"""Soft mode of the mask kernel (csrc/swb_masks.cuh, swb_render_soft_masks) against the CPU
restatement tests/soft_mask_oracle.py, count for count.

- Every raster of test_gpu_render_geometry.CASES (convex and concave pools, 1 to 32 slots), plus
  test_gpu_masks.EXTRA and the huge-sprite cases with anti_aliasing <= 15 (w273h15a15 at 32 slots,
  w4095h1a1), into sentinel-filled buffers at byte offsets that are not 16-byte aligned, whose guard
  bytes must survive; permuted and repeated records against the live result.  The aa = 20 cases
  are refused, with nothing launched.
- Episodes of a BatchedEnvironment with PILRenderer, SpriteMasks, SpriteCoverage, SoftSpriteMasks
  and SpriteFactors through auto-resets, with the host and the device scene sampler: the soft masks
  equal the oracle on the downloaded state and keep their properties against the same step's mask;
  expand leaves; a checkpoint round trip.
- One launch per call and nothing else changes; every refusal enqueues nothing.
- The drop-in Environment on a sprite list.
"""
import collections
import ctypes

import numpy as np
import pytest

from oracle import oracle
from tests import mask_oracle, soft_mask_oracle
from tests import test_gpu_masks as gm
from tests import test_gpu_render_geometry as geo

gpu = pytest.mark.gpu


def _soft_guarded(eng, W, H, aa, n, skew=0, states=None):
  """render_soft_masks into a guarded uint8 buffer `skew` bytes past a 16-byte boundary; checks the
  guards and returns the result as an array."""
  import torch
  S = eng.n_slots
  nb = n * S * H * W
  big, flat, lo = geo._guarded(nb, eng.device, skew)
  out = flat.view(n, S, H, W)
  launches = eng.launch_count()
  assert eng.render_soft_masks(W, H, aa, states=states, out=out) is out
  assert eng.launch_count() == launches + 1
  torch.cuda.synchronize()
  geo._assert_guards(big, lo, nb, (W, H, aa, skew))
  return out.cpu().numpy()


def _want(sw, W, H, aa):
  rc = oracle.raster_cfg(W, H, aa)
  return np.stack([soft_mask_oracle.render_soft_masks(rc, sw.tab, sw.rec[e]) for e in range(sw.E)])


def _check_sweep(sw, W, H, aa, skews=(0, 7)):
  import torch
  want = _want(sw, W, H, aa)
  rc = oracle.raster_cfg(W, H, aa)
  for e in range(sw.E):
    soft_mask_oracle.check_properties(want[e], mask_oracle.render_masks(rc, sw.tab, sw.rec[e]), aa, e)
  for skew in skews:
    got = _soft_guarded(sw.eng, W, H, aa, sw.E, skew)
    bad = np.argwhere(got != want)
    assert not len(bad), (W, H, aa, skew, len(bad), bad[:4].tolist())
  # records, permuted and repeated, give the soft masks of the envs they were saved from
  perm = torch.from_numpy(np.random.RandomState(sw.E).randint(0, sw.E, sw.E + 3)).to(sw.eng.device)
  states = sw.eng.save_envs().take(perm)
  got = _soft_guarded(sw.eng, W, H, aa, len(states), 13, states=states)
  assert np.array_equal(got, want[perm.cpu().numpy()]), (W, H, aa, 'records')
  return want


def _refused(sw, W, H, aa):
  """aa > 15: refused before anything is enqueued, the buffer untouched."""
  import torch
  from spriteworld_b200 import _native
  eng = sw.eng
  big, flat, lo = geo._guarded(sw.E * eng.n_slots * H * W, eng.device, 5)
  launches = eng.launch_count()
  with pytest.raises(_native.NativeError, match='exceeds 15'):
    eng.render_soft_masks(W, H, aa, out=flat.view(sw.E, eng.n_slots, H, W))
  torch.cuda.synchronize()
  assert eng.launch_count() == launches and bool((big == geo.SENTINEL).all())


@gpu
@pytest.mark.parametrize('case', geo.CASES, ids=[c[0] for c in geo.CASES])
def test_soft_masks_sweep(case):
  sw = geo.Sweep(case, geo._n_sms())
  try:
    want = _check_sweep(sw, sw.W, sw.H, sw.aa)
    if sw.S == 32:
      assert want[:, 31].any()
  finally:
    sw.close()


@gpu
@pytest.mark.parametrize('extra', gm.EXTRA, ids=[c[0] for c in gm.EXTRA])
def test_soft_masks_on_tall_and_4095_canvases(extra):
  cid, W, H, aa, S, E, concave = extra
  sw = geo.Sweep((cid, W, H, aa, (0, 0, 0), S, E, concave, 'edges'), geo._n_sms())
  try:
    if aa > 15:
      _refused(sw, W, H, aa)
    else:
      _check_sweep(sw, W, H, aa, skews=(0, 11))
  finally:
    sw.close()


@gpu
@pytest.mark.parametrize('huge', gm.HUGE, ids=[c[0] for c in gm.HUGE])
def test_soft_masks_of_sprites_with_edges_beyond_int16_rows(huge):
  cid, W, H, aa, S, E = huge
  arrs = mask_oracle.huge_scene_arrays(np.random.RandomState(len(cid) + S), E, S, aa * H)
  sw = geo.Sweep((cid, W, H, aa, (0, 0, 0), S, E, True, 'edges'), geo._n_sms(), arrs=arrs)
  try:
    rc = oracle.raster_cfg(W, H, aa)
    assert max(abs(mask_oracle.canvas_vertices(rc, sw.tab, r)[:, 1]).max() for r in sw.rec[0]) > 40000
    if aa > 15:
      _refused(sw, W, H, aa)
    else:
      _check_sweep(sw, W, H, aa, skews=(0, 3))
  finally:
    sw.close()


def _env(E=48, seed=3, max_episode_length=5, sampler='host'):
  from spriteworld_b200 import action_spaces, environment, renderers
  from spriteworld_b200.configs.cobra import goal_finding_more_targets as cfgmod
  cfg = cfgmod.get_config('train')
  cfg['max_episode_length'] = max_episode_length
  cfg['action_space'] = action_spaces.SelectMove(scale=0.25)
  hsv = renderers.color_maps.hsv_to_rgb
  cfg['renderers'] = collections.OrderedDict([
      ('image', renderers.PILRenderer(image_size=(32, 24), anti_aliasing=1, bg_color=(9, 20, 30),
                                      color_to_rgb=hsv)),
      ('masks', renderers.SpriteMasks(image_size=(32, 24), anti_aliasing=1)),
      ('cover', renderers.SpriteCoverage(image_size=(32, 24), anti_aliasing=1)),
      ('soft', renderers.SoftSpriteMasks(image_size=(32, 24), anti_aliasing=1)),
      ('masks5', renderers.SpriteMasks(image_size=(40, 40), anti_aliasing=5)),
      ('soft5', renderers.SoftSpriteMasks(image_size=(40, 40), anti_aliasing=5)),
      ('factors', renderers.SpriteFactors())])
  kw = dict(refill='sync') if sampler == 'host' else dict(sampler='device', seed=seed)
  return environment.BatchedEnvironment(n_envs=E, pool_depth=5, rng=np.random.RandomState(seed), **kw, **cfg)


def _oracle_soft(env, renderer, states):
  rc = oracle.raster_cfg(renderer.width, renderer.height, renderer.anti_aliasing)
  return np.stack([soft_mask_oracle.render_soft_masks(rc, gm._tab(), sp) for sp in gm._sprites_of(env.engine, states)])


@gpu
@pytest.mark.parametrize('sampler', ['host', 'device'])
def test_episodes_soft_masks_equal_the_oracle_and_keep_their_properties(sampler):
  env = _env(sampler=sampler)
  rng = np.random.RandomState(1)
  ts = env.reset()
  buffers = {k: ts.observation[k].data_ptr() for k in ('soft', 'soft5')}
  lasts = 0
  for t in range(14):
    if t:
      ts = env.step(rng.uniform(0, 1, (env.n_envs, 4)).astype(np.float32))
    lasts += int((ts.step_type.cpu().numpy() == 2).sum())
    states = env.save_envs()
    obs = {k: v.cpu().numpy() if hasattr(v, 'cpu') else v for k, v in ts.observation.items()}
    for name, masks, aa in (('soft', 'masks', 1), ('soft5', 'masks5', 5)):
      assert ts.observation[name].data_ptr() == buffers[name], (t, name)
      want = _oracle_soft(env, env._renderers[name], states)
      assert np.array_equal(obs[name], want), (t, name, int((obs[name] != want).sum()))
      for e in range(env.n_envs):
        soft_mask_oracle.check_properties(obs[name][e], obs[masks][e], aa, (t, name, e))
    # slot k's count is the coverage's visible count at aa 1, and the factors' slots hold them
    visible = ts.observation['cover']['visible'].cpu().numpy()
    assert np.array_equal(obs['soft'].astype(np.int64).sum((2, 3)), visible), t
    occupied = ts.observation['factors']['mask'].cpu().numpy()
    assert not obs['soft5'][~occupied].any(), t
  assert lasts > env.n_envs   # the run went through auto-resets
  env.close()


@gpu
def test_soft_masks_of_leaves_and_after_a_checkpoint():
  import torch
  env = _env(E=32, seed=5, max_episode_length=20)
  rng = np.random.RandomState(2)
  env.reset()
  for _ in range(3):
    env.step(rng.uniform(0, 1, (env.n_envs, 4)).astype(np.float32))
  T, C = 3, 2
  plans = rng.uniform(0, 1, (T, env.n_envs, C, 4)).astype(np.float32)
  _, leaves = env.expand(plans)
  pick = leaves.take(torch.arange(0, 2 * env.n_envs, 2, device=env.engine.device))
  obs, _ = env.observe(pick)
  assert np.array_equal(obs['soft5'].cpu().numpy(), _oracle_soft(env, env._renderers['soft5'], pick))
  sd = env.state_dict()
  saved = {k: env.render()[k].clone() for k in ('soft', 'soft5')}
  env.load_envs(pick)
  out = env.render()
  for k in ('soft', 'soft5'):
    assert torch.equal(obs[k], out[k]), k
  env.load_state_dict(sd)
  out = env.render()
  for k in ('soft', 'soft5'):
    assert torch.equal(out[k], saved[k]), k
  env.close()


@gpu
def test_one_launch_per_call_and_nothing_else_changes():
  import torch
  env = _env(E=16)
  rng = np.random.RandomState(3)
  env.reset()
  env.step(rng.uniform(0, 1, (env.n_envs, 4)).astype(np.float32))
  eng = env.engine
  states = env.save_envs()
  saved = eng.save_state()
  frames = env._frames['image'].clone()
  masks = env._mask_buffers[id(env._renderers['masks'])].clone()
  cover = [t.clone() for t in env._coverage_buffers[id(env._renderers['cover'])]]
  status = eng.render_status().clone()
  rng_state = env._rng.get_state()
  own = env._soft_buffers[id(env._renderers['soft5'])]
  launches = eng.launch_count()
  s = eng.render_soft_masks(40, 40, 5)
  assert eng.launch_count() == launches + 1
  r = eng.render_soft_masks(20, 30, 7, states=states)
  assert eng.launch_count() == launches + 2 and tuple(r.shape) == (16, eng.n_slots, 30, 20)
  obs = env.render_soft_masks(env._renderers['soft5'])
  assert eng.launch_count() == launches + 3 and obs.data_ptr() == own.data_ptr()
  assert torch.equal(eng.save_state(), saved)
  assert torch.equal(env._frames['image'], frames) and torch.equal(eng.render_status(), status)
  assert torch.equal(env._mask_buffers[id(env._renderers['masks'])], masks)
  assert all(torch.equal(a, b) for a, b in zip(env._coverage_buffers[id(env._renderers['cover'])], cover))
  assert all(np.array_equal(a, b) for a, b in zip(env._rng.get_state()[1:], rng_state[1:]))
  assert torch.equal(s, own)
  env.close()


@gpu
def test_refused_calls_enqueue_nothing():
  import torch
  from spriteworld_b200 import _native
  env = _env(E=8)
  env.reset()
  eng = env.engine
  L = eng._lib
  states = env.save_envs()
  torch.cuda.synchronize()
  n, W, H, S = 8, 16, 8, eng.n_slots
  big, flat, lo = geo._guarded(n * S * H * W + 64, eng.device)
  sp = ctypes.c_void_p(flat.data_ptr() + 3)
  rp, rb = ctypes.c_void_p(states.data.data_ptr()), states.data.numel()
  stream = eng._stream()
  odd = ctypes.c_void_p(states.data.data_ptr() + 8)
  cases = [
      ('null', (None, W, H, 1, None, n, 0, sp)),
      ('null output soft', (eng._h, W, H, 1, None, n, 0, None)),
      ('must be >= 1', (eng._h, 0, H, 1, None, n, 0, sp)),
      ('must be >= 1', (eng._h, W, -1, 1, None, n, 0, sp)),
      ('must be >= 1', (eng._h, W, H, 0, None, n, 0, sp)),
      ('exceeds 15', (eng._h, W, H, 16, None, n, 0, sp)),
      ('exceeds 15', (eng._h, 1, 1, 20, None, n, 0, sp)),
      ('4095', (eng._h, 4096, 1, 1, None, n, 0, sp)),
      ('4095', (eng._h, 1, 274, 15, None, n, 0, sp)),
      ('n = -1', (eng._h, W, H, 1, rp, -1, rb, sp)),
      ('must be E', (eng._h, W, H, 1, None, n - 1, 0, sp)),
      ('must be E', (eng._h, W, H, 1, None, 0, 0, sp)),
      ('16-byte aligned', (eng._h, W, H, 1, odd, 2, rb, sp)),
      ('bytes', (eng._h, W, H, 1, rp, n, rb - 16, sp)),
      ('soft overlaps the records', (eng._h, W, H, 1, rp, n, rb, ctypes.c_void_p(states.data.data_ptr() + 32))),
      ('soft overlaps the records', (eng._h, W, H, 1, rp, n, rb, ctypes.c_void_p(states.data.data_ptr() - 5))),
  ]
  launches = eng.launch_count()
  for msg, args in cases:
    assert L.swb_render_soft_masks(*args, stream) != 0, msg
    assert msg.encode() in L.swb_last_error(), (msg, L.swb_last_error())
    assert eng.launch_count() == launches, msg
  # a grid the launch cannot express, checked before any buffer is read: 4000-pixel-wide rows at
  # aa 1 stage 8 mask rows per band, so 2^30 records of 300 rows exceed 2^31 - 1 CTAs
  big_n = 1 << 30
  assert L.swb_render_soft_masks(eng._h, 4000, 300, 1, rp, big_n, big_n * states.record_bytes, sp, stream) != 0
  assert b'2^31' in L.swb_last_error()
  torch.cuda.synchronize()
  assert bool((big == geo.SENTINEL).all())
  assert eng.launch_count() == launches
  # through Python: NativeError (or ValueError before the call), nothing enqueued
  with pytest.raises(_native.NativeError, match='exceeds 15'):
    eng.render_soft_masks(W, H, 16)
  with pytest.raises(_native.NativeError, match='4095'):
    eng.render_soft_masks(2048, 8, 2)
  with pytest.raises(ValueError, match='soft'):
    eng.render_soft_masks(W, H, 1, out=torch.zeros((n, S, W, H), dtype=torch.uint8, device=eng.device))
  with pytest.raises(ValueError, match='states must be EnvStates'):
    eng.render_soft_masks(W, H, 1, states=torch.zeros(4))
  # zero records are checked as any other call, and draw nothing
  empty = states.take(torch.zeros(0, dtype=torch.int64, device=eng.device))
  with pytest.raises(_native.NativeError, match='exceeds 15'):
    eng.render_soft_masks(16, 8, 16, states=empty)
  with pytest.raises(_native.NativeError, match='must be >= 1'):
    eng.render_soft_masks(16, 8, 0, states=empty)
  assert tuple(eng.render_soft_masks(16, 8, 3, states=empty).shape) == (0, S, 8, 16)
  assert eng.launch_count() == launches
  env.close()


@gpu
def test_drop_in_environment_soft_masks_equal_the_oracle_of_its_sprite_list():
  from spriteworld_b200 import environment, renderers
  from spriteworld_b200.configs.cobra import goal_finding_more_targets as cfgmod
  from tests import fixtures
  cfg = cfgmod.get_config('train')
  cfg['renderers'] = collections.OrderedDict([
      ('soft', renderers.SoftSpriteMasks(image_size=(24, 16), anti_aliasing=5)),
      ('masks', renderers.SpriteMasks(image_size=(24, 16), anti_aliasing=5))])
  env = environment.Environment(**cfg)
  rng = np.random.RandomState(4)
  tab = gm._tab()
  ts = env.reset()
  for t in range(8):
    if t:
      ts = env.step(rng.uniform(0, 1, 4))
    sprites = env.state()['sprites']
    got = ts.observation['soft']
    n = len(sprites)
    assert got.shape == (n, 16, 24) and got.dtype == np.uint8
    arrs = dict(x=np.array([s.x for s in sprites]), y=np.array([s.y for s in sprites]),
                shape=np.array([oracle.SHAPE_IDS[s.shape] for s in sprites]),
                angle=np.array([s.angle for s in sprites]), scale=np.array([s.scale for s in sprites]),
                vx=np.zeros(n), vy=np.zeros(n), member=np.zeros(n, np.uint32), pos_f32=np.zeros(n, np.uint8),
                rgb=np.zeros((n, 3), np.uint8))
    want = soft_mask_oracle.render_soft_masks(oracle.raster_cfg(24, 16, 5), tab, fixtures.records_from_arrays(arrs))
    assert np.array_equal(got, want), t
    soft_mask_oracle.check_properties(got, ts.observation['masks'], 5, t)
  env.close()
