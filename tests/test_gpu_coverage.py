"""Coverage mode of the mask kernel (csrc/swb_masks.cuh, swb_render_coverage) against the CPU
restatement tests/coverage_oracle.py, bit for bit and count for count.

- Every raster of test_gpu_render_geometry.CASES (convex and concave pools, 1 to 32 slots, so bit
  31 too), plus test_gpu_masks.EXTRA and the huge-sprite cases, into sentinel-filled buffers at
  4-byte-aligned offsets that are not 16-byte aligned, whose guard bytes must survive; permuted and
  repeated records against the live result.
- Episodes of a BatchedEnvironment with PILRenderer, SpriteMasks, SpriteCoverage and SpriteFactors
  through auto-resets, with the host and the device scene sampler: the coverage equals the oracle
  on the downloaded state, and its highest bit + 1 is the same step's mask; expand leaves; a
  checkpoint round trip.
- One launch per call and nothing else changes; every refusal enqueues nothing.
- The drop-in Environment on a sprite list.
"""
import collections
import ctypes

import numpy as np
import pytest

from oracle import oracle
from tests import coverage_oracle, mask_oracle
from tests import test_gpu_masks as gm
from tests import test_gpu_render_geometry as geo

gpu = pytest.mark.gpu


def _coverage_guarded(eng, W, H, aa, n, skews=(0, 0, 0), states=None):
  """render_coverage into three guarded int32 buffers `skews` bytes past 16-byte boundaries; checks
  the guards and returns the three as arrays."""
  import torch
  S = eng.n_slots
  sizes = (n * H * W * 4, n * S * 4, n * S * 4)
  bufs = [geo._guarded(nb, eng.device, skew) for nb, skew in zip(sizes, skews)]
  out = [flat.view(torch.int32).view(shape) for (_, flat, _), shape in zip(bufs, ((n, H, W), (n, S), (n, S)))]
  for t in out[1:]:
    t.fill_(-7)                     # the call zeroes the counts itself
  launches = eng.launch_count()
  got = eng.render_coverage(W, H, aa, states=states, out=out)
  assert all(g is o for g, o in zip(got, out)) and eng.launch_count() == launches + 1
  torch.cuda.synchronize()
  for (big, _, lo), nb, name in zip(bufs, sizes, ('cover', 'visible', 'area')):
    geo._assert_guards(big, lo, nb, (W, H, aa, skews, name))
  return tuple(t.cpu().numpy() for t in out)


def _want(sw, W, H, aa):
  rc = oracle.raster_cfg(W, H, aa)
  got = [coverage_oracle.render_coverage(rc, sw.tab, sw.rec[e]) for e in range(sw.E)]
  return tuple(np.stack(x) for x in zip(*got))


def _check_sweep(sw, W, H, aa, skews=((0, 0, 0), (4, 8, 12))):
  import torch
  want = _want(sw, W, H, aa)
  # the restatement's own invariants, and the mask restatement
  rc = oracle.raster_cfg(W, H, aa)
  for e in range(sw.E):
    assert np.array_equal(coverage_oracle.modal(want[0][e]), mask_oracle.render_masks(rc, sw.tab, sw.rec[e]))
  assert (want[1] <= want[2]).all()
  for skew in skews:
    got = _coverage_guarded(sw.eng, W, H, aa, sw.E, skew)
    for name, g, w in zip(('cover', 'visible', 'area'), got, want):
      bad = np.argwhere(g != w)
      assert not len(bad), (W, H, aa, skew, name, len(bad), bad[:4].tolist())
  # records, permuted and repeated, give the coverage of the envs they were saved from
  perm = torch.from_numpy(np.random.RandomState(sw.E).randint(0, sw.E, sw.E + 3)).to(sw.eng.device)
  states = sw.eng.save_envs().take(perm)
  got = _coverage_guarded(sw.eng, W, H, aa, len(states), (12, 4, 8), states=states)
  p = perm.cpu().numpy()
  for name, g, w in zip(('cover', 'visible', 'area'), got, want):
    assert np.array_equal(g, w[p]), (W, H, aa, 'records', name)
  return want


@gpu
@pytest.mark.parametrize('case', geo.CASES, ids=[c[0] for c in geo.CASES])
def test_coverage_sweep(case):
  sw = geo.Sweep(case, geo._n_sms())
  try:
    want = _check_sweep(sw, sw.W, sw.H, sw.aa)
    if sw.S == 32:
      assert (want[2][:, 31] > 0).any()   # bit 31, the sign bit, is exercised
  finally:
    sw.close()


@gpu
@pytest.mark.parametrize('extra', gm.EXTRA, ids=[c[0] for c in gm.EXTRA])
def test_coverage_on_tall_and_4095_canvases(extra):
  cid, W, H, aa, S, E, concave = extra
  sw = geo.Sweep((cid, W, H, aa, (0, 0, 0), S, E, concave, 'edges'), geo._n_sms())
  try:
    _check_sweep(sw, W, H, aa, skews=((0, 0, 0), (8, 12, 4)))
  finally:
    sw.close()


@gpu
@pytest.mark.parametrize('huge', gm.HUGE, ids=[c[0] for c in gm.HUGE])
def test_coverage_of_sprites_with_edges_beyond_int16_rows(huge):
  cid, W, H, aa, S, E = huge
  arrs = mask_oracle.huge_scene_arrays(np.random.RandomState(len(cid) + S), E, S, aa * H)
  sw = geo.Sweep((cid, W, H, aa, (0, 0, 0), S, E, True, 'edges'), geo._n_sms(), arrs=arrs)
  try:
    rc = oracle.raster_cfg(W, H, aa)
    assert max(abs(mask_oracle.canvas_vertices(rc, sw.tab, r)[:, 1]).max() for r in sw.rec[0]) > 40000
    _check_sweep(sw, W, H, aa, skews=((0, 0, 0), (4, 4, 4)))
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
      ('fine', renderers.SpriteCoverage(image_size=(40, 40), anti_aliasing=5)),
      ('factors', renderers.SpriteFactors())])
  kw = dict(refill='sync') if sampler == 'host' else dict(sampler='device', seed=seed)
  return environment.BatchedEnvironment(n_envs=E, pool_depth=5, rng=np.random.RandomState(seed), **kw, **cfg)


def _oracle_coverage(env, renderer, states):
  rc = oracle.raster_cfg(renderer.width, renderer.height, renderer.anti_aliasing)
  got = [coverage_oracle.render_coverage(rc, gm._tab(), sp) for sp in gm._sprites_of(env.engine, states)]
  return tuple(np.stack(x) for x in zip(*got))


def _assert_coverage(obs, want, what):
  assert list(obs) == ['cover', 'visible', 'area'], what
  for k, w in zip(obs, want):
    assert np.array_equal(obs[k].cpu().numpy(), w), (what, k)


@gpu
@pytest.mark.parametrize('sampler', ['host', 'device'])
def test_episodes_coverage_equals_the_oracle_and_the_masks(sampler):
  env = _env(sampler=sampler)
  rng = np.random.RandomState(1)
  ts = env.reset()
  buffers = [t.data_ptr() for t in ts.observation['cover'].values()]
  lasts = 0
  for t in range(14):
    if t:
      ts = env.step(rng.uniform(0, 1, (env.n_envs, 4)).astype(np.float32))
    lasts += int((ts.step_type.cpu().numpy() == 2).sum())
    states = env.save_envs()
    for name in ('cover', 'fine'):
      _assert_coverage(ts.observation[name], _oracle_coverage(env, env._renderers[name], states), (t, name))
    assert [v.data_ptr() for v in ts.observation['cover'].values()] == buffers
    cover = ts.observation['cover']['cover'].cpu().numpy()
    m = ts.observation['masks'].cpu().numpy()
    assert np.array_equal(coverage_oracle.modal(cover), m), t
    area = ts.observation['cover']['area'].cpu().numpy()
    occupied = ts.observation['factors']['mask'].cpu().numpy()
    assert (area[~occupied] == 0).all(), t
  assert lasts > env.n_envs   # the run went through auto-resets
  env.close()


@gpu
def test_coverage_of_leaves_and_after_a_checkpoint():
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
  _assert_coverage(obs['fine'], _oracle_coverage(env, env._renderers['fine'], pick), 'leaves')
  sd = env.state_dict()
  saved = {k: {f: v.clone() for f, v in env.render()[k].items()} for k in ('cover', 'fine')}
  env.load_envs(pick)
  out = env.render()
  for k in ('cover', 'fine'):
    for f in ('cover', 'visible', 'area'):
      assert torch.equal(obs[k][f], out[k][f]), (k, f)
  env.load_state_dict(sd)
  out = env.render()
  for k in ('cover', 'fine'):
    for f in ('cover', 'visible', 'area'):
      assert torch.equal(out[k][f], saved[k][f]), (k, f)
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
  status = eng.render_status().clone()
  rng_state = env._rng.get_state()
  own = env._coverage_buffers[id(env._renderers['cover'])]
  launches = eng.launch_count()
  c = eng.render_coverage(32, 24, 1)
  assert eng.launch_count() == launches + 1
  r = eng.render_coverage(20, 30, 7, states=states)
  assert eng.launch_count() == launches + 2 and [tuple(t.shape) for t in r] == [(16, 30, 20), (16, eng.n_slots),
                                                                                (16, eng.n_slots)]
  obs = env.render_coverage(env._renderers['cover'])
  assert eng.launch_count() == launches + 3
  assert [v.data_ptr() for v in obs.values()] == [t.data_ptr() for t in own]
  assert torch.equal(eng.save_state(), saved)
  assert torch.equal(env._frames['image'], frames) and torch.equal(eng.render_status(), status)
  assert torch.equal(env._mask_buffers[id(env._renderers['masks'])], masks)
  assert all(np.array_equal(a, b) for a, b in zip(env._rng.get_state()[1:], rng_state[1:]))
  for a, b in zip(c, own):
    assert torch.equal(a, b)
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
  nc, nv = n * H * W * 4, n * S * 4
  big, flat, lo = geo._guarded(nc + 2 * nv + 64, eng.device)
  base = flat.data_ptr()
  cp, vp, ap = (ctypes.c_void_p(base), ctypes.c_void_p(base + nc), ctypes.c_void_p(base + nc + nv))
  rp, rb = ctypes.c_void_p(states.data.data_ptr()), states.data.numel()
  stream = eng._stream()
  odd = ctypes.c_void_p(states.data.data_ptr() + 8)

  def at(off):
    return ctypes.c_void_p(base + off)
  cases = [
      ('null', (None, W, H, 1, None, n, 0, cp, vp, ap)),
      ('null', (eng._h, W, H, 1, None, n, 0, None, vp, ap)),
      ('null', (eng._h, W, H, 1, None, n, 0, cp, None, ap)),
      ('null', (eng._h, W, H, 1, None, n, 0, cp, vp, None)),
      ('must be >= 1', (eng._h, 0, H, 1, None, n, 0, cp, vp, ap)),
      ('must be >= 1', (eng._h, W, -1, 1, None, n, 0, cp, vp, ap)),
      ('must be >= 1', (eng._h, W, H, 0, None, n, 0, cp, vp, ap)),
      ('4095', (eng._h, 4096, 1, 1, None, n, 0, cp, vp, ap)),
      ('4095', (eng._h, 1, 820, 5, None, n, 0, cp, vp, ap)),
      ('n = -1', (eng._h, W, H, 1, rp, -1, rb, cp, vp, ap)),
      ('must be E', (eng._h, W, H, 1, None, n - 1, 0, cp, vp, ap)),
      ('must be E', (eng._h, W, H, 1, None, 0, 0, cp, vp, ap)),
      ('16-byte aligned', (eng._h, W, H, 1, odd, 2, rb, cp, vp, ap)),
      ('bytes', (eng._h, W, H, 1, rp, n, rb - 16, cp, vp, ap)),
      ('cover is not 4-byte aligned', (eng._h, W, H, 1, None, n, 0, at(2), vp, ap)),
      ('visible is not 4-byte aligned', (eng._h, W, H, 1, None, n, 0, cp, at(nc + 1), ap)),
      ('area is not 4-byte aligned', (eng._h, W, H, 1, None, n, 0, cp, vp, at(nc + nv + 3))),
      ('visible overlaps cover', (eng._h, W, H, 1, None, n, 0, cp, at(nc - 4), ap)),
      ('area overlaps cover', (eng._h, W, H, 1, None, n, 0, cp, vp, at(16))),
      ('area overlaps visible', (eng._h, W, H, 1, None, n, 0, cp, vp, at(nc + nv - 4))),
      ('area overlaps visible', (eng._h, W, H, 1, None, n, 0, cp, vp, vp)),
      ('cover overlaps the records', (eng._h, W, H, 1, rp, n, rb, ctypes.c_void_p(states.data.data_ptr() + 32),
                                      vp, ap)),
      ('visible overlaps the records', (eng._h, W, H, 1, rp, n, rb, cp, rp, ap)),
      ('area overlaps the records', (eng._h, W, H, 1, rp, n, rb, cp, vp,
                                     ctypes.c_void_p(states.data.data_ptr() + rb - 4))),
  ]
  launches = eng.launch_count()
  for msg, args in cases:
    assert L.swb_render_coverage(*args, stream) != 0, msg
    assert msg.encode() in L.swb_last_error(), (msg, L.swb_last_error())
    assert eng.launch_count() == launches, msg
  # a grid the launch cannot express, checked before any buffer is read: a band of coverage holds
  # 16 KiB, so 4000-pixel-wide rows are one band each and 2^30 records of 300 rows exceed 2^31 - 1 CTAs
  big_n = (1 << 30)
  assert L.swb_render_coverage(eng._h, 4000, 300, 1, rp, big_n, big_n * states.record_bytes, cp, vp, ap,
                               stream) != 0
  assert b'2^31' in L.swb_last_error()
  torch.cuda.synchronize()
  assert bool((flat == geo.SENTINEL).all()) and bool((big == geo.SENTINEL).all())
  assert eng.launch_count() == launches
  # through Python: NativeError (or ValueError before the call), nothing enqueued
  with pytest.raises(_native.NativeError, match='4095'):
    eng.render_coverage(2048, 8, 2)
  c = torch.zeros((n, H, W), dtype=torch.int32, device=eng.device)
  v = torch.zeros((n, S), dtype=torch.int32, device=eng.device)
  with pytest.raises(_native.NativeError, match='area overlaps visible'):
    eng.render_coverage(W, H, 1, out=(c, v, v))
  with pytest.raises(ValueError, match='states must be EnvStates'):
    eng.render_coverage(W, H, 1, states=torch.zeros(4))
  # zero records are checked as any other call, and draw nothing
  empty = states.take(torch.zeros(0, dtype=torch.int64, device=eng.device))
  with pytest.raises(_native.NativeError, match='4095'):
    eng.render_coverage(2048, 8, 2, states=empty)
  with pytest.raises(_native.NativeError, match='must be >= 1'):
    eng.render_coverage(16, 8, 0, states=empty)
  got = eng.render_coverage(16, 8, 3, states=empty)
  assert [tuple(t.shape) for t in got] == [(0, 8, 16), (0, S), (0, S)]
  assert eng.launch_count() == launches
  env.close()


@gpu
def test_drop_in_environment_coverage_equals_the_oracle_of_its_sprite_list():
  from spriteworld_b200 import environment, renderers
  from spriteworld_b200.configs.cobra import goal_finding_more_targets as cfgmod
  from tests import fixtures
  cfg = cfgmod.get_config('train')
  cfg['renderers'] = collections.OrderedDict([
      ('cover', renderers.SpriteCoverage(image_size=(24, 16), anti_aliasing=3)),
      ('masks', renderers.SpriteMasks(image_size=(24, 16), anti_aliasing=3))])
  env = environment.Environment(**cfg)
  rng = np.random.RandomState(4)
  tab = gm._tab()
  ts = env.reset()
  for t in range(8):
    if t:
      ts = env.step(rng.uniform(0, 1, 4))
    sprites = env.state()['sprites']
    got = ts.observation['cover']
    assert got['cover'].shape == (16, 24) and got['cover'].dtype == np.int32
    n = len(sprites)
    arrs = dict(x=np.array([s.x for s in sprites]), y=np.array([s.y for s in sprites]),
                shape=np.array([oracle.SHAPE_IDS[s.shape] for s in sprites]),
                angle=np.array([s.angle for s in sprites]), scale=np.array([s.scale for s in sprites]),
                vx=np.zeros(n), vy=np.zeros(n), member=np.zeros(n, np.uint32), pos_f32=np.zeros(n, np.uint8),
                rgb=np.zeros((n, 3), np.uint8))
    want = coverage_oracle.render_coverage(oracle.raster_cfg(24, 16, 3), tab, fixtures.records_from_arrays(arrs))
    for k, w in zip(('cover', 'visible', 'area'), want):
      assert np.array_equal(got[k], w), (t, k)
    assert np.array_equal(coverage_oracle.modal(got['cover']), ts.observation['masks']), t
  env.close()
