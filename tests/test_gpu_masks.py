"""Mask kernel (csrc/swb_masks.cuh, swb_render_masks) against the CPU restatement
tests/mask_oracle.py, bit for bit.

- Every raster of test_gpu_render_geometry.CASES (convex and concave pools, 1 to 32 slots, the
  canvas-side limit, the tall rasters the render kernel refuses), plus anti_aliasing >= 14 on tall
  masks and 4095-pixel canvases, into sentinel-filled buffers whose guard bytes must survive, at
  aligned and odd addresses; permuted records against the live masks.
- Episodes of a BatchedEnvironment with PILRenderer, SpriteMasks and SpriteFactors through
  auto-resets, against the oracle on the downloaded state, with frames = bg / rgb[mask - 1] at
  anti_aliasing 1; expand leaves; a checkpoint round trip.
- One launch per call and nothing else changes; every refusal enqueues nothing.
- The drop-in Environment.
"""
import collections
import ctypes

import numpy as np
import pytest

from oracle import oracle
from tests import mask_oracle
from tests import test_gpu_render_geometry as geo
from tests.oracle_engine import record_sprites as _sprites_of

gpu = pytest.mark.gpu

# (id, W, H, aa, S, E, concave): masks beyond what PILRenderer accepts
EXTRA = [
    ('w10h292a14', 10, 292, 14, 8, 4, True),      # canvas 140 x 4088
    ('w3h204a20', 3, 204, 20, 5, 4, False),       # canvas 60 x 4080
    ('w1h4095a1', 1, 4095, 1, 3, 3, True),
    ('w4095h1a1', 4095, 1, 1, 9, 3, True),
    ('w273h15a15', 273, 15, 15, 32, 2, True),     # canvas 4095 x 225
    ('w2h273a15', 2, 273, 15, 6, 3, False),       # canvas 30 x 4095
]


def _masks_guarded(eng, W, H, aa, n, skew=0, states=None):
  import torch
  nbytes = n * H * W
  big, flat, lo = geo._guarded(nbytes, eng.device, skew)
  out = flat.view(n, H, W)
  launches = eng.launch_count()
  got = eng.render_masks(W, H, aa, states=states, out=out)
  assert got is out and eng.launch_count() == launches + 1
  torch.cuda.synchronize()
  geo._assert_guards(big, lo, nbytes, (W, H, aa, skew))
  return out.cpu().numpy()


def _check_sweep(sw, W, H, aa, skews=(0, 3)):
  rc = oracle.raster_cfg(W, H, aa)
  want = np.stack([mask_oracle.render_masks(rc, sw.tab, sw.rec[e]) for e in range(sw.E)])
  for skew in skews:
    got = _masks_guarded(sw.eng, W, H, aa, sw.E, skew)
    bad = np.argwhere(got != want)
    assert not len(bad), (W, H, aa, skew, len(bad), bad[:4].tolist())
  # records, permuted and repeated, give the masks of the envs they were saved from
  import torch
  perm = torch.from_numpy(np.random.RandomState(sw.E).randint(0, sw.E, sw.E + 3)).to(sw.eng.device)
  states = sw.eng.save_envs().take(perm)
  got = _masks_guarded(sw.eng, W, H, aa, len(states), 5, states=states)
  assert np.array_equal(got, want[perm.cpu().numpy()]), (W, H, aa, 'records')


@gpu
@pytest.mark.parametrize('case', geo.CASES, ids=[c[0] for c in geo.CASES])
def test_masks_sweep(case):
  sw = geo.Sweep(case, geo._n_sms())
  try:
    _check_sweep(sw, sw.W, sw.H, sw.aa)
  finally:
    sw.close()


@gpu
@pytest.mark.parametrize('extra', EXTRA, ids=[c[0] for c in EXTRA])
def test_masks_on_tall_and_4095_canvases(extra):
  cid, W, H, aa, S, E, concave = extra
  case = (cid, W, H, aa, (0, 0, 0), S, E, concave, 'edges')
  sw = geo.Sweep(case, geo._n_sms())
  try:
    _check_sweep(sw, W, H, aa, skews=(0, 7))
  finally:
    sw.close()


# (id, W, H, aa, S, E): sprites thousands of canvases large whose outlines cross the canvas, with
# edges wholly beyond +-32768 canvas rows (mask_oracle.huge_scene_arrays)
HUGE = [
    ('huge_w64h819a5', 64, 819, 5, 5, 6),        # canvas 320 x 4095
    ('huge_w16h16a20', 16, 16, 20, 3, 8),
    ('huge_w101h30a2', 101, 30, 2, 32, 4),
]


@gpu
@pytest.mark.parametrize('huge', HUGE, ids=[c[0] for c in HUGE])
def test_masks_of_sprites_with_edges_beyond_int16_rows(huge):
  cid, W, H, aa, S, E = huge
  arrs = mask_oracle.huge_scene_arrays(np.random.RandomState(len(cid) + S), E, S, aa * H)
  sw = geo.Sweep((cid, W, H, aa, (0, 0, 0), S, E, True, 'edges'), geo._n_sms(), arrs=arrs)
  try:
    rc = oracle.raster_cfg(W, H, aa)
    assert max(abs(mask_oracle.canvas_vertices(rc, sw.tab, r)[:, 1]).max() for r in sw.rec[0]) > 40000
    assert sum(len(np.unique(mask_oracle.render_masks(rc, sw.tab, sw.rec[e]))) > 1 for e in range(E)) >= E // 2
    _check_sweep(sw, W, H, aa, skews=(0, 9))
  finally:
    sw.close()


def _env(E=48, seed=3, max_episode_length=5):
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
      ('fine', renderers.SpriteMasks(image_size=(40, 40), anti_aliasing=5)),
      ('factors', renderers.SpriteFactors())])
  return environment.BatchedEnvironment(n_envs=E, pool_depth=5, rng=np.random.RandomState(seed),
                                        refill='sync', **cfg)


def _tab():
  from spriteworld_b200 import constants
  return oracle.shape_table(constants.SHAPES)


def _oracle_masks(env, renderer, states):
  rc = oracle.raster_cfg(renderer.width, renderer.height, renderer.anti_aliasing)
  tab = _tab()
  return np.stack([mask_oracle.render_masks(rc, tab, sp) for sp in _sprites_of(env.engine, states)])


@gpu
def test_episodes_masks_equal_the_oracle_and_name_the_frame_colours():
  env = _env()
  rng = np.random.RandomState(1)
  ts = env.reset()
  lasts = 0
  for t in range(14):
    if t:
      ts = env.step(rng.uniform(0, 1, (env.n_envs, 4)).astype(np.float32))
    lasts += int((ts.step_type.cpu().numpy() == 2).sum())
    states = env.save_envs()
    for name in ('masks', 'fine'):
      got = ts.observation[name].cpu().numpy()
      assert np.array_equal(got, _oracle_masks(env, env._renderers[name], states)), (t, name)
    m = ts.observation['masks'].cpu().numpy()
    frames = ts.observation['image'].cpu().numpy()
    occupied = ts.observation['factors']['mask'].cpu().numpy()
    sprites = _sprites_of(env.engine, states)
    for e in range(env.n_envs):
      colours = np.concatenate([np.array([[9, 20, 30]], np.uint8), sprites[e]['rgb']])
      assert np.array_equal(frames[e], colours[m[e]]), (t, e)
      ids = np.unique(m[e])
      assert occupied[e, ids[ids > 0] - 1].all(), (t, e)
  assert lasts > env.n_envs   # the run went through auto-resets
  env.close()


@gpu
def test_masks_of_leaves_and_after_a_checkpoint():
  import torch
  env = _env(E=32, seed=5, max_episode_length=20)
  rng = np.random.RandomState(2)
  env.reset()
  for _ in range(3):
    env.step(rng.uniform(0, 1, (env.n_envs, 4)).astype(np.float32))
  # leaves of expand: their masks equal those after load_envs(leaves)
  T, C = 3, 2
  plans = rng.uniform(0, 1, (T, env.n_envs, C, 4)).astype(np.float32)
  _, leaves = env.expand(plans)
  pick = leaves.take(torch.arange(0, 2 * env.n_envs, 2, device=env.engine.device))
  obs, _ = env.observe(pick)
  sd = env.state_dict()
  saved = {k: env.render()[k].clone() for k in ('masks', 'fine')}
  env.load_envs(pick)
  out = env.render()
  for k in ('masks', 'fine'):
    assert torch.equal(obs[k], out[k]), k
  # the checkpoint: masks after load_state_dict equal the saved run's
  env.load_state_dict(sd)
  out = env.render()
  for k in ('masks', 'fine'):
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
  status = eng.render_status().clone()
  launches = eng.launch_count()
  m = eng.render_masks(32, 24, 1)
  assert eng.launch_count() == launches + 1
  r = eng.render_masks(20, 30, 7, states=states)
  assert eng.launch_count() == launches + 2 and tuple(r.shape) == (16, 30, 20)
  assert torch.equal(eng.save_state(), saved)
  assert torch.equal(env._frames['image'], frames) and torch.equal(eng.render_status(), status)
  assert torch.equal(m, env._mask_buffers[id(env._renderers['masks'])])
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
  n, W, H = 8, 16, 8
  big, flat, lo = geo._guarded(n * H * W + 64, eng.device)
  mp = ctypes.c_void_p(flat.data_ptr())
  rp, rb = ctypes.c_void_p(states.data.data_ptr()), states.data.numel()
  stream = eng._stream()
  odd = ctypes.c_void_p(states.data.data_ptr() + 8)
  cases = [
      ('null', (None, W, H, 1, None, n, 0, mp)),
      ('null', (eng._h, W, H, 1, None, n, 0, None)),
      ('must be >= 1', (eng._h, 0, H, 1, None, n, 0, mp)),
      ('must be >= 1', (eng._h, W, -1, 1, None, n, 0, mp)),
      ('must be >= 1', (eng._h, W, H, 0, None, n, 0, mp)),
      ('4095', (eng._h, 4096, 1, 1, None, n, 0, mp)),
      ('4095', (eng._h, 1, 820, 5, None, n, 0, mp)),
      ('n = -1', (eng._h, W, H, 1, rp, -1, rb, mp)),
      ('must be E', (eng._h, W, H, 1, None, n - 1, 0, mp)),
      ('must be E', (eng._h, W, H, 1, None, 0, 0, mp)),
      ('16-byte aligned', (eng._h, W, H, 1, odd, 2, rb, mp)),
      ('bytes', (eng._h, W, H, 1, rp, n, rb - 16, mp)),
      ('overlap', (eng._h, W, H, 1, rp, n, rb, ctypes.c_void_p(states.data.data_ptr() + 32))),
  ]
  launches = eng.launch_count()
  for msg, args in cases:
    assert L.swb_render_masks(*args, stream) != 0, msg
    assert msg.encode() in L.swb_last_error(), (msg, L.swb_last_error())
    assert eng.launch_count() == launches, msg
  # a grid the launch cannot express: 2^31 - 1 bands is checked before any buffer is read
  big_n = (1 << 30)
  assert L.swb_render_masks(eng._h, 1, 300, 1, rp, big_n, big_n * states.record_bytes, mp, stream) != 0
  assert b'2^31' in L.swb_last_error()
  torch.cuda.synchronize()
  assert bool((flat == geo.SENTINEL).all()) and bool((big == geo.SENTINEL).all())
  assert eng.launch_count() == launches
  # through Python: NativeError, nothing enqueued
  with pytest.raises(_native.NativeError, match='4095'):
    eng.render_masks(2048, 8, 2)
  # zero records are checked as any other call, and draw nothing
  empty = states.take(torch.zeros(0, dtype=torch.int64, device=eng.device))
  with pytest.raises(_native.NativeError, match='4095'):
    eng.render_masks(2048, 8, 2, states=empty)
  with pytest.raises(_native.NativeError, match='must be >= 1'):
    eng.render_masks(16, 8, 0, states=empty)
  got = eng.render_masks(16, 8, 3, states=empty)
  assert tuple(got.shape) == (0, 8, 16)
  assert eng.launch_count() == launches
  env.close()


@gpu
def test_drop_in_environment_masks_equal_the_oracle_of_its_sprite_list():
  from spriteworld_b200 import environment, renderers
  from spriteworld_b200.configs.cobra import goal_finding_more_targets as cfgmod
  from tests import fixtures
  cfg = cfgmod.get_config('train')
  cfg['renderers'] = collections.OrderedDict([('masks', renderers.SpriteMasks(image_size=(24, 16), anti_aliasing=3))])
  env = environment.Environment(**cfg)
  rng = np.random.RandomState(4)
  tab = _tab()
  ts = env.reset()
  for t in range(8):
    if t:
      ts = env.step(rng.uniform(0, 1, 4))
    sprites = env.state()['sprites']
    got = ts.observation['masks']
    assert got.shape == (16, 24) and got.dtype == np.uint8
    arrs = dict(x=np.array([s.x for s in sprites]), y=np.array([s.y for s in sprites]),
                shape=np.array([oracle.SHAPE_IDS[s.shape] for s in sprites]),
                angle=np.array([s.angle for s in sprites]), scale=np.array([s.scale for s in sprites]))
    n = len(sprites)
    arrs.update(vx=np.zeros(n), vy=np.zeros(n), member=np.zeros(n, np.uint32), pos_f32=np.zeros(n, np.uint8),
                rgb=np.zeros((n, 3), np.uint8))
    want = mask_oracle.render_masks(oracle.raster_cfg(24, 16, 3), tab, fixtures.records_from_arrays(arrs))
    assert np.array_equal(got, want), t
  env.close()
