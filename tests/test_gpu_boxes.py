"""Box mode of the mask kernel (csrc/swb_masks.cuh, swb_render_boxes) against the CPU restatement
tests/box_oracle.py and against the device's own coverage, box for box and count for count.

- Every raster of test_gpu_render_geometry.CASES (convex and concave pools, 1 to 32 slots, so slot
  31 too), plus test_gpu_masks.EXTRA and the huge-sprite cases, into sentinel-filled buffers at
  4-byte-aligned offsets that are not 16-byte aligned, whose guard bytes must survive; the boxes of
  swb_render_coverage's bits on the same state; permuted and repeated records.
- Episodes of a BatchedEnvironment with SpriteMasks, SpriteCoverage, SpriteBoxes and SpriteFactors
  through auto-resets, with the host and the device scene sampler; expand leaves; a checkpoint
  round trip.
- Two launches per call and nothing else changes; n = 0 and every refusal enqueue nothing.
- The drop-in Environment on a sprite list.
"""
import collections
import ctypes

import numpy as np
import pytest

from oracle import oracle
from tests import box_oracle
from tests import test_gpu_masks as gm
from tests import test_gpu_render_geometry as geo
from tests import mask_oracle

gpu = pytest.mark.gpu
KEYS = ('visible_box', 'amodal_box', 'visible', 'area')


def _boxes_guarded(eng, W, H, aa, n, skews=(0, 0, 0, 0), states=None):
  """render_boxes into four guarded int32 buffers `skews` bytes past 16-byte boundaries; checks the
  guards and the launch count and returns the four as arrays."""
  import torch
  S = eng.n_slots
  shapes = ((n, S, 4), (n, S, 4), (n, S), (n, S))
  sizes = [4 * int(np.prod(s)) for s in shapes]
  bufs = [geo._guarded(nb, eng.device, skew) for nb, skew in zip(sizes, skews)]
  out = [flat.view(torch.int32).view(shape) for (_, flat, _), shape in zip(bufs, shapes)]
  for t in out:
    t.fill_(-7)                     # the call zeroes its outputs itself
  launches = eng.launch_count()
  got = eng.render_boxes(W, H, aa, states=states, out=out)
  assert all(g is o for g, o in zip(got, out)) and eng.launch_count() == launches + (2 if n else 0)
  torch.cuda.synchronize()
  for (big, _, lo), nb, name in zip(bufs, sizes, KEYS):
    geo._assert_guards(big, lo, nb, (W, H, aa, skews, name))
  return tuple(t.cpu().numpy() for t in out)


def _want(sw, W, H, aa):
  rc = oracle.raster_cfg(W, H, aa)
  got = [box_oracle.render_boxes(rc, sw.tab, sw.rec[e]) for e in range(sw.E)]
  return tuple(np.stack(x) for x in zip(*got))


def _assert_same(got, want, what):
  for name, g, w in zip(KEYS, got, want):
    bad = np.argwhere(g != w)
    assert not len(bad), (what, name, len(bad), bad[:4].tolist())


def _check_sweep(sw, W, H, aa, skews=((0, 0, 0, 0), (4, 8, 12, 4))):
  import torch
  want = _want(sw, W, H, aa)
  box_oracle.check_invariants(*want, W, H, (W, H, aa))
  for skew in skews:
    _assert_same(_boxes_guarded(sw.eng, W, H, aa, sw.E, skew), want, (W, H, aa, skew))
  # the device's own coverage of the same state: its bits' boxes and its counts
  cover, visible, area = sw.eng.render_coverage(W, H, aa)
  from_cover = box_oracle.boxes_of_covers(cover.cpu().numpy(), sw.eng.n_slots)
  _assert_same(from_cover[:2] + (visible.cpu().numpy(), area.cpu().numpy()), want, (W, H, aa, 'coverage'))
  _assert_same(from_cover, want, (W, H, aa, 'coverage bits'))
  # records, permuted and repeated, give the boxes of the envs they were saved from
  perm = torch.from_numpy(np.random.RandomState(sw.E).randint(0, sw.E, sw.E + 3)).to(sw.eng.device)
  states = sw.eng.save_envs().take(perm)
  got = _boxes_guarded(sw.eng, W, H, aa, len(states), (12, 4, 8, 4), states=states)
  p = perm.cpu().numpy()
  _assert_same(got, tuple(w[p] for w in want), (W, H, aa, 'records'))
  return want


@gpu
@pytest.mark.parametrize('case', geo.CASES, ids=[c[0] for c in geo.CASES])
def test_boxes_sweep(case):
  sw = geo.Sweep(case, geo._n_sms())
  try:
    want = _check_sweep(sw, sw.W, sw.H, sw.aa)
    if sw.S == 32:
      assert (want[3][:, 31] > 0).any()   # slot 31, the sign bit of the coverage, is exercised
  finally:
    sw.close()


@gpu
@pytest.mark.parametrize('extra', gm.EXTRA, ids=[c[0] for c in gm.EXTRA])
def test_boxes_on_tall_and_4095_canvases(extra):
  cid, W, H, aa, S, E, concave = extra
  sw = geo.Sweep((cid, W, H, aa, (0, 0, 0), S, E, concave, 'edges'), geo._n_sms())
  try:
    _check_sweep(sw, W, H, aa, skews=((0, 0, 0, 0), (8, 12, 4, 8)))
  finally:
    sw.close()


@gpu
@pytest.mark.parametrize('huge', gm.HUGE, ids=[c[0] for c in gm.HUGE])
def test_boxes_of_sprites_with_edges_beyond_int16_rows(huge):
  cid, W, H, aa, S, E = huge
  arrs = mask_oracle.huge_scene_arrays(np.random.RandomState(len(cid) + S), E, S, aa * H)
  sw = geo.Sweep((cid, W, H, aa, (0, 0, 0), S, E, True, 'edges'), geo._n_sms(), arrs=arrs)
  try:
    rc = oracle.raster_cfg(W, H, aa)
    assert max(abs(mask_oracle.canvas_vertices(rc, sw.tab, r)[:, 1]).max() for r in sw.rec[0]) > 40000
    _check_sweep(sw, W, H, aa, skews=((0, 0, 0, 0), (4, 4, 4, 4)))
  finally:
    sw.close()


def _env(E=48, seed=3, max_episode_length=5, sampler='host'):
  from spriteworld_b200 import action_spaces, environment, renderers
  from spriteworld_b200.configs.cobra import goal_finding_more_targets as cfgmod
  cfg = cfgmod.get_config('train')
  cfg['max_episode_length'] = max_episode_length
  cfg['action_space'] = action_spaces.SelectMove(scale=0.25)
  cfg['renderers'] = collections.OrderedDict([
      ('masks', renderers.SpriteMasks(image_size=(32, 24), anti_aliasing=1)),
      ('cover', renderers.SpriteCoverage(image_size=(32, 24), anti_aliasing=1)),
      ('boxes', renderers.SpriteBoxes(image_size=(32, 24), anti_aliasing=1)),
      ('fine', renderers.SpriteBoxes(image_size=(40, 40), anti_aliasing=5)),
      ('factors', renderers.SpriteFactors())])
  kw = dict(refill='sync') if sampler == 'host' else dict(sampler='device', seed=seed)
  return environment.BatchedEnvironment(n_envs=E, pool_depth=5, rng=np.random.RandomState(seed), **kw, **cfg)


def _oracle_boxes(env, renderer, states):
  rc = oracle.raster_cfg(renderer.width, renderer.height, renderer.anti_aliasing)
  got = [box_oracle.render_boxes(rc, gm._tab(), sp) for sp in gm._sprites_of(env.engine, states)]
  return tuple(np.stack(x) for x in zip(*got))


def _assert_boxes(obs, want, what):
  assert tuple(obs) == KEYS, what
  for k, w in zip(obs, want):
    assert np.array_equal(obs[k].cpu().numpy(), w), (what, k)


@gpu
@pytest.mark.parametrize('sampler', ['host', 'device'])
def test_episodes_boxes_equal_the_oracle_and_the_coverage(sampler):
  env = _env(sampler=sampler)
  rng = np.random.RandomState(1)
  ts = env.reset()
  buffers = [t.data_ptr() for t in ts.observation['boxes'].values()]
  S = env.engine.n_slots
  lasts = 0
  for t in range(14):
    if t:
      ts = env.step(rng.uniform(0, 1, (env.n_envs, 4)).astype(np.float32))
    lasts += int((ts.step_type.cpu().numpy() == 2).sum())
    states = env.save_envs()
    for name in ('boxes', 'fine'):
      _assert_boxes(ts.observation[name], _oracle_boxes(env, env._renderers[name], states), (t, name))
    assert [v.data_ptr() for v in ts.observation['boxes'].values()] == buffers
    # the same step's coverage, summarised, is the boxes
    cover = ts.observation['cover']
    _assert_boxes(ts.observation['boxes'], box_oracle.boxes_of_covers(cover['cover'].cpu().numpy(), S), t)
    occupied = ts.observation['factors']['mask'].cpu().numpy()
    assert (ts.observation['boxes']['amodal_box'].cpu().numpy()[~occupied] == 0).all(), t
  assert lasts > env.n_envs   # the run went through auto-resets
  env.close()


@gpu
def test_boxes_of_leaves_and_after_a_checkpoint():
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
  for name in ('boxes', 'fine'):
    _assert_boxes(obs[name], _oracle_boxes(env, env._renderers[name], pick), ('leaves', name))
  sd = env.state_dict()
  saved = {k: {f: v.clone() for f, v in env.render()[k].items()} for k in ('boxes', 'fine')}
  env.load_envs(pick)
  out = env.render()
  for k in ('boxes', 'fine'):
    for f in KEYS:
      assert torch.equal(obs[k][f], out[k][f]), (k, f)
  env.load_state_dict(sd)
  out = env.render()
  for k in ('boxes', 'fine'):
    for f in KEYS:
      assert torch.equal(out[k][f], saved[k][f]), (k, f)
  env.close()


@gpu
def test_two_launches_per_call_and_nothing_else_changes():
  import torch
  env = _env(E=16)
  rng = np.random.RandomState(3)
  env.reset()
  env.step(rng.uniform(0, 1, (env.n_envs, 4)).astype(np.float32))
  eng = env.engine
  states = env.save_envs()
  saved = eng.save_state()
  masks = env._mask_buffers[id(env._renderers['masks'])].clone()
  status = eng.render_status().clone()
  rng_state = env._rng.get_state()
  own = env._mask_buffers[id(env._renderers['boxes'])]
  launches = eng.launch_count()
  b = eng.render_boxes(32, 24, 1)
  assert eng.launch_count() == launches + 2
  r = eng.render_boxes(20, 30, 7, states=states)
  S = eng.n_slots
  assert eng.launch_count() == launches + 4
  assert [tuple(t.shape) for t in r] == [(16, S, 4), (16, S, 4), (16, S), (16, S)]
  obs = env.render_boxes(env._renderers['boxes'])
  assert eng.launch_count() == launches + 6
  assert [v.data_ptr() for v in obs.values()] == [t.data_ptr() for t in own]
  empty = eng.render_boxes(32, 24, 1, states=states[:0])
  assert [tuple(t.shape) for t in empty] == [(0, S, 4), (0, S, 4), (0, S), (0, S)]
  assert eng.launch_count() == launches + 6
  assert torch.equal(eng.save_state(), saved)
  assert torch.equal(eng.render_status(), status)
  assert torch.equal(env._mask_buffers[id(env._renderers['masks'])], masks)
  assert all(np.array_equal(a, c) for a, c in zip(env._rng.get_state()[1:], rng_state[1:]))
  for a, c in zip(b, own):
    assert torch.equal(a, c)
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
  nb, nv = n * S * 16, n * S * 4
  big, flat, lo = geo._guarded(2 * nb + 2 * nv + 64, eng.device)
  base = flat.data_ptr()
  bp, ap = ctypes.c_void_p(base), ctypes.c_void_p(base + nb)
  vp, rp_ = ctypes.c_void_p(base + 2 * nb), ctypes.c_void_p(base + 2 * nb + nv)
  rp, rb = ctypes.c_void_p(states.data.data_ptr()), states.data.numel()
  stream = eng._stream()
  odd = ctypes.c_void_p(states.data.data_ptr() + 8)

  def at(off):
    return ctypes.c_void_p(base + off)
  h = eng._h
  cases = [
      ('null', (None, W, H, 1, None, n, 0, bp, ap, vp, rp_)),
      ('null output visible_box', (h, W, H, 1, None, n, 0, None, ap, vp, rp_)),
      ('null output amodal_box', (h, W, H, 1, None, n, 0, bp, None, vp, rp_)),
      ('null output visible', (h, W, H, 1, None, n, 0, bp, ap, None, rp_)),
      ('null output area', (h, W, H, 1, None, n, 0, bp, ap, vp, None)),
      ('must be >= 1', (h, 0, H, 1, None, n, 0, bp, ap, vp, rp_)),
      ('must be >= 1', (h, W, -1, 1, None, n, 0, bp, ap, vp, rp_)),
      ('must be >= 1', (h, W, H, 0, None, n, 0, bp, ap, vp, rp_)),
      ('4095', (h, 4096, 1, 1, None, n, 0, bp, ap, vp, rp_)),
      ('4095', (h, 1, 820, 5, None, n, 0, bp, ap, vp, rp_)),
      ('n = -1', (h, W, H, 1, rp, -1, rb, bp, ap, vp, rp_)),
      ('must be E', (h, W, H, 1, None, n - 1, 0, bp, ap, vp, rp_)),
      ('must be E', (h, W, H, 1, None, 0, 0, bp, ap, vp, rp_)),
      ('16-byte aligned', (h, W, H, 1, odd, 2, rb, bp, ap, vp, rp_)),
      ('bytes', (h, W, H, 1, rp, n, rb - 16, bp, ap, vp, rp_)),
      ('visible_box is not 4-byte aligned', (h, W, H, 1, None, n, 0, at(2), ap, vp, rp_)),
      ('amodal_box is not 4-byte aligned', (h, W, H, 1, None, n, 0, bp, at(nb + 1), vp, rp_)),
      ('visible is not 4-byte aligned', (h, W, H, 1, None, n, 0, bp, ap, at(2 * nb + 3), rp_)),
      ('area is not 4-byte aligned', (h, W, H, 1, None, n, 0, bp, ap, vp, at(2 * nb + nv + 2))),
      ('amodal_box overlaps visible_box', (h, W, H, 1, None, n, 0, bp, at(nb - 4), vp, rp_)),
      ('visible overlaps visible_box', (h, W, H, 1, None, n, 0, bp, ap, at(16), rp_)),
      ('visible overlaps amodal_box', (h, W, H, 1, None, n, 0, bp, ap, at(2 * nb - 4), rp_)),
      ('area overlaps visible', (h, W, H, 1, None, n, 0, bp, ap, vp, vp)),
      ('visible_box overlaps the records', (h, W, H, 1, rp, n, rb, ctypes.c_void_p(states.data.data_ptr() + 32),
                                            ap, vp, rp_)),
      ('amodal_box overlaps the records', (h, W, H, 1, rp, n, rb, bp, rp, vp, rp_)),
      ('area overlaps the records', (h, W, H, 1, rp, n, rb, bp, ap, vp,
                                     ctypes.c_void_p(states.data.data_ptr() + rb - 4))),
  ]
  launches = eng.launch_count()
  for msg, args in cases:
    assert L.swb_render_boxes(*args, stream) != 0, msg
    assert msg.encode() in L.swb_last_error(), (msg, L.swb_last_error())
    assert eng.launch_count() == launches, msg
  # a grid the launch cannot express, checked before any buffer is read: as for the coverage, a
  # band holds 16 KiB of coverage words, so 2^30 records of 300 rows 4000 pixels wide exceed 2^31 - 1 CTAs
  big_n = (1 << 30)
  assert L.swb_render_boxes(h, 4000, 300, 1, rp, big_n, big_n * states.record_bytes, bp, ap, vp, rp_,
                            stream) != 0
  assert b'2^31' in L.swb_last_error()
  torch.cuda.synchronize()
  assert bool((flat == geo.SENTINEL).all()) and bool((big == geo.SENTINEL).all())
  assert eng.launch_count() == launches
  # through Python: NativeError (or ValueError before the call), nothing enqueued
  with pytest.raises(_native.NativeError, match='4095'):
    eng.render_boxes(2048, 8, 2)
  b4 = torch.zeros((n, S, 4), dtype=torch.int32, device=eng.device)
  v = torch.zeros((n, S), dtype=torch.int32, device=eng.device)
  with pytest.raises(_native.NativeError, match='amodal_box overlaps visible_box'):
    eng.render_boxes(W, H, 1, out=(b4, b4, v, v.clone()))
  with pytest.raises(ValueError, match='states must be EnvStates'):
    eng.render_boxes(W, H, 1, states=torch.zeros(4))
  empty = states.take(torch.zeros(0, dtype=torch.int64, device=eng.device))
  with pytest.raises(_native.NativeError, match='4095'):
    eng.render_boxes(2048, 8, 2, states=empty)
  got = eng.render_boxes(16, 8, 3, states=empty)
  assert [tuple(t.shape) for t in got] == [(0, S, 4), (0, S, 4), (0, S), (0, S)]
  assert eng.launch_count() == launches
  env.close()


@gpu
def test_drop_in_environment_boxes_equal_the_oracle_of_its_sprite_list():
  from spriteworld_b200 import environment, renderers
  from spriteworld_b200.configs.cobra import goal_finding_more_targets as cfgmod
  from tests import fixtures
  cfg = cfgmod.get_config('train')
  cfg['renderers'] = collections.OrderedDict([
      ('boxes', renderers.SpriteBoxes(image_size=(24, 16), anti_aliasing=3)),
      ('masks', renderers.SpriteMasks(image_size=(24, 16), anti_aliasing=3))])
  env = environment.Environment(**cfg)
  rng = np.random.RandomState(4)
  tab = gm._tab()
  ts = env.reset()
  for t in range(8):
    if t:
      ts = env.step(rng.uniform(0, 1, 4))
    sprites = env.state()['sprites']
    got = ts.observation['boxes']
    n = len(sprites)
    assert tuple(got) == KEYS and got['visible_box'].shape == (n, 4) and got['visible_box'].dtype == np.int32
    arrs = dict(x=np.array([s.x for s in sprites]), y=np.array([s.y for s in sprites]),
                shape=np.array([oracle.SHAPE_IDS[s.shape] for s in sprites]),
                angle=np.array([s.angle for s in sprites]), scale=np.array([s.scale for s in sprites]),
                vx=np.zeros(n), vy=np.zeros(n), member=np.zeros(n, np.uint32), pos_f32=np.zeros(n, np.uint8),
                rgb=np.zeros((n, 3), np.uint8))
    want = box_oracle.render_boxes(oracle.raster_cfg(24, 16, 3), tab, fixtures.records_from_arrays(arrs))
    for k, w in zip(KEYS, want):
      assert np.array_equal(got[k], w), (t, k)
    for k in range(n):
      assert np.array_equal(got['visible_box'][k], box_oracle.box(ts.observation['masks'] == k + 1)), (t, k)
  env.close()
