"""Positions inside sprites on the GPU (swb_sample_contained, csrc/swb_contained.cuh).

- The device equals the CPU build of the same source (scene_program.sample_contained_on_host), bit
  for bit, on live envs of four COBRA configs through auto-resets with both scene samplers, on
  permuted records and expand leaves, and at 1, 33 and 4097 rows; a record gives the samples of the
  env it was saved from.
- A float64 SelectMove / DragAndDrop click at a sampled position moves exactly one sprite, at or
  above the sampled slot, by the action's motion.
- A call is one launch, reads only, never synchronises the host, runs next to the asynchronous
  refill; refused calls enqueue nothing.
- Plans whose first click is a contained proposal all move a sprite.
"""
import ctypes
import importlib

import numpy as np
import pytest
import torch

from spriteworld_b200 import _native, action_spaces, environment, renderers, scene_program

pytestmark = pytest.mark.gpu

CONFIGS = ('goal_finding_new_position', 'sorting', 'clustering', 'exploration')
SAMPLERS = {'host': dict(refill='sync'), 'device': dict(sampler='device', seed=17)}


def _env(name='exploration', E=37, sampler='host', max_episode_length=3, action_space=None, refill=None,
         seed=0, factors=True):
  cfg = importlib.import_module('spriteworld_b200.configs.cobra.' + name).get_config('train')
  cfg['max_episode_length'] = max_episode_length
  cfg['renderers'] = {'factors': renderers.SpriteFactors()} if factors else cfg['renderers']
  if action_space is not None:
    cfg['action_space'] = action_space
  kw = dict(SAMPLERS[sampler])
  if refill:
    kw['refill'] = refill
  return environment.BatchedEnvironment(n_envs=E, pool_depth=4, rng=np.random.RandomState(seed), **dict(cfg, **kw))


def _live_rows(env):
  """The rows the live path reads: live positions, and the transform and shape of pool entry
  e * K + cursor[e]."""
  eng = env.engine
  live, pool, K = eng.state_tensors(), eng.pool_tensors(), eng.pool_depth
  entry = torch.arange(0, env.n_envs * K, K, device=eng.device) + live['cursor']
  rows = {k: pool[k].flatten(0, 1).index_select(0, entry).cpu().numpy() for k in ('m00', 'm01', 'm10', 'm11', 'shape')}
  rows['x'], rows['y'] = live['pos_x'].cpu().numpy(), live['pos_y'].cpu().numpy()
  return rows


def _record_rows(states):
  h = states.to_host()
  return dict(x=h['pos_x'], y=h['pos_y'], m00=h['m00'], m01=h['m01'], m10=h['m10'], m11=h['m11'], shape=h['shape'])


def _same(got, want, what):
  gp, gk, gs = (t.cpu().numpy() for t in got)
  wp, wk, ws = want
  assert np.array_equal(gp.view(np.uint64), wp.view(np.uint64)), (what, np.argwhere(gp.view(np.uint64) != wp.view(np.uint64))[:4])
  assert np.array_equal(gk, wk), what
  assert np.array_equal(gs, ws), what


def _check_live(env, seed, what):
  rows = _live_rows(env)
  for n_samples in (None, 1, 3, 64):
    got = env.sample_contained_positions(seed, n_samples)
    want = scene_program.sample_contained_on_host(rows, seed, 1 if n_samples is None else n_samples)
    if n_samples is None:
      assert tuple(got.position.shape) == (env.n_envs, 2) and tuple(got.slot.shape) == (env.n_envs,)
      want = tuple(w[:, 0] for w in want)
    _same(got, want, (what, n_samples))
    assert got.position.dtype == torch.float64 and got.slot.dtype == torch.int8 and got.status.dtype == torch.uint8


@pytest.mark.parametrize('sampler', list(SAMPLERS))
@pytest.mark.parametrize('name', CONFIGS)
def test_live_envs_equal_the_host_build_through_auto_resets(name, sampler):
  env = _env(name, sampler=sampler)
  rng = np.random.RandomState(1)
  _check_live(env, 5, 'before reset')   # about to reset: the scene the env is still on
  env.reset()
  lasts = 0
  for t in range(7):
    ts = env.step(rng.uniform(0, 1, (env.n_envs, 4)).astype(np.float32))
    lasts += int((ts.step_type == _native.STEP_LAST).sum())
    _check_live(env, 2 ** 64 - 1 - t, (name, sampler, t))
  assert lasts > 0
  env.close()


def test_records_equal_the_host_build_and_the_live_envs():
  env = _env('exploration', E=40, max_episode_length=6)
  rng = np.random.RandomState(2)
  env.reset()
  env.step(rng.uniform(0, 1, (env.n_envs, 4)).astype(np.float32))
  states = env.save_envs()
  # record i gives live env i's samples
  live = env.sample_contained_positions(99, 5)
  rec = env.sample_contained_positions(99, 5, states=states)
  for a, b in zip(live, rec):
    assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))
  # permuted and repeated records
  perm = torch.from_numpy(rng.randint(0, env.n_envs, 53)).to(env.engine.device)
  sub = states.take(perm)
  _same(env.sample_contained_positions(7, 4, states=sub),
        scene_program.sample_contained_on_host(_record_rows(sub), 7, 4), 'permuted')
  # expand leaves, and a zero record (an index outside the records): no sprite
  plans = rng.uniform(0, 1, (2, env.n_envs, 3, 4)).astype(np.float32)
  _, leaves = env.expand(plans)
  _same(env.sample_contained_positions(8, 3, states=leaves),
        scene_program.sample_contained_on_host(_record_rows(leaves), 8, 3), 'leaves')
  zero = states.take(torch.tensor([-1, 0], device=env.engine.device))
  got = env.sample_contained_positions(8, 2, states=zero)
  assert (got.status[0] == _native.ENV_NO_SPRITE).all() and (got.slot[0] == -1).all()
  assert torch.isnan(got.position[0]).all() and (got.status[1] == 0).all()
  # zero records draw nothing
  empty = states.take(torch.zeros(0, dtype=torch.int64, device=env.engine.device))
  got = env.sample_contained_positions(8, 2, states=empty)
  assert tuple(got.position.shape) == (0, 2, 2)
  env.close()


@pytest.mark.parametrize('E', [1, 33, 4097])
def test_row_counts(E):
  env = _env('exploration', E=E, sampler='device')
  env.reset()
  _check_live(env, 123456789, E)
  env.close()


def _click_case(kind):
  rng = np.random.RandomState(3)
  space = action_spaces.SelectMove(scale=0.5) if kind == 'select_move' else action_spaces.DragAndDrop(scale=1.0)
  env = _env('exploration', E=64, max_episode_length=50, action_space=space)
  env.reset()
  eng = env.engine
  moved_total = 0
  for t in range(4):
    cp = env.sample_contained_positions(1000 + t)
    assert (cp.status == 0).all()
    before = {k: v.cpu().numpy().copy() for k, v in eng.state_tensors().items()}
    pos = cp.position.cpu().numpy()
    x0, y0 = before['pos_x'], before['pos_y']
    k = cp.slot.cpu().numpy()
    # a motion toward the frame's centre, by a random fraction
    target = np.stack([x0[np.arange(env.n_envs), k], y0[np.arange(env.n_envs), k]], 1)
    frac = rng.uniform(0.1, 0.9, (env.n_envs, 1))
    motion = (0.5 - target) * frac
    if kind == 'select_move':
      tail = motion / 0.5 + 0.5
      mx, my = (tail[:, 0] - 0.5) * 0.5, (tail[:, 1] - 0.5) * 0.5
    else:
      tail = pos + motion
      mx, my = (tail[:, 0] - pos[:, 0]) * 1.0, (tail[:, 1] - pos[:, 1]) * 1.0
    actions = np.concatenate([pos, tail], 1).astype(np.float64)
    ts = env.step(actions)
    assert (ts.step_type == _native.STEP_MID).all()
    after = {k2: v.cpu().numpy() for k2, v in eng.state_tensors().items()}
    f32 = _live_rows_pos_f32(env)
    for e in range(env.n_envs):
      changed = np.flatnonzero((after['pos_x'][e] != x0[e]) | (after['pos_y'][e] != y0[e]))
      assert len(changed) == 1, (kind, t, e, changed)
      j = int(changed[0])
      assert j >= k[e], (kind, t, e)
      nx, ny = x0[e, j] + mx[e], y0[e, j] + my[e]
      if f32[e, j]:
        nx, ny = float(np.float32(nx)), float(np.float32(ny))
      nx, ny = min(max(nx, 0.0), 1.0), min(max(ny, 0.0), 1.0)   # keep_in_frame
      assert after['pos_x'][e, j] == nx and after['pos_y'][e, j] == ny, (kind, t, e)
      moved_total += 1
  assert moved_total == 4 * env.n_envs
  env.close()


def _live_rows_pos_f32(env):
  eng = env.engine
  live, pool, K = eng.state_tensors(), eng.pool_tensors(), eng.pool_depth
  entry = torch.arange(0, env.n_envs * K, K, device=eng.device) + live['cursor']
  return pool['pos_f32'].flatten(0, 1).index_select(0, entry).cpu().numpy()


@pytest.mark.parametrize('kind', ['select_move', 'drag_and_drop'])
def test_a_click_at_the_sample_moves_the_sampled_sprite_or_one_above(kind):
  _click_case(kind)


def _no_sync(fn):
  prev = torch.cuda.get_sync_debug_mode()
  torch.cuda.set_sync_debug_mode('error')
  try:
    return fn()
  finally:
    torch.cuda.set_sync_debug_mode(prev)


def test_read_only_one_launch_and_no_host_sync_next_to_the_async_refill():
  env = _env('exploration', E=48, max_episode_length=2, refill='async', factors=False)
  eng = env.engine
  rng = np.random.RandomState(4)
  env.reset()
  refills = 0
  for t in range(8):
    env.step(rng.uniform(0, 1, (env.n_envs, 4)).astype(np.float32))
    refills += env._inflight is not None
    # enqueued while the refill may still be sampling and uploading on its side stream
    launches = eng.launch_count()
    a = _no_sync(lambda: env.sample_contained_positions(t, 16))
    assert eng.launch_count() == launches + 1
    env._land(True)     # no refill in flight from here to the end of the iteration
    torch.cuda.synchronize()
    _same(a, scene_program.sample_contained_on_host(_live_rows(env), t, 16), t)
    saved = eng.save_state()
    frames = {k: v.clone() for k, v in env._frames.items()}
    rng_state = env._rng.get_state()
    stats = env.refill_stats()
    launches = eng.launch_count()
    b = _no_sync(lambda: env.sample_contained_positions(t))
    assert eng.launch_count() == launches + 1
    torch.cuda.synchronize()
    assert torch.equal(eng.save_state(), saved)
    for k, v in frames.items():
      assert torch.equal(env._frames[k], v), k
    st = env._rng.get_state()
    assert all(np.array_equal(np.asarray(x), np.asarray(y)) for x, y in zip(st, rng_state))
    assert env.refill_stats() == stats
    assert torch.equal(b.position, a.position[:, 0]) and torch.equal(b.slot, a.slot[:, 0])
  assert refills > 0
  env.close()


def test_refused_calls_enqueue_nothing():
  env = _env('exploration', E=8)
  env.reset()
  eng = env.engine
  L = eng._lib
  states = env.save_envs()
  pos = torch.empty((8, 4, 2), dtype=torch.float64, device=eng.device)
  slot = torch.empty((8, 4), dtype=torch.int8, device=eng.device)
  status = torch.empty((8, 4), dtype=torch.uint8, device=eng.device)
  outs = [ctypes.c_void_p(t.data_ptr()) for t in (pos, slot, status)]
  rp, rb = ctypes.c_void_p(states.data.data_ptr()), states.data.numel()
  odd = ctypes.c_void_p(states.data.data_ptr() + 8)
  stream = eng._stream()
  torch.cuda.synchronize()
  cases = [
      ('null engine', (None, None, 8, 0, 4, 1, *outs)),
      ('null output', (eng._h, None, 8, 0, 4, 1, None, outs[1], outs[2])),
      ('null output', (eng._h, None, 8, 0, 4, 1, outs[0], None, outs[2])),
      ('null output', (eng._h, rp, 8, rb, 4, 1, outs[0], outs[1], None)),
      ('n_samples = 0', (eng._h, None, 8, 0, 0, 1, *outs)),
      ('n_samples = -3', (eng._h, rp, 8, rb, -3, 1, *outs)),
      ('2^31 - 1', (eng._h, rp, 65536, 65536 * states.record_bytes, 32768, 1, *outs)),
      ('must be E', (eng._h, None, 7, 0, 4, 1, *outs)),
      ('must be E', (eng._h, None, 0, 0, 4, 1, *outs)),
      ('n = -1', (eng._h, rp, -1, rb, 4, 1, *outs)),
      ('16-byte aligned', (eng._h, odd, 2, rb, 4, 1, *outs)),
      ('bytes', (eng._h, rp, 8, rb - 16, 4, 1, *outs)),
      ('position is not 8-byte aligned', (eng._h, None, 8, 0, 4, 1, ctypes.c_void_p(pos.data_ptr() + 4),
                                          outs[1], outs[2])),
      ('position overlaps the records', (eng._h, rp, 8, rb, 4, 1, ctypes.c_void_p(states.data.data_ptr() + 16),
                                         outs[1], outs[2])),
      ('status overlaps slot', (eng._h, rp, 8, rb, 4, 1, outs[0], outs[1], ctypes.c_void_p(slot.data_ptr() + 31))),
  ]
  records = states.data.clone()
  launches = eng.launch_count()
  for msg, args in cases:
    assert L.swb_sample_contained(*args, stream) != 0, msg
    assert msg.encode() in L.swb_last_error(), (msg, L.swb_last_error())
    assert eng.launch_count() == launches, msg
  torch.cuda.synchronize()
  assert torch.equal(states.data, records)
  # zero records are accepted and draw nothing
  assert L.swb_sample_contained(eng._h, rp, 0, 0, 4, 1, *outs, stream) == 0
  assert eng.launch_count() == launches
  # through Python
  for bad in (-1, 2 ** 64, 1.5, None, True):
    with pytest.raises(ValueError, match='seed'):
      eng.sample_contained(bad)
  for bad in (0, -2, 2 ** 31, 2.0):
    with pytest.raises(ValueError, match='n_samples'):
      eng.sample_contained(1, bad)
  with pytest.raises(ValueError):
    eng.sample_contained(1, states=states[:3].data)
  assert eng.launch_count() == launches
  env.close()


def _plans_moving(env, first, C):
  """(n_envs, C) bool: which plans' first step moves a sprite (expand with T = 1, leaf positions
  against the roots')."""
  E = env.n_envs
  _, leaves = env.expand(first[None])
  roots = env.save_envs().to_host()
  h = leaves.to_host()
  rx = np.repeat(roots['pos_x'], C, 0)
  ry = np.repeat(roots['pos_y'], C, 0)
  moved = ((h['pos_x'] != rx) | (h['pos_y'] != ry)).any(1)
  return moved.reshape(E, C)


def test_contained_proposals_move_a_sprite_on_every_first_step():
  env = _env('goal_finding_new_position', E=256, max_episode_length=20, sampler='device')
  env.reset()
  rng = np.random.RandomState(6)
  E, C, T = env.n_envs, 16, 3
  # T * C samples per root, reshaped to (T, n, C, 2): the first clicks of a random-shooting level
  cp = env.sample_contained_positions(42, T * C)
  assert (cp.status == 0).all()
  clicks = cp.position.reshape(E, T, C, 2).permute(1, 0, 2, 3)
  motion = torch.from_numpy(rng.uniform(0, 1, (T, E, C, 2))).to(clicks.device)
  plans = torch.cat([clicks, motion], -1).contiguous()
  moved = _plans_moving(env, plans[0], C)
  uniform = torch.from_numpy(rng.uniform(0, 1, (E, C, 4))).to(clicks.device)
  moved_uniform = _plans_moving(env, uniform, C)
  print('first steps that move a sprite: contained proposals %.4f, uniform clicks %.4f'
        % (moved.mean(), moved_uniform.mean()))
  assert moved.all()
  res = env.rollout(plans)
  assert tuple(res.reward.shape) == (T, E, C)
  env.close()
