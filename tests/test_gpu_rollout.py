"""The rollout kernel (csrc/swb_rollout.cuh, swb_rollout), bit for bit.

Entry [t, e, c] of a rollout is what the t-th Engine.step with candidate c's actions reports for
an env in the state env e has when the rollout runs, up to and including the plan's first LAST;
everything after it, and every entry of an env about to reset, is padding.  Checked against the
step kernel -- an engine of n_envs x C envs loaded from the saved records and stepped T times --
and against the CPU oracle in its sqrt mode stepped from the decoded records, over the step sweep's
cases: every action kind and dtype, FindGoalPosition, Clustering with its error statuses, a
MetaAggregated root, mixed float32 / float64 positions, velocities, keep_in_frame off, 1 and 32
slots, bad Embodied directions, and envs at different step counts.  A rollout changes nothing:
state, pool, scene_serial, statuses and the refill bookkeeping are as they were, and it adds one
launch.  Calls the C-ABI refuses enqueue nothing.
"""
import ctypes

import numpy as np
import pytest
import torch

from spriteworld_b200 import _native

gpu = pytest.mark.gpu
PAD = dict(reward=0.0, step_type=_native.STEP_NONE, success=0, status=0)
NAMES = ('reward', 'step_type', 'success', 'status')


def _host(res):
  return {k: getattr(res, k).cpu().numpy().copy() for k in NAMES}


def _bits(a):
  return a.view(np.int64) if a.dtype == np.float64 else a


def _stepped(eng, make_engine, plans):
  """(outputs (T, E, C) of T Engine.step calls on an engine of E x C envs loaded from eng's saved
  records, the mask of their live steps, the saved records of the E x C envs)."""
  T, E, C = plans.shape[:3]
  ids = np.repeat(np.arange(E), C)
  saved = eng.save_envs()[ids]
  big = make_engine(E * C)
  big.load_envs(saved)
  out = {k: [] for k in NAMES}
  for t in range(T):
    res = big.step(torch.from_numpy(np.ascontiguousarray(plans[t].reshape((E * C,) + plans.shape[3:]))).to(big.device))
    for k, v in _host(res).items():
      out[k].append(v.reshape(E, C))
  big.close()
  out = {k: np.stack(v) for k, v in out.items()}
  st = out['step_type']
  lasts_before = np.cumsum(st == _native.STEP_LAST, 0) - (st == _native.STEP_LAST)
  started = np.cumsum(st == _native.STEP_FIRST, 0) > 0     # an env about to reset starts a scene
  return out, (lasts_before == 0) & ~started, saved


def _assert_rollout(got, want, mask, what, nan_bits=True):
  for k in NAMES:
    expect = np.where(mask, want[k], np.asarray(PAD[k], want[k].dtype))
    if k == 'reward' and not nan_bits:
      assert np.array_equal(got[k], expect, equal_nan=True), (what, k)
    else:
      assert np.array_equal(_bits(got[k]), _bits(expect)), (what, k)


def _rollout(eng, plans):
  return _host(eng.rollout(torch.from_numpy(np.ascontiguousarray(plans)).to(eng.device)))


# -- the step sweep's cases ---------------------------------------------------------------------

SWEEP = ['select_f32_s1_e1', 'select_f64_s2', 'drag_f32_s5_mixed', 'drag_f64_s8_mixed', 'embodied_s7',
         'embodied_s32_f64', 'edges_keep', 'edges_free', 'goal_filters', 'clustering_f32',
         'clustering_f64', 'meta_all_aggs', 'wide_f64_cost', 'select_f64_s32_many']
# statuses that must show up in live entries, and cases that must end plans by timeout at several t
WANT_STATUS = {'embodied_s7': 4, 'embodied_s32_f64': 4, 'clustering_f32': 1 | 2, 'clustering_f64': 1 | 2}


@gpu
@pytest.mark.parametrize('name', SWEEP)
def test_rollout_matches_the_step_kernel_and_the_oracle(name):
  from spriteworld_b200 import constants, engine
  from tests import test_gpu_step_sweep as sweep
  from tests.test_gpu_env_states import _oracle_from_records
  case = next(c for c in sweep.CASES if c['name'] == name)
  arrs, nodes, action, acts = sweep._setup(case)
  eng = sweep._engine(case, nodes, arrs, action)
  E, mel = case['E'], case['mel']
  for a in acts[:3]:                                  # past the first reset, some envs moved
    eng.step(torch.from_numpy(np.ascontiguousarray(a)).to(eng.device))
  # envs at different step counts (timeouts fall at different t); a few about to reset
  rng = np.random.RandomState(len(name))
  count = rng.randint(0, mel, E).astype(np.int32)
  reset_next = eng.download_state()['reset_next'] | (rng.rand(E) < 0.1)
  eng.upload_state(step_count=count, reset_next=reset_next.astype(np.uint8))
  T, C = 8, 3
  plans = sweep.case_actions(case, arrs, rng, T * C)
  plans = np.ascontiguousarray(plans.reshape((T, C, E) + plans.shape[2:]).swapaxes(1, 2))

  def make_engine(n):
    return engine.Engine(n, case['S'], 1, action, nodes, constants.SHAPES, keep_in_frame=case['keep'],
                         max_episode_length=mel)

  got = _rollout(eng, plans)
  want, mask, saved = _stepped(eng, make_engine, plans)
  _assert_rollout(got, want, mask, 'step kernel')
  assert not mask[:, reset_next > 0].any()
  if E >= 33:
    assert mask[0].any() and mask[0].sum() > mask[-1].sum()      # plans ended inside the window
  assert np.bitwise_or.reduce(got['status'][mask]) & WANT_STATUS.get(name, 0) == WANT_STATUS.get(name, 0)
  if name == 'edges_free':      # keep_in_frame off: plans that end out of frame, unsolved
    last = mask & (got['step_type'] == _native.STEP_LAST)
    t_of = np.broadcast_to(np.arange(T)[:, None, None], mask.shape)
    timeout = count[None, :, None] + t_of + 1 >= mel
    assert (last & (got['success'] == 0) & ~timeout).any()
  if E <= 300:                  # the CPU oracle, stepped from the decoded records
    bo = _oracle_from_records(saved.to_host(), action, nodes, case['keep'], mel, None)
    ref = {k: [] for k in NAMES}
    for t in range(T):
      bo.step(plans[t].reshape((E * C,) + plans.shape[3:]))
      for k, v in zip(NAMES, (bo.reward, bo.step_type, bo.success, bo.err)):
        ref[k].append(v.reshape(E, C).copy())
    _assert_rollout(got, {k: np.stack(v) for k, v in ref.items()}, mask, 'oracle', nan_bits=False)
  eng.close()


# -- shapes -------------------------------------------------------------------------------------

def _c2(n_envs, seed, mel=6, pool_depth=3):
  from spriteworld_b200 import workloads
  wl = workloads.GoalFinding()
  eng, raster, _ = workloads.build_engine(wl, n_envs, pool_depth, seed=seed, max_episode_length=mel)
  return wl, eng, raster


def _c2_engine(wl, mel):
  from spriteworld_b200 import constants, engine
  return lambda n: engine.Engine(n, wl.n_slots, 1, wl.action, wl.nodes, constants.SHAPES,
                                 max_episode_length=mel)


@gpu
@pytest.mark.parametrize('E,T,C,mel', [(1, 1, 1, 6), (301, 1, 1, 6), (301, 3, 1, 6), (7, 4, 5, 6),
                                       (66, 15, 2, 6), (4096, 5, 64, 20)],
                         ids=['one', 'odd_envs_t1', 'odd_envs', 'odd_plans', 't_beyond_the_episode', 'c2_c64'])
def test_rollout_shapes(E, T, C, mel):
  wl, eng, raster = _c2(E, 5, mel)
  rng = np.random.RandomState(E + T)
  for a in wl.sample_actions(rng, 3, E):
    eng.step(torch.from_numpy(a).to(eng.device))
  plans = rng.uniform(0, 1, (T, E, C, 4)).astype(np.float32)
  got = _rollout(eng, plans)
  want, mask, _ = _stepped(eng, _c2_engine(wl, mel), plans)
  _assert_rollout(got, want, mask, (E, T, C))
  assert mask[0].mean() > 0.9
  if T > mel:
    assert mask[mel - 3].any() and not mask[mel:].any()     # no plan outlives the episode
  eng.close()


# -- read-only ----------------------------------------------------------------------------------

def _everything(eng):
  torch.cuda.synchronize(eng.device)
  out = dict(eng.download_state())
  out['scene_serial'] = eng.download_state_serial()
  out['render_status'] = eng.render_status().cpu().numpy().copy()
  out['ids_status'] = eng.env_ids_status().cpu().numpy().copy()
  for k, v in eng.pool_tensors().items():
    out['pool_' + k] = v.cpu().numpy().copy()
  return out


@gpu
def test_rollout_changes_nothing_and_is_one_launch():
  wl, eng, raster = _c2(300, 7)
  _, twin, twin_raster = _c2(300, 7)
  rng = np.random.RandomState(3)
  acts = [torch.from_numpy(a).to(eng.device) for a in wl.sample_actions(rng, 9, 300)]
  for a in acts[:4]:
    eng.step(a, raster)
    twin.step(a, twin_raster)
  before, launches = _everything(eng), eng.launch_count()
  plans = torch.from_numpy(rng.uniform(0, 1, (6, 300, 4, 4))).to(eng.device)
  first = _host(eng.rollout(plans))
  assert eng.launch_count() == launches + 1
  again = _host(eng.rollout(plans.clone()))
  assert eng.launch_count() == launches + 2
  after = _everything(eng)
  for k, v in before.items():
    assert np.array_equal(v, after[k], equal_nan=True), k
  for k in NAMES:
    assert np.array_equal(_bits(first[k]), _bits(again[k])), k
  # the engine goes on as its twin that never rolled out
  for a in acts[4:]:
    got, want = eng.step(a, raster), twin.step(a, twin_raster)
    for k in NAMES:
      assert torch.equal(getattr(got, k), getattr(want, k)), k
    assert torch.equal(got.frames, want.frames)
    eng.rollout(plans)
  eng.close()
  twin.close()


def _batched(sampler, refill, noise_scale=None):
  from spriteworld_b200 import action_spaces, environment
  from spriteworld_b200.configs.cobra import goal_finding_more_targets as cfgmod
  cfg = cfgmod.get_config('train')
  cfg['max_episode_length'] = 4
  cfg['action_space'] = action_spaces.SelectMove(scale=0.25, noise_scale=noise_scale)
  kw = dict(sampler='device', seed=11) if sampler == 'device' else dict(refill=refill)
  return environment.BatchedEnvironment(n_envs=64, pool_depth=6, rng=np.random.RandomState(2), **kw, **cfg)


@gpu
@pytest.mark.parametrize('sampler,refill', [('host', 'async'), ('host', 'sync'), ('device', None)])
def test_rollouts_leave_the_refill_alone(sampler, refill):
  env = _batched(sampler, refill)
  rng = np.random.RandomState(4)
  env.reset()
  for t in range(30):
    env.step(rng.uniform(0, 1, (64, 4)).astype(np.float32))
    if getattr(env, '_inflight', None) is not None:
      env._inflight['future'].result()          # the refill thread is idle from here on
    torch.cuda.synchronize()
    stats = env.refill_stats()
    book = (env._t, env._resets, env._safe_step, env._safe_resets)
    launches = env.engine.launch_count()
    for _ in range(3):
      r = env.rollout(rng.uniform(0, 1, (5, 64, 2, 4)))
    assert tuple(r.reward.shape) == (5, 64, 2) and r.discount.dtype == torch.float32
    assert env.refill_stats() == stats and book == (env._t, env._resets, env._safe_step, env._safe_resets)
    assert env.engine.launch_count() == launches + 3
  env.close()


@gpu
def test_rollouts_between_steps_of_a_noisy_device_sampled_run_change_no_timestep():
  runs = []
  for with_rollouts in (False, True):
    env = _batched('device', None, noise_scale=0.05)
    rng = np.random.RandomState(6)
    env.reset()
    steps = []
    for t in range(12):
      a = rng.uniform(0, 1, (64, 4)).astype(np.float32)
      plans = rng.uniform(0, 1, (3, 64, 2, 4)).astype(np.float32)
      if with_rollouts:
        env.rollout(plans)
      ts = env.step(a)
      steps.append({k: getattr(ts, k).cpu().numpy().copy() for k in ('step_type', 'reward', 'success', 'status')})
      steps[-1]['image'] = ts.observation['image'].cpu().numpy().copy()
    runs.append((steps, env._rng.get_state()))
    env.close()
  for a, b in zip(runs[0][0], runs[1][0]):
    for k in a:
      assert np.array_equal(a[k], b[k], equal_nan=True), k
  assert np.array_equal(runs[0][1][1], runs[1][1][1]) and runs[0][1][2:] == runs[1][1][2:]


# -- refusals -----------------------------------------------------------------------------------

@gpu
def test_refused_rollouts_enqueue_nothing():
  from spriteworld_b200 import constants, engine
  from tests.test_gpu_launch_checks import E, _assert_unchanged, _engine, _snapshot
  T, C = 3, 2
  for kind, dtype, good, bad_dtypes in (
      ('select_move', torch.float32, _native.DTYPE_F32, (_native.DTYPE_I32, _native.DTYPE_I64)),
      ('embodied', torch.int32, _native.DTYPE_I32, (_native.DTYPE_F32, _native.DTYPE_F64))):
    eng = _engine(kind)
    cols = 2 if kind == 'embodied' else 4
    acts = torch.zeros((T, E, C, cols), dtype=dtype, device=eng.device)
    eng.step(acts[0, :, 0].contiguous())
    res = eng.rollout(acts)
    out = _native.StepOut(res.reward.data_ptr(), res.step_type.data_ptr(), res.success.data_ptr(),
                          res.status.data_ptr())
    before = _snapshot(eng)
    ptr = ctypes.c_void_p(acts.data_ptr())

    def refused(match, actions=ptr, dt=good, n_steps=T, n_candidates=C, outputs=out):
      rc = eng._lib.swb_rollout(eng._h, actions, dt, n_steps, n_candidates,
                                ctypes.byref(outputs) if outputs is not None else None, eng._stream())
      assert rc != 0 and match in eng._lib.swb_last_error(), eng._lib.swb_last_error()
      _assert_unchanged(eng, before)

    refused(b'null', actions=None)
    refused(b'null', outputs=None)
    for field in ('reward', 'step_type', 'success', 'status'):
      holes = _native.StepOut(out.reward, out.step_type, out.success, out.status)
      setattr(holes, field, None)
      refused(b'every swb_step_out pointer', outputs=holes)
    for dt in bad_dtypes:
      refused(b'Embodied' if kind == 'embodied' else b'float32 or float64', dt=dt)
    for n in (0, -1, -2 ** 31):
      refused(b'>= 1', n_steps=n)
      refused(b'>= 1', n_candidates=n)
    # E = 4 envs: 2^29 steps x 1 candidate is one entry beyond the limit of 2^31 - 1 per call
    refused(b'entries per call', n_steps=2 ** 29, n_candidates=1)
    refused(b'entries per call', n_steps=1, n_candidates=2 ** 29)
    refused(b'entries per call', n_steps=2 ** 31 - 1, n_candidates=2 ** 31 - 1)
    # the same state is scored by a call that is not refused: one launch more
    assert eng._lib.swb_rollout(eng._h, ptr, good, T, C, ctypes.byref(out), eng._stream()) == 0
    assert _snapshot(eng)[1] == before[1] + 1
    with pytest.raises(ValueError):
      eng.rollout(acts[:, :, :, :1].contiguous())
    with pytest.raises(ValueError):
      eng.rollout(acts.transpose(0, 2))          # not contiguous
    with pytest.raises(ValueError):
      eng.rollout(acts.cpu())
    with pytest.raises(ValueError):
      eng.rollout(acts.to(torch.float64 if kind == 'embodied' else torch.int32))
    _assert_unchanged(eng, (before[0], before[1] + 1))
    eng.close()


# -- the returns mean what they say --------------------------------------------------------------

def _play(planner, n_envs=256, T=3, C=32, steps=20):
  """Mean return of the first episode of every env of goal_finding under random-shooting MPC: each
  step C plans of T clicks per env are sampled on the device (half of the clicks on a sprite), scored
  by one rollout, and the first action of the chosen plan is stepped."""
  wl, eng, _ = _c2(n_envs, 21, mel=steps)
  E, S = n_envs, wl.n_slots
  gen = torch.Generator(device=eng.device)
  gen.manual_seed(0)
  rows = torch.arange(E, device=eng.device)
  live = eng.state_tensors()
  eng.step(torch.zeros((E, 4), device=eng.device))               # FIRST
  ret = torch.zeros(E, dtype=torch.float64, device=eng.device)
  alive = torch.ones(E, dtype=torch.bool, device=eng.device)
  for _ in range(steps):
    plans = torch.rand((T, E, C, 4), device=eng.device, generator=gen)
    slot = torch.randint(0, S, (T, E, C), device=eng.device, generator=gen)
    on = torch.rand((T, E, C), device=eng.device, generator=gen) < 0.5
    for k, pos in ((0, live['pos_x']), (1, live['pos_y'])):
      at = pos.to(torch.float32)[rows[None, :, None], slot]
      plans[..., k] = torch.where(on, at, plans[..., k])
    returns = eng.rollout(plans).reward.sum(0)                    # (E, C)
    best = returns.argmax(1) if planner == 'mpc' else torch.zeros(E, dtype=torch.long, device=eng.device)
    res = eng.step(plans[0, rows, best].contiguous())
    ret += torch.where(alive, res.reward, torch.zeros_like(res.reward))
    alive &= res.step_type == _native.STEP_MID
  eng.close()
  assert not alive.any()
  return float(ret.mean().item())


@gpu
def test_random_shooting_with_rollout_returns_beats_ignoring_them():
  mpc, blind = _play('mpc'), _play('first')
  assert np.isfinite(mpc) and np.isfinite(blind) and mpc > blind, (mpc, blind)
