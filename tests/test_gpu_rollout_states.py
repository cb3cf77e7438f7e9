"""Rollouts from env records and their leaves (csrc/swb_rollout.cuh, swb_rollout_states), bit for bit.

A rollout from records equals the rollout from the live envs the records were saved from; leaf
r * C + c equals, byte for byte, the saved record of an engine loaded from root r and stepped
through plan c's live steps (and the CPU oracle's state stepped from the decoded roots); a plan
continued from its leaf equals the longer plan.  Records roll out on engines of any width and pool
depth, nothing but the outputs and leaves is written, a call is one launch, refused calls enqueue
nothing, and a beam search runs level after level on the device without the host waiting.
"""
import ctypes

import numpy as np
import pytest
import torch

from spriteworld_b200 import _native
from tests.test_gpu_rollout import NAMES, SWEEP, _assert_rollout, _bits, _c2, _everything, _host

gpu = pytest.mark.gpu


def _t(eng, a):
  return torch.from_numpy(np.ascontiguousarray(a)).to(eng.device)


def _outputs_and_leaves(res):
  return _host(res), res.leaves.data.cpu().numpy().copy()


def _same(a, b, what):
  (oa, la), (ob, lb) = a, b
  for k in NAMES:
    assert np.array_equal(_bits(oa[k]), _bits(ob[k])), (what, k)
  assert np.array_equal(la, lb), (what, 'leaves')


def _stepped(roots, make_engine, plans):
  """(outputs (T, R, C) of T Engine.step calls on an engine of R x C envs loaded from the repeated
  roots, the mask of their live steps, the saved record of each plan after its last live step --
  its root if it has none)."""
  T, R, C = plans.shape[:3]
  rep = roots[np.repeat(np.arange(R), C)]
  big = make_engine(R * C)
  big.load_envs(rep)
  out = {k: [] for k in NAMES}
  saves = []
  for t in range(T):
    res = big.step(torch.from_numpy(np.ascontiguousarray(plans[t].reshape((R * C,) + plans.shape[3:]))).to(big.device))
    for k, v in _host(res).items():
      out[k].append(v.reshape(R, C))
    saves.append(big.save_envs().data.cpu().numpy().copy())
  big.close()
  out = {k: np.stack(v) for k, v in out.items()}
  st = out['step_type']
  lasts_before = np.cumsum(st == _native.STEP_LAST, 0) - (st == _native.STEP_LAST)
  started = np.cumsum(st == _native.STEP_FIRST, 0) > 0
  mask = (lasts_before == 0) & ~started
  n_live = mask.sum(0).reshape(-1)
  leaves = rep.data.cpu().numpy().copy()
  for i in np.nonzero(n_live)[0]:
    leaves[i] = saves[n_live[i] - 1][i]
  return out, mask, leaves


# -- 1, 2: roots from records equal live roots; leaves equal stepping ---------------------------

@gpu
@pytest.mark.parametrize('name', SWEEP)
def test_record_roots_and_leaves_match_live_roots_the_step_kernel_and_the_oracle(name):
  from spriteworld_b200 import constants, engine
  from tests import test_gpu_step_sweep as sweep
  from tests.test_gpu_env_states import _oracle_from_records
  case = next(c for c in sweep.CASES if c['name'] == name)
  arrs, nodes, action, acts = sweep._setup(case)
  eng = sweep._engine(case, nodes, arrs, action)
  E, mel = case['E'], case['mel']
  for a in acts[:3]:
    eng.step(_t(eng, a))
  rng = np.random.RandomState(len(name) + 1)
  count = rng.randint(0, mel, E).astype(np.int32)
  reset_next = eng.download_state()['reset_next'] | (rng.rand(E) < 0.1)
  eng.upload_state(step_count=count, reset_next=reset_next.astype(np.uint8))
  T, C = 8, 3
  plans = sweep.case_actions(case, arrs, rng, T * C)
  plans = np.ascontiguousarray(plans.reshape((T, C, E) + plans.shape[2:]).swapaxes(1, 2))
  pt = _t(eng, plans)
  roots = eng.save_envs()
  root_bytes = roots.data.clone()
  live = _outputs_and_leaves(eng.rollout(pt, leaves=True))
  rec = _outputs_and_leaves(eng.rollout(pt, states=roots, leaves=True))
  _same(live, rec, 'live roots')
  assert torch.equal(roots.data, root_bytes)
  plain = _host(eng.rollout(pt, states=roots))                    # no leaves: the same outputs
  _same((plain, rec[1]), rec, 'without leaves')

  def make_engine(n):
    return engine.Engine(n, case['S'], 1, action, nodes, constants.SHAPES, keep_in_frame=case['keep'],
                         max_episode_length=mel)

  want, mask, want_leaves = _stepped(roots, make_engine, plans)
  _assert_rollout(rec[0], want, mask, 'step kernel')
  assert np.array_equal(rec[1], want_leaves), 'leaves against stepping'
  h = engine.EnvStates(torch.from_numpy(rec[1]), 1, roots.signature, roots.n_slots).to_host()
  n_live = mask.sum(0).reshape(-1)
  root_rep = np.repeat(reset_next > 0, C)
  assert (n_live[root_rep] == 0).all() and (h['reset_next'][root_rep] == 1).all()   # own leaf
  if E >= 33:                   # plans that ended on a LAST inside the window
    assert (h['reset_next'][~root_rep] == 1).any()
  if E <= 300:                  # the CPU oracle, stepped from the decoded roots
    bo = _oracle_from_records(roots[np.repeat(np.arange(E), C)].to_host(), action, nodes, case['keep'], mel, None)
    ref = {k: [] for k in NAMES}
    ox, oy, oc = bo.cur['x'].copy(), bo.cur['y'].copy(), bo.step_count.copy()
    for t in range(T):
      bo.step(plans[t].reshape((E * C,) + plans.shape[3:]))
      for k, v in zip(NAMES, (bo.reward, bo.step_type, bo.success, bo.err)):
        ref[k].append(v.reshape(E, C).copy())
      m = mask[t].reshape(-1)
      ox[m], oy[m], oc[m] = bo.cur['x'][m], bo.cur['y'][m], bo.step_count[m]
    _assert_rollout(rec[0], {k: np.stack(v) for k, v in ref.items()}, mask, 'oracle', nan_bits=False)
    for k, v in (('pos_x', ox), ('pos_y', oy), ('step_count', oc)):
      assert np.array_equal(h[k], v), ('oracle leaves', k)
  eng.close()


# -- 3: composition ------------------------------------------------------------------------------

@gpu
def test_a_plan_continued_from_its_leaf_equals_the_longer_plan():
  E, T1, T2, C = 300, 3, 5, 8
  wl, eng, _ = _c2(E, 13, mel=12)
  rng = np.random.RandomState(5)
  for a in wl.sample_actions(rng, 2, E):
    eng.step(_t(eng, a))
  eng.upload_state(step_count=rng.randint(0, 12, E).astype(np.int32))   # timeouts at every t
  plans = rng.uniform(0, 1, (T1 + T2, E, C, 4)).astype(np.float32)
  whole = _host(eng.rollout(_t(eng, plans)))
  head = eng.rollout(_t(eng, plans[:T1]), leaves=True)
  tail = eng.rollout(_t(eng, plans[T1:].reshape(T2, E * C, 1, 4)), states=head.leaves)
  head, tail = _host(head), _host(tail)
  ended = (head['step_type'] == _native.STEP_LAST).any(0)
  assert ended.any() and (~ended).any()
  for k in NAMES:                # a plan that ended in its first T1 steps continues as padding
    got = np.concatenate([head[k], tail[k].reshape(T2, E, C)])
    assert np.array_equal(_bits(got), _bits(whole[k])), k
  eng.close()


# -- 4: width and engines ------------------------------------------------------------------------

@gpu
def test_records_roll_out_on_an_engine_of_any_width_and_pool_depth():
  E, T, C = 4096, 5, 4
  wl, eng, _ = _c2(E, 17, mel=20, pool_depth=3)
  _, small, _ = _c2(4, 18, mel=20, pool_depth=5)
  rng = np.random.RandomState(7)
  for a in wl.sample_actions(rng, 3, E):
    eng.step(_t(eng, a))
  roots = eng.save_envs()
  plans = _t(eng, rng.uniform(0, 1, (T, E, C, 4)).astype(np.float32))
  own = _outputs_and_leaves(eng.rollout(plans, leaves=True))
  before = _everything(small)
  res = small.rollout(plans, states=roots, leaves=True)
  assert res.leaves.span_class == roots.span_class and res.leaves.signature == roots.signature
  _same(_outputs_and_leaves(res), own, '4096 records on 4 envs')
  after = _everything(small)
  for k, v in before.items():
    assert np.array_equal(v, after[k], equal_nan=True), k
  eng.close()
  small.close()


# -- 5: read-only, one launch --------------------------------------------------------------------

@gpu
def test_record_rollouts_change_nothing_and_are_one_launch():
  from tests.test_gpu_rollout import _batched
  wl, eng, raster = _c2(300, 7)
  rng = np.random.RandomState(3)
  for a in wl.sample_actions(rng, 4, 300):
    eng.step(_t(eng, a), raster)
  roots = eng.save_envs()[::3]
  root_bytes = roots.data.clone()
  plans = _t(eng, rng.uniform(0, 1, (6, len(roots), 4, 4)))
  live_plans = _t(eng, rng.uniform(0, 1, (6, 300, 4, 4)))
  before, launches = _everything(eng), eng.launch_count()
  for i, (p, kw) in enumerate(((plans, dict(states=roots)), (plans, dict(states=roots, leaves=True)),
                               (live_plans, dict(leaves=True)))):
    eng.rollout(p, **kw)
    assert eng.launch_count() == launches + i + 1, kw
  after = _everything(eng)
  for k, v in before.items():
    assert np.array_equal(v, after[k], equal_nan=True), k
  assert torch.equal(roots.data, root_bytes)
  eng.close()
  env = _batched('device', None)
  env.reset()
  for _ in range(5):
    env.step(rng.uniform(0, 1, (64, 4)).astype(np.float32))
  torch.cuda.synchronize()
  stats, book = env.refill_stats(), (env._t, env._resets, env._safe_step, env._safe_resets)
  state, launches = env.engine.download_state(), env.engine.launch_count()
  r, leaves = env.expand(rng.uniform(0, 1, (3, 64, 2, 4)))
  r2, leaves2 = env.expand(rng.uniform(0, 1, (3, 128, 2, 4)), states=leaves)
  assert tuple(r2.reward.shape) == (3, 128, 2) and len(leaves2) == 256
  assert env.engine.launch_count() == launches + 2
  assert env.refill_stats() == stats and book == (env._t, env._resets, env._safe_step, env._safe_resets)
  for k, v in env.engine.download_state().items():
    assert np.array_equal(v, state[k]), k
  env.close()


# -- 6: refusals ---------------------------------------------------------------------------------

@gpu
def test_refused_record_rollouts_enqueue_nothing():
  from spriteworld_b200 import constants, engine
  from tests.test_gpu_launch_checks import E, _assert_unchanged, _engine, _snapshot
  T, C = 3, 2
  eng = _engine()
  acts = torch.zeros((T, E, C, 4), dtype=torch.float32, device=eng.device)
  eng.step(acts[0, :, 0].contiguous())
  roots = eng.save_envs()
  rb = eng.record_bytes
  buf = torch.zeros((E * C + E + 1) * rb, dtype=torch.uint8, device=eng.device)   # room to overlap
  res = eng.rollout(acts)
  out = _native.StepOut(res.reward.data_ptr(), res.step_type.data_ptr(), res.success.data_ptr(),
                        res.status.data_ptr())
  before = _snapshot(eng)
  span = ctypes.c_int32(-5)
  R = roots.data.data_ptr()
  L = buf.data_ptr()

  def call(roots=R, n_roots=E, roots_bytes=E * rb, actions=acts.data_ptr(), dt=_native.DTYPE_F32,
           n_steps=T, n_candidates=C, outputs=out, leaves=L, leaves_bytes=E * C * rb, engine=eng._h):
    return eng._lib.swb_rollout_states(engine, roots, n_roots, roots_bytes, actions, dt, n_steps, n_candidates,
                                       ctypes.byref(outputs) if outputs is not None else None, leaves,
                                       leaves_bytes, ctypes.byref(span), eng._stream())

  def refused(match, **kw):
    assert call(**kw) != 0 and match in eng._lib.swb_last_error(), (kw, eng._lib.swb_last_error())
    _assert_unchanged(eng, before)
    assert span.value == -5

  refused(b'null', engine=None)
  refused(b'null', actions=None)
  refused(b'null', outputs=None)
  refused(b'float32 or float64', dt=_native.DTYPE_I32)
  for n in (0, -1):
    refused(b'>= 1', n_steps=n)
    refused(b'>= 1', n_candidates=n)
    refused(b'n_roots', n_roots=n)
  refused(b'n_roots', roots=None, n_roots=E + 1)                  # live roots: n_roots must be E
  refused(b'entries per call', n_roots=2 ** 30, n_candidates=2, n_steps=1)    # 2^31 plans
  refused(b'entries per call', n_roots=2 ** 29, n_candidates=2, n_steps=2)
  refused(b'entries per call', n_roots=2 ** 31 - 1, n_candidates=2 ** 31 - 1)
  refused(b'roots is not 16-byte aligned', roots=R + 8)
  refused(b'records need', roots_bytes=E * rb - 1)
  refused(b'leaves is not 16-byte aligned', leaves=L + 4)
  refused(b'records need', leaves_bytes=E * C * rb - 1)
  refused(b'overlap', leaves=R, leaves_bytes=E * C * rb)           # the same buffer
  refused(b'overlap', roots=L + (E * C - 1) * rb)                 # roots from the last leaf on
  refused(b'overlap', roots=L, leaves=L + (E - 1) * rb)           # leaves from the last root on

  def outputs(**kw):   # `out` with some arrays replaced by pointers
    ptrs = dict(reward=out.reward, step_type=out.step_type, success=out.success, status=out.status)
    return _native.StepOut(**dict(ptrs, **kw))
  refused(b'reward is not 8-byte aligned', outputs=outputs(reward=out.reward + 4))
  refused(b'leaves overlaps status', outputs=outputs(status=L + (E * C - 1) * rb))
  refused(b'success overlaps the roots', outputs=outputs(success=R + E * rb - 1))
  refused(b'status overlaps step_type', outputs=outputs(status=out.step_type + T * E * C - 1))
  assert call(roots=L + E * C * rb) == 0 and span.value == -5     # adjacent: accepted
  assert call(roots=None) == 0 and span.value == roots.span_class  # live roots: the engine's
  assert _snapshot(eng)[1] == before[1] + 2
  other = engine.Engine(E, 2, 1, dict(kind='select_move', scale=0.05), [dict(kind='no_reward')],
                        constants.SHAPES, max_episode_length=77)
  with pytest.raises(ValueError, match='another configuration'):
    eng.rollout(acts, states=other.save_envs())
  with pytest.raises(ValueError, match='another configuration'):
    eng.rollout(acts, leaves=other.save_envs(list(range(E)) * C))
  with pytest.raises(ValueError):
    eng.rollout(acts[:, :3].contiguous(), states=roots)             # plans of 3 roots, 4 roots
  with pytest.raises(ValueError):
    eng.rollout(acts, leaves=roots)                                 # E records, E x C plans
  _assert_unchanged(eng, (before[0], before[1] + 2))
  other.close()
  eng.close()


# -- 7: a beam search on the device --------------------------------------------------------------

def _level_return(reward):
  """Sum over t of (T, n, C) rewards, left to right, as the replay below adds them."""
  ret = reward[0]
  for t in range(1, reward.shape[0]):
    ret = ret + reward[t]
  return ret


@gpu
def test_device_beam_search_enqueues_without_the_host_and_claims_true_returns():
  from spriteworld_b200 import action_spaces, environment
  from spriteworld_b200.configs.cobra import goal_finding_more_targets as cfgmod
  E, B, C, D, T = 64, 4, 16, 3, 2
  cfg = cfgmod.get_config('train')
  cfg['max_episode_length'] = 7        # two steps before the search: timeouts inside it
  cfg['action_space'] = action_spaces.SelectMove(scale=0.5)
  env = environment.BatchedEnvironment(n_envs=E, pool_depth=4, sampler='device', seed=3, **cfg)
  env.reset()
  rng = np.random.RandomState(2)
  for _ in range(2):
    env.step(rng.uniform(0, 1, (E, 4)).astype(np.float32))
  dev = env.engine.device
  roots = env.save_envs()
  gen = torch.Generator(device=dev)

  def search():
    gen.manual_seed(1)
    frontier, width = roots, 1
    score = torch.zeros(E, dtype=torch.float64, device=dev)
    picked = []                                       # per level: (leaf index, plans)
    for _ in range(D):
      plans = torch.rand((T, E * width, C, 4), device=dev, generator=gen)
      r, leaves = env.expand(plans, states=frontier)
      total = (score[:, None] + _level_return(r.reward)).view(E, width * C)
      score, best = total.topk(B, dim=1)              # per env, over its width x C children
      leaf = (best + torch.arange(E, device=dev)[:, None] * (width * C)).view(-1)
      frontier, width = leaves.take(leaf), B
      score = score.reshape(-1)
      picked.append((leaf, plans))
    return score, picked

  search()                  # loads every kernel it uses: a kernel's first launch may wait
  torch.cuda.synchronize()
  launches = env.engine.launch_count()
  torch.cuda._sleep(1 << 31)                          # about a second of device time
  score, picked = search()
  done = torch.cuda.Event()
  done.record()
  assert not done.query()                             # everything above was enqueued while busy
  assert env.engine.launch_count() == launches + D
  torch.cuda.synchronize()
  # the best beam of every env: follow its leaves back to the root, collecting the plans' actions
  score = score.view(E, B)
  beam = score.argmax(1).cpu().numpy() + np.arange(E) * B
  claimed = score.view(-1).cpu().numpy()[beam]
  actions = []
  for leaf, plans in reversed(picked):
    i = leaf.cpu().numpy()[beam]
    actions.append(plans.cpu().numpy()[:, i // C, i % C])
    beam = i // C
  assert np.array_equal(beam, np.arange(E))
  actions = np.concatenate(actions[::-1])           # (D * T, E, 4)
  # replay with Engine.step on the engine loaded from the roots, counting rewards up to the first
  # LAST, summed in the order the search summed them
  eng = env.engine
  eng.load_envs(roots)
  got = np.zeros(E)
  alive = np.ones(E, bool)
  for d in range(D):
    ret = []
    for t in range(T):
      res = eng.step(torch.from_numpy(np.ascontiguousarray(actions[d * T + t])).to(dev))
      ret.append(np.where(alive, res.reward.cpu().numpy(), 0.0))
      alive &= res.step_type.cpu().numpy() == _native.STEP_MID
    got = got + _level_return(np.stack(ret))
  assert not alive.all()                              # beams that ended inside the search
  assert np.array_equal(got.view(np.int64), claimed.view(np.int64)), (got, claimed)
  env.close()
