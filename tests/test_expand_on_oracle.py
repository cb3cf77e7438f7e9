"""CPU tier of rollouts from env records and of their leaves: BatchedEnvironment.expand,
BatchedEnvironment.rollout(states=...) and EnvStates.take, on the oracle-backed engine double
extended here with Engine.rollout's `states` and `leaves` (ExpandOracleEngine: BatchOracle over the
decoded roots, stepped T times, each plan's end state written into a copy of its root's record).

What runs on the host is under test: the argument checks, the shapes of what comes back, the
leaves' layout, signature and span class, that an expansion leaves the environment and its `rng`
alone, and the gather by device indices.  The kernel is tests/test_gpu_rollout_states.py's.
"""
import numpy as np
import pytest
import torch

from oracle import oracle
from spriteworld_b200 import _native
from spriteworld_b200 import engine as engine_lib
from tests import oracle_engine
from tests.test_env_states_on_oracle import StatesOracleEngine
from tests.test_rollout_on_oracle import RolloutOracleEngine

_Engine = engine_lib.Engine   # the device engine, for its host-side checks


def _set_field(data, n_slots, name, values):
  """Writes `values` (one per record) into field `name` of the (n, record_bytes) uint8 array."""
  for field, off, dtype, shape in engine_lib.record_layout(n_slots)[0]:
    if field == name:
      nbytes = dtype.itemsize * int(np.prod(shape, dtype=np.int64))
      data[:, off:off + nbytes] = np.ascontiguousarray(values, dtype).reshape(len(data), -1).view(np.uint8)


class ExpandOracleEngine(RolloutOracleEngine, StatesOracleEngine):
  """The oracle double with Engine.rollout's record roots and leaves."""

  def rollout(self, actions, out=None, states=None, leaves=None):
    if states is None and leaves is None:
      return super().rollout(actions, out)
    if states is not None and not isinstance(states, engine_lib.EnvStates):
      raise ValueError('states must be EnvStates')
    n = self.n_envs if states is None else len(states)
    engine_lib.action_dtype(self.action_kind, n, actions, plans=True)
    if states is not None:
      _Engine.check_states(self, states, n)
    roots = self.save_envs() if states is None else states
    a = np.ascontiguousarray(actions.numpy())
    T, _, C = a.shape[:3]
    if leaves is True:
      leaves = engine_lib.EnvStates(torch.zeros((n * C, self.record_bytes), dtype=torch.uint8), 1,
                                    self.signature, self.n_slots)
    elif leaves is not None:
      _Engine.check_states(self, leaves, n * C)
    out, res = engine_lib.rollout_outputs(out, T, n, C, self.device)
    h = roots.to_host()
    pool = oracle_engine.record_sprites(self, roots)[:, None]   # each root at its live positions
    sub = oracle.BatchOracle(self._cfg, self._tab, None, np.repeat(pool, C, 0))
    sub.step_count[:] = np.repeat(h['step_count'], C)
    sub.reset_next[:] = 0
    live = np.repeat(h['reset_next'] == 0, C)
    end_x, end_y = sub.cur['x'].copy(), sub.cur['y'].copy()
    end_count, end_last = sub.step_count.copy(), np.zeros(n * C, np.uint8)
    for name, pad in (('reward', 0.0), ('step_type', _native.STEP_NONE), ('success', 0), ('status', 0)):
      getattr(res, name).fill_(pad)
    for t in range(T):
      sub.step(a[t].reshape(n * C, -1))
      for name, got in (('reward', sub.reward), ('step_type', sub.step_type), ('success', sub.success),
                        ('status', sub.err)):
        getattr(res, name)[t].view(-1).numpy()[live] = got[live]
      end_x[live], end_y[live] = sub.cur['x'][live], sub.cur['y'][live]
      end_count[live] = sub.step_count[live]
      end_last[live] = sub.step_type[live] == _native.STEP_LAST
      live = live & (sub.step_type != _native.STEP_LAST)
    if leaves is not None:
      data = np.repeat(roots.data.numpy(), C, 0)
      moved = np.repeat(h['reset_next'] == 0, C)
      for name, v in (('pos_x', end_x), ('pos_y', end_y), ('step_count', end_count), ('reset_next', end_last)):
        part = data[moved]
        _set_field(part, self.n_slots, name, v[moved])
        data[moved] = part
      leaves.data.numpy()[:] = data
      leaves.span_class = roots.span_class
    res.leaves = leaves
    self._launches += 1
    return res


@pytest.fixture(autouse=True)
def _expand_engine(monkeypatch):
  oracle_engine.install(monkeypatch)
  monkeypatch.setattr(engine_lib, 'Engine', ExpandOracleEngine)


def _env(E=6, K=5, seed=3, max_episode_length=9, noise_scale=None):
  from spriteworld_b200 import action_spaces, environment
  from spriteworld_b200.configs.cobra import goal_finding_more_targets as cfgmod
  cfg = cfgmod.get_config('train')
  cfg['action_space'] = action_spaces.SelectMove(scale=0.25, motion_cost=0.1, noise_scale=noise_scale)
  cfg['max_episode_length'] = max_episode_length
  return environment.BatchedEnvironment(n_envs=E, pool_depth=K, rng=np.random.RandomState(seed),
                                        refill='sync', **cfg)


def _started(env, steps, seed):
  """env after reset(), `steps` random steps, and one env flagged to reset."""
  rng = np.random.RandomState(seed)
  env.reset()
  for _ in range(steps):
    env.step(rng.uniform(0, 1, (env.n_envs, 4)).astype(np.float32))
  env.engine._bo.reset_next[1] = 1
  return rng


def _same_rollout(a, b):
  for name in a._fields:
    assert np.array_equal(getattr(a, name).numpy(), getattr(b, name).numpy(), equal_nan=True), name


def test_expand_from_the_live_envs_matches_rollout_and_stepping():
  E, T, C = 6, 5, 3
  env = _env(E=E)
  rng = _started(env, 3, 1)
  plans = rng.uniform(0, 1, (T, E, C, 4))
  roots = env.save_envs()
  r, leaves = env.expand(plans)
  _same_rollout(r, env.rollout(plans))
  assert isinstance(leaves, engine_lib.EnvStates) and len(leaves) == E * C
  assert leaves.signature == roots.signature and leaves.span_class == roots.span_class
  # leaf e * C + c: the record after plan c's last live step from a load of root e
  live_steps = ((r.step_type.numpy() == _native.STEP_MID) | (r.step_type.numpy() == _native.STEP_LAST)).sum(0)
  want = np.repeat(roots.data.numpy(), C, 0).reshape(E, C, -1).copy()
  for c in range(C):
    env.load_envs(roots)
    for t in range(T):
      env.step(plans[t, :, c])
      done = live_steps[:, c] == t + 1
      want[done, c] = env.save_envs().data.numpy()[done]
  assert (live_steps[1] == 0).all()                       # the root about to reset is its own leaf
  assert np.array_equal(leaves.data.numpy(), want.reshape(E * C, -1))
  h = leaves.to_host()
  assert (h['reset_next'].reshape(E, C)[live_steps > 0] ==
          (r.step_type.numpy() == _native.STEP_LAST).any(0)[live_steps > 0]).all()
  env.close()


def test_rollout_from_records_equals_the_live_rollout_on_any_width():
  E, T, C = 6, 4, 2
  env = _env(E=E)
  rng = _started(env, 2, 2)
  plans = rng.uniform(0, 1, (T, E, C, 4)).astype(np.float32)
  roots = env.save_envs()
  _same_rollout(env.rollout(plans, states=roots), env.rollout(plans))
  launches = env.engine.launch_count()
  few = env.rollout(plans[:, [4, 2, 1]], states=roots[[4, 2, 1]])   # 3 roots on 6 envs
  assert tuple(few.reward.shape) == (T, 3, C) and env.engine.launch_count() == launches + 1
  full = env.rollout(plans)
  for name in few._fields:
    assert np.array_equal(getattr(few, name).numpy(), getattr(full, name).numpy()[:, [4, 2, 1]],
                          equal_nan=True), name
  many = engine_lib.EnvStates.cat([roots] * 3)                       # 18 roots on 6 envs
  r, leaves = env.expand(np.concatenate([plans] * 3, 1), states=many)
  assert tuple(r.reward.shape) == (T, 3 * E, C) and len(leaves) == 3 * E * C
  with pytest.raises(ValueError):
    env.rollout(plans, states=roots[:3])                             # plans of 6 roots, 3 roots
  env.close()


def test_expanding_a_leaf_continues_the_plan():
  """T1 + T2 steps of a plan equal T1 steps, then T2 steps from its leaf."""
  E, T1, T2 = 5, 2, 3
  env = _env(E=E, max_episode_length=30)
  rng = _started(env, 1, 3)
  plans = rng.uniform(0.3, 0.7, (T1 + T2, E, 1, 4))
  whole = env.rollout(plans)
  head, leaves = env.expand(plans[:T1])
  tail = env.rollout(plans[T1:], states=leaves)
  no_last = ~(head.step_type.numpy() == _native.STEP_LAST).any(0)[:, 0]
  for name in whole._fields:
    got = np.concatenate([getattr(head, name).numpy(), getattr(tail, name).numpy()])
    assert np.array_equal(got[:, no_last], getattr(whole, name).numpy()[:, no_last], equal_nan=True), name
  env.close()


def test_expand_changes_neither_the_environment_nor_its_rng():
  E, T, C = 4, 3, 2
  env = _env(E=E, noise_scale=0.05)
  rng = _started(env, 2, 4)
  state = (env._t, env._resets, env._safe_step, env.refill_stats(), env._rng.get_state()[1].copy())
  before = env.save_envs().data.clone()
  r, leaves = env.expand(rng.uniform(0, 1, (T, E, C, 4)))
  again = (env._t, env._resets, env._safe_step, env.refill_stats(), env._rng.get_state()[1])
  assert state[:4] == again[:4] and np.array_equal(state[4], again[4])
  assert torch.equal(env.save_envs().data, before)
  env.close()


def test_leaves_in_place_and_refusals():
  E, T, C = 4, 2, 3
  env, other = _env(E=E), _env(E=E, max_episode_length=10)
  rng = _started(env, 1, 5)
  other.reset()
  eng = env.engine
  plans = torch.from_numpy(rng.uniform(0, 1, (T, E, C, 4)))
  roots = env.save_envs()
  mine = engine_lib.EnvStates(torch.full((E * C, eng.record_bytes), 7, dtype=torch.uint8), 4,
                              roots.signature, roots.n_slots)
  res = eng.rollout(plans, states=roots, leaves=mine)
  assert res.leaves is mine and mine.span_class == roots.span_class
  assert torch.equal(mine.data, eng.rollout(plans, leaves=True).leaves.data)
  assert eng.rollout(plans).leaves is None and eng.rollout(plans, states=roots).leaves is None
  with pytest.raises(ValueError, match='another configuration'):
    eng.rollout(plans, states=other.save_envs())
  with pytest.raises(ValueError, match='another configuration'):
    env.expand(plans, states=other.save_envs())
  with pytest.raises(ValueError):
    eng.rollout(plans, states=roots.data)                             # not EnvStates
  with pytest.raises(ValueError):
    eng.rollout(plans, leaves=mine[:E * C - 1])                       # one leaf short
  with pytest.raises(ValueError, match='another configuration'):
    eng.rollout(plans, leaves=engine_lib.EnvStates(mine.data, 1, b'other', mine.n_slots))
  env.close()
  other.close()


def test_take_gathers_by_device_indices_and_zeroes_the_ones_outside():
  env = _env(E=6)
  _started(env, 2, 6)
  s = env.save_envs()
  n = len(s)
  for dtype in (torch.int32, torch.int64):
    idx = torch.tensor([5, 0, 0, -1, n, 2 ** 31 - 1 if dtype == torch.int32 else 2 ** 40, 3], dtype=dtype)
    got = s.take(idx)
    assert len(got) == len(idx) and got.signature == s.signature and got.span_class == s.span_class
    d = got.data.numpy()
    for i, j in enumerate(idx.tolist()):
      want = s.data.numpy()[j] if 0 <= j < n else np.zeros(s.record_bytes, np.uint8)
      assert np.array_equal(d[i], want), (dtype, i)
  assert len(s.take(torch.zeros(0, dtype=torch.int64))) == 0
  empty = s[0:0]
  assert np.array_equal(empty.take(torch.tensor([0, -3])).data.numpy(), np.zeros((2, s.record_bytes), np.uint8))
  zero = s.take(torch.tensor([-1]))
  env.load_envs(zero, [2])                                            # loads as an env of empty slots
  assert (env.save_envs([2]).to_host()['shape'] == 0).all()
  for bad in (torch.tensor([0.0, 1.0]), torch.tensor([[0, 1]]), [0, 1], np.array([0, 1]),
              torch.tensor([0, 1], dtype=torch.int16), torch.empty(2, dtype=torch.int64, device='meta')):
    with pytest.raises(ValueError):
      s.take(bad)
  env.close()
