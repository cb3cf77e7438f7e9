"""CPU tier of rollout trajectories: BatchedEnvironment.rollout_trajectory and Engine.rollout's
`trajectory`, on the oracle-backed engine double extended here (TrajectoryOracleEngine: record
(t * n + r) * C + c is the double's own leaf r * C + c of the rollout of actions[:t + 1]).

What runs on the host is under test: the shapes and the record index of what comes back, the
signature and span class, that the last slice is expand's leaves, that a trajectory leaves the
environment, its rings and its `rng` alone, and that every refusal is raised before anything is
enqueued.  The kernel is tests/test_gpu_trajectory.py's.
"""
import numpy as np
import pytest
import torch

from spriteworld_b200 import _native
from spriteworld_b200 import engine as engine_lib
from tests import oracle_engine
from tests.test_expand_on_oracle import ExpandOracleEngine, _env, _same_rollout, _started

_Engine = engine_lib.Engine   # the device engine, for its host-side checks


class TrajectoryOracleEngine(ExpandOracleEngine):
  """The expand double with Engine.rollout's `trajectory`, built from the double's own leaves."""

  def rollout(self, actions, out=None, states=None, leaves=None, trajectory=None):
    if trajectory is None:
      return super().rollout(actions, out, states, leaves)
    if leaves is not None:
      raise ValueError('trajectory and leaves are exclusive')
    n = self.n_envs if states is None else len(states)
    engine_lib.action_dtype(self.action_kind, n, actions, plans=True)
    if states is not None:
      _Engine.check_states(self, states, n)
    T, _, C = actions.shape[:3]
    if trajectory is True:
      trajectory = engine_lib.EnvStates(torch.zeros((T * n * C, self.record_bytes), dtype=torch.uint8), 1,
                                        self.signature, self.n_slots)
    else:
      _Engine.check_states(self, trajectory, T * n * C)
    launches = self._launches
    for t in range(T):
      res = super().rollout(actions[:t + 1].contiguous(), out if t == T - 1 else None, states, True)
      trajectory.data[t * n * C:(t + 1) * n * C] = res.leaves.data
    trajectory.span_class = res.leaves.span_class
    res.leaves, res.trajectory = None, trajectory
    self._launches = launches + 1
    return res


@pytest.fixture(autouse=True)
def _trajectory_engine(monkeypatch):
  oracle_engine.install(monkeypatch)
  monkeypatch.setattr(engine_lib, 'Engine', TrajectoryOracleEngine)


def test_trajectory_is_every_prefix_leaf_and_its_last_slice_is_the_leaves():
  E, T, C = 6, 5, 3
  env = _env(E=E, max_episode_length=7)
  rng = _started(env, 3, 1)
  plans = rng.uniform(0, 1, (T, E, C, 4))
  roots = env.save_envs()
  launches = env.engine.launch_count()
  r, traj = env.rollout_trajectory(plans)
  assert env.engine.launch_count() == launches + 1
  _same_rollout(r, env.rollout(plans))
  assert isinstance(traj, engine_lib.EnvStates) and len(traj) == T * E * C
  assert traj.signature == roots.signature and traj.span_class == roots.span_class
  data = traj.data.numpy().reshape(T, E, C, -1)
  for t in range(T):
    _, leaves = env.expand(plans[:t + 1])
    assert np.array_equal(data[t].reshape(E * C, -1), leaves.data.numpy()), t
  _, leaves = env.expand(plans)
  assert np.array_equal(traj[(T - 1) * E * C:].data.numpy(), leaves.data.numpy())
  # record (t * E + e) * C + c: the state after step t of plan c from env e
  h = traj.to_host()
  st = r.step_type.numpy()
  live = (st == _native.STEP_MID) | (st == _native.STEP_LAST)
  n_live = np.cumsum(live, 0)
  count0 = roots.to_host()['step_count']
  assert np.array_equal(h['step_count'].reshape(T, E, C), count0[None, :, None] + n_live)
  ended = np.cumsum(st == _native.STEP_LAST, 0) > 0
  assert np.array_equal(h['reset_next'].reshape(T, E, C)[:, [0, 2, 3, 4, 5]], ended[:, [0, 2, 3, 4, 5]])
  assert (h['reset_next'].reshape(T, E, C)[:, 1] == 1).all()           # the root about to reset
  assert ended.any() and (~ended[-1]).any()
  for t in range(T):                                                    # its own record at every t
    assert np.array_equal(data[t, 1], np.repeat(roots.data.numpy()[1:2], C, 0))
  env.close()


def test_trajectory_from_records_matches_the_live_roots_on_any_width():
  E, T, C = 6, 4, 2
  env = _env(E=E)
  rng = _started(env, 2, 2)
  plans = rng.uniform(0, 1, (T, E, C, 4)).astype(np.float32)
  roots = env.save_envs()
  r_live, live = env.rollout_trajectory(plans)
  r_rec, rec = env.rollout_trajectory(plans, states=roots)
  _same_rollout(r_live, r_rec)
  assert torch.equal(live.data, rec.data)
  # narrow, then trace: the chosen plans of 3 roots, C = 1
  idx = torch.tensor([4, 2, 1])
  best = torch.from_numpy(plans[:, [4, 2, 1], 1:2].copy())
  r3, few = env.rollout_trajectory(best, states=roots.take(idx))
  assert tuple(r3.reward.shape) == (T, 3, 1) and len(few) == T * 3
  want = live.data.numpy().reshape(T, E, C, -1)[:, [4, 2, 1], 1]
  assert np.array_equal(few.data.numpy().reshape(T, 3, -1), want)
  many = engine_lib.EnvStates.cat([roots] * 3)                          # 18 roots on 6 envs
  r18, traj18 = env.rollout_trajectory(np.concatenate([plans] * 3, 1), states=many)
  assert tuple(r18.reward.shape) == (T, 3 * E, C) and len(traj18) == T * 3 * E * C
  env.close()


def test_trajectory_changes_neither_the_environment_nor_its_rng():
  E, T, C = 4, 3, 2
  env = _env(E=E, noise_scale=0.05)
  rng = _started(env, 2, 4)
  state = (env._t, env._resets, env._safe_step, env.refill_stats(), env._rng.get_state()[1].copy())
  before = env.save_envs().data.clone()
  pool = {k: v.clone() for k, v in env.engine.pool_tensors().items()}
  plans = rng.uniform(0, 1, (T, E, C, 4))
  r, traj = env.rollout_trajectory(plans)
  r2, traj2 = env.rollout_trajectory(plans)                              # no noise: the same twice
  _same_rollout(r, r2)
  assert torch.equal(traj.data, traj2.data)
  again = (env._t, env._resets, env._safe_step, env.refill_stats(), env._rng.get_state()[1])
  assert state[:4] == again[:4] and np.array_equal(state[4], again[4])
  assert torch.equal(env.save_envs().data, before)
  for k, v in env.engine.pool_tensors().items():
    assert torch.equal(v, pool[k]), k
  env.close()


def test_trajectory_in_place_and_refusals_before_anything_is_enqueued():
  E, T, C = 4, 2, 3
  env, other = _env(E=E), _env(E=E, max_episode_length=10)
  rng = _started(env, 1, 5)
  other.reset()
  eng = env.engine
  plans = torch.from_numpy(rng.uniform(0, 1, (T, E, C, 4)))
  roots = env.save_envs()
  mine = engine_lib.EnvStates(torch.full((T * E * C, eng.record_bytes), 7, dtype=torch.uint8), 4,
                              roots.signature, roots.n_slots)
  res = eng.rollout(plans, states=roots, trajectory=mine)
  assert res.trajectory is mine and res.leaves is None and mine.span_class == roots.span_class
  assert torch.equal(mine.data, eng.rollout(plans, trajectory=True).trajectory.data)
  assert eng.rollout(plans).trajectory is None and eng.rollout(plans, leaves=True).trajectory is None
  before, launches = env.save_envs().data.clone(), eng.launch_count()
  bad = [
      dict(trajectory=True, leaves=True),                                          # exclusive
      dict(trajectory=mine, leaves=True),
      dict(trajectory=mine[:T * E * C - 1]),                                       # one record short
      dict(trajectory=engine_lib.EnvStates(mine.data, 1, b'other', mine.n_slots)),  # another engine's
      dict(trajectory=mine.data),                                                  # not EnvStates
      dict(trajectory=True, states=other.save_envs()),
      dict(trajectory=True, states=roots.data),
      dict(trajectory=True, states=roots[:3]),                                     # plans of 4 roots
  ]
  for kw in bad:
    with pytest.raises(ValueError):
      eng.rollout(plans, **kw)
  for a in (plans[:, :, :0], plans[:0], plans[..., :3], plans.to(torch.int32)):  # C or T < 1, columns, dtype
    with pytest.raises(ValueError):
      eng.rollout(a, trajectory=True)
    with pytest.raises(ValueError):
      env.rollout_trajectory(a)
  with pytest.raises(ValueError, match='another configuration'):
    env.rollout_trajectory(plans, states=other.save_envs())
  assert eng.launch_count() == launches
  assert torch.equal(env.save_envs().data, before)
  env.close()
  other.close()
