"""CPU tier of BatchedEnvironment.rollout, on the oracle-backed engine double extended here with
`rollout` (RolloutOracleEngine, built from BatchOracle on copies of the live state).

What runs on the host is under test: the action conversion and the shape and dtype checks, the
shapes, dtypes and padding of what comes back, the discount, and that a rollout leaves the
environment's bookkeeping and its `rng` alone.  The kernel is tests/test_gpu_rollout.py's.
"""
import numpy as np
import pytest
import torch

from oracle import oracle
from spriteworld_b200 import _native
from spriteworld_b200 import engine as engine_lib
from tests import oracle_engine


class RolloutOracleEngine(oracle_engine.OracleEngine):
  """The oracle double with Engine.rollout: every (env, candidate) is an env of a BatchOracle over a
  one-scene pool, a copy of the live state, stepped T times; entries after a plan's first LAST, and
  every entry of an env about to reset, are padding."""

  def rollout(self, actions, out=None):
    engine_lib.action_dtype(self.action_kind, self.n_envs, actions, plans=True)
    a = np.ascontiguousarray(actions.numpy())
    T, E, C = a.shape[:3]
    out, res = engine_lib.rollout_outputs(out, T, E, C, self.device)
    bo = self._bo
    pool = np.repeat(bo.pool[np.arange(E), bo.cursor], C, 0)[:, None]
    sub = oracle.BatchOracle(self._cfg, self._tab, None, pool)
    sub.cur[:] = np.repeat(bo.cur, C, 0)
    sub.step_count[:] = np.repeat(bo.step_count, C)
    sub.reset_next[:] = 0
    live = np.repeat(bo.reset_next == 0, C)
    for name, pad in (('reward', 0.0), ('step_type', _native.STEP_NONE), ('success', 0), ('status', 0)):
      getattr(res, name).fill_(pad)
    for t in range(T):
      sub.step(a[t].reshape(E * C, -1))
      for name, got in (('reward', sub.reward), ('step_type', sub.step_type), ('success', sub.success),
                        ('status', sub.err)):
        getattr(res, name)[t].view(-1).numpy()[live] = got[live]
      live = live & (sub.step_type != _native.STEP_LAST)
    self._launches += 1
    return res


@pytest.fixture(autouse=True)
def _oracle_engine(monkeypatch):
  oracle_engine.install(monkeypatch)
  monkeypatch.setattr(engine_lib, 'Engine', RolloutOracleEngine)


def _env(E=6, K=5, seed=3, max_episode_length=20, noise_scale=None, embodied=False):
  from spriteworld_b200 import action_spaces, environment
  if embodied:
    from spriteworld_b200.configs.examples import goal_finding_embodied as cfgmod
    cfg = cfgmod.get_config('train')
  else:
    from spriteworld_b200.configs.cobra import goal_finding_more_targets as cfgmod
    cfg = cfgmod.get_config('train')
    cfg['action_space'] = action_spaces.SelectMove(scale=0.25, motion_cost=0.1, noise_scale=noise_scale)
  cfg['max_episode_length'] = max_episode_length
  return environment.BatchedEnvironment(n_envs=E, pool_depth=K, rng=np.random.RandomState(seed),
                                        refill='sync', **cfg)


def _is_padding(r, where):
  return ((r.step_type.numpy()[where] == _native.STEP_NONE).all() and (r.reward.numpy()[where] == 0).all()
          and (r.success.numpy()[where] == 0).all() and (r.status.numpy()[where] == 0).all()
          and (r.discount.numpy()[where] == 0).all())


def test_shapes_dtypes_padding_and_timeout_from_the_own_step_count():
  E, T, C, mel = 6, 9, 3, 7
  env = _env(E=E, max_episode_length=mel)
  rng = np.random.RandomState(0)
  plans = rng.uniform(0, 1, (T, E, C, 4)).astype(np.float32)
  # before the first reset every env is about to reset: nothing to plan in
  r = env.rollout(plans)
  assert _is_padding(r, np.ones((T, E, C), bool))
  env.reset()
  for _ in range(3):                       # step_count 3: four steps left of the seven
    ts = env.step(rng.uniform(0, 1, (E, 4)).astype(np.float32))
  live_env = ts.step_type.numpy() != _native.STEP_LAST
  assert live_env.any()
  r = env.rollout(plans)
  for name, dtype in (('reward', torch.float64), ('step_type', torch.int8), ('success', torch.uint8),
                      ('status', torch.uint8), ('discount', torch.float32)):
    t = getattr(r, name)
    assert t.dtype == dtype and tuple(t.shape) == (T, E, C), name
  st = r.step_type.numpy()
  assert _is_padding(r, np.broadcast_to(~live_env[None, :, None], st.shape))
  n_live = ((st == _native.STEP_MID) | (st == _native.STEP_LAST)).sum(0)
  assert (n_live[live_env] <= mel - 3).all() and (n_live[live_env] == mel - 3).any()
  assert (n_live[live_env] >= 1).all()
  for e in np.nonzero(live_env)[0]:
    for c in range(C):
      n = n_live[e, c]
      assert (st[:n - 1, e, c] == _native.STEP_MID).all() and st[n - 1, e, c] == _native.STEP_LAST
      assert (r.discount.numpy()[:n - 1, e, c] == 1).all() and r.discount.numpy()[n - 1, e, c] == 0
      assert _is_padding(r, (slice(n, None), e, c))
  # the first step of every candidate is the step the env would take
  ts = env.step(plans[0, :, 1])
  assert np.array_equal(ts.reward.numpy()[live_env].view(np.int64),
                        r.reward.numpy()[0, :, 1][live_env].view(np.int64))
  assert np.array_equal(ts.step_type.numpy()[live_env], st[0, :, 1][live_env])
  env.close()


def test_rollout_follows_steps_of_a_twin_environment():
  """Entry [t, e, c] is what the t-th step with candidate c's actions reports."""
  E, T, C = 5, 6, 2
  rng = np.random.RandomState(1)
  plans = rng.uniform(0, 1, (T, E, C, 4))           # float64
  envs = [_env(E=E, seed=11, max_episode_length=5) for _ in range(C + 1)]
  for env in envs:
    env.reset()
    env.step(np.full((E, 4), 0.5))
  r = envs[C].rollout(torch.from_numpy(plans))
  for c in range(C):
    live = np.ones(E, bool)
    for t in range(T):
      ts = envs[c].step(plans[t, :, c])
      for name in ('reward', 'step_type', 'success', 'status', 'discount'):
        assert np.array_equal(getattr(ts, name).numpy()[live], getattr(r, name).numpy()[t, :, c][live],
                              equal_nan=True), (name, t, c)
      live &= ts.step_type.numpy() != _native.STEP_LAST
      if t + 1 < T:
        assert _is_padding(r, (t + 1, ~live, c))
  for env in envs:
    env.close()


def _timesteps(noise_scale, with_rollouts, embodied=False):
  E = 4
  np.random.seed(17)     # whatever the config draws from the global generator
  env = _env(E=E, seed=5, max_episode_length=6, noise_scale=noise_scale, embodied=embodied)
  rng = np.random.RandomState(2)

  def host(ts):          # a timestep's tensors are views the next step overwrites
    return {k: (getattr(ts, k).numpy().copy() if k != 'observation' else ts.observation['image'].numpy().copy())
            for k in ts._fields}

  out = [host(env.reset())]
  for t in range(15):
    if embodied:
      a = np.stack([rng.randint(0, 2, E), rng.randint(0, 4, E)], -1)
      plans = np.stack([rng.randint(0, 2, (3, E, 2)), rng.randint(0, 5, (3, E, 2))], -1)
    else:
      a = rng.uniform(0, 1, (E, 4)).astype(np.float32)
      plans = rng.uniform(0, 1, (3, E, 2, 4))
    if with_rollouts:
      state = (env._t, env._resets, env._safe_step, env.refill_stats(), env.engine.download_state())
      env.rollout(plans)
      again = (env._t, env._resets, env._safe_step, env.refill_stats(), env.engine.download_state())
      assert state[:4] == again[:4]
      for k, v in state[4].items():
        assert np.array_equal(v, again[4][k]), k
    out.append(host(env.step(a)))
  rng_state = env._rng.get_state()
  env.close()
  assert len({ts['step_type'].tobytes() for ts in out}) > 2      # episodes ended and restarted
  return out, rng_state


@pytest.mark.parametrize('embodied', [False, True], ids=['noisy_select_move', 'embodied'])
def test_rollouts_between_steps_change_neither_the_timesteps_nor_the_rng(embodied):
  plain, rng_plain = _timesteps(0.05, False, embodied)
  mixed, rng_mixed = _timesteps(0.05, True, embodied)
  for a, b in zip(plain, mixed):
    for k in a:
      assert np.array_equal(a[k], b[k], equal_nan=True), k
  assert rng_plain[0] == rng_mixed[0] and np.array_equal(rng_plain[1], rng_mixed[1])
  assert rng_plain[2:] == rng_mixed[2:]


def test_embodied_bad_direction_goes_on():
  E, T, C = 3, 4, 2
  env = _env(E=E, embodied=True)
  env.reset()
  plans = np.zeros((T, E, C, 2), np.int64)
  plans[1, :, 0, 1] = 7                    # a direction the reference raises KeyError for
  r = env.rollout(plans)
  assert (r.status.numpy()[1, :, 0] == _native.ENV_BAD_ACTION).all()
  assert np.isnan(r.reward.numpy()[1, :, 0]).all()
  assert (r.step_type.numpy()[1:3, :, 0] == _native.STEP_MID).all()
  assert (r.status.numpy()[:, :, 1] == 0).all() and not np.isnan(r.reward.numpy()[2:, :, 0]).any()
  env.close()


def test_rejected_inputs():
  E = 4
  env = _env(E=E)
  env.reset()
  z = lambda *shape: np.zeros(shape, np.float32)
  for bad in (z(E, 4), z(3, E, 4), z(2, 3, E, 2, 4),     # wrong rank
              z(3, E + 1, 2, 4),                          # wrong n_envs
              z(3, E, 2, 3), z(3, E, 2, 2),               # wrong columns
              z(0, E, 2, 4), z(3, E, 0, 4)):              # T = 0, C = 0
    with pytest.raises(ValueError):
      env.rollout(bad)
    with pytest.raises(ValueError):
      env.rollout(torch.from_numpy(bad))
  with pytest.raises(ValueError):
    env.rollout(torch.zeros((3, E, 2, 4), dtype=torch.float16))
  env.rollout(z(3, E, 2, 4))
  env.close()
  emb = _env(E=E, embodied=True)
  emb.reset()
  with pytest.raises(ValueError):
    emb.rollout(torch.zeros((3, E, 2, 2), dtype=torch.float32))   # float actions for Embodied
  with pytest.raises(ValueError):
    emb.rollout(torch.zeros((3, E, 2, 2), dtype=torch.int64))
  with pytest.raises(ValueError):
    emb.rollout(np.zeros((3, E, 2, 4), np.int32))
  emb.rollout(torch.zeros((3, E, 2, 2), dtype=torch.int32))
  emb.close()


def test_packed_output_buffer():
  from spriteworld_b200 import engine as engine_lib
  E, T, C = 4, 3, 2
  env = _env(E=E)
  env.reset()
  a = torch.rand((T, E, C, 4), dtype=torch.float64)
  want = env.engine.rollout(a)
  buf = torch.zeros(T * E * C * engine_lib.OUT_BYTES_PER_ENV, dtype=torch.uint8)
  got = env.engine.rollout(a, out=buf)
  assert got.reward.data_ptr() == buf.data_ptr()
  for name in ('reward', 'step_type', 'success', 'status'):
    assert torch.equal(getattr(got, name), getattr(want, name)), name
  with pytest.raises(ValueError):
    env.engine.rollout(a, out=buf[:-1])
  with pytest.raises(ValueError):
    env.engine.rollout(a, out=buf.view(torch.int8))
  env.close()
