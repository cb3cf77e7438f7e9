"""CPU tier of whole-run checkpoints (BatchedEnvironment.state_dict / load_state_dict): the host
layer on the oracle-backed engine double, extended here with save_state / load_state over
BatchOracle's rings, counters and live positions.

What runs on the host is under test: the refill bookkeeping and underflow guard, the action-noise
and refill-block RandomStates, the snapshot schedule of the asynchronous refill, the fingerprint
and its refusals, and torch.save / torch.load of the dict.  The engine's own checkpoint (layout,
checks, copies) is tests/test_gpu_checkpoint.py's.  The asynchronous refill's jobs run at once here
(_NowExecutor), so that its refill timing, and with it the run, is deterministic.
"""
import collections
import concurrent.futures
import io

import numpy as np
import pytest
import torch

from spriteworld_b200 import _native
from spriteworld_b200 import engine as engine_lib
from tests import oracle_engine

E, K = 8, 4


class CheckpointOracleEngine(oracle_engine.OracleEngine):
  """The oracle double with an engine checkpoint: the state the device engine keeps (live
  positions, cursor, step_count, scene_serial, reset_next and every ring), nothing else."""

  def __init__(self, n_envs, n_slots, pool_depth, action, nodes, shapes, keep_in_frame=True,
               max_episode_length=1000, device=0):
    super().__init__(n_envs, n_slots, pool_depth, action, nodes, shapes, keep_in_frame,
                     max_episode_length, device)
    self.signature = engine_lib.config_signature(engine_lib.make_config(
        n_envs, n_slots, pool_depth, action, nodes, shapes, keep_in_frame, max_episode_length, 0))

  def _parts(self):
    bo = self._bo
    return [np.array([self.n_envs, self.pool_depth, self.n_slots], np.int64), bo.cur['x'], bo.cur['y'],
            bo.cursor, bo.step_count, self._serial, bo.reset_next, bo.pool, self._factors]

  def save_state(self):
    parts = [np.ascontiguousarray(p).reshape(-1).view(np.uint8) for p in self._parts()]
    return torch.from_numpy(np.concatenate(parts))

  def load_state(self, state):
    data, off = state.numpy(), 0
    loaded = []
    for p in self._parts():
      p = np.ascontiguousarray(p)
      loaded.append(data[off:off + p.nbytes].copy().view(p.dtype).reshape(p.shape))
      off += p.nbytes
    if off != len(data) or not np.array_equal(loaded[0], self._parts()[0]):
      raise _native.NativeError('swb_load_engine: checkpoint of another engine')
    bo = self._bo
    _, x, y, bo.cursor[:], bo.step_count[:], self._serial[:], bo.reset_next[:], bo.pool[:], self._factors[:] = loaded
    # the live sprites are the ring entries the envs are on, at their live positions
    bo.cur[:] = bo.pool[np.arange(self.n_envs), bo.cursor]
    bo.cur['x'], bo.cur['y'] = x, y
    self._last_cursor = bo.cursor.astype(np.int64).copy()


class _NowExecutor(object):
  """Runs every refill job when it is submitted."""

  def submit(self, fn, *args):
    future = concurrent.futures.Future()
    future.set_result(fn(*args))
    return future

  def shutdown(self, wait=True):
    pass


@pytest.fixture(autouse=True)
def _checkpoint_engine(monkeypatch):
  oracle_engine.install(monkeypatch)
  monkeypatch.setattr(engine_lib, 'Engine', CheckpointOracleEngine)


def _cfg(max_episode_length=5, image_size=(24, 24), scale=0.5, goal=(0.5, 0.5)):
  from spriteworld_b200 import action_spaces, renderers, tasks
  from spriteworld_b200.configs.cobra import goal_finding_more_targets as cfgmod
  from spriteworld_b200 import factor_distributions as distribs
  cfg = cfgmod.get_config('train')
  cfg['max_episode_length'] = max_episode_length
  cfg['action_space'] = action_spaces.SelectMove(scale=scale, noise_scale=0.05)
  cfg['task'] = tasks.FindGoalPosition(filter_distrib=distribs.Continuous('c0', 0., 0.4), goal_position=goal,
                                       terminate_distance=0.05)
  color = cfg['renderers']['image'].color_to_rgb
  cfg['renderers'] = collections.OrderedDict([
      ('image', renderers.PILRenderer(image_size=image_size, anti_aliasing=2, color_to_rgb=color)),
      ('factors', renderers.SpriteFactors(('x', 'y', 'shape', 'scale', 'c0', 'x_vel')))])
  return cfg


def _env(refill='sync', seed=3, n_envs=E, pool_depth=K, refill_threads=3, n_slots=None, **kw):
  from spriteworld_b200 import environment
  env = environment.BatchedEnvironment(n_envs=n_envs, pool_depth=pool_depth, rng=np.random.RandomState(seed),
                                       refill=refill, refill_threads=refill_threads, n_slots=n_slots,
                                       **_cfg(**kw))
  if env._worker is not None:
    env._worker.shutdown(wait=True)
    env._worker = _NowExecutor()
  return env


def _outputs(ts):
  out = dict(step_type=ts.step_type, reward=ts.reward, discount=ts.discount, success=ts.success,
             status=ts.status, image=ts.observation['image'])
  out.update(('factor_' + k, v) for k, v in ts.observation['factors'].items())
  return {k: v.numpy().copy() for k, v in out.items()}


def _run(env, actions):
  return [_outputs(env.step(a)) for a in actions]


def _same(want, got):
  assert len(want) == len(got)
  for t, (w, g) in enumerate(zip(want, got)):
    for k in w:
      assert np.array_equal(w[k], g[k], equal_nan=True), (t, k)


def _observed(env):
  """What the env shows of its state without stepping: frames, factor observations, ring state."""
  out = {'image': env.render()['image'].numpy().copy()}
  out.update(('factor_' + k, v.numpy().copy()) for k, v in env.factor_tensors(('x', 'y', 'shape', 'c0')).items())
  out.update((k, np.asarray(v).copy()) for k, v in env.engine.download_state().items())
  return out


@pytest.mark.parametrize('refill', ['sync', 'async'])
def test_resume_equals_the_uninterrupted_run_and_rewinds(refill):
  n0, n1 = 13, 40
  acts = np.random.RandomState(1).uniform(0, 1, (n0 + n1, E, 4)).astype(np.float32)
  a = _env(refill, seed=3)
  a.reset()
  _run(a, acts[:n0])
  assert (a.engine.download_state()['step_count'] > 0).any()     # mid-episode
  sd = a.state_dict()
  observed = _observed(a)
  refills, serial = a.refill_stats()['refills'], a.engine.download_state_serial().copy()
  want = _run(a, acts[n0:])
  firsts = sum(int((w['step_type'] == 0).sum()) for w in want)
  assert firsts >= 3 * E                                            # episode boundaries ...
  assert a.refill_stats()['refills'] >= refills + 3                 # ... and refills after the checkpoint
  assert (a.engine.download_state_serial() - serial).min() >= K     # every ring turned over

  buf = io.BytesIO()
  torch.save(sd, buf)
  buf.seek(0)
  back = torch.load(buf)                                            # weights_only=True
  b = _env(refill, seed=77)                                         # another rng: other scenes, other noise
  b.load_state_dict(back)
  got_observed = _observed(b)
  for k in observed:
    assert np.array_equal(observed[k], got_observed[k]), k
  _same(want, _run(b, acts[n0:]))

  a.load_state_dict(sd)                                             # rewind the run itself
  _same(want, _run(a, acts[n0:]))
  a.close(); b.close()


def test_state_dict_holds_only_what_weights_only_loads():
  env = _env('async', seed=5)
  env.reset()
  _run(env, np.random.RandomState(2).uniform(0, 1, (6, E, 4)).astype(np.float32))
  sd = env.state_dict()

  def walk(v):
    if isinstance(v, dict):
      assert all(isinstance(k, str) for k in v)
      return all(walk(x) for x in v.values())
    if isinstance(v, (list, tuple)):
      return all(walk(x) for x in v)
    return v is None or isinstance(v, (torch.Tensor, bool, int, float, str, bytes))

  assert walk(sd)
  assert len(sd['block_rngs']) == 3 and sd['rng'][0] == 'MT19937'
  assert sd['engine'].dtype == torch.uint8 and sd['engine'].device.type == 'cpu'
  env.close()


def test_default_rng_is_numpys_global_state():
  from spriteworld_b200 import environment
  np.random.seed(11)
  a = environment.BatchedEnvironment(n_envs=E, pool_depth=K, refill='sync', **_cfg())
  a.reset()
  acts = np.random.RandomState(4).uniform(0, 1, (20, E, 4)).astype(np.float32)
  _run(a, acts[:5])
  sd = a.state_dict()
  want = _run(a, acts[5:])
  np.random.seed(12345)                                              # the global stream moves on
  a.load_state_dict(sd)                                              # and is set back
  _same(want, _run(a, acts[5:]))
  a.close()


_MISMATCHES = [
    ('n_envs', dict(n_envs=E + 2)),
    ('pool_depth', dict(pool_depth=K + 1)),
    ('n_slots', dict(n_slots=12)),
    ('signature', dict(goal=(0.2, 0.8))),            # the task
    ('signature', dict(scale=0.3)),                  # the action space
    ('rasters', dict(image_size=(20, 24))),
    ('refill', dict(refill='async')),
]


@pytest.mark.parametrize('key,kw', _MISMATCHES + [('refill_blocks', dict(refill='async', refill_threads=2)),
                                                  ('sampler', None)])
def test_a_mismatch_is_refused_and_changes_nothing(key, kw):
  base = dict(refill='async', refill_threads=3) if key == 'refill_blocks' else {}
  a = _env(seed=3, **base)
  a.reset()
  _run(a, np.random.RandomState(2).uniform(0, 1, (4, E, 4)).astype(np.float32))
  sd = a.state_dict()
  if kw is None:                                   # a device-sampler checkpoint
    sd = dict(sd, fingerprint=dict(sd['fingerprint'], sampler='device'))
    b = _env(seed=9)
  else:
    b = _env(seed=9, **dict(base, **kw))
  b.reset()
  before = (b.engine.save_state().clone(), b._rng.get_state()[1].copy(), b._t, b._resets, b._safe_step)
  with pytest.raises(ValueError, match=key):
    b.load_state_dict(sd)
  after = (b.engine.save_state(), b._rng.get_state()[1], b._t, b._resets, b._safe_step)
  assert torch.equal(before[0], after[0]) and np.array_equal(before[1], after[1])
  assert before[2:] == after[2:]
  a.close(); b.close()
