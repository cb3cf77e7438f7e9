"""CPU tier of env records (save / load / copy): the BatchedEnvironment surface on the oracle-backed
engine double, extended here with save_envs / load_envs / copy_envs over BatchOracle's `cur` and
`pool` in NumPy, in the record layout of include/spriteworld_b200.h (engine.record_layout).

What runs on the host is under test: the id conversion, the signature check, EnvStates slicing,
concatenation and serialisation, the factor observations following a load, and the scene ring
bookkeeping of both refill modes around loads.  The device kernels are tests/test_gpu_env_states.py's.
"""
import io

import numpy as np
import pytest
import torch

from spriteworld_b200 import engine as engine_lib
from tests import oracle_engine

_Engine = engine_lib.Engine   # the device engine, for its host-side checks
_F64 = ('x0', 'y0', 'm00', 'm01', 'm10', 'm11', 'vx', 'vy')


class StatesOracleEngine(oracle_engine.OracleEngine):
  """The oracle double with env records."""

  def __init__(self, n_envs, n_slots, pool_depth, action, nodes, shapes, keep_in_frame=True,
               max_episode_length=1000, device=0):
    super().__init__(n_envs, n_slots, pool_depth, action, nodes, shapes, keep_in_frame,
                     max_episode_length, device)
    self.signature = engine_lib.config_signature(engine_lib.make_config(
        n_envs, n_slots, pool_depth, action, nodes, shapes, keep_in_frame, max_episode_length, 0))
    self._factors = np.zeros((self.n_envs, self.pool_depth, self.n_slots, 5), np.float32)
    self._spans = 1

  @property
  def record_bytes(self):
    return engine_lib.record_layout(self.n_slots)[1]

  def upload_scenes(self, scenes, env_ids, ring_slots):
    super().upload_scenes(scenes, env_ids, ring_slots)
    if 'factors' in scenes:
      self._factors[np.asarray(env_ids), np.asarray(ring_slots)] = scenes['factors']
    if (np.asarray(scenes['shape']) > 6).any():
      self._spans = 4

  def _ids(self, ids, distinct):
    ids = np.arange(self.n_envs, dtype=np.int32) if ids is None else engine_lib.env_ids_array(ids)
    if len(ids) and (ids.min() < 0 or ids.max() >= self.n_envs):
      raise _native_error('env id out of range')
    if distinct and len(np.unique(ids)) != len(ids):
      raise _native_error('destination env id appears twice')
    return ids.astype(np.int64)

  def save_envs(self, env_ids=None):
    ids = self._ids(env_ids, False)
    bo, n = self._bo, len(ids)
    cur = bo.pool[ids, bo.cursor[ids]]
    layout, rb = engine_lib.record_layout(self.n_slots)
    vals = {f: cur[f[:-1] if f in ('x0', 'y0') else f] for f in _F64}
    vals.update(pos_x=bo.cur['x'][ids], pos_y=bo.cur['y'][ids], member=cur['member'],
                rgb=np.concatenate([cur['rgb'], np.zeros(cur['rgb'].shape[:-1] + (1,), np.uint8)],
                                   -1).view('<u4')[..., 0],
                factors=self._factors[ids, bo.cursor[ids]].transpose(0, 2, 1),
                step_count=bo.step_count[ids], reset_next=bo.reset_next[ids],
                shape=cur['shape'], pos_f32=cur['pos_f32'])
    data = np.zeros((n, rb), np.uint8)
    for name, off, dtype, shape in layout:
      nbytes = dtype.itemsize * int(np.prod(shape, dtype=np.int64))
      data[:, off:off + nbytes] = np.ascontiguousarray(vals[name], dtype).reshape(n, -1).view(np.uint8)
    return engine_lib.EnvStates(torch.from_numpy(data), self._spans, self.signature, self.n_slots)

  def load_envs(self, states, env_ids=None):
    ids = self._ids(env_ids, True)
    _Engine.check_states(self, states, len(ids))
    bo, h = self._bo, states.to_host()
    k = bo.cursor[ids]
    for f in _F64:
      bo.pool[f[:-1] if f in ('x0', 'y0') else f][ids, k] = h[f]
    for f in ('member', 'rgb', 'shape', 'pos_f32'):
      bo.pool[f][ids, k] = h[f]
    self._factors[ids, k] = h['factors']
    bo.cur[ids] = bo.pool[ids, k]
    bo.cur['x'][ids], bo.cur['y'][ids] = h['pos_x'], h['pos_y']
    bo.step_count[ids], bo.reset_next[ids] = h['step_count'], h['reset_next']
    self._spans = max(self._spans, states.span_class)

  def copy_envs(self, src_ids, dst_ids):
    src, dst = self._ids(src_ids, False), self._ids(dst_ids, True)
    if len(src) != len(dst):
      raise ValueError('copy_envs: %d sources, %d destinations' % (len(src), len(dst)))
    self.load_envs(self.save_envs(src), dst)   # every read before any write


def _native_error(msg):
  from spriteworld_b200 import _native
  return _native.NativeError(msg)


@pytest.fixture(autouse=True)
def _states_engine(monkeypatch):
  oracle_engine.install(monkeypatch)
  monkeypatch.setattr(engine_lib, 'Engine', StatesOracleEngine)


def _env(E=12, K=5, seed=3, max_episode_length=20, refill='sync', factors=False):
  from spriteworld_b200 import environment, renderers
  from spriteworld_b200.configs.cobra import goal_finding_more_targets as cfgmod
  cfg = cfgmod.get_config('train')
  cfg['max_episode_length'] = max_episode_length
  if factors:
    cfg['renderers'] = dict(cfg['renderers'], factors=renderers.SpriteFactors())
  return environment.BatchedEnvironment(n_envs=E, pool_depth=K, rng=np.random.RandomState(seed),
                                        refill=refill, **cfg)


def _run(env, steps, seed):
  rng = np.random.RandomState(seed)
  for _ in range(steps):
    env.step(rng.uniform(0, 1, (env.n_envs, 4)).astype(np.float32))


def _host(env):
  """The whole observable state of every env: its record, decoded, and its frame."""
  h = env.save_envs().to_host()
  frames = env.render()['image'].numpy().copy()
  return h, frames


def _same_envs(a, b, ia, ib):
  (ha, fa), (hb, fb) = a, b
  for k in ha:
    assert np.array_equal(ha[k][ia], hb[k][ib]), k
  assert np.array_equal(fa[ia], fb[ib])


@pytest.mark.parametrize('kind', ['shift', 'subset'])
def test_copy_reads_the_state_from_before_the_call(kind):
  env = _env()
  env.reset()
  _run(env, 4, 1)
  E = env.n_envs
  if kind == 'shift':
    src = np.arange(E)
    dst = (src + 1) % E
  else:
    rng = np.random.RandomState(7)
    dst = rng.choice(E, 7, replace=False)
    src = np.concatenate([dst[3:], rng.choice(E, 3)])   # reads envs that are also written
  before = _host(env)
  cursor = env.engine.download_state()['cursor'].copy()
  env.copy_envs(list(src), torch.as_tensor(dst))
  after = _host(env)
  _same_envs(before, after, src, dst)
  untouched = np.setdiff1d(np.arange(E), dst)
  _same_envs(before, after, untouched, untouched)
  assert np.array_equal(env.engine.download_state()['cursor'], cursor)   # cursors stay
  env.close()


def test_load_refuses_records_of_another_configuration():
  a, b = _env(max_episode_length=20), _env(max_episode_length=21)
  a.reset(); b.reset()
  states = a.save_envs()
  before = b.save_envs().data.clone()
  with pytest.raises(ValueError, match='another configuration'):
    b.load_envs(states)
  assert torch.equal(b.save_envs().data, before)
  with pytest.raises(ValueError):
    a.load_envs(states[:3], [0, 1])     # two ids, three records
  a.load_envs(states[:3], [5, 6, 7])
  with pytest.raises(ValueError):
    a.copy_envs([0, 1], [2])
  a.close(); b.close()


def test_env_states_slice_concatenate_and_serialise():
  env = _env()
  env.reset()
  _run(env, 3, 2)
  s = env.save_envs()
  assert len(s) == env.n_envs and s.record_bytes == env.engine.record_bytes
  assert s.record_bytes % 16 == 0
  h = s.to_host()
  pieces = [s[:4], s[[9, 4]], s[7], s[-1]]
  cat = engine_lib.EnvStates.cat(pieces)
  order = [0, 1, 2, 3, 9, 4, 7, env.n_envs - 1]
  assert len(cat) == len(order)
  hc = cat.to_host()
  for k in h:
    assert np.array_equal(hc[k], h[k][order]), k
  buf = io.BytesIO()
  torch.save(cat, buf)
  buf.seek(0)
  back = torch.load(buf)                 # weights_only: EnvStates is an allowed global
  assert isinstance(back, engine_lib.EnvStates) and torch.equal(back.data, cat.data)
  assert back.signature == cat.signature and back.span_class == cat.span_class
  # records loaded anywhere: env 0 <- what env 9 was
  env.load_envs(cat[4:5], [0])
  assert np.array_equal(env.save_envs([0]).data.numpy(), s[9].data.numpy())
  with pytest.raises(ValueError):
    engine_lib.EnvStates.cat([s, engine_lib.EnvStates(s.data, 1, b'other', s.n_slots)])
  env.close()


def test_factor_tensors_follow_a_load():
  env = _env(factors=True)
  env.reset()
  saved = env.save_envs()
  want = {k: v.clone() for k, v in env.factor_tensors(('x', 'y', 'shape', 'scale', 'c0', 'x_vel')).items()}
  _run(env, 25, 4)                       # episodes of 20 steps: every env is on another scene
  dst = np.arange(env.n_envs)[::-1].copy()
  env.load_envs(saved, dst)
  got = env.factor_tensors(('x', 'y', 'shape', 'scale', 'c0', 'x_vel'))
  for k in want:
    assert torch.equal(got[k][dst], want[k]), k
  env.copy_envs([0], [1])
  got2 = env.factor_tensors(('shape', 'c0'))
  assert torch.equal(got2['c0'][1], got2['c0'][0])
  env.close()


@pytest.mark.parametrize('refill', ['sync', 'async'])
def test_load_in_place_then_auto_reset_continues_the_own_ring(refill):
  """Records loaded into the ids they came from replay the saved episode, and after its LAST each
  env starts the next scene of its own ring; the refill bookkeeping is untouched by the load."""
  E, K = 16, 6
  env = _env(E=E, K=K, max_episode_length=3, refill=refill)
  eng = env.engine
  uploads = np.ones((E, K), np.int64)
  pushed = eng.upload_scenes

  def upload(batch, env_ids, ring_slots):
    np.add.at(uploads, (np.asarray(env_ids), np.asarray(ring_slots)), 1)
    return pushed(batch, env_ids, ring_slots)

  eng.upload_scenes = upload
  env.reset()
  rng = np.random.RandomState(9)
  last = eng._bo.cursor.astype(np.int64).copy()
  absolute = last.copy()                 # reset() started scene 1 of every ring
  for t in range(40):
    if t % 5 == 2:
      saved = env.save_envs()
    if t % 5 == 4:
      upto = env._refilled_upto.copy()
      env.load_envs(saved)
      assert np.array_equal(env._refilled_upto, upto)
      # a loaded env is on its own ring slot still
      assert np.array_equal(eng._bo.cursor.astype(np.int64), last)
    ts = env.step(rng.uniform(0, 1, (E, 4)).astype(np.float32))
    cur = eng._bo.cursor.astype(np.int64)
    started = cur != last
    absolute += (cur - last) % K
    last = cur
    # every scene an env starts is the next of its own ring, uploaded for exactly this visit
    assert np.array_equal(uploads[np.arange(E), absolute % K], absolute // K + 1), t
    first = ts.step_type.numpy() == 0
    assert np.array_equal(first, started), t
    pool = eng._bo.pool[np.arange(E), cur]
    assert np.array_equal(eng._bo.cur['x'][first], pool['x'][first]), t
  assert absolute.min() >= K
  env.close()


@pytest.mark.parametrize('refill', ['sync', 'async'])
def test_loads_of_a_record_about_to_reset_keep_every_scene_fresh(refill):
  """A record saved on a LAST step (reset_next = 1) starts the env's next ring scene on the next
  step.  Loaded before every step, it makes the env start a scene on every step; the ring's
  underflow guard counts each load as a reset, so every scene started is one uploaded for exactly
  that visit of its ring slot, never a leftover of the previous lap."""
  E, K = 8, 6
  env = _env(E=E, K=K, max_episode_length=3, refill=refill)
  eng = env.engine
  uploads = np.ones((E, K), np.int64)
  pushed = eng.upload_scenes

  def upload(batch, env_ids, ring_slots):
    np.add.at(uploads, (np.asarray(env_ids), np.asarray(ring_slots)), 1)
    return pushed(batch, env_ids, ring_slots)

  eng.upload_scenes = upload
  rng = np.random.RandomState(13)
  ts = env.reset()
  while ts.step_type.numpy()[0] != 2:        # env 0 ends an episode
    ts = env.step(rng.uniform(0, 1, (E, 4)).astype(np.float32))
  at_last = env.save_envs([0])
  assert at_last.to_host()['reset_next'][0] == 1
  last = eng._bo.cursor.astype(np.int64).copy()
  absolute = eng.download_state_serial().astype(np.int64)
  starts = 0
  for t in range(40):
    env.load_envs(at_last, [0])
    if t % 2:
      env.copy_envs([0], [1])              # env 1 too: a copy of a record about to reset
    ts = env.step(rng.uniform(0, 1, (E, 4)).astype(np.float32))
    cur = eng._bo.cursor.astype(np.int64)
    absolute += (cur - last) % K
    starts += int(cur[0] != last[0])
    last = cur
    assert np.array_equal(uploads[np.arange(E), absolute % K], absolute // K + 1), t
  assert starts == 40                        # env 0 started a scene after every load
  env.close()
