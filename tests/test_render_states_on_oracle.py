"""CPU tier of the frames of env records: Engine.render_states, BatchedEnvironment.observe,
BatchedEnvironment.factor_tensors(states) and SpriteFactors.render_states, on the oracle-backed
engine double extended here with swb_render_states (RenderStatesOracleEngine: the records decoded
and drawn one by one with oracle.render).

What runs on the host is under test: Engine.render_states' argument checks and the call it makes,
the keys, order, shapes and dtypes of observe(), the status OR over rasters, the refusal of a
renderer without a record form before anything is enqueued, and the factor observations of records
against those of the envs they are loaded into, sanitised shape ids included.  The kernel is
tests/test_gpu_render_states.py's.
"""
import collections
import ctypes

import numpy as np
import pytest
import torch

from oracle import oracle
from spriteworld_b200 import _native
from spriteworld_b200 import engine as engine_lib
from tests import oracle_engine
from tests.test_env_states_on_oracle import StatesOracleEngine
from tests.test_expand_on_oracle import _set_field

_Engine = engine_lib.Engine


def _fake_overflow(n, width):
  """The double's render status: ENV_SPAN_OVERFLOW on records i with (i + width) % 3 == 0, so
  that rasters of different widths flag different records."""
  return np.where((np.arange(n) + width) % 3 == 0, _native.ENV_SPAN_OVERFLOW, 0).astype(np.uint8)


class _RenderLib(oracle_engine._Lib):

  def swb_render_states(self, eng, raster, records, n, records_bytes, span_class, frames, status, stream):
    assert records_bytes == n * eng.record_bytes and span_class in (1, 4)
    if n == 0:
      return 0
    sprites = oracle_engine.record_sprites(eng, oracle_engine.states_at(eng, records, n))
    r = eng._rasters[raster]
    out = np.ctypeslib.as_array((ctypes.c_uint8 * (n * r.height * r.width * 3)).from_address(frames.value))
    out = out.reshape(n, r.height, r.width, 3)
    for i in range(n):
      out[i] = oracle.render(r.rc, eng._tab, sprites[i])
    st = np.ctypeslib.as_array((ctypes.c_uint8 * n).from_address(status.value))
    st[:] = _fake_overflow(n, r.width)
    eng._launches += 1
    return 0


class RenderStatesOracleEngine(StatesOracleEngine):
  """The oracle double with swb_render_states under the real Engine.render_states, and shape ids
  sanitised on load as swb_load_envs sanitises them."""

  check_states = _Engine.check_states
  _check_frames = _Engine._check_frames
  render_states = _Engine.render_states

  def __init__(self, *args, **kw):
    super().__init__(*args, **kw)
    self._lib, self._rasters = _RenderLib(), {}

  def render_status(self):   # the live renders of the double never overflow
    return torch.zeros(self.n_envs, dtype=torch.uint8)

  def load_envs(self, states, env_ids=None):
    super().load_envs(states, env_ids)
    ids = self._ids(env_ids, True)
    bo = self._bo
    bo.pool['shape'][ids, bo.cursor[ids]] = oracle_engine._SHAPE_IDS[bo.pool['shape'][ids, bo.cursor[ids]]]
    bo.cur['shape'][ids] = oracle_engine._SHAPE_IDS[bo.cur['shape'][ids]]


class RenderStatesOracleRaster(oracle_engine.OracleRaster):

  def __init__(self, engine, *args, **kw):
    super().__init__(engine, *args, **kw)
    self._h = id(self)
    engine._rasters[self._h] = self


@pytest.fixture(autouse=True)
def _render_engine(monkeypatch):
  oracle_engine.install(monkeypatch)
  monkeypatch.setattr(engine_lib, 'Engine', RenderStatesOracleEngine)
  monkeypatch.setattr(engine_lib, 'Raster', RenderStatesOracleRaster)


def _env(renderers, E=6, K=5, seed=3):
  from spriteworld_b200 import action_spaces, environment
  from spriteworld_b200.configs.cobra import goal_finding_more_targets as cfgmod
  cfg = cfgmod.get_config('train')
  cfg['action_space'] = action_spaces.SelectMove(scale=0.25, motion_cost=0.1)
  cfg['max_episode_length'] = 9
  cfg['renderers'] = renderers
  return environment.BatchedEnvironment(n_envs=E, pool_depth=K, rng=np.random.RandomState(seed),
                                        refill='sync', **cfg)


def _renderers(*names):
  from spriteworld_b200 import renderers
  hsv = renderers.color_maps.hsv_to_rgb
  make = dict(image=lambda: renderers.PILRenderer(image_size=(16, 16), anti_aliasing=2, color_to_rgb=hsv),
              small=lambda: renderers.PILRenderer(image_size=(8, 6), color_to_rgb=hsv, bg_color=(9, 9, 9)),
              factors=lambda: renderers.SpriteFactors(),
              success=lambda: renderers.Success())
  return collections.OrderedDict((n, make[n]()) for n in names)


def _started(env, steps=3, seed=1):
  rng = np.random.RandomState(seed)
  env.reset()
  for _ in range(steps):
    env.step(rng.uniform(0, 1, (env.n_envs, 4)).astype(np.float32))
  return rng


def test_observe_returns_every_renderer_in_order():
  env = _env(_renderers('small', 'factors', 'image'))
  _started(env)
  states = env.save_envs()[[5, 0, 0, 3, 1, 2, 4]]
  launches = env.engine.launch_count()
  obs, status = env.observe(states)
  assert list(obs) == ['small', 'factors', 'image']
  assert env.engine.launch_count() == launches + 2          # one per raster
  assert obs['small'].dtype == torch.uint8 and tuple(obs['small'].shape) == (7, 6, 8, 3)
  assert obs['image'].dtype == torch.uint8 and tuple(obs['image'].shape) == (7, 16, 16, 3)
  assert obs['image'].data_ptr() != env._frames['image'].data_ptr()
  f = obs['factors']
  assert list(f) == list(env._renderers['factors']._factors) + ['mask']
  for k, v in f.items():
    assert tuple(v.shape) == (7, env.engine.n_slots) and v.dtype == (torch.bool if k == 'mask' else torch.float32)
  # the status is the OR over the two rasters
  assert np.array_equal(status.numpy(), _fake_overflow(7, 8) | _fake_overflow(7, 16))
  assert status.dtype == torch.uint8 and tuple(status.shape) == (7,)
  env.close()


def test_observe_frames_equal_load_and_render():
  env = _env(_renderers('image', 'small'))
  _started(env, seed=4)
  states = env.save_envs()[[3, 1, 4, 0, 5, 2]]
  obs, _ = env.observe(states)
  env.load_envs(states)
  for k, v in env.render().items():
    assert torch.equal(obs[k], v), k
  env.close()


def test_a_renderer_without_a_record_form_is_refused_before_anything_is_enqueued():
  env = _env(_renderers('image', 'success'))
  _started(env)
  states = env.save_envs()
  launches = env.engine.launch_count()
  with pytest.raises(NotImplementedError, match='success'):
    env.observe(states)
  assert env.engine.launch_count() == launches
  env.close()


def test_render_states_checks_its_arguments():
  env = _env(_renderers('image'))
  _started(env)
  eng, raster = env.engine, env._rasters['image']
  states = env.save_envs()
  launches = eng.launch_count()
  with pytest.raises(ValueError, match='EnvStates'):
    eng.render_states(raster, states.data)
  with pytest.raises(ValueError, match='EnvStates must hold'):
    eng.render_states(raster, engine_lib.EnvStates(states.data[:, :-16].contiguous(), 1, states.signature,
                                                   states.n_slots))
  other = engine_lib.EnvStates(states.data, 1, b'x' * len(states.signature), states.n_slots)
  with pytest.raises(ValueError, match='another configuration'):
    eng.render_states(raster, other)
  n = len(states)
  for bad in (torch.zeros((n, 16, 16, 3), dtype=torch.int32), torch.zeros((n, 16, 15, 3), dtype=torch.uint8),
              torch.zeros((n - 1, 16, 16, 3), dtype=torch.uint8), np.zeros((n, 16, 16, 3), np.uint8),
              torch.zeros((n, 16, 3, 16), dtype=torch.uint8).transpose(2, 3)):
    with pytest.raises(ValueError, match='frames'):
      eng.render_states(raster, states, frames=bad)
  for bad in (torch.zeros(n, dtype=torch.int32), torch.zeros(n + 1, dtype=torch.uint8),
              torch.zeros((n, 1), dtype=torch.uint8), torch.zeros(2 * n, dtype=torch.uint8)[::2]):
    with pytest.raises(ValueError, match='status'):
      eng.render_states(raster, states, status=bad)
  assert eng.launch_count() == launches
  frames = torch.zeros((n, 16, 16, 3), dtype=torch.uint8)
  status = torch.zeros(n, dtype=torch.uint8)
  got = eng.render_states(raster, states, frames, status)
  assert got[0] is frames and got[1] is status and eng.launch_count() == launches + 1
  env.close()


def test_factor_tensors_of_records_equal_those_after_a_load():
  from spriteworld_b200 import renderers
  env = _env(_renderers('image', 'factors'), E=8)
  _started(env, steps=4, seed=6)
  states = env.save_envs()[[7, 2, 2, 5, 0, 1, 6, 3]]
  data = states.data.numpy().copy()
  shape = states.to_host()['shape']
  shape[0, :] = 255
  shape[3, 0] = 13
  shape[5, -1] = 200
  _set_field(data, env.engine.n_slots, 'shape', shape)
  states = engine_lib.EnvStates(torch.from_numpy(data), states.span_class, states.signature, states.n_slots)
  names = ('x', 'y', 'shape', 'angle', 'scale', 'c0', 'c1', 'c2', 'x_vel', 'y_vel')
  direct = env.factor_tensors(names, states)
  by_renderer = renderers.SpriteFactors(names).render_states(env, states)
  observed = env.observe(states)[0]['factors']
  assert not direct['mask'][0].any()
  env.load_envs(states)
  loaded = env.factor_tensors(names)
  assert list(direct) == list(loaded) == list(names) + ['mask']
  for k in loaded:
    for got in (direct, by_renderer, observed):
      assert got[k].dtype == loaded[k].dtype and torch.equal(got[k], loaded[k]), k
  env.close()
