"""CPU doubles of engine.Engine / engine.Raster backed by the oracle (test infrastructure).

The package has no CPU path: its host layer (environment.Environment, the plugin protocol in
_direct.py, task/action compilation, scene packing) always drives the CUDA engine.  To run that
host layer in the CPU tier of the test-suite -- e.g. under the reference's own test files -- these
doubles implement the engine's Python surface on top of oracle.BatchOracle, which follows the
same scene-pool protocol.  They are installed by tests only (install()); nothing in the product
imports this module.
"""
import ctypes

import numpy as np
import torch

from oracle import oracle
from spriteworld_b200 import _native
from spriteworld_b200 import engine as engine_lib
from tests import fixtures

_FIELDS = ('x', 'y', 'm00', 'm01', 'm10', 'm11', 'vx', 'vy', 'member', 'shape', 'pos_f32', 'rgb')


class _Lib(object):
  """The two C-ABI entry points _direct.py calls through the engine handle."""

  def swb_eval_task(self, eng, out, stream):
    bo = eng._bo
    for e in range(eng.n_envs):
      r, s, err = oracle.task_eval(eng._cfg, bo.cur[e])
      bo.reward[e], bo.success[e], bo.err[e] = r, int(s), err
    return 0

  def swb_apply_action(self, eng, ptr, dtype, out, stream):
    bo = eng._bo
    n = 2 if dtype == _native.DTYPE_I32 else 4
    ctype = {_native.DTYPE_I32: ctypes.c_int32, _native.DTYPE_F32: ctypes.c_float,
             _native.DTYPE_F64: ctypes.c_double}[dtype]
    a = np.ctypeslib.as_array((ctype * (n * eng.n_envs)).from_address(ptr.value)).reshape(
        eng.n_envs, n)
    bo.err[:] = 0
    for e in range(eng.n_envs):
      try:
        cost, _ = oracle.action_step(eng._cfg, eng._tab, bo.cur[e], a[e],
                                     dtype == _native.DTYPE_F32)
      except KeyError:
        cost = 0.0
        bo.err[e] |= _native.ENV_BAD_ACTION
      bo.reward[e] = cost
    return 0


class OracleRaster(object):

  def __init__(self, engine, width, height, anti_aliasing=1, bg_color=(0, 0, 0)):
    self.engine = engine
    self.width, self.height, self.anti_aliasing = int(width), int(height), int(anti_aliasing)
    self.rc = oracle.raster_cfg(width, height, anti_aliasing, bg_color)

  def new_frames(self):
    return torch.empty((self.engine.n_envs, self.height, self.width, 3), dtype=torch.uint8)

  def close(self):
    pass


class OracleEngine(object):

  def __init__(self, n_envs, n_slots, pool_depth, action, nodes, shapes, keep_in_frame=True,
               max_episode_length=1000, device=0):
    self.n_envs, self.n_slots, self.pool_depth = int(n_envs), int(n_slots), int(pool_depth)
    self.device = torch.device('cpu')
    self.action_kind = engine_lib.ACTIONS[action['kind']].kind
    # the engine's FindGoalPosition distance: the correctly rounded sqrt
    self._cfg = oracle.with_device_sqrt(fixtures.env_cfg_from_meta(dict(
        action=dict(kind=action['kind'], scale=float(action['scale']),
                    motion_cost=float(action.get('motion_cost', 0.0))),
        keep_in_frame=bool(keep_in_frame),
        max_episode_length=int(min(max_episode_length, 2 ** 31 - 1)), nodes=nodes)))
    self._tab = oracle.shape_table(shapes)
    pool = np.zeros((self.n_envs, self.pool_depth, self.n_slots), oracle.SPRITE_DTYPE)
    self._bo = oracle.BatchOracle(self._cfg, self._tab, None, pool)
    self._bo.reset_next[:] = 0
    bo = self._bo
    self._reward = torch.from_numpy(bo.reward)
    self._step_type = torch.from_numpy(bo.step_type)
    self._success = torch.from_numpy(bo.success)
    self._status = torch.from_numpy(bo.err)
    self._lib, self._h, self._out = _Lib(), self, None
    self._launches = 0
    self._serial = np.zeros(self.n_envs, np.int64)       # scenes started (engine: scene_serial)
    self._last_cursor = bo.cursor.astype(np.int64).copy()

  def _stream(self):
    return None

  def close(self):
    pass

  def upload_scenes(self, scenes, env_ids, ring_slots):
    env_ids, ring_slots = np.asarray(env_ids, np.int64), np.asarray(ring_slots, np.int64)
    n, S = len(env_ids), self.n_slots
    assert len(ring_slots) == n and (ring_slots >= 0).all() and (ring_slots < self.pool_depth).all()
    for f in _FIELDS:   # the shapes engine.Engine.upload_scenes insists on
      tail = (3,) if f == 'rgb' else ()
      assert np.shape(scenes[f]) == (n, S) + tail, (f, np.shape(scenes[f]), (n, S) + tail)
      self._bo.pool[f][env_ids, ring_slots] = scenes[f]

  def upload_state(self, pos_x=None, pos_y=None, cursor=None, step_count=None, reset_next=None):
    bo = self._bo
    if cursor is not None:
      bo.cursor[:] = np.asarray(cursor, np.int32)
      self._last_cursor = bo.cursor.astype(np.int64).copy()
    # static factors of the live scene follow the cursor; positions are the live ones
    live_x, live_y = bo.cur['x'].copy(), bo.cur['y'].copy()
    bo.cur[:] = bo.pool[np.arange(self.n_envs), bo.cursor]
    bo.cur['x'] = live_x if pos_x is None else np.asarray(pos_x, np.float64).reshape(live_x.shape)
    bo.cur['y'] = live_y if pos_y is None else np.asarray(pos_y, np.float64).reshape(live_y.shape)
    if step_count is not None:
      bo.step_count[:] = np.asarray(step_count, np.int32)
    if reset_next is not None:
      bo.reset_next[:] = np.asarray(reset_next, np.uint8)

  def request_reset(self, mask=None):
    if mask is None:
      self._bo.reset_next[:] = 1
    else:
      self._bo.reset_next[np.asarray(mask, bool)] = 1

  def step(self, actions, raster=None, frames=None):
    engine_lib.action_dtype(self.action_kind, self.n_envs, actions)   # what Engine.step accepts
    a = np.ascontiguousarray(actions.numpy())
    self._bo.step(a)   # a bad Embodied direction sets ENV_BAD_ACTION, like the engine
    self._launches += 1
    cur = self._bo.cursor.astype(np.int64)
    self._serial += (cur != self._last_cursor)          # at most one scene per step
    self._last_cursor = cur
    if raster is not None:
      frames = self.render(raster, frames)
    return engine_lib.StepResult(self._reward, self._step_type, self._success, self._status, frames)

  def render(self, raster, frames=None):
    if frames is None:
      frames = raster.new_frames()
    out = frames.numpy()
    for e in range(self.n_envs):
      out[e] = oracle.render(raster.rc, self._tab, self._bo.cur[e])
    self._launches += 1
    return frames

  def download_state(self):
    bo = self._bo
    return dict(pos_x=bo.cur['x'].copy(), pos_y=bo.cur['y'].copy(), cursor=bo.cursor.copy(),
                step_count=bo.step_count.copy(), reset_next=bo.reset_next.copy())

  def check_render(self):
    pass

  # the asynchronous refill's engine surface: no streams here, so a snapshot is a copy taken at
  # once and every event has already happened
  def snapshot_scene_serial(self):
    serial = self._serial.copy()

    class _Snapshot(object):
      def ready(self):
        return True

      def wait(self):
        return serial

    return _Snapshot()

  def side_stream_context(self):
    import contextlib
    return contextlib.nullcontext()

  def record_side_event(self):
    return None

  def wait_event(self, event):
    pass

  def download_state_serial(self):
    return self._serial.copy()

  def state_tensors(self):
    bo = self._bo
    return dict(pos_x=torch.from_numpy(bo.cur['x'].copy()), pos_y=torch.from_numpy(bo.cur['y'].copy()),
                cursor=torch.from_numpy(bo.cursor), step_count=torch.from_numpy(bo.step_count),
                reset_next=torch.from_numpy(bo.reset_next))

  def launch_count(self):
    return self._launches


def install(monkeypatch):
  """Routes the package's host layer to the oracle doubles for the duration of a test."""
  monkeypatch.setattr(engine_lib, 'Engine', OracleEngine)
  monkeypatch.setattr(engine_lib, 'Raster', OracleRaster)
  monkeypatch.setattr(torch.cuda, 'synchronize', lambda *a, **k: None)
  from spriteworld_b200 import _direct
  monkeypatch.setattr(_direct, '_engines', type(_direct._engines)())
  monkeypatch.setattr(_direct, '_rasters', {})
