"""Thin Python owner of one swb_engine (one per GPU).

PyTorch is used only for device memory and streams: action, reward, flag and frame
buffers are torch tensors whose `data_ptr()` is handed to the C-ABI
(include/spriteworld_b200.h).  All compute happens in the CUDA library.
"""
import collections
import ctypes

import numpy as np
import torch

from spriteworld_b200 import _native

SCENE_FIELDS_F64 = ('x', 'y', 'm00', 'm01', 'm10', 'm11', 'vx', 'vy')


def _as_ptr(a):
  return ctypes.c_void_p(a.ctypes.data)


class _DevicePointer(object):
  """Minimal __cuda_array_interface__ carrier so torch can alias engine-owned memory."""

  def __init__(self, ptr, shape, typestr):
    self.__cuda_array_interface__ = dict(shape=tuple(shape), typestr=typestr,
                                         data=(int(ptr), False), version=2)


class StepResult(object):
  """Per-env outputs of one step, as device tensors (valid until the next step)."""
  __slots__ = ('reward', 'step_type', 'success', 'status', 'frames')

  def __init__(self, reward, step_type, success, status, frames=None):
    self.reward, self.step_type, self.success = reward, step_type, success
    self.status, self.frames = status, frames


class RolloutResult(object):
  """Outputs of a rollout, (T, n_envs, C) each: reward float64, step_type int8 (STEP_MID, STEP_LAST
  or, after a plan's first LAST and for an env about to reset, STEP_NONE with reward 0), success
  and status uint8.  The caller's own tensors: no later call overwrites them.  `leaves`: None, or
  the EnvStates of the state each plan ends in (record r * C + c: root r's plan c).  `trajectory`:
  None, or the EnvStates of the state after every step (record (t * n + r) * C + c: root r's plan c
  after step t, its end state once the plan has ended)."""
  __slots__ = ('reward', 'step_type', 'success', 'status', 'leaves', 'trajectory')

  def __init__(self, reward, step_type, success, status, leaves=None, trajectory=None):
    self.reward, self.step_type, self.success, self.status = reward, step_type, success, status
    self.leaves, self.trajectory = leaves, trajectory


OUT_BYTES_PER_ENV = 8 + 1 + 1 + 1


def split_outputs(buf, n_envs):
  """Views (reward f64, step_type i8, success u8, status u8) of a packed output buffer of
  n_envs * OUT_BYTES_PER_ENV bytes (layout: all rewards, then all step types, ...); of a
  (n, n_envs * OUT_BYTES_PER_ENV) buffer, n such buffers, copies of n * n_envs outputs each."""
  E = int(n_envs)
  reward = buf[..., :8 * E].contiguous().view(torch.float64).reshape(-1)
  step_type = buf[..., 8 * E:9 * E].reshape(-1).view(torch.int8)
  success = buf[..., 9 * E:10 * E].reshape(-1)
  status = buf[..., 10 * E:11 * E].reshape(-1)
  return reward, step_type, success, status


ActionSpec = collections.namedtuple('ActionSpec', ['kind', 'columns', 'dtypes'])

# What the engine accepts per action kind: (E, columns) actions of one of `dtypes` (dtype name ->
# swb action dtype), as device tensors (step, step_gather) or host arrays (step_host)
_FLOATS = {'float32': _native.DTYPE_F32, 'float64': _native.DTYPE_F64}
ACTIONS = {'select_move': ActionSpec(_native.ACT_SELECT_MOVE, 4, _FLOATS),
           'drag_and_drop': ActionSpec(_native.ACT_DRAG_AND_DROP, 4, _FLOATS),
           'embodied': ActionSpec(_native.ACT_EMBODIED, 2, {'int32': _native.DTYPE_I32})}
_SPECS = {spec.kind: spec for spec in ACTIONS.values()}   # the same table by swb action kind


def action_dtype(action_kind, n_envs, actions, device=None, plans=False):
  """The swb action dtype of `actions` (tensor or array) for `n_envs` envs of swb `action_kind`;
  with `device`, a contiguous tensor on it; with `plans`, the (T, n_envs, C, columns) actions of a
  rollout, T and C at least 1.  ValueError otherwise: nothing is converted."""
  if device is not None and not (isinstance(actions, torch.Tensor) and actions.device == device
                                 and actions.is_contiguous()):
    raise ValueError('actions must be a contiguous tensor on %s, got %s'
                     % (device, _describe(actions)))
  spec = _SPECS[action_kind]
  name = str(actions.dtype).replace('torch.', '')
  shape, got = (int(n_envs), spec.columns), tuple(actions.shape)
  if plans:
    ok = len(got) == 4 and got[1::2] == shape and got[0] >= 1 and got[2] >= 1
    shape = ('T >= 1', shape[0], 'C >= 1', shape[1])
  else:
    ok = got == shape
  if not ok or name not in spec.dtypes:
    raise ValueError('actions must have shape %s and dtype %s, got %s %s' % (
        shape, ' or '.join(spec.dtypes), name, got))
  return spec.dtypes[name]


def rollout_outputs(out, n_steps, n_envs, n_candidates, device):
  """(packed buffer, RolloutResult of its views) for a rollout of that size: `out`, or if it is None
  a new uint8 tensor, of n_steps * n_envs * n_candidates * OUT_BYTES_PER_ENV bytes on `device`, laid
  out as split_outputs reads it."""
  shape = (int(n_steps), int(n_envs), int(n_candidates))
  n = shape[0] * shape[1] * shape[2]
  if out is None:
    out = torch.empty(n * OUT_BYTES_PER_ENV, dtype=torch.uint8, device=device)
  _check_output(out, 'out', torch.uint8, (n * OUT_BYTES_PER_ENV,), device, align=8)
  return out, RolloutResult(*[v.view(shape) for v in split_outputs(out, n)])


def _check_output(t, name, dtype, shape, device, align=1):
  """ValueError naming `name` unless `t` is a contiguous tensor of `dtype` and `shape` on `device`,
  `align`-byte aligned: a kernel writes the whole shape from t.data_ptr(), so anything else would be
  written out of bounds or scrambled."""
  shape = tuple(shape)
  if (not isinstance(t, torch.Tensor) or t.dtype != dtype or t.device != device or tuple(t.shape) != shape
      or not t.is_contiguous() or t.data_ptr() % align):
    raise ValueError('%s must be a contiguous%s %s tensor of shape %s on %s, got %s' % (
        name, ', %d-byte aligned' % align if align > 1 else '', str(dtype).replace('torch.', ''), shape,
        device, _describe(t)))


def _address(t):
  """ctypes pointer to tensor t's data.  An empty tensor may have no address, and the C-ABI refuses a
  null buffer even where it reads and writes nothing; any aligned address stands in for it then."""
  return ctypes.c_void_p(t.data_ptr() or 256)


def _rows(engine, states, live=True):
  """(n, records pointer or None, bytes) of a call on `states`: EnvStates of n records `engine` can
  read, or where the call takes the live envs (`live`) None for its n_envs envs.  ValueError
  otherwise."""
  if states is None and live:
    return engine.n_envs, None, 0
  if not isinstance(states, EnvStates):
    raise ValueError('states must be EnvStates, got %s' % type(states).__name__)
  engine.check_states(states, len(states))
  return len(states), _address(states.data), states.data.numel()


# What each sprite-mask observation writes: its C-ABI call, then the name, dtype and axes of each
# output, over n rows, S slots and H x W pixels (a digit: an axis of that constant size).
# Engine.render_masks, render_coverage, render_soft_masks and render_boxes take and return one
# output as a tensor, several as a tuple.
_MASK_KINDS = {
    'masks': ('swb_render_masks', (('masks', torch.uint8, 'nHW'),)),
    'coverage': ('swb_render_coverage', (('cover', torch.int32, 'nHW'), ('visible', torch.int32, 'nS'),
                                         ('area', torch.int32, 'nS'))),
    'soft': ('swb_render_soft_masks', (('soft', torch.uint8, 'nSHW'),)),
    'boxes': ('swb_render_boxes', (('visible_box', torch.int32, 'nS4'), ('amodal_box', torch.int32, 'nS4'),
                                   ('visible', torch.int32, 'nS'), ('area', torch.int32, 'nS'))),
}


def _mask_outputs(kind, n, n_slots, height, width):
  """[(name, dtype, shape)] of the outputs of sprite-mask observation `kind` for n rows."""
  size = dict(n=n, S=n_slots, H=height, W=width)
  return [(name, dtype, tuple(int(a) if a.isdigit() else size[a] for a in axes))
          for name, dtype, axes in _MASK_KINDS[kind][1]]


def _new_mask_outputs(engine, kind, n, width, height):
  """New tensors on `engine`'s device for what sprite-mask observation `kind` writes for n rows, in
  the form its call takes as `out`."""
  t = [torch.empty(shape, dtype=dtype, device=engine.device)
       for _, dtype, shape in _mask_outputs(kind, n, engine.n_slots, max(int(height), 0), max(int(width), 0))]
  return t[0] if len(t) == 1 else tuple(t)


def _render_sprite_masks(engine, kind, width, height, anti_aliasing=1, states=None, out=None):
  """The body of Engine.render_masks, render_coverage, render_soft_masks and render_boxes, for
  observation `kind`."""
  n, rec, rec_bytes = _rows(engine, states)
  W, H, aa = int(width), int(height), int(anti_aliasing)
  spec = _mask_outputs(kind, n, engine.n_slots, H, W)
  if out is None:
    out = _new_mask_outputs(engine, kind, n, W, H)
  elif len(spec) == 1:
    _check_output(out, *spec[0], engine.device)
  else:
    if not isinstance(out, (tuple, list)) or len(out) != len(spec):
      what = 'triple' if len(spec) == 3 else '%d-tuple' % len(spec)
      raise ValueError('out must be a (%s) %s, got %s' % (', '.join(s[0] for s in spec), what, type(out).__name__))
    for t, s in zip(out, spec):
      _check_output(t, *s, engine.device)
    out = tuple(out)
  call = getattr(engine._lib, _MASK_KINDS[kind][0])
  _native.check(call(engine._h, W, H, aa, rec, n, rec_bytes,
                     *[_address(t) for t in ((out,) if len(spec) == 1 else out)], engine._stream()))
  return out


def host_actions(kind, actions):
  """Host actions (array-like, one row per env) as a contiguous array the engine accepts.
  SelectMove / DragAndDrop: float32 stays float32, anything else becomes float64.  Embodied: int32
  (carry != 0, direction); a direction that is not an integer in 0..3 becomes -1, so the step
  reports ENV_BAD_ACTION (the reference's KeyError) rather than a wrapped or truncated move."""
  a = np.asarray(actions)
  if kind != 'embodied':
    return np.ascontiguousarray(a if a.dtype == np.float32 else a.astype(np.float64))
  if a.ndim == 0 or a.shape[-1] != 2:
    raise ValueError('Embodied actions must be (carry, direction) rows, got shape %s' % (a.shape,))
  valid = np.isin(a[..., 1], (0, 1, 2, 3))
  out = np.full(a.shape, -1, np.int32)
  out[..., 0] = a[..., 0] != 0
  out[..., 1][valid] = a[..., 1][valid]
  return out


def zero_actions(kind, n_envs):
  """All-zero host actions, for a step that resets every env (and so ignores them)."""
  return host_actions(kind, np.zeros((int(n_envs), ACTIONS[kind].columns), np.float32))


class SerialSnapshot(object):
  """scene_serial of every env as of the steps enqueued when it was requested; `wait()` blocks
  the calling host thread (not the step stream) until the copy has landed."""

  def __init__(self, host, event):
    self._host, self._event = host, event

  def ready(self):
    """True once the copy has landed (never blocks)."""
    return self._event.query()

  def wait(self):
    self._event.synchronize()
    return self._host.numpy().astype(np.int64)


class Raster(object):
  """PILRenderer(image_size=(width, height), anti_aliasing, bg_color) on the device."""

  def __init__(self, engine, width, height, anti_aliasing=1, bg_color=(0, 0, 0)):
    self.engine = engine
    self.width, self.height, self.anti_aliasing = int(width), int(height), int(anti_aliasing)
    bg = (ctypes.c_uint8 * 3)(*[int(c) for c in bg_color])
    h = ctypes.c_void_p()
    _native.check(engine._lib.swb_raster_create(engine._h, self.width, self.height,
                                                self.anti_aliasing, bg, ctypes.byref(h)))
    self._h = h

  def new_frames(self):
    return torch.empty((self.engine.n_envs, self.height, self.width, 3), dtype=torch.uint8,
                       device=self.engine.device)

  def close(self):
    if self._h:
      self.engine._lib.swb_raster_destroy(self._h)
      self._h = None

  def __del__(self):
    try:
      self.close()
    except Exception:  # pragma: no cover
      pass


class Engine(object):

  def __init__(self, n_envs, n_slots, pool_depth, action, nodes, shapes, keep_in_frame=True,
               max_episode_length=1000, device=0):
    """Args:
      action: dict(kind='select_move'|'drag_and_drop'|'embodied', scale=.., motion_cost=..)
      nodes: post-order list of task-node dicts (see tasks.compile_task)
      shapes: dict name -> (V, 2) float64 vertex arrays (constants.SHAPES)
    """
    if not torch.cuda.is_available():
      raise _native.NativeError('spriteworld_b200 needs a CUDA device; there is no CPU path')
    self._lib = _native.load()
    self.n_envs, self.n_slots, self.pool_depth = int(n_envs), int(n_slots), int(pool_depth)
    self.device = torch.device('cuda', device)
    self.action_kind = ACTIONS[action['kind']].kind
    cfg = make_config(n_envs, n_slots, pool_depth, action, nodes, shapes, keep_in_frame,
                      max_episode_length, device)
    self.signature = config_signature(cfg)
    h = ctypes.c_void_p()
    _native.check(self._lib.swb_engine_create(ctypes.byref(cfg), ctypes.byref(h)))
    self._h = h
    gp, ng = ctypes.c_void_p(), ctypes.c_int32()
    _native.check(self._lib.swb_pool_goal_pointer(h, ctypes.byref(gp), ctypes.byref(ng)))
    self.n_goals = ng.value   # G: goal slots per scene (sampled FindGoalPosition goals)
    E = self.n_envs
    # the four per-env outputs of a step are slices of ONE buffer (11 bytes per env: reward f64,
    # step_type i8, success u8, status u8), so that a multi-GPU gather moves them in one piece
    self.out_bytes = torch.zeros(E * OUT_BYTES_PER_ENV, dtype=torch.uint8, device=self.device)
    self._reward, self._step_type, self._success, self._status = split_outputs(self.out_bytes, E)
    self._out = _native.StepOut(self._reward.data_ptr(), self._step_type.data_ptr(),
                                self._success.data_ptr(), self._status.data_ptr())

  # -- lifetime -------------------------------------------------------------------
  def close(self):
    if getattr(self, '_h', None):
      self._lib.swb_engine_destroy(self._h)
      self._h = None

  def __del__(self):
    try:
      self.close()
    except Exception:  # pragma: no cover
      pass

  def _stream(self):
    return ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

  # -- scenes -----------------------------------------------------------------------
  def upload_scenes(self, scenes, env_ids, ring_slots):
    """scenes: dict of numpy arrays shaped (n, S[, ...]) (see scene.SceneBatch.arrays)."""
    n = len(env_ids)
    S = self.n_slots
    keep = []

    def arr(name, dtype, tail=()):
      a = np.ascontiguousarray(scenes[name], dtype=dtype)
      assert a.shape == (n, S) + tail, (name, a.shape, (n, S) + tail)
      keep.append(a)
      return a.ctypes.data

    soa = _native.SceneSoA()
    for f in SCENE_FIELDS_F64:
      setattr(soa, f, arr(f, np.float64))
    soa.member = arr('member', np.uint32)
    soa.shape = arr('shape', np.uint8)
    soa.pos_f32 = arr('pos_f32', np.uint8)
    soa.rgb = arr('rgb', np.uint8, (3,))
    soa.factors = arr('factors', np.float32, (5,)) if 'factors' in scenes else None
    if self.n_goals:
      goal = np.ascontiguousarray(scenes['goal'], dtype=np.float64)
      assert goal.shape == (n, self.n_goals, 2), ('goal', goal.shape, (n, self.n_goals, 2))
      keep.append(goal)
      soa.goal = goal.ctypes.data
    env_ids = np.ascontiguousarray(env_ids, dtype=np.int32)
    ring_slots = np.ascontiguousarray(ring_slots, dtype=np.int32)
    _native.check(self._lib.swb_upload_scenes(self._h, ctypes.byref(soa), _as_ptr(env_ids),
                                              _as_ptr(ring_slots), n, self._stream()))

  def scene_serial(self):
    """Zero-copy int32 (E,) view of how many scenes each env has started (monotonic)."""
    if getattr(self, '_serial_view', None) is None:
      p = ctypes.c_void_p()
      _native.check(self._lib.swb_scene_serial_pointer(self._h, ctypes.byref(p)))
      self._serial_view = torch.as_tensor(_DevicePointer(p.value, (self.n_envs,), '<i4'),
                                          device=self.device)
    return self._serial_view

  def side_stream(self):
    """The engine's stream for work that must not hold up the step stream (scene refills)."""
    if getattr(self, '_side', None) is None:
      self._side = torch.cuda.Stream(device=self.device)
    return self._side

  def snapshot_scene_serial(self):
    """Asynchronous device->pinned copy of scene_serial, ordered after the work enqueued so far
    on the current stream and issued on the side stream.  Returns a SerialSnapshot."""
    if getattr(self, '_serial_host', None) is None:
      # a ring of pinned buffers: the batched environment keeps its last dozen snapshots around
      self._serial_host = [torch.empty(self.n_envs, dtype=torch.int32).pin_memory() for _ in range(16)]
      self._serial_i = 0
    side = self.side_stream()
    ev = torch.cuda.Event()
    ev.record(torch.cuda.current_stream(self.device))
    side.wait_event(ev)
    host = self._serial_host[self._serial_i]
    self._serial_i = (self._serial_i + 1) % len(self._serial_host)
    with torch.cuda.stream(side):
      host.copy_(self.scene_serial(), non_blocking=True)
      done = torch.cuda.Event()
      done.record(side)
    return SerialSnapshot(host, done)

  def side_stream_context(self):
    """Context in which this thread's CUDA work (scene uploads, pool bookkeeping) goes to the
    side stream of this engine's device."""
    torch.cuda.set_device(self.device)
    return torch.cuda.stream(self.side_stream())

  def record_side_event(self):
    """An event after the work enqueued so far on the side stream (for wait_event)."""
    done = torch.cuda.Event()
    done.record(self.side_stream())
    return done

  def download_state_serial(self):
    """scene_serial as a host array, after everything enqueued so far (synchronous)."""
    return self.scene_serial().cpu().numpy().astype(np.int64)

  def wait_event(self, event):
    """Makes the current (step) stream wait for `event` without blocking the host."""
    torch.cuda.current_stream(self.device).wait_event(event)

  def request_reset(self, mask=None):
    ptr = None
    if mask is not None:
      mask = mask.to(device=self.device, dtype=torch.uint8).contiguous()
      ptr = ctypes.c_void_p(mask.data_ptr())
    _native.check(self._lib.swb_request_reset(self._h, ptr, self._stream()))

  # -- stepping ---------------------------------------------------------------------
  def _check_frames(self, frames, raster, n_frames):
    """ValueError unless `frames` holds n_frames frames of `raster` as the render kernel writes them."""
    _check_output(frames, 'frames', torch.uint8, (n_frames, raster.height, raster.width, 3), self.device)

  def step(self, actions, raster=None, frames=None):
    """One Environment.step for every env.  `actions`: device tensor."""
    dt = action_dtype(self.action_kind, self.n_envs, actions, self.device)
    if raster is None:
      _native.check(self._lib.swb_step(self._h, ctypes.c_void_p(actions.data_ptr()), dt,
                                       ctypes.byref(self._out), self._stream()))
    else:
      if frames is None:
        frames = raster.new_frames()
      self._check_frames(frames, raster, self.n_envs)
      _native.check(self._lib.swb_step_render(
          self._h, raster._h, ctypes.c_void_p(actions.data_ptr()), dt, ctypes.byref(self._out),
          ctypes.c_void_p(frames.data_ptr()), self._stream()))
    return StepResult(self._reward, self._step_type, self._success, self._status, frames)

  def rollout(self, actions, out=None, states=None, leaves=None, trajectory=None):
    """What each of C candidate action sequences of T steps would earn from the state every env is
    in now, in one launch that changes nothing (swb_rollout).  `actions`: device tensor
    (T, n_envs, C, columns) of a dtype step() takes.  Returns a RolloutResult; with `out`, a packed
    uint8 tensor of T * n_envs * C * OUT_BYTES_PER_ENV bytes, its tensors are views of that.

    `states`: EnvStates of n roots of this engine's configuration (any n >= 1) to plan from instead
    of the live envs; actions and outputs are then (T, n, C, ...).  `leaves`: True for new
    EnvStates of the n * C states the plans end in (RolloutResult.leaves), or EnvStates of n * C
    records to fill in place; record r * C + c is what save_envs would return after loading root r
    and stepping plan c's live steps.  Leaves carry the roots' span class.  Still one launch
    (swb_rollout_states).

    `trajectory`: True for new EnvStates of the T * n * C states after every step
    (RolloutResult.trajectory), or EnvStates of T * n * C records to fill in place; record
    (t * n + r) * C + c is leaf r * C + c of the same call with actions[:t + 1], so the last n * C
    records are the leaves.  Not with `leaves`.  Still one launch (swb_rollout_trajectory)."""
    if trajectory is not None and leaves is not None:
      raise ValueError('trajectory and leaves are exclusive: the leaves are the last n * C records of '
                       'the trajectory')
    n, roots, roots_bytes = _rows(self, states)
    dt = action_dtype(self.action_kind, n, actions, self.device, plans=True)
    T, _, C, _ = actions.shape
    records, n_records = (leaves, n * C) if trajectory is None else (trajectory, T * n * C)
    if records is True:
      records = EnvStates(torch.empty((n_records, self.record_bytes), dtype=torch.uint8, device=self.device),
                          1, self.signature, self.n_slots, self.n_goals)
    elif records is not None:
      self.check_states(records, n_records)
    out, res = rollout_outputs(out, T, n, C, self.device)
    ptrs = _native.StepOut(res.reward.data_ptr(), res.step_type.data_ptr(), res.success.data_ptr(),
                           res.status.data_ptr())
    if states is None and records is None:
      _native.check(self._lib.swb_rollout(self._h, ctypes.c_void_p(actions.data_ptr()), dt, T, C,
                                          ctypes.byref(ptrs), self._stream()))
      return res
    span = ctypes.c_int32(1 if states is None else states.span_class)
    dst = (None, 0) if records is None else (ctypes.c_void_p(records.data.data_ptr()), records.data.numel())
    call = self._lib.swb_rollout_states if trajectory is None else self._lib.swb_rollout_trajectory
    _native.check(call(self._h, roots, n, roots_bytes, ctypes.c_void_p(actions.data_ptr()), dt, T, C,
                       ctypes.byref(ptrs), dst[0], dst[1], ctypes.byref(span), self._stream()))
    if records is not None:
      records.span_class = span.value
    if trajectory is None:
      res.leaves = records
    else:
      res.trajectory = records
    return res

  def step_gather(self, actions, raster, targets):
    """Environment.step for every env with the frame gather fused into the render kernel:
    each finished frame is stored into every rank's gathered buffer (`targets`, a
    distributed.PeerFrames slot) over NVLink peer memory.  Returns the StepResult with the
    local rank's gathered tensor as `frames`; it is whole after `targets.barrier()`."""
    dt = action_dtype(self.action_kind, self.n_envs, actions, self.device)
    ptrs, n, env_offset, local = targets
    self._check_frames(local, raster, int(n) * self.n_envs)
    _native.check(self._lib.swb_step_render_gather(
        self._h, raster._h, ctypes.c_void_p(actions.data_ptr()), dt, ctypes.byref(self._out),
        ptrs, n, env_offset, self._stream()))
    return StepResult(self._reward, self._step_type, self._success, self._status, local)

  def render(self, raster, frames=None):
    if frames is None:
      frames = raster.new_frames()
    self._check_frames(frames, raster, self.n_envs)
    _native.check(self._lib.swb_render(self._h, raster._h, ctypes.c_void_p(frames.data_ptr()),
                                       self._stream()))
    return frames

  def render_states(self, raster, states, frames=None, status=None):
    """The frames of env records without loading them (swb_render_states): frame i is what
    render() would draw after load_envs of record i, status[i] its render status
    (ENV_SPAN_OVERFLOW).  `states`: EnvStates of any n records of this engine's configuration.
    Returns (frames (n, H, W, 3) uint8, status (n,) uint8) on this device, new unless given.  One
    launch on the current stream; no env, frame buffer, render_status() or span class changes."""
    n, rec, rec_bytes = _rows(self, states, live=False)
    if frames is None:
      frames = torch.empty((n, raster.height, raster.width, 3), dtype=torch.uint8, device=self.device)
    self._check_frames(frames, raster, n)
    if status is None:
      status = torch.empty(n, dtype=torch.uint8, device=self.device)
    _check_output(status, 'status', torch.uint8, (n,), self.device)
    _native.check(self._lib.swb_render_states(
        self._h, raster._h, rec, n, rec_bytes, states.span_class, _address(frames), _address(status),
        self._stream()))
    return frames, status

  def render_windows(self, raster, windows, states=None, frames=None, status=None, draw=None):
    """The scene seen through windows (swb_render_windows): frame (i, v) is `raster`'s PILRenderer
    frame of row i with the window windows[i, v] = (x0, y0, x1, y1) of scene coordinates stretched
    over the whole raster, so (0, 0, 1, 1) draws what render() / render_states() draw.  Rows are the
    live envs (n = n_envs), or with `states` EnvStates of any n records, as if loaded.  `windows`: a
    contiguous float64 (n, V, 4) tensor on this device, V >= 1.  Returns (frames (n, V, H, W, 3)
    uint8, status (n, V) uint8: ENV_BAD_WINDOW for an empty or non-finite window or a vertex 2^30
    canvas pixels or more away, whose frame is zeros, and ENV_SPAN_OVERFLOW), new unless given.  One
    launch on the current stream; nothing else changes.

    `draw` (swb_render_views): a contiguous bool (n, V, n_slots) tensor on this device; view (i, v)
    then draws only the slots s with draw[i, v, s], as if every other slot were empty, and its
    status counts those slots only.  None draws every slot."""
    n, rec, rec_bytes = _rows(self, states)
    if not isinstance(windows, torch.Tensor) or windows.dim() != 3 or windows.shape[-1] != 4 or windows.shape[1] < 1:
      raise ValueError('windows must be a float64 (n, V, 4) tensor with V >= 1, got %s' % _describe(windows))
    V = int(windows.shape[1])
    _check_output(windows, 'windows', torch.float64, (n, V, 4), self.device, align=8)
    if draw is not None:
      _check_output(draw, 'draw', torch.bool, (n, V, self.n_slots), self.device)
    if frames is None:
      frames = torch.empty((n, V, raster.height, raster.width, 3), dtype=torch.uint8, device=self.device)
    _check_output(frames, 'frames', torch.uint8, (n, V, raster.height, raster.width, 3), self.device)
    if status is None:
      status = torch.empty((n, V), dtype=torch.uint8, device=self.device)
    _check_output(status, 'status', torch.uint8, (n, V), self.device)
    span = 1 if states is None else states.span_class
    if draw is None:
      _native.check(self._lib.swb_render_windows(
          self._h, raster._h, rec, n, rec_bytes, span, _address(windows), V, _address(frames), _address(status),
          self._stream()))
    else:
      _native.check(self._lib.swb_render_views(
          self._h, raster._h, rec, n, rec_bytes, span, _address(windows), _address(draw), V, _address(frames),
          _address(status), self._stream()))
    return frames, status

  def render_masks(self, width, height, anti_aliasing=1, states=None, out=None):
    """Sprite instance masks (swb_render_masks): uint8 (n, height, width), pixel value k + 1 where
    slot k is the top-most sprite covering the pixel's sample point on PILRenderer's
    anti_aliasing-times canvas, 0 where none does (renderers.SpriteMasks).  Of the live envs (n =
    n_envs), or with `states` of EnvStates of any n records, as if loaded.  Into `out` if given
    (a contiguous uint8 tensor of that shape on this device), else a new tensor.  One launch on the
    current stream; nothing else changes."""
    return _render_sprite_masks(self, 'masks', width, height, anti_aliasing, states, out)

  def render_coverage(self, width, height, anti_aliasing=1, states=None, out=None):
    """Amodal sprite coverage (swb_render_coverage): (cover, visible, area), int32 (n, height,
    width), (n, n_slots) and (n, n_slots).  Bit k of a cover pixel is set where slot k's polygon
    covers the pixel's sample point (the one render_masks samples), whether or not a sprite above
    hides it; visible[i, k] counts the pixels where slot k is the top-most covering sprite (the mask
    render_masks draws is k + 1 there), area[i, k] those where bit k is set (renderers.SpriteCoverage).
    Of the live envs (n = n_envs), or with `states` of EnvStates of any n records, as if loaded.
    Into `out` if given (a triple of contiguous int32 tensors of those shapes on this device), else
    new tensors.  One launch on the current stream (after zeroing the counts); nothing else changes."""
    return _render_sprite_masks(self, 'coverage', width, height, anti_aliasing, states, out)

  def render_soft_masks(self, width, height, anti_aliasing=1, states=None, out=None):
    """Soft sprite masks (swb_render_soft_masks): uint8 (n, n_slots, height, width), where
    soft[i, k, r, c] counts the canvas pixels of mask pixel (r, c)'s anti_aliasing x anti_aliasing
    block on PILRenderer's canvas whose top-most covering sprite is slot k (the pixel render_masks
    draws k + 1 at samples the block's centre one); soft / anti_aliasing**2 is the slot's share of
    the pixel (renderers.SoftSpriteMasks).  anti_aliasing at most 15.  Of the live envs (n =
    n_envs), or with `states` of EnvStates of any n records, as if loaded.  Into `out` if given (a
    contiguous uint8 tensor of that shape on this device), else a new tensor.  One launch on the
    current stream; nothing else changes."""
    return _render_sprite_masks(self, 'soft', width, height, anti_aliasing, states, out)

  def render_boxes(self, width, height, anti_aliasing=1, states=None, out=None):
    """Sprite bounding boxes (swb_render_boxes): (visible_box, amodal_box, visible, area), int32
    (n, n_slots, 4), (n, n_slots, 4), (n, n_slots) and (n, n_slots).  Over the pixels where slot k
    is the top-most covering sprite (the mask render_masks draws is k + 1) and over those where its
    bit of render_coverage's cover is set: the half-open pixel box (x0, y0, x1, y1) = (min column,
    min row, max column + 1, max row + 1), (0, 0, 0, 0) for no pixel, and the pixel counts, which
    are render_coverage's (renderers.SpriteBoxes).  Of the live envs (n = n_envs), or with `states`
    of EnvStates of any n records, as if loaded.  Into `out` if given (a 4-tuple of contiguous
    int32 tensors of those shapes on this device), else new tensors.  Two launches on the current
    stream (after zeroing the four outputs); nothing else changes."""
    return _render_sprite_masks(self, 'boxes', width, height, anti_aliasing, states, out)

  def render_status(self):
    """Zero-copy uint8 (E,) view of the per-env status of the last render() (ENV_SPAN_OVERFLOW)."""
    if getattr(self, '_render_status_view', None) is None:
      p = ctypes.c_void_p()
      _native.check(self._lib.swb_render_status_pointer(self._h, ctypes.byref(p)))
      self._render_status_view = torch.as_tensor(_DevicePointer(p.value, (self.n_envs,), '|u1'),
                                                 device=self.device)
    return self._render_status_view

  def check_render(self):
    """Raises if the last render() overflowed its span tables for any env (the frame would be
    wrong).  Synchronises."""
    if int(self.render_status().max().item()) & _native.ENV_SPAN_OVERFLOW:
      raise _native.NativeError(
          'render: a canvas row has more crossings, spans or visible segments than the engine '
          'was sized for (once a star or spoke shape is uploaded, at most 16 visible segments '
          'per canvas row; see DESIGN.md section 8)')

  def step_host(self, actions, raster=None, want_frames=True, out=None):
    """Whole call with HOST buffers (numpy in, numpy out): H2D, step, render, D2H, sync.

    `out`: optional dict of preallocated (ideally pinned) numpy arrays reward/step_type/
    success/status/frames to receive the results.
    """
    # swb_step_host reads E rows of 2 int32 or 4 floats from the buffer: check what step() checks
    a = np.ascontiguousarray(actions)
    dt = action_dtype(self.action_kind, self.n_envs, a)
    E = self.n_envs
    out = out or {}
    reward = out.get('reward') if 'reward' in out else np.empty(E, np.float64)
    step_type = out.get('step_type') if 'step_type' in out else np.empty(E, np.int8)
    success = out.get('success') if 'success' in out else np.empty(E, np.uint8)
    status = out.get('status') if 'status' in out else np.empty(E, np.uint8)
    frames = None
    if raster is not None and want_frames:
      frames = (out.get('frames') if 'frames' in out
                else np.empty((E, raster.height, raster.width, 3), np.uint8))
    _native.check(self._lib.swb_step_host(
        self._h, raster._h if raster is not None else None, _as_ptr(a), dt, _as_ptr(reward),
        _as_ptr(step_type), _as_ptr(success), _as_ptr(status),
        _as_ptr(frames) if frames is not None else None, self._stream()))
    return reward, step_type, success, status, frames

  # -- state ------------------------------------------------------------------------
  def download_state(self):
    E, S = self.n_envs, self.n_slots
    px, py = np.empty((E, S)), np.empty((E, S))
    cursor, count = np.empty(E, np.int32), np.empty(E, np.int32)
    reset_next = np.empty(E, np.uint8)
    _native.check(self._lib.swb_download_state(self._h, _as_ptr(px), _as_ptr(py), _as_ptr(cursor),
                                               _as_ptr(count), _as_ptr(reset_next),
                                               self._stream()))
    return dict(pos_x=px, pos_y=py, cursor=cursor, step_count=count, reset_next=reset_next)

  def upload_state(self, pos_x=None, pos_y=None, cursor=None, step_count=None, reset_next=None):
    def p(a, dtype):
      if a is None:
        return None, None
      a = np.ascontiguousarray(a, dtype=dtype)
      return a, _as_ptr(a)
    k1, a1 = p(pos_x, np.float64)
    k2, a2 = p(pos_y, np.float64)
    k3, a3 = p(cursor, np.int32)
    k4, a4 = p(step_count, np.int32)
    k5, a5 = p(reset_next, np.uint8)
    _native.check(self._lib.swb_upload_state(self._h, a1, a2, a3, a4, a5, self._stream()))

  def state_tensors(self):
    """Zero-copy torch views of the live device state: pos_x/pos_y (E, S) float64,
    cursor/step_count (E,) int32, reset_next (E,) uint8."""
    ptrs = [ctypes.c_void_p() for _ in range(5)]
    _native.check(self._lib.swb_state_pointers(self._h, *[ctypes.byref(p) for p in ptrs]))
    E, S = self.n_envs, self.n_slots
    spec = [('pos_x', (E, S), '<f8'), ('pos_y', (E, S), '<f8'), ('cursor', (E,), '<i4'),
            ('step_count', (E,), '<i4'), ('reset_next', (E,), '|u1')]
    out = {}
    for (name, shape, typestr), ptr in zip(spec, ptrs):
      out[name] = torch.as_tensor(_DevicePointer(ptr.value, shape, typestr), device=self.device)
    return out

  # -- checkpoints ------------------------------------------------------------------
  def state_bytes(self):
    """Bytes of this engine's checkpoint (swb_engine_state_bytes)."""
    return int(self._lib.swb_engine_state_bytes(self._h))

  def save_state(self):
    """The whole engine state -- live positions and counters, every ring's scenes, the device
    sampler's refill bookkeeping -- as a CPU uint8 tensor in the self-describing layout of
    include/spriteworld_b200.h (swb_save_engine), after the work enqueued on the current stream.
    Synchronises that stream; changes nothing."""
    out = torch.empty(self.state_bytes(), dtype=torch.uint8)
    _native.check(self._lib.swb_save_engine(self._h, ctypes.c_void_p(out.data_ptr()), out.numel(),
                                            self._stream()))
    return out

  def load_state(self, state):
    """Loads a save_state() of an engine of this configuration (same n_envs, pool_depth and
    signature, and a device sampler of the same seed and env_offset, or none on both sides).  The
    library checks every byte before anything is enqueued and raises NativeError naming the first
    bad field, index and value; the copies go to the current stream."""
    if (not isinstance(state, torch.Tensor) or state.dtype != torch.uint8 or state.device.type != 'cpu'
        or state.dim() != 1):
      raise ValueError('state must be a one-dimensional CPU uint8 tensor (save_state()), got %s'
                       % _describe(state))
    state = state.contiguous()
    _native.check(self._lib.swb_load_engine(self._h, ctypes.c_void_p(state.data_ptr()), state.numel(),
                                            self._stream()))

  # -- env records ------------------------------------------------------------------
  # Ids are lists, ndarrays or tensors; with check='host' (the default) the library checks them on
  # the host, so a CUDA tensor of ids costs a device-to-host copy (env_ids_array).  With
  # check='device' the ids are an int32 or int64 tensor on this engine's device, checked by kernels
  # without the host waiting for them: a refused call changes nothing, and check_env_ids() reports
  # it.  The work goes to the current stream.
  @property
  def record_bytes(self):
    """Bytes of one env record (include/spriteworld_b200.h)."""
    return int(self._lib.swb_env_record_bytes(self._h))

  def _all_or(self, env_ids):
    return np.arange(self.n_envs, dtype=np.int32) if env_ids is None else env_ids_array(env_ids)

  def save_envs(self, env_ids=None, check='host'):
    """EnvStates of envs `env_ids` (default: all, in order), on this engine's device.  With
    check='device', a save refused on the device returns zero records."""
    rb = self.record_bytes
    span = ctypes.c_int32()
    if device_checked(check, env_ids):
      ids, dt = self._dev_ids(env_ids, 'save_envs')
      data = torch.empty((ids.numel(), rb), dtype=torch.uint8, device=self.device)
      _native.check(self._lib.swb_save_envs_dev(self._h, ctypes.c_void_p(ids.data_ptr()), dt, ids.numel(),
                                                ctypes.c_void_p(data.data_ptr()), data.numel(),
                                                ctypes.byref(span), self._stream()))
      return EnvStates(data, span.value, self.signature, self.n_slots, self.n_goals)
    ids = self._all_or(env_ids)
    data = torch.empty((len(ids), rb), dtype=torch.uint8, device=self.device)
    _native.check(self._lib.swb_save_envs(self._h, _as_ptr(ids), len(ids), ctypes.c_void_p(data.data_ptr()),
                                          data.numel(), ctypes.byref(span), self._stream()))
    return EnvStates(data, span.value, self.signature, self.n_slots, self.n_goals)

  def check_states(self, states, n):
    """ValueError unless `states` holds n records that this engine can load."""
    if not isinstance(states, EnvStates):
      raise ValueError('expected EnvStates, got %s' % type(states).__name__)
    if states.signature != self.signature:
      raise ValueError('EnvStates were saved by an engine of another configuration (slot count, '
                       'action space, task tree, shape table, keep_in_frame or max_episode_length)')
    d = states.data
    if (d.dtype != torch.uint8 or d.device != self.device or tuple(d.shape) != (n, self.record_bytes)
        or not d.is_contiguous() or d.data_ptr() % 16):
      raise ValueError('EnvStates must hold a contiguous, 16-byte aligned uint8 (%d, %d) tensor on '
                       '%s, got %s' % (n, self.record_bytes, self.device, _describe(d)))

  def load_envs(self, states, env_ids=None, check='host'):
    """Env env_ids[i] <- record i of `states` (default ids: all envs, in order; distinct)."""
    if device_checked(check, env_ids):
      ids, dt = self._dev_ids(env_ids, 'load_envs')
      self.check_states(states, ids.numel())
      _native.check(self._lib.swb_load_envs_dev(self._h, ctypes.c_void_p(ids.data_ptr()), dt, ids.numel(),
                                                ctypes.c_void_p(states.data.data_ptr()), states.data.numel(),
                                                states.span_class, self._stream()))
      return
    ids = self._all_or(env_ids)
    self.check_states(states, len(ids))
    _native.check(self._lib.swb_load_envs(self._h, _as_ptr(ids), len(ids),
                                          ctypes.c_void_p(states.data.data_ptr()), states.data.numel(),
                                          states.span_class, self._stream()))

  def copy_envs(self, src_ids, dst_ids, check='host'):
    """Env dst_ids[i] <- env src_ids[i]; every read sees the state from before the call."""
    if device_checked(check, src_ids):
      src, dt = self._dev_ids(src_ids, 'copy_envs')
      dst, dt_dst = self._dev_ids(dst_ids, 'copy_envs')
      if src.numel() != dst.numel():
        raise ValueError('copy_envs: %d sources, %d destinations' % (src.numel(), dst.numel()))
      if dt != dt_dst:    # one id type per call: widen the int32 side on the device
        src, dst, dt = src.long(), dst.long(), _native.DTYPE_I64
      _native.check(self._lib.swb_copy_envs_dev(self._h, ctypes.c_void_p(src.data_ptr()),
                                                ctypes.c_void_p(dst.data_ptr()), dt, src.numel(),
                                                self._stream()))
      return
    src, dst = env_ids_array(src_ids), env_ids_array(dst_ids)
    if len(src) != len(dst):
      raise ValueError('copy_envs: %d sources, %d destinations' % (len(src), len(dst)))
    _native.check(self._lib.swb_copy_envs(self._h, _as_ptr(src), _as_ptr(dst), len(src), self._stream()))

  def _dev_ids(self, ids, fn):
    """(contiguous ids, swb id dtype) of a device-checked call.  Nothing here reads the ids or
    waits for the device; a non-contiguous tensor is made contiguous on the device."""
    if not (isinstance(ids, torch.Tensor) and ids.device == self.device and ids.dtype in _ID_DTYPES
            and ids.dim() == 1):
      raise ValueError("%s with check='device' takes one-dimensional int32 or int64 ids on %s, got %s"
                       % (fn, self.device, _describe(ids)))
    return ids.contiguous(), _ID_DTYPES[ids.dtype]

  def env_ids_status(self):
    """Zero-copy uint8 (32,) view of the engine's swb_ids_status record (include/spriteworld_b200.h)."""
    if getattr(self, '_ids_status_view', None) is None:
      p = ctypes.c_void_p()
      _native.check(self._lib.swb_env_ids_status_pointer(self._h, ctypes.byref(p)))
      self._ids_status_view = torch.as_tensor(_DevicePointer(p.value, (_IDS_STATUS.itemsize,), '|u1'),
                                              device=self.device)
    return self._ids_status_view

  def env_ids_ok(self):
    """0-dim bool device tensor: True if the last device-checked record call passed its id checks.
    Read in stream order, it masks work that follows a call without waiting for it."""
    return self.env_ids_status()[:4].view(torch.int32)[0] != 0

  def check_env_ids(self):
    """Raises ValueError naming the call, the argument, the position, the id and the reason if a
    device-checked save_envs / load_envs / copy_envs has been refused since the last check (the
    first such), and clears the record.  Synchronises."""
    view = self.env_ids_status()
    rec = view.cpu().numpy().view(_IDS_STATUS)[0]
    if not rec['failed']:
      return
    view[4:].zero_()
    fn = _IDS_CALLS[int(rec['call'])]
    arg = ('src_ids', 'dst_ids')[int(rec['arg'])] if fn == 'copy_envs' else 'env_ids'
    why = ('is out of range [0, %d)' % self.n_envs if rec['reason'] == _native.IDS_OUT_OF_RANGE
           else 'repeats a destination at a lower position')
    raise ValueError('%s: %s[%d] = %d %s' % (fn, arg, int(rec['position']), int(rec['value']), why))

  # -- device scene sampler ---------------------------------------------------------------
  def load_sampler(self, program, seed, env_offset=0):
    """Gives the engine a scene_program.SceneProgram and a seed; env e is global env
    env_offset + e.  Synchronises; no scene is sampled until refill_device() or sample_scenes()."""
    from spriteworld_b200 import scene_program
    if self._lib.swb_sampler_sizeof_program() != ctypes.sizeof(scene_program.Program):
      raise _native.NativeError('ABI mismatch: swb_scene_program')
    _native.check(self._lib.swb_sampler_load(self._h, ctypes.byref(program.struct),
                                             int(seed) & (2 ** 64 - 1), int(env_offset)))
    self._program = program
    self._refilled_view = self._sampler_status_view = None

  def sample_scenes(self, env_ids, scene_idx):
    """Scenes (env_ids[i], scene_idx[i]) (global env ids, absolute scene indices) as device
    tensors: the fields of a scene batch shaped (n, S[, ...]) plus 'factor_value' float64 and
    'factor_kind' uint8 (n, S, 10), and with sampled goals 'goal' float64 (n, G, 2).  The pool is
    not touched."""
    from spriteworld_b200 import scene_program
    ids = torch.as_tensor(env_ids, dtype=torch.int64, device=self.device).contiguous()
    idx = torch.as_tensor(scene_idx, dtype=torch.int64, device=self.device).contiguous()
    if ids.dim() != 1 or ids.shape != idx.shape:
      raise ValueError('env_ids and scene_idx must be one-dimensional and of one length')
    n, S = ids.numel(), self.n_slots
    f64 = dict(dtype=torch.float64, device=self.device)
    out = {f: torch.zeros((n, S), **f64) for f in SCENE_FIELDS_F64}
    out['member'] = torch.zeros((n, S), dtype=torch.int32, device=self.device)
    for f in ('shape', 'pos_f32'):
      out[f] = torch.zeros((n, S), dtype=torch.uint8, device=self.device)
    out['rgb'] = torch.zeros((n, S, 3), dtype=torch.uint8, device=self.device)
    out['factors'] = torch.zeros((n, S, 5), dtype=torch.float32, device=self.device)
    out['factor_value'] = torch.zeros((n, S, 10), **f64)
    out['factor_kind'] = torch.zeros((n, S, 10), dtype=torch.uint8, device=self.device)
    if self.n_goals:
      out['goal'] = torch.zeros((n, self.n_goals, 2), **f64)
    st = scene_program.sample_out_struct(out, lambda t: t.data_ptr())
    _native.check(self._lib.swb_sample_scenes(self._h, ctypes.c_void_p(ids.data_ptr()),
                                              ctypes.c_void_p(idx.data_ptr()), n, ctypes.byref(st),
                                              self._stream()))
    return out

  def refill_device(self):
    """Enqueues the device refill: every env's ring up to scene_serial + K - 1."""
    _native.check(self._lib.swb_refill_device(self._h, self._stream()))

  def pool_tensors(self):
    """Zero-copy views of the scene pool, shaped (E, K, S[, ...]): x .. vy float64, member int32,
    shape and pos_f32 uint8, rgb uint8 (E, K, S, 4) (r, g, b, 0), factors float32 (E, K, S, 5), and
    with sampled goals (n_goals = G > 0) goal float64 (E, K, G, 2)."""
    if getattr(self, '_pool_views', None) is None:
      vp = ctypes.c_void_p
      f64 = (vp * 8)()
      ptrs = [vp() for _ in range(5)]
      _native.check(self._lib.swb_pool_pointers(self._h, f64, *[ctypes.byref(p) for p in ptrs]))
      E, K, S = self.n_envs, self.pool_depth, self.n_slots

      def view(p, typestr, tail=()):
        return torch.as_tensor(_DevicePointer(p, (E, K, S) + tail, typestr), device=self.device)

      out = {f: view(f64[i], '<f8') for i, f in enumerate(SCENE_FIELDS_F64)}
      out['member'] = view(ptrs[0].value, '<i4')
      out['shape'] = view(ptrs[1].value, '|u1')
      out['pos_f32'] = view(ptrs[2].value, '|u1')
      out['rgb'] = view(ptrs[3].value, '|u1', (4,))
      out['factors'] = view(ptrs[4].value, '<f4', (5,))
      if self.n_goals:
        gp, ng = ctypes.c_void_p(), ctypes.c_int32()
        _native.check(self._lib.swb_pool_goal_pointer(self._h, ctypes.byref(gp), ctypes.byref(ng)))
        out['goal'] = torch.as_tensor(_DevicePointer(gp.value, (E, K, self.n_goals, 2), '<f8'),
                                      device=self.device)
      self._pool_views = out
    return self._pool_views

  def _sampler_views(self):
    if getattr(self, '_refilled_view', None) is None:
      p, q = ctypes.c_void_p(), ctypes.c_void_p()
      _native.check(self._lib.swb_sampler_pointers(self._h, ctypes.byref(p), ctypes.byref(q)))
      self._refilled_view = torch.as_tensor(_DevicePointer(p.value, (self.n_envs,), '<i8'),
                                            device=self.device)
      self._sampler_status_view = torch.as_tensor(_DevicePointer(q.value, (3,), '<i8'),
                                                  device=self.device)
    return self._refilled_view, self._sampler_status_view

  def refilled_upto(self):
    """Zero-copy int64 (E,) view: the newest scene each env's ring holds (-1: none yet)."""
    return self._sampler_views()[0]

  def check_sampler(self):
    """Raises the reference's ValueError if a rejection loop of the device sampler ran out of
    tries since the last check (the first such; its scene was left empty), and clears the record.
    Synchronises."""
    view = self._sampler_views()[1]
    rec = view.cpu().numpy()
    if not rec[0] & 0xFFFFFFFF:
      return
    view.zero_()
    op = int(rec[0] >> 32)
    err = self._program.error(op)
    raise ValueError('%s (env %d, scene %d)' % (err.args[0], int(rec[1]), int(rec[2])))

  # -- sampled goals ----------------------------------------------------------------------
  def _check_goals(self, goals, n, fn):
    """ValueError unless `goals` is a contiguous float64 (n, G, 2) tensor on this engine's device."""
    if not self.n_goals:
      raise ValueError('%s: the task tree samples no goals' % fn)
    if (not isinstance(goals, torch.Tensor) or goals.dtype != torch.float64 or goals.device != self.device
        or tuple(goals.shape) != (n, self.n_goals, 2)):
      raise ValueError('%s takes float64 goals (%d, %d, 2) on %s, got %s'
                       % (fn, n, self.n_goals, self.device, _describe(goals)))
    return goals.contiguous()

  def set_goals(self, goals, env_ids=None, check='host'):
    """The goals of the scene env env_ids[i] is on <- goals[i] (default ids: all envs, in order;
    distinct), until the env starts its next scene.  `goals`: float64 (n, G, 2) on this engine's
    device.  Ids as load_envs takes them; with check='device' a refused call changes nothing and
    check_env_ids() reports it."""
    if device_checked(check, env_ids):
      ids, dt = self._dev_ids(env_ids, 'set_goals')
      goals = self._check_goals(goals, ids.numel(), 'set_goals')
      _native.check(self._lib.swb_set_goals_dev(self._h, ctypes.c_void_p(ids.data_ptr()), dt, ids.numel(),
                                                ctypes.c_void_p(goals.data_ptr()), self._stream()))
      return
    ids = self._all_or(env_ids)
    goals = self._check_goals(goals, len(ids), 'set_goals')
    _native.check(self._lib.swb_set_goals(self._h, _as_ptr(ids), len(ids), ctypes.c_void_p(goals.data_ptr()),
                                          self._stream()))

  def evaluate(self, states, goals=None):
    """(reward float64, success uint8, status uint8) device tensors (n,): the task tree's value on
    each record of `states` at its live positions (no action cost), with goals[i] (float64
    (n, G, 2) on this engine's device) in place of record i's goals if given.  One launch; reads
    only."""
    n, rec, rec_bytes = _rows(self, states, live=False)
    if goals is not None:
      goals = self._check_goals(goals, n, 'evaluate')
    reward = torch.empty(n, dtype=torch.float64, device=self.device)
    success = torch.empty(n, dtype=torch.uint8, device=self.device)
    status = torch.empty(n, dtype=torch.uint8, device=self.device)
    _native.check(self._lib.swb_evaluate_states(
        self._h, rec, n, rec_bytes, None if goals is None else ctypes.c_void_p(goals.data_ptr()),
        *[_address(t) for t in (reward, success, status)], self._stream()))
    return reward, success, status

  def sample_contained(self, seed, n_samples=1, states=None):
    """Positions inside sprites (swb_sample_contained): n_samples draws per row of the live envs
    (n = n_envs), or of the records of EnvStates `states`.  Sample s of row i picks one of the
    row's sprites uniformly and rejection-samples a point of it, from the Philox stream
    (seed, SWB_CONTAINED_DOMAIN) at counter (block, s, i, 0): a pure function of (seed, i, s, the
    row's state).  Returns new tensors on this device: position float64 (n, n_samples, 2), slot int8
    (n, n_samples) and status uint8 (n, n_samples) (ENV_NO_SPRITE, ENV_SAMPLE_TRIES; a failed
    sample has position NaN and slot -1).  One launch on the current stream; reads only."""
    if isinstance(seed, (bool, np.bool_)) or not isinstance(seed, (int, np.integer)) or not 0 <= seed < 2 ** 64:
      raise ValueError('seed must be an int in [0, 2^64), got %r' % (seed,))
    n, rec, rec_bytes = _rows(self, states)
    if isinstance(n_samples, (bool, np.bool_)) or not isinstance(n_samples, (int, np.integer)) or not (
        1 <= n_samples < 2 ** 31):
      raise ValueError('n_samples must be an int in [1, 2^31), got %r' % (n_samples,))
    n_samples = int(n_samples)
    position = torch.empty((n, n_samples, 2), dtype=torch.float64, device=self.device)
    slot = torch.empty((n, n_samples), dtype=torch.int8, device=self.device)
    status = torch.empty((n, n_samples), dtype=torch.uint8, device=self.device)
    _native.check(self._lib.swb_sample_contained(
        self._h, rec, n, rec_bytes, n_samples, int(seed), *[_address(t) for t in (position, slot, status)],
        self._stream()))
    return position, slot, status

  # -- env records from factor values ----------------------------------------------------
  def span_class(self):
    """The engine's spans per sprite row, as save_envs reports it: 1 while every uploaded or loaded
    shape is convex, else 4.  Enqueues nothing."""
    span = ctypes.c_int32()
    _native.check(self._lib.swb_save_envs(self._h, None, 0, None, 0, ctypes.byref(span), self._stream()))
    return span.value

  def load_packer(self, program):
    """Gives the engine the packer of make_states (scene_program.compile_packer: task filters, colour
    map and angle table).  Synchronises."""
    from spriteworld_b200 import scene_program
    if self._lib.swb_sampler_sizeof_program() != ctypes.sizeof(scene_program.Program):
      raise _native.NativeError('ABI mismatch: swb_scene_program')
    _native.check(self._lib.swb_packer_load(self._h, ctypes.byref(program.struct)))
    self._packer = program

  def make_states(self, factors, goals=None, step_count=None, span_class=None, out=None):
    """Env records of scenes chosen by the caller (swb_make_states): (EnvStates, status uint8 (n,)).

    `factors`: dict keyed by a subset of sprite.FACTOR_NAMES.  'shape' is required, (n, n_slots),
    ShapeType ids with 0 for an empty slot; every other value broadcasts to (n, n_slots).  All are
    tensors on this device of dtype float32, float64, int8, int16, int32, int64 or uint8; an omitted
    factor is Sprite's default.  Record i is what save_envs would save of an env right after the
    reset step of an episode whose scene is [Sprite(**factors at (i, j)) for its occupied slots j],
    packed with the loaded packer's filters and colour map, with step_count[i] (int32 (n,), default
    zeros) and goals[i] (float64 (n, G, 2), required when G > 0).  status[i] holds the
    scene_program.MAKE_* bits of a refused record, which is written as zeros.

    `span_class`: 1 or 4, the EnvStates' span class.  None reads one device flag back -- the call's
    only host synchronisation -- and gives 4 if an accepted record holds a star or spoke, else
    span_class().  `out`: EnvStates of n records to fill instead of new ones.  One launch on the
    current stream; nothing of the engine changes."""
    from spriteworld_b200 import scene_program, sprite
    packer = getattr(self, '_packer', None)
    if packer is None:
      raise ValueError('make_states: no packer loaded (load_packer)')
    if not isinstance(factors, dict) or 'shape' not in factors:
      raise ValueError("make_states: factors must be a dict with a 'shape' entry")
    unknown = sorted(set(factors) - set(sprite.FACTOR_NAMES))
    if unknown:
      raise ValueError('make_states: unknown factors %s (factors are %s)' % (unknown, ', '.join(sprite.FACTOR_NAMES)))
    shape = factors['shape']
    if not isinstance(shape, torch.Tensor) or shape.dim() != 2 or shape.shape[1] != self.n_slots:
      raise ValueError("make_states: factors['shape'] must be a (n, %d) tensor, got %s"
                       % (self.n_slots, _describe(shape)))
    n = int(shape.shape[0])
    for name, t in factors.items():
      if (not isinstance(t, torch.Tensor) or t.device != self.device or t.dtype not in _MAKE_DTYPES
          or not _broadcasts(t.shape, (n, self.n_slots))):
        raise ValueError('make_states: factors[%r] must be a float32, float64, int8, int16, int32, int64 or '
                         'uint8 tensor on %s that broadcasts to (%d, %d), got %s'
                         % (name, self.device, n, self.n_slots, _describe(t)))
    if packer.struct.color_mode == scene_program.COLOR_HSV:
      kinds = [factors[c].dtype if c in factors else None for c in ('c0', 'c1', 'c2')]
      if len(set(kinds)) != 1 or kinds[0] not in (None, torch.float32, torch.float64):
        raise ValueError('make_states: under hsv_to_rgb the colours c0, c1, c2 must be all float32, all '
                         'float64 or all omitted, got %s' % [str(k).replace('torch.', '') for k in kinds])
    if goals is not None or self.n_goals:
      if goals is None:
        raise ValueError('make_states: the task samples %d goals per scene: goals (n, %d, 2) are required'
                         % (self.n_goals, self.n_goals))
      goals = self._check_goals(goals, n, 'make_states')
    if step_count is not None:
      _check_output(step_count, 'step_count', torch.int32, (n,), self.device, align=4)
    if span_class not in (None, 1, 4):
      raise ValueError('make_states: span_class must be None, 1 or 4, got %r' % (span_class,))
    if out is None:
      out = EnvStates(torch.empty((n, self.record_bytes), dtype=torch.uint8, device=self.device), 1,
                      self.signature, self.n_slots, self.n_goals)
    else:
      self.check_states(out, n)
    status = torch.empty(n, dtype=torch.uint8, device=self.device)
    flag = torch.empty(1, dtype=torch.uint8, device=self.device) if span_class is None else None
    cols, keep = scene_program.FactorColumns(), []
    for f, name in enumerate(sprite.FACTOR_NAMES):
      if name in factors:
        t = factors[name].expand(n, self.n_slots).contiguous()
        keep.append(t)
        cols.col[f], cols.kind[f] = _address(t).value, _MAKE_DTYPES[t.dtype]
    _native.check(self._lib.swb_make_states(
        self._h, ctypes.byref(cols), n, None if goals is None else _address(goals),
        None if step_count is None else _address(step_count), _address(out.data), out.data.numel(),
        _address(status), None if flag is None else _address(flag), self._stream()))
    if span_class is None:
      span_class = 4 if n and int(flag.item()) else self.span_class()
    out.span_class = span_class
    return out, status

  def launch_count(self):
    return int(self._lib.swb_launch_count(self._h))


def make_config(n_envs, n_slots, pool_depth, action, nodes, shapes, keep_in_frame=True,
                max_episode_length=1000, device=0):
  """The swb_config of an engine (see Engine)."""
  cfg = _native.Config()
  cfg.device = device
  cfg.n_envs, cfg.n_slots, cfg.pool_depth = int(n_envs), int(n_slots), int(pool_depth)
  cfg.action_kind = ACTIONS[action['kind']].kind
  cfg.action_scale = float(action['scale'])
  cfg.motion_cost = float(action.get('motion_cost', 0.0))
  cfg.keep_in_frame = int(bool(keep_in_frame))
  cfg.max_episode_length = int(min(max_episode_length, 2 ** 31 - 1))
  fill_task_nodes(cfg, nodes)
  fill_shapes(cfg, shapes)
  return cfg


def config_signature(cfg):
  """The bytes of `cfg` with n_envs, pool_depth and device zeroed: engines with equal signatures
  step and render an env record alike, so records of one load into the other."""
  sig = _native.Config()
  ctypes.memmove(ctypes.byref(sig), ctypes.byref(cfg), ctypes.sizeof(_native.Config))
  sig.n_envs = sig.pool_depth = sig.device = 0
  return bytes(sig)


def record_layout(n_slots, n_goals=0):
  """(fields, record bytes) of an env record of an engine with n_slots slots and n_goals sampled
  goals: fields is a list of (name, byte offset, NumPy dtype, shape within one record).  The table
  of include/spriteworld_b200.h; `factors` is (5, S) there: scale, angle, c0, c1, c2.  With
  n_goals = G > 0 the record ends in `goal` float64 (G, 2)."""
  S, G = int(n_slots), int(n_goals)
  fields, off = [], 0
  for name in ('x0', 'y0', 'm00', 'm01', 'm10', 'm11', 'vx', 'vy', 'pos_x', 'pos_y'):
    fields.append((name, off, np.dtype('<f8'), (S,)))
    off += 8 * S
  for name, dtype, shape in (('member', '<u4', (S,)), ('rgb', '<u4', (S,)), ('factors', '<f4', (5, S)),
                             ('step_count', '<i4', ()), ('reset_next', 'u1', ()),
                             ('shape', 'u1', (S,)), ('pos_f32', 'u1', (S,))):
    dtype = np.dtype(dtype)
    fields.append((name, off, dtype, shape))
    off += dtype.itemsize * int(np.prod(shape, dtype=np.int64))
  if G:
    off = (off + 7) // 8 * 8
    fields.append(('goal', off, np.dtype('<f8'), (G, 2)))
    off += 16 * G
  return fields, (off + 15) // 16 * 16


_ID_DTYPES = {torch.int32: _native.DTYPE_I32, torch.int64: _native.DTYPE_I64}
# the dtypes of make_states' factor columns and their SWB_FT_* kinds
_MAKE_DTYPES = {torch.float32: 1, torch.float64: 2, torch.int8: 3, torch.int16: 4, torch.int32: 5,
                torch.int64: 6, torch.uint8: 7}


def _broadcasts(shape, to):
  """True if a tensor of `shape` broadcasts to `to` (without growing its rank beyond it)."""
  shape = tuple(shape)
  return len(shape) <= len(to) and all(a in (1, b) for a, b in zip(shape[::-1], to[::-1]))
# swb_ids_status
_IDS_STATUS = np.dtype([('ok', '<u4'), ('failed', '<u4'), ('call', '<i4'), ('arg', '<i4'), ('reason', '<i4'),
                        ('position', '<i4'), ('value', '<i8')])
_IDS_CALLS = {_native.IDS_CALL_SAVE: 'save_envs', _native.IDS_CALL_LOAD: 'load_envs',
              _native.IDS_CALL_COPY: 'copy_envs', _native.IDS_CALL_SET_GOALS: 'set_goals'}


def device_checked(check, env_ids):
  """True for a record call that takes device ids checked on the device: check='device' with ids
  given (env_ids=None, all envs, takes the host path).  ValueError for another `check`."""
  if check not in ('host', 'device'):
    raise ValueError("check must be 'host' or 'device', got %r" % (check,))
  return check == 'device' and env_ids is not None


_TORCH_DTYPES = {np.dtype('<f8'): torch.float64, np.dtype('<f4'): torch.float32,
                 np.dtype('<i4'): torch.int32, np.dtype('<u4'): torch.int32, np.dtype('u1'): torch.uint8}


def env_ids_array(ids):
  """Host int32 array of env ids from a list, ndarray or tensor.  A CUDA tensor costs a
  device-to-host copy, which waits for the work enqueued on its stream."""
  if isinstance(ids, torch.Tensor):
    ids = ids.detach().cpu().numpy()
  a = np.asarray(ids)
  if a.ndim != 1:
    raise ValueError('env ids must be one-dimensional, got shape %s' % (a.shape,))
  if a.size and not np.issubdtype(a.dtype, np.integer):
    raise ValueError('env ids must be integers, got %s' % a.dtype)
  if a.size and (a.min() < -2 ** 31 or a.max() >= 2 ** 31):
    raise ValueError('env id out of range')
  return np.ascontiguousarray(a, np.int32)


class EnvStates(object):
  """Env records saved on the device (Engine.save_envs): a (n, record_bytes) uint8 tensor, the
  span class the records need (1: convex shapes only, 4: stars or spokes) and the signature of
  the engine configuration they belong to (config_signature).

  len(), indexing and slicing (a device gather; an int keeps one record), take() (a gather by a
  device index tensor, without host synchronisation), `to(device)`, EnvStates.cat() and
  torch.save / torch.load; to_host() decodes the records into NumPy arrays."""

  def __init__(self, data, span_class, signature, n_slots, n_goals=0):
    self.data, self.span_class = data, int(span_class)
    self.signature, self.n_slots, self.n_goals = bytes(signature), int(n_slots), int(n_goals)

  @property
  def record_bytes(self):
    return int(self.data.shape[1])

  def __len__(self):
    return int(self.data.shape[0])

  def __getitem__(self, idx):
    if isinstance(idx, (int, np.integer)):
      idx = slice(idx, idx + 1 if idx != -1 else None)
    elif not isinstance(idx, slice):
      idx = torch.as_tensor(env_ids_array(idx).astype(np.int64), device=self.data.device)
    return EnvStates(self.data[idx].contiguous(), self.span_class, self.signature, self.n_slots, self.n_goals)

  def take(self, index):
    """EnvStates whose record i is record index[i]: a gather on the device that never waits for
    it, for indices the device computes (a top-k over rollout returns, say).  `index`: a
    one-dimensional int32 or int64 tensor on the records' device.  An entry outside [0, len(self))
    gives a zero record, which loads as an env with only empty slots."""
    if (not isinstance(index, torch.Tensor) or index.dim() != 1 or
        index.dtype not in (torch.int32, torch.int64) or index.device != self.data.device):
      raise ValueError('take needs a one-dimensional int32 or int64 tensor on %s, got %s'
                       % (self.data.device, _describe(index)))
    n = len(self)
    if n == 0:
      data = self.data.new_zeros((index.numel(), self.record_bytes))
    else:
      index = index.long()
      inside = (index >= 0) & (index < n)
      # clamped, so that no index outside the records reaches the gather
      data = self.data.index_select(0, index.clamp(0, n - 1)).masked_fill_(~inside[:, None], 0)
    return EnvStates(data, self.span_class, self.signature, self.n_slots, self.n_goals)

  def to(self, device):
    return EnvStates(self.data.to(device), self.span_class, self.signature, self.n_slots, self.n_goals)

  @staticmethod
  def cat(states):
    """One EnvStates of the records of `states` (a sequence of EnvStates of one configuration)."""
    states = list(states)
    if not states or any(s.signature != states[0].signature for s in states):
      raise ValueError('EnvStates.cat needs at least one EnvStates, all of one engine configuration')
    return EnvStates(torch.cat([s.data for s in states]), max(s.span_class for s in states),
                     states[0].signature, states[0].n_slots, states[0].n_goals)

  def fields(self):
    """dict name -> device tensor view (n,) + shape of every field (uint32 fields as int32)."""
    layout, _ = record_layout(self.n_slots, self.n_goals)
    n, out = len(self), {}
    for name, off, dtype, shape in layout:
      nbytes = dtype.itemsize * int(np.prod(shape, dtype=np.int64))
      out[name] = self.data[:, off:off + nbytes].view(_TORCH_DTYPES[dtype]).reshape((n,) + shape)
    return out

  def to_host(self):
    """dict of NumPy arrays, one per field: x0 .. vy, pos_x, pos_y (n, S) float64, member (n, S)
    uint32, rgb (n, S, 3) uint8, factors (n, S, 5) float32, shape and pos_f32 (n, S) uint8,
    step_count (n,) int32, reset_next (n,) uint8, and goal (n, G, 2) float64 with sampled goals."""
    out = {name: t.cpu().numpy().copy() for name, t in self.fields().items()}
    out['member'] = out['member'].view(np.uint32)
    out['rgb'] = out['rgb'].view(np.uint32)[..., None].view(np.uint8)[..., :3].copy()
    out['factors'] = np.ascontiguousarray(out['factors'].transpose(0, 2, 1))
    return out


torch.serialization.add_safe_globals([EnvStates])   # torch.load(..., weights_only=True)


def _describe(t):
  if not isinstance(t, torch.Tensor):
    return type(t).__name__
  return '%s %s on %s%s' % (t.dtype, tuple(t.shape), t.device,
                            '' if t.is_contiguous() else ' (not contiguous)')


def fill_task_nodes(cfg, nodes):
  if not 1 <= len(nodes) <= _native.MAX_NODES:
    raise ValueError('task tree has %d nodes (max %d)' % (len(nodes), _native.MAX_NODES))
  cfg.n_nodes = len(nodes)
  for i, nd in enumerate(nodes):
    n = cfg.nodes[i]
    kind = nd['kind']
    if kind == 'find_goal':
      n.kind = _native.TASK_FIND_GOAL
      n.filter_slot = int(nd['filter_slot'])
      n.goal[0], n.goal[1] = [float(v) for v in nd['goal']]
      n.weights[0], n.weights[1] = [float(v) for v in nd['weights']]
      n.terminate_distance = float(nd['terminate_distance'])
      n.terminate_bonus = float(nd['terminate_bonus'])
      n.raw_reward_multiplier = float(nd['raw_reward_multiplier'])
      n.sparse_reward = int(bool(nd['sparse_reward']))
      n.goal_slot = int(nd.get('goal_slot', -1))
    elif kind == 'clustering':
      n.kind = _native.TASK_CLUSTERING
      slots = nd['cluster_slots']
      if len(slots) > _native.MAX_CHILDREN:
        raise ValueError('at most %d clusters' % _native.MAX_CHILDREN)
      n.n_clusters = len(slots)
      for j, s in enumerate(slots):
        n.cluster_slots[j] = int(s)
      n.termination_threshold = float(nd['termination_threshold'])
      n.terminate_bonus = float(nd['terminate_bonus'])
      n.sparse_reward = int(bool(nd['sparse_reward']))
      n.reward_range = float(nd['reward_range'])
    elif kind == 'meta':
      n.kind = _native.TASK_META
      kids = nd['children']
      if len(kids) > _native.MAX_CHILDREN:
        raise ValueError('at most %d subtasks' % _native.MAX_CHILDREN)
      n.n_children = len(kids)
      for j, c in enumerate(kids):
        n.children[j] = int(c)
      n.aggregator = _native.AGG[nd['aggregator']]
      n.criterion = _native.CRIT[nd['criterion']]
      n.terminate_bonus = float(nd['terminate_bonus'])
    elif kind == 'no_reward':
      n.kind = _native.TASK_NO_REWARD
    else:
      raise ValueError('unknown task node kind %r' % (kind,))


SHAPE_IDS = {
    'triangle': 1, 'square': 2, 'pentagon': 3, 'hexagon': 4, 'octagon': 5, 'circle': 6,
    'star_4': 7, 'star_5': 8, 'star_6': 9, 'spoke_4': 10, 'spoke_5': 11, 'spoke_6': 12,
}


def shape_id_table(shapes):
  """uint8 (256,) NumPy array: id -> the id an env record's shape id `id` loads as (swb_load_envs),
  i.e. itself for a shape with a vertex table of at least 3 vertices in `shapes`, else 0 (an
  empty slot)."""
  table = np.zeros(256, np.uint8)
  for name, sid in SHAPE_IDS.items():
    if len(shapes[name]) >= 3:
      table[sid] = sid
  return table


def fill_shapes(cfg, shapes):
  for name, sid in SHAPE_IDS.items():
    v = np.asarray(shapes[name], dtype=np.float64)
    if v.ndim != 2 or v.shape[1] != 2 or len(v) > _native.MAX_VERTS:
      raise ValueError('bad vertex table for %s' % name)
    cfg.shape_n_verts[sid] = len(v)
    for i in range(len(v)):
      cfg.shape_verts[sid][i][0] = float(v[i, 0])
      cfg.shape_verts[sid][i][1] = float(v[i, 1])
