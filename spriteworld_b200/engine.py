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


def action_dtype(action_kind, n_envs, actions, device=None):
  """The swb action dtype of `actions` (tensor or array) for `n_envs` envs of swb `action_kind`;
  with `device`, a contiguous tensor on it.  ValueError otherwise: nothing is converted."""
  if device is not None and not (isinstance(actions, torch.Tensor) and actions.device == device
                                 and actions.is_contiguous()):
    raise ValueError('actions must be a contiguous tensor on %s, got %s'
                     % (device, _describe(actions)))
  spec = _SPECS[action_kind]
  name = str(actions.dtype).replace('torch.', '')
  shape = (int(n_envs), spec.columns)
  if tuple(actions.shape) != shape or name not in spec.dtypes:
    raise ValueError('actions must have shape %s and dtype %s, got %s %s' % (
        shape, ' or '.join(spec.dtypes), name, tuple(actions.shape)))
  return spec.dtypes[name]


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
    """The render kernel writes n_frames * H * W * 3 bytes from frames.data_ptr(): anything but
    a contiguous uint8 tensor of exactly that shape on this device would be written out of
    bounds or scrambled."""
    shape = (n_frames, raster.height, raster.width, 3)
    if (not isinstance(frames, torch.Tensor) or frames.dtype != torch.uint8 or
        frames.device != self.device or tuple(frames.shape) != shape or
        not frames.is_contiguous()):
      raise ValueError('frames must be a contiguous uint8 tensor of shape %s on %s, got %s' % (
          shape, self.device, _describe(frames)))

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
      return EnvStates(data, span.value, self.signature, self.n_slots)
    ids = self._all_or(env_ids)
    data = torch.empty((len(ids), rb), dtype=torch.uint8, device=self.device)
    _native.check(self._lib.swb_save_envs(self._h, _as_ptr(ids), len(ids), ctypes.c_void_p(data.data_ptr()),
                                          data.numel(), ctypes.byref(span), self._stream()))
    return EnvStates(data, span.value, self.signature, self.n_slots)

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
    'factor_kind' uint8 (n, S, 10).  The pool is not touched."""
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
    st = scene_program.sample_out_struct(out, lambda t: t.data_ptr())
    _native.check(self._lib.swb_sample_scenes(self._h, ctypes.c_void_p(ids.data_ptr()),
                                              ctypes.c_void_p(idx.data_ptr()), n, ctypes.byref(st),
                                              self._stream()))
    return out

  def refill_device(self, static_rows=None):
    """Enqueues the device refill: every env's ring up to scene_serial + K - 1.  static_rows: an
    optional float32 (E, K, S, 8) device tensor that gets the static factors of every slot written
    (shape, scale, angle, c0, c1, c2, vx, vy)."""
    ptr = None
    if static_rows is not None:
      E, K, S = self.n_envs, self.pool_depth, self.n_slots
      if not (static_rows.dtype == torch.float32 and tuple(static_rows.shape) == (E, K, S, 8)
              and static_rows.device == self.device and static_rows.is_contiguous()):
        raise ValueError('static_rows must be a contiguous float32 (%d, %d, %d, 8) tensor on %s'
                         % (E, K, S, self.device))
      ptr = ctypes.c_void_p(static_rows.data_ptr())
    _native.check(self._lib.swb_refill_device(self._h, ptr, self._stream()))

  def pool_tensors(self):
    """Zero-copy views of the scene pool, shaped (E, K, S[, ...]): x .. vy float64, member int32,
    shape and pos_f32 uint8, rgb uint8 (E, K, S, 4) (r, g, b, 0), factors float32 (E, K, S, 5)."""
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
    return out

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


def record_layout(n_slots):
  """(fields, record bytes) of an env record of an engine with n_slots slots: fields is a list of
  (name, byte offset, NumPy dtype, shape within one record).  The table of
  include/spriteworld_b200.h; `factors` is (5, S) there: scale, angle, c0, c1, c2."""
  S = int(n_slots)
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
  return fields, (off + 15) // 16 * 16


_ID_DTYPES = {torch.int32: _native.DTYPE_I32, torch.int64: _native.DTYPE_I64}
# swb_ids_status
_IDS_STATUS = np.dtype([('ok', '<u4'), ('failed', '<u4'), ('call', '<i4'), ('arg', '<i4'), ('reason', '<i4'),
                        ('position', '<i4'), ('value', '<i8')])
_IDS_CALLS = {_native.IDS_CALL_SAVE: 'save_envs', _native.IDS_CALL_LOAD: 'load_envs',
              _native.IDS_CALL_COPY: 'copy_envs'}


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

  len(), indexing and slicing (a device gather; an int keeps one record), `to(device)`,
  EnvStates.cat() and torch.save / torch.load; to_host() decodes the records into NumPy arrays."""

  def __init__(self, data, span_class, signature, n_slots):
    self.data, self.span_class = data, int(span_class)
    self.signature, self.n_slots = bytes(signature), int(n_slots)

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
    return EnvStates(self.data[idx].contiguous(), self.span_class, self.signature, self.n_slots)

  def to(self, device):
    return EnvStates(self.data.to(device), self.span_class, self.signature, self.n_slots)

  @staticmethod
  def cat(states):
    """One EnvStates of the records of `states` (a sequence of EnvStates of one configuration)."""
    states = list(states)
    if not states or any(s.signature != states[0].signature for s in states):
      raise ValueError('EnvStates.cat needs at least one EnvStates, all of one engine configuration')
    return EnvStates(torch.cat([s.data for s in states]), max(s.span_class for s in states),
                     states[0].signature, states[0].n_slots)

  def fields(self):
    """dict name -> device tensor view (n,) + shape of every field (uint32 fields as int32)."""
    layout, _ = record_layout(self.n_slots)
    n, out = len(self), {}
    for name, off, dtype, shape in layout:
      nbytes = dtype.itemsize * int(np.prod(shape, dtype=np.int64))
      out[name] = self.data[:, off:off + nbytes].view(_TORCH_DTYPES[dtype]).reshape((n,) + shape)
    return out

  def to_host(self):
    """dict of NumPy arrays, one per field: x0 .. vy, pos_x, pos_y (n, S) float64, member (n, S)
    uint32, rgb (n, S, 3) uint8, factors (n, S, 5) float32, shape and pos_f32 (n, S) uint8,
    step_count (n,) int32, reset_next (n,) uint8."""
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


def fill_shapes(cfg, shapes):
  for name, sid in SHAPE_IDS.items():
    v = np.asarray(shapes[name], dtype=np.float64)
    if v.ndim != 2 or v.shape[1] != 2 or len(v) > _native.MAX_VERTS:
      raise ValueError('bad vertex table for %s' % name)
    cfg.shape_n_verts[sid] = len(v)
    for i in range(len(v)):
      cfg.shape_verts[sid][i][0] = float(v[i, 0])
      cfg.shape_verts[sid][i][1] = float(v[i, 1])
