"""Thin Python owner of one swb_engine (one per GPU).

PyTorch is used only for device memory and streams: action, reward, flag and frame
buffers are torch tensors whose `data_ptr()` is handed to the C-ABI
(include/spriteworld_b200.h).  All compute happens in the CUDA library.
"""
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
  n_envs * OUT_BYTES_PER_ENV bytes (layout: all rewards, then all step types, ...)."""
  E = int(n_envs)
  reward = buf[:8 * E].view(torch.float64)
  step_type = buf[8 * E:9 * E].view(torch.int8)
  success = buf[9 * E:10 * E]
  status = buf[10 * E:11 * E]
  return reward, step_type, success, status


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
    self.action_kind = {'select_move': _native.ACT_SELECT_MOVE,
                        'drag_and_drop': _native.ACT_DRAG_AND_DROP,
                        'embodied': _native.ACT_EMBODIED}[action['kind']]
    cfg = _native.Config()
    cfg.device = device
    cfg.n_envs, cfg.n_slots, cfg.pool_depth = self.n_envs, self.n_slots, self.pool_depth
    cfg.action_kind = self.action_kind
    cfg.action_scale = float(action['scale'])
    cfg.motion_cost = float(action.get('motion_cost', 0.0))
    cfg.keep_in_frame = int(bool(keep_in_frame))
    cfg.max_episode_length = int(min(max_episode_length, 2 ** 31 - 1))
    fill_task_nodes(cfg, nodes)
    fill_shapes(cfg, shapes)
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
  def _action_dtype(self, actions):
    if self.action_kind == _native.ACT_EMBODIED:
      if actions.dtype != torch.int32 or tuple(actions.shape) != (self.n_envs, 2):
        raise ValueError('Embodied actions must be an int32 tensor of shape (E, 2)')
      return _native.DTYPE_I32
    if tuple(actions.shape) != (self.n_envs, 4):
      raise ValueError('actions must have shape (E, 4)')
    if actions.dtype == torch.float32:
      return _native.DTYPE_F32
    if actions.dtype == torch.float64:
      return _native.DTYPE_F64
    raise ValueError('actions must be float32 or float64')

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
    if actions.device != self.device or not actions.is_contiguous():
      raise ValueError('actions must be a contiguous tensor on %s' % self.device)
    dt = self._action_dtype(actions)
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
    if actions.device != self.device or not actions.is_contiguous():
      raise ValueError('actions must be a contiguous tensor on %s' % self.device)
    dt = self._action_dtype(actions)
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
    a = np.ascontiguousarray(actions)
    if self.action_kind == _native.ACT_EMBODIED:
      a = np.ascontiguousarray(a, dtype=np.int32)
      dt = _native.DTYPE_I32
    elif a.dtype == np.float32:
      dt = _native.DTYPE_F32
    else:
      a = np.ascontiguousarray(a, dtype=np.float64)
      dt = _native.DTYPE_F64
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

  def launch_count(self):
    return int(self._lib.swb_launch_count(self._h))


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
