"""ctypes binding of include/spriteworld_b200.h.

There is no CPU fallback: if the CUDA library is missing or does not load, importing the
engine fails loudly (build it with `python -m spriteworld_b200.build`).
"""
import ctypes
import os

MAX_VERTS = 32
NUM_SHAPES = 13
MAX_CHILDREN = 16
MAX_NODES = 32
MAX_SLOTS = 32
MAX_FILTERS = 32

ACT_SELECT_MOVE, ACT_DRAG_AND_DROP, ACT_EMBODIED = 0, 1, 2
DTYPE_F32, DTYPE_F64, DTYPE_I32, DTYPE_I64 = 0, 1, 2, 3
TASK_NO_REWARD, TASK_FIND_GOAL, TASK_CLUSTERING, TASK_META = 0, 1, 2, 3
AGG = {'sum': 0, 'max': 1, 'min': 2, 'mean': 3}
CRIT = {'all': 0, 'any': 1}
STEP_FIRST, STEP_MID, STEP_LAST = 0, 1, 2
ENV_OK, ENV_CLUSTER_LABELS, ENV_CLUSTER_ZERODIV, ENV_BAD_ACTION, ENV_SPAN_OVERFLOW = 0, 1, 2, 4, 8
IDS_CALL_SAVE, IDS_CALL_LOAD, IDS_CALL_COPY = 0, 1, 2
IDS_OUT_OF_RANGE, IDS_REPEATED = 1, 2

_c32, _f64, _u8p = ctypes.c_int32, ctypes.c_double, ctypes.POINTER(ctypes.c_uint8)


class TaskNode(ctypes.Structure):
  _fields_ = [
      ('kind', _c32), ('filter_slot', _c32),
      ('goal', _f64 * 2), ('weights', _f64 * 2),
      ('terminate_distance', _f64), ('terminate_bonus', _f64),
      ('raw_reward_multiplier', _f64), ('sparse_reward', _c32),
      ('n_clusters', _c32), ('cluster_slots', _c32 * MAX_CHILDREN),
      ('termination_threshold', _f64), ('reward_range', _f64),
      ('n_children', _c32), ('children', _c32 * MAX_CHILDREN),
      ('aggregator', _c32), ('criterion', _c32),
  ]


class Config(ctypes.Structure):
  _fields_ = [
      ('device', _c32), ('n_envs', _c32), ('n_slots', _c32), ('pool_depth', _c32),
      ('action_kind', _c32), ('action_scale', _f64), ('motion_cost', _f64),
      ('keep_in_frame', _c32), ('max_episode_length', _c32),
      ('n_nodes', _c32), ('nodes', TaskNode * MAX_NODES),
      ('shape_n_verts', _c32 * NUM_SHAPES),
      ('shape_verts', _f64 * 2 * MAX_VERTS * NUM_SHAPES),
  ]


class SceneSoA(ctypes.Structure):
  _fields_ = [(n, ctypes.c_void_p) for n in
              ('x', 'y', 'm00', 'm01', 'm10', 'm11', 'vx', 'vy', 'member', 'shape', 'pos_f32',
               'rgb', 'factors')]


class StepOut(ctypes.Structure):
  _fields_ = [('reward', ctypes.c_void_p), ('step_type', ctypes.c_void_p),
              ('success', ctypes.c_void_p), ('status', ctypes.c_void_p)]


# SPRITEWORLD_B200_LIB points at another build of the same library (debug / experiment builds)
_LIB_PATH = os.environ.get('SPRITEWORLD_B200_LIB') or os.path.join(
    os.path.dirname(os.path.abspath(__file__)), 'csrc', 'libspriteworld_b200.so')
_lib = None


MAX_PEERS = 8            # SWB_MAX_PEERS
IPC_HANDLE_BYTES = 64    # SWB_IPC_HANDLE_BYTES


class NativeError(RuntimeError):
  pass


def lib_path():
  return _LIB_PATH


def load():
  """Loads the CUDA library (once).  Raises if it has not been built."""
  global _lib
  if _lib is not None:
    return _lib
  if not os.path.exists(_LIB_PATH):
    raise NativeError(
        'spriteworld_b200: %s is missing. Build it with `python -m spriteworld_b200.build` '
        '(nvcc, sm_90a). There is no CPU fallback.' % _LIB_PATH)
  L = ctypes.CDLL(_LIB_PATH)
  vp, ci = ctypes.c_void_p, ctypes.c_int32
  L.swb_last_error.restype = ctypes.c_char_p
  L.swb_engine_create.argtypes = [ctypes.POINTER(Config), ctypes.POINTER(vp)]
  L.swb_engine_destroy.argtypes = [vp]
  L.swb_engine_destroy.restype = None
  L.swb_upload_scenes.argtypes = [vp, ctypes.POINTER(SceneSoA), vp, vp, ci, vp]
  L.swb_request_reset.argtypes = [vp, vp, vp]
  L.swb_step.argtypes = [vp, vp, ci, ctypes.POINTER(StepOut), vp]
  L.swb_eval_task.argtypes = [vp, ctypes.POINTER(StepOut), vp]
  L.swb_apply_action.argtypes = [vp, vp, ci, ctypes.POINTER(StepOut), vp]
  L.swb_raster_create.argtypes = [vp, ci, ci, ci, vp, ctypes.POINTER(vp)]
  L.swb_raster_destroy.argtypes = [vp]
  L.swb_raster_destroy.restype = None
  L.swb_render.argtypes = [vp, vp, vp, vp]
  L.swb_step_render.argtypes = [vp, vp, vp, ci, ctypes.POINTER(StepOut), vp, vp]
  L.swb_step_host.argtypes = [vp, vp, vp, ci, vp, vp, vp, vp, vp, vp]
  L.swb_step_render_gather.argtypes = [vp, vp, vp, ci, ctypes.POINTER(StepOut), ctypes.POINTER(vp), ci,
                                       ctypes.c_int64, vp]
  L.swb_ipc_alloc.argtypes = [ci, ctypes.c_uint64, ctypes.POINTER(vp), vp]
  L.swb_ipc_free.argtypes = [vp]
  L.swb_ipc_open.argtypes = [ci, vp, ctypes.POINTER(vp)]
  L.swb_ipc_close.argtypes = [vp]
  L.swb_peer_copy.argtypes = [vp, vp, ctypes.c_uint64, vp]
  L.swb_state_pointers.argtypes = [vp] + [ctypes.POINTER(vp)] * 5
  L.swb_scene_serial_pointer.argtypes = [vp, ctypes.POINTER(vp)]
  L.swb_render_status_pointer.argtypes = [vp, ctypes.POINTER(vp)]
  L.swb_download_state.argtypes = [vp, vp, vp, vp, vp, vp, vp]
  L.swb_upload_state.argtypes = [vp, vp, vp, vp, vp, vp, vp]
  L.swb_env_record_bytes.argtypes = [vp]
  L.swb_env_record_bytes.restype = ctypes.c_int64
  L.swb_save_envs.argtypes = [vp, vp, ci, vp, ctypes.c_uint64, ctypes.POINTER(ci), vp]
  L.swb_load_envs.argtypes = [vp, vp, ci, vp, ctypes.c_uint64, ci, vp]
  L.swb_copy_envs.argtypes = [vp, vp, vp, ci, vp]
  L.swb_save_envs_dev.argtypes = [vp, vp, ci, ci, vp, ctypes.c_uint64, ctypes.POINTER(ci), vp]
  L.swb_load_envs_dev.argtypes = [vp, vp, ci, ci, vp, ctypes.c_uint64, ci, vp]
  L.swb_copy_envs_dev.argtypes = [vp, vp, vp, ci, ci, vp]
  L.swb_env_ids_status_pointer.argtypes = [vp, ctypes.POINTER(vp)]
  L.swb_launch_count.argtypes = [vp]
  L.swb_launch_count.restype = ctypes.c_int64
  L.swb_sampler_load.argtypes = [vp, vp, ctypes.c_uint64, ctypes.c_int64]
  L.swb_sample_scenes.argtypes = [vp, vp, vp, ci, vp, vp]
  L.swb_refill_device.argtypes = [vp, vp, vp]
  L.swb_pool_pointers.argtypes = [vp, vp] + [ctypes.POINTER(vp)] * 5
  L.swb_sampler_pointers.argtypes = [vp, ctypes.POINTER(vp), ctypes.POINTER(vp)]
  if L.swb_sizeof_config() != ctypes.sizeof(Config):
    raise NativeError('ABI mismatch: swb_config is %d bytes in the library, %d in the binding'
                      % (L.swb_sizeof_config(), ctypes.sizeof(Config)))
  if L.swb_sizeof_task_node() != ctypes.sizeof(TaskNode):
    raise NativeError('ABI mismatch: swb_task_node')
  _lib = L
  return L


EXPORTS = (
    'swb_last_error', 'swb_version', 'swb_sizeof_config', 'swb_sizeof_task_node',
    'swb_engine_create', 'swb_engine_destroy', 'swb_upload_scenes', 'swb_request_reset',
    'swb_step', 'swb_eval_task', 'swb_apply_action', 'swb_raster_create', 'swb_raster_destroy', 'swb_render', 'swb_step_render',
    'swb_step_render_gather', 'swb_ipc_alloc', 'swb_ipc_free', 'swb_ipc_open', 'swb_ipc_close', 'swb_peer_copy',
    'swb_step_host', 'swb_state_pointers', 'swb_scene_serial_pointer', 'swb_render_status_pointer', 'swb_download_state', 'swb_upload_state',
    'swb_env_record_bytes', 'swb_save_envs', 'swb_load_envs', 'swb_copy_envs', 'swb_save_envs_dev',
    'swb_load_envs_dev', 'swb_copy_envs_dev', 'swb_env_ids_status_pointer', 'swb_launch_count',
    'swb_sampler_sizeof_program', 'swb_sampler_load', 'swb_sample_scenes', 'swb_refill_device',
    'swb_sampler_pointers', 'swb_pool_pointers')


def check(rc):
  if rc != 0:
    raise NativeError(load().swb_last_error().decode('utf-8', 'replace'))
