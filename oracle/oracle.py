"""ctypes front-end of the CPU oracle (test infrastructure, NOT product code).

Importers allowed: tests/, __graft_entry__.smoke(), bench.py's CPU-baseline /
`--impl reference` arm.  The product package `spriteworld_b200` never imports this.

The C sources restate the reference's Environment.step() hot path
(oracle/sw_env_oracle.c) and the two Pillow stages under it
(oracle/sw_raster_oracle.c); this module only marshals data.
"""
import ctypes
import math
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, '_build', 'libsw_oracle.so')

MAX_VERTS = 32
NUM_SHAPES = 13
MAX_CHILDREN = 16
MAX_NODES = 32

ACT_SELECT_MOVE, ACT_DRAG_AND_DROP, ACT_EMBODIED = 0, 1, 2
TASK_NO_REWARD, TASK_FIND_GOAL, TASK_CLUSTERING, TASK_META = 0, 1, 2, 3
AGG = {'sum': 0, 'max': 1, 'min': 2, 'mean': 3}
CRIT = {'all': 0, 'any': 1}
STEP_FIRST, STEP_MID, STEP_LAST = 0, 1, 2

SHAPE_IDS = {  # constants.py:43-56
    'triangle': 1, 'square': 2, 'pentagon': 3, 'hexagon': 4, 'octagon': 5,
    'circle': 6, 'star_4': 7, 'star_5': 8, 'star_6': 9, 'spoke_4': 10,
    'spoke_5': 11, 'spoke_6': 12,
}

SPRITE_DTYPE = np.dtype([
    ('x', '<f8'), ('y', '<f8'),
    ('m00', '<f8'), ('m01', '<f8'), ('m10', '<f8'), ('m11', '<f8'),
    ('vx', '<f8'), ('vy', '<f8'),
    ('member', '<u4'), ('shape', 'u1'), ('pos_f32', 'u1'),
    ('rgb', 'u1', (3,)), ('pad', 'u1', (3,)),
], align=True)


class ShapeTable(ctypes.Structure):
  _fields_ = [('n_verts', ctypes.c_int32 * NUM_SHAPES),
              ('verts', ctypes.c_double * 2 * MAX_VERTS * NUM_SHAPES)]


class TaskNode(ctypes.Structure):
  _fields_ = [
      ('kind', ctypes.c_int32), ('filter_slot', ctypes.c_int32),
      ('goal', ctypes.c_double * 2), ('weights', ctypes.c_double * 2),
      ('terminate_distance', ctypes.c_double), ('terminate_bonus', ctypes.c_double),
      ('raw_reward_multiplier', ctypes.c_double), ('sparse_reward', ctypes.c_int32),
      ('n_clusters', ctypes.c_int32), ('cluster_slots', ctypes.c_int32 * MAX_CHILDREN),
      ('termination_threshold', ctypes.c_double), ('reward_range', ctypes.c_double),
      ('n_children', ctypes.c_int32), ('children', ctypes.c_int32 * MAX_CHILDREN),
      ('aggregator', ctypes.c_int32), ('criterion', ctypes.c_int32),
  ]


class EnvCfg(ctypes.Structure):
  _fields_ = [
      ('action_kind', ctypes.c_int32), ('action_scale', ctypes.c_double),
      ('motion_cost', ctypes.c_double), ('keep_in_frame', ctypes.c_int32),
      ('max_episode_length', ctypes.c_int32), ('n_nodes', ctypes.c_int32),
      ('nodes', TaskNode * MAX_NODES),
  ]


class RasterCfg(ctypes.Structure):
  _fields_ = [('width', ctypes.c_int32), ('height', ctypes.c_int32),
              ('anti_aliasing', ctypes.c_int32), ('bg', ctypes.c_uint8 * 3),
              ('pad', ctypes.c_uint8)]


def build(force=False):
  """Compiles oracle/_build/libsw_oracle.so with gcc (make)."""
  srcs = [os.path.join(_HERE, f) for f in
          ('sw_raster_oracle.c', 'sw_env_oracle.c', 'sw_oracle.h', 'Makefile')]
  stale = (not os.path.exists(_LIB_PATH) or
           any(os.path.getmtime(s) > os.path.getmtime(_LIB_PATH) for s in srcs))
  if force or stale:
    subprocess.check_call(['make', '-s', '-C', _HERE] + (['-B'] if force else []))
  return _LIB_PATH


_lib = None


def lib():
  global _lib
  if _lib is None:
    build()
    L = ctypes.CDLL(_LIB_PATH)
    vp, ci = ctypes.c_void_p, ctypes.c_int
    L.swo_polygon_fill.argtypes = [vp, ci, ci, vp, ci, vp, ci]
    L.swo_polygon_fill.restype = None
    L.swo_lanczos_resize.argtypes = [vp, ci, ci, vp, ci, ci, vp]
    L.swo_lanczos_resize.restype = None
    L.swo_lanczos_ksize.argtypes = [ci, ci]
    L.swo_lanczos_coeffs.argtypes = [ci, ci, vp, vp]
    L.swo_lanczos_coeffs.restype = None
    L.swo_hsv_to_rgb_f32.argtypes = [ctypes.c_float] * 3 + [vp]
    L.swo_hsv_to_rgb_f64.argtypes = [ctypes.c_double] * 3 + [vp]
    L.swo_contains_offset.argtypes = [vp, vp, ctypes.c_double, ctypes.c_double]
    L.swo_action_step.argtypes = [vp, vp, vp, ci, vp, ci, vp, vp]
    L.swo_task_eval.argtypes = [vp, vp, ci, vp, vp, vp]
    L.swo_task_eval.restype = None
    L.swo_render.argtypes = [vp, vp, vp, ci, vp, vp]
    L.swo_render.restype = None
    L.swo_env_step.argtypes = [vp, vp, vp, ci, vp, vp, ci, vp, vp, vp, vp]
    L.swo_batch_step.argtypes = [vp, vp, vp, ci, ci, vp, vp, vp, vp, vp, vp, ci,
                                 vp, vp, vp, vp, vp, ci, ci]
    assert L.swo_sizeof_sprite() == SPRITE_DTYPE.itemsize, (
        L.swo_sizeof_sprite(), SPRITE_DTYPE.itemsize)
    assert L.swo_sizeof_env_cfg() == ctypes.sizeof(EnvCfg)
    assert L.swo_sizeof_task_node() == ctypes.sizeof(TaskNode)
    assert L.swo_sizeof_shape_table() == ctypes.sizeof(ShapeTable)
    _lib = L
  return _lib


def _p(a):
  return a.ctypes.data_as(ctypes.c_void_p)


# ---------------------------------------------------------------------------
# Raster stages
# ---------------------------------------------------------------------------

def polygon_fill(canvas, xy, rgb, corner_join=1):
  """In-place ImageDraw.polygon restatement on an (H, W, 3) uint8 canvas."""
  assert canvas.dtype == np.uint8 and canvas.flags.c_contiguous
  xy = np.ascontiguousarray(xy, dtype=np.float64)
  col = np.ascontiguousarray(rgb, dtype=np.uint8)
  h, w = canvas.shape[:2]
  lib().swo_polygon_fill(_p(canvas), w, h, _p(xy), len(xy), _p(col), corner_join)
  return canvas


def lanczos_resize(img, out_w, out_h, return_hpass=False):
  """Image.resize(..., LANCZOS).  return_hpass: also the first pass's image when both sizes
  change: (h, out_w) for the horizontal pass, or (out_h, w) for an image more than 100 times
  taller than wide, which Pillow shrinks vertically first."""
  img = np.ascontiguousarray(img, dtype=np.uint8)
  h, w = img.shape[:2]
  out = np.empty((out_h, out_w, 3), np.uint8)
  mid = (out_h, w) if h > 100 * w and out_h < h else (h, out_w)
  tmp = np.empty(mid + (3,), np.uint8) if return_hpass else None
  lib().swo_lanczos_resize(_p(img), w, h, _p(out), out_w, out_h,
                           _p(tmp) if tmp is not None else None)
  return (out, tmp) if return_hpass else out


def lanczos_coeffs(in_size, out_size):
  ks = lib().swo_lanczos_ksize(in_size, out_size)
  bounds = np.zeros((out_size, 2), np.int32)
  kk = np.zeros((out_size, ks), np.int32)
  lib().swo_lanczos_coeffs(in_size, out_size, _p(bounds), _p(kk))
  return bounds, kk


def hsv_to_rgb(c0, c1, c2, f32):
  out = np.zeros(3, np.uint8)
  if f32:
    lib().swo_hsv_to_rgb_f32(float(np.float32(c0)), float(np.float32(c1)),
                             float(np.float32(c2)), _p(out))
  else:
    lib().swo_hsv_to_rgb_f64(float(c0), float(c1), float(c2), _p(out))
  return out


# ---------------------------------------------------------------------------
# Marshalling helpers
# ---------------------------------------------------------------------------

def shape_table(shapes_dict):
  """shapes_dict: name -> (V, 2) float64 (constants.SHAPES, generated by numpy)."""
  tab = ShapeTable()
  for name, sid in SHAPE_IDS.items():
    v = np.asarray(shapes_dict[name], np.float64)
    assert len(v) <= MAX_VERTS
    tab.n_verts[sid] = len(v)
    for i in range(len(v)):
      tab.verts[sid][i][0] = float(v[i, 0])
      tab.verts[sid][i][1] = float(v[i, 1])
  return tab


def centred_matrix(scale, angle):
  """(Affine2D().scale(s) + Affine2D().rotate_deg(a)).get_matrix() (sprite.py:96-101)."""
  s = float(scale)
  th = math.radians(angle)
  a, b = math.cos(th), math.sin(th)
  return a * s, (-b) * s, b * s, a * s


def sprite_record(x, y, shape, angle, scale, rgb, vx=0.0, vy=0.0, member=0, pos_f32=None):
  rec = np.zeros((), SPRITE_DTYPE)
  if pos_f32 is None:
    pos_f32 = isinstance(x, np.float32) and isinstance(y, np.float32)
  rec['x'], rec['y'] = float(x), float(y)
  rec['m00'], rec['m01'], rec['m10'], rec['m11'] = centred_matrix(scale, angle)
  rec['vx'], rec['vy'] = float(vx), float(vy)
  rec['member'] = member
  rec['shape'] = SHAPE_IDS[shape] if isinstance(shape, str) else int(shape)
  rec['pos_f32'] = 1 if pos_f32 else 0
  rec['rgb'] = np.asarray(rgb, np.uint8)
  return rec


def render(raster_cfg, tab, sprites):
  """sprites: 1-D SPRITE_DTYPE array (back to front).  Returns (H, W, 3) uint8 frame."""
  sprites = np.ascontiguousarray(sprites, dtype=SPRITE_DTYPE)
  frame = np.empty((raster_cfg.height, raster_cfg.width, 3), np.uint8)
  lib().swo_render(ctypes.byref(raster_cfg), ctypes.byref(tab), _p(sprites), len(sprites),
                   _p(frame), None)
  return frame


def raster_cfg(width, height, anti_aliasing=1, bg=(0, 0, 0)):
  rc = RasterCfg()
  rc.width, rc.height, rc.anti_aliasing = width, height, anti_aliasing
  rc.bg[0], rc.bg[1], rc.bg[2] = [int(c) for c in bg]
  return rc


def contains_offset(tab, sprite, tx, ty):
  s = np.ascontiguousarray(sprite, dtype=SPRITE_DTYPE).reshape(1)
  return bool(lib().swo_contains_offset(ctypes.byref(tab), _p(s), float(tx), float(ty)))


def action_step(cfg, tab, sprites, action, action_is_f32):
  """In-place action on a 1-D SPRITE_DTYPE array.  Returns (cost, moved slots)."""
  cost = ctypes.c_double()
  moved = (ctypes.c_int * 2)()
  a = np.ascontiguousarray(action)
  rc = lib().swo_action_step(ctypes.byref(cfg), ctypes.byref(tab), _p(sprites), len(sprites),
                             _p(a), int(action_is_f32), ctypes.byref(cost), moved)
  if rc:
    raise KeyError(int(a[1]))
  return cost.value, (moved[0], moved[1])


def task_eval(cfg, sprites):
  r, s, e = ctypes.c_double(), ctypes.c_int(), ctypes.c_int()
  lib().swo_task_eval(ctypes.byref(cfg), _p(sprites), len(sprites), ctypes.byref(r),
                      ctypes.byref(s), ctypes.byref(e))
  return r.value, bool(s.value), e.value


def env_step(cfg, tab, sprites, step_count, action, action_is_f32):
  """One Environment.step after the reset check.  Returns dict of outputs."""
  sc = ctypes.c_int32(step_count)
  r = ctypes.c_double()
  st, su, er = ctypes.c_int8(), ctypes.c_uint8(), ctypes.c_uint8()
  a = np.ascontiguousarray(action)
  rc = lib().swo_env_step(ctypes.byref(cfg), ctypes.byref(tab), _p(sprites), len(sprites),
                          ctypes.byref(sc), _p(a), int(action_is_f32), ctypes.byref(r),
                          ctypes.byref(st), ctypes.byref(su), ctypes.byref(er))
  if rc:
    raise KeyError(int(a[1]))
  return dict(step_count=sc.value, reward=r.value, step_type=st.value,
              success=bool(su.value), err=er.value)


class BatchOracle(object):
  """E envs x S slots with a K-deep scene pool; mirrors the GPU engine's protocol."""

  def __init__(self, cfg, tab, raster, pool):
    """pool: (E, K, S) SPRITE_DTYPE array of pre-sampled scenes (slot 0 = constructor's)."""
    self.cfg, self.tab, self.raster = cfg, tab, raster
    self.pool = np.ascontiguousarray(pool, dtype=SPRITE_DTYPE)
    self.E, self.K, self.S = self.pool.shape
    self.cur = self.pool[:, 0, :].copy()
    self.cursor = np.zeros(self.E, np.int32)
    self.step_count = np.zeros(self.E, np.int32)
    self.reset_next = np.ones(self.E, np.uint8)
    self.reward = np.zeros(self.E, np.float64)
    self.step_type = np.zeros(self.E, np.int8)
    self.success = np.zeros(self.E, np.uint8)
    self.err = np.zeros(self.E, np.uint8)
    self.frames = (np.zeros((self.E, raster.height, raster.width, 3), np.uint8)
                   if raster is not None else None)

  def step(self, actions, e0=0, e1=None):
    e1 = self.E if e1 is None else e1
    a = np.ascontiguousarray(actions)
    f32 = a.dtype == np.float32
    if self.cfg.action_kind == ACT_EMBODIED:
      assert a.dtype == np.int32
    rc = lib().swo_batch_step(
        ctypes.byref(self.cfg), ctypes.byref(self.tab),
        ctypes.byref(self.raster) if self.raster is not None else None,
        self.S, self.K, _p(self.cur), _p(self.pool), _p(self.cursor), _p(self.step_count),
        _p(self.reset_next), _p(a), int(f32), _p(self.reward), _p(self.step_type),
        _p(self.success), _p(self.err),
        _p(self.frames) if self.frames is not None else None, e0, e1)
    if rc:
      raise KeyError('bad Embodied action')
    return self
