"""Host-side scene batches: what `init_sprites()` returned, reduced to the struct-of-arrays
the engine uploads (include/spriteworld_b200.h: swb_scene_soa).

A scene batch is a dict of numpy arrays shaped (n_scenes, n_slots[, ...]):
  x, y            float64   initial position (float32-valued where pos_f32)
  m00..m11        float64   centred-path transform, scale then rotate (sprite.py:96-101)
  vx, vy          float64   velocity
  member          uint32    bit i = task filter i contains the sprite (tasks.py:136,201)
  shape           uint8     ShapeType id, 0 = empty slot (slots are padded at the FRONT)
  pos_f32         uint8     the reference's position ndarray would be float32
  rgb             uint8 x3  color_to_rgb(sprite.color) (pil_renderer.py:82)
  factors         float32x5 scale, angle, c0, c1, c2 (for factor observations)
"""
import math

import numpy as np

from spriteworld_b200 import _host_pack

F64_FIELDS = ('x', 'y', 'm00', 'm01', 'm10', 'm11', 'vx', 'vy')


def transform_matrix(scale, angle):
  """Matrix of Affine2D().scale(s) + Affine2D().rotate_deg(a) (sprite.py:96-101).

  rotate_deg goes through math.radians / math.cos / math.sin (libm), and the composite
  matrix is rotate . scale, whose entries are single products.
  """
  s = float(scale)
  th = math.radians(angle)
  c, sn = math.cos(th), math.sin(th)
  return c * s, (-sn) * s, sn * s, c * s


_matrix_cache = {}


def transform_matrices(scale, angle):
  """Vectorised transform_matrix over arrays: the scalar function runs once per distinct
  (scale, angle) bit pattern (configs use few) and the results are scattered back."""
  scale = np.ascontiguousarray(scale, dtype=np.float64)
  angle = np.ascontiguousarray(angle, dtype=np.float64)
  if scale.size == 0:
    return np.empty(scale.shape + (4,), np.float64)
  sb, ab = scale.reshape(-1).view(np.int64), angle.reshape(-1).view(np.int64)
  if sb.min() == sb.max() and ab.min() == ab.max():   # one (scale, angle) bit pattern for all
    key = (float(scale.reshape(-1)[0]), float(angle.reshape(-1)[0]))
    m = transform_matrix(key[0], key[1])
    return np.broadcast_to(np.array(m, np.float64), scale.shape + (4,)).copy()
  # distinct by bit pattern (0.0 and -0.0 stay apart: they give differently signed zeros);
  # two 1-D uniques and one over the combined small index are much cheaper than a row-wise one
  us, inv_s = np.unique(scale.reshape(-1).view(np.int64), return_inverse=True)
  ua, inv_a = np.unique(angle.reshape(-1).view(np.int64), return_inverse=True)
  pair_ids, inverse = np.unique(inv_s.reshape(-1) * len(ua) + inv_a.reshape(-1), return_inverse=True)
  us, ua = us.view(np.float64), ua.view(np.float64)
  mats = np.empty((pair_ids.shape[0], 4), np.float64)
  for i, pid in enumerate(pair_ids):
    key = (us[pid // len(ua)], ua[pid % len(ua)])
    m = _matrix_cache.get(key)
    if m is None:
      m = transform_matrix(key[0], key[1])
      if len(_matrix_cache) < 65536:
        _matrix_cache[key] = m
    mats[i] = m
  return mats[inverse.reshape(-1)].reshape(scale.shape + (4,))


def empty_batch(n_scenes, n_slots, zero=True):
  """zero=False: uninitialised arrays, for a caller that fills every slot."""
  new = np.zeros if zero else np.empty
  b = {f: new((n_scenes, n_slots), np.float64) for f in F64_FIELDS}
  b['member'] = new((n_scenes, n_slots), np.uint32)
  b['shape'] = new((n_scenes, n_slots), np.uint8)
  b['pos_f32'] = new((n_scenes, n_slots), np.uint8)
  b['rgb'] = new((n_scenes, n_slots, 3), np.uint8)
  b['factors'] = new((n_scenes, n_slots, 5), np.float32)
  return b


def batch_from_factor_arrays(x, y, pos_f32, shape, angle, scale, c0, c1, c2, vx, vy, member, rgb):
  """All arguments are arrays shaped (n, S) (rgb: (n, S, 3)); shape 0 marks empty slots."""
  x = np.asarray(x, np.float64)
  b = empty_batch(*x.shape)
  b['x'][:], b['y'][:] = x, np.asarray(y, np.float64)
  b['vx'][:], b['vy'][:] = vx, vy
  b['member'][:], b['shape'][:], b['pos_f32'][:] = member, shape, pos_f32
  b['rgb'][:] = rgb
  m = transform_matrices(scale, angle)
  occupied = b['shape'] > 0
  for i, f in enumerate(('m00', 'm01', 'm10', 'm11')):
    b[f][:] = np.where(occupied, m[..., i], 0.0)
  b['factors'][..., 0], b['factors'][..., 1] = scale, angle
  b['factors'][..., 2], b['factors'][..., 3], b['factors'][..., 4] = c0, c1, c2
  return b


# ---------------------------------------------------------------------------------
# SceneLayout (sprite_generators.py) -> scene arrays
# ---------------------------------------------------------------------------------

_DEFAULTS = dict(x=0.5, y=0.5, shape='square', angle=0, scale=0.1, c0=0, c1=0, c2=0,
                 x_vel=0.0, y_vel=0.0)   # Sprite.__init__ defaults (sprite.py:56-66)


def _default_column(default, rows):
  """`rows` copies of a Sprite.__init__ default, typed like factor_distributions._as_column
  types a list of them: float -> float64, int -> int64, anything else an object column."""
  if isinstance(default, float):
    return np.full(rows, default, np.float64)
  if isinstance(default, int):
    return np.full(rows, default, np.int64)
  out = np.empty(rows, dtype=object)
  out[:] = [default] * rows
  return out


def _full_columns(table):
  """The ten factor columns of a SpriteTable, defaults filled in, typed like
  `Sprite.factors` would type them (positions are float32 only if x and y both are)."""
  cols = {}
  for name, default in _DEFAULTS.items():
    col = table.columns.get(name)
    cols[name] = _default_column(default, table.rows) if col is None else col
  x, y = cols['x'], cols['y']
  if not (x.dtype == np.float32 and y.dtype == np.float32):
    # np.array([x, y]) promotes: anything that is not float32 + float32 becomes float64
    if x.dtype != object:
      cols['x'] = x.astype(np.float64)
    if y.dtype != object:
      cols['y'] = y.astype(np.float64)
  return cols


def _numeric(col):
  if col.dtype == object:
    return np.array([float(v) for v in col], np.float64)
  return col.astype(np.float64)


def _is_f32(col):
  if col.dtype == object:
    return np.array([isinstance(v, np.float32) for v in col], bool)
  return np.full(len(col), col.dtype == np.float32, bool)


_SHAPE_ID_CACHE = {}


def _shape_ids(col):
  from spriteworld_b200 import constants
  if col.dtype != object and np.issubdtype(col.dtype, np.integer):
    return col.astype(np.uint8)
  # Object column of names.  Discrete.sample_batch indexes a small typed column of candidates, so
  # the elements are a handful of distinct Python objects repeated: map each distinct POINTER once
  # (the column's buffer is an array of PyObject*), instead of one dict lookup per element.
  table = _SHAPE_ID_CACHE
  if len(col) >= 256 and col.flags.c_contiguous:
    import ctypes
    ptrs = np.ctypeslib.as_array((ctypes.c_size_t * len(col)).from_address(col.ctypes.data))
    uniq, inverse = np.unique(ptrs, return_inverse=True)
    if len(uniq) <= 64:
      first = np.zeros(len(uniq), np.int64)
      first[inverse[::-1]] = np.arange(len(col) - 1, -1, -1)   # an element index per distinct object
      ids = np.empty(len(uniq), np.uint8)
      for k, i in enumerate(first):
        v = col[i]
        if v not in table:
          table[v] = int(constants.ShapeType[str(v)])
        ids[k] = table[v]
      return ids[inverse.reshape(-1)]
  try:
    return np.fromiter(map(table.__getitem__, col.tolist()), np.uint8, len(col))
  except KeyError:
    for v in set(col.tolist()):
      table[v] = int(constants.ShapeType[str(v)])
    return np.fromiter(map(table.__getitem__, col.tolist()), np.uint8, len(col))


def _table_rgb(cols, color_to_rgb, num=None):
  from spriteworld_b200.renderers import color_maps
  c = [cols['c0'], cols['c1'], cols['c2']]
  rows = len(c[0])
  if color_to_rgb is None:   # colours are already RGB (pil_renderer.py:53-55)
    return np.stack([_numeric(a).astype(np.int64) for a in c], -1).astype(np.uint8)
  homogeneous = all(a.dtype != object for a in c) and len({a.dtype for a in c}) == 1
  if color_to_rgb is color_maps.hsv_to_rgb and homogeneous and c[0].dtype in (
      np.dtype(np.float32), np.dtype(np.float64)):
    if num is not None:
      return color_maps.hsv_to_rgb_batch(num['c0'], num['c1'], num['c2'], c[0].dtype == np.float32)
    return color_maps.hsv_to_rgb_batch(_numeric(c[0]), _numeric(c[1]), _numeric(c[2]),
                                       c[0].dtype == np.float32)
  out = np.zeros((rows, 3), np.uint8)   # arbitrary callable or mixed scalar types
  for i in range(rows):
    out[i] = [int(v) for v in color_to_rgb((c[0][i], c[1][i], c[2][i]))]
  return out


def draw_goals(goal_distribs, n, rng):
  """float64 (n, G, 2): the goals of n scenes, drawn per goal slot in slot order, each slot's n
  goals with one goal_distrib.sample_batch(n, rng) call.  None without goal distributions."""
  if not goal_distribs:
    return None
  out = np.empty((n, len(goal_distribs), 2), np.float64)
  for g, d in enumerate(goal_distribs):
    cols = d.sample_batch(n, rng)
    out[:, g, 0] = np.asarray(cols['x'], dtype=np.float64)
    out[:, g, 1] = np.asarray(cols['y'], dtype=np.float64)
  return out


def arrays_from_layout(layout, n_slots, filters=(), color_to_rgb=None):
  """SceneLayout -> scene batch (n, n_slots), sprites right-aligned (empty slots first).

  Args:
    layout: sprite_generators.SceneLayout.
    n_slots: sprite slots per env.
    filters: task filter distributions; bit i of `member` = filters[i].contains(sprite).
    color_to_rgb: the PILRenderer's colour map (None, color_maps.hsv_to_rgb or a callable).
  """
  if layout.n and int(layout.count.max()) > n_slots:
    raise ValueError('a scene has %d sprites but the engine has %d slots'
                     % (int(layout.count.max()), n_slots))
  tables, offsets = _merged_tables(layout.tables)
  n = layout.n
  valid = layout.valid()
  full = bool(valid.all()) and layout.width == n_slots    # every slot of every scene gets written
  b = empty_batch(n, n_slots, zero=not full)
  if full:
    flat_dst = None
    tab, row = layout.ref_table.reshape(-1), layout.ref_row.reshape(-1)
  else:
    scene_i, slot_j = np.nonzero(valid)
    flat_dst = scene_i * n_slots + (n_slots - layout.count[scene_i] + slot_j)
    tab, row = layout.ref_table[valid], layout.ref_row[valid]
  if offsets is not None:
    row = row + offsets[tab]                        # the tables were concatenated into one
    tab = None
  if (tab is None or len(tables) == 1) and tables and tables[0].rows and _host_pack.pack(
      tables[0], filters, color_to_rgb, row, flat_dst, b):
    return b                                        # one native pass over the sprites
  per_table = [None if t.rows == 0 else _table_arrays(t, filters, color_to_rgb) for t in tables]
  fields = ('x', 'y', 'm00', 'm01', 'm10', 'm11', 'vx', 'vy', 'member', 'shape', 'pos_f32', 'rgb', 'factors')
  for t, data in enumerate(per_table):
    if data is None:
      continue
    if tab is None:
      dst, ri = flat_dst, row
    else:
      sel = tab == t
      dst, ri = (np.flatnonzero(sel) if flat_dst is None else flat_dst[sel]), row[sel]
    for f in fields:
      out = b[f].reshape((n * n_slots,) + b[f].shape[2:])
      if dst is None and data[f].dtype == out.dtype:
        np.take(data[f], ri, axis=0, out=out)     # straight into the batch, no temporary
      elif dst is None:
        out[...] = data[f][ri]
      else:
        out[dst] = data[f][ri]
  return b


def _merged_tables(tables):
  """Concatenates the layout's sprite tables into one when their columns have the same names
  and dtypes (the usual case: several generate_sprites over the same factor names), so that
  the per-table work (filters, transforms, colour map) runs once.  Returns (tables, row offset
  of each original table or None)."""
  live = [t for t in tables if t.rows]
  if len(live) < 2:
    return tables, None
  keys = set(live[0].columns)
  if any(set(t.columns) != keys for t in live[1:]):
    return tables, None
  for k in keys:
    if len({t.columns[k].dtype for t in live}) != 1:
      return tables, None
  from spriteworld_b200 import sprite_generators
  offsets = np.zeros(len(tables), np.int64)
  run = 0
  for i, t in enumerate(tables):
    offsets[i] = run
    run += t.rows
  merged = sprite_generators.SpriteTable(
      {k: np.concatenate([t.columns[k] for t in live]) for k in keys}, run)
  return [merged], offsets


def _factor_columns(num):
  out = np.empty((len(num['scale']), 5), np.float32)
  for i, k in enumerate(('scale', 'angle', 'c0', 'c1', 'c2')):
    out[:, i] = num[k]     # through float64, like the stacked form it replaces
  return out


class _NumericCache(dict):
  """cols[name] as float64, converted once per table (several consumers want the same columns)."""

  def __init__(self, cols):
    super().__init__()
    self._cols = cols

  def __missing__(self, name):
    v = _numeric(self._cols[name])
    self[name] = v
    return v


def _table_arrays(table, filters, color_to_rgb):
  cols = _full_columns(table)
  num = _NumericCache(cols)
  member = np.zeros(table.rows, np.uint32)
  for bit, f in enumerate(filters):
    member |= np.asarray(f.contains_batch(cols), bool).astype(np.uint32) << np.uint32(bit)
  if '_transform' in table.columns:
    m = table.columns['_transform']
  else:
    m = transform_matrices(num['scale'], num['angle'])
  pos_f32 = table.columns.get('_pos_f32')
  if pos_f32 is None:
    pos_f32 = _is_f32(cols['x']) & _is_f32(cols['y'])
  return dict(
      x=num['x'], y=num['y'], m00=m[:, 0], m01=m[:, 1], m10=m[:, 2],
      m11=m[:, 3], vx=num['x_vel'], vy=num['y_vel'], member=member,
      shape=_shape_ids(cols['shape']), pos_f32=pos_f32.astype(np.uint8),
      rgb=_table_rgb(cols, color_to_rgb, num), factors=_factor_columns(num))
