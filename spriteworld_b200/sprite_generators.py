"""Generators of sprite lists from factor distributions.

Same four combinators as the reference's `spriteworld/sprite_generators.py:27-128`
(`generate_sprites`, `chain_generators`, `sample_generator`, `shuffle`).  Each returns a
`SpriteGenerator`: calling it yields one list of `Sprite`s with the same draws from
`np.random`, in the same order, as the reference; `.batch(n, rng)` samples `n` scenes at
once into a `SceneLayout` (typed factor tables + a (scene, slot) -> row index), which is
what the batched Environment uploads when many envs reset in the same step.
"""
import numpy as np

from spriteworld_b200 import sprite as sprite_lib


class SpriteTable(object):
  """`rows` sprites as typed factor columns (one homogeneous dtype per factor)."""

  def __init__(self, columns, rows):
    self.columns = columns
    self.rows = rows

  def take(self, index):
    return SpriteTable({k: v[index] for k, v in self.columns.items()}, len(index))


class SceneLayout(object):
  """n scenes; scene i has count[i] sprites, slot j (back to front) is row
  ref_row[i, j] of tables[ref_table[i, j]]."""

  def __init__(self, tables, count, ref_table, ref_row):
    self.tables, self.count = tables, np.asarray(count, np.int64)
    self.ref_table, self.ref_row = ref_table, ref_row

  @property
  def n(self):
    return len(self.count)

  @property
  def width(self):
    return self.ref_row.shape[1]

  def valid(self):
    v = getattr(self, '_valid', None)
    if v is None or v.shape != self.ref_row.shape:
      v = np.arange(self.width)[None, :] < self.count[:, None]
      self._valid = v
    return v

  def rows_of(self, index):
    """Sub-layout of the given scenes (tables are shared)."""
    return SceneLayout(self.tables, self.count[index], self.ref_table[index], self.ref_row[index])


def _ragged_concat(a, b):
  """Slot-wise concatenation of two layouts over the same scenes."""
  n = a.n
  tables = a.tables + b.tables
  count = a.count + b.count
  if n and a.valid().all() and b.valid().all():   # no padding on either side: plain concatenation
    return SceneLayout(tables, count,
                       np.concatenate([a.ref_table, b.ref_table + len(a.tables)], axis=1),
                       np.concatenate([a.ref_row, b.ref_row], axis=1))
  width = int(count.max()) if n else 0
  ref_table = np.zeros((n, width), np.int64)
  ref_row = np.zeros((n, width), np.int64)
  va, vb = a.valid(), b.valid()
  ia, ja = np.nonzero(va)
  ref_table[ia, ja], ref_row[ia, ja] = a.ref_table[va], a.ref_row[va]
  ib, jb = np.nonzero(vb)
  ref_table[ib, jb + a.count[ib]] = b.ref_table[vb] + len(a.tables)
  ref_row[ib, jb + a.count[ib]] = b.ref_row[vb]
  return SceneLayout(tables, count, ref_table, ref_row)


def _stack_scenes(parts, where, n):
  """Layouts for disjoint scene subsets `where[k]` -> one layout over n scenes."""
  tables, count = [], np.zeros(n, np.int64)
  width = max([p.width for p in parts] + [0])
  ref_table = np.zeros((n, width), np.int64)
  ref_row = np.zeros((n, width), np.int64)
  for p, rows in zip(parts, where):
    count[rows] = p.count
    ref_table[rows, :p.width] = p.ref_table + len(tables)
    ref_row[rows, :p.width] = p.ref_row
    tables = tables + p.tables
  return SceneLayout(tables, count, ref_table, ref_row)


class SpriteGenerator(object):
  """Callable returning a list of sprites; `.batch(n)` returns a SceneLayout.

  `max_sprites` is an upper bound of the sprites in one scene, or None when a count is drawn
  by a user callable (the batched environment sizes its sprite slots from it)."""

  def __init__(self, one, many, max_sprites=None, spec=None):
    self._one, self._many = one, many
    self.max_sprites = max_sprites
    self._spec = spec   # what scene_program.compile_program flattens for the device sampler

  def __call__(self):
    return self._one()

  def batch(self, n, rng=None):
    return self._many(n, np.random if rng is None else rng)


def batch_of(generator, n, rng=None):
  """SceneLayout of n scenes from any sprite generator; plain callables are called n times."""
  if isinstance(generator, SpriteGenerator):
    return generator.batch(n, rng)
  return layout_from_sprite_lists([generator() for _ in range(n)])


def layout_from_sprite_lists(scenes):
  """Builds a SceneLayout from Python lists of Sprite objects (slow path)."""
  flat = [s for sc in scenes for s in sc]
  cols = {name: _column([getattr(s, name) for s in flat]) for name in sprite_lib.FACTOR_NAMES}
  cols['_transform'] = np.array([s.transform for s in flat], np.float64).reshape(len(flat), 4)
  cols['_pos_f32'] = np.array([s.position.dtype == np.float32 for s in flat], bool)
  count = np.array([len(sc) for sc in scenes], np.int64)
  width = int(count.max()) if len(count) else 0
  ref_row = np.zeros((len(scenes), width), np.int64)
  start = np.concatenate([[0], np.cumsum(count)[:-1]]) if len(count) else np.zeros(0, np.int64)
  for i, c in enumerate(count):
    ref_row[i, :c] = start[i] + np.arange(c)
  return SceneLayout([SpriteTable(cols, len(flat))], count, np.zeros_like(ref_row), ref_row)


def _column(values):
  from spriteworld_b200.factor_distributions import _as_column
  return _as_column(values)


class uniform_count(object):
  """A sprite count drawn as np.random.randint(lo, hi): picklable, and compilable for the device
  sampler (a lambda count runs on the host only)."""

  def __init__(self, lo, hi):
    self.lo, self.hi = int(lo), int(hi)
    if self.hi <= self.lo:
      raise ValueError('uniform_count needs lo < hi, got (%d, %d)' % (self.lo, self.hi))

  def __call__(self):
    return np.random.randint(self.lo, self.hi)

  def __repr__(self):
    return 'uniform_count(%d, %d)' % (self.lo, self.hi)


def generate_sprites(factor_dist, num_sprites=1):
  """`num_sprites` (int or callable returning int) sprites drawn i.i.d. from `factor_dist`."""

  def how_many():
    return num_sprites() if callable(num_sprites) else num_sprites

  def one():
    return [sprite_lib.Sprite(**factor_dist.sample()) for _ in range(how_many())]

  def many(n, rng):
    if not callable(num_sprites):   # every scene has the same count: row i*num + j, no padding
      count = np.full(n, num_sprites, np.int64)
      total = n * int(num_sprites)
      cols = factor_dist.sample_batch(total, rng=rng) if total else {}
      ref_row = np.arange(total, dtype=np.int64).reshape(n, int(num_sprites))
      return SceneLayout([SpriteTable(cols, total)], count, np.zeros_like(ref_row), ref_row)
    count = np.array([num_sprites() for _ in range(n)], np.int64)
    total = int(count.sum())
    cols = factor_dist.sample_batch(total, rng=rng) if total else {}
    width = int(count.max()) if n else 0
    start = np.concatenate([[0], np.cumsum(count)[:-1]]) if n else np.zeros(0, np.int64)
    ref_row = start[:, None] + np.arange(width)[None, :]
    ref_row = np.where(np.arange(width)[None, :] < count[:, None], ref_row, 0)
    return SceneLayout([SpriteTable(cols, total)], count, np.zeros_like(ref_row), ref_row)

  return SpriteGenerator(one, many, None if callable(num_sprites) else int(num_sprites),
                         spec=('sprites', factor_dist, num_sprites))


def _bounds(generators):
  return [getattr(g, 'max_sprites', None) for g in generators]


def chain_generators(*sprite_generators):
  """Concatenates the outputs of several generators ("AND")."""

  def one():
    out = []
    for g in sprite_generators:
      out.extend(g())
    return out

  def many(n, rng):
    layout = batch_of(sprite_generators[0], n, rng)
    for g in sprite_generators[1:]:
      layout = _ragged_concat(layout, batch_of(g, n, rng))
    return layout

  bounds = _bounds(sprite_generators)
  return SpriteGenerator(one, many, None if None in bounds else sum(bounds),
                         spec=('chain', sprite_generators))


def sample_generator(sprite_generators, p=None):
  """Each call picks one generator at random ("OR") and returns its output."""

  def one():
    return sprite_generators[np.random.choice(len(sprite_generators), p=p)]()

  def many(n, rng):
    which = rng.choice(len(sprite_generators), size=n, p=p)
    parts, where = [], []
    for i, g in enumerate(sprite_generators):
      rows = np.flatnonzero(which == i)
      if len(rows):
        parts.append(batch_of(g, len(rows), rng))
        where.append(rows)
    return _stack_scenes(parts, where, n)

  bounds = _bounds(sprite_generators)
  return SpriteGenerator(one, many, None if None in bounds else max(bounds),
                         spec=('sample', sprite_generators, p))


def shuffle(sprite_generator):
  """Randomises the z-order of the generated sprites (occlusion carries no information)."""

  def one():
    sprites = sprite_generator()
    order = np.arange(len(sprites))
    np.random.shuffle(order)
    return [sprites[i] for i in order]

  def many(n, rng):
    layout = batch_of(sprite_generator, n, rng)
    keys = rng.uniform(size=(layout.n, layout.width))
    keys = np.where(layout.valid(), keys, np.inf)     # empty slots stay at the end
    order = np.argsort(keys, axis=1, kind='stable')
    rows = np.arange(layout.n)[:, None]
    return SceneLayout(layout.tables, layout.count, layout.ref_table[rows, order],
                       layout.ref_row[rows, order])

  return SpriteGenerator(one, many, getattr(sprite_generator, 'max_sprites', None),
                         spec=('shuffle', sprite_generator))
