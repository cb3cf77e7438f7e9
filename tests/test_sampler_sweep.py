"""The device scene sampler over every program op, factor dtype and colour path, against a NumPy
restatement of it (no GPU needed).

The programs are seeded random scene generators built from the package's own combinators and
distributions, plus hand-written cases at the edges where float-to-integer conversions and
rejection loops go wrong.  scene_program.sample_on_host (csrc/swb_sampler.cuh built for the CPU)
must equal `restate`, bit for bit: every pool field and the drawn factor table.  `restate` walks
the generator and distribution objects themselves, independent of compile_program and of the C++
source; Sprite objects and scene.arrays_from_layout (the host sampler's packing) are the spec for
every pool field.

The word consumption of a scene (g, a) under seed s, the contract both builds follow:
  stream   np.random.Philox(counter=(a << 64) + (g << 128) - 1, key=(s, DOMAIN)): successive
           words 0, 1, 2, ...; each `draw` below takes the next word.
  uniform  (w >> 11) * 2**-53                    below(n)  (w * n) >> 64
  choice   over probabilities p: cdf = cumsum(p) / sum; the first index whose cdf entry exceeds
           one uniform (np.searchsorted(cdf, u, 'right')), clamped to len(p) - 1
  generate_sprites(d, n)      n sprites, in order; uniform_count(lo, hi): lo + below(hi - lo) first
  chain_generators(*gs)       each generator in order
  sample_generator(gs, p)     one choice (uniform weights when p is None), then that generator
  shuffle(g)                  g, then Fisher-Yates over g's sprites from the top:
                              for i = last .. first + 1: swap i with first + below(i - first + 1)
  Continuous(k, lo, hi, dt)   one uniform u; np.asarray(lo + (hi - lo) * u).astype(dt)[()]
  Discrete(k, c, probs)       below(len(c)) without probs, one choice with them
  Product(cs)                 each component in order
  Mixture(cs, probs)          one choice, then that component
  Intersection(cs, i)         draw cs[i] until every component contains the draw
  SetMinus(b, h)              draw b until h does not contain the draw
  Selection(b, f)             draw b until f contains the draw
A rejection loop gives up after factor_distributions._MAX_TRIES draws: the scene is then empty.
"""
import colorsys
import functools

import numpy as np
import pytest

from spriteworld_b200 import constants, scene, scene_program
from spriteworld_b200 import factor_distributions as distribs
from spriteworld_b200 import sprite as sprite_lib
from spriteworld_b200 import sprite_generators as gen
from spriteworld_b200.renderers import color_maps

DOMAIN = 0x53574253434e4531   # SWB_SAMPLER_DOMAIN
M64 = 2 ** 64 - 1
FIELDS = ('x', 'y', 'm00', 'm01', 'm10', 'm11', 'vx', 'vy', 'member', 'shape', 'pos_f32', 'rgb',
          'factors', 'factor_value', 'factor_kind')
# SWB_FT_* of include/spriteworld_b200.h, restated
FT = {np.float32: 1, np.float64: 2, np.int8: 3, np.int16: 4, np.int32: 5, np.int64: 6, np.uint8: 7,
      np.uint16: 8, np.uint32: 9, np.uint64: 10}
FT_SHAPE, FT_PYFLOAT, FT_PYINT = 11, 12, 13
OPS = (list(range(0, 6)) + list(range(10, 17)) + list(range(20, 26)))
DEFAULTS = dict(x=0.5, y=0.5, shape='square', angle=0, scale=0.1, c0=0, c1=0, c2=0, x_vel=0.0,
                y_vel=0.0)
FACTORS = tuple(DEFAULTS)
INT_DTYPES = ('int8', 'int16', 'int32', 'int64', 'uint8', 'uint16', 'uint32', 'uint64')
FLOAT_DTYPES = ('float32', 'float64')
SHAPES = tuple(constants.SHAPE_NAMES)


def bits(a):
  a = np.ascontiguousarray(a)
  return a.view(np.uint8) if a.dtype.kind == 'f' else a


# -- the restatement -----------------------------------------------------------------------------


class Words(object):
  """The draw words of scene (g, a) under `seed`."""

  def __init__(self, seed, g, a):
    c = ((int(g) << 128) + (int(a) << 64) - 1) % (1 << 256)
    ctr = np.array([(c >> (64 * i)) & M64 for i in range(4)], np.uint64)
    self._bg = np.random.Philox(counter=ctr, key=np.array([int(seed) & M64, DOMAIN], np.uint64))
    self._buf, self._pos = [], 0

  def next(self):
    if self._pos == len(self._buf):
      self._buf, self._pos = self._bg.random_raw(16).tolist(), 0
    self._pos += 1
    return self._buf[self._pos - 1]

  def uniform(self):
    return (self.next() >> 11) * 2.0 ** -53

  def below(self, n):
    return (self.next() * int(n)) >> 64

  def choice(self, p):
    cdf = np.cumsum(np.array(p, np.float64))
    cdf /= cdf[-1]
    return min(int(np.searchsorted(cdf, self.uniform(), side='right')), len(cdf) - 1)


class RejectionFailed(Exception):

  def __init__(self, dist):
    super().__init__(str(dist))
    self.dist = dist


def draw(d, w, stats):
  """One spec of distribution `d` (dict factor -> value, typed as the host sampler types it)."""
  if isinstance(d, distribs.Continuous):
    lo, hi = float(d.minval), float(d.maxval)
    return {d.key: np.asarray(lo + (hi - lo) * w.uniform()).astype(d.dtype)[()]}
  if isinstance(d, distribs.Discrete):
    n = len(d.candidates)
    return {d.key: d.candidates[w.below(n) if d.probs is None else w.choice(d.probs)]}
  if isinstance(d, distribs.Product):
    spec = {}
    for c in d.components:
      spec.update(draw(c, w, stats))
    return spec
  if isinstance(d, distribs.Mixture):
    return draw(d.components[w.choice(d.probs)], w, stats)
  if isinstance(d, distribs.Intersection):
    source, accept = d.components[d.index_for_sampling], d.contains
  else:   # SetMinus, Selection
    source = d.base
    accept = lambda s: d._other.contains(s) == d._keep_if_inside  # noqa: E731
  for _ in range(distribs._MAX_TRIES):
    spec = draw(source, w, stats)
    if accept(spec):
      return spec
    stats['retries'] += 1
    if stats['retries'] > stats['limit']:
      raise _TooSlow()
  raise RejectionFailed(d)


class _TooSlow(Exception):
  pass


def generate(g, w, out, stats):
  """Appends the factor specs of generator `g`'s sprites to `out`, back to front."""
  spec = g._spec
  if spec[0] == 'sprites':
    _, d, num = spec
    n = num.lo + w.below(num.hi - num.lo) if isinstance(num, gen.uniform_count) else int(num)
    for _ in range(n):
      out.append(draw(d, w, stats))
  elif spec[0] == 'chain':
    for child in spec[1]:
      generate(child, w, out, stats)
  elif spec[0] == 'sample':
    children, p = spec[1], spec[2]
    n = len(children)
    generate(children[w.choice(np.ones(n) / n if p is None else p)], w, out, stats)
  else:   # shuffle
    lo = len(out)
    generate(spec[1], w, out, stats)
    for i in range(len(out) - 1, lo, -1):
      j = lo + w.below(i - lo + 1)
      out[i], out[j] = out[j], out[i]


def _kind(v):
  if isinstance(v, str):
    return FT_SHAPE
  if isinstance(v, np.generic):
    return FT[type(v)]
  return FT[np.float64] if isinstance(v, float) else FT[np.int64]


def _value(v):
  return float(int(constants.ShapeType[v])) if isinstance(v, str) else float(v)


def restate(case, seed, env_ids, scene_idx, n_slots, stats=None, stop_at_failure=False):
  """(arrays of scene_program.empty_sample, (index, distribution) of the first scene whose
  rejection loop ran out of tries, or None) for scenes (env_ids[i], scene_idx[i])."""
  stats = stats if stats is not None else _new_stats()
  n = len(env_ids)
  out = scene_program.empty_sample(n, n_slots)
  fail = None
  for i in range(n):
    specs = []
    try:
      generate(case.gen, Words(seed, env_ids[i], scene_idx[i]), specs, stats)
    except RejectionFailed as e:
      specs = []
      if fail is None:
        fail = (i, e.dist)
    stats['sprites'].append(len(specs))
    full = [dict(DEFAULTS, **s) for s in specs]
    if case.cmap is not None:
      for f in full:
        rgb = colorsys.hsv_to_rgb(float(f['c0']), float(f['c1']), float(f['c2']))
        stats['neg_hsv'] += min(rgb) < 0
        stats['hsv_over_int32'] += max(abs(c) for c in rgb) * 255 >= 2 ** 31
    b = scene.arrays_from_layout(gen.layout_from_sprite_lists([[sprite_lib.Sprite(**s) for s in specs]]),
                                 n_slots, case.filters, case.cmap)
    for k, v in b.items():
      out[k][i] = v[0]
    for j, f in enumerate(full):
      slot = n_slots - len(full) + j
      out['factor_value'][i, slot] = [_value(f[k]) for k in FACTORS]
      out['factor_kind'][i, slot] = [_kind(f[k]) for k in FACTORS]
    if fail is not None and stop_at_failure:
      return {k: v[:i + 1] for k, v in out.items()}, fail
  return out, fail


def _new_stats():
  return dict(retries=0, neg_hsv=0, hsv_over_int32=0, sprites=[], limit=float('inf'))


def assert_same(got, want, what):
  for k in FIELDS:
    g, r = bits(got[k]), bits(want[k])
    if k == 'member':
      g = g.view(np.uint32)
    if not np.array_equal(g, r):
      bad = np.flatnonzero((g != r).reshape(len(r), -1).any(1))
      raise AssertionError('%s: field %s differs in %d scenes, first scene %d: %r vs %r' % (
          what, k, len(bad), bad[0], got[k][bad[0]], want[k][bad[0]]))


def scene_ids(n):
  """n (env id, scene index) pairs: small ones, and some near 2**62 and 2**63 - 1."""
  rng = np.random.RandomState(n)
  big = [2 ** 63 - 1, 2 ** 63 - 2, 2 ** 62, 2 ** 62 - 1, 0, 1]
  k = n - 2 * len(big)
  ids = np.concatenate([np.arange(k) % 11, big, rng.randint(2 ** 62 - 64, 2 ** 62 + 64, len(big))])
  idx = np.concatenate([np.arange(k) // 11, big[::-1], rng.randint(0, 2 ** 62, len(big))])
  return ids.astype(np.int64), idx.astype(np.int64)


SEEDS = (7, 2 ** 64 - 3)


# -- the programs ----------------------------------------------------------------------------------


class Case(object):

  def __init__(self, name, init_sprites, filters=(), cmap=None, impossible=False):
    self.name, self.gen, self.filters, self.cmap = name, init_sprites, list(filters), cmap
    self.impossible = impossible
    self.program = scene_program.compile_program(init_sprites, self.filters, cmap)


C, D, P = distribs.Continuous, distribs.Discrete, distribs.Product
HSV = color_maps.hsv_to_rgb


def _hsv(h, s, v, dtype='float64'):
  return [C('c0', h[0], h[1], dtype), C('c1', s[0], s[1], dtype), C('c2', v[0], v[1], dtype)]


def _pos(dtype='float64'):
  return [C('x', 0.05, 0.95, dtype), C('y', 0.05, 0.95, dtype), C('scale', 0.05, 0.2)]


def _edge_cases():
  out = []
  f_hue = [C('c0', -0.5, 0.0), C('c0', 0.0, 1.0), D('c0', [np.float32(-0.25), -0.25]), C('c1', 1.0, 3.0)]
  for dt in FLOAT_DTYPES:
    out.append(Case('hue_below_0_' + dt, gen.generate_sprites(P(_pos() + _hsv((-0.5, 0.0), (0.3, 1.0), (0.2, 1.0), dt)), 6),
                    f_hue, HSV))
    out.append(Case('hue_above_1_' + dt, gen.generate_sprites(P(_pos() + _hsv((1.0, 2.0), (0.0, 1.0), (0.0, 1.0), dt)), 6),
                    f_hue, HSV))
    out.append(Case('saturation_above_1_' + dt, gen.generate_sprites(
        P(_pos() + _hsv((0.0, 1.0), (1.0, 2.0), (0.1, 1.0), dt)), 6), f_hue, HSV))
    out.append(Case('value_below_0_' + dt, gen.generate_sprites(
        P(_pos() + _hsv((-0.2, 1.2), (0.0, 1.5), (-3.0, 0.0), dt)), 6), f_hue, HSV))
    out.append(Case('value_past_int32_' + dt, gen.generate_sprites(
        P(_pos() + _hsv((-0.3, 1.3), (0.0, 1.5), (1e6, 1e11), dt)), 6), f_hue, HSV))
    t = np.dtype(dt).type
    out.append(Case('saturation_0_' + dt, gen.generate_sprites(P(_pos() + [
        C('c0', -0.5, 2.0, dt), D('c1', [t(0.0), t(0.5)]), C('c2', -2.0, 2.0, dt)]), 6), (), HSV))
  out.append(Case('rgb_float_1e19', gen.generate_sprites(P(_pos() + [
      C('c0', -1e19, 1e19, 'float64'), D('c1', [1e19, -1e19, 300.7, -3.2, -2.0 ** 63, 2.0 ** 63]),
      C('c2', -1e19, 1e19, 'float32')]), 8), [C('c0', 0, 1e19), C('c2', -1e19, 0)]))
  u64 = [C('c0', 2 ** 63, 2 ** 64 - 4096, 'uint64'), C('c1', 0, 2 ** 64 - 4096, 'uint64'),
         C('scale', 2 ** 63, 2 ** 64 - 4096, 'uint64'), C('x_vel', 0, 2 ** 64 - 4096, 'uint64')]
  out.append(Case('uint64_above_2_63', gen.generate_sprites(P(_pos()[:2] + u64), 8), [
      C('c0', 0.5, 1.5e19), C('c1', 2 ** 53, 1e30), C('c1', np.uint64(2 ** 63 + 2 ** 20), np.uint64(2 ** 64 - 2 ** 12)),
      C('scale', np.int64(0), np.float32(1.5e19)), D('c0', [np.uint64(2 ** 63), 17]),
      C('x_vel', np.int64(-5), np.int64(2 ** 62)), C('c1', -1, np.float64(1e19))]))
  ints = [C('c0', -2 ** 63, -2 ** 63 + 2 ** 20, 'int64'), C('c1', 2 ** 63 - 2 ** 20, 2 ** 63 - 1024, 'int64'),
          C('c2', -128, 128, 'int8'), C('scale', 0, 256, 'uint8'), C('x_vel', -2 ** 15, 2 ** 15, 'int16'),
          C('y_vel', 0, 2 ** 16, 'uint16')]
  out.append(Case('integer_limits', gen.generate_sprites(P(_pos()[:2] + ints), 8), [
      C('c0', -2 ** 53, 0), C('c1', np.int64(2 ** 63 - 2 ** 19), np.uint64(2 ** 63)), C('c2', -1, 1000),
      C('scale', np.int8(-1), np.uint8(200)), D('x_vel', [0, -1, np.int16(-2), 2.0]), C('y_vel', 300, 70000)]))
  ints32 = [C('c0', -2 ** 31, 2 ** 31, 'int32'), C('c1', 0, 2 ** 32, 'uint32'), C('c2', 2 ** 31, 2 ** 32, 'uint32')]
  out.append(Case('integer_limits_32', gen.generate_sprites(P(_pos()[:2] + ints32), 8),
                  [C('c0', np.float32(-2 ** 31), 0), C('c2', np.uint32(2 ** 31 + 5), 2 ** 32)]))
  ang = distribs.Mixture([D('angle', [-0.0, 0.0]), C('angle', -30, 20, 'int16'), C('angle', -200, -100, 'int32'),
                          D('angle', [np.float32(-45.5), np.float32(0.0), np.float32(-0.0)])], probs=[0.4, 0.3, 0.2, 0.1])
  out.append(Case('angles', gen.generate_sprites(P(_pos() + [ang]), 8), [D('angle', [0, -0.0, -30])]))
  out.append(Case('x_float32_y_float64', gen.generate_sprites(P([
      D('x', [np.float32(0.9), np.float32(0.25)]), C('y', 0, 1, 'float64'), C('c0', 0, 255)]), 6),
      [C('x', 0, 0.9), C('y', 0, np.float32(0.5)), D('x', [np.float32(0.9), 0.9])]))
  sel = distribs.Selection(P([C('scale', 0, 1, 'float64'), C('c0', 0, 1)]), C('scale', 0.5, 0.51))
  inter = distribs.Intersection([C('c1', 0, 1, 'float64'), C('c1', 0.2, 0.21)], index_for_sampling=0)
  out.append(Case('rejection_one_percent', gen.generate_sprites(P([sel, inter]), 3), [C('c0', 0.5, 1)]))
  nested = distribs.SetMinus(
      distribs.Selection(distribs.Mixture([P([C('x', 0, 1), C('c0', 0, 1, 'float64')]),
                                           P([D('x', [0.1, 0.9]), C('c0', -1, 1, 'float64')])], probs=[0.3, 0.7]),
                         C('c0', 0, 0.5)),
      distribs.Intersection([C('x', 0, 0.5), C('x', 0.25, 1)], index_for_sampling=1))
  out.append(Case('rejection_in_rejection', gen.shuffle(gen.generate_sprites(nested, gen.uniform_count(1, 6))),
                  [nested, distribs.Mixture([C('c0', 0, 0.1), D('c0', [0.1])])]))
  body = P(_pos() + [C('c0', 0, 1, 'float32'), C('c1', 0, 1, 'float32'), C('c2', 0, 1, 'float32')])
  out.append(Case('zero_sprites', gen.chain_generators(gen.generate_sprites(body, 0),
                                                       gen.generate_sprites(body, gen.uniform_count(0, 1))), (), HSV))
  bit_filters = [C('scale', 0.05 + 0.15 * k / 32, 0.05 + 0.15 * (k + 2) / 32) for k in range(31)] + [C('c0', 0.5, 1)]
  out.append(Case('32_sprites_32_filters', gen.shuffle(gen.chain_generators(
      gen.generate_sprites(body, 16), gen.shuffle(gen.generate_sprites(body, gen.uniform_count(10, 17))))),
      bit_filters, HSV))
  gens = [gen.generate_sprites(body, k) for k in (1, 2, 3, 4)]
  out.append(Case('sample_generator_zero_p', gen.sample_generator(gens, p=[0.0, 0.7, 0.0, 0.3]),
                  [C('c0', 0.25, 0.75)], HSV))
  npk = [D('c0', [t(v) for v in (1, 7, 100)], probs=[0.5, 0.0, 0.5]) for t in FT if t not in (np.uint64,)]
  out.append(Case('numpy_scalar_candidates', gen.sample_generator(
      [gen.generate_sprites(P(_pos()[:2] + [d]), 2) for d in npk] +
      [gen.generate_sprites(P(_pos()[:2] + [D('c0', [np.uint64(2 ** 63), np.uint64(3)], probs=[0.0, 1.0])]), 1)]),
      [D('c0', [np.uint8(7), 100.0, np.float32(1)]), C('c0', np.int8(1), np.uint16(100))]))
  out.append(Case('p_or', gen.generate_sprites(P(_pos() + [C('c0', 0, 1), D('shape', list(SHAPES[:4]))]), 5), [
      distribs.Mixture([C('c0', 0, 0.3), D('c0', [0.5])]),
      distribs.Mixture([D('shape', [SHAPES[0]]), D('shape', [SHAPES[2], 'nonshape'])]),
      distribs.SetMinus(C('c0', 0, 1), C('c0', 0.2, 0.4))]))
  out.append(Case('float32_int_bound', gen.generate_sprites(P([C('scale', 1.6e7, 1.8e7, 'float32'),
                                                               D('c0', [np.float32(16777217), np.float32(0.5)])]), 4),
                  [C('scale', 16777217, 2 ** 25), C('c0', 16777217, 16777218)]))
  base = P([C('x', 0.2, 0.4), C('y', 0.2, 0.4)] + [C(c, 0.5, 0.6) for c in ('c0', 'c1', 'c2')])
  ok = gen.generate_sprites(base, 2)
  out.append(Case('impossible', gen.sample_generator([ok, gen.generate_sprites(
      distribs.SetMinus(base, C('x', 0.0, 1.0)), 1)], p=[0.8, 0.2]), impossible=True))
  inner = distribs.Selection(C('c0', 0.0, 1.0), C('c0', 2.0, 3.0))
  out.append(Case('impossible_nested', gen.chain_generators(ok, gen.generate_sprites(
      distribs.Selection(P([inner, C('x', 0, 1)]), C('x', 0.0, 0.5)), 1)), [C('c0', 0, 1)], impossible=True))
  return out


# -- random programs -------------------------------------------------------------------------------


def _fits(v, dt):
  info = np.iinfo(dt)
  return info.min <= v <= info.max


def _exact_int(v, lo=-2 ** 63, hi=2 ** 64 - 1):
  """An integer near v that float64 holds exactly, within [lo, hi]."""
  v = int(float(min(max(int(v), lo), hi)))
  return v if lo <= v <= hi else int(np.nextafter(float(v), 0))


class _Random(object):
  """A seeded random scene generator over the package's combinators and distributions."""

  def __init__(self, seed):
    self.rng = np.random.RandomState(seed)
    self.hsv = self.rng.rand() < 0.5

  def pick(self, seq):
    return seq[self.rng.randint(len(seq))]

  def probs(self, n):
    p = self.rng.rand(n) * (self.rng.rand(n) < 0.7)
    if p.sum() == 0:
      p[self.rng.randint(n)] = 1.0
    return list(p / p.sum())

  def constant(self, v, weak_values=False):
    """v as a constant of a random kind: Python float or int, or a NumPy scalar.  Not float32
    against Python-scalar values (`weak_values`): in a scene whose column for the key mixes types
    those compare as weak scalars, in float32, and in a typed column as float64 or int64."""
    kind = self.pick(('float', 'int', 'float64') + ('float32',) * (not weak_values) + INT_DTYPES)
    if kind == 'float':
      return float(v)
    if kind in ('float32', 'float64'):
      return np.dtype(kind).type(v)
    if not np.isfinite(v):
      return float(v)
    if kind == 'int':
      return int(min(max(v, -2 ** 53), 2 ** 53))
    info = np.iinfo(kind)
    return np.dtype(kind).type(_exact_int(np.floor(v), int(info.min), int(info.max)))

  def int_range(self, dt):
    info = np.iinfo(dt)
    lo_max = min(int(info.max), 2 ** 63 - 1024 if dt == 'int64' else 2 ** 64 - 4096)
    m = self.rng.randint(4)
    if m == 0:
      lo = int(info.min) if self.rng.rand() < 0.5 else 0
      return lo, lo + self.rng.randint(1, 200)
    if m == 1:
      return int(info.min), _exact_int(int(info.min) + (lo_max - int(info.min)) * self.rng.rand() + 1)
    if m == 2:
      return _exact_int(int(info.min) + (lo_max - int(info.min)) * self.rng.rand()), lo_max + (lo_max == info.max)
    return int(info.min), lo_max + (lo_max == info.max)

  def leaf(self, key, color_dt):
    r = self.rng
    if key == 'shape':
      names = list(r.choice(SHAPES, r.randint(1, 5), replace=False))
      return D('shape', names, probs=self.probs(len(names)) if r.rand() < 0.4 else None)
    if key in ('c0', 'c1', 'c2') and color_dt is not None:
      t = np.dtype(color_dt).type
      if r.rand() < 0.6:
        lo = r.uniform(-0.6, 1.2)
        return C(key, lo, lo + r.uniform(0.05, 1.2), color_dt)
      vals = r.uniform(-0.6, 2.0, r.randint(1, 5))
      cands = [t(v) for v in vals] if color_dt == 'float32' else [self.pick((float, np.float64))(v) for v in vals]
      return D(key, cands, probs=self.probs(len(cands)) if r.rand() < 0.4 else None)
    if key == 'angle':
      if r.rand() < 0.5:
        dt = self.pick(INT_DTYPES)
        info = np.iinfo(dt)
        lo = max(int(info.min), -400) + r.randint(0, 300)
        return C('angle', lo, min(lo + r.randint(1, 200), int(info.max) + 1), dt)
      kind = self.pick(('float', 'int', 'float32') + INT_DTYPES)
      vals = [-0.0, 0.0, 45.0, -30.0, 90.0, 12.5, 200.0, 7.0]
      vals = [vals[i] for i in r.choice(len(vals), r.randint(1, 5), replace=False)]
      if kind in INT_DTYPES:
        vals = [abs(v) if kind[0] == 'u' else v for v in vals]
        cands = [np.dtype(kind).type(v) for v in vals if _fits(v, kind)] or [np.dtype(kind).type(7)]
      else:
        cands = [dict(float=float, int=lambda v: int(v), float32=np.float32)[kind](v) for v in vals]
      return D('angle', cands, probs=self.probs(len(cands)) if r.rand() < 0.3 else None)
    if r.rand() < 0.6:
      dt = self.pick(FLOAT_DTYPES + INT_DTYPES if key not in ('x', 'y') else FLOAT_DTYPES + INT_DTYPES[:7])
      if dt in FLOAT_DTYPES:
        lo = r.uniform(-1, 1) * 10.0 ** r.randint(0, 4 if key in ('x', 'y', 'scale') else 20)
        return C(key, lo, lo + abs(lo) * r.rand() + r.uniform(0.01, 2), dt)
      lo, hi = self.int_range(dt)
      return C(key, lo, hi, dt)
    kind = self.pick(('float', 'int', 'float32', 'float64') + INT_DTYPES if key not in ('x', 'y')
                     else ('float', 'float32', 'float64') + INT_DTYPES[:7])
    n = r.randint(1, 6)
    if kind == 'float':
      cands = list(r.uniform(-3, 3, n))
      cands = [float(v) for v in cands]
    elif kind == 'int':
      cands = [int(v) for v in r.randint(-2 ** 40, 2 ** 40, n)]
    elif kind in FLOAT_DTYPES:
      cands = [np.dtype(kind).type(v) for v in r.uniform(-1e3, 1e3, n)]
    else:
      info = np.iinfo(kind)
      cands = [np.dtype(kind).type(_exact_int(int(info.min) + (int(info.max) - int(info.min)) * r.rand(),
                                              int(info.min), int(info.max))) for _ in range(n)]
    return D(key, cands, probs=self.probs(n) if r.rand() < 0.4 else None)

  def values(self, d, n=48):
    """n host draws of d: dict key -> list of values."""
    w, stats = Words(self.rng.randint(1 << 30), 0, 0), dict(_new_stats(), limit=400)
    specs = [draw(d, w, stats) for _ in range(n)]
    return {k: [s[k] for s in specs] for k in d.keys}

  def predicate(self, key, vals, keep):
    """A distribution over `key` containing about a `keep` fraction of `vals`."""
    r = self.rng
    weak = any(not isinstance(v, np.generic) for v in vals)
    uniq = list({(type(v), v): v for v in vals}.values())
    if key == 'shape' or (len(uniq) <= 8 and r.rand() < 0.6):
      k = max(1, int(round(keep * len(uniq))))
      cands = [uniq[i] for i in r.choice(len(uniq), k, replace=False)]
      if key != 'shape':
        cands = [self.constant(float(v), weak) if r.rand() < 0.3 else v for v in cands]
      return D(key, cands)
    x = np.sort(np.array([float(v) for v in vals]))
    a = r.uniform(0, 1 - keep)
    lo, hi = x[int(a * (len(x) - 1))], x[min(len(x) - 1, int((a + keep) * (len(x) - 1)) + 1)]
    if r.rand() < 0.2:
      lo = -np.inf
    return C(key, self.constant(lo, weak), self.constant(np.nextafter(hi, np.inf) if hi == lo else hi, weak))

  def dist(self, keys, depth, color_dt):
    r = self.rng
    if len(keys) == 1 and (depth >= 3 or r.rand() < 0.5):
      return self.leaf(keys[0], color_dt)
    u = r.rand()
    if len(keys) > 1 and (u < 0.45 or depth >= 3):
      cut = sorted(r.choice(np.arange(1, len(keys)), min(len(keys) - 1, r.randint(1, 3)), replace=False))
      groups = np.split(np.array(keys), cut)
      return P([self.dist(list(g), depth + 1, color_dt) for g in groups])
    if u < 0.65:
      n = r.randint(2, 4)
      return distribs.Mixture([self.dist(keys, depth + 1, color_dt) for _ in range(n)], probs=self.probs(n))
    base = self.dist(keys, depth + 1, color_dt)
    vals = self.values(base)
    sub = [k for k in keys if r.rand() < 0.5] or [keys[0]]
    if u < 0.78 and len(keys) <= 3:
      other = P([self.predicate(k, vals[k], 0.85) for k in keys]) if len(keys) > 1 else self.predicate(keys[0], vals[keys[0]], 0.7)
      comps = [other, base] if r.rand() < 0.5 else [base, other]
      return distribs.Intersection(comps, index_for_sampling=comps.index(base))
    part = P([self.predicate(k, vals[k], 0.6) for k in sub]) if len(sub) > 1 else self.predicate(sub[0], vals[sub[0]], 0.6)
    if u < 0.9:
      return distribs.SetMinus(base, part)
    return distribs.Selection(base, part)

  def generator(self, depth, budget, leaves):
    r = self.rng
    u = r.rand()
    if depth >= 3 or u < 0.35 or budget < 4:
      keys = [k for k in FACTORS if r.rand() < 0.35]
      color_dt = None
      if self.hsv:
        color_dt = self.pick(FLOAT_DTYPES)
        keys = sorted(set(keys) | {'c0', 'c1', 'c2'}, key=FACTORS.index)
      keys = keys or [self.pick(FACTORS)]
      d = self.dist([str(k) for k in r.permutation(keys)], 0, color_dt)
      leaves.append(d)
      most = min(budget, r.randint(0, 7))
      if r.rand() < 0.5:
        lo = r.randint(0, most + 1)
        return gen.generate_sprites(d, gen.uniform_count(lo, r.randint(lo + 1, most + 2))), most + 1
      return gen.generate_sprites(d, most), most
    if u < 0.6:
      parts, total = [], 0
      for _ in range(r.randint(2, 4)):
        g, m = self.generator(depth + 1, (budget - total) // 2, leaves)
        parts.append(g)
        total += m
      return gen.chain_generators(*parts), total
    if u < 0.85:
      n = r.randint(2, 4)
      parts = [self.generator(depth + 1, budget, leaves) for _ in range(n)]
      p = self.probs(n) if r.rand() < 0.6 else None
      return gen.sample_generator([g for g, _ in parts], p=p), max(m for _, m in parts)
    g, m = self.generator(depth + 1, budget, leaves)
    return gen.shuffle(g), m

  def filters(self, leaves):
    r = self.rng
    pool = {k: [v] for k, v in DEFAULTS.items()}
    for d in leaves:
      for k, v in self.values(d, 24).items():
        pool[k] += v
    out = []
    for _ in range(r.randint(0, 9) if r.rand() < 0.8 else 32):
      k = self.pick(FACTORS)
      form = r.randint(6)
      if form == 0 and k != 'shape':
        k2 = self.pick([f for f in FACTORS if f != k])
        out.append(P([self.predicate(k, pool[k], 0.5), self.predicate(k2, pool[k2], 0.7)]))
      elif form == 1:
        out.append(distribs.Intersection([self.predicate(k, pool[k], 0.7), self.predicate(k, pool[k], 0.7)]))
      elif form == 2:
        out.append(distribs.Mixture([self.predicate(k, pool[k], 0.3), self.predicate(k, pool[k], 0.3)]))
      elif form == 3:
        out.append(distribs.SetMinus(self.predicate(k, pool[k], 0.8), self.predicate(k, pool[k], 0.3)))
      elif form == 4:
        out.append(distribs.Selection(self.predicate(k, pool[k], 0.8), self.predicate(k, pool[k], 0.5)))
      else:
        out.append(self.predicate(k, pool[k], 0.5))
    return out


N_RANDOM = 40


@functools.lru_cache(maxsize=None)
def random_case(i):
  """Random program i: the first draw from seed 1000 + i (and on) that compiles and whose
  rejection loops all accept within the CPU build's tries on the test's scenes."""
  for attempt in range(50):
    b = _Random(1000 + 97 * i + attempt)
    leaves = []
    try:
      g, _ = b.generator(0, 32, leaves)
      case = Case('random_%d' % i, g, b.filters(leaves), HSV if b.hsv else None)
    except (NotImplementedError, ValueError, RejectionFailed, _TooSlow):
      continue
    ids, idx = scene_ids(64)
    if scene_program.sample_on_host(case.program, SEEDS[0], ids, idx, 32)[1] is not None:
      continue
    try:   # the restatement draws in Python: keep its rejection loops short
      restate(case, SEEDS[0], ids[:6], idx[:6], 32, dict(_new_stats(), limit=150))
    except _TooSlow:
      continue
    return case
  raise AssertionError('no program for random case %d' % i)


@functools.lru_cache(maxsize=None)
def edge_cases():
  return {c.name: c for c in _edge_cases()}


CASE_NAMES = ['random_%d' % i for i in range(N_RANDOM)] + [c.name for c in _edge_cases()]


def case(name):
  return random_case(int(name.split('_')[1])) if name.startswith('random_') else edge_cases()[name]


_STATS = {}


@functools.lru_cache(maxsize=None)
def host_and_restatement(name, seed):
  """(sample_on_host, restate) of the test's scenes with `seed` (impossible programs: the
  restatement stops after its first failing scene)."""
  c = case(name)
  ids, idx = scene_ids(64)
  S = max(1, c.program.max_sprites)
  got = scene_program.sample_on_host(c.program, seed, ids, idx, S)
  stats = _STATS.setdefault(name, _new_stats())
  want = restate(c, seed, ids, idx, S, stats, stop_at_failure=c.impossible)
  return got, want


# -- the tests -------------------------------------------------------------------------------------


def test_words_equal_philox_host():
  for g, a in ((0, 0), (0, 1), (2 ** 63 - 1, 0), (5, 2 ** 63 - 1), (2 ** 62, 2 ** 62 + 3)):
    w = Words(99, g, a)
    for block in range(3):
      ref = scene_program.philox_host([block, a, g, 0], [99, DOMAIN])
      assert [w.next() for _ in range(4)] == [int(v) for v in ref], (g, a, block)


@pytest.mark.parametrize('name', CASE_NAMES)
@pytest.mark.parametrize("seed", SEEDS[:1])
def test_cpu_build_equals_numpy_restatement(name, seed):
  c = case(name)
  (got, got_fail), (want, want_fail) = host_and_restatement(name, seed)
  if c.impossible:
    assert got_fail is not None and want_fail is not None
    i, dist = want_fail
    assert got_fail[0] == i and c.program.describe(got_fail[1]) == str(dist)
    got = {k: v[:i + 1] for k, v in got.items()}
  else:
    assert got_fail is None and want_fail is None
  assert_same(got, want, name)


def _ops(prog):
  p = prog.struct
  return [p.ops[i] for i in range(p.n_ops)]


def test_sweep_covers_every_op_kind_and_edge():
  names = CASE_NAMES
  ops, draw_kinds, const_kinds, modes = set(), set(), set(), set()
  for n in names:
    prog = case(n).program
    modes.add(prog.struct.color_mode)
    for o in _ops(prog):
      ops.add(o.op)
      if o.op in (scene_program.D_CONT, scene_program.D_DISC):
        draw_kinds.add(o.dtype)
      if o.op == scene_program.P_CONT:
        const_kinds |= {o.a, o.b}
      if o.op == scene_program.P_DISC:
        const_kinds |= {prog.struct.const_kind[o.a + j] for j in range(o.b)}
  assert ops == set(OPS), sorted(set(OPS) - ops)
  assert draw_kinds >= set(range(1, 12)), sorted(set(range(1, 12)) - draw_kinds)
  assert const_kinds >= set(range(1, 14)), sorted(set(range(1, 14)) - const_kinds)
  assert modes == {scene_program.COLOR_RGB, scene_program.COLOR_HSV}
  # the edges were reached in the drawn scenes
  for n in names:
    host_and_restatement(n, SEEDS[0])
  total = lambda k: sum(s[k] for s in _STATS.values())  # noqa: E731
  assert total('retries') > 1000 and total('neg_hsv') > 100 and total('hsv_over_int32') > 10
  sprites = [k for s in _STATS.values() for k in s['sprites']]
  assert 0 in sprites and 32 in sprites
  u64_high = member31 = rgb_1e19 = 0
  for n in names:
    (got, _), _ = host_and_restatement(n, SEEDS[0])
    if True:
      u64_high += int(((got['factor_kind'] == FT[np.uint64]) & (got['factor_value'] >= 2.0 ** 63)).sum())
      member31 += int((got['member'] >> 31).sum())
      if n == 'rgb_float_1e19':
        rgb_1e19 += int((np.abs(got['factor_value'][..., 5:8]) >= 2.0 ** 63).sum())
  assert u64_high > 100 and member31 > 10 and rgb_1e19 > 100
  assert any(case(n).program.max_sprites == 32 for n in names)


def test_integer_constants_float64_cannot_hold_are_refused():
  g = gen.generate_sprites(C('c0', 0, 2 ** 64 - 4096, 'uint64'), 1)
  for bad in (np.uint64(2 ** 63 + 1), np.int64(2 ** 62 + 1), np.int64(-2 ** 60 - 3)):
    with pytest.raises(NotImplementedError, match='float64'):
      scene_program.compile_program(g, [C('c0', bad, 2 ** 53)])
    with pytest.raises(NotImplementedError, match='float64'):
      scene_program.compile_program(gen.generate_sprites(D('c0', [bad]), 1))
  scene_program.compile_program(g, [C('c0', np.uint64(2 ** 63 + 2 ** 11), np.int64(-2 ** 62))])
