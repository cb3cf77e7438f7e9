"""Scene generators compiled for the device sampler.

`compile_program(init_sprites, filters, color_to_rgb)` flattens a scene generator -- the
combinators of sprite_generators.py over the distributions of factor_distributions.py -- into the
POD `swb_scene_program` of include/spriteworld_b200.h, the way tasks.compile() flattens a task
tree.  The device runs it one scene per thread (csrc/swb_sampler.cuh): scene `a` of global env `g`
is a pure function of (seed, g, a), drawn from Philox4x64-10 with the same distribution as the
host sampler draws it, and packed exactly as scene.arrays_from_layout packs the same factors.

What does not compile raises NotImplementedError naming the part: plain callables (a lambda
sprite count: use sprite_generators.uniform_count), colour maps other than None and
color_maps.hsv_to_rgb, colour triples of mixed dtypes, angles drawn from a float Continuous (the
transform's cos / sin come from a host table over the finite angle set), and programs beyond the
header's size limits.

`sample_on_host` runs the same sampler source built for the CPU (libswb_sampler_host.so): the
restatement the device is tested against, and a way to draw the device's scenes without a GPU.
`sample_contained_on_host` is the same for the contained-position sampler (swb_contained.cuh).
"""
import ctypes
import math
import os

import numpy as np

from spriteworld_b200 import constants
from spriteworld_b200 import factor_distributions as fd
from spriteworld_b200 import scene as scene_lib
from spriteworld_b200 import sprite_generators as gen

MAX_OPS, MAX_CONSTS, MAX_ANGLES, MAX_STACK, MAX_FILTERS, MAX_SLOTS = 512, 1024, 1024, 16, 32, 32
MAX_GOALS = 8   # SWB_MAX_GOALS
DOMAIN = 0x53574253434e4531   # SWB_SAMPLER_DOMAIN: second Philox key word of the scene stream

FT_NONE, FT_F32, FT_F64 = 0, 1, 2
FT_SHAPE, FT_PYFLOAT, FT_PYINT = 11, 12, 13
_NP_KINDS = {np.dtype(np.float32): 1, np.dtype(np.float64): 2, np.dtype(np.int8): 3,
             np.dtype(np.int16): 4, np.dtype(np.int32): 5, np.dtype(np.int64): 6,
             np.dtype(np.uint8): 7, np.dtype(np.uint16): 8, np.dtype(np.uint32): 9,
             np.dtype(np.uint64): 10}
KIND_DTYPES = {k: d for d, k in _NP_KINDS.items()}
_INT_KINDS = set(range(3, 11))

(G_END, G_SPRITES, G_MARK, G_SHUFFLE, G_CHOOSE, G_JUMP) = range(6)
(D_RET, D_CONT, D_DISC, D_MIX, D_JUMP, D_REJ_BEGIN, D_REJ_END) = range(10, 17)
(P_RET, P_CONT, P_DISC, P_AND, P_OR, P_NOT) = range(20, 26)
COLOR_RGB, COLOR_HSV = 0, 1
FACTORS = ('x', 'y', 'shape', 'angle', 'scale', 'c0', 'c1', 'c2', 'x_vel', 'y_vel')
_KEY = {name: i for i, name in enumerate(FACTORS)}
# kinds of the Sprite.__init__ defaults as scene._default_column types them
_DEFAULT_KINDS = dict(x=FT_F64, y=FT_F64, shape=FT_SHAPE, angle=6, scale=FT_F64, c0=6, c1=6, c2=6,
                      x_vel=FT_F64, y_vel=FT_F64)

_c32, _f64 = ctypes.c_int32, ctypes.c_double


class ProgOp(ctypes.Structure):
  _fields_ = [('op', _c32), ('key', _c32), ('dtype', _c32), ('a', _c32), ('b', _c32), ('c', _c32),
              ('lo', _f64), ('hi', _f64)]


class Program(ctypes.Structure):
  _fields_ = [('n_ops', _c32), ('n_consts', _c32), ('n_angles', _c32), ('n_filters', _c32),
              ('max_sprites', _c32), ('color_mode', _c32), ('filter_pc', _c32 * MAX_FILTERS),
              ('ops', ProgOp * MAX_OPS), ('consts', _f64 * MAX_CONSTS), ('const_kind', _c32 * MAX_CONSTS),
              ('angle', _f64 * MAX_ANGLES), ('angle_cos', _f64 * MAX_ANGLES),
              ('angle_sin', _f64 * MAX_ANGLES), ('n_goals', _c32), ('goal_pc', _c32 * MAX_GOALS)]


class SampleOut(ctypes.Structure):
  _fields_ = [(n, ctypes.c_void_p) for n in
              ('x', 'y', 'm00', 'm01', 'm10', 'm11', 'vx', 'vy', 'member', 'shape', 'pos_f32', 'rgb',
               'factors', 'factor_value', 'factor_kind', 'goal')]


class FactorColumns(ctypes.Structure):
  """swb_factor_columns: a pointer and an SWB_FT_* kind per factor (NULL: Sprite's default)."""
  _fields_ = [('col', ctypes.c_void_p * len(FACTORS)), ('kind', _c32 * len(FACTORS))]


# the dtypes a factor column of swb_make_states may have, and their SWB_FT_* kinds
MAKE_KINDS = {np.dtype(t): _NP_KINDS[np.dtype(t)]
              for t in (np.float32, np.float64, np.int8, np.int16, np.int32, np.int64, np.uint8)}
MAKE_ANGLE, MAKE_SHAPE, MAKE_HOLE, MAKE_INT, MAKE_STEP = 1, 2, 4, 8, 16   # SWB_MAKE_*


class SceneProgram(object):
  """A compiled scene generator: `struct` (the ctypes swb_scene_program), `max_sprites`, and
  `describe(op)`, the distribution a rejection loop draws from (for the reference's error)."""

  def __init__(self, struct, max_sprites, rejections):
    self.struct = struct
    self.max_sprites = max_sprites
    self._rejections = rejections

  def describe(self, op):
    return self._rejections.get(int(op), 'op %d' % int(op))

  def error(self, op):
    """The reference's ValueError for a rejection loop that ran out of tries."""
    return ValueError('Maximum number of tried exceeded when trying to sample from {}.'.format(
        self.describe(op)))


def _refuse(what):
  raise NotImplementedError('the device sampler cannot compile %s' % what)


def _const_kind(v, what):
  """Kind of a bound or candidate as NumPy compares it (Python scalars are weak, NEP 50)."""
  if isinstance(v, (bool, np.bool_)):
    _refuse('boolean %s %r' % (what, v))
  if isinstance(v, np.generic):
    kind = _NP_KINDS.get(v.dtype)
    if kind is None:
      _refuse('%s %r of dtype %s' % (what, v, v.dtype))
    if kind in _INT_KINDS and int(float(v)) != int(v):
      _refuse('%s %r: an integer float64 cannot hold exactly (the sampler compares in float64)'
              % (what, v))
    return kind
  if isinstance(v, float):
    return FT_PYFLOAT
  if isinstance(v, int):
    if abs(v) > 2 ** 53:
      _refuse('%s %r beyond 2**53' % (what, v))
    return FT_PYINT
  _refuse('%s %r of type %s' % (what, v, type(v).__name__))


def _key(k):
  if k not in _KEY:
    _refuse('factor %r (factors are %s)' % (k, ', '.join(FACTORS)))
  return _KEY[k]


def _cdf(p):
  """np.random.choice's table: cumsum, divided by its last entry."""
  cdf = np.cumsum(np.array(p, dtype=np.double))
  cdf /= cdf[-1]
  return cdf


class _Compiler(object):

  def __init__(self):
    self.ops, self.consts, self.kinds = [], [], []
    self.pending_dist, self.pending_pred = [], []
    self.pred_pc = {}   # op of each distribution's predicate code, by id
    self.angles = {}   # angle values by bit pattern (0.0 and -0.0 are distinct)
    self.angle(0.0)    # the default angle 0
    self.rejections = {}

  def op(self, op, key=0, dtype=0, a=0, b=0, c=0, lo=0.0, hi=0.0):
    self.ops.append(dict(op=op, key=key, dtype=dtype, a=a, b=b, c=c, lo=float(lo), hi=float(hi)))
    return len(self.ops) - 1

  def angle(self, v):
    v = float(v)
    self.angles[np.float64(v).tobytes()] = v

  def const(self, values, kinds):
    off = len(self.consts)
    self.consts.extend(float(v) for v in values)
    self.kinds.extend(kinds)
    return off

  # -- generators ------------------------------------------------------------------------
  def gen(self, g):
    spec = getattr(g, '_spec', None)
    if spec is None:
      _refuse('the sprite generator %r: plain callables run on the host only; compose '
              'generate_sprites / chain_generators / sample_generator / shuffle' % (g,))
    kind = spec[0]
    if kind == 'sprites':
      _, dist, num = spec
      if isinstance(num, gen.uniform_count):
        i = self.op(G_SPRITES, dtype=1, b=num.lo, c=num.hi)
        most = num.hi - 1
      elif callable(num):
        _refuse('the sprite count %r: a callable count runs on the host only; use '
                'sprite_generators.uniform_count(lo, hi) for np.random.randint(lo, hi)' % (num,))
      else:
        i = self.op(G_SPRITES, b=int(num))
        most = int(num)
      self.pending_dist.append((i, dist))
      return most
    if kind == 'chain':
      return sum(self.gen(child) for child in spec[1])
    if kind == 'sample':
      _, children, p = spec
      n = len(children)
      self.op(G_CHOOSE, b=n, c=self.const(_cdf(np.ones(n) / n if p is None else p), [FT_F64] * n))
      jumps = [self.op(G_JUMP) for _ in range(n)]
      ends, most = [], 0
      for j, child in zip(jumps, children):
        self.ops[j]['a'] = len(self.ops)
        most = max(most, self.gen(child))
        ends.append(self.op(G_JUMP))
      for e in ends:
        self.ops[e]['a'] = len(self.ops)
      return most
    if kind == 'shuffle':
      self.op(G_MARK)
      most = self.gen(spec[1])
      self.op(G_SHUFFLE)
      return most
    _refuse('generator kind %r' % kind)

  # -- distributions (sampling) ----------------------------------------------------------
  def dist(self, d):
    if isinstance(d, fd.Continuous):
      key = _key(d.key)
      dt = np.dtype(d.dtype)
      kind = _NP_KINDS.get(dt)
      if kind is None:
        _refuse('Continuous(%r) of dtype %s' % (d.key, dt))
      lo, hi = float(d.minval), float(d.maxval)
      if kind in _INT_KINDS:
        info = np.iinfo(dt)
        # draws lie in [lo, hi): the largest truncates to ceil(hi) - 1
        if not (info.min <= math.trunc(lo) and math.ceil(hi) - 1 <= info.max):
          _refuse('Continuous(%r, %r, %r, dtype=%s): the range does not fit the dtype'
                  % (d.key, d.minval, d.maxval, dt))
      if d.key == 'angle':
        if kind not in _INT_KINDS:
          _refuse('angle drawn from a float Continuous: angles must come from a finite set '
                  '(an integer dtype, a Discrete, or the default 0)')
        if math.trunc(hi) - math.trunc(lo) + 1 > MAX_ANGLES:
          _refuse('an angle range of more than %d values' % MAX_ANGLES)
        for v in range(math.trunc(lo), math.trunc(hi) + 1):   # hi too: a draw can round up to it
          self.angle(v)
      self.op(D_CONT, key=key, dtype=kind, lo=lo, hi=hi)
    elif isinstance(d, fd.Discrete):
      key = _key(d.key)
      kind, values = self._candidates(d)
      if d.key == 'angle':
        for v in values:
          self.angle(v)
      off = self.const(values, [kind] * len(values))
      cdf = -1 if d.probs is None else self.const(_cdf(d.probs), [FT_F64] * len(values))
      self.op(D_DISC, key=key, dtype=kind, a=off, b=len(values), c=cdf)
    elif isinstance(d, fd.Product):
      for c in d.components:
        self.dist(c)
    elif isinstance(d, fd.Mixture):
      n = len(d.components)
      self.op(D_MIX, b=n, c=self.const(_cdf(d.probs), [FT_F64] * n))
      jumps = [self.op(D_JUMP) for _ in range(n)]
      ends = []
      for j, c in zip(jumps, d.components):
        self.ops[j]['a'] = len(self.ops)
        self.dist(c)
        ends.append(self.op(D_JUMP))
      for e in ends:
        self.ops[e]['a'] = len(self.ops)
    elif isinstance(d, (fd.Intersection, fd.SetMinus, fd.Selection)):
      self.op(D_REJ_BEGIN)
      if isinstance(d, fd.Intersection):
        self.dist(d.components[d.index_for_sampling])
        pred, keep = d, 1
      else:
        self.dist(d.base)
        pred, keep = d._other, int(d._keep_if_inside)
      i = self.op(D_REJ_END, b=keep)
      self.pending_pred.append((i, pred))
      self.rejections[i] = str(d)
    else:
      _refuse('the distribution %s' % type(d).__name__)

  def _candidates(self, d):
    """(kind of the drawn column, values) of a Discrete, typed as factor_distributions._as_column
    types its candidates."""
    cands = list(d.candidates)
    if not cands:
      _refuse('an empty Discrete(%r)' % d.key)
    if all(isinstance(v, str) for v in cands):
      if d.key != 'shape':
        _refuse('names as values of factor %r' % d.key)
      bad = [v for v in cands if v not in constants.SHAPE_NAMES]
      if bad:
        _refuse('shape names %s' % bad)
      return FT_SHAPE, [int(constants.ShapeType[v]) for v in cands]
    if d.key == 'shape':
      _refuse('shape values that are not shape names: %r' % (cands,))
    types = set(type(v) for v in cands)
    if types <= {float, np.float64}:
      kind = FT_F64
    elif types <= {int, np.int64}:
      kind = _NP_KINDS[np.dtype(np.int64)]
    elif len(types) == 1 and issubclass(next(iter(types)), np.generic):
      kind = _NP_KINDS.get(np.dtype(next(iter(types))))
      if kind is None:
        _refuse('Discrete(%r) candidates of dtype %s' % (d.key, np.dtype(next(iter(types)))))
    else:
      _refuse('Discrete(%r) with candidates of mixed types %s' % (d.key, sorted(t.__name__ for t in types)))
    for v in cands:
      _const_kind(v, 'candidate')
    return kind, [float(v) for v in cands]

  # -- predicates (containment) ------------------------------------------------------------
  def predicate(self, d):
    """Op index of the predicate code of `d` (containment), emitted once per distribution object."""
    if id(d) not in self.pred_pc:
      if _stack_depth(d) > MAX_STACK:
        _refuse('a containment test nested more than %d deep' % MAX_STACK)
      self.pred_pc[id(d)] = len(self.ops)
      self.pred(d)
      self.op(P_RET)
    return self.pred_pc[id(d)]

  def pred(self, d):
    if isinstance(d, fd.Continuous):
      self.op(P_CONT, key=_key(d.key), a=_const_kind(d.minval, 'bound'), b=_const_kind(d.maxval, 'bound'),
              lo=float(d.minval), hi=float(d.maxval))
    elif isinstance(d, fd.Discrete):
      values, kinds = [], []
      for v in d.candidates:
        if isinstance(v, str):
          values.append(int(constants.ShapeType[v]) if v in constants.SHAPE_NAMES else -1)
          kinds.append(FT_SHAPE)
        else:
          values.append(float(v))
          kinds.append(_const_kind(v, 'candidate'))
      if not values:
        _refuse('an empty Discrete(%r)' % d.key)
      self.op(P_DISC, key=_key(d.key), a=self.const(values, kinds), b=len(values))
    elif isinstance(d, (fd.Product, fd.Intersection, fd.Mixture)):
      join = P_OR if isinstance(d, fd.Mixture) else P_AND
      for i, c in enumerate(d.components):
        self.pred(c)
        if i:
          self.op(join, b=2)
    elif isinstance(d, fd.SetMinus):
      self.pred(d.base)
      self.pred(d.hold_out)
      self.op(P_NOT)
      self.op(P_AND, b=2)
    elif isinstance(d, fd.Selection):
      self.pred(d.base)
      self.pred(d.filtering)
      self.op(P_AND, b=2)
    else:
      _refuse('containment in %s' % type(d).__name__)


def _stack_depth(d):
  if isinstance(d, (fd.Product, fd.Intersection, fd.Mixture)):
    return max([_stack_depth(d.components[0])] + [1 + _stack_depth(c) for c in d.components[1:]])
  if isinstance(d, fd.SetMinus):
    return max(_stack_depth(d.base), 1 + _stack_depth(d.hold_out))
  if isinstance(d, fd.Selection):
    return max(_stack_depth(d.base), 1 + _stack_depth(d.filtering))
  return 1


def _rejection_depth(d):
  if isinstance(d, (fd.Product, fd.Mixture)):
    return max(_rejection_depth(c) for c in d.components)
  if isinstance(d, fd.Intersection):
    return 1 + _rejection_depth(d.components[d.index_for_sampling])
  if isinstance(d, (fd.SetMinus, fd.Selection)):
    return 1 + _rejection_depth(d.base)
  return 0


def _key_kinds(d):
  """dict factor -> set of kinds a sprite drawn from `d` can have."""
  if isinstance(d, fd.Continuous):
    return {d.key: {_NP_KINDS.get(np.dtype(d.dtype))}}
  if isinstance(d, fd.Discrete):
    return {d.key: {_Compiler()._candidates(d)[0]}}
  if isinstance(d, fd.Intersection):
    return _key_kinds(d.components[d.index_for_sampling])
  if isinstance(d, (fd.SetMinus, fd.Selection)):
    return _key_kinds(d.base)
  out = {}
  for c in d.components:
    for k, v in _key_kinds(c).items():
      out.setdefault(k, set()).update(v)
  return out


def _leaf_dists(g):
  spec = getattr(g, '_spec', None)
  if spec is None:
    return []
  if spec[0] == 'sprites':
    return [spec[1]]
  if spec[0] in ('chain', 'sample'):
    return [d for child in spec[1] for d in _leaf_dists(child)]
  return _leaf_dists(spec[1])


def _generator_depth(g):
  spec = getattr(g, '_spec', None)
  if spec is None or spec[0] == 'sprites':
    return 0
  if spec[0] == 'shuffle':
    return 1 + _generator_depth(spec[1])
  return max([_generator_depth(c) for c in spec[1]] + [0])


def compile_program(init_sprites, filters=(), color_to_rgb=None, goals=()):
  """SceneProgram of a scene generator, the task's filter distributions (bit i of `member` is
  filters[i]), the PILRenderers' colour map and the task's goal distributions (goal slot i is drawn
  by goals[i], after the scene's sprites; tasks.AbstractTask.goal_distributions)."""
  color_mode = _color_mode(color_to_rgb, filters)
  if len(goals) > MAX_GOALS:
    _refuse('more than %d sampled goals' % MAX_GOALS)
  for d in goals:
    if set(d.keys) != {'x', 'y'}:
      _refuse("a goal distribution over %s (it must be over exactly {'x', 'y'})" % sorted(d.keys))
    if _rejection_depth(d) > MAX_STACK:
      _refuse('rejection samplers nested more than %d deep' % MAX_STACK)
  c = _Compiler()
  most = c.gen(init_sprites)
  c.op(G_END)
  if most > MAX_SLOTS:
    _refuse('scenes of up to %d sprites (the engine has at most %d slots)' % (most, MAX_SLOTS))
  if _generator_depth(init_sprites) > MAX_STACK:
    _refuse('shuffles nested more than %d deep' % MAX_STACK)
  for dist in _leaf_dists(init_sprites):
    kinds = {k: _key_kinds(dist).get(k, {_DEFAULT_KINDS[k]}) for k in FACTORS if k in _DEFAULT_KINDS}
    if kinds['shape'] != {FT_SHAPE}:
      _refuse('shape values that are not shape names')
    if color_mode == COLOR_HSV:
      triple = [kinds[k] for k in ('c0', 'c1', 'c2')]
      if not (all(t == {FT_F32} for t in triple) or all(t == {FT_F64} for t in triple)):
        _refuse('colour factors (c0, c1, c2) of mixed or integer dtypes %s under hsv_to_rgb: the '
                'three must all be float32 or all float64' % [sorted(t) for t in triple])
    if _rejection_depth(dist) > MAX_STACK:
      _refuse('rejection samplers nested more than %d deep' % MAX_STACK)
  # distribution code, then predicate code
  done = {}
  for i, dist in c.pending_dist:
    if id(dist) not in done:
      done[id(dist)] = len(c.ops)
      c.dist(dist)
      c.op(D_RET)
    c.ops[i]['a'] = done[id(dist)]
  goal_pcs = []
  for dist in goals:
    if id(dist) not in done:
      done[id(dist)] = len(c.ops)
      c.dist(dist)
      c.op(D_RET)
    goal_pcs.append(done[id(dist)])
  for i, d in c.pending_pred:
    c.ops[i]['a'] = c.predicate(d)
  filter_pcs = [c.predicate(f) for f in filters]
  return SceneProgram(_program_struct(c, most, color_mode, filter_pcs, goal_pcs), most, c.rejections)


def _color_mode(color_to_rgb, filters):
  """COLOR_RGB or COLOR_HSV of a PILRenderer colour map; refuses other maps and too many filters."""
  from spriteworld_b200.renderers import color_maps
  if color_to_rgb is None:
    mode = COLOR_RGB
  elif color_to_rgb is color_maps.hsv_to_rgb:
    mode = COLOR_HSV
  else:
    _refuse('the colour map %r: only None (RGB colours) and color_maps.hsv_to_rgb' % (color_to_rgb,))
  if len(filters) > MAX_FILTERS:
    _refuse('more than %d task filters' % MAX_FILTERS)
  return mode


def _program_struct(c, most, color_mode, filter_pcs, goal_pcs):
  """The swb_scene_program of compiler `c`'s code, constants and angles."""
  if len(c.ops) > MAX_OPS or len(c.consts) > MAX_CONSTS or len(c.angles) > MAX_ANGLES:
    _refuse('a program of %d ops, %d constants and %d angles (limits %d, %d, %d)'
            % (len(c.ops), len(c.consts), len(c.angles), MAX_OPS, MAX_CONSTS, MAX_ANGLES))
  p = Program()
  p.n_ops, p.n_consts, p.n_filters = len(c.ops), len(c.consts), len(filter_pcs)
  p.max_sprites, p.color_mode = most, color_mode
  for i, pc in enumerate(filter_pcs):
    p.filter_pc[i] = pc
  p.n_goals = len(goal_pcs)
  for i, pc in enumerate(goal_pcs):
    p.goal_pc[i] = pc
  for i, o in enumerate(c.ops):
    for k, v in o.items():
      setattr(p.ops[i], k, v)
  for i, (v, k) in enumerate(zip(c.consts, c.kinds)):
    p.consts[i], p.const_kind[i] = v, k
  # angles ascending, -0.0 before 0.0; cos / sin as scene.transform_matrix takes them
  angles = sorted(c.angles.values(), key=lambda a: (a, not math.copysign(1.0, a) < 0))
  p.n_angles = len(angles)
  for i, a in enumerate(angles):
    th = math.radians(a)
    p.angle[i], p.angle_cos[i], p.angle_sin[i] = a, math.cos(th), math.sin(th)
  return p


PACKER_ANGLES = tuple(range(-360, 361))   # the integer angles a packer takes (and -0.0)


def compile_packer(filters=(), color_to_rgb=None):
  """SceneProgram of the packer of Engine.make_states: no generator (its code is a lone G_END), the
  task's filter distributions (bit i of `member` is filters[i]) as compile_program compiles them,
  the colour map's mode, and the angle table of every integer angle in [-360, 360] and -0.0 (libm's
  cos / sin of their radians, as scene.transform_matrix takes them).  NotImplementedError for a
  colour map other than None and color_maps.hsv_to_rgb, more than MAX_FILTERS filters, or a filter
  compile_program refuses."""
  color_mode = _color_mode(color_to_rgb, filters)
  c = _Compiler()
  c.op(G_END)
  for a in PACKER_ANGLES + (-0.0,):
    c.angle(a)
  filter_pcs = [c.predicate(f) for f in filters]
  return SceneProgram(_program_struct(c, 0, color_mode, filter_pcs, []), 0, {})


# -- the CPU build of the sampler ----------------------------------------------------------

_host = None


def _host_lib():
  global _host
  if _host is None:
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'csrc', 'libswb_sampler_host.so')
    if not os.path.exists(path):
      raise RuntimeError('%s is missing: build it with `python -m spriteworld_b200.build`' % path)
    L = ctypes.CDLL(path)
    vp = ctypes.c_void_p
    L.swb_host_philox.argtypes = [vp, ctypes.c_uint64, ctypes.c_uint64, vp]
    L.swb_host_philox.restype = None
    L.swb_host_sample_scenes.argtypes = [vp, ctypes.c_uint64, ctypes.c_int32, vp, vp, ctypes.c_int64,
                                         vp, vp, vp]
    L.swb_host_sample_scenes.restype = ctypes.c_int64
    L.swb_host_sample_contained.argtypes = [vp] * 7 + [ctypes.c_int32, ctypes.c_int32, vp, vp, ctypes.c_int32,
                                                        ctypes.c_uint64, vp, vp, vp]
    L.swb_host_sample_contained.restype = None
    L.swb_host_make_states.argtypes = [vp, vp, ctypes.c_int32, ctypes.c_int32, ctypes.c_int32, vp, vp, vp,
                                       ctypes.c_uint64, vp, vp]
    L.swb_host_make_states.restype = None
    if L.swb_host_sampler_sizeof_program() != ctypes.sizeof(Program):
      raise RuntimeError('ABI mismatch: swb_scene_program')
    _host = L
  return _host


def philox_host(counter, key):
  """Philox4x64-10 of one counter block (4 uint64 words) under a 2-word key."""
  ctr = np.ascontiguousarray(counter, np.uint64)
  out = np.zeros(4, np.uint64)
  _host_lib().swb_host_philox(ctr.ctypes.data, int(key[0]), int(key[1]), out.ctypes.data)
  return out


def empty_sample(n, n_slots, n_goals=0):
  """Host arrays of swb_sample_out for n scenes: a scene batch plus the drawn factor table and,
  for n_goals > 0, the goals (n, n_goals, 2)."""
  b = scene_lib.empty_batch(n, n_slots)
  if n_goals:
    b['goal'] = np.zeros((n, n_goals, 2), np.float64)
  b['factor_value'] = np.zeros((n, n_slots, len(FACTORS)), np.float64)
  b['factor_kind'] = np.zeros((n, n_slots, len(FACTORS)), np.uint8)
  return b


def sample_out_struct(arrays, ptr=lambda a: a.ctypes.data):
  out = SampleOut()
  for name, _ in SampleOut._fields_:
    setattr(out, name, ptr(arrays[name]) if name in arrays else None)   # goal: optional
  return out


def sample_on_host(program, seed, env_ids, scene_idx, n_slots):
  """Scenes (env_ids[i], scene_idx[i]) as the device samples them, drawn on the CPU.  Returns
  (arrays of empty_sample, index of the first scene whose rejection loop ran out of tries, and
  its op; or None)."""
  env_ids = np.ascontiguousarray(env_ids, np.int64)
  scene_idx = np.ascontiguousarray(scene_idx, np.int64)
  n = len(env_ids)
  b = empty_sample(n, n_slots, program.struct.n_goals)
  op, idx = ctypes.c_int32(-1), ctypes.c_int64(-1)
  failures = _host_lib().swb_host_sample_scenes(
      ctypes.byref(program.struct), int(seed) & (2 ** 64 - 1), int(n_slots), env_ids.ctypes.data,
      scene_idx.ctypes.data, n, ctypes.byref(sample_out_struct(b)), ctypes.byref(op), ctypes.byref(idx))
  return b, ((int(idx.value), int(op.value)) if failures else None)


def make_states_on_host(packer, columns, n_slots, n_goals=0, goals=None, step_count=None):
  """swb_make_states on the CPU, built from the kernel's own source (swb_make_states.cuh): `columns`
  is a dict factor name -> (n, S) array of a MAKE_KINDS dtype ('shape' required; a missing factor
  takes Sprite's default), goals float64 (n, n_goals, 2), step_count int32 (n,) or None for zeros.
  Returns (records uint8 (n, record bytes), status uint8 (n,), span flag: True if an accepted record
  holds a star or spoke)."""
  from spriteworld_b200 import engine
  shape = np.asarray(columns['shape'])
  n, S = shape.shape
  assert S == n_slots, (S, n_slots)
  cols, keep = FactorColumns(), []
  for f, name in enumerate(FACTORS):
    if name in columns:
      a = np.ascontiguousarray(columns[name])
      assert a.shape == (n, S) and a.dtype in MAKE_KINDS, (name, a.shape, a.dtype)
      keep.append(a)
      cols.col[f], cols.kind[f] = a.ctypes.data, MAKE_KINDS[a.dtype]
  _, rb = engine.record_layout(S, n_goals)
  records = np.zeros((n, rb), np.uint8)
  status = np.zeros(n, np.uint8)
  flag = np.zeros(1, np.uint8)
  g = None if not n_goals else np.ascontiguousarray(goals, np.float64).reshape(n, n_goals, 2)
  sc = None if step_count is None else np.ascontiguousarray(step_count, np.int32).reshape(n)
  _host_lib().swb_host_make_states(
      ctypes.byref(packer.struct), ctypes.byref(cols), n, S, int(n_goals), None if g is None else g.ctypes.data,
      None if sc is None else sc.ctypes.data, records.ctypes.data, rb, status.ctypes.data, flag.ctypes.data)
  return records, status, bool(flag[0])


def shape_table(shapes=None):
  """(verts float64 (13, 32, 2), n_verts int32 (13,)): the engine's shape table (swb_config) of
  `shapes` (default constants.SHAPES), indexed by ShapeType id."""
  shapes = constants.SHAPES if shapes is None else shapes
  verts = np.zeros((len(constants.SHAPE_NAMES) + 1, 32, 2), np.float64)
  n_verts = np.zeros(len(constants.SHAPE_NAMES) + 1, np.int32)
  for sid, name in enumerate(constants.SHAPE_NAMES, 1):
    v = np.asarray(shapes[name], np.float64)
    verts[sid, :len(v)], n_verts[sid] = v, len(v)
  return verts, n_verts


def sample_contained_on_host(rows, seed, n_samples=1, shapes=None):
  """swb_sample_contained on the CPU, built from the kernel's own source (swb_contained.cuh):
  `rows` is a dict of (n, S) arrays x, y (live positions), m00, m01, m10, m11 and shape (raw ids,
  sanitised as a record load sanitises them).  Returns (position float64 (n, n_samples, 2), slot
  int8 (n, n_samples), status uint8 (n, n_samples)), what the device returns for those rows."""
  f64 = {k: np.ascontiguousarray(rows[k], np.float64) for k in ('x', 'y', 'm00', 'm01', 'm10', 'm11')}
  shape = np.ascontiguousarray(rows['shape'], np.uint8)
  n, S = shape.shape
  verts, n_verts = shape_table(shapes)
  position = np.zeros((n, n_samples, 2), np.float64)
  slot = np.zeros((n, n_samples), np.int8)
  status = np.zeros((n, n_samples), np.uint8)
  _host_lib().swb_host_sample_contained(
      *[f64[k].ctypes.data for k in ('x', 'y', 'm00', 'm01', 'm10', 'm11')], shape.ctypes.data, n, S,
      verts.ctypes.data, n_verts.ctypes.data, int(n_samples), int(seed) & (2 ** 64 - 1), position.ctypes.data,
      slot.ctypes.data, status.ctypes.data)
  return position, slot, status


def layout_from_factor_table(values, kinds):
  """SceneLayout of a drawn factor table ((n, S, 10) values and SWB_FT_* kinds, empty slots
  first): each sprite's factors as NumPy columns of their kind, one SpriteTable per combination of
  kinds -- what scene.arrays_from_layout takes."""
  n, S, _ = values.shape
  occupied = kinds[..., 2] != FT_NONE
  count = occupied.sum(1)
  width = int(count.max()) if n else 0
  ref_table = np.zeros((n, width), np.int64)
  ref_row = np.zeros((n, width), np.int64)
  si, sj = np.nonzero(occupied)
  slot = sj - (S - count[si])
  sig = kinds[si, sj]
  uniq, which = np.unique(sig, axis=0, return_inverse=True)
  which = which.reshape(-1)
  tables = []
  for t, ks in enumerate(uniq):
    rows = np.flatnonzero(which == t)
    cols = {}
    for f, name in enumerate(FACTORS):
      v = values[si[rows], sj[rows], f]
      if ks[f] == FT_SHAPE:
        col = np.empty(len(rows), dtype=object)
        col[:] = [constants.SHAPE_NAMES[int(i) - 1] for i in v]
      else:
        col = v.astype(KIND_DTYPES[int(ks[f])])
      cols[name] = col
    tables.append(gen.SpriteTable(cols, len(rows)))
    ref_table[si[rows], slot[rows]] = t
    ref_row[si[rows], slot[rows]] = np.arange(len(rows))
  return gen.SceneLayout(tables, count, ref_table, ref_row)
