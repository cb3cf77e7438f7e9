"""Env records from factor values (swb_make_states), the record maker built for the CPU
(scene_program.make_states_on_host, csrc/swb_make_states.cuh), against the host packer, byte for
byte: record i is the sprite list [Sprite(**factors at (i, j)) for the occupied slots j] packed by
scene.arrays_from_layout with the same filters and colour map, assembled into record bytes with
engine.record_layout, live position = initial position, reset_next = 0, step_count and goals as
given.  A record with a SWB_MAKE_* bit is zeros.  No GPU needed; tests/test_gpu_make_states.py
holds the kernel to this build.
"""
import importlib
import math
import types

import numpy as np
import pytest
import torch

from spriteworld_b200 import constants, environment, scene, scene_program, sprite_generators as gen
from spriteworld_b200 import engine as engine_lib
from spriteworld_b200 import factor_distributions as distribs
from spriteworld_b200 import sprite as sprite_lib
from spriteworld_b200.renderers import color_maps

CONFIGS = ['cobra.' + n for n in ('clustering', 'exploration', 'goal_finding_more_distractors',
                                  'goal_finding_more_targets', 'goal_finding_new_position',
                                  'goal_finding_new_shape', 'sorting')] + \
          ['examples.' + n for n in ('goal_finding_clustering', 'goal_finding_embodied',
                                     'goal_finding_random_goal')]
FACTORS = sprite_lib.FACTOR_NAMES
DTYPES = (np.float32, np.float64, np.int8, np.int16, np.int32, np.int64, np.uint8)
FLOATS = (np.float32, np.float64)
ANGLE, SHAPE, HOLE, INT, STEP = (scene_program.MAKE_ANGLE, scene_program.MAKE_SHAPE, scene_program.MAKE_HOLE,
                                 scene_program.MAKE_INT, scene_program.MAKE_STEP)


# -- the restatement -------------------------------------------------------------------------------


def restate_status(columns, step_count=None):
  """SWB_MAKE_* bits of each record, from the contract."""
  shape = np.asarray(columns['shape'])
  n, S = shape.shape
  out = np.zeros(n, np.uint8)
  for i in range(n):
    occ = []
    for j in range(S):
      v = float(shape[i, j])
      if not (0 <= v <= 12 and v == int(v)):
        out[i] |= SHAPE
        occ.append(False)
        continue
      occ.append(v != 0)
      if v == 0:
        continue
      if 'angle' in columns:
        a = float(columns['angle'][i, j])
        if not (-360 <= a <= 360 and a == int(a)):
          out[i] |= ANGLE
      for name, col in columns.items():
        if name != 'shape' and col.dtype == np.int64 and abs(int(col[i, j])) > 2 ** 53:
          out[i] |= INT
    first = occ.index(True) if True in occ else S
    if not all(occ[first:]):
      out[i] |= HOLE
    if step_count is not None and step_count[i] < 0:
      out[i] |= STEP
  return out


def host_packer_records(columns, S, filters=(), cmap=None, G=0, goals=None, step_count=None):
  """(records, status): the sprite lists packed by scene.arrays_from_layout, as record bytes."""
  shape = np.asarray(columns['shape'])
  n = shape.shape[0]
  status = restate_status(columns, step_count)
  scenes = []
  for i in range(n):
    sc = []
    for j in range(S):
      if status[i] or shape[i, j] == 0:
        continue
      kw = {k: columns[k][i, j] for k in columns if k != 'shape'}
      kw['shape'] = constants.SHAPE_NAMES[int(shape[i, j]) - 1]
      sc.append(sprite_lib.Sprite(**kw))
    scenes.append(sc)
  if any(scenes):
    b = scene.arrays_from_layout(gen.layout_from_sprite_lists(scenes), S, filters, cmap)
  else:
    b = scene.empty_batch(n, S)
  fields, rb = engine_lib.record_layout(S, G)
  rgb = b['rgb'].astype(np.uint32)
  values = dict(x0=b['x'], y0=b['y'], m00=b['m00'], m01=b['m01'], m10=b['m10'], m11=b['m11'], vx=b['vx'],
                vy=b['vy'], pos_x=b['x'], pos_y=b['y'], member=b['member'],
                rgb=rgb[..., 0] | rgb[..., 1] << 8 | rgb[..., 2] << 16,
                factors=b['factors'].transpose(0, 2, 1),
                step_count=np.zeros(n, np.int32) if step_count is None else step_count,
                reset_next=np.zeros(n, np.uint8), shape=b['shape'], pos_f32=b['pos_f32'])
  if G:
    values['goal'] = goals
  rec = np.zeros((n, rb), np.uint8)
  for name, off, dtype, shp in fields:
    v = np.ascontiguousarray(np.asarray(values[name]).astype(dtype)).reshape(n, -1).view(np.uint8)
    rec[:, off:off + v.shape[1]] = v
  rec[status != 0] = 0
  return rec, status


def check(columns, S, filters=(), cmap=None, G=0, goals=None, step_count=None, what=''):
  packer = scene_program.compile_packer(filters, cmap)
  got, got_status, flag = scene_program.make_states_on_host(packer, columns, S, G, goals, step_count)
  want, want_status = host_packer_records(columns, S, filters, cmap, G, goals, step_count)
  assert np.array_equal(got_status, want_status), (what, got_status, want_status)
  bad = np.flatnonzero((got != want).any(1))
  assert not len(bad), (what, 'record %d of %d differs at bytes %s' % (
      bad[0], len(got), np.flatnonzero(got[bad[0]] != want[bad[0]])[:8]))
  shape = np.asarray(columns['shape'])
  stars = ((shape >= 7) & (shape <= 12) & (want_status[:, None] == 0)).any()
  assert flag == bool(stars), what
  return got, got_status


# -- factor columns --------------------------------------------------------------------------------


def _values(rng, name, dtype, n, S, hsv=False):
  """(n, S) values of factor `name` in `dtype` that the packer accepts."""
  dt = np.dtype(dtype)
  if name == 'angle':
    if dt.kind == 'f':
      v = rng.randint(-360, 361, (n, S)).astype(dt)
      v[rng.rand(n, S) < 0.1] = -0.0
      return v
    info = np.iinfo(dt)
    return rng.randint(max(int(info.min), -360), min(int(info.max), 360) + 1, (n, S)).astype(dt)
  if dt.kind == 'f':
    lo, hi = dict(x=(-0.2, 1.2), y=(-0.2, 1.2), scale=(0.0, 0.3), x_vel=(-0.1, 0.1), y_vel=(-0.1, 0.1)).get(
        name, (-0.5, 1.5) if hsv else (-300.0, 300.0))
    return rng.uniform(lo, hi, (n, S)).astype(dt)
  info = np.iinfo(dt)
  lo, hi = (0, 2) if name in ('x', 'y', 'scale') else (max(int(info.min), -1000), min(int(info.max), 1000))
  return rng.randint(lo, hi + 1, (n, S)).astype(dt)


def _shapes(rng, n, S, dtype=np.uint8):
  """Shape ids 1 .. 12 right-aligned in S slots, 0 .. S sprites per scene."""
  k = rng.randint(0, S + 1, n)
  shape = np.where(np.arange(S)[None, :] >= (S - k)[:, None], rng.randint(1, 13, (n, S)), 0)
  return shape.astype(dtype)


def random_columns(rng, n, S, hsv=False, dtypes=DTYPES, omit=0.2):
  cols = {'shape': _shapes(rng, n, S, dtypes[rng.randint(len(dtypes))])}
  color_dt = FLOATS[rng.randint(2)] if hsv else None
  for name in FACTORS:
    if name == 'shape' or rng.rand() < omit:
      continue
    if name in ('c0', 'c1', 'c2') and hsv:
      continue
    cols[name] = _values(rng, name, dtypes[rng.randint(len(dtypes))], n, S)
  if hsv and rng.rand() > omit:
    for name in ('c0', 'c1', 'c2'):
      cols[name] = _values(rng, name, color_dt, n, S, hsv=True)
  return cols


def _config(name):
  cfg = importlib.import_module('spriteworld_b200.configs.' + name).get_config('train')
  _, filters = cfg['task'].compile()
  pil, _ = environment._split_renderers(cfg['renderers'])
  return cfg, list(filters), environment._color_map(pil)


# -- the tests -------------------------------------------------------------------------------------


@pytest.mark.parametrize('name', CONFIGS)
def test_config_filters_and_colour_map(name):
  cfg, filters, cmap = _config(name)
  rng = np.random.RandomState(len(name))
  # the config's own scenes, as columns of their factors' dtypes, and random columns
  np.random.seed(len(name))
  scenes = [cfg['init_sprites']() for _ in range(32)]
  S = max(len(sc) for sc in scenes)
  b = scene.arrays_from_layout(gen.layout_from_sprite_lists(scenes), S)
  cols = {'shape': b['shape'], 'x': b['x'], 'y': b['y'], 'scale': b['factors'][..., 0].astype(np.float64),
          'angle': b['factors'][..., 1].astype(np.int64)}
  color_dt = np.float64 if cmap is not None else np.int64
  for k, c in enumerate(('c0', 'c1', 'c2')):
    cols[c] = np.array([[0 if j < S - len(sc) else getattr(sc[j - (S - len(sc))], c) for j in range(S)]
                        for sc in scenes]).astype(color_dt)
  check(cols, S, filters, cmap, what=name)
  for trial in range(4):
    check(random_columns(rng, 48, S, hsv=cmap is not None), S, filters, cmap, what=(name, trial))


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('cmap', [None, color_maps.hsv_to_rgb])
def test_every_dtype(dtype, cmap):
  _, filters, _ = _config('cobra.goal_finding_more_targets')
  filters = filters + [distribs.Continuous('x', 0.2, 0.8), distribs.Discrete('shape', ['triangle', 'star_5']),
                       distribs.Continuous('c1', np.float32(0.25), 0.75), distribs.Continuous('angle', -90, 90)]
  rng = np.random.RandomState(7)
  S = 6
  hsv = cmap is not None
  cols = {'shape': _shapes(rng, 64, S, dtype)}
  for name in FACTORS[1:]:
    if hsv and name in ('c0', 'c1', 'c2') and dtype not in FLOATS:
      continue
    cols[name] = _values(rng, name, dtype, 64, S, hsv)
  check(cols, S, filters, cmap, what=np.dtype(dtype).name)


@pytest.mark.parametrize('angle_dtype', [np.float64, np.float32, np.int16, np.int32, np.int64])
def test_every_shape_and_every_integer_angle(angle_dtype):
  angles = np.array(list(range(-360, 361)) + [0.0, -0.0] * 4)
  if np.dtype(angle_dtype).kind != 'f':
    angles = angles[:721]
  n, S = len(angles), 13
  shape = np.tile(np.arange(13, dtype=np.int32), (n, 1))
  shape[:, 0] = 0                                             # ids 1 .. 12 in slots 1 .. 12
  cols = {'shape': shape, 'angle': np.repeat(angles[:, None], S, 1).astype(angle_dtype),
          'scale': np.full((n, S), 0.13), 'x': np.full((n, S), 0.4, np.float32), 'y': np.full((n, S), 0.6, np.float32)}
  got, status = check(cols, S, [distribs.Discrete('angle', [0, -0.0, -30])], what=np.dtype(angle_dtype).name)
  assert not status.any()
  if np.dtype(angle_dtype).kind == 'f':   # -0.0 and 0.0 give differently signed m01 = -sin * scale
    m01 = got[:, 24 * S:32 * S].copy().view(np.float64)[:, 1]
    assert np.signbit(m01[-1]) != np.signbit(m01[-2])


def test_default_factors():
  rng = np.random.RandomState(3)
  S = 5
  check({'shape': _shapes(rng, 40, S)}, S, [distribs.Continuous('x', 0.4, 0.6)], what='shape only')
  check({'shape': _shapes(rng, 40, S)}, S, [distribs.Continuous('c0', 0, 1)], color_maps.hsv_to_rgb,
        what='shape only, hsv')
  for omit in FACTORS[:2] + FACTORS[3:]:
    cols = random_columns(rng, 40, S, omit=0.0)
    del cols[omit]
    check(cols, S, [distribs.Continuous(omit, 0.0, 0.5)], what=omit)


@pytest.mark.parametrize('S', range(1, 33))
def test_slot_counts(S):
  rng = np.random.RandomState(S)
  check(random_columns(rng, 9, S), S, [distribs.Continuous('y', 0.2, 0.5)], what=S)


@pytest.mark.parametrize('G', [0, 2])
def test_goals_and_step_counts(G):
  rng = np.random.RandomState(G)
  n, S = 30, 4
  goals = rng.uniform(-1, 2, (n, G, 2)) if G else None
  step = rng.randint(0, 1000, n).astype(np.int32)
  check(random_columns(rng, n, S), S, G=G, goals=goals, step_count=step)
  check(random_columns(rng, n, S), S, G=G, goals=goals)


def test_each_status_bit_zeroes_its_record():
  S = 3
  ok = np.array([0, 1, 8], np.float64)
  cases = [  # (factor, slot, value, bit)
      ('angle', 2, 0.5, ANGLE), ('angle', 1, 361.0, ANGLE), ('angle', 2, -360.5, ANGLE),
      ('angle', 2, np.nan, ANGLE), ('angle', 1, np.inf, ANGLE),
      ('shape', 2, 13.0, SHAPE | HOLE), ('shape', 1, 2.5, SHAPE), ('shape', 0, -1.0, SHAPE),
      ('shape', 2, np.nan, SHAPE | HOLE)]
  n = len(cases) + 4
  cols = {'shape': np.tile(ok, (n, 1)), 'angle': np.zeros((n, S)), 'c0': np.zeros((n, S), np.int64),
          'scale': np.full((n, S), 0.2)}
  for i, (name, j, v, _) in enumerate(cases):
    cols[name][i, j] = v
  cols['shape'][len(cases), 2] = 0                              # a hole after slot 1
  cols['c0'][len(cases) + 1, 2] = 2 ** 53 + 1                    # beyond 2^53
  cols['c0'][len(cases) + 2, 2] = -2 ** 53                       # held exactly: accepted
  cols['c0'][len(cases) + 3, 0] = 2 ** 62                        # in an empty slot: accepted
  cols['angle'][len(cases) + 3, 0] = 0.5
  step = np.zeros(n, np.int32)
  step[len(cases) + 2] = -1
  rec, status = check(cols, S, step_count=step)
  want = [b for _, _, _, b in cases] + [HOLE, INT, STEP, 0]
  assert status.tolist() == want
  assert not rec[status != 0].any() and rec[status == 0].any(1).all()


def test_the_span_flag_counts_accepted_stars_only():
  S = 2
  cols = {'shape': np.array([[0, 2], [0, 9]], np.int8), 'angle': np.array([[0, 0], [0, 0]], np.int8)}
  check(cols, S)                                        # a star: the flag is set
  cols['shape'][1, 0] = 13                              # ... unless its record is refused
  _, status = check(cols, S)
  assert status.tolist() == [0, SHAPE]


def test_compile_packer():
  p = scene_program.compile_packer().struct
  angles = [p.angle[i] for i in range(p.n_angles)]
  assert p.n_angles == 722 and p.n_ops == 1 and p.ops[0].op == scene_program.G_END and p.max_sprites == 0
  assert math.copysign(1, angles[360]) < 0 and angles[360:362] == [0.0, 0.0] and angles[0] == -360 and angles[-1] == 360
  assert all(p.angle_cos[i] == math.cos(math.radians(a)) for i, a in enumerate(angles))
  f = [distribs.Continuous('c0', 0, 0.5)]
  a = scene_program.compile_packer(f, color_maps.hsv_to_rgb).struct
  assert a.color_mode == scene_program.COLOR_HSV and a.n_filters == 1
  with pytest.raises(NotImplementedError, match='colour map'):
    scene_program.compile_packer(f, lambda c: c)
  with pytest.raises(NotImplementedError, match='filters'):
    scene_program.compile_packer([distribs.Continuous('x', 0, 1)] * 33)
  with pytest.raises(NotImplementedError, match='containment'):
    scene_program.compile_packer([object()])


# -- the Python layer's refusals, on an engine double ----------------------------------------------


class _Lib(object):

  def __init__(self):
    self.calls = 0

  def swb_make_states(self, *args):
    self.calls += 1
    return 0


def _double(G=0, cmap=None):
  eng = types.SimpleNamespace(n_slots=3, n_goals=G, device=torch.device('cpu'), signature=b'sig', record_bytes=336,
                              _lib=_Lib(), _h=None, _stream=lambda: None,
                              _packer=scene_program.compile_packer((), cmap))
  for name in ('make_states', '_check_goals', 'check_states'):
    setattr(eng, name, getattr(engine_lib.Engine, name).__get__(eng))
  eng.span_class = lambda: 1
  return eng


def test_python_refusals_enqueue_nothing():
  eng = _double()
  shape = torch.zeros((4, 3), dtype=torch.uint8)
  bad = [
      (dict(factors={}), "'shape'"),
      (dict(factors={'shape': torch.zeros((4, 2))}), r'\(n, 3\)'),
      (dict(factors={'shape': shape, 'size': torch.zeros(3)}), 'unknown factors'),
      (dict(factors={'shape': shape, 'x': torch.zeros((4, 3), dtype=torch.bool)}), "factors\\['x'\\]"),
      (dict(factors={'shape': shape, 'x': torch.zeros((5, 3))}), "factors\\['x'\\]"),
      (dict(factors={'shape': shape, 'x': np.zeros((4, 3))}), "factors\\['x'\\]"),
      (dict(factors={'shape': shape.to(torch.uint16)}), "factors\\['shape'\\]"),
      (dict(factors={'shape': shape}, goals=torch.zeros((4, 1, 2), dtype=torch.float64)), 'samples no goals'),
      (dict(factors={'shape': shape}, step_count=torch.zeros(4, dtype=torch.int64)), 'step_count'),
      (dict(factors={'shape': shape}, span_class=2), 'span_class'),
  ]
  for kw, msg in bad:
    with pytest.raises(ValueError, match=msg):
      eng.make_states(**kw)
  g = _double(G=1)
  with pytest.raises(ValueError, match='goals'):
    g.make_states({'shape': shape})
  with pytest.raises(ValueError, match='goals'):
    g.make_states({'shape': shape}, goals=torch.zeros((4, 2, 2), dtype=torch.float64))
  h = _double(cmap=color_maps.hsv_to_rgb)
  for colours in ({'c0': torch.zeros(3)}, {'c0': torch.zeros(3), 'c1': torch.zeros(3),
                                            'c2': torch.zeros(3, dtype=torch.float64)},
                  {c: torch.zeros(3, dtype=torch.int32) for c in ('c0', 'c1', 'c2')}):
    with pytest.raises(ValueError, match='hsv_to_rgb'):
      h.make_states(dict(shape=shape, **colours))
  assert eng._lib.calls == g._lib.calls == h._lib.calls == 0
  # accepted: the columns broadcast, the call is made once
  states, status = h.make_states(dict(shape=shape, **{c: torch.zeros(1, 3) for c in ('c0', 'c1', 'c2')}),
                                 span_class=4)
  assert h._lib.calls == 1 and states.span_class == 4 and status.shape == (4,)


def test_environment_refuses_other_colour_maps_before_anything():
  eng = _double()
  env = types.SimpleNamespace(_packer=None, _filters=[], _color_to_rgb=lambda c: c, _engine=eng)
  with pytest.raises(NotImplementedError, match='colour map'):
    environment.BatchedEnvironment.make_states(env, {'shape': torch.zeros((1, 3))})
  assert env._packer is None and eng._lib.calls == 0
