"""Env records from factor values on the device (csrc/swb_make_states.cuh, swb_make_states), byte
for byte.

The kernel equals the CPU build of the same source (tests/test_make_states_on_host.py holds that
build to the host packer) for 0, 1, 33 and 4097 records and every column dtype, into guarded
buffers.  Made records equal what save_envs saves right after the reset step of the same scenes --
drawn by the device sampler (fed the factor values and kinds it drew) or by a fixed init_sprites --
with and without sampled goals, and so every record observation, relabelling, planning call and
load gives equal results.  Stars infer span class 4 and render the oracle's frames.  A call is one
launch, synchronises only to infer the span class, changes nothing, and a refused call enqueues
nothing.
"""
import ctypes

import numpy as np
import pytest
import torch

from spriteworld_b200 import _native, environment, scene_program, sprite as sprite_lib
from spriteworld_b200 import engine as engine_lib
from tests import test_make_states_on_host as on_host
from tests.test_gpu_rollout import _everything
from tests.test_gpu_trajectory import _env_cfg

gpu = pytest.mark.gpu
DTYPES = on_host.DTYPES


def _env(kind='goal_finding', sampler='device', E=16, **kw):
  cfg = _env_cfg(kind)
  cfg.update(kw)
  return environment.BatchedEnvironment(n_envs=E, pool_depth=4, sampler=sampler, seed=5, **cfg)


def _tensors(cols, device):
  return {k: torch.from_numpy(np.ascontiguousarray(v)).to(device) for k, v in cols.items()}


def _records(states):
  torch.cuda.synchronize()
  return states.data.cpu().numpy()


# -- 1: the kernel against the CPU build -----------------------------------------------------------

@gpu
@pytest.mark.parametrize('n', [0, 1, 33, 4097])
def test_device_equals_the_cpu_build_into_guarded_buffers(n):
  env = _env()
  eng, S = env.engine, env.engine.n_slots
  hsv = env._color_to_rgb is not None
  rng = np.random.RandomState(n)
  rb = eng.record_bytes
  for dtype in DTYPES:
    cols = on_host.random_columns(rng, n, S, hsv=hsv, dtypes=(dtype,), omit=0.1)
    if n:   # some refused records and some stars
      cols['shape'][rng.rand(n) < 0.05, -1] = 13
      cols['shape'][rng.rand(n) < 0.1, -1] = 8
    step = rng.randint(-2, 100, n).astype(np.int32)
    guard = torch.full((n + 2, rb), 0xA5, dtype=torch.uint8, device=eng.device)
    out = engine_lib.EnvStates(guard[1:n + 1], 1, eng.signature, S)
    states, status = env.make_states(_tensors(cols, eng.device), step_count=torch.from_numpy(step).to(eng.device))
    states2, status2 = eng.make_states(_tensors(cols, eng.device), step_count=torch.from_numpy(step).to(eng.device),
                                       span_class=1, out=out)
    want, want_status, flag = scene_program.make_states_on_host(env._packer, cols, S, 0, None, step)
    g = guard.cpu().numpy()
    assert (g[0] == 0xA5).all() and (g[-1] == 0xA5).all(), np.dtype(dtype).name
    assert np.array_equal(g[1:n + 1], want) and np.array_equal(_records(states), want), np.dtype(dtype).name
    assert np.array_equal(status.cpu().numpy(), want_status) and np.array_equal(status2.cpu().numpy(), want_status)
    assert states.span_class == (4 if flag else eng.span_class()) and states2 is out and out.span_class == 1
  env.close()


# -- 2: made records are what save_envs saves after the FIRST step ---------------------------------

_KIND_DTYPES = dict(scene_program.KIND_DTYPES)
_KIND_DTYPES.update({scene_program.FT_PYFLOAT: np.dtype(np.float64), scene_program.FT_PYINT: np.dtype(np.int64),
                     scene_program.FT_SHAPE: np.dtype(np.uint8)})


def _columns_of_drawn(values, kinds):
  """Factor columns of a drawn factor table (n, S, 10): each factor in its drawn kind's dtype (one
  kind per factor over the occupied slots), defaults (kind NONE in empty slots) as zeros."""
  occ = kinds[..., 2] != scene_program.FT_NONE
  cols = {}
  for f, name in enumerate(sprite_lib.FACTOR_NAMES):
    ks = set(kinds[..., f][occ].tolist()) or {scene_program.FT_F64}
    assert len(ks) == 1, (name, ks)
    cols[name] = np.where(occ, values[..., f], 0).astype(_KIND_DTYPES[ks.pop()])
  return cols


def _fixed_sprites():
  f32 = np.float32
  return [sprite_lib.Sprite(x=f32(0.2 + 0.1 * k), y=f32(0.7 - 0.1 * k), shape=('triangle', 'square', 'star_4')[k],
                            angle=(-30, 0, 45)[k], scale=(0.1, 0.2, 0.15)[k], c0=f32(0.1 * k), c1=f32(0.9),
                            c2=f32(0.5 + 0.2 * k)) for k in range(3)]


def _fixed_columns(n, S):
  sprites = _fixed_sprites()
  cols = {name: np.zeros((n, S), np.float32) for name in ('x', 'y', 'c0', 'c1', 'c2')}
  cols.update(shape=np.zeros((n, S), np.uint8), angle=np.zeros((n, S), np.int64), scale=np.zeros((n, S)))
  for k, s in enumerate(sprites):
    j = S - len(sprites) + k
    for name in cols:
      cols[name][:, j] = (engine_lib.SHAPE_IDS[s.shape] if name == 'shape' else getattr(s, name))
  return cols


def _made_and_saved(sampler, kind):
  if sampler == 'device':
    env = _env(kind)
  else:
    env = _env(kind, sampler='host', init_sprites=_fixed_sprites, refill='sync')
  env.reset()
  eng, E, S = env.engine, env.n_envs, env.engine.n_slots
  saved = env.save_envs()
  if sampler == 'device':
    serial = eng.download_state_serial()
    b, fail = scene_program.sample_on_host(env._program, env.seed, np.arange(E), serial, S)
    assert fail is None
    cols = _columns_of_drawn(b['factor_value'], b['factor_kind'])
  else:
    cols = _fixed_columns(E, S)
  goals = env.goal_tensor().clone() if eng.n_goals else None
  made, status = env.make_states(_tensors(cols, eng.device), goals=goals)
  assert not status.any()
  assert np.array_equal(_records(made), _records(saved)), (sampler, kind)
  assert made.span_class == saved.span_class or (made.span_class == 4) == _has_stars(cols)
  return env, made, saved


def _has_stars(cols):
  return bool(((cols['shape'] >= 7) & (cols['shape'] <= 12)).any())


def _same(a, b, what):
  if isinstance(a, torch.Tensor):
    assert torch.equal(a, b) or (a.is_floating_point() and torch.equal(a.isnan(), b.isnan()) and
                                 torch.equal(a.nan_to_num(), b.nan_to_num())), what
  elif isinstance(a, dict):
    assert a.keys() == b.keys(), what
    for k in a:
      _same(a[k], b[k], (what, k))
  else:
    assert len(a) == len(b), what
    for i, (x, y) in enumerate(zip(a, b)):
      _same(x, y, (what, i))


@gpu
@pytest.mark.parametrize('sampler,kind', [('device', 'goal_finding'), ('device', 'goals'), ('device', 'sorting'),
                                          ('host', 'goal_finding'), ('host', 'goals')])
def test_made_records_equal_saved_records_and_give_equal_results(sampler, kind):
  env, made, saved = _made_and_saved(sampler, kind)
  eng, E = env.engine, env.n_envs
  rng = np.random.RandomState(1)
  plans = rng.uniform(0, 1, (4, E, 3, 4)).astype(np.float32)
  for name, fn in [('observe', lambda s: env.observe(s)),
                   ('factor_tensors', lambda s: env.factor_tensors(sprite_lib.FACTOR_NAMES, s)),
                   ('goal_tensor', lambda s: env.goal_tensor(s)),
                   ('evaluate', lambda s: env.evaluate(s)),
                   ('contained', lambda s: env.sample_contained_positions(7, 3, s)),
                   ('rollout', lambda s: env.rollout(plans, s)),
                   ('expand', lambda s: (env.expand(plans, s)[0], env.expand(plans, s)[1].data))]:
    _same(fn(made), fn(saved), name)
  for r in env._renderers.values():   # masks, coverage, soft masks and boxes of any raster size
    for call in (env.render_masks, env.render_coverage, env.render_soft_masks, env.render_boxes):
      if hasattr(r, 'width') and hasattr(r, 'anti_aliasing'):
        _same(call(r, made), call(r, saved), call.__name__)
  # loaded and stepped: as envs loaded from the saved records
  out = []
  for states in (made, saved):
    env.load_envs(states)
    steps = []
    for t in range(4):
      ts = env.step(plans[t, :, 0])
      steps.append([ts.step_type.clone(), ts.reward.clone()] + [v.clone() for v in ts.observation.values()
                                                                if isinstance(v, torch.Tensor)])
    out.append(steps)
  # compared while the loaded episode lasts: after a LAST each env starts the next scene of its ring,
  # which the first pass has used up
  alive = torch.ones(E, dtype=torch.bool, device=eng.device)
  for t in range(4):
    for a, b in zip(out[0][t], out[1][t]):
      _same(a[alive], b[alive], ('load and step', t))
    alive &= out[0][t][0] == _native.STEP_MID
  env.close()


# -- 3: stars --------------------------------------------------------------------------------------

@gpu
def test_stars_infer_span_class_4_and_render_the_oracles_frames():
  from oracle import oracle
  from spriteworld_b200 import constants
  from tests.oracle_engine import record_sprites
  env = _env(E=8)
  eng, S = env.engine, env.engine.n_slots
  assert eng.span_class() == 1
  rng = np.random.RandomState(9)
  n = 40
  cols = on_host.random_columns(rng, n, S, hsv=True, dtypes=(np.float64,), omit=0.0)
  cols['shape'] = np.tile(np.arange(S, dtype=np.int16) + 7, (n, 1)) % 13
  cols['shape'][cols['shape'] == 0] = 12
  cols['scale'] = rng.uniform(0.1, 0.4, (n, S))
  made, status = env.make_states(_tensors(cols, eng.device))
  assert not status.any() and made.span_class == 4 and eng.span_class() == 1
  obs, st = env.observe(made)
  torch.cuda.synchronize()
  assert not st.any()
  img = env._rasters['image']
  rc = oracle.raster_cfg(img.width, img.height, img.anti_aliasing)
  tab = oracle.shape_table(constants.SHAPES)
  sprites = record_sprites(eng, made)
  frames = obs['image'].cpu().numpy()
  for i in range(0, n, 3):
    assert np.array_equal(frames[i], oracle.render(rc, tab, sprites[i])), i
  # class 1 given: the stars overflow the span tables, flagged, never a silent wrong frame
  cheap, _ = env.make_states(_tensors(cols, eng.device), span_class=1)
  _, st1 = env.observe(cheap)
  assert (st1.cpu().numpy() & _native.ENV_SPAN_OVERFLOW).any()
  env.close()


# -- 4: one launch, no synchronisation with a span class, nothing changes, refusals -------------------

@gpu
def test_one_launch_no_sync_with_span_class_and_nothing_changes():
  env = _env(E=12)
  env.reset()
  eng, S = env.engine, env.engine.n_slots
  cols = _tensors(on_host.random_columns(np.random.RandomState(2), 50, S, hsv=True, omit=0.0), eng.device)
  env.make_states(cols, span_class=1)   # loads the packer
  book = (env._t, env._resets, env._safe_step, env.refill_stats())
  frames = {k: v.clone() for k, v in env._frames.items()}
  rng_state = env._rng.get_state()[1].copy()
  before, launches = _everything(eng), eng.launch_count()
  torch.cuda.set_sync_debug_mode('error')
  try:
    made, _ = env.make_states(cols, span_class=4)
    assert eng.launch_count() == launches + 1
    with pytest.raises(RuntimeError):
      env.make_states(cols)      # the inferred span class reads a flag back
  finally:
    torch.cuda.set_sync_debug_mode('default')
  assert eng.launch_count() == launches + 2 and made.span_class == 4
  after = _everything(eng)
  for k, v in before.items():
    assert np.array_equal(v, after[k], equal_nan=True), k
  assert book == (env._t, env._resets, env._safe_step, env.refill_stats())
  assert all(torch.equal(v, env._frames[k]) for k, v in frames.items())
  assert np.array_equal(rng_state, env._rng.get_state()[1])
  # refusals: Python's, then the library's, enqueue nothing
  shape = cols['shape']
  for kw in (dict(factors={'x': cols['x']}), dict(factors=dict(cols, c0=cols['c0'].to(torch.int32))),
             dict(factors=cols, goals=torch.zeros((50, 1, 2), dtype=torch.float64, device=eng.device)),
             dict(factors=dict(cols, shape=shape[:, :1]))):
    with pytest.raises(ValueError):
      env.make_states(**kw)
  lib, rb = eng._lib, eng.record_bytes
  rec = torch.zeros((50, rb), dtype=torch.uint8, device=eng.device)
  status = torch.zeros(50, dtype=torch.uint8, device=eng.device)
  c = scene_program.FactorColumns()
  c.col[2], c.kind[2] = shape.data_ptr(), engine_lib._MAKE_DTYPES[shape.dtype]

  def call(cols=c, n=50, records=rec.data_ptr(), records_bytes=rec.numel(), status=status.data_ptr(), flag=None):
    return lib.swb_make_states(eng._h, ctypes.byref(cols), n, None, None, records, records_bytes, status, flag,
                               eng._stream())

  assert call() == 0
  refused = [dict(n=-1), dict(records=rec.data_ptr() + 8), dict(records_bytes=rec.numel() - 1),
             dict(status=rec.data_ptr()), dict(flag=status.data_ptr() + 3), dict(status=shape.data_ptr()),
             dict(records=None)]
  bad = scene_program.FactorColumns()
  bad.col[2], bad.kind[2] = shape.data_ptr(), 9     # uint32: not a column kind
  refused.append(dict(cols=bad))
  bad2 = scene_program.FactorColumns()
  bad2.col[0], bad2.kind[0] = shape.data_ptr(), 1   # no shape column
  refused.append(dict(cols=bad2))
  launches = eng.launch_count()
  for kw in refused:
    assert call(**kw) != 0, kw
  assert eng.launch_count() == launches
  after2 = _everything(eng)
  for k, v in before.items():
    assert np.array_equal(v, after2[k], equal_nan=True), k
  env.close()
