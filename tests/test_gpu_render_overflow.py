"""The render kernel's SWB_ENV_SPAN_OVERFLOW flag on each side of every phase-B capacity.

Polygons registered under shape names of either span class (ids 1..6 convex, 7..12 concave:
the engine keeps one span per sprite row until an id above 6 is uploaded) are built on the
canvas so that one row holds exactly CAP crossings or one more pair, M runs of one sprite's
fill or one more.  (Crossing counts are even: every scanned edge through a row is matched by
one back, and an edge ending on an interior row counts twice, so the first count past CAP is
CAP + 2.)  Each sits in its own env beside envs of ordinary sprites.  Through render, step,
step_host, step_gather and render_states, every env's status must be what
tests/span_overflow.py restates and every unflagged env must match the oracle bit for bit;
check_render raises exactly for the flagged ones.  The segment-table side is
test_gpu_render_geometry.test_segment_capacity_boundary.
"""
import numpy as np
import pytest

from oracle import oracle
from tests import fixtures, span_overflow
from tests import test_gpu_render_geometry as geo

W, H, AA = 64, 64, 2
CW, CH = W * AA, H * AA
Y = 60          # the canvas row the crossing and span boundaries sit on
S = 3           # slots per env: the boundary polygon alone, or ordinary sprites


def _to_shape(pts):
  """Canvas pixel corners -> vertices of a sprite at (0, 0), scale 1, angle 0: each lands
  half a pixel inside its pixel, so that Pillow's truncation gives it back exactly."""
  p = np.asarray(pts, np.float64)
  return np.stack([(p[:, 0] + 0.5) / CW, (p[:, 1] + 0.5) / CH], 1)


def spikes(up, down):
  """The rectangle x 20..100, rows 40..80, whose left side has `up` spikes up to row Y - 1 and
  `down` spikes down to row Y + 1 at its vertex on row Y.  On row Y the lower left edge counts
  once, the upper one twice, an up spike 4, a down spike 2, the right side once: 4 + 4 up +
  2 down crossings, and the fill is one run."""
  pts = [(20, 40), (100, 40), (100, 80), (20, 80), (20, Y)]
  pts += [(20, Y + 1), (20, Y)] * down + [(20, Y - 1), (20, Y)] * up
  return pts


def step_left():
  """Wide on top, a step on the left at row Y: the crossing spans of row Y, [20, 20] and
  [50, 100], are disjoint, and the horizontal edge 20..50 of that row joins them into one run."""
  return [(20, 40), (100, 40), (100, 80), (50, 80), (50, Y), (20, Y)]


def notch():
  """The rectangle with a notch from the top edge down to row Y: two runs on rows 41..59."""
  return [(20, 40), (50, 40), (50, Y), (70, Y), (70, 40), (100, 40), (100, 80), (20, 80)]


def comb(teeth):
  """A bar on rows 40..50 with `teeth` teeth down to row 80: as many runs on rows 51..79."""
  right = 10 + 20 * teeth - 10
  pts = [(10, 40), (right, 40)]
  for t in range(teeth - 1, -1, -1):
    x0 = 10 + 20 * t
    pts += [(x0 + 10, 80), (x0, 80)]
    if t:
      pts += [(x0, 50), (x0 - 10, 50)]
  return pts


# (env name, shape name it is registered as, canvas polygon, restated maxima that matter,
#  conditions it must flag)
CONVEX_BOUNDARY = [
    ('crossings_8', 'triangle', spikes(1, 0), dict(crossings=8, spans=1), ()),
    ('crossings_10', 'square', spikes(1, 1), dict(crossings=10, spans=1), ('crossings',)),
    ('spans_1_joined', 'pentagon', step_left(), dict(spans=1), ()),
    ('spans_2', 'hexagon', notch(), dict(spans=2), ('spans',)),
]
CONCAVE_BOUNDARY = [
    ('crossings_16', 'star_4', spikes(3, 0), dict(crossings=16, spans=1), ()),
    ('crossings_18', 'star_5', spikes(3, 1), dict(crossings=18, spans=1), ('crossings',)),
    ('spans_4', 'star_6', comb(4), dict(spans=4), ()),
    ('spans_5', 'spoke_4', comb(5), dict(spans=5), ('spans',)),
]
# ordinary sprites in the envs beside them: shape ids the boundary polygons do not replace
NEIGHBOUR_IDS = {False: (5, 6), True: (1, 2, 3, 11, 12)}
N_NEIGHBOURS = 6


def _shapes(boundary):
  from spriteworld_b200 import constants
  shapes = dict(constants.SHAPES)
  for _, name, pts, _, _ in boundary:
    shapes[name] = _to_shape(pts)
  return shapes


def _arrays(boundary, concave):
  """One env per boundary polygon (slot 0, the other slots empty), then N_NEIGHBOURS envs of
  ordinary sprites, boundary envs and neighbours interleaved."""
  n = len(boundary) + N_NEIGHBOURS
  a = geo._empty_arrays(n, S)
  rng = np.random.RandomState(7 + concave)
  order = rng.permutation(n)
  for i, (_, name, _, _, _) in enumerate(boundary):
    e = order[i]
    a['shape'][e, 0] = oracle.SHAPE_IDS[name]
    a['scale'][e, 0] = 1.0
    a['rgb'][e, 0] = (250, 120, 30)
  for e in order[len(boundary):]:
    a['x'][e] = geo._f32(rng.uniform(0.1, 0.9, S))
    a['y'][e] = geo._f32(rng.uniform(0.1, 0.9, S))
    a['shape'][e] = rng.choice(NEIGHBOUR_IDS[concave], S)
    a['scale'][e] = rng.uniform(0.1, 0.3, S)
    a['angle'][e] = rng.randint(0, 360, S)
    a['rgb'][e] = rng.randint(0, 256, (S, 3))
  return a, order[:len(boundary)]


CLASSES = [('convex', CONVEX_BOUNDARY, False), ('concave', CONCAVE_BOUNDARY, True)]


@pytest.mark.parametrize('cls, boundary, concave', CLASSES, ids=[c[0] for c in CLASSES])
def test_boundary_polygons_restate_as_built(cls, boundary, concave):
  """The restatement puts each polygon where it was built: its maxima, its conditions; and
  the neighbours are within every table."""
  M = 4 if concave else 1
  shapes = _shapes(boundary)
  a, envs = _arrays(boundary, concave)
  rec = fixtures.records_from_arrays(a)
  for (name, _, _, want, flags), e in zip(boundary, envs):
    got = span_overflow.restate(W, H, AA, rec[e], shapes, M)
    for k, v in want.items():
      assert got[k] == v, (name, k, got)
    assert span_overflow.conditions(got, M, span_overflow.segcap(S, M)) == flags, (name, got)
  for e in sorted(set(range(len(rec))) - set(envs)):
    got = span_overflow.restate(W, H, AA, rec[e], shapes, M)
    assert not span_overflow.conditions(got, M, span_overflow.segcap(S, M)), (e, got)


@pytest.mark.gpu
@pytest.mark.parametrize('cls, boundary, concave', CLASSES, ids=[c[0] for c in CLASSES])
def test_overflow_flag_on_each_side_of_every_capacity(cls, boundary, concave):
  import torch
  from spriteworld_b200 import _native, engine
  from tests import test_gpu_render_states as states_test
  a, envs = _arrays(boundary, concave)
  E = len(a['x'])
  case = ('overflow_' + cls, W, H, AA, (0, 0, 0), S, E, concave, None)
  sw = geo.Sweep(case, geo._n_sms(), arrs=a, shapes=_shapes(boundary))
  try:
    raster = engine.Raster(sw.eng, W, H, AA, sw.bg)
    flagged = [e for e in range(E) if sw.overflow(e)]
    assert flagged == sorted(e for (_, _, _, _, f), e in zip(boundary, envs) if f), flagged
    # render, step, step_host, step_gather (two targets): status exact, the others bit-exact
    assert geo._run_modes(sw, raster) == [E - len(flagged)] * 5
    # records of the same envs, permuted and repeated
    n_exact, n_within = states_test._render_permuted(sw, raster)
    assert n_exact == [n_within] * 2
    # check_render: every env loaded with one env's record raises exactly when that env is flagged
    saved = sw.eng.save_envs()
    for e in range(E):
      sw.eng.load_envs(saved[np.full(E, e)])
      frames = sw.eng.render(raster).cpu().numpy()
      status = sw.eng.render_status().cpu().numpy()
      assert (status == (_native.ENV_SPAN_OVERFLOW if e in flagged else 0)).all(), (e, status)
      if e in flagged:
        with pytest.raises(_native.NativeError):
          sw.eng.check_render()
      else:
        sw.eng.check_render()
        assert (frames == sw.ref(e)[0]).all(), e
    torch.cuda.synchronize()
    raster.close()
  finally:
    sw.close()
