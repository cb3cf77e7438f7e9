"""The phase-B capacities the render layout relies on hold for every shipped shape, and the
restatement of the overflow flag (tests/span_overflow.py) counts what is known.

RenderLayout keeps CAP crossings and M spans per (sprite, canvas row): 8 and 1 while every
shape is convex, 16 and 4 once a star or spoke is uploaded.  Nothing in the kernel checks
that the shipped shapes stay within them except the overflow flag itself, so sweep every
shape of constants.SHAPES over angles, scales (sub-pixel ones included) and positions (on the
canvas edges too, where truncation toward zero folds the vertices on either side of x = 0 or
y = 0 onto the same column or row) on a square and a flat raster, and check the maxima.  The
one excess is a six-armed star or spoke across y = 0: row 0 then holds 18 crossings, and the
kernel flags the env instead of rendering it.
"""
import numpy as np

from oracle import oracle
from spriteworld_b200 import constants
from tests import fixtures, span_overflow
from tests.test_gpu_render_geometry import stripes

ANGLES = [0.0, 45.0, 90.0, 135.0, 180.0, 270.0, 7.0, 33.3, 61.0, 101.5, 222.2, 301.0]
SCALES = [3e-4, 1.5e-3, 6e-3, 0.02, 0.07, 0.2, 0.45, 1.3]
POSITIONS = [(0.5, 0.5), (0.0, 0.0), (0.001, 0.5), (0.5, -0.001), (1.0, 1.0), (0.999, 0.3),
             (-0.004, 1.002), (0.37, 0.61)]
RASTERS = [(32, 32, 5), (110, 8, 5)]    # (W, H, aa): square, and 550 x 40 canvas rows
SIX_ARMED = ('star_6', 'spoke_6')


def test_shipped_shapes_stay_within_crossing_and_span_capacities():
  maxima, folded = {}, set()
  for W, H, aa in RASTERS:
    CW, CH = W * aa, H * aa
    rows = np.arange(CH)
    for name, verts in constants.SHAPES.items():
      M = span_overflow.span_class([oracle.SHAPE_IDS[name]])
      cap, M = span_overflow.limits(M)
      most = maxima.setdefault(name, [0, 0])
      for angle in ANGLES:
        for scale in SCALES:
          for x, y in POSITIONS:
            r = oracle.sprite_record(x, y, name, angle, scale, (1, 1, 1))
            xy = span_overflow.canvas_xy(r, verts, CW, CH)
            ivx, ivy = span_overflow.int_vertices(xy)
            pymin, p_ymax = span_overflow.sprite_rows(ivy, CH)
            mine = rows[(rows >= pymin) & (rows <= min(p_ymax, CH - 1))]
            c = span_overflow.crossings(ivx, ivy, CH, mine)
            # every edge through a row is matched by one back: the first count past CAP is CAP + 2
            assert (c % 2 == 0).all(), (name, angle, scale, x, y, c)
            c, n = span_overflow.sprite_maxima(xy, W, H, aa, M)
            where = (name, (W, H, aa), angle, scale, (x, y))
            if c > cap:
              # the one known excess: a six-armed star or spoke across y = 0, where truncation
              # toward zero puts the vertices of canvas rows -1 and 0 on row 0 (flagged)
              assert name in SIX_ARMED and ivy.min() < 0 <= ivy.max() and c == cap + 2, where
              folded.add(where)
            assert n <= M, where + ('spans', n, M)
            most[0], most[1] = max(most[0], c), max(most[1], n)
  print('most crossings, spans per (sprite, canvas row):',
        ', '.join('%s %d %d' % (k, v[0], v[1]) for k, v in maxima.items()))
  print('beyond CAP (folded on row 0): %d placements' % len(folded))
  assert {w[0] for w in folded} == set(SIX_ARMED)
  # the sweep reaches what the capacities are there for: vertex rows of convex shapes, several
  # spans of the concave ones
  assert max(maxima[k][0] for k in ('triangle', 'square', 'circle')) == 6
  assert max(maxima[k][1] for k in oracle.SHAPE_IDS if oracle.SHAPE_IDS[k] > 6) >= 3


def test_restatement_counts_the_stripes_pieces():
  """Squares in front of a large square cut its pieces on the rows they cover: 17, 16 and 15
  visible pieces, each within its tables but the 17-piece row beyond 16 segments."""
  for n_inside, straddle, star, pieces in ((8, False, False, 17), (8, False, True, 17),
                                           (7, True, True, 16), (7, False, False, 15)):
    a = stripes(n_inside, straddle, star)
    rec = fixtures.records_from_arrays(a)[0]
    M = span_overflow.span_class(a['shape'])
    got = span_overflow.restate(64, 64, 5, rec, constants.SHAPES, M)
    assert got['pieces'] == pieces, (n_inside, straddle, star, got)
    S = len(rec)
    want = ('pieces',) if star and pieces > 16 else ()
    assert span_overflow.conditions(got, M, span_overflow.segcap(S, M)) == want, got
    # the same scenes on a 64 x 100 raster (two bands) count the same
    assert span_overflow.restate(64, 100, 5, rec, constants.SHAPES, M)['pieces'] == pieces


def test_full_window_restates_the_frame_maxima():
  """restate through the window (0, 0, 1, 1) is restate of the frame, on the scenes of every case
  of the geometry, wide anti-aliasing and far sweeps (the first envs of each, and the ones whose
  frame overflows): u = (wx - 0) * (CW / 1) is CW * wx exactly."""
  from tests import test_gpu_render_far as far
  from tests import test_gpu_render_geometry as geo
  from tests import test_gpu_render_wide_aa as wide
  n_flagged = 0
  cases = ([(c, geo.case_arrays(c, geo._n_envs(c, geo.H100_SMS))) for c in geo.CASES + wide.CASES]
           + [(c, far.case_arrays(c)) for c in far.CASES])
  for case, arrs in cases:
    cid, W, H, aa, bg, S, _, concave, kind = case
    recs = fixtures.records_from_arrays(arrs)
    M = 4 if concave else 1
    for e in range(min(len(recs), 3)):
      want = span_overflow.restate(W, H, aa, recs[e], constants.SHAPES, M)
      got = span_overflow.restate(W, H, aa, recs[e], constants.SHAPES, M, window=(0.0, 0.0, 1.0, 1.0))
      assert got == want, (cid, e, got, want)
      n_flagged += bool(span_overflow.conditions(want, M, 16))
  assert n_flagged > 0


def test_bands_and_scratch_match_the_layout():
  # one band of 64 rows at aa 5: canvas rows 0..319; 100 rows: two bands that overlap
  assert span_overflow.bands(64, 5) == [(0, 320)]
  b = span_overflow.bands(100, 5)
  assert len(b) == 2 and b[0][0] == 0 and b[1][1] == 500 and b[1][0] < b[0][1]
  # RenderLayout::scratch_bytes at 64x64 aa 5 (convex and concave pools) and 128x128 aa 5
  assert span_overflow.phase_b_scratch(64, 64, 5, 1) == 22848
  assert span_overflow.phase_b_scratch(64, 64, 5, 4) == 25600
  assert span_overflow.phase_b_scratch(128, 128, 5, 1) == 35136
  assert [span_overflow.segcap(S, 1) for S in (1, 2, 9, 32)] == [3, 3, 17, 63]
  assert span_overflow.segcap(32, 1, exact=False) == 16 and span_overflow.segcap(2, 4) == 16
  m = dict(crossings=8, spans=1, pieces=6)
  assert span_overflow.describe(m, 1, 5) == 'crossings 8/8, spans 1/1, pieces 6/5'
  assert span_overflow.conditions(m, 1, 5) == ('pieces',) and span_overflow.conditions(m, 4, 16) == ()
