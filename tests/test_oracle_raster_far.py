"""Pins the oracle's Pillow stages (oracle/sw_raster_oracle.c) against the installed Pillow on
sprites whose canvas coordinates go far past int16, up to 2^30, and checks that the scenes of
tests/test_gpu_render_far.py reach what the render kernel's 16-bit packing special-cases.

  * oracle.polygon_fill against ImageDraw.polygon for the 12 Spriteworld shapes with vertex
    magnitudes in [2^15, 2^16), [2^16, 2^24) and [2^24, 2^30): huge sprites whose outline crosses
    the canvas, long thin sprites with one far vertex, and sprites wholly off the canvas on each
    side, on canvases of 64, 320, 2560 and 4095 pixels a side.  Above 2^24 the edge walk's float
    (y - y0) * dx rounds; at 2^30 x1 - x0 could overflow int32 in Pillow's C code, so the bands
    stop below it.
  * oracle.render (polygon fill and LANCZOS) against Pillow's resize(LANCZOS) for whole frames
    of such scenes at anti_aliasing 1, 5 and 10.
  * test_far_scenes_reach_the_int16_special_cases recomputes, from the GPU scenes, edges that
    cross the canvas from beyond +-32768 rows, horizontal edges on a canvas row with ends beyond
    +-32768 columns, corner joins on a canvas row whose edges end beyond int16, and sprites
    covering the whole canvas that phase B takes in chunks.
"""
import numpy as np
import pytest

from oracle import oracle
from tests import fixtures, mask_oracle
from tests import test_gpu_render_far as far
from tests import test_gpu_render_geometry as geo

PIL = pytest.importorskip('PIL')
from PIL import Image, ImageDraw  # noqa: E402

INT16 = far.INT16
BANDS = ((1 << 15, 1 << 16), (1 << 16, 1 << 24), (1 << 24, 1 << 30))
# (W, H) canvases, every side of 64, 320, 2560 and 4095 pixels among them
CANVASES = ((64, 64), (320, 320), (2560, 64), (64, 2560), (4095, 320), (320, 4095), (2560, 2560),
            (4095, 64), (64, 4095))
SIDES = ('left', 'right', 'above', 'below')


def _pil_polygon(w, h, xy, rgb):
  im = Image.new('RGB', (w, h))
  ImageDraw.Draw(im).polygon([tuple(v) for v in xy], fill=tuple(rgb))
  return np.array(im)


def _rotate(v, ang):
  c, s = np.cos(np.radians(ang)), np.sin(np.radians(ang))
  return v @ np.array([[c, s], [-s, c]])


def _magnitude(xy):
  return float(np.abs(np.trunc(xy)).max())


def _in_band(xy, band):
  return band[0] <= _magnitude(xy) < band[1]


def _crossing(rng, verts, w, h, band):
  """A sprite a random magnitude of `band` across with a random point of one of its edges inside
  the canvas."""
  for _ in range(100):
    m = float(np.exp(rng.uniform(np.log(band[0]), np.log(band[1]))))
    v = _rotate(verts, rng.uniform(0, 360))
    v = v * (m / np.abs(v).max() / 2 * rng.uniform(1.0, 2.0))
    i, t = rng.randint(len(v)), rng.rand()
    p = v[i] + t * (v[(i + 1) % len(v)] - v[i])
    xy = v - p + rng.uniform(0, 1, 2) * (w, h)
    if _in_band(xy, band):
      return xy
  raise AssertionError(('no crossing sprite in', band))


def _thin(rng, verts, w, h, band):
  """An ordinary sprite on the canvas with one vertex moved out to a magnitude of `band`: two
  long edges meeting far away."""
  for _ in range(100):
    v = _rotate(verts, rng.uniform(0, 360)) * rng.uniform(0.05, 0.5) * min(w, h)
    xy = v + rng.uniform(0.2, 0.8, 2) * (w, h)
    m = float(np.exp(rng.uniform(np.log(band[0]), np.log(band[1]))))
    d = rng.uniform(0, 2 * np.pi)
    xy[rng.randint(len(xy))] = (m * np.cos(d), m * np.sin(d))
    if _in_band(xy, band):
      return xy
  raise AssertionError(('no thin sprite in', band))


def _off(rng, verts, w, h, band, side):
  """A sprite wholly off the canvas on `side`, its far vertices at a magnitude of `band`; one
  time in three just clear of the canvas edge."""
  for _ in range(100):
    m = float(np.exp(rng.uniform(np.log(band[0]), np.log(band[1]))))
    v = _rotate(verts, rng.uniform(0, 360))
    v = v * (m * rng.uniform(0.1, 1.0) / np.abs(v).max() / 2)
    lo, hi = np.trunc(v.min(0)), np.trunc(v.max(0))
    gap = 1.0 if rng.rand() < 1 / 3 else float(np.exp(rng.uniform(0, np.log(m))))
    pos = rng.uniform(-0.5, 1.5, 2) * (w, h)
    if side == 'left':
      pos[0] = -hi[0] - gap
    elif side == 'right':
      pos[0] = w - lo[0] + gap
    elif side == 'above':
      pos[1] = -hi[1] - gap
    else:
      pos[1] = h - lo[1] + gap
    xy = v + np.trunc(pos)
    iv = np.trunc(xy)
    off = {'left': iv[:, 0].max() < 0, 'right': iv[:, 0].min() >= w,
           'above': iv[:, 1].max() < 0, 'below': iv[:, 1].min() >= h}[side]
    if off and _in_band(xy, band):
      return xy
  raise AssertionError(('no off-canvas sprite in', band, side))


def test_polygon_fill_matches_pillow_far_spriteworld_shapes():
  shapes, _ = fixtures.render_cases()
  rng = np.random.RandomState(2024)
  n, n_drawn, n_canvases = 0, 0, set()
  for si, (name, verts) in enumerate(shapes.items()):
    for bi, band in enumerate(BANDS):
      kinds = [('cross', None)] * 2 + [('thin', None)] * 2 + [('off', s) for s in SIDES]
      for ki, (kind, side) in enumerate(kinds):
        w, h = CANVASES[(si + 3 * bi + ki) % len(CANVASES)]
        n_canvases.update((w, h))
        if kind == 'cross':
          xy = _crossing(rng, verts, w, h, band)
        elif kind == 'thin':
          xy = _thin(rng, verts, w, h, band)
        else:
          xy = _off(rng, verts, w, h, band, side)
        ref = _pil_polygon(w, h, xy, (9, 200, 77))
        got = oracle.polygon_fill(np.zeros((h, w, 3), np.uint8), xy, (9, 200, 77))
        assert np.array_equal(got, ref), (name, band, kind, side, w, h, xy.tolist())
        n += 1
        n_drawn += bool(ref.any())
        if kind == 'off':
          assert not ref.any(), (name, band, side, w, h)
  assert n == 12 * 3 * 8 and n_canvases == {64, 320, 2560, 4095}
  # the crossing and thin sprites draw on the canvas (not every one covers a pixel centre)
  assert n_drawn >= 0.8 * 12 * 3 * 4, n_drawn


# (W, H, aa, bg, S, E, pool, kind) of whole frames
FRAMES = [
    (64, 64, 1, (0, 0, 0), 9, 3, 'all', 'far'),
    (41, 33, 1, (200, 10, 30), 5, 3, 'convex', 'huge'),
    (64, 64, 5, (255, 255, 255), 9, 3, 'all', 'far'),
    (33, 17, 5, (90, 90, 90), 5, 3, 'all', 'huge'),
    (64, 64, 10, (5, 6, 7), 9, 2, 'convex', 'far'),
    (100, 20, 10, (0, 0, 255), 5, 2, 'all', 'huge'),
]


def _pillow_frame(W, H, aa, bg, tab, sprites):
  """PILRenderer's frame with Pillow: every sprite drawn on the aa-times larger canvas at the
  vertices the oracle computes, resize((W, H), LANCZOS), np.flipud."""
  rc = oracle.raster_cfg(W, H, aa)
  im = Image.new('RGB', (aa * W, aa * H), tuple(bg))
  draw = ImageDraw.Draw(im)
  for sp in sprites:
    if sp['shape']:
      draw.polygon([tuple(v) for v in mask_oracle.canvas_vertices(rc, tab, sp)],
                   fill=tuple(int(c) for c in sp['rgb']))
  return np.flipud(np.array(im.resize((W, H), Image.LANCZOS)))


def test_render_matches_pillow_on_far_scenes():
  from spriteworld_b200 import constants
  tab = oracle.shape_table(constants.SHAPES)
  seen_aa = set()
  for W, H, aa, bg, S, E, pool, kind in FRAMES:
    rng = np.random.RandomState(W * H + aa)
    shapes = far.ALL_SHAPES if pool == 'all' else far.CONVEX
    if kind == 'huge':
      a = far.far_scene_arrays(rng, E, S, aa * W, aa * H, shapes, (40000, 120000),
                               kinds=('cross',), side=aa * H, p_small=0)
    else:
      a = far.far_scene_arrays(rng, E, S, aa * W, aa * H, shapes, (far.INT16, far.LIMIT / 2))
    rec = fixtures.records_from_arrays(a)
    rc = oracle.raster_cfg(W, H, aa, bg)
    assert far.INT16 < far.max_canvas_coordinate(('', W, H, aa), rec) < far.LIMIT
    for e in range(E):
      got = oracle.render(rc, tab, rec[e])
      ref = _pillow_frame(W, H, aa, bg, tab, rec[e])
      assert np.array_equal(got, ref), (W, H, aa, kind, e, int((got != ref).any(-1).sum()))
    seen_aa.add(aa)
  assert seen_aa == {1, 5, 10}


# ---------------------------------------------------------------------------------------
# what the scenes of tests/test_gpu_render_far.py reach
# ---------------------------------------------------------------------------------------

def _f32_x_at(y, y0, dx, x0):
  """Pillow's edge walk: float32 (y - y0) * dx, plus float32 x0."""
  return np.float32(np.float32(y - y0) * dx) + np.float32(x0)


def _roundf(v):
  return np.sign(v) * np.floor(np.abs(v) + np.float32(0.5))


def sprite_paths(iv, CW, CH):
  """What phase A of the render kernel meets for one sprite of integer vertices iv (n, 2): the
  set of int16 special cases it reaches."""
  x0, y0 = iv[:, 0], iv[:, 1]
  x1, y1 = np.roll(x0, -1), np.roll(y0, -1)
  n = len(iv)
  exists = np.ones(n, bool)
  exists[-1] = x0[-1] != x0[0] or y0[-1] != y0[0]
  scanned = exists & (y0 != y1)
  ymin, ymax = np.minimum(y0, y1), np.maximum(y0, y1)
  out = set()
  # edges whose rows cross the canvas from beyond the int16 range
  crosses = scanned & (ymin < CH) & (ymax >= 0)
  if (crosses & (ymin < -INT16)).any():
    out.add('edge_from_below_int16')
  if (crosses & (ymax > INT16 - 1)).any():
    out.add('edge_to_above_int16')
  # horizontal edges drawn on a canvas row, their ends beyond +-32768 columns
  hl = exists & (y0 == y1) & (y0 >= 0) & (y0 < CH)
  lo, hi = np.minimum(x0, x1), np.maximum(x0, x1)
  if (hl & ((lo < -INT16) | (hi > INT16 - 1))).any():
    out.add('hline_end_beyond_int16')
  if (hl & (lo < -INT16) & (hi > INT16 - 1)).any():
    out.add('hline_both_ends_beyond_int16')
  # corner joins (csrc/swb_render.cuh phase A, oracle/sw_raster_oracle.c): edge i and an earlier
  # edge k with slopes of one sign both starting on canvas row y, or both ending on the
  # polygon's last row, their crossings there rounding alike
  dx = np.zeros(n, np.float32)
  dx[scanned] = (x1 - x0)[scanned].astype(np.float32) / (y1 - y0)[scanned].astype(np.float32)
  p_ymax = min(max(0, int(y0.max())), CH)
  for i in np.flatnonzero(scanned):
    for start in (True, False):
      y = int(ymin[i]) if start else p_ymax
      if not (0 <= y < CH) or (not start and ymax[i] != p_ymax):
        continue
      for k in np.flatnonzero(scanned[:i]):
        if np.sign(dx[k]) != np.sign(dx[i]) or dx[i] == 0:
          continue
        if (ymin[k] if start else ymax[k]) != y:
          continue
        if _roundf(_f32_x_at(y, y0[i], dx[i], x0[i])) != _roundf(_f32_x_at(y, y0[k], dx[k], x0[k])):
          continue
        far_end = (ymax[[i, k]] > INT16 - 1) if start else (ymin[[i, k]] < -INT16)
        if far_end.any():
          out.add('corner_join_%s_beyond_int16' % ('start' if start else 'end'))
        break
  # a bounding box over the whole canvas
  if x0.min() <= 0 and x0.max() >= CW - 1 and y0.min() <= 0 and y0.max() >= CH - 1:
    out.add('covers_canvas')
  return out



def test_far_scenes_reach_the_int16_special_cases():
  paths = set()
  cases = list(far.CASES) + [(cid, W, H, 1, (0, 0, 0), S, E, concave, kind)
                             for cid, W, H, S, E, concave, kind in far.MASK_CASES]
  for case in cases:
    cid, W, H, aa, bg, S, E, concave, kind = case
    rec = fixtures.records_from_arrays(far.case_arrays(case))
    CW, CH = W * aa, H * aa
    assert far.max_canvas_coordinate(case, rec) < far.LIMIT, cid
    for e in range(E):
      for s, iv in far.canvas_int_vertices(case, rec[e]):
        for p in sprite_paths(iv, CW, CH):
          paths.add(p)
          paths.add('%s_%s' % (p, 'wide' if aa >= far.WIDE_AA else 'narrow'))
      if aa < far.WIDE_AA and geo.phase_b_chunked(W, H, aa, concave, rec[e]):
        paths.add('phase_b_chunked_%s' % ('concave' if concave else 'convex'))
  need = {'edge_from_below_int16', 'edge_to_above_int16', 'hline_end_beyond_int16',
          'hline_both_ends_beyond_int16', 'corner_join_start_beyond_int16',
          'corner_join_end_beyond_int16', 'covers_canvas', 'phase_b_chunked_convex',
          'phase_b_chunked_concave'}
  need |= {'%s_%s' % (p, w) for p in ('edge_from_below_int16', 'edge_to_above_int16',
                                      'hline_end_beyond_int16', 'corner_join_start_beyond_int16',
                                      'covers_canvas') for w in ('narrow', 'wide')}
  assert need <= paths, sorted(need - paths)


def test_sprite_paths_on_known_polygons():
  # a triangle from far above to far below the canvas, its apex on row 10
  iv = np.array([[30, 10], [50000, 40000], [-20000, -40000]])
  assert {'edge_from_below_int16', 'edge_to_above_int16', 'covers_canvas'} <= sprite_paths(iv, 64, 64)
  # a huge square at angle 0 whose top edge lies on canvas row 5
  iv = np.array([[100000, 5], [-100000, 5], [-100000, 200005], [100000, 200005]])
  p = sprite_paths(iv, 64, 64)
  assert 'hline_both_ends_beyond_int16' in p and 'covers_canvas' not in p
  # an acute corner on row 3 whose edges both run down to the right, ending beyond int16
  iv = np.array([[10, 3], [200000, 40000], [100000, 40000]])
  assert 'corner_join_start_beyond_int16' in sprite_paths(iv, 64, 64)
  # its mirror image on the last row of a polygon that ends on the canvas
  iv = np.array([[10, 60], [200000, -40000], [100000, -40000]])
  assert 'corner_join_end_beyond_int16' in sprite_paths(iv, 64, 64)
