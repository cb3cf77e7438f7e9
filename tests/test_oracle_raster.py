"""Pins the oracle's two Pillow stages (oracle/sw_raster_oracle.c):
  * against the installed Pillow, differentially (Pillow is where the reference's pixels
    are decided: pil_renderer.py:83-84);
  * against frames produced by the reference itself (tests/golden/render_cases.npz);
  * against the literals in the reference's own tests/renderers/pil_renderer_test.py.
"""
import math

import numpy as np
import pytest

from oracle import oracle
from tests import fixtures

# (output width, output height, anti_aliasing) of tests/test_gpu_render_geometry.py's sweep:
# frames with short bands, partial blocks, column tails and canvas sides of 4095 pixels
SWEEP_GEOMETRIES = ((33, 17, 3), (50, 50, 5), (64, 65, 5), (64, 100, 5), (36, 70, 3),
                    (7, 130, 4), (101, 30, 2), (1, 1, 1), (1, 1, 5), (2, 3, 5), (819, 8, 5),
                    (8, 819, 5))
# Image.resize shrinks an image more than 100 times taller than wide vertically first: the
# oracle follows that rule on both sides of the H = 100 W boundary
TALL_GEOMETRIES = ((8, 819, 5), (8, 1023, 4), (8, 1300, 3), (1, 101, 2), (1, 150, 3),
                   (2, 250, 2), (3, 400, 5), (4, 401, 3), (1, 200, 5), (1, 100, 3), (8, 800, 5))

PIL = pytest.importorskip('PIL')
from PIL import Image, ImageDraw  # noqa: E402


def _pil_polygon(w, h, xy, rgb):
  im = Image.new('RGB', (w, h))
  ImageDraw.Draw(im).polygon([tuple(v) for v in xy], fill=tuple(rgb))
  return np.array(im)


def test_lanczos_golden_vector():
  # SURVEY.md App. B: interior tap vector for 320->64 and 640->128, xmin = 5*xx - 12
  golden = [3986, 14634, 24820, 23080, 0, -44124, -94487, -123412, -99278, 0, 174543,
            397113, 618288, 781320, 841337, 781320, 618288, 397113, 174543, 0, -99278,
            -123412, -94487, -44124, 0, 23080, 24820, 14634, 3986, 0]
  for n_in, n_out in ((320, 64), (640, 128)):
    bounds, kk = oracle.lanczos_coeffs(n_in, n_out)
    for xx in range(3, n_out - 3):
      assert bounds[xx, 0] == 5 * xx - 12 and bounds[xx, 1] == 30
      assert kk[xx, :30].tolist() == golden
    assert bounds[0].tolist() == [0, 18] and bounds[1].tolist() == [0, 23]
    assert bounds[2].tolist() == [0, 28]
    assert [int(b) for b in bounds[-3:, 1]] == [27, 22, 17]


def test_lanczos_matches_pillow():
  rng = np.random.RandomState(3)
  for t in range(24):
    o = int(rng.choice([16, 64, 128, 37]))
    aa = int(rng.choice([2, 3, 5, 5, 5, 4, 7]))
    oh = o if rng.rand() < .6 else int(rng.choice([16, 64, 24]))
    w, h = o * aa, oh * aa
    if t % 2:
      img = rng.randint(0, 256, (h, w, 3)).astype(np.uint8)
    else:
      img = np.zeros((h, w, 3), np.uint8)
      for _ in range(6):
        x0, y0 = rng.randint(0, w), rng.randint(0, h)
        img[y0:y0 + rng.randint(1, h), x0:x0 + rng.randint(1, w)] = rng.randint(0, 256, 3)
    ref = np.array(Image.fromarray(img).resize((o, oh), Image.LANCZOS))
    assert np.array_equal(oracle.lanczos_resize(img, o, oh), ref)
  for t, (o, oh, aa) in enumerate((SWEEP_GEOMETRIES + TALL_GEOMETRIES) * 2):
    w, h = o * aa, oh * aa
    if t % 2:
      img = rng.randint(0, 256, (h, w, 3)).astype(np.uint8)
    else:   # saturated rectangles: the LANCZOS overshoot clips at both ends
      img = np.full((h, w, 3), 255 * (t % 4 == 0), np.uint8)
      for _ in range(6):
        x0, y0 = rng.randint(0, w), rng.randint(0, h)
        img[y0:y0 + rng.randint(1, h + 1), x0:x0 + rng.randint(1, w + 1)] = 255 * rng.randint(0, 2, 3)
    ref = np.array(Image.fromarray(img).resize((o, oh), Image.LANCZOS))
    assert np.array_equal(oracle.lanczos_resize(img, o, oh), ref), (o, oh, aa)


def test_polygon_fill_matches_pillow_spriteworld_shapes():
  shapes, _ = fixtures.render_cases()
  rng = np.random.RandomState(123)
  n_without = 0
  for name, verts in shapes.items():
    for _ in range(250):
      w = int(rng.choice([64, 320, 640]))
      h = w if rng.rand() < 0.7 else int(rng.choice([64, 320, 640]))
      s = float(np.exp(rng.uniform(np.log(0.005), np.log(0.6))))
      ang = rng.uniform(0, 360) if rng.rand() < 0.7 else float(rng.randint(0, 360))
      c, sn = math.cos(math.radians(ang)), math.sin(math.radians(ang))
      pos = rng.uniform(-0.1, 1.1, 2)
      xy = ((verts * s) @ np.array([[c, sn], [-sn, c]]) + pos) * np.array([w, h])
      ref = _pil_polygon(w, h, xy, (9, 200, 77))
      got = oracle.polygon_fill(np.zeros((h, w, 3), np.uint8), xy, (9, 200, 77))
      assert np.array_equal(got, ref), (name, w, h, s, ang, pos)
      plain = oracle.polygon_fill(np.zeros((h, w, 3), np.uint8), xy, (9, 200, 77),
                                  corner_join=0)
      n_without += not np.array_equal(plain, ref)
    # the canvases of the render sweep, angles on multiples of 45 degrees half of the time
    for o, oh, aa in SWEEP_GEOMETRIES:
      w, h = o * aa, oh * aa
      for _ in range(4):
        s = float(np.exp(rng.uniform(np.log(0.001), np.log(2.0))))
        ang = 45.0 * rng.randint(8) if rng.rand() < 0.5 else rng.uniform(0, 360)
        c, sn = math.cos(math.radians(ang)), math.sin(math.radians(ang))
        pos = rng.uniform(-0.2, 1.2, 2)
        xy = ((verts * s) @ np.array([[c, sn], [-sn, c]]) + pos) * np.array([w, h])
        ref = _pil_polygon(w, h, xy, (255, 0, 255))
        got = oracle.polygon_fill(np.zeros((h, w, 3), np.uint8), xy, (255, 0, 255))
        assert np.array_equal(got, ref), (name, w, h, s, ang, pos)
  # the corner-joining refinement is not optional: some instances need it
  assert n_without > 0


def test_polygon_fill_matches_pillow_random_polygons():
  rng = np.random.RandomState(9)
  bad = 0
  n = 4000
  sweep = [d * aa for o, oh, aa in SWEEP_GEOMETRIES for d in (o, oh)]
  for i in range(n):
    w, h = int(rng.choice([16, 64, 320])), int(rng.choice([16, 64, 320]))
    if i % 8 == 7:   # every eighth polygon on a canvas of the render sweep
      w, h = int(rng.choice(sweep)), int(rng.choice(sweep))
    kind, nv = rng.randint(3), rng.randint(3, 10)
    if kind == 0:  # convex, float coordinates, partly off canvas
      ang = np.sort(rng.uniform(0, 2 * np.pi, nv))
      r, c = rng.uniform(0.05, 0.6) * w, rng.uniform(-0.1, 1.1, 2) * w
      xy = np.stack([c[0] + r * np.cos(ang), c[1] + r * np.sin(ang)], 1)
    elif kind == 1:  # star-like simple polygons on integer coordinates
      ang = np.sort(rng.uniform(0, 2 * np.pi, nv))
      r, c = rng.uniform(0.05, 0.6, nv) * w, rng.uniform(0, 1, 2) * w
      xy = np.floor(np.stack([c[0] + r * np.cos(ang), c[1] + r * np.sin(ang)], 1))
    else:  # arbitrary (self-intersecting)
      xy = rng.uniform(-0.2, 1.2, (nv, 2)) * np.array([w, h])
    ref = _pil_polygon(w, h, xy, (1, 2, 3))
    got = oracle.polygon_fill(np.zeros((h, w, 3), np.uint8), xy, (1, 2, 3))
    bad += not np.array_equal(got, ref)
  # Residual: zero-area spikes made of exactly repeated vertices (never produced by
  # Spriteworld shapes) -- see DESIGN.md.  Everything else is bit-exact.
  assert bad <= n // 1000, bad


def test_render_matches_reference_frames():
  shapes, cases = fixtures.render_cases()
  tab = oracle.shape_table(shapes)
  for meta, arrs, frame in cases:
    rec = fixtures.records_from_arrays(arrs)
    rc = oracle.raster_cfg(meta['width'], meta['height'], meta['aa'], meta['bg'])
    got = oracle.render(rc, tab, rec)
    assert got.shape == frame.shape, meta['name']
    assert np.array_equal(got, frame), (meta['name'], int(np.abs(
        got.astype(int) - frame.astype(int)).max()))


def test_reference_renderer_test_literals():
  """tests/renderers/pil_renderer_test.py:49-88 expectations, on the oracle's output."""
  shapes, cases = fixtures.render_cases()
  tab = oracle.shape_table(shapes)
  by_name = {m['name']: (m, a) for m, a, _ in cases}

  def rend(name):
    meta, arrs = by_name[name]
    rc = oracle.raster_cfg(meta['width'], meta['height'], meta['aa'], meta['bg'])
    return oracle.render(rc, tab, fixtures.records_from_arrays(arrs))

  assert list(rend('ref_test_bg_64')[5, 5]) == [5, 6, 7]                      # :49-53
  img = rend('ref_test_basic_64')                                             # :55-59
  assert list(img[32, 32]) == [255, 0, 0] and list(img[32, 50]) == [0, 255, 0]
  img = rend('ref_test_aa5_16')                                               # :61-72
  assert list(img[4, 6]) == [0, 0, 0] and list(img[6, 6]) == [255, 0, 0]
  assert all(img[5, 6] >= [50, 0, 0]) and all(img[5, 6] <= [120, 30, 0])
  assert all(img[7, 6] >= [200, 0, 0]) and all(img[7, 6] <= [255, 50, 0])
  img = rend('ref_test_aa1_16')                                               # :74-78
  assert list(img[4, 6]) == [0, 0, 0] and list(img[6, 6]) == [255, 0, 0]
  assert list(img[7, 6]) == [255, 0, 0]
  assert list(rend('ref_test_hsv_64')[32, 32]) == [114, 127, 63]              # :80-88


def test_hsv_to_rgb_matches_colorsys():
  import colorsys
  rng = np.random.RandomState(0)
  for _ in range(20000):
    c = rng.uniform(0, 1, 3).astype(np.float32)
    ref = (255 * np.array(colorsys.hsv_to_rgb(*c))).astype(np.uint8)   # color_maps.py:28
    assert ref.dtype == np.uint8 and np.array(colorsys.hsv_to_rgb(*c)).dtype == np.float32
    assert np.array_equal(oracle.hsv_to_rgb(c[0], c[1], c[2], True), ref), c
    cd = [float(v) for v in rng.uniform(0, 1, 3)]
    refd = (255 * np.array(colorsys.hsv_to_rgb(*cd))).astype(np.uint8)
    assert np.array_equal(oracle.hsv_to_rgb(cd[0], cd[1], cd[2], False), refd), cd
  assert list(oracle.hsv_to_rgb(1.0, 0.0, 1.0, False)) == [255, 255, 255]
