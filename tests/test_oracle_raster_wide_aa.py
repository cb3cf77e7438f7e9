"""The oracle's two Pillow stages and the render kernel's resampling tables at anti_aliasing 6
and more (CPU tier):
  * oracle.render against the reference's own frames (tests/golden/wide_aa/, written by
    tests/golden/make_golden_wide_aa.py);
  * the oracle against Pillow's Image.resize(LANCZOS) and ImageDraw.polygon on the canvases of
    tests/test_gpu_render_wide_aa.py's sweep;
  * swb_tables.h through tests/native/check_vfrag_wide.cpp: vertical-pass fragments against the
    direct convolution, prefix tables, k-steps and tile blocks per factor.
"""
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import oracle
from tests import fixtures
from tests.test_gpu_render_wide_aa import CASES, REFUSED, tile_blocks, v_nks, wide_render_cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# (output width, output height, anti_aliasing) of the sweep's rendered cases and of the golden file
SWEEP_GEOMETRIES = sorted({(c[1], c[2], c[3]) for c in CASES if c[0] not in REFUSED} |
                          {(64, 64, a) for a in (11, 12)} | {(72, 40, 9)})


def test_render_matches_reference_frames_wide_aa():
  shapes, cases = wide_render_cases()
  tab = oracle.shape_table(shapes)
  assert {m['aa'] for m, _, _ in cases} >= {6, 7, 8, 9, 10, 13, 20}
  for meta, arrs, frame in cases:
    rc = oracle.raster_cfg(meta['width'], meta['height'], meta['aa'], meta['bg'])
    got = oracle.render(rc, tab, fixtures.records_from_arrays(arrs))
    assert got.shape == frame.shape, meta['name']
    assert np.array_equal(got, frame), (meta['name'], int((got != frame).sum()))


PIL = pytest.importorskip('PIL')
from PIL import Image, ImageDraw  # noqa: E402


def test_lanczos_matches_pillow_wide_aa():
  rng = np.random.RandomState(31)
  for t, (o, oh, aa) in enumerate(SWEEP_GEOMETRIES * 2):
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


def test_polygon_fill_matches_pillow_wide_aa():
  shapes, _ = fixtures.render_cases()
  rng = np.random.RandomState(77)
  for name, verts in shapes.items():
    for o, oh, aa in SWEEP_GEOMETRIES:
      w, h = o * aa, oh * aa
      for _ in range(2):
        s = float(np.exp(rng.uniform(np.log(0.001), np.log(2.0))))
        ang = 45.0 * rng.randint(8) if rng.rand() < 0.5 else rng.uniform(0, 360)
        c, sn = math.cos(math.radians(ang)), math.sin(math.radians(ang))
        pos = rng.uniform(-0.2, 1.2, 2)
        xy = ((verts * s) @ np.array([[c, sn], [-sn, c]]) + pos) * np.array([w, h])
        im = Image.new('RGB', (w, h))
        ImageDraw.Draw(im).polygon([tuple(v) for v in xy], fill=(255, 0, 255))
        got = oracle.polygon_fill(np.zeros((h, w, 3), np.uint8), xy, (255, 0, 255))
        assert np.array_equal(got, np.array(im)), (name, w, h, s, ang, pos)


def _cuda_include():
  for d in (os.environ.get('CUDA_HOME'), '/usr/local/cuda'):
    if d and os.path.exists(os.path.join(d, 'include', 'cuda_runtime.h')):
      return os.path.join(d, 'include')
  return None


def test_wide_vertical_fragments_and_tables(tmp_path):
  cxx, inc = shutil.which('g++'), _cuda_include()
  if not cxx or not inc:
    pytest.skip('needs g++ and the CUDA headers')
  exe = str(tmp_path / 'check_vfrag_wide')
  src = os.path.join(ROOT, 'tests', 'native', 'check_vfrag_wide.cpp')
  build = subprocess.run([cxx, '-std=c++17', '-O1', '-I', inc, '-o', exe, src], capture_output=True, text=True)
  assert build.returncode == 0, build.stderr[-2000:]
  run = subprocess.run([exe], capture_output=True, text=True, timeout=300)
  assert run.returncode == 0, run.stdout + run.stderr
  pat = re.compile(r'(\d+) -> (\d+): aa (\d+), window (\d+), prefix stride (\d+), k-steps (\d+), '
                   r'tile blocks (\d+), one-block span (\d+), classes \d+, prefix errors (\d+), '
                   r'mismatches (\d+)$')
  rows = [tuple(map(int, m.groups())) for m in map(pat.match, run.stdout.splitlines()) if m]
  assert len(rows) >= 20, run.stdout
  seen = set()
  for n_in, n_out, aa, win, stride, nks, tb, span, perr, bad in rows:
    assert perr == 0 and bad == 0, (n_out, aa)
    assert n_in == n_out * aa and stride == win + 1
    assert win <= 6 * aa
    # the C++ tables and the Python restatement the GPU sweep is planned with agree
    assert (nks, tb) == (v_nks(n_out, aa), tile_blocks(n_out, aa)), (n_out, aa)
    assert (tb == 0) == (span > 176), (n_out, aa)
    seen.add((n_out, aa, tb, nks))
  # the table of the factors: (tile blocks, k-steps) of 64- and 100-row frames
  want = {6: (3, 3), 7: (2, 3), 8: (2, 4), 9: (1, 4), 10: (1, 5), 11: (1, 5), 12: (1, 5),
          13: (1, 6), 14: (0, 6)}
  for aa, (tb, nks) in want.items():
    assert {(64, aa, tb, nks), (100, aa, tb, nks)} <= seen, aa
  assert (8, 20, 3, 5) in seen and (315, 13, 1, 6) in seen
