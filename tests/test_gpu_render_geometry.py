"""Render kernel (csrc/swb_render.cuh) against the CPU oracle over the geometry the kernel
branches on: raster sizes whose bands, 8-row blocks and column tiles end short, frames whose
bands take the per-byte write-out instead of the bulk copy (and launches that mix the two),
slot counts up to 32, concave shapes in the pool, scenes built to hit the edges of scan
conversion and filtering, and enough envs that every persistent CTA claims several items.

Every frame buffer is a slice of a larger tensor pre-filled with a sentinel byte, so an
unwritten band or a stray store shows up instead of matching a background by chance; the
guard bytes on both sides must come back untouched.  Frames are compared bit-exact.

CASES is the sweep; test_case_table_covers_render_paths recomputes, from the host formulas of
swb_raster_create and check_render, which kernel paths each case reaches and fails if
the table stops covering one of them.
"""
import ctypes

import numpy as np
import pytest

from oracle import oracle
from tests import fixtures, span_overflow

SENTINEL = 0xA5
GUARD = 256                 # sentinel bytes on each side of a frame buffer; a multiple of 16
BAND_ROWS = 64              # swb_raster_create: output rows per band
R_CTAS_PER_SM = 5           # render CTAs resident per SM (SWB_RENDER_CTAS)
R_WARPS = 8                 # warps per render CTA: phase A gives each warp S / 8 sprites
H100_SMS = 132
CONVEX = tuple(range(1, 7))         # triangle .. circle
CONCAVE = tuple(range(7, 13))       # star_4 .. spoke_6

# (id, W, H, aa, bg, S, E, concave, scene).  E = None: enough envs that every CTA of the
# persistent grid claims about three (env, band) items (see _n_envs).
CASES = [
    # every item takes the per-byte write-out; grey background with n_bytes % 16 != 0 (u32 fill)
    ('w33h17a3', 33, 17, 3, (90, 90, 90), 9, 40, True, 'edges'),
    # per-byte write-out, non-grey background (byte fill)
    ('w50h50a5', 50, 50, 5, (10, 200, 30), 8, 40, False, 'edges'),
    # bands of 64 and 1 rows
    ('w64h65a5', 64, 65, 5, (0, 0, 0), 17, 40, True, 'edges'),
    # bands of 64 and 36 rows: a partial last block of eight rows
    ('w64h100a5', 64, 100, 5, (255, 255, 255), 32, 24, False, 'edges'),
    # bulk and per-byte items in one launch, every CTA claiming several items of unequal bands
    ('w36h70a3', 36, 70, 3, (0, 0, 255), 9, None, True, 'edges'),
    ('w7h130a4', 7, 130, 4, (255, 0, 0), 17, None, False, 'edges'),
    # W > 64: column tiles and H-pass column pairs with tails
    ('w101h30a2', 101, 30, 2, (40, 40, 40), 32, 40, True, 'edges'),
    ('w1h1a1', 1, 1, 1, (7, 7, 7), 1, 16, False, 'edges'),
    ('w1h1a5', 1, 1, 5, (0, 255, 0), 8, 16, True, 'edges'),
    ('w2h3a5', 2, 3, 5, (255, 255, 255), 1, 16, True, 'edges'),
    # canvas side at its limit of 4095 pixels
    ('w819h8a5', 819, 8, 5, (5, 6, 7), 8, 8, True, 'edges'),
    ('w41h819a5', 41, 819, 5, (5, 6, 7), 9, 8, False, 'edges'),
    # more than 100 times taller than wide: Pillow resizes vertically first, the kernel does not,
    # so aa > 1 is refused; H = 100 W, and any height at aa = 1 (no resize), still render
    ('w8h819a5', 8, 819, 5, (5, 6, 7), 9, 8, False, 'edges'),
    ('w1h101a2', 1, 101, 2, (5, 6, 7), 8, 8, True, 'edges'),
    ('w1h100a3', 1, 100, 3, (5, 6, 7), 8, 8, True, 'edges'),
    ('w1h150a1', 1, 150, 1, (5, 6, 7), 8, 8, False, 'edges'),
    # the exact segment table of 32 convex slots does not fit beside a 550-wide staged frame:
    # the launch falls back to 16 visible segments per canvas row instead of refusing
    ('w550h64a5', 550, 64, 5, (0, 0, 0), 32, 8, False, 'full'),
    ('w550h64a5_edges', 550, 64, 5, (0, 0, 0), 32, 8, False, 'edges'),
    # sprites that each span every canvas row: phase B works through the sprites in chunks
    ('full_convex', 64, 64, 5, (0, 0, 0), 9, 16, False, 'full'),
    ('full_concave', 64, 64, 5, (255, 255, 255), 17, 16, True, 'full'),
    # 17 visible pieces on one canvas row from nine convex sprites
    ('stripes', 64, 64, 5, (0, 0, 0), 9, 16, False, 'stripes'),
    ('stripes_h100', 64, 100, 5, (0, 0, 0), 9, 16, False, 'stripes'),
]
# Raster(...) refuses these with NativeError instead of rendering them
REFUSED = {'w8h819a5', 'w1h101a2'}
# cases whose segment table is capped at 16 although every shape is convex
SEGCAP_16 = {'w550h64a5', 'w550h64a5_edges'}
# known kernel defects the sweep has found and that are not fixed yet (case id -> xfail mark)
KNOWN_DEFECTS = {}


def _n_envs(case, n_sms):
  _, W, H, aa, bg, S, E, concave, scene = case
  if E is not None:
    return E
  n_bands = -(-H // min(H, BAND_ROWS))
  return -(-3 * n_sms * R_CTAS_PER_SM // n_bands)


# ---------------------------------------------------------------------------------------
# host formulas of swb_raster_create / check_render / enqueue_render / render_kernel phase D
# ---------------------------------------------------------------------------------------

def render_plan(W, H, S, E, n_sms=H100_SMS, base=0):
  """What one launch does: bands, items, grid and, per item, whether phase D can hand the band
  to the bulk copy (size and destination address multiples of 16).  `base`: the frame buffer's
  address modulo 16."""
  band_rows = H if H <= BAND_ROWS else BAND_ROWS
  n_bands = -(-H // band_rows)
  row_bytes = 3 * W
  heights = [min(band_rows, H - b * band_rows) for b in range(n_bands)]
  bulk = []
  for e in range(E):
    for b in range(n_bands):
      yo_b1 = min((b + 1) * band_rows, H)
      n_bytes = heights[b] * row_bytes
      band_off = e * H * row_bytes + (H - yo_b1) * row_bytes
      bulk.append(n_bytes % 16 == 0 and (base + band_off) % 16 == 0)
  n_items = E * n_bands
  return dict(n_bands=n_bands, heights=heights, n_items=n_items,
              grid=min(n_items, n_sms * R_CTAS_PER_SM), bulk=np.array(bulk),
              sprites_per_warp=-(-S // R_WARPS))


def test_case_table_covers_render_paths():
  paths = set()
  for case in CASES:
    cid, W, H, aa, bg, S, _, concave, scene = case
    if cid in REFUSED:
      assert aa > 1 and H > 100 * W, cid
      paths.add('refused_tall')
      continue
    if aa > 1 and H == 100 * W:
      paths.add('tall_boundary_renders')
    if cid in SEGCAP_16:
      paths.add('segcap_fallback')
    E = _n_envs(case, H100_SMS)
    p = render_plan(W, H, S, E)
    grey = bg[0] == bg[1] == bg[2]
    if not p['bulk'].any():
      paths.add('all_fallback')
    if p['bulk'].any() and not p['bulk'].all():
      paths.add('mixed_bulk_fallback')
    for h in p['heights']:
      if grey and (h * W * 3) % 16:
        paths.add('fill_u32')
      if not grey and not p['bulk'].all():
        paths.add('fill_bytes_fallback')
    if H % 8:
      paths.add('partial_block')
    if p['heights'][-1] == 1 and p['n_bands'] > 1:
      paths.add('one_row_band')
    if p['n_bands'] > 1 and p['heights'][-1] % 8 and p['heights'][-1] > 1:
      paths.add('short_band')
    if W > 64:
      paths.add('wide')
    if W * aa == 4095:
      paths.add('canvas_limit_w')
    if H * aa == 4095:
      paths.add('canvas_limit_h')
    if W * H == 1:
      paths.add('single_pixel_aa%d' % min(aa, 2))
    if p['n_items'] >= 3 * p['grid'] and len(set(p['heights'])) > 1 and not p['bulk'].all():
      paths.add('persistent_unequal_bands_mixed')
    paths.add('S%d_%s' % (S, 'concave' if concave else 'convex'))
    paths.add('sprites_per_warp_%d' % p['sprites_per_warp'])
    if scene == 'full' and all(phase_b_chunked(W, H, aa, concave, rec)
                               for rec in fixtures.records_from_arrays(case_arrays(case, E))):
      paths.add('phase_b_chunks_%s' % ('concave' if concave else 'convex'))
    if scene == 'stripes':
      paths.add('stripes_%s' % ('multiband' if p['n_bands'] > 1 else 'oneband'))
  need = {'all_fallback', 'mixed_bulk_fallback', 'fill_u32', 'fill_bytes_fallback',
          'partial_block', 'one_row_band', 'short_band', 'wide', 'canvas_limit_w',
          'canvas_limit_h', 'single_pixel_aa1', 'single_pixel_aa2',
          'persistent_unequal_bands_mixed', 'phase_b_chunks_concave', 'phase_b_chunks_convex',
          'stripes_oneband', 'stripes_multiband', 'refused_tall', 'tall_boundary_renders',
          'segcap_fallback'}
  need |= {'S%d_%s' % (s, k) for s in (1, 8, 9, 17, 32) for k in ('convex', 'concave')}
  need |= {'sprites_per_warp_%d' % k for k in (1, 2, 3, 4)}
  assert need <= paths, sorted(need - paths)
  # the geometries the sweep is there for
  sizes = {(c[1], c[2], c[3]) for c in CASES}
  assert {(33, 17, 3), (50, 50, 5), (64, 65, 5), (64, 100, 5), (36, 70, 3), (7, 130, 4),
          (101, 30, 2), (1, 1, 1), (1, 1, 5), (2, 3, 5), (819, 8, 5), (8, 819, 5)} <= sizes


def _axis_windows(n_in, n_out):
  """Per output: (first input, input count) of its LANCZOS window (swb_tables.h build_axis)."""
  bounds, _ = oracle.lanczos_coeffs(n_in, n_out)
  return bounds[:, 0], bounds[:, 1]


def phase_b_scratch(W, H, aa, concave):
  """RenderLayout::scratch_bytes: the H tile (or more, so that phase B can hold one sprite
  spanning every canvas row of a band) and the staged frame, each rounded to 16 bytes."""
  band_rows = min(H, BAND_ROWS)
  wmin, wlen = _axis_windows(H * aa, H)
  rows = max(int(wmin[min(y0 + band_rows, H) - 1] + wlen[min(y0 + band_rows, H) - 1]
                 - (wmin[y0] & ~3)) for y0 in range(0, H, band_rows))
  M, cap = (4, 16) if concave else (1, 8)
  r16 = lambda b: (b + 15) & ~15
  frame = band_rows * W * 3
  ht = 60 * 44 * 4                       # HT_WORDS words of the H tile
  if ht + r16(frame) < (cap + M) * 4 * rows:
    ht = (cap + M) * 4 * rows - frame
  return r16(ht) + r16(frame)


def phase_b_chunked(W, H, aa, concave, rec):
  """Whether phase B of band 0 takes this scene's sprites in several chunks: their crossing
  lists (CAP words per canvas row a sprite spans) and spans (M words per row of the band) do
  not fit the scratch area together."""
  from spriteworld_b200 import constants
  M, cap = (4, 16) if concave else (1, 8)
  CH = H * aa
  wmin, wlen = _axis_windows(CH, H)
  yo_b1 = min(H, BAND_ROWS)
  row_b0, row_b1 = int(wmin[0]) & ~3, int(wmin[yo_b1 - 1] + wlen[yo_b1 - 1])
  names = {v: k for k, v in oracle.SHAPE_IDS.items()}
  rows_all = 0
  for r in rec:
    if not r['shape']:
      continue
    v = np.asarray(constants.SHAPES[names[int(r['shape'])]], np.float64)
    ivy = np.trunc(CH * (((r['m10'] * v[:, 0] + r['m11'] * v[:, 1]) + 0.0) + r['y'])).astype(int)
    pymin, pymax = max(min(CH - 1, ivy.min()), 0), min(max(0, ivy.max()), CH)
    r0, r1 = max(pymin, row_b0), min(pymax, CH - 1, row_b1 - 1)
    rows_all += max(0, r1 - r0 + 1)
  need = rows_all * cap * 4 + len(rec) * (row_b1 - row_b0) * M * 4
  return need > phase_b_scratch(W, H, aa, concave)


def test_render_plan_matches_known_geometries():
  # 64x64 frames: one band, every item bulk; 128x128: two equal bands, every item bulk
  p = render_plan(64, 64, 5, 4096)
  assert p['n_bands'] == 1 and p['bulk'].all() and p['grid'] == 660
  p = render_plan(128, 128, 8, 4096)
  assert p['heights'] == [64, 64] and p['bulk'].all() and p['sprites_per_warp'] == 1
  # 36x70: bands of 64 and 6 rows; the 6-row band is never bulk, the 64-row band of odd envs is
  p = render_plan(36, 70, 9, 4)
  assert p['heights'] == [64, 6] and p['bulk'].tolist() == [False, False, True, False] * 2
  assert not render_plan(64, 64, 5, 4, base=1)['bulk'].any()
  # RenderLayout::scratch_bytes at 64x64 aa 5 (convex and concave pools) and 128x128 aa 5
  assert phase_b_scratch(64, 64, 5, False) == 22848 and phase_b_scratch(64, 64, 5, True) == 25600
  assert phase_b_scratch(128, 128, 5, False) == 35136


# ---------------------------------------------------------------------------------------
# scenes
# ---------------------------------------------------------------------------------------

def _f32(a):
  return np.asarray(a, np.float32).astype(np.float64)


def _empty_arrays(E, S):
  z = np.zeros((E, S))
  return dict(x=z.copy(), y=z.copy(), pos_f32=np.ones((E, S), np.uint8),
              shape=np.zeros((E, S), np.uint8), angle=z.copy(), scale=z.copy(),
              c0=z.copy(), c1=z.copy(), c2=z.copy(), vx=z.copy(), vy=z.copy(),
              member=np.zeros((E, S), np.uint32), rgb=np.zeros((E, S, 3), np.uint8))


def _pick_shapes(rng, size, concave):
  pool = CONVEX + CONCAVE if concave else CONVEX
  return rng.choice(pool, size)


def scene_edges(rng, E, S, bg, concave):
  """Per slot, at random: off-frame, on an edge or corner, or inside; sub-pixel, ordinary or
  larger than the frame; angles at multiples of 45 degrees half of the time; colour equal to
  the background, from {0, 255}^3, or random; some slots empty, some identical to the slot
  below them."""
  a = _empty_arrays(E, S)
  edge_pos = np.array([-0.3, -0.05, 0.0, 0.01, 0.99, 1.0, 1.05, 1.3])
  for e in range(E):
    for s in range(S):
      u = rng.rand()
      if u < 0.15 and s > 0:   # identical stacked sprite
        for k in a:
          a[k][e, s] = a[k][e, s - 1]
        continue
      kind = rng.randint(4)
      x, y = rng.uniform(-0.2, 1.2, 2)
      if kind == 1:
        x = rng.choice(edge_pos)
      elif kind == 2:
        y = rng.choice(edge_pos)
      elif kind == 3:
        x, y = rng.choice(edge_pos, 2)
      a['x'][e, s], a['y'][e, s] = _f32(x), _f32(y)
      v = rng.rand()
      a['scale'][e, s] = (rng.uniform(5e-4, 2e-3) if v < 0.1 else
                          rng.uniform(1.0, 2.5) if v < 0.2 else
                          np.exp(rng.uniform(np.log(0.02), np.log(0.4))))
      a['angle'][e, s] = 45.0 * rng.randint(8) if rng.rand() < 0.5 else float(rng.randint(360))
      a['shape'][e, s] = 0 if rng.rand() < 0.05 else _pick_shapes(rng, 1, concave)[0]
      c = rng.rand()
      a['rgb'][e, s] = (bg if c < 0.3 else 255 * rng.randint(0, 2, 3) if c < 0.6
                        else rng.randint(0, 256, 3))
  a['shape'][:, -1] = np.maximum(a['shape'][:, -1], 1)
  return a


def scene_full(rng, E, S, bg, concave):
  """Sprites taller than the frame, each covering every canvas row, at columns spread over
  and beyond the frame so that they overlap partly."""
  a = _empty_arrays(E, S)
  a['x'][:] = _f32(rng.uniform(-0.6, 1.6, (E, S)))
  a['y'][:] = _f32(rng.uniform(0.45, 0.55, (E, S)))
  a['scale'][:] = rng.uniform(1.2, 1.6, (E, S))
  a['angle'][:] = rng.randint(0, 360, (E, S))
  a['shape'][:] = rng.choice((2, 5, 6, 7, 8) if concave else (2, 5, 6), (E, S))
  a['rgb'][:] = 255 * rng.randint(0, 2, (E, S, 3))
  a['rgb'][:, ::3] = rng.randint(0, 256, a['rgb'][:, ::3].shape)
  return a


def stripes(n_inside, straddle, star, y=0.5):
  """Squares on one line in front of a large square: a square at scale 0.9 centred at
  (0.5, 0.5), behind n_inside squares at scale 0.05 on x = 0.1, 0.2, ... (or 0.2, 0.3, ...
  with a ninth square straddling the large square's left edge), y = `y`.  Every small square
  cuts the large one's pieces on the rows it covers: 2 n_inside + 1 (+ 1 for the straddling
  one) visible pieces.  `star`: one more slot, a small star far below the line."""
  xs = [0.1 * (i + 1) for i in range(n_inside)]
  if straddle:
    xs = [0.05] + [0.1 * (i + 2) for i in range(n_inside)]
  sl = [(0.5, 0.5, 2, 0.9, (200, 30, 90))] + [(x, y, 2, 0.05, (20 * i, 250, 10)) for i, x in enumerate(xs)]
  if star:
    sl = [(0.5, 0.1, 7, 0.05, (255, 255, 255))] + sl
  a = _empty_arrays(1, len(sl))
  for s, (x, yy, shape, scale, rgb) in enumerate(sl):
    a['x'][0, s], a['y'][0, s] = _f32(x), _f32(yy)
    a['shape'][0, s], a['scale'][0, s], a['rgb'][0, s] = shape, scale, rgb
  return a


def scene_stripes(rng, E, S, bg, concave):
  assert S == 9 and not concave
  rows = []
  for e in range(E):
    r = stripes(8, False, False, y=0.5 + rng.uniform(-0.3, 0.3))
    r['angle'][:] = 90.0 * rng.randint(0, 4, r['angle'].shape)
    r['rgb'][0, 1:] = rng.randint(0, 256, (S - 1, 3))
    rows.append(r)
  return {k: np.concatenate([r[k] for r in rows]) for k in rows[0]}


SCENES = dict(edges=scene_edges, full=scene_full, stripes=scene_stripes)


def case_arrays(case, E):
  """The scenes of a case, one per env (seeded by the case id)."""
  cid, W, H, aa, bg, S, _, concave, kind = case
  rng = np.random.RandomState(sum(map(ord, cid)))
  return _ensure_concave(SCENES[kind](rng, E, S, bg, concave), rng, concave)


def _ensure_concave(a, rng, concave):
  """An engine sizes its span tables for concave shapes once one is uploaded: make the pool
  contain one exactly when the case asks for it."""
  if concave and not np.isin(a['shape'], CONCAVE).any():
    a['shape'][0, 0] = CONCAVE[0]
  if not concave:
    assert not np.isin(a['shape'], CONCAVE).any()
  return a


def visible_pieces(W, H, aa, rec, shapes):
  """Most visible pieces on any canvas row (what the kernel's per-row segment table holds):
  the sprites scan-converted by the oracle's Pillow restatement onto a label canvas, back to
  front, and the runs of equal non-background labels counted per row."""
  CW, CH = W * aa, H * aa
  lab = np.zeros((CH, CW, 3), np.uint8)
  names = {v: k for k, v in oracle.SHAPE_IDS.items()}
  for s, r in enumerate(rec):
    if not r['shape']:
      continue
    v = np.asarray(shapes[names[int(r['shape'])]], np.float64)
    cx = (r['m00'] * v[:, 0] + r['m01'] * v[:, 1]) + 0.0
    cy = (r['m10'] * v[:, 0] + r['m11'] * v[:, 1]) + 0.0
    xy = np.stack([CW * (cx + r['x']), CH * (cy + r['y'])], 1)
    oracle.polygon_fill(lab, xy, (s + 1, 0, 0))
  L = lab[..., 0]
  starts = (L != 0) & np.concatenate([np.ones((CH, 1), bool), L[:, 1:] != L[:, :-1]], 1)
  return int(starts.sum(1).max())


def test_stripes_scenes_have_the_intended_piece_counts():
  from spriteworld_b200 import constants
  for n_inside, straddle, star, pieces in ((8, False, False, 17), (8, False, True, 17),
                                           (7, True, True, 16), (7, False, False, 15)):
    rec = fixtures.records_from_arrays(stripes(n_inside, straddle, star))[0]
    assert visible_pieces(64, 64, 5, rec, constants.SHAPES) == pieces, (n_inside, straddle)


# ---------------------------------------------------------------------------------------
# running the engine
# ---------------------------------------------------------------------------------------

def _guarded(n_bytes, device, skew=0):
  """A flat uint8 tensor of n_bytes filled with the sentinel, `skew` bytes past a 16-byte
  boundary, inside a larger tensor with GUARD sentinel bytes on both sides."""
  import torch
  big = torch.full((n_bytes + 2 * GUARD + 16,), SENTINEL, dtype=torch.uint8, device=device)
  pad = (-big.data_ptr()) % 16
  lo = GUARD + pad + skew
  return big, big[lo:lo + n_bytes], lo


def _assert_guards(big, lo, n_bytes, where):
  hi = lo + n_bytes
  assert bool((big[:lo] == SENTINEL).all()) and bool((big[hi:] == SENTINEL).all()), (
      where, 'store outside the frame buffer')


class Sweep(object):
  """One case: the engine with its scenes uploaded, and the oracle's frames of every env and
  the restated phase-B maxima (tests/span_overflow.py) that decide its status (each computed
  once, on first use).  `arrs` and `shapes`: scenes and shape table other than the case's own."""

  def __init__(self, case, n_sms, arrs=None, shapes=None):
    import torch
    from spriteworld_b200 import constants, engine, scene
    self.case = case
    cid, self.W, self.H, self.aa, self.bg, self.S, _, concave, kind = case
    self.E = E = _n_envs(case, n_sms)
    if arrs is None:
      arrs = case_arrays(case, E)
    shapes = constants.SHAPES if shapes is None else shapes
    self.M = 4 if concave else 1
    self.segcap = span_overflow.segcap(self.S, self.M, exact=cid not in SEGCAP_16)
    self.eng = engine.Engine(E, self.S, 1, dict(kind='select_move', scale=1.0),
                             [dict(kind='no_reward')], shapes, keep_in_frame=False)
    b = scene.batch_from_factor_arrays(
        arrs['x'], arrs['y'], arrs['pos_f32'], arrs['shape'], arrs['angle'], arrs['scale'],
        arrs['c0'], arrs['c1'], arrs['c2'], arrs['vx'], arrs['vy'], arrs['member'], arrs['rgb'])
    self.eng.upload_scenes(b, np.arange(E), np.zeros(E, int))
    self.eng.upload_state(pos_x=b['x'], pos_y=b['y'], cursor=np.zeros(E), step_count=np.zeros(E),
                          reset_next=np.zeros(E))
    self.pos = (b['x'].copy(), b['y'].copy())
    self.rec = fixtures.records_from_arrays(arrs)
    self.shapes = shapes
    self.tab = oracle.shape_table(shapes)
    self.rc = oracle.raster_cfg(self.W, self.H, self.aa, self.bg)
    self._ref, self._maxima = {}, {}
    self.actions = torch.full((E, 4), 0.5, dtype=torch.float32, device=self.eng.device)

  def ref(self, e):
    """The oracle's frame of env e, and the restated maxima of phase B's capacities."""
    if e not in self._ref:
      self._ref[e] = oracle.render(self.rc, self.tab, self.rec[e])
      self._maxima[e] = span_overflow.restate(self.W, self.H, self.aa, self.rec[e], self.shapes,
                                              self.M)
    return self._ref[e], self._maxima[e]

  def overflow(self, e):
    """The conditions that must flag env e under this sweep's span class and segment table."""
    return span_overflow.conditions(self.ref(e)[1], self.M, self.segcap)

  def within(self, e):
    return not self.overflow(e)

  def check(self, frames, status, where):
    """frames: (E, H, W, 3) uint8 numpy; status: (E,) uint8 numpy.  Every env is flagged
    exactly when the restatement says so; every other env has status 0 and the oracle's frame."""
    from spriteworld_b200 import _native
    over = (status & _native.ENV_SPAN_OVERFLOW) != 0
    n_exact = 0
    for e in range(self.E):
      ref, maxima = self.ref(int(e))
      want = self.overflow(int(e))
      assert over[e] == bool(want), (where, int(e), 'status %d' % status[e], 'restated %s' % (want,),
                                     span_overflow.describe(maxima, self.M, self.segcap))
      if want:
        continue    # beyond phase B's tables: the frame is not defined
      assert status[e] == 0, (where, int(e), int(status[e]), maxima)
      diff = frames[e] != ref
      assert not diff.any(), (where, int(e), int(diff.sum()), np.argwhere(diff)[:4].tolist())
      n_exact += 1
    return n_exact

  def unmoved(self):
    st = self.eng.download_state()
    return np.array_equal(st['pos_x'], self.pos[0]) and np.array_equal(st['pos_y'], self.pos[1])

  def close(self):
    self.eng.close()


def _n_sms():
  import torch
  return torch.cuda.get_device_properties(0).multi_processor_count


def _run_modes(sw, raster, skew=0):
  """Engine.render, Engine.step (actions that move nothing), step_host (env chunks) and
  step_gather into two buffers of this device (render_kernel<true>), each into sentinel-filled
  guarded buffers.  Returns, per write-out, the number of envs compared bit-exact."""
  import torch
  E, H, W = sw.E, sw.H, sw.W
  n = E * H * W * 3
  dev = sw.eng.device
  cid = sw.case[0]
  n_exact = []
  # render
  big, flat, lo = _guarded(n, dev, skew)
  frames = flat.view(E, H, W, 3)
  sw.eng.render(raster, frames)
  status = sw.eng.render_status().cpu().numpy()
  _assert_guards(big, lo, n, (cid, 'render'))
  n_exact.append(sw.check(frames.cpu().numpy(), status, (cid, 'render', skew)))
  # step
  big, flat, lo = _guarded(n, dev, skew)
  res = sw.eng.step(sw.actions, raster, flat.view(E, H, W, 3))
  fr, status = res.frames.cpu().numpy(), res.status.cpu().numpy()
  _assert_guards(big, lo, n, (cid, 'step'))
  assert sw.unmoved(), (cid, 'the step moved a sprite')
  n_exact.append(sw.check(fr, status, (cid, 'step', skew)))
  # step_host: frames rendered in env chunks into the engine's own buffer, copied out per chunk
  hbig = np.full(n + 2 * GUARD + 1, SENTINEL, np.uint8)
  hfr = hbig[GUARD + skew:GUARD + skew + n].reshape(E, H, W, 3)
  _, _, _, status, fr = sw.eng.step_host(sw.actions.cpu().numpy(), raster, out=dict(frames=hfr))
  assert fr is hfr
  assert (hbig[:GUARD + skew] == SENTINEL).all() and (hbig[GUARD + skew + n:] == SENTINEL).all()
  assert sw.unmoved(), (cid, 'the step moved a sprite')
  n_exact.append(sw.check(fr, status, (cid, 'host', skew)))
  # step_gather: every frame stored into two [2E] buffers at env index e (render_kernel<true>);
  # with skew, the second target starts `skew` bytes past a 16-byte boundary
  bufs = [_guarded(2 * n, dev, 0), _guarded(2 * n, dev, skew)]
  ptrs = (ctypes.c_void_p * 2)(bufs[0][1].data_ptr(), bufs[1][1].data_ptr())
  local = bufs[0][1].view(2 * E, H, W, 3)
  res = sw.eng.step_gather(sw.actions, raster, (ptrs, 2, 0, local))
  torch.cuda.synchronize()
  status = res.status.cpu().numpy()
  for k, (big, flat, lo) in enumerate(bufs):
    _assert_guards(big, lo, 2 * n, (cid, 'gather', k))
    assert bool((flat[n:] == SENTINEL).all()), (cid, 'gather', k, 'store past env E - 1')
    n_exact.append(sw.check(flat[:n].view(E, H, W, 3).cpu().numpy(), status,
                            (cid, 'gather', k, skew)))
  assert sw.unmoved(), (cid, 'the step moved a sprite')
  return n_exact


@pytest.mark.gpu
@pytest.mark.parametrize('case', [pytest.param(c, id=c[0], marks=KNOWN_DEFECTS.get(c[0], ()))
                                  for c in CASES])
def test_geometry_sweep(case):
  from spriteworld_b200 import _native, engine
  sw = Sweep(case, _n_sms())
  try:
    try:
      raster = engine.Raster(sw.eng, sw.W, sw.H, sw.aa, sw.bg)
      n_exact = _run_modes(sw, raster)
    except _native.NativeError as ex:
      assert case[0] in REFUSED, (case[0], 'refused: %s' % ex)
      return
    assert case[0] not in REFUSED, (case[0], 'rendered, but the table says it is refused')
    # the sweep must not pass by flagging envs: at least 90 % of them are within the segment
    # table, and every write-out path renders every one of those exactly
    n_within = sum(sw.within(e) for e in range(sw.E))
    assert n_within >= 0.9 * sw.E and n_exact == [n_within] * 5, (case[0], n_exact, n_within, sw.E)
    raster.close()
  finally:
    sw.close()


@pytest.mark.gpu
@pytest.mark.parametrize('cid', ['w36h70a3', 'stripes', 'w33h17a3'])
def test_frames_at_odd_addresses(cid):
  """Frame buffers one byte past a 16-byte boundary: phase D must not hand a misaligned
  destination to the bulk copy (64x64 frames would otherwise go through it whole)."""
  from spriteworld_b200 import engine
  case = [c for c in CASES if c[0] == cid][0]
  sw = Sweep(case, _n_sms())
  raster = engine.Raster(sw.eng, sw.W, sw.H, sw.aa, sw.bg)
  n_within = sum(sw.within(e) for e in range(sw.E))
  assert n_within > 0 and _run_modes(sw, raster, skew=1) == [n_within] * 5
  raster.close()
  sw.close()


@pytest.mark.gpu
def test_segment_capacity_boundary():
  """With a star in the pool (16 visible segments per canvas row) a row of 16 pieces renders
  exact and a row of 17 is flagged for its env alone; with convex shapes only the same 17-piece
  row renders exact."""
  import torch
  from spriteworld_b200 import _native, constants, engine, renderers, scene, sprite
  tab = oracle.shape_table(constants.SHAPES)
  rc = oracle.raster_cfg(64, 64, 5)

  def run(rows):
    arrs = {k: np.concatenate([r[k] for r in rows]) for k in rows[0]}
    E, S = arrs['x'].shape
    eng = engine.Engine(E, S, 1, dict(kind='select_move', scale=1.0), [dict(kind='no_reward')],
                        constants.SHAPES)
    b = scene.batch_from_factor_arrays(
        arrs['x'], arrs['y'], arrs['pos_f32'], arrs['shape'], arrs['angle'], arrs['scale'],
        arrs['c0'], arrs['c1'], arrs['c2'], arrs['vx'], arrs['vy'], arrs['member'], arrs['rgb'])
    eng.upload_scenes(b, np.arange(E), np.zeros(E, int))
    eng.upload_state(pos_x=b['x'], pos_y=b['y'], cursor=np.zeros(E), step_count=np.zeros(E),
                     reset_next=np.zeros(E))
    r = engine.Raster(eng, 64, 64, 5)
    big, flat, lo = _guarded(E * 64 * 64 * 3, eng.device)
    frames = eng.render(r, flat.view(E, 64, 64, 3)).cpu().numpy()
    _assert_guards(big, lo, E * 64 * 64 * 3, 'capacity')
    status = eng.render_status().cpu().numpy()
    refs = [oracle.render(rc, tab, rec) for rec in fixtures.records_from_arrays(arrs)]
    return eng, r, frames, status, refs

  # star in the pool: 16 pieces exact, 17 flagged for env 1 only
  eng, r, frames, status, refs = run([stripes(7, True, True), stripes(8, False, True),
                                      stripes(7, True, True), stripes(7, True, True, y=0.3)])
  assert status.tolist() == [0, _native.ENV_SPAN_OVERFLOW, 0, 0], status
  for e in (0, 2, 3):
    assert np.array_equal(frames[e], refs[e]), e
  with pytest.raises(_native.NativeError):
    eng.check_render()
  r.close()
  eng.close()
  # convex shapes only: 2S - 1 segments per row, the 17-piece row is exact
  eng, r, frames, status, refs = run([stripes(8, False, False)] * 3)
  assert not status.any(), status
  for e in range(3):
    assert np.array_equal(frames[e], refs[e]), e
  eng.check_render()
  r.close()
  eng.close()
  # the drop-in renderer raises on the 17-piece row with a star, renders it without one
  def sprites(star):
    a = stripes(8, False, star)
    return [sprite.Sprite(x=float(a['x'][0, s]), y=float(a['y'][0, s]),
                          shape=oracle_name(int(a['shape'][0, s])), scale=float(a['scale'][0, s]),
                          c0=int(a['rgb'][0, s, 0]), c1=int(a['rgb'][0, s, 1]),
                          c2=int(a['rgb'][0, s, 2])) for s in range(a['x'].shape[1])]
  with pytest.raises(RuntimeError):
    renderers.PILRenderer(image_size=(64, 64), anti_aliasing=5).render(sprites(True))
  got = renderers.PILRenderer(image_size=(64, 64), anti_aliasing=5).render(sprites(False))
  a = stripes(8, False, False)
  assert np.array_equal(got, oracle.render(rc, tab, fixtures.records_from_arrays(a)[0]))
  torch.cuda.synchronize()


def oracle_name(shape_id):
  return {v: k for k, v in oracle.SHAPE_IDS.items()}[shape_id]


@pytest.mark.gpu
def test_frames_argument_is_checked():
  import torch
  from spriteworld_b200 import constants, engine
  E = 4
  eng = engine.Engine(E, 2, 1, dict(kind='select_move', scale=1.0), [dict(kind='no_reward')],
                      constants.SHAPES)
  r = engine.Raster(eng, 16, 8, 2)
  acts = torch.full((E, 4), 0.5, device=eng.device)
  dev = eng.device
  bad = [torch.zeros((E, 8, 16, 3), dtype=torch.uint8),                      # host memory
         torch.zeros((E, 8, 16, 3), dtype=torch.float32, device=dev),        # dtype
         torch.zeros((E + 1, 8, 16, 3), dtype=torch.uint8, device=dev),      # too many frames
         torch.zeros((E, 16, 8, 3), dtype=torch.uint8, device=dev),          # W and H swapped
         torch.zeros((E * 8 * 16 * 3,), dtype=torch.uint8, device=dev),      # flat
         torch.zeros((E, 16, 16, 3), dtype=torch.uint8, device=dev)[:, ::2],  # not contiguous
         np.zeros((E, 8, 16, 3), np.uint8)]
  for fr in bad:
    with pytest.raises(ValueError):
      eng.render(r, fr)
    with pytest.raises(ValueError):
      eng.step(acts, r, fr)
  ptrs = (ctypes.c_void_p * 2)(0, 0)
  for fr in bad + [torch.zeros((E, 8, 16, 3), dtype=torch.uint8, device=dev)]:   # gather: 2E frames
    with pytest.raises(ValueError):
      eng.step_gather(acts, r, (ptrs, 2, 0, fr))
  assert eng.render(r, torch.zeros((E, 8, 16, 3), dtype=torch.uint8, device=dev)).shape == (E, 8, 16, 3)
  r.close()
  eng.close()
