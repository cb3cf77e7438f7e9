"""CPU restatement of the render kernel's SWB_ENV_SPAN_OVERFLOW flag (csrc/swb_render.cuh,
phase B), from Pillow's scan conversion as the oracle restates it.

The kernel flags an env when one of its bands does not fit phase B's tables:
  - crossings: more than CAP crossings of one sprite on one canvas row (B1's crossing list);
  - spans: more than M runs of one sprite's own fill on one canvas row (B1's span list; with
    M = 1 a second disjoint run);
  - pieces: more than segcap visible pieces on one canvas row (B2's segment table);
  - chunk: one sprite's crossing lists and spans do not fit the scratch area.  check_render
    refuses every raster where that could happen, so `restate` asserts that it does not.

CAP and M follow the span class of the engine's shapes: M = 1 and CAP = 8 while every shape is
convex (ids 1..6), M = 4 and CAP = 16 once a star or spoke (ids > 6) is uploaded.  segcap is
the launch's: 2S - 1 (at least 3) with convex shapes only, 16 with concave shapes or where the
exact table does not fit in shared memory beside the staged frame.

`restate` returns the quantity of each condition, maximised over every canvas row a band of the
raster scans, and `conditions` those beyond their limit: the env is flagged exactly when that
is not empty.
"""
import numpy as np

from oracle import oracle

BAND_ROWS = 64              # swb_raster_create: output rows per band
HT_BYTES = 60 * 44 * 4      # HT_WORDS words of the H tile
CONDITIONS = ('crossings', 'spans', 'pieces')


def limits(M):
  """(CAP, M): crossings and spans kept per (sprite, canvas row) for span class M."""
  assert M in (1, 4), M
  return (16 if M > 1 else 8), M


def span_class(shape_ids):
  """1 while every shape id is convex, 4 once a star or spoke id (> 6) is present."""
  return 4 if (np.asarray(shape_ids) > 6).any() else 1


def segcap(S, M, exact=True):
  """RenderLayout::segcap: visible segments kept per canvas row.  exact = False: the launch
  fell back to 16 because the exact table did not fit."""
  if M > 1:
    return 16
  cap = max(3, 2 * S - 1)
  return cap if exact else min(cap, 16)


def axis_windows(n_in, n_out):
  """Per output: (first input, input count) of its LANCZOS window (swb_tables.h build_axis)."""
  bounds, _ = oracle.lanczos_coeffs(n_in, n_out)
  return bounds[:, 0].astype(int), bounds[:, 1].astype(int)


def bands(H, aa):
  """Per band: the canvas rows [row_b0, row_b1) its vertical windows touch, counted from a
  multiple of four (render_kernel: row_b0 = win_min[yo_b0] & ~3)."""
  band_rows = min(H, BAND_ROWS)
  wmin, wlen = axis_windows(H * aa, H)
  out = []
  for yo_b0 in range(0, H, band_rows):
    yo_b1 = min(yo_b0 + band_rows, H)
    out.append((int(wmin[yo_b0]) & ~3, int(wmin[yo_b1 - 1] + wlen[yo_b1 - 1])))
  return out


def phase_b_scratch(W, H, aa, M):
  """RenderLayout::scratch_bytes: the H tile (or more, so that phase B can hold one sprite
  spanning every canvas row of a band) and the staged frame, each rounded to 16 bytes."""
  cap, M = limits(M)
  rows = max(b1 - b0 for b0, b1 in bands(H, aa))
  r16 = lambda b: (b + 15) & ~15
  frame = min(H, BAND_ROWS) * W * 3
  ht = HT_BYTES
  if ht + r16(frame) < (cap + M) * 4 * rows:
    ht = (cap + M) * 4 * rows - frame
  return r16(ht) + r16(frame)


def canvas_xy(r, verts, CW, CH):
  """(V, 2) canvas coordinates of one sprite record's vertices, as phase A and Pillow compute
  them: the centred path (a*x + c*y) + 0, plus the position, times the canvas side."""
  v = np.asarray(verts, np.float64)
  cx = (r['m00'] * v[:, 0] + r['m01'] * v[:, 1]) + 0.0
  cy = (r['m10'] * v[:, 0] + r['m11'] * v[:, 1]) + 0.0
  return np.stack([CW * (cx + r['x']), CH * (cy + r['y'])], 1)


def int_vertices(xy):
  """Pillow's integer vertices: each coordinate truncated toward zero ((int) in C)."""
  iv = np.trunc(xy).astype(np.int64)
  return iv[:, 0], iv[:, 1]


def sprite_rows(ivy, CH):
  """Pillow's scanned rows of a polygon: [pymin, p_ymax] with ymin = min(CH - 1, vertices),
  ymax = max(0, vertices), clipped to [0, CH]."""
  return max(min(CH - 1, int(ivy.min())), 0), min(max(0, int(ivy.max())), CH)


def crossings(ivx, ivy, CH, rows):
  """Crossings B1 keeps for one sprite on each of `rows`: every scanned edge (y0 != y1) with
  ymin <= y <= ymax, twice where it ends on a row above the polygon's last row.  The closing
  edge exists only where the last vertex differs from the first."""
  x1, y1 = np.roll(ivx, -1), np.roll(ivy, -1)
  exists = np.ones(len(ivy), bool)
  exists[-1] = ivx[-1] != ivx[0] or ivy[-1] != ivy[0]
  scanned = exists & (ivy != y1)
  ymin, ymax = np.minimum(ivy, y1), np.maximum(ivy, y1)
  p_ymax = sprite_rows(ivy, CH)[1]
  y = np.asarray(rows, np.int64)[:, None]
  on = scanned & (ymin <= y) & (y <= ymax)
  twice = on & (y == ymax) & (y < p_ymax)
  return (on.astype(int) + twice).sum(1)


def runs(mask):
  """Per row of a 2-D boolean mask: its runs of True."""
  starts = mask.copy()
  starts[:, 1:] &= ~mask[:, :-1]
  return starts.sum(1)


def sprite_maxima(xy, W, H, aa, M):
  """Most crossings and most runs of one sprite's own fill (the Pillow restatement of the
  oracle, clipped to the canvas, horizontal edges included) on any canvas row a band scans.
  Asserts that the sprite fits phase B's scratch area alone."""
  cap, M = limits(M)
  CW, CH = W * aa, H * aa
  ivx, ivy = int_vertices(xy)
  pymin, p_ymax = sprite_rows(ivy, CH)
  scratch = phase_b_scratch(W, H, aa, M)
  rows = set()
  for b0, b1 in bands(H, aa):
    r0, r1 = max(pymin, b0), min(p_ymax, CH - 1, b1 - 1)
    rows.update(range(r0, r1 + 1))
    # chunk: check_render sizes the scratch area so that one sprite always fits
    rcnt = max(0, r1 - r0 + 1)
    assert rcnt * cap * 4 + (b1 - b0) * M * 4 <= scratch, ('chunk', rcnt, b1 - b0, scratch)
  if not rows:
    return 0, 0
  rows = np.array(sorted(rows))
  own = np.zeros((CH, CW, 3), np.uint8)
  oracle.polygon_fill(own, xy, (1, 0, 0))
  return int(crossings(ivx, ivy, CH, rows).max()), int(runs(own[rows, :, 0] != 0).max())


_TABLES = {}


def _shape_table(shapes):
  key = tuple((k, np.asarray(v, np.float64).tobytes()) for k, v in sorted(shapes.items()))
  if key not in _TABLES:
    _TABLES[key] = oracle.shape_table(shapes)
  return _TABLES[key]


def restate(W, H, aa, rec, shapes, M, window=None):
  """The quantities phase B compares with its capacities, for one env.  rec: its sprite
  records, back to front; shapes: name -> vertices of the engine's shape table; M: the
  launch's span class.  Returns dict(crossings, spans, pieces): the maxima over every sprite
  and every canvas row a band of the raster scans (the status is the OR over the bands).

  window: (x0, y0, x1, y1) of swb_render_windows.  The vertices are then the window-space ones
  of tests/window_oracle.py; bands, capacities and conditions are the same.  An item flagged
  ENV_BAD_WINDOW has no phase B: every maximum is 0."""
  from tests import window_oracle
  CW, CH = W * aa, H * aa
  if window is not None:
    rc, tab = oracle.raster_cfg(W, H, aa), _shape_table(shapes)
    if window_oracle.bad_window(rc, tab, rec, window):
      return dict(crossings=0, spans=0, pieces=0)
  scanned = np.zeros(CH, bool)
  for b0, b1 in bands(H, aa):
    scanned[b0:b1] = True
  rows = np.flatnonzero(scanned)
  names = {v: k for k, v in oracle.SHAPE_IDS.items()}
  lab = np.zeros((CH, CW, 3), np.uint8)   # the painter's algorithm, label s + 1 per sprite
  out = dict(crossings=0, spans=0, pieces=0)
  for s, r in enumerate(rec):
    if not r['shape']:
      continue
    if window is None:
      xy = canvas_xy(r, shapes[names[int(r['shape'])]], CW, CH)
    else:
      xy = window_oracle.window_vertices(rc, tab, r, window)
    c, n = sprite_maxima(xy, W, H, aa, M)
    out['crossings'], out['spans'] = max(out['crossings'], c), max(out['spans'], n)
    oracle.polygon_fill(lab, xy, (s + 1, 0, 0))
  L = lab[rows, :, 0]
  starts = (L != 0) & np.concatenate([np.ones((len(rows), 1), bool), L[:, 1:] != L[:, :-1]], 1)
  out['pieces'] = int(starts.sum(1).max())
  return out


def conditions(maxima, M, seg_cap):
  """The conditions of `restate`'s maxima that set SWB_ENV_SPAN_OVERFLOW under span class M
  and a segment table of seg_cap; empty: the frame is rendered exactly."""
  cap, M = limits(M)
  return tuple(k for k, lim in zip(CONDITIONS, (cap, M, seg_cap)) if maxima[k] > lim)


def describe(maxima, M, seg_cap):
  """'crossings 8/8, spans 1/1, pieces 3/5': each condition's maximum against its limit."""
  cap, M = limits(M)
  return ', '.join('%s %d/%d' % (k, maxima[k], lim) for k, lim in zip(CONDITIONS, (cap, M, seg_cap)))
