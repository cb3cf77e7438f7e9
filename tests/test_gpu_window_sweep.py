"""Windows (render_kernel<., ., ., true>, swb_render_windows) over every raster of the render sweeps,
against the CPU restatements: tests/window_oracle.py for frames and ENV_BAD_WINDOW, and
tests/span_overflow.py (restate with a window) for ENV_SPAN_OVERFLOW.

Every non-refused case of the geometry, wide anti-aliasing and far sweeps is drawn through windows:
its live envs and its records (permuted and repeated, n > E, some with edited shape bytes and
positions), with V = 1, 3 and 7 distinct windows per row, into sentinel-guarded buffers at aligned
and odd addresses.  Each view's window comes from a family built on the CPU from the row's own
world vertices (`plan`):
  full      -- (0, 0, 1, 1), some corners -0.0;
  random    -- zoom 1/4 .. 64, anisotropic, partly or wholly off the scene;
  zoomout   -- zoom 1/4 about the scene, where sprites shrink to a few canvas pixels and crowd the
               rows (each phase-B overflow condition);
  edge, corner, flat -- zoom so far that a sprite is 2^15 .. 2^29 canvas units across, centred on
               a point of one of its edges, on a vertex, or on a horizontal edge: int16 clamps of
               edge rows, horizontal edges, output regions and corner joins, through a window;
  int16     -- a chosen vertex at exactly 32767.5, 32768, -32768.5 or -32769 canvas units;
  limit     -- the vertex of largest magnitude at exactly nextafter(2^30, 0), 2^30 - 1, 2^30 or
               nextafter(2^30, inf), either sign, either axis: phase A's |u| < 2^30;
  rounding  -- windows found by search where the specified u = (wx - x0) * (CW / (x1 - x0))
               truncates to another integer than ((wx - x0) * CW) / (x1 - x0) or than the fused
               fma(wx, sx, -(x0 * sx)) would;
  edge cases -- width 1e-12, a width that overflows to inf, a subnormal width, wholly off the
               scene, NaN, inf and empty windows.
Records rows 0 .. 6 are edited: shape bytes 13 and 255 (sanitised on read to empty slots), empty
slots at NaN, infinite and far positions (never flagged), occupied slots at NaN and +-inf
positions (always flagged).

Every item's status must be the restated BAD_WINDOW | SPAN_OVERFLOW.  The restated BAD_WINDOW bit
is cheap and checked on every item; the frame and the overflow bit are compared on every item the
device or the restatement flags, every item of the edge families and edited rows, and a seeded
sample of the rest sized to a canvas budget (`_pick`).  Items with status 0 must be the
restatement's frame bit for bit, BAD_WINDOW frames are zero, and SPAN_OVERFLOW frames are not
defined.  test_case_table_covers_the_window_paths runs the same plans on the CPU alone and fails if
the compared items stop reaching what the sweep is there for.
"""
import fractions
import math

import numpy as np
import pytest

from oracle import oracle
from spriteworld_b200 import _native
from tests import fixtures, span_overflow
from tests import test_gpu_render_far as far
from tests import test_gpu_render_geometry as geo
from tests import test_gpu_render_wide_aa as wide
from tests import window_oracle as wo

gpu = pytest.mark.gpu

LIMIT = wo.LIMIT
INT16 = 2.0 ** 15
BAD_WINDOW, SPAN_OVERFLOW = _native.ENV_BAD_WINDOW, _native.ENV_SPAN_OVERFLOW
RUNS = (('live', 3), ('records', 1), ('records', 7))
PIXEL_BUDGET = 6e7                    # canvas pixels x sprites per run for the sampled items
SAMPLE = (4, 16)                      # sampled items per run, at least and at most
LIMIT_T = (np.nextafter(LIMIT, 0.0), LIMIT - 1.0, LIMIT, np.nextafter(LIMIT, np.inf))
INT16_T = (32767.5, 32768.0, -32768.5, -32769.0)
EDGE_FAMILIES = {'edge', 'corner', 'flat', 'int16', 'limit', 'rounding', 'tiny', 'inf_width',
                 'subnormal', 'offscene', 'nan', 'inf', 'empty', 'zoomout', 'fold'}


def _cases():
  out = [('geo', c) for c in geo.CASES if c[0] not in geo.REFUSED]
  out += [('wide', c) for c in wide.CASES if c[0] not in wide.REFUSED]
  out += [('far', c) for c in far.CASES]
  assert len({c[0] for _, c in out}) == len(out)
  return out


CASES = _cases()


class Case(object):
  """A case's scenes and raster on the CPU: records, shape table, span class and segment table."""

  def __init__(self, sweep, case):
    from spriteworld_b200 import constants
    self.sweep, self.case = sweep, case
    cid, self.W, self.H, self.aa, self.bg, self.S, _, concave, _ = case
    if sweep == 'far':
      self.arrs = far.case_arrays(case)
    else:
      self.arrs = geo.case_arrays(case, geo._n_envs(case, geo.H100_SMS))
    self.rec = fixtures.records_from_arrays(self.arrs)
    self.E = len(self.rec)
    self.shapes = constants.SHAPES
    self.tab = oracle.shape_table(self.shapes)
    self.rc = oracle.raster_cfg(self.W, self.H, self.aa, self.bg)
    self.CW, self.CH = self.W * self.aa, self.H * self.aa
    self.M = 4 if concave else 1
    if self.aa >= far.WIDE_AA:
      self.segcap = wide.render_layout(self.W, self.H, self.aa, self.S, concave)[1]
    else:
      self.segcap = span_overflow.segcap(self.S, self.M, exact=cid not in geo.SEGCAP_16)
    nv = np.zeros(256, int)
    vt = np.zeros((256, oracle.MAX_VERTS, 2))
    for k in range(1, 13):
      n = self.tab.n_verts[k]
      nv[k] = n
      vt[k, :n] = [[self.tab.verts[k][i][0], self.tab.verts[k][i][1]] for i in range(n)]
    self.nv, self.vt = nv, vt


def _permutation(E):
  """2E + 3 record indices, reversed and repeated, none at its own position."""
  i = np.arange(2 * E + 3)
  perm = (E - 1 - i) % E
  return np.where(perm == i, (i + 1) % E, perm)


# record edits: row -> [(slot, shape byte or None, x or None, y or None)]; slot -1 is the last slot,
# which every case's scenes occupy
def _edits(S):
  even = [(s, 13, None, None) for s in range(0, S, 2)]
  odd = [(s, 255, None, None) for s in range(1, S, 2)] or [(0, 255, None, None)]
  return {0: even, 1: odd,
          2: [(0, 0, np.nan, np.nan)] + ([(1, 13, np.inf, -np.inf)] if S > 1 else []),
          3: [(0, 0, 1e30, -1e300)] + ([(1, 255, -1e300, np.nan)] if S > 1 else []),
          4: [(-1, None, np.nan, None)],
          5: [(-1, None, None, np.inf)],
          6: [(-1, None, -np.inf, None)]}


def _sprites(c, source):
  """(rows, sprites (n, S) as the kernel reads them, edited rows): shape bytes sanitised."""
  if source == 'live':
    return np.arange(c.E), c.rec.copy(), {}
  rows = _permutation(c.E)
  sp = c.rec[rows].copy()
  edits = _edits(c.S)
  for i, ed in edits.items():
    for s, shape, x, y in ed:
      if shape is not None:
        sp['shape'][i, s] = shape if shape <= 12 else 0
      if x is not None:
        sp['x'][i, s] = x
      if y is not None:
        sp['y'][i, s] = y
  return rows, sp, edits


def world(c, sp):
  """(wx, wy, valid) (n, S, MAX_VERTS): world vertices of every slot, as window_oracle.world_vertices
  computes them, and whether the vertex belongs to an occupied slot."""
  sh = sp['shape'].astype(int)
  v = c.vt[sh]
  with np.errstate(all='ignore'):
    cx = (sp['m00'][..., None] * v[..., 0] + sp['m01'][..., None] * v[..., 1]) + 0.0
    cy = (sp['m10'][..., None] * v[..., 0] + sp['m11'][..., None] * v[..., 1]) + 0.0
    wx, wy = cx + sp['x'][..., None], cy + sp['y'][..., None]
  valid = (sh[..., None] != 0) & (np.arange(v.shape[2]) < c.nv[sh][..., None])
  return wx, wy, valid


def transform(c, wx, wy, win):
  """Window-space (u, v) of world vertices (n, S, K) through windows (n, V, 4): (n, V, S, K)."""
  x0, y0, x1, y1 = (win[..., k][..., None, None] for k in range(4))
  with np.errstate(all='ignore'):
    return ((wx[:, None] - x0) * (c.CW / (x1 - x0)), (wy[:, None] - y0) * (c.CH / (y1 - y0)))


def bad_flags(c, wx, wy, valid, win):
  """ENV_BAD_WINDOW of every item (n, V), as window_oracle.bad_window decides it."""
  x0, y0, x1, y1 = (win[..., k] for k in range(4))
  ok = np.isfinite(win).all(-1) & (x1 > x0) & (y1 > y0)
  u, v = transform(c, wx, wy, win)
  with np.errstate(all='ignore'):
    inside = (np.abs(u) < LIMIT) & (np.abs(v) < LIMIT)
  return ~ok | (valid[:, None] & ~inside).any((2, 3))


# ---------------------------------------------------------------------------------------------
# window families
# ---------------------------------------------------------------------------------------------

def exact_axis(w, T, C):
  """(a0, a1): an axis interval whose transform takes world coordinate w to exactly T: a1 - a0 is
  C 2^-k and w - a0 is T 2^-k, both exact, so that C / (a1 - a0) is 2^k and u = T.  None if no k
  near the natural one gives exact operations."""
  if not np.isfinite(w) or w == 0.0:
    return None
  E = math.frexp(abs(w))[1]
  k0 = math.ceil(math.log2(abs(T))) - E
  for k in range(k0 - 1, k0 + 12):
    D = T * 2.0 ** -k
    a0 = w - D
    a1 = a0 + C * 2.0 ** -k
    if a1 - a0 == C * 2.0 ** -k and w - a0 == D and (w - a0) * (C / (a1 - a0)) == T:
      return a0, a1
  return None


def _fma_u(w, a0, C, a1):
  """fma(w, sx, -(a0 * sx)) with sx = C / (a1 - a0): one rounding of the exact w sx - fl(a0 sx)."""
  sx = C / (a1 - a0)
  p = a0 * sx
  return float(fractions.Fraction(w) * fractions.Fraction(sx) - fractions.Fraction(p))


def rounding_axis(rng, ws, C, kind, tries=64):
  """(a0, a1, w): an axis interval and one of the world coordinates `ws` whose specified u truncates
  to another integer than the other formula `kind` ('reordered': ((w - a0) * C) / (a1 - a0);
  'fma': fma(w, sx, -(a0 sx))) gives, with u inside the canvas.  None if the search finds none."""
  ws = ws[np.isfinite(ws)]
  if not len(ws):
    return None
  for _ in range(tries):
    n = 4096
    w = rng.choice(ws, n)
    zoom = np.exp(rng.uniform(0.0, np.log(16.0), n))
    width = 1.0 / zoom
    target = rng.randint(1, max(2, int(C)), n).astype(np.float64)
    a0 = w - target * width / C
    # step a0 a few ulps either way, so that u crosses the integer
    a0 = (a0.view(np.int64) + rng.randint(-6, 7, n) * np.where(a0 < 0, -1, 1)).view(np.float64)
    a1 = a0 + width
    u = (w - a0) * (C / (a1 - a0))
    near = np.abs(u - np.round(u)) <= 8 * np.spacing(u)
    if kind == 'reordered':
      alt = ((w - a0) * C) / (a1 - a0)
      hit = np.flatnonzero(near & (np.trunc(u) != np.trunc(alt)) & (u > 0) & (u < C))
      if len(hit):
        i = hit[0]
        return a0[i], a1[i], w[i]
    else:
      for i in np.flatnonzero(near & (u > 0) & (u < C))[:64]:
        if np.trunc(_fma_u(w[i], a0[i], C, a1[i])) != np.trunc(u[i]):
          return a0[i], a1[i], w[i]
  return None


def _far_zoom(rng, c, wx, wy, valid, family):
  """A window zoomed so far that one sprite is 2^15 .. 2^29 canvas units across, centred on a point
  of one of its edges ('edge'), on a vertex ('corner') or on a horizontal edge ('flat'), with every
  occupied vertex of the row below 2^29.  None if the row has no such sprite."""
  occ = np.flatnonzero(valid.any(1) & np.isfinite(np.where(valid, wx + wy, 0.0)).all(1))
  if not len(occ):
    return None
  s = rng.choice(occ)
  n = int(valid[s].sum())
  px, py = wx[s, :n], wy[s, :n]
  if family == 'flat':
    flat = [i for i in range(n) if py[i] == py[(i + 1) % n] and px[i] != px[(i + 1) % n]]
    if not flat:
      return None
    i = flat[rng.randint(len(flat))]
    t = rng.rand()
  else:
    i, t = rng.randint(n), (0.0 if family == 'corner' else rng.rand())
  j = (i + 1) % n
  p = np.array([px[i] + t * (px[j] - px[i]), py[i] + t * (py[j] - py[i])])
  allx, ally = wx[valid], wy[valid]
  if not (np.isfinite(allx).all() and np.isfinite(ally).all()):
    return None
  diam = max(px.max() - px.min(), py.max() - py.min())
  if diam <= 0:
    return None
  # canvas units per world unit: the sprite 2^15.5 .. 2^29 across, every vertex below 2^28.5
  reach = max(np.abs(allx - p[0]).max(), np.abs(ally - p[1]).max(), 1e-300)
  sx = min(2.0 ** rng.uniform(15.5, 29) / diam, 2.0 ** 28.5 / reach)
  ww, hh = c.CW / sx, c.CH / sx * rng.choice([1.0, 0.5, 2.0])
  cx, cy = p[0] + rng.uniform(-0.3, 0.3) * ww, p[1] + rng.uniform(-0.3, 0.3) * hh
  return (cx - ww / 2, cy - hh / 2, cx + ww / 2, cy + hh / 2)


SIX_ARMED = (oracle.SHAPE_IDS['star_6'], oracle.SHAPE_IDS['spoke_6'])


def _fold(rng, c, sp, wx, wy, valid, tries=4096):
  """A window that puts a six-armed star or spoke of the row across canvas row 0, found by search
  among sizes, aspects and offsets, so that truncation toward zero folds its vertices on rows -1 and
  0 onto row 0: more crossings on that row than CAP (the known excess of tests/test_span_overflow_bounds).
  None if the row has no such sprite or the search finds none."""
  cap = span_overflow.limits(c.M)[0]
  occ = [s for s in range(c.S) if sp['shape'][s] in SIX_ARMED and np.isfinite(wx[s][valid[s]]).all()
         and np.isfinite(wy[s][valid[s]]).all()]
  if not occ:
    return None
  s = occ[rng.randint(len(occ))]
  n = int(valid[s].sum())
  px, py = wx[s, :n], wy[s, :n]
  diam = max(np.ptp(px), np.ptp(py))
  sx = np.exp(rng.uniform(np.log(5.0), np.log(1000.0), tries)) / diam
  sy = sx * np.where(rng.rand(tries) < 0.5, 1.0, np.exp(rng.uniform(np.log(0.25), np.log(4.0), tries)))
  cx, cy = float(sp['x'][s]), float(sp['y'][s])
  x0 = cx - rng.uniform(0, c.CW, tries) / sx
  y0 = cy - rng.uniform(-1.0, 1.0, tries) / sy
  x1, y1 = x0 + c.CW / sx, y0 + c.CH / sy
  iu = np.trunc((px - x0[:, None]) * (c.CW / (x1 - x0))[:, None])
  iv = np.trunc((py - y0[:, None]) * (c.CH / (y1 - y0))[:, None])
  iu1, iv1 = np.roll(iu, -1, 1), np.roll(iv, -1, 1)
  exists = np.ones_like(iu, bool)
  exists[:, -1] = (iu[:, -1] != iu[:, 0]) | (iv[:, -1] != iv[:, 0])
  scanned = exists & (iv != iv1)
  ymin, ymax = np.minimum(iv, iv1), np.maximum(iv, iv1)
  p_ymax = np.minimum(np.maximum(0, iv.max(1)), c.CH)[:, None]
  on = scanned & (ymin <= 0) & (0 <= ymax)
  count = (on.astype(int) + (on & (ymax == 0) & (0 < p_ymax))).sum(1)
  hit = np.flatnonzero(count > cap)
  if not len(hit):
    return None
  k = hit[0]
  return (x0[k], y0[k], x1[k], y1[k]), dict(crossings=int(count[k]))


def _exact_window(rng, c, wx, wy, valid, Ts, extreme):
  """A window that takes one occupied vertex of the row exactly to T (one of Ts) on one axis; the
  other axis is the unit interval.  extreme: the vertex of largest magnitude on that axis, so that
  no other vertex is further out.  Returns (window, T, axis) or None."""
  for _ in range(8):
    T = float(Ts[rng.randint(len(Ts))])
    axis = rng.randint(2)
    ws = (wx if axis == 0 else wy)[valid]
    ws = ws[np.isfinite(ws) & (ws != 0)]
    if not len(ws):
      return None
    if extreme:
      cand = [ws[np.argmax(np.abs(ws))]]
      T = math.copysign(T, cand[0])
    else:
      cand = ws[np.sign(ws) == np.sign(T)]
      if not len(cand):
        continue
      cand = [rng.choice(cand)]
    C = c.CW if axis == 0 else c.CH
    iv = exact_axis(cand[0], T, float(C))
    if iv is None:
      continue
    win = (iv[0], 0.0, iv[1], 1.0) if axis == 0 else (0.0, iv[0], 1.0, iv[1])
    return win, T, axis
  return None


SPECIAL = ('edge', 'corner', 'flat', 'int16', 'limit', 'rounding', 'zoomout', 'fold')
ONE_OFF = ('tiny', 'inf_width', 'subnormal', 'offscene', 'nan', 'inf', 'empty', 'negzero')


def plan(c, source, V, seed):
  """The windows of one run: (rows, sprites, edits, windows (n, V, 4), family (n, V) str, info
  (n, V) dict).  A deterministic function of the case and the run, so that the CPU coverage test
  sees the device test's items."""
  rng = np.random.RandomState(seed)
  rows, sp, edits = _sprites(c, source)
  n = len(rows)
  wx, wy, valid = world(c, sp)
  win = np.zeros((n, V, 4))
  fam = np.empty((n, V), object)
  info = np.empty((n, V), object)
  # the rest: full, random and zoom-out windows
  zoom = np.exp(rng.uniform(np.log(0.25), np.log(64.0), (n, V)))
  aspect = rng.choice([1.0, 0.5, 2.5], (n, V))
  cx, cy = rng.uniform(-0.5, 1.5, (n, V)), rng.uniform(-0.5, 1.5, (n, V))
  w, h = 1.0 / zoom, aspect / zoom
  win[:] = np.stack([cx - w / 2, cy - h / 2, cx + w / 2, cy + h / 2], -1)
  fam[:] = 'random'
  full = rng.rand(n, V) < 0.1
  win[full] = (0.0, 0.0, 1.0, 1.0)
  fam[full] = 'full'
  for i in range(n):
    for v in range(V):
      info[i, v] = {}
  # the edge families, at items spread over the run
  items = rng.permutation(n * V)
  k = 0
  want = [f for f in SPECIAL for _ in range(3)] + list(ONE_OFF)
  for f in want:
    if k >= len(items):
      break
    i, v = divmod(int(items[k]), V)
    k += 1
    got = _family(rng, c, f, sp[i], wx[i], wy[i], valid[i])
    if got is None:
      continue
    win[i, v], info[i, v] = got
    fam[i, v] = f
  return rows, sp, edits, win, fam, info


def _family(rng, c, f, sp, wx, wy, valid):
  """(window, info) of family f for one row, or None."""
  if f == 'fold':
    return _fold(rng, c, sp, wx, wy, valid)
  if f == 'zoomout':
    cx, cy = 0.5 + rng.uniform(-0.3, 0.3, 2)
    return (cx - 2.0, cy - 2.0, cx + 2.0, cy + 2.0), {}
  if f in ('edge', 'corner', 'flat'):
    w = _far_zoom(rng, c, wx, wy, valid, f)
    return None if w is None else (w, {})
  if f in ('int16', 'limit'):
    got = _exact_window(rng, c, wx, wy, valid, INT16_T if f == 'int16' else LIMIT_T, f == 'limit')
    if got is None:
      return None
    return got[0], dict(T=got[1], axis=got[2])
  if f == 'rounding':
    kind = ('reordered', 'fma')[rng.randint(2)]
    axis = rng.randint(2)
    C = float(c.CW if axis == 0 else c.CH)
    got = rounding_axis(rng, (wx if axis == 0 else wy)[valid], C, kind)
    if got is None:
      return None
    a0, a1, w = got
    win = (a0, 0.0, a1, 1.0) if axis == 0 else (0.0, a0, 1.0, a1)
    return win, dict(kind=kind, axis=axis, w=w)
  x = float(wx[valid][0]) if valid.any() and np.isfinite(wx[valid][0]) else 0.5
  return {'tiny': ((x, 0.0, x + 1e-12, 1.0), {}),
          'inf_width': ((-1e308, 0.0, 1e308, 1.0), {}),
          'subnormal': ((0.0, 0.25, 5e-324, 0.75), {}),
          'offscene': ((4.0, -7.5, 4.5, -7.0), {}),
          'nan': ((0.0, np.nan, 1.0, 1.0), {}),
          'inf': ((-np.inf, 0.0, 1.0, 1.0), {}),
          'empty': ((0.3, 0.6, 0.7, 0.6), {}),
          'negzero': ((-0.0, -0.0, 1.0, 1.0), {})}[f]


def _pick(c, fam, bad, edits, flagged, seed):
  """Items (i, v) compared with the oracle: every item the device or the restatement flags, every
  item of an edge family or an edited row, and a seeded sample of the rest sized to PIXEL_BUDGET."""
  n, V = fam.shape
  special = bad | flagged | np.isin(fam, list(EDGE_FAMILIES))
  if edits:
    special[list(edits)] = True
  cost = float(c.CW * c.CH * (c.S + 3))
  n_rest = int((~special).sum())
  p = min(1.0, min(SAMPLE[1], max(SAMPLE[0], PIXEL_BUDGET / cost)) / max(1, n_rest))
  u = np.random.RandomState(seed).rand(n, V)
  return np.argwhere(special | (u < p))


def _seed(cid, source, V):
  return (sum(map(ord, cid)) * 31 + V * 7 + (source == 'records')) % (2 ** 31)


def expected(c, sp, win, i, v):
  """(frame, status) the restatements give item (i, v)."""
  frame, bad = wo.render_window(c.rc, c.tab, sp[i], win[i, v])
  if bad:
    return frame, BAD_WINDOW
  m = span_overflow.restate(c.W, c.H, c.aa, sp[i], c.shapes, c.M, window=win[i, v])
  return frame, (SPAN_OVERFLOW if span_overflow.conditions(m, c.M, c.segcap) else 0), m


# ---------------------------------------------------------------------------------------------
# the device
# ---------------------------------------------------------------------------------------------

def _set_field(data, S, name, rows, slot, value):
  from spriteworld_b200 import engine
  for field, off, dtype, shape in engine.record_layout(S)[0]:
    if field == name:
      a = data[:, off:off + dtype.itemsize * S].view(dtype)
      a[rows, slot] = value
      return
  raise KeyError(name)


def _records(sw, c, rows, edits):
  """The permuted records of the engine with the edits applied to their bytes."""
  import torch
  from spriteworld_b200 import engine
  states = sw.eng.save_envs().take(torch.from_numpy(rows).to(sw.eng.device))
  data = states.data.cpu().numpy().copy()
  for i, ed in edits.items():
    for s, shape, x, y in ed:
      s = s % c.S
      if shape is not None:
        _set_field(data, c.S, 'shape', i, s, shape)
      if x is not None:
        _set_field(data, c.S, 'pos_x', i, s, x)
      if y is not None:
        _set_field(data, c.S, 'pos_y', i, s, y)
  return engine.EnvStates(torch.from_numpy(data).to(sw.eng.device), states.span_class, states.signature, c.S)


def _run(sw, c, raster, source, V):
  """One run on the device against the restatements; returns the counts it compared."""
  import torch
  cid = c.case[0]
  seed = _seed(cid, source, V)
  rows, sp, edits, win, fam, info = plan(c, source, V, seed)
  n, H, W = len(rows), c.H, c.W
  states = None if source == 'live' else _records(sw, c, rows, edits)
  windows = torch.from_numpy(win).to(sw.eng.device).contiguous()
  wx, wy, valid = world(c, sp)
  bad = bad_flags(c, wx, wy, valid, win)
  out = []
  for skew in (0, 1):
    fbig, fflat, flo = geo._guarded(n * V * H * W * 3, sw.eng.device, skew)
    sbig, sflat, slo = geo._guarded(n * V, sw.eng.device, skew)
    frames, status = sw.eng.render_windows(raster, windows, states, fflat.view(n, V, H, W, 3), sflat.view(n, V))
    geo._assert_guards(fbig, flo, n * V * H * W * 3, (cid, source, V, 'frames', skew))
    geo._assert_guards(sbig, slo, n * V, (cid, source, V, 'status', skew))
    out.append((frames.cpu().numpy(), status.cpu().numpy()))
  (f0, s0), (f1, s1) = out
  assert np.array_equal(s0, s1), (cid, source, V, 'status differs between skews')
  # BAD_WINDOW restated on every item
  dev_bad = (s0 & BAD_WINDOW) != 0
  where = np.argwhere(dev_bad != bad)
  assert not len(where), (cid, source, V, 'BAD_WINDOW', [(int(i), int(v), fam[i, v], win[i, v].tolist())
                                                         for i, v in where[:4]])
  assert not (s0 & (0xFF ^ (BAD_WINDOW | SPAN_OVERFLOW))).any(), (cid, source, V, np.unique(s0))
  counts = dict(items=n * V, compared=0, exact=0, bad=int(bad.sum()), overflow=0)
  for i, v in _pick(c, fam, bad, edits, s0 != 0, seed + 1):
    got = expected(c, sp, win, i, v)
    frame, want = got[0], got[1]
    what = (cid, source, V, int(i), int(v), fam[i, v], win[i, v].tolist())
    assert int(s0[i, v]) == want, what + ('status %d, restated %d' % (s0[i, v], want),
                                          span_overflow.describe(got[2], c.M, c.segcap) if len(got) > 2 else '')
    counts['compared'] += 1
    if want == SPAN_OVERFLOW:
      counts['overflow'] += 1
      continue
    for skew, f in ((0, f0), (1, f1)):
      diff = f[i, v] != frame
      assert not diff.any(), what + (skew, int(diff.sum()))
    counts['exact'] += want == 0
  return counts


def _sweep(c):
  sw = geo.Sweep(c.case, geo.H100_SMS, arrs=c.arrs)
  sw.segcap = c.segcap
  return sw


@gpu
@pytest.mark.parametrize('case', [pytest.param(c, id=c[1][0]) for c in CASES])
def test_window_sweep(case):
  from spriteworld_b200 import engine
  c = Case(*case)
  sw = _sweep(c)
  try:
    raster = engine.Raster(sw.eng, c.W, c.H, c.aa, c.bg)
    for source, V in RUNS:
      counts = _run(sw, c, raster, source, V)
      assert counts['exact'] > 0, (c.case[0], source, V, counts)
    assert sw.unmoved()
    raster.close()
  finally:
    sw.close()


# ---------------------------------------------------------------------------------------------
# the CPU tier: what the compared items reach
# ---------------------------------------------------------------------------------------------

def _int16_reach(c, sp, win, i, v):
  """(axis beyond int16 x, y, corner join beyond int16) of the item's integer window vertices."""
  reach = set()
  for s in range(sp.shape[1]):
    if not sp['shape'][i, s]:
      continue
    iv = np.trunc(wo.window_vertices(c.rc, c.tab, sp[i, s], win[i, v])).astype(np.int64)
    if (np.abs(iv[:, 0]) > 32767).any():
      reach.add('int16_x')
    if (np.abs(iv[:, 1]) > 32767).any():
      reach.add('int16_y')
    # a corner join on a canvas row: a vertex on a canvas row both of whose edges leave it
    # downwards with slopes of one sign, one of them ending beyond int16
    n = len(iv)
    for k in range(n):
      a, b = iv[k - 1] - iv[k], iv[(k + 1) % n] - iv[k]
      if (0 <= iv[k, 1] < c.CH and a[1] > 0 and b[1] > 0 and a[0] * b[0] > 0
          and max(abs(iv[k - 1, 1]), abs(iv[(k + 1) % n, 1])) > 32767):
        reach.add('corner_join_int16')
  return reach


def test_case_table_covers_the_window_paths():
  paths = set()
  for sweep, case in CASES:
    c = Case(sweep, case)
    multiband = c.H > geo.BAND_ROWS
    paths.add('wide' if c.aa >= far.WIDE_AA else 'narrow')
    for source, V in RUNS:
      seed = _seed(case[0], source, V)
      rows, sp, edits, win, fam, info = plan(c, source, V, seed)
      wx, wy, valid = world(c, sp)
      bad = bad_flags(c, wx, wy, valid, win)
      if edits:
        paths.add('sanitised_shapes')
        assert bad[4].all() and bad[5].all() and bad[6].all(), case[0]
        if not (bad[2].all() and bad[3].all()):
          paths.add('empty_slots_at_nonfinite_positions_unflagged')
      for i, v in _pick(c, fam, bad, edits, np.zeros_like(bad), seed + 1):
        paths.add(source)
        if multiband and V > 1:
          paths.add('multiband_V>1')
        x0, y0, x1, y1 = win[i, v]
        if bad[i, v]:
          if not np.isfinite(win[i, v]).all():
            paths.add('bad_nonfinite_window')
          elif not (x1 > x0 and y1 > y0):
            paths.add('bad_empty_window')
          else:
            u, vv = transform(c, wx[i:i + 1], wy[i:i + 1], win[i:i + 1, v:v + 1])
            uv = np.concatenate([u[0, 0][valid[i]], vv[0, 0][valid[i]]])
            paths.add('bad_vertex_nan' if np.isnan(uv).any() else 'bad_vertex_limit')
          if fam[i, v] == 'limit':
            paths.add('limit_exact' if abs(info[i, v]['T']) == LIMIT else 'limit_above')
          continue
        if fam[i, v] == 'limit':
          paths.add('limit_below')
          if info[i, v]['T'] == LIMIT_T[0]:
            paths.add('limit_nextafter_below')
        if fam[i, v] == 'rounding':
          paths.add('rounding_' + info[i, v]['kind'])
        if fam[i, v] in ('edge', 'corner', 'flat', 'int16'):
          paths |= _int16_reach(c, sp, win, i, v)
        if fam[i, v] in ('zoomout', 'random', 'full', 'fold'):
          m = span_overflow.restate(c.W, c.H, c.aa, sp[i], c.shapes, c.M, window=win[i, v])
          paths |= {'overflow_' + k for k in span_overflow.conditions(m, c.M, c.segcap)}
  need = {'bad_nonfinite_window', 'bad_empty_window', 'bad_vertex_nan', 'bad_vertex_limit',
          'limit_below', 'limit_nextafter_below', 'limit_exact', 'limit_above',
          'overflow_crossings', 'overflow_pieces',
          'int16_x', 'int16_y', 'corner_join_int16', 'multiband_V>1', 'narrow', 'wide',
          'live', 'records', 'sanitised_shapes', 'empty_slots_at_nonfinite_positions_unflagged', 'rounding_reordered', 'rounding_fma'}
  assert need <= paths, sorted(need - paths)
