"""CPU restatement of frames seen through windows (swb_render_windows, render_kernel<., ., ., true>,
renderers.SpriteGlimpses): test infrastructure, built on the oracle's Pillow polygon fill and
LANCZOS resize (oracle.polygon_fill, oracle.lanczos_resize, which tests/test_oracle_raster.py pins
against Pillow).

The definition: for window (x0, y0, x1, y1) on a W x H raster at anti_aliasing aa, CW = aa W and
CH = aa H, a world vertex (wx, wy) -- PILRenderer's vertex before its multiply by the canvas size
-- goes to
    sx = CW / (x1 - x0);  u = (wx - x0) * sx         (each op float64, round to nearest)
    sy = CH / (y1 - y0);  v = (wy - y0) * sy
and Pillow truncates (u, v).  Then PILRenderer's pipeline: every sprite back to front on a bg
canvas of CW x CH, resize((W, H), LANCZOS), flipud.  With (0, 0, 1, 1), u = CW * wx exactly, so the
frame is PILRenderer's.  The item is flagged ENV_BAD_WINDOW (frame zeros) when the window is not
finite or empty, or an occupied slot has a vertex with u or v NaN or |u| or |v| >= 2^30.
"""
import numpy as np

from oracle import oracle

LIMIT = 2.0 ** 30


def world_vertices(tab, sprite):
  """(n, 2) float64 world vertices (centred vertex + position), the arithmetic of
  tests/mask_oracle.canvas_vertices before its canvas multiply."""
  shape = int(sprite['shape'])
  n = tab.n_verts[shape]
  v = np.array([[tab.verts[shape][i][0], tab.verts[shape][i][1]] for i in range(n)], np.float64).reshape(n, 2)
  cx = (sprite['m00'] * v[:, 0] + sprite['m01'] * v[:, 1]) + 0.0
  cy = (sprite['m10'] * v[:, 0] + sprite['m11'] * v[:, 1]) + 0.0
  return np.stack([cx + sprite['x'], cy + sprite['y']], 1)


def window_vertices(raster_cfg, tab, sprite, window):
  """(n, 2) float64 window-space canvas vertices (u, v) of one sprite."""
  aa = raster_cfg.anti_aliasing
  CW, CH = float(aa * raster_cfg.width), float(aa * raster_cfg.height)
  x0, y0, x1, y1 = (np.float64(c) for c in window)
  w = world_vertices(tab, sprite)
  with np.errstate(all='ignore'):
    sx, sy = CW / (x1 - x0), CH / (y1 - y0)
    return np.stack([(w[:, 0] - x0) * sx, (w[:, 1] - y0) * sy], 1)


def window_ok(window):
  x0, y0, x1, y1 = (float(c) for c in window)
  return bool(np.isfinite([x0, y0, x1, y1]).all() and x1 > x0 and y1 > y0)


def bad_window(raster_cfg, tab, sprites, window):
  """True if the item is flagged ENV_BAD_WINDOW."""
  if not window_ok(window):
    return True
  for sp in np.asarray(sprites, oracle.SPRITE_DTYPE).reshape(-1):
    if sp['shape']:
      uv = window_vertices(raster_cfg, tab, sp, window)
      if not (np.abs(uv) < LIMIT).all():   # NaN fails too
        return True
  return False


def render_window(raster_cfg, tab, sprites, window):
  """(frame (H, W, 3) uint8, bad): the frame of 1-D oracle.SPRITE_DTYPE `sprites` (back to front)
  seen through `window`; zeros and bad = True for a flagged item."""
  W, H, aa = raster_cfg.width, raster_cfg.height, raster_cfg.anti_aliasing
  sprites = np.asarray(sprites, oracle.SPRITE_DTYPE).reshape(-1)
  if bad_window(raster_cfg, tab, sprites, window):
    return np.zeros((H, W, 3), np.uint8), True
  canvas = np.empty((aa * H, aa * W, 3), np.uint8)
  canvas[:] = np.asarray(raster_cfg.bg, np.uint8)
  for sp in sprites:
    if sp['shape']:
      oracle.polygon_fill(canvas, window_vertices(raster_cfg, tab, sp, window), sp['rgb'])
  return np.ascontiguousarray(oracle.lanczos_resize(canvas, W, H)[::-1]), False


def pillow_window(sprites, width, height, anti_aliasing, window, bg=(0, 0, 0), color_to_rgb=None):
  """The definition itself, with Pillow, on Sprite objects (back to front)."""
  from PIL import Image, ImageDraw
  CW, CH = anti_aliasing * width, anti_aliasing * height
  x0, y0, x1, y1 = (np.float64(c) for c in window)
  canvas = Image.new('RGB', (CW, CH), tuple(int(c) for c in bg))
  draw = ImageDraw.Draw(canvas)
  for s in sprites:
    w = np.asarray(s.vertices, np.float64)
    uv = np.stack([(w[:, 0] - x0) * (CW / (x1 - x0)), (w[:, 1] - y0) * (CH / (y1 - y0))], 1)
    color = tuple(int(c) for c in (color_to_rgb(s.color) if color_to_rgb else s.color))
    draw.polygon([tuple(p) for p in uv], fill=color)
  return np.flipud(np.asarray(canvas.resize((width, height), Image.LANCZOS)))


# ---------------------------------------------------------------------------------------------
# the mask double (tests/mask_oracle.py) with swb_render_windows and Engine.render_windows
# ---------------------------------------------------------------------------------------------

def _swb_render_windows(self, eng, raster, records, n, records_bytes, span_class, windows, n_views, frames,
                        status, stream):
  import ctypes
  from spriteworld_b200 import _native
  from tests import oracle_engine
  assert span_class in (1, 4) and n_views >= 1
  assert (records is None and n == eng.n_envs) or (records is not None and n >= 0)
  if n == 0:
    return 0
  r = eng._rasters[raster]
  H, W, items = r.height, r.width, n * n_views
  assert windows.value % 8 == 0
  for p, nb in ((frames.value, items * H * W * 3), (status.value, items)):   # outputs disjoint from windows
    assert not (p < windows.value + items * 32 and windows.value < p + nb), 'windows overlap an output'
  if records is None:
    scenes = [eng._bo.cur[e] for e in range(n)]
  else:
    assert records_bytes >= n * eng.record_bytes
    scenes = oracle_engine.record_sprites(eng, oracle_engine.states_at(eng, records, n))
  win = np.ctypeslib.as_array((ctypes.c_double * (items * 4)).from_address(windows.value)).reshape(n, n_views, 4)
  out = np.ctypeslib.as_array((ctypes.c_uint8 * (items * H * W * 3)).from_address(frames.value))
  out = out.reshape(n, n_views, H, W, 3)
  st = np.ctypeslib.as_array((ctypes.c_uint8 * items).from_address(status.value)).reshape(n, n_views)
  for i, sprites in enumerate(scenes):
    for v in range(n_views):
      out[i, v], bad = render_window(r.rc, eng._tab, sprites, win[i, v])
      st[i, v] = _native.ENV_BAD_WINDOW if bad else 0
  eng._launches += 1
  return 0


def _lib_with_windows():
  from spriteworld_b200 import engine as engine_lib
  from tests import mask_oracle
  mask_engine, raster = mask_oracle._lib_with_masks()

  class WindowOracleEngine(mask_engine):
    """The mask double with swb_render_windows under the real Engine.render_windows."""

    render_windows = engine_lib.Engine.render_windows
    _lib_cls = None

    def __init__(self, *args, **kw):
      super().__init__(*args, **kw)
      cls = type(self)
      if cls._lib_cls is None:
        cls._lib_cls = type('WindowLib', (type(self._lib),), {'swb_render_windows': _swb_render_windows})
      self._lib = cls._lib_cls()

  return WindowOracleEngine, raster


_DOUBLE = None


def install(monkeypatch):
  """Routes the package's host layer to the mask double with swb_render_windows for the duration of a
  test: what tests/mask_oracle.install does, plus Engine.render_windows (the real one, over the
  restatement above), so that SpriteGlimpses and BatchedEnvironment.render_windows run on the CPU."""
  global _DOUBLE
  from spriteworld_b200 import engine as engine_lib
  from tests import mask_oracle
  if _DOUBLE is None:
    _DOUBLE = _lib_with_windows()
  mask_oracle.install(monkeypatch)
  monkeypatch.setattr(engine_lib, 'Engine', _DOUBLE[0])
  monkeypatch.setattr(engine_lib, 'Raster', _DOUBLE[1])
