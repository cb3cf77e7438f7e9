"""CPU restatement of views with only some sprites drawn (swb_render_views, the `draw` of
render_kernel<., ., ., true>, renderers.SpriteLayers): test infrastructure over
tests/window_oracle.py's restatement of windows, which tests/test_oracle_windows.py pins against
Pillow.

The definition: the view (window, draw) of a row is tests/window_oracle.render_window of the row in
which every slot s with draw[s] == 0 is an empty slot (shape 0).  The sprites drawn keep their
back-to-front order, and the bad-window test looks at drawn occupied slots only.  Through Pillow it
is window_oracle.pillow_window of the sprite list with the undrawn sprites removed.
"""
import numpy as np

from oracle import oracle
from tests import window_oracle as wo


def drawn_sprites(sprites, draw):
  """Copy of the 1-D oracle.SPRITE_DTYPE `sprites` with every slot s whose draw[s] is zero emptied."""
  out = np.array(np.asarray(sprites, oracle.SPRITE_DTYPE).reshape(-1))
  out['shape'][~np.asarray(draw, bool).reshape(-1)] = 0
  return out


def render_layer(raster_cfg, tab, sprites, window, draw):
  """(frame (H, W, 3) uint8, bad) of the view `window` of `sprites` with the slots `draw` drawn."""
  return wo.render_window(raster_cfg, tab, drawn_sprites(sprites, draw), window)


# ---------------------------------------------------------------------------------------------
# the window double (tests/window_oracle.py) with swb_render_views
# ---------------------------------------------------------------------------------------------

def _swb_render_views(self, eng, raster, records, n, records_bytes, span_class, windows, draw, n_views, frames,
                      status, stream):
  import ctypes
  from spriteworld_b200 import _native
  from tests import oracle_engine
  assert span_class in (1, 4) and n_views >= 1 and draw is not None and draw.value
  assert (records is None and n == eng.n_envs) or (records is not None and n >= 0)
  if n == 0:
    return 0
  r = eng._rasters[raster]
  H, W, S, items = r.height, r.width, eng.n_slots, n * n_views
  assert windows.value % 8 == 0
  for p, nb in ((frames.value, items * H * W * 3), (status.value, items)):   # outputs disjoint from the inputs
    assert not (p < windows.value + items * 32 and windows.value < p + nb), 'windows overlap an output'
    assert not (p < draw.value + items * S and draw.value < p + nb), 'draw overlaps an output'
  if records is None:
    scenes = [eng._bo.cur[e] for e in range(n)]
  else:
    assert records_bytes >= n * eng.record_bytes
    scenes = oracle_engine.record_sprites(eng, oracle_engine.states_at(eng, records, n))
  win = np.ctypeslib.as_array((ctypes.c_double * (items * 4)).from_address(windows.value)).reshape(n, n_views, 4)
  drw = np.ctypeslib.as_array((ctypes.c_uint8 * (items * S)).from_address(draw.value)).reshape(n, n_views, S)
  out = np.ctypeslib.as_array((ctypes.c_uint8 * (items * H * W * 3)).from_address(frames.value))
  out = out.reshape(n, n_views, H, W, 3)
  st = np.ctypeslib.as_array((ctypes.c_uint8 * items).from_address(status.value)).reshape(n, n_views)
  for i, sprites in enumerate(scenes):
    for v in range(n_views):
      out[i, v], bad = render_layer(r.rc, eng._tab, sprites, win[i, v], drw[i, v])
      st[i, v] = _native.ENV_BAD_WINDOW if bad else 0
  eng._launches += 1
  return 0


def _lib_with_views():
  window_engine, raster = wo._lib_with_windows()

  class LayerOracleEngine(window_engine):
    """The window double with swb_render_views under the real Engine.render_windows."""

    _views_lib_cls = None

    def __init__(self, *args, **kw):
      super().__init__(*args, **kw)
      cls = type(self)
      if cls._views_lib_cls is None:
        cls._views_lib_cls = type('ViewLib', (type(self._lib),), {'swb_render_views': _swb_render_views})
      self._lib = cls._views_lib_cls()

  return LayerOracleEngine, raster


_DOUBLE = None


def install(monkeypatch):
  """Routes the package's host layer to the window double with swb_render_views for the duration of
  a test: what tests/window_oracle.install does, plus the `draw` of Engine.render_windows (the real
  one, over the restatement above), so that SpriteLayers and render_windows(draw=...) run on the
  CPU."""
  global _DOUBLE
  from spriteworld_b200 import engine as engine_lib
  if _DOUBLE is None:
    _DOUBLE = _lib_with_views()
  wo.install(monkeypatch)
  monkeypatch.setattr(engine_lib, 'Engine', _DOUBLE[0])
  monkeypatch.setattr(engine_lib, 'Raster', _DOUBLE[1])
