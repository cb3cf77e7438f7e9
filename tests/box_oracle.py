"""CPU restatement of the sprite bounding boxes (renderers.SpriteBoxes, the mask kernel's box mode in
csrc/swb_masks.cuh): test infrastructure, built on the coverage restatement tests/coverage_oracle.py.

box(P) of a set P of pixels (i, j) is (min j, min i, max j + 1, max i + 1), half-open (x0, y0, x1, y1)
in pixels of the flipped image, and (0, 0, 0, 0) for an empty P.  For slot k, visible_box is box of
the pixels whose highest set bit of the coverage is k (the SpriteMasks mask is k + 1 there) and
amodal_box box of those whose bit k is set; visible and area count them, as SpriteCoverage does.
"""
import ctypes

import numpy as np

from tests import coverage_oracle, mask_oracle

_Engine = mask_oracle._Engine


def box(plane):
  """int32 (4,) box of the True pixels of a 2-D plane: row and column extents."""
  rows, cols = np.flatnonzero(plane.any(1)), np.flatnonzero(plane.any(0))
  if not len(rows):
    return np.zeros(4, np.int32)
  return np.array([cols[0], rows[0], cols[-1] + 1, rows[-1] + 1], np.int32)


def boxes_of_cover(cover, n_slots):
  """(visible_box, amodal_box, visible, area) of an (H, W) int32 coverage: int32 (n_slots, 4) twice,
  then int32 (n_slots,) twice."""
  bits = np.asarray(cover).view(np.uint32)
  top = coverage_oracle.modal(cover)
  visible_box = np.stack([box(top == k + 1) for k in range(n_slots)]).reshape(n_slots, 4)
  amodal_box = np.stack([box((bits >> np.uint32(k)) & 1 == 1) for k in range(n_slots)]).reshape(n_slots, 4)
  return (visible_box, amodal_box) + coverage_oracle.counts(cover, n_slots)


def boxes_of_covers(covers, n_slots):
  """boxes_of_cover of each of n coverages (n, H, W) at once: int32 (n, n_slots, 4) twice, then
  int32 (n, n_slots) twice."""
  bits = np.asarray(covers).view(np.uint32)
  top = coverage_oracle.modal(covers)
  n, H, W = bits.shape
  vb, ab = np.zeros((n, n_slots, 4), np.int32), np.zeros((n, n_slots, 4), np.int32)
  visible, area = np.zeros((n, n_slots), np.int32), np.zeros((n, n_slots), np.int32)
  for k in range(n_slots):
    for b, count, plane in ((vb, visible, top == k + 1), (ab, area, (bits >> np.uint32(k)) & 1 == 1)):
      rows, cols = plane.any(2), plane.any(1)
      full = rows.any(1)
      b[full, k] = np.stack([cols.argmax(1), rows.argmax(1), W - cols[:, ::-1].argmax(1),
                             H - rows[:, ::-1].argmax(1)], 1)[full]
      count[:, k] = plane.reshape(n, -1).sum(1)
  return vb, ab, visible, area


def render_boxes(raster_cfg, tab, sprites):
  """sprites: 1-D oracle.SPRITE_DTYPE array, one per slot.  Returns (visible_box, amodal_box,
  visible, area) of their coverage."""
  cover, _, _ = coverage_oracle.render_coverage(raster_cfg, tab, sprites)
  return boxes_of_cover(cover, len(np.asarray(sprites).reshape(-1)))


def pillow_boxes(sprites, width, height, anti_aliasing):
  """The definition itself, on Sprite objects: Pillow's coverage planes, the top-most set bit of
  each pixel, and each box as torchvision.ops.masks_to_boxes writes it, plus (0, 0, 1, 1)."""
  cover = coverage_oracle.pillow_coverage(sprites, width, height, anti_aliasing)
  top = coverage_oracle.modal(cover)
  n = len(sprites)
  out = np.zeros((2, n, 4), np.int32)
  for k in range(n):
    for which, plane in enumerate((top == k + 1, (cover.view(np.uint32) >> np.uint32(k)) & 1 == 1)):
      y, x = np.nonzero(plane)
      if len(x):
        out[which, k] = (x.min(), y.min(), x.max() + 1, y.max() + 1)
  visible = np.array([(top == k + 1).sum() for k in range(n)], np.int32)
  area = np.array([((cover.view(np.uint32) >> np.uint32(k)) & 1).sum() for k in range(n)], np.int32)
  return out[0], out[1], visible, area


def check_invariants(visible_box, amodal_box, visible, area, width, height, what=()):
  """What SpriteBoxes states of any observation, over a leading slot axis (any leading axes)."""
  vb, ab = np.asarray(visible_box).reshape(-1, 4), np.asarray(amodal_box).reshape(-1, 4)
  v, a = np.asarray(visible).reshape(-1), np.asarray(area).reshape(-1)
  assert (v <= a).all(), what
  for b, c in ((vb, v), (ab, a)):
    empty = c == 0
    assert (b[empty] == 0).all(), what
    full = b[~empty]
    assert (full[:, 0] >= 0).all() and (full[:, 1] >= 0).all(), what
    assert (full[:, 0] < full[:, 2]).all() and (full[:, 1] < full[:, 3]).all(), what
    assert (full[:, 2] <= width).all() and (full[:, 3] <= height).all(), what
    size = (full[:, 2] - full[:, 0]).astype(np.int64) * (full[:, 3] - full[:, 1])
    assert (size >= c[~empty]).all(), what
  seen = v > 0   # the visible box lies in the amodal box
  assert (vb[seen, :2] >= ab[seen, :2]).all() and (vb[seen, 2:] <= ab[seen, 2:]).all(), what


# ---------------------------------------------------------------------------------------------
# the mask double (tests/mask_oracle.py) with swb_render_boxes and Engine.render_boxes
# ---------------------------------------------------------------------------------------------

def _swb_render_boxes(self, eng, width, height, aa, records, n, records_bytes, visible_box, amodal_box,
                      visible, area, stream):
  S = eng.n_slots
  rc = self._draw(eng, width, height, aa, records, n, records_bytes,
                  [(visible_box, ctypes.c_int32, (S, 4)), (amodal_box, ctypes.c_int32, (S, 4)),
                   (visible, ctypes.c_int32, (S,)), (area, ctypes.c_int32, (S,))], render_boxes)
  if rc == 0 and n > 0:
    eng._launches += 1   # the call is two launches: the mask kernel and the decoding of the boxes
  return rc


def _lib_with_boxes():
  mask_engine, raster = mask_oracle._lib_with_masks()

  class BoxOracleEngine(mask_engine):
    """The mask double with swb_render_boxes under the real Engine.render_boxes."""

    render_boxes = _Engine.render_boxes
    _lib_cls = None

    def __init__(self, *args, **kw):
      super().__init__(*args, **kw)
      cls = type(self)
      if cls._lib_cls is None:
        cls._lib_cls = type('BoxLib', (type(self._lib),), {'swb_render_boxes': _swb_render_boxes})
      self._lib = cls._lib_cls()

  return BoxOracleEngine, raster


_DOUBLE = None


def install(monkeypatch):
  """Routes the package's host layer to the mask double with SpriteBoxes for the duration of a test:
  what tests/mask_oracle.install does, plus swb_render_boxes."""
  global _DOUBLE
  from spriteworld_b200 import engine as engine_lib
  if _DOUBLE is None:
    _DOUBLE = _lib_with_boxes()
  mask_oracle.install(monkeypatch)
  monkeypatch.setattr(engine_lib, 'Engine', _DOUBLE[0])
  monkeypatch.setattr(engine_lib, 'Raster', _DOUBLE[1])
