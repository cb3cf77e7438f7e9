"""CPU restatement of the amodal sprite coverage (renderers.SpriteCoverage, the mask kernel's
coverage mode in csrc/swb_masks.cuh): test infrastructure, built on the oracle's Pillow polygon fill
(oracle.polygon_fill, the restatement tests/test_oracle_raster.py pins against Pillow), as
tests/mask_oracle.py is.

The definition, in Pillow: every sprite drawn ALONE with fill 1 into its own zero 'L' canvas of
aa*W x aa*H pixels at the integer vertices PILRenderer draws, then resize((W, H), NEAREST) -- which
for an integer factor picks canvas pixel aa*j + aa//2 on both axes -- and np.flipud, gives bit k's
plane for sprite k.  visible[k] counts the pixels whose highest set bit is k, area[k] those whose
bit k is set.
"""
import numpy as np

from oracle import oracle
from tests import mask_oracle


def counts(cover, n_slots):
  """(visible, area), int32 (n_slots,) each, of an (H, W) int32 coverage."""
  c = np.asarray(cover).view(np.uint32)
  bits = (c[None] >> np.arange(n_slots, dtype=np.uint32)[:, None, None]) & 1
  area = bits.reshape(n_slots, c.size).sum(1).astype(np.int32)
  top = modal(cover)
  visible = np.bincount(top.reshape(-1), minlength=n_slots + 1)[1:n_slots + 1].astype(np.int32)
  return visible, area


def modal(cover):
  """The highest set bit + 1 of every pixel, 0 where cover is 0 (the SpriteMasks mask, as int64)."""
  c = np.asarray(cover).view(np.uint32).astype(np.int64)
  top = np.zeros(c.shape, np.int64)
  for k in range(32):
    top[(c >> k) & 1 == 1] = k + 1
  return top


def render_coverage(raster_cfg, tab, sprites):
  """sprites: 1-D oracle.SPRITE_DTYPE array, one per slot.  Returns (cover, visible, area): the
  (H, W) int32 coverage, bit k set where slot k's fill covers the pixel's sample point, and the
  int32 (S,) counts."""
  aa, W, H = raster_cfg.anti_aliasing, raster_cfg.width, raster_cfg.height
  sprites = np.asarray(sprites, oracle.SPRITE_DTYPE).reshape(-1)
  assert len(sprites) <= 32
  canvas = np.zeros((aa * H, aa * W, 3), np.uint8)
  cover = np.zeros((H, W), np.uint32)
  h = aa // 2
  for s, sp in enumerate(sprites):
    if not sp['shape']:
      continue
    canvas[...] = 0
    oracle.polygon_fill(canvas, mask_oracle.canvas_vertices(raster_cfg, tab, sp), (1, 0, 0))
    cover |= canvas[h::aa, h::aa, 0][::-1].astype(np.uint32) << np.uint32(s)
  cover = np.ascontiguousarray(cover).view(np.int32)
  return (cover,) + counts(cover, len(sprites))


def pillow_coverage(sprites, width, height, anti_aliasing):
  """The definition itself, with Pillow, on Sprite objects: (H, W) int32, bit i for sprites[i]."""
  from PIL import Image, ImageDraw
  cover = np.zeros((height, width), np.uint32)
  for k, s in enumerate(sprites):
    canvas = Image.new('L', (anti_aliasing * width, anti_aliasing * height), 0)
    ImageDraw.Draw(canvas).polygon([tuple(v) for v in canvas.size * s.vertices], fill=1)
    plane = np.flipud(np.asarray(canvas.resize((width, height), Image.NEAREST)))
    cover |= plane.astype(np.uint32) << np.uint32(k)
  return cover.view(np.int32)
