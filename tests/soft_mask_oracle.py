"""CPU restatement of the soft sprite masks (renderers.SoftSpriteMasks, the mask kernel's soft mode
in csrc/swb_masks.cuh): test infrastructure, built on the oracle's Pillow polygon fill
(oracle.polygon_fill, the restatement tests/test_oracle_raster.py pins against Pillow), as
tests/mask_oracle.py is.

The definition, in Pillow: the label canvas of mask_oracle.pillow_masks (every sprite back to
front, fill k + 1, into a zero 'L' canvas of aa*W x aa*H pixels) before its resize;
L = np.flipud(canvas).reshape(H, aa, W, aa); soft[k] = (L == k + 1).sum((1, 3)).
"""
import numpy as np

from oracle import oracle
from tests import mask_oracle


def block_counts(labels, n_slots, W, H, aa):
  """(n_slots, H, W) uint8 counts of labels k + 1 in each aa x aa block of an (aa H, aa W) label
  canvas whose rows are already flipped."""
  L = np.asarray(labels).reshape(H, aa, W, aa)
  out = np.zeros((n_slots, H, W), np.uint8)
  for k in range(n_slots):
    out[k] = (L == k + 1).sum((1, 3))
  return out


def render_soft_masks(raster_cfg, tab, sprites):
  """sprites: 1-D oracle.SPRITE_DTYPE array, one per slot (back to front).  Returns the (S, H, W)
  uint8 soft masks: per slot, the canvas pixels of each pixel's aa x aa block where it is top-most."""
  aa, W, H = raster_cfg.anti_aliasing, raster_cfg.width, raster_cfg.height
  sprites = np.asarray(sprites, oracle.SPRITE_DTYPE).reshape(-1)
  assert aa <= 15 and len(sprites) <= 32
  canvas = np.zeros((aa * H, aa * W, 3), np.uint8)
  for s, sp in enumerate(sprites):
    if sp['shape']:
      oracle.polygon_fill(canvas, mask_oracle.canvas_vertices(raster_cfg, tab, sp), (s + 1, 0, 0))
  return block_counts(canvas[::-1, :, 0], len(sprites), W, H, aa)


def pillow_soft_masks(sprites, width, height, anti_aliasing):
  """The definition itself, with Pillow, on Sprite objects (back to front): (len(sprites), H, W)."""
  from PIL import Image, ImageDraw
  canvas = Image.new('L', (anti_aliasing * width, anti_aliasing * height), 0)
  draw = ImageDraw.Draw(canvas)
  for k, s in enumerate(sprites):
    draw.polygon([tuple(v) for v in canvas.size * s.vertices], fill=k + 1)
  return block_counts(np.flipud(np.asarray(canvas)), len(sprites), width, height, anti_aliasing)


def check_properties(soft, mask, aa, what=()):
  """The properties SoftSpriteMasks states against the SpriteMasks mask of the same state: at aa 1
  soft[k] == (mask == k + 1); at any aa, mask == k + 1 implies soft[k] >= 1, mask == 0 implies a
  background sample, and the counts of a pixel sum to at most aa**2."""
  soft, mask = np.asarray(soft), np.asarray(mask)
  S = soft.shape[0]
  total = soft.astype(np.int64).sum(0)
  assert (total <= aa * aa).all(), what
  assert (total[mask == 0] < aa * aa).all(), what
  for k in range(S):
    if aa == 1:
      assert np.array_equal(soft[k], (mask == k + 1).astype(np.uint8)), (what, k)
    assert (soft[k][mask == k + 1] >= 1).all(), (what, k)
