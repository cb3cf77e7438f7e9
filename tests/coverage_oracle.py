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
from spriteworld_b200 import engine as _engine
from tests import mask_oracle

_ENGINE_RENDER_COVERAGE = _engine.Engine.render_coverage   # the real one, whatever a test patches later


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


# ---------------------------------------------------------------------------------------------
# the mask double (tests/mask_oracle.py) with swb_render_coverage
# ---------------------------------------------------------------------------------------------

def _scenes(eng, records, n, records_bytes):
  """The oracle sprite arrays of the double's live envs (records None) or of n env records, as the
  mask double's swb_render_masks reads them."""
  import ctypes

  import torch

  from spriteworld_b200 import engine as engine_lib
  from tests import test_render_states_on_oracle as rs
  from tests.test_expand_on_oracle import _POOL_FIELDS
  if records is None:
    return [eng._bo.cur[e] for e in range(n)]
  assert records_bytes >= n * eng.record_bytes
  rec = np.ctypeslib.as_array((ctypes.c_uint8 * (n * eng.record_bytes)).from_address(records.value))
  h = engine_lib.EnvStates(torch.from_numpy(rec.reshape(n, -1).copy()), 1, eng.signature,
                           eng.n_slots).to_host()
  scenes = []
  for i in range(n):
    sprites = np.zeros(eng.n_slots, oracle.SPRITE_DTYPE)
    for f, g in _POOL_FIELDS:
      sprites[f] = h[g][i]
    sprites['x'], sprites['y'] = h['pos_x'][i], h['pos_y'][i]
    sprites['shape'] = rs._SHAPE_IDS[sprites['shape']]
    scenes.append(sprites)
  return scenes


class _CoverageLib(object):
  """The mask double's library plus swb_render_coverage."""

  def __init__(self, inner):
    self._inner = inner

  def __getattr__(self, name):
    return getattr(self._inner, name)

  def swb_render_coverage(self, eng, width, height, aa, records, n, records_bytes, cover, visible, area,
                          stream):
    import ctypes
    assert min(width, height, aa) >= 1 and aa * max(width, height) <= 4095
    assert n >= 0 and (records is not None or n == eng.n_envs)
    S = eng.n_slots
    spans = [(cover.value, n * height * width * 4), (visible.value, n * S * 4), (area.value, n * S * 4)]
    for i, (p, nb) in enumerate(spans):
      assert p % 4 == 0
      for q, mb in spans[:i]:
        assert not (p < q + mb and q < p + nb), 'outputs overlap'
    if n == 0:
      return 0
    scenes = _scenes(eng, records, n, records_bytes)

    def view(p, count):
      return np.ctypeslib.as_array((ctypes.c_int32 * count).from_address(p))

    out_c = view(cover.value, n * height * width).reshape(n, height, width)
    out_v, out_a = view(visible.value, n * S).reshape(n, S), view(area.value, n * S).reshape(n, S)
    rc = oracle.raster_cfg(width, height, aa)
    for i, sprites in enumerate(scenes):
      out_c[i], out_v[i], out_a[i] = render_coverage(rc, eng._tab, sprites)
    eng._launches += 1
    return 0


def _lib_with_coverage():
  MaskOracleEngine, Raster = mask_oracle._lib_with_masks()

  class CoverageOracleEngine(MaskOracleEngine):
    """The mask double with swb_render_coverage under the real Engine.render_coverage."""

    render_coverage = _ENGINE_RENDER_COVERAGE

    def __init__(self, *args, **kw):
      super().__init__(*args, **kw)
      self._lib = _CoverageLib(self._lib)

  return CoverageOracleEngine, Raster


_DOUBLE = None


def install(monkeypatch):
  """Routes the package's host layer to the oracle double with masks and coverage for the duration
  of a test: what tests/mask_oracle.install does, plus SpriteCoverage."""
  global _DOUBLE
  from spriteworld_b200 import engine as engine_lib
  if _DOUBLE is None:
    _DOUBLE = _lib_with_coverage()
  mask_oracle.install(monkeypatch)
  monkeypatch.setattr(engine_lib, 'Engine', _DOUBLE[0])
  monkeypatch.setattr(engine_lib, 'Raster', _DOUBLE[1])
