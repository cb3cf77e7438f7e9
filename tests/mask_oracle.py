"""CPU restatement of the sprite instance masks (renderers.SpriteMasks, csrc/swb_masks.cuh): test
infrastructure, built on the oracle's Pillow polygon fill (oracle.polygon_fill, the restatement
tests/test_oracle_raster.py pins against Pillow).

The definition, in Pillow: every sprite, back to front, filled with its slot + 1 into a zero 'L'
canvas of aa*W x aa*H pixels at the integer vertices PILRenderer draws, then resize((W, H), NEAREST)
-- which for an integer factor picks canvas pixel aa*j + aa//2 on both axes -- and np.flipud.
"""
import numpy as np

from oracle import oracle
from spriteworld_b200 import engine as _engine

_Engine = _engine.Engine   # the real one, whatever a test patches later


def canvas_vertices(raster_cfg, tab, sprite):
  """(n, 2) float64 canvas vertices canvas_size * (centred vertex + position), the arithmetic of the
  oracle's render (sw_env_oracle.c centred_vertex and render_ws)."""
  aa = raster_cfg.anti_aliasing
  CW, CH = aa * raster_cfg.width, aa * raster_cfg.height
  shape = int(sprite['shape'])
  n = tab.n_verts[shape]
  v = np.array([[tab.verts[shape][i][0], tab.verts[shape][i][1]] for i in range(n)], np.float64)
  cx = (sprite['m00'] * v[:, 0] + sprite['m01'] * v[:, 1]) + 0.0
  cy = (sprite['m10'] * v[:, 0] + sprite['m11'] * v[:, 1]) + 0.0
  return np.stack([float(CW) * (cx + sprite['x']), float(CH) * (cy + sprite['y'])], 1)


def render_masks(raster_cfg, tab, sprites):
  """sprites: 1-D oracle.SPRITE_DTYPE array (back to front).  Returns the (H, W) uint8 mask: slot + 1
  of the top-most sprite covering each pixel's sample point, 0 where none does."""
  aa, W, H = raster_cfg.anti_aliasing, raster_cfg.width, raster_cfg.height
  canvas = np.zeros((aa * H, aa * W, 3), np.uint8)
  for s, sp in enumerate(np.asarray(sprites, oracle.SPRITE_DTYPE).reshape(-1)):
    if sp['shape']:
      oracle.polygon_fill(canvas, canvas_vertices(raster_cfg, tab, sp), (s + 1, 0, 0))
  h = aa // 2
  return np.ascontiguousarray(canvas[h::aa, h::aa, 0][::-1])


def pillow_masks(sprites, width, height, anti_aliasing):
  """The definition itself, with Pillow, on Sprite objects (back to front)."""
  from PIL import Image, ImageDraw
  canvas = Image.new('L', (anti_aliasing * width, anti_aliasing * height), 0)
  draw = ImageDraw.Draw(canvas)
  for k, s in enumerate(sprites):
    draw.polygon([tuple(v) for v in canvas.size * s.vertices], fill=k + 1)
  return np.flipud(np.asarray(canvas.resize((width, height), Image.NEAREST)))


def huge_scene_arrays(rng, E, S, CH):
  """Factor arrays (E, S) of sprites far larger than the canvas whose outlines cross it: at a scale
  whose diameter is 40k to 120k canvas rows, each sprite is placed so that a random point of one of
  its edges lands inside the canvas.  Many of its edges then lie wholly beyond +-32768 canvas rows
  (beyond int16) while one crosses the canvas."""
  from spriteworld_b200 import constants
  names = {v: k for k, v in oracle.SHAPE_IDS.items()}
  z = np.zeros((E, S))
  a = dict(x=z.copy(), y=z.copy(), pos_f32=np.zeros((E, S), np.uint8),
           shape=rng.randint(1, 13, (E, S)).astype(np.uint8), angle=rng.uniform(0, 360, (E, S)),
           scale=z.copy(), c0=z.copy(), c1=z.copy(), c2=z.copy(), vx=z.copy(), vy=z.copy(),
           member=np.zeros((E, S), np.uint32), rgb=rng.randint(0, 256, (E, S, 3)).astype(np.uint8))
  for e in range(E):
    for s in range(S):
      v = np.asarray(constants.SHAPES[names[int(a['shape'][e, s])]], np.float64)
      scale = rng.uniform(40000, 120000) / CH / (2 * np.hypot(v[:, 0], v[:, 1]).max())
      m00, m01, m10, m11 = oracle.centred_matrix(scale, a['angle'][e, s])
      c = np.stack([m00 * v[:, 0] + m01 * v[:, 1], m10 * v[:, 0] + m11 * v[:, 1]], 1)
      i, t = rng.randint(len(c)), rng.rand()
      p = c[i] + t * (c[(i + 1) % len(c)] - c[i])           # a point of edge i, centred
      a['scale'][e, s] = scale
      a['x'][e, s], a['y'][e, s] = rng.uniform(0.1, 0.9, 2) - p
  return a


# ---------------------------------------------------------------------------------------------
# the oracle-backed engine double (tests/oracle_engine.py) with env records, swb_render_masks,
# swb_render_coverage and swb_render_soft_masks
# ---------------------------------------------------------------------------------------------

def _lib_with_masks():
  import ctypes

  from tests import coverage_oracle, oracle_engine, soft_mask_oracle
  from tests import test_render_states_on_oracle as rs

  class MaskLib(rs._RenderLib):

    def _draw(self, eng, width, height, aa, records, n, records_bytes, outs, render):
      """A mask call: outs are (ctypes pointer, ctypes type, shape of one row) of each output, and
      render(raster_cfg, tab, sprites) gives one row of each (a tuple of several)."""
      assert min(width, height, aa) >= 1 and aa * max(width, height) <= 4095
      assert n >= 0 and (records is not None or n == eng.n_envs)
      spans = [(p.value, ctypes.sizeof(ct), n * int(np.prod(shape)) * ctypes.sizeof(ct)) for p, ct, shape in outs]
      for i, (p, align, nb) in enumerate(spans):
        assert p and p % align == 0
        for q, _, mb in spans[:i]:
          assert not (p < q + mb and q < p + nb), 'outputs overlap'
      if n == 0:
        return 0
      if records is None:
        scenes = [eng._bo.cur[e] for e in range(n)]
      else:
        assert records_bytes >= n * eng.record_bytes
        scenes = oracle_engine.record_sprites(eng, oracle_engine.states_at(eng, records, n))
      views = [np.ctypeslib.as_array((ct * (n * int(np.prod(shape)))).from_address(p.value)).reshape((n,) + shape)
               for p, ct, shape in outs]
      rc = oracle.raster_cfg(width, height, aa)
      for i, sprites in enumerate(scenes):
        rows = render(rc, eng._tab, sprites)
        for view, row in zip(views, rows if isinstance(rows, tuple) else (rows,)):
          view[i] = row
      eng._launches += 1
      return 0

    def swb_render_masks(self, eng, width, height, aa, records, n, records_bytes, masks, stream):
      return self._draw(eng, width, height, aa, records, n, records_bytes,
                        [(masks, ctypes.c_uint8, (height, width))], render_masks)

    def swb_render_coverage(self, eng, width, height, aa, records, n, records_bytes, cover, visible, area,
                            stream):
      S = eng.n_slots
      return self._draw(eng, width, height, aa, records, n, records_bytes,
                        [(cover, ctypes.c_int32, (height, width)), (visible, ctypes.c_int32, (S,)),
                         (area, ctypes.c_int32, (S,))], coverage_oracle.render_coverage)

    def swb_render_soft_masks(self, eng, width, height, aa, records, n, records_bytes, soft, stream):
      assert aa <= 15
      return self._draw(eng, width, height, aa, records, n, records_bytes,
                        [(soft, ctypes.c_uint8, (eng.n_slots, height, width))], soft_mask_oracle.render_soft_masks)

  class MaskOracleEngine(rs.RenderStatesOracleEngine):
    """The records double with the mask calls under the real Engine.render_masks, render_coverage
    and render_soft_masks."""

    render_masks = _Engine.render_masks
    render_coverage = _Engine.render_coverage
    render_soft_masks = _Engine.render_soft_masks

    def __init__(self, *args, **kw):
      super().__init__(*args, **kw)
      self._lib = MaskLib()

  return MaskOracleEngine, rs.RenderStatesOracleRaster


_DOUBLE = None


def install(monkeypatch):
  """Routes the package's host layer to the oracle double with SpriteMasks, SpriteCoverage and
  SoftSpriteMasks (and env records, and swb_render_states) for the duration of a test: what
  tests/oracle_engine.install does, plus the mask calls."""
  global _DOUBLE
  from spriteworld_b200 import engine as engine_lib
  from tests import oracle_engine
  if _DOUBLE is None:
    _DOUBLE = _lib_with_masks()
  oracle_engine.install(monkeypatch)
  monkeypatch.setattr(engine_lib, 'Engine', _DOUBLE[0])
  monkeypatch.setattr(engine_lib, 'Raster', _DOUBLE[1])
