"""The window restatement (tests/window_oracle.py) against Pillow itself and against oracle.render:
the definition of swb_render_windows and renderers.SpriteGlimpses, pinned on the CPU before the
kernel is held to it (tests/test_gpu_windows.py)."""
import numpy as np
import pytest

from oracle import oracle
from spriteworld_b200 import constants
from spriteworld_b200 import sprite as sprite_lib
from tests import window_oracle as wo

PIL = pytest.importorskip('PIL')

SHAPES = [n for n in oracle.SHAPE_IDS if oracle.SHAPE_IDS[n]]
TAB = oracle.shape_table(constants.SHAPES)


def _scene(rng, n, far=False):
  """(Sprite list, SPRITE_DTYPE records) of n random sprites, every shape in turn."""
  sprites, recs = [], []
  for k in range(n):
    shape = SHAPES[(k + rng.randint(len(SHAPES))) % len(SHAPES)]
    x, y = rng.uniform(-0.3, 1.3, 2) if not far else rng.uniform(-40, 40, 2)
    angle, scale = float(rng.uniform(0, 360)), float(np.exp(rng.uniform(np.log(0.02), np.log(0.4))))
    rgb = tuple(int(c) for c in rng.randint(0, 256, 3))
    sprites.append(sprite_lib.Sprite(x=x, y=y, shape=shape, angle=angle, scale=scale, c0=rgb[0], c1=rgb[1],
                                     c2=rgb[2]))
    recs.append(oracle.sprite_record(x, y, oracle.SHAPE_IDS[shape], angle, scale, rgb))
  return sprites, np.array(recs, oracle.SPRITE_DTYPE).reshape(-1)


def _window(rng, zoom, aspect=1.0, off=False):
  w, h = 1.0 / zoom, aspect / zoom
  cx, cy = (rng.uniform(1.5, 3.0, 2) * rng.choice([-1, 1], 2)) if off else rng.uniform(-0.2, 1.2, 2)
  return (cx - 0.5 * w, cy - 0.5 * h, cx + 0.5 * w, cy + 0.5 * h)


def test_full_scene_window_is_the_oracle_frame():
  rng = np.random.RandomState(5)
  for W, H, aa, bg in ((64, 64, 1, (0, 0, 0)), (32, 48, 3, (9, 30, 200)), (20, 12, 7, (255, 255, 255))):
    rc = oracle.raster_cfg(W, H, aa, bg)
    for _ in range(6):
      _, recs = _scene(rng, rng.randint(1, 9))
      got, bad = wo.render_window(rc, TAB, recs, (0.0, 0.0, 1.0, 1.0))
      assert not bad and np.array_equal(got, oracle.render(rc, TAB, recs)), (W, H, aa)


@pytest.mark.parametrize('aa', list(range(1, 14)) + [14, 20])
def test_windows_match_pillow(aa):
  rng = np.random.RandomState(100 + aa)
  W, H = (24, 16) if aa < 14 else (12, 8)   # aa >= 14: short frames keep the canvas small
  n_checked = 0
  for t in range(10):
    zoom = float(np.exp(rng.uniform(np.log(0.25), np.log(64.0))))
    window = _window(rng, zoom, aspect=rng.choice([1.0, 0.5, 3.0]), off=t == 9)
    sprites, recs = _scene(rng, 1 + t % 5, far=t == 8)
    rc = oracle.raster_cfg(W, H, aa, (17, 80, 140))
    got, bad = wo.render_window(rc, TAB, recs, window)
    if bad:
      continue
    ref = wo.pillow_window(sprites, W, H, aa, window, bg=(17, 80, 140))
    assert np.array_equal(got, ref), (aa, zoom, window)
    n_checked += 1
  assert n_checked >= 8


def test_every_shape_zoomed_on_itself():
  rng = np.random.RandomState(7)
  for shape in SHAPES:
    for zoom in (0.25, 1.0, 8.0, 64.0):
      s = sprite_lib.Sprite(x=0.4, y=0.6, shape=shape, angle=float(rng.uniform(0, 360)), scale=0.13,
                            c0=200, c1=40, c2=90)
      rec = np.array([oracle.sprite_record(0.4, 0.6, oracle.SHAPE_IDS[shape], s.angle, 0.13, (200, 40, 90))],
                     oracle.SPRITE_DTYPE)
      win = (0.4 - 0.5 / zoom, 0.6 - 0.5 / zoom, 0.4 + 0.5 / zoom, 0.6 + 0.5 / zoom)
      rc = oracle.raster_cfg(32, 32, 5)
      got, bad = wo.render_window(rc, TAB, rec, win)
      assert not bad and np.array_equal(got, wo.pillow_window([s], 32, 32, 5, win)), (shape, zoom)


def test_far_zoom_windows_match_pillow():
  """Windows zoomed so far that the sprites reach 2^15 .. 2^29 canvas units from the window's origin,
  both signs on both axes, crossing the canvas: the restatement is Pillow's frame, and no vertex is
  flagged (every one stays below 2^30)."""
  rng = np.random.RandomState(11)
  W, H, aa = 16, 12, 3
  rc = oracle.raster_cfg(W, H, aa, (3, 4, 5))
  reach = []
  for t in range(8):
    sprites, recs = _scene(rng, 2)
    s = sprites[t % 2]
    v = np.asarray(s.vertices, np.float64)
    k = rng.randint(len(v))
    p = v[k] + rng.rand() * (v[(k + 1) % len(v)] - v[k])     # a point of one of its edges
    allv = np.concatenate([np.asarray(q.vertices, np.float64) for q in sprites])
    far = 2.0 ** rng.uniform(15, 29)
    sx = min(far / np.ptp(v, 0).max(), 2.0 ** 29 / np.abs(allv - p).max())
    w, h = W * aa / sx, H * aa / sx
    win = (p[0] - w * rng.uniform(0.2, 0.8), p[1] - h * rng.uniform(0.2, 0.8))
    win = win + (win[0] + w, win[1] + h)
    got, bad = wo.render_window(rc, TAB, recs, win)
    assert not bad, (t, win)
    assert np.array_equal(got, wo.pillow_window(sprites, W, H, aa, win, bg=(3, 4, 5))), (t, win)
    reach.append(max(np.abs(wo.window_vertices(rc, TAB, r, win)).max() for r in recs))
  assert max(reach) > 2.0 ** 28 and min(reach) > 2.0 ** 15, reach


def test_bad_window_conditions():
  rc = oracle.raster_cfg(16, 16, 2)
  _, recs = _scene(np.random.RandomState(3), 3)
  for win in ((0.5, 0.0, 0.5, 1.0), (0.6, 0.0, 0.5, 1.0), (0.0, 1.0, 1.0, 0.0), (np.nan, 0, 1, 1),
              (0, 0, np.inf, 1), (-np.inf, 0, 1, 1)):
    frame, bad = wo.render_window(rc, TAB, recs, win)
    assert bad and not frame.any(), win
  # a window so small that a vertex lands 2^30 canvas pixels or more from its origin
  x = float(recs['x'][0])
  tiny = (x, 0.0, x + 1e-12, 1.0)
  assert wo.bad_window(rc, TAB, recs, tiny)
  # empty slots are not looked at
  empty = recs.copy()
  empty['shape'] = 0
  assert not wo.bad_window(rc, TAB, empty, tiny)
  assert not wo.bad_window(rc, TAB, recs, (0.0, 0.0, 1.0, 1.0))
