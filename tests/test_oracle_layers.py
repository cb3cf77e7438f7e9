"""The layer restatement (tests/layer_oracle.py) against Pillow itself: the definition of
swb_render_views and renderers.SpriteLayers, pinned on the CPU before the kernel is held to it
(tests/test_gpu_layers.py)."""
import numpy as np
import pytest

from oracle import oracle
from spriteworld_b200 import sprite as sprite_lib
from tests import coverage_oracle
from tests import layer_oracle as lo
from tests import window_oracle as wo
from tests.test_oracle_windows import SHAPES, TAB, _scene, _window

PIL = pytest.importorskip('PIL')

FULL = (0.0, 0.0, 1.0, 1.0)


def _subsets(rng, n):
  """Draw masks of n slots: none, all, each singleton, each complement of one, and random ones."""
  out = [np.zeros(n, bool), np.ones(n, bool)]
  for k in range(n):
    one = np.zeros(n, bool)
    one[k] = True
    out += [one, ~one]
  out += [rng.rand(n) < 0.5 for _ in range(3)]
  return out


def _pillow(sprites, draw, W, H, aa, window, bg):
  return wo.pillow_window([s for s, d in zip(sprites, draw) if d], W, H, aa, window, bg=bg)


@pytest.mark.parametrize('aa', list(range(1, 14)) + [14, 20])
def test_layers_match_pillow(aa):
  rng = np.random.RandomState(300 + aa)
  W, H = (24, 16) if aa < 14 else (12, 8)   # aa >= 14: short frames keep the canvas small
  bg = (17, 80, 140)
  rc = oracle.raster_cfg(W, H, aa, bg)
  n_checked = 0
  for t in range(4):
    sprites, recs = _scene(rng, 2 + t)
    zoom = float(np.exp(rng.uniform(np.log(0.5), np.log(16.0))))
    for window in (FULL, _window(rng, zoom)):
      for draw in _subsets(rng, len(recs)):
        got, bad = lo.render_layer(rc, TAB, recs, window, draw)
        if bad:
          continue
        assert np.array_equal(got, _pillow(sprites, draw, W, H, aa, window, bg)), (aa, t, window, draw)
        n_checked += 1
  assert n_checked >= 80


def test_every_shape_alone_and_removed():
  rng = np.random.RandomState(8)
  rc = oracle.raster_cfg(32, 32, 5, (5, 6, 7))
  for shape in SHAPES:
    sprites, recs = _scene(rng, 3)
    k = rng.randint(3)
    recs['shape'][k] = oracle.SHAPE_IDS[shape]
    s = sprites[k]
    sprites[k] = sprite_lib.Sprite(x=float(recs['x'][k]), y=float(recs['y'][k]), shape=shape, angle=s.angle,
                                   scale=s.scale, c0=s.color[0], c1=s.color[1], c2=s.color[2])
    one = np.arange(3) == k
    x, y = float(recs['x'][k]), float(recs['y'][k])
    for window in (FULL, (x - 0.1, y - 0.1, x + 0.1, y + 0.1)):
      for draw in (one, ~one):
        got, bad = lo.render_layer(rc, TAB, recs, window, draw)
        assert not bad and np.array_equal(got, _pillow(sprites, draw, 32, 32, 5, window, (5, 6, 7))), (shape, draw)


def test_all_drawn_is_the_window_frame_and_none_drawn_the_background():
  rng = np.random.RandomState(9)
  for W, H, aa, bg in ((16, 12, 1, (0, 0, 0)), (20, 20, 4, (9, 30, 200)), (12, 8, 7, (255, 255, 255))):
    rc = oracle.raster_cfg(W, H, aa, bg)
    for t in range(4):
      _, recs = _scene(rng, 1 + 2 * t)
      for window in (FULL, _window(rng, 3.0)):
        assert all(np.array_equal(a, b) for a, b in zip(
            lo.render_layer(rc, TAB, recs, window, np.ones(len(recs), bool)), wo.render_window(rc, TAB, recs, window)))
        got, bad = lo.render_layer(rc, TAB, recs, window, np.zeros(len(recs), bool))
        assert not bad and (got == np.asarray(bg, np.uint8)).all()
      # the full window with every slot drawn is the oracle's frame
      assert np.array_equal(lo.render_layer(rc, TAB, recs, FULL, np.ones(len(recs), bool))[0],
                            oracle.render(rc, TAB, recs))


def test_one_hot_layers_at_aa_1_are_the_coverage_bits():
  rng = np.random.RandomState(10)
  bg = np.array([12, 34, 56], np.uint8)
  for W, H in ((16, 16), (33, 17), (8, 40)):
    rc = oracle.raster_cfg(W, H, 1, tuple(bg))
    for t in range(3):
      _, recs = _scene(rng, 2 + 2 * t)
      cover = coverage_oracle.render_coverage(rc, TAB, recs)[0]
      for k in range(len(recs)):
        got, bad = lo.render_layer(rc, TAB, recs, FULL, np.arange(len(recs)) == k)
        rgb = np.asarray(recs['rgb'][k], np.uint8)
        want = np.where(((cover >> k) & 1).astype(bool)[..., None], rgb, bg)
        assert not bad and np.array_equal(got, want), (W, H, t, k)


def test_a_far_sprite_left_out_does_not_flag_the_view():
  rc = oracle.raster_cfg(16, 16, 2)
  _, recs = _scene(np.random.RandomState(3), 3)
  recs['x'][1] = 2.0 ** 40     # every vertex of slot 1 is 2^30 canvas pixels or more away
  for window in (FULL, (0.2, 0.2, 0.6, 0.6)):
    assert lo.render_layer(rc, TAB, recs, window, np.ones(3, bool))[1]
    frame, bad = lo.render_layer(rc, TAB, recs, window, np.array([True, False, True]))
    assert not bad and np.array_equal(frame, wo.render_window(rc, TAB, lo.drawn_sprites(recs, [1, 0, 1]), window)[0])
    # the far sprite drawn alone flags its view, whose frame is zeros
    frame, bad = lo.render_layer(rc, TAB, recs, window, np.array([False, True, False]))
    assert bad and not frame.any()
