"""The contained-position sampler (csrc/swb_contained.cuh) built for the CPU
(scene_program.sample_contained_on_host) against a NumPy restatement of its contract, bit for bit,
and the distribution it draws.

The contract, for sample s of row i under seed `seed`:
  sprites  the slots whose shape id has a vertex table, in slot order; m of them (none: NO_SPRITE)
  stream   np.random.Philox(counter=(s << 64) + (i << 128) - 1, key=(seed, CONTAINED_DOMAIN)),
           successive words; uniform = (w >> 11) * 2**-53
  choice   k = (word * m) >> 64, the k-th sprite
  box      lo / hi = min / max of the centred vertices (m00 ax + m01 ay) + 0.0, (m10 ax + m11 ay) + 0.0
  tries    ux, uy; c = pos + (lo + (hi - lo) u); accepted if sprite.polygon_contains(centred, c - pos);
           CONTAINED_MAX_TRIES tries at most (SAMPLE_TRIES)
The reference's sprite.Sprite.contains_point holds every accepted position inside its sprite.
"""
import importlib

import numpy as np
import pytest
from scipy import stats

from spriteworld_b200 import _native, constants, scene, scene_program
from spriteworld_b200 import sprite as sprite_lib
from spriteworld_b200 import sprite_generators as gen

M64 = (1 << 64) - 1
CONFIGS = ['cobra.' + n for n in ('clustering', 'exploration', 'goal_finding_more_distractors',
                                  'goal_finding_more_targets', 'goal_finding_new_position',
                                  'goal_finding_new_shape', 'sorting')] + \
          ['examples.' + n for n in ('goal_finding_clustering', 'goal_finding_embodied',
                                     'goal_finding_random_goal')]
FIELDS = ('x', 'y', 'm00', 'm01', 'm10', 'm11')


class Words(object):
  """The draw words of sample s of row i under `seed`."""

  def __init__(self, seed, i, s):
    c = ((int(i) << 128) + (int(s) << 64) - 1) % (1 << 256)
    ctr = np.array([(c >> (64 * q)) & M64 for q in range(4)], np.uint64)
    self._bg = np.random.Philox(counter=ctr, key=np.array([int(seed) & M64, _native.CONTAINED_DOMAIN], np.uint64))
    self._buf, self._pos = [], 0

  def next(self):
    if self._pos == len(self._buf):
      self._buf, self._pos = self._bg.random_raw(16).tolist(), 0
    self._pos += 1
    return self._buf[self._pos - 1]

  def uniform(self):
    return (self.next() >> 11) * 2.0 ** -53


_NAMES = (None,) + constants.SHAPE_NAMES


def restate(rows, seed, n_samples, max_tries=_native.CONTAINED_MAX_TRIES):
  """(position, slot, status) of the contract above, in NumPy and Python floats."""
  shape = np.asarray(rows['shape'])
  n, S = shape.shape
  pos = np.full((n, n_samples, 2), np.nan)
  slot = np.full((n, n_samples), -1, np.int8)
  status = np.zeros((n, n_samples), np.uint8)
  for i in range(n):
    occupied = [j for j in range(S) if 0 < shape[i, j] < len(_NAMES)]
    for s in range(n_samples):
      if not occupied:
        status[i, s] = _native.ENV_NO_SPRITE
        continue
      w = Words(seed, i, s)
      j = occupied[(w.next() * len(occupied)) >> 64]
      x, y = float(rows['x'][i, j]), float(rows['y'][i, j])
      matrix = np.array([[rows['m00'][i, j], rows['m01'][i, j]], [rows['m10'][i, j], rows['m11'][i, j]]])
      centred = sprite_lib._apply(matrix, constants.SHAPES[_NAMES[shape[i, j]]])
      lo, hi = centred.min(0), centred.max(0)
      status[i, s] = _native.ENV_SAMPLE_TRIES
      for _ in range(max_tries):
        ux = w.uniform()
        uy = w.uniform()
        cx = x + (float(lo[0]) + (float(hi[0]) - float(lo[0])) * ux)
        cy = y + (float(lo[1]) + (float(hi[1]) - float(lo[1])) * uy)
        if sprite_lib.polygon_contains(centred, cx - x, cy - y):
          pos[i, s], slot[i, s], status[i, s] = (cx, cy), j, 0
          break
  return pos, slot, status


def _assert_same(got, want, what):
  gp, gk, gs = got
  wp, wk, ws = want
  assert np.array_equal(gp.view(np.uint64), wp.view(np.uint64)), (what, np.argwhere(gp.view(np.uint64) != wp.view(np.uint64))[:4])
  assert np.array_equal(gk, wk) and np.array_equal(gs, ws), what


def _rows_of_sprites(scenes, S):
  """Scene batch (n, S) of lists of Sprite objects, packed by scene.arrays_from_layout."""
  return scene.arrays_from_layout(gen.layout_from_sprite_lists(scenes), S)


def _check_inside(scenes, S, got):
  """Every accepted position is inside its slot's sprite by Sprite.contains_point."""
  pos, slot, status = got
  for i, sc in enumerate(scenes):
    for s in range(pos.shape[1]):
      if status[i, s] == 0:
        sp = sc[int(slot[i, s]) - (S - len(sc))]
        assert sp.contains_point(pos[i, s]), (i, s)


@pytest.mark.parametrize('name', CONFIGS)
def test_config_scenes_equal_the_restatement(name):
  cfg = importlib.import_module('spriteworld_b200.configs.' + name).get_config('train')
  init = cfg['init_sprites']
  np.random.seed(len(name))
  scenes = [init() for _ in range(24)]
  S = max(getattr(init, 'max_sprites', 0) or 0, max(len(sc) for sc in scenes))
  rows = _rows_of_sprites(scenes, S)
  for seed, n_samples in ((0, 3), (2 ** 64 - 1, 2), (12345678901234567, 5)):
    got = scene_program.sample_contained_on_host(rows, seed, n_samples)
    _assert_same(got, restate(rows, seed, n_samples), (name, seed))
    _check_inside(scenes, S, got)
    assert (got[2] == 0).all()


def _shape_scenes(angles, f32, xy=(0.4, 0.6), scale=0.13):
  """One scene per shape and angle: the shape alone, at a float32 or float64 position."""
  scenes = []
  for name in constants.SHAPE_NAMES:
    for a in angles:
      x, y = (np.float32(xy[0]), np.float32(xy[1])) if f32 else xy
      scenes.append([sprite_lib.Sprite(x=x, y=y, shape=name, angle=a, scale=scale)])
  return scenes


@pytest.mark.parametrize('f32', [False, True], ids=['f64', 'f32'])
def test_every_shape_at_every_angle_equals_the_restatement(f32):
  angles = list(range(0, 360, 15)) + [7.3, 101.25, -33.0, 359.9]
  scenes = _shape_scenes(angles, f32)
  rows = _rows_of_sprites(scenes, 1)
  assert (rows['pos_f32'] == (1 if f32 else 0)).all()
  got = scene_program.sample_contained_on_host(rows, 77, 4)
  _assert_same(got, restate(rows, 77, 4), f32)
  _check_inside(scenes, 1, got)
  assert (got[2] == 0).all()


def test_out_of_frame_mixed_and_empty_scenes_equal_the_restatement():
  rng = np.random.RandomState(5)
  scenes = []
  for i in range(40):
    n = i % 5     # every fifth scene is empty
    scenes.append([sprite_lib.Sprite(x=rng.uniform(-0.3, 1.3), y=rng.uniform(-0.3, 1.3),
                                     shape=constants.SHAPE_NAMES[rng.randint(12)], angle=rng.uniform(0, 360),
                                     scale=rng.uniform(0.02, 0.4)) for _ in range(n)])
  scenes.append([])
  rows = _rows_of_sprites(scenes, 6)
  got = scene_program.sample_contained_on_host(rows, 9, 6)
  _assert_same(got, restate(rows, 9, 6), 'mixed')
  _check_inside(scenes, 6, got)
  assert ((got[0][..., 0] < 0) | (got[0][..., 0] > 1)).any()   # positions beyond the frame are kept
  empty = np.array([len(sc) == 0 for sc in scenes])
  assert (got[2][empty] == _native.ENV_NO_SPRITE).all() and (got[2][~empty] == 0).all()
  assert np.isnan(got[0][empty]).all() and (got[1][empty] == -1).all()


def test_shape_ids_without_a_vertex_table_are_empty_slots():
  rows = _rows_of_sprites([[sprite_lib.Sprite(shape='circle'), sprite_lib.Sprite(shape='square', x=0.2)]], 4)
  rows['shape'][0, 0] = 13
  rows['shape'][0, 1] = 255
  got = scene_program.sample_contained_on_host(rows, 3, 50)
  _assert_same(got, restate(rows, 3, 50), 'sanitised')
  assert set(got[1].ravel().tolist()) == {2, 3}
  rows['shape'][0, 2:] = 0
  got = scene_program.sample_contained_on_host(rows, 3, 2)
  assert (got[2] == _native.ENV_NO_SPRITE).all() and np.isnan(got[0]).all() and (got[1] == -1).all()


def test_a_scale_0_sprite_runs_out_of_tries():
  rows = _rows_of_sprites([[sprite_lib.Sprite(shape='square', scale=0.0)],
                           [sprite_lib.Sprite(shape='square', scale=0.1)]], 1)
  pos, slot, status = scene_program.sample_contained_on_host(rows, 1, 2)
  assert (status[0] == _native.ENV_SAMPLE_TRIES).all() and np.isnan(pos[0]).all() and (slot[0] == -1).all()
  assert (status[1] == 0).all()
  # the restatement agrees at a smaller try count: the host build stops only after 10^6
  assert (restate(rows, 1, 2, max_tries=1000)[2][0] == _native.ENV_SAMPLE_TRIES).all()


def test_sample_0_and_rows_do_not_depend_on_the_sample_count():
  scenes = _shape_scenes([0, 45], False)
  rows = _rows_of_sprites(scenes, 1)
  a = scene_program.sample_contained_on_host(rows, 11, 1)
  b = scene_program.sample_contained_on_host(rows, 11, 9)
  for x, y in zip(a, b):
    assert np.array_equal(x[:, 0], y[:, 0])
  c = scene_program.sample_contained_on_host(rows, 12, 1)
  assert not np.array_equal(a[0], c[0])


def test_slots_are_chosen_uniformly():
  # five sprites of very different sizes: the choice is per sprite, not per area
  scales = (0.02, 0.3, 0.1, 0.05, 0.2)
  sc = [sprite_lib.Sprite(x=0.1 * k + 0.2, shape=constants.SHAPE_NAMES[k], scale=v) for k, v in enumerate(scales)]
  rows = _rows_of_sprites([sc], 8)
  _, slot, status = scene_program.sample_contained_on_host(rows, 21, 50000)
  assert (status == 0).all()
  counts = np.bincount(slot.ravel(), minlength=8)
  assert (counts[:3] == 0).all()
  assert stats.chisquare(counts[3:]).pvalue > 1e-3, counts


def _half_area(poly, axis, cut):
  """Exact area of the polygon's part with coordinate `axis` below `cut` (half-plane clip)."""
  out = []
  n = len(poly)
  for q in range(n):
    a, b = poly[q], poly[(q + 1) % n]
    ina, inb = a[axis] < cut, b[axis] < cut
    if ina:
      out.append(a)
    if ina != inb:
      t = (cut - a[axis]) / (b[axis] - a[axis])
      out.append(a + t * (b - a))
  return _area(np.array(out)) if len(out) >= 3 else 0.0


def _area(p):
  x, y = p[:, 0], p[:, 1]
  return 0.5 * abs(np.dot(x, np.roll(y, -1)) - np.dot(y, np.roll(x, -1)))


@pytest.mark.parametrize('angle', [0, 37.5])
def test_points_are_uniform_over_each_shape(angle):
  N = 200000
  for name in constants.SHAPE_NAMES:
    sp = sprite_lib.Sprite(x=0.5, y=0.5, shape=name, angle=angle, scale=0.2)
    rows = _rows_of_sprites([[sp]], 1)
    pos, _, status = scene_program.sample_contained_on_host(rows, 31, N)
    assert (status == 0).all()
    c = sp.centred_vertices
    lo, hi = c.min(0), c.max(0)
    total = _area(c)
    for axis in (0, 1):
      mid = 0.5 * (lo[axis] + hi[axis])
      p = _half_area(c, axis, mid) / total
      share = float(np.mean(pos[0, :, axis] - 0.5 < mid))
      sigma = np.sqrt(p * (1 - p) / N)
      assert abs(share - p) < 4 * sigma, (name, angle, axis, share, p)
