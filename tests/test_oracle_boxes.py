"""CPU tier of the sprite bounding boxes (renderers.SpriteBoxes).

1. The restatement tests/box_oracle.py uses (the coverage restatement's planes, each box from its row
   and column extents) equals the definition written with Pillow itself (Pillow's coverage planes,
   boxes as torchvision.ops.masks_to_boxes writes them): all twelve shapes, random angles, scales and
   positions partly and wholly off the canvas, stars and spokes across y = 0, sprites with edges
   beyond +-32768 canvas rows, anti_aliasing up to 20, non-square and 1-pixel sizes, up to 32 slots
   (bit 31 included), hidden, empty and out-of-frame sprites.
2. The stated invariants: the visible box lies in the amodal box, visible <= area, a count is 0
   exactly where its box is, and the counts are the coverage restatement's.
3. The host layer -- Engine.render_boxes' checks, SpriteBoxes in a BatchedEnvironment (step,
   observe, render, specs), the drop-in Environment and the gym wrappers -- on the oracle-backed
   engine double with swb_render_boxes (tests/box_oracle.install).  The kernel is
   tests/test_gpu_boxes.py's.
"""
import collections

import numpy as np
import pytest
import torch

from oracle import oracle
from spriteworld_b200 import engine as engine_lib
from tests import box_oracle, coverage_oracle, mask_oracle
from tests import test_oracle_coverage as oc
from tests import test_oracle_masks as om
from tests import test_render_states_on_oracle as rs

TAB = om.TAB
KEYS = ['visible_box', 'amodal_box', 'visible', 'area']


def _check(rec, W, H, aa, sprites=None, what=()):
  """The restatement of records `rec` against the Pillow definition (given the Sprite objects), the
  coverage restatement and the invariants; returns (visible_box, amodal_box, visible, area)."""
  rc = oracle.raster_cfg(W, H, aa)
  got = box_oracle.render_boxes(rc, TAB, rec)
  n = len(rec)
  assert [g.shape for g in got] == [(n, 4), (n, 4), (n,), (n,)], what
  assert all(g.dtype == np.int32 for g in got), what
  if sprites is not None:
    want = box_oracle.pillow_boxes(sprites, W, H, aa)
    for k, g, w in zip(KEYS, got, want):
      assert np.array_equal(g, w), (what, k, np.argwhere(g != w)[:4].tolist())
  _, visible, area = coverage_oracle.render_coverage(rc, TAB, rec)
  assert np.array_equal(got[2], visible) and np.array_equal(got[3], area), what
  box_oracle.check_invariants(*got, W, H, what)
  return got


@pytest.mark.parametrize('aa', [1, 2, 3, 5, 10, 13, 20])
def test_oracle_boxes_equal_the_pillow_definition(aa):
  rng = np.random.RandomState(300 + aa)
  for W, H in om.SIZES:
    for n in (1, 5, 32):
      sprites, rec = om._sprites(rng, n)
      _check(rec, W, H, aa, sprites, (aa, W, H, n))
    sprites, rec = oc._every_shape(rng)
    _check(rec, W, H, aa, sprites, (aa, W, H, 'shapes'))


def test_box_of_a_plane_is_masks_to_boxes_plus_one():
  plane = np.zeros((7, 9), bool)
  assert box_oracle.box(plane).tolist() == [0, 0, 0, 0]
  plane[2, 3] = plane[5, 1] = True
  assert box_oracle.box(plane).tolist() == [1, 2, 4, 6]
  plane[:] = True
  assert box_oracle.box(plane).tolist() == [0, 0, 9, 7]


def test_slot_31_and_hidden_sprites_keep_their_amodal_boxes():
  """32 sprites over the same centre, each smaller than the one below: the amodal box of each holds
  the boxes of those above it, slot 31 (the sign bit) has its own box, and the visible box of a
  sprite wholly hidden under a larger one is zero."""
  from spriteworld_b200 import sprite
  rng = np.random.RandomState(3)
  sprites, _ = om._sprites(rng, 32)
  sprites = [sprite.Sprite(x=0.5, y=0.5, shape=s.shape, angle=s.angle, scale=0.6 - 0.015 * k)
             for k, s in enumerate(sprites)]
  vb, ab, visible, area = _check(oc._records(sprites), 16, 16, 3, sprites, 'nested')
  assert area[31] > 0 and (ab[31] > 0).any() and visible[31] == area[31]
  assert (area > 0).all() and (visible < area).any()
  # a small square under a big one, and the big one alone: hidden has a zero visible box only
  hidden = [sprite.Sprite(x=0.5, y=0.5, shape='square', scale=0.1),
            sprite.Sprite(x=0.5, y=0.5, shape='square', scale=0.5)]
  vb, ab, visible, area = _check(oc._records(hidden), 20, 20, 2, hidden, 'hidden')
  assert visible[0] == 0 and (vb[0] == 0).all() and area[0] > 0 and (ab[0] > 0).all()
  assert (ab[0, :2] >= ab[1, :2]).all() and (ab[0, 2:] <= ab[1, 2:]).all()


def test_empty_and_out_of_frame_sprites_have_zero_boxes():
  from spriteworld_b200 import sprite
  rng = np.random.RandomState(5)
  sprites, _ = om._sprites(rng, 6)
  sprites[3] = sprite.Sprite(x=5.0, y=-4.0, shape='square', scale=0.1)   # wholly out of frame
  rec = oc._records(sprites)
  rec[0]['shape'] = 0                             # an empty slot, padded at the front
  vb, ab, visible, area = _check(rec, 12, 9, 2, what='empty')
  for k in (0, 3):
    assert (vb[k] == 0).all() and (ab[k] == 0).all() and visible[k] == 0 and area[k] == 0


def test_stars_and_spokes_across_y0_equal_the_pillow_definition():
  rng = np.random.RandomState(19)
  for aa in (1, 2, 5, 13):
    for W, H in ((16, 16), (9, 4)):
      sprites, rec = om._sprites(rng, 12, y_range=(-0.08, 0.08), shapes=om.STARS)
      _check(rec, W, H, aa, sprites, (aa, W, H))


def test_sprites_with_edges_beyond_int16_rows_equal_the_pillow_definition():
  from spriteworld_b200 import sprite
  from tests import fixtures
  rng = np.random.RandomState(29)
  names = {v: k for k, v in oracle.SHAPE_IDS.items()}
  n_crossing = 0
  for W, H, aa in ((16, 16, 20), (24, 9, 13), (7, 30, 5)):
    a = mask_oracle.huge_scene_arrays(rng, 6, 3, aa * H)
    for e in range(6):
      sprites = [sprite.Sprite(x=a['x'][e, s], y=a['y'][e, s], shape=names[int(a['shape'][e, s])],
                               angle=a['angle'][e, s], scale=a['scale'][e, s]) for s in range(3)]
      rec = fixtures.records_from_arrays({k: v[e] for k, v in a.items()})
      assert max(abs(mask_oracle.canvas_vertices(oracle.raster_cfg(W, H, aa), TAB, r)[:, 1]).max()
                 for r in rec) > 40000
      _, ab, _, area = _check(rec, W, H, aa, sprites, (W, H, aa, e))
      crossing = (0 < area) & (area < W * H)
      n_crossing += int(crossing.any())
  assert n_crossing >= 6   # outlines do cross the canvases


# ---------------------------------------------------------------------------------------------
# host layer on the engine double
# ---------------------------------------------------------------------------------------------

@pytest.fixture
def double(monkeypatch):
  box_oracle.install(monkeypatch)


def _renderers(**boxes):
  from spriteworld_b200 import renderers
  hsv = renderers.color_maps.hsv_to_rgb
  out = collections.OrderedDict(image=renderers.PILRenderer(image_size=(16, 12), color_to_rgb=hsv))
  out['masks'] = renderers.SpriteMasks(image_size=(16, 12), anti_aliasing=1)
  for name, (size, aa) in boxes.items():
    out[name] = renderers.SpriteBoxes(image_size=size, anti_aliasing=aa)
  out['factors'] = renderers.SpriteFactors()
  return out


def _oracle_boxes(env, renderer):
  """Boxes of the double's live envs by the restatement."""
  rc = oracle.raster_cfg(renderer.width, renderer.height, renderer.anti_aliasing)
  bo = env.engine._bo
  got = [box_oracle.render_boxes(rc, env.engine._tab, bo.cur[e]) for e in range(env.n_envs)]
  return tuple(np.stack(x) for x in zip(*got))


def _assert_equal(obs, want, what):
  assert list(obs) == KEYS, what
  for k, w in zip(obs, want):
    assert obs[k].dtype == torch.int32, (what, k)
    assert np.array_equal(obs[k].numpy(), w), (what, k)


def test_sprite_boxes_in_a_batched_environment(double):
  env = rs._env(_renderers(boxes=((16, 12), 1), fine=((9, 14), 3)), E=6)
  S = env.engine.n_slots
  spec = env.observation_spec()
  assert list(spec['boxes']) == KEYS
  assert spec['boxes']['visible_box'].shape == spec['boxes']['amodal_box'].shape == (S, 4)
  assert spec['fine']['amodal_box'].maximum[0].tolist() == [9, 14, 9, 14]
  assert spec['boxes']['visible'].shape == spec['boxes']['area'].shape == (S,)
  rng = np.random.RandomState(2)
  ts = env.reset()
  buffers = {k: [t.data_ptr() for t in ts.observation[k].values()] for k in ('boxes', 'fine')}
  for t in range(12):
    if t:
      ts = env.step(rng.uniform(0, 1, (env.n_envs, 4)).astype(np.float32))
    assert list(ts.observation) == ['image', 'masks', 'boxes', 'fine', 'factors']
    for name in ('boxes', 'fine'):
      obs = ts.observation[name]
      assert [v.data_ptr() for v in obs.values()] == buffers[name]   # the env's buffers, every step
      _assert_equal(obs, _oracle_boxes(env, env._renderers[name]), (t, name))
      for k, v in spec[name].items():
        for e in range(env.n_envs):
          v.validate(obs[k][e].numpy())
    # the visible boxes and counts of the same step are those of its mask
    m = ts.observation['masks'].numpy()
    b = ts.observation['boxes']
    for e in range(env.n_envs):
      for k in range(S):
        assert np.array_equal(b['visible_box'][e, k].numpy(), box_oracle.box(m[e] == k + 1)), (t, e, k)
    occupied = ts.observation['factors']['mask'].numpy()
    assert (b['area'].numpy()[~occupied] == 0).all(), t     # slots index the factors' slot axis
    assert (b['amodal_box'].numpy()[~occupied] == 0).all(), t
  env.close()


def test_observe_and_render_give_the_boxes_of_records(double):
  env = rs._env(_renderers(boxes=((16, 12), 2)), E=6)
  rs._started(env, steps=4, seed=5)
  states = env.save_envs()[[4, 4, 1, 0, 5, 3, 2]]
  launches = env.engine.launch_count()
  obs, _ = env.observe(states)
  assert list(obs) == ['image', 'masks', 'boxes', 'factors']
  assert env.engine.launch_count() == launches + 4    # frames, masks, and two for the boxes
  c = obs['boxes']
  S = env.engine.n_slots
  assert [tuple(v.shape) for v in c.values()] == [(7, S, 4), (7, S, 4), (7, S), (7, S)]
  own = env._mask_buffers[id(env._renderers['boxes'])]
  assert all(v.data_ptr() != b.data_ptr() for v, b in zip(c.values(), own))
  by_renderer = env._renderers['boxes'].render_states(env, states)
  for k in c:
    assert torch.equal(by_renderer[k], c[k]), k
  by_env = env.render_boxes(env._renderers['boxes'], states)
  for k in c:
    assert torch.equal(by_env[k], c[k]), k
  env.load_envs(states[:6])
  out = env.render()
  assert list(out) == ['image', 'masks', 'boxes']
  assert [v.data_ptr() for v in out['boxes'].values()] == [b.data_ptr() for b in own]
  for k in c:
    assert torch.equal(out['boxes'][k], c[k][:6]), k
  live = env.render_boxes(env._renderers['boxes'])
  assert [v.data_ptr() for v in live.values()] == [b.data_ptr() for b in own]
  # and the coverage of the same records, summarised, is the boxes
  from spriteworld_b200 import renderers
  cover = env.render_coverage(renderers.SpriteCoverage(image_size=(16, 12), anti_aliasing=2), states)
  for e in range(len(states)):
    want = box_oracle.boxes_of_cover(cover['cover'][e].numpy(), S)
    for k, w in zip(KEYS, want):
      assert np.array_equal(c[k][e].numpy(), w), (e, k)
  env.close()


def test_render_boxes_checks_its_arguments(double):
  env = rs._env(_renderers(boxes=((16, 12), 1)), E=6)
  rs._started(env)
  eng = env.engine
  states = env.save_envs()
  launches = eng.launch_count()
  n, S = eng.n_envs, eng.n_slots
  with pytest.raises(ValueError, match='EnvStates'):
    eng.render_boxes(16, 12, 1, states=states.data)
  other = engine_lib.EnvStates(states.data, 1, b'x' * len(states.signature), states.n_slots)
  with pytest.raises(ValueError, match='another configuration'):
    eng.render_boxes(16, 12, 1, states=other)

  def good():
    return [torch.zeros((n, S, 4), dtype=torch.int32), torch.zeros((n, S, 4), dtype=torch.int32),
            torch.zeros((n, S), dtype=torch.int32), torch.zeros((n, S), dtype=torch.int32)]
  with pytest.raises(ValueError, match='4-tuple'):
    eng.render_boxes(16, 12, 1, out=good()[0])
  with pytest.raises(ValueError, match='4-tuple'):
    eng.render_boxes(16, 12, 1, out=good()[:3])
  for i, name in enumerate(KEYS):
    shape = good()[i].shape
    wrong = [torch.zeros(shape, dtype=torch.uint8), torch.zeros(shape[::-1], dtype=torch.int32),
             torch.zeros((n - 1,) + tuple(shape[1:]), dtype=torch.int32), np.zeros(shape, np.int32),
             torch.zeros(shape[::-1], dtype=torch.int32).t() if len(shape) == 2 else
             torch.zeros((n, 4, S), dtype=torch.int32).transpose(1, 2)]
    for bad in wrong:
      out = good()
      out[i] = bad
      with pytest.raises(ValueError, match=name):
        eng.render_boxes(16, 12, 1, out=out)
  assert eng.launch_count() == launches
  out = good()
  got = eng.render_boxes(16, 12, 1, out=out)
  assert all(g is o for g, o in zip(got, out)) and eng.launch_count() == launches + 2
  empty = eng.render_boxes(16, 12, 1, states=states[:0])
  assert [tuple(t.shape) for t in empty] == [(0, S, 4), (0, S, 4), (0, S), (0, S)]
  assert eng.launch_count() == launches + 2
  env.close()


def test_sprite_boxes_arguments_and_specs():
  from spriteworld_b200 import gym_wrapper, renderers
  r = renderers.SpriteBoxes(image_size=(10, 4), anti_aliasing=409)
  spec = r.observation_spec()
  assert list(spec) == KEYS
  assert spec['visible_box'].shape == spec['amodal_box'].shape == (0, 4)
  assert spec['visible'].shape == (0,) and spec['area'].dtype == np.int32
  spec = r._spec(3)
  for k in ('visible_box', 'amodal_box'):
    assert spec[k].dtype == np.int32 and spec[k].shape == (3, 4)
    assert (np.asarray(spec[k].minimum) == 0).all()
    assert np.broadcast_to(spec[k].maximum, (3, 4)).tolist() == [[10, 4, 10, 4]] * 3
    spec[k].validate(np.array([[0, 0, 10, 4]] * 3, np.int32))
    with pytest.raises(ValueError):
      spec[k].validate(np.array([[0, 0, 10, 5]] * 3, np.int32))
    # the per-column bounds survive the conversion to a gym space
    space = gym_wrapper._spec_to_space(spec[k])
    assert space.shape == (3, 4) and space.dtype == np.int32
    assert np.asarray(space.low).tolist() == [[0] * 4] * 3
    assert np.asarray(space.high).tolist() == [[10, 4, 10, 4]] * 3
    assert space.contains(np.array([[1, 2, 10, 4]] * 3, np.int32))
    assert not space.contains(np.array([[1, 2, 5, 5]] * 3, np.int32))
  assert spec['visible'].maximum == spec['area'].maximum == 40
  for size, aa in (((0, 4), 1), ((4, 4), 0), ((4096, 1), 1), ((10, 4), 410), ((4,), 1)):
    with pytest.raises(ValueError):
      renderers.SpriteBoxes(image_size=size, anti_aliasing=aa)


def test_sprite_boxes_render_a_sprite_list(double):
  from spriteworld_b200 import renderers
  rng = np.random.RandomState(21)
  for n, size, aa in ((0, (6, 5), 2), (1, (16, 12), 1), (7, (9, 14), 3), (32, (5, 5), 20)):
    sprites, _ = om._sprites(rng, n) if n else ([], None)
    r = renderers.SpriteBoxes(image_size=size, anti_aliasing=aa)
    got = r.render(sprites)
    want = box_oracle.pillow_boxes(sprites, size[0], size[1], aa)
    assert list(got) == KEYS
    for k, w in zip(KEYS, want):
      assert got[k].dtype == np.int32 and np.array_equal(got[k], w.reshape(got[k].shape)), (n, size, aa, k)
    assert r.observation_spec()['visible_box'].shape == (n, 4)


def test_gym_wrapper_of_the_drop_in_environment_describes_and_returns_the_boxes(double):
  from spriteworld_b200 import environment, gym_wrapper, renderers
  from spriteworld_b200.configs.cobra import goal_finding_more_targets as cfgmod
  cfg = cfgmod.get_config('train')
  cfg['renderers'] = collections.OrderedDict([
      ('boxes', renderers.SpriteBoxes(image_size=(16, 12), anti_aliasing=3)),
      ('masks', renderers.SpriteMasks(image_size=(16, 12), anti_aliasing=3))])
  np.random.seed(9)
  wrapped = gym_wrapper.GymWrapper(environment.Environment(**cfg))
  space = wrapped.observation_space.spaces['boxes']
  n = len(wrapped.state()['sprites'])
  assert space.spaces['visible_box'].shape == (n, 4) and space.spaces['amodal_box'].dtype == np.int32
  assert np.asarray(space.spaces['amodal_box'].high)[0].tolist() == [16, 12, 16, 12]
  assert space.spaces['visible'].shape == (n,) and int(np.max(space.spaces['area'].high)) == 12 * 16
  for t in range(4):
    obs, _, _, _ = wrapped.step(np.array([0.3, 0.4, 0.6, 0.7]))
    sprites = wrapped.state()['sprites']
    b = obs['boxes']
    assert isinstance(b, dict) and list(b) == KEYS, t
    want = box_oracle.pillow_boxes(sprites, 16, 12, 3)
    for k, w in zip(KEYS, want):
      assert b[k].dtype == np.int32 and np.array_equal(b[k], w), (t, k)
      assert space.spaces[k].contains(b[k]), (t, k)
    for k in range(n):
      assert np.array_equal(b['visible_box'][k], box_oracle.box(obs['masks'] == k + 1)), (t, k)
  wrapped.close()


def test_vector_gym_wrapper_describes_and_returns_the_boxes(double):
  from spriteworld_b200 import gym_wrapper
  env = rs._env(_renderers(boxes=((16, 12), 1)), E=4)
  S = env.engine.n_slots
  vec = gym_wrapper.VectorGymWrapper(env)
  space = vec.single_observation_space.spaces['boxes']
  assert space.spaces['visible_box'].shape == space.spaces['amodal_box'].shape == (S, 4)
  assert np.asarray(space.spaces['visible_box'].high)[0].tolist() == [16, 12, 16, 12]
  assert space.spaces['visible'].shape == space.spaces['area'].shape == (S,)
  obs = vec.reset()
  assert tuple(obs['boxes']['amodal_box'].shape) == (4, S, 4) and tuple(obs['boxes']['area'].shape) == (4, S)
  obs, _, _, _ = vec.step(np.random.RandomState(0).uniform(0, 1, (4, 4)).astype(np.float32))
  _assert_equal(obs['boxes'], _oracle_boxes(env, env._renderers['boxes']), 'vector step')
  for e in range(4):
    for k in KEYS:
      assert space.spaces[k].contains(obs['boxes'][k][e].numpy()), (e, k)
  vec.close()
