"""CPU tier of the soft sprite masks (renderers.SoftSpriteMasks).

1. The restatement tests/soft_mask_oracle.py uses (the oracle's Pillow polygon fill of the label
   canvas, counted per aa x aa block) equals the definition written with Pillow itself, count for
   count: all twelve shapes, random angles, scales and positions partly and wholly off the canvas,
   stars and spokes across y = 0, sprites with edges beyond +-32768 canvas rows, anti_aliasing 1 to
   15, odd and 1-pixel sizes, empty slots and 32 slots.
2. The properties SoftSpriteMasks states, against tests/mask_oracle.py's masks and
   tests/coverage_oracle.py's coverage: at aa 1 the soft mask is the mask's indicator; the mask's
   sample is one of the aa**2; counts sum to at most aa**2; empty, out-of-frame and hidden sprites
   are zero; soft[k].sum() is slot k's visible canvas area.
3. The host layer -- Engine.render_soft_masks' checks, SoftSpriteMasks in a BatchedEnvironment
   (step, observe, render, specs), the drop-in Environment and the gym wrappers -- on the
   oracle-backed engine double with swb_render_soft_masks (tests/mask_oracle.install).  The kernel
   is tests/test_gpu_soft_masks.py's.
"""
import collections

import numpy as np
import pytest
import torch

from oracle import oracle
from spriteworld_b200 import engine as engine_lib
from tests import coverage_oracle, mask_oracle, soft_mask_oracle
from tests import test_oracle_masks as om
from tests import test_render_states_on_oracle as rs

TAB = om.TAB
ODD_SIZES = [(15, 15), (23, 9), (7, 19), (1, 1), (1, 5), (11, 1)]


def _check(rec, W, H, aa, sprites=None, what=()):
  """The restatement of records `rec` against the Pillow definition (given the Sprite objects), the
  mask and the coverage restatements; returns the soft masks."""
  rc = oracle.raster_cfg(W, H, aa)
  soft = soft_mask_oracle.render_soft_masks(rc, TAB, rec)
  assert soft.shape == (len(rec), H, W) and soft.dtype == np.uint8, what
  if sprites is not None:
    want = soft_mask_oracle.pillow_soft_masks(sprites, W, H, aa)
    assert np.array_equal(soft, want), (what, np.argwhere(soft != want)[:4].tolist())
  mask = mask_oracle.render_masks(rc, TAB, rec)
  soft_mask_oracle.check_properties(soft, mask, aa, what)
  # a slot covers no sample of a pixel whose sample its coverage bit misses only if it is hidden or
  # absent there; where it is the top-most at the sample it owns that sample
  _, visible, area = coverage_oracle.render_coverage(rc, TAB, rec)
  for k in range(len(rec)):
    if area[k] == 0 and aa == 1:
      assert not soft[k].any(), (what, k)
    assert int((soft[k] > 0).sum()) >= int(visible[k]), (what, k)
  return soft


def _every_shape(rng):
  sprites, recs = [], []
  for name in rng.permutation(om.SHAPES):
    s, r = om._sprites(rng, 1, shapes=(name,))
    sprites += s
    recs.append(r)
  return sprites, np.concatenate(recs)


@pytest.mark.parametrize('aa', list(range(1, 16)))
def test_oracle_soft_masks_equal_the_pillow_definition(aa):
  rng = np.random.RandomState(300 + aa)
  for W, H in ODD_SIZES:
    for n in (1, 5, 32):
      sprites, rec = om._sprites(rng, n)
      _check(rec, W, H, aa, sprites, (aa, W, H, n))
    sprites, rec = _every_shape(rng)
    _check(rec, W, H, aa, sprites, (aa, W, H, 'shapes'))


def test_stars_and_spokes_across_y0_equal_the_pillow_definition():
  rng = np.random.RandomState(31)
  for aa in (1, 2, 5, 13, 15):
    for W, H in ((15, 15), (9, 5)):
      sprites, rec = om._sprites(rng, 12, y_range=(-0.08, 0.08), shapes=om.STARS)
      _check(rec, W, H, aa, sprites, (aa, W, H))


def test_sprites_with_edges_beyond_int16_rows_equal_the_pillow_definition():
  from spriteworld_b200 import sprite
  from tests import fixtures
  rng = np.random.RandomState(37)
  names = {v: k for k, v in oracle.SHAPE_IDS.items()}
  n_crossing = 0
  for W, H, aa in ((15, 15, 15), (23, 9, 13), (7, 29, 5)):
    a = mask_oracle.huge_scene_arrays(rng, 6, 3, aa * H)
    for e in range(6):
      sprites = [sprite.Sprite(x=a['x'][e, s], y=a['y'][e, s], shape=names[int(a['shape'][e, s])],
                               angle=a['angle'][e, s], scale=a['scale'][e, s]) for s in range(3)]
      rec = fixtures.records_from_arrays({k: v[e] for k, v in a.items()})
      assert max(abs(mask_oracle.canvas_vertices(oracle.raster_cfg(W, H, aa), TAB, r)[:, 1]).max()
                 for r in rec) > 40000
      soft = _check(rec, W, H, aa, sprites, (W, H, aa, e))
      total = soft.astype(np.int64).sum(0)
      n_crossing += int(((total > 0) & (total < aa * aa)).any())   # an outline inside a pixel
  assert n_crossing >= 6


def _records(sprites):
  from tests import fixtures
  n = len(sprites)
  z = np.zeros(n)
  return fixtures.records_from_arrays(dict(
      x=np.array([s.x for s in sprites]), y=np.array([s.y for s in sprites]),
      shape=np.array([oracle.SHAPE_IDS[s.shape] for s in sprites]), angle=np.array([s.angle for s in sprites]),
      scale=np.array([s.scale for s in sprites]), vx=z, vy=z, member=np.zeros(n, np.uint32),
      pos_f32=np.zeros(n, np.uint8), rgb=np.zeros((n, 3), np.uint8)))


def test_empty_out_of_frame_and_hidden_sprites_are_zero():
  from spriteworld_b200 import sprite
  rng = np.random.RandomState(5)
  sprites, _ = om._sprites(rng, 6)
  sprites[3] = sprite.Sprite(x=5.0, y=-4.0, shape='square', scale=0.1)      # wholly out of frame
  sprites[2] = sprite.Sprite(x=0.5, y=0.5, shape='circle', scale=0.05)      # wholly hidden by 5
  sprites[5] = sprite.Sprite(x=0.5, y=0.5, shape='square', scale=0.5)
  rec = _records(sprites)
  rec[0]['shape'] = 0                                                       # an empty slot
  for aa in (1, 4, 15):
    soft = _check(rec, 13, 9, aa, what=('zero', aa))
    for k in (0, 2, 3):
      assert not soft[k].any(), (aa, k)
    assert soft[5].any()


def test_visible_area_is_the_sum_of_the_counts():
  """soft[k].sum() is slot k's visible canvas area: the label canvas's count of k + 1."""
  rng = np.random.RandomState(41)
  for aa in (1, 3, 5, 15):
    sprites, rec = om._sprites(rng, 9)
    soft = soft_mask_oracle.pillow_soft_masks(sprites, 17, 11, aa)
    from PIL import Image, ImageDraw
    canvas = Image.new('L', (17 * aa, 11 * aa), 0)
    draw = ImageDraw.Draw(canvas)
    for k, s in enumerate(sprites):
      draw.polygon([tuple(v) for v in canvas.size * s.vertices], fill=k + 1)
    area = np.bincount(np.asarray(canvas).reshape(-1), minlength=10)[1:10]
    assert np.array_equal(soft.astype(np.int64).sum((1, 2)), area), aa


def test_32_nested_slots_and_mixed_pixels():
  """32 sprites over one centre, each smaller than the one below: every ring is visible, and the
  pixels on the outlines mix several slots."""
  from spriteworld_b200 import sprite
  rng = np.random.RandomState(3)
  sprites, _ = om._sprites(rng, 32)
  sprites = [sprite.Sprite(x=0.5, y=0.5, shape=s.shape, angle=s.angle, scale=0.6 - 0.015 * k)
             for k, s in enumerate(sprites)]
  soft = _check(_records(sprites), 31, 31, 5, sprites, 'nested')
  assert soft[31].any()
  assert ((soft > 0).sum(0) >= 3).any()


# ---------------------------------------------------------------------------------------------
# host layer on the engine double
# ---------------------------------------------------------------------------------------------

@pytest.fixture
def double(monkeypatch):
  mask_oracle.install(monkeypatch)


def _renderers(**soft):
  from spriteworld_b200 import renderers
  hsv = renderers.color_maps.hsv_to_rgb
  out = collections.OrderedDict(image=renderers.PILRenderer(image_size=(16, 12), color_to_rgb=hsv))
  out['masks'] = renderers.SpriteMasks(image_size=(16, 12), anti_aliasing=3)
  for name, (size, aa) in soft.items():
    out[name] = renderers.SoftSpriteMasks(image_size=size, anti_aliasing=aa)
  out['factors'] = renderers.SpriteFactors()
  return out


def _oracle_soft(env, renderer):
  rc = oracle.raster_cfg(renderer.width, renderer.height, renderer.anti_aliasing)
  bo = env.engine._bo
  return np.stack([soft_mask_oracle.render_soft_masks(rc, env.engine._tab, bo.cur[e]) for e in range(env.n_envs)])


def test_soft_sprite_masks_in_a_batched_environment(double):
  env = rs._env(_renderers(soft=((16, 12), 3), fine=((9, 14), 2)), E=6)
  S = env.engine.n_slots
  spec = env.observation_spec()
  assert spec['soft'].shape == (S, 12, 16) and spec['soft'].dtype == np.uint8
  assert spec['soft'].minimum == 0 and spec['soft'].maximum == 9 and spec['fine'].maximum == 4
  assert spec['fine'].shape == (S, 14, 9)
  rng = np.random.RandomState(2)
  ts = env.reset()
  buffers = {k: ts.observation[k].data_ptr() for k in ('soft', 'fine')}
  for t in range(12):
    if t:
      ts = env.step(rng.uniform(0, 1, (env.n_envs, 4)).astype(np.float32))
    assert list(ts.observation) == ['image', 'masks', 'soft', 'fine', 'factors']
    for name in ('soft', 'fine'):
      obs = ts.observation[name]
      assert obs.data_ptr() == buffers[name] and obs.dtype == torch.uint8, (t, name)
      assert np.array_equal(obs.numpy(), _oracle_soft(env, env._renderers[name])), (t, name)
    m = ts.observation['masks'].numpy()
    for e in range(env.n_envs):
      soft_mask_oracle.check_properties(ts.observation['soft'][e].numpy(), m[e], 3, (t, e))
    occupied = ts.observation['factors']['mask'].numpy()
    assert not ts.observation['soft'].numpy()[~occupied].any(), t   # slots are the factors' slots
  env.close()


def test_observe_and_render_give_the_soft_masks_of_records(double):
  env = rs._env(_renderers(soft=((16, 12), 2)), E=6)
  rs._started(env, steps=4, seed=5)
  states = env.save_envs()[[4, 4, 1, 0, 5, 3, 2]]
  launches = env.engine.launch_count()
  obs, _ = env.observe(states)
  assert list(obs) == ['image', 'masks', 'soft', 'factors']
  assert env.engine.launch_count() == launches + 3
  soft = obs['soft']
  assert tuple(soft.shape) == (7, env.engine.n_slots, 12, 16) and soft.dtype == torch.uint8
  own = env._soft_buffers[id(env._renderers['soft'])]
  assert soft.data_ptr() != own.data_ptr()
  assert torch.equal(env._renderers['soft'].render_states(env, states), soft)
  env.load_envs(states[:6])
  out = env.render()
  assert list(out) == ['image', 'masks', 'soft']
  assert out['soft'].data_ptr() == own.data_ptr()
  assert torch.equal(out['soft'], soft[:6])
  assert np.array_equal(out['soft'].numpy(), _oracle_soft(env, env._renderers['soft']))
  env.close()


def test_render_soft_masks_checks_its_arguments(double):
  env = rs._env(_renderers(soft=((16, 12), 1)), E=6)
  rs._started(env)
  eng = env.engine
  states = env.save_envs()
  launches = eng.launch_count()
  n, S = eng.n_envs, eng.n_slots
  with pytest.raises(ValueError, match='EnvStates'):
    eng.render_soft_masks(16, 12, 1, states=states.data)
  other = engine_lib.EnvStates(states.data, 1, b'x' * len(states.signature), states.n_slots)
  with pytest.raises(ValueError, match='another configuration'):
    eng.render_soft_masks(16, 12, 1, states=other)
  for bad in (torch.zeros((n, S, 12, 16), dtype=torch.int32), torch.zeros((n, 12, 16), dtype=torch.uint8),
              torch.zeros((n, S, 16, 12), dtype=torch.uint8), torch.zeros((n - 1, S, 12, 16), dtype=torch.uint8),
              np.zeros((n, S, 12, 16), np.uint8),
              torch.zeros((n, S, 16, 12), dtype=torch.uint8).transpose(2, 3)):
    with pytest.raises(ValueError, match='soft'):
      eng.render_soft_masks(16, 12, 1, out=bad)
  assert eng.launch_count() == launches
  out = torch.zeros((n, S, 12, 16), dtype=torch.uint8)
  assert eng.render_soft_masks(16, 12, 1, out=out) is out and eng.launch_count() == launches + 1
  empty = eng.render_soft_masks(16, 12, 1, states=states[:0])
  assert tuple(empty.shape) == (0, S, 12, 16) and eng.launch_count() == launches + 1
  env.close()


def test_soft_sprite_masks_arguments_and_specs():
  from spriteworld_b200 import renderers
  r = renderers.SoftSpriteMasks(image_size=(10, 4), anti_aliasing=15)
  spec = r.observation_spec()
  assert spec.shape == (0, 4, 10) and spec.dtype == np.uint8 and spec.minimum == 0 and spec.maximum == 225
  assert r.width == 10 and r.height == 4 and r.anti_aliasing == 15
  assert renderers.SoftSpriteMasks(image_size=(273, 273), anti_aliasing=15).width == 273
  with pytest.raises(ValueError, match='exceeds 15'):
    renderers.SoftSpriteMasks(image_size=(10, 4), anti_aliasing=16)
  for size, aa in (((0, 4), 1), ((4, 4), 0), ((4096, 1), 1), ((274, 1), 15), ((1, 274), 15), ((4,), 1),
                   ((4, 4), 20)):
    with pytest.raises(ValueError):
      renderers.SoftSpriteMasks(image_size=size, anti_aliasing=aa)


def test_soft_sprite_masks_render_a_sprite_list(double):
  from spriteworld_b200 import renderers
  rng = np.random.RandomState(21)
  for n, size, aa in ((0, (6, 5), 2), (1, (16, 12), 1), (7, (9, 14), 3), (32, (5, 5), 15)):
    sprites, _ = om._sprites(rng, n) if n else ([], None)
    r = renderers.SoftSpriteMasks(image_size=size, anti_aliasing=aa)
    got = r.render(sprites)
    want = soft_mask_oracle.pillow_soft_masks(sprites, size[0], size[1], aa)
    assert got.dtype == np.uint8 and got.shape == (n, size[1], size[0]), (n, size, aa)
    assert np.array_equal(got, want), (n, size, aa)
    assert r.observation_spec().shape == (n, size[1], size[0])


def test_gym_wrapper_of_the_drop_in_environment_describes_and_returns_the_soft_masks(double):
  from spriteworld_b200 import environment, gym_wrapper, renderers
  from spriteworld_b200.configs.cobra import goal_finding_more_targets as cfgmod
  cfg = cfgmod.get_config('train')
  cfg['renderers'] = collections.OrderedDict([
      ('soft', renderers.SoftSpriteMasks(image_size=(16, 12), anti_aliasing=5)),
      ('masks', renderers.SpriteMasks(image_size=(16, 12), anti_aliasing=5))])
  np.random.seed(9)
  env = environment.Environment(**cfg)
  wrapped = gym_wrapper.GymWrapper(env)
  n = len(wrapped.state()['sprites'])
  assert env.observation_spec()['soft'].shape == (n, 12, 16)
  space = wrapped.observation_space.spaces['soft']
  assert space.shape == (n, 12, 16) and space.dtype == np.uint8
  for t in range(4):
    obs, _, _, _ = wrapped.step(np.array([0.3, 0.4, 0.6, 0.7]))
    sprites = wrapped.state()['sprites']
    assert obs['soft'].shape == (n, 12, 16) and obs['soft'].dtype == np.uint8, t
    assert np.array_equal(obs['soft'], soft_mask_oracle.pillow_soft_masks(sprites, 16, 12, 5)), t
    soft_mask_oracle.check_properties(obs['soft'], obs['masks'], 5, t)
  wrapped.close()


def test_vector_gym_wrapper_describes_and_returns_the_soft_masks(double):
  from spriteworld_b200 import gym_wrapper
  env = rs._env(_renderers(soft=((16, 12), 4)), E=4)
  S = env.engine.n_slots
  vec = gym_wrapper.VectorGymWrapper(env)
  space = vec.single_observation_space.spaces['soft']
  assert space.shape == (S, 12, 16) and space.dtype == np.uint8
  assert int(np.min(space.low)) == 0 and int(np.max(space.high)) == 16
  obs = vec.reset()
  assert tuple(obs['soft'].shape) == (4, S, 12, 16)
  obs, _, _, _ = vec.step(np.random.RandomState(0).uniform(0, 1, (4, 4)).astype(np.float32))
  assert np.array_equal(obs['soft'].numpy(), _oracle_soft(env, env._renderers['soft']))
  vec.close()
