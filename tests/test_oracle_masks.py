"""CPU tier of the sprite instance masks (renderers.SpriteMasks).

1. The restatement tests/mask_oracle.py uses (the oracle's Pillow polygon fill on a label canvas,
   sampled at aa*j + aa//2 and flipped) equals the definition written with Pillow itself, bit for
   bit: every shape, random angles, scales and positions partly and wholly off the canvas, stars
   and spokes across y = 0, anti_aliasing up to 20, non-square and 1-pixel sizes, up to 32 slots.
2. At anti_aliasing = 1 the oracle's frames are bg where the mask is 0 and the colour of sprite
   mask - 1 elsewhere.
3. The host layer -- Engine.render_masks' checks, SpriteMasks in a BatchedEnvironment (step,
   observe, render, specs) and in the gym wrappers' spaces -- on the oracle-backed engine double,
   with swb_render_masks, swb_render_coverage and swb_render_soft_masks (tests/mask_oracle.install).
   The kernel is tests/test_gpu_masks.py's.
"""
import collections

import numpy as np
import pytest
import torch

from oracle import oracle
from spriteworld_b200 import constants
from spriteworld_b200 import engine as engine_lib
from tests import fixtures, mask_oracle
from tests import test_render_states_on_oracle as rs

SHAPES = tuple(oracle.SHAPE_IDS)          # the twelve shapes, ids 1 .. 12
STARS = ('star_4', 'star_5', 'star_6', 'spoke_4', 'spoke_5', 'spoke_6')
TAB = oracle.shape_table(constants.SHAPES)


def _sprites(rng, n, y_range=(-0.4, 1.4), shapes=SHAPES):
  """Random Sprite objects and their oracle records: positions on, across and off the canvas,
  sub-pixel to larger-than-canvas scales, random and axis-aligned angles."""
  from spriteworld_b200 import sprite
  out, arrs = [], collections.defaultdict(list)
  for _ in range(n):
    x, y = rng.uniform(-0.4, 1.4), rng.uniform(*y_range)
    v = rng.rand()
    scale = rng.uniform(1e-3, 5e-3) if v < 0.1 else rng.uniform(0.8, 2.0) if v < 0.2 else rng.uniform(0.03, 0.4)
    angle = 45.0 * rng.randint(8) if rng.rand() < 0.3 else float(rng.uniform(0, 360))
    name = shapes[rng.randint(len(shapes))]
    out.append(sprite.Sprite(x=x, y=y, shape=name, angle=angle, scale=scale))
    for k, val in (('x', x), ('y', y), ('shape', oracle.SHAPE_IDS[name]), ('angle', angle), ('scale', scale)):
      arrs[k].append(val)
  a = {k: np.array(v) for k, v in arrs.items()}
  z = np.zeros(n)
  a.update(vx=z, vy=z, member=np.zeros(n, np.uint32), pos_f32=np.zeros(n, np.uint8),
           rgb=rng.randint(0, 256, (n, 3)).astype(np.uint8))
  return out, fixtures.records_from_arrays(a)


SIZES = [(16, 16), (24, 9), (7, 20), (1, 1), (1, 6), (11, 1)]


@pytest.mark.parametrize('aa', [1, 2, 3, 5, 10, 13, 20])
def test_oracle_masks_equal_the_pillow_definition(aa):
  rng = np.random.RandomState(100 + aa)
  for W, H in SIZES:
    for n in (1, 5, 32):
      sprites, rec = _sprites(rng, n)
      want = mask_oracle.pillow_masks(sprites, W, H, aa)
      got = mask_oracle.render_masks(oracle.raster_cfg(W, H, aa), TAB, rec)
      assert got.shape == (H, W) and got.dtype == np.uint8
      assert np.array_equal(got, want), (aa, W, H, n, np.argwhere(got != want)[:4].tolist())


def test_stars_and_spokes_across_y0_equal_the_pillow_definition():
  rng = np.random.RandomState(7)
  for aa in (1, 2, 5, 13):
    for W, H in ((16, 16), (9, 4)):
      sprites, rec = _sprites(rng, 12, y_range=(-0.08, 0.08), shapes=STARS)
      want = mask_oracle.pillow_masks(sprites, W, H, aa)
      got = mask_oracle.render_masks(oracle.raster_cfg(W, H, aa), TAB, rec)
      assert np.array_equal(got, want), (aa, W, H)


def test_sprites_with_edges_beyond_int16_rows_equal_the_pillow_definition():
  """Sprites thousands of canvases large whose outlines cross the canvas: many of their edges lie
  wholly beyond +-32768 canvas rows (the row range the kernel packs into 16 bits)."""
  from spriteworld_b200 import sprite
  rng = np.random.RandomState(13)
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
      want = mask_oracle.pillow_masks(sprites, W, H, aa)
      got = mask_oracle.render_masks(oracle.raster_cfg(W, H, aa), TAB, rec)
      assert np.array_equal(got, want), (W, H, aa, e)
      n_crossing += int(len(np.unique(got)) > 1)
  assert n_crossing >= 6   # outlines do cross the canvases: masks that are not one id throughout


def test_masks_name_the_colours_of_frames_at_anti_aliasing_1():
  rng = np.random.RandomState(11)
  for W, H in ((16, 16), (13, 7), (1, 1)):
    for n in (3, 32):
      _, rec = _sprites(rng, n)
      bg = rng.randint(0, 256, 3).astype(np.uint8)
      frame = oracle.render(oracle.raster_cfg(W, H, 1, bg), TAB, rec)
      mask = mask_oracle.render_masks(oracle.raster_cfg(W, H, 1), TAB, rec)
      colours = np.concatenate([bg[None], rec['rgb']])
      assert np.array_equal(frame, colours[mask]), (W, H, n)


# ---------------------------------------------------------------------------------------------
# host layer on the engine double
# ---------------------------------------------------------------------------------------------

@pytest.fixture(autouse=True)
def _mask_engine(monkeypatch):
  mask_oracle.install(monkeypatch)


def _renderers(**masks):
  from spriteworld_b200 import renderers
  hsv = renderers.color_maps.hsv_to_rgb
  out = collections.OrderedDict(image=renderers.PILRenderer(image_size=(16, 12), color_to_rgb=hsv))
  for name, (size, aa) in masks.items():
    out[name] = renderers.SpriteMasks(image_size=size, anti_aliasing=aa)
  out['factors'] = renderers.SpriteFactors()
  return out


def _oracle_masks(env, renderer):
  """Masks of the double's live envs by the restatement, (n_envs, H, W)."""
  rc = oracle.raster_cfg(renderer.width, renderer.height, renderer.anti_aliasing)
  bo = env.engine._bo
  return np.stack([mask_oracle.render_masks(rc, env.engine._tab, bo.cur[e]) for e in range(env.n_envs)])


def test_sprite_masks_in_a_batched_environment():
  env = rs._env(_renderers(masks=((16, 12), 1), fine=((9, 14), 3)), E=6)
  spec = env.observation_spec()
  assert spec['masks'].shape == (12, 16) and spec['masks'].dtype == np.uint8
  assert spec['fine'].shape == (14, 9)
  rng = np.random.RandomState(2)
  ts = env.reset()
  buffers = {k: ts.observation[k].data_ptr() for k in ('masks', 'fine')}
  for t in range(12):
    if t:
      ts = env.step(rng.uniform(0, 1, (env.n_envs, 4)).astype(np.float32))
    assert list(ts.observation) == ['image', 'masks', 'fine', 'factors']
    for name in ('masks', 'fine'):
      m = ts.observation[name]
      assert m.dtype == torch.uint8 and m.data_ptr() == buffers[name]   # the env's buffer, every step
      assert np.array_equal(m.numpy(), _oracle_masks(env, env._renderers[name])), (t, name)
    # ids index the slot axis of the factors: every visible id is an occupied slot
    occupied = ts.observation['factors']['mask'].numpy()
    m = ts.observation['masks'].numpy()
    for e in range(env.n_envs):
      ids = np.unique(m[e])
      assert occupied[e, ids[ids > 0] - 1].all()
    # at anti_aliasing 1 the frame is bg / rgb[mask - 1]
    frames = ts.observation['image'].numpy()
    rgb = env.engine._bo.cur['rgb']
    for e in range(env.n_envs):
      colours = np.concatenate([np.zeros((1, 3), np.uint8), rgb[e]])
      assert np.array_equal(frames[e], colours[m[e]]), (t, e)
  env.close()


def test_observe_and_render_give_the_masks_of_records():
  env = rs._env(_renderers(masks=((16, 12), 2)), E=6)
  rs._started(env, steps=4, seed=5)
  states = env.save_envs()[[4, 4, 1, 0, 5, 3, 2]]
  launches = env.engine.launch_count()
  obs, _ = env.observe(states)
  assert list(obs) == ['image', 'masks', 'factors']
  assert env.engine.launch_count() == launches + 2
  m = obs['masks']
  assert tuple(m.shape) == (7, 12, 16) and m.dtype == torch.uint8
  assert m.data_ptr() != env._mask_buffers[id(env._renderers['masks'])].data_ptr()
  by_renderer = env._renderers['masks'].render_states(env, states)
  assert torch.equal(by_renderer, m)
  env.load_envs(states[:6])
  out = env.render()
  assert list(out) == ['image', 'masks']
  assert out['masks'].data_ptr() == env._mask_buffers[id(env._renderers['masks'])].data_ptr()
  assert torch.equal(out['masks'], m[:6])
  env.close()


def test_render_masks_checks_its_arguments():
  env = rs._env(_renderers(masks=((16, 12), 1)), E=6)
  rs._started(env)
  eng = env.engine
  states = env.save_envs()
  launches = eng.launch_count()
  with pytest.raises(ValueError, match='EnvStates'):
    eng.render_masks(16, 12, 1, states=states.data)
  other = engine_lib.EnvStates(states.data, 1, b'x' * len(states.signature), states.n_slots)
  with pytest.raises(ValueError, match='another configuration'):
    eng.render_masks(16, 12, 1, states=other)
  n = eng.n_envs
  for bad in (torch.zeros((n, 12, 16), dtype=torch.int32), torch.zeros((n, 16, 12), dtype=torch.uint8),
              torch.zeros((n - 1, 12, 16), dtype=torch.uint8), np.zeros((n, 12, 16), np.uint8),
              torch.zeros((n, 16, 12), dtype=torch.uint8).transpose(1, 2)):
    with pytest.raises(ValueError, match='masks'):
      eng.render_masks(16, 12, 1, out=bad)
  assert eng.launch_count() == launches
  out = torch.zeros((n, 12, 16), dtype=torch.uint8)
  assert eng.render_masks(16, 12, 1, out=out) is out and eng.launch_count() == launches + 1
  empty = eng.render_masks(16, 12, 1, states=states[:0])
  assert tuple(empty.shape) == (0, 12, 16) and eng.launch_count() == launches + 1
  env.close()


def test_sprite_masks_arguments_and_specs():
  from spriteworld_b200 import renderers
  r = renderers.SpriteMasks(image_size=(10, 4), anti_aliasing=409)
  assert r.observation_spec().shape == (4, 10) and r.observation_spec().dtype == np.uint8
  for size, aa in (((0, 4), 1), ((4, 4), 0), ((4096, 1), 1), ((10, 4), 410), ((4,), 1)):
    with pytest.raises(ValueError):
      renderers.SpriteMasks(image_size=size, anti_aliasing=aa)


def test_sprite_masks_render_a_sprite_list():
  from spriteworld_b200 import renderers
  rng = np.random.RandomState(21)
  for n, size, aa in ((1, (16, 12), 1), (7, (9, 14), 3), (32, (5, 5), 20)):
    sprites, _ = _sprites(rng, n)
    got = renderers.SpriteMasks(image_size=size, anti_aliasing=aa).render(sprites)
    assert np.array_equal(got, mask_oracle.pillow_masks(sprites, size[0], size[1], aa)), (n, size, aa)


def test_gym_wrapper_of_the_drop_in_environment_describes_and_returns_the_masks():
  from spriteworld_b200 import environment, gym_wrapper, renderers
  from spriteworld_b200.configs.cobra import goal_finding_more_targets as cfgmod
  cfg = cfgmod.get_config('train')
  cfg['renderers'] = collections.OrderedDict([('masks', renderers.SpriteMasks(image_size=(16, 12),
                                                                              anti_aliasing=3))])
  np.random.seed(9)
  wrapped = gym_wrapper.GymWrapper(environment.Environment(**cfg))
  space = wrapped.observation_space.spaces['masks']
  assert space.shape == (12, 16) and space.dtype == np.uint8
  obs, _, _, _ = wrapped.step(np.array([0.3, 0.4, 0.6, 0.7]))
  sprites = wrapped.state()['sprites']
  assert obs['masks'].shape == (12, 16) and obs['masks'].dtype == np.uint8
  assert np.array_equal(obs['masks'], mask_oracle.pillow_masks(sprites, 16, 12, 3))
  wrapped.close()


def test_gym_wrappers_describe_the_masks():
  from spriteworld_b200 import gym_wrapper
  env = rs._env(_renderers(masks=((16, 12), 1)), E=4)
  vec = gym_wrapper.VectorGymWrapper(env)
  space = vec.single_observation_space.spaces['masks']
  assert space.shape == (12, 16) and space.dtype == np.uint8
  assert int(np.min(space.low)) == 0 and int(np.max(space.high)) == 255
  obs = vec.reset()
  assert tuple(obs['masks'].shape) == (4, 12, 16)
  vec.close()
