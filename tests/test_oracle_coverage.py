"""CPU tier of the amodal sprite coverage (renderers.SpriteCoverage).

1. The restatement tests/coverage_oracle.py uses (the oracle's Pillow polygon fill, one canvas per
   sprite, sampled at aa*j + aa//2 and flipped) equals the definition written with Pillow itself, bit
   for bit: all twelve shapes, random angles, scales and positions partly and wholly off the canvas,
   stars and spokes across y = 0, sprites with edges beyond +-32768 canvas rows, anti_aliasing up to
   20, non-square and 1-pixel sizes, up to 32 slots (bit 31 included).
2. Its highest set bit + 1 is the mask of tests/mask_oracle.py, visible is that mask's bincount and
   area each bit's popcount; visible <= area, and empty or out-of-frame sprites have no bits.
3. The host layer -- Engine.render_coverage's checks, SpriteCoverage in a BatchedEnvironment (step,
   observe, render, specs), the drop-in Environment and the gym wrappers -- on the oracle-backed
   engine double with swb_render_coverage (tests/mask_oracle.install).  The kernel is
   tests/test_gpu_coverage.py's.
"""
import collections

import numpy as np
import pytest
import torch

from oracle import oracle
from spriteworld_b200 import engine as engine_lib
from tests import coverage_oracle, mask_oracle
from tests import test_oracle_masks as om
from tests import test_render_states_on_oracle as rs

TAB = om.TAB


def _every_shape(rng):
  """One random sprite of each of the twelve shapes, in a random order, and their records."""
  sprites, recs = [], []
  for name in rng.permutation(om.SHAPES):
    s, r = om._sprites(rng, 1, shapes=(name,))
    sprites += s
    recs.append(r)
  return sprites, np.concatenate(recs)


def _check(rec, W, H, aa, sprites=None, what=()):
  """The restatement of records `rec` against the Pillow definition (given the Sprite objects) and
  against the mask restatement; returns the coverage."""
  rc = oracle.raster_cfg(W, H, aa)
  cover, visible, area = coverage_oracle.render_coverage(rc, TAB, rec)
  assert cover.shape == (H, W) and cover.dtype == np.int32, what
  assert visible.shape == area.shape == (len(rec),) and visible.dtype == area.dtype == np.int32, what
  if sprites is not None:
    want = coverage_oracle.pillow_coverage(sprites, W, H, aa)
    assert np.array_equal(cover, want), (what, np.argwhere(cover != want)[:4].tolist())
  mask = mask_oracle.render_masks(rc, TAB, rec)
  assert np.array_equal(coverage_oracle.modal(cover), mask), what
  assert np.array_equal(visible, np.bincount(mask.reshape(-1), minlength=len(rec) + 1)[1:]), what
  bits = cover.view(np.uint32)
  for k in range(len(rec)):
    assert area[k] == int(((bits >> np.uint32(k)) & 1).sum()), (what, k)
  assert (visible <= area).all(), what
  return cover, visible, area


@pytest.mark.parametrize('aa', [1, 2, 3, 5, 10, 13, 20])
def test_oracle_coverage_equals_the_pillow_definition(aa):
  rng = np.random.RandomState(200 + aa)
  for W, H in om.SIZES:
    for n in (1, 5, 32):
      sprites, rec = om._sprites(rng, n)
      _check(rec, W, H, aa, sprites, (aa, W, H, n))
    sprites, rec = _every_shape(rng)
    _check(rec, W, H, aa, sprites, (aa, W, H, 'shapes'))


def _records(sprites):
  """Oracle records of Sprite objects."""
  from tests import fixtures
  n = len(sprites)
  z = np.zeros(n)
  return fixtures.records_from_arrays(dict(
      x=np.array([s.x for s in sprites]), y=np.array([s.y for s in sprites]),
      shape=np.array([oracle.SHAPE_IDS[s.shape] for s in sprites]), angle=np.array([s.angle for s in sprites]),
      scale=np.array([s.scale for s in sprites]), vx=z, vy=z, member=np.zeros(n, np.uint32),
      pos_f32=np.zeros(n, np.uint8), rgb=np.zeros((n, 3), np.uint8)))


def test_bit_31_and_hidden_sprites_keep_their_bits():
  """32 sprites over the same centre, each smaller than the one below: every one but the top is
  partly hidden and keeps its whole silhouette, and bit 31 (the sign bit) is slot 31's."""
  from spriteworld_b200 import sprite
  rng = np.random.RandomState(3)
  sprites, _ = om._sprites(rng, 32)
  sprites = [sprite.Sprite(x=0.5, y=0.5, shape=s.shape, angle=s.angle, scale=0.6 - 0.015 * k)
             for k, s in enumerate(sprites)]
  cover, visible, area = _check(_records(sprites), 16, 16, 3, sprites, 'nested')
  assert (cover < 0).any()                       # bit 31 set somewhere
  assert (area > 0).all() and (visible < area).any()


def test_empty_and_out_of_frame_sprites_have_no_bits():
  from spriteworld_b200 import sprite
  rng = np.random.RandomState(5)
  sprites, _ = om._sprites(rng, 6)
  sprites[3] = sprite.Sprite(x=5.0, y=-4.0, shape='square', scale=0.1)   # wholly out of frame
  rec = _records(sprites)
  rec[0]['shape'] = 0                             # an empty slot, padded at the front
  cover, visible, area = _check(rec, 12, 9, 2, what='empty')
  bits = cover.view(np.uint32)
  for k in (0, 3):
    assert not ((bits >> np.uint32(k)) & 1).any() and visible[k] == 0 and area[k] == 0


def test_stars_and_spokes_across_y0_equal_the_pillow_definition():
  rng = np.random.RandomState(17)
  for aa in (1, 2, 5, 13):
    for W, H in ((16, 16), (9, 4)):
      sprites, rec = om._sprites(rng, 12, y_range=(-0.08, 0.08), shapes=om.STARS)
      _check(rec, W, H, aa, sprites, (aa, W, H))


def test_sprites_with_edges_beyond_int16_rows_equal_the_pillow_definition():
  from spriteworld_b200 import sprite
  from tests import fixtures
  rng = np.random.RandomState(23)
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
      cover, _, area = _check(rec, W, H, aa, sprites, (W, H, aa, e))
      n_crossing += int(0 < area.max() < W * H)
  assert n_crossing >= 6   # outlines do cross the canvases


# ---------------------------------------------------------------------------------------------
# host layer on the engine double
# ---------------------------------------------------------------------------------------------

@pytest.fixture
def double(monkeypatch):
  mask_oracle.install(monkeypatch)


def _renderers(**cover):
  from spriteworld_b200 import renderers
  hsv = renderers.color_maps.hsv_to_rgb
  out = collections.OrderedDict(image=renderers.PILRenderer(image_size=(16, 12), color_to_rgb=hsv))
  out['masks'] = renderers.SpriteMasks(image_size=(16, 12), anti_aliasing=1)
  for name, (size, aa) in cover.items():
    out[name] = renderers.SpriteCoverage(image_size=size, anti_aliasing=aa)
  out['factors'] = renderers.SpriteFactors()
  return out


def _oracle_coverage(env, renderer):
  """Coverage of the double's live envs by the restatement."""
  rc = oracle.raster_cfg(renderer.width, renderer.height, renderer.anti_aliasing)
  bo = env.engine._bo
  got = [coverage_oracle.render_coverage(rc, env.engine._tab, bo.cur[e]) for e in range(env.n_envs)]
  return tuple(np.stack(x) for x in zip(*got))


def _assert_equal(obs, want, what):
  assert list(obs) == ['cover', 'visible', 'area'], what
  for k, w in zip(obs, want):
    assert obs[k].dtype == torch.int32, (what, k)
    assert np.array_equal(obs[k].numpy(), w), (what, k)


def test_sprite_coverage_in_a_batched_environment(double):
  env = rs._env(_renderers(cover=((16, 12), 1), fine=((9, 14), 3)), E=6)
  S = env.engine.n_slots
  spec = env.observation_spec()
  assert spec['cover']['cover'].shape == (12, 16) and spec['cover']['cover'].dtype == np.int32
  assert spec['fine']['cover'].shape == (14, 9)
  assert spec['cover']['visible'].shape == spec['cover']['area'].shape == (S,)
  rng = np.random.RandomState(2)
  ts = env.reset()
  buffers = {k: [t.data_ptr() for t in ts.observation[k].values()] for k in ('cover', 'fine')}
  for t in range(12):
    if t:
      ts = env.step(rng.uniform(0, 1, (env.n_envs, 4)).astype(np.float32))
    assert list(ts.observation) == ['image', 'masks', 'cover', 'fine', 'factors']
    for name in ('cover', 'fine'):
      obs = ts.observation[name]
      assert [v.data_ptr() for v in obs.values()] == buffers[name]   # the env's buffers, every step
      _assert_equal(obs, _oracle_coverage(env, env._renderers[name]), (t, name))
    # the mask of the same step is the highest bit + 1, its bincount is visible
    cover = ts.observation['cover']['cover'].numpy()
    m = ts.observation['masks'].numpy()
    assert np.array_equal(coverage_oracle.modal(cover), m), t
    occupied = ts.observation['factors']['mask'].numpy()
    area = ts.observation['cover']['area'].numpy()
    assert (area[~occupied] == 0).all(), t     # bits index the factors' slot axis
  env.close()


def test_observe_and_render_give_the_coverage_of_records(double):
  env = rs._env(_renderers(cover=((16, 12), 2)), E=6)
  rs._started(env, steps=4, seed=5)
  states = env.save_envs()[[4, 4, 1, 0, 5, 3, 2]]
  launches = env.engine.launch_count()
  obs, _ = env.observe(states)
  assert list(obs) == ['image', 'masks', 'cover', 'factors']
  assert env.engine.launch_count() == launches + 3
  c = obs['cover']
  assert tuple(c['cover'].shape) == (7, 12, 16) and tuple(c['visible'].shape) == (7, env.engine.n_slots)
  own = env._coverage_buffers[id(env._renderers['cover'])]
  assert all(v.data_ptr() != b.data_ptr() for v, b in zip(c.values(), own))
  by_renderer = env._renderers['cover'].render_states(env, states)
  for k in c:
    assert torch.equal(by_renderer[k], c[k]), k
  env.load_envs(states[:6])
  out = env.render()
  assert list(out) == ['image', 'masks', 'cover']
  assert [v.data_ptr() for v in out['cover'].values()] == [b.data_ptr() for b in own]
  for k in c:
    assert torch.equal(out['cover'][k], c[k][:6]), k
  from spriteworld_b200 import renderers
  masks = env.render_masks(renderers.SpriteMasks(image_size=(16, 12), anti_aliasing=2))
  assert np.array_equal(masks.numpy(), coverage_oracle.modal(out['cover']['cover'].numpy()))
  env.close()


def test_render_coverage_checks_its_arguments(double):
  env = rs._env(_renderers(cover=((16, 12), 1)), E=6)
  rs._started(env)
  eng = env.engine
  states = env.save_envs()
  launches = eng.launch_count()
  n, S = eng.n_envs, eng.n_slots
  with pytest.raises(ValueError, match='EnvStates'):
    eng.render_coverage(16, 12, 1, states=states.data)
  other = engine_lib.EnvStates(states.data, 1, b'x' * len(states.signature), states.n_slots)
  with pytest.raises(ValueError, match='another configuration'):
    eng.render_coverage(16, 12, 1, states=other)

  def good():
    return [torch.zeros((n, 12, 16), dtype=torch.int32), torch.zeros((n, S), dtype=torch.int32),
            torch.zeros((n, S), dtype=torch.int32)]
  with pytest.raises(ValueError, match='triple'):
    eng.render_coverage(16, 12, 1, out=good()[0])
  with pytest.raises(ValueError, match='triple'):
    eng.render_coverage(16, 12, 1, out=good()[:2])
  for i, name in enumerate(('cover', 'visible', 'area')):
    shape = good()[i].shape
    wrong = [torch.zeros(shape, dtype=torch.uint8), torch.zeros(shape[::-1], dtype=torch.int32),
             torch.zeros((n - 1,) + tuple(shape[1:]), dtype=torch.int32), np.zeros(shape, np.int32),
             torch.zeros(shape[::-1], dtype=torch.int32).t() if len(shape) == 2 else
             torch.zeros((n, 16, 12), dtype=torch.int32).transpose(1, 2)]
    for bad in wrong:
      out = good()
      out[i] = bad
      with pytest.raises(ValueError, match=name):
        eng.render_coverage(16, 12, 1, out=out)
  assert eng.launch_count() == launches
  out = good()
  got = eng.render_coverage(16, 12, 1, out=out)
  assert all(g is o for g, o in zip(got, out)) and eng.launch_count() == launches + 1
  empty = eng.render_coverage(16, 12, 1, states=states[:0])
  assert [tuple(t.shape) for t in empty] == [(0, 12, 16), (0, S), (0, S)]
  assert eng.launch_count() == launches + 1
  env.close()


def test_sprite_coverage_arguments_and_specs():
  from spriteworld_b200 import renderers
  r = renderers.SpriteCoverage(image_size=(10, 4), anti_aliasing=409)
  spec = r.observation_spec()
  assert list(spec) == ['cover', 'visible', 'area']
  assert spec['cover'].shape == (4, 10) and spec['cover'].dtype == np.int32
  assert spec['visible'].shape == (0,) and spec['area'].dtype == np.int32
  for size, aa in (((0, 4), 1), ((4, 4), 0), ((4096, 1), 1), ((10, 4), 410), ((4,), 1)):
    with pytest.raises(ValueError):
      renderers.SpriteCoverage(image_size=size, anti_aliasing=aa)


def test_sprite_coverage_renders_a_sprite_list(double):
  from spriteworld_b200 import renderers
  rng = np.random.RandomState(21)
  for n, size, aa in ((0, (6, 5), 2), (1, (16, 12), 1), (7, (9, 14), 3), (32, (5, 5), 20)):
    sprites, _ = om._sprites(rng, n) if n else ([], None)
    r = renderers.SpriteCoverage(image_size=size, anti_aliasing=aa)
    got = r.render(sprites)
    want = coverage_oracle.pillow_coverage(sprites, size[0], size[1], aa)
    assert list(got) == ['cover', 'visible', 'area']
    assert got['cover'].dtype == np.int32 and np.array_equal(got['cover'], want), (n, size, aa)
    assert np.array_equal((got['visible'], got['area']), coverage_oracle.counts(want, n)), (n, size, aa)
    assert r.observation_spec()['visible'].shape == (n,)


def test_gym_wrapper_of_the_drop_in_environment_describes_and_returns_the_coverage(double):
  from spriteworld_b200 import environment, gym_wrapper, renderers
  from spriteworld_b200.configs.cobra import goal_finding_more_targets as cfgmod
  cfg = cfgmod.get_config('train')
  cfg['renderers'] = collections.OrderedDict([
      ('cover', renderers.SpriteCoverage(image_size=(16, 12), anti_aliasing=3)),
      ('masks', renderers.SpriteMasks(image_size=(16, 12), anti_aliasing=3))])
  np.random.seed(9)
  wrapped = gym_wrapper.GymWrapper(environment.Environment(**cfg))
  space = wrapped.observation_space.spaces['cover']
  n = len(wrapped.state()['sprites'])
  assert space.spaces['cover'].shape == (12, 16) and space.spaces['cover'].dtype == np.int32
  assert space.spaces['visible'].shape == (n,) and int(np.max(space.spaces['area'].high)) == 12 * 16
  for t in range(4):
    obs, _, _, _ = wrapped.step(np.array([0.3, 0.4, 0.6, 0.7]))
    sprites = wrapped.state()['sprites']
    c = obs['cover']
    assert isinstance(c, dict) and list(c) == ['cover', 'visible', 'area'], t
    assert c['cover'].shape == (12, 16) and c['cover'].dtype == np.int32
    assert np.array_equal(c['cover'], coverage_oracle.pillow_coverage(sprites, 16, 12, 3)), t
    assert np.array_equal(coverage_oracle.modal(c['cover']), obs['masks']), t
    assert np.array_equal(c['visible'], np.bincount(obs['masks'].reshape(-1), minlength=n + 1)[1:]), t
  wrapped.close()


def test_vector_gym_wrapper_describes_and_returns_the_coverage(double):
  from spriteworld_b200 import gym_wrapper
  env = rs._env(_renderers(cover=((16, 12), 1)), E=4)
  S = env.engine.n_slots
  vec = gym_wrapper.VectorGymWrapper(env)
  space = vec.single_observation_space.spaces['cover']
  assert space.spaces['cover'].shape == (12, 16) and space.spaces['cover'].dtype == np.int32
  assert space.spaces['visible'].shape == space.spaces['area'].shape == (S,)
  assert int(np.min(space.spaces['cover'].low)) == -2 ** 31 and int(np.max(space.spaces['cover'].high)) == 2 ** 31 - 1
  obs = vec.reset()
  assert tuple(obs['cover']['cover'].shape) == (4, 12, 16) and tuple(obs['cover']['area'].shape) == (4, S)
  obs, _, _, _ = vec.step(np.random.RandomState(0).uniform(0, 1, (4, 4)).astype(np.float32))
  _assert_equal(obs['cover'], _oracle_coverage(env, env._renderers['cover']), 'vector step')
  vec.close()
