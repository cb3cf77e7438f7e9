"""CPU tier of the layer observations: renderers.SpriteLayers and the `draw` of Engine.render_windows
and BatchedEnvironment.render_windows, on the oracle-backed engine double with swb_render_views
(tests/layer_oracle.install: each view drawn by the restatement tests/test_oracle_layers.py pins
against Pillow).

What runs on the host is under test: the one-hot draw and full windows SpriteLayers builds, the
env's buffers and status, observe() and render(), the draw broadcasting and argument checks (each
refused before anything is enqueued), the specs and both gym wrappers, the one-env Environment
through _direct.render_views, and the sharded refusal.  The kernel is tests/test_gpu_layers.py's.
"""
import collections

import numpy as np
import pytest
import torch

from oracle import oracle
from spriteworld_b200 import _native
from tests import layer_oracle as lo
from tests import test_render_states_on_oracle as rs
from tests import window_oracle as wo

FULL = (0.0, 0.0, 1.0, 1.0)


@pytest.fixture
def double(monkeypatch):
  lo.install(monkeypatch)


def _renderers(**layers):
  from spriteworld_b200 import renderers
  hsv = renderers.color_maps.hsv_to_rgb
  out = collections.OrderedDict(image=renderers.PILRenderer(image_size=(16, 12), color_to_rgb=hsv))
  for name, kw in layers.items():
    out[name] = renderers.SpriteLayers(color_to_rgb=hsv, **kw)
  out['factors'] = renderers.SpriteFactors()
  return out


def _oracle_layers(env, renderer, sprites=None):
  """Layers of the double's live envs (or of (n, S) oracle sprites) by the restatement."""
  if sprites is None:
    sprites = env.engine._bo.cur
  S = sprites.shape[1]
  idx = renderer.slot_indices(S)
  rc = oracle.raster_cfg(renderer.width, renderer.height, renderer.anti_aliasing, renderer.bg_color)
  return np.array([[lo.render_layer(rc, env.engine._tab, sprites[e], FULL, np.arange(S) == k)[0] for k in idx]
                   for e in range(len(sprites))], np.uint8)


LAYERS = dict(layers=dict(image_size=(10, 8), anti_aliasing=3, bg_color=(20, 30, 40)),
              some=dict(image_size=(12, 12), anti_aliasing=2, slots=[-1, 0]))


def test_sprite_layers_in_a_batched_environment(double):
  env = rs._env(_renderers(**LAYERS), E=6)
  S = env.engine.n_slots
  spec = env.observation_spec()
  assert spec['layers'].shape == (S, 8, 10, 3) and spec['some'].shape == (2, 12, 12, 3)
  assert spec['layers'].dtype == np.uint8
  rng = np.random.RandomState(2)
  ts = env.reset()
  ptrs = {k: ts.observation[k].data_ptr() for k in LAYERS}
  resets = 0
  for t in range(14):
    if t:
      ts = env.step(rng.uniform(0, 1, (env.n_envs, 4)).astype(np.float32))
    resets += int((ts.step_type == _native.STEP_FIRST).sum())
    assert list(ts.observation) == ['image', 'layers', 'some', 'factors']
    for name in LAYERS:
      obs = ts.observation[name]
      assert obs.data_ptr() == ptrs[name], (t, name)   # the env's buffer, every step
      assert np.array_equal(obs.numpy(), _oracle_layers(env, env._renderers[name])), (t, name)
      for e in range(env.n_envs):
        spec[name].validate(obs[e].numpy())
    # an empty slot's layer is the background
    empty = ~ts.observation['factors']['mask'].numpy().astype(bool)
    assert (ts.observation['layers'].numpy()[empty] == np.array([20, 30, 40], np.uint8)).all()
    assert not (ts.status.numpy() & _native.ENV_BAD_WINDOW).any()
  assert resets > env.n_envs      # episodes ended and restarted
  env.close()


def test_observe_and_render_give_the_layers_of_records(double):
  from tests import oracle_engine
  env = rs._env(_renderers(**LAYERS), E=6)
  rs._started(env, steps=4, seed=5)
  states = env.save_envs()[[4, 4, 1, 0, 5, 3, 2]]
  launches = env.engine.launch_count()
  obs, status = env.observe(states)
  assert list(obs) == ['image', 'layers', 'some', 'factors']
  assert env.engine.launch_count() == launches + 3     # the frames and one launch per SpriteLayers
  # the double's frames report a made-up span overflow (rs._fake_overflow); the layers add nothing
  assert np.array_equal(status.numpy(), rs._fake_overflow(7, 16))
  sprites = oracle_engine.record_sprites(env.engine, states)
  for name in LAYERS:
    r = env._renderers[name]
    assert np.array_equal(obs[name].numpy(), _oracle_layers(env, r, sprites)), name
    assert obs[name].data_ptr() != env._glimpse_buffers[id(r)][0].data_ptr()
    assert torch.equal(r.render_states(env, states), obs[name])
  env.load_envs(states[:6])
  out = env.render()
  assert list(out) == ['image', 'layers', 'some']
  for name in LAYERS:
    assert out[name].data_ptr() == env._glimpse_buffers[id(env._renderers[name])][0].data_ptr()
    assert torch.equal(out[name], obs[name][:6]), name
  env.close()


def test_render_windows_with_draw(double):
  from tests import oracle_engine
  env = rs._env(_renderers(**LAYERS), E=6)
  rs._started(env)
  S = env.engine.n_slots
  image, layers = env._renderers['image'], env._renderers['layers']
  win = torch.tensor([[list(FULL), [0.2, 0.1, 0.6, 0.5]]], dtype=torch.float64).repeat(6, 1, 1)
  rng = np.random.RandomState(4)
  draw = torch.from_numpy(rng.rand(6, 2, S) < 0.5)
  frames, status = env.render_windows(win, image, draw=draw)
  assert frames.shape == (6, 2, 12, 16, 3) and not status.any()
  sprites = env.engine._bo.cur
  rc = oracle.raster_cfg(16, 12, 1)
  for e in range(6):
    for v in range(2):
      want, _ = lo.render_layer(rc, env.engine._tab, sprites[e], win[e, v].tolist(), draw[e, v].numpy())
      assert np.array_equal(frames[e, v].numpy(), want), (e, v)
  # every slot drawn is the window frame; none drawn is the background
  full, _ = env.render_windows(win, image)
  assert torch.equal(env.render_windows(win, image, draw=torch.ones(S, dtype=torch.bool))[0], full)
  assert not env.render_windows(win, image, draw=torch.zeros((), dtype=torch.bool))[0].any()
  # broadcasting: one draw per slot, per view, per row
  for d, full_shape in ((draw[0, 0], (1, 1, S)), (draw[0], (1, 2, S)), (draw[:, :1], (6, 1, S))):
    got, _ = env.render_windows(win, image, draw=d)
    want, _ = env.render_windows(win, image, draw=d.reshape(full_shape).expand(6, 2, S).contiguous())
    assert torch.equal(got, want)
  # records, and a SpriteLayers renderer: the scene without slot k through its raster
  states = env.save_envs()[[2, 0]]
  without = ~torch.eye(S, dtype=torch.bool)[:2].unsqueeze(0)        # view v: every slot but v
  f2, _ = env.render_windows(win[:2], layers, states, draw=without)
  rc = oracle.raster_cfg(10, 8, 3, (20, 30, 40))
  rec = oracle_engine.record_sprites(env.engine, states)
  for i in range(2):
    for v in range(2):
      want, _ = lo.render_layer(rc, env.engine._tab, rec[i], win[i, v].tolist(), without[0, v].numpy())
      assert np.array_equal(f2[i, v].numpy(), want), (i, v)
  env.close()


def test_draw_arguments_are_checked_before_anything_is_enqueued(double):
  from spriteworld_b200 import renderers
  env = rs._env(_renderers(**LAYERS), E=6)
  rs._started(env)
  eng, raster = env.engine, env._rasters['image']
  image = env._renderers['image']
  n, S = eng.n_envs, eng.n_slots
  launches = eng.launch_count()
  win = torch.zeros((n, 2, 4), dtype=torch.float64)
  win[..., 2:] = 1.0
  draw = torch.ones((n, 2, S), dtype=torch.bool)
  # Engine.render_windows: a contiguous bool (n, V, n_slots) tensor on the engine's device
  for d in (draw.to(torch.uint8), draw[:, :, :-1].contiguous(), draw[:1], draw[:, :1].contiguous(),
            torch.ones((n, 2, S + 1), dtype=torch.bool), draw.transpose(0, 1).contiguous().transpose(0, 1),
            draw[0].expand(n, 2, S), draw.to('meta'), draw.numpy()):
    with pytest.raises(ValueError, match='draw'):
      eng.render_windows(raster, win, draw=d)
  # BatchedEnvironment.render_windows: any bool tensor on the device that broadcasts
  for d in (draw.to(torch.uint8), torch.ones((n, 3, S), dtype=torch.bool), torch.ones(S + 1, dtype=torch.bool),
            torch.ones((2, n, 2, S), dtype=torch.bool), draw.to('meta'), draw.numpy(), [True] * S):
    with pytest.raises(ValueError, match='draw'):
      env.render_windows(win, image, draw=d)
  # the windows are still checked first, and the renderer
  with pytest.raises(ValueError, match='windows'):
    env.render_windows(win[:, :, :3], image, draw=draw)
  with pytest.raises(ValueError, match='PILRenderer or SpriteGlimpses'):
    env.render_windows(win, renderers.SpriteMasks(image_size=(16, 12)), draw=draw)
  with pytest.raises(ValueError, match='color_to_rgb'):
    env.render_windows(win, renderers.SpriteLayers(image_size=(16, 12)), draw=draw)
  assert eng.launch_count() == launches
  env.render_windows(win, env._renderers['layers'], draw=draw[0])
  eng.render_windows(raster, win, draw=draw)
  assert eng.launch_count() == launches + 2
  env.close()


def test_sprite_layers_arguments_and_specs(double):
  from spriteworld_b200 import renderers
  for kw in (dict(image_size=(0, 4)), dict(anti_aliasing=0), dict(image_size=(4,)), dict(slots=[])):
    with pytest.raises(ValueError):
      renderers.SpriteLayers(**kw)
  g = renderers.SpriteLayers(image_size=(7, 5), slots=[-1, 0, 2])
  assert g.slot_indices(4) == [3, 0, 2]
  with pytest.raises(IndexError):
    g.slot_indices(2)
  x = torch.tensor([[0.1, 0.2, 0.3, 0.4]] * 2, dtype=torch.float64)
  w, d = g.views(x, 1 - x)
  assert w.shape == (2, 3, 4) and w.dtype == torch.float64 and w.is_contiguous()
  assert (w == torch.tensor(FULL, dtype=torch.float64)).all()
  assert d.dtype == torch.bool and d.is_contiguous() and d.shape == (2, 3, 4)
  assert d[0].int().tolist() == [[0, 0, 0, 1], [1, 0, 0, 0], [0, 0, 1, 0]] and torch.equal(d[0], d[1])
  w, d = renderers.SpriteLayers().views(x, x)
  assert torch.equal(d, torch.eye(4, dtype=torch.bool).expand(2, 4, 4))
  # a slot the engine does not have fails the constructor
  with pytest.raises(IndexError):
    rs._env(_renderers(far=dict(slots=[40])), E=2)
  # colours are packed at upload: one colour map for the PILRenderers and SpriteLayers
  r = _renderers()
  r['l'] = renderers.SpriteLayers()
  with pytest.raises(NotImplementedError, match='color_to_rgb'):
    rs._env(r, E=2)


def test_sprite_layers_render_a_sprite_list(double):
  from spriteworld_b200 import renderers, sprite
  rng = np.random.RandomState(21)
  for n, slots, aa in ((0, None, 2), (1, [-1], 1), (5, None, 3), (5, [4, 0, -2], 2)):
    sprites = [sprite.Sprite(x=rng.uniform(0, 1), y=rng.uniform(0, 1), shape=['triangle', 'square', 'star_5'][k % 3],
                             angle=float(rng.uniform(0, 360)), scale=0.2, c0=255, c1=k * 40, c2=90)
               for k in range(n)]
    g = renderers.SpriteLayers(image_size=(12, 10), anti_aliasing=aa, bg_color=(1, 2, 3), slots=slots)
    got = g.render(sprites)
    idx = g.slot_indices(n)
    assert got.shape == (len(idx), 10, 12, 3) and got.dtype == np.uint8
    assert g.observation_spec().shape == got.shape
    for v, k in enumerate(idx):
      assert np.array_equal(got[v], wo.pillow_window([sprites[k]], 12, 10, aa, FULL, bg=(1, 2, 3))), (n, slots, v)


def _layer_cfg():
  from spriteworld_b200 import renderers
  from spriteworld_b200.configs.cobra import goal_finding_more_targets as cfgmod
  cfg = cfgmod.get_config('train')
  hsv = renderers.color_maps.hsv_to_rgb
  cfg['renderers'] = collections.OrderedDict([
      ('image', renderers.PILRenderer(image_size=(16, 12), color_to_rgb=hsv)),
      ('layers', renderers.SpriteLayers(image_size=(8, 6), anti_aliasing=2, color_to_rgb=hsv))])
  return cfg


def test_gym_wrapper_of_the_drop_in_environment_returns_the_layers(double):
  from spriteworld_b200 import environment, gym_wrapper
  np.random.seed(9)
  cfg = _layer_cfg()
  hsv = cfg['renderers']['layers'].color_to_rgb
  wrapped = gym_wrapper.GymWrapper(environment.Environment(**cfg))
  space = wrapped.observation_space.spaces['layers']
  n = len(wrapped.state()['sprites'])
  assert space.shape == (n, 6, 8, 3) and space.dtype == np.uint8
  for t in range(4):
    obs, _, _, _ = wrapped.step(np.array([0.3, 0.4, 0.6, 0.7]))
    sprites = wrapped.state()['sprites']
    g = obs['layers']
    assert g.shape == space.shape == (len(sprites), 6, 8, 3) and g.dtype == space.dtype, t
    for k, s in enumerate(sprites):
      assert np.array_equal(g[k], wo.pillow_window([s], 8, 6, 2, FULL, color_to_rgb=hsv)), (t, k)
  wrapped.close()


def test_vector_gym_wrapper_returns_the_layers(double):
  from spriteworld_b200 import gym_wrapper
  env = rs._env(_renderers(**LAYERS), E=4)
  S = env.engine.n_slots
  vec = gym_wrapper.VectorGymWrapper(env)
  space = vec.single_observation_space.spaces['layers']
  assert space.shape == (S, 8, 10, 3) and space.dtype == np.uint8
  assert vec.single_observation_space.spaces['some'].shape == (2, 12, 12, 3)
  obs = vec.reset()
  assert tuple(obs['layers'].shape) == (4, S, 8, 10, 3)
  obs, _, _, _ = vec.step(np.random.RandomState(0).uniform(0, 1, (4, 4)).astype(np.float32))
  assert np.array_equal(np.asarray(obs['layers']), _oracle_layers(env, env._renderers['layers']))
  for e in range(4):
    assert space.contains(np.asarray(obs['layers'][e])), e
  vec.close()


def test_sharded_environment_refuses_sprite_layers():
  from spriteworld_b200 import environment
  with pytest.raises(NotImplementedError, match='SpriteLayers'):
    environment.ShardedBatchedEnvironment(8, **_layer_cfg())
