"""CPU tier of the window observations: renderers.SpriteGlimpses, Engine.render_windows and
BatchedEnvironment.render_windows on the oracle-backed engine double with swb_render_windows
(tests/window_oracle.install: each view drawn by the restatement tests/test_oracle_windows.py pins
against Pillow).

What runs on the host is under test: the windows SpriteGlimpses builds from live positions and from
records, the env's buffers and status, observe() and render(), the argument checks of
Engine.render_windows and BatchedEnvironment.render_windows (each refused before anything is
enqueued), the raster cache and its release, the specs and both gym wrappers, the one-env
Environment through _direct.render_glimpses, and the sharded refusal.  The kernel is
tests/test_gpu_windows.py's.
"""
import collections

import numpy as np
import pytest
import torch

from oracle import oracle
from spriteworld_b200 import _native
from tests import test_render_states_on_oracle as rs
from tests import window_oracle as wo


@pytest.fixture
def double(monkeypatch):
  wo.install(monkeypatch)


def _renderers(**glimpses):
  from spriteworld_b200 import renderers
  hsv = renderers.color_maps.hsv_to_rgb
  out = collections.OrderedDict(image=renderers.PILRenderer(image_size=(16, 12), color_to_rgb=hsv))
  for name, kw in glimpses.items():
    out[name] = renderers.SpriteGlimpses(color_to_rgb=hsv, **kw)
  out['factors'] = renderers.SpriteFactors()
  return out


def _oracle_glimpses(env, renderer, sprites=None):
  """(views, bad) of the double's live envs (or of (n, S) oracle sprites) by the restatement."""
  if sprites is None:
    sprites = env.engine._bo.cur
  win = renderer.windows(torch.from_numpy(np.ascontiguousarray(sprites['x'])),
                         torch.from_numpy(np.ascontiguousarray(sprites['y']))).numpy()
  rc = oracle.raster_cfg(renderer.width, renderer.height, renderer.anti_aliasing, renderer.bg_color)
  got = [[wo.render_window(rc, env.engine._tab, sprites[e], win[e, v]) for v in range(win.shape[1])]
         for e in range(len(sprites))]
  return (np.array([[f for f, _ in row] for row in got], np.uint8),
          np.array([[b for _, b in row] for row in got], bool))


GLIMPSES = dict(glimpses=dict(image_size=(10, 8), anti_aliasing=3, window_size=(0.3, 0.2)),
                body=dict(image_size=(12, 12), anti_aliasing=2, window_size=(0.5, 0.5), slots=[-1, 0]))


def test_sprite_glimpses_in_a_batched_environment(double):
  env = rs._env(_renderers(**GLIMPSES), E=6)
  S = env.engine.n_slots
  spec = env.observation_spec()
  assert spec['glimpses'].shape == (S, 8, 10, 3) and spec['body'].shape == (2, 12, 12, 3)
  assert spec['glimpses'].dtype == np.uint8
  rng = np.random.RandomState(2)
  ts = env.reset()
  ptrs = {k: ts.observation[k].data_ptr() for k in GLIMPSES}
  resets = 0
  for t in range(14):
    if t:
      ts = env.step(rng.uniform(0, 1, (env.n_envs, 4)).astype(np.float32))
    resets += int((ts.step_type == _native.STEP_FIRST).sum())
    assert list(ts.observation) == ['image', 'glimpses', 'body', 'factors']
    for name in GLIMPSES:
      obs = ts.observation[name]
      assert obs.data_ptr() == ptrs[name], (t, name)   # the env's buffer, every step
      want, bad = _oracle_glimpses(env, env._renderers[name])
      assert not bad.any() and np.array_equal(obs.numpy(), want), (t, name)
      for e in range(env.n_envs):
        spec[name].validate(obs[e].numpy())
    assert not (ts.status.numpy() & _native.ENV_BAD_WINDOW).any()
  assert resets > env.n_envs      # episodes ended and restarted
  env.close()


def test_bad_views_are_zeros_and_reach_the_step_status(double):
  # a window this small puts every vertex of the sprite it is centred on past 2^30 canvas pixels
  env = rs._env(_renderers(tiny=dict(image_size=(8, 8), window_size=(1e-12, 1e-12), slots=[-1])), E=4)
  ts = env.reset()
  occupied = ts.observation['factors']['mask'][:, -1].numpy()
  assert occupied.all()
  assert (ts.status.numpy() & _native.ENV_BAD_WINDOW).all()
  assert not ts.observation['tiny'].any()
  obs, status = env.observe(env.save_envs())
  assert (status.numpy() & _native.ENV_BAD_WINDOW).all() and not obs['tiny'].any()
  env.close()


def test_observe_and_render_give_the_glimpses_of_records(double):
  env = rs._env(_renderers(**GLIMPSES), E=6)
  rs._started(env, steps=4, seed=5)
  states = env.save_envs()[[4, 4, 1, 0, 5, 3, 2]]
  launches = env.engine.launch_count()
  obs, status = env.observe(states)
  assert list(obs) == ['image', 'glimpses', 'body', 'factors']
  assert env.engine.launch_count() == launches + 3     # the frames and one launch per SpriteGlimpses
  # the double's frames report a made-up span overflow (rs._fake_overflow); the views add nothing
  assert np.array_equal(status.numpy(), rs._fake_overflow(7, 16))
  from tests import oracle_engine
  sprites = oracle_engine.record_sprites(env.engine, states)
  for name in GLIMPSES:
    r = env._renderers[name]
    want, _ = _oracle_glimpses(env, r, sprites)
    assert np.array_equal(obs[name].numpy(), want), name
    assert obs[name].data_ptr() != env._glimpse_buffers[id(r)][0].data_ptr()
    assert torch.equal(r.render_states(env, states), obs[name])
  env.load_envs(states[:6])
  out = env.render()
  assert list(out) == ['image', 'glimpses', 'body']
  for name in GLIMPSES:
    assert out[name].data_ptr() == env._glimpse_buffers[id(env._renderers[name])][0].data_ptr()
    assert torch.equal(out[name], obs[name][:6]), name
  env.close()


def test_render_windows_of_the_environment(double, monkeypatch):
  from spriteworld_b200 import renderers
  env = rs._env(_renderers(**GLIMPSES), E=6)
  rs._started(env)
  image = env._renderers['image']
  win = torch.tensor([[[0.0, 0.0, 1.0, 1.0], [0.2, 0.1, 0.4, 0.5]]], dtype=torch.float64).repeat(6, 1, 1)
  frames, status = env.render_windows(win, image)
  assert frames.shape == (6, 2, 12, 16, 3) and not status.any()
  assert torch.equal(frames[:, 0], env.render()['image'])    # the full window is the frame
  sprites = env.engine._bo.cur
  for e in range(6):
    want, _ = wo.render_window(oracle.raster_cfg(16, 12, 1), env.engine._tab, sprites[e], win[e, 1].tolist())
    assert np.array_equal(frames[e, 1].numpy(), want), e
  states = env.save_envs()[[2, 0]]
  f2, _ = env.render_windows(win[:2], image, states)
  assert torch.equal(f2, frames[[2, 0]])
  # one raster per (W, H, aa, bg): the PILRenderer's and each SpriteGlimpses' (made by the
  # constructor), shared by renderers that draw alike; all closed with the env
  same = renderers.PILRenderer(image_size=(16, 12), color_to_rgb=image.color_to_rgb)
  env.render_windows(win, same)
  assert len(env._window_rasters) == 3
  with pytest.raises(ValueError, match='PILRenderer or SpriteGlimpses'):
    env.render_windows(win, renderers.SpriteMasks(image_size=(16, 12)))
  with pytest.raises(ValueError, match='color_to_rgb'):
    env.render_windows(win, renderers.PILRenderer(image_size=(16, 12)))
  closed = []
  for r in env._window_rasters.values():
    monkeypatch.setattr(r, 'close', lambda r=r: closed.append(r))
  rasters = list(env._window_rasters.values())
  env.close()
  assert closed == rasters


def test_render_windows_checks_its_arguments(double):
  env = rs._env(_renderers(**GLIMPSES), E=6)
  rs._started(env)
  eng, raster = env.engine, env._rasters['image']
  n = eng.n_envs
  launches = eng.launch_count()
  win = torch.zeros((n, 2, 4), dtype=torch.float64)
  win[..., 2:] = 1.0
  odd = torch.zeros(n * 2 * 4 + 1, dtype=torch.float64)[1:].view(n, 2, 4)   # contiguous, 8-byte aligned
  misaligned = torch.frombuffer(bytearray(n * 2 * 32 + 4), dtype=torch.float64, offset=4, count=n * 8).view(n, 2, 4)
  assert misaligned.is_contiguous() and misaligned.data_ptr() % 8
  bad = [win.float(), win.to(torch.int64), win[:, :, :3].contiguous(), win[:-1], win[:, :0],
         win.view(n, 8), win.transpose(1, 2).contiguous().transpose(1, 2),          # (n, 2, 4), not contiguous
         torch.zeros((2, n, 4), dtype=torch.float64).transpose(0, 1),            # the same
         misaligned, win.to('meta'), win.numpy()]
  assert tuple(bad[6].shape) == (n, 2, 4) and not bad[6].is_contiguous()
  for w in bad:
    with pytest.raises(ValueError, match='windows'):
      eng.render_windows(raster, w)
  with pytest.raises(ValueError, match='EnvStates'):
    eng.render_windows(raster, win, states=env.save_envs().data)
  states = env.save_envs()[[0, 1, 2]]
  with pytest.raises(ValueError, match='windows'):
    eng.render_windows(raster, win, states)                   # n = 6 windows for 3 records
  H, W = raster.height, raster.width
  for f in (torch.zeros((n, 2, H, W, 3), dtype=torch.int32), torch.zeros((n, 1, H, W, 3), dtype=torch.uint8),
            torch.zeros((n, 2, W, H, 3), dtype=torch.uint8), torch.zeros((2, n, H, W, 3), dtype=torch.uint8)
            .transpose(0, 1)):
    with pytest.raises(ValueError, match='frames'):
      eng.render_windows(raster, win, frames=f)
  for s in (torch.zeros((n, 2), dtype=torch.int32), torch.zeros(n * 2, dtype=torch.uint8),
            torch.zeros((2, n), dtype=torch.uint8).t()):
    with pytest.raises(ValueError, match='status'):
      eng.render_windows(raster, win, status=s)
  assert eng.launch_count() == launches
  frames, status = eng.render_windows(raster, odd)
  assert eng.launch_count() == launches + 1
  got = eng.render_windows(raster, win[:3].contiguous(), states)
  assert got[0].shape == (3, 2, H, W, 3) and eng.launch_count() == launches + 2
  env.close()


def test_sprite_glimpses_arguments_and_specs(double):
  from spriteworld_b200 import renderers
  for kw in (dict(image_size=(0, 4)), dict(anti_aliasing=0), dict(image_size=(4,)), dict(window_size=(0, 1)),
             dict(window_size=(np.inf, 1)), dict(window_size=(np.nan, 1)), dict(window_size=(1,)), dict(slots=[])):
    with pytest.raises(ValueError):
      renderers.SpriteGlimpses(**kw)
  g = renderers.SpriteGlimpses(image_size=(7, 5), slots=[-1, 0, 2])
  assert g.slot_indices(4) == [3, 0, 2]
  with pytest.raises(IndexError):
    g.slot_indices(2)
  x = torch.tensor([[0.1, 0.2, 0.3, 0.4]], dtype=torch.float64)
  w = g.windows(x, 1 - x)
  assert w.shape == (1, 3, 4) and w.dtype == torch.float64 and w.is_contiguous()
  assert w[0, 0].tolist() == [0.4 - 0.125, 0.6 - 0.125, 0.4 + 0.125, 0.6 + 0.125]
  # a slot the engine does not have fails the constructor
  with pytest.raises(IndexError):
    rs._env(_renderers(far=dict(slots=[40])), E=2)
  # colours are packed at upload: one colour map for the PILRenderers and SpriteGlimpses
  r = _renderers()
  r['g'] = renderers.SpriteGlimpses()
  with pytest.raises(NotImplementedError, match='color_to_rgb'):
    rs._env(r, E=2)


def test_sprite_glimpses_render_a_sprite_list(double):
  from spriteworld_b200 import renderers, sprite
  rng = np.random.RandomState(21)
  for n, slots, aa in ((0, None, 2), (1, [-1], 1), (5, None, 3), (5, [4, 0, -2], 2)):
    sprites = [sprite.Sprite(x=rng.uniform(0, 1), y=rng.uniform(0, 1), shape=['triangle', 'square', 'star_5'][k % 3],
                             angle=float(rng.uniform(0, 360)), scale=0.1, c0=255, c1=k * 40, c2=90)
               for k in range(n)]
    g = renderers.SpriteGlimpses(image_size=(12, 10), anti_aliasing=aa, window_size=(0.3, 0.4), slots=slots)
    got = g.render(sprites)
    idx = g.slot_indices(n)
    assert got.shape == (len(idx), 10, 12, 3) and got.dtype == np.uint8
    assert g.observation_spec().shape == got.shape
    for v, k in enumerate(idx):
      x, y = (float(c) for c in sprites[k].position)
      win = (x - 0.15, y - 0.2, x + 0.15, y + 0.2)
      assert np.array_equal(got[v], wo.pillow_window(sprites, 12, 10, aa, win)), (n, slots, v)


def _glimpse_cfg():
  from spriteworld_b200 import renderers
  from spriteworld_b200.configs.cobra import goal_finding_more_targets as cfgmod
  cfg = cfgmod.get_config('train')
  hsv = renderers.color_maps.hsv_to_rgb
  cfg['renderers'] = collections.OrderedDict([
      ('image', renderers.PILRenderer(image_size=(16, 12), color_to_rgb=hsv)),
      ('glimpses', renderers.SpriteGlimpses(image_size=(8, 6), anti_aliasing=2, color_to_rgb=hsv,
                                            window_size=(0.25, 0.25)))])
  return cfg


def test_gym_wrapper_of_the_drop_in_environment_returns_the_glimpses(double):
  from spriteworld_b200 import environment, gym_wrapper
  np.random.seed(9)
  cfg = _glimpse_cfg()
  hsv = cfg['renderers']['glimpses'].color_to_rgb
  wrapped = gym_wrapper.GymWrapper(environment.Environment(**cfg))
  space = wrapped.observation_space.spaces['glimpses']
  n = len(wrapped.state()['sprites'])
  assert space.shape == (n, 6, 8, 3) and space.dtype == np.uint8
  for t in range(4):
    obs, _, _, _ = wrapped.step(np.array([0.3, 0.4, 0.6, 0.7]))
    sprites = wrapped.state()['sprites']
    g = obs['glimpses']
    # the wrapper describes array observations as the reference's does (shape and dtype)
    assert g.shape == space.shape == (len(sprites), 6, 8, 3) and g.dtype == space.dtype, t
    for k, s in enumerate(sprites):
      x, y = (float(c) for c in s.position)   # float64 windows, as SpriteGlimpses builds them
      want = wo.pillow_window(sprites, 8, 6, 2, (x - 0.125, y - 0.125, x + 0.125, y + 0.125), color_to_rgb=hsv)
      assert np.array_equal(g[k], want), (t, k)
  wrapped.close()


def test_vector_gym_wrapper_returns_the_glimpses(double):
  from spriteworld_b200 import gym_wrapper
  env = rs._env(_renderers(**GLIMPSES), E=4)
  S = env.engine.n_slots
  vec = gym_wrapper.VectorGymWrapper(env)
  space = vec.single_observation_space.spaces['glimpses']
  assert space.shape == (S, 8, 10, 3) and space.dtype == np.uint8
  assert vec.single_observation_space.spaces['body'].shape == (2, 12, 12, 3)
  obs = vec.reset()
  assert tuple(obs['glimpses'].shape) == (4, S, 8, 10, 3)
  obs, _, _, _ = vec.step(np.random.RandomState(0).uniform(0, 1, (4, 4)).astype(np.float32))
  want, _ = _oracle_glimpses(env, env._renderers['glimpses'])
  assert np.array_equal(np.asarray(obs['glimpses']), want)
  for e in range(4):
    assert space.contains(np.asarray(obs['glimpses'][e])), e
  vec.close()


def test_sharded_environment_refuses_sprite_glimpses():
  from spriteworld_b200 import environment
  with pytest.raises(NotImplementedError, match='SpriteGlimpses'):
    environment.ShardedBatchedEnvironment(8, **_glimpse_cfg())
