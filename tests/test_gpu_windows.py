"""Frames seen through windows (render_kernel<., ., ., true>, swb_render_windows, Engine.render_windows,
renderers.SpriteGlimpses), bit for bit against the render kernel's own frames and against the CPU
restatement tests/window_oracle.py (pinned against Pillow by tests/test_oracle_windows.py)."""
import numpy as np
import pytest
import torch

from oracle import oracle
from spriteworld_b200 import _native
from tests import test_gpu_render_geometry as geo
from tests import test_gpu_render_wide_aa as wide
from tests import window_oracle as wo

gpu = pytest.mark.gpu
FULL = (0.0, 0.0, 1.0, 1.0)


def _full_windows(n, V, device):
  return torch.tensor(FULL, dtype=torch.float64, device=device).repeat(n, V, 1).contiguous()


def _identity(sw, raster):
  """render_windows of (0, 0, 1, 1) with V = 1 and 3 equals render (live) and render_states
  (permuted records), frames and status."""
  from tests.test_gpu_render_states import _permutation
  eng = sw.eng
  frames = eng.render(raster).clone()
  status = eng.render_status().clone()
  perm = torch.from_numpy(_permutation(sw.E)).to(eng.device)
  states = eng.save_envs().take(perm)
  rframes, rstatus = eng.render_states(raster, states)
  for V in (1, 3):
    got, st = eng.render_windows(raster, _full_windows(sw.E, V, eng.device))
    assert torch.equal(got, frames[:, None].expand_as(got)), (sw.case[0], V)
    assert torch.equal(st, status[:, None].expand_as(st)), (sw.case[0], V)
    got, st = eng.render_windows(raster, _full_windows(len(states), V, eng.device), states)
    assert torch.equal(got, rframes[:, None].expand_as(got)), (sw.case[0], V, 'records')
    assert torch.equal(st, rstatus[:, None].expand_as(st)), (sw.case[0], V, 'records')
  assert sw.unmoved()


@gpu
@pytest.mark.parametrize('case', [pytest.param(c, id=c[0]) for c in geo.CASES])
def test_full_window_is_the_frame(case):
  from spriteworld_b200 import engine
  sw = geo.Sweep(case, geo._n_sms())
  try:
    try:
      raster = engine.Raster(sw.eng, sw.W, sw.H, sw.aa, sw.bg)
    except _native.NativeError:
      assert case[0] in geo.REFUSED
      return
    _identity(sw, raster)
    raster.close()
  finally:
    sw.close()


@gpu
@pytest.mark.parametrize('case', [pytest.param(c, id=c[0]) for c in wide.CASES if c[0] not in wide.REFUSED])
def test_full_window_is_the_frame_on_wide_rasters(case):
  from spriteworld_b200 import engine
  sw = geo.Sweep(case, geo._n_sms())
  try:
    raster = engine.Raster(sw.eng, sw.W, sw.H, sw.aa, sw.bg)
    _identity(sw, raster)
    raster.close()
  finally:
    sw.close()


def _random_windows(rng, n, V):
  """Zoom 1/4 .. 64, anisotropic, partly or wholly off the scene."""
  zoom = np.exp(rng.uniform(np.log(0.25), np.log(64.0), (n, V)))
  aspect = rng.choice([1.0, 0.5, 2.5], (n, V))
  cx, cy = rng.uniform(-0.5, 1.5, (n, V)), rng.uniform(-0.5, 1.5, (n, V))
  w, h = 1.0 / zoom, aspect / zoom
  return np.stack([cx - w / 2, cy - h / 2, cx + w / 2, cy + h / 2], -1)


def _check_against_oracle(sw, raster, rows, states, where, V=3, seed=0):
  """Windows of `rows` (env index per row) into guarded buffers at skew 0 and 1: every item is
  either span-overflowed, or flagged BAD_WINDOW exactly as the restatement says with a zero
  frame, or the restatement's frame.  Returns the number of items compared exactly."""
  rng = np.random.RandomState(seed)
  n, H, W = len(rows), sw.H, sw.W
  win = _random_windows(rng, n, V)
  windows = torch.from_numpy(win).to(sw.eng.device).contiguous()
  n_exact = 0
  for skew in (0, 1):
    fbig, fflat, flo = geo._guarded(n * V * H * W * 3, sw.eng.device, skew)
    sbig, sflat, slo = geo._guarded(n * V, sw.eng.device, skew)
    frames, status = sw.eng.render_windows(raster, windows, states, fflat.view(n, V, H, W, 3), sflat.view(n, V))
    geo._assert_guards(fbig, flo, n * V * H * W * 3, (where, 'frames', skew))
    geo._assert_guards(sbig, slo, n * V, (where, 'status', skew))
    frames, status = frames.cpu().numpy(), status.cpu().numpy()
    for i in range(n):
      rec = sw.rec[int(rows[i])]
      for v in range(V):
        st = int(status[i, v])
        if st & _native.ENV_SPAN_OVERFLOW:
          continue
        want, bad = wo.render_window(sw.rc, sw.tab, rec, win[i, v])
        assert bool(st & _native.ENV_BAD_WINDOW) == bad, (where, i, v, st, win[i, v])
        diff = frames[i, v] != want
        assert not diff.any(), (where, skew, i, v, win[i, v].tolist(), int(diff.sum()))
        n_exact += 1
  return n_exact


ORACLE_CASES = [c for c in geo.CASES if c[0] not in geo.REFUSED][:6]


@gpu
@pytest.mark.parametrize('case', [pytest.param(c, id=c[0]) for c in ORACLE_CASES]
                         + [pytest.param(c, id=c[0]) for c in wide.CASES if c[0] not in wide.REFUSED][:2])
def test_zoomed_windows_of_records_match_the_restatement(case):
  from spriteworld_b200 import engine
  sw = geo.Sweep(case, geo._n_sms())
  try:
    raster = engine.Raster(sw.eng, sw.W, sw.H, sw.aa, sw.bg)
    E = sw.E
    perm = (E - 1 - np.arange(min(E, 24) + 3)) % E
    states = sw.eng.save_envs().take(torch.from_numpy(perm).to(sw.eng.device))
    assert _check_against_oracle(sw, raster, perm, states, (case[0], 'records'), seed=1) > 0
    assert sw.unmoved()
    raster.close()
  finally:
    sw.close()


@gpu
def test_live_windows_match_the_restatement():
  from spriteworld_b200 import engine
  case = ORACLE_CASES[0]
  sw = geo.Sweep(case, geo._n_sms())
  try:
    raster = engine.Raster(sw.eng, sw.W, sw.H, sw.aa, sw.bg)
    n = _check_against_oracle(sw, raster, np.arange(sw.E), None, (case[0], 'all live'), V=2, seed=2)
    assert n > 0
    raster.close()
  finally:
    sw.close()


@gpu
def test_bad_windows_are_flagged_and_zeroed():
  from spriteworld_b200 import engine
  case = ORACLE_CASES[0]
  sw = geo.Sweep(case, geo._n_sms())
  try:
    raster = engine.Raster(sw.eng, sw.W, sw.H, sw.aa, sw.bg)
    E, V = sw.E, 4
    win = np.tile(np.array(FULL), (E, V, 1))
    x = float(sw.rec[1]['x'][-1])
    win[0, 1] = (0.5, 0.0, 0.5, 1.0)
    win[0, 2] = (np.nan, 0.0, 1.0, 1.0)
    win[1, 0] = (0.0, 0.0, np.inf, 1.0)
    win[1, 3] = (x, 0.0, x + 1e-12, 1.0)
    win[2, 2] = (0.0, 0.7, 1.0, 0.2)
    frames, status = sw.eng.render_windows(raster, torch.from_numpy(win).to(sw.eng.device))
    full = sw.eng.render(raster)
    frames, status, full = frames.cpu().numpy(), status.cpu().numpy(), full.cpu().numpy()
    for i in range(E):
      for v in range(V):
        bad = wo.bad_window(sw.rc, sw.tab, sw.rec[i], win[i, v])
        assert bool(status[i, v] & _native.ENV_BAD_WINDOW) == bad, (i, v, win[i, v])
        if bad:
          assert not frames[i, v].any()
        elif not status[i, v]:
          assert np.array_equal(frames[i, v], full[i]), (i, v)
    assert status[0, 1] and status[0, 2] and status[1, 0] and status[2, 2]
    raster.close()
  finally:
    sw.close()


def _glimpse_env(E=16, seed=3, sampler='host', config='cobra'):
  from spriteworld_b200 import environment, renderers
  if config == 'cobra':
    from spriteworld_b200.configs.cobra import goal_finding_more_targets as cfgmod
    cfg = cfgmod.get_config('train')
  else:
    from spriteworld_b200.configs.examples import goal_finding_embodied as cfgmod
    cfg = cfgmod.get_config('train')
  hsv = renderers.color_maps.hsv_to_rgb
  cfg['renderers'] = dict(
      image=renderers.PILRenderer(image_size=(32, 32), anti_aliasing=2, color_to_rgb=hsv),
      glimpses=renderers.SpriteGlimpses(image_size=(16, 16), anti_aliasing=3, color_to_rgb=hsv,
                                        window_size=(0.25, 0.2), slots=[0, -1, 2]),
      factors=renderers.SpriteFactors())
  cfg['max_episode_length'] = 6
  return environment.BatchedEnvironment(n_envs=E, pool_depth=5, rng=np.random.RandomState(seed),
                                        sampler=sampler, seed=seed, **cfg)


@gpu
@pytest.mark.parametrize('sampler', ['host', 'device'])
def test_glimpses_through_episodes(sampler):
  env = _glimpse_env(sampler=sampler)
  try:
    g = env._renderers['glimpses']
    raster = env._window_raster(g)
    rng = np.random.RandomState(0)
    ts = env.reset()
    for t in range(14):
      obs = ts.observation['glimpses']
      assert obs.shape == (env.n_envs, 3, 16, 16, 3)
      pos = env.engine.state_tensors()
      win = g.windows(pos['pos_x'], pos['pos_y'])
      want, st = env.engine.render_windows(raster, win)
      assert torch.equal(obs, want) and not st.any(), t
      if t % 5 == 0:   # the oracle on a sample of envs
        states = env.save_envs()
        recs = _oracle_records(env, states)
        for e in (0, env.n_envs - 1):
          for v in range(3):
            ref, bad = wo.render_window(oracle_rc(g), _tab(), recs[e], win[e, v].tolist())
            assert not bad and np.array_equal(obs[e, v].cpu().numpy(), ref), (t, e, v)
      a = torch.from_numpy(rng.uniform(0, 1, (env.n_envs, 4)).astype(np.float32))
      ts = env.step(a)
    # observe() of records equals the glimpses of those records loaded into envs
    states = env.save_envs().take(torch.arange(env.n_envs - 1, -1, -1, device=env.engine.device))
    obs, status = env.observe(states)
    env.load_envs(states)
    assert torch.equal(obs['glimpses'], env.render()['glimpses'])
  finally:
    env.close()


def oracle_rc(g):
  return oracle.raster_cfg(g.width, g.height, g.anti_aliasing, g.bg_color)


def _tab():
  from spriteworld_b200 import constants
  return oracle.shape_table(constants.SHAPES)


def _oracle_records(env, states):
  h = states.to_host()
  recs = []
  for i in range(len(states)):
    r = np.zeros(env.engine.n_slots, dtype=oracle.SPRITE_DTYPE)
    r['x'], r['y'] = h['pos_x'][i], h['pos_y'][i]
    for f in ('m00', 'm01', 'm10', 'm11'):
      r[f] = h[f][i]
    r['shape'] = h['shape'][i]
    r['rgb'] = h['rgb'][i]
    recs.append(r)
  return recs


@gpu
def test_egocentric_embodied_views_centre_on_the_body():
  from spriteworld_b200 import environment, renderers
  from spriteworld_b200.configs.examples import goal_finding_embodied as cfgmod
  cfg = cfgmod.get_config('train')
  body = renderers.SpriteGlimpses(image_size=(64, 64), anti_aliasing=5, window_size=(0.5, 0.5), slots=[-1])
  cfg['renderers'] = dict(ego=body)
  env = environment.BatchedEnvironment(n_envs=32, pool_depth=4, rng=np.random.RandomState(1), **cfg)
  try:
    rng = np.random.RandomState(2)
    ts = env.reset()
    tab, rc = _tab(), oracle_rc(body)
    for t in range(8):
      obs = ts.observation['ego'].cpu().numpy()
      recs = _oracle_records(env, env.save_envs())
      pos = env.engine.state_tensors()
      win = body.windows(pos['pos_x'], pos['pos_y']).cpu().numpy()
      for e in range(env.n_envs):
        alone = recs[e][-1:]
        ref, bad = wo.render_window(rc, tab, alone, win[e, 0])
        assert not bad and np.array_equal(obs[e, 0, 31:33, 31:33], ref[31:33, 31:33]), (t, e)
      a = torch.from_numpy(np.stack([rng.randint(0, 2, env.n_envs), rng.randint(0, 4, env.n_envs)], 1)
                           .astype(np.int32))
      ts = env.step(a)
  finally:
    env.close()


@gpu
def test_render_windows_is_read_only_one_launch_and_refuses_before_enqueuing():
  from spriteworld_b200 import engine
  case = ORACLE_CASES[0]
  sw = geo.Sweep(case, geo._n_sms())
  try:
    eng = sw.eng
    raster = engine.Raster(eng, sw.W, sw.H, sw.aa, sw.bg)
    frames = eng.render(raster).clone()
    status = eng.render_status().clone()
    state = eng.save_state()
    win = _full_windows(sw.E, 2, eng.device)
    torch.cuda.synchronize()
    n0 = eng.launch_count()
    eng.render_windows(raster, win)
    assert eng.launch_count() == n0 + 1
    states = eng.save_envs()
    n0 = eng.launch_count()
    eng.render_windows(raster, _full_windows(3, 2, eng.device), states.take(torch.tensor([0, 1, 2], device=eng.device)))
    assert eng.launch_count() == n0 + 1
    torch.cuda.synchronize()
    assert torch.equal(eng.render_status(), status) and sw.unmoved()
    assert all(torch.equal(a, b) if isinstance(a, torch.Tensor) else True
               for a, b in zip(_flat(eng.save_state()), _flat(state)))
    n0 = eng.launch_count()
    # (torch makes no float64 CUDA tensor at a misaligned address: the C-ABI refusal of one is below)
    strided = torch.zeros((2, sw.E, 4), dtype=torch.float64, device=eng.device).transpose(0, 1)
    assert tuple(strided.shape) == tuple(win.shape) and not strided.is_contiguous()
    bad = [win.float(), win[:, :, :3], win[:-1], win.transpose(0, 1), win.cpu(), win[:, :0], strided]
    for w in bad:
      with pytest.raises((ValueError, _native.NativeError)):
        eng.render_windows(raster, w)
    with pytest.raises(ValueError):
      eng.render_windows(raster, win, frames=torch.empty(1, dtype=torch.uint8, device=eng.device))
    with pytest.raises(ValueError):
      eng.render_windows(raster, win, status=torch.empty((sw.E, 3), dtype=torch.uint8, device=eng.device))
    L, h = eng._lib, eng._h
    import ctypes
    f = torch.empty((sw.E, 2, sw.H, sw.W, 3), dtype=torch.uint8, device=eng.device)
    s = torch.empty((sw.E, 2), dtype=torch.uint8, device=eng.device)
    args = lambda **k: [k.get('eng', h), raster._h, None, k.get('n', sw.E), 0, 1,
                        ctypes.c_void_p(k.get('win', win.data_ptr())), k.get('V', 2),
                        ctypes.c_void_p(f.data_ptr()), ctypes.c_void_p(s.data_ptr()), eng._stream()]
    for k in (dict(n=sw.E - 1), dict(V=0), dict(win=0), dict(win=win.data_ptr() + 4),
              dict(win=f.data_ptr())):
      assert L.swb_render_windows(*args(**k)) != 0, k
    assert eng.launch_count() == n0
    assert torch.equal(eng.render(raster), frames)
    raster.close()
  finally:
    sw.close()


def _flat(x):
  if isinstance(x, dict):
    return [v for k in sorted(x) for v in _flat(x[k])]
  if isinstance(x, (list, tuple)):
    return [v for i in x for v in _flat(i)]
  return [x]


def _no_sync(fn):
  prev = torch.cuda.get_sync_debug_mode()
  torch.cuda.set_sync_debug_mode('error')
  try:
    return fn()
  finally:
    torch.cuda.set_sync_debug_mode(prev)


@gpu
def test_glimpses_of_steps_and_records_do_not_synchronise():
  env = _glimpse_env(E=32)
  try:
    g = env._renderers['glimpses']
    rng = np.random.RandomState(3)
    dev = env.engine.device
    acts = [torch.from_numpy(rng.uniform(0, 1, (env.n_envs, 4)).astype(np.float32)).to(dev) for _ in range(3)]
    env.reset()
    states = env.save_envs()
    res = env.engine.step(acts[0], env._rasters['image'], env._frames['image'])
    env.observe(states)    # SpriteFactors uploads its shape-id table on first use
    torch.cuda.synchronize()
    launches = env.engine.launch_count()
    view = _no_sync(lambda: g.render_batch(env, res))                  # what every step does
    obs, status = _no_sync(lambda: env.observe(states))
    win = g.windows(env.engine.state_tensors()['pos_x'], env.engine.state_tensors()['pos_y'])
    frames, st = _no_sync(lambda: env.render_windows(win, g))
    assert env.engine.launch_count() == launches + 1 + 2 + 1          # observe: the frames and the views
    torch.cuda.synchronize()
    assert torch.equal(view, frames) and not st.any()
    env.load_envs(states)
    assert torch.equal(obs['glimpses'], env.render()['glimpses'])
  finally:
    env.close()


@gpu
def test_render_windows_of_the_environment_and_the_one_env_environment():
  from spriteworld_b200 import environment, renderers
  env = _glimpse_env(E=8)
  try:
    env.reset()
    image = env._renderers['image']
    win = torch.tensor([[0.0, 0.0, 1.0, 1.0], [0.3, 0.2, 0.45, 0.4]], dtype=torch.float64,
                       device=env.engine.device).repeat(env.n_envs, 1, 1)
    frames, status = env.render_windows(win, image)
    assert torch.equal(frames[:, 0], env.render()['image']) and not status.any()
    recs = _oracle_records(env, env.save_envs())
    rc = oracle.raster_cfg(image.width, image.height, image.anti_aliasing, image.bg_color)
    for e in range(env.n_envs):
      ref, bad = wo.render_window(rc, _tab(), recs[e], win[e, 1].tolist())
      assert not bad and np.array_equal(frames[e, 1].cpu().numpy(), ref), e
    with pytest.raises(ValueError, match='color_to_rgb'):
      env.render_windows(win, renderers.PILRenderer(image_size=(8, 8)))
  finally:
    env.close()
  # the one-env Environment: SpriteGlimpses.render through _direct.render_glimpses
  from spriteworld_b200.configs.cobra import goal_finding_more_targets as cfgmod
  cfg = cfgmod.get_config('train')
  hsv = renderers.color_maps.hsv_to_rgb
  cfg['renderers'] = dict(glimpses=renderers.SpriteGlimpses(image_size=(16, 12), anti_aliasing=3, color_to_rgb=hsv,
                                                            window_size=(0.25, 0.3)))
  np.random.seed(4)
  one = environment.Environment(**cfg)
  for t in range(3):
    ts = one.step(np.array([0.3, 0.4, 0.6, 0.7]))
    sprites = one.state()['sprites']
    g = ts.observation['glimpses']
    assert g.shape == (len(sprites), 12, 16, 3)
    for k, s in enumerate(sprites):
      x, y = (float(c) for c in s.position)   # float64 windows, as SpriteGlimpses builds them
      want = wo.pillow_window(sprites, 16, 12, 3, (x - 0.125, y - 0.15, x + 0.125, y + 0.15), color_to_rgb=hsv)
      assert np.array_equal(g[k], want), (t, k)
  one.close()
