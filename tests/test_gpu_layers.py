"""Views with only some sprites drawn (the `draw` of render_kernel<., ., ., true>, swb_render_views,
Engine.render_windows(draw=...), renderers.SpriteLayers) on the device.

Device against device: over every case and window of the window sweep (tests/test_gpu_window_sweep.py),
swb_render_views with a random draw equals, byte for byte, swb_render_windows of the same records with
each undrawn slot's shape byte set to 0, and an all-ones draw equals swb_render_windows.  Against the
restatements: a sample of the views against tests/layer_oracle.py and tests/span_overflow.py on the
drawn subset.  Then the properties (layers at aa = 1 against the device's own coverage, the empty
subset, a far sprite left out) and the environment paths.
"""
import ctypes

import numpy as np
import pytest
import torch

from oracle import oracle
from spriteworld_b200 import _native
from tests import layer_oracle as lo
from tests import test_gpu_render_geometry as geo
from tests import test_gpu_window_sweep as ws
from tests import test_gpu_windows as gw

gpu = pytest.mark.gpu
FULL = (0.0, 0.0, 1.0, 1.0)


def _random_draw(rng, n, V, S):
  """(n, V, S) draw masks: random subsets, with every row's first view all drawn and its second none."""
  d = rng.rand(n, V, S) < rng.uniform(0.2, 0.8, (n, V, 1))
  if V > 1:
    d[:, 0] = True
    d[:, 1] = False
  return d


def _emptied(c, states, undrawn):
  """EnvStates `states` with slot s's shape byte 0 in every record i where undrawn[i, s]."""
  from spriteworld_b200 import engine
  data = states.data.cpu().numpy().copy()
  for s in range(c.S):
    if undrawn[:, s].any():
      ws._set_field(data, c.S, 'shape', np.flatnonzero(undrawn[:, s]), s, 0)
  return engine.EnvStates(torch.from_numpy(data).to(states.data.device), states.span_class, states.signature, c.S)


def _views(sw, raster, windows, states, draw, n, V, c, skew, where):
  """swb_render_views into guarded buffers at `skew`: (frames, status) on the host."""
  H, W = c.H, c.W
  fbig, fflat, flo = geo._guarded(n * V * H * W * 3, sw.eng.device, skew)
  sbig, sflat, slo = geo._guarded(n * V, sw.eng.device, skew)
  frames, status = sw.eng.render_windows(raster, windows, states, fflat.view(n, V, H, W, 3), sflat.view(n, V),
                                         draw=draw)
  geo._assert_guards(fbig, flo, n * V * H * W * 3, where + ('frames', skew))
  geo._assert_guards(sbig, slo, n * V, where + ('status', skew))
  return frames.cpu().numpy(), status.cpu().numpy()


def _restated(c, sp, win, draw, i, v):
  """(frame, status) the restatements give view (i, v) of (n, S) sprites `sp` with draw[i, v]."""
  spv = sp.copy()
  spv[i] = lo.drawn_sprites(sp[i], draw[i, v])
  got = ws.expected(c, spv, win, i, v)
  return got[0], got[1]


def _run(sw, c, raster, source, V):
  cid = c.case[0]
  seed = ws._seed(cid, source, V)
  rows, sp, edits, win, fam, _ = ws.plan(c, source, V, seed)
  n, S = len(rows), c.S
  live_states = sw.eng.save_envs()
  states = None if source == 'live' else ws._records(sw, c, rows, edits)
  base = live_states if source == 'live' else states
  windows = torch.from_numpy(win).to(sw.eng.device).contiguous()
  rng = np.random.RandomState(seed + 7)
  draw = _random_draw(rng, n, V, S)
  draw_t = torch.from_numpy(draw).to(sw.eng.device)
  where = (cid, source, V)
  (f0, s0), (f1, s1) = (_views(sw, raster, windows, states, draw_t, n, V, c, skew, where) for skew in (0, 1))
  assert np.array_equal(s0, s1) and np.array_equal(f0, f1), where + ('skews differ',)
  # each view against swb_render_windows of the records with the undrawn slots emptied
  for v in range(V):
    ref_states = _emptied(c, base, ~draw[:, v])
    rf, rs = sw.eng.render_windows(raster, windows[:, v:v + 1].contiguous(), ref_states)
    rf, rs = rf[:, 0].cpu().numpy(), rs[:, 0].cpu().numpy()
    assert np.array_equal(s0[:, v], rs), where + (v, np.flatnonzero(s0[:, v] != rs)[:4])
    if source == 'live':
      # live rows against records: a frame with SPAN_OVERFLOW is not defined, so not compared
      ok = (rs & ws.SPAN_OVERFLOW) == 0
      assert np.array_equal(f0[ok, v], rf[ok]), where + (v,)
    else:
      assert np.array_equal(f0[:, v], rf), where + (v,)
  # every slot drawn is swb_render_windows, frames and status
  ones = torch.ones((n, V, S), dtype=torch.bool, device=sw.eng.device)
  af, ast = sw.eng.render_windows(raster, windows, states, draw=ones)
  wf, wst = sw.eng.render_windows(raster, windows, states)
  assert torch.equal(af, wf) and torch.equal(ast, wst), where + ('all drawn',)
  # a sample against the restatements: every flagged view up to 6, and 3 others
  flagged = np.argwhere(s0 != 0)
  others = np.argwhere(s0 == 0)
  pick = list(flagged[rng.permutation(len(flagged))[:6]]) + list(others[rng.permutation(len(others))[:3]])
  for i, v in pick:
    frame, want = _restated(c, sp, win, draw, i, v)
    assert int(s0[i, v]) == want, where + (int(i), int(v), fam[i, v], int(s0[i, v]), want)
    if want != ws.SPAN_OVERFLOW:
      assert np.array_equal(f0[i, v], frame), where + (int(i), int(v), fam[i, v])
  return int((s0 == 0).sum())


@gpu
@pytest.mark.parametrize('case', [pytest.param(c, id=c[1][0]) for c in ws.CASES])
def test_views_are_windows_of_the_emptied_records(case):
  from spriteworld_b200 import engine
  c = ws.Case(*case)
  sw = ws._sweep(c)
  try:
    raster = engine.Raster(sw.eng, c.W, c.H, c.aa, c.bg)
    for source, V in ws.RUNS:
      assert _run(sw, c, raster, source, V) > 0, (c.case[0], source, V)
    assert sw.unmoved()
    raster.close()
  finally:
    sw.close()


# ---------------------------------------------------------------------------------------------
# properties
# ---------------------------------------------------------------------------------------------

def _layer_env(E=16, seed=3, sampler='host', aa=3):
  from spriteworld_b200 import environment, renderers
  from spriteworld_b200.configs.cobra import goal_finding_more_targets as cfgmod
  cfg = cfgmod.get_config('train')
  hsv = renderers.color_maps.hsv_to_rgb
  cfg['renderers'] = dict(
      image=renderers.PILRenderer(image_size=(32, 32), anti_aliasing=2, color_to_rgb=hsv),
      layers=renderers.SpriteLayers(image_size=(24, 20), anti_aliasing=aa, bg_color=(10, 20, 30), color_to_rgb=hsv),
      some=renderers.SpriteLayers(image_size=(16, 16), anti_aliasing=2, color_to_rgb=hsv, slots=[-1, 0]),
      factors=renderers.SpriteFactors())
  cfg['max_episode_length'] = 6
  return environment.BatchedEnvironment(n_envs=E, pool_depth=5, rng=np.random.RandomState(seed),
                                        sampler=sampler, seed=seed, **cfg)


def _oracle_layers(env, renderer, states):
  recs = gw._oracle_records(env, states)
  S = env.engine.n_slots
  rc = oracle.raster_cfg(renderer.width, renderer.height, renderer.anti_aliasing, renderer.bg_color)
  tab = gw._tab()
  return np.array([[lo.render_layer(rc, tab, r, FULL, np.arange(S) == k)[0] for k in renderer.slot_indices(S)]
                   for r in recs], np.uint8)


@gpu
def test_one_hot_layers_at_aa_1_are_the_device_coverage():
  env = _layer_env(E=24, aa=1)
  try:
    rng = np.random.RandomState(1)
    env.reset()
    for _ in range(3):
      env.step(torch.from_numpy(rng.uniform(0, 1, (env.n_envs, 4)).astype(np.float32)))
    layers = env.render()['layers'].cpu().numpy()
    cover = env.engine.render_coverage(24, 20, 1)[0].cpu().numpy()
    rgb = env.save_envs().to_host()['rgb']
    bg = np.array([10, 20, 30], np.uint8)
    for k in range(env.engine.n_slots):
      bit = ((cover >> k) & 1).astype(bool)[..., None]
      want = np.where(bit, rgb[:, k, None, None, :], bg)
      assert np.array_equal(layers[:, k], want), k
  finally:
    env.close()


@gpu
def test_the_empty_subset_is_the_background_and_a_far_sprite_left_out_is_not_flagged():
  from spriteworld_b200 import engine
  env = _layer_env(E=8)
  try:
    env.reset()
    eng, S = env.engine, env.engine.n_slots
    image = env._renderers['image']
    win = torch.tensor([FULL, (0.2, 0.3, 0.5, 0.6)], dtype=torch.float64, device=eng.device).repeat(8, 1, 1)
    frames, status = env.render_windows(win, image, draw=torch.zeros((), dtype=torch.bool, device=eng.device))
    assert not status.any() and (frames == 0).all()      # the image's background is black
    f2, _ = env.render_windows(win, env._renderers['layers'],
                               draw=torch.zeros((), dtype=torch.bool, device=eng.device))
    assert (f2 == torch.tensor([10, 20, 30], dtype=torch.uint8, device=eng.device)).all()
    # slot k of every record 2^40 away: drawn it flags the view, left out it does not
    states = eng.save_envs()
    data = states.data.cpu().numpy().copy()
    occupied = states.to_host()['shape'] != 0
    k = int(np.argmax(occupied.sum(0)))
    rows = occupied[:, k]
    assert rows.any()
    ws._set_field(data, S, 'pos_x', np.arange(8), k, 2.0 ** 40)
    far = engine.EnvStates(torch.from_numpy(data).to(eng.device), states.span_class, states.signature, S)
    every = torch.ones(S, dtype=torch.bool, device=eng.device)
    without = every.clone()
    without[k] = False
    f, st = env.render_windows(win, image, far, draw=every)
    flagged = (st.cpu().numpy() & _native.ENV_BAD_WINDOW) != 0
    assert (flagged == rows[:, None]).all() and not f[torch.from_numpy(rows).to(eng.device)].any()
    f, st = env.render_windows(win, image, far, draw=without)
    assert not st.any()
    ref, _ = env.render_windows(win, image, states, draw=without)
    assert torch.equal(f, ref)
    # SpriteLayers of the far records: only layer k is flagged and zero
    obs, status = env.observe(far)
    assert (((status.cpu().numpy() & _native.ENV_BAD_WINDOW) != 0) == rows).all()
    lay = obs['layers'].cpu().numpy()
    assert not lay[rows, k].any()
    others = [s for s in range(S) if s != k]
    assert np.array_equal(lay[:, others], env.observe(states)[0]['layers'].cpu().numpy()[:, others])
  finally:
    env.close()


# ---------------------------------------------------------------------------------------------
# environment paths
# ---------------------------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize('sampler', ['host', 'device'])
def test_sprite_layers_through_episodes(sampler):
  env = _layer_env(sampler=sampler)
  try:
    S = env.engine.n_slots
    rng = np.random.RandomState(0)
    ts = env.reset()
    for t in range(14):
      obs = ts.observation['layers']
      assert obs.shape == (env.n_envs, S, 20, 24, 3) and ts.observation['some'].shape == (env.n_envs, 2, 16, 16, 3)
      assert not (ts.status.cpu().numpy() & _native.ENV_BAD_WINDOW).any()
      if t % 5 == 0:   # the oracle on a sample of envs
        states = env.save_envs()
        sample = torch.tensor([0, env.n_envs - 1], device=env.engine.device)
        want = _oracle_layers(env, env._renderers['layers'], states.take(sample))
        assert np.array_equal(obs[sample].cpu().numpy(), want), t
        want = _oracle_layers(env, env._renderers['some'], states.take(sample))
        assert np.array_equal(ts.observation['some'][sample].cpu().numpy(), want), t
      ts = env.step(torch.from_numpy(rng.uniform(0, 1, (env.n_envs, 4)).astype(np.float32)))
    # observe() of records, and of expand's leaves, equals the layers of those records loaded
    states = env.save_envs().take(torch.arange(env.n_envs - 1, -1, -1, device=env.engine.device))
    _, leaves = env.expand(rng.uniform(0, 1, (3, env.n_envs, 2, 4)))
    for recs in (states, leaves.take(torch.arange(env.n_envs, device=env.engine.device) * 2 + 1)):
      obs, status = env.observe(recs)
      env.load_envs(recs)
      out = env.render()
      assert torch.equal(obs['layers'], out['layers']) and torch.equal(obs['some'], out['some'])
      want = _oracle_layers(env, env._renderers['layers'], recs.take(torch.tensor([1], device=env.engine.device)))
      assert np.array_equal(obs['layers'][1:2].cpu().numpy(), want)
  finally:
    env.close()


@gpu
def test_views_are_read_only_one_launch_and_refusals_enqueue_nothing():
  from spriteworld_b200 import engine
  case = gw.ORACLE_CASES[0]
  sw = geo.Sweep(case, geo._n_sms())
  try:
    eng, S = sw.eng, sw.S
    raster = engine.Raster(eng, sw.W, sw.H, sw.aa, sw.bg)
    frames = eng.render(raster).clone()
    status = eng.render_status().clone()
    state = eng.save_state()
    win = gw._full_windows(sw.E, 2, eng.device)
    draw = torch.from_numpy(np.random.RandomState(0).rand(sw.E, 2, S) < 0.5).to(eng.device)
    torch.cuda.synchronize()
    n0 = eng.launch_count()
    eng.render_windows(raster, win, draw=draw)
    assert eng.launch_count() == n0 + 1
    states = eng.save_envs()
    n0 = eng.launch_count()
    three = states.take(torch.tensor([0, 1, 2], device=eng.device))
    eng.render_windows(raster, gw._full_windows(3, 2, eng.device), three, draw=draw[:3].contiguous())
    assert eng.launch_count() == n0 + 1
    torch.cuda.synchronize()
    assert torch.equal(eng.render_status(), status) and sw.unmoved()
    assert all(torch.equal(a, b) if isinstance(a, torch.Tensor) else True
               for a, b in zip(gw._flat(eng.save_state()), gw._flat(state)))
    n0 = eng.launch_count()
    for d in (draw.to(torch.uint8), draw[:, :, :-1], draw.cpu(), draw[:1], draw.transpose(0, 1)):
      with pytest.raises(ValueError, match='draw'):
        eng.render_windows(raster, win, draw=d)
    # the C-ABI: everything swb_render_windows refuses, a null draw, a draw over the outputs
    L, h = eng._lib, eng._h
    f = torch.empty((sw.E, 2, sw.H, sw.W, 3), dtype=torch.uint8, device=eng.device)
    s = torch.empty((sw.E, 2), dtype=torch.uint8, device=eng.device)
    args = lambda **k: [k.get('eng', h), raster._h, None, k.get('n', sw.E), 0, 1,
                        ctypes.c_void_p(k.get('win', win.data_ptr())), ctypes.c_void_p(k.get('draw', draw.data_ptr())),
                        k.get('V', 2), ctypes.c_void_p(f.data_ptr()), ctypes.c_void_p(s.data_ptr()), eng._stream()]
    for k in (dict(n=sw.E - 1), dict(V=0), dict(win=0), dict(win=win.data_ptr() + 4), dict(win=f.data_ptr()),
              dict(draw=0), dict(draw=f.data_ptr() + 1), dict(draw=s.data_ptr()),
              dict(draw=f.data_ptr() + f.numel() - 1)):
      assert L.swb_render_views(*args(**k)) != 0, k
    assert b'draw' in L.swb_last_error()
    assert eng.launch_count() == n0
    assert L.swb_render_views(*args()) == 0 and eng.launch_count() == n0 + 1
    assert torch.equal(eng.render(raster), frames)
    raster.close()
  finally:
    sw.close()


@gpu
def test_layers_of_steps_and_records_do_not_synchronise():
  env = _layer_env(E=32)
  try:
    g = env._renderers['layers']
    rng = np.random.RandomState(3)
    dev = env.engine.device
    acts = [torch.from_numpy(rng.uniform(0, 1, (env.n_envs, 4)).astype(np.float32)).to(dev) for _ in range(3)]
    env.reset()
    states = env.save_envs()
    res = env.engine.step(acts[0], env._rasters['image'], env._frames['image'])
    env.observe(states)    # SpriteFactors uploads its shape-id table on first use
    image = env._renderers['image']
    win = torch.tensor([FULL, (0.1, 0.1, 0.4, 0.4)], dtype=torch.float64, device=dev).repeat(env.n_envs, 1, 1)
    draw = torch.rand((env.n_envs, 1, env.engine.n_slots), device=dev) < 0.5
    torch.cuda.synchronize()
    launches = env.engine.launch_count()
    view = _no_sync(lambda: g.render_batch(env, res))                  # what every step does
    obs, status = _no_sync(lambda: env.observe(states))
    frames, st = _no_sync(lambda: env.render_windows(win, image, draw=draw))
    assert env.engine.launch_count() == launches + 1 + 3 + 1          # observe: the frames and two layer views
    torch.cuda.synchronize()
    assert not st.any()
    assert torch.equal(view.clone(), g.render_states(env, env.save_envs()))
    env.load_envs(states)
    assert torch.equal(obs['layers'], env.render()['layers'])
  finally:
    env.close()


_no_sync = gw._no_sync


@gpu
def test_the_one_env_environment_draws_each_sprite_alone():
  from spriteworld_b200 import environment, renderers
  from spriteworld_b200.configs.cobra import goal_finding_more_targets as cfgmod
  from tests import window_oracle as wo
  cfg = cfgmod.get_config('train')
  hsv = renderers.color_maps.hsv_to_rgb
  cfg['renderers'] = dict(layers=renderers.SpriteLayers(image_size=(16, 12), anti_aliasing=3, color_to_rgb=hsv))
  np.random.seed(4)
  one = environment.Environment(**cfg)
  for t in range(3):
    ts = one.step(np.array([0.3, 0.4, 0.6, 0.7]))
    sprites = one.state()['sprites']
    g = ts.observation['layers']
    assert g.shape == (len(sprites), 12, 16, 3)
    for k, s in enumerate(sprites):
      assert np.array_equal(g[k], wo.pillow_window([s], 16, 12, 3, FULL, color_to_rgb=hsv)), (t, k)
  one.close()
