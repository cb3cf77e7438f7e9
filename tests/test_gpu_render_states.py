"""Frames of env records without loading them (render_kernel<., ., true>, swb_render_states), bit for bit.

Records saved from the render sweeps' engines, permuted so that no record index equals its env
index and repeated past E, render as the oracle renders the envs they were saved from, at aligned
and odd frame addresses, on narrow and wide rasters.  Leaves of expand() render as the step kernel
rendered each plan's last live step.  Stars rendered by a convex-only engine, sanitised shape ids
and zero records render as a load would make them.  A call changes nothing but its outputs, is one
launch, and a refused one enqueues nothing.  observe() runs inside a device beam search without
the host waiting, and next to the asynchronous refill without changing a run.
"""
import collections
import ctypes

import numpy as np
import pytest
import torch

from spriteworld_b200 import _native
from tests import test_gpu_render_geometry as geo
from tests import test_gpu_render_wide_aa as wide
from tests.test_gpu_rollout import SWEEP

gpu = pytest.mark.gpu


class _Permuted(object):
  """Sweep.check's view of records `perm` of a Sweep: frame i is env perm[i]'s."""

  def __init__(self, sw, perm):
    self.sw, self.perm, self.E, self.M, self.segcap = sw, perm, len(perm), sw.M, sw.segcap

  def ref(self, i):
    return self.sw.ref(int(self.perm[i]))

  overflow = geo.Sweep.overflow
  within = geo.Sweep.within
  check = geo.Sweep.check


def _permutation(E):
  """2E + 3 env indices, reversed and repeated, none at its own position."""
  i = np.arange(2 * E + 3)
  perm = (E - 1 - i) % E
  return np.where(perm == i, (i + 1) % E, perm)


def _render_permuted(sw, raster):
  """Renders the permuted records into guarded buffers at skew 0 and 1; returns the frames
  compared bit-exact per skew."""
  perm = _permutation(sw.E)
  states = sw.eng.save_envs().take(torch.from_numpy(perm).to(sw.eng.device))
  n, H, W = len(perm), sw.H, sw.W
  view = _Permuted(sw, perm)
  n_exact = []
  for skew in (0, 1):
    fbig, fflat, flo = geo._guarded(n * H * W * 3, sw.eng.device, skew)
    sbig, sflat, slo = geo._guarded(n, sw.eng.device, skew)
    frames, status = sw.eng.render_states(raster, states, fflat.view(n, H, W, 3), sflat)
    assert frames.data_ptr() == fflat.data_ptr() and status.data_ptr() == sflat.data_ptr()
    geo._assert_guards(fbig, flo, n * H * W * 3, (sw.case[0], 'frames', skew))
    geo._assert_guards(sbig, slo, n, (sw.case[0], 'status', skew))
    n_exact.append(view.check(frames.cpu().numpy(), status.cpu().numpy(), (sw.case[0], 'records', skew)))
  assert sw.unmoved()
  n_within = sum(view.within(i) for i in range(n))
  return n_exact, n_within


# -- 1, 2: the render sweeps, from records ---------------------------------------------------------

@gpu
@pytest.mark.parametrize('case', [pytest.param(c, id=c[0], marks=geo.KNOWN_DEFECTS.get(c[0], ()))
                                  for c in geo.CASES])
def test_records_render_as_the_oracle_renders_their_envs(case):
  from spriteworld_b200 import engine
  sw = geo.Sweep(case, geo._n_sms())
  try:
    try:
      raster = engine.Raster(sw.eng, sw.W, sw.H, sw.aa, sw.bg)
    except _native.NativeError as ex:
      assert case[0] in geo.REFUSED, (case[0], 'refused: %s' % ex)
      return
    assert case[0] not in geo.REFUSED
    n_exact, n_within = _render_permuted(sw, raster)
    assert n_within >= 0.9 * (2 * sw.E + 3) and n_exact == [n_within] * 2, (case[0], n_exact, n_within)
    raster.close()
  finally:
    sw.close()


@gpu
@pytest.mark.parametrize('case', [pytest.param(c, id=c[0]) for c in wide.CASES if c[0] not in wide.REFUSED])
def test_records_render_on_wide_rasters(case):
  from spriteworld_b200 import engine
  cid, W, H, aa, bg, S, E, concave, scene = case
  sw = geo.Sweep(case, geo._n_sms())
  try:
    sw.segcap = wide.render_layout(W, H, aa, S, concave)[1]
    raster = engine.Raster(sw.eng, W, H, aa, bg)
    n_exact, n_within = _render_permuted(sw, raster)
    assert n_within >= 0.9 * (2 * sw.E + 3) and n_exact == [n_within] * 2, (cid, n_exact, n_within)
    raster.close()
  finally:
    sw.close()


# -- 3: leaves --------------------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize('name', SWEEP)
def test_leaves_render_as_the_step_kernel_rendered_their_last_live_step(name):
  from spriteworld_b200 import constants, engine
  from tests import test_gpu_step_sweep as sweep
  case = next(c for c in sweep.CASES if c['name'] == name)
  arrs, nodes, action, acts = sweep._setup(case)
  eng = sweep._engine(case, nodes, arrs, action)
  E, mel = case['E'], case['mel']
  for a in acts[:3]:
    eng.step(torch.from_numpy(np.ascontiguousarray(a)).to(eng.device))
  rng = np.random.RandomState(len(name))
  eng.upload_state(step_count=rng.randint(0, mel, E).astype(np.int32),
                   reset_next=(eng.download_state()['reset_next'] | (rng.rand(E) < 0.1)).astype(np.uint8))
  T, C = 6, 3
  plans = sweep.case_actions(case, arrs, rng, T * C)
  plans = np.ascontiguousarray(plans.reshape((T, C, E) + plans.shape[2:]).swapaxes(1, 2))
  roots = eng.save_envs()
  leaves = eng.rollout(torch.from_numpy(plans).to(eng.device), states=roots, leaves=True).leaves
  raster = engine.Raster(eng, 40, 24, 3, (20, 30, 40))
  got, got_status = eng.render_states(raster, leaves)
  got, got_status = got.cpu().numpy(), got_status.cpu().numpy()
  # the engine of E x C envs loaded from the repeated roots, stepped with frames
  big = engine.Engine(E * C, case['S'], 1, action, nodes, constants.SHAPES, keep_in_frame=case['keep'],
                      max_episode_length=mel)
  big_raster = engine.Raster(big, 40, 24, 3, (20, 30, 40))
  big.load_envs(roots[np.repeat(np.arange(E), C)])
  frames = [big.render(big_raster).cpu().numpy()]
  status = [big.render_status().cpu().numpy().copy()]
  step_type = []
  for t in range(T):
    res = big.step(torch.from_numpy(np.ascontiguousarray(plans[t].reshape((E * C,) + plans.shape[3:]))).to(big.device),
                   big_raster)
    frames.append(res.frames.cpu().numpy())
    status.append(res.status.cpu().numpy() & _native.ENV_SPAN_OVERFLOW)
    step_type.append(res.step_type.cpu().numpy())
  st = np.stack(step_type)
  lasts_before = np.cumsum(st == _native.STEP_LAST, 0) - (st == _native.STEP_LAST)
  started = np.cumsum(st == _native.STEP_FIRST, 0) > 0
  n_live = ((lasts_before == 0) & ~started).sum(0)
  for i in range(E * C):
    assert np.array_equal(got[i], frames[n_live[i]][i]), (name, i, int(n_live[i]))
    assert got_status[i] == status[n_live[i]][i], (name, i)
  for r in (raster, big_raster):
    r.close()
  big.close()
  eng.close()


# -- 4: a span class the engine has not seen --------------------------------------------------------

@gpu
def test_stars_render_on_a_convex_only_engine_for_that_call_only():
  from spriteworld_b200 import constants, engine
  case = next(c for c in geo.CASES if c[0] == 'w64h65a5')      # stars in the pool, S = 17
  sw = geo.Sweep(case, geo._n_sms())
  states = sw.eng.save_envs()
  assert states.span_class == 4
  convex = engine.Engine(3, sw.S, 1, dict(kind='select_move', scale=1.0), [dict(kind='no_reward')],
                         constants.SHAPES, keep_in_frame=False)
  raster = engine.Raster(convex, sw.W, sw.H, sw.aa, sw.bg)
  frames, status = convex.render_states(raster, states)
  n_exact = sw.check(frames.cpu().numpy(), status.cpu().numpy(), 'convex engine')
  assert n_exact >= 0.9 * sw.E
  assert convex.save_envs().span_class == 1
  raster.close()
  convex.close()
  sw.close()


# -- 5: sanitised and zero records ------------------------------------------------------------------

@gpu
def test_sanitised_shape_ids_and_zero_records_render_as_a_load_makes_them():
  from spriteworld_b200 import engine
  from tests.test_expand_on_oracle import _set_field
  case = next(c for c in geo.CASES if c[0] == 'full_concave')
  sw = geo.Sweep(case, geo._n_sms())
  raster = engine.Raster(sw.eng, sw.W, sw.H, sw.aa, sw.bg)
  states = sw.eng.save_envs()
  data = states.data.cpu().numpy().copy()
  shape = states.to_host()['shape']
  shape[0, :] = 255
  shape[1, ::2] = 13
  shape[2, 1::3] = 200
  _set_field(data, sw.S, 'shape', shape)
  bad = engine.EnvStates(torch.from_numpy(data).to(sw.eng.device), states.span_class, states.signature, sw.S)
  got, got_status = sw.eng.render_states(raster, bad)
  sw.eng.load_envs(bad)
  want = sw.eng.render(raster)
  assert torch.equal(got, want) and torch.equal(got_status, sw.eng.render_status())
  assert bool((got[0] == torch.tensor(sw.bg, dtype=torch.uint8, device=got.device)).all())
  # out-of-range take() indices give zero records: background only, status 0
  zero = states.take(torch.tensor([-1, sw.E, 10 ** 6], device=sw.eng.device))
  frames, status = sw.eng.render_states(raster, zero)
  bg = torch.tensor(sw.bg, dtype=torch.uint8, device=frames.device)
  assert bool((frames == bg).all()) and not bool(status.any())
  raster.close()
  sw.close()


# -- 6: read-only, one launch -----------------------------------------------------------------------

def _env(E=32, refill='sync', seed=3, factors=False):
  from spriteworld_b200 import action_spaces, environment, renderers
  from spriteworld_b200.configs.cobra import goal_finding_more_targets as cfgmod
  cfg = cfgmod.get_config('train')
  cfg['max_episode_length'] = 6
  cfg['action_space'] = action_spaces.SelectMove(scale=0.25, noise_scale=0.05)
  if factors:
    cfg['renderers'] = collections.OrderedDict([
        ('factors', renderers.SpriteFactors()), ('image', cfg['renderers']['image']),
        ('small', renderers.PILRenderer(image_size=(24, 20), anti_aliasing=2,
                                        color_to_rgb=renderers.color_maps.hsv_to_rgb))])
  return environment.BatchedEnvironment(n_envs=E, pool_depth=5, rng=np.random.RandomState(seed),
                                        refill=refill, **cfg)


def _live(env):
  eng = env.engine
  torch.cuda.synchronize(eng.device)
  out = {k: v.cpu().numpy().copy() for k, v in eng.state_tensors().items()}
  out.update({'pool_' + k: v.cpu().numpy().copy() for k, v in eng.pool_tensors().items()})
  out.update({'frames_' + k: v.cpu().numpy().copy() for k, v in env._frames.items()})
  out['render_status'] = eng.render_status().cpu().numpy().copy()
  out['scene_serial'] = eng.download_state_serial()
  return out


@gpu
def test_observe_changes_nothing_and_is_one_launch_per_raster():
  from spriteworld_b200 import renderers
  env = _env(factors=True)
  rng = np.random.RandomState(1)
  env.reset()
  for _ in range(4):
    env.step(rng.uniform(0, 1, (env.n_envs, 4)).astype(np.float32))
  states = env.save_envs()
  states = states.take(torch.from_numpy(rng.randint(0, env.n_envs, 50)).to(env.engine.device))
  before, launches = _live(env), env.engine.launch_count()
  book = (env._t, env._resets, env._safe_step, env._safe_resets, env.refill_stats())
  rng_state = env._rng.get_state()[1].copy()
  obs, status = env.observe(states)
  assert list(obs) == ['factors', 'image', 'small']
  assert env.engine.launch_count() == launches + 2
  after = _live(env)
  for k, v in before.items():
    assert np.array_equal(v, after[k]), k
  assert book == (env._t, env._resets, env._safe_step, env._safe_resets, env.refill_stats())
  assert np.array_equal(rng_state, env._rng.get_state()[1])
  assert obs['image'].data_ptr() != env._frames['image'].data_ptr()
  assert tuple(obs['image'].shape) == (50, 64, 64, 3) and tuple(obs['small'].shape) == (50, 20, 24, 3)
  assert tuple(status.shape) == (50,) and status.dtype == torch.uint8
  # n = 0 enqueues nothing
  frames, st = env.engine.render_states(env._rasters['image'], states[0:0])
  assert tuple(frames.shape) == (0, 64, 64, 3) and env.engine.launch_count() == launches + 2
  # the factors of the records are those of the envs after loading them
  names = ('x', 'y', 'shape', 'angle', 'scale', 'c0', 'c1', 'c2', 'x_vel', 'y_vel')
  direct = env.factor_tensors(names, states[:env.n_envs])
  sf = renderers.SpriteFactors().render_states(env, states[:env.n_envs])
  frames = {k: obs[k][:env.n_envs].clone() for k in ('image', 'small')}
  env.load_envs(states[:env.n_envs])
  loaded = env.factor_tensors(names)
  for k in names + ('mask',):
    assert torch.equal(direct[k], loaded[k]) and torch.equal(sf[k], loaded[k]), k
    assert torch.equal(obs['factors'][k][:env.n_envs], loaded[k]), k
  for k, v in env.render().items():
    assert torch.equal(frames[k], v), k
  env.close()


# -- 7: refusals ------------------------------------------------------------------------------------

@gpu
def test_refused_calls_enqueue_nothing():
  from spriteworld_b200 import constants, engine
  from tests.test_gpu_launch_checks import E, _assert_unchanged, _engine, _snapshot
  eng = _engine()
  raster = engine.Raster(eng, 16, 16, 2)
  eng.step(torch.full((E, 4), 0.5, device=eng.device))
  states = eng.save_envs()
  rb, n = eng.record_bytes, E
  fb = n * 16 * 16 * 3
  buf = torch.zeros(n * rb + fb + 64, dtype=torch.uint8, device=eng.device)
  frames = torch.full((fb,), 7, dtype=torch.uint8, device=eng.device)
  status = torch.full((n,), 7, dtype=torch.uint8, device=eng.device)
  R, F, S = states.data.data_ptr(), frames.data_ptr(), status.data_ptr()
  before = _snapshot(eng)

  def call(records=R, n=n, records_bytes=n * rb, span=1, frames=F, status=S, engine=eng._h, raster=raster._h):
    return eng._lib.swb_render_states(engine, raster, records, n, records_bytes, span, frames, status,
                                      eng._stream())

  def refused(match, **kw):
    assert call(**kw) != 0 and match in eng._lib.swb_last_error(), (kw, eng._lib.swb_last_error())
    _assert_unchanged(eng, before)

  refused(b'null', engine=None)
  refused(b'null', raster=None)
  refused(b'n = -1', n=-1)
  refused(b'null', records=None)
  refused(b'records is not 16-byte aligned', records=R + 8)
  refused(b'records need', records_bytes=n * rb - 1)
  for span in (0, 2, 3, 5):
    refused(b'span_class', span=span)
  refused(b'null', frames=None)
  refused(b'null', status=None)
  B = buf.data_ptr() + (-buf.data_ptr()) % 16
  refused(b'frames overlap', records=B, frames=B + n * rb - 1)
  refused(b'frames overlap', records=B + 16, frames=B)
  refused(b'status overlaps', records=B, status=B + (n - 1) * rb)
  refused(b'status overlaps frames', status=F + fb - 1)
  tall = engine.Raster(eng, 4, 65, 1)                               # two bands per frame
  refused(b'exceed', raster=tall._h, n=2 ** 30, records_bytes=2 ** 30 * rb, frames=16, status=32)
  other = engine.Engine(E, 2, 1, dict(kind='select_move', scale=0.05), [dict(kind='no_reward')], constants.SHAPES)
  foreign = engine.Raster(other, 16, 16, 2)
  refused(b'another engine', raster=foreign._h)
  assert call(n=0, records=None, frames=None, status=None) == 0
  _assert_unchanged(eng, before)
  assert bool((frames == 7).all()) and bool((status == 7).all())
  # the Python checks
  longer = engine.Engine(E, 2, 1, dict(kind='select_move', scale=0.05), [dict(kind='no_reward')],
                         constants.SHAPES, max_episode_length=77)
  with pytest.raises(ValueError, match='another configuration'):
    eng.render_states(raster, longer.save_envs())
  longer.close()
  with pytest.raises(ValueError):
    eng.render_states(raster, states.data)
  for bad in (torch.zeros((n, 16, 16, 3), dtype=torch.int32, device=eng.device),
              torch.zeros((n, 16, 17, 3), dtype=torch.uint8, device=eng.device),
              torch.zeros((n + 1, 16, 16, 3), dtype=torch.uint8, device=eng.device),
              torch.zeros((n, 16, 16, 3), dtype=torch.uint8),
              torch.zeros((n, 16, 3, 16), dtype=torch.uint8, device=eng.device).transpose(2, 3)):
    with pytest.raises(ValueError, match='frames'):
      eng.render_states(raster, states, frames=bad)
  for bad in (torch.zeros(n, dtype=torch.int32, device=eng.device), torch.zeros(n + 1, dtype=torch.uint8, device=eng.device),
              torch.zeros(n, dtype=torch.uint8)):
    with pytest.raises(ValueError, match='status'):
      eng.render_states(raster, states, status=bad)
  _assert_unchanged(eng, before)
  for r in (raster, tall, foreign):
    r.close()
  other.close()
  eng.close()


# -- 8: a beam search that looks at its frontier -----------------------------------------------------

@gpu
def test_device_beam_search_observes_every_level_without_the_host():
  from spriteworld_b200 import action_spaces, environment
  from spriteworld_b200.configs.cobra import goal_finding_more_targets as cfgmod
  from tests.test_gpu_rollout_states import _level_return
  E, B, C, D, T = 64, 4, 16, 3, 2
  cfg = cfgmod.get_config('train')
  cfg['max_episode_length'] = 7
  cfg['action_space'] = action_spaces.SelectMove(scale=0.5)
  env = environment.BatchedEnvironment(n_envs=E, pool_depth=4, sampler='device', seed=3, **cfg)
  env.reset()
  rng = np.random.RandomState(2)
  for _ in range(2):
    env.step(rng.uniform(0, 1, (E, 4)).astype(np.float32))
  dev = env.engine.device
  roots = env.save_envs()
  gen = torch.Generator(device=dev)
  n_rasters = len(env._rasters)

  def search():
    gen.manual_seed(1)
    frontier, width = roots, 1
    score = torch.zeros(E, dtype=torch.float64, device=dev)
    for _ in range(D):
      obs, _ = env.observe(frontier)
      value = obs['image'].view(len(frontier), -1).to(torch.float64).mean(1) * 1e-6   # a stand-in value net
      plans = torch.rand((T, E * width, C, 4), device=dev, generator=gen)
      r, leaves = env.expand(plans, states=frontier)
      total = ((score + value)[:, None] + _level_return(r.reward)).view(E, width * C)
      score, best = total.topk(B, dim=1)
      leaf = (best + torch.arange(E, device=dev)[:, None] * (width * C)).view(-1)
      frontier, width = leaves.take(leaf), B
      score = score.reshape(-1)
    return frontier

  search()
  torch.cuda.synchronize()
  launches = env.engine.launch_count()
  torch.cuda._sleep(1 << 31)
  frontier = search()
  assert env.engine.launch_count() == launches + D * (1 + n_rasters)
  frames = env.observe(frontier)[0]['image']
  done = torch.cuda.Event()
  done.record()
  assert not done.query()                             # everything above was enqueued while busy
  torch.cuda.synchronize()
  # the final frontier's frames: E * B records, loaded E at a time into the env and rendered
  for i in range(B):
    env.load_envs(frontier[i * E:(i + 1) * E])
    assert torch.equal(env.render()['image'], frames[i * E:(i + 1) * E]), i
  env.close()


# -- 9: next to the asynchronous refill ---------------------------------------------------------------

@gpu
def test_observing_records_does_not_change_an_asynchronous_run():
  a, b = _env(E=48, refill='async', seed=9), _env(E=48, refill='async', seed=9)
  rng = np.random.RandomState(4)
  ts_a, ts_b = a.reset(), b.reset()
  for t in range(40):
    obs, _ = a.observe(a.save_envs())
    actions = rng.uniform(0, 1, (48, 4)).astype(np.float32)
    ts_a, ts_b = a.step(actions), b.step(actions)
    for k in ('step_type', 'reward', 'discount', 'success', 'status'):
      assert torch.equal(getattr(ts_a, k), getattr(ts_b, k)), (t, k)
    assert torch.equal(ts_a.observation['image'], ts_b.observation['image']), t
  a.close()
  b.close()
