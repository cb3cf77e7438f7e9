"""Rollout trajectories (csrc/swb_rollout.cuh, swb_rollout_trajectory), byte for byte.

Record (t * n + r) * C + c of a trajectory is leaf r * C + c of the rollout of the first t + 1
steps: checked against expand(actions[:t + 1]) for every t, over every action kind and dtype, a bad
Embodied direction, Clustering, a MetaAggregated root, plans that end early, roots about to reset,
live and record roots, the sorting task, sampled goals and a pool of stars (span class 4).  The
outputs are rollout's, bit for bit.  observe() of slice t equals the frames and masks a live env
shows after loading the root and stepping the plan's live steps, and the CPU oracle's.  A call is
one launch, changes nothing, and a refused call enqueues nothing.
"""
import ctypes

import numpy as np
import pytest
import torch

from oracle import oracle
from spriteworld_b200 import _native
from tests.test_gpu_rollout import NAMES, _bits, _everything, _host

gpu = pytest.mark.gpu


def _t(eng, a):
  return torch.from_numpy(np.ascontiguousarray(a)).to(eng.device)


def _check(eng, plans, states=None):
  """The trajectory of `plans` (device tensor) from `states` (None: the live envs), checked against
  rollout and against expand of every prefix, and shown to be one launch that changes nothing.
  Returns (outputs on the host, trajectory EnvStates)."""
  T, n, C = plans.shape[:3]
  before, launches = _everything(eng), eng.launch_count()
  res = eng.rollout(plans, states=states, trajectory=True)
  assert eng.launch_count() == launches + 1 and res.leaves is None
  after = _everything(eng)
  for k, v in before.items():
    assert np.array_equal(v, after[k], equal_nan=True), k
  traj = res.trajectory
  assert len(traj) == T * n * C and traj.signature == eng.signature
  got, want = _host(res), _host(eng.rollout(plans, states=states))
  for k in NAMES:
    assert np.array_equal(_bits(got[k]), _bits(want[k])), k
  data = traj.data.cpu().numpy().reshape(T, n * C, -1)
  for t in range(T):
    leaves = eng.rollout(plans[:t + 1].contiguous(), states=states, leaves=True).leaves
    assert leaves.span_class == traj.span_class
    assert np.array_equal(data[t], leaves.data.cpu().numpy()), t
  return got, traj


# -- 1: every prefix, over the step sweep's paths ------------------------------------------------

CASES = ['select_f32_s1_e1', 'select_f64_s2', 'drag_f32_s5_mixed', 'drag_f64_s8_mixed', 'embodied_s7',
         'clustering_f32', 'meta_all_aggs', 'edges_free']


@gpu
@pytest.mark.parametrize('name', CASES)
def test_every_slice_is_the_leaf_of_that_prefix(name):
  from tests import test_gpu_step_sweep as sweep
  case = next(c for c in sweep.CASES if c['name'] == name)
  arrs, nodes, action, acts = sweep._setup(case)
  eng = sweep._engine(case, nodes, arrs, action)
  E, mel = case['E'], case['mel']
  for a in acts[:3]:
    eng.step(_t(eng, a))
  rng = np.random.RandomState(len(name) + 7)
  eng.upload_state(step_count=rng.randint(0, mel, E).astype(np.int32),
                   reset_next=(eng.download_state()['reset_next'] | (rng.rand(E) < 0.1)).astype(np.uint8))
  T, C = 7, 3
  plans = sweep.case_actions(case, arrs, rng, T * C)
  plans = _t(eng, plans.reshape((T, C, E) + plans.shape[2:]).swapaxes(1, 2))
  roots = eng.save_envs()
  live_out, live = _check(eng, plans)
  rec_out, rec = _check(eng, plans, roots)
  assert torch.equal(live.data, rec.data) and live.span_class == roots.span_class
  for k in NAMES:
    assert np.array_equal(_bits(live_out[k]), _bits(rec_out[k])), k
  h = rec.to_host()
  resetting = np.repeat(roots.to_host()['reset_next'] > 0, C)
  root_rep = roots.data.cpu().numpy()[np.repeat(np.arange(E), C)]
  data = rec.data.cpu().numpy().reshape(T, E * C, -1)
  for t in range(T):                      # a root about to reset is its own record at every t
    assert np.array_equal(data[t][resetting], root_rep[resetting]), t
  st = rec_out['step_type'].reshape(T, E * C)
  ended = np.cumsum(st == _native.STEP_LAST, 0) > 0
  assert np.array_equal(h['reset_next'].reshape(T, E * C)[:, ~resetting], ended[:, ~resetting])
  if E >= 33:                             # plans that ended inside the window
    assert ended[-1, ~resetting].any()
  if name == 'embodied_s7':
    assert (rec_out['status'] & _native.ENV_BAD_ACTION).any()
  eng.close()


# -- 2: observations of every step against live envs and the oracle ------------------------------

def _env_cfg(kind):
  from spriteworld_b200 import renderers
  from spriteworld_b200.configs.cobra import goal_finding_more_targets, sorting
  if kind == 'goals':
    from tests.test_gpu_goals import _cfg
    cfg = _cfg(max_episode_length=9)
    cfg['renderers'] = dict(cfg['renderers'], image=goal_finding_more_targets.get_config('train')['renderers']['image'])
  else:
    cfg = dict((sorting if kind == 'sorting' else goal_finding_more_targets).get_config('train'))
    cfg['max_episode_length'] = 9
  cfg['renderers'] = dict(cfg['renderers'], mask=renderers.SpriteMasks(image_size=(40, 24), anti_aliasing=3))
  return cfg


@gpu
@pytest.mark.parametrize('kind,dtype', [('goal_finding', np.float32), ('goal_finding', np.float64),
                                        ('sorting', np.float32), ('goals', np.float64)])
def test_observations_of_every_step_equal_a_live_env_and_the_oracle(kind, dtype):
  from spriteworld_b200 import constants, environment
  from tests import mask_oracle
  from tests.oracle_engine import record_sprites
  E, T, C = 24, 6, 3
  env = environment.BatchedEnvironment(n_envs=E, pool_depth=4, sampler='device', seed=11, **_env_cfg(kind))
  eng = env.engine
  assert (eng.n_goals > 0) == (kind == 'goals')
  env.reset()
  rng = np.random.RandomState(4)
  for _ in range(3):
    env.step(rng.uniform(0, 1, (E, 4)).astype(np.float32))
  roots = env.save_envs()
  plans = rng.uniform(0, 1, (T, E, C, 4)).astype(dtype)
  book = (env._t, env._resets, env._safe_step, env.refill_stats())
  frames = {k: v.clone() for k, v in env._frames.items()}
  launches = eng.launch_count()
  r, traj = env.rollout_trajectory(plans)
  assert eng.launch_count() == launches + 1
  assert book == (env._t, env._resets, env._safe_step, env.refill_stats())
  assert all(torch.equal(v, env._frames[k]) for k, v in frames.items())
  rr = env.rollout(plans)
  for k in r._fields:
    assert np.array_equal(_bits(getattr(r, k).cpu().numpy()), _bits(getattr(rr, k).cpu().numpy())), k
  _check(eng, _t(eng, plans), roots)
  obs, status = env.observe(traj)
  torch.cuda.synchronize()
  image = obs['image'].cpu().numpy().reshape(T, E, C, *obs['image'].shape[1:])
  mask = obs['mask'].cpu().numpy().reshape(T, E, C, *obs['mask'].shape[1:])
  st = r.step_type.cpu().numpy()
  # a live env loaded from the roots and stepped through plan c, compared while the plan is live
  n_cmp = 0
  for c in range(C):
    env.load_envs(roots)
    alive = roots.to_host()['reset_next'] == 0
    for t in range(T):
      ts = env.step(np.ascontiguousarray(plans[t, :, c]))
      got_st = ts.step_type.cpu().numpy()
      assert np.array_equal(got_st[alive], st[t, alive, c])
      for name, ours in (('image', image), ('mask', mask)):
        theirs = ts.observation[name].cpu().numpy()
        assert np.array_equal(ours[t, alive, c], theirs[alive]), (name, t, c)
      n_cmp += int(alive.sum())
      alive &= got_st == _native.STEP_MID
  assert n_cmp > E * C
  # the CPU oracle's frames and masks of the last slice
  last = traj[(T - 1) * E * C:]
  sprites = record_sprites(eng, last)
  tab = oracle.shape_table(constants.SHAPES)
  img = env._rasters['image']
  rc = oracle.raster_cfg(img.width, img.height, img.anti_aliasing)
  rcm = oracle.raster_cfg(40, 24, 3)
  for i in range(0, E * C, 5):
    assert np.array_equal(image[T - 1].reshape(E * C, *image.shape[3:])[i], oracle.render(rc, tab, sprites[i])), i
    assert np.array_equal(mask[T - 1].reshape(E * C, *mask.shape[3:])[i],
                          mask_oracle.render_masks(rcm, tab, sprites[i])), i
  env.close()


# -- 3: stars ------------------------------------------------------------------------------------

@gpu
def test_a_pool_of_stars_keeps_span_class_4_and_renders_every_step():
  from spriteworld_b200 import engine
  from tests import test_gpu_render_geometry as geo
  case = next(c for c in geo.CASES if c[0] == 'w64h65a5')      # stars in the pool
  sw = geo.Sweep(case, geo._n_sms())
  eng = sw.eng
  roots = eng.save_envs()
  assert roots.span_class == 4
  rng = np.random.RandomState(2)
  T, C = 3, 2
  plans = _t(eng, rng.uniform(0, 1, (T, sw.E, C, 4)).astype(np.float32))
  _, live = _check(eng, plans)
  _, rec = _check(eng, plans, roots)
  assert live.span_class == 4 and rec.span_class == 4 and torch.equal(live.data, rec.data)
  raster = engine.Raster(eng, sw.W, sw.H, sw.aa, sw.bg)
  leaves = eng.rollout(plans, states=roots, leaves=True).leaves
  got, got_status = eng.render_states(raster, rec[(T - 1) * sw.E * C:])
  want, want_status = eng.render_states(raster, leaves)
  assert torch.equal(got, want) and torch.equal(got_status, want_status)
  raster.close()
  sw.close()


# -- 4: refusals ---------------------------------------------------------------------------------

@gpu
def test_refused_trajectories_enqueue_nothing():
  from spriteworld_b200 import engine
  from tests.test_gpu_launch_checks import E, _assert_unchanged, _engine, _snapshot
  T, C = 3, 2
  eng = _engine()
  acts = torch.zeros((T, E, C, 4), dtype=torch.float32, device=eng.device)
  eng.step(acts[0, :, 0].contiguous())
  roots = eng.save_envs()
  rb = eng.record_bytes
  n_rec = T * E * C
  buf = torch.zeros((n_rec + E + 1) * rb, dtype=torch.uint8, device=eng.device)   # room to overlap
  res = eng.rollout(acts)
  out = _native.StepOut(res.reward.data_ptr(), res.step_type.data_ptr(), res.success.data_ptr(),
                        res.status.data_ptr())
  before = _snapshot(eng)
  span = ctypes.c_int32(-5)
  R, L = roots.data.data_ptr(), buf.data_ptr()

  def call(roots=R, n_roots=E, roots_bytes=E * rb, n_steps=T, n_candidates=C, outputs=out, records=L,
           records_bytes=n_rec * rb):
    return eng._lib.swb_rollout_trajectory(eng._h, roots, n_roots, roots_bytes, acts.data_ptr(), _native.DTYPE_F32,
                                           n_steps, n_candidates, ctypes.byref(outputs), records, records_bytes,
                                           ctypes.byref(span), eng._stream())

  def refused(match, **kw):
    assert call(**kw) != 0 and match in eng._lib.swb_last_error(), (kw, eng._lib.swb_last_error())
    _assert_unchanged(eng, before)
    assert span.value == -5

  refused(b'null output records', records=None)
  refused(b'records is not 16-byte aligned', records=L + 8)
  refused(b'records need', records_bytes=n_rec * rb - 1)                    # one record short
  refused(b'records need', records_bytes=(n_rec - 1) * rb)
  refused(b'overlap', roots=L + (n_rec - 1) * rb)                           # roots on the last record
  refused(b'overlap', records=R)                                            # the roots' own buffer
  refused(b'records overlaps status', outputs=_native.StepOut(out.reward, out.step_type, out.success,
                                                              L + (n_rec - 1) * rb))
  for n in (0, -1):
    refused(b'>= 1', n_steps=n)
    refused(b'>= 1', n_candidates=n)
    refused(b'n_roots', n_roots=n)
  refused(b'entries per call', n_roots=2 ** 30, n_candidates=2, n_steps=1)
  assert call(roots=L + n_rec * rb) == 0 and span.value == -5              # adjacent: accepted
  assert call(roots=None) == 0 and span.value == roots.span_class           # live roots: the engine's
  assert _snapshot(eng)[1] == before[1] + 2
  with pytest.raises(ValueError):
    eng.rollout(acts, leaves=True, trajectory=True)
  with pytest.raises(ValueError):                                           # E records short
    eng.rollout(acts, trajectory=engine.EnvStates(buf[:(n_rec - E) * rb].view(n_rec - E, rb), roots.span_class,
                                                  roots.signature, roots.n_slots))
  _assert_unchanged(eng, (before[0], before[1] + 2))
  eng.close()
