"""Env records with device-checked id lists (check='device'), bit for bit.

A device-checked save, load or copy computes what the host-checked one computes, for int32 and
int64 ids, and the host does not wait for the ids.  Ids the device refuses -- out of range, in
the id type's own width, or a repeated destination -- change nothing, a refused save returns zero
records, Engine.check_env_ids() names the lowest failing position, and the next call runs
normally.  Host-visible faults (dtype, device, shape, counts, span class) are refused before
anything is enqueued.  Next to the asynchronous refill a device-checked resample keeps every env
on its own pool entry, and factor observations follow an accepted call and ignore a refused one.
"""
import re

import numpy as np
import pytest
import torch

from oracle import oracle

gpu = pytest.mark.gpu

ID_DTYPES = {'int32': torch.int32, 'int64': torch.int64}


def _c2(seed=1, n_envs=None, mel=6):
  from spriteworld_b200 import workloads
  wl = workloads.WORKLOADS['c2']()
  eng, raster, _ = workloads.build_engine(wl, n_envs or wl.n_envs, 4, seed=seed, max_episode_length=mel)
  return wl, eng, raster


def _step(eng, raster, acts):
  out = []
  for a in acts:
    frames = raster.new_frames()
    res = eng.step(torch.from_numpy(np.ascontiguousarray(a)).to(eng.device), raster, frames)
    out.append(dict(reward=res.reward.cpu().numpy().view(np.int64).copy(),
                    step_type=res.step_type.cpu().numpy().copy(), success=res.success.cpu().numpy().copy(),
                    status=res.status.cpu().numpy().copy(), frames=frames.cpu().numpy().copy()))
  return out


def _dev(ids, eng, dtype):
  return torch.as_tensor(np.asarray(ids), device=eng.device).to(dtype)


@gpu
@pytest.mark.parametrize('id_dtype', sorted(ID_DTYPES))
def test_device_checked_calls_compute_what_host_checked_calls_compute(id_dtype):
  """Two C2 engines built alike: every call host-checked on A, device-checked on B; then both
  states step alike, outputs and frames bit for bit."""
  wl, A, ra = _c2(seed=11)
  _, B, rb = _c2(seed=11)
  E, dt = A.n_envs, ID_DTYPES[id_dtype]
  acts = wl.sample_actions(np.random.RandomState(3), 12, E)
  assert all(np.array_equal(x[k], y[k]) for x, y in zip(_step(A, ra, acts[:4]), _step(B, rb, acts[:4]))
             for k in x)
  rng = np.random.RandomState(4)
  gen = torch.Generator(device=B.device)
  gen.manual_seed(5)

  def same(what):
    assert torch.equal(A.save_envs().data, B.save_envs().data), what

  same('start')
  for what, ids in (('save with repeats', rng.randint(0, E, 777)), ('save permutation', rng.permutation(E))):
    sa, sb = A.save_envs(ids), B.save_envs(_dev(ids, B, dt), check='device')
    assert torch.equal(sa.data, sb.data) and sa.span_class == sb.span_class, what
  recs = A.save_envs(rng.randint(0, E, 1000))
  dst = rng.choice(E, 1000, replace=False)
  A.load_envs(recs, dst)
  B.load_envs(recs, _dev(dst, B, dt), check='device')
  same('load')
  half = E // 2
  sub = rng.choice(E, 300, replace=False)
  copies = [
      ('sources with repeats, disjoint', rng.randint(0, half, 500), half + rng.choice(half, 500, replace=False)),
      ('overlapping', np.concatenate([sub[100:], rng.randint(0, E, 100)]), sub),
      ('disjoint', np.arange(0, 200), np.arange(E - 200, E)),
      ('permutation', np.arange(E), rng.permutation(E)),
      ('shift by one', np.arange(E), np.roll(np.arange(E), 1)),
  ]
  for what, src, dst in copies:
    A.copy_envs(src, dst)
    B.copy_envs(_dev(src, B, dt), _dev(dst, B, dt), check='device')
    same(what)
  # resampling: every env replaced by a draw, with replacement, from weights on the device
  src = torch.multinomial(torch.rand(E, device=B.device, generator=gen), E, replacement=True,
                          generator=gen).to(dt)
  dst = torch.arange(E, device=B.device, dtype=dt)
  B.copy_envs(src, dst, check='device')
  A.copy_envs(src.cpu().numpy(), np.arange(E))
  same('multinomial resample')
  B.check_env_ids()
  outa, outb = _step(A, ra, acts[4:]), _step(B, rb, acts[4:])
  for t, (x, y) in enumerate(zip(outa, outb)):
    for k in x:
      assert np.array_equal(x[k], y[k]), (t, k)


@gpu
def test_device_checked_calls_do_not_wait_for_the_device():
  wl, eng, raster = _c2(seed=2, n_envs=1024)
  E = eng.n_envs
  ids = torch.arange(E, device=eng.device)
  shifted = torch.roll(ids, 1)
  s = eng.save_envs(ids, check='device')
  eng.copy_envs(ids, shifted, check='device')        # engine scratch grows here, once
  torch.cuda.synchronize()
  launches = eng.launch_count()
  torch.cuda._sleep(1 << 31)                          # about a second of device time
  s2 = eng.save_envs(ids, check='device')
  eng.load_envs(s, shifted, check='device')
  eng.copy_envs(shifted, ids, check='device')
  done = torch.cuda.Event()
  done.record()
  assert not done.query()
  assert eng.launch_count() == launches + 2 + 3 + 3
  torch.cuda.synchronize()
  eng.check_env_ids()
  assert len(s2) == E


@gpu
def test_batched_environment_forms_do_not_synchronise():
  from tests import test_env_states_on_oracle as cpu
  env = cpu._env(E=48, K=5, seed=9, refill='sync', factors=True)
  rng = np.random.RandomState(1)
  for _ in range(3):
    env.step(rng.uniform(0, 1, (env.n_envs, 4)).astype(np.float32))
  dev = env.engine.device
  ids = torch.arange(env.n_envs, device=dev)
  bad = torch.tensor([-1, 0], device=dev)     # (a host-to-device copy: made before the mode is set)
  torch.cuda.synchronize()
  prev = torch.cuda.get_sync_debug_mode()
  torch.cuda.set_sync_debug_mode('error')
  try:
    s = env.save_envs(ids, check='device')
    env.load_envs(s, torch.flip(ids, (0,)), check='device')
    env.copy_envs(ids[:10].int(), ids[20:30], check='device')
    env.copy_envs(bad, ids[:2], check='device')    # refused
  finally:
    torch.cuda.set_sync_debug_mode(prev)
  with pytest.raises(ValueError, match=re.escape('copy_envs: src_ids[0] = -1')):
    env.engine.check_env_ids()
  env.close()


def _refusal_cases(E):
  """(name, call, id dtype, ids..., expected message prefix).  Every case fails at two positions;
  the lower one is reported."""
  ids = np.random.RandomState(7).choice(E, 16, replace=False).astype(np.int64)

  def bad(v, at=(5, 9)):
    a = ids.copy()
    a[list(at)] = v
    return a

  rep = ids.copy()
  rep[9], rep[12] = rep[5], rep[2]           # positions 9 and 12 repeat lower ones: 9 is reported
  return [
      ('save -1', 'save', 'int32', bad(-1), 'save_envs: env_ids[5] = -1 is out of range'),
      ('save E', 'save', 'int64', bad(E), 'save_envs: env_ids[5] = %d is out of range' % E),
      ('save 2**32+1', 'save', 'int64', bad(2 ** 32 + 1), 'save_envs: env_ids[5] = 4294967297 is out'),
      ('load E', 'load', 'int32', bad(E), 'load_envs: env_ids[5] = %d is out' % E),
      ('load 2**31', 'load', 'int64', bad(2 ** 31), 'load_envs: env_ids[5] = 2147483648 is out'),
      ('load 2**32+1', 'load', 'int64', bad(2 ** 32 + 1), 'load_envs: env_ids[5] = 4294967297 is out'),
      ('load repeat', 'load', 'int32', rep, 'load_envs: env_ids[9] = %d repeats a destination' % ids[5]),
      ('copy src -1', 'copy_src', 'int32', bad(-1), 'copy_envs: src_ids[5] = -1 is out'),
      ('copy dst E', 'copy_dst', 'int64', bad(E), 'copy_envs: dst_ids[5] = %d is out' % E),
      ('copy src 2**32+1', 'copy_src', 'int64', bad(2 ** 32 + 1), 'copy_envs: src_ids[5] = 4294967297 is'),
      ('copy repeat', 'copy_dst', 'int64', rep, 'copy_envs: dst_ids[9] = %d repeats a destination' % ids[5]),
  ], ids


@gpu
def test_refused_ids_change_nothing_and_are_reported():
  wl, eng, raster = _c2(seed=3, n_envs=256)
  E = eng.n_envs
  _step(eng, raster, wl.sample_actions(np.random.RandomState(2), 3, E))
  cases, good = _refusal_cases(E)
  src_ok = np.random.RandomState(8).randint(0, E, len(good))
  recs = eng.save_envs(src_ok)
  for name, call, id_dtype, ids, msg in cases:
    dt = ID_DTYPES[id_dtype]
    before = eng.save_envs().data.clone()
    frames = eng.render(raster).clone()
    t = torch.as_tensor(ids, device=eng.device).to(dt) if dt == torch.int64 else \
        torch.as_tensor(ids.astype(np.int32), device=eng.device)
    if call == 'save':
      out = eng.save_envs(t, check='device')
      assert len(out) == len(ids) and not out.data.any(), name
    elif call == 'load':
      eng.load_envs(recs, t, check='device')
    elif call == 'copy_src':
      eng.copy_envs(t, _dev(good, eng, dt), check='device')
    else:
      eng.copy_envs(_dev(src_ok, eng, dt), t, check='device')
    assert torch.equal(eng.save_envs().data, before), name
    assert torch.equal(eng.render(raster), frames), name
    with pytest.raises(ValueError, match=re.escape(msg)):
      eng.check_env_ids()
    eng.check_env_ids()                                 # cleared
    # the next call runs normally
    eng.copy_envs(_dev(src_ok, eng, dt), _dev(good, eng, dt), check='device')
    after = eng.save_envs().data
    g = torch.as_tensor(good, device=eng.device)
    assert torch.equal(after[g], before[torch.as_tensor(src_ok, device=eng.device)]), name
    eng.check_env_ids()
    eng.load_envs(engine_states(eng, before), check='host')
  # the first refused call since the last check is the one reported
  bad = torch.tensor([0, E], device=eng.device)
  eng.save_envs(bad, check='device')
  eng.load_envs(recs[:2], torch.tensor([3, 3], device=eng.device), check='device')
  with pytest.raises(ValueError, match=re.escape('save_envs: env_ids[1] = %d' % E)):
    eng.check_env_ids()
  eng.check_env_ids()


def engine_states(eng, data):
  from spriteworld_b200 import engine as engine_lib
  return engine_lib.EnvStates(data, 1, eng.signature, eng.n_slots)


@gpu
def test_claims_do_not_leak_into_the_next_call():
  """A destination of call k is a fresh destination in call k + 1, whatever the calls between."""
  wl, eng, raster = _c2(seed=4, n_envs=128)
  _step(eng, raster, wl.sample_actions(np.random.RandomState(3), 2, eng.n_envs))
  dev = eng.device
  dst = torch.tensor([7, 9, 11], device=dev)
  for k in range(4):
    before = eng.save_envs().data.clone()
    src = torch.tensor([k, k + 20, k + 40], device=dev)
    if k % 2:
      eng.copy_envs(src, dst, check='device')
    else:
      eng.load_envs(eng.save_envs(src), dst.int(), check='device')
    eng.check_env_ids()
    assert torch.equal(eng.save_envs().data[dst], before[src]), k
  eng.save_envs(torch.tensor([1, 1, 1], device=dev), check='device')   # repeats are fine in a save
  eng.check_env_ids()


@gpu
def test_host_visible_faults_are_refused_before_anything_is_enqueued():
  from spriteworld_b200 import _native
  from spriteworld_b200 import engine as engine_lib
  wl, eng, raster = _c2(seed=5, n_envs=64)
  E, dev = eng.n_envs, eng.device
  s = eng.save_envs(np.arange(4))
  torch.cuda.synchronize()
  launches = eng.launch_count()
  ok = torch.arange(4, device=dev)
  wrong = [torch.arange(4, device=dev, dtype=torch.float32), torch.arange(4, device=dev, dtype=torch.uint8),
           torch.arange(4), torch.empty(4, dtype=torch.int64, device='meta'), ok.reshape(2, 2),
           np.arange(4), [0, 1, 2, 3]]
  if torch.cuda.device_count() > 1:
    wrong.append(torch.arange(4, device='cuda:1'))
  for w in wrong:
    for call in (lambda: eng.save_envs(w, check='device'), lambda: eng.load_envs(s, w, check='device'),
                 lambda: eng.copy_envs(w, ok, check='device'), lambda: eng.copy_envs(ok, w, check='device')):
      with pytest.raises(ValueError, match="check='device'"):
        call()
  refused = [
      (ValueError, lambda: eng.load_envs(s, ok[:3], check='device')),                # count
      (ValueError, lambda: eng.copy_envs(ok, ok[:3], check='device')),
      (ValueError, lambda: eng.save_envs(ok, check='gpu')),
      (_native.NativeError, lambda: eng.load_envs(engine_lib.EnvStates(s.data, 2, s.signature, s.n_slots), ok,
                                                  check='device')),                # span class
      # the C-ABI's own checks: a host pointer, an id dtype, a short buffer
      (_native.NativeError, lambda: _native.check(eng._lib.swb_copy_envs_dev(
          eng._h, ok.cpu().numpy().ctypes.data, ok.data_ptr(), _native.DTYPE_I64, 4, eng._stream()))),
      (_native.NativeError, lambda: _native.check(eng._lib.swb_load_envs_dev(
          eng._h, ok.data_ptr(), _native.DTYPE_F32, 4, s.data.data_ptr(), s.data.numel(), 1, eng._stream()))),
      (_native.NativeError, lambda: _native.check(eng._lib.swb_load_envs_dev(
          eng._h, ok.data_ptr(), _native.DTYPE_I64, 4, s.data.data_ptr(), s.data.numel() - 1, 1,
          eng._stream()))),
  ]
  for i, (exc, call) in enumerate(refused):
    with pytest.raises(exc):
      call()
    assert eng.launch_count() == launches, i
  # n == 0 launches nothing
  none = torch.empty(0, dtype=torch.int64, device=dev)
  assert len(eng.save_envs(none, check='device')) == 0
  eng.load_envs(s[:0], none, check='device')
  eng.copy_envs(none, none, check='device')
  assert eng.launch_count() == launches
  eng.check_env_ids()


@gpu
def test_device_resampling_every_step_next_to_the_refill(monkeypatch):
  """test_gpu_env_states.test_copies_every_step_next_to_the_refill with the asynchronous refill and
  ids drawn on the device: after every step a device-checked resample, and each env's record
  checked against the host mirror of the pool and each frame against the oracle's render."""
  import threading
  from spriteworld_b200 import constants
  from spriteworld_b200 import engine as engine_lib
  from tests import test_env_states_on_oracle as cpu
  E, K, T = 32, 6, 200
  static = {'x0': 'x', 'y0': 'y', 'm00': 'm00', 'm01': 'm01', 'm10': 'm10', 'm11': 'm11',
            'vx': 'vx', 'vy': 'vy', 'member': 'member', 'shape': 'shape', 'pos_f32': 'pos_f32',
            'rgb': 'rgb', 'factors': 'factors'}
  mirror, lock = {}, threading.Lock()
  pushed = engine_lib.Engine.upload_scenes

  def upload(self, scenes, env_ids, ring_slots):
    with lock:
      for f, g in static.items():
        a = np.asarray(scenes[g])
        if f not in mirror:
          mirror[f] = np.zeros((self.n_envs, K) + a.shape[1:], a.dtype)
        mirror[f][np.asarray(env_ids), np.asarray(ring_slots)] = a
    return pushed(self, scenes, env_ids, ring_slots)

  monkeypatch.setattr(engine_lib.Engine, 'upload_scenes', upload)
  env = cpu._env(E=E, K=K, seed=8, max_episode_length=3, refill='async')
  dev = env.engine.device
  gen = torch.Generator(device=dev)
  gen.manual_seed(13)
  tab, rc = oracle.shape_table(constants.SHAPES), oracle.raster_cfg(64, 64, 5)
  rng = np.random.RandomState(12)
  h = env.save_envs().to_host()
  expect = {f: h[f].copy() for f in static}
  rows = np.arange(E)
  for t in range(T):
    a = rng.uniform(0, 1, (E, 4)).astype(np.float32)
    ts = env.step(a)
    frames = ts.observation['image'].cpu().numpy()
    first = ts.step_type.cpu().numpy() == 0
    h = env.save_envs().to_host()
    cursor = env.engine.download_state()['cursor'].astype(np.int64)
    with lock:
      for f in static:
        expect[f][first] = mirror[f][rows, cursor][first]
    for f in static:
      assert np.array_equal(h[f], expect[f]), (t, f)
    for e in range(E):
      rec = np.zeros(env.engine.n_slots, oracle.SPRITE_DTYPE)
      for f, g in (('x', 'pos_x'), ('y', 'pos_y'), ('m00', 'm00'), ('m01', 'm01'), ('m10', 'm10'),
                   ('m11', 'm11'), ('shape', 'shape'), ('rgb', 'rgb')):
        rec[f] = h[g][e]
      assert np.array_equal(frames[e], oracle.render(rc, tab, rec)), (t, e)
    n = int(rng.randint(1, E))
    weights = torch.rand(E, device=dev, generator=gen)
    src = torch.multinomial(weights, n, replacement=True, generator=gen)
    dst = torch.randperm(E, device=dev, generator=gen)[:n]
    env.copy_envs(src, dst.int() if t % 2 else dst, check='device')
    s, d = src.cpu().numpy(), dst.cpu().numpy()       # bookkeeping, after the call
    for f in static:
      expect[f][d] = expect[f][s]
  env.engine.check_env_ids()
  assert env.refill_stats()['refills'] >= 5
  env.close()


FACTORS = ('x', 'y', 'shape', 'angle', 'scale', 'c0', 'c1', 'c2', 'x_vel', 'y_vel')


@gpu
def test_factor_observations_follow_device_checked_calls():
  from tests import test_env_states_on_oracle as cpu
  A = cpu._env(E=40, K=5, seed=6, refill='sync', factors=True)
  B = cpu._env(E=40, K=5, seed=6, refill='sync', factors=True)
  E, dev = A.n_envs, B.engine.device
  rng = np.random.RandomState(2)

  def step_both():
    a = rng.uniform(0, 1, (E, 4)).astype(np.float32)
    A.step(a)
    B.step(a)

  def factors(env):
    return {k: v.clone() for k, v in env.factor_tensors(FACTORS).items()}

  def same(what):
    fa, fb = factors(A), factors(B)
    for k in fa:
      assert torch.equal(fa[k], fb[k]), (what, k)

  for _ in range(3):
    step_both()
  same('start')
  ids = rng.choice(E, 12, replace=False)
  recs = A.save_envs(rng.randint(0, E, 12))
  A.load_envs(recs, ids)
  B.load_envs(recs, torch.as_tensor(ids, device=dev), check='device')
  same('load')
  src, dst = rng.randint(0, E, 15), rng.choice(E, 15, replace=False)
  A.copy_envs(src, dst)
  B.copy_envs(torch.as_tensor(src, device=dev).int(), torch.as_tensor(dst, device=dev).int(), check='device')
  same('copy')
  step_both()
  same('step')
  # refused calls: factors unchanged, no device assert
  before = factors(B)
  big = torch.tensor([0, 2 ** 32 + 1, 3], device=dev)
  B.copy_envs(big, torch.tensor([5, 6, 7], device=dev), check='device')
  B.copy_envs(torch.tensor([1, 2, 3], device=dev), torch.tensor([E, -7, 4], device=dev), check='device')
  B.load_envs(recs[:3], torch.tensor([8, 8, 9], device=dev), check='device')
  torch.cuda.synchronize()
  after = factors(B)
  for k in before:
    assert torch.equal(before[k], after[k]), k
  with pytest.raises(ValueError, match=re.escape('copy_envs: src_ids[1] = 4294967297')):
    B.engine.check_env_ids()
  A.close()
  B.close()
