"""Env records on the device (swb_save_envs / swb_load_envs / swb_copy_envs), bit for bit.

A saved record replays its episode: stepped with the same actions, a loaded env reports what the
env it was saved from reported after the save, up to and including the episode's first LAST, and
so does the CPU oracle stepped from the decoded record (EnvStates.to_host) in its sqrt mode.  A
copy makes every destination what its source was before the call, also where the id sets
overlap.  Records move between engines of one configuration whatever their env count and pool,
and a record holding a star renders exactly in an engine that has only seen convex shapes.  Next
to the asynchronous refill, a loaded or copied env keeps its current pool entry: the refill
never writes it.  A refused call enqueues nothing.
"""
import ctypes

import numpy as np
import pytest
import torch

from oracle import oracle
from tests import fixtures

gpu = pytest.mark.gpu


def _oracle_from_records(h, action, nodes, keep, mel, rc):
  """BatchOracle whose envs are the decoded records `h`: a one-scene pool, live state restored."""
  from spriteworld_b200 import constants
  n, S = h['shape'].shape
  pool = np.zeros((n, 1, S), oracle.SPRITE_DTYPE)
  p = pool[:, 0]
  for f, g in (('x', 'x0'), ('y', 'y0'), ('m00', 'm00'), ('m01', 'm01'), ('m10', 'm10'),
               ('m11', 'm11'), ('vx', 'vx'), ('vy', 'vy'), ('member', 'member'), ('shape', 'shape'),
               ('pos_f32', 'pos_f32'), ('rgb', 'rgb')):
    p[f] = h[g]
  cfg = oracle.with_device_sqrt(fixtures.env_cfg_from_meta(dict(
      action=action, keep_in_frame=keep, max_episode_length=mel, nodes=nodes)))
  bo = oracle.BatchOracle(cfg, oracle.shape_table(constants.SHAPES), rc, pool)
  bo.cur['x'], bo.cur['y'] = h['pos_x'], h['pos_y']
  bo.step_count[:], bo.reset_next[:] = h['step_count'], h['reset_next']
  return bo


def _outputs(res, frames):
  return dict(reward=res.reward.cpu().numpy().copy(), step_type=res.step_type.cpu().numpy().copy(),
              success=res.success.cpu().numpy().copy(), status=res.status.cpu().numpy().copy(),
              frames=frames.cpu().numpy().copy())


def _run(eng, raster, acts):
  out = []
  for a in acts:
    frames = raster.new_frames()
    out.append(_outputs(eng.step(torch.from_numpy(np.ascontiguousarray(a)).to(eng.device), raster, frames),
                        frames))
  return out


def _live_mask(first_run):
  """(T, E): steps up to and including each env's first LAST, before any FIRST (a reset goes to the
  env's next ring scene, which is not part of the record)."""
  st = np.stack([o['step_type'] for o in first_run])
  done = np.cumsum(st == 2, 0) - (st == 2)          # LASTs strictly before step t
  started = np.cumsum(st == 0, 0) > 0
  return (done == 0) & ~started


def _compare(a, b, mask, what, nan_bits=True):
  for t in range(len(a)):
    m = mask[t]
    for k in ('step_type', 'success', 'status'):
      assert np.array_equal(a[t][k][m], b[t][k][m]), (what, k, t)
    ra, rb = a[t]['reward'][m], b[t]['reward'][m]
    if nan_bits:
      assert np.array_equal(ra.view(np.int64), rb.view(np.int64)), (what, 'reward', t)
    else:
      assert np.array_equal(ra, rb, equal_nan=True), (what, 'reward', t)
    ok = m & ((a[t]['status'] & 8) == 0)            # frames of envs whose spans fit
    assert np.array_equal(a[t]['frames'][ok], b[t]['frames'][ok]), (what, 'frames', t)


def _replay(eng, raster, acts, t0, action, nodes, keep, mel, rc):
  """Steps t0 actions, saves, steps the rest, loads, steps the rest again; checks the replay and
  the oracle stepped from the decoded records.  Returns the saved EnvStates, the live mask and
  the replay's outputs."""
  _run(eng, raster, acts[:t0])
  saved = eng.save_envs()
  first = _run(eng, raster, acts[t0:])
  eng.load_envs(saved)
  again = _run(eng, raster, acts[t0:])
  mask = _live_mask(first)
  _compare(first, again, mask, 'replay')
  h = saved.to_host()
  bo = _oracle_from_records(h, action, nodes, keep, mel, rc)
  ref = []
  for a in acts[t0:]:
    bo.step(a)
    ref.append(dict(reward=bo.reward.copy(), step_type=bo.step_type.copy(), success=bo.success.copy(),
                    status=bo.err.copy(), frames=bo.frames.copy()))
  for r, o in zip(ref, again):
    r['status'] = r['status'] | (o['status'] & 8)  # the oracle has no span limit
  _compare(again, ref, mask, 'oracle', nan_bits=False)
  # an env saved about to reset restarts: FIRST, on the next scene of its own ring
  resetting = h['reset_next'] == 1
  assert (again[0]['step_type'][resetting] == 0).all()
  return saved, mask, again


def _c2(n_envs, pool_depth, seed, mel=6):
  from spriteworld_b200 import workloads
  wl = workloads.GoalFinding()
  eng, raster, _ = workloads.build_engine(wl, n_envs, pool_depth, seed=seed, max_episode_length=mel)
  return wl, eng, raster


@gpu
def test_round_trip_is_the_identity():
  wl, eng, raster = _c2(300, 4, 1)
  acts = wl.sample_actions(np.random.RandomState(0), 5, eng.n_envs)
  _run(eng, raster, acts)
  before = eng.download_state()
  s = eng.save_envs()
  assert s.data.shape == (300, eng.record_bytes) and eng.record_bytes % 16 == 0
  eng.load_envs(s)
  again = eng.save_envs()
  assert torch.equal(again.data, s.data)
  after = eng.download_state()
  for k in before:
    assert np.array_equal(before[k], after[k]), k


@gpu
def test_replay_of_c2_matches_itself_and_the_oracle():
  wl, eng, raster = _c2(512, 4, 2, mel=10)          # saved 6 steps into a 10-step episode
  acts = wl.sample_actions(np.random.RandomState(1), 7 + 12, eng.n_envs)
  _, mask, _ = _replay(eng, raster, acts, 7, wl.action, wl.nodes, True, 10,
                       oracle.raster_cfg(64, 64, wl.anti_aliasing))
  assert 0 < mask[0].sum() and mask[-1].sum() < mask[0].sum()   # episodes ended inside the window


def _sweep_case(name):
  from tests import test_gpu_step_sweep as sweep
  return next(c for c in sweep.CASES if c['name'] == name)


# the step sweep's scenes and tasks: every action kind and dtype, filters, Clustering with both
# error statuses, MetaAggregated, mixed pos_f32, S = 1 .. 32, and records saved about to reset
FIELD_CASES = ['select_f32_s1_e1', 'select_f64_s2', 'drag_f32_s5_mixed', 'embodied_s7',
               'goal_filters', 'clustering_f32', 'meta_all_aggs', 'episode_len1']


def _sweep_engine(name):
  from spriteworld_b200 import engine
  from tests import test_gpu_step_sweep as sweep
  case = _sweep_case(name)
  arrs, nodes, action, acts = sweep._setup(case)
  rng = np.random.RandomState(5)
  shp = arrs['shape'].shape
  arrs['rgb'] = rng.randint(0, 256, shp + (3,)).astype(np.uint8)     # every field distinct
  arrs['c0'], arrs['c1'], arrs['c2'] = rng.rand(*shp), rng.rand(*shp), rng.rand(*shp)
  eng = sweep._engine(case, nodes, arrs, action)
  raster = engine.Raster(eng, 32, 32, 2)
  return case, nodes, action, acts, eng, raster


@gpu
@pytest.mark.parametrize('name', FIELD_CASES)
def test_every_field_replays_and_copies(name):
  case, nodes, action, acts, eng, raster = _sweep_engine(name)
  t0 = 3 if case['mel'] > 2 else 2
  saved, mask, again = _replay(eng, raster, acts, t0, action, nodes, case['keep'], case['mel'],
                               oracle.raster_cfg(32, 32, 2))
  h = saved.to_host()
  if name == 'episode_len1':
    assert h['reset_next'].any()
  # the statuses the case exists for show up inside the replayed window
  status = np.bitwise_or.reduce(np.stack([o['status'] for o in again])[mask])
  want = {'embodied_s7': 4, 'clustering_f32': 1 | 2}.get(name, 0)
  assert status & want == want
  _check_copy(eng, raster, np.arange(eng.n_envs), (np.arange(eng.n_envs) + 1) % eng.n_envs)


def _eval(eng):
  from spriteworld_b200 import _native
  _native.check(eng._lib.swb_eval_task(eng._h, ctypes.byref(eng._out), eng._stream()))
  return (eng._reward.cpu().numpy().copy(), eng._success.cpu().numpy().copy(),
          eng._status.cpu().numpy().copy())


def _check_copy(eng, raster, src, dst):
  """Copies src -> dst and checks each destination against its source before the call: record,
  frame, task reward, success and status."""
  rec = eng.save_envs().data.clone()
  frames = eng.render(raster).clone()
  r, s, st = _eval(eng)
  launches = eng.launch_count()
  eng.copy_envs(src, dst)
  overlap = len(np.intersect1d(src, dst)) > 0
  assert eng.launch_count() == launches + (2 if overlap else 1)
  rec2 = eng.save_envs().data
  assert torch.equal(rec2[torch.as_tensor(dst, device=eng.device).long()],
                     rec[torch.as_tensor(src, device=eng.device).long()])
  frames2 = eng.render(raster)
  assert torch.equal(frames2[torch.as_tensor(dst).long()], frames[torch.as_tensor(src).long()])
  r2, s2, st2 = _eval(eng)
  assert np.array_equal(r2[dst].view(np.int64), r[src].view(np.int64))
  assert np.array_equal(s2[dst], s[src]) and np.array_equal(st2[dst], st[src])
  rest = np.setdiff1d(np.arange(eng.n_envs), dst)
  assert torch.equal(rec2[torch.as_tensor(rest, device=eng.device).long()],
                     rec[torch.as_tensor(rest, device=eng.device).long()])


@gpu
def test_copy_with_overlap():
  wl, eng, raster = _c2(257, 3, 3)
  _run(eng, raster, wl.sample_actions(np.random.RandomState(2), 4, eng.n_envs))
  E = eng.n_envs
  _check_copy(eng, raster, np.arange(E), (np.arange(E) + 1) % E)
  rng = np.random.RandomState(3)
  dst = rng.choice(E, 60, replace=False)
  src = np.concatenate([dst[20:], rng.choice(E, 20)])
  _check_copy(eng, raster, src, dst)
  rest = np.setdiff1d(np.arange(E), np.concatenate([src, dst]))[:30]
  _check_copy(eng, raster, rest[:15], rest[15:])      # disjoint: one kernel


@gpu
def test_records_move_between_engines():
  """Records of engine A (stars and spokes among its shapes) loaded into engine B of another env
  count and pool depth that has only seen convex shapes: B renders them exactly, unflagged, and
  continues them as A does."""
  from spriteworld_b200 import engine as engine_lib
  from spriteworld_b200 import constants, workloads
  wl = workloads.GoalFinding()
  rng = np.random.RandomState(4)
  EA, KA, EB, KB = 96, 3, 200, 5
  scenes = wl.sample_scenes(rng, EA * KA)
  scenes['shape'][:] = rng.randint(1, 13, scenes['shape'].shape)
  mk = lambda E, K: engine_lib.Engine(E, wl.n_slots, K, wl.action, wl.nodes, constants.SHAPES,
                                      max_episode_length=6)
  A, B = mk(EA, KA), mk(EB, KB)
  A.upload_scenes(scenes, np.repeat(np.arange(EA), KA), np.tile(np.arange(KA), EA))
  B.upload_scenes(wl.sample_scenes(rng, EB * KB), np.repeat(np.arange(EB), KB), np.tile(np.arange(KB), EB))
  ra, rb = engine_lib.Raster(A, 64, 64, 5), engine_lib.Raster(B, 64, 64, 5)
  acts = wl.sample_actions(rng, 14, EB)
  _run(A, ra, acts[:4, :EA])
  _run(B, rb, acts[:4])
  saved = A.save_envs()
  assert saved.span_class == 4
  ids = rng.choice(EB, EA, replace=False)
  B.load_envs(saved, ids)
  assert torch.equal(B.save_envs(ids).data, saved.data)
  fa, fb = A.render(ra), B.render(rb)
  assert int(B.render_status().max().item()) == 0
  assert torch.equal(fb[torch.as_tensor(ids).long()], fa)
  outa = _run(A, ra, acts[4:, :EA])
  actb = acts[4:].copy()
  actb[:, ids] = acts[4:, :EA]
  outb = _run(B, rb, actb)
  mask = _live_mask(outa)
  for o in outb:
    for k in o:
      o[k] = o[k][ids]
  _compare(outa, outb, mask, 'across engines')
  assert all((o['status'] & 8 == 0).all() for o in outb)


@gpu
@pytest.mark.parametrize('refill', ['async', 'sync'])
def test_copies_every_step_next_to_the_refill(refill, monkeypatch):
  """max_episode_length 3, K = 6 and random copies after every step for 200 steps.

  A host mirror of the pool follows every upload.  After every step each env's record must hold
  the scene it should be on: the mirror's entry at its cursor if it started a scene this step,
  otherwise what it held after the last step and copy.  A refill writing the pool entry an env is
  on would break that.  Each frame must also be the oracle's render of the record.  With
  refill='sync' the outputs also equal the CPU double's, step for step."""
  import threading
  from spriteworld_b200 import constants
  from spriteworld_b200 import engine as engine_lib
  from tests import oracle_engine
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
  env = cpu._env(E=E, K=K, seed=8, max_episode_length=3, refill=refill)
  twin = None
  if refill == 'sync':
    with monkeypatch.context() as m:
      oracle_engine.install(m)
      m.setattr(engine_lib, 'Engine', cpu.StatesOracleEngine)
      twin = cpu._env(E=E, K=K, seed=8, max_episode_length=3, refill='sync')
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
    if twin is not None:
      tt = twin.step(a)
      for k in ('step_type', 'reward', 'success', 'status'):
        assert np.array_equal(getattr(ts, k).cpu().numpy(), getattr(tt, k).numpy()), (t, k)
      assert np.array_equal(frames, tt.observation['image'].numpy()), t
    n = rng.randint(1, E // 2)
    dst = rng.choice(E, n, replace=False)
    src = rng.choice(E, n)
    env.copy_envs(src, dst)
    for f in static:
      expect[f][dst] = expect[f][src]
    if twin is not None:
      twin.copy_envs(src, dst)
  assert env.refill_stats()['refills'] >= 5
  env.close()
  if twin is not None:
    twin.close()


@gpu
def test_refused_calls_enqueue_nothing():
  from spriteworld_b200 import _native
  from spriteworld_b200 import engine as engine_lib
  from spriteworld_b200 import constants, workloads
  wl, eng, raster = _c2(64, 3, 5)
  _run(eng, raster, wl.sample_actions(np.random.RandomState(6), 3, eng.n_envs))
  s = eng.save_envs()
  torch.cuda.synchronize()
  launches = eng.launch_count()
  L, h, rb = eng._lib, eng._h, eng.record_bytes
  ids = np.arange(4, dtype=np.int32)
  p = lambda a: ctypes.c_void_p(a.ctypes.data)
  refused = [
      lambda: eng.save_envs([0, 64]),
      lambda: eng.save_envs([-1]),
      lambda: eng.load_envs(s[:2], [3, 3]),
      lambda: eng.load_envs(s[:2], [0, 64]),
      lambda: eng.copy_envs([0, 1], [2, 2]),
      lambda: eng.copy_envs([0, 99], [1, 2]),
      lambda: _native.check(L.swb_save_envs(h, p(ids), 4, ctypes.c_void_p(s.data.data_ptr()), 4 * rb - 1,
                                            ctypes.byref(ctypes.c_int32()), eng._stream())),
      lambda: _native.check(L.swb_load_envs(h, p(ids), 4, ctypes.c_void_p(s.data.data_ptr()), 3 * rb, 1,
                                            eng._stream())),
      lambda: _native.check(L.swb_load_envs(h, p(ids), 4, ctypes.c_void_p(s.data.data_ptr()), 4 * rb, 2,
                                            eng._stream())),
      lambda: _native.check(L.swb_copy_envs(h, None, p(ids), 4, eng._stream())),
      lambda: _native.check(L.swb_save_envs(h, p(ids), 4, ctypes.c_void_p(s.data.data_ptr() + 8), 4 * rb,
                                            ctypes.byref(ctypes.c_int32()), eng._stream())),
      lambda: _native.check(L.swb_load_envs(h, p(ids), 4, ctypes.c_void_p(s.data.data_ptr() + 8), 4 * rb, 1,
                                            eng._stream())),
  ]
  for i, call in enumerate(refused):
    with pytest.raises(_native.NativeError):
      call()
    assert eng.launch_count() == launches, i
  # records at an address the kernels cannot read f64 fields from
  shifted = torch.zeros(4 * rb + 8, dtype=torch.uint8, device=eng.device)[8:].view(4, rb)
  with pytest.raises(ValueError, match='aligned'):
    eng.load_envs(engine_lib.EnvStates(shifted, s.span_class, s.signature, s.n_slots), ids)
  assert eng.launch_count() == launches
  other = engine_lib.Engine(8, wl.n_slots, 3, wl.action, wl.nodes, constants.SHAPES,
                            max_episode_length=7)
  with pytest.raises(ValueError, match='another configuration'):
    other.load_envs(s[:8])
  assert other.launch_count() == 0
  assert torch.equal(eng.save_envs().data, s.data)
  # n == 0: nothing to do, no launch
  eng.copy_envs([], [])
  eng.load_envs(s[:0], [])
  assert len(eng.save_envs([])) == 0
  assert eng.launch_count() == launches + 1


@gpu
def test_a_shape_id_without_a_vertex_table_loads_as_an_empty_slot():
  """Records not written by swb_save_envs: an out-of-range shape id never reaches the shape table."""
  from spriteworld_b200 import engine as engine_lib
  wl, eng, raster = _c2(16, 3, 7)
  _run(eng, raster, wl.sample_actions(np.random.RandomState(8), 2, eng.n_envs))
  s = eng.save_envs()
  layout = {name: off for name, off, _, _ in engine_lib.record_layout(eng.n_slots)[0]}
  bad = s.data.clone()
  bad[:, layout['shape']] = 200
  bad[:, layout['shape'] + 1] = 13
  eng.load_envs(engine_lib.EnvStates(bad, s.span_class, s.signature, s.n_slots))
  h, h0 = eng.save_envs().to_host(), s.to_host()
  assert (h['shape'][:, :2] == 0).all()
  assert np.array_equal(h['shape'][:, 2:], h0['shape'][:, 2:])
  cleared = s.to_host()
  cleared['shape'][:, :2] = 0
  rec = np.zeros((eng.n_envs, eng.n_slots), oracle.SPRITE_DTYPE)
  for f, g in (('x', 'pos_x'), ('y', 'pos_y'), ('m00', 'm00'), ('m01', 'm01'), ('m10', 'm10'),
               ('m11', 'm11'), ('shape', 'shape'), ('rgb', 'rgb')):
    rec[f] = cleared[g]
  from spriteworld_b200 import constants
  tab, rc = oracle.shape_table(constants.SHAPES), oracle.raster_cfg(64, 64, 5)
  frames = eng.render(raster).cpu().numpy()
  for e in range(eng.n_envs):
    assert np.array_equal(frames[e], oracle.render(rc, tab, rec[e]))
