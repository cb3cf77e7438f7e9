"""Whole-run checkpoints on the GPU: the engine checkpoint of the C-ABI (swb_save_engine /
swb_load_engine) and BatchedEnvironment.state_dict / load_state_dict built on it.

A run resumed from a checkpoint in a fresh environment (another rng, and for the device sampler
another seed, which the load replaces) must give, bit for bit, what the uninterrupted run gave --
every raster's frames, reward, step type, discount, success, status and factor observations -- for
at least three episodes per env after the checkpoint, with the device sampler and with the host
sampler's sync refill; with the async refill, up to the scenes the rings held at the checkpoint.
render(), rollout(), expand() and observe() after a load equal their results before the save.  The
C-ABI's saves are byte-identical and read-only, and every corrupt buffer is refused, naming its
field, with nothing enqueued.
"""
import collections
import ctypes
import io
import os

import numpy as np
import pytest
import torch

from spriteworld_b200 import _native, constants, environment, renderers
from spriteworld_b200 import engine as engine_lib
from spriteworld_b200.configs.cobra import clustering, goal_finding_more_targets, sorting

pytestmark = pytest.mark.gpu

FACTORS = ('x', 'y', 'shape', 'angle', 'scale', 'c0', 'x_vel')


def _cfg(name, two_rasters, max_episode_length):
  mod = dict(goal=goal_finding_more_targets, clustering=clustering, sorting=sorting)[name]
  cfg = dict(mod.get_config('train'))
  cfg.pop('metadata', None)
  cfg['max_episode_length'] = max_episode_length
  rs = collections.OrderedDict(cfg['renderers'])
  if two_rasters:
    rs['small'] = renderers.PILRenderer(image_size=(40, 24), anti_aliasing=3, bg_color=(20, 40, 60),
                                        color_to_rgb=rs['image'].color_to_rgb)
  rs['factors'] = renderers.SpriteFactors(FACTORS)
  cfg['renderers'] = rs
  return cfg


def _env(name='goal', n_envs=1024, sampler='device', refill=None, rng_seed=0, seed=5, two_rasters=False,
         max_episode_length=5, pool_depth=6, **kw):
  extra = dict(seed=seed) if sampler == 'device' else dict(refill=refill, refill_threads=4)
  return environment.BatchedEnvironment(n_envs=n_envs, pool_depth=pool_depth, sampler=sampler,
                                        rng=np.random.RandomState(rng_seed),
                                        **dict(_cfg(name, two_rasters, max_episode_length), **extra, **kw))


def _outputs(ts):
  out = dict(step_type=ts.step_type, reward=ts.reward, discount=ts.discount, success=ts.success,
             status=ts.status)
  for name, obs in ts.observation.items():
    if isinstance(obs, dict):
      out.update(('%s.%s' % (name, k), v) for k, v in obs.items())
    else:
      out[name] = obs
  return {k: v.cpu().numpy().copy() for k, v in out.items()}


def _actions(rng, T, E):
  return torch.from_numpy(rng.uniform(0, 1, (T, E, 4)).astype(np.float32)).cuda()


def _run(env, actions):
  return [_outputs(env.step(a)) for a in actions]


def _same(want, got, mask=None):
  assert len(want) == len(got)
  for t, (w, g) in enumerate(zip(want, got)):
    m = slice(None) if mask is None else mask[t]
    for k in w:
      assert np.array_equal(w[k][m], g[k][m], equal_nan=True), (t, k)


def _observed(env, plans):
  """What the env shows of its state without stepping: every raster's frames, the factor
  observations, the decoded records, a rollout, an expand and an observe of the records."""
  out = {'render.' + k: v.cpu().numpy().copy() for k, v in env.render().items()}
  out.update(('factors.' + k, v.cpu().numpy().copy()) for k, v in env.factor_tensors(FACTORS).items())
  states = env.save_envs()
  out.update(('record.' + k, v) for k, v in states.to_host().items())
  out.update(('rollout.' + k, v.cpu().numpy().copy()) for k, v in env.rollout(plans)._asdict().items())
  res, leaves = env.expand(plans)
  out.update(('expand.' + k, v.cpu().numpy().copy()) for k, v in res._asdict().items())
  out['expand.leaves'] = leaves.data.cpu().numpy().copy()
  obs, status = env.observe(leaves)
  out['observe.status'] = status.cpu().numpy().copy()
  for name, o in obs.items():
    items = o.items() if isinstance(o, dict) else [('', o)]
    out.update(('observe.%s.%s' % (name, k), v.cpu().numpy().copy()) for k, v in items)
  return out


def _same_observed(a, b):
  assert set(a) == set(b)
  for k in a:
    assert np.array_equal(a[k], b[k], equal_nan=True), k


CASES = [('goal', 'device', None, False), ('goal', 'host', 'sync', False),
         ('clustering', 'device', None, True), ('sorting', 'host', 'sync', True)]


@pytest.mark.parametrize('name,sampler,refill,two_rasters', CASES)
def test_resume_is_bit_exact_for_three_episodes_per_env(name, sampler, refill, two_rasters):
  E = 1024 if name == 'goal' else 256
  n0, n1 = 9, 24                     # episodes of at most 5 steps + the FIRST step
  rng = np.random.RandomState(3)
  acts = _actions(rng, n0 + n1, E)
  plans = _actions(rng, 4 * 3, E).reshape(4, E, 3, 4)
  a = _env(name, E, sampler, refill, two_rasters=two_rasters)
  a._action_space._noise_scale = 0.05          # noise draws from rng are part of the run
  a.reset()
  _run(a, acts[:n0])
  assert (a.engine.download_state()['step_count'] > 0).any()
  sd = a.state_dict()
  before = _observed(a, plans)
  want = _run(a, acts[n0:])
  firsts = np.sum([w['step_type'] == 0 for w in want], axis=0)
  assert firsts.min() >= 3, firsts.min()          # every env started three more episodes

  buf = io.BytesIO()
  torch.save(sd, buf)
  buf.seek(0)
  b = _env(name, E, sampler, refill, rng_seed=99, seed=6, two_rasters=two_rasters)
  b._action_space._noise_scale = 0.05
  b.reset()
  _run(b, acts[:2])
  b.load_state_dict(torch.load(buf))
  if sampler == 'device':
    assert b.seed == a.seed
  _same_observed(before, _observed(b, plans))
  _same(want, _run(b, acts[n0:]))

  a.load_state_dict(sd)                            # rewind
  _same(want, _run(a, acts[n0:]))
  a.close(); b.close()


def _until_in_flight(env, acts):
  """Steps until the async refill has a job in flight; returns the steps taken."""
  for t in range(len(acts)):
    if env._inflight is not None and not env._inflight['future'].done():
      return t
    env.step(acts[t])
  return len(acts)


def test_async_resume_is_bit_exact_up_to_the_saved_horizon():
  E, K = 512, 8
  rng = np.random.RandomState(4)
  n0, n1 = 12, 30
  acts = _actions(rng, n0 + 40 + n1, E)
  a = _env('goal', E, 'host', 'async', pool_depth=K, max_episode_length=4)
  a.reset()
  _run(a, acts[:n0])
  t0 = n0 + _until_in_flight(a, acts[n0:n0 + 40])
  in_flight = a._inflight is not None
  sd = a.state_dict()                              # lands the refill in flight
  assert a._inflight is None
  horizon = sd['host']['refilled_upto'].numpy()
  cont = acts[t0:t0 + n1]
  want, serial = [], []
  for x in cont:
    want.append(_outputs(a.step(x)))
    serial.append(a.engine.download_state_serial())
  mask = [s <= horizon for s in serial]            # envs still on scenes their ring held
  assert mask[0].all()
  crossed = sum(int(((w['step_type'] == 0) & m).sum()) for w, m in zip(want, mask))
  assert crossed >= E // 2                         # episode boundaries inside the horizon

  b = _env('goal', E, 'host', 'async', rng_seed=42, pool_depth=K, max_episode_length=4)
  b.reset()
  _until_in_flight(b, acts[:40])
  b_in_flight = b._inflight is not None
  b.load_state_dict(sd)                            # lands b's own refill first
  _same(want, _run(b, cont), mask)
  assert in_flight and b_in_flight                 # both paths were exercised
  a.close(); b.close()


def _stars_engine(E=16, K=2, spans_star=True, seed=1):
  from spriteworld_b200 import scene
  rng = np.random.RandomState(seed)
  S = 6
  eng = engine_lib.Engine(E, S, K, dict(kind='select_move', scale=0.5), [dict(kind='no_reward')],
                          constants.SHAPES, keep_in_frame=False)
  n = E * K
  z = np.zeros((n, S))
  shapes = rng.randint(7, 13, (n, S)) if spans_star else rng.randint(1, 7, (n, S))
  b = scene.batch_from_factor_arrays(
      rng.uniform(0.1, 0.9, (n, S)), rng.uniform(0.1, 0.9, (n, S)), np.zeros((n, S), np.uint8), shapes,
      rng.randint(0, 360, (n, S)), rng.uniform(0.1, 0.4, (n, S)), z, z, z, z, z, np.zeros((n, S), np.uint32),
      rng.randint(0, 256, (n, S, 3)))
  eng.upload_scenes(b, np.repeat(np.arange(E), K), np.tile(np.arange(K), E))
  eng.upload_state(pos_x=b['x'][::K], pos_y=b['y'][::K], cursor=np.zeros(E), step_count=np.zeros(E),
                   reset_next=np.zeros(E))
  return eng


def test_span_class_travels_with_the_checkpoint():
  a = _stars_engine(spans_star=True)
  ra = engine_lib.Raster(a, 64, 64, 5)
  a.step(torch.full((a.n_envs, 4), 0.6, device='cuda'))
  want, want_status = a.render(ra).cpu().numpy(), a.render_status().cpu().numpy().copy()
  state = a.save_state()
  assert int.from_bytes(state[24:28].numpy().tobytes(), 'little') == 4
  b = _stars_engine(spans_star=False, seed=2)     # convex only: span class 1
  assert b.save_envs([0]).span_class == 1
  rb = engine_lib.Raster(b, 64, 64, 5)
  b.load_state(state)
  assert b.save_envs([0]).span_class == 4
  assert np.array_equal(b.render(rb).cpu().numpy(), want)
  assert np.array_equal(b.render_status().cpu().numpy(), want_status)
  ra.close(); rb.close(); a.close(); b.close()


def _layout(E, K, S):
  """Offsets of the checkpoint fields, restated from the table of include/spriteworld_b200.h."""
  a16 = lambda n: (n + 15) // 16 * 16
  off, o = {}, a16(56 + ctypes.sizeof(_native.Config))
  ES, EKS = E * S, E * K * S
  for name, nbytes in ([('pos_x', 8 * ES), ('pos_y', 8 * ES), ('cursor', 4 * E), ('step_count', 4 * E),
                        ('scene_serial', 4 * E), ('reset_next', E)] +
                       [(f, 8 * EKS) for f in ('x', 'y', 'm00', 'm01', 'm10', 'm11', 'vx', 'vy')] +
                       [('member', 4 * EKS), ('rgb', 4 * EKS), ('factors', 20 * EKS), ('shape', EKS),
                        ('pos_f32', EKS), ('refilled_upto', 8 * E)]):
    off[name] = o
    o = a16(o + nbytes)
  return off, o


def _put(state, off, dtype, value):
  b = np.asarray([value], dtype).tobytes()
  state[off:off + len(b)] = torch.frombuffer(bytearray(b), dtype=torch.uint8)


@pytest.mark.parametrize('sampler', ['host', 'device'])
def test_saves_are_byte_identical_read_only_and_laid_out_as_documented(sampler):
  env = _env('goal', 64, sampler, 'sync', pool_depth=5)
  env.reset()
  _run(env, _actions(np.random.RandomState(5), 7, 64))
  eng = env.engine
  E, K, S = eng.n_envs, eng.pool_depth, eng.n_slots
  off, total = _layout(E, K, S)
  n = eng.launch_count()
  s1, s2 = eng.save_state(), eng.save_state()
  assert eng.launch_count() == n
  assert torch.equal(s1, s2) and s1.numel() == total == eng.state_bytes()
  h = s1.numpy()
  assert h[:8].tobytes() == b'SWBCKPT\0'
  assert list(h[8:28].view('<i4')) == [1, E, K, S, 1]
  assert h[28:32].view('<i4')[0] == (sampler == 'device')
  sig = bytes(h[56:56 + ctypes.sizeof(_native.Config)])
  assert sig == eng.signature
  live = eng.download_state()
  assert np.array_equal(h[off['pos_x']:off['pos_x'] + 8 * E * S].view('<f8').reshape(E, S), live['pos_x'])
  assert np.array_equal(h[off['cursor']:off['cursor'] + 4 * E].view('<i4'), live['cursor'])
  assert np.array_equal(h[off['scene_serial']:off['scene_serial'] + 4 * E].view('<i4'),
                        eng.download_state_serial())
  pool = eng.pool_tensors()
  assert np.array_equal(h[off['shape']:off['shape'] + E * K * S].reshape(E, K, S), pool['shape'].cpu().numpy())
  upto = h[off['refilled_upto']:off['refilled_upto'] + 8 * E].view('<i8')
  if sampler == 'device':
    assert np.array_equal(upto, eng.refilled_upto().cpu().numpy())
  else:
    assert (upto == -1).all()
  # 94 bytes per pool entry and 16 S + 21 per env, plus header and padding
  assert 0 <= total - (94 * E * K * S + (16 * S + 21) * E) <= 56 + ctypes.sizeof(_native.Config) + 16 * 20
  # a save of the loaded state is the same bytes
  eng.load_state(s1)
  assert torch.equal(eng.save_state(), s1)
  env.close()


def test_corrupt_buffers_are_refused_naming_the_field_and_enqueue_nothing():
  env = _env('goal', 64, 'device', pool_depth=5)
  env.reset()
  _run(env, _actions(np.random.RandomState(6), 4, 64))
  eng = env.engine
  E, K, S = eng.n_envs, eng.pool_depth, eng.n_slots
  off, total = _layout(E, K, S)
  good = eng.save_state()

  def edit(fn):
    s = good.clone()
    fn(s)
    return s

  cases = [
      ('magic', edit(lambda s: _put(s, 0, 'u1', ord('X')))),
      ('version', edit(lambda s: _put(s, 8, '<u4', 2))),
      ('too few', good[:40].clone()),
      ('size', good[:-16].clone()),
      ('size', torch.cat([good, torch.zeros(16, dtype=torch.uint8)])),
      ('E = ', edit(lambda s: _put(s, 12, '<i4', E + 1))),
      ('K = ', edit(lambda s: _put(s, 16, '<i4', K + 1))),
      ('S = ', edit(lambda s: _put(s, 20, '<i4', S - 1))),
      ('span_class', edit(lambda s: _put(s, 24, '<i4', 3))),
      ('sampler', edit(lambda s: _put(s, 28, '<i4', 0))),
      ('seed', edit(lambda s: _put(s, 32, '<u8', env.seed + 1))),
      ('env_offset', edit(lambda s: _put(s, 40, '<i8', 3))),
      ('signature', edit(lambda s: _put(s, 56 + _native.Config.max_episode_length.offset, '<i4', 7))),
      ('cursor\\[3\\] = %d' % K, edit(lambda s: _put(s, off['cursor'] + 12, '<i4', K))),
      ('cursor\\[0\\] = -1', edit(lambda s: _put(s, off['cursor'], '<i4', -1))),
      ('scene_serial\\[5\\] = -1', edit(lambda s: _put(s, off['scene_serial'] + 20, '<i4', -1))),
      ('reset_next\\[7\\] = 2', edit(lambda s: _put(s, off['reset_next'] + 7, 'u1', 2))),
      ('shape\\[%d\\] = 200' % (S + 1), edit(lambda s: _put(s, off['shape'] + S + 1, 'u1', 200))),
      ('shape\\[0\\] = 13', edit(lambda s: _put(s, off['shape'], 'u1', 13))),
      ('refilled_upto\\[2\\] = -2', edit(lambda s: _put(s, off['refilled_upto'] + 16, '<i8', -2))),
  ]
  torch.cuda.synchronize()
  n = eng.launch_count()
  for match, bad in cases:
    with pytest.raises(_native.NativeError, match=match):
      eng.load_state(bad)
  assert eng.launch_count() == n
  assert torch.equal(eng.save_state(), good)
  # a checkpoint of an engine without a sampler, and of another configuration
  other = _env('goal', 64, 'host', 'sync', pool_depth=5, n_slots=S)
  with pytest.raises(_native.NativeError, match='sampler'):
    other.engine.load_state(good)
  longer = _env('goal', 64, 'device', pool_depth=5, max_episode_length=6, n_slots=S)
  with pytest.raises(_native.NativeError, match='signature'):
    longer.engine.load_state(good)
  with pytest.raises(ValueError):
    eng.load_state(good.cuda())
  assert torch.equal(eng.save_state(), good)
  env.close(); other.close(); longer.close()


def test_environment_mismatches_are_refused_before_anything_changes():
  a = _env('goal', 64, 'device', pool_depth=5)
  a.reset()
  sd = a.state_dict()
  S = a.engine.n_slots
  for kw, key in ((dict(sampler='host', refill='sync', n_slots=S), 'sampler'),
                  (dict(two_rasters=True, n_slots=S), 'renderers'), (dict(name='sorting'), 'n_slots|signature')):
    args = dict(dict(name='goal', n_envs=64, sampler='device', pool_depth=5, seed=9), **kw)
    b = _env(**args)
    b.reset()
    before = b.engine.save_state()
    with pytest.raises(ValueError, match=key):
      b.load_state_dict(sd)
    assert torch.equal(b.engine.save_state(), before)
    if args['sampler'] == 'device':
      assert b.seed == 9
    b.close()
  a.close()


E_TOTAL = 128


def _sharded_worker(rank, world, port, path, ret):
  import torch.distributed as dist
  os.environ['MASTER_ADDR'] = '127.0.0.1'
  os.environ['MASTER_PORT'] = str(port)
  dist.init_process_group('gloo', rank=rank, world_size=world)
  try:
    torch.cuda.set_device(0)
    cfg = dict(sorting.get_config('train'))
    cfg.pop('metadata', None)
    cfg['max_episode_length'] = 5
    rng = np.random.RandomState(11)
    acts = rng.uniform(0, 1, (40, E_TOTAL, 4)).astype(np.float32)

    def run(env, xs):
      out = []
      for x in xs:
        ts = env.step(x)
        out.append({k: v.cpu().numpy().copy() for k, v in
                    dict(step_type=ts.step_type, reward=ts.reward, success=ts.success, status=ts.status,
                         image=ts.observation['image']).items()})
        dist.barrier()   # nobody overwrites a frame slot a peer is still copying
      return out

    env = environment.ShardedBatchedEnvironment(E_TOTAL, device=0, seed=5, host_barrier=True, pool_depth=4,
                                                refill='sync', **cfg)
    env.reset()
    run(env, acts[:7])
    torch.save(env.state_dict(), os.path.join(path, 'rank%d.pt' % rank))
    want = run(env, acts[7:])
    env.close()
    fresh = environment.ShardedBatchedEnvironment(E_TOTAL, device=0, seed=8, host_barrier=True, pool_depth=4,
                                                  refill='sync', **cfg)
    dist.barrier()
    try:
      fresh.load_state_dict(torch.load(os.path.join(path, 'rank%d.pt' % (1 - rank))))
      refused = False
    except ValueError as e:
      refused = 'rank' in str(e)
    fresh.load_state_dict(torch.load(os.path.join(path, 'rank%d.pt' % rank)))
    got = run(fresh, acts[7:])
    ok = refused and all(np.array_equal(w[k], g[k], equal_nan=True) for w, g in zip(want, got) for k in w)
    ok = ok and sum(int((w['step_type'] == 0).sum()) for w in want) >= 3 * E_TOTAL
    ret[rank] = bool(ok)
    fresh.close()
  finally:
    dist.destroy_process_group()


def test_sharded_checkpoint_resumes_each_rank_and_refuses_another_ranks_file(tmp_path):
  import torch.multiprocessing as mp
  world = 2
  port = 29500 + (os.getpid() + 1733) % 2000
  with mp.Manager() as m:
    ret = m.dict()
    mp.spawn(_sharded_worker, args=(world, port, str(tmp_path), ret), nprocs=world, join=True)
    assert dict(ret) == {0: True, 1: True}
