"""BatchedEnvironment(sampler='device') and the sampler kernels on the GPU, against the CPU build
of the same sampler (scene_program.sample_on_host), which tests/test_scene_program.py holds to
NumPy's Philox, scene.arrays_from_layout and the host sampler's distribution."""
import numpy as np
import pytest
import torch

from spriteworld_b200 import environment, scene_program
from spriteworld_b200 import factor_distributions as distribs
from spriteworld_b200 import sprite_generators as gen
from spriteworld_b200.configs.cobra import goal_finding_more_distractors
from tests.test_scene_program import CONFIGS, bits, compiled

pytestmark = pytest.mark.gpu


def _env(pool_depth=8, n_envs=64, seed=7, config=None, **kw):
  cfg = dict(config or goal_finding_more_distractors.get_config('train'))
  cfg.pop('metadata', None)
  return environment.BatchedEnvironment(n_envs=n_envs, pool_depth=pool_depth, sampler='device',
                                        seed=seed, rng=np.random.RandomState(0), **dict(cfg, **kw))


@pytest.mark.parametrize('name,mode', CONFIGS)
def test_sample_scenes_equals_cpu_build(name, mode):
  cfg, filters, cmap, prog = compiled(name, mode)
  env = _env(n_envs=4, config=cfg)
  try:
    rng = np.random.RandomState(2)
    ids = np.concatenate([np.arange(512), rng.randint(0, 2 ** 62, 512), [2 ** 63 - 1]])
    idx = np.concatenate([np.arange(512) % 5, rng.randint(0, 2 ** 62, 512), [2 ** 63 - 1]])
    out = env.engine.sample_scenes(ids, idx)
    ref, fail = scene_program.sample_on_host(prog, env.seed, ids, idx, env.engine.n_slots)
    assert fail is None
    for k, v in out.items():
      v = v.cpu().numpy()
      if k == 'member':
        v = v.view(np.uint32)
      assert np.array_equal(bits(v), bits(ref[k])), k
  finally:
    env.close()


POOL_FIELDS = ('x', 'y', 'm00', 'm01', 'm10', 'm11', 'vx', 'vy', 'member', 'shape', 'pos_f32', 'rgb',
               'factors')


def _pool_numpy(eng):
  pool = {k: v.cpu().numpy() for k, v in eng.pool_tensors().items()}
  pool['member'] = pool['member'].view(np.uint32)
  pool['rgb'] = pool['rgb'][..., :3]
  return pool


def _ring_check(env, res, written=(), env_offset=0):
  """Every field of the pool entries an env's ring holds -- its fresh scenes serial+1 ..
  refilled_upto, and the scene it is on unless a load or copy has written that entry (`written`)
  -- equals the CPU build's scene (env_offset + e, a); envs on a FIRST step show that scene's
  initial positions."""
  eng = env.engine
  K = env._K
  serial = eng.scene_serial().cpu().numpy().astype(np.int64)
  upto = eng.refilled_upto().cpu().numpy()
  assert (upto >= serial).all() and (upto - serial <= K - 1).all()
  envs, scenes = [], []
  for e in range(eng.n_envs):
    lo = serial[e] + (1 if e in written else 0)
    envs.extend([e] * int(upto[e] + 1 - lo))
    scenes.extend(range(lo, upto[e] + 1))
  envs, scenes = np.array(envs, np.int64), np.array(scenes, np.int64)
  ref, _ = scene_program.sample_on_host(env._program, env.seed, envs + env_offset, scenes, eng.n_slots)
  pool = _pool_numpy(eng)
  for f in POOL_FIELDS:
    assert np.array_equal(bits(pool[f][envs, scenes % K]), bits(ref[f])), f
  first = np.flatnonzero(res.step_type.cpu().numpy() == 0)
  first = np.array([e for e in first if e not in written], np.int64)
  if len(first):
    cur, _ = scene_program.sample_on_host(env._program, env.seed, first + env_offset, serial[first],
                                          eng.n_slots)
    live = eng.state_tensors()
    assert np.array_equal(live['pos_x'].cpu().numpy()[first], cur['x'])
    assert np.array_equal(live['pos_y'].cpu().numpy()[first], cur['y'])
  return len(envs)


class _Written(object):
  """Envs whose current pool entry a load or copy has written since their last scene start."""

  def __init__(self, env):
    self.env, self.envs = env, set()
    self.serial = env.engine.scene_serial().cpu().numpy().copy()

  def step_done(self):
    serial = self.env.engine.scene_serial().cpu().numpy()
    self.envs -= set(np.flatnonzero(serial != self.serial).tolist())
    self.serial = serial.copy()

  def add(self, ids):
    self.envs |= set(int(i) for i in ids)


def test_same_seed_same_episodes_whatever_pool_depth_and_timing():
  a, b = _env(pool_depth=4), _env(pool_depth=32)
  try:
    rng = np.random.RandomState(5)
    for t in range(200):
      act = rng.uniform(0, 1, (64, 4)).astype(np.float32)
      if t % 17 == 3:
        torch.cuda._sleep(2000000)
      ra, rb = a.step(act), b.step(act)
      for f in ('step_type', 'reward', 'success', 'status'):
        assert torch.equal(getattr(ra, f), getattr(rb, f)), (t, f)
      assert torch.equal(ra.observation['image'], rb.observation['image']), t
      _ring_check(a, ra)
      _ring_check(b, rb)
    assert a.refill_stats()['mode'] == 'device' and a.refill_stats()['launches'] > 0
  finally:
    a.close()
    b.close()


def test_resets_loads_and_copies_next_to_the_device_refill():
  env = _env(pool_depth=4)
  try:
    rng = np.random.RandomState(8)
    written = _Written(env)
    saved = None
    checked = 0
    for t in range(150):
      if t % 9 == 0:
        res = env.reset()
      else:
        res = env.step(rng.uniform(0, 1, (64, 4)).astype(np.float32))
      torch.cuda.synchronize()
      written.step_done()
      if t == 20:
        saved = env.save_envs(np.arange(16, 24))
      if t % 11 == 5:
        env.copy_envs(np.arange(8), np.arange(8, 16))
        written.add(range(8, 16))
      if saved is not None and t % 13 == 7:
        env.load_envs(saved, np.arange(40, 48))
        written.add(range(40, 48))
      checked += _ring_check(env, res, written.envs)
    assert checked > 64 * 100
    env.check_sampler()
  finally:
    env.close()


def test_episodes_match_the_oracle_stepped_from_the_same_scenes():
  from oracle import oracle
  from spriteworld_b200 import constants
  from tests import fixtures
  cfg = dict(goal_finding_more_distractors.get_config('train'))
  env = _env(pool_depth=4, config=cfg, max_episode_length=7)
  try:
    eng, E, K, S = env.engine, env.n_envs, env._K, env.engine.n_slots
    pool = np.zeros((E, K, S), oracle.SPRITE_DTYPE)
    fields = ('x', 'y', 'm00', 'm01', 'm10', 'm11', 'vx', 'vy', 'member', 'shape', 'pos_f32', 'rgb')
    have = np.full(E, -1, np.int64)

    def refill_mirror():
      upto = eng.refilled_upto().cpu().numpy()
      envs = np.repeat(np.arange(E), upto - have)
      scenes = np.concatenate([np.arange(have[e] + 1, upto[e] + 1) for e in range(E)]).astype(np.int64)
      if len(envs):
        ref, _ = scene_program.sample_on_host(env._program, env.seed, envs, scenes, S)
        for f in fields:
          pool[f][envs, scenes % K] = ref[f]
      have[:] = upto

    nodes, _ = cfg['task'].compile()
    ocfg = oracle.with_device_sqrt(fixtures.env_cfg_from_meta(dict(
        action=cfg['action_space'].compile(), keep_in_frame=True, max_episode_length=7, nodes=nodes)))
    refill_mirror()
    bo = oracle.BatchOracle(ocfg, oracle.shape_table(constants.SHAPES), oracle.raster_cfg(64, 64, 5), pool)
    bo.pool = pool
    rng = np.random.RandomState(3)
    n_first = 0
    for t in range(60):
      a = rng.uniform(0, 1, (E, 4)).astype(np.float32)
      ts = env.step(a)
      torch.cuda.synchronize()
      refill_mirror()          # the refill ran on the device before this step
      bo.step(a)
      assert np.array_equal(ts.step_type.cpu().numpy(), bo.step_type), t
      assert np.array_equal(ts.reward.cpu().numpy(), bo.reward, equal_nan=True), t
      assert np.array_equal(ts.success.cpu().numpy(), bo.success), t
      assert np.array_equal(ts.observation['image'].cpu().numpy(), bo.frames), t
      n_first += int((bo.step_type == 0).sum())
    assert n_first > 5 * E
  finally:
    env.close()


def test_factor_and_success_observations_equal_the_host_packing():
  from spriteworld_b200 import renderers as sw_renderers
  from spriteworld_b200 import scene
  cfg = dict(goal_finding_more_distractors.get_config('train'))
  cfg['renderers'] = dict(cfg['renderers'], factors=sw_renderers.SpriteFactors(),
                          success=sw_renderers.Success())
  env = _env(pool_depth=4, config=cfg, max_episode_length=5)
  _, filters = cfg['task'].compile()
  try:
    rng = np.random.RandomState(4)
    written = _Written(env)
    for t in range(40):
      ts = env.step(rng.uniform(0, 1, (64, 4)).astype(np.float32))
      torch.cuda.synchronize()
      written.step_done()
      if t == 17:
        env.copy_envs(np.arange(4), np.arange(4, 8))
        written.add(range(4, 8))
      serial = env.engine.scene_serial().cpu().numpy().astype(np.int64)
      envs = np.array([e for e in range(64) if e not in written.envs], np.int64)
      ref, _ = scene_program.sample_on_host(env._program, env.seed, envs, serial[envs], env.engine.n_slots)
      host = scene.arrays_from_layout(
          scene_program.layout_from_factor_table(ref['factor_value'], ref['factor_kind']),
          env.engine.n_slots, filters, env._color_to_rgb)
      got = {k: v.cpu().numpy()[envs] for k, v in ts.observation['factors'].items()}
      want = dict(shape=host['shape'].astype(np.float32), x_vel=host['vx'].astype(np.float32),
                  y_vel=host['vy'].astype(np.float32))
      for i, f in enumerate(('scale', 'angle', 'c0', 'c1', 'c2')):
        want[f] = host['factors'][..., i]
      for f, v in want.items():
        assert np.array_equal(bits(got[f]), bits(v)), (t, f)
      assert np.array_equal(got['mask'], host['shape'] > 0)
      live = env.engine.state_tensors()
      assert np.array_equal(got['x'], live['pos_x'].cpu().numpy()[envs].astype(np.float32))
      assert ts.observation['success'].dtype == torch.bool
      assert torch.equal(ts.observation['success'], ts.success.to(bool))
  finally:
    env.close()


def test_no_host_sync_across_device_steps():
  env = _env()
  try:
    act = torch.rand((64, 4), device=env.engine.device)
    env.step(act)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
      for _ in range(40):
        env.step(act)
    finally:
      torch.cuda.set_sync_debug_mode(0)
  finally:
    env.close()


def test_impossible_set_minus_is_reported_and_steps_go_on():
  base = distribs.Product([distribs.Continuous('x', 0.2, 0.4), distribs.Continuous('y', 0.2, 0.4)] +
                          [distribs.Continuous(c, 0.5, 0.6) for c in ('c0', 'c1', 'c2')])
  impossible = distribs.SetMinus(base, distribs.Continuous('x', 0.0, 1.0))
  cfg = dict(goal_finding_more_distractors.get_config('train'))
  cfg['init_sprites'] = gen.generate_sprites(impossible, 1)
  env = _env(n_envs=8, config=cfg)
  try:
    with pytest.raises(ValueError, match='Maximum number of tried exceeded'):
      env.check_sampler()
    env.check_sampler()   # cleared
    for _ in range(5):
      res = env.step(np.full((8, 4), 0.5, np.float32))
    torch.cuda.synchronize()
    assert (env.engine.state_tensors()['pos_x'].cpu().numpy() == 0).all()   # empty scenes
    assert res.step_type.shape == (8,)
  finally:
    env.close()


def _sharded_worker(rank, world, port, ret):
  import os
  import torch.distributed as dist
  os.environ['MASTER_ADDR'] = '127.0.0.1'
  os.environ['MASTER_PORT'] = str(port)
  dist.init_process_group('gloo', rank=rank, world_size=world)
  try:
    from spriteworld_b200.configs.cobra import sorting
    torch.cuda.set_device(0)
    cfg = dict(sorting.get_config('train'), max_episode_length=7)
    cfg.pop('metadata')
    n_total = 64
    sharded = environment.ShardedBatchedEnvironment(n_total, device=0, seed=5, host_barrier=True,
                                                    pool_depth=4, sampler='device', **cfg)
    whole = environment.BatchedEnvironment(n_envs=n_total, device=0, pool_depth=4, sampler='device',
                                           seed=5, **cfg)
    rng = np.random.RandomState(11)
    ok, n_first = True, 0
    for t in range(40):
      a = rng.uniform(0, 1, (n_total, 4)).astype(np.float32)
      ts, tw = sharded.step(a), whole.step(a)
      torch.cuda.synchronize()
      for f in ('step_type', 'reward', 'success', 'status'):
        ok = ok and torch.equal(getattr(ts, f).cpu(), getattr(tw, f).cpu())
      ok = ok and torch.equal(ts.observation['image'].cpu(), tw.observation['image'].cpu())
      n_first += int((tw.step_type == 0).sum().item())
      dist.barrier()
    local = sharded.local
    ok = ok and local.refill_stats()['mode'] == 'device' and local.seed == 5
    ret[rank] = bool(ok) and n_first > 3 * n_total
    whole.close()
    sharded.close()
  finally:
    dist.destroy_process_group()


def test_sharded_run_equals_the_one_gpu_run():
  import os
  import torch.multiprocessing as mp
  world = 2
  port = 29500 + (os.getpid() + 1733) % 2000
  with mp.Manager() as m:
    ret = m.dict()
    mp.spawn(_sharded_worker, args=(world, port, ret), nprocs=world, join=True)
    assert dict(ret) == {0: True, 1: True}
