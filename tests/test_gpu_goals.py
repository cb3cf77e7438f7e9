"""Sampled FindGoalPosition goals on the GPU.

The contract every test here checks: an env whose goals are (gx, gy) steps and evaluates bit for bit
as an env whose task is the same tree with those goals as constants.  The reference is a one-env
engine of that constant-goal tree, loaded with the env's record (the goal-free prefix of it) before
each step.  The tree is a MetaAggregated of two sampled goal nodes and a constant one.
"""
import io

import numpy as np
import pytest
import torch

from spriteworld_b200 import _native, constants, environment, renderers, scene, scene_program
from spriteworld_b200 import sprite_generators, tasks
from spriteworld_b200 import engine as engine_lib
from spriteworld_b200 import factor_distributions as distribs
from spriteworld_b200.configs.examples import goal_finding_random_goal

pytestmark = pytest.mark.gpu


def _box(lo, hi):
  return distribs.Product((distribs.Continuous('x', lo, hi), distribs.Continuous('y', lo, hi)))


GOAL_A, GOAL_B = _box(0.1, 0.9), _box(0.3, 0.7)


def _cfg(max_episode_length=6):
  cfg = dict(goal_finding_random_goal.get_config('train'))
  cfg.pop('metadata')
  target_hue = distribs.Continuous('c0', 0., 0.4)
  cfg['task'] = tasks.MetaAggregated([
      tasks.FindGoalPosition(filter_distrib=target_hue, goal_position=GOAL_A, terminate_distance=0.2),
      tasks.FindGoalPosition(goal_position=(0.4, 0.6), terminate_distance=0.3),
      tasks.FindGoalPosition(goal_position=GOAL_B, terminate_distance=0.25)], reward_aggregator='sum')
  cfg['renderers'] = {'goal': renderers.GoalPositions(),
                      'factors': renderers.SpriteFactors(('x', 'y', 'c0'))}
  cfg['max_episode_length'] = max_episode_length
  return cfg


SAMPLERS = {'sync': dict(refill='sync'), 'async': dict(refill='async', refill_threads=2),
            'procs': dict(refill='async', refill_threads=2, refill_procs=2),
            'device': dict(sampler='device', seed=5)}


def _env(n_envs=16, refill='sync', rng_seed=0, **kw):
  kw = dict(SAMPLERS[refill], **kw)
  return environment.BatchedEnvironment(n_envs=n_envs, pool_depth=4, rng=np.random.RandomState(rng_seed),
                                        **dict(_cfg(), **kw))


class Reference(object):
  """One-env engines of the constant-goal tree, one per goal set, fed goal-free records."""

  def __init__(self, env):
    self.env, self.eng = env, env.engine
    self.nodes, _ = env._task.compile()
    self.S = self.eng.n_slots
    self.rb0 = engine_lib.record_layout(self.S)[1]
    self.engines = {}

  def engine(self, goals):
    key = goals.tobytes()
    if key not in self.engines:
      nodes = []
      for nd in self.nodes:
        nd = dict(nd)
        if 'goal_slot' in nd:
          g = nd.pop('goal_slot')
          nd.pop('goal_distrib')
          nd['goal'] = [float(goals[g, 0]), float(goals[g, 1])]
        nodes.append(nd)
      self.engines[key] = engine_lib.Engine(1, self.S, 1, self.env._action_space.compile(), nodes,
                                            constants.SHAPES, max_episode_length=6)
    return self.engines[key]

  def load(self, states, i, goals):
    ref = self.engine(goals)
    rec = states.data[i:i + 1, :self.rb0].clone()
    rec[:, 110 * self.S + 5:] = 0
    ref.load_envs(engine_lib.EnvStates(rec.contiguous(), states.span_class, ref.signature, self.S), [0])
    return ref

  def eval_task(self, ref):
    _native.check(ref._lib.swb_eval_task(ref._h, ref._out, ref._stream()))
    return ref._reward.item(), ref._success.item(), ref._status.item()


def _same(a, b):
  return a == b or (np.isnan(a) and np.isnan(b))


def _eq(a, b):
  """Bit-equal tensors, NaN equal to NaN."""
  if a.is_floating_point():
    a, b = a.nan_to_num(7.5), b.nan_to_num(7.5)
  return torch.equal(a, b)


@pytest.mark.parametrize('refill', sorted(SAMPLERS))
def test_steps_match_the_constant_goal_tree_through_resets_and_set_goals(refill):
  env = _env(refill=refill)
  eng, E = env.engine, env.n_envs
  ref = Reference(env)
  rng = np.random.RandomState(1)
  env.reset()
  firsts = 0
  for t in range(40):
    if t == 10:   # out-of-distribution goals, host ids
      ids = np.arange(0, E, 2)
      set_to = torch.full((len(ids), 2, 2), 0.05, dtype=torch.float64, device=eng.device)
      env.set_goals(set_to, ids)
      assert torch.equal(env.goal_tensor()[torch.as_tensor(ids, device=eng.device)], set_to)
    if t == 20:   # device ids
      ids = torch.arange(1, E, 2, device=eng.device)
      set_to = torch.rand((len(ids), 2, 2), dtype=torch.float64, device=eng.device)
      env.set_goals(set_to, ids, check='device')
      eng.check_env_ids()
      assert torch.equal(env.goal_tensor()[ids], set_to)
    before = env.save_envs()
    goals_before = env.goal_tensor().cpu().numpy()
    assert np.array_equal(before.to_host()['goal'], goals_before)
    actions = rng.uniform(0, 1, (E, 4))
    ts = env.step(actions)
    torch.cuda.synchronize()
    st = {k: v.cpu().numpy() for k, v in eng.state_tensors().items()}
    obs_goal = ts.observation['goal'].cpu().numpy()
    after = env.save_envs()
    for e in range(E):
      if ts.step_type[e].item() == _native.STEP_FIRST:
        firsts += 1
        if t > 10:   # a reset brings a drawn goal
          assert GOAL_A.contains(dict(x=obs_goal[e, 0, 0], y=obs_goal[e, 0, 1]))
          assert GOAL_B.contains(dict(x=obs_goal[e, 1, 0], y=obs_goal[e, 1, 1]))
        # success and status of a FIRST step are the task's on the new scene with its goals
        _, succ, status = ref.eval_task(ref.load(after, e, obs_goal[e]))
        assert ts.reward[e].item() == 0.0
        assert succ == ts.success[e].item() and status == ts.status[e].item(), (t, e)
        continue
      assert np.array_equal(obs_goal[e], goals_before[e])   # an episode keeps its goals
      r = ref.load(before, e, goals_before[e])
      res = r.step(torch.from_numpy(actions[e:e + 1]).to(eng.device))
      assert _same(res.reward.item(), ts.reward[e].item()), (t, e)
      assert res.step_type.item() == ts.step_type[e].item()
      assert res.success.item() == ts.success[e].item()
      assert res.status.item() == ts.status[e].item()
      rs = r.download_state()
      assert np.array_equal(rs['pos_x'][0], st['pos_x'][e]) and np.array_equal(rs['pos_y'][0], st['pos_y'][e])
  assert firsts > 2 * E   # several auto-resets per env


def test_set_goals_refusals_change_nothing():
  env = _env(n_envs=8)
  eng = env.engine
  env.reset()
  torch.cuda.synchronize()
  goals0, launches = env.goal_tensor().clone(), eng.launch_count()
  good = torch.zeros((2, 2, 2), dtype=torch.float64, device=eng.device)
  for bad_goals, ids in ((good[:, :1], [0, 1]), (good.float(), [0, 1]), (good.cpu(), [0, 1]), (good, [0])):
    with pytest.raises(ValueError):
      env.set_goals(bad_goals, ids)
  for ids in ([0, 8], [1, 1], [-1, 2]):
    with pytest.raises(_native.NativeError):
      env.set_goals(good, ids)
  assert eng.launch_count() == launches
  # device ids out of range: refused on the device, all or nothing
  env.set_goals(good, torch.tensor([3, 99], device=eng.device), check='device')
  torch.cuda.synchronize()
  assert torch.equal(env.goal_tensor(), goals0)
  with pytest.raises(ValueError, match='set_goals'):
    eng.check_env_ids()


def test_evaluate_refusals_change_nothing():
  env = _env(n_envs=8)
  eng = env.engine
  env.reset()
  states = env.save_envs()
  n, rb = len(states), states.record_bytes
  no_goals = engine_lib.Engine(n, eng.n_slots, 1, env._action_space.compile(), [dict(kind='no_reward')],
                               constants.SHAPES)
  goals = torch.zeros((n, eng.n_goals, 2), dtype=torch.float64, device=eng.device)
  out = torch.full((16 * n,), 7, dtype=torch.uint8, device=eng.device)   # reward, success, status
  records = states.data.clone()
  R, O, G = states.data.data_ptr(), out.data_ptr(), goals.data_ptr()
  torch.cuda.synchronize()
  launches = eng.launch_count(), no_goals.launch_count()

  def call(engine=eng._h, records=R, n=n, records_bytes=n * rb, goals=G, reward=O, success=O + 8 * n,
           status=O + 9 * n):
    return eng._lib.swb_evaluate_states(engine, records, n, records_bytes, goals, reward, success, status,
                                        eng._stream())

  def refused(match, **kw):
    assert call(**kw) != 0 and match in eng._lib.swb_last_error(), (kw, eng._lib.swb_last_error())
    assert (eng.launch_count(), no_goals.launch_count()) == launches

  refused(b'null', engine=None)
  refused(b'null', records=None)
  for name in ('reward', 'success', 'status'):
    refused(b'null', **{name: None})
  refused(b'n = -1', n=-1)
  refused(b'records is not 16-byte aligned', records=R + 8)
  refused(b'records need', records_bytes=n * rb - 1)
  refused(b'G = 0', engine=no_goals._h)
  refused(b'goals are not 8-byte aligned', goals=G + 4)
  refused(b'reward overlaps the records', reward=R + 16)
  refused(b'status overlaps the records', status=R + n * rb - 1)
  refused(b'reward is not 8-byte aligned', reward=O + 4)
  refused(b'status overlaps success', status=O + 9 * n - 1)
  torch.cuda.synchronize()
  assert bool((out == 7).all()) and torch.equal(states.data, records)
  assert call(n=0) == 0 and eng.launch_count() == launches[0]
  assert call() == 0 and eng.launch_count() == launches[0] + 1
  no_goals.close()


def test_evaluate_relabels_records_as_the_constant_goal_tree():
  env = _env(n_envs=32)
  eng = env.engine
  ref = Reference(env)
  env.reset()
  rng = np.random.RandomState(2)
  for _ in range(3):
    env.step(rng.uniform(0, 1, (env.n_envs, 4)))
  states = env.save_envs()
  # goals=None: the step's task value of the live envs
  out = eng._out
  _native.check(eng._lib.swb_eval_task(eng._h, out, eng._stream()))
  live = (eng._reward.clone(), eng._success.clone(), eng._status.clone())
  snapshot, launches = eng.save_state(), eng.launch_count()
  own = env.evaluate(states)
  assert eng.launch_count() == launches + 1
  for a, b in zip(own, live):
    assert _eq(a, b)
  n = 200
  pick = torch.as_tensor(rng.randint(0, len(states), n), device=eng.device)
  recs = states.take(pick)
  goals = torch.as_tensor(rng.uniform(-0.2, 1.2, (n, 2, 2)), device=eng.device)
  reward, success, status = env.evaluate(recs, goals)
  assert eng.launch_count() == launches + 2
  assert torch.equal(eng.save_state(), snapshot)   # read-only
  g = goals.cpu().numpy()
  for i in range(n):
    want = ref.eval_task(ref.load(recs, i, g[i]))
    assert _same(reward[i].item(), want[0]) and success[i].item() == want[1] and status[i].item() == want[2]
  with pytest.raises(ValueError):
    env.evaluate(recs, goals[:, :1])


def test_records_rollout_expand_and_observe_carry_goals():
  env = _env(n_envs=16)
  eng = env.engine
  env.reset()
  rng = np.random.RandomState(4)
  env.step(rng.uniform(0, 1, (16, 4)))
  states = env.save_envs()
  goals = env.goal_tensor().clone()
  obs, _ = env.observe(states)
  assert torch.equal(obs['goal'], goals)
  # load into permuted envs (host and device ids) and copy: goals follow the records
  perm = np.random.RandomState(5).permutation(16)
  env.load_envs(states, perm)
  assert torch.equal(env.goal_tensor()[torch.as_tensor(perm, device=eng.device)], goals)
  env.load_envs(states, torch.as_tensor(perm[::-1].copy(), device=eng.device), check='device')
  assert torch.equal(env.goal_tensor()[torch.as_tensor(perm[::-1].copy(), device=eng.device)], goals)
  env.load_envs(states)
  env.copy_envs([0, 1, 2], [5, 6, 7])
  env.copy_envs(torch.tensor([3], device=eng.device), torch.tensor([3 + 8], device=eng.device), check='device')
  want = goals.clone()
  want[5:8] = goals[0:3]
  want[11] = goals[3]
  assert torch.equal(env.goal_tensor(), want)
  env.load_envs(states)
  # rollouts from live envs and from their records agree; leaves keep their roots' goals
  plans = rng.uniform(0, 1, (5, 16, 3, 4))
  live = env.rollout(plans)
  rec = env.rollout(plans, states)
  for f in ('reward', 'step_type', 'success', 'status'):
    assert _eq(getattr(live, f), getattr(rec, f))
  res, leaves = env.expand(plans, states)
  assert torch.equal(leaves.fields()['goal'], goals.repeat_interleave(3, 0))
  # a leaf is what an env loaded from its root and stepped through the plan would save
  C = 3
  big = _env(n_envs=16 * C, rng_seed=9)
  big.load_envs(states.take(torch.arange(16, device=eng.device).repeat_interleave(C)))
  for t in range(5):
    big.engine.step(torch.from_numpy(plans[t].reshape(16 * C, 4)).to(eng.device))
  got = big.save_envs()
  live_leaf = res.step_type.cpu().numpy()   # plans that ended early stop being stepped in `big` too
  ended = (live_leaf == _native.STEP_LAST).any(0).reshape(-1)
  keep = torch.as_tensor(~ended, device=eng.device)
  assert torch.equal(got.data[keep], leaves.data[keep])


@pytest.mark.parametrize('refill', ['sync', 'device'])
def test_checkpoint_resumes_bit_exact_with_goals(refill):
  env = _env(n_envs=64, refill=refill)
  rng = np.random.RandomState(6)
  acts = rng.uniform(0, 1, (30, 64, 4))
  env.reset()
  for t in range(5):
    env.step(acts[t])
  buf = io.BytesIO()
  torch.save(env.state_dict(), buf)
  first = []
  for t in range(5, 30):
    ts = env.step(acts[t])
    first.append((ts.reward.clone(), ts.step_type.clone(), ts.observation['goal'].clone()))
  other = _env(n_envs=64, refill=refill, rng_seed=11)
  other.load_state_dict(torch.load(io.BytesIO(buf.getvalue()), weights_only=True))
  for t in range(5, 30):
    ts = other.step(acts[t])
    r, s, g = first[t - 5]
    assert _eq(ts.reward, r) and torch.equal(ts.step_type, s)
    assert torch.equal(ts.observation['goal'], g)


def test_goal_free_engines_and_device_sampler():
  cfg = _cfg()
  goal_env = environment.BatchedEnvironment(n_envs=4, sampler='device', seed=1, **cfg)
  plain_program = scene_program.compile_program(goal_env._init_sprites, goal_env._filters,
                                                goal_env._color_to_rgb)
  with pytest.raises(_native.NativeError, match='goal slots'):   # a program that draws no goals
    goal_env.engine.load_sampler(plain_program, 1)
  plain = dict(cfg, task=tasks.FindGoalPosition(goal_position=(0.5, 0.5)))
  env = environment.BatchedEnvironment(n_envs=4, **plain)
  assert env.engine.n_goals == 0 and 'goal' not in env.engine.pool_tensors()
  assert env.engine.record_bytes == (110 * env.engine.n_slots + 5 + 15) // 16 * 16
  assert env.reset().observation['goal'].shape == (4, 0, 2)
  goal_env = environment.BatchedEnvironment(n_envs=4, **cfg)
  G = goal_env.engine.n_goals
  assert G == 2 and goal_env.engine.record_bytes == engine_lib.record_layout(goal_env.engine.n_slots, G)[1]
  gym_spec = goal_env._other['goal'].batch_observation_spec(goal_env)
  assert gym_spec.shape == (2, 2) and gym_spec.dtype == np.float64


def test_host_goals_replay_the_rng_after_the_scenes():
  env = _env(n_envs=8, rng_seed=3)
  eng = env.engine
  rs = np.random.RandomState(3)
  sprite_generators.batch_of(env._init_sprites, 8 * 4, rs)
  want = scene.draw_goals(env._task.goal_distributions(), 8 * 4, rs)
  got = eng.pool_tensors()['goal'].cpu().numpy().reshape(8 * 4, 2, 2)
  assert np.array_equal(got, want)


def test_device_goals_equal_the_host_build_and_leave_the_sprites_alone():
  env = _env(n_envs=8, refill='device')
  eng, S = env.engine, env.engine.n_slots
  ids, idx = np.repeat(np.arange(8), 50), np.tile(np.arange(50), 8)
  dev = eng.sample_scenes(ids, idx)
  host, fail = scene_program.sample_on_host(env._program, env.seed, ids, idx, S)
  assert fail is None
  goals = dev['goal'].cpu().numpy()
  assert goals.shape == (400, 2, 2) and np.array_equal(goals, host['goal'])
  for g, d in enumerate((GOAL_A, GOAL_B)):
    assert all(d.contains(dict(x=x, y=y)) for x, y in goals[:, g])
  plain = scene_program.compile_program(env._init_sprites, env._filters, env._color_to_rgb)
  base, _ = scene_program.sample_on_host(plain, env.seed, ids, idx, S)
  for f in ('x', 'y', 'm00', 'm11', 'vx', 'member', 'shape', 'rgb', 'factors', 'factor_value'):
    assert np.array_equal(base[f], host[f]), f
    assert np.array_equal(dev[f].cpu().numpy().view(base[f].dtype), base[f]), f
  # the pool's rings hold the same draws: env e's scene a in ring slot a % K
  pool = eng.pool_tensors()['goal'].cpu().numpy()
  ref, _ = scene_program.sample_on_host(env._program, env.seed, np.repeat(np.arange(8), 4),
                                        np.tile(np.arange(4), 8), S)
  assert np.array_equal(pool.reshape(32, 2, 2), ref['goal'])


def test_expand_from_live_roots_keeps_their_goals():
  env = _env(n_envs=16)
  env.reset()
  env.step(np.random.RandomState(8).uniform(0, 1, (16, 4)))
  plans = np.random.RandomState(9).uniform(0, 1, (4, 16, 3, 4))
  res, leaves = env.expand(plans)
  _, from_records = env.expand(plans, env.save_envs())
  assert torch.equal(leaves.fields()['goal'], env.goal_tensor().repeat_interleave(3, 0))
  assert torch.equal(leaves.data, from_records.data)
