"""Sampled FindGoalPosition goals on the host: goal slots, refusals, the host draw and the record
layout (no GPU needed)."""
import numpy as np
import pytest

from spriteworld_b200 import engine as engine_lib
from spriteworld_b200 import environment
from spriteworld_b200 import factor_distributions as distribs
from spriteworld_b200 import scene
from spriteworld_b200 import tasks
from spriteworld_b200.configs.examples import goal_finding_random_goal


def _box(lo, hi):
  return distribs.Product((distribs.Continuous('x', lo, hi), distribs.Continuous('y', lo, hi)))


def test_goal_slots_follow_post_order_and_constant_nodes_are_unchanged():
  d = _box(0.1, 0.9)
  const = tasks.FindGoalPosition(goal_position=(0.3, 0.7))
  tree = tasks.MetaAggregated([tasks.FindGoalPosition(goal_position=d), const,
                               tasks.FindGoalPosition(goal_position=d)])
  nodes, filters = tree.compile()
  assert [nd.get('goal_slot') for nd in nodes] == [0, None, 1, None]
  assert tree.goal_distributions() == [d, d]      # one object in two nodes: two slots
  # a constant goal's node is the dict it always was
  assert nodes[1] == const.compile()[0][0]
  assert set(nodes[1]) == {'kind', 'filter_slot', 'goal', 'weights', 'terminate_distance',
                           'terminate_bonus', 'raw_reward_multiplier', 'sparse_reward'}
  assert const.goal_distributions() == []


def test_bad_goal_distributions_and_too_many_slots_are_refused():
  three = distribs.Product((distribs.Continuous('x', 0, 1), distribs.Continuous('y', 0, 1),
                            distribs.Continuous('c0', 0, 1)))
  for bad in (distribs.Continuous('x', 0, 1), three):
    with pytest.raises(ValueError, match="exactly {'x', 'y'}"):
      tasks.FindGoalPosition(goal_position=bad)
  d = _box(0.1, 0.9)
  tasks.MetaAggregated([tasks.FindGoalPosition(goal_position=d) for _ in range(8)]).compile()
  with pytest.raises(NotImplementedError, match='at most 8'):
    tasks.MetaAggregated([tasks.FindGoalPosition(goal_position=d) for _ in range(9)]).compile()


def test_reward_and_the_one_env_environment_refuse_sampled_goals():
  cfg = goal_finding_random_goal.get_config('train')
  with pytest.raises(NotImplementedError, match='sampled goals'):
    cfg['task'].reward([])
  with pytest.raises(NotImplementedError, match='sampled goals'):
    cfg['task'].success([])
  with pytest.raises(NotImplementedError, match='sampled goals'):
    environment.Environment(cfg['task'], cfg['action_space'], cfg['renderers'], cfg['init_sprites'])


def test_draw_goals_replays_sample_batch_per_slot_after_the_scenes():
  a, b = _box(0.1, 0.9), _box(0.5, 0.9)
  rng = np.random.RandomState(3)
  copy = np.random.RandomState()
  copy.set_state(rng.get_state())
  goals = scene.draw_goals([a, b], 37, rng)
  assert goals.dtype == np.float64 and goals.shape == (37, 2, 2)
  for g, d in enumerate((a, b)):
    cols = d.sample_batch(37, copy)
    assert np.array_equal(goals[:, g, 0], cols['x']) and np.array_equal(goals[:, g, 1], cols['y'])
    assert all(d.contains({'x': x, 'y': y}) for x, y in goals[:, g])
  assert np.array_equal(rng.randint(0, 2 ** 31 - 1, 4), copy.randint(0, 2 ** 31 - 1, 4))
  assert scene.draw_goals([], 5, rng) is None


def test_record_layout_appends_goals_and_keeps_the_goal_free_size():
  for S in (1, 3, 5, 32):
    fields, nbytes = engine_lib.record_layout(S)
    assert nbytes == (110 * S + 5 + 15) // 16 * 16
    assert engine_lib.record_layout(S, 0) == (fields, nbytes)
    for G in (1, 2, 8):
      gf, gbytes = engine_lib.record_layout(S, G)
      assert gf[:-1] == fields
      name, off, dtype, shape = gf[-1]
      assert name == 'goal' and off % 8 == 0 and off >= 110 * S + 5 and shape == (G, 2)
      assert gbytes == (off + 16 * G + 15) // 16 * 16


def test_test_mode_goals_lie_in_the_held_out_quadrant():
  cfg = goal_finding_random_goal.get_config('test')
  d, = cfg['task'].goal_distributions()
  goals = scene.draw_goals([d], 500, np.random.RandomState(0))
  assert (goals >= 0.5).all() and (goals < 0.9).all()


def test_sharded_environment_refuses_goal_positions_before_it_needs_a_process_group():
  cfg = goal_finding_random_goal.get_config('train')
  with pytest.raises(NotImplementedError, match='GoalPositions'):
    environment.ShardedBatchedEnvironment(4, **cfg)


def test_host_build_of_the_device_sampler_draws_goals_after_the_sprites():
  from spriteworld_b200 import scene_program
  cfg = goal_finding_random_goal.get_config('test')
  task = cfg['task']
  _, filters = task.compile()
  cmap = cfg['renderers']['image'].color_to_rgb
  goals = task.goal_distributions()
  prog = scene_program.compile_program(cfg['init_sprites'], filters, cmap, goals)
  plain = scene_program.compile_program(cfg['init_sprites'], filters, cmap)
  ids, idx = np.repeat(np.arange(20), 10), np.tile(np.arange(10), 20)
  with_goals, fail = scene_program.sample_on_host(prog, 7, ids, idx, 2)
  without, _ = scene_program.sample_on_host(plain, 7, ids, idx, 2)
  assert fail is None and 'goal' not in without
  for f in without:
    assert np.array_equal(with_goals[f], without[f]), f
  g = with_goals['goal']
  assert g.shape == (200, 1, 2) and all(goals[0].contains({'x': x, 'y': y}) for x, y in g[:, 0])
  assert len({tuple(v) for v in g[:, 0]}) == 200   # a draw per scene
  again, _ = scene_program.sample_on_host(prog, 7, ids[::-1], idx[::-1], 2)
  assert np.array_equal(again['goal'][::-1], g)   # a pure function of (seed, env, scene)
