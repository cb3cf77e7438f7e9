"""Goal finding with a goal drawn per episode: the scene of cobra/goal_finding_new_position, with
the FindGoalPosition goal drawn with every scene -- uniformly from [0.1, 0.9)^2 in train, from the
held-out upper-right quadrant [0.5, 0.9)^2 in test -- and observed through GoalPositions.  For
goal-conditioned policies; BatchedEnvironment only (the one-env Environment has no sampled goals)."""
from spriteworld_b200 import factor_distributions as distribs
from spriteworld_b200 import renderers as sw_renderers
from spriteworld_b200 import tasks
from spriteworld_b200.configs.cobra import common
from spriteworld_b200.configs.cobra import goal_finding_new_position


def _box(lo, hi):
  return distribs.Product((distribs.Continuous('x', lo, hi), distribs.Continuous('y', lo, hi)))


MODES_GOALS = {
    'train': _box(0.1, 0.9),
    'test': _box(0.5, 0.9),
}


def get_config(mode='train'):
  config = goal_finding_new_position.get_config('train')
  target_hue = distribs.Continuous('c0', 0., 0.4)
  config['task'] = tasks.FindGoalPosition(
      filter_distrib=target_hue, goal_position=MODES_GOALS[mode],
      terminate_distance=goal_finding_new_position.TERMINATE_DISTANCE)
  config['renderers'] = dict(common.renderers(), goal=sw_renderers.GoalPositions())
  config['metadata'] = {'name': 'goal_finding_random_goal.py', 'mode': mode}
  return config
