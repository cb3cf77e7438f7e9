"""Tasks: reward and success functions over the sprites of an env.

Same classes and constructor signatures as the reference's `spriteworld/tasks.py`
(NoReward :70-81, FindGoalPosition :84-158, Clustering :161-245, MetaAggregated :248-296).
A task here is a *description*: `compile()` flattens the task tree into the POD nodes of
`swb_config` (include/spriteworld_b200.h) and the list of filter distributions whose
membership is precomputed per sprite at reset.  A FindGoalPosition whose goal is a distribution
over ('x', 'y') gets a goal slot: its goal is drawn with every scene and stored in the scene pool
entry (goal_distributions() lists them in slot order).  The arithmetic itself runs in the step
kernel (csrc/swb_step.cuh).  `reward(sprites)` / `success(sprites)` on a Python sprite
list are kept for the plugin protocol; they evaluate on the GPU through a one-env engine
(_direct.py) -- there is no CPU implementation of the task math in this package.
"""
import abc

import numpy as np

MAX_GOALS = 8   # SWB_MAX_GOALS: sampled goals per task tree
_AGGREGATORS = ('sum', 'max', 'min', 'mean')
_CRITERIA = ('all', 'any')


class AbstractTask(abc.ABC):

  @abc.abstractmethod
  def _emit(self, nodes, filters):
    """Appends this task's node(s) to `nodes` (post-order); returns the node index."""

  def compile(self):
    """Returns (nodes, filters): POD node dicts, root last, and the distinct filter
    distributions in slot order (bit i of a sprite's `member` mask <-> filters[i]).  A
    find_goal node's `goal_slot` is -1 for a constant goal, else the index of its distribution
    in goal_distributions()."""
    nodes, filters = [], []
    self._emit(nodes, filters)
    slot = 0
    for nd in nodes:   # a constant goal's node has neither key: its dict is as it always was
      if 'goal_distrib' in nd:
        nd['goal_slot'] = slot
        slot += 1
    if slot > MAX_GOALS:
      raise NotImplementedError('task tree has %d sampled goals; at most %d (SWB_MAX_GOALS) are '
                                'supported' % (slot, MAX_GOALS))
    return nodes, filters

  def goal_distributions(self):
    """The goal distributions of the tree's sampled goals, in goal-slot order (node post-order;
    one distribution object used by two nodes gives two slots)."""
    nodes, _ = self.compile()
    return [nd['goal_distrib'] for nd in nodes if 'goal_distrib' in nd]

  def _constant_goals(self, where):
    """NotImplementedError if the tree samples goals: `where` has no per-scene goal."""
    if self.goal_distributions():
      raise NotImplementedError(
          '%s does not support sampled goals (FindGoalPosition with a goal distribution); use '
          'BatchedEnvironment' % where)

  def _filters_static(self):
    """Task filters must depend only on factors that do not change during an episode."""
    _, filters = self.compile()
    for f in filters:
      moving = set(f.keys) & {'x', 'y'}
      if moving:
        raise NotImplementedError(
            'task filter on %s: filters are evaluated once per reset; position-dependent '
            'filters are not supported' % sorted(moving))
    return filters

  def reward(self, sprites):
    from spriteworld_b200 import _direct
    return _direct.task_value(self, sprites)[0]

  def success(self, sprites):
    from spriteworld_b200 import _direct
    return _direct.task_value(self, sprites)[1]


def _slot(filters, distrib):
  if distrib is None:
    return -1
  for i, f in enumerate(filters):
    if f is distrib:
      return i
  filters.append(distrib)
  return len(filters) - 1


class NoReward(AbstractTask):
  """No task: reward 0, never successful."""

  def __init__(self):
    pass

  def _emit(self, nodes, filters):
    nodes.append(dict(kind='no_reward'))
    return len(nodes) - 1

  def reward(self, unused_sprites):
    return 0.0

  def success(self, unused_sprites):
    return False


class FindGoalPosition(AbstractTask):
  """Bring every sprite selected by `filter_distrib` to `goal_position`: an (x, y) pair, or a
  factor distribution over exactly {'x', 'y'} from which each scene draws its own goal
  (BatchedEnvironment only)."""

  def __init__(self, filter_distrib=None, goal_position=(0.5, 0.5), terminate_distance=0.05,
               terminate_bonus=0.0, weights_dimensions=(1, 1), sparse_reward=False,
               raw_reward_multiplier=50):
    self._filter_distrib = filter_distrib
    if hasattr(goal_position, 'sample_batch'):
      keys = getattr(goal_position, 'keys', None)
      if keys is None or set(keys) != {'x', 'y'}:
        raise ValueError("a goal distribution must have keys exactly {'x', 'y'}, got %r"
                         % (sorted(keys) if keys is not None else None,))
      self._goal_distrib, self._goal_position = goal_position, np.full(2, np.nan)
    else:
      self._goal_distrib, self._goal_position = None, np.asarray(goal_position)
    self._terminate_bonus = terminate_bonus
    self._terminate_distance = terminate_distance
    self._sparse_reward = sparse_reward
    self._weights_dimensions = np.asarray(weights_dimensions)
    self._raw_reward_multiplier = raw_reward_multiplier

  def _emit(self, nodes, filters):
    sampled = {} if self._goal_distrib is None else dict(goal_distrib=self._goal_distrib)
    nodes.append(dict(
        kind='find_goal', filter_slot=_slot(filters, self._filter_distrib),
        goal=[float(v) for v in self._goal_position], **sampled,
        weights=[float(v) for v in self._weights_dimensions],
        terminate_distance=float(self._terminate_distance),
        terminate_bonus=float(self._terminate_bonus),
        raw_reward_multiplier=float(self._raw_reward_multiplier),
        sparse_reward=bool(self._sparse_reward)))
    return len(nodes) - 1


class Clustering(AbstractTask):
  """Cluster sprites by the given factor distributions (inverse Davies-Bouldin index)."""

  def __init__(self, cluster_distribs, termination_threshold=2.5, terminate_bonus=0.0,
               sparse_reward=False, reward_range=10):
    self._cluster_distribs = cluster_distribs
    self._num_clusters = len(cluster_distribs)
    self._termination_threshold = termination_threshold
    self._terminate_bonus = terminate_bonus
    self._sparse_reward = sparse_reward
    self._reward_range = reward_range

  def _emit(self, nodes, filters):
    nodes.append(dict(
        kind='clustering', cluster_slots=[_slot(filters, d) for d in self._cluster_distribs],
        termination_threshold=float(self._termination_threshold),
        terminate_bonus=float(self._terminate_bonus), sparse_reward=bool(self._sparse_reward),
        reward_range=float(self._reward_range)))
    return len(nodes) - 1


class MetaAggregated(AbstractTask):
  """Combines subtasks: rewards by nan-sum/max/min/mean, termination by all/any."""
  REWARD_AGGREGATOR = {'sum': np.nansum, 'max': np.nanmax, 'min': np.nanmin, 'mean': np.nanmean}
  TERMINATION_CRITERION = {'all': np.all, 'any': np.any}

  def __init__(self, subtasks, reward_aggregator='sum', termination_criterion='all',
               terminate_bonus=0.0):
    if reward_aggregator not in _AGGREGATORS:
      raise ValueError('Unknown reward_aggregator. {} not in {}'.format(
          reward_aggregator, MetaAggregated.REWARD_AGGREGATOR))
    if termination_criterion not in _CRITERIA:
      raise ValueError('Unknown termination_criterion. {} not in {}'.format(
          termination_criterion, MetaAggregated.TERMINATION_CRITERION))
    self._subtasks = subtasks
    self._aggregator_name = reward_aggregator
    self._criterion_name = termination_criterion
    self._reward_aggregator = MetaAggregated.REWARD_AGGREGATOR[reward_aggregator]
    self._termination_criterion = MetaAggregated.TERMINATION_CRITERION[termination_criterion]
    self._terminate_bonus = terminate_bonus

  def _emit(self, nodes, filters):
    children = [t._emit(nodes, filters) for t in self._subtasks]
    nodes.append(dict(kind='meta', children=children, aggregator=self._aggregator_name,
                      criterion=self._criterion_name,
                      terminate_bonus=float(self._terminate_bonus)))
    return len(nodes) - 1
