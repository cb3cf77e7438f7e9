"""Environment configs of the whole-step episodes in tests/golden/actions/actions.npz.

`episode_configs(sw)` builds them from either package: `sw` is a namespace with the modules
action_spaces, tasks, factor_distributions, sprite_generators and renderers, taken from the
reference (make_golden_actions.py) or from spriteworld_b200 (tests/test_gpu_actions.py, which
swaps the scene generator for a replay of the recorded scenes and drops the action noise in
favour of the recorded noisy actions).

Every config has motion cost 0.7, keep_in_frame off and 64x64 frames at anti-aliasing 5.
Scales of 1 to 3 let a click in [-3, 4] fling a sprite to a position of about +-10.
"""

FRAME = (64, 64)
AA = 5


def _renderer(sw):
  return {'image': sw.renderers.PILRenderer(image_size=FRAME, anti_aliasing=AA,
                                            color_to_rgb=sw.renderers.color_maps.hsv_to_rgb)}


def _factors(sw, c0=(0., 1.)):
  d = sw.factor_distributions
  return d.Product([
      d.Continuous('x', 0.2, 0.8), d.Continuous('y', 0.2, 0.8),
      d.Discrete('shape', ['square', 'triangle', 'star_5', 'spoke_4', 'circle']),
      d.Continuous('scale', 0.1, 0.25), d.Discrete('angle', [0, 30, 77]),
      d.Continuous('c0', c0[0], c0[1]), d.Continuous('c1', 0.3, 1.),
      d.Continuous('c2', 0.9, 1.),
  ])


def episode_configs(sw, noise_scale=0.05):
  """[(name, make_config)]: one config per root task kind.  `noise_scale` is the
  SelectMove noise of the 'find_goal_noisy' config (None: no noise)."""
  d, t, a, g = sw.factor_distributions, sw.tasks, sw.action_spaces, sw.sprite_generators

  def find_goal_noisy():
    return dict(
        task=t.FindGoalPosition(filter_distrib=d.Continuous('c0', 0., 0.6),
                                goal_position=(0.4, 0.6), terminate_distance=0.1,
                                terminate_bonus=2.0),
        action_space=a.SelectMove(scale=3.0, motion_cost=0.7, noise_scale=noise_scale),
        renderers=_renderer(sw), init_sprites=g.generate_sprites(_factors(sw), num_sprites=4),
        keep_in_frame=False, max_episode_length=8)

  def clustering():
    lo, hi = (0., 0.5), (0.5, 1.)
    return dict(
        task=t.Clustering([d.Continuous('c0', *lo), d.Continuous('c0', *hi)],
                          termination_threshold=4.0),
        action_space=a.DragAndDrop(scale=1.0, motion_cost=0.7),
        renderers=_renderer(sw),
        init_sprites=g.chain_generators(
            g.generate_sprites(_factors(sw, lo), num_sprites=2),
            g.generate_sprites(_factors(sw, hi), num_sprites=2)),
        keep_in_frame=False, max_episode_length=8)

  def meta():
    return dict(
        task=t.MetaAggregated([
            t.FindGoalPosition(filter_distrib=d.Continuous('c0', 0., 0.5),
                               goal_position=(0.3, 0.6), terminate_distance=0.2),
            t.FindGoalPosition(filter_distrib=d.Continuous('c0', 0.5, 1.),
                               goal_position=(0.7, 0.4), sparse_reward=True),
        ], reward_aggregator='mean', termination_criterion='all', terminate_bonus=1.5),
        action_space=a.SelectMove(scale=3.0, motion_cost=0.7),
        renderers=_renderer(sw), init_sprites=g.generate_sprites(_factors(sw), num_sprites=4),
        keep_in_frame=False, max_episode_length=8)

  def no_reward():
    return dict(
        task=t.NoReward(), action_space=a.DragAndDrop(scale=1.5, motion_cost=0.7),
        renderers=_renderer(sw), init_sprites=g.generate_sprites(_factors(sw), num_sprites=3),
        keep_in_frame=False, max_episode_length=8)

  return [('find_goal_noisy', find_goal_noisy), ('clustering', clustering), ('meta', meta),
          ('no_reward', no_reward)]
