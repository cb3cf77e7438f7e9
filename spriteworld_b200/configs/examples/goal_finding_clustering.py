"""Clustering by shape combined with two goal-finding subtasks, RGB integer colours,
rotated stars and spokes (reference: configs/examples/goal_finding_clustering.py)."""
import os

from spriteworld_b200 import action_spaces
from spriteworld_b200 import factor_distributions as distribs
from spriteworld_b200 import renderers as sw_renderers
from spriteworld_b200 import sprite_generators as gen
from spriteworld_b200 import tasks


def _int(key, lo, hi, dtype='int32'):
  return distribs.Continuous(key, lo, hi, dtype=dtype)


def get_config(mode='train'):
  pose = distribs.Product([distribs.Continuous('x', 0.1, 0.9), distribs.Continuous('y', 0.1, 0.9),
                           _int('angle', 0, 360)])
  held_out_scale = distribs.Continuous('scale', 0.08, 0.12)
  green_blue = distribs.Product([_int('c1', 64, 256), _int('c2', 64, 256)])
  if mode == 'train':
    goal_scale = distribs.SetMinus(distribs.Continuous('scale', 0.05, 0.15), held_out_scale)
    cluster_colors = distribs.Product([_int('c0', 128, 256), green_blue])
  elif mode == 'test':
    goal_scale = held_out_scale
    cluster_colors = distribs.Product([_int('c0', 0, 128), green_blue])
  else:
    raise ValueError('Invalid mode {}. Mode must be "train" or "test".'.format(mode))

  generators = []
  cluster_shapes = [distribs.Discrete('shape', [s]) for s in ['triangle', 'square', 'pentagon']]
  for shape in cluster_shapes:
    factors = distribs.Product([pose, cluster_colors, shape,
                                distribs.Continuous('scale', 0.08, 0.12)])
    generators.append(gen.generate_sprites(factors, num_sprites=2))

  goal_colors = [
      distribs.Product([_int('c0', 192, 256), _int('c1', 0, 128), _int('c2', 64, 128)]),
      distribs.Product([_int('c0', 0, 128), _int('c1', 192, 256), _int('c2', 64, 128)]),
  ]
  goal_positions = [(0., 0.5), (1., 0.5)]
  goal_shapes = distribs.Discrete('shape', ['spoke_4', 'star_4'])
  for colors in goal_colors:
    factors = distribs.Product([pose, goal_scale, goal_shapes, colors])
    generators.append(gen.generate_sprites(factors,
                                           num_sprites=gen.uniform_count(1, 3)))

  distractor = distribs.Product([
      pose, distribs.Discrete('shape', ['circle']), _int('c0', 64, 256, 'uint8'),
      _int('c1', 64, 256, 'uint8'), _int('c2', 64, 256, 'uint8'),
      distribs.Continuous('scale', 0.08, 0.12)])
  generators.append(gen.generate_sprites(distractor,
                                         num_sprites=gen.uniform_count(0, 3)))
  sprite_gen = gen.shuffle(gen.chain_generators(*generators))

  subtasks = [tasks.Clustering(cluster_shapes, terminate_bonus=0., reward_range=10.)]
  for colors, goal in zip(goal_colors, goal_positions):
    subtasks.append(tasks.FindGoalPosition(
        distribs.Product([colors, goal_shapes]), goal_position=goal, weights_dimensions=(1, 0),
        terminate_distance=0.15, raw_reward_multiplier=30))
  return {
      'task': tasks.MetaAggregated(subtasks, reward_aggregator='sum',
                                   termination_criterion='all'),
      'action_space': action_spaces.SelectMove(scale=0.5),
      'renderers': {'image': sw_renderers.PILRenderer(image_size=(64, 64), anti_aliasing=5)},
      'init_sprites': sprite_gen,
      'max_episode_length': 50,
      'metadata': {'name': os.path.basename(__file__), 'mode': mode},
  }
