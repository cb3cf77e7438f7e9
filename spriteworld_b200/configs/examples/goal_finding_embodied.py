"""Goal finding with an embodied agent: 1-3 targets and 1-3 distractors in random z-order,
plus the agent's body (a small white circle) always in front
(reference: configs/examples/goal_finding_embodied.py)."""
import os

from spriteworld_b200 import action_spaces
from spriteworld_b200 import factor_distributions as distribs
from spriteworld_b200 import renderers as sw_renderers
from spriteworld_b200 import sprite_generators as gen
from spriteworld_b200 import tasks

TERMINATE_DISTANCE = 0.075
NUM_TARGETS = gen.uniform_count(1, 4)
NUM_DISTRACTORS = gen.uniform_count(1, 4)


def get_config(mode=None):
  del mode
  position = [distribs.Continuous('x', 0.1, 0.9), distribs.Continuous('y', 0.1, 0.9)]
  shared = distribs.Product(position + [
      distribs.Discrete('shape', ['square', 'triangle', 'circle']),
      distribs.Discrete('scale', [0.13]),
      distribs.Continuous('c1', 0.3, 1.),
      distribs.Continuous('c2', 0.9, 1.),
  ])
  target_hue = distribs.Continuous('c0', 0., 0.4)
  distractor_hue = distribs.Continuous('c0', 0.5, 0.9)
  objects = gen.shuffle(gen.chain_generators(
      gen.generate_sprites(distribs.Product([target_hue, shared]), num_sprites=NUM_TARGETS),
      gen.generate_sprites(distribs.Product([distractor_hue, shared]),
                           num_sprites=NUM_DISTRACTORS)))
  body = distribs.Product(position + [
      distribs.Discrete('shape', ['circle']),
      distribs.Discrete('scale', [0.07]),
      distribs.Discrete('c0', [1.]),
      distribs.Discrete('c1', [0.]),
      distribs.Discrete('c2', [1.]),
  ])
  sprite_gen = gen.chain_generators(objects, gen.generate_sprites(body, num_sprites=1))
  return {
      'task': tasks.FindGoalPosition(filter_distrib=target_hue,
                                     terminate_distance=TERMINATE_DISTANCE),
      'action_space': action_spaces.Embodied(step_size=0.05),
      'renderers': {'image': sw_renderers.PILRenderer(
          image_size=(64, 64), anti_aliasing=5,
          color_to_rgb=sw_renderers.color_maps.hsv_to_rgb)},
      'init_sprites': sprite_gen,
      'max_episode_length': 50,
      'metadata': {'name': os.path.basename(__file__)},
  }
