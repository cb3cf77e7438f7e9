"""Task-free exploration: 1-6 random sprites, no reward, 10-step episodes
(reference: configs/cobra/exploration.py)."""

from spriteworld_b200 import factor_distributions as distribs
from spriteworld_b200 import sprite_generators as gen
from spriteworld_b200 import tasks
from spriteworld_b200.configs.cobra import common


def get_config(mode=None):
  del mode
  factors = distribs.Product([
      distribs.Continuous('x', 0.1, 0.9),
      distribs.Continuous('y', 0.1, 0.9),
      distribs.Discrete('shape', list(common.SHAPES)),
      distribs.Discrete('scale', [0.13]),
      distribs.Continuous('c0', 0., 1.),
      distribs.Continuous('c1', 0.3, 1.),
      distribs.Continuous('c2', 0.9, 1.),
  ])
  sprite_gen = gen.generate_sprites(factors, num_sprites=gen.uniform_count(1, 7))
  return common.config(tasks.NoReward(), sprite_gen, 10, __file__, None)
