"""Non-pixel observations derived from the sprite state.

Reference: renderers/handcrafted.py:29-131 (SpriteFactors, SpritePassthrough, Success).
In the batched Environment these read the struct-of-arrays state directly
(`render_batch`); `render(sprites, global_state)` keeps the per-env protocol.
"""
import collections

import numpy as np

from spriteworld_b200 import constants
from spriteworld_b200 import sprite as sprite_lib
from spriteworld_b200._dm_env import specs
from spriteworld_b200.renderers import abstract_renderer


class SpritePassthrough(abstract_renderer.AbstractRenderer):
  """Returns the sprites unchanged."""

  def __init__(self):
    self._observation_spec = None

  def render(self, sprites=(), global_state=None):
    self._observation_spec = specs.Array(shape=(len(sprites),), dtype=object)
    return sprites

  def observation_spec(self):
    return self._observation_spec


class SpriteFactors(abstract_renderer.AbstractRenderer):
  """List of per-sprite factor dicts (shape as ShapeType id), optionally a subset."""

  def __init__(self, factors=('x', 'y', 'shape', 'angle', 'scale', 'c0', 'c1', 'c2', 'x_vel',
                              'y_vel')):
    if not set(factors).issubset(set(sprite_lib.FACTOR_NAMES)):   # handcrafted.py:41-43
      raise ValueError('Factors have to belong to {}.'.format(sprite_lib.FACTOR_NAMES))
    self._num_sprites = None
    self._factors = factors
    self._per_object_spec = {f: specs.Array(shape=(), dtype=np.float32) for f in factors}

  def render(self, sprites=(), global_state=None):
    self._num_sprites = len(sprites)

    def value(sprite, name):
      if name == 'shape':
        return np.float32(int(constants.ShapeType[sprite.shape]))
      return np.float32(getattr(sprite, name))

    return [collections.OrderedDict((f, value(s, f)) for f in self._factors) for s in sprites]

  def observation_spec(self):
    return [self._per_object_spec for _ in range(self._num_sprites)]

  def render_batch(self, env, res):
    """Batched form: dict factor -> float32 (n_envs, n_slots) device tensor, plus 'mask'
    (slot occupied).  Empty slots are padded at the front (the last slot is top-most)."""
    return env.factor_tensors(self._factors)

  def render_states(self, env, states):
    """render_batch of env records (EnvStates) instead of the live envs: dict factor -> float32
    (n, n_slots) device tensor plus 'mask', what render_batch would return after
    env.load_envs(states)."""
    return env.factor_tensors(self._factors, states)

  def batch_observation_spec(self, env):
    n = env.engine.n_slots
    spec = {f: specs.Array(shape=(n,), dtype=np.float32) for f in self._factors}
    spec['mask'] = specs.Array(shape=(n,), dtype=bool)
    return spec


class Success(abstract_renderer.AbstractRenderer):
  """global_state['success'] as an observation."""

  def __init__(self):
    self._observation_spec = specs.Array(shape=(), dtype=bool)

  def render(self, sprites=(), global_state=None):
    return global_state['success']

  def render_batch(self, env, res):
    return res.success.to(bool)

  def observation_spec(self):
    return self._observation_spec
