"""Action spaces: how an agent's action moves sprites.

Same classes and constructor signatures as the reference's `spriteworld/action_spaces.py`
(SelectMove :27-111, DragAndDrop :114-137, Embodied :140-221).  As with tasks, an action
space here describes the computation (`compile()` -> kind/scale/motion_cost of
`swb_config`); hit tests and pose updates run in the step kernel.  The per-call protocol
method `step(action, sprites, keep_in_frame)` on a Python sprite list goes through a
one-env engine on the GPU (_direct.py) and writes the new positions back into the sprites.
"""
import numpy as np

from spriteworld_b200._dm_env import specs


class SelectMove(object):
  """Two clicks [x0, y0, x1, y1] in [0, 1]: the top-most sprite containing (x0, y0) moves by
  scale * ([x1, y1] - 0.5)."""
  _kind = 'select_move'

  def __init__(self, scale=1.0, motion_cost=0.0, noise_scale=None):
    self._scale = scale
    self._motion_cost = motion_cost
    self._noise_scale = noise_scale
    self._action_spec = specs.BoundedArray(shape=(4,), dtype=np.float32, minimum=0.0, maximum=1.0)

  def compile(self):
    return dict(kind=self._kind, scale=float(self._scale), motion_cost=float(self._motion_cost))

  def get_motion(self, action):
    return (action[2:] - 0.5) * self._scale

  def get_sprite_from_position(self, position, sprites):
    """Top-most sprite containing `position`, or None (action_spaces.py:77-81)."""
    for sprite in sprites[::-1]:
      if sprite.contains_point(position):
        return sprite
    return None

  def apply_noise_to_action(self, action):
    """Adds N(0, noise_scale) to the action if noise_scale is set (host side, np.random)."""
    if self._noise_scale:
      return action + np.random.normal(loc=0.0, scale=self._noise_scale, size=action.shape)
    return action

  def step(self, action, sprites, keep_in_frame):
    from spriteworld_b200 import _direct
    return _direct.action_step(self, self.apply_noise_to_action(np.asarray(action)), sprites,
                               keep_in_frame)

  def sample(self):
    return np.random.uniform(0., 1., size=(4,))

  def action_spec(self):
    return self._action_spec


class DragAndDrop(SelectMove):
  """Like SelectMove but the motion is scale * ([x1, y1] - [x0, y0])."""
  _kind = 'drag_and_drop'

  def get_motion(self, action):
    return (action[2:] - action[:2]) * self._scale


class Embodied(object):
  """sprites[-1] is the agent's body.  action = (carry in {0, 1}, direction in {0: up,
  1: left, 2: down, 3: right}); a carried sprite is the top-most one under the body."""
  _kind = 'embodied'

  def __init__(self, step_size=0.05, motion_cost=0.):
    self._step_size = step_size
    self._motion_cost = motion_cost
    self._action_spec = [specs.DiscreteArray(num_values=2, dtype=np.int64),
                         specs.DiscreteArray(num_values=4, dtype=np.int64)]
    d = self._step_size
    self.action_to_motion = {0: np.array([0, d]), 1: np.array([-d, 0]),
                             2: np.array([0, -d]), 3: np.array([d, 0])}

  def compile(self):
    return dict(kind=self._kind, scale=float(self._step_size),
                motion_cost=float(self._motion_cost))

  def get_body_sprite(self, sprites):
    return sprites[-1]

  def get_non_body_sprites(self, sprites):
    return sprites[:-1]

  def get_carried_sprite(self, sprites):
    """Top-most non-body sprite under the body's position, or None (action_spaces.py:180-185)."""
    body_position = self.get_body_sprite(sprites).position
    for sprite in self.get_non_body_sprites(sprites)[::-1]:
      if sprite.contains_point(body_position):
        return sprite
    return None

  def step(self, action, sprites, keep_in_frame):
    if action[1] not in self.action_to_motion:
      raise KeyError(action[1])
    from spriteworld_b200 import _direct
    return _direct.action_step(self, action, sprites, keep_in_frame)

  def sample(self):
    return [np.random.randint(0, 2), np.random.randint(0, 4)]

  def action_spec(self):
    return self._action_spec
