"""OpenAI-gym style front end (reference: spriteworld/gym_wrapper.py:42-135).

`GymWrapper(env)` adapts a single `Environment`; `gym`/`gymnasium` are imported lazily
and only for their `spaces` (neither is required: a minimal Box/Discrete/Dict/Tuple
stand-in is used when absent).  `VectorGymWrapper` is the same surface over a
`BatchedEnvironment`, returning device tensors.
"""
import numpy as np

from spriteworld_b200 import _dm_env as dm_env


def _spaces():
  for name in ('gymnasium', 'gym'):
    try:
      mod = __import__(name)
      return mod.spaces
    except ImportError:
      continue
  return _MiniSpaces


class _MiniSpaces(object):
  """Just enough of gym.spaces to describe Spriteworld's action/observation spaces."""

  class Box(object):

    def __init__(self, low, high, shape=None, dtype=np.float32):
      self.dtype = np.dtype(dtype)
      self.shape = tuple(shape) if shape is not None else np.shape(low)
      with np.errstate(invalid='ignore'):   # infinite bounds of integer boxes, as gym allows
        self.low = np.broadcast_to(np.asarray(low).astype(self.dtype), self.shape)
        self.high = np.broadcast_to(np.asarray(high).astype(self.dtype), self.shape)

    def sample(self):
      return np.random.uniform(self.low, self.high).astype(self.dtype)

    def contains(self, x):
      x = np.asarray(x)
      return x.shape == self.shape and bool(np.all(x >= self.low) and np.all(x <= self.high))

    def __eq__(self, other):
      return (isinstance(other, type(self)) and self.shape == other.shape and
              self.dtype == other.dtype and np.array_equal(self.low, other.low) and
              np.array_equal(self.high, other.high))

    __hash__ = None

  class Discrete(object):

    def __init__(self, n):
      self.n = int(n)
      self.shape = ()
      self.dtype = np.dtype(np.int64)

    def sample(self):
      return np.random.randint(self.n)

    def contains(self, x):
      return 0 <= int(x) < self.n

    def __eq__(self, other):
      return isinstance(other, type(self)) and self.n == other.n

    __hash__ = None

  class Dict(dict):

    def __init__(self, spaces):
      super().__init__(spaces)
      self.spaces = dict(spaces)

    def sample(self):
      return {k: s.sample() for k, s in self.spaces.items()}

  class Tuple(tuple):

    def __new__(cls, spaces):
      return super().__new__(cls, spaces)

    @property
    def spaces(self):
      return tuple(self)

    def sample(self):
      return tuple(s.sample() for s in self)


def _spec_to_space(spec):
  spaces = _spaces()
  if isinstance(spec, (list, tuple)):
    return spaces.Tuple([_spec_to_space(s) for s in spec])
  if isinstance(spec, dict):
    return spaces.Dict({k: _spec_to_space(v) for k, v in spec.items()})
  if hasattr(spec, 'num_values'):
    return spaces.Discrete(spec.num_values)
  if hasattr(spec, 'minimum'):
    low, high = np.broadcast_to(spec.minimum, spec.shape), np.broadcast_to(spec.maximum, spec.shape)
    if low.size and (low.min() != low.max() or high.min() != high.max()):
      # bounds per element (SpriteBoxes: x in [0, W], y in [0, H]) stay per element
      return spaces.Box(low=low, high=high, shape=spec.shape, dtype=spec.dtype)
    return spaces.Box(low=float(np.min(spec.minimum)), high=float(np.max(spec.maximum)),
                      shape=spec.shape, dtype=spec.dtype)
  if spec.dtype == np.uint8:
    return spaces.Box(low=0, high=255, shape=spec.shape, dtype=spec.dtype)
  if spec.dtype == bool:
    return spaces.Box(low=0.0, high=1.0, shape=spec.shape, dtype=np.float32)
  return spaces.Box(low=-np.inf, high=np.inf, shape=spec.shape, dtype=spec.dtype)


class GymWrapper(object):
  """gym.Env-like view of a dm_env style Environment (gym_wrapper.py:42-135).

  Observations are a dict with the keys of the environment's `renderers`; rendering always
  happens, so render() only returns the last 'image' observation."""
  metadata = {'render.modes': ['rgb_array']}

  def __init__(self, env):
    self._env = env
    self._last_render = None
    self._action_space = None
    self._observation_space = None
    # like the reference (:57-58): a reset sets up the observation specs -- and draws one
    # scene from init_sprites, which a seeded run must not skip
    self._env.reset()

  def __getattr__(self, name):
    return getattr(self._env, name)

  @property
  def observation_space(self):
    if self._observation_space is None:
      spaces = _spaces()
      components = {}
      for key, value in self._env.observation_spec().items():
        if hasattr(value, 'shape'):   # :67-68, whatever the dtype
          components[key] = spaces.Box(-np.inf, np.inf, value.shape, dtype=value.dtype)
        else:                          # per-sprite factor lists: no counterpart in the reference
          components[key] = _spec_to_space(value)
      self._observation_space = spaces.Dict(components)
    return self._observation_space

  @property
  def action_space(self):
    if self._action_space is None:
      self._action_space = _spec_to_space(self._env.action_spec())
    return self._action_space

  def _process_obs(self, obs):
    for k, v in obs.items():
      if isinstance(v, dict):         # SpriteCoverage, SpriteBoxes: a dict of arrays, as its space describes
        obs[k] = type(v)((kk, np.asarray(vv)) for kk, vv in v.items())
        continue
      obs[k] = np.asarray(v)
      if obs[k].dtype == bool:       # boolean 'success' becomes float32 (:83-85)
        obs[k] = obs[k].astype(np.float32)
      if k == 'image':
        self._last_render = obs[k]
    return obs

  def step(self, action):
    """-> (obs dict, reward, done, {'discount': ...}) (:91-110)."""
    ts = self._env.step(action)
    obs = self._process_obs(ts.observation)
    return obs, ts.reward or 0, ts.last(), {'discount': ts.discount}

  def reset(self):
    return self._process_obs(self._env.reset().observation)

  def render(self, mode='rgb_array'):
    del mode   # always the last RGB observation (:123-133)
    return self._last_render

  def close(self):
    if hasattr(self._env, 'close'):
      self._env.close()


class VectorGymWrapper(object):
  """(obs, reward, done, info) over a BatchedEnvironment; all values are device tensors."""

  def __init__(self, env):
    self._env = env
    self.num_envs = env.n_envs
    self.single_action_space = _spec_to_space(env.action_spec())
    self.single_observation_space = _spec_to_space(env.observation_spec())

  def reset(self):
    return self._env.reset().observation

  def step(self, actions):
    ts = self._env.step(actions)
    done = ts.step_type == int(dm_env.StepType.LAST)
    return ts.observation, ts.reward, done, {'discount': ts.discount, 'success': ts.success,
                                             'first': ts.step_type == int(dm_env.StepType.FIRST)}

  def close(self):
    self._env.close()
