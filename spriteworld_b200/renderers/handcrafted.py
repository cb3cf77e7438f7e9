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


class _SpriteMaskRenderer(abstract_renderer.AbstractRenderer):
  """What SpriteMasks, SpriteCoverage, SoftSpriteMasks and SpriteBoxes share: image_size=(W, H) and
  anti_aliasing, whose canvas may not exceed 4095 pixels per side, drawn by the mask kernel as
  observation `_kind` (engine._render_sprite_masks); `_observation` shapes what it writes
  and `_spec(n)` describes that for n sprites."""

  def __init__(self, image_size=(64, 64), anti_aliasing=1):
    self._image_size = tuple(int(v) for v in image_size)
    self._anti_aliasing = int(anti_aliasing)
    if len(self._image_size) != 2 or min(self._image_size) < 1 or self._anti_aliasing < 1:
      raise ValueError('image_size must be (width, height) >= 1 and anti_aliasing >= 1, got %r, %r'
                       % (image_size, anti_aliasing))
    if self._anti_aliasing * max(self._image_size) > 4095:
      raise ValueError('the canvas (anti_aliasing * image_size) exceeds 4095 pixels per side')
    self._num_sprites = 0

  @property
  def width(self):
    return self._image_size[0]

  @property
  def height(self):
    return self._image_size[1]

  @property
  def anti_aliasing(self):
    return self._anti_aliasing

  @staticmethod
  def _observation(out, slots=slice(None)):
    """The observation of the engine's outputs `out`, keeping `slots` of any slot axis."""
    return out

  def render(self, sprites=(), global_state=None):
    from spriteworld_b200 import _direct
    self._num_sprites = len(sprites)
    return _direct.render_sprite_masks(self, list(sprites))

  def observation_spec(self):
    """The spec of the last render's sprite count (as SpriteFactors')."""
    return self._spec(self._num_sprites)

  def render_batch(self, env, res):
    """Batched form: the observation of every env, in buffers of `env` that every step (and
    env.render()) overwrites, as it does the frames."""
    return env._render_sprite_masks(type(self), self)

  def render_states(self, env, states):
    """The observation of env records (EnvStates) without loading them, in new tensors."""
    return env._render_sprite_masks(type(self), self, states)

  def batch_observation_spec(self, env):
    return self._spec(env.engine.n_slots)


class SpriteMasks(_SpriteMaskRenderer):
  """Instance masks: which sprite is visible at each pixel of a PILRenderer frame.

  Observes uint8 (H, W) for image_size=(W, H) (width, height as PILRenderer hands them to Pillow):
  k + 1 where sprite k is the top-most sprite covering the pixel's sample point, 0 where none does.
  Mask pixel (i, j) samples canvas pixel (aa j + aa//2, aa (H-1-i) + aa//2) of the aa W x aa H
  canvas PILRenderer draws on, with the same integer vertices and Pillow's fill rules, so at
  anti_aliasing=1 a frame is bg where the mask is 0 and the colour of sprite mask-1 elsewhere.
  Drawn by the mask kernel (csrc/swb_masks.cuh).

  Ids: in a BatchedEnvironment, slots of SpriteFactors.render_batch (empty slots, padded at the
  front, are never visible), so factors[f][e, mask - 1] is the visible sprite's factor; on a sprite
  list (`render`, the drop-in Environment), indices into the list.  Any anti_aliasing is accepted
  whose canvas sides stay within 4095 pixels."""

  _kind = 'masks'

  def _spec(self, n):
    return specs.Array(shape=(self.height, self.width), dtype=np.uint8)


class SpriteCoverage(_SpriteMaskRenderer):
  """Amodal sprite coverage: every sprite covering each pixel of a PILRenderer frame, hidden or not,
  with per-sprite visible and total pixel counts.

  Observes a dict for image_size=(W, H) and S sprites:
    'cover'    int32 (H, W): bit k is set where sprite k's Pillow polygon fill covers the pixel's
               sample point, whether or not a sprite above hides it (bit 31 is the sign bit).  The
               sample point, integer vertices and fill rules are SpriteMasks': canvas pixel
               (aa j + aa//2, aa (H-1-i) + aa//2) of the aa W x aa H canvas PILRenderer draws on.
    'visible'  int32 (S,): per sprite, the pixels where it is the top-most covering sprite, which
               is (SpriteMasks mask == k + 1).sum().
    'area'     int32 (S,): per sprite, the pixels whose bit k is set.
  So the SpriteMasks mask is the highest set bit + 1 (0 where cover is 0), visible <= area, and
  empty slots and sprites wholly out of frame have no bits and zero counts.  In Pillow, bit k's
  plane is sprite k drawn alone with fill 1 into a zero 'L' canvas of aa W x aa H, then
  resize((W, H), NEAREST) and np.flipud.  Drawn by the mask kernel's coverage mode
  (csrc/swb_masks.cuh), which also counts.

  Bits: in a BatchedEnvironment, S is n_slots and bit k is slot k of SpriteFactors.render_batch;
  on a sprite list (`render`, the drop-in Environment), bit i is sprites[i].  The same arguments
  and limits as SpriteMasks."""

  _kind = 'coverage'

  def _spec(self, n):
    i32, npx = np.iinfo(np.int32), self.height * self.width
    return collections.OrderedDict([
        ('cover', specs.BoundedArray(shape=(self.height, self.width), dtype=np.int32, minimum=i32.min,
                                     maximum=i32.max)),
        ('visible', specs.BoundedArray(shape=(n,), dtype=np.int32, minimum=0, maximum=npx)),
        ('area', specs.BoundedArray(shape=(n,), dtype=np.int32, minimum=0, maximum=npx))])

  @staticmethod
  def _observation(out, slots=slice(None)):
    cover, visible, area = out
    return collections.OrderedDict([('cover', cover), ('visible', visible[..., slots]), ('area', area[..., slots])])


class SoftSpriteMasks(_SpriteMaskRenderer):
  """Soft instance masks: how much of each pixel of a PILRenderer frame each sprite owns.

  Observes uint8 (S, H, W) for image_size=(W, H) and S sprites: soft[k, i, j] is the number of
  canvas pixels (aa j + u, aa (H-1-i) + v), u, v in [0, aa), of the aa W x aa H canvas PILRenderer
  draws on whose top-most covering sprite is sprite k, with SpriteMasks' integer vertices and
  Pillow fill rules.  So soft / aa**2 is the fraction of the pixel sprite k owns, aa**2 -
  soft.sum(0) counts the background's samples, and soft[k].sum() / aa**2 is sprite k's visible
  area in frame pixels, below pixel precision.  In Pillow: draw the label canvas (every sprite back
  to front, fill k + 1, into a zero 'L' image of aa W x aa H), L = np.flipud(canvas).reshape(H, aa,
  W, aa), soft[k] = (L == k + 1).sum((1, 3)).

  At anti_aliasing=1, soft[k] == (SpriteMasks mask == k + 1); at any aa the sample SpriteMasks reads
  is one of the aa**2, so mask == k + 1 implies soft[k] >= 1.  Empty slots and sprites out of frame
  or wholly hidden are zero.  This is a box filter of the label canvas: the frame is LANCZOS
  filtered, so it is not in general the composite sum_k rgb_k soft_k / aa**2.  Drawn by the mask
  kernel's soft mode (csrc/swb_masks.cuh).

  Slots: in a BatchedEnvironment, S is n_slots and k is slot k of SpriteFactors.render_batch; on a
  sprite list (`render`, the drop-in Environment), k is the list index.  SpriteMasks' arguments
  and limits, and anti_aliasing at most 15, so that the aa**2 samples of a pixel fit a byte."""

  _kind = 'soft'

  def __init__(self, image_size=(64, 64), anti_aliasing=1):
    super().__init__(image_size, anti_aliasing)
    if self._anti_aliasing > 15:
      raise ValueError('anti_aliasing %d exceeds 15: a pixel\'s anti_aliasing**2 sample count must '
                       'fit a uint8' % self._anti_aliasing)

  def _spec(self, n):
    return specs.BoundedArray(shape=(n, self.height, self.width), dtype=np.uint8, minimum=0,
                              maximum=self._anti_aliasing ** 2)

  @staticmethod
  def _observation(out, slots=slice(None)):
    return out[..., slots, :, :]


class SpriteBoxes(_SpriteMaskRenderer):
  """Sprite bounding boxes: where each sprite is visible and where it lies, hidden or not, in a
  PILRenderer frame, as pixel boxes with pixel counts.

  Observes a dict for image_size=(W, H) and S sprites:
    'visible_box'  int32 (S, 4): box(V_k), V_k the pixels (i, j) where sprite k is the top-most
                   covering sprite (SpriteMasks mask == k + 1).
    'amodal_box'   int32 (S, 4): box(A_k), A_k the pixels whose bit k of SpriteCoverage's 'cover'
                   is set, whether or not a sprite above hides them.
    'visible'      int32 (S,): |V_k|, SpriteCoverage's 'visible'.
    'area'         int32 (S,): |A_k|, SpriteCoverage's 'area'.
  box(P) = (min j, min i, max j + 1, max i + 1): half-open (x0, y0, x1, y1) in pixels of the
  observed (flipped) image, x the column and y the row from the top; (0, 0, 0, 0) for an empty P.
  For a non-empty plane that is torchvision.ops.masks_to_boxes(plane) + (0, 0, 1, 1).  So the
  visible box lies in the amodal box, visible <= area, a count is 0 exactly where its box is, and
  (x1 - x0) * (y1 - y0) >= the count.  Empty slots and sprites wholly out of frame have zero boxes
  and counts; wholly hidden sprites a zero visible box.  The sample point, integer vertices and
  fill rules are SpriteMasks'.  Reduced inside the mask kernel's box mode (csrc/swb_masks.cuh):
  no per-pixel output is written.

  Slots: in a BatchedEnvironment, S is n_slots and k is slot k of SpriteFactors.render_batch; on a
  sprite list (`render`, the drop-in Environment), k is the list index.  The same arguments and
  limits as SpriteMasks."""

  _kind = 'boxes'

  def _spec(self, n):
    W, H, npx = self.width, self.height, self.height * self.width
    box = specs.BoundedArray(shape=(n, 4), dtype=np.int32, minimum=0,
                             maximum=np.broadcast_to(np.array([W, H, W, H], np.int32), (n, 4)))
    return collections.OrderedDict([
        ('visible_box', box), ('amodal_box', box),
        ('visible', specs.BoundedArray(shape=(n,), dtype=np.int32, minimum=0, maximum=npx)),
        ('area', specs.BoundedArray(shape=(n,), dtype=np.int32, minimum=0, maximum=npx))])

  @staticmethod
  def _observation(out, slots=slice(None)):
    visible_box, amodal_box, visible, area = out
    return collections.OrderedDict([('visible_box', visible_box[..., slots, :]),
                                    ('amodal_box', amodal_box[..., slots, :]),
                                    ('visible', visible[..., slots]), ('area', area[..., slots])])


class GoalPositions(abstract_renderer.AbstractRenderer):
  """The goals of the task's sampled FindGoalPosition nodes: float64 (G, 2), (x, y) per goal slot
  (tasks.AbstractTask.goal_distributions order).  A task with constant goals only has G = 0."""

  def __init__(self):
    self._observation_spec = specs.Array(shape=(0, 2), dtype=np.float64)

  def render(self, sprites=(), global_state=None):
    # the one-env Environment refuses sampled goals, so its tasks have none
    return np.zeros((0, 2), np.float64)

  def observation_spec(self):
    return self._observation_spec

  def render_batch(self, env, res):
    """Batched form: float64 (n_envs, G, 2) device tensor of the goals of the scene each env is on."""
    return env.goal_tensor()

  def render_states(self, env, states):
    """The goals of env records (EnvStates): a new float64 (n, G, 2) tensor."""
    return env.goal_tensor(states)

  def batch_observation_spec(self, env):
    return specs.Array(shape=(env.n_goals, 2), dtype=np.float64)


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
