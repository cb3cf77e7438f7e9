"""SpriteGlimpses and SpriteLayers: PILRenderer frames of views of some sprites.

Crop encoders, glimpse models and per-object reconstruction targets need each sprite large; an
egocentric, partially observable Embodied agent needs the scene around its body.  Both are the
scene seen through a window (x0, y0, x1, y1) of scene coordinates, drawn at the raster's full size
by the render kernel's window instantiation (Engine.render_windows), so no large frame is rendered
and cropped.  Slot decoders need each sprite's own pixels, and object-level saliency needs the scene
with a sprite taken out: both are the scene with only some slots drawn (Engine.render_windows'
`draw`), so no scene is edited and uploaded again.
"""
import numpy as np
import torch

from spriteworld_b200._dm_env import specs
from spriteworld_b200.renderers import abstract_renderer


class _SpriteViews(abstract_renderer.AbstractRenderer):
  """The renderer protocol of views of chosen slots, each a PILRenderer frame (same anti_aliasing,
  bg_color and color_to_rgb) through a window with some slots drawn.  Subclasses supply `views`:
  the windows and the slots drawn of each row's views."""

  def __init__(self, image_size, anti_aliasing, bg_color, color_to_rgb, slots):
    self._image_size = tuple(int(v) for v in image_size)
    self._anti_aliasing = int(anti_aliasing)
    if len(self._image_size) != 2 or min(self._image_size) < 1 or self._anti_aliasing < 1:
      raise ValueError('image_size must be (width, height) >= 1 and anti_aliasing >= 1, got %r, %r'
                       % (image_size, anti_aliasing))
    self._slots = None if slots is None else tuple(int(s) for s in slots)
    if self._slots is not None and not self._slots:
      raise ValueError('slots must name at least one slot, or be None for all')
    self._color_to_rgb = color_to_rgb
    self._bg_color = (0, 0, 0) if bg_color is None else tuple(int(c) for c in bg_color)
    self._num_views = 0

  @property
  def width(self):
    return self._image_size[0]

  @property
  def height(self):
    return self._image_size[1]

  @property
  def anti_aliasing(self):
    return self._anti_aliasing

  @property
  def bg_color(self):
    return self._bg_color

  @property
  def color_to_rgb(self):
    return self._color_to_rgb

  def slot_indices(self, n_slots):
    """The slots observed, as indices in [0, n_slots).  IndexError for one out of range."""
    if self._slots is None:
      return list(range(n_slots))
    out = []
    for s in self._slots:
      if not -n_slots <= s < n_slots:
        raise IndexError('slot %d out of range for %d slots' % (s, n_slots))
      out.append(s % n_slots)
    return out

  def views(self, pos_x, pos_y):
    """(windows float64 (n, V, 4), draw bool (n, V, n_slots) or None for every slot) of the rows
    whose positions are pos_x, pos_y (n, n_slots), both contiguous on their device.  Built with
    device fills and views only: a copy from pageable host memory would wait for the stream."""
    raise NotImplementedError

  def _spec(self, n_views):
    return specs.Array(shape=(n_views, self.height, self.width, 3), dtype=np.uint8)

  # -- plugin protocol ---------------------------------------------------------------
  def render(self, sprites=(), global_state=None):
    from spriteworld_b200 import _direct
    out = _direct.render_views(self, list(sprites))
    self._num_views = len(out)
    return out

  def observation_spec(self):
    """The spec of the last render's view count."""
    return self._spec(self._num_views)

  def render_batch(self, env, res):
    """Batched form: uint8 (n_envs, V, H, W, 3) views of every env, in a buffer of `env` that every
    step (and env.render()) overwrites, as it does the frames.  The step's status (res.status) gets
    each env's view status ORed in (ENV_BAD_WINDOW, ENV_SPAN_OVERFLOW)."""
    return env._render_views(self, status=None if res is None else res.status)

  def render_states(self, env, states):
    """The views of env records (EnvStates) without loading them, in a new tensor."""
    return env._render_views(self, states)

  def batch_observation_spec(self, env):
    return self._spec(len(self.slot_indices(env.engine.n_slots)))


class SpriteGlimpses(_SpriteViews):
  """Observes uint8 (V, H, W, 3) for image_size=(W, H): view v is the PILRenderer frame (same
  anti_aliasing, bg_color and color_to_rgb) of the window_size=(w, h) window centred on the live
  position (x, y) of slot slots[v]: x0 = x - 0.5 w, x1 = x + 0.5 w, and likewise y, in float64.
  The window is stretched over the whole raster: a world vertex wx goes to the canvas column
  trunc((wx - x0) * (aa W / (x1 - x0))), and everything else is PILRenderer's, so the window
  (0, 0, 1, 1) would draw PILRenderer's frame byte for byte.

  slots=None means every slot; negative indices count from the end, so slots=[-1] of an Embodied
  environment is the egocentric view of the body (the last, top-most slot).  An empty slot's view
  is the window around that slot's stored position: mask it with SpriteFactors' 'mask'.  In a
  BatchedEnvironment slots are engine slots (SpriteFactors.render_batch's); on a sprite list
  (`render`, the drop-in Environment) they index the list.  A view whose window has a vertex 2^30
  canvas pixels or more from its origin is all zeros, on every path; in a BatchedEnvironment the
  step's status (and observe()'s) then has ENV_BAD_WINDOW, and ENV_SPAN_OVERFLOW where a view
  overflowed the render kernel's span tables."""

  def __init__(self, image_size=(64, 64), anti_aliasing=1, bg_color=None, color_to_rgb=None,
               window_size=(0.25, 0.25), slots=None):
    super().__init__(image_size, anti_aliasing, bg_color, color_to_rgb, slots)
    self._window_size = tuple(float(v) for v in window_size)
    if len(self._window_size) != 2 or not all(np.isfinite(v) and v > 0 for v in self._window_size):
      raise ValueError('window_size must be (w, h), finite and > 0, got %r' % (window_size,))

  @property
  def window_size(self):
    return self._window_size

  def windows(self, pos_x, pos_y):
    """float64 (n, V, 4) windows centred on the slots of positions pos_x, pos_y (n, n_slots).  Built
    from views of the position columns, so that no index array is copied to the device (a copy from
    pageable host memory would wait for the stream)."""
    idx = self.slot_indices(pos_x.shape[1])
    if idx == list(range(pos_x.shape[1])):
      x, y = pos_x, pos_y
    else:
      x, y = torch.stack([pos_x[:, s] for s in idx], 1), torch.stack([pos_y[:, s] for s in idx], 1)
    x, y = x.to(torch.float64), y.to(torch.float64)
    hw, hh = 0.5 * self._window_size[0], 0.5 * self._window_size[1]
    return torch.stack([x - hw, y - hh, x + hw, y + hh], -1).contiguous()

  def views(self, pos_x, pos_y):
    return self.windows(pos_x, pos_y), None


class SpriteLayers(_SpriteViews):
  """Observes uint8 (V, H, W, 3) for image_size=(W, H): view v is the PILRenderer frame (same
  anti_aliasing, bg_color and color_to_rgb) of slot slots[v] drawn alone on the background, the
  frame PILRenderer draws of a sprite list holding that sprite only.  Amodal per-object RGB: where
  another sprite covers it, its own pixels show.  An empty slot's layer is the background.  At
  anti_aliasing 1, slot k's layer is its colour where SpriteCoverage's `cover` has bit k set and
  the background elsewhere.

  slots=None means every slot; negative indices count from the end.  In a BatchedEnvironment slots
  are engine slots (SpriteFactors.render_batch's); on a sprite list (`render`, the drop-in
  Environment) they index the list.  A layer whose sprite has a vertex 2^30 canvas pixels or more
  from the origin is all zeros, on every path; in a BatchedEnvironment the step's status (and
  observe()'s) then has ENV_BAD_WINDOW, and ENV_SPAN_OVERFLOW where a layer overflowed the render
  kernel's span tables.  Other subsets of the
  scene -- the scene without sprite k, a glimpse of one sprite without its occluders -- are
  BatchedEnvironment.render_windows(windows, renderer, draw=...)."""

  def __init__(self, image_size=(64, 64), anti_aliasing=1, bg_color=None, color_to_rgb=None, slots=None):
    super().__init__(image_size, anti_aliasing, bg_color, color_to_rgb, slots)

  def views(self, pos_x, pos_y):
    """The full-scene window (0, 0, 1, 1) for every view, and a one-hot draw: view v draws slot
    slots[v] only."""
    n, S = pos_x.shape
    idx = self.slot_indices(S)
    windows = torch.zeros((n, len(idx), 4), dtype=torch.float64, device=pos_x.device)
    windows[..., 2:] = 1.0
    eye = torch.eye(S, dtype=torch.bool, device=pos_x.device)
    one_hot = eye if idx == list(range(S)) else torch.stack([eye[s] for s in idx])
    return windows, one_hot.expand(n, len(idx), S).contiguous()
