"""Per-call plugin protocol on Python sprite lists, executed on the GPU.

The reference's `action_space.step(action, sprites, keep_in_frame)`,
`task.reward(sprites)`, `task.success(sprites)` and `renderer.render(sprites)`
(environment.py:94-102 call sites) operate on one env's sprite list.  Here they upload
the list as a one-env scene, run the corresponding entry point of the C-ABI
(swb_apply_action / swb_eval_task / swb_render) and, for actions, write the new
positions back into the `Sprite` objects.  Engines are cached per configuration.
There is deliberately no CPU implementation of this math in the package.
"""
import collections
import ctypes
import json

import numpy as np
import torch

from spriteworld_b200 import _native, constants, scene
from spriteworld_b200 import engine as engine_lib
from spriteworld_b200 import sprite_generators

_DUMMY_ACTION = dict(kind='select_move', scale=1.0, motion_cost=0.0)
_NO_TASK = [dict(kind='no_reward')]
_MAX_CACHED = 32
_engines = collections.OrderedDict()
_rasters = {}


def _engine(n_slots, action, nodes, keep_in_frame):
  key = json.dumps([n_slots, action, nodes, bool(keep_in_frame)], sort_keys=True)
  eng = _engines.get(key)
  if eng is None:
    eng = engine_lib.Engine(1, n_slots, 1, action, nodes, constants.SHAPES,
                            keep_in_frame=keep_in_frame, max_episode_length=2 ** 31 - 1)
    _engines[key] = eng
    while len(_engines) > _MAX_CACHED:
      _, old = _engines.popitem(last=False)
      for k in [k for k in _rasters if k[0] is old]:
        _rasters.pop(k).close()
      old.close()
  else:
    _engines.move_to_end(key)
  return eng


def _load(eng, sprites, filters=(), color_to_rgb=None):
  layout = sprite_generators.layout_from_sprite_lists([list(sprites)])
  batch = scene.arrays_from_layout(layout, eng.n_slots, filters, color_to_rgb)
  eng.upload_scenes(batch, [0], [0])
  eng.upload_state(pos_x=batch['x'], pos_y=batch['y'], cursor=[0], step_count=[0],
                   reset_next=[0])
  return batch


def _load_for_task(eng, sprites, filters):
  """Like _load, for task evaluation: needs of a sprite only what the reference's tasks touch,
  `.position` and -- when the task filters -- `.factors` (tasks.py:126-158,196-205), so the
  same duck-typed stand-ins work."""
  n, S = len(sprites), eng.n_slots
  batch = scene.empty_batch(1, S)
  for j, s in enumerate(sprites):
    k = S - n + j
    pos = np.asarray(s.position)
    batch['x'][0, k], batch['y'][0, k] = float(pos[0]), float(pos[1])
    batch['pos_f32'][0, k] = 1 if pos.dtype == np.float32 else 0
    batch['shape'][0, k] = 1                     # any occupied slot; the task never looks at it
    batch['m00'][0, k] = batch['m11'][0, k] = 1.0
    member = 0
    for bit, f in enumerate(filters):
      if f.contains(s.factors):
        member |= 1 << bit
    batch['member'][0, k] = member
  eng.upload_scenes(batch, [0], [0])
  eng.upload_state(pos_x=batch['x'], pos_y=batch['y'], cursor=[0], step_count=[0],
                   reset_next=[0])
  return batch


def _raise_for_status(status):
  if status & _native.ENV_CLUSTER_LABELS:
    raise ValueError('Number of labels is invalid for the Davies-Bouldin score: clustering '
                     'needs 2 <= populated clusters <= sprites - 1')
  if status & _native.ENV_CLUSTER_ZERODIV:
    raise ZeroDivisionError('float division by zero')
  if status & _native.ENV_BAD_ACTION:
    raise KeyError('bad Embodied action')
  if status & _native.ENV_SPAN_OVERFLOW:
    raise RuntimeError('renderer span table overflow')


def task_value(task, sprites):
  """(reward, success) of `task` on a Python sprite list."""
  nodes, filters = task.compile()
  task._filters_static()
  sprites = list(sprites)
  eng = _engine(max(1, len(sprites)), _DUMMY_ACTION, nodes, True)
  _load_for_task(eng, sprites, filters)
  _native.check(eng._lib.swb_eval_task(eng._h, eng._out, eng._stream()))
  torch.cuda.synchronize(eng.device)
  _raise_for_status(int(eng._status[0].item()))
  return float(eng._reward[0].item()), bool(eng._success[0].item())


def action_step(action_space, action, sprites, keep_in_frame):
  """Applies the action to the sprites (positions are written back); returns the cost."""
  sprites = list(sprites)
  cfg = action_space.compile()
  if not sprites:
    if cfg['kind'] == 'embodied':
      raise IndexError('list index out of range')   # sprites[-1] in the reference
  eng = _engine(max(1, len(sprites)), cfg, _NO_TASK, keep_in_frame)
  _load(eng, sprites)
  a = engine_lib.host_actions(cfg['kind'], np.reshape(action, (1, -1)))
  dtype = engine_lib.action_dtype(eng.action_kind, 1, a)
  t = torch.from_numpy(a).to(eng.device)
  _native.check(eng._lib.swb_apply_action(eng._h, ctypes.c_void_p(t.data_ptr()), dtype, eng._out,
                                          eng._stream()))
  state = eng.download_state()
  _raise_for_status(int(eng._status[0].item()))
  n, S = len(sprites), eng.n_slots
  for j, s in enumerate(sprites):
    k = S - n + j
    s._position[0] = state['pos_x'][0, k]
    s._position[1] = state['pos_y'][0, k]
  cost = float(eng._reward[0].item())
  if dtype == _native.DTYPE_F32:
    return np.float32(cost)
  return cost


def render(renderer, sprites):
  """(H, W, 3) uint8 frame of a Python sprite list."""
  eng = _engine(max(1, len(sprites)), _DUMMY_ACTION, _NO_TASK, True)
  _load(eng, sprites, (), renderer.color_to_rgb)
  key = (eng, renderer.width, renderer.height, renderer.anti_aliasing, renderer.bg_color)
  raster = _rasters.get(key)
  if raster is None:
    raster = engine_lib.Raster(eng, renderer.width, renderer.height, renderer.anti_aliasing,
                               renderer.bg_color)
    _rasters[key] = raster
  frames = eng.render(raster)
  eng.check_render()
  return frames[0].cpu().numpy()
