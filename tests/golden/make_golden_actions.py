"""Generates tests/golden/actions/actions.npz by RUNNING THE UNMODIFIED REFERENCE.

Run in the build container only (needs /root/reference):

    python tests/golden/make_golden_actions.py

The click action path of SelectMove and DragAndDrop, outside the narrow inputs of the episode
fixtures.  Two parts:

  single steps  `action_space.step(action, sprites, keep_in_frame)` of the reference on a list
                of three Sprites, sampled over action dtype (float32, float64), scale (0.25,
                0.5, 1, 3), motion cost (0, 0.25, 0.7, 1e-3), keep_in_frame and sprite position
                dtype, with actions uniform in [0, 1] and in [-3, 4], clicks on a sprite's
                centre and just inside a vertex, exact 0 / 0.5 / 1 with their nextafter
                neighbours, -0.0 and subnormals, NaN and +-inf in any subset of the four
                components, and +-1e30.  Per case: the cost (its exact float64 bits; a float32
                cost widened), which sprite moved (-1: none) and every position afterwards.
  episodes      short Environment episodes of the configs of action_configs.py, one per root
                task kind, with float64 actions of which some fling sprites to about +-10.
                'find_goal_noisy' draws SelectMove noise from np.random as the reference does;
                `ep_applied` is the action each step actually applied (after the noise), so a
                replay needs no np.random.  Frames (64x64, anti-aliasing 5) of every step that
                ends an episode.

Hit tests in the reference run through matplotlib's point-in-path, which oracle/refshim
replaces with a stand-in where matplotlib is absent.  This fixture therefore pins the motion,
cost, clipping and termination arithmetic of the action path, not matplotlib's hit test.

The NumPy, OpenBLAS and Pillow versions are stored in `meta`: the float64 cost is
np.linalg.norm, whose rounding is OpenBLAS's (DESIGN.md section 5).  SWB_GOLDEN_OUT redirects
the output directory (tests/test_golden_actions_reproducible.py).
"""
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402  (loads the reference)
import action_configs  # noqa: E402

OUT = os.environ.get('SWB_GOLDEN_OUT') or os.path.join(HERE, 'actions')

KINDS = ('select_move', 'drag_and_drop')
SCALES = (0.25, 0.5, 1.0, 3.0)
COSTS = (0.0, 0.25, 0.7, 1e-3)
MODES = ('uniform', 'wide', 'centre', 'vertex', 'special', 'nonfinite', 'large')
N_SLOTS = 3
SHAPES = sorted(mg.constants.SHAPES)


def versions():
  import PIL
  blas = np.show_config(mode='dicts')['Build Dependencies']['blas']
  return dict(numpy=np.__version__, blas=blas.get('name'), blas_version=blas.get('version'),
              openblas_config=blas.get('openblas configuration'), pillow=PIL.__version__)


def _specials(dt):
  one, half, zero = dt(1), dt(0.5), dt(0)
  tiny = np.finfo(dt).smallest_subnormal
  vals = [zero, -zero, half, one, tiny, -tiny]
  for v in (zero, half, one):
    vals += [np.nextafter(v, dt(-2)), np.nextafter(v, dt(2))]
  return np.array(vals, dt)


def _action(mode, dt, rng, sprites):
  a = rng.uniform(0, 1, 4)
  if mode == 'wide':
    a = rng.uniform(-3, 4, 4)
  elif mode in ('centre', 'vertex', 'nonfinite'):
    s = sprites[rng.randint(len(sprites))]
    p = s.position.astype(np.float64)
    if mode == 'vertex':
      v = s._centered_path.vertices
      p = p + 0.98 * v[rng.randint(len(v))]
    a[:2] = p
  a = a.astype(dt)
  if mode == 'special':
    sp = _specials(dt)
    a = sp[rng.randint(len(sp), size=4)]
  elif mode == 'nonfinite':
    mask = rng.randint(1, 16)                  # any non-empty subset of the components
    for i in range(4):
      if mask >> i & 1:
        a[i] = dt(rng.choice([np.nan, np.inf, -np.inf]))
  elif mode == 'large':
    i = rng.randint(4)
    a[i] = dt(rng.choice([1e30, -1e30]))
  return a


def single_steps(seed=31, reps=12):
  rng = np.random.RandomState(seed)
  rows = []
  for f32 in (True, False):
    dt = np.float32 if f32 else np.float64
    for scale in SCALES:
      for cost in COSTS:
        for keep in (True, False):
          for mode in MODES:
            for _ in range(reps):
              kind = KINDS[rng.randint(2)]
              pos_f32 = rng.rand(N_SLOTS) < 0.5
              sprites = []
              for k in range(N_SLOTS):
                x, y = rng.uniform(0.15, 0.85, 2)
                if pos_f32[k]:
                  x, y = np.float32(x), np.float32(y)
                sprites.append(mg.sprite_lib.Sprite(
                    x=x, y=y, shape=str(SHAPES[rng.randint(len(SHAPES))]),
                    angle=int(rng.choice([0, 30, 45, 77])),
                    scale=float(rng.choice([0.1, 0.2, 0.3]))))
              a = _action(mode, dt, rng, sprites)
              before = mg.positions(sprites, N_SLOTS)
              moved = []
              for k, s in enumerate(sprites):
                s.move = (lambda motion, keep_in_frame=False, _s=s, _k=k:
                          (moved.append(_k), type(_s).move(_s, motion, keep_in_frame)))
              space = (mg.action_spaces.SelectMove if kind == 'select_move'
                       else mg.action_spaces.DragAndDrop)(scale=scale, motion_cost=cost)
              with np.errstate(all='ignore'):
                c = space.step(np.array(a), sprites, keep)
              assert isinstance(c, dt) and len(moved) <= 1, (type(c), moved)
              rows.append(dict(
                  kind=KINDS.index(kind), scale=scale, motion_cost=cost, keep=keep, f32=f32,
                  mode=MODES.index(mode), action=a.astype(np.float64), before=before,
                  pos_f32=pos_f32, shape=[mg.SHAPE_IDS[s.shape] for s in sprites],
                  angle=[float(s.angle) for s in sprites],
                  sprite_scale=[float(s.scale) for s in sprites],
                  cost=np.float64(c), moved=moved[0] if moved else -1,
                  after=mg.positions(sprites, N_SLOTS)))
  out = {}
  for k in rows[0]:
    out['ss_' + k] = np.array([r[k] for r in rows])
  out['ss_pos_f32'] = out['ss_pos_f32'].astype(np.uint8)
  out['ss_shape'] = out['ss_shape'].astype(np.uint8)
  for k in ('kind', 'mode', 'keep', 'f32'):
    out['ss_' + k] = out['ss_' + k].astype(np.uint8)
  out['ss_moved'] = out['ss_moved'].astype(np.int8)
  return out


def _reference_modules():
  ref = sys.modules['spriteworld']
  return types.SimpleNamespace(
      action_spaces=ref.action_spaces, tasks=ref.tasks,
      factor_distributions=ref.factor_distributions,
      sprite_generators=ref.sprite_generators, renderers=ref.renderers)


def episodes(n_envs=3, n_steps=24, seed=41):
  """Environment episodes; per config c: `ep<c>_*` arrays, laid out as in episodes_<cfg>.npz,
  plus `applied` (the noisy actions) and the frames of the steps that end an episode."""
  sw = _reference_modules()
  out = {}
  names = []
  for ci, (name, make) in enumerate(action_configs.episode_configs(sw)):
    names.append(name)
    rng = np.random.RandomState(seed + ci)
    scene_log = [[] for _ in range(n_envs)]
    envs, applied_log = [], [None] * n_envs
    meta = None
    for e in range(n_envs):
      np.random.seed(2000 + 10 * ci + e)
      cfg = make()
      filters = mg.collect_filters(cfg['task'])
      rend = cfg['renderers']['image']
      base = cfg['init_sprites']

      def logged_gen(_base=base, _log=scene_log[e], _f=filters, _r=rend):
        sprites = _base()
        _log.append(mg.sprites_to_arrays(sprites, N_SLOTS + 1, _f, _r._color_to_rgb))
        return sprites

      cfg['init_sprites'] = logged_gen
      space = cfg['action_space']
      noise = space._noise_scale

      def logged_noise(action, _f=space.apply_noise_to_action, _e=e):
        applied_log[_e] = _f(action)
        return applied_log[_e]

      space.apply_noise_to_action = logged_noise
      envs.append(mg.environment.Environment(**cfg))
      if meta is None:
        kind = 'drag_and_drop' if isinstance(space, sw.action_spaces.DragAndDrop) else 'select_move'
        meta = dict(name=name, n_slots=N_SLOTS + 1, noise_scale=noise,
                    action=dict(kind=kind, scale=float(space._scale),
                                motion_cost=float(space._motion_cost)),
                    keep_in_frame=bool(cfg['keep_in_frame']),
                    max_episode_length=int(cfg['max_episode_length']),
                    nodes=mg.task_nodes(cfg['task'], filters), n_filters=len(filters),
                    width=action_configs.FRAME[0], height=action_configs.FRAME[1],
                    aa=action_configs.AA, bg=[0, 0, 0])
    S = N_SLOTS + 1
    actions = rng.uniform(0, 1, (n_steps, n_envs, 4))
    applied = np.full((n_steps, n_envs, 4), np.nan)
    pos = np.zeros((n_steps, n_envs, S, 2))
    reward = np.zeros((n_steps, n_envs))
    step_type = np.zeros((n_steps, n_envs), np.int8)
    success = np.zeros((n_steps, n_envs), np.uint8)
    scene_idx = np.zeros((n_steps, n_envs), np.int32)
    frames, frame_at = [], []
    for t in range(n_steps):
      for e, env in enumerate(envs):
        u = rng.rand()
        if u < 0.4 and env._sprites:          # a click on a sprite, moved within the frame
          s = env._sprites[rng.randint(len(env._sprites))]
          actions[t, e, :2] = s.position + rng.uniform(-0.02, 0.02, 2)
        elif u < 0.7 and env._sprites:        # a click on a sprite that flings it far out
          s = env._sprites[rng.randint(len(env._sprites))]
          actions[t, e, :2] = s.position
          actions[t, e, 2:] = rng.uniform(-3, 4, 2)
        applied_log[e] = None
        with np.errstate(all='ignore'):
          ts = env.step(actions[t, e].copy())
        if applied_log[e] is not None:
          applied[t, e] = applied_log[e]
        pos[t, e] = mg.positions(env._sprites, S)
        reward[t, e] = 0.0 if ts.reward is None else float(ts.reward)
        step_type[t, e] = int(ts.step_type)
        success[t, e] = bool(env.success())
        scene_idx[t, e] = len(scene_log[e]) - 1
        if ts.last() and np.isfinite(pos[t, e]).all():
          frames.append(ts.observation['image'])
          frame_at.append((t, e))
    p = 'ep%d_' % ci
    out.update({p + 'meta': np.array(json.dumps(meta)), p + 'actions': actions,
                p + 'applied': applied, p + 'pos': pos, p + 'reward': reward,
                p + 'step_type': step_type, p + 'success': success, p + 'scene_idx': scene_idx,
                p + 'frames': np.array(frames, np.uint8).reshape(-1, 64, 64, 3),
                p + 'frame_at': np.array(frame_at, np.int32).reshape(-1, 2)})
    n_scenes = max(len(l) for l in scene_log)
    for f in mg.FIELDS:
      proto = scene_log[0][0][f]
      arr = np.zeros((n_envs, n_scenes) + proto.shape, proto.dtype)
      for e in range(n_envs):
        for k, sc in enumerate(scene_log[e]):
          arr[e, k] = sc[f]
      out[p + 'scene_' + f] = arr
    print('%s: %d LAST, %d frames, %d scenes max' % (name, (step_type == 2).sum(), len(frames),
                                                     n_scenes))
  out['ep_names'] = np.array(names)
  return out


def main():
  blob = dict(meta=np.array(json.dumps(dict(versions(), kinds=KINDS, modes=MODES,
                                            n_slots=N_SLOTS))))
  blob.update(single_steps())
  blob.update(episodes())
  blob.update(mg.shapes_blob())
  os.makedirs(OUT, exist_ok=True)
  path = os.path.join(OUT, 'actions.npz')
  np.savez_compressed(path, **blob)
  print('actions.npz: %d single steps, %.0f KB' % (len(blob['ss_cost']),
                                                   os.path.getsize(path) / 1024))


if __name__ == '__main__':
  main()
