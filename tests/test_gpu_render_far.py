"""Render kernel (csrc/swb_render.cuh) on sprites whose canvas coordinates go far past int16,
against the CPU oracle, bit for bit.

Phase A packs each edge's row range into 16 bits (ymin, ymax clamped to [-32768, 32767]) and keeps
horizontal edges and output regions as shorts; the corner-join groups, the doubling of crossings
on interior rows and phase B's row tests read the clamped values.  The scenes here reach what that
packing special-cases: edges that cross the canvas from beyond +-32768 rows, horizontal edges on
a canvas row whose ends lie beyond +-32768 columns, corner joins on a canvas row whose edges end
beyond int16, sprites wholly off the canvas far out on every side, and sprites that cover every
canvas row, so that phase B takes them in chunks.  tests/test_oracle_raster_far.py pins the oracle
to Pillow on such scenes and checks that they reach each of those cases.

  * every write-out of the render kernel (render, step, step_host, step_gather into two targets)
    into sentinel-guarded buffers, aligned and at an odd address, on narrow (aa <= 5) and wide
    rasters: each env is flagged exactly as tests/span_overflow.py restates it, or its frame is
    the oracle's;
  * the same scenes as env records (render_states, the records instantiation);
  * at anti_aliasing 1, frames against the mask kernel: background where the mask is 0, the
    sprite's colour elsewhere;
  * episodes of SelectMove and DragAndDrop with keep_in_frame off whose sprites the velocity update
    and clicks carry past 2^15 canvas units and on, against oracle.BatchOracle at every step.
"""
import numpy as np
import pytest

from oracle import oracle
from tests import fixtures, mask_oracle
from tests import test_gpu_render_geometry as geo

gpu = pytest.mark.gpu

INT16 = 1 << 15
LIMIT = 1 << 30             # canvas coordinates stay below this: x1 - x0 fits in int32
CONVEX = geo.CONVEX
ALL_SHAPES = geo.CONVEX + geo.CONCAVE
WIDE_AA = 6                 # rasters of anti_aliasing 6 and more render in render_kernel<., true>

# (id, W, H, aa, bg, S, E, concave, scene), as in test_gpu_render_geometry.CASES.  'huge': sprites
# 40k to 120k canvas rows across whose outlines cross the canvas (as mask_oracle.huge_scene_arrays);
# 'far': sprites up to 2^29 canvas units across, crossing the canvas, touching it at a corner
# or a horizontal edge, wholly off it on every side, and a few ordinary ones in front.
CASES = [
    # narrow rasters
    ('huge_w64h64a5_s9', 64, 64, 5, (0, 0, 0), 9, 12, False, 'huge'),
    ('far_w64h64a5_s32', 64, 64, 5, (255, 255, 255), 32, 6, True, 'far'),
    ('huge_w33h17a3_s1', 33, 17, 3, (90, 90, 90), 1, 24, True, 'huge'),
    ('far_w33h17a3_s9', 33, 17, 3, (10, 200, 30), 9, 16, False, 'far'),
    ('huge_w101h30a2_s32', 101, 30, 2, (40, 40, 40), 32, 6, True, 'huge'),
    ('far_w101h30a2_s1', 101, 30, 2, (0, 0, 255), 1, 24, False, 'far'),
    ('huge_w41h819a5_s9', 41, 819, 5, (5, 6, 7), 9, 4, True, 'huge'),          # canvas 205 x 4095
    ('far_w41h819a5_s32', 41, 819, 5, (5, 6, 7), 32, 3, False, 'far'),
    # wide rasters
    ('huge_w64h64a10_s32', 64, 64, 10, (0, 0, 0), 32, 4, False, 'huge'),
    ('far_w64h64a10_s9', 64, 64, 10, (255, 0, 0), 9, 8, True, 'far'),
    ('huge_w315h8a13_s9', 315, 8, 13, (5, 6, 7), 9, 6, True, 'huge'),          # canvas 4095 x 104
    ('far_w315h8a13_s1', 315, 8, 13, (5, 6, 7), 1, 16, False, 'far'),
    ('huge_w64h8a20_s1', 64, 8, 20, (0, 0, 255), 1, 16, True, 'huge'),
    ('far_w64h8a20_s32', 64, 8, 20, (0, 0, 0), 32, 4, False, 'far'),
]


# ---------------------------------------------------------------------------------------
# scenes
# ---------------------------------------------------------------------------------------

def _shape_verts(shape_id):
  from spriteworld_b200 import constants
  return np.asarray(constants.SHAPES[geo.oracle_name(int(shape_id))], np.float64)


def _centred(v, scale, angle):
  m00, m01, m10, m11 = oracle.centred_matrix(scale, angle)
  return np.stack([(m00 * v[:, 0] + m01 * v[:, 1]) + 0.0, (m10 * v[:, 0] + m11 * v[:, 1]) + 0.0], 1)


def _corner_angle(rng, v, k):
  """An angle (degrees) at which vertex k of shape v is a corner both of whose edges leave it
  downwards (larger y) with slopes of one sign, or None if none of 64 tries is."""
  for _ in range(64):
    ang = rng.uniform(0, 360)
    c = _centred(v, 1.0, ang)
    d0, d1 = c[k - 1] - c[k], c[(k + 1) % len(c)] - c[k]
    if d0[1] > 0 and d1[1] > 0 and d0[0] * d1[0] > 0:
      return ang
  return None


def _place(a, e, s, shape, scale, angle, rgb):
  a['shape'][e, s], a['scale'][e, s], a['angle'][e, s] = shape, scale, angle
  a['rgb'][e, s] = rgb


KINDS = ('cross', 'corner', 'flat', 'off')


def far_scene_arrays(rng, E, S, CW, CH, pool, reach, kinds=KINDS, side=None, p_small=0.1):
  """Factor arrays (E, S) of sprites `reach` = (lo, hi) canvas units across (log-uniform,
  measured along `side`, by default the canvas's longer side), drawn from the shape ids `pool`,
  each slot one of `kinds`:
    cross  -- a random point of one of its edges inside the canvas;
    corner -- a vertex whose two edges both leave it downwards with slopes of one sign (a
              corner join) on a canvas row, at an angle found by search;
    flat   -- at a multiple of 90 degrees, one of its horizontal edges on a canvas row;
    off    -- wholly off the canvas on one side (left, right, above, below), up to `hi` away;
  or, with probability p_small from slot 2 on, an ordinary sprite inside the canvas.  Every
  canvas coordinate stays below 2^30 in magnitude while hi <= 2^29 along the longer side."""
  side = float(max(CW, CH) if side is None else side)
  z = np.zeros((E, S))
  a = dict(x=z.copy(), y=z.copy(), pos_f32=np.zeros((E, S), np.uint8),
           shape=np.zeros((E, S), np.uint8), angle=z.copy(), scale=z.copy(), c0=z.copy(),
           c1=z.copy(), c2=z.copy(), vx=z.copy(), vy=z.copy(), member=np.zeros((E, S), np.uint32),
           rgb=np.zeros((E, S, 3), np.uint8))
  for e in range(E):
    for s in range(S):
      rgb = rng.randint(0, 256, 3)
      if s >= 2 and rng.rand() < p_small:
        shape = rng.choice(pool)
        _place(a, e, s, shape, rng.uniform(0.05, 0.3), rng.uniform(0, 360), rgb)
        a['x'][e, s], a['y'][e, s] = rng.uniform(0.1, 0.9, 2)
        continue
      kind = kinds[(e + s) % len(kinds)] if rng.rand() < 0.6 else kinds[rng.randint(len(kinds))]
      D = float(np.exp(rng.uniform(np.log(reach[0]), np.log(reach[1]))))
      shape = int(rng.choice(pool))
      v = _shape_verts(shape)
      scale = D / side / (2 * np.hypot(v[:, 0], v[:, 1]).max())
      in_canvas = rng.uniform(0.0, 1.0, 2)             # world point placed in the canvas
      if kind == 'corner':
        k = rng.randint(len(v))
        angle = _corner_angle(rng, v, k)
        if angle is None:
          kind = 'cross'
        else:
          c = _centred(v, scale, angle)
          p = c[k]
      if kind == 'flat':
        angle = 90.0 * rng.randint(4)
        c = _centred(v, scale, angle)
        flat = [i for i in range(len(c)) if abs(c[i, 1] - c[(i + 1) % len(c), 1]) < 1e-12 * scale]
        if flat:
          i = flat[rng.randint(len(flat))]
          p = c[i] + rng.rand() * (c[(i + 1) % len(c)] - c[i])
        else:
          kind = 'cross'
      if kind == 'cross':
        angle = rng.uniform(0, 360)
        c = _centred(v, scale, angle)
        i, t = rng.randint(len(c)), rng.rand()
        p = c[i] + t * (c[(i + 1) % len(c)] - c[i])
      if kind == 'off':
        angle = rng.uniform(0, 360)
        c = _centred(v, scale, angle)
        lo, hi = c.min(0), c.max(0)
        gap = float(np.exp(rng.uniform(np.log(1.0), np.log(reach[1] / 2)))) / side
        if rng.rand() < 0.25:
          gap = rng.choice([0.5, 2.0]) / side           # just clear of the canvas
        where = rng.randint(4)
        pos = rng.uniform(-0.5, 1.5, 2)
        if where == 0:
          pos[0] = -hi[0] - gap
        elif where == 1:
          pos[0] = 1.0 - lo[0] + gap
        elif where == 2:
          pos[1] = -hi[1] - gap
        else:
          pos[1] = 1.0 - lo[1] + gap
        _place(a, e, s, shape, scale, angle, rgb)
        a['x'][e, s], a['y'][e, s] = pos
        continue
      _place(a, e, s, shape, scale, angle, rgb)
      a['x'][e, s], a['y'][e, s] = in_canvas - p
  a['shape'][:, -1] = np.maximum(a['shape'][:, -1], pool[0])
  return a


def case_arrays(case):
  """The scenes of a case, one per env (seeded by the case id)."""
  cid, W, H, aa, bg, S, E, concave, kind = case
  rng = np.random.RandomState(sum(map(ord, cid)))
  if kind == 'huge' and concave:
    a = mask_oracle.huge_scene_arrays(rng, E, S, aa * H)
  elif kind == 'huge':     # the same, from the convex shapes
    a = far_scene_arrays(rng, E, S, aa * W, aa * H, CONVEX, (40000, 120000), kinds=('cross',),
                         side=aa * H, p_small=0)
  else:
    a = far_scene_arrays(rng, E, S, aa * W, aa * H, ALL_SHAPES if concave else CONVEX,
                         (INT16, LIMIT / 2))
  return geo._ensure_concave(a, rng, concave)


def canvas_int_vertices(case, rec_row):
  """Per occupied slot of one env: (slot, (n, 2) int64 vertices Pillow draws), as phase A and
  the oracle compute them."""
  cid, W, H, aa = case[:4]
  rc = oracle.raster_cfg(W, H, aa)
  tab = _tab()
  return [(s, np.trunc(mask_oracle.canvas_vertices(rc, tab, r)).astype(np.int64))
          for s, r in enumerate(rec_row) if r['shape']]


_TAB = []


def _tab():
  from spriteworld_b200 import constants
  if not _TAB:
    _TAB.append(oracle.shape_table(constants.SHAPES))
  return _TAB[0]


def max_canvas_coordinate(case, rec):
  return max(int(np.abs(iv).max()) for row in rec for _, iv in canvas_int_vertices(case, row))


# ---------------------------------------------------------------------------------------
# running the engine
# ---------------------------------------------------------------------------------------

def _sweep(case):
  """geo.Sweep of a case, with the segment table of the raster's path (built once per case)."""
  from tests import test_gpu_render_wide_aa as wide
  cid, W, H, aa, bg, S, E, concave, kind = case
  sw = geo.Sweep(case, geo._n_sms(), arrs=case_arrays(case))
  if aa >= WIDE_AA:
    sw.segcap = wide.render_layout(W, H, aa, S, concave)[1]
  return sw


def _reaches_the_regime(sw):
  rc = oracle.raster_cfg(sw.W, sw.H, sw.aa)
  assert max(abs(mask_oracle.canvas_vertices(rc, sw.tab, r)[:, 1]).max()
             for r in sw.rec[0] if r['shape']) > 40000, sw.case[0]
  assert max_canvas_coordinate(sw.case, sw.rec) < LIMIT, sw.case[0]


@gpu
@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_far_sprites_through_every_write_out(case):
  from spriteworld_b200 import engine
  sw = _sweep(case)
  try:
    _reaches_the_regime(sw)
    raster = engine.Raster(sw.eng, sw.W, sw.H, sw.aa, sw.bg)
    n_within = sum(sw.within(e) for e in range(sw.E))
    assert n_within >= 0.9 * sw.E, (case[0], n_within, sw.E)
    for skew in ((0, 1) if case[5] != 1 else (0,)):
      n_exact = geo._run_modes(sw, raster, skew)
      assert n_exact == [n_within] * 5, (case[0], skew, n_exact, n_within)
    raster.close()
  finally:
    sw.close()


@gpu
@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_far_sprites_from_env_records(case):
  """The records instantiation on the same scenes, permuted and repeated, at aligned and odd
  addresses, equals the live frames (the oracle's) bit for bit."""
  from spriteworld_b200 import engine
  from tests import test_gpu_render_states as rs
  sw = _sweep(case)
  try:
    raster = engine.Raster(sw.eng, sw.W, sw.H, sw.aa, sw.bg)
    live = sw.eng.render(raster).cpu().numpy()
    status = sw.eng.render_status().cpu().numpy()
    sw.check(live, status, (case[0], 'live'))
    n_exact, n_within = rs._render_permuted(sw, raster)
    assert n_within >= 0.9 * (2 * sw.E + 3) and n_exact == [n_within] * 2, (case[0], n_exact, n_within)
    raster.close()
  finally:
    sw.close()


# at anti_aliasing 1 a frame is the canvas itself: background where the mask is 0, rgb[mask - 1]
# elsewhere.  (id, W, H, S, E, concave, scene)
MASK_CASES = [
    ('huge_w64h64a1', 64, 64, 9, 12, True, 'huge'),
    ('far_w64h64a1', 64, 64, 32, 6, False, 'far'),
    ('far_w101h30a1', 101, 30, 9, 12, True, 'far'),
    ('huge_w41h1000a1', 41, 1000, 5, 4, False, 'huge'),
]


@gpu
@pytest.mark.parametrize('mc', MASK_CASES, ids=[c[0] for c in MASK_CASES])
def test_frames_at_aa1_are_the_masks_coloured(mc):
  from spriteworld_b200 import engine
  cid, W, H, S, E, concave, kind = mc
  bg = (17, 34, 51)
  case = (cid, W, H, 1, bg, S, E, concave, kind)
  sw = _sweep(case)
  try:
    _reaches_the_regime(sw)
    raster = engine.Raster(sw.eng, W, H, 1, bg)
    frames = sw.eng.render(raster).cpu().numpy()
    status = sw.eng.render_status().cpu().numpy()
    masks = sw.eng.render_masks(W, H, 1).cpu().numpy()
    n_within = sw.check(frames, status, (cid, 'render'))
    assert n_within >= 0.9 * E, (cid, n_within)
    n_drawn = 0
    for e in range(E):
      if status[e]:
        continue
      colours = np.concatenate([np.array([bg], np.uint8), sw.rec[e]['rgb']])
      # frames are stored top row first, masks flipped as PILRenderer does; both as Pillow draws
      assert np.array_equal(frames[e], colours[masks[e]]), (cid, e, int((frames[e] != colours[masks[e]]).any(-1).sum()))
      n_drawn += int((masks[e] > 0).any())
    assert n_drawn >= E // 2, (cid, n_drawn)
    raster.close()
  finally:
    sw.close()


# ---------------------------------------------------------------------------------------
# sprites flown out by the step kernel
# ---------------------------------------------------------------------------------------

def _flight_scenes(rng, E, S, CW):
  """Per env, slot 0: a square, hexagon, star or spoke 4 to 6 times 2^15 canvas units across,
  centred near the frame's centre (a sprite whose centre leaves [0, 1]^2 ends the episode), with
  a velocity of 0.01 to 0.02 frames per step along a diagonal d; slots 1..S-1: ordinary sprites
  inside [0.3, 0.7]^2 in front of it.  Returns the arrays and d (E, 2)."""
  a = geo._empty_arrays(E, S)
  d = rng.choice([-1.0, 1.0], (E, 2))
  for e in range(E):
    shape = (2, 4, 7, 10)[e % 4]
    rmax = np.hypot(*_shape_verts(shape).T).max()
    a['shape'][e, 0], a['angle'][e, 0] = shape, rng.uniform(0, 360)
    a['scale'][e, 0] = rng.uniform(2.0, 3.0) * INT16 / CW / rmax
    a['x'][e, 0], a['y'][e, 0] = 0.5 + 0.05 * d[e]
    a['vx'][e, 0], a['vy'][e, 0] = rng.uniform(0.01, 0.02, 2) * d[e]
    for s in range(1, S):
      a['shape'][e, s] = rng.choice(ALL_SHAPES)
      a['scale'][e, s], a['angle'][e, s] = rng.uniform(0.05, 0.15), rng.uniform(0, 360)
      a['x'][e, s], a['y'][e, s] = rng.uniform(0.3, 0.7, 2)
  a['rgb'][:] = rng.randint(0, 256, (E, S, 3))
  return a, d


def _outward(case, sprites, d):
  """Per env: how far the sprite's integer canvas vertices reach along the diagonal d (E, 2)."""
  return np.array([max((iv * d[e]).max() for _, iv in canvas_int_vertices(case, sprites[e]))
                   for e in range(len(sprites))])


def _click(kind, at, move, scale, dtype):
  """Actions clicking `at` (E, 2) and moving what they select by `move` (E, 2): SelectMove moves
  by scale * (a[2:] - 0.5), DragAndDrop by scale * (a[2:] - a[:2])."""
  a = np.zeros((len(at), 4))
  a[:, :2] = at
  a[:, 2:] = (0.5 if kind == 'select_move' else at) + move / scale
  return a.astype(dtype)


@gpu
@pytest.mark.parametrize('kind', ['select_move', 'drag_and_drop'])
@pytest.mark.parametrize('raster', [(256, 256, 10), (64, 64, 5)], ids=['w256a10', 'w64a5'])
def test_sprites_carried_out_by_the_step_kernel(kind, raster):
  """Within one episode the velocity update and clicks on a frame corner carry the huge sprite
  outward (its canvas coordinates past 2^15 and growing every step); then a click flings the
  sprite in front 1000 frames out, which ends the episode with that sprite drawn where it went,
  and the env resets.  Positions, rewards, step types and every frame against the oracle."""
  import torch
  from spriteworld_b200 import constants, engine, scene
  W, H, aa = raster
  E, S, K, T_IN = 16, 4, 1, 9
  scale = 2.0
  rng = np.random.RandomState(W + aa + len(kind))
  arrs, d = _flight_scenes(rng, E, S, W * aa)
  action = dict(kind=kind, scale=scale, motion_cost=0.3)
  nodes = [dict(kind='find_goal', filter_slot=-1, goal=[0.5, 0.5], weights=[1.0, 1.0],
                terminate_distance=0.0, terminate_bonus=0.0, raw_reward_multiplier=1.0,
                sparse_reward=False)]
  eng = engine.Engine(E, S, K, action, nodes, constants.SHAPES, keep_in_frame=False,
                      max_episode_length=T_IN + 10)
  b = scene.batch_from_factor_arrays(
      arrs['x'], arrs['y'], arrs['pos_f32'], arrs['shape'], arrs['angle'], arrs['scale'],
      arrs['c0'], arrs['c1'], arrs['c2'], arrs['vx'], arrs['vy'], arrs['member'], arrs['rgb'])
  eng.upload_scenes(b, np.arange(E), np.zeros(E, int))
  r = engine.Raster(eng, W, H, aa, (3, 4, 5))
  meta = dict(action=action, keep_in_frame=False, max_episode_length=T_IN + 10, nodes=nodes)
  bo = oracle.BatchOracle(oracle.with_device_sqrt(fixtures.env_cfg_from_meta(meta)), _tab(),
                          oracle.raster_cfg(W, H, aa, (3, 4, 5)),
                          fixtures.records_from_arrays(arrs).reshape(E, K, S))
  # a frame corner, away from the sprites in front: only the huge sprite is under it
  corner = 0.5 + 0.45 * d
  plan = ['reset'] + ['carry'] * T_IN + ['fling', 'reset', 'carry']
  huge, flung, types = [], [], []
  try:
    for t, what in enumerate(plan):
      dtype = np.float32 if t % 2 else np.float64
      if what == 'carry':
        a = _click(kind, corner, rng.uniform(0.005, 0.01, (E, 2)) * d, scale, dtype)
      elif what == 'fling':
        at = np.stack([bo.cur['x'][:, S - 1], bo.cur['y'][:, S - 1]], 1)
        a = _click(kind, at, rng.uniform(500, 1000, (E, 2)) * rng.choice([-1, 1], (E, 2)), scale,
                   dtype)
      else:
        a = np.full((E, 4), 0.5, dtype)
      res = eng.step(torch.from_numpy(a).to(eng.device), r)
      bo.step(a)
      torch.cuda.synchronize()
      st = eng.download_state()
      where = (kind, raster, t, what)
      assert np.array_equal(res.step_type.cpu().numpy(), bo.step_type), where
      assert np.array_equal(st['pos_x'], bo.cur['x']) and np.array_equal(st['pos_y'], bo.cur['y']), where
      assert np.array_equal(res.reward.cpu().numpy(), bo.reward), where
      status, frames = res.status.cpu().numpy(), res.frames.cpu().numpy()
      assert not status.any(), (where, status)
      for e in range(E):
        assert np.array_equal(frames[e], bo.frames[e]), where + (e, int((frames[e] != bo.frames[e]).any(-1).sum()))
      types.append(bo.step_type.copy())
      huge.append(_outward(('', W, H, aa), bo.cur[:, :1], d))
      flung.append(max_canvas_coordinate(('', W, H, aa), bo.cur[:, S - 1:]))
  finally:
    r.close()
    eng.close()
  # one episode of T_IN steps whose canvas coordinates pass 2^15 and grow every step, within the
  # int32 contract; the fling ends it with the flung sprite beyond int16 too
  assert all((types[t] == oracle.STEP_MID).all() for t in range(1, T_IN + 1)), types
  assert (INT16 < huge[1]).all() and all((b > c).all() for b, c in zip(huge[2:T_IN + 1], huge[1:T_IN])), huge
  assert (types[T_IN + 1] == oracle.STEP_LAST).all() and INT16 < flung[T_IN + 1] < LIMIT, flung
  assert max(h.max() for h in huge) < LIMIT, huge
