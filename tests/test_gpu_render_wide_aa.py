"""Render kernel at anti_aliasing 6 and more against the CPU oracle.

Windows of 6 * anti_aliasing canvas rows make a phase-C tile hold fewer blocks of eight output
rows (RasterDev::tile_blocks: 3, 2 or 1, whichever fits the H tile's 176 canvas rows), the
prefix table a longer stride, and the vertical pass more k-steps (3 to 6); such rasters render
in render_kernel<., true>, the aa <= 5 path stays as it was.  CASES sweeps those
over frame sizes, bands, column tiles, slot counts and pools with and without stars and spokes;
each case runs through every write-out of tests/test_gpu_render_geometry.py and must match the
oracle bit for bit.  test_case_table_covers_wide_paths recomputes the tables of
swb_raster_create in Python and fails if the sweep stops reaching one of them.

Also: the reference's own frames (tests/golden/wide_aa/render_cases_wide_aa.npz) through
PILRenderer.render, the demo's renderer (256x256, anti_aliasing 10, hsv_to_rgb) through
Environment and BatchedEnvironment, and the refusal of a raster whose windows do not fit.
"""
import json
import os

import numpy as np
import pytest

from oracle import oracle
from tests import fixtures
from tests import test_gpu_render_geometry as geo

TILE_BLOCKS = 3              # most blocks of eight output rows per phase-C tile
TILE_ROWS = 4 * 44           # canvas rows of the H tile (4 * HT_ROWW)
NARROW_PREFIX_STRIDE = 33    # prefix-table stride of windows up to 32 taps (kNarrowPrefixStride)
MAX_SMEM = 232448            # H100 opt-in shared memory per CTA

# (id, W, H, aa, bg, S, E, concave, scene), as in test_gpu_render_geometry.CASES
CASES = [
    ('w64h64a6', 64, 64, 6, (0, 0, 0), 9, 24, True, 'edges'),             # 3 blocks, 3 k-steps
    ('w64h64a7', 64, 64, 7, (90, 90, 90), 17, 24, False, 'edges'),        # 2 blocks, 3 k-steps
    ('w64h100a8', 64, 100, 8, (255, 255, 255), 32, 16, True, 'edges'),    # 2 blocks, 4 k-steps
    ('w64h64a8_s32', 64, 64, 8, (0, 0, 0), 32, 16, False, 'edges'),
    ('w128h128a9', 128, 128, 9, (10, 200, 30), 9, 8, False, 'edges'),     # 1 block, 4 k-steps
    ('w64h64a10', 64, 64, 10, (0, 0, 0), 1, 24, False, 'edges'),          # 1 block, 5 k-steps
    ('w100h100a10', 100, 100, 10, (40, 40, 40), 17, 8, True, 'edges'),
    ('w256h256a10', 256, 256, 10, (0, 0, 0), 9, 4, True, 'edges'),
    ('stripes_a10', 64, 64, 10, (0, 0, 0), 9, 16, False, 'stripes'),
    ('w64h64a13_full', 64, 64, 13, (5, 6, 7), 32, 8, False, 'full'),     # 1 block, 6 k-steps
    ('w315h8a13', 315, 8, 13, (5, 6, 7), 8, 8, True, 'edges'),            # 4095-pixel canvas side
    ('w64h8a20', 64, 8, 20, (0, 0, 255), 1, 16, True, 'edges'),           # accepted above aa 13
    ('w64h64a14', 64, 64, 14, (0, 0, 0), 9, 4, False, 'edges'),           # one block > 176 rows
]
REFUSED = {'w64h64a14'}


# ---------------------------------------------------------------------------------------
# host formulas of swb_tables.h / swb_raster_create / RenderLayout
# ---------------------------------------------------------------------------------------

def axis(n_in, n_out):
  """(win_min, win_len, taps) of build_axis."""
  bounds, kk = oracle.lanczos_coeffs(n_in, n_out)
  return bounds[:, 0].astype(int), bounds[:, 1].astype(int), kk


def tile_span(wmin, wlen, H, tb):
  band_rows = min(H, geo.BAND_ROWS)
  span = 0
  for y0 in range(0, H, band_rows):
    y1 = min(y0 + band_rows, H) - 1
    for t0 in range(y0, y1 + 1, 8):
      t1 = min(t0 + 8 * tb - 1, y1)
      span = max(span, wmin[t1] + wlen[t1] - (wmin[t0] & ~3))
  return span


def tile_blocks(H, aa):
  """choose_tile_blocks: 0 where swb_raster_create refuses the raster."""
  wmin, wlen, _ = axis(H * aa, H)
  tb = TILE_BLOCKS
  while tb > 0 and tile_span(wmin, wlen, H, tb) > TILE_ROWS:
    tb -= 1
  return tb


def v_nks(H, aa):
  """build_vfrag's k-steps: 32 canvas rows each, trailing zero taps left out."""
  wmin, wlen, kk = axis(H * aa, H)
  nks = 1
  for b in range(0, H, 8):
    o = wmin[b] & ~3
    end = o + 1
    for yo in range(b, min(b + 8, H)):
      last = wlen[yo] - 1
      while last > 0 and kk[yo][last] == 0:
        last -= 1
      end = max(end, wmin[yo] + last + 1)
    nks = max(nks, (end - o + 31) // 32)
  return nks


def render_layout(W, H, aa, S, concave):
  """RenderLayout (csrc/swb_render.cuh) as check_render picks it: (total bytes, segcap)."""
  band_rows = min(H, geo.BAND_ROWS)
  wmin, wlen, _ = axis(H * aa, H)
  rows = max(wmin[min(y0 + band_rows, H) - 1] + wlen[min(y0 + band_rows, H) - 1] - (wmin[y0] & ~3)
             for y0 in range(0, H, band_rows))
  xmin, xlen, xk = axis(W * aa, W)
  ncx = len({tuple(xk[i][:xlen[i]]) for i in range(W)})
  pstride = max(int(xlen.max()) + 1, NARROW_PREFIX_STRIDE)
  nks = v_nks(H, aa)
  M = 4 if concave else 1

  def layout(exact):
    o = 0

    def take(n):
      nonlocal o
      r = o
      o += (n + 15) & ~15
      return r
    for n in (S * 16, S * 18 * 4, S * 32 * 8, S * 32 * 12, S * 32 * 4, S * 32 * 6, S * 8):
      take(n)
    segcap = 16 if M > 1 else max(3, 2 * S - 1)
    if not exact:
      segcap = min(segcap, 16)
    take(((rows + 3) & ~3) + 8)
    take(rows * segcap * 4)
    take(ncx * pstride * 4)
    take(W * 4)
    take(band_rows * 4)
    cap = 16 if M > 1 else 8
    frame = band_rows * W * 3
    ht = 60 * 44 * 4
    if ht + ((frame + 15) & ~15) < (cap + M) * 4 * rows:
      ht = (cap + M) * 4 * rows - frame
    off_scratch = take(ht)
    take(frame)
    o = max(o, off_scratch + (64 * 44 + 8 * nks) * 4)
    return o, segcap
  total, segcap = layout(True)
  if total > MAX_SMEM and segcap > 16:
    total, segcap = layout(False)
  return total, segcap


def test_case_table_covers_wide_paths():
  paths = set()
  for case in CASES:
    cid, W, H, aa, bg, S, E, concave, scene = case
    tb = tile_blocks(H, aa)
    assert (tb == 0) == (cid in REFUSED), cid
    if tb == 0:
      paths.add('refused')
      continue
    nks = v_nks(H, aa)
    total, _ = render_layout(W, H, aa, S, concave)
    assert total <= MAX_SMEM, (cid, total)
    paths |= {'tile_blocks_%d' % tb, 'k_steps_%d' % nks, 'aa_%d' % aa,
              'S%d_%s' % (S, 'concave' if concave else 'convex')}
    if aa > 13:
      paths.add('accepted_above_13')
    if W * aa == 4095 or H * aa == 4095:
      paths.add('canvas_limit')
    if H > geo.BAND_ROWS and H % geo.BAND_ROWS:
      paths.add('partial_band')
    if W > 64:
      paths.add('column_tiles')
    if W == H:
      paths.add('square_%d' % W)
  need = {'refused', 'accepted_above_13', 'canvas_limit', 'partial_band', 'column_tiles',
          'square_64', 'square_128', 'square_256'}
  need |= {'tile_blocks_%d' % k for k in (1, 2, 3)} | {'k_steps_%d' % k for k in (3, 4, 5, 6)}
  need |= {'aa_%d' % k for k in (6, 7, 8, 9, 10, 13)}
  need |= {'S%d_%s' % (s, k) for s in (1, 9, 17, 32) for k in ('convex', 'concave')}
  assert need <= paths, sorted(need - paths)


def test_tables_match_the_known_factors():
  # 64-row frames (100 rows give the same): tile blocks and k-steps per anti_aliasing
  want = {6: (3, 3), 7: (2, 3), 8: (2, 4), 9: (1, 4), 10: (1, 5), 11: (1, 5), 12: (1, 5),
          13: (1, 6)}
  for aa, (tb, nks) in want.items():
    for H in (64, 100):
      assert (tile_blocks(H, aa), v_nks(H, aa)) == (tb, nks), (H, aa)
  assert tile_blocks(64, 14) == 0 and tile_blocks(8, 20) == 3 and v_nks(8, 20) == 5
  # every raster the kernel rendered before keeps three blocks per tile
  for H in (1, 7, 17, 64, 65, 100, 130, 819):
    for aa in range(1, 6):
      if H * aa <= 4095:
        assert tile_blocks(H, aa) == 3, (H, aa)
  # the demo's renderer with a nine-slot convex pool: 120,064 B, one CTA per SM (an H100 SM has
  # 233,472 B of shared memory, 1 KB of it reserved per CTA)
  total, segcap = render_layout(256, 256, 10, 9, False)
  assert segcap == 17 and total == 120064 and 2 * (total + 1024) > 233472, total


# ---------------------------------------------------------------------------------------
# the sweep on the GPU
# ---------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize('case', [pytest.param(c, id=c[0]) for c in CASES])
def test_wide_aa_sweep(case):
  from spriteworld_b200 import _native, engine
  cid, W, H, aa, bg, S, E, concave, scene = case
  sw = geo.Sweep(case, geo._n_sms())
  try:
    if cid in REFUSED:
      with pytest.raises(_native.NativeError, match='176'):
        engine.Raster(sw.eng, W, H, aa, bg)
      return
    sw.segcap = render_layout(W, H, aa, S, concave)[1]
    raster = engine.Raster(sw.eng, W, H, aa, bg)
    n_exact = geo._run_modes(sw, raster)
    n_within = sum(sw.ref(e)[1] <= sw.segcap for e in range(sw.E))
    assert n_within >= 0.9 * sw.E and n_exact == [n_within] * 5, (cid, n_exact, n_within, sw.E)
    raster.close()
  finally:
    sw.close()


@pytest.mark.gpu
def test_refused_raster_enqueues_nothing():
  """64x64 at anti_aliasing 14: the vertical windows of one block of eight output rows span 183
  canvas rows, more than the H tile's 176.  swb_raster_create refuses it, naming the limit,
  and the engine has launched nothing and changed nothing."""
  import torch
  from spriteworld_b200 import _native, constants, engine
  eng = engine.Engine(4, 2, 1, dict(kind='select_move', scale=0.05), [dict(kind='no_reward')],
                      constants.SHAPES)
  eng.step(torch.full((4, 4), 0.75, device=eng.device))
  torch.cuda.synchronize(eng.device)
  state, launches = eng.download_state(), eng.launch_count()
  with pytest.raises(_native.NativeError, match='183 canvas rows.*176'):
    engine.Raster(eng, 64, 64, 14)
  torch.cuda.synchronize(eng.device)
  assert eng.launch_count() == launches
  for k, v in eng.download_state().items():
    assert np.array_equal(v, state[k]), k
  # the same frame height one step lower renders
  engine.Raster(eng, 64, 64, 13).close()
  eng.close()


# ---------------------------------------------------------------------------------------
# frames of the reference
# ---------------------------------------------------------------------------------------

def wide_render_cases():
  """tests/golden/wide_aa/render_cases_wide_aa.npz (make_golden_wide_aa.py): (meta, factor
  arrays, frame) per case."""
  blob = fixtures.load(os.path.join('wide_aa', 'render_cases_wide_aa.npz'))
  out = []
  for i in range(len(blob['names'])):
    meta = json.loads(str(blob['meta_%d' % i]))
    out.append((meta, {f: blob['%s_%d' % (f, i)] for f in fixtures.FIELDS}, blob['frame_%d' % i]))
  return fixtures.shapes_of(blob), out


@pytest.mark.gpu
def test_reference_frames_through_pil_renderer():
  from spriteworld_b200 import renderers, sprite
  names = {v: k for k, v in oracle.SHAPE_IDS.items()}
  _, cases = wide_render_cases()
  for meta, arrs, frame in cases:
    sprites = []
    for k in range(len(arrs['x'])):
      if not arrs['shape'][k]:
        continue
      pos = np.float32 if arrs['pos_f32'][k] else float
      col = np.float32 if arrs['color_f32'][k] else float
      sprites.append(sprite.Sprite(x=pos(arrs['x'][k]), y=pos(arrs['y'][k]),
                                   shape=names[int(arrs['shape'][k])], angle=arrs['angle'][k],
                                   scale=arrs['scale'][k], c0=col(arrs['c0'][k]),
                                   c1=col(arrs['c1'][k]), c2=col(arrs['c2'][k])))
    ctr = renderers.color_maps.hsv_to_rgb if meta['color_map'] == 'hsv' else None
    r = renderers.PILRenderer(image_size=(meta['width'], meta['height']),
                              anti_aliasing=meta['aa'], bg_color=tuple(meta['bg']),
                              color_to_rgb=ctr)
    got = r.render(sprites)
    assert np.array_equal(got, frame), (meta['name'], int((got != frame).sum()))


# ---------------------------------------------------------------------------------------
# the demo's renderer through the environments
# ---------------------------------------------------------------------------------------

def _demo_config(max_episode_length):
  from spriteworld_b200 import renderers
  from spriteworld_b200.configs.cobra import clustering
  cfg = clustering.get_config('train')
  cfg['renderers'] = {
      'image': renderers.PILRenderer(image_size=(256, 256), anti_aliasing=10,
                                     color_to_rgb=renderers.color_maps.hsv_to_rgb),
      'success': renderers.Success()}
  cfg['max_episode_length'] = max_episode_length
  return cfg


def _oracle_for(cfg, pool):
  from spriteworld_b200 import constants
  nodes, _ = cfg['task'].compile()
  meta = dict(action=cfg['action_space'].compile(), keep_in_frame=True,
              max_episode_length=cfg['max_episode_length'], nodes=nodes)
  ocfg = oracle.with_device_sqrt(fixtures.env_cfg_from_meta(meta))
  bo = oracle.BatchOracle(ocfg, oracle.shape_table(constants.SHAPES),
                          oracle.raster_cfg(256, 256, 10), pool)
  bo.pool = pool            # share the live mirror (refills land in it)
  return bo


def _mirror(eng, E, K):
  """A host copy of the engine's scene pool, kept current by wrapping upload_scenes."""
  pool = np.zeros((E, K, eng.n_slots), oracle.SPRITE_DTYPE)
  orig = eng.upload_scenes

  def upload(batch, env_ids, ring_slots):
    for f in ('x', 'y', 'm00', 'm01', 'm10', 'm11', 'vx', 'vy', 'member', 'shape', 'pos_f32', 'rgb'):
      pool[f][np.asarray(env_ids), np.asarray(ring_slots)] = batch[f]
    return orig(batch, env_ids, ring_slots)
  eng.upload_scenes = upload
  return pool


@pytest.mark.gpu
def test_demo_renderer_batched_environment():
  from spriteworld_b200 import environment, scene, sprite_generators
  E, K, T = 4, 3, 24
  cfg = _demo_config(max_episode_length=7)
  env = environment.BatchedEnvironment(n_envs=E, pool_depth=K, rng=np.random.RandomState(3), **cfg)
  eng = env.engine
  pool = _mirror(eng, E, K)
  # the constructor uploaded the first K scenes per env already: sample them again
  first = sprite_generators.batch_of(cfg['init_sprites'], E * K, np.random.RandomState(3))
  _, filters = cfg['task'].compile()
  b0 = scene.arrays_from_layout(first, eng.n_slots, filters, cfg['renderers']['image'].color_to_rgb)
  for f in ('x', 'y', 'm00', 'm01', 'm10', 'm11', 'vx', 'vy', 'member', 'shape', 'pos_f32', 'rgb'):
    pool[f][np.repeat(np.arange(E), K), np.tile(np.arange(K), E)] = b0[f]
  bo = _oracle_for(cfg, pool)
  rng = np.random.RandomState(11)
  n_first = 0
  for t in range(T):
    a = rng.uniform(0, 1, (E, 4)).astype(np.float32)
    ts = env.step(a)
    bo.step(a)
    st = ts.step_type.cpu().numpy()
    assert np.array_equal(st, bo.step_type), t
    n_first += int((st == 0).sum())
    assert np.array_equal(ts.reward.cpu().numpy(), bo.reward, equal_nan=True), t
    assert np.array_equal(ts.observation['success'].cpu().numpy(), bo.success.astype(bool)), t
    assert ts.observation['image'].shape == (E, 256, 256, 3)
    assert np.array_equal(ts.observation['image'].cpu().numpy(), bo.frames), t
  assert n_first > E            # episodes ended and restarted
  env.close()


@pytest.mark.gpu
def test_demo_renderer_environment():
  """The drop-in Environment with the demo's renderers: every frame is the oracle's frame of the
  sprites the environment holds after the step (positions synced from the device), and episodes
  end and restart on the step cadence of max_episode_length."""
  from spriteworld_b200 import constants, environment
  cfg = _demo_config(max_episode_length=6)
  ctr = cfg['renderers']['image'].color_to_rgb
  tab = oracle.shape_table(constants.SHAPES)
  rc = oracle.raster_cfg(256, 256, 10)
  np.random.seed(5)
  env = environment.Environment(**cfg)
  rng = np.random.RandomState(2)
  kinds = []
  for t in range(20):
    ts = env.step(rng.uniform(0, 1, 4).astype(np.float32))
    kinds.append(int(ts.step_type))
    sprites = env.state()['sprites']
    S = len(sprites)
    arrs = {k: np.zeros(S) for k in ('x', 'y', 'angle', 'scale', 'vx', 'vy')}
    arrs.update(pos_f32=np.zeros(S, np.uint8), shape=np.zeros(S, np.uint8),
                member=np.zeros(S, np.uint32), rgb=np.zeros((S, 3), np.uint8))
    for k, s in enumerate(sprites):
      arrs['x'][k], arrs['y'][k] = float(s.position[0]), float(s.position[1])
      arrs['angle'][k], arrs['scale'][k] = float(s.angle), float(s.scale)
      arrs['shape'][k] = oracle.SHAPE_IDS[s.shape]
      arrs['rgb'][k] = [int(c) for c in ctr(s.color)]
    want = oracle.render(rc, tab, fixtures.records_from_arrays(arrs))
    assert np.array_equal(ts.observation['image'], want), t
    assert isinstance(ts.observation['success'], (bool, np.bool_))
  # FIRST, then at most six steps to the episode's LAST (success may end it sooner)
  assert kinds.count(0) >= 3 and kinds[0] == 0, kinds
  env.close()
