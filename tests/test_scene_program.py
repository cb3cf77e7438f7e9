"""The device scene sampler's program compiler and its CPU build (no GPU needed).

scene_program.sample_on_host runs csrc/swb_sampler.cuh built for the CPU, the same source the
kernels run.  Here it is held to three independent specifications: np.random.Philox for the random
stream, scene.arrays_from_layout for the packing of its own drawn factors, and the host sampler
(init_sprites.batch) for the distribution of scenes.
"""
import importlib

import numpy as np
import pytest
from scipy import stats

from spriteworld_b200 import environment, scene, scene_program
from spriteworld_b200 import factor_distributions as distribs
from spriteworld_b200 import sprite_generators as gen
from spriteworld_b200.renderers import color_maps

CONFIGS = [('cobra.clustering', 'train'), ('cobra.clustering', 'test'), ('cobra.exploration', None),
           ('cobra.goal_finding_more_distractors', 'train'), ('cobra.goal_finding_more_distractors', 'test'),
           ('cobra.goal_finding_more_targets', 'train'), ('cobra.goal_finding_more_targets', 'test'),
           ('cobra.goal_finding_new_position', 'train'), ('cobra.goal_finding_new_position', 'test'),
           ('cobra.goal_finding_new_shape', 'train'), ('cobra.goal_finding_new_shape', 'test'),
           ('cobra.sorting', 'train'), ('cobra.sorting', 'test'),
           ('examples.goal_finding_clustering', 'train'), ('examples.goal_finding_clustering', 'test'),
           ('examples.goal_finding_embodied', None)]


def compiled(name, mode):
  cfg = importlib.import_module('spriteworld_b200.configs.' + name).get_config(mode)
  _, filters = cfg['task'].compile()
  cmap = environment._color_map(environment._split_renderers(cfg['renderers'])[0])
  return cfg, filters, cmap, scene_program.compile_program(cfg['init_sprites'], filters, cmap)


def bits(a):
  a = np.ascontiguousarray(a)
  return a.view(np.uint8) if a.dtype.kind == 'f' else a


def assert_packs_like_host(b, S, filters, cmap):
  layout = scene_program.layout_from_factor_table(b['factor_value'], b['factor_kind'])
  ref = scene.arrays_from_layout(layout, S, filters, cmap)
  for k in ref:
    assert np.array_equal(bits(ref[k]), bits(b[k])), k


@pytest.mark.parametrize('name,mode', CONFIGS)
def test_config_compiles_and_packs_like_arrays_from_layout(name, mode):
  _, filters, cmap, prog = compiled(name, mode)
  S = prog.max_sprites
  rng = np.random.RandomState(1)
  ids = np.concatenate([np.arange(1000), rng.randint(0, 2 ** 62, 1000)])
  idx = np.concatenate([np.arange(1000) % 7, rng.randint(0, 2 ** 62, 1000)])
  b, fail = scene_program.sample_on_host(prog, 99, ids, idx, S)
  assert fail is None
  assert (b['shape'] > 0).sum(1).min() >= 1
  assert_packs_like_host(b, S, filters, cmap)


def test_philox_equals_numpy():
  rng = np.random.RandomState(0)
  for _ in range(50):
    ctr = rng.randint(0, 2 ** 63, 4, dtype=np.uint64)
    ctr[0] |= 1
    key = [int(rng.randint(0, 2 ** 63, dtype=np.uint64)), scene_program.DOMAIN]
    ref = np.random.Philox(counter=[int(ctr[0]) - 1, int(ctr[1]), int(ctr[2]), int(ctr[3])],
                           key=key).random_raw(4)
    assert np.array_equal(scene_program.philox_host(ctr, key), ref)


def _program(init_sprites, filters=(), cmap=None):
  return scene_program.compile_program(init_sprites, filters, cmap)


def test_float32_bounds_and_rgb_paths():
  # np.array([np.float32(0.9)]) < 0.9 is False (the bound is cast to float32), but the float64
  # 0.8999999761581421 < 0.9 is True
  hue = distribs.Continuous('c0', 0.0, 0.9)
  parts = [distribs.Discrete('c0', [np.float32(0.9)]), distribs.Discrete('c0', [0.8999999761581421])]
  for c0, member in zip(parts, (0, 1)):
    g = gen.generate_sprites(distribs.Product([c0, distribs.Discrete('c1', [0.5]),
                                               distribs.Discrete('c2', [0.5])]), 2)
    if c0.candidates[0].__class__ is np.float32:
      g = gen.generate_sprites(distribs.Product([c0, distribs.Continuous('c1', 0, 1),
                                                 distribs.Continuous('c2', 0, 1)]), 2)
    prog = _program(g, [hue], color_maps.hsv_to_rgb)
    b, _ = scene_program.sample_on_host(prog, 5, np.arange(64), np.zeros(64), 2)
    assert (b['member'] == member).all()
    assert_packs_like_host(b, 2, [hue], color_maps.hsv_to_rgb)
  # x float32 but y float64: scene._full_columns promotes both to float64 before the filters, so
  # the float32 0.9 is inside [0, 0.9) as a float64
  g = gen.generate_sprites(distribs.Product([
      distribs.Discrete('x', [np.float32(0.9)]), distribs.Continuous('y', 0, 1, dtype='float64'),
      distribs.Continuous('c0', 0, 1), distribs.Continuous('c1', 0, 1), distribs.Continuous('c2', 0, 1)]), 2)
  xf = distribs.Continuous('x', 0, 0.9)
  b, _ = scene_program.sample_on_host(_program(g, [xf], color_maps.hsv_to_rgb), 5, np.arange(64),
                                      np.zeros(64), 2)
  assert (b['member'] == 1).all() and (b['pos_f32'] == 0).all()
  assert_packs_like_host(b, 2, [xf], color_maps.hsv_to_rgb)
  # angle -0.0 and 0.0 are distinct table entries: they give differently signed zeros.  (Compared
  # with scene.transform_matrix itself: the memo of scene.transform_matrices keys on float values,
  # so within one process it returns whichever of the two zeros it met first.)
  g = gen.generate_sprites(distribs.Discrete('angle', [-0.0, 0.0, 90.0]), 3)
  b, _ = scene_program.sample_on_host(_program(g), 8, np.arange(200), np.zeros(200), 3)
  angle = b['factor_value'][..., 3].reshape(-1)
  assert np.signbit(angle).any() and not np.signbit(angle).all()
  want = np.array([scene.transform_matrix(0.1, a) for a in angle]).reshape(200, 3, 4)
  for i, f in enumerate(('m00', 'm01', 'm10', 'm11')):
    assert np.array_equal(bits(b[f]), bits(want[..., i])), f
  # RGB integer colours wrap through int64 -> uint8; float64 HSV colours
  for factors, cmap in (([distribs.Continuous('c0', 200, 400, dtype='int64'),
                          distribs.Continuous('c1', -20, 20, dtype='int32'),
                          distribs.Continuous('c2', 0, 256, dtype='uint8')], None),
                        ([distribs.Continuous('c0', 0, 1, dtype='float64'),
                          distribs.Continuous('c1', 0, 1, dtype='float64'),
                          distribs.Discrete('c2', [0.0, 1.0])], color_maps.hsv_to_rgb)):
    g = gen.shuffle(gen.generate_sprites(distribs.Product(factors + [
        distribs.Discrete('angle', [0, 45, -30]), distribs.Continuous('scale', 0.1, 0.2)]),
        gen.uniform_count(0, 5)))
    prog = _program(g, [distribs.Continuous('c0', 250, 300)], cmap)
    b, _ = scene_program.sample_on_host(prog, 6, np.arange(500), np.arange(500), 4)
    assert_packs_like_host(b, 4, [distribs.Continuous('c0', 250, 300)], cmap)


def test_refusals():
  body = distribs.Product([distribs.Continuous('x', 0, 1), distribs.Continuous('c0', 0, 1)])
  with pytest.raises(NotImplementedError, match='uniform_count'):
    _program(gen.generate_sprites(body, lambda: np.random.randint(1, 3)))
  with pytest.raises(NotImplementedError, match='plain callables'):
    _program(lambda: [])
  with pytest.raises(NotImplementedError, match='colour map'):
    _program(gen.generate_sprites(body, 1), (), lambda c: (0, 0, 0))
  with pytest.raises(NotImplementedError, match='mixed or integer'):
    _program(gen.generate_sprites(body, 1), (), color_maps.hsv_to_rgb)
  with pytest.raises(NotImplementedError, match='finite set'):
    _program(gen.generate_sprites(distribs.Continuous('angle', 0, 360), 1))
  with pytest.raises(NotImplementedError, match='slots'):
    _program(gen.generate_sprites(body, 40))
  with pytest.raises(NotImplementedError, match='limits'):
    _program(gen.generate_sprites(distribs.Discrete('scale', list(np.linspace(0, 1, 2000))), 1))


def test_uniform_count_draws_like_randint():
  np.random.seed(3)
  a = [gen.uniform_count(1, 7)() for _ in range(100)]
  np.random.seed(3)
  assert a == [np.random.randint(1, 7) for _ in range(100)]
  import pickle
  assert pickle.loads(pickle.dumps(gen.uniform_count(1, 7)))() in range(1, 7)


# Marginals against the host sampler, 20 000 scenes per side at fixed seeds.  Every comparison
# must have p > 1e-4: two-sample KS for continuous columns, chi-square for counts, shapes, the
# scenes' sets of member values (sample_generator's choices), every factor per (member value,
# shape) group of sprites (per generator), and the per-slot rate of each member bit (the shuffle
# order).
P_MIN = 1e-4
N_SCENES = 20000


def _chi2(a, b):
  keys = sorted(set(a) | set(b))
  table = np.array([[a.get(k, 0) for k in keys], [b.get(k, 0) for k in keys]])
  table = table[:, table.sum(0) > 0]
  if table.shape[1] < 2:
    return 1.0
  return stats.chi2_contingency(table)[1]


def _counts(v):
  u, c = np.unique(v, return_counts=True)
  return dict(zip(u.tolist(), c.tolist()))


@pytest.mark.parametrize('name,mode', CONFIGS)
def test_marginals_match_host_sampler(name, mode):
  cfg, filters, cmap, prog = compiled(name, mode)
  S = prog.max_sprites
  dev, _ = scene_program.sample_on_host(prog, 2024, np.arange(N_SCENES) // 4, np.arange(N_SCENES) % 4, S)
  np.random.seed(11)
  host = scene.arrays_from_layout(gen.batch_of(cfg['init_sprites'], N_SCENES, np.random.RandomState(12)),
                                  S, filters, cmap)
  occ_d, occ_h = dev['shape'] > 0, host['shape'] > 0
  assert _chi2(_counts(occ_d.sum(1)), _counts(occ_h.sum(1))) > P_MIN, 'sprite count'
  assert _chi2(_counts(dev['shape'][occ_d]), _counts(host['shape'][occ_h])) > P_MIN, 'shape'
  # the generators of the shipped configs differ in their filter membership (targets and
  # distractors, one colour band per cluster or subtask), so the factors are compared per member
  # value and per shape: each group is one generator's sprites (or a union of generators that
  # draw alike), and a misrouted choice or jump moves sprites between groups
  # which generators a scene drew from (sample_generator's choice): its set of member values
  sig_d = [frozenset(r[o].tolist()) for r, o in zip(dev['member'], occ_d)]
  sig_h = [frozenset(r[o].tolist()) for r, o in zip(host['member'], occ_h)]
  assert _chi2(_counts(np.array([hash(v) for v in sig_d])), _counts(np.array([hash(v) for v in sig_h]))) > P_MIN
  mem_d, mem_h = dev['member'][occ_d], host['member'][occ_h]
  shp_d, shp_h = dev['shape'][occ_d], host['shape'][occ_h]
  for m in np.unique(mem_h):
    for sh in np.unique(shp_h):
      gd, gh = (mem_d == m) & (shp_d == sh), (mem_h == m) & (shp_h == sh)
      if gh.sum() < 200:
        continue
      cols_d = [dev['x'][occ_d], dev['y'][occ_d]] + [dev['factors'][..., i][occ_d] for i in range(5)]
      cols_h = [host['x'][occ_h], host['y'][occ_h]] + [host['factors'][..., i][occ_h] for i in range(5)]
      for f, cd, ch in zip(('x', 'y', 'scale', 'angle', 'c0', 'c1', 'c2'), cols_d, cols_h):
        d, h = cd[gd], ch[gh]
        if np.unique(h).size > 50:
          assert stats.ks_2samp(d, h).pvalue > P_MIN, (f, m, sh)
        else:
          assert _chi2(_counts(d), _counts(h)) > P_MIN, (f, m, sh)
  for bit in range(len(filters)):
    for slot in range(S):
      m_d = (dev['member'][:, slot] >> bit) & 1
      m_h = (host['member'][:, slot] >> bit) & 1
      a = {0: int((occ_d[:, slot] & (m_d == 0)).sum()), 1: int(m_d.sum()), 2: int((~occ_d[:, slot]).sum())}
      b = {0: int((occ_h[:, slot] & (m_h == 0)).sum()), 1: int(m_h.sum()), 2: int((~occ_h[:, slot]).sum())}
      assert _chi2(a, b) > P_MIN, ('member bit', bit, 'slot', slot)
