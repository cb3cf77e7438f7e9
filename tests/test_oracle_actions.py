"""CPU tier: the oracle's click action path against the reference (tests/golden/actions/).

actions.npz holds single SelectMove / DragAndDrop steps of the reference on three sprites,
over action and position dtypes, scales, motion costs, keep_in_frame and actions in and far
outside [0, 1], exact 0 / 0.5 / 1 and their neighbours, signed zeros, subnormals, NaN, +-inf
and 1e30; and short Environment episodes with float64 actions, motion cost 0.7, action noise
and sprites flung to about +-10 (make_golden_actions.py).  Everything here is bit for bit:
a cost, reward or position matches when its float64 bits are equal, or when both are NaN.
"""
import json

import numpy as np
import pytest

from oracle import oracle
from tests import fixtures

KIND = (oracle.ACT_SELECT_MOVE, oracle.ACT_DRAG_AND_DROP)


class ActionCases(object):
  """tests/golden/actions/actions.npz."""

  def __init__(self):
    blob = fixtures.load('actions/actions.npz')
    self.blob = blob
    self.meta = json.loads(str(blob['meta']))
    self.ss = {k[3:]: blob[k] for k in blob.files if k.startswith('ss_')}
    self.n = len(self.ss['cost'])
    self.shapes = fixtures.shapes_of(blob)
    self.episode_names = [str(n) for n in blob['ep_names']]

  def records(self, i, positions=None):
    """The three sprites of single step i (positions before the step unless given)."""
    ss = self.ss
    p = ss['before'][i] if positions is None else positions
    z = np.zeros(len(p))
    return fixtures.records_from_arrays(dict(
        x=p[:, 0].copy(), y=p[:, 1].copy(), vx=z, vy=z, member=np.zeros(len(p), np.uint32),
        shape=ss['shape'][i], pos_f32=ss['pos_f32'][i], rgb=np.zeros((len(p), 3), np.uint8),
        scale=ss['sprite_scale'][i], angle=ss['angle'][i]))

  def action(self, i):
    a = self.ss['action'][i]
    return a.astype(np.float32) if self.ss['f32'][i] else a.copy()

  def cfg(self, i, nodes=None):
    ss = self.ss
    cfg = fixtures.env_cfg_from_meta(dict(
        action=dict(kind=('select_move', 'drag_and_drop')[ss['kind'][i]],
                    scale=float(ss['scale'][i]), motion_cost=float(ss['motion_cost'][i])),
        keep_in_frame=bool(ss['keep'][i]), max_episode_length=1000,
        nodes=nodes or [dict(kind='no_reward')]))
    return cfg

  def expected_env_step(self, i):
    """What Environment.step makes of single step i under a NoReward task with zero velocities:
    the velocity update adds 0.0 to every position (so -0.0 becomes 0.0), the reward is
    cost + 0.0 in the cost's dtype, and any position outside [0, 1] (NaN included) ends the
    episode (sprite.py:135-138)."""
    ss = self.ss
    pos = ss['after'][i] + 0.0
    if ss['f32'][i]:
      reward = np.float64(np.float32(ss['cost'][i]) + 0.0)
    else:
      reward = ss['cost'][i] + 0.0
    oof = any(not (np.all(p >= [0., 0.]) and np.all(p <= [1., 1.])) for p in pos)
    return pos, reward, oracle.STEP_LAST if oof else oracle.STEP_MID

  def episode(self, c):
    b, p = self.blob, 'ep%d_' % c
    ep = {k[len(p):]: b[k] for k in b.files if k.startswith(p)}
    ep['meta'] = json.loads(str(ep['meta']))
    ep['scenes'] = {f: ep.pop('scene_' + f) for f in fixtures.FIELDS}
    return ep


def same_bits(a, b):
  """Elementwise: equal float64 bits, or both NaN."""
  a = np.ascontiguousarray(a, np.float64)
  b = np.ascontiguousarray(b, np.float64)
  return (a.view(np.uint64) == b.view(np.uint64)) | (np.isnan(a) & np.isnan(b))


@pytest.fixture(scope='module')
def cases():
  return ActionCases()


def _describe(cases, i):
  ss = cases.ss
  return dict(case=i, kind=cases.meta['kinds'][ss['kind'][i]], f32=bool(ss['f32'][i]),
              scale=float(ss['scale'][i]), motion_cost=float(ss['motion_cost'][i]),
              keep=bool(ss['keep'][i]), mode=cases.meta['modes'][ss['mode'][i]],
              action=cases.action(i).tolist())


def test_fixture_covers_the_action_inputs(cases):
  ss = cases.ss
  combos = {(int(k), float(s), float(c), int(kp), int(f)) for k, s, c, kp, f in zip(
      ss['kind'], ss['scale'], ss['motion_cost'], ss['keep'], ss['f32'])}
  assert len(combos) == 2 * 4 * 4 * 2 * 2
  assert set(cases.meta['modes']) == {'uniform', 'wide', 'centre', 'vertex', 'special',
                                      'nonfinite', 'large'}
  a = ss['action']
  for i in range(4):
    for v in (np.nan, np.inf, -np.inf):
      assert (np.isnan(a[:, i]) if v != v else a[:, i] == v).any(), (i, v)
  assert (~np.isfinite(a)).all(1).any()
  assert (np.signbit(a) & (a == 0)).any() and ((a != 0) & (np.abs(a) < 1e-300)).any()
  assert (ss['moved'] >= 0).sum() > cases.n // 4
  assert {0, 1} <= set(ss['pos_f32'].reshape(-1).tolist())
  # the float64 cost is np.linalg.norm's: fused, and apart from the unfused formula somewhere
  f64 = (ss['f32'] == 0) & (ss['motion_cost'] > 0)
  m = _motion(ss)
  with np.errstate(all='ignore'):
    unfused = -ss['motion_cost'] * np.sqrt(m[:, 0] * m[:, 0] + m[:, 1] * m[:, 1])
  assert (~same_bits(unfused, ss['cost']) & f64).sum() > 20


def _motion(ss):
  a = ss['action']
  with np.errstate(all='ignore'):
    d = np.where(ss['kind'][:, None] == 0, a[:, 2:] - 0.5, a[:, 2:] - a[:, :2])
    return d * ss['scale'][:, None]


def test_action_step_matches_reference(cases):
  tab = oracle.shape_table(cases.shapes)
  bad = []
  for i in range(cases.n):
    sp = cases.records(i)
    cost, moved = oracle.action_step(cases.cfg(i), tab, sp, cases.action(i),
                                     bool(cases.ss['f32'][i]))
    ok_cost = same_bits(cost, cases.ss['cost'][i])
    ok_moved = moved[0] == cases.ss['moved'][i]
    got = np.stack([sp['x'], sp['y']], 1)
    ok_pos = same_bits(got, cases.ss['after'][i]).all()
    if not (ok_cost and ok_moved and ok_pos):
      bad.append(dict(_describe(cases, i), cost=(cost.hex(), float(cases.ss['cost'][i]).hex()),
                      moved=(moved[0], int(cases.ss['moved'][i])),
                      pos=(got.tolist(), cases.ss['after'][i].tolist())))
  assert not bad, '%d of %d cases differ; first: %r' % (len(bad), cases.n, bad[:3])


def test_env_step_matches_reference(cases):
  tab = oracle.shape_table(cases.shapes)
  bad = []
  for i in range(cases.n):
    sp = cases.records(i)
    out = oracle.env_step(cases.cfg(i), tab, sp, 0, cases.action(i), bool(cases.ss['f32'][i]))
    pos, reward, step_type = cases.expected_env_step(i)
    got = np.stack([sp['x'], sp['y']], 1)
    if not (same_bits(out['reward'], reward) and out['step_type'] == step_type and
            same_bits(got, pos).all() and out['err'] == 0 and out['step_count'] == 1):
      bad.append(dict(_describe(cases, i), got=out, want=(reward, step_type)))
  assert not bad, '%d of %d cases differ; first: %r' % (len(bad), cases.n, bad[:3])


@pytest.mark.parametrize('c', range(4))
def test_episodes_match_reference(cases, c):
  """The oracle in the reference's pow distance mode, fed the actions the reference applied."""
  ep = cases.episode(c)
  meta = ep['meta']
  cfg = fixtures.env_cfg_from_meta(meta)
  tab = oracle.shape_table(cases.shapes)
  bo = oracle.BatchOracle(cfg, tab, None, fixtures.records_from_arrays(ep['scenes']))
  T, E = ep['reward'].shape
  for t in range(T):
    bo.step(ep['applied'][t])
    where = (meta['name'], t)
    assert np.array_equal(bo.step_type, ep['step_type'][t]), where
    assert np.array_equal(bo.cursor, ep['scene_idx'][t]), where
    assert np.array_equal(bo.success, ep['success'][t]), where
    assert (bo.err == 0).all(), where
    assert same_bits(bo.reward, ep['reward'][t]).all(), where
    occ = bo.cur['shape'] > 0
    got = np.stack([bo.cur['x'], bo.cur['y']], -1)
    assert same_bits(got[occ], ep['pos'][t][occ]).all(), where


def test_episodes_cover_what_they_are_for(cases):
  kinds = set()
  n_far = n_noisy = 0
  for c in range(len(cases.episode_names)):
    ep = cases.episode(c)
    meta = ep['meta']
    kinds.add(meta['nodes'][-1]['kind'])
    assert meta['action']['motion_cost'] == 0.7 and not meta['keep_in_frame']
    assert ep['actions'].dtype == np.float64 and len(ep['frames']) > 0
    n_far += int((np.abs(ep['pos'][ep['step_type'] == 2]) > 5).any(-1).any(-1).sum())
    if meta['noise_scale']:
      done = ~np.isnan(ep['applied'][..., 0])
      n_noisy += int((ep['applied'][done] != ep['actions'][done]).all(-1).sum())
  assert kinds == {'find_goal', 'clustering', 'meta', 'no_reward'}
  assert n_far >= 10 and n_noisy >= 20


def test_render_far_out_of_frame_matches_reference(cases):
  tab = oracle.shape_table(cases.shapes)
  n = 0
  for c in range(len(cases.episode_names)):
    ep = cases.episode(c)
    meta = ep['meta']
    rc = oracle.raster_cfg(meta['width'], meta['height'], meta['aa'], meta['bg'])
    pool = fixtures.records_from_arrays(ep['scenes'])
    for (t, e), frame in zip(ep['frame_at'], ep['frames']):
      sp = pool[e, ep['scene_idx'][t, e]].copy()
      sp['x'], sp['y'] = ep['pos'][t, e, :, 0], ep['pos'][t, e, :, 1]
      got = oracle.render(rc, tab, sp)
      assert np.array_equal(got, frame), (meta['name'], int(t), int(e))
      n += 1
  assert n >= 40


def test_numpy_norm_on_this_host_reproduces_the_fixture(cases):
  """The float64 cost is -motion_cost * np.linalg.norm(motion), whose rounding belongs to the
  BLAS NumPy was built with.  On the NumPy and OpenBLAS the fixture was made with, NumPy here
  must give the recorded bits; elsewhere the comparison says nothing about this project."""
  meta = cases.meta
  blas = np.show_config(mode='dicts')['Build Dependencies']['blas']
  have = (np.__version__, blas.get('name'), blas.get('version'))
  want = (meta['numpy'], meta['blas'], meta['blas_version'])
  if have != want:
    pytest.skip('NumPy / BLAS here is %r, the fixture was made with %r' % (have, want))
  ss = cases.ss
  m = _motion(ss)
  f64 = np.nonzero(ss['f32'] == 0)[0]
  with np.errstate(all='ignore'):
    got = np.array([-ss['motion_cost'][i] * np.linalg.norm(m[i]) for i in f64])
  assert same_bits(got, ss['cost'][f64]).all()
