"""The step kernel (csrc/swb_step.cuh) swept over its paths against the CPU oracle, bit for bit.

Each case of CASES builds seeded scenes and actions and runs T steps through Engine.step and
Engine.step_host.  After every step it compares with oracle.BatchOracle in its sqrt-distance
mode (oracle.with_device_sqrt, the engine's FindGoalPosition distance): positions of the
occupied slots, cursor, step_count, reset_next, scene_serial, step type, success, status and
reward (positions and rewards NaN-aware).  Action-only cases also run through swb_apply_action (mode 2) and
swb_eval_task (mode 1) the way _direct.py calls them.  Clicks are in [0, 1], or (case_actions)
far outside it with a float64 motion cost, or carry NaN and +-inf components.

A bad Embodied direction follows the reference's state after its KeyError
(environment.py:93-95): the step is counted, nothing moves (no velocity update either), the
env reports reward NaN, step type MID and SWB_ENV_BAD_ACTION, and the unchanged scene is what
gets rendered.

Separate tests: the hit test on the vertices and edges of every shape against the oracle and
against exact rational arithmetic, and the Clustering metric against scikit-learn's
(tests/golden/clustering_metric.npz).  test_case_table_covers_the_step_paths runs without a GPU.
"""
import ctypes
import zlib
from fractions import Fraction

import numpy as np
import pytest

from oracle import oracle
from tests import fixtures

gpu = pytest.mark.gpu
INT32_MIN = -2 ** 31
AGGS = ('sum', 'mean', 'max', 'min')


def _case(name, S, E, action, dtype, T=12, K=2, nodes='goal', pos='f32', keep=True, mel=50,
          empty='front', vel=0.0, reset_mask=(), edge_pos=False, filter_sizes=(), direct=False,
          expect=(), actions='unit', scale=None, motion_cost=None):
  """expect: events (see _count) the case must produce at least once, besides FIRST steps.
  actions: see case_actions.  scale, motion_cost: the action space's, instead of drawn ones."""
  return dict(name=name, S=S, E=E, action=action, dtype=dtype, T=T, K=K, nodes=nodes, pos=pos,
              keep=keep, mel=mel, empty=empty, vel=vel, reset_mask=tuple(reset_mask),
              edge_pos=edge_pos, filter_sizes=tuple(filter_sizes), direct=direct,
              expect=tuple(expect), actions=actions, scale=scale, motion_cost=motion_cost)


CASES = [
    _case('select_f32_s1_e1', 1, 1, 'select_move', 'f32', direct=True),
    _case('select_f64_s2', 2, 3, 'select_move', 'f64', direct=True),
    _case('drag_f32_s5_mixed', 5, 5, 'drag_and_drop', 'f32', pos='mixed', direct=True),
    _case('drag_f64_s8_mixed', 8, 9, 'drag_and_drop', 'f64', pos='mixed', direct=True),
    _case('select_f32_s9_interleaved', 9, 17, 'select_move', 'f32', pos='mixed', empty='interleaved'),
    _case('select_f64_s17_f64pos', 17, 33, 'select_move', 'f64', pos='f64', empty='interleaved'),
    _case('drag_f32_s31', 31, 65, 'drag_and_drop', 'f32', pos='mixed', empty='interleaved'),
    _case('select_f64_s32_many', 32, 2049, 'select_move', 'f64', pos='mixed', T=6),
    _case('embodied_s7', 7, 33, 'embodied', 'i32', pos='mixed', T=16, direct=True,
          expect=('bad',)),
    _case('embodied_s32_f64', 32, 129, 'embodied', 'i32', pos='f64', T=10, expect=('bad',)),
    _case('edges_keep', 5, 65, 'select_move', 'f64', pos='mixed', edge_pos=True, vel=0.05),
    _case('edges_free', 5, 65, 'drag_and_drop', 'f32', pos='mixed', edge_pos=True, vel=0.05,
          keep=False, mel=4, nodes='goal_centre', expect=('last', 'success_and_oof')),
    _case('goal_filters', 32, 129, 'select_move', 'f32', pos='mixed',
          filter_sizes=(0, 1, 7, 8, 9, 15, 16, 17, 32), nodes='goal_filters'),
    _case('clustering_f32', 32, 257, 'select_move', 'f32', nodes='clustering', pos='f32',
          expect=('labels', 'zerodiv')),
    _case('clustering_f64', 32, 257, 'drag_and_drop', 'f64', nodes='clustering', pos='mixed',
          expect=('labels', 'zerodiv')),
    _case('clustering_small', 3, 65, 'select_move', 'f32', nodes='clustering', pos='f64',
          expect=('labels',)),
    _case('meta_all_aggs', 17, 65, 'select_move', 'f64', nodes='meta', pos='mixed'),
    _case('meta_nested_32_nodes', 32, 65, 'drag_and_drop', 'f32', nodes='meta_big', pos='mixed'),
    _case('episode_len1', 4, 33, 'select_move', 'f32', mel=1, K=3, T=9, expect=('last',)),
    _case('episode_len2_ring', 4, 33, 'embodied', 'i32', mel=2, K=3, T=20,
          expect=('last', 'bad')),
    _case('reset_mask', 6, 41, 'select_move', 'f64', mel=5, K=3, T=14, vel=0.02,
          reset_mask=(3, 4, 9), expect=('last', 'reset_on_last', 'reset_mid')),
    # clicks far outside [0, 1] and non-finite components, with a float64 motion cost
    _case('wide_f64_cost', 9, 65, 'select_move', 'f64', pos='mixed', keep=False, actions='wide',
          scale=3.0, motion_cost=0.7, direct=True, expect=('last',)),
    _case('nonfinite_f32', 5, 65, 'drag_and_drop', 'f32', pos='mixed', keep=False,
          actions='nonfinite', scale=3.0, motion_cost=0.7, direct=True, expect=('last',)),
    _case('nonfinite_f64_s32', 32, 129, 'select_move', 'f64', pos='mixed', keep=False,
          actions='nonfinite', scale=3.0, motion_cost=0.7, expect=('last',)),
    _case('nonfinite_f64_keep', 5, 33, 'drag_and_drop', 'f64', pos='mixed', actions='nonfinite',
          motion_cost=0.0),
]


# -- scenes, tasks and actions ------------------------------------------------------------------

def _scene_arrays(case, rng):
  E, K, S = case['E'], case['K'], case['S']
  shp = (E, K, S)
  shape = rng.randint(1, 13, shp).astype(np.uint8)
  if S > 2 and case['empty'] == 'front':
    shape[..., :rng.randint(0, S // 3 + 1)] = 0
  elif S > 2 and case['empty'] == 'interleaved':
    shape[rng.rand(*shp) < 0.25] = 0
  shape[..., -1] = np.maximum(shape[..., -1], 1)          # the Embodied body, and >= 1 sprite
  x, y = rng.uniform(0.05, 0.95, shp), rng.uniform(0.05, 0.95, shp)
  if case['edge_pos']:
    special = np.array([0.0, -0.0, 1.0, np.nextafter(1.0, 2.0), np.nextafter(0.0, -1.0),
                        np.nextafter(np.float32(1.0), np.float32(2.0)).astype(np.float64)])
    m = rng.rand(*shp) < 0.5
    x[m] = special[rng.randint(0, len(special), m.sum())]
    m = rng.rand(*shp) < 0.5
    y[m] = special[rng.randint(0, len(special), m.sum())]
  if case['pos'] == 'f32':
    f32 = np.ones(shp, np.uint8)
  elif case['pos'] == 'f64':
    f32 = np.zeros(shp, np.uint8)
  else:
    f32 = (rng.rand(*shp) < 0.5).astype(np.uint8)
  x = np.where(f32 > 0, x.astype(np.float32).astype(np.float64), x)
  y = np.where(f32 > 0, y.astype(np.float32).astype(np.float64), y)
  v = case['vel']
  member = rng.randint(0, 2 ** 16, shp).astype(np.uint32)
  if case['filter_sizes']:
    # filter bit i holds exactly filter_sizes[i] of the occupied sprites (fewer if S is short)
    member[:] = 0
    for i, k in enumerate(case['filter_sizes']):
      for e in range(E):
        for c in range(K):
          occ = np.nonzero(shape[e, c])[0]
          pick = rng.permutation(occ)[:k] if rng.rand() < 0.8 else occ[:k]
          member[e, c, pick] |= np.uint32(1 << i)
  elif case['nodes'] == 'clustering':
    lab = rng.randint(0, 16 if rng.rand() < 0.5 else 3, shp)
    member = np.where(rng.rand(*shp) < 0.1, 0, 1 << lab).astype(np.uint32)
    # a tenth of the envs: every sprite in cluster 0 (ValueError); another tenth: each cluster
    # on one point of its own, exact in float32 (all intra distances 0: ZeroDivisionError)
    one = rng.rand(E) < 0.1
    member[one] = 1
    flat = (rng.rand(E) < 0.1) & ~one
    grid = rng.randint(4, 60, (16, 2)) / 64.0
    x[flat], y[flat] = grid[lab[flat], 0], grid[lab[flat], 1]
  return dict(
      x=x, y=y, pos_f32=f32, shape=shape, angle=rng.choice([0., 30., 45., 90., 77.], shp),
      scale=rng.choice([0.05, 0.1, 0.2, 0.4], shp), c0=np.zeros(shp), c1=np.zeros(shp),
      c2=np.zeros(shp), color_f32=np.zeros(shp, np.uint8),
      vx=rng.choice([0., v, -v], shp) if v else np.zeros(shp),
      vy=rng.choice([0., v, -v], shp) if v else np.zeros(shp), member=member,
      rgb=np.zeros(shp + (3,), np.uint8))


def _goal(filter_slot, rng, sparse=False):
  return dict(kind='find_goal', filter_slot=int(filter_slot),
              goal=[float(rng.uniform(0, 1)), float(rng.uniform(0, 1))],
              weights=[float(rng.choice([1.0, 0.5, 2.0])), float(rng.choice([1.0, 0.25]))],
              terminate_distance=float(rng.choice([0.05, 0.3, 2.0])),
              terminate_bonus=float(rng.choice([0.0, 1.5])), raw_reward_multiplier=50.0,
              sparse_reward=bool(sparse))


def _clustering(rng, n):
  return dict(kind='clustering', cluster_slots=list(range(n)),
              termination_threshold=float(rng.choice([0.5, 2.5, 100.0])),
              terminate_bonus=float(rng.choice([0.0, 1.0])), sparse_reward=bool(rng.rand() < 0.3),
              reward_range=10.0)


def _meta(children, agg, crit, bonus=0.5):
  return dict(kind='meta', children=list(children), aggregator=agg, criterion=crit,
              terminate_bonus=bonus)


def case_nodes(case, rng):
  kind = case['nodes']
  if kind == 'goal':
    return [_goal(-1, rng)]
  if kind == 'goal_centre':   # succeeds while the sprites of filter 0 stay near the centre
    return [dict(_goal(0, rng), goal=[0.5, 0.5], terminate_distance=0.45)]
  if kind == 'goal_filters':   # one node per filter size, dense and sparse, summed
    nodes = [_goal(i, rng, sparse=(i % 2 == 1)) for i in range(len(case['filter_sizes']))]
    return nodes + [_meta(range(len(nodes)), 'sum', 'all', 0.0)]
  if kind == 'clustering':
    return [_clustering(rng, 16 if case['S'] > 3 else 2)]
  if kind == 'meta':         # every aggregator with both criteria; empty filter 20 -> NaN child
    leaves = [_goal(-1, rng), _goal(0, rng, sparse=True), _goal(20, rng), _goal(1, rng)]
    nodes = list(leaves)
    for agg in AGGS:
      for crit in ('all', 'any'):
        nodes.append(_meta(range(4), agg, crit))
    nodes.append(_meta(range(4, len(nodes)), 'mean', 'any', 1.0))   # nested
    return nodes
  if kind == 'meta_big':     # 32 nodes, a 16-child MetaAggregated, nesting three deep
    leaves = [_goal(i % 18, rng, sparse=(i % 3 == 0)) for i in range(16)]
    nodes = list(leaves)
    nodes.append(_meta(range(16), 'max', 'any'))                      # 16
    for j, agg in enumerate(AGGS * 3):                                # 17..28
      nodes.append(_meta([j, j + 1, 16], agg, ('all', 'any')[j % 2]))
    nodes.append(_meta(range(17, 29), 'min', 'all'))                  # 29
    nodes.append(_meta([29, 16, 3], 'sum', 'any'))                    # 30
    nodes.append(_meta([30, 29], 'mean', 'all', 2.0))                 # 31
    return nodes
  raise ValueError(kind)


def case_actions(case, arrs, rng, T):
  """(T, E, 4) float clicks -- half of them on a sprite of the env's first scene -- or (T, E, 2)
  int32 Embodied actions with carry 0, 1, 2, -1 and, mid-episode, bad directions.

  case['actions'] of clicks: 'unit' in [0, 1]; 'wide' with every component in [-3, 4] (the
  click position too, when it is not on a sprite); 'nonfinite' as 'unit', with NaN, +inf or
  -inf in a random subset of the components of a third of the actions."""
  E = case['E']
  if case['action'] == 'embodied':
    a = np.zeros((T, E, 2), np.int32)
    a[..., 0] = rng.choice([0, 1, 2, -1], (T, E))
    a[..., 1] = rng.randint(0, 4, (T, E))
    bad = rng.rand(T, E) < 0.12
    bad[0] = False
    a[..., 1][bad] = rng.choice([-1, 4, INT32_MIN], bad.sum())
    return a
  a = rng.uniform(0, 1, (T, E, 4))
  if case['actions'] == 'wide':
    a = rng.uniform(-3, 4, (T, E, 4))
  occ = arrs['shape'][:, 0] > 0
  for t in range(T):
    for e in range(E):
      if rng.rand() < 0.5:
        s = rng.choice(np.nonzero(occ[e])[0])
        a[t, e, 0] = arrs['x'][e, 0, s] + rng.normal(0, 0.01)
        a[t, e, 1] = arrs['y'][e, 0, s] + rng.normal(0, 0.01)
  if case['actions'] == 'nonfinite':
    hit = rng.rand(T, E) < 1 / 3.
    comp = rng.rand(T, E, 4) < 0.4
    vals = np.array([np.nan, np.inf, -np.inf])[rng.randint(0, 3, (T, E, 4))]
    a = np.where(hit[..., None] & comp, vals, a)
  return a.astype(np.float32 if case['dtype'] == 'f32' else np.float64)


# -- the runs -----------------------------------------------------------------------------------

def _reset_mask(case, t):
  return np.random.RandomState(t).rand(case['E']) < 0.5


def _count_mask(ev, bo, mask):
  """A masked reset on an env that has just terminated, and on one in mid-episode."""
  ev['reset_on_last'] += int((mask & (bo.reset_next == 1)).sum())
  ev['reset_mid'] += int((mask & (bo.reset_next == 0) & (bo.step_count > 0)).sum())


def _count(ev, bo):
  """What the oracle's last step did, per event."""
  st, err = bo.step_type, bo.err
  ev['first'] += int((st == oracle.STEP_FIRST).sum())
  ev['last'] += int((st == oracle.STEP_LAST).sum())
  ev['bad'] += int(((err & oracle.ERR_BAD_ACTION) > 0).sum())
  ev['labels'] += int(((err & oracle.ERR_CLUSTER_LABELS) > 0).sum())
  ev['zerodiv'] += int(((err & oracle.ERR_CLUSTER_ZERODIV) > 0).sum())
  c = bo.cur
  oof = ((c['shape'] > 0) & ~((c['x'] >= 0) & (c['y'] >= 0) & (c['x'] <= 1) & (c['y'] <= 1))).any(1)
  ev['success_and_oof'] += int(((st == oracle.STEP_LAST) & (bo.success > 0) & oof).sum())


def _new_events():
  return dict.fromkeys(('first', 'last', 'bad', 'labels', 'zerodiv', 'success_and_oof',
                        'reset_on_last', 'reset_mid'), 0)


def oracle_events(case):
  """Runs a case on the oracle alone (no GPU) and counts its events."""
  arrs, nodes, action, acts = _setup(case)
  bo = _oracle(case, nodes, arrs, action)
  ev = _new_events()
  for t in range(case['T']):
    if t in case['reset_mask']:
      mask = _reset_mask(case, t)
      _count_mask(ev, bo, mask)
      bo.reset_next[mask] = 1
    bo.step(acts[t])
    _count(ev, bo)
  return ev

def _engine(case, nodes, arrs, action):
  from spriteworld_b200 import constants, engine, scene
  E, K, S = case['E'], case['K'], case['S']
  eng = engine.Engine(E, S, K, action, nodes, constants.SHAPES, keep_in_frame=case['keep'],
                      max_episode_length=case['mel'])
  flat = {k: v.reshape((E * K,) + v.shape[2:]) for k, v in arrs.items()}
  b = scene.batch_from_factor_arrays(
      flat['x'], flat['y'], flat['pos_f32'], flat['shape'], flat['angle'], flat['scale'],
      flat['c0'], flat['c1'], flat['c2'], flat['vx'], flat['vy'], flat['member'], flat['rgb'])
  eng.upload_scenes(b, np.repeat(np.arange(E), K), np.tile(np.arange(K), E))
  return eng


def _oracle(case, nodes, arrs, action):
  from spriteworld_b200 import constants
  cfg = oracle.with_device_sqrt(fixtures.env_cfg_from_meta(dict(
      action=action, keep_in_frame=case['keep'], max_episode_length=case['mel'], nodes=nodes)))
  return oracle.BatchOracle(cfg, oracle.shape_table(constants.SHAPES), None,
                            fixtures.records_from_arrays(arrs))


def _setup(case):
  rng = np.random.RandomState(zlib.crc32(case['name'].encode()))
  arrs = _scene_arrays(case, rng)
  nodes = case_nodes(case, rng)
  action = dict(kind=case['action'], scale=float(rng.choice([0.5, 1.0])),
                motion_cost=float(rng.choice([0.0, 0.25])))
  if case['action'] == 'embodied':
    action['scale'] = 0.05
  if case['scale'] is not None:
    action['scale'] = case['scale']
  if case['motion_cost'] is not None:
    action['motion_cost'] = case['motion_cost']
  acts = case_actions(case, arrs, rng, case['T'])
  return arrs, nodes, action, acts


@gpu
@pytest.mark.parametrize('host', [False, True], ids=['device', 'host'])
@pytest.mark.parametrize('case', CASES, ids=[c['name'] for c in CASES])
def test_step_matches_oracle(case, host):
  import torch
  arrs, nodes, action, acts = _setup(case)
  eng = _engine(case, nodes, arrs, action)
  bo = _oracle(case, nodes, arrs, action)
  serial0 = eng.download_state_serial()
  n_first = np.zeros(case['E'], np.int64)
  seen = _new_events()
  for t in range(case['T']):
    if t in case['reset_mask']:
      mask = _reset_mask(case, t)
      _count_mask(seen, bo, mask)
      eng.request_reset(torch.from_numpy(mask.astype(np.uint8)))
      bo.reset_next[mask] = 1
    if host:
      reward, step_type, success, status, _ = eng.step_host(acts[t])
    else:
      res = eng.step(torch.from_numpy(acts[t]).to(eng.device))
      reward, step_type, success, status = (a.cpu().numpy() for a in (
          res.reward, res.step_type, res.success, res.status))
    bo.step(acts[t])
    st = eng.download_state()
    where = (case['name'], t)
    assert np.array_equal(step_type, bo.step_type), where
    assert np.array_equal(success, bo.success), where
    assert np.array_equal(status, bo.err), where
    assert np.array_equal(reward, bo.reward, equal_nan=True), where
    assert np.array_equal(st['cursor'], bo.cursor), where
    assert np.array_equal(st['step_count'], bo.step_count), where
    assert np.array_equal(st['reset_next'], bo.reset_next), where
    occ = bo.cur['shape'] > 0
    assert np.array_equal(st['pos_x'][occ], bo.cur['x'][occ], equal_nan=True), where
    assert np.array_equal(st['pos_y'][occ], bo.cur['y'][occ], equal_nan=True), where
    n_first += bo.step_type == oracle.STEP_FIRST
    assert np.array_equal(eng.download_state_serial() - serial0, n_first), where
    _count(seen, bo)
  eng.close()
  # the case did what it is there for
  assert seen['first'] >= case['E']
  for event in case['expect']:
    assert seen[event] > 0, (case['name'], event)


@gpu
@pytest.mark.parametrize('case', [c for c in CASES if c['direct']], ids=lambda c: c['name'])
def test_apply_action_and_eval_task_match_oracle(case):
  """swb_apply_action (mode 2) and swb_eval_task (mode 1) on the live state, as _direct.py
  calls them, against oracle.action_step / oracle.task_eval."""
  import torch
  from spriteworld_b200 import _native
  arrs, nodes, action, acts = _setup(case)
  eng = _engine(case, nodes, arrs, action)
  bo = _oracle(case, nodes, arrs, action)
  E = case['E']
  cur = bo.pool[:, 0].copy()
  eng.upload_state(pos_x=cur['x'], pos_y=cur['y'], cursor=np.zeros(E), step_count=np.zeros(E),
                   reset_next=np.zeros(E))
  dtype = {'f32': _native.DTYPE_F32, 'f64': _native.DTYPE_F64, 'i32': _native.DTYPE_I32}[case['dtype']]
  for t in range(case['T']):
    a = torch.from_numpy(np.ascontiguousarray(acts[t])).to(eng.device)
    _native.check(eng._lib.swb_apply_action(eng._h, ctypes.c_void_p(a.data_ptr()), dtype,
                                            eng._out, eng._stream()))
    st = eng.download_state()
    cost = eng._reward.cpu().numpy()
    status = eng._status.cpu().numpy()
    for e in range(E):
      try:
        want_cost, _ = oracle.action_step(bo.cfg, bo.tab, cur[e], acts[t][e], case['dtype'] == 'f32')
        assert status[e] == 0 and np.array_equal(cost[e], want_cost, equal_nan=True), (
            case['name'], t, e)
      except KeyError:
        assert status[e] == _native.ENV_BAD_ACTION and cost[e] == 0.0, (case['name'], t, e)
    occ = cur['shape'] > 0
    assert np.array_equal(st['pos_x'][occ], cur['x'][occ], equal_nan=True), (case['name'], t)
    assert np.array_equal(st['pos_y'][occ], cur['y'][occ], equal_nan=True), (case['name'], t)
    _native.check(eng._lib.swb_eval_task(eng._h, eng._out, eng._stream()))
    got_r, got_s, got_e = (a.cpu().numpy() for a in (eng._reward, eng._success, eng._status))
    for e in range(E):
      r, s, err = oracle.task_eval(bo.cfg, cur[e])
      assert np.array_equal(got_r[e], r, equal_nan=True), (case['name'], t, e)
      assert got_s[e] == s and got_e[e] == err, (case['name'], t, e)
  eng.close()


# -- Clustering against scikit-learn ------------------------------------------------------------

@gpu
def test_eval_task_clustering_matches_oracle_and_scikit_learn():
  from spriteworld_b200 import _native, constants, engine, scene
  cm = fixtures.ClusteringMetric()
  arrs = cm.scenes()
  nodes = [cm.node()]
  eng = engine.Engine(cm.L, 32, 1, dict(kind='select_move', scale=1.0, motion_cost=0.0), nodes,
                      constants.SHAPES)
  b = scene.batch_from_factor_arrays(
      arrs['x'], arrs['y'], arrs['pos_f32'], arrs['shape'], arrs['angle'], arrs['scale'],
      arrs['c0'], arrs['c1'], arrs['c2'], arrs['vx'], arrs['vy'], arrs['member'], arrs['rgb'])
  eng.upload_scenes(b, np.arange(cm.L), np.zeros(cm.L, int))
  eng.upload_state(pos_x=b['x'], pos_y=b['y'], cursor=np.zeros(cm.L), step_count=np.zeros(cm.L),
                   reset_next=np.zeros(cm.L))
  _native.check(eng._lib.swb_eval_task(eng._h, eng._out, eng._stream()))
  got, status = eng._reward.cpu().numpy(), eng._status.cpu().numpy()
  eng.close()
  cfg = fixtures.env_cfg_from_meta(dict(action=dict(kind='select_move', scale=1.0, motion_cost=0.0),
                                        keep_in_frame=True, max_episode_length=10, nodes=nodes))
  rec = fixtures.records_from_arrays(arrs)
  want = np.array([oracle.task_eval(cfg, rec[i])[0] for i in range(cm.L)])
  assert np.array_equal(got, want, equal_nan=True)                      # = the oracle, exactly
  assert np.array_equal(status, cm.err)                                  # the same exceptions
  ok = cm.err == 0
  assert np.array_equal(got[ok], cm.metric[ok])                          # = scikit-learn


# -- hit-test boundaries ------------------------------------------------------------------------

ANGLES = (0., 30., 45., 77., 90., 180., 359.)
SCALES = (1e-3, 0.1, 0.5, 2.0)


def _clicks(verts, pos, rng, af32):
  """Click points (world coordinates) at the transformed vertices, edge midpoints, their +-1 ULP
  neighbours in x and in y, the centre and random points."""
  n = len(verts)
  base = [verts, 0.5 * (verts + np.roll(verts, -1, 0))]
  pts = np.concatenate(base) + pos
  dt = np.float32 if af32 else np.float64
  pts = pts.astype(dt)
  out = [pts]
  for axis in (0, 1):
    for d in (-np.inf, np.inf):
      q = pts.copy()
      q[:, axis] = np.nextafter(q[:, axis], dt(d))
      out.append(q)
  out.append(np.array([pos], dt))
  out.append((pos + rng.uniform(-1, 1, (max(4, n // 2), 2)) * np.abs(verts).max()).astype(dt))
  return np.concatenate(out)


def _exact_inside(tx, ty, cv):
  """Even-odd test of (tx, ty) against the polygon cv in exact rationals, and the smallest
  relative distance of the point from an edge's line among the edges its ray crosses."""
  X, Y = Fraction(tx), Fraction(ty)
  inside, margin = False, None
  n = len(cv)
  for i in range(n):
    ax, ay = Fraction(cv[i][0]), Fraction(cv[i][1])
    bx, by = Fraction(cv[(i + 1) % n][0]), Fraction(cv[(i + 1) % n][1])
    if (ay > Y) != (by > Y):
      xc = ax + (Y - ay) * (bx - ax) / (by - ay)
      if X < xc:
        inside = not inside
    cross = (bx - ax) * (Y - ay) - (by - ay) * (X - ax)
    length = abs(bx - ax) + abs(by - ay)
    rel = abs(cross) / (length * length) if length else Fraction(0)
    margin = rel if margin is None else min(margin, rel)
    if ay == Y or by == Y:
      margin = Fraction(0)
  return inside, margin


@gpu
@pytest.mark.parametrize('af32', [True, False], ids=['f32_action', 'f64_action'])
def test_hit_test_boundaries(af32):
  """One sprite per env (plus, in half the envs, a second overlapping sprite drawn on top of
  it, for the top-most-first order), a click with non-zero motion and keep_in_frame off, so a
  hit is a move.  The kernel agrees with the oracle's action_step on every click, and with an
  exact even-odd test wherever the click is not within a relative 1e-9 of an edge."""
  import torch
  from spriteworld_b200 import _native, constants, engine, scene
  rng = np.random.RandomState(5 if af32 else 6)
  tab = oracle.shape_table(constants.SHAPES)
  rows = []   # (shape, angle, scale, pos, pos_f32, click, second sprite?)
  for sid in range(1, 13):
    for ang in ANGLES:
      for sc in SCALES:
        for pf32 in (True, False):
          pos = rng.uniform(0.2, 0.8, 2)
          if pf32:
            pos = pos.astype(np.float32).astype(np.float64)
          m = oracle.centred_matrix(sc, ang)
          v = np.array([tab.verts[sid][i][:] for i in range(tab.n_verts[sid])])
          cv = np.stack([(m[0] * v[:, 0] + m[1] * v[:, 1]) + 0.0,
                         (m[2] * v[:, 0] + m[3] * v[:, 1]) + 0.0], 1)
          for c in _clicks(cv, pos, rng, af32):
            rows.append((sid, ang, sc, pos, pf32, c, rng.rand() < 0.5))
  E = len(rows)
  S = 2
  z = np.zeros((E, S))
  arrs = dict(x=z.copy(), y=z.copy(), pos_f32=np.zeros((E, S), np.uint8),
              shape=np.zeros((E, S), np.uint8), angle=z.copy(), scale=np.full((E, S), 0.1),
              c0=z.copy(), c1=z.copy(), c2=z.copy(), vx=z.copy(), vy=z.copy(),
              member=np.zeros((E, S), np.uint32), rgb=np.zeros((E, S, 3), np.uint8))
  acts = np.zeros((E, 4), np.float32 if af32 else np.float64)
  for e, (sid, ang, sc, pos, pf32, c, two) in enumerate(rows):
    k = 0 if two else 1       # the sprite under test sits below the second one, if any
    arrs['shape'][e, k], arrs['angle'][e, k], arrs['scale'][e, k] = sid, ang, sc
    arrs['x'][e, k], arrs['y'][e, k], arrs['pos_f32'][e, k] = pos[0], pos[1], pf32
    if two:
      arrs['shape'][e, 1], arrs['angle'][e, 1], arrs['scale'][e, 1] = 2, 0.0, sc * 0.5
      arrs['x'][e, 1], arrs['y'][e, 1], arrs['pos_f32'][e, 1] = pos[0] + sc * 0.3, pos[1], pf32
    acts[e] = (c[0], c[1], 0.75, 0.25)
  action = dict(kind='select_move', scale=1.0, motion_cost=0.0)
  eng = engine.Engine(E, S, 1, action, [dict(kind='no_reward')], constants.SHAPES,
                      keep_in_frame=False)
  b = scene.batch_from_factor_arrays(
      arrs['x'], arrs['y'], arrs['pos_f32'], arrs['shape'], arrs['angle'], arrs['scale'],
      arrs['c0'], arrs['c1'], arrs['c2'], arrs['vx'], arrs['vy'], arrs['member'], arrs['rgb'])
  eng.upload_scenes(b, np.arange(E), np.zeros(E, int))
  eng.upload_state(pos_x=b['x'], pos_y=b['y'], cursor=np.zeros(E), step_count=np.zeros(E),
                   reset_next=np.zeros(E))
  a = torch.from_numpy(acts).to(eng.device)
  _native.check(eng._lib.swb_apply_action(
      eng._h, ctypes.c_void_p(a.data_ptr()), _native.DTYPE_F32 if af32 else _native.DTYPE_F64,
      eng._out, eng._stream()))
  st = eng.download_state()
  eng.close()
  moved = (st['pos_x'] != b['x']) | (st['pos_y'] != b['y'])
  rec = fixtures.records_from_arrays(arrs)
  cfg = fixtures.env_cfg_from_meta(dict(action=action, keep_in_frame=False, max_episode_length=10,
                                        nodes=[dict(kind='no_reward')]))
  n_in = n_checked = 0
  for e, (sid, ang, sc, pos, pf32, c, two) in enumerate(rows):
    sp = rec[e].copy()
    oracle.action_step(cfg, tab, sp, acts[e], af32)
    want = (sp['x'] != rec[e]['x']) | (sp['y'] != rec[e]['y'])
    assert np.array_equal(moved[e], want), (e, sid, ang, sc, pf32, c.tolist(), two)
    k = 0 if two else 1
    if two and moved[e, 1]:
      continue                # the click went to the sprite on top
    n_in += bool(moved[e, k])
    if e % 7 == 0:            # the exact test is slow: every seventh click
      p_f32 = bool(af32) and pf32
      tx = float(np.float32(c[0]) - np.float32(pos[0])) if p_f32 else float(c[0]) - float(pos[0])
      ty = float(np.float32(c[1]) - np.float32(pos[1])) if p_f32 else float(c[1]) - float(pos[1])
      m = oracle.centred_matrix(sc, ang)
      v = [(tab.verts[sid][i][0], tab.verts[sid][i][1]) for i in range(tab.n_verts[sid])]
      cv = [((m[0] * vx + m[1] * vy) + 0.0, (m[2] * vx + m[3] * vy) + 0.0) for vx, vy in v]
      inside, margin = _exact_inside(tx, ty, cv)
      if margin > Fraction(1, 10 ** 9):
        n_checked += 1
        assert bool(moved[e, k]) == inside, (e, sid, ang, sc, pf32, c.tolist())
  assert n_in > E // 10 and n_checked > 300


# -- the table covers what it should ------------------------------------------------------------

def test_case_table_covers_the_step_paths():
  """Runs without a GPU: fails if CASES stops covering one of the paths of the step kernel."""
  Ss = {c['S'] for c in CASES}
  assert {1, 2, 5, 8, 9, 17, 31, 32} <= Ss
  Es = {c['E'] for c in CASES}
  assert {1, 3, 5} <= Es and any(e % 4 == 1 and e > 5 for e in Es) and max(Es) >= 2000
  combos = {(c['action'], c['dtype']) for c in CASES}
  assert {('select_move', 'f32'), ('select_move', 'f64'), ('drag_and_drop', 'f32'),
          ('drag_and_drop', 'f64'), ('embodied', 'i32')} <= combos
  assert {(c['dtype'], c['pos']) for c in CASES} >= {('f32', 'mixed'), ('f64', 'mixed')}
  assert {c['empty'] for c in CASES} >= {'front', 'interleaved'}
  assert any(c['edge_pos'] and c['keep'] for c in CASES)
  assert any(c['edge_pos'] and not c['keep'] for c in CASES)
  sizes = set().union(*[c['filter_sizes'] for c in CASES])
  assert {0, 1, 7, 8, 9, 15, 16, 17, 32} <= sizes
  kinds = {c['nodes'] for c in CASES}
  assert {'goal', 'goal_filters', 'clustering', 'meta', 'meta_big'} <= kinds
  assert {(c['nodes'], c['pos']) for c in CASES if c['nodes'] == 'clustering'} >= {
      ('clustering', 'f32'), ('clustering', 'mixed')}
  rng = np.random.RandomState(0)
  big = case_nodes([c for c in CASES if c['nodes'] == 'meta_big'][0], rng)
  assert len(big) == 32 and max(len(n.get('children', ())) for n in big) == 16
  metas = [n for c in CASES if c['nodes'].startswith('meta')
           for n in case_nodes(c, np.random.RandomState(0)) if n['kind'] == 'meta']
  assert {(n['aggregator'], n['criterion']) for n in metas} >= {
      (a, k) for a in AGGS for k in ('all', 'any')}
  assert {1, 2} <= {c['mel'] for c in CASES}
  assert any(c['K'] == 3 and c['mel'] <= 2 and c['T'] >= 6 * c['mel'] for c in CASES)
  assert any(c['reset_mask'] for c in CASES)
  emb = [c for c in CASES if c['action'] == 'embodied']
  a = case_actions(emb[0], None, np.random.RandomState(0), 40)
  assert set(np.unique(a[..., 0])) == {-1, 0, 1, 2}
  assert {-1, 4, INT32_MIN} <= set(np.unique(a[..., 1]).tolist())
  assert any(c['direct'] for c in CASES if c['action'] == 'embodied')
  assert {c['dtype'] for c in CASES if c['direct']} == {'f32', 'f64', 'i32'}
  # a float64 cost with a nonzero motion cost (np.linalg.norm's fused dot), clicks outside
  # [0, 1] and non-finite action components, with keep_in_frame off and on
  f64_cost, nonfinite, wide = set(), set(), set()
  for c in CASES:
    if c['action'] == 'embodied':
      continue
    _, _, action, acts = _setup(c)
    if c['dtype'] == 'f64' and action['motion_cost'] > 0:
      f64_cost.add(c['name'])
    if not np.isfinite(acts).all():
      nonfinite.add((c['dtype'], c['keep']))
    if ((acts < 0) | (acts > 1)).any() and action['motion_cost'] > 0 and action['scale'] > 1:
      wide.add(c['dtype'])
  assert f64_cost and 'f64' in wide
  assert {('f32', False), ('f64', False), ('f64', True)} <= nonfinite
  # the events the step path must meet somewhere in the table, checked on the oracle
  expected = {e for c in CASES for e in c['expect']}
  assert expected >= {'bad', 'labels', 'zerodiv', 'last', 'success_and_oof', 'reset_on_last',
                      'reset_mid'}
  for c in CASES:
    if c['expect']:
      ev = oracle_events(c)
      for event in c['expect']:
        assert ev[event] > 0, (c['name'], event, ev)
