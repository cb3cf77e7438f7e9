"""Env record evaluation (evaluate_kernel in csrc/swb_rollout.cuh, swb_evaluate_states) against the CPU
oracle, bit for bit, over every task tree of the step sweep (tests/test_gpu_step_sweep.py).

1. Every case of the step sweep runs its T steps and saves every env after each step (and after each
   masked reset request).  Evaluated, the records give the oracle's task_eval in its sqrt mode
   (oracle.with_device_sqrt) on the sprites decoded from them: reward bit for bit (NaN equal to
   NaN), success and status exactly.  Compared are every record about to reset, every record with a
   sprite outside [0, 1] or at a non-finite position, and a seeded sample of the rest (_pick).
2. The same records, loaded into an engine of the same configuration, give the same values through
   swb_eval_task (step_kernel mode 1): record staging equals live staging on every task tree.
3. The 1600 Clustering layouts of tests/golden/clustering_metric.npz, saved as records, give
   scikit-learn's metric exactly, the float64 metric for float32 layouts too.
4. Trees of FindGoalPosition nodes with 1, 3 and 8 goal slots under MetaAggregated evaluate as the
   constant-goal tree with the record's goals, or the overriding goals, substituted (DESIGN §3.3a).
5. Edited shape bytes (13, 255, an id the engine has no vertex table for) evaluate as a load
   sanitises them; permuted and repeated records, counts 0 to 4097, outputs at unaligned addresses
   inside guarded buffers; one launch per call, none for n = 0, and the engine unchanged.
6. Every live step of a rollout without motion cost reports what evaluate says of its trajectory
   record.
test_case_table_covers_the_evaluate_paths runs without a GPU.
"""
import zlib

import numpy as np
import pytest

from oracle import oracle
from tests import fixtures
from tests import test_gpu_step_sweep as sweep

gpu = pytest.mark.gpu
MAX_PICK = 1200        # records of one case compared with the oracle, about
LACKING = 'star_5'     # the shape _lacking_shapes() has no vertex table for
# (name, step-sweep case whose records are evaluated, {node index: goal slot})
GOAL_TREES = [
    ('g1', 'meta_all_aggs', {3: 0}),
    ('g3', 'meta_all_aggs', {0: 2, 1: 0, 3: 1}),
    ('g8', 'meta_nested_32_nodes', {1: 5, 2: 0, 4: 7, 5: 1, 7: 3, 8: 6, 10: 2, 11: 4}),
]
# (step-sweep case whose records get edited shape bytes, task tree to evaluate them on: None for the
# case's own)
EDITS = [('clustering_f64', None), ('meta_all_aggs', None), ('drag_f64_s8_mixed', [dict(kind='no_reward')])]


def _named(name):
  return next(c for c in sweep.CASES if c['name'] == name)


def _seed(case, k):
  return (zlib.crc32(case['name'].encode()) + k) % 2 ** 32


def _lacking_shapes():
  from spriteworld_b200 import constants
  return dict(constants.SHAPES, **{LACKING: np.zeros((0, 2))})


def _cfg(case, action, nodes):
  """The oracle's configuration of a tree, in sqrt mode; a node's goal is its `goal` entry."""
  return oracle.with_device_sqrt(fixtures.env_cfg_from_meta(dict(
      action=action, keep_in_frame=case['keep'], max_episode_length=case['mel'], nodes=nodes)))


def _constant_goals(nodes, goals):
  """The tree with goal slot g's node taking goals[g] as its constant goal."""
  return [dict(nd, goal=[float(goals[nd['goal_slot'], 0]), float(goals[nd['goal_slot'], 1])])
          if nd.get('goal_slot', -1) >= 0 else nd for nd in nodes]


# -- which records meet the oracle --------------------------------------------------------------

def _far(x, y, shape):
  """Records with an occupied slot outside [0, 1] or at a non-finite position."""
  return ((shape > 0) & ~((x >= 0) & (x <= 1) & (y >= 0) & (y <= 1))).any(1)


def _pick(case, x, y, shape, reset_next):
  """Indices of the records compared with the oracle: every record about to reset, every record with
  an occupied slot outside [0, 1] or at a non-finite position, and a seeded sample of the rest; about
  MAX_PICK in all.  x, y, shape: (n, S) as the records hold them (shape sanitised); reset_next (n,)."""
  special = (reset_next == 1) | _far(x, y, shape)
  rng = np.random.RandomState(_seed(case, 1))
  u = rng.rand(len(x))
  n_sp = int(special.sum())
  p_sp = min(1.0, MAX_PICK / 2 / max(1, n_sp))
  p_rest = min(1.0, (MAX_PICK - p_sp * n_sp) / max(1, len(x) - n_sp))
  return np.nonzero(np.where(special, u < p_sp, u < p_rest))[0]


def _oracle_saves(case):
  """The oracle's run of a case, saved as _saved saves it: (cfg, sprites (n, S), reset_next (n,))."""
  arrs, nodes, action, acts = sweep._setup(case)
  bo = sweep._oracle(case, nodes, arrs, action)
  cur, rn = [], []
  for t in range(case['T']):
    if t in case['reset_mask']:
      bo.reset_next[sweep._reset_mask(case, t)] = 1
      cur.append(bo.cur.copy())
      rn.append(bo.reset_next.copy())
    bo.step(acts[t])
    cur.append(bo.cur.copy())
    rn.append(bo.reset_next.copy())
  return bo.cfg, np.concatenate(cur), np.concatenate(rn)


def _oracle_values(cfgs, sprites):
  """oracle.task_eval of each row of `sprites` (n, S) under cfgs[i] (or one cfg for all)."""
  out = [oracle.task_eval(cfgs if isinstance(cfgs, oracle.EnvCfg) else cfgs[i], sprites[i])
         for i in range(len(sprites))]
  return (np.array([o[0] for o in out], np.float64), np.array([o[1] for o in out], np.uint8),
          np.array([o[2] for o in out], np.uint8))


# -- the device side ----------------------------------------------------------------------------

def _bits(a):
  """float64 values as int64 bits, every NaN as one NaN."""
  a = np.asarray(a, np.float64)
  return np.where(np.isnan(a), np.nan, a).view(np.int64)


def _assert_same(got, want, where):
  """(reward, success, status) host arrays: reward bit for bit, NaN equal to NaN; the rest exactly."""
  bad = (_bits(got[0]) != _bits(want[0])) | (got[1] != want[1]) | (got[2] != want[2])
  i = np.nonzero(bad)[0][:4]
  assert not bad.any(), (where, int(bad.sum()), i, [(g[i], w[i]) for g, w in zip(got, want)])


def _host(outputs):
  return tuple(t.cpu().numpy() for t in outputs)


def _saved(case):
  """The case's engine after its T steps, and the EnvStates saved after every step and after every
  masked reset request (record k * E + e: env e at save k)."""
  import torch
  from spriteworld_b200 import engine
  arrs, nodes, action, acts = sweep._setup(case)
  eng = sweep._engine(case, nodes, arrs, action)
  saves = []
  for t in range(case['T']):
    if t in case['reset_mask']:
      eng.request_reset(torch.from_numpy(sweep._reset_mask(case, t).astype(np.uint8)))
      saves.append(eng.save_envs())
    eng.step(torch.from_numpy(acts[t]).to(eng.device))
    saves.append(eng.save_envs())
  return eng, engine.EnvStates.cat(saves), (arrs, nodes, action, acts)


def _sprites(host, idx, shape_ids):
  """Oracle sprite arrays (len(idx), S) of records idx of EnvStates.to_host() output, with the shape
  ids a load makes of them (shape_ids: engine.shape_id_table)."""
  f = host['factors'][idx]
  rec = fixtures.records_from_arrays(dict(
      x=host['pos_x'][idx], y=host['pos_y'][idx], vx=host['vx'][idx], vy=host['vy'][idx],
      member=host['member'][idx], shape=shape_ids[host['shape'][idx]], pos_f32=host['pos_f32'][idx],
      rgb=host['rgb'][idx], scale=f[..., 0], angle=f[..., 1]))
  for k in ('m00', 'm01', 'm10', 'm11'):
    rec[k] = host[k][idx]
  return rec


def _eval_task(eng):
  """swb_eval_task (step_kernel mode 1): the task value of every live env."""
  from spriteworld_b200 import _native
  _native.check(eng._lib.swb_eval_task(eng._h, eng._out, eng._stream()))
  return _host((eng._reward, eng._success, eng._status))


def _two_paths(case, action, nodes, states, shapes=None, goals=None):
  """(evaluate, swb_eval_task after load_envs) of `states` on a new engine of the case's configuration
  with task tree `nodes` and one env per record; evaluate with `goals` if given.  Each is checked to
  be one launch; evaluate changes nothing of the engine."""
  import torch
  from spriteworld_b200 import constants, engine
  G = states.n_goals
  eng = engine.Engine(len(states), case['S'], 1, action, nodes, constants.SHAPES if shapes is None else shapes,
                      keep_in_frame=case['keep'], max_episode_length=case['mel'])
  assert eng.n_goals == G
  states = engine.EnvStates(states.data, states.span_class, eng.signature, case['S'], G)
  before, launches = eng.save_state(), eng.launch_count()
  got = _host(eng.evaluate(states, None if goals is None else torch.from_numpy(goals).to(eng.device)))
  assert eng.launch_count() == launches + 1 and torch.equal(eng.save_state(), before)
  eng.load_envs(states)
  launches = eng.launch_count()
  live = _eval_task(eng)
  assert eng.launch_count() == launches + 1
  eng.close()
  return got, live


# -- 1, 2: records of every step-sweep case -----------------------------------------------------

@gpu
@pytest.mark.parametrize('case', sweep.CASES, ids=[c['name'] for c in sweep.CASES])
def test_saved_records_evaluate_as_the_oracle(case):
  from spriteworld_b200 import constants, engine
  eng, states, (arrs, nodes, action, _) = _saved(case)
  launches = eng.launch_count()
  got = _host(eng.evaluate(states))
  assert eng.launch_count() == launches + 1
  host = states.to_host()
  ids = engine.shape_id_table(constants.SHAPES)
  pick = _pick(case, host['pos_x'], host['pos_y'], ids[host['shape']], host['reset_next'])
  assert (host['reset_next'][pick] == 1).any() or case['mel'] > case['T'], case['name']
  want = _oracle_values(_cfg(case, action, nodes), _sprites(host, pick, ids))
  _assert_same(tuple(a[pick] for a in got), want, case['name'])
  eng.close()


@gpu
@pytest.mark.parametrize('case', sweep.CASES, ids=[c['name'] for c in sweep.CASES])
def test_saved_records_evaluate_as_the_envs_they_load_into(case):
  eng, states, (_, nodes, action, _) = _saved(case)
  eng.close()
  got, live = _two_paths(case, action, nodes, states)
  _assert_same(got, live, case['name'])


# -- 3: Clustering against scikit-learn ---------------------------------------------------------

@gpu
def test_clustering_records_evaluate_as_scikit_learn():
  """Rewards of the Clustering layouts are scikit-learn's 1 / davies_bouldin_score, errors its
  exceptions; layouts of float32 positions give the float64 metric, not a float32-rounded one."""
  from spriteworld_b200 import constants, engine, scene
  cm = fixtures.ClusteringMetric()
  arrs = cm.scenes()
  nodes = [cm.node()]
  action = dict(kind='select_move', scale=1.0, motion_cost=0.0)
  eng = engine.Engine(cm.L, 32, 1, action, nodes, constants.SHAPES)
  b = scene.batch_from_factor_arrays(
      arrs['x'], arrs['y'], arrs['pos_f32'], arrs['shape'], arrs['angle'], arrs['scale'],
      arrs['c0'], arrs['c1'], arrs['c2'], arrs['vx'], arrs['vy'], arrs['member'], arrs['rgb'])
  eng.upload_scenes(b, np.arange(cm.L), np.zeros(cm.L, int))
  eng.upload_state(pos_x=b['x'], pos_y=b['y'], cursor=np.zeros(cm.L), step_count=np.zeros(cm.L),
                   reset_next=np.zeros(cm.L))
  states = eng.save_envs()
  reward, success, status = got = _host(eng.evaluate(states))
  eng.close()
  ok = cm.err == 0
  assert np.array_equal(status, cm.err)
  assert np.array_equal(_bits(reward[ok]), _bits(cm.metric[ok]))
  assert np.isnan(reward[~ok]).all() and ok.sum() > 1000 and (~ok).sum() > 10
  # the layouts whose positions are all float32, and among them metrics float32 cannot hold
  occ = arrs['shape'] > 0
  all_f32 = ((arrs['pos_f32'] > 0) | ~occ).all(1)
  mixed = ((arrs['pos_f32'] > 0) & occ).any(1) & ~all_f32
  rounds = cm.metric.astype(np.float32).astype(np.float64) != cm.metric
  assert (ok & all_f32 & rounds).sum() > 100 and (ok & mixed).sum() > 100 and (ok & ~all_f32 & ~mixed).sum() > 100
  host = states.to_host()
  want = _oracle_values(_cfg(dict(keep=True, mel=10), action, nodes),
                        _sprites(host, np.arange(cm.L), engine.shape_id_table(constants.SHAPES)))
  _assert_same(got, want, 'clustering_metric')
  assert (success[ok] == 1).all()


# -- 4: goals -----------------------------------------------------------------------------------

def _goal_tree_nodes(tree):
  """The task tree of GOAL_TREES entry `tree`: its case's tree with goal slots on the named nodes."""
  _, name, slots = tree
  case = _named(name)
  _, nodes, action, _ = sweep._setup(case)
  assert all(nodes[i]['kind'] == 'find_goal' for i in slots)
  return case, action, [dict(nd, goal_slot=slots[i]) if i in slots else nd for i, nd in enumerate(nodes)]


def _override_goals(n, G, rng):
  """Goals (n, G, 2) with a different value in every slot, many outside [0, 1], and -0.0 and 0.0."""
  g = rng.uniform(-0.75, 1.75, (n, G, 2))
  g[::4, 0, 0] = -0.0
  g[1::4, -1, 1] = -0.0
  g[2::4, G // 2, 0] = 0.0
  return g


@gpu
@pytest.mark.parametrize('tree', GOAL_TREES, ids=[t[0] for t in GOAL_TREES])
def test_goals_of_records_and_overriding_goals_evaluate_as_the_constant_goal_tree(tree):
  import torch
  from spriteworld_b200 import constants, engine
  case, action, nodes = _goal_tree_nodes(tree)
  G = len(tree[2])
  eng, states, _ = _saved(case)
  eng.close()
  rng = np.random.RandomState(_seed(case, 3) + G)
  n = len(states)
  # the goal-free records with goals appended, as a G-goal engine saves them
  fields, rb = engine.record_layout(case['S'], G)
  off = {f[0]: f[1] for f in fields}
  slots_end = off['pos_f32'] + case['S']
  own = rng.uniform(0, 1, (n, G, 2))
  data = np.zeros((n, rb), np.uint8)
  data[:, :slots_end] = states.data.cpu().numpy()[:, :slots_end]
  data[:, off['goal']:off['goal'] + 16 * G] = own.reshape(n, 2 * G).view(np.uint8)
  recs = engine.EnvStates(torch.from_numpy(data).to(states.data.device), states.span_class, b'', case['S'], G)
  got, live = _two_paths(case, action, nodes, recs)
  _assert_same(got, live, (tree[0], 'own goals, live'))
  assert np.array_equal(recs.to_host()['goal'], own)
  over = _override_goals(n, G, rng)
  got_over, _ = _two_paths(case, action, nodes, recs, goals=over)
  host = recs.to_host()
  pick = np.sort(rng.choice(n, min(n, 400), replace=False))
  sprites = _sprites(host, pick, engine.shape_id_table(constants.SHAPES))
  for goals, values, what in ((own, got, 'own goals'), (over, got_over, 'overriding goals')):
    cfgs = [_cfg(case, action, _constant_goals(nodes, goals[i])) for i in pick]
    _assert_same(tuple(a[pick] for a in values), _oracle_values(cfgs, sprites), (tree[0], what))
  # the goals decide the values
  assert not np.array_equal(_bits(got[0]), _bits(got_over[0]))


# -- 5: record shapes and edges -----------------------------------------------------------------

def _edit_shapes(host, rng):
  """Shape bytes (n, S) with 13, 255 and LACKING's id in some occupied slots and a pentagon in some
  empty ones."""
  from spriteworld_b200 import engine
  shape = host['shape'].copy()
  occ, u = shape > 0, rng.rand(*shape.shape)
  shape[occ & (u < 0.15)] = 13
  shape[occ & (u >= 0.15) & (u < 0.3)] = 255
  shape[occ & (u >= 0.3) & (u < 0.45)] = engine.SHAPE_IDS[LACKING]
  shape[~occ & (u < 0.3)] = engine.SHAPE_IDS['pentagon']
  return shape


@gpu
@pytest.mark.parametrize('edit', EDITS, ids=[e[0] for e in EDITS])
def test_edited_shape_bytes_evaluate_as_a_load_sanitises_them(edit):
  import torch
  from spriteworld_b200 import constants, engine
  from tests.test_expand_on_oracle import _set_field
  name, tree = edit
  case = _named(name)
  eng, states, (_, nodes, action, _) = _saved(case)
  eng.close()
  nodes = nodes if tree is None else tree
  host = states.to_host()
  rng = np.random.RandomState(_seed(case, 4))
  shape = _edit_shapes(host, rng)
  data = states.data.cpu().numpy().copy()
  _set_field(data, case['S'], 'shape', shape)
  edited = engine.EnvStates(torch.from_numpy(data).to(states.data.device), states.span_class, b'', case['S'])
  host = edited.to_host()
  pick = np.sort(rng.choice(len(states), min(len(states), 600), replace=False))
  cfg = _cfg(case, action, nodes)
  for label, shapes in (('all shapes', constants.SHAPES), ('no ' + LACKING, _lacking_shapes())):
    got, live = _two_paths(case, action, nodes, edited, shapes=shapes)
    _assert_same(got, live, (name, label, 'live'))
    want = _oracle_values(cfg, _sprites(host, pick, engine.shape_id_table(shapes)))
    _assert_same(tuple(a[pick] for a in got), want, (name, label))


@gpu
def test_permuted_repeated_and_counted_records_and_guarded_outputs():
  import torch
  from spriteworld_b200 import constants, engine
  from tests import test_gpu_render_geometry as geo
  case = _named('clustering_f32')
  eng, states, (_, nodes, action, _) = _saved(case)
  dev, N, S = eng.device, len(states), case['S']
  snapshot = eng.save_state()
  base = _host(eng.evaluate(states))
  # reversed, repeated past N, and indices outside [0, N): zero records, all slots empty
  i = np.arange(2 * N + 3)
  perm = np.concatenate([(N - 1 - i) % N, [-1, N, 10 ** 6]])
  got = _host(eng.evaluate(states.take(torch.from_numpy(perm).to(dev))))
  inside = perm[:-3]
  _assert_same(tuple(a[:-3] for a in got), tuple(a[inside] for a in base), 'permuted')
  zero = np.zeros((3, S), oracle.SPRITE_DTYPE)
  _assert_same(tuple(a[-3:] for a in got), _oracle_values(_cfg(case, action, nodes), zero), 'zero records')
  # counts around the four warps of a CTA, and a grid with a tail
  rng = np.random.RandomState(_seed(case, 5))
  for n in (0, 1, 3, 4, 5, 4097):
    idx = rng.randint(0, N, n)
    sub = states.take(torch.from_numpy(idx).to(dev))
    launches = eng.launch_count()
    out = _host(eng.evaluate(sub))
    assert eng.launch_count() == launches + (n > 0), n
    assert all(len(a) == n for a in out)
    _assert_same(out, tuple(a[idx] for a in base), ('count', n))
  # swb_evaluate_states into guarded buffers: reward 8 bytes past a 16-byte boundary, success and
  # status at odd addresses
  n = 4097
  sub = states.take(torch.from_numpy(rng.randint(0, N, n)).to(dev))
  want = _host(eng.evaluate(sub))
  rbig, rflat, rlo = geo._guarded(8 * n, dev, 8)
  sbig, sflat, slo = geo._guarded(n, dev, 1)
  ebig, eflat, elo = geo._guarded(n, dev, 3)
  launches = eng.launch_count()
  assert eng._lib.swb_evaluate_states(eng._h, sub.data.data_ptr(), n, sub.data.numel(), None, rflat.data_ptr(),
                                      sflat.data_ptr(), eflat.data_ptr(), eng._stream()) == 0
  assert eng.launch_count() == launches + 1
  torch.cuda.synchronize(dev)
  for big, lo, nb, what in ((rbig, rlo, 8 * n, 'reward'), (sbig, slo, n, 'success'), (ebig, elo, n, 'status')):
    geo._assert_guards(big, lo, nb, what)
  got = (rflat.cpu().numpy().copy().view(np.float64), sflat.cpu().numpy(), eflat.cpu().numpy())
  _assert_same(got, want, 'guarded')
  assert torch.equal(eng.save_state(), snapshot)
  eng.close()
  # the sample has what it is there for: NaN rewards, both success values, repeated records
  assert np.isnan(base[0]).any() and set(base[1].tolist()) == {0, 1}


# -- 6: rollout steps against their trajectory records ------------------------------------------

@gpu
@pytest.mark.parametrize('case', sweep.CASES, ids=[c['name'] for c in sweep.CASES])
def test_rollout_steps_evaluate_as_their_trajectory_records(case):
  """Without motion cost a live step's reward is the task value of the state it reaches -- with a
  float32 click on a Clustering root the float32 sum of DESIGN §5, float32(value) -- except where a
  non-finite action component makes the cost NaN."""
  import torch
  from spriteworld_b200 import _native
  case = dict(case, motion_cost=0.0)
  eng, states, (arrs, nodes, action, _) = _saved(case)
  rng = np.random.RandomState(_seed(case, 6))
  E, T, C = case['E'], 6, 3
  n = min(64, len(states))
  roots = np.sort(rng.choice(len(states), n, replace=False))
  acts = sweep.case_actions(case, arrs, rng, T * C)
  plans = np.ascontiguousarray(acts.reshape((T, C, E) + acts.shape[2:])[:, :, roots % E].swapaxes(1, 2))
  res = eng.rollout(torch.from_numpy(plans).to(eng.device), states=states[roots], trajectory=True)
  reward, success, status = _host(eng.evaluate(res.trajectory))
  step_type, got_r, got_s, got_e = (a.reshape(-1) for a in _host((res.step_type, res.reward, res.success,
                                                                    res.status)))
  ok = (step_type != _native.STEP_NONE) & ((got_e & _native.ENV_BAD_ACTION) == 0)
  finite = np.isfinite(plans).all(-1).reshape(-1) if plans.dtype != np.int32 else np.ones_like(ok)
  if case['dtype'] == 'f32' and nodes[-1]['kind'] == 'clustering':
    reward = reward.astype(np.float32).astype(np.float64)
  assert ok.sum() > 0 and (ok & finite).sum() > 0
  _assert_same((got_r[ok & finite], got_s[ok & finite], got_e[ok & finite]),
               (reward[ok & finite], success[ok & finite], status[ok & finite]), case['name'])
  assert np.array_equal(got_s[ok], success[ok]) and np.array_equal(got_e[ok], status[ok])
  eng.close()


# -- 7: the table covers what it should ---------------------------------------------------------

def test_case_table_covers_the_evaluate_paths():
  """Runs without a GPU: fails if the records compared with the oracle stop reaching a task kind, an
  aggregator, a success value, a task status, a record about to reset, a sanitised shape or a goal
  count."""
  from spriteworld_b200 import constants, engine
  success, statuses, nan_rewards, n_reset, far = {}, set(), 0, 0, set()
  for case in sweep.CASES:
    cfg, cur, rn = _oracle_saves(case)
    pick = _pick(case, cur['x'], cur['y'], cur['shape'], rn)
    assert len(pick) <= 1.1 * MAX_PICK, case['name']
    n_reset += int((rn[pick] == 1).sum())
    if _far(cur['x'][pick], cur['y'][pick], cur['shape'][pick]).any():
      far.add(case['name'])
    kind = sweep.case_nodes(case, np.random.RandomState(0))[-1]['kind']
    r, s, e = _oracle_values(cfg, cur[pick])
    success.setdefault(kind, set()).update(s.tolist())
    statuses.update(e.tolist())
    nan_rewards += int(np.isnan(r).sum())
  assert success == {k: {0, 1} for k in ('find_goal', 'clustering', 'meta')}, success
  assert {0, oracle.ERR_CLUSTER_LABELS, oracle.ERR_CLUSTER_ZERODIV} <= statuses and nan_rewards > 0
  assert n_reset > 100
  assert {c['name'] for c in sweep.CASES if c['actions'] in ('wide', 'nonfinite') or c['edge_pos']} <= far, far
  # every aggregator under both criteria, in the step sweep's trees and in a goal tree
  metas = [nd for c in sweep.CASES for nd in sweep.case_nodes(c, np.random.RandomState(0)) if nd['kind'] == 'meta']
  assert {(nd['aggregator'], nd['criterion']) for nd in metas} >= {
      (a, k) for a in sweep.AGGS for k in ('all', 'any')}
  # NoReward, sanitised shapes: 13, 255 and an id the engine lacks, on both shape tables
  assert any(tree == [dict(kind='no_reward')] for _, tree in EDITS)
  assert any(name.startswith('clustering') for name, _ in EDITS)
  full, lacking = engine.shape_id_table(constants.SHAPES), engine.shape_id_table(_lacking_shapes())
  lid = engine.SHAPE_IDS[LACKING]
  assert full[lid] == lid and lacking[lid] == 0 and full[13] == full[255] == 0
  shape = _edit_shapes(dict(shape=np.tile([0, 1, 2, 3, 4, 5, 6, 7], (64, 4)).astype(np.uint8)),
                       np.random.RandomState(0))
  assert {13, 255, lid, engine.SHAPE_IDS['pentagon']} <= set(np.unique(shape).tolist())
  # G = 0 (every case) and G = 1 and G > 1, with goal slots out of node order
  goal_counts = set()
  for tree in GOAL_TREES:
    slots = sorted(tree[2].values())
    assert slots == list(range(len(slots))) and list(tree[2].values()) != slots or len(slots) == 1
    case = _named(tree[1])
    nodes = sweep.case_nodes(case, np.random.RandomState(0))
    assert all(nodes[i]['kind'] == 'find_goal' and nodes[i]['filter_slot'] != 20 for i in tree[2])
    assert nodes[-1]['kind'] == 'meta'
    goal_counts.add(len(slots))
  assert 1 in goal_counts and max(goal_counts) >= 2
  g = _override_goals(8, 3, np.random.RandomState(0))
  assert (np.signbit(g) & (g == 0)).any() and ((g < 0) | (g > 1)).any()
  assert all(len(np.unique(g[i])) == g[i].size for i in range(4, 8))
