"""swb_engine_create checks every field of its swb_config before its first CUDA call: a malformed
config is refused with the message of its own check, with or without a GPU, and no engine is
made.  Every config names a device that does not exist, so none of them can make an engine."""
import ctypes

import pytest

from spriteworld_b200 import _native

NO_DEVICE = 1 << 20


def _config():
  """2 envs x 3 slots, SelectMove, a Meta node over FindGoal (goal slot 0) and Clustering."""
  cfg = _native.Config()
  cfg.device = NO_DEVICE
  cfg.n_envs, cfg.n_slots, cfg.pool_depth = 2, 3, 2
  cfg.action_kind, cfg.action_scale, cfg.max_episode_length = _native.ACT_SELECT_MOVE, 1.0, 10
  cfg.n_nodes = 3
  goal, clusters, meta = cfg.nodes[0], cfg.nodes[1], cfg.nodes[2]
  goal.kind, goal.goal_slot = _native.TASK_FIND_GOAL, 0
  clusters.kind, clusters.n_clusters = _native.TASK_CLUSTERING, 2
  meta.kind, meta.n_children = _native.TASK_META, 2
  meta.children[0], meta.children[1] = 0, 1
  cfg.shape_n_verts[1] = 3
  return cfg


def _fields(part, **fields):
  """Sets `fields` of part(cfg): the config or one of its nodes."""
  def mutate(cfg):
    for name, value in fields.items():
      setattr(part(cfg), name, value)
  return mutate


def _item(array, j, value):
  """Sets element j of the array array(cfg)."""
  def mutate(cfg):
    array(cfg)[j] = value
  return mutate


CFG = lambda c: c
GOAL, CLUSTERS, META = (lambda c: c.nodes[0]), (lambda c: c.nodes[1]), (lambda c: c.nodes[2])

CASES = {
    'n_envs': (_fields(CFG, n_envs=0), 'n_envs must be >= 1'),
    'n_slots': (_fields(CFG, n_slots=33), 'n_slots must be in [1, 32], got 33'),
    'pool_depth': (_fields(CFG, pool_depth=0), 'pool_depth must be >= 1'),
    'n_nodes': (_fields(CFG, n_nodes=0), 'bad n_nodes 0'),
    'n_nodes_over': (_fields(CFG, n_nodes=33), 'bad n_nodes 33'),
    'n_children': (_fields(META, n_children=17), 'bad n_children'),
    'tree_order': (_item(lambda c: c.nodes[2].children, 1, 2), 'task tree is not post-order'),
    'n_clusters': (_fields(CLUSTERS, n_clusters=0), 'bad n_clusters'),
    'filter_slot': (_fields(GOAL, filter_slot=32), 'bad filter_slot'),
    'goal_slot': (_fields(GOAL, goal_slot=8), 'node 0: goal_slot 8 outside [-1, 8) (SWB_MAX_GOALS)'),
    'goal_slot_twice': (_fields(CLUSTERS, kind=_native.TASK_FIND_GOAL, goal_slot=0),
                        'goal_slot 0 belongs to nodes 0 and 1'),
    'goal_slot_missing': (_fields(GOAL, goal_slot=1), 'goal slots must be 0 .. 1, slot 0 has no node'),
    'task_kind': (_fields(CLUSTERS, kind=7), 'unknown task kind 7'),
    'action_kind': (_fields(CFG, action_kind=3), 'bad action_kind'),
    'shape_verts': (_item(lambda c: c.shape_n_verts, 5, _native.MAX_VERTS + 1), 'shape 5 has 33 vertices (max 32)'),
    'shape_verts_negative': (_item(lambda c: c.shape_n_verts, 12, -1), 'shape 12 has -1 vertices (max 32)'),
}


def _create(cfg):
  L = _native.load()
  h = ctypes.c_void_p()
  rc = L.swb_engine_create(ctypes.byref(cfg), ctypes.byref(h))
  return rc, L.swb_last_error().decode(), h.value


def test_the_base_config_passes_every_check():
  rc, msg, h = _create(_config())
  assert rc != 0 and h is None
  assert 'device' in msg.lower(), msg


@pytest.mark.parametrize('case', sorted(CASES))
def test_a_malformed_config_is_refused_with_its_own_message(case):
  mutate, want = CASES[case]
  cfg = _config()
  mutate(cfg)
  rc, msg, h = _create(cfg)
  assert rc != 0 and h is None
  assert msg == want
