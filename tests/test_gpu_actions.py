"""The click action path on the device against the reference's recorded steps
(tests/golden/actions/actions.npz, made by make_golden_actions.py), bit for bit.

  * every single step of the fixture through Engine.step (mode 0: NoReward task, velocities
    zero), Engine.step_host, and the action-only launch (mode 2) behind the drop-in
    action_space.step: costs, rewards, positions, step types and statuses;
  * the drop-in Environment replaying the recorded episodes, the noisy one included, with the
    actions the reference applied after its noise: positions, step types and frames against the
    fixture, rewards against the oracle in the engine's sqrt distance mode (which equals the
    reference's pow mode bit for bit on these episodes except where pow(x, .5) is not sqrt(x);
    tests/test_oracle_actions.py pins the pow mode to the reference);
  * BatchedEnvironment with SelectMove(noise_scale=0.05, motion_cost=0.7) against the oracle fed
    the same noise from an identically seeded generator.

Nothing here reads the reference or np.random's global stream.
"""
import ctypes
import types

import numpy as np
import pytest

from oracle import oracle
from tests import fixtures
from tests.test_oracle_actions import ActionCases, same_bits

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def cases():
  return ActionCases()


def _groups(cases):
  """Single steps grouped by engine configuration: (kind, scale, motion_cost, keep) -> ids."""
  ss = cases.ss
  out = {}
  for i in range(cases.n):
    key = (int(ss['kind'][i]), float(ss['scale'][i]), float(ss['motion_cost'][i]),
           bool(ss['keep'][i]))
    out.setdefault(key, []).append(i)
  return out


def _engine_for(cases, key, ids):
  from spriteworld_b200 import engine, scene
  kind, scale, cost, keep = key
  action = dict(kind=('select_move', 'drag_and_drop')[kind], scale=scale, motion_cost=cost)
  E, S = len(ids), cases.meta['n_slots']
  eng = engine.Engine(E, S, 1, action, [dict(kind='no_reward')], cases.shapes,
                      keep_in_frame=keep, max_episode_length=1000)
  ss = cases.ss
  z = np.zeros((E, S))
  before = ss['before'][ids]
  b = scene.batch_from_factor_arrays(
      before[..., 0], before[..., 1], ss['pos_f32'][ids], ss['shape'][ids], ss['angle'][ids],
      ss['sprite_scale'][ids], z, z, z, z, z, np.zeros((E, S), np.uint32),
      np.zeros((E, S, 3), np.uint8))
  eng.upload_scenes(b, np.arange(E), np.zeros(E, int))
  return eng, b


def test_single_steps_through_engine_step_and_step_host(cases):
  import torch
  from spriteworld_b200 import _native
  checked = 0
  for key, ids in _groups(cases).items():
    ids = np.array(ids)
    eng, b = _engine_for(cases, key, ids)
    for f32 in (True, False):
      sel = ids[cases.ss['f32'][ids] == int(f32)]
      rows = np.nonzero(cases.ss['f32'][ids] == int(f32))[0]
      acts = np.zeros((len(ids), 4), np.float32 if f32 else np.float64)
      acts[rows] = cases.ss['action'][sel]
      want = [cases.expected_env_step(i) for i in sel]
      for path in ('device', 'host', 'apply'):
        eng.upload_state(pos_x=b['x'], pos_y=b['y'], cursor=np.zeros(len(ids)),
                         step_count=np.zeros(len(ids)), reset_next=np.zeros(len(ids)))
        if path == 'host':
          reward, step_type, _, status, _ = eng.step_host(acts)
        elif path == 'device':
          res = eng.step(torch.from_numpy(acts).to(eng.device))
          reward, step_type, status = (a.cpu().numpy() for a in (res.reward, res.step_type,
                                                                 res.status))
        else:
          t = torch.from_numpy(acts).to(eng.device)
          _native.check(eng._lib.swb_apply_action(
              eng._h, ctypes.c_void_p(t.data_ptr()),
              _native.DTYPE_F32 if f32 else _native.DTYPE_F64, eng._out, eng._stream()))
          reward, step_type, status = (a.cpu().numpy() for a in (eng._reward, eng._step_type,
                                                                 eng._status))
        st = eng.download_state()
        pos = np.stack([st['pos_x'], st['pos_y']], -1)[rows]
        where = (key, f32, path)
        assert (status[rows] == 0).all(), where
        if path == 'apply':
          bad = ~same_bits(reward[rows], cases.ss['cost'][sel])
          assert not bad.any(), (where, sel[bad][:5].tolist())
          bad = ~same_bits(pos, cases.ss['after'][sel]).all((1, 2))
          assert not bad.any(), (where, sel[bad][:5].tolist())
        else:
          bad = ~same_bits(reward[rows], np.array([w[1] for w in want]))
          assert not bad.any(), (where, sel[bad][:5].tolist())
          assert np.array_equal(step_type[rows], [w[2] for w in want]), where
          bad = ~same_bits(pos, np.array([w[0] for w in want])).all((1, 2))
          assert not bad.any(), (where, sel[bad][:5].tolist())
        checked += len(sel)
    eng.close()
  assert checked == 3 * cases.n


def test_single_steps_through_the_drop_in_action_space(cases):
  """action_space.step on Python sprite lists (the mode 2 launch of _direct.action_step)."""
  from spriteworld_b200 import action_spaces, sprite
  ss = cases.ss
  for i in range(0, cases.n, 3):
    sprites = []
    for k in range(cases.meta['n_slots']):
      x, y = ss['before'][i, k]
      if ss['pos_f32'][i, k]:
        x, y = np.float32(x), np.float32(y)
      sprites.append(sprite.Sprite(x=x, y=y, shape=fixtures.SHAPE_NAMES[ss['shape'][i, k] - 1],
                                   angle=ss['angle'][i, k], scale=ss['sprite_scale'][i, k]))
    space = (action_spaces.SelectMove, action_spaces.DragAndDrop)[ss['kind'][i]](
        scale=float(ss['scale'][i]), motion_cost=float(ss['motion_cost'][i]))
    with np.errstate(all='ignore'):
      cost = space.step(cases.action(i), sprites, bool(ss['keep'][i]))
    assert isinstance(cost, np.float32) == bool(ss['f32'][i]), i
    assert same_bits(cost, ss['cost'][i]), (i, float(cost), float(ss['cost'][i]))
    got = np.array([[float(s.position[0]), float(s.position[1])] for s in sprites])
    assert same_bits(got, ss['after'][i]).all(), i


def _project_modules():
  from spriteworld_b200 import (action_spaces, factor_distributions, renderers,
                                sprite_generators, tasks)
  return types.SimpleNamespace(action_spaces=action_spaces, tasks=tasks,
                               factor_distributions=factor_distributions,
                               sprite_generators=sprite_generators, renderers=renderers)


def _action_configs():
  import importlib.util
  import os
  path = os.path.join(fixtures.GOLDEN, 'action_configs.py')
  spec = importlib.util.spec_from_file_location('swb_action_configs', path)
  mod = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(mod)
  return mod


def _replay_scenes(scenes, e):
  """init_sprites that returns env e's recorded scenes in order, as the reference drew them."""
  from spriteworld_b200 import sprite
  k = [0]

  def gen():
    out = []
    for s in range(scenes['shape'].shape[2]):
      if not scenes['shape'][e, k[0], s]:
        continue
      f = {name: scenes[name][e, k[0], s] for name in fixtures.FIELDS}
      pos = (np.float32 if f['pos_f32'] else float)
      col = (np.float32 if f['color_f32'] else float)
      out.append(sprite.Sprite(
          x=pos(f['x']), y=pos(f['y']), shape=fixtures.SHAPE_NAMES[f['shape'] - 1],
          angle=float(f['angle']), scale=float(f['scale']), c0=col(f['c0']), c1=col(f['c1']),
          c2=col(f['c2']), x_vel=float(f['vx']), y_vel=float(f['vy'])))
    k[0] += 1
    return out
  return gen


@pytest.mark.parametrize('c', range(4))
def test_dropin_environment_replays_reference_episode(cases, c):
  from spriteworld_b200 import environment
  ep = cases.episode(c)
  meta = ep['meta']
  make = dict(_action_configs().episode_configs(_project_modules(), noise_scale=None))[meta['name']]
  T, E = ep['reward'].shape
  bo = oracle.BatchOracle(oracle.with_device_sqrt(fixtures.env_cfg_from_meta(meta)),
                          oracle.shape_table(cases.shapes), None,
                          fixtures.records_from_arrays(ep['scenes']))
  want_reward = [bo.step(ep['applied'][t]).reward.copy() for t in range(T)]
  envs = []
  for e in range(E):
    cfg = make()
    cfg['init_sprites'] = _replay_scenes(ep['scenes'], e)
    envs.append(environment.Environment(**cfg))
  frames = {(int(t), int(e)): f for (t, e), f in zip(ep['frame_at'], ep['frames'])}
  S = meta['n_slots']
  for t in range(T):
    for e, env in enumerate(envs):
      a = ep['applied'][t, e]
      with np.errstate(all='ignore'):
        ts = env.step(ep['actions'][t, e] if np.isnan(a).all() else a)
      where = (meta['name'], t, e)
      assert int(ts.step_type) == ep['step_type'][t, e], where
      if not ts.first():
        assert same_bits(ts.reward, want_reward[t][e]), (where, ts.reward, want_reward[t][e])
      n = len(env.state()['sprites'])
      got = np.array([[float(s.x), float(s.y)] for s in env.state()['sprites']])
      assert same_bits(got, ep['pos'][t, e, S - n:]).all(), where
      assert bool(env.success()) == bool(ep['success'][t, e]), where
      if (t, e) in frames:
        assert np.array_equal(ts.observation['image'], frames[(t, e)]), where
  for env in envs:
    env.close()


def test_batched_environment_action_noise_matches_oracle():
  """SelectMove(noise_scale=0.05, motion_cost=0.7, scale=3) with keep_in_frame off: the oracle
  is fed float32 actions plus the noise of a generator in the state the environment's is in."""
  from spriteworld_b200 import action_spaces, constants, environment, scene, sprite_generators
  from spriteworld_b200.configs.cobra import goal_finding_more_targets as cfgmod
  E, K, T = 64, 6, 3
  cfg = cfgmod.get_config('train')
  cfg['action_space'] = action_spaces.SelectMove(scale=3.0, noise_scale=0.05, motion_cost=0.7)
  cfg['keep_in_frame'] = False
  env = environment.BatchedEnvironment(n_envs=E, pool_depth=K, rng=np.random.RandomState(3),
                                       **cfg)
  eng = env.engine
  S = eng.n_slots
  pool = np.zeros((E, K, S), oracle.SPRITE_DTYPE)

  def record(batch, env_ids, ring_slots):
    for f in ('x', 'y', 'm00', 'm01', 'm10', 'm11', 'vx', 'vy', 'member', 'shape', 'pos_f32',
              'rgb'):
      pool[f][np.asarray(env_ids), np.asarray(ring_slots)] = batch[f]

  orig_upload = eng.upload_scenes

  def upload(batch, env_ids, ring_slots):
    record(batch, env_ids, ring_slots)
    return orig_upload(batch, env_ids, ring_slots)

  eng.upload_scenes = upload
  twin = np.random.RandomState(3)
  first = sprite_generators.batch_of(cfg['init_sprites'], E * K, twin)
  nodes, filters = cfg['task'].compile()
  record(scene.arrays_from_layout(first, S, filters, cfg['renderers']['image'].color_to_rgb),
         np.repeat(np.arange(E), K), np.tile(np.arange(K), E))
  twin.set_state(env._rng.get_state())
  meta = dict(action=cfg['action_space'].compile(), keep_in_frame=False,
              max_episode_length=cfg['max_episode_length'], nodes=nodes)
  bo = oracle.BatchOracle(oracle.with_device_sqrt(fixtures.env_cfg_from_meta(meta)),
                          oracle.shape_table(constants.SHAPES), oracle.raster_cfg(64, 64, 5), pool)
  bo.pool = pool
  env.reset()
  bo.step(np.zeros((E, 4)))
  twin.normal(size=(E, 4))                   # reset() stepped once with a dummy action
  rng = np.random.RandomState(11)
  n_cost = 0
  for t in range(T):
    a = rng.uniform(0, 1, (E, 4)).astype(np.float32)
    ts = env.step(a)
    pre = a + twin.normal(loc=0.0, scale=0.05, size=(E, 4))
    bo.step(pre)
    assert np.array_equal(ts.step_type.cpu().numpy(), bo.step_type), t
    assert same_bits(ts.reward.cpu().numpy(), bo.reward).all(), t
    assert np.array_equal(ts.observation['image'].cpu().numpy(), bo.frames), t
    st = eng.download_state()
    occ = bo.cur['shape'] > 0
    assert same_bits(st['pos_x'][occ], bo.cur['x'][occ]).all(), t
    n_cost += int((bo.step_type == oracle.STEP_MID).sum())
  assert n_cost > E
  env.close()
