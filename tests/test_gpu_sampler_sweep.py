"""The device scene sampler on the GPU over the programs of tests/test_sampler_sweep.py: every
program op, factor dtype and colour path, against the CPU build of the same source and, on a
subset, against the NumPy restatement directly; the refill kernel through BatchedEnvironment; and
the failure record of a rejection loop that runs out of tries."""
import re

import numpy as np
import pytest

from spriteworld_b200 import constants, environment, scene_program, tasks
from spriteworld_b200 import engine as engine_lib
from spriteworld_b200 import factor_distributions as distribs
from spriteworld_b200 import sprite_generators as gen
from spriteworld_b200.configs.cobra import goal_finding_more_distractors
from spriteworld_b200.renderers import PILRenderer
from tests import test_sampler_sweep as sweep
from tests.test_gpu_device_sampler import _ring_check

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def engines():
  """One engine per slot count, reloaded with each program."""
  made = {}
  cfg = goal_finding_more_distractors.get_config('train')
  nodes, _ = cfg['task'].compile()

  def get(S):
    if S not in made:
      made[S] = engine_lib.Engine(4, S, 4, cfg['action_space'].compile(), nodes, constants.SHAPES)
    return made[S]

  yield get
  for eng in made.values():
    eng.close()


def _scenes():
  rng = np.random.RandomState(2)
  ids = np.concatenate([np.arange(256) % 19, rng.randint(0, 2 ** 62, 24), [2 ** 63 - 1, 2 ** 62, 0]])
  idx = np.concatenate([np.arange(256) // 19, rng.randint(0, 2 ** 62, 24), [2 ** 63 - 1, 2 ** 63 - 1, 2 ** 62]])
  return ids.astype(np.int64), idx.astype(np.int64)


def _numpy(out):
  return {k: v.cpu().numpy() for k, v in out.items()}


@pytest.mark.parametrize('name', sweep.CASE_NAMES)
def test_device_equals_cpu_build(name, engines):
  c = sweep.case(name)
  most = c.program.max_sprites
  ids, idx = _scenes()
  for S in sorted({1, max(1, most), 32} if most <= 1 else {most, 32}):
    eng = engines(S)
    for seed in sweep.SEEDS:
      eng.load_sampler(c.program, seed)
      got = _numpy(eng.sample_scenes(ids, idx))
      ref, fail = scene_program.sample_on_host(c.program, seed, ids, idx, S)
      if c.impossible:
        assert fail is not None
        with pytest.raises(ValueError, match='Maximum number of tried exceeded') as err:
          eng.check_sampler()
        # the same op as the CPU build, and a scene the CPU build fails too
        assert c.program.describe(fail[1]) in str(err.value)
        g, a = (int(v) for v in re.search(r'\(env (\d+), scene (\d+)\)$', str(err.value)).groups())
        assert scene_program.sample_on_host(c.program, seed, [g], [a], S)[1] is not None
      else:
        assert fail is None
        eng.check_sampler()
      sweep.assert_same(got, ref, '%s S=%d seed=%d' % (name, S, seed))


@pytest.mark.parametrize('name', list(dict.fromkeys(sweep.CASE_NAMES[::4] + [
    'hue_below_0_float32', 'value_past_int32_float32', 'rgb_float_1e19', 'uint64_above_2_63', 'impossible'])))
def test_device_equals_numpy_restatement(name, engines):
  c = sweep.case(name)
  S = max(1, c.program.max_sprites)
  ids, idx = sweep.scene_ids(64)
  eng = engines(S)
  eng.load_sampler(c.program, sweep.SEEDS[0])
  got = _numpy(eng.sample_scenes(ids, idx))
  _, (want, want_fail) = sweep.host_and_restatement(name, sweep.SEEDS[0])
  if c.impossible:
    assert want_fail is not None
    with pytest.raises(ValueError, match='Maximum number of tried exceeded'):
      eng.check_sampler()
    got = {k: v[:len(want['x'])] for k, v in got.items()}
  else:
    eng.check_sampler()
  sweep.assert_same(got, want, name)


def _uint64_rgb():
  C = distribs.Continuous
  body = distribs.Product([C('x', 0.1, 0.9), C('y', 0.1, 0.9), C('scale', 0.05, 0.2),
                           C('c0', 2 ** 63, 2 ** 64 - 4096, 'uint64'), C('c1', 0, 2 ** 64 - 4096, 'uint64'),
                           C('c2', -1e19, 1e19, 'float64')])
  return sweep.Case('uint64_rgb', gen.shuffle(gen.generate_sprites(body, gen.uniform_count(1, 6))),
                    [C('c0', 0.5, 1.5e19), C('c1', np.uint64(2 ** 63), 1e30), C('c2', 0, 1e19)])


REFILL = ['hue_below_0_float32', 'value_past_int32_float64', 'saturation_above_1_float32', 'p_or',
          'sample_generator_zero_p', 'angles', 'rejection_one_percent', 'zero_sprites', 'uint64_rgb']


@pytest.mark.parametrize('name', REFILL)
def test_refill_rings_equal_cpu_build(name):
  c = _uint64_rgb() if name == 'uint64_rgb' else sweep.case(name)
  task = (tasks.MetaAggregated([tasks.FindGoalPosition(f) for f in c.filters]) if c.filters
          else tasks.NoReward())
  cfg = goal_finding_more_distractors.get_config('train')
  env = environment.BatchedEnvironment(
      task=task, action_space=cfg['action_space'],
      renderers={'image': PILRenderer(image_size=(32, 32), color_to_rgb=c.cmap)},
      init_sprites=c.gen, max_episode_length=3, n_envs=32, pool_depth=4, sampler='device', seed=13,
      rng=np.random.RandomState(0))
  try:
    rng = np.random.RandomState(1)
    checked = 0
    for _ in range(24):
      res = env.step(rng.uniform(0, 1, (32, 4)).astype(np.float32))
      checked += _ring_check(env, res)
    assert checked > 32 * 24
    env.check_sampler()
  finally:
    env.close()
