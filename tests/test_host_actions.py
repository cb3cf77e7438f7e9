"""CPU tier: how host actions become what the engine accepts (engine.host_actions), through every
host entry point, on the oracle-backed engine double (tests/oracle_engine.py).

An Embodied direction is valid only if it equals an integer in 0..3; anything else is the
reference's KeyError (action_spaces.py:203) and must never be wrapped or truncated into a valid
direction on its way to the device.  A carry is truthy as in the reference's `if carry:`.
"""
import numpy as np
import pytest

from tests import oracle_engine

BAD_DIRECTIONS = [2 ** 32 + 1, 1.5, -1, 4, float('nan')]


@pytest.fixture(autouse=True)
def _oracle_engine(monkeypatch):
  oracle_engine.install(monkeypatch)


def _body_over_sprite():
  """The body (last) sits on a square: a carry moves both (tests/action_spaces_test.py)."""
  from spriteworld_b200 import sprite
  return [sprite.Sprite(x=p[0], y=p[1], shape='square', scale=0.15)
          for p in ([0.5, 0.5], [0.45, 0.55])]


def _positions(sprites):
  return [np.array(s.position) for s in sprites]


def test_host_actions_conversion():
  from spriteworld_b200 import engine
  conv = lambda kind, a: engine.host_actions(kind, np.asarray(a))
  got = conv('embodied', [[0, 1.0], [2 ** 32, 2 ** 32 + 1], [0.5, 1.5], [-0.0, float('nan')],
                          [True, 3], [0, -1], [7, 4]])
  assert got.dtype == np.int32 and got.flags.c_contiguous
  assert got.tolist() == [[0, 1], [1, -1], [1, -1], [0, -1], [1, 3], [0, -1], [1, -1]]
  assert conv('embodied', np.array([[2 ** 33, 2]], np.uint64)).tolist() == [[1, 2]]
  for kind in ('select_move', 'drag_and_drop'):
    assert conv(kind, np.zeros((2, 4), np.float32)).dtype == np.float32
    for dtype in (np.float16, np.int32, np.int64, np.float64):
      assert conv(kind, np.ones((2, 4), dtype)).dtype == np.float64
  with pytest.raises(ValueError):
    conv('embodied', np.zeros((2, 4)))
  for kind in engine.ACTIONS:
    zero = engine.zero_actions(kind, 3)
    assert not zero.any()
    spec = engine.ACTIONS[kind]
    assert engine.action_dtype(spec.kind, 3, zero) == spec.dtypes[zero.dtype.name]


@pytest.mark.parametrize('direction', BAD_DIRECTIONS)
def test_embodied_step_refuses_bad_directions(direction):
  from spriteworld_b200 import _direct, action_spaces
  space = action_spaces.Embodied(step_size=0.1)
  sprites = _body_over_sprite()
  before = _positions(sprites)
  with pytest.raises(KeyError):
    space.step((0, direction), sprites, keep_in_frame=True)
  # past the host check as well: the step reports the env's bad action, nothing moves
  with pytest.raises(KeyError):
    _direct.action_step(space, np.array([1, direction]), sprites, True)
  assert all(np.array_equal(a, b) for a, b in zip(before, _positions(sprites)))


@pytest.mark.parametrize('carry', [2 ** 32, 0.5, -1, True])
def test_embodied_truthy_carry_carries(carry):
  from spriteworld_b200 import _direct, action_spaces
  space = action_spaces.Embodied(step_size=0.1)
  for step in (space.step, lambda a, s, k: _direct.action_step(space, np.array(a), s, k)):
    sprites = _body_over_sprite()
    step((carry, 3), sprites, True)
    assert np.allclose([s.position for s in sprites], [[0.6, 0.5], [0.55, 0.55]], atol=1e-12)


@pytest.mark.parametrize('dtype', [np.int64, np.float64])
def test_batched_embodied_bad_directions_set_bad_action(dtype):
  from spriteworld_b200 import _native, environment
  from spriteworld_b200.configs.examples import goal_finding_embodied
  E = 8
  env = environment.BatchedEnvironment(n_envs=E, pool_depth=4, rng=np.random.RandomState(2),
                                       **goal_finding_embodied.get_config())
  env.reset()
  actions = np.zeros((E, 2), dtype)
  actions[:, 0] = [0, 2 ** 32, 0, 1, 0, 0.5 if dtype == np.float64 else 3, 0, 1]
  actions[:, 1] = [0, 1, 2, 3, 0, 1, 2, 3]
  bad = np.array([1, 4, 6]) if dtype == np.int64 else np.array([2, 5, 7])
  actions[bad, 1] = 2 ** 32 + 1 if dtype == np.int64 else [1.5, 2.5, 0.25]
  before = env.engine.download_state()
  ts = env.step(actions)
  after = env.engine.download_state()
  status = ts.status.numpy()
  flagged = np.flatnonzero(status & _native.ENV_BAD_ACTION)
  assert flagged.tolist() == bad.tolist(), status
  good = np.setdiff1d(np.arange(E), bad)
  for k in ('pos_x', 'pos_y'):
    assert np.array_equal(after[k][bad], before[k][bad])
  moved = (after['pos_x'] != before['pos_x']) | (after['pos_y'] != before['pos_y'])
  assert moved[good].any(axis=1).all()        # every valid direction moved the body
  env.close()
