"""The reference's own test files, run against spriteworld_b200 (CPU tier).

`spriteworld` is aliased to `spriteworld_b200`, so every `from spriteworld import ...` in the
reference's tests/ resolves to this package, unmodified.  The modules that only touch host code
(factor distributions, sprite generators, shapes, sprites, handcrafted renderers) run as they
are; the ones that call tasks, action spaces, the PIL renderer or whole environments need the
device, so here the engine is replaced by the oracle-backed double (tests/oracle_engine.py):
what is under test is this package's host layer -- task / action compilation, scene packing,
the plugin protocol, the config modules -- the device arithmetic has its own parity tests
(`-m gpu`).  The runs of the reference's test files are skipped where the reference is not
installed (SPRITEWORLD_REFERENCE).
"""
import importlib
import importlib.abc
import importlib.util
import os
import sys
import unittest

import pytest

REF_TESTS = os.path.join(os.environ.get('SPRITEWORLD_REFERENCE', '/root/reference'), 'tests')

needs_reference = pytest.mark.skipif(not os.path.isdir(REF_TESTS), reason='reference tests not present')


class _Alias(importlib.abc.MetaPathFinder, importlib.abc.Loader):
  """spriteworld[.x.y] -> spriteworld_b200[.x.y]"""

  def find_spec(self, name, path, target=None):
    if name == 'spriteworld' or name.startswith('spriteworld.'):
      return importlib.util.spec_from_loader(name, self)
    return None

  def create_module(self, spec):
    return importlib.import_module('spriteworld_b200' + spec.name[len('spriteworld'):])

  def exec_module(self, module):
    pass


def _third_party_stand_ins():
  """dm_env (with test_utils) and gym are absent from this image.  The reference's tests get
  them as views of what the package itself uses in their place: its dm_env surface
  (spriteworld_b200._dm_env), its minimal gym spaces, and a restatement of dm_env's
  EnvironmentTestMixin (oracle/refshim/standins/dm_env/test_utils.py)."""
  import types
  from oracle.refshim import loader
  from spriteworld_b200 import _dm_env, gym_wrapper
  mods = {}
  if importlib.util.find_spec('dm_env') is None:
    dm = types.ModuleType('dm_env')
    for name in ('Environment', 'TimeStep', 'StepType', 'restart', 'transition', 'termination'):
      setattr(dm, name, getattr(_dm_env, name))
    specs = types.ModuleType('dm_env.specs')
    for name in ('Array', 'BoundedArray', 'DiscreteArray'):
      setattr(specs, name, getattr(_dm_env.specs, name))
    spec = importlib.util.spec_from_file_location(
        'dm_env.test_utils', os.path.join(loader._STANDINS, 'dm_env', 'test_utils.py'))
    test_utils = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(test_utils)
    dm.specs, dm.test_utils = specs, test_utils
    mods.update({'dm_env': dm, 'dm_env.specs': specs, 'dm_env.test_utils': test_utils})
  if importlib.util.find_spec('gym') is None and importlib.util.find_spec('gymnasium') is None:
    gym = types.ModuleType('gym')
    spaces = types.ModuleType('gym.spaces')
    for name in ('Box', 'Discrete', 'Dict', 'Tuple'):
      setattr(spaces, name, getattr(gym_wrapper._MiniSpaces, name))
    gym.spaces = spaces
    mods.update({'gym': gym, 'gym.spaces': spaces})
  return mods


@pytest.fixture
def reference_alias():
  from oracle.refshim import loader
  loader._patch_aliases()   # np.cast / mock aliases the reference's tests rely on
  finder = _Alias()
  sys.meta_path.insert(0, finder)
  stand_ins = _third_party_stand_ins()
  sys.modules.update(stand_ins)
  yield
  sys.meta_path.remove(finder)
  for name in stand_ins:
    sys.modules.pop(name, None)
  for name in [n for n in sys.modules if n == 'spriteworld' or n.startswith('spriteworld.')]:
    del sys.modules[name]


def _run(rel):
  path = os.path.join(REF_TESTS, rel + '.py')
  spec = importlib.util.spec_from_file_location('reference_' + rel.replace('/', '_'), path)
  mod = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(mod)
  suite = unittest.defaultTestLoader.loadTestsFromModule(mod)
  result = unittest.TestResult()
  suite.run(result)
  problems = ['%s: %s' % (t.id(), tb.strip().splitlines()[-1]) for t, tb in
              result.failures + result.errors]
  return result.testsRun, problems


@needs_reference
@pytest.mark.parametrize('rel,n_tests', [
    ('factor_distributions_test', 39), ('sprite_generators_test', 7), ('shapes_test', 21),
    ('sprite_test', 16), ('renderers/handcrafted_test', 24)])
def test_reference_host_tests(reference_alias, rel, n_tests):
  ran, problems = _run(rel)
  assert not problems, '\n'.join(problems)
  assert ran == n_tests


@needs_reference
@pytest.mark.parametrize('rel,n_tests', [
    ('tasks_test', 85), ('action_spaces_test', 30), ('renderers/pil_renderer_test', 5),
    ('configs/configs_test', 8), ('environment_test', 7), ('gym_wrapper_test', 2)])
def test_reference_protocol_tests_on_oracle_engine(reference_alias, monkeypatch, rel, n_tests):
  from tests import oracle_engine
  oracle_engine.install(monkeypatch)
  ran, problems = _run(rel)
  assert not problems, '\n'.join(problems)
  assert ran == n_tests


def test_public_surface_of_the_reference_is_present():
  """Every public class, function, method and constructor parameter of the reference's modules
  on and around the path (as recorded from the reference in tests/golden/reference_surface.json
  by tests/golden/make_golden.py) exists under the same name in spriteworld_b200."""
  import inspect
  import json
  with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden',
                         'reference_surface.json')) as f:
    surface = json.load(f)
  missing = []
  for m, names in sorted(surface.items()):
    ours = importlib.import_module('spriteworld_b200.' + m)
    for name, entry in sorted(names.items()):
      if not hasattr(ours, name):
        missing.append('%s.%s' % (m, name))
        continue
      mine = getattr(ours, name)
      missing += ['%s.%s.%s' % (m, name, a) for a in entry.get('attrs', ()) if not hasattr(mine, a)]
      for key, fn in (('init', lambda: mine.__init__), ('params', lambda: mine)):
        if key in entry:
          have = [p for p in inspect.signature(fn()).parameters if p != 'self']
          if entry[key] != have[:len(entry[key])]:
            missing.append('%s.%s(%s)' % (m, name, ', '.join(entry[key])))
  assert not missing, missing
