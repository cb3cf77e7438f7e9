"""The committed fixtures are what tests/golden/make_golden.py produces from the unmodified
reference today (CPU tier; skipped where /root/reference does not exist)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
REFERENCE = os.environ.get('SPRITEWORLD_REFERENCE', '/root/reference')


@pytest.mark.skipif(not os.path.isdir(os.path.join(REFERENCE, 'spriteworld')),
                    reason='reference not present')
def test_make_golden_reproduces_the_committed_fixtures(tmp_path):
  env = dict(os.environ, SWB_GOLDEN_OUT=str(tmp_path))
  out = subprocess.run([sys.executable, os.path.join(GOLDEN, 'make_golden.py')], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=900)
  assert out.returncode == 0, out.stderr[-2000:]
  names = sorted(f for f in os.listdir(GOLDEN) if f.endswith(('.npz', '.json')))
  assert names == sorted(f for f in os.listdir(str(tmp_path)) if f.endswith(('.npz', '.json')))
  for name in [n for n in names if n.endswith('.json')]:
    with open(os.path.join(GOLDEN, name)) as f_have, open(os.path.join(str(tmp_path), name)) as f_made:
      assert json.load(f_have) == json.load(f_made), name
  for name in [n for n in names if n.endswith('.npz')]:
    have = np.load(os.path.join(GOLDEN, name), allow_pickle=True)
    made = np.load(os.path.join(str(tmp_path), name), allow_pickle=True)
    assert set(have.files) == set(made.files), name
    for key in have.files:
      assert np.array_equal(have[key], made[key]), (name, key)
