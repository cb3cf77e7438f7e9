"""The committed frames of tests/golden/wide_aa/ are what tests/golden/make_golden_wide_aa.py
produces from the unmodified reference today (CPU tier; skipped where /root/reference does not
exist)."""
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
def test_make_golden_wide_aa_reproduces_the_committed_frames(tmp_path):
  env = dict(os.environ, SWB_GOLDEN_OUT=str(tmp_path))
  out = subprocess.run([sys.executable, os.path.join(GOLDEN, 'make_golden_wide_aa.py')], cwd=ROOT,
                       env=env, capture_output=True, text=True, timeout=900)
  assert out.returncode == 0, out.stderr[-2000:]
  have_dir = os.path.join(GOLDEN, 'wide_aa')
  names = sorted(os.listdir(have_dir))
  assert names == ['render_cases_wide_aa.npz'] and sorted(os.listdir(str(tmp_path))) == names
  have = np.load(os.path.join(have_dir, names[0]), allow_pickle=False)
  made = np.load(os.path.join(str(tmp_path), names[0]), allow_pickle=False)
  assert set(have.files) == set(made.files)
  for key in have.files:
    assert np.array_equal(have[key], made[key]), key
