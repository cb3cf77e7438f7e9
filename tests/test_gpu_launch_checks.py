"""A call the C-ABI refuses -- bad arguments, or a raster that cannot launch -- has enqueued
nothing: no kernel, no copy, no change to the engine's state or launch count
(include/spriteworld_b200.h).  Rasters that could never launch are refused when created."""
import ctypes

import numpy as np
import pytest

E = 4


def _engine(kind='select_move'):
  from spriteworld_b200 import constants, engine
  return engine.Engine(E, 2, 1, dict(kind=kind, scale=0.05), [dict(kind='no_reward')],
                       constants.SHAPES)


def _snapshot(eng):
  import torch
  torch.cuda.synchronize(eng.device)
  return eng.download_state(), eng.launch_count()


def _assert_unchanged(eng, before):
  state, launches = _snapshot(eng)
  assert launches == before[1]
  for k, v in before[0].items():
    assert np.array_equal(state[k], v), k


@pytest.mark.gpu
def test_raster_that_can_never_launch_is_refused_at_creation():
  from spriteworld_b200 import _native, engine
  eng = _engine()
  # 64 rows x 1365 columns x 3 bytes of staged band alone exceed the H100's 232,448 B opt-in
  with pytest.raises(_native.NativeError):
    engine.Raster(eng, 1365, 64, 3)
  engine.Raster(eng, 64, 64, 5).close()
  eng.close()


@pytest.mark.gpu
def test_raster_of_another_engine_enqueues_nothing():
  import torch
  from spriteworld_b200 import _native, engine
  a, b = _engine(), _engine()
  raster_b = engine.Raster(b, 16, 8, 2)
  acts = torch.full((E, 4), 0.75, device=a.device)
  frames = raster_b.new_frames()
  ptrs = (ctypes.c_void_p * 1)(frames.data_ptr())
  a.step(acts)                     # every env past its first reset: a step advances its counters
  before = _snapshot(a)
  calls = [lambda: a.step(acts, raster_b, frames),
           lambda: a.step_host(acts.cpu().numpy(), raster_b),
           lambda: a.step_host(acts.cpu().numpy(), raster_b, want_frames=False),
           lambda: a.step_gather(acts, raster_b, (ptrs, 1, 0, frames)),
           lambda: a.render(raster_b, frames)]
  for call in calls:
    with pytest.raises(_native.NativeError, match='another engine'):
      call()
    _assert_unchanged(a, before)
  # the same state moves on a step that is not refused
  a.step(acts)
  state, launches = _snapshot(a)
  assert launches == before[1] + 1 and not np.array_equal(state['step_count'], before[0]['step_count'])
  raster_b.close()
  a.close()
  b.close()


@pytest.mark.gpu
def test_step_host_checks_the_dtype_before_copying_actions():
  from spriteworld_b200 import _native
  from spriteworld_b200.engine import _as_ptr
  eng = _engine('embodied')
  acts = np.zeros((E, 2), np.int32)          # 8 B per env; float64 would read 32 B per env
  before = _snapshot(eng)
  for dt in (_native.DTYPE_F64, _native.DTYPE_F32):
    rc = eng._lib.swb_step_host(eng._h, None, _as_ptr(acts), dt, None, None, None, None, None,
                                eng._stream())
    assert rc != 0
    assert b'Embodied' in eng._lib.swb_last_error()
    _assert_unchanged(eng, before)
  assert eng._lib.swb_step_host(eng._h, None, _as_ptr(acts), _native.DTYPE_I32, None, None, None,
                                None, None, eng._stream()) == 0
  assert _snapshot(eng)[1] == before[1] + 1
  eng.close()
