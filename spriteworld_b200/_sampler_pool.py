"""Worker processes that sample and pack scenes for the batched environment's refill.

`init_sprites()` stays on the host (north_star), and in Python: a scene costs about 2-3 us to
draw and pack with NumPy, GIL-bound, so threads do not scale it.  At C2's reset rate (every env
every 20 steps) the ~18.6 M env-steps/s of C2 on an H100 want ~0.9 M scenes/s, more than one
core draws.
Each worker holds the generator, the task filters and the colour map (sent once, cloudpickle:
generators are closures), receives (n, seed) and writes the packed scene arrays
(scene.arrays_from_layout: what the in-process path uploads) into its block of POSIX shared
memory; only a few bytes travel through the pipe (pickling the arrays through it cost as much
as drawing them).  Workers import NumPy and this package's host modules only (no torch, no
CUDA) and run single-threaded.
"""
import multiprocessing as mp
import os
import threading
from multiprocessing import shared_memory

import numpy as np

# (field, dtype, trailing shape) of a scene batch, in the order they lie in a worker's block
_FIELDS = (('x', np.float64, ()), ('y', np.float64, ()), ('m00', np.float64, ()),
           ('m01', np.float64, ()), ('m10', np.float64, ()), ('m11', np.float64, ()),
           ('vx', np.float64, ()), ('vy', np.float64, ()), ('factors', np.float32, (5,)),
           ('member', np.uint32, ()), ('rgb', np.uint8, (3,)), ('shape', np.uint8, ()),
           ('pos_f32', np.uint8, ()))


def _views(buf, cap, n_slots, n):
  """name -> (n, n_slots[, ...]) array over the first n scenes of a block laid out for `cap`."""
  out, off = {}, 0
  for name, dtype, tail in _FIELDS:
    count = cap * n_slots * int(np.prod(tail, dtype=np.int64))
    a = np.frombuffer(buf, dtype=dtype, count=count, offset=off).reshape((cap, n_slots) + tail)
    out[name] = a[:n]
    off += (count * np.dtype(dtype).itemsize + 63) & ~63
  return out


def _block_bytes(cap, n_slots):
  off = 0
  for _, dtype, tail in _FIELDS:
    off += (cap * n_slots * int(np.prod(tail, dtype=np.int64)) * np.dtype(dtype).itemsize + 63) & ~63
  return off


def _worker_main(conn, payload, shm_name, cap):
  import time

  import cloudpickle
  from spriteworld_b200 import scene, sprite_generators
  init_sprites, n_slots, filters, color_to_rgb, goal_distribs = cloudpickle.loads(payload)
  shm = shared_memory.SharedMemory(name=shm_name)
  try:
    while True:
      try:
        msg = conn.recv()
      except EOFError:
        return
      if msg is None:
        return
      n, seed = msg
      try:
        t0 = time.perf_counter()
        np.random.seed(seed ^ 0x5BD1E995)    # generators whose callables draw from the global stream
        rng = np.random.RandomState(seed)
        layout = sprite_generators.batch_of(init_sprites, n, rng)
        goals = scene.draw_goals(goal_distribs, n, rng)   # right after the scenes, same stream
        batch = scene.arrays_from_layout(layout, n_slots, filters, color_to_rgb)
        if n <= cap:
          for name, view in _views(shm.buf, cap, n_slots, n).items():
            view[...] = batch[name]
          conn.send(('shm', (n, goals), time.perf_counter() - t0))
        else:   # larger than the block: through the pipe
          if goals is not None:
            batch['goal'] = goals
          conn.send(('pickle', batch, time.perf_counter() - t0))
      except Exception as ex:   # reported to the caller, the worker lives on
        conn.send(('error', ex, 0.0))
  finally:
    # leave without running destructors: NumPy views of the block are still alive in this frame,
    # and SharedMemory.__del__ would complain about them (the parent owns and unlinks the block)
    os._exit(0)


class SamplerPool(object):

  def __init__(self, n_procs, init_sprites, n_slots, filters, color_to_rgb, capacity=16384,
               goal_distribs=()):
    """capacity: scenes a worker's shared-memory block holds (larger requests fall back to
    pickling through the pipe).  goal_distribs: the task's goal distributions; a block's goals
    are drawn right after its scenes (scene.draw_goals) and come back as its 'goal' array."""
    import cloudpickle
    payload = cloudpickle.dumps((init_sprites, n_slots, list(filters), color_to_rgb, list(goal_distribs)))
    ctx = mp.get_context('spawn')
    self._conns, self._procs, self._locks, self._shm = [], [], [], []
    self._n_slots, self._cap = int(n_slots), int(capacity)
    self.worker_seconds = 0.0   # time the workers spent sampling and packing (summed)
    # The workers run single-threaded NumPy.  Without this every worker starts an OpenBLAS/OpenMP
    # pool of one thread per visible CPU, and a container may see many more CPUs than it may use:
    # hundreds of threads spinning at start-up exhaust the container's CPU quota and the cgroup
    # throttles the whole process tree for seconds.
    pinned = ('OMP_NUM_THREADS', 'OPENBLAS_NUM_THREADS', 'MKL_NUM_THREADS', 'NUMEXPR_NUM_THREADS')
    saved = {k: os.environ.get(k) for k in pinned}
    os.environ.update({k: '1' for k in pinned})
    n_procs = int(n_procs)
    try:
      for w in range(n_procs):
        shm = shared_memory.SharedMemory(create=True, size=_block_bytes(self._cap, self._n_slots))
        parent, child = ctx.Pipe()
        p = ctx.Process(target=_worker_main, args=(child, payload, shm.name, self._cap), daemon=True)
        p.start()
        child.close()
        self._conns.append(parent)
        self._procs.append(p)
        self._shm.append(shm)
        self._locks.append(threading.Lock())
    finally:
      for k, v in saved.items():
        if v is None:
          os.environ.pop(k, None)
        else:
          os.environ[k] = v

  def __len__(self):
    return len(self._procs)

  def request(self, worker, n, seed):
    """Asynchronous half of sample(): the worker starts drawing; collect() returns its arrays.
    One outstanding request per worker."""
    self._conns[worker].send((int(n), int(seed)))

  def collect(self, worker):
    """The arrays of the worker's outstanding request.  They are views of the worker's shared
    block: valid until the next request() to the same worker."""
    kind, out, seconds = self._conns[worker].recv()
    self.worker_seconds += seconds
    if kind == 'error':
      raise out
    if kind == 'shm':
      n, goals = out
      views = _views(self._shm[worker].buf, self._cap, self._n_slots, n)
      if goals is not None:
        views['goal'] = goals
      return views
    return out

  def sample(self, worker, n, seed):
    """request() + collect() (blocking; call it from one thread per worker to keep all busy)."""
    with self._locks[worker]:
      self.request(worker, n, seed)
      return self.collect(worker)

  def close(self):
    for c in self._conns:
      try:
        c.send(None)
        c.close()
      except Exception:  # pragma: no cover
        pass
    for p in self._procs:
      p.join(timeout=2)
      if p.is_alive():  # pragma: no cover
        p.terminate()
    for shm in self._shm:
      try:
        shm.unlink()
      except Exception:  # pragma: no cover
        pass
      try:
        shm.close()
      except BufferError:
        # a caller still holds views of the block: leave the mapping to them (it goes when they
        # do) and keep SharedMemory.__del__ from trying again
        shm._buf = None
        shm._mmap = None
    self._conns, self._procs, self._shm = [], [], []
