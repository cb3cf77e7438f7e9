"""Spriteworld environments on the H100 engine.

`Environment` is the drop-in for the reference's `spriteworld/environment.py:27-161`: same
constructor, `reset()/step()/observation_spec()/action_spec()/state()/success()`, dm_env
TimeSteps with NumPy observations, same auto-reset cadence and the same calls to
`init_sprites()` (hence the same draws from `np.random`) -- but every step runs on the
GPU through the C-ABI.

`BatchedEnvironment` advances `n_envs` independent copies of that environment in
lockstep: actions, rewards, step types and frames are device tensors, scenes come from a
device-resident pool of host-sampled scenes (`init_sprites.batch(n)`) that the step kernel
draws from when an env auto-resets, so no host work sits between two steps except the
periodic pool refill.
"""
import collections

import numpy as np
import torch

from spriteworld_b200 import _dm_env as dm_env
from spriteworld_b200 import _native, constants, scene
from spriteworld_b200 import engine as engine_lib
from spriteworld_b200 import sprite_generators
from spriteworld_b200.renderers import pil_renderer


def _split_renderers(renderers):
  pil = collections.OrderedDict()
  other = collections.OrderedDict()
  for name, r in renderers.items():
    (pil if isinstance(r, pil_renderer.PILRenderer) else other)[name] = r
  return pil, other


def _color_map(pil_renderers):
  maps = {id(r.color_to_rgb): r.color_to_rgb for r in pil_renderers.values()}
  if len(maps) > 1:
    raise NotImplementedError('all PILRenderers of one Environment must share color_to_rgb')
  return next(iter(maps.values())) if maps else None


def tune_host_allocator(threshold_bytes=1 << 30):
  """Opt-in, process-wide: keeps glibc from serving NumPy's temporaries (a few hundred KB each
  in the scene sampler) through mmap/munmap.  Each munmap shoots down TLB entries on every CPU a
  thread of the process has run on, and a process that drives a GPU has many threads (CUDA,
  OpenBLAS, OpenMP pools): the sampler was measured 3.6x slower late in a process than in a
  fresh one.  With the mmap threshold raised the arrays come from the heap instead.  Returns
  True if mallopt accepted both settings (Linux/glibc only)."""
  import ctypes
  try:
    libc = ctypes.CDLL('libc.so.6')
    M_TRIM_THRESHOLD, M_MMAP_THRESHOLD = -1, -3
    return bool(libc.mallopt(M_MMAP_THRESHOLD, int(threshold_bytes)) and
                libc.mallopt(M_TRIM_THRESHOLD, int(threshold_bytes)))
  except (OSError, AttributeError):
    return False


def _require_compilable(task, action_space):
  """The reference's task / action-space protocol is duck-typed (any object with reward/success
  or step/action_spec works there, on the host).  Here both run on the device, so they must be
  this package's classes (or subclasses that keep `compile()`): say so instead of failing
  with an AttributeError (DESIGN.md section 8)."""
  for what, obj, need in (('task', task, ('compile', '_filters_static')),
                          ('action_space', action_space, ('compile',))):
    missing = [m for m in need if not hasattr(obj, m)]
    if missing:
      raise NotImplementedError(
          '%s %r cannot run on the device: it has no %s(). User-defined tasks and action spaces '
          '(the reference accepts any duck-typed object) are out of scope of the GPU engine; '
          'compose spriteworld_b200.tasks / action_spaces classes instead.'
          % (what, type(obj).__name__, '/'.join(missing)))


class Environment(dm_env.Environment):
  """One Spriteworld environment (drop-in for the reference class)."""

  def __init__(self, task, action_space, renderers, init_sprites, keep_in_frame=True,
               max_episode_length=1000, metadata=None, device=0, max_sprites=None):
    self._task = task
    self._action_space = action_space
    self._renderers = renderers
    self._init_sprites = init_sprites
    self._keep_in_frame = keep_in_frame
    self._max_episode_length = max_episode_length
    self._metadata = metadata
    self._device = device
    _require_compilable(task, action_space)
    self._pil, self._other = _split_renderers(renderers)
    self._color_to_rgb = _color_map(self._pil)
    self._nodes, self._filters = task.compile()
    task._filters_static()
    self._engine = None
    self._rasters = {}
    self._max_sprites = max_sprites
    self._sprites = self._init_sprites()            # environment.py:68
    self._step_count = 0
    self._reset_next_step = True
    self._renderers_initialized = False
    self._ring = 0
    self._last = None          # (reward, step_type, success) of the last device step
    self._load_scene(first=True)

  # -- engine plumbing ---------------------------------------------------------------
  def _ensure_engine(self, n_sprites):
    """(Re)creates the one-env engine if it has too few sprite slots. Returns True if new."""
    if self._engine is not None and n_sprites <= self._engine.n_slots:
      return False
    slots = max(8, n_sprites, self._max_sprites or 0)
    if self._engine is not None:
      for r in self._rasters.values():
        r.close()
      self._engine.close()
    self._engine = engine_lib.Engine(
        1, slots, 2, self._action_space.compile(), self._nodes, constants.SHAPES,
        keep_in_frame=self._keep_in_frame,
        max_episode_length=int(min(self._max_episode_length, 2 ** 31 - 1)), device=self._device)
    self._rasters = {
        name: engine_lib.Raster(self._engine, r.width, r.height, r.anti_aliasing, r.bg_color)
        for name, r in self._pil.items()}
    return True

  def _load_scene(self, first=False):
    """Uploads self._sprites: as the live scene (constructor) or as the scene the next
    reset step switches to (ring of two slots)."""
    fresh = self._ensure_engine(len(self._sprites))
    eng = self._engine
    layout = sprite_generators.layout_from_sprite_lists([self._sprites])
    batch = scene.arrays_from_layout(layout, eng.n_slots, self._filters, self._color_to_rgb)
    if first or fresh:
      eng.upload_scenes(batch, [0], [0])
      eng.upload_state(pos_x=batch['x'], pos_y=batch['y'], cursor=[0], step_count=[0],
                       reset_next=[1])
      self._ring = 0
    if not first:
      self._ring = (self._ring + 1) % 2
      eng.upload_scenes(batch, [0], [self._ring])

  def _sync_sprites(self):
    """Copies the device positions into the host Sprite objects."""
    state = self._engine.download_state()
    n, S = len(self._sprites), self._engine.n_slots
    for j, s in enumerate(self._sprites):
      s._position[0] = state['pos_x'][0, S - n + j]
      s._position[1] = state['pos_y'][0, S - n + j]

  def _device_action(self, action):
    kind = self._action_space.compile()['kind']
    if kind == 'embodied':
      if action[1] not in (0, 1, 2, 3):
        raise KeyError(action[1])
      a = np.array([[int(bool(action[0])), int(action[1])]], np.int32)
    else:
      a = np.asarray(self._action_space.apply_noise_to_action(np.asarray(action)))
      a = a.reshape(1, 4)
      if a.dtype != np.float32:
        a = a.astype(np.float64)
    return torch.from_numpy(np.ascontiguousarray(a)).to(self._engine.device)

  def _run_step(self, action_tensor):
    eng = self._engine
    res = eng.step(action_tensor)
    frames = {}
    for name, r in self._rasters.items():
      frames[name] = eng.render(r)
      eng.check_render()
    torch.cuda.synchronize(eng.device)
    status = int(res.status[0].item())
    if status & _native.ENV_CLUSTER_LABELS:
      raise ValueError('Number of labels is invalid for the Davies-Bouldin score')
    if status & _native.ENV_CLUSTER_ZERODIV:
      raise ZeroDivisionError('float division by zero')
    self._last = (float(res.reward[0].item()), int(res.step_type[0].item()),
                  bool(res.success[0].item()))
    self._sync_sprites()
    return {name: f[0].cpu().numpy() for name, f in frames.items()}

  def _dummy_action(self):
    if self._action_space.compile()['kind'] == 'embodied':
      return torch.zeros((1, 2), dtype=torch.int32, device=self._engine.device)
    return torch.zeros((1, 4), dtype=torch.float32, device=self._engine.device)

  # -- dm_env API ----------------------------------------------------------------------
  def reset(self):
    self._sprites = self._init_sprites()            # environment.py:75
    self._step_count = 0
    self._reset_next_step = False
    self._load_scene()
    self._engine.request_reset()
    images = self._run_step(self._dummy_action())
    return dm_env.restart(self._observation(images))

  def success(self):
    return self._task.success(self._sprites) if self._last is None else self._last[2]

  def should_terminate(self):
    """What the device decides each step, evaluated on the host objects (environment.py:83-86)."""
    timeout = self._step_count >= self._max_episode_length
    out_of_frame = any(sprite.out_of_frame for sprite in self._sprites)
    return bool(self.success() or out_of_frame or timeout)

  def step(self, action):
    if self._reset_next_step:
      return self.reset()
    self._step_count += 1
    images = self._run_step(self._device_action(action))
    reward, step_type, _ = self._last
    observation = self._observation(images)
    if step_type == _native.STEP_LAST:
      self._reset_next_step = True
      return dm_env.termination(reward=reward, observation=observation)
    return dm_env.transition(reward=reward, observation=observation)

  def sample_contained_position(self):
    sprite = self._sprites[np.random.randint(len(self._sprites))]
    return sprite.sample_contained_position()

  def state(self):
    global_state = {'success': self.success()}
    if self._metadata:
      global_state['metadata'] = self._metadata
    return {'sprites': self._sprites, 'global_state': global_state}

  def _observation(self, images):
    state = self.state() if self._other else None
    out = {}
    for name in self._renderers:
      if name in images:
        out[name] = images[name]
      else:
        out[name] = self._other[name].render(**state)
    return out

  def observation(self):
    """Observation of the current state (renders on the device)."""
    eng = self._engine
    frames = {}
    for name, r in self._rasters.items():
      frames[name] = eng.render(r)
      eng.check_render()
    torch.cuda.synchronize(eng.device)
    return self._observation({name: f[0].cpu().numpy() for name, f in frames.items()})

  def observation_spec(self):
    if not self._renderers_initialized:
      self.observation()
      self._renderers_initialized = True
    return {name: r.observation_spec() for name, r in self._renderers.items()}

  def action_spec(self):
    return self._action_space.action_spec()

  @property
  def action_space(self):
    return self._action_space

  def close(self):
    if self._engine is not None:
      for r in self._rasters.values():
        r.close()
      self._engine.close()
      self._engine = None


BatchedTimeStep = collections.namedtuple(
    'BatchedTimeStep', ['step_type', 'reward', 'discount', 'observation', 'success', 'status'])


class BatchedEnvironment(object):
  """`n_envs` Spriteworld environments advanced in lockstep on one GPU.

  step(actions) takes a (n_envs, 4) float32/float64 or (n_envs, 2) int32 array/tensor and
  returns a BatchedTimeStep of device tensors: step_type int8 (dm_env.StepType values),
  reward float64 (0 on FIRST), discount float32 (1 MID/FIRST, 0 LAST), observation dict
  name -> uint8 (n_envs, H, W, 3), success uint8, status uint8 (per-env task errors the
  reference would raise: _native.ENV_*).
  """

  def __init__(self, task, action_space, renderers, init_sprites, keep_in_frame=True,
               max_episode_length=1000, metadata=None, n_envs=1, n_slots=None, pool_depth=8,
               device=0, rng=None, refill=None, refill_threads=1, refill_procs=0):
    """Args beyond the reference's Environment:
      n_envs: environments advanced in lockstep.
      n_slots: sprite slots per env; default: the generator's own bound (`max_sprites`), or,
        when a user callable draws the sprite count, the largest count seen in a probe sample.
      pool_depth: K, scenes kept per env on the device (the ring auto-resets draw from).
      refill: 'async' (default on CUDA: host threads sample and upload consumed ring slots
        over a side stream, the step stream waits only if a ring would underflow) or 'sync'.
      refill_threads: blocks of envs an asynchronous refill is split into (each has its own
        RandomState drawn from `rng`, so what a block draws does not depend on timing).
      refill_procs: worker processes that sample and pack the blocks' scenes at the same time
        (_sampler_pool; NumPy sampling is GIL-bound, threads do not scale it).  0 (default): the
        refill thread samples block after block.  Opt-in: next to a stepping process the
        workers have been seen running one after the other (DESIGN.md section 4).
    """
    self._task, self._action_space = task, action_space
    self._renderers = renderers
    self._init_sprites = init_sprites
    self._metadata = metadata
    self.n_envs = int(n_envs)
    self._rng = rng if rng is not None else np.random
    _require_compilable(task, action_space)
    self._pil, self._other = _split_renderers(renderers)
    unsupported = [n for n, r in self._other.items() if not hasattr(r, 'render_batch')]
    if unsupported:
      raise NotImplementedError('renderers %s have no batched form' % unsupported)
    self._color_to_rgb = _color_map(self._pil)
    self._nodes, self._filters = task.compile()
    task._filters_static()
    self._K = max(3, int(pool_depth))
    E, K = self.n_envs, self._K
    first = self._sample(E * K)
    slots = n_slots or getattr(init_sprites, 'max_sprites', None)
    if not slots:
      # the count is drawn by a user callable: size the slots from a probe sample, so that a
      # later refill cannot meet a larger scene in the middle of a run
      probe = self._sample(4096)
      slots = max(1, int(first.count.max()), int(probe.count.max()))
    slots = max(1, int(slots))
    self._engine = engine_lib.Engine(
        E, slots, K, action_space.compile(), self._nodes, constants.SHAPES,
        keep_in_frame=keep_in_frame,
        max_episode_length=int(min(max_episode_length, 2 ** 31 - 1)), device=device)
    self._rasters = collections.OrderedDict(
        (name, engine_lib.Raster(self._engine, r.width, r.height, r.anti_aliasing, r.bg_color))
        for name, r in self._pil.items())
    self._frames = {name: r.new_frames() for name, r in self._rasters.items()}
    batch0 = self._upload(first, np.repeat(np.arange(E), K), np.tile(np.arange(K), E))
    # env e starts on its scene 0 (the constructor's sample, environment.py:68) and is about
    # to reset (environment.py:70)
    self._engine.upload_state(pos_x=batch0['x'][::K], pos_y=batch0['y'][::K],
                              cursor=np.zeros(E), step_count=np.zeros(E), reset_next=np.ones(E))
    # Ring bookkeeping in absolute scene indices: scene a of an env lives in ring slot a % K;
    # the device counts the scenes an env has started (scene_serial), so "serial" is the scene
    # it is on and scenes serial+1 .. _refilled_upto are fresh.  A refill brings every env up
    # to serial + K - 1 (the slot of the scene before the current one).
    self._refilled_upto = np.full(E, K - 1, np.int64)
    if refill is None:
      refill = 'async' if self._engine.device.type == 'cuda' else 'sync'
    if refill not in ('async', 'sync'):
      raise ValueError("refill must be 'async' or 'sync'")
    self._refill_mode = refill
    # Underflow guard.  Between the snapshot a landed refill was computed from (step _safe_step,
    # explicit resets so far _safe_resets) and step t an env can have started at most
    # ceil((t - _safe_step) / 2) + (resets since) scenes: an auto-reset takes a LAST and a
    # FIRST step, an explicit reset() one step.  K - 1 fresh scenes were there at the snapshot.
    self._t = 0                    # steps enqueued
    self._resets = 0               # explicit reset() calls
    self._safe_step, self._safe_resets = 0, 0
    self._period = max(1, (K - 2) // 2 if refill == 'async' else 2 * (K - 2))
    self._inflight = None          # async: dict(snapshot step/resets, future)
    # async: the last snapshots of scene_serial, (step, resets, SerialSnapshot).  They are taken
    # every few steps, ahead of need: the step stream runs tens of steps behind the host, and a
    # refill that had to wait for a snapshot ordered behind everything enqueued would leave the
    # sampler idle for that long; it starts from the newest snapshot that has already landed.
    self._snaps = collections.deque(maxlen=12)
    self._snap_every = max(1, (K - 2) // 4)
    self._last_snap = -(1 << 30)
    self._worker = None
    self._stats = dict(refills=0, scenes=0, host_seconds=0.0, blocked_seconds=0.0, blocked=0,
                       collect_seconds=0.0, upload_seconds=0.0)
    if refill == 'async':
      import concurrent.futures
      self._worker = concurrent.futures.ThreadPoolExecutor(1, thread_name_prefix='swb-refill')
      n_thr = max(1, min(max(int(refill_threads), int(refill_procs or 0)), E))
      # one RandomState per block of envs, so that the blocks' draws do not depend on timing
      # (never `rng` itself: the step thread draws the action noise from it)
      self._block_rngs = [np.random.RandomState(self._rng.randint(0, 2 ** 31 - 1))
                          for _ in range(n_thr)]
      self._block_edges = np.linspace(0, E, len(self._block_rngs) + 1).astype(np.int64)
      self._pool = None
      if refill_procs:
        from spriteworld_b200 import _sampler_pool
        self._pool = _sampler_pool.SamplerPool(min(int(refill_procs), n_thr), init_sprites, slots,
                                               self._filters, self._color_to_rgb)

  # -- scenes ----------------------------------------------------------------------------
  def _sample(self, n):
    return sprite_generators.batch_of(self._init_sprites, n, self._rng)

  def _upload(self, layout, env_ids, ring_slots, batch=None):
    if batch is None:
      batch = scene.arrays_from_layout(layout, self._engine.n_slots, self._filters,
                                       self._color_to_rgb)
    self._engine.upload_scenes(batch, env_ids, ring_slots)
    if self._other:   # static factors of the pooled scenes, for factor observations
      E, K, S = self.n_envs, self._K, self._engine.n_slots
      if getattr(self, '_pool_static', None) is None:
        self._pool_static = torch.zeros((E, K, S, 8), dtype=torch.float32,
                                        device=self._engine.device)
      static = np.concatenate([batch['shape'][..., None].astype(np.float32), batch['factors'],
                               batch['vx'][..., None].astype(np.float32),
                               batch['vy'][..., None].astype(np.float32)], -1)
      e = torch.as_tensor(np.asarray(env_ids), device=self._engine.device, dtype=torch.long)
      k = torch.as_tensor(np.asarray(ring_slots), device=self._engine.device, dtype=torch.long)
      self._pool_static[e, k] = torch.from_numpy(static).to(self._engine.device)
    return batch

  _STATIC_COLUMNS = {'shape': 0, 'scale': 1, 'angle': 2, 'c0': 3, 'c1': 4, 'c2': 5,
                     'x_vel': 6, 'y_vel': 7}

  def factor_tensors(self, factors):
    """dict factor name -> float32 (n_envs, n_slots) tensor of the current scenes + 'mask'."""
    live = self._engine.state_tensors()
    rows = torch.arange(self.n_envs, device=self._engine.device)
    static = self._pool_static[rows, live['cursor'].long()]      # (E, S, 8)
    out = collections.OrderedDict()
    for name in factors:
      if name == 'x':
        out[name] = live['pos_x'].to(torch.float32)
      elif name == 'y':
        out[name] = live['pos_y'].to(torch.float32)
      else:
        out[name] = static[..., self._STATIC_COLUMNS[name]]
    out['mask'] = static[..., 0] > 0
    return out

  def _plan_block(self, serial, lo, hi):
    """Ring slots of envs [lo, hi) to refill so that every ring reaches serial + K - 1:
    (env ids, absolute scene indices, new `refilled_upto`) or None."""
    K = self._K
    upto = self._refilled_upto[lo:hi]
    want_upto = np.asarray(serial, np.int64)[lo:hi] + (K - 1)
    n_new = np.maximum(want_upto - upto, 0)
    total = int(n_new.sum())
    if total <= 0:
      return None
    env_ids = np.repeat(np.arange(lo, hi), n_new)
    # 1..n_new[e] for every env, concatenated
    offs = np.arange(total) - np.repeat(np.cumsum(n_new) - n_new, n_new) + 1
    absolute = np.repeat(upto, n_new) + offs
    return env_ids, absolute, np.maximum(upto, want_upto)

  def _refill_from(self, serial, rng=None):
    """Synchronous form: samples (in this thread, from `rng`) and uploads what brings every
    env's ring up to serial + K - 1.  Returns the number of scenes uploaded."""
    plan = self._plan_block(serial, 0, self.n_envs)
    if plan is None:
      return 0
    env_ids, absolute, upto = plan
    layout = sprite_generators.batch_of(self._init_sprites, len(env_ids),
                                        self._rng if rng is None else rng)
    self._upload(layout, env_ids, absolute % self._K)
    self._refilled_upto[:] = upto
    return len(env_ids)

  def _refill_job(self, snapshot):
    """Worker thread: wait for the snapshot copy (not for the step stream), have the blocks'
    scenes drawn and packed -- all worker processes at once, or here, block after block --
    and upload them over the side stream.  Returns the event after which they are in the pool."""
    import time
    serial = snapshot.wait()
    t0 = time.perf_counter()
    eng = self._engine
    K, n = self._K, 0
    edges = self._block_edges
    plans = [self._plan_block(serial, int(edges[i]), int(edges[i + 1])) for i in range(len(edges) - 1)]
    with eng.side_stream_context():
      if self._pool is not None:
        # every worker draws its block at the same time; collect and upload in block order
        for i, plan in enumerate(plans):
          if plan is not None:
            self._pool.request(i % len(self._pool), len(plan[0]), self._block_rngs[i].randint(0, 2 ** 31 - 1))
            if (i + 1) % len(self._pool) == 0 or i + 1 == len(plans):
              for j in range(i - i % len(self._pool), i + 1):
                if plans[j] is not None:
                  tc = time.perf_counter()
                  batch = self._pool.collect(j % len(self._pool))
                  t1 = time.perf_counter()
                  self._stats['collect_seconds'] += t1 - tc   # waiting for the worker's block
                  self._upload(None, plans[j][0], plans[j][1] % K, batch=batch)
                  self._stats['upload_seconds'] += time.perf_counter() - t1
      else:
        for i, plan in enumerate(plans):
          if plan is not None:
            layout = sprite_generators.batch_of(self._init_sprites, len(plan[0]), self._block_rngs[i])
            self._upload(layout, plan[0], plan[1] % K)
      for i, plan in enumerate(plans):
        if plan is not None:
          self._refilled_upto[int(edges[i]):int(edges[i + 1])] = plan[2]
          n += len(plan[0])
      done = eng.record_side_event()
    self._stats['host_seconds'] += time.perf_counter() - t0
    self._stats['refills'] += 1
    self._stats['scenes'] += n
    return done

  def _risk(self, t):
    """Upper bound of the scenes an env can have started by step t since the last landed refill."""
    return (t - self._safe_step + 1) // 2 + (self._resets - self._safe_resets)

  def _land(self, block):
    """Absorbs the in-flight refill if it is finished (or waits for it): the step stream waits
    on its upload event, the guard moves to its snapshot."""
    job = self._inflight
    if job is None or not (block or job['future'].done()):
      return
    if not job['future'].done():
      import time
      t0 = time.perf_counter()
      job['future'].result()
      self._stats['blocked_seconds'] += time.perf_counter() - t0
      self._stats['blocked'] += 1
    self._engine.wait_event(job['future'].result())
    self._safe_step, self._safe_resets = job['step'], job['resets']
    self._inflight = None

  def _snapshot(self):
    self._snaps.append((self._t, self._resets, self._engine.snapshot_scene_serial()))
    self._last_snap = self._t

  def _request(self):
    """Starts a refill from the newest snapshot that has landed (or, if none newer than the last
    refill has, from the oldest pending one: it lands first)."""
    fresh = [rec for rec in self._snaps if rec[0] > self._safe_step]
    if not fresh:
      self._snapshot()
      fresh = [self._snaps[-1]]
    landed = [rec for rec in fresh if rec[2].ready()]
    step, resets, snapshot = landed[-1] if landed else fresh[0]
    self._inflight = dict(step=step, resets=resets,
                          future=self._worker.submit(self._refill_job, snapshot))

  def _keep_ring_fresh(self):
    """Called before a step is enqueued."""
    K = self._K
    if self._refill_mode == 'sync':
      if self._t - self._safe_step >= self._period or self._risk(self._t + 1) > K - 1:
        import time
        t0 = time.perf_counter()
        serial = self._engine.download_state_serial()
        self._stats['scenes'] += self._refill_from(serial)
        self._stats['refills'] += 1
        self._stats['host_seconds'] += time.perf_counter() - t0
        self._safe_step, self._safe_resets = self._t, self._resets
      return
    self._land(block=False)
    if self._t - self._last_snap >= self._snap_every:
      self._snapshot()
    if self._inflight is None and self._t - self._safe_step >= self._period:
      self._request()
    while self._risk(self._t + 1) > K - 1:   # this step could run a ring dry: wait for scenes
      if self._inflight is None:
        self._request()
      self._land(block=True)

  def refill_stats(self):
    """Counters of the scene-ring refill: refills, scenes sampled, host seconds spent sampling
    and packing, and how often / how long a step had to wait for scenes."""
    return dict(self._stats, mode=self._refill_mode, pool_depth=self._K,
                threads=len(getattr(self, '_block_rngs', [None])),
                procs=len(self._pool) if getattr(self, '_pool', None) is not None else 0)

  # -- API ---------------------------------------------------------------------------------
  @property
  def engine(self):
    return self._engine

  def _to_device(self, actions):
    dev = self._engine.device
    if isinstance(actions, torch.Tensor):
      t = actions
    else:
      a = np.asarray(actions)
      if self._action_space.compile()['kind'] == 'embodied':
        a = a.astype(np.int32)
      elif a.dtype != np.float32:
        a = a.astype(np.float64)
      t = torch.from_numpy(np.ascontiguousarray(a))
    t = t.to(dev)
    noise_scale = getattr(self._action_space, '_noise_scale', None)
    if noise_scale and self._action_space.compile()['kind'] != 'embodied':
      # SelectMove.apply_noise_to_action (action_spaces.py:69-75), one draw per env; like
      # there, float32 actions become float64 by the addition
      noise = self._rng.normal(loc=0.0, scale=noise_scale, size=(self.n_envs, 4))
      t = t.to(torch.float64) + torch.from_numpy(noise).to(dev)
    return t.contiguous()

  def _timestep(self, res):
    obs = collections.OrderedDict()
    for name in self._renderers:
      if name in self._frames:
        obs[name] = self._frames[name]
      else:
        obs[name] = self._other[name].render_batch(self, res)
    discount = (res.step_type != _native.STEP_LAST).to(torch.float32)
    return BatchedTimeStep(res.step_type, res.reward, discount, obs, res.success, res.status)

  def step(self, actions):
    eng = self._engine
    self._keep_ring_fresh()
    self._t += 1
    t = self._to_device(actions)
    names = list(self._rasters)
    if names:
      res = eng.step(t, self._rasters[names[0]], self._frames[names[0]])
      for name in names[1:]:
        eng.render(self._rasters[name], self._frames[name])
        res.status.bitwise_or_(eng.render_status())   # span overflow of the extra rasters
    else:
      res = eng.step(t)
    return self._timestep(res)

  def reset(self):
    """Restarts every env from its next pooled scene; returns the FIRST timestep."""
    self._resets += 1
    self._engine.request_reset()
    kind = self._action_space.compile()['kind']
    shape, dtype = ((self.n_envs, 2), torch.int32) if kind == 'embodied' else (
        (self.n_envs, 4), torch.float32)
    return self.step(torch.zeros(shape, dtype=dtype, device=self._engine.device))

  def observation_spec(self):
    """Per-env specs (the leading n_envs axis of the batched observations is not included)."""
    return {name: (r.batch_observation_spec(self) if hasattr(r, 'batch_observation_spec')
                   else r.observation_spec()) for name, r in self._renderers.items()}

  def action_spec(self):
    return self._action_space.action_spec()

  @property
  def action_space(self):
    return self._action_space

  def close(self):
    if self._worker is not None:
      if self._inflight is not None:
        try:
          self._inflight['future'].result()
        except Exception:  # pragma: no cover
          pass
        self._inflight = None
      self._worker.shutdown(wait=True)
      self._worker = None
      if self._pool is not None:
        self._pool.close()
        self._pool = None
    if self._engine.device.type == 'cuda':
      torch.cuda.synchronize(self._engine.device)
    for r in self._rasters.values():
      r.close()
    self._engine.close()


class ShardedBatchedEnvironment(object):
  """`n_envs_total` environments sharded by env index over the ranks of a process group, one
  BatchedEnvironment (one GPU) per rank; every rank's step() returns the BatchedTimeStep of
  ALL envs, ordered by global env index.

  The path's single collective is the gather of a step's outputs (SURVEY 8(e)):
    * the frames are stored into every rank's gathered buffer by the render kernel itself, over
      NVLink peer memory (distributed.PeerFrames, swb_step_render_gather);
    * reward, step type, success and status (11 bytes per env, one packed buffer per rank) ride
      along as ONE NCCL all-gather enqueued behind the kernel, which is also the completion
      barrier of the frame stores: it cannot finish on a rank before every rank's kernel has.
  Requires n_envs_total % world_size == 0 (equal shards; distributed.StepGatherer pads
  otherwise).  `actions` may be this rank's shard (E_local, ...) or the global batch.

  host_barrier=True (tests with several ranks on one device, where NCCL refuses to run):
  device synchronise + host barrier, outputs gathered through the host.
  """

  def __init__(self, n_envs_total, group=None, device=None, seed=0, frame_slots=2,
               host_barrier=False, **config):
    import torch.distributed as dist
    from spriteworld_b200 import distributed
    self.group = group
    self.world = dist.get_world_size(group)
    self.rank = dist.get_rank(group)
    self.n_envs_total = int(n_envs_total)
    if self.n_envs_total % self.world:
      raise ValueError('n_envs_total (%d) must be a multiple of the world size (%d)'
                       % (self.n_envs_total, self.world))
    self.env_start, self.n_local = distributed.env_shard(self.n_envs_total, self.rank, self.world)
    if device is None:
      device = torch.cuda.current_device()
    self.host_barrier = host_barrier
    # every rank draws its own scenes: same seed, rank-specific stream
    self.local = BatchedEnvironment(n_envs=self.n_local, device=device,
                                    rng=np.random.RandomState((int(seed) + 7919 * self.rank) % (2 ** 31)),
                                    **config)
    eng = self.local.engine
    names = list(self.local._rasters)
    if len(names) != 1:
      raise NotImplementedError('ShardedBatchedEnvironment gathers exactly one PILRenderer observation')
    self._image = names[0]
    r = self.local._rasters[self._image]
    self._peer = distributed.PeerFrames(self.n_local, (r.height, r.width, 3), eng.device,
                                        n_slots=max(2, int(frame_slots)), group=group,
                                        host_barrier=host_barrier)
    self._out_all = torch.empty(self.world * self.n_local * engine_lib.OUT_BYTES_PER_ENV,
                                dtype=torch.uint8, device=eng.device)
    self._t = 0

  @property
  def engine(self):
    return self.local.engine

  def _local_actions(self, actions):
    n = actions.shape[0]
    if n == self.n_envs_total and self.world > 1:
      return actions[self.env_start:self.env_start + self.n_local]
    return actions

  def step(self, actions):
    import torch.distributed as dist
    env, eng = self.local, self.local.engine
    env._keep_ring_fresh()
    env._t += 1
    t = env._to_device(self._local_actions(actions))
    targets = self._peer.slot(self._t)
    res = eng.step_gather(t, env._rasters[self._image], targets)
    E, W = self.n_local, self.world
    if self.host_barrier:
      self._peer.barrier()
      parts = [torch.empty_like(eng.out_bytes, device='cpu') for _ in range(W)]
      dist.all_gather(parts, eng.out_bytes.cpu(), group=self.group)
      self._out_all.copy_(torch.cat(parts))
    else:
      # the step's one collective besides the frame stores; completes only after every rank's
      # render kernel (and with it its peer stores) has
      dist.all_gather_into_tensor(self._out_all, eng.out_bytes, group=self.group)
    self._t += 1
    per_rank = self._out_all.view(W, engine_lib.OUT_BYTES_PER_ENV * E)
    reward = per_rank[:, :8 * E].contiguous().view(torch.float64).reshape(W * E)
    step_type = per_rank[:, 8 * E:9 * E].reshape(W * E).view(torch.int8)
    success = per_rank[:, 9 * E:10 * E].reshape(W * E)
    status = per_rank[:, 10 * E:11 * E].reshape(W * E)
    discount = (step_type != _native.STEP_LAST).to(torch.float32)
    obs = collections.OrderedDict([(self._image, res.frames)])
    return BatchedTimeStep(step_type, reward, discount, obs, success, status)

  def reset(self):
    env = self.local
    env._resets += 1
    env.engine.request_reset()
    kind = env._action_space.compile()['kind']
    shape, dtype = ((self.n_local, 2), torch.int32) if kind == 'embodied' else (
        (self.n_local, 4), torch.float32)
    return self.step(torch.zeros(shape, dtype=dtype, device=env.engine.device))

  def observation_spec(self):
    return self.local.observation_spec()

  def action_spec(self):
    return self.local.action_spec()

  def close(self):
    if self.local.engine.device.type == 'cuda':
      torch.cuda.synchronize(self.local.engine.device)
    self._peer.close()
    self.local.close()
