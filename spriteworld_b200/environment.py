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
from spriteworld_b200.renderers import glimpses, handcrafted, pil_renderer


def _split_renderers(renderers):
  pil = collections.OrderedDict()
  other = collections.OrderedDict()
  for name, r in renderers.items():
    (pil if isinstance(r, pil_renderer.PILRenderer) else other)[name] = r
  return pil, other


def _color_map(pil_renderers):
  """The one colour map of `pil_renderers` (PILRenderers, and in a BatchedEnvironment also
  SpriteGlimpses and SpriteLayers: colours are packed into the scenes at upload), or None."""
  maps = {id(r.color_to_rgb): r.color_to_rgb for r in pil_renderers.values()}
  if len(maps) > 1:
    raise NotImplementedError('all PILRenderers, SpriteGlimpses and SpriteLayers of one Environment must share '
                              'color_to_rgb')
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


def _rng_state(rng):
  """The state of a RandomState (or of the np.random module: NumPy's global state) as
  (str, int64 tensor, int, int, float), which torch.load(weights_only=True) reads back."""
  name, keys, pos, has_gauss, cached = rng.get_state()
  return (str(name), torch.from_numpy(np.asarray(keys).astype(np.int64)), int(pos), int(has_gauss),
          float(cached))


def _set_rng_state(rng, state):
  name, keys, pos, has_gauss, cached = state
  rng.set_state((str(name), keys.numpy().astype(np.uint32), int(pos), int(has_gauss), float(cached)))


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
    task._constant_goals('the one-env Environment')
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
        keep_in_frame=self._keep_in_frame, max_episode_length=self._max_episode_length,
        device=self._device)
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
    else:
      action = self._action_space.apply_noise_to_action(np.asarray(action))
    a = engine_lib.host_actions(kind, np.reshape(action, (1, -1)))
    return torch.from_numpy(a).to(self._engine.device)

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

  # -- dm_env API ----------------------------------------------------------------------
  def reset(self):
    self._sprites = self._init_sprites()            # environment.py:75
    self._step_count = 0
    self._reset_next_step = False
    self._load_scene()
    self._engine.request_reset()
    zero = engine_lib.zero_actions(self._action_space.compile()['kind'], 1)
    images = self._run_step(torch.from_numpy(zero).to(self._engine.device))
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


BatchedRollout = collections.namedtuple(
    'BatchedRollout', ['step_type', 'reward', 'discount', 'success', 'status'])


ContainedPositions = collections.namedtuple('ContainedPositions', ['position', 'slot', 'status'])


class BatchedEnvironment(object):
  """`n_envs` Spriteworld environments advanced in lockstep on one GPU.

  step(actions) takes a (n_envs, 4) float32/float64 or (n_envs, 2) int32 array/tensor and
  returns a BatchedTimeStep of device tensors: step_type int8 (dm_env.StepType values),
  reward float64 (0 on FIRST), discount float32 (1 MID/FIRST, 0 LAST), observation dict
  name -> uint8 (n_envs, H, W, 3), success uint8, status uint8 (per-env task errors the
  reference would raise: _native.ENV_*).

  rollout(actions) scores plans without stepping: for (T, n_envs, C, 4) or (T, n_envs, C, 2)
  actions it returns a BatchedRollout of (T, n_envs, C) device tensors, entry [t, e, c] being what
  step t of candidate c would report for env e from the state it is in now.  No env changes.
  rollout(actions, states) plans from saved env records instead, and expand(actions, states) also
  returns the state each plan ends in, as records: one level of a search tree.
  rollout_trajectory(actions, states) returns the state after every step instead, for the
  observations of each imagined step.
  """

  def __init__(self, task, action_space, renderers, init_sprites, keep_in_frame=True,
               max_episode_length=1000, metadata=None, n_envs=1, n_slots=None, pool_depth=8,
               device=0, rng=None, refill=None, refill_threads=1, refill_procs=0, sampler='host',
               seed=None, env_offset=0):
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
      sampler: 'host' (default: scenes drawn by init_sprites' NumPy sampler, as the reference
        draws them for a given seed) or 'device': init_sprites compiled to a program
        (scene_program.compile_program) that the GPU runs.  Scene a of env e is then a pure
        function of (seed, env_offset + e, a): the same distribution as the host's, drawn from
        its own stream, independent of timing; refills are kernels on the step stream, with no
        host thread.  `refill`, `refill_threads` and `refill_procs` do not apply.
      seed: the device sampler's seed (default: drawn from `rng`).
      env_offset: the global id of env 0 for the device sampler (a shard's first env).
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
    self._views = collections.OrderedDict(
        (n, r) for n, r in self._other.items() if isinstance(r, glimpses._SpriteViews))
    self._color_to_rgb = _color_map(collections.OrderedDict(list(self._pil.items()) + list(self._views.items())))
    self._nodes, self._filters = task.compile()
    task._filters_static()
    self._goal_distribs = task.goal_distributions()
    self._K = max(3, int(pool_depth))
    E, K = self.n_envs, self._K
    if sampler not in ('host', 'device'):
      raise ValueError("sampler must be 'host' or 'device'")
    self._sampler = sampler
    if sampler == 'device':
      from spriteworld_b200 import scene_program
      self._program = scene_program.compile_program(init_sprites, self._filters, self._color_to_rgb,
                                                    self._goal_distribs)
      slots = n_slots or self._program.max_sprites
    else:
      first, first_goals = self._sample(E * K)
      slots = n_slots or getattr(init_sprites, 'max_sprites', None)
      if not slots:
        # the count is drawn by a user callable: size the slots from a probe sample, so that a
        # later refill cannot meet a larger scene in the middle of a run
        probe, _ = self._sample(4096)
        slots = max(1, int(first.count.max()), int(probe.count.max()))
    slots = max(1, int(slots))
    self._engine = engine_lib.Engine(
        E, slots, K, action_space.compile(), self._nodes, constants.SHAPES,
        keep_in_frame=keep_in_frame, max_episode_length=max_episode_length, device=device)
    self._rasters = collections.OrderedDict(
        (name, engine_lib.Raster(self._engine, r.width, r.height, r.anti_aliasing, r.bg_color))
        for name, r in self._pil.items())
    self._frames = {name: r.new_frames() for name, r in self._rasters.items()}
    # the outputs of each SpriteMasks, SpriteCoverage, SoftSpriteMasks and SpriteBoxes renderer by
    # id(renderer), overwritten every step like the frames: one dict, also under the coverage and
    # soft-mask buffer names the test suite reads them by
    self._mask_buffers = {
        id(r): engine_lib._new_mask_outputs(self._engine, r._kind, E, r.width, r.height)
        for r in self._other.values() if isinstance(r, handcrafted._SpriteMaskRenderer)}
    self._coverage_buffers = self._soft_buffers = self._mask_buffers
    # rasters of render_windows by (W, H, aa, bg), those of the SpriteGlimpses and SpriteLayers
    # renderers made here (a raster the engine refuses fails the constructor, not a step), and each
    # such renderer's views and their status by id(renderer), overwritten every step like the frames
    self._window_rasters = {}
    self._glimpse_buffers = {}
    for r in self._views.values():
      self._window_raster(r)
      V = len(r.slot_indices(slots))
      self._glimpse_buffers[id(r)] = (
          torch.empty((E, V, r.height, r.width, 3), dtype=torch.uint8, device=self._engine.device),
          torch.empty((E, V), dtype=torch.uint8, device=self._engine.device))
    if sampler == 'device':
      self._init_device_sampler(seed, env_offset)
      return
    batch0 = self._upload(first, np.repeat(np.arange(E), K), np.tile(np.arange(K), E), goals=first_goals)
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
    # A load or copy counts as an explicit reset: a record saved about to reset (reset_next = 1)
    # makes the env start its next ring scene on the next step, as reset() does.
    self._t = 0                    # steps enqueued
    self._resets = 0               # explicit reset() calls, load_envs and copy_envs calls
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
                                               self._filters, self._color_to_rgb,
                                               goal_distribs=self._goal_distribs)

  def _init_device_sampler(self, seed, env_offset):
    E, K = self.n_envs, self._K
    self.seed = int(self._rng.randint(0, 2 ** 31 - 1)) if seed is None else int(seed)
    self._env_offset = int(env_offset)
    self._engine.load_sampler(self._program, self.seed, env_offset)
    # every ring gets scenes 0 .. K-1; env e starts on its scene 0 and is about to reset
    self._engine.refill_device()
    first = self._engine.sample_scenes(np.arange(E) + int(env_offset), np.zeros(E))
    self._engine.upload_state(pos_x=first['x'].cpu().numpy(), pos_y=first['y'].cpu().numpy(),
                              cursor=np.zeros(E), step_count=np.zeros(E), reset_next=np.ones(E))
    self._refill_mode = 'device'
    self._t, self._resets = 0, 0
    self._safe_step, self._safe_resets = 0, 0
    # a launch is stream-ordered before the next step: it covers everything up to that step
    self._period = max(1, 2 * (K - 2))
    self._worker = None
    self._stats = dict(refills=0)

  def check_sampler(self):
    """sampler='device': raises the reference's ValueError if a rejection loop ran out of tries
    (that scene was left empty) since the last check.  Synchronises."""
    self._engine.check_sampler()

  # -- scenes ----------------------------------------------------------------------------
  def _sample(self, n, rng=None):
    """(SceneLayout of n scenes, their goals (n, G, 2) or None), the goals drawn right after the
    scenes from the same RandomState (default: `rng`)."""
    rng = self._rng if rng is None else rng
    layout = sprite_generators.batch_of(self._init_sprites, n, rng)
    return layout, scene.draw_goals(self._goal_distribs, n, rng)

  def _upload(self, layout, env_ids, ring_slots, batch=None, goals=None):
    if batch is None:
      batch = scene.arrays_from_layout(layout, self._engine.n_slots, self._filters,
                                       self._color_to_rgb)
    if goals is not None:
      batch['goal'] = goals
    self._engine.upload_scenes(batch, env_ids, ring_slots)
    return batch

  _FACTOR_COLUMNS = {'scale': 0, 'angle': 1, 'c0': 2, 'c1': 3, 'c2': 4}   # of the pool's `factors`

  def factor_tensors(self, factors, states=None):
    """dict factor name -> float32 (n_envs, n_slots) tensor of the current scenes + 'mask': x and y
    are the live positions, the rest is read from the pool entry each env is on.

    With `states` (EnvStates of n records) the same dict of (n, n_slots) tensors is read from the
    records on their device, without a host synchronisation: what factor_tensors() would return
    after load_envs(states), shape ids sanitised as a load sanitises them."""
    if states is not None:
      return self._record_factor_tensors(factors, states)
    eng = self._engine
    live, pool, K = eng.state_tensors(), eng.pool_tensors(), eng.pool_depth
    entry = torch.arange(0, self.n_envs * K, K, device=eng.device) + live['cursor']   # env * K + cursor

    def at(field):   # (n_envs, n_slots[, 5]): the field of the pool entry each env is on
      return pool[field].flatten(0, 1).index_select(0, entry)

    shape, columns = at('shape'), None
    out = collections.OrderedDict()
    for name in factors:
      if name in ('x', 'y'):
        out[name] = live['pos_' + name].to(torch.float32)
      elif name in ('x_vel', 'y_vel'):
        out[name] = at('v' + name[0]).to(torch.float32)
      elif name == 'shape':
        out[name] = shape.to(torch.float32)
      else:
        columns = at('factors') if columns is None else columns
        out[name] = columns[..., self._FACTOR_COLUMNS[name]]
    out['mask'] = shape > 0
    return out

  @property
  def n_goals(self):
    """G: goals drawn per scene (the task's FindGoalPosition nodes with a goal distribution)."""
    return len(self._goal_distribs)

  def goal_tensor(self, states=None):
    """float64 (n_envs, G, 2) device tensor: the goals of the scene each env is on (GoalPositions),
    or with `states` (EnvStates of n records) a new (n, G, 2) tensor of the records' goals."""
    eng = self._engine
    if states is not None:
      eng.check_states(states, len(states))
      if not self.n_goals:
        return torch.zeros((len(states), 0, 2), dtype=torch.float64, device=states.data.device)
      return states.fields()['goal'].clone()
    if not self.n_goals:
      return torch.zeros((self.n_envs, 0, 2), dtype=torch.float64, device=eng.device)
    views = getattr(self, '_goal_views', None)
    if views is None:   # zero-copy views and the entry base e * K, made once
      K = eng.pool_depth
      views = self._goal_views = (torch.arange(0, self.n_envs * K, K, dtype=torch.int32, device=eng.device),
                                  eng.state_tensors()['cursor'], eng.pool_tensors()['goal'].flatten(0, 1))
    base, cursor, goal = views
    return goal.index_select(0, base + cursor)

  def set_goals(self, goals, env_ids=None, check='host'):
    """The goals of the scene env env_ids[i] is on <- goals[i] (float64 (n, G, 2) on the engine's
    device; default ids: all envs, in order; distinct), on the step stream.  The env keeps them
    until it starts its next scene, which brings a drawn goal.  Ids as load_envs takes them; a
    device-checked call is all or nothing (Engine.check_env_ids reports a refused one).  It writes
    only the pool entry each env is on, as a load does, and counts against the ring's refill guard
    like a load.

    An env whose last step was LAST is still on the finished scene: goals set now are replaced by
    the next scene's drawn goals at the reset that follows.  To choose the goal of an env's next
    episode, set it after the FIRST step of that episode (the reset step observes no reward)."""
    if engine_lib.device_checked(check, env_ids):
      self._engine.set_goals(goals, env_ids, check='device')
    else:
      self._engine.set_goals(goals, env_ids)
    self._resets += 1

  def evaluate(self, states, goals=None):
    """Relabels env records: (reward float64, success uint8, status uint8) device tensors (n,),
    the task's value on each record of `states` (EnvStates) at its live positions -- without the
    step's action cost -- with goals[i] (float64 (n, G, 2) on the engine's device) in place of
    record i's goals, or the records' own goals if `goals` is None.  One launch on the current
    stream, no host synchronisation; no env, ring or `rng` changes."""
    return self._engine.evaluate(states, goals)

  def sample_contained_positions(self, seed, n_samples=None, states=None):
    """Positions inside sprites for random agents and plan proposals, drawn on the device: what
    Environment.sample_contained_position() draws for one env -- a sprite chosen uniformly (not by
    area), then a point of it by rejection from its bounding box -- for every env, or for every
    record of EnvStates `states`.  Returns ContainedPositions(position float64, slot int8, status
    uint8) of new device tensors: shapes (n, 2), (n,), (n,) with n_samples=None, ready for
    actions[:, :2], or (n, n_samples, 2), (n, n_samples), (n, n_samples) for an int; sample 0 of
    those equals the n_samples=None call.  slot indexes the slot axis of SpriteFactors and
    SpriteMasks.  A row without sprites gives status ENV_NO_SPRITE, a sprite no draw lands in (scale
    0) ENV_SAMPLE_TRIES, each with position NaN and slot -1.

    Each sample is a pure function of (seed, row, sample index, the row's state), from the
    device's own Philox stream: nothing is drawn from `rng` and nothing is kept, so there is nothing
    to checkpoint.  Envs sample the scene they are on, also an env about to reset (whose next step
    replaces it).  A float64 SelectMove / DragAndDrop action clicking `position` grabs `slot` or a
    sprite above it; with the action space's noise_scale, step() adds noise to the click first, and
    the grab is no longer certain.  One launch on the current stream, read-only (no env, ring, frame
    or refill state changes) and without host synchronisation."""
    position, slot, status = self._engine.sample_contained(seed, 1 if n_samples is None else n_samples, states)
    if n_samples is None:
      return ContainedPositions(position[:, 0], slot[:, 0], status[:, 0])
    return ContainedPositions(position, slot, status)

  def _record_factor_tensors(self, factors, states):
    if not isinstance(states, engine_lib.EnvStates):
      raise ValueError('states must be EnvStates, got %s' % type(states).__name__)
    self._engine.check_states(states, len(states))
    fields, dev = states.fields(), states.data.device
    table = getattr(self, '_shape_ids', None)
    if table is None or table.device != dev:
      table = self._shape_ids = torch.from_numpy(engine_lib.shape_id_table(constants.SHAPES)).to(dev)
    shape = table[fields['shape'].long()]
    out = collections.OrderedDict()
    for name in factors:
      if name in ('x', 'y'):
        out[name] = fields['pos_' + name].to(torch.float32)
      elif name in ('x_vel', 'y_vel'):
        out[name] = fields['v' + name[0]].to(torch.float32)
      elif name == 'shape':
        out[name] = shape.to(torch.float32)
      else:
        out[name] = fields['factors'][:, self._FACTOR_COLUMNS[name]].clone()
    out['mask'] = shape > 0
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
    layout, goals = self._sample(len(env_ids), rng)
    self._upload(layout, env_ids, absolute % self._K, goals=goals)
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
            layout, goals = self._sample(len(plan[0]), self._block_rngs[i])
            self._upload(layout, plan[0], plan[1] % K, goals=goals)
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
    if self._refill_mode == 'device':
      if self._t - self._safe_step >= self._period or self._risk(self._t + 1) > K - 1:
        self._engine.refill_device()
        self._stats['refills'] += 1
        self._safe_step, self._safe_resets = self._t, self._resets
      return
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
    if self._refill_mode == 'device':
      return dict(mode='device', launches=self._stats['refills'], pool_depth=self._K, seed=self.seed)
    return dict(self._stats, mode=self._refill_mode, pool_depth=self._K,
                threads=len(getattr(self, '_block_rngs', [None])),
                procs=len(self._pool) if getattr(self, '_pool', None) is not None else 0)

  # -- API ---------------------------------------------------------------------------------
  @property
  def engine(self):
    return self._engine

  def _to_device(self, actions):
    """Host actions through engine.host_actions; tensors are moved, not converted."""
    dev = self._engine.device
    kind = self._action_space.compile()['kind']
    if not isinstance(actions, torch.Tensor):
      actions = torch.from_numpy(engine_lib.host_actions(kind, actions))
    t = actions.to(dev)
    noise_scale = getattr(self._action_space, '_noise_scale', None)
    if noise_scale and kind != 'embodied':
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
    return self.step(engine_lib.zero_actions(self._action_space.compile()['kind'], self.n_envs))

  # -- env records -------------------------------------------------------------------------
  # On the step stream, after everything enqueued so far.  A record holds an env's current scene
  # and episode counters, not its place in the scene ring: a loaded env plays the saved episode
  # out, then starts the next scene of its own ring.  A record with reset_next = 1 starts that
  # scene on the next step, as reset() does, so every load or copy counts as a reset against the
  # ring's underflow guard (_risk): with loads before every step the ring is refilled more often
  # rather than an env running onto a ring slot that has not been refilled.
  # Ids: lists, ndarrays or tensors (a CUDA tensor costs a device-to-host copy), or with
  # check='device' int32 / int64 tensors on the engine's device, checked there without a wait
  # (Engine.check_env_ids reports a refused call).  A device-checked load or copy counts as a
  # reset whether or not the device refuses it.
  def save_envs(self, env_ids=None, check='host'):
    """engine.EnvStates of envs `env_ids` (default: all, in order)."""
    if engine_lib.device_checked(check, env_ids):
      return self._engine.save_envs(env_ids, check='device')
    return self._engine.save_envs(env_ids)

  def load_envs(self, states, env_ids=None, check='host'):
    """Env env_ids[i] <- record i of `states` (default ids: all envs, in order)."""
    if engine_lib.device_checked(check, env_ids):
      self._engine.load_envs(states, env_ids, check='device')
    else:
      self._engine.load_envs(states, env_ids)
    self._resets += 1

  def copy_envs(self, src_ids, dst_ids, check='host'):
    """Env dst_ids[i] <- env src_ids[i]; every read sees the state from before the call."""
    if engine_lib.device_checked(check, src_ids):
      self._engine.copy_envs(src_ids, dst_ids, check='device')
    else:
      self._engine.copy_envs(src_ids, dst_ids)
    self._resets += 1

  def make_states(self, factors, goals=None, step_count=None, span_class=None):
    """Env records of scenes the caller chose: (EnvStates, status uint8 (n,)), made on the device
    from factor tensors, for datasets from factor samples, interventions on one factor of one
    sprite, fixed evaluation suites (load_envs) and rendering predicted factors.

    `factors`: dict keyed by a subset of sprite.FACTOR_NAMES.  'shape' (n, n_slots) is required:
    constants.ShapeType ids, 0 for an empty slot, in any of the dtypes below (the float32 'shape' of
    factor_tensors goes straight back in).  Every other value broadcasts to (n, n_slots).  All are
    tensors on the engine's device of dtype float32, float64, int8, int16, int32, int64 or uint8; an
    omitted factor is Sprite's default (x = y = 0.5, angle 0, scale 0.1, colours 0, velocities 0.0).
    Under color_maps.hsv_to_rgb c0, c1 and c2 are all float32, all float64 or all omitted.  `goals`:
    float64 (n, G, 2), required when the task samples goals (G > 0) and refused otherwise.
    `step_count`: int32 (n,), default zeros.

    Record i is, byte for byte, what save_envs saves of an env that has just taken the reset (FIRST)
    step of an episode -- with step_count[i] in place of 0 -- whose scene is
    [Sprite(**factors at (i, j)) for the occupied slots j, in slot order], packed with this
    environment's task filters and colour map, and whose goals are goals[i].  A scene of k sprites
    fills slots n_slots - k .. n_slots - 1.  status[i] holds the scene_program.MAKE_* bits of a
    refused record, which is written as zeros (an env with only empty slots): MAKE_ANGLE, an
    occupied slot's angle is not an integer in [-360, 360]; MAKE_SHAPE, a shape value is not an
    integer in 0 .. 12; MAKE_HOLE, an empty slot after an occupied one; MAKE_INT, an occupied slot's
    integer factor of magnitude above 2^53; MAKE_STEP, step_count < 0.

    `span_class` (1 or 4) is the records' span class.  None reads one device flag back -- the call's
    only host synchronisation -- and gives 4 if a record holds a star or spoke, else the engine's.
    A caller who passes it avoids the read; stars made under class 1 render with ENV_SPAN_OVERFLOW
    set, never as a wrong frame.

    One launch on the current stream (the first call also uploads the packer, synchronising once).
    Read-only: no env, scene ring, frame buffer or `rng` changes, and nothing counts against the
    ring's refill.  A colour map other than None and hsv_to_rgb raises NotImplementedError."""
    if getattr(self, '_packer', None) is None:
      from spriteworld_b200 import scene_program
      packer = scene_program.compile_packer(self._filters, self._color_to_rgb)
      self._engine.load_packer(packer)
      self._packer = packer
    return self._engine.make_states(factors, goals, step_count, span_class)

  def rollout(self, actions, states=None):
    """Scores C candidate action sequences of T steps per env from the state every env is in now,
    in one kernel launch, and leaves every env as it is: no position, counter, scene ring or
    frame changes, so nothing here counts against the ring's refill.  With `states` (EnvStates of
    n roots saved by an environment of this configuration) the plans start from those records
    instead, and actions and outputs are (T, n, C, ...).

    `actions`: (T, n_envs, C, 4) float32 / float64 or (T, n_envs, C, 2) int32, array or tensor, as
    step() takes them per env.  Returns a BatchedRollout of (T, n_envs, C) device tensors the
    caller owns.  Entry [t, e, c] is, bit for bit, what step(actions[t, :, c]) would report for env
    e after the steps before it: step_type int8, reward float64, success and status uint8, and
    discount float32 (1 on MID, 0 on LAST and on padding).  A plan ends with its first LAST (the
    task solved, a sprite out of frame, or max_episode_length counted from the env's own step
    count); the entries after it are padding -- step_type _native.STEP_NONE, reward 0 -- so
    reward.sum(0) is each plan's return.  An env that is about to reset (before the first reset(),
    or after a LAST) has no episode to plan in: all its entries are padding.

    A rollout evaluates the noiseless model: the action space's `noise_scale` is not applied and
    nothing is drawn from `rng`, so the timesteps of a run are bit-identical with and without
    rollouts between its steps."""
    if states is None:
      return self._batched_rollout(self._engine.rollout(self._plans(actions)))
    return self._batched_rollout(self._engine.rollout(self._plans(actions), states=states))

  def expand(self, actions, states=None):
    """One level of a search tree: rollout(actions, states) that also returns the state every plan
    ends in, as (BatchedRollout, EnvStates).  Leaf r * C + c is root r's plan c (the roots are the
    live envs without `states`): what save_envs would return after loading the root and stepping
    the plan's live steps -- its final positions and step count, and reset_next = 1 if the plan
    ended on a LAST, so that a leaf's own rollouts are all padding.  Leaves go back in as `states`
    (narrowed with EnvStates.take, say), with nothing on the host between levels.

    As rollout(): no noise, no `rng` draw, and no env or scene ring changes; loading a leaf later
    (load_envs) counts as a reset, as every load does."""
    res = self._engine.rollout(self._plans(actions), states=states, leaves=True)
    return self._batched_rollout(res), res.leaves

  def rollout_trajectory(self, actions, states=None):
    """rollout(actions, states) that also returns the state after every step of every plan, as
    (BatchedRollout, EnvStates) of T * n * C records, in one launch.  Record (t * n + r) * C + c is
    the leaf expand(actions[:t + 1], states) returns for root r's plan c: after a plan's first LAST
    every record repeats its end state, a root about to reset is its own record at every t, and the
    last n * C records are expand's leaves.  observe(trajectory) then gives every step's
    observations; reshape them to (T, n, C, ...).

    As rollout(): no noise, no `rng` draw, and no env or scene ring changes.  The records take
    T * n * C * engine.record_bytes bytes: to trace a few plans out of many, roll out first, pick
    the plans, and trace those from the roots they start in (states.take)."""
    res = self._engine.rollout(self._plans(actions), states=states, trajectory=True)
    return self._batched_rollout(res), res.trajectory

  def _plans(self, actions):
    """Rollout actions as a contiguous tensor on the engine's device (host actions through
    engine.host_actions), without noise."""
    kind = self._action_space.compile()['kind']
    if not isinstance(actions, torch.Tensor):
      actions = torch.from_numpy(engine_lib.host_actions(kind, actions))
    return actions.to(self._engine.device).contiguous()

  @staticmethod
  def _batched_rollout(res):
    discount = (res.step_type == _native.STEP_MID).to(torch.float32)
    return BatchedRollout(res.step_type, res.reward, discount, res.success, res.status)

  def render(self):
    """Re-renders every PILRenderer, SpriteMasks, SpriteCoverage, SoftSpriteMasks and SpriteBoxes
    observation of the current state (a loaded one, say) into this environment's buffers, and
    returns them: dict name -> uint8 (n_envs, H, W, 3) frames, then uint8 (n_envs, H, W) masks,
    coverage dicts, uint8 (n_envs, n_slots, H, W) soft masks, box dicts and uint8
    (n_envs, V, H, W, 3) SpriteGlimpses and SpriteLayers views, in renderer order."""
    out = collections.OrderedDict()
    for name, r in self._rasters.items():
      out[name] = self._engine.render(r, self._frames[name])
    for name, r in self._other.items():
      if isinstance(r, handcrafted._SpriteMaskRenderer):
        out[name] = self._render_sprite_masks(type(r), r)
      elif isinstance(r, glimpses._SpriteViews):
        out[name] = self._render_views(r)
    return out

  def render_windows(self, windows, renderer, states=None, draw=None):
    """The scene seen through windows (Engine.render_windows) on the current stream: (frames uint8
    (n, V, H, W, 3), status uint8 (n, V)) for a float64 (n, V, 4) device tensor of windows
    (x0, y0, x1, y1), each drawn as `renderer` (a PILRenderer, SpriteGlimpses or SpriteLayers whose
    colour map is this environment's) draws its frame, with the window stretched over the whole
    raster.  Rows are the live envs (n = n_envs), or with `states` EnvStates of any n records, as if
    loaded.  Status holds ENV_BAD_WINDOW (an empty or non-finite window, or a vertex 2^30 canvas
    pixels or more away; the frame is zeros) and ENV_SPAN_OVERFLOW.  New tensors; one launch,
    read-only.

    `draw`: a bool tensor on this environment's device that broadcasts to (n, V, n_slots); view
    (i, v) then draws only the slots s with draw[i, v, s], as if the others were empty (the scene
    without sprite k, a sprite without its occluders), and its status counts those slots only.
    None draws every slot."""
    if not isinstance(renderer, (pil_renderer.PILRenderer, glimpses._SpriteViews)):
      raise ValueError('renderer must be a PILRenderer or SpriteGlimpses or SpriteLayers, got %s'
                       % type(renderer).__name__)
    if renderer.color_to_rgb is not self._color_to_rgb:
      raise ValueError("renderer's color_to_rgb is not this environment's: colours are packed at upload")
    if draw is not None:
      draw = self._broadcast_draw(draw, windows)
    return self._engine.render_windows(self._window_raster(renderer), windows, states, draw=draw)

  def _broadcast_draw(self, draw, windows):
    """`draw` broadcast to (n, V, n_slots) for windows (n, V, 4), contiguous on the device.  A
    `windows` that is not (n, V, 4) is left to Engine.render_windows to refuse."""
    eng = self._engine
    if not isinstance(draw, torch.Tensor) or draw.dtype != torch.bool or draw.device != eng.device:
      raise ValueError('draw must be a bool tensor on %s, got %s' % (eng.device, engine_lib._describe(draw)))
    if not isinstance(windows, torch.Tensor) or windows.dim() != 3:
      return draw
    shape = (int(windows.shape[0]), int(windows.shape[1]), eng.n_slots)
    try:
      ok = torch.broadcast_shapes(draw.shape, shape) == shape
    except RuntimeError:
      ok = False
    if not ok:
      raise ValueError('draw must broadcast to (n, V, n_slots) = %s, got %s' % (shape, engine_lib._describe(draw)))
    return draw.expand(shape).contiguous()

  def _window_raster(self, renderer):
    """The Raster of render_windows for `renderer`'s size, anti_aliasing and background."""
    key = (renderer.width, renderer.height, renderer.anti_aliasing, tuple(renderer.bg_color))
    r = self._window_rasters.get(key)
    if r is None:
      r = self._window_rasters[key] = engine_lib.Raster(self._engine, *key)
    return r

  def _render_views(self, renderer, states=None, status=None):
    """SpriteGlimpses or SpriteLayers `renderer`'s views on the current stream: of the live envs
    into this environment's buffers for the renderer (new tensors for one it does not own), or of
    EnvStates `states` into a new tensor.  `status` (uint8 (n,)), if given, is ORed in place with
    each row's view status (ENV_BAD_WINDOW, ENV_SPAN_OVERFLOW)."""
    pos = self._engine.state_tensors() if states is None else states.fields()
    frames, st = self._glimpse_buffers.get(id(renderer), (None, None)) if states is None else (None, None)
    windows, draw = renderer.views(pos['pos_x'], pos['pos_y'])
    frames, st = self._engine.render_windows(self._window_raster(renderer), windows, states, frames, st, draw)
    if status is not None:
      status.bitwise_or_(st.amax(1))
    return frames

  def _render_sprite_masks(self, cls, renderer, states=None):
    """`renderer`'s observation as a `cls` (SpriteMasks, SpriteCoverage, SoftSpriteMasks or
    SpriteBoxes) on the current stream: of the live envs into this environment's buffers for the
    renderer (new tensors for a renderer it does not own), or of EnvStates `states` into new
    tensors."""
    # only a renderer of this kind has buffers of this kind's form
    out = self._mask_buffers.get(id(renderer)) if states is None and isinstance(renderer, cls) else None
    return cls._observation(engine_lib._render_sprite_masks(
        self._engine, cls._kind, renderer.width, renderer.height, renderer.anti_aliasing, states=states, out=out))

  def render_masks(self, renderer, states=None):
    """SpriteMasks `renderer`'s masks (Engine.render_masks) on the current stream: of the live envs
    into this environment's buffer for the renderer (a new tensor for a renderer it does not own),
    or of EnvStates `states` into a new uint8 (n, H, W) tensor."""
    return self._render_sprite_masks(handcrafted.SpriteMasks, renderer, states)

  def render_coverage(self, renderer, states=None):
    """SpriteCoverage `renderer`'s observation (Engine.render_coverage) on the current stream: dict
    'cover' int32 (n, H, W), 'visible' and 'area' int32 (n, n_slots).  Of the live envs into this
    environment's buffers for the renderer (new tensors for a renderer it does not own), or of
    EnvStates `states` into new tensors."""
    return self._render_sprite_masks(handcrafted.SpriteCoverage, renderer, states)

  def render_soft_masks(self, renderer, states=None):
    """SoftSpriteMasks `renderer`'s soft masks (Engine.render_soft_masks) on the current stream: of
    the live envs into this environment's buffer for the renderer (a new tensor for a renderer it
    does not own), or of EnvStates `states` into a new uint8 (n, n_slots, H, W) tensor."""
    return self._render_sprite_masks(handcrafted.SoftSpriteMasks, renderer, states)

  def render_boxes(self, renderer, states=None):
    """SpriteBoxes `renderer`'s observation (Engine.render_boxes) on the current stream: dict
    'visible_box' and 'amodal_box' int32 (n, n_slots, 4), 'visible' and 'area' int32 (n, n_slots).
    Of the live envs into this environment's buffers for the renderer (new tensors for a renderer
    it does not own), or of EnvStates `states` into new tensors."""
    return self._render_sprite_masks(handcrafted.SpriteBoxes, renderer, states)

  def observe(self, states):
    """The observations of env records without loading them: (observation, status) for EnvStates
    `states` of n records, observation an OrderedDict in renderer order of what step() would
    observe for envs that load_envs(states) had loaded -- PILRenderer frames as new uint8
    (n, H, W, 3) tensors (one render launch per raster; never this environment's own frame
    buffers), SpriteFactors dicts of (n, n_slots) tensors, SpriteMasks, SpriteCoverage and
    SoftSpriteMasks observations in new tensors (one launch each), SpriteBoxes observations in new
    tensors (two launches each), SpriteGlimpses and SpriteLayers views as new uint8
    (n, V, H, W, 3) tensors -- and status uint8 (n,), the OR over the rasters of their render status
    (_native.ENV_SPAN_OVERFLOW) and over the views of theirs (also _native.ENV_BAD_WINDOW).

    Enqueued on the current stream without a host synchronisation.  Read-only: no env, scene ring,
    frame buffer or `rng` changes, and nothing counts against the ring's refill.  A renderer
    without a record form (Success: success is a task evaluation, which rollout and expand
    report) raises NotImplementedError before anything is enqueued."""
    missing = [name for name, r in self._other.items() if not hasattr(r, 'render_states')]
    if missing:
      raise NotImplementedError('renderers %s have no record form: observe() cannot render them' % missing)
    eng = self._engine
    eng.check_states(states, len(states))
    status, obs = None, collections.OrderedDict()
    for name in self._renderers:
      if name in self._rasters:
        frames, st = eng.render_states(self._rasters[name], states)
        obs[name] = frames
        status = st if status is None else status.bitwise_or_(st)
      elif name in self._views:
        if status is None:
          status = torch.zeros(len(states), dtype=torch.uint8, device=eng.device)
        obs[name] = self._render_views(self._views[name], states, status)
      else:
        obs[name] = self._other[name].render_states(self, states)
    if status is None:
      status = torch.zeros(len(states), dtype=torch.uint8, device=eng.device)
    return obs, status

  # -- checkpoints -------------------------------------------------------------------------
  def state_dict(self):
    """A checkpoint of the whole run, to resume it exactly (load_state_dict), across episode
    boundaries: the engine's state (Engine.save_state: live sprites, counters, every scene ring,
    the device sampler's bookkeeping), the host's refill bookkeeping and underflow guard, the
    state of `rng` (action noise, the sync refill's scenes) and of every asynchronous refill
    block's RandomState, and the device sampler's seed and env_offset, with a fingerprint of the
    environment's configuration.  Only tensors, Python scalars, strings, bytes, tuples, lists and
    dicts: torch.save writes it and torch.load with weights_only=True reads it back.

    Lands an asynchronous refill in flight first (and so may wait for it), so that the rings match
    the bookkeeping, and restarts the schedule of scene_serial snapshots (pending snapshots are not
    state; load_state_dict restarts it the same way).  Synchronises the current stream.

    Not carried over: unreported device sampler failures and refused device-checked id reports --
    call check_sampler() / engine.check_env_ids() first to have those raised -- and the frame
    buffers of the last step (render() recomputes them from the state).  With the default `rng`
    (the np.random module) the state saved is NumPy's global one.  A host-sampler fingerprint
    cannot cover `init_sprites`, a Python callable: resuming with another generator is not
    detected."""
    if self._refill_mode == 'async':
      self._land(block=True)
      self._restart_snapshots()
    host = dict(t=self._t, resets=self._resets, safe_step=self._safe_step, safe_resets=self._safe_resets,
                stats=dict(self._stats))
    if self._sampler == 'host':
      host['refilled_upto'] = torch.from_numpy(self._refilled_upto.copy())
    return dict(
        fingerprint=self._fingerprint(), engine=self._engine.save_state(), host=host,
        rng=_rng_state(self._rng), block_rngs=[_rng_state(r) for r in getattr(self, '_block_rngs', ())],
        sampler=(self.seed, self._env_offset) if self._sampler == 'device' else None)

  def load_state_dict(self, sd):
    """Resumes the run a state_dict() was taken of, in an environment constructed with the same
    arguments (a fresh one, in another process or on another device index too, or this one: a
    rewind).  Afterwards steps with the same actions give, bit for bit, what the saved run gave
    after the checkpoint -- with sampler='device' or refill='sync' for as many episodes as are
    stepped; with refill='async' while every env is on a scene its ring held at the checkpoint,
    since refill timing decides which env gets which newly drawn scene -- and render(),
    factor_tensors(), rollout(), expand(), observe() and save_envs() give what they gave at the
    checkpoint.

    Raises ValueError naming the first difference of configuration before anything changes.  Then
    lands this environment's own refill in flight, reloads the device sampler if its seed or
    env_offset differ, loads the engine and restores the host bookkeeping and the RNG states
    (NumPy's global state with the default `rng`)."""
    fp, got = self._fingerprint(), sd.get('fingerprint') if isinstance(sd, dict) else None
    if not isinstance(got, dict):
      raise ValueError('not a BatchedEnvironment state_dict')
    for key, mine in fp.items():
      if got.get(key) != mine:
        shown = ((got.get(key), mine) if not isinstance(mine, bytes) else ('other bytes', 'its own'))
        raise ValueError('state_dict was taken of another configuration: %s is %r there, %r here'
                         % ((key,) + shown))
    if self._refill_mode == 'async':
      self._land(block=True)       # no upload of this env's may land on the loaded pool
    eng = self._engine
    if self._sampler == 'device' and tuple(sd['sampler']) != (self.seed, self._env_offset):
      seed, env_offset = (int(v) for v in sd['sampler'])
      backup = eng.save_state()
      eng.load_sampler(self._program, seed, env_offset)
      try:
        eng.load_state(sd['engine'])
      except Exception:
        eng.load_sampler(self._program, self.seed, self._env_offset)
        eng.load_state(backup)
        raise
      self.seed, self._env_offset = seed, env_offset
    else:
      eng.load_state(sd['engine'])
    host = sd['host']
    self._t, self._resets = int(host['t']), int(host['resets'])
    self._safe_step, self._safe_resets = int(host['safe_step']), int(host['safe_resets'])
    self._stats = dict(host['stats'])
    if self._sampler == 'host':
      self._refilled_upto[:] = host['refilled_upto'].numpy()
    _set_rng_state(self._rng, sd['rng'])
    for r, st in zip(getattr(self, '_block_rngs', ()), sd['block_rngs']):
      _set_rng_state(r, st)
    if self._refill_mode == 'async':
      self._restart_snapshots()

  def _restart_snapshots(self):
    """Drops the pending scene_serial snapshots; the next step takes a fresh one."""
    self._snaps.clear()
    self._last_snap = -(1 << 30)

  def _fingerprint(self):
    """What load_state_dict compares: everything that decides how the saved state steps."""
    fp = dict(n_envs=self.n_envs, pool_depth=self._K, n_slots=self._engine.n_slots,
              signature=bytes(self._engine.signature), sampler=self._sampler, refill=self._refill_mode,
              refill_blocks=len(getattr(self, '_block_rngs', ())),
              refill_procs=len(self._pool) if getattr(self, '_pool', None) is not None else 0,
              renderers=list(self._renderers),
              rasters=[(name, int(r.width), int(r.height), int(r.anti_aliasing),
                        tuple(int(c) for c in r.bg_color)) for name, r in self._pil.items()])
    if self._sampler == 'device':
      fp['program'] = bytes(self._program.struct)
    if self._goal_distribs:
      fp['goals'] = [str(d) for d in self._goal_distribs]
    return fp

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
    for r in list(self._rasters.values()) + list(self._window_rasters.values()):
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
    if any(isinstance(r, handcrafted.GoalPositions) for r in dict(config.get('renderers') or {}).values()):
      raise NotImplementedError('ShardedBatchedEnvironment does not gather GoalPositions across ranks; '
                                "each rank's goals are self.local.goal_tensor()")
    for cls in (glimpses.SpriteGlimpses, glimpses.SpriteLayers):
      if any(isinstance(r, cls) for r in dict(config.get('renderers') or {}).values()):
        raise NotImplementedError('ShardedBatchedEnvironment does not gather %s across ranks; '
                                  "each rank's are in self.local's observations" % cls.__name__)
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
    if config.get('sampler', 'host') == 'device':
      # scenes are functions of (seed, global env id): every rank takes the common seed and the
      # global id of its first env, so the run draws what a one-GPU run over all envs draws
      config = dict(config, env_offset=self.env_start)
      if config.get('seed') is None:
        config['seed'] = int(seed)
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
    reward, step_type, success, status = engine_lib.split_outputs(self._out_all.view(W, -1), E)
    discount = (step_type != _native.STEP_LAST).to(torch.float32)
    obs = collections.OrderedDict([(self._image, res.frames)])
    return BatchedTimeStep(step_type, reward, discount, obs, success, status)

  def reset(self):
    env = self.local
    env._resets += 1
    env.engine.request_reset()
    return self.step(engine_lib.zero_actions(env._action_space.compile()['kind'], self.n_local))

  def state_dict(self):
    """This rank's checkpoint: the local BatchedEnvironment.state_dict() with the sharding it
    belongs to.  Every rank saves and loads its own (at the same step); loading into another
    sharding -- another rank, world size or env count -- is refused."""
    return dict(rank=self.rank, world=self.world, n_envs_total=self.n_envs_total, env_start=self.env_start,
                t=self._t, local=self.local.state_dict())

  def load_state_dict(self, sd):
    """Resumes this rank from its own state_dict() (see BatchedEnvironment.load_state_dict)."""
    for key in ('rank', 'world', 'n_envs_total', 'env_start'):
      if sd.get(key) != getattr(self, key):
        raise ValueError('state_dict was taken of another sharding: %s is %r there, %r here'
                         % (key, sd.get(key), getattr(self, key)))
    self.local.load_state_dict(sd['local'])
    self._t = int(sd['t'])

  def observation_spec(self):
    return self.local.observation_spec()

  def action_spec(self):
    return self.local.action_spec()

  def close(self):
    if self.local.engine.device.type == 'cuda':
      torch.cuda.synchronize(self.local.engine.device)
    self._peer.close()
    self.local.close()
