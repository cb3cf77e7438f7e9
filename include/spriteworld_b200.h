/*
 * spriteworld_b200 -- C-ABI of the H100-native batched Spriteworld step+render engine.
 *
 * The reference (google-deepmind/spriteworld) has no FFI: its boundary for this path is
 * three duck-typed Python protocols called from Environment.step
 * (spriteworld/environment.py:88-108):
 *     action_space.step(action, sprites, keep_in_frame)   action_spaces.py:83-104, 187-214
 *     task.reward(sprites) / task.success(sprites)        tasks.py:140-158, 217-245, 288-296
 *     renderer.render(sprites, global_state)              renderers/pil_renderer.py:67-91
 * This header is what a ctypes/cffi binding of that path binds instead (see
 * INTEGRATION.md): plain pointers and sizes, no torch types, int return codes
 * (0 = ok) with the message available from swb_last_error().
 *
 * Ownership: the caller owns action / output / frame buffers (device pointers unless a
 * function says "host"); the engine owns the sprite state (struct-of-arrays), the scene
 * pool, per-env counters and all scratch.  One engine per GPU; not thread-safe per
 * engine; all work is enqueued on the caller's stream (a cudaStream_t passed as void*).
 *
 * A call its checks refuse -- bad arguments, or a raster that cannot launch -- has enqueued
 * nothing: no kernel, no copy, no change to swb_launch_count.  (A CUDA runtime error raised after
 * work was enqueued can leave part of a call done.)
 */
#ifndef SPRITEWORLD_B200_H_
#define SPRITEWORLD_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SWB_MAX_VERTS 32    /* largest shape: 30-gon "circle" (constants.py:33) */
#define SWB_NUM_SHAPES 13   /* ShapeType 1..12 (constants.py:43-56); 0 = empty slot */
#define SWB_MAX_CHILDREN 16
#define SWB_MAX_NODES 32
#define SWB_MAX_SLOTS 32    /* sprites per env */
#define SWB_MAX_FILTERS 32  /* distinct task filter distributions (bits of `member`) */
#define SWB_MAX_GOALS 8     /* sampled FindGoalPosition goals per task tree (goal slots) */
#define SWB_MAX_PEERS 8     /* ranks whose frame buffers one render launch can write */
#define SWB_IPC_HANDLE_BYTES 64

/* action spaces (action_spaces.py) */
enum { SWB_ACT_SELECT_MOVE = 0, SWB_ACT_DRAG_AND_DROP = 1, SWB_ACT_EMBODIED = 2 };
/* action dtypes accepted by swb_step: SelectMove/DragAndDrop take [E][4] f32 or f64
 * (action_spaces.py:62-63,106-108); Embodied takes [E][2] int32 (carry, direction).
 * Device id lists of the swb_*_envs_dev calls are SWB_DTYPE_I32 or SWB_DTYPE_I64. */
enum { SWB_DTYPE_F32 = 0, SWB_DTYPE_F64 = 1, SWB_DTYPE_I32 = 2, SWB_DTYPE_I64 = 3 };
/* tasks (tasks.py) */
enum { SWB_TASK_NO_REWARD = 0, SWB_TASK_FIND_GOAL = 1, SWB_TASK_CLUSTERING = 2, SWB_TASK_META = 3 };
enum { SWB_AGG_SUM = 0, SWB_AGG_MAX = 1, SWB_AGG_MIN = 2, SWB_AGG_MEAN = 3 };
enum { SWB_CRIT_ALL = 0, SWB_CRIT_ANY = 1 };
/* dm_env.StepType; SWB_STEP_NONE: no step (the padding of swb_rollout) */
enum { SWB_STEP_NONE = -1, SWB_STEP_FIRST = 0, SWB_STEP_MID = 1, SWB_STEP_LAST = 2 };
/* per-env status written to swb_step_out.status (the reference raises instead) */
enum {
  SWB_ENV_OK = 0,
  SWB_ENV_CLUSTER_LABELS = 1,  /* sklearn ValueError: needs 2 <= n_labels <= n_samples-1 */
  SWB_ENV_CLUSTER_ZERODIV = 2, /* davies_bouldin_score == 0 -> 1./0. (tasks.py:215) */
  SWB_ENV_BAD_ACTION = 4,      /* Embodied direction not in 0..3 -> KeyError (action_spaces.py:203) */
  SWB_ENV_SPAN_OVERFLOW = 8,   /* renderer: more spans on a canvas row than the engine was sized for */
  SWB_ENV_NO_SPRITE = 16,      /* swb_sample_contained: the row has no sprite (np.random.randint(0) raises) */
  SWB_ENV_SAMPLE_TRIES = 32,   /* swb_sample_contained: SWB_CONTAINED_MAX_TRIES draws, none inside (sprite.py) */
  SWB_ENV_BAD_WINDOW = 64      /* swb_render_windows: empty or non-finite window, or a vertex at 2^30 or beyond */
};

/* One node of the flattened task tree, post-order, root last. */
typedef struct {
  int32_t kind;
  /* FindGoalPosition (tasks.py:87-113) */
  int32_t filter_slot; /* bit index into `member`; -1: filter_distrib is None */
  double goal[2];
  double weights[2];
  double terminate_distance;
  double terminate_bonus; /* also Clustering / MetaAggregated */
  double raw_reward_multiplier;
  int32_t sparse_reward; /* also Clustering */
  /* Clustering (tasks.py:164-194) */
  int32_t n_clusters;
  int32_t cluster_slots[SWB_MAX_CHILDREN];
  double termination_threshold;
  double reward_range;
  /* MetaAggregated (tasks.py:258-286) */
  int32_t n_children;
  int32_t children[SWB_MAX_CHILDREN]; /* node indices < this node's index */
  int32_t aggregator;
  int32_t criterion;
  /* FindGoalPosition: -1 = the constant `goal`; g in [0, SWB_MAX_GOALS) = the goal drawn with the
   * env's scene, goal slot g of the pool entry the env is on.  The engine's G (goals per scene) is
   * the largest slot + 1; slots 0 .. G-1 must each belong to exactly one node.  Added in version 11
   * in the struct's tail padding (its size did not change): bindings check swb_version() >= 11, and
   * a zero-filled FIND_GOAL node is a sampled goal, whose engine then refuses scene uploads without
   * swb_scene_soa.goal. */
  int32_t goal_slot;
} swb_task_node;

typedef struct {
  int32_t device;     /* CUDA device ordinal */
  int32_t n_envs;     /* E */
  int32_t n_slots;    /* S: sprite slots per env; slot S-1 is the top-most / Embodied body */
  int32_t pool_depth; /* K: pre-sampled scenes per env (ring) */
  /* action space */
  int32_t action_kind;
  double action_scale; /* SelectMove/DragAndDrop `scale`, Embodied `step_size` */
  double motion_cost;
  /* Environment (environment.py:34-70) */
  int32_t keep_in_frame;
  int32_t max_episode_length;
  /* task tree */
  int32_t n_nodes;
  swb_task_node nodes[SWB_MAX_NODES];
  /* unit-area vertex tables generated by the caller with the reference's NumPy
   * expressions (shapes.py:34-116 via constants.py:27-40) */
  int32_t shape_n_verts[SWB_NUM_SHAPES];
  double shape_verts[SWB_NUM_SHAPES][SWB_MAX_VERTS][2];
} swb_config;

/*
 * Host-side struct-of-arrays view of `n` scenes x S slots, index = scene * S + slot.
 * A scene is what one init_sprites() call returned (environment.py:75), already reduced
 * to what the step path needs.  Slots are ordered back to front; pad EMPTY slots
 * (shape 0) at the front.
 */
typedef struct {
  const double *x, *y;                   /* initial position (float32-valued iff pos_f32) */
  const double *m00, *m01, *m10, *m11;   /* centred-path transform: scale then rotate (sprite.py:96-101) */
  const double *vx, *vy;                 /* velocity (sprite.py:92) */
  const uint32_t *member;                /* bit i: filter distribution i contains the sprite */
  const uint8_t *shape;                  /* ShapeType, 0 = empty slot */
  const uint8_t *pos_f32;                /* 1: the reference's position ndarray is float32 */
  const uint8_t *rgb;                    /* [n*S*3] color_to_rgb(sprite.color) (pil_renderer.py:82) */
  const float *factors;                  /* optional [n*S*5]: scale, angle, c0, c1, c2 for factor observations */
  const double *goal;                    /* [n*G*2]: (x, y) of every goal slot of scene i at (i*G + g)*2;
                                            required when the engine has G > 0 goal slots, else ignored */
} swb_scene_soa;

/* Per-step outputs, device pointers, one element per env (swb_rollout: per step, env and candidate). */
typedef struct {
  double *reward;      /* action cost + task.reward (environment.py:101); 0 on FIRST */
  int8_t *step_type;   /* SWB_STEP_* */
  uint8_t *success;    /* task.success(sprites) (environment.py:80-81) */
  uint8_t *status;     /* SWB_ENV_* bits */
} swb_step_out;

typedef struct swb_engine swb_engine;
typedef struct swb_raster swb_raster;

const char *swb_last_error(void);
int swb_version(void);
/* sizeof(swb_config) / sizeof(swb_task_node) as compiled, for bindings to check their mirror structs */
int swb_sizeof_config(void);
int swb_sizeof_task_node(void);

int swb_engine_create(const swb_config *cfg, swb_engine **out);
void swb_engine_destroy(swb_engine *eng);

/*
 * Uploads `n` scenes into the pool.  scene i goes to env `env_ids[i]`, ring slot
 * `ring_slots[i]`.  Host pointers, free to reuse when the call returns: the arrays are packed
 * into a pinned staging block of the engine (two alternate), which one asynchronous copy and one
 * scatter kernel on `stream` move into the pool.  The call does not wait for the device; work
 * enqueued on `stream` afterwards sees the scenes, other streams need an event.
 * (reset(): init_sprites() on the host, environment.py:74-78)
 */
int swb_upload_scenes(swb_engine *eng, const swb_scene_soa *scenes, const int32_t *env_ids,
                      const int32_t *ring_slots, int32_t n, void *stream);

/* Forces every env (or those with mask[e] != 0, device pointer, may be NULL) to restart
 * from its next pooled scene on the next swb_step: sets the reset flag. */
int swb_request_reset(swb_engine *eng, const uint8_t *mask, void *stream);

/*
 * One Environment.step for all E envs (environment.py:88-108): envs whose reset flag is
 * set ignore their action, advance their ring cursor, load that scene and return FIRST;
 * the others apply the action, the velocity update, the task and the termination test.
 * `actions`: device pointer, [E][4] f32/f64 or [E][2] i32 per `action_dtype`.
 */
int swb_step(swb_engine *eng, const void *actions, int32_t action_dtype, const swb_step_out *out,
             void *stream);

/* task.reward(sprites) / task.success(sprites) of the live state, nothing else
 * (tasks.py:35-67): out->reward = task reward (no action cost), out->success. */
int swb_eval_task(swb_engine *eng, const swb_step_out *out, void *stream);

/* action_space.step(action, sprites, keep_in_frame) only (action_spaces.py:83-104,
 * 187-214): moves the clicked/carried/body sprites, out->reward = the action's cost.
 * No velocity update, task evaluation, counters or auto-reset. */
int swb_apply_action(swb_engine *eng, const void *actions, int32_t action_dtype,
                     const swb_step_out *out, void *stream);

/*
 * Scores candidate action sequences without changing anything: for every env e and candidate c,
 * the n_steps steps actions[0 .. n_steps-1][e][c] applied one after the other to a copy of the
 * state env e is in when the call runs.  One kernel, one warp per (env, candidate).
 * `actions`: device pointer, [n_steps][E][n_candidates][4] f32/f64 or [..][2] i32 per
 * `action_dtype`, as swb_step takes them.  `out`: device pointers to [n_steps][E][n_candidates]
 * elements each, the caller's.
 *
 * Entry [t][e][c] is what swb_step would report at step t of that plan -- reward with action
 * cost, step type from success, out of frame or max_episode_length counted from the env's own
 * step_count, success, status (a bad Embodied direction is counted, moves nothing, reports NaN
 * and SWB_ENV_BAD_ACTION, and the plan goes on) -- up to and including the plan's first
 * SWB_STEP_LAST.  The entries after it are padding: step type SWB_STEP_NONE, reward 0.0, success
 * 0, status 0; a rollout never starts another scene.  An env whose reset flag is set has no
 * episode to plan in (its next swb_step ignores the action and starts a new scene): all its
 * entries are padding.  Summed over t, `reward` is each plan's return.
 *
 * Read-only: positions, cursor, step_count, the reset flag, scene_serial, the pool and the
 * render and id status are as they were.  n_steps and n_candidates must be >= 1 and
 * n_steps * E * n_candidates at most SWB_ROLLOUT_MAX_ENTRIES; a refused call enqueues nothing.
 */
#define SWB_ROLLOUT_MAX_ENTRIES 2147483647 /* entries per output array of one swb_rollout */
int swb_rollout(swb_engine *eng, const void *actions, int32_t action_dtype, int32_t n_steps,
                int32_t n_candidates, const swb_step_out *out, void *stream);

/* Renderer: PILRenderer(image_size=(width,height), anti_aliasing, bg_color)
 * (renderers/pil_renderer.py:32-65).  Frame layout: [E][height][width][3] uint8.  Any
 * anti_aliasing >= 1 whose canvas sides stay within 4095 pixels is accepted where its resampling
 * tables fit the render kernel: the vertical tap windows of one block of eight output rows must
 * span at most 176 canvas rows.  That holds for every factor up to 13 at any frame size, and
 * above 13 for frames short enough.  Refuses a raster that does not fit, naming the limit, and a
 * raster whose render launch would not fit in shared memory even with convex shapes only; with
 * a star or spoke uploaded later a launch can still be refused. */
int swb_raster_create(swb_engine *eng, int32_t width, int32_t height, int32_t anti_aliasing,
                      const uint8_t bg_rgb[3], swb_raster **out);
void swb_raster_destroy(swb_raster *r);

/* Renders the current sprites of every env (pil_renderer.py:67-91). */
int swb_render(swb_engine *eng, swb_raster *r, uint8_t *frames, void *stream);

/* swb_step immediately followed by swb_render on the same stream. */
int swb_step_render(swb_engine *eng, swb_raster *r, const void *actions, int32_t action_dtype,
                    const swb_step_out *out, uint8_t *frames, void *stream);

/*
 * Multi-GPU frame gather fused into the render kernel (the path's one collective, SURVEY 8(e):
 * "one gather of frames per step" after environment.py:102).  Every rank passes the same
 * list of `n_dst` gathered buffers, each [n_ranks * E][height][width][3] uint8 -- its own
 * and its peers', opened with swb_ipc_open -- and the render kernel stores each finished
 * frame at env index `env_offset + e` (env_offset = rank * E) in all of them with the
 * 128-bit stores of its write-out phase, over NVLink peer memory.  The stores are complete
 * when the kernel is; a cross-rank barrier after it (the caller's, e.g. a one-element
 * all-reduce) makes every buffer whole.  n_dst <= SWB_MAX_PEERS.
 */
int swb_step_render_gather(swb_engine *eng, swb_raster *r, const void *actions,
                           int32_t action_dtype, const swb_step_out *out, uint8_t *const *dst,
                           int32_t n_dst, int64_t env_offset, void *stream);

/* Device buffers other processes can map: cudaMalloc + cudaIpcGetMemHandle, and the peer's
 * side of it.  `handle` is SWB_IPC_HANDLE_BYTES opaque bytes to ship to the other ranks. */
int swb_ipc_alloc(int32_t device, uint64_t bytes, void **ptr, uint8_t *handle);
int swb_ipc_free(void *ptr);
int swb_ipc_open(int32_t device, const uint8_t *handle, void **ptr);
int swb_ipc_close(void *ptr);
/* Asynchronous device-to-device copy on `stream`; either side may be a buffer opened with
 * swb_ipc_open (the copy engine then moves the bytes over NVLink). */
int swb_peer_copy(void *dst, const void *src, uint64_t bytes, void *stream);

/*
 * Host-buffer convenience for the whole call a binding makes per step: copies `actions`
 * host->device, steps, renders, copies outputs and frames device->host, synchronises.
 * Any of frames/reward/step_type/success/status may be NULL to skip that copy.
 */
int swb_step_host(swb_engine *eng, swb_raster *r, const void *actions, int32_t action_dtype,
                  double *reward, int8_t *step_type, uint8_t *success, uint8_t *status,
                  uint8_t *frames, void *stream);

/* Device pointers to the live struct-of-arrays state (for zero-copy observation views).
 * pos_x/pos_y: [E*S] double; shape: [E*S] u8 (of the env's current scene);
 * cursor/step_count: [E] int32; reset_next: [E] u8. */
int swb_state_pointers(swb_engine *eng, double **pos_x, double **pos_y, int32_t **cursor,
                       int32_t **step_count, uint8_t **reset_next);

/* Device pointer to the per-env status of the last swb_render (SWB_ENV_SPAN_OVERFLOW): [E] u8.
 * swb_step_render / swb_step_host report the same bit through swb_step_out.status. */
int swb_render_status_pointer(swb_engine *eng, uint8_t **render_status);

/* Device pointer to scene_serial: [E] int32, how many scenes each env has started (monotonic;
 * the env's ring slot is `cursor`).  Lets a host refill thread tell how far every env's ring
 * has been consumed without the modulo ambiguity of the cursor. */
int swb_scene_serial_pointer(swb_engine *eng, int32_t **scene_serial);

/* Copies the current state to host arrays (any may be NULL). pos: [E*S] each. */
int swb_download_state(swb_engine *eng, double *pos_x, double *pos_y, int32_t *cursor,
                       int32_t *step_count, uint8_t *reset_next, void *stream);

/* Overwrites the live positions / counters from host arrays (any may be NULL). */
int swb_upload_state(swb_engine *eng, const double *pos_x, const double *pos_y,
                     const int32_t *cursor, const int32_t *step_count, const uint8_t *reset_next,
                     void *stream);

/*
 * Env records: save, load and copy the state of envs on the device.
 *
 * An env record is everything that decides an env's future steps and frames within its current
 * episode: the sprite records of its current scene (the pool entry at (env, cursor)), its live
 * positions, step_count and reset_next.  cursor and scene_serial are not in it: they stay with
 * the env a record is loaded into, which plays the saved episode out and then starts the next
 * scene of its own ring.  A load or copy writes only the pool entry at the destination's cursor.
 * A record with reset_next = 1 (saved on a LAST step, say) starts the env's next ring scene on the
 * next swb_step, as swb_request_reset does: a caller that refills rings as they are consumed
 * counts a load or copy as a reset (environment.BatchedEnvironment does).
 *
 * Records are record-major, swb_env_record_bytes() (a multiple of 16) apart, so that record
 * sets can be sliced and concatenated and a record loaded into any env of any engine created
 * with the same swb_config apart from n_envs, pool_depth and device.  One record, S = n_slots,
 * every field's S values contiguous, little-endian:
 *
 *   offset      type      count   field
 *   0           double    8 x S   x0, y0, m00, m01, m10, m11, vx, vy of the current scene
 *   64 S        double    2 x S   pos_x, pos_y (live positions)
 *   80 S        uint32    S       member
 *   84 S        uint32    S       rgb (r | g << 8 | b << 16)
 *   88 S        float     5 x S   factors: scale[S], angle[S], c0[S], c1[S], c2[S]
 *   108 S       int32     1       step_count
 *   108 S + 4   uint8     1       reset_next
 *   108 S + 5   uint8     S       shape
 *   109 S + 5   uint8     S       pos_f32
 *   110 S + 5   zero      ..      padding up to swb_env_record_bytes(), when G = 0
 *
 * An engine with G > 0 goal slots appends the goals of the current scene, and swb_env_record_bytes()
 * grows accordingly (it is unchanged for G = 0):
 *
 *   P = 110 S + 5 rounded up to 8
 *   P           double    2 x G   goal (x, y) of goal slot g at P + 16 g
 *   P + 16 G    zero      ..      padding up to swb_env_record_bytes()
 *
 * Id arrays are HOST pointers, checked on the host; a call its checks refuse enqueues nothing.
 * (swb_save_envs_dev and its siblings below take device ids, checked on the device.)
 * Record buffers are device pointers aligned to 16 bytes.  The ids reach the device through a
 * pinned staging block of these calls (free to reuse when the call returns); the work is enqueued
 * on `stream`.  n == 0 enqueues nothing.
 *
 * Records are not validated beyond their shape ids: a shape id without a vertex table loads as an
 * empty slot.  Any other byte of a record that swb_save_envs of an engine of the same
 * configuration did not write -- and a span_class lower than its shapes need -- gives undefined
 * steps and frames.
 *
 * Read-only record calls (swb_rollout_states, swb_rollout_trajectory, swb_render_states, swb_render_masks,
 * swb_render_coverage, swb_render_soft_masks, swb_render_boxes, swb_evaluate_states,
 * swb_sample_contained) read n rows: n records of this
 * engine's layout in a device record buffer of records_bytes bytes or, where a call takes them,
 * the E live envs for records == NULL, and then n == E.  Each of them is refused, enqueuing
 * nothing, for a null engine, n < 0, records == NULL where the call takes no live envs, a record
 * buffer not 16-byte aligned or smaller than n records, an output that is null or not aligned to
 * its element type, or an output that overlaps another output or the records it reads.  Each
 * call's comment lists what it refuses besides.
 */
int64_t swb_env_record_bytes(const swb_engine *eng);

/* Record i <- env env_ids[i] (ids in [0, E), repeats allowed), into the device buffer `dst` of at
 * least n * swb_env_record_bytes() bytes.  *span_class <- the engine's spans per sprite row:
 * 1 while every uploaded or loaded shape is convex, else 4; pass it to swb_load_envs. */
int swb_save_envs(swb_engine *eng, const int32_t *env_ids, int32_t n, void *dst, uint64_t dst_bytes,
                  int32_t *span_class, void *stream);

/* Env env_ids[i] <- record i, from the device buffer `src` of at least n * swb_env_record_bytes()
 * bytes holding records saved by swb_save_envs of an engine with the same configuration.  Ids in
 * [0, E), distinct.  span_class (1 or 4, as saved) raises the engine's spans per sprite row as an
 * upload of a star or spoke does. */
int swb_load_envs(swb_engine *eng, const int32_t *env_ids, int32_t n, const void *src, uint64_t src_bytes,
                  int32_t span_class, void *stream);

/*
 * swb_rollout from any set of env records, and the state each plan ends in as a record: one level
 * of a search tree in one launch, with nothing on the host between levels.
 *
 * Roots: `roots` NULL means the E live envs, and then n_roots must be E.  Otherwise `roots` is a
 * device buffer of roots_bytes bytes holding n_roots >= 1 records (independent of E) in the
 * layout above; a root is staged as the env a swb_load_envs of it would make, so a root with
 * reset_next set has no episode to plan in and all its entries are padding.  `actions` are
 * [n_steps][n_roots][n_candidates][4] f32/f64 or [..][2] i32; every output of `out` is
 * [n_steps][n_roots][n_candidates], with the meaning swb_rollout gives it.
 *
 * Leaves: `leaves` NULL means none.  Otherwise it is a device buffer of leaves_bytes bytes, and
 * record r * n_candidates + c becomes, byte for byte, what swb_save_envs would save of an env
 * loaded from root r that then took plan c's live steps through swb_step: the root's scene, the
 * final positions, step_count after the steps counted (bad Embodied steps included) and
 * reset_next = 1 iff the plan's last live step was SWB_STEP_LAST (a root about to reset is its
 * own leaf).  *span_class (if span_class is not NULL) <- for live roots the engine's spans per
 * sprite row, as swb_save_envs reports it; with record roots it is not written: the leaves need
 * the span class of their roots.
 *
 * A read-only record call (above) with the roots as its rows, and the leaves and every array of
 * `out` as its outputs.  Refused besides: what swb_rollout refuses, with n_roots in place of E (so
 * n_steps * n_roots * n_candidates at most SWB_ROLLOUT_MAX_ENTRIES), record roots with
 * n_roots < 1, and leaves not 16-byte aligned or smaller than n_roots * n_candidates records.  An
 * accepted call is one launch, leaves included.  Read-only but for `out` and `leaves`, as
 * swb_rollout.
 *
 * Records are not validated beyond their shape ids: a shape id without a vertex table loads as an
 * empty slot.  Any other byte of a record that swb_save_envs of an engine of the same
 * configuration did not write gives undefined outputs and leaves.
 */
int swb_rollout_states(swb_engine *eng, const void *roots, int32_t n_roots, uint64_t roots_bytes,
                       const void *actions, int32_t action_dtype, int32_t n_steps, int32_t n_candidates,
                       const swb_step_out *out, void *leaves, uint64_t leaves_bytes,
                       int32_t *span_class, void *stream);

/*
 * swb_rollout_states with the state after every step of every plan: trajectories of the candidate
 * plans in one launch, for the frames, masks, boxes or task values of each imagined step.
 *
 * Roots, actions, `out` and *span_class are as swb_rollout_states has them, and `out` is bit for bit
 * what it writes.  `records` (required) is a device buffer of records_bytes bytes: record
 * (t * n_roots + r) * n_candidates + c is, byte for byte, leaf r * n_candidates + c of
 * swb_rollout_states called with the same roots and only the first t + 1 steps of the actions.  So
 * after a plan's first SWB_STEP_LAST every record repeats its end state (reset_next = 1), a root
 * about to reset is its own record at every t, every record keeps its root's goals, and the last
 * n_roots * n_candidates records are the leaves.
 *
 * A read-only record call (above) with the roots as its rows, and `records` and every array of
 * `out` as its outputs.  Refused besides: what swb_rollout_states refuses, records NULL, and
 * records not 16-byte aligned or smaller than n_steps * n_roots * n_candidates records.  An
 * accepted call is one launch.  Read-only but for `out` and `records`, as swb_rollout.
 */
int swb_rollout_trajectory(swb_engine *eng, const void *roots, int32_t n_roots, uint64_t roots_bytes,
                           const void *actions, int32_t action_dtype, int32_t n_steps, int32_t n_candidates,
                           const swb_step_out *out, void *records, uint64_t records_bytes,
                           int32_t *span_class, void *stream);

/*
 * The frames of env records without loading them into envs: frame i (of [n][height][width][3]
 * uint8 `frames`) is, byte for byte, what swb_render would draw for an env swb_load_envs had
 * loaded record i into, and status[i] is that env's render status (SWB_ENV_SPAN_OVERFLOW).
 * `records`: a device buffer of records_bytes bytes holding n records (independent of E) in the
 * layout above, with span_class (1 or 4) as saved.  One launch; status is zeroed on the stream
 * first.  n == 0 enqueues nothing.
 *
 * Read-only: no env, pool entry, counter, render status or span class of the engine changes.
 * Records of stars or spokes rendered by an engine whose shapes are all convex get the concave
 * span tables for this call only.  A read-only record call (above) without live envs, whose
 * outputs are frames and status; with n == 0 it checks nothing but the engine and raster.  Refused
 * besides: a null raster, a span_class other than 1 or 4, n * (the raster's bands of 64 rows) above
 * 2^31 - 1, or a render launch that would not fit (as swb_render is refused).  Records are not
 * validated beyond their shape ids, as in swb_load_envs.
 */
int swb_render_states(swb_engine *eng, swb_raster *r, const void *records, int32_t n,
                      uint64_t records_bytes, int32_t span_class, uint8_t *frames,
                      uint8_t *status, void *stream);

/*
 * The scene seen through windows: n_views frames of each row, each the raster's PILRenderer frame of
 * the window (x0, y0, x1, y1) of scene coordinates instead of the unit square.  Zoomed sprite
 * glimpses, egocentric views.
 *
 * Rows: `records` NULL means the E live envs (then n must be E), else n records as in
 * swb_render_states, with span_class (1 or 4) as saved; live rows pass 1 and render with the
 * engine's own spans per sprite row, as swb_render does.
 * windows[(i * n_views + v) * 4 + 0..3] (device f64, 8-byte aligned) is the window of view v of row
 * i; frames [n][n_views][height][width][3] u8 and status [n][n_views] u8 (SWB_ENV_* bits) are the
 * item's.  With CW = aa * width, CH = aa * height, a world vertex (wx, wy) -- the one swb_render
 * multiplies by CW and CH -- goes to the canvas vertex (trunc(u), trunc(v)) with
 *   sx = CW / (x1 - x0);  u = (wx - x0) * sx       (each op float64, round to nearest)
 *   sy = CH / (y1 - y0);  v = (wy - y0) * sy
 * and everything after that is swb_render's: so the window (0, 0, 1, 1) draws swb_render's (or
 * swb_render_states') frame byte for byte.  An item whose window is not finite or has x1 <= x0 or
 * y1 <= y0, or with an occupied slot whose vertex has u or v NaN or |u| or |v| >= 2^30, gets
 * SWB_ENV_BAD_WINDOW and a frame of zeros; a span overflow sets SWB_ENV_SPAN_OVERFLOW as in
 * swb_render_states.  One memset of status and one launch; n == 0 enqueues nothing.
 *
 * Read-only as swb_render_states.  Refused besides what swb_render_states refuses (for live rows,
 * what swb_render refuses): live rows with n != E, n_views < 1, n * n_views * (the raster's bands)
 * above 2^31 - 1, and windows that are null, not 8-byte aligned, or overlap the outputs or the records.
 */
int swb_render_windows(swb_engine *eng, swb_raster *r, const void *records, int32_t n,
                       uint64_t records_bytes, int32_t span_class, const double *windows, int32_t n_views,
                       uint8_t *frames, uint8_t *status, void *stream);

/*
 * Views of chosen sprites: swb_render_windows with only some slots drawn.  Sprite layers (one slot
 * drawn alone), scenes with sprites removed, glimpses of a sprite without its occluders.
 *
 * draw[(i * n_views + v) * S + s] (device u8, S the engine's slot count) is nonzero where slot s is
 * drawn in view v of row i.  The view's frame and status are swb_render_windows' of the row in
 * which every undrawn slot is an empty slot (shape 0; a record's undrawn slot is not read beyond
 * its draw byte): the sprites drawn keep their back-to-front order, no slot drawn gives the
 * background, every slot drawn gives swb_render_windows' frame byte for byte.  SWB_ENV_BAD_WINDOW
 * and SWB_ENV_SPAN_OVERFLOW count drawn slots only.
 *
 * Refused besides what swb_render_windows refuses: a null draw, and a draw that overlaps frames or
 * status.  A refused call enqueues nothing.
 */
int swb_render_views(swb_engine *eng, swb_raster *r, const void *records, int32_t n, uint64_t records_bytes,
                     int32_t span_class, const double *windows, const uint8_t *draw, int32_t n_views,
                     uint8_t *frames, uint8_t *status, void *stream);

/*
 * Sprite instance masks (renderers.SpriteMasks): which sprite is visible at each pixel.  `masks`
 * is [n][height][width] uint8; mask i's pixel (r, c) is k + 1 if slot k is the top-most sprite whose
 * Pillow polygon fill -- the integer vertices int(canvas_size * vertex) PILRenderer draws at this
 * width, height and anti_aliasing -- covers canvas pixel (aa c + aa/2, aa (height-1-r) + aa/2) of
 * the aa*width x aa*height canvas, and 0 if none does.  Rows are flipped as frames are.  Ids index
 * the slot axis; empty slots are never visible.
 *
 * records == NULL: the E live envs, with n == E.  Otherwise n records (any n) of this engine's
 * layout in a device buffer of records_bytes bytes, drawn as if loaded into envs (shape ids
 * sanitised as swb_load_envs does).  The mask is exact for every shape: there is no span table and
 * no status.  Any anti_aliasing whose canvas sides stay within 4095 pixels is accepted.
 *
 * An accepted call with n > 0 is one launch on `stream`; n == 0 enqueues nothing.  Read-only: no
 * env, pool entry, counter, frame buffer, render status or span class changes.  A read-only record
 * call (above) whose output is masks.  Refused besides, width, height and canvas first: width,
 * height or anti_aliasing < 1, a canvas side above 4095, or an n whose bands (of at most 128 mask
 * rows) exceed 2^31 - 1 CTAs.
 */
int swb_render_masks(swb_engine *eng, int32_t width, int32_t height, int32_t anti_aliasing,
                     const void *records, int32_t n, uint64_t records_bytes, uint8_t *masks,
                     void *stream);

/*
 * Amodal sprite coverage (renderers.SpriteCoverage): every sprite covering each pixel, hidden or
 * not.  `cover` is [n][height][width] int32; bit k of pixel (r, c) is set if slot k's Pillow polygon
 * fill covers the sample point swb_render_masks uses for that pixel, whether or not a sprite above
 * hides it (bit 31 is the sign bit).  So the mask swb_render_masks draws is the highest set bit + 1,
 * or 0 where cover is 0.  `visible` and `area` are [n][S] int32: for each slot, the number of
 * pixels where it is the top-most covering sprite, and the number where its bit is set.  Empty
 * slots and sprites wholly out of frame have no bits and zero counts.
 *
 * Records, sizes and n as swb_render_masks takes them (records == NULL: the E live envs, n == E).
 * An accepted call with n > 0 zeroes visible and area on `stream` and is then one launch there;
 * the counts are integer sums, exact and independent of scheduling.  n == 0 enqueues nothing.
 * Read-only as swb_render_masks, with cover, visible and area as outputs.  Refused besides: what
 * swb_render_masks refuses, with bands of at most 128 mask rows and 16 KiB of coverage.
 */
int swb_render_coverage(swb_engine *eng, int32_t width, int32_t height, int32_t anti_aliasing,
                        const void *records, int32_t n, uint64_t records_bytes, int32_t *cover,
                        int32_t *visible, int32_t *area, void *stream);

/*
 * Soft sprite masks (renderers.SoftSpriteMasks): how much of each pixel each sprite owns.  `soft`
 * is [n][S][height][width] uint8; soft[i][k][r][c] is the number of canvas pixels
 * (aa c + u, aa (height-1-r) + v), u and v in [0, aa), of the aa*width x aa*height canvas whose
 * top-most covering sprite is slot k, with the integer vertices and Pillow fill rules of
 * swb_render_masks.  So soft / aa^2 is the fraction of the pixel's box the slot owns, aa^2 minus the
 * sum over the slots is the background's count, the sample swb_render_masks reads (u = v = aa/2) is
 * one of them, and at anti_aliasing 1 soft[i][k] is (mask == k + 1).  Empty slots and sprites out
 * of frame or wholly hidden are zero.  A box filter of the label canvas: the frames are LANCZOS
 * filtered, so they are not the soft masks' composite of sprite colours.
 *
 * Records, sizes and n as swb_render_masks takes them (records == NULL: the E live envs, n == E).
 * An accepted call with n > 0 is one launch on `stream` that writes every byte of `soft`; n == 0
 * enqueues nothing.  Read-only as swb_render_masks, with soft as its output.  Refused besides: what
 * swb_render_masks refuses, anti_aliasing above 15 (aa^2 = 225 is the largest count a byte holds),
 * with bands of at most 128 canvas rows and 32 KiB of staged canvas (or one mask row).
 */
int swb_render_soft_masks(swb_engine *eng, int32_t width, int32_t height, int32_t anti_aliasing,
                          const void *records, int32_t n, uint64_t records_bytes, uint8_t *soft,
                          void *stream);

/*
 * Sprite bounding boxes (renderers.SpriteBoxes): the per-slot summaries of swb_render_coverage
 * without its per-pixel output.  `visible_box` and `amodal_box` are [n][S][4] int32, `visible` and
 * `area` [n][S] int32.  For slot k of row i, with V the pixels (r, c) where it is the top-most
 * covering sprite (mask == k + 1 in swb_render_masks) and A those where its bit is set in
 * swb_render_coverage's cover: visible_box = box(V), amodal_box = box(A), visible = |V| and
 * area = |A|, where box(P) = (min c, min r, max c + 1, max r + 1) -- half-open (x0, y0, x1, y1) in
 * pixels of the flipped image -- and (0, 0, 0, 0) for an empty P.  So the visible box lies in the
 * amodal box, visible <= area, and a count is 0 iff its box is.  The counts equal
 * swb_render_coverage's.  Bit 31 (slot 31) is a slot like any other.
 *
 * Records, sizes and n as swb_render_masks takes them (records == NULL: the E live envs, n == E).
 * An accepted call with n > 0 zeroes the four outputs on `stream` (four memsets), then is two
 * launches there: the mask kernel, which sends integer atomics per band and slot, and a kernel that
 * decodes the boxes' mins.  The outputs are exact and independent of scheduling.  n == 0 enqueues
 * nothing.  Read-only as swb_render_masks, with visible_box, amodal_box, visible and area as outputs.
 * Refused besides: what swb_render_coverage refuses.
 */
int swb_render_boxes(swb_engine *eng, int32_t width, int32_t height, int32_t anti_aliasing,
                     const void *records, int32_t n, uint64_t records_bytes, int32_t *visible_box,
                     int32_t *amodal_box, int32_t *visible, int32_t *area, void *stream);

/* Env dst_ids[i] <- env src_ids[i].  Ids in [0, E), destinations distinct.  Every read sees the
 * state from before the call, also where the two sets overlap (then the records go through
 * device scratch of the engine: two kernels instead of one). */
int swb_copy_envs(swb_engine *eng, const int32_t *src_ids, const int32_t *dst_ids, int32_t n, void *stream);

/*
 * Device-checked id lists: the same three calls with ids in DEVICE memory of the engine's device,
 * SWB_DTYPE_I32 or SWB_DTYPE_I64 per `id_dtype`, checked by kernels, so that the host never waits
 * for ids the device computes (an argmax, a top-k, a multinomial draw).  The host checks only what
 * it sees without reading device memory -- the pointers, `id_dtype`, that the ids are device
 * memory of the engine's device aligned to their type, n, the record buffer's size and alignment,
 * span_class -- and a call those checks refuse enqueues nothing.  n == 0 enqueues nothing.
 *
 * The kernels apply the host path's rules: every id in [0, E), compared in the id type's own width
 * (an int64 2^32 + 1 is out of range, not 1), and destination ids distinct (load, copy).  A call is
 * all or nothing: if any id fails, no env, pool entry or counter changes, and a save writes zero
 * bytes into every one of its n records (a zero record loads as an env with only empty slots).  A
 * refused id never indexes engine memory, and the calls after a refused one run normally.  A load
 * refused on the device has still raised the engine's span class (renders stay exact).
 *
 * Failures are reported in the engine's swb_ids_status record (swb_env_ids_status_pointer): `ok`
 * is rewritten by every device-checked call, and the fields after it hold the first failure since
 * the caller last zeroed `failed`: calls are stream-ordered, so the earliest refused call, and
 * within it the lowest failing position (arguments in the call's order at equal positions).  For a
 * repeat that is the lowest position whose id also appears at a lower position.
 *
 * A copy saves every source to engine scratch, then loads the destinations from it: every read
 * sees the state from before the call, whatever the overlap.  Scratch grows to n records the
 * first time a copy needs more; that growth synchronises the device, later copies of at most that
 * many ids do not.  Kernels per call: save 2, load 3, copy 3.  Device-checked calls of one engine
 * are ordered on one stream at a time (they share the scratch, the status record and the claim
 * array that checks distinctness).
 */
enum { SWB_IDS_CALL_SAVE = 0, SWB_IDS_CALL_LOAD = 1, SWB_IDS_CALL_COPY = 2, SWB_IDS_CALL_SET_GOALS = 3 };
enum { SWB_IDS_OUT_OF_RANGE = 1, SWB_IDS_REPEATED = 2 };
typedef struct {
  uint32_t ok;       /* 1: the last device-checked call passed its id checks; 0: it was refused */
  uint32_t failed;   /* 1: the fields below hold the first refused call since the caller zeroed this */
  int32_t call;      /* SWB_IDS_CALL_* */
  int32_t arg;       /* the id argument: 0 = env_ids (save, load) or src_ids (copy), 1 = dst_ids */
  int32_t reason;    /* SWB_IDS_OUT_OF_RANGE or SWB_IDS_REPEATED */
  int32_t position;  /* index into that argument */
  int64_t value;     /* the id there */
} swb_ids_status;

int swb_save_envs_dev(swb_engine *eng, const void *env_ids, int32_t id_dtype, int32_t n, void *dst,
                      uint64_t dst_bytes, int32_t *span_class, void *stream);
int swb_load_envs_dev(swb_engine *eng, const void *env_ids, int32_t id_dtype, int32_t n, const void *src,
                      uint64_t src_bytes, int32_t span_class, void *stream);
int swb_copy_envs_dev(swb_engine *eng, const void *src_ids, const void *dst_ids, int32_t id_dtype, int32_t n,
                      void *stream);
/* Device pointer to the engine's swb_ids_status record (zeroed at engine creation). */
int swb_env_ids_status_pointer(swb_engine *eng, swb_ids_status **status);

/*
 * Device scene sampler.
 *
 * A swb_scene_program is a scene generator (init_sprites) flattened into code for one thread:
 * spriteworld_b200/scene_program.py builds it from generate_sprites / chain_generators /
 * sample_generator / shuffle over Continuous / Discrete / Product / Mixture / SetMinus /
 * Intersection / Selection, together with the task's filter distributions.  Scene `a` of global env
 * `g` is a pure function of (seed, g, a): Philox4x64-10 with key (seed, SWB_SAMPLER_DOMAIN) and
 * counter (block, a, g, 0), block = 0, 1, ... giving the scene's 64-bit draw words four at a time
 * (csrc/swb_sampler.cuh).  Every scene is packed as swb_upload_scenes would store the same
 * sprites packed on the host (scene.arrays_from_layout).
 *
 * Code layout.  ops[0 ..] is the generator, run once per scene:
 *   G_SPRITES  a = distribution code, dtype = 0: b sprites, 1: np.random.randint(b, c) sprites
 *   G_MARK / G_SHUFFLE   uniform permutation of the sprites appended between the two
 *   G_CHOOSE   c = cdf (consts), b = n; followed by n G_JUMPs, one per generator
 *   G_JUMP     a = target;   G_END
 * Distribution code draws one sprite's factors, ending in D_RET:
 *   D_CONT     key, dtype, lo + (hi - lo) * u in float64 (u: 53 bits), then .astype(dtype)
 *   D_DISC     key, dtype, a = candidates (consts), b = n, c = cdf or -1 (uniform)
 *   D_MIX      c = cdf, b = n; followed by n D_JUMPs;   D_JUMP a = target
 *   D_REJ_BEGIN .. D_REJ_END  a = predicate, b = 1 keep inside / 0 keep outside: redraw the code
 *              between them until accepted, at most SWB_SAMPLER_MAX_TRIES times
 * Predicate code (containment, postfix over a bool stack) ends in P_RET:
 *   P_CONT     key, lo (kind a) <= v < hi (kind b);  P_DISC key, a = candidates, b = n
 *   P_AND / P_OR  b = operands;  P_NOT
 * Values and constants carry a kind (SWB_FT_*): the NumPy dtype of the value, or for constants a
 * Python float / int, which compares against a float32 value in float32 (NEP 50).
 */
#define SWB_PROG_MAX_OPS 512
#define SWB_PROG_MAX_CONSTS 1024
#define SWB_PROG_MAX_ANGLES 1024
#define SWB_PROG_MAX_STACK 16          /* nesting of shuffles, rejections and predicate operands */
#define SWB_SAMPLER_MAX_TRIES 100000   /* factor_distributions._MAX_TRIES */
#define SWB_SAMPLER_DOMAIN 0x53574253434e4531ULL   /* second key word of the scene stream */
enum {
  SWB_FT_NONE = 0, SWB_FT_F32 = 1, SWB_FT_F64 = 2,
  SWB_FT_I8 = 3, SWB_FT_I16 = 4, SWB_FT_I32 = 5, SWB_FT_I64 = 6,
  SWB_FT_U8 = 7, SWB_FT_U16 = 8, SWB_FT_U32 = 9, SWB_FT_U64 = 10,
  SWB_FT_SHAPE = 11,    /* a shape name; the value is its ShapeType id */
  SWB_FT_PYFLOAT = 12, SWB_FT_PYINT = 13   /* constants only */
};
enum {
  SWB_OP_G_END = 0, SWB_OP_G_SPRITES, SWB_OP_G_MARK, SWB_OP_G_SHUFFLE, SWB_OP_G_CHOOSE, SWB_OP_G_JUMP,
  SWB_OP_D_RET = 10, SWB_OP_D_CONT, SWB_OP_D_DISC, SWB_OP_D_MIX, SWB_OP_D_JUMP, SWB_OP_D_REJ_BEGIN,
  SWB_OP_D_REJ_END,
  SWB_OP_P_RET = 20, SWB_OP_P_CONT, SWB_OP_P_DISC, SWB_OP_P_AND, SWB_OP_P_OR, SWB_OP_P_NOT
};
enum { SWB_COLOR_RGB = 0, SWB_COLOR_HSV = 1 };

typedef struct {
  int32_t op, key, dtype, a, b, c;
  double lo, hi;
} swb_prog_op;

typedef struct {
  int32_t n_ops, n_consts, n_angles, n_filters;
  int32_t max_sprites;  /* most sprites one scene can have */
  int32_t color_mode;   /* SWB_COLOR_RGB: colours are RGB (int64, then uint8); SWB_COLOR_HSV */
  int32_t filter_pc[SWB_MAX_FILTERS];  /* predicate of member bit i */
  swb_prog_op ops[SWB_PROG_MAX_OPS];
  double consts[SWB_PROG_MAX_CONSTS];
  int32_t const_kind[SWB_PROG_MAX_CONSTS];
  /* every angle value the code can draw, ascending (-0.0 before 0.0), with libm's
   * cos / sin of its radians (scene.transform_matrix) */
  double angle[SWB_PROG_MAX_ANGLES], angle_cos[SWB_PROG_MAX_ANGLES], angle_sin[SWB_PROG_MAX_ANGLES];
  /* sampled FindGoalPosition goals: goal slot g is drawn by the distribution code at goal_pc[g] (its
   * x and y), after the scene's sprites, from the same stream.  n_goals must equal the engine's G. */
  int32_t n_goals;
  int32_t goal_pc[SWB_MAX_GOALS];
} swb_scene_program;

/* Output of swb_sample_scenes: device pointers, [n * S] per field (rgb [n * S * 3], factors
 * [n * S * 5]), the fields of swb_scene_soa.  factor_value / factor_kind: [n * S * 10] drawn
 * factors (x, y, shape, angle, scale, c0, c1, c2, x_vel, y_vel) with their SWB_FT_* kind, kind
 * SWB_FT_NONE in empty slots. */
typedef struct {
  double *x, *y, *m00, *m01, *m10, *m11, *vx, *vy;
  uint32_t *member;
  uint8_t *shape, *pos_f32, *rgb;
  float *factors;
  double *factor_value;
  uint8_t *factor_kind;
  double *goal;   /* [n * G * 2] goals (x, y) per goal slot; may be NULL (then not written) */
} swb_sample_out;

/* The first rejection loop that ran out of tries, since the caller last zeroed `failed`.  The
 * scene it was drawing is left with every slot empty. */
typedef struct {
  uint32_t failed;
  int32_t op;       /* the D_REJ_END op */
  int64_t env;      /* global env id */
  int64_t scene;    /* absolute scene index */
} swb_sampler_status;

int swb_sampler_sizeof_program(void);

/* Gives the engine a program and a seed; env e of this engine is global env env_offset + e.
 * The program's max_sprites must fit n_slots.  Synchronises.  Resets the refill bookkeeping:
 * refilled_upto[e] = -1 (no scene sampled). */
int swb_sampler_load(swb_engine *eng, const swb_scene_program *prog, uint64_t seed, int64_t env_offset);

/* Samples scenes (env_ids[i], scene_idx[i]) -- int64 device arrays, global env ids, any values
 * >= 0 -- into `out`, without touching the pool. */
int swb_sample_scenes(swb_engine *eng, const int64_t *env_ids, const int64_t *scene_idx, int32_t n,
                      const swb_sample_out *out, void *stream);

/* Refill on the device: for every env, samples scenes refilled_upto[e] + 1 .. scene_serial[e] + K - 1
 * into ring slots a % K and advances refilled_upto[e].  One kernel on `stream`, no host wait. */
int swb_refill_device(swb_engine *eng, void *stream);

/* Device pointers to the scene pool, entry (env, ring slot, slot) at ((env * K + ring) * S + slot):
 * f64[0..7] = x, y, m00, m01, m10, m11, vx, vy; rgb packed r | g << 8 | b << 16; factors 5 per slot. */
int swb_pool_pointers(swb_engine *eng, double **f64, uint32_t **member, uint8_t **shape, uint8_t **pos_f32,
                      uint32_t **rgb, float **factors);

/*
 * Sampled goals.  A FindGoalPosition node with goal_slot g >= 0 reads its goal from the scene the
 * env is on: goal slot g of pool entry (env, ring slot), (x, y) at ((env * K + ring) * G + g) * 2.
 * An env stepped with goal (gx, gy) steps bit for bit as one whose node has goal_slot -1 and
 * goal = {gx, gy}.  Goals arrive with the scenes (swb_scene_soa.goal) and travel in env records
 * and checkpoints.  An engine with G = 0 allocates no goal array.
 *
 * swb_pool_goal_pointer: *goal <- the device array [E * K * G * 2] f64 (NULL when G = 0),
 * *n_goals <- G.
 */
int swb_pool_goal_pointer(swb_engine *eng, double **goal, int32_t *n_goals);

/*
 * Overwrites the goals of the scene each listed env is on: env env_ids[i] (ids in [0, E), distinct)
 * gets goals[i * G * 2 .. (i + 1) * G * 2) (device f64) in pool entry (env, cursor).  The env keeps
 * them until it starts its next scene, which brings that scene's goals.  Like swb_load_envs it writes
 * only the entry at the env's cursor.  Host ids are checked on the host; swb_set_goals_dev takes
 * device ids (SWB_DTYPE_I32 / I64) checked by kernels with the rules and status record of the _dev
 * record calls (call SWB_IDS_CALL_SET_GOALS, all or nothing).  Refused, enqueuing nothing: G = 0,
 * n < 0, null or unaligned pointers, bad host ids.  n == 0 enqueues nothing.
 */
int swb_set_goals(swb_engine *eng, const int32_t *env_ids, int32_t n, const double *goals, void *stream);
int swb_set_goals_dev(swb_engine *eng, const void *env_ids, int32_t id_dtype, int32_t n, const double *goals,
                      void *stream);

/*
 * The task tree's value on env records, as swb_eval_task gives it for a live env (no action cost):
 * reward[i], success[i] and status[i] of record i at its live positions, with the record's goals, or
 * with goals[i * G * 2 .. (i + 1) * G * 2) (device f64) in their place when `goals` is not NULL.
 * One launch; read-only: no env, pool entry, counter or record changes.  A read-only record call
 * (above) without live envs, whose outputs are reward, success and status.  Refused besides: goals
 * given with G = 0 or not 8-byte aligned.  n == 0 enqueues nothing.
 */
int swb_evaluate_states(swb_engine *eng, const void *records, int32_t n, uint64_t records_bytes,
                        const double *goals, double *reward, uint8_t *success, uint8_t *status, void *stream);

/*
 * Positions inside sprites (Environment.sample_contained_position, for random agents and plan
 * proposals): n_samples draws per row, of the E live envs (records == NULL, n == E) or of n env
 * records of this engine's layout (records_bytes bytes, 16-byte aligned, shape ids sanitised as
 * swb_load_envs does).  Sample s of row i:
 *   - the row's sprites are its slots with a non-zero shape id, in slot order; m of them.  m == 0:
 *     status SWB_ENV_NO_SPRITE.
 *   - draws come from Philox4x64-10 with key (seed, SWB_CONTAINED_DOMAIN) and counter
 *     (block, s, i, 0), words consumed in order as the scene sampler consumes them: word 0 picks
 *     sprite k = mulhi64(word, m), the k-th occupied slot.
 *   - lo / hi: the min / max over the shape's vertices of the centred path (m00 ax + m01 ay) + 0.0
 *     (and likewise y).  Each try draws ux, then uy (53-bit uniforms) and proposes
 *     c = pos + (lo + (hi - lo) u) in float64; it is accepted if the step kernel's even-odd hit test
 *     of c - pos finds it inside the sprite.  After SWB_CONTAINED_MAX_TRIES tries: status
 *     SWB_ENV_SAMPLE_TRIES (a sprite of scale 0, say).
 * position[(i * n_samples + s) * 2 + 0/1] (f64), slot[i * n_samples + s] (i8) and status (u8) are
 * device arrays of the caller; a failed sample has position NaN and slot -1.  Live envs sample the
 * scene they are on (pool entry (e, cursor)) at their live positions, also an env about to reset.
 * A float64 SelectMove / DragAndDrop action whose click is the returned position grabs the sampled
 * slot or a sprite above it, as c - pos is what swb_step computes from it (action noise aside).
 *
 * Each sample is a pure function of (seed, i, s, the row's state): nothing is kept between calls.
 * An accepted call with n > 0 is one launch on `stream`; n == 0 enqueues nothing.  Read-only: no
 * env, pool entry, counter or frame changes.  A read-only record call (above) whose outputs are
 * position, slot and status.  Refused besides: n_samples < 1, n * n_samples above 2^31 - 1.
 */
#define SWB_CONTAINED_MAX_TRIES 1000000          /* sprite.py _MAX_TRIES */
#define SWB_CONTAINED_DOMAIN 0x535742434e544431ULL  /* second key word of the contained-position stream */
int swb_sample_contained(swb_engine *eng, const void *records, int32_t n, uint64_t records_bytes,
                         int32_t n_samples, uint64_t seed, double *position, int8_t *slot, uint8_t *status,
                         void *stream);

/* Device pointers: refilled_upto [E] int64, and the engine's swb_sampler_status. */
int swb_sampler_pointers(swb_engine *eng, int64_t **refilled_upto, swb_sampler_status **status);

/*
 * Env records from factor values: scenes the caller chose, packed on the device.
 *
 * swb_packer_load gives the engine the packer of swb_make_states: a swb_scene_program of which only
 * the filters (bit i of `member` is filter_pc[i]'s predicate), color_mode and angle table are used
 * (scene_program.compile_packer builds it: its generator code is a lone G_END).  The angle table
 * must hold every integer in [-360, 360] and -0.0, with libm's cos / sin of their radians.  It is
 * the engine's own copy, apart from the device sampler's program.  Synchronises.
 *
 * swb_make_states writes n records (record i at i * swb_env_record_bytes() of `records`).  Record
 * i is, byte for byte, what swb_save_envs saves of an env that has just taken the reset (FIRST)
 * step of an episode whose scene is the sprite list [Sprite(**factors at (i, j)) for the occupied
 * slots j, in slot order], packed by the host packer (scene.arrays_from_layout) with the packer's
 * filters and colour map, with step_count[i] in place of 0 and goals[i] as its goals: live
 * position = initial position, reset_next = 0, every padding byte zero.
 *
 * Columns: cols->col[f] is a device array [n][S] of factor f (x, y, shape, angle, scale, c0, c1, c2,
 * x_vel, y_vel), element (i, j) at i * S + j, of dtype cols->kind[f] (SWB_FT_F32, F64, I8, I16, I32,
 * I64 or U8), aligned to it; or NULL for Sprite's default as a Python scalar (x = y = 0.5, angle 0,
 * scale 0.1, c0 = c1 = c2 = 0, x_vel = y_vel = 0.0), kind SWB_FT_PYFLOAT or SWB_FT_PYINT.  The shape
 * column is required: ShapeType ids, 0 for an empty slot, in any of those dtypes.  Under
 * SWB_COLOR_HSV the colour columns are all F32, all F64 or all NULL.  goals: device f64
 * [n][G][2], required when G > 0 and refused when G = 0.  step_count: device int32 [n], or NULL for
 * zeros.
 *
 * status[i] (device uint8 [n]) gets the SWB_MAKE_* bits of record i; a record with any bit set is
 * written as zeros (it loads as an env with only empty slots).  span_flag (device uint8, may be
 * NULL) is zeroed on `stream` and then set to 1 if an accepted record holds a star or spoke
 * (ShapeType 7 .. 12): such records need span class 4 (swb_load_envs, swb_render_states).
 *
 * An accepted call with n > 0 is (after the span_flag memset) one launch on `stream`, one warp per
 * record; n == 0 enqueues nothing.  Read-only for the engine: no env, pool entry, counter, frame
 * buffer or span class changes.  Refused, enqueuing nothing: a null engine, no packer loaded, n < 0,
 * null cols or shape column, a column of another kind or not aligned to it, a mixed HSV triple,
 * goals missing for G > 0 or given for G = 0 or not 8-byte aligned, step_count not 4-byte aligned,
 * records null, not 16-byte aligned or smaller than n records, a null status, and outputs (records,
 * status, span_flag) that overlap each other or the inputs.
 */
enum {
  SWB_MAKE_ANGLE = 1,  /* an occupied slot's angle is not an integer in [-360, 360] */
  SWB_MAKE_SHAPE = 2,  /* a shape value is not an integer in 0 .. 12 */
  SWB_MAKE_HOLE = 4,   /* an empty slot after an occupied one (a scene fills slots S - n .. S - 1) */
  SWB_MAKE_INT = 8,    /* an occupied slot's integer factor of magnitude above 2^53 */
  SWB_MAKE_STEP = 16   /* step_count < 0 */
};
typedef struct {
  const void *col[10];  /* x, y, shape, angle, scale, c0, c1, c2, x_vel, y_vel; NULL: the default */
  int32_t kind[10];     /* SWB_FT_* of each given column */
} swb_factor_columns;

int swb_packer_load(swb_engine *eng, const swb_scene_program *prog);
int swb_make_states(swb_engine *eng, const swb_factor_columns *cols, int32_t n, const double *goals,
                    const int32_t *step_count, void *records, uint64_t records_bytes, uint8_t *status,
                    uint8_t *span_flag, void *stream);

/*
 * Engine checkpoints: the whole state of an engine -- live positions and counters, every scene of
 * every ring and the device sampler's refill bookkeeping -- as one self-describing buffer in HOST
 * memory, to write to disk and load into an engine of the same configuration (in another process
 * or on another device index too), which then steps and renders exactly as the saved one would
 * have.  Render status, id status and sampler status records are transient and not in it.
 *
 * Layout, little-endian.  A header, then field-major arrays, each from the next multiple of 16
 * bytes; every padding byte is zero.  C = sizeof(swb_config), H = 56 + C rounded up to 16:
 *
 *   offset   type      count       field
 *   0        char      8           magic "SWBCKPT\0"
 *   8        uint32    1           layout version (1)
 *   12       int32     3           E, K, S (n_envs, pool_depth, n_slots)
 *   24       int32     1           span class: 1 or 4, as swb_save_envs reports it
 *   28       int32     1           1: a device sampler is loaded (swb_sampler_load), else 0
 *   32       uint64    1           its seed (0 without)
 *   40       int64     1           its env_offset (0 without)
 *   48       uint32    1           C
 *   52       zero      4
 *   56       bytes     C           config signature: the engine's swb_config with n_envs, pool_depth
 *                                  and device zeroed
 *   H        double    E*S x 2     pos_x, pos_y
 *   ..       int32     E x 3       cursor, step_count, scene_serial
 *   ..       uint8     E           reset_next
 *   ..       double    E*K*S x 8   the pool: x, y, m00, m01, m10, m11, vx, vy, entry (env, ring
 *                                  slot, slot) at (env * K + ring) * S + slot, as swb_pool_pointers
 *   ..       uint32    E*K*S x 2   member, rgb (r | g << 8 | b << 16)
 *   ..       float     E*K*S*5     factors, 5 per entry
 *   ..       uint8     E*K*S x 2   shape, pos_f32
 *   ..       int64     E           refilled_upto (-1 throughout without a device sampler)
 *   ..       double    E*K*G x 2   goals of every pool entry, as swb_pool_goal_pointer (absent when G = 0;
 *                                  G is part of the signature through the nodes' goal_slot)
 *
 * That is about 94 bytes per pool entry and 16 S + 21 bytes per env; swb_engine_state_bytes()
 * gives the exact size.
 *
 * swb_save_engine copies the state as it stands after the work enqueued on `stream` so far,
 * synchronises that stream and returns when `host_dst` (at least swb_engine_state_bytes() bytes)
 * is complete.  It reads only: no state changes and swb_launch_count does not move.
 *
 * swb_load_engine checks the whole buffer on the host before anything is enqueued, and refuses it,
 * naming the field, the index and the value, for: a wrong magic, version, size, E, K, S or
 * signature; a span class other than 1 or 4; a sampler that disagrees with the engine's (a
 * checkpoint saved with a device sampler loads only into an engine whose loaded sampler has the
 * same seed and env_offset, one saved without only into an engine without); a cursor outside
 * [0, K); scene_serial < 0; refilled_upto < -1; reset_next other than 0 or 1; and a pool shape id
 * >= SWB_NUM_SHAPES or without a vertex table.  A checkpoint is outside input: where record loads
 * sanitise shape ids, this load refuses, since a bad cursor or shape id would make later kernels
 * index out of bounds.  An accepted buffer is copied into the engine on `stream` through a pinned
 * staging block of the engine (the caller may reuse `host_src` when the call returns), and the
 * engine's span class is raised to the saved one, as swb_load_envs raises it.
 *
 * Neither call may run while a scene upload (swb_upload_scenes) or refill of the same engine is
 * in flight on another stream: the caller orders them first (environment.BatchedEnvironment lands
 * its asynchronous refill before it saves or loads).
 */
int64_t swb_engine_state_bytes(const swb_engine *eng);
int swb_save_engine(swb_engine *eng, void *host_dst, uint64_t dst_bytes, void *stream);
int swb_load_engine(swb_engine *eng, const void *host_src, uint64_t src_bytes, void *stream);

/* Number of kernels this library has launched since engine creation. */
int64_t swb_launch_count(const swb_engine *eng);

#ifdef __cplusplus
}
#endif
#endif /* SPRITEWORLD_B200_H_ */
