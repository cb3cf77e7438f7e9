// Rollout kernel: what C candidate action sequences of T steps would earn from a set of root
// states, without changing any env, and optionally the state each plan ends in.
//
// One warp per (root, candidate), warp index w = r * C + c.  A root is either live env r -- its
// current scene, the pool entry at (r, cursor), with the live positions (swb_rollout) -- or record
// r of a device buffer of env records (swb_rollout_states).  The warp stages the root's scene into
// shared memory once and runs T steps of step_kernel's own action, velocity, task and termination
// code (swb_step.cuh) on that copy.  Entry [t][r][c] of the outputs is what Environment.step would
// report at step t; after the plan's first LAST, and for a root about to reset, the entries are
// padding (SWB_STEP_NONE, reward 0, success 0, status 0).
//
// Leaves: when a warp is done (after step T, after the plan's first LAST, or at once for a root
// about to reset) lanes < S write record w: the record swb_save_envs would save of an env that
// started in the root state and took the plan's live steps -- the root's scene, the final
// positions, step_count after the counted steps and reset_next = 1 iff the last of them was LAST.
// Leaves and roots share the record format, so one launch is one level of a search tree.  A leaf
// keeps its root's goals.
//
// Trajectories (swb_rollout_trajectory): record t * R * C + w of io.leaves is the leaf of the same
// plan cut after step t.  Lanes < S write it after each live step, and the warp's final record
// fills the entries after the plan's first LAST (all T of them for a root about to reset).  The
// scene fields come from the root at each write, not from registers held across the step loop.
//
// Actions are [T][R][C][A]: at a step the warps of a CTA read consecutive rows, every lane the
// row of its warp (one broadcast transaction), and the row of step t + 1 is loaded before step t
// is evaluated, so its latency hides behind lane 0's task evaluation.
#pragma once
#include "swb_states.cuh"
#include "swb_step.cuh"

namespace swb {

constexpr int ROLLOUT_WARPS = 4;

// The record buffers of a rollout: roots (n_roots records) unless the roots are the live envs,
// leaves (n_roots * C records, or T * n_roots * C for a trajectory) if asked for.  Each
// instantiation of rollout_kernel reads only the members its template arguments use.
struct RolloutRecords {
  const unsigned char *roots;
  unsigned char *leaves;
  size_t record_bytes;
  int n_roots;
};

// Root record `rec` in the warp's WarpSprites, as stage_sprites stages an env's pool entry with
// its live positions and goals (shape ids sanitised by read_record); *vx, *vy: lane s holds slot s's
// velocity.
__device__ __forceinline__ void stage_record(const DevState &st, WarpSprites &ws, int S,
                                             const unsigned char *rec, int lane, double *vx, double *vy) {
  if (lane < 2 * st.G) ws.goal[lane] = record_goals(rec, S, st.G)[lane];
  *vx = 0.; *vy = 0.;
  if (lane < S) {
    const SlotRecord r = read_record(st, rec, lane);
    ws.shape[lane] = r.shape;
    ws.f32[lane] = r.pos_f32;
    ws.member[lane] = r.member;
    ws.m00[lane] = r.f64[M00]; ws.m01[lane] = r.f64[M01];
    ws.m10[lane] = r.f64[M10]; ws.m11[lane] = r.f64[M11];
    ws.x[lane] = r.f64[POS_X]; ws.y[lane] = r.f64[POS_Y];
    *vx = r.f64[VX]; *vy = r.f64[VY];
  }
  __syncwarp();
}

// Slot `lane` of the record a plan from root e (record `root`, else live env e) has reached: the
// root's slot read now, with the positions in ws, step_count `count` (lane 0's copy is the one
// write_record stores) and reset_next `last` -- unless the root was resetting, which takes no step.
template <bool kRecordRoots>
__device__ __forceinline__ SlotRecord plan_record(const DevState &st, const WarpSprites &ws,
                                                  const unsigned char *root, int e, int lane, bool resetting,
                                                  int count, bool last) {
  SlotRecord r = kRecordRoots ? read_record(st, root, lane) : read_state(st, e, lane);
  if (!resetting) {
    r.f64[POS_X] = ws.x[lane];
    r.f64[POS_Y] = ws.y[lane];
    r.step_count = count;
    r.reset_next = last ? 1 : 0;
  }
  return r;
}

// kRecordRoots: roots are io.roots (else the E live envs); kLeaves: write io.leaves; kTrajectory
// (with kLeaves false): write the T * R * C records of every step into io.leaves.
template <bool kRecordRoots, bool kLeaves, bool kTrajectory = false>
__global__ void __launch_bounds__(ROLLOUT_WARPS * 32)
rollout_kernel(DevState st, const StepCfg *__restrict__ step_cfg, const void *__restrict__ actions,
               int action_dtype, int T, int C, swb_step_out out, RolloutRecords io) {
  const StepCfg &c_step = *step_cfg;
  __shared__ WarpSprites s_ws[ROLLOUT_WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int w = blockIdx.x * ROLLOUT_WARPS + warp;
  // T * R * C fits an int32 (swb_rollout and swb_rollout_states check it)
  const int EC = (kRecordRoots ? io.n_roots : st.E) * C;
  if (w >= EC) return;
  const int e = w / C;
  WarpSprites &ws = s_ws[warp];
  const int S = st.S;
  const RecordLayout L(S);
  const unsigned char *root = kRecordRoots ? io.roots + (size_t)e * io.record_bytes : nullptr;
  // else the env's next step starts another scene: nothing to plan in
  const bool resetting = kRecordRoots ? root[L.reset_next()] != 0 : st.reset_next[e] != 0;
  // a leaf (every trajectory entry) keeps its root's goals: stored now, before the plan keeps
  // registers busy
  if ((kLeaves || kTrajectory) && lane < 2 * st.G) {
    const double g = (kRecordRoots ? record_goals(root, S, st.G) : state_goals(st, e))[lane];
    for (int p = 0; p < (kTrajectory ? T : 1); ++p)
      record_goals(io.leaves + ((size_t)p * EC + w) * io.record_bytes, S, st.G)[lane] = g;
  }
  int t = 0, count = 0;
  bool ended = false;
  if (!resetting) {
    double vx, vy;
    if (kRecordRoots) {
      stage_record(st, ws, S, root, lane, &vx, &vy);
      count = *reinterpret_cast<const int32_t *>(root + L.step_count());
    } else {
      stage_sprites(st, ws, S, e, e * st.K + st.cursor[e], false, lane, &vx, &vy);
      count = st.step_count[e];
    }
    ActionRow next = load_action(actions, action_dtype, (size_t)w);
    while (t < T) {
      const ActionRow row = next;
      if (t + 1 < T) next = load_action(actions, action_dtype, (size_t)(t + 1) * EC + w);
      int status = 0;
      const double cost = apply_action(st, c_step, ws, S, row, action_dtype, lane, &status);
      velocity_update(c_step, ws, S, lane, vx, vy, status);
      int step_type = 0;
      if (lane == 0) {
        double tr, reward;
        int succ;
        task_eval(c_step, ws, S, &tr, &succ, &status);
        step_type = finish_step(c_step, ws, S, action_dtype, cost, tr, succ, status, &count, &reward);
        const size_t i = (size_t)t * EC + w;
        out.reward[i] = reward;
        out.step_type[i] = (int8_t)step_type;
        out.success[i] = (uint8_t)succ;
        out.status[i] = (uint8_t)status;
      }
      step_type = __shfl_sync(0xFFFFFFFFu, step_type, 0);
      if (kTrajectory && lane < S)
        write_record(io.leaves + ((size_t)t * EC + w) * io.record_bytes, S, st.G, lane,
                     plan_record<kRecordRoots>(st, ws, root, e, lane, resetting, count, step_type == SWB_STEP_LAST));
      t++;
      if (step_type == SWB_STEP_LAST) {
        ended = true;
        break;
      }
    }
  }
  for (int p = t + lane; p < T; p += 32) {
    const size_t i = (size_t)p * EC + w;
    out.reward[i] = 0.0;
    out.step_type[i] = (int8_t)SWB_STEP_NONE;
    out.success[i] = 0;
    out.status[i] = 0;
  }
  if (kTrajectory && lane < S && t < T) {
    // the end state repeats: the plan's last record, or the root itself
    const SlotRecord end = plan_record<kRecordRoots>(st, ws, root, e, lane, resetting, count, ended);
    for (int p = t; p < T; ++p) write_record(io.leaves + ((size_t)p * EC + w) * io.record_bytes, S, st.G, lane, end);
  }
  if (kLeaves && lane < S)
    write_record(io.leaves + (size_t)w * io.record_bytes, S, st.G, lane,
                 plan_record<kRecordRoots>(st, ws, root, e, lane, resetting, count, ended));
}

// swb_evaluate_states: the task tree's value on record i (one warp each) at its live positions, with
// row i of `goals` in place of the record's goals when `goals` is not null.  Read-only.
__global__ void __launch_bounds__(ROLLOUT_WARPS * 32)
evaluate_kernel(DevState st, const StepCfg *__restrict__ step_cfg, const unsigned char *__restrict__ recs,
                size_t record_bytes, int n, const double *__restrict__ goals, double *__restrict__ reward,
                uint8_t *__restrict__ success, uint8_t *__restrict__ status) {
  __shared__ WarpSprites s_ws[ROLLOUT_WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * ROLLOUT_WARPS + warp;
  if (i >= n) return;
  WarpSprites &ws = s_ws[warp];
  double vx, vy;
  stage_record(st, ws, st.S, recs + (size_t)i * record_bytes, lane, &vx, &vy);
  if (goals && lane < 2 * st.G) ws.goal[lane] = goals[(size_t)i * 2 * st.G + lane];
  __syncwarp();
  if (lane == 0) {
    double tr;
    int succ, stat = 0;
    task_eval(*step_cfg, ws, st.S, &tr, &succ, &stat);
    reward[i] = tr;
    success[i] = (uint8_t)succ;
    status[i] = (uint8_t)stat;
  }
}

}  // namespace swb
