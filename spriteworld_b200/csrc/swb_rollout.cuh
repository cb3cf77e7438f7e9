// Rollout kernel: what C candidate action sequences of T steps would earn from the state every
// env is in now, without changing that state.
//
// One warp per (env, candidate), warp index w = e * C + c.  The warp stages the env's current
// scene -- the pool entry at (e, cursor) with the live positions -- into shared memory once and
// runs T steps of step_kernel's own action, velocity, task and termination code
// (swb_step.cuh) on that copy.  Entry [t][e][c] of the outputs is what Environment.step would
// report at step t; after the plan's first LAST, and for an env about to reset, the entries are
// padding (SWB_STEP_NONE, reward 0, success 0, status 0).  The kernel writes the outputs only.
//
// Actions are [T][E][C][A]: at a step the warps of a CTA read consecutive rows, every lane the
// row of its warp (one broadcast transaction), and the row of step t + 1 is loaded before step t
// is evaluated, so its latency hides behind lane 0's task evaluation.
#pragma once
#include "swb_step.cuh"

namespace swb {

constexpr int ROLLOUT_WARPS = 4;

__global__ void __launch_bounds__(ROLLOUT_WARPS * 32)
rollout_kernel(DevState st, const StepCfg *__restrict__ step_cfg, const void *__restrict__ actions,
               int action_dtype, int T, int C, swb_step_out out) {
  const StepCfg &c_step = *step_cfg;
  __shared__ WarpSprites s_ws[ROLLOUT_WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int w = blockIdx.x * ROLLOUT_WARPS + warp;
  const int EC = st.E * C;  // T * E * C fits an int32 (swb_rollout checks it)
  if (w >= EC) return;
  const int e = w / C;
  WarpSprites &ws = s_ws[warp];
  const int S = st.S;
  int t = 0;
  if (!st.reset_next[e]) {  // else the env's next step starts another scene: nothing to plan in
    double vx, vy;
    stage_sprites(st, ws, S, e, (e * st.K + st.cursor[e]) * S, false, lane, &vx, &vy);
    int count = st.step_count[e];
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
      t++;
      if (step_type == SWB_STEP_LAST) break;
    }
  }
  for (int p = t + lane; p < T; p += 32) {
    const size_t i = (size_t)p * EC + w;
    out.reward[i] = 0.0;
    out.step_type[i] = (int8_t)SWB_STEP_NONE;
    out.success[i] = 0;
    out.status[i] = 0;
  }
}

}  // namespace swb
