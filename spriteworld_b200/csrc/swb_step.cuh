// Step kernel: Environment.step minus the renderer, for E envs (environment.py:88-108).
//
// One warp per env.  The env's sprites (<= 32 slots) are staged in shared memory;
// lanes work edge-parallel in the hit tests (sprite.py:113-115 -> matplotlib
// point_in_path, even-odd crossings in fp64), slot-parallel in the velocity update
// (sprite.py:109-111) and lane 0 evaluates the task tree serially, in the reference's
// summation order (tasks.py).  fp64 throughout; float32 where the reference's NumPy
// dtypes make it float32 (App. C of SURVEY.md); no FMA contraction (-fmad=false and
// explicit _rn intrinsics).
#pragma once
#include "swb_device.cuh"

namespace swb {

constexpr int STEP_WARPS = 4;

struct WarpSprites {
  double x[SWB_MAX_SLOTS], y[SWB_MAX_SLOTS];
  double m00[SWB_MAX_SLOTS], m01[SWB_MAX_SLOTS], m10[SWB_MAX_SLOTS], m11[SWB_MAX_SLOTS];
  uint32_t member[SWB_MAX_SLOTS];
  uint8_t shape[SWB_MAX_SLOTS], f32[SWB_MAX_SLOTS];
  double goal[2 * SWB_MAX_GOALS];  // the scene's sampled goals (x, y) per goal slot; G of them staged
};

// numpy pairwise_sum: < 8 sequential, <= 128 eight accumulators
__device__ double np_sum(const double *a, int n) {
  if (n < 8) {
    double res = 0.;
    for (int i = 0; i < n; i++) res = __dadd_rn(res, a[i]);
    return res;
  }
  double r[8];
  int i;
  for (i = 0; i < 8; i++) r[i] = a[i];
  for (i = 8; i < n - (n % 8); i += 8)
    for (int j = 0; j < 8; j++) r[j] = __dadd_rn(r[j], a[i + j]);
  double res = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])),
                         __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
  for (; i < n; i++) res = __dadd_rn(res, a[i]);
  return res;
}

// the same for a float32 array: np.mean of float32 sums in float32
__device__ float np_sum_f32(const float *a, int n) {
  if (n < 8) {
    float res = 0.f;
    for (int i = 0; i < n; i++) res = __fadd_rn(res, a[i]);
    return res;
  }
  float r[8];
  int i;
  for (i = 0; i < 8; i++) r[i] = a[i];
  for (i = 8; i < n - (n % 8); i += 8)
    for (int j = 0; j < 8; j++) r[j] = __fadd_rn(r[j], a[i + j]);
  float res = __fadd_rn(__fadd_rn(__fadd_rn(r[0], r[1]), __fadd_rn(r[2], r[3])),
                        __fadd_rn(__fadd_rn(r[4], r[5]), __fadd_rn(r[6], r[7])));
  for (; i < n; i++) res = __fadd_rn(res, a[i]);
  return res;
}

// X @ Y.T of two 2-feature rows as scikit-learn gets it from OpenBLAS on x86-64 with FMA:
// gemv (cluster of >= 2 points against its centroid) fuses the first product into the second,
// dot (one-point cluster) and gemm (centroid against centroid) the second into the first --
// except, for 12 to 15 centroids, the entries of the first 12 rows and columns that touch rows
// 8..11, which its tail kernel sums unfused.  Products of float32 values are exact in float64,
// so for float32 positions all of these are the plain sum of products (DESIGN.md section 5).
__device__ __forceinline__ double blas_dot2_gemv(double x0, double x1, double y0, double y1) {
  return __fma_rn(x0, y0, __dmul_rn(x1, y1));
}
__device__ __forceinline__ double blas_dot2_dot(double x0, double x1, double y0, double y1) {
  return __fma_rn(x1, y1, __dmul_rn(x0, y0));
}
__device__ __forceinline__ double blas_dot2_gemm(int i, int j, int k, double x0, double x1,
                                                 double y0, double y1) {
  if (k >= 12 && k <= 15 && i < 12 && j < 12 && (i >= 8 || j >= 8))
    return __dadd_rn(__dmul_rn(x0, y0), __dmul_rn(x1, y1));
  return __fma_rn(x1, y1, __dmul_rn(x0, y0));
}

// `point - self.position` (sprite.py:115): float32 subtraction iff both are float32
__device__ __forceinline__ double offset_component(double p, bool p_f32, double q, bool q_f32) {
  if (p_f32 && q_f32) return (double)__fsub_rn((float)p, (float)q);
  return __dsub_rn(p, q);
}

// Warp-cooperative Sprite.contains_point: lane i tests edge i -> i+1 (closing edge included).
__device__ bool warp_contains(const DevState &st, const WarpSprites &ws, int s, double tx,
                              double ty, int lane) {
  const int shape = ws.shape[s];
  const int n = st.shape_n[shape];
  bool toggle = false;
  if (n >= 3 && lane < n) {
    const double *v = st.shape_verts + (size_t)shape * SWB_MAX_VERTS * 2;
    const int j = (lane + 1 == n) ? 0 : lane + 1;
    const double ax = v[2 * lane], ay = v[2 * lane + 1], bx = v[2 * j], by = v[2 * j + 1];
    const double m00 = ws.m00[s], m01 = ws.m01[s], m10 = ws.m10[s], m11 = ws.m11[s];
    const double vx0 = __dadd_rn(__dadd_rn(__dmul_rn(m00, ax), __dmul_rn(m01, ay)), 0.0);
    const double vy0 = __dadd_rn(__dadd_rn(__dmul_rn(m10, ax), __dmul_rn(m11, ay)), 0.0);
    const double vx1 = __dadd_rn(__dadd_rn(__dmul_rn(m00, bx), __dmul_rn(m01, by)), 0.0);
    const double vy1 = __dadd_rn(__dadd_rn(__dmul_rn(m10, bx), __dmul_rn(m11, by)), 0.0);
    const bool yf0 = vy0 >= ty, yf1 = vy1 >= ty;
    if (yf0 != yf1) {
      const double lhs = __dmul_rn(__dsub_rn(vy1, ty), __dsub_rn(vx0, vx1));
      const double rhs = __dmul_rn(__dsub_rn(vx1, tx), __dsub_rn(vy0, vy1));
      toggle = ((lhs >= rhs) == yf1);
    }
  }
  const unsigned b = __ballot_sync(0xFFFFFFFFu, toggle);
  return (__popc(b) & 1) != 0;
}

// Sprite.move (sprite.py:103-107)
__device__ __forceinline__ void sprite_move(WarpSprites &ws, int s, double mx, double my, bool keep) {
  double nx = __dadd_rn(ws.x[s], mx), ny = __dadd_rn(ws.y[s], my);
  if (ws.f32[s]) {
    nx = (double)(float)nx;
    ny = (double)(float)ny;
  }
  if (keep) {
    nx = nx < 0.0 ? 0.0 : (nx > 1.0 ? 1.0 : nx);
    ny = ny < 0.0 ? 0.0 : (ny > 1.0 ? 1.0 : ny);
  }
  ws.x[s] = nx;
  ws.y[s] = ny;
}

struct TaskVal {
  double reward;
  int success;
};

// tasks.py:126-158.  The goal is the node's constant, or for goal_slot >= 0 the env's staged goal:
// the same arithmetic on another operand, so an env whose goal is (gx, gy) gets the value of the
// constant-goal node with goal = {gx, gy}.
__device__ TaskVal find_goal(const swb_task_node &nd, const WarpSprites &ws, int S) {
  double rewards[SWB_MAX_SLOTS];
  int n = 0;
  bool all_nonneg = true;
  for (int s = 0; s < S; s++) {
    if (!ws.shape[s]) continue;
    if (nd.filter_slot >= 0 && !((ws.member[s] >> nd.filter_slot) & 1u)) continue;
    const int g = nd.goal_slot;
    const double gx = g >= 0 ? ws.goal[2 * g] : nd.goal[0], gy = g >= 0 ? ws.goal[2 * g + 1] : nd.goal[1];
    const double dx = __dsub_rn(ws.x[s], gx), dy = __dsub_rn(ws.y[s], gy);
    const double t0 = __dmul_rn(nd.weights[0], __dmul_rn(dx, dx));
    const double t1 = __dmul_rn(nd.weights[1], __dmul_rn(dy, dy));
    const double tot = __dadd_rn(__dadd_rn(0., t0), t1);
    // the reference computes np.float64 ** 0.5 = libm pow(x, .5); sqrt is the correctly
    // rounded value and differs from glibc's pow in ~0.08% of inputs by 1 ULP (DESIGN.md)
    const double dist = sqrt(tot);
    const double r = __dmul_rn(nd.raw_reward_multiplier, __dsub_rn(nd.terminate_distance, dist));
    if (!(r >= 0)) all_nonneg = false;
    rewards[n++] = r;
  }
  TaskVal out;
  out.success = all_nonneg;
  if (n == 0) {
    out.reward = nan("");
    return out;
  }
  const double dense = np_sum(rewards, n);
  double reward = 0.;
  if (all_nonneg) {
    reward = __dadd_rn(reward, nd.terminate_bonus);
    reward = __dadd_rn(reward, dense);
  } else if (!nd.sparse_reward) {
    reward = __dadd_rn(reward, dense);
  }
  out.reward = reward;
  return out;
}

// sklearn.metrics.davies_bouldin_score as called from tasks.py:207-215, with the float32
// intermediate roundings scikit-learn applies to float32 positions.
__device__ int davies_bouldin_metric(const double *px, const double *py, const int *label, int n,
                                     int n_clusters, bool all_f32, double *metric) {
  bool present[SWB_MAX_CHILDREN];
  int relabel[SWB_MAX_CHILDREN];
  int k = 0;
  for (int c = 0; c < n_clusters; c++) {
    present[c] = false;
    for (int i = 0; i < n; i++) if (label[i] == c) present[c] = true;
    relabel[c] = present[c] ? k++ : -1;
  }
  if (!(1 < k && k < n)) return SWB_ENV_CLUSTER_LABELS;
  double cen[SWB_MAX_CHILDREN][2], intra[SWB_MAX_CHILDREN];
  for (int c = 0; c < n_clusters; c++) {
    if (!present[c]) continue;
    const int kk = relabel[c];
    int cnt = 0;
    double cx, cy, mean_d;
    if (all_f32) {
      float sx = 0.f, sy = 0.f;
      bool first = true;
      for (int i = 0; i < n; i++) {
        if (label[i] != c) continue;
        if (first) { sx = (float)px[i]; sy = (float)py[i]; first = false; }
        else { sx = __fadd_rn(sx, (float)px[i]); sy = __fadd_rn(sy, (float)py[i]); }
        cnt++;
      }
      cx = (double)__fdiv_rn(sx, (float)cnt);
      cy = (double)__fdiv_rn(sy, (float)cnt);
      float dist[SWB_MAX_SLOTS];
      int m = 0;
      const double yy = __dadd_rn(__dmul_rn(cx, cx), __dmul_rn(cy, cy));
      for (int i = 0; i < n; i++) {
        if (label[i] != c) continue;
        const double xx = __dadd_rn(__dmul_rn(px[i], px[i]), __dmul_rn(py[i], py[i]));
        double d = __dmul_rn(-2.0, blas_dot2_gemv(px[i], py[i], cx, cy));
        d = __dadd_rn(d, xx);
        d = __dadd_rn(d, yy);
        float df = (float)d;
        if (df < 0.f) df = 0.f;
        dist[m++] = __fsqrt_rn(df);
      }
      mean_d = (double)__fdiv_rn(np_sum_f32(dist, m), (float)cnt);
    } else {
      double sx = 0., sy = 0.;
      bool first = true;
      for (int i = 0; i < n; i++) {
        if (label[i] != c) continue;
        if (first) { sx = px[i]; sy = py[i]; first = false; }
        else { sx = __dadd_rn(sx, px[i]); sy = __dadd_rn(sy, py[i]); }
        cnt++;
      }
      cx = __ddiv_rn(sx, (double)cnt);
      cy = __ddiv_rn(sy, (double)cnt);
      double dist[SWB_MAX_SLOTS];
      int m = 0;
      const double yy = __dadd_rn(__dmul_rn(cx, cx), __dmul_rn(cy, cy));
      for (int i = 0; i < n; i++) {
        if (label[i] != c) continue;
        const double xx = __dadd_rn(__dmul_rn(px[i], px[i]), __dmul_rn(py[i], py[i]));
        const double dot = cnt == 1 ? blas_dot2_dot(px[i], py[i], cx, cy)
                                    : blas_dot2_gemv(px[i], py[i], cx, cy);
        double d = __dmul_rn(-2.0, dot);
        d = __dadd_rn(d, xx);
        d = __dadd_rn(d, yy);
        if (d < 0.) d = 0.;
        dist[m++] = __dsqrt_rn(d);
      }
      mean_d = __ddiv_rn(np_sum(dist, m), (double)cnt);
    }
    cen[kk][0] = cx; cen[kk][1] = cy; intra[kk] = mean_d;
  }
  bool all_intra_zero = true, all_cd_zero = true;
  for (int i = 0; i < k; i++) if (!(fabs(intra[i]) <= 1e-8)) all_intra_zero = false;
  double cd[SWB_MAX_CHILDREN][SWB_MAX_CHILDREN];
  for (int i = 0; i < k; i++) {
    const double xi = __dadd_rn(__dmul_rn(cen[i][0], cen[i][0]), __dmul_rn(cen[i][1], cen[i][1]));
    for (int j = 0; j < k; j++) {
      const double xj = __dadd_rn(__dmul_rn(cen[j][0], cen[j][0]), __dmul_rn(cen[j][1], cen[j][1]));
      double d = __dmul_rn(-2.0, blas_dot2_gemm(i, j, k, cen[i][0], cen[i][1], cen[j][0], cen[j][1]));
      d = __dadd_rn(d, xi);
      d = __dadd_rn(d, xj);
      if (d < 0.) d = 0.;
      if (i == j) d = 0.;
      cd[i][j] = __dsqrt_rn(d);
      if (!(fabs(cd[i][j]) <= 1e-8)) all_cd_zero = false;
    }
  }
  if (all_intra_zero || all_cd_zero) return SWB_ENV_CLUSTER_ZERODIV;
  double scores[SWB_MAX_CHILDREN];
  for (int i = 0; i < k; i++) {
    double best = -INFINITY;
    for (int j = 0; j < k; j++) {
      const double dd = cd[i][j] == 0 ? INFINITY : cd[i][j];
      const double v = __ddiv_rn(__dadd_rn(intra[i], intra[j]), dd);
      if (v > best) best = v;
    }
    scores[i] = best;
  }
  const double score = __ddiv_rn(np_sum(scores, k), (double)k);
  if (score == 0.0) return SWB_ENV_CLUSTER_ZERODIV;
  *metric = __ddiv_rn(1., score);
  return SWB_ENV_OK;
}

// tasks.py:196-245
__device__ TaskVal clustering(const swb_task_node &nd, const WarpSprites &ws, int S, int *status) {
  double px[SWB_MAX_SLOTS], py[SWB_MAX_SLOTS];
  int label[SWB_MAX_SLOTS];
  int n = 0;
  bool all_f32 = true;
  for (int s = 0; s < S; s++) {
    if (!ws.shape[s]) continue;
    int lab = -1;
    for (int c = 0; c < nd.n_clusters; c++) {
      if ((ws.member[s] >> nd.cluster_slots[c]) & 1u) { lab = c; break; }
    }
    if (!ws.f32[s]) all_f32 = false;
    if (lab < 0) continue;
    px[n] = ws.x[s]; py[n] = ws.y[s]; label[n] = lab; n++;
  }
  TaskVal out;
  double metric = 0.;
  const int err = davies_bouldin_metric(px, py, label, n, nd.n_clusters, all_f32, &metric);
  if (err) {
    *status |= err;
    out.reward = nan("");
    out.success = 0;
    return out;
  }
  const double dense = __ddiv_rn(__dmul_rn(__dsub_rn(metric, nd.termination_threshold), nd.reward_range), 2.);
  double reward = 0.;
  out.success = metric >= nd.termination_threshold;
  if (out.success) {
    reward = __dadd_rn(reward, nd.terminate_bonus);
    reward = __dadd_rn(reward, dense);
  } else if (!nd.sparse_reward) {
    reward = __dadd_rn(reward, dense);
  }
  out.reward = reward;
  return out;
}

// whole task tree; root = last node (tasks.py:288-296 for MetaAggregated)
__device__ void task_eval(const StepCfg &c_step, const WarpSprites &ws, int S, double *reward,
                          int *success, int *status) {
  TaskVal val[SWB_MAX_NODES];
  const int nn = c_step.n_nodes;
  for (int i = 0; i < nn; i++) {
    const swb_task_node &nd = c_step.nodes[i];
    if (nd.kind == SWB_TASK_FIND_GOAL) {
      val[i] = find_goal(nd, ws, S);
    } else if (nd.kind == SWB_TASK_CLUSTERING) {
      val[i] = clustering(nd, ws, S, status);
    } else if (nd.kind == SWB_TASK_META) {
      double r[SWB_MAX_CHILDREN];
      int cnt_nonnan = 0;
      bool all_s = true, any_s = false;
      const int nc = nd.n_children;
      for (int c = 0; c < nc; c++) {
        const TaskVal cv = val[nd.children[c]];
        r[c] = cv.reward;
        if (!isnan(cv.reward)) cnt_nonnan++;
        all_s = all_s && cv.success;
        any_s = any_s || cv.success;
      }
      double agg;
      if (nd.aggregator == SWB_AGG_SUM || nd.aggregator == SWB_AGG_MEAN) {
        double z[SWB_MAX_CHILDREN];
        for (int c = 0; c < nc; c++) z[c] = isnan(r[c]) ? 0. : r[c];
        agg = np_sum(z, nc);
        if (nd.aggregator == SWB_AGG_MEAN) agg = cnt_nonnan ? __ddiv_rn(agg, (double)cnt_nonnan) : nan("");
      } else {
        agg = nan("");
        for (int c = 0; c < nc; c++) {
          if (isnan(r[c])) continue;
          if (isnan(agg)) agg = r[c];
          else if (nd.aggregator == SWB_AGG_MAX) agg = r[c] > agg ? r[c] : agg;
          else agg = r[c] < agg ? r[c] : agg;
        }
      }
      const int succ = nd.criterion == SWB_CRIT_ALL ? all_s : any_s;
      agg = __dadd_rn(agg, __dmul_rn(nd.terminate_bonus, (double)succ));
      val[i].reward = agg;
      val[i].success = succ;
    } else {
      val[i].reward = 0.0;
      val[i].success = 0;
    }
  }
  *reward = val[nn - 1].reward;
  *success = val[nn - 1].success;
}

// One env's row of `actions` in registers, as raw 32-bit words: 2 of an int32 row, 4 of a float32
// row, 8 of a float64 row.
struct ActionRow {
  uint32_t w[8];
};

__device__ __forceinline__ ActionRow load_action(const void *__restrict__ actions, int action_dtype,
                                                 size_t row) {
  ActionRow r = {};
  if (action_dtype == SWB_DTYPE_I32) {
    const int32_t *a = reinterpret_cast<const int32_t *>(actions) + 2 * row;
    r.w[0] = (uint32_t)a[0]; r.w[1] = (uint32_t)a[1];
  } else if (action_dtype == SWB_DTYPE_F32) {
    const float *a = reinterpret_cast<const float *>(actions) + 4 * row;
    for (int i = 0; i < 4; i++) r.w[i] = __float_as_uint(a[i]);
  } else {
    const double *a = reinterpret_cast<const double *>(actions) + 4 * row;
    for (int i = 0; i < 4; i++) {
      r.w[2 * i] = (uint32_t)__double2loint(a[i]);
      r.w[2 * i + 1] = (uint32_t)__double2hiint(a[i]);
    }
  }
  return r;
}

// action_space.step of one action on the warp's sprites (every lane calls it): moves the clicked /
// carried / body sprite, returns the action's cost; a bad Embodied direction sets
// SWB_ENV_BAD_ACTION in *status and moves nothing.  The warp is synchronised on return.
__device__ __forceinline__ double apply_action(const DevState &st, const StepCfg &c_step, WarpSprites &ws,
                                               int S, const ActionRow &row, int action_dtype, int lane,
                                               int *status) {
  double cost = 0.;
  const bool keep = c_step.keep_in_frame != 0;
  if (c_step.action_kind == SWB_ACT_EMBODIED) {  // action_spaces.py:187-214
    const bool carry = row.w[0] != 0;
    const int dir = (int)row.w[1];
    const double step = c_step.action_scale;
    double mx = 0., my = 0.;
    if (dir == 0) my = step;
    else if (dir == 1) mx = -step;
    else if (dir == 2) my = -step;
    else if (dir == 3) mx = step;
    else *status |= SWB_ENV_BAD_ACTION;
    if (!(*status & SWB_ENV_BAD_ACTION)) {
      const int body = S - 1;
      if (carry) {  // :180-185
        for (int s = body - 1; s >= 0; s--) {
          if (!ws.shape[s]) continue;
          const double tx = offset_component(ws.x[body], ws.f32[body], ws.x[s], ws.f32[s]);
          const double ty = offset_component(ws.y[body], ws.f32[body], ws.y[s], ws.f32[s]);
          if (warp_contains(st, ws, s, tx, ty, lane)) {
            __syncwarp();  // every lane is done reading the pose lane 0 overwrites
            if (lane == 0) sprite_move(ws, s, mx, my, keep);
            break;
          }
        }
        __syncwarp();
      }
      if (lane == 0) sprite_move(ws, body, mx, my, keep);
      cost = __dmul_rn(-c_step.motion_cost, c_step.action_scale);
    }
  } else {  // SelectMove :83-104 / DragAndDrop :133-137
    double px, py, mx, my, norm;
    const bool af32 = action_dtype == SWB_DTYPE_F32;
    if (af32) {
      float a[4];
      for (int i = 0; i < 4; i++) a[i] = __uint_as_float(row.w[i]);
      const float fsc = (float)c_step.action_scale;
      float d0, d1;
      if (c_step.action_kind == SWB_ACT_SELECT_MOVE) {
        d0 = __fsub_rn(a[2], 0.5f); d1 = __fsub_rn(a[3], 0.5f);
      } else {
        d0 = __fsub_rn(a[2], a[0]); d1 = __fsub_rn(a[3], a[1]);
      }
      const float m0 = __fmul_rn(d0, fsc), m1 = __fmul_rn(d1, fsc);
      px = a[0]; py = a[1]; mx = m0; my = m1;
      norm = (double)__fsqrt_rn(__fadd_rn(__fmul_rn(m0, m0), __fmul_rn(m1, m1)));
    } else {
      double a[4];
      for (int i = 0; i < 4; i++) a[i] = __hiloint2double((int)row.w[2 * i + 1], (int)row.w[2 * i]);
      if (c_step.action_kind == SWB_ACT_SELECT_MOVE) {
        mx = __dmul_rn(__dsub_rn(a[2], 0.5), c_step.action_scale);
        my = __dmul_rn(__dsub_rn(a[3], 0.5), c_step.action_scale);
      } else {
        mx = __dmul_rn(__dsub_rn(a[2], a[0]), c_step.action_scale);
        my = __dmul_rn(__dsub_rn(a[3], a[1]), c_step.action_scale);
      }
      px = a[0]; py = a[1];
      // np.linalg.norm of a float64 2-vector is sqrt(x.dot(x)), and OpenBLAS ddot fuses the
      // second product into the first: fma(my, my, mx * mx) (DESIGN.md section 5)
      norm = __dsqrt_rn(__fma_rn(my, my, __dmul_rn(mx, mx)));
    }
    for (int s = S - 1; s >= 0; s--) {  // :77-81 top-most first
      if (!ws.shape[s]) continue;
      const double tx = offset_component(px, af32, ws.x[s], ws.f32[s]);
      const double ty = offset_component(py, af32, ws.y[s], ws.f32[s]);
      if (warp_contains(st, ws, s, tx, ty, lane)) {
        __syncwarp();
        if (lane == 0) sprite_move(ws, s, mx, my, keep);
        break;
      }
    }
    if (af32) cost = (double)__fmul_rn((float)(-c_step.motion_cost), (float)norm);
    else cost = __dmul_rn(-c_step.motion_cost, norm);
  }
  __syncwarp();
  return cost;
}

// velocity update of every sprite (environment.py:98-99), slot-parallel; the reference's KeyError
// skips it.  The warp is synchronised on return.
__device__ __forceinline__ void velocity_update(const StepCfg &c_step, WarpSprites &ws, int S, int lane,
                                                double vx, double vy, int status) {
  if (!(status & SWB_ENV_BAD_ACTION) && lane < S && ws.shape[lane])
    sprite_move(ws, lane, vx, vy, c_step.keep_in_frame != 0);
  __syncwarp();
}

// The end of Environment.step for one env (one lane calls it) after its action, velocity update
// and task: counts the step in *count, returns the step type and sets *reward.
__device__ __forceinline__ int finish_step(const StepCfg &c_step, const WarpSprites &ws, int S,
                                           int action_dtype, double cost, double tr, int succ,
                                           int status, int *count, double *reward) {
  *count += 1;  // :93
  if (status & SWB_ENV_BAD_ACTION) {
    // the reference's state after the KeyError: the step is counted (:93), nothing moved
    *reward = nan("");
    return SWB_STEP_MID;
  }
  bool oof = false;
  for (int s = 0; s < S; s++) {
    if (!ws.shape[s]) continue;
    if (!((ws.x[s] >= 0.0 && ws.y[s] >= 0.0) && (ws.x[s] <= 1.0 && ws.y[s] <= 1.0))) oof = true;
  }
  const bool timeout = *count >= c_step.max_episode_length;  // :84
  // :101.  A float32 click costs an np.float32; Clustering's reward is a Python float, so
  // NumPy 2 adds the two in float32.  Every other root returns np.float64 (or 0.0, which
  // leaves the float32 cost unchanged either way).
  const bool f32_sum = action_dtype == SWB_DTYPE_F32 && c_step.action_kind != SWB_ACT_EMBODIED &&
                       c_step.nodes[c_step.n_nodes - 1].kind == SWB_TASK_CLUSTERING;
  *reward = f32_sum ? (double)__fadd_rn((float)cost, (float)tr) : __dadd_rn(cost, tr);
  return (succ || oof || timeout) ? SWB_STEP_LAST : SWB_STEP_MID;
}

// The env's current scene -- pool entry `entry` = e * K + ring slot -- in the warp's WarpSprites, with
// the pool's initial positions (`from_pool`) or the live ones, and its goals; *vx, *vy: lane s holds
// slot s's velocity.
__device__ __forceinline__ void stage_sprites(const DevState &st, WarpSprites &ws, int S, int e, int entry,
                                              bool from_pool, int lane, double *vx, double *vy) {
  const int scene0 = entry * S;
  if (lane < 2 * st.G) ws.goal[lane] = st.p_goal[(size_t)entry * st.G * 2 + lane];
  *vx = 0.; *vy = 0.;
  if (lane < S) {
    const int sc = scene0 + lane;
    ws.shape[lane] = st.p_shape[sc];
    ws.f32[lane] = st.p_pos_f32[sc];
    ws.member[lane] = st.p_member[sc];
    ws.m00[lane] = st.p_m00[sc]; ws.m01[lane] = st.p_m01[sc];
    ws.m10[lane] = st.p_m10[sc]; ws.m11[lane] = st.p_m11[sc];
    if (from_pool) {
      ws.x[lane] = st.p_x[sc]; ws.y[lane] = st.p_y[sc];
    } else {
      ws.x[lane] = st.pos_x[e * S + lane]; ws.y[lane] = st.pos_y[e * S + lane];
      *vx = st.p_vx[sc]; *vy = st.p_vy[sc];
    }
  }
  __syncwarp();
}

__global__ void __launch_bounds__(STEP_WARPS * 32)
step_kernel(DevState st, const StepCfg *__restrict__ step_cfg, const void *__restrict__ actions,
            int action_dtype, swb_step_out out, int mode) {
  // the engine's own copy of the action space / episode / task tree, in global memory: a
  // kernel of engine A queued behind a launch of engine B still reads A's table
  const StepCfg &c_step = *step_cfg;
  // the render kernel that follows on the stream may start to become resident (it waits for
  // this grid to complete before it reads anything a step writes)
  asm volatile("griddepcontrol.launch_dependents;");
  // mode 0: Environment.step; 1: task.reward/success of the live state only;
  // 2: action_space.step only (no velocity update, task or counters)
  __shared__ WarpSprites s_ws[STEP_WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int e = blockIdx.x * STEP_WARPS + warp;
  if (e >= st.E) return;
  WarpSprites &ws = s_ws[warp];
  const int S = st.S;
  const bool resetting = mode == 0 && st.reset_next[e] != 0;
  int cursor = st.cursor[e];
  if (resetting) cursor = (cursor + 1) % st.K;  // environment.py:90-91 -> reset() :74-78
  double vx, vy;
  stage_sprites(st, ws, S, e, e * st.K + cursor, resetting, lane, &vx, &vy);

  double cost = 0.;
  int status = 0;
  if (!resetting && mode != 1) {
    cost = apply_action(st, c_step, ws, S, load_action(actions, action_dtype, (size_t)e), action_dtype,
                        lane, &status);
    if (mode == 0) velocity_update(c_step, ws, S, lane, vx, vy, status);
  }

  if (mode != 1 && lane < S) {
    st.pos_x[e * S + lane] = ws.x[lane];
    st.pos_y[e * S + lane] = ws.y[lane];
  }
  if (mode == 2) {
    if (lane == 0) {
      out.reward[e] = cost;
      out.step_type[e] = (int8_t)SWB_STEP_MID;
      out.success[e] = 0;
      out.status[e] = (uint8_t)status;
    }
    return;
  }
  if (lane == 0) {
    double tr;
    int succ;
    task_eval(c_step, ws, S, &tr, &succ, &status);
    if (mode == 1) {
      out.reward[e] = tr;
      out.step_type[e] = (int8_t)SWB_STEP_MID;
      out.success[e] = (uint8_t)succ;
      out.status[e] = (uint8_t)status;
      return;
    }
    int step_type = SWB_STEP_FIRST;
    int count = 0;
    double reward = 0.0;
    if (!resetting) {
      count = st.step_count[e];
      step_type = finish_step(c_step, ws, S, action_dtype, cost, tr, succ, status, &count, &reward);
    }
    out.reward[e] = reward;
    st.cursor[e] = cursor;
    if (resetting) st.scene_serial[e] += 1;  // monotonic: the host's refill bookkeeping reads it
    st.step_count[e] = count;
    st.reset_next[e] = (step_type == SWB_STEP_LAST) ? 1 : 0;
    out.step_type[e] = (int8_t)step_type;
    out.success[e] = (uint8_t)succ;
    out.status[e] = (uint8_t)status;
  }
}

// sets the reset flag of every env (mask == nullptr) or of the masked ones
__global__ void request_reset_kernel(DevState st, const uint8_t *__restrict__ mask) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e < st.E && (mask == nullptr || mask[e])) st.reset_next[e] = 1;
}

}  // namespace swb
