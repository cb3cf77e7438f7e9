/*
 * ORACLE (test infrastructure, not product code) -- CPU restatement of the reference's
 * Environment.step() hot path, one env at a time, plus a batch driver with the same
 * scene-pool auto-reset protocol the GPU engine uses.  Every function cites the
 * reference file:line it follows (paths relative to /root/reference/spriteworld/).
 *
 * Pinned by tests/test_oracle_env.py against the tests/golden fixtures, which were generated
 * by running the UNMODIFIED reference (tests/golden/make_golden.py, via oracle/refshim).
 * matplotlib is absent from this image, so hit tests / vertex transforms of the
 * reference run through oracle/refshim/standins/matplotlib (a restatement of
 * matplotlib's C++ point_in_path / affine_transform); that residual risk is stated in
 * DESIGN.md.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's CPU-baseline/reference arm may
 * load this library.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "sw_oracle.h"

#define SWO_API __attribute__((visibility("default")))
#define SWO_MAX_SLOTS_CLUSTER 256 /* sprites one Clustering node looks at */

void swo_polygon_fill(uint8_t *canvas, int W, int H, const double *xy, int n, const uint8_t *rgb,
                      int corner_join);
void swo_lanczos_resize(const uint8_t *in, int inW, int inH, uint8_t *out, int outW, int outH,
                        uint8_t *tmp_h);

/* ---- numpy reductions ---------------------------------------------------- */

/* numpy pairwise_sum (umath loops): < 8 sequential; <= 128 eight accumulators. */
static double np_sum(const double *a, int n) {
  if (n < 8) {
    double res = 0.;
    for (int i = 0; i < n; i++) res += a[i];
    return res;
  }
  if (n <= 128) {
    double r[8];
    int i;
    for (i = 0; i < 8; i++) r[i] = a[i];
    for (i = 8; i < n - (n % 8); i += 8)
      for (int j = 0; j < 8; j++) r[j] += a[i + j];
    double res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
    for (; i < n; i++) res += a[i];
    return res;
  }
  int n2 = n / 2;
  n2 -= n2 % 8;
  return np_sum(a, n2) + np_sum(a + n2, n - n2);
}

/* the same for a float32 array: np.mean of float32 sums in float32 */
static float np_sum_f32(const float *a, int n) {
  if (n > 128) {
    int n2 = n / 2;
    n2 -= n2 % 8;
    volatile float s = np_sum_f32(a, n2) + np_sum_f32(a + n2, n - n2);
    return s;
  }
  if (n < 8) {
    volatile float res = 0.f;
    for (int i = 0; i < n; i++) res = res + a[i];
    return res;
  }
  volatile float r[8];
  int i;
  for (i = 0; i < 8; i++) r[i] = a[i];
  for (i = 8; i < n - (n % 8); i += 8)
    for (int j = 0; j < 8; j++) r[j] = r[j] + a[i + j];
  volatile float r01 = r[0] + r[1], r23 = r[2] + r[3], r45 = r[4] + r[5], r67 = r[6] + r[7];
  volatile float lo = r01 + r23, hi = r45 + r67;
  volatile float res = lo + hi;
  for (; i < n; i++) res = res + a[i];
  return res;
}

/* ---- colour map: renderers/color_maps.py:26-28 -------------------------- */

/* colorsys.hsv_to_rgb evaluated in float32 (numpy float32 scalars stay float32),
 * then (255 * np.array(rgb)).astype(np.uint8) -> truncation. */
SWO_API void swo_hsv_to_rgb_f32(float h, float s, float v, uint8_t *out) {
  volatile float r, g, b;
  if (s == 0.0f) {
    r = g = b = v;
  } else {
    volatile float h6 = h * 6.0f;
    int i = (int)h6;
    volatile float f = h6 - (float)i;
    volatile float one_s = 1.0f - s;
    volatile float p = v * one_s;
    volatile float sf = s * f;
    volatile float one_sf = 1.0f - sf;
    volatile float q = v * one_sf;
    volatile float one_f = 1.0f - f;
    volatile float s1f = s * one_f;
    volatile float one_s1f = 1.0f - s1f;
    volatile float t = v * one_s1f;
    i = i % 6;
    switch (i) {
      case 0: r = v; g = t; b = p; break;
      case 1: r = q; g = v; b = p; break;
      case 2: r = p; g = v; b = t; break;
      case 3: r = p; g = q; b = v; break;
      case 4: r = t; g = p; b = v; break;
      default: r = v; g = p; b = q; break;
    }
  }
  volatile float r255 = 255.0f * r, g255 = 255.0f * g, b255 = 255.0f * b;
  out[0] = (uint8_t)(int)r255;
  out[1] = (uint8_t)(int)g255;
  out[2] = (uint8_t)(int)b255;
}

SWO_API void swo_hsv_to_rgb_f64(double h, double s, double v, uint8_t *out) {
  double r, g, b;
  if (s == 0.0) {
    r = g = b = v;
  } else {
    double h6 = h * 6.0;
    int i = (int)h6;
    double f = h6 - i;
    double p = v * (1.0 - s);
    double q = v * (1.0 - s * f);
    double t = v * (1.0 - s * (1.0 - f));
    i = i % 6;
    switch (i) {
      case 0: r = v; g = t; b = p; break;
      case 1: r = q; g = v; b = p; break;
      case 2: r = p; g = v; b = t; break;
      case 3: r = p; g = q; b = v; break;
      case 4: r = t; g = p; b = v; break;
      default: r = v; g = p; b = q; break;
    }
  }
  out[0] = (uint8_t)(int)(255 * r);
  out[1] = (uint8_t)(int)(255 * g);
  out[2] = (uint8_t)(int)(255 * b);
}

/* ---- sprite geometry: sprite.py ------------------------------------------ */

/* sprite.py:96-101 -- centred path vertex i: (m00*x + m01*y) + 0, (m10*x + m11*y) + 0 */
static void centred_vertex(const swo_shape_table *tab, const swo_sprite *sp, int i, double *cx,
                           double *cy) {
  double vx = tab->verts[sp->shape][i][0], vy = tab->verts[sp->shape][i][1];
  *cx = (sp->m00 * vx + sp->m01 * vy) + 0.0;
  *cy = (sp->m10 * vx + sp->m11 * vy) + 0.0;
}

/* sprite.py:113-115 via matplotlib point_in_path: even-odd crossings, float64.
 * (tx, ty) = point - position, already formed by the caller in the right dtype. */
SWO_API int swo_contains_offset(const swo_shape_table *tab, const swo_sprite *sp, double tx,
                                double ty) {
  int n = tab->n_verts[sp->shape];
  if (n < 3) return 0;
  double sx, sy;
  centred_vertex(tab, sp, 0, &sx, &sy);
  double vx0 = sx, vy0 = sy;
  int yflag0 = vy0 >= ty;
  int inside = 0;
  for (int i = 1; i <= n; i++) {
    double vx1, vy1;
    if (i < n) centred_vertex(tab, sp, i, &vx1, &vy1);
    else { vx1 = sx; vy1 = sy; }
    int yflag1 = vy1 >= ty;
    if (yflag0 != yflag1) {
      if (((vy1 - ty) * (vx0 - vx1) >= (vx1 - tx) * (vy0 - vy1)) == yflag1) inside = !inside;
    }
    yflag0 = yflag1;
    vx0 = vx1;
    vy0 = vy1;
  }
  return inside;
}

/* `point - self.position` (sprite.py:115): float32 subtraction iff both are float32 */
static double offset_component(double p, int p_f32, double q, int q_f32) {
  if (p_f32 && q_f32) {
    volatile float d = (float)p - (float)q;
    return (double)d;
  }
  return p - q;
}

/* sprite.py:103-107 */
static void sprite_move(swo_sprite *sp, double mx, double my, int keep_in_frame) {
  double nx = sp->x + mx, ny = sp->y + my;
  if (sp->pos_f32) {
    nx = (double)(float)nx;
    ny = (double)(float)ny;
  }
  if (keep_in_frame) { /* np.clip(pos, 0.0, 1.0) */
    nx = nx < 0.0 ? 0.0 : (nx > 1.0 ? 1.0 : nx);
    ny = ny < 0.0 ? 0.0 : (ny > 1.0 ? 1.0 : ny);
  }
  sp->x = nx;
  sp->y = ny;
}

/* sprite.py:135-138 */
static int out_of_frame(const swo_sprite *sp) {
  return !((sp->x >= 0.0 && sp->y >= 0.0) && (sp->x <= 1.0 && sp->y <= 1.0));
}

/* ---- action spaces: action_spaces.py ------------------------------------- */

/* returns 0 ok, 1 = KeyError (bad Embodied action).  moved[0..1]: slots moved (-1 none). */
SWO_API int swo_action_step(const swo_env_cfg *cfg, const swo_shape_table *tab, swo_sprite *sp,
                            int S, const void *action, int action_is_f32, double *cost,
                            int *moved) {
  moved[0] = moved[1] = -1;
  int keep = cfg->keep_in_frame;
  if (cfg->action_kind == SWO_ACT_EMBODIED) {
    /* action_spaces.py:187-214 */
    const int32_t *a = (const int32_t *)action;
    int carry = a[0] != 0;
    double step = cfg->action_scale, mx, my;
    switch (a[1]) { /* :165-170 */
      case 0: mx = 0.0; my = step; break;
      case 1: mx = -step; my = 0.0; break;
      case 2: mx = 0.0; my = -step; break;
      case 3: mx = step; my = 0.0; break;
      default: return 1;
    }
    int body = S - 1;
    if (carry) { /* :180-185 top-most of sprites[:-1] containing the body centre */
      for (int s = body - 1; s >= 0; s--) {
        if (!sp[s].shape) continue;
        double tx = offset_component(sp[body].x, sp[body].pos_f32, sp[s].x, sp[s].pos_f32);
        double ty = offset_component(sp[body].y, sp[body].pos_f32, sp[s].y, sp[s].pos_f32);
        if (swo_contains_offset(tab, &sp[s], tx, ty)) {
          sprite_move(&sp[s], mx, my, keep);
          moved[1] = s;
          break;
        }
      }
    }
    sprite_move(&sp[body], mx, my, keep);
    moved[0] = body;
    *cost = -cfg->motion_cost * cfg->action_scale;
    return 0;
  }
  /* SelectMove :83-104 / DragAndDrop :133-137 */
  double px, py, mx, my, norm;
  if (action_is_f32) {
    const float *a = (const float *)action;
    volatile float fsc = (float)cfg->action_scale;
    volatile float d0, d1;
    if (cfg->action_kind == SWO_ACT_SELECT_MOVE) {
      d0 = a[2] - 0.5f;
      d1 = a[3] - 0.5f;
    } else {
      d0 = a[2] - a[0];
      d1 = a[3] - a[1];
    }
    volatile float m0 = d0 * fsc, m1 = d1 * fsc;
    px = a[0]; py = a[1]; mx = m0; my = m1;
    volatile float q0 = m0 * m0, q1 = m1 * m1;
    volatile float ss = q0 + q1;
    norm = (double)sqrtf(ss);
  } else {
    const double *a = (const double *)action;
    if (cfg->action_kind == SWO_ACT_SELECT_MOVE) {
      mx = (a[2] - 0.5) * cfg->action_scale;
      my = (a[3] - 0.5) * cfg->action_scale;
    } else {
      mx = (a[2] - a[0]) * cfg->action_scale;
      my = (a[3] - a[1]) * cfg->action_scale;
    }
    px = a[0]; py = a[1];
    /* np.linalg.norm = sqrt(x.dot(x)); OpenBLAS ddot of two elements is fma(m1, m1, m0 * m0).
     * This file builds with -ffp-contract=off, so the fusion is spelled out. */
    norm = sqrt(fma(my, my, mx * mx));
  }
  for (int s = S - 1; s >= 0; s--) { /* :77-81 top-most first */
    if (!sp[s].shape) continue;
    double tx = offset_component(px, action_is_f32, sp[s].x, sp[s].pos_f32);
    double ty = offset_component(py, action_is_f32, sp[s].y, sp[s].pos_f32);
    if (swo_contains_offset(tab, &sp[s], tx, ty)) {
      sprite_move(&sp[s], mx, my, keep);
      moved[0] = s;
      break;
    }
  }
  if (action_is_f32) {
    volatile float c = (float)(-cfg->motion_cost) * (float)norm;
    *cost = (double)c;
  } else {
    *cost = -cfg->motion_cost * norm;
  }
  return 0;
}

/* ---- tasks: tasks.py ------------------------------------------------------ */

typedef struct { double reward; int success; } task_val;

/* tasks.py:126-158 */
static task_val find_goal(const swo_task_node *nd, const swo_sprite *sp, int S, int use_sqrt) {
  double rewards[256];
  int n = 0, all_nonneg = 1;
  for (int s = 0; s < S; s++) {
    if (!sp[s].shape) continue;
    if (nd->filter_slot >= 0 && !((sp[s].member >> nd->filter_slot) & 1u)) continue;
    double dx = sp[s].x - nd->goal[0], dy = sp[s].y - nd->goal[1];
    double t0 = nd->weights[0] * (dx * dx), t1 = nd->weights[1] * (dy * dy);
    double tot = 0.;
    tot += t0;
    tot += t1;
    /* np.float64 ** 0.5 -> libm pow; the engine's sqrt differs from glibc's pow by 1 ULP
     * in ~0.08 % of inputs (swo_env_cfg.distance_sqrt) */
    double dist = use_sqrt ? sqrt(tot) : pow(tot, 0.5);
    double r = nd->raw_reward_multiplier * (nd->terminate_distance - dist);
    if (!(r >= 0)) all_nonneg = 0;
    rewards[n++] = r;
  }
  task_val out;
  out.success = all_nonneg; /* all([]) is True */
  if (n == 0) {
    out.reward = NAN;
    return out;
  }
  double dense = np_sum(rewards, n);
  double reward = 0.;
  if (all_nonneg) {
    reward += nd->terminate_bonus;
    reward += dense;
  } else if (!nd->sparse_reward) {
    reward += dense;
  }
  out.reward = reward;
  return out;
}

/* X @ Y.T of two 2-feature rows as OpenBLAS computes it on x86-64 with FMA (the numpy wheels'
 * BLAS): gemv (a cluster of >= 2 points against its centroid) fuses the first product into the
 * second; dot (a one-point cluster) and gemm (centroid against centroid) the second into the
 * first -- except, for 12 to 15 centroids, the entries of the first 12 rows and columns that
 * touch rows 8..11, which its tail kernel sums unfused.  Products of float32 values are exact in
 * float64, so for float32 positions all of these are the plain sum of products.  DESIGN.md
 * section 5. */
static double blas_dot2_gemv(double x0, double x1, double y0, double y1) {
  return fma(x0, y0, x1 * y1);
}
static double blas_dot2_dot(double x0, double x1, double y0, double y1) {
  return fma(x1, y1, x0 * y0);
}
static double blas_dot2_gemm(int i, int j, int k, double x0, double x1, double y0, double y1) {
  if (k >= 12 && k <= 15 && i < 12 && j < 12 && (i >= 8 || j >= 8)) return x0 * y0 + x1 * y1;
  return fma(x1, y1, x0 * y0);
}

/* sklearn.metrics.davies_bouldin_score as called from tasks.py:207-215.
 * all_f32: the positions array is float32 (every sprite position float32).
 * Intra-cluster distances are averaged with np.mean's pairwise sum (8 accumulators from 8
 * points on), centroids with a sequential sum (a mean over axis 0).
 * returns 0 ok, SWO_ERR_* otherwise. */
static int davies_bouldin_metric(const double *px, const double *py, const int *label, int n,
                                 int n_clusters, int all_f32, double *metric) {
  int present[SWO_MAX_CHILDREN], relabel[SWO_MAX_CHILDREN];
  int k = 0;
  for (int c = 0; c < n_clusters; c++) {
    present[c] = 0;
    for (int i = 0; i < n; i++) if (label[i] == c) present[c] = 1;
    relabel[c] = present[c] ? k++ : -1;
  }
  if (!(1 < k && k < n)) return SWO_ERR_CLUSTER_LABELS;
  double cen[SWO_MAX_CHILDREN][2], intra[SWO_MAX_CHILDREN];
  for (int c = 0; c < n_clusters; c++) {
    if (!present[c]) continue;
    int kk = relabel[c], cnt = 0;
    double cx, cy, mean_d;
    if (all_f32) {
      volatile float sx = 0.f, sy = 0.f; /* float32 mean over axis 0: sequential */
      int first = 1;
      for (int i = 0; i < n; i++) {
        if (label[i] != c) continue;
        if (first) { sx = (float)px[i]; sy = (float)py[i]; first = 0; }
        else { sx = sx + (float)px[i]; sy = sy + (float)py[i]; }
        cnt++;
      }
      volatile float mx = sx / (float)cnt, my = sy / (float)cnt;
      cx = mx; cy = my;
      /* euclidean_distances float32 path: -2 x.y + |x|^2 + |y|^2 in float64, cast to
       * float32, clamp at 0, float32 sqrt; then float32 mean */
      float dist[SWO_MAX_SLOTS_CLUSTER];
      int m = 0;
      double yy = cx * cx + cy * cy;
      for (int i = 0; i < n; i++) {
        if (label[i] != c) continue;
        double xx = px[i] * px[i] + py[i] * py[i];
        double d = -2.0 * blas_dot2_gemv(px[i], py[i], cx, cy);
        d += xx;
        d += yy;
        volatile float df = (float)d;
        if (df < 0.f) df = 0.f;
        volatile float sq = sqrtf(df);
        dist[m++] = sq;
      }
      volatile float acc = np_sum_f32(dist, m);
      volatile float md = acc / (float)cnt;
      mean_d = md;
    } else {
      double sx = 0., sy = 0.;
      int first = 1;
      for (int i = 0; i < n; i++) {
        if (label[i] != c) continue;
        if (first) { sx = px[i]; sy = py[i]; first = 0; } else { sx += px[i]; sy += py[i]; }
        cnt++;
      }
      cx = sx / cnt; cy = sy / cnt;
      double dist[SWO_MAX_SLOTS_CLUSTER], yy = cx * cx + cy * cy;
      int m = 0;
      for (int i = 0; i < n; i++) {
        if (label[i] != c) continue;
        double xx = px[i] * px[i] + py[i] * py[i];
        double dot = cnt == 1 ? blas_dot2_dot(px[i], py[i], cx, cy)
                              : blas_dot2_gemv(px[i], py[i], cx, cy);
        double d = -2.0 * dot;
        d += xx;
        d += yy;
        if (d < 0.) d = 0.;
        dist[m++] = sqrt(d);
      }
      mean_d = np_sum(dist, m) / cnt;
    }
    cen[kk][0] = cx; cen[kk][1] = cy; intra[kk] = mean_d;
  }
  /* centroid distances (float64 path, diagonal forced to 0) */
  double cd[SWO_MAX_CHILDREN][SWO_MAX_CHILDREN];
  int all_intra_zero = 1, all_cd_zero = 1;
  for (int i = 0; i < k; i++) if (!(fabs(intra[i]) <= 1e-8)) all_intra_zero = 0;
  for (int i = 0; i < k; i++) {
    double xi = cen[i][0] * cen[i][0] + cen[i][1] * cen[i][1];
    for (int j = 0; j < k; j++) {
      double xj = cen[j][0] * cen[j][0] + cen[j][1] * cen[j][1];
      double d = -2.0 * blas_dot2_gemm(i, j, k, cen[i][0], cen[i][1], cen[j][0], cen[j][1]);
      d += xi;
      d += xj;
      if (d < 0.) d = 0.;
      if (i == j) d = 0.;
      cd[i][j] = sqrt(d);
      if (!(fabs(cd[i][j]) <= 1e-8)) all_cd_zero = 0;
    }
  }
  if (all_intra_zero || all_cd_zero) return SWO_ERR_CLUSTER_ZERODIV; /* score 0.0 -> 1./0. */
  double scores[SWO_MAX_CHILDREN];
  for (int i = 0; i < k; i++) {
    double best = -INFINITY;
    for (int j = 0; j < k; j++) {
      double dd = cd[i][j] == 0 ? INFINITY : cd[i][j];
      double v = (intra[i] + intra[j]) / dd;
      if (v > best) best = v;
    }
    scores[i] = best;
  }
  double score = np_sum(scores, k) / k;
  if (score == 0.0) return SWO_ERR_CLUSTER_ZERODIV;
  *metric = 1. / score;
  return SWO_ERR_NONE;
}

/* tasks.py:196-245 */
static task_val clustering(const swo_task_node *nd, const swo_sprite *sp, int S, int *err) {
  double px[SWO_MAX_SLOTS_CLUSTER], py[SWO_MAX_SLOTS_CLUSTER];
  int label[SWO_MAX_SLOTS_CLUSTER], n = 0, all_f32 = 1;
  for (int s = 0; s < S; s++) {
    if (!sp[s].shape) continue;
    int lab = -1;
    for (int c = 0; c < nd->n_clusters; c++) {
      if ((sp[s].member >> nd->cluster_slots[c]) & 1u) { lab = c; break; }
    }
    if (!sp[s].pos_f32) all_f32 = 0; /* np.array([...positions]) promotes to float64 */
    if (lab < 0) continue;
    px[n] = sp[s].x; py[n] = sp[s].y; label[n] = lab; n++;
  }
  task_val out;
  double metric = 0.;
  int e = davies_bouldin_metric(px, py, label, n, nd->n_clusters, all_f32, &metric);
  if (e) {
    *err = e;
    out.reward = NAN;
    out.success = 0;
    return out;
  }
  double dense = (metric - nd->termination_threshold) * nd->reward_range / 2.;
  double reward = 0.;
  out.success = metric >= nd->termination_threshold;
  if (out.success) {
    reward += nd->terminate_bonus;
    reward += dense;
  } else if (!nd->sparse_reward) {
    reward += dense;
  }
  out.reward = reward;
  return out;
}

/* evaluates the whole tree; root = last node.  tasks.py:288-296 for MetaAggregated. */
SWO_API void swo_task_eval(const swo_env_cfg *cfg, const swo_sprite *sp, int S, double *reward,
                           int *success, int *err) {
  task_val val[SWO_MAX_NODES];
  *err = 0;
  for (int i = 0; i < cfg->n_nodes; i++) {
    const swo_task_node *nd = &cfg->nodes[i];
    switch (nd->kind) {
      case SWO_TASK_FIND_GOAL: val[i] = find_goal(nd, sp, S, cfg->distance_sqrt); break;
      case SWO_TASK_CLUSTERING: val[i] = clustering(nd, sp, S, err); break;
      case SWO_TASK_META: {
        double r[SWO_MAX_CHILDREN];
        int nn = 0, cnt_nonnan = 0, all_s = 1, any_s = 0;
        for (int c = 0; c < nd->n_children; c++) {
          task_val cv = val[nd->children[c]];
          r[nn++] = cv.reward;
          if (!isnan(cv.reward)) cnt_nonnan++;
          all_s = all_s && cv.success;
          any_s = any_s || cv.success;
        }
        double agg;
        if (nd->aggregator == SWO_AGG_SUM || nd->aggregator == SWO_AGG_MEAN) {
          double z[SWO_MAX_CHILDREN];
          for (int c = 0; c < nn; c++) z[c] = isnan(r[c]) ? 0. : r[c];
          agg = np_sum(z, nn);
          if (nd->aggregator == SWO_AGG_MEAN) agg = cnt_nonnan ? agg / cnt_nonnan : NAN;
        } else {
          agg = NAN;
          for (int c = 0; c < nn; c++) {
            if (isnan(r[c])) continue;
            if (isnan(agg)) agg = r[c];
            else if (nd->aggregator == SWO_AGG_MAX) agg = r[c] > agg ? r[c] : agg;
            else agg = r[c] < agg ? r[c] : agg;
          }
        }
        int succ = nd->criterion == SWO_CRIT_ALL ? all_s : any_s;
        agg += nd->terminate_bonus * (double)succ;
        val[i].reward = agg;
        val[i].success = succ;
        break;
      }
      default: val[i].reward = 0.0; val[i].success = 0; break; /* NoReward tasks.py:70-81 */
    }
  }
  *reward = val[cfg->n_nodes - 1].reward;
  *success = val[cfg->n_nodes - 1].success;
}

/* ---- renderer: renderers/pil_renderer.py:67-91 ---------------------------- */

/* frame: H x W x 3, already flipped (np.flipud).  canvas scratch: (aa*H)*(aa*W)*3 bytes. */
static void render_ws(const swo_raster_cfg *rc, const swo_shape_table *tab, const swo_sprite *sp,
                      int S, uint8_t *frame, uint8_t *canvas, uint8_t *hbuf, uint8_t *small) {
  int CW = rc->anti_aliasing * rc->width, CH = rc->anti_aliasing * rc->height;
  for (size_t i = 0; i < (size_t)CW * CH; i++) { /* canvas.paste(bg) :79 */
    canvas[3 * i] = rc->bg[0]; canvas[3 * i + 1] = rc->bg[1]; canvas[3 * i + 2] = rc->bg[2];
  }
  double xy[2 * SWO_MAX_VERTS];
  for (int s = 0; s < S; s++) { /* back to front :80-83 */
    if (!sp[s].shape) continue;
    int n = tab->n_verts[sp[s].shape];
    for (int i = 0; i < n; i++) {
      double cx, cy;
      centred_vertex(tab, &sp[s], i, &cx, &cy);
      /* Sprite.vertices (sprite.py:128-133): translate by float(position) */
      double wx = cx + sp[s].x, wy = cy + sp[s].y;
      xy[2 * i] = (double)CW * wx; /* canvas_size * vertices :81 */
      xy[2 * i + 1] = (double)CH * wy;
    }
    swo_polygon_fill(canvas, CW, CH, xy, n, sp[s].rgb, 1);
  }
  swo_lanczos_resize(canvas, CW, CH, small, rc->width, rc->height, hbuf); /* :84 */
  size_t row = (size_t)rc->width * 3;
  for (int y = 0; y < rc->height; y++) /* np.flipud :90 */
    memcpy(frame + (size_t)(rc->height - 1 - y) * row, small + (size_t)y * row, row);
}

/* Scratch of one render: the aa-times canvas, the horizontal-pass image and the unflipped
 * frame.  Kept per thread and only ever grown: the batch driver is called once per step from
 * every worker thread, and a 300 KB malloc/free pair per call goes through mmap/munmap, which
 * serialises the threads on the process's address-space lock. */
static __thread uint8_t *tls_ws = NULL;
static __thread size_t tls_ws_cap = 0;

static void workspace(const swo_raster_cfg *rc, uint8_t **canvas, uint8_t **hbuf, uint8_t **small) {
  size_t CW = (size_t)rc->anti_aliasing * rc->width, CH = (size_t)rc->anti_aliasing * rc->height;
  size_t n_canvas = CW * CH * 3, n_h = CH * rc->width * 3, n_small = (size_t)rc->width * rc->height * 3;
  size_t need = n_canvas + n_h + n_small;
  if (need > tls_ws_cap) {
    free(tls_ws);
    tls_ws = (uint8_t *)malloc(need);
    tls_ws_cap = need;
  }
  *canvas = tls_ws;
  *hbuf = tls_ws + n_canvas;
  *small = tls_ws + n_canvas + n_h;
}

/* frame: H x W x 3, already flipped (np.flipud).  canvas: optional caller scratch of
 * (aa*H)*(aa*W)*3 bytes that receives the anti-aliasing canvas (tests look at it). */
SWO_API void swo_render(const swo_raster_cfg *rc, const swo_shape_table *tab, const swo_sprite *sp,
                        int S, uint8_t *frame, uint8_t *canvas) {
  uint8_t *ws_canvas, *hbuf, *small;
  workspace(rc, &ws_canvas, &hbuf, &small);
  render_ws(rc, tab, sp, S, frame, canvas ? canvas : ws_canvas, hbuf, small);
}

/* ---- environment: environment.py:74-108 ----------------------------------- */

/* One env, one step AFTER the reset check.  Returns 0, or 1 for a bad Embodied action. */
SWO_API int swo_env_step(const swo_env_cfg *cfg, const swo_shape_table *tab, swo_sprite *sp, int S,
                         int32_t *step_count, const void *action, int action_is_f32,
                         double *reward, int8_t *step_type, uint8_t *success, uint8_t *err) {
  double cost = 0.;
  int moved[2];
  *step_count += 1; /* :93 */
  int rc = swo_action_step(cfg, tab, sp, S, action, action_is_f32, &cost, moved); /* :94-95 */
  if (rc) return rc;
  for (int s = 0; s < S; s++) /* :98-99 */
    if (sp[s].shape) sprite_move(&sp[s], sp[s].vx, sp[s].vy, cfg->keep_in_frame);
  double tr;
  int succ, e;
  swo_task_eval(cfg, sp, S, &tr, &succ, &e);
  /* :101.  A float32 click costs an np.float32; Clustering's reward is a Python float, so NumPy 2
   * adds the two in float32.  Every other root returns np.float64 (or 0.0, which leaves the
   * float32 cost unchanged either way). */
  if (action_is_f32 && cfg->action_kind != SWO_ACT_EMBODIED &&
      cfg->nodes[cfg->n_nodes - 1].kind == SWO_TASK_CLUSTERING) {
    volatile float sum = (float)cost + (float)tr;
    *reward = sum;
  } else {
    *reward = cost + tr;
  }
  int timeout = *step_count >= cfg->max_episode_length; /* :84 */
  int oof = 0;
  for (int s = 0; s < S; s++) if (sp[s].shape && out_of_frame(&sp[s])) oof = 1;
  *success = (uint8_t)succ;
  *err = (uint8_t)e;
  *step_type = (succ || oof || timeout) ? SWO_STEP_LAST : SWO_STEP_MID; /* :104-108 */
  return 0;
}

/*
 * Batch driver over envs [e0, e1) with the scene-pool auto-reset protocol:
 * pool holds K pre-sampled scenes per env (host-sampled by init_sprites); an env whose
 * reset_next flag is set ignores its action, advances its cursor, copies the scene and
 * returns FIRST (environment.py:90-91, 74-78).  Returns 1 if some env had a bad Embodied
 * action (its status carries SWO_ERR_BAD_ACTION), else 0.
 */
SWO_API int swo_batch_step(const swo_env_cfg *cfg, const swo_shape_table *tab,
                           const swo_raster_cfg *rc, int S, int K, swo_sprite *cur,
                           const swo_sprite *pool, int32_t *cursor, int32_t *step_count,
                           uint8_t *reset_next, const void *actions, int action_is_f32,
                           double *reward, int8_t *step_type, uint8_t *success, uint8_t *err,
                           uint8_t *frames, int e0, int e1) {
  size_t astride = cfg->action_kind == SWO_ACT_EMBODIED ? 2 * sizeof(int32_t)
                   : (action_is_f32 ? 4 * sizeof(float) : 4 * sizeof(double));
  uint8_t *canvas = NULL, *hbuf = NULL, *small = NULL;
  size_t fbytes = 0;
  if (rc && frames) {
    workspace(rc, &canvas, &hbuf, &small);
    fbytes = (size_t)rc->width * rc->height * 3;
  }
  int bad = 0;
  for (int e = e0; e < e1; e++) {
    swo_sprite *sp = cur + (size_t)e * S;
    if (reset_next[e]) {
      cursor[e] = (cursor[e] + 1) % K;
      memcpy(sp, pool + ((size_t)e * K + cursor[e]) * S, sizeof(swo_sprite) * S);
      step_count[e] = 0;
      reset_next[e] = 0;
      double tr;
      int succ, er;
      swo_task_eval(cfg, sp, S, &tr, &succ, &er);
      reward[e] = 0.0;
      step_type[e] = SWO_STEP_FIRST;
      success[e] = (uint8_t)succ;
      err[e] = (uint8_t)er;
    } else {
      int r = swo_env_step(cfg, tab, sp, S, &step_count[e], (const char *)actions + astride * e,
                           action_is_f32, &reward[e], &step_type[e], &success[e], &err[e]);
      if (r) {
        /* the reference's state after a caught KeyError: the step is counted (:93), nothing
         * moved; the env reports it and the unchanged scene is rendered */
        double tr;
        int succ, er;
        swo_task_eval(cfg, sp, S, &tr, &succ, &er);
        reward[e] = NAN;
        step_type[e] = SWO_STEP_MID;
        success[e] = (uint8_t)succ;
        err[e] = (uint8_t)(er | SWO_ERR_BAD_ACTION);
        bad = r;
      }
      if (step_type[e] == SWO_STEP_LAST) reset_next[e] = 1;
    }
    if (canvas) render_ws(rc, tab, sp, S, frames + fbytes * e, canvas, hbuf, small);
  }
  return bad;
}

SWO_API int swo_sizeof_sprite(void) { return (int)sizeof(swo_sprite); }
SWO_API int swo_sizeof_env_cfg(void) { return (int)sizeof(swo_env_cfg); }
SWO_API int swo_sizeof_task_node(void) { return (int)sizeof(swo_task_node); }
SWO_API int swo_sizeof_shape_table(void) { return (int)sizeof(swo_shape_table); }
