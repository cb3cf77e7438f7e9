// Device-side data layout shared by the step and render kernels.
//
// HBM layout (all arrays owned by swb_engine, struct-of-arrays):
//   live state   pos_x, pos_y            [E*S] f64   (float32-valued where pos_f32)
//                cursor, step_count      [E]   i32
//                reset_next              [E]   u8
//                scene_serial            [E]   i32  (how many scenes the env has started)
//   scene pool   x0,y0,m00..m11,vx,vy    [E*K*S] f64
//                member                  [E*K*S] u32
//                shape,pos_f32           [E*K*S] u8
//                rgb                     [E*K*S] u32 (r | g<<8 | b<<16)
//                factors                 [E*K*S*5] f32 (scale, angle, c0, c1, c2)
//                goal                    [E*K*G*2] f64 (sampled FindGoalPosition goals; only when G > 0)
//   index of (env e, ring slot k, sprite slot s) = (e*K + k)*S + s; goal slot g: ((e*K + k)*G + g)*2
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "../../include/spriteworld_b200.h"

namespace swb {

struct DevState {
  int E, S, K;
  double *pos_x, *pos_y;
  int32_t *cursor, *step_count;
  uint8_t *reset_next;
  int32_t *scene_serial;   // [E] scenes the env has started so far (monotonic; ring slot = cursor)
  uint8_t *render_status;  // [E] SWB_ENV_SPAN_OVERFLOW from the last render
  double *p_x, *p_y, *p_m00, *p_m01, *p_m10, *p_m11, *p_vx, *p_vy;
  uint32_t *p_member;
  uint8_t *p_shape, *p_pos_f32;
  uint32_t *p_rgb;
  float *p_factors;
  int G;            // goal slots per scene (0: every goal of the task tree is a constant)
  double *p_goal;   // null when G == 0
  const double *shape_verts;  // [13][32][2]
  const int32_t *shape_n;     // [13]
};

// action space + episode + task tree; every engine keeps its own copy in device memory and
// hands the step kernel a pointer to it.
struct StepCfg {
  int32_t action_kind;
  double action_scale;
  double motion_cost;
  int32_t keep_in_frame;
  int32_t max_episode_length;
  int32_t n_nodes;
  swb_task_node nodes[SWB_MAX_NODES];
};

// Prefix-table stride of windows up to 32 taps (anti_aliasing <= 5), the stride the render
// kernel's narrow instantiation is compiled for; longer windows take their length + 1.
constexpr int kNarrowPrefixStride = 33;

// Resampling tables for one axis (Pillow precompute_coeffs / normalize_coeffs_8bpc).
struct AxisTables {
  const int16_t *win_min;    // [n_out]  first input index of the tap window
  const uint8_t *win_len;    // [n_out]  taps (6 * anti_aliasing at most, <= 255)
  const uint8_t *win_cls;    // [n_out]  class = distinct tap vector
  const int32_t *prefix;     // [n_cls][RasterDev::prefix_stride] prefix sums of the tap vector, prefix[len] = total
  const int16_t *first_out;  // [n_in] first output whose window contains input index i
  const int16_t *last_out;   // [n_in] last  output whose window contains input index i
};

struct RasterDev {
  int W, H, aa, CW, CH;
  uint32_t bg;  // r | g<<8 | b<<16
  int band_rows;  // output rows per CTA
  int n_bands;
  int max_spans;  // spans kept per (sprite, canvas row)
  int ncls_x, ncls_y;  // distinct tap vectors per axis
  int prefix_stride;   // entries per class of ax.prefix: the longest horizontal window + 1, >= 33
  int tile_blocks;     // blocks of eight output rows per phase-C tile (3, 2 or 1): the most whose
                       // vertical windows fit the H tile's 4 * HT_ROWW canvas rows in every band
  // vertical pass on the integer tensor pipe (mma.sync m16n8k32 u8 x s8 -> s32): per block of
  // eight output rows the 22-bit tap matrix, cut into three signed 8-bit limbs and laid out as
  // the instruction's B fragments (see swb_tables.h build_vfrag)
  int v_nks;                 // k-steps (32 canvas rows each) a block's taps span (1..6)
  const uint8_t *v_blk_cls;  // [ceil(H/8)] class (distinct coefficient matrix) of each block
  const uint2 *v_frag;       // [n_cls][v_nks][3 limbs][32 lanes] {b0, b1}
  AxisTables ax, ay;
};

}  // namespace swb
