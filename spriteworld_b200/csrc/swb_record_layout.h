// Byte offsets of the fields of one env record (the table in include/spriteworld_b200.h).  Plain
// C++ for host and device: the record kernels (swb_states.cuh) and the record maker
// (swb_make_states.cuh, also built for the CPU) lay records out through it.
#pragma once
#include <stddef.h>

#ifdef __CUDACC__
#define SWB_LAYOUT_HD __host__ __device__
#else
#define SWB_LAYOUT_HD
#endif

namespace swb {

// Byte offsets of the fields of one record of an engine with S slots and G goal slots.
struct RecordLayout {
  int S, G;
  SWB_LAYOUT_HD explicit RecordLayout(int S_, int G_ = 0) : S(S_), G(G_) {}
  // x0, y0, m00, m01, m10, m11, vx, vy, pos_x, pos_y: f64 [10][S] from offset 0
  SWB_LAYOUT_HD size_t member() const { return 80 * (size_t)S; }      // u32 [S]
  SWB_LAYOUT_HD size_t rgb() const { return 84 * (size_t)S; }         // u32 [S]
  SWB_LAYOUT_HD size_t factors() const { return 88 * (size_t)S; }     // f32 [5][S]
  SWB_LAYOUT_HD size_t step_count() const { return 108 * (size_t)S; } // i32
  SWB_LAYOUT_HD size_t reset_next() const { return 108 * (size_t)S + 4; }  // u8
  SWB_LAYOUT_HD size_t shape() const { return 108 * (size_t)S + 5; }  // u8 [S]
  SWB_LAYOUT_HD size_t pos_f32() const { return 109 * (size_t)S + 5; }  // u8 [S]
  SWB_LAYOUT_HD size_t goals() const { return (110 * (size_t)S + 5 + 7) & ~(size_t)7; }  // f64 [G][2]
  SWB_LAYOUT_HD size_t used() const { return G ? goals() + 16 * (size_t)G : 110 * (size_t)S + 5; }
  SWB_LAYOUT_HD size_t bytes() const { return (used() + 15) & ~(size_t)15; }  // zero padded
};

}  // namespace swb
