// The env record format (the table in include/spriteworld_b200.h): byte offsets of its fields,
// one slot of a record in registers, and the one writer of a record.  Plain C++ for host and
// device: the record kernels (swb_states.cuh, swb_rollout.cuh) and the record maker
// (swb_make_states.cuh, also built for the CPU) lay records out through it.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include "../../include/spriteworld_b200.h"

#ifdef __CUDACC__
#define SWB_LAYOUT_HD __host__ __device__ __forceinline__
#else
#define SWB_LAYOUT_HD inline
#endif

namespace swb {

// The ten float64 arrays of a record, [S] values each from offset 0, in this order: the pool
// entry's position, centred-path transform and velocity, then the live position.
enum RecordF64 : int { X0, Y0, M00, M01, M10, M11, VX, VY, POS_X, POS_Y, N_F64 };

// Byte offsets of the fields of one record of an engine with S slots and G goal slots.
struct RecordLayout {
  int S, G;
  SWB_LAYOUT_HD explicit RecordLayout(int S_, int G_ = 0) : S(S_), G(G_) {}
  // slot s of float64 array a (RecordF64), as an index in doubles from the record's start
  SWB_LAYOUT_HD int f64_at(int a, int s) const { return a * S + s; }
  SWB_LAYOUT_HD size_t member() const { return 80 * (size_t)S; }      // u32 [S]
  SWB_LAYOUT_HD size_t rgb() const { return 84 * (size_t)S; }         // u32 [S]
  SWB_LAYOUT_HD size_t factors() const { return 88 * (size_t)S; }     // f32 [5][S]
  SWB_LAYOUT_HD size_t step_count() const { return 108 * (size_t)S; } // i32
  SWB_LAYOUT_HD size_t reset_next() const { return 108 * (size_t)S + 4; }  // u8
  SWB_LAYOUT_HD size_t shape() const { return 108 * (size_t)S + 5; }  // u8 [S]
  SWB_LAYOUT_HD size_t pos_f32() const { return 109 * (size_t)S + 5; }  // u8 [S]
  SWB_LAYOUT_HD size_t slots_end() const { return 110 * (size_t)S + 5; }  // end of the fields above
  SWB_LAYOUT_HD size_t goals() const { return (slots_end() + 7) & ~(size_t)7; }  // f64 [G][2]
  SWB_LAYOUT_HD size_t used() const { return G ? goals() + 16 * (size_t)G : slots_end(); }
  SWB_LAYOUT_HD size_t bytes() const { return (used() + 15) & ~(size_t)15; }  // zero padded
};

// One slot of a record in registers; the per-record fields ride along in every slot's copy.
struct SlotRecord {
  double f64[N_F64];   // indexed by RecordF64
  uint32_t member, rgb;
  float factors[5];
  uint8_t shape, pos_f32, reset_next;
  int32_t step_count;
};

// A shape id without a vertex table (shape_n: the engine's vertex counts, [SWB_NUM_SHAPES]) is an
// empty slot (0), so that no kernel indexes the shape table with a record's shape byte.
SWB_LAYOUT_HD int sanitize_shape(int shape, const int32_t *shape_n) {
  return shape < SWB_NUM_SHAPES && shape_n[shape] >= 3 ? shape : 0;
}

// Slot s of a record.  Slot 0 also stores the per-record fields and zeroes the padding after the
// slot fields, around the goals (which write_goals stores, in any order with this): saved bytes
// are deterministic.
SWB_LAYOUT_HD void write_record(unsigned char *rec, int S, int G, int s, const SlotRecord &r) {
  const RecordLayout L(S, G);
  for (int a = 0; a < N_F64; ++a) reinterpret_cast<double *>(rec)[L.f64_at(a, s)] = r.f64[a];
  reinterpret_cast<uint32_t *>(rec + L.member())[s] = r.member;
  reinterpret_cast<uint32_t *>(rec + L.rgb())[s] = r.rgb;
  for (int f = 0; f < 5; ++f) reinterpret_cast<float *>(rec + L.factors())[f * S + s] = r.factors[f];
  rec[L.shape() + s] = r.shape;
  rec[L.pos_f32() + s] = r.pos_f32;
  if (s == 0) {
    *reinterpret_cast<int32_t *>(rec + L.step_count()) = r.step_count;
    rec[L.reset_next()] = r.reset_next;
    const size_t g0 = G ? L.goals() : L.bytes(), g1 = G ? L.used() : L.bytes();
    for (size_t b = L.slots_end(); b < g0; ++b) rec[b] = 0;
    for (size_t b = g1; b < L.bytes(); ++b) rec[b] = 0;
  }
}

// The goals (G x (x, y)) of a record, and a copy of G of them (zeros when src is null).
SWB_LAYOUT_HD double *record_goals(unsigned char *rec, int S, int G) {
  return reinterpret_cast<double *>(rec + RecordLayout(S, G).goals());
}
SWB_LAYOUT_HD const double *record_goals(const unsigned char *rec, int S, int G) {
  return reinterpret_cast<const double *>(rec + RecordLayout(S, G).goals());
}
SWB_LAYOUT_HD void write_goals(double *dst, const double *src, int G) {
  for (int i = 0; i < 2 * G; ++i) dst[i] = src ? src[i] : 0.;
}

}  // namespace swb
