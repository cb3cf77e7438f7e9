// Env records from factor columns (swb_make_states): the device scene sampler's packer
// (swb_sampler::pack_sprite) fed with the caller's factor values instead of Philox draws.
//
// Plain C++ for host and device (SWB_HD), as swb_sampler.cuh: the CUDA library runs it one warp
// per record, one lane per slot (make_states_kernel), and csrc/swb_sampler_host.cpp builds the same
// functions for the CPU (swb_host_make_states), the restatement the tests hold the kernel to.  A
// record is made in three steps: read_slot per slot (its factors and its SWB_MAKE_* bits),
// record_status over the record's slots, then swb::write_record of make_slot per slot and
// swb::write_goals once.
#pragma once
#include "swb_record_layout.h"
#include "swb_sampler.cuh"

namespace swb_make {

using swb_sampler::Packed;
using swb_sampler::Sprite;

// A factor column's element k as float64; `big` <- an integer of magnitude above 2^53 (the packer
// compares in float64, which cannot hold it exactly).
SWB_HD double column_value(const void *col, int kind, size_t k, bool &big) {
  switch (kind) {
    case SWB_FT_F32: return (double)static_cast<const float *>(col)[k];
    case SWB_FT_F64: return static_cast<const double *>(col)[k];
    case SWB_FT_I8: return (double)static_cast<const int8_t *>(col)[k];
    case SWB_FT_I16: return (double)static_cast<const int16_t *>(col)[k];
    case SWB_FT_I32: return (double)static_cast<const int32_t *>(col)[k];
    case SWB_FT_I64: {
      const int64_t v = static_cast<const int64_t *>(col)[k];
      big = v > (int64_t(1) << 53) || v < -(int64_t(1) << 53);
      return (double)v;
    }
    default: return (double)static_cast<const uint8_t *>(col)[k];  // SWB_FT_U8
  }
}

// Sprite.__init__'s defaults as the Python scalars they are (sprite.py)
SWB_HD void default_factor(int f, double &v, uint8_t &kind) {
  const double val[swb_sampler::kFactors] = {0.5, 0.5, 0.0, 0.0, 0.1, 0.0, 0.0, 0.0, 0.0, 0.0};
  const bool is_int = f == swb_sampler::F_ANGLE || f == swb_sampler::F_C0 || f == swb_sampler::F_C1 ||
                      f == swb_sampler::F_C2;
  v = val[f];
  kind = (uint8_t)(is_int ? SWB_FT_PYINT : SWB_FT_PYFLOAT);
}

// Slot k = i * S + j of the columns as a Sprite.  Returns its SWB_MAKE_* bits; occupied <- a valid
// non-zero shape id, concave <- a star or spoke.
SWB_HD uint32_t read_slot(const swb_factor_columns &c, size_t k, Sprite &s, bool &occupied, bool &concave) {
  bool big = false;
  for (int f = 0; f < swb_sampler::kFactors; ++f) {
    if (c.col[f]) {
      bool b = false;
      s.val[f] = column_value(c.col[f], c.kind[f], k, b);
      s.kind[f] = (uint8_t)c.kind[f];
      if (f != swb_sampler::F_SHAPE) big = big || b;
    } else {
      default_factor(f, s.val[f], s.kind[f]);
    }
  }
  uint32_t bits = 0;
  const double shape = s.val[swb_sampler::F_SHAPE];   // NaN fails both range tests
  const bool shape_ok = shape >= 0.0 && shape <= 12.0 && shape == (double)(int)shape;
  s.kind[swb_sampler::F_SHAPE] = (uint8_t)SWB_FT_SHAPE;
  if (!shape_ok) bits |= SWB_MAKE_SHAPE;
  occupied = shape_ok && shape != 0.0;
  concave = occupied && shape >= 7.0;
  if (occupied) {
    const double a = s.val[swb_sampler::F_ANGLE];
    if (!(a >= -360.0 && a <= 360.0 && a == (double)(int)a)) bits |= SWB_MAKE_ANGLE;
    if (big) bits |= SWB_MAKE_INT;
  }
  return bits;
}

// The SWB_MAKE_* bits of a record: the OR of its slots' bits, a hole in `occupied` (bit j: slot j
// is occupied; the occupied slots must be S - n .. S - 1), and a negative step count.
SWB_HD uint32_t record_status(uint32_t slot_bits, uint32_t occupied, int S, int32_t step) {
  const uint64_t m = occupied, full = (uint64_t(1) << S) - 1;
  uint32_t bits = slot_bits;
  if (m && (m | (m - 1)) != full) bits |= SWB_MAKE_HOLE;   // m - 1 fills the bits below the lowest
  if (step < 0) bits |= SWB_MAKE_STEP;
  return bits;
}

// A record's slot: the sprite's packed fields, or an empty slot's (also every slot of a refused
// record), with live position = initial, step_count `step` and reset_next = 0.
SWB_HD swb::SlotRecord make_slot(const swb_scene_program &p, const Sprite &s, bool occupied, uint32_t status,
                                 int32_t step) {
  Packed o;
  if (occupied && !status) swb_sampler::pack_sprite(p, s, o);
  else swb_sampler::empty_slot(o);
  swb::SlotRecord r;
  r.f64[swb::X0] = r.f64[swb::POS_X] = o.x;
  r.f64[swb::Y0] = r.f64[swb::POS_Y] = o.y;
  r.f64[swb::M00] = o.m00; r.f64[swb::M01] = o.m01; r.f64[swb::M10] = o.m10; r.f64[swb::M11] = o.m11;
  r.f64[swb::VX] = o.vx; r.f64[swb::VY] = o.vy;
  r.member = o.member;
  r.rgb = (uint32_t)o.rgb[0] | ((uint32_t)o.rgb[1] << 8) | ((uint32_t)o.rgb[2] << 16);
  for (int f = 0; f < 5; ++f) r.factors[f] = o.factors[f];
  r.shape = o.shape;
  r.pos_f32 = o.pos_f32;
  r.reset_next = 0;
  r.step_count = step;
  return r;
}

}  // namespace swb_make

#ifdef __CUDACC__
namespace swb {

constexpr int MAKE_WARPS = 4;   // records per CTA of make_states_kernel

// swb_make_states: warp r makes record r, lane j its slot j.
__global__ void __launch_bounds__(MAKE_WARPS * 32) make_states_kernel(
    const swb_scene_program *__restrict__ prog, swb_factor_columns cols, int n, int S, int G,
    const double *__restrict__ goals, const int32_t *__restrict__ step_count, unsigned char *__restrict__ records,
    size_t record_bytes, uint8_t *__restrict__ status, uint8_t *__restrict__ span_flag) {
  const int r = (int)((blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5), j = threadIdx.x & 31;
  if (r >= n) return;   // whole warps
  swb_sampler::Sprite s;
  bool occupied = false, concave = false;
  uint32_t bits = 0;
  if (j < S) bits = swb_make::read_slot(cols, (size_t)r * S + j, s, occupied, concave);
  const uint32_t occ = __ballot_sync(0xFFFFFFFFu, occupied);
  const uint32_t any_bits = __reduce_or_sync(0xFFFFFFFFu, bits);
  const bool any_concave = __any_sync(0xFFFFFFFFu, concave);
  const int32_t step = step_count ? step_count[r] : 0;
  const uint32_t st = swb_make::record_status(any_bits, occ, S, step);
  unsigned char *rec = records + (size_t)r * record_bytes;
  // lane 0's per-record stores first, so that nothing they need stays live across the packer
  if (j == 0) {
    write_goals(record_goals(rec, S, G), st || !G ? nullptr : goals + (size_t)r * G * 2, G);
    status[r] = (uint8_t)st;
    if (span_flag && any_concave && !st) *span_flag = 1;
  }
  if (j < S) write_record(rec, S, G, j, swb_make::make_slot(*prog, s, occupied, st, st ? 0 : step));
}

}  // namespace swb
#endif
