// Positions inside sprites: Environment.sample_contained_position for every row of a batch
// (swb_sample_contained, include/spriteworld_b200.h).
//
// Sample s of row i (a live env or an env record) picks one of the row's sprites uniformly -- the
// reference's self._sprites[np.random.randint(len)], empty slots padded at the front -- and then
// rejection-samples the sprite's centred bounding box until the step kernel's hit test accepts the
// point (sprite.py sample_contained_position).  Draws come from the scene sampler's counter-based
// Stream (swb_sampler.cuh) under the key (seed, SWB_CONTAINED_DOMAIN) and counter (block, s, i, 0),
// so a sample is a pure function of (seed, i, s, the row's state) and never aliases a scene draw.
//
// sample_contained is plain C++ for host and device (SWB_HD): contained_kernel runs it on the GPU,
// and csrc/swb_sampler_host.cpp builds it for the CPU as the restatement the tests compare the
// kernel against.  Both builds run without contraction, so every double operation rounds alike.
//
// The hit test is the even-odd test of warp_contains (swb_step.cuh), restated serially: the step
// kernel tests a float64 click c against slot k with c - pos in float64, so a click at the returned
// position grabs slot k or a sprite above it.
#pragma once
#include "swb_record_layout.h"
#include "swb_sampler.cuh"

namespace swb_contained {

// The fields of the chosen slot: live position and centred-path transform.
struct Sprite {
  double x, y, m00, m01, m10, m11;
};

// Vertex j of the centred path, as warp_contains transforms it: (m00 ax + m01 ay) + 0.0.
SWB_HD void centred(const Sprite &sp, const double *v, int j, double &cx, double &cy) {
  const double ax = v[2 * j], ay = v[2 * j + 1];
  cx = (sp.m00 * ax + sp.m01 * ay) + 0.0;
  cy = (sp.m10 * ax + sp.m11 * ay) + 0.0;
}

// warp_contains of (tx, ty) relative to the sprite's position: the parity of the edges i -> i+1
// (closing edge included) whose even-odd test toggles.  Edges are visited from the closing one on,
// so each vertex is transformed once.
SWB_HD bool contains(const Sprite &sp, const double *v, int n, double tx, double ty) {
  double x0, y0;
  centred(sp, v, n - 1, x0, y0);
  bool inside = false;
  for (int j = 0; j < n; ++j) {
    double x1, y1;
    centred(sp, v, j, x1, y1);
    const bool yf0 = y0 >= ty, yf1 = y1 >= ty;
    if (yf0 != yf1) {
      const double lhs = (y1 - ty) * (x0 - x1);
      const double rhs = (x1 - tx) * (y0 - y1);
      if ((lhs >= rhs) == yf1) inside = !inside;
    }
    x0 = x1;
    y0 = y1;
  }
  return inside;
}

// Sample s of row i.  `shape_at(j)` gives slot j's shape id (0 .. S-1), `sprite_at(j)` slot j's
// Sprite; only the chosen slot's sprite is read.  verts / nverts: the engine's shape table
// ([SWB_NUM_SHAPES][SWB_MAX_VERTS][2], [SWB_NUM_SHAPES]).  Writes pos[0..1] and *slot, returns the
// status (SWB_ENV_OK, SWB_ENV_NO_SPRITE or SWB_ENV_SAMPLE_TRIES).
template <typename ShapeAt, typename SpriteAt>
SWB_HD int sample_contained(uint64_t seed, uint64_t i, uint64_t s, int S, const double *verts,
                            const int32_t *nverts, const ShapeAt &shape_at, const SpriteAt &sprite_at,
                            double *pos, int8_t *slot) {
  pos[0] = pos[1] = nan("");
  *slot = -1;
  int m = 0;
  for (int j = 0; j < S; ++j) m += swb::sanitize_shape(shape_at(j), nverts) != 0;
  if (m == 0) return SWB_ENV_NO_SPRITE;
  swb_sampler::Stream rng;
  rng.init(seed, i, s, SWB_CONTAINED_DOMAIN);
  int k = (int)rng.below(m);
  int j = 0, shape = 0;
  for (;; ++j) {
    shape = swb::sanitize_shape(shape_at(j), nverts);
    if (shape && k-- == 0) break;
  }
  const Sprite sp = sprite_at(j);
  const double *v = verts + (size_t)shape * SWB_MAX_VERTS * 2;
  const int n = nverts[shape];
  double lox, loy, hix, hiy;
  centred(sp, v, 0, lox, loy);
  hix = lox;
  hiy = loy;
  for (int q = 1; q < n; ++q) {
    double cx, cy;
    centred(sp, v, q, cx, cy);
    lox = cx < lox ? cx : lox; hix = cx > hix ? cx : hix;
    loy = cy < loy ? cy : loy; hiy = cy > hiy ? cy : hiy;
  }
  const double wx = hix - lox, wy = hiy - loy;
  for (int t = 0; t < SWB_CONTAINED_MAX_TRIES; ++t) {
    const double ux = rng.uniform();
    const double uy = rng.uniform();
    // NumPy's uniform(lo, hi) added to the position, then the offset apply_action tests
    const double cx = sp.x + (lox + wx * ux), cy = sp.y + (loy + wy * uy);
    if (contains(sp, v, n, cx - sp.x, cy - sp.y)) {
      pos[0] = cx;
      pos[1] = cy;
      *slot = (int8_t)j;
      return SWB_ENV_OK;
    }
  }
  return SWB_ENV_SAMPLE_TRIES;
}

}  // namespace swb_contained

#ifdef __CUDACC__
#include "swb_states.cuh"

namespace swb {

constexpr int CT_THREADS = 128;

// One thread per (row, sample), t = i * n_samples + s: the n_samples threads of a row are
// neighbours and share its shape bytes in L1.  Live rows read pool entry (e, cursor[e]) and the
// live positions, as factor_tensors and the render kernel do; record rows read the record.
template <bool kRecords>
__global__ void __launch_bounds__(CT_THREADS)
contained_kernel(DevState st, const unsigned char *__restrict__ records, size_t record_bytes, int n,
                 int n_samples, uint64_t seed, double *__restrict__ position, int8_t *__restrict__ slot,
                 uint8_t *__restrict__ status) {
  const int64_t t = (int64_t)blockIdx.x * CT_THREADS + threadIdx.x;
  if (t >= (int64_t)n * n_samples) return;
  const int i = (int)(t / n_samples), s = (int)(t - (int64_t)i * n_samples);
  const int S = st.S;
  const unsigned char *const rec = kRecords ? records + (size_t)i * record_bytes : nullptr;
  const size_t entry = kRecords ? 0 : ((size_t)i * st.K + st.cursor[i]) * S;
  auto shape_at = [&](int j) -> int {
    return kRecords ? read_record(st, rec, j).shape : st.p_shape[entry + j];
  };
  auto sprite_at = [&](int j) {
    swb_contained::Sprite sp;
    if (kRecords) {
      const SlotRecord r = read_record(st, rec, j);
      sp.x = r.f64[POS_X]; sp.y = r.f64[POS_Y];
      sp.m00 = r.f64[M00]; sp.m01 = r.f64[M01]; sp.m10 = r.f64[M10]; sp.m11 = r.f64[M11];
    } else {
      sp.x = st.pos_x[(size_t)i * S + j]; sp.y = st.pos_y[(size_t)i * S + j];
      sp.m00 = st.p_m00[entry + j]; sp.m01 = st.p_m01[entry + j];
      sp.m10 = st.p_m10[entry + j]; sp.m11 = st.p_m11[entry + j];
    }
    return sp;
  };
  double pos[2];
  int8_t k;
  const int stat = swb_contained::sample_contained(seed, (uint64_t)i, (uint64_t)s, S, st.shape_verts, st.shape_n,
                                                   shape_at, sprite_at, pos, &k);
  position[2 * t] = pos[0];
  position[2 * t + 1] = pos[1];
  slot[t] = k;
  status[t] = (uint8_t)stat;
}

}  // namespace swb
#endif
