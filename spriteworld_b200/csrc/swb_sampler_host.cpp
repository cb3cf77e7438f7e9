// The device scene sampler (swb_sampler.cuh), contained-position sampler (swb_contained.cuh) and
// record maker (swb_make_states.cuh) built for the CPU: the restatement the tests hold the CUDA
// kernels to, and a way to draw the device's scenes without a GPU.  Same source, no
// contraction (-ffp-contract=off), so it computes what the kernels compute, bit for bit.
#include "swb_contained.cuh"
#include "swb_make_states.cuh"
#include "swb_sampler.cuh"

extern "C" {

int swb_host_sampler_sizeof_program(void) { return (int)sizeof(swb_scene_program); }

// Philox4x64-10 of one counter block (for checking against np.random.Philox).
void swb_host_philox(const uint64_t ctr[4], uint64_t k0, uint64_t k1, uint64_t out[4]) {
  for (int i = 0; i < 4; ++i) out[i] = ctr[i];
  swb_sampler::philox4x64_10(out, k0, k1);
}

// swb_sample_scenes on the host, into host arrays laid out as swb_sample_out.  Returns the number
// of scenes whose rejection loop ran out of tries; fail_op / fail_index (may be null) get the first.
int64_t swb_host_sample_scenes(const swb_scene_program *prog, uint64_t seed, int32_t S, const int64_t *env_ids,
                               const int64_t *scene_idx, int64_t n, const swb_sample_out *out,
                               int32_t *fail_op, int64_t *fail_index) {
  int64_t failures = 0;
  swb_sampler::Scene sc;
  double goal[2 * SWB_MAX_GOALS];
  for (int64_t i = 0; i < n; ++i) {
    const int bad = swb_sampler::sample_and_pack(
        *prog, seed, (uint64_t)env_ids[i], (uint64_t)scene_idx[i], S, sc, goal,
        [&](int slot, const swb_sampler::Packed &o, const swb_sampler::Sprite *s) {
          const size_t d = (size_t)i * S + slot;
          out->x[d] = o.x; out->y[d] = o.y;
          out->m00[d] = o.m00; out->m01[d] = o.m01; out->m10[d] = o.m10; out->m11[d] = o.m11;
          out->vx[d] = o.vx; out->vy[d] = o.vy;
          out->member[d] = o.member; out->shape[d] = o.shape; out->pos_f32[d] = o.pos_f32;
          for (int c = 0; c < 3; ++c) out->rgb[d * 3 + c] = o.rgb[c];
          for (int f = 0; f < 5; ++f) out->factors[d * 5 + f] = o.factors[f];
          for (int f = 0; f < swb_sampler::kFactors; ++f) {
            out->factor_value[d * swb_sampler::kFactors + f] = s ? s->val[f] : 0.0;
            out->factor_kind[d * swb_sampler::kFactors + f] = s ? s->kind[f] : (uint8_t)SWB_FT_NONE;
          }
        });
    if (out->goal)
      for (int j = 0; j < 2 * prog->n_goals; ++j) out->goal[(size_t)i * 2 * prog->n_goals + j] = goal[j];
    if (bad >= 0) {
      if (!failures) {
        if (fail_op) *fail_op = bad;
        if (fail_index) *fail_index = i;
      }
      ++failures;
    }
  }
  return failures;
}

// swb_sample_contained on the host, over n rows of S packed slots each (row i's slot j at i * S + j:
// live position x, y, centred-path transform m00 .. m11, shape id) with the engine's shape table
// verts [SWB_NUM_SHAPES][SWB_MAX_VERTS][2], nverts [SWB_NUM_SHAPES].  Outputs as the device call
// lays them out: position [n][n_samples][2], slot and status [n][n_samples].
void swb_host_sample_contained(const double *x, const double *y, const double *m00, const double *m01,
                               const double *m10, const double *m11, const uint8_t *shape, int32_t n,
                               int32_t S, const double *verts, const int32_t *nverts, int32_t n_samples,
                               uint64_t seed, double *position, int8_t *slot, uint8_t *status) {
  for (int64_t i = 0; i < n; ++i) {
    const size_t r = (size_t)i * S;
    auto shape_at = [&](int j) -> int { return shape[r + j]; };
    auto sprite_at = [&](int j) {
      return swb_contained::Sprite{x[r + j], y[r + j], m00[r + j], m01[r + j], m10[r + j], m11[r + j]};
    };
    for (int64_t s = 0; s < n_samples; ++s) {
      const int64_t t = i * n_samples + s;
      status[t] = (uint8_t)swb_contained::sample_contained(seed, (uint64_t)i, (uint64_t)s, S, verts, nverts,
                                                           shape_at, sprite_at, position + 2 * t, slot + t);
    }
  }
}

// swb_make_states on the host, over host arrays laid out as the device call takes them (columns
// [n][S], goals [n][G][2] or null for G = 0, step_count [n] or null), into n records of
// record_bytes bytes each, status [n] and *span_flag (may be null; set to 1 if an accepted record
// holds a star or spoke, else left as it is).
void swb_host_make_states(const swb_scene_program *prog, const swb_factor_columns *cols, int32_t n, int32_t S,
                          int32_t G, const double *goals, const int32_t *step_count, unsigned char *records,
                          uint64_t record_bytes, uint8_t *status, uint8_t *span_flag) {
  swb_sampler::Sprite s[SWB_MAX_SLOTS];
  bool occupied[SWB_MAX_SLOTS];
  for (int64_t r = 0; r < n; ++r) {
    uint32_t occ = 0, bits = 0;
    bool any_concave = false;
    for (int j = 0; j < S; ++j) {
      bool concave = false;
      bits |= swb_make::read_slot(*cols, (size_t)r * S + j, s[j], occupied[j], concave);
      occ |= (uint32_t)occupied[j] << j;
      any_concave = any_concave || concave;
    }
    const int32_t step = step_count ? step_count[r] : 0;
    const uint32_t st = swb_make::record_status(bits, occ, S, step);
    unsigned char *rec = records + (size_t)r * record_bytes;
    for (int j = 0; j < S; ++j)
      swb::write_record(rec, S, G, j, swb_make::make_slot(*prog, s[j], occupied[j], st, st ? 0 : step));
    swb::write_goals(swb::record_goals(rec, S, G), st || !G ? nullptr : goals + (size_t)r * G * 2, G);
    status[r] = (uint8_t)st;
    if (span_flag && any_concave && !st) *span_flag = 1;
  }
}

}  // extern "C"
