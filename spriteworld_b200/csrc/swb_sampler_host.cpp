// The device scene sampler (swb_sampler.cuh) built for the CPU: the restatement the tests hold the
// CUDA kernels to, and a way to draw the device's scenes without a GPU.  Same source, no
// contraction (-ffp-contract=off), so it computes what the kernels compute, bit for bit.
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
  for (int64_t i = 0; i < n; ++i) {
    const int bad = swb_sampler::sample_and_pack(
        *prog, seed, (uint64_t)env_ids[i], (uint64_t)scene_idx[i], S, sc,
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

}  // extern "C"
