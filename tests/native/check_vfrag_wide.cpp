// Host-only check of the resampling tables at anti_aliasing 6 and more (swb_tables.h).
//
// For each (canvas rows, output rows) pair: the vertical-pass fragments are expanded back
// through the register layout of mma.sync.m16n8k32, exactly as tests/native/check_vfrag.cpp
// does, and compared with the direct convolution with Pillow's 22-bit taps; every class of the
// prefix table must run from 0 to the sum of its taps and stay there up to the table's stride.
// Prints one line per pair with the k-step count and the phase-C tile blocks the render kernel
// would use (0: swb_raster_create refuses the raster); exit code 1 on any mismatch.
#include <cstdio>
#include <cstdlib>

#include "../../spriteworld_b200/csrc/swb_tables.h"

using namespace swb;

constexpr int kBandRows = 64;       // swb_raster_create: output rows per band
constexpr int kTileBlocks = 3;      // TILE_BLOCKS
constexpr int kTileRows = 4 * 44;   // canvas rows of the H tile (4 * HT_ROWW)

static long prefix_errors(const AxisHost &ax) {
  long bad = 0;
  if (ax.prefix_stride != std::max(ax.max_len + 1, kNarrowPrefixStride) ||
      (int)ax.prefix.size() != ax.n_cls * ax.prefix_stride)
    return 1;
  for (int xx = 0; xx < ax.n_out; ++xx) {
    const int32_t *P = ax.prefix.data() + (size_t)ax.win_cls[xx] * ax.prefix_stride;
    int32_t run = 0;
    for (int i = 0; i < ax.prefix_stride; ++i) {
      bad += P[i] != run;
      if (i < ax.win_len[xx]) run += ax.taps[xx][i];
    }
    int32_t sum = 0;
    for (int32_t t : ax.taps[xx]) sum += t;
    bad += P[ax.win_len[xx]] != sum;
  }
  return bad;
}

int main() {
  // {output rows, anti_aliasing}: 64- and 100-row frames at 6..14, the 315-pixel side of a
  // 4095-pixel canvas at 13, and a short frame above 13
  const int cfgs[][2] = {{64, 6},  {64, 7},  {64, 8},  {64, 9},  {64, 10},  {64, 11},  {64, 12},
                         {64, 13}, {64, 14}, {100, 6}, {100, 7}, {100, 8}, {100, 9}, {100, 10},
                         {100, 11}, {100, 12}, {100, 13}, {100, 14}, {315, 13}, {128, 10},
                         {256, 10}, {8, 20}};
  long total_bad = 0;
  srand(4321);
  for (const auto &c : cfgs) {
    const int n_out = c[0], aa = c[1], n_in = n_out * aa;
    AxisHost ay;
    std::string err;
    if (!build_axis(n_in, n_out, &ay, &err)) { printf("axis %d->%d: %s\n", n_in, n_out, err.c_str()); return 1; }
    const long pbad = prefix_errors(ay);
    const int tb = choose_tile_blocks(ay, n_out <= kBandRows ? n_out : kBandRows, kTileBlocks, kTileRows);
    VFragHost vf;
    if (!build_vfrag(ay, &vf, &err)) { printf("vfrag %d->%d: %s\n", n_in, n_out, err.c_str()); return 1; }
    const int n_blk = (n_out + 7) / 8;
    long bad = 0;
    for (int b = 0; b < n_blk; ++b) {
      const int o = ay.win_min[8 * b] & ~3;
      std::vector<int> h(n_in + 32 * vf.nks + 8);
      for (auto &v : h) v = rand() & 255;
      const uint32_t *f = vf.frag.data() + (size_t)vf.blk_cls[b] * vf.nks * 3 * 32 * 2;
      for (int g = 0; g < 8; ++g) {
        const int yo = 8 * b + g;
        if (yo >= n_out) continue;
        int32_t acc[3] = {0, 0, 0};
        for (int ks = 0; ks < vf.nks; ++ks)
          for (int t = 0; t < 4; ++t)
            for (int half = 0; half < 2; ++half)
              for (int i = 0; i < 4; ++i) {
                const int row = o + 32 * ks + 16 * half + 4 * t + i;
                const int hv = row < (int)h.size() ? h[row] : 0;
                for (int limb = 0; limb < 3; ++limb) {
                  const uint32_t w = f[(((size_t)ks * 3 + limb) * 32 + (g * 4 + t)) * 2 + half];
                  acc[limb] += hv * (int)(int8_t)((w >> (8 * i)) & 255u);
                }
              }
        const int32_t got = (int32_t)((uint32_t)acc[0] + ((uint32_t)acc[1] << 8) + ((uint32_t)acc[2] << 16));
        int64_t want = 0;
        for (int i = 0; i < ay.win_len[yo]; ++i) want += (int64_t)ay.taps[yo][i] * h[ay.win_min[yo] + i];
        if (want != got) ++bad;
      }
    }
    printf("%d -> %d: aa %d, window %d, prefix stride %d, k-steps %d, tile blocks %d, one-block span %d, "
           "classes %d, prefix errors %ld, mismatches %ld\n",
           n_in, n_out, aa, ay.max_len, ay.prefix_stride, vf.nks, tb,
           tile_span(ay, n_out <= kBandRows ? n_out : kBandRows, 1), vf.n_cls, pbad, bad);
    total_bad += bad + pbad;
  }
  return total_bad ? 1 : 0;
}
