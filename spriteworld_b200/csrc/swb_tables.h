// Host-side construction of the resampling tables the render kernel consumes.
//
// Restates Pillow's Resample.c precompute_coeffs + normalize_coeffs_8bpc for the LANCZOS
// filter (the arithmetic behind `canvas.resize(image_size, Image.ANTIALIAS)`,
// renderers/pil_renderer.py:84): support 3*scale, window [int(c-s+.5), int(c+s+.5)),
// taps normalised in double and quantised to 22-bit fixed point.  On top of the raw taps
// the kernel wants: a class id per output (outputs with identical tap vectors share one
// table), prefix sums per class (horizontal pass over piecewise-constant rows; one row of
// max_len + 1 entries per class, at least 33: 33 up to 5x, 37 at 6x, 61 at 10x), the
// inverse maps "input index -> first/last output whose window contains it" and, for the
// vertical pass, the tap matrix of every block of eight outputs as tensor-core fragments.
#pragma once
#include <algorithm>
#include <array>
#include <cmath>
#include <cstdint>
#include <map>
#include <string>
#include <vector>

#include "swb_device.cuh"

namespace swb {

constexpr int kPrecisionBits = 32 - 8 - 2;  // Pillow PRECISION_BITS

struct AxisHost {
  int n_in = 0, n_out = 0, n_cls = 0, max_len = 0;
  int prefix_stride = 1;         // max(max_len + 1, kNarrowPrefixStride)
  std::vector<int16_t> win_min;
  std::vector<uint8_t> win_len, win_cls;
  std::vector<int32_t> prefix;   // [n_cls][prefix_stride]
  std::vector<int16_t> first_out, last_out;
  std::vector<std::vector<int32_t>> taps;  // per output, for tests
};

inline double sinc_filter(double x) {
  if (x == 0.0) return 1.0;
  x = x * M_PI;
  return std::sin(x) / x;
}
inline double lanczos_filter(double x) {
  if (-3.0 <= x && x < 3.0) return sinc_filter(x) * sinc_filter(x / 3);
  return 0.0;
}

inline bool build_axis(int n_in, int n_out, AxisHost *ax, std::string *err) {
  ax->n_in = n_in;
  ax->n_out = n_out;
  ax->win_min.assign(n_out, 0);
  ax->win_len.assign(n_out, 0);
  ax->win_cls.assign(n_out, 0);
  ax->taps.assign(n_out, {});
  if (n_in == n_out) {
    // Image.resize returns a plain copy when the size does not change (anti_aliasing=1)
    for (int xx = 0; xx < n_out; ++xx) {
      ax->win_min[xx] = (int16_t)xx;
      ax->win_len[xx] = 1;
      ax->taps[xx] = {1 << kPrecisionBits};
    }
  } else {
    const double scale = (double)n_in / n_out;
    const double filterscale = scale < 1.0 ? 1.0 : scale;
    const double support = 3.0 * filterscale;
    const int ksize = (int)std::ceil(support) * 2 + 1;
    std::vector<double> k(ksize);
    for (int xx = 0; xx < n_out; ++xx) {
      const double center = (xx + 0.5) * scale;
      double ww = 0.0;
      const double ss = 1.0 / filterscale;
      int xmin = (int)(center - support + 0.5);
      if (xmin < 0) xmin = 0;
      int xmax = (int)(center + support + 0.5);
      if (xmax > n_in) xmax = n_in;
      xmax -= xmin;
      for (int x = 0; x < xmax; ++x) {
        const double w = lanczos_filter((x + xmin - center + 0.5) * ss);
        k[x] = w;
        ww += w;
      }
      for (int x = 0; x < xmax; ++x)
        if (ww != 0.0) k[x] /= ww;
      if (xmax > 255) {  // win_len and the kernel's packed windows hold 8 bits
        *err = "tap window of " + std::to_string(xmax) + " > 255 taps";
        return false;
      }
      ax->win_min[xx] = (int16_t)xmin;
      ax->win_len[xx] = (uint8_t)xmax;
      ax->taps[xx].resize(xmax);
      for (int x = 0; x < xmax; ++x) {
        const double v = k[x] * (1 << kPrecisionBits);
        ax->taps[xx][x] = (v < 0) ? (int)(-0.5 + v) : (int)(0.5 + v);
      }
    }
  }
  // classes
  std::map<std::vector<int32_t>, int> cls;
  for (int xx = 0; xx < n_out; ++xx) {
    auto it = cls.find(ax->taps[xx]);
    int id;
    if (it == cls.end()) {
      id = (int)cls.size();
      cls.emplace(ax->taps[xx], id);
    } else {
      id = it->second;
    }
    if (id > 255) {
      *err = "more than 256 distinct tap vectors on one axis";
      return false;
    }
    ax->win_cls[xx] = (uint8_t)id;
    ax->max_len = std::max<int>(ax->max_len, ax->win_len[xx]);
  }
  ax->n_cls = (int)cls.size();
  ax->prefix_stride = std::max(ax->max_len + 1, kNarrowPrefixStride);
  ax->prefix.assign((size_t)ax->n_cls * ax->prefix_stride, 0);
  for (const auto &kv : cls) {
    const std::vector<int32_t> &t = kv.first;
    int32_t *P = ax->prefix.data() + (size_t)kv.second * ax->prefix_stride;
    int32_t run = 0;
    for (int i = 0; i < ax->prefix_stride; ++i) {
      P[i] = run;
      if (i < (int)t.size()) run += t[i];
    }
  }
  // inverse maps
  ax->first_out.assign(n_in, (int16_t)(n_out - 1));
  ax->last_out.assign(n_in, 0);
  std::vector<char> seen(n_in, 0);
  for (int xx = 0; xx < n_out; ++xx) {
    for (int i = ax->win_min[xx]; i < ax->win_min[xx] + ax->win_len[xx]; ++i) {
      if (!seen[i]) {
        seen[i] = 1;
        ax->first_out[i] = (int16_t)xx;
        ax->last_out[i] = (int16_t)xx;
      } else {
        ax->first_out[i] = std::min<int16_t>(ax->first_out[i], (int16_t)xx);
        ax->last_out[i] = std::max<int16_t>(ax->last_out[i], (int16_t)xx);
      }
    }
  }
  // an input index no window touches contributes to no output: map it to an empty range
  for (int i = 0; i < n_in; ++i)
    if (!seen[i]) {
      ax->first_out[i] = 1;
      ax->last_out[i] = 0;
    }
  return true;
}

// Canvas rows the vertical tap windows of a phase-C tile of `tb` blocks of eight output rows span
// at most.  Bands are `band_rows` output rows; a tile may start at any block of a band and never
// crosses into the next one, and its rows are counted from a multiple of four (the H tile packs
// four canvas rows into a word).
inline int tile_span(const AxisHost &ay, int band_rows, int tb) {
  int span = 0;
  for (int y0 = 0; y0 < ay.n_out; y0 += band_rows) {
    const int y1 = std::min(y0 + band_rows, ay.n_out) - 1;
    for (int t0 = y0; t0 <= y1; t0 += 8) {
      const int t1 = std::min(t0 + 8 * tb - 1, y1);
      span = std::max(span, ay.win_min[t1] + ay.win_len[t1] - (ay.win_min[t0] & ~3));
    }
  }
  return span;
}

// Blocks per phase-C tile: the largest tb <= max_blocks whose tiles span at most max_rows canvas
// rows, or 0 if not even one block fits.
inline int choose_tile_blocks(const AxisHost &ay, int band_rows, int max_blocks, int max_rows) {
  int tb = max_blocks;
  while (tb > 0 && tile_span(ay, band_rows, tb) > max_rows) --tb;
  return tb;
}

// Vertical pass as a banded integer contraction on the tensor pipe.
//
// out[yo][n] = clip8((2^21 + sum_r K[yo][r] * Hval[r][n]) >> 22), Hval uint8, K the 22-bit taps
// (Pillow ImagingResampleVertical_8bpc).  The render kernel evaluates it per block of eight
// output rows with mma.sync.m16n8k32 (A = 16 H columns x 32 canvas rows of uint8, B = 32
// canvas rows x 8 output rows of int8, int32 accumulators): K = l0 + 2^8 l1 + 2^16 l2 with
// l0, l1 in [-128, 127], one MMA per limb, recombined with shifts -- exact in int32 because
// the true sum is below 2^31.  A block's canvas rows are addressed from the 4-aligned row
// o = win_min[8b] & ~3 (four consecutive canvas rows share one 32-bit word of the H tile).
// Blocks with the same matrix share a class; per class the fragments are stored in the
// register layout of the instruction: lane (g = lane/4, t = lane%4) holds for output row g
// b0 = limb(K[8b+g][o + 32ks + 4t + 0..3]) and b1 = the same 16 rows further.
struct VFragHost {
  int nks = 1, n_cls = 0;
  std::vector<uint8_t> blk_cls;   // [ceil(n_out/8)]
  std::vector<uint32_t> frag;     // [n_cls][nks][3][32][2]
};

inline bool build_vfrag(const AxisHost &ay, VFragHost *vf, std::string *err) {
  const int n_blk = (ay.n_out + 7) / 8;
  auto coef = [&](int yo, int r) -> int32_t {
    if (yo >= ay.n_out) return 0;
    const int i = r - ay.win_min[yo];
    return (i >= 0 && i < (int)ay.win_len[yo]) ? ay.taps[yo][i] : 0;
  };
  int nks = 1;
  for (int b = 0; b < n_blk; ++b) {
    const int o = ay.win_min[8 * b] & ~3;
    int end = o + 1;
    for (int j = 0; j < 8 && 8 * b + j < ay.n_out; ++j) {
      const int yo = 8 * b + j;
      int last = (int)ay.win_len[yo] - 1;  // trailing zero taps need no k-step (5x LANCZOS: tap 29)
      while (last > 0 && ay.taps[yo][last] == 0) --last;
      end = std::max(end, ay.win_min[yo] + last + 1);
    }
    nks = std::max(nks, (end - o + 31) / 32);
  }
  vf->nks = nks;
  vf->blk_cls.assign(n_blk, 0);
  std::map<std::vector<uint32_t>, int> classes;
  std::vector<std::vector<uint32_t>> ordered;
  for (int b = 0; b < n_blk; ++b) {
    const int o = ay.win_min[8 * b] & ~3;
    std::vector<uint32_t> f((size_t)nks * 3 * 32 * 2, 0u);
    for (int ks = 0; ks < nks; ++ks)
      for (int lane = 0; lane < 32; ++lane) {
        const int g = lane >> 2, t = lane & 3;
        for (int half = 0; half < 2; ++half) {
          uint32_t w[3] = {0u, 0u, 0u};
          for (int i = 0; i < 4; ++i) {
            const int32_t k = coef(8 * b + g, o + 32 * ks + 16 * half + 4 * t + i);
            const int32_t l0 = ((k + 128) & 255) - 128;
            const int32_t k1 = (k - l0) >> 8;
            const int32_t l1 = ((k1 + 128) & 255) - 128;
            const int32_t l2 = (k1 - l1) >> 8;
            if (l2 < -128 || l2 > 127) {
              *err = "resampling coefficient does not fit three signed 8-bit limbs";
              return false;
            }
            w[0] |= (uint32_t)(uint8_t)(int8_t)l0 << (8 * i);
            w[1] |= (uint32_t)(uint8_t)(int8_t)l1 << (8 * i);
            w[2] |= (uint32_t)(uint8_t)(int8_t)l2 << (8 * i);
          }
          for (int limb = 0; limb < 3; ++limb)
            f[(((size_t)ks * 3 + limb) * 32 + lane) * 2 + half] = w[limb];
        }
      }
    auto it = classes.find(f);
    int id;
    if (it == classes.end()) {
      id = (int)classes.size();
      if (id > 255) {
        *err = "more than 256 distinct vertical tap blocks";
        return false;
      }
      classes.emplace(f, id);
      ordered.push_back(f);
    } else {
      id = it->second;
    }
    vf->blk_cls[b] = (uint8_t)id;
  }
  vf->n_cls = (int)ordered.size();
  vf->frag.clear();
  for (const auto &f : ordered) vf->frag.insert(vf->frag.end(), f.begin(), f.end());
  return true;
}

}  // namespace swb
