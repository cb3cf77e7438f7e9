// Counter-based scene sampler: scene `a` of global env `g` is a pure function of (seed, g, a).
//
// The scene generator (init_sprites) arrives flattened into a swb_scene_program
// (include/spriteworld_b200.h; built by spriteworld_b200/scene_program.py).  One thread runs the
// program for one scene: it draws the sprites' factors, then packs them into the pool's
// struct-of-arrays exactly as scene.arrays_from_layout packs the same factor values.
//
// This file is plain C++ for host and device (SWB_HD): the CUDA library runs it in its kernels,
// and csrc/swb_sampler_host.cpp builds the same source for the CPU, as the restatement the tests
// compare the device against.  Both builds run without contraction (-fmad=false,
// -ffp-contract=off), so every double and float operation rounds as NumPy's does.
//
// Random numbers: Philox4x64-10 (Salmon et al., SC'11), the generator of np.random.Philox, with
//   key     = (seed, SWB_SAMPLER_DOMAIN)
//   counter = (block, a, g, 0)
// Block b gives the scene's draw words 4b .. 4b+3, in order; a scene consumes its words one by one
// from word 0.  np.random.Philox(counter=(b - 1, a, g, 0), key=(seed, SWB_SAMPLER_DOMAIN))
// .random_raw(4) gives block b for b >= 1 (NumPy increments the counter before each block).
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/spriteworld_b200.h"

#ifdef __CUDACC__
#define SWB_HD __host__ __device__ __forceinline__
#else
#define SWB_HD inline
#endif

namespace swb_sampler {

static const uint64_t kPhiloxM0 = 0xD2E7470EE14C6C93ULL, kPhiloxM1 = 0xCA5A826395121157ULL;
static const uint64_t kPhiloxW0 = 0x9E3779B97F4A7C15ULL, kPhiloxW1 = 0xBB67AE8584CAA73BULL;
enum { kFactors = 10 };  // x, y, shape, angle, scale, c0, c1, c2, x_vel, y_vel (sprite.py)
enum { F_X = 0, F_Y = 1, F_SHAPE = 2, F_ANGLE = 3, F_SCALE = 4, F_C0 = 5, F_C1 = 6, F_C2 = 7,
       F_VX = 8, F_VY = 9 };

SWB_HD uint64_t mulhi64(uint64_t a, uint64_t b) {
#ifdef __CUDA_ARCH__
  return __umul64hi(a, b);
#else
  return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}

// Philox4x64 with 10 rounds: ctr <- f(ctr, key), in place.
SWB_HD void philox4x64_10(uint64_t ctr[4], uint64_t k0, uint64_t k1) {
  for (int r = 0; r < 10; ++r) {
    if (r) { k0 += kPhiloxW0; k1 += kPhiloxW1; }
    const uint64_t lo0 = kPhiloxM0 * ctr[0], hi0 = mulhi64(kPhiloxM0, ctr[0]);
    const uint64_t lo1 = kPhiloxM1 * ctr[2], hi1 = mulhi64(kPhiloxM1, ctr[2]);
    const uint64_t c1 = ctr[1], c3 = ctr[3];
    ctr[0] = hi1 ^ c1 ^ k0;
    ctr[1] = lo1;
    ctr[2] = hi0 ^ c3 ^ k1;
    ctr[3] = lo0;
  }
}

// The draw stream of one scene (key word 1 = SWB_SAMPLER_DOMAIN), or of another counter-based
// stream of the library under its own domain word (swb_contained.cuh).
struct Stream {
  uint64_t key, domain, g, a, block;
  uint64_t buf[4];
  int pos;
  SWB_HD void init(uint64_t seed, uint64_t g_, uint64_t a_, uint64_t domain_ = SWB_SAMPLER_DOMAIN) {
    key = seed; domain = domain_; g = g_; a = a_; block = 0; pos = 4;
  }
  SWB_HD uint64_t next() {
    if (pos == 4) {
      buf[0] = block++; buf[1] = a; buf[2] = g; buf[3] = 0;
      philox4x64_10(buf, key, domain);
      pos = 0;
    }
    return buf[pos++];
  }
  // NumPy's random_sample / next_double: 53 random bits
  SWB_HD double uniform() { return (double)(next() >> 11) * (1.0 / 9007199254740992.0); }
  // an index in [0, n): the high word of a 64x64-bit product (bias below n / 2^64)
  SWB_HD int64_t below(int64_t n) { return (int64_t)mulhi64(next(), (uint64_t)n); }
};

// Float-to-integer conversions as NumPy's astype makes them on x86-64: truncation toward zero,
// and INT32_MIN / INT64_MIN for a value out of range or NaN (what cvttsd2si returns).  C++ leaves
// such conversions undefined and the device's cvt instructions saturate, so both builds convert
// through these.
SWB_HD int32_t trunc_i32(double v) {
  return (v > -2147483649.0 && v < 2147483648.0) ? (int32_t)v : INT32_MIN;
}
SWB_HD int64_t trunc_i64(double v) {
  return (v >= -9223372036854775808.0 && v < 9223372036854775808.0) ? (int64_t)v : INT64_MIN;
}
// astype(np.uint64): values from 2^63 up are converted less 2^63, and the top bit set again
SWB_HD uint64_t trunc_u64(double v) {
  return v >= 9223372036854775808.0
             ? (uint64_t)trunc_i64(v - 9223372036854775808.0) ^ 0x8000000000000000ULL
             : (uint64_t)trunc_i64(v);
}
// astype(np.uint8) of a float: through int32, so -153.2 gives 103 and anything beyond int32 gives 0
SWB_HD uint8_t float_to_u8(double v) { return (uint8_t)trunc_i32(v); }

SWB_HD bool small_int(int k) {
  return k == SWB_FT_I8 || k == SWB_FT_U8 || k == SWB_FT_I16 || k == SWB_FT_U16;
}

// value (numpy scalar of kind `vk`) against a constant of kind `ck` (a Python float or int, or a
// numpy scalar), as NumPy compares them: a Python float or int meeting a float32 value is cast to
// float32 (NEP 50), anything else compares exactly -- in float64, which holds every value a draw
// can have and every constant compile_program accepts (it refuses integers float64 cannot hold).
// Returns -1, 0 or 1; 2 if the two do not compare (a shape name against a number).
SWB_HD int compare(double v, int vk, double c, int ck) {
  if (vk == SWB_FT_SHAPE || ck == SWB_FT_SHAPE)
    return (vk == ck) ? (v == c ? 0 : (v < c ? -1 : 1)) : 2;
  if (vk == SWB_FT_F32 && (ck == SWB_FT_PYFLOAT || ck == SWB_FT_PYINT || ck == SWB_FT_F32)) {
    const float a = (float)v, b = (float)c;
    return a == b ? 0 : (a < b ? -1 : 1);
  }
  return v == c ? 0 : (v < c ? -1 : 1);
}

// .astype(dtype) of a float64 draw: integer dtypes truncate (the program's ranges fit the type;
// a draw that rounds up to `hi` wraps as the conversion through int64 does)
SWB_HD double cast_draw(double v, int kind) {
  switch (kind) {
    case SWB_FT_F32: return (double)(float)v;
    case SWB_FT_F64: return v;
    case SWB_FT_U64: return (double)trunc_u64(v);
    default: break;
  }
  const int64_t i = trunc_i64(v);
  switch (kind) {
    case SWB_FT_I8: return (double)(int8_t)i;
    case SWB_FT_I16: return (double)(int16_t)i;
    case SWB_FT_I32: return (double)(int32_t)i;
    case SWB_FT_U8: return (double)(uint8_t)i;
    case SWB_FT_U16: return (double)(uint16_t)i;
    case SWB_FT_U32: return (double)(uint32_t)i;
    default: return (double)i;
  }
}

struct Sprite {
  double val[kFactors];
  uint8_t kind[kFactors];
};

SWB_HD void set_defaults(Sprite &s) {
  // Sprite.__init__ defaults (sprite.py), typed as scene._default_column types them
  const double v[kFactors] = {0.5, 0.5, 2.0 /* ShapeType.square */, 0.0, 0.1, 0.0, 0.0, 0.0, 0.0, 0.0};
  const uint8_t k[kFactors] = {SWB_FT_F64, SWB_FT_F64, SWB_FT_SHAPE, SWB_FT_I64, SWB_FT_F64,
                               SWB_FT_I64, SWB_FT_I64, SWB_FT_I64, SWB_FT_F64, SWB_FT_F64};
  for (int f = 0; f < kFactors; ++f) { s.val[f] = v[f]; s.kind[f] = k[f]; }
}

// Evaluates the predicate code at `pc` (containment in a distribution) on one sprite.
SWB_HD bool contains(const swb_scene_program &p, int pc, const Sprite &s) {
  bool stack[SWB_PROG_MAX_STACK];
  int sp = 0;
  for (;; ++pc) {
    const swb_prog_op &o = p.ops[pc];
    switch (o.op) {
      case SWB_OP_P_CONT: {
        const int lo = compare(s.val[o.key], s.kind[o.key], o.lo, o.a);
        const int hi = compare(s.val[o.key], s.kind[o.key], o.hi, o.b);
        stack[sp++] = (lo == 0 || lo == 1) && hi == -1;
        break;
      }
      case SWB_OP_P_DISC: {
        bool in = false;
        for (int i = 0; i < o.b && !in; ++i)
          in = compare(s.val[o.key], s.kind[o.key], p.consts[o.a + i], p.const_kind[o.a + i]) == 0;
        stack[sp++] = in;
        break;
      }
      case SWB_OP_P_AND: case SWB_OP_P_OR: {
        bool r = o.op == SWB_OP_P_AND;
        for (int i = 0; i < o.b; ++i) {
          const bool x = stack[--sp];
          r = (o.op == SWB_OP_P_AND) ? (r && x) : (r || x);
        }
        stack[sp++] = r;
        break;
      }
      case SWB_OP_P_NOT: stack[sp - 1] = !stack[sp - 1]; break;
      default: return sp ? stack[sp - 1] : false;  // SWB_OP_P_RET
    }
  }
}

// The cdf search of np.random.choice: the first index whose cdf entry exceeds u.
SWB_HD int cdf_index(const double *cdf, int n, double u) {
  int i = 0;
  while (i < n - 1 && !(cdf[i] > u)) ++i;
  return i;
}

// Draws one sprite's factors with the distribution code at `pc`.  Returns -1, or the program
// op of a rejection loop that ran out of tries.
SWB_HD int sample_sprite(const swb_scene_program &p, int pc, Stream &rng, Sprite &s) {
  int rej_pc[SWB_PROG_MAX_STACK];
  int32_t rej_tries[SWB_PROG_MAX_STACK];
  int rp = 0;
  for (;;) {
    const swb_prog_op &o = p.ops[pc];
    switch (o.op) {
      case SWB_OP_D_CONT: {
        const double u = rng.uniform();
        s.val[o.key] = cast_draw(o.lo + (o.hi - o.lo) * u, o.dtype);
        s.kind[o.key] = (uint8_t)o.dtype;
        ++pc;
        break;
      }
      case SWB_OP_D_DISC: {
        const int i = o.c < 0 ? (int)rng.below(o.b) : cdf_index(p.consts + o.c, o.b, rng.uniform());
        s.val[o.key] = p.consts[o.a + i];
        s.kind[o.key] = (uint8_t)o.dtype;
        ++pc;
        break;
      }
      case SWB_OP_D_MIX:   // followed by o.b D_JUMPs, one per component
        pc = pc + 1 + cdf_index(p.consts + o.c, o.b, rng.uniform());
        break;
      case SWB_OP_D_JUMP: pc = o.a; break;
      case SWB_OP_D_REJ_BEGIN:
        rej_pc[rp] = pc + 1;
        rej_tries[rp++] = 0;
        ++pc;
        break;
      case SWB_OP_D_REJ_END: {
        const bool accept = contains(p, o.a, s) == (o.b != 0);
        if (accept) { --rp; ++pc; break; }
        if (++rej_tries[rp - 1] >= SWB_SAMPLER_MAX_TRIES) return pc;
        pc = rej_pc[rp - 1];
        break;
      }
      default: return -1;  // SWB_OP_D_RET
    }
  }
}

// A scene's sprites in back-to-front order: n of them, sprite order[i] at position i.
struct Scene {
  Sprite spr[SWB_MAX_SLOTS];
  int order[SWB_MAX_SLOTS];
  int n;
};

// Runs the generator code of the program (from op 0).  Returns -1, or the op of a failed
// rejection loop (the scene is then empty).
SWB_HD int sample_scene(const swb_scene_program &p, Stream &rng, Scene &sc) {
  int marks[SWB_PROG_MAX_STACK];
  int mp = 0;
  bool overflow = false;
  sc.n = 0;
  for (int pc = 0;;) {
    const swb_prog_op &o = p.ops[pc];
    switch (o.op) {
      case SWB_OP_G_SPRITES: {
        int count = o.dtype ? (int)(o.b + rng.below((int64_t)o.c - o.b)) : o.b;
        // a program whose counts exceed the slot bound (not one compile_program builds) keeps the
        // first SWB_MAX_SLOTS sprites; sample_and_pack then leaves such a scene empty
        if (count > SWB_MAX_SLOTS - sc.n) { count = SWB_MAX_SLOTS - sc.n; overflow = true; }
        for (int j = 0; j < count; ++j) {
          Sprite &s = sc.spr[sc.n];
          set_defaults(s);
          const int bad = sample_sprite(p, o.a, rng, s);
          if (bad >= 0) { sc.n = 0; return bad; }
          sc.order[sc.n] = sc.n;
          ++sc.n;
        }
        ++pc;
        break;
      }
      case SWB_OP_G_MARK: marks[mp++] = sc.n; ++pc; break;
      case SWB_OP_G_SHUFFLE: {  // Fisher-Yates over the positions since the matching mark
        const int lo = marks[--mp];
        for (int i = sc.n - 1; i > lo; --i) {
          const int j = lo + (int)rng.below(i - lo + 1);
          const int t = sc.order[i]; sc.order[i] = sc.order[j]; sc.order[j] = t;
        }
        ++pc;
        break;
      }
      case SWB_OP_G_CHOOSE:   // followed by o.b G_JUMPs, one per generator
        pc = pc + 1 + cdf_index(p.consts + o.c, o.b, rng.uniform());
        break;
      case SWB_OP_G_JUMP: pc = o.a; break;
      default:  // SWB_OP_G_END
        if (overflow) sc.n = SWB_MAX_SLOTS + 1;
        return -1;
    }
  }
}

// (cos, sin) of an angle value: the program's table, built on the host with libm
// (scene.transform_matrix).  The table is sorted by value; equal values are told apart by sign.
SWB_HD void angle_cs(const swb_scene_program &p, double angle, double &c, double &s) {
  int lo = 0, hi = p.n_angles;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (p.angle[mid] < angle) lo = mid + 1; else hi = mid;
  }
  for (int i = lo; i < p.n_angles && p.angle[i] == angle; ++i)
    if (signbit(p.angle[i]) == signbit(angle)) { c = p.angle_cos[i]; s = p.angle_sin[i]; return; }
  c = 1.0; s = 0.0;  // not reached: the program holds every angle its code can draw
}

template <typename T>
SWB_HD void hsv_to_rgb(T h, T s, T v, uint8_t out[3]) {
  // colorsys.hsv_to_rgb, then (255 * rgb).astype(uint8) (color_maps.py, swb_host_pack.c)
  const T one = (T)1.0, six = (T)6.0, scale = (T)255;
  const T h6 = h * six;
  const int64_t it = trunc_i64((double)h6);
  const T f = h6 - (T)it;
  const T sf = s * f;
  const T pp = v * (one - s);
  const T q = v * (one - sf);
  const T omf = one - f;
  const T somf = s * omf;
  const T t = v * (one - somf);
  int64_t m = it % 6;
  if (m < 0) m += 6;
  T r, g, b;
  switch (m) {
    case 0: r = v; g = t; b = pp; break;
    case 1: r = q; g = v; b = pp; break;
    case 2: r = pp; g = v; b = t; break;
    case 3: r = pp; g = q; b = v; break;
    case 4: r = t; g = pp; b = v; break;
    default: r = v; g = pp; b = q; break;
  }
  if (s == (T)0) { r = v; g = v; b = v; }
  out[0] = float_to_u8((double)(scale * r));
  out[1] = float_to_u8((double)(scale * g));
  out[2] = float_to_u8((double)(scale * b));
}

// One packed slot, the fields of swb_scene_soa.
struct Packed {
  double x, y, m00, m01, m10, m11, vx, vy;
  uint32_t member;
  uint8_t shape, pos_f32, rgb[3];
  float factors[5];
};

// scene._table_arrays for one sprite.
SWB_HD void pack_sprite(const swb_scene_program &p, const Sprite &s, Packed &o) {
  o.x = s.val[F_X];
  o.y = s.val[F_Y];
  o.vx = s.val[F_VX];
  o.vy = s.val[F_VY];
  const double scale = s.val[F_SCALE];
  double c, sn;
  angle_cs(p, s.val[F_ANGLE], c, sn);
  o.m00 = c * scale; o.m01 = (-sn) * scale; o.m10 = sn * scale; o.m11 = c * scale;
  // the filters see the sprite's position, np.array([x, y]): float32 if one is float32 and the
  // other float32 or an integer float32 holds (at most 16 bits), float64 (or an integer dtype,
  // which compares alike) otherwise
  const int kx = s.kind[F_X], ky = s.kind[F_Y];
  const bool pos_f32 = (kx == SWB_FT_F32 && (ky == SWB_FT_F32 || small_int(ky))) ||
                       (ky == SWB_FT_F32 && small_int(kx));
  Sprite t = s;
  t.kind[F_X] = t.kind[F_Y] = (uint8_t)(pos_f32 ? SWB_FT_F32 : SWB_FT_F64);
  uint32_t member = 0;
  for (int f = 0; f < p.n_filters; ++f)
    if (contains(p, p.filter_pc[f], t)) member |= 1u << f;
  o.member = member;
  o.shape = (uint8_t)s.val[F_SHAPE];
  o.pos_f32 = pos_f32;
  const double c0 = s.val[F_C0], c1 = s.val[F_C1], c2 = s.val[F_C2];
  if (p.color_mode == SWB_COLOR_HSV) {
    if (s.kind[F_C0] == SWB_FT_F32) hsv_to_rgb<float>((float)c0, (float)c1, (float)c2, o.rgb);
    else hsv_to_rgb<double>(c0, c1, c2, o.rgb);
  } else {  // RGB values: through int64, then uint8 with wraparound
    o.rgb[0] = (uint8_t)trunc_i64(c0); o.rgb[1] = (uint8_t)trunc_i64(c1); o.rgb[2] = (uint8_t)trunc_i64(c2);
  }
  o.factors[0] = (float)scale; o.factors[1] = (float)s.val[F_ANGLE];
  o.factors[2] = (float)c0; o.factors[3] = (float)c1; o.factors[4] = (float)c2;
}

SWB_HD void empty_slot(Packed &o) {
  o.x = o.y = o.m00 = o.m01 = o.m10 = o.m11 = o.vx = o.vy = 0.0;
  o.member = 0;
  o.shape = o.pos_f32 = 0;
  o.rgb[0] = o.rgb[1] = o.rgb[2] = 0;
  for (int f = 0; f < 5; ++f) o.factors[f] = 0.f;
}

// The scene's goals, drawn after its sprites from the same stream: goal slot i is the (x, y) that
// the distribution code at goal_pc[i] draws.  Returns -1, or the op of a failed rejection loop
// (that goal is then (0, 0)).
SWB_HD int sample_goals(const swb_scene_program &p, Stream &rng, double *goal) {
  int bad = -1;
  for (int i = 0; i < p.n_goals; ++i) {
    Sprite s;
    set_defaults(s);
    const int b = sample_sprite(p, p.goal_pc[i], rng, s);
    if (b >= 0 && bad < 0) bad = b;
    goal[2 * i] = b >= 0 ? 0.0 : s.val[F_X];
    goal[2 * i + 1] = b >= 0 ? 0.0 : s.val[F_Y];
  }
  return bad;
}

// Samples scene (g, a) and hands every one of its S slots to `put(slot, packed, sprite or null)`,
// empty slots first, and its goals to goal[0 .. 2 * n_goals).  Returns -1, or the op of a failed
// rejection loop (all slots empty then, if it was the sprites').  The goals come after the sprites,
// so a program's sprites do not depend on its goals.
template <typename Put>
SWB_HD int sample_and_pack(const swb_scene_program &p, uint64_t seed, uint64_t g, uint64_t a, int S,
                           Scene &sc, double *goal, Put &&put) {
  Stream rng;
  rng.init(seed, g, a);
  int bad = sample_scene(p, rng, sc);
  const int bad_goal = sample_goals(p, rng, goal);
  if (bad < 0) bad = bad_goal;
  const int n = sc.n <= S ? sc.n : 0;
  Packed o;
  for (int j = 0; j < S - n; ++j) {
    empty_slot(o);
    put(j, o, (const Sprite *)nullptr);
  }
  for (int i = 0; i < n; ++i) {
    const Sprite &s = sc.spr[sc.order[i]];
    pack_sprite(p, s, o);
    put(S - n + i, o, &s);
  }
  return bad;
}

}  // namespace swb_sampler
