// Render kernel: PILRenderer.render for E envs (renderers/pil_renderer.py:67-91).
//
// One CTA renders one band of one frame.  Nothing of the aa-times supersampled canvas is
// ever materialised; the CTA works on what Pillow's two stages are functions of:
//
//   A  vertices   int(canvas * (R.S.v + pos)) in fp64 (sprite.py:128-133, pil_renderer.py:81,
//                 Pillow's (int) truncation), then Pillow's edge records (float32 dx) and,
//                 per edge, the value Pillow's corner-joining refinement would overwrite
//                 its crossing with on its first row / on the polygon's last row.
//   B  spans      Pillow's scan conversion.  B1 is edge-parallel: every edge drops its
//                 float32 crossing (twice where it ends on an interior row) into the
//                 crossing list of each canvas row it spans.  B2 is row-parallel: per
//                 sprite, front to back, sort the list, pair it up with Pillow's
//                 ROUND_UP/ROUND_DOWN rule, add horizontal edges, and fold the spans into
//                 the row's list of VISIBLE segments (x range + sprite), i.e. the painter's
//                 algorithm resolved once per canvas row.
//   C  per sprite region (the outputs whose 2-D tap window can see the sprite), in tiles of
//      up to rd.tile_blocks (3; 2 or 1 where the vertical windows are too long for three)
//      blocks of eight output rows x 20 columns:
//        H  horizontal LANCZOS pass of the canvas rows the tile needs.  A canvas row is
//           piecewise constant, so an output is bg*K + sum_segments (colour-bg) * (P[b]-P[a])
//           with P the prefix sums of the 22-bit tap vector and [a, b) the segment clamped
//           to the tap window (branch-free), clip8'ed like Pillow's uint8 intermediate.
//           A thread owns two columns of four consecutive canvas rows and stores the four
//           uint8 results of a (column, channel) as one word: the H tile is laid out
//           [column*3 + channel][canvas row / 4], i.e. as the k-contiguous A operand of
//        V  the vertical pass on the integer tensor pipe: per block of eight output rows a
//           banded contraction out[yo][n] = sum_r K[yo][r] * H[r][n], mma.sync.m16n8k32
//           u8 x s8 -> s32 with the 22-bit taps cut into three signed 8-bit limbs (exact:
//           the sums stay below 2^31), clip8, written into the frame staged in shared memory.
//   D  the staged frame (background + tiles), rows flipped (np.flipud, pil_renderer.py:90),
//      goes to HBM through the bulk-copy engine.
//
// The kernel is persistent: a CTA claims (env, band) items from a counter until none is
// left, so the axis tables are loaded once per CTA, a frame's write-out overlaps the next
// frame's set-up, and no SM idles in a last partial wave.
//
// All pixel arithmetic is integer and associative, so the result is bit-identical to
// Pillow's; the float32 edge arithmetic uses explicit _rn intrinsics (no FMA).
#pragma once
#include <climits>

#include "swb_device.cuh"

namespace swb {

constexpr int R_THREADS = 256;
#ifndef SWB_RENDER_CTAS
#define SWB_RENDER_CTAS 5
#endif
constexpr int R_CTAS_PER_SM = SWB_RENDER_CTAS;  // resident CTAs per SM the register budget is set for
constexpr int R_CTAS_PER_SM_WIDE = 2;            // the same for render_kernel<., true>
constexpr int H_NC = 2;           // output columns one H-pass thread owns
constexpr int TILE_X_MAX = 20;    // output columns per tile
constexpr int TILE_BLOCKS = 3;    // most blocks of eight output rows per tile (RasterDev::tile_blocks)
constexpr int V_KS_NARROW = 3;    // most V-pass k-steps of render_kernel<., false>;
                                  // render_kernel<., true> takes up to V_KS_WIDE
constexpr int V_KS_WIDE = 6;      // a one-block tile spans at most 4 * HT_ROWW = 176 canvas rows: 6 k-steps
constexpr int HT_N = 3 * TILE_X_MAX;  // (column, channel) rows of the H tile; the fourth MMA row tile of 16
                                  // reads four rows (and a k-step's tail) past it, into the staged frame
                                  // that follows in shared memory: values that are never stored
constexpr int HT_ROWW = 44;       // words per row = 176 canvas rows; = 4 mod 8: fragment loads hit 32 banks
constexpr int HT_WORDS = HT_N * HT_ROWW;
constexpr int MAX_ROW_SPANS = 12;
constexpr int EV = SWB_MAX_VERTS;  // edge slots per sprite
static_assert(EV == 32, "phase A maps one lane to one vertex / edge");

// Where a frame goes.  Normally one buffer; with the frame gather fused into the kernel
// (swb_step_render_gather) one buffer per rank, each an [n_ranks * E] frame array reached
// over NVLink peer memory, written at env index env_offset + e.
struct RenderTargets {
  uint8_t *dst[SWB_MAX_PEERS];
  int n;
  int env_offset;
  int self;  // index of this rank's own buffer in dst
};

// Whether a raster needs render_kernel<., true>: tables beyond those of anti_aliasing <= 5
inline bool render_wide(const RasterDev &rd) {
  return rd.v_nks > V_KS_NARROW || rd.tile_blocks != TILE_BLOCKS || rd.prefix_stride != kNarrowPrefixStride;
}

struct RenderLayout {
  int S, rows, M, band_rows, W, aa, ncx, ncy, cap;
  int off_meta, off_edge_i, off_edge_f, off_edge_yr, off_hl, off_region;
  int off_nseg, off_segs, off_prefix, off_xwin, off_ywin, off_scratch, off_frame, total;
  int scratch_bytes, segcap;
  // exact_segs: with convex shapes only, size the segment table for every row a scene can
  // produce (2S-1 pieces); false caps it at 16 like the concave case
  // pstride: entries per class of the horizontal prefix table; nks: the raster's V-pass k-steps
  __host__ __device__ RenderLayout(int S_, int rows_, int M_, int band_rows_, int W_, int aa_,
                                   int ncx_, int ncy_, int pstride, int nks, bool exact_segs = true)
      : S(S_), rows(rows_), M(M_), band_rows(band_rows_), W(W_), aa(aa_), ncx(ncx_), ncy(ncy_) {
    int o = 0;
    auto take = [&](int bytes) { int r = o; o += (bytes + 15) & ~15; return r; };
    take(S * 16);                          // offset 0: colour - background per channel (int4 per sprite)
    off_meta = take(S * (10 + 8) * 4);     // 10 plan ints + 8 active-edge masks per sprite
    off_edge_i = take(S * EV * 2 * 4);     // x0, y0
    off_edge_f = take(S * EV * 3 * 4);     // dx, ovs (override on the first row), ove (on the last row)
    off_edge_yr = take(S * EV * 4);        // ymin | ymax<<16 of non-horizontal edges, empty otherwise
    off_hl = take(S * EV * 3 * 2);         // horizontal edges: y, xmin, xmax (int16)
    off_region = take(S * 4 * 2);
    // visible segments kept per canvas row: n one-span sprites leave at most 2n-1 pieces, so
    // with convex shapes only (M == 1) the exact table never overflows.  With several spans
    // per sprite row, or where the exact table does not fit, it is capped at 16: a row with
    // more visible pieces sets SWB_ENV_SPAN_OVERFLOW (DESIGN §8)
    segcap = M > 1 ? 16 : (2 * S - 1 < 3 ? 3 : 2 * S - 1);
    if (!exact_segs && segcap > 16) segcap = 16;
    off_nseg = take(((rows + 3) & ~3) + 8);  // +: quads of the H pass may end past the last row
    off_segs = take(rows * segcap * 4);
    off_prefix = take(ncx * pstride * 4);
    off_xwin = take(W * 4);                // per output column: win_min | len<<16 | cls<<24
    off_ywin = take(band_rows * 4);
    cap = (M > 1) ? 16 : 8;                // crossings kept per (sprite, row)
    // scratch = H tile + staged frame; phase B aliases it with the per-row crossing lists and
    // spans of a chunk of sprites, so it must hold at least one sprite spanning every row
    const int frame_bytes = band_rows * W * 3;
    const int need_b = (cap + M) * 4 * rows;
    int ht_bytes = HT_WORDS * 4;           // one word = four canvas rows of one (column, channel)
    if (ht_bytes + ((frame_bytes + 15) & ~15) < need_b) ht_bytes = need_b - frame_bytes;
    off_scratch = take(ht_bytes);
    off_frame = take(frame_bytes);
    scratch_bytes = o - off_scratch;
    // The V pass reads, for H-tile row n <= 63 (see HT_N), the words kw + 8 ks + (lane & 3) + {0, 4},
    // ks < nks, of that row: kw, the block's first word, is < HT_ROWW (the block's windows lie in
    // the tile), so the last word read is below 63 * HT_ROWW + HT_ROWW + 8 nks.  Words past a
    // block's window (the next H-tile row, the staged frame, this tail) meet zero taps: they
    // must be addressable shared memory, nothing more
    const int v_words = 64 * HT_ROWW + 8 * nks;
    if (o < off_scratch + v_words * 4) o = off_scratch + v_words * 4;
    total = o;
  }
};

__device__ __forceinline__ int round_up_f(float f) {
  return f >= 0.0f ? (int)floorf(__fadd_rn(f, 0.5f)) : -(int)floorf(__fadd_rn(fabsf(f), 0.5f));
}
__device__ __forceinline__ int round_down_f(float f) {
  return f >= 0.0f ? (int)ceilf(__fsub_rn(f, 0.5f)) : -(int)ceilf(__fsub_rn(fabsf(f), 0.5f));
}
__device__ __forceinline__ float edge_x_at(int y, int y0, float dx, int x0) {
  return __fadd_rn(__fmul_rn((float)(y - y0), dx), (float)x0);
}
__device__ __forceinline__ uint32_t clip8_q22(int v) {  // Pillow clip8: (v >> 22) clamped to 0..255
  uint32_t r;
  asm("cvt.sat.u8.s32 %0, %1;" : "=r"(r) : "r"(v >> 22));
  return r;
}
__device__ __forceinline__ uint32_t lds_u8(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts_u32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.u32 [%0], %1;" : : "r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ int lds_s32(uint32_t addr) {
  int v;
  // volatile: must not be scheduled across the barriers that publish the tables it reads
  asm volatile("ld.shared.s32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}

// merges [xs, xe] into a small unsorted list of disjoint, non-adjacent spans
__device__ __forceinline__ void add_span(int *lxs, int *lxe, int &n, int xs, int xe, bool &ovf) {
  for (int i = 0; i < n;) {
    if (xs <= lxe[i] + 1 && lxs[i] <= xe + 1) {
      xs = min(xs, lxs[i]);
      xe = max(xe, lxe[i]);
      lxs[i] = lxs[n - 1];
      lxe[i] = lxe[n - 1];
      --n;
      i = 0;
    } else {
      ++i;
    }
  }
  if (n < MAX_ROW_SPANS) {
    lxs[n] = xs;
    lxe[n] = xe;
    ++n;
  } else {
    ovf = true;
  }
}

// c_inv20[d] = 2^20 / d + 1: x / d == (x * c_inv20[d]) >> 20 for 0 <= x < 2^20 / d (d <= 64)
__constant__ uint32_t c_inv20[65] = {
    0u, 1048577u, 524289u, 349526u, 262145u, 209716u, 174763u, 149797u,
    131073u, 116509u, 104858u, 95326u, 87382u, 80660u, 74899u, 69906u,
    65537u, 61681u, 58255u, 55189u, 52429u, 49933u, 47663u, 45591u,
    43691u, 41944u, 40330u, 38837u, 37450u, 36158u, 34953u, 33826u,
    32769u, 31776u, 30841u, 29960u, 29128u, 28340u, 27595u, 26887u,
    26215u, 25576u, 24967u, 24386u, 23832u, 23302u, 22796u, 22311u,
    21846u, 21400u, 20972u, 20561u, 20165u, 19785u, 19419u, 19066u,
    18725u, 18397u, 18079u, 17773u, 17477u, 17190u, 16913u, 16645u,
    16385u};
__device__ __forceinline__ int div20(int x, int d) { return (int)(((uint32_t)x * c_inv20[d]) >> 20); }

// Debug-only phase timers (nvcc -DSWB_PHASE_CLOCKS): thread 0 of every CTA adds the cycles
// between consecutive marks to g_phase_clk[id].  Not part of the shipped library.
#ifdef SWB_PHASE_CLOCKS
__device__ unsigned long long g_phase_clk[16];
#define SWB_MARK(id)                                                              \
  do {                                                                            \
    if (tid == 0) {                                                               \
      const long long now_ = clock64();                                           \
      atomicAdd(&g_phase_clk[id], (unsigned long long)(now_ - mark_));            \
      mark_ = now_;                                                               \
    }                                                                             \
  } while (0)
#else
#define SWB_MARK(id) do { } while (0)
#endif

__device__ __forceinline__ int4 lds_v4(uint32_t addr) {
  int4 v;
  asm volatile("ld.shared.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts_u8(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.u8 [%0], %1;" : : "r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
  uint32_t r;
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(sel));
  return r;
}
// Pillow clip8 of a 22-bit fixed-point sum; the result register holds 0..255 (no re-masking)
__device__ __forceinline__ uint32_t sat_u8_q22(int v) {
  return (uint32_t)__vimin_s32_relu(v >> 22, 255);  // max(min(v >> 22, 255), 0), one instruction
}
__device__ __forceinline__ uint32_t lds_u32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
// D(16x8, s32) += A(16x32, u8, row) * B(32x8, s8, col): the integer tensor pipe (SASS IMMA)
__device__ __forceinline__ void mma_u8s8(int (&d)[4], const uint32_t (&a)[4], const uint2 b) {
  asm volatile(
      "mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
      "{%0,%1,%2,%3};"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b.x), "r"(b.y));
}

// The kernel's dynamic shared memory, at namespace scope so that its shared-window address
// can be taken by name (mov.u32 r, symbol: a link-time constant; converting a generic pointer
// costs extra instructions and is rematerialised at every use)
extern __shared__ __align__(16) unsigned char g_render_smem[];
__device__ __forceinline__ uint32_t render_smem_base() {
  uint32_t a;
  asm("mov.u32 %0, _ZN3swb13g_render_smemE;" : "=r"(a));
  return a;
}
__constant__ uint32_t c_prmt_insert[4] = {0x3214u, 0x3240u, 0x3410u, 0x4210u};  // byte i <- byte 0 of b

// Persistent: CTAs claim (env, band) items with atomicAdd(work_counter) - work_base until
// none is left (the host advances work_base by n_items + gridDim.x per launch, so the
// counter never needs a reset).
// kPeers: also store the frame into the other ranks' buffers.
// kWide: the raster's tables go beyond those of anti_aliasing <= 5 (render_wide): the tile plan
// takes rd.tile_blocks, the H pass the prefix stride rd.prefix_stride and the V pass up to
// V_KS_WIDE k-steps.  The narrow instantiation has TILE_BLOCKS, kNarrowPrefixStride and
// V_KS_NARROW compiled in: the code of the aa <= 5 path does not change with the wide one
// (reading the stride and tile blocks at run time cost it 0.4 % at C2).  Wide rasters' staged
// frames and segment tables leave room for few CTAs per SM anyway, so their register budget is
// set for R_CTAS_PER_SM_WIDE
template <bool kPeers, bool kWide>
__global__ void __launch_bounds__(R_THREADS, kWide ? R_CTAS_PER_SM_WIDE : R_CTAS_PER_SM)
render_kernel(DevState st, RasterDev rd, const RenderLayout L, const RenderTargets targets,
              int env_base, int n_items, unsigned *work_counter, unsigned work_base) {
  unsigned char *const smem = g_render_smem;
  const int tid = threadIdx.x;
  const int S = st.S;

  // per-sprite plan (ints): vertex count, last polygon row, first row / row count in this
  // band, horizontal-edge count, bucket shift of the active-edge masks, colour - background,
  // tile plan of the region, "has a corner join"
  int *s_nv = reinterpret_cast<int *>(smem + L.off_meta);
  int *s_pymax = s_nv + S, *s_r0 = s_pymax + S, *s_rcnt = s_r0 + S, *s_nh = s_rcnt + S;
  int *s_bsh = s_nh + S;
  int *s_pny = s_bsh + S, *s_pnx = s_pny + S;
  int *s_hasov = s_pnx + S;
  unsigned *s_emask = reinterpret_cast<unsigned *>(s_hasov + S);  // [S][8] active edges per row bucket
  int4 *s_dcol = reinterpret_cast<int4 *>(smem);  // [SWB_MAX_SLOTS] at offset 0: its address is a constant
  // edge table: start vertex, slope, corner-join overrides on the first / last row
  int *e_x0 = reinterpret_cast<int *>(smem + L.off_edge_i);
  int *e_y0 = e_x0 + S * EV;
  float *e_dx = reinterpret_cast<float *>(smem + L.off_edge_f);
  float *e_ovs = e_dx + S * EV, *e_ove = e_ovs + S * EV;
  uint32_t *e_yr = reinterpret_cast<uint32_t *>(smem + L.off_edge_yr);
  short *s_hl = reinterpret_cast<short *>(smem + L.off_hl);  // [S][EV][3]
  short *s_region = reinterpret_cast<short *>(smem + L.off_region);  // [S][4] yo0,yo1,xo0,xo1
  uint8_t *s_nseg = smem + L.off_nseg;
  uint32_t *s_segs = reinterpret_cast<uint32_t *>(smem + L.off_segs);  // xs | (xe+1)<<12 | sprite<<25
  const int SEGCAP = L.segcap;
  const int M = rd.max_spans;
  int32_t *s_prefix = reinterpret_cast<int32_t *>(smem + L.off_prefix);
  uint32_t *s_xwin = reinterpret_cast<uint32_t *>(smem + L.off_xwin);
  uint32_t *s_ywin = reinterpret_cast<uint32_t *>(smem + L.off_ywin);
  uint8_t *s_frame = smem + L.off_frame;
  // phase-B view of the scratch area: per-row crossing lists
  const int CAP = L.cap;
  __shared__ int4 s_tile[2][2];  // tile descriptors, one tile ahead (phase C)
  __shared__ int s_it[4];        // the walking warp's state (sprite, row tile, column tile)
  __shared__ int s_overflow;
  __shared__ int s_item;
  __shared__ uint8_t *s_dst[SWB_MAX_PEERS];  // kPeers: the targets, indexable at run time

  constexpr unsigned FULL = 0xFFFFFFFFu;
  constexpr int NWARP = R_THREADS / 32;
  const int lane = tid & 31, warp = tid >> 5;

  // ---- once per CTA: the axis tables ------------------------------------------------------
  if (kPeers && tid < SWB_MAX_PEERS) s_dst[tid] = targets.dst[tid];
#pragma unroll 1
  for (int i = tid; i < rd.ncls_x * (kWide ? rd.prefix_stride : kNarrowPrefixStride); i += R_THREADS)
    s_prefix[i] = rd.ax.prefix[i];
#pragma unroll 1
  for (int i = tid; i < rd.W; i += R_THREADS)
    s_xwin[i] = (uint32_t)(uint16_t)rd.ax.win_min[i] | ((uint32_t)rd.ax.win_len[i] << 16) |
                ((uint32_t)rd.ax.win_cls[i] << 24);
#pragma unroll 1
  for (int i = tid; i < (((L.rows + 3) & ~3) + 8) / 4; i += R_THREADS) reinterpret_cast<uint32_t *>(s_nseg)[i] = 0u;
  int band_loaded = -1;
  bool copy_pending = false;  // thread 0: the previous frame's bulk copy may still read s_frame

  // Launched behind this step's step_kernel as a programmatic dependent launch (swb_api.cu), the
  // CTA got here while that grid may still be running: wait until it has completed and its
  // positions / cursors are visible.  Returns at once for an ordinary launch.
  asm volatile("griddepcontrol.wait;" ::: "memory");
#ifdef SWB_PHASE_CLOCKS
  long long mark_ = clock64();
#endif
  for (;;) {
  if (tid == 0) s_item = (int)(atomicAdd(work_counter, 1u) - work_base);
  __syncthreads();
  const int item = s_item;
  if (item >= n_items) break;
  const int band = rd.n_bands > 1 ? item % rd.n_bands : 0;
  const int e = env_base + (rd.n_bands > 1 ? item / rd.n_bands : item);  // frames is indexed by the absolute env id

  const int yo_b0 = band * rd.band_rows;
  const int yo_b1 = min(yo_b0 + rd.band_rows, rd.H);
  const int n_yo = yo_b1 - yo_b0;
  // canvas rows this band's vertical windows can touch, from a row that is a multiple of four
  // (the H tile packs four consecutive canvas rows into a word)
  const int row_b0 = rd.ay.win_min[yo_b0] & ~3;
  const int row_b1 = rd.ay.win_min[yo_b1 - 1] + rd.ay.win_len[yo_b1 - 1];  // exclusive
  const int n_rows = row_b1 - row_b0;

  // ---- phase A: a warp per sprite, a lane per vertex / edge ------------------------------
  // Everything Pillow derives from the vertex list before it scans rows: integer vertices,
  // the edge table (add_edge), horizontal edges, extents, the corner joins -- plus this
  // kernel's own per-sprite plan (rows, output region, tiles, active-edge masks).  Neighbour
  // vertices come by shuffle, extents by warp reductions, "edges that share a start row" by
  // match_any; nothing leaves the warp until the barrier that ends the phase.
  if (tid == 0) s_overflow = 0;
  const int cur = st.cursor[e];
  // per-frame tables first: their loads overlap the sprite records' dependent loads below
#pragma unroll 1
  for (int i = tid; i < (n_rows + 3) / 4; i += R_THREADS) reinterpret_cast<uint32_t *>(s_nseg)[i] = 0u;
  if (band != band_loaded) {
#pragma unroll 1
    for (int i = tid; i < n_yo; i += R_THREADS)
      s_ywin[i] = (uint32_t)(uint16_t)rd.ay.win_min[yo_b0 + i] | ((uint32_t)rd.ay.win_len[yo_b0 + i] << 16) |
                  ((uint32_t)rd.ay.win_cls[yo_b0 + i] << 24);
    band_loaded = band;
  }
  for (int s = warp; s < S; s += NWARP) {
    // sprite record of this env's current scene (warp-uniform loads)
    const int scene = (e * st.K + cur) * S + s;
    const int shape = st.p_shape[scene];
    const uint32_t col = st.p_rgb[scene];
    const double px = st.pos_x[e * S + s], py = st.pos_y[e * S + s];
    const double m00 = st.p_m00[scene], m01 = st.p_m01[scene];
    const double m10 = st.p_m10[scene], m11 = st.p_m11[scene];
    const int nv = shape ? st.shape_n[shape] : 0;
    const int t = s * EV + lane;
    // integer canvas vertex of this lane
    int ivx = 0, ivy = 0;
    if (lane < nv) {
      const double2 v = reinterpret_cast<const double2 *>(st.shape_verts)[(size_t)shape * EV + lane];
      // centred path (sprite.py:96-101): (a*x + c*y) + 0 ; world (sprite.py:128-133): + pos
      const double cx = __dadd_rn(__dadd_rn(__dmul_rn(m00, v.x), __dmul_rn(m01, v.y)), 0.0);
      const double cy = __dadd_rn(__dadd_rn(__dmul_rn(m10, v.x), __dmul_rn(m11, v.y)), 0.0);
      const double wx = __dadd_rn(cx, px), wy = __dadd_rn(cy, py);
      // canvas_size * vertices (pil_renderer.py:81), then Pillow's (int) cast
      ivx = __double2int_rz(__dmul_rn((double)rd.CW, wx));
      ivy = __double2int_rz(__dmul_rn((double)rd.CH, wy));
    }
    // edge lane -> lane+1 (Pillow add_edge); the closing edge exists only if the last vertex
    // differs from the first
    const int jn = (lane + 1 >= nv) ? 0 : lane + 1;
    const int x0 = ivx, y0 = ivy;
    const int x1 = __shfl_sync(FULL, ivx, jn), y1 = __shfl_sync(FULL, ivy, jn);
    const bool exists = lane < nv && ((lane + 1 < nv) || (x0 != x1 || y0 != y1));
    const bool scanned = exists && y0 != y1;
    const int ymin = min(y0, y1), ymax = max(y0, y1);
    const float dx = scanned ? __fdiv_rn((float)(x1 - x0), (float)(y1 - y0)) : 0.0f;
    // horizontal edges are drawn directly as hline(xmin, y, xmax)
    const int hxs = max(min(x0, x1), 0), hxe = min(max(x0, x1), rd.CW - 1);
    const bool hline = exists && y0 == y1 && y0 >= 0 && y0 < rd.CH && hxs <= hxe;
    const unsigned hmask = __ballot_sync(FULL, hline);
    if (hline) {
      short *h = s_hl + ((size_t)s * EV + __popc(hmask & ((1u << lane) - 1u))) * 3;
      h[0] = (short)y0; h[1] = (short)hxs; h[2] = (short)hxe;
    }
    // rows the edge crosses, clamped to int16 (canvas rows are < 4096); empty if not scanned
    const uint32_t yr = scanned ? ((uint32_t)(uint16_t)(short)max(ymin, -32768) |
                                   ((uint32_t)(uint16_t)(short)min(ymax, 32767) << 16))
                                : 0x80007FFFu;
    e_x0[t] = x0;
    e_y0[t] = y0;
    e_dx[t] = dx;
    e_yr[t] = yr;
    e_ovs[t] = nanf("");
    e_ove[t] = nanf("");
    // extents over the vertices
    const bool isv = lane < nv;
    const int xmn = __reduce_min_sync(FULL, isv ? ivx : INT_MAX), xmx = __reduce_max_sync(FULL, isv ? ivx : INT_MIN);
    const int ymn = __reduce_min_sync(FULL, isv ? ivy : INT_MAX), ymx = __reduce_max_sync(FULL, isv ? ivy : INT_MIN);
    // Pillow: ymin = min(ysize-1, edges), ymax = max(0, edges); then clip to [0, ysize]
    const int pymin = max(min(rd.CH - 1, ymn), 0), p_ymax = min(max(0, ymx), rd.CH);
    const int r0 = max(pymin, row_b0), r1 = min(min(p_ymax, rd.CH - 1), row_b1 - 1);
    const int rcnt = (nv > 0 && r1 >= r0) ? (r1 - r0 + 1) : 0;
    // active-edge masks of eight equal row buckets: B1 only looks at the edges of its bucket
    const int bsh = rcnt > 8 ? (32 - __clz(rcnt - 1) - 3) : 0;
    unsigned my_bucket = 0;
#pragma unroll
    for (int b = 0; b < 8; ++b) {
      const int lo = r0 + (b << bsh), hi = lo + (1 << bsh) - 1;
      const unsigned m = __ballot_sync(FULL, scanned && ymin <= hi && ymax >= lo);
      if (lane == b) my_bucket = m;
    }
    if (lane < 8) s_emask[s * 8 + lane] = my_bucket;
    __syncwarp();  // the edge table of this sprite is visible to the join search below

    // corner joins ("connect discontiguous corners"): edge i and the FIRST earlier edge k
    // that leaves the same corner in the same x direction -- both starting on row y, or both
    // ending on the polygon's last row -- move k's crossing on that row towards the adjacent
    // row's span (oracle/sw_raster_oracle.c).  Applied in B1 through e_ovs / e_ove.
    const unsigned lt = (1u << lane) - 1u;
    const unsigned pos = __ballot_sync(FULL, scanned && dx > 0.0f);
    const unsigned neg = __ballot_sync(FULL, scanned && dx < 0.0f);
    const unsigned same_dir = dx > 0.0f ? pos : (dx < 0.0f ? neg : 0u);
    const unsigned start_grp = __match_any_sync(FULL, scanned ? (int)(short)(yr & 0xFFFFu) : (0x40000000 | lane));
    const unsigned end_grp = __ballot_sync(FULL, scanned && (int)(short)(yr >> 16) == p_ymax);
    bool any_join = false;
#pragma unroll
    for (int pass = 0; pass < 2; ++pass) {
      const int y = pass == 0 ? ymin : p_ymax;
      unsigned cand = (pass == 0 ? start_grp : end_grp) & lt & same_dir;
      if (!scanned || (pass == 1 && ymax != p_ymax) || y < 0 || y >= rd.CH) cand = 0;
      int jk = -1;
      float jv = 0.0f;
      if (cand) {
        const float x = edge_x_at(y, y0, dx, x0);
        while (cand) {
          const int k = __ffs(cand) - 1;
          cand &= cand - 1;
          const int u = s * EV + k;
          const float odx = e_dx[u];
          const int oy0 = e_y0[u], ox0 = e_x0[u];
          const float ox = edge_x_at(y, oy0, odx, ox0);
          if (roundf(x) != roundf(ox)) continue;
          const int off = (y == p_ymax) ? -1 : 1;
          const float adj = edge_x_at(y + off, y0, dx, x0);
          const float adjo = edge_x_at(y + off, oy0, odx, ox0);
          const bool right = (y == ymax) ? (dx < 0.0f) : (dx > 0.0f);
          float nvx = right ? __fsub_rn(fminf(adj, adjo), 1.0f) : __fadd_rn(fmaxf(adj, adjo), 1.0f);
          nvx = floorf(__fadd_rn(nvx, 0.5f));
          jv = right ? fmaxf(nvx, x) : fminf(nvx, x);
          jk = k;
          break;
        }
      }
      // several later edges may pick the same k: the last one in table order wins
      const unsigned grp = __match_any_sync(FULL, jk >= 0 ? jk : (64 + lane));
      if (jk >= 0 && (grp >> lane) == 1u) {
        (pass == 0 ? e_ovs : e_ove)[s * EV + jk] = jv;
      }
      any_join |= __any_sync(FULL, jk >= 0);
    }

    if (lane == 0) {
      s_nv[s] = nv;
      // colour - background per channel
      s_dcol[s] = make_int4((int)(col & 255u) - (int)(rd.bg & 255u),
                            (int)((col >> 8) & 255u) - (int)((rd.bg >> 8) & 255u),
                            (int)((col >> 16) & 255u) - (int)((rd.bg >> 16) & 255u), 0);
      s_nh[s] = __popc(hmask);
      s_hasov[s] = any_join ? 1 : 0;
      s_pymax[s] = p_ymax;
      s_r0[s] = r0;
      s_rcnt[s] = rcnt;
      s_bsh[s] = bsh;
      // output region whose 2-D tap window can see this sprite's bounding box
      short yo0 = 0, yo1 = -1, xo0 = 0, xo1 = -1;
      if (nv > 0 && xmx >= 0 && xmn < rd.CW && ymx >= 0 && ymn < rd.CH) {
        const int cx0 = max(xmn, 0), cx1 = min(xmx, rd.CW - 1);
        const int cy0 = max(ymn, 0), cy1 = min(ymx, rd.CH - 1);
        xo0 = rd.ax.first_out[cx0]; xo1 = rd.ax.last_out[cx1];
        yo0 = max((int)rd.ay.first_out[cy0], yo_b0);
        yo1 = min((int)rd.ay.last_out[cy1], yo_b1 - 1);
      }
      s_region[s * 4 + 0] = yo0; s_region[s * 4 + 1] = yo1;
      s_region[s * 4 + 2] = xo0; s_region[s * 4 + 3] = xo1;
      // tile plan: the blocks of eight output rows the region touches, in equal groups of at
      // most rd.tile_blocks; equal column blocks of at most TILE_X_MAX (columns need no halo)
      int pny = 1, pnx = 1;
      if (yo1 >= yo0 && xo1 >= xo0) {
        const int nb = (yo1 >> 3) - (yo0 >> 3) + 1, rw = xo1 - xo0 + 1;  // nb <= 8: bands have <= 64 rows
        const int tb = kWide ? rd.tile_blocks : TILE_BLOCKS;
        const int nty = div20(nb + tb - 1, tb);
        pny = div20(nb + nty - 1, nty);
        const int ntx = div20(rw + TILE_X_MAX - 1, TILE_X_MAX);  // rw <= 4096
        pnx = ntx <= 64 ? div20(rw + ntx - 1, ntx) : (rw + ntx - 1) / ntx;
      }
      s_pny[s] = pny; s_pnx[s] = pnx;
    }
  }
  // the previous frame's write-out must have read the staged frame before phase B reuses the
  // scratch area it lives in
  if (tid == 0 && copy_pending) {
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
    copy_pending = false;
  }
  __syncthreads();
  SWB_MARK(3);

  // ---- phase B: visible segments per canvas row -----------------------------------------
  // B1 (sprite, row)-parallel: Pillow's scan conversion of one canvas row of one sprite
  //    (crossings of the edges that span the row, with the corner-join overrides; sort;
  //    ROUND_UP/ROUND_DOWN pairing; horizontal edges) -> <= M merged spans.
  // B2 row-parallel: fold the sprites' spans front to back into the row's visible segments.
  // Sprites are taken front to back in chunks whose scratch (crossing lists + spans) fits.
  for (int s_hi = S; s_hi > 0;) {
    int s_lo = s_hi, rows_used = 0;
    if (s_hi == S && S <= 32) {  // common case: every sprite fits in one chunk
      const int rows_all = __reduce_add_sync(FULL, lane < S ? s_rcnt[lane] : 0);
      if (rows_all * CAP * 4 + S * n_rows * M * 4 <= L.scratch_bytes) { s_lo = 0; rows_used = rows_all; }
    }
    while (s_lo > 0) {
      const int rows_next = rows_used + s_rcnt[s_lo - 1];
      const int need = rows_next * CAP * 4 + (s_hi - s_lo + 1) * n_rows * M * 4;
      if (s_lo != s_hi && need > L.scratch_bytes) break;
      rows_used = rows_next;
      --s_lo;
    }
    uint32_t *s_spans = reinterpret_cast<uint32_t *>(smem + L.off_scratch) + rows_used * CAP;
    const bool fits = rows_used * CAP * 4 + (s_hi - s_lo) * n_rows * M * 4 <= L.scratch_bytes;
    if (!fits) { s_overflow = 1; }
    SWB_MARK(4);
    // B1
    for (int t = tid; fits && t < rows_used; t += R_THREADS) {
      int s = s_lo, rem = t;
      while (rem >= s_rcnt[s]) { rem -= s_rcnt[s]; ++s; }
      const int y = s_r0[s] + rem;
      const int base = s * EV, p_ymax = s_pymax[s];
      const bool hasov = s_hasov[s] != 0;
      float *xx = reinterpret_cast<float *>(smem + L.off_scratch) + (size_t)t * CAP;
      int j = 0;
      bool ovf = false;
      // edges whose rows overlap this row's bucket, in table order
      unsigned active = s_emask[s * 8 + (rem >> s_bsh[s])];
      while (active) {
        const int u = base + __ffs(active) - 1;
        active &= active - 1;
        const uint32_t yr = e_yr[u];
        const int ymin = (int)(short)(yr & 0xFFFFu), ymax = (int)(short)(yr >> 16);
        if (y < ymin || y > ymax) continue;
        float x = edge_x_at(y, e_y0[u], e_dx[u], e_x0[u]);
        if (hasov) {  // corner-join overrides (rare: acute same-direction corners only)
          if (y == ymin) { const float o = e_ovs[u]; if (!isnan(o)) x = o; }
          if (y == p_ymax && y == ymax) { const float o = e_ove[u]; if (!isnan(o)) x = o; }
        }
        const int twice = (y == ymax && y < p_ymax) ? 2 : 1;  // edge ending on an interior row
        if (j + twice <= CAP) {
          xx[j] = x;
          if (twice == 2) xx[j + 1] = x;
          j += twice;
        } else {
          ovf = true;
        }
      }
      for (int a = 1; a < j; ++a) {  // insertion sort, ascending
        const float v = xx[a];
        int b = a - 1;
        while (b >= 0 && xx[b] > v) { xx[b + 1] = xx[b]; --b; }
        xx[b + 1] = v;
      }
      uint32_t *dst = s_spans + ((size_t)(s - s_lo) * n_rows + (y - row_b0)) * M;
      const int nh = s_nh[s];
      if (M == 1) {
        // convex shapes: every span of the row merges into one [lo, hi] (kept in registers)
        int lo = 1, hi = 0;
        auto merge1 = [&](int xs, int xe) {
          if (lo > hi) { lo = xs; hi = xe; }
          else if (xs <= hi + 1 && lo <= xe + 1) { lo = min(lo, xs); hi = max(hi, xe); }
          else ovf = true;  // a second, disjoint span: the engine was sized for convex shapes
        };
        int x_pos = 0;
        for (int i = 1; i < j; i += 2) {
          const int x_end = round_down_f(xx[i]);
          if (x_end < x_pos) continue;
          if (xx[i - 1] > (float)x_pos) {
            x_pos = round_up_f(xx[i - 1]);
            if (x_end < x_pos) continue;
          }
          const int xs = max(x_pos, 0), xe = min(x_end, rd.CW - 1);
          if (xs <= xe) merge1(xs, xe);
          x_pos = x_end + 1;
        }
        for (int h = 0; h < nh; ++h) {
          const short *hl = s_hl + ((size_t)s * EV + h) * 3;
          if (hl[0] == y) merge1(hl[1], hl[2]);
        }
        dst[0] = lo <= hi ? ((uint32_t)lo | ((uint32_t)hi << 16)) : 0x0000FFFFu;
      } else {
        int lxs[MAX_ROW_SPANS], lxe[MAX_ROW_SPANS];
        int n = 0;
        int x_pos = 0;
        for (int i = 1; i < j; i += 2) {
          const int x_end = round_down_f(xx[i]);
          if (x_end < x_pos) continue;
          if (xx[i - 1] > (float)x_pos) {
            x_pos = round_up_f(xx[i - 1]);
            if (x_end < x_pos) continue;
          }
          const int xs = max(x_pos, 0), xe = min(x_end, rd.CW - 1);
          if (xs <= xe) add_span(lxs, lxe, n, xs, xe, ovf);
          x_pos = x_end + 1;
        }
        for (int h = 0; h < nh; ++h) {
          const short *hl = s_hl + ((size_t)s * EV + h) * 3;
          if (hl[0] == y) add_span(lxs, lxe, n, hl[1], hl[2], ovf);
        }
        if (n > M) ovf = true;
        for (int k = 0; k < M; ++k)
          dst[k] = k < n ? ((uint32_t)lxs[k] | ((uint32_t)lxe[k] << 16)) : 0x0000FFFFu;
      }
      if (ovf) s_overflow = 1;
    }
    __syncthreads();
    SWB_MARK(5);
    // B2
    for (int ry = tid; fits && ry < n_rows; ry += R_THREADS) {
      const int y = row_b0 + ry;
      uint32_t *seg = s_segs + (size_t)ry * SEGCAP;
      int nseg = s_nseg[ry];
      bool ovf = false;
      for (int s = s_hi - 1; s >= s_lo; --s) {
        const int rem = y - s_r0[s];
        if (rem < 0 || rem >= s_rcnt[s]) continue;
        const uint32_t *spn = s_spans + ((size_t)(s - s_lo) * n_rows + ry) * M;
        for (int k = 0; k < M; ++k) {
          const uint32_t w = spn[k];
          const int b = (int)(w >> 16);
          int cursor = (int)(w & 0xFFFFu);
          // the span minus what nearer sprites already cover, kept sorted by x
          for (int i = 0; i <= nseg && cursor <= b; ++i) {
            int gap_end = b;
            int next_cursor = b + 1;
            if (i < nseg) {
              const int xs = (int)(seg[i] & 0xFFFu), xe = (int)((seg[i] >> 12) & 0x1FFFu) - 1;
              if (xe < cursor) continue;
              gap_end = min(b, xs - 1);
              next_cursor = xe + 1;
            }
            if (cursor <= gap_end) {
              if (nseg < SEGCAP) {
                for (int m = nseg; m > i; --m) seg[m] = seg[m - 1];
                seg[i] = (uint32_t)cursor | ((uint32_t)(gap_end + 1) << 12) | ((uint32_t)s << 25);
                ++nseg;
                ++i;  // the segment we compared against moved one slot up
              } else {
                ovf = true;
              }
            }
            cursor = max(cursor, next_cursor);
          }
        }
      }
      s_nseg[ry] = (uint8_t)nseg;
      if (ovf) s_overflow = 1;
    }
    __syncthreads();
    SWB_MARK(6);
    s_hi = s_lo;
  }

  {  // background fill of the staged frame (the scratch area is free again)
    const uint32_t r = rd.bg & 255u, g = (rd.bg >> 8) & 255u, b = (rd.bg >> 16) & 255u;
    const int n_bytes = n_yo * rd.W * 3;
    if (r == g && g == b) {
      const uint32_t w = r * 0x01010101u;
      if ((n_bytes & 15) == 0) {
        uint4 *f128 = reinterpret_cast<uint4 *>(s_frame);
#pragma unroll 1
        for (int i = tid; i < (n_bytes >> 4); i += R_THREADS) f128[i] = make_uint4(w, w, w, w);
      } else {
        uint32_t *f32 = reinterpret_cast<uint32_t *>(s_frame);
        for (int i = tid; i < (n_bytes + 3) / 4; i += R_THREADS) f32[i] = w;
      }
    } else {
      for (int i = tid; i < n_yo * rd.W; i += R_THREADS) {
        s_frame[3 * i] = (uint8_t)r; s_frame[3 * i + 1] = (uint8_t)g; s_frame[3 * i + 2] = (uint8_t)b;
      }
    }
  }
  SWB_MARK(7);

  // ---- phase C: per sprite region, in tiles of <= rd.tile_blocks blocks of eight output rows
  // x <= TILE_X_MAX columns.  Blocks are aligned to multiples of eight output rows of the
  // frame, so that a block's tap matrix is one of a few classes (rd.v_blk_cls); outputs of a
  // block outside the region are computed from whatever the H tile holds and not stored.
  const int bg_r = rd.bg & 255u, bg_g = (rd.bg >> 8) & 255u, bg_b = (rd.bg >> 16) & 255u;
  const uint32_t sm0 = render_smem_base();
  const uint32_t ht0 = sm0 + (uint32_t)L.off_scratch, sm_frame = sm0 + (uint32_t)L.off_frame;
  const uint32_t sm_prefix = sm0 + (uint32_t)L.off_prefix, sm_nseg = sm0 + (uint32_t)L.off_nseg;
  const uint32_t sm_segs = sm0 + (uint32_t)L.off_segs;
  // V pass: this thread's row of the H tile (16 (warp & 3) + lane / 4) and its byte offset
  // there (k words lane % 4 ...), fixed for the whole kernel
  const int v_n0 = 16 * (warp & 3) + (lane >> 2);
  const uint32_t v_aoff = (uint32_t)(v_n0 * HT_ROWW + (lane & 3)) * 4u;
  const int row_bytes = rd.W * 3;
  // The tile loop is driven by the last warp alone: it walks (sprite, row tile, column tile) and
  // publishes each tile as a descriptor of eight words one tile ahead (during the previous
  // tile's H pass; the barriers of the loop order it), so the other seven warps do not repeat
  // the walk and the scalar arithmetic behind a tile.
  //   d0 = (tx0, nx (0: no more tiles), tb0 | nblk << 8 | yo_first << 16 | yo_last << 24  [band-relative], tr0)
  //   d1 = (q0 | q1 << 8, x4lo, x4hi, 2^20 / cs + 1)
  // (the iterator's state lives in shared memory: registers are per thread, and only one warp walks)
  if (tid == (NWARP - 1) * 32) { s_it[0] = -1; s_it[1] = 0; s_it[2] = 0; }
  __syncwarp();
  auto next_tile = [&](int slot) {   // one warp only
    int it_s = s_it[0], it_tb0 = s_it[1], it_tx0 = s_it[2];
    int it_ryo0 = 0, it_ryo1 = -1, it_rxo0 = 0, it_rxo1 = -1, it_nb = 1, it_nxb = 1;
    if (it_s >= 0) {
      it_ryo0 = s_region[it_s * 4 + 0]; it_ryo1 = s_region[it_s * 4 + 1];
      it_rxo0 = s_region[it_s * 4 + 2]; it_rxo1 = s_region[it_s * 4 + 3];
      it_nb = s_pny[it_s]; it_nxb = s_pnx[it_s];
    }
    // advance: next column tile, else next row tile, else the next sprite with a region
    it_tx0 += it_nxb;
    if (it_s < 0 || it_tx0 > it_rxo1) {
      it_tb0 += it_nb;
      it_tx0 = it_rxo0;
      if (it_s < 0 || it_tb0 > (it_ryo1 >> 3)) {
        for (++it_s; it_s < S; ++it_s) {
          it_ryo0 = s_region[it_s * 4 + 0]; it_ryo1 = s_region[it_s * 4 + 1];
          it_rxo0 = s_region[it_s * 4 + 2]; it_rxo1 = s_region[it_s * 4 + 3];
          if (it_ryo1 >= it_ryo0 && it_rxo1 >= it_rxo0) break;
        }
        if (it_s >= S) {
          if (lane == 0) s_tile[slot][0] = make_int4(0, 0, 0, 0);
          return;
        }
        it_nb = s_pny[it_s]; it_nxb = s_pnx[it_s];
        it_tb0 = it_ryo0 >> 3;
        it_tx0 = it_rxo0;
      }
    }
    const int tb0 = it_tb0, tb1 = min(tb0 + it_nb - 1, it_ryo1 >> 3);
    const int tx0 = it_tx0, nx = min(it_nxb, it_rxo1 - tx0 + 1);
    // outputs of the region inside this tile, the canvas rows their windows span, and the
    // tile's row origin: the 4-aligned first row of its first block
    const int yo_first = max(it_ryo0, tb0 << 3), yo_last = min(it_ryo1, (tb1 << 3) + 7);
    const int tr0 = (int)(int16_t)(s_ywin[(tb0 << 3) - yo_b0] & 0xFFFFu) & ~3;
    const uint32_t ywl = s_ywin[yo_last - yo_b0];
    const int q0 = ((int)(int16_t)(s_ywin[yo_first - yo_b0] & 0xFFFFu) - tr0) >> 2;
    const int q1 = ((int)(int16_t)(ywl & 0xFFFFu) + (int)((ywl >> 16) & 0xFFu) - 1 - tr0) >> 2;
    // [x4lo, x4hi): the tile's tap windows in bytes of the prefix table (4 * canvas x)
    const uint32_t xwa = s_xwin[tx0], xwb = s_xwin[tx0 + nx - 1];
    const int x4lo = (int)(int16_t)(xwa & 0xFFFFu) << 2;
    const int x4hi = ((int)(int16_t)(xwb & 0xFFFFu) + (int)((xwb >> 16) & 0xFFu)) << 2;
    __syncwarp();  // every lane has read the state lane 0 overwrites
    if (lane == 0) {
      s_it[0] = it_s; s_it[1] = it_tb0; s_it[2] = it_tx0;
      s_tile[slot][0] = make_int4(tx0, nx,
                                  (tb0 - (yo_b0 >> 3)) | ((tb1 - tb0 + 1) << 8) | ((yo_first - yo_b0) << 16) |
                                      ((yo_last - yo_b0) << 24),
                                  tr0);
      s_tile[slot][1] = make_int4(q0 | (q1 << 8), x4lo, x4hi, (int)c_inv20[(nx + H_NC - 1) / H_NC]);
    }
  };
  if (warp == NWARP - 1) next_tile(0);
  // the background (and later the tiles) is written through the generic proxy; the bulk copy of
  // phase D reads the staged frame through the async proxy
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();  // also: the staged frame's background is in place
  for (int tile = 0;; ++tile) {
        const int4 d0 = s_tile[tile & 1][0], d1 = s_tile[tile & 1][1];
        const int nx = d0.y;
        if (nx == 0) break;
        const int tx0 = d0.x, tr0 = d0.w;
        const int tb0 = (yo_b0 >> 3) + (d0.z & 255), tb1 = tb0 + ((d0.z >> 8) & 255) - 1;
        const int yo_first = yo_b0 + ((d0.z >> 16) & 255), yo_last = yo_b0 + ((d0.z >> 24) & 255);
        const int q0 = d1.x & 255, q1 = d1.x >> 8;
        const int x4lo = d1.y, x4hi = d1.z;
        // ---- H pass: a thread owns NC columns (c0, c0 + cs) of a quad of canvas rows and
        // strides over the quads, so the window start/length and tap prefix table are loop
        // invariants and a row's segment records are decoded once for its columns; the four
        // uint8 results of a (column, channel) leave as one word ----
        {
          const int cs = (nx + H_NC - 1) / H_NC;  // column stride = threads per quad
          const uint32_t inv_cs = (uint32_t)d1.w;
          const int qgroup = (int)(((uint32_t)tid * inv_cs) >> 20);  // tid / cs
          const int c0 = tid - qgroup * cs;
          const int qstride = (int)(((uint32_t)R_THREADS * inv_cs) >> 20);  // quads per pass
          // (consecutive thread groups take consecutive quads on purpose: the sprite's own rows then
          // fill whole warps; spreading them over all warps for balance at the barrier was measured
          // 13 % slower -- every warp then runs the segment loop half empty)
          const int qslot = qgroup;
          if (qgroup < qstride) {
            // per column: prefix-table window [plo, phi] (shared byte addresses) and the offset
            // that maps 4*x to the address of P[x - xmin]; clamping the sum to [plo, phi] is
            // the clamp of x to the tap window
            int poff[H_NC], plo[H_NC], phi[H_NC], kk[H_NC];
#pragma unroll
            for (int q = 0; q < H_NC; ++q) {
              const int c = c0 + q * cs;
              const uint32_t xw = s_xwin[tx0 + (c < nx ? c : c0)];
              plo[q] = (int)(sm_prefix + (xw >> 24) * (uint32_t)(kWide ? rd.prefix_stride : kNarrowPrefixStride) * 4u);
              phi[q] = plo[q] + (int)(((xw >> 16) & 0xFFu) << 2);
              poff[q] = plo[q] - ((int)(int16_t)(xw & 0xFFFFu) << 2);
              kk[q] = lds_s32((uint32_t)phi[q]);  // sum of the window's taps
            }
            const bool on1 = c0 + cs < nx;
            // raw shared-window addresses, advanced by one pass of quads per iteration
            const int rel0 = tr0 - row_b0 + ((q0 + qslot) << 2);  // first canvas row of the quad, band-relative
            uint32_t nseg_addr = sm_nseg + (uint32_t)rel0;
            uint32_t seg_quad = sm_segs + (uint32_t)(rel0 * SEGCAP) * 4u;
            uint32_t ht_addr = ht0 + (uint32_t)(3 * c0 * HT_ROWW + q0 + qslot) * 4u;
            const uint32_t seg_row_step = (uint32_t)SEGCAP * 4u;
            const uint32_t seg_step = (uint32_t)(qstride * 4 * SEGCAP) * 4u;
            const uint32_t ht_col = (uint32_t)(3 * cs * HT_ROWW) * 4u;
            const uint32_t bgw_r = (uint32_t)bg_r * 0x01010101u, bgw_g = (uint32_t)bg_g * 0x01010101u,
                           bgw_b = (uint32_t)bg_b * 0x01010101u;
            for (int qq = q0 + qslot; qq <= q1; qq += qstride, nseg_addr += (uint32_t)(qstride << 2),
                     seg_quad += seg_step, ht_addr += (uint32_t)(qstride << 2)) {
              const uint32_t nseg4 = lds_u32(nseg_addr);  // segment counts of the quad's four rows
              uint32_t wr[H_NC], wg[H_NC], wb[H_NC];
#pragma unroll
              for (int q = 0; q < H_NC; ++q) { wr[q] = bgw_r; wg[q] = bgw_g; wb[q] = bgw_b; }
              if (nseg4) {
                uint32_t seg_addr0 = seg_quad;
#pragma unroll 1
                for (int i = 0; i < 4; ++i, seg_addr0 += seg_row_step) {
                  int j = (int)((nseg4 >> (8 * i)) & 255u);
                  if (!j) continue;
                  uint32_t seg_addr = seg_addr0;
                  uint32_t w;
                  // skip the segments left of every tap window of the tile
                  for (;;) {
                    w = lds_u32(seg_addr);
                    if ((int)((w >> 10) & 0x7FFCu) > x4lo) break;
                    seg_addr += 4u;
                    if (--j == 0) break;
                  }
                  if (j == 0 || (int)((w << 2) & 0x3FFCu) >= x4hi) continue;  // the row shows this tile background only
                  int ar[H_NC], ag[H_NC], ab[H_NC];
#pragma unroll
                  for (int q = 0; q < H_NC; ++q) {
                    ar[q] = bg_r * kk[q] + (1 << 21);
                    ag[q] = bg_g * kk[q] + (1 << 21);
                    ab[q] = bg_b * kk[q] + (1 << 21);
                  }
#pragma unroll 1
                  for (;;) {
                    const int xs4 = (int)((w << 2) & 0x3FFCu), xe4 = (int)((w >> 10) & 0x7FFCu);  // 4*xs, 4*(xe+1)
                    const int4 d = lds_v4(sm0 + ((w >> 21) & 0x7F0u));  // colour - background of the segment's sprite
#pragma unroll
                    for (int q = 0; q < H_NC; ++q) {
                      const int a = min(max(xs4 + poff[q], plo[q]), phi[q]);
                      const int b = min(max(xe4 + poff[q], plo[q]), phi[q]);
                      const int wt = lds_s32((uint32_t)b) - lds_s32((uint32_t)a);
                      ar[q] += d.x * wt; ag[q] += d.y * wt; ab[q] += d.z * wt;
                    }
                    if (--j == 0) break;
                    seg_addr += 4u;
                    w = lds_u32(seg_addr);
                    if ((int)((w << 2) & 0x3FFCu) >= x4hi) break;  // right of every tap window: so are the rest
                  }
                  // byte i of the words <- clip8 (Pillow's uint8 intermediate)
                  const uint32_t psel = c_prmt_insert[i];
#pragma unroll
                  for (int q = 0; q < H_NC; ++q) {
                    wr[q] = prmt(wr[q], sat_u8_q22(ar[q]), psel);
                    wg[q] = prmt(wg[q], sat_u8_q22(ag[q]), psel);
                    wb[q] = prmt(wb[q], sat_u8_q22(ab[q]), psel);
                  }
                }
              }
              sts_u32(ht_addr, wr[0]);
              sts_u32(ht_addr + HT_ROWW * 4u, wg[0]);
              sts_u32(ht_addr + 2u * HT_ROWW * 4u, wb[0]);
              if (on1) {
                sts_u32(ht_addr + ht_col, wr[1]);
                sts_u32(ht_addr + ht_col + HT_ROWW * 4u, wg[1]);
                sts_u32(ht_addr + ht_col + 2u * HT_ROWW * 4u, wb[1]);
              }
            }
          }
        }
        // The last warp's quads are the tile's last canvas rows, usually background below the
        // sprite: it is done early and publishes the next tile's descriptor while the warps on the
        // sprite's rows are still in their segment loops (read after two more barriers).
        if (warp == NWARP - 1) next_tile((tile + 1) & 1);
        __syncthreads();
        SWB_MARK(8);
        // ---- V pass on the tensor pipe: a warp takes 16 (column, channel) rows of the H tile x
        // one block of eight output rows: A = H values (16 x 32 canvas rows per k-step, uint8),
        // B = the block's taps as three int8 limbs (fragments prebuilt on the host), three
        // int32 accumulators recombined as d0 + 2^8 d1 + 2^16 d2 (+ 2^21, >> 22, clip8) ----
        {
          // warp w owns row tile mt = w & 3 (16 (column, channel) rows) for the whole kernel and
          // block w >> 2 of the tile; warps 0..3 also take a third block
          const int nks = rd.v_nks;
          const int n3 = 3 * nx;
          const bool pn0 = v_n0 < n3, pn1 = v_n0 + 8 < n3;
          if (16 * (warp & 3) < n3) {  // warp-uniform (mma.sync needs the whole warp); rows past n3 are not stored
#pragma unroll 1
            for (int jb = warp >> 2; jb <= tb1 - tb0; jb += 2) {
              const int yo_blk = (tb0 + jb) << 3;
              // k origin of the block inside the tile, in words of four canvas rows
              const int kw = (((int)(int16_t)(s_ywin[yo_blk - yo_b0] & 0xFFFFu) & ~3) - tr0) >> 2;
              const uint32_t cls = __ldg(rd.v_blk_cls + (yo_blk >> 3));
              const uint2 *cf = rd.v_frag + (cls * (uint32_t)nks * 96u + (uint32_t)lane);
              const uint32_t a_addr = ht0 + v_aoff + (uint32_t)kw * 4u;
              int d0[4] = {1 << 21, 1 << 21, 1 << 21, 1 << 21}, d1[4] = {0, 0, 0, 0}, d2[4] = {0, 0, 0, 0};
#pragma unroll
              for (int ks = 0; ks < (kWide ? V_KS_WIDE : V_KS_NARROW); ++ks) {  // v_nks <= this
                if (ks < nks) {
                  uint32_t a[4];
                  a[0] = lds_u32(a_addr + 32u * ks);
                  a[1] = lds_u32(a_addr + 32u * ks + 8u * HT_ROWW * 4u);
                  a[2] = lds_u32(a_addr + 32u * ks + 16u);
                  a[3] = lds_u32(a_addr + 32u * ks + 8u * HT_ROWW * 4u + 16u);
                  const uint2 b0 = __ldg(cf + (ks * 3 + 0) * 32);
                  const uint2 b1 = __ldg(cf + (ks * 3 + 1) * 32);
                  const uint2 b2 = __ldg(cf + (ks * 3 + 2) * 32);
                  mma_u8s8(d0, a, b0);
                  mma_u8s8(d1, a, b1);
                  mma_u8s8(d2, a, b2);
                }
              }
              // accumulator r: row n = n0 (+8 for r >= 2), output row yo0 + (r & 1).  Staged in
              // destination order: output row yo is row H-1-yo of the frame (np.flipud)
              const int yo0 = yo_blk + 2 * (lane & 3);
              const uint32_t f_addr = sm_frame + (uint32_t)((yo_b1 - 1 - yo0) * row_bytes + 3 * tx0 + v_n0);
              const bool py0 = (unsigned)(yo0 - yo_first) <= (unsigned)(yo_last - yo_first);
              const bool py1 = (unsigned)(yo0 + 1 - yo_first) <= (unsigned)(yo_last - yo_first);
              if (pn0 && py0) sts_u8(f_addr, sat_u8_q22(d0[0] + (d1[0] << 8) + (d2[0] << 16)));
              if (pn0 && py1) sts_u8(f_addr - (uint32_t)row_bytes, sat_u8_q22(d0[1] + (d1[1] << 8) + (d2[1] << 16)));
              if (pn1 && py0) sts_u8(f_addr + 8u, sat_u8_q22(d0[2] + (d1[2] << 8) + (d2[2] << 16)));
              if (pn1 && py1) sts_u8(f_addr - (uint32_t)row_bytes + 8u, sat_u8_q22(d0[3] + (d1[3] << 8) + (d2[3] << 16)));
            }
          }
        }
        // the tiles are written through the generic proxy; the bulk copy of phase D reads them
        // through the async proxy
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
        SWB_MARK(9);
  }

  // ---- phase D: staged frame -> HBM.  The frame is staged in destination order (rows already
  // flipped, np.flipud), so the band is one contiguous block: one thread hands it to the
  // bulk-copy engine (TMA, cp.async.bulk shared -> global), once per target; the engine reads
  // the staged frame while the CTA sets up its next frame (the wait is at the end of phase A).
  // With several targets the same block also goes to the other ranks' buffers over NVLink
  // peer memory: the frame gather of the multi-GPU path is issued by the kernel that produced
  // the frame and costs it one instruction per rank ----------------------------------------
  const int n_bytes = n_yo * row_bytes;
  const size_t band_off = (size_t)(targets.env_offset + e) * rd.H * row_bytes + (size_t)(rd.H - yo_b1) * row_bytes;
  // the bulk copy needs a 16-byte aligned size and destination address in every target; the
  // caller's buffers may start anywhere (a view at an odd offset), so test the address itself
  bool bulk = (n_bytes & 15) == 0;
  for (int i = 0; i < (kPeers ? targets.n : 1); ++i)
    bulk &= (((uintptr_t)(kPeers ? s_dst[i] : targets.dst[0]) + band_off) & 15) == 0;
  if (bulk) {
    if (tid == 0) {
      const uint32_t src = (uint32_t)__cvta_generic_to_shared(s_frame);
      // peers in an order rotated by rank and frame, so that at any moment the ranks' copies are
      // spread over all receivers instead of all hitting rank 0 first, then rank 1, ...
      int t = 0;
      if (kPeers) {  // (self + 1 + item) mod n without a division (n <= 8)
        t = targets.self + 1 + (int)((unsigned)item & 7u);
        while (t >= targets.n) t -= targets.n;
      }
      for (int i = 0; i < (kPeers ? targets.n : 1); ++i) {
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                     : : "l"((kPeers ? s_dst[t] : targets.dst[0]) + band_off), "r"(src), "r"(n_bytes) : "memory");
        if (kPeers && ++t == targets.n) t = 0;
      }
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      copy_pending = true;
    }
  } else {
    for (int i = tid; i < n_bytes; i += R_THREADS) {
      const uint8_t val = s_frame[i];
      targets.dst[0][band_off + i] = val;
      if (kPeers)
        for (int t = 1; t < targets.n; ++t) targets.dst[t][band_off + i] = val;
    }
  }
  // several bands of one env may race here, but they all OR in the same bit
  if (tid == 0 && s_overflow) st.render_status[e] |= (uint8_t)SWB_ENV_SPAN_OVERFLOW;
  SWB_MARK(10);
  }  // item loop
  // the CTA's shared memory must stay until the engine has read it
  if (tid == 0 && copy_pending) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}

}  // namespace swb
