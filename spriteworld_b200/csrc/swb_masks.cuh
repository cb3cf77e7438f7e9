// Mask kernel: which sprite is visible at each pixel (renderers.SpriteMasks, swb_render_masks),
// which sprites cover it (renderers.SpriteCoverage, swb_render_coverage), and how many of its
// anti-aliasing samples each sprite owns (renderers.SoftSpriteMasks, swb_render_soft_masks).
//
// Mask pixel (i, j) of a W x H mask at anti_aliasing aa is the slot + 1 of the top-most sprite
// whose Pillow polygon fill covers canvas pixel (aa j + aa/2, aa (H-1-i) + aa/2) of the aa W x aa H
// canvas PILRenderer draws on, or 0 (what Image.resize(NEAREST) of a label canvas picks, flipped
// like the frames).  Only Pillow's scan conversion is needed, not its LANCZOS filter, and only one
// canvas row per mask row.  The coverage of the same pixel (MASK_COVER) is the int32 whose bit k is
// set where slot k's fill covers that canvas pixel, whether or not a sprite above hides it, so the
// mask is its highest set bit + 1; with it come per-slot counts of the pixels where the slot is the
// top-most covering sprite (visible) and where its bit is set (area).  The soft mask (MASK_SOFT) is
// [S][H][W] uint8: soft[k][i][j] counts the canvas pixels (aa j + u, aa (H-1-i) + v), u, v in
// [0, aa), whose top-most covering sprite is slot k -- all aa^2 samples of the pixel, not only the
// centre one, so aa <= 15 keeps a count in a byte.  The boxes (MASK_BOX) are the coverage's
// per-slot summaries without the coverage: for each slot, the half-open pixel box (x0, y0, x1, y1)
// of the pixels where it is the top-most covering sprite (visible) and of those where its bit is
// set (amodal), with the two counts; (0, 0, 0, 0) for no pixel.
//
// One CTA draws one band of mask rows of one env (or record):
//   A  a warp per sprite, a lane per vertex: the integer canvas vertices, Pillow's edge records,
//      horizontal edges and corner-join overrides -- the arithmetic of render_kernel's phase A
//      (swb_render.cuh), restated here without that kernel's tile and bucket plan.
//   B  a thread per canvas row scan-converts it for every sprite, back to front: the crossings of
//      the edges spanning the row (an edge ending on an interior row counts twice), sorted and
//      paired with ROUND_UP / ROUND_DOWN, plus the horizontal edges on the row.  Label and cover:
//      a thread per mask row takes its one canvas row, and each canvas span [xs, xe] paints
//      slot + 1 (MASK_COVER: ORs 1 << slot) into the mask columns whose sample aa j + aa/2 lies in
//      it, in a row staged in shared memory.  Soft: a thread per canvas row of the band's aa
//      canvas rows per mask row paints slot + 1 over the whole span, into a staged label row of
//      the canvas.  One scan serves all three modes; only the rows and the paint differ.
//   C  label and cover: the staged band goes out with 16-byte stores (single pixels at its ends).
//      MASK_COVER: each warp counts its pixels per slot with ballots, the CTA sums the warps in
//      shared memory and adds its sums to the outputs with one integer atomic per (band, slot).
//      Soft: a thread per mask pixel collects the labels of its aa x aa block as a 32-bit set,
//      counts the samples of each label in it, and writes one byte to each of the S slot planes;
//      consecutive threads take consecutive columns, so each plane's stores coalesce.
//      Box: the staged band (painted as in MASK_COVER) never leaves the CTA.  Each warp takes
//      32 consecutive pixels at a time; per slot present, two ballots give the amodal and visible
//      lanes, whose first and last set lanes give the row extent (pixels are in raster order) and,
//      where the 32 pixels lie on one row, the column extent; else __reduce_max_sync gives it.
//      The warps combine in shared memory, and each (band, slot) sends integer atomicMax /
//      atomicAdd to the outputs, which hold the mins as MK_BOX_KEY - min so that a zeroed output
//      is the identity; box_finish_kernel turns them back.
// A sprite row has at most 2 crossings per edge, 2 * SWB_MAX_VERTS in all, and every one is kept:
// the masks are exact for every shape, and there is no overflow status.
//
// Nothing but the outputs (MASK_COVER: the coverage and its counts; MASK_BOX: the boxes and the
// counts) is written, every byte of them: no env, pool entry, frame or render status changes.
#pragma once
#include <climits>
#include <type_traits>

#include "swb_device.cuh"
#include "swb_render.cuh"
#include "swb_states.cuh"

namespace swb {

constexpr int MK_THREADS = 128;          // threads per CTA = most mask rows per band
constexpr int MK_STAGE_BYTES = 16384;    // staged bytes per band (fewer rows for wide or coverage masks)
constexpr int MK_SOFT_STAGE_BYTES = 32768;  // soft: staged canvas labels per band (at least one mask row's)
constexpr int MK_SOFT_MAX_AA = 15;       // soft: aa^2 samples per pixel fit a uint8 count
constexpr int MK_XCAP = 2 * EV;          // crossings one sprite row can have
constexpr int MK_BOX_KEY = 4096;         // box: a min m is held as MK_BOX_KEY - m >= 2 (m <= 4094)

// What the mask kernel draws: the uint8 mask, the int32 coverage and its counts, the uint8 soft
// mask [S][H][W], or the per-slot boxes and counts of the coverage.
enum MaskMode { MASK_LABEL, MASK_COVER, MASK_SOFT, MASK_BOX };

// A mask raster and the shared-memory layout of one CTA.  MASK_COVER: staged pixels are the 4-byte
// coverage words, and the CTA keeps per-slot counts.  MASK_BOX: the staged band and its rows are
// MASK_COVER's (the staging budget and a thread per mask row), though it is never written out, and
// the CTA keeps the counts and 8 encoded box fields per slot.  MASK_SOFT: the band's aa canvas rows per mask
// row are staged as CW label bytes each, and band_rows * aa <= MK_THREADS (a thread per canvas row);
// one mask row (at most 15 * 4095 bytes) is always staged, whatever MK_SOFT_STAGE_BYTES says.
struct MaskLayout {
  int S, W, H, aa, CW, CH, band_rows, n_bands;
  int off_edge, off_hl, off_meta, off_xx, off_stage, total;
  __host__ __device__ MaskLayout(int S_, int W_, int H_, int aa_, MaskMode mode = MASK_LABEL)
      : S(S_), W(W_), H(H_), aa(aa_) {
    const bool cover = mode == MASK_COVER, soft = mode == MASK_SOFT, box = mode == MASK_BOX;
    const int px = cover || box ? 4 : 1;  // bytes per staged pixel
    CW = aa * W;
    CH = aa * H;
    if (soft) {
      // the fewest bands of at most the budget's rows, then rows spread evenly over them
      int most = MK_SOFT_STAGE_BYTES / (aa * CW);
      if (most > MK_THREADS / aa) most = MK_THREADS / aa;
      if (most < 1) most = 1;
      n_bands = (H + most - 1) / most;
      band_rows = (H + n_bands - 1) / n_bands;
    } else {
      band_rows = MK_STAGE_BYTES / (px * W);
      if (band_rows < 1) band_rows = 1;
      if (band_rows > MK_THREADS) band_rows = MK_THREADS;
      if (band_rows > H) band_rows = H;
      n_bands = (H + band_rows - 1) / band_rows;
    }
    int o = 0;
    auto take = [&](int bytes) { int r = o; o += (bytes + 15) & ~15; return r; };
    off_edge = take(S * EV * 6 * 4);        // x0, y0 (int), dx, ovs, ove (float), yr (u32)
    off_hl = take(S * EV * 3 * 2);          // horizontal edges: y, xmin, xmax (int16)
    off_meta = take(S * 5 * 4);             // nv, nh, has-join, p_ymax, ymin | ymax << 16
    off_xx = take(MK_XCAP * MK_THREADS * 4);  // crossings, [k][thread]
    if (soft)
      off_stage = take(band_rows * aa * CW);  // canvas labels, [band_rows * aa][CW]
    else
      off_stage = take(band_rows * W * px + 16);  // staged band, placed at the output's address mod 16
    if (cover) take(S * 2 * 4);             // the band's visible [S], area [S] (int), at cnt_offset()
    if (box) take(S * 10 * 4);              // and box: then the encoded boxes [8][S], see mask_kernel
    total = o;
  }
  // cover and box: where the band's counts are, right after the staged band
  __host__ __device__ int cnt_offset() const { return off_stage + ((band_rows * W * 4 + 16 + 15) & ~15); }
};

// The per-slot counts of the coverage, [n][S] int32 each, and (MASK_BOX) its per-slot boxes,
// [n][S][4] int32 each, encoded as box_finish_kernel reads them; all zeroed before the launch.
struct CoverCounts {
  int32_t *visible, *area;
  int32_t *visible_box, *amodal_box;
};

// MASK_LABEL: `masks` is the [n][H][W] uint8 mask.  MASK_COVER: `masks` is the [n][H][W] int32
// coverage, and `counts` receives its per-slot counts.  MASK_SOFT: `masks` is the [n][S][H][W]
// uint8 soft mask.  MASK_BOX: `masks` is unused, and `counts` receives the counts and the encoded
// boxes.  `counts` is read in MASK_COVER and MASK_BOX only.
template <bool kRecords, MaskMode kMode>
__global__ void __launch_bounds__(MK_THREADS)
mask_kernel(DevState st, const MaskLayout L, uint8_t *__restrict__ masks, const RenderRecords recs,
            const CoverCounts counts) {
  constexpr bool kCover = kMode == MASK_COVER, kSoft = kMode == MASK_SOFT, kBox = kMode == MASK_BOX;
  constexpr bool kBits = kCover || kBox;  // staged pixels are coverage words
  extern __shared__ __align__(16) unsigned char g_mask_smem[];
  unsigned char *const smem = g_mask_smem;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr unsigned FULL = 0xFFFFFFFFu;
  constexpr int NWARP = MK_THREADS / 32;
  const int S = L.S;
  const size_t item = blockIdx.x;
  const size_t e = item / (unsigned)L.n_bands;
  const int band = (int)(item - e * (unsigned)L.n_bands);

  int *e_x0 = reinterpret_cast<int *>(smem + L.off_edge);
  int *e_y0 = e_x0 + S * EV;
  float *e_dx = reinterpret_cast<float *>(e_y0 + S * EV);
  float *e_ovs = e_dx + S * EV, *e_ove = e_ovs + S * EV;
  uint32_t *e_yr = reinterpret_cast<uint32_t *>(e_ove + S * EV);
  short *s_hl = reinterpret_cast<short *>(smem + L.off_hl);  // [S][EV][3]
  int *s_nv = reinterpret_cast<int *>(smem + L.off_meta);
  int *s_nh = s_nv + S, *s_hasov = s_nh + S, *s_pymax = s_hasov + S;
  uint32_t *s_yext = reinterpret_cast<uint32_t *>(s_pymax + S);
  float *xx = reinterpret_cast<float *>(smem + L.off_xx) + tid;  // crossing k at xx[k * MK_THREADS]
  using Px = std::conditional_t<kBits, uint32_t, uint8_t>;       // a staged pixel

  // ---- phase A: a warp per sprite, a lane per vertex / edge (render_kernel phase A) ----------
  const int cur = kRecords ? 0 : st.cursor[e];
  const unsigned char *const rec = kRecords ? recs.rec + e * recs.record_bytes : nullptr;
  for (int s = warp; s < S; s += NWARP) {
    const size_t scene = (e * st.K + cur) * S + s;
    const SlotRecord r = kRecords ? read_record(st, rec, s) : SlotRecord{};
    const int shape = kRecords ? r.shape : st.p_shape[scene];
    const double px = kRecords ? r.f64[POS_X] : st.pos_x[e * S + s];
    const double py = kRecords ? r.f64[POS_Y] : st.pos_y[e * S + s];
    const double m00 = kRecords ? r.f64[M00] : st.p_m00[scene];
    const double m01 = kRecords ? r.f64[M01] : st.p_m01[scene];
    const double m10 = kRecords ? r.f64[M10] : st.p_m10[scene];
    const double m11 = kRecords ? r.f64[M11] : st.p_m11[scene];
    const int nv = shape ? st.shape_n[shape] : 0;
    const int t = s * EV + lane;
    int ivx = 0, ivy = 0;
    if (lane < nv) {
      const double2 v = reinterpret_cast<const double2 *>(st.shape_verts)[(size_t)shape * EV + lane];
      // centred path (sprite.py:96-101), world position, canvas_size * vertices, Pillow's (int)
      const double cx = __dadd_rn(__dadd_rn(__dmul_rn(m00, v.x), __dmul_rn(m01, v.y)), 0.0);
      const double cy = __dadd_rn(__dadd_rn(__dmul_rn(m10, v.x), __dmul_rn(m11, v.y)), 0.0);
      const double wx = __dadd_rn(cx, px), wy = __dadd_rn(cy, py);
      ivx = __double2int_rz(__dmul_rn((double)L.CW, wx));
      ivy = __double2int_rz(__dmul_rn((double)L.CH, wy));
    }
    // edge lane -> lane+1 (Pillow add_edge); the closing edge only if the polygon is not closed
    const int jn = (lane + 1 >= nv) ? 0 : lane + 1;
    const int x0 = ivx, y0 = ivy;
    const int x1 = __shfl_sync(FULL, ivx, jn), y1 = __shfl_sync(FULL, ivy, jn);
    const bool exists = lane < nv && ((lane + 1 < nv) || (x0 != x1 || y0 != y1));
    const bool scanned = exists && y0 != y1;
    const int ymin = min(y0, y1), ymax = max(y0, y1);
    const float dx = scanned ? __fdiv_rn((float)(x1 - x0), (float)(y1 - y0)) : 0.0f;
    // horizontal edges are drawn directly as hline(xmin, y, xmax), clipped to the canvas
    const int hxs = max(min(x0, x1), 0), hxe = min(max(x0, x1), L.CW - 1);
    const bool hline = exists && y0 == y1 && y0 >= 0 && y0 < L.CH && hxs <= hxe;
    const unsigned hmask = __ballot_sync(FULL, hline);
    if (hline) {
      short *h = s_hl + ((size_t)s * EV + __popc(hmask & ((1u << lane) - 1u))) * 3;
      h[0] = (short)y0; h[1] = (short)hxs; h[2] = (short)hxe;
    }
    // rows the edge crosses, both ends clamped to [-1, CH]: canvas rows are 0 .. CH-1, so the
    // clamped range holds exactly the canvas rows the true one does, and a clamped end equals a
    // canvas row only where the true end does (the tests of phase B and the join search below).
    // Empty (no row) if not scanned
    const uint32_t yr = scanned ? ((uint32_t)(uint16_t)(short)min(max(ymin, -1), L.CH) |
                                   ((uint32_t)(uint16_t)(short)min(max(ymax, -1), L.CH) << 16))
                                : 0x80007FFFu;
    e_x0[t] = x0;
    e_y0[t] = y0;
    e_dx[t] = dx;
    e_yr[t] = yr;
    e_ovs[t] = nanf("");
    e_ove[t] = nanf("");
    const bool isv = lane < nv;
    const int ymn = __reduce_min_sync(FULL, isv ? ivy : INT_MAX), ymx = __reduce_max_sync(FULL, isv ? ivy : INT_MIN);
    // Pillow's last polygon row: max(0, edges), clipped to ysize
    const int p_ymax = min(max(0, ymx), L.CH);
    __syncwarp();  // the edge table of this sprite is visible to the join search below

    // corner joins: edge i and the FIRST earlier edge k leaving the same corner in the same x
    // direction -- both starting on row y, or both ending on the polygon's last row -- move k's
    // crossing on that row (oracle/sw_raster_oracle.c, render_kernel phase A)
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
      if (!scanned || (pass == 1 && ymax != p_ymax) || y < 0 || y >= L.CH) cand = 0;
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
      if (jk >= 0 && (grp >> lane) == 1u) (pass == 0 ? e_ovs : e_ove)[s * EV + jk] = jv;
      any_join |= __any_sync(FULL, jk >= 0);
    }
    if (lane == 0) {
      s_nv[s] = nv;
      s_nh[s] = __popc(hmask);
      s_hasov[s] = any_join ? 1 : 0;
      s_pymax[s] = p_ymax;
      // the canvas rows any edge or horizontal edge of the sprite is on, clamped to [-1, 32767]
      // (canvas rows are 0 .. 4094); none without vertices
      s_yext[s] = nv > 0 ? ((uint32_t)(uint16_t)(short)min(max(ymn, -1), 32767) |
                            ((uint32_t)(uint16_t)(short)min(max(ymx, -1), 32767) << 16))
                         : 0x8000FFFFu;
    }
  }


  // the band's output rows [i0, i0 + nb) are pixels [g, g + nb * W) of the masks; the band is
  // staged from s_stage + (its address mod 16), so that staged and global addresses agree modulo 16.
  // kSoft: the stage holds the band's canvas rows aa (H-1-i) + v, v in [0, aa), of mask rows i in
  // [i0, i0 + nb) as label rows stage[((i - i0) aa + v) CW + x] (0: no sprite), from s_stage
  const int i0 = band * L.band_rows;
  const int nb = min(L.band_rows, L.H - i0);
  const size_t g = (e * (size_t)L.H + (size_t)i0) * (size_t)L.W;
  const int npx = nb * L.W;
  Px *const gdst = reinterpret_cast<Px *>(masks) + g;
  const int mis = kSoft || kBox ? 0 : (int)(reinterpret_cast<uintptr_t>(gdst) & 15u);
  Px *const stage = reinterpret_cast<Px *>(smem + L.off_stage + mis);
  // kCover: visible [S], area [S]; kBox: then the boxes [8][S]
  int *const s_cnt = reinterpret_cast<int *>(smem + L.cnt_offset());
  const int nstage = kSoft ? nb * L.aa * L.CW : npx;  // staged pixels
  if constexpr (kSoft)
    for (int i = tid; i < (nstage >> 4); i += MK_THREADS) reinterpret_cast<uint4 *>(stage)[i] = make_uint4(0, 0, 0, 0);
  for (int i = (kSoft ? nstage & ~15 : 0) + tid; i < nstage; i += MK_THREADS) stage[i] = 0;
  if (kCover && tid < 2 * S) s_cnt[tid] = 0;
  if constexpr (kBox)
    for (int i = tid; i < 10 * S; i += MK_THREADS) s_cnt[i] = 0;
  __syncthreads();

  // ---- phase B: a thread per mask row, its one canvas row, sprites back to front (kSoft: a
  // thread per canvas row of the band, nb * aa <= MK_THREADS by MaskLayout) ---------------------
  if (tid < (kSoft ? nb * L.aa : nb)) {
    const int i = i0 + (kSoft ? tid / L.aa : tid);
    // canvas row of mask row i (always on the canvas): its sample row, kSoft its row tid mod aa
    const int y = L.aa * (L.H - 1 - i) + (kSoft ? tid - (i - i0) * L.aa : L.aa / 2);
    const int half = L.aa / 2;
    Px *const row = stage + (size_t)tid * (kSoft ? L.CW : L.W);
    // paints the mask columns j with xs <= aa j + aa/2 <= xe (0 <= xs <= xe < CW); kSoft: the
    // canvas pixels xs .. xe
    auto paint = [&](int xs, int xe, Px label) {
      if constexpr (kSoft) {
#pragma unroll 1
        for (int x = xs; x <= xe; ++x) row[x] = label;
      } else {
        const int jlo = (xs - half + L.aa - 1) / L.aa, jhi = (xe - half + L.aa) / L.aa - 1;
        for (int j = jlo; j <= jhi; ++j) {
          if constexpr (kBits) row[j] |= label;
          else row[j] = label;
        }
      }
    };
#pragma unroll 1
    for (int s = 0; s < S; ++s) {
      const uint32_t ext = s_yext[s];
      if (y < (int)(short)(ext & 0xFFFFu) || y > (int)(short)(ext >> 16)) continue;
      const Px label = kBits ? (Px)(1u << s) : (Px)(s + 1);
      const int nv = s_nv[s], p_ymax = s_pymax[s];
      const bool hasov = s_hasov[s] != 0;
      int j = 0;
#pragma unroll 1
      for (int k = 0; k < nv; ++k) {
        const int u = s * EV + k;
        const uint32_t yr = e_yr[u];
        const int ymin = (int)(short)(yr & 0xFFFFu), ymax = (int)(short)(yr >> 16);
        if (y < ymin || y > ymax) continue;
        float x = edge_x_at(y, e_y0[u], e_dx[u], e_x0[u]);
        if (hasov) {
          if (y == ymin) { const float o = e_ovs[u]; if (!isnan(o)) x = o; }
          if (y == p_ymax && y == ymax) { const float o = e_ove[u]; if (!isnan(o)) x = o; }
        }
        xx[j++ * MK_THREADS] = x;
        if (y == ymax && y < p_ymax) xx[j++ * MK_THREADS] = x;  // edge ending on an interior row
      }
#pragma unroll 1
      for (int a = 1; a < j; ++a) {  // insertion sort, ascending
        const float v = xx[a * MK_THREADS];
        int b = a - 1;
        while (b >= 0 && xx[b * MK_THREADS] > v) { xx[(b + 1) * MK_THREADS] = xx[b * MK_THREADS]; --b; }
        xx[(b + 1) * MK_THREADS] = v;
      }
      int x_pos = 0;
#pragma unroll 1
      for (int a = 1; a < j; a += 2) {
        const int x_end = round_down_f(xx[a * MK_THREADS]);
        if (x_end < x_pos) continue;
        const float xa = xx[(a - 1) * MK_THREADS];
        if (xa > (float)x_pos) {
          x_pos = round_up_f(xa);
          if (x_end < x_pos) continue;
        }
        const int xs = max(x_pos, 0), xe = min(x_end, L.CW - 1);
        if (xs <= xe) paint(xs, xe, label);
        x_pos = x_end + 1;
      }
      const int nh = s_nh[s];
#pragma unroll 1
      for (int h = 0; h < nh; ++h) {
        const short *hl = s_hl + ((size_t)s * EV + h) * 3;
        if (hl[0] == y) paint(hl[1], hl[2], label);
      }
    }
  }
  __syncthreads();

  if constexpr (kSoft) {
    // ---- soft phase C: a thread per mask pixel (i0 + r, j), its aa x aa block of labels ------
    const int aa = L.aa, CW = L.CW, aa2 = aa * aa;
    const size_t plane = (size_t)L.H * L.W;
    for (int p = tid; p < npx; p += MK_THREADS) {
      const int r = p / L.W, j = p - r * L.W;
      const uint8_t *const blk = stage + (size_t)r * aa * CW + aa * j;
      uint32_t present = 0;  // bit s: label s + 1 is in the block
      bool bg = false;       // a sample no sprite covers
#pragma unroll 1
      for (int v = 0; v < aa; ++v)
#pragma unroll 1
        for (int u = 0; u < aa; ++u) {
          const int l = blk[v * CW + u];
          if (l) present |= 1u << (l - 1);
          else bg = true;
        }
      const bool one = !bg && (present & (present - 1u)) == 0u;  // one label on every sample
      uint8_t *dst = masks + (e * (size_t)S * L.H + (size_t)(i0 + r)) * L.W + j;
#pragma unroll 1
      for (int s = 0; s < S; ++s, dst += plane) {
        int c = 0;
        if ((present >> s) & 1u) {
          if (one) {
            c = aa2;
          } else {
#pragma unroll 1
            for (int v = 0; v < aa; ++v)
#pragma unroll 1
              for (int u = 0; u < aa; ++u) c += blk[v * CW + u] == s + 1;
          }
        }
        *dst = (uint8_t)c;
      }
    }
    return;
  }

  if constexpr (kBox) {
    // ---- box phase C: lane s keeps slot s's counts and encoded boxes over its warp's pixels --
    // box fields: K - x0, K - y0, x1, y1 (K = MK_BOX_KEY), all 0 while the slot has no pixel
    constexpr int K = MK_BOX_KEY;
    int vis = 0, area = 0, vb[4] = {0, 0, 0, 0}, ab[4] = {0, 0, 0, 0};
    for (int p0 = warp * 32; p0 < npx; p0 += MK_THREADS) {
      const int p = p0 + lane;
      const uint32_t c = p < npx ? stage[p] : 0u;
      const int top = c ? 31 - __clz(c) : -1;  // the top-most covering slot
      const int r0 = p0 / L.W, c0 = p0 - r0 * L.W, j = p % L.W;
      // warp-uniform: all 32 pixels are on band row r0, from column c0, so the first and last set
      // lanes of a ballot give its columns; else (W < 32, or pixels on two rows) reductions do
      const bool one_row = c0 + 32 <= L.W;
      for (unsigned any = __reduce_or_sync(FULL, c); any; any &= any - 1u) {
        const int s = __ffs(any) - 1;
        const bool in_a = (c >> s) & 1u, in_v = top == s;
        const unsigned am = __ballot_sync(FULL, in_a), vm = __ballot_sync(FULL, in_v);
        int ax0, ax1, vx0 = 0, vx1 = 0;  // K - x0 and x1 of the amodal and visible lanes
        if (one_row) {
          ax0 = K - (c0 + __ffs(am) - 1);
          ax1 = c0 + 32 - __clz(am);
          if (vm) {
            vx0 = K - (c0 + __ffs(vm) - 1);
            vx1 = c0 + 32 - __clz(vm);
          }
        } else {
          ax0 = __reduce_max_sync(FULL, in_a ? K - j : 0);
          ax1 = __reduce_max_sync(FULL, in_a ? j + 1 : 0);
          if (vm) {
            vx0 = __reduce_max_sync(FULL, in_v ? K - j : 0);
            vx1 = __reduce_max_sync(FULL, in_v ? j + 1 : 0);
          }
        }
        if (lane == s) {
          // raster order: the first and last set lanes hold the top and bottom rows
          area += __popc(am);
          ab[0] = max(ab[0], ax0);
          ab[1] = max(ab[1], K - (i0 + (one_row ? r0 : (p0 + __ffs(am) - 1) / L.W)));
          ab[2] = max(ab[2], ax1);
          ab[3] = max(ab[3], i0 + (one_row ? r0 : (p0 + 31 - __clz(am)) / L.W) + 1);
          if (vm) {
            vis += __popc(vm);
            vb[0] = max(vb[0], vx0);
            vb[1] = max(vb[1], K - (i0 + (one_row ? r0 : (p0 + __ffs(vm) - 1) / L.W)));
            vb[2] = max(vb[2], vx1);
            vb[3] = max(vb[3], i0 + (one_row ? r0 : (p0 + 31 - __clz(vm)) / L.W) + 1);
          }
        }
      }
    }
    if (area) {  // vis <= area, and only slots < S have bits
      atomicAdd(&s_cnt[lane], vis);
      atomicAdd(&s_cnt[S + lane], area);
#pragma unroll
      for (int f = 0; f < 4; ++f) {
        atomicMax(&s_cnt[(2 + f) * S + lane], vb[f]);
        atomicMax(&s_cnt[(6 + f) * S + lane], ab[f]);
      }
    }
    __syncthreads();
    // s_cnt[q * S + s]: q = 0 visible, 1 area, 2..5 the visible box, 6..9 the amodal box
    for (int i = tid; i < 10 * S; i += MK_THREADS) {
      const int v = s_cnt[i], q = i / S, s = i - q * S;
      if (!v) continue;
      const size_t o = e * S + s;
      if (q == 0) atomicAdd(&counts.visible[o], v);
      else if (q == 1) atomicAdd(&counts.area[o], v);
      else if (q < 6) atomicMax(&counts.visible_box[o * 4 + (q - 2)], v);
      else atomicMax(&counts.amodal_box[o * 4 + (q - 6)], v);
    }
    return;
  }

  // ---- phase C: the staged band to the masks -------------------------------------------------
  constexpr int LOG16 = kCover ? 2 : 4;  // log2 of the pixels per 16-byte store
  const int head = min(((16 - mis) & 15) / (int)sizeof(Px), npx);
  const int n16 = (npx - head) >> LOG16;
  const int tail0 = head + (n16 << LOG16);
  for (int i = tid; i < head; i += MK_THREADS) gdst[i] = stage[i];
  const uint4 *src16 = reinterpret_cast<const uint4 *>(stage + head);
  uint4 *dst16 = reinterpret_cast<uint4 *>(gdst + head);
  for (int i = tid; i < n16; i += MK_THREADS) dst16[i] = src16[i];
  for (int i = tail0 + tid; i < npx; i += MK_THREADS) gdst[i] = stage[i];

  if constexpr (kCover) {
    // lane s counts slot s over its warp's pixels: a ballot per slot that any of 32 pixels has
    int vis = 0, area = 0;
    for (int p0 = warp * 32; p0 < npx; p0 += MK_THREADS) {
      const uint32_t c = p0 + lane < npx ? stage[p0 + lane] : 0u;
      const int top = c ? 31 - __clz(c) : -1;  // the top-most covering slot
      for (unsigned any = __reduce_or_sync(FULL, c); any; any &= any - 1u) {
        const int s = __ffs(any) - 1;
        const int a = __popc(__ballot_sync(FULL, (c >> s) & 1u));
        const int v = __popc(__ballot_sync(FULL, top == s));
        if (lane == s) { area += a; vis += v; }
      }
    }
    if (area) {  // vis <= area, and only slots < S have bits
      atomicAdd(&s_cnt[lane], vis);
      atomicAdd(&s_cnt[S + lane], area);
    }
    __syncthreads();
    if (tid < S) {
      const int v = s_cnt[tid], a = s_cnt[S + tid];
      if (v) atomicAdd(&counts.visible[e * S + tid], v);
      if (a) atomicAdd(&counts.area[e * S + tid], a);
    }
  }
}

constexpr int BOX_FINISH_THREADS = 256;

// MASK_BOX, after mask_kernel: box i < n_boxes of visible_box, then box i - n_boxes of amodal_box
// ([n][S][4] int32 each, n_boxes = n S), from MK_BOX_KEY - x0, MK_BOX_KEY - y0 back to x0, y0.  A
// box no pixel reached is all 0 and stays so; any other has both fields >= 2.
__global__ void __launch_bounds__(BOX_FINISH_THREADS)
box_finish_kernel(int32_t *__restrict__ visible_box, int32_t *__restrict__ amodal_box, size_t n_boxes) {
  const size_t i = (size_t)blockIdx.x * BOX_FINISH_THREADS + threadIdx.x;
  if (i >= 2 * n_boxes) return;
  int32_t *const b = i < n_boxes ? visible_box + 4 * i : amodal_box + 4 * (i - n_boxes);
  if (b[0]) {
    b[0] = MK_BOX_KEY - b[0];
    b[1] = MK_BOX_KEY - b[1];
  }
}

}  // namespace swb
