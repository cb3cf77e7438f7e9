// C-ABI of the engine (include/spriteworld_b200.h): engine/raster lifetime, scene upload,
// kernel launches.  No torch types; plain CUDA runtime.
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "swb_device.cuh"
#include "swb_render.cuh"
#include "swb_step.cuh"
#include "swb_tables.h"

using namespace swb;

namespace {

thread_local std::string g_error;

int fail(const char *fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_error = buf;
  return 1;
}

#define CUDA_TRY(expr)                                                              \
  do {                                                                              \
    cudaError_t _e = (expr);                                                        \
    if (_e != cudaSuccess)                                                          \
      return fail("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

template <typename T>
cudaError_t dev_alloc(T **p, size_t n) {
  cudaError_t e = cudaMalloc(reinterpret_cast<void **>(p), (n ? n : 1) * sizeof(T));
  if (e == cudaSuccess) e = cudaMemset(*p, 0, (n ? n : 1) * sizeof(T));
  return e;
}

}  // namespace

// One staging slot of swb_upload_scenes: a pinned host block and its device twin, laid out
// [8 x f64][member u32][rgb u32][factors 5 x f32][dst i32][shape u8][pos_f32 u8] for `cap`
// scenes, moved with ONE cudaMemcpyAsync and scattered into the pool by one kernel.
struct UploadSlot {
  size_t cap = 0;          // scenes
  size_t bytes = 0;
  unsigned char *host = nullptr, *dev = nullptr;
  cudaEvent_t done = nullptr;  // recorded after the scatter kernel that reads `dev`
  bool in_flight = false;
};

struct swb_engine {
  swb_config cfg;
  StepCfg step_cfg;
  StepCfg *d_step_cfg = nullptr;  // device copy the step kernel reads (per engine)
  unsigned *d_work = nullptr;     // render kernel's work counter (monotonic, see render_kernel)
  unsigned work_base = 0;         // its value when the next launch starts
  int n_sms = 1;
  DevState st;
  int device = 0;
  int max_spans = 1;  // 1 while every uploaded shape is convex, else 4
  int64_t launches = 0;
  // staging for scene uploads (pinned host + device), grown on demand, double-buffered
  UploadSlot upload_slots[2];
  int upload_next = 0;
  std::vector<void *> owned;
  // buffers of swb_step_host
  void *h_actions = nullptr;
  swb_step_out h_out = {nullptr, nullptr, nullptr, nullptr};
  uint8_t *h_frames = nullptr;
  size_t h_frames_bytes = 0;
  cudaStream_t copy_stream = nullptr;  // D2H of frame chunks overlaps the render of the next chunk
  cudaEvent_t chunk_done[8] = {};
  cudaEvent_t copies_done = nullptr;
};

struct swb_raster {
  swb_engine *eng;
  RasterDev rd;
  AxisHost ax, ay;
  int smem_rows = 0;
  std::vector<void *> owned;
};

namespace {

__global__ void scatter_scenes_kernel(DevState st, int n, const int32_t *__restrict__ dst,
                                      const double *__restrict__ f64, size_t f64_stride,
                                      const uint32_t *__restrict__ member,
                                      const uint8_t *__restrict__ shape,
                                      const uint8_t *__restrict__ pos_f32,
                                      const uint32_t *__restrict__ rgb,
                                      const float *__restrict__ factors) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * st.S) return;
  const int sc = i / st.S, s = i - sc * st.S;
  const size_t d = (size_t)dst[sc] * st.S + s;
  st.p_x[d] = f64[0 * f64_stride + i];
  st.p_y[d] = f64[1 * f64_stride + i];
  st.p_m00[d] = f64[2 * f64_stride + i];
  st.p_m01[d] = f64[3 * f64_stride + i];
  st.p_m10[d] = f64[4 * f64_stride + i];
  st.p_m11[d] = f64[5 * f64_stride + i];
  st.p_vx[d] = f64[6 * f64_stride + i];
  st.p_vy[d] = f64[7 * f64_stride + i];
  st.p_member[d] = member[i];
  st.p_shape[d] = shape[i];
  st.p_pos_f32[d] = pos_f32[i];
  st.p_rgb[d] = rgb[i];
  for (int f = 0; f < 5; ++f) st.p_factors[d * 5 + f] = factors[(size_t)i * 5 + f];
}

template <typename T>
int upload_vec(swb_raster *r, const std::vector<T> &v, const T **out) {
  T *p = nullptr;
  CUDA_TRY(cudaMalloc(reinterpret_cast<void **>(&p), std::max<size_t>(v.size(), 1) * sizeof(T)));
  r->owned.push_back(p);
  CUDA_TRY(cudaMemcpy(p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
  *out = p;
  return 0;
}

int upload_axis(swb_raster *r, const AxisHost &h, AxisTables *d) {
  if (upload_vec(r, h.win_min, &d->win_min)) return 1;
  if (upload_vec(r, h.win_len, &d->win_len)) return 1;
  if (upload_vec(r, h.win_cls, &d->win_cls)) return 1;
  if (upload_vec(r, h.prefix, &d->prefix)) return 1;
  if (upload_vec(r, h.first_out, &d->first_out)) return 1;
  if (upload_vec(r, h.last_out, &d->last_out)) return 1;
  return 0;
}

}  // namespace

extern "C" {

const char *swb_last_error(void) { return g_error.c_str(); }
int swb_version(void) { return 1; }
int swb_sizeof_config(void) { return (int)sizeof(swb_config); }
int swb_sizeof_task_node(void) { return (int)sizeof(swb_task_node); }

int swb_engine_create(const swb_config *cfg, swb_engine **out) {
  if (!cfg || !out) return fail("swb_engine_create: null argument");
  if (cfg->n_envs < 1) return fail("n_envs must be >= 1");
  if (cfg->n_slots < 1 || cfg->n_slots > SWB_MAX_SLOTS)
    return fail("n_slots must be in [1, %d], got %d", SWB_MAX_SLOTS, cfg->n_slots);
  if (cfg->pool_depth < 1) return fail("pool_depth must be >= 1");
  if (cfg->n_nodes < 1 || cfg->n_nodes > SWB_MAX_NODES) return fail("bad n_nodes %d", cfg->n_nodes);
  for (int i = 0; i < cfg->n_nodes; ++i) {
    const swb_task_node &nd = cfg->nodes[i];
    if (nd.kind == SWB_TASK_META) {
      if (nd.n_children < 0 || nd.n_children > SWB_MAX_CHILDREN) return fail("bad n_children");
      for (int c = 0; c < nd.n_children; ++c)
        if (nd.children[c] < 0 || nd.children[c] >= i) return fail("task tree is not post-order");
    } else if (nd.kind == SWB_TASK_CLUSTERING) {
      if (nd.n_clusters < 1 || nd.n_clusters > SWB_MAX_CHILDREN) return fail("bad n_clusters");
    } else if (nd.kind == SWB_TASK_FIND_GOAL) {
      if (nd.filter_slot >= SWB_MAX_FILTERS) return fail("bad filter_slot");
    } else if (nd.kind != SWB_TASK_NO_REWARD) {
      return fail("unknown task kind %d", nd.kind);
    }
  }
  if (cfg->action_kind < 0 || cfg->action_kind > SWB_ACT_EMBODIED) return fail("bad action_kind");
  int n_dev = 0;
  CUDA_TRY(cudaGetDeviceCount(&n_dev));
  if (cfg->device < 0 || cfg->device >= n_dev) return fail("no CUDA device %d", cfg->device);
  CUDA_TRY(cudaSetDevice(cfg->device));

  swb_engine *eng = new swb_engine();
  eng->cfg = *cfg;
  eng->device = cfg->device;
  if (cudaDeviceGetAttribute(&eng->n_sms, cudaDevAttrMultiProcessorCount, cfg->device) != cudaSuccess ||
      eng->n_sms < 1)
    eng->n_sms = 132;
  StepCfg &sc = eng->step_cfg;
  memset(&sc, 0, sizeof sc);
  sc.action_kind = cfg->action_kind;
  sc.action_scale = cfg->action_scale;
  sc.motion_cost = cfg->motion_cost;
  sc.keep_in_frame = cfg->keep_in_frame;
  sc.max_episode_length = cfg->max_episode_length;
  sc.n_nodes = cfg->n_nodes;
  memcpy(sc.nodes, cfg->nodes, sizeof(swb_task_node) * cfg->n_nodes);

  DevState &st = eng->st;
  memset(&st, 0, sizeof st);
  st.E = cfg->n_envs;
  st.S = cfg->n_slots;
  st.K = cfg->pool_depth;
  const size_t ES = (size_t)st.E * st.S, EKS = ES * st.K;
  bool ok = true;
  auto A = [&](auto **p, size_t n) {
    if (ok && dev_alloc(p, n) != cudaSuccess) ok = false;
    if (ok) eng->owned.push_back(*p);
  };
  A(&st.pos_x, ES); A(&st.pos_y, ES);
  A(&st.cursor, st.E); A(&st.step_count, st.E);
  A(&st.reset_next, st.E + 4); A(&st.render_status, st.E + 4);
  A(&st.p_x, EKS); A(&st.p_y, EKS);
  A(&st.p_m00, EKS); A(&st.p_m01, EKS); A(&st.p_m10, EKS); A(&st.p_m11, EKS);
  A(&st.p_vx, EKS); A(&st.p_vy, EKS);
  A(&st.p_member, EKS); A(&st.p_shape, EKS); A(&st.p_pos_f32, EKS); A(&st.p_rgb, EKS);
  A(&st.p_factors, EKS * 5);
  double *d_verts = nullptr;
  int32_t *d_nv = nullptr;
  A(&eng->d_step_cfg, 1);
  A(&eng->d_work, 1);
  A(&st.scene_serial, st.E);
  A(&d_verts, (size_t)SWB_NUM_SHAPES * SWB_MAX_VERTS * 2);
  A(&d_nv, SWB_NUM_SHAPES);
  if (!ok) {
    swb_engine_destroy(eng);
    return fail("device allocation failed: %s", cudaGetErrorString(cudaGetLastError()));
  }
  for (int s = 1; s < SWB_NUM_SHAPES; ++s)
    if (cfg->shape_n_verts[s] < 0 || cfg->shape_n_verts[s] > SWB_MAX_VERTS) {
      swb_engine_destroy(eng);
      return fail("shape %d has %d vertices (max %d)", s, cfg->shape_n_verts[s], SWB_MAX_VERTS);
    }
  CUDA_TRY(cudaMemcpy(eng->d_step_cfg, &eng->step_cfg, sizeof(StepCfg), cudaMemcpyHostToDevice));
  CUDA_TRY(cudaMemcpy(d_verts, cfg->shape_verts, sizeof cfg->shape_verts, cudaMemcpyHostToDevice));
  CUDA_TRY(cudaMemcpy(d_nv, cfg->shape_n_verts, sizeof cfg->shape_n_verts, cudaMemcpyHostToDevice));
  st.shape_verts = d_verts;
  st.shape_n = d_nv;
  // every env starts "about to reset" (environment.py:70)
  CUDA_TRY(cudaMemset(st.reset_next, 1, st.E));
  *out = eng;
  return 0;
}

void swb_engine_destroy(swb_engine *eng) {
  if (!eng) return;
  cudaSetDevice(eng->device);
  for (void *p : eng->owned) cudaFree(p);
  for (auto &slot : eng->upload_slots) {
    if (slot.in_flight) cudaEventSynchronize(slot.done);
    if (slot.host) cudaFreeHost(slot.host);
    if (slot.dev) cudaFree(slot.dev);
    if (slot.done) cudaEventDestroy(slot.done);
  }
  cudaFree(eng->h_actions); cudaFree(eng->h_out.reward); cudaFree(eng->h_out.step_type);
  cudaFree(eng->h_out.success); cudaFree(eng->h_out.status); cudaFree(eng->h_frames);
  if (eng->copy_stream) cudaStreamDestroy(eng->copy_stream);
  for (auto &ev : eng->chunk_done) if (ev) cudaEventDestroy(ev);
  if (eng->copies_done) cudaEventDestroy(eng->copies_done);
  delete eng;
}

static size_t upload_layout(size_t cap, int S, size_t off[7]) {
  const size_t capS = cap * S;
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o += (bytes + 255) & ~(size_t)255; return r; };
  off[0] = take(capS * 8 * sizeof(double));   // f64 x 8
  off[1] = take(capS * sizeof(uint32_t));     // member
  off[2] = take(capS * sizeof(uint32_t));     // rgb
  off[3] = take(capS * 5 * sizeof(float));    // factors
  off[4] = take(cap * sizeof(int32_t));       // dst
  off[5] = take(capS);                        // shape
  off[6] = take(capS);                        // pos_f32
  return o;
}

int swb_upload_scenes(swb_engine *eng, const swb_scene_soa *sc, const int32_t *env_ids,
                      const int32_t *ring_slots, int32_t n, void *stream_) {
  if (!eng || !sc || !env_ids || !ring_slots) return fail("swb_upload_scenes: null argument");
  if (n <= 0) return 0;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  CUDA_TRY(cudaSetDevice(eng->device));
  const int S = eng->st.S;
  const size_t nS = (size_t)n * S;
  const double *f64_src[8] = {sc->x, sc->y, sc->m00, sc->m01, sc->m10, sc->m11, sc->vx, sc->vy};
  for (int a = 0; a < 8; ++a)
    if (!f64_src[a]) return fail("swb_upload_scenes: null f64 array %d", a);
  if (!sc->member || !sc->shape || !sc->pos_f32 || !sc->rgb) return fail("swb_upload_scenes: null array");
  for (int i = 0; i < n; ++i) {
    if (env_ids[i] < 0 || env_ids[i] >= eng->st.E) return fail("env id %d out of range", env_ids[i]);
    if (ring_slots[i] < 0 || ring_slots[i] >= eng->st.K) return fail("ring slot %d out of range", ring_slots[i]);
  }
  for (size_t i = 0; i < nS; ++i) {
    const int sh = sc->shape[i];
    if (sh >= SWB_NUM_SHAPES) return fail("shape id %d out of range", sh);
    if (sh > 6) eng->max_spans = 4;  // stars / spokes: several spans per canvas row
    if (sh && eng->cfg.shape_n_verts[sh] < 3) return fail("shape %d has no vertex table", sh);
  }
  // two staging slots alternate, so the host packs upload i+1 while upload i is in flight; a
  // slot is reused only after the scatter kernel that read it has finished (its event)
  UploadSlot &slot = eng->upload_slots[eng->upload_next];
  eng->upload_next ^= 1;
  if (slot.in_flight) {
    CUDA_TRY(cudaEventSynchronize(slot.done));
    slot.in_flight = false;
  }
  if ((size_t)n > slot.cap) {
    if (slot.host) cudaFreeHost(slot.host);
    if (slot.dev) cudaFree(slot.dev);
    slot.host = slot.dev = nullptr;
    slot.cap = 0;
    size_t off[7];
    const size_t cap = std::max<size_t>((size_t)n, 256);
    const size_t bytes = upload_layout(cap, S, off);
    CUDA_TRY(cudaMallocHost(reinterpret_cast<void **>(&slot.host), bytes));
    CUDA_TRY(cudaMalloc(reinterpret_cast<void **>(&slot.dev), bytes));
    if (!slot.done) CUDA_TRY(cudaEventCreateWithFlags(&slot.done, cudaEventDisableTiming));
    slot.cap = cap;
    slot.bytes = bytes;
  }
  size_t off[7];
  upload_layout(slot.cap, S, off);
  const size_t stride = slot.cap * S;
  unsigned char *h = slot.host;
  for (int a = 0; a < 8; ++a)
    memcpy(h + off[0] + a * stride * sizeof(double), f64_src[a], nS * sizeof(double));
  memcpy(h + off[1], sc->member, nS * sizeof(uint32_t));
  uint32_t *rgb = reinterpret_cast<uint32_t *>(h + off[2]);
  for (size_t i = 0; i < nS; ++i)
    rgb[i] = (uint32_t)sc->rgb[3 * i] | ((uint32_t)sc->rgb[3 * i + 1] << 8) | ((uint32_t)sc->rgb[3 * i + 2] << 16);
  if (sc->factors) memcpy(h + off[3], sc->factors, nS * 5 * sizeof(float));
  else memset(h + off[3], 0, nS * 5 * sizeof(float));
  int32_t *dst = reinterpret_cast<int32_t *>(h + off[4]);
  for (int i = 0; i < n; ++i) dst[i] = env_ids[i] * eng->st.K + ring_slots[i];
  memcpy(h + off[5], sc->shape, nS);
  memcpy(h + off[6], sc->pos_f32, nS);
  // everything up to the end of the last used array, in one copy
  CUDA_TRY(cudaMemcpyAsync(slot.dev, slot.host, off[6] + nS, cudaMemcpyHostToDevice, stream));
  const int threads = 256, blocks = (int)((nS + threads - 1) / threads);
  unsigned char *d = slot.dev;
  scatter_scenes_kernel<<<blocks, threads, 0, stream>>>(
      eng->st, n, reinterpret_cast<const int32_t *>(d + off[4]), reinterpret_cast<const double *>(d + off[0]),
      stride, reinterpret_cast<const uint32_t *>(d + off[1]), d + off[5], d + off[6],
      reinterpret_cast<const uint32_t *>(d + off[2]), reinterpret_cast<const float *>(d + off[3]));
  eng->launches++;
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaEventRecord(slot.done, stream));
  slot.in_flight = true;
  return 0;
}

int swb_request_reset(swb_engine *eng, const uint8_t *mask, void *stream_) {
  if (!eng) return fail("null engine");
  CUDA_TRY(cudaSetDevice(eng->device));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  request_reset_kernel<<<(eng->st.E + 255) / 256, 256, 0, stream>>>(eng->st, mask);
  eng->launches++;
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int swb_step(swb_engine *eng, const void *actions, int32_t action_dtype, const swb_step_out *out,
             void *stream_) {
  if (!eng || !actions || !out) return fail("swb_step: null argument");
  if (!out->reward || !out->step_type || !out->success || !out->status)
    return fail("swb_step: every swb_step_out pointer must be set");
  const bool emb = eng->cfg.action_kind == SWB_ACT_EMBODIED;
  if (emb && action_dtype != SWB_DTYPE_I32) return fail("Embodied actions must be int32 [E][2]");
  if (!emb && action_dtype != SWB_DTYPE_F32 && action_dtype != SWB_DTYPE_F64)
    return fail("SelectMove/DragAndDrop actions must be float32 or float64 [E][4]");
  CUDA_TRY(cudaSetDevice(eng->device));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int blocks = (eng->st.E + STEP_WARPS - 1) / STEP_WARPS;
  step_kernel<<<blocks, STEP_WARPS * 32, 0, stream>>>(eng->st, eng->d_step_cfg, actions, action_dtype, *out, 0);
  eng->launches++;
  CUDA_TRY(cudaGetLastError());
  return 0;
}

static int launch_partial(swb_engine *eng, const void *actions, int32_t action_dtype,
                          const swb_step_out *out, void *stream_, int mode) {
  if (!eng || !out) return fail("null argument");
  if (!out->reward || !out->step_type || !out->success || !out->status)
    return fail("every swb_step_out pointer must be set");
  CUDA_TRY(cudaSetDevice(eng->device));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int blocks = (eng->st.E + STEP_WARPS - 1) / STEP_WARPS;
  step_kernel<<<blocks, STEP_WARPS * 32, 0, stream>>>(eng->st, eng->d_step_cfg, actions, action_dtype, *out, mode);
  eng->launches++;
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int swb_eval_task(swb_engine *eng, const swb_step_out *out, void *stream) {
  return launch_partial(eng, nullptr, SWB_DTYPE_F32, out, stream, 1);
}

int swb_apply_action(swb_engine *eng, const void *actions, int32_t action_dtype,
                     const swb_step_out *out, void *stream) {
  if (!actions) return fail("swb_apply_action: null actions");
  const bool emb = eng && eng->cfg.action_kind == SWB_ACT_EMBODIED;
  if (emb && action_dtype != SWB_DTYPE_I32) return fail("Embodied actions must be int32 [E][2]");
  if (!emb && action_dtype != SWB_DTYPE_F32 && action_dtype != SWB_DTYPE_F64)
    return fail("SelectMove/DragAndDrop actions must be float32 or float64 [E][4]");
  return launch_partial(eng, actions, action_dtype, out, stream, 2);
}

int swb_raster_create(swb_engine *eng, int32_t width, int32_t height, int32_t aa,
                      const uint8_t bg_rgb[3], swb_raster **out) {
  if (!eng || !out) return fail("swb_raster_create: null argument");
  if (width < 1 || height < 1 || width > 4096 || height > 4096) return fail("bad image size %dx%d", width, height);
  if (aa < 1) return fail("anti_aliasing must be >= 1");
  if ((int64_t)width * aa > 4095 || (int64_t)height * aa > 4095)
    return fail("canvas %dx%d exceeds 4095 pixels per side", width * aa, height * aa);
  // Image.resize shrinks a canvas more than 100 times taller than wide vertically first
  // (Pillow 12.2.0), which rounds differently from the kernel's horizontal-then-vertical passes
  if (aa > 1 && height > (int64_t)width * 100)
    return fail("image %dx%d is more than 100 times taller than wide; with anti_aliasing > 1 "
                "Pillow resizes such frames vertically first, which the render kernel does not",
                width, height);
  CUDA_TRY(cudaSetDevice(eng->device));
  swb_raster *r = new swb_raster();
  r->eng = eng;
  std::string err;
  if (!build_axis(width * aa, width, &r->ax, &err) || !build_axis(height * aa, height, &r->ay, &err)) {
    delete r;
    return fail("%s", err.c_str());
  }
  RasterDev &rd = r->rd;
  rd.W = width; rd.H = height; rd.aa = aa; rd.CW = width * aa; rd.CH = height * aa;
  rd.bg = bg_rgb ? ((uint32_t)bg_rgb[0] | ((uint32_t)bg_rgb[1] << 8) | ((uint32_t)bg_rgb[2] << 16)) : 0u;
  rd.band_rows = height <= 64 ? height : 64;
  rd.n_bands = (height + rd.band_rows - 1) / rd.band_rows;
  rd.max_spans = 1;
  rd.ncls_x = r->ax.n_cls;
  rd.ncls_y = r->ay.n_cls;
  int rows = 0;
  for (int b = 0; b < rd.n_bands; ++b) {
    const int y0 = b * rd.band_rows, y1 = std::min(y0 + rd.band_rows, height) - 1;
    // the kernel counts a band's canvas rows from a multiple of four
    rows = std::max(rows, r->ay.win_min[y1] + r->ay.win_len[y1] - (r->ay.win_min[y0] & ~3));
    // a tile of TILE_BLOCKS blocks of eight output rows must fit the H tile's row length
    for (int t0 = y0; t0 <= y1; t0 += 8) {
      const int t1 = std::min(t0 + 8 * TILE_BLOCKS - 1, y1);
      const int span = r->ay.win_min[t1] + r->ay.win_len[t1] - (r->ay.win_min[t0] & ~3);
      if (span > 4 * HT_ROWW) {
        delete r;
        return fail("vertical tap windows of %d output rows span %d canvas rows (limit %d)",
                    8 * TILE_BLOCKS, span, 4 * HT_ROWW);
      }
    }
  }
  r->smem_rows = rows;
  VFragHost vf;
  if (!build_vfrag(r->ay, &vf, &err)) {
    delete r;
    return fail("%s", err.c_str());
  }
  rd.v_nks = vf.nks;
  const uint32_t *d_frag = nullptr;
  if (upload_axis(r, r->ax, &rd.ax) || upload_axis(r, r->ay, &rd.ay) ||
      upload_vec(r, vf.blk_cls, &rd.v_blk_cls) || upload_vec(r, vf.frag, &d_frag)) {
    swb_raster_destroy(r);
    return 1;
  }
  rd.v_frag = reinterpret_cast<const uint2 *>(d_frag);  // cudaMalloc: 256-byte aligned
  *out = r;
  return 0;
}

void swb_raster_destroy(swb_raster *r) {
  if (!r) return;
  for (void *p : r->owned) cudaFree(p);
  delete r;
}

// after_step: the launch follows this step's step_kernel on the stream.  It is then made a
// programmatic dependent launch: the render CTAs may become resident and load their tables while
// the step kernel's last CTAs run (step_kernel signals griddepcontrol.launch_dependents at once),
// and wait (griddepcontrol.wait, after their set-up) until the step grid has completed and its
// writes are visible.
static int launch_render_targets(swb_engine *eng, swb_raster *r, const RenderTargets &targets,
                                 uint8_t *status, cudaStream_t stream, int env_base = 0,
                                 int env_count = -1, bool after_step = false) {
  if (r->eng != eng) return fail("raster belongs to another engine");
  RasterDev rd = r->rd;
  rd.max_spans = eng->max_spans;
  int max_smem = 0;
  CUDA_TRY(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, eng->device));
  RenderLayout L(eng->st.S, r->smem_rows, rd.max_spans, rd.band_rows, rd.W, rd.aa, rd.ncls_x, rd.ncls_y);
  // many convex slots on a wide raster: rather than refuse the raster, keep 16 visible segments
  // per canvas row as with concave shapes (a row with more is flagged, see RenderLayout)
  if (L.total > max_smem && L.segcap > 16)
    L = RenderLayout(eng->st.S, r->smem_rows, rd.max_spans, rd.band_rows, rd.W, rd.aa, rd.ncls_x,
                     rd.ncls_y, false);
  if ((L.cap + rd.max_spans) * 4 * r->smem_rows > L.scratch_bytes)
    return fail("render scratch (%d B) cannot hold one sprite spanning %d canvas rows", L.scratch_bytes,
                r->smem_rows);
  if (L.total > max_smem)
    return fail("render needs %d B of shared memory per CTA (limit %d): too many sprite slots / too large a canvas",
                L.total, max_smem);
  auto kernel = targets.n > 1 ? render_kernel<true> : render_kernel<false>;
  CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, L.total));
  DevState st = eng->st;
  st.render_status = status;
  if (env_count < 0) env_count = eng->st.E - env_base;
  if (env_count <= 0) return 0;
  // persistent CTAs: one per resident slot (or per item if there are fewer), claiming
  // (env, band) items from the engine's counter; see render_kernel
  const int n_items = env_count * rd.n_bands;
  const int grid = std::min(n_items, eng->n_sms * R_CTAS_PER_SM);
  cudaLaunchConfig_t lc = {};
  lc.gridDim = dim3(grid);
  lc.blockDim = dim3(R_THREADS);
  lc.dynamicSmemBytes = (size_t)L.total;
  lc.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  lc.attrs = attr;
  lc.numAttrs = after_step ? 1 : 0;
  CUDA_TRY(cudaLaunchKernelEx(&lc, kernel, st, rd, L, targets, env_base, n_items, eng->d_work, eng->work_base));
  eng->work_base += (unsigned)(n_items + grid);  // every CTA's last claim fails
  eng->launches++;
  CUDA_TRY(cudaGetLastError());
  return 0;
}

static int launch_render(swb_engine *eng, swb_raster *r, uint8_t *frames, uint8_t *status,
                         cudaStream_t stream, int env_base = 0, int env_count = -1,
                         bool after_step = false) {
  RenderTargets targets{};
  targets.dst[0] = frames;
  targets.n = 1;
  targets.env_offset = 0;
  targets.self = 0;
  return launch_render_targets(eng, r, targets, status, stream, env_base, env_count, after_step);
}

int swb_render(swb_engine *eng, swb_raster *r, uint8_t *frames, void *stream_) {
  if (!eng || !r || !frames) return fail("swb_render: null argument");
  CUDA_TRY(cudaSetDevice(eng->device));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  CUDA_TRY(cudaMemsetAsync(eng->st.render_status, 0, eng->st.E, stream));
  return launch_render(eng, r, frames, eng->st.render_status, stream);
}

int swb_step_render(swb_engine *eng, swb_raster *r, const void *actions, int32_t action_dtype,
                    const swb_step_out *out, uint8_t *frames, void *stream_) {
  if (!r || !frames) return fail("swb_step_render: null argument");
  if (swb_step(eng, actions, action_dtype, out, stream_)) return 1;
  return launch_render(eng, r, frames, out->status, static_cast<cudaStream_t>(stream_), 0, -1, true);
}

int swb_step_render_gather(swb_engine *eng, swb_raster *r, const void *actions,
                           int32_t action_dtype, const swb_step_out *out, uint8_t *const *dst,
                           int32_t n_dst, int64_t env_offset, void *stream_) {
  if (!r || !dst) return fail("swb_step_render_gather: null argument");
  if (n_dst < 1 || n_dst > SWB_MAX_PEERS)
    return fail("swb_step_render_gather: n_dst = %d, expected 1..%d", n_dst, SWB_MAX_PEERS);
  if (env_offset < 0 || env_offset > INT32_MAX - (eng ? eng->st.E : 0))
    return fail("swb_step_render_gather: env_offset out of range");
  RenderTargets targets{};
  for (int i = 0; i < n_dst; ++i) {
    if (!dst[i]) return fail("swb_step_render_gather: dst[%d] is null", i);
    targets.dst[i] = dst[i];
  }
  targets.n = n_dst;
  targets.env_offset = (int)env_offset;
  targets.self = (int)((env_offset / (eng ? eng->st.E : 1)) % n_dst);
  if (swb_step(eng, actions, action_dtype, out, stream_)) return 1;
  return launch_render_targets(eng, r, targets, out->status, static_cast<cudaStream_t>(stream_), 0, -1, true);
}

int swb_ipc_alloc(int32_t device, uint64_t bytes, void **ptr, uint8_t *handle) {
  if (!ptr || !handle || !bytes) return fail("swb_ipc_alloc: bad argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == SWB_IPC_HANDLE_BYTES, "IPC handle size");
  CUDA_TRY(cudaSetDevice(device));
  void *p = nullptr;
  CUDA_TRY(cudaMalloc(&p, bytes));
  cudaIpcMemHandle_t h;
  cudaError_t err = cudaIpcGetMemHandle(&h, p);
  if (err != cudaSuccess) {
    cudaFree(p);
    return fail("cudaIpcGetMemHandle: %s", cudaGetErrorString(err));
  }
  memcpy(handle, &h, sizeof(h));
  *ptr = p;
  return 0;
}

int swb_ipc_free(void *ptr) {
  if (ptr) CUDA_TRY(cudaFree(ptr));
  return 0;
}

int swb_ipc_open(int32_t device, const uint8_t *handle, void **ptr) {
  if (!ptr || !handle) return fail("swb_ipc_open: null argument");
  CUDA_TRY(cudaSetDevice(device));
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, sizeof(h));
  void *p = nullptr;
  CUDA_TRY(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
  *ptr = p;
  return 0;
}

int swb_peer_copy(void *dst, const void *src, uint64_t bytes, void *stream) {
  if (!dst || !src) return fail("swb_peer_copy: null argument");
  CUDA_TRY(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(stream)));
  return 0;
}

int swb_ipc_close(void *ptr) {
  if (ptr) CUDA_TRY(cudaIpcCloseMemHandle(ptr));
  return 0;
}

int swb_step_host(swb_engine *eng, swb_raster *r, const void *actions, int32_t action_dtype,
                  double *reward, int8_t *step_type, uint8_t *success, uint8_t *status,
                  uint8_t *frames, void *stream_) {
  if (!eng || !actions) return fail("swb_step_host: null argument");
  CUDA_TRY(cudaSetDevice(eng->device));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int E = eng->st.E;
  if (!eng->h_actions) {
    CUDA_TRY(cudaMalloc(&eng->h_actions, (size_t)E * 4 * sizeof(double)));
    CUDA_TRY(cudaMalloc(&eng->h_out.reward, (size_t)E * sizeof(double)));
    CUDA_TRY(cudaMalloc(&eng->h_out.step_type, E + 4));
    CUDA_TRY(cudaMalloc(&eng->h_out.success, E + 4));
    CUDA_TRY(cudaMalloc(&eng->h_out.status, E + 4));
  }
  const size_t abytes = action_dtype == SWB_DTYPE_I32 ? (size_t)E * 2 * 4
                        : (action_dtype == SWB_DTYPE_F32 ? (size_t)E * 16 : (size_t)E * 32);
  CUDA_TRY(cudaMemcpyAsync(eng->h_actions, actions, abytes, cudaMemcpyHostToDevice, stream));
  if (r) {
    const size_t fbytes = (size_t)E * r->rd.H * r->rd.W * 3;
    if (fbytes > eng->h_frames_bytes) {
      CUDA_TRY(cudaStreamSynchronize(stream));
      cudaFree(eng->h_frames);
      eng->h_frames_bytes = 0;
      CUDA_TRY(cudaMalloc(&eng->h_frames, fbytes));
      // written only by the render kernel's bulk copies, which initcheck does not track: zero
      // it once so that the tool sees every byte the D2H copies read as initialised
      CUDA_TRY(cudaMemsetAsync(eng->h_frames, 0, fbytes, stream));
      eng->h_frames_bytes = fbytes;
    }
    if (swb_step(eng, eng->h_actions, action_dtype, &eng->h_out, stream)) return 1;
    if (!frames) {
      if (launch_render(eng, r, eng->h_frames, eng->h_out.status, stream, 0, -1, true)) return 1;
    } else {
      // render in env chunks; each chunk's frames go to the host on a second stream while
      // the next chunk renders
      if (!eng->copy_stream) {
        CUDA_TRY(cudaStreamCreateWithFlags(&eng->copy_stream, cudaStreamNonBlocking));
        for (auto &ev : eng->chunk_done) CUDA_TRY(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
        CUDA_TRY(cudaEventCreateWithFlags(&eng->copies_done, cudaEventDisableTiming));
      }
      const size_t per_env = (size_t)r->rd.H * r->rd.W * 3;
      const int n_chunks = E >= 1024 ? 8 : (E >= 64 ? 2 : 1);
      for (int c = 0; c < n_chunks; ++c) {
        const int e0 = (int)((int64_t)E * c / n_chunks), e1 = (int)((int64_t)E * (c + 1) / n_chunks);
        if (launch_render(eng, r, eng->h_frames, eng->h_out.status, stream, e0, e1 - e0, c == 0)) return 1;
        CUDA_TRY(cudaEventRecord(eng->chunk_done[c], stream));
        CUDA_TRY(cudaStreamWaitEvent(eng->copy_stream, eng->chunk_done[c], 0));
        CUDA_TRY(cudaMemcpyAsync(frames + per_env * e0, eng->h_frames + per_env * e0, per_env * (e1 - e0),
                                 cudaMemcpyDeviceToHost, eng->copy_stream));
      }
      CUDA_TRY(cudaEventRecord(eng->copies_done, eng->copy_stream));
      CUDA_TRY(cudaStreamWaitEvent(stream, eng->copies_done, 0));
    }
  } else {
    if (swb_step(eng, eng->h_actions, action_dtype, &eng->h_out, stream)) return 1;
  }
  if (reward) CUDA_TRY(cudaMemcpyAsync(reward, eng->h_out.reward, (size_t)E * sizeof(double), cudaMemcpyDeviceToHost, stream));
  if (step_type) CUDA_TRY(cudaMemcpyAsync(step_type, eng->h_out.step_type, E, cudaMemcpyDeviceToHost, stream));
  if (success) CUDA_TRY(cudaMemcpyAsync(success, eng->h_out.success, E, cudaMemcpyDeviceToHost, stream));
  if (status) CUDA_TRY(cudaMemcpyAsync(status, eng->h_out.status, E, cudaMemcpyDeviceToHost, stream));
  CUDA_TRY(cudaStreamSynchronize(stream));
  return 0;
}

int swb_state_pointers(swb_engine *eng, double **pos_x, double **pos_y, int32_t **cursor,
                       int32_t **step_count, uint8_t **reset_next) {
  if (!eng) return fail("null engine");
  if (pos_x) *pos_x = eng->st.pos_x;
  if (pos_y) *pos_y = eng->st.pos_y;
  if (cursor) *cursor = eng->st.cursor;
  if (step_count) *step_count = eng->st.step_count;
  if (reset_next) *reset_next = eng->st.reset_next;
  return 0;
}

int swb_render_status_pointer(swb_engine *eng, uint8_t **render_status) {
  if (!eng || !render_status) return fail("swb_render_status_pointer: null argument");
  *render_status = eng->st.render_status;
  return 0;
}

int swb_scene_serial_pointer(swb_engine *eng, int32_t **scene_serial) {
  if (!eng || !scene_serial) return fail("swb_scene_serial_pointer: null argument");
  *scene_serial = eng->st.scene_serial;
  return 0;
}

int swb_download_state(swb_engine *eng, double *pos_x, double *pos_y, int32_t *cursor,
                       int32_t *step_count, uint8_t *reset_next, void *stream_) {
  if (!eng) return fail("null engine");
  CUDA_TRY(cudaSetDevice(eng->device));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const size_t ES = (size_t)eng->st.E * eng->st.S;
  if (pos_x) CUDA_TRY(cudaMemcpyAsync(pos_x, eng->st.pos_x, ES * 8, cudaMemcpyDeviceToHost, stream));
  if (pos_y) CUDA_TRY(cudaMemcpyAsync(pos_y, eng->st.pos_y, ES * 8, cudaMemcpyDeviceToHost, stream));
  if (cursor) CUDA_TRY(cudaMemcpyAsync(cursor, eng->st.cursor, eng->st.E * 4, cudaMemcpyDeviceToHost, stream));
  if (step_count) CUDA_TRY(cudaMemcpyAsync(step_count, eng->st.step_count, eng->st.E * 4, cudaMemcpyDeviceToHost, stream));
  if (reset_next) CUDA_TRY(cudaMemcpyAsync(reset_next, eng->st.reset_next, eng->st.E, cudaMemcpyDeviceToHost, stream));
  CUDA_TRY(cudaStreamSynchronize(stream));
  return 0;
}

int swb_upload_state(swb_engine *eng, const double *pos_x, const double *pos_y, const int32_t *cursor,
                     const int32_t *step_count, const uint8_t *reset_next, void *stream_) {
  if (!eng) return fail("null engine");
  CUDA_TRY(cudaSetDevice(eng->device));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const size_t ES = (size_t)eng->st.E * eng->st.S;
  if (pos_x) CUDA_TRY(cudaMemcpyAsync(eng->st.pos_x, pos_x, ES * 8, cudaMemcpyHostToDevice, stream));
  if (pos_y) CUDA_TRY(cudaMemcpyAsync(eng->st.pos_y, pos_y, ES * 8, cudaMemcpyHostToDevice, stream));
  if (cursor) CUDA_TRY(cudaMemcpyAsync(eng->st.cursor, cursor, eng->st.E * 4, cudaMemcpyHostToDevice, stream));
  if (step_count) CUDA_TRY(cudaMemcpyAsync(eng->st.step_count, step_count, eng->st.E * 4, cudaMemcpyHostToDevice, stream));
  if (reset_next) CUDA_TRY(cudaMemcpyAsync(eng->st.reset_next, reset_next, eng->st.E, cudaMemcpyHostToDevice, stream));
  CUDA_TRY(cudaStreamSynchronize(stream));
  return 0;
}

#ifdef SWB_PHASE_CLOCKS
// debug build only: cumulative cycles per render phase (see SWB_MARK); resets the counters
int swb_debug_phase_clocks(unsigned long long *out16) {
  unsigned long long zero[16] = {0};
  if (cudaMemcpyFromSymbol(out16, swb::g_phase_clk, sizeof(zero)) != cudaSuccess) return 1;
  return cudaMemcpyToSymbol(swb::g_phase_clk, zero, sizeof(zero)) != cudaSuccess;
}
#endif

int64_t swb_launch_count(const swb_engine *eng) { return eng ? eng->launches : 0; }

}  // extern "C"
