// C-ABI of the engine (include/spriteworld_b200.h): engine/raster lifetime, scene upload,
// kernel launches.  No torch types; plain CUDA runtime.
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <optional>
#include <string>
#include <vector>

#include "swb_device.cuh"
#include "swb_render.cuh"
#include "swb_sampler.cuh"
#include "swb_states.cuh"
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

// Pinned staging of the env ids of swb_save_envs / swb_load_envs / swb_copy_envs and its device
// twin, `cap` int32 each; two alternate, so the host stages call i+1 while call i's copy is queued.
struct IdSlot {
  size_t cap = 0;
  int32_t *host = nullptr, *dev = nullptr;
  cudaEvent_t done = nullptr;  // recorded after the kernels that read `dev`
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
  // env records: id staging, and the records of an overlapping swb_copy_envs (grown on demand)
  IdSlot id_slots[2];
  int id_next = 0;
  unsigned char *d_records = nullptr;
  size_t records_bytes = 0;
  // device-checked id lists (IdCall in swb_states.cuh): claims, the failure word, the status record
  unsigned long long *d_id_claim = nullptr, *d_id_fail = nullptr;
  swb_ids_status *d_id_status = nullptr;
  uint32_t id_seq = 0;
  // device scene sampler (swb_sampler_load): program, refill bookkeeping, first failure
  swb_scene_program *d_prog = nullptr;
  uint64_t seed = 0;
  int64_t env_offset = 0;
  int64_t *d_refilled_upto = nullptr;
  swb_sampler_status *d_sampler_status = nullptr;
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
int swb_version(void) { return 4; }
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
  A(&eng->d_id_claim, st.E); A(&eng->d_id_fail, 1); A(&eng->d_id_status, 1);
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
  CUDA_TRY(cudaMemset(eng->d_id_claim, 0xFF, (size_t)st.E * sizeof(unsigned long long)));
  CUDA_TRY(cudaMemset(eng->d_id_fail, 0xFF, sizeof(unsigned long long)));
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
  for (auto &slot : eng->id_slots) {
    if (slot.in_flight) cudaEventSynchronize(slot.done);
    if (slot.host) cudaFreeHost(slot.host);
    if (slot.dev) cudaFree(slot.dev);
    if (slot.done) cudaEventDestroy(slot.done);
  }
  cudaFree(eng->d_records);
  cudaFree(eng->d_prog); cudaFree(eng->d_refilled_upto); cudaFree(eng->d_sampler_status);
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

enum { STEP_WHOLE = 0, STEP_TASK = 1, STEP_ACTION = 2 };  // step_kernel modes

// What a step_kernel launch reads from its caller: the engine, every output pointer and, unless
// it evaluates the task only, actions of a dtype the engine's action kind takes.
static int check_step(const swb_engine *eng, const void *actions, int32_t action_dtype,
                      const swb_step_out *out, int mode) {
  if (!eng || !out || (mode != STEP_TASK && !actions)) return fail("step: null argument");
  if (!out->reward || !out->step_type || !out->success || !out->status)
    return fail("step: every swb_step_out pointer must be set");
  if (mode == STEP_TASK) return 0;
  const bool emb = eng->cfg.action_kind == SWB_ACT_EMBODIED;
  if (emb && action_dtype != SWB_DTYPE_I32) return fail("Embodied actions must be int32 [E][2]");
  if (!emb && action_dtype != SWB_DTYPE_F32 && action_dtype != SWB_DTYPE_F64)
    return fail("SelectMove/DragAndDrop actions must be float32 or float64 [E][4]");
  return 0;
}

// Enqueues step_kernel over every env, after check_step has passed.
static int launch_step(swb_engine *eng, const void *actions, int32_t action_dtype,
                       const swb_step_out &out, cudaStream_t stream, int mode) {
  CUDA_TRY(cudaSetDevice(eng->device));
  const int blocks = (eng->st.E + STEP_WARPS - 1) / STEP_WARPS;
  step_kernel<<<blocks, STEP_WARPS * 32, 0, stream>>>(eng->st, eng->d_step_cfg, actions, action_dtype, out, mode);
  eng->launches++;
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int swb_step(swb_engine *eng, const void *actions, int32_t action_dtype, const swb_step_out *out,
             void *stream) {
  if (check_step(eng, actions, action_dtype, out, STEP_WHOLE)) return 1;
  return launch_step(eng, actions, action_dtype, *out, static_cast<cudaStream_t>(stream), STEP_WHOLE);
}

int swb_eval_task(swb_engine *eng, const swb_step_out *out, void *stream) {
  if (check_step(eng, nullptr, SWB_DTYPE_F32, out, STEP_TASK)) return 1;
  return launch_step(eng, nullptr, SWB_DTYPE_F32, *out, static_cast<cudaStream_t>(stream), STEP_TASK);
}

int swb_apply_action(swb_engine *eng, const void *actions, int32_t action_dtype,
                     const swb_step_out *out, void *stream) {
  if (check_step(eng, actions, action_dtype, out, STEP_ACTION)) return 1;
  return launch_step(eng, actions, action_dtype, *out, static_cast<cudaStream_t>(stream), STEP_ACTION);
}

// The checks of a render launch of raster `r` by `eng` with `max_spans` spans per sprite row;
// on success *plan is the shared-memory layout the launch needs.  Every entry point that renders
// runs them before it enqueues anything; swb_raster_create runs them for a convex-only pool.
static int check_render(const swb_engine *eng, const swb_raster *r, int max_spans,
                        std::optional<RenderLayout> *plan) {
  if (r->eng != eng) return fail("raster belongs to another engine");
  const RasterDev &rd = r->rd;
  int max_smem = 0;
  CUDA_TRY(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, eng->device));
  RenderLayout L(eng->st.S, r->smem_rows, max_spans, rd.band_rows, rd.W, rd.aa, rd.ncls_x, rd.ncls_y,
                 rd.prefix_stride, rd.v_nks);
  // many convex slots on a wide raster: rather than refuse the raster, keep 16 visible segments
  // per canvas row as with concave shapes (a row with more is flagged, see RenderLayout)
  if (L.total > max_smem && L.segcap > 16)
    L = RenderLayout(eng->st.S, r->smem_rows, max_spans, rd.band_rows, rd.W, rd.aa, rd.ncls_x,
                     rd.ncls_y, rd.prefix_stride, rd.v_nks, false);
  if ((L.cap + max_spans) * 4 * r->smem_rows > L.scratch_bytes)
    return fail("render scratch (%d B) cannot hold one sprite spanning %d canvas rows", L.scratch_bytes,
                r->smem_rows);
  if (L.total > max_smem)
    return fail("render needs %d B of shared memory per CTA (limit %d): too many sprite slots / too large a canvas",
                L.total, max_smem);
  plan->emplace(L);
  return 0;
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
  rd.prefix_stride = r->ax.prefix_stride;
  int rows = 0;
  for (int b = 0; b < rd.n_bands; ++b) {
    const int y0 = b * rd.band_rows, y1 = std::min(y0 + rd.band_rows, height) - 1;
    // the kernel counts a band's canvas rows from a multiple of four
    rows = std::max(rows, r->ay.win_min[y1] + r->ay.win_len[y1] - (r->ay.win_min[y0] & ~3));
  }
  r->smem_rows = rows;
  // a tile's canvas rows must fit the H tile's row length: as many blocks per tile as fit
  rd.tile_blocks = choose_tile_blocks(r->ay, rd.band_rows, TILE_BLOCKS, 4 * HT_ROWW);
  if (rd.tile_blocks == 0) {
    const int span = tile_span(r->ay, rd.band_rows, 1);
    delete r;
    return fail("vertical tap windows of 8 output rows span %d canvas rows, more than the %d of the "
                "render kernel's H tile (anti_aliasing %d is too large for a frame %d rows high)",
                span, 4 * HT_ROWW, aa, height);
  }
  VFragHost vf;
  if (!build_vfrag(r->ay, &vf, &err)) {
    delete r;
    return fail("%s", err.c_str());
  }
  if (vf.nks > V_KS_WIDE) {  // cannot happen: one block's windows fit 4 * HT_ROWW canvas rows
    delete r;
    return fail("vertical pass needs %d k-steps (limit %d)", vf.nks, V_KS_WIDE);
  }
  rd.v_nks = vf.nks;
  // refuse a raster that cannot render even convex shapes (a star or spoke may still fail later)
  std::optional<RenderLayout> plan;
  if (check_render(eng, r, 1, &plan)) {
    delete r;
    return 1;
  }
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

// Enqueues render_kernel for envs [env_base, env_base + env_count) with a layout check_render
// returned.  after_step: the launch follows this step's step_kernel on the stream.  It is then
// made a programmatic dependent launch: the render CTAs may become resident and load their tables
// while the step kernel's last CTAs run (step_kernel signals griddepcontrol.launch_dependents at
// once), and wait (griddepcontrol.wait, after their set-up) until the step grid has completed and
// its writes are visible.
static int enqueue_render(swb_engine *eng, const swb_raster *r, const RenderLayout &L,
                          const RenderTargets &targets, uint8_t *status, cudaStream_t stream,
                          int env_base, int env_count, bool after_step) {
  RasterDev rd = r->rd;
  rd.max_spans = L.M;
  // the wide instantiation only for rasters whose tables the narrow one was not compiled for
  const bool wide = render_wide(rd);
  auto kernel = targets.n > 1 ? (wide ? render_kernel<true, true> : render_kernel<true, false>)
                              : (wide ? render_kernel<false, true> : render_kernel<false, false>);
  CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, L.total));
  DevState st = eng->st;
  st.render_status = status;
  // persistent CTAs: one per resident slot (or per item if there are fewer), claiming
  // (env, band) items from the engine's counter; see render_kernel
  const int n_items = env_count * rd.n_bands;
  const int grid = std::min(n_items, eng->n_sms * (wide ? R_CTAS_PER_SM_WIDE : R_CTAS_PER_SM));
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

int swb_render(swb_engine *eng, swb_raster *r, uint8_t *frames, void *stream_) {
  if (!eng || !r || !frames) return fail("swb_render: null argument");
  std::optional<RenderLayout> plan;
  if (check_render(eng, r, eng->max_spans, &plan)) return 1;
  CUDA_TRY(cudaSetDevice(eng->device));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  CUDA_TRY(cudaMemsetAsync(eng->st.render_status, 0, eng->st.E, stream));
  return enqueue_render(eng, r, *plan, RenderTargets{{frames}, 1, 0, 0}, eng->st.render_status, stream,
                        0, eng->st.E, false);
}

int swb_step_render(swb_engine *eng, swb_raster *r, const void *actions, int32_t action_dtype,
                    const swb_step_out *out, uint8_t *frames, void *stream) {
  if (!eng || !r || !frames) return fail("swb_step_render: null argument");
  uint8_t *const dst[1] = {frames};  // one target at env offset 0: the frames of this engine alone
  return swb_step_render_gather(eng, r, actions, action_dtype, out, dst, 1, 0, stream);
}

int swb_step_render_gather(swb_engine *eng, swb_raster *r, const void *actions,
                           int32_t action_dtype, const swb_step_out *out, uint8_t *const *dst,
                           int32_t n_dst, int64_t env_offset, void *stream_) {
  if (!eng || !r || !dst) return fail("swb_step_render_gather: null argument");
  if (n_dst < 1 || n_dst > SWB_MAX_PEERS)
    return fail("swb_step_render_gather: n_dst = %d, expected 1..%d", n_dst, SWB_MAX_PEERS);
  if (env_offset < 0 || env_offset > INT32_MAX - eng->st.E)
    return fail("swb_step_render_gather: env_offset out of range");
  RenderTargets targets{{}, n_dst, (int)env_offset, (int)((env_offset / eng->st.E) % n_dst)};
  for (int i = 0; i < n_dst; ++i) {
    if (!dst[i]) return fail("swb_step_render_gather: dst[%d] is null", i);
    targets.dst[i] = dst[i];
  }
  std::optional<RenderLayout> plan;
  if (check_step(eng, actions, action_dtype, out, STEP_WHOLE) ||
      check_render(eng, r, eng->max_spans, &plan))
    return 1;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (launch_step(eng, actions, action_dtype, *out, stream, STEP_WHOLE)) return 1;
  return enqueue_render(eng, r, *plan, targets, out->status, stream, 0, eng->st.E, true);
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
  if (!eng) return fail("swb_step_host: null argument");
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
  std::optional<RenderLayout> plan;
  if (check_step(eng, actions, action_dtype, &eng->h_out, STEP_WHOLE) ||
      (r && check_render(eng, r, eng->max_spans, &plan)))
    return 1;
  // [E][2] int32 or [E][4] float32 / float64, as checked
  const size_t abytes = (size_t)E * (action_dtype == SWB_DTYPE_I32 ? 8 : action_dtype == SWB_DTYPE_F32 ? 16 : 32);
  CUDA_TRY(cudaMemcpyAsync(eng->h_actions, actions, abytes, cudaMemcpyHostToDevice, stream));
  const size_t fbytes = r ? (size_t)E * r->rd.H * r->rd.W * 3 : 0;
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
  if (launch_step(eng, eng->h_actions, action_dtype, eng->h_out, stream, STEP_WHOLE)) return 1;
  if (r) {
    const RenderTargets targets{{eng->h_frames}, 1, 0, 0};
    if (!frames) {
      if (enqueue_render(eng, r, *plan, targets, eng->h_out.status, stream, 0, E, true)) return 1;
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
        if (enqueue_render(eng, r, *plan, targets, eng->h_out.status, stream, e0, e1 - e0, c == 0)) return 1;
        CUDA_TRY(cudaEventRecord(eng->chunk_done[c], stream));
        CUDA_TRY(cudaStreamWaitEvent(eng->copy_stream, eng->chunk_done[c], 0));
        CUDA_TRY(cudaMemcpyAsync(frames + per_env * e0, eng->h_frames + per_env * e0, per_env * (e1 - e0),
                                 cudaMemcpyDeviceToHost, eng->copy_stream));
      }
      CUDA_TRY(cudaEventRecord(eng->copies_done, eng->copy_stream));
      CUDA_TRY(cudaStreamWaitEvent(stream, eng->copies_done, 0));
    }
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

}  // extern "C"

// Env ids of a record call: every id in [0, E); with `mark`, no id twice (destinations), and each
// id is marked in it.
static int check_env_ids(const swb_engine *eng, const char *fn, const int32_t *ids, int32_t n,
                         std::vector<uint8_t> *mark) {
  for (int32_t i = 0; i < n; ++i) {
    if (ids[i] < 0 || ids[i] >= eng->st.E)
      return fail("%s: env id %d out of range [0, %d)", fn, ids[i], eng->st.E);
    if (mark) {
      if ((*mark)[ids[i]]) return fail("%s: destination env id %d appears twice", fn, ids[i]);
      (*mark)[ids[i]] = 1;
    }
  }
  return 0;
}

// Moves `n` ids from `a` (and `n` from `b`, if given) into a staging slot and enqueues one copy of
// them to its device twin; the caller enqueues the kernels that read them, then finish_ids.
static int stage_ids(swb_engine *eng, const int32_t *a, const int32_t *b, int32_t n, cudaStream_t stream,
                     IdSlot **out) {
  IdSlot &slot = eng->id_slots[eng->id_next];
  eng->id_next ^= 1;
  if (slot.in_flight) {
    CUDA_TRY(cudaEventSynchronize(slot.done));
    slot.in_flight = false;
  }
  const size_t need = 2 * (size_t)n;
  if (need > slot.cap) {
    if (slot.host) cudaFreeHost(slot.host);
    if (slot.dev) cudaFree(slot.dev);
    slot.host = slot.dev = nullptr;
    slot.cap = 0;
    const size_t cap = std::max<size_t>(need, 1024);
    CUDA_TRY(cudaMallocHost(reinterpret_cast<void **>(&slot.host), cap * sizeof(int32_t)));
    CUDA_TRY(cudaMalloc(reinterpret_cast<void **>(&slot.dev), cap * sizeof(int32_t)));
    if (!slot.done) CUDA_TRY(cudaEventCreateWithFlags(&slot.done, cudaEventDisableTiming));
    slot.cap = cap;
  }
  memcpy(slot.host, a, n * sizeof(int32_t));
  if (b) memcpy(slot.host + n, b, n * sizeof(int32_t));
  CUDA_TRY(cudaMemcpyAsync(slot.dev, slot.host, (b ? 2 : 1) * n * sizeof(int32_t), cudaMemcpyHostToDevice,
                           stream));
  *out = &slot;
  return 0;
}

static int finish_ids(IdSlot *slot, cudaStream_t stream) {
  CUDA_TRY(cudaEventRecord(slot->done, stream));
  slot->in_flight = true;
  return 0;
}

static int launch_save(swb_engine *eng, const int32_t *d_ids, int32_t n, void *dst, cudaStream_t stream) {
  const int threads = 256, blocks = (int)(((size_t)n * eng->st.S + threads - 1) / threads);
  save_envs_kernel<<<blocks, threads, 0, stream>>>(eng->st, n, d_ids, static_cast<unsigned char *>(dst),
                                                   RecordLayout(eng->st.S).bytes());
  eng->launches++;
  CUDA_TRY(cudaGetLastError());
  return 0;
}

static int launch_load(swb_engine *eng, const int32_t *d_ids, int32_t n, const void *src,
                       cudaStream_t stream) {
  const int threads = 256, blocks = (int)(((size_t)n * eng->st.S + threads - 1) / threads);
  load_envs_kernel<<<blocks, threads, 0, stream>>>(eng->st, n, d_ids, static_cast<const unsigned char *>(src),
                                                   RecordLayout(eng->st.S).bytes());
  eng->launches++;
  CUDA_TRY(cudaGetLastError());
  return 0;
}

// Engine scratch of at least `need` bytes for the records of a copy.
static int grow_records(swb_engine *eng, size_t need) {
  if (need <= eng->records_bytes) return 0;
  if (eng->d_records) {
    CUDA_TRY(cudaDeviceSynchronize());  // an earlier copy on any stream may still read it
    cudaFree(eng->d_records);
    eng->d_records = nullptr;
    eng->records_bytes = 0;
  }
  CUDA_TRY(cudaMalloc(reinterpret_cast<void **>(&eng->d_records), need));
  eng->records_bytes = need;
  return 0;
}

// Host checks of a device id list: everything the host sees without reading device memory.
static int check_dev_ids(const swb_engine *eng, const char *fn, const void *ids, int32_t id_dtype) {
  if (!ids) return fail("%s: null argument", fn);
  if (id_dtype != SWB_DTYPE_I32 && id_dtype != SWB_DTYPE_I64)
    return fail("%s: id_dtype must be SWB_DTYPE_I32 or SWB_DTYPE_I64, got %d", fn, id_dtype);
  if (reinterpret_cast<uintptr_t>(ids) % (id_dtype == SWB_DTYPE_I64 ? 8 : 4))
    return fail("%s: ids are not aligned to their type", fn);
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, ids) != cudaSuccess) {
    cudaGetLastError();
    return fail("%s: ids are not device memory", fn);
  }
  if ((at.type != cudaMemoryTypeDevice && at.type != cudaMemoryTypeManaged) || at.device != eng->device)
    return fail("%s: ids must be device memory of device %d", fn, eng->device);
  return 0;
}

// The IdCall of the next device-checked call; enqueues nothing but, once every 2^32 - 2 calls,
// the reset of the claims and the failure word that lets the sequence number start over.
static int begin_id_call(swb_engine *eng, int call, const void *a, const void *b, int dst_arg, int32_t n,
                         cudaStream_t stream, IdCall *c) {
  if (++eng->id_seq == 0xFFFFFFFFu) {
    CUDA_TRY(cudaMemsetAsync(eng->d_id_claim, 0xFF, (size_t)eng->st.E * sizeof(unsigned long long), stream));
    CUDA_TRY(cudaMemsetAsync(eng->d_id_fail, 0xFF, sizeof(unsigned long long), stream));
    eng->id_seq = 1;
  }
  c->ids[0] = a;
  c->ids[1] = b;
  c->n = n;
  c->dst_arg = dst_arg;
  c->call = call;
  c->hi = (unsigned long long)(~eng->id_seq) << 32;
  c->claim = eng->d_id_claim;
  c->fail = eng->d_id_fail;
  c->status = eng->d_id_status;
  return 0;
}

static unsigned grid_of(size_t threads) { return (unsigned)((threads + 255) / 256); }

template <typename T>
static int enqueue_save_dev(swb_engine *eng, const IdCall &c, void *dst, cudaStream_t stream) {
  const size_t rb = RecordLayout(eng->st.S).bytes();
  check_ids_kernel<T><<<grid_of(c.n), 256, 0, stream>>>(c, eng->st.E);
  save_envs_dev_kernel<T><<<grid_of((size_t)c.n * eng->st.S), 256, 0, stream>>>(
      eng->st, c, static_cast<unsigned char *>(dst), rb);
  eng->launches += 2;
  CUDA_TRY(cudaGetLastError());
  return 0;
}

template <typename T>
static int enqueue_load_dev(swb_engine *eng, const IdCall &c, const void *src, cudaStream_t stream) {
  const size_t rb = RecordLayout(eng->st.S).bytes();
  check_ids_kernel<T><<<grid_of(c.n), 256, 0, stream>>>(c, eng->st.E);
  repeat_ids_kernel<T><<<grid_of(c.n), 256, 0, stream>>>(c, eng->st.E);
  load_envs_dev_kernel<T><<<grid_of((size_t)c.n * eng->st.S), 256, 0, stream>>>(
      eng->st, c, static_cast<const unsigned char *>(src), rb);
  eng->launches += 3;
  CUDA_TRY(cudaGetLastError());
  return 0;
}

template <typename T>
static int enqueue_copy_dev(swb_engine *eng, const IdCall &c, cudaStream_t stream) {
  const size_t rb = RecordLayout(eng->st.S).bytes();
  check_ids_kernel<T><<<grid_of(2 * (size_t)c.n), 256, 0, stream>>>(c, eng->st.E);
  stage_copy_dev_kernel<T><<<grid_of((size_t)c.n * eng->st.S), 256, 0, stream>>>(eng->st, c, eng->d_records, rb);
  load_envs_dev_kernel<T><<<grid_of((size_t)c.n * eng->st.S), 256, 0, stream>>>(eng->st, c, eng->d_records, rb);
  eng->launches += 3;
  CUDA_TRY(cudaGetLastError());
  return 0;
}

extern "C" {

int64_t swb_env_record_bytes(const swb_engine *eng) {
  if (!eng) {
    fail("swb_env_record_bytes: null engine");
    return -1;
  }
  return (int64_t)RecordLayout(eng->st.S).bytes();
}

int swb_save_envs(swb_engine *eng, const int32_t *env_ids, int32_t n, void *dst, uint64_t dst_bytes,
                  int32_t *span_class, void *stream_) {
  if (!eng || !span_class) return fail("swb_save_envs: null argument");
  if (n < 0) return fail("swb_save_envs: n = %d", n);
  if (n == 0) {
    *span_class = eng->max_spans;
    return 0;
  }
  if (!env_ids || !dst) return fail("swb_save_envs: null argument");
  if (reinterpret_cast<uintptr_t>(dst) % 16) return fail("swb_save_envs: dst is not 16-byte aligned");
  const uint64_t need = (uint64_t)n * RecordLayout(eng->st.S).bytes();
  if (dst_bytes < need)
    return fail("swb_save_envs: %d records need %llu bytes, the buffer has %llu", n,
                (unsigned long long)need, (unsigned long long)dst_bytes);
  if (check_env_ids(eng, "swb_save_envs", env_ids, n, nullptr)) return 1;
  CUDA_TRY(cudaSetDevice(eng->device));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  IdSlot *slot = nullptr;
  if (stage_ids(eng, env_ids, nullptr, n, stream, &slot) || launch_save(eng, slot->dev, n, dst, stream))
    return 1;
  *span_class = eng->max_spans;
  return finish_ids(slot, stream);
}

int swb_load_envs(swb_engine *eng, const int32_t *env_ids, int32_t n, const void *src, uint64_t src_bytes,
                  int32_t span_class, void *stream_) {
  if (!eng) return fail("swb_load_envs: null engine");
  if (n < 0) return fail("swb_load_envs: n = %d", n);
  if (span_class != 1 && span_class != 4)
    return fail("swb_load_envs: span_class must be 1 or 4, got %d", span_class);
  if (n == 0) return 0;
  if (!env_ids || !src) return fail("swb_load_envs: null argument");
  if (reinterpret_cast<uintptr_t>(src) % 16) return fail("swb_load_envs: src is not 16-byte aligned");
  const uint64_t need = (uint64_t)n * RecordLayout(eng->st.S).bytes();
  if (src_bytes < need)
    return fail("swb_load_envs: %d records need %llu bytes, the buffer has %llu", n,
                (unsigned long long)need, (unsigned long long)src_bytes);
  std::vector<uint8_t> mark(eng->st.E, 0);
  if (check_env_ids(eng, "swb_load_envs", env_ids, n, &mark)) return 1;
  CUDA_TRY(cudaSetDevice(eng->device));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  // records of stars or spokes need the concave span tables, as if their scenes were uploaded
  eng->max_spans = std::max(eng->max_spans, (int)span_class);
  IdSlot *slot = nullptr;
  if (stage_ids(eng, env_ids, nullptr, n, stream, &slot) || launch_load(eng, slot->dev, n, src, stream))
    return 1;
  return finish_ids(slot, stream);
}

int swb_copy_envs(swb_engine *eng, const int32_t *src_ids, const int32_t *dst_ids, int32_t n, void *stream_) {
  if (!eng) return fail("swb_copy_envs: null engine");
  if (n < 0) return fail("swb_copy_envs: n = %d", n);
  if (n == 0) return 0;
  if (!src_ids || !dst_ids) return fail("swb_copy_envs: null argument");
  std::vector<uint8_t> mark(eng->st.E, 0);
  if (check_env_ids(eng, "swb_copy_envs", dst_ids, n, &mark) ||
      check_env_ids(eng, "swb_copy_envs", src_ids, n, nullptr))
    return 1;
  bool overlap = false;
  for (int32_t i = 0; i < n && !overlap; ++i) overlap = mark[src_ids[i]] != 0;
  CUDA_TRY(cudaSetDevice(eng->device));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  // an env both read and written: every source is saved to engine scratch before any destination
  // is written, so every read sees the state from before the call
  if (grow_records(eng, overlap ? (size_t)n * RecordLayout(eng->st.S).bytes() : 0)) return 1;
  IdSlot *slot = nullptr;
  if (stage_ids(eng, src_ids, dst_ids, n, stream, &slot)) return 1;
  if (!overlap) {
    const int threads = 256, blocks = (int)(((size_t)n * eng->st.S + threads - 1) / threads);
    copy_envs_kernel<<<blocks, threads, 0, stream>>>(eng->st, n, slot->dev, slot->dev + n);
    eng->launches++;
    CUDA_TRY(cudaGetLastError());
    return finish_ids(slot, stream);
  }
  if (launch_save(eng, slot->dev, n, eng->d_records, stream) ||
      launch_load(eng, slot->dev + n, n, eng->d_records, stream))
    return 1;
  return finish_ids(slot, stream);
}

int swb_save_envs_dev(swb_engine *eng, const void *env_ids, int32_t id_dtype, int32_t n, void *dst,
                      uint64_t dst_bytes, int32_t *span_class, void *stream_) {
  if (!eng || !span_class) return fail("swb_save_envs_dev: null argument");
  if (n < 0) return fail("swb_save_envs_dev: n = %d", n);
  if (n == 0) {
    *span_class = eng->max_spans;
    return 0;
  }
  if (!dst) return fail("swb_save_envs_dev: null argument");
  if (check_dev_ids(eng, "swb_save_envs_dev", env_ids, id_dtype)) return 1;
  if (reinterpret_cast<uintptr_t>(dst) % 16) return fail("swb_save_envs_dev: dst is not 16-byte aligned");
  const uint64_t need = (uint64_t)n * RecordLayout(eng->st.S).bytes();
  if (dst_bytes < need)
    return fail("swb_save_envs_dev: %d records need %llu bytes, the buffer has %llu", n,
                (unsigned long long)need, (unsigned long long)dst_bytes);
  CUDA_TRY(cudaSetDevice(eng->device));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  IdCall c;
  if (begin_id_call(eng, SWB_IDS_CALL_SAVE, env_ids, nullptr, -1, n, stream, &c)) return 1;
  if (id_dtype == SWB_DTYPE_I64 ? enqueue_save_dev<int64_t>(eng, c, dst, stream)
                                : enqueue_save_dev<int32_t>(eng, c, dst, stream))
    return 1;
  *span_class = eng->max_spans;
  return 0;
}

int swb_load_envs_dev(swb_engine *eng, const void *env_ids, int32_t id_dtype, int32_t n, const void *src,
                      uint64_t src_bytes, int32_t span_class, void *stream_) {
  if (!eng) return fail("swb_load_envs_dev: null engine");
  if (n < 0) return fail("swb_load_envs_dev: n = %d", n);
  if (span_class != 1 && span_class != 4)
    return fail("swb_load_envs_dev: span_class must be 1 or 4, got %d", span_class);
  if (n == 0) return 0;
  if (!src) return fail("swb_load_envs_dev: null argument");
  if (check_dev_ids(eng, "swb_load_envs_dev", env_ids, id_dtype)) return 1;
  if (reinterpret_cast<uintptr_t>(src) % 16) return fail("swb_load_envs_dev: src is not 16-byte aligned");
  const uint64_t need = (uint64_t)n * RecordLayout(eng->st.S).bytes();
  if (src_bytes < need)
    return fail("swb_load_envs_dev: %d records need %llu bytes, the buffer has %llu", n,
                (unsigned long long)need, (unsigned long long)src_bytes);
  CUDA_TRY(cudaSetDevice(eng->device));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  eng->max_spans = std::max(eng->max_spans, (int)span_class);
  IdCall c;
  if (begin_id_call(eng, SWB_IDS_CALL_LOAD, env_ids, nullptr, 0, n, stream, &c)) return 1;
  return id_dtype == SWB_DTYPE_I64 ? enqueue_load_dev<int64_t>(eng, c, src, stream)
                                   : enqueue_load_dev<int32_t>(eng, c, src, stream);
}

int swb_copy_envs_dev(swb_engine *eng, const void *src_ids, const void *dst_ids, int32_t id_dtype, int32_t n,
                      void *stream_) {
  if (!eng) return fail("swb_copy_envs_dev: null engine");
  if (n < 0) return fail("swb_copy_envs_dev: n = %d", n);
  if (n == 0) return 0;
  if (check_dev_ids(eng, "swb_copy_envs_dev", src_ids, id_dtype) ||
      check_dev_ids(eng, "swb_copy_envs_dev", dst_ids, id_dtype))
    return 1;
  CUDA_TRY(cudaSetDevice(eng->device));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (grow_records(eng, (size_t)n * RecordLayout(eng->st.S).bytes())) return 1;
  IdCall c;
  if (begin_id_call(eng, SWB_IDS_CALL_COPY, src_ids, dst_ids, 1, n, stream, &c)) return 1;
  return id_dtype == SWB_DTYPE_I64 ? enqueue_copy_dev<int64_t>(eng, c, stream)
                                   : enqueue_copy_dev<int32_t>(eng, c, stream);
}

int swb_env_ids_status_pointer(swb_engine *eng, swb_ids_status **status) {
  if (!eng || !status) return fail("swb_env_ids_status_pointer: null argument");
  *status = eng->d_id_status;
  return 0;
}

}  // extern "C"

namespace {

// Records a rejection loop that ran out of tries, unless an earlier one is recorded.
__device__ void sampler_fail(swb_sampler_status *st, int op, int64_t g, int64_t a) {
  if (atomicCAS(&st->failed, 0u, 1u) == 0u) {
    st->op = op;
    st->env = g;
    st->scene = a;
  }
}

// swb_sample_scenes: one thread per requested scene.
__global__ void sample_scenes_kernel(const swb_scene_program *__restrict__ prog, uint64_t seed, int S,
                                     const int64_t *__restrict__ env_ids,
                                     const int64_t *__restrict__ scene_idx, int n, swb_sample_out out,
                                     swb_sampler_status *status) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t g = env_ids[i], a = scene_idx[i];
  swb_sampler::Scene sc;
  const int bad = swb_sampler::sample_and_pack(
      *prog, seed, (uint64_t)g, (uint64_t)a, S, sc,
      [&](int slot, const swb_sampler::Packed &o, const swb_sampler::Sprite *s) {
        const size_t d = (size_t)i * S + slot;
        out.x[d] = o.x; out.y[d] = o.y;
        out.m00[d] = o.m00; out.m01[d] = o.m01; out.m10[d] = o.m10; out.m11[d] = o.m11;
        out.vx[d] = o.vx; out.vy[d] = o.vy;
        out.member[d] = o.member; out.shape[d] = o.shape; out.pos_f32[d] = o.pos_f32;
        for (int c = 0; c < 3; ++c) out.rgb[d * 3 + c] = o.rgb[c];
        for (int f = 0; f < 5; ++f) out.factors[d * 5 + f] = o.factors[f];
        for (int f = 0; f < swb_sampler::kFactors; ++f) {
          out.factor_value[d * swb_sampler::kFactors + f] = s ? s->val[f] : 0.0;
          out.factor_kind[d * swb_sampler::kFactors + f] = s ? s->kind[f] : (uint8_t)SWB_FT_NONE;
        }
      });
  if (bad >= 0) sampler_fail(status, bad, g, a);
}

// swb_refill_device: one thread per env, scenes refilled_upto + 1 .. scene_serial + K - 1 into the
// ring.  The scene the env is on (ring slot serial % K) is never among them.
__global__ void refill_device_kernel(const swb_scene_program *__restrict__ prog, uint64_t seed,
                                     int64_t env_offset, DevState st, int64_t *refilled_upto,
                                     swb_sampler_status *status, float *static_rows) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= st.E) return;
  const int64_t serial = st.scene_serial[e], want = serial + st.K - 1;
  const int64_t g = env_offset + e;
  // from the first scene not sampled yet, never below the one after the current scene (scene 0
  // itself is sampled by the first refill after swb_sampler_load)
  const int64_t lo = refilled_upto[e] < 0 ? serial : serial + 1;
  int64_t a = refilled_upto[e] + 1;
  if (a < lo) a = lo;
  for (; a <= want; ++a) {
    const size_t base = ((size_t)e * st.K + (size_t)(a % st.K)) * st.S;
    swb_sampler::Scene sc;
    const int bad = swb_sampler::sample_and_pack(
        *prog, seed, (uint64_t)g, (uint64_t)a, st.S, sc,
        [&](int slot, const swb_sampler::Packed &o, const swb_sampler::Sprite *) {
          const size_t d = base + slot;
          st.p_x[d] = o.x; st.p_y[d] = o.y;
          st.p_m00[d] = o.m00; st.p_m01[d] = o.m01; st.p_m10[d] = o.m10; st.p_m11[d] = o.m11;
          st.p_vx[d] = o.vx; st.p_vy[d] = o.vy;
          st.p_member[d] = o.member; st.p_shape[d] = o.shape; st.p_pos_f32[d] = o.pos_f32;
          st.p_rgb[d] = (uint32_t)o.rgb[0] | ((uint32_t)o.rgb[1] << 8) | ((uint32_t)o.rgb[2] << 16);
          for (int f = 0; f < 5; ++f) st.p_factors[d * 5 + f] = o.factors[f];
          if (static_rows) {   // shape, scale, angle, c0, c1, c2, vx, vy as float32
            float *r = static_rows + d * 8;
            r[0] = (float)o.shape;
            for (int f = 0; f < 5; ++f) r[1 + f] = o.factors[f];
            r[6] = (float)o.vx;
            r[7] = (float)o.vy;
          }
        });
    if (bad >= 0) sampler_fail(status, bad, g, a);
  }
  if (want > refilled_upto[e]) refilled_upto[e] = want;
}

// What the kernels rely on: every op, jump, constant and angle index inside the program.
int check_program(const swb_scene_program &p, int S) {
  if (p.n_ops < 1 || p.n_ops > SWB_PROG_MAX_OPS) return fail("program: n_ops %d out of range", p.n_ops);
  if (p.n_consts < 0 || p.n_consts > SWB_PROG_MAX_CONSTS) return fail("program: n_consts out of range");
  if (p.n_angles < 1 || p.n_angles > SWB_PROG_MAX_ANGLES) return fail("program: n_angles out of range");
  if (p.n_filters < 0 || p.n_filters > SWB_MAX_FILTERS) return fail("program: n_filters out of range");
  if (p.max_sprites < 0 || p.max_sprites > S)
    return fail("program: scenes of up to %d sprites do not fit %d slots", p.max_sprites, S);
  auto pc_ok = [&](int pc) { return pc >= 0 && pc < p.n_ops; };
  auto consts_ok = [&](int off, int n) { return n >= 1 && off >= 0 && off + n <= p.n_consts; };
  for (int f = 0; f < p.n_filters; ++f)
    if (!pc_ok(p.filter_pc[f])) return fail("program: filter %d has no code", f);
  for (int i = 0; i < p.n_ops; ++i) {
    const swb_prog_op &o = p.ops[i];
    const bool key_ok = o.key >= 0 && o.key < swb_sampler::kFactors;
    bool ok = true;
    switch (o.op) {
      case SWB_OP_G_END: case SWB_OP_G_MARK: case SWB_OP_G_SHUFFLE: case SWB_OP_D_RET:
      case SWB_OP_D_REJ_BEGIN: case SWB_OP_P_RET: case SWB_OP_P_NOT: break;
      case SWB_OP_G_SPRITES: ok = pc_ok(o.a) && o.b >= 0 && (o.dtype == 0 || o.c > o.b); break;
      case SWB_OP_G_CHOOSE: case SWB_OP_D_MIX: ok = consts_ok(o.c, o.b) && i + o.b < p.n_ops; break;
      case SWB_OP_G_JUMP: case SWB_OP_D_JUMP: ok = pc_ok(o.a); break;
      case SWB_OP_D_CONT: ok = key_ok; break;
      case SWB_OP_D_DISC: ok = key_ok && consts_ok(o.a, o.b) && (o.c < 0 || consts_ok(o.c, o.b)); break;
      case SWB_OP_D_REJ_END: ok = pc_ok(o.a); break;
      case SWB_OP_P_CONT: ok = key_ok; break;
      case SWB_OP_P_DISC: ok = key_ok && consts_ok(o.a, o.b); break;
      case SWB_OP_P_AND: case SWB_OP_P_OR: ok = o.b >= 1 && o.b <= SWB_PROG_MAX_STACK; break;
      default: ok = false;
    }
    if (!ok) return fail("program: op %d (code %d) is malformed", i, o.op);
  }
  return 0;
}

}  // namespace

extern "C" {

int swb_sampler_sizeof_program(void) { return (int)sizeof(swb_scene_program); }

int swb_sampler_load(swb_engine *eng, const swb_scene_program *prog, uint64_t seed, int64_t env_offset) {
  if (!eng || !prog) return fail("swb_sampler_load: null argument");
  if (env_offset < 0) return fail("swb_sampler_load: env_offset must be >= 0");
  if (check_program(*prog, eng->st.S)) return 1;
  CUDA_TRY(cudaSetDevice(eng->device));
  if (!eng->d_prog) {  // all three or none: the other calls test d_prog alone
    swb_scene_program *prog_d = nullptr;
    int64_t *upto_d = nullptr;
    swb_sampler_status *status_d = nullptr;
    if (dev_alloc(&prog_d, 1) != cudaSuccess || dev_alloc(&upto_d, eng->st.E) != cudaSuccess ||
        dev_alloc(&status_d, 1) != cudaSuccess) {
      cudaFree(prog_d); cudaFree(upto_d); cudaFree(status_d);
      return fail("swb_sampler_load: device allocation failed");
    }
    eng->d_prog = prog_d;
    eng->d_refilled_upto = upto_d;
    eng->d_sampler_status = status_d;
  }
  CUDA_TRY(cudaDeviceSynchronize());
  CUDA_TRY(cudaMemcpy(eng->d_prog, prog, sizeof(swb_scene_program), cudaMemcpyHostToDevice));
  CUDA_TRY(cudaMemset(eng->d_refilled_upto, 0xFF, (size_t)eng->st.E * sizeof(int64_t)));
  eng->seed = seed;
  eng->env_offset = env_offset;
  return 0;
}

int swb_sample_scenes(swb_engine *eng, const int64_t *env_ids, const int64_t *scene_idx, int32_t n,
                      const swb_sample_out *out, void *stream_) {
  if (!eng || !out) return fail("swb_sample_scenes: null argument");
  if (!eng->d_prog) return fail("swb_sample_scenes: no program (swb_sampler_load)");
  if (n < 0) return fail("swb_sample_scenes: n < 0");
  if (n == 0) return 0;
  if (!env_ids || !scene_idx || !out->x || !out->y || !out->m00 || !out->m01 || !out->m10 || !out->m11 ||
      !out->vx || !out->vy || !out->member || !out->shape || !out->pos_f32 || !out->rgb || !out->factors ||
      !out->factor_value || !out->factor_kind)
    return fail("swb_sample_scenes: every pointer must be set");
  CUDA_TRY(cudaSetDevice(eng->device));
  const int threads = 128;
  sample_scenes_kernel<<<(n + threads - 1) / threads, threads, 0, static_cast<cudaStream_t>(stream_)>>>(
      eng->d_prog, eng->seed, eng->st.S, env_ids, scene_idx, n, *out, eng->d_sampler_status);
  eng->launches++;
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int swb_refill_device(swb_engine *eng, float *static_rows, void *stream_) {
  if (!eng) return fail("swb_refill_device: null engine");
  if (!eng->d_prog) return fail("swb_refill_device: no program (swb_sampler_load)");
  CUDA_TRY(cudaSetDevice(eng->device));
  const int threads = 64;
  refill_device_kernel<<<(eng->st.E + threads - 1) / threads, threads, 0, static_cast<cudaStream_t>(stream_)>>>(
      eng->d_prog, eng->seed, eng->env_offset, eng->st, eng->d_refilled_upto, eng->d_sampler_status,
      static_rows);
  eng->launches++;
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int swb_sampler_pointers(swb_engine *eng, int64_t **refilled_upto, swb_sampler_status **status) {
  if (!eng) return fail("swb_sampler_pointers: null engine");
  if (!eng->d_prog) return fail("swb_sampler_pointers: no program (swb_sampler_load)");
  if (refilled_upto) *refilled_upto = eng->d_refilled_upto;
  if (status) *status = eng->d_sampler_status;
  return 0;
}

int swb_pool_pointers(swb_engine *eng, double **f64, uint32_t **member, uint8_t **shape, uint8_t **pos_f32,
                      uint32_t **rgb, float **factors) {
  if (!eng || !f64 || !member || !shape || !pos_f32 || !rgb || !factors)
    return fail("swb_pool_pointers: null argument");
  const DevState &st = eng->st;
  double *p[8] = {st.p_x, st.p_y, st.p_m00, st.p_m01, st.p_m10, st.p_m11, st.p_vx, st.p_vy};
  for (int i = 0; i < 8; ++i) f64[i] = p[i];
  *member = st.p_member; *shape = st.p_shape; *pos_f32 = st.p_pos_f32; *rgb = st.p_rgb;
  *factors = st.p_factors;
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
