// C-ABI of the engine (include/spriteworld_b200.h): engine/raster lifetime, scene upload,
// kernel launches.  No torch types; plain CUDA runtime.
#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <memory>
#include <optional>
#include <string>
#include <type_traits>
#include <vector>

#include "swb_contained.cuh"
#include "swb_device.cuh"
#include "swb_make_states.cuh"
#include "swb_masks.cuh"
#include "swb_render.cuh"
#include "swb_rollout.cuh"
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

}  // namespace

// Owners of CUDA resources: each releases its resource when destroyed; they move but do not copy.
struct FreeDev { void operator()(void *p) const { cudaFree(p); } };
struct FreeHost { void operator()(void *p) const { cudaFreeHost(p); } };
struct DestroyEvent { void operator()(cudaEvent_t e) const { cudaEventDestroy(e); } };
struct DestroyStream { void operator()(cudaStream_t s) const { cudaStreamDestroy(s); } };
template <typename T> using DevPtr = std::unique_ptr<T, FreeDev>;
template <typename T> using HostPtr = std::unique_ptr<T, FreeHost>;
using Event = std::unique_ptr<std::remove_pointer_t<cudaEvent_t>, DestroyEvent>;
using Stream = std::unique_ptr<std::remove_pointer_t<cudaStream_t>, DestroyStream>;

// *out <- a device array of n T (at least one), zero-filled unless `zero` is false.  The fill runs
// on the legacy default stream and may finish after the call has returned.
template <typename T>
static cudaError_t dev_alloc(DevPtr<T> *out, size_t n, bool zero = true) {
  const size_t bytes = (n ? n : 1) * sizeof(T);
  void *p = nullptr;
  cudaError_t e = cudaMalloc(&p, bytes);
  if (e == cudaSuccess) out->reset(static_cast<T *>(p));
  return e == cudaSuccess && zero ? cudaMemset(p, 0, bytes) : e;
}

static cudaError_t make_event(Event *out) {
  cudaEvent_t e = nullptr;
  const cudaError_t err = cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
  if (err == cudaSuccess) out->reset(e);
  return err;
}

// A buffer of at least the bytes last asked for.  grow(need, wait) keeps it if it holds `need`
// bytes; else it calls wait(), which returns once nothing may still read the old bytes, frees them
// and allocates `need` bytes.  If that allocation fails, the buffer is empty.
template <typename Owner, cudaError_t (*Alloc)(void **, size_t)>
struct Growable {
  Owner buf;
  size_t bytes = 0;
  unsigned char *get() const { return buf.get(); }
  template <typename Wait>
  cudaError_t grow(size_t need, Wait wait) {
    if (need <= bytes) return cudaSuccess;
    cudaError_t e = buf ? wait() : cudaSuccess;
    if (e != cudaSuccess) return e;
    buf.reset();
    bytes = 0;
    void *p = nullptr;
    if ((e = Alloc(&p, need)) != cudaSuccess) return e;
    buf.reset(static_cast<unsigned char *>(p));
    bytes = need;
    return cudaSuccess;
  }
};
using DevBuffer = Growable<DevPtr<unsigned char>, cudaMalloc>;
using HostBuffer = Growable<HostPtr<unsigned char>, cudaMallocHost>;
// The wait of a grow whose caller has already waited for every reader of the buffer.
constexpr auto kWaited = [] { return cudaSuccess; };

// The work that reads a buffer the host writes: an event recorded after the last of it.  wait()
// returns once that work has finished (at once if none was recorded), with an event ready for the
// next record().  The destructor waits too, so the buffers declared before an InFlight outlive
// their readers.
struct InFlight {
  Event done;
  cudaError_t wait() { return done ? cudaEventSynchronize(done.get()) : make_event(&done); }
  cudaError_t record(cudaStream_t stream) { return cudaEventRecord(done.get(), stream); }
  ~InFlight() { if (done) cudaEventSynchronize(done.get()); }
};

// A pinned host block and its device twin, grown on demand.  Two alternate (Staging::slots), so
// the host fills call i+1 while call i's copy is queued; a slot is reused only after its event.
struct StagingSlot {
  HostBuffer host;
  DevBuffer dev;
  InFlight readers;  // the kernels that read `dev`
};

struct Staging {
  StagingSlot slots[2];
  int next = 0;
};

// The device scene sampler (swb_sampler_load): program, refill bookkeeping, first failure.
struct SamplerDev {
  DevPtr<swb_scene_program> prog;
  DevPtr<int64_t> refilled_upto;
  DevPtr<swb_sampler_status> status;
};

// swb_step_host's device copies of the actions and of the step outputs
struct StepHostDev {
  DevPtr<double> actions, reward;
  DevPtr<int8_t> step_type;
  DevPtr<uint8_t> success, status;
  swb_step_out out() const { return {reward.get(), step_type.get(), success.get(), status.get()}; }
};

// swb_step_host's second stream: the D2H of frame chunks overlaps the render of the next chunk
struct ChunkCopies {
  Stream stream;
  Event chunk_done[8], copies_done;
};

struct swb_engine {
  swb_config cfg;
  StepCfg step_cfg;
  DevPtr<StepCfg> d_step_cfg;  // device copy the step kernel reads (per engine)
  DevPtr<unsigned> d_work;     // render kernel's work counter (monotonic, see render_kernel)
  unsigned work_base = 0;      // its value when the next launch starts
  int n_sms = 1;
  DevState st;
  // the arrays of st; declared before every owner whose destructor waits for copies into them
  std::vector<DevPtr<void>> arrays;
  int device = 0;
  int max_spans = 1;  // 1 while every uploaded shape is convex, else 4
  int64_t launches = 0;
  // scene uploads (from the refill thread, on its stream) and the ids of host-checked record
  // calls (on the step stream) stage apart, so that neither waits for or overwrites the other
  Staging upload_staging, id_staging;
  DevBuffer records;  // the records of a copy through engine scratch
  // device-checked id lists (IdCall in swb_states.cuh): claims, the failure word, the status record
  DevPtr<unsigned long long> d_id_claim, d_id_fail;
  DevPtr<swb_ids_status> d_id_status;
  uint32_t id_seq = 0;
  std::unique_ptr<SamplerDev> sampler;  // null until swb_sampler_load
  uint64_t seed = 0;
  int64_t env_offset = 0;
  // the packer of swb_make_states (swb_packer_load): filters, colour mode and angle table
  DevPtr<swb_scene_program> d_packer;
  bool packer_hsv = false;
  // buffers of swb_step_host, each group made on first use
  std::unique_ptr<StepHostDev> step_host;
  DevBuffer h_frames;
  std::unique_ptr<ChunkCopies> chunk_copies;
  // pinned staging of swb_save_engine / swb_load_engine; `ckpt_done` is recorded after the copies
  // of the last load, which read it after the call has returned
  HostBuffer h_ckpt;
  InFlight ckpt_done;
};

struct swb_raster {
  swb_engine *eng;
  RasterDev rd;
  AxisHost ax, ay;
  int smem_rows = 0;
  std::vector<DevPtr<void>> tables;  // the device arrays of rd
};

namespace {

__global__ void scatter_scenes_kernel(DevState st, int n, const int32_t *__restrict__ dst,
                                      const double *__restrict__ f64, size_t f64_stride,
                                      const uint32_t *__restrict__ member,
                                      const uint8_t *__restrict__ shape,
                                      const uint8_t *__restrict__ pos_f32,
                                      const uint32_t *__restrict__ rgb,
                                      const float *__restrict__ factors,
                                      const double *__restrict__ goal) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * st.S) return;
  const int sc = i / st.S, s = i - sc * st.S;
  if (s == 0)
    for (int j = 0; j < 2 * st.G; ++j) st.p_goal[(size_t)dst[sc] * st.G * 2 + j] = goal[(size_t)sc * st.G * 2 + j];
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
  DevPtr<T> p;
  CUDA_TRY(dev_alloc(&p, v.size(), false));
  CUDA_TRY(cudaMemcpy(p.get(), v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
  *out = p.get();
  r->tables.push_back(std::move(p));
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
int swb_version(void) { return 19; }
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
      if (nd.goal_slot < -1 || nd.goal_slot >= SWB_MAX_GOALS)
        return fail("node %d: goal_slot %d outside [-1, %d) (SWB_MAX_GOALS)", i, nd.goal_slot, SWB_MAX_GOALS);
    } else if (nd.kind != SWB_TASK_NO_REWARD) {
      return fail("unknown task kind %d", nd.kind);
    }
  }
  // goal slots 0 .. G-1, one node each
  int n_goals = 0, goal_nodes[SWB_MAX_GOALS];
  for (int g = 0; g < SWB_MAX_GOALS; ++g) goal_nodes[g] = -1;
  for (int i = 0; i < cfg->n_nodes; ++i) {
    const swb_task_node &nd = cfg->nodes[i];
    if (nd.kind != SWB_TASK_FIND_GOAL || nd.goal_slot < 0) continue;
    if (goal_nodes[nd.goal_slot] >= 0)
      return fail("goal_slot %d belongs to nodes %d and %d", nd.goal_slot, goal_nodes[nd.goal_slot], i);
    goal_nodes[nd.goal_slot] = i;
    n_goals = std::max(n_goals, nd.goal_slot + 1);
  }
  for (int g = 0; g < n_goals; ++g)
    if (goal_nodes[g] < 0) return fail("goal slots must be 0 .. %d, slot %d has no node", n_goals - 1, g);
  if (cfg->action_kind < 0 || cfg->action_kind > SWB_ACT_EMBODIED) return fail("bad action_kind");
  for (int s = 1; s < SWB_NUM_SHAPES; ++s)
    if (cfg->shape_n_verts[s] < 0 || cfg->shape_n_verts[s] > SWB_MAX_VERTS)
      return fail("shape %d has %d vertices (max %d)", s, cfg->shape_n_verts[s], SWB_MAX_VERTS);
  int n_dev = 0;
  CUDA_TRY(cudaGetDeviceCount(&n_dev));
  if (cfg->device < 0 || cfg->device >= n_dev) return fail("no CUDA device %d", cfg->device);
  CUDA_TRY(cudaSetDevice(cfg->device));

  std::unique_ptr<swb_engine> eng(new swb_engine());
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
  st.G = n_goals;
  const size_t ES = (size_t)st.E * st.S, EKS = ES * st.K;
  bool ok = true;
  auto own = [&](auto *owner, size_t n) { ok = ok && dev_alloc(owner, n) == cudaSuccess; };
  auto A = [&](auto **p, size_t n) {  // an array of st
    DevPtr<std::remove_pointer_t<std::remove_pointer_t<decltype(p)>>> a;
    own(&a, n);
    *p = a.get();
    eng->arrays.push_back(std::move(a));
  };
  A(&st.pos_x, ES); A(&st.pos_y, ES);
  A(&st.cursor, st.E); A(&st.step_count, st.E);
  A(&st.reset_next, st.E + 4); A(&st.render_status, st.E + 4);
  A(&st.p_x, EKS); A(&st.p_y, EKS);
  A(&st.p_m00, EKS); A(&st.p_m01, EKS); A(&st.p_m10, EKS); A(&st.p_m11, EKS);
  A(&st.p_vx, EKS); A(&st.p_vy, EKS);
  A(&st.p_member, EKS); A(&st.p_shape, EKS); A(&st.p_pos_f32, EKS); A(&st.p_rgb, EKS);
  A(&st.p_factors, EKS * 5);
  if (st.G) A(&st.p_goal, (size_t)st.E * st.K * st.G * 2);
  double *d_verts = nullptr;
  int32_t *d_nv = nullptr;
  own(&eng->d_step_cfg, 1);
  own(&eng->d_work, 1);
  A(&st.scene_serial, st.E);
  A(&d_verts, (size_t)SWB_NUM_SHAPES * SWB_MAX_VERTS * 2);
  A(&d_nv, SWB_NUM_SHAPES);
  own(&eng->d_id_claim, st.E); own(&eng->d_id_fail, 1); own(&eng->d_id_status, 1);
  if (!ok) return fail("device allocation failed: %s", cudaGetErrorString(cudaGetLastError()));
  CUDA_TRY(cudaMemcpy(eng->d_step_cfg.get(), &eng->step_cfg, sizeof(StepCfg), cudaMemcpyHostToDevice));
  CUDA_TRY(cudaMemcpy(d_verts, cfg->shape_verts, sizeof cfg->shape_verts, cudaMemcpyHostToDevice));
  CUDA_TRY(cudaMemcpy(d_nv, cfg->shape_n_verts, sizeof cfg->shape_n_verts, cudaMemcpyHostToDevice));
  st.shape_verts = d_verts;
  st.shape_n = d_nv;
  // every env starts "about to reset" (environment.py:70)
  CUDA_TRY(cudaMemset(st.reset_next, 1, st.E));
  CUDA_TRY(cudaMemset(eng->d_id_claim.get(), 0xFF, (size_t)st.E * sizeof(unsigned long long)));
  CUDA_TRY(cudaMemset(eng->d_id_fail.get(), 0xFF, sizeof(unsigned long long)));
  *out = eng.release();
  return 0;
}

void swb_engine_destroy(swb_engine *eng) {
  if (!eng) return;
  cudaSetDevice(eng->device);
  delete eng;
}

// The next slot of `staging`, of at least `need` bytes, once the kernels that last read it have
// finished.  The caller enqueues the copy to `dev` and the kernels that read it, then records them
// as the slot's readers.
static int take_slot(Staging &staging, size_t need, StagingSlot **out) {
  StagingSlot &slot = staging.slots[staging.next];
  staging.next ^= 1;
  CUDA_TRY(slot.readers.wait());  // the host rewrites the slot whether or not it grows
  const size_t bytes = std::max<size_t>(need, 4096);
  CUDA_TRY(slot.host.grow(bytes, kWaited));
  CUDA_TRY(slot.dev.grow(bytes, kWaited));
  *out = &slot;
  return 0;
}

// An upload of n scenes in its staging slot: [8 x f64][member u32][rgb u32][factors 5 x f32]
// [dst i32][shape u8][pos_f32 u8][goal G x 2 f64], each array 256-byte aligned, moved with ONE
// cudaMemcpyAsync and scattered into the pool by one kernel.
static size_t upload_layout(size_t n, int S, int G, size_t off[8]) {
  const size_t nS = n * S;
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o += (bytes + 255) & ~(size_t)255; return r; };
  off[0] = take(nS * 8 * sizeof(double));   // f64 x 8
  off[1] = take(nS * sizeof(uint32_t));     // member
  off[2] = take(nS * sizeof(uint32_t));     // rgb
  off[3] = take(nS * 5 * sizeof(float));    // factors
  off[4] = take(n * sizeof(int32_t));       // dst
  off[5] = take(nS);                        // shape
  off[6] = take(nS);                        // pos_f32
  off[7] = take(n * G * 2 * sizeof(double)); // goal
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
  const int G = eng->st.G;
  if (G && !sc->goal) return fail("swb_upload_scenes: the task samples %d goals per scene, goal is null", G);
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
  size_t off[8];
  StagingSlot *slot = nullptr;
  if (take_slot(eng->upload_staging, upload_layout(n, S, G, off), &slot)) return 1;
  unsigned char *h = slot->host.get();
  for (int a = 0; a < 8; ++a)
    memcpy(h + off[0] + a * nS * sizeof(double), f64_src[a], nS * sizeof(double));
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
  if (G) memcpy(h + off[7], sc->goal, (size_t)n * G * 2 * sizeof(double));
  // everything up to the end of the last used array, in one copy
  const size_t end = G ? off[7] + (size_t)n * G * 2 * sizeof(double) : off[6] + nS;
  CUDA_TRY(cudaMemcpyAsync(slot->dev.get(), h, end, cudaMemcpyHostToDevice, stream));
  const int threads = 256, blocks = (int)((nS + threads - 1) / threads);
  unsigned char *d = slot->dev.get();
  scatter_scenes_kernel<<<blocks, threads, 0, stream>>>(
      eng->st, n, reinterpret_cast<const int32_t *>(d + off[4]), reinterpret_cast<const double *>(d + off[0]),
      nS, reinterpret_cast<const uint32_t *>(d + off[1]), d + off[5], d + off[6],
      reinterpret_cast<const uint32_t *>(d + off[2]), reinterpret_cast<const float *>(d + off[3]),
      reinterpret_cast<const double *>(d + off[7]));
  eng->launches++;
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(slot->readers.record(stream));
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
  step_kernel<<<blocks, STEP_WARPS * 32, 0, stream>>>(eng->st, eng->d_step_cfg.get(), actions, action_dtype, out,
                                                      mode);
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

// The checks of a rollout from n_roots roots (`what`: "envs" for the live envs, else "roots") that
// every rollout entry point makes.  T * n_roots * C <= SWB_ROLLOUT_MAX_ENTRIES also keeps the
// kernel's warp index n_roots * C within an int32.
static_assert(SWB_ROLLOUT_MAX_ENTRIES <= 2147483647, "rollout indices are int32");
static int check_rollout(const swb_engine *eng, const char *fn, const char *what, const void *actions,
                         int32_t action_dtype, int32_t n_steps, int32_t n_candidates, int32_t n_roots,
                         const swb_step_out *out) {
  if (check_step(eng, actions, action_dtype, out, STEP_WHOLE)) return 1;
  if (n_steps < 1 || n_candidates < 1)
    return fail("%s: n_steps = %d and n_candidates = %d must both be >= 1", fn, n_steps, n_candidates);
  const int64_t plans = (int64_t)n_roots * n_candidates;
  if (plans > SWB_ROLLOUT_MAX_ENTRIES / n_steps)
    return fail("%s: %d steps x %d %s x %d candidates exceed %d entries per call", fn, n_steps, n_roots,
                what, n_candidates, SWB_ROLLOUT_MAX_ENTRIES);
  return 0;
}

// Enqueues the one rollout_kernel launch of a checked call: roots from io.roots unless it is null
// (the live envs), leaves into io.leaves unless it is null -- every step's records with `trajectory`.
static int enqueue_rollout(swb_engine *eng, const void *actions, int32_t action_dtype, int32_t n_steps,
                           int32_t n_candidates, const swb_step_out &out, RolloutRecords io,
                           cudaStream_t stream, bool trajectory = false) {
  CUDA_TRY(cudaSetDevice(eng->device));
  const int64_t plans = (int64_t)(io.roots ? io.n_roots : eng->st.E) * n_candidates;
  const unsigned blocks = (unsigned)((plans + ROLLOUT_WARPS - 1) / ROLLOUT_WARPS);
  auto kernel = trajectory ? (io.roots ? rollout_kernel<true, false, true> : rollout_kernel<false, false, true>)
                : io.roots ? (io.leaves ? rollout_kernel<true, true> : rollout_kernel<true, false>)
                           : (io.leaves ? rollout_kernel<false, true> : rollout_kernel<false, false>);
  kernel<<<blocks, ROLLOUT_WARPS * 32, 0, stream>>>(eng->st, eng->d_step_cfg.get(), actions, action_dtype,
                                                    n_steps, n_candidates, out, io);
  eng->launches++;
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int swb_rollout(swb_engine *eng, const void *actions, int32_t action_dtype, int32_t n_steps,
                int32_t n_candidates, const swb_step_out *out, void *stream) {
  if (check_rollout(eng, "swb_rollout", "envs", actions, action_dtype, n_steps, n_candidates,
                    eng ? eng->st.E : 0, out))
    return 1;
  return enqueue_rollout(eng, actions, action_dtype, n_steps, n_candidates, *out, RolloutRecords{},
                         static_cast<cudaStream_t>(stream));
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
  std::unique_ptr<swb_raster> r(new swb_raster());
  r->eng = eng;
  std::string err;
  if (!build_axis(width * aa, width, &r->ax, &err) || !build_axis(height * aa, height, &r->ay, &err))
    return fail("%s", err.c_str());
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
  if (rd.tile_blocks == 0)
    return fail("vertical tap windows of 8 output rows span %d canvas rows, more than the %d of the "
                "render kernel's H tile (anti_aliasing %d is too large for a frame %d rows high)",
                tile_span(r->ay, rd.band_rows, 1), 4 * HT_ROWW, aa, height);
  VFragHost vf;
  if (!build_vfrag(r->ay, &vf, &err)) return fail("%s", err.c_str());
  if (vf.nks > V_KS_WIDE)  // cannot happen: one block's windows fit 4 * HT_ROWW canvas rows
    return fail("vertical pass needs %d k-steps (limit %d)", vf.nks, V_KS_WIDE);
  rd.v_nks = vf.nks;
  // refuse a raster that cannot render even convex shapes (a star or spoke may still fail later)
  std::optional<RenderLayout> plan;
  if (check_render(eng, r.get(), 1, &plan)) return 1;
  const uint32_t *d_frag = nullptr;
  if (upload_axis(r.get(), r->ax, &rd.ax) || upload_axis(r.get(), r->ay, &rd.ay) ||
      upload_vec(r.get(), vf.blk_cls, &rd.v_blk_cls) || upload_vec(r.get(), vf.frag, &d_frag))
    return 1;
  rd.v_frag = reinterpret_cast<const uint2 *>(d_frag);  // cudaMalloc: 256-byte aligned
  *out = r.release();
  return 0;
}

void swb_raster_destroy(swb_raster *r) { delete r; }

// Enqueues render_kernel for envs [env_base, env_base + env_count) with a layout check_render
// returned.  after_step: the launch follows this step's step_kernel on the stream.  It is then
// made a programmatic dependent launch: the render CTAs may become resident and load their tables
// while the step kernel's last CTAs run (step_kernel signals griddepcontrol.launch_dependents at
// once), and wait (griddepcontrol.wait, after their set-up) until the step grid has completed and
// its writes are visible.  With recs.rec set, the items are records [0, env_count) of recs instead
// of live envs (swb_render_states; one target, env_base 0, status [env_count]).  With wins.win set,
// each of the env_count rows is drawn wins.V times (swb_render_windows; one target, env_base 0,
// status [env_count * V]).
static int enqueue_render(swb_engine *eng, const swb_raster *r, const RenderLayout &L,
                          const RenderTargets &targets, uint8_t *status, cudaStream_t stream,
                          int env_base, int env_count, bool after_step,
                          const RenderRecords &recs = RenderRecords{nullptr, 0},
                          const RenderWindows &wins = RenderWindows{nullptr, 1}) {
  RasterDev rd = r->rd;
  rd.max_spans = L.M;
  // the wide instantiation only for rasters whose tables the narrow one was not compiled for
  const bool wide = render_wide(rd);
  auto kernel = wins.win ? (recs.rec ? (wide ? render_kernel<false, true, true, true>
                                             : render_kernel<false, false, true, true>)
                                     : (wide ? render_kernel<false, true, false, true>
                                             : render_kernel<false, false, false, true>))
                : recs.rec ? (wide ? render_kernel<false, true, true> : render_kernel<false, false, true>)
                : targets.n > 1 ? (wide ? render_kernel<true, true, false> : render_kernel<true, false, false>)
                                : (wide ? render_kernel<false, true, false> : render_kernel<false, false, false>);
  CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, L.total));
  DevState st = eng->st;
  st.render_status = status;
  // persistent CTAs: one per resident slot (or per item if there are fewer), claiming
  // (env, band) items from the engine's counter; see render_kernel
  const int n_items = env_count * wins.V * rd.n_bands;
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
  CUDA_TRY(cudaLaunchKernelEx(&lc, kernel, st, rd, L, targets, env_base, n_items, eng->d_work.get(),
                              eng->work_base, recs, wins));
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
  if (!eng->step_host) {
    auto h = std::make_unique<StepHostDev>();
    // not zero-filled: nothing would order the fill before the writes that follow on `stream`
    CUDA_TRY(dev_alloc(&h->actions, (size_t)E * 4, false));
    CUDA_TRY(dev_alloc(&h->reward, E, false));
    CUDA_TRY(dev_alloc(&h->step_type, E + 4, false));
    CUDA_TRY(dev_alloc(&h->success, E + 4, false));
    CUDA_TRY(dev_alloc(&h->status, E + 4, false));
    eng->step_host = std::move(h);
  }
  const swb_step_out h_out = eng->step_host->out();
  std::optional<RenderLayout> plan;
  if (check_step(eng, actions, action_dtype, &h_out, STEP_WHOLE) ||
      (r && check_render(eng, r, eng->max_spans, &plan)))
    return 1;
  // [E][2] int32 or [E][4] float32 / float64, as checked
  const size_t abytes = (size_t)E * (action_dtype == SWB_DTYPE_I32 ? 8 : action_dtype == SWB_DTYPE_F32 ? 16 : 32);
  CUDA_TRY(cudaMemcpyAsync(eng->step_host->actions.get(), actions, abytes, cudaMemcpyHostToDevice, stream));
  const size_t fbytes = r ? (size_t)E * r->rd.H * r->rd.W * 3 : 0;
  if (fbytes > eng->h_frames.bytes) {
    CUDA_TRY(eng->h_frames.grow(fbytes, [&] { return cudaStreamSynchronize(stream); }));
    // written only by the render kernel's bulk copies, which initcheck does not track: zero
    // it once so that the tool sees every byte the D2H copies read as initialised
    CUDA_TRY(cudaMemsetAsync(eng->h_frames.get(), 0, fbytes, stream));
  }
  if (launch_step(eng, eng->step_host->actions.get(), action_dtype, h_out, stream, STEP_WHOLE)) return 1;
  if (r) {
    const RenderTargets targets{{eng->h_frames.get()}, 1, 0, 0};
    if (!frames) {
      if (enqueue_render(eng, r, *plan, targets, h_out.status, stream, 0, E, true)) return 1;
    } else {
      // render in env chunks; each chunk's frames go to the host on a second stream while
      // the next chunk renders
      if (!eng->chunk_copies) {
        auto c = std::make_unique<ChunkCopies>();
        cudaStream_t s = nullptr;
        CUDA_TRY(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
        c->stream.reset(s);
        for (Event &ev : c->chunk_done) CUDA_TRY(make_event(&ev));
        CUDA_TRY(make_event(&c->copies_done));
        eng->chunk_copies = std::move(c);
      }
      const ChunkCopies &cc = *eng->chunk_copies;
      const size_t per_env = (size_t)r->rd.H * r->rd.W * 3;
      const int n_chunks = E >= 1024 ? 8 : (E >= 64 ? 2 : 1);
      for (int c = 0; c < n_chunks; ++c) {
        const int e0 = (int)((int64_t)E * c / n_chunks), e1 = (int)((int64_t)E * (c + 1) / n_chunks);
        if (enqueue_render(eng, r, *plan, targets, h_out.status, stream, e0, e1 - e0, c == 0)) return 1;
        CUDA_TRY(cudaEventRecord(cc.chunk_done[c].get(), stream));
        CUDA_TRY(cudaStreamWaitEvent(cc.stream.get(), cc.chunk_done[c].get(), 0));
        CUDA_TRY(cudaMemcpyAsync(frames + per_env * e0, eng->h_frames.get() + per_env * e0, per_env * (e1 - e0),
                                 cudaMemcpyDeviceToHost, cc.stream.get()));
      }
      CUDA_TRY(cudaEventRecord(cc.copies_done.get(), cc.stream.get()));
      CUDA_TRY(cudaStreamWaitEvent(stream, cc.copies_done.get(), 0));
    }
  }
  if (reward) CUDA_TRY(cudaMemcpyAsync(reward, h_out.reward, (size_t)E * sizeof(double), cudaMemcpyDeviceToHost, stream));
  if (step_type) CUDA_TRY(cudaMemcpyAsync(step_type, h_out.step_type, E, cudaMemcpyDeviceToHost, stream));
  if (success) CUDA_TRY(cudaMemcpyAsync(success, h_out.success, E, cudaMemcpyDeviceToHost, stream));
  if (status) CUDA_TRY(cudaMemcpyAsync(status, h_out.status, E, cudaMemcpyDeviceToHost, stream));
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

// A record buffer `name` of fn that must hold n records: 16-byte aligned and large enough.
static int check_record_buffer(const swb_engine *eng, const char *fn, const char *name, const void *rec,
                               uint64_t rec_bytes, int64_t n) {
  if (reinterpret_cast<uintptr_t>(rec) % 16) return fail("%s: %s is not 16-byte aligned", fn, name);
  const uint64_t need = (uint64_t)n * RecordLayout(eng->st.S, eng->st.G).bytes();
  if (rec_bytes < need)
    return fail("%s: %lld records need %llu bytes, the buffer has %llu", fn, (long long)n,
                (unsigned long long)need, (unsigned long long)rec_bytes);
  return 0;
}

// The argument checks every save, load and copy makes before it checks its ids: the engine, n, a
// load's span class and, for n > 0, the id pointers and the record buffer of a save (dst) or a load
// (src): set, 16-byte aligned and n records long.  `call` is SWB_IDS_CALL_*; `fn` names the entry point.
static int check_record_args(const swb_engine *eng, const char *fn, int call, int32_t n, const void *ids0,
                             const void *ids1, const void *rec, uint64_t rec_bytes, int32_t span_class) {
  if (!eng) return fail("%s: null engine", fn);
  if (n < 0) return fail("%s: n = %d", fn, n);
  if (call == SWB_IDS_CALL_LOAD && span_class != 1 && span_class != 4)
    return fail("%s: span_class must be 1 or 4, got %d", fn, span_class);
  if (n == 0) return 0;
  if (!ids0 || (call == SWB_IDS_CALL_COPY ? !ids1 : !rec)) return fail("%s: null argument", fn);
  if (call == SWB_IDS_CALL_COPY) return 0;
  return check_record_buffer(eng, fn, call == SWB_IDS_CALL_SAVE ? "dst" : "src", rec, rec_bytes, n);
}

// Host ids of a record call: every id in [0, E); with `mark`, no id twice (destinations), and each
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

// Copies `n` host ids from `a` (and `n` from `b`, if given) into an id staging slot, enqueues their
// copy to its device twin, and makes *c the IdCall of them, checked on the host.  The kernels that
// read them are then recorded as (*slot)->readers.
static int stage_ids(swb_engine *eng, const int32_t *a, const int32_t *b, int32_t n, int dst_arg,
                     cudaStream_t stream, IdCall *c, StagingSlot **slot) {
  const size_t bytes = (b ? 2 : 1) * (size_t)n * sizeof(int32_t);
  if (take_slot(eng->id_staging, bytes, slot)) return 1;
  int32_t *h = reinterpret_cast<int32_t *>((*slot)->host.get());
  memcpy(h, a, n * sizeof(int32_t));
  if (b) memcpy(h + n, b, n * sizeof(int32_t));
  CUDA_TRY(cudaMemcpyAsync((*slot)->dev.get(), h, bytes, cudaMemcpyHostToDevice, stream));
  const int32_t *d = reinterpret_cast<const int32_t *>((*slot)->dev.get());
  *c = IdCall{{d, b ? d + n : nullptr}, n, dst_arg, true};
  return 0;
}

// Host checks of a device id list: everything the host sees without reading device memory.
static int check_dev_ids(const swb_engine *eng, const char *fn, const void *ids, int32_t id_dtype) {
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
    CUDA_TRY(cudaMemsetAsync(eng->d_id_claim.get(), 0xFF, (size_t)eng->st.E * sizeof(unsigned long long), stream));
    CUDA_TRY(cudaMemsetAsync(eng->d_id_fail.get(), 0xFF, sizeof(unsigned long long), stream));
    eng->id_seq = 1;
  }
  *c = IdCall{{a, b}, n, dst_arg, false, call, (unsigned long long)(~eng->id_seq) << 32, eng->d_id_claim.get(),
              eng->d_id_fail.get(), eng->d_id_status.get()};
  return 0;
}

static unsigned grid_of(size_t threads) { return (unsigned)((threads + 255) / 256); }

// The check kernels of device-checked ids `c`, enqueued before the kernels that use them: every id
// in range and, with kDistinct (ids that are destinations), none repeated.  Host-checked ids need none.
template <typename T, bool kDistinct>
static void enqueue_id_checks(swb_engine *eng, const IdCall &c, cudaStream_t stream) {
  if (c.host_checked) return;
  check_ids_kernel<T><<<grid_of(c.n), 256, 0, stream>>>(c, eng->st.E);
  if constexpr (kDistinct) repeat_ids_kernel<T><<<grid_of(c.n), 256, 0, stream>>>(c, eng->st.E);
  eng->launches += kDistinct ? 2 : 1;
}

// The kernels of a save, load or copy of the ids `c`, checked on the host or, by the check kernels
// enqueued first, on the device.
template <typename T>
static int enqueue_save(swb_engine *eng, const IdCall &c, void *dst, cudaStream_t stream) {
  enqueue_id_checks<T, false>(eng, c, stream);
  save_envs_kernel<T><<<grid_of((size_t)c.n * eng->st.S), 256, 0, stream>>>(
      eng->st, c, static_cast<unsigned char *>(dst), RecordLayout(eng->st.S, eng->st.G).bytes());
  eng->launches++;
  CUDA_TRY(cudaGetLastError());
  return 0;
}

template <typename T>
static int enqueue_load(swb_engine *eng, const IdCall &c, const void *src, cudaStream_t stream) {
  enqueue_id_checks<T, true>(eng, c, stream);
  load_envs_kernel<T><<<grid_of((size_t)c.n * eng->st.S), 256, 0, stream>>>(
      eng->st, c, static_cast<const unsigned char *>(src), RecordLayout(eng->st.S, eng->st.G).bytes());
  eng->launches++;
  CUDA_TRY(cudaGetLastError());
  return 0;
}

// `disjoint`: the host found no env among both sources and destinations, so one kernel copies.
// Otherwise every source is saved to engine scratch before any destination is written, so every
// read sees the state from before the call.
template <typename T>
static int enqueue_copy(swb_engine *eng, const IdCall &c, bool disjoint, cudaStream_t stream) {
  const size_t threads = (size_t)c.n * eng->st.S, rb = RecordLayout(eng->st.S, eng->st.G).bytes();
  if (disjoint) {
    copy_envs_kernel<<<grid_of(threads), 256, 0, stream>>>(eng->st, c);
    eng->launches++;
  } else {
    // an earlier copy on any stream may still read the scratch
    CUDA_TRY(eng->records.grow(c.n * rb, [] { return cudaDeviceSynchronize(); }));
    if (c.host_checked) {
      save_envs_kernel<T><<<grid_of(threads), 256, 0, stream>>>(eng->st, c, eng->records.get(), rb);
    } else {
      check_ids_kernel<T><<<grid_of(2 * (size_t)c.n), 256, 0, stream>>>(c, eng->st.E);
      stage_copy_dev_kernel<T><<<grid_of(threads), 256, 0, stream>>>(eng->st, c, eng->records.get(), rb);
      eng->launches++;
    }
    load_envs_kernel<T><<<grid_of(threads), 256, 0, stream>>>(eng->st, c, eng->records.get(), rb);
    eng->launches += 2;
  }
  CUDA_TRY(cudaGetLastError());
  return 0;
}

template <typename T>
static int enqueue_set_goals(swb_engine *eng, const IdCall &c, const double *goals, cudaStream_t stream) {
  enqueue_id_checks<T, true>(eng, c, stream);
  set_goals_kernel<T><<<grid_of((size_t)c.n * 2 * eng->st.G), 256, 0, stream>>>(eng->st, c, goals);
  eng->launches++;
  CUDA_TRY(cudaGetLastError());
  return 0;
}

// The ids of a save, load, copy or set_goals: host int32 arrays, or device arrays of `dtype`
// (SWB_DTYPE_I32 or SWB_DTYPE_I64).  ids[1] holds the destinations of a copy and is null otherwise.
struct EnvIds {
  const void *ids[2];
  bool host;
  int32_t dtype;
};

static EnvIds host_ids(const int32_t *a, const int32_t *b = nullptr) { return EnvIds{{a, b}, true, SWB_DTYPE_I32}; }
static EnvIds dev_ids(const void *a, const void *b, int32_t dtype) { return EnvIds{{a, b}, false, dtype}; }

// Checks the n ids of `call` (SWB_IDS_CALL_*), then calls enqueue(c, T(), disjoint) with their
// IdCall c and id type T.  Host ids: every id in [0, E) and the destinations distinct, checked before
// anything is enqueued; then staged, their slot's readers recorded after `enqueue`; `disjoint` says that
// no env is among both the sources and the destinations.  Device ids: check_dev_ids, then the next
// device-checked call (begin_id_call), whose kernels check them; `disjoint` is false.
template <typename Enqueue>
static int run_ids(swb_engine *eng, const char *fn, int call, const EnvIds &ids, int32_t n,
                   cudaStream_t stream, Enqueue enqueue) {
  const int n_args = ids.ids[1] ? 2 : 1;
  const int dst_arg = call == SWB_IDS_CALL_SAVE ? -1 : call == SWB_IDS_CALL_COPY ? 1 : 0;
  IdCall c;
  if (ids.host) {
    const int32_t *src = static_cast<const int32_t *>(ids.ids[0]), *dst = static_cast<const int32_t *>(ids.ids[1]);
    std::vector<uint8_t> mark(dst_arg >= 0 ? eng->st.E : 0, 0);
    if (dst_arg >= 0 && check_env_ids(eng, fn, dst_arg ? dst : src, n, &mark)) return 1;
    if (dst_arg != 0 && check_env_ids(eng, fn, src, n, nullptr)) return 1;  // argument 0 holds sources
    bool disjoint = true;
    for (int32_t i = 0; dst && i < n && disjoint; ++i) disjoint = !mark[src[i]];
    CUDA_TRY(cudaSetDevice(eng->device));
    StagingSlot *slot = nullptr;
    if (stage_ids(eng, src, dst, n, dst_arg, stream, &c, &slot) || enqueue(c, int32_t(), disjoint)) return 1;
    CUDA_TRY(slot->readers.record(stream));
    return 0;
  }
  for (int a = 0; a < n_args; ++a)
    if (check_dev_ids(eng, fn, ids.ids[a], ids.dtype)) return 1;
  CUDA_TRY(cudaSetDevice(eng->device));
  if (begin_id_call(eng, call, ids.ids[0], ids.ids[1], dst_arg, n, stream, &c)) return 1;
  return ids.dtype == SWB_DTYPE_I64 ? enqueue(c, int64_t(), false) : enqueue(c, int32_t(), false);
}

static int save_envs(swb_engine *eng, const char *fn, const EnvIds &ids, int32_t n, void *dst, uint64_t dst_bytes,
                     int32_t *span_class, cudaStream_t stream) {
  if (!eng || !span_class) return fail("%s: null argument", fn);
  if (check_record_args(eng, fn, SWB_IDS_CALL_SAVE, n, ids.ids[0], nullptr, dst, dst_bytes, 0)) return 1;
  *span_class = eng->max_spans;
  if (n == 0) return 0;
  return run_ids(eng, fn, SWB_IDS_CALL_SAVE, ids, n, stream, [&](const IdCall &c, auto id, bool) {
    return enqueue_save<decltype(id)>(eng, c, dst, stream);
  });
}

static int load_envs(swb_engine *eng, const char *fn, const EnvIds &ids, int32_t n, const void *src,
                     uint64_t src_bytes, int32_t span_class, cudaStream_t stream) {
  if (check_record_args(eng, fn, SWB_IDS_CALL_LOAD, n, ids.ids[0], nullptr, src, src_bytes, span_class)) return 1;
  if (n == 0) return 0;
  return run_ids(eng, fn, SWB_IDS_CALL_LOAD, ids, n, stream, [&](const IdCall &c, auto id, bool) {
    // records of stars or spokes need the concave span tables, as if their scenes were uploaded
    eng->max_spans = std::max(eng->max_spans, (int)span_class);
    return enqueue_load<decltype(id)>(eng, c, src, stream);
  });
}

static int copy_envs(swb_engine *eng, const char *fn, const EnvIds &ids, int32_t n, cudaStream_t stream) {
  if (check_record_args(eng, fn, SWB_IDS_CALL_COPY, n, ids.ids[0], ids.ids[1], nullptr, 0, 0)) return 1;
  if (n == 0) return 0;
  return run_ids(eng, fn, SWB_IDS_CALL_COPY, ids, n, stream, [&](const IdCall &c, auto id, bool disjoint) {
    return enqueue_copy<decltype(id)>(eng, c, disjoint, stream);
  });
}

static int set_goals(swb_engine *eng, const char *fn, const EnvIds &ids, int32_t n, const double *goals,
                     cudaStream_t stream) {
  if (!eng) return fail("%s: null engine", fn);
  if (!eng->st.G) return fail("%s: the task tree samples no goals (G = 0)", fn);
  if (n < 0) return fail("%s: n = %d", fn, n);
  if (n == 0) return 0;
  if (!ids.ids[0] || !goals) return fail("%s: null argument", fn);
  if (reinterpret_cast<uintptr_t>(goals) % 8) return fail("%s: goals are not 8-byte aligned", fn);
  return run_ids(eng, fn, SWB_IDS_CALL_SET_GOALS, ids, n, stream, [&](const IdCall &c, auto id, bool) {
    return enqueue_set_goals<decltype(id)>(eng, c, goals, stream);
  });
}

// The rows a read-only record call reads: n >= 0 records in fn's record buffer `name`, or, where
// the call takes them (live_ok), the E live envs for records == NULL, and then n == E.
static int check_rows(const swb_engine *eng, const char *fn, const char *name, const void *records, int32_t n,
                      uint64_t records_bytes, bool live_ok) {
  if (!eng) return fail("%s: null engine", fn);
  if (n < 0) return fail("%s: n = %d", fn, n);
  if (records) return check_record_buffer(eng, fn, name, records, records_bytes, n);
  if (!live_ok) return fail("%s: null %s", fn, name);
  if (n != eng->st.E) return fail("%s: n = %d must be E = %d when the rows are the live envs", fn, n, eng->st.E);
  return 0;
}

// `bytes` bytes at `ptr`, which hold elements aligned to `align` bytes.
struct Span {
  const char *name;
  const void *ptr;
  uint64_t bytes;
  unsigned align;
};

static bool overlap(const Span &a, const Span &b) {
  const uint64_t a0 = reinterpret_cast<uintptr_t>(a.ptr), b0 = reinterpret_cast<uintptr_t>(b.ptr);
  return a0 < b0 + b.bytes && b0 < a0 + a.bytes;
}

// The outputs outs[0 .. n_outs) of a read-only record call: each set, aligned to its elements, and
// disjoint from every other output and from the rows it reads (rows.ptr NULL: the live envs).  An
// output that overlaps the rows would race with the kernel's reads of them.
static int check_outputs(const char *fn, const Span *outs, int n_outs, const Span &rows) {
  for (int i = 0; i < n_outs; ++i) {
    const Span &o = outs[i];
    if (!o.ptr) return fail("%s: null output %s", fn, o.name);
    if (reinterpret_cast<uintptr_t>(o.ptr) % o.align) return fail("%s: %s is not %u-byte aligned", fn, o.name, o.align);
    for (int j = 0; j < i; ++j)
      if (overlap(o, outs[j])) return fail("%s: %s overlaps %s", fn, o.name, outs[j].name);
    if (rows.ptr && overlap(o, rows)) return fail("%s: %s overlaps %s", fn, o.name, rows.name);
  }
  return 0;
}

// swb_render_masks, swb_render_coverage, swb_render_soft_masks and swb_render_boxes: the image sizes
// first (soft masks: aa <= 15), then the rows, then the grid of n rows of bands, then the outputs --
// `out`, the per-pixel output of the mode (none for MASK_BOX), MASK_BOX's two boxes, and for
// MASK_COVER and MASK_BOX the counts.  Counts and boxes are zeroed on the stream before the launch,
// and MASK_BOX's boxes are decoded by a second launch after it.
template <MaskMode kMode>
static int render_mask_call(swb_engine *eng, const char *fn, int32_t width, int32_t height, int32_t anti_aliasing,
                            const void *records, int32_t n, uint64_t records_bytes, void *out, int32_t *visible,
                            int32_t *area, int32_t *visible_box, int32_t *amodal_box, cudaStream_t stream) {
  constexpr bool counted = kMode == MASK_COVER || kMode == MASK_BOX;
  if (width < 1 || height < 1 || anti_aliasing < 1)
    return fail("%s: width %d, height %d and anti_aliasing %d must be >= 1", fn, width, height, anti_aliasing);
  if (kMode == MASK_SOFT && anti_aliasing > MK_SOFT_MAX_AA)
    return fail("%s: anti_aliasing %d exceeds %d: a pixel's anti_aliasing^2 sample count must fit a uint8", fn,
                anti_aliasing, MK_SOFT_MAX_AA);
  if ((int64_t)anti_aliasing * width > 4095 || (int64_t)anti_aliasing * height > 4095)
    return fail("%s: canvas %lld x %lld exceeds 4095 pixels per side", fn, (long long)anti_aliasing * width,
                (long long)anti_aliasing * height);
  if (check_rows(eng, fn, "records", records, n, records_bytes, true)) return 1;
  const MaskLayout L(eng->st.S, width, height, anti_aliasing, kMode);
  if ((int64_t)n * L.n_bands > INT32_MAX)
    return fail("%s: n = %d rows of %d bands each exceed 2^31 - 1 CTAs", fn, n, L.n_bands);
  const uint64_t rb = RecordLayout(eng->st.S, eng->st.G).bytes();
  // `out` holds a byte per pixel, a 4-byte word per pixel (MASK_COVER) or a byte per pixel and slot (MASK_SOFT)
  const char *name = kMode == MASK_LABEL ? "masks" : kMode == MASK_COVER ? "cover" : "soft";
  const unsigned px = kMode == MASK_COVER ? 4 : 1;
  const uint64_t bytes = (uint64_t)n * height * width * px * (kMode == MASK_SOFT ? eng->st.S : 1);
  const uint64_t counts = (uint64_t)n * eng->st.S * 4, boxes = 4 * counts;
  Span outs[4];
  int n_outs = 0;
  if (kMode == MASK_BOX) {
    outs[n_outs++] = {"visible_box", visible_box, boxes, 4};
    outs[n_outs++] = {"amodal_box", amodal_box, boxes, 4};
  } else {
    outs[n_outs++] = {name, out, bytes, px};
  }
  if (counted) {
    outs[n_outs++] = {"visible", visible, counts, 4};
    outs[n_outs++] = {"area", area, counts, 4};
  }
  if (check_outputs(fn, outs, n_outs, Span{"the records", records, n * rb, 16})) return 1;
  if (n == 0) return 0;
  CUDA_TRY(cudaSetDevice(eng->device));
  auto kernel = records ? mask_kernel<true, kMode> : mask_kernel<false, kMode>;
  CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, L.total));
  if (counted) {
    CUDA_TRY(cudaMemsetAsync(visible, 0, (size_t)counts, stream));
    CUDA_TRY(cudaMemsetAsync(area, 0, (size_t)counts, stream));
  }
  if (kMode == MASK_BOX) {
    CUDA_TRY(cudaMemsetAsync(visible_box, 0, (size_t)boxes, stream));
    CUDA_TRY(cudaMemsetAsync(amodal_box, 0, (size_t)boxes, stream));
  }
  kernel<<<(unsigned)((int64_t)n * L.n_bands), MK_THREADS, L.total, stream>>>(
      eng->st, L, static_cast<uint8_t *>(out), RenderRecords{static_cast<const unsigned char *>(records), (size_t)rb},
      CoverCounts{visible, area, visible_box, amodal_box});
  eng->launches++;
  CUDA_TRY(cudaGetLastError());
  if (kMode == MASK_BOX) {
    const size_t n_boxes = (size_t)n * eng->st.S;
    box_finish_kernel<<<(unsigned)((2 * n_boxes + BOX_FINISH_THREADS - 1) / BOX_FINISH_THREADS),
                        BOX_FINISH_THREADS, 0, stream>>>(visible_box, amodal_box, n_boxes);
    eng->launches++;
    CUDA_TRY(cudaGetLastError());
  }
  return 0;
}

extern "C" {

int64_t swb_env_record_bytes(const swb_engine *eng) {
  if (!eng) {
    fail("swb_env_record_bytes: null engine");
    return -1;
  }
  return (int64_t)RecordLayout(eng->st.S, eng->st.G).bytes();
}

int swb_save_envs(swb_engine *eng, const int32_t *env_ids, int32_t n, void *dst, uint64_t dst_bytes,
                  int32_t *span_class, void *stream) {
  return save_envs(eng, "swb_save_envs", host_ids(env_ids), n, dst, dst_bytes, span_class,
                   static_cast<cudaStream_t>(stream));
}

int swb_save_envs_dev(swb_engine *eng, const void *env_ids, int32_t id_dtype, int32_t n, void *dst,
                      uint64_t dst_bytes, int32_t *span_class, void *stream) {
  return save_envs(eng, "swb_save_envs_dev", dev_ids(env_ids, nullptr, id_dtype), n, dst, dst_bytes, span_class,
                   static_cast<cudaStream_t>(stream));
}

int swb_load_envs(swb_engine *eng, const int32_t *env_ids, int32_t n, const void *src, uint64_t src_bytes,
                  int32_t span_class, void *stream) {
  return load_envs(eng, "swb_load_envs", host_ids(env_ids), n, src, src_bytes, span_class,
                   static_cast<cudaStream_t>(stream));
}

int swb_load_envs_dev(swb_engine *eng, const void *env_ids, int32_t id_dtype, int32_t n, const void *src,
                      uint64_t src_bytes, int32_t span_class, void *stream) {
  return load_envs(eng, "swb_load_envs_dev", dev_ids(env_ids, nullptr, id_dtype), n, src, src_bytes, span_class,
                   static_cast<cudaStream_t>(stream));
}

int swb_copy_envs(swb_engine *eng, const int32_t *src_ids, const int32_t *dst_ids, int32_t n, void *stream) {
  return copy_envs(eng, "swb_copy_envs", host_ids(src_ids, dst_ids), n, static_cast<cudaStream_t>(stream));
}

int swb_copy_envs_dev(swb_engine *eng, const void *src_ids, const void *dst_ids, int32_t id_dtype, int32_t n,
                      void *stream) {
  return copy_envs(eng, "swb_copy_envs_dev", dev_ids(src_ids, dst_ids, id_dtype), n,
                   static_cast<cudaStream_t>(stream));
}

int swb_pool_goal_pointer(swb_engine *eng, double **goal, int32_t *n_goals) {
  if (!eng || !goal || !n_goals) return fail("swb_pool_goal_pointer: null argument");
  *goal = eng->st.p_goal;
  *n_goals = eng->st.G;
  return 0;
}

int swb_set_goals(swb_engine *eng, const int32_t *env_ids, int32_t n, const double *goals, void *stream) {
  return set_goals(eng, "swb_set_goals", host_ids(env_ids), n, goals, static_cast<cudaStream_t>(stream));
}

int swb_set_goals_dev(swb_engine *eng, const void *env_ids, int32_t id_dtype, int32_t n, const double *goals,
                      void *stream) {
  return set_goals(eng, "swb_set_goals_dev", dev_ids(env_ids, nullptr, id_dtype), n, goals,
                   static_cast<cudaStream_t>(stream));
}

int swb_evaluate_states(swb_engine *eng, const void *records, int32_t n, uint64_t records_bytes,
                        const double *goals, double *reward, uint8_t *success, uint8_t *status, void *stream_) {
  static const char fn[] = "swb_evaluate_states";
  if (check_rows(eng, fn, "records", records, n, records_bytes, false)) return 1;
  if (goals && !eng->st.G) return fail("%s: goals given, but the task tree samples no goals (G = 0)", fn);
  if (n == 0) return 0;
  if (reinterpret_cast<uintptr_t>(goals) % 8) return fail("%s: goals are not 8-byte aligned", fn);
  const uint64_t rb = RecordLayout(eng->st.S, eng->st.G).bytes();
  const Span outs[] = {{"reward", reward, 8 * (uint64_t)n, 8}, {"success", success, (uint64_t)n, 1},
                       {"status", status, (uint64_t)n, 1}};
  if (check_outputs(fn, outs, 3, Span{"the records", records, n * rb, 16})) return 1;
  CUDA_TRY(cudaSetDevice(eng->device));
  const unsigned blocks = (unsigned)(((int64_t)n + ROLLOUT_WARPS - 1) / ROLLOUT_WARPS);
  evaluate_kernel<<<blocks, ROLLOUT_WARPS * 32, 0, static_cast<cudaStream_t>(stream_)>>>(
      eng->st, eng->d_step_cfg.get(), static_cast<const unsigned char *>(records), (size_t)rb, n, goals, reward,
      success, status);
  eng->launches++;
  CUDA_TRY(cudaGetLastError());
  return 0;
}

}  // extern "C"

// swb_rollout_states and swb_rollout_trajectory: the rollout, roots and output checks, then one
// launch.  `records` are the leaves (NULL: none), or with `trajectory` the n_steps records of
// every plan, which the call requires.
static int rollout_records_call(swb_engine *eng, const char *fn, const void *roots, int32_t n_roots,
                                uint64_t roots_bytes, const void *actions, int32_t action_dtype, int32_t n_steps,
                                int32_t n_candidates, const swb_step_out *out, void *records,
                                uint64_t records_bytes, int32_t *span_class, cudaStream_t stream,
                                bool trajectory) {
  const char *name = trajectory ? "records" : "leaves";
  if (!eng) return fail("%s: null engine", fn);
  if (roots ? n_roots < 1 : n_roots != eng->st.E)
    return roots ? fail("%s: n_roots = %d must be >= 1", fn, n_roots)
                 : fail("%s: n_roots = %d must be E = %d when the roots are the live envs", fn, n_roots,
                        eng->st.E);
  if (check_rollout(eng, fn, roots ? "roots" : "envs", actions, action_dtype, n_steps, n_candidates, n_roots,
                    out) ||
      check_rows(eng, fn, "roots", roots, n_roots, roots_bytes, true))
    return 1;
  if (trajectory && !records) return fail("%s: null output records", fn);
  const uint64_t rb = RecordLayout(eng->st.S, eng->st.G).bytes();
  const uint64_t plans = (uint64_t)n_roots * n_candidates, entries = plans * n_steps;
  const uint64_t n_records = trajectory ? entries : plans;
  if (records && check_record_buffer(eng, fn, name, records, records_bytes, (int64_t)n_records)) return 1;
  const Span outs[] = {{"reward", out->reward, 8 * entries, 8}, {"step_type", out->step_type, entries, 1},
                       {"success", out->success, entries, 1}, {"status", out->status, entries, 1},
                       {name, records, n_records * rb, 16}};
  if (check_outputs(fn, outs, records ? 5 : 4, Span{"the roots", roots, n_roots * rb, 16})) return 1;
  if (!roots && span_class) *span_class = eng->max_spans;
  return enqueue_rollout(eng, actions, action_dtype, n_steps, n_candidates, *out,
                         RolloutRecords{static_cast<const unsigned char *>(roots),
                                        static_cast<unsigned char *>(records), (size_t)rb, n_roots},
                         stream, trajectory);
}

extern "C" {

int swb_rollout_states(swb_engine *eng, const void *roots, int32_t n_roots, uint64_t roots_bytes,
                       const void *actions, int32_t action_dtype, int32_t n_steps, int32_t n_candidates,
                       const swb_step_out *out, void *leaves, uint64_t leaves_bytes, int32_t *span_class,
                       void *stream) {
  return rollout_records_call(eng, "swb_rollout_states", roots, n_roots, roots_bytes, actions, action_dtype,
                              n_steps, n_candidates, out, leaves, leaves_bytes, span_class,
                              static_cast<cudaStream_t>(stream), false);
}

int swb_rollout_trajectory(swb_engine *eng, const void *roots, int32_t n_roots, uint64_t roots_bytes,
                           const void *actions, int32_t action_dtype, int32_t n_steps, int32_t n_candidates,
                           const swb_step_out *out, void *records, uint64_t records_bytes, int32_t *span_class,
                           void *stream) {
  return rollout_records_call(eng, "swb_rollout_trajectory", roots, n_roots, roots_bytes, actions, action_dtype,
                              n_steps, n_candidates, out, records, records_bytes, span_class,
                              static_cast<cudaStream_t>(stream), true);
}

int swb_render_states(swb_engine *eng, swb_raster *r, const void *records, int32_t n, uint64_t records_bytes,
                      int32_t span_class, uint8_t *frames, uint8_t *status, void *stream_) {
  static const char fn[] = "swb_render_states";
  if (!eng || !r) return fail("%s: null engine or raster", fn);
  if (n == 0) return 0;  // nothing is read or drawn: the buffers may be null
  if (check_rows(eng, fn, "records", records, n, records_bytes, false)) return 1;
  if (span_class != 1 && span_class != 4) return fail("%s: span_class must be 1 or 4, got %d", fn, span_class);
  const RasterDev &rd = r->rd;
  // n_items and the kernel's item index are int
  if ((int64_t)n * rd.n_bands > INT32_MAX)
    return fail("%s: n = %d records of %d bands each exceed 2^31 - 1 render items", fn, n, rd.n_bands);
  const uint64_t rb = RecordLayout(eng->st.S, eng->st.G).bytes();
  const Span outs[] = {{"frames", frames, (uint64_t)n * rd.H * rd.W * 3, 1}, {"status", status, (uint64_t)n, 1}};
  if (check_outputs(fn, outs, 2, Span{"the records", records, n * rb, 16})) return 1;
  // read-only: records of stars or spokes get the concave span tables for this launch only
  std::optional<RenderLayout> plan;
  if (check_render(eng, r, std::max(eng->max_spans, (int)span_class), &plan)) return 1;
  CUDA_TRY(cudaSetDevice(eng->device));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  CUDA_TRY(cudaMemsetAsync(status, 0, (size_t)n, stream));
  return enqueue_render(eng, r, *plan, RenderTargets{{frames}, 1, 0, 0}, status, stream, 0, n, false,
                        RenderRecords{static_cast<const unsigned char *>(records), (size_t)rb});
}

// swb_render_windows (draw NULL: every slot drawn) and swb_render_views (draw [n][n_views][S]).
static int render_views_call(const char *fn, swb_engine *eng, swb_raster *r, const void *records, int32_t n,
                             uint64_t records_bytes, int32_t span_class, const double *windows,
                             const uint8_t *draw, int32_t n_views, uint8_t *frames, uint8_t *status,
                             void *stream_) {
  if (!eng || !r) return fail("%s: null engine or raster", fn);
  if (check_rows(eng, fn, "records", records, n, records_bytes, true)) return 1;
  if (span_class != 1 && span_class != 4) return fail("%s: span_class must be 1 or 4, got %d", fn, span_class);
  if (n_views < 1) return fail("%s: n_views = %d must be >= 1", fn, n_views);
  const RasterDev &rd = r->rd;
  // n_items and the kernel's item index are int
  if ((int64_t)n * n_views * rd.n_bands > INT32_MAX)
    return fail("%s: n = %d rows of %d views of %d bands each exceed 2^31 - 1 render items", fn, n, n_views,
                rd.n_bands);
  if (n == 0) return 0;
  if (!windows) return fail("%s: null windows", fn);
  if (reinterpret_cast<uintptr_t>(windows) % 8) return fail("%s: windows are not 8-byte aligned", fn);
  const uint64_t rb = RecordLayout(eng->st.S, eng->st.G).bytes(), items = (uint64_t)n * n_views;
  const Span outs[] = {{"frames", frames, items * rd.H * rd.W * 3, 1}, {"status", status, items, 1},
                       {"windows", windows, items * 32, 8}};
  if (check_outputs(fn, outs, 3, Span{"the records", records, records ? n * rb : 0, 16})) return 1;
  if (draw) {  // read-only like the windows and records: only the outputs may not overlap it
    const Span d{"draw", draw, items * eng->st.S, 1};
    for (int i = 0; i < 2; ++i)
      if (overlap(d, outs[i])) return fail("%s: draw overlaps %s", fn, outs[i].name);
  }
  std::optional<RenderLayout> plan;
  if (check_render(eng, r, std::max(eng->max_spans, (int)span_class), &plan)) return 1;
  CUDA_TRY(cudaSetDevice(eng->device));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  CUDA_TRY(cudaMemsetAsync(status, 0, (size_t)items, stream));
  return enqueue_render(eng, r, *plan, RenderTargets{{frames}, 1, 0, 0}, status, stream, 0, n, false,
                        RenderRecords{static_cast<const unsigned char *>(records), (size_t)rb},
                        RenderWindows{windows, n_views, draw});
}

int swb_render_windows(swb_engine *eng, swb_raster *r, const void *records, int32_t n, uint64_t records_bytes,
                       int32_t span_class, const double *windows, int32_t n_views, uint8_t *frames,
                       uint8_t *status, void *stream) {
  return render_views_call("swb_render_windows", eng, r, records, n, records_bytes, span_class, windows, nullptr,
                           n_views, frames, status, stream);
}

int swb_render_views(swb_engine *eng, swb_raster *r, const void *records, int32_t n, uint64_t records_bytes,
                     int32_t span_class, const double *windows, const uint8_t *draw, int32_t n_views,
                     uint8_t *frames, uint8_t *status, void *stream) {
  if (!draw) return fail("swb_render_views: null draw");
  return render_views_call("swb_render_views", eng, r, records, n, records_bytes, span_class, windows, draw,
                           n_views, frames, status, stream);
}

int swb_render_masks(swb_engine *eng, int32_t width, int32_t height, int32_t anti_aliasing,
                     const void *records, int32_t n, uint64_t records_bytes, uint8_t *masks, void *stream) {
  return render_mask_call<MASK_LABEL>(eng, "swb_render_masks", width, height, anti_aliasing, records, n,
                                      records_bytes, masks, nullptr, nullptr, nullptr, nullptr,
                                      static_cast<cudaStream_t>(stream));
}

int swb_render_coverage(swb_engine *eng, int32_t width, int32_t height, int32_t anti_aliasing,
                        const void *records, int32_t n, uint64_t records_bytes, int32_t *cover,
                        int32_t *visible, int32_t *area, void *stream) {
  return render_mask_call<MASK_COVER>(eng, "swb_render_coverage", width, height, anti_aliasing, records, n,
                                      records_bytes, cover, visible, area, nullptr, nullptr,
                                      static_cast<cudaStream_t>(stream));
}

int swb_render_soft_masks(swb_engine *eng, int32_t width, int32_t height, int32_t anti_aliasing,
                          const void *records, int32_t n, uint64_t records_bytes, uint8_t *soft, void *stream) {
  return render_mask_call<MASK_SOFT>(eng, "swb_render_soft_masks", width, height, anti_aliasing, records, n,
                                     records_bytes, soft, nullptr, nullptr, nullptr, nullptr,
                                     static_cast<cudaStream_t>(stream));
}

int swb_render_boxes(swb_engine *eng, int32_t width, int32_t height, int32_t anti_aliasing,
                     const void *records, int32_t n, uint64_t records_bytes, int32_t *visible_box,
                     int32_t *amodal_box, int32_t *visible, int32_t *area, void *stream) {
  return render_mask_call<MASK_BOX>(eng, "swb_render_boxes", width, height, anti_aliasing, records, n,
                                    records_bytes, nullptr, visible, area, visible_box, amodal_box,
                                    static_cast<cudaStream_t>(stream));
}

int swb_sample_contained(swb_engine *eng, const void *records, int32_t n, uint64_t records_bytes,
                         int32_t n_samples, uint64_t seed, double *position, int8_t *slot, uint8_t *status,
                         void *stream_) {
  static const char fn[] = "swb_sample_contained";
  if (check_rows(eng, fn, "records", records, n, records_bytes, true)) return 1;
  if (n_samples < 1) return fail("%s: n_samples = %d must be >= 1", fn, n_samples);
  // the kernel's thread index and the output arrays' entries are one per (row, sample)
  if ((int64_t)n * n_samples > INT32_MAX)
    return fail("%s: n = %d rows of %d samples exceed 2^31 - 1 samples", fn, n, n_samples);
  if (n == 0) return 0;
  const uint64_t rb = RecordLayout(eng->st.S, eng->st.G).bytes(), total = (uint64_t)n * n_samples;
  const Span outs[] = {{"position", position, 16 * total, 8}, {"slot", slot, total, 1},
                       {"status", status, total, 1}};
  if (check_outputs(fn, outs, 3, Span{"the records", records, n * rb, 16})) return 1;
  CUDA_TRY(cudaSetDevice(eng->device));
  auto kernel = records ? contained_kernel<true> : contained_kernel<false>;
  kernel<<<(unsigned)((total + CT_THREADS - 1) / CT_THREADS), CT_THREADS, 0, static_cast<cudaStream_t>(stream_)>>>(
      eng->st, static_cast<const unsigned char *>(records), (size_t)rb, n, n_samples, seed, position, slot,
      status);
  eng->launches++;
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int swb_env_ids_status_pointer(swb_engine *eng, swb_ids_status **status) {
  if (!eng || !status) return fail("swb_env_ids_status_pointer: null argument");
  *status = eng->d_id_status.get();
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
  double goal[2 * SWB_MAX_GOALS];
  const int bad = swb_sampler::sample_and_pack(
      *prog, seed, (uint64_t)g, (uint64_t)a, S, sc, goal,
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
  if (out.goal)
    for (int j = 0; j < 2 * prog->n_goals; ++j) out.goal[(size_t)i * 2 * prog->n_goals + j] = goal[j];
  if (bad >= 0) sampler_fail(status, bad, g, a);
}

// swb_refill_device: one thread per env, scenes refilled_upto + 1 .. scene_serial + K - 1 into the
// ring.  The scene the env is on (ring slot serial % K) is never among them.
__global__ void refill_device_kernel(const swb_scene_program *__restrict__ prog, uint64_t seed,
                                     int64_t env_offset, DevState st, int64_t *refilled_upto,
                                     swb_sampler_status *status) {
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
    double goal[2 * SWB_MAX_GOALS];
    const int bad = swb_sampler::sample_and_pack(
        *prog, seed, (uint64_t)g, (uint64_t)a, st.S, sc, goal,
        [&](int slot, const swb_sampler::Packed &o, const swb_sampler::Sprite *) {
          const size_t d = base + slot;
          st.p_x[d] = o.x; st.p_y[d] = o.y;
          st.p_m00[d] = o.m00; st.p_m01[d] = o.m01; st.p_m10[d] = o.m10; st.p_m11[d] = o.m11;
          st.p_vx[d] = o.vx; st.p_vy[d] = o.vy;
          st.p_member[d] = o.member; st.p_shape[d] = o.shape; st.p_pos_f32[d] = o.pos_f32;
          st.p_rgb[d] = (uint32_t)o.rgb[0] | ((uint32_t)o.rgb[1] << 8) | ((uint32_t)o.rgb[2] << 16);
          for (int f = 0; f < 5; ++f) st.p_factors[d * 5 + f] = o.factors[f];
        });
    const size_t gb = ((size_t)e * st.K + (size_t)(a % st.K)) * st.G * 2;
    for (int j = 0; j < 2 * st.G; ++j) st.p_goal[gb + j] = goal[j];
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
  if (p.n_goals < 0 || p.n_goals > SWB_MAX_GOALS) return fail("program: n_goals %d out of range", p.n_goals);
  for (int i = 0; i < p.n_goals; ++i)
    if (!pc_ok(p.goal_pc[i])) return fail("program: goal %d has no code", i);
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
  if (prog->n_goals != eng->st.G)
    return fail("swb_sampler_load: the program draws %d goals per scene, the task tree has %d goal slots",
                prog->n_goals, eng->st.G);
  CUDA_TRY(cudaSetDevice(eng->device));
  // a first load publishes the sampler once its program is on the device
  std::unique_ptr<SamplerDev> fresh;
  if (!eng->sampler) {
    fresh = std::make_unique<SamplerDev>();
    if (dev_alloc(&fresh->prog, 1) != cudaSuccess || dev_alloc(&fresh->refilled_upto, eng->st.E) != cudaSuccess ||
        dev_alloc(&fresh->status, 1) != cudaSuccess)
      return fail("swb_sampler_load: device allocation failed");
  }
  const SamplerDev &s = fresh ? *fresh : *eng->sampler;
  CUDA_TRY(cudaDeviceSynchronize());
  CUDA_TRY(cudaMemcpy(s.prog.get(), prog, sizeof(swb_scene_program), cudaMemcpyHostToDevice));
  CUDA_TRY(cudaMemset(s.refilled_upto.get(), 0xFF, (size_t)eng->st.E * sizeof(int64_t)));
  if (fresh) eng->sampler = std::move(fresh);
  eng->seed = seed;
  eng->env_offset = env_offset;
  return 0;
}

int swb_sample_scenes(swb_engine *eng, const int64_t *env_ids, const int64_t *scene_idx, int32_t n,
                      const swb_sample_out *out, void *stream_) {
  if (!eng || !out) return fail("swb_sample_scenes: null argument");
  if (!eng->sampler) return fail("swb_sample_scenes: no program (swb_sampler_load)");
  if (n < 0) return fail("swb_sample_scenes: n < 0");
  if (n == 0) return 0;
  if (!env_ids || !scene_idx || !out->x || !out->y || !out->m00 || !out->m01 || !out->m10 || !out->m11 ||
      !out->vx || !out->vy || !out->member || !out->shape || !out->pos_f32 || !out->rgb || !out->factors ||
      !out->factor_value || !out->factor_kind)
    return fail("swb_sample_scenes: every pointer must be set");
  CUDA_TRY(cudaSetDevice(eng->device));
  const int threads = 128;
  sample_scenes_kernel<<<(n + threads - 1) / threads, threads, 0, static_cast<cudaStream_t>(stream_)>>>(
      eng->sampler->prog.get(), eng->seed, eng->st.S, env_ids, scene_idx, n, *out, eng->sampler->status.get());
  eng->launches++;
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int swb_refill_device(swb_engine *eng, void *stream_) {
  if (!eng) return fail("swb_refill_device: null engine");
  if (!eng->sampler) return fail("swb_refill_device: no program (swb_sampler_load)");
  CUDA_TRY(cudaSetDevice(eng->device));
  const int threads = 64;
  const SamplerDev &s = *eng->sampler;
  refill_device_kernel<<<(eng->st.E + threads - 1) / threads, threads, 0, static_cast<cudaStream_t>(stream_)>>>(
      s.prog.get(), eng->seed, eng->env_offset, eng->st, s.refilled_upto.get(), s.status.get());
  eng->launches++;
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int swb_sampler_pointers(swb_engine *eng, int64_t **refilled_upto, swb_sampler_status **status) {
  if (!eng) return fail("swb_sampler_pointers: null engine");
  if (!eng->sampler) return fail("swb_sampler_pointers: no program (swb_sampler_load)");
  if (refilled_upto) *refilled_upto = eng->sampler->refilled_upto.get();
  if (status) *status = eng->sampler->status.get();
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

int swb_packer_load(swb_engine *eng, const swb_scene_program *prog) {
  static const char fn[] = "swb_packer_load";
  if (!eng || !prog) return fail("%s: null argument", fn);
  if (check_program(*prog, eng->st.S)) return 1;
  if (prog->color_mode != SWB_COLOR_RGB && prog->color_mode != SWB_COLOR_HSV)
    return fail("%s: color_mode %d is neither SWB_COLOR_RGB nor SWB_COLOR_HSV", fn, prog->color_mode);
  // make_states_kernel looks up only angles it has checked to be integers in [-360, 360]
  auto has = [&](double a) {
    for (int i = 0; i < prog->n_angles; ++i)
      if (prog->angle[i] == a && std::signbit(prog->angle[i]) == std::signbit(a)) return true;
    return false;
  };
  if (!has(-0.0)) return fail("%s: the angle table lacks -0.0", fn);
  for (int a = -360; a <= 360; ++a)
    if (!has((double)a)) return fail("%s: the angle table lacks %d", fn, a);
  CUDA_TRY(cudaSetDevice(eng->device));
  // a first load publishes the packer once it is on the device
  DevPtr<swb_scene_program> fresh;
  if (!eng->d_packer && dev_alloc(&fresh, 1) != cudaSuccess) return fail("%s: device allocation failed", fn);
  CUDA_TRY(cudaDeviceSynchronize());  // a make_states call in flight may still read the old packer
  CUDA_TRY(cudaMemcpy(fresh ? fresh.get() : eng->d_packer.get(), prog, sizeof(swb_scene_program),
                      cudaMemcpyHostToDevice));
  if (fresh) eng->d_packer = std::move(fresh);
  eng->packer_hsv = prog->color_mode == SWB_COLOR_HSV;
  return 0;
}

int swb_make_states(swb_engine *eng, const swb_factor_columns *cols, int32_t n, const double *goals,
                    const int32_t *step_count, void *records, uint64_t records_bytes, uint8_t *status,
                    uint8_t *span_flag, void *stream_) {
  static const char fn[] = "swb_make_states";
  static const char *const names[swb_sampler::kFactors] = {"x", "y", "shape", "angle", "scale",
                                                          "c0", "c1", "c2", "x_vel", "y_vel"};
  if (!eng) return fail("%s: null engine", fn);
  if (!eng->d_packer) return fail("%s: no packer (swb_packer_load)", fn);
  if (n < 0) return fail("%s: n = %d", fn, n);
  if (!cols) return fail("%s: null cols", fn);
  if (!cols->col[swb_sampler::F_SHAPE]) return fail("%s: the shape column is required", fn);
  const int S = eng->st.S, G = eng->st.G;
  const uint64_t cells = (uint64_t)n * S;
  Span ins[swb_sampler::kFactors + 2];
  int n_ins = 0;
  for (int f = 0; f < swb_sampler::kFactors; ++f) {
    if (!cols->col[f]) continue;
    unsigned size = 0;
    switch (cols->kind[f]) {
      case SWB_FT_F64: case SWB_FT_I64: size = 8; break;
      case SWB_FT_F32: case SWB_FT_I32: size = 4; break;
      case SWB_FT_I16: size = 2; break;
      case SWB_FT_I8: case SWB_FT_U8: size = 1; break;
      default: return fail("%s: column %s has kind %d: not SWB_FT_F32, F64, I8, I16, I32, I64 or U8", fn,
                           names[f], cols->kind[f]);
    }
    if (reinterpret_cast<uintptr_t>(cols->col[f]) % size)
      return fail("%s: column %s is not %u-byte aligned", fn, names[f], size);
    ins[n_ins++] = Span{names[f], cols->col[f], cells * size, size};
  }
  // hsv_to_rgb takes the triple in one dtype (the device sampler refuses the same mixes)
  if (eng->packer_hsv) {
    auto color_kind = [&](int f) { return cols->col[f] ? cols->kind[f] : (int)SWB_FT_NONE; };
    const int k0 = color_kind(swb_sampler::F_C0);
    if (k0 != color_kind(swb_sampler::F_C1) || k0 != color_kind(swb_sampler::F_C2) ||
        (k0 != SWB_FT_NONE && k0 != SWB_FT_F32 && k0 != SWB_FT_F64))
      return fail("%s: under hsv_to_rgb the colour columns c0, c1, c2 must be all float32, all float64 or all "
                  "omitted, got kinds %d, %d, %d", fn, k0, color_kind(swb_sampler::F_C1),
                  color_kind(swb_sampler::F_C2));
  }
  if (G ? !goals : goals != nullptr)
    return G ? fail("%s: the task tree samples %d goals per scene: goals are required", fn, G)
             : fail("%s: goals given, but the task tree samples no goals (G = 0)", fn);
  if (reinterpret_cast<uintptr_t>(goals) % 8) return fail("%s: goals are not 8-byte aligned", fn);
  if (reinterpret_cast<uintptr_t>(step_count) % 4) return fail("%s: step_count is not 4-byte aligned", fn);
  if (goals) ins[n_ins++] = Span{"goals", goals, (uint64_t)n * G * 16, 8};
  if (step_count) ins[n_ins++] = Span{"step_count", step_count, (uint64_t)n * 4, 4};
  if (!records) return fail("%s: null records", fn);
  if (check_record_buffer(eng, fn, "records", records, records_bytes, n)) return 1;
  const uint64_t rb = RecordLayout(S, G).bytes();
  Span outs[3] = {{"records", records, n * rb, 16}, {"status", status, (uint64_t)n, 1}};
  const int n_outs = span_flag ? 3 : 2;
  if (span_flag) outs[2] = Span{"span_flag", span_flag, 1, 1};
  if (check_outputs(fn, outs, n_outs, Span{nullptr, nullptr, 0, 1})) return 1;
  for (int i = 0; i < n_outs; ++i)
    for (int k = 0; k < n_ins; ++k)
      if (overlap(outs[i], ins[k])) return fail("%s: %s overlaps %s", fn, outs[i].name, ins[k].name);
  if (n == 0) return 0;
  CUDA_TRY(cudaSetDevice(eng->device));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (span_flag) CUDA_TRY(cudaMemsetAsync(span_flag, 0, 1, stream));
  const unsigned blocks = (unsigned)(((int64_t)n + MAKE_WARPS - 1) / MAKE_WARPS);
  make_states_kernel<<<blocks, MAKE_WARPS * 32, 0, stream>>>(
      eng->d_packer.get(), *cols, n, S, G, goals, step_count, static_cast<unsigned char *>(records), (size_t)rb, status,
      span_flag);
  eng->launches++;
  CUDA_TRY(cudaGetLastError());
  return 0;
}

}  // extern "C"

// Engine checkpoints (swb_save_engine / swb_load_engine): the header, then every field of
// CkptLayout from a 16-byte boundary, in the order of the table in include/spriteworld_b200.h.
namespace {

constexpr char kCkptMagic[8] = {'S', 'W', 'B', 'C', 'K', 'P', 'T', '\0'};
constexpr uint32_t kCkptVersion = 1;
constexpr size_t kCkptFixed = 56;  // header bytes before the config signature

struct CkptHeader {
  char magic[8];
  uint32_t version;
  int32_t E, K, S, span_class, sampler;
  uint64_t seed;
  int64_t env_offset;
  uint32_t config_bytes, zero;
};
static_assert(sizeof(CkptHeader) == kCkptFixed, "checkpoint header layout");

size_t align16(size_t n) { return (n + 15) & ~(size_t)15; }

struct CkptField {
  const char *name;
  void *dev;      // the engine's array (refilled_upto: null without a sampler)
  size_t elem;    // bytes per element
  size_t count;
  size_t off = 0;
  size_t bytes() const { return elem * count; }
};

struct CkptLayout {
  enum { POS_X, POS_Y, CURSOR, STEP_COUNT, SCENE_SERIAL, RESET_NEXT, P_X, P_Y, P_M00, P_M01, P_M10, P_M11,
         P_VX, P_VY, MEMBER, RGB, FACTORS, SHAPE, POS_F32, REFILLED_UPTO, GOAL, N };
  CkptField f[N];
  size_t header = 0, total = 0;

  explicit CkptLayout(const swb_engine *eng) {
    const DevState &st = eng->st;
    const size_t E = st.E, ES = E * st.S, EKS = ES * st.K;
    const CkptField init[N] = {
        {"pos_x", st.pos_x, 8, ES}, {"pos_y", st.pos_y, 8, ES},
        {"cursor", st.cursor, 4, E}, {"step_count", st.step_count, 4, E},
        {"scene_serial", st.scene_serial, 4, E}, {"reset_next", st.reset_next, 1, E},
        {"x", st.p_x, 8, EKS}, {"y", st.p_y, 8, EKS}, {"m00", st.p_m00, 8, EKS}, {"m01", st.p_m01, 8, EKS},
        {"m10", st.p_m10, 8, EKS}, {"m11", st.p_m11, 8, EKS}, {"vx", st.p_vx, 8, EKS}, {"vy", st.p_vy, 8, EKS},
        {"member", st.p_member, 4, EKS}, {"rgb", st.p_rgb, 4, EKS}, {"factors", st.p_factors, 4, EKS * 5},
        {"shape", st.p_shape, 1, EKS}, {"pos_f32", st.p_pos_f32, 1, EKS},
        {"refilled_upto", eng->sampler ? eng->sampler->refilled_upto.get() : nullptr, 8, E},
        {"goal", st.p_goal, 8, E * st.K * st.G * 2}};   // no bytes when G == 0
    header = align16(kCkptFixed + sizeof(swb_config));
    size_t o = header;
    for (int i = 0; i < N; ++i) {
      f[i] = init[i];
      f[i].off = o;
      o = align16(o + f[i].bytes());
    }
    total = o;
  }
};

// The config signature of an engine: its swb_config with n_envs, pool_depth and device zeroed
// (engine.config_signature).
swb_config signature_of(const swb_engine *eng) {
  swb_config sig;
  memcpy(&sig, &eng->cfg, sizeof sig);
  sig.n_envs = sig.pool_depth = sig.device = 0;
  return sig;
}

template <typename T>
const T *ckpt_array(const unsigned char *buf, const CkptField &f) {
  return reinterpret_cast<const T *>(buf + f.off);
}

// Every check of swb_load_engine on a checkpoint `s` of n bytes (the staging copy, so that every
// field is aligned), before anything is enqueued.  *stars <- some pool shape is a star or spoke.
int check_checkpoint(const swb_engine *eng, const unsigned char *s, uint64_t n, const CkptLayout &L,
                     bool *stars) {
  static const char fn[] = "swb_load_engine";
  const DevState &st = eng->st;
  if (n < kCkptFixed) return fail("%s: %llu bytes are too few for the header", fn, (unsigned long long)n);
  CkptHeader h;
  memcpy(&h, s, sizeof h);
  if (memcmp(h.magic, kCkptMagic, sizeof h.magic)) return fail("%s: magic: not an engine checkpoint", fn);
  if (h.version != kCkptVersion)
    return fail("%s: version = %u, this library reads version %u", fn, h.version, kCkptVersion);
  if (h.E != st.E) return fail("%s: E = %d, the engine has n_envs = %d", fn, h.E, st.E);
  if (h.K != st.K) return fail("%s: K = %d, the engine has pool_depth = %d", fn, h.K, st.K);
  if (h.S != st.S) return fail("%s: S = %d, the engine has n_slots = %d", fn, h.S, st.S);
  if (h.config_bytes != sizeof(swb_config))
    return fail("%s: config_bytes = %u, sizeof(swb_config) is %zu", fn, h.config_bytes, sizeof(swb_config));
  if (n != L.total)
    return fail("%s: size = %llu bytes, a checkpoint of this engine has %llu", fn, (unsigned long long)n,
                (unsigned long long)L.total);
  const swb_config sig = signature_of(eng);
  const unsigned char *a = s + kCkptFixed, *b = reinterpret_cast<const unsigned char *>(&sig);
  for (size_t i = 0; i < sizeof sig; ++i)
    if (a[i] != b[i])
      return fail("%s: signature: the swb_config differs from the engine's at byte %zu (the engine's "
                  "configuration is another)", fn, i);
  if (h.span_class != 1 && h.span_class != 4)
    return fail("%s: span_class = %d, expected 1 or 4", fn, h.span_class);
  if (h.sampler != 0 && h.sampler != 1) return fail("%s: sampler = %d, expected 0 or 1", fn, h.sampler);
  const bool has = eng->sampler != nullptr;
  if (h.sampler != (int)has)
    return fail("%s: sampler: the checkpoint was saved %s a device sampler, the engine has %s", fn,
                h.sampler ? "with" : "without", has ? "one (swb_sampler_load)" : "none");
  if (has && h.seed != eng->seed)
    return fail("%s: seed = %llu, the engine's sampler has seed %llu", fn, (unsigned long long)h.seed,
                (unsigned long long)eng->seed);
  if (has && h.env_offset != eng->env_offset)
    return fail("%s: env_offset = %lld, the engine's sampler has env_offset %lld", fn,
                (long long)h.env_offset, (long long)eng->env_offset);
  const CkptField *f = L.f;
  const int32_t *cursor = ckpt_array<int32_t>(s, f[CkptLayout::CURSOR]);
  const int32_t *serial = ckpt_array<int32_t>(s, f[CkptLayout::SCENE_SERIAL]);
  const uint8_t *reset_next = ckpt_array<uint8_t>(s, f[CkptLayout::RESET_NEXT]);
  const int64_t *upto = ckpt_array<int64_t>(s, f[CkptLayout::REFILLED_UPTO]);
  for (int e = 0; e < st.E; ++e) {
    if (cursor[e] < 0 || cursor[e] >= st.K)
      return fail("%s: cursor[%d] = %d is outside [0, %d)", fn, e, cursor[e], st.K);
    if (serial[e] < 0) return fail("%s: scene_serial[%d] = %d is negative", fn, e, serial[e]);
    if (reset_next[e] > 1) return fail("%s: reset_next[%d] = %d is not 0 or 1", fn, e, reset_next[e]);
    if (upto[e] < -1) return fail("%s: refilled_upto[%d] = %lld is below -1", fn, e, (long long)upto[e]);
  }
  const uint8_t *shape = ckpt_array<uint8_t>(s, f[CkptLayout::SHAPE]);
  *stars = false;
  for (size_t i = 0; i < f[CkptLayout::SHAPE].count; ++i) {
    const int sh = shape[i];
    if (sh >= SWB_NUM_SHAPES || (sh && eng->cfg.shape_n_verts[sh] < 3))
      return fail("%s: shape[%zu] = %d (env %zu, ring slot %zu, slot %zu) %s", fn, i, sh,
                  i / st.S / st.K, i / st.S % st.K, i % st.S,
                  sh >= SWB_NUM_SHAPES ? "is not a shape id" : "has no vertex table");
    *stars = *stars || sh > 6;
  }
  return 0;
}

}  // namespace

extern "C" {

int64_t swb_engine_state_bytes(const swb_engine *eng) {
  if (!eng) {
    fail("swb_engine_state_bytes: null engine");
    return -1;
  }
  return (int64_t)CkptLayout(eng).total;
}

int swb_save_engine(swb_engine *eng, void *host_dst, uint64_t dst_bytes, void *stream_) {
  static const char fn[] = "swb_save_engine";
  if (!eng || !host_dst) return fail("%s: null argument", fn);
  const CkptLayout L(eng);
  if (dst_bytes < L.total)
    return fail("%s: the checkpoint has %llu bytes, the buffer %llu", fn, (unsigned long long)L.total,
                (unsigned long long)dst_bytes);
  CUDA_TRY(cudaSetDevice(eng->device));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  CUDA_TRY(eng->ckpt_done.wait());  // the copies of the last load may still read the staging
  CUDA_TRY(eng->h_ckpt.grow(L.total, kWaited));
  unsigned char *h = eng->h_ckpt.get();
  memset(h, 0, L.total);  // padding included: two saves of one state are byte-identical
  CkptHeader hd;
  memset(&hd, 0, sizeof hd);
  memcpy(hd.magic, kCkptMagic, sizeof hd.magic);
  hd.version = kCkptVersion;
  hd.E = eng->st.E; hd.K = eng->st.K; hd.S = eng->st.S;
  hd.span_class = eng->max_spans;
  hd.sampler = eng->sampler != nullptr;
  hd.seed = hd.sampler ? eng->seed : 0;
  hd.env_offset = hd.sampler ? eng->env_offset : 0;
  hd.config_bytes = sizeof(swb_config);
  memcpy(h, &hd, sizeof hd);
  const swb_config sig = signature_of(eng);
  memcpy(h + kCkptFixed, &sig, sizeof sig);
  for (const CkptField &f : L.f)
    if (f.dev) CUDA_TRY(cudaMemcpyAsync(h + f.off, f.dev, f.bytes(), cudaMemcpyDeviceToHost, stream));
  const CkptField &upto = L.f[CkptLayout::REFILLED_UPTO];
  if (!upto.dev) memset(h + upto.off, 0xFF, upto.bytes());  // -1: no scene sampled on the device
  CUDA_TRY(cudaStreamSynchronize(stream));
  memcpy(host_dst, h, L.total);
  return 0;
}

int swb_load_engine(swb_engine *eng, const void *host_src, uint64_t src_bytes, void *stream_) {
  static const char fn[] = "swb_load_engine";
  if (!eng || !host_src) return fail("%s: null argument", fn);
  const CkptLayout L(eng);
  CUDA_TRY(cudaSetDevice(eng->device));
  // checked in the staging copy: the caller's buffer may be reused once the call returns, and
  // every field of the copy is aligned
  CUDA_TRY(eng->ckpt_done.wait());
  CUDA_TRY(eng->h_ckpt.grow(std::max<size_t>(L.total, kCkptFixed), kWaited));
  unsigned char *h = eng->h_ckpt.get();
  memcpy(h, host_src, std::min<uint64_t>(src_bytes, L.total));
  bool stars = false;
  if (check_checkpoint(eng, h, src_bytes, L, &stars)) return 1;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  CkptHeader hd;
  memcpy(&hd, h, sizeof hd);
  // as swb_load_envs raises it; a pool holding a star or spoke needs the concave tables anyway
  eng->max_spans = std::max({eng->max_spans, (int)hd.span_class, stars ? 4 : 1});
  for (const CkptField &f : L.f)
    if (f.dev) CUDA_TRY(cudaMemcpyAsync(f.dev, h + f.off, f.bytes(), cudaMemcpyHostToDevice, stream));
  CUDA_TRY(eng->ckpt_done.record(stream));
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
