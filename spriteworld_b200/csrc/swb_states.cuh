// Env records: the save / load / copy kernels of swb_save_envs, swb_load_envs and swb_copy_envs.
//
// An env record is everything that decides an env's future steps and frames within its current
// episode: the sprite records of its current scene (the pool entry at (e, cursor[e])), its live
// positions, step_count and reset_next.  Records are record-major (record i starts at
// i * record_bytes), so that a record saved at index i can be loaded into any env.  Within a
// record every field's S values are contiguous (RecordLayout; the header documents the table).
//
// cursor and scene_serial are not part of a record: they stay with the env a record is loaded
// into, so a loaded env plays the saved episode out and then starts the next scene of its own ring.
//
// Why this is safe next to the asynchronous scene refill (environment.BatchedEnvironment), which
// uploads ring slots on a side stream: a load or copy writes only the pool entry at cursor[dst],
// the scene s_now = scene_serial[dst] the env is on, and never a refill target.  A refill planned
// from a snapshot s_old <= s_now writes absolute scenes a with refilled_upto < a <= s_old + K - 1
// < s_now + K.  The refill that uploaded s_now itself had landed -- the step stream waited on its
// event (the _risk guard) -- before the env could start s_now; every later refill writes a > s_now.
// So no refill in flight writes a scene congruent to s_now mod K.  That needs the guard to bound
// how fast an env starts scenes, and a record saved about to reset (reset_next = 1) starts the
// next one on the next step, as a reset does: the batched environment counts every load and copy
// as a reset against the guard.
#pragma once
#include <cstdint>

#include "swb_device.cuh"

namespace swb {

// Byte offsets of the fields of one record of an engine with S slots.
struct RecordLayout {
  int S;
  __host__ __device__ explicit RecordLayout(int S_) : S(S_) {}
  // x0, y0, m00, m01, m10, m11, vx, vy, pos_x, pos_y: f64 [10][S] from offset 0
  __host__ __device__ size_t member() const { return 80 * (size_t)S; }      // u32 [S]
  __host__ __device__ size_t rgb() const { return 84 * (size_t)S; }         // u32 [S]
  __host__ __device__ size_t factors() const { return 88 * (size_t)S; }     // f32 [5][S]
  __host__ __device__ size_t step_count() const { return 108 * (size_t)S; } // i32
  __host__ __device__ size_t reset_next() const { return 108 * (size_t)S + 4; }  // u8
  __host__ __device__ size_t shape() const { return 108 * (size_t)S + 5; }  // u8 [S]
  __host__ __device__ size_t pos_f32() const { return 109 * (size_t)S + 5; }  // u8 [S]
  __host__ __device__ size_t used() const { return 110 * (size_t)S + 5; }
  __host__ __device__ size_t bytes() const { return (used() + 15) & ~(size_t)15; }  // zero padded
};

// One slot of a record in registers; the per-env fields ride along in every slot's copy.
struct SlotRecord {
  double f64[10];
  uint32_t member, rgb;
  float factors[5];
  uint8_t shape, pos_f32, reset_next;
  int32_t step_count;
};

__device__ __forceinline__ SlotRecord read_state(const DevState &st, int e, int s) {
  SlotRecord r;
  const size_t p = ((size_t)e * st.K + st.cursor[e]) * st.S + s, l = (size_t)e * st.S + s;
  r.f64[0] = st.p_x[p]; r.f64[1] = st.p_y[p];
  r.f64[2] = st.p_m00[p]; r.f64[3] = st.p_m01[p]; r.f64[4] = st.p_m10[p]; r.f64[5] = st.p_m11[p];
  r.f64[6] = st.p_vx[p]; r.f64[7] = st.p_vy[p];
  r.f64[8] = st.pos_x[l]; r.f64[9] = st.pos_y[l];
  r.member = st.p_member[p];
  r.rgb = st.p_rgb[p];
#pragma unroll
  for (int f = 0; f < 5; ++f) r.factors[f] = st.p_factors[p * 5 + f];
  r.shape = st.p_shape[p];
  r.pos_f32 = st.p_pos_f32[p];
  r.step_count = st.step_count[e];
  r.reset_next = st.reset_next[e];
  return r;
}

__device__ __forceinline__ void write_state(const DevState &st, int e, int s, const SlotRecord &r) {
  const size_t p = ((size_t)e * st.K + st.cursor[e]) * st.S + s, l = (size_t)e * st.S + s;
  st.p_x[p] = r.f64[0]; st.p_y[p] = r.f64[1];
  st.p_m00[p] = r.f64[2]; st.p_m01[p] = r.f64[3]; st.p_m10[p] = r.f64[4]; st.p_m11[p] = r.f64[5];
  st.p_vx[p] = r.f64[6]; st.p_vy[p] = r.f64[7];
  st.pos_x[l] = r.f64[8]; st.pos_y[l] = r.f64[9];
  st.p_member[p] = r.member;
  st.p_rgb[p] = r.rgb;
#pragma unroll
  for (int f = 0; f < 5; ++f) st.p_factors[p * 5 + f] = r.factors[f];
  st.p_shape[p] = r.shape;
  st.p_pos_f32[p] = r.pos_f32;
  if (s == 0) {
    st.step_count[e] = r.step_count;
    st.reset_next[e] = r.reset_next;
  }
}

// A shape id without a vertex table (a record that swb_save_envs did not write) loads as an empty
// slot, so that no kernel indexes the shape table with it.
__device__ __forceinline__ SlotRecord read_record(const DevState &st, const unsigned char *rec, int s) {
  const int S = st.S;
  const RecordLayout L(S);
  SlotRecord r;
  const double *f64 = reinterpret_cast<const double *>(rec);
#pragma unroll
  for (int a = 0; a < 10; ++a) r.f64[a] = f64[a * S + s];
  r.member = reinterpret_cast<const uint32_t *>(rec + L.member())[s];
  r.rgb = reinterpret_cast<const uint32_t *>(rec + L.rgb())[s];
#pragma unroll
  for (int f = 0; f < 5; ++f) r.factors[f] = reinterpret_cast<const float *>(rec + L.factors())[f * S + s];
  const int shape = rec[L.shape() + s];
  r.shape = shape < SWB_NUM_SHAPES && st.shape_n[shape] >= 3 ? shape : 0;
  r.pos_f32 = rec[L.pos_f32() + s];
  r.step_count = *reinterpret_cast<const int32_t *>(rec + L.step_count());
  r.reset_next = rec[L.reset_next()];
  return r;
}

__device__ __forceinline__ void write_record(unsigned char *rec, int S, int s, const SlotRecord &r) {
  const RecordLayout L(S);
  double *f64 = reinterpret_cast<double *>(rec);
#pragma unroll
  for (int a = 0; a < 10; ++a) f64[a * S + s] = r.f64[a];
  reinterpret_cast<uint32_t *>(rec + L.member())[s] = r.member;
  reinterpret_cast<uint32_t *>(rec + L.rgb())[s] = r.rgb;
#pragma unroll
  for (int f = 0; f < 5; ++f) reinterpret_cast<float *>(rec + L.factors())[f * S + s] = r.factors[f];
  rec[L.shape() + s] = r.shape;
  rec[L.pos_f32() + s] = r.pos_f32;
  if (s == 0) {
    *reinterpret_cast<int32_t *>(rec + L.step_count()) = r.step_count;
    rec[L.reset_next()] = r.reset_next;
    for (size_t b = L.used(); b < L.bytes(); ++b) rec[b] = 0;  // saved bytes are deterministic
  }
}

// One thread per (record, slot), as scatter_scenes_kernel.  record i <- env ids[i]
__global__ void save_envs_kernel(DevState st, int n, const int32_t *__restrict__ ids,
                                 unsigned char *__restrict__ rec, size_t record_bytes) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * st.S) return;
  const int r = i / st.S, s = i - r * st.S;
  write_record(rec + (size_t)r * record_bytes, st.S, s, read_state(st, ids[r], s));
}

// env ids[i] <- record i (ids distinct)
__global__ void load_envs_kernel(DevState st, int n, const int32_t *__restrict__ ids,
                                 const unsigned char *__restrict__ rec, size_t record_bytes) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * st.S) return;
  const int r = i / st.S, s = i - r * st.S;
  write_state(st, ids[r], s, read_record(st, rec + (size_t)r * record_bytes, s));
}

// env dst[i] <- env src[i], for id sets that do not overlap (no thread reads what another writes)
__global__ void copy_envs_kernel(DevState st, int n, const int32_t *__restrict__ src,
                                 const int32_t *__restrict__ dst) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * st.S) return;
  const int r = i / st.S, s = i - r * st.S;
  write_state(st, dst[r], s, read_state(st, src[r], s));
}

// Device-checked id lists (swb_save_envs_dev / swb_load_envs_dev / swb_copy_envs_dev).
//
// Every call k of an engine gets a sequence number seq (1 .. 2^32 - 2, so that hi = ~seq never
// equals the all-ones initial value) and keys hi << 32 | low: a later call's keys are smaller.
// Failing positions atomicMin the key hi | (position << 1 | argument) into one engine word, so
// that word holds a key of call k exactly when call k failed, and then the lowest failing position
// of it.  A destination id claims its env with atomicMin(claim[id], hi | position); after that
// pass a destination whose claim is not its own key repeats an id at a lower position.  Neither
// word needs clearing between calls: the next call's keys replace the last one's.
struct IdCall {
  const void *ids[2];          // id arguments 0 and 1 (copy: src, dst; else ids[1] is null)
  int n;
  int dst_arg;                 // the argument whose ids must be distinct, or -1 (save)
  int call;                    // SWB_IDS_CALL_*
  unsigned long long hi;       // ~seq << 32
  unsigned long long *claim;   // [E]
  unsigned long long *fail;    // [1]
  swb_ids_status *status;
};

template <typename T>
__device__ __forceinline__ bool id_in_range(T id, int E) {
  return id >= 0 && id < static_cast<T>(E);   // in T's width: an int64 2^32 + 1 does not wrap
}

// Argument a's ids (a select, not an index: an indexed kernel parameter array goes to the stack)
template <typename T>
__device__ __forceinline__ const T *ids_of(const IdCall &c, int a) {
  return static_cast<const T *>(a ? c.ids[1] : c.ids[0]);
}

__device__ __forceinline__ bool call_refused(const IdCall &c) {
  return (*c.fail >> 32) == (c.hi >> 32);
}

// Thread 0 of a call's last kernel: the ok word, and the call's first failure if none is recorded.
template <typename T>
__device__ void report_ids(const IdCall &c, int E) {
  const unsigned long long f = *c.fail;
  const bool bad = (f >> 32) == (c.hi >> 32);
  swb_ids_status *s = c.status;
  s->ok = bad ? 0u : 1u;
  if (!bad || s->failed) return;
  const unsigned low = (unsigned)f;
  const int a = (int)(low & 1u), p = (int)(low >> 1);
  const T id = ids_of<T>(c, a)[p];
  s->call = c.call;
  s->arg = a;
  s->reason = id_in_range(id, E) ? SWB_IDS_REPEATED : SWB_IDS_OUT_OF_RANGE;
  s->position = p;
  s->value = (int64_t)id;
  s->failed = 1u;
}

// One thread per (argument, position): range check, and the claims of destination ids.
template <typename T>
__global__ void check_ids_kernel(IdCall c, int E) {
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int n_args = c.ids[1] ? 2 : 1;
  if (t >= (size_t)n_args * c.n) return;
  const int a = (int)(t / c.n), p = (int)(t - (size_t)a * c.n);
  const T id = ids_of<T>(c, a)[p];
  if (!id_in_range(id, E))
    atomicMin(c.fail, c.hi | ((unsigned long long)p << 1 | (unsigned)a));
  else if (a == c.dst_arg)
    atomicMin(c.claim + id, c.hi | (unsigned)p);
}

// After check_ids_kernel: a destination whose claim is another position's repeats an id.
template <typename T>
__device__ __forceinline__ void check_repeat(const IdCall &c, int E, int p) {
  const T id = ids_of<T>(c, c.dst_arg)[p];
  if (id_in_range(id, E) && c.claim[id] != (c.hi | (unsigned)p))
    atomicMin(c.fail, c.hi | ((unsigned long long)p << 1 | (unsigned)c.dst_arg));
}

template <typename T>
__global__ void repeat_ids_kernel(IdCall c, int E) {
  const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p < (size_t)c.n) check_repeat<T>(c, E, (int)p);
}

// record i <- env ids[i], or zeros in every record of a refused call
template <typename T>
__global__ void save_envs_dev_kernel(DevState st, IdCall c, unsigned char *__restrict__ rec,
                                     size_t record_bytes) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) report_ids<T>(c, st.E);
  if (i >= (size_t)c.n * st.S) return;
  const int r = (int)(i / st.S), s = (int)(i - (size_t)r * st.S);
  const int id = (int)ids_of<T>(c, 0)[r];
  write_record(rec + (size_t)r * record_bytes, st.S, s, call_refused(c) ? SlotRecord{} : read_state(st, id, s));
}

// Copy, first half: the repeat check of the destinations, and record i <- env src[i] in engine
// scratch for every source in range (the load below reads none of it if the call is refused).
template <typename T>
__global__ void stage_copy_dev_kernel(DevState st, IdCall c, unsigned char *__restrict__ rec,
                                      size_t record_bytes) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)c.n * st.S) return;
  const int r = (int)(i / st.S), s = (int)(i - (size_t)r * st.S);
  if (s == 0) check_repeat<T>(c, st.E, r);
  const T id = ids_of<T>(c, 0)[r];
  if (id_in_range(id, st.E)) write_record(rec + (size_t)r * record_bytes, st.S, s, read_state(st, (int)id, s));
}

// env ids[dst_arg][i] <- record i, unless the call is refused
template <typename T>
__global__ void load_envs_dev_kernel(DevState st, IdCall c, const unsigned char *__restrict__ rec,
                                     size_t record_bytes) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) report_ids<T>(c, st.E);
  if (i >= (size_t)c.n * st.S || call_refused(c)) return;
  const int r = (int)(i / st.S), s = (int)(i - (size_t)r * st.S);
  const int id = (int)ids_of<T>(c, c.dst_arg)[r];
  write_state(st, id, s, read_record(st, rec + (size_t)r * record_bytes, s));
}

}  // namespace swb
