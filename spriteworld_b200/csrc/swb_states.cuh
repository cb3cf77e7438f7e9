// Env records: the kernels of swb_save_envs, swb_load_envs and swb_copy_envs and of their _dev
// variants.  save_envs_kernel<T> and load_envs_kernel<T> serve both; copy_envs_kernel copies
// host-checked ids that do not overlap; device-checked ids add check_ids_kernel<T>,
// repeat_ids_kernel<T> and stage_copy_dev_kernel<T>.
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
#include "swb_record_layout.h"

namespace swb {

__device__ __forceinline__ SlotRecord read_state(const DevState &st, int e, int s) {
  SlotRecord r;
  const size_t p = ((size_t)e * st.K + st.cursor[e]) * st.S + s, l = (size_t)e * st.S + s;
  r.f64[X0] = st.p_x[p]; r.f64[Y0] = st.p_y[p];
  r.f64[M00] = st.p_m00[p]; r.f64[M01] = st.p_m01[p]; r.f64[M10] = st.p_m10[p]; r.f64[M11] = st.p_m11[p];
  r.f64[VX] = st.p_vx[p]; r.f64[VY] = st.p_vy[p];
  r.f64[POS_X] = st.pos_x[l]; r.f64[POS_Y] = st.pos_y[l];
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
  st.p_x[p] = r.f64[X0]; st.p_y[p] = r.f64[Y0];
  st.p_m00[p] = r.f64[M00]; st.p_m01[p] = r.f64[M01]; st.p_m10[p] = r.f64[M10]; st.p_m11[p] = r.f64[M11];
  st.p_vx[p] = r.f64[VX]; st.p_vy[p] = r.f64[VY];
  st.pos_x[l] = r.f64[POS_X]; st.pos_y[l] = r.f64[POS_Y];
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

// Slot s of a record, with its shape id sanitised as a load sanitises it.  Every kernel that reads
// records reads them through this; the loads of fields a kernel does not use are dead code.
__device__ __forceinline__ SlotRecord read_record(const DevState &st, const unsigned char *rec, int s) {
  const int S = st.S;
  const RecordLayout L(S);
  SlotRecord r;
#pragma unroll
  for (int a = 0; a < N_F64; ++a) r.f64[a] = reinterpret_cast<const double *>(rec)[L.f64_at(a, s)];
  r.member = reinterpret_cast<const uint32_t *>(rec + L.member())[s];
  r.rgb = reinterpret_cast<const uint32_t *>(rec + L.rgb())[s];
#pragma unroll
  for (int f = 0; f < 5; ++f) r.factors[f] = reinterpret_cast<const float *>(rec + L.factors())[f * S + s];
  r.shape = sanitize_shape(rec[L.shape() + s], st.shape_n);
  r.pos_f32 = rec[L.pos_f32() + s];
  r.step_count = *reinterpret_cast<const int32_t *>(rec + L.step_count());
  r.reset_next = rec[L.reset_next()];
  return r;
}

// The goals (G x (x, y)) of the scene env e is on.
__device__ __forceinline__ double *state_goals(const DevState &st, int e) {
  return st.p_goal + ((size_t)e * st.K + st.cursor[e]) * st.G * 2;
}

// The id lists of a record call (and of swb_set_goals) (swb_save_envs / swb_load_envs / swb_copy_envs and their _dev
// variants).  Ids checked on the host (host_checked) are int32 and all valid: no check kernel runs
// before the call's kernels, the call is never refused and reports nothing.
//
// Device-checked ids: every call k of an engine gets a sequence number seq (1 .. 2^32 - 2, so that
// hi = ~seq never equals the all-ones initial value) and keys hi << 32 | low: a later call's keys
// are smaller.  Failing positions atomicMin the key hi | (position << 1 | argument) into one engine
// word, so that word holds a key of call k exactly when call k failed, and then the lowest failing
// position of it.  A destination id claims its env with atomicMin(claim[id], hi | position); after
// that pass a destination whose claim is not its own key repeats an id at a lower position.
// Neither word needs clearing between calls: the next call's keys replace the last one's.
struct IdCall {
  const void *ids[2];          // id arguments 0 and 1 (copy: src, dst; else ids[1] is null)
  int n;
  int dst_arg;                 // the argument whose ids must be distinct, or -1 (save)
  bool host_checked;
  // device-checked ids only
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
  return !c.host_checked && (*c.fail >> 32) == (c.hi >> 32);
}

// Thread 0 of a device-checked call's last kernel: the ok word, and the call's first failure if
// none is recorded.
template <typename T>
__device__ void report_ids(const IdCall &c, int E) {
  if (c.host_checked) return;
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

// One thread per (record, slot), as scatter_scenes_kernel.  record i <- env ids[0][i], or zeros
// in every record of a refused call
template <typename T>
__global__ void save_envs_kernel(DevState st, IdCall c, unsigned char *__restrict__ rec,
                                 size_t record_bytes) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) report_ids<T>(c, st.E);
  if (i >= (size_t)c.n * st.S) return;
  const int r = (int)(i / st.S), s = (int)(i - (size_t)r * st.S);
  const int id = (int)ids_of<T>(c, 0)[r];
  const bool refused = call_refused(c);
  unsigned char *dst = rec + (size_t)r * record_bytes;
  write_record(dst, st.S, st.G, s, refused ? SlotRecord{} : read_state(st, id, s));
  if (s == 0 && st.G) write_goals(record_goals(dst, st.S, st.G), refused ? nullptr : state_goals(st, id), st.G);
}

// Device-checked copy, first half: the repeat check of the destinations, and record i <- env
// src[i] in engine scratch for every source in range (the load below reads none of it if the call
// is refused).
template <typename T>
__global__ void stage_copy_dev_kernel(DevState st, IdCall c, unsigned char *__restrict__ rec,
                                      size_t record_bytes) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)c.n * st.S) return;
  const int r = (int)(i / st.S), s = (int)(i - (size_t)r * st.S);
  if (s == 0) check_repeat<T>(c, st.E, r);
  const T id = ids_of<T>(c, 0)[r];
  if (id_in_range(id, st.E)) {
    unsigned char *dst = rec + (size_t)r * record_bytes;
    write_record(dst, st.S, st.G, s, read_state(st, (int)id, s));
    if (s == 0 && st.G) write_goals(record_goals(dst, st.S, st.G), state_goals(st, (int)id), st.G);
  }
}

// env ids[dst_arg][i] <- record i (ids distinct), unless the call is refused
template <typename T>
__global__ void load_envs_kernel(DevState st, IdCall c, const unsigned char *__restrict__ rec,
                                 size_t record_bytes) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) report_ids<T>(c, st.E);
  if (i >= (size_t)c.n * st.S || call_refused(c)) return;
  const int r = (int)(i / st.S), s = (int)(i - (size_t)r * st.S);
  const int id = (int)ids_of<T>(c, c.dst_arg)[r];
  const unsigned char *src = rec + (size_t)r * record_bytes;
  write_state(st, id, s, read_record(st, src, s));
  if (s == 0 && st.G) write_goals(state_goals(st, id), record_goals(src, st.S, st.G), st.G);
}

// Host-checked copy of id sets that do not overlap (no thread reads what another writes):
// env dst[i] <- env src[i] in one pass, without scratch
__global__ void copy_envs_kernel(DevState st, IdCall c) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.n * st.S) return;
  const int r = i / st.S, s = i - r * st.S;
  const int src = ids_of<int32_t>(c, 0)[r], dst = ids_of<int32_t>(c, 1)[r];
  write_state(st, dst, s, read_state(st, src, s));
  if (s == 0 && st.G) write_goals(state_goals(st, dst), state_goals(st, src), st.G);
}

// swb_set_goals / swb_set_goals_dev: one thread per (id, goal value); env ids[0][i] <- goals of row i,
// unless the call is refused
template <typename T>
__global__ void set_goals_kernel(DevState st, IdCall c, const double *__restrict__ goals) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) report_ids<T>(c, st.E);
  const size_t per = 2 * (size_t)st.G;
  if (i >= (size_t)c.n * per || call_refused(c)) return;
  const int r = (int)(i / per), j = (int)(i - (size_t)r * per);
  state_goals(st, (int)ids_of<T>(c, 0)[r])[j] = goals[i];
}

}  // namespace swb
