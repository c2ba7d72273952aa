// sm_90a device code of the collective engine: inter-GPU synchronisation on
// flag pads, eager slot transfers, NVLS (multimem) and peer-to-peer
// collective bodies with the reduction fused into the transfer.  `run_work`
// executes one WorkItem cooperatively on `nctas` CTAs; it is called both by
// the per-call kernel (direct launch) and by the persistent engine kernel.
//
// Reference counterparts: the DMP data loops and RX-buffer matching
// (kernels/cclo/hls/dma_mover/dma_mover.cpp:433-927, rxbuf_offload/*.cpp), the
// arithmetic and cast plugins (kernels/plugins/reduce_ops, hp_compression) and
// the firmware collectives (ccl_offload_control.c:531-2218).  Algorithms are
// NVSwitch-native instead: one-shot through eager slots for small messages,
// two-shot with in-switch reduction (multimem.ld_reduce + multimem.st) or peer
// loads/stores for large ones; no rings or trees — every peer is one hop away.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>

#include "accl/cuda/devtypes.hpp"
#include "accl/device/primitives.cuh"

namespace accl {
namespace cuda {
namespace k {

using namespace accl::dev;

constexpr int BLOCK = 512;

__device__ __forceinline__ uint32_t esize_of(uint32_t dtype) { return dtype_bytes(static_cast<dataType>(dtype)); }

// ------------------------------------------------------------------ context
struct Ctx {
  const DevWorld &w;
  const WorkItem &it;
  int cta, nctas;
  Ctrl *me;           // my control block
  uint32_t *err;      // shared-memory error word of this CTA
  uint64_t timeout_ns;
  struct PtrTable *tab; // shared-memory pointer table of this CTA
  __device__ char *heap(uint32_t grank) const { return w.window + static_cast<uint64_t>(grank) * w.heap_bytes; }
  __device__ Ctrl *ctrl(uint32_t grank) const { return reinterpret_cast<Ctrl *>(heap(grank)); }
  __device__ PadBank &pads() const { return me->pad[it.bank]; }
  __device__ PadBank &pads_of(uint32_t grank) const { return ctrl(grank)->pad[it.bank]; }
  __device__ StageBank &stg() const { return me->stg[it.bank]; }
  __device__ StageBank &stg_of(uint32_t grank) const { return ctrl(grank)->stg[it.bank]; }
  __device__ uint32_t kind_word() const { return (it.desc.scenario & 0xFFu) | (it.comm_sig << 8); }
  __device__ uint32_t P() const { return it.comm_size; }
  __device__ uint32_t r() const { return it.comm_rank; }
  __device__ uint32_t g(uint32_t comm_rank) const { return it.members[comm_rank]; }
};

// spin until *p >= target (wrap-safe); false + error bit on timeout
__device__ __forceinline__ bool wait_ge(const uint32_t *p, uint32_t target, const Ctx &c, uint32_t errbit) {
  uint32_t spins = 0;
  uint64_t t0 = 0;
  while (static_cast<int32_t>(ld_acquire_sys(p) - target) < 0) {
    ++spins;
    if (spins > 32) nanosleep(spins > 4096 ? 256 : 32);
    if ((spins & 0x3FF) == 0) {
      const uint64_t now = globaltimer_ns();
      if (t0 == 0) t0 = now;
      else if (now - t0 > c.timeout_ns) {
        atomicOr(c.err, errbit);
        return false;
      }
    }
  }
  return true;
}

// ------------------------------------------------------ sync-pad meetings
// A meeting of this rank with one peer on channel `ch` of the call's bank (global rank `peer`): each side posts
// (sent += 1, optionally a record, then the release of the peer's `sig`), then takes the peer's post (expect += 1)
// once `sig` has reached it.  The pad layout and the record format are known only to the helpers below.  They are
// per thread and never call __syncthreads: a CTA serves its peers with one thread each, the fused plugins one lane each
// (meet_peers, below), and the engine polls with `pad_arrived` instead of blocking.

// which fields of the record a post carries: none (a bare signal), off0 + kind, or off0 + off2 + kind
enum PadRec : uint32_t { REC_NONE, REC_OFF0, REC_OFFS };

__device__ __forceinline__ void pad_post(const Ctx &c, uint32_t ch, uint32_t peer, PadRec rec, uint64_t off0, uint64_t off2,
                                         uint32_t kind) {
  PadBank &mine = c.pads();
  PadBank &theirs = c.pads_of(peer);
  const uint32_t v = mine.sent[ch][peer] + 1;
  mine.sent[ch][peer] = v;
  if (rec != REC_NONE) {
    SyncRec *rr = &theirs.rec[ch][c.w.rank];
    st_relaxed_sys(&rr->off0, off0);
    if (rec == REC_OFFS) st_relaxed_sys(&rr->off2, off2);
    st_relaxed_sys(&rr->kind, kind);
  }
  st_release_sys(&theirs.sig[ch][c.w.rank], v);
}

// has the peer's next post landed?
__device__ __forceinline__ bool pad_arrived(const Ctx &c, uint32_t ch, uint32_t peer) {
  const PadBank &mine = c.pads();
  return static_cast<int32_t>(ld_acquire_sys(&mine.sig[ch][peer]) - (mine.expect[ch][peer] + 1)) >= 0;
}

// take the peer's next post (after pad_arrived); returns its number
__device__ __forceinline__ uint32_t pad_take(const Ctx &c, uint32_t ch, uint32_t peer) {
  PadBank &mine = c.pads();
  const uint32_t e = mine.expect[ch][peer] + 1;
  mine.expect[ch][peer] = e;
  return e;
}

// take the peer's next post and wait for it; false + RECEIVE_TIMEOUT_ERROR on timeout.  The post counts as taken
// either way, so the next meeting waits for the peer's next post.
__device__ __forceinline__ bool pad_wait(const Ctx &c, uint32_t ch, uint32_t peer) {
  const uint32_t e = pad_take(c, ch, peer);
  return wait_ge(&c.pads().sig[ch][peer], e, c, RECEIVE_TIMEOUT_ERROR);
}

// the record of the post just taken, as far as `rec` says the peer wrote it
__device__ __forceinline__ SyncRec pad_rec(const Ctx &c, uint32_t ch, uint32_t peer, PadRec rec) {
  const SyncRec *mr = &c.pads().rec[ch][peer];
  SyncRec r{};
  r.off0 = ld_relaxed_sys(&mr->off0);
  if (rec == REC_OFFS) r.off2 = ld_relaxed_sys(&mr->off2);
  r.kind = ld_relaxed_sys(&mr->kind);
  return r;
}

// Symmetric synchronisation of this CTA's channel with the same channel of
// every communicator peer.  Optionally carries (off0, off2) to the peers —
// the rendezvous address exchange — and returns theirs in shared arrays.
// All threads of the CTA must call it.
__device__ __forceinline__ void chan_sync(const Ctx &c, bool exchange, uint64_t my_off0, uint64_t my_off2,
                                          uint64_t *s_off0, uint64_t *s_off2) {
  __syncthreads(); // every thread's prior writes happen-before the release below
  const uint32_t t = threadIdx.x;
  const uint32_t ch = static_cast<uint32_t>(c.cta);
  if (t == c.r()) {
    if (exchange) {
      s_off0[t] = my_off0;
      s_off2[t] = my_off2;
    }
  } else if (t < c.P()) {
    const uint32_t peer = c.g(t);
    pad_post(c, ch, peer, exchange ? REC_OFFS : REC_NONE, my_off0, my_off2, c.kind_word());
    if (pad_wait(c, ch, peer) && exchange) {
      const SyncRec r = pad_rec(c, ch, peer, REC_OFFS);
      s_off0[t] = r.off0;
      s_off2[t] = r.off2;
      // a peer in a different operation, or in a different communicator that hashes onto this bank
      if (r.kind != c.kind_word()) atomicOr(c.err, PACK_SEQ_NUMBER_ERROR);
    }
  }
  __syncthreads();
}

// pairwise variant for send/recv in direct mode: only (me, peer) take part; kinds differ by design
// `post_rec` = false: signal only.  The second meeting of a transfer must NOT rewrite the record: the peer may not have
// read the first one yet (the receiver runs straight from its first into its second meeting).
__device__ __forceinline__ void pair_sync(const Ctx &c, uint32_t peer_comm_rank, uint64_t my_off, uint32_t my_kind,
                                          uint64_t *peer_off, uint32_t *peer_kind, bool post_rec = true) {
  __syncthreads();
  if (threadIdx.x == 0) {
    const uint32_t ch = static_cast<uint32_t>(c.cta);
    const uint32_t peer = c.g(peer_comm_rank);
    pad_post(c, ch, peer, post_rec ? REC_OFF0 : REC_NONE, my_off, 0, my_kind);
    if (pad_wait(c, ch, peer)) {
      const SyncRec r = pad_rec(c, ch, peer, REC_OFF0);
      *peer_off = r.off0;
      *peer_kind = r.kind;
    } else {
      *peer_off = INVALID_OFF;
      *peer_kind = 0xFFFFFFFFu;
    }
  }
  __syncthreads();
}

// ------------------------------------------------ fused plugin kernels
// The fused plugins (plugin_gemm_rs.cu, plugin_ag_gemm.cu, plugin_ar_rmsnorm.cu) meet their peers on the sync pads of
// channel MAX_CH-1, bank 0, through an identity communicator whose kind word names the plugin, and coordinate their
// grid through a flag block in device memory that the host zeroes on the stream before every launch
// (plugin_flags, launch.hpp).  Words of the block; a plugin's own words start at FLAG_PLUGIN.
enum PluginFlag : uint32_t {
  FLAG_RELEASE, // the entry meeting is over: FLAG_MASK is valid
  FLAG_DONE,    // CTAs that have finished
  FLAG_ERR,     // error bits of the grid
  FLAG_MASK,    // meet_peers' mask
  FLAG_PLUGIN
};

// The identity communicator of a plugin kernel (world ranks, channel MAX_CH-1 of bank 0).  scenario and comm_sig make
// up its kind word: a peer inside another plugin reports PACK_SEQ_NUMBER_ERROR.
__device__ __forceinline__ void plugin_item(WorkItem &it, const DevWorld &w, uint32_t scenario, uint32_t comm_sig, uint32_t timeout_us) {
  it.comm_size = w.world;
  it.comm_rank = w.rank;
  for (uint32_t r = 0; r < static_cast<uint32_t>(ACCL_MAX_RANKS); ++r) it.members[r] = static_cast<uint8_t>(r < w.world ? r : 0);
  it.desc.scenario = scenario;
  it.timeout_us = timeout_us;
  it.bank = 0;
  it.comm_sig = comm_sig;
}

// Entry meeting of a plugin kernel, called by one whole warp: lane q meets rank q on channel MAX_CH-1 and posts
// (off0, off2) with `rec` (REC_OFF0: off0 only).  Returns the ranks whose post carries this kernel's kind word and the
// same offsets; this rank's bit is always set.  A peer in another plugin sets PACK_SEQ_NUMBER_ERROR, one whose offsets
// differ DMA_MISMATCH_ERROR, one that does not answer within the call timeout RECEIVE_TIMEOUT_ERROR.
__device__ __forceinline__ uint32_t meet_peers(const Ctx &c, PadRec rec, uint64_t off0, uint64_t off2) {
  const uint32_t lane = threadIdx.x % 32, ch = MAX_CH - 1;
  bool ok = lane == c.w.rank;
  if (lane < c.w.world && lane != c.w.rank) {
    pad_post(c, ch, lane, rec, off0, off2, c.kind_word());
    if (pad_wait(c, ch, lane)) {
      const SyncRec r = pad_rec(c, ch, lane, rec);
      if (r.kind != c.kind_word())
        atomicOr(c.err, PACK_SEQ_NUMBER_ERROR);
      else if (r.off0 != off0 || (rec == REC_OFFS && r.off2 != off2))
        atomicOr(c.err, DMA_MISMATCH_ERROR);
      else
        ok = true;
    }
  }
  return __ballot_sync(0xffffffffu, ok);
}

// Release the grid after the entry meeting (one thread): publish the mask of meet_peers, then the release.
__device__ __forceinline__ void release_grid(unsigned int *flags, uint32_t mask) {
  flags[FLAG_MASK] = mask;
  __threadfence();
  st_release_gpu(&flags[FLAG_RELEASE], 1u);
}

// Wait for release_grid (one thread) and return its mask; on timeout RECEIVE_TIMEOUT_ERROR and this rank alone.
__device__ __forceinline__ uint32_t wait_grid(const unsigned int *flags, const Ctx &c) {
  const bool released = wait_ge(&flags[FLAG_RELEASE], 1u, c, RECEIVE_TIMEOUT_ERROR);
  return (released ? *reinterpret_cast<const volatile unsigned int *>(&flags[FLAG_MASK]) : 0u) | (1u << c.w.rank);
}

// Exit of a plugin kernel, called by every thread of every CTA once the CTA's work is done: OR the CTA's error bits
// into the block and count the CTA finished.  The last CTA of the grid meets every peer once more when `meet` (so no
// rank rewrites what a peer still reads, or leaves while a peer still writes into it) and publishes the error bits of
// the grid to `status` (0: success; may be null).  s_last: a shared word of the CTA, declared with its other shared
// words (a shared variable of its own here moves the kernel's shared layout, which cost the RMSNorm kernel a register).
__device__ __forceinline__ void plugin_exit(const Ctx &c, unsigned int *flags, uint32_t *status, bool meet, uint32_t &s_last) {
  __syncthreads();
  if (threadIdx.x == 0) {
    if (*c.err) atomicOr(&flags[FLAG_ERR], *c.err);
    // GPU scope suffices: every write into a peer is followed by __threadfence_system() in the thread that made it,
    // before the CTA gets here.  A system-scope fence here cost the RMSNorm kernel ~2 us a call on an H100.
    __threadfence(); // this CTA's writes are performed before it counts itself finished
    s_last = atomicAdd(&flags[FLAG_DONE], 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  if (meet) chan_sync(c, false, 0, 0, nullptr, nullptr);
  if (threadIdx.x == 0 && status) *status = atomicOr(&flags[FLAG_ERR], *c.err) | *c.err;
}

// ------------------------------------------------------ exchange patterns
// The eight collectives as exchange patterns, shared by the eager slot ring (collectives.cuh), the one-way
// staged exchanges (staged.cuh) and the rendezvous data phases.  PAT_NONE: not a collective.
enum Pattern : uint32_t {
  PAT_ALLREDUCE, PAT_REDUCE_SCATTER, PAT_ALLGATHER, PAT_BCAST, PAT_SCATTER, PAT_GATHER, PAT_REDUCE, PAT_ALLTOALL, PAT_NONE
};

__device__ __forceinline__ Pattern pattern_of(operation op) {
  switch (op) {
  case operation::allreduce: return PAT_ALLREDUCE;
  case operation::reduce_scatter: return PAT_REDUCE_SCATTER;
  case operation::allgather: return PAT_ALLGATHER;
  case operation::bcast: return PAT_BCAST;
  case operation::scatter: return PAT_SCATTER;
  case operation::gather: return PAT_GATHER;
  case operation::reduce: return PAT_REDUCE;
  case operation::alltoall: return PAT_ALLTOALL;
  default: return PAT_NONE;
  }
}

// who pushes to whom in a one-way exchange of pattern `pat` (communicator ranks)
struct Roles {
  Pattern pat;
  uint32_t P, me, root;
  __device__ bool pushes_to(uint32_t q) const {
    if (q == me) return false;
    switch (pat) {
    case PAT_ALLREDUCE: case PAT_ALLGATHER: case PAT_REDUCE_SCATTER: case PAT_ALLTOALL: return true;
    case PAT_BCAST: case PAT_SCATTER: return me == root;
    case PAT_GATHER: case PAT_REDUCE: return q == root;
    default: return false;
    }
  }
  __device__ bool expects_from(uint32_t q) const {
    if (q == me) return false;
    switch (pat) {
    case PAT_ALLREDUCE: case PAT_ALLGATHER: case PAT_REDUCE_SCATTER: case PAT_ALLTOALL: return true;
    case PAT_BCAST: case PAT_SCATTER: return me != root && q == root;
    case PAT_GATHER: case PAT_REDUCE: return me == root;
    default: return false;
    }
  }
  // does every destination get the same bytes of my source buffer?
  __device__ bool same_src() const {
    return pat == PAT_ALLREDUCE || pat == PAT_ALLGATHER || pat == PAT_BCAST || pat == PAT_GATHER || pat == PAT_REDUCE;
  }
};

// ------------------------------------------------------- typed arithmetic
template <typename T> struct Tr;
template <> struct Tr<float> {
  using A = float;
  static __device__ __forceinline__ A up(float x) { return x; }
  static __device__ __forceinline__ float down(A x) { return x; }
};
template <> struct Tr<double> {
  using A = double;
  static __device__ __forceinline__ A up(double x) { return x; }
  static __device__ __forceinline__ double down(A x) { return x; }
};
template <> struct Tr<int32_t> {
  using A = int32_t;
  static __device__ __forceinline__ A up(int32_t x) { return x; }
  static __device__ __forceinline__ int32_t down(A x) { return x; }
};
template <> struct Tr<int64_t> {
  using A = int64_t;
  static __device__ __forceinline__ A up(int64_t x) { return x; }
  static __device__ __forceinline__ int64_t down(A x) { return x; }
};
template <> struct Tr<__half> {
  using A = float;
  static __device__ __forceinline__ A up(__half x) { return __half2float(x); }
  static __device__ __forceinline__ __half down(A x) { return __float2half_rn(x); }
};
template <> struct Tr<__nv_bfloat16> {
  using A = float;
  static __device__ __forceinline__ A up(__nv_bfloat16 x) { return __bfloat162float(x); }
  static __device__ __forceinline__ __nv_bfloat16 down(A x) { return __float2bfloat16_rn(x); }
};
template <> struct Tr<__nv_fp8_e4m3> {
  using A = float;
  static __device__ __forceinline__ A up(__nv_fp8_e4m3 x) { return static_cast<float>(x); }
  static __device__ __forceinline__ __nv_fp8_e4m3 down(A x) { return __nv_fp8_e4m3(x); }
};
template <> struct Tr<__nv_fp8_e5m2> {
  using A = float;
  static __device__ __forceinline__ A up(__nv_fp8_e5m2 x) { return static_cast<float>(x); }
  static __device__ __forceinline__ __nv_fp8_e5m2 down(A x) { return __nv_fp8_e5m2(x); }
};

struct OpSum {
  template <typename A> static __device__ __forceinline__ A apply(A a, A b) { return a + b; }
};
struct OpMax {
  template <typename A> static __device__ __forceinline__ A apply(A a, A b) { return a > b ? a : b; }
};

template <typename T> struct VecOf {
  static constexpr int N = 16 / sizeof(T);
  using A = typename Tr<T>::A;
  static __device__ __forceinline__ void unpack(const Vec16 &v, A (&a)[N]) {
    const T *e = reinterpret_cast<const T *>(&v);
#pragma unroll
    for (int i = 0; i < N; ++i) a[i] = Tr<T>::up(e[i]);
  }
  static __device__ __forceinline__ Vec16 pack(const A (&a)[N]) {
    Vec16 v;
    T *e = reinterpret_cast<T *>(&v);
#pragma unroll
    for (int i = 0; i < N; ++i) e[i] = Tr<T>::down(a[i]);
    return v;
  }
};

// 16-bit floats: widen / narrow two lanes per 32-bit word (bf16 -> f32 is a shift, the narrowing
// is one cvt.rn.*x2 per pair) instead of eight scalar conversions per 16 bytes.  The SM reduce
// paths are ALU-limited for 16-bit types otherwise.
template <> struct VecOf<__nv_bfloat16> {
  static constexpr int N = 8;
  using A = float;
  static __device__ __forceinline__ void unpack(const Vec16 &v, A (&a)[N]) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      a[2 * i] = __uint_as_float(w[i] << 16);
      a[2 * i + 1] = __uint_as_float(w[i] & 0xFFFF0000u);
    }
  }
  static __device__ __forceinline__ Vec16 pack(const A (&a)[N]) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      __nv_bfloat162 p = __floats2bfloat162_rn(a[2 * i], a[2 * i + 1]);
      w[i] = *reinterpret_cast<uint32_t *>(&p);
    }
    return Vec16{w[0], w[1], w[2], w[3]};
  }
};
template <> struct VecOf<__half> {
  static constexpr int N = 8;
  using A = float;
  static __device__ __forceinline__ void unpack(const Vec16 &v, A (&a)[N]) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __half22float2(*reinterpret_cast<const __half2 *>(&w[i]));
      a[2 * i] = f.x;
      a[2 * i + 1] = f.y;
    }
  }
  static __device__ __forceinline__ Vec16 pack(const A (&a)[N]) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      __half2 p = __floats2half2_rn(a[2 * i], a[2 * i + 1]);
      w[i] = *reinterpret_cast<uint32_t *>(&p);
    }
    return Vec16{w[0], w[1], w[2], w[3]};
  }
};

// Pointer table of one data-movement step.  Lives in shared memory so that
// rank-indexed accesses never turn into local-memory arrays.
struct PtrTable {
  const char *src[ACCL_MAX_RANKS];
  char *dst[ACCL_MAX_RANKS];
};

// Core reduce loop: for every element i < n, dst[q][i] = op over p of
// src[p][i], for q < ndst.  Sources and destinations may live on peers.  Work
// is split over (cta, nctas).  NP > 0 fixes the source count at compile time
// (loads of all peers are issued back to back); NP == 0 uses the runtime np.
template <typename T, typename Op, int NP>
__device__ __forceinline__ void reduce_core(const PtrTable &t, int np_rt, int ndst, size_t n, int cta, int nctas) {
  using V = VecOf<T>;
  const int np = NP > 0 ? NP : np_rt;
  bool aligned = true;
  for (int p = 0; p < np; ++p) aligned = aligned && (reinterpret_cast<uintptr_t>(t.src[p]) & 15) == 0;
  for (int q = 0; q < ndst; ++q) aligned = aligned && (reinterpret_cast<uintptr_t>(t.dst[q]) & 15) == 0;
  const size_t stride = static_cast<size_t>(nctas) * blockDim.x;
  const size_t tid = static_cast<size_t>(cta) * blockDim.x + threadIdx.x;
  size_t done = 0;
  if (aligned) {
    const size_t nvec = n / V::N;
    if (NP > 0) {
      const char *sp[NP > 0 ? NP : 1];
#pragma unroll
      for (int p = 0; p < NP; ++p) sp[p] = t.src[p];
      // vectors per thread in flight: enough bytes outstanding to cover the NVLink round trip
      constexpr int U = NP <= 2 ? 4 : (NP <= 4 ? 2 : 1);
      size_t i = tid;
      for (; i + (U - 1) * stride < nvec; i += U * stride) {
        Vec16 in[U][NP > 0 ? NP : 1];
#pragma unroll
        for (int u = 0; u < U; ++u)
#pragma unroll
          for (int p = 0; p < NP; ++p) in[u][p] = ld_relaxed_sys16(sp[p] + (i + u * stride) * 16);
        Vec16 out[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          typename V::A acc[V::N], x[V::N];
          V::unpack(in[u][0], acc);
#pragma unroll
          for (int p = 1; p < NP; ++p) {
            V::unpack(in[u][p], x);
#pragma unroll
            for (int e = 0; e < V::N; ++e) acc[e] = Op::apply(acc[e], x[e]);
          }
          out[u] = V::pack(acc);
        }
        for (int q = 0; q < ndst; ++q) {
          char *d = t.dst[q];
#pragma unroll
          for (int u = 0; u < U; ++u) st_relaxed_sys16(d + (i + u * stride) * 16, out[u]);
        }
      }
      for (; i < nvec; i += stride) {
        typename V::A acc[V::N], x[V::N];
        V::unpack(ld_relaxed_sys16(sp[0] + i * 16), acc);
#pragma unroll
        for (int p = 1; p < NP; ++p) {
          V::unpack(ld_relaxed_sys16(sp[p] + i * 16), x);
#pragma unroll
          for (int e = 0; e < V::N; ++e) acc[e] = Op::apply(acc[e], x[e]);
        }
        const Vec16 o = V::pack(acc);
        for (int q = 0; q < ndst; ++q) st_relaxed_sys16(t.dst[q] + i * 16, o);
      }
    } else {
      for (size_t i = tid; i < nvec; i += stride) {
        typename V::A acc[V::N], x[V::N];
        V::unpack(ld_relaxed_sys16(t.src[0] + i * 16), acc);
        for (int p = 1; p < np; ++p) {
          V::unpack(ld_relaxed_sys16(t.src[p] + i * 16), x);
#pragma unroll
          for (int e = 0; e < V::N; ++e) acc[e] = Op::apply(acc[e], x[e]);
        }
        const Vec16 o = V::pack(acc);
        for (int q = 0; q < ndst; ++q) st_relaxed_sys16(t.dst[q] + i * 16, o);
      }
    }
    done = nvec * V::N;
  }
  for (size_t i = done + tid; i < n; i += stride) {
    typename Tr<T>::A acc = Tr<T>::up(reinterpret_cast<const volatile T *>(t.src[0])[i]);
    for (int p = 1; p < np; ++p) acc = Op::apply(acc, Tr<T>::up(reinterpret_cast<const volatile T *>(t.src[p])[i]));
    const T o = Tr<T>::down(acc);
    for (int q = 0; q < ndst; ++q) reinterpret_cast<T *>(t.dst[q])[i] = o;
  }
}

template <typename T, typename Op>
__device__ __forceinline__ void reduce_np(const PtrTable &t, int np, int ndst, size_t n, int cta, int nctas) {
  switch (np) {
  case 2: reduce_core<T, Op, 2>(t, np, ndst, n, cta, nctas); break;
  case 4: reduce_core<T, Op, 4>(t, np, ndst, n, cta, nctas); break;
  case 8: reduce_core<T, Op, 8>(t, np, ndst, n, cta, nctas); break;
  default: reduce_core<T, Op, 0>(t, np, ndst, n, cta, nctas); break;
  }
}

// The one place where (dtype, function) select typed code.  All threads of
// the CTA call it with a table that is already visible (after __syncthreads).
static __device__ __noinline__ void reduce_dispatch(const PtrTable *t, int np, int ndst, size_t n, uint32_t dtype, uint32_t func,
                                             int cta, int nctas, uint32_t *err) {
  const bool sum = func == static_cast<uint32_t>(reduceFunction::SUM);
#define ACCL_RD(TYPE)                                                         \
  if (sum) reduce_np<TYPE, OpSum>(*t, np, ndst, n, cta, nctas);               \
  else reduce_np<TYPE, OpMax>(*t, np, ndst, n, cta, nctas);
  switch (static_cast<dataType>(dtype)) {
  case dataType::float32: ACCL_RD(float); break;
  case dataType::float16: ACCL_RD(__half); break;
  case dataType::bfloat16: ACCL_RD(__nv_bfloat16); break;
  case dataType::float64: ACCL_RD(double); break;
  case dataType::int32: ACCL_RD(int32_t); break;
  case dataType::int64: ACCL_RD(int64_t); break;
  default:
    if (threadIdx.x == 0) atomicOr(err, ARITH_ERROR);
    break;
  }
#undef ACCL_RD
}

// byte copy t->src[0] -> t->dst[0..ndst) (push / broadcast), 16-byte path when aligned
static __device__ __noinline__ void copy_dispatch(const PtrTable *t, int ndst, size_t bytes, int cta, int nctas) {
  const char *src = t->src[0];
  bool aligned = (reinterpret_cast<uintptr_t>(src) & 15) == 0;
  for (int q = 0; q < ndst; ++q) aligned = aligned && (reinterpret_cast<uintptr_t>(t->dst[q]) & 15) == 0;
  const size_t stride = static_cast<size_t>(nctas) * blockDim.x;
  const size_t tid = static_cast<size_t>(cta) * blockDim.x + threadIdx.x;
  size_t done = 0;
  if (aligned) {
    const size_t nvec = bytes / 16;
    size_t i = tid;
    for (; i + 3 * stride < nvec; i += 4 * stride) {
      Vec16 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = ld_relaxed_sys16(src + (i + u * stride) * 16);
      for (int q = 0; q < ndst; ++q) {
        char *d = t->dst[q];
#pragma unroll
        for (int u = 0; u < 4; ++u) st_relaxed_sys16(d + (i + u * stride) * 16, v[u]);
      }
    }
    for (; i < nvec; i += stride) {
      const Vec16 v = ld_relaxed_sys16(src + i * 16);
      for (int q = 0; q < ndst; ++q) st_relaxed_sys16(t->dst[q] + i * 16, v);
    }
    done = nvec * 16;
  }
  for (size_t i = done + tid; i < bytes; i += stride) {
    const char b = *reinterpret_cast<const volatile char *>(src + i);
    for (int q = 0; q < ndst; ++q) t->dst[q][i] = b;
  }
}

// single source / single destination copy without a table (whole-CTA helper)
__device__ __forceinline__ void copy_simple(char *dst, const char *src, size_t bytes, int cta, int nctas) {
  const bool aligned = ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0;
  const size_t stride = static_cast<size_t>(nctas) * blockDim.x;
  const size_t tid = static_cast<size_t>(cta) * blockDim.x + threadIdx.x;
  size_t done = 0;
  if (aligned) {
    const size_t nvec = bytes / 16;
    size_t i = tid;
    for (; i + 7 * stride < nvec; i += 8 * stride) {
      Vec16 v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) v[u] = ld_relaxed_sys16(src + (i + u * stride) * 16);
#pragma unroll
      for (int u = 0; u < 8; ++u) st_relaxed_sys16(dst + (i + u * stride) * 16, v[u]);
    }
    for (; i < nvec; i += stride) st_relaxed_sys16(dst + i * 16, ld_relaxed_sys16(src + i * 16));
    done = nvec * 16;
  }
  for (size_t i = done + tid; i < bytes; i += stride) dst[i] = *reinterpret_cast<const volatile char *>(src + i);
}

// ------------------------------------------------------------- NVLS bodies
enum class NvOp { add_f32, add_f16, add_bf16, max_f16, max_bf16, none };

__device__ __forceinline__ NvOp nvls_op(uint32_t dtype, uint32_t func) {
  const dataType t = static_cast<dataType>(dtype);
  const bool sum = func == static_cast<uint32_t>(reduceFunction::SUM);
  if (t == dataType::float32) return sum ? NvOp::add_f32 : NvOp::none; // no f32 max in the switch
  if (t == dataType::float16) return sum ? NvOp::add_f16 : NvOp::max_f16;
  if (t == dataType::bfloat16) return sum ? NvOp::add_bf16 : NvOp::max_bf16;
  return NvOp::none;
}

template <NvOp OP> __device__ __forceinline__ Vec16 nv_ld(const void *mc) {
  if (OP == NvOp::add_f32) return multimem_ld_reduce_add_f32(mc);
  if (OP == NvOp::add_f16) return multimem_ld_reduce_add_f16(mc);
  if (OP == NvOp::add_bf16) return multimem_ld_reduce_add_bf16(mc);
  if (OP == NvOp::max_f16) return multimem_ld_reduce_max_f16(mc);
  return multimem_ld_reduce_max_bf16(mc);
}

// out[i] = switch-reduce(in[i]) for vectors [v0, v1); out is a multicast
// address (two-shot allreduce) or a local address (reduce_scatter / reduce).
// U x 16 B per thread are in flight (in-switch reductions have a long round trip).
template <NvOp OP, bool MC_OUT, int U>
__device__ __forceinline__ void nvls_reduce_range(const char *mc_in, char *out, size_t v0, size_t v1, int cta, int nctas) {
  const size_t stride = static_cast<size_t>(nctas) * blockDim.x;
  size_t i = v0 + static_cast<size_t>(cta) * blockDim.x + threadIdx.x;
  for (; i + (U - 1) * stride < v1; i += U * stride) {
    Vec16 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) v[u] = nv_ld<OP>(mc_in + (i + u * stride) * 16);
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (MC_OUT) multimem_st16(out + (i + u * stride) * 16, v[u]);
      else st_stream(out + (i + u * stride) * 16, v[u]);
    }
  }
  for (; i < v1; i += stride) {
    const Vec16 v = nv_ld<OP>(mc_in + i * 16);
    if (MC_OUT) multimem_st16(out + i * 16, v);
    else st_stream(out + i * 16, v);
  }
}

template <NvOp OP, bool MC_OUT>
__device__ __forceinline__ void nvls_reduce_unroll(uint32_t unroll, const char *mc_in, char *out, size_t v0, size_t v1, int cta,
                                                   int nctas) {
  if (unroll == 4) nvls_reduce_range<OP, MC_OUT, 4>(mc_in, out, v0, v1, cta, nctas);
  else if (unroll == 2) nvls_reduce_range<OP, MC_OUT, 2>(mc_in, out, v0, v1, cta, nctas);
  else if (unroll == 16) nvls_reduce_range<OP, MC_OUT, 16>(mc_in, out, v0, v1, cta, nctas);
  else nvls_reduce_range<OP, MC_OUT, 8>(mc_in, out, v0, v1, cta, nctas);
}

template <bool MC_OUT>
__device__ __noinline__ void nvls_reduce_dispatch(NvOp op, uint32_t unroll, const char *mc_in, char *out, size_t v0, size_t v1, int cta,
                                                  int nctas) {
  switch (op) {
  case NvOp::add_f32: nvls_reduce_unroll<NvOp::add_f32, MC_OUT>(unroll, mc_in, out, v0, v1, cta, nctas); break;
  case NvOp::add_f16: nvls_reduce_unroll<NvOp::add_f16, MC_OUT>(unroll, mc_in, out, v0, v1, cta, nctas); break;
  case NvOp::add_bf16: nvls_reduce_unroll<NvOp::add_bf16, MC_OUT>(unroll, mc_in, out, v0, v1, cta, nctas); break;
  case NvOp::max_f16: nvls_reduce_unroll<NvOp::max_f16, MC_OUT>(unroll, mc_in, out, v0, v1, cta, nctas); break;
  case NvOp::max_bf16: nvls_reduce_unroll<NvOp::max_bf16, MC_OUT>(unroll, mc_in, out, v0, v1, cta, nctas); break;
  default: break;
  }
}

// local src -> multicast dst (allgather / bcast through the switch)
__device__ __forceinline__ void nvls_bcast_range(const char *src, char *mc_out, size_t nvec, int cta, int nctas) {
  const size_t stride = static_cast<size_t>(nctas) * blockDim.x;
  size_t i = static_cast<size_t>(cta) * blockDim.x + threadIdx.x;
  for (; i + 7 * stride < nvec; i += 8 * stride) {
    Vec16 v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) v[u] = ld_stream(src + (i + u * stride) * 16);
#pragma unroll
    for (int u = 0; u < 8; ++u) multimem_st16(mc_out + (i + u * stride) * 16, v[u]);
  }
  for (; i < nvec; i += stride) multimem_st16(mc_out + i * 16, ld_stream(src + i * 16));
}

// generic element conversion through float/double (cast lanes); slow path
__device__ __forceinline__ double load_as_double(const void *p, uint32_t dtype, size_t i) {
  switch (static_cast<dataType>(dtype)) {
  case dataType::float32: return reinterpret_cast<const float *>(p)[i];
  case dataType::float64: return reinterpret_cast<const double *>(p)[i];
  case dataType::float16: return __half2float(reinterpret_cast<const __half *>(p)[i]);
  case dataType::bfloat16: return __bfloat162float(reinterpret_cast<const __nv_bfloat16 *>(p)[i]);
  case dataType::float8_e4m3: return static_cast<float>(reinterpret_cast<const __nv_fp8_e4m3 *>(p)[i]);
  case dataType::float8_e5m2: return static_cast<float>(reinterpret_cast<const __nv_fp8_e5m2 *>(p)[i]);
  case dataType::int32: return reinterpret_cast<const int32_t *>(p)[i];
  case dataType::int64: return static_cast<double>(reinterpret_cast<const int64_t *>(p)[i]);
  default: return 0.0;
  }
}
__device__ __forceinline__ void store_from_double(void *p, uint32_t dtype, size_t i, double v) {
  switch (static_cast<dataType>(dtype)) {
  case dataType::float32: reinterpret_cast<float *>(p)[i] = static_cast<float>(v); break;
  case dataType::float64: reinterpret_cast<double *>(p)[i] = v; break;
  case dataType::float16: reinterpret_cast<__half *>(p)[i] = __float2half_rn(static_cast<float>(v)); break;
  case dataType::bfloat16: reinterpret_cast<__nv_bfloat16 *>(p)[i] = __float2bfloat16_rn(static_cast<float>(v)); break;
  case dataType::float8_e4m3: reinterpret_cast<__nv_fp8_e4m3 *>(p)[i] = __nv_fp8_e4m3(static_cast<float>(v)); break;
  case dataType::float8_e5m2: reinterpret_cast<__nv_fp8_e5m2 *>(p)[i] = __nv_fp8_e5m2(static_cast<float>(v)); break;
  case dataType::int32: reinterpret_cast<int32_t *>(p)[i] = static_cast<int32_t>(v); break;
  case dataType::int64: reinterpret_cast<int64_t *>(p)[i] = static_cast<int64_t>(v); break;
  default: break;
  }
}

} // namespace k
} // namespace cuda
} // namespace accl
