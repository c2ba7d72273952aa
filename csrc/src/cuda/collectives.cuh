// Collective and primitive bodies executed by `run_work` (see kernels.cuh).
// Two protocol families, selected per call exactly like the reference
// firmware does (eager iff small, or compressed; ccl_offload_control.c:587,
// 808,1878):
//   * eager: data is pushed into the destination's slot ring (the RX
//     buffers), flagged with a per-(channel, src) sequence counter, consumed
//     and acknowledged (credit return).  One network hop, works for every
//     dtype / wire-dtype combination, segmented by slot size.
//   * rendezvous: peers exchange buffer offsets on the sync pads (the
//     address hand-shake), then move data straight between user buffers with
//     multimem (in-switch reduce/broadcast) or peer loads/stores, and meet
//     again on the pads.
#pragma once
#include "kernels.cuh"

namespace accl {
namespace cuda {
namespace k {

// ---------------------------------------------------------------- helpers
__device__ __forceinline__ uint32_t esize(uint32_t dtype) { return esize_of(dtype); }
__device__ __forceinline__ bool is_fp8_dt(uint32_t dtype) {
  return dtype == static_cast<uint32_t>(dataType::float8_e4m3) || dtype == static_cast<uint32_t>(dataType::float8_e5m2);
}
// bytes of n elements in wire representation (block-scaled fp8 appends fp32 scales, 4-byte aligned)
__device__ __forceinline__ uint64_t wire_bytes(uint32_t wdt, uint32_t rl, uint64_t n) {
  uint64_t b = n * esize(wdt);
  if (is_fp8_dt(wdt) && rl) b = ((b + 3) & ~3ull) + 4 * ((n + (1u << rl) - 1) >> rl);
  return b;
}

// Convert n elements src(src_t) -> dst(dst_t) with the whole CTA.  Identical
// types take the vector copy path.  A block-scaled fp8 destination gets one
// scale per 2^rl elements (computed by the 32 lanes of a warp when rl == 5).
__device__ __forceinline__ void cast_copy(void *dst, uint32_t dst_t, const void *src, uint32_t src_t, size_t n, uint32_t rl) {
  if (dst_t == src_t && !(is_fp8_dt(dst_t) && rl)) {
    copy_simple(static_cast<char *>(dst), static_cast<const char *>(src), n * esize(dst_t), 0, 1);
    return;
  }
  const bool dst_scaled = is_fp8_dt(dst_t) && rl, src_scaled = is_fp8_dt(src_t) && rl;
  const float *src_scales = reinterpret_cast<const float *>(static_cast<const char *>(src) + ((n * esize(src_t) + 3) & ~3ull));
  float *dst_scales = reinterpret_cast<float *>(static_cast<char *>(dst) + ((n * esize(dst_t) + 3) & ~3ull));
  if (dst_scaled && rl == 5) {
    const float fmax = dst_t == static_cast<uint32_t>(dataType::float8_e4m3) ? 448.f : 57344.f;
    const size_t nblk = (n + 31) / 32;
    for (size_t b = threadIdx.x / 32; b < nblk; b += blockDim.x / 32) {
      const size_t i = b * 32 + (threadIdx.x & 31);
      float x = 0.f;
      if (i < n) x = static_cast<float>(load_as_double(src, src_t, i)) * (src_scaled ? src_scales[i >> rl] : 1.f);
      float m = fabsf(x);
#pragma unroll
      for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
      const float scale = m > 0.f ? m / fmax : 1.f;
      if (i < n) store_from_double(dst, dst_t, i, x / scale);
      if ((threadIdx.x & 31) == 0) dst_scales[b] = scale;
    }
    return;
  }
  for (size_t i = threadIdx.x; i < n; i += blockDim.x) {
    double x = load_as_double(src, src_t, i);
    if (src_scaled) x *= src_scales[i >> rl];
    store_from_double(dst, dst_t, i, x);
  }
}

__device__ __forceinline__ double wire_load(const void *p, uint32_t wdt, uint32_t rl, size_t n, size_t i) {
  double x = load_as_double(p, wdt, i);
  if (is_fp8_dt(wdt) && rl)
    x *= reinterpret_cast<const float *>(static_cast<const char *>(p) + ((n * esize(wdt) + 3) & ~3ull))[i >> rl];
  return x;
}

// ------------------------------------------------------------ local calls
__device__ __noinline__ void op_copy(const Ctx &c) {
  const WorkItem &it = c.it;
  const uint32_t cf = it.desc.compression_flags;
  const uint32_t st = (cf & 1) ? it.cdtype : it.udtype, dt = (cf & 4) ? it.cdtype : it.udtype;
  const char *src = c.heap(c.w.rank) + it.desc.addr0();
  char *dst = c.heap(c.w.rank) + it.desc.addr2();
  const size_t n = it.desc.count;
  if (st == dt) {
    copy_simple(dst, src, n * esize(st), c.cta, c.nctas);
  } else {
    const size_t stride = static_cast<size_t>(c.nctas) * blockDim.x;
    for (size_t i = static_cast<size_t>(c.cta) * blockDim.x + threadIdx.x; i < n; i += stride)
      store_from_double(dst, dt, i, load_as_double(src, st, i));
  }
}

__device__ __noinline__ void op_combine(const Ctx &c) {
  const WorkItem &it = c.it;
  const uint32_t cf = it.desc.compression_flags;
  const uint32_t t0 = (cf & 1) ? it.cdtype : it.udtype, t1 = (cf & 2) ? it.cdtype : it.udtype,
                 tr = (cf & 4) ? it.cdtype : it.udtype;
  const char *a = c.heap(c.w.rank) + it.desc.addr0();
  const char *b = c.heap(c.w.rank) + it.desc.addr1();
  char *d = c.heap(c.w.rank) + it.desc.addr2();
  const size_t n = it.desc.count;
  if (t0 == t1 && t1 == tr) {
    __syncthreads();
    if (threadIdx.x == 0) {
      c.tab->src[0] = a;
      c.tab->src[1] = b;
      c.tab->dst[0] = d;
    }
    __syncthreads();
    reduce_dispatch(c.tab, 2, 1, n, t0, it.desc.function, c.cta, c.nctas, c.err);
    return;
  }
  const uint32_t at = it.arith_compressed ? it.cdtype : it.udtype;
  const bool sum = it.desc.function == static_cast<uint32_t>(reduceFunction::SUM);
  const size_t stride = static_cast<size_t>(c.nctas) * blockDim.x;
  for (size_t i = static_cast<size_t>(c.cta) * blockDim.x + threadIdx.x; i < n; i += stride) {
    double x = load_as_double(a, t0, i), y = load_as_double(b, t1, i);
    double r = sum ? x + y : (x > y ? x : y);
    if (at != static_cast<uint32_t>(dataType::float64)) r = static_cast<float>(r);
    store_from_double(d, tr, i, r);
  }
}

// ------------------------------------------------------------ eager slots
// The slot-ring handshake with one peer (global rank) on channel `ch`, per thread: message v from me to `peer` goes
// into slot v % depth of my column of its ring, once the peer has handed back the credit for message v - depth; a
// header describes it and the release of `egr_sig` announces it.  The counters, the header format and the slot
// addressing are known only to these helpers.
constexpr uint32_t EGR_LOST = 0xFFFFFFFFu; // egr_arrive: the message did not come in time

// may message sent + 1 be written? (its slot held message sent + 1 - depth, which must have been consumed)
__device__ __forceinline__ bool egr_credit_ok(const Ctx &c, uint32_t ch, uint32_t peer) {
  const uint32_t v = c.me->egr_sent[ch][peer] + 1;
  return v <= c.w.egr_depth || static_cast<int32_t>(ld_acquire_sys(&c.me->egr_ack[ch][peer]) - (v - c.w.egr_depth)) >= 0;
}

// wait for the credit of the next message; returns its number (DEQUEUE_BUFFER_TIMEOUT_ERROR on timeout)
__device__ __forceinline__ uint32_t egr_credit_wait(const Ctx &c, uint32_t ch, uint32_t peer) {
  const uint32_t v = c.me->egr_sent[ch][peer] + 1;
  if (v > c.w.egr_depth) wait_ge(&c.me->egr_ack[ch][peer], v - c.w.egr_depth, c, DEQUEUE_BUFFER_TIMEOUT_ERROR);
  return v;
}

// where message v to `peer` goes
__device__ __forceinline__ char *egr_tx_slot(const Ctx &c, uint32_t ch, uint32_t peer, uint32_t v) {
  return c.heap(peer) + egr_slot_off(c.w, ch, v % c.w.egr_depth, c.w.rank);
}

// Announce message v (its payload is in the slot): header, then the release of the arrival counter.  `fence` adds a
// fence.acq_rel.sys between the two.  egr_collective asks for it, because other threads of its CTA wrote the payload.
// egr_p2p's payload is written by the whole CTA as well, yet it has never issued the fence: the difference is
// inherited, not derived, and is kept as it is.
__device__ __forceinline__ void egr_publish(const Ctx &c, uint32_t ch, uint32_t peer, uint32_t v, uint32_t tag, uint32_t wire_t,
                                            uint32_t elems, bool fence) {
  Ctrl *pc = c.ctrl(peer);
  EgrHdr *h = &pc->egr_hdr[ch][v % c.w.egr_depth][c.w.rank];
  st_relaxed_sys(&h->tag, tag);
  st_relaxed_sys(&h->bytes, static_cast<uint32_t>(wire_bytes(wire_t, c.it.ratio_log, elems)));
  st_relaxed_sys(&h->elems, elems);
  st_relaxed_sys(&h->kind, c.it.desc.scenario | (wire_t << 8));
  if (fence) fence_acq_rel_sys();
  st_release_sys(&pc->egr_sig[ch][c.w.rank], v);
  c.me->egr_sent[ch][peer] = v;
}

// has the next message of `peer` arrived?
__device__ __forceinline__ bool egr_arrived(const Ctx &c, uint32_t ch, uint32_t peer) {
  return static_cast<int32_t>(ld_acquire_sys(&c.me->egr_sig[ch][peer]) - (c.me->egr_expect[ch][peer] + 1)) >= 0;
}

// Wait for the next message of `peer` and check its header against the tag, element count and wire dtype this call
// expects.  Returns its number, or EGR_LOST on timeout; the message counts as consumed either way.
__device__ __forceinline__ uint32_t egr_arrive(const Ctx &c, uint32_t ch, uint32_t peer, uint32_t want_tag, uint32_t want_elems,
                                               uint32_t wire_t) {
  const uint32_t e = c.me->egr_expect[ch][peer] + 1;
  const bool ok = wait_ge(&c.me->egr_sig[ch][peer], e, c, RECEIVE_TIMEOUT_ERROR);
  if (ok) {
    const EgrHdr *h = &c.me->egr_hdr[ch][e % c.w.egr_depth][peer];
    const uint32_t tag = ld_relaxed_sys(&h->tag);
    if (want_tag != TAG_ANY && tag != TAG_ANY && tag != want_tag) atomicOr(c.err, DMA_TAG_MISMATCH_ERROR);
    if (ld_relaxed_sys(&h->elems) != want_elems) atomicOr(c.err, DMA_NOT_EXPECTED_BTT_ERROR);
    if ((ld_relaxed_sys(&h->kind) >> 8) != wire_t) atomicOr(c.err, COMPRESSION_ERROR);
  }
  c.me->egr_expect[ch][peer] = e;
  return ok ? e : EGR_LOST;
}

// where message e from `peer` is
__device__ __forceinline__ const char *egr_rx_slot(const Ctx &c, uint32_t ch, uint32_t peer, uint32_t e) {
  return c.heap(c.w.rank) + egr_slot_off(c.w, ch, e % c.w.egr_depth, peer);
}

// the last consumed message of `peer` has been read out: hand its credit back
__device__ __forceinline__ void egr_credit_return(const Ctx &c, uint32_t ch, uint32_t peer) {
  st_relaxed_sys(&c.ctrl(peer)->egr_ack[ch][c.w.rank], c.me->egr_expect[ch][peer]);
}

// segment geometry shared by both ends: the block of `count` elements is cut
// into nctas equal parts (one per channel), each part into slot-sized segments
__device__ __forceinline__ uint32_t egr_seg_elems(const Ctx &c, uint32_t wire_t) {
  const uint32_t rl = c.it.ratio_log;
  if (is_fp8_dt(wire_t) && rl) return c.w.egr_slot_bytes / ((1u << rl) + 4) * (1u << rl);
  return c.w.egr_slot_bytes / esize(wire_t);
}

struct EgrPlan {
  size_t part_off, part_elems;
  uint32_t seg;
};
__device__ __forceinline__ EgrPlan egr_plan(const Ctx &c, size_t count, uint32_t wire_t) {
  EgrPlan p;
  const size_t per = (count + c.nctas - 1) / c.nctas;
  // keep parts 16-byte aligned for the vector paths
  const size_t al = 16;
  const size_t per_al = (per + al - 1) / al * al;
  p.part_off = static_cast<size_t>(c.cta) * per_al;
  p.part_elems = p.part_off >= count ? 0 : (count - p.part_off < per_al ? count - p.part_off : per_al);
  p.seg = egr_seg_elems(c, wire_t);
  return p;
}

// reduce my local block with the slots of all peers into dst (comm-rank order
// so every rank produces bit-identical sums)
__device__ __forceinline__ void egr_reduce_consume(const Ctx &c, const char *local, uint32_t local_t, const char *const *slots,
                                                    uint32_t wire_t, char *dst, uint32_t dst_t, uint32_t n) {
  const uint32_t P = c.P();
  const uint32_t rl = c.it.ratio_log;
  if (local_t == wire_t && wire_t == dst_t && !is_fp8_dt(wire_t)) {
    __syncthreads();
    if (threadIdx.x < P) {
      const uint32_t q = threadIdx.x;
      c.tab->src[q] = q == c.r() ? local : slots[q];
    }
    if (threadIdx.x == 0) c.tab->dst[0] = dst;
    __syncthreads();
    reduce_dispatch(c.tab, static_cast<int>(P), 1, n, wire_t, c.it.desc.function, 0, 1, c.err);
    return;
  }
  const bool sum = c.it.desc.function == static_cast<uint32_t>(reduceFunction::SUM);
  const uint32_t at = c.it.arith_compressed ? c.it.cdtype : c.it.udtype;
  for (size_t i = threadIdx.x; i < n; i += blockDim.x) {
    double acc = 0;
    for (uint32_t q = 0; q < P; ++q) {
      const double x = q == c.r() ? load_as_double(local, local_t, i) : wire_load(slots[q], wire_t, rl, n, i);
      if (q == 0) acc = x;
      else acc = sum ? acc + x : (acc > x ? acc : x);
      if (at == static_cast<uint32_t>(dataType::float16)) acc = __half2float(__float2half_rn(static_cast<float>(acc)));
      else if (at != static_cast<uint32_t>(dataType::float64)) acc = static_cast<float>(acc);
    }
    store_from_double(dst, dst_t, i, acc);
  }
}

// One generic eager exchange.  Per segment: push what each peer needs from
// me, wait for what I need from each peer, consume, acknowledge.  Flag
// traffic (credits, headers, arrival counters, acks) is handled by one thread
// per peer in parallel so the latency does not grow with the world size.
__device__ __noinline__ void egr_collective(const Ctx &c, Pattern pat, uint32_t *s_tmp, const char **s_slots) {
  const WorkItem &it = c.it;
  const uint32_t P = c.P(), me = c.r(), root = it.desc.root_src_dst;
  const uint32_t cf = it.desc.compression_flags;
  const uint32_t src_t = (cf & 1) ? it.cdtype : it.udtype, dst_t = (cf & 4) ? it.cdtype : it.udtype;
  const uint32_t wire_t = (cf & 8) ? it.cdtype : it.udtype;
  const size_t count = it.desc.count;
  const char *src = c.heap(c.w.rank) + it.desc.addr0();
  char *dst = c.heap(c.w.rank) + it.desc.addr2();
  if (pat == PAT_BCAST) dst = const_cast<char *>(src); // bcast works in place on addr0
  const EgrPlan pl = egr_plan(c, count, wire_t);
  const uint32_t tag = it.desc.tag;
  const size_t se = esize(src_t), de = esize(dst_t);
  const uint32_t ch = static_cast<uint32_t>(c.cta);
  __shared__ uint32_t s_v[ACCL_MAX_RANKS];
  (void)s_tmp;
  const uint32_t t = threadIdx.x;
  const Roles ro{pat, P, me, root};
  const bool same_src = ro.same_src();

  for (size_t off = 0; off < pl.part_elems; off += pl.seg) {
    const uint32_t n = static_cast<uint32_t>(pl.part_elems - off < pl.seg ? pl.part_elems - off : pl.seg);
    const size_t e0 = pl.part_off + off; // element offset inside a block
    __syncthreads();
    if (t < ACCL_MAX_RANKS) s_slots[t] = nullptr;
    // ---- push phase: credits in parallel
    if (t < P && ro.pushes_to(t)) s_v[t] = egr_credit_wait(c, ch, c.g(t));
    __syncthreads();
    if (same_src && src_t == wire_t && !is_fp8_dt(wire_t)) {
      // one read of my block, stores fan out to every destination slot
      int nd = 0;
      if (t == 0) {
        for (uint32_t k = 1; k < P; ++k) {
          const uint32_t q = (me + k) % P;
          if (ro.pushes_to(q)) c.tab->dst[nd++] = egr_tx_slot(c, ch, c.g(q), s_v[q]);
        }
        c.tab->src[0] = src + e0 * se;
        *s_tmp = static_cast<uint32_t>(nd);
      }
      __syncthreads();
      nd = static_cast<int>(*s_tmp);
      if (nd) copy_dispatch(c.tab, nd, static_cast<size_t>(n) * se, 0, 1);
    } else {
      for (uint32_t k = 1; k < P; ++k) {
        const uint32_t q = (me + k) % P; // stagger destinations across ranks
        if (!ro.pushes_to(q)) continue;
        const char *from = same_src ? src + e0 * se : src + (static_cast<size_t>(q) * count + e0) * se;
        cast_copy(egr_tx_slot(c, ch, c.g(q), s_v[q]), wire_t, from, src_t, n, it.ratio_log);
      }
    }
    __syncthreads();
    // headers + arrival flags in parallel; the payload was written by other threads of this CTA (ordered by the barrier above)
    if (t < P && ro.pushes_to(t)) egr_publish(c, ch, c.g(t), s_v[t], tag, wire_t, n, true);
    // ---- wait phase: one thread per expected peer
    if (t < P && ro.expects_from(t)) {
      const uint32_t peer = c.g(t), e = egr_arrive(c, ch, peer, tag, n, wire_t);
      if (e != EGR_LOST) s_slots[t] = egr_rx_slot(c, ch, peer, e);
    }
    __syncthreads();
    bool ok = *c.err == 0;
    // ---- consume phase
    if (ok) {
      switch (pat) {
      case PAT_ALLREDUCE:
        egr_reduce_consume(c, src + e0 * se, src_t, s_slots, wire_t, dst + e0 * de, dst_t, n);
        break;
      case PAT_REDUCE_SCATTER:
        egr_reduce_consume(c, src + (static_cast<size_t>(me) * count + e0) * se, src_t, s_slots, wire_t, dst + e0 * de, dst_t, n);
        break;
      case PAT_REDUCE:
        if (me == root) egr_reduce_consume(c, src + e0 * se, src_t, s_slots, wire_t, dst + e0 * de, dst_t, n);
        break;
      case PAT_ALLGATHER: case PAT_GATHER: case PAT_ALLTOALL:
        if (pat != PAT_GATHER || me == root)
          for (uint32_t q = 0; q < P; ++q) {
            char *to = dst + (static_cast<size_t>(q) * count + e0) * de;
            if (q == me) {
              const char *own = pat == PAT_ALLTOALL ? src + (static_cast<size_t>(me) * count + e0) * se : src + e0 * se;
              cast_copy(to, dst_t, own, src_t, n, it.ratio_log);
            } else if (s_slots[q]) {
              cast_copy(to, dst_t, s_slots[q], wire_t, n, it.ratio_log);
            }
          }
        break;
      case PAT_BCAST:
        if (me != root && s_slots[root]) cast_copy(dst + e0 * se, src_t, s_slots[root], wire_t, n, it.ratio_log);
        break;
      case PAT_SCATTER:
        if (me == root) cast_copy(dst + e0 * de, dst_t, src + (static_cast<size_t>(me) * count + e0) * se, src_t, n, it.ratio_log);
        else if (s_slots[root]) cast_copy(dst + e0 * de, dst_t, s_slots[root], wire_t, n, it.ratio_log);
        break;
      }
    }
    // ---- credits back to the senders
    __syncthreads();
    if (t < P && s_slots[t]) egr_credit_return(c, ch, c.g(t));
  }
  __syncthreads();
}

// Eager point-to-point: CTA 0 moves the message segment by segment through channel 0 of the slot ring, its thread 0
// keeps the handshake.  Starts `progress` elements in and returns how far it got: the element count when done (or when
// a segment did not arrive in time, with the error set).  `park`: return early instead of blocking at the first
// missing credit (send) or segment (recv), so that the engine can step other calls and come back.
__device__ __noinline__ unsigned long long egr_p2p(const Ctx &c, bool sending, bool park, unsigned long long progress, uint32_t *s_tmp) {
  const WorkItem &it = c.it;
  if (c.cta != 0) return progress;
  const uint32_t cf = it.desc.compression_flags;
  const uint32_t src_t = (cf & 1) ? it.cdtype : it.udtype, dst_t = (cf & 4) ? it.cdtype : it.udtype;
  const uint32_t wire_t = (cf & 8) ? it.cdtype : it.udtype;
  const uint32_t peer = c.g(it.desc.root_src_dst);
  const unsigned long long count = it.desc.count;
  const uint32_t seg = egr_seg_elems(c, wire_t);
  while (progress < count) {
    const uint32_t n = static_cast<uint32_t>(count - progress < seg ? count - progress : seg);
    __syncthreads(); // s_tmp may still be read by stragglers of the previous step
    if (park) {
      if (threadIdx.x == 0) *s_tmp = sending ? egr_credit_ok(c, 0, peer) : egr_arrived(c, 0, peer);
      __syncthreads();
      if (!*s_tmp) return progress;
      __syncthreads();
    }
    if (threadIdx.x == 0) *s_tmp = sending ? egr_credit_wait(c, 0, peer) : egr_arrive(c, 0, peer, it.desc.tag, n, wire_t);
    __syncthreads();
    const uint32_t v = *s_tmp;
    if (sending) {
      cast_copy(egr_tx_slot(c, 0, peer, v), wire_t, c.heap(c.w.rank) + it.desc.addr0() + progress * esize(src_t), src_t, n,
                it.ratio_log);
      __syncthreads();
      if (threadIdx.x == 0) egr_publish(c, 0, peer, v, it.desc.tag, wire_t, n, false);
    } else {
      if (v == EGR_LOST) return count;
      cast_copy(c.heap(c.w.rank) + it.desc.addr2() + progress * esize(dst_t), dst_t, egr_rx_slot(c, 0, peer, v), wire_t, n,
                it.ratio_log);
      __syncthreads();
      if (threadIdx.x == 0) egr_credit_return(c, 0, peer);
    }
    __syncthreads();
    progress += n;
  }
  return progress;
}

// ------------------------------------------------------ rendezvous bodies
__device__ __forceinline__ bool all_equal(const uint64_t *v, uint32_t P) {
  bool eq = true;
  for (uint32_t q = 1; q < P; ++q) eq = eq && v[q] == v[0];
  return eq;
}

// fill the CTA's pointer table: src[k] / dst[k] for k < P, rotated so that my
// own buffers come first (staggers the peers each rank touches first)
__device__ __forceinline__ void fill_table(const Ctx &c, const uint64_t *s_off0, const uint64_t *s_off2, uint64_t src_add,
                                           uint64_t dst_add, bool rotate) {
  __syncthreads();
  if (threadIdx.x < c.P()) {
    const uint32_t k = threadIdx.x;
    const uint32_t q = rotate ? (c.r() + k) % c.P() : k;
    if (s_off0) c.tab->src[k] = c.heap(c.g(q)) + s_off0[q] + src_add;
    if (s_off2) c.tab->dst[k] = c.heap(c.g(q)) + s_off2[q] + dst_add;
  }
  __syncthreads();
}

// allreduce, two-shot.  NVLS: the switch reduces my shard (multimem.ld_reduce)
// and broadcasts it (multimem.st).  P2P: pull my shard from every peer,
// reduce on the SM, store it into every peer's destination.
// `rvb_*` are the data phases between the entry and the exit meeting, dispatched by `run_body` (run_work.cuh):
// the direct-launch kernel brackets them with chan_sync, the persistent engine runs them as moves on its worker CTAs.
__device__ __noinline__ void rvb_allreduce(const Ctx &c, const uint64_t *s_off0, const uint64_t *s_off2) {
  const WorkItem &it = c.it;
  const uint32_t P = c.P(), me = c.r();
  const uint32_t dt = it.udtype;
  const size_t count = it.desc.count, es = esize(dt);
  const size_t per_vec = 16 / es;
  const size_t nvec = count / per_vec;
  const size_t shard = (nvec + P - 1) / P;
  const size_t v0 = static_cast<size_t>(me) * shard < nvec ? static_cast<size_t>(me) * shard : nvec;
  const size_t v1 = v0 + shard < nvec ? v0 + shard : nvec;
  const NvOp nop = nvls_op(dt, it.desc.function);
  const bool sym = all_equal(s_off0, P) && all_equal(s_off2, P) && (s_off0[0] & 15) == 0 && (s_off2[0] & 15) == 0;
  const bool nv = (it.flags & WF_USE_MC) && it.algo == ALGO_NVLS && nop != NvOp::none && sym;
  if (nv) {
    nvls_reduce_dispatch<true>(nop, it.nvls_unroll, c.w.mc + s_off0[0], c.w.mc + s_off2[0], v0, v1, c.cta, c.nctas);
  } else {
    fill_table(c, s_off0, s_off2, v0 * 16, v0 * 16, true);
    reduce_dispatch(c.tab, static_cast<int>(P), static_cast<int>(P), (v1 - v0) * per_vec, dt, it.desc.function, c.cta,
                    c.nctas, c.err);
  }
  // sub-vector tail: communicator rank 0 handles it element-wise for everybody
  const size_t tail0 = nvec * per_vec;
  if (tail0 < count && me == 0 && c.cta == 0) {
    fill_table(c, s_off0, s_off2, tail0 * es, tail0 * es, false);
    reduce_dispatch(c.tab, static_cast<int>(P), static_cast<int>(P), count - tail0, dt, it.desc.function, 0, 1, c.err);
  }
}

// every rank pulls everything and reduces locally: no second hop, for
// messages too big for the slots but small enough that latency dominates
__device__ __noinline__ void rvb_allreduce_oneshot(const Ctx &c, const uint64_t *s_off0, const uint64_t *s_off2) {
  const WorkItem &it = c.it;
  const uint32_t P = c.P();
  // In place on ANY rank (source == destination): that rank's result stores would race with the peers' reads of
  // its source.  The exchanged offsets are identical everywhere, so all ranks take the two-shot body together
  // (only a shard's owner writes it, after having read it).
  bool inplace = false;
  for (uint32_t q = 0; q < P; ++q) inplace = inplace || s_off0[q] == s_off2[q];
  if (inplace) {
    rvb_allreduce(c, s_off0, s_off2);
    return;
  }
  const NvOp nop = nvls_op(it.udtype, it.desc.function);
  const size_t es = esize(it.udtype), per_vec = 16 / es, nvec = it.desc.count / per_vec;
  const bool sym = all_equal(s_off0, P) && (s_off0[0] & 15) == 0 && (it.desc.addr2() & 15) == 0;
  size_t done = 0;
  if ((it.flags & WF_USE_MC) && nop != NvOp::none && sym) {
    nvls_reduce_dispatch<false>(nop, it.nvls_unroll, c.w.mc + s_off0[0], c.heap(c.w.rank) + it.desc.addr2(), 0, nvec, c.cta, c.nctas);
    done = nvec * per_vec;
  }
  if (done < it.desc.count) {
    fill_table(c, s_off0, nullptr, done * es, 0, false); // communicator-rank order: identical sums everywhere
    if (threadIdx.x == 0) c.tab->dst[0] = c.heap(c.w.rank) + it.desc.addr2() + done * es;
    __syncthreads();
    reduce_dispatch(c.tab, static_cast<int>(P), 1, it.desc.count - done, it.udtype, it.desc.function, c.cta, c.nctas, c.err);
  }
}

__device__ __noinline__ void rvb_reduce_scatter(const Ctx &c, const uint64_t *s_off0, const uint64_t *s_off2) {
  (void)s_off2;
  const WorkItem &it = c.it;
  const uint32_t P = c.P(), me = c.r();
  const size_t count = it.desc.count, es = esize(it.udtype);
  const size_t blk_bytes = count * es;
  const NvOp nop = nvls_op(it.udtype, it.desc.function);
  char *dst = c.heap(c.w.rank) + it.desc.addr2();
  const bool sym = all_equal(s_off0, P) && ((s_off0[0] + me * blk_bytes) & 15) == 0 && (it.desc.addr2() & 15) == 0;
  size_t done = 0;
  if ((it.flags & WF_USE_MC) && it.algo == ALGO_NVLS && nop != NvOp::none && sym) {
    const size_t nvec = blk_bytes / 16;
    nvls_reduce_dispatch<false>(nop, it.nvls_unroll, c.w.mc + s_off0[0] + me * blk_bytes, dst, 0, nvec, c.cta, c.nctas);
    done = nvec * 16 / es;
  }
  if (done < count) {
    fill_table(c, s_off0, nullptr, me * blk_bytes + done * es, 0, true);
    if (threadIdx.x == 0) c.tab->dst[0] = dst + done * es;
    __syncthreads();
    reduce_dispatch(c.tab, static_cast<int>(P), 1, count - done, it.udtype, it.desc.function, c.cta, c.nctas, c.err);
  }
}

__device__ __noinline__ void rv_bcast_pipelined(const Ctx &c, const uint64_t *s_off);

// push-style data movement shared by allgather / bcast / scatter / gather / alltoall.
// `stepwise_ok`: the caller can run the pipelined broadcast, which meets the peers between chunks (direct launches
// only: inside the engine every wait must be a parked step, so it takes the single-pass body).
__device__ __noinline__ void rvb_move(const Ctx &c, Pattern pat, const uint64_t *s_off0, const uint64_t *s_off2, bool stepwise_ok) {
  (void)s_off0;
  const WorkItem &it = c.it;
  const uint32_t P = c.P(), me = c.r(), root = it.desc.root_src_dst;
  const size_t blk = static_cast<size_t>(it.desc.count) * esize(it.udtype);
  const char *src = c.heap(c.w.rank) + it.desc.addr0();
  const bool mc_ok = (it.flags & WF_USE_MC) && it.algo == ALGO_NVLS && all_equal(s_off2, P) && (blk & 15) == 0 &&
                     (s_off2[0] & 15) == 0 && (it.desc.addr0() & 15) == 0;
  bool bcast_pipelined = stepwise_ok && pat == PAT_BCAST && P >= 3 && blk >= (128u << 20) && (blk & 15) == 0;
  for (uint32_t q = 0; q < P; ++q) bcast_pipelined = bcast_pipelined && (s_off2[q] & 15) == 0;
  switch (pat) {
  case PAT_ALLGATHER:
    if (mc_ok) {
      nvls_bcast_range(src, c.w.mc + s_off2[0] + me * blk, blk / 16, c.cta, c.nctas);
    } else {
      fill_table(c, nullptr, s_off2, 0, me * blk, true);
      if (threadIdx.x == 0) c.tab->src[0] = src;
      __syncthreads();
      copy_dispatch(c.tab, static_cast<int>(P), blk, c.cta, c.nctas);
    }
    break;
  case PAT_BCAST:
    if (bcast_pipelined) {
      rv_bcast_pipelined(c, s_off2);
    } else if (me == root) {
      if (mc_ok) {
        // the multicast store also rewrites the root's own copy with identical bytes
        nvls_bcast_range(src, c.w.mc + s_off2[0], blk / 16, c.cta, c.nctas);
      } else {
        fill_table(c, nullptr, s_off2, 0, 0, true); // dst[0] is my own buffer: skip it
        if (threadIdx.x == 0) {
          c.tab->src[0] = src;
          for (uint32_t k = 1; k < P; ++k) c.tab->dst[k - 1] = c.tab->dst[k];
        }
        __syncthreads();
        copy_dispatch(c.tab, static_cast<int>(P) - 1, blk, c.cta, c.nctas);
      }
    }
    break;
  case PAT_SCATTER:
    if (me == root)
      for (uint32_t k = 0; k < P; ++k) {
        // CTAs visit the destinations in different orders: all P switch ports are fed at once
        // instead of bursting one block at a time into a single port
        const uint32_t q = (me + k + static_cast<uint32_t>(c.cta)) % P;
        copy_simple(c.heap(c.g(q)) + s_off2[q], src + q * blk, blk, c.cta, c.nctas);
      }
    break;
  case PAT_GATHER:
    copy_simple(c.heap(c.g(root)) + s_off2[root] + me * blk, src, blk, c.cta, c.nctas);
    break;
  case PAT_ALLTOALL:
    for (uint32_t k = 0; k < P; ++k) {
      const uint32_t q = (me + k + static_cast<uint32_t>(c.cta)) % P;
      copy_simple(c.heap(c.g(q)) + s_off2[q] + me * blk, src + q * blk, blk, c.cta, c.nctas);
    }
    break;
  default: break;
  }
}

// ---------------------------------------------------------------- alltoallv
// The counts of an alltoallv live in device memory (int64: P send counts, then P receive counts, in elements).  At
// the entry meeting a rank publishes the heap offset of its counts in the off0 slot (the push bodies never read a
// peer's source offset) and its receive buffer in off2.  A rank whose counts fail the checks only it can make (a
// negative count, more than its buffers hold) publishes A2AV_REJECT instead, so that every rank fails the call.
// INVALID_OFF already means "this peer timed out".
constexpr uint64_t A2AV_REJECT = ~0ull - 1;

// What this rank publishes in off0 (every calling thread computes the same value).  Relaxed .sys loads: the engine
// kernel outlives the host writes to a counts buffer, so nothing may come from a stale L1 line.
__device__ __noinline__ uint64_t a2av_entry_off(const char *heap, const WorkItem &it) {
  const uint64_t *cnt = reinterpret_cast<const uint64_t *>(heap + it.desc.addr1());
  const uint32_t P = it.comm_size;
  const int64_t scap = it.desc.root_src_dst, rcap = it.desc.count;
  int64_t s = 0, r = 0;
  bool ok = true;
  for (uint32_t q = 0; q < P; ++q) {
    const int64_t a = static_cast<int64_t>(ld_relaxed_sys(cnt + q)), b = static_cast<int64_t>(ld_relaxed_sys(cnt + P + q));
    ok = ok && a >= 0 && a <= scap && b >= 0 && b <= rcap; // bounded first: the sums below cannot overflow
    s += ok ? a : 0;
    r += ok ? b : 0;
  }
  return ok && s <= scap && r <= rcap ? it.desc.addr1() : A2AV_REJECT;
}

__device__ __forceinline__ int64_t a2av_count(const Ctx &c, const uint64_t *s_off0, uint32_t p, uint32_t i) {
  return static_cast<int64_t>(ld_relaxed_sys(reinterpret_cast<const uint64_t *>(c.heap(c.g(p)) + s_off0[p]) + i));
}

// `bytes` from src to dst split over (cta, nctas) on the widest path the two addresses allow: 16-byte vectors when
// they are congruent mod 16 (head and tail peeled), 4-byte words when congruent mod 4, else bytes.  Arbitrary
// element counts put the blocks at arbitrary byte offsets, where copy_simple would fall back to single bytes.
__device__ __forceinline__ void copy_congruent(char *dst, const char *src, size_t bytes, int cta, int nctas) {
  const uintptr_t d = reinterpret_cast<uintptr_t>(dst), x = d ^ reinterpret_cast<uintptr_t>(src);
  const size_t g = (x & 15) == 0 ? 16 : ((x & 3) == 0 ? 4 : 1);
  size_t head = (g - (d & (g - 1))) & (g - 1);
  if (head > bytes) head = bytes;
  const size_t body = (bytes - head) / g * g;
  const size_t stride = static_cast<size_t>(nctas) * blockDim.x;
  const size_t tid = static_cast<size_t>(cta) * blockDim.x + threadIdx.x;
  for (size_t i = tid; i < head; i += stride) dst[i] = *reinterpret_cast<const volatile char *>(src + i);
  for (size_t i = head + body + tid; i < bytes; i += stride) dst[i] = *reinterpret_cast<const volatile char *>(src + i);
  if (g == 4) {
    uint32_t *dw = reinterpret_cast<uint32_t *>(dst + head);
    const volatile uint32_t *sw = reinterpret_cast<const volatile uint32_t *>(src + head);
    for (size_t i = tid; i < body / 4; i += stride) dw[i] = sw[i];
  } else {
    copy_simple(dst + head, src + head, body, cta, nctas); // g == 16: the vector path; g == 1: bytes
  }
}

// Data phase of alltoallv.  Every CTA checks the whole count matrix from the peers' counts buffers (at most 2 x 16 x
// 16 loads), so all ranks reach the same verdict; the peers wrote their counts with stream-ordered work before their
// kernels started, and nobody leaves the exit meeting before everybody has read them.  Then each CTA pushes its
// share of every block, starting at a different destination.
__device__ __noinline__ void rvb_alltoallv(const Ctx &c, const uint64_t *s_off0, const uint64_t *s_off2) {
  __shared__ uint64_t s_len[ACCL_MAX_RANKS];
  __shared__ uint32_t s_bad;
  const WorkItem &it = c.it;
  const uint32_t P = c.P(), me = c.r(), t = threadIdx.x;
  const size_t es = esize(it.udtype);
  __syncthreads();
  if (t == 0) s_bad = 0;
  __syncthreads();
  if (t < P && (s_off0[t] == A2AV_REJECT || s_off0[t] > c.w.heap_bytes - 16ull * P)) s_bad = 1;
  __syncthreads();
  if (!s_bad)
    for (uint32_t i = t; i < P * P; i += blockDim.x) {
      const uint32_t p = i / P, q = i % P; // p's send count to q against q's receive count from p
      if (a2av_count(c, s_off0, p, q) != a2av_count(c, s_off0, q, P + p)) s_bad = 1;
    }
  __syncthreads();
  if (s_bad) {
    if (t == 0) atomicOr(c.err, DMA_SIZE_ERROR);
    return;
  }
  if (t < P) {
    // my block for q: at the prefix of my send counts in my source, after the blocks of q's lower senders in q's
    // destination
    const uint32_t q = t;
    uint64_t so = 0, dof = 0;
    for (uint32_t j = 0; j < q; ++j) so += a2av_count(c, s_off0, me, j);
    for (uint32_t p = 0; p < me; ++p) dof += a2av_count(c, s_off0, q, P + p);
    c.tab->src[q] = c.heap(c.w.rank) + it.desc.addr0() + so * es;
    c.tab->dst[q] = c.heap(c.g(q)) + s_off2[q] + dof * es;
    s_len[q] = a2av_count(c, s_off0, me, q) * es;
  }
  __syncthreads();
  for (uint32_t k = 0; k < P; ++k) {
    const uint32_t q = (me + k + static_cast<uint32_t>(c.cta)) % P; // all switch ports fed at once
    copy_congruent(c.tab->dst[q], c.tab->src[q], s_len[q], c.cta, c.nctas);
  }
}

// reduce to root.  Small: the root pulls (or lets the switch reduce) everything.  Large
// (P >= 3): the P-1 other ranks each reduce one slice and store it into the root's buffer,
// so the root's inbound link carries N bytes instead of (P-1) N.
__device__ __noinline__ void rvb_reduce(const Ctx &c, const uint64_t *s_off0, const uint64_t *s_off2) {
  const WorkItem &it = c.it;
  const uint32_t P = c.P(), me = c.r(), root = it.desc.root_src_dst;
  const size_t es = esize(it.udtype), count = it.desc.count;
  const NvOp nop = nvls_op(it.udtype, it.desc.function);
  const bool sym = all_equal(s_off0, P) && (s_off0[0] & 15) == 0 && (s_off2[root] & 15) == 0;
  const bool use_mc = (it.flags & WF_USE_MC) && it.algo == ALGO_NVLS && nop != NvOp::none && sym;
  char *root_dst = c.heap(c.g(root)) + s_off2[root];
  const size_t nvec = count * es / 16;
  // all ranks take the same decision: it only depends on the call and on the (identical) geometry
  const bool distributed = P >= 3 && count * es >= (1u << 20) && (s_off2[root] & 15) == 0;
  size_t done = 0;
  if (distributed) {
    if (me != root) {
      const uint32_t j = (me + P - root - 1) % P; // my index among the P-1 workers
      const size_t per = (nvec + (P - 1) - 1) / (P - 1);
      const size_t v0 = j * per < nvec ? j * per : nvec, v1 = v0 + per < nvec ? v0 + per : nvec;
      // peer pulls: every worker's inbound link carries ~N, like the root's, instead of letting the switch reduce
      // the slices
      fill_table(c, s_off0, nullptr, v0 * 16, 0, true);
      if (threadIdx.x == 0) c.tab->dst[0] = root_dst + v0 * 16;
      __syncthreads();
      reduce_dispatch(c.tab, static_cast<int>(P), 1, (v1 - v0) * (16 / es), it.udtype, it.desc.function, c.cta, c.nctas, c.err);
    }
    done = nvec * 16 / es; // the sub-vector tail (if any) is reduced by the root below
  } else if (me == root && use_mc) {
    nvls_reduce_dispatch<false>(nop, it.nvls_unroll, c.w.mc + s_off0[0], root_dst, 0, nvec, c.cta, c.nctas);
    done = nvec * 16 / es;
  }
  if (me == root && done < count) {
    fill_table(c, s_off0, nullptr, done * es, 0, false);
    if (threadIdx.x == 0) c.tab->dst[0] = root_dst + done * es;
    __syncthreads();
    reduce_dispatch(c.tab, static_cast<int>(P), 1, count - done, it.udtype, it.desc.function, c.cta, c.nctas, c.err);
  }
}

// Large broadcast, software-pipelined in two overlapping stages: the root deals slice j of its
// buffer to worker j (root outbound = N in total); worker j forwards what it received to the other
// workers (worker inbound = N, outbound = N (P-2)/(P-1)).  Chunk c is forwarded while chunk c+1 is
// dealt, each CTA running its own stripe of every slice with its own flags.
__device__ __noinline__ void rv_bcast_pipelined(const Ctx &c, const uint64_t *s_off) {
  const WorkItem &it = c.it;
  const uint32_t P = c.P(), me = c.r(), root = it.desc.root_src_dst;
  const size_t nvec = static_cast<size_t>(it.desc.count) * esize(it.udtype) / 16;
  const uint32_t W = P - 1;                       // workers
  const size_t per_slice = (nvec + W - 1) / W;    // vectors per worker slice
  const size_t per_cta = (per_slice + c.nctas - 1) / c.nctas;
  // per (slice, CTA) step: about 1/8 of the stripe, between 32 KiB and 256 KiB (pipeline depth vs sync cost)
  size_t CH = per_cta / 8;
  CH = CH < 2048 ? 2048 : (CH > 16384 ? 16384 : CH);
  const size_t steps = (per_cta + CH - 1) / CH;
  const uint32_t j_me = (me + P - root - 1) % P;  // my worker index (unused on the root)
  const char *src = c.heap(c.w.rank) + s_off[me];
  auto range = [&](uint32_t j, size_t step, size_t &a, size_t &b) {
    a = j * per_slice + static_cast<size_t>(c.cta) * per_cta + step * CH;
    b = a + CH;
    const size_t lim_cta = j * per_slice + (static_cast<size_t>(c.cta) + 1) * per_cta;
    const size_t lim_slice = (j + 1) * per_slice < nvec ? (j + 1) * per_slice : nvec;
    if (b > lim_cta) b = lim_cta;
    if (b > lim_slice) b = lim_slice;
  };
  for (size_t st = 0; st <= steps; ++st) {
    if (me == root && st < steps) {
      for (uint32_t k = 0; k < W; ++k) {
        const uint32_t j = (k + static_cast<uint32_t>(c.cta)) % W; // CTAs start on different workers
        const uint32_t q = (root + 1 + j) % P;
        size_t a, b;
        range(j, st, a, b);
        if (a < b) copy_simple(c.heap(c.g(q)) + s_off[q] + a * 16, src + a * 16, (b - a) * 16, 0, 1);
      }
    } else if (me != root && st >= 1 && W >= 2) {
      size_t a, b;
      range(j_me, st - 1, a, b);
      if (a < b) {
        __syncthreads();
        if (threadIdx.x == 0) {
          int nd = 0;
          for (uint32_t k = 1; k < W; ++k) { // the other workers, starting after me
            const uint32_t q = (root + 1 + (j_me + k) % W) % P;
            c.tab->dst[nd++] = c.heap(c.g(q)) + s_off[q] + a * 16;
          }
          c.tab->src[0] = src + a * 16; // what the root stored here one step ago
        }
        __syncthreads();
        copy_dispatch(c.tab, static_cast<int>(W) - 1, (b - a) * 16, 0, 1);
      }
    }
    chan_sync(c, false, 0, 0, nullptr, nullptr);
  }
}

// rendezvous send / recv: a pair of ranks meets on the pads, the receiver
// announces its buffer, the sender stores straight into it
__device__ __noinline__ void rv_send(const Ctx &c, uint64_t *s_pair) {
  const WorkItem &it = c.it;
  uint32_t *kind = reinterpret_cast<uint32_t *>(s_pair + 1);
  pair_sync(c, it.desc.root_src_dst, it.desc.addr0(), static_cast<uint32_t>(operation::send), s_pair, kind);
  if (*kind != static_cast<uint32_t>(operation::recv)) {
    if (threadIdx.x == 0 && *kind != 0xFFFFFFFFu) atomicOr(c.err, PACK_SEQ_NUMBER_ERROR);
  } else {
    copy_simple(c.heap(c.g(it.desc.root_src_dst)) + *s_pair, c.heap(c.w.rank) + it.desc.addr0(),
                static_cast<size_t>(it.desc.count) * esize(it.udtype), c.cta, c.nctas);
  }
  __shared__ uint64_t s_o;
  __shared__ uint32_t s_k;
  pair_sync(c, it.desc.root_src_dst, 0, static_cast<uint32_t>(operation::send), &s_o, &s_k, false);
}

__device__ __noinline__ void rv_recv(const Ctx &c, uint64_t *s_pair) {
  const WorkItem &it = c.it;
  uint32_t *kind = reinterpret_cast<uint32_t *>(s_pair + 1);
  pair_sync(c, it.desc.root_src_dst, it.desc.addr2(), static_cast<uint32_t>(operation::recv), s_pair, kind);
  if (*kind != static_cast<uint32_t>(operation::send) && *kind != 0xFFFFFFFFu && threadIdx.x == 0)
    atomicOr(c.err, PACK_SEQ_NUMBER_ERROR);
  __shared__ uint64_t s_o;
  __shared__ uint32_t s_k;
  pair_sync(c, it.desc.root_src_dst, 0, static_cast<uint32_t>(operation::recv), &s_o, &s_k, false);
}

} // namespace k
} // namespace cuda
} // namespace accl
