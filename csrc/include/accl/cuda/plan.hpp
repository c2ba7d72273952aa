// Call planning shared by the host (direct launches, host ring) and the
// engine's control CTA (device-issued commands): decode communicator and
// arithmetic configuration from exchange memory, pick protocol, algorithm and
// CTA count.  Must be a pure function of the call and of configuration that
// is identical on all ranks, because both ends of every transfer derive their
// behaviour from it independently.
//
// Reference: the per-call decisions at the top of every firmware collective
// (eager vs rendezvous: ccl_offload_control.c:587,667,808,1009,1142,1314,1523,
// 1768,1878; tree/flat selection from the tuning registers, accl.cpp:1198-1208).
// On an NVSwitch domain the choices are eager-slots / one-shot / two-shot and
// in-switch (NVLS) vs peer load-store instead of ring / flat / binary tree.
#pragma once
#include "accl/cuda/devtypes.hpp"

namespace accl {
namespace cuda {

struct PlanCfg {
  uint32_t max_ctas;
  uint32_t nvls_min_ranks;
  uint32_t has_mc;
  uint32_t heap_world;
  uint64_t oneshot_max_bytes;
  // bit i set: operation code i may use the in-switch (multimem) algorithm.  Default: allreduce,
  // bcast and reduce: allgather and reduce_scatter move less data per link with peer stores / loads
  // than through the switch.
  uint32_t nvls_ops;
  uint32_t nvls_ctas;      // channel cap of the NVLS two-shot all-reduce (fewer, fatter CTAs win through the switch)
  uint32_t stg_bytes;      // staging region per (bank, parity, source) of ALGO_STAGED; 0: protocol off
  uint32_t ll_bytes;       // same for ALGO_LL
  uint32_t ll_max_bytes;   // flag-in-data protocol while message x (P - 1) peers stays within this many bytes
  uint32_t ll_oneshot_max; // all-reduce: everybody-sends-everything (one hop) up to this size, two hops above
  uint32_t wire_min_bytes; // compressed-wire calls at least this big use the fused two-shot (0: always the slot ring)
  uint32_t staged_max_bytes; // per-peer messages up to this size that do not fit the LL protocol use ALGO_STAGED
                             // (0: they go to the slot ring / rendezvous instead)
  uint32_t engine_mode;    // calls run inside the persistent engine: prefer ONE channel when the message fits it
                           // (the control CTA executes it inline, no hand-over to the workers)
  uint32_t nvls_unroll;    // 16-byte multimem accesses in flight per thread of the NVLS bodies: 2, 4, 8 or 16
};
constexpr uint32_t NVLS_OPS_DEFAULT = (1u << static_cast<uint32_t>(operation::allreduce)) |
                                      (1u << static_cast<uint32_t>(operation::bcast)) |
                                      (1u << static_cast<uint32_t>(operation::reduce));

ACCL_HD uint32_t plan_ctas(uint64_t bytes, uint64_t per_cta, uint32_t cap) {
  uint64_t n = (bytes + per_cta - 1) / per_cta;
  if (n < 1) n = 1;
  if (n > cap) n = cap;
  return static_cast<uint32_t>(n);
}

// One-way staged protocols (staged.cuh): does a per-peer message of `m` bytes fit, and on how many channels?
// Every channel owns a fixed 1 / STG_CH slice of the staging region.  Returns 0 when it does not fit.
ACCL_HD uint32_t plan_staged_ctas(uint64_t m, bool ll, const PlanCfg &cfg, uint32_t cap) {
  if (!ll && m > cfg.staged_max_bytes) return 0;
  const uint64_t region = ll ? cfg.ll_bytes : cfg.stg_bytes;
  const uint64_t slice = (region / static_cast<uint64_t>(STG_CH)) & ~127ull;
  if (!slice) return 0;
  const uint64_t unit = ll ? 8 : 16;                       // payload granule of a part (staged.cuh stg_part)
  const uint64_t units = (m + unit - 1) / unit;
  const uint64_t per_slice = slice / 16;                   // LL: 8 payload bytes per 16-byte line; plain: 16 per 16
  uint64_t need = (units + per_slice - 1) / per_slice;     // channels needed for capacity
  uint64_t want = ll ? (units + 511) / 512 : (m + (32u << 10) - 1) / (32u << 10); // channels wanted for parallelism
  const uint64_t lim = cap < static_cast<uint32_t>(STG_CH) ? cap : static_cast<uint32_t>(STG_CH);
  if (need < 1) need = 1;
  if (need > lim) return 0;
  if (cfg.engine_mode && need == 1 && units <= 2048) want = 1;
  if (want < need) want = need;
  if (want > lim) want = lim;
  // parts are ceil(units / n): re-check capacity for the chosen n
  while (want < lim && (units + want - 1) / want > per_slice) ++want;
  if ((units + want - 1) / want > per_slice) return 0;
  return static_cast<uint32_t>(want);
}

ACCL_HD void plan_call(const uint32_t *exch, const PlanCfg &cfg, WorkItem &w) {
  const operation op = static_cast<operation>(w.desc.scenario);
  const uint64_t ubytes = static_cast<uint64_t>(w.desc.count) * dtype_bytes(static_cast<dataType>(w.udtype));
  const uint32_t P = w.comm_size;
  const uint32_t cap = cfg.max_ctas < static_cast<uint32_t>(MAX_CH) ? cfg.max_ctas : static_cast<uint32_t>(MAX_CH);
  w.flags = cfg.has_mc ? WF_USE_MC : 0;
  w.nvls_unroll = cfg.nvls_unroll;
  if (op == operation::nop || op == operation::config) {
    w.algo = ALGO_LOCAL;
    w.n_ctas = 1;
    return;
  }
  if (op == operation::copy || op == operation::combine) {
    w.algo = ALGO_LOCAL;
    w.n_ctas = plan_ctas(ubytes, 256u << 10, 264); // local: no sync channels involved, fill the chip (132 SMs) twice
    return;
  }
  if (op == operation::barrier) {
    w.algo = ALGO_P2P;
    w.n_ctas = 1;
    return;
  }
  if (op == operation::alltoallv) {
    // the block sizes live in device memory and `count` is this rank's receive capacity, which differs between
    // ranks: every channel decision here must come from configuration alone, or the ranks' grids (and with them
    // the per-channel meetings) would disagree.  Always the rendezvous push between user buffers.
    w.algo = ALGO_P2P;
    w.n_ctas = cap;
    return;
  }
  uint64_t moved = ubytes; // payload a rank moves, for sizing
  if (op == operation::allgather || op == operation::reduce_scatter || op == operation::alltoall ||
      op == operation::scatter || op == operation::gather)
    moved = ubytes * P;
  const bool compressed = w.desc.compression_flags != 0;
  const bool p2p = op == operation::send || op == operation::recv;
  const bool eager = compressed || ubytes <= exch[exchmem::MAX_EAGER_SIZE / 4];
  bool eager_ok = eager;
  if (eager && !compressed && !p2p && ubytes && cfg.ll_bytes) {
    // one-way staged exchange: flag-in-data (LL) while it fits, payload + release flag when enabled
    uint64_t m = ubytes;
    uint32_t extra = 0;
    bool ok = true;
    if (op == operation::allreduce) {
      if (ubytes <= cfg.ll_oneshot_max || ubytes % (16ull * P) != 0) extra = WF_ONESHOT; // everybody receives everything
      else m = ubytes / P;                                                               // shards: reduce-scatter + all-gather
      // a one-shot of a large odd-sized message would move P x the bytes: leave it to the other paths
      if ((extra & WF_ONESHOT) && ubytes > 4ull * cfg.ll_oneshot_max && ubytes > (256u << 10)) ok = false;
    }
    if (ok) {
      // flag-in-data doubles the wire bytes, and a rank pushes its message to P - 1 peers: the budget is on the fan-out
      uint32_t n = m * (P > 1 ? P - 1 : 1) <= cfg.ll_max_bytes ? plan_staged_ctas(m, true, cfg, cap) : 0;
      if (n) {
        w.algo = ALGO_LL;
      } else {
        n = plan_staged_ctas(m, false, cfg, cap);
        if (n) w.algo = ALGO_STAGED;
      }
      if (n) {
        w.flags |= extra;
        w.n_ctas = n;
        return;
      }
    }
    // does not fit (or is too fat for) the staging regions: through the slot ring only while that is one or two
    // segments (every segment costs a credit + header + flag round), else the rendezvous algorithms
    if (ubytes > 2ull * exch[exchmem::EAGER_RX_BUF_SIZE / 4]) eager_ok = false;
  }
  // compressed wire, uncompressed operands, large message: the cast is fused into the two-shot exchange
  // (compress.cuh) instead of pushing segment after segment through the slot ring
  if (compressed && w.desc.compression_flags == 8u && cfg.wire_min_bytes && ubytes >= cfg.wire_min_bytes && P > 1 &&
      (op == operation::allreduce || op == operation::reduce_scatter || op == operation::allgather)) {
    const dataType u = static_cast<dataType>(w.udtype), c = static_cast<dataType>(w.cdtype);
    const bool c16 = c == dataType::float16 || c == dataType::bfloat16;
    const bool c8 = c == dataType::float8_e4m3 || c == dataType::float8_e5m2;
    const bool ok = (u == dataType::float32 && (c16 || c8)) || ((u == dataType::float16 || u == dataType::bfloat16) && c8);
    if (ok && (!c8 || w.ratio_log == 0 || w.ratio_log == 5)) {
      w.algo = ALGO_WIRE;
      w.n_ctas = plan_ctas(moved, 128u << 10, cap);
      return;
    }
  }
  if (eager_ok) {
    w.algo = ALGO_EAGER;
    const uint32_t ecap = cap < static_cast<uint32_t>(EGR_CH) ? cap : static_cast<uint32_t>(EGR_CH);
    w.n_ctas = p2p ? 1 : plan_ctas(ubytes, 16u << 10, ecap);
    return;
  }
  const bool nvls = cfg.has_mc && P >= cfg.nvls_min_ranks && P == cfg.heap_world &&
                    ((cfg.nvls_ops >> static_cast<uint32_t>(op)) & 1u);
  w.algo = nvls ? ALGO_NVLS : ALGO_P2P;
  // one-shot (everybody pulls everything) moves P x the bytes of two-shot: only while latency dominates
  if (op == operation::allreduce && ubytes * P <= cfg.oneshot_max_bytes) w.algo = ALGO_P2P_ONESHOT;
  if (p2p) w.algo = ALGO_P2P;
  uint32_t c = cap;
  // two-shot all-reduce through the switch is fastest with FEW channels and short bursts (bench/tune.py sweeps the
  // channel count and the accesses in flight); peer loads / stores want every channel they can get
  if (op == operation::allreduce && w.algo == ALGO_NVLS && cfg.nvls_ctas && c > cfg.nvls_ctas) c = cfg.nvls_ctas;
  w.n_ctas = plan_ctas(moved, 128u << 10, c);
}

// signature of a communicator's member list (identical on all members): names its protocol-state bank
ACCL_HD uint32_t comm_signature(const uint8_t *members, uint32_t n) {
  uint32_t h = 2166136261u ^ n;
  for (uint32_t i = 0; i < n; ++i) h = (h ^ members[i]) * 16777619u;
  h ^= h >> 15;
  return h & 0xFFFFFFu;
}

// Decode + plan.  Returns an error word (0 = ok).
ACCL_HD uint32_t build_work_item_hd(const uint32_t *exch, const PlanCfg &cfg, uint32_t world, const CallDesc &d,
                                    uint32_t timeout_us, WorkItem &w) {
  w.desc = d;
  w.scratch_off = 0;
  w.scratch_bytes = 0;
  w.req_slot = 0;
  w.req_seq = 0;
  const uint32_t ci = d.comm;
  if (ci >= static_cast<uint32_t>(ACCL_MAX_COMMUNICATORS)) return CONFIG_SWITCH_ERROR;
  w.comm_size = exch[exchmem::comm_offset(ci) / 4];
  w.comm_rank = exch[exchmem::comm_offset(ci) / 4 + 1];
  if (w.comm_size == 0 || w.comm_size > static_cast<uint32_t>(ACCL_MAX_RANKS)) return CONFIG_SWITCH_ERROR;
  for (uint32_t r = 0; r < static_cast<uint32_t>(ACCL_MAX_RANKS); ++r) {
    uint32_t g = 0;
    if (r < w.comm_size) {
      g = exch[exchmem::comm_rank_offset(ci, r, exchmem::CR_SESSION) / 4];
      if (g >= world) return CONFIG_SWITCH_ERROR;
    }
    w.members[r] = static_cast<uint8_t>(g);
  }
  if (d.arithcfg >= exchmem::MAX_ARITHCFG) return ARITH_ERROR;
  const uint32_t ab = exchmem::arith_offset(d.arithcfg, 0) / 4;
  w.udtype = exch[ab + exchmem::AC_UNCOMPRESSED_BYTES] >> 16;
  w.cdtype = exch[ab + exchmem::AC_COMPRESSED_BYTES] >> 16;
  w.ratio_log = exch[ab + exchmem::AC_RATIO_LOG];
  w.arith_compressed = exch[ab + exchmem::AC_ARITH_COMPRESSED];
  w.timeout_us = timeout_us;
  w.comm_sig = comm_signature(w.members, w.comm_size);
  w.bank = w.comm_sig % static_cast<uint32_t>(N_BANKS);
  w.hc_ptr = 0;
  const operation op = static_cast<operation>(d.scenario);
  const bool rooted = op == operation::send || op == operation::recv || op == operation::bcast ||
                      op == operation::scatter || op == operation::gather || op == operation::reduce;
  if (rooted && d.root_src_dst >= w.comm_size) return CONFIG_SWITCH_ERROR;
  // a communicator of one: every collective degenerates to a local copy (alltoallv excepted: its size is in device
  // memory, its body validates and copies it)
  if (w.comm_size == 1 && op != operation::copy && op != operation::combine && op != operation::nop &&
      op != operation::config && op != operation::alltoallv) {
    if (op == operation::barrier || op == operation::bcast) w.desc.scenario = static_cast<uint32_t>(operation::nop);
    else if (op == operation::send || op == operation::recv) return CONFIG_SWITCH_ERROR; // no loop-back slots to self
    else w.desc.scenario = static_cast<uint32_t>(operation::copy);
  }
  plan_call(exch, cfg, w);
  return 0;
}

} // namespace cuda
} // namespace accl
