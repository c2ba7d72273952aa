// run_work: execute one WorkItem with `nctas` cooperating CTAs.
#pragma once
#include "collectives.cuh"
#include "staged.cuh"
#include "compress.cuh"

namespace accl {
namespace cuda {
namespace k {

// The data phase of a rendezvous collective with the buffer offsets already exchanged, and the local calls.  The
// direct launch runs it between its entry and exit meetings (run_work below); the engine's worker CTAs run it for an
// MV_BODY move.  `stepwise`: the body may meet the peers between chunks (the pipelined broadcast); false inside the
// engine, where every wait must be a parked step.
__device__ __noinline__ void run_body(const Ctx &c, const uint64_t *off0, const uint64_t *off2, bool stepwise) {
  const WorkItem &it = c.it;
  const operation op = static_cast<operation>(it.desc.scenario);
  switch (op) {
  case operation::copy: op_copy(c); break;
  case operation::combine: op_combine(c); break;
  case operation::allreduce:
    if (it.algo == ALGO_P2P_ONESHOT) rvb_allreduce_oneshot(c, off0, off2);
    else rvb_allreduce(c, off0, off2);
    break;
  case operation::reduce_scatter: rvb_reduce_scatter(c, off0, off2); break;
  case operation::reduce: rvb_reduce(c, off0, off2); break;
  case operation::allgather:
  case operation::bcast:
  case operation::scatter:
  case operation::gather:
  case operation::alltoall: rvb_move(c, pattern_of(op), off0, off2, stepwise); break;
  default: // (alltoallv here rather than as a case of its own: fewer registers saved around the calls above)
    if (op == operation::alltoallv) rvb_alltoallv(c, off0, off2);
    else if (threadIdx.x == 0) atomicOr(c.err, COLLECTIVE_NOT_IMPLEMENTED);
    break;
  }
}

__device__ __noinline__ void run_work(const DevWorld &w, const WorkItem &it, int cta, int nctas, uint32_t *s_err) {
  __shared__ uint64_t s_off0[ACCL_MAX_RANKS], s_off2[ACCL_MAX_RANKS];
  __shared__ const char *s_slots[ACCL_MAX_RANKS];
  __shared__ uint32_t s_tmp;
  __shared__ PtrTable s_tab;
  Ctx c{w, it, cta, nctas, reinterpret_cast<Ctrl *>(w.window + static_cast<uint64_t>(w.rank) * w.heap_bytes), s_err,
        static_cast<uint64_t>(it.timeout_us) * 1000ull, &s_tab};
  const operation op = static_cast<operation>(it.desc.scenario);
  const Pattern pat = pattern_of(op);
  const bool eager = it.algo == ALGO_EAGER;
  if ((it.algo == ALGO_LL || it.algo == ALGO_STAGED) && pat != PAT_NONE) {
    // one-way staged exchange (one hop, no meetings): staged.cuh
    stg_collective(c, pat, &s_tmp);
    return;
  }
  if (it.algo == ALGO_WIRE) {
    wire_collective(c);
    return;
  }
  switch (op) {
  case operation::nop:
  case operation::config: return;
  case operation::copy: op_copy(c); return;
  case operation::combine: op_combine(c); return;
  case operation::send:
    if (eager) egr_p2p(c, true, false, 0, &s_tmp);
    else rv_send(c, s_off0);
    return;
  case operation::recv:
    if (eager) egr_p2p(c, false, false, 0, &s_tmp);
    else rv_recv(c, s_off0);
    return;
  case operation::barrier:
    chan_sync(c, false, 0, 0, nullptr, nullptr);
    return;
  default: break;
  }
  const bool a2av = op == operation::alltoallv;
  if (pat == PAT_NONE && !a2av) {
    if (threadIdx.x == 0) atomicOr(s_err, COLLECTIVE_NOT_IMPLEMENTED);
    return;
  }
  if (eager) {
    egr_collective(c, pat, &s_tmp, s_slots);
    return;
  }
  // rendezvous: entry meeting with the address exchange, data phase, exit meeting (the engine's step_call runs the
  // same three steps).  Bcast keeps its buffer in addr0 on every rank; the others receive into addr2.  Alltoallv
  // publishes its counts (or its rejection) in the off0 slot.
  const uint64_t my_off0 = a2av ? a2av_entry_off(c.heap(w.rank), it) : it.desc.addr0();
  chan_sync(c, true, my_off0, pat == PAT_BCAST ? it.desc.addr0() : it.desc.addr2(), s_off0, s_off2);
  if (*c.err == 0) run_body(c, s_off0, s_off2, true);
  chan_sync(c, false, 0, 0, nullptr, nullptr);
}

} // namespace k
} // namespace cuda
} // namespace accl
