// The persistent collective engine: one long-running sm_90a kernel per GPU
// that owns a command queue in device memory and drives the calls itself.
//
//   control CTA (last block)   the "firmware".  Fetches commands from the ring (host proxies and plugin
//                              kernels take tickets in it: the client arbiter), plans device-issued
//                              descriptors from the device copy of exchange memory, and runs every call as a
//                              RESUMABLE STATE MACHINE: a call that cannot make progress — the receiver of a
//                              rendezvous send has not announced its buffer yet, a peer has not entered a
//                              collective, an eager credit is missing — returns NOT_READY, keeps its
//                              `step`, and the next call is tried.  Calls are retired out of order.
//   worker CTAs                the data movers (the reference's DMP).  They execute MOVES handed over by
//                              the control CTA: the data phase of a collective with all buffer offsets
//                              resolved, a point-to-point payload copy, or a whole one-way exchange.
//
// Reference counterpart: the continuously running CCLO — wait_for_call round-robining the new-call and retry
// queues (ccl_offload_control.c:2264-2288), `current_step` saved with a parked call (:34, :2336, :2460-2478),
// the rendezvous mailbox (:142-408), move instructions issued to the data mover (:413-527), hostctrl
// (kernels/plugins/hostctrl/hostctrl.cpp:22-63) and client_arbiter (kernels/plugins/client_arbiter).
//
// Host calls reach the engine through a one-warp PROXY kernel launched on the caller's stream (the hostctrl
// block: it turns kernel arguments into a command-ring entry, so the call is ordered after the work already
// queued on that stream) which then, for everything but asynchronous point-to-point calls, waits for the
// engine's status word — later work on the stream sees the result, exactly like a direct launch.
//
// The kernel parks itself after `idle_us` without work so that device-wide synchronisation (cudaDeviceSynchronize,
// cudaFree, ...) cannot hang; the host relaunches it on the next submit (Dekker-style handshake on `submitted` /
// `state` in pinned memory).
#include "accl/cuda/engine.hpp"

#include <atomic>
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <stdexcept>
#include <thread>

#include "accl/common.hpp"
#include "accl/cuda/cudadevice.hpp"
#include "accl/cuda/driver_api.hpp"
#include "accl/cuda/plan.hpp"
#include "accl/device/api.cuh"
#include "run_work.cuh"

namespace accl {
namespace cuda {

__device__ __forceinline__ void publish_completion(HostCompletion *hc, uint32_t seq, uint32_t rc, unsigned long long dur) {
  asm volatile("st.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(hc), "r"(seq), "r"(rc), "r"(static_cast<uint32_t>(dur)),
               "r"(static_cast<uint32_t>(dur >> 32))
               : "memory");
}

enum EngineState : uint32_t { ENG_STOPPED = 0, ENG_RUNNING = 1, ENG_EXITING = 2 };

// lives in pinned, device-mapped host memory
struct HostRing {
  volatile unsigned long long submitted; // commands the host has handed to proxy kernels so far
  volatile uint32_t state;               // EngineState, written by the control CTA
  volatile uint32_t pins;                // device-side clients active: do not park
  volatile uint32_t stop;                // host asks the engine to leave now
  volatile uint32_t idle_us;
  volatile uint32_t clients;             // device-side client kernels launched so far (Ctrl::clients_done catches up)
};

__device__ __forceinline__ EngineArea *engine_area(const DevWorld &w) {
  return reinterpret_cast<EngineArea *>(w.window + static_cast<uint64_t>(w.rank) * w.heap_bytes + CTRL_BYTES / 2);
}
__device__ __forceinline__ Ctrl *my_ctrl(const DevWorld &w) {
  return reinterpret_cast<Ctrl *>(w.window + static_cast<uint64_t>(w.rank) * w.heap_bytes);
}

// copy a WorkItem or MoveDesc as 8-byte words, with threads [0, stride) of the caller (the CTA or one warp)
template <typename T> __device__ __forceinline__ void copy_words(T *dst, const T *src, uint32_t stride) {
  static_assert(sizeof(T) % 8 == 0, "copied as whole 8-byte words");
  const unsigned long long *s = reinterpret_cast<const unsigned long long *>(src);
  unsigned long long *d = reinterpret_cast<unsigned long long *>(dst);
  for (uint32_t i = threadIdx.x; i < sizeof(T) / 8; i += stride) d[i] = s[i];
}

// ------------------------------------------------------------------ workers
// Move i is complete when all `nworkers` CTAs have passed it (participants after executing their share).
__device__ void engine_worker(const DevWorld &w, int nworkers) {
  __shared__ uint32_t s_err;
  __shared__ MoveDesc s_mv;
  __shared__ unsigned long long s_seq;
  __shared__ uint32_t s_exit;
  __shared__ k::PtrTable s_tab;
  Ctrl *me = my_ctrl(w);
  EngineArea *ea = engine_area(w);
  if (threadIdx.x == 0) s_seq = dev::ld_acquire_gpu(&me->move_tail); // resume where the previous instance stopped (nothing is pending at a park)
  __syncthreads();
  unsigned long long next = s_seq;
  for (;;) {
    if (threadIdx.x == 0) {
      uint32_t spins = 0, ex = 0;
      while (dev::ld_acquire_gpu(&me->move_tail) <= next) {
        if (dev::ld_relaxed_sys(&me->engine_exit)) {
          ex = 1;
          break;
        }
        if (++spins > 256) dev::nanosleep(spins > 8192 ? 400 : 20);
      }
      s_exit = ex;
      s_err = 0;
    }
    __syncthreads();
    if (s_exit) return;
    const uint32_t slot = static_cast<uint32_t>(next % MOVE_SLOTS);
    copy_words(&s_mv, &ea->move_ring[slot], blockDim.x);
    __syncthreads();
    const int nctas = static_cast<int>(s_mv.n_ctas);
    if (static_cast<int>(blockIdx.x) < nctas) {
      switch (s_mv.kind) {
      case MV_BODY: {
        const k::Ctx c{w, s_mv.item, static_cast<int>(blockIdx.x), nctas, me, &s_err,
                       static_cast<uint64_t>(s_mv.item.timeout_us) * 1000ull, &s_tab};
        k::run_body(c, s_mv.off0, s_mv.off2, false);
        break;
      }
      case MV_WORK: k::run_work(w, s_mv.item, blockIdx.x, nctas, &s_err); break;
      case MV_COPY:
        k::copy_simple(reinterpret_cast<char *>(s_mv.b), reinterpret_cast<const char *>(s_mv.a), s_mv.c, blockIdx.x, nctas);
        break;
      default: break;
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      if (s_err) atomicOr(&me->move_err[slot], s_err);
      __threadfence_system(); // my stores (possibly to peers) are performed before the move counts as done
      atomicAdd(&me->move_done[slot], 1ull);
    }
    ++next;
    __syncthreads();
  }
  (void)nworkers;
}

// ------------------------------------------------------------------ control
enum StepResult : uint32_t { SR_DONE = 0, SR_NOT_READY = 1 };

struct Call { // one call in flight (running or parked) — lives in the control CTA's shared memory
  WorkItem item;
  uint64_t off0[ACCL_MAX_RANKS], off2[ACCL_MAX_RANKS]; // rendezvous: buffer offsets of every member
  unsigned long long ticket1; // command ring ticket + 1
  unsigned long long t_start; // %globaltimer when the call was fetched
  unsigned long long move_id; // outstanding move (valid in the "wait for move" steps)
  unsigned long long progress; // eager point-to-point: elements already transferred
  uint32_t step;   // current_step: where to resume
  uint32_t active;
  uint32_t err;
  uint32_t body_err; // rendezvous collectives: error of the data phase, reported once the exit meeting is done
  uint32_t note_slot, note_seq; // rendezvous point-to-point
};

struct EngCtx {
  const DevWorld &w;
  Ctrl *me;
  EngineArea *ea;
  int nworkers;
  unsigned long long *moves_issued; // shared-memory counter (== Ctrl::move_tail)
  uint32_t *s_flag;                 // shared scratch word for CTA-wide decisions
};

__device__ __forceinline__ bool is_collective(uint32_t scenario) {
  const operation op = static_cast<operation>(scenario);
  return op == operation::bcast || op == operation::scatter || op == operation::gather || op == operation::reduce ||
         op == operation::allgather || op == operation::allreduce || op == operation::reduce_scatter ||
         op == operation::barrier || op == operation::alltoall || op == operation::alltoallv;
}

// all threads; returns thread 0's value
__device__ __forceinline__ uint32_t bcast0(const EngCtx &e, uint32_t v) {
  __syncthreads();
  if (threadIdx.x == 0) *e.s_flag = v;
  __syncthreads();
  return *e.s_flag;
}

// ---- moves
// issue one move to the workers; false when the ring slot is still in use (caller parks)
__device__ bool move_issue(const EngCtx &e, Call &cl, uint32_t kind, uint32_t n_ctas, uint64_t a, uint64_t b, uint64_t c) {
  const unsigned long long id = *e.moves_issued;
  const uint32_t slot = static_cast<uint32_t>(id % MOVE_SLOTS);
  const unsigned long long prev_uses = id / MOVE_SLOTS;
  uint32_t ok = 0;
  if (threadIdx.x == 0)
    ok = dev::ld_acquire_gpu(&e.me->move_done[slot]) >= prev_uses * static_cast<unsigned long long>(e.nworkers) ? 1u : 0u;
  ok = bcast0(e, ok);
  if (!ok) return false;
  MoveDesc *mv = &e.ea->move_ring[slot];
  copy_words(&mv->item, &cl.item, blockDim.x);
  if (threadIdx.x < ACCL_MAX_RANKS) {
    mv->off0[threadIdx.x] = cl.off0[threadIdx.x];
    mv->off2[threadIdx.x] = cl.off2[threadIdx.x];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mv->kind = kind;
    mv->n_ctas = n_ctas < static_cast<uint32_t>(e.nworkers) ? n_ctas : static_cast<uint32_t>(e.nworkers);
    mv->item.n_ctas = mv->n_ctas;
    mv->a = a;
    mv->b = b;
    mv->c = c;
    e.me->move_err[slot] = 0;
    __threadfence();
    cl.move_id = id;
    *e.moves_issued = id + 1;
    dev::st_release_gpu(&e.me->move_tail, id + 1);
  }
  __syncthreads();
  return true;
}

__device__ bool move_finished(const EngCtx &e, Call &cl) {
  uint32_t done = 0;
  if (threadIdx.x == 0) {
    const uint32_t slot = static_cast<uint32_t>(cl.move_id % MOVE_SLOTS);
    const unsigned long long need = (cl.move_id / MOVE_SLOTS + 1) * static_cast<unsigned long long>(e.nworkers);
    if (dev::ld_acquire_gpu(&e.me->move_done[slot]) >= need) {
      done = 1;
      cl.err |= e.me->move_err[slot];
    }
  }
  return bcast0(e, done) != 0;
}

// ---- rendezvous meetings on the engine's own channel of the call's bank, split into post and poll
constexpr int ENG_CH = MAX_CH - 2; // (MAX_CH - 1 belongs to the GEMM plugin)

// the call as the device helpers see it (one CTA; the meetings name their channel themselves)
__device__ __forceinline__ k::Ctx call_ctx(const EngCtx &e, const Call &cl, uint32_t *err) {
  return k::Ctx{e.w, cl.item, 0, 1, e.me, err, static_cast<uint64_t>(cl.item.timeout_us) * 1000ull, nullptr};
}

__device__ void meet_post(const EngCtx &e, Call &cl, bool exchange, uint64_t off0, uint64_t off2) {
  const k::Ctx c = call_ctx(e, cl, &cl.err);
  __syncthreads();
  const uint32_t t = threadIdx.x;
  if (t == c.r()) {
    cl.off0[t] = off0;
    cl.off2[t] = off2;
  } else if (t < c.P()) {
    k::pad_post(c, ENG_CH, c.g(t), exchange ? k::REC_OFFS : k::REC_NONE, off0, off2, c.kind_word());
  }
  __syncthreads();
}

// true once every member has posted its side of the meeting (then the offsets are in cl.off0 / off2).  All or
// nothing: no post is taken before every peer's has arrived, so a parked meeting is polled again from scratch.
__device__ bool meet_poll(const EngCtx &e, Call &cl, bool exchange) {
  const k::Ctx c = call_ctx(e, cl, &cl.err);
  const uint32_t t = threadIdx.x;
  const bool peer = t < c.P() && t != c.r();
  const bool all = __syncthreads_and(!peer || k::pad_arrived(c, ENG_CH, c.g(t))) != 0;
  if (all && peer) {
    k::pad_take(c, ENG_CH, c.g(t));
    if (exchange) {
      const SyncRec r = k::pad_rec(c, ENG_CH, c.g(t), k::REC_OFFS);
      cl.off0[t] = r.off0;
      cl.off2[t] = r.off2;
      if (r.kind != c.kind_word()) atomicOr(c.err, PACK_SEQ_NUMBER_ERROR);
    }
  }
  __syncthreads();
  return all;
}

// ---- one step of one call (all threads of the control CTA; uniform result)
__device__ uint32_t step_call(const EngCtx &e, Call &cl, uint32_t *s_err) {
  const WorkItem &it = cl.item;
  const operation op = static_cast<operation>(it.desc.scenario);
  const uint32_t t = threadIdx.x;
  char *heap = e.w.window + static_cast<uint64_t>(e.w.rank) * e.w.heap_bytes;

  if (op == operation::nop || op == operation::config) return SR_DONE;

  // ---------------- local data movement: one wait-free move
  if (op == operation::copy || op == operation::combine) {
    if (cl.step == 0) {
      if (!move_issue(e, cl, MV_BODY, it.n_ctas, 0, 0, 0)) return SR_NOT_READY;
      cl.step = 1;
    }
    return move_finished(e, cl) ? SR_DONE : SR_NOT_READY;
  }

  // ---------------- point to point
  if (op == operation::send || op == operation::recv) {
    const bool sending = op == operation::send;
    const uint32_t peer_cr = it.desc.root_src_dst;
    const uint32_t peer = it.members[peer_cr];
    Ctrl *pc = reinterpret_cast<Ctrl *>(e.w.window + static_cast<uint64_t>(peer) * e.w.heap_bytes);
    if (it.algo == ALGO_EAGER) {
      // a missing credit (sender) or a segment that has not arrived yet (receiver) parks the call with `progress`
      const unsigned long long done = k::egr_p2p(call_ctx(e, cl, s_err), sending, true, cl.progress, e.s_flag);
      __syncthreads();
      if (t == 0) cl.progress = done;
      return done < it.desc.count ? SR_NOT_READY : SR_DONE;
    }
    // rendezvous through the address mailbox
    if (!sending) {
      if (cl.step == 0) {
        uint32_t ok = 0;
        if (t == 0) {
          const uint32_t seq = e.me->note_posted[peer] + 1;
          const uint32_t slot = (seq - 1) % P2P_NOTES;
          // the slot's previous note (seq - P2P_NOTES) must have been served
          if (seq <= static_cast<uint32_t>(P2P_NOTES) ||
              static_cast<int32_t>(dev::ld_acquire_sys(&e.me->note_done[peer][slot]) - (seq - P2P_NOTES)) >= 0) {
            P2pNote *n = &pc->note[e.w.rank][slot];
            dev::st_relaxed_sys(&n->addr, it.desc.addr2());
            dev::st_relaxed_sys(&n->count, it.desc.count);
            dev::st_relaxed_sys(&n->tag, it.desc.tag);
            dev::st_relaxed_sys(&n->dtype, it.udtype);
            dev::st_release_sys(&n->seq, seq);
            e.me->note_posted[peer] = seq;
            cl.note_slot = slot;
            cl.note_seq = seq;
            ok = 1;
          }
        }
        if (!bcast0(e, ok)) return SR_NOT_READY;
        cl.step = 1;
      }
      uint32_t done = 0;
      if (t == 0) done = dev::ld_acquire_sys(&e.me->note_done[peer][cl.note_slot]) == cl.note_seq ? 1u : 0u;
      return bcast0(e, done) ? SR_DONE : SR_NOT_READY;
    }
    // sender
    if (cl.step == 0) {
      uint32_t found = 0;
      if (t == 0) {
        // oldest note of this receiver that no earlier send of mine has taken and whose tag matches
        uint32_t best_seq = 0, best_slot = 0;
        for (uint32_t j = 0; j < static_cast<uint32_t>(P2P_NOTES); ++j) {
          const P2pNote *n = &e.me->note[peer][j];
          const uint32_t sq = dev::ld_acquire_sys(&n->seq);
          if (sq == 0 || static_cast<int32_t>(sq - e.me->note_taken[peer][j]) <= 0) continue;
          const uint32_t ntag = dev::ld_relaxed_sys(&n->tag);
          if (!(it.desc.tag == TAG_ANY || ntag == TAG_ANY || ntag == it.desc.tag)) continue;
          if (best_seq == 0 || static_cast<int32_t>(sq - best_seq) < 0) {
            best_seq = sq;
            best_slot = j;
          }
        }
        if (best_seq) {
          const P2pNote *n = &e.me->note[peer][best_slot];
          if (dev::ld_relaxed_sys(&n->count) != it.desc.count) cl.err |= DMA_NOT_EXPECTED_BTT_ERROR;
          if (dev::ld_relaxed_sys(&n->dtype) != it.udtype) cl.err |= COMPRESSION_ERROR;
          cl.off2[0] = dev::ld_relaxed_sys(&n->addr);
          e.me->note_taken[peer][best_slot] = best_seq;
          cl.note_slot = best_slot;
          cl.note_seq = best_seq;
          found = 1;
        }
      }
      if (!bcast0(e, found)) return SR_NOT_READY;
      cl.step = 1;
    }
    if (cl.step == 1) {
      const uint64_t bytes = cl.err ? 0 : static_cast<uint64_t>(it.desc.count) * k::esize(it.udtype);
      char *dst = e.w.window + static_cast<uint64_t>(peer) * e.w.heap_bytes + cl.off2[0];
      if (!move_issue(e, cl, MV_COPY, it.n_ctas, reinterpret_cast<uint64_t>(heap + it.desc.addr0()), reinterpret_cast<uint64_t>(dst), bytes))
        return SR_NOT_READY;
      cl.step = 2;
    }
    if (!move_finished(e, cl)) return SR_NOT_READY;
    // payload has landed (workers fenced before reporting): tell the receiver (RNDZVS_WR_DONE)
    if (t == 0) dev::st_release_sys(&pc->note_done[e.w.rank][cl.note_slot], cl.note_seq);
    __syncthreads();
    return SR_DONE;
  }

  // ---------------- collectives
  if (op == operation::barrier) {
    if (cl.step == 0) {
      meet_post(e, cl, false, 0, 0);
      cl.step = 1;
    }
    return meet_poll(e, cl, false) ? SR_DONE : SR_NOT_READY;
  }
  if (it.algo == ALGO_LL || it.algo == ALGO_STAGED || it.algo == ALGO_EAGER || it.algo == ALGO_WIRE) {
    // one-way exchanges: everything they wait for is pushed by the peers at the START of the same collective,
    // so they run to completion — inline when one channel is enough, else as one move on the workers
    if (it.n_ctas <= 1) {
      k::run_work(e.w, it, 0, 1, s_err);
      __syncthreads();
      return SR_DONE;
    }
    if (cl.step == 0) {
      if (!move_issue(e, cl, MV_WORK, it.n_ctas, 0, 0, 0)) return SR_NOT_READY;
      cl.step = 1;
    }
    return move_finished(e, cl) ? SR_DONE : SR_NOT_READY;
  }
  // rendezvous: entry meeting (parked until every member has entered), wait-free data phase on the workers,
  // exit meeting (parked until every member is done with my buffers)
  if (cl.step == 0) {
    const uint64_t my_dst = op == operation::bcast ? it.desc.addr0() : it.desc.addr2();
    // alltoallv: the counts offset (or its local rejection, decided when the call was fetched) in the off0 slot
    const uint64_t my_src = op == operation::alltoallv ? cl.off0[it.comm_rank] : it.desc.addr0();
    meet_post(e, cl, true, my_src, my_dst);
    cl.step = 1;
  }
  if (cl.step == 1) {
    if (!meet_poll(e, cl, true)) return SR_NOT_READY;
    cl.step = 2;
  }
  if (cl.step == 2) {
    if (!move_issue(e, cl, MV_BODY, it.n_ctas, 0, 0, 0)) return SR_NOT_READY;
    cl.step = 3;
  }
  if (cl.step == 3) {
    if (!move_finished(e, cl)) return SR_NOT_READY;
    // a failed data phase (a rejected alltoallv) still meets its peers on the way out: a call retired before its exit
    // meeting would leave that meeting to pair with the entry meeting of the next call on the bank
    if (t == 0) {
      cl.body_err = cl.err;
      cl.err = 0;
    }
    meet_post(e, cl, false, 0, 0);
    cl.step = 4;
  }
  if (!meet_poll(e, cl, false)) return SR_NOT_READY;
  if (t == 0) cl.err |= cl.body_err;
  return SR_DONE;
}

// Ordering rules between calls in flight: collectives of one bank run one at a time in arrival order (their
// counters are sequential); the slot-ring collectives share one set of counters; eager point-to-point calls
// towards the same peer keep their order (sequence numbers).  Everything else may overtake.
__device__ bool blocked_by(const Call &later, const Call &earlier) {
  const WorkItem &a = later.item, &b = earlier.item;
  const bool ca = is_collective(a.desc.scenario), cb = is_collective(b.desc.scenario);
  if (ca && cb) return a.bank == b.bank || (a.algo == ALGO_EAGER && b.algo == ALGO_EAGER);
  const bool pa = a.desc.scenario == static_cast<uint32_t>(operation::send) || a.desc.scenario == static_cast<uint32_t>(operation::recv);
  if (pa && a.desc.scenario == b.desc.scenario && a.algo == ALGO_EAGER && b.algo == ALGO_EAGER)
    return a.members[a.desc.root_src_dst] == b.members[b.desc.root_src_dst];
  // slot-ring collectives and eager point-to-point share channel 0 of the slot rings
  if ((ca && a.algo == ALGO_EAGER && !cb && b.algo == ALGO_EAGER) || (cb && b.algo == ALGO_EAGER && pa && a.algo == ALGO_EAGER)) return true;
  return false;
}

__device__ void engine_control(const DevWorld &w, HostRing *hr, int nworkers) {
  __shared__ Call s_calls[MAX_ACTIVE];
  __shared__ uint32_t s_order[MAX_ACTIVE]; // active slots, oldest first
  __shared__ uint32_t s_nactive;
  __shared__ uint32_t s_flag, s_err, s_leave;
  __shared__ unsigned long long s_moves, s_host_fetched;
  Ctrl *me = my_ctrl(w);
  EngineArea *ea = engine_area(w);
  const uint32_t t = threadIdx.x;
  PlanCfg pcfg;
  memcpy(&pcfg, me->plan_cfg_words, sizeof(PlanCfg));
  if (t < MAX_ACTIVE) s_calls[t].active = 0;
  if (t == 0) {
    s_nactive = 0;
    s_moves = dev::ld_acquire_gpu(&me->move_tail);
    s_host_fetched = me->host_fetched;
    s_leave = 0;
    hr->state = ENG_RUNNING;
  }
  __syncthreads();
  EngCtx e{w, me, ea, nworkers, &s_moves, &s_flag};
  unsigned long long fetched = me->cmd_fetched;
  unsigned long long last_work_ns = dev::globaltimer_ns();
  const uint32_t idle_us = hr->idle_us;
  for (;;) {
    bool progressed = false;
    // ---- fetch new commands while there is room (at most a few per pass: a fresh command is stepped right away)
    for (int nf = 0; nf < 4; ++nf) {
      uint32_t have = 0;
      if (t == 0 && s_nactive < static_cast<uint32_t>(MAX_ACTIVE))
        have = dev::ld_acquire_sys(&me->cmd_ready[fetched % RING_SLOTS]) == fetched + 1 ? 1u : 0u;
      if (!bcast0(e, have)) break;
      // free slot (uniform: every thread scans the same shared state)
      uint32_t slot = 0;
      while (s_calls[slot].active) ++slot;
      Call &cl = s_calls[slot];
      copy_words(&cl.item, &ea->cmd_ring[fetched % RING_SLOTS].item, blockDim.x);
      __syncthreads();
      if (t == 0) {
        cl.err = 0;
        cl.body_err = 0;
        if (!(cl.item.flags & WF_PLANNED)) {
          // device-issued descriptor: decode + plan here, from the device copy of exchange memory
          const CallDesc d = cl.item.desc;
          WorkItem wi;
          const uint32_t err = build_work_item_hd(me->exch, pcfg, w.world, d, me->engine_timeout_us, wi);
          if (err) {
            wi.desc.scenario = static_cast<uint32_t>(operation::nop);
            wi.algo = ALGO_LOCAL;
            wi.n_ctas = 1;
            cl.err = err;
          }
          cl.item = wi;
        } else {
          s_host_fetched += 1;
        }
        cl.item.flags |= WF_ENGINE;
        // alltoallv: this rank's own check of its counts, published at the entry meeting (collectives.cuh)
        if (cl.item.desc.scenario == static_cast<uint32_t>(operation::alltoallv))
          cl.off0[cl.item.comm_rank] = k::a2av_entry_off(w.window + static_cast<uint64_t>(w.rank) * w.heap_bytes, cl.item);
        cl.ticket1 = fetched + 1;
        cl.t_start = dev::globaltimer_ns();
        cl.step = 0;
        cl.progress = 0;
        cl.move_id = 0;
        cl.note_slot = cl.note_seq = 0;
        cl.active = 1;
        s_order[s_nactive] = slot;
        s_nactive += 1;
        // producers wait on cmd_fetched only when the ring is full: plain stores, ordered by the fences of later steps
        me->cmd_fetched = fetched + 1;
        me->host_fetched = s_host_fetched;
      }
      __syncthreads();
      ++fetched;
      progressed = true;
      if (s_nactive == 1) break; // nothing else in flight: run it now
    }
    // ---- step every call in flight, oldest first
    for (uint32_t i = 0; i < s_nactive; ++i) {
      const uint32_t slot = s_order[i];
      Call &cl = s_calls[slot];
      bool blocked = false;
      for (uint32_t j = 0; j < i && !blocked; ++j) blocked = blocked_by(cl, s_calls[s_order[j]]);
      if (blocked) continue;
      if (t == 0) s_err = 0;
      __syncthreads();
      uint32_t r = cl.err ? SR_DONE : step_call(e, cl, &s_err);
      __syncthreads();
      if (r == SR_NOT_READY) {
        // parked: give up on it once its wait budget is spent (reference: *_TIMEOUT_ERROR)
        uint32_t expired = 0;
        if (t == 0) {
          me->eng_parks += 1;
          expired = dev::globaltimer_ns() - cl.t_start > static_cast<unsigned long long>(cl.item.timeout_us) * 1000ull ? 1u : 0u;
          if (expired) cl.err |= RECEIVE_TIMEOUT_ERROR;
        }
        if (!bcast0(e, expired)) continue;
      }
      // ---- retire
      if (t == 0) {
        const uint32_t rc = cl.err | s_err;
        const unsigned long long dur = dev::globaltimer_ns() - cl.t_start;
        me->exch[exchmem::RETCODE / 4] = rc;
        me->exch[exchmem::PERFCNT_LO / 4] = static_cast<uint32_t>(dur);
        if (cl.item.hc_ptr) publish_completion(reinterpret_cast<HostCompletion *>(cl.item.hc_ptr), cl.item.req_seq, rc, dur);
        dev::st_release_sys(&me->cmd_status[(cl.ticket1 - 1) % RING_SLOTS], cl.ticket1 | (static_cast<unsigned long long>(rc) << 32));
        me->eng_calls_done += 1;
        cl.active = 0;
        for (uint32_t j = i; j + 1 < s_nactive; ++j) s_order[j] = s_order[j + 1];
        s_nactive -= 1;
      }
      __syncthreads();
      --i; // the list moved up
      progressed = true;
    }
    if (progressed) {
      last_work_ns = dev::globaltimer_ns();
      continue;
    }
    // ---- idle: park after idle_us unless pinned or calls are in flight; leave when told to stop.  The host-side
    // words live in pinned host memory (a PCIe round trip each): they are only looked at after 20 us without work,
    // so polling the command ring stays a device-memory loop.
    if (t == 0) {
      uint32_t leave = 0;
      const unsigned long long idle_ns = dev::globaltimer_ns() - last_work_ns;
      if (idle_ns > 20000ull) {
        const uint32_t stop = hr->stop;
        const bool idle_long = idle_us != 0 && idle_ns > static_cast<unsigned long long>(idle_us) * 1000ull;
        if (stop || (idle_long && s_nactive == 0 && hr->pins == 0 && hr->clients == dev::ld_acquire_sys(&me->clients_done))) {
          hr->state = ENG_EXITING;
          dev::fence_sc_sys();
          // Dekker handshake with the host (submit / pin / client_begin write their word, fence, then read `state`): everything
          // that may have changed since the decision above is read again AFTER `state = EXITING` has been published
          const bool pending = hr->submitted != s_host_fetched || dev::ld_acquire_sys(&me->cmd_ready[fetched % RING_SLOTS]) == fetched + 1 ||
                               hr->pins != 0 || hr->clients != dev::ld_acquire_sys(&me->clients_done);
          if ((pending || s_nactive != 0) && !stop) hr->state = ENG_RUNNING; // a submit raced with parking: keep going
          else leave = 1;
        }
        if (!leave && idle_ns > 100000ull) dev::nanosleep(s_nactive ? 20 : 100); // back off after 100 us of nothing
      }
      s_leave = leave;
    }
    __syncthreads();
    if (s_leave) {
      if (t == 0) {
        dev::st_release_sys(&me->engine_exit, 1u);
        __threadfence_system();
        hr->state = ENG_STOPPED;
      }
      return;
    }
  }
}

__global__ void __launch_bounds__(k::BLOCK) k_engine(DevWorld w, HostRing *hr, int nworkers) {
  if (static_cast<int>(blockIdx.x) == nworkers) engine_control(w, hr, nworkers);
  else engine_worker(w, nworkers);
}

__global__ void k_engine_prepare(DevWorld w, PlanCfg cfg, uint32_t timeout_us) {
  Ctrl *me = my_ctrl(w);
  memcpy(me->plan_cfg_words, &cfg, sizeof(PlanCfg));
  me->engine_timeout_us = timeout_us;
  me->engine_exit = 0;
}

// The host-call proxy (hostctrl): places a planned work item in the command ring in stream order and, if
// `wait_done`, holds the stream until the engine has retired it.
__global__ void __launch_bounds__(32) k_submit(DevWorld w, WorkItem item, int wait_done) {
  asm volatile("griddepcontrol.wait;" ::: "memory"); // (programmatic dependent launch, see k_call)
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  Ctrl *me = my_ctrl(w);
  EngineArea *ea = engine_area(w);
  unsigned long long t = 0;
  const unsigned long long budget_ns = static_cast<unsigned long long>(item.timeout_us) * 1000ull;
  if (threadIdx.x == 0) {
    t = atomicAdd(&me->cmd_tail, 1ull);
    const unsigned long long t0 = dev::globaltimer_ns();
    while (t >= dev::ld_acquire_sys(&me->cmd_fetched) + RING_SLOTS) { // ring full
      dev::nanosleep(100);
      if (dev::globaltimer_ns() - t0 > budget_ns) break; // no engine is consuming (a tool serialising kernels?): give up
    }
  }
  t = __shfl_sync(0xffffffffu, t, 0);
  copy_words(&ea->cmd_ring[t % RING_SLOTS].item, &item, 32);
  __syncwarp();
  if (threadIdx.x == 0) {
    __threadfence();
    dev::st_release_sys(&me->cmd_ready[t % RING_SLOTS], t + 1);
    if (wait_done) {
      const unsigned long long *st = &me->cmd_status[t % RING_SLOTS];
      const unsigned long long t0 = dev::globaltimer_ns();
      uint32_t spins = 0;
      // (>=: a later occupant of the slot may have retired already if 128 calls overtook a parked one)
      while (static_cast<int32_t>(static_cast<uint32_t>(dev::ld_acquire_sys(st)) - static_cast<uint32_t>(t + 1)) < 0) {
        if (++spins > 64) dev::nanosleep(spins > 1024 ? 200 : 20);
        // the engine retires a call within its wait budget (parked calls time out there); twice that without an
        // answer means no engine is running next to this proxy
        if ((spins & 0x3FF) == 0 && dev::globaltimer_ns() - t0 > 2 * budget_ns + 1000000ull) break;
      }
    }
  }
}

// ------------------------------------------------------ direct-launch path
// One kernel per call, stream-ordered like any other CUDA work; shares every
// device function with the engine above (one translation unit, one copy).
__global__ void __launch_bounds__(k::BLOCK) k_call(DevWorld w, WorkItem it, HostCompletion *hc) {
  __shared__ uint32_t s_err;
  // Programmatic dependent launch: this kernel may have been scheduled while its predecessor on the stream was still
  // draining (the launch latency of back-to-back collectives overlaps the previous one's tail); nothing is read
  // before the predecessor has completed.  The successor is released right after, so at most one is ever pre-staged.
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const unsigned long long t0 = dev::globaltimer_ns();
  if (threadIdx.x == 0) s_err = 0;
  __syncthreads();
  k::run_work(w, it, blockIdx.x, gridDim.x, &s_err);
  __syncthreads();
  if (threadIdx.x == 0) {
    Ctrl *me = my_ctrl(w);
    if (blockIdx.x == 0) { // stream helper kernels that ran before this call report through it
      const uint32_t se = me->strm_err;
      if (se) {
        s_err |= se;
        me->strm_err = 0;
      }
    }
    const unsigned long long t1 = dev::globaltimer_ns();
    if (it.flags & WF_CHAIN) {
      // a later kernel of the same lowered call reports for all of them
      if (s_err) atomicOr(&me->strm_err, s_err);
    } else if (gridDim.x == 1) {
      if (hc) publish_completion(hc, it.req_seq, s_err, t1 - t0);
    } else {
      Completion *cp = &me->comp[it.req_slot];
      if (s_err) atomicOr(&cp->retcode, s_err);
      atomicMin(&cp->t_start, t0);
      atomicMax(&cp->t_end, t1);
      __threadfence();
      if (atomicAdd(&cp->done_ctas, 1u) == gridDim.x - 1) {
        // last CTA out: publish to the host and recycle the record
        __threadfence();
        const uint32_t rc = cp->retcode;
        const unsigned long long dur = cp->t_end - cp->t_start;
        cp->retcode = 0;
        cp->done_ctas = 0;
        cp->t_start = ~0ull;
        cp->t_end = 0;
        if (hc) publish_completion(hc, it.req_seq, rc, dur);
      }
    }
  }
}

cudaError_t launch_call(const DevWorld &w, const WorkItem &item, HostCompletion *hc_dev, cudaStream_t stream) {
  static const bool pdl = [] {
    const char *e = std::getenv("ACCL_PDL");
    return !e || std::atoi(e) != 0;
  }();
  cudaLaunchConfig_t lc = {};
  lc.gridDim = dim3(item.n_ctas);
  lc.blockDim = dim3(k::BLOCK);
  lc.stream = stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  lc.attrs = at;
  lc.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&lc, k_call, w, item, hc_dev);
}

__global__ void k_reset_ctrl(DevWorld w) {
  Ctrl *me = my_ctrl(w);
  // everything after the exchange memory is protocol state
  uint32_t *p = reinterpret_cast<uint32_t *>(&me->pad[0]);
  const size_t n = (sizeof(Ctrl) - offsetof(Ctrl, pad)) / 4;
  for (size_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) p[i] = 0;
  // LL staging: a stale line must never carry a sequence number that will be used again
  uint4 *ll = reinterpret_cast<uint4 *>(w.window + static_cast<uint64_t>(w.rank) * w.heap_bytes + w.ll_off);
  const size_t nl = stg_area_bytes(w.world, w.ll_bytes) / 16;
  for (size_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nl; i += static_cast<size_t>(gridDim.x) * blockDim.x) ll[i] = make_uint4(0, 0, 0, 0);
}
__global__ void k_init_comp(DevWorld w) {
  Ctrl *me = my_ctrl(w);
  for (int i = threadIdx.x; i < N_REQ_SLOTS; i += blockDim.x) me->comp[i].t_start = ~0ull;
}

cudaError_t launch_reset_ctrl(const DevWorld &w, cudaStream_t stream) {
  k_reset_ctrl<<<64, 256, 0, stream>>>(w);
  k_init_comp<<<1, 256, 0, stream>>>(w);
  return cudaGetLastError();
}

// ---------------------------------------------------------------- stream port
// FIFO -> local buffer / local buffer -> FIFO of rank dst_rank (my own: RES_STREAM results; a peer's:
// stream_put).  One CTA each; the bodies are the device API's Data port (accl/device/api.cuh).
__global__ void __launch_bounds__(512) k_stream_pop(DevWorld w, uint64_t dst_off, uint64_t bytes, uint32_t strm, uint32_t timeout_us) {
  char *heap = w.window + static_cast<uint64_t>(w.rank) * w.heap_bytes;
  device::Data port(w, strm);
  const uint32_t e = port.pull(heap + dst_off, bytes, static_cast<uint64_t>(timeout_us) * 1000ull);
  if (e && threadIdx.x == 0) atomicOr(&reinterpret_cast<Ctrl *>(heap)->strm_err, e);
}

__global__ void __launch_bounds__(512) k_stream_push(DevWorld w, uint32_t dst_rank, uint64_t src_off, uint64_t bytes, uint32_t strm,
                                                     uint32_t timeout_us) {
  char *heap = w.window + static_cast<uint64_t>(w.rank) * w.heap_bytes;
  device::Data port(w, strm);
  const uint32_t e = port.push(heap + src_off, bytes, static_cast<int>(dst_rank), static_cast<uint64_t>(timeout_us) * 1000ull);
  if (e && threadIdx.x == 0) atomicOr(&reinterpret_cast<Ctrl *>(heap)->strm_err, e);
}

cudaError_t launch_stream_pop(const DevWorld &w, uint64_t dst_off, uint64_t bytes, uint32_t strm, uint32_t timeout_us, cudaStream_t stream) {
  k_stream_pop<<<1, 512, 0, stream>>>(w, dst_off, bytes, strm, timeout_us);
  return cudaGetLastError();
}
cudaError_t launch_stream_push(const DevWorld &w, uint32_t dst_rank, uint64_t src_off, uint64_t bytes, uint32_t strm, uint32_t timeout_us,
                               cudaStream_t stream) {
  k_stream_push<<<1, 512, 0, stream>>>(w, dst_rank, src_off, bytes, strm, timeout_us);
  return cudaGetLastError();
}

void preload_engine_kernels() {
  cudaFuncAttributes a;
  cudaFuncGetAttributes(&a, k_stream_pop);
  cudaFuncGetAttributes(&a, k_stream_push);
  cudaFuncGetAttributes(&a, k_engine);
  cudaFuncGetAttributes(&a, k_engine_prepare);
  cudaFuncGetAttributes(&a, k_submit);
  cudaFuncGetAttributes(&a, k_call);
  cudaFuncGetAttributes(&a, k_reset_ctrl);
  cudaFuncGetAttributes(&a, k_init_comp);
}

// --------------------------------------------------------------------- host
struct Engine::Impl {
  HostRing *ring = nullptr, *ring_dev = nullptr;
  cudaStream_t stream = nullptr;
  unsigned long long submitted = 0;
  int nworkers = 0;
  std::mutex m;
};

static_assert(sizeof(PlanCfg) <= sizeof(((Ctrl *)nullptr)->plan_cfg_words), "PlanCfg must fit plan_cfg_words");

Engine::Engine(CudaDevice &dev) : dev_(dev), impl_(new Impl()) {
  ACCL_CUDART(cudaSetDevice(dev_.device()));
  ACCL_CUDART(cudaHostAlloc(reinterpret_cast<void **>(&impl_->ring), sizeof(HostRing), cudaHostAllocMapped | cudaHostAllocPortable));
  std::memset(impl_->ring, 0, sizeof(HostRing));
  ACCL_CUDART(cudaHostGetDevicePointer(reinterpret_cast<void **>(&impl_->ring_dev), impl_->ring, 0));
  int lo = 0, hi = 0;
  cudaDeviceGetStreamPriorityRange(&lo, &hi);
  ACCL_CUDART(cudaStreamCreateWithPriority(&impl_->stream, cudaStreamNonBlocking, hi));
  // leave SMs for the proxies and for the application: the engine never takes the whole chip
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev_.device());
  int nw = dev_.config().engine_workers > 0 ? dev_.config().engine_workers : dev_.config().max_ctas;
  nw = std::max(1, std::min(nw, std::max(1, sms - 16)));
  impl_->nworkers = nw;
  impl_->ring->idle_us = static_cast<uint32_t>(dev_.config().engine_idle_us);
  impl_->ring->state = ENG_STOPPED;
}

Engine::~Engine() {
  try {
    stop();
  } catch (...) {
  }
  if (impl_) {
    cudaSetDevice(dev_.device());
    if (impl_->stream) cudaStreamDestroy(impl_->stream);
    // the ring is pinned host memory: cudaFreeHost synchronises the device, which is fine here
    if (impl_->ring) cudaFreeHost(impl_->ring);
  }
  delete impl_;
}

int Engine::workers() const { return impl_->nworkers; }

void Engine::launch_locked() {
  HostRing *r = impl_->ring;
  ACCL_CUDART(cudaSetDevice(dev_.device()));
  r->stop = 0;
  r->state = ENG_RUNNING; // optimistic: the kernel re-asserts it
  std::atomic_thread_fence(std::memory_order_seq_cst);
  k_engine_prepare<<<1, 1, 0, impl_->stream>>>(dev_.world(), dev_.plan_cfg(), dev_.timeout_us());
  k_engine<<<impl_->nworkers + 1, k::BLOCK, 0, impl_->stream>>>(dev_.world(), impl_->ring_dev, impl_->nworkers);
  ACCL_CUDART(cudaGetLastError());
}

// make sure an engine instance is (or will be) alive for everything submitted so far
void Engine::ensure_running_locked() {
  HostRing *r = impl_->ring;
  std::atomic_thread_fence(std::memory_order_seq_cst);
  for (;;) {
    const uint32_t st = r->state;
    if (st == ENG_RUNNING) return;
    if (st == ENG_STOPPED) {
      launch_locked();
      return;
    }
    std::this_thread::yield(); // EXITING: it either resumes or stops within microseconds
  }
}

void Engine::stop() {
  if (!impl_ || !impl_->ring) return;
  std::lock_guard<std::mutex> g(impl_->m);
  HostRing *r = impl_->ring;
  cudaSetDevice(dev_.device());
  if (r->state != ENG_STOPPED) {
    r->stop = 1;
    std::atomic_thread_fence(std::memory_order_seq_cst);
  }
  cudaStreamSynchronize(impl_->stream);
  r->state = ENG_STOPPED;
  r->stop = 0;
}

void Engine::pin() {
  std::lock_guard<std::mutex> g(impl_->m);
  impl_->ring->pins = impl_->ring->pins + 1;
  std::atomic_thread_fence(std::memory_order_seq_cst);
  ensure_running_locked();
}

void Engine::client_begin() {
  std::lock_guard<std::mutex> g(impl_->m);
  impl_->ring->clients = impl_->ring->clients + 1;
  std::atomic_thread_fence(std::memory_order_seq_cst);
  ensure_running_locked();
}

void Engine::clients_reset() {
  std::lock_guard<std::mutex> g(impl_->m);
  impl_->ring->clients = 0;
}

void Engine::unpin() {
  std::lock_guard<std::mutex> g(impl_->m);
  if (impl_->ring->pins) impl_->ring->pins = impl_->ring->pins - 1;
}

void Engine::submit(const WorkItem &w, HostCompletion *hc, cudaStream_t s, bool stream_waits) {
  std::lock_guard<std::mutex> g(impl_->m);
  HostRing *r = impl_->ring;
  WorkItem item = w;
  item.hc_ptr = reinterpret_cast<uint64_t>(hc);
  item.flags |= WF_ENGINE | WF_PLANNED;
  impl_->submitted += 1;
  r->submitted = impl_->submitted;
  std::atomic_thread_fence(std::memory_order_seq_cst);
  ensure_running_locked();
  cudaLaunchConfig_t lc = {};
  lc.gridDim = dim3(1);
  lc.blockDim = dim3(32);
  lc.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  lc.attrs = at;
  lc.numAttrs = 1;
  ACCL_CUDART(cudaLaunchKernelEx(&lc, k_submit, dev_.world(), item, stream_waits ? 1 : 0));
}

} // namespace cuda
} // namespace accl
