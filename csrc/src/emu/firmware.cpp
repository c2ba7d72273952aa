// Emulator control plane: protocol selection (eager vs rendezvous) and the
// collective algorithms, expressed as move instructions for the data mover
// and rendezvous mailbox operations.
//
// Behavioural model: the reference firmware
// (kernels/cclo/fw/sw_apps/ccl_offload_control/src/ccl_offload_control.c):
// eager = segmented sends into the peer's RX buffers, ring/daisy-chain
// algorithms with fused receive-reduce(-send); rendezvous = address exchange,
// one-sided write, completion note, flat/binomial trees, with calls that
// cannot progress parked in the retry queue (NOT_READY) and resumed at their
// saved step.  The code below is an independent formulation of those
// behaviours (resumable `Steps` instead of current_step gotos).
#include <algorithm>
#include <atomic>
#include <cstring>

#include "accl/common.hpp"
#include "accl/cuda/plan.hpp" // the H100 backend's call planner (host / device shared, plain C++): one-hop schedule selection
#include "engine_ctx.hpp"

namespace accl {
namespace emu {

namespace {
constexpr uint32_t BARRIER_TAG = 0xBA221E20u;

Operand imm(uint64_t addr, bool compressed = false) {
  Operand o;
  o.mode = MOVE_IMMEDIATE;
  o.addr = addr;
  o.compressed = compressed;
  return o;
}
Operand stream_op() {
  Operand o;
  o.mode = MOVE_STREAM;
  return o;
}
Operand next_of(const Operand &o) { // how the following segment addresses the same operand
  Operand n = o;
  if (o.mode == MOVE_IMMEDIATE || o.mode == MOVE_STRIDE || o.mode == MOVE_REPEAT) n.mode = MOVE_INCREMENT;
  return n;
}
bool tag_match(uint32_t want, uint32_t have) { return want == TAG_ANY || have == TAG_ANY || want == have; }
} // namespace

// Ordering among calls in flight (the reference runs one call at a time; this engine keeps many): a call that
// has not started yet must wait while an OLDER parked call competes for the same mailbox events —
//  * point to point: an elder send to the same (communicator, destination) / recv from the same source:
//    messages of one pair are matched in issue order (non-overtaking), whatever their tags;
//  * collectives: any elder collective on the same communicator (their notes carry no per-call identity).
// Without this a younger call dispatched at the wrong moment takes the address / completion note meant for its
// elder (found by the point-to-point property test: three parked sends, same peer, same tag).
bool Engine::elder_conflict(const EmuCall &c) {
  const operation op = static_cast<operation>(c.desc.scenario);
  const bool p2p = op == operation::send || op == operation::recv;
  const bool coll = op == operation::bcast || op == operation::scatter || op == operation::gather || op == operation::allgather ||
                    op == operation::reduce || op == operation::reduce_scatter || op == operation::allreduce ||
                    op == operation::alltoall || op == operation::alltoallv;
  if (!p2p && !coll) return false;
  std::lock_guard<std::mutex> g(q_m_);
  const size_t n = std::min(older_parked_, retry_calls_.size());
  for (size_t i = 0; i < n; ++i) {
    const CallDesc &e = retry_calls_[i].desc;
    if (e.comm != c.desc.comm) continue;
    const operation eo = static_cast<operation>(e.scenario);
    if (p2p) {
      // regardless of tags: the other side may match with TAG_ANY, so a pair's messages stay in issue order
      if (eo == op && e.root_src_dst == c.desc.root_src_dst) return true;
    } else {
      if (eo == operation::bcast || eo == operation::scatter || eo == operation::gather || eo == operation::allgather ||
          eo == operation::reduce || eo == operation::reduce_scatter || eo == operation::allreduce || eo == operation::alltoall ||
          eo == operation::alltoallv)
        return true;
    }
  }
  return false;
}

uint32_t Engine::dispatch(EmuCall &c) {
  const operation op = static_cast<operation>(c.desc.scenario);
  // collectives: checked here; point to point: only the rendezvous form waits for its elders (fw_send / fw_recv) —
  // an eager send must never park, or younger eager traffic to the same peer would take its sequence number
  if (op != operation::send && op != operation::recv && c.step == 0 && c.mask == 0 && elder_conflict(c)) return NOT_READY_ERROR;
  switch (op) {
  case operation::config: return fw_config(c);
  case operation::nop: return 0;
  case operation::copy: return fw_copy(c);
  case operation::combine: return fw_combine(c);
  case operation::send: return fw_send(c);
  case operation::recv: return fw_recv(c);
  case operation::bcast: return fw_bcast(c);
  case operation::scatter: return fw_scatter(c);
  case operation::gather: return fw_gather(c);
  case operation::allgather: return fw_allgather(c);
  case operation::reduce: return fw_reduce(c);
  case operation::reduce_scatter: return fw_reduce_scatter(c);
  case operation::allreduce: return fw_allreduce(c);
  case operation::barrier: return fw_barrier(c);
  case operation::alltoall: return fw_alltoall(c);
  case operation::alltoallv: return fw_alltoallv(c);
  }
  return COLLECTIVE_NOT_IMPLEMENTED;
}

uint32_t Engine::fw_config(EmuCall &c) {
  switch (static_cast<cfgFunc>(c.desc.function)) {
  case cfgFunc::reset_periph:
    soft_reset();
    return 0;
  case cfgFunc::enable_pkt: {
    std::lock_guard<std::mutex> g(rx_m_);
    {
      std::lock_guard<std::mutex> e(exch_m_);
      exch_[exchmem::PKT_ENABLED / 4] = 1;
      const uint32_t n = exch_[exchmem::EAGER_RX_BUF_COUNT / 4];
      for (uint32_t i = 0; i < n; ++i) // post every idle buffer (rxbuf_enqueue)
        if (exch_[exchmem::rxbuf_offset(i, exchmem::RX_STATUS) / 4] == exchmem::RX_IDLE)
          exch_[exchmem::rxbuf_offset(i, exchmem::RX_STATUS) / 4] = exchmem::RX_ENQUEUED;
    }
    rx_try_fill_locked();
    return 0;
  }
  case cfgFunc::set_timeout:
    write_exch(exchmem::TIMEOUT, c.desc.count);
    return 0;
  case cfgFunc::set_max_eager_msg_size:
    if (c.desc.count < read_exch(exchmem::EAGER_RX_BUF_SIZE)) return EAGER_THRESHOLD_INVALID;
    write_exch(exchmem::MAX_EAGER_SIZE, c.desc.count);
    return 0;
  case cfgFunc::set_max_rendezvous_msg_size:
    if (c.desc.count <= read_exch(exchmem::MAX_EAGER_SIZE)) return RENDEZVOUS_THRESHOLD_INVALID;
    write_exch(exchmem::MAX_RENDEZVOUS_SIZE, c.desc.count);
    return 0;
  }
  return COLLECTIVE_NOT_IMPLEMENTED;
}

// ------------------------------------------------------------- primitives
uint32_t Engine::seg_elems(const Ctx &x) const {
  const dataType w = x.eth_c ? x.ar.c : x.ar.u;
  if (is_fp8(w) && x.ar.ratio_log > 0) {
    const uint32_t blk = 1u << x.ar.ratio_log;
    return x.rxbuf_size / (blk + 4) * blk;
  }
  return x.rxbuf_size / std::max(1u, dtype_bytes(w));
}

uint32_t Engine::egr_send(Ctx &x, uint32_t dst, Operand src, uint32_t count, uint32_t tag, bool to_stream,
                          uint32_t strm) {
  const uint32_t seg = seg_elems(x);
  if (seg == 0) return DMA_SIZE_ERROR;
  uint32_t err = 0;
  for (uint32_t off = 0; off < count && !err; off += seg) {
    Move m;
    m.op0 = off == 0 ? src : next_of(src);
    m.count = std::min(seg, count - off);
    m.res_remote = true;
    m.res.mode = to_stream ? MOVE_STREAM : MOVE_IMMEDIATE;
    m.strm = strm;
    m.dst_rank = dst;
    m.tx_tag = tag;
    m.eth_compressed = x.eth_c;
    err |= execute(x, m);
  }
  return err;
}

uint32_t Engine::egr_recv(Ctx &x, uint32_t src, Operand dst, uint32_t count, uint32_t tag, bool to_stream,
                          uint32_t strm) {
  const uint32_t seg = seg_elems(x);
  if (seg == 0) return DMA_SIZE_ERROR;
  uint32_t err = 0;
  for (uint32_t off = 0; off < count && !err; off += seg) {
    Move m;
    m.op0.mode = MOVE_ON_RECV;
    m.rx_src = src;
    m.rx_tag = tag;
    m.count = std::min(seg, count - off);
    m.eth_compressed = x.eth_c;
    if (to_stream) {
      m.res.mode = MOVE_STREAM;
      m.strm = strm;
    } else {
      m.res = off == 0 ? dst : next_of(dst);
    }
    err |= execute(x, m);
  }
  return err;
}

uint32_t Engine::egr_recv_reduce(Ctx &x, uint32_t src, Operand local, Operand dst, uint32_t count, uint32_t tag) {
  const uint32_t seg = seg_elems(x);
  if (seg == 0) return DMA_SIZE_ERROR;
  uint32_t err = 0;
  for (uint32_t off = 0; off < count && !err; off += seg) {
    Move m;
    m.op0 = off == 0 ? local : next_of(local);
    m.op1.mode = MOVE_ON_RECV;
    m.rx_src = src;
    m.rx_tag = tag;
    m.count = std::min(seg, count - off);
    m.func = x.fn();
    m.eth_compressed = x.eth_c;
    if (dst.mode == MOVE_STREAM) {
      m.res.mode = MOVE_STREAM;
      m.strm = x.stream_id();
    } else {
      m.res = off == 0 ? dst : next_of(dst);
    }
    err |= execute(x, m);
  }
  return err;
}

uint32_t Engine::egr_recv_reduce_send(Ctx &x, uint32_t src, Operand local, uint32_t dst_rank, uint32_t count,
                                      uint32_t tag) {
  const uint32_t seg = seg_elems(x);
  if (seg == 0) return DMA_SIZE_ERROR;
  uint32_t err = 0;
  for (uint32_t off = 0; off < count && !err; off += seg) {
    Move m;
    m.op0 = off == 0 ? local : next_of(local);
    m.op1.mode = MOVE_ON_RECV;
    m.rx_src = src;
    m.rx_tag = tag;
    m.count = std::min(seg, count - off);
    m.func = x.fn();
    m.eth_compressed = x.eth_c;
    m.res_remote = true;
    m.res.mode = MOVE_IMMEDIATE;
    m.dst_rank = dst_rank;
    m.tx_tag = tag;
    err |= execute(x, m);
  }
  return err;
}

// which kind of call a mailbox note belongs to (carried in the otherwise unused seqn field of note packets)
template <typename C> static uint32_t note_kind(const C &x) {
  return (x.op == operation::send || x.op == operation::recv) ? 1u : (0x100u | static_cast<uint32_t>(x.op));
}

void Engine::rndzv_post_addr(Ctx &x, uint32_t to_rank, uint64_t vaddr, uint32_t count, uint32_t tag) {
  Packet p;
  p.hdr.msg_type = static_cast<uint32_t>(MsgType::RNDZVS_INIT);
  p.hdr.src = static_cast<uint32_t>(rank_);
  p.hdr.dst = x.comm.session[to_rank];
  p.hdr.tag = tag;
  p.hdr.vaddr = vaddr;
  p.hdr.count = count;
  p.hdr.comm_sig = x.comm.sig;
  p.hdr.host = vaddr >= HOST_BASE;
  p.hdr.seqn = note_kind(x);
  fabric_->send(std::move(p));
}

// A parked call is being retired with a timeout: remove the mailbox entries that belong to it, here and (for a
// rendezvous receive, whose address note sits in the sender's mailbox) at the peer.
void Engine::purge_notes_of(EmuCall &c) {
  Ctx x;
  uint32_t e = 0;
  if (!decode(c, x, e)) return;
  const bool p2p = x.op == operation::send || x.op == operation::recv;
  {
    std::lock_guard<std::mutex> g(q_m_);
    const uint32_t peer = p2p && x.root < x.comm.size ? x.comm.session[x.root] : 0;
    addr_notes_.remove_if([&](const AddrNote &n) {
      return n.comm_sig == x.comm.sig && n.kind == note_kind(x) && (!p2p || (n.src == peer && tag_match(x.tag, n.tag)));
    });
    done_notes_.remove_if([&](const DoneNote &n) {
      return n.comm_sig == x.comm.sig && n.kind == note_kind(x) && (!p2p || (n.src == peer && tag_match(x.tag, n.tag)));
    });
  }
  if (x.op == operation::recv && !x.eager && c.step != 0 && x.root < x.comm.size) {
    Packet p;
    p.hdr.msg_type = static_cast<uint32_t>(MsgType::RNDZVS_CANCEL);
    p.hdr.src = static_cast<uint32_t>(rank_);
    p.hdr.dst = x.comm.session[x.root];
    p.hdr.tag = x.tag;
    p.hdr.vaddr = x.a2;
    p.hdr.comm_sig = x.comm.sig;
    p.hdr.seqn = note_kind(x);
    fabric_->send(std::move(p));
  }
}

bool Engine::rndzv_take_addr(Ctx &x, uint32_t from_rank, uint32_t tag, uint64_t &vaddr) {
  std::lock_guard<std::mutex> g(q_m_);
  const uint32_t src = x.comm.session[from_rank];
  for (auto it = addr_notes_.begin(); it != addr_notes_.end(); ++it)
    if (it->comm_sig == x.comm.sig && it->src == src && it->kind == note_kind(x) && tag_match(tag, it->tag)) {
      vaddr = it->vaddr;
      addr_notes_.erase(it);
      return true;
    }
  return false;
}

bool Engine::rndzv_take_any_addr(Ctx &x, uint32_t exclude_mask, uint32_t tag, uint32_t &from_rank, uint64_t &vaddr) {
  std::lock_guard<std::mutex> g(q_m_);
  for (auto it = addr_notes_.begin(); it != addr_notes_.end(); ++it) {
    if (it->comm_sig != x.comm.sig || it->kind != note_kind(x) || !tag_match(tag, it->tag)) continue;
    for (uint32_t r = 0; r < x.comm.size; ++r)
      if (x.comm.session[r] == it->src && !(exclude_mask & (1u << r))) {
        from_rank = r;
        vaddr = it->vaddr;
        addr_notes_.erase(it);
        return true;
      }
  }
  return false;
}

uint32_t Engine::rndzv_write(Ctx &x, uint32_t dst_rank, uint64_t src_addr, uint64_t vaddr, uint32_t count,
                             uint32_t tag) {
  Move m;
  m.op0 = imm(src_addr);
  m.count = count;
  m.res_remote = true;
  m.rendezvous = true;
  m.res.mode = MOVE_IMMEDIATE;
  m.dst_rank = dst_rank;
  m.remote_vaddr = vaddr;
  m.tx_tag = tag;
  uint32_t err = count ? execute(x, m) : 0;
  Packet p; // completion note follows the data on the same ordered channel
  p.hdr.msg_type = static_cast<uint32_t>(MsgType::RNDZVS_WR_DONE);
  p.hdr.src = static_cast<uint32_t>(rank_);
  p.hdr.dst = x.comm.session[dst_rank];
  p.hdr.tag = tag;
  p.hdr.comm_sig = x.comm.sig;
  p.hdr.seqn = note_kind(x);
  fabric_->send(std::move(p));
  return err;
}

bool Engine::rndzv_take_done(Ctx &x, uint32_t from_rank, uint32_t tag) {
  std::lock_guard<std::mutex> g(q_m_);
  const uint32_t src = x.comm.session[from_rank];
  for (auto it = done_notes_.begin(); it != done_notes_.end(); ++it)
    if (it->comm_sig == x.comm.sig && it->src == src && it->barrier == (tag == BARRIER_TAG) && it->kind == note_kind(x) &&
        tag_match(tag, it->tag)) {
      done_notes_.erase(it);
      return true;
    }
  return false;
}

bool Engine::rndzv_take_any_done(Ctx &x, uint32_t exclude_mask, uint32_t tag, uint32_t &from_rank) {
  std::lock_guard<std::mutex> g(q_m_);
  for (auto it = done_notes_.begin(); it != done_notes_.end(); ++it) {
    if (it->comm_sig != x.comm.sig || it->barrier != (tag == BARRIER_TAG) || it->kind != note_kind(x) || !tag_match(tag, it->tag)) continue;
    for (uint32_t r = 0; r < x.comm.size; ++r)
      if (x.comm.session[r] == it->src && !(exclude_mask & (1u << r))) {
        from_rank = r;
        done_notes_.erase(it);
        return true;
      }
  }
  return false;
}

#define FW_DECODE(x)                                                         \
  Ctx x;                                                                     \
  {                                                                          \
    uint32_t _e = 0;                                                         \
    if (!decode(c, x, _e)) return _e;                                        \
  }

// ------------------------------------------------------- local primitives
uint32_t Engine::fw_copy(EmuCall &c) {
  FW_DECODE(x);
  Move m;
  m.op0 = x.op0_stream() ? stream_op() : imm(x.a0, x.op0_c());
  m.res = x.res_stream() ? stream_op() : imm(x.a2, x.res_c());
  m.strm = x.stream_id();
  m.count = x.count;
  return execute(x, m);
}

uint32_t Engine::fw_combine(EmuCall &c) {
  FW_DECODE(x);
  Move m;
  m.op0 = x.op0_stream() ? stream_op() : imm(x.a0, x.op0_c());
  m.op1 = imm(x.a1, x.op1_c());
  m.res = x.res_stream() ? stream_op() : imm(x.a2, x.res_c());
  m.strm = x.stream_id();
  m.count = x.count;
  m.func = x.fn();
  return execute(x, m);
}

// ---------------------------------------------------------- point to point
uint32_t Engine::fw_send(EmuCall &c) {
  FW_DECODE(x);
  if (x.root >= x.comm.size) return CONFIG_SWITCH_ERROR;
  if (!x.eager) {
    // rendezvous: elder rendezvous sends to the same peer go first (non-overtaking) ...
    if (c.step == 0 && c.mask == 0 && elder_conflict(c)) return NOT_READY_ERROR;
    // ... then we need the receiver's address; park until it shows up
    uint64_t vaddr = 0;
    if (!rndzv_take_addr(x, x.root, x.tag, vaddr)) return NOT_READY_ERROR;
    return rndzv_write(x, x.root, x.a0, vaddr, x.count, x.tag);
  }
  Operand src = x.op0_stream() ? stream_op() : imm(x.a0, x.op0_c());
  // RES_STREAM on a send == stream_put: lands in stream `tag` of the peer
  return egr_send(x, x.root, src, x.count, x.tag, x.res_stream(), x.res_stream() ? x.tag : 0);
}

uint32_t Engine::fw_recv(EmuCall &c) {
  FW_DECODE(x);
  if (x.root >= x.comm.size) return CONFIG_SWITCH_ERROR;
  if (!x.eager) {
    if (c.step == 0 && c.mask == 0 && elder_conflict(c)) return NOT_READY_ERROR; // elder receives from this source first
    Steps st(c.step);
    st([&] { rndzv_post_addr(x, x.root, x.a2, x.count * x.ubytes(), x.tag); return true; });
    if (!st([&] { return rndzv_take_done(x, x.root, x.tag); })) return NOT_READY_ERROR;
    return 0;
  }
  return egr_recv(x, x.root, imm(x.a2, x.res_c()), x.count, x.tag, x.res_stream(), x.stream_id());
}

// --------------------------------------------------------------- broadcast
uint32_t Engine::fw_bcast(EmuCall &c) {
  FW_DECODE(x);
  const uint32_t P = x.comm.size, me = x.comm.local_rank, root = x.root;
  if (P == 1) return 0;
  if (x.eager) {
    if (me == root) {
      // segment-major so every peer streams at the same pace
      const uint32_t seg = seg_elems(x);
      if (!seg) return DMA_SIZE_ERROR;
      uint32_t err = 0;
      for (uint32_t off = 0; off < x.count && !err; off += seg) {
        const uint32_t n = std::min(seg, x.count - off);
        bool first_peer = true;
        for (uint32_t r = 0; r < P && !err; ++r) {
          if (r == root) continue;
          Move m;
          m.op0 = imm(x.a0, x.op0_c());
          if (x.op0_stream()) m.op0 = stream_op(); // a streamed source can only feed one peer
          else if (!first_peer) m.op0.mode = MOVE_REPEAT;      // same segment again for the next peer
          else if (off != 0) m.op0.mode = MOVE_INCREMENT;      // next segment
          first_peer = false;
          m.count = n;
          m.res_remote = true;
          m.res.mode = MOVE_IMMEDIATE;
          m.dst_rank = r;
          m.tx_tag = x.tag;
          m.eth_compressed = x.eth_c;
          err |= execute(x, m);
        }
      }
      return err;
    }
    return egr_recv(x, root, imm(x.a0, x.op0_c()), x.count, x.tag, x.res_stream(), x.stream_id());
  }
  // ---- rendezvous
  const uint32_t flat_max = read_exch(exchmem::ONE_HOP_SCHEDULES) ? ~0u : read_exch(exchmem::BCAST_FLAT_TREE_MAX_RANKS);
  Steps st(c.step);
  if (P <= flat_max) {
    // flat tree: peers announce their buffers, root serves them in arrival order
    if (me == root) {
      const uint32_t all = ((1u << P) - 1) & ~(1u << root);
      while (c.mask != all) {
        uint32_t from = 0;
        uint64_t vaddr = 0;
        if (!rndzv_take_any_addr(x, c.mask | (1u << root), x.tag, from, vaddr)) return NOT_READY_ERROR;
        uint32_t err = rndzv_write(x, from, x.a0, vaddr, x.count, x.tag);
        if (err) return err;
        c.mask |= 1u << from;
      }
      return 0;
    }
    st([&] { rndzv_post_addr(x, root, x.a0, x.count * x.ubytes(), x.tag); return true; });
    if (!st([&] { return rndzv_take_done(x, root, x.tag); })) return NOT_READY_ERROR;
    return 0;
  }
  // binomial tree over ranks normalised so that the root is 0
  const uint32_t v = (me + P - root) % P;
  uint32_t err = 0;
  // receive from parent: the highest set bit of v
  if (v != 0) {
    uint32_t hb = 1;
    while ((hb << 1) <= v) hb <<= 1;
    const uint32_t parent = ((v - hb) + root) % P;
    st([&] { rndzv_post_addr(x, parent, x.a0, x.count * x.ubytes(), x.tag); return true; });
    if (!st([&] { return rndzv_take_done(x, parent, x.tag); })) return NOT_READY_ERROR;
  }
  // forward to children v + 2^k for 2^k > v
  uint32_t k = 1;
  while (k <= v) k <<= 1;
  for (; v + k < P; k <<= 1) {
    const uint32_t child = (v + k + root) % P;
    if (!st([&] {
          uint64_t vaddr = 0;
          if (!rndzv_take_addr(x, child, x.tag, vaddr)) return false;
          err |= rndzv_write(x, child, x.a0, vaddr, x.count, x.tag);
          return true;
        }))
      return NOT_READY_ERROR;
  }
  return err;
}

// ----------------------------------------------------------------- scatter
uint32_t Engine::fw_scatter(EmuCall &c) {
  FW_DECODE(x);
  const uint32_t P = x.comm.size, me = x.comm.local_rank, root = x.root;
  const uint64_t slice_bytes = x.op_bytes(x.op0_c(), x.count);
  if (x.eager) {
    if (me == root) {
      uint32_t err = 0;
      for (uint32_t r = 0; r < P && !err; ++r) {
        if (r == root) { // own slice: local copy
          Move m;
          m.op0 = imm(x.a0 + r * slice_bytes, x.op0_c());
          m.res = x.res_stream() ? stream_op() : imm(x.a2, x.res_c());
          m.strm = x.stream_id();
          m.count = x.count;
          err |= execute(x, m);
        } else {
          err |= egr_send(x, r, imm(x.a0 + r * slice_bytes, x.op0_c()), x.count, x.tag, false, 0);
        }
      }
      return err;
    }
    return egr_recv(x, root, imm(x.a2, x.res_c()), x.count, x.tag, x.res_stream(), x.stream_id());
  }
  Steps st(c.step);
  if (me == root) {
    uint32_t err = 0;
    st([&] {
      Move m;
      m.op0 = imm(x.a0 + root * slice_bytes);
      m.res = imm(x.a2);
      m.count = x.count;
      err |= execute(x, m);
      return true;
    });
    if (err) return err;
    const uint32_t all = ((1u << P) - 1) & ~(1u << root);
    while (c.mask != all) {
      uint32_t from = 0;
      uint64_t vaddr = 0;
      if (!rndzv_take_any_addr(x, c.mask | (1u << root), x.tag, from, vaddr)) return NOT_READY_ERROR;
      err = rndzv_write(x, from, x.a0 + from * slice_bytes, vaddr, x.count, x.tag);
      if (err) return err;
      c.mask |= 1u << from;
    }
    return 0;
  }
  st([&] { rndzv_post_addr(x, root, x.a2, x.count * x.ubytes(), x.tag); return true; });
  if (!st([&] { return rndzv_take_done(x, root, x.tag); })) return NOT_READY_ERROR;
  return 0;
}

// ------------------------------------------------------------------ gather
uint32_t Engine::fw_gather(EmuCall &c) {
  FW_DECODE(x);
  const uint32_t P = x.comm.size, me = x.comm.local_rank, root = x.root;
  const uint64_t slot_bytes = x.op_bytes(x.res_c(), x.count);
  if (x.eager && one_hop(x, 0)) {
    // fan-in: everybody sends its block straight to the root
    if (me != root) return egr_send(x, root, imm(x.a0), x.count, x.tag, false, 0);
    Move m;
    m.op0 = imm(x.a0);
    m.res = imm(x.a2 + root * slot_bytes);
    m.count = x.count;
    uint32_t err = execute(x, m);
    for (uint32_t k = 1; k < P && !err; ++k) {
      const uint32_t from = (root + P - k) % P;
      err |= egr_recv(x, from, imm(x.a2 + from * slot_bytes), x.count, x.tag, false, 0);
    }
    return err;
  }
  if (x.eager) {
    // daisy chain towards the root: r -> r+1 -> ... -> root.  A rank first
    // injects its own block, then relays the blocks of the ranks behind it.
    const uint32_t next = (me + 1) % P, prev = (me + P - 1) % P;
    const uint32_t dist = (root + P - me) % P; // hops from me to the root
    uint32_t err = 0;
    if (me == root) {
      Move m; // own contribution
      m.op0 = x.op0_stream() ? stream_op() : imm(x.a0, x.op0_c());
      m.res = imm(x.a2 + root * slot_bytes, x.res_c());
      m.count = x.count;
      err |= execute(x, m);
      for (uint32_t k = 1; k < P && !err; ++k) { // k-th arrival originates k hops upstream
        const uint32_t origin = (root + P - k) % P;
        err |= egr_recv(x, prev, imm(x.a2 + origin * slot_bytes, x.res_c()), x.count, x.tag, false, 0);
      }
      return err;
    }
    err |= egr_send(x, next, x.op0_stream() ? stream_op() : imm(x.a0, x.op0_c()), x.count, x.tag, false, 0);
    // relay P-1-dist blocks through a scratch buffer
    for (uint32_t k = 0; k + dist + 1 < P && !err; ++k) {
      // relay segment by segment: no scratch beyond the RX buffer is needed
      const uint32_t seg = seg_elems(x);
      for (uint32_t off = 0; off < x.count && !err; off += seg) {
        Move m; // receive one segment and forward it unchanged
        m.op0.mode = MOVE_ON_RECV;
        m.rx_src = prev;
        m.rx_tag = x.tag;
        m.count = std::min(seg, x.count - off);
        m.eth_compressed = x.eth_c;
        m.res_remote = true;
        m.res.mode = MOVE_IMMEDIATE;
        m.dst_rank = next;
        m.tx_tag = x.tag;
        err |= execute(x, m);
      }
    }
    return err;
  }
  // ---- rendezvous: root exposes up to `fanin` slots at a time
  Steps st(c.step);
  if (me == root) {
    uint32_t err = 0;
    st([&] {
      Move m;
      m.op0 = imm(x.a0);
      m.res = imm(x.a2 + root * slot_bytes);
      m.count = x.count;
      err |= execute(x, m);
      return true;
    });
    if (err) return err;
    uint32_t fanin = P - 1;
    if (x.count * x.ubytes() > read_exch(exchmem::GATHER_FLAT_TREE_MAX_COUNT) && !read_exch(exchmem::ONE_HOP_SCHEDULES))
      fanin = std::max(1u, read_exch(exchmem::GATHER_FLAT_TREE_MAX_FANIN));
    // peers are admitted in rank order, `fanin` outstanding at a time:
    // c.mask = peers whose completion has been collected; the admission
    // window is recomputed from it on every attempt
    const uint32_t all = ((1u << P) - 1) & ~(1u << root);
    // number of peers already posted is tracked in the step counter beyond step 1
    std::vector<uint32_t> order;
    for (uint32_t k = 1; k < P; ++k) order.push_back((root + k) % P);
    for (;;) {
      const uint32_t done_cnt = static_cast<uint32_t>(__builtin_popcount(c.mask));
      uint32_t posted = c.step - 1; // step 0 was the local copy
      while (posted < order.size() && posted < done_cnt + fanin) {
        const uint32_t r = order[posted];
        rndzv_post_addr(x, r, x.a2 + r * slot_bytes, x.count * x.ubytes(), x.tag);
        ++posted;
        ++c.step;
      }
      if (c.mask == all) return 0;
      uint32_t from = 0;
      if (!rndzv_take_any_done(x, c.mask | (1u << root), x.tag, from)) return NOT_READY_ERROR;
      c.mask |= 1u << from;
    }
  }
  uint64_t vaddr = 0;
  if (!rndzv_take_addr(x, root, x.tag, vaddr)) return NOT_READY_ERROR;
  return rndzv_write(x, root, x.a0, vaddr, x.count, x.tag);
}

// ---------------------------------------------------------------------------------------------------------------
// One-hop schedules (exchmem::ONE_HOP_SCHEDULES != 0): the exchanges the H100 backend runs on an NVSwitch domain,
// where every peer is one hop away — all-gather: every rank delivers its block straight to every peer;
// reduce-scatter: every rank delivers block q to its owner q, the owner reduces; all-reduce: everybody-sends-everything
// while small (or when the count does not split), reduce-scatter + all-gather above (plan.hpp: WF_ONESHOT /
// two-shot); rooted collectives take their flat forms.  Same primitives as the reference-style algorithms below
// (eager sends into RX buffers; address note, one-sided write, completion note), so the CPU suite exercises the
// data flow and the in-place hazards of the GPU schedules.  Uncompressed, non-stream calls only (as on the GPU, where
// compressed / stream calls take other paths); everything else keeps the ring / tree forms.
namespace {
std::atomic<uint64_t> g_one_hop_dispatches{0}; // process-wide statistics (ranks as threads share them): shown by debug_state
std::atomic<uint64_t> g_allreduce_one_shot{0}, g_allreduce_two_shot{0};
}
uint64_t one_hop_dispatches() { return g_one_hop_dispatches.load(); }
uint64_t one_hop_allreduce_forms(bool two_shot) { return two_shot ? g_allreduce_two_shot.load() : g_allreduce_one_shot.load(); }

bool Engine::one_hop(const Ctx &x, uint64_t landing_bytes) {
  if (!read_exch(exchmem::ONE_HOP_SCHEDULES) || x.cflags || x.sflags || x.comm.size < 2) return false;
  if (!x.eager && landing_bytes > x.spare_size) return false;
  if (x.call && x.call->step == 0 && x.call->mask == 0) g_one_hop_dispatches.fetch_add(1); // first attempt of the call
  return true;
}

// Every rank delivers `count` elements at own_block to slot `me` of every peer's dst_base (slots of blk_bytes).
// step / mask: resumable state of a parked call (mask bits 0-15: peers written, bits 16-20: completions collected).
uint32_t Engine::onehop_gather(Ctx &x, uint32_t &step, uint32_t &mask, uint64_t own_block, uint64_t dst_base, uint64_t blk_bytes,
                               uint32_t count, uint32_t last_extra) {
  const uint32_t P = x.comm.size, me = x.comm.local_rank;
  auto count_of = [&](uint32_t q) { return count + (q == P - 1 ? last_extra : 0); };
  uint32_t err = 0;
  if (x.eager) {
    for (uint32_t k = 1; k < P && !err; ++k) err |= egr_send(x, (me + k) % P, imm(own_block), count_of(me), x.tag, false, 0);
    for (uint32_t k = 1; k < P && !err; ++k) {
      const uint32_t from = (me + P - k) % P;
      err |= egr_recv(x, from, imm(dst_base + from * blk_bytes), count_of(from), x.tag, false, 0);
    }
    return err;
  }
  Steps st(step);
  st([&] {
    for (uint32_t r = 0; r < P; ++r)
      if (r != me) rndzv_post_addr(x, r, dst_base + r * blk_bytes, count_of(r) * x.ubytes(), x.tag);
    return true;
  });
  const uint32_t all = ((1u << P) - 1) & ~(1u << me);
  while ((mask & 0xFFFFu) != all) {
    uint32_t to = 0;
    uint64_t vaddr = 0;
    if (!rndzv_take_any_addr(x, (mask & 0xFFFFu) | (1u << me), x.tag, to, vaddr)) return NOT_READY_ERROR;
    err = rndzv_write(x, to, own_block, vaddr, count_of(me), x.tag);
    if (err) return err;
    mask |= 1u << to;
  }
  while (((mask >> 16) & 0x1Fu) != P - 1) {
    uint32_t from = 0;
    if (!rndzv_take_any_done(x, 1u << me, x.tag, from)) return NOT_READY_ERROR;
    mask += 1u << 16;
  }
  return 0;
}

// Every rank q contributes `count` elements at src_base + owner * src_stride to every owner (src_stride 0: the same
// vector to everybody — one-shot all-reduce); this rank reduces the P contributions for itself into dst.
// Rendezvous form: contributions land one at a time in scratch 0 and are folded ping-pong through scratch 1 / 2; the
// fold that writes dst waits until this rank has delivered all of its own contributions (dst may alias the source).
uint32_t Engine::onehop_reduce(Ctx &x, uint32_t &step, uint32_t &mask, uint64_t src_base, uint64_t src_stride, uint64_t dst,
                               uint32_t count, uint32_t last_extra) {
  const uint32_t P = x.comm.size, me = x.comm.local_rank;
  auto count_of = [&](uint32_t q) { return count + (q == P - 1 ? last_extra : 0); };
  const uint32_t mine = count_of(me);
  uint32_t err = 0;
  if (x.eager) {
    for (uint32_t k = 1; k < P && !err; ++k) {
      const uint32_t to = (me + k) % P;
      err |= egr_send(x, to, imm(src_base + to * src_stride), count_of(to), x.tag, false, 0);
    }
    Operand acc = imm(src_base + me * src_stride);
    for (uint32_t k = 1; k < P && !err; ++k) {
      err |= egr_recv_reduce(x, (me + P - k) % P, acc, imm(dst), mine, x.tag);
      acc = imm(dst);
    }
    return err;
  }
  // step: 2 * contributions folded + (address for the next one posted); mask bits 0-15: owners written to
  const uint32_t all = ((1u << P) - 1) & ~(1u << me);
  for (;;) {
    bool progressed = false;
    while ((mask & 0xFFFFu) != all) { // sender role: serve whichever owner has exposed its landing buffer
      uint32_t to = 0;
      uint64_t vaddr = 0;
      if (!rndzv_take_any_addr(x, (mask & 0xFFFFu) | (1u << me), x.tag, to, vaddr)) break;
      err = rndzv_write(x, to, src_base + to * src_stride, vaddr, count_of(to), x.tag);
      if (err) return err;
      mask |= 1u << to;
      progressed = true;
    }
    const uint32_t served = step >> 1;
    if (served < P - 1) { // owner role
      const uint32_t from = (me + P - 1 - served) % P;
      if (!(step & 1u)) {
        rndzv_post_addr(x, from, x.spare[0], mine * x.ubytes(), x.tag);
        step |= 1u;
        progressed = true;
      }
      const bool last = served + 1 == P - 1;
      if ((!last || (mask & 0xFFFFu) == all) && rndzv_take_done(x, from, x.tag)) {
        Move m;
        m.op0 = imm(served == 0 ? src_base + me * src_stride : x.spare[1 + (served & 1)]);
        m.op1 = imm(x.spare[0]);
        m.res = imm(last ? dst : x.spare[1 + ((served + 1) & 1)]);
        m.count = mine;
        m.func = x.fn();
        err = execute(x, m);
        if (err) return err;
        step = (served + 1) << 1;
        progressed = true;
      }
    }
    if ((step >> 1) == P - 1 && (mask & 0xFFFFu) == all) return 0;
    if (!progressed) return NOT_READY_ERROR;
  }
}

// --------------------------------------------------------------- allgather
uint32_t Engine::fw_allgather(EmuCall &c) {
  FW_DECODE(x);
  const uint32_t P = x.comm.size, me = x.comm.local_rank;
  const uint64_t slot_bytes = x.op_bytes(x.res_c(), x.count);
  const uint32_t next = (me + 1) % P, prev = (me + P - 1) % P;
  uint32_t err = 0;
  if (one_hop(x, 0)) {
    if (!(c.mask & 0x80000000u)) { // own block into place, once
      Move m;
      m.op0 = imm(x.a0);
      m.res = imm(x.a2 + me * slot_bytes);
      m.count = x.count;
      err = execute(x, m);
      if (err) return err;
      c.mask |= 0x80000000u;
    }
    uint32_t mask = c.mask & 0x7FFFFFFFu;
    err = onehop_gather(x, c.step, mask, x.a2 + me * slot_bytes, x.a2, slot_bytes, x.count);
    c.mask = mask | 0x80000000u;
    return err;
  }
  if (x.eager) {
    Move m; // own block into place
    m.op0 = x.op0_stream() ? stream_op() : imm(x.a0, x.op0_c());
    m.res = imm(x.a2 + me * slot_bytes, x.res_c());
    m.count = x.count;
    err |= execute(x, m);
    // ring: in step s forward the block that originated s hops upstream
    for (uint32_t s = 0; s + 1 < P && !err; ++s) {
      const uint32_t send_origin = (me + P - s) % P;
      const uint32_t recv_origin = (me + P - s - 1) % P;
      err |= egr_send(x, next, imm(x.a2 + send_origin * slot_bytes, x.res_c()), x.count, x.tag, false, 0);
      // blocking receive before the next relay: the relay reads what this writes
      if (!err) err |= egr_recv(x, prev, imm(x.a2 + recv_origin * slot_bytes, x.res_c()), x.count, x.tag, false, 0);
    }
    return err;
  }
  // ---- rendezvous ring: expose the slot the upstream neighbour will fill,
  // write my current block downstream, wait for the upstream block
  Steps st(c.step);
  st([&] {
    Move m;
    m.op0 = imm(x.a0);
    m.res = imm(x.a2 + me * slot_bytes);
    m.count = x.count;
    err |= execute(x, m);
    return true;
  });
  for (uint32_t s = 0; s + 1 < P; ++s) {
    const uint32_t send_origin = (me + P - s) % P;
    const uint32_t recv_origin = (me + P - s - 1) % P;
    st([&] { rndzv_post_addr(x, prev, x.a2 + recv_origin * slot_bytes, x.count * x.ubytes(), x.tag); return true; });
    if (!st([&] {
          uint64_t vaddr = 0;
          if (!rndzv_take_addr(x, next, x.tag, vaddr)) return false;
          err |= rndzv_write(x, next, x.a2 + send_origin * slot_bytes, vaddr, x.count, x.tag);
          return true;
        }))
      return NOT_READY_ERROR;
    if (!st([&] { return rndzv_take_done(x, prev, x.tag); })) return NOT_READY_ERROR;
  }
  return err;
}

// ------------------------------------------------------------------ reduce
uint32_t Engine::fw_reduce(EmuCall &c) {
  FW_DECODE(x);
  const uint32_t P = x.comm.size, me = x.comm.local_rank, root = x.root;
  Operand src = x.op0_stream() ? stream_op() : imm(x.a0, x.op0_c());
  Operand dst = x.res_stream() ? stream_op() : imm(x.a2, x.res_c());
  if (P == 1) {
    Move m;
    m.op0 = src;
    m.res = dst;
    m.strm = x.stream_id();
    m.count = x.count;
    return execute(x, m);
  }
  if (x.eager && one_hop(x, 0)) {
    // fan-in: everybody sends to the root, which folds the contributions in as they are matched
    if (me != root) return egr_send(x, root, src, x.count, x.tag, false, 0);
    uint32_t err = 0;
    Operand acc = src;
    for (uint32_t k = 1; k < P && !err; ++k) {
      err |= egr_recv_reduce(x, (root + P - k) % P, acc, dst, x.count, x.tag);
      acc = dst;
    }
    return err;
  }
  if (x.eager) {
    // chain root+1 -> root+2 -> ... -> root, each hop folds in its own data
    const uint32_t next = (me + 1) % P, prev = (me + P - 1) % P;
    if (me == (root + 1) % P) return egr_send(x, next, src, x.count, x.tag, false, 0);
    if (me == root) return egr_recv_reduce(x, prev, src, dst, x.count, x.tag);
    return egr_recv_reduce_send(x, prev, src, next, x.count, x.tag);
  }
  // ---- rendezvous, processed in chunks that fit the scratch buffers
  const uint32_t chunk_max = std::max(1u, x.spare_size / std::max(1u, x.ubytes()));
  const uint32_t flat_ranks = read_exch(exchmem::REDUCE_FLAT_TREE_MAX_RANKS);
  const uint32_t flat_count = read_exch(exchmem::REDUCE_FLAT_TREE_MAX_COUNT);
  const bool flat = P <= flat_ranks || x.count * x.ubytes() <= flat_count || read_exch(exchmem::ONE_HOP_SCHEDULES);
  Steps st(c.step);
  uint32_t err = 0;
  for (uint32_t off = 0; off < x.count; off += chunk_max) {
    const uint32_t n = std::min(chunk_max, x.count - off);
    const uint64_t boff = static_cast<uint64_t>(off) * x.ubytes();
    if (flat) {
      if (me != root) {
        if (!st([&] {
              uint64_t vaddr = 0;
              if (!rndzv_take_addr(x, root, x.tag, vaddr)) return false;
              err |= rndzv_write(x, root, x.a0 + boff, vaddr, n, x.tag);
              return true;
            }))
          return NOT_READY_ERROR;
        continue;
      }
      // root: land each peer's block in scratch 0, accumulate ping-pong in scratch 1/2
      uint64_t acc = x.a0 + boff;
      uint32_t served = 0;
      for (uint32_t r = 0; r < P; ++r) {
        if (r == root) continue;
        st([&] { rndzv_post_addr(x, r, x.spare[0], n * x.ubytes(), x.tag); return true; });
        if (!st([&] { return rndzv_take_done(x, r, x.tag); })) return NOT_READY_ERROR;
        ++served;
        const bool last = served == P - 1;
        const uint64_t out = last ? x.a2 + boff : x.spare[1 + (served & 1)];
        st([&] {
          Move m;
          m.op0 = imm(acc);
          m.op1 = imm(x.spare[0]);
          m.res = imm(out);
          m.count = n;
          m.func = x.fn();
          err |= execute(x, m);
          return true;
        });
        acc = out;
      }
    } else {
      // binomial tree towards the root over normalised ranks
      const uint32_t v = (me + P - root) % P;
      uint64_t acc = x.a0 + boff;
      uint32_t folds = 0;
      bool sent = false;
      for (uint32_t k = 1; k < P && !sent; k <<= 1) {
        if (v & k) {
          const uint32_t parent = ((v - k) + root) % P;
          if (!st([&] {
                uint64_t vaddr = 0;
                if (!rndzv_take_addr(x, parent, x.tag, vaddr)) return false;
                err |= rndzv_write(x, parent, acc, vaddr, n, x.tag);
                return true;
              }))
            return NOT_READY_ERROR;
          sent = true;
        } else if (v + k < P) {
          const uint32_t child = (v + k + root) % P;
          st([&] { rndzv_post_addr(x, child, x.spare[0], n * x.ubytes(), x.tag); return true; });
          if (!st([&] { return rndzv_take_done(x, child, x.tag); })) return NOT_READY_ERROR;
          ++folds;
          // the root's last fold lands in the destination
          bool last = v == 0;
          for (uint32_t kk = k << 1; kk < P && last; kk <<= 1)
            if (v + kk < P) last = false;
          const uint64_t out = last ? x.a2 + boff : x.spare[1 + (folds & 1)];
          st([&] {
            Move m;
            m.op0 = imm(acc);
            m.op1 = imm(x.spare[0]);
            m.res = imm(out);
            m.count = n;
            m.func = x.fn();
            err |= execute(x, m);
            return true;
          });
          acc = out;
        }
      }
    }
  }
  return err;
}

// ---------------------------------------------------------- reduce_scatter
uint32_t Engine::fw_reduce_scatter(EmuCall &c) {
  FW_DECODE(x);
  const uint32_t P = x.comm.size, me = x.comm.local_rank;
  const uint64_t blk = x.op_bytes(x.op0_c(), x.count);
  if (P == 1) {
    Move m;
    m.op0 = imm(x.a0, x.op0_c());
    m.res = imm(x.a2, x.res_c());
    m.count = x.count;
    return execute(x, m);
  }
  if (one_hop(x, blk)) return onehop_reduce(x, c.step, c.mask, x.a0, blk, x.a2, x.count);
  if (!x.eager) {
    // rendezvous: reduce count*P to rank 0 (in scratch-sized chunks), then scatter.
    // Both phases are resumable sub-calls sharing this call's step counter.
    // phase boundary kept in bit 31 of the mask
    if (!(c.mask & 0x80000000u)) {
      EmuCall sub = c;
      sub.desc.scenario = static_cast<uint32_t>(operation::reduce);
      sub.desc.count = x.count * P;
      sub.desc.root_src_dst = 0;
      sub.desc.set_addr(2, x.a0); // rank 0 reduces in place into its send buffer
      uint32_t rc = fw_reduce(sub);
      c.step = sub.step;
      c.mask = sub.mask;
      if (rc) return rc;
      c.step = 0;
      c.mask = 0x80000000u;
    }
    EmuCall sub = c;
    sub.desc.scenario = static_cast<uint32_t>(operation::scatter);
    sub.desc.root_src_dst = 0;
    sub.mask = c.mask & 0x7FFFFFFFu;
    uint32_t rc = fw_scatter(sub);
    c.step = sub.step;
    c.mask = sub.mask | 0x80000000u;
    return rc;
  }
  // eager ring: step s sends block (me-1-s), receives+reduces block (me-2-s);
  // after P-1 steps block `me` is complete here
  const uint32_t next = (me + 1) % P, prev = (me + P - 1) % P;
  uint32_t err = egr_send(x, next, imm(x.a0 + ((me + P - 1) % P) * blk, x.op0_c()), x.count, x.tag, false, 0);
  for (uint32_t s = 0; s + 1 < P && !err; ++s) {
    const uint32_t b = (me + 2 * P - 2 - s) % P;
    Operand local = imm(x.a0 + b * blk, x.op0_c());
    if (s + 2 < P) err |= egr_recv_reduce_send(x, prev, local, next, x.count, x.tag);
    else err |= egr_recv_reduce(x, prev, local, x.res_stream() ? stream_op() : imm(x.a2, x.res_c()), x.count, x.tag);
  }
  return err;
}

// --------------------------------------------------------------- allreduce
uint32_t Engine::fw_allreduce(EmuCall &c) {
  FW_DECODE(x);
  const uint32_t P = x.comm.size, me = x.comm.local_rank;
  if (P == 1) {
    Move m;
    m.op0 = imm(x.a0, x.op0_c());
    m.res = imm(x.a2, x.res_c());
    m.count = x.count;
    return execute(x, m);
  }
  {
    // one hop (everybody sends everything) or two (reduce-scatter + all-gather): what the CUDA backend's planner decides for
    // this call — flag-in-data / slot-ring class: WF_ONESHOT rule; rendezvous class: one-shot while bytes * P <= 2 MiB
    const uint64_t bytes = static_cast<uint64_t>(x.count) * x.ubytes();
    uint32_t ex[16] = {};
    ex[exchmem::MAX_EAGER_SIZE / 4] = x.max_eager;
    ex[exchmem::EAGER_RX_BUF_SIZE / 4] = x.rxbuf_size;
    cuda::PlanCfg pc{};
    pc.max_ctas = 128;
    pc.nvls_min_ranks = 3;
    pc.has_mc = 1;
    pc.heap_world = P;
    pc.oneshot_max_bytes = 2u << 20;
    pc.nvls_ops = cuda::NVLS_OPS_DEFAULT;
    pc.nvls_ctas = 32;
    pc.ll_bytes = 2u << 20;
    pc.ll_max_bytes = 2u << 20;
    pc.ll_oneshot_max = 32u << 10;
    cuda::WorkItem wi{};
    wi.desc = c.desc;
    wi.comm_size = P;
    wi.udtype = static_cast<uint32_t>(x.ar.u);
    wi.cdtype = static_cast<uint32_t>(x.ar.c);
    cuda::plan_call(ex, pc, wi);
    const bool planner_oneshot = wi.algo == cuda::ALGO_P2P_ONESHOT || wi.algo == cuda::ALGO_EAGER ||
                                 ((wi.algo == cuda::ALGO_LL || wi.algo == cuda::ALGO_STAGED) && (wi.flags & cuda::WF_ONESHOT));
    // two hops with a count that does not split: the last rank's shard absorbs the remainder (as on the GPU)
    const uint32_t shard = x.count / P, extra = x.count % P;
    const bool oneshot = planner_oneshot || shard == 0;
    if (one_hop(x, oneshot ? bytes : static_cast<uint64_t>(shard + extra) * x.ubytes())) {
      if (c.step == 0 && c.mask == 0) (oneshot ? g_allreduce_one_shot : g_allreduce_two_shot).fetch_add(1);
      if (oneshot) return onehop_reduce(x, c.step, c.mask, x.a0, 0, x.a2, x.count);
      // reduce-scatter into my shard of the result, then all-gather the shards (phase in bit 31 of the mask)
      const uint64_t sb = static_cast<uint64_t>(shard) * x.ubytes();
      if (!(c.mask & 0x80000000u)) {
        uint32_t rc = onehop_reduce(x, c.step, c.mask, x.a0, sb, x.a2 + me * sb, shard, extra);
        if (rc) return rc;
        c.step = 0;
        c.mask = 0x80000000u;
      }
      uint32_t mask = c.mask & 0x7FFFFFFFu;
      uint32_t rc = onehop_gather(x, c.step, mask, x.a2 + me * sb, x.a2, sb, shard, extra);
      c.mask = mask | 0x80000000u;
      return rc;
    }
  }
  if (!x.eager) {
    // rendezvous: reduce to rank 0, then broadcast from it
    if (!(c.mask & 0x80000000u)) {
      EmuCall sub = c;
      sub.desc.scenario = static_cast<uint32_t>(operation::reduce);
      sub.desc.root_src_dst = 0;
      sub.mask = c.mask;
      uint32_t rc = fw_reduce(sub);
      c.step = sub.step;
      c.mask = sub.mask;
      if (rc) return rc;
      c.step = 0;
      c.mask = 0x80000000u;
    }
    EmuCall sub = c;
    sub.desc.scenario = static_cast<uint32_t>(operation::bcast);
    sub.desc.root_src_dst = 0;
    sub.desc.set_addr(0, x.a2);
    sub.mask = c.mask & 0x7FFFFFFFu;
    uint32_t rc = fw_bcast(sub);
    c.step = sub.step;
    c.mask = sub.mask | 0x80000000u;
    return rc;
  }
  // eager: ring reduce-scatter followed by ring allgather on P blocks of
  // ceil(count/P) elements; the last block may be shorter (or empty)
  const uint32_t next = (me + 1) % P, prev = (me + P - 1) % P;
  const uint32_t bulk = (x.count + P - 1) / P;
  auto blk_count = [&](uint32_t b) -> uint32_t {
    const uint64_t start = static_cast<uint64_t>(b) * bulk;
    if (start >= x.count) return 0;
    return static_cast<uint32_t>(std::min<uint64_t>(bulk, x.count - start));
  };
  const uint64_t src_eb = dtype_bytes(x.op0_c() ? x.ar.c : x.ar.u), dst_eb = dtype_bytes(x.res_c() ? x.ar.c : x.ar.u);
  if ((is_fp8(x.ar.c) && (x.op0_c() || x.res_c()))) return COMPRESSION_ERROR; // block-scaled buffers cannot be sliced
  auto src_at = [&](uint32_t b) { return imm(x.a0 + static_cast<uint64_t>(b) * bulk * src_eb, x.op0_c()); };
  auto dst_at = [&](uint32_t b) { return imm(x.a2 + static_cast<uint64_t>(b) * bulk * dst_eb, x.res_c()); };
  uint32_t err = 0;
  {
    const uint32_t b = (me + P - 1) % P;
    if (blk_count(b)) err |= egr_send(x, next, src_at(b), blk_count(b), x.tag, false, 0);
  }
  for (uint32_t s = 0; s + 1 < P && !err; ++s) {
    const uint32_t b = (me + 2 * P - 2 - s) % P;
    if (!blk_count(b)) continue;
    if (s + 2 < P) err |= egr_recv_reduce_send(x, prev, src_at(b), next, blk_count(b), x.tag);
    else err |= egr_recv_reduce(x, prev, src_at(b), dst_at(b), blk_count(b), x.tag); // b == me
  }
  // allgather phase: block `me` is final in dst; circulate
  for (uint32_t s = 0; s + 1 < P && !err; ++s) {
    const uint32_t sb = (me + P - s) % P, rb = (me + P - s - 1) % P;
    if (blk_count(sb)) err |= egr_send(x, next, dst_at(sb), blk_count(sb), x.tag, false, 0);
    if (!err && blk_count(rb)) err |= egr_recv(x, prev, dst_at(rb), blk_count(rb), x.tag, false, 0);
  }
  return err;
}

// ----------------------------------------------------------------- barrier
uint32_t Engine::fw_barrier(EmuCall &c) {
  FW_DECODE(x);
  const uint32_t P = x.comm.size, me = x.comm.local_rank;
  // calls parked before the barrier must drain first (younger ones parked behind it do not hold it up)
  if (older_parked_ != 0 && c.step == 0 && c.mask == 0) return NOT_READY_ERROR;
  if (P == 1) return 0;
  auto notify = [&](uint32_t to) {
    Packet p;
    p.hdr.msg_type = static_cast<uint32_t>(MsgType::RNDZVS_WR_DONE);
    p.hdr.src = static_cast<uint32_t>(rank_);
    p.hdr.dst = x.comm.session[to];
    p.hdr.tag = BARRIER_TAG;
    p.hdr.strm = 1; // marks a barrier token so data completions never match it
    p.hdr.comm_sig = x.comm.sig;
    p.hdr.seqn = note_kind(x);
    fabric_->send(std::move(p));
  };
  Steps st(c.step);
  if (me == 0) {
    const uint32_t all = ((1u << P) - 1) & ~1u;
    while ((c.mask & all) != all) { // gather arrivals
      uint32_t from = 0;
      if (!rndzv_take_any_done(x, c.mask | 1u, BARRIER_TAG, from)) return NOT_READY_ERROR;
      c.mask |= 1u << from;
    }
    for (uint32_t r = 1; r < P; ++r) notify(r); // release
    return 0;
  }
  st([&] { notify(0); return true; });
  if (!st([&] { return rndzv_take_done(x, 0, BARRIER_TAG); })) return NOT_READY_ERROR;
  return 0;
}

// ---------------------------------------------------------------- alltoall
uint32_t Engine::fw_alltoall(EmuCall &c) {
  FW_DECODE(x);
  const uint32_t P = x.comm.size, me = x.comm.local_rank;
  const uint64_t sblk = x.op_bytes(x.op0_c(), x.count), rblk = x.op_bytes(x.res_c(), x.count);
  uint32_t err = 0;
  if (x.eager) {
    // beyond the reference (which only implements the rendezvous form): pairwise
    // eager exchange, sends first (they are buffered at the receivers)
    Move m;
    m.op0 = imm(x.a0 + me * sblk, x.op0_c());
    m.res = imm(x.a2 + me * rblk, x.res_c());
    m.count = x.count;
    err |= execute(x, m);
    for (uint32_t k = 1; k < P && !err; ++k) {
      const uint32_t to = (me + k) % P;
      err |= egr_send(x, to, imm(x.a0 + to * sblk, x.op0_c()), x.count, x.tag, false, 0);
    }
    for (uint32_t k = 1; k < P && !err; ++k) {
      const uint32_t from = (me + P - k) % P;
      err |= egr_recv(x, from, imm(x.a2 + from * rblk, x.res_c()), x.count, x.tag, false, 0);
    }
    return err;
  }
  Steps st(c.step);
  st([&] {
    Move m;
    m.op0 = imm(x.a0 + me * sblk);
    m.res = imm(x.a2 + me * rblk);
    m.count = x.count;
    err |= execute(x, m);
    for (uint32_t r = 0; r < P; ++r)
      if (r != me) rndzv_post_addr(x, r, x.a2 + r * rblk, x.count * x.ubytes(), x.tag);
    return true;
  });
  if (err) return err;
  // low 16 bits of mask: peers written to; high 16 bits: completions collected
  const uint32_t all = ((1u << P) - 1) & ~(1u << me);
  while ((c.mask & 0xFFFFu) != all) {
    uint32_t from = 0;
    uint64_t vaddr = 0;
    if (!rndzv_take_any_addr(x, (c.mask & 0xFFFFu) | (1u << me), x.tag, from, vaddr)) return NOT_READY_ERROR;
    err = rndzv_write(x, from, x.a0 + from * sblk, vaddr, x.count, x.tag);
    if (err) return err;
    c.mask |= 1u << from;
  }
  while (((c.mask >> 16) & 0xFFFFu) != all) {
    uint32_t from = 0;
    if (!rndzv_take_any_done(x, ((c.mask >> 16) & 0xFFFFu) | (1u << me), x.tag, from)) return NOT_READY_ERROR;
    c.mask |= 1u << (16 + from);
  }
  return 0;
}

// --------------------------------------------------------------- alltoallv
// Beyond the reference.  Counts in memory at a1 (int64: P send counts, then P receive counts, in elements);
// capacities in `count` (receive) and `root_src_dst` (send).  One exchange before any data moves: every rank
// announces its receive buffer to every peer together with its whole count vector and its capacities, so each rank
// checks the same matrix and reaches the same verdict (all-or-nothing: an invalid call writes nothing anywhere).
// Then the blocks go straight into the receivers' buffers as one-sided writes, each followed by its completion
// note.  The same schedule serves the eager and rendezvous sizes and the one-hop mode.
uint32_t Engine::fw_alltoallv(EmuCall &c) {
  FW_DECODE(x);
  const uint32_t P = x.comm.size, me = x.comm.local_rank;
  const uint64_t es = x.ubytes();
  const size_t row_words = 2 * static_cast<size_t>(P) + 2; // counts, send capacity, receive capacity
  auto my_row = [&] {
    std::vector<int64_t> v(row_words, 0);
    uint32_t e = 0;
    const uint8_t *p = mem_ptr(x.a1, 2 * P * sizeof(int64_t), e);
    if (p) std::memcpy(v.data(), p, 2 * P * sizeof(int64_t));
    v[2 * P] = p ? static_cast<int64_t>(x.root) : -1; // unreadable counts: a negative capacity rejects the call
    v[2 * P + 1] = static_cast<int64_t>(x.count);
    return v;
  };
  Steps st(c.step);
  st([&] {
    const std::vector<int64_t> v = my_row();
    for (uint32_t r = 0; r < P; ++r) {
      if (r == me) continue;
      Packet p;
      p.hdr.msg_type = static_cast<uint32_t>(MsgType::RNDZVS_INIT);
      p.hdr.src = static_cast<uint32_t>(rank_);
      p.hdr.dst = x.comm.session[r];
      p.hdr.tag = x.tag;
      p.hdr.vaddr = x.a2;
      p.hdr.comm_sig = x.comm.sig;
      p.hdr.host = x.a2 >= HOST_BASE;
      p.hdr.seqn = note_kind(x);
      p.payload.resize(row_words * sizeof(int64_t));
      std::memcpy(p.payload.data(), v.data(), p.payload.size());
      fabric_->send(std::move(p));
    }
    return true;
  });
  uint32_t err = 0;
  if (!st([&] {
        // every peer's announcement, or none of them (a parked call keeps nothing but its step)
        std::vector<std::vector<int64_t>> rows(P);
        std::vector<uint64_t> dst_base(P, x.a2);
        {
          std::lock_guard<std::mutex> g(q_m_);
          std::vector<std::list<AddrNote>::iterator> found(P, addr_notes_.end());
          uint32_t n = 0;
          for (auto it = addr_notes_.begin(); it != addr_notes_.end(); ++it) {
            if (it->comm_sig != x.comm.sig || it->kind != note_kind(x)) continue;
            for (uint32_t r = 0; r < P; ++r)
              if (r != me && found[r] == addr_notes_.end() && x.comm.session[r] == it->src) {
                found[r] = it;
                ++n;
                break;
              }
          }
          if (n + 1 != P) return false;
          for (uint32_t r = 0; r < P; ++r) {
            if (r == me) continue;
            rows[r].assign(row_words, -1);
            if (found[r]->payload.size() == row_words * sizeof(int64_t))
              std::memcpy(rows[r].data(), found[r]->payload.data(), found[r]->payload.size());
            dst_base[r] = found[r]->vaddr;
            addr_notes_.erase(found[r]);
          }
        }
        rows[me] = my_row();
        bool ok = true;
        for (uint32_t p = 0; p < P && ok; ++p) { // each rank's own checks ...
          const std::vector<int64_t> &v = rows[p];
          int64_t s = 0, r = 0;
          for (uint32_t q = 0; q < P && ok; ++q) {
            ok = v[q] >= 0 && v[P + q] >= 0 && v[q] <= v[2 * P] && v[P + q] <= v[2 * P + 1];
            s += ok ? v[q] : 0;
            r += ok ? v[P + q] : 0;
          }
          ok = ok && s <= v[2 * P] && r <= v[2 * P + 1];
        }
        for (uint32_t p = 0; p < P && ok; ++p) // ... and every send count against its receiver's count
          for (uint32_t q = 0; q < P && ok; ++q) ok = rows[p][q] == rows[q][P + p];
        if (!ok) {
          err = DMA_SIZE_ERROR;
          return true;
        }
        uint64_t src_off = 0;
        for (uint32_t q = 0; q < P; ++q) { // (after a failed write too: every peer gets its completion note)
          uint64_t dst_off = 0; // after the blocks of q's lower senders
          for (uint32_t p = 0; p < me; ++p) dst_off += static_cast<uint64_t>(rows[q][P + p]);
          const uint32_t n = static_cast<uint32_t>(rows[me][q]);
          if (q == me) {
            if (n) {
              Move m;
              m.op0 = imm(x.a0 + src_off * es);
              m.res = imm(x.a2 + dst_off * es);
              m.count = n;
              err |= execute(x, m);
            }
          } else {
            err |= rndzv_write(x, q, x.a0 + src_off * es, dst_base[q] + dst_off * es, n, x.tag);
          }
          src_off += n;
        }
        return true;
      }))
    return NOT_READY_ERROR;
  if (err) return err;
  // only valid calls get here (an invalid one returned above on every rank): collect the completion notes
  const uint32_t all = ((1u << P) - 1) & ~(1u << me);
  while ((c.mask & all) != all) {
    uint32_t from = 0;
    if (!rndzv_take_any_done(x, c.mask | (1u << me), x.tag, from)) return NOT_READY_ERROR;
    c.mask |= 1u << from;
  }
  return 0;
}

} // namespace emu
} // namespace accl
