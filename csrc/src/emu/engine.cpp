#include "accl/emu/engine.hpp"

#include <sys/mman.h>

#include <algorithm>
#include <cstring>
#include <sstream>

#include "accl/common.hpp"
#include "engine_ctx.hpp"

namespace accl {
namespace emu {

static uint64_t now_ns() {
  return static_cast<uint64_t>(
      std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count());
}

// ------------------------------------------------------------------- Arena
Arena::Arena(uint64_t base, size_t capacity) : base_(base), cap_(capacity), mem_(nullptr), alloc_(base, capacity) {
  void *p = ::mmap(nullptr, capacity, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
  if (p == MAP_FAILED) throw std::bad_alloc();
  mem_ = static_cast<uint8_t *>(p);
}
Arena::~Arena() {
  if (mem_) ::munmap(mem_, cap_);
}

// ---------------------------------------------------------------- ByteFifo
void ByteFifo::push(const void *data, size_t n) {
  const uint8_t *b = static_cast<const uint8_t *>(data);
  {
    std::lock_guard<std::mutex> g(m_);
    q_.insert(q_.end(), b, b + n);
  }
  cv_.notify_all();
}
bool ByteFifo::pop(void *out, size_t n, std::chrono::microseconds timeout) {
  std::unique_lock<std::mutex> lk(m_);
  if (!cv_.wait_for(lk, timeout, [&] { return q_.size() >= n; })) return false;
  uint8_t *o = static_cast<uint8_t *>(out);
  std::copy(q_.begin(), q_.begin() + static_cast<std::ptrdiff_t>(n), o);
  q_.erase(q_.begin(), q_.begin() + static_cast<std::ptrdiff_t>(n));
  return true;
}
size_t ByteFifo::size() {
  std::lock_guard<std::mutex> g(m_);
  return q_.size();
}

// ------------------------------------------------------------------ Engine
Engine::Engine(int global_rank, int world, std::shared_ptr<Fabric> fabric, size_t dev_mem_bytes, size_t host_mem_bytes)
    : rank_(global_rank), world_(world), fabric_(std::move(fabric)), dev_(DEV_BASE, dev_mem_bytes),
      host_(HOST_BASE, host_mem_bytes) {
  exch_[exchmem::HWID / 4] = CAP_DMA | CAP_ARITH | CAP_COMPRESSION | CAP_STREAMS | CAP_RENDEZVOUS | CAP_FP8;
  fabric_->attach(rank_, [this](Packet &&p) { on_packet(std::move(p)); });
  control_ = std::thread([this] { control_loop(); });
  ingress_ = std::thread([this] { ingress_loop(); });
}

Engine::~Engine() {
  stop_ = true;
  q_cv_.notify_all();
  in_cv_.notify_all();
  rx_cv_.notify_all();
  if (control_.joinable()) control_.join();
  if (ingress_.joinable()) ingress_.join();
  fabric_->detach(rank_);
}

uint32_t Engine::read_exch(uint32_t off) {
  if (off >= exchmem::SIZE_BYTES || (off & 3)) throw std::out_of_range("exchange memory read out of range");
  std::lock_guard<std::mutex> g(exch_m_);
  return exch_[off / 4];
}
void Engine::write_exch(uint32_t off, uint32_t v) {
  if (off >= exchmem::SIZE_BYTES || (off & 3)) throw std::out_of_range("exchange memory write out of range");
  std::lock_guard<std::mutex> g(exch_m_);
  exch_[off / 4] = v;
}

uint64_t Engine::mem_alloc(size_t bytes, bool host) { return host ? host_.alloc(bytes) : dev_.alloc(bytes); }
void Engine::mem_free(uint64_t addr) {
  if (addr >= HOST_BASE) host_.free(addr);
  else dev_.free(addr);
}
uint8_t *Engine::mem_ptr(uint64_t addr, size_t len, uint32_t &err) {
  if (dev_.contains(addr, len)) return dev_.ptr(addr);
  if (host_.contains(addr, len)) return host_.ptr(addr);
  err |= DMA_DECODE_ERROR;
  return nullptr;
}
void Engine::mem_write(uint64_t addr, const void *src, size_t len) {
  uint32_t e = 0;
  uint8_t *p = mem_ptr(addr, len, e);
  if (!p) throw std::out_of_range("emulator mem_write outside simulated memory");
  std::memcpy(p, src, len);
}
void Engine::mem_read(uint64_t addr, void *dst, size_t len) {
  uint32_t e = 0;
  uint8_t *p = mem_ptr(addr, len, e);
  if (!p) throw std::out_of_range("emulator mem_read outside simulated memory");
  std::memcpy(dst, p, len);
}

void Engine::submit(EmuCall &&c) {
  c.t0_ns = 0;
  {
    std::lock_guard<std::mutex> g(q_m_);
    new_calls_.push_back(std::move(c));
  }
  q_cv_.notify_all();
}

void Engine::kernel_push(const void *data, size_t bytes) { krnl_to_cclo_.push(data, bytes); }
bool Engine::kernel_pull(uint32_t strm, void *out, size_t bytes, int timeout_ms) {
  return out_stream(strm).pop(out, bytes, std::chrono::milliseconds(timeout_ms));
}
ByteFifo &Engine::out_stream(uint32_t id) {
  std::lock_guard<std::mutex> g(strm_m_);
  auto &p = cclo_to_krnl_[id];
  if (!p) p.reset(new ByteFifo());
  return *p;
}

uint32_t Engine::timeout_us() {
  uint32_t t = read_exch(exchmem::TIMEOUT);
  return t ? t : 1000000u;
}

// --------------------------------------------------------------- control
void Engine::control_loop() {
  // Parked calls are kept in issue order and retried oldest first: two calls that wait for the same kind of
  // event (e.g. several rendezvous sends to one peer with one tag, all waiting for an address note) must be
  // served in the order they were issued — the non-overtaking rule of point-to-point messages.  A pass walks
  // the list once; a fresh call is only admitted after a pass (or an empty list) and parks behind its elders.
  uint64_t seen_events = 0;
  size_t cursor = 0;       // next parked call to try in this pass
  bool progressed = false; // did this pass retire anything?
  bool from_retry = false; // where the call being dispatched came from
  while (!stop_) {
    EmuCall c;
    bool have = false;
    {
      std::unique_lock<std::mutex> lk(q_m_);
      if (cursor >= retry_calls_.size() && new_calls_.empty()) {
        // a full pass over the parked calls and nothing new
        if (!progressed || retry_calls_.empty()) {
          // nothing runnable: sleep until a call, a mailbox event or a tick
          q_cv_.wait_for(lk, std::chrono::milliseconds(retry_calls_.empty() ? 50 : 1), [&] {
            return stop_.load() || !new_calls_.empty() || (!retry_calls_.empty() && mailbox_events_ != seen_events);
          });
        }
        cursor = 0;
        progressed = false;
      }
      if (stop_) break;
      if (mailbox_events_ != seen_events) {
        // something arrived: the oldest parked call gets the first look at it
        seen_events = mailbox_events_;
        cursor = 0;
      }
      if (cursor < retry_calls_.size()) {
        c = std::move(retry_calls_[cursor]);
        retry_calls_.erase(retry_calls_.begin() + static_cast<std::ptrdiff_t>(cursor));
        older_parked_ = cursor;
        from_retry = true;
        have = true;
      } else if (!new_calls_.empty()) {
        c = std::move(new_calls_.front());
        new_calls_.pop_front();
        older_parked_ = retry_calls_.size();
        from_retry = false;
        have = true;
        cursor = 0; // after a fresh call, start the next pass with the oldest parked call
        progressed = false;
      }
    }
    if (!have) continue;
    if (c.t0_ns == 0) {
      c.t0_ns = now_ns();
      if (c.req) c.req->set_status(operationStatus::EXECUTING);
    }
    uint32_t rc;
    try {
      rc = dispatch(c);
    } catch (const std::exception &e) {
      ACCL_ERROR_LOG("emulator rank " << rank_ << ": " << e.what());
      rc = DMA_INTERNAL_ERROR;
    }
    if (rc == NOT_READY_ERROR) {
      // park it; give up after a generous deadline so a broken test fails instead of hanging
      const uint64_t waited_us = (now_ns() - c.t0_ns) / 1000;
      if (waited_us > std::max<uint64_t>(60ull * 1000000ull, 2ull * timeout_us())) {
        rc = RECEIVE_TIMEOUT_ERROR;
        purge_notes_of(c); // what it posted to peers / what peers addressed to it must not be matched by a later call
      } else {
        std::lock_guard<std::mutex> g(q_m_);
        if (from_retry) {
          // back to its place in the issue order; the pass moves on to the next one
          const size_t at = std::min(older_parked_, retry_calls_.size());
          retry_calls_.insert(retry_calls_.begin() + static_cast<std::ptrdiff_t>(at), std::move(c));
          cursor = at + 1;
        } else {
          retry_calls_.push_back(std::move(c)); // the youngest
        }
        continue;
      }
    }
    progressed = true;
    if (from_retry) cursor = older_parked_; // the list closed up behind the retired call
    const uint64_t dur = now_ns() - c.t0_ns;
    write_exch(exchmem::RETCODE, rc);
    write_exch(exchmem::PERFCNT_LO, static_cast<uint32_t>(dur));
    write_exch(exchmem::PERFCNT_HI, static_cast<uint32_t>(dur >> 32));
    if (c.req) c.req->complete(rc, dur); // first: completion hooks may read the request's outcome
    if (c.on_done) c.on_done(rc);
  }
  // fail whatever is still queued so waiters wake up
  std::lock_guard<std::mutex> g(q_m_);
  for (auto *q : {&new_calls_, &retry_calls_})
    for (auto &c : *q) {
      if (c.req) c.req->complete(NOT_READY_ERROR, 0);
      if (c.on_done) c.on_done(NOT_READY_ERROR);
    }
}

void Engine::soft_reset() {
  std::deque<EmuCall> parked;
  {
    std::lock_guard<std::mutex> g(q_m_);
    parked.swap(retry_calls_);
    addr_notes_.clear();
    done_notes_.clear();
  }
  for (auto &c : parked) {
    if (c.req) c.req->complete(NOT_READY_ERROR, 0);
    if (c.on_done) c.on_done(NOT_READY_ERROR);
  }
  {
    std::lock_guard<std::mutex> g(rx_m_);
    rx_overflow_.clear();
    std::lock_guard<std::mutex> e(exch_m_);
    const uint32_t n = exch_[exchmem::EAGER_RX_BUF_COUNT / 4];
    for (uint32_t i = 0; i < n && i < exchmem::MAX_RXBUFS; ++i)
      exch_[exchmem::rxbuf_offset(i, exchmem::RX_STATUS) / 4] = exchmem::RX_IDLE;
    const uint32_t nc = exch_[exchmem::NUM_COMMUNICATORS / 4];
    for (uint32_t c = 0; c < nc && c < static_cast<uint32_t>(ACCL_MAX_COMMUNICATORS); ++c)
      for (uint32_t r = 0; r < static_cast<uint32_t>(ACCL_MAX_RANKS); ++r) {
        exch_[exchmem::comm_rank_offset(c, r, exchmem::CR_INBOUND_SEQ) / 4] = 0;
        exch_[exchmem::comm_rank_offset(c, r, exchmem::CR_OUTBOUND_SEQ) / 4] = 0;
      }
    exch_[exchmem::CFGRDY / 4] = 0;
    exch_[exchmem::PKT_ENABLED / 4] = 0;
  }
  for (int s = 0; s < 3; ++s) prev_addr_[s] = prev_bytes_[s] = 0;
}

// --------------------------------------------------------------- ingress
void Engine::on_packet(Packet &&p) {
  {
    std::lock_guard<std::mutex> g(in_m_);
    inbox_.push_back(std::move(p));
  }
  in_cv_.notify_one();
}

// place arrived eager messages into posted RX buffers (rx_m_ held)
void Engine::rx_try_fill_locked() {
  while (!rx_overflow_.empty()) {
    Packet &p = rx_overflow_.front();
    int slot = -1;
    uint32_t maxlen = 0;
    uint64_t addr = 0;
    {
      std::lock_guard<std::mutex> e(exch_m_);
      const uint32_t n = exch_[exchmem::EAGER_RX_BUF_COUNT / 4];
      for (uint32_t i = 0; i < n; ++i)
        if (exch_[exchmem::rxbuf_offset(i, exchmem::RX_STATUS) / 4] == exchmem::RX_ENQUEUED) {
          slot = static_cast<int>(i);
          maxlen = exch_[exchmem::rxbuf_offset(i, exchmem::RX_MAX_LEN) / 4];
          addr = (static_cast<uint64_t>(exch_[exchmem::rxbuf_offset(i, exchmem::RX_ADDR_HI) / 4]) << 32) |
                 exch_[exchmem::rxbuf_offset(i, exchmem::RX_ADDR_LO) / 4];
          break;
        }
    }
    if (slot < 0) return; // every buffer busy: message waits (back-pressure)
    uint32_t status = exchmem::RX_RESERVED;
    uint32_t e = 0;
    uint8_t *dst = mem_ptr(addr, p.payload.size(), e);
    if (p.payload.size() > maxlen || !dst) status = exchmem::RX_ERROR;
    else if (!p.payload.empty()) std::memcpy(dst, p.payload.data(), p.payload.size());
    if (rx_meta_.size() <= static_cast<size_t>(slot)) rx_meta_.resize(static_cast<size_t>(slot) + 1);
    rx_meta_[static_cast<size_t>(slot)] = RxMeta{p.hdr.comm_sig, p.hdr.elems, p.hdr.dtypes};
    {
      std::lock_guard<std::mutex> g(exch_m_);
      const uint32_t s = static_cast<uint32_t>(slot);
      exch_[exchmem::rxbuf_offset(s, exchmem::RX_TAG) / 4] = p.hdr.tag;
      exch_[exchmem::rxbuf_offset(s, exchmem::RX_LEN) / 4] = static_cast<uint32_t>(p.payload.size());
      exch_[exchmem::rxbuf_offset(s, exchmem::RX_SRC) / 4] = p.hdr.src;
      exch_[exchmem::rxbuf_offset(s, exchmem::RX_SEQ) / 4] = p.hdr.seqn;
      exch_[exchmem::rxbuf_offset(s, exchmem::RX_STATUS) / 4] = status;
    }
    rx_overflow_.pop_front();
    rx_cv_.notify_all();
  }
}

void Engine::ingress_loop() {
  while (!stop_) {
    Packet p;
    {
      std::unique_lock<std::mutex> lk(in_m_);
      in_cv_.wait_for(lk, std::chrono::milliseconds(50), [&] { return stop_.load() || !inbox_.empty(); });
      if (stop_) break;
      if (inbox_.empty()) continue;
      p = std::move(inbox_.front());
      inbox_.pop_front();
    }
    switch (static_cast<MsgType>(p.hdr.msg_type)) {
    case MsgType::EGR_MSG:
      if (p.hdr.strm != 0) {
        // streamed eager message: bypasses the RX buffers, goes to the user stream
        if (loopback_) krnl_to_cclo_.push(p.payload.data(), p.payload.size());
        else out_stream(p.hdr.strm).push(p.payload.data(), p.payload.size());
      } else {
        std::lock_guard<std::mutex> g(rx_m_);
        rx_overflow_.push_back(std::move(p));
        rx_try_fill_locked();
        if (!rx_overflow_.empty()) rx_cv_.notify_all(); // pool exhausted: a seeker may want to swap this one in
      }
      break;
    case MsgType::RNDZVS_MSG: {
      uint32_t e = 0;
      uint8_t *dst = mem_ptr(p.hdr.vaddr, p.payload.size(), e);
      if (dst && !p.payload.empty()) std::memcpy(dst, p.payload.data(), p.payload.size());
      else if (!dst) ACCL_ERROR_LOG("emulator rank " << rank_ << ": rendezvous write outside memory");
      break;
    }
    case MsgType::RNDZVS_INIT: {
      std::lock_guard<std::mutex> g(q_m_);
      addr_notes_.push_back(AddrNote{p.hdr.comm_sig, p.hdr.src, p.hdr.tag, p.hdr.count, p.hdr.vaddr, p.hdr.seqn, std::move(p.payload)});
      ++mailbox_events_;
      q_cv_.notify_all();
      break;
    }
    case MsgType::RNDZVS_WR_DONE: {
      std::lock_guard<std::mutex> g(q_m_);
      done_notes_.push_back(DoneNote{p.hdr.comm_sig, p.hdr.src, p.hdr.tag, p.hdr.strm != 0, p.hdr.seqn});
      ++mailbox_events_;
      q_cv_.notify_all();
      break;
    }
    case MsgType::RNDZVS_CANCEL: {
      // the receive that announced this buffer gave up: a later send with the same tag must not write into it
      std::lock_guard<std::mutex> g(q_m_);
      for (auto it = addr_notes_.begin(); it != addr_notes_.end(); ++it)
        if (it->comm_sig == p.hdr.comm_sig && it->src == p.hdr.src && it->tag == p.hdr.tag && it->kind == p.hdr.seqn &&
            it->vaddr == p.hdr.vaddr) {
          addr_notes_.erase(it);
          break;
        }
      break;
    }
    }
  }
}

// find the eager message (src, tag, seqn) among RESERVED buffers; blocks up to timeout
int Engine::rx_seek(uint32_t comm_sig, uint32_t src_global, uint32_t tag, uint32_t seqn, uint64_t tmo_us) {
  std::unique_lock<std::mutex> lk(rx_m_);
  int found = -1;
  auto scan = [&] {
    std::lock_guard<std::mutex> e(exch_m_);
    const uint32_t n = exch_[exchmem::EAGER_RX_BUF_COUNT / 4];
    for (uint32_t i = 0; i < n; ++i) {
      const uint32_t st = exch_[exchmem::rxbuf_offset(i, exchmem::RX_STATUS) / 4];
      if (st != exchmem::RX_RESERVED && st != exchmem::RX_ERROR) continue;
      if (exch_[exchmem::rxbuf_offset(i, exchmem::RX_SRC) / 4] != src_global) continue;
      if (exch_[exchmem::rxbuf_offset(i, exchmem::RX_SEQ) / 4] != seqn) continue;
      if (i < rx_meta_.size() && rx_meta_[i].comm_sig != comm_sig) continue;
      const uint32_t btag = exch_[exchmem::rxbuf_offset(i, exchmem::RX_TAG) / 4];
      if (tag != TAG_ANY && btag != tag) continue;
      found = static_cast<int>(i);
      return true;
    }
    return false;
  };
  // The pool fills in arrival order.  When it is exhausted by messages nobody is asking for yet (many
  // peers, few buffers: all-to-all, gather fan-in) the one being sought may sit in the overflow queue
  // forever.  Swap it in: a parked message goes back to the queue, the sought one takes its buffer.
  auto swap_in = [&]() -> bool {
    for (auto it = rx_overflow_.begin(); it != rx_overflow_.end(); ++it) {
      const Packet &p = *it;
      if (p.hdr.src != src_global || p.hdr.seqn != seqn || p.hdr.comm_sig != comm_sig) continue;
      if (tag != TAG_ANY && p.hdr.tag != tag) continue;
      std::lock_guard<std::mutex> e(exch_m_);
      const uint32_t n = exch_[exchmem::EAGER_RX_BUF_COUNT / 4];
      for (uint32_t i = 0; i < n; ++i) {
        if (exch_[exchmem::rxbuf_offset(i, exchmem::RX_STATUS) / 4] != exchmem::RX_RESERVED) continue;
        const uint32_t maxlen = exch_[exchmem::rxbuf_offset(i, exchmem::RX_MAX_LEN) / 4];
        if (p.payload.size() > maxlen) continue;
        const uint64_t addr = (static_cast<uint64_t>(exch_[exchmem::rxbuf_offset(i, exchmem::RX_ADDR_HI) / 4]) << 32) |
                              exch_[exchmem::rxbuf_offset(i, exchmem::RX_ADDR_LO) / 4];
        uint32_t err = 0;
        uint8_t *buf = mem_ptr(addr, maxlen, err);
        if (!buf) continue;
        // evict buffer i into a packet ...
        Packet parked;
        parked.hdr.src = exch_[exchmem::rxbuf_offset(i, exchmem::RX_SRC) / 4];
        parked.hdr.dst = static_cast<uint32_t>(rank_);
        parked.hdr.seqn = exch_[exchmem::rxbuf_offset(i, exchmem::RX_SEQ) / 4];
        parked.hdr.tag = exch_[exchmem::rxbuf_offset(i, exchmem::RX_TAG) / 4];
        const uint32_t len = exch_[exchmem::rxbuf_offset(i, exchmem::RX_LEN) / 4];
        if (i < rx_meta_.size()) {
          parked.hdr.comm_sig = rx_meta_[i].comm_sig;
          parked.hdr.elems = rx_meta_[i].elems;
          parked.hdr.dtypes = rx_meta_[i].dtypes;
        }
        parked.payload.assign(buf, buf + len);
        // ... and land the sought message in its place
        if (!p.payload.empty()) std::memcpy(buf, p.payload.data(), p.payload.size());
        if (rx_meta_.size() <= i) rx_meta_.resize(i + 1);
        rx_meta_[i] = RxMeta{p.hdr.comm_sig, p.hdr.elems, p.hdr.dtypes};
        exch_[exchmem::rxbuf_offset(i, exchmem::RX_TAG) / 4] = p.hdr.tag;
        exch_[exchmem::rxbuf_offset(i, exchmem::RX_LEN) / 4] = static_cast<uint32_t>(p.payload.size());
        exch_[exchmem::rxbuf_offset(i, exchmem::RX_SRC) / 4] = p.hdr.src;
        exch_[exchmem::rxbuf_offset(i, exchmem::RX_SEQ) / 4] = p.hdr.seqn;
        rx_overflow_.erase(it);
        rx_overflow_.push_back(std::move(parked));
        found = static_cast<int>(i);
        return true;
      }
      return false; // sought message is here but no buffer can take it
    }
    return false;
  };
  const auto deadline = std::chrono::steady_clock::now() + std::chrono::microseconds(tmo_us);
  while (!stop_.load()) {
    if (scan()) break;
    if (!rx_overflow_.empty() && swap_in()) break;
    // Wait in short slices.  Between slices let parked rendezvous sends go out: the peer we are waiting for may
    // itself be waiting for one of them (A: isend(rendezvous) then eager recv / collective; B: recv, then the
    // matching eager send) — this thread is the only one that can move them.
    const auto now = std::chrono::steady_clock::now();
    if (now >= deadline) break;
    const auto slice = std::min<std::chrono::steady_clock::duration>(deadline - now, std::chrono::microseconds(200));
    rx_cv_.wait_for(lk, slice);
    lk.unlock();
    progress_parked_sends();
    lk.lock();
  }
  return found;
}

// Nested progress from inside a blocking eager wait (control thread only): try every parked point-to-point
// send once, in issue order.  A rendezvous send never blocks (it returns NOT_READY while the receiver's address
// note is missing), so this cannot recurse into another wait.
void Engine::progress_parked_sends() {
  size_t idx = 0;
  for (;;) {
    EmuCall c;
    {
      std::lock_guard<std::mutex> g(q_m_);
      while (idx < retry_calls_.size() && static_cast<operation>(retry_calls_[idx].desc.scenario) != operation::send) ++idx;
      if (idx >= retry_calls_.size()) return;
      c = std::move(retry_calls_[idx]);
      retry_calls_.erase(retry_calls_.begin() + static_cast<std::ptrdiff_t>(idx));
    }
    // the interrupted call's view of the data mover and of the queue must survive
    const size_t saved_older = older_parked_;
    uint64_t sa[3], sb[3];
    std::memcpy(sa, prev_addr_, sizeof(sa));
    std::memcpy(sb, prev_bytes_, sizeof(sb));
    older_parked_ = idx;
    uint32_t rc;
    try {
      rc = dispatch(c);
    } catch (const std::exception &e) {
      ACCL_ERROR_LOG("emulator rank " << rank_ << ": " << e.what());
      rc = DMA_INTERNAL_ERROR;
    }
    older_parked_ = saved_older;
    std::memcpy(prev_addr_, sa, sizeof(sa));
    std::memcpy(prev_bytes_, sb, sizeof(sb));
    if (rc == NOT_READY_ERROR) {
      std::lock_guard<std::mutex> g(q_m_);
      const size_t at = std::min(idx, retry_calls_.size());
      retry_calls_.insert(retry_calls_.begin() + static_cast<std::ptrdiff_t>(at), std::move(c));
      idx = at + 1;
    } else {
      const uint64_t dur = now_ns() - c.t0_ns;
      if (c.req) c.req->complete(rc, dur);
      if (c.on_done) c.on_done(rc);
      // the list closed up: idx already points at the next candidate; an elder of the interrupted call is gone,
      // so that call's own position (and re-insert point) moves down by one
      if (idx < older_parked_) --older_parked_;
    }
  }
}

void Engine::rx_release(int idx) {
  std::lock_guard<std::mutex> g(rx_m_);
  {
    std::lock_guard<std::mutex> e(exch_m_);
    // released buffers are re-posted immediately (rxbuf_enqueue)
    exch_[exchmem::rxbuf_offset(static_cast<uint32_t>(idx), exchmem::RX_STATUS) / 4] =
        exch_[exchmem::PKT_ENABLED / 4] ? exchmem::RX_ENQUEUED : exchmem::RX_IDLE;
  }
  rx_try_fill_locked();
}

// ---------------------------------------------------------------- decode
static uint32_t comm_signature(const CommView &c) {
  uint32_t h = 2166136261u;
  for (uint32_t r = 0; r < c.size; ++r) h = (h ^ (c.session[r] + 1)) * 16777619u;
  return h ? h : 1;
}

bool Engine::decode(EmuCall &c, Ctx &x, uint32_t &err) {
  const CallDesc &d = c.desc;
  x.call = &c;
  x.op = static_cast<operation>(d.scenario);
  x.count = d.count;
  x.root = d.root_src_dst;
  x.tag = d.tag;
  x.func = d.function;
  x.cflags = d.compression_flags;
  x.sflags = d.stream_flags();
  x.hflags = d.host_flags();
  x.a0 = d.addr0();
  x.a1 = d.addr1();
  x.a2 = d.addr2();
  std::lock_guard<std::mutex> g(exch_m_);
  if (d.comm >= static_cast<uint32_t>(ACCL_MAX_COMMUNICATORS)) {
    err |= CONFIG_SWITCH_ERROR;
    return false;
  }
  const uint32_t cb = exchmem::comm_offset(d.comm) / 4;
  x.comm.index = d.comm;
  x.comm.size = exch_[cb];
  x.comm.local_rank = exch_[cb + 1];
  if (x.comm.size > static_cast<uint32_t>(ACCL_MAX_RANKS)) {
    err |= CONFIG_SWITCH_ERROR;
    return false;
  }
  for (uint32_t r = 0; r < x.comm.size; ++r)
    x.comm.session[r] = exch_[exchmem::comm_rank_offset(d.comm, r, exchmem::CR_SESSION) / 4];
  // Two communicators over the same members (e.g. a "sub"-communicator of everybody next to the global
  // one) have separate sequence spaces, so their messages must not match each other's receives: mix in how
  // many earlier table entries have the identical member list.  Every member creates the communicators of
  // a given set collectively and in the same order, so all of them derive the same instance number.
  uint32_t instance = 0;
  for (uint32_t ci = 0; ci < d.comm; ++ci) {
    if (exch_[exchmem::comm_offset(ci) / 4] != x.comm.size) continue;
    bool same = true;
    for (uint32_t r = 0; r < x.comm.size && same; ++r)
      same = exch_[exchmem::comm_rank_offset(ci, r, exchmem::CR_SESSION) / 4] == x.comm.session[r];
    instance += same ? 1u : 0u;
  }
  x.comm.sig = comm_signature(x.comm) ^ (instance * 0x9E3779B9u);
  if (x.comm.sig == 0) x.comm.sig = 1;
  if (d.arithcfg >= exchmem::MAX_ARITHCFG) {
    err |= ARITH_ERROR;
    return false;
  }
  const uint32_t ab = exchmem::arith_offset(d.arithcfg, 0) / 4;
  x.ar.u = static_cast<dataType>(exch_[ab + exchmem::AC_UNCOMPRESSED_BYTES] >> 16);
  x.ar.c = static_cast<dataType>(exch_[ab + exchmem::AC_COMPRESSED_BYTES] >> 16);
  x.ar.ratio_log = exch_[ab + exchmem::AC_RATIO_LOG];
  x.ar.arith_compressed = exch_[ab + exchmem::AC_ARITH_COMPRESSED] != 0;
  x.max_eager = exch_[exchmem::MAX_EAGER_SIZE / 4];
  x.max_rndzv = exch_[exchmem::MAX_RENDEZVOUS_SIZE / 4];
  x.rxbuf_size = exch_[exchmem::EAGER_RX_BUF_SIZE / 4];
  x.spare_size = exch_[exchmem::SPARE_BUF_SIZE / 4];
  for (int i = 0; i < 3; ++i)
    x.spare[i] = (static_cast<uint64_t>(exch_[(exchmem::SPARE_BUF_BASE + 8 * i + 4) / 4]) << 32) |
                 exch_[(exchmem::SPARE_BUF_BASE + 8 * i) / 4];
  x.eth_c = x.cflags & static_cast<uint32_t>(compressionFlags::ETH_COMPRESSED);
  const uint64_t bytes = static_cast<uint64_t>(x.count) * dtype_bytes(x.ar.u);
  // eager iff small, or any compression, or any stream operand
  x.eager = bytes <= x.max_eager || x.cflags != 0 || x.sflags != 0;
  return true;
}

// ------------------------------------------------------------- data mover
uint64_t Engine::resolve(int slot, const Operand &o, size_t bytes, const Ctx &x) {
  uint64_t a = 0;
  switch (o.mode) {
  case MOVE_IMMEDIATE: a = o.addr; break;
  case MOVE_INCREMENT: a = prev_addr_[slot] + prev_bytes_[slot]; break;
  case MOVE_REPEAT: a = prev_addr_[slot]; break;
  case MOVE_STRIDE:
    a = static_cast<uint64_t>(static_cast<int64_t>(prev_addr_[slot]) +
                              o.stride * static_cast<int64_t>(dtype_bytes(o.compressed ? x.ar.c : x.ar.u)));
    break;
  default: return 0;
  }
  prev_addr_[slot] = a;
  prev_bytes_[slot] = bytes;
  return a;
}

uint32_t Engine::execute(Ctx &x, const Move &m) {
  uint32_t err = 0;
  const dataType U = x.ar.u, C = x.ar.c;
  const uint32_t rl = x.ar.ratio_log;
  const size_t n = m.count;
  if (n == 0) { // address-register priming
    if (m.op0.mode == MOVE_IMMEDIATE) { prev_addr_[0] = m.op0.addr; prev_bytes_[0] = 0; }
    if (m.op1.mode == MOVE_IMMEDIATE) { prev_addr_[1] = m.op1.addr; prev_bytes_[1] = 0; }
    if (m.res.mode == MOVE_IMMEDIATE) { prev_addr_[2] = m.res.addr; prev_bytes_[2] = 0; }
    return 0;
  }
  const dataType wire_t = m.eth_compressed ? C : U;
  const uint32_t dtypes_word = static_cast<uint32_t>(wire_t) | (static_cast<uint32_t>(U) << 8) | (rl << 16);

  auto fetch = [&](int slot, const Operand &o, std::vector<uint8_t> &buf, dataType &t) -> bool {
    if (o.mode == MOVE_NONE) return true;
    if (o.mode == MOVE_STREAM) {
      t = o.compressed ? C : U;
      buf.resize(repr_bytes(t, n, rl));
      if (!krnl_to_cclo_.pop(buf.data(), buf.size(), std::chrono::microseconds(timeout_us()))) {
        err |= KRNL_TIMEOUT_STS_ERROR;
        return false;
      }
      return true;
    }
    if (o.mode == MOVE_ON_RECV) {
      t = wire_t;
      const uint32_t src_global = x.comm.session[m.rx_src];
      const uint32_t seq_off = exchmem::comm_rank_offset(x.comm.index, m.rx_src, exchmem::CR_INBOUND_SEQ);
      const uint32_t seqn = read_exch(seq_off);
      int idx = rx_seek(x.comm.sig, src_global, m.rx_tag, seqn, timeout_us());
      if (idx < 0) {
        err |= RECEIVE_TIMEOUT_ERROR;
        return false;
      }
      const uint32_t i = static_cast<uint32_t>(idx);
      const uint32_t st = read_exch(exchmem::rxbuf_offset(i, exchmem::RX_STATUS));
      const uint32_t len = read_exch(exchmem::rxbuf_offset(i, exchmem::RX_LEN));
      const uint64_t addr = (static_cast<uint64_t>(read_exch(exchmem::rxbuf_offset(i, exchmem::RX_ADDR_HI))) << 32) |
                            read_exch(exchmem::rxbuf_offset(i, exchmem::RX_ADDR_LO));
      const size_t want = repr_bytes(t, n, rl);
      if (st == exchmem::RX_ERROR) err |= DEQUEUE_BUFFER_SPARE_BUFFER_STATUS_ERROR;
      if (len != want) err |= DMA_NOT_EXPECTED_BTT_ERROR;
      {
        std::lock_guard<std::mutex> g(rx_m_);
        if (i < rx_meta_.size() && rx_meta_[i].dtypes != dtypes_word) err |= COMPRESSION_ERROR;
      }
      if (!err) {
        buf.resize(want);
        uint32_t e = 0;
        uint8_t *p = mem_ptr(addr, want, e);
        if (p) std::memcpy(buf.data(), p, want);
        err |= e;
      }
      write_exch(seq_off, seqn + 1);
      rx_release(idx);
      return err == 0;
    }
    t = o.compressed ? C : U;
    const size_t bytes = repr_bytes(t, n, rl);
    const uint64_t a = resolve(slot, o, bytes, x);
    uint8_t *p = mem_ptr(a, bytes, err);
    if (!p) return false;
    buf.assign(p, p + bytes);
    return true;
  };

  std::vector<uint8_t> b0, b1, r;
  dataType t0 = U, t1 = U, tr = U;
  if (!fetch(0, m.op0, b0, t0)) return err ? err : DMA_INTERNAL_ERROR;
  if (!fetch(1, m.op1, b1, t1)) return err ? err : DMA_INTERNAL_ERROR;

  if (m.op0.mode != MOVE_NONE && m.op1.mode != MOVE_NONE) {
    const dataType A = x.ar.arith_compressed ? C : U;
    if (is_fp8(A)) return ARITH_ERROR;
    std::vector<uint8_t> a0(repr_bytes(A, n, 0)), a1(repr_bytes(A, n, 0));
    convert_buffer(b0.data(), t0, a0.data(), A, n, rl);
    convert_buffer(b1.data(), t1, a1.data(), A, n, rl);
    r.resize(a0.size());
    reduce_buffer(a0.data(), a1.data(), r.data(), A, n, m.func);
    tr = A;
  } else if (m.op0.mode != MOVE_NONE) {
    r.swap(b0);
    tr = t0;
  } else if (m.op1.mode != MOVE_NONE) {
    r.swap(b1);
    tr = t1;
  } else {
    return DMA_DECODE_ERROR;
  }

  auto to_repr = [&](dataType target) {
    if (target == tr) return;
    std::vector<uint8_t> o(repr_bytes(target, n, rl));
    convert_buffer(r.data(), tr, o.data(), target, n, rl);
    r.swap(o);
    tr = target;
  };

  if (m.res_remote) {
    to_repr(wire_t);
    Packet p;
    p.hdr.count = static_cast<uint32_t>(r.size());
    p.hdr.tag = m.tx_tag;
    p.hdr.src = static_cast<uint32_t>(rank_);
    p.hdr.dst = x.comm.session[m.dst_rank];
    p.hdr.comm_sig = x.comm.sig;
    p.hdr.elems = static_cast<uint32_t>(n);
    p.hdr.dtypes = dtypes_word;
    if (m.rendezvous) {
      p.hdr.msg_type = static_cast<uint32_t>(MsgType::RNDZVS_MSG);
      p.hdr.vaddr = m.remote_vaddr;
    } else {
      p.hdr.msg_type = static_cast<uint32_t>(MsgType::EGR_MSG);
      p.hdr.strm = m.res.mode == MOVE_STREAM ? m.strm : 0;
      if (p.hdr.strm == 0) {
        // ordered delivery per (communicator, peer): take and bump the outbound sequence number
        const uint32_t off = exchmem::comm_rank_offset(x.comm.index, m.dst_rank, exchmem::CR_OUTBOUND_SEQ);
        std::lock_guard<std::mutex> g(exch_m_);
        p.hdr.seqn = exch_[off / 4]++;
      } else if (m.eth_compressed) {
        // stream consumers see plain elements: decompress before it leaves
        to_repr(U);
        p.hdr.count = static_cast<uint32_t>(r.size());
      }
    }
    p.payload.swap(r);
    fabric_->send(std::move(p));
    return err;
  }
  if (m.res.mode == MOVE_STREAM) {
    to_repr(m.res.compressed ? C : U);
    if (loopback_) krnl_to_cclo_.push(r.data(), r.size());
    else out_stream(m.strm).push(r.data(), r.size());
    return err;
  }
  to_repr(m.res.compressed ? C : U);
  const uint64_t a = resolve(2, m.res, r.size(), x);
  uint8_t *p = mem_ptr(a, r.size(), err);
  if (p) std::memcpy(p, r.data(), r.size());
  return err;
}

uint64_t one_hop_dispatches();              // firmware.cpp
uint64_t one_hop_allreduce_forms(bool two_shot);

std::string Engine::debug_state() {
  std::ostringstream o;
  std::lock_guard<std::mutex> g(q_m_);
  o << "emulator rank " << rank_ << ": new=" << new_calls_.size() << " parked=" << retry_calls_.size()
    << " addr_notes=" << addr_notes_.size() << " done_notes=" << done_notes_.size()
    << " one_hop_dispatches=" << one_hop_dispatches() << " allreduce_one_shot=" << one_hop_allreduce_forms(false)
    << " allreduce_two_shot=" << one_hop_allreduce_forms(true);
  for (const auto &c : retry_calls_)
    o << "\n  parked: " << operation_name(static_cast<operation>(c.desc.scenario)) << " count=" << c.desc.count
      << " peer/root=" << c.desc.root_src_dst << " tag=" << c.desc.tag << " step=" << c.step << " mask=0x" << std::hex << c.mask
      << std::dec;
  for (const auto &n : addr_notes_) o << "\n  addr note: from " << n.src << " tag=" << n.tag << " count=" << n.count;
  for (const auto &n : done_notes_) o << "\n  done note: from " << n.src << " tag=" << n.tag << (n.barrier ? " (barrier token)" : "");
  return o.str();
}

} // namespace emu
} // namespace accl
