// CPU model of one collective engine ("CCLO"): simulated device + host
// memory, exchange memory, a command queue with a retry queue for parked
// rendezvous calls, a data mover that executes move micro-instructions, an
// eager RX-buffer pool with (src, tag, seqn) matching, rendezvous mailboxes,
// and device-side stream ports.  One Engine per rank; engines talk through a
// Fabric.
//
// Functional counterpart of the reference's `cclo_emu`
// (test/model/emulator/cclo_emu.cpp:57-506), i.e. of the MicroBlaze firmware
// (kernels/cclo/fw/sw_apps/ccl_offload_control/src/ccl_offload_control.c) plus
// the HLS data plane (kernels/cclo/hls/dma_mover, rxbuf_offload, eth_intf).
// The structure is this library's own: three threads (control, ingress,
// nothing else) instead of ~45 free-running block threads, packets instead of
// 64-byte beats, and resumable step machines instead of firmware gotos.
#pragma once
#include <atomic>
#include <condition_variable>
#include <deque>
#include <functional>
#include <string>
#include <list>
#include <map>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>

#include "accl/allocator.hpp"
#include "accl/cclo.hpp"
#include "accl/emu/fabric.hpp"
#include "accl/exchmem.hpp"
#include "accl/request.hpp"

namespace accl {
namespace emu {

// addresses >= HOST_BASE refer to the simulated host memory arena
constexpr uint64_t DEV_BASE = 0x1000;
constexpr uint64_t HOST_BASE = 1ull << 40;

// Simulated memory arena backed by lazily committed anonymous pages.
class Arena {
public:
  Arena(uint64_t base, size_t capacity);
  ~Arena();
  uint64_t alloc(size_t bytes) { return alloc_.alloc(bytes, 64); }
  void free(uint64_t addr) { alloc_.free(addr); }
  bool contains(uint64_t addr, size_t len) const { return addr >= base_ && addr + len <= base_ + cap_; }
  uint8_t *ptr(uint64_t addr) { return mem_ + (addr - base_); }
  uint64_t base() const { return base_; }

private:
  uint64_t base_;
  size_t cap_;
  uint8_t *mem_;
  RangeAllocator alloc_;
};

// Byte FIFO with blocking pop: models an AXI stream between a user kernel
// and the engine.
class ByteFifo {
public:
  void push(const void *data, size_t n);
  bool pop(void *out, size_t n, std::chrono::microseconds timeout);
  size_t size();

private:
  std::mutex m_;
  std::condition_variable cv_;
  std::deque<uint8_t> q_;
};

enum MoveMode : uint8_t {
  MOVE_NONE = 0,
  MOVE_STREAM = 1,    // operand comes from / result goes to a stream port
  MOVE_IMMEDIATE = 2, // explicit address
  MOVE_ON_RECV = 3,   // operand is the next matching eager message
  MOVE_INCREMENT = 4, // previous address + previous length
  MOVE_REPEAT = 5,    // previous address again
  MOVE_STRIDE = 6     // previous address + stride elements
};

struct Operand {
  MoveMode mode = MOVE_NONE;
  uint64_t addr = 0;
  int64_t stride = 0;     // elements, for MOVE_STRIDE
  bool compressed = false; // operand memory holds the compressed representation
};

// One data-mover instruction (the reference's variable-length DMP word
// stream, dma_mover.cpp:355-421, as a struct).
struct Move {
  Operand op0, op1, res;
  uint32_t count = 0; // elements; 0 = prime address registers only
  reduceFunction func = reduceFunction::SUM;
  bool res_remote = false;  // result leaves through the fabric
  bool rendezvous = false;  // remote result is a one-sided write to remote_vaddr
  bool eth_compressed = false;
  uint32_t rx_src = 0, rx_tag = TAG_ANY; // for MOVE_ON_RECV operands (communicator rank)
  uint32_t dst_rank = 0, tx_tag = TAG_ANY;
  uint32_t strm = 0; // stream id for stream results (local or remote)
  uint64_t remote_vaddr = 0;
};

struct ArithView {
  dataType u = dataType::none, c = dataType::none;
  uint32_t ratio_log = 0;
  bool arith_compressed = false;
};

struct CommView {
  uint32_t index = 0, size = 0, local_rank = 0, sig = 0;
  uint32_t session[ACCL_MAX_RANKS] = {}; // global rank id per member
};

struct EmuCall {
  CallDesc desc{};
  std::shared_ptr<BaseRequest> req; // null for device-issued calls
  uint32_t step = 0;                // resume point of a parked call
  uint32_t mask = 0;                // peers already served (any-order phases)
  uint64_t t0_ns = 0;
  int client = 0;                   // 0 = host controller, 1.. = device-side clients
  std::function<void(uint32_t)> on_done; // device-side completion hook
};

class Engine {
public:
  Engine(int global_rank, int world, std::shared_ptr<Fabric> fabric, size_t dev_mem_bytes, size_t host_mem_bytes);
  ~Engine();

  int rank() const { return rank_; }
  int world() const { return world_; }

  // ---- MMIO-style access to exchange memory
  uint32_t read_exch(uint32_t byte_off);
  void write_exch(uint32_t byte_off, uint32_t v);

  // ---- memory
  uint64_t mem_alloc(size_t bytes, bool host);
  void mem_free(uint64_t addr);
  void mem_write(uint64_t addr, const void *src, size_t len);
  void mem_read(uint64_t addr, void *dst, size_t len);

  // ---- command ingress (the 2:1 client arbiter: host + device-side clients)
  void submit(EmuCall &&call);

  // ---- device-side stream ports (what a user kernel sees)
  void kernel_push(const void *data, size_t bytes);                 // kernel -> engine
  bool kernel_pull(uint32_t strm, void *out, size_t bytes, int timeout_ms); // engine -> kernel
  void set_kernel_loopback(bool on) { loopback_ = on; }

  std::string debug_state();

private:
  // ---- threads
  void control_loop();
  void ingress_loop();
  void on_packet(Packet &&p);

  // ---- firmware: one handler per scenario; return error word or NOT_READY_ERROR
  uint32_t dispatch(EmuCall &c);
  bool elder_conflict(const EmuCall &c);
  void progress_parked_sends();
  uint32_t fw_config(EmuCall &c);
  uint32_t fw_copy(EmuCall &c);
  uint32_t fw_combine(EmuCall &c);
  uint32_t fw_send(EmuCall &c);
  uint32_t fw_recv(EmuCall &c);
  uint32_t fw_bcast(EmuCall &c);
  uint32_t fw_scatter(EmuCall &c);
  uint32_t fw_gather(EmuCall &c);
  uint32_t fw_allgather(EmuCall &c);
  uint32_t fw_reduce(EmuCall &c);
  uint32_t fw_reduce_scatter(EmuCall &c);
  uint32_t fw_allreduce(EmuCall &c);
  uint32_t fw_barrier(EmuCall &c);
  uint32_t fw_alltoall(EmuCall &c);
  uint32_t fw_alltoallv(EmuCall &c);
  void soft_reset();

  struct Ctx; // decoded call context (engine.cpp)
  bool decode(EmuCall &c, Ctx &x, uint32_t &err);
  // one-hop schedules (exchmem::ONE_HOP_SCHEDULES): what the H100 backend's planner picks on an NVSwitch domain
  bool one_hop(const Ctx &x, uint64_t landing_bytes);
  // `last_extra`: elements the last rank's block has on top of `count` (two-shot all-reduce of a count that does not split)
  uint32_t onehop_gather(Ctx &x, uint32_t &step, uint32_t &mask, uint64_t own_block, uint64_t dst_base, uint64_t blk_bytes, uint32_t count,
                         uint32_t last_extra = 0);
  uint32_t onehop_reduce(Ctx &x, uint32_t &step, uint32_t &mask, uint64_t src_base, uint64_t src_stride, uint64_t dst, uint32_t count,
                         uint32_t last_extra = 0);
  void purge_notes_of(EmuCall &c);

  // eager building blocks (blocking, like the DMP)
  uint32_t egr_send(Ctx &x, uint32_t dst, Operand src, uint32_t count, uint32_t tag, bool to_stream, uint32_t strm);
  uint32_t egr_recv(Ctx &x, uint32_t src, Operand dst, uint32_t count, uint32_t tag, bool to_stream, uint32_t strm);
  uint32_t egr_recv_reduce(Ctx &x, uint32_t src, Operand local, Operand dst, uint32_t count, uint32_t tag);
  uint32_t egr_recv_reduce_send(Ctx &x, uint32_t src, Operand local, uint32_t dst_rank, uint32_t count, uint32_t tag);
  uint32_t seg_elems(const Ctx &x) const;

  // rendezvous building blocks (non-blocking; false = not ready)
  void rndzv_post_addr(Ctx &x, uint32_t src_rank, uint64_t vaddr, uint32_t count, uint32_t tag);
  bool rndzv_take_addr(Ctx &x, uint32_t from_rank, uint32_t tag, uint64_t &vaddr);
  bool rndzv_take_any_addr(Ctx &x, uint32_t exclude_mask, uint32_t tag, uint32_t &from_rank, uint64_t &vaddr);
  uint32_t rndzv_write(Ctx &x, uint32_t dst_rank, uint64_t src_addr, uint64_t vaddr, uint32_t count, uint32_t tag);
  bool rndzv_take_done(Ctx &x, uint32_t from_rank, uint32_t tag);
  bool rndzv_take_any_done(Ctx &x, uint32_t exclude_mask, uint32_t tag, uint32_t &from_rank);

  // ---- data mover
  uint32_t execute(Ctx &x, const Move &m);
  uint64_t resolve(int slot, const Operand &o, size_t bytes, const Ctx &x);
  uint8_t *mem_ptr(uint64_t addr, size_t len, uint32_t &err);
  int rx_seek(uint32_t comm_sig, uint32_t src_global, uint32_t tag, uint32_t seqn, uint64_t timeout_us);
  void rx_release(int idx);
  void rx_try_fill_locked();
  uint32_t timeout_us();

  int rank_, world_;
  std::shared_ptr<Fabric> fabric_;
  Arena dev_, host_;

  std::mutex exch_m_;
  uint32_t exch_[exchmem::SIZE_WORDS] = {};

  // command queues
  std::mutex q_m_;
  std::condition_variable q_cv_;
  std::deque<EmuCall> new_calls_, retry_calls_;
  size_t older_parked_ = 0; // parked calls issued before the one being dispatched (control thread only)
  std::atomic<bool> stop_{false};
  std::thread control_, ingress_;

  // ingress
  std::mutex in_m_;
  std::condition_variable in_cv_;
  std::deque<Packet> inbox_;

  // eager rx state (guarded by rx_m_)
  std::mutex rx_m_;
  std::condition_variable rx_cv_;
  struct RxMeta { uint32_t comm_sig = 0, elems = 0, dtypes = 0; };
  std::vector<RxMeta> rx_meta_;
  std::deque<Packet> rx_overflow_;

  // rendezvous mailboxes (guarded by q_m_ so arrivals wake the control loop)
  // kind: what posted the note (1 = point to point, 0x100 | opcode = that collective) — a send must never take
  // the address a collective announced with TAG_ANY, and vice versa
  // payload: what an alltoallv announces with its buffer (its counts and capacities)
  struct AddrNote { uint32_t comm_sig, src, tag, count; uint64_t vaddr; uint32_t kind; std::vector<uint8_t> payload; };
  struct DoneNote { uint32_t comm_sig, src, tag; bool barrier; uint32_t kind; };
  std::list<AddrNote> addr_notes_;
  std::list<DoneNote> done_notes_;
  uint64_t mailbox_events_ = 0;

  // data-mover address registers
  uint64_t prev_addr_[3] = {0, 0, 0};
  uint64_t prev_bytes_[3] = {0, 0, 0};

  // streams
  ByteFifo krnl_to_cclo_;
  std::mutex strm_m_;
  std::map<uint32_t, std::unique_ptr<ByteFifo>> cclo_to_krnl_;
  ByteFifo &out_stream(uint32_t id);
  bool loopback_ = true;
};

} // namespace emu
} // namespace accl
