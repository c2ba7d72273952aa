// Backend abstraction: what the ACCL facade needs from "a device running a
// collective engine".  Two implementations ship: EmuDevice (CPU emulator of
// the engine, ranks as threads or processes) and CudaDevice (H100: symmetric
// NVLink heap, direct-launch kernels and the persistent engine kernel).
//
// Counterpart of the reference's pure-virtual CCLO with its XRT / Coyote /
// Sim implementations (driver/xrt/include/accl/cclo.hpp:41-201).  `Options`
// is the same canonical call descriptor; the additions are buffer allocation
// (each backend owns its memory) and an optional stream for stream-ordered
// execution on GPUs.
#pragma once
#include <chrono>
#include <memory>
#include <string>
#include <vector>

#include "accl/buffer.hpp"
#include "accl/constants.hpp"

namespace accl {

// The 16-word descriptor that actually reaches an engine (host ring, device
// ring or emulator command fifo).  Word order of the first 15 words matches
// the reference's stream ABI (driver/hls/accl_hls.h:134-198):
// scenario, count, comm, root_src_dst, function, tag, arithcfg,
// compression_flags, stream_flags|host_flags<<8, addr a/b/c as lo/hi pairs.
//
// alltoallv reuses two words: addr0 = send buffer, addr1 = int64 counts (2P), addr2 = receive buffer;
// `count` = receive capacity and `root_src_dst` (unused: no root) = send capacity, both in elements.
struct alignas(64) CallDesc {
  uint32_t scenario;
  uint32_t count;
  uint32_t comm;
  uint32_t root_src_dst;
  uint32_t function;
  uint32_t tag;
  uint32_t arithcfg;
  uint32_t compression_flags;
  uint32_t stream_host_flags;
  uint32_t addr0_lo, addr0_hi;
  uint32_t addr1_lo, addr1_hi;
  uint32_t addr2_lo, addr2_hi;
  uint32_t aux; // 16th word: resume step for parked calls / producer cookie

  ACCL_HD uint64_t addr0() const { return (static_cast<uint64_t>(addr0_hi) << 32) | addr0_lo; }
  ACCL_HD uint64_t addr1() const { return (static_cast<uint64_t>(addr1_hi) << 32) | addr1_lo; }
  ACCL_HD uint64_t addr2() const { return (static_cast<uint64_t>(addr2_hi) << 32) | addr2_lo; }
  ACCL_HD uint32_t stream_flags() const { return stream_host_flags & 0xFF; }
  ACCL_HD uint32_t host_flags() const { return (stream_host_flags >> 8) & 0xFF; }
  ACCL_HD void set_addr(int i, uint64_t a) {
    uint32_t lo = static_cast<uint32_t>(a), hi = static_cast<uint32_t>(a >> 32);
    if (i == 0) { addr0_lo = lo; addr0_hi = hi; }
    else if (i == 1) { addr1_lo = lo; addr1_hi = hi; }
    else { addr2_lo = lo; addr2_hi = hi; }
  }
};
static_assert(sizeof(CallDesc) == 64, "CallDesc must be one 64-byte record");

class CCLO {
public:
  struct Options {
    operation scenario = operation::nop;
    unsigned int count = 0; // elements
    communicatorId comm = GLOBAL_COMM;
    unsigned int root_src_dst = 0;
    cfgFunc cfg_function = cfgFunc::reset_periph;
    reduceFunction reduce_function = reduceFunction::SUM;
    unsigned int tag = TAG_ANY;
    addr_t arithcfg_addr = 0; // index of the arith config entry
    dataType compress_dtype = dataType::none;
    compressionFlags compression_flags = compressionFlags::NO_COMPRESSION;
    streamFlags stream_flags = streamFlags::NO_STREAM;
    hostFlags host_flags = hostFlags::NO_HOST;
    BaseBuffer *addr_0 = nullptr;
    BaseBuffer *addr_1 = nullptr;
    BaseBuffer *addr_2 = nullptr;
    dataType data_type_io_0 = dataType::none;
    dataType data_type_io_1 = dataType::none;
    dataType data_type_io_2 = dataType::none;
    std::vector<ACCLRequest *> waitfor;
    // GPU only: enqueue on this cudaStream_t instead of the backend's own stream
    void *stream = nullptr;
  };

  virtual ~CCLO() = default;

  // run to completion / start asynchronously; both return a request handle
  virtual ACCLRequest *call(const Options &options) = 0;
  virtual ACCLRequest *start(const Options &options) = 0;

  // exchange-memory access (byte offsets, 32-bit words; see exchmem.hpp)
  virtual val_t read(addr_t offset) = 0;
  virtual void write(addr_t offset, val_t val) = 0;

  virtual void wait(ACCLRequest *request) = 0;
  // false on timeout
  virtual bool wait(ACCLRequest *request, std::chrono::milliseconds timeout) = 0;
  virtual bool test(ACCLRequest *request) = 0;
  virtual void free_request(ACCLRequest *request) = 0;
  virtual val_t get_retcode(ACCLRequest *request) = 0;
  virtual uint64_t get_duration(ACCLRequest *request) = 0; // ns, engine-measured

  virtual deviceType get_device_type() = 0;
  virtual std::string describe() = 0;
  virtual void printDebug() {}
  // GPU backends: stream on which subsequent calls and buffer syncs are enqueued
  virtual void set_stream(void *stream) { (void)stream; }

  // Optional fast path for blocking calls whose operands live on the host: overlap the
  // host->device staging, the collective and the device->host read-back chunk by chunk.
  // Returns nullptr when the backend (or this call) does not support it.
  virtual ACCLRequest *call_host_pipelined(const Options &options) {
    (void)options;
    return nullptr;
  }

  // backend-owned memory
  virtual std::shared_ptr<BufferStorage> allocate(size_t bytes, bufferKind kind) = 0;
  // wrap caller-owned host memory (mirror is the caller's array)
  virtual std::shared_ptr<BufferStorage> wrap_host(void *host_ptr, size_t bytes) = 0;

  // called by the facade once ranks are known, before any configuration
  // write; lets the backend size per-peer structures
  virtual void attach(int world_size, int local_rank) = 0;
};

// Fill the engine descriptor from resolved options (shared by all backends).
CallDesc make_call_desc(const CCLO::Options &o);

} // namespace accl
