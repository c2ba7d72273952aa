// accl::ACCL — the user-facing collective API.
//
// Method names, argument order, defaults and the data-movement conventions
// (host-resident data unless from_fpga/to_fpga say otherwise; per-rank element
// counts; sync vs async with request handles) follow the reference facade
// ACCL::ACCL (driver/xrt/include/accl.hpp:45-1133, src/accl.cpp) so code
// written against it ports by changing the constructor.  "fpga" in argument
// names means "device" (a H100 here).
#pragma once
#include <atomic>
#include <chrono>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "accl/arithconfig.hpp"
#include "accl/buffer.hpp"
#include "accl/cclo.hpp"
#include "accl/communicator.hpp"
#include "accl/constants.hpp"

namespace accl {

class ACCL {
public:
  // Takes ownership of a backend (EmuDevice, CudaDevice).
  explicit ACCL(std::unique_ptr<CCLO> device, const arithConfigMap &arith_config = default_arith_config());
  ~ACCL();
  ACCL(const ACCL &) = delete;
  ACCL &operator=(const ACCL &) = delete;
  // true while this object is alive: lets request handles held elsewhere (language bindings) release themselves
  // in their destructors without touching a destroyed engine
  std::shared_ptr<std::atomic<bool>> alive_token() const { return alive_; }

  // Configure the engine: eager RX buffers, rendezvous scratch, global
  // communicator, arithmetic table, tuning registers, thresholds; then enable
  // the data plane.  Defaults as the reference (accl.hpp:102-104).
  void initialize(const std::vector<rank_t> &ranks, int local_rank, int n_egr_rx_bufs = 16,
                  addr_t egr_rx_buf_size = 1024, addr_t max_egr_size = 1024,
                  addr_t max_rndzv_size = 32 * 1024);
  void soft_reset();
  void deinit();
  unsigned int parse_hwid();

  // ---- configuration calls
  ACCLRequest *set_timeout(unsigned int value, bool run_async = false, std::vector<ACCLRequest *> waitfor = {});
  ACCLRequest *set_max_eager_msg_size(unsigned int value, bool run_async = false, std::vector<ACCLRequest *> waitfor = {});
  ACCLRequest *set_max_rendezvous_msg_size(unsigned int value, bool run_async = false, std::vector<ACCLRequest *> waitfor = {});
  // Emulator: run all-gather / reduce-scatter / all-reduce as one-hop exchanges and the rooted collectives in their flat
  // forms — the schedules the H100 backend executes on an NVSwitch domain — instead of the reference's rings and trees.
  // Set it identically on every rank (before or after initialize).  The CUDA backend always runs one-hop schedules.
  void set_one_hop_schedules(bool on);
  bool one_hop_schedules() const { return one_hop_schedules_; }
  ACCLRequest *nop(bool run_async = false, std::vector<ACCLRequest *> waitfor = {});

  // ---- primitives
  ACCLRequest *send(BaseBuffer &srcbuf, unsigned int count, unsigned int dst, unsigned int tag = TAG_ANY,
                    communicatorId comm_id = GLOBAL_COMM, bool from_fpga = false,
                    dataType compress_dtype = dataType::none, bool run_async = false,
                    std::vector<ACCLRequest *> waitfor = {});
  // source is the device-side stream port
  ACCLRequest *send(dataType src_data_type, unsigned int count, unsigned int dst, unsigned int tag = TAG_ANY,
                    communicatorId comm_id = GLOBAL_COMM, dataType compress_dtype = dataType::none,
                    bool run_async = false, std::vector<ACCLRequest *> waitfor = {});
  // one-sided: lands in stream `stream_id` of rank dst, no matching recv
  ACCLRequest *stream_put(BaseBuffer &srcbuf, unsigned int count, unsigned int dst, unsigned int stream_id,
                          communicatorId comm_id = GLOBAL_COMM, bool from_fpga = false,
                          dataType compress_dtype = dataType::none, bool run_async = false,
                          std::vector<ACCLRequest *> waitfor = {});
  ACCLRequest *stream_put(dataType src_data_type, unsigned int count, unsigned int dst, unsigned int stream_id,
                          communicatorId comm_id = GLOBAL_COMM, dataType compress_dtype = dataType::none,
                          bool run_async = false, std::vector<ACCLRequest *> waitfor = {});
  ACCLRequest *recv(BaseBuffer &dstbuf, unsigned int count, unsigned int src, unsigned int tag = TAG_ANY,
                    communicatorId comm_id = GLOBAL_COMM, bool to_fpga = false,
                    dataType compress_dtype = dataType::none, bool run_async = false,
                    std::vector<ACCLRequest *> waitfor = {});
  ACCLRequest *recv(dataType dst_data_type, unsigned int count, unsigned int src, unsigned int tag = TAG_ANY,
                    communicatorId comm_id = GLOBAL_COMM, dataType compress_dtype = dataType::none,
                    bool run_async = false, std::vector<ACCLRequest *> waitfor = {});
  ACCLRequest *copy(BaseBuffer &srcbuf, BaseBuffer &dstbuf, unsigned int count, bool from_fpga = false,
                    bool to_fpga = false, bool run_async = false, std::vector<ACCLRequest *> waitfor = {});
  ACCLRequest *copy_from_stream(BaseBuffer &dstbuf, unsigned int count, bool to_fpga = false,
                                bool run_async = false, std::vector<ACCLRequest *> waitfor = {});
  ACCLRequest *copy_to_stream(BaseBuffer &srcbuf, unsigned int count, bool from_fpga = false,
                              bool run_async = false, std::vector<ACCLRequest *> waitfor = {});
  ACCLRequest *copy_from_to_stream(dataType data_type, unsigned int count, bool run_async = false,
                                   std::vector<ACCLRequest *> waitfor = {});
  ACCLRequest *combine(unsigned int count, reduceFunction function, BaseBuffer &val1, BaseBuffer &val2,
                       BaseBuffer &result, bool val1_from_fpga = false, bool val2_from_fpga = false,
                       bool to_fpga = false, bool run_async = false, std::vector<ACCLRequest *> waitfor = {});

  // ---- collectives
  ACCLRequest *bcast(BaseBuffer &buf, unsigned int count, unsigned int root, communicatorId comm_id = GLOBAL_COMM,
                     bool from_fpga = false, bool to_fpga = false, dataType compress_dtype = dataType::none,
                     bool run_async = false, std::vector<ACCLRequest *> waitfor = {});
  ACCLRequest *scatter(BaseBuffer &sendbuf, BaseBuffer &recvbuf, unsigned int count, unsigned int root,
                       communicatorId comm_id = GLOBAL_COMM, bool from_fpga = false, bool to_fpga = false,
                       dataType compress_dtype = dataType::none, bool run_async = false,
                       std::vector<ACCLRequest *> waitfor = {});
  ACCLRequest *gather(BaseBuffer &sendbuf, BaseBuffer &recvbuf, unsigned int count, unsigned int root,
                      communicatorId comm_id = GLOBAL_COMM, bool from_fpga = false, bool to_fpga = false,
                      dataType compress_dtype = dataType::none, bool run_async = false,
                      std::vector<ACCLRequest *> waitfor = {});
  ACCLRequest *allgather(BaseBuffer &sendbuf, BaseBuffer &recvbuf, unsigned int count,
                         communicatorId comm_id = GLOBAL_COMM, bool from_fpga = false, bool to_fpga = false,
                         dataType compress_dtype = dataType::none, bool run_async = false,
                         std::vector<ACCLRequest *> waitfor = {});
  ACCLRequest *reduce(BaseBuffer &sendbuf, BaseBuffer &recvbuf, unsigned int count, unsigned int root,
                      reduceFunction func, communicatorId comm_id = GLOBAL_COMM, bool from_fpga = false,
                      bool to_fpga = false, dataType compress_dtype = dataType::none, bool run_async = false,
                      std::vector<ACCLRequest *> waitfor = {});
  // stream -> memory
  ACCLRequest *reduce(dataType src_data_type, BaseBuffer &recvbuf, unsigned int count, unsigned int root,
                      reduceFunction func, communicatorId comm_id = GLOBAL_COMM, bool to_fpga = false,
                      dataType compress_dtype = dataType::none, bool run_async = false,
                      std::vector<ACCLRequest *> waitfor = {});
  // memory -> stream
  ACCLRequest *reduce(BaseBuffer &sendbuf, dataType dst_data_type, unsigned int count, unsigned int root,
                      reduceFunction func, communicatorId comm_id = GLOBAL_COMM, bool from_fpga = false,
                      dataType compress_dtype = dataType::none, bool run_async = false,
                      std::vector<ACCLRequest *> waitfor = {});
  // stream -> stream
  ACCLRequest *reduce(dataType src_data_type, dataType dst_data_type, unsigned int count, unsigned int root,
                      reduceFunction func, communicatorId comm_id = GLOBAL_COMM,
                      dataType compress_dtype = dataType::none, bool run_async = false,
                      std::vector<ACCLRequest *> waitfor = {});
  ACCLRequest *allreduce(BaseBuffer &sendbuf, BaseBuffer &recvbuf, unsigned int count, reduceFunction func,
                         communicatorId comm_id = GLOBAL_COMM, bool from_fpga = false, bool to_fpga = false,
                         dataType compress_dtype = dataType::none, bool run_async = false,
                         std::vector<ACCLRequest *> waitfor = {});
  ACCLRequest *reduce_scatter(BaseBuffer &sendbuf, BaseBuffer &recvbuf, unsigned int count, reduceFunction func,
                              communicatorId comm_id = GLOBAL_COMM, bool from_fpga = false, bool to_fpga = false,
                              dataType compress_dtype = dataType::none, bool run_async = false,
                              std::vector<ACCLRequest *> waitfor = {});
  ACCLRequest *alltoall(BaseBuffer &sendbuf, BaseBuffer &recvbuf, unsigned int count,
                        communicatorId comm_id = GLOBAL_COMM, bool from_fpga = false, bool to_fpga = false,
                        dataType compress_dtype = dataType::none, bool run_async = false,
                        std::vector<ACCLRequest *> waitfor = {});
  // Uneven all-to-all.  `counts` (int64, at least 2P elements, P = communicator size) is read by the engine:
  // counts[q] = elements this rank sends to rank q, counts[P + p] = elements it receives from rank p.  Blocks are
  // packed in rank order (exclusive prefix sums of the counts) in both buffers; their lengths are the capacities.
  // An inconsistent count matrix anywhere in the communicator fails the call with DMA_SIZE_ERROR on every rank
  // without writing any receive buffer.
  ACCLRequest *alltoallv(BaseBuffer &sendbuf, BaseBuffer &recvbuf, BaseBuffer &counts,
                         communicatorId comm_id = GLOBAL_COMM, bool from_fpga = false, bool to_fpga = false,
                         bool run_async = false, std::vector<ACCLRequest *> waitfor = {});
  ACCLRequest *barrier(communicatorId comm_id = GLOBAL_COMM, std::vector<ACCLRequest *> waitfor = {});

  // ---- requests
  void wait(ACCLRequest *request) { cclo->wait(request); }
  bool wait(ACCLRequest *request, std::chrono::milliseconds timeout) { return cclo->wait(request, timeout); }
  bool test(ACCLRequest *request) { return cclo->test(request); }
  uint64_t get_duration(ACCLRequest *request) { return cclo->get_duration(request); }
  val_t get_retcode(ACCLRequest *request) { return cclo->get_retcode(request); }
  void free_request(ACCLRequest *request);

  // ---- communicators
  std::vector<rank_t> get_comm_group(communicatorId comm_id);
  unsigned int get_comm_rank(communicatorId comm_id);
  communicatorId create_communicator(const std::vector<rank_t> &ranks, int local_rank);
  std::string dump_communicator();
  addr_t get_communicator_addr(communicatorId comm_id = GLOBAL_COMM);
  addr_t get_arithmetic_config_addr(std::pair<dataType, dataType> id);

  // ---- buffers
  template <typename dtype> std::unique_ptr<Buffer<dtype>> create_buffer(size_t length, dataType type) {
    return make_buffer<dtype>(length, type, bufferKind::device);
  }
  template <typename dtype> std::unique_ptr<Buffer<dtype>> create_buffer_host(size_t length, dataType type) {
    return make_buffer<dtype>(length, type, bufferKind::host_only);
  }
  template <typename dtype> std::unique_ptr<Buffer<dtype>> create_buffer_p2p(size_t length, dataType type) {
    return make_buffer<dtype>(length, type, bufferKind::p2p);
  }
  // wrap caller-owned host memory
  template <typename dtype>
  std::unique_ptr<Buffer<dtype>> create_buffer(dtype *host_buffer, size_t length, dataType type) {
    auto st = cclo->wrap_host(host_buffer, length * sizeof(dtype));
    return std::unique_ptr<Buffer<dtype>>(new Buffer<dtype>(st, 0, length, type));
  }
  // type-erased variant used by the language bindings
  std::unique_ptr<BaseBuffer> create_buffer_any(size_t length, dataType type, bufferKind kind = bufferKind::device);
  std::unique_ptr<BaseBuffer> wrap_buffer_any(void *host_ptr, size_t length, dataType type);

  // ---- introspection
  std::string dump_exchange_memory();
  std::string dump_eager_rx_buffers(bool dump_data = false);
  deviceType get_device_type() { return cclo->get_device_type(); }
  CCLO *device() { return cclo.get(); }
  addr_t max_eager_size() const { return max_eager_size_; }
  addr_t max_rendezvous_size() const { return max_rndzv_size_; }
  // GPU: enqueue subsequent calls on this cudaStream_t (nullptr = backend stream)
  void set_stream(void *stream) {
    stream_ = stream;
    cclo->set_stream(stream);
  }
  void *get_stream() const { return stream_; }

  // no-ops kept for source compatibility (TCP session management in the reference)
  void open_port(communicatorId = GLOBAL_COMM) {}
  void open_con(communicatorId = GLOBAL_COMM) {}
  void close_con(communicatorId = GLOBAL_COMM) {}

private:
  template <typename dtype> std::unique_ptr<Buffer<dtype>> make_buffer(size_t length, dataType type, bufferKind kind) {
    auto st = cclo->allocate(length * sizeof(dtype), kind);
    return std::unique_ptr<Buffer<dtype>>(new Buffer<dtype>(st, 0, length, type));
  }
  void configure_arithmetic();
  void setup_eager_rx_buffers(size_t n_egr_rx_bufs, addr_t egr_rx_buf_size);
  void setup_rendezvous_spare_buffers(addr_t rndzv_spare_buf_size);
  void configure_tuning_parameters();
  bool one_hop_schedules_ = false;
  void configure_communicator(const std::vector<rank_t> &ranks, int local_rank);
  void check_return_value(const std::string &function_name, ACCLRequest *request);
  void prepare_call(CCLO::Options &options);
  ACCLRequest *call_async(CCLO::Options &options);
  ACCLRequest *call_sync(CCLO::Options &options);
  ACCLRequest *config_call(cfgFunc fn, unsigned int value, bool run_async, std::vector<ACCLRequest *> &waitfor);
  Communicator &comm(communicatorId id);

  std::unique_ptr<CCLO> cclo;
  arithConfigMap arith_config;
  // one extra exchange-memory entry, outside `arith_config`: the element width of 1-byte payloads (int8, fp8) that
  // alltoallv moves as bytes; every other call on such buffers is still refused by the lookup in prepare_call
  ArithConfig byte_move_config_{dataType::int8, dataType::int8, 0, false};
  std::vector<Communicator> communicators;
  std::vector<std::shared_ptr<BufferStorage>> eager_rx_buffers;
  std::vector<std::shared_ptr<BufferStorage>> spare_buffers;
  DummyBuffer dummy_buffer;
  addr_t max_eager_size_ = 0, max_rndzv_size_ = 0, eager_rx_buf_size_ = 0;
  bool config_rdy = false;
  void *stream_ = nullptr;
  int trace_rank_ = 0; // pid of this instance's events in ACCL_TRACE output
  std::shared_ptr<std::atomic<bool>> alive_ = std::make_shared<std::atomic<bool>>(true);
};

} // namespace accl
