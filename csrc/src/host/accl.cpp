#include "accl/accl.hpp"

#include <algorithm>
#include <iomanip>
#include <set>
#include <sstream>
#include <stdexcept>

#include "accl/exchmem.hpp"

namespace accl {

CallDesc make_call_desc(const CCLO::Options &o) {
  CallDesc d{};
  d.scenario = static_cast<uint32_t>(o.scenario);
  d.count = o.count;
  d.comm = o.comm;
  d.root_src_dst = o.root_src_dst;
  d.function = o.scenario == operation::config ? static_cast<uint32_t>(o.cfg_function)
                                                : static_cast<uint32_t>(o.reduce_function);
  d.tag = o.tag;
  d.arithcfg = static_cast<uint32_t>(o.arithcfg_addr);
  d.compression_flags = static_cast<uint32_t>(o.compression_flags);
  d.stream_host_flags = static_cast<uint32_t>(o.stream_flags) | (static_cast<uint32_t>(o.host_flags) << 8);
  d.set_addr(0, o.addr_0 ? o.addr_0->address() : 0);
  d.set_addr(1, o.addr_1 ? o.addr_1->address() : 0);
  d.set_addr(2, o.addr_2 ? o.addr_2->address() : 0);
  d.aux = 0;
  return d;
}

ACCL::ACCL(std::unique_ptr<CCLO> device, const arithConfigMap &ac) : cclo(std::move(device)), arith_config(ac) {}

ACCL::~ACCL() {
  alive_->store(false);
  try {
    deinit();
  } catch (...) {
  }
}

void ACCL::deinit() {
  if (!cclo) return;
  if (config_rdy) {
    try {
      soft_reset();
    } catch (...) {
    }
  }
  eager_rx_buffers.clear();
  spare_buffers.clear();
  communicators.clear();
  config_rdy = false;
}

void ACCL::soft_reset() {
  CCLO::Options o;
  o.scenario = operation::config;
  o.cfg_function = cfgFunc::reset_periph;
  prepare_call(o);
  ACCLRequest *h = cclo->start(o);
  // the engine must acknowledge a reset promptly even with parked calls
  bool ok = cclo->wait(h, std::chrono::milliseconds(2000));
  if (ok) cclo->free_request(h);
  else ACCL_WARN_LOG("soft_reset: engine did not acknowledge within 2 s");
}

unsigned int ACCL::parse_hwid() {
  unsigned int hwid = cclo->read(exchmem::HWID);
  ACCL_DEBUG_LOG("HWID 0x" << std::hex << hwid << std::dec << " dma=" << !!(hwid & CAP_DMA)
                           << " arith=" << !!(hwid & CAP_ARITH) << " compression=" << !!(hwid & CAP_COMPRESSION)
                           << " streams=" << !!(hwid & CAP_STREAMS) << " rendezvous=" << !!(hwid & CAP_RENDEZVOUS)
                           << " nvls=" << !!(hwid & CAP_NVLS_MULTICAST) << " engine=" << !!(hwid & CAP_PERSISTENT_ENGINE)
                           << " fp8=" << !!(hwid & CAP_FP8));
  return hwid;
}

void ACCL::initialize(const std::vector<rank_t> &ranks, int local_rank, int n_egr_rx_bufs, addr_t egr_rx_buf_size,
                      addr_t max_egr_size, addr_t max_rndzv_size) {
  if (ranks.empty() || local_rank < 0 || local_rank >= static_cast<int>(ranks.size()))
    throw std::invalid_argument("initialize: bad rank table / local rank");
  if (ranks.size() > static_cast<size_t>(ACCL_MAX_RANKS))
    throw std::invalid_argument("initialize: more than ACCL_MAX_RANKS ranks");
  trace_rank_ = local_rank;
  cclo->attach(static_cast<int>(ranks.size()), ranks[static_cast<size_t>(local_rank)].session_id);
  parse_hwid();
  if (cclo->read(exchmem::CFGRDY) != 0)
    throw std::runtime_error("CCLO appears configured, might be in use. Please reset the engine before re-initializing.");

  setup_eager_rx_buffers(static_cast<size_t>(n_egr_rx_bufs), egr_rx_buf_size);
  setup_rendezvous_spare_buffers(max_rndzv_size);
  configure_communicator(ranks, local_rank);
  configure_arithmetic();
  configure_tuning_parameters();

  cclo->write(exchmem::CFGRDY, 1);
  config_rdy = true;
  set_timeout(1000000);
  set_max_eager_msg_size(static_cast<unsigned int>(max_egr_size));
  set_max_rendezvous_msg_size(static_cast<unsigned int>(max_rndzv_size));

  CCLO::Options o;
  o.scenario = operation::config;
  o.cfg_function = cfgFunc::enable_pkt;
  ACCLRequest *h = call_sync(o);
  check_return_value("enable_pkt", h);
  cclo->free_request(h);
  ACCL_DEBUG_LOG("initialized: " << cclo->describe());
}

void ACCL::setup_eager_rx_buffers(size_t n, addr_t size) {
  if (n > exchmem::MAX_RXBUFS) throw std::invalid_argument("too many eager rx buffers");
  eager_rx_buf_size_ = size;
  cclo->write(exchmem::EAGER_RX_BUF_SIZE, static_cast<val_t>(size));
  eager_rx_buffers.clear();
  for (size_t i = 0; i < n; ++i) {
    auto st = cclo->allocate(static_cast<size_t>(size), bufferKind::p2p);
    eager_rx_buffers.push_back(st);
    const addr_t a = st->device_addr();
    cclo->write(exchmem::rxbuf_offset(static_cast<uint32_t>(i), exchmem::RX_STATUS), exchmem::RX_IDLE);
    cclo->write(exchmem::rxbuf_offset(static_cast<uint32_t>(i), exchmem::RX_ADDR_LO), static_cast<val_t>(a));
    cclo->write(exchmem::rxbuf_offset(static_cast<uint32_t>(i), exchmem::RX_ADDR_HI), static_cast<val_t>(a >> 32));
    cclo->write(exchmem::rxbuf_offset(static_cast<uint32_t>(i), exchmem::RX_MAX_LEN), static_cast<val_t>(size));
    for (uint32_t w : {exchmem::RX_TAG, exchmem::RX_LEN, exchmem::RX_SRC, exchmem::RX_SEQ})
      cclo->write(exchmem::rxbuf_offset(static_cast<uint32_t>(i), w), 0);
  }
  // the count goes last: it tells the engine the table is complete
  cclo->write(exchmem::EAGER_RX_BUF_COUNT, static_cast<val_t>(n));
}

void ACCL::setup_rendezvous_spare_buffers(addr_t size) {
  // scratch for tree reductions / staging; engines chunk through it, so cap it
  // like the reference's bring-up code does (accl_network_utils.cpp:521: 4 MB)
  size = std::min<addr_t>(size, 4u << 20);
  spare_buffers.clear();
  cclo->write(exchmem::SPARE_BUF_SIZE, static_cast<val_t>(size));
  for (uint32_t i = 0; i < exchmem::NUM_SPARE_BUFS; ++i) {
    auto st = cclo->allocate(static_cast<size_t>(std::max<addr_t>(size, 64)), bufferKind::p2p);
    spare_buffers.push_back(st);
    const addr_t a = st->device_addr();
    cclo->write(exchmem::SPARE_BUF_BASE + i * 8, static_cast<val_t>(a));
    cclo->write(exchmem::SPARE_BUF_BASE + i * 8 + 4, static_cast<val_t>(a >> 32));
  }
}

void ACCL::configure_tuning_parameters() {
  // defaults of the reference (accl.cpp:1198-1208): fan-in 2 above 32 KB for
  // gather, flat-tree bcast up to 3 ranks, flat-tree reduce up to 4 ranks or
  // small messages.  The GPU backend maps these onto one-shot/two-shot
  // crossovers; the emulator uses them literally.
  cclo->write(exchmem::GATHER_FLAT_TREE_MAX_FANIN, 2);
  cclo->write(exchmem::GATHER_FLAT_TREE_MAX_COUNT, 32 * 1024);
  cclo->write(exchmem::BCAST_FLAT_TREE_MAX_RANKS, 3);
  cclo->write(exchmem::REDUCE_FLAT_TREE_MAX_RANKS, 4);
  cclo->write(exchmem::REDUCE_FLAT_TREE_MAX_COUNT, 32 * 1024);
  cclo->write(exchmem::ONE_HOP_SCHEDULES, one_hop_schedules_ ? 1 : 0);
}

void ACCL::set_one_hop_schedules(bool on) {
  one_hop_schedules_ = on;
  cclo->write(exchmem::ONE_HOP_SCHEDULES, on ? 1 : 0);
}

void ACCL::configure_arithmetic() {
  uint32_t idx = 0;
  for (auto &kv : arith_config) {
    if (idx >= exchmem::MAX_ARITHCFG) throw std::runtime_error("too many arithmetic configurations");
    uint32_t w[ARITHCFG_WORDS];
    serialize_arithconfig(kv.second, w);
    for (int i = 0; i < ARITHCFG_WORDS; ++i) cclo->write(exchmem::arith_offset(idx, static_cast<uint32_t>(i)), w[i]);
    kv.second.exchmem_addr = idx;
    ++idx;
  }
  if (idx >= exchmem::MAX_ARITHCFG) throw std::runtime_error("too many arithmetic configurations");
  uint32_t w[ARITHCFG_WORDS];
  serialize_arithconfig(byte_move_config_, w);
  for (int i = 0; i < ARITHCFG_WORDS; ++i) cclo->write(exchmem::arith_offset(idx, static_cast<uint32_t>(i)), w[i]);
  byte_move_config_.exchmem_addr = idx++;
  cclo->write(exchmem::NUM_ARITHCFG, idx);
}

void ACCL::configure_communicator(const std::vector<rank_t> &ranks, int local_rank) {
  if (communicators.size() >= static_cast<size_t>(ACCL_MAX_COMMUNICATORS))
    throw std::runtime_error("too many communicators");
  communicators.emplace_back(cclo.get(), ranks, static_cast<unsigned int>(local_rank),
                             static_cast<unsigned int>(communicators.size()));
  cclo->write(exchmem::NUM_COMMUNICATORS, static_cast<val_t>(communicators.size()));
}

communicatorId ACCL::create_communicator(const std::vector<rank_t> &ranks, int local_rank) {
  configure_communicator(ranks, local_rank);
  return static_cast<communicatorId>(communicators.size() - 1);
}

Communicator &ACCL::comm(communicatorId id) {
  if (id >= communicators.size()) throw std::out_of_range("unknown communicator id " + std::to_string(id));
  return communicators[id];
}
std::vector<rank_t> ACCL::get_comm_group(communicatorId id) { return comm(id).get_ranks(); }
unsigned int ACCL::get_comm_rank(communicatorId id) { return comm(id).local_rank(); }
addr_t ACCL::get_communicator_addr(communicatorId id) { return comm(id).communicators_addr(); }
addr_t ACCL::get_arithmetic_config_addr(std::pair<dataType, dataType> id) { return arith_config.at(id).exchmem_addr; }

std::string ACCL::dump_communicator() {
  std::ostringstream o;
  for (size_t i = 0; i < communicators.size(); ++i) o << "Communicator " << i << ":\n" << communicators[i].dump();
  return o.str();
}

std::string ACCL::dump_exchange_memory() {
  std::ostringstream o;
  o << "exchange mem:" << std::hex << std::setfill('0');
  for (uint32_t a = 0; a < exchmem::SIZE_BYTES; a += 16) {
    uint32_t w[4];
    bool nz = false;
    for (int i = 0; i < 4; ++i) nz |= (w[i] = cclo->read(a + 4u * static_cast<uint32_t>(i))) != 0;
    if (!nz) continue; // keep the dump readable: skip all-zero lines
    o << "\n0x" << std::setw(4) << a << ":";
    for (int i = 0; i < 4; ++i) o << " " << std::setw(8) << w[i];
  }
  o << std::dec << "\n";
  return o.str();
}

std::string ACCL::dump_eager_rx_buffers(bool dump_data) {
  std::ostringstream o;
  const uint32_t n = cclo->read(exchmem::EAGER_RX_BUF_COUNT);
  o << "eager rx buffers: " << n << " x " << cclo->read(exchmem::EAGER_RX_BUF_SIZE) << " B\n";
  static const char *st[] = {"IDLE", "ENQUEUED", "RESERVED", "ERROR"};
  for (uint32_t i = 0; i < n; ++i) {
    const uint32_t s = cclo->read(exchmem::rxbuf_offset(i, exchmem::RX_STATUS));
    const uint64_t a = (static_cast<uint64_t>(cclo->read(exchmem::rxbuf_offset(i, exchmem::RX_ADDR_HI))) << 32) |
                       cclo->read(exchmem::rxbuf_offset(i, exchmem::RX_ADDR_LO));
    o << "Spare RX Buffer " << i << ":\t address: 0x" << std::hex << a << std::dec << " \t status: "
      << (s < 4 ? st[s] : "?") << " \t occupancy: " << cclo->read(exchmem::rxbuf_offset(i, exchmem::RX_LEN)) << "/"
      << cclo->read(exchmem::rxbuf_offset(i, exchmem::RX_MAX_LEN))
      << " \t tag: " << cclo->read(exchmem::rxbuf_offset(i, exchmem::RX_TAG))
      << " \t src: " << cclo->read(exchmem::rxbuf_offset(i, exchmem::RX_SRC))
      << " \t seq: " << cclo->read(exchmem::rxbuf_offset(i, exchmem::RX_SEQ));
    if (dump_data && i < eager_rx_buffers.size() && eager_rx_buffers[i]->host_ptr()) {
      auto &b = eager_rx_buffers[i];
      b->from_device(0, b->bytes());
      o << " \t data: [" << std::hex;
      const unsigned char *p = static_cast<const unsigned char *>(b->host_ptr());
      for (size_t k = 0; k < std::min<size_t>(b->bytes(), 32); ++k) o << std::setw(2) << std::setfill('0') << +p[k];
      o << std::dec << "…]";
    }
    o << "\n";
  }
  return o.str();
}

// ------------------------------------------------------------ call plumbing
void ACCL::check_return_value(const std::string &fn, ACCLRequest *request) {
  val_t rc = cclo->get_retcode(request);
  if (rc != 0) {
    std::string msg = "CCLO @" + fn + ": " + error_word_to_string(rc) + " (0x";
    std::ostringstream h;
    h << std::hex << rc;
    free_request(request);
    throw std::runtime_error(msg + h.str() + ")");
  }
}

void ACCL::prepare_call(CCLO::Options &o) {
  if (!o.addr_0) { o.addr_0 = &dummy_buffer; }
  if (!o.addr_1) { o.addr_1 = &dummy_buffer; }
  if (!o.addr_2) { o.addr_2 = &dummy_buffer; }
  if (o.stream == nullptr) o.stream = stream_;
  if (o.data_type_io_0 == dataType::none) o.data_type_io_0 = o.addr_0->type();
  if (o.data_type_io_1 == dataType::none) o.data_type_io_1 = o.addr_1->type();
  if (o.data_type_io_2 == dataType::none) o.data_type_io_2 = o.addr_2->type();

  std::set<dataType> dtypes;
  for (dataType t : {o.data_type_io_0, o.data_type_io_1, o.data_type_io_2})
    if (t != dataType::none) dtypes.insert(t);
  dtypes.erase(dataType::none);

  o.host_flags = hostFlags::NO_HOST;
  if (o.addr_0->is_host_only()) o.host_flags |= hostFlags::OP0_HOST;
  if (o.addr_1->is_host_only()) o.host_flags |= hostFlags::OP1_HOST;
  if (o.addr_2->is_host_only()) o.host_flags |= hostFlags::RES_HOST;

  o.compression_flags = compressionFlags::NO_COMPRESSION;
  const ArithConfig *cfg = nullptr;
  if (dtypes.empty()) {
    // config / nop / barrier: any entry will do, take the first
    cfg = &arith_config.begin()->second;
  } else if (dtypes.size() == 1) {
    dataType t = *dtypes.begin();
    if (o.compress_dtype == dataType::none || o.compress_dtype == t) {
      const auto it = arith_config.find({t, t});
      if (it != arith_config.end()) cfg = &it->second;
      else if (o.scenario == operation::alltoallv && dtype_bytes(t) == 1) cfg = &byte_move_config_;
      else cfg = &arith_config.at({t, t}); // (throws: no configuration for this type)
    } else {
      cfg = &arith_config.at({t, o.compress_dtype});
      o.compression_flags |= compressionFlags::ETH_COMPRESSED;
    }
  } else if (dtypes.size() == 2) {
    // mixed operand types: the narrower one is the "compressed" representation
    auto it = dtypes.begin();
    dataType a = *it++, b = *it;
    dataType unc = dtype_bits(a) >= dtype_bits(b) ? a : b;
    dataType cmp = unc == a ? b : a;
    cfg = &arith_config.at({unc, cmp});
    if (o.data_type_io_0 == cmp) o.compression_flags |= compressionFlags::OP0_COMPRESSED;
    if (o.data_type_io_1 == cmp) o.compression_flags |= compressionFlags::OP1_COMPRESSED;
    if (o.data_type_io_2 == cmp) o.compression_flags |= compressionFlags::RES_COMPRESSED;
    // with operands already mixed, the wire uses the compressed type too
    if (o.compress_dtype == cmp) o.compression_flags |= compressionFlags::ETH_COMPRESSED;
  } else {
    throw std::runtime_error("unsupported: more than two data types in one call");
  }
  o.arithcfg_addr = cfg->exchmem_addr;
}

namespace {
// tracing hooks around the backend's start / call (no cost unless ACCL_TRACE / ACCL_NVTX are set)
template <typename F> ACCLRequest *traced(const CCLO::Options &o, int rank, F &&issue) {
  Tracer &t = Tracer::get();
  if (!Tracer::enabled() && !Tracer::nvtx()) return issue();
  const char *name = operation_name(o.scenario);
  t.range_push(name);
  const uint64_t t0 = t.now_ns();
  ACCLRequest *h = issue();
  const uint64_t cost = t.now_ns() - t0;
  t.range_pop();
  if (Tracer::enabled()) t.issue(h, rank, name, o.count, static_cast<unsigned>(o.comm), cost);
  return h;
}
} // namespace

ACCLRequest *ACCL::call_async(CCLO::Options &o) {
  if (!config_rdy && o.scenario != operation::config)
    throw std::runtime_error("ACCL not initialized");
  prepare_call(o);
  return traced(o, trace_rank_, [&] { return cclo->start(o); });
}

ACCLRequest *ACCL::call_sync(CCLO::Options &o) {
  if (!config_rdy && o.scenario != operation::config)
    throw std::runtime_error("ACCL not initialized");
  prepare_call(o);
  ACCLRequest *h = traced(o, trace_rank_, [&] { return cclo->call(o); });
  if (Tracer::enabled()) Tracer::get().complete(h, cclo->get_retcode(h), cclo->get_duration(h));
  return h;
}

void ACCL::free_request(ACCLRequest *request) {
  if (Tracer::enabled() && request) {
    try {
      if (cclo->test(request)) Tracer::get().complete(request, cclo->get_retcode(request), cclo->get_duration(request));
    } catch (...) { // already freed / unknown: nothing to record
    }
  }
  cclo->free_request(request);
}

ACCLRequest *ACCL::config_call(cfgFunc fn, unsigned int value, bool run_async, std::vector<ACCLRequest *> &waitfor) {
  CCLO::Options o;
  o.scenario = operation::config;
  o.cfg_function = fn;
  o.count = value;
  o.waitfor = waitfor;
  ACCLRequest *h = call_async(o);
  if (!run_async) {
    cclo->wait(h);
    check_return_value(std::string("config"), h);
  }
  return h;
}

ACCLRequest *ACCL::set_timeout(unsigned int value, bool run_async, std::vector<ACCLRequest *> waitfor) {
  return config_call(cfgFunc::set_timeout, value, run_async, waitfor);
}
ACCLRequest *ACCL::set_max_eager_msg_size(unsigned int value, bool run_async, std::vector<ACCLRequest *> waitfor) {
  ACCLRequest *h = config_call(cfgFunc::set_max_eager_msg_size, value, run_async, waitfor);
  max_eager_size_ = value;
  return h;
}
ACCLRequest *ACCL::set_max_rendezvous_msg_size(unsigned int value, bool run_async, std::vector<ACCLRequest *> waitfor) {
  ACCLRequest *h = config_call(cfgFunc::set_max_rendezvous_msg_size, value, run_async, waitfor);
  max_rndzv_size_ = value;
  return h;
}

ACCLRequest *ACCL::nop(bool run_async, std::vector<ACCLRequest *> waitfor) {
  CCLO::Options o;
  o.scenario = operation::nop;
  o.waitfor = waitfor;
  ACCLRequest *h = call_async(o);
  if (!run_async) {
    cclo->wait(h);
    check_return_value("nop", h);
  }
  return h;
}

namespace {
bool zero_count(const char *fn, unsigned int count) {
  if (count == 0) {
    ACCL_WARN_LOG("zero size buffer passed to " << fn << "; nothing to do");
    return true;
  }
  return false;
}
void warn_async_sync(const char *fn) {
  ACCL_WARN_LOG("ACCL: async run of " << fn << " with host-resident result: sync_from_device() the buffer yourself after wait()");
}
} // namespace

#define ACCL_FINISH(fn_name, handle, run_async, post_sync)                   \
  do {                                                                       \
    if (run_async) return handle;                                            \
    cclo->wait(handle);                                                      \
    if (Tracer::enabled())                                                   \
      Tracer::get().complete(handle, cclo->get_retcode(handle), cclo->get_duration(handle)); \
    post_sync;                                                               \
    check_return_value(fn_name, handle);                                     \
    return handle;                                                           \
  } while (0)

ACCLRequest *ACCL::send(BaseBuffer &srcbuf, unsigned int count, unsigned int dst, unsigned int tag,
                        communicatorId comm_id, bool from_fpga, dataType compress_dtype, bool run_async,
                        std::vector<ACCLRequest *> waitfor) {
  if (zero_count("send", count)) return nullptr;
  auto src = srcbuf.slice(0, count);
  if (!from_fpga) src->sync_to_device();
  CCLO::Options o;
  o.scenario = operation::send;
  o.comm = comm(comm_id).index();
  o.addr_0 = src.get();
  o.count = count;
  o.root_src_dst = dst;
  o.tag = tag;
  o.compress_dtype = compress_dtype;
  o.waitfor = waitfor;
  ACCLRequest *h = call_async(o);
  ACCL_FINISH("send", h, run_async, (void)0);
}

ACCLRequest *ACCL::send(dataType src_data_type, unsigned int count, unsigned int dst, unsigned int tag,
                        communicatorId comm_id, dataType compress_dtype, bool run_async,
                        std::vector<ACCLRequest *> waitfor) {
  if (zero_count("send", count)) return nullptr;
  CCLO::Options o;
  o.scenario = operation::send;
  o.comm = comm(comm_id).index();
  o.data_type_io_0 = src_data_type;
  o.stream_flags = streamFlags::OP0_STREAM;
  o.count = count;
  o.root_src_dst = dst;
  o.tag = tag;
  o.compress_dtype = compress_dtype;
  o.waitfor = waitfor;
  ACCLRequest *h = call_async(o);
  ACCL_FINISH("send", h, run_async, (void)0);
}

ACCLRequest *ACCL::stream_put(BaseBuffer &srcbuf, unsigned int count, unsigned int dst, unsigned int stream_id,
                              communicatorId comm_id, bool from_fpga, dataType compress_dtype, bool run_async,
                              std::vector<ACCLRequest *> waitfor) {
  if (stream_id < STREAM_ID_MIN || stream_id > STREAM_ID_MAX)
    throw std::invalid_argument("Stream ID must be in [9, 246]; 0-8 are reserved");
  if (zero_count("stream_put", count)) return nullptr;
  auto src = srcbuf.slice(0, count);
  if (!from_fpga) src->sync_to_device();
  CCLO::Options o;
  o.scenario = operation::send;
  o.comm = comm(comm_id).index();
  o.addr_0 = src.get();
  o.data_type_io_2 = srcbuf.type();
  o.stream_flags = streamFlags::RES_STREAM;
  o.count = count;
  o.root_src_dst = dst;
  o.tag = stream_id;
  o.compress_dtype = compress_dtype;
  o.waitfor = waitfor;
  ACCLRequest *h = call_async(o);
  ACCL_FINISH("stream_put", h, run_async, (void)0);
}

ACCLRequest *ACCL::stream_put(dataType src_data_type, unsigned int count, unsigned int dst, unsigned int stream_id,
                              communicatorId comm_id, dataType compress_dtype, bool run_async,
                              std::vector<ACCLRequest *> waitfor) {
  if (stream_id < STREAM_ID_MIN || stream_id > STREAM_ID_MAX)
    throw std::invalid_argument("Stream ID must be in [9, 246]; 0-8 are reserved");
  if (zero_count("stream_put", count)) return nullptr;
  CCLO::Options o;
  o.scenario = operation::send;
  o.comm = comm(comm_id).index();
  o.data_type_io_0 = src_data_type;
  o.data_type_io_2 = src_data_type;
  o.stream_flags = streamFlags::OP0_STREAM | streamFlags::RES_STREAM;
  o.count = count;
  o.root_src_dst = dst;
  o.tag = stream_id;
  o.compress_dtype = compress_dtype;
  o.waitfor = waitfor;
  ACCLRequest *h = call_async(o);
  ACCL_FINISH("stream_put", h, run_async, (void)0);
}

ACCLRequest *ACCL::recv(BaseBuffer &dstbuf, unsigned int count, unsigned int src, unsigned int tag,
                        communicatorId comm_id, bool to_fpga, dataType compress_dtype, bool run_async,
                        std::vector<ACCLRequest *> waitfor) {
  if (zero_count("recv", count)) return nullptr;
  if (!to_fpga && run_async) warn_async_sync("recv");
  auto dst = dstbuf.slice(0, count);
  CCLO::Options o;
  o.scenario = operation::recv;
  o.comm = comm(comm_id).index();
  o.addr_2 = dst.get();
  o.count = count;
  o.root_src_dst = src;
  o.tag = tag;
  o.compress_dtype = compress_dtype;
  o.waitfor = waitfor;
  ACCLRequest *h = call_async(o);
  ACCL_FINISH("recv", h, run_async, if (!to_fpga) dst->sync_from_device());
}

ACCLRequest *ACCL::recv(dataType dst_data_type, unsigned int count, unsigned int src, unsigned int tag,
                        communicatorId comm_id, dataType compress_dtype, bool run_async,
                        std::vector<ACCLRequest *> waitfor) {
  if (zero_count("recv", count)) return nullptr;
  CCLO::Options o;
  o.scenario = operation::recv;
  o.comm = comm(comm_id).index();
  o.data_type_io_2 = dst_data_type;
  o.stream_flags = streamFlags::RES_STREAM;
  o.count = count;
  o.root_src_dst = src;
  o.tag = tag;
  o.compress_dtype = compress_dtype;
  o.waitfor = waitfor;
  ACCLRequest *h = call_async(o);
  ACCL_FINISH("recv", h, run_async, (void)0);
}

ACCLRequest *ACCL::copy(BaseBuffer &srcbuf, BaseBuffer &dstbuf, unsigned int count, bool from_fpga, bool to_fpga,
                        bool run_async, std::vector<ACCLRequest *> waitfor) {
  if (zero_count("copy", count)) return nullptr;
  if (!to_fpga && run_async) warn_async_sync("copy");
  auto src = srcbuf.slice(0, count);
  auto dst = dstbuf.slice(0, count);
  if (!from_fpga) src->sync_to_device();
  CCLO::Options o;
  o.scenario = operation::copy;
  o.addr_0 = src.get();
  o.addr_2 = dst.get();
  o.count = count;
  o.waitfor = waitfor;
  ACCLRequest *h = call_async(o);
  ACCL_FINISH("copy", h, run_async, if (!to_fpga) dst->sync_from_device());
}

ACCLRequest *ACCL::copy_from_stream(BaseBuffer &dstbuf, unsigned int count, bool to_fpga, bool run_async,
                                    std::vector<ACCLRequest *> waitfor) {
  if (zero_count("copy_from_stream", count)) return nullptr;
  auto dst = dstbuf.slice(0, count);
  CCLO::Options o;
  o.scenario = operation::copy;
  o.addr_2 = dst.get();
  o.data_type_io_0 = dstbuf.type();
  o.stream_flags = streamFlags::OP0_STREAM;
  o.count = count;
  o.waitfor = waitfor;
  ACCLRequest *h = call_async(o);
  ACCL_FINISH("copy_from_stream", h, run_async, if (!to_fpga) dst->sync_from_device());
}

ACCLRequest *ACCL::copy_to_stream(BaseBuffer &srcbuf, unsigned int count, bool from_fpga, bool run_async,
                                  std::vector<ACCLRequest *> waitfor) {
  if (zero_count("copy_to_stream", count)) return nullptr;
  auto src = srcbuf.slice(0, count);
  if (!from_fpga) src->sync_to_device();
  CCLO::Options o;
  o.scenario = operation::copy;
  o.addr_0 = src.get();
  o.data_type_io_2 = srcbuf.type();
  o.stream_flags = streamFlags::RES_STREAM;
  o.count = count;
  o.waitfor = waitfor;
  ACCLRequest *h = call_async(o);
  ACCL_FINISH("copy_to_stream", h, run_async, (void)0);
}

ACCLRequest *ACCL::copy_from_to_stream(dataType data_type, unsigned int count, bool run_async,
                                       std::vector<ACCLRequest *> waitfor) {
  if (zero_count("copy_from_to_stream", count)) return nullptr;
  CCLO::Options o;
  o.scenario = operation::copy;
  o.data_type_io_0 = data_type;
  o.data_type_io_2 = data_type;
  o.stream_flags = streamFlags::OP0_STREAM | streamFlags::RES_STREAM;
  o.count = count;
  o.waitfor = waitfor;
  ACCLRequest *h = call_async(o);
  ACCL_FINISH("copy_from_to_stream", h, run_async, (void)0);
}

ACCLRequest *ACCL::combine(unsigned int count, reduceFunction function, BaseBuffer &val1, BaseBuffer &val2,
                           BaseBuffer &result, bool val1_from_fpga, bool val2_from_fpga, bool to_fpga,
                           bool run_async, std::vector<ACCLRequest *> waitfor) {
  if (zero_count("combine", count)) return nullptr;
  if (!to_fpga && run_async) warn_async_sync("combine");
  auto a = val1.slice(0, count);
  auto b = val2.slice(0, count);
  auto r = result.slice(0, count);
  if (!val1_from_fpga) a->sync_to_device();
  if (!val2_from_fpga) b->sync_to_device();
  CCLO::Options o;
  o.scenario = operation::combine;
  o.addr_0 = a.get();
  o.addr_1 = b.get();
  o.addr_2 = r.get();
  o.reduce_function = function;
  o.count = count;
  o.waitfor = waitfor;
  ACCLRequest *h = call_async(o);
  ACCL_FINISH("combine", h, run_async, if (!to_fpga) r->sync_from_device());
}

ACCLRequest *ACCL::bcast(BaseBuffer &buf, unsigned int count, unsigned int root, communicatorId comm_id,
                         bool from_fpga, bool to_fpga, dataType compress_dtype, bool run_async,
                         std::vector<ACCLRequest *> waitfor) {
  if (zero_count("bcast", count)) return nullptr;
  Communicator &c = comm(comm_id);
  const bool is_root = c.local_rank() == root;
  if (!to_fpga && !is_root && run_async) warn_async_sync("bcast");
  auto b = buf.slice(0, count);
  if (is_root && !from_fpga) b->sync_to_device();
  CCLO::Options o;
  o.scenario = operation::bcast;
  o.comm = c.index();
  o.addr_0 = b.get();
  o.count = count;
  o.root_src_dst = root;
  o.compress_dtype = compress_dtype;
  o.waitfor = waitfor;
  ACCLRequest *h = call_async(o);
  ACCL_FINISH("bcast", h, run_async, if (!to_fpga && !is_root) b->sync_from_device());
}

ACCLRequest *ACCL::scatter(BaseBuffer &sendbuf, BaseBuffer &recvbuf, unsigned int count, unsigned int root,
                           communicatorId comm_id, bool from_fpga, bool to_fpga, dataType compress_dtype,
                           bool run_async, std::vector<ACCLRequest *> waitfor) {
  if (zero_count("scatter", count)) return nullptr;
  Communicator &c = comm(comm_id);
  const bool is_root = c.local_rank() == root;
  if (!to_fpga && run_async) warn_async_sync("scatter");
  std::unique_ptr<BaseBuffer> s;
  if (is_root) {
    s = sendbuf.slice(0, static_cast<size_t>(count) * c.size());
    if (!from_fpga) s->sync_to_device();
  }
  auto r = recvbuf.slice(0, count);
  CCLO::Options o;
  o.scenario = operation::scatter;
  o.comm = c.index();
  o.addr_0 = is_root ? s.get() : nullptr;
  o.data_type_io_0 = sendbuf.type();
  o.addr_2 = r.get();
  o.count = count;
  o.root_src_dst = root;
  o.compress_dtype = compress_dtype;
  o.waitfor = waitfor;
  ACCLRequest *h = call_async(o);
  ACCL_FINISH("scatter", h, run_async, if (!to_fpga) r->sync_from_device());
}

ACCLRequest *ACCL::gather(BaseBuffer &sendbuf, BaseBuffer &recvbuf, unsigned int count, unsigned int root,
                          communicatorId comm_id, bool from_fpga, bool to_fpga, dataType compress_dtype,
                          bool run_async, std::vector<ACCLRequest *> waitfor) {
  if (zero_count("gather", count)) return nullptr;
  Communicator &c = comm(comm_id);
  const bool is_root = c.local_rank() == root;
  if (!to_fpga && is_root && run_async) warn_async_sync("gather");
  if (eager_rx_buffers.size() < c.size() - 1 && count * dtype_bytes(sendbuf.type()) <= max_eager_size_)
    ACCL_WARN_LOG("ACCL: gather: fewer eager rx buffers than peers; large fan-in may stall");
  auto s = sendbuf.slice(0, count);
  if (!from_fpga) s->sync_to_device();
  std::unique_ptr<BaseBuffer> r;
  if (is_root) r = recvbuf.slice(0, static_cast<size_t>(count) * c.size());
  CCLO::Options o;
  o.scenario = operation::gather;
  o.comm = c.index();
  o.addr_0 = s.get();
  o.addr_2 = is_root ? r.get() : nullptr;
  o.data_type_io_2 = recvbuf.type();
  o.count = count;
  o.root_src_dst = root;
  o.compress_dtype = compress_dtype;
  o.waitfor = waitfor;
  ACCLRequest *h = call_async(o);
  ACCL_FINISH("gather", h, run_async, if (!to_fpga && is_root) r->sync_from_device());
}

ACCLRequest *ACCL::allgather(BaseBuffer &sendbuf, BaseBuffer &recvbuf, unsigned int count, communicatorId comm_id,
                             bool from_fpga, bool to_fpga, dataType compress_dtype, bool run_async,
                             std::vector<ACCLRequest *> waitfor) {
  if (zero_count("allgather", count)) return nullptr;
  Communicator &c = comm(comm_id);
  if (!to_fpga && run_async) warn_async_sync("allgather");
  auto s = sendbuf.slice(0, count);
  auto r = recvbuf.slice(0, static_cast<size_t>(count) * c.size());
  if (!from_fpga) s->sync_to_device();
  CCLO::Options o;
  o.scenario = operation::allgather;
  o.comm = c.index();
  o.addr_0 = s.get();
  o.addr_2 = r.get();
  o.count = count;
  o.compress_dtype = compress_dtype;
  o.waitfor = waitfor;
  ACCLRequest *h = call_async(o);
  ACCL_FINISH("allgather", h, run_async, if (!to_fpga) r->sync_from_device());
}

ACCLRequest *ACCL::reduce(BaseBuffer &sendbuf, BaseBuffer &recvbuf, unsigned int count, unsigned int root,
                          reduceFunction func, communicatorId comm_id, bool from_fpga, bool to_fpga,
                          dataType compress_dtype, bool run_async, std::vector<ACCLRequest *> waitfor) {
  if (zero_count("reduce", count)) return nullptr;
  Communicator &c = comm(comm_id);
  const bool is_root = c.local_rank() == root;
  if (!to_fpga && is_root && run_async) warn_async_sync("reduce");
  auto s = sendbuf.slice(0, count);
  auto r = recvbuf.slice(0, count);
  if (!from_fpga) s->sync_to_device();
  CCLO::Options o;
  o.scenario = operation::reduce;
  o.comm = c.index();
  o.addr_0 = s.get();
  o.addr_2 = is_root ? r.get() : nullptr;
  o.data_type_io_2 = recvbuf.type();
  o.count = count;
  o.reduce_function = func;
  o.root_src_dst = root;
  o.compress_dtype = compress_dtype;
  o.waitfor = waitfor;
  ACCLRequest *h = call_async(o);
  ACCL_FINISH("reduce", h, run_async, if (!to_fpga && is_root) r->sync_from_device());
}

ACCLRequest *ACCL::reduce(dataType src_data_type, BaseBuffer &recvbuf, unsigned int count, unsigned int root,
                          reduceFunction func, communicatorId comm_id, bool to_fpga, dataType compress_dtype,
                          bool run_async, std::vector<ACCLRequest *> waitfor) {
  if (zero_count("reduce", count)) return nullptr;
  Communicator &c = comm(comm_id);
  const bool is_root = c.local_rank() == root;
  auto r = recvbuf.slice(0, count);
  CCLO::Options o;
  o.scenario = operation::reduce;
  o.comm = c.index();
  o.data_type_io_0 = src_data_type;
  o.stream_flags = streamFlags::OP0_STREAM;
  o.addr_2 = is_root ? r.get() : nullptr;
  o.data_type_io_2 = recvbuf.type();
  o.count = count;
  o.reduce_function = func;
  o.root_src_dst = root;
  o.compress_dtype = compress_dtype;
  o.waitfor = waitfor;
  ACCLRequest *h = call_async(o);
  ACCL_FINISH("reduce", h, run_async, if (!to_fpga && is_root) r->sync_from_device());
}

ACCLRequest *ACCL::reduce(BaseBuffer &sendbuf, dataType dst_data_type, unsigned int count, unsigned int root,
                          reduceFunction func, communicatorId comm_id, bool from_fpga, dataType compress_dtype,
                          bool run_async, std::vector<ACCLRequest *> waitfor) {
  if (zero_count("reduce", count)) return nullptr;
  Communicator &c = comm(comm_id);
  auto s = sendbuf.slice(0, count);
  if (!from_fpga) s->sync_to_device();
  CCLO::Options o;
  o.scenario = operation::reduce;
  o.comm = c.index();
  o.addr_0 = s.get();
  o.data_type_io_2 = dst_data_type;
  o.stream_flags = streamFlags::RES_STREAM;
  o.count = count;
  o.reduce_function = func;
  o.root_src_dst = root;
  o.compress_dtype = compress_dtype;
  o.waitfor = waitfor;
  ACCLRequest *h = call_async(o);
  ACCL_FINISH("reduce", h, run_async, (void)0);
}

ACCLRequest *ACCL::reduce(dataType src_data_type, dataType dst_data_type, unsigned int count, unsigned int root,
                          reduceFunction func, communicatorId comm_id, dataType compress_dtype, bool run_async,
                          std::vector<ACCLRequest *> waitfor) {
  if (zero_count("reduce", count)) return nullptr;
  Communicator &c = comm(comm_id);
  CCLO::Options o;
  o.scenario = operation::reduce;
  o.comm = c.index();
  o.data_type_io_0 = src_data_type;
  o.data_type_io_2 = dst_data_type;
  o.stream_flags = streamFlags::OP0_STREAM | streamFlags::RES_STREAM;
  o.count = count;
  o.reduce_function = func;
  o.root_src_dst = root;
  o.compress_dtype = compress_dtype;
  o.waitfor = waitfor;
  ACCLRequest *h = call_async(o);
  ACCL_FINISH("reduce", h, run_async, (void)0);
}

ACCLRequest *ACCL::allreduce(BaseBuffer &sendbuf, BaseBuffer &recvbuf, unsigned int count, reduceFunction func,
                             communicatorId comm_id, bool from_fpga, bool to_fpga, dataType compress_dtype,
                             bool run_async, std::vector<ACCLRequest *> waitfor) {
  if (zero_count("allreduce", count)) return nullptr;
  Communicator &c = comm(comm_id);
  if (!to_fpga && run_async) warn_async_sync("allreduce");
  auto s = sendbuf.slice(0, count);
  auto r = recvbuf.slice(0, count);
  CCLO::Options o;
  o.scenario = operation::allreduce;
  o.comm = c.index();
  o.addr_0 = s.get();
  o.addr_2 = r.get();
  o.count = count;
  o.reduce_function = func;
  o.compress_dtype = compress_dtype;
  o.waitfor = waitfor;
  if (!from_fpga && !to_fpga && !run_async && config_rdy) {
    // host-resident operands, blocking call: let the backend overlap H2D / collective / D2H
    prepare_call(o);
    if (ACCLRequest *ph = cclo->call_host_pipelined(o)) {
      check_return_value("allreduce", ph);
      return ph;
    }
  }
  if (!from_fpga) s->sync_to_device();
  ACCLRequest *h = call_async(o);
  ACCL_FINISH("allreduce", h, run_async, if (!to_fpga) r->sync_from_device());
}

ACCLRequest *ACCL::reduce_scatter(BaseBuffer &sendbuf, BaseBuffer &recvbuf, unsigned int count,
                                  reduceFunction func, communicatorId comm_id, bool from_fpga, bool to_fpga,
                                  dataType compress_dtype, bool run_async, std::vector<ACCLRequest *> waitfor) {
  if (zero_count("reduce_scatter", count)) return nullptr;
  Communicator &c = comm(comm_id);
  if (!to_fpga && run_async) warn_async_sync("reduce_scatter");
  auto s = sendbuf.slice(0, static_cast<size_t>(count) * c.size());
  auto r = recvbuf.slice(0, count);
  if (!from_fpga) s->sync_to_device();
  CCLO::Options o;
  o.scenario = operation::reduce_scatter;
  o.comm = c.index();
  o.addr_0 = s.get();
  o.addr_2 = r.get();
  o.count = count;
  o.reduce_function = func;
  o.compress_dtype = compress_dtype;
  o.waitfor = waitfor;
  ACCLRequest *h = call_async(o);
  ACCL_FINISH("reduce_scatter", h, run_async, if (!to_fpga) r->sync_from_device());
}

ACCLRequest *ACCL::alltoall(BaseBuffer &sendbuf, BaseBuffer &recvbuf, unsigned int count, communicatorId comm_id,
                            bool from_fpga, bool to_fpga, dataType compress_dtype, bool run_async,
                            std::vector<ACCLRequest *> waitfor) {
  if (zero_count("alltoall", count)) return nullptr;
  Communicator &c = comm(comm_id);
  if (!to_fpga && run_async) warn_async_sync("alltoall");
  auto s = sendbuf.slice(0, static_cast<size_t>(count) * c.size());
  auto r = recvbuf.slice(0, static_cast<size_t>(count) * c.size());
  if (!from_fpga) s->sync_to_device();
  CCLO::Options o;
  o.scenario = operation::alltoall;
  o.comm = c.index();
  o.addr_0 = s.get();
  o.addr_2 = r.get();
  o.count = count;
  o.compress_dtype = compress_dtype;
  o.waitfor = waitfor;
  ACCLRequest *h = call_async(o);
  ACCL_FINISH("alltoall", h, run_async, if (!to_fpga) r->sync_from_device());
}

ACCLRequest *ACCL::alltoallv(BaseBuffer &sendbuf, BaseBuffer &recvbuf, BaseBuffer &counts, communicatorId comm_id,
                             bool from_fpga, bool to_fpga, bool run_async, std::vector<ACCLRequest *> waitfor) {
  Communicator &c = comm(comm_id);
  if (counts.type() != dataType::int64 || counts.length() < 2 * static_cast<size_t>(c.size()))
    throw std::invalid_argument("alltoallv: counts must be an int64 buffer of at least 2 x communicator size elements");
  if (counts.is_host_only() && cclo->get_device_type() == deviceType::cuda)
    throw std::invalid_argument("alltoallv: counts must live in device memory (the engine reads them)");
  if (sendbuf.type() != recvbuf.type()) throw std::invalid_argument("alltoallv: send and receive buffers differ in type");
  // the capacities travel in 32-bit descriptor words: recv in `count`, send in `root_src_dst`
  if (sendbuf.length() > 0xFFFFFFFFull || recvbuf.length() > 0xFFFFFFFFull)
    throw std::invalid_argument("alltoallv: buffers longer than 2^32 - 1 elements");
  if (!to_fpga && run_async) warn_async_sync("alltoallv");
  if (!from_fpga) {
    sendbuf.sync_to_device();
    counts.sync_to_device();
  }
  CCLO::Options o;
  o.scenario = operation::alltoallv;
  o.comm = c.index();
  o.addr_0 = &sendbuf;
  o.addr_1 = &counts;
  o.addr_2 = &recvbuf;
  o.data_type_io_1 = sendbuf.type(); // the counts' own type does not select the arithmetic configuration
  o.count = static_cast<unsigned int>(recvbuf.length());
  o.root_src_dst = static_cast<unsigned int>(sendbuf.length());
  o.waitfor = waitfor;
  ACCLRequest *h = call_async(o);
  ACCL_FINISH("alltoallv", h, run_async, if (!to_fpga) recvbuf.sync_from_device());
}

ACCLRequest *ACCL::barrier(communicatorId comm_id, std::vector<ACCLRequest *> waitfor) {
  CCLO::Options o;
  o.scenario = operation::barrier;
  o.comm = comm(comm_id).index();
  o.waitfor = waitfor;
  ACCLRequest *h = call_sync(o);
  check_return_value("barrier", h);
  return h;
}

std::unique_ptr<BaseBuffer> ACCL::create_buffer_any(size_t length, dataType type, bufferKind kind) {
  auto st = cclo->allocate(length * dtype_bytes(type), kind);
  return std::unique_ptr<BaseBuffer>(new BaseBuffer(st, 0, length * dtype_bytes(type), type));
}

std::unique_ptr<BaseBuffer> ACCL::wrap_buffer_any(void *host_ptr, size_t length, dataType type) {
  auto st = cclo->wrap_host(host_ptr, length * dtype_bytes(type));
  return std::unique_ptr<BaseBuffer>(new BaseBuffer(st, 0, length * dtype_bytes(type), type));
}

} // namespace accl
