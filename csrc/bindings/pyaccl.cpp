// Python bindings (pybind11) for the C++ library: enums, rank_t, buffers,
// the ACCL facade, backend factories (emulator in-process / socket, CUDA) and
// the device-API test harness.  Blocking calls release the GIL so that ranks
// driven from Python threads make progress concurrently.
//
// The reference has no Python surface; this is the "Python/torch surface"
// item of SURVEY.md §7.2 step 9.
#include <pybind11/functional.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <execinfo.h>
#include <signal.h>
#include <unistd.h>

#include <cstring>
#include <future>

#include "accl/accl.hpp"
#include "accl/bootstrap.hpp"
#include "accl/emu/emudevice.hpp"
#include "accl/emu/remote.hpp"
#include "accl/emu/softfloat.hpp"
#include "accl/exchmem.hpp"
#ifdef ACCL_WITH_CUDA
#include "accl/cuda/cudadevice.hpp"
#include "accl/cuda/plugins.hpp"
#endif

namespace py = pybind11;
using namespace accl;

namespace {

// Handle of one started call.  Dropping the Python object releases the request in the engine's registry (a
// training loop issuing asynchronous calls and never calling free() must not grow it without bound).
struct PyRequest {
  ACCL *owner = nullptr;
  ACCLRequest *h = nullptr;
  std::shared_ptr<std::atomic<bool>> alive;
  PyRequest() = default;
  PyRequest(ACCL *o, ACCLRequest *r) : owner(o), h(r), alive(o ? o->alive_token() : nullptr) {}
  PyRequest(PyRequest &&o) noexcept : owner(o.owner), h(o.h), alive(std::move(o.alive)) { o.h = nullptr; }
  PyRequest &operator=(PyRequest &&o) noexcept {
    release();
    owner = o.owner;
    h = o.h;
    alive = std::move(o.alive);
    o.h = nullptr;
    return *this;
  }
  PyRequest(const PyRequest &) = delete;
  PyRequest &operator=(const PyRequest &) = delete;
  ~PyRequest() { release(); }
  void release() {
    if (owner && h && alive && alive->load()) {
      try {
        owner->free_request(h);
      } catch (...) {
      }
    }
    h = nullptr;
  }
  bool valid() const { return owner && h && alive && alive->load(); }
};

PyRequest wrap(ACCL &a, ACCLRequest *h) { return PyRequest(&a, h); }

using gil_release = py::call_guard<py::gil_scoped_release>;

} // namespace

static void accl_segv_handler(int sig) {
  void *frames[64];
  int n = backtrace(frames, 64);
  const char msg[] = "\n[accl] fatal signal, native backtrace:\n";
  (void)!write(2, msg, sizeof(msg) - 1);
  backtrace_symbols_fd(frames, n, 2);
  signal(sig, SIG_DFL);
  raise(sig);
}

PYBIND11_MODULE(_C, m) {
  if (getenv("ACCL_SEGV_TRACE")) {
    signal(SIGSEGV, accl_segv_handler);
    signal(SIGABRT, accl_segv_handler);
  }
  m.doc() = "accl_b200 native core: ACCL-compatible collectives for H100 (NVLink/NVSwitch) with a CPU emulator backend";

  py::enum_<dataType>(m, "DataType")
      .value("none", dataType::none).value("int8", dataType::int8).value("float16", dataType::float16)
      .value("float32", dataType::float32).value("float64", dataType::float64).value("int32", dataType::int32)
      .value("int64", dataType::int64).value("bfloat16", dataType::bfloat16)
      .value("float8_e4m3", dataType::float8_e4m3).value("float8_e5m2", dataType::float8_e5m2);
  py::enum_<reduceFunction>(m, "ReduceFunction").value("SUM", reduceFunction::SUM).value("MAX", reduceFunction::MAX);
  py::enum_<operation>(m, "Operation")
      .value("config", operation::config).value("copy", operation::copy).value("combine", operation::combine)
      .value("send", operation::send).value("recv", operation::recv).value("bcast", operation::bcast)
      .value("scatter", operation::scatter).value("gather", operation::gather).value("reduce", operation::reduce)
      .value("allgather", operation::allgather).value("allreduce", operation::allreduce)
      .value("reduce_scatter", operation::reduce_scatter).value("barrier", operation::barrier)
      .value("alltoall", operation::alltoall).value("alltoallv", operation::alltoallv).value("nop", operation::nop);
  py::enum_<bufferKind>(m, "BufferKind")
      .value("device", bufferKind::device).value("host_only", bufferKind::host_only).value("p2p", bufferKind::p2p);
  py::enum_<deviceType>(m, "DeviceType").value("emulator", deviceType::emulator).value("cuda", deviceType::cuda);
  m.attr("TAG_ANY") = py::int_(TAG_ANY);
  m.attr("GLOBAL_COMM") = py::int_(GLOBAL_COMM);
  m.attr("NOT_READY_ERROR") = py::int_(static_cast<uint32_t>(NOT_READY_ERROR));
  m.def("dtype_bytes", [](dataType t) { return dtype_bytes(t); });
  m.def("error_to_string", [](uint32_t w) { return error_word_to_string(w); });
  m.def("set_log_level", [](int l) { Log::get().set_level(l); });

  py::class_<rank_t>(m, "Rank")
      .def(py::init<std::string, int, int, addr_t>(), py::arg("ip") = "127.0.0.1", py::arg("port") = 0,
           py::arg("session_id") = 0, py::arg("max_segment_size") = 0)
      .def_readwrite("ip", &rank_t::ip).def_readwrite("port", &rank_t::port)
      .def_readwrite("session_id", &rank_t::session_id).def_readwrite("max_segment_size", &rank_t::max_segment_size);

  py::class_<PyRequest>(m, "Request")
      .def("wait", [](PyRequest &r) { if (r.valid()) r.owner->wait(r.h); }, gil_release())
      .def("wait_for", [](PyRequest &r, int ms) { return r.valid() ? r.owner->wait(r.h, std::chrono::milliseconds(ms)) : true; }, gil_release())
      .def("test", [](PyRequest &r) { return r.valid() ? r.owner->test(r.h) : true; })
      .def("duration_ns", [](PyRequest &r) { return r.valid() ? r.owner->get_duration(r.h) : 0; })
      .def("retcode", [](PyRequest &r) { return r.valid() ? r.owner->get_retcode(r.h) : 0u; })
      .def("free", [](PyRequest &r) { r.release(); })
      .def_property_readonly("valid", &PyRequest::valid);

  py::class_<BaseBuffer>(m, "Buffer")
      .def_property_readonly("size", &BaseBuffer::size)
      .def_property_readonly("length", &BaseBuffer::length)
      .def_property_readonly("dtype", &BaseBuffer::type)
      .def_property_readonly("address", &BaseBuffer::address)
      .def_property_readonly("device_ptr", [](BaseBuffer &b) { return reinterpret_cast<uintptr_t>(b.device_ptr()); })
      .def_property_readonly("host_ptr", [](BaseBuffer &b) { return reinterpret_cast<uintptr_t>(b.byte_array()); })
      .def_property_readonly("is_host_only", &BaseBuffer::is_host_only)
      .def_property_readonly("is_simulated", &BaseBuffer::is_simulated)
      // writable view of the host side (wrap with numpy / torch.frombuffer)
      .def("host_view", [](BaseBuffer &b) {
        if (!b.byte_array()) throw std::runtime_error("buffer has no host side");
        return py::memoryview::from_memory(b.byte_array(), static_cast<py::ssize_t>(b.size()), false);
      }, py::keep_alive<0, 1>())
      .def("sync_to_device", &BaseBuffer::sync_to_device, gil_release())
      .def("sync_from_device", &BaseBuffer::sync_from_device, gil_release())
      .def("slice", [](BaseBuffer &b, size_t s, size_t e) { return b.slice(s, e); })
      .def("free", &BaseBuffer::free_buffer);

  py::class_<ACCL>(m, "ACCL")
      .def("initialize", &ACCL::initialize, py::arg("ranks"), py::arg("local_rank"), py::arg("n_egr_rx_bufs") = 16,
           py::arg("egr_rx_buf_size") = 1024, py::arg("max_egr_size") = 1024, py::arg("max_rndzv_size") = 32 * 1024,
           gil_release())
      .def("deinit", &ACCL::deinit, gil_release())
      .def("soft_reset", &ACCL::soft_reset, gil_release())
      .def("parse_hwid", &ACCL::parse_hwid)
      .def("device_type", &ACCL::get_device_type)
      .def("describe", [](ACCL &a) { return a.device()->describe(); })
      .def("set_stream", [](ACCL &a, uintptr_t s) { a.set_stream(reinterpret_cast<void *>(s)); })
      .def("create_buffer", [](ACCL &a, size_t n, dataType t, bufferKind k) { return a.create_buffer_any(n, t, k); },
           py::arg("length"), py::arg("dtype"), py::arg("kind") = bufferKind::device, py::keep_alive<0, 1>())
      .def("wrap_buffer", [](ACCL &a, uintptr_t host_ptr, size_t n, dataType t) {
        return a.wrap_buffer_any(reinterpret_cast<void *>(host_ptr), n, t);
      }, py::keep_alive<0, 1>())
      .def("set_timeout", [](ACCL &a, unsigned v) { a.free_request(a.set_timeout(v)); }, gil_release())
      .def("set_max_eager_msg_size", [](ACCL &a, unsigned v) { a.free_request(a.set_max_eager_msg_size(v)); }, gil_release())
      .def("set_one_hop_schedules", &ACCL::set_one_hop_schedules)
      .def("set_max_rendezvous_msg_size", [](ACCL &a, unsigned v) { a.free_request(a.set_max_rendezvous_msg_size(v)); }, gil_release())
      .def("nop", [](ACCL &a, bool async_) { return wrap(a, a.nop(async_)); }, py::arg("run_async") = false, gil_release())
      .def("send", [](ACCL &a, BaseBuffer &b, unsigned count, unsigned dst, unsigned tag, unsigned comm, bool from_fpga,
                      dataType cd, bool async_) { return wrap(a, a.send(b, count, dst, tag, comm, from_fpga, cd, async_)); },
           py::arg("srcbuf"), py::arg("count"), py::arg("dst"), py::arg("tag") = TAG_ANY, py::arg("comm_id") = GLOBAL_COMM,
           py::arg("from_fpga") = false, py::arg("compress_dtype") = dataType::none, py::arg("run_async") = false, gil_release())
      .def("send_from_stream", [](ACCL &a, dataType t, unsigned count, unsigned dst, unsigned tag, unsigned comm, dataType cd,
                                  bool async_) { return wrap(a, a.send(t, count, dst, tag, comm, cd, async_)); },
           py::arg("src_data_type"), py::arg("count"), py::arg("dst"), py::arg("tag") = TAG_ANY,
           py::arg("comm_id") = GLOBAL_COMM, py::arg("compress_dtype") = dataType::none, py::arg("run_async") = false, gil_release())
      .def("stream_put", [](ACCL &a, BaseBuffer &b, unsigned count, unsigned dst, unsigned stream_id, unsigned comm,
                            bool from_fpga, dataType cd, bool async_) {
        return wrap(a, a.stream_put(b, count, dst, stream_id, comm, from_fpga, cd, async_));
      }, py::arg("srcbuf"), py::arg("count"), py::arg("dst"), py::arg("stream_id"), py::arg("comm_id") = GLOBAL_COMM,
           py::arg("from_fpga") = false, py::arg("compress_dtype") = dataType::none, py::arg("run_async") = false, gil_release())
      .def("stream_put_from_stream", [](ACCL &a, dataType t, unsigned count, unsigned dst, unsigned stream_id, unsigned comm,
                                        dataType cd, bool async_) {
        return wrap(a, a.stream_put(t, count, dst, stream_id, comm, cd, async_));
      }, py::arg("src_data_type"), py::arg("count"), py::arg("dst"), py::arg("stream_id"), py::arg("comm_id") = GLOBAL_COMM,
           py::arg("compress_dtype") = dataType::none, py::arg("run_async") = false, gil_release())
      .def("recv", [](ACCL &a, BaseBuffer &b, unsigned count, unsigned src, unsigned tag, unsigned comm, bool to_fpga,
                      dataType cd, bool async_) { return wrap(a, a.recv(b, count, src, tag, comm, to_fpga, cd, async_)); },
           py::arg("dstbuf"), py::arg("count"), py::arg("src"), py::arg("tag") = TAG_ANY, py::arg("comm_id") = GLOBAL_COMM,
           py::arg("to_fpga") = false, py::arg("compress_dtype") = dataType::none, py::arg("run_async") = false, gil_release())
      .def("recv_to_stream", [](ACCL &a, dataType t, unsigned count, unsigned src, unsigned tag, unsigned comm, dataType cd,
                                bool async_) { return wrap(a, a.recv(t, count, src, tag, comm, cd, async_)); },
           py::arg("dst_data_type"), py::arg("count"), py::arg("src"), py::arg("tag") = TAG_ANY,
           py::arg("comm_id") = GLOBAL_COMM, py::arg("compress_dtype") = dataType::none, py::arg("run_async") = false, gil_release())
      .def("copy", [](ACCL &a, BaseBuffer &s, BaseBuffer &d, unsigned count, bool from_fpga, bool to_fpga, bool async_) {
        return wrap(a, a.copy(s, d, count, from_fpga, to_fpga, async_));
      }, py::arg("srcbuf"), py::arg("dstbuf"), py::arg("count"), py::arg("from_fpga") = false, py::arg("to_fpga") = false,
           py::arg("run_async") = false, gil_release())
      .def("copy_from_stream", [](ACCL &a, BaseBuffer &d, unsigned count, bool to_fpga, bool async_) {
        return wrap(a, a.copy_from_stream(d, count, to_fpga, async_));
      }, py::arg("dstbuf"), py::arg("count"), py::arg("to_fpga") = false, py::arg("run_async") = false, gil_release())
      .def("copy_to_stream", [](ACCL &a, BaseBuffer &s, unsigned count, bool from_fpga, bool async_) {
        return wrap(a, a.copy_to_stream(s, count, from_fpga, async_));
      }, py::arg("srcbuf"), py::arg("count"), py::arg("from_fpga") = false, py::arg("run_async") = false, gil_release())
      .def("copy_from_to_stream", [](ACCL &a, dataType t, unsigned count, bool async_) {
        return wrap(a, a.copy_from_to_stream(t, count, async_));
      }, py::arg("data_type"), py::arg("count"), py::arg("run_async") = false, gil_release())
      .def("combine", [](ACCL &a, unsigned count, reduceFunction f, BaseBuffer &v1, BaseBuffer &v2, BaseBuffer &r,
                         bool f1, bool f2, bool to_fpga, bool async_) {
        return wrap(a, a.combine(count, f, v1, v2, r, f1, f2, to_fpga, async_));
      }, py::arg("count"), py::arg("function"), py::arg("val1"), py::arg("val2"), py::arg("result"),
           py::arg("val1_from_fpga") = false, py::arg("val2_from_fpga") = false, py::arg("to_fpga") = false,
           py::arg("run_async") = false, gil_release())
      .def("bcast", [](ACCL &a, BaseBuffer &b, unsigned count, unsigned root, unsigned comm, bool from_fpga, bool to_fpga,
                       dataType cd, bool async_) { return wrap(a, a.bcast(b, count, root, comm, from_fpga, to_fpga, cd, async_)); },
           py::arg("buf"), py::arg("count"), py::arg("root"), py::arg("comm_id") = GLOBAL_COMM, py::arg("from_fpga") = false,
           py::arg("to_fpga") = false, py::arg("compress_dtype") = dataType::none, py::arg("run_async") = false, gil_release())
      .def("scatter", [](ACCL &a, BaseBuffer &s, BaseBuffer &r, unsigned count, unsigned root, unsigned comm, bool from_fpga,
                         bool to_fpga, dataType cd, bool async_) {
        return wrap(a, a.scatter(s, r, count, root, comm, from_fpga, to_fpga, cd, async_));
      }, py::arg("sendbuf"), py::arg("recvbuf"), py::arg("count"), py::arg("root"), py::arg("comm_id") = GLOBAL_COMM,
           py::arg("from_fpga") = false, py::arg("to_fpga") = false, py::arg("compress_dtype") = dataType::none,
           py::arg("run_async") = false, gil_release())
      .def("gather", [](ACCL &a, BaseBuffer &s, BaseBuffer &r, unsigned count, unsigned root, unsigned comm, bool from_fpga,
                        bool to_fpga, dataType cd, bool async_) {
        return wrap(a, a.gather(s, r, count, root, comm, from_fpga, to_fpga, cd, async_));
      }, py::arg("sendbuf"), py::arg("recvbuf"), py::arg("count"), py::arg("root"), py::arg("comm_id") = GLOBAL_COMM,
           py::arg("from_fpga") = false, py::arg("to_fpga") = false, py::arg("compress_dtype") = dataType::none,
           py::arg("run_async") = false, gil_release())
      .def("allgather", [](ACCL &a, BaseBuffer &s, BaseBuffer &r, unsigned count, unsigned comm, bool from_fpga, bool to_fpga,
                           dataType cd, bool async_) {
        return wrap(a, a.allgather(s, r, count, comm, from_fpga, to_fpga, cd, async_));
      }, py::arg("sendbuf"), py::arg("recvbuf"), py::arg("count"), py::arg("comm_id") = GLOBAL_COMM,
           py::arg("from_fpga") = false, py::arg("to_fpga") = false, py::arg("compress_dtype") = dataType::none,
           py::arg("run_async") = false, gil_release())
      .def("reduce", [](ACCL &a, BaseBuffer &s, BaseBuffer &r, unsigned count, unsigned root, reduceFunction f, unsigned comm,
                        bool from_fpga, bool to_fpga, dataType cd, bool async_) {
        return wrap(a, a.reduce(s, r, count, root, f, comm, from_fpga, to_fpga, cd, async_));
      }, py::arg("sendbuf"), py::arg("recvbuf"), py::arg("count"), py::arg("root"), py::arg("func") = reduceFunction::SUM,
           py::arg("comm_id") = GLOBAL_COMM, py::arg("from_fpga") = false, py::arg("to_fpga") = false,
           py::arg("compress_dtype") = dataType::none, py::arg("run_async") = false, gil_release())
      .def("reduce_stream2mem", [](ACCL &a, dataType st, BaseBuffer &r, unsigned count, unsigned root, reduceFunction f,
                                   unsigned comm, bool to_fpga, dataType cd, bool async_) {
        return wrap(a, a.reduce(st, r, count, root, f, comm, to_fpga, cd, async_));
      }, py::arg("src_data_type"), py::arg("recvbuf"), py::arg("count"), py::arg("root"), py::arg("func") = reduceFunction::SUM,
           py::arg("comm_id") = GLOBAL_COMM, py::arg("to_fpga") = false, py::arg("compress_dtype") = dataType::none,
           py::arg("run_async") = false, gil_release())
      .def("reduce_mem2stream", [](ACCL &a, BaseBuffer &s, dataType dt, unsigned count, unsigned root, reduceFunction f,
                                   unsigned comm, bool from_fpga, dataType cd, bool async_) {
        return wrap(a, a.reduce(s, dt, count, root, f, comm, from_fpga, cd, async_));
      }, py::arg("sendbuf"), py::arg("dst_data_type"), py::arg("count"), py::arg("root"), py::arg("func") = reduceFunction::SUM,
           py::arg("comm_id") = GLOBAL_COMM, py::arg("from_fpga") = false, py::arg("compress_dtype") = dataType::none,
           py::arg("run_async") = false, gil_release())
      .def("reduce_stream2stream", [](ACCL &a, dataType st, dataType dt, unsigned count, unsigned root, reduceFunction f,
                                      unsigned comm, dataType cd, bool async_) {
        return wrap(a, a.reduce(st, dt, count, root, f, comm, cd, async_));
      }, py::arg("src_data_type"), py::arg("dst_data_type"), py::arg("count"), py::arg("root"),
           py::arg("func") = reduceFunction::SUM, py::arg("comm_id") = GLOBAL_COMM,
           py::arg("compress_dtype") = dataType::none, py::arg("run_async") = false, gil_release())
      .def("allreduce", [](ACCL &a, BaseBuffer &s, BaseBuffer &r, unsigned count, reduceFunction f, unsigned comm,
                           bool from_fpga, bool to_fpga, dataType cd, bool async_) {
        return wrap(a, a.allreduce(s, r, count, f, comm, from_fpga, to_fpga, cd, async_));
      }, py::arg("sendbuf"), py::arg("recvbuf"), py::arg("count"), py::arg("func") = reduceFunction::SUM,
           py::arg("comm_id") = GLOBAL_COMM, py::arg("from_fpga") = false, py::arg("to_fpga") = false,
           py::arg("compress_dtype") = dataType::none, py::arg("run_async") = false, gil_release())
      .def("reduce_scatter", [](ACCL &a, BaseBuffer &s, BaseBuffer &r, unsigned count, reduceFunction f, unsigned comm,
                                bool from_fpga, bool to_fpga, dataType cd, bool async_) {
        return wrap(a, a.reduce_scatter(s, r, count, f, comm, from_fpga, to_fpga, cd, async_));
      }, py::arg("sendbuf"), py::arg("recvbuf"), py::arg("count"), py::arg("func") = reduceFunction::SUM,
           py::arg("comm_id") = GLOBAL_COMM, py::arg("from_fpga") = false, py::arg("to_fpga") = false,
           py::arg("compress_dtype") = dataType::none, py::arg("run_async") = false, gil_release())
      .def("alltoall", [](ACCL &a, BaseBuffer &s, BaseBuffer &r, unsigned count, unsigned comm, bool from_fpga, bool to_fpga,
                          dataType cd, bool async_) {
        return wrap(a, a.alltoall(s, r, count, comm, from_fpga, to_fpga, cd, async_));
      }, py::arg("sendbuf"), py::arg("recvbuf"), py::arg("count"), py::arg("comm_id") = GLOBAL_COMM,
           py::arg("from_fpga") = false, py::arg("to_fpga") = false, py::arg("compress_dtype") = dataType::none,
           py::arg("run_async") = false, gil_release())
      .def("alltoallv", [](ACCL &a, BaseBuffer &s, BaseBuffer &r, BaseBuffer &counts, unsigned comm, bool from_fpga, bool to_fpga,
                           bool async_) { return wrap(a, a.alltoallv(s, r, counts, comm, from_fpga, to_fpga, async_)); },
           py::arg("sendbuf"), py::arg("recvbuf"), py::arg("counts"), py::arg("comm_id") = GLOBAL_COMM,
           py::arg("from_fpga") = false, py::arg("to_fpga") = false, py::arg("run_async") = false, gil_release())
      .def("barrier", [](ACCL &a, unsigned comm) { a.free_request(a.barrier(comm)); }, py::arg("comm_id") = GLOBAL_COMM, gil_release())
      .def("create_communicator", &ACCL::create_communicator, py::arg("ranks"), py::arg("local_rank"))
      .def("get_comm_group", &ACCL::get_comm_group)
      .def("get_comm_rank", &ACCL::get_comm_rank)
      .def("get_communicator_addr", &ACCL::get_communicator_addr, py::arg("comm_id") = GLOBAL_COMM)
      .def("get_arithmetic_config_addr", [](ACCL &a, dataType u, dataType c) { return a.get_arithmetic_config_addr({u, c}); })
      .def("dump_communicator", &ACCL::dump_communicator)
      .def("dump_exchange_memory", &ACCL::dump_exchange_memory)
      .def("dump_eager_rx_buffers", &ACCL::dump_eager_rx_buffers, py::arg("dump_data") = false)
      .def("read_exchmem", [](ACCL &a, uint32_t off) { return a.device()->read(off); })
      .def_property_readonly("max_eager_size", &ACCL::max_eager_size)
      .def_property_readonly("max_rendezvous_size", &ACCL::max_rendezvous_size)
      // ---- emulator-only: device-side stream ports (the BFM of the reference)
      .def("emu_kernel_push", [](ACCL &a, py::bytes data) {
        std::string s = data;
        if (auto *rd = dynamic_cast<emu::RemoteDevice *>(a.device())) {
          py::gil_scoped_release rel;
          rd->kernel_push(s.data(), s.size());
          return;
        }
        auto *d = dynamic_cast<emu::EmuDevice *>(a.device());
        if (!d) throw std::runtime_error("not an emulator backend");
        d->engine().kernel_push(s.data(), s.size());
      })
      .def("emu_kernel_pull", [](ACCL &a, unsigned strm, size_t bytes, int timeout_ms) {
        auto *d = dynamic_cast<emu::EmuDevice *>(a.device());
        auto *rd = dynamic_cast<emu::RemoteDevice *>(a.device());
        if (!d && !rd) throw std::runtime_error("not an emulator backend");
        std::string out(bytes, '\0');
        bool ok;
        {
          py::gil_scoped_release rel;
          ok = rd ? rd->kernel_pull(strm, &out[0], bytes, timeout_ms) : d->engine().kernel_pull(strm, &out[0], bytes, timeout_ms);
        }
        if (!ok) throw std::runtime_error("emu_kernel_pull: timed out");
        return py::bytes(out);
      }, py::arg("stream_id"), py::arg("nbytes"), py::arg("timeout_ms") = 5000)
      .def("emu_set_kernel_loopback", [](ACCL &a, bool on) {
        if (auto *rd = dynamic_cast<emu::RemoteDevice *>(a.device())) {
          rd->set_kernel_loopback(on);
          return;
        }
        auto *d = dynamic_cast<emu::EmuDevice *>(a.device());
        if (!d) throw std::runtime_error("not an emulator backend");
        d->engine().set_kernel_loopback(on);
      })
      // device-issued call through the emulator's second command port
      .def("emu_device_call", [](ACCL &a, std::vector<uint32_t> words) {
        auto *d = dynamic_cast<emu::EmuDevice *>(a.device());
        if (!d) throw std::runtime_error("not an emulator backend");
        if (words.size() != 15 && words.size() != 16) throw std::invalid_argument("a call descriptor has 15 words");
        words.resize(16, 0);
        emu::EmuCall c;
        std::memcpy(&c.desc, words.data(), 64);
        c.client = 1;
        auto done = std::make_shared<std::promise<uint32_t>>();
        auto fut = done->get_future();
        c.on_done = [done](uint32_t rc) { done->set_value(rc); };
        d->engine().submit(std::move(c));
        py::gil_scoped_release rel;
        return fut.get();
      });

  // ---- backend factories
  m.def("make_emu_world", [](int world, size_t mem_mb) {
    std::vector<std::unique_ptr<ACCL>> out;
    for (auto &d : emu::make_inproc_world(world, mem_mb << 20)) out.emplace_back(new ACCL(std::move(d)));
    return out;
  }, py::arg("world_size"), py::arg("mem_mb") = 256);
  m.def("make_emu_socket", [](int rank, int world, const std::string &addr, int base_port, size_t mem_mb) {
    auto fabric = std::make_shared<emu::SocketFabric>(rank, world, addr, base_port);
    return std::unique_ptr<ACCL>(new ACCL(std::unique_ptr<CCLO>(new emu::EmuDevice(fabric, rank, world, mem_mb << 20))));
  }, py::arg("rank"), py::arg("world_size"), py::arg("addr") = "127.0.0.1", py::arg("base_port") = 5500,
        py::arg("mem_mb") = 256, gil_release());

  // driver side of a stand-alone engine process (build/bin/cclo_emu) listening on addr:ctrl_port
  m.def("make_emu_remote", [](int rank, int world, const std::string &addr, int ctrl_port, int connect_timeout_s) {
    return std::unique_ptr<ACCL>(
        new ACCL(std::unique_ptr<CCLO>(new emu::RemoteDevice(addr, ctrl_port, rank, world, connect_timeout_s))));
  }, py::arg("rank"), py::arg("world_size"), py::arg("addr") = "127.0.0.1", py::arg("ctrl_port") = 6500,
        py::arg("connect_timeout_s") = 60, gil_release());
  m.def("emu_remote_shutdown", [](ACCL &a) {
    auto *rd = dynamic_cast<emu::RemoteDevice *>(a.device());
    if (!rd) throw std::runtime_error("not a remote emulator backend");
    rd->shutdown_engine();
  }, gil_release());
  m.def("emu_debug_state", [](ACCL &a) {
    if (auto *rd = dynamic_cast<emu::RemoteDevice *>(a.device())) return rd->debug_state();
    auto *d = dynamic_cast<emu::EmuDevice *>(a.device());
    if (!d) throw std::runtime_error("not an emulator backend");
    return d->engine().debug_state();
  }, gil_release());
  m.def("emu_remote_debug_state", [](ACCL &a) {
    auto *rd = dynamic_cast<emu::RemoteDevice *>(a.device());
    if (!rd) throw std::runtime_error("not a remote emulator backend");
    return rd->debug_state();
  }, gil_release());

  // ---- rank tables
  m.def("generate_ranks", [](const std::vector<std::string> &ips, int base_port, addr_t rxbuf_size) {
    return generate_ranks(ips, base_port, rxbuf_size);
  }, py::arg("ips"), py::arg("base_port") = 5500, py::arg("rxbuf_size") = 1024);
  m.def("generate_ranks_from_file", [](const std::string &path, int base_port, addr_t rxbuf_size) {
    return generate_ranks(path, base_port, rxbuf_size);
  }, py::arg("config_file"), py::arg("base_port") = 5500, py::arg("rxbuf_size") = 1024);
  m.def("get_ips", [](const std::string &path) { return get_ips(path); });

  // ---- numerics helpers used by tests as the reference for narrow floats
  m.def("encode_float", [](float f, dataType t) -> uint32_t {
    switch (t) {
    case dataType::float16: return emu::F16::encode(f);
    case dataType::bfloat16: return emu::BF16::encode(f);
    case dataType::float8_e4m3: return emu::F8E4M3::encode(f);
    case dataType::float8_e5m2: return emu::F8E5M2::encode(f);
    default: throw std::invalid_argument("encode_float: not a narrow float type");
    }
  });
  m.def("decode_float", [](uint32_t u, dataType t) -> float {
    switch (t) {
    case dataType::float16: return emu::F16::decode(u);
    case dataType::bfloat16: return emu::BF16::decode(u);
    case dataType::float8_e4m3: return emu::F8E4M3::decode(u);
    case dataType::float8_e5m2: return emu::F8E5M2::decode(u);
    default: throw std::invalid_argument("decode_float: not a narrow float type");
    }
  });

#ifdef ACCL_WITH_CUDA
  accl::cuda::bind_cuda(m);
#endif
  m.attr("with_cuda") =
#ifdef ACCL_WITH_CUDA
      true;
#else
      false;
#endif
}
