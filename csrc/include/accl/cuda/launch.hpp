// Host-callable entry points of the CUDA translation units (kernel launches).
#pragma once
#include <cuda_runtime.h>

#include "accl/cuda/devtypes.hpp"

namespace accl {
namespace cuda {

// host-visible mirror of a finished call (pinned, written by the last CTA)
// One 16-byte record, written by the device with a single vector store (one PCIe write): no
// system-scope fence on the kernel's critical path.
struct alignas(16) HostCompletion {
  volatile uint32_t seq;      // request sequence the record belongs to
  volatile uint32_t retcode;
  volatile unsigned long long duration_ns; // %globaltimer: last CTA out - first CTA in
};

// one call, one kernel: `item.n_ctas` CTAs cooperate, completion goes to hc (device-visible pinned pointer)
cudaError_t launch_call(const DevWorld &w, const WorkItem &item, HostCompletion *hc_dev, cudaStream_t stream);

// Force-load every kernel of the library now.  With CUDA's lazy module loading the first
// launch of a kernel may synchronise the context, which deadlocks against a resident
// persistent engine (or a peer rank's spinning kernel on the same GPU).
void preload_engine_kernels();
void preload_gemm_rs_kernels();
void preload_ag_gemm_kernels();
void preload_vadd_kernels();
void preload_ar_rmsnorm_kernels();

class CudaDevice;
// The flag block of fused plugin `plugin` on `dev` (layout: PluginFlag, kernels.cuh): `words` uint32 words of device
// memory, allocated at the first call and zeroed on `stream` at every call, so each launch finds it zeroed and the
// launch can be captured in a CUDA graph.  Each plugin passes its own tag and the same `words` every time.
unsigned int *plugin_flags(CudaDevice &dev, char plugin, uint32_t words, cudaStream_t stream);

// Device-side stream port (the user-kernel <-> engine AXI streams of the reference): a byte
// FIFO in the heap.  pop: FIFO -> dst (local heap offset); push: src -> FIFO of rank `dst_rank`.
cudaError_t launch_stream_pop(const DevWorld &w, uint64_t dst_off, uint64_t bytes, uint32_t stream_id, uint32_t timeout_us,
                              cudaStream_t stream);
cudaError_t launch_stream_push(const DevWorld &w, uint32_t dst_rank, uint64_t src_off, uint64_t bytes, uint32_t stream_id,
                               uint32_t timeout_us, cudaStream_t stream);

// zero the protocol state of my control block (soft reset)
cudaError_t launch_reset_ctrl(const DevWorld &w, cudaStream_t stream);

} // namespace cuda
} // namespace accl
