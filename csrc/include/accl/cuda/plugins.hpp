// Device-API plugins: compute kernels that talk to the collective machinery
// themselves (the reference's kernels/plugins/vadd_put pattern, plus the
// north-star wgmma GEMM whose epilogue feeds a reduce-scatter, and the wgmma GEMM fed by an all-gather).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "accl/cuda/devtypes.hpp"

namespace accl {
namespace cuda {

class CudaDevice;

struct GemmRsArgs {
  const void *a;     // [M, K] bf16 row-major (this rank's K-slice of the activations)
  const void *w;     // [N, K] bf16 row-major (this rank's K-slice of the weight, nn.Linear layout), or [K, N] with w_kn
  uint64_t out_off;  // heap offset of this rank's [M / P, N] output shard (bf16, or fp32 with out_f32)
  uint32_t m, n, k;
  int variant = 0;   // 0: automatic, 1: one CTA per 128 x 256 tile, 2: CTA pair (cluster of 2, W tile multicast) per 256 x 256 tile
  bool out_f32 = false; // shard is fp32: the P partial products are added without intermediate rounding
  uint32_t *status_dev = nullptr; // device word that receives the error bits (0: success) when the kernel ends; may be null
  bool w_kn = false; // w is [K, N] (N contiguous), e.g. an nn.Linear weight in its own backward pass: C = A * W
};

// C = A * W^T (A * W with w_kn) computed tile by tile on the tensor cores (TMA -> smem ->
// wgmma -> register accumulators); every finished accumulator tile is converted
// to bf16, staged in shared memory and added straight into its owner rank's
// output shard over NVLink by the TMA unit (cp.reduce.async.bulk.tensor .add on
// the peer-mapped heap): reduce-scatter along M with no intermediate buffer
// and no separate collective.  The shard must sit at out_off on every rank: no tile is added into a peer whose
// shard is elsewhere, and the call reports DMA_MISMATCH_ERROR.  With non-zero status bits the shard is not a valid
// result.  Returns after enqueueing.
cudaError_t launch_gemm_rs(CudaDevice &dev, const GemmRsArgs &args, cudaStream_t stream);

// most 128 x 256 tiles of one GEMM -> all-reduce call: the size of its counter block, in uint32 words
constexpr uint32_t GEMM_AR_MAX_TILES = 16384;

struct GemmArArgs {
  const void *a;     // [M, K] bf16 row-major (this rank's K-slice of the activations)
  const void *w;     // [N, K] bf16 row-major (this rank's K-slice of the weight, nn.Linear layout), or [K, N] with w_kn
  uint64_t out_off;  // heap offset of the full [M, N] result (bf16, or fp32 with out_f32), the same on every rank
  uint64_t cnt_off;  // heap offset of GEMM_AR_MAX_TILES uint32 arrival counters, the same on every rank
  uint32_t m, n, k;
  int variant = 0;   // 0: automatic, 1: one CTA per 128 x 256 tile, 2: CTA pair per 256 x 256 tile (M % 256 == 0)
  bool out_f32 = false; // C is fp32: the P partial products are added without intermediate rounding
  uint32_t *status_dev = nullptr; // device word that receives the error bits (0: success) when the kernel ends; may be null
  bool w_kn = false; // w is [K, N] (N contiguous): C = sum_r A_r W_r
};

// C = sum over ranks of A_r * W_r^T (A_r * W_r with w_kn), the same bits in every rank's heap at out_off: the GEMM ->
// reduce-scatter kernel with a two-shot all-reduce epilogue.  Every tile has one owner rank; each rank adds its
// partial tile into the owner's C (TMA reduce-add over NVLink) and signals a per-tile counter in the owner's heap, and
// the owner copies each complete tile into every peer's C.  C and the counter block must sit at the same offsets on
// every rank: a peer where either differs gets no adds and no copies, and the call reports DMA_MISMATCH_ERROR.  With
// non-zero status bits C is not a valid result.  Throws std::invalid_argument before enqueueing anything unless
// M % 128 == 0 (256 for the CTA pair), N % 256 == 0, K % 64 == 0, (M / 128) (N / 256) <= GEMM_AR_MAX_TILES and both
// regions are 16-byte aligned inside the heap.  Returns after enqueueing.
cudaError_t launch_gemm_ar(CudaDevice &dev, const GemmArArgs &args, cudaStream_t stream);

struct AgGemmArgs {
  uint64_t a_off;        // heap offset of this rank's [M / P, K] bf16 shard of the activations (the same on every rank)
  const void *w;         // [N, K] bf16 row-major (this rank's output features, nn.Linear layout), or [K, N] with w_kn
  void *gathered;        // [M, K] bf16: receives every rank's shard in rank order
  void *out;             // [M, N] bf16
  uint32_t m, n, k;
  uint32_t *status_dev;  // device word that receives the error bits (0: success) when the kernel ends; may be null
  bool w_kn = false;     // w is [K, N] (N contiguous), e.g. an nn.Linear weight in its own backward pass: C = A * W
};

// C = allgather_M(A_shard) * W^T (* W with w_kn): the first half of a sequence-parallel column-parallel linear layer.  One
// persistent wgmma kernel computes the tiles of this rank's own rows first while spare warps pull the peers'
// shards over NVLink into `gathered`, 128 rows at a time and in the order the tiles consume them; a tile of peer rows
// waits only for its own 128 rows.  Throws std::invalid_argument before enqueueing anything unless
// M % (128 * P) == 0, N % 256 == 0, K % 64 == 0, M / 128 <= 1024 and every pointer and a_off are 16-byte aligned.
// Returns after enqueueing.
cudaError_t launch_ag_gemm(CudaDevice &dev, const AgGemmArgs &args, cudaStream_t stream);

// widest row of one all-reduce -> RMSNorm call, in elements
constexpr uint32_t AR_MAX_H = 16384;

struct ArRmsNormArgs {
  uint64_t x_off;         // heap offset of this rank's [M, H] bf16 partial sums (the same on every rank); only read
  const void *residual;   // [M, H] bf16, the same values on every rank, or null; may be residual_out itself
  const void *gamma;      // [H] bf16 RMSNorm gain
  uint64_t h_off;         // heap offset of residual_out [M, H] bf16 (the same on every rank)
  void *out;              // [M, H] bf16
  uint32_t m, h;
  float eps;
  uint32_t *status_dev;   // device word that receives the error bits (0: success) when the kernel ends; may be null
};

// residual_out = bf16(sum over ranks of x_r, in rank order, + residual) and out = RMSNorm(residual_out) * gamma, in
// one kernel: the all-reduce result is normalised while it is still in registers.  One-shot (every rank pulls every
// row) while M H 2 P <= CudaConfig::oneshot_max_bytes, else two-shot (each rank reduces its M / P rows, pushes them
// into every peer's residual_out, and every rank normalises all rows); both forms give the same bits.  x and
// residual_out must sit at the same offsets on every rank: a peer where either differs is neither read nor written,
// and the call reports DMA_MISMATCH_ERROR.  Throws std::invalid_argument before enqueueing anything unless M >= 1,
// H % 8 == 0, 8 <= H <= AR_MAX_H, eps is finite and >= 0, both heap regions are 16-byte aligned inside the heap and
// do not overlap, every pointer is 16-byte aligned and residual is residual_out or does not overlap it.  Returns
// after enqueueing.
cudaError_t launch_ar_rmsnorm(CudaDevice &dev, const ArRmsNormArgs &args, cudaStream_t stream);

// vector add whose result feeds an all-reduce issued by the kernel itself through the device API (engine must be
// enabled): out = allreduce_sum(x + y).  The vector is produced in chunks of `chunk_elems` (0: 1 Mi elements); each
// finished chunk is handed to the engine at once (all_reduce_async) while the kernel computes the next one.
cudaError_t launch_vadd_allreduce(CudaDevice &dev, uint64_t x_off, uint64_t y_off, uint64_t tmp_off, uint64_t out_off,
                                  uint32_t count, uint32_t chunk_elems, uint32_t comm_adr, uint32_t dpcfg_adr, uint32_t *status_dev,
                                  cudaStream_t stream);

// the reference's vadd_put: src + 1 is pushed tile by tile into stream `stream_id` of rank `dst_rank` while computing
cudaError_t launch_vadd_put(CudaDevice &dev, uint64_t src_off, uint32_t count, uint32_t dst_rank, uint32_t stream_id,
                            uint32_t *status_dev, cudaStream_t stream);
// consumer of a stream: `count` fp32 of stream `stream_id` -> heap offset dst_off
cudaError_t launch_stream_pull(CudaDevice &dev, uint64_t dst_off, uint32_t count, uint32_t stream_id, uint32_t *status_dev,
                               cudaStream_t stream);

// user kernel in the stream path: pulls `count` fp32 from this rank's stream FIFO, optionally adds one,
// pushes them back (reference kernels/plugins/loopback).  scratch_off: heap scratch of count * 4 bytes.
cudaError_t launch_loopback(CudaDevice &dev, uint64_t scratch_off, uint32_t count, bool add_one, uint32_t *status_dev,
                            cudaStream_t stream);

} // namespace cuda
} // namespace accl
