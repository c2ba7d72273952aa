// All-gather -> GEMM plugin: the column-parallel half of a sequence-parallel tensor-parallel block (the row-parallel
// half is the GEMM -> reduce-scatter plugin, plugin_gemm_rs.cu).
//
// Each rank holds A_r, its [M/P, K] rows of the activations (bf16, in the symmetric heap at the same offset on every
// rank), and W_r [N_r, K], its output features (bf16, nn.Linear layout).  The op computes
//   C[M, N_r] = allgather_M(A_r) W_r^T        (bf16 out, fp32 accumulation)
// and leaves the gathered activations [M, K] in rank order, which backward passes reuse.  W_r may also be stored
// [K, N_r] (N contiguous, AgGemmArgs::w_kn): an nn.Linear weight used in its own backward pass,
// dX_r = allgather_M(dY_r) W_r.  It is loaded in 64-column boxes and fed to wgmma MN-major (k_plugin_ag_gemm<true>).
//
// One persistent, warp-specialised sm_90a kernel per rank, one CTA per 128 x 256 tile on every SM, with the 4-stage
// TMA -> mbarrier -> wgmma.m64n256k16 pipeline of the single-CTA GEMM -> reduce-scatter kernel (wgmma.cuh):
//   warpgroup 0, warp 0     TMA producer: A tiles of own rows from the local shard, A tiles of peer rows from
//                           `gathered` once their rows have arrived, W tiles from W
//   warpgroup 0, warps 1-3  PULL the peers' shards into `gathered` through the peer-mapped heap with 16-byte loads
//                           and stores, one 128-row chunk at a time in the order the tiles consume them (rank me+1
//                           first, then me+2, ...; own rows last, since no tile waits for them).  Every CTA copies its
//                           slice of a chunk and counts it in ready[row block]
//   warpgroups 1, 2         consumers: wgmma into registers, then bf16 -> 128B-swizzled smem -> TMA tensor store into C
// Tiles of own rows come first, so the tensor cores start at once; peer rows follow in pull order.  After the entry
// meeting every wait is on local memory.
// Meetings on the sync pads of channel MAX_CH-1: at entry CTA 0 exchanges the shard offsets with every peer (one lane
// per peer) and releases the copy warps of the grid; at exit the last CTA to finish meets the peers again, so no rank
// writes its shard on its stream before every peer has read it.
// The pipeline and the epilogue live in wgmma.cuh; the entry meeting, the grid release and the exit in kernels.cuh.
// This file keeps the pull, the tile order and its ready[] waits, and the host launch code.
#include <cuda.h>
#include <cuda_bf16.h>

#include <algorithm>

#include "accl/cuda/cudadevice.hpp"
#include "accl/cuda/driver_api.hpp"
#include "accl/cuda/launch.hpp"
#include "accl/cuda/plugins.hpp"
#include "accl/device/api.cuh"
#include "kernels.cuh"
#include "wgmma.cuh"

namespace accl {
namespace cuda {

namespace {
constexpr uint32_t AG_MAX_ROW_BLOCKS = 1024; // M / 128 of one call
// flag block (kernels.cuh, PluginFlag); own words: [AG_READY, AG_READY + M/128) ready[row block], the CTAs that have
// copied their slice of those 128 rows into `gathered`
constexpr uint32_t AG_READY = 64;
constexpr uint32_t AG_FLAG_WORDS = AG_READY + AG_MAX_ROW_BLOCKS;
constexpr int COPY_THREADS = 96; // warps 1-3
} // namespace

struct AgGemmParams {
  DevWorld w;
  uint64_t a_off;
  char *gathered;
  uint32_t m, n, k;
  uint32_t timeout_us;
  unsigned int *flags;
  uint32_t *status;
};

// this thread's share of one chunk: 16-byte vectors i, i + stride, ...; four loads in flight before their stores
__device__ __forceinline__ void copy_slice(const char *src, char *dst, size_t nvec, size_t i, size_t stride) {
  for (; i + 3 * stride < nvec; i += 4 * stride) {
    const dev::Vec16 v0 = dev::ld_volatile16(src + i * 16);
    const dev::Vec16 v1 = dev::ld_volatile16(src + (i + stride) * 16);
    const dev::Vec16 v2 = dev::ld_volatile16(src + (i + 2 * stride) * 16);
    const dev::Vec16 v3 = dev::ld_volatile16(src + (i + 3 * stride) * 16);
    dev::st_stream(dst + i * 16, v0);
    dev::st_stream(dst + (i + stride) * 16, v1);
    dev::st_stream(dst + (i + 2 * stride) * 16, v2);
    dev::st_stream(dst + (i + 3 * stride) * 16, v3);
  }
  for (; i < nvec; i += stride) dev::st_stream(dst + i * 16, dev::ld_volatile16(src + i * 16));
}

template <bool KN>
__global__ void __launch_bounds__(g::THREADS, 1)
k_plugin_ag_gemm(const __grid_constant__ CUtensorMap tmap_own, const __grid_constant__ CUtensorMap tmap_gathered,
                 const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_c, AgGemmParams p) {
  using namespace g;
  constexpr int GROUP_M = 16;
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint32_t s_err, s_readable, s_last;
  __shared__ WorkItem s_item; // identity communicator for the sync pads

  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const uint32_t P = p.w.world, me = p.w.rank, G = gridDim.x;
  const uint32_t tiles_m = p.m / BM, tiles_n = p.n / BN, num_tiles = tiles_m * tiles_n;
  const uint32_t k_blocks = p.k / BK;
  const uint32_t blocks_per_rank = tiles_m / P; // 128-row chunks of one shard
  char *my_heap = p.w.window + static_cast<uint64_t>(me) * p.w.heap_bytes;
  unsigned int *ready = p.flags + AG_READY;

  // ---------------- one-time setup
  const Smem sm = gemm_smem<false>(smem_raw);
  if (threadIdx.x == 0) {
    s_err = 0;
    k::plugin_item(s_item, p.w, 0x41, 0x414747u, p.timeout_us); // 'A'
  }
  if (warp == 0 && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap_own)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap_gathered)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap_w)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap_c)) : "memory");
  }
  __syncthreads();

  k::Ctx ctx{p.w, s_item, MAX_CH - 1, 1, reinterpret_cast<Ctrl *>(my_heap), &s_err, static_cast<uint64_t>(p.timeout_us) * 1000ull, nullptr};

  if (warp >= 1 && warp <= 3) {
    // ===== pull the shards into `gathered`
    if (blockIdx.x == 0 && warp == 1) {
      // entry meeting with every peer, one lane each: exchange the shard offsets.  A peer that does not answer, is in
      // another operation or has its shard elsewhere is not read.
      const uint32_t mask = k::meet_peers(ctx, k::REC_OFF0, p.a_off, 0);
      if (lane == 0) k::release_grid(p.flags, mask); // release the copy warps of every CTA
    }
    const uint32_t ct = threadIdx.x - 32;
    if (ct == 0) s_readable = k::wait_grid(p.flags, ctx);
    asm volatile("bar.sync 1, 96;" ::: "memory"); // warps 1-3 only
    const uint32_t readable = s_readable;
    const size_t chunk_bytes = static_cast<size_t>(BM) * p.k * 2;
    const size_t nvec = chunk_bytes / 16;
    const size_t first = static_cast<size_t>(blockIdx.x) * COPY_THREADS + ct, stride = static_cast<size_t>(G) * COPY_THREADS;
    for (uint32_t dq = 1; dq <= P; ++dq) {
      const uint32_t q = (me + dq) % P; // pull order; dq == P: own rows
      const char *src = p.w.window + static_cast<uint64_t>(q) * p.w.heap_bytes + p.a_off;
      for (uint32_t j = 0; j < blocks_per_rank; ++j) {
        const uint32_t rb = q * blocks_per_rank + j; // row block of `gathered`
        // a shard that may not be read is skipped: its chunks are counted all the same, so nothing waits for them
        if ((readable >> q) & 1u) copy_slice(src + j * chunk_bytes, p.gathered + rb * chunk_bytes, nvec, first, stride);
        asm volatile("fence.proxy.async.global;" ::: "memory"); // the TMA unit reads these rows
        __threadfence();
        asm volatile("bar.sync 1, 96;" ::: "memory");
        if (ct == 0) asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(&ready[rb]) : "memory");
      }
    }
  } else if (warp == 0) {
    // ===== TMA producer
    uint32_t stage = 0, phase = 0;
    bool waiting = true; // false after a timed-out chunk: the chunks still missing are skipped
    for (uint32_t t = blockIdx.x; t < num_tiles; t += G) {
      uint32_t mo, nb;
      tile_coords<GROUP_M>(t, tiles_m, tiles_n, mo, nb);
      const bool own = mo < blocks_per_rank;
      const uint32_t mb = (mo + me * blocks_per_rank) % tiles_m; // own rows first, then the peers' in pull order
      if (lane == 0 && !own && waiting) {
        waiting = k::wait_ge(&ready[mb], G, ctx, RECEIVE_TIMEOUT_ERROR); // every CTA has copied its slice
        asm volatile("fence.proxy.async.global;" ::: "memory");
      }
      __syncwarp();
      produce_tile<false, KN>(sm, own ? &tmap_own : &tmap_gathered, static_cast<int>((own ? mo : mb) * BM), &tmap_w, nb, k_blocks, 0,
                              stage, phase, lane);
    }
  } else {
    // ===== consumers: wgmma into registers, then registers -> bf16 -> swizzled smem -> TMA store into C
    const uint32_t wg = warp / 4 - 1; // rows [64 wg, 64 wg + 64) of the CTA's 128
    const uint32_t wi = warp % 4;     // this warp's 16 of them
    uint8_t *my_epi = sm.epi + (warp - 4) * 2 * EPI_BUF_BYTES;
    uint32_t stage = 0, phase = 0, ebuf = 0;
    float d[128];
#pragma unroll
    for (int i = 0; i < 128; ++i) d[i] = 0.f;
    for (uint32_t t = blockIdx.x; t < num_tiles; t += G) {
      uint32_t mo, nb;
      tile_coords<GROUP_M>(t, tiles_m, tiles_n, mo, nb);
      const uint32_t mb = (mo + me * blocks_per_rank) % tiles_m;
      consume_tile<false, KN>(sm, d, wg, k_blocks, 0, stage, phase);
      const uint32_t row0 = mb * BM + wg * 64 + wi * EPI_ROWS; // first of this warp's 16 rows of C
      epilogue_tile<false, false>(d, my_epi, ebuf, lane, &tmap_c, static_cast<int>(nb * BN), static_cast<int>(row0));
    }
    if (lane == 0) device::emit_flush(); // all my stores have been written
    __syncwarp();
  }

  // ---------------- teardown: a CTA has finished once its copies and its tiles are done; the last one meets the peers
  // (every CTA of this rank has read what it needed of the peers' shards: when all ranks meet there, each may
  // overwrite its shard)
  k::plugin_exit(ctx, p.flags, p.status, true, s_last);
}

// ----------------------------------------------------------------------- host
void preload_ag_gemm_kernels() {
  cudaFuncAttributes a;
  cudaFuncGetAttributes(&a, k_plugin_ag_gemm<false>);
  cudaFuncGetAttributes(&a, k_plugin_ag_gemm<true>);
  cudaFuncSetAttribute(k_plugin_ag_gemm<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, g::SMEM_BYTES);
  cudaFuncSetAttribute(k_plugin_ag_gemm<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, g::SMEM_BYTES);
}

cudaError_t launch_ag_gemm(CudaDevice &dev, const AgGemmArgs &a, cudaStream_t stream) {
  using namespace g;
  const DevWorld &w = dev.world();
  const uint32_t P = w.world;
  if (!a.m || !a.n || !a.k || a.m % (BM * P) || a.n % BN || a.k % BK)
    throw std::invalid_argument("ag_gemm: need M % (128*world) == 0, N % 256 == 0, K % 64 == 0, none of them zero");
  if (a.m / BM > AG_MAX_ROW_BLOCKS) throw std::invalid_argument("ag_gemm: M / 128 is above 1024");
  auto aligned = [](const void *ptr) { return ptr && reinterpret_cast<uintptr_t>(ptr) % 16 == 0; };
  if (a.a_off % 16 || !aligned(a.w) || !aligned(a.gathered) || !aligned(a.out))
    throw std::invalid_argument("ag_gemm: the shard offset and the w, gathered and out pointers must be 16-byte aligned");
  if (a.a_off + static_cast<uint64_t>(a.m / P) * a.k * 2 > w.heap_bytes)
    throw std::invalid_argument("ag_gemm: the shard does not fit in the symmetric heap at that offset");
  ACCL_CUDART(cudaSetDevice(dev.device()));
  const CUtensorMap t_own = make_map(w.window + static_cast<uint64_t>(w.rank) * w.heap_bytes + a.a_off, a.m / P, a.k, BM, BK);
  const CUtensorMap t_gathered = make_map(a.gathered, a.m, a.k, BM, BK);
  const CUtensorMap t_w = a.w_kn ? make_map(a.w, a.k, a.n, BK, 64) : make_map(a.w, a.n, a.k, BN, BK);
  const CUtensorMap t_c = make_map(a.out, a.m, a.n, EPI_ROWS, 64);
  AgGemmParams p;
  p.w = w;
  p.a_off = a.a_off;
  p.gathered = static_cast<char *>(a.gathered);
  p.m = a.m;
  p.n = a.n;
  p.k = a.k;
  p.timeout_us = dev.timeout_us();
  p.flags = plugin_flags(dev, 'A', AG_FLAG_WORDS, stream);
  p.status = a.status_dev;
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev.device());
  const uint32_t tiles = (a.m / BM) * (a.n / BN);
  const auto kernel = a.w_kn ? k_plugin_ag_gemm<true> : k_plugin_ag_gemm<false>;
  cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
  cudaLaunchConfig_t lc = {};
  // every CTA copies a slice of every chunk and waits for the others' slices: the whole grid must be resident, one CTA per SM
  lc.gridDim = dim3(std::min<uint32_t>(static_cast<uint32_t>(sms), tiles));
  lc.blockDim = dim3(THREADS);
  lc.dynamicSmemBytes = SMEM_BYTES;
  lc.stream = stream;
  return cudaLaunchKernelEx(&lc, kernel, t_own, t_gathered, t_w, t_c, p);
}

} // namespace cuda
} // namespace accl
