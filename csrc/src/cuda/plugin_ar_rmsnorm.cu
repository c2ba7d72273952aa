// All-reduce -> residual add -> RMSNorm plugin: the step that ends every row-parallel matmul of a transformer block
// whose activations are replicated on every rank.
//
// Each rank holds x_r [M, H], its unreduced partial sums (bf16, in the symmetric heap at the same offset on every
// rank), the replicated residual [M, H] and the RMSNorm gain [H].  Per element and per row:
//   acc = x_0 + x_1 + ... + x_{P-1} (+ residual)      fp32, ranks added in rank order
//   h   = bf16_rn(acc)                                 -> residual_out (heap, same offset on every rank)
//   y   = bf16_rn((h * rsqrt(mean(h^2) + eps)) * w)    -> out
// so the reduced rows are normalised while they are still in registers, in one kernel instead of an all-reduce, an
// add and a norm.  A row of up to AR_MAX_H elements is held by one CTA, AR_VPT 16-byte vectors per thread.
//
// Two forms of one kernel, chosen on the host by the all-reduce rule of plan.hpp (CudaConfig::oneshot_max_bytes):
//   one-shot (M H 2 P <= oneshot_max_bytes)  every rank pulls every row of every peer's x and computes all M rows.
//                 The last CTA to finish meets the peers again, so no rank rewrites its x while a peer reads it.
//   two-shot      rank o owns rows [o M / P, (o + 1) M / P).  Phase 1: the owner pulls its rows from every peer, adds
//                 its own copy of the residual, and writes h into its own and every peer's residual_out.  A grid
//                 barrier and a meeting with the peers follow.  Phase 2: every rank normalises all M rows of its local
//                 residual_out.  After the middle meeting nobody reads this rank's x or writes its heap, so no exit
//                 meeting is needed.  Each rank moves 2 (P - 1) / P of the rows over NVLink instead of (P - 1).
// Both forms round h once and run the same norm code (norm_row) on the same bf16 h: their results are bit-identical.
// World 1 always takes the one-shot body: a local fused residual add + RMSNorm with no meeting.
//
// Meetings on the sync pads of channel MAX_CH-1, bank 0, one lane per peer as in the GEMM plugins, with the kind
// word 'N' / "ARN": the entry meeting exchanges the offsets of x and residual_out.  A peer in another plugin reports
// PACK_SEQ_NUMBER_ERROR; a peer where either offset differs is neither read nor written, and both report
// DMA_MISMATCH_ERROR.  The result is released to the grid through flags in device memory zeroed before the launch.
// The identity communicator, the grid release, the exit and the flag layout are the other fused plugins' (kernels.cuh).
#include <cuda_bf16.h>

#include <algorithm>
#include <cmath>

#include "accl/cuda/cudadevice.hpp"
#include "accl/cuda/driver_api.hpp"
#include "accl/cuda/launch.hpp"
#include "accl/cuda/plugins.hpp"
#include "kernels.cuh"

namespace accl {
namespace cuda {

namespace {
constexpr int AR_THREADS = 512;
constexpr int AR_VPT = AR_MAX_H / 8 / AR_THREADS; // 16-byte vectors of a row per thread
static_assert(AR_VPT * 8 * AR_THREADS == static_cast<int>(AR_MAX_H), "a row of AR_MAX_H elements fills the block");
// flag block (kernels.cuh, PluginFlag); own words of the two-shot form: CTAs done with phase 1, and the middle release
constexpr uint32_t AR_PHASE1 = k::FLAG_PLUGIN, AR_MIDDLE = AR_PHASE1 + 1, AR_FLAG_WORDS = AR_MIDDLE + 1;
} // namespace

struct ArRmsNormParams {
  DevWorld w;
  uint64_t x_off, h_off;
  const __nv_bfloat16 *residual; // null: no residual; may be residual_out itself
  const __nv_bfloat16 *gamma;
  __nv_bfloat16 *out;
  uint32_t m, h;
  float eps;
  uint32_t timeout_us;
  uint32_t two_shot;
  unsigned int *flags;
  uint32_t *status;
};

__device__ __forceinline__ float bf_lo(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf_hi(uint32_t v) { return __uint_as_float(v & 0xFFFF0000u); }
__device__ __forceinline__ uint32_t pack_bf2(float lo, float hi) {
  const __nv_bfloat162 b = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<const uint32_t *>(&b);
}
__device__ __forceinline__ void add_vec(float (&a)[8], const dev::Vec16 &v) {
  const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    a[2 * i] += bf_lo(u[i]);
    a[2 * i + 1] += bf_hi(u[i]);
  }
}

// h = bf16_rn(sum over the ranks in `ok`, in rank order, of their x row, + residual row) for this thread's vectors
// v = threadIdx.x + k AR_THREADS < nvec.  Peer rows are read with strong 16-byte loads, two ranks' vectors in flight.
__device__ __forceinline__ void reduce_row(const ArRmsNormParams &p, uint32_t ok, uint64_t row, uint32_t nvec,
                                           dev::Vec16 (&hv)[AR_VPT]) {
  const uint32_t P = p.w.world;
  const uint64_t row_off = p.x_off + row * p.h * 2;
  float acc[AR_VPT][8];
#pragma unroll
  for (int k = 0; k < AR_VPT; ++k)
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[k][i] = 0.f;
  for (uint32_t q = 0; q < P; q += 2) {
    const bool has0 = (ok >> q) & 1u, has1 = q + 1 < P && ((ok >> (q + 1)) & 1u);
    const char *s0 = p.w.window + static_cast<uint64_t>(q) * p.w.heap_bytes + row_off;
    const char *s1 = s0 + p.w.heap_bytes;
    dev::Vec16 a[AR_VPT], b[AR_VPT];
#pragma unroll
    for (int k = 0; k < AR_VPT; ++k) {
      const uint32_t v = threadIdx.x + k * AR_THREADS;
      if (v < nvec && has0) a[k] = dev::ld_volatile16(s0 + v * 16);
      if (v < nvec && has1) b[k] = dev::ld_volatile16(s1 + v * 16);
    }
#pragma unroll
    for (int k = 0; k < AR_VPT; ++k) {
      const uint32_t v = threadIdx.x + k * AR_THREADS;
      if (v < nvec && has0) add_vec(acc[k], a[k]);
      if (v < nvec && has1) add_vec(acc[k], b[k]);
    }
  }
  if (p.residual) {
    const char *r = reinterpret_cast<const char *>(p.residual) + row * p.h * 2;
#pragma unroll
    for (int k = 0; k < AR_VPT; ++k) {
      const uint32_t v = threadIdx.x + k * AR_THREADS;
      if (v < nvec) add_vec(acc[k], dev::ld_volatile16(r + v * 16)); // (may be this rank's residual_out: coherent)
    }
  }
#pragma unroll
  for (int k = 0; k < AR_VPT; ++k)
    hv[k] = dev::Vec16{pack_bf2(acc[k][0], acc[k][1]), pack_bf2(acc[k][2], acc[k][3]), pack_bf2(acc[k][4], acc[k][5]),
                       pack_bf2(acc[k][6], acc[k][7])};
}

// y = bf16_rn((h rstd) w), rstd = rsqrt(sum(h^2) / H + eps), for one row held by the block.  The sum runs over a fixed
// tree (each thread's vectors in order, a warp butterfly, the warps in order), so both forms and every rank compute
// the same bits from the same h.  Every thread of the block must call it.
__device__ __forceinline__ void norm_row(const ArRmsNormParams &p, uint64_t row, uint32_t nvec, const dev::Vec16 (&hv)[AR_VPT],
                                         float *s_red) {
  float ss = 0.f;
#pragma unroll
  for (int k = 0; k < AR_VPT; ++k) {
    if (threadIdx.x + k * AR_THREADS < nvec) {
      const uint32_t u[4] = {hv[k].x, hv[k].y, hv[k].z, hv[k].w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        ss = fmaf(bf_lo(u[i]), bf_lo(u[i]), ss);
        ss = fmaf(bf_hi(u[i]), bf_hi(u[i]), ss);
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  __syncthreads(); // the previous row's readers of s_red are done
  if (threadIdx.x % 32 == 0) s_red[threadIdx.x / 32] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int i = 0; i < AR_THREADS / 32; ++i) tot += s_red[i];
  const float rstd = rsqrtf(__fadd_rn(__fdiv_rn(tot, static_cast<float>(p.h)), p.eps));
  const char *gam = reinterpret_cast<const char *>(p.gamma);
  char *dst = reinterpret_cast<char *>(p.out) + row * p.h * 2;
#pragma unroll
  for (int k = 0; k < AR_VPT; ++k) {
    const uint32_t v = threadIdx.x + k * AR_THREADS;
    if (v < nvec) {
      const dev::Vec16 g = *reinterpret_cast<const dev::Vec16 *>(gam + v * 16);
      const uint32_t u[4] = {hv[k].x, hv[k].y, hv[k].z, hv[k].w}, gu[4] = {g.x, g.y, g.z, g.w};
      uint32_t y[4];
#pragma unroll
      for (int i = 0; i < 4; ++i)
        y[i] = pack_bf2(__fmul_rn(__fmul_rn(bf_lo(u[i]), rstd), bf_lo(gu[i])), __fmul_rn(__fmul_rn(bf_hi(u[i]), rstd), bf_hi(gu[i])));
      dev::st_stream(dst + v * 16, dev::Vec16{y[0], y[1], y[2], y[3]});
    }
  }
}

// wait for a grid release flag; on timeout the error bit is set and the caller goes on
__device__ __forceinline__ void wait_release(unsigned int *flag, const k::Ctx &ctx) {
  if (threadIdx.x == 0) k::wait_ge(flag, 1u, ctx, RECEIVE_TIMEOUT_ERROR);
  __syncthreads();
}

__global__ void __launch_bounds__(AR_THREADS, 1) k_plugin_ar_rmsnorm(ArRmsNormParams p) {
  __shared__ uint32_t s_err, s_ok, s_last;
  __shared__ float s_red[AR_THREADS / 32];
  __shared__ WorkItem s_item; // identity communicator for the sync pads

  const uint32_t P = p.w.world, me = p.w.rank, G = gridDim.x;
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const uint32_t nvec = p.h / 8;
  char *my_heap = p.w.window + static_cast<uint64_t>(me) * p.w.heap_bytes;

  if (threadIdx.x == 0) {
    s_err = 0;
    k::plugin_item(s_item, p.w, 0x4E, 0x41524Eu, p.timeout_us); // 'N' (the GEMM plugins use 'A', 'G' and 'R')
  }
  __syncthreads();
  k::Ctx ctx{p.w, s_item, MAX_CH - 1, 1, reinterpret_cast<Ctrl *>(my_heap), &s_err, static_cast<uint64_t>(p.timeout_us) * 1000ull, nullptr};

  // ---------------- entry meeting (CTA 0, one lane per peer): x and residual_out must sit at the same offsets.  It does
  // what k::meet_peers and k::wait_grid do, written out: with those helpers ptxas schedules the reduce and norm loops
  // differently (120 registers instead of 119) and calls of 2048-8192 rows ran 3-9% slower on an H100 (700 W).
  if (P > 1 && blockIdx.x == 0 && warp == 0) {
    bool ok = static_cast<uint32_t>(lane) == me;
    if (static_cast<uint32_t>(lane) < P && static_cast<uint32_t>(lane) != me) {
      k::pad_post(ctx, MAX_CH - 1, lane, k::REC_OFFS, p.x_off, p.h_off, ctx.kind_word());
      if (k::pad_wait(ctx, MAX_CH - 1, lane)) {
        const SyncRec r = k::pad_rec(ctx, MAX_CH - 1, lane, k::REC_OFFS);
        if (r.kind != ctx.kind_word()) {
          atomicOr(&s_err, PACK_SEQ_NUMBER_ERROR);
        } else if (r.off0 != p.x_off || r.off2 != p.h_off) {
          atomicOr(&s_err, DMA_MISMATCH_ERROR);
        } else {
          ok = true;
        }
      }
    }
    const uint32_t mask = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) k::release_grid(p.flags, mask); // no CTA touches a peer before this release
  }
  if (P > 1) {
    wait_release(&p.flags[k::FLAG_RELEASE], ctx);
    if (threadIdx.x == 0) s_ok = *reinterpret_cast<volatile unsigned int *>(&p.flags[k::FLAG_MASK]) | (1u << me);
  } else if (threadIdx.x == 0) {
    s_ok = 1u;
  }
  __syncthreads();
  const uint32_t ok = s_ok;

  dev::Vec16 hv[AR_VPT];
  if (!p.two_shot) {
    // ===== one-shot: every rank reduces and normalises every row
    for (uint64_t row = blockIdx.x; row < p.m; row += G) {
      reduce_row(p, ok, row, nvec, hv);
      char *hrow = my_heap + p.h_off + row * p.h * 2;
#pragma unroll
      for (int k = 0; k < AR_VPT; ++k) {
        const uint32_t v = threadIdx.x + k * AR_THREADS;
        if (v < nvec) dev::st_stream(hrow + v * 16, hv[k]);
      }
      norm_row(p, row, nvec, hv, s_red);
    }
  } else {
    // ===== two-shot, phase 1: reduce the rows this rank owns and push h into every peer's residual_out
    const uint64_t lo = static_cast<uint64_t>(me) * p.m / P, hi = static_cast<uint64_t>(me + 1) * p.m / P;
    for (uint64_t row = lo + blockIdx.x; row < hi; row += G) {
      reduce_row(p, ok, row, nvec, hv);
      const uint64_t hrow = p.h_off + row * p.h * 2;
      for (uint32_t q = 0; q < P; ++q) {
        if (!((ok >> q) & 1u)) continue;
        char *dst = p.w.window + static_cast<uint64_t>(q) * p.w.heap_bytes + hrow;
#pragma unroll
        for (int k = 0; k < AR_VPT; ++k) {
          const uint32_t v = threadIdx.x + k * AR_THREADS;
          if (v < nvec) dev::st_stream(dst + v * 16, hv[k]);
        }
      }
    }
    // every CTA's pushes are performed before it arrives; CTA 0 then meets every peer once more
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) atomicAdd(&p.flags[AR_PHASE1], 1u);
    if (blockIdx.x == 0 && warp == 0) {
      if (lane == 0) k::wait_ge(&p.flags[AR_PHASE1], G, ctx, RECEIVE_TIMEOUT_ERROR);
      __syncwarp();
      __threadfence_system();
      if (static_cast<uint32_t>(lane) < P && static_cast<uint32_t>(lane) != me) {
        k::pad_post(ctx, MAX_CH - 1, lane, k::REC_NONE, 0, 0, ctx.kind_word());
        k::pad_wait(ctx, MAX_CH - 1, lane);
      }
      __syncwarp();
      if (lane == 0) dev::st_release_gpu(&p.flags[AR_MIDDLE], 1u);
    }
    wait_release(&p.flags[AR_MIDDLE], ctx);
    // ===== phase 2: every row of the local residual_out, written by this rank's and the peers' CTAs
    for (uint64_t row = blockIdx.x; row < p.m; row += G) {
      const char *hrow = my_heap + p.h_off + row * p.h * 2;
#pragma unroll
      for (int k = 0; k < AR_VPT; ++k) {
        const uint32_t v = threadIdx.x + k * AR_THREADS;
        if (v < nvec) hv[k] = dev::ld_volatile16(hrow + v * 16);
      }
      norm_row(p, row, nvec, hv, s_red);
    }
  }

  // ---------------- teardown: the last CTA to finish publishes the status.  One-shot, it meets the peers first: every
  // CTA of this rank has read what it needed of the peers' x, so when all ranks meet there, each may rewrite its x.
  k::plugin_exit(ctx, p.flags, p.status, P > 1 && !p.two_shot, s_last);
}

// ----------------------------------------------------------------------- host
void preload_ar_rmsnorm_kernels() {
  cudaFuncAttributes a;
  cudaFuncGetAttributes(&a, k_plugin_ar_rmsnorm);
}

cudaError_t launch_ar_rmsnorm(CudaDevice &dev, const ArRmsNormArgs &a, cudaStream_t stream) {
  const DevWorld &w = dev.world();
  const uint32_t P = w.world;
  if (!a.m || a.h % 8 || a.h < 8 || a.h > AR_MAX_H)
    throw std::invalid_argument("ar_rmsnorm: need M >= 1, H % 8 == 0 and 8 <= H <= 16384");
  if (!(a.eps >= 0.f) || !std::isfinite(a.eps)) throw std::invalid_argument("ar_rmsnorm: eps must be finite and non-negative");
  const uint64_t bytes = static_cast<uint64_t>(a.m) * a.h * 2;
  if (a.x_off % 16 || a.h_off % 16 || a.x_off + bytes > w.heap_bytes || a.h_off + bytes > w.heap_bytes)
    throw std::invalid_argument("ar_rmsnorm: x and residual_out must be 16-byte aligned and inside the symmetric heap");
  if (a.x_off < a.h_off + bytes && a.h_off < a.x_off + bytes) throw std::invalid_argument("ar_rmsnorm: x and residual_out overlap");
  auto aligned = [](const void *ptr) { return ptr && reinterpret_cast<uintptr_t>(ptr) % 16 == 0; };
  if (!aligned(a.gamma) || !aligned(a.out) || (a.residual && !aligned(a.residual)))
    throw std::invalid_argument("ar_rmsnorm: the residual, gamma and out pointers must be 16-byte aligned");
  const char *h_ptr = static_cast<const char *>(dev.heap().local()) + a.h_off;
  const char *r_ptr = static_cast<const char *>(a.residual);
  if (r_ptr && r_ptr != h_ptr && r_ptr < h_ptr + bytes && h_ptr < r_ptr + bytes)
    throw std::invalid_argument("ar_rmsnorm: residual overlaps residual_out without being the same tensor");
  ACCL_CUDART(cudaSetDevice(dev.device()));
  ArRmsNormParams p;
  p.w = w;
  p.x_off = a.x_off;
  p.h_off = a.h_off;
  p.residual = static_cast<const __nv_bfloat16 *>(a.residual);
  p.gamma = static_cast<const __nv_bfloat16 *>(a.gamma);
  p.out = static_cast<__nv_bfloat16 *>(a.out);
  p.m = a.m;
  p.h = a.h;
  p.eps = a.eps;
  p.timeout_us = dev.timeout_us();
  // the all-reduce planner's rule (plan.hpp): one-shot while bytes x ranks fit oneshot_max_bytes
  p.two_shot = P > 1 && bytes * P > dev.config().oneshot_max_bytes ? 1u : 0u;
  p.status = a.status_dev;
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev.device());
  // the kernel spins on grid-wide flags and waits for its peers: every CTA of every rank on this GPU must be resident
  const uint32_t grid = std::min<uint32_t>(std::min<uint32_t>(static_cast<uint32_t>(std::max(dev.config().max_ctas, 1)),
                                                              static_cast<uint32_t>(std::max(sms, 1))), a.m);
  p.flags = plugin_flags(dev, 'N', AR_FLAG_WORDS, stream);
  k_plugin_ar_rmsnorm<<<grid, AR_THREADS, 0, stream>>>(p);
  return cudaGetLastError();
}

} // namespace cuda
} // namespace accl
