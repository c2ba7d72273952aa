// The sm_90a GEMM machinery shared by the fused GEMM plugins (plugin_gemm_rs.cu, plugin_ag_gemm.cu): tile shape and
// shared-memory budget of one CTA, mbarrier / TMA / wgmma / shared-memory-descriptor helpers and their CTA-pair
// (cluster of 2) flavours, the shared-memory carve-up, the TMA -> mbarrier -> wgmma pipeline of one tile
// (produce_tile / consume_tile), the L2 tile order, the 128B-swizzled epilogue (epilogue_tile), plus the host-side
// tensor-map encoder.  Tile orders, grids and meetings stay with each plugin.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>

#include <stdexcept>
#include <string>

#include "accl/cuda/driver_api.hpp"
#include "accl/device/api.cuh"

namespace accl {
namespace cuda {

namespace g {
constexpr int BM = 128, BN = 256, BK = 64;
constexpr int STAGES = 4;
constexpr int WGMMA_K = 16;
constexpr int A_STAGE_BYTES = BM * BK * 2;  // 16 KB
constexpr int B_STAGE_BYTES = BN * BK * 2;  // 32 KB
constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
constexpr int CONSUMER_WARPS = 8;
constexpr int EPI_ROWS = 16;                         // rows of one warp's share of a wgmma accumulator
constexpr int EPI_BUF_BYTES = EPI_ROWS * 128;        // 16 rows x one 128-byte swizzle row = 2 KB
constexpr int EPI_BYTES = CONSUMER_WARPS * 2 /*double buffer*/ * EPI_BUF_BYTES;
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + EPI_BYTES + 1024 /*align*/ + 256 /*barriers*/;
constexpr int THREADS = 384;

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE;\n"
      "bra WAIT_LOOP;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}

__device__ __forceinline__ void tma_load_2d(void *smem_dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

// one 16-row box of staged shared memory -> global memory by the TMA unit (a bulk group of this thread)
__device__ __forceinline__ void tma_store_2d(const CUtensorMap *map, const void *smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(reinterpret_cast<uint64_t>(map)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}

// ---- CTA-pair (cluster of 2) flavours of the primitives
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// the TMA unit writes the box at the same shared-memory offset in every CTA of `mask` and signals the barrier at
// the same offset in each of them
__device__ __forceinline__ void tma_load_2d_multicast(void *smem_dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1,
                                                      uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(
          smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(mask)
      : "memory");
}
// arrive on the barrier at this shared-memory offset in CTA `cta` of the cluster
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t *bar, uint32_t cta) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(bar)), "r"(cta));
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}

// PAIR: a CTA pair computes one 256 x 256 tile, each CTA 128 rows of it, and each loads half of the W tile, multicast
// into both CTAs
template <bool PAIR> struct Cfg {
  static constexpr int BN_LOAD = PAIR ? BN / 2 : BN;          // W rows this CTA loads per stage
  static constexpr int TILE_M = PAIR ? 2 * BM : BM;           // rows of one output tile
};

// K-major, 128B-swizzled shared-memory matrix descriptor (sm_90 wgmma format): rows of 128 bytes, 8-row groups
// 1024 bytes apart; the leading byte offset is unused for swizzled K-major operands
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);      // start address >> 4
  d |= static_cast<uint64_t>(1) << 16;                          // leading byte offset
  d |= static_cast<uint64_t>(1024 >> 4) << 32;                  // stride byte offset: 8 rows x 128 B
  d |= static_cast<uint64_t>(1) << 62;                          // SWIZZLE_128B
  return d;
}

// MN-major, 128B-swizzled descriptor for a B operand stored [K, N] (N contiguous) and loaded as boxes of 64 columns x
// 64 K-rows: a swizzle atom is 8 K-rows of 128 bytes (64 columns); atoms along N sit one box (8 KB, leading byte
// offset) apart, 8-row groups along K 1 KB (stride byte offset) apart.  One K=16 step is 16 rows = 2048 bytes.
__device__ __forceinline__ uint64_t make_smem_desc_mn(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);      // start address >> 4
  d |= static_cast<uint64_t>(8192 >> 4) << 16;                  // leading byte offset: next 64 columns
  d |= static_cast<uint64_t>(1024 >> 4) << 32;                  // stride byte offset: next 8 K-rows
  d |= static_cast<uint64_t>(1) << 62;                          // SWIZZLE_128B
  return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D[64 x 256] (+)= A[64 x 16] B[256 x 16]^T, bf16 operands in smem, fp32 D in registers (warpgroup-wide).  A is
// K-major; B is K-major (TNSP_B = 0, desc_b from make_smem_desc) or MN-major (TNSP_B = 1, make_smem_desc_mn).
// Thread t of the warpgroup holds rows 16*(t/32) + (t%32)/4 (+8) and columns 8*j + 2*(t%4) (+1), j = 0..31:
// d[4j], d[4j+1] on the first row, d[4j+2], d[4j+3] on the second.
template <int TNSP_B = 0>
__device__ __forceinline__ void wgmma_m64n256k16(float (&d)[128], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %130, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
      "%128, %129, p, 1, 1, 0, %131;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate), "n"(TNSP_B)
      : "memory");
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t *>(&v);
}

// The dynamic shared memory of a GEMM CTA, 1024-byte aligned for the 128B swizzle: the A stages, the W stages, the
// epilogue buffers of the consumer warps, then the full / empty barriers of the stage ring.
struct Smem {
  uint8_t *a, *b, *epi;
  uint64_t *full, *empty;
};

// Carve up the dynamic shared memory; thread 0 also initialises the stage barriers.  The caller's __syncthreads (and
// for a pair its cluster_sync) makes them visible before anything waits on or signals them.
template <bool PAIR> __device__ __forceinline__ Smem gemm_smem(uint8_t *raw) {
  uint8_t *base = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint64_t *bars = reinterpret_cast<uint64_t *>(base + STAGES * STAGE_BYTES + EPI_BYTES);
  const Smem s{base, base + STAGES * A_STAGE_BYTES, base + STAGES * STAGE_BYTES, bars, bars + STAGES};
  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&s.full[i], 1);             // the producer's arrive.expect_tx
      mbar_init(&s.empty[i], PAIR ? 4 : 2); // one arrival per consumer warpgroup (pair: of both CTAs)
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  return s;
}

// TMA producer, lane 0 of its warp: the k-loop of one tile into the stage ring.  A: 128 rows from row_a of map_a.
// W: this CTA's BN_LOAD rows (nk) or columns (kn, boxes of 64 columns x 64 K-rows, one 8 KB column of swizzle atoms
// each) from column nb * BN; a pair multicasts its half into both CTAs (cr: this CTA's rank in the pair).
template <bool PAIR, bool KN>
__device__ __forceinline__ void produce_tile(const Smem &s, const CUtensorMap *map_a, int row_a, const CUtensorMap *map_w, uint32_t nb,
                                             uint32_t k_blocks, uint32_t cr, uint32_t &stage, uint32_t &phase, int lane) {
  using C = Cfg<PAIR>;
  for (uint32_t kb = 0; kb < k_blocks; ++kb) {
    if (lane == 0) {
      mbar_wait(&s.empty[stage], phase ^ 1); // pair: the stage is free in BOTH CTAs
      mbar_expect_tx(&s.full[stage], STAGE_BYTES);
      tma_load_2d(s.a + stage * A_STAGE_BYTES, map_a, &s.full[stage], static_cast<int>(kb * BK), row_a);
      if constexpr (KN) {
#pragma unroll
        for (int j = 0; j < C::BN_LOAD / 64; ++j) {
          uint8_t *dst = s.b + stage * B_STAGE_BYTES + cr * (C::BN_LOAD * BK * 2) + j * (64 * BK * 2);
          const int n0 = static_cast<int>(nb * BN + cr * C::BN_LOAD + 64 * j), k0 = static_cast<int>(kb * BK);
          if (PAIR)
            tma_load_2d_multicast(dst, map_w, &s.full[stage], n0, k0, 0x3);
          else
            tma_load_2d(dst, map_w, &s.full[stage], n0, k0);
        }
      } else if (PAIR) {
        tma_load_2d_multicast(s.b + stage * B_STAGE_BYTES + cr * (C::BN_LOAD * BK * 2), map_w, &s.full[stage],
                              static_cast<int>(kb * BK), static_cast<int>(nb * BN + cr * C::BN_LOAD), 0x3);
      } else {
        tma_load_2d(s.b + stage * B_STAGE_BYTES, map_w, &s.full[stage], static_cast<int>(kb * BK), static_cast<int>(nb * BN));
      }
    }
    __syncwarp();
    if (++stage == STAGES) {
      stage = 0;
      phase ^= 1;
    }
  }
}

// Consumer warpgroup wg: the k-loop of one tile into d (rows [64 wg, 64 wg + 64) of the CTA's 128).  A stage is
// released once its MMAs have retired, by one arrival of the warpgroup (pair: on the barriers of both CTAs, since the
// peer's producer multicasts into it too).  Returns after every MMA of the tile has retired.
template <bool PAIR, bool KN>
__device__ __forceinline__ void consume_tile(const Smem &s, float (&d)[128], uint32_t wg, uint32_t k_blocks, uint32_t cr, uint32_t &stage,
                                             uint32_t &phase) {
  const bool signaller = threadIdx.x % 128 == 0;
  auto release = [&](uint32_t st) {
    if (signaller) {
      mbar_arrive(&s.empty[st]);
      if (PAIR) mbar_arrive_cluster(&s.empty[st], cr ^ 1u);
    }
  };
  uint32_t prev = 0;
  for (uint32_t kb = 0; kb < k_blocks; ++kb) {
    mbar_wait(&s.full[stage], phase);
    const uint64_t da = make_smem_desc(smem_u32(s.a + stage * A_STAGE_BYTES + wg * 64 * 128));
    const uint32_t b_addr = smem_u32(s.b + stage * B_STAGE_BYTES);
    const uint64_t db = KN ? make_smem_desc_mn(b_addr) : make_smem_desc(b_addr);
    constexpr uint64_t DB_STEP = KN ? 128 : 2; // per K=16 step, >> 4: 16 K-rows of 128 B (MN-major), 32 B (K-major)
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BK / WGMMA_K; ++kk) // A: +32 bytes (>>4 = 2) per K=16 step inside the swizzle atom
      wgmma_m64n256k16<KN ? 1 : 0>(d, da + 2 * kk, db + DB_STEP * kk, (kb | kk) ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<1>(); // the previous stage's MMAs have retired: it may be refilled
    if (kb > 0) release(prev);
    prev = stage;
    if (++stage == STAGES) {
      stage = 0;
      phase ^= 1;
    }
  }
  wgmma_wait<0>();
  release(prev);
}
} // namespace g

// Tile order: groups of GROUP_M tile rows are swept column by column, so the tiles in flight (one per SM) form a
// near-square patch whose A rows and W rows are read from L2 by many CTAs at once.  A plain row-major sweep keeps
// all of W in flight at once and leaves the tensor cores waiting on L2 misses.
template <int GROUP_M>
__device__ __forceinline__ void tile_coords(uint32_t t, uint32_t tiles_m, uint32_t tiles_n, uint32_t &mo, uint32_t &nb) {
  const uint32_t width = GROUP_M * tiles_n;
  const uint32_t group = t / width, first_m = group * GROUP_M;
  const uint32_t gsize = tiles_m - first_m < static_cast<uint32_t>(GROUP_M) ? tiles_m - first_m : static_cast<uint32_t>(GROUP_M);
  const uint32_t in = t % width;
  mo = first_m + in % gsize;
  nb = in / gsize;
}

// One epilogue chunk: this warp's 16 accumulator rows x COLS columns (chunk C of the 256) -> the shard's element type,
// staged in 128B-swizzled shared memory (16-byte chunk index XOR row % 8) for the collective
// (device API: reduce_scatter_emit_tile).
template <bool F32, int C>
__device__ __forceinline__ void epilogue_chunk(const float (&d)[128], uint8_t *buf, int lane) {
  const int r0 = lane / 4, q = lane % 4; // rows r0 and r0 + 8 (same swizzle phase)
  if (F32) {
    // 32 fp32 columns = one 128-byte row
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const int j = 4 * C + jj;
      const int chunk = (2 * jj + (q >> 1)) ^ r0;
      const int off = chunk * 16 + 8 * (q & 1);
      *reinterpret_cast<float2 *>(buf + r0 * 128 + off) = make_float2(d[4 * j], d[4 * j + 1]);
      *reinterpret_cast<float2 *>(buf + (r0 + 8) * 128 + off) = make_float2(d[4 * j + 2], d[4 * j + 3]);
    }
  } else {
    // 64 bf16 columns = one 128-byte row
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      const int j = 8 * C + jj;
      const int off = (jj ^ r0) * 16 + 4 * q;
      *reinterpret_cast<uint32_t *>(buf + r0 * 128 + off) = g::pack_bf16x2(d[4 * j], d[4 * j + 1]);
      *reinterpret_cast<uint32_t *>(buf + (r0 + 8) * 128 + off) = g::pack_bf16x2(d[4 * j + 2], d[4 * j + 3]);
    }
  }
}

// The epilogue of one warp: its 16 accumulator rows, chunk by chunk (C of the 256 columns), through the warp's two
// buffers `epi` (ebuf: the next one) to the TMA unit, which adds each box into the memory of `map`
// (device API: reduce_scatter_emit_tile) with REDUCE, else stores it there.
template <bool F32, bool REDUCE, int C = 0>
__device__ __forceinline__ void epilogue_tile(const float (&d)[128], uint8_t *epi, uint32_t &ebuf, int lane, const CUtensorMap *map,
                                              int col0, int row) {
  constexpr int COLS = F32 ? 32 : 64;
  if constexpr (C < g::BN / COLS) {
    uint8_t *buf = epi + ebuf * g::EPI_BUF_BYTES;
    // the TMA unit must be done READING this buffer (handed over two chunks ago)
    if (lane == 0) device::emit_wait_read<1>();
    __syncwarp();
    epilogue_chunk<F32, C>(d, buf, lane);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); // generic-proxy writes -> visible to the TMA unit
    __syncwarp();
    if (lane == 0) {
      if constexpr (REDUCE)
        device::reduce_scatter_emit_tile(map, buf, col0 + C * COLS, row);
      else
        g::tma_store_2d(map, buf, col0 + C * COLS, row);
    }
    ebuf ^= 1;
    epilogue_tile<F32, REDUCE, C + 1>(d, epi, ebuf, lane, map, col0, row);
  }
}

// ------------------------------------------------------------------ host: 2-D bf16 / fp32 tensor maps
using EncodeFn = CUresult (*)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                              const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                              CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline EncodeFn encode_fn() {
  static EncodeFn fn = [] {
    void *p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || !p)
      throw std::runtime_error("cuTensorMapEncodeTiled unavailable");
    return reinterpret_cast<EncodeFn>(p);
  }();
  return fn;
}

inline CUtensorMap make_map(const void *base, uint64_t rows, uint64_t cols, uint32_t box_rows, uint32_t box_cols, bool f32 = false) {
  CUtensorMap m;
  const uint64_t es = f32 ? 4 : 2;
  const cuuint64_t dims[2] = {cols, rows};           // innermost first
  const cuuint64_t strides[1] = {cols * es};         // bytes between rows
  const cuuint32_t box[2] = {box_cols, box_rows};
  const cuuint32_t estr[2] = {1, 1};
  CUresult r = encode_fn()(&m, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void *>(base), dims,
                           strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                           CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw std::runtime_error("cuTensorMapEncodeTiled failed: " + cu_error_string(r));
  return m;
}

} // namespace cuda
} // namespace accl
