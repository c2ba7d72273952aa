// GEMM -> reduce-scatter plugin (BASELINE config #5, the north-star fused path).
//
// Each rank holds a K-slice of a row-parallel linear layer: A_r [M, K_r] and
// W_r [N, K_r] (bf16, K contiguous).  The full product is C = sum_r A_r W_r^T,
// reduce-scattered along M: rank o ends up with rows [o*M/P, (o+1)*M/P).
// W_r may also be stored [K_r, N] (N contiguous, GemmRsArgs::w_kn): an nn.Linear weight used in its own backward
// pass, dX = RS_M(dY W).  It is loaded in 64-column boxes and fed to wgmma MN-major (KN kernels); nothing else changes.
//
// One persistent, warp-specialised sm_90a kernel per rank, in two flavours selected at run time
// (GemmRsArgs::variant, default: the CTA pair when the shape allows it):
//   * single CTA per 128 x 256 tile, and
//   * CTA PAIR per 256 x 256 tile (cluster of 2): each CTA computes 128 rows against the same 256 rows of W and
//     loads half of that W tile, multicast by the TMA unit into the shared memory of both CTAs, so W is fetched
//     from L2 once per 256 rows of output,
// each with a bf16 or an fp32 reduction of the partial tiles (the TMA unit adds in the shard's element type: fp32
// shards accumulate the P partial products without intermediate rounding).
// Roles of the 3 warpgroups of a CTA:
//   warpgroup 0, warp 0   TMA producer: cp.async.bulk.tensor 2D loads of 128x64 (A) and 256x64 (W) bf16 tiles,
//                         128B-swizzled, into a 4-stage smem ring, signalling mbarriers with complete_tx
//   warpgroup 0, warps 1-3  zero this rank's output shard and meet the peers (see below)
//   warpgroups 1, 2       consumers: each issues wgmma.mma_async m64n256k16 (bf16 in, fp32 accumulators in
//                         registers) for 64 of the tile's 128 rows straight from the swizzled smem stages, releases
//                         a stage once its MMAs have retired, then runs the epilogue: each warp converts its 16 rows
//                         to the shard's element type, stages 16 x 128-byte boxes in 128B-swizzled smem and hands
//                         them to the TMA unit as cp.reduce.async.bulk.tensor ... .add whose tensor map points at
//                         the OWNER rank's output shard in the peer-mapped symmetric heap — the tile goes into the
//                         collective as it leaves the tensor core, coalesced by hardware, with no SM store
//                         instructions on the NVLink path.  The producer keeps loading the next tile meanwhile.
// Tiles are visited owner-rotated (peers' rows first, own rows last) so the
// NVLink traffic overlaps the remaining math.  Shards are zeroed in-kernel and
// two flag barriers over the sync pads (channel MAX_CH-1) bracket the adds.
// The pipeline, the CTA-pair helpers and the epilogue live in wgmma.cuh; the entry meeting, the grid release and the
// exit in kernels.cuh.  This file keeps the tile orders, the zeroing, the all-reduce signal and broadcast, and the host
// launch code.
//
// GEMM -> ALL-REDUCE (AR kernels, launch_gemm_ar): the same kernel with a two-shot all-reduce epilogue.  Every rank
// ends with the same full C [M, N] at out_off of its heap.
//   reduce     every output tile has one owner rank (ar_tile_of_slot); each rank adds its partial of every tile into
//              the owner's copy of the tile with the reduce-scatter epilogue above.  The owner zeroes only its own tiles.
//   signal     a consumer warp whose adds into a tile have completed adds 1 to the tile's arrival counter in the
//              owner's heap (at cnt_off).  It does so lazily, at its next tile's epilogue or at the end, so it never
//              waits on NVLink for adds it has just issued.
//   broadcast  on the owner, warps 1-3 (idle after zeroing) poll their local counters; a tile with all P * TILE_M / 16
//              arrivals is copied with 16-byte stores into the same tile of every peer's C, so every replica holds the
//              owner's bits.  The exit meeting of the last CTA keeps every rank in the kernel until all pushes into
//              it have landed.
// Each rank sends 2 (P - 1) / P of C, as a ring or two-shot all-reduce does.
//
// The reference has no GEMM; its mechanism for compute-initiated communication
// is kernels/plugins/vadd_put/vadd_put.cpp (data.push + stream_put from inside
// the compute kernel).  Baseline to beat: cuBLAS GEMM + NCCL reduce_scatter.
#include <cuda.h>
#include <cuda_bf16.h>

#include <cstdlib>
#include <cstring>

#include "accl/cuda/cudadevice.hpp"
#include "accl/cuda/driver_api.hpp"
#include "accl/cuda/launch.hpp"
#include "accl/cuda/plugins.hpp"
#include "accl/device/api.cuh"
#include "kernels.cuh"
#include "wgmma.cuh"

namespace accl {
namespace cuda {

struct alignas(64) OutMaps {
  CUtensorMap m[ACCL_MAX_RANKS]; // owner rank o: its [M/P, N] shard through my peer mapping
};

// flag block (kernels.cuh, PluginFlag) of both epilogues; their own word: CTAs whose warps 1-3 have zeroed their part of C
constexpr uint32_t GEMM_ZEROED = k::FLAG_PLUGIN, GEMM_FLAG_WORDS = GEMM_ZEROED + 1;

struct GemmRsParams {
  DevWorld w;
  uint64_t out_off;
  uint32_t m, n, k;
  uint32_t timeout_us;
  unsigned int *flags; // the flag block, zeroed before every launch
  uint32_t *status;    // receives the error bits (0: success) when the kernel ends; may be null
};

struct GemmArParams : GemmRsParams {
  uint64_t cnt_off; // heap offset of the per-tile arrival counters, zeroed before every launch
};
template <bool AR> struct ParamsOf { using type = GemmRsParams; };
template <> struct ParamsOf<true> { using type = GemmArParams; };

// GEMM -> all-reduce tile order.  Tile t (the L2-grouped order of tile_coords) is owned by rank t % P.  Slot s of the
// grid's sweep is tile P (s / P) + (s + me + 1) % P on rank `me`: within every block of P consecutive tiles the ranks
// visit the P owners in rotated order, so at any slot they add into P different owners (no incast), and all ranks
// reach a tile within P slots of one another (tiles complete steadily and their broadcast overlaps the math).  The
// last block may be short; its slots past the last tile are skipped.
__device__ __forceinline__ uint32_t ar_tile_of_slot(uint32_t s, uint32_t P, uint32_t me) { return s - s % P + (s % P + me + 1) % P; }


// GEMM -> all-reduce broadcast: one warp copies a finished TILE_M x 256 tile of its own C into the same tile of every
// peer's C, 16 bytes per lane and access, four loads in flight.  `base`: the tile's offset from the start of a heap.
template <int TILE_M, bool F32>
__device__ __forceinline__ void ar_push_tile(const DevWorld &w, uint32_t me, uint64_t base, uint32_t n, int lane) {
  constexpr uint32_t ES = F32 ? 4 : 2, ROW_VECS = g::BN * ES / 16, TILE_VECS = TILE_M * ROW_VECS;
  const char *src = w.window + static_cast<uint64_t>(me) * w.heap_bytes + base;
  for (uint32_t v = lane; v < TILE_VECS; v += 4 * 32) {
    dev::Vec16 x[4];
    uint64_t off[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint32_t vj = v + 32 * j;
      off[j] = static_cast<uint64_t>(vj / ROW_VECS) * n * ES + (vj % ROW_VECS) * 16;
      x[j] = dev::ld_volatile16(src + off[j]);
    }
    for (uint32_t q = 0; q < w.world; ++q) {
      if (q == me) continue;
      char *dst = w.window + static_cast<uint64_t>(q) * w.heap_bytes + base;
#pragma unroll
      for (int j = 0; j < 4; ++j) dev::st_stream(dst + off[j], x[j]);
    }
  }
}

template <bool PAIR, bool F32, bool KN, bool AR>
__global__ void __launch_bounds__(g::THREADS, 1)
k_plugin_gemm_rs(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                 const __grid_constant__ OutMaps out_maps, typename ParamsOf<AR>::type p) {
  using namespace g;
  using C = Cfg<PAIR>;
  constexpr int GROUP_M = PAIR ? 8 : 16;
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint32_t s_err, s_last;
  __shared__ WorkItem s_item; // identity communicator for the sync pads

  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const uint32_t cr = PAIR ? cluster_ctarank() : 0; // 0 = leader of the pair
  const uint32_t unit = PAIR ? blockIdx.x / 2 : blockIdx.x, num_units = PAIR ? gridDim.x / 2 : gridDim.x;
  const uint32_t P = p.w.world, me = p.w.rank;
  const uint32_t tiles_m = p.m / C::TILE_M, tiles_n = p.n / BN, num_tiles = tiles_m * tiles_n;
  const uint32_t num_slots = AR ? (num_tiles + P - 1) / P * P : num_tiles; // all-reduce: see ar_tile_of_slot
  const uint32_t k_blocks = p.k / BK;
  const uint32_t rows_per_rank = p.m / P, tiles_m_per_rank = tiles_m / P;
  char *my_heap = p.w.window + static_cast<uint64_t>(me) * p.w.heap_bytes;

  // ---------------- one-time setup
  const Smem sm = gemm_smem<PAIR>(smem_raw);
  if (threadIdx.x == 0) {
    s_err = 0;
    k::plugin_item(s_item, p.w, AR ? 0x52 : 0x47, AR ? 0x474152u : 0x47454Du, p.timeout_us); // 'R' (all-reduce) / 'G'
  }
  if (warp == 0 && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap_a)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap_b)) : "memory");
  }
  __syncthreads();
  if (PAIR) cluster_sync(); // the peer's barriers are initialised before anything signals them

  // ---------------- zero my output shard and meet the peers — WITHOUT holding back the math: the TMA producer
  // (warp 0) and the consumers go straight to the main loop; warps 1-3 zero the shard (the reduce-adds accumulate
  // into it), warp 3 of CTA 0 then exchanges the shard offsets with the peers on the sync pads and releases the
  // epilogues of the whole grid.  The first tile's accumulator is ready long after (K / 64 stages of MMAs).
  k::Ctx ctx{p.w, s_item, MAX_CH - 1, 1, reinterpret_cast<Ctrl *>(my_heap), &s_err, static_cast<uint64_t>(p.timeout_us) * 1000ull, nullptr};
  // all-reduce: tiles owned by this rank (me, me + P, ...) and the offset of a tile's first element in C
  constexpr uint32_t ES = F32 ? 4 : 2;
  const uint32_t owned = num_tiles > me ? (num_tiles - me + P - 1) / P : 0;
  auto tile_base = [&](uint32_t t) {
    uint32_t mo, nb;
    tile_coords<GROUP_M>(t, tiles_m, tiles_n, mo, nb);
    return p.out_off + (static_cast<uint64_t>(mo) * C::TILE_M * p.n + nb * BN) * ES;
  };
  if (warp >= 1 && warp <= 3) {
    dev::Vec16 z{0, 0, 0, 0};
    if constexpr (AR) {
      // zero the tiles this rank owns (the adds accumulate into them); its other tiles are overwritten by the owners
      constexpr uint32_t ROW_VECS = BN * ES / 16;
      for (uint32_t i = blockIdx.x; i < owned; i += gridDim.x) {
        char *tile = my_heap + tile_base(me + i * P);
        for (uint32_t v = threadIdx.x - 32; v < C::TILE_M * ROW_VECS; v += 96)
          dev::st_stream(tile + static_cast<uint64_t>(v / ROW_VECS) * p.n * ES + (v % ROW_VECS) * 16, z);
      }
    } else {
      char *shard = my_heap + p.out_off;
      const size_t nvec = static_cast<size_t>(rows_per_rank) * p.n * (F32 ? 4 : 2) / 16;
      const size_t zt = static_cast<size_t>(blockIdx.x) * 96 + (threadIdx.x - 32), zstride = static_cast<size_t>(gridDim.x) * 96;
      for (size_t i = zt; i < nvec; i += zstride) dev::st_stream(shard + i * 16, z);
    }
    asm volatile("fence.proxy.async.global;" ::: "memory"); // the zeros are read by the TMA unit's reduce-adds
    __threadfence();
    asm volatile("bar.sync 1, 96;" ::: "memory"); // warps 1-3 only
    if (threadIdx.x == 32) atomicAdd(&p.flags[GEMM_ZEROED], 1u);
    if (blockIdx.x == 0 && warp == 3) {
      // the whole grid has zeroed -> meet every peer.  The output tensor maps assume the shard (all-reduce: C and the
      // counter block) sits at the same offset in every heap: a peer that does not answer, is in another operation or
      // has it elsewhere gets no reduce-adds.
      if (lane == 0) k::wait_ge(&p.flags[GEMM_ZEROED], gridDim.x, ctx, RECEIVE_TIMEOUT_ERROR);
      __syncwarp();
      __threadfence();
      uint64_t off2 = 0;
      if constexpr (AR) off2 = p.cnt_off;
      const uint32_t mask = k::meet_peers(ctx, AR ? k::REC_OFFS : k::REC_OFF0, p.out_off, off2);
      if (lane == 0) k::release_grid(p.flags, mask); // release the epilogues of every CTA
    }
    if constexpr (AR) {
      // ===== broadcast: this rank's owned tiles, round robin over the grid's warps 1-3, each once all P ranks' consumer
      // warps have signalled it.  Nothing is pushed unless every peer's C and counters sit where this rank's do (a
      // peer that differs gets no pushes, and the tiles it would have added are never complete).
      uint32_t mask = 0;
      if (lane == 0) mask = k::wait_grid(p.flags, ctx);
      mask = __shfl_sync(0xffffffffu, mask, 0);
      __threadfence();
      if (mask == (2u << (P - 1)) - 1u && P > 1) {
        const uint32_t *cnt = reinterpret_cast<const uint32_t *>(my_heap + p.cnt_off);
        const uint32_t want = P * (C::TILE_M / EPI_ROWS); // one arrival per consumer warp of every rank
        bool waiting = true; // false after a timed-out tile: the rest are skipped
        for (uint32_t i = blockIdx.x + gridDim.x * (warp - 1); i < owned && waiting; i += 3 * gridDim.x) {
          const uint32_t t = me + i * P;
          if (lane == 0) waiting = k::wait_ge(&cnt[t], want, ctx, RECEIVE_TIMEOUT_ERROR);
          waiting = __shfl_sync(0xffffffffu, waiting, 0);
          __syncwarp(); // lane 0's acquire of the counter happens before every lane's loads of the tile
          if (waiting) ar_push_tile<C::TILE_M, F32>(p.w, me, tile_base(t), p.n, lane);
        }
        __threadfence_system(); // the pushes are performed before this CTA counts itself finished
      }
    }
  }

  // ---------------- warp-specialised main loop
  if (warp == 0) {
    // ===== TMA producer (pair: each CTA its 128 rows of A, and its half of W multicast to both CTAs)
    uint32_t stage = 0, phase = 0;
    for (uint32_t s = unit; s < num_slots; s += num_units) {
      uint32_t t = s;
      if constexpr (AR) {
        t = ar_tile_of_slot(s, P, me);
        if (t >= num_tiles) continue;
      }
      uint32_t mo, nb;
      tile_coords<GROUP_M>(t, tiles_m, tiles_n, mo, nb);
      const uint32_t mb = AR ? mo : (mo + (me + 1) * tiles_m_per_rank) % tiles_m; // peers' rows first, mine last
      produce_tile<PAIR, KN>(sm, &tmap_a, static_cast<int>(mb * C::TILE_M + cr * BM), &tmap_b, nb, k_blocks, cr, stage, phase, lane);
    }
  } else if (warp >= 4) {
    // ===== consumers: wgmma into registers, then registers -> shard element type -> swizzled smem -> collective
    const uint32_t wg = warp / 4 - 1;   // rows [64 wg, 64 wg + 64) of the CTA's 128
    const uint32_t wi = warp % 4;       // this warp's 16 of them
    uint8_t *my_epi = sm.epi + (warp - 4) * 2 * EPI_BUF_BYTES;
    uint32_t stage = 0, phase = 0, ebuf = 0;
    uint32_t owners_ok = 0; // owners whose shard sits at out_off, the only ones this warp adds into; 0: not yet released
    float d[128];
#pragma unroll
    for (int i = 0; i < 128; ++i) d[i] = 0.f;
    uint32_t pending = ~0u; // all-reduce: the tile whose adds this warp has issued but not yet signalled
    // Signal `pending`: its adds have been performed at the owner (wait_group without .read waits for the writes, not
    // only the reads of shared memory), fence.proxy.async orders those async-proxy writes before this thread's
    // generic-proxy accesses, and the release red then makes them visible (release cumulativity, PTX memory model)
    // to any thread that acquires the counter at system scope — the owner's broadcast warp.
    auto signal = [&]() {
      if constexpr (AR) {
        if (lane == 0 && pending != ~0u && P > 1) { // (one rank: nothing is broadcast, nobody reads the counters)
          device::emit_flush();
          asm volatile("fence.proxy.async.global;" ::: "memory");
          dev::red_release_sys_add(reinterpret_cast<uint32_t *>(p.w.window + static_cast<uint64_t>(pending % P) * p.w.heap_bytes +
                                                                p.cnt_off) + pending, 1u);
        }
        pending = ~0u;
      }
    };
    for (uint32_t s = unit; s < num_slots; s += num_units) {
      uint32_t t = s;
      if constexpr (AR) {
        t = ar_tile_of_slot(s, P, me);
        if (t >= num_tiles) continue;
      }
      uint32_t mo, nb;
      tile_coords<GROUP_M>(t, tiles_m, tiles_n, mo, nb);
      const uint32_t mb = AR ? mo : (mo + (me + 1) * tiles_m_per_rank) % tiles_m;
      consume_tile<PAIR, KN>(sm, d, wg, k_blocks, cr, stage, phase);

      if (!owners_ok) {
        if (lane == 0) owners_ok = k::wait_grid(p.flags, ctx);
        owners_ok = __shfl_sync(0xffffffffu, owners_ok, 0);
        __threadfence();
        // every shard has been zeroed with generic stores: order them before this warp's TMA reduce-adds
        asm volatile("fence.proxy.async.global;" ::: "memory");
      }
      const uint32_t row0 = mb * C::TILE_M + cr * BM + wg * 64 + wi * EPI_ROWS; // first of this warp's 16 rows
      if constexpr (AR) {
        // the previous tile's adds were issued a whole mainloop ago: signalling it now does not wait on NVLink
        signal();
        const uint32_t owner = t % P;
        if ((owners_ok >> owner) & 1u) {
          epilogue_tile<F32, true>(d, my_epi, ebuf, lane, &out_maps.m[owner], static_cast<int>(nb * BN), static_cast<int>(row0));
          pending = t;
        }
      } else {
        const uint32_t owner = row0 / rows_per_rank;                              // a warp's rows never straddle owners
        const int local_row0 = static_cast<int>(row0 - owner * rows_per_rank);
        if ((owners_ok >> owner) & 1u) epilogue_tile<F32, true>(d, my_epi, ebuf, lane, &out_maps.m[owner], static_cast<int>(nb * BN), local_row0);
      }
    }
    signal(); // all-reduce: the last tile
    if (lane == 0) device::emit_flush(); // all my reductions have completed
    __syncwarp();
    __threadfence_system(); // my adds are performed before this CTA reports completion
  }

  // ---------------- teardown: the last CTA of the grid meets the peers again (every CTA of this rank has added and
  // pushed its tiles: when all ranks meet there, every shard is complete)
  if (PAIR) cluster_sync(); // nobody exits while the peer may still signal its barriers or write its smem
  k::plugin_exit(ctx, p.flags, p.status, true, s_last);
}

// ----------------------------------------------------------------------- host
namespace {
template <bool PAIR, bool F32, bool KN, bool AR> void set_smem_attr() {
  cudaFuncSetAttribute(k_plugin_gemm_rs<PAIR, F32, KN, AR>, cudaFuncAttributeMaxDynamicSharedMemorySize, g::SMEM_BYTES);
}
template <bool KN, bool AR> void preload_layout() {
  cudaFuncAttributes a;
  cudaFuncGetAttributes(&a, k_plugin_gemm_rs<false, false, KN, AR>);
  cudaFuncGetAttributes(&a, k_plugin_gemm_rs<false, true, KN, AR>);
  cudaFuncGetAttributes(&a, k_plugin_gemm_rs<true, false, KN, AR>);
  cudaFuncGetAttributes(&a, k_plugin_gemm_rs<true, true, KN, AR>);
  set_smem_attr<false, false, KN, AR>();
  set_smem_attr<false, true, KN, AR>();
  set_smem_attr<true, false, KN, AR>();
  set_smem_attr<true, true, KN, AR>();
}
} // namespace

void preload_gemm_rs_kernels() {
  preload_layout<false, false>();
  preload_layout<true, false>();
  preload_layout<false, true>();
  preload_layout<true, true>();
}

template <bool PAIR, bool F32, bool KN, bool AR>
static cudaError_t launch_variant(const CUtensorMap &ta, const CUtensorMap &tb, const OutMaps &om, const typename ParamsOf<AR>::type &p,
                                  uint32_t tiles, int sms, cudaStream_t stream) {
  using namespace g;
  set_smem_attr<PAIR, F32, KN, AR>();
  cudaLaunchConfig_t lc = {};
  lc.blockDim = dim3(THREADS);
  lc.dynamicSmemBytes = SMEM_BYTES;
  lc.stream = stream;
  cudaLaunchAttribute at[1];
  if (PAIR) {
    uint32_t pairs = std::min<uint32_t>(static_cast<uint32_t>(sms) / 2, tiles);
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = 2;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    lc.attrs = at;
    lc.numAttrs = 1;
    lc.gridDim = dim3(2 * pairs);
    // the kernel spins on grid-wide flags: every cluster must be resident at once
    int max_clusters = 0;
    if (cudaOccupancyMaxActiveClusters(&max_clusters, k_plugin_gemm_rs<PAIR, F32, KN, AR>, &lc) == cudaSuccess && max_clusters > 0)
      pairs = std::min<uint32_t>(pairs, static_cast<uint32_t>(max_clusters));
    lc.gridDim = dim3(2 * pairs);
  } else {
    lc.gridDim = dim3(std::min<uint32_t>(static_cast<uint32_t>(sms), tiles));
  }
  return cudaLaunchKernelEx(&lc, k_plugin_gemm_rs<PAIR, F32, KN, AR>, ta, tb, om, p);
}

// the eight kernels of one epilogue (AR: all-reduce, else reduce-scatter)
template <bool AR>
static cudaError_t launch_kernel(bool pair, bool f32, bool kn, const CUtensorMap &ta, const CUtensorMap &tb, const OutMaps &om,
                                 const typename ParamsOf<AR>::type &p, uint32_t tiles, int sms, cudaStream_t stream) {
  if (kn) {
    if (pair) return f32 ? launch_variant<true, true, true, AR>(ta, tb, om, p, tiles, sms, stream) : launch_variant<true, false, true, AR>(ta, tb, om, p, tiles, sms, stream);
    return f32 ? launch_variant<false, true, true, AR>(ta, tb, om, p, tiles, sms, stream) : launch_variant<false, false, true, AR>(ta, tb, om, p, tiles, sms, stream);
  }
  if (pair) return f32 ? launch_variant<true, true, false, AR>(ta, tb, om, p, tiles, sms, stream) : launch_variant<true, false, false, AR>(ta, tb, om, p, tiles, sms, stream);
  return f32 ? launch_variant<false, true, false, AR>(ta, tb, om, p, tiles, sms, stream) : launch_variant<false, false, false, AR>(ta, tb, om, p, tiles, sms, stream);
}

// variant: 0 = automatic, 1 = single CTA, 2 = pair; ACCL_GEMM_VARIANT overrides the automatic choice
static int chosen_variant(int variant) {
  static const int env_variant = [] {
    const char *e = std::getenv("ACCL_GEMM_VARIANT");
    return e ? std::atoi(e) : 0;
  }();
  return variant ? variant : env_variant;
}

// The launch of either epilogue once its arguments are checked.  Owner o's output, shard_rows x N, sits at out_off of
// its heap (symmetric allocation; verified in-kernel: an owner whose output is elsewhere gets no adds and the call
// reports DMA_MISMATCH_ERROR).  pair_ok: M suits the CTA-pair kernel; pair_error: what to throw when it is forced anyway.
template <bool AR, typename Args>
static cudaError_t launch_gemm(CudaDevice &dev, const Args &a, uint32_t shard_rows, bool pair_ok, const char *pair_error,
                               cudaStream_t stream) {
  using namespace g;
  const DevWorld &w = dev.world();
  ACCL_CUDART(cudaSetDevice(dev.device()));
  const int variant = chosen_variant(a.variant);
  if (variant == 2 && !pair_ok) throw std::invalid_argument(pair_error);
  const bool pair = variant == 2 || (variant == 0 && pair_ok);
  const bool f32 = a.out_f32;
  const CUtensorMap ta = make_map(a.a, a.m, a.k, BM, BK);
  // each CTA of a pair loads half of the N tile; a [K, N] weight goes in boxes of 64 columns x 64 K-rows
  const CUtensorMap tb = a.w_kn ? make_map(a.w, a.k, a.n, BK, 64) : make_map(a.w, a.n, a.k, pair ? BN / 2 : BN, BK);
  OutMaps om;
  std::memset(&om, 0, sizeof(om));
  for (uint32_t o = 0; o < w.world; ++o)
    om.m[o] = make_map(w.window + static_cast<uint64_t>(o) * w.heap_bytes + a.out_off, shard_rows, a.n, EPI_ROWS, f32 ? 32 : 64, f32);
  typename ParamsOf<AR>::type p;
  p.w = w;
  p.out_off = a.out_off;
  p.m = a.m;
  p.n = a.n;
  p.k = a.k;
  p.timeout_us = dev.timeout_us();
  p.flags = plugin_flags(dev, 'G', GEMM_FLAG_WORDS, stream);
  p.status = a.status_dev;
  const uint32_t tiles = (a.m / (pair ? 2 * BM : BM)) * (a.n / BN);
  if constexpr (AR) {
    p.cnt_off = a.cnt_off;
    // the peers add into these counters only after this launch has met them, i.e. after the memset
    ACCL_CUDART(cudaMemsetAsync(w.window + static_cast<uint64_t>(w.rank) * w.heap_bytes + a.cnt_off, 0, tiles * sizeof(uint32_t), stream));
  }
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev.device());
  return launch_kernel<AR>(pair, f32, a.w_kn, ta, tb, om, p, tiles, sms, stream);
}

cudaError_t launch_gemm_rs(CudaDevice &dev, const GemmRsArgs &a, cudaStream_t stream) {
  using namespace g;
  const uint32_t P = dev.world().world;
  if (a.m % (BM * P) || a.n % BN || a.k % BK)
    throw std::invalid_argument("gemm_rs: need M % (128*world) == 0, N % 256 == 0, K % 64 == 0");
  // CTA-pair kernel: 256-row tiles must not straddle shard owners
  return launch_gemm<false>(dev, a, a.m / P, a.m % (2 * BM * P) == 0, "gemm_rs: the CTA-pair kernel needs M % (256*world) == 0", stream);
}

cudaError_t launch_gemm_ar(CudaDevice &dev, const GemmArArgs &a, cudaStream_t stream) {
  using namespace g;
  const DevWorld &w = dev.world();
  if (!a.m || !a.n || !a.k || a.m % BM || a.n % BN || a.k % BK)
    throw std::invalid_argument("gemm_ar: need M % 128 == 0, N % 256 == 0, K % 64 == 0, none of them zero");
  if (static_cast<uint64_t>(a.m / BM) * (a.n / BN) > GEMM_AR_MAX_TILES)
    throw std::invalid_argument("gemm_ar: more than GEMM_AR_MAX_TILES 128 x 256 tiles");
  const uint64_t c_bytes = static_cast<uint64_t>(a.m) * a.n * (a.out_f32 ? 4 : 2);
  if (a.out_off % 16 || a.cnt_off % 16 || a.out_off + c_bytes > w.heap_bytes || a.cnt_off + GEMM_AR_MAX_TILES * 4ull > w.heap_bytes)
    throw std::invalid_argument("gemm_ar: C and the counter block must be 16-byte aligned and inside the symmetric heap");
  return launch_gemm<true>(dev, a, a.m, a.m % (2 * BM) == 0, "gemm_ar: the CTA-pair kernel needs M % 256 == 0", stream);
}

} // namespace cuda
} // namespace accl
