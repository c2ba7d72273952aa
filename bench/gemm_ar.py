"""GEMM -> all-reduce: the fused wgmma plugin (ops.gemm_all_reduce) against the unfused ways to get the same C on every rank.

  python bench/gemm_ar.py --check                  # 1 GPU, 8192^3: fused vs cuBLAS, and vs the GEMM -> reduce-scatter kernel
  python -m torch.distributed.run --nproc-per-node N ... bench/gemm_ar.py --gm 8192 --gn 8192 --gk 1024

Per rank: A[M, K] and W[N, K] bf16 (its K-slice); result: C = sum_r A_r W_r^T [M, N] on every rank.  Compared in one
process: the fused kernel, cuBLAS + accl all-reduce, cuBLAS + NCCL all-reduce, and gemm_reduce_scatter + accl
all-gather.  Reports device-timed ms (CUDA events, max over ranks), TFLOP/s per GPU and the fraction of the roofline
max(FLOPs / BF16_PEAK, NVLink bytes / LINK_BPS), naming the bound.  Both peaks are NVIDIA's H100 SXM data-sheet figures
(700 W, dense bf16; NVLink 4 per direction), not measurements; the card's name and power limit are read in the same run.
--repeats R alternates the fused kernel and gemm_reduce_scatter R times (world 1: the same GEMM, different epilogue).
"""
import argparse
import json
import os
import subprocess
import sys

BF16_PEAK = 989.4e12  # H100 SXM data sheet, dense bf16 FLOP/s
LINK_BPS = 450e9      # H100 SXM data sheet, NVLink 4 bytes/s per direction per GPU

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import accl_b200 as A  # noqa: E402
from accl_b200.ops import gemm_all_reduce, gemm_reduce_scatter  # noqa: E402
from accl_b200.parallel import TensorGroup  # noqa: E402


def card(local):
    """(name, power limit) of this rank's GPU, read now."""
    name = torch.cuda.get_device_name(local)
    try:
        limit = subprocess.run(["nvidia-smi", "-i", str(local), "--query-gpu=power.limit", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit or "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gm", dest="m", type=int, default=8192)
    ap.add_argument("--gn", dest="n", type=int, default=8192)
    ap.add_argument("--gk", dest="k", type=int, default=8192, help="K per rank")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=1, help="alternate fused / gemm_reduce_scatter this many times")
    ap.add_argument("--check", action="store_true", help="compare the fused result with cuBLAS + NCCL")
    ap.add_argument("--variant", type=int, default=0, help="0 auto, 1 single CTA per tile, 2 CTA pair (cluster of 2)")
    ap.add_argument("--f32", action="store_true", help="fp32 C (fp32 accumulation of the partial products)")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    M, N, K = a.m, a.n, a.k
    es = 4 if a.f32 else 2
    heap_mb = (3 * M * N * es >> 20) + 384
    acc = A.cuda_rank(rank, world, local, heap_mb=max(512, heap_mb), max_ctas=32)
    acc.initialize(n_egr_rx_bufs=4, egr_rx_buf_size=16 << 10, max_egr_size=16 << 10, max_rndzv_size=1 << 30)
    group = TensorGroup(acc)
    out_dtype = torch.float32 if a.f32 else torch.bfloat16

    g = torch.Generator(device="cuda").manual_seed(7 + rank)
    x = (torch.randn(M, K, device="cuda", generator=g) * 0.25).bfloat16()
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.25).bfloat16()
    out = acc.create_buffer(M * N, out_dtype)
    c_heap = group.empty(M, N, dtype=torch.bfloat16)      # cuBLAS writes here, accl all-reduces in place
    shard = acc.create_buffer(M // world * N, out_dtype) if M % (128 * world) == 0 else None
    gathered = group.empty(M, N, dtype=out_dtype)
    c_nccl = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")

    def timed(fn, iters):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(iters):
            fn()
        e.record()
        torch.cuda.synchronize()
        ms = s.elapsed_time(e) / iters
        if world > 1:
            t = torch.tensor([ms], device="cuda", dtype=torch.float64)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            ms = float(t.item())
        return ms

    def fused():
        gemm_all_reduce(acc, x, w, out, variant=a.variant)

    def cublas_accl():
        torch.matmul(x, w.t(), out=c_heap)
        if world > 1:
            group.all_reduce(c_heap)

    def cublas_nccl():
        torch.matmul(x, w.t(), out=c_nccl)
        if world > 1:
            dist.all_reduce(c_nccl)

    def rs_ag():
        gemm_reduce_scatter(acc, x, w, shard, variant=a.variant)
        if world > 1:
            group.all_gather_into_tensor(gathered, shard.dev[:M // world * N])

    fused_ms, rs_ms = [], []
    for _ in range(a.repeats):
        fused_ms.append(timed(fused, a.iters))
        if shard is not None:
            rs_ms.append(timed(rs_ag, a.iters))
    ms_accl = timed(cublas_accl, a.iters)
    ms_nccl = timed(cublas_nccl, a.iters)
    group.check(block=True)
    ms_f = min(fused_ms)
    flops = 2.0 * M * N * K
    nvlink_bytes = 2.0 * (world - 1) / world * M * N * es  # two-shot: partials to the owners, finished tiles back
    t_flops, t_link = flops / BF16_PEAK, nvlink_bytes / LINK_BPS
    t_roof = max(t_flops, t_link) * 1e3
    err = replicas_equal = None
    if a.check:
        st = group.plugin_status()
        gemm_all_reduce(acc, x, w, out, variant=a.variant, status=st)
        cublas_nccl()
        torch.cuda.synchronize()
        got = out.dev.view(M, N)
        err = float((got.float() - c_nccl.float()).abs().max())
        assert int(st.item()) == 0, f"status {int(st.item()):#x}"
        if world > 1:
            # every replica holds the same bits: compare a checksum of the raw words
            words = got.view(torch.int32 if a.f32 else torch.int16).to(torch.int64)
            h = torch.stack([words.sum(), (words * torch.arange(words.numel(), device="cuda").view(M, N) % 1000003).sum()])
            hs = [torch.empty_like(h) for _ in range(world)]
            dist.all_gather(hs, h)
            replicas_equal = all(torch.equal(hs[0], v) for v in hs)
    name, limit = card(local)
    if rank == 0:
        row = dict(op="gemm_all_reduce", m=M, n=N, k_per_rank=K, world=world, variant=a.variant,
                   out_dtype="fp32" if a.f32 else "bf16", fused_ms=ms_f, fused_ms_runs=fused_ms,
                   gemm_rs_allgather_ms_runs=rs_ms, cublas_accl_allreduce_ms=ms_accl, cublas_nccl_allreduce_ms=ms_nccl,
                   fused_tflops=flops / ms_f * 1e-9, speedup_vs_cublas_nccl=ms_nccl / ms_f,
                   roofline_ms=t_roof, roofline_bound="bf16 tensor-core FLOP/s" if t_flops >= t_link else "NVLink bytes/s",
                   frac_of_roofline=t_roof / ms_f, peak_source="H100 SXM data sheet (700 W)",
                   bf16_peak_tflops=BF16_PEAK * 1e-12, link_GBps=LINK_BPS * 1e-9, gpu=name, power_limit=limit,
                   max_abs_err_vs_cublas_nccl=err, replicas_bit_identical=replicas_equal)
        print(json.dumps(row), flush=True)
        if a.out:
            os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
            with open(a.out, "a") as fh:
                fh.write(json.dumps(row) + "\n")
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
