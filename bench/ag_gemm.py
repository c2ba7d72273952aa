"""All-gather -> GEMM: fused wgmma plugin vs NCCL all_gather_into_tensor + cuBLAS matmul.

  python bench/ag_gemm.py --check                 # 1 GPU: fused kernel vs copy + cuBLAS, and vs gemm_reduce_scatter
  python -m torch.distributed.run --nproc-per-node N ... bench/ag_gemm.py --gm 8192 --gn 8192 --gk 8192

Per rank: A_r [M/P, K] (its rows of the activations, in the symmetric heap) and W_r [N, K] bf16; result:
C [M, N] = all_gather_M(A_r) W_r^T, plus the gathered [M, K].  Reports device-timed ms (CUDA events, max over ranks),
TFLOP/s per GPU and the fraction of the roofline max(FLOPs / BF16_PEAK, NVLink bytes / LINK_BPS).  Both peaks are
NVIDIA's H100 SXM data-sheet figures (700 W, dense bf16; NVLink 4 per direction), not measurements: a card with a lower
power limit or clock reaches less.  The card's name and power limit are read in the same run and printed with the result.

At one rank the fused kernel runs the same mainloop as the single-CTA GEMM -> reduce-scatter kernel (variant 1) at the
same shape, which is timed in the same process as the reference for the fused kernel's own overheads (the local copy
into `gathered` against the shard zeroing of the reduce-scatter).
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
from accl_b200.ops import all_gather_gemm, gemm_reduce_scatter  # noqa: E402


def card(local):
    """Name and power limit of this GPU, read now (a number is only worth something with what it was measured on)."""
    name, limit = torch.cuda.get_device_name(local), None
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(local), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        if q.returncode == 0 and q.stdout.strip():
            name, limit = (v.strip() for v in q.stdout.strip().split(",", 1))
    except (OSError, subprocess.SubprocessError):
        pass
    return name, limit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gm", dest="m", type=int, default=8192, help="M over all ranks")
    ap.add_argument("--gn", dest="n", type=int, default=8192, help="N of this rank")
    ap.add_argument("--gk", dest="k", type=int, default=8192)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--check", action="store_true", help="compare the fused result with the unfused one")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    M, N, K = a.m, a.n, a.k
    heap_mb = (M // world * K * 2 >> 20) + 1 + ((M * N * 2 >> 20) + 1 if world == 1 else 0)
    acc = A.cuda_rank(rank, world, local, heap_mb=max(512, heap_mb + 384), max_ctas=32)
    acc.initialize(n_egr_rx_bufs=4, egr_rx_buf_size=16 << 10, max_egr_size=16 << 10, max_rndzv_size=1 << 30)

    g = torch.Generator(device="cuda").manual_seed(7 + rank)
    shard_buf = acc.create_buffer(M // world * K, torch.bfloat16)
    shard = shard_buf.dev.view(M // world, K)
    shard.copy_(torch.randn(M // world, K, device="cuda", generator=g) * 0.25)
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.25).bfloat16()
    out = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    gathered = torch.empty(M, K, dtype=torch.bfloat16, device="cuda")
    ref_out = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    ref_gathered = torch.empty(M, K, dtype=torch.bfloat16, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")

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
        all_gather_gemm(acc, shard, w, out=out, gathered=gathered, status=status)

    def baseline():
        if world > 1:
            dist.all_gather_into_tensor(ref_gathered, shard)
        else:
            ref_gathered.copy_(shard)
        torch.matmul(ref_gathered, w.t(), out=ref_out)

    ms_f = timed(fused, a.iters)
    ms_b = timed(baseline, a.iters)
    ms_rs = None
    if world == 1:
        rs_out = acc.create_buffer(M * N, torch.bfloat16)
        ms_rs = timed(lambda: gemm_reduce_scatter(acc, shard, w, rs_out, variant=1), a.iters)
    flops = 2.0 * M * N * K
    nvlink_bytes = M // world * K * 2 * (world - 1)  # peers' shards pulled into this GPU
    t_roof = max(flops / BF16_PEAK, nvlink_bytes / LINK_BPS) * 1e3
    err = gathered_equal = None
    if a.check:
        status.fill_(-1)
        fused()
        baseline()
        torch.cuda.synchronize()
        assert int(status.item()) == 0, f"all_gather_gemm status 0x{int(status.item()) & 0xffffffff:x}"
        gathered_equal = bool(torch.equal(gathered, ref_gathered))
        err = float((out.float() - ref_out.float()).abs().max())
    name, limit = card(local)
    if rank == 0:
        row = dict(op="all_gather_gemm", m=M, n_per_rank=N, k=K, world=world, gpu=name, power_limit=limit,
                   fused_ms=ms_f, nccl_cublas_ms=ms_b, gemm_rs_v1_world1_ms=ms_rs,
                   fused_tflops=flops / ms_f * 1e-9, nccl_cublas_tflops=flops / ms_b * 1e-9,
                   gemm_rs_v1_tflops=flops / ms_rs * 1e-9 if ms_rs else None,
                   fused_vs_gemm_rs_v1=ms_f / ms_rs if ms_rs else None,
                   speedup_vs_nccl_cublas=ms_b / ms_f, roofline_ms=t_roof, frac_of_roofline=t_roof / ms_f,
                   peak_source="H100 SXM data sheet (700 W)", bf16_peak_tflops=BF16_PEAK * 1e-12, link_GBps=LINK_BPS * 1e-9,
                   max_abs_err_vs_nccl_cublas=err, gathered_equal=gathered_equal)
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
