"""One forward + backward of each sequence-parallel linear: the [K, N] ("kn") fused input gradient against a transposed
weight copy + the [N, K] kernel, and against NCCL + cuBLAS.

  python bench/tp_backward.py                      # 1 GPU, world 1
  python -m torch.distributed.run --nproc-per-node 8 bench/tp_backward.py

Shapes (per rank P): tokens T, hidden H, FFN F.
  column (SeqParallelColumnLinear): x_r [T/P, H], W_r [F/P, H]; y = AG(x) W_r^T; dX_r = RS(dY W_r); dW_r = dY^T AG(x)
  row    (RowParallelLinear):       x_r [T, F/P], W_r [H, F/P]; y_r = RS(x_r W_r^T); dX_r = AG(dY_r) W_r; dW_r = AG(dY_r)^T x_r
Arms, each one forward + backward with the weight gradient a cuBLAS matmul:
  fused       the fused plugins, the input gradient reading W_r as [K, N] (w_layout="kn")
  transpose   the same, but the input gradient on W_r.t().contiguous() with the [N, K] kernel (a copy per step)
  nccl_cublas NCCL all_gather / reduce_scatter (a local copy at world 1) + cuBLAS matmuls
  layer       the fused arm through the autograd layers themselves (RowParallelLinear / SeqParallelColumnLinear)
The arms' outputs and gradients are compared before timing: fused and transpose must be bit-identical, nccl_cublas is
reported as a max abs difference.  Timing: CUDA events over --iters steps per arm, warm-up first, arms alternated over
--repeats rounds; the JSON row gives the median and the min-max spread per arm, with the card's name and power limit
read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import accl_b200 as A  # noqa: E402
from accl_b200.ops import all_gather_gemm, gemm_reduce_scatter  # noqa: E402
from accl_b200.parallel import RowParallelLinear, SeqParallelColumnLinear, TensorGroup  # noqa: E402


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
    ap.add_argument("--tokens", type=int, default=8192)
    ap.add_argument("--hidden", type=int, default=8192)
    ap.add_argument("--ffn", type=int, default=28672)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    T, H, F = a.tokens, a.hidden, a.ffn
    Fr, m = F // world, T // world
    dev = torch.device("cuda", local)
    heap_mb = 4 * (T * max(H, Fr) * 2 >> 20) + 512
    acc = A.cuda_rank(rank, world, local, heap_mb=heap_mb, max_ctas=32)
    acc.initialize(n_egr_rx_bufs=4, egr_rx_buf_size=16 << 10, max_egr_size=16 << 10, max_rndzv_size=1 << 30)
    group = TensorGroup(acc)
    col, row = SeqParallelColumnLinear(group, H, Fr), RowParallelLinear(group, Fr, H)
    g = torch.Generator(device=dev).manual_seed(11 + rank)
    x_col = torch.randn(m, H, device=dev, generator=g).bfloat16()          # column input shard
    dy_col = (torch.randn(T, Fr, device=dev, generator=g) * 0.1).bfloat16()
    x_row = (torch.randn(T, Fr, device=dev, generator=g) * 0.5).bfloat16()  # row input: the full sequence
    dy_row = (torch.randn(m, H, device=dev, generator=g) * 0.1).bfloat16()
    W1, W2 = col.weight.detach(), row.weight.detach()
    # heap operands of the explicit fused arms, allocated in the same order on every rank
    shard = acc.create_buffer(m * H, torch.bfloat16).dev.view(m, H)
    dxc = acc.create_buffer(m * H, torch.bfloat16)
    yr = acc.create_buffer(m * H, torch.bfloat16)
    dy_shard = acc.create_buffer(m * H, torch.bfloat16).dev.view(m, H)
    status = torch.zeros(1, dtype=torch.int32, device=dev)

    def fused(transpose):
        lay = "nk" if transpose else "kn"
        # column
        shard.copy_(x_col)
        y1, gathered = all_gather_gemm(acc, shard, W1, status=status)
        w1 = W1.t().contiguous() if transpose else W1
        gemm_reduce_scatter(acc, dy_col, w1, dxc, status=status, w_layout=lay)
        dw1 = dy_col.t() @ gathered
        # row
        gemm_reduce_scatter(acc, x_row, W2, yr, status=status)
        dy_shard.copy_(dy_row)
        w2 = W2.t().contiguous() if transpose else W2
        dx2, gdy = all_gather_gemm(acc, dy_shard, w2, status=status, w_layout=lay)
        dw2 = gdy.t() @ x_row
        return y1, dxc.dev.view(m, H), dw1, yr.dev.view(m, H), dx2, dw2

    def all_gather(t):
        if world == 1:
            return t.clone()
        out = torch.empty(t.shape[0] * world, *t.shape[1:], dtype=t.dtype, device=dev)
        dist.all_gather_into_tensor(out, t)
        return out

    def reduce_scatter(t):
        if world == 1:
            return t
        out = torch.empty(t.shape[0] // world, *t.shape[1:], dtype=t.dtype, device=dev)
        dist.reduce_scatter_tensor(out, t)
        return out

    def nccl_cublas():
        gathered = all_gather(x_col)
        y1 = gathered @ W1.t()
        dx1 = reduce_scatter(dy_col @ W1)
        dw1 = dy_col.t() @ gathered
        y2 = reduce_scatter(x_row @ W2.t())
        gdy = all_gather(dy_row)
        dx2 = gdy @ W2
        dw2 = gdy.t() @ x_row
        return y1, dx1, dw1, y2, dx2, dw2

    xc, xr = x_col.clone().requires_grad_(), x_row.clone().requires_grad_()

    def layer():
        col(xc).backward(dy_col)
        row(xr).backward(dy_row)

    arms = {"fused": lambda: fused(False), "transpose": lambda: fused(True), "nccl_cublas": nccl_cublas, "layer": layer}

    # ---- results agree before anything is timed
    names = ("y_col", "dx_col", "dw_col", "y_row", "dx_row", "dw_row")
    f = [t.clone() for t in fused(False)]
    t_ = [t.clone() for t in fused(True)]
    n = nccl_cublas()
    torch.cuda.synchronize()
    assert int(status.item()) == 0, f"fused status 0x{int(status.item()) & 0xffffffff:x}"
    identical = {k: bool(torch.equal(x, y)) for k, x, y in zip(names, f, t_)}
    assert all(identical.values()), f"kn and the transposed copy differ: {identical}"
    diff = {k: float((x.float() - y.float()).abs().max()) for k, x, y in zip(names, f, n)}
    scale = {k: float(y.float().abs().max()) for k, y in zip(names, n)}
    for p in (col.weight, row.weight):
        p.grad = None
    layer()
    torch.cuda.synchronize()
    group.check(block=True)
    layer_equal = all(bool(torch.equal(x, y)) for x, y in ((xc.grad, f[1]), (col.weight.grad, f[2]), (xr.grad, f[4]),
                                                           (row.weight.grad, f[5])))

    # ---- timing: warm-up, then rounds with the arms alternated
    def timed(fn):
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(a.iters):
            fn()
        e.record()
        torch.cuda.synchronize()
        ms = s.elapsed_time(e) / a.iters
        if world > 1:
            t = torch.tensor([ms], device=dev, dtype=torch.float64)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            ms = float(t.item())
        return ms

    for fn in arms.values():
        for _ in range(2):
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(a.repeats):
        for k, fn in arms.items():
            times[k].append(timed(fn))
    group.check(block=True)
    assert int(status.item()) == 0
    name, limit = card(local)
    if rank == 0:
        med = {k: statistics.median(v) for k, v in times.items()}
        flops = 2 * 2.0 * T * Fr * H * 3  # per layer: forward, input gradient, weight gradient
        row_ = dict(op="tp_backward", tokens=T, hidden=H, ffn=F, world=world, gpu=name, power_limit=limit,
                    iters=a.iters, repeats=a.repeats,
                    ms_median={k: round(v, 4) for k, v in med.items()},
                    ms_spread={k: [round(min(v), 4), round(max(v), 4)] for k, v in times.items()},
                    tflops_median={k: round(flops / v * 1e-9, 1) for k, v in med.items()},
                    fused_vs_transpose=round(med["transpose"] / med["fused"], 4),
                    fused_vs_nccl_cublas=round(med["nccl_cublas"] / med["fused"], 4),
                    kn_equals_transposed_copy=True, layer_equals_fused=layer_equal,
                    max_abs_diff_vs_nccl_cublas=diff, max_abs_nccl_cublas=scale)
        print(json.dumps(row_), flush=True)
        if a.out:
            os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
            with open(a.out, "a") as fh:
                fh.write(json.dumps(row_) + "\n")
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
