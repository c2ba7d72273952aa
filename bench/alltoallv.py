"""alltoallv against NCCL's all_to_all_single on the same uneven splits, one rank per GPU.

    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 --master-port 29531 \
        bench/alltoallv.py [--tokens 8192] [--hidden 4096] [--iters 50] [--warmup 10]

Workloads (bf16 rows of `hidden`):
  * moe   dropless MoE dispatch: every rank routes `tokens` tokens top-2 over P expert ranks with seeded, skewed
          router probabilities, so the blocks differ per pair and some ranks receive far more than others;
  * even  the same number of rows to every rank (what `alltoall` covers), for comparison.
Both libraries move the same splits; their outputs are compared bit for bit before any number is printed.  Times
are CUDA events over `iters` back-to-back calls after `warmup`, max over ranks.  algbw = bytes a rank sends
(its own block included) / time; bytes_out = what leaves the GPU (own block excluded), max over ranks.  The card
name and power limit are read in the same run and written with the numbers to results/alltoallv_<P>.json.
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def splits(workload, rank, world, tokens, seed=0):
    """Rows this rank sends to each rank."""
    if workload == "even":
        return [2 * tokens // world] * world
    g = torch.Generator().manual_seed(seed + 1000 * rank)
    skew = torch.linspace(2.0, 0.0, world)                        # lower expert ranks are hotter
    logits = torch.randn(tokens, world, generator=g) + skew
    top2 = logits.topk(min(2, world), dim=1).indices.reshape(-1)
    return torch.bincount(top2, minlength=world).tolist()


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    dist.barrier()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    t = torch.tensor([a.elapsed_time(b) / iters], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return t.item()


def card(local):
    out = subprocess.run(["nvidia-smi", "-i", str(local), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    name, _, power = out.partition(",")
    return name.strip(), power.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=8192, help="tokens per rank (each routed to 2 experts)")
    ap.add_argument("--hidden", type=int, default=4096)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default="results")
    args = ap.parse_args()
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    from accl_b200.parallel import TensorGroup, init_from_env
    acc = init_from_env("cuda")
    grp = TensorGroup(acc)
    name, power = card(local)
    rows_out = []
    for workload in ("moe", "even"):
        send = splits(workload, rank, world, args.tokens)
        send_t = torch.tensor(send, dtype=torch.int64, device=dev)
        recv_t = torch.empty_like(send_t)
        dist.all_to_all_single(recv_t, send_t)                       # the receivers' row counts
        recv = recv_t.tolist()
        h = args.hidden
        g = torch.Generator(device="cpu").manual_seed(rank)
        inp = grp.empty(sum(send) * h, dtype=torch.bfloat16).view(sum(send), h)    # zero-copy operand in the heap
        inp.copy_(torch.randn(sum(send), h, generator=g).to(torch.bfloat16))
        out_accl = grp.empty(sum(recv) * h, dtype=torch.bfloat16).view(sum(recv), h)
        out_nccl = torch.empty(sum(recv), h, dtype=torch.bfloat16, device=dev)
        sc, rc = send_t * h, recv_t * h
        out_accl.zero_()
        grp.all_to_all_v(out_accl.view(-1), inp.view(-1), sc, rc)
        dist.all_to_all_single(out_nccl, inp, recv, send)
        grp.check(block=True)
        torch.cuda.synchronize()
        same = torch.tensor([int(torch.equal(out_accl, out_nccl))], device=dev)
        dist.all_reduce(same, op=dist.ReduceOp.MIN)
        if not same.item():
            raise SystemExit(f"{workload}: accl and nccl outputs differ")
        ms_accl = timed(lambda: grp.all_to_all_v(out_accl.view(-1), inp.view(-1), sc, rc), args.iters, args.warmup)
        grp.check(block=True)
        ms_nccl = timed(lambda: dist.all_to_all_single(out_nccl, inp, recv, send), args.iters, args.warmup)
        esz = 2 * h
        sent = torch.tensor([sum(send) * esz, (sum(send) - send[rank]) * esz], dtype=torch.float64, device=dev)
        dist.all_reduce(sent, op=dist.ReduceOp.MAX)
        for impl, ms in (("accl", ms_accl), ("nccl", ms_nccl)):
            row = dict(impl=impl, workload=workload, world=world, hidden=h, tokens_per_rank=args.tokens, dtype="bfloat16",
                       us=ms * 1e3, algbw_GBps=sent[0].item() / ms * 1e-6, bytes_out_per_gpu=int(sent[1].item()),
                       out_GBps=sent[1].item() / ms * 1e-6, bit_identical=True, card=name, power_limit=power)
            rows_out.append(row)
            if rank == 0:
                print(json.dumps(row), flush=True)
    if rank == 0:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, f"alltoallv_{world}.json"), "w") as f:
            json.dump(rows_out, f, indent=1)
    acc.deinit()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
