"""Worker of the multi-process alltoallv tests (tests/test_alltoallv.py, tests/test_cuda_alltoallv.py): one process
per rank on the "accl" torch.distributed backend; uneven all_to_all_single, then the raw alltoallv in four dtypes."""
import faulthandler, os, sys
faulthandler.dump_traceback_later(int(os.environ.get("PG_WATCHDOG_S", 90)), exit=True)  # a hang prints where, then exits
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch, torch.distributed as dist
import accl_b200.parallel.process_group  # noqa
import accl_b200.parallel  # noqa
import accl_b200 as A  # noqa: E402
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
use_cuda = torch.cuda.is_available() and A._C.with_cuda and A._C.cuda_driver_available()
dev = "cpu"
if use_cuda:
    os.environ["LOCAL_RANK"] = str(int(os.environ.get("LOCAL_RANK", rank)) % torch.cuda.device_count())  # ranks may share a GPU
    torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
    dev = torch.device("cuda", int(os.environ["LOCAL_RANK"]))
port = os.environ.get("PG_PORT") or str(int(os.environ.get("MASTER_PORT", 29500)) + 7)
if "TORCHELASTIC_RUN_ID" in os.environ:
    dist.init_process_group("accl", init_method="env://", rank=rank, world_size=world)
else:
    dist.init_process_group("accl", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)


def rows(p, q):  # rows rank p sends to rank q (zeros included)
    return (3 * p + 5 * q + 1) % 4


hidden = 3
for dtype in (torch.float32, torch.bfloat16):
    in_splits = [rows(rank, q) for q in range(world)]
    out_splits = [rows(p, rank) for p in range(world)]
    inp = torch.cat([torch.full((rows(rank, q), hidden), 100.0 * rank + q) for q in range(world)]).to(dtype).to(dev)
    out = torch.full((sum(out_splits), hidden), -1.0, dtype=dtype, device=dev)
    dist.all_to_all_single(out, inp, out_splits, in_splits)
    ref = torch.cat([torch.full((rows(p, rank), hidden), 100.0 * p + rank) for p in range(world)]).to(dtype)
    assert torch.equal(out.cpu(), ref), (out, ref)
    # one side even, the other given
    even = torch.arange(2 * world * hidden, dtype=dtype, device=dev).view(2 * world, hidden) + 1000 * rank
    got = torch.empty_like(even)
    dist.all_to_all_single(got, even, [2] * world, [])
    ref = torch.cat([torch.arange(2 * world * hidden, dtype=torch.float32).view(2 * world, hidden)[2 * rank:2 * rank + 2] + 1000 * p
                     for p in range(world)]).to(dtype)
    assert torch.equal(got.cpu(), ref)
# rank 0 sends nothing (input of zero rows) but receives from everybody
zin = [0] * world if rank == 0 else [rank + q for q in range(world)]
zout = [0 if p == 0 else p + rank for p in range(world)]
inp = torch.cat([torch.full((zin[q], hidden), 10.0 * rank + q) for q in range(world)]).reshape(-1, hidden).to(dev)
out = torch.full((sum(zout), hidden), -1.0, device=dev)
dist.all_to_all_single(out, inp, zout, zin)
ref = torch.cat([torch.full((zout[p], hidden), 10.0 * p + rank) for p in range(world)]).reshape(-1, hidden)
assert torch.equal(out.cpu(), ref), (out, ref)

# the raw alltoallv on this rank's engine, one process per rank: seeded matrices in four dtypes
acc = accl_b200.parallel.process_group._primary["accl"]
for i, dt in enumerate((torch.int8, torch.float16, torch.float32, torch.int64)):
    g = torch.Generator().manual_seed(99 + i)
    m = torch.randint(0, 40, (world, world), generator=g)
    m[i % world, :] = 0
    scap, rcap = int(m[rank].sum()) + 3, int(m[:, rank].sum()) + 1
    s, d, cnt = acc.create_buffer(scap, dt), acc.create_buffer(rcap, dt), acc.create_buffer(2 * world, torch.int64)
    src = [torch.randint(-100, 100, (int(m[p].sum()) + 3,), generator=torch.Generator().manual_seed(7 * p + i)).to(dt) for p in range(world)]
    counts = torch.cat([m[rank], m[:, rank]]).to(torch.int64)
    if acc.is_cuda:
        s.dev.copy_(src[rank].to(dev)); cnt.dev.copy_(counts.to(dev))
        acc.alltoallv(s, d, cnt, from_fpga=True, to_fpga=True)
        torch.cuda.current_stream().synchronize()
        got = d.dev.cpu()
    else:
        s.host[:] = src[rank]; cnt.host[:] = counts
        acc.alltoallv(s, d, cnt)
        got = d.host.clone()
    n = int(m[:, rank].sum())
    ref = torch.cat([src[p][int(m[p, :rank].sum()):int(m[p, :rank + 1].sum())] for p in range(world)])
    assert torch.equal(got[:n], ref), (dt, got[:n], ref)
dist.barrier()
print(f"a2av rank {rank}: ok", flush=True)
dist.destroy_process_group()
