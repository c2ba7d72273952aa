"""GPU tests of alltoallv on the CUDA backend (rvb_alltoallv, csrc/src/cuda/collectives.cuh): seeded uneven count
matrices from a few bytes to several MiB per peer, aligned and unaligned block offsets, direct launches and the
persistent engine, zero-copy and staged torch tensors (TensorGroup.all_to_all_v, also asynchronous calls followed by a barrier), the
MoE dispatch / combine round trip, CUDA-graph replay with counts rewritten on the device,
all-or-nothing rejection of inconsistent counts, and the "accl" torch.distributed backend with uneven splits.
Ranks share cuda:0 when the box has one GPU (few channels, so that their kernels are co-resident).  A rank waits for
its own stream only: a device-wide synchronise would also wait for the peers' kernels, which wait for this rank."""
import os
import random
import subprocess
import sys
import threading

import numpy as np
import pytest
import torch

import accl_b200 as A
from accl_b200.parallel import TensorGroup
from accl_b200.parallel.strategies import moe_combine_v, moe_dispatch_v

pytestmark = pytest.mark.gpu
NGPU = torch.cuda.device_count() if torch.cuda.is_available() else 0
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG = dict(n_egr_rx_bufs=4, egr_rx_buf_size=16 << 10, max_egr_size=64 << 10, max_rndzv_size=1 << 30)
SENTINEL = 77


def run(world, fn, engine=False, shared=True, heap_mb=256):
    devs = [0] * world if shared else list(range(world))
    opts = dict(heap_mb=heap_mb, max_ctas=4, engine=engine)
    if engine:
        opts["engine_workers"] = 4
    return A.run_cuda_ranks(devs, fn, CFG, **opts)


def count_matrix(world, seed, sizes):
    g = np.random.default_rng(seed)
    m = g.choice(np.array(sizes, dtype=np.int64), size=(world, world))
    m[seed % world, :] = 0   # one rank sends nothing
    return m


def payload(n, rank, dtype, salt=0):
    g = torch.Generator().manual_seed(8765 + 31 * rank + salt)
    return torch.randint(-100, 100, (max(n, 1),), generator=g).to(dtype)[:n]


def expected(m, r, scap, rcap, dtype, salt=0):
    out = torch.full((rcap[r],), SENTINEL, dtype=dtype)
    off = 0
    for p in range(m.shape[0]):
        s0 = int(m[p, :r].sum())
        out[off:off + m[p, r]] = payload(scap[p], p, dtype, salt)[s0:s0 + m[p, r]]
        off += int(m[p, r])
    return out


def one_call(a, m, r, scap, rcap, dtype, salt=0):
    w = m.shape[0]
    dev = a.cuda_device
    s, d, cnt = a.create_buffer(scap[r], dtype), a.create_buffer(rcap[r], dtype), a.create_buffer(2 * w, torch.int64)
    s.dev.copy_(payload(scap[r], r, dtype, salt).cuda(dev))
    d.dev.fill_(SENTINEL)
    cnt.dev.copy_(torch.from_numpy(np.concatenate([m[r], m[:, r]]).astype(np.int64)).cuda(dev))
    a.alltoallv(s, d, cnt, from_fpga=True, to_fpga=True)
    torch.cuda.current_stream(dev).synchronize()
    assert torch.equal(d.dev.cpu(), expected(m, r, scap, rcap, dtype, salt)), (r, dtype, salt)


# sizes in elements: a few bytes up to several MiB per peer (fp32: 3 MiB = 786432), odd counts put blocks at unaligned offsets
SMALL = [0, 1, 3, 17, 1000]
LARGE = [0, 5, 4096, 65537, 786432]


@pytest.mark.parametrize("engine", [False, True], ids=["direct", "engine"])
@pytest.mark.parametrize("world", [2, 3, 4])
def test_alltoallv_shared_gpu(world, engine):
    def fn(a, r, w):
        for i, (sizes, dtype) in enumerate([(SMALL, torch.int8), (SMALL, torch.float16), (LARGE, torch.float32),
                                            ([0, 4, 64, 4096], torch.float32), (LARGE, torch.int8)]):
            m = count_matrix(w, 10 * w + i, sizes)
            scap = [int(m[p].sum()) + 3 * p + 1 for p in range(w)]     # a different capacity on every rank
            rcap = [int(m[:, p].sum()) + 5 * p + 2 for p in range(w)]
            one_call(a, m, r, scap, rcap, dtype, salt=i)
        a.barrier()
    run(world, fn, engine)


@pytest.mark.multigpu
@pytest.mark.parametrize("engine", [False, True], ids=["direct", "engine"])
def test_alltoallv_one_rank_per_gpu(engine):
    world = min(NGPU, 8)

    def fn(a, r, w):
        for i, (sizes, dtype) in enumerate([(SMALL, torch.int8), (LARGE, torch.float32), (LARGE, torch.bfloat16)]):
            m = count_matrix(w, 100 + i, sizes)
            scap = [int(m[p].sum()) + p for p in range(w)]
            rcap = [int(m[:, p].sum()) + 2 * p for p in range(w)]
            one_call(a, m, r, scap, rcap, dtype, salt=i)
    A.run_cuda_ranks(list(range(world)), fn, CFG, heap_mb=512, max_ctas=32, engine=engine,
                     **({"engine_workers": 32} if engine else {}))


@pytest.mark.parametrize("engine", [False, True], ids=["direct", "engine"])
@pytest.mark.parametrize("kind", ["mismatch", "negative", "send_capacity", "recv_capacity"])
def test_alltoallv_invalid_counts(kind, engine):
    world = 3

    def fn(a, r, w):
        dev = a.cuda_device
        m = np.array([[4, 9, 2], [7, 1, 5], [3, 6, 8]], dtype=np.int64)
        scap = [int(m[p].sum()) for p in range(w)]
        rcap = [int(m[:, p].sum()) for p in range(w)]
        send, recv = m[r].copy(), m[:, r].copy()
        if kind == "mismatch" and r == 0:
            send[1] += 1
            scap[0] += 1
        if kind == "negative":
            if r == 1:
                send[2] = -2
            if r == 2:
                recv[1] = -2
        if kind == "send_capacity":
            scap[2] -= 1
        if kind == "recv_capacity":
            rcap[1] -= 1
        s, d, cnt = a.create_buffer(scap[r]), a.create_buffer(rcap[r]), a.create_buffer(2 * w, torch.int64)
        s.dev.copy_(payload(scap[r], r, torch.float32).cuda(dev))
        d.dev.fill_(SENTINEL)
        cnt.dev.copy_(torch.from_numpy(np.concatenate([send, recv])).cuda(dev))
        with pytest.raises(RuntimeError, match="DMA_SIZE_ERROR"):
            a.alltoallv(s, d, cnt, from_fpga=True, to_fpga=True)
        torch.cuda.current_stream(dev).synchronize()
        assert torch.all(d.dev == SENTINEL).item(), f"rank {r}: a rejected call wrote the receive buffer"
        # the next valid call on the same communicator
        scap = [int(m[p].sum()) for p in range(w)]
        rcap = [int(m[:, p].sum()) for p in range(w)]
        one_call(a, m, r, scap, rcap, torch.float32)
    run(world, fn, engine)


def test_alltoallv_cuda_graph_replay_with_new_counts():
    world, cap = 3, 4096
    # capturing synchronises the whole device: nobody replays (a kernel waiting for the peers) before all have captured
    captured = threading.Barrier(world)

    def fn(a, r, w):
        dev = a.cuda_device
        s, d, cnt = a.create_buffer(cap), a.create_buffer(cap), a.create_buffer(2 * w, torch.int64)
        st = torch.cuda.Stream(dev)
        with torch.cuda.stream(st):
            m0 = count_matrix(w, 0, [1, 2, 3])
            cnt.dev.copy_(torch.from_numpy(np.concatenate([m0[r], m0[:, r]])).cuda(dev))
            a.alltoallv(s, d, cnt, from_fpga=True, to_fpga=True, run_async=True).free()   # warm-up outside the graph
            st.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=st, capture_error_mode="thread_local"):
                a.alltoallv(s, d, cnt, from_fpga=True, to_fpga=True, run_async=True).free()
            captured.wait()
            for it in range(4):
                m = count_matrix(w, 50 + it, [0, 1, 33, 300, 1000])
                s.dev.copy_(payload(cap, r, torch.float32, salt=it).cuda(dev))   # rewritten on the device
                d.dev.fill_(SENTINEL)
                cnt.dev.copy_(torch.from_numpy(np.concatenate([m[r], m[:, r]])).cuda(dev))
                g.replay()
                st.synchronize()
                assert torch.equal(d.dev.cpu(), expected(m, r, [cap] * w, [cap] * w, torch.float32, salt=it)), it
        a.barrier()
    run(world, fn)


@pytest.mark.parametrize("engine", [False, True], ids=["direct", "engine"])
def test_tensor_group_zero_copy_and_staged(engine):
    world = 3

    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        grp = TensorGroup(a)
        m = count_matrix(w, 7, [0, 1, 9, 1000, 20000])
        sc, rc = [int(m[p].sum()) for p in range(w)], [int(m[:, p].sum()) + 4 for p in range(w)]
        sends = torch.from_numpy(m[r].copy()).to(dev)
        recvs = torch.from_numpy(m[:, r].copy()).to(dev)
        for heap in (True, False):
            inp = grp.empty(sc[r], dtype=torch.bfloat16) if heap else torch.empty(sc[r], dtype=torch.bfloat16, device=dev)
            out = grp.empty(rc[r], dtype=torch.bfloat16) if heap else torch.empty(rc[r], dtype=torch.bfloat16, device=dev)
            inp.copy_(payload(sc[r], r, torch.bfloat16).to(dev))
            out.fill_(SENTINEL)
            grp.all_to_all_v(out, inp, sends, recvs)
            grp.check(block=True)
            torch.cuda.current_stream(dev).synchronize()
            n = int(m[:, r].sum())   # (a staged output's tail beyond the received blocks is not defined)
            assert torch.equal(out[:n].cpu(), expected(m, r, sc, rc, torch.bfloat16)[:n]), ("heap" if heap else "staged")
        # several asynchronous calls back to back, then a barrier right away
        outs = []
        for i in range(4):
            inp = torch.empty(sc[r], dtype=torch.bfloat16, device=dev)
            inp.copy_(payload(sc[r], r, torch.bfloat16, salt=i).to(dev))
            outs.append(torch.full((rc[r],), SENTINEL, dtype=torch.bfloat16, device=dev))
            grp.all_to_all_v(outs[-1], inp, sends, recvs)
        a.barrier()
        grp.check(block=True)
        torch.cuda.current_stream(dev).synchronize()
        n = int(m[:, r].sum())
        for i, out in enumerate(outs):
            assert torch.equal(out[:n].cpu(), expected(m, r, sc, rc, torch.bfloat16, salt=i)[:n]), ("async", i)
    run(world, fn, engine)


@pytest.mark.parametrize("engine", [False, True], ids=["direct", "engine"])
def test_moe_dispatch_combine_v_round_trip(engine):
    world, hidden, tokens = 3, 64, 40

    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        grp = TensorGroup(a)
        dests = [torch.randint(0, w, (tokens,), generator=torch.Generator().manual_seed(p)) for p in range(w)]
        dests[1][:] = 0                                                        # rank 1 routes everything to rank 0
        rows = torch.stack([torch.bincount(d, minlength=w) for d in dests])     # rows[p, q]: p routes to q
        x = torch.randn(tokens, hidden, generator=torch.Generator().manual_seed(100 + r))[torch.argsort(dests[r], stable=True)].to(dev)
        send_counts = rows[r].to(dev)
        for step in range(2):
            recv, recv_counts = moe_dispatch_v(grp, x, send_counts, capacity=tokens * w)
            back = moe_combine_v(grp, recv * 3, recv_counts, send_counts, tokens)
            grp.check(block=True)
            torch.cuda.current_stream(dev).synchronize()
            assert torch.equal(recv_counts.cpu(), rows[:, r]), (step, recv_counts, rows[:, r])
            assert torch.equal(back.cpu(), (x * 3).cpu()), step
        a.barrier()
    run(world, fn, engine)


@pytest.mark.parametrize("mode", ["direct", "engine"])
def test_torch_distributed_all_to_all_single_uneven_on_gpus(mode):
    world = 2
    env = dict(os.environ, PG_PORT=str(random.randint(20000, 30000)), CUDA_DEVICE_MAX_CONNECTIONS="32",
               ACCL_PG_ENGINE="1" if mode == "engine" else "0", ACCL_MAX_CTAS="4")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr",
                        "127.0.0.1", "--master-port", str(random.randint(30001, 40000)),
                        os.path.join(ROOT, "tests", "helpers", "a2av_worker.py")], cwd=ROOT, env=env, capture_output=True,
                       text=True, timeout=200)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert r.stdout.count(": ok") == world
