"""alltoallv (uneven all-to-all, per-peer counts in engine memory) on the CPU emulator: seeded count matrices
checked bit for bit against a Python reference, all-or-nothing rejection of inconsistent counts, the CUDA
planner's decisions for it, the torch front ends (TensorGroup, MoE dispatch / combine, the "accl"
torch.distributed backend)."""
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

import accl_b200 as A
from accl_b200.parallel import TensorGroup
from accl_b200.parallel.strategies import moe_combine_v, moe_dispatch_v

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EAGER = dict(n_egr_rx_bufs=16, egr_rx_buf_size=1024, max_egr_size=1 << 20, max_rndzv_size=1 << 24)
RNDZV = dict(n_egr_rx_bufs=16, egr_rx_buf_size=64, max_egr_size=64, max_rndzv_size=32 * 1024)
PROTOCOLS = [pytest.param(EAGER, id="eager"), pytest.param(RNDZV, id="rndzv")]
DTYPES = [torch.int8, torch.float16, torch.float32, torch.int64]
SENTINEL = 77


def count_matrix(world, seed, max_blk=60):
    """m[p, q] = elements rank p sends to rank q: zeros, 1-element blocks, odd sizes, one rank sending nothing."""
    g = np.random.default_rng(seed)
    m = g.integers(2, max_blk, size=(world, world))
    m[g.random((world, world)) < 0.25] = 0
    m[g.random((world, world)) < 0.15] = 1
    if world > 1:
        m[seed % world, :] = 0
    return m


def payload(n, rank, dtype, salt=0):
    g = torch.Generator().manual_seed(4321 + 31 * rank + salt)
    return torch.randint(-100, 100, (max(n, 1),), generator=g).to(dtype)[:n]


def capacities(m, seed):
    """Send / receive capacities per rank: the counts' sums plus a different slack on every rank."""
    g = np.random.default_rng(seed + 99)
    w = m.shape[0]
    return [int(m[r].sum()) + int(g.integers(1, 9)) for r in range(w)], [int(m[:, r].sum()) + int(g.integers(1, 9)) for r in range(w)]


def expected(m, r, scap, rcap, dtype, salt=0):
    w = m.shape[0]
    out = torch.full((rcap[r],), SENTINEL, dtype=dtype)
    off = 0
    for p in range(w):
        src = payload(scap[p], p, dtype, salt)
        s0 = int(m[p, :r].sum())
        out[off:off + m[p, r]] = src[s0:s0 + m[p, r]]
        off += int(m[p, r])
    return out


def setup_rank(a, m, r, scap, rcap, dtype, salt=0):
    w = m.shape[0]
    s, d = a.create_buffer(scap[r], dtype), a.create_buffer(rcap[r], dtype)
    cnt = a.create_buffer(2 * w, torch.int64)
    s.host[:] = payload(scap[r], r, dtype, salt)
    d.host[:] = SENTINEL
    d.sync_to_device()   # the receive buffer's untouched tail must read back as the sentinel
    cnt.host[:w] = torch.from_numpy(m[r].astype(np.int64))
    cnt.host[w:] = torch.from_numpy(m[:, r].astype(np.int64))
    return s, d, cnt


@pytest.mark.parametrize("cfg", PROTOCOLS)
@pytest.mark.parametrize("world", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("dtype", DTYPES)
def test_alltoallv_matrix(cfg, world, dtype):
    seed = world * 7 + DTYPES.index(dtype)
    m = count_matrix(world, seed)
    scap, rcap = capacities(m, seed)

    def fn(a, r, w):
        s, d, cnt = setup_rank(a, m, r, scap, rcap, dtype)
        a.alltoallv(s, d, cnt)
        assert torch.equal(d.host, expected(m, r, scap, rcap, dtype)), f"rank {r}"
        # the same buffers again with the transposed matrix: counts are read per call
        mt = m.T.copy()
        s2, d2, cnt2 = setup_rank(a, mt, r, [int(x) for x in rcap], [int(x) for x in scap], dtype, salt=1)
        a.alltoallv(s2, d2, cnt2)
        assert torch.equal(d2.host, expected(mt, r, rcap, scap, dtype, salt=1))
    A.run_ranks(world, fn, cfg)


def test_alltoallv_one_hop_schedules():
    m = count_matrix(4, 3)
    scap, rcap = capacities(m, 3)

    def fn(a, r, w):
        a.set_one_hop_schedules(True)
        s, d, cnt = setup_rank(a, m, r, scap, rcap, torch.float32)
        a.alltoallv(s, d, cnt)
        assert torch.equal(d.host, expected(m, r, scap, rcap, torch.float32))
    A.run_ranks(4, fn, RNDZV)


@pytest.mark.parametrize("cfg", PROTOCOLS)
def test_alltoallv_sub_communicator(cfg):
    group = [0, 2, 3]
    m = count_matrix(3, 11)
    scap, rcap = capacities(m, 11)

    def fn(a, r, w):
        ranks = A.Accl.generate_ranks(w)
        if r not in group:
            a.barrier()
            return
        comm = a.create_communicator([ranks[g] for g in group], group.index(r))
        me = group.index(r)
        s, d, cnt = setup_rank(a, m, me, scap, rcap, torch.float32)
        a.alltoallv(s, d, cnt, comm_id=comm)
        assert torch.equal(d.host, expected(m, me, scap, rcap, torch.float32))
        a.barrier()
    A.run_ranks(4, fn, cfg)


def _break(kind, m, scap, rcap):
    m, scap, rcap = m.copy(), list(scap), list(rcap)
    if kind == "mismatch":       # rank 0 sends one more element to rank 1 than rank 1 expects
        m_send = m.copy()
        m_send[0, 1] += 1
        scap[0] += 1             # rank 0's own checks pass: only the matrix shows the disagreement
        return m_send, m, scap, rcap
    if kind == "negative":       # consistent on both sides, but negative
        m[1, 2] = -3
    elif kind == "send_capacity":
        scap[2] = int(m[2].sum()) - 1
    elif kind == "recv_capacity":
        rcap[1] = int(m[:, 1].sum()) - 1
    return m, m, scap, rcap


@pytest.mark.parametrize("cfg", PROTOCOLS)
@pytest.mark.parametrize("kind", ["mismatch", "negative", "send_capacity", "recv_capacity"])
def test_alltoallv_invalid_counts(cfg, kind):
    world = 3
    m = count_matrix(world, 5, max_blk=30)
    m[m == 0] = 2  # every block non-empty: a write anywhere would show in the sentinel check
    scap, rcap = capacities(m, 5)
    m_send, m_recv, bscap, brcap = _break(kind, m, scap, rcap)
    bscap = [max(c, 1) for c in bscap]
    brcap = [max(c, 1) for c in brcap]

    def fn(a, r, w):
        s, d = a.create_buffer(bscap[r], torch.float32), a.create_buffer(brcap[r], torch.float32)
        cnt = a.create_buffer(2 * w, torch.int64)
        s.host[:] = payload(bscap[r], r, torch.float32)
        d.host[:] = SENTINEL
        d.sync_to_device()
        cnt.host[:w] = torch.from_numpy(m_send[r].astype(np.int64))
        cnt.host[w:] = torch.from_numpy(m_recv[:, r].astype(np.int64))
        with pytest.raises(RuntimeError, match="DMA_SIZE_ERROR"):
            a.alltoallv(s, d, cnt)
        d.sync_from_device()
        assert torch.all(d.host == SENTINEL), f"rank {r}: receive buffer written by a rejected call"
        # the communicator is usable right after
        s2, d2, cnt2 = setup_rank(a, m, r, scap, rcap, torch.float32)
        a.alltoallv(s2, d2, cnt2)
        assert torch.equal(d2.host, expected(m, r, scap, rcap, torch.float32))
    A.run_ranks(world, fn, cfg)


def test_alltoallv_host_checks():
    def fn(a, r, w):
        s, d = a.create_buffer(8), a.create_buffer(8)
        with pytest.raises(ValueError):
            a.alltoallv(s, d, a.create_buffer(2 * w, torch.int32))      # counts must be int64
        with pytest.raises(ValueError):
            a.alltoallv(s, d, a.create_buffer(2 * w - 1, torch.int64))  # at least 2P of them
        with pytest.raises(ValueError):
            a.alltoallv(s, a.create_buffer(8, torch.float16), a.create_buffer(2 * w, torch.int64))
        # 1-byte payloads are moved by alltoallv only: an int8 reduction is still refused on the host
        x, y = a.create_buffer(8, torch.int8), a.create_buffer(8, torch.int8)
        with pytest.raises(IndexError):
            a.allreduce(x, y, 8)
        with pytest.raises(IndexError):
            a.reduce_scatter(x, y, 4)
    A.run_ranks(2, fn, EAGER)


# ------------------------------------------------------------------ planner
@pytest.mark.skipif(not A._C.with_cuda, reason="built without the CUDA backend")
@pytest.mark.parametrize("world", [1, 2, 5, 8])
@pytest.mark.parametrize("max_ctas", [4, 8, 128])
@pytest.mark.parametrize("engine_mode", [False, True])
def test_plan_alltoallv(world, max_ctas, engine_mode):
    Op = A._C.Operation
    plans = [A._C.cuda_plan(Op.alltoallv, n, A.DataType.float32, world, max_ctas=max_ctas, engine_mode=engine_mode)
             for n in (0, 1, 100, 16 << 10, 1 << 20, (1 << 32) - 1)]
    assert all(p["algo"] == "p2p" for p in plans)                 # never NVLS, never the slot ring or staged exchanges
    assert len({p["n_ctas"] for p in plans}) == 1                  # the receive capacity differs per rank: not a factor
    assert plans[0]["n_ctas"] == max_ctas


# ------------------------------------------------------------- torch layers
def test_tensor_group_all_to_all_v():
    world = 3
    m = count_matrix(world, 21)

    def fn(a, r, w):
        g = TensorGroup(a)
        inp = payload(int(m[r].sum()), r, torch.float32)
        out = torch.full((int(m[:, r].sum()) + 5,), float(SENTINEL))
        g.all_to_all_v(out, inp, torch.from_numpy(m[r].astype(np.int64)), torch.from_numpy(m[:, r].astype(np.int64)))
        ref = expected(m, r, [int(m[p].sum()) for p in range(w)], [out.numel()] * w, torch.float32)
        n = int(m[:, r].sum())   # (a staged output's tail beyond the received blocks is not defined)
        assert torch.equal(out[:n], ref[:n])
    A.run_ranks(world, fn, EAGER)


@pytest.mark.parametrize("cfg", PROTOCOLS)
def test_moe_dispatch_combine_v_round_trip(cfg):
    world, hidden, tokens = 4, 6, 10

    def fn(a, r, w):
        g = TensorGroup(a)
        gen = torch.Generator().manual_seed(r)
        dest = torch.randint(0, w, (tokens,), generator=gen)
        dest[dest == (r + 1) % w] = r            # some expert rank gets nothing from me
        order = torch.argsort(dest, stable=True)
        x = torch.randn(tokens, hidden, generator=gen)[order]
        send_counts = torch.bincount(dest, minlength=w).to(torch.int64)
        recv, recv_counts = moe_dispatch_v(g, x, send_counts, capacity=tokens * w)
        assert int(recv_counts.sum()) <= tokens * w
        y = recv * 2 + 1                             # the "expert"
        back = moe_combine_v(g, y, recv_counts, send_counts, tokens)
        assert torch.equal(back, x * 2 + 1)
    A.run_ranks(world, fn, cfg)


@pytest.mark.parametrize("world", [2, 3])
def test_torch_distributed_all_to_all_single_uneven(world):
    """dist.all_to_all_single(out, inp, out_splits, in_splits) on the "accl" backend, one emulator process per rank."""
    env = dict(os.environ, PG_PORT=str(random.randint(20000, 40000)), CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-m", "accl_b200.models.emulator", "-n", str(world), "--", sys.executable,
                        os.path.join(ROOT, "tests", "helpers", "a2av_worker.py")], cwd=ROOT, env=env, capture_output=True,
                       text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert r.stdout.count(": ok") == world
