"""GPU tests of the fused all-gather -> wgmma GEMM plugin and the sequence-parallel column-parallel linear."""
import pytest
import torch

import accl_b200 as A
from accl_b200.ops import all_gather_gemm

pytestmark = pytest.mark.gpu
NGPU = torch.cuda.device_count() if torch.cuda.is_available() else 0
CFG = dict(n_egr_rx_bufs=4, egr_rx_buf_size=16 << 10, max_egr_size=64 << 10, max_rndzv_size=1 << 30)
DMA_MISMATCH_ERROR = 1 << 0  # accl/constants.hpp


def devices(world):
    return [r % max(NGPU, 1) for r in range(world)]


def close(a, b, rtol, atol):
    return torch.allclose(a.cpu().double(), b.cpu().double(), rtol=rtol, atol=atol)


def heap_shard(a, m, k):
    """An [m, k] bf16 tensor in the symmetric heap (same offset on every rank when allocated in the same order)."""
    buf = a.create_buffer(m * k, torch.bfloat16)
    t = buf.dev.view(m, k)
    t._buf = buf
    return t


def status_of(a):
    return torch.full((1,), -1, dtype=torch.int32, device=torch.device("cuda", a.cuda_device))


def check_result(res, N):
    """res: per rank (shard, w, out, gathered, status) on the CPU; out against an fp32 matmul of the same bf16 operands,
    gathered bit for bit against the concatenated shards."""
    full = torch.cat([shard for shard, *_ in res])
    for r, (_, w, out, gathered, status) in enumerate(res):
        assert status == 0, (r, hex(status))
        assert torch.equal(gathered, full), r
        ref = full.float() @ w.float().t()
        assert out.shape == (full.shape[0], N)
        assert close(out, ref, 2e-2, 2e-1), (r, (out.float() - ref).abs().max())


@pytest.mark.parametrize("world", [1, 2])
def test_all_gather_gemm_matches_fp32_reference(world):
    M, N, K = 512 * world, 512, 320   # several tiles per rank, a K that is not a multiple of the stage depth

    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        g = torch.Generator().manual_seed(200 + r)
        shard = heap_shard(a, M // w, K)
        shard.copy_((torch.randn(M // w, K, generator=g) * 0.5).bfloat16())
        wt = (torch.randn(N, K, generator=g) * 0.5).bfloat16().to(dev)
        st = status_of(a)
        out, gathered = all_gather_gemm(a, shard, wt, status=st)
        torch.cuda.current_stream().synchronize()
        return shard.cpu(), wt.cpu(), out.cpu(), gathered.cpu(), int(st.item())

    check_result(A.run_cuda_ranks(devices(world), fn, CFG, heap_mb=64, max_ctas=4), N)


def test_all_gather_gemm_with_more_tiles_than_sms():
    """The persistent loop: several tiles per CTA, the accumulator restarted after each TMA-store epilogue."""
    M, N, K = 4096, 4096, 320

    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        g = torch.Generator().manual_seed(9)
        shard = heap_shard(a, M, K)
        shard.copy_((torch.randn(M, K, generator=g) * 0.5).bfloat16())
        wt = (torch.randn(N, K, generator=g) * 0.5).bfloat16().to(dev)
        st = status_of(a)
        out, gathered = all_gather_gemm(a, shard, wt, status=st)
        torch.cuda.current_stream().synchronize()
        return shard.cpu(), wt.cpu(), out.cpu(), gathered.cpu(), int(st.item())

    check_result(A.run_cuda_ranks([0], fn, CFG, heap_mb=256, max_ctas=4), N)


def test_all_gather_gemm_back_to_back_calls_rewrite_the_shard():
    """Three calls on the same buffers; each rank rewrites its shard on the stream right after the previous call.  Every
    result must be its own iteration's: the exit meeting keeps a peer from overwriting a shard still being read, and the
    flags are reset before every launch."""
    M, N, K = 1024, 512, 320

    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        shard = heap_shard(a, M // w, K)
        wt = (torch.randn(N, K, generator=torch.Generator().manual_seed(300 + r)) * 0.5).bfloat16().to(dev)
        out = torch.empty(M, N, dtype=torch.bfloat16, device=dev)
        gathered = torch.empty(M, K, dtype=torch.bfloat16, device=dev)
        its = []
        for it in range(3):
            g = torch.Generator(device=dev).manual_seed(1000 * it + r)
            shard.copy_(torch.randn(M // w, K, generator=g, device=dev) * 0.5)
            x = shard.clone()
            st = status_of(a)
            all_gather_gemm(a, shard, wt, out=out, gathered=gathered, status=st)
            its.append((x, out.clone(), gathered.clone(), st))
        torch.cuda.current_stream().synchronize()
        return [(x.cpu(), wt.cpu(), o.cpu(), gth.cpu(), int(st.item())) for x, o, gth, st in its]

    res = A.run_cuda_ranks(devices(2), fn, CFG, heap_mb=64, max_ctas=4)
    for it in range(3):
        check_result([per_rank[it] for per_rank in res], N)


def test_all_gather_gemm_reports_a_shard_offset_mismatch_and_recovers():
    """Rank 1's shard sits one buffer further into the heap: neither rank reads the other's shard and both report
    DMA_MISMATCH_ERROR.  Once the heaps line up again the next call succeeds."""
    M, N, K = 512, 256, 128

    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        g = torch.Generator().manual_seed(400 + r)
        wt = (torch.randn(N, K, generator=g) * 0.5).bfloat16().to(dev)
        extra = heap_shard(a, M // w, K) if r == 1 else None
        bad = heap_shard(a, M // w, K)
        bad.copy_((torch.randn(M // w, K, generator=g) * 0.5).bfloat16())
        st_bad = status_of(a)
        all_gather_gemm(a, bad, wt, status=st_bad)
        if r == 0:
            extra = heap_shard(a, M // w, K)
        shard = heap_shard(a, M // w, K)
        shard.copy_((torch.randn(M // w, K, generator=g) * 0.5).bfloat16())
        st = status_of(a)
        out, gathered = all_gather_gemm(a, shard, wt, status=st)
        torch.cuda.current_stream().synchronize()
        del extra
        return int(st_bad.item()), (shard.cpu(), wt.cpu(), out.cpu(), gathered.cpu(), int(st.item()))

    res = A.run_cuda_ranks(devices(2), fn, CFG, heap_mb=64, max_ctas=4)
    for r, (bad_status, _) in enumerate(res):
        assert bad_status != -1 and bad_status & DMA_MISMATCH_ERROR, (r, hex(bad_status))
    check_result([good for _, good in res], N)


def test_all_gather_gemm_rejects_bad_arguments():
    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        K, N = 128, 256
        shard = heap_shard(a, 128, K)
        wt = torch.zeros(N, K, dtype=torch.bfloat16, device=dev)
        st = status_of(a)
        bad = {
            "shard outside the heap": lambda: all_gather_gemm(a, torch.zeros(128, K, dtype=torch.bfloat16, device=dev), wt),
            "fp32 weight": lambda: all_gather_gemm(a, shard, wt.float()),
            "fp32 shard": lambda: all_gather_gemm(a, a.create_buffer(128 * K, torch.float32).dev.view(128, K), wt),
            "M % 128": lambda: all_gather_gemm(a, heap_shard(a, 64, K), wt, status=st),
            "N % 256": lambda: all_gather_gemm(a, shard, wt[:128], status=st),
            "K % 64": lambda: all_gather_gemm(a, heap_shard(a, 128, 96), torch.zeros(N, 96, dtype=torch.bfloat16, device=dev),
                                              status=st),
            "K mismatch": lambda: all_gather_gemm(a, shard, torch.zeros(N, 64, dtype=torch.bfloat16, device=dev)),
            "out shape": lambda: all_gather_gemm(a, shard, wt, out=torch.empty(128, 128, dtype=torch.bfloat16, device=dev)),
        }
        # out overlapping the shard: both carved out of one heap buffer
        both = a.create_buffer(128 * K + 128 * N, torch.bfloat16).dev
        bad["out overlapping the shard"] = lambda: all_gather_gemm(a, both[:128 * K].view(128, K), wt,
                                                                   out=both[64 * K:64 * K + 128 * N].view(128, N), status=st)
        for what, call in bad.items():
            try:
                call()
            except ValueError:
                continue
            raise AssertionError(f"no ValueError for: {what}")
        torch.cuda.current_stream().synchronize()
        assert int(st.item()) == -1  # nothing was enqueued
        return True

    assert A.run_cuda_ranks([0], fn, CFG, heap_mb=64, max_ctas=4)[0]


def test_sequence_parallel_mlp_matches_unsharded_reference():
    """SeqParallelColumnLinear -> GELU -> RowParallelLinear at world 2 against the fp32 MLP on the full sequence."""
    from accl_b200.parallel import RowParallelLinear, SeqParallelColumnLinear, TensorGroup
    S, H, F = 512, 256, 1024   # sequence, hidden, FFN width over both ranks

    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        g = TensorGroup(a)
        up = SeqParallelColumnLinear(g, H, F // w)
        down = RowParallelLinear(g, F // w, H)
        x = torch.randn(S // w, H, generator=torch.Generator().manual_seed(500 + r)).bfloat16().to(dev)
        y = down(torch.nn.functional.gelu(up(x)))
        torch.cuda.current_stream().synchronize()
        return x.float().cpu(), up.weight.float().cpu(), down.weight.float().cpu(), y.float().cpu()

    res = A.run_cuda_ranks(devices(2), fn, CFG, heap_mb=64, max_ctas=4)
    x = torch.cat([x for x, *_ in res])
    w1 = torch.cat([w1 for _, w1, _, _ in res])          # [F, H]: the ranks' output features in rank order
    w2 = torch.cat([w2 for _, _, w2, _ in res], dim=1)   # [H, F]: the ranks' input features in rank order
    ref = torch.nn.functional.gelu(x @ w1.t()) @ w2.t()
    rows = S // 2
    for r, (_, _, _, y) in enumerate(res):
        assert close(y, ref[r * rows:(r + 1) * rows], 5e-2, 2e-2), (r, (y - ref[r * rows:(r + 1) * rows]).abs().max())
