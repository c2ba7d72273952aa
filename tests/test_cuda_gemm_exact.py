"""Exact tests of the two fused wgmma GEMM plugins (GEMM -> reduce-scatter and all-gather -> GEMM) against an fp64
reference computed on the CPU, at the depths, tile orders and world sizes where the TMA -> mbarrier -> wgmma pipeline
can go wrong.

Three kinds of operands:
* dense: bf16 integers in {-2..2}.  Every product and every partial sum is an integer far below 2^24, so fp32
  accumulation is exact in any order: an fp32 shard equals the reference, and a bf16 result equals the reference
  rounded once to bf16.  A misplaced element, a lost or doubled K-block, a stale accumulator, a wrong owner row or any
  rounding of the accumulator in mid-K shows up as an inequality.
* sparse: rows of A with at most 8 nonzeros in {-1, 1}, W in {-4..4}.  Every rank's partial is an integer of magnitude
  <= 32 and every sum of up to 8 of them <= 256, which bf16 represents exactly: a bf16 shard whose partials the TMA
  unit adds in bf16, in arrival order, equals the reference.
* random: randn * 0.5, checked against a per-element error bound computed from the same operands.

Every GPU test carries its own `gpu` mark, so the CPU test of the helpers at the end runs without a GPU.
"""
import pytest
import torch

import accl_b200 as A
from accl_b200.ops import all_gather_gemm, gemm_reduce_scatter

NGPU = torch.cuda.device_count() if torch.cuda.is_available() else 0
CFG = dict(n_egr_rx_bufs=4, egr_rx_buf_size=16 << 10, max_egr_size=64 << 10, max_rndzv_size=1 << 30)
DMA_MISMATCH_ERROR = 1 << 0  # accl/constants.hpp

BM, BN, BK = 128, 256, 64  # wgmma.cuh: tile rows of one CTA, tile columns, K-block
# one K-block; fewer K-blocks than the 4 ring stages; the ring wraps exactly; several wraps and a remainder; the
# depth of bench/gemm_rs.py and bench/ag_gemm.py
KS = (64, 192, 256, 576, 8192)
RANDOM_KS = (64, 576, 8192)
# rows per world size.  Tile rows are swept in groups of 16 (single-CTA tiles, ag-gemm) or 8 (pair tiles):
# 2560 = 20 single / 10 pair tile rows (16 + 4, 8 + 2), 2304 = 18 / 9 (16 + 2, 8 + 1), 3072 = 24 / 12 (16 + 8, 8 + 4)
M_OF_WORLD = {1: 2560, 2: 1024, 3: 2304, 4: 3072}
# (world, N): one column tile; an odd column-tile count; at world 1 also more tiles than SMs (160 single, 80 pair)
SHAPES = [(1, 256), (1, 768), (1, 2048), (2, 256), (2, 768), (3, 256), (3, 768), (4, 256), (4, 768)]
GUARD_ROWS = 16  # rows of sentinel before and after every output
SENTINEL = -12288.0  # exact in bf16 and fp32, and no result of these operands


def devices(world):
    return [r % max(NGPU, 1) for r in range(world)]


def status_of(a):
    return torch.full((1,), -1, dtype=torch.int32, device=torch.device("cuda", a.cuda_device))


# ------------------------------------------------------------------------------------------------ grid budget
def grid_ctas(kernel, M, N, sms):
    """CTAs of one rank's launch, sized as launch_variant (plugin_gemm_rs.cu) and launch_ag_gemm size the grid:
    "single" (gemm_rs variant 1, ag-gemm) one CTA per 128 x 256 tile, "pair" (gemm_rs variant 2) two per 256 x 256."""
    if kernel == "pair":
        return 2 * min(sms // 2, (M // (2 * BM)) * (N // BN))
    return min(sms, (M // BM) * (N // BN))


def over_budget(kernel, M, N, devs, sms):
    """Why the case may not run with rank r on GPU devs[r], or None.  Both kernels are persistent, one CTA per SM, and
    wait for their peers: grids of ranks sharing a GPU must all be resident at once or they can only time out.  The
    pair kernel keeps a quarter of the SMs spare because its cluster placement cannot see the other ranks' kernels
    (a judgement, not a measurement)."""
    per_gpu = max(devs.count(d) for d in devs)
    if per_gpu == 1:
        return None
    need = per_gpu * grid_ctas(kernel, M, N, sms)
    limit = sms * 3 // 4 if kernel == "pair" else sms
    if need <= limit:
        return None
    return (f"over the shared-GPU budget: {per_gpu} ranks x {need // per_gpu} {kernel}-kernel CTAs = {need} > {limit} "
            f"of {sms} SMs")


def skip_over_budget(kernel, M, N, devs):
    why = over_budget(kernel, M, N, devs, torch.cuda.get_device_properties(devs[0]).multi_processor_count)
    if why:
        pytest.skip(why)


# ------------------------------------------------------------------------------------------------ operands
def dense_operands(M, N, K, P, seed):
    """bf16 integers in {-2..2}: every sum over K and P ranks is an integer below 2^24, exact in fp32."""
    assert 4 * K * P < 1 << 24
    g = torch.Generator().manual_seed(seed)
    return (torch.randint(-2, 3, (M, K), generator=g, dtype=torch.int8).bfloat16(),
            torch.randint(-2, 3, (N, K), generator=g, dtype=torch.int8).bfloat16())


def sparse_operands(M, N, K, P, seed):
    """At most 8 nonzeros in {-1, 1} per row of A, W in {-4..4}: |partial| <= 8 * 4 = 32, and a sum of P <= 8 partials
    in any order stays an integer of magnitude <= 256, which bf16 represents exactly."""
    assert 2 <= P <= 8 and P * 8 * 4 <= 256
    g = torch.Generator().manual_seed(seed)
    a = torch.zeros(M, K)
    a.scatter_(1, torch.randint(0, K, (M, 8), generator=g), torch.randint(0, 2, (M, 8), generator=g).float() * 2 - 1)
    w = torch.randint(-4, 5, (N, K), generator=g).float()
    assert int((a != 0).sum(1).max()) <= 8 and float(a.abs().max()) <= 1 and float(w.abs().max()) <= 4
    return a.bfloat16(), w.bfloat16()


def random_operands(M, N, K, P, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(M, K, generator=g) * 0.5).bfloat16(), (torch.randn(N, K, generator=g) * 0.5).bfloat16()


OPERANDS = {"dense": dense_operands, "sparse": sparse_operands, "random": random_operands}


def seed_of(*key):
    s = 17
    for k in key:
        s = (s * 1_000_003 + k) % (1 << 62)
    return s


# ------------------------------------------------------------------------------------------------ checks
def error_bound(abs_prod, K, P, bf16_roundings):
    """Per-element bound on |result - exact| for operands whose |A_r| |W_r|^T summed over ranks is `abs_prod` (fp64).
    fp32 accumulation over K, and the fp32 adds of P partials: (K + P - 1) 2^-23 abs_prod, twice gamma to allow for a
    truncating accumulator.  Each bf16 rounding of a value v adds at most 2^-8 |v|, and |v| <= abs_prod (1 + 2^-8)^n."""
    acc = (K + P - 1) * 2.0 ** -23 * abs_prod
    return acc + bf16_roundings * 2.0 ** -8 * (1 + 2.0 ** -8) ** bf16_roundings * (abs_prod + acc)


def cublas_note(parts):
    """Whether cuBLAS's bf16 GEMM of the same operands rounds the exact product correctly: tells a kernel bug from
    tensor cores that do not accumulate these integers exactly."""
    if not torch.cuda.is_available():
        return "cuBLAS not checked (no GPU)"
    dev = torch.device("cuda", 0)
    keep = torch.backends.cuda.matmul.allow_bf16_reduced_precision_reduction
    torch.backends.cuda.matmul.allow_bf16_reduced_precision_reduction = False
    try:
        exact = all(torch.equal(torch.matmul(a.to(dev), w.to(dev).t()).cpu(), (a.double() @ w.double().t()).float().bfloat16())
                    for a, w in parts)
    finally:
        torch.backends.cuda.matmul.allow_bf16_reduced_precision_reduction = keep
    return f"cuBLAS bf16 GEMM of the same operands {'is' if exact else 'is NOT'} exact at this shape"


def exact_failure(what, got, want, row0, tile_m, parts):
    """None when `got` equals `want` bit for bit, else a report: the number of wrong elements, the first wrong one in
    C's coordinates with its tile, and the (rank, K-block) whose contribution equals the error (a lost or doubled
    block).  `row0` is the row of C that got[0] holds; parts: every rank's (A_r, W_r) with C = sum_r A_r W_r^T."""
    if torch.equal(got, want):
        return None
    bad = (got.double() != want.double()) | torch.isnan(got.double())
    i, j = (int(v) for v in bad.nonzero()[0])
    row = row0 + i
    diff = float(got[i, j].double() - want[i, j].double())
    blocks = []
    for r, (a, w) in enumerate(parts):
        contrib = (a[row].double() * w[j].double()).view(-1, BK).sum(1)
        blocks += [(r, kb) for kb, c in enumerate(contrib.tolist()) if c != 0 and abs(c) == abs(diff)]
    return (f"{what}: {int(bad.sum())} of {bad.numel()} elements wrong; first at C[{row}, {j}] (tile row {row // tile_m}, "
            f"tile column {j // BN}, row {row % tile_m} / column {j % BN} inside it): got {float(got[i, j])}, want "
            f"{float(want[i, j])}; (rank, K-block) contributing exactly the difference: {blocks or 'none'}; "
            f"{cublas_note(parts)}")


def bound_failure(what, got, ref, bound, row0):
    err = (got.double() - ref).abs()
    over = err > bound
    if not bool(over.any()):
        return None
    i, j = (int(v) for v in over.nonzero()[0])
    return (f"{what}: {int(over.sum())} elements outside the error bound; first at C[{row0 + i}, {j}]: error "
            f"{float(err[i, j]):.4g} > bound {float(bound[i, j]):.4g}")


def cases_for(kinds_exact):
    return [(K, kind) for K in KS for kind in kinds_exact] + [(K, "random") for K in RANDOM_KS]


# ------------------------------------------------------------------------------------------------ GEMM -> reduce-scatter
RS_KERNELS = [(1, torch.bfloat16), (1, torch.float32), (2, torch.bfloat16), (2, torch.float32)]
RS_IDS = ["single-bf16", "single-fp32", "pair-bf16", "pair-fp32"]


def run_gemm_rs_cases(world, M, N, cases, variant, out_dtype, tag):
    """One rank start-up for all cases.  Each call gets fresh sentinel-filled heap buffers before and after its shard;
    the previous call's buffers stay alive, so every call also sees another out_off.  Returns per rank per case
    (A_r, W_r, shard, status, guards intact)."""

    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        keep, res = None, []
        for K, kind in cases:
            x, wt = OPERANDS[kind](M, N, K, w, seed_of(tag, world, N, K, len(kind), r))
            rows = M // w
            pre, out, post = (a.create_buffer(n, out_dtype) for n in (GUARD_ROWS * N, rows * N, GUARD_ROWS * N))
            for b in (pre, out, post):
                b.dev.fill_(SENTINEL)  # the kernel zeroes the shard itself
            st = status_of(a)
            gemm_reduce_scatter(a, x.to(dev), wt.to(dev), out, variant=variant, status=st)
            torch.cuda.current_stream().synchronize()
            guards = bool((pre.dev == SENTINEL).all()) and bool((post.dev == SENTINEL).all())
            res.append((x, wt, out.dev.view(rows, N).cpu(), int(st.item()), guards))
            keep = (pre, out, post)
        del keep
        return res

    return A.run_cuda_ranks(devices(world), fn, CFG, timeout=600.0, heap_mb=256 if world == 1 else 128, max_ctas=4)


def check_gemm_rs_case(what, per_rank, M, N, K, kind, out_dtype, tile_m):
    P = len(per_rank)
    parts = [(x, wt) for x, wt, *_ in per_rank]
    ref = sum(x.double() @ wt.double().t() for x, wt in parts)
    abs_prod = sum(x.double().abs() @ wt.double().abs().t() for x, wt in parts) if kind == "random" else None
    rows = M // P
    for o, (_, _, shard, status, guards) in enumerate(per_rank):
        label = f"{what} K={K} {kind} rank {o}"
        assert status == 0, f"{label}: status {status:#x}"
        assert guards, f"{label}: the heap buffers around the shard were written"
        ref_o = ref[o * rows:(o + 1) * rows]
        if kind == "random":
            bound = error_bound(abs_prod[o * rows:(o + 1) * rows], K, P, 0 if out_dtype == torch.float32 else P)
            msg = bound_failure(label, shard, ref_o, bound, o * rows)
        else:
            want = ref_o.float() if out_dtype == torch.float32 else ref_o.float().bfloat16()
            msg = exact_failure(label, shard, want, o * rows, tile_m, parts)
        assert msg is None, msg


@pytest.mark.gpu
@pytest.mark.parametrize("world,N", SHAPES, ids=[f"world{w}-N{n}" for w, n in SHAPES])
@pytest.mark.parametrize("variant,out_dtype", RS_KERNELS, ids=RS_IDS)
def test_gemm_reduce_scatter_is_exact(variant, out_dtype, world, N):
    """Both kernels, bf16 and fp32 shards, at every K of KS: exact for integer operands (dense, or sparse for bf16
    shards at world > 1, whose partials are added in bf16), within the computed bound for random ones."""
    M = M_OF_WORLD[world]
    kernel = "pair" if variant == 2 else "single"
    skip_over_budget(kernel, M, N, devices(world))
    exact = "sparse" if out_dtype == torch.bfloat16 and world > 1 else "dense"
    cases = cases_for([exact])
    res = run_gemm_rs_cases(world, M, N, cases, variant, out_dtype, tag=variant * 2 + (out_dtype == torch.float32))
    what = f"gemm_rs {kernel} {str(out_dtype)[6:]} world {world} M={M} N={N}"
    for i, (K, kind) in enumerate(cases):
        check_gemm_rs_case(what, [per_rank[i] for per_rank in res], M, N, K, kind, out_dtype, 2 * BM if variant == 2 else BM)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", [1, 2], ids=["single", "pair"])
def test_gemm_reduce_scatter_back_to_back_calls_rewrite_the_operands(variant):
    """Three calls into the same shard at world 2, the operands rewritten on the stream between calls: the in-kernel
    zeroing must not race a peer's late reduce-adds, and the flags must be reset for every launch."""
    M, N, K = 1024, 512, 576

    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        g = torch.Generator(device=dev).manual_seed(600 + r)
        out = a.create_buffer(M // w * N, torch.float32)
        x = torch.empty(M, K, dtype=torch.bfloat16, device=dev)
        wt = torch.empty(N, K, dtype=torch.bfloat16, device=dev)
        its = []
        for _ in range(3):
            x.copy_(torch.randint(-2, 3, (M, K), generator=g, device=dev))
            wt.copy_(torch.randint(-2, 3, (N, K), generator=g, device=dev))
            st = status_of(a)
            gemm_reduce_scatter(a, x, wt, out, variant=variant, status=st)
            its.append((x.clone(), wt.clone(), out.dev.view(M // w, N).clone(), st))
        torch.cuda.current_stream().synchronize()
        return [(xi.cpu(), wi.cpu(), o.cpu(), int(st.item()), True) for xi, wi, o, st in its]

    res = A.run_cuda_ranks(devices(2), fn, CFG, heap_mb=64, max_ctas=4)
    for it in range(3):
        check_gemm_rs_case(f"gemm_rs back-to-back call {it}", [per_rank[it] for per_rank in res], M, N, K, "dense",
                           torch.float32, 2 * BM if variant == 2 else BM)


@pytest.mark.gpu
def test_gemm_reduce_scatter_reports_a_shard_offset_mismatch_and_contains_it():
    """Rank 0 allocates (out, extra), rank 1 (extra, out): each rank's shard sits where the peer keeps `extra`.  Both
    calls report DMA_MISMATCH_ERROR and neither rank adds into the peer's `extra`; a following call on shards that line
    up is exact."""
    M, N, K = 1024, 256, 128

    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        x, wt = dense_operands(M, N, K, w, 700 + r)
        x, wt = x.to(dev), wt.to(dev)
        n = M // w * N
        first, second = a.create_buffer(n, torch.float32), a.create_buffer(n, torch.float32)
        out, extra = (first, second) if r == 0 else (second, first)
        extra.dev.fill_(SENTINEL)
        torch.cuda.current_stream().synchronize()
        a.barrier()  # the peer's sentinel is in place before anything could add into it
        st_bad = status_of(a)
        gemm_reduce_scatter(a, x, wt, out, status=st_bad)
        torch.cuda.current_stream().synchronize()
        intact = bool((extra.dev == SENTINEL).all())
        good = a.create_buffer(n, torch.float32)
        st = status_of(a)
        gemm_reduce_scatter(a, x, wt, good, status=st)
        torch.cuda.current_stream().synchronize()
        return int(st_bad.item()), intact, (x.cpu(), wt.cpu(), good.dev.view(M // w, N).cpu(), int(st.item()), True)

    res = A.run_cuda_ranks(devices(2), fn, CFG, heap_mb=64, max_ctas=4)
    for r, (bad_status, intact, _) in enumerate(res):
        assert intact, f"rank {r}: the peer's partial products landed in this rank's `extra` buffer"
        assert bad_status != -1 and bad_status & DMA_MISMATCH_ERROR, (r, hex(bad_status))
    check_gemm_rs_case("gemm_rs after a mismatch", [good for *_, good in res], M, N, K, "dense", torch.float32, 2 * BM)


@pytest.mark.gpu
def test_gemm_reduce_scatter_rejects_bad_arguments():
    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        M, N, K = 256, 256, 128
        x = torch.zeros(M, K, dtype=torch.bfloat16, device=dev)
        wt = torch.zeros(N, K, dtype=torch.bfloat16, device=dev)
        out = a.create_buffer(M * N, torch.bfloat16)
        st = status_of(a)
        bad = {
            "fp32 a": lambda: gemm_reduce_scatter(a, x.float(), wt, out),
            "fp32 w": lambda: gemm_reduce_scatter(a, x, wt.float(), out),
            "a on the CPU": lambda: gemm_reduce_scatter(a, x.cpu(), wt, out, status=st),
            "1-D a": lambda: gemm_reduce_scatter(a, x.view(-1), wt, out, status=st),
            "non-contiguous a": lambda: gemm_reduce_scatter(a, x.t(), torch.zeros(N, M, dtype=torch.bfloat16, device=dev),
                                                            out, status=st),
            "K mismatch": lambda: gemm_reduce_scatter(a, x, wt[:, :64].contiguous(), out, status=st),
            "M % 128": lambda: gemm_reduce_scatter(a, x[:192], wt, out, status=st),
            "N % 256": lambda: gemm_reduce_scatter(a, x, wt[:128], out, status=st),
            "K % 64": lambda: gemm_reduce_scatter(a, x[:, :96].contiguous(), wt[:, :96].contiguous(), out, status=st),
            "pair variant, M % 256": lambda: gemm_reduce_scatter(a, x[:128], wt, out, variant=2, status=st),
            "unknown variant": lambda: gemm_reduce_scatter(a, x, wt, out, variant=3, status=st),
            "out too small": lambda: gemm_reduce_scatter(a, x, wt, a.create_buffer(M * N - 1, torch.bfloat16), status=st),
            "out is a plain tensor": lambda: gemm_reduce_scatter(a, x, wt, torch.empty(M * N, dtype=torch.bfloat16,
                                                                                       device=dev), status=st),
            "fp16 out": lambda: gemm_reduce_scatter(a, x, wt, a.create_buffer(M * N, torch.float16), status=st),
            "out_dtype disagrees with out": lambda: gemm_reduce_scatter(a, x, wt, out, out_dtype=torch.float32, status=st),
            "int64 status": lambda: gemm_reduce_scatter(a, x, wt, out, status=torch.zeros(1, dtype=torch.int64, device=dev)),
        }
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


# ------------------------------------------------------------------------------------------------ all-gather -> GEMM
def run_ag_gemm_cases(world, M, N, cases, tag):
    """One rank start-up for all cases; a fresh heap shard per call (the previous one kept alive), `out` and `gathered`
    carved out of the middle of sentinel-filled tensors.  Returns per rank per case
    (shard, W_r, out, gathered, status, guards intact)."""

    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        keep, res = None, []
        for K, kind in cases:
            s, wt = OPERANDS[kind](M // w, N, K, w, seed_of(tag, world, N, K, len(kind), r))
            buf = a.create_buffer(M // w * K, torch.bfloat16)
            shard = buf.dev.view(M // w, K)
            shard.copy_(s.to(dev))
            out_all = torch.full((M + 2 * GUARD_ROWS, N), SENTINEL, dtype=torch.bfloat16, device=dev)
            gathered_all = torch.full((M + 2 * GUARD_ROWS, K), SENTINEL, dtype=torch.bfloat16, device=dev)
            st = status_of(a)
            out, gathered = all_gather_gemm(a, shard, wt.to(dev), out=out_all[GUARD_ROWS:GUARD_ROWS + M],
                                            gathered=gathered_all[GUARD_ROWS:GUARD_ROWS + M], status=st)
            torch.cuda.current_stream().synchronize()
            guards = all(bool((t[:GUARD_ROWS] == SENTINEL).all()) and bool((t[GUARD_ROWS + M:] == SENTINEL).all())
                         for t in (out_all, gathered_all))
            res.append((s, wt, out.cpu(), gathered.cpu(), int(st.item()), guards))
            keep = buf
        del keep
        return res

    return A.run_cuda_ranks(devices(world), fn, CFG, timeout=600.0, heap_mb=256 if world == 1 else 128, max_ctas=4)


def check_ag_gemm_case(what, per_rank, M, N, K, kind):
    full = torch.cat([s for s, *_ in per_rank])
    for r, (_, wt, out, gathered, status, guards) in enumerate(per_rank):
        label = f"{what} K={K} {kind} rank {r}"
        assert status == 0, f"{label}: status {status:#x}"
        assert guards, f"{label}: the memory around out or gathered was written"
        assert torch.equal(gathered, full), f"{label}: gathered is not the shards in rank order"
        ref = full.double() @ wt.double().t()
        if kind == "random":
            bound = error_bound(full.double().abs() @ wt.double().abs().t(), K, 1, 1)
            msg = bound_failure(label, out, ref, bound, 0)
        else:
            msg = exact_failure(label, out, ref.float().bfloat16(), 0, BM, [(full, wt)])
        assert msg is None, msg


@pytest.mark.gpu
@pytest.mark.parametrize("world,N", SHAPES, ids=[f"world{w}-N{n}" for w, n in SHAPES])
def test_all_gather_gemm_is_exact(world, N):
    """bf16 out of dense integer operands equals the reference rounded once; random operands stay within the bound;
    `gathered` is bit-identical to the shards in rank order."""
    M = M_OF_WORLD[world]
    skip_over_budget("single", M, N, devices(world))
    cases = cases_for(["dense"])
    res = run_ag_gemm_cases(world, M, N, cases, tag=9)
    for i, (K, kind) in enumerate(cases):
        check_ag_gemm_case(f"ag_gemm world {world} M={M} N={N}", [per_rank[i] for per_rank in res], M, N, K, kind)


@pytest.mark.gpu
def test_all_gather_gemm_at_the_row_block_limit():
    """M / 128 = 1024 uses the last ready[] word; 1025 row blocks raise ValueError before anything is enqueued."""
    M, N, K = 1024 * BM, 256, 64
    res = run_ag_gemm_cases(1, M, N, [(K, "dense")], tag=10)
    check_ag_gemm_case(f"ag_gemm world 1 M={M} N={N}", [res[0][0]], M, N, K, "dense")

    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        shard = a.create_buffer((M + BM) * K, torch.bfloat16).dev.view(M + BM, K)
        st = status_of(a)
        with pytest.raises(ValueError):
            all_gather_gemm(a, shard, torch.zeros(N, K, dtype=torch.bfloat16, device=dev), status=st)
        torch.cuda.current_stream().synchronize()
        return int(st.item())

    assert A.run_cuda_ranks([0], fn, CFG, heap_mb=256, max_ctas=4)[0] == -1


# ------------------------------------------------------------------------------------------------ CPU: the helpers
def test_operand_generators_grid_budget_and_diagnostics_on_the_cpu():
    # the exactness arguments hold: integer partials, fp32-exact dense sums, bf16-exact sparse sums over 8 ranks
    parts = [sparse_operands(128, 256, 576, 8, seed_of(1, r)) for r in range(8)]
    partials = [a.double() @ w.double().t() for a, w in parts]
    assert max(float(p.abs().max()) for p in partials) <= 32
    assert float(sum(p.abs() for p in partials).max()) <= 256
    running = torch.zeros_like(partials[0]).bfloat16()
    for p in reversed(partials):  # bf16 adds in some arrival order
        running = running + p.bfloat16()
    assert torch.equal(running.double(), sum(partials))
    a, w = dense_operands(128, 256, 8192, 4, 3)
    ref = a.double() @ w.double().t()
    assert torch.equal((a.float() @ w.float().t()).double(), ref)

    # the exact check catches an accumulator rounded to bf16 after every K-block at the benchmark depth
    acc = torch.zeros(128, 256)
    for kb in range(8192 // BK):
        acc = (acc + a[:, kb * BK:(kb + 1) * BK].float() @ w[:, kb * BK:(kb + 1) * BK].float().t()).bfloat16().float()
    assert not torch.equal(acc.bfloat16(), ref.float().bfloat16())

    # a lost K-block is named in the report
    got = ref.float().clone()
    a0, w0 = a[0, 5 * BK:6 * BK].double(), w[7, 5 * BK:6 * BK].double()
    got[0, 7] -= float(a0 @ w0)
    msg = exact_failure("lost block", got, ref.float(), 0, BM, [(a, w)])
    assert msg is not None and "C[0, 7]" in msg and "(0, 5)" in msg
    assert exact_failure("same", ref.float(), ref.float(), 0, BM, [(a, w)]) is None

    # the random-operand bound covers a correct computation with a single bf16 rounding
    a, w = random_operands(128, 256, 576, 1, 4)
    ref = a.double() @ w.double().t()
    assert bound_failure("ok", (a.float() @ w.float().t()).bfloat16(), ref,
                         error_bound(a.double().abs() @ w.double().abs().t(), 576, 1, 1), 0) is None

    # the launchers' grids: min(SMs, tiles) single, 2 min(SMs / 2, pair tiles) pair
    assert grid_ctas("single", 2304, 256, 132) == 18 and grid_ctas("pair", 2304, 256, 132) == 18
    assert grid_ctas("single", 3072, 256, 132) == 24 and grid_ctas("pair", 3072, 256, 132) == 24
    assert grid_ctas("single", 2560, 2048, 132) == 132 and grid_ctas("pair", 2560, 2048, 132) == 132
    assert grid_ctas("pair", 2560, 2048, 131) == 130
    # world 3 and 4 at N = 256 fit one GPU (54 and 96 CTAs), N = 768 needs distinct GPUs
    for kernel in ("single", "pair"):
        assert over_budget(kernel, 2304, 256, [0] * 3, 132) is None
        assert over_budget(kernel, 3072, 256, [0] * 4, 132) is None
        assert over_budget(kernel, 2304, 768, [0] * 3, 132) is not None
        assert over_budget(kernel, 3072, 768, [0, 1, 2, 3], 132) is None
    assert over_budget("single", 2560, 2048, [0], 132) is None
    assert over_budget("pair", 2048, 768, [0, 0], 132) is None          # 2 x 48 = 96 <= 99
    assert over_budget("single", 2560, 768, [0, 0], 132) is None        # 2 x 60 = 120 <= 132
    assert over_budget("pair", 2560, 768, [0, 0], 132) is not None      # 2 x 60 = 120 > 99, the pair kernel's margin
    assert over_budget("single", 2048, 1280, [0, 0], 132) is not None   # 2 x 80 = 160 > 132
