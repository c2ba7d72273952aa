"""GPU tests of the fused GEMM -> all-reduce plugin (ops.gemm_all_reduce) and of the tensor-parallel linears with
replicated activations that run on it.

* ops: every rank's C against the fp64 reference (exact for integer operands, within the computed bound for random
  ones, as tests/test_cuda_gemm_exact.py does for gemm_reduce_scatter), every replica bit-identical to rank 0's, "kn"
  bit-identical to "nk" on W^T for integer operands, and at world 1 bit-identical to gemm_reduce_scatter.  M is a
  multiple of 128 (256 for the CTA pair) but not of 128 P, and the tile count is not a multiple of P, so the last block
  of the tile order is short.  Guard buffers around every C.
* back-to-back calls, a C at another heap offset on one rank, bad arguments.
* layers at world 1 and 2: gradients against fp32 autograd with the fused calls counted, a fused forward with a
  fallback backward, two micro-batches, and an offset mismatch in backward reported by TensorGroup.check.
"""
import threading

import pytest
import torch

import accl_b200 as A
import accl_b200.ops as ops
from accl_b200.ops import gemm_all_reduce, gemm_reduce_scatter
from accl_b200.parallel import ReplicatedColumnParallelLinear, ReplicatedRowParallelLinear, TensorGroup
from test_cuda_gemm_exact import (BM, CFG, DMA_MISMATCH_ERROR, GUARD_ROWS, OPERANDS, RS_IDS, RS_KERNELS, SENTINEL,
                                  bound_failure, devices, error_bound, exact_failure, seed_of, skip_over_budget,
                                  status_of)

pytestmark = pytest.mark.gpu

KS = (64, 192, 576, 8192)
RANDOM_KS = (576, 8192)
# M % 256 == 0 (both kernels) but M % (128 P) != 0 for P > 1; tiles of 128 x 256 / 256 x 256 per 256 columns:
# world 2: 10 / 5, world 3: 16 / 8, world 4: 20 / 10 -- a short last block of the tile order somewhere in every world
M_OF_WORLD = {1: 2560, 2: 1280, 3: 2048, 4: 2560}
SHAPES = [(1, 256), (1, 768), (2, 256), (2, 768), (3, 256), (3, 768), (4, 256), (4, 768)]


def cases_for(exact_kind):
    return [(K, exact_kind) for K in KS] + [(K, "random") for K in RANDOM_KS]


def guarded(a, n, dtype):
    """(pre, out, post) heap buffers, all sentinel-filled: the kernel writes only `out`."""
    bufs = tuple(a.create_buffer(k, dtype) for k in (GUARD_ROWS * 256, n, GUARD_ROWS * 256))
    for b in bufs:
        b.dev.fill_(SENTINEL)
    return bufs


def intact(pre, post):
    return bool((pre.dev == SENTINEL).all()) and bool((post.dev == SENTINEL).all())


# ------------------------------------------------------------------------------------------------ ops
def run_cases(world, M, N, cases, variant, out_dtype, tag):
    """Per case a "kn" call on W^T [K, N] and an "nk" call on W [N, K] (and at world 1 gemm_reduce_scatter on W), each
    into fresh guarded heap buffers.  Returns per rank per case (A_r, W_r, {name: (C, status, guards intact)})."""

    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        keep, res = [], []
        for K, kind in cases:
            x, wt = OPERANDS[kind](M, N, K, w, seed_of(tag, world, N, K, len(kind), r))
            xd, wd = x.to(dev), wt.to(dev)
            calls = {"kn": lambda out, st: gemm_all_reduce(a, xd, wd.t().contiguous(), out, variant=variant, status=st,
                                                           w_layout="kn"),
                     "nk": lambda out, st: gemm_all_reduce(a, xd, wd, out, variant=variant, status=st)}
            if w == 1:
                calls["rs"] = lambda out, st: gemm_reduce_scatter(a, xd, wd, out, variant=variant, status=st)
            got = {}
            for name, call in calls.items():
                pre, out, post = guarded(a, M * N, out_dtype)
                st = status_of(a)
                call(out, st)
                got[name] = (pre, out, post, st)
                keep.append((pre, out, post))
            torch.cuda.current_stream().synchronize()
            res.append((x, wt, {name: (out.dev.view(M, N).cpu(), int(st.item()), intact(pre, post))
                                for name, (pre, out, post, st) in got.items()}))
        del keep
        return res

    return A.run_cuda_ranks(devices(world), fn, CFG, timeout=600.0, heap_mb=256 if world == 1 else 160, max_ctas=4)


def check_case(what, per_rank, M, N, K, kind, out_dtype, tile_m):
    P = len(per_rank)
    parts = [(x, wt) for x, wt, _ in per_rank]
    ref = sum(x.double() @ wt.double().t() for x, wt in parts)
    if kind == "random":
        bound = error_bound(sum(x.double().abs() @ wt.double().abs().t() for x, wt in parts), K, P,
                            0 if out_dtype == torch.float32 else P)
    want = ref.float() if out_dtype == torch.float32 else ref.float().bfloat16()
    c0 = per_rank[0][2]["nk"][0]
    for r, (_, _, got) in enumerate(per_rank):
        for name, (c, status, guards) in got.items():
            label = f"{what} K={K} {kind} {name} rank {r}"
            assert status == 0, f"{label}: status {status:#x}"
            assert guards, f"{label}: the heap buffers around C were written"
            if name == "rs":
                continue
            msg = bound_failure(label, c, ref, bound, 0) if kind == "random" else exact_failure(label, c, want, 0, tile_m, parts)
            assert msg is None, msg
        # one owner's bits in every replica; "kn" and "nk" run the same MMAs on the same values, and integer partials
        # sum to the same bits in any arrival order
        assert torch.equal(got["nk"][0], c0), f"{what} K={K} {kind}: rank {r}'s C differs from rank 0's"
        if "kn" not in got:
            continue
        assert torch.equal(got["kn"][0], per_rank[0][2]["kn"][0]), f"{what} K={K} {kind}: rank {r}'s kn C differs from rank 0's"
        if kind != "random":
            assert torch.equal(got["kn"][0], got["nk"][0]), f"{what} K={K} {kind} rank {r}: kn differs from nk on W^T"
        if "rs" in got:
            assert torch.equal(got["rs"][0], got["nk"][0]), f"{what} K={K} {kind}: differs from gemm_reduce_scatter"


@pytest.mark.parametrize("world,N", SHAPES, ids=[f"world{w}-N{n}" for w, n in SHAPES])
@pytest.mark.parametrize("variant,out_dtype", RS_KERNELS, ids=RS_IDS)
def test_gemm_all_reduce_is_exact_and_replicated(variant, out_dtype, world, N):
    M = M_OF_WORLD[world]
    kernel = "pair" if variant == 2 else "single"
    skip_over_budget(kernel, M, N, devices(world))
    cases = cases_for("sparse" if out_dtype == torch.bfloat16 and world > 1 else "dense")
    res = run_cases(world, M, N, cases, variant, out_dtype, tag=40 + variant * 2 + (out_dtype == torch.float32))
    what = f"gemm_ar {kernel} {str(out_dtype)[6:]} world {world} M={M} N={N}"
    for i, (K, kind) in enumerate(cases):
        check_case(what, [per[i] for per in res], M, N, K, kind, out_dtype, 2 * BM if variant == 2 else BM)


@pytest.mark.parametrize("world", [2, 3, 4])
@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_gemm_all_reduce_replicas_are_bit_identical(world, out_dtype):
    """Random operands, where P independent sums would differ in the last bits: every rank holds the owner's bits."""
    M, N, K = 1024, 512, 1024

    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        g = torch.Generator(device=dev).manual_seed(800 + r)
        x = torch.randn(M, K, generator=g, device=dev).bfloat16()
        wt = torch.randn(N, K, generator=g, device=dev).bfloat16()
        outs = []
        for _ in range(2):
            st = status_of(a)
            outs.append((gemm_all_reduce(a, x, wt, out_dtype=out_dtype, status=st), st))
        torch.cuda.current_stream().synchronize()
        return [(out.dev.view(M, N).cpu(), int(st.item())) for out, st in outs]

    res = A.run_cuda_ranks(devices(world), fn, CFG, heap_mb=64, max_ctas=4)
    for call in range(2):
        for r, per in enumerate(res):
            c, status = per[call]
            assert status == 0, (r, call, hex(status))
            assert torch.equal(c, res[0][call][0]), f"call {call}: rank {r}'s C differs from rank 0's"


@pytest.mark.parametrize("variant", [1, 2], ids=["single", "pair"])
def test_gemm_all_reduce_back_to_back_calls_rewrite_the_operands(variant):
    """Three calls into the same C at world 2, the operands rewritten on the stream between calls: the zeroing, the
    counters and the broadcast of one call must not race the next."""
    M, N, K = 1280, 512, 576

    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        g = torch.Generator(device=dev).manual_seed(900 + r)
        out = a.create_buffer(M * N, torch.float32)
        x = torch.empty(M, K, dtype=torch.bfloat16, device=dev)
        wt = torch.empty(N, K, dtype=torch.bfloat16, device=dev)
        its = []
        for _ in range(3):
            x.copy_(torch.randint(-2, 3, (M, K), generator=g, device=dev))
            wt.copy_(torch.randint(-2, 3, (N, K), generator=g, device=dev))
            st = status_of(a)
            gemm_all_reduce(a, x, wt, out, variant=variant, status=st)
            its.append((x.clone(), wt.clone(), out.dev.view(M, N).clone(), st))
        torch.cuda.current_stream().synchronize()  # (a host wait inside the loop would hold the GIL the peer needs)
        return [(xi.cpu(), wi.cpu(), {"nk": (o.cpu(), int(st.item()), True)}) for xi, wi, o, st in its]

    res = A.run_cuda_ranks(devices(2), fn, CFG, heap_mb=64, max_ctas=4)
    for it in range(3):
        check_case(f"gemm_ar back-to-back call {it}", [per[it] for per in res], M, N, K, "dense", torch.float32,
                   2 * BM if variant == 2 else BM)


def test_gemm_all_reduce_reports_an_offset_mismatch_and_contains_it():
    """Rank 0 allocates (out, extra), rank 1 (extra, out): each rank's C sits where the peer keeps `extra`.  Both calls
    report DMA_MISMATCH_ERROR and neither rank writes into the peer's `extra`; a following call on buffers that line up
    is exact."""
    M, N, K = 1280, 256, 128

    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        x, wt = OPERANDS["dense"](M, N, K, w, 700 + r)
        x, wt = x.to(dev), wt.to(dev)
        first, second = a.create_buffer(M * N, torch.float32), a.create_buffer(M * N, torch.float32)
        out, extra = (first, second) if r == 0 else (second, first)
        extra.dev.fill_(SENTINEL)
        torch.cuda.current_stream().synchronize()
        a.barrier()  # the peer's sentinel is in place before anything could write into it
        st_bad = status_of(a)
        gemm_all_reduce(a, x, wt, out, status=st_bad)
        torch.cuda.current_stream().synchronize()
        untouched = bool((extra.dev == SENTINEL).all())
        good = a.create_buffer(M * N, torch.float32)
        st = status_of(a)
        gemm_all_reduce(a, x, wt, good, status=st)
        torch.cuda.current_stream().synchronize()
        return int(st_bad.item()), untouched, (x.cpu(), wt.cpu(), {"nk": (good.dev.view(M, N).cpu(), int(st.item()), True)})

    res = A.run_cuda_ranks(devices(2), fn, CFG, heap_mb=64, max_ctas=4)
    for r, (bad_status, untouched, _) in enumerate(res):
        assert untouched, f"rank {r}: the peer wrote into this rank's `extra` buffer"
        assert bad_status != -1 and bad_status & DMA_MISMATCH_ERROR, (r, hex(bad_status))
    check_case("gemm_ar after a mismatch", [good for *_, good in res], M, N, K, "dense", torch.float32, 2 * BM)


def test_gemm_all_reduce_rejects_bad_arguments():
    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        M, N, K = 256, 256, 128
        x = torch.zeros(M, K, dtype=torch.bfloat16, device=dev)
        wt = torch.zeros(N, K, dtype=torch.bfloat16, device=dev)
        out = a.create_buffer(M * N, torch.bfloat16)
        st = status_of(a)
        big_m, big_n = 128 * 513, 256 * 32  # 16416 tiles of 128 x 256, over the counter block's 16384
        bad = {
            "fp32 a": lambda: gemm_all_reduce(a, x.float(), wt, out, status=st),
            "fp32 w": lambda: gemm_all_reduce(a, x, wt.float(), out, status=st),
            "a on the CPU": lambda: gemm_all_reduce(a, x.cpu(), wt, out, status=st),
            "1-D a": lambda: gemm_all_reduce(a, x.view(-1), wt, out, status=st),
            "non-contiguous a": lambda: gemm_all_reduce(a, x.t(), torch.zeros(N, M, dtype=torch.bfloat16, device=dev),
                                                        out, status=st),
            "K mismatch": lambda: gemm_all_reduce(a, x, wt[:, :64].contiguous(), out, status=st),
            "M % 128": lambda: gemm_all_reduce(a, x[:192], wt, out, status=st),
            "N % 256": lambda: gemm_all_reduce(a, x, wt[:128], out, status=st),
            "K % 64": lambda: gemm_all_reduce(a, x[:, :96].contiguous(), wt[:, :96].contiguous(), out, status=st),
            "pair variant, M % 256": lambda: gemm_all_reduce(a, x[:128], wt, out, variant=2, status=st),
            "unknown variant": lambda: gemm_all_reduce(a, x, wt, out, variant=3, status=st),
            "unknown layout": lambda: gemm_all_reduce(a, x, wt, out, status=st, w_layout="t"),
            "kn, K mismatch": lambda: gemm_all_reduce(a, x, wt, out, status=st, w_layout="kn"),
            "out too small": lambda: gemm_all_reduce(a, x, wt, a.create_buffer(M * N - 1, torch.bfloat16), status=st),
            "out is a plain tensor": lambda: gemm_all_reduce(a, x, wt, torch.empty(M * N, dtype=torch.bfloat16,
                                                                                   device=dev), status=st),
            "fp16 out": lambda: gemm_all_reduce(a, x, wt, a.create_buffer(M * N, torch.float16), status=st),
            "out_dtype disagrees with out": lambda: gemm_all_reduce(a, x, wt, out, out_dtype=torch.float32, status=st),
            "int64 status": lambda: gemm_all_reduce(a, x, wt, out, status=torch.zeros(1, dtype=torch.int64, device=dev)),
            "over the tile limit": lambda: gemm_all_reduce(a, torch.zeros(big_m, 64, dtype=torch.bfloat16, device=dev),
                                                           torch.zeros(big_n, 64, dtype=torch.bfloat16, device=dev),
                                                           status=st),
        }
        for what, call in bad.items():
            try:
                call()
            except ValueError:
                continue
            raise AssertionError(f"no ValueError for: {what}")
        torch.cuda.current_stream().synchronize()
        return int(st.item())

    assert A.run_cuda_ranks([0], fn, CFG, heap_mb=64, max_ctas=4)[0] == -1  # nothing was enqueued


# ------------------------------------------------------------------------------------------------ layers
@pytest.fixture
def fused_calls(monkeypatch):
    """Counts the fused gemm_all_reduce calls by w_layout across the rank threads."""
    calls, lock = [], threading.Lock()
    real = ops.gemm_all_reduce

    def counting(*args, **kw):
        with lock:
            calls.append(("gemm_ar", kw.get("w_layout", "nk")))
        return real(*args, **kw)

    monkeypatch.setattr(ops, "gemm_all_reduce", counting)
    return calls


def rand(seed, *shape, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


def rel_err(got, ref):
    return float((got.double() - ref.double()).abs().max() / ref.double().abs().max())


def load_kernels(forward_local, xs, gys):
    """Runs the step's local math once on copies of the operands, so every kernel it needs is loaded before any fused
    call.  With ranks sharing one GPU in one process, loading a module can wait for the kernels running in the context,
    among them a peer's fused kernel that waits for this rank: the load would stall until that kernel's timeout."""
    for _ in range(2):  # the second pass accumulates into .grad
        for x, gy in zip(xs, gys):
            forward_local(x.detach().clone().requires_grad_()).backward(gy)
    torch.cuda.current_stream().synchronize()


def run_layers(world, build, micro_batches=1):
    """build(group, rank, world, device, micro_batches) -> (modules, forward, local forward on detached weight copies,
    inputs, upstream gradients).  Runs every forward, then the backwards in reverse order, syncs and checks the group's
    status word.  Returns per rank (inputs, weights, outputs, input grads, weight grads) on the CPU in fp32."""

    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        g = TensorGroup(a)
        mods, forward, local, xs, gys = build(g, r, w, dev, micro_batches)
        load_kernels(local, xs, gys)
        ys = [forward(x) for x in xs]
        for y, gy in reversed(list(zip(ys, gys))):
            y.backward(gy)
        torch.cuda.current_stream().synchronize()
        g.check(block=True)  # raises on a non-zero status of any fused call
        cpu = lambda t: t.detach().float().cpu()  # noqa: E731
        return ([cpu(x) for x in xs], [cpu(m.weight) for m in mods], [cpu(y) for y in ys], [cpu(x.grad) for x in xs],
                [cpu(m.weight.grad) for m in mods])

    return A.run_cuda_ranks(devices(world), fn, CFG, heap_mb=64, max_ctas=4)


def copies(mods):
    return [m.weight.detach().clone().requires_grad_() for m in mods]


@pytest.mark.parametrize("world", [1, 2])
def test_replicated_row_linear_forward_runs_on_the_all_reduce_kernel(world, fused_calls):
    m, Kr, N, seed = 256, 192, 256, 6000

    def build(g, r, w, dev, mbs):
        lin = ReplicatedRowParallelLinear(g, Kr, N)
        xs = [rand(seed + 10 * i + r, m, Kr).bfloat16().to(dev).requires_grad_() for i in range(mbs)]
        gys = [rand(seed + 100 + 10 * i, m, N, scale=0.1).bfloat16().to(dev) for i in range(mbs)]
        (wc,) = copies([lin])
        return [lin], lin, (lambda x: x @ wc.t()), xs, gys

    res = run_layers(world, build)
    X = torch.cat([xs[0] for xs, *_ in res], dim=1).requires_grad_()
    W = torch.cat([ws[0] for _, ws, *_ in res], dim=1).requires_grad_()
    gy = rand(seed + 100, m, N, scale=0.1).bfloat16().float()
    Y = X @ W.t()
    (Y * gy).sum().backward()
    for r, (_, _, ys, dxs, dws) in enumerate(res):
        assert torch.equal(ys[0], res[0][2][0]), f"rank {r}'s output differs from rank 0's"
        assert rel_err(ys[0], Y.detach()) < 1e-2, r
        assert rel_err(dxs[0], X.grad[:, r * Kr:(r + 1) * Kr]) < 1e-2, r
        assert rel_err(dws[0], W.grad[:, r * Kr:(r + 1) * Kr]) < 1e-2, r
    assert fused_calls == [("gemm_ar", "nk")] * world, fused_calls


@pytest.mark.parametrize("world", [1, 2])
def test_replicated_column_linear_backward_runs_on_the_kn_all_reduce_kernel(world, fused_calls):
    m, H, Nr, seed = 256, 256, 192, 7000

    def build(g, r, w, dev, mbs):
        lin = ReplicatedColumnParallelLinear(g, H, Nr)
        xs = [rand(seed + 10 * i, m, H).bfloat16().to(dev).requires_grad_() for i in range(mbs)]
        gys = [rand(seed + 100 + 10 * i + r, m, Nr, scale=0.1).bfloat16().to(dev) for i in range(mbs)]
        (wc,) = copies([lin])
        return [lin], lin, (lambda x: x @ wc.t()), xs, gys

    res = run_layers(world, build)
    X = rand(seed, m, H).bfloat16().float().requires_grad_()
    W = torch.cat([ws[0] for _, ws, *_ in res]).requires_grad_()
    gy = torch.cat([rand(seed + 100 + r, m, Nr, scale=0.1).bfloat16().float() for r in range(world)], dim=1)
    Y = X @ W.t()
    (Y * gy).sum().backward()
    for r, (_, _, ys, dxs, dws) in enumerate(res):
        assert rel_err(ys[0], Y.detach()[:, r * Nr:(r + 1) * Nr]) < 1e-2, r
        assert torch.equal(dxs[0], res[0][3][0]), f"rank {r}'s input gradient differs from rank 0's"
        assert rel_err(dxs[0], X.grad) < 1e-2, r
        assert rel_err(dws[0], W.grad[r * Nr:(r + 1) * Nr]) < 1e-2, r
    assert fused_calls == [("gemm_ar", "kn")] * world, fused_calls


def mlp_build(H_in, F, H_out, seed):
    """ReplicatedColumnParallelLinear(H_in -> F / P) -> GELU -> ReplicatedRowParallelLinear(F / P -> H_out)."""
    def build(g, r, w, dev, mbs):
        up, down = ReplicatedColumnParallelLinear(g, H_in, F // w), ReplicatedRowParallelLinear(g, F // w, H_out)
        xs = [rand(seed + 10 * i, 256, H_in).bfloat16().to(dev).requires_grad_() for i in range(mbs)]
        gys = [rand(seed + 100 + 10 * i, 256, H_out, scale=0.1).bfloat16().to(dev) for i in range(mbs)]
        w1, w2 = copies([up, down])
        return ([up, down], (lambda x: down(torch.nn.functional.gelu(up(x)))),
                (lambda x: torch.nn.functional.gelu(x @ w1.t()) @ w2.t()), xs, gys)
    return build


def check_mlp(res, world, micro_batches, H_in, F, H_out, seed):
    W1 = torch.cat([ws[0] for _, ws, *_ in res]).requires_grad_()
    W2 = torch.cat([ws[1] for _, ws, *_ in res], dim=1).requires_grad_()
    Xs = []
    for i in range(micro_batches):
        X = rand(seed + 10 * i, 256, H_in).bfloat16().float().requires_grad_()
        gy = rand(seed + 100 + 10 * i, 256, H_out, scale=0.1).bfloat16().float()
        Y = torch.nn.functional.gelu(X @ W1.t()) @ W2.t()
        (Y * gy).sum().backward()
        Xs.append((X, Y.detach()))
    n = F // world
    for r, (_, _, ys, dxs, dws) in enumerate(res):
        for i, (X, Y) in enumerate(Xs):
            assert rel_err(ys[i], Y) < 3e-2, (r, i)
            assert rel_err(dxs[i], X.grad) < 3e-2, (r, i)
        assert rel_err(dws[0], W1.grad[r * n:(r + 1) * n]) < 3e-2, r
        assert rel_err(dws[1], W2.grad[:, r * n:(r + 1) * n]) < 3e-2, r


@pytest.mark.parametrize("world,micro_batches", [(1, 1), (2, 1), (2, 2)], ids=["world1", "world2", "world2-2mb"])
def test_replicated_mlp_gradients_match_the_unsharded_reference(world, micro_batches, fused_calls):
    """Column -> GELU -> row; with two micro-batches both forwards run before either backward."""
    H, F, seed = 256, 512, 8000
    res = run_layers(world, mlp_build(H, F, H, seed), micro_batches)
    check_mlp(res, world, micro_batches, H, F, H, seed)
    per_pass = [("gemm_ar", "nk"), ("gemm_ar", "kn")]
    assert sorted(fused_calls) == sorted(per_pass * world * micro_batches), fused_calls


def test_replicated_mlp_fused_forward_with_fallback_backward(fused_calls):
    """Input width 192: the row layer's forward fuses (N = 256), the column layer's input gradient cannot (K % 256) and
    runs matmul + all_reduce."""
    world, H_in, F, H_out, seed = 2, 192, 512, 256, 9000
    res = run_layers(world, mlp_build(H_in, F, H_out, seed))
    check_mlp(res, world, 1, H_in, F, H_out, seed)
    assert fused_calls == [("gemm_ar", "nk")] * world, fused_calls


def test_replicated_column_offset_mismatch_in_backward_is_reported_at_check():
    """The column layer's backward heap buffer sits at different offsets on the two ranks (allocated around a pad in
    opposite orders): the fused all-reduce of the input gradient reports DMA_MISMATCH_ERROR, and
    TensorGroup.check(block=True) raises."""
    m, H, Nr = 256, 256, 256

    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        g = TensorGroup(a)
        lin = ReplicatedColumnParallelLinear(g, H, Nr)
        first, second = a.create_buffer(m * H, torch.bfloat16), a.create_buffer(m * H, torch.bfloat16)
        lin._dx, pad = (first, second) if r == 0 else (second, first)
        x = rand(5000, m, H).bfloat16().to(dev).requires_grad_()
        (wc,) = copies([lin])
        load_kernels(lambda t: t @ wc.t(), [x], [torch.ones(m, Nr, dtype=torch.bfloat16, device=dev)])
        y = lin(x)
        y.backward(torch.ones_like(y))
        torch.cuda.current_stream().synchronize()
        try:
            g.check(block=True)
        except RuntimeError as e:
            return str(e), pad is not None
        return None, True

    for r, (err, _) in enumerate(A.run_cuda_ranks(devices(2), fn, CFG, heap_mb=64, max_ctas=4)):
        assert err is not None and "DMA_MISMATCH_ERROR" in err, (r, err)
