"""GPU tests of the [K, N] ("kn") weight layout of the two fused wgmma GEMM plugins, and of the backward passes of the
sequence-parallel linears that run on them.

* ops: "kn" on W [K, N] against the fp64 reference (exact for integer operands, within the computed bound for random
  ones, as tests/test_cuda_gemm_exact.py does for "nk"), and bit for bit against "nk" on W^T: the same wgmma
  instruction on the same values, only the B operand's shared-memory layout differs (for gemm_reduce_scatter wherever
  the reduction of the ranks' partials does not depend on their arrival order).
* layers at world 1 and 2: gradients against single-process fp32 autograd on the unsharded problem, with the fused
  calls counted, a fused forward with a fallback backward, two micro-batches before backward, and a shard-offset
  mismatch in backward reported by TensorGroup.check.
"""
import threading

import pytest
import torch

import accl_b200 as A
import accl_b200.ops as ops
from accl_b200.ops import all_gather_gemm, gemm_reduce_scatter
from accl_b200.parallel import RowParallelLinear, SeqParallelColumnLinear, TensorGroup
from test_cuda_gemm_exact import (BM, CFG, GUARD_ROWS, M_OF_WORLD, OPERANDS, RS_IDS, RS_KERNELS, SENTINEL,
                                  check_ag_gemm_case, check_gemm_rs_case, devices, seed_of, skip_over_budget, status_of)

pytestmark = pytest.mark.gpu

KN_KS = (64, 192, 576, 8192)
KN_RANDOM_KS = (576, 8192)
KN_SHAPES = [(1, 256), (1, 768), (2, 256), (2, 768), (3, 256), (3, 768), (4, 256), (4, 768)]


def kn_cases(exact_kind):
    return [(K, exact_kind) for K in KN_KS] + [(K, "random") for K in KN_RANDOM_KS]


# ------------------------------------------------------------------------------------------------ ops
def run_gemm_rs_kn_cases(world, M, N, cases, variant, out_dtype, tag):
    """Per case a "kn" call on W^T [K, N] and an "nk" call on W [N, K], each into fresh sentinel-guarded heap buffers.
    Returns per rank per case ((A_r, W_r, kn shard, kn status, guards intact), nk shard, nk status)."""

    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        keep, res = [], []
        for K, kind in cases:
            x, wt = OPERANDS[kind](M, N, K, w, seed_of(tag, world, N, K, len(kind), r))
            x, wt = x.to(dev), wt.to(dev)
            w_kn = wt.t().contiguous()
            rows = M // w
            got = []
            for layout, wmat in (("kn", w_kn), ("nk", wt)):
                pre, out, post = (a.create_buffer(n, out_dtype) for n in (GUARD_ROWS * N, rows * N, GUARD_ROWS * N))
                for b in (pre, out, post):
                    b.dev.fill_(SENTINEL)
                st = status_of(a)
                gemm_reduce_scatter(a, x, wmat, out, variant=variant, status=st, w_layout=layout)
                got.append((pre, out, post, st))
                keep.append((pre, out, post))
            torch.cuda.current_stream().synchronize()
            (pre, out, post, st), (_, out_nk, _, st_nk) = got
            guards = bool((pre.dev == SENTINEL).all()) and bool((post.dev == SENTINEL).all())
            res.append(((x.cpu(), wt.cpu(), out.dev.view(rows, N).cpu(), int(st.item()), guards),
                        out_nk.dev.view(rows, N).cpu(), int(st_nk.item())))
        del keep
        return res

    return A.run_cuda_ranks(devices(world), fn, CFG, timeout=600.0, heap_mb=256 if world == 1 else 128, max_ctas=4)


@pytest.mark.parametrize("world,N", KN_SHAPES, ids=[f"world{w}-N{n}" for w, n in KN_SHAPES])
@pytest.mark.parametrize("variant,out_dtype", RS_KERNELS, ids=RS_IDS)
def test_gemm_reduce_scatter_kn_is_exact_and_equals_nk(variant, out_dtype, world, N):
    M = M_OF_WORLD[world]
    kernel = "pair" if variant == 2 else "single"
    skip_over_budget(kernel, M, N, devices(world))
    cases = kn_cases("sparse" if out_dtype == torch.bfloat16 and world > 1 else "dense")
    res = run_gemm_rs_kn_cases(world, M, N, cases, variant, out_dtype, tag=20 + variant * 2 + (out_dtype == torch.float32))
    what = f"gemm_rs kn {kernel} {str(out_dtype)[6:]} world {world} M={M} N={N}"
    for i, (K, kind) in enumerate(cases):
        per_rank = [per[i] for per in res]
        check_gemm_rs_case(what, [kn for kn, _, _ in per_rank], M, N, K, kind, out_dtype, 2 * BM if variant == 2 else BM)
        # the TMA unit adds the ranks' partial tiles into a shard in arrival order, which differs from call to call: with
        # random operands and three or more partials the rounded sum depends on it (two calls of "nk" differ too), so
        # kn and nk are compared bit for bit where the sum is order-independent: integer operands, or world <= 2
        order_free = kind != "random" or world <= 2
        for r, ((_, _, shard, _, _), shard_nk, st_nk) in enumerate(per_rank):
            assert st_nk == 0, f"{what} K={K} {kind} rank {r}: nk status {st_nk:#x}"
            assert not order_free or torch.equal(shard, shard_nk), f"{what} K={K} {kind} rank {r}: kn differs from nk on W^T"


def run_ag_gemm_kn_cases(world, M, N, cases, tag):
    """Per case an "nk" call on W [N, K] and a "kn" call on W^T [K, N] over the same heap shard, out and gathered carved
    out of sentinel-filled tensors.  Returns per rank per case ((shard, W_r, kn out, kn gathered, kn status, guards
    intact), nk out, nk status)."""

    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        keep, res = [], []
        for K, kind in cases:
            s, wt = OPERANDS[kind](M // w, N, K, w, seed_of(tag, world, N, K, len(kind), r))
            wt = wt.to(dev)
            buf = a.create_buffer(M // w * K, torch.bfloat16)
            shard = buf.dev.view(M // w, K)
            shard.copy_(s.to(dev))
            keep.append(buf)
            got = []
            for layout, wmat in (("kn", wt.t().contiguous()), ("nk", wt)):
                out_all = torch.full((M + 2 * GUARD_ROWS, N), SENTINEL, dtype=torch.bfloat16, device=dev)
                gathered_all = torch.full((M + 2 * GUARD_ROWS, K), SENTINEL, dtype=torch.bfloat16, device=dev)
                st = status_of(a)
                out, gathered = all_gather_gemm(a, shard, wmat, out=out_all[GUARD_ROWS:GUARD_ROWS + M],
                                                gathered=gathered_all[GUARD_ROWS:GUARD_ROWS + M], status=st, w_layout=layout)
                got.append((out_all, gathered_all, out, gathered, st))
            torch.cuda.current_stream().synchronize()
            (out_all, gathered_all, out, gathered, st), (_, _, out_nk, _, st_nk) = got
            guards = all(bool((t[:GUARD_ROWS] == SENTINEL).all()) and bool((t[GUARD_ROWS + M:] == SENTINEL).all())
                         for t in (out_all, gathered_all))
            res.append(((s, wt.cpu(), out.cpu(), gathered.cpu(), int(st.item()), guards), out_nk.cpu(), int(st_nk.item())))
        del keep
        return res

    return A.run_cuda_ranks(devices(world), fn, CFG, timeout=600.0, heap_mb=256 if world == 1 else 128, max_ctas=4)


@pytest.mark.parametrize("world,N", KN_SHAPES, ids=[f"world{w}-N{n}" for w, n in KN_SHAPES])
def test_all_gather_gemm_kn_is_exact_and_equals_nk(world, N):
    M = M_OF_WORLD[world]
    skip_over_budget("single", M, N, devices(world))
    cases = kn_cases("dense")
    res = run_ag_gemm_kn_cases(world, M, N, cases, tag=29)
    what = f"ag_gemm kn world {world} M={M} N={N}"
    for i, (K, kind) in enumerate(cases):
        per_rank = [per[i] for per in res]
        check_ag_gemm_case(what, [kn for kn, _, _ in per_rank], M, N, K, kind)
        for r, ((_, _, out, _, _, _), out_nk, st_nk) in enumerate(per_rank):
            assert st_nk == 0, f"{what} K={K} {kind} rank {r}: nk status {st_nk:#x}"
            assert torch.equal(out, out_nk), f"{what} K={K} {kind} rank {r}: kn differs from nk on W^T"


def test_kn_layout_rejects_bad_arguments():
    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        M, N, K = 256, 256, 128
        x = torch.zeros(M, K, dtype=torch.bfloat16, device=dev)
        w_kn = torch.zeros(K, N, dtype=torch.bfloat16, device=dev)
        out = a.create_buffer(M * N, torch.bfloat16)
        shard = a.create_buffer(M * K, torch.bfloat16).dev.view(M, K)
        st = status_of(a)
        bad = {
            "unknown layout": lambda: gemm_reduce_scatter(a, x, w_kn, out, status=st, w_layout="t"),
            "nk-shaped w as kn": lambda: gemm_reduce_scatter(a, x, torch.zeros(N, 64, dtype=torch.bfloat16, device=dev),
                                                             out, status=st, w_layout="kn"),
            "kn, N % 256": lambda: gemm_reduce_scatter(a, x, w_kn[:, :128].contiguous(), out, status=st, w_layout="kn"),
            "kn, K % 64": lambda: gemm_reduce_scatter(a, x[:, :96].contiguous(), w_kn[:96].contiguous(), out, status=st,
                                                      w_layout="kn"),
            "ag unknown layout": lambda: all_gather_gemm(a, shard, w_kn, status=st, w_layout="NK"),
            "ag kn, K mismatch": lambda: all_gather_gemm(a, shard, w_kn[:64].contiguous(), status=st, w_layout="kn"),
            "ag kn, N % 256": lambda: all_gather_gemm(a, shard, w_kn[:, :128].contiguous(), status=st, w_layout="kn"),
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
    """Counts the fused plugin calls by (op, w_layout) across the rank threads."""
    calls, lock = [], threading.Lock()

    def counting(name, fn):
        def wrapper(*args, **kw):
            with lock:
                calls.append((name, kw.get("w_layout", "nk")))
            return fn(*args, **kw)
        return wrapper

    monkeypatch.setattr(ops, "gemm_reduce_scatter", counting("gemm_rs", ops.gemm_reduce_scatter))
    monkeypatch.setattr(ops, "all_gather_gemm", counting("ag_gemm", ops.all_gather_gemm))
    return calls


def rand(seed, *shape, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


def rel_err(got, ref):
    return float((got.double() - ref.double()).abs().max() / ref.double().abs().max())


def load_kernels(mods, xs, gys, world):
    """Runs the local matmuls, GELU and gradient accumulation of the step once on an unsharded replica, so their
    kernels are loaded before any fused call.  With ranks sharing one GPU in one process, loading a module can wait for
    the kernels running in the context, among them a peer's fused kernel that waits for this rank: the load would
    stall until that kernel's timeout (one process per GPU, as in training, does not share a context with its peers)."""
    ws = [m.weight.detach().clone().requires_grad_() for m in mods]
    for _ in range(2):  # the second pass accumulates into .grad
        for x, gy in zip(xs, gys):
            h = x.detach().repeat(world, 1) if isinstance(mods[0], SeqParallelColumnLinear) else x.detach()
            h = h.requires_grad_()
            y = h @ ws[0].t()
            if len(ws) == 2:
                y = torch.nn.functional.gelu(y) @ ws[1].t()
            y.backward(torch.cat([gy] * (y.shape[0] // gy.shape[0]))[:, :y.shape[1]].contiguous())
    torch.cuda.current_stream().synchronize()


def run_layers(world, build, micro_batches=1):
    """build(group, rank, world, device, micro_batches) -> (modules, forward, inputs, upstream gradients), one input
    and one upstream gradient per micro-batch.  Runs every
    forward, then the backwards in reverse order, syncs and checks the group's status word.  Returns per rank
    (inputs, weights, outputs, input grads, weight grads) on the CPU in fp32."""

    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        g = TensorGroup(a)
        mods, forward, xs, gys = build(g, r, w, dev, micro_batches)
        load_kernels(mods, xs, gys, w)
        ys = [forward(x) for x in xs]
        for y, gy in reversed(list(zip(ys, gys))):
            y.backward(gy)
        torch.cuda.current_stream().synchronize()
        g.check(block=True)  # raises on a non-zero status of any fused call
        cpu = lambda t: t.detach().float().cpu()  # noqa: E731
        return ([cpu(x) for x in xs], [cpu(m.weight) for m in mods], [cpu(y) for y in ys], [cpu(x.grad) for x in xs],
                [cpu(m.weight.grad) for m in mods])

    return A.run_cuda_ranks(devices(world), fn, CFG, heap_mb=64, max_ctas=4)


def column_build(S, H, Nr, seed):
    def build(g, r, w, dev, mbs):
        lin = SeqParallelColumnLinear(g, H, Nr)
        xs = [rand(seed + 10 * i + r, S, H).bfloat16().to(dev).requires_grad_() for i in range(mbs)]
        gys = [rand(seed + 100 + 10 * i + r, S * w, Nr, scale=0.1).bfloat16().to(dev) for i in range(mbs)]
        return [lin], lin, xs, gys
    return build


def row_build(Mr, Kr, N, seed):
    """Mr: output rows per rank (the input has Mr * world rows)."""
    def build(g, r, w, dev, mbs):
        lin = RowParallelLinear(g, Kr, N)
        xs = [rand(seed + 10 * i + r, Mr * w, Kr).bfloat16().to(dev).requires_grad_() for i in range(mbs)]
        gys = [rand(seed + 100 + 10 * i + r, Mr, N, scale=0.1).bfloat16().to(dev) for i in range(mbs)]
        return [lin], lin, xs, gys
    return build


@pytest.mark.parametrize("world", [1, 2])
def test_column_linear_backward_runs_on_the_kn_reduce_scatter_kernel(world, fused_calls):
    S, H, Nr, seed = 256, 256, 256, 1000
    res = run_layers(world, column_build(S, H, Nr, seed))
    X = torch.cat([xs[0] for xs, *_ in res]).requires_grad_()
    W = torch.cat([ws[0] for _, ws, *_ in res]).requires_grad_()
    gy = torch.cat([rand(seed + 100 + r, S * world, Nr, scale=0.1).bfloat16().float() for r in range(world)], dim=1)
    Y = X @ W.t()
    (Y * gy).sum().backward()
    for r, (_, _, ys, dxs, dws) in enumerate(res):
        assert rel_err(ys[0], Y.detach()[:, r * Nr:(r + 1) * Nr]) < 1e-2, r
        assert rel_err(dxs[0], X.grad[r * S:(r + 1) * S]) < 1e-2, r
        assert rel_err(dws[0], W.grad[r * Nr:(r + 1) * Nr]) < 1e-2, r
    assert sorted(fused_calls) == sorted([("ag_gemm", "nk"), ("gemm_rs", "kn")] * world), fused_calls


@pytest.mark.parametrize("world", [1, 2])
def test_row_linear_backward_runs_on_the_kn_all_gather_kernel(world, fused_calls):
    Mr, Kr, N, seed = 256, 256, 256, 2000
    res = run_layers(world, row_build(Mr, Kr, N, seed))
    X = torch.cat([xs[0] for xs, *_ in res], dim=1).requires_grad_()
    W = torch.cat([ws[0] for _, ws, *_ in res], dim=1).requires_grad_()
    gy = torch.cat([rand(seed + 100 + r, Mr, N, scale=0.1).bfloat16().float() for r in range(world)])
    Y = X @ W.t()
    (Y * gy).sum().backward()
    for r, (_, _, ys, dxs, dws) in enumerate(res):
        assert rel_err(ys[0], Y.detach()[r * Mr:(r + 1) * Mr]) < 1e-2, r
        assert rel_err(dxs[0], X.grad[:, r * Kr:(r + 1) * Kr]) < 1e-2, r
        assert rel_err(dws[0], W.grad[:, r * Kr:(r + 1) * Kr]) < 1e-2, r
    assert sorted(fused_calls) == sorted([("ag_gemm", "kn"), ("gemm_rs", "nk")] * world), fused_calls


def test_row_linear_fused_forward_with_fallback_backward(fused_calls):
    """K_r = 192: the forward fuses (K_r % 64), the backward cannot (K_r % 256) and runs all_gather + matmul."""
    world, Mr, Kr, N, seed = 2, 256, 192, 256, 3000
    res = run_layers(world, row_build(Mr, Kr, N, seed))
    X = torch.cat([xs[0] for xs, *_ in res], dim=1).requires_grad_()
    W = torch.cat([ws[0] for _, ws, *_ in res], dim=1).requires_grad_()
    gy = torch.cat([rand(seed + 100 + r, Mr, N, scale=0.1).bfloat16().float() for r in range(world)])
    Y = X @ W.t()
    (Y * gy).sum().backward()
    for r, (_, _, ys, dxs, dws) in enumerate(res):
        assert rel_err(ys[0], Y.detach()[r * Mr:(r + 1) * Mr]) < 1e-2, r
        assert rel_err(dxs[0], X.grad[:, r * Kr:(r + 1) * Kr]) < 1e-2, r
        assert rel_err(dws[0], W.grad[:, r * Kr:(r + 1) * Kr]) < 1e-2, r
    assert fused_calls == [("gemm_rs", "nk")] * world, fused_calls


@pytest.mark.parametrize("world,micro_batches", [(1, 1), (2, 1), (2, 2)], ids=["world1", "world2", "world2-2mb"])
def test_mlp_gradients_match_the_unsharded_reference(world, micro_batches, fused_calls):
    """Column -> GELU -> row; with two micro-batches both forwards run before either backward."""
    S, H, F, seed = 256, 256, 512, 4000

    def build(g, r, w, dev, mbs):
        up, down = SeqParallelColumnLinear(g, H, F // w), RowParallelLinear(g, F // w, H)
        xs = [rand(seed + 10 * i + r, S, H).bfloat16().to(dev).requires_grad_() for i in range(mbs)]
        gys = [rand(seed + 100 + 10 * i + r, S, H, scale=0.1).bfloat16().to(dev) for i in range(mbs)]
        return [up, down], (lambda x: down(torch.nn.functional.gelu(up(x)))), xs, gys

    res = run_layers(world, build, micro_batches)
    W1 = torch.cat([ws[0] for _, ws, *_ in res]).requires_grad_()
    W2 = torch.cat([ws[1] for _, ws, *_ in res], dim=1).requires_grad_()
    Xs = []
    for i in range(micro_batches):
        X = torch.cat([xs[i] for xs, *_ in res]).requires_grad_()
        gy = torch.cat([rand(seed + 100 + 10 * i + r, S, H, scale=0.1).bfloat16().float() for r in range(world)])
        Y = torch.nn.functional.gelu(X @ W1.t()) @ W2.t()
        (Y * gy).sum().backward()
        Xs.append((X, Y.detach()))
    n = F // world
    for r, (_, _, ys, dxs, dws) in enumerate(res):
        for i, (X, Y) in enumerate(Xs):
            assert rel_err(ys[i], Y[r * S:(r + 1) * S]) < 3e-2, (r, i)
            assert rel_err(dxs[i], X.grad[r * S:(r + 1) * S]) < 3e-2, (r, i)
        assert rel_err(dws[0], W1.grad[r * n:(r + 1) * n]) < 3e-2, r
        assert rel_err(dws[1], W2.grad[:, r * n:(r + 1) * n]) < 3e-2, r
    per_pass = [("ag_gemm", "nk"), ("gemm_rs", "nk"), ("ag_gemm", "kn"), ("gemm_rs", "kn")]
    assert sorted(fused_calls) == sorted(per_pass * world * micro_batches), fused_calls


def test_shard_offset_mismatch_in_backward_is_reported_at_check():
    """The column layer's backward heap buffer sits at different offsets on the two ranks (allocated around a pad in
    opposite orders, so every later buffer lines up again): the forward is clean, the backward's fused reduce-scatter
    reports DMA_MISMATCH_ERROR, and TensorGroup.check(block=True) raises."""
    S, H, Nr = 256, 256, 256

    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        g = TensorGroup(a)
        lin = SeqParallelColumnLinear(g, H, Nr)
        first, second = a.create_buffer(S * H, torch.bfloat16), a.create_buffer(S * H, torch.bfloat16)
        lin._dx_shard, pad = (first, second) if r == 0 else (second, first)
        x = rand(5000 + r, S, H).bfloat16().to(dev).requires_grad_()
        y = lin(x)
        torch.cuda.current_stream().synchronize()
        g.check(block=True)  # the forward's shards line up
        y.backward(torch.ones_like(y))
        torch.cuda.current_stream().synchronize()
        try:
            g.check(block=True)
        except RuntimeError as e:
            return str(e), pad is not None
        return None, True

    for r, (err, _) in enumerate(A.run_cuda_ranks(devices(2), fn, CFG, heap_mb=64, max_ctas=4)):
        assert err is not None and "DMA_MISMATCH_ERROR" in err, (r, err)
