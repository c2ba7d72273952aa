"""GPU tests of the fused all-reduce -> residual add -> RMSNorm plugin (ops.all_reduce_rmsnorm) and of the
AllReduceRMSNorm layer that runs on it.  Ranks are threads (run_cuda_ranks) on the GPUs present, max_ctas=4.

* ops: residual_out bit-equal to the fp32 rank-order sum rounded once to bf16, out a faithful rounding of the fp64
  RMSNorm of residual_out, every replica bit-identical to rank 0's, the one-shot and two-shot forms (forced with the
  "oneshot_max_bytes" knob) bit-identical to each other, x unchanged, sentinel guards around residual_out and out.
  M covers one row, M < P and M not a multiple of P; H the narrowest and widest rows; a row of zeros exercises eps;
  without a residual, with one, and updated in place (residual_out is residual).
* back-to-back calls with x rewritten on the stream right after each call, an x at another heap offset on one rank,
  bad arguments.
* the layer at world 1 and 2: the fused call counted, gradients against fp32 autograd, two micro-batches, and an offset
  mismatch reported by TensorGroup.check.
"""
import threading

import pytest
import torch

import accl_b200 as A
import accl_b200.ops as ops
from accl_b200.ops import all_reduce_rmsnorm
from accl_b200.parallel import AllReduceRMSNorm, TensorGroup
from test_cuda_gemm_exact import CFG, DMA_MISMATCH_ERROR, SENTINEL, devices, status_of

pytestmark = pytest.mark.gpu

EPS = 1e-6
GUARD = 4096  # sentinel elements before and after every output
FORMS = {"oneshot": 1 << 40, "twoshot": 0}  # oneshot_max_bytes that forces each form
# (M, H): one row; M < P for P > 2; M not a multiple of 2, 3 or 4; the widest and the narrowest rows
CASES = [(1, 16384), (2, 4096), (7, 16384), (128, 8), (1000, 1032), (4096, 1032)]
RESIDUALS = ("none", "separate", "inplace")


def operands(M, H, P, seed):
    """Per rank x_r, the replicated residual and gain.  Row M // 2 is zero in every x_r and in the residual (for M > 1):
    its h is zero and its norm is eps alone."""
    g = torch.Generator().manual_seed(seed)
    xs = [torch.randn(M, H, generator=g).bfloat16() for _ in range(P)]
    res = torch.randn(M, H, generator=g).bfloat16()
    gamma = (1 + 0.5 * torch.randn(H, generator=g)).bfloat16()
    if M > 1:
        for x in xs:
            x[M // 2] = 0
        res[M // 2] = 0
    return xs, res, gamma


def reference_h(xs, res):
    acc = xs[0].float()
    for x in xs[1:]:
        acc += x.float()
    if res is not None:
        acc += res.float()
    return acc.bfloat16()


def faithful_failure(label, got, h, gamma, eps=EPS):
    """None when every element of `got` is one of the two bf16 neighbours of the fp64 RMSNorm of h (the value itself
    when it is a bf16 number), else a message naming the first element that is not."""
    hd = h.double()
    yd = hd * torch.rsqrt((hd * hd).mean(-1, keepdim=True) + eps) * gamma.double()
    bits = yd.view(torch.int64)
    low = bits & -(1 << 45)  # bf16 keeps 7 of fp64's 52 fraction bits: truncate toward zero
    lo, hi = low.view(torch.float64), (low + (1 << 45)).view(torch.float64)
    g = got.double()
    ok = (g == lo) | ((g == hi) & (lo != yd))
    if bool(ok.all()):
        return None
    r, c = (~ok).nonzero()[0].tolist()
    return (f"{label}: out[{r}, {c}] = {float(g[r, c])!r}, the fp64 value is {float(yd[r, c])!r} "
            f"({int((~ok).sum())} elements not faithfully rounded)")


def warm(dev):
    """Runs the torch kernels the rank threads use around the fused calls once, so none is loaded between calls.  With
    ranks sharing one GPU in one process, loading a module can wait for the kernels running in the context, among them
    a peer's fused kernel that waits for this rank's next call.  For the same reason the tests stage every operand on
    the device, and meet on a thread barrier, before the first fused call: a copy from pageable host memory waits for
    the rank's stream, and a rank thread that waits there keeps its peers from launching."""
    t = torch.full((64,), SENTINEL, dtype=torch.bfloat16, device=dev)
    t.fill_(0)
    bool((t == SENTINEL).all())
    bool(t.any())
    t.clone()
    torch.full((1,), -1, dtype=torch.int32, device=dev)
    torch.cuda.current_stream().synchronize()


def guarded_heap(a, n):
    """(pre, mid, post) bf16 heap buffers, pre and post sentinel-filled."""
    bufs = tuple(a.create_buffer(k, torch.bfloat16) for k in (GUARD, n, GUARD))
    bufs[0].dev.fill_(SENTINEL)
    bufs[2].dev.fill_(SENTINEL)
    return bufs


def run_ops(world, cases, seed):
    """Per case, per form and per residual mode, one call into fresh guarded outputs.  Returns per rank per case
    {(form, mode): (h, out, status, guards intact, x unchanged)} on the CPU."""

    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        warm(dev)
        staged = []
        for i, (M, H) in enumerate(cases):
            xs, res, gamma = operands(M, H, w, seed + i)
            staged.append((xs[r].to(dev), res.to(dev), gamma.to(dev)))
        torch.cuda.current_stream().synchronize()
        ready.wait()
        res_all = []
        for i, (M, H) in enumerate(cases):
            x_d, res_d, gamma_d = staged[i]
            xbuf = a.create_buffer(M * H, torch.bfloat16)
            x = xbuf.dev.view(M, H)
            x.copy_(x_d)
            got = {}
            for form, limit in FORMS.items():
                a.set_tuning("oneshot_max_bytes", limit)
                for mode in RESIDUALS:
                    pre, hb, post = guarded_heap(a, M * H)
                    h = hb.dev.view(M, H)
                    out_full = torch.full(((M + 2 * (GUARD // H + 1)) * H,), SENTINEL, dtype=torch.bfloat16, device=dev)
                    o0 = (GUARD // H + 1) * H
                    out = out_full[o0:o0 + M * H].view(M, H)
                    residual = None
                    if mode == "separate":
                        residual = res_d
                    elif mode == "inplace":
                        h.copy_(res_d)
                        residual = h
                    st = status_of(a)
                    y, h_ret = all_reduce_rmsnorm(a, x, gamma_d, residual, EPS, out=out, residual_out=h, status=st)
                    assert y is out and h_ret is h
                    got[(form, mode)] = (pre, hb, post, out_full, o0, st)
            torch.cuda.current_stream().synchronize()
            x_same = bool((x == x_d).all())
            per = {}
            for key, (pre, hb, post, out_full, o0, st) in got.items():
                guards = (bool((pre.dev == SENTINEL).all()) and bool((post.dev == SENTINEL).all()) and
                          bool((out_full[:o0] == SENTINEL).all()) and bool((out_full[o0 + M * H:] == SENTINEL).all()))
                per[key] = (hb.dev.view(M, H).cpu(), out_full[o0:o0 + M * H].view(M, H).cpu(), int(st.item()), guards,
                            x_same)
            res_all.append(per)
            del got, x, xbuf
        a.set_tuning("oneshot_max_bytes", 2048 << 10)
        return res_all

    ready = threading.Barrier(world)
    return A.run_cuda_ranks(devices(world), fn, CFG, timeout=600.0, heap_mb=512, max_ctas=4)


def check_ops(world, cases, seed, res):
    for i, (M, H) in enumerate(cases):
        xs, rz, gamma = operands(M, H, world, seed + i)
        for mode in RESIDUALS:
            want_h = reference_h(xs, None if mode == "none" else rz)
            for form in FORMS:
                for r in range(world):
                    h, out, status, guards, x_same = res[r][i][(form, mode)]
                    label = f"world {world} M={M} H={H} {form} residual {mode} rank {r}"
                    assert status == 0, f"{label}: status {status:#x}"
                    assert guards, f"{label}: a guard around residual_out or out was written"
                    assert x_same, f"{label}: x changed"
                    if not torch.equal(h, want_h):
                        bad = (h.float() != want_h.float()).nonzero()[0].tolist()
                        raise AssertionError(f"{label}: residual_out[{bad[0]}, {bad[1]}] = {float(h[tuple(bad)])}, "
                                             f"want {float(want_h[tuple(bad)])}")
                    msg = faithful_failure(label, out, want_h, gamma)
                    assert msg is None, msg
                    h0, out0 = res[0][i][(form, mode)][:2]
                    assert torch.equal(h, h0), f"{label}: residual_out differs from rank 0's"
                    assert torch.equal(out, out0), f"{label}: out differs from rank 0's"
                one, two = res[0][i][("oneshot", mode)][1], res[0][i][("twoshot", mode)][1]
                assert torch.equal(one, two), f"world {world} M={M} H={H} residual {mode}: one-shot and two-shot differ"
            if M > 1:
                assert not res[0][i][("oneshot", mode)][1][M // 2].any(), "the zero row's norm is not zero"


@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_all_reduce_rmsnorm_is_exact_replicated_and_form_independent(world):
    seed = 100 * world
    check_ops(world, CASES, seed, run_ops(world, CASES, seed))


@pytest.mark.parametrize("world", [2, 3])
def test_all_reduce_rmsnorm_back_to_back_calls_with_x_rewritten(world):
    """Three calls per form into the same residual_out; each rank rewrites x on its stream right after every call.  The
    one-shot exit meeting and the two-shot middle meeting must keep the peers' reads ahead of the rewrite."""
    M, H = 96, 4096

    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        warm(dev)
        staged = {}
        for j in range(len(FORMS)):
            for it in range(3):
                xs, res, gamma = operands(M, H, w, 7000 + 10 * j + it)
                staged[j, it] = (xs[r].to(dev), res.to(dev), gamma.to(dev))
        x = a.create_buffer(M * H, torch.bfloat16).dev.view(M, H)
        h = a.create_buffer(M * H, torch.bfloat16).dev.view(M, H)
        out = torch.empty(M, H, dtype=torch.bfloat16, device=dev)
        torch.cuda.current_stream().synchronize()
        ready.wait()
        runs = []
        for j, (form, limit) in enumerate(FORMS.items()):
            a.set_tuning("oneshot_max_bytes", limit)
            for it in range(3):
                x_d, res_d, gamma_d = staged[j, it]
                x.copy_(x_d)
                st = status_of(a)
                all_reduce_rmsnorm(a, x, gamma_d, res_d, EPS, out=out, residual_out=h, status=st)
                x.fill_(SENTINEL)  # the next call's operands come from a fresh generator
                runs.append((form, it, h.clone(), out.clone(), st))
        torch.cuda.current_stream().synchronize()
        return [(form, it, hh.cpu(), oo.cpu(), int(st.item())) for form, it, hh, oo, st in runs]

    ready = threading.Barrier(world)
    res = A.run_cuda_ranks(devices(world), fn, CFG, heap_mb=64, max_ctas=4)
    for k, (form, it, *_rest) in enumerate(res[0]):
        xs, rz, gamma = operands(M, H, world, 7000 + 10 * list(FORMS).index(form) + it)
        want_h = reference_h(xs, rz)
        for r in range(world):
            _, _, h, out, status = res[r][k]
            label = f"world {world} {form} call {it} rank {r}"
            assert status == 0, f"{label}: status {status:#x}"
            assert torch.equal(h, want_h), f"{label}: residual_out is not the rank-order sum"
            msg = faithful_failure(label, out, want_h, gamma)
            assert msg is None, msg


@pytest.mark.parametrize("form", list(FORMS))
def test_all_reduce_rmsnorm_reports_an_offset_mismatch_and_contains_it(form):
    """World 3; rank 2's x sits at another heap offset.  Every rank reports DMA_MISMATCH_ERROR, nobody writes outside its
    residual_out, and a following call on buffers that line up is exact."""
    world, M, H = 3, 12, 1024

    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        warm(dev)
        a.set_tuning("oneshot_max_bytes", FORMS[form])
        xs, res, gamma = operands(M, H, w, 9100)
        x_d, res, gamma = xs[r].to(dev), res.to(dev), gamma.to(dev)
        pre, hb, post = guarded_heap(a, M * H)
        first, second = a.create_buffer(M * H, torch.bfloat16), a.create_buffer(M * H, torch.bfloat16)
        xbuf, pad = (first, second) if r < 2 else (second, first)
        pad.dev.fill_(SENTINEL)
        xbuf.dev.copy_(x_d.view(-1))
        torch.cuda.current_stream().synchronize()
        ready.wait()  # every rank's sentinels are in place before any call could write
        st_bad = status_of(a)
        all_reduce_rmsnorm(a, xbuf.dev.view(M, H), gamma, res, EPS, residual_out=hb.dev.view(M, H),
                           status=st_bad)
        torch.cuda.current_stream().synchronize()
        intact = (bool((pre.dev == SENTINEL).all()) and bool((post.dev == SENTINEL).all()) and
                  bool((pad.dev == SENTINEL).all()))
        x = a.create_buffer(M * H, torch.bfloat16).dev.view(M, H)
        x.copy_(x_d)
        st = status_of(a)
        out, h = all_reduce_rmsnorm(a, x, gamma, res, EPS, status=st)
        torch.cuda.current_stream().synchronize()
        return int(st_bad.item()), intact, int(st.item()), h.cpu(), out.cpu()

    ready = threading.Barrier(world)
    res = A.run_cuda_ranks(devices(world), fn, CFG, heap_mb=64, max_ctas=4)
    xs, rz, gamma = operands(M, H, world, 9100)
    want_h = reference_h(xs, rz)
    for r, (bad, intact, status, h, out) in enumerate(res):
        assert bad != -1 and bad & DMA_MISMATCH_ERROR, (r, hex(bad))
        assert intact, f"rank {r}: a guard or the pad buffer was written"
        assert status == 0, (r, hex(status))
        assert torch.equal(h, want_h), f"rank {r}: the call after the mismatch is not exact"
        msg = faithful_failure(f"rank {r} after the mismatch", out, want_h, gamma)
        assert msg is None, msg


def test_all_reduce_rmsnorm_rejects_bad_arguments():
    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        M, H = 4, 64
        xb = a.create_buffer(2 * M * H, torch.bfloat16)
        x = xb.dev[:M * H].view(M, H)
        hb = a.create_buffer(2 * M * H, torch.bfloat16)
        h = hb.dev[:M * H].view(M, H)
        gamma = torch.ones(H, dtype=torch.bfloat16, device=dev)
        res = torch.zeros(M, H, dtype=torch.bfloat16, device=dev)
        out = torch.empty(M, H, dtype=torch.bfloat16, device=dev)
        st = status_of(a)
        plain = torch.zeros(M, H, dtype=torch.bfloat16, device=dev)
        wide = a.create_buffer(2 * 16392, torch.bfloat16).dev.view(2, 16392)
        bad = {
            "x outside the heap": lambda: all_reduce_rmsnorm(a, plain, gamma, status=st),
            "fp32 x": lambda: all_reduce_rmsnorm(a, xb.dev.view(torch.float32)[:M * H // 2].view(M, H // 2),
                                                 gamma[:H // 2], status=st),
            "1-D x": lambda: all_reduce_rmsnorm(a, x.view(-1), gamma, status=st),
            "non-contiguous x": lambda: all_reduce_rmsnorm(a, xb.dev.view(2 * M, H)[::2], gamma, status=st),
            "H % 8": lambda: all_reduce_rmsnorm(a, xb.dev[:M * 60].view(M, 60), gamma[:60], status=st),
            "H above 16384": lambda: all_reduce_rmsnorm(a, wide, torch.ones(16392, dtype=torch.bfloat16, device=dev),
                                                        status=st),
            "no rows": lambda: all_reduce_rmsnorm(a, xb.dev[:0].view(0, H), gamma, status=st),
            "misaligned x": lambda: all_reduce_rmsnorm(a, xb.dev[4:4 + M * H].view(M, H), gamma, status=st),
            "fp32 weight": lambda: all_reduce_rmsnorm(a, x, gamma.float(), status=st),
            "weight of the wrong length": lambda: all_reduce_rmsnorm(a, x, gamma[:32], status=st),
            "weight on the CPU": lambda: all_reduce_rmsnorm(a, x, gamma.cpu(), status=st),
            "residual of the wrong shape": lambda: all_reduce_rmsnorm(a, x, gamma, res[:2], status=st),
            "fp32 residual": lambda: all_reduce_rmsnorm(a, x, gamma, res.float(), status=st),
            "residual_out outside the heap": lambda: all_reduce_rmsnorm(a, x, gamma, residual_out=plain, status=st),
            "residual_out overlaps x": lambda: all_reduce_rmsnorm(a, x, gamma, residual_out=xb.dev[H:H + M * H].view(M, H),
                                                                  status=st),
            "residual_out partly overlaps residual": lambda: all_reduce_rmsnorm(
                a, x, gamma, hb.dev[H:H + M * H].view(M, H), residual_out=h, status=st),
            "residual_out of the wrong shape": lambda: all_reduce_rmsnorm(a, x, gamma, residual_out=hb.dev[:2 * H]
                                                                          .view(2, H), status=st),
            "out overlaps residual": lambda: all_reduce_rmsnorm(a, x, gamma, res, out=res, status=st),
            "out overlaps residual_out": lambda: all_reduce_rmsnorm(a, x, gamma, out=h, residual_out=h, status=st),
            "out overlaps x": lambda: all_reduce_rmsnorm(a, x, gamma, out=x, status=st),
            "fp32 out": lambda: all_reduce_rmsnorm(a, x, gamma, out=out.float(), status=st),
            "negative eps": lambda: all_reduce_rmsnorm(a, x, gamma, eps=-1e-6, status=st),
            "infinite eps": lambda: all_reduce_rmsnorm(a, x, gamma, eps=float("inf"), status=st),
            "int64 status": lambda: all_reduce_rmsnorm(a, x, gamma, status=torch.zeros(1, dtype=torch.int64, device=dev)),
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


# ------------------------------------------------------------------------------------------------ layer
@pytest.fixture
def fused_calls(monkeypatch):
    """Counts the fused all_reduce_rmsnorm calls across the rank threads."""
    calls, lock = [], threading.Lock()
    real = ops.all_reduce_rmsnorm

    def counting(*args, **kw):
        with lock:
            calls.append("ar_rmsnorm")
        return real(*args, **kw)

    monkeypatch.setattr(ops, "all_reduce_rmsnorm", counting)
    return calls


def rand(seed, *shape, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


def rel_err(got, ref):
    return float((got.double() - ref.double()).abs().max() / ref.double().abs().max())


def load_kernels(m, hidden, dev):
    """Runs the layer's local torch math once, so every kernel it needs is loaded before any fused call.  With ranks
    sharing one GPU in one process, loading a module can wait for the kernels running in the context, among them a
    peer's fused kernel that waits for this rank."""
    from accl_b200.parallel import _rms_norm_backward
    h = torch.randn(m, hidden, device=dev).bfloat16().requires_grad_()
    wt = torch.ones(hidden, dtype=torch.bfloat16, device=dev, requires_grad=True)
    for _ in range(2):  # the second pass accumulates into .grad
        y = torch.nn.functional.rms_norm(h.float(), (hidden,), wt.float(), EPS).bfloat16()
        (y.float() * h.float()).sum().backward()
        dh, dw = _rms_norm_backward(h.detach(), wt.detach(), EPS, y.detach(), h.detach())
        (dh.to(torch.bfloat16) + h.detach().clone()).sum()
        dw.to(torch.bfloat16)
    torch.zeros(1, dtype=torch.int32, device=dev).bitwise_or_(torch.zeros(1, dtype=torch.int32, device=dev))
    torch.cuda.current_stream().synchronize()


def run_layer(world, m, hidden, micro_batches, seed, partial_in_heap=False):
    """Per rank: AllReduceRMSNorm on partials (bf16, requires grad) and a shared residual; every forward, then the
    backwards in reverse order, with a loss on both y and h.  Returns per rank (partials, [(y, h)], dpartials,
    dresiduals, dweight) on the CPU in fp32."""

    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        g = TensorGroup(a)
        norm = AllReduceRMSNorm(g, hidden)
        with torch.no_grad():
            norm.weight.copy_(1 + 0.25 * rand(seed + 1, hidden))
        load_kernels(m, hidden, dev)
        staged = [tuple(t.bfloat16().to(dev) for t in (rand(seed + 10 * i + r, m, hidden), rand(seed + 100 + i, m, hidden),
                                                      rand(seed + 200 + i, m, hidden),
                                                      rand(seed + 300 + i, m, hidden, scale=0.5)))
                  for i in range(micro_batches)]
        torch.cuda.current_stream().synchronize()
        ready.wait()
        xs, rs, outs = [], [], []
        for i in range(micro_batches):
            x = staged[i][0].clone()
            if partial_in_heap:
                xb = g.empty(m, hidden, dtype=torch.bfloat16)
                xb.copy_(x)
                x = xb
            x.requires_grad_()
            res = staged[i][1].clone().requires_grad_()
            xs.append(x)
            rs.append(res)
            outs.append(norm(x, res))
        for i, (y, h) in reversed(list(enumerate(outs))):
            torch.autograd.backward([y, h], [staged[i][2], staged[i][3]])
        torch.cuda.current_stream().synchronize()
        g.check(block=True)  # raises on a non-zero status of any fused call
        cpu = lambda t: t.detach().float().cpu()  # noqa: E731
        return ([cpu(x) for x in xs], [(cpu(y), cpu(h)) for y, h in outs], [cpu(x.grad) for x in xs],
                [cpu(res.grad) for res in rs], cpu(norm.weight.grad))

    ready = threading.Barrier(world)
    return A.run_cuda_ranks(devices(world), fn, CFG, heap_mb=64, max_ctas=4)


@pytest.mark.parametrize("world,micro_batches,in_heap", [(1, 1, False), (2, 1, False), (2, 2, False), (2, 1, True)],
                         ids=["world1", "world2", "world2-2mb", "world2-partial-in-heap"])
def test_all_reduce_rmsnorm_layer_runs_fused_and_matches_fp32_autograd(world, micro_batches, in_heap, fused_calls):
    m, hidden, seed = 24, 1024, 4000
    res = run_layer(world, m, hidden, micro_batches, seed, in_heap)
    gamma = (1 + 0.25 * rand(seed + 1, hidden)).bfloat16().float().requires_grad_()
    for i in range(micro_batches):
        parts = [per[0][i].clone().requires_grad_() for per in res]
        resid = rand(seed + 100 + i, m, hidden).bfloat16().float().requires_grad_()
        h = sum(parts) + resid
        y = torch.nn.functional.rms_norm(h, (hidden,), gamma, EPS)
        gy = rand(seed + 200 + i, m, hidden).bfloat16().float()
        gh = rand(seed + 300 + i, m, hidden, scale=0.5).bfloat16().float()
        torch.autograd.backward([y, h], [gy, gh])
        for r, (_, outs, dxs, drs, _) in enumerate(res):
            assert torch.equal(outs[i][0], res[0][1][i][0]) and torch.equal(outs[i][1], res[0][1][i][1]), \
                f"rank {r}'s outputs differ from rank 0's"
            assert rel_err(outs[i][0], y.detach()) < 1e-2, (r, i)
            assert rel_err(outs[i][1], h.detach()) < 1e-2, (r, i)
            assert rel_err(dxs[i], parts[r].grad) < 2e-2, (r, i)
            assert rel_err(drs[i], resid.grad) < 2e-2, (r, i)
    for r, per in enumerate(res):
        assert rel_err(per[4], gamma.grad) < 2e-2, r
    assert fused_calls == ["ar_rmsnorm"] * world * micro_batches, fused_calls


def test_all_reduce_rmsnorm_layer_offset_mismatch_is_reported_at_check():
    """The layer's residual-stream heap buffer sits at different offsets on the two ranks (allocated around a pad in
    opposite orders): the fused call reports DMA_MISMATCH_ERROR, and TensorGroup.check(block=True) raises."""
    m, hidden = 16, 512

    def fn(a, r, w):
        dev = torch.device("cuda", a.cuda_device)
        g = TensorGroup(a)
        norm = AllReduceRMSNorm(g, hidden)
        load_kernels(m, hidden, dev)
        first, second = a.create_buffer(m * hidden, torch.bfloat16), a.create_buffer(m * hidden, torch.bfloat16)
        norm._h, pad = (first, second) if r == 0 else (second, first)
        x = rand(5000 + r, m, hidden).bfloat16().to(dev).requires_grad_()
        torch.cuda.current_stream().synchronize()
        ready.wait()
        y, h = norm(x)
        y.sum().backward()
        torch.cuda.current_stream().synchronize()
        try:
            g.check(block=True)
        except RuntimeError as e:
            return str(e), pad is not None
        return None, True

    ready = threading.Barrier(2)
    for r, (err, _) in enumerate(A.run_cuda_ranks(devices(2), fn, CFG, heap_mb=64, max_ctas=4)):
        assert err is not None and "DMA_MISMATCH_ERROR" in err, (r, err)
