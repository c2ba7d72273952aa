"""AllReduceRMSNorm on the CPU emulator, at world 3 in fp32: the all_reduce + add + torch rms_norm path every backend
takes when the fused all-reduce -> RMSNorm kernel does not apply, and the layer's local backward, checked against
single-process autograd on the unsharded computation.  Also the choice of the fused kernel."""
import pytest
import torch

import accl_b200 as A
from accl_b200.parallel import AllReduceRMSNorm, ReplicatedColumnParallelLinear, TensorGroup, ar_rmsnorm_fused

CFG = dict(n_egr_rx_bufs=16, egr_rx_buf_size=1024, max_egr_size=1024, max_rndzv_size=1 << 20)
W = 3
M, H, F = 5, 16, 18  # rows (replicated), hidden width, FFN width over all ranks
EPS = 1e-5


def rand(seed, *shape):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def close(a, b):
    return torch.allclose(a, b, rtol=1e-4, atol=1e-5)


def reference(partials, residual, weight, gy, gh):
    """Unsharded autograd: y = rms_norm(sum(partials) + residual) * weight, h = sum(partials) + residual."""
    parts = [p.clone().requires_grad_() for p in partials]
    res = None if residual is None else residual.clone().requires_grad_()
    wt = weight.clone().requires_grad_()
    h = sum(parts)
    if res is not None:
        h = h + res
    y = torch.nn.functional.rms_norm(h, (h.shape[-1],), wt, EPS)
    ((y * gy).sum() + (h * gh).sum()).backward()
    return y.detach(), h.detach(), [p.grad for p in parts], None if res is None else res.grad, wt.grad


def run_layer(with_residual, micro_batches):
    """Every micro-batch's forward before any backward, backwards in reverse order; the loss reads both y and h."""
    gys = [rand(10 + i, M, H) for i in range(micro_batches)]
    ghs = [rand(20 + i, M, H) * 0.5 for i in range(micro_batches)]
    residuals = [rand(30 + i, M, H) if with_residual else None for i in range(micro_batches)]
    gamma = 1 + 0.1 * rand(40, H)

    def fn(a, r, w):
        norm = AllReduceRMSNorm(TensorGroup(a), H, eps=EPS, dtype=torch.float32)
        with torch.no_grad():
            norm.weight.copy_(gamma)
        xs = [rand(100 + 10 * i + r, M, H).requires_grad_() for i in range(micro_batches)]
        rs = [None if res is None else res.clone().requires_grad_() for res in residuals]
        outs = [norm(x, res) for x, res in zip(xs, rs)]
        for y, h in outs:
            assert y.grad_fn is not None and h.grad_fn is not None and y.shape == h.shape == (M, H)
        for (y, h), gy, gh in reversed(list(zip(outs, gys, ghs))):
            ((y * gy).sum() + (h * gh).sum()).backward()
        return ([x.detach() for x in xs], [(y.detach(), h.detach()) for y, h in outs], [x.grad for x in xs],
                [None if res is None else res.grad for res in rs], norm.weight.grad)

    res = A.run_ranks(W, fn, CFG)
    dw_total = 0
    for i in range(micro_batches):
        y, h, dparts, dres, dw = reference([per[0][i] for per in res], residuals[i], gamma, gys[i], ghs[i])
        dw_total = dw_total + dw
        for r, (_, outs, dxs, drs, _) in enumerate(res):
            assert close(outs[i][0], y), (r, i)
            assert close(outs[i][1], h), (r, i)
            assert close(dxs[i], dparts[r]), (r, i)  # dpartial = dh on every rank
            if with_residual:
                assert close(drs[i], dres), (r, i)
            else:
                assert drs[i] is None
    for r, per in enumerate(res):
        assert close(per[4], dw_total), r


def test_all_reduce_rmsnorm_layer_matches_unsharded_autograd():
    run_layer(True, 1)


def test_all_reduce_rmsnorm_layer_without_residual():
    run_layer(False, 1)


def test_all_reduce_rmsnorm_layer_two_forwards_before_two_backwards():
    run_layer(True, 2)


def test_column_gelu_matmul_all_reduce_rmsnorm_block_matches_unsharded_block():
    """ReplicatedColumnParallelLinear(H -> F / P) -> GELU -> local matmul with W2_r [H, F / P] -> AllReduceRMSNorm with
    the block input as the residual, against the same block unsharded."""
    x0, gy, gh = rand(1, M, H), rand(2, M, H), rand(3, M, H)
    gamma = 1 + 0.1 * rand(4, H)

    def fn(a, r, w):
        g = TensorGroup(a)
        up = ReplicatedColumnParallelLinear(g, H, F // w, dtype=torch.float32)
        w2 = torch.nn.Parameter(rand(60 + r, H, F // w) * 0.2)
        norm = AllReduceRMSNorm(g, H, eps=EPS, dtype=torch.float32)
        with torch.no_grad():
            norm.weight.copy_(gamma)
        x = x0.clone().requires_grad_()
        y, h = norm(torch.nn.functional.linear(torch.nn.functional.gelu(up(x)), w2), x)
        ((y * gy).sum() + (h * gh).sum()).backward()
        return (up.weight.detach().clone(), w2.detach().clone(), y.detach(), h.detach(), x.grad, up.weight.grad, w2.grad,
                norm.weight.grad)

    res = A.run_ranks(W, fn, CFG)
    x = x0.clone().requires_grad_()
    w1 = torch.cat([per[0] for per in res]).requires_grad_()
    w2 = torch.cat([per[1] for per in res], dim=1).requires_grad_()
    wt = gamma.clone().requires_grad_()
    h = torch.nn.functional.gelu(x @ w1.t()) @ w2.t() + x
    y = torch.nn.functional.rms_norm(h, (H,), wt, EPS)
    ((y * gy).sum() + (h * gh).sum()).backward()
    n = F // W
    for r, (_, _, yr, hr, dx, dw1, dw2, dg) in enumerate(res):
        assert close(yr, y.detach()) and close(hr, h.detach()), r
        assert close(dx, x.grad), r
        assert close(dw1, w1.grad[r * n:(r + 1) * n]), r
        assert close(dw2, w2.grad[:, r * n:(r + 1) * n]), r
        assert close(dg, wt.grad), r


def test_all_reduce_rmsnorm_layer_under_no_grad_and_inference_mode_builds_no_graph():
    def fn(a, r, w):
        norm = AllReduceRMSNorm(TensorGroup(a), H, eps=EPS, dtype=torch.float32)
        x, res = rand(70 + r, M, H), rand(80, M, H)
        y, h = norm(x, res)
        with torch.no_grad():
            y_ng, h_ng = norm(x, res)
        with torch.inference_mode():
            y_inf, h_inf = norm(x, res)
        return (y.grad_fn is not None, y_ng.grad_fn, h_ng.grad_fn, y_inf.grad_fn,
                torch.equal(y.detach(), y_ng) and torch.equal(h.detach(), h_ng),
                torch.equal(y_ng, y_inf) and torch.equal(h_ng, h_inf))

    for has_fn, y_ng_fn, h_ng_fn, inf_fn, same_ng, same_inf in A.run_ranks(W, fn, CFG):
        assert has_fn and y_ng_fn is None and h_ng_fn is None and inf_fn is None and same_ng and same_inf


def test_all_reduce_rmsnorm_layer_weight_starts_at_ones():
    def fn(a, r, w):
        norm = AllReduceRMSNorm(TensorGroup(a), H, dtype=torch.float32)
        return norm.weight.detach().clone(), isinstance(norm.weight, torch.nn.Parameter), norm.eps

    for wt, is_param, eps in A.run_ranks(W, fn, CFG):
        assert is_param and torch.equal(wt, torch.ones(H)) and eps == 1e-6


def test_all_reduce_rmsnorm_layer_chooses_the_fused_kernel():
    bf16, f32 = torch.bfloat16, torch.float32
    assert ar_rmsnorm_fused(True, 0, bf16, 1, 4096)       # decode-sized m
    assert ar_rmsnorm_fused(True, 0, bf16, 8192, 8192)
    assert ar_rmsnorm_fused(True, 0, bf16, 7, 8)          # the narrowest row
    assert ar_rmsnorm_fused(True, 0, bf16, 3, 16384)      # the widest row
    assert not ar_rmsnorm_fused(True, 0, bf16, 3, 16384 + 8)
    assert not ar_rmsnorm_fused(True, 0, bf16, 3, 4100)   # hidden % 8
    assert not ar_rmsnorm_fused(True, 0, bf16, 3, 4)
    assert not ar_rmsnorm_fused(True, 0, bf16, 0, 4096)
    assert not ar_rmsnorm_fused(True, 1, bf16, 64, 4096)  # sub-communicator
    assert not ar_rmsnorm_fused(False, 0, bf16, 64, 4096)  # emulator
    assert not ar_rmsnorm_fused(True, 0, f32, 64, 4096)
    assert not ar_rmsnorm_fused(True, 0, None, 64, 4096)  # partial, weight or residual of different dtypes


def test_rmsnorm_width_limit_matches_the_extension():
    from accl_b200 import _C
    from accl_b200.ops.plugins import AR_RMSNORM_MAX_H
    if not getattr(_C, "with_cuda", False):
        pytest.skip("the extension was built without the CUDA backend")
    assert _C.ar_rmsnorm_max_h == AR_RMSNORM_MAX_H
