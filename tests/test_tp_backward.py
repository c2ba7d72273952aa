"""Backward passes of the sequence-parallel linears on the CPU emulator, at world 3 in fp32: the all-gather / matmul /
reduce-scatter path every backend takes when the fused kernels do not apply, checked against single-process autograd
on the unsharded layer and the full sequence.  Also the per-pass choice between the fused kernels and that path."""
import torch

import accl_b200 as A
from accl_b200.parallel import (RowParallelLinear, SeqParallelColumnLinear, TensorGroup, column_backward_fused,
                                column_forward_fused, row_backward_fused, row_forward_fused)

CFG = dict(n_egr_rx_bufs=16, egr_rx_buf_size=1024, max_egr_size=1024, max_rndzv_size=1 << 20)
W = 3
S, H, F = 4, 12, 18  # rows of sequence per rank, hidden width, FFN width over all ranks


def rand(seed, *shape):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def close(a, b):
    return torch.allclose(a, b, rtol=1e-4, atol=1e-5)


def test_column_linear_gradients_match_unsharded_autograd():
    gy = rand(1, S * W, F)  # upstream gradient of the full output

    def fn(a, r, w):
        lin = SeqParallelColumnLinear(TensorGroup(a), H, F // w, dtype=torch.float32)
        x = rand(10 + r, S, H).requires_grad_()
        y = lin(x)
        assert y.grad_fn is not None and y.shape == (S * w, F // w)
        (y * gy[:, r * (F // w):(r + 1) * (F // w)]).sum().backward()
        return x.detach(), lin.weight.detach().clone(), y.detach(), x.grad, lin.weight.grad

    res = A.run_ranks(W, fn, CFG)
    x = torch.cat([x for x, *_ in res]).requires_grad_()
    wt = torch.cat([wt for _, wt, *_ in res]).requires_grad_()
    y = x @ wt.t()
    (y * gy).sum().backward()
    n = F // W
    for r, (_, _, yr, dx, dw) in enumerate(res):
        assert close(yr, y.detach()[:, r * n:(r + 1) * n]), r
        assert close(dx, x.grad[r * S:(r + 1) * S]), r
        assert close(dw, wt.grad[r * n:(r + 1) * n]), r


def test_row_linear_gradients_match_unsharded_autograd():
    M, N = S * W, H
    gy = rand(2, M, N)

    def fn(a, r, w):
        lin = RowParallelLinear(TensorGroup(a), F // w, N, dtype=torch.float32)
        x = rand(20 + r, M, F // w).requires_grad_()
        y = lin(x)
        assert y.grad_fn is not None and y.shape == (M // w, N)
        (y * gy[r * (M // w):(r + 1) * (M // w)]).sum().backward()
        return x.detach(), lin.weight.detach().clone(), y.detach(), x.grad, lin.weight.grad

    res = A.run_ranks(W, fn, CFG)
    x = torch.cat([x for x, *_ in res], dim=1).requires_grad_()
    wt = torch.cat([wt for _, wt, *_ in res], dim=1).requires_grad_()
    y = x @ wt.t()
    (y * gy).sum().backward()
    k, rows = F // W, M // W
    for r, (_, _, yr, dx, dw) in enumerate(res):
        assert close(yr, y.detach()[r * rows:(r + 1) * rows]), r
        assert close(dx, x.grad[:, r * k:(r + 1) * k]), r
        assert close(dw, wt.grad[:, r * k:(r + 1) * k]), r


def mlp_reference(res, gys):
    """Single-process autograd of gelu(X W1^T) W2^T on the full sequence, one backward per micro-batch."""
    w1 = torch.cat([w1 for _, w1, _, _ in res]).requires_grad_()          # [F, H]: the ranks' FFN features in order
    w2 = torch.cat([w2 for _, _, w2, _ in res], dim=1).requires_grad_()   # [H, F]
    xs, ys = [], []
    for i, gy in enumerate(gys):
        x = torch.cat([per[0][i] for per in res]).requires_grad_()
        y = torch.nn.functional.gelu(x @ w1.t()) @ w2.t()
        (y * gy).sum().backward()
        xs.append(x)
        ys.append(y.detach())
    return xs, ys, w1.grad, w2.grad


def run_mlp(micro_batches):
    """Column -> GELU -> row at world 3; every micro-batch runs forward before any backward, backwards in reverse
    order (as with activation recomputation or pipelined micro-batches)."""
    gys = [rand(30 + i, S * W, H) for i in range(micro_batches)]

    def fn(a, r, w):
        g = TensorGroup(a)
        up = SeqParallelColumnLinear(g, H, F // w, dtype=torch.float32)
        down = RowParallelLinear(g, F // w, H, dtype=torch.float32)
        xs = [rand(40 + 10 * i + r, S, H).requires_grad_() for i in range(micro_batches)]
        ys = [down(torch.nn.functional.gelu(up(x))) for x in xs]
        for y, gy in reversed(list(zip(ys, gys))):
            (y * gy[r * S:(r + 1) * S]).sum().backward()
        return ([x.detach() for x in xs], up.weight.detach().clone(), down.weight.detach().clone(),
                ([y.detach() for y in ys], [x.grad for x in xs], up.weight.grad, down.weight.grad))

    res = A.run_ranks(W, fn, CFG)
    xs, ys, dw1, dw2 = mlp_reference(res, gys)
    n = F // W
    for r, (_, _, _, (yr, dxr, dw1r, dw2r)) in enumerate(res):
        for i in range(micro_batches):
            assert close(yr[i], ys[i][r * S:(r + 1) * S]), (r, i)
            assert close(dxr[i], xs[i].grad[r * S:(r + 1) * S]), (r, i)
        assert close(dw1r, dw1[r * n:(r + 1) * n]), r
        assert close(dw2r, dw2[:, r * n:(r + 1) * n]), r


def test_mlp_gradients_match_unsharded_autograd():
    run_mlp(1)


def test_two_forwards_before_two_backwards_accumulate_the_right_gradients():
    run_mlp(2)


def test_no_grad_and_inference_mode_keep_the_graph_free_path():
    def fn(a, r, w):
        g = TensorGroup(a)
        up = SeqParallelColumnLinear(g, H, F // w, dtype=torch.float32)
        down = RowParallelLinear(g, F // w, H, dtype=torch.float32)
        x = rand(50 + r, S, H)
        y_grad = down(up(x))
        with torch.no_grad():
            y_ng = down(up(x))
        with torch.inference_mode():
            y_inf = down(up(x))
        return y_grad.grad_fn is not None, y_ng.grad_fn, y_inf.grad_fn, torch.equal(y_grad.detach(), y_ng), \
            torch.equal(y_ng, y_inf)

    for has_fn, ng_fn, inf_fn, same_ng, same_inf in A.run_ranks(W, fn, CFG):
        assert has_fn and ng_fn is None and inf_fn is None and same_ng and same_inf


def test_forward_and_backward_choose_the_fused_kernels_independently():
    bf16, f32 = torch.bfloat16, torch.float32
    # RowParallelLinear [m, K_r] -> [m / P, N]: forward N % 256 and K_r % 64, backward K_r % 256 and N % 64
    assert row_forward_fused(True, bf16, 1024, 2, 512, 64)
    assert not row_backward_fused(True, 0, bf16, 1024, 2, 512, 64)          # K_r = 64: fused forward, fallback backward
    assert row_backward_fused(True, 0, bf16, 1024, 2, 64, 256)
    assert not row_forward_fused(True, bf16, 1024, 2, 64, 256)              # N = 64: fallback forward, fused backward
    assert row_forward_fused(True, bf16, 8192, 8, 8192, 3584)               # FFN 28672 / 8 in, hidden 8192 out
    assert row_backward_fused(True, 0, bf16, 8192, 8, 8192, 3584)
    assert not row_backward_fused(True, 0, bf16, 8192, 8, 8192, 1088)       # K_r = 17 * 64
    assert not row_backward_fused(True, 0, bf16, 1024 + 128, 2, 256, 256)   # m % (128 P)
    assert not row_backward_fused(True, 0, bf16, 128 * 1025, 1, 256, 256)   # the all-gather plugin's 1024 row blocks
    assert not row_backward_fused(True, 1, bf16, 1024, 2, 256, 256)         # sub-communicator
    assert not row_backward_fused(False, 0, bf16, 1024, 2, 256, 256)        # emulator
    assert not row_backward_fused(True, 0, f32, 1024, 2, 256, 256)
    assert not row_backward_fused(True, 0, None, 1024, 2, 256, 256)         # x and weight of different dtypes
    # SeqParallelColumnLinear [m, K] -> [m P, N_r]: forward N_r % 256 and K % 64, backward K % 256 and N_r % 64
    assert column_forward_fused(True, 0, bf16, 512, 2, 64, 256)
    assert not column_backward_fused(True, 0, bf16, 512, 2, 64, 256)       # K = 64: fused forward, fallback backward
    assert column_backward_fused(True, 0, bf16, 512, 2, 256, 64)
    assert not column_forward_fused(True, 0, bf16, 512, 2, 256, 64)
    assert column_backward_fused(True, 0, bf16, 1024, 8, 8192, 3584)       # hidden 8192 in, FFN 28672 / 8 out
    assert column_backward_fused(True, 0, bf16, 1024, 8, 8192, 1088)       # N_r = 17 * 64: only the backward fuses
    assert not column_forward_fused(True, 0, bf16, 1024, 8, 8192, 1088)
    assert not column_backward_fused(True, 0, bf16, 512 + 64, 2, 256, 256)  # m % 128
    assert not column_backward_fused(True, 1, bf16, 512, 2, 256, 256)
    assert not column_backward_fused(False, 0, bf16, 512, 2, 256, 256)
    assert not column_backward_fused(True, 0, f32, 512, 2, 256, 256)
    assert not column_forward_fused(True, 0, bf16, 128 * 513, 2, 64, 256)   # m P / 128 > 1024
