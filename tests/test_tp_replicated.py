"""Tensor-parallel linears with replicated activations on the CPU emulator, at world 3 in fp32: the matmul + all-reduce
path every backend takes when the fused GEMM -> all-reduce kernel does not apply, checked against single-process
autograd on the unsharded layers.  Also the per-pass choice of the fused kernel, and a model of the kernel's tile
ownership and visit order (plugin_gemm_rs.cu, ar_tile_of_slot)."""
import pytest
import torch

import accl_b200 as A
from accl_b200.ops.plugins import GEMM_AR_MAX_TILES
from accl_b200.parallel import (ReplicatedColumnParallelLinear, ReplicatedRowParallelLinear, TensorGroup,
                                column_ar_backward_fused, row_ar_forward_fused)

CFG = dict(n_egr_rx_bufs=16, egr_rx_buf_size=1024, max_egr_size=1024, max_rndzv_size=1 << 20)
W = 3
M, H, F = 5, 12, 18  # rows (replicated), hidden width, FFN width over all ranks


def rand(seed, *shape):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def close(a, b):
    return torch.allclose(a, b, rtol=1e-4, atol=1e-5)


def test_replicated_column_linear_gradients_match_unsharded_autograd():
    x0, gy = rand(1, M, H), rand(2, M, F)

    def fn(a, r, w):
        lin = ReplicatedColumnParallelLinear(TensorGroup(a), H, F // w, dtype=torch.float32)
        x = x0.clone().requires_grad_()
        y = lin(x)
        assert y.grad_fn is not None and y.shape == (M, F // w)
        (y * gy[:, r * (F // w):(r + 1) * (F // w)]).sum().backward()
        return lin.weight.detach().clone(), y.detach(), x.grad, lin.weight.grad

    res = A.run_ranks(W, fn, CFG)
    x = x0.clone().requires_grad_()
    wt = torch.cat([wt for wt, *_ in res]).requires_grad_()
    y = x @ wt.t()
    (y * gy).sum().backward()
    n = F // W
    for r, (_, yr, dx, dw) in enumerate(res):
        assert close(yr, y.detach()[:, r * n:(r + 1) * n]), r
        assert close(dx, x.grad), r  # the all-reduced input gradient, the same on every rank
        assert close(dw, wt.grad[r * n:(r + 1) * n]), r


def test_replicated_row_linear_gradients_match_unsharded_autograd():
    gy = rand(3, M, H)

    def fn(a, r, w):
        lin = ReplicatedRowParallelLinear(TensorGroup(a), F // w, H, dtype=torch.float32)
        x = rand(20 + r, M, F // w).requires_grad_()
        y = lin(x)
        assert y.grad_fn is not None and y.shape == (M, H)
        (y * gy).sum().backward()
        return x.detach(), lin.weight.detach().clone(), y.detach(), x.grad, lin.weight.grad

    res = A.run_ranks(W, fn, CFG)
    x = torch.cat([x for x, *_ in res], dim=1).requires_grad_()
    wt = torch.cat([wt for _, wt, *_ in res], dim=1).requires_grad_()
    y = x @ wt.t()
    (y * gy).sum().backward()
    k = F // W
    for r, (_, _, yr, dx, dw) in enumerate(res):
        assert close(yr, y.detach()), r
        assert close(dx, x.grad[:, r * k:(r + 1) * k]), r
        assert close(dw, wt.grad[:, r * k:(r + 1) * k]), r


def run_mlp(micro_batches):
    """Column -> GELU -> row at world 3 on a replicated input; every micro-batch runs forward before any backward,
    backwards in reverse order."""
    xs0 = [rand(40 + i, M, H) for i in range(micro_batches)]
    gys = [rand(30 + i, M, H) for i in range(micro_batches)]

    def fn(a, r, w):
        g = TensorGroup(a)
        up = ReplicatedColumnParallelLinear(g, H, F // w, dtype=torch.float32)
        down = ReplicatedRowParallelLinear(g, F // w, H, dtype=torch.float32)
        xs = [x.clone().requires_grad_() for x in xs0]
        ys = [down(torch.nn.functional.gelu(up(x))) for x in xs]
        for y, gy in reversed(list(zip(ys, gys))):
            (y * gy).sum().backward()
        return (up.weight.detach().clone(), down.weight.detach().clone(),
                ([y.detach() for y in ys], [x.grad for x in xs], up.weight.grad, down.weight.grad))

    res = A.run_ranks(W, fn, CFG)
    w1 = torch.cat([w1 for w1, _, _ in res]).requires_grad_()
    w2 = torch.cat([w2 for _, w2, _ in res], dim=1).requires_grad_()
    xs, ys = [], []
    for x0, gy in zip(xs0, gys):
        x = x0.clone().requires_grad_()
        y = torch.nn.functional.gelu(x @ w1.t()) @ w2.t()
        (y * gy).sum().backward()
        xs.append(x)
        ys.append(y.detach())
    n = F // W
    for r, (_, _, (yr, dxr, dw1r, dw2r)) in enumerate(res):
        for i in range(micro_batches):
            assert close(yr[i], ys[i]), (r, i)
            assert close(dxr[i], xs[i].grad), (r, i)
        assert close(dw1r, w1.grad[r * n:(r + 1) * n]), r
        assert close(dw2r, w2.grad[:, r * n:(r + 1) * n]), r


def test_replicated_mlp_gradients_match_unsharded_autograd():
    run_mlp(1)


def test_replicated_mlp_two_forwards_before_two_backwards():
    run_mlp(2)


def test_replicated_layers_under_no_grad_and_inference_mode_build_no_graph():
    def fn(a, r, w):
        g = TensorGroup(a)
        up = ReplicatedColumnParallelLinear(g, H, F // w, dtype=torch.float32)
        down = ReplicatedRowParallelLinear(g, F // w, H, dtype=torch.float32)
        x = rand(50, M, H)
        y_grad = down(up(x))
        with torch.no_grad():
            y_ng = down(up(x))
        with torch.inference_mode():
            y_inf = down(up(x))
        return y_grad.grad_fn is not None, y_ng.grad_fn, y_inf.grad_fn, torch.equal(y_grad.detach(), y_ng), \
            torch.equal(y_ng, y_inf)

    for has_fn, ng_fn, inf_fn, same_ng, same_inf in A.run_ranks(W, fn, CFG):
        assert has_fn and ng_fn is None and inf_fn is None and same_ng and same_inf


def test_replicated_layers_choose_the_fused_kernel():
    bf16, f32 = torch.bfloat16, torch.float32
    # ReplicatedRowParallelLinear [m, K_r] -> [m, N]: forward fused for m % 128, N % 256, K_r % 64
    assert row_ar_forward_fused(True, 0, bf16, 128, 256, 64)
    assert row_ar_forward_fused(True, 0, bf16, 8192 + 128, 8192, 3584)   # m % (128 P) is not needed
    assert not row_ar_forward_fused(True, 0, bf16, 64, 8192, 3584)       # decode-sized m
    assert not row_ar_forward_fused(True, 0, bf16, 192, 8192, 3584)      # m % 128
    assert not row_ar_forward_fused(True, 0, bf16, 1024, 8192 + 64, 3584)
    assert not row_ar_forward_fused(True, 0, bf16, 1024, 8192, 3584 + 32)
    assert not row_ar_forward_fused(True, 1, bf16, 1024, 8192, 3584)     # sub-communicator
    assert not row_ar_forward_fused(False, 0, bf16, 1024, 8192, 3584)    # emulator
    assert not row_ar_forward_fused(True, 0, f32, 1024, 8192, 3584)
    assert not row_ar_forward_fused(True, 0, None, 1024, 8192, 3584)     # x and weight of different dtypes
    assert row_ar_forward_fused(True, 0, bf16, 128 * 512, 256 * 32, 64)  # exactly the tile limit
    assert not row_ar_forward_fused(True, 0, bf16, 128 * 513, 256 * 32, 64)
    # ReplicatedColumnParallelLinear [m, K] -> [m, N_r]: backward dX [m, K] fused for m % 128, K % 256, N_r % 64
    assert column_ar_backward_fused(True, 0, bf16, 128, 256, 64)
    assert column_ar_backward_fused(True, 0, bf16, 1024, 8192, 28672 // 8)
    assert column_ar_backward_fused(True, 0, bf16, 1024, 8192, 17 * 64)
    assert not column_ar_backward_fused(True, 0, bf16, 64, 8192, 3584)
    assert not column_ar_backward_fused(True, 0, bf16, 1024, 8192 + 64, 3584)
    assert not column_ar_backward_fused(True, 0, bf16, 1024, 8192, 3584 + 32)
    assert not column_ar_backward_fused(True, 1, bf16, 1024, 8192, 3584)
    assert not column_ar_backward_fused(False, 0, bf16, 1024, 8192, 3584)
    assert not column_ar_backward_fused(True, 0, f32, 1024, 8192, 3584)


# ------------------------------------------------------------------------------------------------ tile order model
def ar_tile_of_slot(s, P, me):
    """plugin_gemm_rs.cu: the tile rank `me` computes at slot s of the sweep; tile t is owned by rank t % P."""
    return s - s % P + (s % P + me + 1) % P


@pytest.mark.parametrize("P", [1, 2, 3, 4, 5, 8])
def test_all_reduce_tile_ownership_and_visit_order(P):
    for tiles in [1, 2, 3, 7, 8, 9, 16, 17, 64, 100, 2048, 2049]:
        slots = (tiles + P - 1) // P * P
        owners = [t % P for t in range(tiles)]
        # every tile has exactly one owner, and the owners are balanced
        counts = [owners.count(o) for o in range(P)]
        assert max(counts) - min(counts) <= 1, (tiles, P, counts)
        visits = [[ar_tile_of_slot(s, P, me) for s in range(slots)] for me in range(P)]
        for me in range(P):
            # each rank computes every tile exactly once (slots past the last tile are skipped)
            assert sorted(t for t in visits[me] if t < tiles) == list(range(tiles)), (tiles, P, me)
        for s in range(slots):
            # at any slot the ranks add into different owners: no incast
            targets = [visits[me][s] % P for me in range(P) if visits[me][s] < tiles]
            assert len(set(targets)) == len(targets), (tiles, P, s)
        for t in range(tiles):
            # all ranks reach a tile within P slots of one another
            reach = [visits[me].index(t) for me in range(P)]
            assert max(reach) - min(reach) < P, (tiles, P, t)


def test_counter_block_limit_matches_the_extension():
    from accl_b200 import _C
    if not getattr(_C, "with_cuda", False):
        pytest.skip("the extension was built without the CUDA backend")
    assert _C.gemm_ar_max_tiles == GEMM_AR_MAX_TILES
