"""SeqParallelColumnLinear on the CPU emulator: the all-gather + matmul path every backend without the fused kernel takes."""
import torch

import accl_b200 as A
from accl_b200.parallel import SeqParallelColumnLinear, TensorGroup

CFG = dict(n_egr_rx_bufs=16, egr_rx_buf_size=1024, max_egr_size=1024, max_rndzv_size=1 << 20)
W = 3


def test_seq_parallel_column_linear_gathers_the_sequence():
    m, k, n = 5, 24, 8

    def fn(a, r, w):
        lin = SeqParallelColumnLinear(TensorGroup(a), k, n, dtype=torch.float32)
        x = torch.randn(m, k, generator=torch.Generator().manual_seed(10 + r))
        y = lin(x)
        assert y.shape == (m * w, n)
        return x, lin.weight.detach().clone(), y

    res = A.run_ranks(W, fn, CFG)
    full = torch.cat([x for x, _, _ in res])
    for r, (_, wt, y) in enumerate(res):
        assert torch.allclose(y, full @ wt.t(), rtol=1e-5, atol=1e-5), r
