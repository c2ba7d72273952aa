"""Reference implementations of the parallelism strategies the collectives exist for (SURVEY 2.8: the
reference ships only the primitives).  Each is a few lines over `TensorGroup`, runs unchanged on the CPU
emulator and on H100, and is covered by tests/test_parallel.py.

* `ZeroOptimizer`            ZeRO-1 / FSDP-style step: reduce_scatter(grads) -> local shard update -> all_gather(params)
* `ColumnParallelLinear`     Megatron column-parallel linear (local GEMM; optional all_gather of the output)
* `pipeline_send` / `pipeline_recv`   tagged activation hand-off between pipeline stages
* `moe_dispatch` / `moe_combine`      expert-parallel token exchange (all_to_all, equal capacity per expert rank)
* `moe_dispatch_v` / `moe_combine_v`  dropless token exchange (alltoallv: routed row counts stay on the device)
* `ulysses_seq_to_head` / `ulysses_head_to_seq`   DeepSpeed-Ulysses re-sharding sequence <-> heads (all_to_all)
"""
import torch

from . import GradBucket, TensorGroup


class ZeroOptimizer:
    """SGD with the optimizer state and the update sharded over the group (ZeRO stage 1).

    params: list of tensors (updated in place).  Gradients are written into `grad_views` (views of one flat
    bucket living in engine memory), then `step()` = reduce_scatter -> update my shard -> all_gather."""

    def __init__(self, group: TensorGroup, params, lr=0.1, momentum=0.0):
        self.group, self.params, self.lr, self.momentum = group, list(params), lr, momentum
        n = sum(p.numel() for p in self.params)
        self.bucket = GradBucket(group, n, dtype=torch.float32)
        self.grad_views = self.bucket.views([tuple(p.shape) for p in self.params])
        self.shard_len = self.bucket.numel // group.world
        self.flat_params = group.empty(self.bucket.numel)
        self.flat_params.zero_()
        off = 0
        for p in self.params:
            self.flat_params[off:off + p.numel()].copy_(p.detach().reshape(-1).float())
            off += p.numel()
        self.velocity = torch.zeros(self.shard_len, dtype=torch.float32, device=self.flat_params.device)
        self._shard_in = group.empty(self.shard_len)

    def step(self):
        g, r = self.group, self.group.rank
        grad_shard = self.bucket.reduce_scatter()                 # sum over ranks of my 1/P of the gradients
        grad_shard = grad_shard / g.world
        mine = self.flat_params[r * self.shard_len:(r + 1) * self.shard_len]
        if self.momentum:
            self.velocity.mul_(self.momentum).add_(grad_shard)
            grad_shard = self.velocity
        self._shard_in.copy_(mine - self.lr * grad_shard)         # update only what I own
        g.all_gather_into_tensor(self.flat_params, self._shard_in)
        off = 0
        for p in self.params:
            p.data.copy_(self.flat_params[off:off + p.numel()].view_as(p))
            off += p.numel()


class ColumnParallelLinear(torch.nn.Module):
    """y_r = x @ W_r^T with the output features split over ranks; `gather_output` all-gathers them."""

    def __init__(self, group: TensorGroup, in_features, out_features_per_rank, gather_output=False, dtype=torch.float32,
                 device="cpu"):
        super().__init__()
        self.group, self.gather_output = group, gather_output
        self.weight = torch.nn.Parameter(torch.empty(out_features_per_rank, in_features, dtype=dtype, device=device))
        torch.nn.init.normal_(self.weight, std=0.02)

    @torch.no_grad()
    def forward(self, x):
        y = x @ self.weight.t()
        if not self.gather_output:
            return y
        P = self.group.world
        out = torch.empty(P, *y.shape, dtype=y.dtype, device=y.device)
        self.group.all_gather_into_tensor(out, y.contiguous())
        return out.movedim(0, -2).reshape(*y.shape[:-1], P * y.shape[-1])


def pipeline_send(group: TensorGroup, act: torch.Tensor, dst_stage: int, microbatch: int):
    """Hand an activation to the next stage; the tag carries the micro-batch index (1F1B schedules keep
    several in flight).  Returns the request (asynchronous: wait before reusing `act`)."""
    return group.send(act, dst_stage, tag=microbatch & 0xFFFF)


def pipeline_recv(group: TensorGroup, act: torch.Tensor, src_stage: int, microbatch: int):
    return group.recv(act, src_stage, tag=microbatch & 0xFFFF)


def moe_dispatch(group: TensorGroup, tokens_by_dest: torch.Tensor):
    """tokens_by_dest[q] = the (capacity, hidden) block this rank routes to expert rank q.
    Returns recv[q] = the block rank q routed to me."""
    out = torch.empty_like(tokens_by_dest)
    group.all_to_all_single(out.view(-1), tokens_by_dest.contiguous().view(-1))
    return out


def moe_combine(group: TensorGroup, expert_out_by_src: torch.Tensor):
    """Inverse of `moe_dispatch`: send every processed block back to the rank it came from."""
    return moe_dispatch(group, expert_out_by_src)


def moe_dispatch_v(group: TensorGroup, tokens: torch.Tensor, send_counts: torch.Tensor, capacity: int):
    """Dropless dispatch.  tokens: [N, hidden], rows grouped by destination rank in rank order; send_counts: int64
    rows per destination (on the device for the CUDA backend).  The row counts are exchanged first (one int64 per
    peer), then the rows move with alltoallv into a [capacity, hidden] buffer; no step waits for the host.
    Returns (recv_tokens, recv_counts): recv_counts[p] rows from rank p, packed in rank order."""
    hidden = tokens.shape[1]
    send_counts = send_counts.to(torch.int64).contiguous()
    recv_counts = torch.empty_like(send_counts)
    group.all_to_all_single(recv_counts, send_counts)
    recv = torch.empty(capacity, hidden, dtype=tokens.dtype, device=tokens.device)
    group.all_to_all_v(recv.view(-1), tokens.contiguous().view(-1), send_counts * hidden, recv_counts * hidden)
    return recv, recv_counts


def moe_combine_v(group: TensorGroup, expert_out: torch.Tensor, recv_counts: torch.Tensor, send_counts: torch.Tensor,
                  num_tokens: int):
    """Inverse of `moe_dispatch_v`: the rows of `expert_out` ([capacity, hidden], recv_counts[p] rows from rank p)
    go back to the ranks they came from.  Returns [num_tokens, hidden] in the original dispatch order."""
    hidden = expert_out.shape[1]
    out = torch.empty(num_tokens, hidden, dtype=expert_out.dtype, device=expert_out.device)
    group.all_to_all_v(out.view(-1), expert_out.contiguous().view(-1), recv_counts.to(torch.int64) * hidden,
                       send_counts.to(torch.int64) * hidden)
    return out


def ulysses_seq_to_head(group: TensorGroup, x: torch.Tensor):
    """[S/P, H, D] (sequence-sharded, all heads) -> [S, H/P, D] (full sequence, my heads)."""
    P = group.world
    s, h, d = x.shape
    send = x.view(s, P, h // P, d).transpose(0, 1).contiguous()          # [P, S/P, H/P, D]: block q goes to rank q
    recv = torch.empty_like(send)
    group.all_to_all_single(recv.view(-1), send.view(-1))
    return recv.reshape(P * s, h // P, d)                                 # blocks arrive in rank (= sequence) order


def ulysses_head_to_seq(group: TensorGroup, x: torch.Tensor):
    """[S, H/P, D] -> [S/P, H, D]: the inverse re-sharding after attention."""
    P = group.world
    s, hp, d = x.shape
    send = x.view(P, s // P, hp, d).contiguous()                          # block q = sequence chunk q
    recv = torch.empty_like(send)
    group.all_to_all_single(recv.view(-1), send.view(-1))
    return recv.transpose(0, 1).reshape(s // P, P * hp, d)                # [S/P, P, H/P, D] -> heads in rank order
