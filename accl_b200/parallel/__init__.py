"""Parallelism building blocks on top of the collective API.

The reference is a communication library and implements no model-parallel
strategy itself (SURVEY §2.8); it supplies the primitives they are built from.
This module packages those primitives the way training / serving code consumes
them on a H100 node:

* `init_from_env`        one rank per process (torchrun): pick the backend, build the world
* `TensorGroup`          torch-tensor front end: all_reduce / all_gather / reduce_scatter /
                         broadcast / all_to_all (even or uneven) / send / recv on CUDA tensors (zero-copy when the
                         tensor already lives in the symmetric heap, staged otherwise)
* `GradBucket`           DP / ZeRO gradient bucket living in the heap: fill, then one all-reduce
                         (or reduce_scatter + all_gather) per bucket, stream ordered
* `RowParallelLinear`    TP row-parallel linear whose GEMM epilogue IS the reduce-scatter
                         (wgmma plugin), sequence-parallel output; its input gradient runs on the all-gather plugin
* `SeqParallelColumnLinear`  its counterpart: TP column-parallel linear on a sequence-parallel input whose all-gather
                         feeds the GEMM inside one kernel (wgmma plugin); its input gradient runs on the
                         reduce-scatter plugin
* `ReplicatedRowParallelLinear` / `ReplicatedColumnParallelLinear`  the same pair with activations replicated on every
                         rank (plain Megatron TP): the row layer's forward and the column layer's input gradient end
                         in an all-reduce that runs inside the GEMM (accl_b200.ops.gemm_all_reduce)
* `AllReduceRMSNorm`     all-reduce of a row-parallel matmul's partial sums, residual add and RMSNorm in one kernel
                         (accl_b200.ops.all_reduce_rmsnorm)
* `ring_exchange`        neighbour send/recv step for context-parallel / ring-attention schedules
* `process_group`        `torch.distributed` backend "accl" (import accl_b200.parallel.process_group): the standard
                         ProcessGroup interface incl. DistributedDataParallel on top of this library
* `strategies`           ZeRO-1 optimizer step, column-parallel linear, pipeline hand-off, MoE dispatch / combine,
                         Ulysses sequence <-> head re-sharding (accl_b200/parallel/strategies.py)
"""
import os

import torch

from .. import _C
from ..core import Accl, Buffer, SUM, cuda_rank, socket_rank
from ..ops.plugins import AR_RMSNORM_MAX_H, GEMM_AR_MAX_TILES
from ..utils.dtypes import to_accl


def init_from_env(backend=None, **kw):
    """RANK / WORLD_SIZE / LOCAL_RANK / MASTER_ADDR / MASTER_PORT -> an initialised `Accl`.

    backend: "cuda" (default when a GPU and the CUDA backend are available) or "emulator".
    Extra keyword arguments go to `initialize` (eager / rendezvous geometry)."""
    if backend is None:
        backend = "cuda" if (torch.cuda.is_available() and _C.with_cuda and _C.cuda_driver_available()) else "emulator"
    init_keys = ("n_egr_rx_bufs", "egr_rx_buf_size", "max_egr_size", "max_rndzv_size")
    init_kw = {k: kw.pop(k) for k in list(kw) if k in init_keys}
    if backend == "cuda":
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
        if "engine" not in kw and os.environ.get("ACCL_PG_ENGINE") is not None:
            kw["engine"] = os.environ["ACCL_PG_ENGINE"] not in ("", "0")
        if "max_ctas" not in kw and os.environ.get("ACCL_MAX_CTAS"):
            kw["max_ctas"] = int(os.environ["ACCL_MAX_CTAS"])  # channel cap (default 128; the planner sizes every call)
        if "heap_mb" not in kw and os.environ.get("ACCL_HEAP_MB"):
            kw["heap_mb"] = int(os.environ["ACCL_HEAP_MB"])   # symmetric heap per rank (default 1024)
        acc = cuda_rank(**kw)
        init_kw.setdefault("n_egr_rx_bufs", 4)
        init_kw.setdefault("egr_rx_buf_size", 64 << 10)
        init_kw.setdefault("max_egr_size", 64 << 10)
        init_kw.setdefault("max_rndzv_size", 1 << 30)
    else:
        acc = socket_rank(**kw)
    acc.initialize(**init_kw)
    if backend != "cuda" and os.environ.get("ACCL_EMU_ONE_HOP", "0") not in ("", "0"):
        acc.set_one_hop_schedules(True)   # emulator: the H100 backend's schedules instead of the reference's rings / trees
    return acc


class TensorGroup:
    """torch.distributed-flavoured calls on top of one `Accl` (device-resident tensors)."""

    def __init__(self, accl: Accl, comm_id=0, scratch_bytes=64 << 20):
        self.accl = accl
        self.comm_id = comm_id
        self.world = len(accl.get_comm_group(comm_id))
        self.rank = accl.get_comm_rank(comm_id)
        self._scratch = {}
        self._wrapped = {}  # heap-resident torch tensors seen so far -> Buffer views
        self._scratch_bytes = scratch_bytes
        # CUDA: operands are device resident and calls are stream ordered.  Emulator: the tensor side of a
        # buffer is its host mirror, so calls are blocking and sync to / from the engine's memory themselves.
        self._res = bool(accl.is_cuda)
        self._async = bool(accl.is_cuda)
        # engine mode: asynchronous point-to-point calls do not hold the stream (they may stay parked until the peer posts
        # its side), so a staged receive has to be waited for on the host before its staging buffer is read
        self._engine = bool(accl.is_cuda) and "mode=engine" in accl.describe()
        self._pending = []  # asynchronous requests whose return code has not been looked at yet
        self._plugin_status = None  # int32 device word: OR of the status bits of every fused plugin call (CUDA)

    # -- request bookkeeping ---------------------------------------------------
    def _track(self, req):
        """Keep an asynchronous request until it has completed, then check its return code: a device-side timeout,
        tag mismatch or protocol error must not go unnoticed while training continues on garbage."""
        if req is None or not hasattr(req, "test"):
            return req
        self._pending.append(req)
        self.check(block=len(self._pending) > 64)
        return req

    def plugin_status(self):
        """A fresh 1-element int32 status tensor for one fused plugin call (ops.gemm_reduce_scatter /
        ops.all_gather_gemm); pass it to the call, then to `note_plugin_status`."""
        return torch.zeros(1, dtype=torch.int32, device=torch.device("cuda", self.accl.cuda_device))

    def note_plugin_status(self, status):
        """OR a fused call's status word into this group's, stream ordered: nothing waits for the host, so it may run
        inside autograd's backward.  `check(block=True)` and `barrier()` raise when the word is non-zero."""
        if self._plugin_status is None:
            self._plugin_status = torch.zeros_like(status)
        self._plugin_status.bitwise_or_(status)

    def check(self, block=False):
        """Raise if any finished call reported an error; with block=True wait for everything outstanding, including the
        fused plugin calls of this group's layers (their status word is read then, and cleared)."""
        if block and self._plugin_status is not None:
            bits = int(self._plugin_status.item())
            if bits:
                self._plugin_status.zero_()
                raise RuntimeError(f"fused GEMM plugin call failed on rank {self.rank}: {_C.error_to_string(bits)} "
                                   f"(0x{bits:x})")
        keep = []
        for r in self._pending:
            if block:
                r.wait()
            if block or r.test():
                rc = r.retcode()
                if rc:
                    self._pending = [q for q in self._pending if q is not r]
                    raise RuntimeError(f"accl call failed on rank {self.rank}: {_C.error_to_string(rc)} (0x{rc:x})")
            else:
                keep.append(r)
        self._pending = keep

    def _t(self, buf):
        """The torch tensor aliasing a buffer on this backend."""
        return buf.dev if self._res else buf.host

    # -- heap-resident tensors -------------------------------------------
    def empty(self, *shape, dtype=torch.float32):
        """A tensor allocated in the symmetric heap: zero-copy operand of every collective."""
        n = 1
        for s in shape:
            n *= s
        buf = self.accl.create_buffer(n, dtype)
        t = self._t(buf).view(*shape)
        t._accl_buffer = buf
        return t

    def _buffer_of(self, t: torch.Tensor, role):
        buf = getattr(t, "_accl_buffer", None)
        if buf is not None and buf.length == t.numel():
            return buf, False
        if self._res and t.is_contiguous() and self.accl.heap_contains(t):
            # memory from the heap pool (Accl.heap_mem_pool): zero-copy, the view is cached by address
            key = (t.data_ptr(), t.numel(), t.dtype)
            buf = self._wrapped.get(key)
            if buf is None:
                if len(self._wrapped) > 256:
                    self._wrapped.clear()
                buf = self._wrapped[key] = self.accl.wrap_device(t)
            return buf, False
        # stage through ONE cached heap buffer per (role, dtype); it grows to the largest tensor seen (calls carry
        # their own element counts, so a longer buffer is fine).  Reuse is safe: staging copies and collectives are
        # ordered on the caller's stream.
        key = (role, t.dtype)
        cur = self._scratch.get(key)
        if cur is None or cur.length < t.numel():
            self._scratch.pop(key, None)
            cur = None  # the old allocation returns to the heap (same order on every rank) before the new one is made
            self._scratch[key] = self.accl.create_buffer(t.numel(), t.dtype)
        return self._scratch[key], True

    def _chunks(self, t: torch.Tensor):
        """Element-wise collectives on a tensor outside the heap that is larger than the staging budget: contiguous
        views of at most `scratch_bytes` each (None when the tensor can go in one piece)."""
        if getattr(t, "_accl_buffer", None) is not None or t.numel() * t.element_size() <= self._scratch_bytes:
            return None
        if self._res and self.accl.heap_contains(t):
            return None
        step = max(1, self._scratch_bytes // t.element_size())
        flat = t.view(-1) if t.is_contiguous() else None
        if flat is None:
            return None
        return [flat[o:o + step] for o in range(0, t.numel(), step)]

    def _run(self, fn, src: torch.Tensor, dst: torch.Tensor, src_elems, dst_elems):
        sb, s_staged = self._buffer_of(src, "s")
        db, d_staged = (sb, s_staged) if dst is src else self._buffer_of(dst, "d")
        if s_staged:
            self._t(sb)[:src.numel()].copy_(src.reshape(-1))
        req = self._track(fn(sb, db))
        if d_staged:
            dst.copy_(self._t(db)[:dst.numel()].view_as(dst))  # (works for non-contiguous destinations too)
        return req

    # -- collectives ---------------------------------------------------------
    def all_reduce(self, t: torch.Tensor, op=SUM):
        parts = self._chunks(t)
        if parts:
            for p in parts:
                req = self.all_reduce(p, op)
            return req
        n = t.numel()
        return self._run(lambda s, d: self.accl.allreduce(s, d, n, op, self.comm_id, self._res, self._res, run_async=self._async), t, t, n, n)

    def broadcast(self, t: torch.Tensor, root=0):
        parts = self._chunks(t)
        if parts:
            for p in parts:
                req = self.broadcast(p, root)
            return req
        n = t.numel()
        return self._run(lambda s, d: self.accl.bcast(s, n, root, self.comm_id, self._res, self._res, run_async=self._async), t, t, n, n)

    def all_gather_into_tensor(self, out: torch.Tensor, inp: torch.Tensor):
        n = inp.numel()
        return self._run(lambda s, d: self.accl.allgather(s, d, n, self.comm_id, self._res, self._res, run_async=self._async), inp, out, n, n * self.world)

    def reduce_scatter_tensor(self, out: torch.Tensor, inp: torch.Tensor, op=SUM):
        n = out.numel()
        return self._run(lambda s, d: self.accl.reduce_scatter(s, d, n, op, self.comm_id, self._res, self._res, run_async=self._async), inp, out, n * self.world, n)

    def all_to_all_single(self, out: torch.Tensor, inp: torch.Tensor):
        n = inp.numel() // self.world
        return self._run(lambda s, d: self.accl.alltoall(s, d, n, self.comm_id, self._res, self._res, run_async=self._async), inp, out, n * self.world, n * self.world)

    def all_to_all_v(self, out: torch.Tensor, inp: torch.Tensor, send_counts: torch.Tensor, recv_counts: torch.Tensor):
        """Uneven all-to-all in elements: send_counts[q] elements of `inp` go to rank q and recv_counts[p] elements
        from rank p land in `out`, both packed in rank order.  The counts are int64 tensors of `world` elements (on
        the GPU for the CUDA backend); they are packed with device copies and read by the engine, so nothing waits
        for the host.  Capacities are inp.numel() and out.numel().  The elements of `out` past the received blocks
        keep their values when `out` lives in the heap; a staged `out` gets the staging buffer's there (undefined)."""
        P = self.world
        cb = self._scratch.get(("counts", P))
        if cb is None:
            cb = self._scratch[("counts", P)] = self.accl.create_buffer(2 * P, torch.int64)
        ct = self._t(cb)
        ct[:P].copy_(send_counts.reshape(-1))
        ct[P:2 * P].copy_(recv_counts.reshape(-1))

        def fn(s, d):
            # a staging buffer may be longer than the tensor: the capacities are the tensors' own lengths
            s = s if s.length == inp.numel() else s.slice(0, inp.numel())
            d = d if d.length == out.numel() else d.slice(0, out.numel())
            return self.accl.alltoallv(s, d, cb, self.comm_id, self._res, self._res, run_async=self._async)
        # a rank may send or receive nothing: stage through one element, pass a capacity of zero
        src, dst = (inp if inp.numel() else inp.new_empty(1)), (out if out.numel() else out.new_empty(1))
        return self._run(fn, src, dst, inp.numel(), out.numel())

    def send(self, t: torch.Tensor, dst, tag=0):
        sb, staged = self._buffer_of(t, "s")
        if staged:
            self._t(sb)[:t.numel()].copy_(t.reshape(-1))
        # always asynchronous: a blocking rendezvous send would wait for the peer's recv
        return self._track(self.accl.send(sb, t.numel(), dst, tag, self.comm_id, self._res, run_async=True))

    def recv(self, t: torch.Tensor, src, tag=0):
        db, staged = self._buffer_of(t, "d")
        req = self._track(self.accl.recv(db, t.numel(), src, tag, self.comm_id, self._res, run_async=self._async))
        if staged:
            if self._engine and req is not None:
                req.wait()
            t.copy_(self._t(db)[:t.numel()].view_as(t))
        return req

    def barrier(self):
        self.accl.barrier(self.comm_id)
        self.check(block=True)


class GradBucket:
    """A flat gradient bucket in the symmetric heap (DP all-reduce or ZeRO reduce_scatter)."""

    def __init__(self, group: TensorGroup, numel, dtype=torch.bfloat16):
        self.group = group
        self.numel = (numel + group.world - 1) // group.world * group.world
        self.flat = group.empty(self.numel, dtype=dtype)
        self.flat.zero_()

    def views(self, shapes):
        """Carve parameter-shaped gradient views out of the bucket."""
        out, off = [], 0
        for shp in shapes:
            n = 1
            for s in shp:
                n *= s
            out.append(self.flat[off:off + n].view(*shp))
            off += n
        return out

    def all_reduce(self, average=True):
        req = self.group.all_reduce(self.flat)
        if average:
            self.flat.div_(self.group.world)
        return req

    def reduce_scatter(self):
        shard = self.flat.view(self.group.world, -1)[self.group.rank]
        buf = self.flat._accl_buffer
        n = self.numel // self.group.world
        out = self.group.empty(n, dtype=self.flat.dtype)
        g = self.group
        g._track(g.accl.reduce_scatter(buf, out._accl_buffer, n, SUM, g.comm_id, g._res, g._res, run_async=g._async))
        del shard
        return out


def row_forward_fused(cuda, dtype, m, world, out_features, in_features_per_rank):
    """Whether RowParallelLinear's forward runs on ops.gemm_reduce_scatter: [m, K_r] @ [N, K_r]^T, reduce-scattered."""
    return (cuda and dtype == torch.bfloat16 and m % (128 * world) == 0 and out_features % 256 == 0 and
            in_features_per_rank % 64 == 0)


def row_backward_fused(cuda, comm_id, dtype, m, world, out_features, in_features_per_rank):
    """Whether RowParallelLinear's input gradient runs on ops.all_gather_gemm: dX_r = all_gather(dY_shard) @ W_r, the
    weight [N, K_r] read as [K, N] ("kn"): output columns K_r % 256, contraction N % 64."""
    return (cuda and comm_id == 0 and dtype == torch.bfloat16 and m % (128 * world) == 0 and m // 128 <= 1024 and
            in_features_per_rank % 256 == 0 and out_features % 64 == 0)


def column_forward_fused(cuda, comm_id, dtype, m, world, in_features, out_features_per_rank):
    """Whether SeqParallelColumnLinear's forward runs on ops.all_gather_gemm: all_gather(x [m, K]) @ [N_r, K]^T."""
    return (cuda and comm_id == 0 and dtype == torch.bfloat16 and m % 128 == 0 and m * world // 128 <= 1024 and
            out_features_per_rank % 256 == 0 and in_features % 64 == 0)


def column_backward_fused(cuda, comm_id, dtype, m, world, in_features, out_features_per_rank):
    """Whether SeqParallelColumnLinear's input gradient runs on ops.gemm_reduce_scatter: dX_shard =
    reduce_scatter(dY [m P, N_r] @ W), the weight [N_r, K] read as [K, N] ("kn"): output columns K % 256, contraction
    N_r % 64."""
    return (cuda and comm_id == 0 and dtype == torch.bfloat16 and m % 128 == 0 and in_features % 256 == 0 and
            out_features_per_rank % 64 == 0)


def _ar_fits(m, n):
    return m % 128 == 0 and n % 256 == 0 and (m // 128) * (n // 256) <= GEMM_AR_MAX_TILES


def row_ar_forward_fused(cuda, comm_id, dtype, m, out_features, in_features_per_rank):
    """Whether ReplicatedRowParallelLinear's forward runs on ops.gemm_all_reduce: all_reduce([m, K_r] @ [N, K_r]^T).
    Decode-sized m < 128 and every m % 128 != 0 take matmul + all_reduce."""
    return (cuda and comm_id == 0 and dtype == torch.bfloat16 and _ar_fits(m, out_features) and
            in_features_per_rank % 64 == 0)


def column_ar_backward_fused(cuda, comm_id, dtype, m, in_features, out_features_per_rank):
    """Whether ReplicatedColumnParallelLinear's input gradient runs on ops.gemm_all_reduce: dX = all_reduce(dY [m, N_r]
    @ W_r), the weight [N_r, K] read as [K, N] ("kn"): output columns K % 256, contraction N_r % 64."""
    return (cuda and comm_id == 0 and dtype == torch.bfloat16 and _ar_fits(m, in_features) and
            out_features_per_rank % 64 == 0)


def _heap_buffer(layer, attr, n):
    """The layer's heap buffer `attr` of n bf16 elements, (re)allocated here: in forward, in the rank's own thread and
    in layer order, so it sits at the same heap offset on every rank."""
    buf = getattr(layer, attr)
    if buf is None or buf.length != n:
        buf = layer.group.accl.create_buffer(n, torch.bfloat16)
        setattr(layer, attr, buf)
    return buf


def _dtype_of(x, weight):
    return x.dtype if x.dtype == weight.dtype else None


def _wants_grad(x, weight):
    return torch.is_grad_enabled() and (x.requires_grad or weight.requires_grad)


class _RowParallelFn(torch.autograd.Function):
    """y_shard = reduce_scatter(x_r W_r^T); dX_r = all_gather(dY_shard) W_r, dW_r = all_gather(dY_shard)^T x_r."""

    @staticmethod
    def forward(ctx, x, weight, layer):
        group = layer.group
        m, k = x.shape
        n, P = weight.shape[0], group.world
        cuda = bool(group.accl.is_cuda)
        ctx.layer, ctx.m = layer, m
        ctx.bwd_fused = row_backward_fused(cuda, group.comm_id, _dtype_of(x, weight), m, P, n, k)
        ctx.dy_buf = _heap_buffer(layer, "_dy_shard", m // P * n) if ctx.bwd_fused else None
        ctx.save_for_backward(x, weight)
        return layer._forward(x, weight, training=True)

    @staticmethod
    def backward(ctx, dy):
        from ..ops import all_gather_gemm
        x, weight = ctx.saved_tensors
        group = ctx.layer.group
        dy = dy.contiguous()
        dx = None
        if ctx.bwd_fused:
            shard = ctx.dy_buf.dev.view(dy.shape)
            shard.copy_(dy)
            st = group.plugin_status()
            dx, gathered = all_gather_gemm(group.accl, shard, weight.detach(), status=st, w_layout="kn")
            group.note_plugin_status(st)
        else:
            gathered = torch.empty(ctx.m, dy.shape[1], dtype=dy.dtype, device=dy.device)
            group.all_gather_into_tensor(gathered, dy)
            if ctx.needs_input_grad[0]:
                dx = gathered @ weight
        dw = gathered.t() @ x if ctx.needs_input_grad[1] else None
        return (dx if ctx.needs_input_grad[0] else None), dw, None


class _ColumnParallelFn(torch.autograd.Function):
    """y = all_gather(x_r) W_r^T; dX_r = reduce_scatter(dY W_r), dW_r = dY^T all_gather(x_r)."""

    @staticmethod
    def forward(ctx, x, weight, layer):
        group = layer.group
        m, k = x.shape
        n, P = weight.shape[0], group.world
        cuda = bool(group.accl.is_cuda)
        ctx.layer, ctx.m = layer, m
        ctx.bwd_fused = column_backward_fused(cuda, group.comm_id, _dtype_of(x, weight), m, P, k, n)
        ctx.dx_buf = _heap_buffer(layer, "_dx_shard", m * k) if ctx.bwd_fused and ctx.needs_input_grad[0] else None
        out, gathered = layer._forward(x, weight, training=True)
        ctx.save_for_backward(gathered, weight)
        return out

    @staticmethod
    def backward(ctx, dy):
        from ..ops import gemm_reduce_scatter
        gathered, weight = ctx.saved_tensors
        group = ctx.layer.group
        dy = dy.contiguous()
        dx = None
        if ctx.needs_input_grad[0]:
            if ctx.bwd_fused:
                st = group.plugin_status()
                gemm_reduce_scatter(group.accl, dy, weight.detach(), ctx.dx_buf, status=st, w_layout="kn")
                group.note_plugin_status(st)
                # the heap buffer is rewritten by the next backward through this layer
                dx = ctx.dx_buf.dev.view(ctx.m, weight.shape[1]).clone()
            else:
                dx = torch.empty(ctx.m, weight.shape[1], dtype=dy.dtype, device=dy.device)
                group.reduce_scatter_tensor(dx, (dy @ weight).contiguous())
        dw = dy.t() @ gathered if ctx.needs_input_grad[1] else None
        return dx, dw, None


class RowParallelLinear(torch.nn.Module):
    """y = reduce_scatter_over_ranks(x_r @ W_r^T): Megatron row-parallel linear with a sequence-parallel
    output shard.  On the CUDA backend the GEMM (wgmma) emits its tiles straight into the owner rank's
    shard over NVLink (accl_b200.ops.gemm_reduce_scatter); elsewhere falls back to matmul + reduce_scatter.
    Trainable: with grad enabled the input gradient dX_r = all_gather(dY_shard) @ W_r runs on
    accl_b200.ops.all_gather_gemm reading W_r as [K, N] (no transposed copy) when the shape allows it
    (`row_backward_fused`), else on all_gather + matmul; dW_r = all_gather(dY_shard)^T @ x_r is a local matmul.
    Every rank must build its layers and run them in the same order (the heap buffers sit at the same offset on every
    rank), and fused-call errors surface at `group.check(block=True)` / `group.barrier()`."""

    def __init__(self, group: TensorGroup, in_features_per_rank, out_features, dtype=torch.bfloat16, device=None):
        super().__init__()
        self.group = group
        dev = device if device is not None else (torch.device("cuda", group.accl.cuda_device) if group.accl.is_cuda else "cpu")
        self.weight = torch.nn.Parameter(torch.empty(out_features, in_features_per_rank, dtype=dtype, device=dev))
        torch.nn.init.normal_(self.weight, std=0.02)
        self._out = None
        self._dy_shard = None  # heap buffer of the fused backward's all-gather operand

    def forward(self, x):
        if _wants_grad(x, self.weight):
            return _RowParallelFn.apply(x, self.weight, self)
        with torch.no_grad():
            return self._forward(x, self.weight)

    def _forward(self, x, weight, training=False):
        """training: the fused call reports into the group's status word, and the result is copied out of the layer's
        heap buffer, which the next call rewrites (micro-batches, recomputation)."""
        from ..ops import gemm_reduce_scatter
        m = x.shape[0]
        P = self.group.world
        if row_forward_fused(bool(self.group.accl.is_cuda), x.dtype, m, P, weight.shape[0], weight.shape[1]):
            if self._out is None or self._out.length != m // P * weight.shape[0]:
                self._out = self.group.accl.create_buffer(m // P * weight.shape[0], torch.bfloat16)
            if training:
                st = self.group.plugin_status()
                gemm_reduce_scatter(self.group.accl, x.contiguous(), weight.detach(), self._out, status=st)
                self.group.note_plugin_status(st)
                return self._out.dev.view(m // P, weight.shape[0]).clone()
            gemm_reduce_scatter(self.group.accl, x.contiguous(), weight.data, self._out)
            return self._out.dev.view(m // P, weight.shape[0])
        full = x @ weight.t()
        out = torch.empty(m // P, weight.shape[0], dtype=full.dtype, device=full.device)
        self.group.reduce_scatter_tensor(out, full)
        return out


class SeqParallelColumnLinear(torch.nn.Module):
    """y = all_gather_over_ranks(x_r) @ W_r^T: Megatron column-parallel linear on a sequence-parallel input shard,
    the counterpart of `RowParallelLinear`.  forward(x_shard [m, in_features]) returns [m * P, out_features_per_rank].
    On the CUDA backend (bf16, m % 128 == 0, out_features_per_rank % 256 == 0, in_features % 64 == 0) the shard is
    copied into a heap buffer the layer keeps and one kernel gathers the rows while the GEMM runs
    (accl_b200.ops.all_gather_gemm); elsewhere falls back to all_gather + matmul.  Every rank must build its layers
    and run them in the same order (the heap buffer sits at the same offset on every rank).
    Trainable: with grad enabled the input gradient dX_shard = reduce_scatter(dY @ W_r) runs on
    accl_b200.ops.gemm_reduce_scatter reading W_r as [K, N] (no transposed copy) when the shape allows it
    (`column_backward_fused`), else on matmul + reduce_scatter; dW_r = dY^T @ gathered reuses the gathered input the
    forward returns.  Fused-call errors surface at `group.check(block=True)` / `group.barrier()`."""

    def __init__(self, group: TensorGroup, in_features, out_features_per_rank, dtype=torch.bfloat16, device=None):
        super().__init__()
        self.group = group
        dev = device if device is not None else (torch.device("cuda", group.accl.cuda_device) if group.accl.is_cuda else "cpu")
        self.weight = torch.nn.Parameter(torch.empty(out_features_per_rank, in_features, dtype=dtype, device=dev))
        torch.nn.init.normal_(self.weight, std=0.02)
        self._shard = None
        self._dx_shard = None  # heap buffer of the fused backward's reduce-scattered input gradient

    def forward(self, x):
        if _wants_grad(x, self.weight):
            return _ColumnParallelFn.apply(x, self.weight, self)
        with torch.no_grad():
            return self._forward(x, self.weight)[0]

    def _forward(self, x, weight, training=False):
        """(y, the gathered input [m P, in_features]); training: the fused call reports into the group's status word."""
        from ..ops import all_gather_gemm
        m, k = x.shape
        P = self.group.world
        n = weight.shape[0]
        if column_forward_fused(bool(self.group.accl.is_cuda), self.group.comm_id, _dtype_of(x, weight), m, P, k, n):
            if self._shard is None or self._shard.length != m * k:
                self._shard = self.group.accl.create_buffer(m * k, torch.bfloat16)
            shard = self._shard.dev.view(m, k)
            shard.copy_(x)
            if training:
                st = self.group.plugin_status()
                out, gathered = all_gather_gemm(self.group.accl, shard, weight.detach(), status=st)
                self.group.note_plugin_status(st)
                return out, gathered
            return all_gather_gemm(self.group.accl, shard, weight.data)
        full = torch.empty(m * P, k, dtype=x.dtype, device=x.device)
        self.group.all_gather_into_tensor(full, x.contiguous())
        return full @ weight.t(), full


class _ReplicatedRowFn(torch.autograd.Function):
    """y = all_reduce(x_r W_r^T); dX_r = dY W_r, dW_r = dY^T x_r (dY is replicated: no communication)."""

    @staticmethod
    def forward(ctx, x, weight, layer):
        ctx.save_for_backward(x, weight)
        return layer._forward(x, weight, training=True)

    @staticmethod
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        dx = dy @ weight if ctx.needs_input_grad[0] else None
        dw = dy.t() @ x if ctx.needs_input_grad[1] else None
        return dx, dw, None


class _ReplicatedColumnFn(torch.autograd.Function):
    """y_r = x W_r^T; dX = all_reduce(dY_r W_r), dW_r = dY_r^T x."""

    @staticmethod
    def forward(ctx, x, weight, layer):
        group = layer.group
        m, k = x.shape
        cuda = bool(group.accl.is_cuda)
        ctx.layer, ctx.m = layer, m
        ctx.bwd_fused = column_ar_backward_fused(cuda, group.comm_id, _dtype_of(x, weight), m, k, weight.shape[0])
        ctx.dx_buf = _heap_buffer(layer, "_dx", m * k) if ctx.bwd_fused and ctx.needs_input_grad[0] else None
        ctx.save_for_backward(x, weight)
        return x @ weight.t()

    @staticmethod
    def backward(ctx, dy):
        from ..ops import gemm_all_reduce
        x, weight = ctx.saved_tensors
        group = ctx.layer.group
        dy = dy.contiguous()
        dx = None
        if ctx.needs_input_grad[0]:
            if ctx.dx_buf is not None:
                st = group.plugin_status()
                gemm_all_reduce(group.accl, dy, weight.detach(), ctx.dx_buf, status=st, w_layout="kn")
                group.note_plugin_status(st)
                # the heap buffer is rewritten by the next backward through this layer
                dx = ctx.dx_buf.dev.view(ctx.m, weight.shape[1]).clone()
            else:
                dx = (dy @ weight).contiguous()
                group.all_reduce(dx)
        dw = dy.t() @ x if ctx.needs_input_grad[1] else None
        return dx, dw, None


class ReplicatedRowParallelLinear(torch.nn.Module):
    """y = all_reduce_over_ranks(x_r @ W_r^T): Megatron row-parallel linear whose output [m, out_features] is replicated
    on every rank (the non-sequence-parallel counterpart of `RowParallelLinear`).  On the CUDA backend (bf16, m % 128 ==
    0, out_features % 256 == 0, in_features_per_rank % 64 == 0, `row_ar_forward_fused`) the all-reduce runs inside the
    GEMM (accl_b200.ops.gemm_all_reduce) into a heap buffer the layer keeps, and every rank gets the same bits;
    elsewhere (emulator, fp32, decode-sized m < 128) it falls back to matmul + all_reduce.
    Trainable: dX_r = dY @ W_r and dW_r = dY^T @ x_r are local matmuls.  Every rank must build its layers and run them
    in the same order (the heap buffer sits at the same offset on every rank), and fused-call errors surface at
    `group.check(block=True)` / `group.barrier()`."""

    def __init__(self, group: TensorGroup, in_features_per_rank, out_features, dtype=torch.bfloat16, device=None):
        super().__init__()
        self.group = group
        dev = device if device is not None else (torch.device("cuda", group.accl.cuda_device) if group.accl.is_cuda else "cpu")
        self.weight = torch.nn.Parameter(torch.empty(out_features, in_features_per_rank, dtype=dtype, device=dev))
        torch.nn.init.normal_(self.weight, std=0.02)
        self._out = None

    def forward(self, x):
        if _wants_grad(x, self.weight):
            return _ReplicatedRowFn.apply(x, self.weight, self)
        with torch.no_grad():
            return self._forward(x, self.weight)

    def _forward(self, x, weight, training=False):
        """training: the fused call reports into the group's status word, and the result is copied out of the layer's
        heap buffer, which the next call rewrites (micro-batches, recomputation)."""
        from ..ops import gemm_all_reduce
        m, k = x.shape
        n = weight.shape[0]
        g = self.group
        if row_ar_forward_fused(bool(g.accl.is_cuda), g.comm_id, _dtype_of(x, weight), m, n, k):
            out = _heap_buffer(self, "_out", m * n)
            if training:
                st = g.plugin_status()
                gemm_all_reduce(g.accl, x.contiguous(), weight.detach(), out, status=st)
                g.note_plugin_status(st)
                return out.dev.view(m, n).clone()
            gemm_all_reduce(g.accl, x.contiguous(), weight.data, out)
            return out.dev.view(m, n)
        y = (x @ weight.t()).contiguous()
        g.all_reduce(y)
        return y


class ReplicatedColumnParallelLinear(torch.nn.Module):
    """y_r = x @ W_r^T: Megatron column-parallel linear on an input [m, in_features] replicated on every rank; returns
    this rank's [m, out_features_per_rank] features with no communication in forward (the non-sequence-parallel
    counterpart of `SeqParallelColumnLinear`).  Trainable: the input gradient dX = all_reduce(dY_r @ W_r) runs on
    accl_b200.ops.gemm_all_reduce reading W_r as [K, N] (no transposed copy) when the shape allows it
    (`column_ar_backward_fused`), else on matmul + all_reduce; dW_r = dY_r^T @ x is a local matmul.  Every rank must
    build its layers and run them in the same order, and fused-call errors surface at `group.check(block=True)` /
    `group.barrier()`."""

    def __init__(self, group: TensorGroup, in_features, out_features_per_rank, dtype=torch.bfloat16, device=None):
        super().__init__()
        self.group = group
        dev = device if device is not None else (torch.device("cuda", group.accl.cuda_device) if group.accl.is_cuda else "cpu")
        self.weight = torch.nn.Parameter(torch.empty(out_features_per_rank, in_features, dtype=dtype, device=dev))
        torch.nn.init.normal_(self.weight, std=0.02)
        self._dx = None  # heap buffer of the fused backward's all-reduced input gradient

    def forward(self, x):
        if _wants_grad(x, self.weight):
            return _ReplicatedColumnFn.apply(x, self.weight, self)
        with torch.no_grad():
            return x @ self.weight.t()


def ar_rmsnorm_fused(cuda, comm_id, dtype, m, hidden):
    """Whether AllReduceRMSNorm's forward runs on ops.all_reduce_rmsnorm: bf16 rows of 8 to 16384 features, a multiple
    of 8, on the world communicator of the CUDA backend."""
    return (cuda and comm_id == 0 and dtype == torch.bfloat16 and m >= 1 and hidden % 8 == 0 and
            8 <= hidden <= AR_RMSNORM_MAX_H)


def _rms_norm_backward(h, weight, eps, dy, dh_out):
    """(dh, dweight) of y = rms_norm(h) * weight, from the saved h (fp32 math; rstd is recomputed)."""
    hf = h.float()
    rstd = torch.rsqrt(hf.pow(2).mean(-1, keepdim=True) + eps)
    hhat = hf * rstd
    dyf = dy.float()
    g = dyf * weight.float()
    dh = rstd * (g - hhat * (g * hhat).mean(-1, keepdim=True))
    if dh_out is not None:
        dh = dh + dh_out.float()
    return dh, (dyf * hhat).sum(0)


class _ArRmsNormFn(torch.autograd.Function):
    """(y, h) = (rms_norm(h) * weight, all_reduce(partial) + residual).  y and h are replicated, so the backward is local:
    dpartial = dresidual = dh, with dh = rstd (dy w - h^ mean(dy w h^)) + dh_out and dweight = sum_rows dy h^."""

    @staticmethod
    def forward(ctx, partial, residual, weight, layer):
        y, h = layer._forward(partial, residual, weight, training=True)
        ctx.eps, ctx.has_residual = layer.eps, residual is not None
        ctx.save_for_backward(h, weight)
        return y, h

    @staticmethod
    def backward(ctx, dy, dh_out):
        h, weight = ctx.saved_tensors
        dh, dw = _rms_norm_backward(h, weight, ctx.eps, dy, dh_out)
        dh = dh.to(h.dtype)
        return dh, (dh if ctx.has_residual else None), dw.to(weight.dtype), None


class AllReduceRMSNorm(torch.nn.Module):
    """(y, h) = (RMSNorm(h) * weight, all_reduce_over_ranks(partial) + residual): the step after the row-parallel matmul of
    a transformer block whose activations are replicated on every rank.  forward(partial [m, hidden], residual=None):
    `partial` is this rank's unreduced output of a local matmul (F.linear(x_r, W_r)), `h` the new residual stream
    and `y` its normalisation, both replicated.
    On the CUDA backend (bf16, hidden % 8 == 0, 8 <= hidden <= 16384, `ar_rmsnorm_fused`) the all-reduce, the residual
    add and the norm run in one kernel (accl_b200.ops.all_reduce_rmsnorm) and every rank gets the same bits: `partial`
    is read in place when it lives in the symmetric heap, else it is copied into a heap buffer the layer keeps, and `h`
    is written into a second heap buffer the layer keeps.  The fused call rounds h to bf16 once; the fallback
    (emulator, fp32, other shapes: all_reduce, add, torch rms_norm) rounds the all-reduce result and then its sum with
    the residual.
    Trainable: the backward is local torch math (y and h are replicated), dpartial = dresidual = dh.  With grad enabled
    the fused call's status goes into the group's word (raised at `group.check(block=True)` / `group.barrier()`) and h is
    copied out of the heap buffer; under no_grad / inference_mode h is a view of the heap buffer, which the layer's next
    call rewrites (`residual=h` from the previous call is updated in place).  Every rank must build its layers and run
    them in the same order (the heap buffers sit at the same offset on every rank)."""

    def __init__(self, group: TensorGroup, hidden, eps=1e-6, dtype=torch.bfloat16, device=None):
        super().__init__()
        self.group = group
        self.eps = eps
        dev = device if device is not None else (torch.device("cuda", group.accl.cuda_device) if group.accl.is_cuda else "cpu")
        self.weight = torch.nn.Parameter(torch.ones(hidden, dtype=dtype, device=dev))
        self._x = None  # heap buffer of a partial that does not live in the heap
        self._h = None  # heap buffer of the residual stream

    def forward(self, partial, residual=None):
        if torch.is_grad_enabled() and (partial.requires_grad or self.weight.requires_grad or
                                        (residual is not None and residual.requires_grad)):
            return _ArRmsNormFn.apply(partial, residual, self.weight, self)
        with torch.no_grad():
            return self._forward(partial, residual, self.weight)

    def _forward(self, partial, residual, weight, training=False):
        """training: the fused call reports into the group's status word, and h is copied out of the heap buffer."""
        from ..ops import all_reduce_rmsnorm
        m, n = partial.shape
        g = self.group
        dtype = _dtype_of(partial, weight)
        if residual is not None and residual.dtype != dtype:
            dtype = None
        if ar_rmsnorm_fused(bool(g.accl.is_cuda), g.comm_id, dtype, m, n):
            if partial.is_contiguous() and g.accl.heap_contains(partial) and partial.data_ptr() % 16 == 0:
                x = partial
            else:
                x = _heap_buffer(self, "_x", m * n).dev.view(m, n)
                x.copy_(partial)
            h = _heap_buffer(self, "_h", m * n).dev.view(m, n)
            res = None if residual is None else residual.detach()
            if res is not None and not (res.is_contiguous() and res.data_ptr() % 16 == 0):
                res = res.contiguous()
            st = g.plugin_status() if training else None
            y, h = all_reduce_rmsnorm(g.accl, x, weight.detach(), res, self.eps, residual_out=h, status=st)
            if training:
                g.note_plugin_status(st)
                return y, h.clone()
            return y, h
        s = partial.detach().clone().contiguous()
        g.all_reduce(s)
        h = s if residual is None else s + residual.detach()
        return torch.nn.functional.rms_norm(h, (n,), weight.detach(), self.eps), h


def ring_exchange(group: TensorGroup, send_t: torch.Tensor, recv_t: torch.Tensor, tag=0):
    """One step of a ring schedule (context parallelism / ring attention): pass a block to the next
    rank while receiving the previous rank's block.  Even ranks send first (legal for both protocols)."""
    nxt, prv = (group.rank + 1) % group.world, (group.rank - 1) % group.world
    if group.rank % 2 == 0:
        s = group.send(send_t, nxt, tag)
        r = group.recv(recv_t, prv, tag)
    else:
        r = group.recv(recv_t, prv, tag)
        s = group.send(send_t, nxt, tag)
    return s, r
