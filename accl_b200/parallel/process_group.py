"""`torch.distributed` backend "accl": the collectives of this library behind the standard ProcessGroup
interface, so existing `torch.distributed` code (including DistributedDataParallel) runs on it unchanged.

    import accl_b200.parallel.process_group          # registers the backend
    dist.init_process_group("accl", init_method="tcp://127.0.0.1:29500", rank=r, world_size=w)
    dist.all_reduce(t)

One rank per process.  The engine is chosen like `init_from_env`: the CUDA backend when a GPU and the sm_90a
extension are available (tensors must then be CUDA tensors; calls are stream ordered and their Work objects
complete immediately, like NCCL's), otherwise the CPU emulator over loopback TCP (calls are blocking).
SURVEY 7.2 step 9 ("optional ProcessGroup shim for drop-in comparison").
"""
import math
import os

import torch
import torch.distributed as dist
from torch._C._distributed_c10d import (AllgatherOptions, AllreduceCoalescedOptions, AllreduceOptions, AllToAllOptions,
                                        BarrierOptions, BroadcastOptions, GatherOptions, ReduceOptions,
                                        ReduceScatterOptions, ScatterOptions, _create_work_from_future)
from torch.futures import Future

from ..core import MAX, SUM
from . import TensorGroup, init_from_env


def _done(result):
    fut = Future()
    fut.set_result(result)
    return _create_work_from_future(fut)


def _cuda_device_of(x):
    if isinstance(x, torch.Tensor):
        return x.device if x.is_cuda else None
    if isinstance(x, (list, tuple)):
        for y in x:
            d = _cuda_device_of(y)
            if d is not None:
                return d
    return None


class AcclProcessGroup(dist.ProcessGroup):
    def __init__(self, rank, world_size, accl, comm_id=0):
        super().__init__(rank, world_size)
        self._rank, self._world = rank, world_size
        self.accl = accl
        self.group = TensorGroup(accl, comm_id)
        self._comm_stream = None   # CUDA: collectives run here so that they overlap the caller's compute (like NCCL's)
        self._overlap = os.environ.get("ACCL_PG_OVERLAP", "1") not in ("", "0")

    def _join(self):
        """Ops that run on the caller's stream share staging buffers with the communication stream: order after it."""
        if self._comm_stream is not None:
            torch.cuda.current_stream(self._comm_stream.device).wait_stream(self._comm_stream)

    def _run(self, tensors, fn):
        """Run `fn` (which issues the collective and any staging copies) and return its Work.  CUDA tensors: on this
        group's communication stream, ordered after what the caller has queued so far; the Work's future carries the
        completion event, so `work.wait()` / `fut.then(...)` order the caller's stream after the collective without
        blocking the host — DDP's backward keeps running while a bucket is being reduced."""
        dev = _cuda_device_of(tensors) if self.accl.is_cuda else None
        if dev is None or not self._overlap:
            fn()
            return _done(tensors)
        if self._comm_stream is None:
            self._comm_stream = torch.cuda.Stream(device=dev, priority=-1)
        cs = self._comm_stream
        cs.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(cs):
            fn()
            fut = Future(devices=[dev])
            fut.set_result(tensors)          # records the completion event on the communication stream
        for t in (tensors if isinstance(tensors, (list, tuple)) else [tensors]):
            if isinstance(t, torch.Tensor) and t.is_cuda:
                t.record_stream(cs)
        return _create_work_from_future(fut)

    # -- identity ------------------------------------------------------------
    def getBackendName(self):
        return "accl"

    def size(self):
        return self._world

    def __repr__(self):
        return f"AcclProcessGroup(rank={self._rank}, world={self._world}, {self.accl.describe()})"

    # -- helpers ----------------------------------------------------------------
    @staticmethod
    def _op(opts):
        op = getattr(opts, "reduceOp", dist.ReduceOp.SUM)
        if op == dist.ReduceOp.SUM:
            return SUM, None
        if op == dist.ReduceOp.MAX:
            return MAX, None
        if op == dist.ReduceOp.AVG:
            return SUM, "avg"
        raise NotImplementedError(f"accl backend: reduce op {op} (SUM, MAX and AVG are supported)")

    def _finish(self, t, post):
        if post == "avg":
            t.div_(self._world)

    # -- collectives ----------------------------------------------------------------
    def allreduce(self, tensor_list, opts=AllreduceOptions()):
        fn, post = self._op(opts)

        def go():
            for t in tensor_list:
                self.group.all_reduce(t, fn)
                self._finish(t, post)
        return self._run(tensor_list, go)

    def allreduce_coalesced(self, tensor_list, opts=AllreduceCoalescedOptions()):
        return self.allreduce(tensor_list, opts)

    def broadcast(self, tensor_list, opts=BroadcastOptions()):
        def go():
            for t in tensor_list:
                self.group.broadcast(t, opts.rootRank)
        return self._run(tensor_list, go)

    def reduce(self, tensor_list, opts=ReduceOptions()):
        self._join()
        fn, post = self._op(opts)
        for t in tensor_list:
            n = t.numel()
            flat = t.reshape(-1) if t.is_contiguous() else t.contiguous().view(-1)
            sb, _ = self.group._buffer_of(flat, "s")
            db, _ = self.group._buffer_of(flat, "d")
            self.group._t(sb)[:n].copy_(flat)
            self.group._track(self.accl.reduce(sb, db, n, opts.rootRank, fn, self.group.comm_id, self.group._res,
                                               self.group._res, run_async=self.group._async))
            if self._rank == opts.rootRank:
                t.copy_(self.group._t(db)[:n].view_as(t))
                self._finish(t, post)
        return _done(tensor_list)

    def _allgather_base(self, output_tensor, input_tensor, opts=AllgatherOptions()):
        return self._run([output_tensor, input_tensor], lambda: self.group.all_gather_into_tensor(output_tensor, input_tensor.contiguous()))

    def allgather(self, output_tensors, input_tensor, opts=AllgatherOptions()):
        self._join()
        for outs, inp in zip(output_tensors, input_tensor):
            flat = torch.empty(self._world * inp.numel(), dtype=inp.dtype, device=inp.device)
            self.group.all_gather_into_tensor(flat, inp.contiguous())
            for o, chunk in zip(outs, flat.chunk(self._world)):
                o.copy_(chunk.view_as(o))
        return _done(output_tensors)

    def allgather_into_tensor_coalesced(self, output_tensor_list, input_tensor_list, opts=AllgatherOptions()):
        for o, i in zip(output_tensor_list, input_tensor_list):
            self._allgather_base(o, i, opts).wait()   # (orders the caller's stream after the communication stream)
        return _done(output_tensor_list)

    def _reduce_scatter_base(self, output_tensor, input_tensor, opts=ReduceScatterOptions()):
        fn, post = self._op(opts)

        def go():
            self.group.reduce_scatter_tensor(output_tensor, input_tensor.contiguous(), fn)
            self._finish(output_tensor, post)
        return self._run([output_tensor, input_tensor], go)

    def reduce_scatter(self, output_tensors, scatter_lists, opts=ReduceScatterOptions()):
        for out, parts in zip(output_tensors, scatter_lists):
            self._reduce_scatter_base(out, torch.cat([p.reshape(-1) for p in parts]), opts).wait()
        return _done(output_tensors)

    def reduce_scatter_tensor_coalesced(self, output_tensors, input_tensors, opts=ReduceScatterOptions()):
        for o, i in zip(output_tensors, input_tensors):
            self._reduce_scatter_base(o, i, opts).wait()
        return _done(output_tensors)

    def alltoall_base(self, output_buffer, input_buffer, output_split_sizes, input_split_sizes, opts=AllToAllOptions()):
        self._join()
        if not output_split_sizes and not input_split_sizes:
            self.group.all_to_all_single(output_buffer, input_buffer.contiguous())
            return _done(output_buffer)
        # uneven: splits are dim-0 rows (an empty list means even splits); the engine takes element counts
        P = self._world
        row = math.prod(input_buffer.shape[1:])   # from the trailing dimensions: a rank may send zero rows
        if math.prod(output_buffer.shape[1:]) != row:
            raise ValueError("accl backend: all_to_all_single with input and output rows of different sizes")
        in_splits = list(input_split_sizes) or [input_buffer.shape[0] // P] * P
        out_splits = list(output_split_sizes) or [output_buffer.shape[0] // P] * P
        dev = input_buffer.device if self.accl.is_cuda else "cpu"
        counts = torch.tensor(in_splits + out_splits, dtype=torch.int64, device=dev) * row
        self.group.all_to_all_v(output_buffer, input_buffer.contiguous(), counts[:P], counts[P:])
        return _done(output_buffer)

    def alltoall(self, output_tensor_list, input_tensor_list, opts=AllToAllOptions()):
        self._join()
        inp = torch.cat([t.reshape(-1) for t in input_tensor_list])
        out = torch.empty_like(inp)
        self.group.all_to_all_single(out, inp)
        for o, chunk in zip(output_tensor_list, out.chunk(self._world)):
            o.copy_(chunk.view_as(o))
        return _done(output_tensor_list)

    def gather(self, output_tensors, input_tensors, opts=GatherOptions()):
        self._join()
        inp = input_tensors[0].contiguous()
        n = inp.numel()
        sb, _ = self.group._buffer_of(inp.view(-1), "s")
        db = self.accl.create_buffer(n * self._world, inp.dtype)
        self.group._t(sb)[:n].copy_(inp.view(-1))
        self.group._track(self.accl.gather(sb, db, n, opts.rootRank, self.group.comm_id, self.group._res, self.group._res,
                                           run_async=self.group._async))
        if self._rank == opts.rootRank:
            for o, chunk in zip(output_tensors[0], self.group._t(db).chunk(self._world)):
                o.copy_(chunk.view_as(o))
        return _done(output_tensors)

    def scatter(self, output_tensors, input_tensors, opts=ScatterOptions()):
        self._join()
        out = output_tensors[0]
        n = out.numel()
        sb = self.accl.create_buffer(n * self._world, out.dtype)
        db, _ = self.group._buffer_of(out.reshape(-1), "d")
        if self._rank == opts.rootRank:
            self.group._t(sb).copy_(torch.cat([t.reshape(-1) for t in input_tensors[0]]))
        self.group._track(self.accl.scatter(sb, db, n, opts.rootRank, self.group.comm_id, self.group._res, self.group._res,
                                            run_async=self.group._async))
        out.copy_(self.group._t(db)[:n].view_as(out))
        return _done(output_tensors)

    def barrier(self, opts=BarrierOptions()):
        self._join()
        self.group.barrier()
        return _done(None)

    # -- point to point ----------------------------------------------------------------
    def send(self, tensors, dst, tag=0):
        self._join()
        reqs = [self.group.send(t.contiguous(), dst, tag) for t in tensors]
        for r in reqs:      # asynchronous issue (a rendezvous send completes when the peer has posted its recv)
            r.wait()
        return _done(None)

    def recv(self, tensors, src, tag=0):
        self._join()
        for t in tensors:
            self.group.recv(t, src, tag)
        return _done(tensors)


_primary = {}  # the world-sized engine of this process: sub-groups are communicators on it


def _create(opts, pg_options=None):
    """Backend constructor (extended API).  The default group builds the engine: ranks meet over a private TCP
    rendezvous whose port is published through the store that torch.distributed hands us (so `init_method` /
    the store decide, not only the environment).  Every further group (`dist.new_group(ranks)`) becomes a
    communicator on that engine (accl::ACCL::create_communicator) with its own protocol-state bank."""
    store, rank, size = opts.store, opts.group_rank, opts.group_size
    ranks = list(getattr(opts, "global_ranks_in_group", []) or range(size))
    if "accl" not in _primary:
        if ranks != list(range(size)):
            raise NotImplementedError("accl backend: the first process group must span all ranks (default group)")
        os.environ["RANK"] = str(rank)
        os.environ["WORLD_SIZE"] = str(size)
        # publish / fetch the bootstrap port through the store (rank 0 derives it from MASTER_PORT or picks 29637)
        if rank == 0:
            port = int(os.environ.get("ACCL_PORT", int(os.environ.get("MASTER_PORT", 29500)) + 137))
            store.set("accl_bootstrap_port", str(port))
        port = int(store.get("accl_bootstrap_port").decode())
        os.environ["ACCL_PORT"] = str(port)
        os.environ["ACCL_EMU_PORT"] = str(port)
        accl = init_from_env(None)
        assert accl.rank == rank and accl.world == size, "accl backend: rank / world size disagree with init_process_group"
        _primary["accl"] = accl
        _primary["ranks"] = accl.generate_ranks(size)
        _primary["pg"] = AcclProcessGroup(rank, size, accl)
        return _primary["pg"]
    accl = _primary["accl"]
    if ranks == list(range(accl.world)):
        # another world-sized group: its own communicator (and bank) so it can be used concurrently
        comm = accl.create_communicator(list(_primary["ranks"]), accl.rank)
        return AcclProcessGroup(rank, size, accl, comm)
    if accl.rank not in ranks:
        raise NotImplementedError("accl backend: this rank is not a member of the group being created")
    comm = accl.create_communicator([_primary["ranks"][g] for g in ranks], ranks.index(accl.rank))
    return AcclProcessGroup(ranks.index(accl.rank), len(ranks), accl, comm)


def heap_mem_pool():
    """`torch.cuda.MemPool` over the symmetric heap of the default "accl" group (see `Accl.heap_mem_pool`): build the
    DDP wrapper (or allocate gradient / activation buffers) inside `with torch.cuda.use_mem_pool(pool):` and the
    backend's collectives take those tensors as zero-copy operands instead of staging them through the heap."""
    if "accl" not in _primary:
        raise RuntimeError('init_process_group("accl") first')
    return _primary["accl"].heap_mem_pool()


dist.Backend.register_backend("accl", _create, extended_api=True, devices=["cpu", "cuda"])
