"""Fused compute+collective plugins (CUDA backend).

* gemm_reduce_scatter: row-parallel linear layer — every rank multiplies its
  K-slice on the tensor cores (wgmma) and each finished tile is added straight
  into the owner rank's output shard over NVLink (no intermediate C, no
  separate reduce_scatter kernel).
* gemm_all_reduce: the same GEMM whose epilogue is an all-reduce — each tile is
  added into its owner rank over NVLink, and the owner copies the finished tile
  into every peer, so every rank ends with the same full C.
* all_gather_gemm: the column-parallel counterpart — the GEMM starts on this
  rank's own rows while the kernel pulls the peers' shards over NVLink, and
  each peer tile waits only for its own 128 rows.
* all_reduce_rmsnorm: the step after a row-parallel matmul with replicated
  activations — the partial sums are all-reduced, the residual added and the
  rows RMS-normalised in one kernel, while the reduced rows are in registers.
* vadd_allreduce: the vector-add plugin; the kernel computes x + y chunk by
  chunk and hands every finished chunk to the persistent engine itself
  (device API, all_reduce_async) while it computes the next one.
* vadd_put / stream_pull: the reference's vadd_put example — x + 1 pushed into
  a stream of the destination rank while computing; the consumer drains it.
"""
import torch

from .. import _C
from ..core import Accl, Buffer
from ..utils.dtypes import to_torch


def _stream_handle(accl):
    h = torch.cuda.current_stream(accl.cuda_device).cuda_stream
    return h if h else 1  # cudaStreamLegacy


def gemm_reduce_scatter(accl: Accl, a: torch.Tensor, w: torch.Tensor, out: Buffer = None, variant: int = 0,
                        out_dtype=None, status: torch.Tensor = None, w_layout: str = "nk") -> Buffer:
    """out[M/P, N] (in the symmetric heap) = reduce_scatter over ranks of a[M, K_r] @ w[N, K_r]^T.

    `a` and `w` are this rank's K-slices (bf16, contiguous, on this rank's GPU).  w_layout "nk" (default): `w` is
    [N, K_r] (nn.Linear layout); "kn": `w` is [K_r, N] and the product is a @ w, e.g. an nn.Linear weight in its own
    backward pass, dX = reduce_scatter(dY @ W), without a transposed copy.
    Needs M % (128 * world) == 0, N % 256 == 0, K_r % 64 == 0.  Stream ordered.
    The shard is bf16 (partials added in bf16 by the TMA unit) or, with an fp32 `out` buffer / out_dtype, fp32
    (the P partial products are accumulated without intermediate rounding); out_dtype defaults to `out`'s dtype, or
    bf16.  `out` must sit at the same heap offset on every rank: allocate it in the same order everywhere.
    variant: 0 automatic, 1 one CTA per 128 x 256 tile, 2 CTA pair (cluster of 2 sharing each W tile) per
    256 x 256 tile (needs M % (256 * world) == 0).
    `status`, optional 1-element int32 CUDA tensor, receives the error bits when the kernel ends (0: success); with
    non-zero bits the shard is not a valid result.  A shard at a different heap offset on some peer sets
    DMA_MISMATCH_ERROR (bit 0) on both ranks, and neither adds into the other's heap.
    Raises ValueError for a wrong dtype, shape, layout or device, or an `out` that is not a large enough heap buffer.
    """
    device = torch.device("cuda", accl.cuda_device)
    _check_operand("gemm_reduce_scatter", "a", a, device)
    _check_operand("gemm_reduce_scatter", "w", w, device)
    kn = _is_kn("gemm_reduce_scatter", w_layout)
    M, K = a.shape
    N, w_k = (w.shape[1], w.shape[0]) if kn else (w.shape[0], w.shape[1])
    P = accl.world
    if w_k != K:
        raise ValueError(f"gemm_reduce_scatter: w has K = {w_k}, a has K = {K}")
    if M % (128 * P) or N % 256 or K % 64 or not (M and N and K):
        raise ValueError(f"gemm_reduce_scatter: need M % (128 * {P}) == 0, N % 256 == 0, K % 64 == 0, none of them zero; "
                         f"got M = {M}, N = {N}, K = {K}")
    if variant not in (0, 1, 2):
        raise ValueError(f"gemm_reduce_scatter: variant must be 0, 1 or 2, got {variant}")
    if variant == 2 and M % (256 * P):
        raise ValueError(f"gemm_reduce_scatter: the CTA-pair variant needs M % (256 * {P}) == 0, got M = {M}")
    if out_dtype not in (None, torch.bfloat16, torch.float32):
        raise ValueError(f"gemm_reduce_scatter: out_dtype must be torch.bfloat16 or torch.float32, got {out_dtype}")
    if out is None:
        out = accl.create_buffer(M // P * N, out_dtype or torch.bfloat16)
    if not isinstance(out, Buffer) or not accl.heap_contains(_device_view(out)):
        raise ValueError("gemm_reduce_scatter: out must be a buffer in the symmetric heap (accl.create_buffer)")
    dt = to_torch(out.dtype)
    if dt not in (torch.bfloat16, torch.float32) or (out_dtype is not None and dt != out_dtype):
        raise ValueError(f"gemm_reduce_scatter: out is {dt}; it must be bf16 or fp32"
                         + (f" and match out_dtype = {out_dtype}" if out_dtype is not None else ""))
    if out.length < M // P * N:
        raise ValueError(f"gemm_reduce_scatter: out holds {out.length} elements, the shard needs {M // P * N}")
    status_ptr = _status_ptr("gemm_reduce_scatter", status, device)
    _C.gemm_reduce_scatter(accl.impl, a.data_ptr(), w.data_ptr(), out.impl, M, N, K, _stream_handle(accl), variant,
                           status_ptr, kn)
    return out


GEMM_AR_MAX_TILES = 16384  # plugins.hpp: most 128 x 256 tiles of one gemm_all_reduce call


def _gemm_ar_counters(accl: Accl) -> Buffer:
    """The heap block of per-tile arrival counters gemm_all_reduce signals in, allocated at this Accl's first call (in
    the same order on every rank, so at the same offset) and kept; the kernel verifies the offsets match."""
    cnt = getattr(accl, "_gemm_ar_counters", None)
    if cnt is None:
        cnt = accl._gemm_ar_counters = accl.create_buffer(GEMM_AR_MAX_TILES, torch.int32)
    return cnt


def gemm_all_reduce(accl: Accl, a: torch.Tensor, w: torch.Tensor, out: Buffer = None, variant: int = 0, out_dtype=None,
                    status: torch.Tensor = None, w_layout: str = "nk") -> Buffer:
    """out[M, N] (in the symmetric heap) = all_reduce over ranks of a[M, K_r] @ w[N, K_r]^T, the same bits on every rank.

    `a` and `w` are this rank's K-slices (bf16, contiguous, on this rank's GPU).  w_layout "nk" (default): `w` is
    [N, K_r] (nn.Linear layout); "kn": `w` is [K_r, N] and the product is a @ w, e.g. an nn.Linear weight in its own
    backward pass, dX = all_reduce(dY @ W), without a transposed copy.
    Needs M % 128 == 0, N % 256 == 0, K_r % 64 == 0 and (M / 128) (N / 256) <= 16384 tiles.  Stream ordered.
    One kernel: every rank adds its partial of each 128 x 256 (or 256 x 256) tile into the tile's owner rank over
    NVLink, and the owner copies the finished tile into every peer's `out`, so all replicas are bit-identical.
    `out` is bf16 (partials added in bf16 by the TMA unit) or, with an fp32 `out` buffer / out_dtype, fp32 (the P
    partial products are accumulated without intermediate rounding); out_dtype defaults to `out`'s dtype, or bf16.
    `out` must sit at the same heap offset on every rank: allocate it in the same order everywhere.
    variant: 0 automatic, 1 one CTA per 128 x 256 tile, 2 CTA pair per 256 x 256 tile (needs M % 256 == 0).
    `status`, optional 1-element int32 CUDA tensor, receives the error bits when the kernel ends (0: success); with
    non-zero bits `out` is not a valid result.  An `out` at a different heap offset on some peer sets
    DMA_MISMATCH_ERROR (bit 0) on both ranks, and neither writes into the other's heap.
    Raises ValueError for a wrong dtype, shape, layout or device, too many tiles, or an `out` that is not a large
    enough heap buffer.
    """
    op = "gemm_all_reduce"
    device = torch.device("cuda", accl.cuda_device)
    _check_operand(op, "a", a, device)
    _check_operand(op, "w", w, device)
    kn = _is_kn(op, w_layout)
    M, K = a.shape
    N, w_k = (w.shape[1], w.shape[0]) if kn else (w.shape[0], w.shape[1])
    if w_k != K:
        raise ValueError(f"{op}: w has K = {w_k}, a has K = {K}")
    if M % 128 or N % 256 or K % 64 or not (M and N and K):
        raise ValueError(f"{op}: need M % 128 == 0, N % 256 == 0, K % 64 == 0, none of them zero; got M = {M}, N = {N}, K = {K}")
    if (M // 128) * (N // 256) > GEMM_AR_MAX_TILES:
        raise ValueError(f"{op}: M = {M}, N = {N} is {(M // 128) * (N // 256)} tiles of 128 x 256, more than {GEMM_AR_MAX_TILES}")
    if variant not in (0, 1, 2):
        raise ValueError(f"{op}: variant must be 0, 1 or 2, got {variant}")
    if variant == 2 and M % 256:
        raise ValueError(f"{op}: the CTA-pair variant needs M % 256 == 0, got M = {M}")
    if out_dtype not in (None, torch.bfloat16, torch.float32):
        raise ValueError(f"{op}: out_dtype must be torch.bfloat16 or torch.float32, got {out_dtype}")
    if out is not None and (not isinstance(out, Buffer) or not accl.heap_contains(_device_view(out))):
        raise ValueError(f"{op}: out must be a buffer in the symmetric heap (accl.create_buffer)")
    if out is not None:
        dt = to_torch(out.dtype)
        if dt not in (torch.bfloat16, torch.float32) or (out_dtype is not None and dt != out_dtype):
            raise ValueError(f"{op}: out is {dt}; it must be bf16 or fp32"
                             + (f" and match out_dtype = {out_dtype}" if out_dtype is not None else ""))
        if out.length < M * N:
            raise ValueError(f"{op}: out holds {out.length} elements, the result needs {M * N}")
    status_ptr = _status_ptr(op, status, device)
    counters = _gemm_ar_counters(accl)
    if out is None:
        out = accl.create_buffer(M * N, out_dtype or torch.bfloat16)
    _C.gemm_all_reduce(accl.impl, a.data_ptr(), w.data_ptr(), out.impl, counters.impl, M, N, K, _stream_handle(accl),
                       variant, status_ptr, kn)
    return out


def _is_kn(op, w_layout):
    if w_layout not in ("nk", "kn"):
        raise ValueError(f'{op}: w_layout must be "nk" or "kn", got {w_layout!r}')
    return w_layout == "kn"


def _device_view(buf: Buffer):
    try:
        return buf.dev
    except RuntimeError:  # a host-only buffer
        return None


def _check_operand(op, name, t, device):
    if not isinstance(t, torch.Tensor) or t.device != device:
        raise ValueError(f"{op}: {name} must be a tensor on {device}")
    if t.dtype != torch.bfloat16 or t.dim() != 2 or not t.is_contiguous():
        raise ValueError(f"{op}: {name} must be a contiguous 2-D bf16 tensor, got {t.dtype} {tuple(t.shape)}")


def _status_ptr(op, status, device):
    if status is None:
        return 0
    if not (isinstance(status, torch.Tensor) and status.device == device and status.dtype == torch.int32 and
            status.numel() == 1):
        raise ValueError(f"{op}: status must be a 1-element int32 tensor on {device}")
    return status.data_ptr()


def _overlap(a: torch.Tensor, b: torch.Tensor) -> bool:
    a0, b0 = a.data_ptr(), b.data_ptr()
    return a0 < b0 + b.numel() * b.element_size() and b0 < a0 + a.numel() * a.element_size()


def all_gather_gemm(accl: Accl, a_shard: torch.Tensor, w: torch.Tensor, out: torch.Tensor = None,
                    gathered: torch.Tensor = None, status: torch.Tensor = None, w_layout: str = "nk"):
    """out[M, N] = all_gather over ranks of a_shard[M/P, K], times w[N, K]^T.  Returns (out, gathered).

    `a_shard` is this rank's rows, a contiguous bf16 tensor in the symmetric heap (a `Buffer.dev` view or a tensor
    from `heap_mem_pool()`), at the same heap offset on every rank: allocate it in the same order everywhere.
    `w` is this rank's output features (bf16, nn.Linear layout); with w_layout "kn" it is [K, N] and the product is
    gathered @ w, e.g. an nn.Linear weight in its own backward pass, dX = all_gather(dY) @ W.  `out` (bf16 [M, N]) and `gathered` (bf16 [M, K],
    every rank's shard in rank order) are ordinary CUDA tensors, allocated when not given.  Needs M % (128 * P) == 0,
    N % 256 == 0, K % 64 == 0 and M <= 128 * 1024.  Stream ordered: a rank may rewrite its shard on the stream right
    after the call.
    `status`, optional 1-element int32 CUDA tensor, receives the error bits when the kernel ends (0: success); a
    shard at a different heap offset on some peer sets DMA_MISMATCH_ERROR (bit 0) on both ranks and is not read.
    Raises ValueError for a shard outside the heap, a wrong dtype, shape or layout, or `out` / `gathered` overlapping
    the shard or each other."""
    if not isinstance(a_shard, torch.Tensor) or not accl.heap_contains(a_shard):
        raise ValueError("all_gather_gemm: a_shard must live in the symmetric heap (a Buffer.dev view or a heap_mem_pool tensor)")
    device = a_shard.device
    _check_operand("all_gather_gemm", "a_shard", a_shard, device)
    _check_operand("all_gather_gemm", "w", w, device)
    kn = _is_kn("all_gather_gemm", w_layout)
    m, K = a_shard.shape
    M, N = m * accl.world, (w.shape[1] if kn else w.shape[0])
    w_k = w.shape[0] if kn else w.shape[1]
    if w_k != K:
        raise ValueError(f"all_gather_gemm: w has K = {w_k}, a_shard has K = {K}")
    if out is None:
        out = torch.empty(M, N, dtype=torch.bfloat16, device=device)
    if gathered is None:
        gathered = torch.empty(M, K, dtype=torch.bfloat16, device=device)
    _check_operand("all_gather_gemm", "out", out, device)
    _check_operand("all_gather_gemm", "gathered", gathered, device)
    if tuple(out.shape) != (M, N) or tuple(gathered.shape) != (M, K):
        raise ValueError(f"all_gather_gemm: need out [{M}, {N}] and gathered [{M}, {K}], "
                         f"got {tuple(out.shape)} and {tuple(gathered.shape)}")
    if _overlap(out, a_shard) or _overlap(gathered, a_shard) or _overlap(out, gathered):
        raise ValueError("all_gather_gemm: out, gathered and a_shard must not overlap")
    status_ptr = _status_ptr("all_gather_gemm", status, device)
    _C.all_gather_gemm(accl.impl, accl.wrap_device(a_shard).impl, w.data_ptr(), gathered.data_ptr(), out.data_ptr(),
                       M, N, K, status_ptr, _stream_handle(accl), kn)
    return out, gathered


AR_RMSNORM_MAX_H = 16384  # plugins.hpp AR_MAX_H: widest row of one all_reduce_rmsnorm call


def all_reduce_rmsnorm(accl: Accl, x: torch.Tensor, weight: torch.Tensor, residual: torch.Tensor = None,
                       eps: float = 1e-6, out: torch.Tensor = None, residual_out: torch.Tensor = None,
                       status: torch.Tensor = None):
    """All-reduce -> residual add -> RMSNorm in one kernel.  Returns (out, residual_out).

        residual_out = bf16(x_0 + x_1 + ... + x_{P-1} + residual)      fp32 sum, ranks added in rank order
        out          = bf16((residual_out * rsqrt(mean(residual_out^2) + eps)) * weight)   per row, in fp32

    `x` [M, H] bf16 is this rank's partial sums (e.g. the output of a row-parallel matmul, x_r @ W_r^T), contiguous,
    in the symmetric heap (a `Buffer.dev` view or a `heap_mem_pool()` tensor) at the same offset on every rank; it is
    only read, and a rank may rewrite it on the stream right after the call.  `residual` [M, H] bf16 (optional) holds
    the same values on every rank; `weight` [H] bf16 is the RMSNorm gain.  `residual_out` [M, H] bf16 must live in the
    heap at the same offset on every rank; it is allocated when not given (the returned tensor keeps its heap buffer
    alive) and may be `residual` itself (in-place update).  `out` [M, H] bf16 is an ordinary CUDA tensor, allocated
    when not given.  Needs H % 8 == 0, 8 <= H <= 16384, M >= 1.  Every rank gets the same bits.
    The sum is rounded to bf16 once, before the norm; matmul + all_reduce + add + rms_norm rounds twice (the
    all-reduce result, then its sum with the residual), so its residual stream can differ in the last bit.
    The kernel is one-shot (every rank pulls every row of every peer) while M H 2 P <= the "oneshot_max_bytes" tuning
    knob, two-shot above it (each rank reduces M / P rows and pushes them into every peer's residual_out); both give
    the same bits.  Stream ordered.
    `status`, optional 1-element int32 CUDA tensor, receives the error bits when the kernel ends (0: success); with
    non-zero bits the results are not valid.  An x or residual_out at a different heap offset on some peer sets
    DMA_MISMATCH_ERROR (bit 0) on both ranks, and neither reads or writes the other's heap.
    Raises ValueError, before anything is enqueued, for a wrong dtype, shape, device or alignment, an x or
    residual_out outside the heap, overlapping tensors (other than residual_out being residual), or a bad eps."""
    op = "all_reduce_rmsnorm"
    if not isinstance(x, torch.Tensor) or not accl.heap_contains(x):
        raise ValueError(f"{op}: x must live in the symmetric heap (a Buffer.dev view or a heap_mem_pool tensor)")
    device = x.device
    _check_operand(op, "x", x, device)
    M, H = x.shape
    if M < 1 or H % 8 or not 8 <= H <= AR_RMSNORM_MAX_H:
        raise ValueError(f"{op}: need M >= 1, H % 8 == 0 and 8 <= H <= {AR_RMSNORM_MAX_H}; got M = {M}, H = {H}")
    if not (isinstance(weight, torch.Tensor) and weight.device == device and weight.dtype == torch.bfloat16 and
            tuple(weight.shape) == (H,) and weight.is_contiguous()):
        raise ValueError(f"{op}: weight must be a contiguous bf16 tensor of shape ({H},) on {device}")
    eps = float(eps)
    if not (eps >= 0.0 and eps < float("inf")):
        raise ValueError(f"{op}: eps must be finite and non-negative, got {eps}")
    for name, t in (("residual", residual), ("residual_out", residual_out), ("out", out)):
        if t is not None:
            _check_operand(op, name, t, device)
            if tuple(t.shape) != (M, H):
                raise ValueError(f"{op}: {name} must be [{M}, {H}], got {tuple(t.shape)}")
    if residual_out is not None and not accl.heap_contains(residual_out):
        raise ValueError(f"{op}: residual_out must live in the symmetric heap (a Buffer.dev view or a heap_mem_pool tensor)")
    if residual_out is not None and (_overlap(residual_out, x) or (
            residual is not None and _overlap(residual_out, residual) and residual_out.data_ptr() != residual.data_ptr())):
        raise ValueError(f"{op}: residual_out must not overlap x, and may overlap residual only by being the same tensor")
    if out is not None and any(t is not None and _overlap(out, t) for t in (x, residual, residual_out, weight)):
        raise ValueError(f"{op}: out must not overlap x, residual, residual_out or weight")
    if any(t is not None and t.data_ptr() % 16 for t in (x, weight, residual, residual_out, out)):
        raise ValueError(f"{op}: every tensor must start at a 16-byte aligned address")
    status_ptr = _status_ptr(op, status, device)
    if residual_out is None:
        buf = accl.create_buffer(M * H, torch.bfloat16)
        residual_out = buf.dev.view(M, H)
        residual_out._accl_buffer = buf
    if out is None:
        out = torch.empty(M, H, dtype=torch.bfloat16, device=device)
    _C.all_reduce_rmsnorm(accl.impl, accl.wrap_device(x).impl, residual.data_ptr() if residual is not None else 0,
                          weight.data_ptr(), accl.wrap_device(residual_out).impl, out.data_ptr(), M, H, eps, status_ptr,
                          _stream_handle(accl))
    return out, residual_out


def vadd_allreduce(accl: Accl, x: Buffer, y: Buffer, out: Buffer, tmp: Buffer = None, count: int = None,
                   chunk_elems: int = 0):
    """out = allreduce_sum(x + y) (fp32), produced and reduced in chunks of `chunk_elems` (0: 1 Mi elements).
    Returns a 1-element int32 CUDA tensor that receives the engine's status word (0 = success) once the kernel
    has finished."""
    count = x.length if count is None else count
    if tmp is None:
        tmp = accl.create_buffer(count, torch.float32)
    status = torch.full((1,), -1, dtype=torch.int32, device=torch.device("cuda", accl.cuda_device))
    _C.vadd_allreduce(accl.impl, x.impl, y.impl, tmp.impl, out.impl, count, status.data_ptr(), _stream_handle(accl),
                      chunk_elems)
    status._keep = tmp
    return status


def vadd_put(accl: Accl, src: Buffer, count: int, dst_rank: int, stream_id: int = 9):
    """The reference's vadd_put user kernel: src + 1 (fp32) is pushed tile by tile into stream `stream_id` of rank
    `dst_rank` while it is being computed (device::Data::push).  Returns the status tensor."""
    status = torch.full((1,), -1, dtype=torch.int32, device=torch.device("cuda", accl.cuda_device))
    _C.vadd_put(accl.impl, src.impl, count, dst_rank, stream_id, status.data_ptr(), _stream_handle(accl))
    return status


def stream_pull(accl: Accl, dst: Buffer, count: int, stream_id: int = 9):
    """Drain `count` fp32 of stream `stream_id` of this rank into `dst` (device::Data::pull).  Returns the status tensor."""
    status = torch.full((1,), -1, dtype=torch.int32, device=torch.device("cuda", accl.cuda_device))
    _C.stream_pull(accl.impl, dst.impl, count, stream_id, status.data_ptr(), _stream_handle(accl))
    return status


def stream_loopback(accl: Accl, count: int, add_one: bool = False, scratch: Buffer = None):
    """Run the loopback user kernel on this rank's stream port: pull `count` fp32 words that a previous
    `copy_to_stream` / `recv_to_stream` / `RES_STREAM` op produced, optionally add one, push them back for a
    following `copy_from_stream` / `send_from_stream` / `OP0_STREAM` op (reference
    kernels/plugins/loopback, test/host/hls_simulator/test.cpp:153).  Returns the status tensor."""
    if scratch is None:
        scratch = accl.create_buffer(count, torch.float32)
    status = torch.full((1,), -1, dtype=torch.int32, device=torch.device("cuda", accl.cuda_device))
    _C.stream_loopback(accl.impl, scratch.impl, count, add_one, status.data_ptr(), _stream_handle(accl))
    status._keep = scratch
    return status
