from .plugins import all_gather_gemm, all_reduce_rmsnorm, gemm_all_reduce, gemm_reduce_scatter, stream_loopback, stream_pull, vadd_allreduce, vadd_put  # noqa: F401
