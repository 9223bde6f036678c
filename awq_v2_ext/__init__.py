"""Drop-in `awq_v2_ext` (awq/modules/linear/gemv_fast.py:5,192-205) on this repository's kernels."""
from autoawq_b200.ext import gemm_forward_cuda_prefill, gemv_forward_cuda_decode  # noqa: F401
