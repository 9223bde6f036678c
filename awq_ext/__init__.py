"""Drop-in `awq_ext` for casper-hansen/AutoAWQ: the reference discovers its kernels with
importlib.import_module("awq_ext") (awq/utils/module.py:4-9; awq/modules/linear/gemm.py:11,
gemv.py:6, awq/modules/fused/norm.py:5, mlp.py:7, moe.py:5, awq/models/base.py:538).  Putting this
package on sys.path before `import awq` routes those call sites to this repository's kernels.
Raises at import when libb200awq.so is missing: there is no CPU fallback."""
from autoawq_b200.ext import (  # noqa: F401
    dequantize_weights_cuda,
    gemm_forward_cuda,
    gemmv2_forward_cuda,
    gemv_forward_cuda,
    grouped_gemm_forward,
    layernorm_forward_cuda,
    moe_alig_block_size,
    silu_and_mul,
    topk_softmax,
)
