"""The reference's CPU path, restated with the same torch operators, for TIMING ONLY
(bench.py `cpu_baseline` and `--impl reference`).  TEST/BENCH INFRASTRUCTURE - never imported by the
product packages.

What the reference executes on a CPU box (no awq_ext, no Triton, no IPEX):
WQLinearMMFunction.forward's naive branch, awq/modules/linear/gemm.py:71-77 (identical to
WQLinear_IPEX's fallback, awq/modules/linear/gemm_ipex.py:105-107): dequantize_gemm
(awq/utils/packing_utils.py:87-102) followed by torch.matmul in fp16, on every call.
The reference checkout is not available where the GPU runs, hence this port; its dequant is checked bit-for-bit
against the numpy oracle (tests/test_oracle_golden.py::test_torch_port_matches_oracle).
"""
from __future__ import annotations

import torch

_SHIFTS = torch.tensor([0, 16, 4, 20, 8, 24, 12, 28], dtype=torch.int32)  # 4 * AWQ_REVERSE_ORDER[j]


def dequantize(qweight: torch.Tensor, qzeros: torch.Tensor, scales: torch.Tensor, group_size: int) -> torch.Tensor:
    iw = ((qweight.unsqueeze(-1) >> _SHIFTS) & 0xF).to(torch.int8).reshape(qweight.shape[0], -1)
    iz = ((qzeros.unsqueeze(-1) >> _SHIFTS) & 0xF).to(torch.int8).reshape(qzeros.shape[0], -1)
    return (iw - iz.repeat_interleave(group_size, dim=0)) * scales.repeat_interleave(group_size, dim=0)


def wqlinear_forward(x: torch.Tensor, qweight, qzeros, scales, group_size: int, bias=None) -> torch.Tensor:
    w = dequantize(qweight, qzeros, scales, group_size)
    out = torch.matmul(x.to(torch.float16), w)
    return out + bias if bias is not None else out
