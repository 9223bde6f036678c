"""Host-side mirror of the reference's quantised-linear modules on this repository's kernels.

Same class names, constructor arguments, buffer names / shapes / dtypes, `from_linear` signature and
forward semantics as awq/modules/linear/{gemm.py:116-298, gemv.py:27-197, gemv_fast.py:68-208}, so the
parity tests read like tests of the reference and a checkpoint's state-dict loads unchanged.  The
reference's own (unmodified) classes work on top of `awq_ext` / `awq_v2_ext` too - that is the real
drop-in point; these mirrors exist because the reference package need not be installed where the kernels run, and because
they skip the reference's "dequantise the whole matrix then cuBLAS" detour for >= 1024 tokens
(gemm.py:48-54): one fused wgmma kernel covers every M.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import ext
from .packing import (
    calculate_zeros_width,
    pack_gemm,
    pack_gemv,
    pack_gemv_fast,
    quantize_to_int,
)

__all__ = ["WQLinear_GEMM", "WQLinear_GEMV", "WQLinear_GEMVFast", "WQLinearMMFunction", "calculate_zeros_width"]


class WQLinearMMFunction(torch.autograd.Function):
    """Forward = fused W4A16 kernel; backward = dX only, through the dequantised weights
    (the reference's contract, gemm.py:24-114: no weight gradient)."""

    @staticmethod
    def forward(ctx, x, qweight, qzeros, scales, w_bit=4, group_size=128, bias=None, out_features=0):
        ctx.save_for_backward(x, qweight, qzeros, scales, bias)
        ctx.out_features = out_features
        out_shape = x.shape[:-1] + (out_features,)
        x = x.to(torch.float16)
        if x.shape[0] == 0:  # gemm.py:44-45
            return torch.zeros(out_shape, dtype=x.dtype, device=x.device)
        out = ext.linear_forward("gemm", x, qweight, scales, qzeros, group_size, bias)
        out = out.reshape(out_shape)
        if out.dim() == 2:  # gemm.py:83-84: always hand back a 3-D tensor
            out = out.unsqueeze(0)
        return out

    @staticmethod
    def backward(ctx, grad_output):
        x, qweight, qzeros, scales, bias = ctx.saved_tensors
        weights = ext.dequantize_weights_cuda(qweight, scales, qzeros, 1, 0, 0, False).to(grad_output.dtype)
        grad_input = None
        if ctx.needs_input_grad[0]:
            grad_input = torch.matmul(grad_output, weights.t())
        return grad_input, None, None, None, None, None, None, None


def _check_bits(w_bit):
    if w_bit not in [4]:
        raise NotImplementedError("Only 4-bit are supported for now.")


class WQLinear_GEMM(nn.Module):
    def __init__(self, w_bit, group_size, in_features, out_features, bias, dev, training=False):
        super().__init__()
        _check_bits(w_bit)
        self.in_features = in_features
        self.out_features = out_features
        self.w_bit = w_bit
        self.group_size = group_size if group_size != -1 else in_features
        self.training = training
        assert self.in_features % self.group_size == 0
        assert out_features % (32 // self.w_bit) == 0
        pack = 32 // self.w_bit
        self.register_buffer("qweight", torch.zeros((in_features, out_features // pack), dtype=torch.int32, device=dev))
        self.register_buffer(
            "qzeros", torch.zeros((in_features // self.group_size, out_features // pack), dtype=torch.int32, device=dev)
        )
        self.register_buffer(
            "scales", torch.zeros((in_features // self.group_size, out_features), dtype=torch.float16, device=dev)
        )
        if bias:
            self.register_buffer("bias", torch.zeros((out_features), dtype=torch.float16, device=dev))
        else:
            self.bias = None

    @classmethod
    def from_linear(cls, linear, w_bit, group_size, init_only=False, scales=None, zeros=None):
        """scales / zeros: [K/G, N] as the reference's quantiser passes them for GEMM (quantizer.py:236-240)."""
        m = cls(w_bit, group_size, linear.in_features, linear.out_features, linear.bias is not None,
                linear.weight.device)
        if init_only:
            return m
        assert scales is not None and zeros is not None
        s_ng, z_ng = scales.t().contiguous(), zeros.t().contiguous()
        iw = quantize_to_int(linear.weight.data, s_ng, z_ng, m.group_size)
        m.qweight, m.qzeros, m.scales = pack_gemm(iw, z_ng, s_ng)
        if linear.bias is not None:
            m.bias = linear.bias.clone().half()
        return m

    def forward(self, x):
        out_shape = x.shape[:-1] + (self.out_features,)
        input_dtype = x.dtype
        if input_dtype != torch.float16:
            x = x.half()
        args = (x, self.qweight, self.qzeros, self.scales, self.w_bit, self.group_size, self.bias, self.out_features)
        if self.training:
            out = WQLinearMMFunction.apply(*args)
        else:
            with torch.no_grad():
                out = WQLinearMMFunction.apply(*args)
        if input_dtype != torch.float16:
            out = out.to(dtype=input_dtype)
        return out.reshape(out_shape)

    def extra_repr(self) -> str:
        return "in_features={}, out_features={}, bias={}, w_bit={}, group_size={}".format(
            self.in_features, self.out_features, self.bias is not None, self.w_bit, self.group_size
        )


class WQLinear_GEMV(nn.Module):
    def __init__(self, w_bit, group_size, in_features, out_features, bias, dev):
        super().__init__()
        _check_bits(w_bit)
        self.in_features = in_features
        self.out_features = out_features
        self.w_bit = w_bit
        self.group_size = group_size if group_size != -1 else in_features
        self.split_k_iters = 8  # read by fuse_qkv (awq/utils/fused_utils.py:86)
        assert self.in_features % self.group_size == 0
        assert out_features % (32 // self.w_bit) == 0
        pack = 32 // self.w_bit
        zw = calculate_zeros_width(in_features, self.group_size)
        self.register_buffer("qweight", torch.zeros((out_features, in_features // pack), dtype=torch.int32, device=dev))
        self.register_buffer("qzeros", torch.zeros((out_features, zw), dtype=torch.int32, device=dev))
        self.register_buffer("scales", torch.zeros((out_features, zw * pack), dtype=torch.float16, device=dev))
        if bias:
            self.register_buffer("bias", torch.zeros((out_features), dtype=torch.float16, device=dev))
        else:
            self.bias = None

    @classmethod
    def from_linear(cls, linear, w_bit, group_size, init_only=False, scales=None, zeros=None):
        """scales / zeros: [N, K/G] (the quantiser's native orientation, gemv.py:78-94)."""
        m = cls(w_bit, group_size, linear.in_features, linear.out_features, linear.bias is not None,
                linear.weight.device)
        if init_only:
            return m
        assert scales is not None and zeros is not None
        iw = quantize_to_int(linear.weight.data, scales, zeros, m.group_size)
        m.qweight, m.qzeros, m.scales = pack_gemv(iw, zeros, scales, m.group_size)
        if linear.bias is not None:
            m.bias = linear.bias.clone().half()
        return m

    @torch.no_grad()
    def forward(self, x):
        out_shape = x.shape[:-1] + (self.out_features,)
        inputs = x.reshape(-1, x.shape[-1])
        input_dtype = inputs.dtype
        if input_dtype != torch.float16:
            inputs = inputs.half()
        out = ext.linear_forward("gemv", inputs, self.qweight, self.scales, self.qzeros, self.group_size)
        if input_dtype != torch.float16:
            out = out.to(dtype=input_dtype)
        out = out + self.bias if self.bias is not None else out  # bias after the cast back (gemv.py:182-185)
        return out.reshape(out_shape)

    def extra_repr(self) -> str:
        return "in_features={}, out_features={}, bias={}, w_bit={}, group_size={}".format(
            self.in_features, self.out_features, self.bias is not None, self.w_bit, self.group_size
        )


class WQLinear_GEMVFast(nn.Module):
    def __init__(self, w_bit, group_size, in_features, out_features, bias, dev):
        super().__init__()
        self.in_features = in_features
        self.out_features = out_features
        self.w_bit = w_bit
        self.group_size = group_size if group_size != -1 else in_features
        self.split_k_iters = 8
        self.interleave = 4
        assert self.in_features % self.group_size == 0
        assert out_features % (32 // self.w_bit) == 0
        assert out_features % self.interleave == 0
        pack = 32 // self.w_bit
        int16_pack = 16 // self.w_bit
        zw = calculate_zeros_width(in_features, self.group_size)
        self.register_buffer(
            "qweight",
            torch.zeros((out_features // self.interleave, in_features // int16_pack * self.interleave),
                        dtype=torch.int16, device=dev),
        )
        self.register_buffer("scales", torch.zeros((zw * pack, out_features), dtype=torch.float16, device=dev))
        self.register_buffer("qzeros", torch.zeros((zw * pack, out_features), dtype=torch.float16, device=dev))
        if bias:
            self.register_buffer("bias", torch.zeros((out_features), dtype=torch.float16, device=dev))
        else:
            self.bias = None

    @classmethod
    def from_linear(cls, linear, w_bit, group_size, init_only=False, scales=None, zeros=None):
        m = cls(w_bit, group_size, linear.in_features, linear.out_features, linear.bias is not None,
                linear.weight.device)
        if init_only:
            return m
        assert scales is not None and zeros is not None
        iw = quantize_to_int(linear.weight.data, scales, zeros, m.group_size)
        m.qweight, m.scales, m.qzeros = pack_gemv_fast(iw, zeros, scales, m.group_size)
        if linear.bias is not None:
            m.bias = linear.bias.clone().half()
        return m

    @torch.no_grad()
    def forward(self, x):
        batch_size, n_tokens, _ = x.shape  # requires a 3-D input, as the reference (gemv_fast.py:190)
        out = ext.linear_forward("fast", x, self.qweight, self.scales, self.qzeros, self.group_size)
        out = out.reshape(batch_size, n_tokens, self.out_features)
        return out + self.bias if self.bias is not None else out
