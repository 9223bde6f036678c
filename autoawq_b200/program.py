"""Decode programs: record the awq_ext-facing operator calls of one decode step, run them as ONE persistent
kernel (csrc/program.cu, C ABI b200awq_program_*).

The recorder exposes the same call names and argument order as `awq_ext` (`layernorm_forward_cuda`,
`gemm_forward_cuda`, `silu_and_mul` - call sites awq/modules/fused/norm.py:33-36, fused/mlp.py:41-55,
fused/moe.py:76), so the code that drives a fused block (awq/modules/fused/block.py:117-170) can be pointed at
a `DecodeProgram` once, and `run()` replays it every token:

    prog = DecodeProgram()
    prog.layernorm_forward_cuda(h, w_norm, xn, eps)      # buffers are captured by address: refill h in place
    qkv = prog.gemm_forward_cuda(xn, qweight, scales, qzeros, 8)
    ...
    prog.build()
    prog.run()                               # one memset + one kernel on torch's current stream

If the sequence does not fit the fused kernel (M != 1, unsupported shape, aliasing) `build()` keeps the op list and
`run()` issues the per-op entry points instead - still the CUDA path, `prog.fused` tells which.

A fused block built for batch size B (every call has B rows) is fused when the program is created with
`DecodeProgram(max_tokens=B)`, B <= 8: one persistent kernel then runs all B tokens (csrc/program_batch.cuh), each
bit-identical to an M = 1 program on that token's row.  Without it, M > 1 replays the per-op kernels as before.
"""
from __future__ import annotations

import ctypes

import torch

from . import _cabi, ext
from ._cabi import B200AwqError, Op, check, lib


class DecodeProgram:
    def __init__(self, max_tokens: int = 1):
        if not 1 <= int(max_tokens) <= 8:
            raise B200AwqError("b200awq: max_tokens must be in 1..8")
        self.max_tokens = int(max_tokens)  # > 1: build() may fuse a sequence recorded with up to this many rows per op
        self._ops: list = []          # (kind, dict of tensors / scalars)
        self._keep: list = []         # every tensor named by an op stays alive with the program
        self._handle = None
        self._built = False
        self._max_n = 0
        self._dev = None
        self.calibration = None       # {"stream_ms", "splitk_ms"} when build() timed both kernels

    # ------------------------------------------------------------------ recording (awq_ext call names)
    def _dev_of(self, t: torch.Tensor):
        ext._require_cuda(t)
        if self._dev is None:
            self._dev = t.device
        elif t.device != self._dev:
            raise B200AwqError("b200awq: a decode program lives on one device")

    def _no_more(self):
        if self._built:
            raise B200AwqError("b200awq: program already built")

    def layernorm_forward_cuda(self, x, weight, out, eps):
        self._no_more()
        self._dev_of(x)
        if x.dtype != torch.float16 or weight.dtype != torch.float16 or out.dtype != torch.float16:
            raise B200AwqError("b200awq: rmsnorm expects float16 tensors")
        if not x.is_contiguous() or not out.is_contiguous() or not weight.is_contiguous():
            raise B200AwqError("b200awq: program rmsnorm expects contiguous tensors")
        hidden = x.shape[-1]
        self._ops.append(("rmsnorm", dict(x=x, weight=weight, out=out, eps=float(eps), rows=x.numel() // hidden,
                                          hidden=hidden)))
        self._keep += [x, weight, out]

    def silu_and_mul(self, out, gate_up):
        self._no_more()
        self._dev_of(out)
        d = out.shape[-1]
        if gate_up.shape[-1] != 2 * d or not gate_up.is_contiguous() or not out.is_contiguous():
            raise B200AwqError("b200awq: silu_and_mul expects contiguous [.., 2d] -> [.., d]")
        self._ops.append(("silu", dict(out=out, gate_up=gate_up, rows=out.numel() // d, d=d)))
        self._keep += [out, gate_up]

    def gemm_forward_cuda(self, x, qweight, scales, qzeros, split_k_iters=8, bias=None):
        self._no_more()
        self._dev_of(x)
        ext._check_w(qweight, torch.int32, "qweight")
        ext._check_w(scales, torch.float16, "scales")
        ext._check_w(qzeros, torch.int32, "qzeros")
        K, N = qweight.shape[0], qweight.shape[1] * 8
        G = K // scales.shape[0]
        x2 = ext._x2d(x, K)
        if x2.data_ptr() != x.data_ptr():
            raise B200AwqError("b200awq: program inputs must be 16-byte aligned rows with unit stride (no copies "
                               "can be recorded)")
        M = x2.shape[0]
        y = torch.empty((M, N), dtype=torch.float16, device=x.device)
        self._ops.append(("linear", dict(x=x2, qweight=qweight, scales=scales, qzeros=qzeros, bias=bias, y=y, M=M, K=K,
                                         N=N, G=G, ldx=x2.stride(0) if M > 1 else K)))
        self._keep += [x, x2, qweight, scales, qzeros, y] + ([bias] if bias is not None else [])
        self._max_n = max(self._max_n, N)
        return y.reshape(x.shape[:-1] + (N,))

    # ------------------------------------------------------------------ build / run
    def _c_ops(self):
        arr = (Op * len(self._ops))()
        for i, (kind, o) in enumerate(self._ops):
            c = arr[i]
            if kind == "rmsnorm":
                c.kind, c.M, c.K, c.eps = _cabi.OP_RMSNORM, o["rows"], o["hidden"], o["eps"]
                c.x, c.weight, c.y = o["x"].data_ptr(), o["weight"].data_ptr(), o["out"].data_ptr()
            elif kind == "silu":
                c.kind, c.M, c.K = _cabi.OP_SILU_AND_MUL, o["rows"], o["d"]
                c.x, c.y = o["gate_up"].data_ptr(), o["out"].data_ptr()
            else:
                c.kind, c.M, c.K, c.N, c.group_size, c.ldx = _cabi.OP_LINEAR_GEMM, o["M"], o["K"], o["N"], o["G"], o["ldx"]
                c.x, c.qweight, c.scales, c.qzeros = (o["x"].data_ptr(), o["qweight"].data_ptr(), o["scales"].data_ptr(),
                                                      o["qzeros"].data_ptr())
                c.bias = o["bias"].data_ptr() if o["bias"] is not None else None
                c.y = o["y"].data_ptr()
        return arr

    def _create(self, arr, kind_knob: int):
        """b200awq_program_create (b200awq_program_create_batched when max_tokens > 1) under knob 14 = kind_knob;
        returns a handle or None (sequence outside that kernel)."""
        prev = lib.b200awq_get_knob(14)
        lib.b200awq_set_knob(14, kind_knob)
        try:
            handle = ctypes.c_void_p()
            with ext._DeviceGuard(self._dev):
                if self.max_tokens > 1:
                    code = lib.b200awq_program_create_batched(arr, len(self._ops), self.max_tokens, ctypes.byref(handle))
                else:
                    code = lib.b200awq_program_create(arr, len(self._ops), ctypes.byref(handle))
        finally:
            lib.b200awq_set_knob(14, prev)
        if code == _cabi.EUNSUPPORTED:
            return None
        check(code, "b200awq_program_create")
        return handle

    def _time(self, handle, runs: int = 5) -> float:
        """Median device time (ms) of one run of `handle` on the current stream (load-time calibration)."""
        dev = self._dev
        with ext._DeviceGuard(dev):
            st = ext._stream(dev)
            ws = ext._workspace(dev, st, lib.b200awq_workspace_bytes(8, 0, (self._max_n + 7) & ~7))
            ts = []
            for i in range(runs + 2):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                check(lib.b200awq_program_run(handle, ws.data_ptr(), ws.numel(), st), "b200awq_program_run")
                e1.record()
                e1.synchronize()
                if i >= 2:
                    ts.append(e0.elapsed_time(e1))
        ts.sort()
        return ts[len(ts) // 2]

    def build(self, calibrate: bool = True) -> "DecodeProgram":
        """Fold the recorded calls into a fused program.  Two kernels can run it: the stream variant (one-time
        re-layout of the weights, output-stationary, csrc/program_stream.cuh) and the split-K kernel on the checkpoint
        layout (csrc/program.cu).  With `calibrate` (default) and knob 14 = 0, both are created when the sequence fits
        both, each is timed on the device (a load-time step, like the re-layout itself; the recorded buffers are
        overwritten by those runs exactly as `run()` would), and the faster one is kept - `calibration` holds the two
        times.  Knob 14 = 1 / 2 forces the split-K / stream kernel.  A sequence with M > 1 rows per op (max_tokens >= M)
        has only the batched stream kernel: nothing to calibrate."""
        self._no_more()
        if not self._ops:
            raise B200AwqError("b200awq: empty program")
        arr = self._c_ops()
        self.calibration = None
        forced = lib.b200awq_get_knob(14)
        if forced in (1, 2) or not calibrate:
            self._handle = self._create(arr, forced)
        else:
            hs, hk = self._create(arr, 2), self._create(arr, 1)
            if hs is not None and hk is not None:
                ts, tk = self._time(hs), self._time(hk)
                self.calibration = {"stream_ms": round(ts, 4), "splitk_ms": round(tk, 4)}
                keep, drop = (hs, hk) if ts <= tk else (hk, hs)
                lib.b200awq_program_destroy(drop)
                self._handle = keep
            else:
                self._handle = hs if hs is not None else hk      # None: per-op replay (still the CUDA path)
        self._built = True
        return self

    @property
    def fused(self) -> bool:
        return self._handle is not None

    @property
    def kind(self) -> str:
        """"stream" (re-laid-out weights, output-stationary kernel), "splitk" (round-1 kernel on the checkpoint
        layout) or "per-op"."""
        if self._handle is None:
            return "per-op"
        return "stream" if lib.b200awq_program_kind(self._handle) == 2 else "splitk"

    @property
    def tokens(self) -> int:
        """Token rows per run (M of the recorded ops; 0 before anything was recorded)."""
        if self._handle is not None:
            return lib.b200awq_program_tokens(self._handle)
        for kind, o in self._ops:
            return o["M"] if kind == "linear" else o["rows"]
        return 0

    @property
    def kernel_ops(self) -> int:
        return lib.b200awq_program_num_ops(self._handle) if self._handle is not None else 0

    @property
    def launches_per_run(self) -> int:
        """Kernels of this library launched by one run()."""
        return 1 if self.fused else len(self._ops)

    def run(self) -> None:
        if not self._built:
            raise B200AwqError("b200awq: build() the program first")
        dev = self._dev
        if self._handle is not None:
            with ext._DeviceGuard(dev):
                st = ext._stream(dev)
                ws = ext._workspace(dev, st, lib.b200awq_workspace_bytes(8, 0, (self._max_n + 7) & ~7))
                code = lib.b200awq_program_run(self._handle, ws.data_ptr(), ws.numel(), st)
            check(code, "b200awq_program_run")
            return
        for kind, o in self._ops:
            if kind == "rmsnorm":
                ext.layernorm_forward_cuda(o["x"], o["weight"], o["out"], o["eps"])
            elif kind == "silu":
                ext.silu_and_mul(o["out"], o["gate_up"])
            else:
                ext.linear_forward("gemm", o["x"], o["qweight"], o["scales"], o["qzeros"], o["G"], o["bias"], out=o["y"])

    @staticmethod
    def abort_record():
        """(code, op, cta, aborted) of the last fused run on this device: the kernel's spin loops give up after 0.5 s
        instead of hanging the GPU and record which wait failed (csrc/program.cu).  Synchronises the device."""
        import numpy as np

        prev = lib.b200awq_get_knob(3)
        lib.b200awq_set_knob(3, 3)
        buf = np.zeros(4, dtype=np.int32)
        try:
            check(lib.b200awq_debug_read(buf.ctypes.data_as(ctypes.c_void_p), buf.nbytes), "b200awq_debug_read")
        finally:
            lib.b200awq_set_knob(3, prev)
        return tuple(int(v) for v in buf)

    def close(self) -> None:
        if self._handle is not None:
            lib.b200awq_program_destroy(self._handle)
            self._handle = None
            self._built = False

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
