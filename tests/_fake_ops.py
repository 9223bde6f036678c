"""Decode-program op lists over fake device addresses, for b200awq_program_plan: program_create's folding for a given SM
count, without any CUDA call.  The folding only compares addresses, so aligned integers stand in for tensors.

An op is a dict of b200awq_op_t fields; `plan` turns a list of them into the C array.  Buffers come from one allocator
for the whole session, so two buffers alias only where a test makes them."""
import ctypes

from autoawq_b200 import _cabi
from autoawq_b200._cabi import lib

_next = [0x10000000]


def buf(nbytes=1 << 16):
    """A fresh 64 KiB-aligned placeholder address with room for `nbytes`."""
    p = _next[0]
    _next[0] += (max(nbytes, 1) + 0xffff) & ~0xffff
    return p


def _out(y, nbytes):
    return buf(nbytes) if y is None else y


def linear(x, K, N, M=1, y=None, ldx=None):
    return dict(kind=_cabi.OP_LINEAR_GEMM, M=M, K=K, N=N, group_size=128, ldx=K if ldx is None else ldx, x=x,
                qweight=buf(K * N // 2), scales=buf(K // 128 * N * 2), qzeros=buf(K // 128 * N // 2),
                y=_out(y, M * N * 2))


def rmsnorm(x, K, M=1, eps=1e-5, y=None, ldx=0):
    return dict(kind=_cabi.OP_RMSNORM, M=M, K=K, eps=eps, ldx=ldx, x=x, weight=buf(K * 2), y=_out(y, M * K * 2))


def add(a, b, K, M=1, y=None):
    return dict(kind=_cabi.OP_ADD, M=M, K=K, x=a, weight=b, y=_out(y, M * K * 2))


def silu(gu, K, M=1, y=None):
    return dict(kind=_cabi.OP_SILU_AND_MUL, M=M, K=K, x=gu, y=_out(y, M * K * 2))


def plan(ops, max_tokens=1, sms=132):
    """(return code, kernel ops) of b200awq_program_plan on the op dicts."""
    arr = (_cabi.Op * len(ops))()
    for c, o in zip(arr, ops):
        for f, v in o.items():
            setattr(c, f, v)
    n = ctypes.c_int(-1)
    rc = lib.b200awq_program_plan(arr, len(ops), max_tokens, sms, 0, ctypes.byref(n))
    return rc, n.value
