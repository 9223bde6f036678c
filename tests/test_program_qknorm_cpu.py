"""Host logic of Qwen3's q / k norm folded into decode programs (B200AWQ_OP_QK_NORM_ROPE_KV), checked without a GPU: the
ctypes descriptor layout, the exported entry point, the folding rules through b200awq_program_plan (ROPE_KV's rules on
the embedded descriptor, plus the norm weights) and the register / spill budget of the new kernel entries.

The plan sequences use fake (aligned integer) pointers: the folding only compares addresses.  Shapes are Qwen3-8B's
(hidden 4096, 32 q heads, 8 kv heads, head_dim 128, intermediate 12288)."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

from autoawq_b200 import _cabi
from autoawq_b200._cabi import lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, EINVAL, EUNSUPPORTED = 0, 1, 2
HID, INTER, H, KV, D, SMS = 4096, 12288, 32, 8, 128, 132
QKV = (H + 2 * KV) * D
S = 2048
_next = [0x30000000]
_KEEP = []


def _buf(nbytes=1 << 16):
    p = _next[0]
    _next[0] += (nbytes + 0xffff) & ~0xffff
    return p


def _lin(x, y=None, k=HID, n=HID, M=1):
    return dict(kind=_cabi.OP_LINEAR_GEMM, M=M, K=k, N=n, group_size=128, ldx=k, x=x, qweight=_buf(), scales=_buf(),
                qzeros=_buf(), y=y or _buf(M * n * 2))


def _norm(x, y=None, k=HID, M=1):
    return dict(kind=_cabi.OP_RMSNORM, M=M, K=k, x=x, weight=_buf(), y=y or _buf(), eps=1e-6)


def _add(a, b, y=None, k=HID, M=1):
    return dict(kind=_cabi.OP_ADD, M=M, K=k, x=a, weight=b, y=y or _buf())


def _silu(gu, y=None, k=INTER, M=1):
    return dict(kind=_cabi.OP_SILU_AND_MUL, M=M, K=k, x=gu, y=y or _buf())


def _qkn(qkv, M=1, n=QKV, heads=(H, KV, D), q_w=None, k_w=None, **over):
    """A QK_NORM_ROPE_KV op on qkv with its own q_out / caches / pos / freqs / norm weights; `over` replaces fields of
    the embedded rope descriptor."""
    h, kv, d = heads
    q = _cabi.QkNormRope()
    r = q.rope
    r.n_heads, r.n_kv_heads, r.head_dim, r.cache_len, r.freqs_len = h, kv, d, S, S
    r.cache_batch_stride = S * kv * d
    cache = 8 * S * kv * d * 2
    r.pos, r.freqs, r.q_out = _buf(), _buf(S * d * 4), _buf()
    r.k_cache, r.v_cache = _buf(cache), _buf(cache)
    for f, v in over.items():
        setattr(r, f, v)
    q.q_norm_weight = _buf() if q_w is None else q_w
    q.k_norm_weight = _buf() if k_w is None else k_w
    q.eps = 1e-6
    _KEEP.append(q)
    return dict(kind=_cabi.OP_QK_NORM_ROPE_KV, M=M, N=n, ldx=n, x=qkv, weight=ctypes.addressof(q)), q


def _plan(ops, max_tokens=1):
    arr = (_cabi.Op * len(ops))()
    for c, o in zip(arr, ops):
        for f, v in o.items():
            setattr(c, f, v)
    kops = ctypes.c_int(-1)
    code = lib.b200awq_program_plan(arr, len(ops), max_tokens, SMS, 0, ctypes.byref(kops))
    return code, kops.value


def _segment(M=1, hid=HID):
    """[o + h, norm2, gate|up, silu, down + h, norm1', qkv', qk-norm-rope'] of a Qwen3 layer (hidden `hid`)."""
    attn, h_in = _buf(), _buf()
    o = _lin(attn, k=H * D, n=hid, M=M)
    h = _add(o["y"], h_in, k=hid, M=M)
    n2 = _norm(h["y"], k=hid, M=M)
    gu = _lin(n2["y"], k=hid, n=2 * INTER, M=M)
    act = _silu(gu["y"], M=M)
    dn = _lin(act["y"], k=INTER, n=hid, M=M)
    out = _add(dn["y"], h["y"], k=hid, M=M)
    n1 = _norm(out["y"], k=hid, M=M)
    qkv = _lin(n1["y"], k=hid, n=QKV, M=M)
    qk, q = _qkn(qkv["y"], M=M)
    return [o, h, n2, gu, act, dn, out, n1, qkv, qk], q


def test_struct_matches_header(tmp_path):
    src = tmp_path / "k.c"
    fields = [f for f, _ in _cabi.QkNormRope._fields_]
    body = " ".join(f'printf("%zu ", offsetof(b200awq_qk_norm_rope_t, {f}));' for f in fields)
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200awq.h"\nint main(void) { ' + body +
                   ' printf("%zu %zu %d %d", sizeof(b200awq_qk_norm_rope_t), sizeof(b200awq_rope_t), '
                   'B200AWQ_OP_QK_NORM_ROPE_KV, B200AWQ_OP_ROPE_KV); return 0; }\n')
    exe = tmp_path / "k"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert got[:len(fields)] == [getattr(_cabi.QkNormRope, f).offset for f in fields]
    assert got[len(fields)] == ctypes.sizeof(_cabi.QkNormRope)
    assert got[len(fields) + 1] == ctypes.sizeof(_cabi.Rope) == 72      # the embedded descriptor is unchanged
    assert got[-2:] == [_cabi.OP_QK_NORM_ROPE_KV, _cabi.OP_ROPE_KV] == [7, 6]


def test_entry_point_is_exported():
    assert "b200awq_qk_norm_rope_kv" in _cabi.SIGNATURES
    fn = getattr(lib, "b200awq_qk_norm_rope_kv")
    assert fn.restype is ctypes.c_int
    # argument checks happen before any CUDA call: a null descriptor / qkv is EINVAL, M = 0 with a valid one is a no-op
    assert fn(None, QKV, None, 1, None) == EINVAL
    _, q = _qkn(_buf())
    assert fn(None, QKV, q, 1, None) == EINVAL
    assert fn(_buf(), QKV, q, 0, None) == OK
    for field in ("q_norm_weight", "k_norm_weight"):
        bad = _cabi.QkNormRope.from_buffer_copy(q)
        setattr(bad, field, 0)
        assert fn(_buf(), QKV, bad, 1, None) == EINVAL, field
    _, q72 = _qkn(_buf(), n=(H + 2 * KV) * 72, heads=(H, KV, 72))
    assert fn(_buf(), (H + 2 * KV) * 72, q72, 1, None) == EUNSUPPORTED       # the summation order needs D % 16 == 0


def test_folds_without_adding_kernel_ops():
    x = _buf()
    n1 = _norm(x)
    qkv = _lin(n1["y"], n=QKV)
    qk, _ = _qkn(qkv["y"])
    assert _plan([n1, qkv]) == (OK, 1)
    assert _plan([n1, qkv, qk]) == (OK, 1)
    for M in (1, 2, 4):
        seg, _ = _segment(M)
        assert _plan(seg, max_tokens=M) == (OK, 4), M
        assert _plan(seg[:-1], max_tokens=M) == (OK, 4), M
    seg, _ = _segment(hid=2560)                      # Qwen3-4B: hidden 2560 != H D = 4096
    assert _plan(seg) == (OK, 4)
    o = _lin(qkv["y"], k=HID)                        # a later linear may read the raw qkv
    assert _plan([n1, qkv, qk, o]) == (OK, 2)


def test_argument_validation():
    qkv = _lin(_buf(), n=QKV)
    qk, _ = _qkn(qkv["y"])
    for field in ("pos", "freqs", "q_out", "k_cache", "v_cache"):
        bad, _ = _qkn(qkv["y"], **{field: 0})
        assert _plan([qkv, bad])[0] == EINVAL, field
    for over in (dict(q_w=0), dict(k_w=0)):
        bad, _ = _qkn(qkv["y"], **over)
        assert _plan([qkv, bad])[0] == EINVAL, over
    assert _plan([qkv, dict(qk, x=0)])[0] == EINVAL
    assert _plan([qkv, dict(qk, weight=0)])[0] == EINVAL
    for over in (dict(head_dim=127), dict(n_heads=0), dict(cache_len=0), dict(cache_batch_stride=S * KV * D - 1)):
        bad, _ = _qkn(qkv["y"], **over)
        assert _plan([qkv, bad])[0] == EINVAL, over
    for over in (dict(q_w=_buf() + 8), dict(k_w=_buf() + 2)):          # misaligned norm weights
        bad, _ = _qkn(qkv["y"], **over)
        assert _plan([qkv, bad])[0] == EUNSUPPORTED, over


def test_rejected_after_anything_but_a_plain_linear():
    x, r = _buf(), _buf()
    n1 = _norm(x, k=QKV)
    qk, _ = _qkn(n1["y"])
    assert _plan([n1, qk, _lin(n1["y"], k=QKV)])[0] == EUNSUPPORTED            # after a glue op
    qkv = _lin(x, n=QKV)
    a = _add(qkv["y"], r, k=QKV)
    qk, _ = _qkn(a["y"])
    assert _plan([qkv, a, qk])[0] == EUNSUPPORTED                              # after an add
    qkv = _lin(x, n=QKV)
    qk, _ = _qkn(qkv["y"])
    qk2, _ = _qkn(qkv["y"])
    assert _plan([qkv, qk, qk2])[0] == EUNSUPPORTED                            # after another rope op
    assert _plan([qk])[0] == EUNSUPPORTED                                      # first op
    gu = _lin(x, n=QKV)                                                        # a gate|up whose product SiLU*mul reads
    qk, _ = _qkn(gu["y"])
    act = _silu(gu["y"], k=QKV // 2)
    assert _plan([gu, qk, act, _lin(act["y"], k=QKV // 2)])[0] == EUNSUPPORTED
    E, k, Hm, Im = 8, 2, QKV, 512                                              # a sparse-MoE block's down op
    d = _cabi.Moe()
    d.E, d.top_k, d.renormalize, d.group_size, d.H, d.I, d.block_size = E, k, 1, 128, Hm, Im, 16
    d.sorted_len = k + E * 15
    d.gate_weight = _buf()
    for f, _ in _cabi.Moe._fields_[9:]:
        setattr(d, f, _buf())
    _KEEP.append(d)
    xn = _norm(x, k=Hm)
    moe = dict(kind=_cabi.OP_SPARSE_MOE, M=1, K=Hm, N=Hm, x=xn["y"], y=_buf(), weight=ctypes.addressof(d))
    qk, _ = _qkn(moe["y"])
    assert _plan([xn, moe])[0] == OK
    assert _plan([xn, moe, qk])[0] == EUNSUPPORTED


def test_rejected_when_qkv_is_not_the_whole_output_or_the_shape_is_off():
    x = _buf()
    qkv = _lin(x, n=QKV)
    qk, _ = _qkn(qkv["y"] + 256, n=QKV - 128)
    assert _plan([qkv, qk])[0] == EUNSUPPORTED                                 # a slice of the linear's output
    qk, _ = _qkn(_buf())
    assert _plan([qkv, qk])[0] == EUNSUPPORTED                                 # not the linear's output at all
    wide = _lin(x, n=QKV + 128)
    qk, _ = _qkn(wide["y"], n=QKV + 128)
    assert _plan([wide, qk])[0] == EUNSUPPORTED                                # N != (H + 2 KV) D
    d72 = (H + 2 * KV) * 72
    q72 = _lin(x, n=d72)
    qk, _ = _qkn(q72["y"], n=d72, heads=(H, KV, 72))
    assert _plan([q72, qk])[0] == EUNSUPPORTED                                 # D % 16 != 0
    d64 = (H + 2 * KV) * 64
    q64 = _lin(x, n=d64)
    qk, _ = _qkn(q64["y"], n=d64, heads=(H, KV, 64))
    assert _plan([q64, qk])[0] == OK


def test_rejected_when_another_op_touches_its_outputs_or_writes_its_inputs():
    x = _buf()
    for field in ("q_out", "k_cache", "v_cache"):
        n1 = _norm(x)
        qkv = _lin(n1["y"], n=QKV)
        qk, q = _qkn(qkv["y"])
        target = getattr(q.rope, field)
        assert _plan([n1, qkv, qk, _lin(target, k=HID)])[0] == EUNSUPPORTED, field           # a later linear reads it
        assert _plan([n1, qkv, qk, _lin(_buf(), y=target, k=HID)])[0] == EUNSUPPORTED, field  # ... writes it
        assert _plan([_norm(_buf(), y=target), _lin(target, k=HID), n1, qkv, qk])[0] == EUNSUPPORTED, field
        o = _lin(_buf())
        assert _plan([n1, qkv, qk, o, _add(o["y"], target)])[0] == EUNSUPPORTED, field
        n1b = _norm(_buf())
        qkv_b = _lin(n1b["y"], n=QKV)
        qk_b, _ = _qkn(qkv_b["y"], **{field: target})                          # a second op writes into it
        assert _plan([n1, qkv, qk, n1b, qkv_b, qk_b])[0] == EUNSUPPORTED, field
        qk_ip, _ = _qkn(qkv["y"], **{field: qkv["y"]})                        # the qkv linear's own output
        assert _plan([n1, qkv, qk_ip])[0] == EUNSUPPORTED, field
    for field in ("q_norm_weight", "k_norm_weight", "pos"):
        n1 = _norm(x)
        qkv = _lin(n1["y"], n=QKV)
        qk, q = _qkn(qkv["y"])
        target = getattr(q, field) if field != "pos" else q.rope.pos
        assert _plan([n1, qkv, qk, _lin(_buf(), y=target)])[0] == EUNSUPPORTED, field       # a program op writes it
        assert _plan([_lin(_buf(), y=target), n1, qkv, qk])[0] == EUNSUPPORTED, field
        assert _plan([n1, qkv, qk, _lin(target, k=HID)])[0] == OK, field                    # reading it is fine
    # the q_out of one layer's op as the next layer's norm weight: a write of a read
    n1 = _norm(x)
    qkv = _lin(n1["y"], n=QKV)
    qk, q = _qkn(qkv["y"])
    n1b = _norm(_buf())
    qkv_b = _lin(n1b["y"], n=QKV)
    qk_b, _ = _qkn(qkv_b["y"], q_w=q.rope.q_out)
    assert _plan([n1, qkv, qk, n1b, qkv_b, qk_b])[0] == EUNSUPPORTED
    # two layers sharing pos, freqs and the norm weights fold
    qk_c, _ = _qkn(qkv_b["y"], pos=q.rope.pos, freqs=q.rope.freqs, q_w=q.q_norm_weight, k_w=q.k_norm_weight)
    assert _plan([n1, qkv, qk, n1b, qkv_b, qk_c]) == (OK, 2)
    # a plain ROPE_KV layer and a q / k norm layer in one program
    r = _cabi.Rope.from_buffer_copy(q.rope)
    r.q_out, r.k_cache, r.v_cache = _buf(), _buf(8 * S * KV * D * 2), _buf(8 * S * KV * D * 2)
    _KEEP.append(r)
    rope_b = dict(kind=_cabi.OP_ROPE_KV, M=1, N=QKV, ldx=QKV, x=qkv_b["y"], weight=ctypes.addressof(r))
    assert _plan([n1, qkv, qk, n1b, qkv_b, rope_b]) == (OK, 2)


@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"), reason="needs nvcc")
def test_qknorm_kernels_register_and_spill_budget(tmp_path):
    """One CTA per SM: the q / k norm entries (288 threads) stay within 168 registers and spill nothing."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    src = os.path.join(ROOT, "autoawq_b200", "csrc", "program.cu")
    out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xptxas",
                          "-v", "-c", src, "-o", str(tmp_path / "program.o")], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-2000:]
    log = out.stderr + out.stdout
    entries = re.findall(r"Compiling entry function '(\S*qknorm_kernel\S*)'[^\n]*\n[^\n]*\n\s*(\d+) bytes stack frame, "
                         r"(\d+) bytes spill stores, (\d+) bytes spill loads\n[^\n]*Used (\d+) registers", log)
    assert len(entries) == 4, log[-1500:]          # stream_qknorm_kernel, stream_batch_qknorm_kernel<2|4|8>
    for name, stack, st, ld, regs in entries:
        assert int(regs) <= 168, f"{name}: {regs} registers"
        assert int(st) == 0 and int(ld) == 0 and int(stack) == 0, f"{name}: spills {st} / {ld}, stack {stack}"
