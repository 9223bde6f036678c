"""Host logic of RoPE + KV-cache append in decode programs (B200AWQ_OP_ROPE_KV), checked without a GPU: the stream
format's rotary column pairing (mode 2), the folding rules through b200awq_program_plan, the ctypes descriptor layout
and the register / spill budget of the new kernel entries.

The plan sequences use fake (aligned integer) pointers: the folding only compares addresses.  Shapes are Llama-3-8B's
(hidden 4096, 32 q heads, 8 kv heads, head_dim 128, intermediate 14336)."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from autoawq_b200 import _cabi
from autoawq_b200._cabi import lib
from oracle import awq_oracle as O
from oracle import stream_format as SF

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, EINVAL, EUNSUPPORTED = 0, 1, 2
HID, INTER, H, KV, D, SMS = 4096, 14336, 32, 8, 128, 132
QKV = (H + 2 * KV) * D
S = 2048
_next = [0x10000000]


def rotary_columns(N, D):
    """[S, 16] original columns of mode 2 (include/b200awq.h): set s of head h = s // (D / 16), t = s % (D / 16), holds
    lo[g] = h D + 8 t + g and hi[g] = lo[g] + D / 2, so RoPE's rotation partners share a lane."""
    s = np.arange(N // 16)[:, None]
    g = np.arange(8)[None, :]
    h, t = s // (D // 16), s % (D // 16)
    lo = h * D + 8 * t + g
    return np.concatenate([lo, lo + D // 2], axis=1)


@pytest.fixture
def rotary_oracle(monkeypatch):
    """oracle/stream_format.py with mode 2 routed to rotary_columns(N, head_dim): pack_stream / simulate_gemv then lay
    out and evaluate the rotary format with the oracle's own fragment and constant code."""
    orig = SF.set_columns
    head = {}

    def cols(N, mode):
        return rotary_columns(N, head["D"]) if mode == 2 else orig(N, mode)

    monkeypatch.setattr(SF, "set_columns", cols)
    return head


def test_rotary_columns_pair_every_column_with_its_partner_once():
    for N, D in [(QKV, 128), (3 * 64 * 4, 64), (16, 16), (2 * 80 * 3, 80)]:
        cols = rotary_columns(N, D)
        assert sorted(cols.reshape(-1).tolist()) == list(range(N)), (N, D)
        lo, hi = cols[:, :8], cols[:, 8:]
        assert np.array_equal(hi - lo, np.full_like(lo, D // 2))
        assert np.all(lo % D < D // 2) and np.array_equal(lo // D, hi // D)   # same head, first half


@pytest.mark.parametrize("K,N,G,D", [(256, 3 * 128, 128, 128), (256, 6 * 64, 64, 64), (128, 4 * 64, 32, 64),
                                     (384, 2 * 128, 128, 128)])
def test_rotary_stream_reproduces_dense_contraction(rotary_oracle, K, N, G, D):
    rotary_oracle["D"] = D
    c = O.make_case(K, N, G, seed=K + N + D, raw=True)
    Gs = c["group_size"]
    st = SF.pack_stream(c["qweight"], c["qzeros"], c["scales"], Gs, 2)
    assert st.size == SF.stream_bytes(K, N, Gs)          # the byte count of every mode
    iw, iz = SF.unpack_gemm_ints(c["qweight"], c["qzeros"])
    w = (iw.astype(np.float64) - np.repeat(iz.astype(np.float64), Gs, axis=0)) * \
        np.repeat(c["scales"].astype(np.float64), Gs, axis=0)
    x = np.random.default_rng(2).standard_normal(K).astype(np.float16)
    np.testing.assert_allclose(SF.simulate_gemv(st, K, N, Gs, x, 2), x.astype(np.float64) @ w, rtol=1e-9, atol=1e-9)
    # and it is a different buffer from mode 0 (the pairing is really applied)
    assert not np.array_equal(st, SF.pack_stream(c["qweight"], c["qzeros"], c["scales"], Gs, 0))


def test_rope_struct_matches_header(tmp_path):
    src = tmp_path / "k.c"
    fields = [f for f, _ in _cabi.Rope._fields_]
    body = " ".join(f'printf("%zu ", offsetof(b200awq_rope_t, {f}));' for f in fields)
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200awq.h"\nint main(void) { ' + body +
                   ' printf("%zu %d", sizeof(b200awq_rope_t), B200AWQ_OP_ROPE_KV); return 0; }\n')
    exe = tmp_path / "k"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert got[:-2] == [getattr(_cabi.Rope, f).offset for f in fields]
    assert got[-2] == ctypes.sizeof(_cabi.Rope)
    assert got[-1] == _cabi.OP_ROPE_KV == 6


# ---------------------------------------------------------------------------------------------- folding (plan)
def _buf(nbytes=1 << 16):
    p = _next[0]
    _next[0] += (nbytes + 0xffff) & ~0xffff
    return p


def _lin(x, y=None, k=HID, n=HID, M=1):
    return dict(kind=_cabi.OP_LINEAR_GEMM, M=M, K=k, N=n, group_size=128, ldx=k, x=x, qweight=_buf(), scales=_buf(),
                qzeros=_buf(), y=y or _buf(M * n * 2))


def _norm(x, y=None, k=HID, M=1):
    return dict(kind=_cabi.OP_RMSNORM, M=M, K=k, x=x, weight=_buf(), y=y or _buf(), eps=1e-5)


def _add(a, b, y=None, k=HID, M=1):
    return dict(kind=_cabi.OP_ADD, M=M, K=k, x=a, weight=b, y=y or _buf())


def _silu(gu, y=None, k=INTER, M=1):
    return dict(kind=_cabi.OP_SILU_AND_MUL, M=M, K=k, x=gu, y=y or _buf())


_KEEP = []


def _rope(qkv, M=1, n=QKV, heads=(H, KV, D), **over):
    """A ROPE_KV op on qkv with its own q_out / caches / pos / freqs; `over` replaces descriptor fields."""
    h, kv, d = heads
    r = _cabi.Rope()
    r.n_heads, r.n_kv_heads, r.head_dim, r.cache_len, r.freqs_len = h, kv, d, S, S
    r.cache_batch_stride = S * kv * d
    cache = 8 * S * kv * d * 2
    r.pos, r.freqs, r.q_out = _buf(), _buf(S * d * 4), _buf()
    r.k_cache, r.v_cache = _buf(cache), _buf(cache)
    for f, v in over.items():
        setattr(r, f, v)
    _KEEP.append(r)
    return dict(kind=_cabi.OP_ROPE_KV, M=M, N=n, ldx=n, x=qkv, weight=ctypes.addressof(r)), r


def _plan(ops, max_tokens=1):
    arr = (_cabi.Op * len(ops))()
    for c, o in zip(arr, ops):
        for f, v in o.items():
            setattr(c, f, v)
    kops = ctypes.c_int(-1)
    code = lib.b200awq_program_plan(arr, len(ops), max_tokens, SMS, 0, ctypes.byref(kops))
    return code, kops.value


def _segment(M=1):
    """[o + h, norm2, gate|up, silu, down + h, norm1', qkv', rope'] of a Llama-3-8B layer."""
    attn, h_in = _buf(), _buf()
    o = _lin(attn, M=M)
    h = _add(o["y"], h_in, M=M)
    n2 = _norm(h["y"], M=M)
    gu = _lin(n2["y"], n=2 * INTER, M=M)
    act = _silu(gu["y"], M=M)
    dn = _lin(act["y"], k=INTER, M=M)
    out = _add(dn["y"], h["y"], M=M)
    n1 = _norm(out["y"], M=M)
    qkv = _lin(n1["y"], n=QKV, M=M)
    rope, r = _rope(qkv["y"], M=M)
    return [o, h, n2, gu, act, dn, out, n1, qkv, rope], r


def test_folds_without_adding_kernel_ops():
    x = _buf()
    n1 = _norm(x)
    qkv = _lin(n1["y"], n=QKV)
    rope, _ = _rope(qkv["y"])
    assert _plan([n1, qkv]) == (OK, 1)
    assert _plan([n1, qkv, rope]) == (OK, 1)
    seg, _ = _segment()
    assert _plan(seg[:-1]) == (OK, 4)
    assert _plan(seg) == (OK, 4)
    for M in (2, 4):
        seg, _ = _segment(M)
        assert _plan(seg, max_tokens=M) == (OK, 4), M
    # a later linear may read the raw qkv (its row keeps the raw values), e.g. an o projection over q
    o = _lin(qkv["y"], k=HID)
    assert _plan([n1, qkv, rope, o]) == (OK, 2)


def test_argument_validation():
    qkv = _lin(_buf(), n=QKV)
    rope, r = _rope(qkv["y"])
    for field in ("pos", "freqs", "q_out", "k_cache", "v_cache"):
        bad, _ = _rope(qkv["y"], **{field: 0})
        assert _plan([qkv, bad])[0] == EINVAL, field
    assert _plan([qkv, dict(rope, x=0)])[0] == EINVAL
    assert _plan([qkv, dict(rope, weight=0)])[0] == EINVAL
    for over in (dict(head_dim=127), dict(n_heads=0), dict(cache_len=0), dict(cache_batch_stride=S * KV * D - 1)):
        bad, _ = _rope(qkv["y"], **over)
        assert _plan([qkv, bad])[0] == EINVAL, over


def test_rejected_after_anything_but_a_plain_linear():
    x, r = _buf(), _buf()
    n1 = _norm(x, k=QKV)
    rope, _ = _rope(n1["y"])
    assert _plan([n1, rope, _lin(n1["y"], k=QKV)])[0] == EUNSUPPORTED              # after a glue op
    qkv = _lin(x, n=QKV)
    a = _add(qkv["y"], r, k=QKV)
    rope, _ = _rope(a["y"])
    assert _plan([qkv, a, rope])[0] == EUNSUPPORTED                              # after an add (the linear carries it)
    qkv = _lin(x, n=QKV)
    rope, _ = _rope(qkv["y"])
    rope2, _ = _rope(qkv["y"])
    assert _plan([qkv, rope, rope2])[0] == EUNSUPPORTED                          # after another ROPE_KV
    assert _plan([rope])[0] == EUNSUPPORTED                                      # first op
    # a gate|up whose product SiLU*mul reads (its row would hold silu(gate) * up)
    gu = _lin(x, n=QKV)
    rope, _ = _rope(gu["y"])
    act = _silu(gu["y"], k=QKV // 2)
    assert _plan([gu, rope, act, _lin(act["y"], k=QKV // 2)])[0] == EUNSUPPORTED
    # a sparse-MoE block's down op
    E, k, Hm, Im = 8, 2, QKV, 512
    d = _cabi.Moe()
    d.E, d.top_k, d.renormalize, d.group_size, d.H, d.I, d.block_size = E, k, 1, 128, Hm, Im, 16
    d.sorted_len = k + E * 15
    d.gate_weight = _buf()
    for f, _ in _cabi.Moe._fields_[9:]:
        setattr(d, f, _buf())
    xn = _norm(x, k=Hm)
    moe = dict(kind=_cabi.OP_SPARSE_MOE, M=1, K=Hm, N=Hm, x=xn["y"], y=_buf(), weight=ctypes.addressof(d))
    rope, _ = _rope(moe["y"])
    assert _plan([xn, moe])[0] == OK
    assert _plan([xn, moe, rope])[0] == EUNSUPPORTED


def test_rejected_when_qkv_is_not_the_whole_output_or_the_shape_is_off():
    x = _buf()
    qkv = _lin(x, n=QKV)
    rope, _ = _rope(qkv["y"] + 256, n=QKV - 128)
    assert _plan([qkv, rope])[0] == EUNSUPPORTED                                 # a slice of the linear's output
    rope, _ = _rope(_buf())
    assert _plan([qkv, rope])[0] == EUNSUPPORTED                                 # not the linear's output at all
    wide = _lin(x, n=QKV + 128)
    rope, _ = _rope(wide["y"])
    assert _plan([wide, rope])[0] == EUNSUPPORTED                                # N != (H + 2 KV) D
    rope, _ = _rope(wide["y"], n=QKV + 128)
    assert _plan([wide, rope])[0] == EUNSUPPORTED
    d72 = (H + 2 * KV) * 72                                                      # D % 16 != 0
    q72 = _lin(x, n=d72)
    rope, _ = _rope(q72["y"], n=d72, heads=(H, KV, 72))
    assert _plan([q72, rope])[0] == EUNSUPPORTED
    d64 = (H + 2 * KV) * 64
    q64 = _lin(x, n=d64)
    rope, _ = _rope(q64["y"], n=d64, heads=(H, KV, 64))
    assert _plan([q64, rope])[0] == OK


def test_rejected_when_another_op_touches_q_out_or_the_caches():
    x = _buf()
    for field in ("q_out", "k_cache", "v_cache"):
        n1 = _norm(x)
        qkv = _lin(n1["y"], n=QKV)
        rope, r = _rope(qkv["y"])
        target = getattr(r, field)
        # a later linear reads it
        assert _plan([n1, qkv, rope, _lin(target, k=HID)])[0] == EUNSUPPORTED, field
        # a later linear writes it
        assert _plan([n1, qkv, rope, _lin(_buf(), y=target, k=HID)])[0] == EUNSUPPORTED, field
        # an earlier glue op writes it / reads it
        assert _plan([_norm(_buf(), y=target), _lin(target, k=HID), n1, qkv, rope])[0] == EUNSUPPORTED, field
        nt = _norm(target)
        assert _plan([nt, _lin(nt["y"], k=HID), n1, qkv, rope])[0] == EUNSUPPORTED, field
        # an add uses it as its residual
        o = _lin(_buf())
        assert _plan([n1, qkv, rope, o, _add(o["y"], target)])[0] == EUNSUPPORTED, field
        # a second ROPE_KV writes into the same buffer
        n1b = _norm(_buf())
        qkv_b = _lin(n1b["y"], n=QKV)
        rope_b, _ = _rope(qkv_b["y"], **{field: target})
        assert _plan([n1, qkv, rope, n1b, qkv_b, rope_b])[0] == EUNSUPPORTED, field
        # the qkv linear's own output (in place)
        rope_ip, _ = _rope(qkv["y"], **{field: qkv["y"]})
        assert _plan([n1, qkv, rope_ip])[0] == EUNSUPPORTED, field
    # a program op writing the position
    n1 = _norm(x)
    qkv = _lin(n1["y"], n=QKV)
    rope, r = _rope(qkv["y"])
    assert _plan([n1, qkv, rope, _lin(_buf(), y=r.pos)])[0] == EUNSUPPORTED
    # two layers sharing pos and freqs fold
    n1b = _norm(_buf())
    qkv_b = _lin(n1b["y"], n=QKV)
    rope_b, _ = _rope(qkv_b["y"], pos=r.pos, freqs=r.freqs)
    assert _plan([n1, qkv, rope, n1b, qkv_b, rope_b]) == (OK, 2)


@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"), reason="needs nvcc")
def test_rope_kernels_register_and_spill_budget(tmp_path):
    """One CTA per SM: the rope entries (288 threads) fit the register file and spill nothing."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    src = os.path.join(ROOT, "autoawq_b200", "csrc", "program.cu")
    out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xptxas",
                          "-v", "-c", src, "-o", str(tmp_path / "program.o")], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-2000:]
    log = out.stderr + out.stdout
    entries = re.findall(r"Compiling entry function '(\S*rope_kernel\S*)'[^\n]*\n[^\n]*\n\s*(\d+) bytes stack frame, "
                         r"(\d+) bytes spill stores, (\d+) bytes spill loads\n[^\n]*Used (\d+) registers", log)
    assert len(entries) == 4, log[-1500:]          # stream_rope_kernel, stream_batch_rope_kernel<2|4|8>
    for name, stack, st, ld, regs in entries:
        assert int(regs) * (32 + 32 * 8) <= 65536, f"{name}: {regs} registers x 288 threads"
        assert int(st) == 0 and int(ld) == 0 and int(stack) == 0, f"{name}: spills {st} / {ld}, stack {stack}"
