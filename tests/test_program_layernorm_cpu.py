"""Host logic of the LayerNorm blocks' decode programs (B200AWQ_OP_LAYER_NORM, _GELU, _GELU_TANH), checked without a GPU:
the header constants against the ctypes mirror, the exported stand-alone entry points and their argument checks, the
folding through b200awq_program_plan (Command-R, StarCoder2 and MPT segments at their real geometry), every rejection,
and the register / spill budget of the new kernel entry.

The plan sequences use fake (aligned integer) pointers: the folding only compares addresses."""
import ctypes
from functools import partial

import pytest

from _fake_ops import add, buf, linear, plan as _fplan, rmsnorm, silu
from _toolchain import entries, header_constants, needs_nvcc
from autoawq_b200 import _cabi
from autoawq_b200._cabi import lib

OK, EINVAL, EUNSUPPORTED = 0, 1, 2
SMS, S = 132, 4096
_plan = partial(_fplan, sms=SMS)
_KEEP = []

# name: (hidden, q heads, kv heads, intermediate, gated MLP, GELU op, rope)
MODELS = {
    "command-r-v01": (8192, 64, 64, 22528, True, None, True),
    "starcoder2-3b": (3072, 24, 2, 12288, False, _cabi.OP_GELU_TANH, True),
    "starcoder2-15b": (6144, 48, 4, 24576, False, _cabi.OP_GELU_TANH, True),
    "mpt-7b": (4096, 32, 32, 16384, False, _cabi.OP_GELU, False),
}


def layer_norm(x, K, M=1, bias=True, y=None):
    return dict(kind=_cabi.OP_LAYER_NORM, M=M, K=K, eps=1e-5, x=x, weight=buf(K * 2), bias=buf(K * 2) if bias else None,
                y=buf(M * K * 2) if y is None else y)


def gelu(x, K, M=1, kind=_cabi.OP_GELU_TANH, y=None):
    return dict(kind=kind, M=M, K=K, x=x, y=buf(M * K * 2) if y is None else y)


def _rope(qkv, H, KV, D=128, M=1):
    r = _cabi.Rope()
    r.n_heads, r.n_kv_heads, r.head_dim, r.cache_len, r.freqs_len = H, KV, D, S, S
    r.cache_batch_stride = S * KV * D
    r.pos, r.freqs, r.q_out = buf(), buf(S * D * 4), buf(M * H * D * 2)
    r.k_cache, r.v_cache = buf(8 * S * KV * D * 2), buf(8 * S * KV * D * 2)
    _KEEP.append(r)
    n = (H + 2 * KV) * D
    return dict(kind=_cabi.OP_ROPE_KV, M=M, N=n, ldx=n, x=qkv, weight=ctypes.addressof(r))


def segment(model, M=1, shared_norm=False):
    """One attention-to-attention segment in the recording order of autoawq_b200/program.py's docstring."""
    hid, H, KV, inter, gated, gk, rope = MODELS[model]
    qkv_n = (H + 2 * KV) * 128
    attn, x = buf(), buf()
    o = linear(attn, H * 128, hid, M=M)
    h = add(o["y"], x, hid, M=M)
    if gated:                                                 # Command-R: parallel residual, xn from the last segment
        xn = buf(hid * 2 * M)
        gu = linear(xn, hid, 2 * inter, M=M)
        act = silu(gu["y"], inter, M=M)
        mlp = [gu, act]
        d = linear(act["y"], inter, hid, M=M)
    else:
        n2 = layer_norm(h["y"], hid, M=M)
        fc = linear(n2["y"], hid, inter, M=M)
        g = gelu(fc["y"], inter, M=M, kind=gk)
        mlp = [n2, fc, g]
        d = linear(g["y"], inter, hid, M=M)
    out = add(d["y"], h["y"], hid, M=M)
    n1 = layer_norm(out["y"], hid, M=M, bias=not gated, y=xn if gated and shared_norm else None)
    qkv = linear(n1["y"], hid, qkv_n, M=M)
    ops = [o, h] + mlp + [d, out, n1, qkv]
    return ops + ([_rope(qkv["y"], H, KV, M=M)] if rope else [])


def test_header_constants_and_entry_points():
    assert header_constants("B200AWQ_OP_LAYER_NORM", "B200AWQ_OP_GELU", "B200AWQ_OP_GELU_TANH",
                            "B200AWQ_OP_MLA_Q_ROPE") == (_cabi.OP_LAYER_NORM, _cabi.OP_GELU, _cabi.OP_GELU_TANH,
                                                         _cabi.OP_MLA_Q_ROPE) == (14, 15, 16, 13)
    for name in ("b200awq_layer_norm", "b200awq_gelu"):
        assert name in _cabi.SIGNATURES and getattr(lib, name).restype is ctypes.c_int
    ln, ge = lib.b200awq_layer_norm, lib.b200awq_gelu
    x, w, b, y = buf(), buf(), buf(), buf()
    # argument checks come before any CUDA call
    assert ln(None, 4096, w, b, y, 1, 4096, 1e-5, None) == EINVAL
    assert ln(x, 4096, None, b, y, 1, 4096, 1e-5, None) == EINVAL
    assert ln(x, 4096, w, b, None, 1, 4096, 1e-5, None) == EINVAL
    assert ln(x, 100, w, b, y, 2, 4096, 1e-5, None) == EINVAL                 # pitch < hidden
    assert ln(x, 4100, w, b, y, 1, 4100, 1e-5, None) == EUNSUPPORTED          # hidden % 8 != 0
    assert ln(x, 4100, w, b, y, 2, 4096, 1e-5, None) == EUNSUPPORTED          # pitch % 8 != 0
    assert ln(x + 8, 4096, w, b, y, 1, 4096, 1e-5, None) == EUNSUPPORTED      # misaligned x
    assert ln(x, 4096, w, b + 2, y, 1, 4096, 1e-5, None) == EUNSUPPORTED      # misaligned bias
    assert ln(x, 4096, w, None, y, 0, 4096, 1e-5, None) == OK                 # no rows: nothing to do
    assert ge(None, y, 1, 64, 1, None) == EINVAL
    assert ge(x, y, 1, 64, 2, None) == EINVAL                                 # approximate is 0 or 1
    assert ge(x, y, 0, 64, 0, None) == OK


@pytest.mark.parametrize("model", sorted(MODELS))
def test_segments_fold_into_four_kernel_ops(model):
    seg = segment(model)
    assert _plan(seg) == (OK, 4)
    if MODELS[model][4]:
        assert _plan(segment(model, shared_norm=True)) == (OK, 4)     # xn and xn' one buffer


def test_glue_folds_like_rmsnorm():
    x = buf()
    n = layer_norm(x, 4096)
    a, b = linear(n["y"], 4096, 4096), linear(n["y"], 4096, 1024)
    assert _plan([n, a, b]) == (OK, 2)                       # every consumer stages it; the first stores y
    assert _plan([n, a, layer_norm(a["y"], 4096, bias=False), linear(buf(), 4096, 4096)])[0] == EUNSUPPORTED  # unused
    src = linear(x, 4096, 6144)
    sl = layer_norm(src["y"] + 2048 * 2, 4096)               # a slice of the previous op's published row
    assert _plan([src, sl, linear(sl["y"], 4096, 4096)]) == (OK, 2)
    fc = linear(x, 4096, 16384)
    g = gelu(fc["y"], 16384, kind=_cabi.OP_GELU)
    assert _plan([fc, g, linear(g["y"], 16384, 4096)]) == (OK, 2)
    assert _plan([fc, g, linear(g["y"], 16384, 4096), linear(g["y"], 16384, 4096)]) == (OK, 3)   # a later reader


def test_rejections():
    x, r = buf(), buf()
    fc = linear(x, 4096, 16384)
    g = gelu(fc["y"], 16384)
    down = linear(g["y"], 16384, 4096)
    assert _plan([fc, g, down]) == (OK, 2)
    # GELU after anything but a plain linear: a glue op, an ADD, a rope finish, a MoE block's down op
    n = rmsnorm(x, 16384)
    assert _plan([n, gelu(n["y"], 16384), linear(buf(), 4096, 4096)])[0] == EUNSUPPORTED
    a = add(fc["y"], r, 16384)
    ga = gelu(a["y"], 16384)
    assert _plan([fc, a, ga, linear(ga["y"], 16384, 4096)])[0] == EUNSUPPORTED
    qkv = linear(x, 4096, 6144)
    rp = _rope(qkv["y"], 32, 8)
    gr = gelu(qkv["y"], 6144)
    assert _plan([qkv, rp, gr, linear(gr["y"], 6144, 4096)])[0] == EUNSUPPORTED
    d = _cabi.Moe()
    d.E, d.top_k, d.renormalize, d.group_size, d.H, d.I, d.block_size = 8, 2, 1, 128, 4096, 1024, 16
    d.sorted_len = 2 + 8 * 15
    d.gate_weight = buf()
    for f, _ in _cabi.Moe._fields_[9:]:
        setattr(d, f, buf())
    _KEEP.append(d)
    xn = rmsnorm(x, 4096)
    moe = dict(kind=_cabi.OP_SPARSE_MOE, M=1, K=4096, N=4096, x=xn["y"], y=buf(), weight=ctypes.addressof(d))
    gm = gelu(moe["y"], 4096)
    assert _plan([xn, moe]) == (OK, 2)
    assert _plan([xn, moe, gm, linear(gm["y"], 4096, 4096)])[0] == EUNSUPPORTED
    # a mode-1 producer: a SiLU*mul of the GELU's output
    s = silu(g["y"], 8192)
    assert _plan([fc, g, s, linear(s["y"], 8192, 4096)])[0] == EUNSUPPORTED
    # an ADD and a GELU on one finish, either order
    ag = add(g["y"], r, 16384)
    assert _plan([fc, g, ag, linear(ag["y"], 16384, 4096)])[0] == EUNSUPPORTED
    # a later read of the raw y: by a linear, a glue op, an ADD's residual
    assert _plan([fc, g, down, linear(fc["y"], 16384, 4096)])[0] == EUNSUPPORTED
    ln_raw = layer_norm(fc["y"], 16384)
    assert _plan([fc, g, down, ln_raw, linear(ln_raw["y"], 16384, 4096)])[0] == EUNSUPPORTED
    o2 = linear(buf(), 4096, 16384)
    assert _plan([fc, g, down, o2, add(o2["y"], fc["y"], 16384)])[0] == EUNSUPPORTED
    # in place, or on part of the linear's output
    gi = gelu(fc["y"], 16384, y=fc["y"])
    assert _plan([fc, gi, linear(gi["y"], 16384, 4096)])[0] == EUNSUPPORTED
    gp = gelu(fc["y"], 8192)
    assert _plan([fc, gp, linear(gp["y"], 8192, 4096)])[0] == EUNSUPPORTED
    assert _plan([gelu(buf(), 4096), linear(buf(), 4096, 4096)])[0] == EUNSUPPORTED     # first op
    # in-place LayerNorm
    li = layer_norm(x, 4096, y=x)
    assert _plan([li, linear(li["y"], 4096, 4096)])[0] == EUNSUPPORTED
    # mixed with MoE, q / k norm or MLA ops
    ln = layer_norm(x, 4096)
    assert _plan([ln, linear(ln["y"], 4096, 4096), xn, moe])[0] == EUNSUPPORTED
    assert _plan([fc, g, down, xn, moe])[0] == EUNSUPPORTED
    q = _cabi.QkNormRope()
    q.rope = _cabi.Rope.from_buffer_copy(ctypes.cast(rp["weight"], ctypes.POINTER(_cabi.Rope)).contents)
    q.q_norm_weight, q.k_norm_weight, q.eps = buf(), buf(), 1e-6
    _KEEP.append(q)
    qkv2 = linear(ln["y"], 4096, 6144)
    qk = dict(kind=_cabi.OP_QK_NORM_ROPE_KV, M=1, N=6144, ldx=6144, x=qkv2["y"], weight=ctypes.addressof(q))
    assert _plan([ln, qkv2, qk])[0] == EUNSUPPORTED
    rn = rmsnorm(x, 4096)
    qkv3 = linear(rn["y"], 4096, 6144)
    assert _plan([rn, qkv3, dict(qk, x=qkv3["y"])]) == (OK, 1)              # the same op under an RMSNorm folds
    m = _cabi.Mla()
    m.n_heads, m.nope_dim, m.rope_dim, m.v_dim, m.kv_lora_rank, m.cache_len, m.freqs_len = 16, 128, 64, 128, 512, S, S
    m.k_batch_stride, m.v_batch_stride, m.v_head_stride = S * 16 * 192, S * 16 * 128, 128
    m.pos, m.freqs, m.k_cache, m.v_cache = buf(), buf(S * 64 * 4), buf(8 * S * 16 * 192 * 2), buf(8 * S * 16 * 128 * 2)
    _KEEP.append(m)
    kvb = linear(ln["y"], 4096, 16 * 256)
    mkv = dict(kind=_cabi.OP_MLA_KV, M=1, N=16 * 256, ldx=16 * 256, x=kvb["y"], weight=ctypes.addressof(m))
    assert _plan([ln, kvb, mkv])[0] == EUNSUPPORTED
    kvb3 = linear(rn["y"], 4096, 16 * 256)
    assert _plan([rn, kvb3, dict(mkv, x=kvb3["y"])]) == (OK, 1)


@pytest.mark.parametrize("model", sorted(MODELS))
def test_batched_programs_are_not_fused(model):
    """Any program created with max_tokens > 1 that holds these ops replays per op, at M = 1 too."""
    for M in (1, 2, 4):
        assert _plan(segment(model, M=M), max_tokens=4)[0] == EUNSUPPORTED, M
    fc = linear(buf(), 4096, 16384, M=2)
    assert _plan([fc, gelu(fc["y"], 16384, M=2), linear(buf(), 16384, 4096, M=2)], max_tokens=2)[0] == EUNSUPPORTED


@needs_nvcc
def test_layernorm_entry_register_and_spill_budget():
    """One 288-thread CTA per SM: stream_layernorm_kernel stays within 168 registers and spills nothing."""
    found = entries("program.cu", r"stream_layernorm_kernel")
    assert len(found) == 1, found
    for name, (regs, stack, st, ld) in found.items():
        assert regs <= 168 and regs * (32 + 8 * 32) <= 65536, f"{name}: {regs} registers"
        assert st == 0 and ld == 0 and stack == 0, f"{name}: spills {st} / {ld}, stack {stack}"
