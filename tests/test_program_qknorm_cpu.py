"""Host logic of Qwen3's q / k norm folded into decode programs (B200AWQ_OP_QK_NORM_ROPE_KV), checked without a GPU: the
ctypes descriptor layout, the exported entry point, the folding rules through b200awq_program_plan (ROPE_KV's rules on
the embedded descriptor, plus the norm weights) and the register / spill budget of the new kernel entries.

The plan sequences use fake (aligned integer) pointers: the folding only compares addresses.  Shapes are Qwen3-8B's
(hidden 4096, 32 q heads, 8 kv heads, head_dim 128, intermediate 12288)."""
import ctypes
from functools import partial

from _fake_ops import add, buf, linear, rmsnorm, silu
from _fake_ops import plan as _fplan
from _toolchain import entries, header_constants, header_layout, mirror_layout, needs_nvcc
from autoawq_b200 import _cabi
from autoawq_b200._cabi import lib

OK, EINVAL, EUNSUPPORTED = 0, 1, 2
HID, INTER, H, KV, D, SMS = 4096, 12288, 32, 8, 128, 132
QKV = (H + 2 * KV) * D
S = 2048
_norm = partial(rmsnorm, eps=1e-6)
_plan = partial(_fplan, sms=SMS)
_KEEP = []


def _qkn(qkv, M=1, n=QKV, heads=(H, KV, D), q_w=None, k_w=None, **over):
    """A QK_NORM_ROPE_KV op on qkv with its own q_out / caches / pos / freqs / norm weights; `over` replaces fields of
    the embedded rope descriptor."""
    h, kv, d = heads
    q = _cabi.QkNormRope()
    r = q.rope
    r.n_heads, r.n_kv_heads, r.head_dim, r.cache_len, r.freqs_len = h, kv, d, S, S
    r.cache_batch_stride = S * kv * d
    cache = 8 * S * kv * d * 2
    r.pos, r.freqs, r.q_out = buf(), buf(S * d * 4), buf()
    r.k_cache, r.v_cache = buf(cache), buf(cache)
    for f, v in over.items():
        setattr(r, f, v)
    q.q_norm_weight = buf() if q_w is None else q_w
    q.k_norm_weight = buf() if k_w is None else k_w
    q.eps = 1e-6
    _KEEP.append(q)
    return dict(kind=_cabi.OP_QK_NORM_ROPE_KV, M=M, N=n, ldx=n, x=qkv, weight=ctypes.addressof(q)), q


def _segment(M=1, hid=HID):
    """[o + h, norm2, gate|up, silu, down + h, norm1', qkv', qk-norm-rope'] of a Qwen3 layer (hidden `hid`)."""
    attn, h_in = buf(), buf()
    o = linear(attn, H * D, hid, M=M)
    h = add(o["y"], h_in, hid, M=M)
    n2 = _norm(h["y"], hid, M=M)
    gu = linear(n2["y"], hid, 2 * INTER, M=M)
    act = silu(gu["y"], INTER, M=M)
    dn = linear(act["y"], INTER, hid, M=M)
    out = add(dn["y"], h["y"], hid, M=M)
    n1 = _norm(out["y"], hid, M=M)
    qkv = linear(n1["y"], hid, QKV, M=M)
    qk, q = _qkn(qkv["y"], M=M)
    return [o, h, n2, gu, act, dn, out, n1, qkv, qk], q


def test_struct_matches_header():
    assert header_layout(_cabi.QkNormRope, "b200awq_qk_norm_rope_t") == mirror_layout(_cabi.QkNormRope)
    assert header_layout(_cabi.Rope, "b200awq_rope_t")["sizeof"] == ctypes.sizeof(_cabi.Rope) == 72  # embedded: unchanged
    assert header_constants("B200AWQ_OP_QK_NORM_ROPE_KV", "B200AWQ_OP_ROPE_KV") == (
        _cabi.OP_QK_NORM_ROPE_KV, _cabi.OP_ROPE_KV) == (7, 6)


def test_entry_point_is_exported():
    assert "b200awq_qk_norm_rope_kv" in _cabi.SIGNATURES
    fn = getattr(lib, "b200awq_qk_norm_rope_kv")
    assert fn.restype is ctypes.c_int
    # argument checks happen before any CUDA call: a null descriptor / qkv is EINVAL, M = 0 with a valid one is a no-op
    assert fn(None, QKV, None, 1, None) == EINVAL
    _, q = _qkn(buf())
    assert fn(None, QKV, q, 1, None) == EINVAL
    assert fn(buf(), QKV, q, 0, None) == OK
    for field in ("q_norm_weight", "k_norm_weight"):
        bad = _cabi.QkNormRope.from_buffer_copy(q)
        setattr(bad, field, 0)
        assert fn(buf(), QKV, bad, 1, None) == EINVAL, field
    _, q72 = _qkn(buf(), n=(H + 2 * KV) * 72, heads=(H, KV, 72))
    assert fn(buf(), (H + 2 * KV) * 72, q72, 1, None) == EUNSUPPORTED       # the summation order needs D % 16 == 0


def test_folds_without_adding_kernel_ops():
    x = buf()
    n1 = _norm(x, HID)
    qkv = linear(n1["y"], HID, QKV)
    qk, _ = _qkn(qkv["y"])
    assert _plan([n1, qkv]) == (OK, 1)
    assert _plan([n1, qkv, qk]) == (OK, 1)
    for M in (1, 2, 4):
        seg, _ = _segment(M)
        assert _plan(seg, max_tokens=M) == (OK, 4), M
        assert _plan(seg[:-1], max_tokens=M) == (OK, 4), M
    seg, _ = _segment(hid=2560)                      # Qwen3-4B: hidden 2560 != H D = 4096
    assert _plan(seg) == (OK, 4)
    o = linear(qkv["y"], HID, HID)                        # a later linear may read the raw qkv
    assert _plan([n1, qkv, qk, o]) == (OK, 2)


def test_argument_validation():
    qkv = linear(buf(), HID, QKV)
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
    for over in (dict(q_w=buf() + 8), dict(k_w=buf() + 2)):          # misaligned norm weights
        bad, _ = _qkn(qkv["y"], **over)
        assert _plan([qkv, bad])[0] == EUNSUPPORTED, over


def test_rejected_after_anything_but_a_plain_linear():
    x, r = buf(), buf()
    n1 = _norm(x, QKV)
    qk, _ = _qkn(n1["y"])
    assert _plan([n1, qk, linear(n1["y"], QKV, HID)])[0] == EUNSUPPORTED            # after a glue op
    qkv = linear(x, HID, QKV)
    a = add(qkv["y"], r, QKV)
    qk, _ = _qkn(a["y"])
    assert _plan([qkv, a, qk])[0] == EUNSUPPORTED                              # after an add
    qkv = linear(x, HID, QKV)
    qk, _ = _qkn(qkv["y"])
    qk2, _ = _qkn(qkv["y"])
    assert _plan([qkv, qk, qk2])[0] == EUNSUPPORTED                            # after another rope op
    assert _plan([qk])[0] == EUNSUPPORTED                                      # first op
    gu = linear(x, HID, QKV)                                                        # a gate|up whose product SiLU*mul reads
    qk, _ = _qkn(gu["y"])
    act = silu(gu["y"], QKV // 2)
    assert _plan([gu, qk, act, linear(act["y"], QKV // 2, HID)])[0] == EUNSUPPORTED
    E, k, Hm, Im = 8, 2, QKV, 512                                              # a sparse-MoE block's down op
    d = _cabi.Moe()
    d.E, d.top_k, d.renormalize, d.group_size, d.H, d.I, d.block_size = E, k, 1, 128, Hm, Im, 16
    d.sorted_len = k + E * 15
    d.gate_weight = buf()
    for f, _ in _cabi.Moe._fields_[9:]:
        setattr(d, f, buf())
    _KEEP.append(d)
    xn = _norm(x, Hm)
    moe = dict(kind=_cabi.OP_SPARSE_MOE, M=1, K=Hm, N=Hm, x=xn["y"], y=buf(), weight=ctypes.addressof(d))
    qk, _ = _qkn(moe["y"])
    assert _plan([xn, moe])[0] == OK
    assert _plan([xn, moe, qk])[0] == EUNSUPPORTED


def test_rejected_when_qkv_is_not_the_whole_output_or_the_shape_is_off():
    x = buf()
    qkv = linear(x, HID, QKV)
    qk, _ = _qkn(qkv["y"] + 256, n=QKV - 128)
    assert _plan([qkv, qk])[0] == EUNSUPPORTED                                 # a slice of the linear's output
    qk, _ = _qkn(buf())
    assert _plan([qkv, qk])[0] == EUNSUPPORTED                                 # not the linear's output at all
    wide = linear(x, HID, QKV + 128)
    qk, _ = _qkn(wide["y"], n=QKV + 128)
    assert _plan([wide, qk])[0] == EUNSUPPORTED                                # N != (H + 2 KV) D
    d72 = (H + 2 * KV) * 72
    q72 = linear(x, HID, d72)
    qk, _ = _qkn(q72["y"], n=d72, heads=(H, KV, 72))
    assert _plan([q72, qk])[0] == EUNSUPPORTED                                 # D % 16 != 0
    d64 = (H + 2 * KV) * 64
    q64 = linear(x, HID, d64)
    qk, _ = _qkn(q64["y"], n=d64, heads=(H, KV, 64))
    assert _plan([q64, qk])[0] == OK


def test_rejected_when_another_op_touches_its_outputs_or_writes_its_inputs():
    x = buf()
    for field in ("q_out", "k_cache", "v_cache"):
        n1 = _norm(x, HID)
        qkv = linear(n1["y"], HID, QKV)
        qk, q = _qkn(qkv["y"])
        target = getattr(q.rope, field)
        assert _plan([n1, qkv, qk, linear(target, HID, HID)])[0] == EUNSUPPORTED, field           # a later linear reads it
        assert _plan([n1, qkv, qk, linear(buf(), HID, HID, y=target)])[0] == EUNSUPPORTED, field  # ... writes it
        assert _plan([_norm(buf(), HID, y=target), linear(target, HID, HID), n1, qkv, qk])[0] == EUNSUPPORTED, field
        o = linear(buf(), HID, HID)
        assert _plan([n1, qkv, qk, o, add(o["y"], target, HID)])[0] == EUNSUPPORTED, field
        n1b = _norm(buf(), HID)
        qkv_b = linear(n1b["y"], HID, QKV)
        qk_b, _ = _qkn(qkv_b["y"], **{field: target})                          # a second op writes into it
        assert _plan([n1, qkv, qk, n1b, qkv_b, qk_b])[0] == EUNSUPPORTED, field
        qk_ip, _ = _qkn(qkv["y"], **{field: qkv["y"]})                        # the qkv linear's own output
        assert _plan([n1, qkv, qk_ip])[0] == EUNSUPPORTED, field
    for field in ("q_norm_weight", "k_norm_weight", "pos"):
        n1 = _norm(x, HID)
        qkv = linear(n1["y"], HID, QKV)
        qk, q = _qkn(qkv["y"])
        target = getattr(q, field) if field != "pos" else q.rope.pos
        assert _plan([n1, qkv, qk, linear(buf(), HID, HID, y=target)])[0] == EUNSUPPORTED, field       # a program op writes it
        assert _plan([linear(buf(), HID, HID, y=target), n1, qkv, qk])[0] == EUNSUPPORTED, field
        assert _plan([n1, qkv, qk, linear(target, HID, HID)])[0] == OK, field                    # reading it is fine
    # the q_out of one layer's op as the next layer's norm weight: a write of a read
    n1 = _norm(x, HID)
    qkv = linear(n1["y"], HID, QKV)
    qk, q = _qkn(qkv["y"])
    n1b = _norm(buf(), HID)
    qkv_b = linear(n1b["y"], HID, QKV)
    qk_b, _ = _qkn(qkv_b["y"], q_w=q.rope.q_out)
    assert _plan([n1, qkv, qk, n1b, qkv_b, qk_b])[0] == EUNSUPPORTED
    # two layers sharing pos, freqs and the norm weights fold
    qk_c, _ = _qkn(qkv_b["y"], pos=q.rope.pos, freqs=q.rope.freqs, q_w=q.q_norm_weight, k_w=q.k_norm_weight)
    assert _plan([n1, qkv, qk, n1b, qkv_b, qk_c]) == (OK, 2)
    # a plain ROPE_KV layer and a q / k norm layer in one program
    r = _cabi.Rope.from_buffer_copy(q.rope)
    r.q_out, r.k_cache, r.v_cache = buf(), buf(8 * S * KV * D * 2), buf(8 * S * KV * D * 2)
    _KEEP.append(r)
    rope_b = dict(kind=_cabi.OP_ROPE_KV, M=1, N=QKV, ldx=QKV, x=qkv_b["y"], weight=ctypes.addressof(r))
    assert _plan([n1, qkv, qk, n1b, qkv_b, rope_b]) == (OK, 2)


@needs_nvcc
def test_qknorm_kernels_register_and_spill_budget():
    """One CTA per SM: the q / k norm entries (288 threads) stay within 168 registers and spill nothing."""
    found = entries("program.cu", r"qknorm_kernel")
    assert len(found) == 4, found          # stream_qknorm_kernel, stream_batch_qknorm_kernel<2|4|8>
    for name, (regs, stack, st, ld) in found.items():
        assert regs <= 168, f"{name}: {regs} registers"
        assert st == 0 and ld == 0 and stack == 0, f"{name}: spills {st} / {ld}, stack {stack}"
