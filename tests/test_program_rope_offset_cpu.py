"""Host logic of RoPE + KV-cache append with a per-sequence rotary offset (B200AWQ_OP_ROPE_KV_OFFSET,
b200awq_rope_kv_offset), checked without a GPU: the constants, exports and descriptor layout, the argument checks of
the stand-alone entry and of the op, the folding through b200awq_program_plan (Qwen2.5-VL-7B, Llama-3-8B, Qwen3-8B and
StableLM segments fold into exactly the kernel ops of the same segment without offsets), the offsets as a read no op
may write, and the register / spill budget of every entry whose finish reads them.

ROPE_KV's and QK_NORM_ROPE_KV's own folding tests are run again with their op builders returning the new kind.  The
plan sequences use fake (aligned integer) pointers."""
import ctypes
import re
from functools import partial

import pytest

import test_program_qknorm_cpu as QK
import test_program_rope_cpu as RK
from _fake_ops import add, buf, linear, plan as _fplan, rmsnorm, silu
from _toolchain import entries, header_constants, header_layout, mirror_layout, needs_nvcc
from autoawq_b200 import _cabi
from autoawq_b200._cabi import lib
from test_program_partial_rope_cpu import STABLELM, stablelm_segment

OK, EINVAL, EUNSUPPORTED = 0, 1, 2
S, SMS = 2048, 132
_plan = partial(_fplan, sms=SMS)
_KEEP = []


def offset(op, T=1, rot_offset=None):
    """The ROPE_KV / QK_NORM_ROPE_KV / _SEQ op dict `op` as a ROPE_KV_OFFSET with T tokens per sequence: a
    b200awq_rope_offset_t embedding a copy of its descriptor (null norm weights for ROPE_KV) and the offsets at
    rot_offset (a fresh buffer when None)."""
    d = _cabi.RopeOffset()
    if op["kind"] in (_cabi.OP_QK_NORM_ROPE_KV, _cabi.OP_QK_NORM_ROPE_KV_SEQ):
        d.qk = _cabi.QkNormRope.from_address(op["weight"])
    else:
        d.qk.rope = _cabi.Rope.from_address(op["weight"])
    d.rot_offset = buf() if rot_offset is None else rot_offset
    _KEEP.append(d)
    return dict(op, kind=_cabi.OP_ROPE_KV_OFFSET, K=T, weight=ctypes.addressof(d)), d


def test_constants_exports_and_layout():
    assert header_constants("B200AWQ_OP_ROPE_KV_OFFSET") == (_cabi.OP_ROPE_KV_OFFSET,) == (19,)
    assert "b200awq_rope_kv_offset" in _cabi.SIGNATURES
    assert lib.b200awq_rope_kv_offset.restype is ctypes.c_int
    lay = header_layout(_cabi.RopeOffset, "b200awq_rope_offset_t")
    assert lay == mirror_layout(_cabi.RopeOffset) == {"sizeof": 104, "qk": 0, "rot_offset": 96}
    assert ctypes.sizeof(_cabi.Rope) == 72 and ctypes.sizeof(_cabi.QkNormRope) == 96   # embedded unchanged


def _desc(norm=False, **over):
    """A stand-alone descriptor of Llama-3-8B heads (with Qwen3's norm weights when norm)."""
    op, d = (QK._qkn if norm else RK._rope)(buf(), **over)
    return offset(op)[1]


def test_stand_alone_argument_checks_before_any_cuda_call():
    QKV = RK.QKV
    for norm in (False, True):
        d = _desc(norm)
        for M, T in ((4, 0), (4, -1), (4, 3), (6, 4), (1, 2)):
            assert lib.b200awq_rope_kv_offset(buf(), QKV, d, M, T, None) == EINVAL, (norm, M, T)
        assert lib.b200awq_rope_kv_offset(None, QKV, d, 4, 2, None) == EINVAL
        assert lib.b200awq_rope_kv_offset(buf(), QKV, None, 4, 2, None) == EINVAL
        assert lib.b200awq_rope_kv_offset(buf(), QKV - 1, d, 4, 2, None) == EINVAL
        assert lib.b200awq_rope_kv_offset(buf(), QKV, d, 0, 3, None) == OK                 # M = 0: nothing to do
        bad = _cabi.RopeOffset.from_buffer_copy(d)
        bad.rot_offset = 0
        assert lib.b200awq_rope_kv_offset(buf(), QKV, bad, 4, 2, None) == EINVAL           # null rot_offset
        assert lib.b200awq_rope_kv_offset(buf(), QKV, bad, 0, 1, None) == EINVAL
    # the embedded descriptor's errors, as the entries without offsets report them
    for over in (dict(head_dim=127), dict(cache_batch_stride=S * RK.KV * RK.D - 1), dict(pos=0), dict(rotary_dim=130),
                 dict(rotary_dim=65)):
        assert lib.b200awq_rope_kv_offset(buf(), QKV, _desc(**over), 4, 2, None) == EINVAL, over
    one = _desc(norm=True)
    one.qk.k_norm_weight = 0                                                                # one norm weight only
    assert lib.b200awq_rope_kv_offset(buf(), QKV, one, 4, 2, None) == EINVAL
    H, KV = RK.H, RK.KV
    assert lib.b200awq_rope_kv_offset(buf(), (H + 2 * KV) * 72, _desc(True, n=(H + 2 * KV) * 72, heads=(H, KV, 72)),
                                      4, 2, None) == EUNSUPPORTED                            # q / k norm, D % 16
    assert lib.b200awq_rope_kv_offset(buf(), QKV, _desc(True, rotary_dim=64), 4, 2, None) == EUNSUPPORTED  # partial


# ---------------------------------------------------------------------------------------------- folding (plan)
QWEN25VL_7B = dict(hid=3584, inter=18944, H=28, KV=4, D=128)


def qwen2_segment(M, hid, inter, H, KV, D):
    """[o + h, norm2, gate|up, silu, down + h, norm1', qkv' (with bias), rope'] of a Qwen2 block (the Qwen2.5-VL
    language model)."""
    n = (H + 2 * KV) * D
    o = linear(buf(), H * D, hid, M=M)
    h = add(o["y"], buf(), hid, M=M)
    n2 = rmsnorm(h["y"], hid, M=M)
    gu = linear(n2["y"], hid, 2 * inter, M=M)
    act = silu(gu["y"], inter, M=M)
    dn = linear(act["y"], inter, hid, M=M)
    out = add(dn["y"], h["y"], hid, M=M)
    n1 = rmsnorm(out["y"], hid, M=M)
    qkv = dict(linear(n1["y"], hid, n, M=M), bias=buf(n * 2))
    rope, _ = RK._rope(qkv["y"], M=M, n=n, heads=(H, KV, D))
    return [o, h, n2, gu, act, dn, out, n1, qkv, rope]


SEGMENTS = {
    "qwen2.5-vl-7b": lambda M: qwen2_segment(M, **QWEN25VL_7B),
    "llama-3-8b": lambda M: RK._segment(M)[0],
    "qwen3-8b": lambda M: QK._segment(M)[0],
}


@pytest.mark.parametrize("model", sorted(SEGMENTS))
@pytest.mark.parametrize("B,T", [(1, 1), (2, 1), (4, 1), (8, 1), (1, 2), (2, 2), (4, 2), (1, 4), (2, 4), (1, 8)])
def test_segment_folds_like_the_segment_without_offsets(model, B, T):
    M = B * T
    seg = SEGMENTS[model](M)
    want = _plan(seg, max_tokens=M)
    assert want == (OK, 4)
    assert _plan(seg[:-1] + [offset(seg[-1], T)[0]], max_tokens=M) == want


@pytest.mark.parametrize("model", sorted(STABLELM))
def test_stablelm_segment_folds_at_one_token(model):
    """LayerNorm staging and partial rotary: the M = 1 LayerNorm kernel's finish reads the offset too."""
    seg = stablelm_segment(model)
    assert _plan(seg) == (OK, 4)
    assert _plan(seg[:-1] + [offset(seg[-1])[0]]) == (OK, 4)


def test_offset_and_seq_len_checks():
    for M, T, code in ((4, 4, OK), (4, 1, OK), (4, 3, EINVAL), (4, 0, EINVAL), (4, -2, EINVAL), (4, 8, EINVAL),
                       (2, 2, OK), (8, 2, OK), (1, 1, OK)):
        for norm in (False, True):
            n1 = rmsnorm(buf(), RK.HID, M=M)
            qkv = linear(n1["y"], RK.HID, RK.QKV, M=M)
            rope, _ = (QK._qkn if norm else RK._rope)(qkv["y"], M=M)
            assert _plan([n1, qkv, offset(rope, T)[0]], max_tokens=8)[0] == code, (M, T, norm)
    n1 = rmsnorm(buf(), RK.HID)
    qkv = linear(n1["y"], RK.HID, RK.QKV)
    rope, _ = RK._rope(qkv["y"])
    assert _plan([n1, qkv, offset(rope, rot_offset=0)[0]])[0] == EINVAL                    # null rot_offset
    assert _plan([n1, qkv, dict(offset(rope)[0], weight=0)])[0] == EINVAL
    # a program created for fewer rows than the step has
    seg = RK._segment(4)[0]
    assert _plan(seg[:-1] + [offset(seg[-1], 2)[0]], max_tokens=2)[0] == EUNSUPPORTED


@pytest.mark.parametrize("B,T", [(1, 1), (4, 1), (2, 2)])
def test_rot_offset_is_a_read_no_op_may_write(B, T):
    """The offsets are read like pos: an op writing any of their B words is rejected, a buffer right after them is
    free, and another ROPE_KV_OFFSET reading them is fine."""
    M = B * T
    HID = RK.HID
    for norm in (False, True):
        offs = buf()
        n1 = rmsnorm(buf(), HID, M=M)
        qkv = linear(n1["y"], HID, RK.QKV, M=M)
        rope, r = (QK._qkn if norm else RK._rope)(qkv["y"], M=M)
        op = offset(rope, T, offs)[0]
        ybytes = M * HID * 2
        for y, code in ((offs, EUNSUPPORTED), (offs + 16 - ybytes, EUNSUPPORTED),
                        (offs + 4 * B, OK), (offs - ybytes, OK)):
            after = linear(buf(), HID, HID, M=M, y=y)
            assert _plan([n1, qkv, op, after], max_tokens=M)[0] == code, (norm, y - offs)
        # two layers sharing pos, freqs and the offsets
        r = r.rope if norm else r
        n1b = rmsnorm(buf(), HID, M=M)
        qkv_b = linear(n1b["y"], HID, RK.QKV, M=M)
        rope_b, _ = (QK._qkn if norm else RK._rope)(qkv_b["y"], M=M, pos=r.pos, freqs=r.freqs)
        assert _plan([n1, qkv, op, n1b, qkv_b, offset(rope_b, T, offs)[0]], max_tokens=M) == (OK, 2), norm


# ROPE_KV's and QK_NORM_ROPE_KV's folding tests with their op builders returning kind 19 at T = 1
def _as_offset(builder):
    def build(*a, **k):
        op, d = builder(*a, **k)
        return offset(op)[0], d
    return build


@pytest.mark.parametrize("name", ["test_folds_without_adding_kernel_ops", "test_argument_validation",
                                  "test_rejected_after_anything_but_a_plain_linear",
                                  "test_rejected_when_qkv_is_not_the_whole_output_or_the_shape_is_off",
                                  "test_rejected_when_another_op_touches_q_out_or_the_caches"])
def test_rope_kv_rules_hold_for_rope_kv_offset(name, monkeypatch):
    monkeypatch.setattr(RK, "_rope", _as_offset(RK._rope))
    getattr(RK, name)()


@pytest.mark.parametrize("name", ["test_folds_without_adding_kernel_ops", "test_argument_validation",
                                  "test_rejected_after_anything_but_a_plain_linear",
                                  "test_rejected_when_qkv_is_not_the_whole_output_or_the_shape_is_off",
                                  "test_rejected_when_another_op_touches_its_outputs_or_writes_its_inputs"])
def test_qk_norm_rope_kv_rules_hold_for_rope_kv_offset(name, monkeypatch):
    monkeypatch.setattr(QK, "_qkn", _as_offset(QK._qkn))
    getattr(QK, name)()


@needs_nvcc
def test_entries_reading_the_offset_keep_their_register_and_spill_budget():
    """The offsets add no kernel entry: every entry with a mode-2 finish reads them and keeps the registers and spills
    it had without them (the M = 1 finish derives the rotary row per pair, program_stream.cuh: sp_rot_row)."""
    want = {"stream_rope_kernel": (167, 0, 0, 0), "stream_layernorm_kernel": (168, 0, 0, 0),
            "stream_qknorm_kernel": (168, 0, 0, 0), "stream_qwen3moe_kernel": (168, 0, 0, 0),
            "stream_deepseek_moe_kernel": (168, 8, 8, 28), "stream_mla_kernel": (168, 16, 12, 28),
            "stream_mla_lora_kernel": (168, 16, 16, 52)}
    found = entries("program.cu", r"stream_(rope|layernorm|qknorm|qwen3moe|deepseek_moe|mla|mla_lora|batch_rope|"
                                  r"batch_qknorm)_kernel")
    assert len(found) == 13, sorted(found)
    for name, got in found.items():
        if m := re.search(r"kernelILi(\d+)E", name):
            assert got == ((165 if m.group(1) == "2" else 162), 0, 0, 0), f"{name}: {got}"
        else:
            key = re.search(r"\d+(stream_\w+?_kernel)", name).group(1)
            assert got == want[key], f"{name}: {got}"
