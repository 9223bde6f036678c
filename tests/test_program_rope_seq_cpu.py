"""Host logic of RoPE + KV-cache append for T tokens per sequence (B200AWQ_OP_ROPE_KV_SEQ / _QK_NORM_ROPE_KV_SEQ,
b200awq_rope_kv_seq / b200awq_qk_norm_rope_kv_seq), checked without a GPU: the constants and exports, the argument
checks of both entries, the folding through b200awq_program_plan (Llama-3-8B, Qwen3-8B and a partial-rotary RMSNorm
segment, the cache extent of B = M / T entries, every rejection) and the register / spill budget of the batched
entries whose finish maps rows to (sequence, position).

ROPE_KV's and QK_NORM_ROPE_KV's own folding tests are run again with their op builders returning the new kinds at
T = 1, which must fold exactly as kinds 6 / 7.  The plan sequences use fake (aligned integer) pointers."""
import ctypes
import re
from functools import partial

import pytest

import test_program_qknorm_cpu as QK
import test_program_rope_cpu as RK
from _fake_ops import buf, linear, plan as _fplan, rmsnorm
from _toolchain import entries, header_constants, needs_nvcc
from autoawq_b200 import _cabi
from autoawq_b200._cabi import lib
from test_program_partial_rope_cpu import layer_norm, llama_segment

OK, EINVAL, EUNSUPPORTED = 0, 1, 2
HID, H, KV, D, S, SMS = 4096, 32, 8, 128, 2048, 132
QKV = (H + 2 * KV) * D
_plan = partial(_fplan, sms=SMS)


def seq(op, T):
    """The ROPE_KV / QK_NORM_ROPE_KV op dict `op` as its _SEQ kind with T tokens per sequence (record: K = T)."""
    kind = {_cabi.OP_ROPE_KV: _cabi.OP_ROPE_KV_SEQ, _cabi.OP_QK_NORM_ROPE_KV: _cabi.OP_QK_NORM_ROPE_KV_SEQ}[op["kind"]]
    return dict(op, kind=kind, K=T)


def test_constants_and_exports():
    assert header_constants("B200AWQ_OP_ROPE_KV_SEQ", "B200AWQ_OP_QK_NORM_ROPE_KV_SEQ") == (
        _cabi.OP_ROPE_KV_SEQ, _cabi.OP_QK_NORM_ROPE_KV_SEQ) == (17, 18)
    for name in ("b200awq_rope_kv_seq", "b200awq_qk_norm_rope_kv_seq"):
        assert name in _cabi.SIGNATURES
        assert getattr(lib, name).restype is ctypes.c_int
    assert ctypes.sizeof(_cabi.Rope) == 72                    # the descriptors are reused unchanged


def test_stand_alone_argument_checks_before_any_cuda_call():
    _, r = RK._rope(buf())
    _, q = QK._qkn(buf())
    for fn, d in ((lib.b200awq_rope_kv_seq, r), (lib.b200awq_qk_norm_rope_kv_seq, q)):
        for M, T in ((4, 0), (4, -1), (4, 3), (6, 4), (1, 2)):
            assert fn(buf(), QKV, d, M, T, None) == EINVAL, (M, T)
        assert fn(None, QKV, d, 4, 2, None) == EINVAL
        assert fn(buf(), QKV, None, 4, 2, None) == EINVAL
        assert fn(buf(), QKV - 1, d, 4, 2, None) == EINVAL        # row pitch under (H + 2 KV) D
        assert fn(buf(), QKV, d, 0, 3, None) == OK                # M = 0: nothing to do
    # the embedded descriptor's errors, as the T = 1 entries report them
    for over, code in ((dict(head_dim=127), EINVAL), (dict(cache_batch_stride=S * KV * D - 1), EINVAL),
                       (dict(pos=0), EINVAL), (dict(rotary_dim=130), EINVAL), (dict(rotary_dim=65), EINVAL)):
        _, bad = RK._rope(buf(), **over)
        assert lib.b200awq_rope_kv_seq(buf(), QKV, bad, 4, 2, None) == code, over
        assert lib.b200awq_rope_kv(buf(), QKV, bad, 4, None) == code, over
    _, q72 = QK._qkn(buf(), n=(H + 2 * KV) * 72, heads=(H, KV, 72))
    assert lib.b200awq_qk_norm_rope_kv_seq(buf(), (H + 2 * KV) * 72, q72, 4, 2, None) == EUNSUPPORTED   # D % 16
    _, qp = QK._qkn(buf(), rotary_dim=64)
    assert lib.b200awq_qk_norm_rope_kv_seq(buf(), QKV, qp, 4, 2, None) == EUNSUPPORTED      # partial rotary
    bad = _cabi.QkNormRope.from_buffer_copy(q)
    bad.k_norm_weight = 0
    assert lib.b200awq_qk_norm_rope_kv_seq(buf(), QKV, bad, 4, 2, None) == EINVAL


# ---------------------------------------------------------------------------------------------- folding (plan)
BT = [(1, 2), (1, 4), (2, 2)]          # (B sequences, T tokens each): M = B T rows


@pytest.mark.parametrize("B,T", BT)
def test_llama_segment_folds_like_rope_kv(B, T):
    M = B * T
    seg, _ = RK._segment(M)
    assert _plan(seg, max_tokens=M) == (OK, 4)
    assert _plan(seg[:-1] + [seq(seg[-1], T)], max_tokens=M) == (OK, 4)


@pytest.mark.parametrize("B,T", BT)
def test_qwen3_segment_folds_like_qk_norm_rope_kv(B, T):
    M = B * T
    seg, _ = QK._segment(M)
    assert _plan(seg, max_tokens=M) == (OK, 4)
    assert _plan(seg[:-1] + [seq(seg[-1], T)], max_tokens=M) == (OK, 4)


@pytest.mark.parametrize("B,T", BT)
def test_partial_rotary_rmsnorm_segment_folds(B, T):
    """StableLM-shaped heads (D = 64, R = 16) in an RMSNorm segment."""
    M = B * T
    seg = llama_segment(M, hid=2048, inter=5632, H=32, KV=32, D=64, R=16)
    assert _plan(seg[:-1] + [seq(seg[-1], T)], max_tokens=M) == (OK, 4)


def test_seq_len_checks():
    for M, T, code in ((4, 4, OK), (4, 1, OK), (4, 3, EINVAL), (4, 0, EINVAL), (4, -2, EINVAL), (4, 8, EINVAL),
                       (2, 2, OK), (8, 2, OK)):
        n1 = rmsnorm(buf(), HID, M=M)
        qkv = linear(n1["y"], HID, QKV, M=M)
        rope, _ = RK._rope(qkv["y"], M=M)
        assert _plan([n1, qkv, seq(rope, T)], max_tokens=8)[0] == code, (M, T)
        qk, _ = QK._qkn(qkv["y"], M=M)
        assert _plan([n1, qkv, seq(qk, T)], max_tokens=8)[0] == code, (M, T)


def test_cache_extent_is_b_entries():
    """The hazard checks see B = M / T cache entries: a buffer right after entry B - 1 is free at T = 2, but inside
    the M entries a ROPE_KV of the same rows would write."""
    M, T = 4, 2
    ent = S * KV * D * 2
    for field in ("k_cache", "v_cache"):
        n1 = rmsnorm(buf(), HID, M=M)
        qkv = linear(n1["y"], HID, QKV, M=M)
        rope, r = RK._rope(qkv["y"], M=M)
        after = linear(buf(), HID, HID, M=M, y=getattr(r, field) + (M // T) * ent)
        assert _plan([n1, qkv, seq(rope, T), after], max_tokens=M) == (OK, 2), field
        assert _plan([n1, qkv, rope, after], max_tokens=M)[0] == EUNSUPPORTED, field
        inside = linear(buf(), HID, HID, M=M, y=getattr(r, field) + (M // T) * ent - 64)
        assert _plan([n1, qkv, seq(rope, T), inside], max_tokens=M)[0] == EUNSUPPORTED, field


def test_rejections_of_multi_token_steps():
    M, T = 4, 2
    # a program created for fewer rows than the step has (an M = 1-sized program, or max_tokens < B T)
    seg, _ = RK._segment(M)
    seg = seg[:-1] + [seq(seg[-1], T)]
    assert _plan(seg, max_tokens=1)[0] == EUNSUPPORTED
    assert _plan(seg, max_tokens=2)[0] == EUNSUPPORTED
    # LayerNorm segments (StableLM with its LayerNorms, Command-R, StarCoder2) replay per op at M > 1
    ln = layer_norm(buf(), 2560, M=M)
    qkv = linear(ln["y"], 2560, 96 * 80, M=M)
    rope, _ = RK._rope(qkv["y"], M=M, n=96 * 80, heads=(32, 32, 80), rotary_dim=20)
    assert _plan([ln, qkv, seq(rope, T)], max_tokens=M)[0] == EUNSUPPORTED
    # a MoE block in the program
    d = _cabi.Moe()
    d.E, d.top_k, d.renormalize, d.group_size, d.H, d.I, d.block_size = 8, 2, 1, 128, HID, 512, 16
    d.sorted_len = 2 * M + 8 * 15
    d.gate_weight = buf()
    for f, _ in _cabi.Moe._fields_[9:]:
        setattr(d, f, buf())
    xn = rmsnorm(buf(), HID, M=M)
    moe = dict(kind=_cabi.OP_SPARSE_MOE, M=M, K=HID, N=HID, x=xn["y"], y=buf(), weight=ctypes.addressof(d))
    n1 = rmsnorm(buf(), HID, M=M)
    qkv = linear(n1["y"], HID, QKV, M=M)
    rope, _ = RK._rope(qkv["y"], M=M)
    assert _plan([xn, moe, n1, qkv, seq(rope, T)], max_tokens=M)[0] == EUNSUPPORTED
    # an MLA op in the program
    m = _cabi.Mla()
    m.n_heads, m.nope_dim, m.rope_dim, m.v_dim, m.kv_lora_rank, m.cache_len, m.freqs_len = 16, 128, 64, 128, 512, S, S
    m.v_head_stride = 128
    m.k_batch_stride, m.v_batch_stride = S * 16 * 192, S * 16 * 128
    m.pos, m.freqs, m.q_out, m.k_cache, m.v_cache = buf(), buf(S * 64 * 4), buf(), buf(8 * S * 16 * 192 * 2), buf()
    kvb = linear(buf(), 512, 16 * 256, M=M)
    mla = dict(kind=_cabi.OP_MLA_KV, M=M, N=16 * 256, ldx=16 * 256, x=kvb["y"], weight=ctypes.addressof(m))
    assert _plan([n1, qkv, seq(rope, T), kvb, mla], max_tokens=M)[0] == EUNSUPPORTED


# ROPE_KV's and QK_NORM_ROPE_KV's folding tests with their op builders returning kind 17 / 18 at T = 1
def _as_seq(builder):
    def build(*a, **k):
        op, d = builder(*a, **k)
        return seq(op, 1), d
    return build


@pytest.mark.parametrize("name", ["test_folds_without_adding_kernel_ops", "test_argument_validation",
                                  "test_rejected_after_anything_but_a_plain_linear",
                                  "test_rejected_when_qkv_is_not_the_whole_output_or_the_shape_is_off",
                                  "test_rejected_when_another_op_touches_q_out_or_the_caches"])
def test_rope_kv_rules_hold_for_rope_kv_seq(name, monkeypatch):
    monkeypatch.setattr(RK, "_rope", _as_seq(RK._rope))
    getattr(RK, name)()


@pytest.mark.parametrize("name", ["test_folds_without_adding_kernel_ops", "test_argument_validation",
                                  "test_rejected_after_anything_but_a_plain_linear",
                                  "test_rejected_when_qkv_is_not_the_whole_output_or_the_shape_is_off",
                                  "test_rejected_when_another_op_touches_its_outputs_or_writes_its_inputs"])
def test_qk_norm_rope_kv_rules_hold_for_qk_norm_rope_kv_seq(name, monkeypatch):
    monkeypatch.setattr(QK, "_qkn", _as_seq(QK._qkn))
    getattr(QK, name)()


@needs_nvcc
def test_batched_rope_entries_register_and_spill_budget():
    """The per-row (sequence, position) map of the batched finish costs no register: stream_batch_rope_kernel and
    stream_batch_qknorm_kernel keep the counts they had with one position per step (165 at MT = 2, 162 at 4 and 8),
    and nothing spills."""
    found = entries("program.cu", r"stream_batch_(rope|qknorm)_kernel")
    assert len(found) == 6, sorted(found)
    for name, (regs, stack, st, ld) in found.items():
        mt = int(re.search(r"kernelILi(\d+)E", name).group(1))
        assert regs == (165 if mt == 2 else 162), f"{name}: {regs} registers"
        assert (stack, st, ld) == (0, 0, 0), f"{name}: stack {stack}, spills {st} / {ld}"
