"""Host logic of RoPE + KV-cache append in decode programs (B200AWQ_OP_ROPE_KV), checked without a GPU: the stream
format's rotary column pairing (mode 2), the folding rules through b200awq_program_plan, the ctypes descriptor layout
and the register / spill budget of the new kernel entries.

The plan sequences use fake (aligned integer) pointers: the folding only compares addresses.  Shapes are Llama-3-8B's
(hidden 4096, 32 q heads, 8 kv heads, head_dim 128, intermediate 14336)."""
import ctypes
from functools import partial

import numpy as np
import pytest

from _fake_ops import add, buf, linear, rmsnorm, silu
from _fake_ops import plan as _fplan
from _toolchain import entries, header_constants, header_layout, mirror_layout, needs_nvcc
from autoawq_b200 import _cabi
from oracle import awq_oracle as O
from oracle import stream_format as SF

OK, EINVAL, EUNSUPPORTED = 0, 1, 2
HID, INTER, H, KV, D, SMS = 4096, 14336, 32, 8, 128, 132
QKV = (H + 2 * KV) * D
S = 2048
_plan = partial(_fplan, sms=SMS)


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


def test_rope_struct_matches_header():
    assert header_layout(_cabi.Rope, "b200awq_rope_t") == mirror_layout(_cabi.Rope)
    assert header_constants("B200AWQ_OP_ROPE_KV") == (_cabi.OP_ROPE_KV,) == (6,)


# ---------------------------------------------------------------------------------------------- folding (plan)
_KEEP = []


def _rope(qkv, M=1, n=QKV, heads=(H, KV, D), **over):
    """A ROPE_KV op on qkv with its own q_out / caches / pos / freqs; `over` replaces descriptor fields."""
    h, kv, d = heads
    r = _cabi.Rope()
    r.n_heads, r.n_kv_heads, r.head_dim, r.cache_len, r.freqs_len = h, kv, d, S, S
    r.cache_batch_stride = S * kv * d
    cache = 8 * S * kv * d * 2
    r.pos, r.freqs, r.q_out = buf(), buf(S * d * 4), buf()
    r.k_cache, r.v_cache = buf(cache), buf(cache)
    for f, v in over.items():
        setattr(r, f, v)
    _KEEP.append(r)
    return dict(kind=_cabi.OP_ROPE_KV, M=M, N=n, ldx=n, x=qkv, weight=ctypes.addressof(r)), r


def _segment(M=1):
    """[o + h, norm2, gate|up, silu, down + h, norm1', qkv', rope'] of a Llama-3-8B layer."""
    attn, h_in = buf(), buf()
    o = linear(attn, HID, HID, M=M)
    h = add(o["y"], h_in, HID, M=M)
    n2 = rmsnorm(h["y"], HID, M=M)
    gu = linear(n2["y"], HID, 2 * INTER, M=M)
    act = silu(gu["y"], INTER, M=M)
    dn = linear(act["y"], INTER, HID, M=M)
    out = add(dn["y"], h["y"], HID, M=M)
    n1 = rmsnorm(out["y"], HID, M=M)
    qkv = linear(n1["y"], HID, QKV, M=M)
    rope, r = _rope(qkv["y"], M=M)
    return [o, h, n2, gu, act, dn, out, n1, qkv, rope], r


def test_folds_without_adding_kernel_ops():
    x = buf()
    n1 = rmsnorm(x, HID)
    qkv = linear(n1["y"], HID, QKV)
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
    o = linear(qkv["y"], HID, HID)
    assert _plan([n1, qkv, rope, o]) == (OK, 2)


def test_argument_validation():
    qkv = linear(buf(), HID, QKV)
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
    x, r = buf(), buf()
    n1 = rmsnorm(x, QKV)
    rope, _ = _rope(n1["y"])
    assert _plan([n1, rope, linear(n1["y"], QKV, HID)])[0] == EUNSUPPORTED              # after a glue op
    qkv = linear(x, HID, QKV)
    a = add(qkv["y"], r, QKV)
    rope, _ = _rope(a["y"])
    assert _plan([qkv, a, rope])[0] == EUNSUPPORTED                              # after an add (the linear carries it)
    qkv = linear(x, HID, QKV)
    rope, _ = _rope(qkv["y"])
    rope2, _ = _rope(qkv["y"])
    assert _plan([qkv, rope, rope2])[0] == EUNSUPPORTED                          # after another ROPE_KV
    assert _plan([rope])[0] == EUNSUPPORTED                                      # first op
    # a gate|up whose product SiLU*mul reads (its row would hold silu(gate) * up)
    gu = linear(x, HID, QKV)
    rope, _ = _rope(gu["y"])
    act = silu(gu["y"], QKV // 2)
    assert _plan([gu, rope, act, linear(act["y"], QKV // 2, HID)])[0] == EUNSUPPORTED
    # a sparse-MoE block's down op
    E, k, Hm, Im = 8, 2, QKV, 512
    d = _cabi.Moe()
    d.E, d.top_k, d.renormalize, d.group_size, d.H, d.I, d.block_size = E, k, 1, 128, Hm, Im, 16
    d.sorted_len = k + E * 15
    d.gate_weight = buf()
    for f, _ in _cabi.Moe._fields_[9:]:
        setattr(d, f, buf())
    xn = rmsnorm(x, Hm)
    moe = dict(kind=_cabi.OP_SPARSE_MOE, M=1, K=Hm, N=Hm, x=xn["y"], y=buf(), weight=ctypes.addressof(d))
    rope, _ = _rope(moe["y"])
    assert _plan([xn, moe])[0] == OK
    assert _plan([xn, moe, rope])[0] == EUNSUPPORTED


def test_rejected_when_qkv_is_not_the_whole_output_or_the_shape_is_off():
    x = buf()
    qkv = linear(x, HID, QKV)
    rope, _ = _rope(qkv["y"] + 256, n=QKV - 128)
    assert _plan([qkv, rope])[0] == EUNSUPPORTED                                 # a slice of the linear's output
    rope, _ = _rope(buf())
    assert _plan([qkv, rope])[0] == EUNSUPPORTED                                 # not the linear's output at all
    wide = linear(x, HID, QKV + 128)
    rope, _ = _rope(wide["y"])
    assert _plan([wide, rope])[0] == EUNSUPPORTED                                # N != (H + 2 KV) D
    rope, _ = _rope(wide["y"], n=QKV + 128)
    assert _plan([wide, rope])[0] == EUNSUPPORTED
    d72 = (H + 2 * KV) * 72                                                      # D % 16 != 0
    q72 = linear(x, HID, d72)
    rope, _ = _rope(q72["y"], n=d72, heads=(H, KV, 72))
    assert _plan([q72, rope])[0] == EUNSUPPORTED
    d64 = (H + 2 * KV) * 64
    q64 = linear(x, HID, d64)
    rope, _ = _rope(q64["y"], n=d64, heads=(H, KV, 64))
    assert _plan([q64, rope])[0] == OK


def test_rejected_when_another_op_touches_q_out_or_the_caches():
    x = buf()
    for field in ("q_out", "k_cache", "v_cache"):
        n1 = rmsnorm(x, HID)
        qkv = linear(n1["y"], HID, QKV)
        rope, r = _rope(qkv["y"])
        target = getattr(r, field)
        # a later linear reads it
        assert _plan([n1, qkv, rope, linear(target, HID, HID)])[0] == EUNSUPPORTED, field
        # a later linear writes it
        assert _plan([n1, qkv, rope, linear(buf(), HID, HID, y=target)])[0] == EUNSUPPORTED, field
        # an earlier glue op writes it / reads it
        assert _plan([rmsnorm(buf(), HID, y=target), linear(target, HID, HID), n1, qkv, rope])[0] == EUNSUPPORTED, field
        nt = rmsnorm(target, HID)
        assert _plan([nt, linear(nt["y"], HID, HID), n1, qkv, rope])[0] == EUNSUPPORTED, field
        # an add uses it as its residual
        o = linear(buf(), HID, HID)
        assert _plan([n1, qkv, rope, o, add(o["y"], target, HID)])[0] == EUNSUPPORTED, field
        # a second ROPE_KV writes into the same buffer
        n1b = rmsnorm(buf(), HID)
        qkv_b = linear(n1b["y"], HID, QKV)
        rope_b, _ = _rope(qkv_b["y"], **{field: target})
        assert _plan([n1, qkv, rope, n1b, qkv_b, rope_b])[0] == EUNSUPPORTED, field
        # the qkv linear's own output (in place)
        rope_ip, _ = _rope(qkv["y"], **{field: qkv["y"]})
        assert _plan([n1, qkv, rope_ip])[0] == EUNSUPPORTED, field
    # a program op writing the position
    n1 = rmsnorm(x, HID)
    qkv = linear(n1["y"], HID, QKV)
    rope, r = _rope(qkv["y"])
    assert _plan([n1, qkv, rope, linear(buf(), HID, HID, y=r.pos)])[0] == EUNSUPPORTED
    # two layers sharing pos and freqs fold
    n1b = rmsnorm(buf(), HID)
    qkv_b = linear(n1b["y"], HID, QKV)
    rope_b, _ = _rope(qkv_b["y"], pos=r.pos, freqs=r.freqs)
    assert _plan([n1, qkv, rope, n1b, qkv_b, rope_b]) == (OK, 2)


@needs_nvcc
def test_rope_kernels_register_and_spill_budget():
    """One CTA per SM: the rope entries (288 threads) fit the register file and spill nothing."""
    found = entries("program.cu", r"rope_kernel")
    assert len(found) == 4, found          # stream_rope_kernel, stream_batch_rope_kernel<2|4|8>
    for name, (regs, stack, st, ld) in found.items():
        assert regs * (32 + 32 * 8) <= 65536, f"{name}: {regs} registers x 288 threads"
        assert st == 0 and ld == 0 and stack == 0, f"{name}: spills {st} / {ld}, stack {stack}"
