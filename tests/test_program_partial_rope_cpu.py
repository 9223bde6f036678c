"""Host logic of partial rotary in RoPE + KV-cache append (b200awq_rope_t.rotary_dim, StableLM), checked without a GPU:
the descriptor layout, the column map of stream mode 2 through the stream-format oracle, the folding of StableLM and
Llama-shaped segments through b200awq_program_plan, the argument checks, and the register / spill budget of every
kernel entry that compiles the mode-2 finish.

The plan sequences use fake (aligned integer) pointers: the folding only compares addresses."""
import ctypes
from functools import partial

import numpy as np
import pytest

from _fake_ops import add, buf, linear, plan as _fplan, rmsnorm, silu
from _toolchain import entries, header_layout, mirror_layout, needs_nvcc
from autoawq_b200 import _cabi
from autoawq_b200._cabi import lib
from oracle import awq_oracle as O
from oracle import stream_format as SF
from test_program_rope_cpu import rotary_columns

OK, EINVAL, EUNSUPPORTED = 0, 1, 2
SMS, S = 132, 2048
_plan = partial(_fplan, sms=SMS)
_KEEP = []
GEOMETRIES = [(64, 16), (80, 20), (160, 40), (128, 64), (128, 128)]   # (head_dim, rotary_dim)

# name: (hidden, q heads, kv heads, head_dim, rotary_dim, intermediate, qkv bias)
STABLELM = {
    "stablelm-2-1.6b": (2048, 32, 32, 64, 16, 5632, True),
    "stablelm-3b-4e1t": (2560, 32, 32, 80, 20, 6912, False),
}


def partial_rotary_columns(N, D, R):
    """[S, 16] original columns of mode 2 with R rotated columns per head (include/b200awq.h, b200awq_rope_t): set s of
    head h = s // (D / 16), t = s % (D / 16), holds the head's pairs p = 8 t + g; pair p < R/2 is (p, p + R/2), pair
    p >= R/2 is (R + q, R + q + (D - R)/2) with q = p - R/2."""
    s = np.arange(N // 16)[:, None]
    g = np.arange(8)[None, :]
    h, p = s // (D // 16), 8 * (s % (D // 16)) + g
    rot = p < R // 2
    lo = np.where(rot, p, p + R // 2)
    hi = np.where(rot, p + R // 2, p + R // 2 + (D - R) // 2)
    return np.concatenate([h * D + lo, h * D + hi], axis=1)


def test_rope_struct_has_rotary_dim_in_place_of_its_padding():
    layout = header_layout(_cabi.Rope, "b200awq_rope_t")
    assert layout == mirror_layout(_cabi.Rope)
    assert layout["sizeof"] == 72 and layout["rotary_dim"] == 20 and layout["cache_batch_stride"] == 24


@pytest.mark.parametrize("D,R", GEOMETRIES)
def test_column_map(D, R):
    N = 6 * D
    cols = partial_rotary_columns(N, D, R)
    assert sorted(cols.reshape(-1).tolist()) == list(range(N))            # every column once
    lo, hi = cols[:, :8] % D, cols[:, 8:] % D
    assert np.array_equal(cols[:, :8] // D, cols[:, 8:] // D)             # both columns in one head
    rot = lo < R // 2
    assert rot.sum() == 6 * R // 2                                        # R/2 rotated pairs per head
    assert np.array_equal(hi[rot], lo[rot] + R // 2)
    assert np.all(lo[~rot] >= R) and np.array_equal(hi[~rot], lo[~rot] + (D - R) // 2)
    if R == D:
        assert np.array_equal(cols, rotary_columns(N, D))                 # full rotary: today's pairing


@pytest.mark.parametrize("D,R", GEOMETRIES)
def test_partial_rotary_stream_reproduces_dense_contraction(D, R, monkeypatch):
    orig = SF.set_columns
    monkeypatch.setattr(SF, "set_columns",
                        lambda n, mode: partial_rotary_columns(n, D, R) if mode == 2 else orig(n, mode))
    K, N, G = 256, 3 * D, 64
    c = O.make_case(K, N, G, seed=D + R, raw=True)
    st = SF.pack_stream(c["qweight"], c["qzeros"], c["scales"], G, 2)
    assert st.size == SF.stream_bytes(K, N, G)
    iw, iz = SF.unpack_gemm_ints(c["qweight"], c["qzeros"])
    w = (iw.astype(np.float64) - np.repeat(iz.astype(np.float64), G, axis=0)) * \
        np.repeat(c["scales"].astype(np.float64), G, axis=0)
    x = np.random.default_rng(3).standard_normal(K).astype(np.float16)
    np.testing.assert_allclose(SF.simulate_gemv(st, K, N, G, x, 2), x.astype(np.float64) @ w, rtol=1e-9, atol=1e-9)


# ---------------------------------------------------------------------------------------------- folding (plan)
def layer_norm(x, K, M=1):
    return dict(kind=_cabi.OP_LAYER_NORM, M=M, K=K, eps=1e-5, x=x, weight=buf(K * 2), bias=buf(K * 2), y=buf(M * K * 2))


def _rope(qkv, H, KV, D, R, M=1, qk_norm=False, **over):
    r = _cabi.Rope()
    r.n_heads, r.n_kv_heads, r.head_dim, r.rotary_dim, r.cache_len, r.freqs_len = H, KV, D, R, S, S
    r.cache_batch_stride = S * KV * D
    r.pos, r.freqs, r.q_out = buf(), buf(S * D * 4), buf(M * H * D * 2)
    r.k_cache, r.v_cache = buf(8 * S * KV * D * 2), buf(8 * S * KV * D * 2)
    for f, v in over.items():
        setattr(r, f, v)
    n = (H + 2 * KV) * D
    if qk_norm:
        q = _cabi.QkNormRope()
        q.rope, q.q_norm_weight, q.k_norm_weight, q.eps = r, buf(D * 2), buf(D * 2), 1e-6
        _KEEP.append(q)
        return dict(kind=_cabi.OP_QK_NORM_ROPE_KV, M=M, N=n, ldx=n, x=qkv, weight=ctypes.addressof(q)), q.rope
    _KEEP.append(r)
    return dict(kind=_cabi.OP_ROPE_KV, M=M, N=n, ldx=n, x=qkv, weight=ctypes.addressof(r)), r


def stablelm_segment(model, M=1):
    """o + x -> h, layer_norm(h), gate|up, silu_and_mul, down + h -> x', layer_norm(x'), qkv', rope_kv_cache."""
    hid, H, KV, D, R, inter, _ = STABLELM[model]
    o = linear(buf(), H * D, hid, M=M)
    h = add(o["y"], buf(), hid, M=M)
    n2 = layer_norm(h["y"], hid, M=M)
    gu = linear(n2["y"], hid, 2 * inter, M=M)
    act = silu(gu["y"], inter, M=M)
    dn = linear(act["y"], inter, hid, M=M)
    out = add(dn["y"], h["y"], hid, M=M)
    n1 = layer_norm(out["y"], hid, M=M)
    qkv = linear(n1["y"], hid, (H + 2 * KV) * D, M=M)
    rope, _ = _rope(qkv["y"], H, KV, D, R, M=M)
    return [o, h, n2, gu, act, dn, out, n1, qkv, rope]


def llama_segment(M, hid=2048, inter=5632, H=32, KV=8, D=128, R=64):
    """The RMSNorm segment of test_program_rope_cpu with rotary_dim R < D."""
    o = linear(buf(), H * D, hid, M=M)
    h = add(o["y"], buf(), hid, M=M)
    n2 = rmsnorm(h["y"], hid, M=M)
    gu = linear(n2["y"], hid, 2 * inter, M=M)
    act = silu(gu["y"], inter, M=M)
    dn = linear(act["y"], inter, hid, M=M)
    out = add(dn["y"], h["y"], hid, M=M)
    n1 = rmsnorm(out["y"], hid, M=M)
    qkv = linear(n1["y"], hid, (H + 2 * KV) * D, M=M)
    rope, _ = _rope(qkv["y"], H, KV, D, R, M=M)
    return [o, h, n2, gu, act, dn, out, n1, qkv, rope]


@pytest.mark.parametrize("model", sorted(STABLELM))
def test_stablelm_segments_fold_into_four_kernel_ops(model):
    seg = stablelm_segment(model)
    assert _plan(seg[:-1]) == (OK, 4)
    assert _plan(seg) == (OK, 4)


@pytest.mark.parametrize("M", [2, 4, 8])
def test_rmsnorm_segment_with_partial_rotary_folds_batched(M):
    assert _plan(llama_segment(M), max_tokens=M) == (OK, 4)


def test_rotary_dim_checks():
    H, KV, D = 32, 32, 80
    qkv = linear(buf(), 2560, (H + 2 * KV) * D)
    for R in (0, 2, 20, 78, 80):
        rope, _ = _rope(qkv["y"], H, KV, D, R)
        assert _plan([qkv, rope]) == (OK, 1), R
    for R in (-2, 19, 82, 160):
        rope, _ = _rope(qkv["y"], H, KV, D, R)
        assert _plan([qkv, rope])[0] == EINVAL, R
    # q / k norm with partial rotary: no model combines them
    qkv = linear(buf(), 4096, 48 * 128)
    rope, _ = _rope(qkv["y"], 32, 8, 128, 64, qk_norm=True)
    assert _plan([qkv, rope])[0] == EUNSUPPORTED
    for R in (0, 128):
        rope, _ = _rope(qkv["y"], 32, 8, 128, R, qk_norm=True)
        assert _plan([qkv, rope]) == (OK, 1), R


def test_stand_alone_entries_check_rotary_dim_before_any_cuda_call():
    H, KV, D = 4, 2, 64
    qkv = buf()
    _, r = _rope(qkv, H, KV, D, 33)
    assert lib.b200awq_rope_kv(qkv, (H + 2 * KV) * D, ctypes.byref(r), 1, None) == EINVAL
    r.rotary_dim = 66
    assert lib.b200awq_rope_kv(qkv, (H + 2 * KV) * D, ctypes.byref(r), 1, None) == EINVAL
    q = _cabi.QkNormRope()
    r.rotary_dim = 32
    q.rope, q.q_norm_weight, q.k_norm_weight, q.eps = r, buf(), buf(), 1e-6
    assert lib.b200awq_qk_norm_rope_kv(qkv, (H + 2 * KV) * D, ctypes.byref(q), 1, None) == EUNSUPPORTED
    pack = lib.b200awq_stream_pack_partial_rotary
    for R in (-2, 15, 66):
        assert pack(buf(), buf(), buf(), buf(), 256, 8 * 64, 128, 64, R, None) == EINVAL, R
    assert pack(buf(), buf(), buf(), buf(), 256, 8 * 72, 128, 72, 16, None) == EUNSUPPORTED   # D % 16 != 0


def test_frequency_table_is_sized_by_the_rotary_dim():
    """A partial table holds S_f x R / 2 pairs: a buffer right after it does not overlap it."""
    H, KV, D, R = 32, 32, 80, 20
    x = buf()
    n1 = rmsnorm(x, 2560)
    qkv = linear(n1["y"], 2560, (H + 2 * KV) * D)
    freqs = buf(S * D * 4)
    rope, _ = _rope(qkv["y"], H, KV, D, R, freqs=freqs)
    after = linear(buf(), 2560, 2560, y=freqs + S * R * 4)
    assert _plan([n1, qkv, rope, after]) == (OK, 2)
    inside = linear(buf(), 2560, 2560, y=freqs + S * R * 4 - 64)
    assert _plan([n1, qkv, rope, inside])[0] == EUNSUPPORTED


@needs_nvcc
def test_mode2_finish_entries_register_and_spill_budget():
    """One 288-thread CTA per SM for every entry that compiles the mode-2 finish.  The MLA and DeepSeek-MoE entries
    spilled before partial rotary (DESIGN.md 3.5i, 3.5k) and keep exactly those spills; every other entry spills
    nothing."""
    names = (r"stream_rope_kernel", r"stream_qknorm_kernel", r"stream_layernorm_kernel", r"stream_qwen3moe_kernel",
             r"stream_deepseek_moe_kernel", r"stream_mla_kernel", r"stream_mla_lora_kernel",
             r"stream_batch_rope_kernel", r"stream_batch_qknorm_kernel")
    found = entries("program.cu", "|".join(names))
    assert len(found) == 13, sorted(found)
    known = {"stream_deepseek_moe_kernel": (8, 8, 28), "stream_mla_kernel": (16, 12, 28),
             "stream_mla_lora_kernel": (16, 16, 52)}
    for name, (regs, stack, st, ld) in found.items():
        assert regs * (32 + 8 * 32) <= 65536, f"{name}: {regs} registers x 288 threads"
        want = next((v for k, v in known.items() if k in name), (0, 0, 0))
        assert (stack, st, ld) == want, f"{name}: stack {stack}, spills {st} / {ld}"
