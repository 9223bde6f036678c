"""Host logic of depth-scaled residual adds in decode programs (B200AWQ_OP_SCALED_ADD: MiniCPM, MiniCPM3, Granite),
checked without a GPU: the ABI constant, the argument checks, the folding of whole Granite / MiniCPM / MiniCPM3
segments through b200awq_program_plan (exactly the kernel ops of the same segment with plain adds), and every rule that
sends a sequence back to the per-op path.

The sequences use fake (aligned integer) pointers: the folding only compares addresses.  The geometries are test shapes
after the public configs (Granite-3.1-8B / 2B, MiniCPM-2B, MiniCPM3-4B)."""
import ctypes
import math

import pytest

from _fake_ops import add, buf, linear, plan, rmsnorm, silu
from _toolchain import header_constants
from autoawq_b200 import _cabi
from test_program_mla_lora_cpu import lora_chain

OK, EINVAL, EUNSUPPORTED = 0, 1, 2
SMS = 132
S = 2048
# hidden, q heads, kv heads, head dim, intermediate
GRANITE_8B = dict(HID=4096, H=32, KV=8, D=128, INTER=12800)
GRANITE_2B = dict(HID=2048, H=32, KV=8, D=64, INTER=8192)
MINICPM_2B = dict(HID=2304, H=36, KV=36, D=64, INTER=5760)
MINICPM3_4B = dict(H=40, DN=64, DR=32, DV=64, C=256, CQ=768, HID=2560, INTER=6400)
ALPHA = 1.4 / math.sqrt(40)
_KEEP = []


def scaled_add(residual, y, K, M=1, alpha=ALPHA, out=None):
    return dict(kind=_cabi.OP_SCALED_ADD, M=M, K=K, eps=alpha, x=residual, weight=y,
                y=buf(M * K * 2) if out is None else out)


def _rope(qkv, g, M):
    r = _cabi.Rope()
    r.n_heads, r.n_kv_heads, r.head_dim, r.cache_len, r.freqs_len = g["H"], g["KV"], g["D"], S, S
    r.cache_batch_stride = S * g["KV"] * g["D"]
    cache = 8 * S * g["KV"] * g["D"] * 2
    r.pos, r.freqs, r.q_out = buf(), buf(S * g["D"] * 4), buf(8 * g["H"] * g["D"] * 2)
    r.k_cache, r.v_cache = buf(cache), buf(cache)
    _KEEP.append(r)
    n = (g["H"] + 2 * g["KV"]) * g["D"]
    return dict(kind=_cabi.OP_ROPE_KV, M=M, N=n, ldx=n, x=qkv, weight=ctypes.addressof(r))


def segment(g, M=1, res=scaled_add):
    """[o, scaled_add, norm2, gate|up, silu, down, scaled_add, norm1', qkv', rope'] of a Granite / MiniCPM layer."""
    HID, I = g["HID"], g["INTER"]
    QKV = (g["H"] + 2 * g["KV"]) * g["D"]
    o = linear(buf(M * g["H"] * g["D"] * 2), g["H"] * g["D"], HID, M=M)
    h = res(buf(M * HID * 2), o["y"], HID, M=M)
    n2 = rmsnorm(h["y"], HID, M=M)
    gu = linear(n2["y"], HID, 2 * I, M=M)
    act = silu(gu["y"], I, M=M)
    dn = linear(act["y"], I, HID, M=M)
    out = res(h["y"], dn["y"], HID, M=M)
    n1 = rmsnorm(out["y"], HID, M=M)
    qkv = linear(n1["y"], HID, QKV, M=M)
    return [o, h, n2, gu, act, dn, out, n1, qkv, _rope(qkv["y"], g, M)]


def minicpm3_segment(M=1, res=scaled_add):
    """[o, scaled_add, norm2, gate|up, silu, down, scaled_add] then the q-LoRA MLA chain of the next layer."""
    g = MINICPM3_4B
    HID, I = g["HID"], g["INTER"]
    o = linear(buf(M * g["H"] * g["DV"] * 2), g["H"] * g["DV"], HID, M=M)
    h = res(buf(M * HID * 2), o["y"], HID, M=M, alpha=1.4 / math.sqrt(62))
    n2 = rmsnorm(h["y"], HID, M=M)
    gu = linear(n2["y"], HID, 2 * I, M=M)
    act = silu(gu["y"], I, M=M)
    dn = linear(act["y"], I, HID, M=M)
    out = res(h["y"], dn["y"], HID, M=M, alpha=1.4 / math.sqrt(62))
    chain, d = lora_chain(g, M, x=out["y"])
    _KEEP.append(d)                      # the ops name the descriptor by address
    return [o, h, n2, gu, act, dn, out] + chain


def _plain(residual, y, K, M=1, alpha=None):
    return add(y, residual, K, M=M)


def test_op_scaled_add_matches_header():
    assert header_constants("B200AWQ_OP_SCALED_ADD") == (_cabi.OP_SCALED_ADD,) == (20,)


@pytest.mark.parametrize("g", [GRANITE_8B, GRANITE_2B, MINICPM_2B], ids=["granite8b", "granite2b", "minicpm2b"])
def test_segments_fold_into_the_kernel_ops_of_plain_adds(g):
    assert plan(segment(g), sms=SMS) == (OK, 4)
    assert plan(segment(g, res=_plain), sms=SMS) == (OK, 4)
    for M in (2, 4):
        assert plan(segment(g, M=M), max_tokens=4, sms=SMS) == (OK, 4), M


def test_minicpm3_segment():
    assert plan(minicpm3_segment(), sms=SMS) == (OK, 6)
    assert plan(minicpm3_segment(res=_plain), sms=SMS) == (OK, 6)
    # batched MLA programs replay per op
    assert plan(minicpm3_segment(M=2), max_tokens=2, sms=SMS)[0] == EUNSUPPORTED


def _rc(ops, **kw):
    return plan(ops, sms=SMS, **kw)[0]


def test_argument_validation():
    K = 4096
    lin = linear(buf(), K, K)
    r = buf()
    assert _rc([lin, scaled_add(r, lin["y"], K)]) == OK
    for alpha in (math.inf, -math.inf, math.nan):
        assert _rc([lin, scaled_add(r, lin["y"], K, alpha=alpha)]) == EINVAL, alpha
    assert _rc([lin, scaled_add(0, lin["y"], K)]) == EINVAL
    assert _rc([lin, scaled_add(r, 0, K)]) == EINVAL
    assert _rc([lin, dict(scaled_add(r, lin["y"], K), y=0)]) == EINVAL
    assert _rc([lin, scaled_add(r, lin["y"], 0)]) == EINVAL
    assert _rc([lin, scaled_add(r, lin["y"], K - 4)]) == EUNSUPPORTED             # K % 8
    assert _rc([lin, scaled_add(r + 8, lin["y"], K)]) == EUNSUPPORTED             # not 16-byte aligned
    assert _rc([lin, scaled_add(r, lin["y"], K, alpha=0.0)]) == OK
    assert _rc([lin, scaled_add(r, lin["y"], K, alpha=-3.0e38)]) == OK


def test_operands_swapped():
    """The scaled operand must be the producer's output; ADD takes either order, SCALED_ADD does not."""
    K = 4096
    lin = linear(buf(), K, K)
    r = buf()
    assert _rc([lin, add(lin["y"], r, K)]) == OK
    assert _rc([lin, add(r, lin["y"], K)]) == OK
    assert _rc([lin, scaled_add(lin["y"], r, K)]) == EUNSUPPORTED
    assert _rc([lin, scaled_add(buf(), buf(), K)]) == EUNSUPPORTED                 # both external
    assert _rc([lin, scaled_add(lin["y"], lin["y"], K)]) == EUNSUPPORTED           # no residual


def test_in_place_output():
    K = 4096
    lin = linear(buf(), K, K)
    r = buf()
    assert _rc([lin, scaled_add(r, lin["y"], K, out=lin["y"])]) == EUNSUPPORTED
    lin = linear(buf(), K, K)
    assert _rc([lin, scaled_add(r, lin["y"], K, out=r)]) == EUNSUPPORTED


def test_output_overlaps_the_producers_source():
    K = 4096
    x = buf()
    lin = linear(x, K, K)
    assert _rc([lin, scaled_add(buf(), lin["y"], K, out=x)]) == EUNSUPPORTED
    nm = rmsnorm(buf(), K)
    lin = linear(nm["y"], K, K)
    assert _rc([nm, lin, scaled_add(buf(), lin["y"], K, out=nm["x"])]) == EUNSUPPORTED


def test_residual_window():
    K = 4096
    chain = [linear(buf(), K, K)]
    for _ in range(5):
        chain.append(linear(chain[-1]["y"], K, K))
    assert _rc(chain[:5] + [scaled_add(chain[0]["y"], chain[4]["y"], K)]) == OK          # four kernel ops back
    assert _rc(chain + [scaled_add(chain[0]["y"], chain[5]["y"], K)]) == EUNSUPPORTED    # five: outside the window


def test_after_a_glue_op_an_add_or_a_moe_block():
    K = 4096
    nm = rmsnorm(buf(), K)
    assert _rc([nm, scaled_add(buf(), nm["y"], K), linear(nm["y"], K, K)]) == EUNSUPPORTED
    lin = linear(buf(), K, K)
    a1 = scaled_add(buf(), lin["y"], K)
    assert _rc([lin, a1, scaled_add(buf(), a1["y"], K)]) == EUNSUPPORTED
    # after a sparse-MoE block's down op: ADD folds, SCALED_ADD replays per op
    H, I, E, k = 1024, 512, 8, 2
    d = _cabi.Moe()
    d.E, d.top_k, d.renormalize, d.group_size, d.H, d.I, d.block_size = E, k, 1, 128, H, I, 16
    d.sorted_len = k + E * 15
    for f, _ in _cabi.Moe._fields_[8:]:
        setattr(d, f, buf())
    _KEEP.append(d)
    nm = rmsnorm(buf(), H)
    moe = dict(kind=_cabi.OP_SPARSE_MOE, M=1, K=H, N=H, x=nm["y"], y=buf(), weight=ctypes.addressof(d))
    assert _rc([nm, moe, add(moe["y"], buf(), H)]) == OK
    assert _rc([nm, moe, scaled_add(buf(), moe["y"], H)]) == EUNSUPPORTED


def test_reading_the_raw_output_under_a_scaled_add():
    K = 4096
    lin = linear(buf(), K, K)
    assert _rc([lin, scaled_add(buf(), lin["y"], K), linear(lin["y"], K, K)]) == EUNSUPPORTED
