"""Host logic of MLA with a q LoRA in decode programs (MLA_K_ROPE / MLA_Q_ROPE), checked without a GPU: the two op
constants and the exports against the header, the folding of the q LoRA chain and of DeepSeek-V3's dense segment through
b200awq_program_plan, every rejection, the residual window with a fused row narrower than the grid, the size checks
against the token rows, fuse_mla_lora_input against the oracle's dequantisation and the register / spill budget of
stream_mla_lora_kernel."""
import ctypes
import re

import numpy as np
import pytest

from _fake_ops import add, buf, linear, plan, rmsnorm, silu
from _toolchain import entries, header_constants, needs_nvcc, sass
from autoawq_b200 import _cabi
from autoawq_b200._cabi import lib

# DeepSeek-V3 attention: H, Dn, Dr, Dv, C, Cq, hidden, intermediate
V3 = dict(H=128, DN=128, DR=64, DV=128, C=512, CQ=1536, HID=7168, INTER=18432)
# a narrower geometry whose fused q_a | kv_a row has fewer 16-column sets (66) than 132 SMs, with Dr = 32
NARROW = dict(H=40, DN=64, DR=32, DV=64, C=256, CQ=768, HID=2560, INTER=6912)


def mla_desc(g, S=2048, Sf=4096, style=0, **kw):
    d = _cabi.Mla()
    d.n_heads, d.nope_dim, d.rope_dim, d.v_dim, d.kv_lora_rank, d.style = g["H"], g["DN"], g["DR"], g["DV"], g["C"], style
    d.cache_len, d.freqs_len = S, Sf
    W = g["DN"] + g["DR"]
    d.k_batch_stride, d.v_batch_stride, d.v_head_stride = S * g["H"] * W, S * g["H"] * g["DV"], g["DV"]
    d.pos, d.freqs, d.q_out = buf(4), buf(Sf * g["DR"] * 4), buf(g["H"] * W * 2)
    d.k_cache, d.v_cache = buf(S * g["H"] * W * 2), buf(S * g["H"] * g["DV"] * 2)
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def lora_chain(g=V3, M=1, d=None, x=None):
    """[norm1, q_a|kv_a, mla_k_rope, rmsnorm(q_a), q_b, mla_q_rope, rmsnorm(c_kv), kv_b, mla_kv]: the start of a
    DeepSeek-V3 attention block.  One descriptor serves the three MLA ops (the caches are shared as a layer shares
    them)."""
    d = d if d is not None else mla_desc(g)
    H, W, C, CQ, DR = g["H"], g["DN"] + g["DR"], g["C"], g["CQ"], g["DR"]
    n_qa, n_qb, n_kv = CQ + C + DR, H * W, H * (g["DN"] + g["DV"])
    norm1 = rmsnorm(x if x is not None else buf(M * g["HID"] * 2), g["HID"], M, eps=1e-6)
    qa = linear(norm1["y"], g["HID"], n_qa, M)
    krope = dict(kind=_cabi.OP_MLA_K_ROPE, M=M, N=n_qa, ldx=n_qa, x=qa["y"], weight=ctypes.addressof(d))
    qnorm = rmsnorm(qa["y"], CQ, M, eps=1e-6)
    qb = linear(qnorm["y"], CQ, n_qb, M)
    qrope = dict(kind=_cabi.OP_MLA_Q_ROPE, M=M, N=n_qb, ldx=n_qb, x=qb["y"], weight=ctypes.addressof(d))
    ckv = rmsnorm(qa["y"] + CQ * 2, C, M, eps=1e-6)
    kvb = linear(ckv["y"], C, n_kv, M)
    kv = dict(kind=_cabi.OP_MLA_KV, M=M, N=n_kv, ldx=n_kv, x=kvb["y"], weight=ctypes.addressof(d))
    return [norm1, qa, krope, qnorm, qb, qrope, ckv, kvb, kv], d


def dense_segment(g=V3, M=1):
    """[o + h, norm2, gate|up, silu, down + h, norm1', q_a|kv_a', k-rope', norm(q_a)', q_b', q-rope', norm(c_kv)',
    kv_b', mla_kv']: a dense DeepSeek-V3 layer's step from one attention call to the next."""
    HID, I = g["HID"], g["INTER"]
    o = linear(buf(M * HID * 2), g["H"] * g["DV"], HID, M)
    h = add(o["y"], buf(M * HID * 2), HID, M)
    norm2 = rmsnorm(h["y"], HID, M, eps=1e-6)
    gu = linear(norm2["y"], HID, 2 * I, M)
    act = silu(gu["y"], I, M)
    down = linear(act["y"], I, HID, M)
    out = add(down["y"], h["y"], HID, M)
    chain, d = lora_chain(g, M, x=out["y"])
    return [o, h, norm2, gu, act, down, out] + chain, d


def test_op_constants_match_header():
    assert header_constants("B200AWQ_OP_MLA_K_ROPE", "B200AWQ_OP_MLA_Q_ROPE") == \
        (_cabi.OP_MLA_K_ROPE, _cabi.OP_MLA_Q_ROPE) == (12, 13)


def test_exports():
    from autoawq_b200 import ext, packing
    from autoawq_b200.program import DecodeProgram

    for name in ("b200awq_mla_k_rope", "b200awq_mla_q_rope"):
        assert name in _cabi.SIGNATURES and hasattr(lib, name)
    for name in ("mla_k_rope", "mla_q_rope"):
        assert name in ext.__all__ and callable(getattr(ext, name))
    assert callable(DecodeProgram.mla_k_rope) and callable(DecodeProgram.mla_q_rope)
    assert callable(packing.fuse_mla_lora_input)


# ------------------------------------------------------------------------------------------------ folding (plan)
@pytest.mark.parametrize("g", [V3, NARROW], ids=["v3", "narrow"])
def test_chain_folds_into_three_kernel_ops(g):
    ops, d = lora_chain(g)
    assert plan(ops) == (0, 3)       # q_a|kv_a (+ K_ROPE), q_b (+ q_a_layernorm, + Q_ROPE), kv_b (+ kv_a_layernorm, + KV)


@pytest.mark.parametrize("g", [V3, NARROW], ids=["v3", "narrow"])
def test_dense_segment_plan(g):
    """The V3 dense segment is 6 kernel ops on 132 SMs (o, gate|up, down, q_a|kv_a', q_b', kv_b') at M = 1; at M = 2 the
    program replays per op."""
    ops, d = dense_segment(g)
    assert plan(ops) == (0, 6)
    ops, d = dense_segment(g, M=2)
    assert plan(ops, max_tokens=2)[0] == 2
    ops, d = lora_chain(g, M=2)
    assert plan(ops, max_tokens=2)[0] == 2


def test_kv_b_poll_counts_for_the_residual_window():
    """A residual read by op 1 from op 0's row, which kv_b (op 4) publishes into again.  Only the staging polls of ops 2..4
    can show that every CTA finished op 1: q_a|kv_a (op 2) reads an external row, q_b polls the fused row (66 sets:
    fewer than the grid, so it does not count), kv_b polls q_b's whole row (240 sets).  That poll is what lets the
    program fold; with q_b's row narrower than the grid as well, the program is refused."""
    g = NARROW
    a = linear(buf(g["HID"] * 2), g["HID"], g["HID"])
    b = linear(a["y"], g["HID"], g["HID"])
    b_res = add(b["y"], a["y"], g["HID"])
    chain, d = lora_chain(g, x=buf(g["HID"] * 2))
    assert plan([a, b, b_res] + chain) == (0, 5)
    assert plan([a, b, b_res] + chain, sms=264)[0] == 2   # q_b's 240 sets no longer cover every CTA


def _reject(mutate, g=V3, rc=2):
    ops, d = lora_chain(g)
    mutate(ops, d)
    assert plan(ops)[0] == rc


def test_rejects_op_before_not_a_plain_linear():
    def glue_in_between(ops, d):     # mla_k_rope after the q_a_layernorm instead of after q_a|kv_a
        ops[2], ops[3] = ops[3], ops[2]
    _reject(glue_in_between)

    def q_rope_before_its_linear(ops, d):
        ops[4], ops[5] = ops[5], ops[4]
    _reject(q_rope_before_its_linear)

    def first(ops, d):
        ops[0] = ops[2]
    _reject(first)


def test_rejects_n_mismatch():
    def no_q_lora(ops, d):           # N = C + Dr: Cq = 0
        d.kv_lora_rank = V3["C"] + V3["CQ"]
    _reject(no_q_lora)

    def q_heads(ops, d):             # q_b's N is not H (Dn + Dr)
        d.n_heads = 64
    _reject(q_heads)


def test_rejects_cq_not_multiple_of_16():
    ops, d = lora_chain()
    ops[1]["N"] = ops[2]["N"] = V3["CQ"] + 8 + V3["C"] + V3["DR"]     # Cq = 1544
    assert plan(ops)[0] == 2


@pytest.mark.parametrize("field", ["DN", "DR", "DV"])
def test_rejects_dims_not_multiple_of_16(field):
    ops, d = lora_chain(dict(V3, **{field: V3[field] - 8}))
    assert plan(ops)[0] == 2


def test_rejects_c_not_multiple_of_16():
    g = dict(V3, C=520)
    ops, d = lora_chain(g)
    for o in ops:                    # (so that K = C = 520 is still a whole number of groups)
        if o["kind"] == _cabi.OP_LINEAR_GEMM and o["K"] == 520:
            o["group_size"] = 8
    assert plan(ops)[0] == 2


@pytest.mark.parametrize("what", ["reads q_out", "writes q_out", "writes k_cache", "writes v_cache", "reads k_cache",
                                  "writes pos", "writes freqs"])
def test_rejects_other_ops_on_outputs_or_writes_of_inputs(what):
    def mutate(ops, d):
        tgt = {"reads q_out": d.q_out, "writes q_out": d.q_out, "writes k_cache": d.k_cache + 4096,
               "writes v_cache": d.v_cache, "reads k_cache": d.k_cache, "writes pos": d.pos,
               "writes freqs": d.freqs}[what]
        if what.startswith("reads"):
            ops[6]["x"] = tgt                # kv_a_layernorm (kv_b's prologue) reads it instead of c_kv
        else:
            ops[7]["y"] = tgt
            ops[8]["x"] = tgt
    _reject(mutate)


def test_rejects_two_k_rotations_on_one_k_cache():
    ops, d = lora_chain()
    ops2, d2 = lora_chain()
    d2.k_cache = d.k_cache
    assert plan(ops + ops2)[0] == 2
    d2.k_cache = buf(2048 * V3["H"] * (V3["DN"] + V3["DR"]) * 2)   # separate caches: two layers' chains fold
    d2.q_out = buf(V3["H"] * (V3["DN"] + V3["DR"]) * 2)
    assert plan(ops + ops2) == (0, 6)


def test_k_rope_and_kv_may_not_share_k_cache_with_another_geometry():
    ops, d = lora_chain()
    dk = mla_desc(V3, k_cache=d.k_cache, cache_len=1024, pos=d.pos)
    dk.k_batch_stride = 1024 * V3["H"] * (V3["DN"] + V3["DR"])
    ops[8]["weight"] = ctypes.addressof(dk)
    assert plan(ops)[0] == 2


def test_rejects_a_program_mixing_mla_rope_and_the_q_lora_ops():
    from test_program_mla_cpu import mla_chain

    ops, d = lora_chain()
    ops2, keep = mla_chain()
    assert plan(ops2)[0] == 0 and plan(ops)[0] == 0
    assert plan(ops + ops2)[0] == 2


@pytest.mark.parametrize("field,op", [("pos", 2), ("k_cache", 2), ("freqs", 2), ("q_out", 5), ("freqs", 5),
                                      ("pos", 5)])
def test_null_pointer_is_einval(field, op):
    ops, d = lora_chain()
    d2 = mla_desc(V3, k_cache=d.k_cache, q_out=d.q_out, pos=d.pos)
    setattr(d2, field, None)
    ops[op]["weight"] = ctypes.addressof(d2)
    assert plan(ops)[0] == 1


def test_k_rope_ignores_q_out_and_q_rope_ignores_the_caches():
    """MLA_K_ROPE writes only k_cache and MLA_Q_ROPE only q_out: a null q_out / k_cache (and no v_cache) fold."""
    ops, d = lora_chain()
    dk = mla_desc(V3, k_cache=d.k_cache, pos=d.pos, q_out=None, v_cache=None)
    dq = mla_desc(V3, q_out=d.q_out, pos=d.pos, k_cache=None, v_cache=None, k_batch_stride=0, kv_lora_rank=0)
    ops[2]["weight"], ops[5]["weight"] = ctypes.addressof(dk), ctypes.addressof(dq)
    assert plan(ops) == (0, 3)


# ------------------------------------------------------------------------------------------------ the kernel entry
@needs_nvcc
def test_entry_register_and_spill_budget():
    """stream_mla_lora_kernel (288 threads, one CTA per SM) fits the register file: 168 registers, like
    stream_mla_kernel, and 16 bytes of spill stores (stream_mla_kernel's 12 and one more value), all made before the unit
    loop.  No spill load or store sits inside the unit loop (between its first and last MMA)."""
    found = entries("program.cu", "stream_mla_lora_kernel")
    assert len(found) == 1, found
    regs, stack, st, ld = next(iter(found.values()))
    assert regs * (32 + 32 * 8) <= 65536 and st <= 16 and stack <= 16, (regs, st, ld, stack)
    lines = sass("program.cu", "stream_mla_lora_kernel").splitlines()
    mma = [i for i, line in enumerate(lines) if "HMMA" in line]
    assert mma
    inside = [line for line in lines[mma[0]:mma[-1]] if re.search(r"\b(LDL|STL)\b", line)]
    assert not inside, inside


# ------------------------------------------------------------------------------------------------ Python-side checks
def _cpu_tensors(M, batch, q_rows=None):
    import torch

    g = NARROW
    W = g["DN"] + g["DR"]
    qa = torch.zeros((M, g["CQ"] + g["C"] + g["DR"]), dtype=torch.float16)
    qb = torch.zeros((M, g["H"] * W), dtype=torch.float16)
    k_cache = torch.zeros((batch, 8, g["H"], W), dtype=torch.float16)
    q_out = None if q_rows is None else torch.zeros((q_rows, g["H"], W), dtype=torch.float16)
    pos = torch.zeros(1, dtype=torch.int32)
    freqs = torch.zeros((16, g["DR"] // 2, 2), dtype=torch.float32)
    return g, qa, qb, k_cache, q_out, pos, freqs


@pytest.mark.parametrize("case", ["k_cache batch", "q_out rows"])
def test_sizes_are_checked_against_the_token_rows(case):
    """The kernels write cache batch entry m and q_out row m for every token row m < M: a smaller cache or q_out is
    refused before any pointer is taken (host tensors: refused for their size before they are refused for living on
    the host)."""
    from autoawq_b200 import ext
    from autoawq_b200._cabi import B200AwqError

    g, qa, qb, k_cache, q_out, pos, freqs = _cpu_tensors(2, 1, 1)
    with pytest.raises(B200AwqError, match=case.split()[0]):
        if case == "k_cache batch":
            ext.mla_k_rope(qa, freqs, pos, k_cache, g["H"], g["DN"], g["DR"], g["C"], g["CQ"], 0)
        else:
            ext.mla_q_rope(qb, freqs, pos, 8, g["H"], g["DN"], g["DR"], 0, q_out=q_out)


def test_sizes_that_fit_reach_the_device_check():
    from autoawq_b200 import ext
    from autoawq_b200._cabi import B200AwqError

    g, qa, qb, k_cache, q_out, pos, freqs = _cpu_tensors(2, 3, 2)
    for call in (lambda: ext.mla_k_rope(qa, freqs, pos, k_cache, g["H"], g["DN"], g["DR"], g["C"], g["CQ"], 1),
                 lambda: ext.mla_q_rope(qb, freqs, pos, 8, g["H"], g["DN"], g["DR"], 0, q_out=q_out)):
        with pytest.raises(B200AwqError, match="CUDA device"):
            call()
    with pytest.raises(B200AwqError, match="qkva"):   # the row width is Cq + C + Dr
        ext.mla_k_rope(qa, freqs, pos, k_cache, g["H"], g["DN"], g["DR"], g["C"], g["CQ"] - 16, 0)


def test_fuse_mla_lora_input_concatenates_the_two_projections():
    """packing.fuse_mla_lora_input: one GEMM-layout linear whose dequantised weight is [W_q_a | W_kv_a] along N, bit for
    bit (the oracle's dequantisation of the fused tensors against that of each projection); an attention without a q
    LoRA is refused."""
    import types

    import torch

    from autoawq_b200 import packing
    from autoawq_b200.linear import WQLinear_GEMM
    from oracle import awq_oracle as O

    g = NARROW
    K, Gs = 256, 128
    gen = torch.Generator().manual_seed(2)

    def lin(N):
        m = WQLinear_GEMM(4, Gs, K, N, False, "cpu")
        m.qweight.copy_(torch.randint(-2**31, 2**31 - 1, m.qweight.shape, dtype=torch.int32, generator=gen))
        m.qzeros.copy_(torch.randint(-2**31, 2**31 - 1, m.qzeros.shape, dtype=torch.int32, generator=gen))
        m.scales.copy_((torch.rand(m.scales.shape, generator=gen) * 0.01).half())
        return m

    n = g["CQ"] + g["C"] + g["DR"]
    attn = types.SimpleNamespace(q_lora_rank=g["CQ"], q_a_proj=lin(g["CQ"]), kv_a_proj_with_mqa=lin(g["C"] + g["DR"]))
    q, s, z, bias = packing.fuse_mla_lora_input(attn)
    assert bias is None and tuple(q.shape) == (K, n // 8) and tuple(s.shape) == (K // Gs, n)

    def deq(qw, sc, qz):
        return O.dequantize_gemm(qw.numpy(), qz.numpy(), sc.numpy(), Gs)

    parts = [deq(m.qweight, m.scales, m.qzeros) for m in (attn.q_a_proj, attn.kv_a_proj_with_mqa)]
    assert np.array_equal(deq(q, s, z).view(np.uint16), np.concatenate(parts, axis=1).view(np.uint16))
    attn.q_lora_rank = None
    with pytest.raises(ValueError):
        packing.fuse_mla_lora_input(attn)
