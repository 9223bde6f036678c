"""Host logic of the MLA ops (MLA_ROPE / MLA_KV) in decode programs, checked without a GPU: the ctypes layout of
b200awq_mla_t and the two op constants against the header, the exports, the mode-3 column map through the stream-format
oracle, the folding of the MLA chain and every rejection through b200awq_program_plan, the register / spill budget of
stream_mla_kernel and the SASS of the pre-existing entries against a given revision."""
import ctypes
import re

import numpy as np
import pytest

from _fake_ops import add, buf, linear, plan, rmsnorm
from _toolchain import entries, header_constants, header_layout, mirror_layout, needs_nvcc, sass, sass_compare
from autoawq_b200 import _cabi
from autoawq_b200._cabi import lib
from oracle import stream_format as SF
from test_program_deepseek_moe_cpu import _desc

# DeepSeek-V2-Lite / Moonlight-16B-A3B attention: H, Dn, Dr, Dv, C, hidden
H, DN, DR, DV, C, HID = 16, 128, 64, 128, 512, 2048
N_QKVA = H * (DN + DR) + C + DR        # 3648
N_KV = H * (DN + DV)                   # 4096


def mode3_columns(N):
    """[S, 16] original column of (set, tile row) in stream mode 3: lo[g] = 16 s + 2 g, hi[g] = lo[g] + 1."""
    s = np.arange(N // 16)[:, None]
    g = np.arange(8)[None, :]
    return np.concatenate([16 * s + 2 * g, 16 * s + 2 * g + 1], axis=1)


def test_layout_and_op_constants_match_header():
    assert header_layout(_cabi.Mla, "b200awq_mla_t") == mirror_layout(_cabi.Mla)
    assert header_constants("B200AWQ_OP_MLA_ROPE", "B200AWQ_OP_MLA_KV") == (_cabi.OP_MLA_ROPE, _cabi.OP_MLA_KV) == (10, 11)


def test_exports():
    from autoawq_b200 import ext, packing
    from autoawq_b200.program import DecodeProgram

    for name in ("b200awq_mla_rope", "b200awq_mla_kv"):
        assert name in _cabi.SIGNATURES and hasattr(lib, name)
    for name in ("mla_rope", "mla_kv_cache", "mla_descriptor"):
        assert name in ext.__all__ and callable(getattr(ext, name))
    assert callable(DecodeProgram.mla_rope) and callable(DecodeProgram.mla_kv_cache)
    assert callable(packing.fuse_mla_input)


def test_mode3_column_map_through_the_oracle():
    """Mode 3 is mode 0 of the linear with its columns reordered so that set s holds (16 s + 2 g, 16 s + 2 g + 1) in
    tile rows (g, 8 + g): the oracle's mode-0 buffer of that reordered linear is the mode-3 buffer (the GPU test compares
    b200awq_stream_pack(mode 3) with it), and its simulated GEMV returns every original column at its own index."""
    rng = np.random.default_rng(3)
    K, N, G = 256, 64, 64
    cols = mode3_columns(N)
    assert sorted(cols.reshape(-1).tolist()) == list(range(N))          # a permutation of the columns
    assert (cols[:, 8:] - cols[:, :8] == 1).all() and (cols[:, :8] % 2 == 0).all()
    qweight = rng.integers(-2**31, 2**31 - 1, (K, N // 8), dtype=np.int64).astype(np.int32)
    qzeros = rng.integers(-2**31, 2**31 - 1, (K // G, N // 8), dtype=np.int64).astype(np.int32)
    scales = (rng.random((K // G, N)) * 0.01 + 0.001).astype(np.float16)
    perm = cols.reshape(-1)                   # mode 0 puts column 16 s + r at (set s, tile row r)
    q2, z2, s2 = permute_linear(qweight, qzeros, scales, perm)
    assert (SF.set_columns(N, 0).reshape(-1) == np.arange(N)).all()
    assert (perm[SF.set_columns(N, 0)] == cols).all()
    x = (rng.standard_normal(K) * 0.5).astype(np.float16)
    y_ref = SF.simulate_gemv(SF.pack_stream(qweight, qzeros, scales, G, 0), K, N, G, x, 0)
    y3 = SF.simulate_gemv(SF.pack_stream(q2, z2, s2, G, 0), K, N, G, x, 0)
    assert np.allclose(y3, y_ref[perm], rtol=0, atol=1e-9)


def permute_linear(qweight, qzeros, scales, perm):
    """GEMM-layout tensors of the linear whose column j is the original column perm[j]."""
    iw, iz = SF.unpack_gemm_ints(qweight, qzeros)

    def pack(ints):
        ints = ints.astype(np.uint32).reshape(ints.shape[0], -1, 8)
        w = np.zeros(ints.shape[:2], dtype=np.uint32)
        for j in range(8):
            w |= ints[..., j] << np.uint32(4 * SF.REV[j])
        return w.view(np.int32)

    return pack(iw[:, perm]), pack(iz[:, perm]), np.ascontiguousarray(scales[:, perm])


# ------------------------------------------------------------------------------------------------ folding (plan)
def mla_desc(S=2048, Sf=4096, style=0, v_head=DV, **kw):
    d = _cabi.Mla()
    d.n_heads, d.nope_dim, d.rope_dim, d.v_dim, d.kv_lora_rank, d.style = H, DN, DR, DV, C, style
    d.cache_len, d.freqs_len = S, Sf
    d.k_batch_stride, d.v_batch_stride, d.v_head_stride = S * H * (DN + DR), S * H * v_head, v_head
    d.pos, d.freqs, d.q_out = buf(4), buf(Sf * DR * 4), buf(H * (DN + DR) * 2)
    d.k_cache, d.v_cache = buf(S * H * (DN + DR) * 2), buf(S * H * v_head * 2)
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def mla_chain(M=1, d_rope=None, d_kv=None):
    """[norm1, q|kv_a, mla_rope, rmsnorm(c_kv), kv_b, mla_kv]: the start of a DeepSeek attention block (no q LoRA)."""
    d = d_rope if d_rope is not None else mla_desc()
    dk = d_kv if d_kv is not None else d
    norm1 = rmsnorm(buf(M * HID * 2), HID, M, eps=1e-6)
    qkva = linear(norm1["y"], HID, N_QKVA, M)
    rope = dict(kind=_cabi.OP_MLA_ROPE, M=M, N=N_QKVA, ldx=N_QKVA, x=qkva["y"], weight=ctypes.addressof(d))
    ckv = rmsnorm(qkva["y"] + H * (DN + DR) * 2, C, M, eps=1e-6)
    kvb = linear(ckv["y"], C, N_KV, M)
    kv = dict(kind=_cabi.OP_MLA_KV, M=M, N=N_KV, ldx=N_KV, x=kvb["y"], weight=ctypes.addressof(dk))
    return [norm1, qkva, rope, ckv, kvb, kv], (d, dk)


def test_chain_folds_into_two_kernel_ops():
    ops, keep = mla_chain()
    assert plan(ops) == (0, 2)          # q|kv_a (+ MLA_ROPE), kv_b (+ kv_a_layernorm as its prologue, + MLA_KV)


@pytest.mark.parametrize("style", [0, 1])
def test_v2_lite_segment_plan(style):
    """[o + h, norm2, deepseek_moe + h, norm1', q|kv_a', mla_rope', rmsnorm(c_kv)', kv_b', mla_kv']: accepted at M = 1
    on 132 SMs (o, gate|up, down, q|kv_a', kv_b'), rejected at M = 2."""
    for M in (1, 2):
        dsk = _desc(scoring=style)
        dsk.moe.sorted_len = 6 * M + 64 * 15
        o = linear(buf(M * HID * 2), HID, HID, M)                        # o_proj
        h = add(o["y"], buf(M * HID * 2), HID, M)
        norm2 = rmsnorm(h["y"], HID, M, eps=1e-6)
        moe = dict(kind=_cabi.OP_DEEPSEEK_MOE, M=M, K=HID, N=HID, x=norm2["y"], y=buf(M * HID * 2),
                   weight=ctypes.addressof(dsk))
        out = add(moe["y"], h["y"], HID, M)
        chain, keep = mla_chain(M)
        chain[0]["x"] = out["y"]
        rc, n = plan([o, h, norm2, moe, out] + chain, max_tokens=M)
        assert (rc, n) == ((0, 5) if M == 1 else (2, 0)), (M, rc, n)
    ops, keep = mla_chain(2)
    assert plan(ops, max_tokens=2)[0] == 2       # the MLA ops alone at M = 2: per op as well


def _reject(mutate, rc=2):
    ops, keep = mla_chain()
    mutate(ops, keep[0])
    assert plan(ops)[0] == rc


def test_rejects_op_before_not_a_plain_linear():
    def glue_in_between(ops, d):   # mla_rope after the rmsnorm instead of after q|kv_a
        ops[2], ops[3] = ops[3], ops[2]
    _reject(glue_in_between)

    def first(ops, d):
        ops[0] = ops[2]
    _reject(first)


def test_rejects_mla_after_a_moe_block():
    dsk = _desc()
    d = mla_desc()
    d.n_heads, d.nope_dim, d.v_dim, d.v_head_stride = 1, 1024, 1024, 1024
    moe = dict(kind=_cabi.OP_DEEPSEEK_MOE, M=1, K=HID, N=HID, x=buf(HID * 2), y=buf(HID * 2), weight=ctypes.addressof(dsk))
    kv = dict(kind=_cabi.OP_MLA_KV, M=1, N=HID, ldx=HID, x=moe["y"], weight=ctypes.addressof(d))
    assert plan([moe, kv])[0] == 2


@pytest.mark.parametrize("field,value", [("n_heads", 8), ("kv_lora_rank", 256), ("rope_dim", 32)])
def test_rejects_n_mismatch(field, value):
    _reject(lambda ops, d: setattr(d, field, value))


@pytest.mark.parametrize("dims", [(120, 64, 128, 512), (128, 56, 128, 512), (128, 64, 120, 512), (128, 64, 128, 520)])
def test_rejects_dims_not_multiple_of_16(dims):
    dn, dr, dv, c = dims
    d = mla_desc(nope_dim=dn, rope_dim=dr, v_dim=dv, kv_lora_rank=c)
    d.k_batch_stride, d.v_batch_stride, d.v_head_stride = 2048 * H * (dn + dr), 2048 * H * dv, dv
    ops, keep = mla_chain(d_rope=d)
    ops[1]["N"] = ops[2]["N"] = H * (dn + dr) + c + dr
    ops[3]["x"] = ops[1]["y"] + H * (dn + dr) * 2
    ops[3]["K"] = ops[4]["K"] = c
    ops[4]["N"] = ops[5]["N"] = H * (dn + dv)
    ops[4]["group_size"] = 8                 # (so that K = C = 520 is still a whole number of groups)
    assert plan(ops)[0] == 2


@pytest.mark.parametrize("what", ["reads q_out", "writes q_out", "writes k_cache", "writes v_cache", "reads v_cache",
                                  "writes pos", "writes freqs"])
def test_rejects_other_ops_on_outputs_or_writes_of_inputs(what):
    def mutate(ops, d):
        tgt = {"reads q_out": d.q_out, "writes q_out": d.q_out, "writes k_cache": d.k_cache + 4096,
               "writes v_cache": d.v_cache, "reads v_cache": d.v_cache, "writes pos": d.pos,
               "writes freqs": d.freqs}[what]
        if what.startswith("reads"):
            ops[3]["x"] = tgt                # kv_a_layernorm (kv_b's prologue) reads it instead of c_kv
        else:
            ops[4]["y"] = tgt
            ops[5]["x"] = tgt
    _reject(mutate)


def test_rejects_two_mla_ropes_on_one_k_cache():
    ops, (d, _) = mla_chain()
    ops2, (d2, _) = mla_chain()
    d2.k_cache = d.k_cache
    both = ops + ops2
    assert plan(both)[0] == 2
    d2.k_cache = buf(2048 * H * (DN + DR) * 2)   # separate caches: two layers' chains in one program fold
    assert plan(both) == (0, 4)


def test_rope_and_kv_may_not_share_k_cache_with_another_geometry():
    d = mla_desc()
    dk = mla_desc(k_cache=d.k_cache, cache_len=1024)
    dk.k_batch_stride, dk.v_batch_stride = 1024 * H * (DN + DR), 1024 * H * DV
    ops, keep = mla_chain(d_rope=d, d_kv=dk)
    assert plan(ops)[0] == 2


@pytest.mark.parametrize("field", ["pos", "k_cache", "q_out", "freqs"])
def test_null_pointer_is_einval(field):
    _reject(lambda ops, d: setattr(d, field, None), rc=1)


def test_kv_op_ignores_rope_only_fields():
    """MLA_KV reads neither freqs nor q_out (a descriptor without them folds); MLA_ROPE reads no v_cache."""
    d = mla_desc()
    dk = mla_desc(k_cache=d.k_cache)
    dk.freqs, dk.q_out, dk.freqs_len, dk.style = None, None, 0, 7
    d.v_cache, d.v_dim = None, 0
    ops, keep = mla_chain(d_rope=d, d_kv=dk)
    assert plan(ops) == (0, 2)


@pytest.mark.parametrize("style", [0, 1])
def test_padded_v_cache_folds(style):
    """A v_cache whose heads are padded to Dn + Dr (FlashAttention-2's layout for Dv < Dqk) is accepted."""
    d = mla_desc(style=style, v_head=DN + DR)
    ops, keep = mla_chain(d_rope=d)
    assert plan(ops) == (0, 2)


# ------------------------------------------------------------------------------------------------ the kernel entry
@needs_nvcc
def test_entry_register_and_spill_budget():
    """stream_mla_kernel (288 threads, one CTA per SM) fits the register file: 168 registers, like
    stream_deepseek_moe_kernel, and 12 bytes of spill stores (the DeepSeek entry's 8 and one more value) made before the
    unit loop.  No spill load or store sits inside the unit loop (between its first and last MMA)."""
    found = entries("program.cu", "stream_mla_kernel")
    assert found
    regs, stack, st, ld = next(iter(found.values()))
    assert regs * (32 + 32 * 8) <= 65536 and st <= 12 and stack <= 16, (regs, st, ld, stack)
    lines = sass("program.cu", "stream_mla_kernel").splitlines()
    mma = [i for i, line in enumerate(lines) if "HMMA" in line]
    assert mma
    inside = [line for line in lines[mma[0]:mma[-1]] if re.search(r"\b(LDL|STL)\b", line)]
    assert not inside, inside


@needs_nvcc
def test_existing_entries_sass_unchanged():
    """With B200AWQ_SASS_BASE set to a git revision (the commit before these ops), every entry both trees have compiles
    to the same SASS (tools/sass_unchanged.py): the MLA code sits behind SP_MLA, its own side table and its own pack
    kernel.  Unset, the test is skipped."""
    res = sass_compare()
    assert res, "no entry to compare"
    assert all(res.values()), [n for n, same in res.items() if not same]


# ------------------------------------------------------------------------------------------------ Python-side checks
def _cpu_ops(M, batch, q_rows=None):
    import torch

    qkva = torch.zeros((M, N_QKVA), dtype=torch.float16)
    kv = torch.zeros((M, N_KV), dtype=torch.float16)
    k_cache = torch.zeros((batch, 8, H, DN + DR), dtype=torch.float16)
    v_cache = torch.zeros((batch, 8, H, DV), dtype=torch.float16)
    q_out = None if q_rows is None else torch.zeros((q_rows, H, DN + DR), dtype=torch.float16)
    pos = torch.zeros(1, dtype=torch.int32)
    freqs = torch.zeros((16, DR // 2, 2), dtype=torch.float32)
    return qkva, kv, k_cache, v_cache, q_out, pos, freqs


@pytest.mark.parametrize("case", ["k_cache batch", "v_cache batch", "q_out rows"])
def test_sizes_are_checked_against_the_token_rows(case):
    """The kernels write cache batch entry m and q_out row m for every token row m < M: a cache with fewer batch
    entries or a q_out of fewer rows is refused before any pointer is taken (checked here on host tensors, which are
    refused for their size before they are refused for living on the host)."""
    from autoawq_b200 import ext
    from autoawq_b200._cabi import B200AwqError

    qkva, kv, k_cache, v_cache, q_out, pos, freqs = _cpu_ops(2, 1 if case == "k_cache batch" else 2,
                                                             1 if case == "q_out rows" else None)
    if case == "v_cache batch":
        v_cache = v_cache[:1]
    with pytest.raises(B200AwqError, match=case.split()[0]):
        if case == "v_cache batch":
            ext.mla_kv_cache(kv, pos, k_cache, v_cache, H, DN, DV)
        else:
            ext.mla_rope(qkva, freqs, pos, k_cache, H, DN, DR, C, 0, q_out=q_out)
    if case == "k_cache batch":
        with pytest.raises(B200AwqError, match="k_cache"):
            ext.mla_kv_cache(kv, pos, k_cache, v_cache, H, DN, DV)


def test_sizes_that_fit_reach_the_device_check():
    """With every size right, the host tensors are refused only for living on the host."""
    from autoawq_b200 import ext
    from autoawq_b200._cabi import B200AwqError

    qkva, kv, k_cache, v_cache, q_out, pos, freqs = _cpu_ops(2, 3, 2)
    for call in (lambda: ext.mla_rope(qkva, freqs, pos, k_cache, H, DN, DR, C, 0, q_out=q_out),
                 lambda: ext.mla_kv_cache(kv, pos, k_cache, v_cache, H, DN, DV)):
        with pytest.raises(B200AwqError, match="CUDA device"):
            call()


@pytest.mark.parametrize("M,ldx,rc", [(2, C, 0), (2, 0, 0), (2, N_QKVA, 2)])
def test_row_strided_rmsnorm_replays_per_op(M, ldx, rc):
    """An RMSNORM over rows of a wider tensor (kv_a_layernorm on the c_kv slice of M > 1 rows) is refused by the fused
    kernels, which stage contiguous rows; a contiguous one (ldx 0 or K) folds."""
    ckv = rmsnorm(buf(M * N_QKVA * 2), C, M, eps=1e-6, ldx=ldx)
    assert plan([ckv, linear(ckv["y"], C, N_KV, M)], max_tokens=M)[0] == rc


def test_fuse_mla_input_concatenates_the_two_projections():
    """packing.fuse_mla_input: one GEMM-layout linear whose dequantised weight is [W_q | W_kv_a] along N, bit for bit
    (the oracle's dequantisation of the fused tensors against that of each projection), and no fused attention module
    with a q LoRA."""
    import types

    import torch

    from autoawq_b200 import packing
    from autoawq_b200.linear import WQLinear_GEMM
    from oracle import awq_oracle as O

    K, Gs = 256, 128
    gen = torch.Generator().manual_seed(1)

    def lin(N):
        m = WQLinear_GEMM(4, Gs, K, N, False, "cpu")
        m.qweight.copy_(torch.randint(-2**31, 2**31 - 1, m.qweight.shape, dtype=torch.int32, generator=gen))
        m.qzeros.copy_(torch.randint(-2**31, 2**31 - 1, m.qzeros.shape, dtype=torch.int32, generator=gen))
        m.scales.copy_((torch.rand(m.scales.shape, generator=gen) * 0.01).half())
        return m

    attn = types.SimpleNamespace(q_lora_rank=None, q_proj=lin(H * (DN + DR)), kv_a_proj_with_mqa=lin(C + DR))
    q, s, z, bias = packing.fuse_mla_input(attn)
    assert bias is None and tuple(q.shape) == (K, N_QKVA // 8) and tuple(s.shape) == (K // Gs, N_QKVA)

    def deq(qw, sc, qz):
        return O.dequantize_gemm(qw.numpy(), qz.numpy(), sc.numpy(), Gs)

    parts = [deq(m.qweight, m.scales, m.qzeros) for m in (attn.q_proj, attn.kv_a_proj_with_mqa)]
    assert np.array_equal(deq(q, s, z).view(np.uint16), np.concatenate(parts, axis=1).view(np.uint16))
    attn.q_lora_rank = 1536
    with pytest.raises(ValueError):
        packing.fuse_mla_input(attn)
