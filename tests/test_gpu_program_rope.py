"""GPU tests of RoPE + KV-cache append (B200AWQ_OP_ROPE_KV): the stand-alone op against the reference's RoPE.forward +
WindowedCache.update_kv (oracle/_ref), the rotary stream format against its numpy restatement, and decode programs that
fold the op into the qkv linear's finish.

Bit-identity and where it stops:
  * the stand-alone op uses the contraction torch's complex multiply has in the common case, but torch does not use one
    contraction for every tensor shape (q and k, batches of 1, 2 or 4 rows go through different loops): a few elements
    (1-2 of 16384 in these cases) come out one fp16 ulp away from any single formula, so the reference comparison
    allows one ulp and reports the counts of each candidate formula when more is seen;
  * a fused program's q and cache rows are bit-identical to the stand-alone op applied to the program's own qkv output;
  * the linears themselves are not bit-identical between a fused program and the per-op replay (different kernels,
    different summation order; a mode-2 column also sits in a different MMA row than in mode 0), so those buffers are
    compared within a tolerance, as the other program tests compare fused linears with the oracle."""
import numpy as np
import pytest
import torch

from test_gpu_program import EPS
from test_gpu_program_moe import Moe
from test_program_rope_cpu import rotary_columns

pytestmark = pytest.mark.gpu

F16 = torch.float16


def _dev():
    return torch.device("cuda:0")


def _linear(K, N, G, seed):
    """Random GEMM-layout AWQ weights with O(1) outputs (the MoE tests' scale recipe)."""
    g = torch.Generator(device=_dev()).manual_seed(seed)
    return (torch.randint(-2**31, 2**31 - 1, (K, N // 8), dtype=torch.int32, device=_dev(), generator=g),
            ((torch.rand((K // G, N), device=_dev(), generator=g) * 0.5 + 0.75) / (6.1 * K**0.5)).half(),
            torch.randint(-2**31, 2**31 - 1, (K // G, N // 8), dtype=torch.int32, device=_dev(), generator=g))


def _freqs(D, S, theta):
    """RoPE.precompute_freqs_cis (awq/modules/fused/attn.py:39-43), on the device like the module's parameter."""
    from _refload import load_reference

    load_reference(shim=True)
    from awq.modules.fused.attn import RoPE

    return RoPE(D, S, _dev(), theta).freqs_cis


def _caches(B, S, KV, D, seed):
    g = torch.Generator(device=_dev()).manual_seed(seed)
    return (torch.randn((B, S, KV, D), device=_dev(), generator=g).half(),
            torch.randn((B, S, KV, D), device=_dev(), generator=g).half())


def _candidates(qkv, freqs, pos, H, KV, D):
    """numpy fp32 evaluations of the complex product (a + ib)(c + is) with each FMA contraction (diagnostics)."""
    x = qkv.float().cpu().numpy().reshape(qkv.shape[0], H + 2 * KV, D)[:, : H + KV].astype(np.float64)
    a, b = x[..., : D // 2], x[..., D // 2:]
    f = torch.view_as_real(freqs)[pos].cpu().numpy().astype(np.float64)
    c, s = f[:, 0], f[:, 1]
    r32 = lambda v: v.astype(np.float32).astype(np.float64)   # noqa: E731
    out = {"no fma": (r32(r32(a * c) - r32(b * s)), r32(r32(a * s) + r32(b * c))),
           "fma(a,c,-bs) fma(b,c,as)": (r32(a * c - r32(b * s)), r32(b * c + r32(a * s))),
           "fma(-b,s,ac) fma(a,s,bc)": (r32(r32(a * c) - b * s), r32(a * s + r32(b * c)))}
    return {k: np.concatenate([re, im], -1).astype(np.float16) for k, (re, im) in out.items()}


# ------------------------------------------------------------------------------------------ stream format
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("G", [64, 128])
def test_stream_pack_rotary_matches_oracle(D, G, monkeypatch):
    from autoawq_b200 import ext
    from oracle import stream_format as SF

    K, N = 512, 6 * D
    qw, sc, qz = _linear(K, N, G, seed=D + G)
    orig = SF.set_columns
    monkeypatch.setattr(SF, "set_columns", lambda n, mode: rotary_columns(n, D) if mode == 2 else orig(n, mode))
    want = SF.pack_stream(qw.cpu().numpy(), qz.cpu().numpy(), sc.cpu().numpy(), G, 2)
    got = ext.stream_pack_rotary(qw, sc, qz, D).cpu().numpy()
    assert np.array_equal(got, want)


# ------------------------------------------------------------------------------------------ the stand-alone op
@pytest.mark.parametrize("M", [1, 2, 4])
def test_rope_kv_cache_matches_reference(M):
    """Llama-3-8B attention shapes (32 / 8 / 128, theta 500000, 2048 positions): q and the written k row within one
    fp16 ulp of RoPE.forward + update_kv, the v row bit-identical; every other cache row untouched."""
    from autoawq_b200 import ext

    _freqs(8, 8, 1.0)                                       # imports the reference package
    from awq.modules.fused.attn import RoPE
    from awq.modules.fused.cache import WindowedCache

    H, KV, D, S = 32, 8, 128, 2048
    rope = RoPE(D, S, _dev(), 500000.0)
    freqs = rope.freqs_cis
    qkv = (torch.randn((M, (H + 2 * KV) * D), device=_dev(), generator=torch.Generator(device=_dev()).manual_seed(M)) * 3
           ).half()
    for p in (0, 1, 1000, 2047):
        cache = WindowedCache(M, H, KV, D, S, _dev())
        cache.k.normal_()
        cache.v.normal_()
        k0, v0 = cache.k.clone(), cache.v.clone()
        kc, vc = cache.k.clone(), cache.v.clone()
        xqkv = qkv.view(M, 1, H + 2 * KV, D)
        xq, xk = rope.forward(xqkv[:, :, :H], xqkv[:, :, H:H + KV], p, 1)
        cache.update_kv(values_store=xqkv[:, :, H + KV:], keys_store=xk, batch_size=M, start_pos=p, seqlen=1)
        pos = torch.tensor([p], dtype=torch.int32, device=_dev())
        q = ext.rope_kv_cache(qkv, freqs, pos, kc, vc, H, KV)
        torch.cuda.synchronize()
        ref_q = xq.reshape(M, H, D)
        got = torch.cat([q, kc[:, p]], 1)
        want = torch.cat([ref_q, cache.k[:, p]], 1)
        ulps = _ulps(got, want)
        if ulps.max() > 1:
            cand = _candidates(qkv, freqs, p, H, KV, D)
            ref = want.cpu().numpy()
            counts = {k: int((v.view(np.uint16) != ref.view(np.uint16)).sum()) for k, v in cand.items()}
            pytest.fail(f"pos {p}: {int((ulps > 1).sum())} elements > 1 ulp; candidate mismatches vs torch: {counts}")
        assert torch.equal(vc, cache.v), f"pos {p}: v cache differs"
        rest = torch.ones(S, dtype=torch.bool, device=_dev())
        rest[p] = False
        assert torch.equal(kc[:, rest], k0[:, rest]) and torch.equal(vc[:, rest], v0[:, rest])


def _ulps(a, b):
    """Distance in fp16 units in the last place (same-sign finite values)."""
    ia, ib = a.view(torch.int16).int(), b.view(torch.int16).int()
    return torch.where((ia < 0) == (ib < 0), (ia - ib).abs(), torch.full_like(ia, 1 << 16))


def test_out_of_range_position_writes_nothing():
    from autoawq_b200 import ext

    H, KV, D, S = 4, 2, 64, 64
    freqs = _freqs(D, S, 10000.0)
    qkv = torch.randn((2, (H + 2 * KV) * D), device=_dev()).half()
    kc, vc = _caches(2, S, KV, D, 1)
    k0, v0 = kc.clone(), vc.clone()
    q = torch.full((2, H, D), 7.0, dtype=F16, device=_dev())
    for p in (S, -1):
        ext.rope_kv_cache(qkv, freqs, torch.tensor([p], dtype=torch.int32, device=_dev()), kc, vc, H, KV, q_out=q)
    torch.cuda.synchronize()
    assert torch.equal(kc, k0) and torch.equal(vc, v0) and bool((q == 7.0).all())


# ------------------------------------------------------------------------------------------ decode programs
class Layer:
    """One decoder layer's weights (GEMM-layout AWQ, random) and its attention geometry."""

    def __init__(self, hidden, inter, H, KV, D, S, seed, G=128):
        self.hidden, self.inter, self.H, self.KV, self.D, self.S = hidden, inter, H, KV, D, S
        self.w = dict(o=_linear(hidden, hidden, G, seed), gu=_linear(hidden, 2 * inter, G, seed + 1),
                      down=_linear(inter, hidden, G, seed + 2), qkv=_linear(hidden, (H + 2 * KV) * D, G, seed + 3))
        g = torch.Generator(device=_dev()).manual_seed(seed + 4)
        self.n1 = (1 + 0.1 * torch.randn(hidden, device=_dev(), generator=g)).half()
        self.n2 = (1 + 0.1 * torch.randn(hidden, device=_dev(), generator=g)).half()
        self.freqs = _freqs(D, S, 500000.0)


def _record_segment(api, L, attn, h_in, pos, kc, vc, moe=None):
    """[o + h, norm2, gate|up, silu, down + h, norm1', qkv', rope'] (Llama) or [o + h, norm2, sparse_moe + h, norm1',
    qkv', rope'] (Mixtral) against `api`; returns the buffers it names."""
    M = attn.shape[0]
    o = api.gemm_forward_cuda(attn, *L.w["o"], 8)
    h = api.add(o, h_in)
    xn2 = torch.empty((M, L.hidden), dtype=F16, device=_dev())
    api.layernorm_forward_cuda(h, L.n2, xn2, EPS)
    bufs = dict(o=o, h=h, xn2=xn2)
    if moe is None:
        gu = api.gemm_forward_cuda(xn2, *L.w["gu"], 8)
        act = torch.empty((M, L.inter), dtype=F16, device=_dev())
        api.silu_and_mul(act, gu)
        dn = api.gemm_forward_cuda(act, *L.w["down"], 8)
        bufs.update(gu=gu, act=act)
    else:
        dn = api.sparse_moe(xn2, moe.gate, moe.w1, moe.w2, moe.top_k)
    out = api.add(dn, h)
    xn = torch.empty((M, L.hidden), dtype=F16, device=_dev())
    api.layernorm_forward_cuda(out, L.n1, xn, EPS)
    qkv = api.gemm_forward_cuda(xn, *L.w["qkv"], 8)
    q = api.rope_kv_cache(qkv, L.freqs, pos, kc, vc, L.H, L.KV)
    bufs.update(dn=dn, out=out, xn=xn, qkv=qkv, q=q, k=kc, v=vc)
    return bufs


def _build(record, M, no_fuse):
    from autoawq_b200 import ext
    from autoawq_b200.program import DecodeProgram

    prev = ext.get_knob(14)
    ext.set_knob(14, 1 if no_fuse else 0)
    try:
        prog = DecodeProgram(max_tokens=M)
        bufs = record(prog)
        prog.build()
    finally:
        ext.set_knob(14, prev)
    return prog, bufs


def _fused_vs_replay(record_with, L, M, runs=(3, 7)):
    """The same program recorded twice (own caches each), fused and per op (the position tensor is shared).  After each
    run at the positions in `runs`: the fused q and cache rows are bit-identical to the stand-alone op on the fused qkv,
    nothing else of the caches changed, and every buffer is within tolerance of the per-op replay."""
    from autoawq_b200 import ext
    from test_gpu_program import _no_abort

    pos = torch.zeros(1, dtype=torch.int32, device=_dev())
    f_prog, f = _build(lambda p: record_with(p, pos, 0), M, False)
    r_prog, r = _build(lambda p: record_with(p, pos, 0), M, True)
    assert f_prog.fused and not r_prog.fused
    assert r_prog.launches_per_run == sum(6 if kind == "moe" else 1 for kind, _ in r_prog._ops)
    for p in runs:
        pos.fill_(p)
        k0, v0 = f["k"].clone(), f["v"].clone()
        f_prog.run()
        r_prog.run()
        torch.cuda.synchronize()
        _no_abort(f"pos {p}")
        rk, rv = k0.clone(), v0.clone()
        rq = ext.rope_kv_cache(f["qkv"], L.freqs, pos, rk, rv, L.H, L.KV)
        torch.cuda.synchronize()
        assert torch.equal(f["q"], rq) and torch.equal(f["k"], rk) and torch.equal(f["v"], rv), f"pos {p}"
        for k in f:
            d = float((f[k].float() - r[k].float()).abs().max())
            assert d <= 0.03 * float(r[k].float().abs().max()) + 0.03, f"pos {p}: {k} differs by {d}"
    return f_prog, f


def test_norm_qkv_rope_program_fuses_and_matches_replay():
    L = Layer(2048, 4096, 16, 4, 128, 256, seed=1)
    x = torch.randn((1, L.hidden), device=_dev()).half()

    def rec(api, pos, seed):
        kc, vc = _caches(1, L.S, L.KV, L.D, 9)
        xn = torch.empty_like(x)
        api.layernorm_forward_cuda(x, L.n1, xn, EPS)
        qkv = api.gemm_forward_cuda(xn, *L.w["qkv"], 8)
        q = api.rope_kv_cache(qkv, L.freqs, pos, kc, vc, L.H, L.KV)
        return dict(xn=xn, qkv=qkv, q=q, k=kc, v=vc)

    prog, f = _fused_vs_replay(rec, L, 1)
    assert prog.kernel_ops == 1 and prog.launches_per_run == 1


@pytest.mark.parametrize("M", [1, 2, 4])
def test_llama_segment_fuses_and_matches_replay(M):
    L = Layer(4096, 14336, 32, 8, 128, 2048, seed=10 + M)
    g = torch.Generator(device=_dev()).manual_seed(M)
    attn = torch.randn((M, L.hidden), device=_dev(), generator=g).half()
    h_in = torch.randn((M, L.hidden), device=_dev(), generator=g).half()

    def rec(api, pos, seed):
        kc, vc = _caches(M, L.S, L.KV, L.D, 5)
        return _record_segment(api, L, attn, h_in, pos, kc, vc)

    prog, _ = _fused_vs_replay(rec, L, M, runs=(0, 1, 1000, 2047))
    assert prog.kernel_ops == 4


def test_mixtral_segment_with_sparse_moe_fuses_and_matches_replay():
    moe = Moe(8, 1024, 768, 128, 2, seed=5)
    L = Layer(1024, 768, 8, 2, 64, 512, seed=30)
    attn = torch.randn((1, L.hidden), device=_dev()).half()
    h_in = torch.randn((1, L.hidden), device=_dev()).half()

    def rec(api, pos, seed):
        kc, vc = _caches(1, L.S, L.KV, L.D, 6)
        return _record_segment(api, L, attn, h_in, pos, kc, vc, moe=moe)

    prog, _ = _fused_vs_replay(rec, L, 1)
    assert prog.kernel_ops == 4


def test_rope_adds_no_kernel_op_and_keeps_the_other_outputs():
    """The same [norm, qkv] with and without a ROPE_KV: same kernel ops, the norm bit-identical, qkv within tolerance
    (mode 2 puts a column in another MMA row than mode 0)."""
    from autoawq_b200.program import DecodeProgram

    L = Layer(2048, 4096, 16, 4, 128, 256, seed=40)
    x = torch.randn((1, L.hidden), device=_dev()).half()
    outs = []
    for with_rope in (False, True):
        prog = DecodeProgram()
        xn = torch.empty_like(x)
        prog.layernorm_forward_cuda(x, L.n1, xn, EPS)
        qkv = prog.gemm_forward_cuda(xn, *L.w["qkv"], 8)
        if with_rope:
            kc, vc = _caches(1, L.S, L.KV, L.D, 1)
            prog.rope_kv_cache(qkv, L.freqs, torch.zeros(1, dtype=torch.int32, device=_dev()), kc, vc, L.H, L.KV)
        prog.build()
        assert prog.fused and prog.kernel_ops == 1
        prog.run()
        torch.cuda.synchronize()
        outs.append((xn.clone(), qkv.clone()))
    assert torch.equal(outs[0][0], outs[1][0])
    d = float((outs[0][1].float() - outs[1][1].float()).abs().max())
    assert d <= 0.03 * float(outs[0][1].float().abs().max()) + 0.03, d


def test_cuda_graph_replay_follows_the_position():
    from autoawq_b200 import ext

    L = Layer(2048, 4096, 16, 4, 128, 256, seed=50)
    x = torch.randn((1, L.hidden), device=_dev()).half()
    pos = torch.zeros(1, dtype=torch.int32, device=_dev())
    kc, vc = _caches(1, L.S, L.KV, L.D, 2)

    def rec(api):
        xn = torch.empty_like(x)
        api.layernorm_forward_cuda(x, L.n1, xn, EPS)
        qkv = api.gemm_forward_cuda(xn, *L.w["qkv"], 8)
        return qkv, api.rope_kv_cache(qkv, L.freqs, pos, kc, vc, L.H, L.KV)

    prog, (qkv, q) = _build(rec, 1, False)
    assert prog.fused
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        prog.run()                                  # warm-up outside the capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        prog.run()
    for p in (5, 6, 200):
        pos.fill_(p)
        k0, v0 = kc.clone(), vc.clone()
        graph.replay()
        torch.cuda.synchronize()
        rk, rv = k0.clone(), v0.clone()
        rq = ext.rope_kv_cache(qkv, L.freqs, pos, rk, rv, L.H, L.KV)
        torch.cuda.synchronize()
        assert torch.equal(q, rq) and torch.equal(kc, rk) and torch.equal(vc, rv), p
        assert not torch.equal(kc[:, p], k0[:, p])


@pytest.mark.parametrize("fuse", [True, False])
def test_out_of_range_position_writes_nothing_in_programs(fuse):
    L = Layer(2048, 4096, 16, 4, 128, 256, seed=60)
    x = torch.randn((1, L.hidden), device=_dev()).half()
    pos = torch.zeros(1, dtype=torch.int32, device=_dev())
    kc, vc = _caches(1, 128, L.KV, L.D, 3)                   # 128 cache rows, 256 frequency rows
    q = torch.full((1, L.H, L.D), 7.0, dtype=F16, device=_dev())

    def rec(api):
        xn = torch.empty_like(x)
        api.layernorm_forward_cuda(x, L.n1, xn, EPS)
        qkv = api.gemm_forward_cuda(xn, *L.w["qkv"], 8)
        api.rope_kv_cache(qkv, L.freqs, pos, kc, vc, L.H, L.KV, q_out=q)

    prog, _ = _build(rec, 1, not fuse)
    assert prog.fused == fuse
    k0, v0 = kc.clone(), vc.clone()
    for p in (128, 256, -1):
        pos.fill_(p)
        prog.run()
    torch.cuda.synchronize()
    assert torch.equal(kc, k0) and torch.equal(vc, v0) and bool((q == 7.0).all())


def test_fallbacks_replay_per_op_correctly():
    """A ROPE_KV after an add, and one whose q_out a later linear reads, replay per op with the stand-alone op's
    results."""
    from autoawq_b200 import ext
    from autoawq_b200.program import DecodeProgram

    L = Layer(2048, 4096, 16, 4, 128, 256, seed=70)
    x = torch.randn((1, L.hidden), device=_dev()).half()
    r = torch.randn((1, (L.H + 2 * L.KV) * L.D), device=_dev()).half()
    pos = torch.tensor([17], dtype=torch.int32, device=_dev())
    for case in ("after_add", "q_out_read"):
        kc, vc = _caches(1, L.S, L.KV, L.D, 4)
        k0, v0 = kc.clone(), vc.clone()
        prog = DecodeProgram()
        xn = torch.empty_like(x)
        prog.layernorm_forward_cuda(x, L.n1, xn, EPS)
        qkv = prog.gemm_forward_cuda(xn, *L.w["qkv"], 8)
        src = prog.add(qkv, r) if case == "after_add" else qkv
        q = prog.rope_kv_cache(src, L.freqs, pos, kc, vc, L.H, L.KV)
        if case == "q_out_read":
            o = prog.gemm_forward_cuda(q.view(1, L.H * L.D), *L.w["o"], 8)
        prog.build()
        assert not prog.fused, case
        prog.run()
        torch.cuda.synchronize()
        rq = ext.rope_kv_cache(src, L.freqs, pos, k0, v0, L.H, L.KV)
        torch.cuda.synchronize()
        assert torch.equal(q, rq) and torch.equal(kc, k0) and torch.equal(vc, v0), case
        if case == "q_out_read":
            assert torch.equal(o, ext.gemm_forward_cuda(rq.view(1, L.H * L.D), *L.w["o"], 8)), case
