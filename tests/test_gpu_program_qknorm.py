"""GPU tests of Qwen3's q / k norm in front of RoPE + KV-cache append (B200AWQ_OP_QK_NORM_ROPE_KV): the stand-alone op
against an ordered-sum oracle (bit for bit) and against transformers' Qwen3RMSNorm followed by the reference's
RoPE.forward + WindowedCache.update_kv, and decode programs that fold the op into the qkv linear's finish.

Bit-identity and where it stops:
  * the op sums each head's squares in one fixed order (include/b200awq.h); the oracle below repeats that order in
    numpy float32 and takes r with torch.rsqrt on the device, then feeds the normalised q / k through the existing
    ext.rope_kv_cache: the op must equal it bit for bit;
  * torch.mean sums in another order, so against the reference chain r may differ in its last bit: q and k are held to
    2 fp16 ulps there, v (never normalised) to bit identity;
  * a fused program's q and cache rows are bit-identical to the stand-alone op applied to the program's own qkv output;
  * the linears are not bit-identical between a fused program and the per-op replay (test_gpu_program_rope.py explains
    why), so the other buffers are compared within the same tolerance as there."""
import numpy as np
import pytest
import torch

from test_gpu_program import EPS
from test_gpu_program_rope import _build, _caches, _freqs, _linear, _ulps

pytestmark = pytest.mark.gpu

F16 = torch.float16
QK_EPS = 1e-6


def _dev():
    return torch.device("cuda:0")


def _norms(D, seed):
    """Qwen3's q_norm / k_norm (transformers' Qwen3RMSNorm) with random fp16 weights around 1."""
    from transformers.models.qwen3.modeling_qwen3 import Qwen3RMSNorm

    g = torch.Generator(device=_dev()).manual_seed(seed)
    out = []
    for _ in range(2):
        n = Qwen3RMSNorm(D, eps=QK_EPS).to(_dev()).half()
        with torch.no_grad():
            n.weight.copy_((1 + 0.2 * torch.randn(D, device=_dev(), generator=g)).half())
        out.append(n)
    return out


def _oracle_norm(qkv, H, KV, D, qn, kn):
    """qkv with every q / k head normalised: the head's sum of squares in the op's order (numpy float32: per pair
    a^2 + b^2, the 8-lane xor butterfly 4, 2, 1 of each set of 8 pairs, the sets in ascending order), r = torch.rsqrt
    on the device, then fp16(w * fp16(x * r))."""
    M = qkv.shape[0]
    x = qkv.cpu().numpy().reshape(M, H + 2 * KV, D)[:, : H + KV].astype(np.float32)
    a, b = x[..., : D // 2], x[..., D // 2:]
    s = (a * a + b * b).reshape(M, H + KV, D // 16, 8)                       # [.., set, lane]
    v = s + s[..., [g ^ 4 for g in range(8)]]
    v = v + v[..., [g ^ 2 for g in range(8)]]
    v = v + v[..., [g ^ 1 for g in range(8)]]
    part = v[..., 0]
    tot = np.zeros((M, H + KV), dtype=np.float32)
    for t in range(D // 16):
        tot = (tot + part[..., t]).astype(np.float32)
    var = (tot * np.float32(1.0 / D)).astype(np.float32) + np.float32(QK_EPS)
    r = torch.rsqrt(torch.from_numpy(var.astype(np.float32)).to(_dev())).cpu().numpy()
    xn = (x * r[..., None]).astype(np.float16).astype(np.float32)
    w = np.stack([qn.weight.detach().float().cpu().numpy()] * H + [kn.weight.detach().float().cpu().numpy()] * KV)
    y = (w[None] * xn).astype(np.float16)
    out = qkv.clone().view(M, H + 2 * KV, D)
    out[:, : H + KV] = torch.from_numpy(y).to(_dev())
    return out.view(M, -1)


# ------------------------------------------------------------------------------------------ the stand-alone op
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("M", [1, 2, 4])
def test_qk_norm_rope_kv_matches_ordered_oracle(M, D):
    from autoawq_b200 import ext

    H, KV, S = 16, 4, 256
    freqs = _freqs(D, S, 1e6)
    qn, kn = _norms(D, seed=D + M)
    g = torch.Generator(device=_dev()).manual_seed(100 * M + D)
    qkv = (torch.randn((M, (H + 2 * KV) * D), device=_dev(), generator=g) * 3).half()
    qkv[0, :D] *= 40                                            # one loud head: large sums of squares
    for p in (0, 77, S - 1):
        pos = torch.tensor([p], dtype=torch.int32, device=_dev())
        kc, vc = _caches(M, S, KV, D, 7)
        rk, rv = kc.clone(), vc.clone()
        q = ext.rope_kv_cache(qkv, freqs, pos, kc, vc, H, KV, q_norm=qn, k_norm=kn)
        rq = ext.rope_kv_cache(_oracle_norm(qkv, H, KV, D, qn, kn), freqs, pos, rk, rv, H, KV)
        torch.cuda.synchronize()
        assert torch.equal(q, rq) and torch.equal(kc, rk) and torch.equal(vc, rv), f"pos {p}"


@pytest.mark.parametrize("M", [1, 2, 4])
def test_qk_norm_rope_kv_matches_reference_chain(M):
    """Qwen3-8B attention shapes (32 / 8 / 128, theta 1e6): Qwen3RMSNorm -> RoPE.forward -> update_kv.  q and the k row
    within 2 fp16 ulps (the mean's summation order differs), the v row bit-identical, every other cache row untouched."""
    from autoawq_b200 import ext

    _freqs(8, 8, 1.0)                                       # imports the reference package
    from awq.modules.fused.attn import RoPE
    from awq.modules.fused.cache import WindowedCache

    H, KV, D, S = 32, 8, 128, 2048
    rope = RoPE(D, S, _dev(), 1e6)
    qn, kn = _norms(D, seed=M)
    g = torch.Generator(device=_dev()).manual_seed(M)
    qkv = (torch.randn((M, (H + 2 * KV) * D), device=_dev(), generator=g) * 3).half()
    for p in (0, 1000, 2047):
        cache = WindowedCache(M, H, KV, D, S, _dev())
        cache.k.normal_()
        cache.v.normal_()
        k0, v0 = cache.k.clone(), cache.v.clone()
        kc, vc = cache.k.clone(), cache.v.clone()
        xqkv = qkv.view(M, 1, H + 2 * KV, D)
        with torch.no_grad():
            xq, xk = qn(xqkv[:, :, :H]), kn(xqkv[:, :, H:H + KV])
            xq, xk = rope.forward(xq, xk, p, 1)
        cache.update_kv(values_store=xqkv[:, :, H + KV:], keys_store=xk, batch_size=M, start_pos=p, seqlen=1)
        pos = torch.tensor([p], dtype=torch.int32, device=_dev())
        q = ext.rope_kv_cache(qkv, rope.freqs_cis, pos, kc, vc, H, KV, q_norm=qn, k_norm=kn)
        torch.cuda.synchronize()
        got = torch.cat([q, kc[:, p]], 1)
        want = torch.cat([xq.reshape(M, H, D), cache.k[:, p]], 1)
        ulps = _ulps(got, want)
        print(f"qk-norm vs reference chain M={M} pos={p}: {int((ulps > 0).sum())} of {ulps.numel()} q/k elements "
              f"differ (max {int(ulps.max())} ulp)")
        assert int(ulps.max()) <= 2, f"pos {p}: {int((ulps > 2).sum())} elements > 2 ulps"
        assert torch.equal(vc, cache.v), f"pos {p}: v cache differs"
        rest = torch.ones(S, dtype=torch.bool, device=_dev())
        rest[p] = False
        assert torch.equal(kc[:, rest], k0[:, rest]) and torch.equal(vc[:, rest], v0[:, rest])


def test_out_of_range_position_writes_nothing():
    from autoawq_b200 import ext

    H, KV, D, S = 4, 2, 64, 64
    freqs = _freqs(D, S, 1e6)
    qn, kn = _norms(D, seed=3)
    qkv = torch.randn((2, (H + 2 * KV) * D), device=_dev()).half()
    kc, vc = _caches(2, S, KV, D, 1)
    k0, v0 = kc.clone(), vc.clone()
    q = torch.full((2, H, D), 7.0, dtype=F16, device=_dev())
    for p in (S, -1):
        ext.rope_kv_cache(qkv, freqs, torch.tensor([p], dtype=torch.int32, device=_dev()), kc, vc, H, KV, q_out=q,
                          q_norm=qn, k_norm=kn)
    torch.cuda.synchronize()
    assert torch.equal(kc, k0) and torch.equal(vc, v0) and bool((q == 7.0).all())


def test_norm_arguments_are_checked():
    from autoawq_b200 import ext
    from autoawq_b200.ext import B200AwqError

    H, KV, D, S = 4, 2, 64, 64
    freqs = _freqs(D, S, 1e6)
    qn, kn = _norms(D, seed=4)
    qkv = torch.randn((1, (H + 2 * KV) * D), device=_dev()).half()
    kc, vc = _caches(1, S, KV, D, 1)
    pos = torch.zeros(1, dtype=torch.int32, device=_dev())
    with pytest.raises(B200AwqError):
        ext.rope_kv_cache(qkv, freqs, pos, kc, vc, H, KV, q_norm=qn)
    with pytest.raises(B200AwqError):
        ext.rope_kv_cache(qkv, freqs, pos, kc, vc, H, KV, k_norm=kn)
    kn.variance_epsilon = 1e-5
    with pytest.raises(B200AwqError):
        ext.rope_kv_cache(qkv, freqs, pos, kc, vc, H, KV, q_norm=qn, k_norm=kn)


# ------------------------------------------------------------------------------------------ decode programs
class Qwen3Layer:
    """One Qwen3 decoder layer's weights (GEMM-layout AWQ, random), its q / k norms and its attention geometry."""

    def __init__(self, hidden, inter, H, KV, D, S, seed, G=128):
        self.hidden, self.inter, self.H, self.KV, self.D, self.S = hidden, inter, H, KV, D, S
        self.w = dict(o=_linear(H * D, hidden, G, seed), gu=_linear(hidden, 2 * inter, G, seed + 1),
                      down=_linear(inter, hidden, G, seed + 2), qkv=_linear(hidden, (H + 2 * KV) * D, G, seed + 3))
        g = torch.Generator(device=_dev()).manual_seed(seed + 4)
        self.n1 = (1 + 0.1 * torch.randn(hidden, device=_dev(), generator=g)).half()
        self.n2 = (1 + 0.1 * torch.randn(hidden, device=_dev(), generator=g)).half()
        self.freqs = _freqs(D, S, 1e6)
        self.qn, self.kn = _norms(D, seed + 5)


def _record_segment(api, L, attn, h_in, pos, kc, vc):
    """[o + h, norm2, gate|up, silu, down + h, norm1', qkv', qk-norm-rope'] of a Qwen3 layer against `api`."""
    M = attn.shape[0]
    o = api.gemm_forward_cuda(attn, *L.w["o"], 8)
    h = api.add(o, h_in)
    xn2 = torch.empty((M, L.hidden), dtype=F16, device=_dev())
    api.layernorm_forward_cuda(h, L.n2, xn2, EPS)
    gu = api.gemm_forward_cuda(xn2, *L.w["gu"], 8)
    act = torch.empty((M, L.inter), dtype=F16, device=_dev())
    api.silu_and_mul(act, gu)
    dn = api.gemm_forward_cuda(act, *L.w["down"], 8)
    out = api.add(dn, h)
    xn = torch.empty((M, L.hidden), dtype=F16, device=_dev())
    api.layernorm_forward_cuda(out, L.n1, xn, EPS)
    qkv = api.gemm_forward_cuda(xn, *L.w["qkv"], 8)
    q = api.rope_kv_cache(qkv, L.freqs, pos, kc, vc, L.H, L.KV, q_norm=L.qn, k_norm=L.kn)
    return dict(o=o, h=h, xn2=xn2, gu=gu, act=act, dn=dn, out=out, xn=xn, qkv=qkv, q=q, k=kc, v=vc)


def _standalone(L, qkv, pos, k0, v0):
    from autoawq_b200 import ext

    rk, rv = k0.clone(), v0.clone()
    rq = ext.rope_kv_cache(qkv, L.freqs, pos, rk, rv, L.H, L.KV, q_norm=L.qn, k_norm=L.kn)
    torch.cuda.synchronize()
    return rq, rk, rv


def _fused_vs_replay(record_with, L, M, runs=(3, 7)):
    """The same program recorded twice (own caches each), fused and per op under knob 14 = 1 (the position tensor is
    shared).  After each run: the fused q and cache rows equal the stand-alone op on the fused qkv bit for bit, and every
    buffer is within tolerance of the per-op replay."""
    from test_gpu_program import _no_abort

    pos = torch.zeros(1, dtype=torch.int32, device=_dev())
    f_prog, f = _build(lambda p: record_with(p, pos), M, False)
    r_prog, r = _build(lambda p: record_with(p, pos), M, True)
    assert f_prog.fused and not r_prog.fused
    for p in runs:
        pos.fill_(p)
        k0, v0 = f["k"].clone(), f["v"].clone()
        f_prog.run()
        r_prog.run()
        torch.cuda.synchronize()
        _no_abort(f"pos {p}")
        rq, rk, rv = _standalone(L, f["qkv"], pos, k0, v0)
        assert torch.equal(f["q"], rq) and torch.equal(f["k"], rk) and torch.equal(f["v"], rv), f"pos {p}"
        for k in f:
            d = float((f[k].float() - r[k].float()).abs().max())
            assert d <= 0.03 * float(r[k].float().abs().max()) + 0.03, f"pos {p}: {k} differs by {d}"
    return f_prog, f


def test_norm_qkv_qknorm_program_fuses_and_matches_standalone():
    L = Qwen3Layer(4096, 12288, 32, 8, 128, 256, seed=1)
    x = torch.randn((1, L.hidden), device=_dev()).half()

    def rec(api, pos):
        kc, vc = _caches(1, L.S, L.KV, L.D, 9)
        xn = torch.empty_like(x)
        api.layernorm_forward_cuda(x, L.n1, xn, EPS)
        qkv = api.gemm_forward_cuda(xn, *L.w["qkv"], 8)
        q = api.rope_kv_cache(qkv, L.freqs, pos, kc, vc, L.H, L.KV, q_norm=L.qn, k_norm=L.kn)
        return dict(xn=xn, qkv=qkv, q=q, k=kc, v=vc)

    prog, _ = _fused_vs_replay(rec, L, 1)
    assert prog.kernel_ops == 1 and prog.launches_per_run == 1


@pytest.mark.parametrize("M", [1, 2, 4])
def test_qwen3_8b_segment_fuses_and_matches(M):
    L = Qwen3Layer(4096, 12288, 32, 8, 128, 2048, seed=10 + M)
    g = torch.Generator(device=_dev()).manual_seed(M)
    attn = torch.randn((M, L.H * L.D), device=_dev(), generator=g).half()
    h_in = torch.randn((M, L.hidden), device=_dev(), generator=g).half()

    def rec(api, pos):
        kc, vc = _caches(M, L.S, L.KV, L.D, 5)
        return _record_segment(api, L, attn, h_in, pos, kc, vc)

    prog, _ = _fused_vs_replay(rec, L, M, runs=(0, 1, 1000, 2047))
    assert prog.kernel_ops == 4


def test_qwen3_4b_segment_fuses_and_matches():
    """hidden 2560 != H D = 4096: o maps 4096 -> 2560, qkv 2560 -> 6144."""
    L = Qwen3Layer(2560, 9728, 32, 8, 128, 512, seed=30)
    attn = torch.randn((1, L.H * L.D), device=_dev()).half()
    h_in = torch.randn((1, L.hidden), device=_dev()).half()

    def rec(api, pos):
        kc, vc = _caches(1, L.S, L.KV, L.D, 6)
        return _record_segment(api, L, attn, h_in, pos, kc, vc)

    prog, _ = _fused_vs_replay(rec, L, 1)
    assert prog.kernel_ops == 4


def test_cuda_graph_replay_follows_the_position():
    L = Qwen3Layer(2048, 4096, 16, 4, 128, 256, seed=50)
    x = torch.randn((1, L.hidden), device=_dev()).half()
    pos = torch.zeros(1, dtype=torch.int32, device=_dev())
    kc, vc = _caches(1, L.S, L.KV, L.D, 2)

    def rec(api):
        xn = torch.empty_like(x)
        api.layernorm_forward_cuda(x, L.n1, xn, EPS)
        qkv = api.gemm_forward_cuda(xn, *L.w["qkv"], 8)
        return qkv, api.rope_kv_cache(qkv, L.freqs, pos, kc, vc, L.H, L.KV, q_norm=L.qn, k_norm=L.kn)

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
        rq, rk, rv = _standalone(L, qkv, pos, k0, v0)
        assert torch.equal(q, rq) and torch.equal(kc, rk) and torch.equal(vc, rv), p
        assert not torch.equal(kc[:, p], k0[:, p])


@pytest.mark.parametrize("fuse", [True, False])
def test_out_of_range_position_writes_nothing_in_programs(fuse):
    L = Qwen3Layer(2048, 4096, 16, 4, 128, 256, seed=60)
    x = torch.randn((1, L.hidden), device=_dev()).half()
    pos = torch.zeros(1, dtype=torch.int32, device=_dev())
    kc, vc = _caches(1, 128, L.KV, L.D, 3)                   # 128 cache rows, 256 frequency rows
    q = torch.full((1, L.H, L.D), 7.0, dtype=F16, device=_dev())

    def rec(api):
        xn = torch.empty_like(x)
        api.layernorm_forward_cuda(x, L.n1, xn, EPS)
        qkv = api.gemm_forward_cuda(xn, *L.w["qkv"], 8)
        api.rope_kv_cache(qkv, L.freqs, pos, kc, vc, L.H, L.KV, q_out=q, q_norm=L.qn, k_norm=L.kn)

    prog, _ = _build(rec, 1, not fuse)
    assert prog.fused == fuse
    k0, v0 = kc.clone(), vc.clone()
    for p in (128, 256, -1):
        pos.fill_(p)
        prog.run()
    torch.cuda.synchronize()
    assert torch.equal(kc, k0) and torch.equal(vc, v0) and bool((q == 7.0).all())


def test_fallbacks_replay_per_op_correctly():
    """A q / k norm op after an add, and one whose q_out a later linear reads, replay per op with the stand-alone op's
    results."""
    from autoawq_b200 import ext
    from autoawq_b200.program import DecodeProgram

    L = Qwen3Layer(2048, 4096, 16, 4, 128, 256, seed=70)
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
        q = prog.rope_kv_cache(src, L.freqs, pos, kc, vc, L.H, L.KV, q_norm=L.qn, k_norm=L.kn)
        if case == "q_out_read":
            o = prog.gemm_forward_cuda(q.view(1, L.H * L.D), *L.w["o"], 8)
        prog.build()
        assert not prog.fused, case
        prog.run()
        torch.cuda.synchronize()
        rq, rk, rv = _standalone(L, src, pos, k0, v0)
        assert torch.equal(q, rq) and torch.equal(kc, rk) and torch.equal(vc, rv), case
        if case == "q_out_read":
            assert torch.equal(o, ext.gemm_forward_cuda(rq.view(1, L.H * L.D), *L.w["o"], 8)), case
