"""GPU tests of partial rotary in RoPE + KV-cache append (b200awq_rope_t.rotary_dim; StableLM's partial_rotary_factor):
the mode-2 packer against the stream-format oracle, the stand-alone op against the reference's RoPE on the rotated
slice (plus the untouched tail and WindowedCache.update_kv) and against transformers' StableLM rotary, and decode
programs of StableLM segments and of an RMSNorm segment with partial rotary.

Bounds: the rotated columns within one fp16 ulp of the reference (torch's loops, DESIGN.md 3.5f), the pass-through
columns and v bit-exact; transformers computes in fp16 with fp16 cos / sin, so it is held to two fp16 ulps at the
largest |x| of each head.  A fused program's q and cache rows are bit-identical to the stand-alone op on the program's
own qkv; its other buffers are compared with the per-op replay within the tolerance of test_gpu_program_layernorm.py."""
import numpy as np
import pytest
import torch

from test_gpu_program import EPS as RMS_EPS
from test_gpu_program import _no_abort
from test_gpu_program_layernorm import _close
from test_gpu_program_rope import _build, _caches, _freqs, _linear, _ulps
from test_program_partial_rope_cpu import GEOMETRIES, STABLELM, partial_rotary_columns

pytestmark = pytest.mark.gpu

F16 = torch.float16
LN_EPS, THETA = 1e-5, 10000.0


def _dev():
    return torch.device("cuda:0")


# ------------------------------------------------------------------------------------------ stream format
@pytest.mark.parametrize("D,R", GEOMETRIES)
def test_stream_pack_partial_rotary_matches_oracle(D, R, monkeypatch):
    from autoawq_b200 import ext
    from oracle import stream_format as SF

    K, N, G = 512, 6 * D, 128
    qw, sc, qz = _linear(K, N, G, seed=D + R)
    orig = SF.set_columns
    monkeypatch.setattr(SF, "set_columns",
                        lambda n, mode: partial_rotary_columns(n, D, R) if mode == 2 else orig(n, mode))
    want = SF.pack_stream(qw.cpu().numpy(), qz.cpu().numpy(), sc.cpu().numpy(), G, 2)
    got = ext.stream_pack_rotary(qw, sc, qz, D, R)
    assert np.array_equal(got.cpu().numpy(), want)
    if R == D:
        assert torch.equal(got, ext.stream_pack_rotary(qw, sc, qz, D))


# ------------------------------------------------------------------------------------------ the stand-alone op
def _reference(qkv, rope, H, KV, D, R, p, M, cache):
    """RoPE(R).forward on the first R columns of q and k, the tail concatenated back, then update_kv.  Returns q."""
    x = qkv.view(M, 1, H + 2 * KV, D)
    xq, xk, xv = x[:, :, :H], x[:, :, H:H + KV], x[:, :, H + KV:]
    rq, rk = rope.forward(xq[..., :R], xk[..., :R], p, 1)
    q, k = torch.cat((rq, xq[..., R:]), -1), torch.cat((rk, xk[..., R:]), -1)
    cache.update_kv(values_store=xv, keys_store=k, batch_size=M, start_pos=p, seqlen=1)
    return q.reshape(M, H, D)


@pytest.mark.parametrize("M", [1, 2, 4])
@pytest.mark.parametrize("H,KV,D,R", [(32, 32, 80, 20), (16, 4, 64, 16), (8, 2, 160, 40), (8, 8, 128, 64)])
def test_rope_kv_cache_partial_matches_reference(M, H, KV, D, R):
    from autoawq_b200 import ext

    _freqs(8, 8, 1.0)                                       # imports the reference package
    from awq.modules.fused.attn import RoPE
    from awq.modules.fused.cache import WindowedCache

    S = 2048
    rope = RoPE(R, S, _dev(), THETA)
    g = torch.Generator(device=_dev()).manual_seed(M * D + R)
    qkv = (torch.randn((M, (H + 2 * KV) * D), device=_dev(), generator=g) * 3).half()
    for p in (0, 1, 1000, S - 1):
        cache = WindowedCache(M, H, KV, D, S, _dev())
        cache.k.normal_()
        cache.v.normal_()
        k0, v0 = cache.k.clone(), cache.v.clone()
        kc, vc = cache.k.clone(), cache.v.clone()
        ref_q = _reference(qkv, rope, H, KV, D, R, p, M, cache)
        pos = torch.tensor([p], dtype=torch.int32, device=_dev())
        q = ext.rope_kv_cache(qkv, rope.freqs_cis, pos, kc, vc, H, KV, head_dim=D)
        torch.cuda.synchronize()
        got, want = torch.cat([q, kc[:, p]], 1), torch.cat([ref_q, cache.k[:, p]], 1)
        assert int(_ulps(got[..., :R], want[..., :R]).max()) <= 1, f"pos {p}"
        assert torch.equal(got[..., R:], want[..., R:]), f"pos {p}: pass-through columns differ"
        assert torch.equal(vc, cache.v), f"pos {p}: v cache differs"
        rest = torch.ones(S, dtype=torch.bool, device=_dev())
        rest[p] = False
        assert torch.equal(kc[:, rest], k0[:, rest]) and torch.equal(vc[:, rest], v0[:, rest]), f"pos {p}"


def test_partial_out_of_range_position_writes_nothing():
    from autoawq_b200 import ext

    H, KV, D, R, S = 4, 2, 80, 20, 64
    short = _freqs(R, 16, THETA)                           # a table shorter than the cache
    qkv = torch.randn((2, (H + 2 * KV) * D), device=_dev()).half()
    kc, vc = _caches(2, S, KV, D, 1)
    k0, v0 = kc.clone(), vc.clone()
    q = torch.full((2, H, D), 7.0, dtype=F16, device=_dev())
    for freqs, p in ((_freqs(R, S, THETA), S), (_freqs(R, S, THETA), -1), (short, 16), (short, 40)):
        ext.rope_kv_cache(qkv, freqs, torch.tensor([p], dtype=torch.int32, device=_dev()), kc, vc, H, KV, q_out=q,
                          head_dim=D)
    torch.cuda.synchronize()
    assert torch.equal(kc, k0) and torch.equal(vc, v0) and bool((q == 7.0).all())


@pytest.mark.parametrize("D,R", [g for g in GEOMETRIES if g[1] < g[0]])
def test_rope_kv_cache_partial_matches_transformers_stablelm(D, R):
    """transformers' StableLmRotaryEmbedding + apply_rotary_pos_emb on the first R columns (StableLmAttention.forward),
    within two fp16 ulps at the largest |x| of each head."""
    from autoawq_b200 import ext
    from transformers import StableLmConfig
    from transformers.models.stablelm.modeling_stablelm import StableLmRotaryEmbedding, apply_rotary_pos_emb

    H, KV, M, S = 8, 8, 2, 2048
    cfg = StableLmConfig(hidden_size=H * D, num_attention_heads=H, num_key_value_heads=KV, partial_rotary_factor=R / D,
                         max_position_embeddings=S, rope_theta=THETA)
    rot = StableLmRotaryEmbedding(cfg, device=_dev())
    freqs = _freqs(R, S, THETA)
    g = torch.Generator(device=_dev()).manual_seed(D + R)
    qkv = (torch.randn((M, (H + 2 * KV) * D), device=_dev(), generator=g) * 3).half()
    worst = 0.0
    for p in (1, 1000, S - 1):
        kc, vc = _caches(M, S, KV, D, 2)
        pos = torch.tensor([p], dtype=torch.int32, device=_dev())
        q = ext.rope_kv_cache(qkv, freqs, pos, kc, vc, H, KV, head_dim=D)
        torch.cuda.synchronize()
        x = qkv.view(M, H + 2 * KV, 1, D)                   # [batch, heads, seq, dim]
        xq, xk = x[:, :H], x[:, H:H + KV]
        cos, sin = rot(qkv, torch.full((M, 1), p, dtype=torch.long, device=_dev()))
        rq, rk = apply_rotary_pos_emb(xq[..., :R], xk[..., :R], cos, sin)
        want = torch.cat([torch.cat((rq, xq[..., R:]), -1), torch.cat((rk, xk[..., R:]), -1)], 1).reshape(M, H + KV, D)
        got = torch.cat([q, kc[:, p]], 1)
        diff = (got.float() - want.float()).abs()
        top = want.float().abs().amax(-1, keepdim=True)
        ulp = torch.exp2(torch.floor(torch.log2(top)) - 10)
        worst = max(worst, float(diff.max()))
        assert bool((diff <= 2 * ulp).all()), f"pos {p}: largest difference {float(diff.max())}"
        assert torch.equal(got[..., R:], want[..., R:])
    print(f"D={D} R={R}: largest difference from transformers {worst}")


# ------------------------------------------------------------------------------------------ decode programs
class StableLmBlock:
    """One StableLM layer's random GEMM-layout AWQ weights, LayerNorms (with bias) and biases at a model's geometry."""

    def __init__(self, model, seed, S=64):
        hid, H, KV, D, R, inter, qkv_bias = STABLELM[model]
        self.hid, self.H, self.KV, self.D, self.R, self.inter, self.S = hid, H, KV, D, R, inter, S
        shapes = dict(o=(H * D, hid), gu=(hid, 2 * inter), down=(inter, hid), qkv=(hid, (H + 2 * KV) * D))
        self.w = {k: _linear(K, N, 128, seed + i) for i, (k, (K, N)) in enumerate(sorted(shapes.items()))}
        g = torch.Generator(device=_dev()).manual_seed(seed + 10)
        self.qkv_bias = (0.05 * torch.randn(shapes["qkv"][1], device=_dev(), generator=g)).half() if qkv_bias else None
        self.ln = {n: ((1 + 0.1 * torch.randn(hid, device=_dev(), generator=g)).half(),
                       (0.05 * torch.randn(hid, device=_dev(), generator=g)).half()) for n in ("n1", "n2")}
        self.freqs = _freqs(R, S, THETA)

    def record(self, api, pos, attn, x):
        """The segment in program.py's StableLM recording order; returns the buffers it names."""
        M = attn.shape[0]
        o = api.gemm_forward_cuda(attn, *self.w["o"], 8)
        h = api.add(o, x)
        hn = torch.empty((M, self.hid), dtype=F16, device=_dev())
        api.layer_norm(h, *self.ln["n2"], hn, LN_EPS)
        gu = api.gemm_forward_cuda(hn, *self.w["gu"], 8)
        act = torch.empty((M, self.inter), dtype=F16, device=_dev())
        api.silu_and_mul(act, gu)
        dn = api.gemm_forward_cuda(act, *self.w["down"], 8)
        out = api.add(dn, h)
        xn = torch.empty((M, self.hid), dtype=F16, device=_dev())
        api.layer_norm(out, *self.ln["n1"], xn, LN_EPS)
        qkv = api.gemm_forward_cuda(xn, *self.w["qkv"], 8, bias=self.qkv_bias)
        kc, vc = _caches(M, self.S, self.KV, self.D, 5)
        q = api.rope_kv_cache(qkv, self.freqs, pos, kc, vc, self.H, self.KV, head_dim=self.D)
        return dict(o=o, h=h, hn=hn, gu=gu, act=act, dn=dn, out=out, xn=xn, qkv=qkv, q=q, k=kc, v=vc)

    def check_fused_ops(self, f, pos):
        """The fused program's LayerNorm outputs and rotation against the stand-alone ops on its own inputs."""
        from autoawq_b200 import ext

        for src, dst, n in (("h", "hn", "n2"), ("out", "xn", "n1")):
            want = torch.empty_like(f[dst])
            ext.layer_norm(f[src], *self.ln[n], want, LN_EPS)
            assert torch.equal(f[dst], want), dst
        k0, v0 = _caches(f["k"].shape[0], self.S, self.KV, self.D, 5)
        rq = ext.rope_kv_cache(f["qkv"], self.freqs, pos, k0, v0, self.H, self.KV, head_dim=self.D)
        assert torch.equal(f["q"], rq) and torch.equal(f["k"], k0) and torch.equal(f["v"], v0)


def _inputs(B, M, seed):
    g = torch.Generator(device=_dev()).manual_seed(seed)
    return ((torch.randn((M, B.H * B.D), device=_dev(), generator=g) * 0.5).half(),
            torch.randn((M, B.hid), device=_dev(), generator=g).half())


@pytest.mark.parametrize("model", sorted(STABLELM))
def test_stablelm_segment_fuses_into_one_launch_and_matches_replay(model):
    B = StableLmBlock(model, seed=len(model))
    attn, x = _inputs(B, 1, 3)
    pos = torch.full((1,), 5, dtype=torch.int32, device=_dev())
    f_prog, f = _build(lambda p: B.record(p, pos, attn, x), 1, False)
    r_prog, r = _build(lambda p: B.record(p, pos, attn, x), 1, True)
    assert f_prog.fused and f_prog.kernel_ops == 4 and f_prog.launches_per_run == 1
    assert not r_prog.fused and r_prog.launches_per_run == len(r_prog._ops)
    f_prog.run()
    r_prog.run()
    torch.cuda.synchronize()
    _no_abort(model)
    B.check_fused_ops(f, pos)
    _close(f, r, f.keys())


def test_stablelm_cuda_graph_replay_follows_the_position():
    B = StableLmBlock("stablelm-3b-4e1t", seed=7)
    attn, x = _inputs(B, 1, 4)
    pos = torch.zeros(1, dtype=torch.int32, device=_dev())
    prog, f = _build(lambda p: B.record(p, pos, attn, x), 1, False)
    assert prog.fused
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        prog.run()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        prog.run()
    k0, v0 = _caches(1, B.S, B.KV, B.D, 5)
    for p in (1, 9, 30):
        pos.fill_(p)
        f["k"].copy_(k0)
        f["v"].copy_(v0)
        graph.replay()
        torch.cuda.synchronize()
        _no_abort(f"pos {p}")
        assert not torch.equal(f["k"][0, p], k0[0, p])
        B.check_fused_ops(f, pos)


def _rms_segment(api, w, n1, n2, freqs, pos, attn, h_in, caches, H, KV, D):
    """[o + h, norm2, gate|up, silu, down + h, norm1', qkv', rope'(head_dim=D)] with a partial table."""
    M, hid = h_in.shape
    o = api.gemm_forward_cuda(attn, *w["o"], 8)
    h = api.add(o, h_in)
    xn2 = torch.empty((M, hid), dtype=F16, device=_dev())
    api.layernorm_forward_cuda(h, n2, xn2, RMS_EPS)
    gu = api.gemm_forward_cuda(xn2, *w["gu"], 8)
    act = torch.empty((M, gu.shape[1] // 2), dtype=F16, device=_dev())
    api.silu_and_mul(act, gu)
    dn = api.gemm_forward_cuda(act, *w["down"], 8)
    out = api.add(dn, h)
    xn = torch.empty((M, hid), dtype=F16, device=_dev())
    api.layernorm_forward_cuda(out, n1, xn, RMS_EPS)
    qkv = api.gemm_forward_cuda(xn, *w["qkv"], 8)
    kc, vc = caches
    q = api.rope_kv_cache(qkv, freqs, pos, kc, vc, H, KV, head_dim=D)
    return dict(o=o, h=h, xn2=xn2, gu=gu, act=act, dn=dn, out=out, xn=xn, qkv=qkv, q=q, k=kc, v=vc)


@pytest.mark.parametrize("M", [2, 4, 8])
def test_rmsnorm_segment_with_partial_rotary_batched_matches_single_rows(M):
    """Fused at M token rows; every row bit-identical to an M = 1 program run on that row alone."""
    hid, inter, H, KV, D, R, S = 2048, 4096, 32, 8, 128, 64, 256
    w = dict(o=_linear(H * D, hid, 128, 1), gu=_linear(hid, 2 * inter, 128, 2), down=_linear(inter, hid, 128, 3),
             qkv=_linear(hid, (H + 2 * KV) * D, 128, 4))
    g = torch.Generator(device=_dev()).manual_seed(M)
    n1, n2 = ((1 + 0.1 * torch.randn(hid, device=_dev(), generator=g)).half() for _ in range(2))
    freqs = _freqs(R, S, 500000.0)
    attn = torch.randn((M, H * D), device=_dev(), generator=g).half()
    h_in = torch.randn((M, hid), device=_dev(), generator=g).half()
    pos = torch.full((1,), 17, dtype=torch.int32, device=_dev())
    caches = _caches(M, S, KV, D, 6)
    k0, v0 = caches[0].clone(), caches[1].clone()
    prog, f = _build(lambda p: _rms_segment(p, w, n1, n2, freqs, pos, attn, h_in, caches, H, KV, D), M, False)
    assert prog.fused and prog.tokens == M and prog.kernel_ops == 4
    prog.run()
    torch.cuda.synchronize()
    _no_abort(f"M={M}")
    for m in range(M):
        one = (k0[m:m + 1].clone(), v0[m:m + 1].clone())
        p1, s = _build(lambda p: _rms_segment(p, w, n1, n2, freqs, pos, attn[m:m + 1], h_in[m:m + 1], one, H, KV, D),
                       1, False)
        assert p1.fused
        p1.run()
        torch.cuda.synchronize()
        for k in f:
            assert torch.equal(f[k][m:m + 1], s[k]), f"M={M} row {m}: {k}"
