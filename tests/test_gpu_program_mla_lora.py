"""MLA with a q LoRA in decode programs (DecodeProgram.mla_k_rope / mla_q_rope, B200AWQ_OP_MLA_K_ROPE / _MLA_Q_ROPE) and
the stand-alone ops (ext.mla_k_rope / ext.mla_q_rope), at DeepSeek-V3 attention shapes (H 128, Dn 128, Dr 64, Dv 128,
C 512, Cq 1536, hidden 7168) and at a narrower geometry whose fused q_a | kv_a row has fewer 16-column sets than SMs
(H 40, Dn 64, Dr 32, Dv 64, C 256, Cq 768, hidden 2560):
  * the stand-alone ops against transformers' apply_rotary_emb (V2, within one fp16 ulp) and
    apply_rotary_pos_emb_interleave (V3, bit-exact), q_nope bit-exact, at M = 1, 2, 4, every other cache row untouched
    and nothing written for a position outside the cache or the table;
  * the fused [norm1, q_a|kv_a, mla_k_rope, norm(q_a), q_b, mla_q_rope, norm(c_kv), kv_b, mla_kv] (three kernel ops)
    bit-identical to the stand-alone ops on the program's own recorded rows;
  * query / key / value states against transformers' DeepseekV2Attention / DeepseekV3Attention with q_lora_rank set;
  * the dense DeepSeek-V3 segment as one launch, within the dense tests' bounds of its knob-14 replay, and in a CUDA
    graph replayed at a moving position;
  * the chain recorded at M = 2, replayed per op, against the stand-alone ops."""
import numpy as np
import pytest
import torch

from autoawq_b200 import ext
from autoawq_b200.program import DecodeProgram
from test_gpu_program import _no_abort
from test_gpu_program_deepseek_moe import _ulps_of_rms
from test_gpu_program_mla import _Capture, _capture_attention, _hf_rot, _ulp_diff
import test_gpu_program_mla as mla_test

pytestmark = pytest.mark.gpu

G, EPS = 128, 1e-6


class Geo:
    def __init__(self, H, DN, DR, DV, C, CQ, HID, INTER):
        self.H, self.DN, self.DR, self.DV, self.C, self.CQ, self.HID, self.INTER = H, DN, DR, DV, C, CQ, HID, INTER
        self.W = DN + DR
        self.N_QA, self.N_QB, self.N_KV = CQ + C + DR, H * self.W, H * (DN + DV)


V3 = Geo(128, 128, 64, 128, 512, 1536, 7168, 18432)
NARROW = Geo(40, 64, 32, 64, 256, 768, 2560, 6912)
GEOS = pytest.mark.parametrize("g", [V3, NARROW], ids=["v3", "narrow"])


def _dev():
    return torch.device("cuda:0")


def _gen(seed):
    return torch.Generator(device=_dev()).manual_seed(seed)


def _lin(K, N, gen):
    return (torch.randint(-2**31, 2**31 - 1, (K, N // 8), dtype=torch.int32, device=_dev(), generator=gen),
            ((torch.rand((K // G, N), device=_dev(), generator=gen) * 0.5 + 0.75) / (6.1 * K**0.5)).half(),
            torch.randint(-2**31, 2**31 - 1, (K // G, N // 8), dtype=torch.int32, device=_dev(), generator=gen))


def _tables(g, S_f, theta=10000.0, scaling=1.2247):
    """(freqs_cis complex64 [S_f, Dr/2], (cos, sin) f32 [S_f, Dr]) with attention_scaling (a yarn mscale) applied."""
    inv = 1.0 / (theta ** (torch.arange(0, g.DR, 2, dtype=torch.int64, device=_dev()).float() / g.DR))
    f = torch.outer(torch.arange(S_f, device=_dev()).float(), inv)
    cis = torch.polar(torch.ones_like(f), f) * scaling
    emb = torch.cat((f, f), dim=-1)
    return cis, (emb.cos() * scaling, emb.sin() * scaling)


def _check_rot(style, got, ref):
    d = _ulp_diff(got, ref)
    assert d.max() <= (1 if style == 0 else 0), d.max()


@GEOS
@pytest.mark.parametrize("style", [0, 1])
@pytest.mark.parametrize("M", [1, 2, 4])
def test_standalone_ops_against_transformers(g, style, M):
    gen = _gen(10 * M + style)
    S, pos = 64, 37
    cis, cs = _tables(g, 128)
    freqs = cis if style == 0 else cs
    qa = (torch.randn((M, g.N_QA), device=_dev(), generator=gen) * 2).half()
    qb = (torch.randn((M, g.N_QB), device=_dev(), generator=gen) * 2).half()
    k_cache = torch.randn((M + 1, S, g.H, g.W), device=_dev(), generator=gen).half()
    k0 = k_cache.clone()
    p = torch.tensor([pos], dtype=torch.int32, device=_dev())
    ext.mla_k_rope(qa, freqs, p, k_cache, g.H, g.DN, g.DR, g.C, g.CQ, style)
    q_out = ext.mla_q_rope(qb, freqs, p, S, g.H, g.DN, g.DR, style)
    torch.cuda.synchronize()
    q = qb.view(M, 1, g.H, g.W).transpose(1, 2)
    q_nope, q_pe = torch.split(q, [g.DN, g.DR], dim=-1)
    k_pe = qa[:, g.CQ + g.C:].view(M, 1, 1, g.DR)
    rq, rk = _hf_rot(style, q_pe, k_pe, cis, cs, pos)
    assert torch.equal(q_out[:, :, :g.DN], q_nope[:, :, 0])
    _check_rot(style, q_out[:, :, g.DN:], rq[:, :, 0])
    _check_rot(style, k_cache[:M, pos, :, g.DN:], rk[:, :, 0].expand(M, g.H, g.DR))
    assert torch.equal(k_cache[:M, pos, :, :g.DN], k0[:M, pos, :, :g.DN])     # k_nope is MLA_KV's
    keep = torch.ones(M + 1, S, dtype=torch.bool, device=_dev())
    keep[:M, pos] = False
    assert torch.equal(k_cache[keep], k0[keep])


@pytest.mark.parametrize("pos,S_f", [(-1, 128), (64, 128), (50, 40)])
def test_out_of_range_position_writes_nothing(pos, S_f):
    g = NARROW
    gen = _gen(7)
    cis, cs = _tables(g, S_f)
    qa = torch.randn((2, g.N_QA), device=_dev(), generator=gen).half()
    qb = torch.randn((2, g.N_QB), device=_dev(), generator=gen).half()
    k_cache = torch.randn((2, 64, g.H, g.W), device=_dev(), generator=gen).half()
    k0 = k_cache.clone()
    q_out = torch.full((2, g.H, g.W), 7.0, dtype=torch.float16, device=_dev())
    p = torch.tensor([pos], dtype=torch.int32, device=_dev())
    for style, f in ((0, cis), (1, cs)):
        ext.mla_k_rope(qa, f, p, k_cache, g.H, g.DN, g.DR, g.C, g.CQ, style)
        ext.mla_q_rope(qb, f, p, 64, g.H, g.DN, g.DR, style, q_out=q_out)
    torch.cuda.synchronize()
    assert (q_out == 7.0).all() and torch.equal(k_cache, k0)


class Attn:
    """The q LoRA MLA chain's weights and buffers: q_a|kv_a, q_b, kv_b (random AWQ-packed), the three norms, caches,
    position."""

    def __init__(self, g, seed, S=256, B=1):
        gen = _gen(seed)
        self.g = g
        self.wqa, self.wqb, self.wkvb = _lin(g.HID, g.N_QA, gen), _lin(g.CQ, g.N_QB, gen), _lin(g.C, g.N_KV, gen)
        self.n1 = (1 + 0.1 * torch.randn(g.HID, device=_dev(), generator=gen)).half()
        self.nq = (1 + 0.1 * torch.randn(g.CQ, device=_dev(), generator=gen)).half()
        self.nkv = (1 + 0.1 * torch.randn(g.C, device=_dev(), generator=gen)).half()
        self.k_cache = torch.zeros((B, S, g.H, g.W), dtype=torch.float16, device=_dev())
        self.v_cache = torch.zeros((B, S, g.H, g.DV), dtype=torch.float16, device=_dev())
        self.pos = torch.tensor([5], dtype=torch.int32, device=_dev())

    def record(self, p, h, style, freqs):
        """[norm1(h), q_a|kv_a, mla_k_rope, norm(q_a), q_b, mla_q_rope, norm(c_kv), kv_b, mla_kv] into program p"""
        g, M = self.g, h.shape[0]
        xn = torch.empty((M, g.HID), dtype=torch.float16, device=_dev())
        qan = torch.empty((M, g.CQ), dtype=torch.float16, device=_dev())
        ckv = torch.empty((M, g.C), dtype=torch.float16, device=_dev())
        p.layernorm_forward_cuda(h, self.n1, xn, EPS)
        qa = p.gemm_forward_cuda(xn, *self.wqa, 8)
        p.mla_k_rope(qa, freqs, self.pos, self.k_cache, g.H, g.DN, g.DR, g.C, g.CQ, style)
        p.layernorm_forward_cuda(qa[:, :g.CQ], self.nq, qan, EPS)
        qb = p.gemm_forward_cuda(qan, *self.wqb, 8)
        q_out = p.mla_q_rope(qb, freqs, self.pos, self.k_cache.shape[1], g.H, g.DN, g.DR, style)
        p.layernorm_forward_cuda(qa[:, g.CQ:g.CQ + g.C], self.nkv, ckv, EPS)
        kv = p.gemm_forward_cuda(ckv, *self.wkvb, 8)
        p.mla_kv_cache(kv, self.pos, self.k_cache, self.v_cache, g.H, g.DN, g.DV)
        return dict(xn=xn, qa=qa, qan=qan, qb=qb, q_out=q_out, ckv=ckv, kv=kv)

    def standalone(self, b, style, freqs, k, v):
        """the stand-alone ops on the recorded rows b into caches k, v: (q_out, normed q_a, normed c_kv)"""
        g = self.g
        ext.mla_k_rope(b["qa"], freqs, self.pos, k, g.H, g.DN, g.DR, g.C, g.CQ, style)
        q2 = ext.mla_q_rope(b["qb"], freqs, self.pos, k.shape[1], g.H, g.DN, g.DR, style)
        ext.mla_kv_cache(b["kv"], self.pos, k, v, g.H, g.DN, g.DV)
        qan, ckv = torch.empty_like(b["qan"]), torch.empty_like(b["ckv"])
        ext.layernorm_forward_cuda(b["qa"][:, :g.CQ].contiguous(), self.nq, qan, EPS)
        ext.layernorm_forward_cuda(b["qa"][:, g.CQ:g.CQ + g.C].contiguous(), self.nkv, ckv, EPS)
        return q2, qan, ckv


@GEOS
@pytest.mark.parametrize("style", [0, 1])
def test_fused_chain_matches_standalone_ops_on_recorded_rows(g, style):
    cis, cs = _tables(g, 512)
    freqs = cis if style == 0 else cs
    a = Attn(g, 20 + style)
    h = torch.randn((1, g.HID), device=_dev(), generator=_gen(3)).half()
    p = DecodeProgram()
    b = a.record(p, h, style, freqs)
    p.build()
    assert p.fused and p.kernel_ops == 3 and p.launches_per_run == 1
    p.run()
    torch.cuda.synchronize()
    _no_abort("mla lora chain")
    pos = int(a.pos.item())
    k2, v2 = torch.zeros_like(a.k_cache), torch.zeros_like(a.v_cache)
    q2, qan, ckv = a.standalone(b, style, freqs, k2, v2)
    torch.cuda.synchronize()
    assert torch.equal(b["q_out"], q2)
    assert torch.equal(a.k_cache, k2) and torch.equal(a.v_cache, v2)
    assert torch.equal(b["qan"], qan) and torch.equal(b["ckv"], ckv)
    assert a.k_cache[0, pos].abs().sum() > 0 and a.v_cache[0, pos].abs().sum() > 0


def _deq(w):
    from oracle import awq_oracle as O

    q, s, z = (t.cpu().numpy() for t in w)
    return torch.from_numpy(O.dequantize_gemm(q, z, s, G).astype(np.float16)).to(_dev())


@GEOS
@pytest.mark.parametrize("version", [2, 3])
def test_states_against_transformers_attention(g, version):
    """query / key / value states of transformers' attention with q_lora_rank set (nn.Linear projections over the
    dequantised weights, both norms with their weights, fp16) against q_out and the cache row the fused chain writes:
    within 8 fp16 ulps of rms, the dense tests' bound; the rotated halves against transformers' own rotation of the
    program's recorded rows within the rotary bound."""
    if version == 2:
        from transformers import DeepseekV2Config as Cfg
        from transformers.models.deepseek_v2.modeling_deepseek_v2 import DeepseekV2Attention as Att
        from transformers.models.deepseek_v2.modeling_deepseek_v2 import DeepseekV2RotaryEmbedding as Rot
    else:
        from transformers import DeepseekV3Config as Cfg
        from transformers.models.deepseek_v3.modeling_deepseek_v3 import DeepseekV3Attention as Att
        from transformers.models.deepseek_v3.modeling_deepseek_v3 import DeepseekV3RotaryEmbedding as Rot
    from transformers import AttentionInterface

    cfg = Cfg(hidden_size=g.HID, num_attention_heads=g.H, num_key_value_heads=g.H, q_lora_rank=g.CQ,
              kv_lora_rank=g.C, qk_nope_head_dim=g.DN, qk_rope_head_dim=g.DR, v_head_dim=g.DV, rms_norm_eps=EPS,
              attention_bias=False, max_position_embeddings=4096, num_hidden_layers=1, vocab_size=128)
    AttentionInterface.register("mla_capture", _capture_attention)
    cfg._attn_implementation = "mla_capture"
    if version == 3:
        cfg.rope_interleave = True
    with torch.random.fork_rng(devices=[]):
        att = Att(cfg, layer_idx=0).to(_dev()).half().eval()
    rot = Rot(cfg, device=_dev())
    a = Attn(g, 40 + version)
    wqa = _deq(a.wqa)
    with torch.no_grad():
        att.q_a_proj.weight.copy_(wqa[:, :g.CQ].t())
        att.kv_a_proj_with_mqa.weight.copy_(wqa[:, g.CQ:].t())
        att.q_b_proj.weight.copy_(_deq(a.wqb).t())
        att.kv_b_proj.weight.copy_(_deq(a.wkvb).t())
        att.q_a_layernorm.weight.copy_(a.nq)
        att.kv_a_layernorm.weight.copy_(a.nkv)
    pos = 5
    a.pos.fill_(pos)
    pid = torch.arange(4096, device=_dev())[None]
    style = 0 if version == 2 else 1
    if style == 0:
        freqs = rot(torch.zeros(1, device=_dev(), dtype=torch.float32), pid)[0]        # complex64 [S, Dr/2]
        pe = freqs[pos:pos + 1][None]
    else:
        freqs = rot(torch.zeros(1, device=_dev(), dtype=torch.float32), pid)           # f32 (cos, sin) [1, S, Dr]
        freqs = (freqs[0][0], freqs[1][0])
        pe = tuple(t[pos:pos + 1][None].half() for t in freqs)
    h = torch.randn((1, g.HID), device=_dev(), generator=_gen(4)).half()
    p = DecodeProgram()
    b = a.record(p, h, style, freqs)
    p.build()
    assert p.fused
    p.run()
    torch.cuda.synchronize()
    _no_abort("mla lora vs transformers")
    cap = mla_test._CAPTURED = _Capture()
    with torch.no_grad():
        att(b["xn"].view(1, 1, g.HID), attention_mask=None, past_key_values=cap, position_embeddings=pe)
    for name, x, ref in (("query", b["q_out"][0], cap.q[0, :, 0]), ("key", a.k_cache[0, pos], cap.k[0, :, 0]),
                         ("value", a.v_cache[0, pos], cap.v[0, :, 0])):
        err, tol = _ulps_of_rms(x, ref, 8)
        assert err <= tol, f"{name}: {err:.3e} > {tol:.3e}"
    q_pe = b["qb"].view(1, 1, g.H, g.W).transpose(1, 2)[..., g.DN:]
    k_pe = b["qa"][:, g.CQ + g.C:].view(1, 1, 1, g.DR)
    rq, rk = _hf_rot(style, q_pe, k_pe, freqs if style == 0 else None, freqs if style == 1 else None, pos)
    _check_rot(style, b["q_out"][0, :, g.DN:], rq[0, :, 0])
    _check_rot(style, a.k_cache[0, pos, :, g.DN:], rk[0, 0, 0].expand(g.H, g.DR))


class Dense:
    """A dense DeepSeek layer's o_proj and MLP weights and its post-attention norm."""

    def __init__(self, g, seed):
        gen = _gen(seed)
        self.wo = _lin(g.H * g.DV, g.HID, gen)
        self.wgu = _lin(g.HID, 2 * g.INTER, gen)
        self.wd = _lin(g.INTER, g.HID, gen)
        self.n2 = (1 + 0.1 * torch.randn(g.HID, device=_dev(), generator=gen)).half()


def _segment(g, dense, a, style, freqs, attn, h, knob14):
    """[o + h, norm2, gate|up, silu, down + h, norm1', q_a|kv_a', k-rope', norm(q_a)', q_b', q-rope', norm(c_kv)',
    kv_b', mla_kv']"""
    hm, xn2, h2 = (torch.empty((1, g.HID), dtype=torch.float16, device=_dev()) for _ in range(3))
    act = torch.empty((1, g.INTER), dtype=torch.float16, device=_dev())
    p = DecodeProgram()
    o = p.gemm_forward_cuda(attn, *dense.wo, 8)
    p.add(o, h, out=hm)
    p.layernorm_forward_cuda(hm, dense.n2, xn2, EPS)
    gu = p.gemm_forward_cuda(xn2, *dense.wgu, 8)
    p.silu_and_mul(act, gu)
    d = p.gemm_forward_cuda(act, *dense.wd, 8)
    p.add(d, hm, out=h2)
    b = a.record(p, h2, style, freqs)
    ext.set_knob(14, 1 if knob14 else 0)
    try:
        p.build()
    finally:
        ext.set_knob(14, 0)
    return p, dict(b, h2=h2)


@pytest.mark.parametrize("g,style", [(V3, 1), (NARROW, 0)], ids=["v3", "narrow"])
def test_dense_segment_one_launch_and_graph_replay(g, style):
    cis, cs = _tables(g, 512)
    freqs = cis if style == 0 else cs
    dense = Dense(g, 11)
    gen = _gen(5)
    attn = torch.randn((1, g.H * g.DV), device=_dev(), generator=gen).half()
    h = torch.randn((1, g.HID), device=_dev(), generator=gen).half()
    af, ar = Attn(g, 30), Attn(g, 30)
    pf, bf = _segment(g, dense, af, style, freqs, attn, h, False)
    pr, br = _segment(g, dense, ar, style, freqs, attn, h, True)
    assert pf.fused and pf.launches_per_run == 1 and pf.kernel_ops == 6 and not pr.fused
    pf.run()
    pr.run()
    torch.cuda.synchronize()
    _no_abort("mla lora segment")
    pos = int(af.pos.item())
    for name, x, y in (("h2", bf["h2"], br["h2"]), ("q_out", bf["q_out"], br["q_out"]),
                       ("k", af.k_cache[0, pos], ar.k_cache[0, pos]), ("v", af.v_cache[0, pos], ar.v_cache[0, pos])):
        err, tol = _ulps_of_rms(x, y, 8)
        assert err <= tol + 1e-3, f"{name}: {err:.3e} > {tol:.3e}"
    # a CUDA graph of the fused segment, replayed at a moving position
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        pf.run()
        torch.cuda.synchronize()
        with torch.cuda.graph(graph, stream=s):
            pf.run()
    torch.cuda.current_stream().wait_stream(s)
    for step in range(3):
        p = 6 + step
        af.pos.fill_(p)
        h.copy_(torch.randn((1, g.HID), device=_dev(), generator=gen).half())
        graph.replay()
        torch.cuda.synchronize()
        k2, v2 = torch.zeros_like(af.k_cache), torch.zeros_like(af.v_cache)
        q2, qan, ckv = af.standalone(bf, style, freqs, k2, v2)
        torch.cuda.synchronize()
        assert torch.equal(q2, bf["q_out"]) and torch.equal(qan, bf["qan"]) and torch.equal(ckv, bf["ckv"]), step
        assert torch.equal(af.k_cache[0, p], k2[0, p]) and torch.equal(af.v_cache[0, p], v2[0, p]), step
        assert af.k_cache[0, p].abs().sum() > 0, step
    _no_abort("mla lora segment graph")


@pytest.mark.parametrize("style", [0, 1])
def test_two_token_chain_replays_per_op(style):
    """The chain recorded at M = 2 through DecodeProgram(max_tokens=2): the norms read slices of two rows (row-strided
    sources) and the MLA ops are outside the fused kernels at M > 1, so run() replays per op.  Every buffer matches the
    stand-alone ops on the recorded rows."""
    g, M = NARROW, 2
    cis, cs = _tables(g, 512)
    freqs = cis if style == 0 else cs
    a = Attn(g, 50 + style, B=M)
    h = torch.randn((M, g.HID), device=_dev(), generator=_gen(6)).half()
    p = DecodeProgram(max_tokens=M)
    b = a.record(p, h, style, freqs)
    p.build()
    assert not p.fused and p.launches_per_run == 9
    p.run()
    torch.cuda.synchronize()
    k2, v2 = torch.zeros_like(a.k_cache), torch.zeros_like(a.v_cache)
    q2, qan, ckv = a.standalone(b, style, freqs, k2, v2)
    torch.cuda.synchronize()
    assert torch.equal(b["q_out"], q2) and torch.equal(b["qan"], qan) and torch.equal(b["ckv"], ckv)
    assert torch.equal(a.k_cache, k2) and torch.equal(a.v_cache, v2)
    pos = int(a.pos.item())
    assert a.k_cache[1, pos].abs().sum() > 0


def test_recorder_refuses_caches_and_q_out_smaller_than_the_rows():
    from autoawq_b200._cabi import B200AwqError

    g = NARROW
    cis, _ = _tables(g, 64)
    pos = torch.zeros(1, dtype=torch.int32, device=_dev())
    qa = torch.zeros((2, g.N_QA), dtype=torch.float16, device=_dev())
    qb = torch.zeros((2, g.N_QB), dtype=torch.float16, device=_dev())
    k1 = torch.zeros((1, 16, g.H, g.W), dtype=torch.float16, device=_dev())
    p = DecodeProgram(max_tokens=2)
    with pytest.raises(B200AwqError, match="k_cache"):
        p.mla_k_rope(qa, cis, pos, k1, g.H, g.DN, g.DR, g.C, g.CQ, 0)
    with pytest.raises(B200AwqError, match="q_out"):
        p.mla_q_rope(qb, cis, pos, 16, g.H, g.DN, g.DR, 0,
                     q_out=torch.empty((1, g.H, g.W), dtype=torch.float16, device=_dev()))


def test_fuse_mla_lora_input_matches_the_two_projections():
    """The fused q_a_proj | kv_a_proj_with_mqa linear from packing.fuse_mla_lora_input against the two WQLinear_GEMM
    modules run on their own: within 2 fp16 ulps of rms."""
    import types

    from autoawq_b200 import packing
    from autoawq_b200.linear import WQLinear_GEMM

    g = V3
    gen = _gen(12)

    def mod(N):
        m = WQLinear_GEMM(4, G, g.HID, N, False, _dev())
        q, s, z = _lin(g.HID, N, gen)
        m.qweight.copy_(q)
        m.scales.copy_(s)
        m.qzeros.copy_(z)
        return m

    attn = types.SimpleNamespace(q_lora_rank=g.CQ, q_a_proj=mod(g.CQ), kv_a_proj_with_mqa=mod(g.C + g.DR))
    q, s, z, bias = packing.fuse_mla_lora_input(attn)
    x = torch.randn((1, g.HID), device=_dev(), generator=gen).half()
    with torch.no_grad():
        ref = torch.cat((attn.q_a_proj(x), attn.kv_a_proj_with_mqa(x)), dim=-1)
    y = ext.linear_forward("gemm", x, q, s, z, G, bias)
    torch.cuda.synchronize()
    err, tol = _ulps_of_rms(y, ref, 2)
    assert err <= tol, f"{err:.3e} > {tol:.3e}"
