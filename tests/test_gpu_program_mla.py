"""MLA glue in decode programs (DecodeProgram.mla_rope / mla_kv_cache, B200AWQ_OP_MLA_ROPE / _MLA_KV) and the stand-alone
ops (ext.mla_rope / ext.mla_kv_cache), at DeepSeek-V2-Lite / Moonlight attention shapes (H 16, Dn 128, Dr 64, Dv 128,
C 512, hidden 2048):
  * b200awq_stream_pack in mode 3 against the stream-format oracle (mode 0 of the column-reordered linear);
  * the stand-alone ops against transformers' own apply_rotary_emb (V2, within one fp16 ulp) and
    apply_rotary_pos_emb_interleave (V3, bit-exact), q_nope, k_nope and v bit-exact, at M = 1, 2, 4, with every other
    cache row untouched and nothing written for a position outside the cache or the table;
  * the fused [norm1, q|kv_a, mla_rope, rmsnorm(c_kv), kv_b, mla_kv] bit-identical to the stand-alone ops on the
    program's own recorded rows;
  * the whole V2-Lite segment in both routing styles as one launch, within the dense tests' bounds of its knob-14
    replay, and in a CUDA graph replayed at a moving position;
  * query / key / value states against transformers' DeepseekV2Attention / DeepseekV3Attention over the dequantised
    weights, captured from the cache's update call."""
import numpy as np
import pytest
import torch

from autoawq_b200 import ext
from autoawq_b200.program import DecodeProgram
from oracle import stream_format as SF
from test_gpu_program import _no_abort
from test_gpu_program_deepseek_moe import DsMoe, _record, _ulps_of_rms
from test_program_mla_cpu import mode3_columns, permute_linear

pytestmark = pytest.mark.gpu

H, DN, DR, DV, C, HID, G = 16, 128, 64, 128, 512, 2048, 128
W = DN + DR
N_QKVA, N_KV = H * W + C + DR, H * (DN + DV)
EPS = 1e-6


def _dev():
    return torch.device("cuda:0")


def _gen(seed):
    return torch.Generator(device=_dev()).manual_seed(seed)


def _lin(K, N, gen):
    return (torch.randint(-2**31, 2**31 - 1, (K, N // 8), dtype=torch.int32, device=_dev(), generator=gen),
            ((torch.rand((K // G, N), device=_dev(), generator=gen) * 0.5 + 0.75) / (6.1 * K**0.5)).half(),
            torch.randint(-2**31, 2**31 - 1, (K // G, N // 8), dtype=torch.int32, device=_dev(), generator=gen))


def _tables(S_f, theta=10000.0, scaling=1.2247):
    """(freqs_cis complex64 [S_f, Dr/2], (cos, sin) f32 [S_f, Dr]) as DeepseekV2RotaryEmbedding /
    DeepseekV3RotaryEmbedding build them, attention_scaling (a yarn mscale) applied."""
    inv = 1.0 / (theta ** (torch.arange(0, DR, 2, dtype=torch.int64, device=_dev()).float() / DR))
    f = torch.outer(torch.arange(S_f, device=_dev()).float(), inv)
    cis = torch.polar(torch.ones_like(f), f) * scaling
    emb = torch.cat((f, f), dim=-1)
    return cis, (emb.cos() * scaling, emb.sin() * scaling)


def _hf_rot(style, q_pe, k_pe, cis, cs, pos):
    """transformers' rotation of q_pe [M, H, 1, Dr] and k_pe [M, 1, 1, Dr] (fp16) at position pos."""
    if style == 0:
        from transformers.models.deepseek_v2.modeling_deepseek_v2 import apply_rotary_emb
        return apply_rotary_emb(q_pe, k_pe, cis[pos:pos + 1][None])
    from transformers.models.deepseek_v3.modeling_deepseek_v3 import apply_rotary_pos_emb_interleave
    cos, sin = (t[pos:pos + 1][None].half() for t in cs)
    return apply_rotary_pos_emb_interleave(q_pe, k_pe, cos, sin)


def _ulp_diff(a, b):
    """|a - b| in fp16 ulps of b, elementwise"""
    a, b = a.float().cpu().numpy(), b.float().cpu().numpy()
    return np.abs(a - b) / np.spacing(np.abs(b).astype(np.float16)).astype(np.float32)


def _caches(B, S, gen, v_head=DV):
    k = torch.randn((B, S, H, W), device=_dev(), generator=gen).half()
    v = torch.randn((B, S, H, v_head), device=_dev(), generator=gen).half()
    return k, v


def test_stream_pack_mode3_against_oracle():
    K, N = 256, N_QKVA
    qw, sc, qz = _lin(K, N, _gen(1))
    got = ext.stream_pack(qw, sc, qz, mode=3).cpu().numpy()
    q2, z2, s2 = permute_linear(qw.cpu().numpy(), qz.cpu().numpy(), sc.cpu().numpy(), mode3_columns(N).reshape(-1))
    assert np.array_equal(got, SF.pack_stream(q2, z2, s2, G, 0))


@pytest.mark.parametrize("style", [0, 1])
@pytest.mark.parametrize("M", [1, 2, 4])
def test_standalone_ops_against_transformers(style, M):
    gen = _gen(10 * M + style)
    S, pos = 64, 37
    cis, cs = _tables(128)
    freqs = cis if style == 0 else cs
    qkva = (torch.randn((M, N_QKVA), device=_dev(), generator=gen) * 2).half()
    kv = torch.randn((M, N_KV), device=_dev(), generator=gen).half()
    k_cache, v_cache = _caches(M + 1, S, gen)
    k0, v0 = k_cache.clone(), v_cache.clone()
    p = torch.tensor([pos], dtype=torch.int32, device=_dev())
    q_out = ext.mla_rope(qkva, freqs, p, k_cache, H, DN, DR, C, style)
    ext.mla_kv_cache(kv, p, k_cache, v_cache, H, DN, DV)
    torch.cuda.synchronize()
    q = qkva[:, :H * W].view(M, 1, H, W).transpose(1, 2)
    q_nope, q_pe = torch.split(q, [DN, DR], dim=-1)
    k_pe = qkva[:, H * W + C:].view(M, 1, 1, DR)
    rq, rk = _hf_rot(style, q_pe, k_pe, cis, cs, pos)
    assert torch.equal(q_out[:, :, :DN], q_nope[:, :, 0])
    dq, dk = _ulp_diff(q_out[:, :, DN:], rq[:, :, 0]), _ulp_diff(k_cache[:M, pos, :, DN:], rk[:, :, 0].expand(M, H, DR))
    if style == 1:
        assert dq.max() == 0 and dk.max() == 0, (dq.max(), dk.max())
    else:
        assert dq.max() <= 1 and dk.max() <= 1, (dq.max(), dk.max())
    kvv = kv.view(M, H, DN + DV)
    assert torch.equal(k_cache[:M, pos, :, :DN], kvv[..., :DN]) and torch.equal(v_cache[:M, pos], kvv[..., DN:])
    keep = torch.ones(M + 1, S, dtype=torch.bool, device=_dev())
    keep[:M, pos] = False
    assert torch.equal(k_cache[keep], k0[keep]) and torch.equal(v_cache[keep], v0[keep])


@pytest.mark.parametrize("pos,S_f", [(-1, 128), (64, 128), (50, 40)])
def test_out_of_range_position_writes_nothing(pos, S_f):
    gen = _gen(7)
    cis, cs = _tables(S_f)
    qkva = torch.randn((2, N_QKVA), device=_dev(), generator=gen).half()
    kv = torch.randn((2, N_KV), device=_dev(), generator=gen).half()
    k_cache, v_cache = _caches(2, 64, gen)
    k0, v0 = k_cache.clone(), v_cache.clone()
    q_out = torch.full((2, H, W), 7.0, dtype=torch.float16, device=_dev())
    p = torch.tensor([pos], dtype=torch.int32, device=_dev())
    for style, f in ((0, cis), (1, cs)):
        ext.mla_rope(qkva, f, p, k_cache, H, DN, DR, C, style, q_out=q_out)
    ext.mla_kv_cache(kv, p, k_cache, v_cache, H, DN, DV)
    torch.cuda.synchronize()
    assert (q_out == 7.0).all() and torch.equal(k_cache[..., DN:], k0[..., DN:])
    if pos < 0 or pos >= 64:
        assert torch.equal(k_cache, k0) and torch.equal(v_cache, v0)
    else:    # MLA_KV reads no frequency table: a position inside the cache is written, and only that row
        kvv = kv.view(2, H, DN + DV)
        assert torch.equal(k_cache[:, pos, :, :DN], kvv[..., :DN]) and torch.equal(v_cache[:, pos], kvv[..., DN:])
        keep = torch.ones(2, 64, dtype=torch.bool, device=_dev())
        keep[:, pos] = False
        assert torch.equal(k_cache[keep], k0[keep]) and torch.equal(v_cache[keep], v0[keep])


class Attn:
    """The MLA chain's weights and buffers: q|kv_a, kv_b (random AWQ-packed), the two norms, caches, position."""

    def __init__(self, seed, S=256, v_head=DV):
        gen = _gen(seed)
        self.wqkva, self.wkvb = _lin(HID, N_QKVA, gen), _lin(C, N_KV, gen)
        self.n1 = (1 + 0.1 * torch.randn(HID, device=_dev(), generator=gen)).half()
        self.nkv = (1 + 0.1 * torch.randn(C, device=_dev(), generator=gen)).half()
        self.k_cache = torch.zeros((1, S, H, W), dtype=torch.float16, device=_dev())
        self.v_cache = torch.zeros((1, S, H, v_head), dtype=torch.float16, device=_dev())
        self.pos = torch.tensor([5], dtype=torch.int32, device=_dev())

    def record(self, p, h, style, freqs):
        """[norm1(h), q|kv_a, mla_rope, rmsnorm(c_kv), kv_b, mla_kv] into program p; returns the recorded buffers."""
        xn = torch.empty((1, HID), dtype=torch.float16, device=_dev())
        ckv = torch.empty((1, C), dtype=torch.float16, device=_dev())
        p.layernorm_forward_cuda(h, self.n1, xn, EPS)
        qkva = p.gemm_forward_cuda(xn, *self.wqkva, 8)
        q_out = p.mla_rope(qkva, freqs, self.pos, self.k_cache, H, DN, DR, C, style)
        p.layernorm_forward_cuda(qkva[:, H * W:H * W + C], self.nkv, ckv, EPS)
        kv = p.gemm_forward_cuda(ckv, *self.wkvb, 8)
        p.mla_kv_cache(kv, self.pos, self.k_cache, self.v_cache, H, DN, DV)
        return dict(xn=xn, qkva=qkva, q_out=q_out, ckv=ckv, kv=kv)


@pytest.mark.parametrize("style", [0, 1])
def test_fused_chain_matches_standalone_ops_on_recorded_rows(style):
    cis, cs = _tables(512)
    freqs = cis if style == 0 else cs
    a = Attn(20 + style, v_head=W)            # v padded to Dn + Dr (FlashAttention-2's layout)
    h = torch.randn((1, HID), device=_dev(), generator=_gen(3)).half()
    p = DecodeProgram()
    b = a.record(p, h, style, freqs)
    p.build()
    assert p.fused and p.kernel_ops == 2 and p.launches_per_run == 1
    p.run()
    torch.cuda.synchronize()
    _no_abort("mla chain")
    pos = int(a.pos.item())
    k2, v2 = torch.zeros_like(a.k_cache), torch.zeros_like(a.v_cache)
    q2 = ext.mla_rope(b["qkva"], freqs, a.pos, k2, H, DN, DR, C, style)
    ext.mla_kv_cache(b["kv"], a.pos, k2, v2, H, DN, DV)
    ckv = torch.empty_like(b["ckv"])
    ext.layernorm_forward_cuda(b["qkva"][:, H * W:H * W + C].contiguous(), a.nkv, ckv, EPS)
    torch.cuda.synchronize()
    assert torch.equal(b["q_out"], q2)
    assert torch.equal(a.k_cache, k2) and torch.equal(a.v_cache, v2)
    assert torch.equal(b["ckv"], ckv)
    assert a.k_cache[0, pos].abs().sum() > 0 and (a.v_cache[0, pos, :, DV:] == 0).all()


def _segment(moe, a, scoring, style, freqs, attn, h, knob14):
    """[o + h, norm2, deepseek_moe + h, norm1', q|kv_a', mla_rope', rmsnorm(c_kv)', kv_b', mla_kv'] at V2-Lite shapes"""
    wo = _lin(H * DV, HID, _gen(9))
    n2 = (1 + 0.1 * torch.randn(HID, device=_dev(), generator=_gen(8))).half()
    hm, xn2, h2 = (torch.empty((1, HID), dtype=torch.float16, device=_dev()) for _ in range(3))
    p = DecodeProgram()
    o = p.gemm_forward_cuda(attn, *wo, 8)
    p.add(o, h, out=hm)
    p.layernorm_forward_cuda(hm, n2, xn2, EPS)
    mo = _record(p, moe, xn2, scoring, 1, 1, scoring == "sigmoid", 1.0 if scoring == "softmax" else 2.446)
    p.add(mo, hm, out=h2)
    b = a.record(p, h2, style, freqs)
    ext.set_knob(14, 1 if knob14 else 0)
    try:
        p.build()
    finally:
        ext.set_knob(14, 0)
    return p, dict(b, h2=h2)


@pytest.mark.parametrize("scoring,style", [("softmax", 0), ("sigmoid", 1)])
def test_v2_lite_segment_one_launch_and_graph_replay(scoring, style):
    cis, cs = _tables(512)
    freqs = cis if style == 0 else cs
    moe = DsMoe(64, HID, 1408, G, 6, 2, seed=11)
    gen = _gen(5)
    attn = torch.randn((1, H * DV), device=_dev(), generator=gen).half()
    h = torch.randn((1, HID), device=_dev(), generator=gen).half()
    af, ar = Attn(30), Attn(30)
    pf, bf = _segment(moe, af, scoring, style, freqs, attn, h, False)
    pr, br = _segment(moe, ar, scoring, style, freqs, attn, h, True)
    assert pf.fused and pf.launches_per_run == 1 and pf.kernel_ops == 5 and not pr.fused
    pf.run()
    pr.run()
    torch.cuda.synchronize()
    _no_abort("mla segment")
    pos = int(af.pos.item())
    same_route = torch.equal(pf.moe_buffers(0)["topk_ids"].sort().values, pr.moe_buffers(0)["topk_ids"].sort().values)
    assert same_route
    for name, x, y in (("q_out", bf["q_out"], br["q_out"]), ("k", af.k_cache[0, pos], ar.k_cache[0, pos]),
                       ("v", af.v_cache[0, pos], ar.v_cache[0, pos]), ("kv", bf["kv"], br["kv"])):
        err, tol = _ulps_of_rms(x, y, 8)
        assert err <= tol + 1e-3, f"{name}: {err:.3e} > {tol:.3e}"
    # a CUDA graph of the fused segment, replayed at a moving position
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        pf.run()
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=s):
            pf.run()
    torch.cuda.current_stream().wait_stream(s)
    for step in range(3):
        p = 6 + step
        af.pos.fill_(p)
        h.copy_(torch.randn((1, HID), device=_dev(), generator=gen).half())
        g.replay()
        torch.cuda.synchronize()
        k2, v2 = torch.zeros_like(af.k_cache), torch.zeros_like(af.v_cache)
        q2 = ext.mla_rope(bf["qkva"], freqs, af.pos, k2, H, DN, DR, C, style)
        ext.mla_kv_cache(bf["kv"], af.pos, k2, v2, H, DN, DV)
        torch.cuda.synchronize()
        assert torch.equal(q2, bf["q_out"]), step
        assert torch.equal(af.k_cache[0, p], k2[0, p]) and torch.equal(af.v_cache[0, p], v2[0, p]), step
        assert af.k_cache[0, p].abs().sum() > 0, step
    _no_abort("mla segment graph")


class _Capture:
    """A cache object whose update() records the key / value states the attention writes (transformers' Cache.update
    signature); the attention function registered below records the query states next to them and returns zeros."""

    def update(self, key_states, value_states, layer_idx, *args, **kwargs):
        self.k, self.v = key_states, value_states
        return key_states, value_states


def _capture_attention(module, query, key, value, attention_mask, **kwargs):
    _CAPTURED.q = query
    b, h, s, _ = query.shape
    return torch.zeros((b, s, h, value.shape[-1]), dtype=query.dtype, device=query.device), None


_CAPTURED = None


def _deq(w):
    from oracle import awq_oracle as O

    q, s, z = (t.cpu().numpy() for t in w)
    return torch.from_numpy(O.dequantize_gemm(q, z, s, G).astype(np.float16)).to(_dev())


@pytest.mark.parametrize("version", [2, 3])
def test_states_against_transformers_attention(version):
    """query / key / value states of transformers' attention (the projections nn.Linear over the dequantised weights,
    kv_a_layernorm with the norm's weight, fp16) against q_out and the cache row the fused chain writes.  Bound: the
    linears' fp64 bound (fp32 accumulation of different orders, a few fp16 ulps of the row's rms), then one rotary ulp."""
    if version == 2:
        from transformers import DeepseekV2Config as Cfg
        from transformers.models.deepseek_v2.modeling_deepseek_v2 import DeepseekV2Attention as Att
        from transformers.models.deepseek_v2.modeling_deepseek_v2 import DeepseekV2RotaryEmbedding as Rot
    else:
        from transformers import DeepseekV3Config as Cfg
        from transformers.models.deepseek_v3.modeling_deepseek_v3 import DeepseekV3Attention as Att
        from transformers.models.deepseek_v3.modeling_deepseek_v3 import DeepseekV3RotaryEmbedding as Rot
    cfg = Cfg(hidden_size=HID, num_attention_heads=H, num_key_value_heads=H, q_lora_rank=None, kv_lora_rank=C,
              qk_nope_head_dim=DN, qk_rope_head_dim=DR, v_head_dim=DV, rms_norm_eps=EPS, attention_bias=False,
              max_position_embeddings=4096, num_hidden_layers=1, vocab_size=128)
    from transformers import AttentionInterface

    AttentionInterface.register("mla_capture", _capture_attention)
    cfg._attn_implementation = "mla_capture"
    if version == 3:
        cfg.rope_interleave = True
    with torch.random.fork_rng(devices=[]):     # (the module's random init leaves the global CPU generator as it was)
        att = Att(cfg, layer_idx=0).to(_dev()).half().eval()
    rot = Rot(cfg, device=_dev())
    a = Attn(40 + version)
    wq = _deq(a.wqkva)
    with torch.no_grad():
        att.q_proj.weight.copy_(wq[:, :H * W].t())
        att.kv_a_proj_with_mqa.weight.copy_(wq[:, H * W:].t())
        att.kv_b_proj.weight.copy_(_deq(a.wkvb).t())
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
    h = torch.randn((1, HID), device=_dev(), generator=_gen(4)).half()
    p = DecodeProgram()
    b = a.record(p, h, style, freqs)
    p.build()
    assert p.fused
    p.run()
    torch.cuda.synchronize()
    _no_abort("mla vs transformers")
    global _CAPTURED
    cap = _CAPTURED = _Capture()
    with torch.no_grad():
        att(b["xn"].view(1, 1, HID), attention_mask=None, past_key_values=cap, position_embeddings=pe)
    for name, x, ref in (("query", b["q_out"][0], cap.q[0, :, 0]), ("key", a.k_cache[0, pos], cap.k[0, :, 0]),
                         ("value", a.v_cache[0, pos], cap.v[0, :, 0])):
        err, tol = _ulps_of_rms(x, ref, 8)
        assert err <= tol, f"{name}: {err:.3e} > {tol:.3e}"
    # the rotated halves against transformers' own rotation of the program's recorded q_pe / k_pe: the rotary bound
    q_pe = b["qkva"][:, :H * W].view(1, 1, H, W).transpose(1, 2)[..., DN:]
    k_pe = b["qkva"][:, H * W + C:].view(1, 1, 1, DR)
    rq, rk = _hf_rot(style, q_pe, k_pe, freqs if style == 0 else None, freqs if style == 1 else None, pos)
    assert _ulp_diff(b["q_out"][0, :, DN:], rq[0, :, 0]).max() <= (1 if style == 0 else 0)
    assert _ulp_diff(a.k_cache[0, pos, :, DN:], rk[0, 0, 0].expand(H, DR)).max() <= (1 if style == 0 else 0)


@pytest.mark.parametrize("style", [0, 1])
def test_two_token_chain_replays_per_op(style):
    """The chain recorded at M = 2 through DecodeProgram(max_tokens=2): kv_a_layernorm reads the c_kv slice of two rows
    (a row-strided source), the MLA ops are outside the fused kernels (M > 1), so build() keeps the op list and run()
    replays it per op.  Every token row matches the stand-alone ops on the recorded rows, and the M = 1 fused program
    on that row alone."""
    M = 2
    cis, cs = _tables(512)
    freqs = cis if style == 0 else cs
    a = Attn(50 + style)
    a.k_cache = torch.zeros((M, 256, H, W), dtype=torch.float16, device=_dev())
    a.v_cache = torch.zeros((M, 256, H, DV), dtype=torch.float16, device=_dev())
    h = torch.randn((M, HID), device=_dev(), generator=_gen(6)).half()
    p = DecodeProgram(max_tokens=M)
    xn = torch.empty((M, HID), dtype=torch.float16, device=_dev())
    ckv = torch.empty((M, C), dtype=torch.float16, device=_dev())
    p.layernorm_forward_cuda(h, a.n1, xn, EPS)
    qkva = p.gemm_forward_cuda(xn, *a.wqkva, 8)
    q_out = p.mla_rope(qkva, freqs, a.pos, a.k_cache, H, DN, DR, C, style)
    p.layernorm_forward_cuda(qkva[:, H * W:H * W + C], a.nkv, ckv, EPS)
    kv = p.gemm_forward_cuda(ckv, *a.wkvb, 8)
    p.mla_kv_cache(kv, a.pos, a.k_cache, a.v_cache, H, DN, DV)
    p.build()
    assert not p.fused
    p.run()
    torch.cuda.synchronize()
    pos = int(a.pos.item())
    ckv2 = torch.empty_like(ckv)
    ext.layernorm_forward_cuda(qkva[:, H * W:H * W + C].contiguous(), a.nkv, ckv2, EPS)
    k2, v2 = torch.zeros_like(a.k_cache), torch.zeros_like(a.v_cache)
    q2 = ext.mla_rope(qkva, freqs, a.pos, k2, H, DN, DR, C, style)
    ext.mla_kv_cache(kv, a.pos, k2, v2, H, DN, DV)
    torch.cuda.synchronize()
    assert torch.equal(ckv, ckv2) and torch.equal(q_out, q2)
    assert torch.equal(a.k_cache, k2) and torch.equal(a.v_cache, v2)
    for m in range(M):
        b1 = Attn(50 + style)
        p1 = DecodeProgram()
        r1 = b1.record(p1, h[m:m + 1].clone(), style, freqs)
        p1.build()
        assert p1.fused
        p1.run()
        torch.cuda.synchronize()
        for name, x, y in (("q_out", q_out[m], r1["q_out"][0]), ("k", a.k_cache[m, pos], b1.k_cache[0, pos]),
                           ("v", a.v_cache[m, pos], b1.v_cache[0, pos])):
            err, tol = _ulps_of_rms(x, y, 8)
            assert err <= tol + 1e-3, f"row {m} {name}: {err:.3e} > {tol:.3e}"


def test_recorder_refuses_caches_and_q_out_smaller_than_the_rows():
    from autoawq_b200._cabi import B200AwqError

    cis, _ = _tables(64)
    pos = torch.zeros(1, dtype=torch.int32, device=_dev())
    qkva = torch.zeros((2, N_QKVA), dtype=torch.float16, device=_dev())
    kv = torch.zeros((2, N_KV), dtype=torch.float16, device=_dev())
    k1 = torch.zeros((1, 16, H, W), dtype=torch.float16, device=_dev())
    k2 = torch.zeros((2, 16, H, W), dtype=torch.float16, device=_dev())
    v1 = torch.zeros((1, 16, H, DV), dtype=torch.float16, device=_dev())
    p = DecodeProgram(max_tokens=2)
    with pytest.raises(B200AwqError, match="k_cache"):
        p.mla_rope(qkva, cis, pos, k1, H, DN, DR, C, 0)
    with pytest.raises(B200AwqError, match="q_out"):
        p.mla_rope(qkva, cis, pos, k2, H, DN, DR, C, 0, q_out=torch.empty((1, H, W), dtype=torch.float16, device=_dev()))
    with pytest.raises(B200AwqError, match="v_cache"):
        p.mla_kv_cache(kv, pos, k2, v1, H, DN, DV)


def test_fuse_mla_input_matches_the_two_projections():
    """The fused q_proj | kv_a_proj_with_mqa linear from packing.fuse_mla_input against the two WQLinear_GEMM modules
    run on their own: within 2 fp16 ulps of rms (the GEMV may cut the K sums differently for another N)."""
    import types

    from autoawq_b200 import packing
    from autoawq_b200.linear import WQLinear_GEMM

    gen = _gen(12)

    def mod(N):
        m = WQLinear_GEMM(4, G, HID, N, False, _dev())
        q, s, z = _lin(HID, N, gen)
        m.qweight.copy_(q)
        m.scales.copy_(s)
        m.qzeros.copy_(z)
        return m

    attn = types.SimpleNamespace(q_lora_rank=None, q_proj=mod(H * W), kv_a_proj_with_mqa=mod(C + DR))
    q, s, z, bias = packing.fuse_mla_input(attn)
    x = torch.randn((1, HID), device=_dev(), generator=gen).half()
    with torch.no_grad():
        ref = torch.cat((attn.q_proj(x), attn.kv_a_proj_with_mqa(x)), dim=-1)
    y = ext.linear_forward("gemm", x, q, s, z, G, bias)
    torch.cuda.synchronize()
    err, tol = _ulps_of_rms(y, ref, 2)
    assert err <= tol, f"{err:.3e} > {tol:.3e}"
