"""Depth-scaled residual adds in decode programs (DecodeProgram.scaled_add, B200AWQ_OP_SCALED_ADD): MiniCPM / MiniCPM3's
h = residual + h * scale_depth / sqrt(num_hidden_layers) and Granite's h = residual + h * residual_multiplier, folded
into the finish of the linear recorded just before, so a whole segment from one attention call to the next is one
launch.  The geometries are test shapes after the public configs (Granite-3.1-8B / 2B, MiniCPM-2B, MiniCPM3-4B):
  * one launch per segment at M = 1, with the kernel ops of the same segment with plain adds;
  * every scaled-add output bit-exact against torch's `residual + y * a` on the program's own raw y, including
    overflow to inf near +-65504, fp16 subnormal results, and an a whose fp16 rounding would change the product;
  * q, the cache rows and the MLA outputs bit-identical to the stand-alone ops on the program's own rows; every other
    buffer within tolerance of the per-op replay;
  * batched Granite-2B segments (M = 2, 4), each row bit-identical to an M = 1 program on that row;
  * a CUDA graph replay that follows pos, a = 1.0 against add, and per-op replay after a MoE block.
The abort record is checked after every run."""
import math

import pytest
import torch

from autoawq_b200 import ext
from autoawq_b200.program import DecodeProgram
from test_gpu_program import EPS, _no_abort
from test_gpu_program_deepseek_moe import _ulps_of_rms
from test_gpu_program_mla_lora import Attn, Dense, Geo, _tables
from test_gpu_program_moe import Moe
from test_gpu_program_rope import Layer, _caches

pytestmark = pytest.mark.gpu

F16 = torch.float16
S = 256
# hidden, intermediate, q heads, kv heads, head dim
GRANITE_8B = (4096, 12800, 32, 8, 128)
GRANITE_2B = (2048, 8192, 32, 8, 64)
MINICPM_2B = (2304, 5760, 36, 36, 64)
MINICPM3_4B = Geo(40, 64, 32, 64, 256, 768, 2560, 6400)


def _dev():
    return torch.device("cuda:0")


def _gen(seed):
    return torch.Generator(device=_dev()).manual_seed(seed)


def _bits(t):
    return t.contiguous().view(torch.int16)


def _torch_scaled(r, y, a):
    return r + y * a


def _assert_scaled_exact(out, r, y, a, what):
    ref = _torch_scaled(r, y, a)
    assert torch.equal(_bits(out), _bits(ref)), f"{what}: not torch's residual + y * a"


def _layer(geo, seed):
    hid, inter, H, KV, D = geo
    return Layer(hid, inter, H, KV, D, S, seed)


def _record(api, L, attn, h_in, pos, kc, vc, a):
    """[o, scaled_add, norm2, gate|up, silu, down, scaled_add, norm1', qkv', rope'] against `api`"""
    M = attn.shape[0]
    o = api.gemm_forward_cuda(attn, *L.w["o"], 8)
    h = api.scaled_add(h_in, o, a)
    xn2 = torch.empty((M, L.hidden), dtype=F16, device=_dev())
    api.layernorm_forward_cuda(h, L.n2, xn2, EPS)
    gu = api.gemm_forward_cuda(xn2, *L.w["gu"], 8)
    act = torch.empty((M, L.inter), dtype=F16, device=_dev())
    api.silu_and_mul(act, gu)
    dn = api.gemm_forward_cuda(act, *L.w["down"], 8)
    out = api.scaled_add(h, dn, a)
    xn = torch.empty((M, L.hidden), dtype=F16, device=_dev())
    api.layernorm_forward_cuda(out, L.n1, xn, EPS)
    qkv = api.gemm_forward_cuda(xn, *L.w["qkv"], 8)
    q = api.rope_kv_cache(qkv, L.freqs, pos, kc, vc, L.H, L.KV)
    return dict(attn=attn, h_in=h_in, o=o, h=h, xn2=xn2, gu=gu, act=act, dn=dn, out=out, xn=xn, qkv=qkv, q=q, k=kc,
                v=vc)


def _build(L, attn, h_in, pos, a, max_tokens=1, no_fuse=False, cache_seed=5):
    prev = ext.get_knob(14)
    ext.set_knob(14, 1 if no_fuse else 0)
    try:
        kc, vc = _caches(attn.shape[0], S, L.KV, L.D, cache_seed)
        prog = DecodeProgram(max_tokens=max_tokens)
        bufs = _record(prog, L, attn, h_in, pos, kc, vc, a)
        prog.build()
    finally:
        ext.set_knob(14, prev)
    return prog, bufs


def _check_exact(f, a, tag):
    """the two scaled adds bit-exact against torch on the program's raw outputs"""
    _assert_scaled_exact(f["h"], f["h_in"], f["o"], a, f"{tag} h")
    _assert_scaled_exact(f["out"], f["h"], f["dn"], a, f"{tag} out")


def _check_rope(L, f, pos, k0, v0, tag):
    """q and the cache rows bit-identical to the stand-alone op on the program's qkv, from the caches before the run"""
    rk, rv = k0.clone(), v0.clone()
    rq = ext.rope_kv_cache(f["qkv"], L.freqs, pos, rk, rv, L.H, L.KV)
    torch.cuda.synchronize()
    assert torch.equal(f["q"], rq) and torch.equal(f["k"], rk) and torch.equal(f["v"], rv), tag


def _close(x, y, what):
    d = float((x.float() - y.float()).abs().max())
    assert d <= 0.03 * float(y.float().abs().max()) + 0.03, f"{what} differs by {d}"


@pytest.mark.parametrize("geo,a", [(GRANITE_8B, 0.22), (GRANITE_2B, 0.22), (MINICPM_2B, 1.4 / math.sqrt(40))],
                         ids=["granite8b", "granite2b", "minicpm2b"])
def test_segment_one_launch_exact_and_replay(geo, a):
    L = _layer(geo, 10 + geo[0] % 97)
    gen = _gen(geo[0])
    attn = torch.randn((1, L.hidden), device=_dev(), generator=gen).half()
    h_in = torch.randn((1, L.hidden), device=_dev(), generator=gen).half()
    pos = torch.zeros(1, dtype=torch.int32, device=_dev())
    fp, f = _build(L, attn, h_in, pos, a)
    rp, r = _build(L, attn, h_in, pos, a, no_fuse=True)
    assert fp.fused and fp.kind == "stream" and fp.kernel_ops == 4 and fp.launches_per_run == 1
    assert not rp.fused and rp.kernel_ops == 0 and rp.launches_per_run == 8 + 2 * 2   # 8 single calls, 2 per scaled_add
    for p in (0, 7, S - 1):
        pos.fill_(p)
        k0, v0 = f["k"].clone(), f["v"].clone()
        fp.run()
        rp.run()
        torch.cuda.synchronize()
        _no_abort(f"pos {p}")
        _check_exact(f, a, f"fused pos {p}")
        _check_exact(r, a, f"per-op pos {p}")
        _check_rope(L, f, pos, k0, v0, f"pos {p}")
        for k in f:
            _close(f[k], r[k], f"pos {p}: {k}")


def _one_linear(K, N, gen):
    return (torch.randint(-2**31, 2**31 - 1, (K, N // 8), dtype=torch.int32, device=_dev(), generator=gen),
            ((torch.rand((K // 128, N), device=_dev(), generator=gen) * 0.5 + 0.75) / (6.1 * K**0.5)).half(),
            torch.randint(-2**31, 2**31 - 1, (K // 128, N // 8), dtype=torch.int32, device=_dev(), generator=gen))


def _linear_then_scaled(w, x, r, a, add=False):
    p = DecodeProgram()
    y = p.gemm_forward_cuda(x, *w, 8)
    out = p.add(y, r) if add else p.scaled_add(r, y, a)
    p.build()
    assert p.fused and p.kernel_ops == 1 and p.launches_per_run == 1
    p.run()
    torch.cuda.synchronize()
    _no_abort("linear + scaled_add")
    return y, out


def test_edge_values_bit_exact():
    """Overflow to inf near +-65504, fp16 subnormal results, and a multiplier whose fp16 rounding changes the product:
    each output bit-exact against torch on the program's raw y."""
    K, N = 2048, 4096
    gen = _gen(3)
    w = _one_linear(K, N, gen)
    x = torch.randn((1, K), device=_dev(), generator=gen).half()
    big = torch.tensor([65504.0, -65504.0, 65000.0, -64992.0], device=_dev()).half().repeat(N // 4).view(1, N)
    tiny = (torch.randint(-8, 9, (1, N), device=_dev(), generator=gen).float() * 2**-24).half()
    cases = [("overflow", big, 64.0), ("product overflow", big, 1.0e6), ("subnormal", tiny, 2.0**-20),
             ("a rounds in fp16", torch.randn((1, N), device=_dev(), generator=gen).half(), 1.4 / math.sqrt(40))]
    for name, r, a in cases:
        y, out = _linear_then_scaled(w, x, r, a)
        _assert_scaled_exact(out, r, y, a, name)
        if name.startswith("overflow"):
            assert torch.isinf(out).any() and torch.isfinite(out).any(), name
        if name == "subnormal":
            sub = (out != 0) & (out.abs() < 2.0**-14)
            assert sub.any(), name
        if name == "a rounds in fp16":
            a16 = float(torch.tensor(a).half())
            assert a16 != a
            assert not torch.equal(_bits(r + y * a16), _bits(out)), "the case does not tell an fp16 multiplier apart"


def test_alpha_one_equals_add():
    K, N = 2048, 4096
    gen = _gen(4)
    w = _one_linear(K, N, gen)
    x = torch.randn((1, K), device=_dev(), generator=gen).half()
    r = torch.randn((1, N), device=_dev(), generator=gen).half()
    y1, s = _linear_then_scaled(w, x, r, 1.0)
    y2, p = _linear_then_scaled(w, x, r, 1.0, add=True)
    assert torch.equal(y1, y2) and torch.equal(_bits(s), _bits(p))


@pytest.mark.parametrize("M", [2, 4])
def test_batched_rows_match_m1_programs(M):
    L = _layer(GRANITE_2B, 70)
    a = 0.22
    gen = _gen(M)
    attn = torch.randn((M, L.hidden), device=_dev(), generator=gen).half()
    h_in = torch.randn((M, L.hidden), device=_dev(), generator=gen).half()
    pos = torch.full((1,), 9, dtype=torch.int32, device=_dev())
    bp, b = _build(L, attn, h_in, pos, a, max_tokens=M)
    assert bp.fused and bp.kernel_ops == 4 and bp.launches_per_run == 1 and bp.tokens == M
    k0, v0 = b["k"].clone(), b["v"].clone()
    bp.run()
    torch.cuda.synchronize()
    _no_abort(f"batched M={M}")
    _check_exact(b, a, f"M={M}")
    _check_rope(L, b, pos, k0, v0, f"M={M}")
    for m in range(M):
        p1, o = _build(L, attn[m:m + 1].clone(), h_in[m:m + 1].clone(), pos, a)
        assert p1.fused
        o["k"].copy_(k0[m:m + 1])
        o["v"].copy_(v0[m:m + 1])
        p1.run()
        torch.cuda.synchronize()
        _no_abort(f"M=1 row {m}")
        for k in ("o", "h", "xn2", "gu", "act", "dn", "out", "xn", "qkv", "q"):
            assert torch.equal(_bits(b[k][m:m + 1]), _bits(o[k].reshape(b[k][m:m + 1].shape))), f"row {m}: {k}"
        assert torch.equal(b["k"][m], o["k"][0]) and torch.equal(b["v"][m], o["v"][0]), f"row {m}: cache"


def test_cuda_graph_replay_follows_pos():
    L = _layer(GRANITE_2B, 80)
    a = 0.22
    gen = _gen(8)
    attn = torch.randn((1, L.hidden), device=_dev(), generator=gen).half()
    h_in = torch.randn((1, L.hidden), device=_dev(), generator=gen).half()
    pos = torch.zeros(1, dtype=torch.int32, device=_dev())
    prog, f = _build(L, attn, h_in, pos, a)
    assert prog.fused
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        prog.run()                                  # warm-up outside the capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        prog.run()
    for p in (3, 4, 100):
        pos.fill_(p)
        h_in.copy_(torch.randn((1, L.hidden), device=_dev(), generator=gen).half())
        k0, v0 = f["k"].clone(), f["v"].clone()
        graph.replay()
        torch.cuda.synchronize()
        _no_abort(f"graph pos {p}")
        _check_exact(f, a, f"graph pos {p}")
        _check_rope(L, f, pos, k0, v0, f"graph pos {p}")
        assert not torch.equal(f["k"][:, p], k0[:, p]), p


def _minicpm3_segment(g, dense, at, freqs, attn, h, a, no_fuse):
    """[o, scaled_add, norm2, gate|up, silu, down, scaled_add] then the q-LoRA MLA chain (norm1', q_a|kv_a', ...)"""
    hm, xn2, h2 = (torch.empty((1, g.HID), dtype=F16, device=_dev()) for _ in range(3))
    act = torch.empty((1, g.INTER), dtype=F16, device=_dev())
    p = DecodeProgram()
    o = p.gemm_forward_cuda(attn, *dense.wo, 8)
    p.scaled_add(h, o, a, out=hm)
    p.layernorm_forward_cuda(hm, dense.n2, xn2, EPS)
    gu = p.gemm_forward_cuda(xn2, *dense.wgu, 8)
    p.silu_and_mul(act, gu)
    d = p.gemm_forward_cuda(act, *dense.wd, 8)
    p.scaled_add(hm, d, a, out=h2)
    b = at.record(p, h2, 0, freqs)
    prev = ext.get_knob(14)
    ext.set_knob(14, 1 if no_fuse else 0)
    try:
        p.build()
    finally:
        ext.set_knob(14, prev)
    return p, dict(b, o=o, hm=hm, xn2=xn2, gu=gu, act=act, d=d, h2=h2)


def test_minicpm3_segment_one_launch():
    g = MINICPM3_4B
    a = 1.4 / math.sqrt(62)
    cis, _ = _tables(g, 512)
    dense = Dense(g, 12)
    gen = _gen(6)
    attn = torch.randn((1, g.H * g.DV), device=_dev(), generator=gen).half()
    h = torch.randn((1, g.HID), device=_dev(), generator=gen).half()
    af, ar = Attn(g, 31), Attn(g, 31)
    pf, bf = _minicpm3_segment(g, dense, af, cis, attn, h, a, False)
    pr, br = _minicpm3_segment(g, dense, ar, cis, attn, h, a, True)
    assert pf.fused and pf.kernel_ops == 6 and pf.launches_per_run == 1 and not pr.fused
    pf.run()
    pr.run()
    torch.cuda.synchronize()
    _no_abort("minicpm3 segment")
    for b, tag in ((bf, "fused"), (br, "per-op")):
        _assert_scaled_exact(b["hm"], h, b["o"], a, f"{tag} h")
        _assert_scaled_exact(b["h2"], b["hm"], b["d"], a, f"{tag} h2")
    pos = int(af.pos.item())
    k2, v2 = torch.zeros_like(af.k_cache), torch.zeros_like(af.v_cache)
    q2, qan, ckv = af.standalone(bf, 0, cis, k2, v2)
    torch.cuda.synchronize()
    assert torch.equal(bf["q_out"], q2) and torch.equal(bf["qan"], qan) and torch.equal(bf["ckv"], ckv)
    assert torch.equal(af.k_cache, k2) and torch.equal(af.v_cache, v2)
    for name, x, y in (("h2", bf["h2"], br["h2"]), ("q_out", bf["q_out"], br["q_out"]),
                       ("k", af.k_cache[0, pos], ar.k_cache[0, pos]), ("v", af.v_cache[0, pos], ar.v_cache[0, pos])):
        err, tol = _ulps_of_rms(x, y, 8)
        assert err <= tol + 1e-3, f"{name}: {err:.3e} > {tol:.3e}"


def test_after_a_moe_block_replays_per_op():
    moe = Moe(8, 1024, 768, 128, 2, seed=5)
    a = 0.22
    gen = _gen(9)
    x = torch.randn((1, 1024), device=_dev(), generator=gen).half()
    r = torch.randn((1, 1024), device=_dev(), generator=gen).half()
    p = DecodeProgram()
    xn = torch.empty_like(x)
    p.layernorm_forward_cuda(x, moe.norm, xn, EPS)
    y = p.sparse_moe(xn, moe.gate, moe.w1, moe.w2, moe.top_k)
    out = p.scaled_add(r, y, a)
    p.build()
    assert not p.fused and p.launches_per_run == 1 + 6 + 2
    p.run()
    torch.cuda.synchronize()
    _assert_scaled_exact(out, r, y, a, "after sparse_moe")


def test_recorder_checks():
    from autoawq_b200._cabi import B200AwqError

    p = DecodeProgram()
    t = torch.zeros((1, 64), dtype=F16, device=_dev())
    for bad in (math.inf, -math.inf, math.nan):
        with pytest.raises(B200AwqError):
            p.scaled_add(t, t.clone(), bad)
    with pytest.raises(B200AwqError):
        p.scaled_add(t, torch.zeros((1, 64), dtype=torch.float32, device=_dev()), 0.5)
    with pytest.raises(B200AwqError):
        p.scaled_add(t, torch.zeros((1, 32), dtype=F16, device=_dev()), 0.5)
    with pytest.raises(B200AwqError):
        p.scaled_add(t, torch.zeros((1, 128), dtype=F16, device=_dev())[:, ::2], 0.5)   # not contiguous
