"""GPU tests of the LayerNorm blocks' ops (B200AWQ_OP_LAYER_NORM, _GELU, _GELU_TANH): the stand-alone kernels against a
numpy oracle of the documented summation order and against torch / transformers, and decode programs of Command-R,
StarCoder2 and MPT segments that fold them (the LayerNorm into a linear's staging, the GELU into its finish).

What is bit-identical: the stand-alone LayerNorm and the oracle (r taken with torch.rsqrt on the device, the same
rsqrtf); a fused program's LayerNorm and GELU outputs and the stand-alone ops on the program's own inputs; its q and
cache rows and ext.rope_kv_cache on its own qkv.  The linears of a fused program and of the per-op replay use different
kernels (summation orders), so those buffers are compared within the tolerance of test_gpu_program_rope.py."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_gpu_program import _no_abort
from test_gpu_program_rope import _build, _caches, _freqs, _linear, _ulps

pytestmark = pytest.mark.gpu

F16 = torch.float16
EPS = 1e-5


def _dev():
    return torch.device("cuda:0")


# ------------------------------------------------------------------------------------------ stand-alone ops
def _ordered_sum(v):
    """include/b200awq.h's order over per-pair terms v [M, K / 2] (float32): thread t < 256 sums the pairs of its
    chunks c = 8 t + 2048 p in order, the warps' lanes meet in the xor butterfly, the 8 warp totals are added in order."""
    M, P = v.shape
    chunks = P // 4
    v = v.reshape(M, chunks, 4)
    s = np.zeros((M, 256), dtype=np.float32)
    for p in range((chunks + 255) // 256):
        j = np.arange(256) + 256 * p
        ok = j < chunks
        for q in range(4):
            s[:, ok] = s[:, ok] + v[:, j[ok], q]
    w = s.reshape(M, 8, 32)
    for off in (16, 8, 4, 2, 1):
        w = w + w[..., np.arange(32) ^ off]
    tot = np.zeros(M, dtype=np.float32)
    for i in range(8):
        tot = tot + w[:, i, 0]
    return tot


def ln_oracle(x, w, b, eps):
    """b200awq_layer_norm in numpy float32, with r = torch.rsqrt on the device (the kernel's rsqrtf)."""
    xf = x.float().cpu().numpy()
    K = xf.shape[1]
    mean = _ordered_sum(xf[:, 0::2] + xf[:, 1::2]) / np.float32(K)
    d = xf - mean[:, None]
    var = _ordered_sum(d[:, 0::2] * d[:, 0::2] + d[:, 1::2] * d[:, 1::2]) / np.float32(K)
    r = torch.rsqrt(torch.from_numpy(var + np.float32(eps)).to(_dev())).cpu().numpy()
    y = (d * r[:, None]) * w.float().cpu().numpy()
    if b is not None:
        y = y + b.float().cpu().numpy()
    return torch.from_numpy(y.astype(np.float16)).to(_dev())


def _near_torch(out, ref):
    """Within one fp16 ulp, or within one fp16 ulp of 1.0 (2^-10) where x is close to the row's mean: torch's mean
    (Welford, another summation order) differs from the two-pass one in its last fp32 bits, and x - mean cancels."""
    return bool(((_ulps(out, ref) <= 1) | ((out.float() - ref.float()).abs() <= 2**-10)).all())


def _rows(M, K, seed, offset=0.0, spread=1.0):
    g = torch.Generator(device=_dev()).manual_seed(seed)
    return (offset + spread * torch.randn((M, K), device=_dev(), generator=g)).half()


@pytest.mark.parametrize("K", [3072, 4096, 6144, 8192])
@pytest.mark.parametrize("M", [1, 2, 4])
@pytest.mark.parametrize("bias", [True, False])
def test_layer_norm_matches_oracle_torch_and_cohere(K, M, bias):
    from autoawq_b200 import ext
    from transformers.models.cohere.modeling_cohere import CohereLayerNorm

    g = torch.Generator(device=_dev()).manual_seed(K + M)
    w = (1 + 0.2 * torch.randn(K, device=_dev(), generator=g)).half()
    b = (0.1 * torch.randn(K, device=_dev(), generator=g)).half() if bias else None
    for x in (_rows(M, K, K * M), _rows(M, K, K * M + 1, offset=100.0)):   # the second: mean 100x the spread
        out = torch.empty_like(x)
        ext.layer_norm(x, w, b, out, EPS)
        assert torch.equal(out, ln_oracle(x, w, b, EPS))
        ref = F.layer_norm(x, (K,), w, b, EPS)
        assert _near_torch(out, ref)
        if not bias:
            cn = CohereLayerNorm(K, eps=EPS, bias=False).to(_dev())
            cn.weight.data = w.clone()
            assert _near_torch(out, cn(x))


@pytest.mark.parametrize("approximate", ["none", "tanh"])
def test_gelu_every_fp16_value(approximate):
    from autoawq_b200 import ext

    x = torch.arange(-32768, 32768, dtype=torch.int32, device=_dev()).to(torch.int16).view(F16).reshape(256, 256)
    out = torch.empty_like(x)
    ext.gelu(out, x, approximate)
    ref = F.gelu(x, approximate=approximate)
    fin = torch.isfinite(ref) & torch.isfinite(out)
    assert torch.equal(torch.isnan(out), torch.isnan(ref))
    assert torch.equal(out[torch.isinf(ref)], ref[torch.isinf(ref)])
    a, r = out[fin], ref[fin]
    zero = (a == 0) & (r == 0)                                     # +0 and -0 count as equal
    assert int(_ulps(a[~zero], r[~zero]).max()) <= 1


# ------------------------------------------------------------------------------------------ decode programs
# name: (hidden, q heads, kv heads, intermediate, Command-R block, GELU approximation, rope, biases)
MODELS = {
    "command-r-v01": (8192, 64, 64, 22528, True, None, True, False),
    "starcoder2-3b": (3072, 24, 2, 12288, False, "tanh", True, True),
    "starcoder2-15b": (6144, 48, 4, 24576, False, "tanh", True, True),
    "mpt-7b": (4096, 32, 32, 16384, False, "none", False, False),
}


class Block:
    """One layer's random GEMM-layout AWQ weights, norms and biases at a model's geometry."""

    def __init__(self, model, seed, S=64):
        hid, H, KV, inter, cohere, approx, rope, biases = MODELS[model]
        self.hid, self.H, self.KV, self.inter, self.cohere, self.approx, self.rope = hid, H, KV, inter, cohere, approx, rope
        self.S, D = S, 128
        qkv_n = (H + 2 * KV) * D
        shapes = dict(o=(H * D, hid), qkv=(hid, qkv_n), down=(inter, hid))
        shapes["gu" if cohere else "fc"] = (hid, 2 * inter if cohere else inter)
        self.w = {k: _linear(K, N, 128, seed + i) for i, (k, (K, N)) in enumerate(sorted(shapes.items()))}
        g = torch.Generator(device=_dev()).manual_seed(seed + 10)
        self.b = {k: (0.05 * torch.randn(N, device=_dev(), generator=g)).half() if biases else None
                  for k, (K, N) in shapes.items()}
        self.ln = {n: ((1 + 0.1 * torch.randn(hid, device=_dev(), generator=g)).half(),
                       (0.05 * torch.randn(hid, device=_dev(), generator=g)).half() if not cohere else None)
                   for n in ("n1", "n2")}
        self.freqs = _freqs(D, S, 8e6 if cohere else 1e5) if rope else None

    def record(self, api, M, pos, attn, x, xn=None):
        """The segment in program.py's recording order; returns the buffers it names (xn: Command-R's normed input,
        read by gate|up and overwritten by the segment's LayerNorm)."""
        o = api.gemm_forward_cuda(attn, *self.w["o"], 8, bias=self.b["o"])
        h = api.add(o, x)
        bufs = dict(o=o, h=h)
        if self.cohere:
            gu = api.gemm_forward_cuda(xn, *self.w["gu"], 8, bias=self.b["gu"])
            act = torch.empty((M, self.inter), dtype=F16, device=_dev())
            api.silu_and_mul(act, gu)
            bufs.update(gu=gu, act=act)
        else:
            hn = torch.empty((M, self.hid), dtype=F16, device=_dev())
            api.layer_norm(h, *self.ln["n2"], hn, EPS)
            fc = api.gemm_forward_cuda(hn, *self.w["fc"], 8, bias=self.b["fc"])
            act = torch.empty_like(fc)
            api.gelu(act, fc, self.approx)
            bufs.update(hn=hn, fc=fc, act=act)
        dn = api.gemm_forward_cuda(act, *self.w["down"], 8, bias=self.b["down"])
        out = api.add(dn, h)
        xn2 = xn if xn is not None else torch.empty((M, self.hid), dtype=F16, device=_dev())
        api.layer_norm(out, *self.ln["n1"], xn2, EPS)
        qkv = api.gemm_forward_cuda(xn2, *self.w["qkv"], 8, bias=self.b["qkv"])
        bufs.update(dn=dn, out=out, xn2=xn2, qkv=qkv)
        if self.rope:
            kc, vc = _caches(M, self.S, self.KV, 128, 5)
            bufs.update(q=api.rope_kv_cache(qkv, self.freqs, pos, kc, vc, self.H, self.KV), k=kc, v=vc)
        return bufs


def _inputs(B, M, seed):
    g = torch.Generator(device=_dev()).manual_seed(seed)
    return ((torch.randn((M, B.H * 128), device=_dev(), generator=g) * 0.5).half(),
            torch.randn((M, B.hid), device=_dev(), generator=g).half(),
            torch.randn((M, B.hid), device=_dev(), generator=g).half())


def _check_fused_ops(B, f, pos):
    """The fused program's LayerNorm / GELU outputs and rotation against the stand-alone ops on its own inputs."""
    from autoawq_b200 import ext

    want = torch.empty_like(f["xn2"])
    ext.layer_norm(f["out"], *B.ln["n1"], want, EPS)
    assert torch.equal(f["xn2"], want)
    if not B.cohere:
        ext.layer_norm(f["h"], *B.ln["n2"], want, EPS)
        assert torch.equal(f["hn"], want)
        act = torch.empty_like(f["fc"])
        ext.gelu(act, f["fc"], B.approx)
        assert torch.equal(f["act"], act)
    if B.rope:
        k0, v0 = _caches(f["k"].shape[0], B.S, B.KV, 128, 5)
        rq = ext.rope_kv_cache(f["qkv"], B.freqs, pos, k0, v0, B.H, B.KV)
        assert torch.equal(f["q"], rq) and torch.equal(f["k"], k0) and torch.equal(f["v"], v0)


def _close(f, r, keys):
    for k in keys:
        d = float((f[k].float() - r[k].float()).abs().max())
        assert d <= 0.03 * float(r[k].float().abs().max()) + 0.03, f"{k} differs by {d}"


@pytest.mark.parametrize("model", sorted(MODELS))
def test_segment_fuses_into_one_launch_and_matches_replay(model):
    B = Block(model, seed=len(model))
    attn, x, xn = _inputs(B, 1, 3)
    pos = torch.full((1,), 5, dtype=torch.int32, device=_dev())
    xf, xr = xn.clone(), xn.clone()
    f_prog, f = _build(lambda p: B.record(p, 1, pos, attn, x, xf if B.cohere else None), 1, False)
    r_prog, r = _build(lambda p: B.record(p, 1, pos, attn, x, xr if B.cohere else None), 1, True)
    assert f_prog.fused and f_prog.kernel_ops == 4 and f_prog.launches_per_run == 1
    assert not r_prog.fused and r_prog.launches_per_run == len(r_prog._ops)
    f_prog.run()
    r_prog.run()
    torch.cuda.synchronize()
    _no_abort(model)
    _check_fused_ops(B, f, pos)
    _close(f, r, f.keys())


def test_cuda_graph_replay_follows_the_position():
    B = Block("starcoder2-3b", seed=7)
    attn, x, _ = _inputs(B, 1, 4)
    pos = torch.zeros(1, dtype=torch.int32, device=_dev())
    prog, f = _build(lambda p: B.record(p, 1, pos, attn, x), 1, False)
    assert prog.fused
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        prog.run()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        prog.run()
    k0, v0 = _caches(1, B.S, B.KV, 128, 5)
    for p in (1, 9, 30):
        pos.fill_(p)
        f["k"].copy_(k0)
        f["v"].copy_(v0)
        graph.replay()
        torch.cuda.synchronize()
        _no_abort(f"pos {p}")
        assert not torch.equal(f["k"][0, p], k0[0, p])
        _check_fused_ops(B, f, pos)


def _reference_segment(B, M, attn, x):
    """The StarCoder2 / MPT segment in torch over dequantized weights, with the stand-alone LayerNorm and F.gelu."""
    from autoawq_b200 import ext

    lin = lambda a, k: (a.float() @ ext.dequantize_weights_cuda(*B.w[k]).float() +   # noqa: E731
                        (B.b[k].float() if B.b[k] is not None else 0)).half()
    h = (lin(attn, "o").float() + x.float()).half()
    hn = ln_oracle(h, *B.ln["n2"], EPS)
    act = F.gelu(lin(hn, "fc"), approximate=B.approx)
    out = (lin(act, "down").float() + h.float()).half()
    return dict(h=h, out=out, qkv=lin(ln_oracle(out, *B.ln["n1"], EPS), "qkv"))


@pytest.mark.parametrize("M", [2, 4])
def test_batched_programs_replay_per_op(M):
    B = Block("starcoder2-3b", seed=11)
    attn, x, _ = _inputs(B, M, 6)
    pos = torch.full((1,), 2, dtype=torch.int32, device=_dev())
    prog, f = _build(lambda p: B.record(p, M, pos, attn, x), 4, False)
    assert not prog.fused and prog.tokens == M and prog.launches_per_run == len(prog._ops)
    prog.run()
    torch.cuda.synchronize()
    assert torch.equal(f["hn"], ln_oracle(f["h"], *B.ln["n2"], EPS))
    assert torch.equal(f["xn2"], ln_oracle(f["out"], *B.ln["n1"], EPS))
    assert int(_ulps(f["act"], F.gelu(f["fc"], approximate="tanh")).max()) <= 1
    _close(f, _reference_segment(B, M, attn, x), ("h", "out", "qkv"))


def test_rejected_sequences_replay_correctly():
    """Sequences program_create does not fuse (tests/test_program_layernorm_cpu.py) replay per op and compute what the
    ops say."""
    from autoawq_b200 import ext
    from autoawq_b200.program import DecodeProgram

    K, N = 1024, 4096
    w1, w2 = _linear(K, N, 128, 21), _linear(N, K, 128, 22)
    x, r = torch.randn((1, K), device=_dev()).half(), torch.randn((1, N), device=_dev()).half()
    deq = lambda w: ext.dequantize_weights_cuda(*w).float()   # noqa: E731

    # each returns the buffers it names and, after a run, the GELU's expected output
    def gelu_after_add(p):                # a GELU after an ADD
        y = p.gemm_forward_cuda(x, *w1, 8)
        a = p.add(y, r)
        g = torch.empty_like(a)
        p.gelu(g, a, "tanh")
        return dict(g=g, z=p.gemm_forward_cuda(g, *w2, 8)), lambda: F.gelu(a, approximate="tanh")

    def raw_y_read(p):                    # the linear's raw y read after its GELU
        y = p.gemm_forward_cuda(x, *w1, 8)
        g = torch.empty_like(y)
        p.gelu(g, y, "none")
        z = p.gemm_forward_cuda(g, *w2, 8)
        return dict(g=g, z=z, z2=p.gemm_forward_cuda(y, *w2, 8)), lambda: F.gelu(y)

    def gelu_in_place(p):
        y = p.gemm_forward_cuda(x, *w1, 8)
        p.gelu(y, y, "tanh")
        return dict(g=y, z=p.gemm_forward_cuda(y, *w2, 8)), lambda: F.gelu(ext.gemm_forward_cuda(x, *w1, 8),
                                                                           approximate="tanh")

    for rec in (gelu_after_add, raw_y_read, gelu_in_place):
        prog = DecodeProgram()
        bufs, want = rec(prog)
        prog.build()
        assert not prog.fused, rec.__name__
        prog.run()
        torch.cuda.synchronize()
        assert int(_ulps(bufs["g"], want()).max()) <= 1, rec.__name__
        zr = (bufs["g"].float() @ deq(w2)).half()
        d = float((bufs["z"].float() - zr.float()).abs().max())
        assert d <= 0.03 * float(zr.float().abs().max()) + 0.03, rec.__name__
