"""GPU tests of residual adds in decode programs (B200AWQ_OP_ADD, DecodeProgram.add): a decoder layer recorded from one
attention call to the next - [o + h_in -> h, norm2(h), gate|up, silu, down + h -> out, norm1'(out), qkv'] - runs as one
persistent kernel with the adds folded into the epilogues of o and down.  Every buffer is checked against the fp64
oracle on its recorded inputs, every add bit-exactly against fp16(a + b), and the whole segment bit-for-bit against the
same linears recorded without adds (today's kernels) plus torch.add."""
import numpy as np
import pytest
import torch

from oracle import awq_oracle as O
from test_gpu_program import EPS, Block, _close, _no_abort, _t
from test_gpu_program_moe import Moe, _check_block

pytestmark = pytest.mark.gpu

F16 = torch.float16


def _dev():
    return torch.device("cuda:0")


def _rand(shape, seed):
    return _t(np.random.default_rng(seed).standard_normal(shape).astype(np.float16))


def _segment(api, b, attn, h_in, add=None):
    """The attention-to-attention segment against `api`; `add(a, b)` records the residual adds (default: api.add)."""
    add = add or api.add
    M = attn.shape[0]
    o = api.gemm_forward_cuda(attn, *b.w["o"], 8)
    h = add(o, h_in)
    xn2 = torch.empty((M, b.hidden), dtype=F16, device=_dev())
    api.layernorm_forward_cuda(h, b.norm2_t, xn2, EPS)
    gu = api.gemm_forward_cuda(xn2, *b.w["gate_up"], 8)
    act = torch.empty((M, b.inter), dtype=F16, device=_dev())
    api.silu_and_mul(act, gu)
    down = api.gemm_forward_cuda(act, *b.w["down"], 8)
    out = add(down, h)
    xn = torch.empty((M, b.hidden), dtype=F16, device=_dev())
    api.layernorm_forward_cuda(out, b.norm1_t, xn, EPS)
    qkv = api.gemm_forward_cuda(xn, *b.w["qkv"], 8)
    return dict(attn=attn, h_in=h_in, o=o, h=h, xn2=xn2, gu=gu, act=act, down=down, out=out, xn=xn, qkv=qkv)


def _fused(b, attn, h_in, max_tokens=1, knob=None):
    from autoawq_b200 import ext
    from autoawq_b200.program import DecodeProgram

    prev = {k: ext.get_knob(k) for k in (knob or {})}
    for k, v in (knob or {}).items():
        ext.set_knob(k, v)
    try:
        prog = DecodeProgram(max_tokens=max_tokens)
        bufs = _segment(prog, b, attn, h_in)
        prog.build()
    finally:
        for k, v in prev.items():
            ext.set_knob(k, v)
    return prog, bufs


def _np(t):
    return t.detach().float().cpu().numpy().astype(np.float16)


def _add_exact(a, b):
    return (a.astype(np.float32) + b.astype(np.float32)).astype(np.float16)


def _check_segment(b, bufs, tag):
    """Each linear against the fp64 oracle on its recorded input, each add bit-exact, the norms against rmsnorm_f64."""
    v = {k: _np(t) for k, t in bufs.items()}
    for name, xin, yout in [("o", v["attn"], v["o"]), ("gate_up", v["xn2"], v["gu"]), ("down", v["act"], v["down"]),
                            ("qkv", v["xn"], v["qkv"])]:
        w = b.np[name]["w"]
        _close(yout, O.gemm_f64(xin, w), np.abs(xin.astype(np.float64)) @ np.abs(w.astype(np.float64)), f"{tag} {name}")
    assert np.array_equal(v["h"].view(np.uint16), _add_exact(v["o"], v["h_in"]).view(np.uint16)), f"{tag}: o + h_in"
    assert np.array_equal(v["out"].view(np.uint16), _add_exact(v["down"], v["h"]).view(np.uint16)), f"{tag}: down + h"
    np.testing.assert_allclose(v["xn2"], O.rmsnorm_f64(v["h"], b.norm2, EPS), rtol=2e-3, atol=2e-3, err_msg=f"{tag} norm2")
    np.testing.assert_allclose(v["xn"], O.rmsnorm_f64(v["out"], b.norm1, EPS), rtol=2e-3, atol=2e-3, err_msg=f"{tag} norm1")
    g64 = v["gu"][:, : b.inter].astype(np.float64)
    np.testing.assert_allclose(v["act"], g64 / (1 + np.exp(-g64)) * v["gu"][:, b.inter:].astype(np.float64),
                               rtol=2e-3, atol=2e-3, err_msg=f"{tag} silu")


def _unfused_reference(b, attn, h_in):
    """The same segment as today's correct split: [o] | torch.add | [norm2, gate|up, silu, down] | torch.add |
    [norm1, qkv], three programs without adds on today's kernels."""
    from autoawq_b200.program import DecodeProgram

    M = attn.shape[0]
    progs = [DecodeProgram(max_tokens=M) for _ in range(3)]
    o = progs[0].gemm_forward_cuda(attn, *b.w["o"], 8)
    h = torch.empty_like(o)
    xn2 = torch.empty((M, b.hidden), dtype=F16, device=_dev())
    progs[1].layernorm_forward_cuda(h, b.norm2_t, xn2, EPS)
    gu = progs[1].gemm_forward_cuda(xn2, *b.w["gate_up"], 8)
    act = torch.empty((M, b.inter), dtype=F16, device=_dev())
    progs[1].silu_and_mul(act, gu)
    down = progs[1].gemm_forward_cuda(act, *b.w["down"], 8)
    out = torch.empty_like(down)
    xn = torch.empty((M, b.hidden), dtype=F16, device=_dev())
    progs[2].layernorm_forward_cuda(out, b.norm1_t, xn, EPS)
    qkv = progs[2].gemm_forward_cuda(xn, *b.w["qkv"], 8)
    for p in progs:
        p.build()
        assert p.fused
    progs[0].run()
    torch.add(o, h_in, out=h)
    progs[1].run()
    torch.add(down, h, out=out)
    progs[2].run()
    torch.cuda.synchronize()
    return progs, dict(attn=attn, h_in=h_in, o=o, h=h, xn2=xn2, gu=gu, act=act, down=down, out=out, xn=xn, qkv=qkv)


def _assert_same(a, b, what):
    for k in a:
        assert torch.equal(a[k], b[k]), f"{what}: {k} differs"


@pytest.mark.parametrize("G", [128, 64])
def test_segment_fuses_and_matches_oracle_and_unfused_programs(G):
    b = Block(2048, 4096, 3072, G, seed=3 + G)
    attn, h_in = _rand((1, 2048), 1), _rand((1, 2048), 2)
    prog, bufs = _fused(b, attn, h_in)
    assert prog.fused and prog.kind == "stream" and prog.kernel_ops == 4 and prog.launches_per_run == 1
    prog.run()
    torch.cuda.synchronize()
    _no_abort("residual segment")
    _check_segment(b, bufs, f"G{G}")
    fused = {k: t.clone() for k, t in bufs.items()}
    _, ref = _unfused_reference(b, attn, h_in)
    _assert_same(fused, ref, "fused vs unfused programs + torch.add")
    # the per-op replay (knob 14 = 1: do not fuse) issues torch.add: the same values
    rp, rbufs = _fused(b, attn, h_in, knob={14: 1})
    assert not rp.fused and rp.kernel_ops == 0
    rp.run()
    torch.cuda.synchronize()
    _check_segment(b, rbufs, f"per-op G{G}")
    assert torch.equal(rbufs["h"], torch.add(rbufs["o"], rbufs["h_in"]))     # the adds, on equal inputs
    assert torch.equal(rbufs["out"], torch.add(rbufs["down"], rbufs["h"]))
    # knob 9 = 12 (12-warp plain kernel) does not change a residual program: it always runs 8 warps x 4 stages
    from autoawq_b200 import ext

    prev = ext.get_knob(9)
    ext.set_knob(9, 12)
    try:
        prog.run()
        torch.cuda.synchronize()
    finally:
        ext.set_knob(9, prev)
    _assert_same(fused, bufs, "knob 9 = 12")
    # two more runs: bit-identical
    prog.run()
    torch.cuda.synchronize()
    _assert_same(fused, bufs, "rerun")


@pytest.mark.parametrize("M", [2, 3, 4])
def test_batched_segment_each_token_matches_m1_program(M):
    b = Block(2048, 4096, 3072, 128, seed=11)
    attn, h_in = _rand((M, 2048), 5), _rand((M, 2048), 6)
    prog, bufs = _fused(b, attn, h_in, max_tokens=M)
    assert prog.fused and prog.tokens == M and prog.kernel_ops == 4
    prog.run()
    torch.cuda.synchronize()
    _no_abort(f"batched M={M}")
    _check_segment(b, bufs, f"M={M}")
    for m in range(M):
        p1, b1 = _fused(b, attn[m:m + 1].clone(), h_in[m:m + 1].clone())
        assert p1.fused
        p1.run()
        torch.cuda.synchronize()
        for k in b1:
            assert torch.equal(bufs[k][m:m + 1], b1[k]), f"M={M} token {m}: {k}"
    # unfused batched programs + torch.add: the same bits
    _, ref = _unfused_reference(b, attn, h_in)
    _assert_same({k: t.clone() for k, t in bufs.items()}, ref, f"M={M} vs unfused")


@pytest.mark.parametrize("M", [1, 4])
def test_llama3_8b_layer_segment_fuses(M):
    b = Block(4096, 14336, 6144, 128, seed=21)
    attn, h_in = _rand((M, 4096), 7), _rand((M, 4096), 8)
    prog, bufs = _fused(b, attn, h_in, max_tokens=M)
    assert prog.fused and prog.kind == "stream" and prog.kernel_ops == 4
    prog.run()
    torch.cuda.synchronize()
    _no_abort("llama3-8b segment")
    _check_segment(b, bufs, f"llama3-8b M={M}")


def test_mixtral_block_residual_fuses_and_matches_replay_and_oracle():
    from autoawq_b200 import ext
    from autoawq_b200.program import DecodeProgram

    moe = Moe(8, 1024, 768, 128, 2, seed=5)
    h = _rand((1, 1024), 9)

    def rec(knob14):
        prev = ext.get_knob(14)
        ext.set_knob(14, knob14)
        try:
            p = DecodeProgram()
            xn = torch.empty_like(h)
            p.layernorm_forward_cuda(h, moe.norm, xn, EPS)
            mo = p.sparse_moe(xn, moe.gate, moe.w1, moe.w2, moe.top_k, True)
            out = p.add(mo, h)
            p.build()
        finally:
            ext.set_knob(14, prev)
        p.run()
        torch.cuda.synchronize()
        return p, xn, mo, out

    p, xn, mo, out = rec(0)
    assert p.fused and p.kernel_ops == 2
    _no_abort("mixtral residual")
    _check_block(moe, xn, p.moe_buffers(0), True, "fused moe + residual")
    assert np.array_equal(_np(out).view(np.uint16), _add_exact(_np(mo), _np(h)).view(np.uint16))
    r, xr, mr, outr = rec(1)
    assert not r.fused
    _check_block(moe, xr, r.moe_buffers(0), True, "per-op moe + residual")
    assert torch.equal(outr, torch.add(mr, h))
    rms = float(outr.float().pow(2).mean().sqrt())
    assert float((outr.float() - out.float()).abs().max()) <= 0.02 * rms + 2e-3


def test_in_program_residual_two_ops_back_and_fallbacks():
    from autoawq_b200.program import DecodeProgram

    b = Block(2048, 4096, 3072, 128, seed=31)
    x = _rand((1, 2048), 12)
    w2 = Block(2048, 2048, 2048, 128, seed=32)

    def chain(window_ops):
        # y0 = x W_o ; y1 = y0 W2 ; ... ; s = last + y0 (the residual `window_ops` kernel ops before last)
        p = DecodeProgram()
        y0 = p.gemm_forward_cuda(x, *b.w["o"], 8)
        y = y0
        for _ in range(window_ops - 1):
            y = p.gemm_forward_cuda(y, *w2.w["o"], 8)
        last = p.gemm_forward_cuda(y, *w2.w["o"], 8)
        s = p.add(last, y0)
        p.build()
        p.run()
        torch.cuda.synchronize()
        return p, dict(y0=y0, last=last, s=s)

    p, t = chain(2)                        # residual two kernel ops back: fused
    assert p.fused and p.kernel_ops == 3
    _no_abort("two back")
    assert torch.equal(t["s"], torch.add(t["last"], t["y0"]))
    p, t = chain(4)                        # four back: the row the producer itself publishes into, fused
    assert p.fused and p.kernel_ops == 5
    _no_abort("four back")
    assert torch.equal(t["s"], torch.add(t["last"], t["y0"]))
    p, t = chain(5)                        # five back: outside the window, per-op replay
    assert not p.fused
    assert torch.equal(t["s"], torch.add(t["last"], t["y0"]))
    # M > max_tokens: per-op replay with correct results
    attn, h_in = _rand((2, 2048), 13), _rand((2, 2048), 14)
    prog, bufs = _fused(b, attn, h_in, max_tokens=1)
    assert not prog.fused
    prog.run()
    torch.cuda.synchronize()
    _check_segment(b, bufs, "M=2 > max_tokens")


def test_aliased_residual_replays_per_op():
    from autoawq_b200.program import DecodeProgram

    b = Block(2048, 2048, 2048, 128, seed=41)
    x, r0 = _rand((1, 2048), 15), _rand((1, 2048), 16)
    r = r0.clone()
    p = DecodeProgram()
    y = p.gemm_forward_cuda(x, *b.w["o"], 8)
    s = p.add(y, r)                                   # external residual r ...
    xn = torch.empty_like(s)
    p.layernorm_forward_cuda(s, b.norm1_t, xn, EPS)
    z = p.gemm_forward_cuda(xn, *b.w["qkv"], 8)
    p.add(z, s, out=r)                                # ... that a later add of the program overwrites
    p.build()
    assert not p.fused
    p.run()
    torch.cuda.synchronize()
    s_ref = torch.add(y, r0)
    assert torch.equal(s, s_ref)
    assert torch.equal(r, torch.add(z, s_ref))


def test_cuda_graph_replay_follows_changed_inputs():
    b = Block(2048, 4096, 3072, 128, seed=51)
    attn, h_in = _rand((1, 2048), 17), _rand((1, 2048), 18)
    prog, bufs = _fused(b, attn, h_in)
    assert prog.fused
    prog.run()
    torch.cuda.synchronize()
    first = {k: t.clone() for k, t in bufs.items()}
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            prog.run()
    torch.cuda.synchronize()
    attn.copy_(_rand((1, 2048), 19))
    h_in.copy_(_rand((1, 2048), 20))
    g.replay()
    torch.cuda.synchronize()
    _no_abort("graph")
    assert not torch.equal(bufs["out"], first["out"])
    _check_segment(b, bufs, "graph replay")
    eager = {k: t.clone() for k, t in bufs.items()}
    prog.run()
    torch.cuda.synchronize()
    _assert_same(eager, bufs, "graph vs eager")
