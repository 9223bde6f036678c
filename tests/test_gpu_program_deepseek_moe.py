"""DeepSeek-MoE expert blocks in M = 1 stream decode programs (DecodeProgram.deepseek_moe, B200AWQ_OP_DEEPSEEK_MOE):
fp32 router logits exchanged across the grid, softmax / sigmoid-with-groups routing, the routed experts and the shared
expert in stream_deepseek_moe_kernel.

Per stage, on the program's own recorded inputs: the logits against the fp64 router matmul, the ids exactly and the fp32
weights within 4 ulps against the routing oracle applied to the recorded logits, gate|up, down and the shared expert
against fp64, SiLU*mul, the per-slot c, the combine and + y_s bit for bit from the recorded tensors.  Then the fused block
against transformers' DeepseekV2Moe / DeepseekV3MoE restated over WQLinear_GEMM and against its per-op replay, and a
V2-Lite segment [o + h, norm2, deepseek_moe + h, norm1', q_proj', kv_a_proj_with_mqa'] as one launch, also replayed in
a CUDA graph."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from autoawq_b200 import ext, packing
from autoawq_b200.linear import WQLinear_GEMM
from autoawq_b200.program import DecodeProgram
from test_gpu_program import _close, _no_abort
from test_gpu_program_moe import Moe, _np
from test_program_deepseek_moe_cpu import route_oracle

pytestmark = pytest.mark.gpu

EPS = 1e-6
# (E, top_k, H, I, n_shared, G, scoring, n_group, topk_group, norm, rsf)
CASES = [(64, 6, 2048, 1408, 2, 128, "softmax", 1, 1, False, 1.0),            # DeepSeek-V2-Lite
         (64, 6, 2048, 1408, 2, 128, "sigmoid", 1, 1, True, 2.446),           # Moonlight-16B-A3B
         (128, 8, 1024, 512, 1, 128, "sigmoid", 8, 4, True, 2.5),             # V3-style groups
         (128, 8, 1024, 512, 2, 64, "sigmoid", 8, 3, False, 1.5)]


def _dev():
    return torch.device("cuda:0")


class DsMoe(Moe):
    """Moe plus a shared expert (the stacked E = 1 tensors of I_s = n_shared I) and a correction bias."""

    def __init__(self, E, H, I, G, top_k, n_shared, seed):
        super().__init__(E, H, I, G, top_k, seed)
        sh = Moe(1, H, n_shared * I, G, 1, seed + 1000)
        self.I_s = n_shared * I
        self.ws1, self.ws2 = tuple(t[0] for t in sh.w1), tuple(t[0] for t in sh.w2)
        self._sh = sh
        g = torch.Generator(device=_dev()).manual_seed(seed + 7)
        self.bias = (torch.randn(E, device=_dev(), generator=g) * 0.05).float()

    def deq_shared(self, which):
        return self._sh.deq(which, 0)


def _record(prog, moe, x, scoring, n_group, topk_group, norm, rsf):
    return prog.deepseek_moe(x, moe.gate, moe.w1, moe.w2, moe.top_k, (moe.ws1, moe.ws2), scoring,
                             e_score_correction_bias=moe.bias if scoring == "sigmoid" else None, n_group=n_group,
                             topk_group=topk_group, norm_topk_prob=norm, routed_scaling_factor=rsf)


@pytest.mark.parametrize("E,k,H,I,nsh,G,scoring,ng,tg,norm,rsf", CASES)
def test_stages_on_recorded_inputs(E, k, H, I, nsh, G, scoring, ng, tg, norm, rsf):
    moe = DsMoe(E, H, I, G, k, nsh, seed=E + k + G)
    x = torch.randn((1, H), device=_dev(), generator=torch.Generator(device=_dev()).manual_seed(E + G)).half()
    prog = DecodeProgram()
    out = _record(prog, moe, x, scoring, ng, tg, norm, rsf)
    prog.build()
    assert prog.fused and prog.kernel_ops == 2
    prog.run()
    torch.cuda.synchronize()
    _no_abort("deepseek_moe")
    b = prog.moe_buffers(0)
    I_s = moe.I_s
    x64 = _np(x).astype(np.float64)[0]
    gw = _np(moe.gate).astype(np.float64)
    ref = gw @ x64
    lg = b["logits"][0].cpu().numpy()
    assert lg.dtype == np.float32
    # fp32 summation of H products: |err| <= H 2^-24 sum |x w| (+ the final rounding)
    assert (np.abs(lg - ref) <= 2**-24 * np.abs(ref) + H * 2**-24 * (np.abs(gw) @ np.abs(x64)) + 1e-7).all(), "logits"
    ids, w = route_oracle(lg, k, scoring, moe.bias.cpu().numpy(), ng, tg, norm, rsf)
    assert (_np(b["topk_ids"])[0] == ids).all(), "ids"
    kw = b["topk_weights"][0].cpu().numpy()
    assert kw.dtype == np.float32
    assert (np.abs(kw - w) <= 4 * np.spacing(np.abs(w))).all(), ("weights", kw, w)
    gu = _np(b["gate_up"])[0]
    act = _np(b["act"])[0].astype(np.float64)
    for s, e in enumerate(ids):
        W1 = moe.deq(1, int(e)).astype(np.float64)
        _close(gu[s * 2 * I:(s + 1) * 2 * I], x64 @ W1, np.abs(x64) @ np.abs(W1), f"gate|up slot {s}")
        W2 = moe.deq(2, int(e)).astype(np.float64)
        a = act[s * I:(s + 1) * I]
        y64 = a @ W2
        _close(_np(b["down"])[0, s], y64 * np.float64(kw[s]), (np.abs(a) @ np.abs(W2)) * abs(float(kw[s])),
               f"down slot {s}")
    Ws1 = moe.deq_shared(1).astype(np.float64)
    _close(gu[k * 2 * I:], x64 @ Ws1, np.abs(x64) @ np.abs(Ws1), "shared gate|up")
    Ws2 = moe.deq_shared(2).astype(np.float64)
    a_s = act[k * I:]
    _close(_np(b["shared_out"])[0], a_s @ Ws2, np.abs(a_s) @ np.abs(Ws2), "shared down")
    # SiLU*mul, c, combine and + y_s, bit for bit from the recorded tensors
    g = b["gate_up"][0, :k * 2 * I].view(k, 2 * I)
    assert torch.equal((F.silu(g[:, :I]) * g[:, I:]).reshape(-1), b["act"][0, :k * I]), "SiLU*mul"
    gs = b["gate_up"][0, k * 2 * I:]
    assert torch.equal(F.silu(gs[:I_s]) * gs[I_s:], b["act"][0, k * I:]), "shared SiLU*mul"
    acc = torch.zeros(H, dtype=torch.float16, device=_dev())
    for s in np.argsort(ids, kind="stable"):
        acc = acc + b["down"][0, int(s)]
    assert torch.equal(acc + b["shared_out"][0], out[0]), "combine + y_s"


def _hf_block(moe, scoring, ng, tg, norm, rsf):
    """transformers' DeepseekV2Moe (softmax, greedy) / DeepseekV3MoE (sigmoid, noaux_tc) forward restated over
    WQLinear_GEMM experts cut from the stacked tensors (5.5's routing code, its Experts loop and shared MLP)."""
    E, H, I, G = moe.E, moe.H, moe.I, moe.G

    def lin(K, N, q, s, z):
        m = WQLinear_GEMM(4, G, K, N, False, _dev())
        m.qweight.copy_(q)
        m.scales.copy_(s)
        m.qzeros.copy_(z)
        return m

    def mlp(w1, w2, i):
        q1, s1, z1 = w1
        gp = lin(H, i, q1[:, : i // 8], s1[:, :i], z1[:, : i // 8])
        up = lin(H, i, q1[:, i // 8:], s1[:, i:], z1[:, i // 8:])
        dp = lin(i, H, *w2)
        return lambda x: dp(F.silu(gp(x)) * up(x))

    experts = [mlp(tuple(t[e] for t in moe.w1), tuple(t[e] for t in moe.w2), I) for e in range(E)]
    shared = mlp(moe.ws1, moe.ws2, moe.I_s)

    def route(router_logits):
        if scoring == "softmax":
            p = router_logits.softmax(dim=-1, dtype=torch.float32)
            w, idx = torch.topk(p, k=moe.top_k, dim=-1, sorted=False)
            return idx, w * rsf
        s = router_logits.sigmoid()
        c = s + moe.bias
        gsc = c.view(-1, ng, E // ng).topk(2, dim=-1)[0].sum(dim=-1)
        gidx = torch.topk(gsc, k=tg, dim=-1, sorted=False)[1]
        gm = torch.zeros_like(gsc).scatter_(1, gidx, 1)
        sm = gm.unsqueeze(-1).expand(-1, ng, E // ng).reshape(-1, E)
        idx = torch.topk(c.masked_fill(~sm.bool(), 0.0), k=moe.top_k, dim=-1, sorted=False)[1]
        w = s.gather(1, idx)
        if norm:
            w = w / (w.sum(dim=-1, keepdim=True) + 1e-20)
        return idx, w * rsf

    def forward(x):
        logits = F.linear(x.float(), moe.gate.float())
        idx, w = route(logits)
        final = torch.zeros_like(x)
        mask = F.one_hot(idx, num_classes=E).permute(2, 1, 0)
        for e in torch.greater(mask.sum(dim=(-1, -2)), 0).nonzero():
            e = int(e[0])
            pos, tok = torch.where(mask[e])
            y = experts[e](x[tok]) * w[tok, pos, None]
            final.index_add_(0, tok, y.to(final.dtype))
        return final + shared(x), idx

    return forward


def _ulps_of_rms(y, ref, n=4):
    """(largest excess of |y - ref| over one fp16 ulp of ref, n fp16 ulps of rms(ref)): both sides round the block's
    output to fp16 on their own, so one ulp of the element itself comes on top of the n ulps of rms."""
    rf = ref.float()
    rms = float(rf.pow(2).mean().sqrt())
    ulp = torch.from_numpy(np.spacing(np.abs(_np(ref)).astype(np.float16)).astype(np.float32)).to(rf.device)
    return float(((y.float() - rf).abs() - ulp.reshape(rf.shape)).max()), n * rms * 2**-10


@pytest.mark.parametrize("E,k,H,I,nsh,G,scoring,ng,tg,norm,rsf", CASES)
def test_against_hf_block_and_per_op_replay(E, k, H, I, nsh, G, scoring, ng, tg, norm, rsf):
    moe = DsMoe(E, H, I, G, k, nsh, seed=3 * E + k)
    x = torch.randn((1, H), device=_dev(), generator=torch.Generator(device=_dev()).manual_seed(3 * E + G)).half()
    prog = DecodeProgram()
    out = _record(prog, moe, x, scoring, ng, tg, norm, rsf)
    prog.build()
    assert prog.fused
    prog.run()
    torch.cuda.synchronize()
    _no_abort("deepseek_moe vs hf")
    with torch.no_grad():
        ref, sel = _hf_block(moe, scoring, ng, tg, norm, rsf)(x)
    b = prog.moe_buffers(0)
    if set(_np(b["topk_ids"][0]).tolist()) == set(_np(sel[0]).tolist()):
        err, tol = _ulps_of_rms(out, ref)
        assert err <= tol, f"out vs HF block: {err:.3e} > {tol:.3e}"
    ext.set_knob(14, 1)
    try:
        rep = DecodeProgram()
        out_r = _record(rep, moe, x, scoring, ng, tg, norm, rsf)
        rep.build()
    finally:
        ext.set_knob(14, 0)
    assert not rep.fused
    rep.run()
    torch.cuda.synchronize()
    br = rep.moe_buffers(0)
    assert set(_np(br["topk_ids"][0]).tolist()) == set(_np(sel[0]).tolist()), "replay routing vs HF"
    if set(_np(br["topk_ids"][0]).tolist()) == set(_np(b["topk_ids"][0]).tolist()):
        err, tol = _ulps_of_rms(out, out_r)
        assert err <= tol, f"fused vs per-op replay: {err:.3e} > {tol:.3e}"


def test_stack_deepseek_experts_round_trip():
    moe = DsMoe(16, 512, 256, 128, 4, 2, seed=3)

    class NS:
        pass

    def mlp(w1, w2, i):
        m = NS()
        for name, (q, s, z) in (("gate_proj", tuple(t[..., : t.shape[-1] // 2] for t in w1)),
                                ("up_proj", tuple(t[..., t.shape[-1] // 2:] for t in w1)), ("down_proj", w2)):
            p = NS()
            p.qweight, p.scales, p.qzeros = q.contiguous(), s.contiguous(), z.contiguous()
            setattr(m, name, p)
        return m

    blk = NS()
    blk.gate = NS()
    blk.gate.weight, blk.gate.e_score_correction_bias = moe.gate, moe.bias
    blk.experts = [mlp(tuple(t[e] for t in moe.w1), tuple(t[e] for t in moe.w2), moe.I) for e in range(16)]
    blk.shared_experts = mlp(moe.ws1, moe.ws2, moe.I_s)
    blk.top_k, blk.n_group, blk.topk_group, blk.norm_topk_prob, blk.routed_scaling_factor = 4, 4, 2, True, 2.0
    gw, w1, w2, k, shared, routing = packing.stack_deepseek_experts(blk)
    assert torch.equal(gw, moe.gate) and k == 4 and routing["scoring"] == "sigmoid" and routing["n_group"] == 4
    for a, b in zip(w1 + w2 + shared[0] + shared[1], moe.w1 + moe.w2 + moe.ws1 + moe.ws2):
        assert torch.equal(a, b)
    x = torch.randn((1, 512), device=_dev(), generator=torch.Generator(device=_dev()).manual_seed(1)).half()
    p1, p2 = DecodeProgram(), DecodeProgram()
    o1 = p1.deepseek_moe(x, gw, w1, w2, k, shared, **routing)
    o2 = _record(p2, moe, x, "sigmoid", 4, 2, True, 2.0)
    p1.build()
    p2.build()
    p1.run()
    p2.run()
    torch.cuda.synchronize()
    assert p1.fused and torch.equal(o1, o2)


def test_v2_lite_segment_is_one_kernel_and_graph_replay():
    """[o + h, norm2, deepseek_moe + h, norm1', q_proj' | kv_a_proj_with_mqa'] at V2-Lite shapes: one launch, every
    buffer within tolerance of the per-op replay, and a CUDA graph of it following a refilled residual.  q_proj and
    kv_a_proj_with_mqa read the same normed row and are recorded as one linear (N = 16 x 192 + 576), as qkv is."""
    H, G = 2048, 128
    moe = DsMoe(64, H, 1408, G, 6, 2, seed=11)
    gen = torch.Generator(device=_dev()).manual_seed(5)

    def lin(K, N):
        return (torch.randint(-2**31, 2**31 - 1, (K, N // 8), dtype=torch.int32, device=_dev(), generator=gen),
                ((torch.rand((K // G, N), device=_dev(), generator=gen) * 0.5 + 0.75) / (6.1 * K**0.5)).half(),
                torch.randint(-2**31, 2**31 - 1, (K // G, N // 8), dtype=torch.int32, device=_dev(), generator=gen))

    wo, wqkv = lin(16 * 128, H), lin(H, 16 * 192 + 576)
    n1, n2 = [(1 + 0.1 * torch.randn(H, device=_dev(), generator=gen)).half() for _ in range(2)]
    attn = torch.randn((1, 16 * 128), device=_dev(), generator=gen).half()
    h = torch.randn((1, H), device=_dev(), generator=gen).half()

    def build(knob14):
        hm, xn2, h2, xn = (torch.empty((1, H), dtype=torch.float16, device=_dev()) for _ in range(4))
        p = DecodeProgram()
        o = p.gemm_forward_cuda(attn, *wo, 8)
        p.add(o, h, out=hm)
        p.layernorm_forward_cuda(hm, n2, xn2, EPS)
        mo = _record(p, moe, xn2, "softmax", 1, 1, False, 1.0)
        p.add(mo, hm, out=h2)
        p.layernorm_forward_cuda(h2, n1, xn, EPS)
        qkv = p.gemm_forward_cuda(xn, *wqkv, 8)
        ext.set_knob(14, 1 if knob14 else 0)
        try:
            p.build()
        finally:
            ext.set_knob(14, 0)
        return p, dict(o=o, hm=hm, xn2=xn2, moe=mo, h2=h2, xn=xn, qkv=qkv)

    pf, bf = build(False)
    pr, br = build(True)
    assert pf.fused and pf.launches_per_run == 1 and pf.kernel_ops == 4 and not pr.fused
    pf.run()
    pr.run()
    torch.cuda.synchronize()
    _no_abort("deepseek-moe segment")
    same_route = torch.equal(pf.moe_buffers(0)["topk_ids"].sort().values, pr.moe_buffers(0)["topk_ids"].sort().values)
    for name in bf:
        if name in ("moe", "h2", "xn", "qkv") and not same_route:
            continue
        err, tol = _ulps_of_rms(bf[name], br[name], 8)
        assert err <= tol + 1e-3, f"{name}: {err:.3e} > {tol:.3e}"
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        pf.run()
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=s):
            pf.run()
    torch.cuda.current_stream().wait_stream(s)
    for i in range(3):
        h.copy_(torch.randn((1, H), device=_dev(), generator=gen).half())
        g.replay()
        torch.cuda.synchronize()
        kg = bf["qkv"].clone()
        pf.run()
        torch.cuda.synchronize()
        assert torch.equal(kg, bf["qkv"]) and kg.abs().sum() > 0, f"graph replay {i}"
    _no_abort("deepseek-moe segment graph")
