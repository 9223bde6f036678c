"""Qwen3-MoE expert blocks in M = 1 stream decode programs (DecodeProgram.qwen3_moe, B200AWQ_OP_QWEN3_MOE): the router
logits exchanged across the grid, the routing and Qwen3MoeSparseMoeBlock's finishes in stream_qwen3moe_kernel.

Per stage, on the program's own recorded inputs: the logits against the fp64 router matmul, the ids and fp16 weights
exactly against the routing oracle applied to the recorded logits, gate|up and down against the fp64 experts, the
SiLU*mul and the combine bit for bit from the recorded gate_up / down.  Then the fused block against its per-op replay
(knob 14 = 1) and against transformers' Qwen3MoeSparseMoeBlock restated over WQLinear_GEMM, a whole attention-to-
attention segment as one kernel (also replayed in a CUDA graph with a moving position), and the per-op fallbacks."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from autoawq_b200 import ext, packing
from autoawq_b200.linear import WQLinear_GEMM
from autoawq_b200.program import DecodeProgram
from test_gpu_program import _close, _no_abort
from test_gpu_program_moe import Moe, _np

pytestmark = pytest.mark.gpu

EPS = 1e-6
CASES = [(128, 8, 2048, 768, 128), (96, 8, 2048, 768, 128), (64, 4, 1024, 512, 128), (64, 4, 1024, 512, 64)]


def _dev():
    return torch.device("cuda:0")


def _routing_oracle(logits, topk, renorm):
    """topk_softmax's arithmetic on the recorded fp16 logits (lane l sums experts l + 32 i in order, then the xor tree),
    the fp32 renormalisation over the slots in slot order and the fp16 cast: (ids, fp16 weights)."""
    E = logits.numel()
    lg = logits.float()
    mx = lg.max()
    p = torch.exp(lg - mx).cpu().numpy().astype(np.float32)     # expf on the device, as the kernel
    lanes = np.zeros(32, dtype=np.float32)
    for lane in range(32):
        for e in range(lane, E, 32):
            lanes[lane] = np.float32(lanes[lane] + p[e])
    for off in (16, 8, 4, 2, 1):
        lanes = np.array([np.float32(lanes[l] + lanes[l ^ off]) for l in range(32)], dtype=np.float32)
    inv = np.float32(1.0) / lanes[0]
    q = p.copy()
    ids, w = [], []
    for _ in range(topk):
        b = int(np.argmax(q))                  # first maximum: ties to the lower expert
        ids.append(b)
        w.append(np.float32(q[b] * inv))
        q[b] = -2.0
    w = np.array(w, dtype=np.float32)
    if renorm:
        s = np.float32(0.0)
        for v in w:
            s = np.float32(s + v)
        w = (w / s).astype(np.float32)
    return np.array(ids), w.astype(np.float16)


def _record(prog, moe, x, renorm=True):
    return prog.qwen3_moe(x, moe.gate, moe.w1, moe.w2, moe.top_k, renorm)


@pytest.mark.parametrize("E,k,H,I,G", CASES)
def test_stages_on_recorded_inputs(E, k, H, I, G):
    moe = Moe(E, H, I, G, k, seed=E + k + G)
    x = torch.randn((1, H), device=_dev()).half()
    prog = DecodeProgram()
    out = _record(prog, moe, x)
    prog.build()
    assert prog.fused and prog.kernel_ops == 2
    prog.run()
    torch.cuda.synchronize()
    _no_abort("qwen3_moe")
    b = prog.moe_buffers(0)
    x64 = _np(x).astype(np.float64)[0]
    gw = _np(moe.gate).astype(np.float64)
    ref = gw @ x64
    lg = _np(b["logits"])[0].astype(np.float64)
    assert (np.abs(lg - ref) <= 2**-10 * np.abs(ref) + 1e-5 * (np.abs(gw) @ np.abs(x64)) + 1e-6).all(), "logits"
    ids, w16 = _routing_oracle(b["logits"][0], k, True)
    assert (_np(b["topk_ids"])[0] == ids).all(), "ids"
    assert (_np(b["topk_weights"])[0].view(np.uint16) == w16.view(np.uint16)).all(), "fp16 weights"
    gu = _np(b["gate_up"])[0]
    act = _np(b["act"])[0].astype(np.float64)
    for s, e in enumerate(ids):
        W1 = moe.deq(1, int(e)).astype(np.float64)
        _close(gu[s], x64 @ W1, np.abs(x64) @ np.abs(W1), f"gate|up slot {s}")
        W2 = moe.deq(2, int(e)).astype(np.float64)
        y64 = act[s] @ W2
        c64 = y64 * np.float64(w16[s])
        _close(_np(b["down"])[0, s], c64, (np.abs(act[s]) @ np.abs(W2)) * abs(float(w16[s])), f"down slot {s}")
    # SiLU*mul and combine, bit for bit from the recorded tensors
    g, u = b["gate_up"][0, :, :I], b["gate_up"][0, :, I:]
    assert torch.equal(F.silu(g) * u, b["act"][0]), "SiLU*mul"
    acc = torch.zeros(H, dtype=torch.float16, device=_dev())
    for s in np.argsort(ids, kind="stable"):
        acc = acc + b["down"][0, int(s)]
    assert torch.equal(acc, out[0]), "combine"


def _hf_block(moe, renorm=True):
    """transformers' Qwen3MoeSparseMoeBlock (4.5x) over WQLinear_GEMM experts cut from the stacked tensors."""
    E, H, I, G = moe.E, moe.H, moe.I, moe.G

    def lin(K, N, q, s, z):
        m = WQLinear_GEMM(4, G, K, N, False, _dev())
        m.qweight.copy_(q)
        m.scales.copy_(s)
        m.qzeros.copy_(z)
        return m

    class Expert(torch.nn.Module):
        def __init__(self, e):
            super().__init__()
            q1, s1, z1 = (t[e] for t in moe.w1)
            self.gate_proj = lin(H, I, q1[:, : I // 8], s1[:, :I], z1[:, : I // 8])
            self.up_proj = lin(H, I, q1[:, I // 8:], s1[:, I:], z1[:, I // 8:])
            self.down_proj = lin(I, H, *(t[e] for t in moe.w2))

        def forward(self, x):
            return self.down_proj(F.silu(self.gate_proj(x)) * self.up_proj(x))

    class Block(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.num_experts, self.top_k, self.norm_topk_prob = E, moe.top_k, renorm
            self.gate = torch.nn.Linear(H, E, bias=False, device=_dev(), dtype=torch.float16)
            self.gate.weight.data.copy_(moe.gate)
            self.experts = torch.nn.ModuleList([Expert(e) for e in range(E)])

        def forward(self, hidden_states):
            router_logits = self.gate(hidden_states)
            routing_weights = F.softmax(router_logits, dim=1, dtype=torch.float)
            routing_weights, selected_experts = torch.topk(routing_weights, self.top_k, dim=-1)
            if self.norm_topk_prob:
                routing_weights /= routing_weights.sum(dim=-1, keepdim=True)
            routing_weights = routing_weights.to(hidden_states.dtype)
            final = torch.zeros_like(hidden_states)
            mask = F.one_hot(selected_experts, num_classes=self.num_experts).permute(2, 1, 0)
            for e in range(self.num_experts):
                idx, top_x = torch.where(mask[e])
                if top_x.numel() == 0:
                    continue
                cur = hidden_states[top_x]
                y = self.experts[e](cur) * routing_weights[top_x, idx, None]
                final.index_add_(0, top_x, y.to(hidden_states.dtype))
            return final, routing_weights, selected_experts, F.softmax(router_logits, dim=1, dtype=torch.float)

    with torch.no_grad():
        return Block()


def _ulps_of_rms(y, ref, n=4):
    rms = float(ref.float().pow(2).mean().sqrt())
    return float((y.float() - ref.float()).abs().max()), n * rms * 2**-10


def test_stack_experts_round_trip():
    moe = Moe(16, 512, 256, 128, 4, seed=3)
    gw, w1, w2, k, norm = packing.stack_experts(_hf_block(moe))
    assert torch.equal(gw, moe.gate) and k == 4 and norm
    for a, b in zip(w1 + w2, moe.w1 + moe.w2):
        assert torch.equal(a, b)


@pytest.mark.parametrize("E,k,H,I,G,M", [(128, 8, 2048, 768, 128, 1), (64, 4, 1024, 512, 64, 1),
                                         (128, 8, 2048, 768, 128, 2), (129, 8, 1024, 512, 128, 1)])
def test_against_hf_block_and_per_op_replay(E, k, H, I, G, M):
    """Fused (M = 1, E <= 128) or per-op (M = 2, E = 129) against the HF restatement; the fused block also against its
    knob-14 replay."""
    moe = Moe(E, H, I, G, k, seed=7 * E + M)
    x = torch.randn((M, H), device=_dev()).half()
    prog = DecodeProgram()
    out = _record(prog, moe, x)
    prog.build()
    assert prog.fused == (M == 1 and E <= 128)
    prog.run()
    torch.cuda.synchronize()
    if prog.fused:
        _no_abort("qwen3_moe vs hf")
    blk = _hf_block(moe)
    with torch.no_grad():
        ref, rw, sel, probs = blk(x)
    b = prog.moe_buffers(0)
    for m in range(M):
        p = probs[m].sort(descending=True).values
        if float(p[k - 1]) != float(p[k]):          # no tie at the cut: the same expert set
            assert set(_np(b["topk_ids"][m]).tolist()) == set(_np(sel[m]).tolist())
    err, tol = _ulps_of_rms(out, ref)
    assert err <= tol, f"out vs HF block: {err:.3e} > {tol:.3e}"
    if prog.fused:
        ext.set_knob(14, 1)
        try:
            rep = DecodeProgram()
            out_r = _record(rep, moe, x)
            rep.build()
        finally:
            ext.set_knob(14, 0)
        assert not rep.fused
        rep.run()
        torch.cuda.synchronize()
        br = rep.moe_buffers(0)
        if torch.equal(br["topk_ids"], b["topk_ids"]):
            err, tol = _ulps_of_rms(out, out_r)
            assert err <= tol, f"fused vs per-op replay: {err:.3e} > {tol:.3e}"
            assert (b["topk_weights"].float() - br["topk_weights"].float()).abs().max() <= 2**-10


def _freqs(D, S, theta):
    inv = 1.0 / (theta ** (torch.arange(0, D, 2, device=_dev()).float() / D))
    return torch.polar(torch.ones(S, D // 2, device=_dev()), torch.outer(torch.arange(S, device=_dev()).float(), inv))


def test_segment_is_one_kernel_and_graph_replay():
    """30B-A3B segment [o + h, norm2, qwen3_moe + hm, norm1', qkv', qk-norm-rope] at M = 1: one launch, every buffer
    within tolerance of the per-op replay, and a CUDA graph of it following a moving position."""
    from transformers.models.qwen3.modeling_qwen3 import Qwen3RMSNorm

    H, NH, KV, D, S, G = 2048, 32, 4, 128, 64, 128
    moe = Moe(128, H, 768, G, 8, seed=11)
    gen = torch.Generator(device=_dev()).manual_seed(5)

    def lin(K, N):
        return (torch.randint(-2**31, 2**31 - 1, (K, N // 8), dtype=torch.int32, device=_dev(), generator=gen),
                ((torch.rand((K // G, N), device=_dev(), generator=gen) * 0.5 + 0.75) / (6.1 * K**0.5)).half(),
                torch.randint(-2**31, 2**31 - 1, (K // G, N // 8), dtype=torch.int32, device=_dev(), generator=gen))

    wo, wqkv = lin(NH * D, H), lin(H, (NH + 2 * KV) * D)
    n1, n2 = [(1 + 0.1 * torch.randn(H, device=_dev(), generator=gen)).half() for _ in range(2)]
    qk = []
    for _ in range(2):
        n = Qwen3RMSNorm(D, eps=EPS).to(_dev()).half()
        with torch.no_grad():
            n.weight.copy_((1 + 0.2 * torch.randn(D, device=_dev(), generator=gen)).half())
        qk.append(n)
    freqs = _freqs(D, S, 1e6)
    attn = torch.randn((1, NH * D), device=_dev(), generator=gen).half()
    h = torch.randn((1, H), device=_dev(), generator=gen).half()

    def build(knob14):
        pos = torch.tensor([3], dtype=torch.int32, device=_dev())
        kc, vc = (torch.zeros((1, S, KV, D), dtype=torch.float16, device=_dev()) for _ in range(2))
        hm, xn2, h2, xn = (torch.empty((1, H), dtype=torch.float16, device=_dev()) for _ in range(4))
        p = DecodeProgram()
        o = p.gemm_forward_cuda(attn, *wo, 8)
        p.add(o, h, out=hm)
        p.layernorm_forward_cuda(hm, n2, xn2, EPS)
        mo = _record(p, moe, xn2)
        p.add(mo, hm, out=h2)
        p.layernorm_forward_cuda(h2, n1, xn, EPS)
        qkv = p.gemm_forward_cuda(xn, *wqkv, 8)
        q = p.rope_kv_cache(qkv, freqs, pos, kc, vc, NH, KV, q_norm=qk[0], k_norm=qk[1])
        ext.set_knob(14, 1 if knob14 else 0)
        try:
            p.build()
        finally:
            ext.set_knob(14, 0)
        return p, dict(o=o, hm=hm, xn2=xn2, moe=mo, h2=h2, xn=xn, qkv=qkv, q=q, k=kc, v=vc), pos

    pf, bf, posf = build(False)
    pr, br, posr = build(True)
    assert pf.fused and pf.launches_per_run == 1 and pf.kernel_ops == 4 and not pr.fused
    pf.run()
    pr.run()
    torch.cuda.synchronize()
    _no_abort("qwen3-moe segment")
    same_route = torch.equal(pf.moe_buffers(0)["topk_ids"], pr.moe_buffers(0)["topk_ids"])
    for name in bf:
        if name in ("moe", "h2", "xn", "qkv", "q", "k", "v") and not same_route:
            continue
        err, tol = _ulps_of_rms(bf[name], br[name], 8)
        assert err <= tol + 1e-3, f"{name}: {err:.3e} > {tol:.3e}"
    # CUDA graph with a moving position: the replayed kernel writes each new cache row as an eager run does
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        pf.run()
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=s):
            pf.run()
    torch.cuda.current_stream().wait_stream(s)
    for p in (4, 5, 6):
        posf.fill_(p)
        g.replay()
        torch.cuda.synchronize()
        kg = bf["k"][0, p].clone()
        bf["k"][0, p].zero_()
        pf.run()
        torch.cuda.synchronize()
        assert torch.equal(kg, bf["k"][0, p]) and kg.abs().sum() > 0, f"graph replay at position {p}"
    _no_abort("qwen3-moe segment graph")
