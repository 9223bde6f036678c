"""Sparse-MoE blocks in M = 1 stream decode programs (DecodeProgram.sparse_moe, B200AWQ_OP_SPARSE_MOE): the routing
prologue and the two expert ops of stream_moe_kernel.  Every tensor the block leaves behind is
checked against the fp64 oracle (oracle/awq_oracle.py) on the program's OWN recorded inputs: the logits against the
router matmul of the recorded normed row, the routing (topk_softmax, renormalisation, moe_align_block_size) against the
oracle applied to the recorded logits, and every expert stage against the dequantised experts the routing selected.
The fused result is also compared with the per-op replay of the same recording."""
import numpy as np
import pytest
import torch

from oracle import awq_oracle as O
from test_gpu_program import _close, _no_abort

pytestmark = pytest.mark.gpu

EPS = 1e-5
BLOCK = 16


def _dev():
    return torch.device("cuda:0")


def _np(t):
    return t.detach().cpu().numpy()


class Moe:
    """One sparse-MoE block with random AWQ-packed stacked experts (the bench's scale recipe keeps O(1) activations)."""

    def __init__(self, E, H, I, G, top_k, seed):
        self.E, self.H, self.I, self.G, self.top_k = E, H, I, G, top_k
        g = torch.Generator(device=_dev()).manual_seed(seed)

        def stacked(K, N):
            return (torch.randint(-2**31, 2**31 - 1, (E, K, N // 8), dtype=torch.int32, device=_dev(), generator=g),
                    ((torch.rand((E, K // G, N), device=_dev(), generator=g) * 0.5 + 0.75) / (6.1 * K**0.5)).half(),
                    torch.randint(-2**31, 2**31 - 1, (E, K // G, N // 8), dtype=torch.int32, device=_dev(), generator=g))

        self.w1, self.w2 = stacked(H, 2 * I), stacked(I, H)
        self.gate = (torch.randn((E, H), device=_dev(), generator=g) * 0.05).half().contiguous()
        self.norm = (1 + 0.1 * torch.randn(H, device=_dev(), generator=g)).half()
        self._deq = {}

    def deq(self, which, e):
        """Expert e's dequantised weight [K, N] fp16 from the oracle (cached)."""
        key = (which, e)
        if key not in self._deq:
            q, s, z = (_np(t[e]) for t in (self.w1 if which == 1 else self.w2))
            self._deq[key] = O.dequantize_gemm(q, z, s, self.G)
        return self._deq[key]


def _record(prog, moe, h, renormalize=True):
    xn = torch.empty_like(h)
    prog.layernorm_forward_cuda(h, moe.norm, xn, EPS)
    out = prog.sparse_moe(xn, moe.gate, moe.w1, moe.w2, moe.top_k, renormalize)
    return xn, out


def _check_block(moe, xn, bufs, renormalize, tag):
    """Every tensor of one block against the oracle on its own recorded inputs (M = 1)."""
    E, k = moe.E, moe.top_k
    x = _np(xn).astype(np.float16)
    # logits: fp32 dots rounded to fp16 -> within fp16 rounding of the fp64 router matmul
    lg = _np(bufs["logits"]).astype(np.float64)
    ref = x.astype(np.float64) @ _np(moe.gate).astype(np.float64).T
    budget = np.abs(x.astype(np.float64)) @ np.abs(_np(moe.gate).astype(np.float64)).T
    assert np.all(np.abs(lg - ref) <= 2.0**-11 * np.abs(ref) + 1e-6 * budget + 1e-6), f"{tag}: logits"
    # routing: the oracle's topk_softmax of the RECORDED logits, exactly; weights within 2e-6
    w_ref, ids_ref, src_ref = O.topk_softmax(lg.astype(np.float32), k)
    if renormalize:
        w_ref = (w_ref.astype(np.float64) / w_ref.astype(np.float64).sum(axis=1, keepdims=True)).astype(np.float32)
    ids = _np(bufs["topk_ids"])
    assert np.array_equal(ids, ids_ref), f"{tag}: topk_ids {ids} vs {ids_ref}"
    np.testing.assert_allclose(_np(bufs["topk_weights"]), w_ref, rtol=0, atol=2e-6, err_msg=f"{tag}: topk_weights")
    assert np.array_equal(_np(bufs["token_expert_indices"]), src_ref), f"{tag}: token_expert_indices"
    s_ref, e_ref, n_ref = O.moe_align_block_size(ids, BLOCK, E)
    assert int(_np(bufs["num_tokens_post_pad"])[0]) == n_ref, f"{tag}: num_tokens_post_pad"
    assert np.array_equal(_np(bufs["sorted_ids"]), s_ref), f"{tag}: sorted_ids"
    assert np.array_equal(_np(bufs["expert_ids"])[: n_ref // BLOCK], e_ref[: n_ref // BLOCK]), f"{tag}: expert_ids"
    # experts, slot by slot, each stage on its recorded input
    gu, act, dn = (_np(bufs[n])[0] for n in ("gate_up", "act", "down"))
    tw = _np(bufs["topk_weights"])[0].astype(np.float64)
    out_ref = np.zeros(moe.H)
    for s in range(k):
        e = int(ids[0, s])
        w1, w2 = moe.deq(1, e), moe.deq(2, e)
        _close(gu[s], O.gemm_f64(x[None], w1)[0], (np.abs(x.astype(np.float64)) @ np.abs(w1.astype(np.float64))),
               f"{tag}: gate_up slot {s}")
        g64, u64 = gu[s, : moe.I].astype(np.float64), gu[s, moe.I:].astype(np.float64)
        np.testing.assert_allclose(act[s], g64 / (1 + np.exp(-g64)) * u64, rtol=2e-3, atol=2e-3, err_msg=f"{tag}: silu {s}")
        a = act[s].astype(np.float16)
        y64 = O.gemm_f64(a[None], w2)[0]
        _close(dn[s].astype(np.float64) / tw[s], y64, np.abs(a.astype(np.float64)) @ np.abs(w2.astype(np.float64)),
               f"{tag}: down slot {s}")
        out_ref += tw[s] * y64
    # out = fp16(sum over slots of the fp16 per-slot outputs), and close to the fp64 block output
    out = _np(bufs["out"])[0].astype(np.float64)
    summed = dn.astype(np.float32).sum(axis=0).astype(np.float16).astype(np.float64)
    assert np.array_equal(out, summed) or np.abs(out - summed).max() <= 2.0**-10 * np.abs(summed).max(), f"{tag}: sum"
    rms = np.sqrt((out_ref**2).mean())
    assert np.abs(out - out_ref).max() <= 0.02 * rms + 2e-3, f"{tag}: out vs oracle, max {np.abs(out - out_ref).max()}"


def _build(moe, h, renormalize=True, kind_knob=None, max_tokens=1):
    from autoawq_b200 import ext
    from autoawq_b200.program import DecodeProgram

    prev = ext.get_knob(14)
    if kind_knob is not None:
        ext.set_knob(14, kind_knob)
    try:
        prog = DecodeProgram(max_tokens=max_tokens)
        xn, out = _record(prog, moe, h, renormalize)
        prog.build()
    finally:
        ext.set_knob(14, prev)
    return prog, xn, out


def _h(H, seed, M=1):
    return torch.from_numpy(np.random.default_rng(seed).standard_normal((M, H)).astype(np.float16)).to(_dev())


CASES = [  # E, H, I, G, top_k
    pytest.param((8, 4096, 14336, 128, 2), id="mixtral"),
    pytest.param((4, 1024, 512, 128, 1), id="E4-top1"),
    pytest.param((64, 512, 256, 128, 6), id="E64-top6"),
    pytest.param((8, 1024, 768, 64, 2), id="E8-top2-g64"),
]


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("renormalize", [True, False])
def test_moe_program_matches_oracle_and_per_op(case, renormalize):
    E, H, I, G, k = case
    if case[0] == 8 and H == 4096 and not renormalize:
        pytest.skip("Mixtral shapes: renormalize=False is covered at the small shapes")
    moe = Moe(E, H, I, G, k, seed=E + k)
    h = _h(H, seed=1)
    prog, xn, out = _build(moe, h, renormalize)
    assert prog.fused and prog.kind == "stream" and prog.kernel_ops == 2
    prog.run()
    torch.cuda.synchronize()
    _no_abort("moe")
    bufs = prog.moe_buffers(0)
    _check_block(moe, xn, bufs, renormalize, f"fused {case}")
    fused = {n: t.clone() for n, t in bufs.items()}
    # the per-op replay of the same recording (knob 14 = 1: do not fuse)
    ref, xn_r, out_r = _build(moe, h, renormalize, kind_knob=1)
    assert not ref.fused and ref.kernel_ops == 0
    ref.run()
    torch.cuda.synchronize()
    rb = ref.moe_buffers(0)
    _check_block(moe, xn_r, rb, renormalize, f"per-op {case}")
    assert torch.equal(xn_r, xn)
    assert torch.equal(rb["topk_ids"], fused["topk_ids"])
    np.testing.assert_allclose(_np(rb["topk_weights"]), _np(fused["topk_weights"]), rtol=0, atol=2e-6)
    rms = float(rb["out"].float().pow(2).mean().sqrt())
    assert float((rb["out"].float() - fused["out"].float()).abs().max()) <= 0.02 * rms + 2e-3


def test_moe_routing_changes_between_runs_and_is_reproducible():
    """Refill the input so that other experts win: a producer that kept stale expert addresses would stream the old
    experts.  Repeated runs are bit-identical, and a CUDA graph of run() replays the same result."""
    moe = Moe(8, 1024, 512, 128, 2, seed=5)
    h = _h(1024, seed=2)
    prog, xn, out = _build(moe, h)
    assert prog.fused
    prog.run()
    torch.cuda.synchronize()
    bufs = prog.moe_buffers(0)
    first = {n: t.clone() for n, t in bufs.items()}
    seen = {tuple(_np(bufs["topk_ids"])[0])}
    for seed in range(3, 12):
        h.copy_(_h(1024, seed=seed))
        prog.run()
        torch.cuda.synchronize()
        _no_abort("refill")
        _check_block(moe, xn, bufs, True, f"refill {seed}")
        seen.add(tuple(_np(bufs["topk_ids"])[0]))
    assert len(seen) > 1, "the refills never changed the routing"
    h.copy_(_h(1024, seed=2))
    prog.run()
    torch.cuda.synchronize()
    for n, t in bufs.items():
        if n != "expert_ids":
            assert torch.equal(t, first[n]), f"run not bit-reproducible: {n}"
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        prog.run()
    torch.cuda.current_stream().wait_stream(s)
    with torch.cuda.graph(g):
        prog.run()
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, first["out"]) and torch.equal(bufs["topk_ids"], first["topk_ids"])


def test_moe_mixtral_chain_each_layer_consistent_with_its_inputs():
    """4 Mixtral-shaped layers of rmsnorm -> qkv -> o -> rmsnorm -> MoE: every layer's routing and output must be
    consistent with its own recorded inputs (the check of the bench's Mixtral leg, in torch on our dequantised
    experts)."""
    from autoawq_b200 import ext
    from autoawq_b200.program import DecodeProgram

    H, I, E, k, QKV, G = 4096, 14336, 8, 2, 6144, 128
    gen = torch.Generator(device=_dev()).manual_seed(77)

    def lin(K, N):
        return (torch.randint(-2**31, 2**31 - 1, (K, N // 8), dtype=torch.int32, device=_dev(), generator=gen),
                ((torch.rand((K // G, N), device=_dev(), generator=gen) * 0.5 + 0.75) / (6.1 * K**0.5)).half(),
                torch.randint(-2**31, 2**31 - 1, (K // G, N // 8), dtype=torch.int32, device=_dev(), generator=gen))

    layers = []
    for li in range(4):
        layers.append(dict(qkv=lin(H, QKV), o=lin(H, H), moe=Moe(E, H, I, G, k, seed=100 + li)))
    prog = DecodeProgram()
    h = _h(H, seed=3)
    x0 = h
    rec = []
    for L in layers:
        xn = torch.empty((1, H), dtype=torch.float16, device=_dev())
        prog.layernorm_forward_cuda(x0, L["moe"].norm, xn, EPS)
        qkv = prog.gemm_forward_cuda(xn, *L["qkv"], 8)
        a = prog.gemm_forward_cuda(qkv[:, :H], *L["o"], 8)
        xn2 = torch.empty((1, H), dtype=torch.float16, device=_dev())
        prog.layernorm_forward_cuda(a, L["moe"].norm, xn2, EPS)
        x0 = prog.sparse_moe(xn2, L["moe"].gate, L["moe"].w1, L["moe"].w2, k)
        rec.append(xn2)
    prog.build()
    assert prog.fused and prog.kernel_ops == 4 * 4
    prog.run()
    torch.cuda.synchronize()
    _no_abort("chain")
    for li, (L, xn2) in enumerate(zip(layers, rec)):
        b = prog.moe_buffers(li)
        m = L["moe"]
        logits = torch.matmul(xn2.float(), m.gate.float().t())
        probs = torch.softmax(logits, dim=-1)
        want = sorted(torch.topk(probs, k, dim=-1).indices.flatten().tolist())
        got = [int(v) for v in b["topk_ids"].flatten().tolist()]
        assert sorted(got) == want, f"L{li}: routed {got}, logits say {want}"
        ref = torch.zeros((1, H), dtype=torch.float32, device=_dev())
        for s, e in enumerate(got):
            w1 = ext.dequantize_weights_cuda(m.w1[0][e], m.w1[1][e], m.w1[2][e], 0, 0, 0, False)
            w2 = ext.dequantize_weights_cuda(m.w2[0][e], m.w2[1][e], m.w2[2][e], 0, 0, 0, False)
            gu = torch.matmul(xn2.float(), w1.float())
            act = (torch.nn.functional.silu(gu[:, :I]) * gu[:, I:]).half().float()
            ref += b["topk_weights"][0, s] * torch.matmul(act, w2.float()).half().float()
        out = b["out"].float()
        rms = float(ref.pow(2).mean().sqrt())
        assert bool(torch.isfinite(out).all()) and float((out - ref).abs().max()) <= 0.03 * rms + 0.02, f"L{li} output"


@pytest.mark.parametrize("what", ["M2", "knob14", "past-lmax"])
def test_moe_envelope_falls_back_to_per_op(what):
    """Outside the fused envelope the recording replays per op - with correct results."""
    if what == "past-lmax":      # top_k x 2I / 16 = 4352 gate|up sets: 33 per CTA on 132 SMs > 32
        moe = Moe(8, 256, 4352, 128, 8, seed=9)
    else:
        moe = Moe(8, 1024, 512, 128, 2, seed=9)
    M = 2 if what == "M2" else 1
    h = _h(moe.H, seed=4, M=M)
    prog, xn, out = _build(moe, h, kind_knob=1 if what == "knob14" else None, max_tokens=M)
    if what == "past-lmax":
        import ctypes

        from autoawq_b200._cabi import lib

        plan = (ctypes.c_int * 8)()
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        assert lib.b200awq_moe_plan(8, 8, 256, 4352, 128, sms, plan) == (2 if sms <= 132 else 0)
        if sms > 132:
            pytest.skip("more SMs than the H100 SXM: the shape fits")
    assert not prog.fused and prog.kind == "per-op"
    prog.run()
    torch.cuda.synchronize()
    bufs = prog.moe_buffers(0)
    if M == 1:
        _check_block(moe, xn, bufs, True, f"per-op {what}")
        return
    # M = 2: each token against the oracle block on its own row (routing per token, no renormalisation differences)
    ids = _np(bufs["topk_ids"])
    w_ref, ids_ref, _ = O.topk_softmax(_np(bufs["logits"]).astype(np.float32), moe.top_k)
    assert np.array_equal(ids, ids_ref)
    for m in range(M):
        x = _np(xn)[m].astype(np.float16)
        tw = _np(bufs["topk_weights"])[m].astype(np.float64)
        ref = sum(tw[s] * O.gemm_f64(
            (lambda g: (g[: moe.I] / (1 + np.exp(-g[: moe.I])) * g[moe.I:]).astype(np.float16))(
                O.gemm_f64(x[None], moe.deq(1, int(ids[m, s])))[0])[None], moe.deq(2, int(ids[m, s])))[0]
            for s in range(moe.top_k))
        out_m = _np(bufs["out"])[m].astype(np.float64)
        rms = np.sqrt((ref**2).mean())
        assert np.abs(out_m - ref).max() <= 0.02 * rms + 2e-3, f"M2 token {m}"
