#!/usr/bin/env python
"""DeepSeek-V2-Lite decode step at bs = 1 (seeded random AWQ weights, g128): per-op replay vs one fused program per
segment, both replayed from CUDA graphs.

27 layers: layer 0 is dense (intermediate size 10944), layers 1..26 are DeepSeek-MoE blocks (E = 64, top-6, I = 1408,
two shared experts, I_s = 2816).  Each layer records [o_proj + h, norm2, mlp + h, norm1', q_proj' | kv_a_proj_with_mqa']
as one DecodeProgram; q_proj and kv_a_proj_with_mqa read the same normed row and are one linear (N = 3072 + 576), as
qkv is.  The dense layer's mlp is gate|up, silu, down with G = 64 (10944 is not a multiple of 128, so that layer is
outside the stream format and replays per op in both arms).  The MLA glue between programs (kv_a_layernorm,
kv_b_proj, rotary, attention) is not part of the programs and not part of this step: the numbers are the programs
alone.

Arms: (a) every program built under knob 14 = 1 (per-op replay through ext / torch), (b) fused.  Each arm is one CUDA
graph of the 27 programs; rounds alternate a and b and the medians are reported.  Self-checks: (b) is one launch per
layer, no abort record, and the first MoE layer's block output of (b) is within 8 fp16 ulps of rms of (a)'s when both
routed the same experts (further down the random stack the arms drift apart, as DESIGN 3.5h describes).  --sigmoid switches the MoE blocks to Moonlight's routing (sigmoid with the correction bias, n_group 1,
norm_topk_prob, routed_scaling_factor 2.446).  Prints one JSON line."""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from autoawq_b200 import ext  # noqa: E402
from autoawq_b200.program import DecodeProgram  # noqa: E402

H, G, E, K_TOP, I, I_S, DENSE_I = 2048, 128, 64, 6, 1408, 2816, 10944
NH, QK_HEAD, V_HEAD, KV_A = 16, 192, 128, 576


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=27)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--sigmoid", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)

    def lin(K, N, lead=(), g=G):
        return (torch.randint(-2**31, 2**31 - 1, lead + (K, N // 8), dtype=torch.int32, device=dev, generator=gen),
                ((torch.rand(lead + (K // g, N), device=dev, generator=gen) * 0.5 + 0.75) / (6.1 * K**0.5)).half(),
                torch.randint(-2**31, 2**31 - 1, lead + (K // g, N // 8), dtype=torch.int32, device=dev, generator=gen))

    def norm_w():
        return (1 + 0.1 * torch.randn(H, device=dev, generator=gen)).half()

    routing = dict(scoring="softmax")
    if a.sigmoid:
        routing = dict(scoring="sigmoid", n_group=1, topk_group=1, norm_topk_prob=True, routed_scaling_factor=2.446)
    layers = []
    for li in range(a.layers):
        L = dict(wo=lin(NH * V_HEAD, H), wqkv=lin(H, NH * QK_HEAD + KV_A), n1=norm_w(), n2=norm_w(),
                 attn=torch.randn((1, NH * V_HEAD), device=dev, generator=gen).half())
        if li == 0:
            L.update(gu=lin(H, 2 * DENSE_I, g=64), down=lin(DENSE_I, H, g=64))
        else:
            L.update(gate=(torch.randn((E, H), device=dev, generator=gen) * 0.05).half(), w1=lin(H, 2 * I, (E,)),
                     w2=lin(I, H, (E,)), shared=(lin(H, 2 * I_S), lin(I_S, H)),
                     bias=(torch.randn(E, device=dev, generator=gen) * 0.05).float())
        layers.append(L)
    h0 = torch.randn((1, H), device=dev, generator=gen).half()

    def build(knob14):
        progs, h = [], h0
        outs = []
        for li, L in enumerate(layers):
            hm, xn2, h2, xn = (torch.empty((1, H), dtype=torch.float16, device=dev) for _ in range(4))
            p = DecodeProgram()
            o = p.gemm_forward_cuda(L["attn"], *L["wo"], 8)
            p.add(o, h, out=hm)
            p.layernorm_forward_cuda(hm, L["n2"], xn2, 1e-6)
            if li == 0:
                gu = p.gemm_forward_cuda(xn2, *L["gu"], 8)
                act = torch.empty((1, DENSE_I), dtype=torch.float16, device=dev)
                p.silu_and_mul(act, gu)
                mo = p.gemm_forward_cuda(act, *L["down"], 8)
            else:
                kw = dict(routing)
                if a.sigmoid:
                    kw["e_score_correction_bias"] = L["bias"]
                mo = p.deepseek_moe(xn2, L["gate"], L["w1"], L["w2"], K_TOP, L["shared"], **kw)
            p.add(mo, hm, out=h2)
            p.layernorm_forward_cuda(h2, L["n1"], xn, 1e-6)
            p.gemm_forward_cuda(xn, *L["wqkv"], 8)
            ext.set_knob(14, 1 if knob14 else 0)
            try:
                p.build()
            finally:
                ext.set_knob(14, 0)
            progs.append(p)
            outs.append(mo)
            h = h2
        return progs, outs

    pa, oa = build(True)
    pb, ob = build(False)
    assert all(p.fused and p.launches_per_run == 1 for p in pb[1:]) and not any(p.fused for p in pa)

    def graph(progs):
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        g = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s):
            for p in progs:
                p.run()
            torch.cuda.synchronize()
            with torch.cuda.graph(g, stream=s):
                for p in progs:
                    p.run()
        torch.cuda.current_stream().wait_stream(s)
        return g

    ga, gb = graph(pa), graph(pb)

    def timed(g):
        st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        g.replay()
        st.record()
        for _ in range(a.steps):
            g.replay()
        en.record()
        torch.cuda.synchronize()
        return st.elapsed_time(en) / a.steps

    ta, tb = [], []
    for _ in range(a.rounds):
        ta.append(timed(ga))
        tb.append(timed(gb))
    rec = DecodeProgram.abort_record()
    assert rec[3] == 0, f"abort record {rec}"
    same = torch.equal(pa[1].moe_buffers(0)["topk_ids"].sort().values, pb[1].moe_buffers(0)["topk_ids"].sort().values)
    ref = oa[1].float()
    err = float((ob[1].float() - ref).abs().max())
    tol = 8 * float(ref.pow(2).mean().sqrt()) * 2**-10
    assert not same or err <= tol, f"fused vs per-op: {err:.3e} > {tol:.3e}"
    props = torch.cuda.get_device_properties(dev)
    print(json.dumps(dict(workload=f"DeepSeek-V2-Lite decode bs=1, {a.layers} layers, programs only (no MLA glue), "
                                   f"{routing['scoring']} routing",
                          gpu=props.name, per_op_ms=round(statistics.median(ta), 4),
                          fused_ms=round(statistics.median(tb), 4),
                          speedup=round(statistics.median(ta) / statistics.median(tb), 3),
                          per_op_rounds=[round(t, 4) for t in ta], fused_rounds=[round(t, 4) for t in tb],
                          first_moe_layer_same_experts=same, first_moe_layer_max_abs_diff=err, self_checks="pass")))


if __name__ == "__main__":
    main()
