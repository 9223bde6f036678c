#!/usr/bin/env python
"""Decode steps of depth-scaled residual models, three ways: one JSON line.

  granite-8b: Granite-3.1-8B-shaped (40 layers, hidden 4096, 32 q / 8 kv heads of 128, intermediate 12800,
      residual_multiplier 0.22, RMSNorm eps 1e-5).  Segment: h = x + o(attn) * a; hn = norm2(h); act = silu(gate) up
      of gate|up(hn); x' = h + down(act) * a; xn' = norm1(x'); qkv'; rope_kv_cache.
  minicpm3-4b: MiniCPM3-4B-shaped (62 layers, hidden 2560, 40 heads, q_lora 768, kv_lora 256, nope 64, rope 32, v 64,
      intermediate 6400, a = 1.4 / sqrt(62)).  The same MLP and scaled adds, then the q-LoRA MLA chain (q_a|kv_a,
      mla_k_rope, q_a_layernorm, q_b, mla_q_rope, kv_a_layernorm, kv_b, mla_kv_cache).
  The geometries are test shapes recalled from the public configs, not read from a checkpoint.

  (a) every segment recorded as in (c) but replayed per op (knob 14 = 1), the whole step in one CUDA graph;
  (b) programs split at each scaled add, with torch's `h = x + y * a` (torch.mul, torch.add) between them: what a
      caller can do without DecodeProgram.scaled_add;
  (c) one program per segment, the scaled adds folded into the finish of o and down (DESIGN.md 3.5p).

g128 seeded random AWQ-packed weights (bench.py's scale recipe).  The attention is a stand-in,
F.scaled_dot_product_attention on torch's math backend over the cache rows 0 .. P, outside every program.  Each variant
is one CUDA graph; the graphs are replayed alternately (rounds x steps after warm-up) and the median round is reported
in ms per step.  A program the stream kernels cannot run replays per op (listed under programs_replayed_per_op).  Card,
power limit and SM clock are read in the same run.

Self-checks: (c)'s last scaled add bit-exact against torch's `h + down * a` on (c)'s own buffers; (c)'s and (b)'s step
outputs within tolerance of (a)'s.

    python tools/scaled_residual_decode_bench.py [--steps 10] [--warmup 3] [--rounds 5] [--pos 1023] [--models ...]
"""
import argparse
import gc
import json
import math
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (graph capture, timing and the clock sampler of the bench)
from tools.batched_decode_bench import _power_limit_w  # noqa: E402

CACHE, GROUP = 2048, 128
MODELS = {
    "granite-8b": dict(layers=40, hid=4096, nh=32, kv=8, d=128, inter=12800, alpha=0.22, eps=1e-5, theta=1e7),
    "minicpm3-4b": dict(layers=62, hid=2560, nh=40, cq=768, c=256, dn=64, dr=32, dv=64, inter=6400,
                        alpha=1.4 / math.sqrt(62), eps=1e-5, theta=1e4),
}


def run_model(name, a):
    import torch
    import torch.nn.functional as F
    from torch.nn.attention import SDPBackend, sdpa_kernel

    from autoawq_b200 import ext
    from autoawq_b200.program import DecodeProgram

    m = MODELS[name]
    mla = "cq" in m
    L, HID, NH, INTER, EPS, AL = m["layers"], m["hid"], m["nh"], m["inter"], m["eps"], m["alpha"]
    dev = torch.device("cuda", 0)
    f16 = torch.float16
    g = torch.Generator(device=dev).manual_seed(0)
    wbytes = 0
    P = a.pos

    def linear(K, N):
        nonlocal wbytes
        qw = torch.randint(-2**31, 2**31 - 1, (K, N // 8), dtype=torch.int32, device=dev, generator=g)
        qz = torch.randint(-2**31, 2**31 - 1, (K // GROUP, N // 8), dtype=torch.int32, device=dev, generator=g)
        s = ((torch.rand((K // GROUP, N), device=dev, generator=g) * 0.5 + 0.75) / (6.1 * K**0.5)).half()
        wbytes += qw.numel() * 4 + qz.numel() * 4 + s.numel() * 2
        return qw, s, qz

    def norm(n):
        return (1 + 0.1 * torch.randn(n, generator=g, device=dev)).half()

    if mla:
        CQ, C, DN, DR, DV = m["cq"], m["c"], m["dn"], m["dr"], m["dv"]
        W = DN + DR
        QD = NH * DV
        w = [dict(o=linear(QD, HID), gu=linear(HID, 2 * INTER), down=linear(INTER, HID), qa=linear(HID, CQ + C + DR),
                  qb=linear(CQ, NH * W), kvb=linear(C, NH * (DN + DV)), n1=norm(HID), n2=norm(HID), nq=norm(CQ),
                  nkv=norm(C)) for _ in range(L)]
        inv = 1.0 / (m["theta"] ** (torch.arange(0, DR, 2, device=dev).float() / DR))
        freqs = torch.polar(torch.ones((CACHE, DR // 2), device=dev), torch.outer(torch.arange(CACHE, device=dev).float(), inv))
        k0 = [torch.randn((1, CACHE, NH, W), generator=g, device=dev, dtype=f16) for _ in range(L)]
        v0 = [torch.randn((1, CACHE, NH, DV), generator=g, device=dev, dtype=f16) for _ in range(L)]
    else:
        KV, D = m["kv"], m["d"]
        QD = NH * D
        w = [dict(o=linear(QD, HID), gu=linear(HID, 2 * INTER), down=linear(INTER, HID),
                  qkv=linear(HID, (NH + 2 * KV) * D), n1=norm(HID), n2=norm(HID)) for _ in range(L)]
        inv = 1.0 / (m["theta"] ** (torch.arange(0, D, 2, device=dev).float() / D))
        freqs = torch.polar(torch.ones((CACHE, D // 2), device=dev), torch.outer(torch.arange(CACHE, device=dev).float(), inv))
        k0 = [torch.randn((1, CACHE, KV, D), generator=g, device=dev, dtype=f16) for _ in range(L)]
        v0 = [torch.randn((1, CACHE, KV, D), generator=g, device=dev, dtype=f16) for _ in range(L)]
    x0 = torch.randn((1, HID), generator=g, device=dev, dtype=f16)
    pos = torch.tensor([P], dtype=torch.int32, device=dev)

    def bufs():
        e = lambda n: torch.empty((1, n), dtype=f16, device=dev)  # noqa: E731
        out = [dict(x=e(HID), xn=e(HID), attn=e(QD), h=e(HID), hn=e(HID), act=e(INTER), k=k0[l].clone(),
                    v=v0[l].clone(), q=torch.empty((1, NH, W if mla else D), dtype=f16, device=dev),
                    ho=e(HID), xo=e(HID)) for l in range(L)]
        if mla:
            for b in out:
                b.update(qan=e(CQ), ckv=e(C))
        return out + [dict(x=e(HID), xn=e(HID))]

    def attention(b):
        q = b["q"].view(1, NH, 1, -1)
        k, v = b["k"][:, : P + 1].transpose(1, 2), b["v"][:, : P + 1].transpose(1, 2)
        with sdpa_kernel([SDPBackend.MATH]):
            o = F.scaled_dot_product_attention(q, k, v, enable_gqa=True)
        b["attn"].copy_(o.reshape(1, QD))

    def head(p, Bs, l):
        """norm1(x) and the attention's input ops of layer l"""
        b = Bs[l]
        p.layernorm_forward_cuda(b["x"], w[l]["n1"], b["xn"], EPS)
        if not mla:
            b["qkv"] = p.gemm_forward_cuda(b["xn"], *w[l]["qkv"], 8)
            p.rope_kv_cache(b["qkv"], freqs, pos, b["k"], b["v"], NH, KV, q_out=b["q"])
            return
        qa = p.gemm_forward_cuda(b["xn"], *w[l]["qa"], 8)
        p.mla_k_rope(qa, freqs, pos, b["k"], NH, DN, DR, C, CQ, 0)
        p.layernorm_forward_cuda(qa[:, :CQ], w[l]["nq"], b["qan"], EPS)
        qb = p.gemm_forward_cuda(b["qan"], *w[l]["qb"], 8)
        p.mla_q_rope(qb, freqs, pos, CACHE, NH, DN, DR, 0, q_out=b["q"])
        p.layernorm_forward_cuda(qa[:, CQ:CQ + C], w[l]["nkv"], b["ckv"], EPS)
        kv = p.gemm_forward_cuda(b["ckv"], *w[l]["kvb"], 8)
        p.mla_kv_cache(kv, pos, b["k"], b["v"], NH, DN, DV)

    def build(progs, no_fuse):
        prev = ext.get_knob(14)
        ext.set_knob(14, 1 if no_fuse else 0)
        try:
            for p in progs:
                p.build()
        finally:
            ext.set_knob(14, prev)
        return progs

    def programs_folded(Bs, no_fuse):
        """(a) / (c): [head(0)], then per layer [o, scaled_add, norm2, gate|up, silu, down, scaled_add, head(l + 1)]"""
        p0 = DecodeProgram()
        head(p0, Bs, 0)
        progs = [p0]
        for l in range(L):
            b, nb = Bs[l], Bs[l + 1]
            p = DecodeProgram()
            b["o"] = p.gemm_forward_cuda(b["attn"], *w[l]["o"], 8)
            p.scaled_add(b["x"], b["o"], AL, out=b["h"])
            p.layernorm_forward_cuda(b["h"], w[l]["n2"], b["hn"], EPS)
            b["gu"] = p.gemm_forward_cuda(b["hn"], *w[l]["gu"], 8)
            p.silu_and_mul(b["act"], b["gu"])
            b["down"] = p.gemm_forward_cuda(b["act"], *w[l]["down"], 8)
            p.scaled_add(b["h"], b["down"], AL, out=nb["x"])
            if l + 1 < L:
                head(p, Bs, l + 1)
            progs.append(p)
        return build(progs, no_fuse)

    def programs_split(Bs):
        """(b): per layer [o] | torch | [norm2, gate|up, silu, down] | torch | [head(l + 1)]"""
        p0 = DecodeProgram()
        head(p0, Bs, 0)
        progs = [[p0]]
        for l in range(L):
            b = Bs[l]
            po, pm = DecodeProgram(), DecodeProgram()
            b["o"] = po.gemm_forward_cuda(b["attn"], *w[l]["o"], 8)
            pm.layernorm_forward_cuda(b["h"], w[l]["n2"], b["hn"], EPS)
            b["gu"] = pm.gemm_forward_cuda(b["hn"], *w[l]["gu"], 8)
            pm.silu_and_mul(b["act"], b["gu"])
            b["down"] = pm.gemm_forward_cuda(b["act"], *w[l]["down"], 8)
            layer = [po, pm]
            if l + 1 < L:
                ph = DecodeProgram()
                head(ph, Bs, l + 1)
                layer.append(ph)
            progs.append(layer)
        for ps in progs:
            build(ps, False)
        return progs

    Ba, Bb, Bc = bufs(), bufs(), bufs()
    for B in (Ba, Bb, Bc):
        B[0]["x"].copy_(x0)
    progs_a, progs_b, progs_c = programs_folded(Ba, True), programs_split(Bb), programs_folded(Bc, False)

    def step_folded(Bs, progs):
        progs[0].run()
        for l in range(L):
            attention(Bs[l])
            progs[l + 1].run()

    def step_split():
        progs_b[0][0].run()
        for l in range(L):
            b, nb = Bb[l], Bb[l + 1]
            attention(b)
            layer = progs_b[l + 1]
            layer[0].run()
            torch.mul(b["o"], AL, out=b["ho"])
            torch.add(b["x"], b["ho"], out=b["h"])
            layer[1].run()
            torch.mul(b["down"], AL, out=b["xo"])
            torch.add(b["h"], b["xo"], out=nb["x"])
            if len(layer) > 2:
                layer[2].run()

    graphs = {}
    with torch.no_grad():
        for vname, fn in (("a_per_op", lambda: step_folded(Ba, progs_a)), ("b_split_torch_scaled_add", step_split),
                          ("c_one_program_per_segment", lambda: step_folded(Bc, progs_c))):
            graphs[vname], _ = bench.capture(torch, fn)
    for gph in graphs.values():
        gph.replay()
    torch.cuda.synchronize()
    last = Bc[L - 1]
    rms = float(Ba[L]["x"].float().pow(2).mean().sqrt())
    d_b = float((Bb[L]["x"].float() - Ba[L]["x"].float()).abs().max())
    d_c = float((Bc[L]["x"].float() - Ba[L]["x"].float()).abs().max())
    ref = last["h"] + last["down"] * AL
    chk = {"c_last_scaled_add_bit_exact_vs_torch": torch.equal(ref.view(torch.int16), Bc[L]["x"].view(torch.int16)),
           "output_rms": round(rms, 4), "b_output_max_abs_diff_vs_a": round(d_b, 5),
           "c_output_max_abs_diff_vs_a": round(d_c, 5),
           "outputs_consistent": bool(torch.isfinite(Bc[L]["x"]).all()) and max(d_b, d_c) <= 0.05 * rms + 0.05}
    chk["all_passed"] = chk["c_last_scaled_add_bit_exact_vs_torch"] and chk["outputs_consistent"]

    for gph in graphs.values():
        for _ in range(a.warmup):
            gph.replay()
    torch.cuda.synchronize()
    sampler = bench.ClockSampler(0)
    sampler.start()
    times = {k: [] for k in graphs}
    t0 = time.time()
    for _ in range(a.rounds):
        for vname, gph in graphs.items():
            times[vname].append(bench.timed(torch, gph.replay, a.steps, 0) / a.steps * 1e3)
    t1 = time.time()
    clocks = sampler.stop(t0, t1)
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    unfused = {"b": [i for i, ps in enumerate(progs_b) for p in ps if not p.fused],
               "c": [i for i, p in enumerate(progs_c) if not p.fused]}
    out = {"model": name, "layers": L, "alpha": AL, "weight_bytes": wbytes, "launches_per_step_c": len(progs_c),
           "kernel_ops_per_segment_c": progs_c[1].kernel_ops, "programs_replayed_per_op": unfused,
           "clocks_during_timing": clocks, "checks": chk,
           "b_over_c": round(med["b_split_torch_scaled_add"] / med["c_one_program_per_segment"], 3),
           "saved_us_per_layer_c_vs_b": round((med["b_split_torch_scaled_add"] - med["c_one_program_per_segment"]) *
                                              1e3 / L, 2),
           "variants": {k: {"ms_per_step": round(med[k], 4), "rounds_ms": [round(t, 4) for t in times[k]]}
                        for k in graphs}}
    del graphs, progs_a, progs_b, progs_c, Ba, Bb, Bc, w, k0, v0
    gc.collect()
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--pos", type=int, default=1023, help="cache row of the step's token")
    ap.add_argument("--models", nargs="*", default=list(MODELS), choices=list(MODELS))
    a = ap.parse_args()

    import torch

    torch.cuda.set_device(0)
    res = {n: run_model(n, a) for n in a.models}
    print(json.dumps({"tool": "scaled_residual_decode_bench", "workload":
                      f"one token at cache row {a.pos} of a {CACHE}-row cache, g128 seeded random weights; attention = "
                      "SDPA math-backend stand-in", "card": torch.cuda.get_device_name(0),
                      "power_limit_w": _power_limit_w(0), "steps": a.steps, "warmup": a.warmup, "rounds": a.rounds,
                      "models": res}), flush=True)


if __name__ == "__main__":
    main()
