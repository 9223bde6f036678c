#!/usr/bin/env python
"""Decode step (bs = 1) of two LayerNorm models, each two ways: one JSON line.

  Command-R v01 (CohereBlock, parallel residual): 40 layers, hidden 8192, 64 q / 64 kv heads of 128, intermediate
      22528, RoPE theta 8e6, CohereLayerNorm without a bias.  Per segment: h = o(attn) + x; act = silu(gate) up of
      gate|up(xn); x' = down(act) + h; xn' = LN(x'); qkv' and RoPE + cache append.
  StarCoder2-15B (LlamaLikeBlock): 40 layers, hidden 6144, 48 q / 4 kv heads of 128, intermediate 24576, theta 1e5,
      nn.LayerNorm and GELUTanh, every linear with a bias.  Per segment: h = o(attn) + x; hn = LN(h); a = gelu(c_fc(hn));
      x' = c_proj(a) + h; xn' = LN(x'); qkv' and RoPE + cache append.

  (a) the split that works without LAYER_NORM / GELU ops: decode programs between every LayerNorm and GELU, with
      transformers' CohereLayerNorm / torch's nn.LayerNorm / transformers' GELUTanh between them (2 programs per layer
      for Command-R, 4 for StarCoder2);
  (b) one program per attention-to-attention segment (DESIGN.md 3.5l).

g128 seeded random weights (bench.py's scale recipe).  The attention is a stand-in, F.scaled_dot_product_attention on
torch's math backend over cache[:, :P + 1] from the rotated q, outside every program and timed alone.  Each variant is
one CUDA graph; the graphs are replayed alternately (rounds x steps after warm-up), the median round is reported with
ms / step, tok/s and GB/s over the step's algorithmic bytes (packed weights, scales, zeros and biases once, the KV rows
the attention reads).  The models run one after the other, with memory freed between them.  Card, power limit and SM
clock are read in the same run.

Self-checks on the last layer of (b): its LayerNorm and GELU outputs bit-identical to the stand-alone ops on (b)'s own
inputs; (b)'s step output within tolerance of (a)'s.

    python tools/layernorm_decode_bench.py [--steps 20] [--warmup 3] [--rounds 5] [--pos 1023] [--layers 40]
"""
import argparse
import gc
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (graph capture, timing and the clock sampler of the bench)
from tools.batched_decode_bench import _power_limit_w  # noqa: E402

CACHE, GROUP, HEAD_DIM, EPS = 2048, 128, 128, 1e-5
MODELS = {
    "command-r-v01": dict(hidden=8192, heads=64, kv=64, inter=22528, theta=8e6, cohere=True),
    "starcoder2-15b": dict(hidden=6144, heads=48, kv=4, inter=24576, theta=1e5, cohere=False),
}


def run_model(name, cfg, a):
    import torch
    import torch.nn.functional as F
    from torch.nn.attention import SDPBackend, sdpa_kernel
    from transformers.activations import GELUTanh
    from transformers.models.cohere.modeling_cohere import CohereLayerNorm

    from autoawq_b200 import ext
    from autoawq_b200.program import DecodeProgram

    dev = torch.device("cuda", 0)
    f16 = torch.float16
    H, I, L, D, P = cfg["hidden"], cfg["inter"], a.layers, HEAD_DIM, a.pos
    NH, KV, cohere = cfg["heads"], cfg["kv"], cfg["cohere"]
    QD, NQKV = NH * D, (NH + 2 * KV) * D
    g = torch.Generator(device=dev).manual_seed(0)
    wbytes = 0

    def linear(K, N):
        nonlocal wbytes
        qw = torch.randint(-2**31, 2**31 - 1, (K, N // 8), dtype=torch.int32, device=dev, generator=g)
        qz = torch.randint(-2**31, 2**31 - 1, (K // GROUP, N // 8), dtype=torch.int32, device=dev, generator=g)
        s = ((torch.rand((K // GROUP, N), device=dev, generator=g) * 0.5 + 0.75) / (6.1 * K**0.5)).half()
        b = None if cohere else (0.02 * torch.randn(N, device=dev, generator=g)).half()
        wbytes += qw.numel() * 4 + qz.numel() * 4 + s.numel() * 2 + (b.numel() * 2 if b is not None else 0)
        return qw, s, qz, b

    def norm():
        if cohere:
            m = CohereLayerNorm(H, eps=EPS, bias=False)
        else:
            m = torch.nn.LayerNorm(H, eps=EPS)
        m = m.to(dev).half()
        with torch.no_grad():
            m.weight.copy_((1 + 0.1 * torch.randn(H, generator=g, device=dev)).half())
            if not cohere:
                m.bias.copy_((0.05 * torch.randn(H, generator=g, device=dev)).half())
        return m

    mlp_in = "gu" if cohere else "fc"
    w = [{"o": linear(QD, H), mlp_in: linear(H, 2 * I if cohere else I), "down": linear(I, H), "qkv": linear(H, NQKV)}
         for _ in range(L)]
    n1 = [norm() for _ in range(L)]
    n2 = [None if cohere else norm() for _ in range(L)]
    gelu_t = GELUTanh()
    inv = 1.0 / (cfg["theta"] ** (torch.arange(0, D, 2, device=dev, dtype=torch.float32) / D))
    freqs = torch.polar(torch.ones((CACHE, D // 2), device=dev), torch.outer(torch.arange(CACHE, device=dev).float(), inv))
    k0 = [torch.randn((1, CACHE, KV, D), generator=g, device=dev, dtype=f16) for _ in range(L)]
    v0 = [torch.randn((1, CACHE, KV, D), generator=g, device=dev, dtype=f16) for _ in range(L)]
    x0 = torch.randn((1, H), generator=g, device=dev, dtype=f16)
    pos = torch.tensor([P], dtype=torch.int32, device=dev)

    def bufs():
        e = lambda n: torch.empty((1, n), dtype=f16, device=dev)  # noqa: E731
        B = [dict(x=e(H), xn=e(H), attn=e(QD), h=e(H), hn=e(H), fc=e(I), act=e(I), q=torch.empty((1, NH, D), dtype=f16,
                  device=dev), k=k0[l].clone(), v=v0[l].clone()) for l in range(L)]
        return B + [dict(x=e(H), xn=e(H))]

    def lin(p, x, l, k):
        qw, s, qz, b = w[l][k]
        return p.gemm_forward_cuda(x, qw, s, qz, 8, bias=b)

    def attention(b):
        k = b["k"][:, : P + 1].transpose(1, 2)
        v = b["v"][:, : P + 1].transpose(1, 2)
        with sdpa_kernel([SDPBackend.MATH]):
            o = F.scaled_dot_product_attention(b["q"].reshape(1, NH, 1, D), k, v, enable_gqa=True)
        b["attn"].copy_(o.reshape(1, QD))

    def head(p, B, l):
        B[l]["qkv"] = lin(p, B[l]["xn"], l, "qkv")
        p.rope_kv_cache(B[l]["qkv"], freqs, pos, B[l]["k"], B[l]["v"], NH, KV, q_out=B[l]["q"])

    def norm_args(m):
        return m.weight, (None if cohere else m.bias)

    # ---- (a): a program between every LayerNorm and GELU, torch between them
    def plan_a(B):
        progs = []

        def new():
            progs.append(DecodeProgram())
            return progs[-1]

        steps = [lambda: B[0]["xn"].copy_(n1[0](B[0]["x"]))]
        p0 = new()
        head(p0, B, 0)
        steps.append(p0.run)
        for l in range(L):
            b, nb = B[l], B[l + 1]
            p = new()
            b["o"] = lin(p, b["attn"], l, "o")
            p.add(b["o"], b["x"], out=b["h"])
            if cohere:
                b["gu"] = lin(p, b["xn"], l, "gu")
                p.silu_and_mul(b["act"], b["gu"])
                b["down"] = lin(p, b["act"], l, "down")
                p.add(b["down"], b["h"], out=nb["x"])
                steps.append(p.run)
            else:
                steps.append(p.run)
                steps.append(lambda b=b, l=l: b["hn"].copy_(n2[l](b["h"])))
                p = new()
                b["fc"] = lin(p, b["hn"], l, "fc")
                steps.append(p.run)
                steps.append(lambda b=b: b["act"].copy_(gelu_t(b["fc"])))
                p = new()
                b["down"] = lin(p, b["act"], l, "down")
                p.add(b["down"], b["h"], out=nb["x"])
                steps.append(p.run)
            if l + 1 < L:
                steps.append(lambda nb=nb, l=l: nb["xn"].copy_(n1[l + 1](nb["x"])))
                p = new()
                head(p, B, l + 1)
                steps.append(p.run)
            if l + 1 < L:
                steps.append(lambda nb=nb: attention(nb))
        for p in progs:
            p.build()
            assert p.fused, "a program of the split did not fuse"
        return progs, steps

    # ---- (b): one program per attention-to-attention segment
    def plan_b(B):
        progs = []
        p0 = DecodeProgram()
        p0.layer_norm(B[0]["x"], *norm_args(n1[0]), B[0]["xn"], EPS)
        head(p0, B, 0)
        progs.append(p0)
        for l in range(L):
            b, nb = B[l], B[l + 1]
            p = DecodeProgram()
            b["o"] = lin(p, b["attn"], l, "o")
            p.add(b["o"], b["x"], out=b["h"])
            if cohere:
                b["gu"] = lin(p, b["xn"], l, "gu")
                p.silu_and_mul(b["act"], b["gu"])
            else:
                p.layer_norm(b["h"], *norm_args(n2[l]), b["hn"], EPS)
                b["fc"] = lin(p, b["hn"], l, "fc")
                p.gelu(b["act"], b["fc"], "tanh")
            b["down"] = lin(p, b["act"], l, "down")
            p.add(b["down"], b["h"], out=nb["x"])
            if l + 1 < L:
                p.layer_norm(nb["x"], *norm_args(n1[l + 1]), nb["xn"], EPS)
                head(p, B, l + 1)
            progs.append(p)
        for p in progs:
            p.build()
            assert p.fused, "a segment program did not fuse"
        steps = [progs[0].run]
        for l in range(L):
            steps.append(lambda b=B[l]: attention(b))
            steps.append(progs[l + 1].run)
        return progs, steps

    Ba, Bb = bufs(), bufs()
    Ba[0]["x"].copy_(x0)
    Bb[0]["x"].copy_(x0)
    Ba[0]["attn"].zero_()
    Bb[0]["attn"].zero_()
    progs_a, steps_a = plan_a(Ba)
    progs_b, steps_b = plan_b(Bb)
    # (a)'s step list runs the attention of layer l + 1 after its head; layer 0's runs after the first head in both
    steps_a.insert(2, lambda: attention(Ba[0]))

    def step_a():
        for s in steps_a:
            s()
        return Ba[L]["x"]

    def step_b():
        for s in steps_b:
            s()
        return Bb[L]["x"]

    def step_attn():
        for l in range(L):
            attention(Bb[l])

    graphs = {}
    with torch.no_grad():
        for vname, fn in (("a_split_programs_plus_torch_ln_gelu", step_a), ("b_one_program_per_segment", step_b),
                          ("attention_stand_in", step_attn)):
            graphs[vname], _ = bench.capture(torch, fn)

    # ---- self-checks after one replay of each graph on identical inputs (the caches were written at the same position)
    for gph in graphs.values():
        gph.replay()
    torch.cuda.synchronize()
    last = L - 1
    b = Bb[last]
    chk = {}
    if not cohere:
        want = torch.empty_like(b["hn"])
        ext.layer_norm(b["h"], n2[last].weight, n2[last].bias, want, EPS)
        act = torch.empty_like(b["fc"])
        ext.gelu(act, b["fc"], "tanh")
        chk["b_last_layer_ln_gelu_bit_identical"] = torch.equal(want, b["hn"]) and torch.equal(act, b["act"])
    want = torch.empty_like(b["xn"])
    ext.layer_norm(Bb[last]["x"], n1[last].weight, None if cohere else n1[last].bias, want, EPS)
    chk["b_last_layer_input_ln_bit_identical"] = torch.equal(want, Bb[last]["xn"])
    d_out = float((Bb[L]["x"].float() - Ba[L]["x"].float()).abs().max())
    rms = float(Ba[L]["x"].float().pow(2).mean().sqrt())
    chk.update({"b_output_max_abs_diff_vs_a": round(d_out, 5), "output_rms": round(rms, 4),
                "b_output_consistent_with_a": bool(torch.isfinite(Bb[L]["x"]).all()) and d_out <= 0.05 * rms + 0.05})

    # ---- timing
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
    kv_bytes = L * 2 * (P + 1) * KV * D * 2
    step_bytes = wbytes + kv_bytes
    table = {}
    for vname in ("a_split_programs_plus_torch_ln_gelu", "b_one_program_per_segment"):
        ms = med[vname]
        table[vname] = {"ms_per_step": round(ms, 4), "tok_s": round(1e3 / ms, 1), "gb_s": round(step_bytes / ms / 1e6, 1),
                        "ms_without_attention": round(ms - med["attention_stand_in"], 4),
                        "program_launches": sum(p.launches_per_run for p in (progs_a if vname[0] == "a" else progs_b)),
                        "rounds_ms": [round(t, 4) for t in times[vname]]}
    table["a_vs_b"] = round(med["a_split_programs_plus_torch_ln_gelu"] / med["b_one_program_per_segment"], 3)
    table["saved_ms_per_layer"] = round((med["a_split_programs_plus_torch_ln_gelu"] -
                                         med["b_one_program_per_segment"]) / L, 5)
    out = {"model": name, "layers": L, "step_bytes": step_bytes, "attention_stand_in_ms": round(med["attention_stand_in"], 4),
           "clocks_during_timing": clocks, "variants": table, "checks": chk}
    del graphs, progs_a, progs_b, steps_a, steps_b, Ba, Bb, w
    gc.collect()
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--pos", type=int, default=1023, help="the fixed decode position P (attention reads P + 1 rows)")
    ap.add_argument("--layers", type=int, default=40)
    ap.add_argument("--models", nargs="*", default=list(MODELS))
    a = ap.parse_args()

    import torch

    torch.cuda.set_device(0)
    res = {n: run_model(n, MODELS[n], a) for n in a.models}
    print(json.dumps({"tool": "layernorm_decode_bench", "workload": f"decode bs=1, position {a.pos} of a {CACHE}-position "
                      "cache, g128 seeded random weights; attention = SDPA math-backend stand-in over cache[:, :P + 1]",
                      "card": torch.cuda.get_device_name(0), "power_limit_w": _power_limit_w(0), "steps": a.steps,
                      "warmup": a.warmup, "rounds": a.rounds, "models": res}), flush=True)


if __name__ == "__main__":
    main()
