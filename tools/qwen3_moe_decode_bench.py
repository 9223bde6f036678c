#!/usr/bin/env python
"""Qwen3-30B-A3B decode step (bs = 1, 48 layers) with Qwen3-MoE expert blocks, two ways: one JSON line.

Per layer: xn = norm1(h); qkv = xn Wqkv; q, k = q_norm(q), k_norm(k); RoPE at position P and the cache append;
attn = ATTENTION STAND-IN; o = attn Wo; hm = o + h; xn2 = norm2(hm); moe = Qwen3-MoE expert block(xn2) (E = 128, top-8,
I = 768, norm_topk_prob); h' = moe + hm.  Shapes: hidden 2048, 32 q / 4 kv heads of 128, RoPE theta 1e6, g128, seeded
random weights (bench.py's scale recipe).  The attention stand-in is qwen3_decode_bench.py's: SDPA on torch's math
backend over cache[:, :P + 1], P fixed (1023 in a 2048-position cache), outside every program and timed alone.

  (a) per_op: the 49 attention-to-attention programs built with knob 14 = 1, so run() replays every op through ext and
      torch (DecodeProgram.qwen3_moe's per-op replay), all captured in one CUDA graph;
  (b) fused: the same 49 programs fused, one persistent kernel per segment (DESIGN.md 3.5h), in one CUDA graph.
The graphs are replayed alternately (rounds x steps after warm-up) and the median round is reported, with GB/s over the
active bytes of a token (attention linears, router and the 8 selected experts of every layer).  Card, power limit and
SM clock are read in the same run.

routing: knob 3 = 2 stamps (program_stream.cuh) of the gate|up op, staged -> routing published ([7] - [2]), median over
runs and the 8 recorded CTAs, in us: the E = 128 exchange of a (b) segment program, and at E = 64 (the first 64 experts
of layer 0) the exchange next to sparse_moe's redundant routing (DESIGN.md 3.5d) on the same weights and row.

mixtral (--mixtral-trees A B ...): tools/moe_decode_bench.py of each source tree (each with its own built library),
run first, alternately, --mixtral-rounds times; its program ms/step per tree.

Self-checks after one replay of each graph on identical inputs: (b)'s last-layer routing against its own logits, its
combine bit-exact from its own per-slot outputs, and (b)'s layer-0 expert-block output within 1 % of rms of (a)'s with
the same experts.  Further down the stack the arms drift apart (the router matmul and the linears round differently per
op and fused, and the random layers amplify it): reported are the first layer where they choose different experts and
the largest block difference before it.

    python tools/qwen3_moe_decode_bench.py [--steps 20] [--warmup 5] [--rounds 5] [--layers 48] [--stamp-runs 20]
                                           [--mixtral-trees DIR ...] [--mixtral-rounds 2]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (graph capture, timing and the clock sampler of the bench)
from tools.batched_decode_bench import DATASHEET_GBS, _power_limit_w  # noqa: E402

HIDDEN, HEADS, KV_HEADS, HEAD_DIM, E, TOPK, INTER, GROUP, CACHE = 2048, 32, 4, 128, 128, 8, 768, 128, 2048
THETA, EPS = 1e6, 1e-6


def _mixtral(trees, rounds, steps, warmup):
    """tools/moe_decode_bench.py of each tree, alternately: {tree: [program ms per run]}."""
    out = {t: [] for t in trees}
    for _ in range(rounds):
        for t in trees:
            r = subprocess.run([sys.executable, os.path.join(t, "tools", "moe_decode_bench.py"), "--steps", str(steps),
                                "--warmup", str(warmup)], capture_output=True, text=True, cwd=t)
            if r.returncode != 0:
                raise SystemExit(f"moe_decode_bench.py in {t} failed:\n{r.stderr[-2000:]}")
            out[t].append(json.loads(r.stdout.strip().splitlines()[-1])["result"]["program_ms"])
    return out


def _stamps(lib, check):
    import numpy as np

    buf = np.zeros(32 * 8 * 8, dtype=np.uint64)
    check(lib.b200awq_debug_read(buf.ctypes.data_as(ctypes.c_void_p), buf.nbytes), "b200awq_debug_read")
    return buf.reshape(32, 8, 8).astype(np.int64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--layers", type=int, default=48)
    ap.add_argument("--pos", type=int, default=1023)
    ap.add_argument("--stamp-runs", type=int, default=20)
    ap.add_argument("--mixtral-trees", nargs="*", default=[])
    ap.add_argument("--mixtral-rounds", type=int, default=2)
    a = ap.parse_args()

    # Mixtral first: its 32 layers (and their stream copies) and this step's weights do not fit one card together
    mixtral = _mixtral([os.path.abspath(t) for t in a.mixtral_trees], a.mixtral_rounds, 30, 5) if a.mixtral_trees else None

    import numpy as np
    import torch
    import torch.nn.functional as F
    from torch.nn.attention import SDPBackend, sdpa_kernel
    from transformers.models.qwen3.modeling_qwen3 import Qwen3RMSNorm

    from autoawq_b200 import ext
    from autoawq_b200._cabi import check, lib
    from autoawq_b200.program import DecodeProgram

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    H, L, D, P, I = HIDDEN, a.layers, HEAD_DIM, a.pos, INTER
    QD = HEADS * D
    f16 = torch.float16
    g = torch.Generator(device=dev).manual_seed(0)

    def linear(K, N, n_exp=None):
        lead = () if n_exp is None else (n_exp,)
        qw = torch.randint(-2**31, 2**31 - 1, lead + (K, N // 8), dtype=torch.int32, device=dev, generator=g)
        qz = torch.randint(-2**31, 2**31 - 1, lead + (K // GROUP, N // 8), dtype=torch.int32, device=dev, generator=g)
        s = (torch.rand(lead + (K // GROUP, N), device=dev, generator=g) * 0.5 + 0.75) / (6.1 * K**0.5)
        return qw, s.half(), qz

    w = [dict(qkv=linear(H, (HEADS + 2 * KV_HEADS) * D), o=linear(QD, H), w1=linear(H, 2 * I, E), w2=linear(I, H, E),
              gate=(torch.randn((E, H), device=dev, generator=g) * 0.05).half()) for _ in range(L)]
    norm1 = [(1 + 0.1 * torch.randn(H, generator=g, device=dev)).half() for _ in range(L)]
    norm2 = [(1 + 0.1 * torch.randn(H, generator=g, device=dev)).half() for _ in range(L)]
    qk_norms = []
    for _ in range(L):
        pair = []
        for _ in range(2):
            n = Qwen3RMSNorm(D, eps=EPS).to(dev).half()
            with torch.no_grad():
                n.weight.copy_((1 + 0.2 * torch.randn(D, generator=g, device=dev)).half())
            pair.append(n)
        qk_norms.append(pair)
    inv = 1.0 / (THETA ** (torch.arange(0, D, 2, device=dev).float() / D))
    freqs = torch.polar(torch.ones(CACHE, D // 2, device=dev), torch.outer(torch.arange(CACHE, device=dev).float(), inv))
    cache0 = [(torch.randn((1, CACHE, KV_HEADS, D), generator=g, device=dev, dtype=f16),
               torch.randn((1, CACHE, KV_HEADS, D), generator=g, device=dev, dtype=f16)) for _ in range(L)]
    h0 = torch.randn((1, H), generator=g, device=dev, dtype=f16)

    def caches():
        return [(k.clone(), v.clone()) for k, v in cache0]

    def attention(q, c, out):
        k = c[0][:, : P + 1].transpose(1, 2)
        v = c[1][:, : P + 1].transpose(1, 2)
        with sdpa_kernel([SDPBackend.MATH]):
            o = F.scaled_dot_product_attention(q.reshape(1, HEADS, 1, D), k, v, enable_gqa=True)
        out.copy_(o.reshape(1, QD))

    def bufs():
        e = lambda n: torch.empty((1, n), dtype=f16, device=dev)  # noqa: E731
        return [dict(h=e(H), xn=e(H), attn=e(QD), hm=e(H), xn2=e(H), q=e(QD)) for _ in range(L)] + [dict(h=e(H))]

    def head(p, B, C, l, pos):
        B[l]["qkv"] = p.gemm_forward_cuda(B[l]["xn"], *w[l]["qkv"], 8)
        qn, kn = qk_norms[l]
        p.rope_kv_cache(B[l]["qkv"], freqs, pos, C[l][0], C[l][1], HEADS, KV_HEADS, q_out=B[l]["q"], q_norm=qn, k_norm=kn)

    def segment(p, B, C, l, pos):
        b = B[l]
        b["o"] = p.gemm_forward_cuda(b["attn"], *w[l]["o"], 8)
        p.add(b["o"], b["h"], out=b["hm"])
        p.layernorm_forward_cuda(b["hm"], norm2[l], b["xn2"], EPS)
        b["moe"] = p.qwen3_moe(b["xn2"], w[l]["gate"], w[l]["w1"], w[l]["w2"], TOPK, True)
        p.add(b["moe"], b["hm"], out=B[l + 1]["h"])
        if l + 1 < L:
            p.layernorm_forward_cuda(B[l + 1]["h"], norm1[l + 1], B[l + 1]["xn"], EPS)
            head(p, B, C, l + 1, pos)

    def programs(B, C, pos, fused):
        p0 = DecodeProgram()
        p0.layernorm_forward_cuda(B[0]["h"], norm1[0], B[0]["xn"], EPS)
        head(p0, B, C, 0, pos)
        plan = [p0]
        for l in range(L):
            p = DecodeProgram()
            segment(p, B, C, l, pos)
            plan.append(p)
        ext.set_knob(14, 0 if fused else 1)
        try:
            for p in plan:
                p.build()
                assert p.fused == fused, "a segment program did not fuse" if fused else "knob 14 = 1 fused a program"
        finally:
            ext.set_knob(14, 0)
        return plan

    pos = torch.tensor([P], dtype=torch.int32, device=dev)
    arms = {}
    for name, fused in (("a_per_op_graph", False), ("b_fused_programs", True)):
        B, C = bufs(), caches()
        B[0]["h"].copy_(h0)
        t = time.time()
        arms[name] = (programs(B, C, pos, fused), B, C, round(time.time() - t, 1))

    def stepper(name):
        plan, B, C, _ = arms[name]

        def step():
            plan[0].run()
            for l in range(L):
                attention(B[l]["q"], C[l], B[l]["attn"])
                plan[l + 1].run()
        return step

    def step_attn():
        _, B, C, _ = arms["b_fused_programs"]
        for l in range(L):
            attention(B[l]["q"], C[l], B[l]["attn"])

    graphs = {}
    for name, fn in (("a_per_op_graph", stepper("a_per_op_graph")), ("b_fused_programs", stepper("b_fused_programs")),
                     ("attention_stand_in", step_attn)):
        graphs[name], _ = bench.capture(torch, fn)

    # ---- self-checks (after one replay of each graph on identical inputs)
    for gph in graphs.values():
        gph.replay()
    torch.cuda.synchronize()
    abort = DecodeProgram.abort_record()
    last = L - 1
    pa, Ba = arms["a_per_op_graph"][0], arms["a_per_op_graph"][1]
    pb, Bb = arms["b_fused_programs"][0], arms["b_fused_programs"][1]
    mb, ma = pb[L].moe_buffers(0), pa[L].moe_buffers(0)
    probs = torch.softmax(mb["logits"].float(), dim=-1)
    want = sorted(torch.topk(probs, TOPK, dim=-1).indices.flatten().tolist())
    got = mb["topk_ids"].flatten().tolist()
    acc = torch.zeros(H, dtype=f16, device=dev)
    for s in sorted(range(TOPK), key=lambda k: got[k]):
        acc = acc + mb["down"][0, s]
    # the two arms' routings drift apart over the layers (the router matmul rounds differently per op and fused):
    # compare the block outputs layer by layer where both chose the same experts
    same = [torch.equal(pb[l + 1].moe_buffers(0)["topk_ids"], pa[l + 1].moe_buffers(0)["topk_ids"]) for l in range(L)]
    rms0 = float(Ba[0]["moe"].float().pow(2).mean().sqrt())
    d0 = float((Bb[0]["moe"].float() - Ba[0]["moe"].float()).abs().max())
    first = next((l for l in range(L) if not same[l]), L)     # before it both arms' inputs still agree closely
    d_same = max([float((Bb[l]["moe"].float() - Ba[l]["moe"].float()).abs().max() /
                        Ba[l]["moe"].float().pow(2).mean().sqrt()) for l in range(first)] or [0.0])
    checks = {"no_abort_record": abort[3] == 0,
              "b_last_layer_routing_matches_its_logits": sorted(got) == want,
              "b_last_layer_combine_bit_exact_from_its_slots": torch.equal(acc, Bb[last]["moe"][0]),
              "layers_with_same_experts_in_a_and_b": int(sum(same)),
              "first_layer_with_different_experts": first if first < L else None,
              "layer0_moe_max_abs_diff_b_vs_a": round(d0, 5), "layer0_moe_rms": round(rms0, 4),
              "max_abs_diff_over_rms_b_vs_a_before_that_layer": round(d_same, 5),
              "b_consistent_with_a": bool(torch.isfinite(Bb[L]["h"]).all()) and same[0] and d0 <= 0.01 * rms0}

    # ---- routing phase: staged -> routing published of a gate|up op
    def routing_us(prog, op):
        vals = []
        was = ext.get_knob(3)
        try:
            ext.set_knob(3, 2)
            for _ in range(a.stamp_runs):
                prog.run()
                torch.cuda.synchronize()
                st = _stamps(lib, check)
                vals.extend(((st[op, :, 7] - st[op, :, 2]) / 1e3).tolist())
        finally:
            ext.set_knob(3, was)
        return {"median_us": round(float(np.median(vals)), 3), "max_us": round(float(np.max(vals)), 3)}

    routing = {"qwen3_moe_E128_exchange": routing_us(pb[1], 1)}     # segment ops: o, gate|up, down, qkv
    x = torch.randn((1, H), generator=g, device=dev, dtype=f16)
    w0 = w[0]
    for name, hf in (("sparse_moe_E64_redundant", False), ("qwen3_moe_E64_exchange", True)):
        p = DecodeProgram()
        args = (x, w0["gate"][:64], tuple(t[:64] for t in w0["w1"]), tuple(t[:64] for t in w0["w2"]), TOPK, True)
        (p.qwen3_moe if hf else p.sparse_moe)(*args)
        p.build()
        assert p.fused
        routing[name] = routing_us(p, 0)
        p.close()
    routing["design_3_5d_mixtral_measured_us"] = 5.0

    # ---- timing: alternate the graphs, `rounds` x `steps` replays each after warm-up
    for gph in graphs.values():
        for _ in range(a.warmup):
            gph.replay()
    torch.cuda.synchronize()
    sampler = bench.ClockSampler(0)
    sampler.start()
    times = {k: [] for k in graphs}
    t0 = time.time()
    for _ in range(a.rounds):
        for name, gph in graphs.items():
            times[name].append(bench.timed(torch, gph.replay, a.steps, 0) / a.steps * 1e3)
    t1 = time.time()
    clocks = sampler.stop(t0, t1)
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    attn_ms = med["attention_stand_in"]
    wb = lambda K, N: K * N // 2 + (K // GROUP) * N * 2 + (K // GROUP) * N // 2  # noqa: E731
    active = L * (wb(H, (HEADS + 2 * KV_HEADS) * D) + wb(QD, H) + E * H * 2 + TOPK * (wb(H, 2 * I) + wb(I, H)))
    table = {}
    for name in ("a_per_op_graph", "b_fused_programs"):
        ms = med[name]
        table[name] = {"ms_per_step": round(ms, 4), "tok_s": round(1e3 / ms, 1),
                       "ms_without_attention": round(ms - attn_ms, 4),
                       "gbs_over_active_bytes_without_attention": round(active / (ms - attn_ms) / 1e6, 1),
                       "build_s": arms[name][3], "rounds_ms": [round(t, 4) for t in times[name]]}
    table["a_vs_b"] = round(med["a_per_op_graph"] / med["b_fused_programs"], 3)
    res = {"tool": "qwen3_moe_decode_bench",
           "workload": f"Qwen3-30B-A3B decode bs=1, {L} layers: q / k norm, RoPE (theta {THETA:g}) and KV-cache append at "
                       f"position {P} of a {CACHE}-position cache, residual adds, Qwen3-MoE block E={E} top-{TOPK} "
                       f"I={I}, g{GROUP}, seeded random weights; attention = SDPA math-backend stand-in over "
                       "cache[:, :P + 1]",
           "card": torch.cuda.get_device_name(dev), "power_limit_w": _power_limit_w(0), "clocks_during_timing": clocks,
           "steps": a.steps, "warmup": a.warmup, "rounds": a.rounds, "active_gb_per_token": round(active / 1e9, 3),
           "datasheet_gbs": DATASHEET_GBS, "attention_stand_in_ms": round(attn_ms, 4), "variants": table,
           "routing_phase": routing, "checks": checks}
    if mixtral is not None:
        res["mixtral_moe_decode_bench_program_ms"] = mixtral
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
