#!/usr/bin/env python
"""Llama-3-8B decode step (bs = 1, 32 layers) WITH the decoder block's residual adds, three ways: one JSON line.

Per layer: xn = norm1(h); qkv = xn Wqkv; attn = ATTENTION STAND-IN(q); o = attn Wo; hm = o + h; xn2 = norm2(hm);
gu = xn2 Wgu; act = silu(gate) up; down = act Wd; h' = down + hm (awq/modules/fused/block.py:117-118).

The attention is a stand-in, not the model's attention: F.scaled_dot_product_attention(q, K, V, enable_gqa=True) with q
taken from qkv[:, :4096] (32 heads x 128) over a fixed, seeded KV cache of 1024 positions (8 KV heads), no RoPE, no
cache append.  By default it runs on torch's math backend: the fused backends are not bit-reproducible from call to
call, and the identity check needs (b) and (c) to see the same attention output.  `--attention fast` times the fused
backends instead (the identity check then reports where run-to-run attention noise first shows).  It stays outside every program (DESIGN.md 7) and is timed on its own, so it can be subtracted.

  (a) per-op: awq_ext-facing launches (PDL on, as bench.py) + torch.add for the adds;
  (b) three programs per layer without adds - [norm1, qkv] | attention | [o] | torch.add | [norm2, gate|up, silu, down]
      | torch.add - today's best correct split (96 programs + 64 adds per step);
  (c) the segments from one attention call to the next with the adds recorded through DecodeProgram.add:
      [norm1, qkv], then per layer [o + h, norm2, gate|up, silu, down + hm, norm1', qkv'] (33 programs, no glue launches).

Each variant is captured in one CUDA graph; the graphs are replayed alternately (rounds x steps after warm-up) and the
median round is reported: ms per step, tok/s, and GB/s over the step's algorithmic bytes (DESIGN.md 2: packed weights +
scales + zeros + activations of the 128 linears) with the stand-in's time subtracted.  Card, power limit and SM clock
are read in the same run.  Self-checks: (c)'s buffers of the last layer and its output bit-identical to (b)'s; the last
layer against torch (bench.py's output_check: act from the stored gate|up, down from the stored act, exact adds).

    python tools/layer_decode_bench.py [--steps 30] [--warmup 5] [--rounds 5] [--attention math|fast]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (shapes, byte accounting, seeded weights, graph capture and timing of the bench)
from tools.batched_decode_bench import _power_limit_w  # noqa: E402

HEADS, KV_HEADS, HEAD_DIM, CTX = 32, 8, 128, 1024
EPS = 1e-5


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--attention", choices=["math", "fast"], default="math",
                    help="stand-in backend: math (bit-reproducible: the (b) / (c) identity is checked) or torch's fused "
                         "backends (faster, not bit-reproducible from call to call)")
    a = ap.parse_args()

    import torch
    import torch.nn.functional as F
    from torch.nn.attention import SDPBackend, sdpa_kernel

    from autoawq_b200.program import DecodeProgram

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    rep = bench.Replica(dev, 1, seed=0)
    ext, H, I, L = rep.ext, bench.HIDDEN, bench.INTER, rep.layers
    f16 = torch.float16
    g = torch.Generator(device=dev).manual_seed(1)
    kv = [(torch.randn((1, KV_HEADS, CTX, HEAD_DIM), generator=g, device=dev, dtype=f16),
           torch.randn((1, KV_HEADS, CTX, HEAD_DIM), generator=g, device=dev, dtype=f16)) for _ in range(L)]
    norm1 = [(1 + 0.1 * torch.randn(H, generator=g, device=dev)).half() for _ in range(L)]
    norm2 = [(1 + 0.1 * torch.randn(H, generator=g, device=dev)).half() for _ in range(L)]
    h0 = rep.h.clone()
    ext.set_knob(4, 1)
    backends = [SDPBackend.MATH] if a.attention == "math" else [SDPBackend.FLASH_ATTENTION, SDPBackend.EFFICIENT_ATTENTION,
                                                                 SDPBackend.CUDNN_ATTENTION, SDPBackend.MATH]

    def attention(qkv, l, out):
        """The stand-in (see the module docstring), into `out` [1, H]."""
        q = qkv[:, :H].reshape(1, HEADS, 1, HEAD_DIM)
        with sdpa_kernel(backends):
            o = F.scaled_dot_product_attention(q, kv[l][0], kv[l][1], enable_gqa=True)
        out.copy_(o.reshape(1, H))

    def bufs():
        e = lambda n: torch.empty((1, n), dtype=f16, device=dev)  # noqa: E731
        return [dict(h=e(H), xn=e(H), attn=e(H), hm=e(H), xn2=e(H), act=e(I)) for _ in range(L)] + [dict(h=e(H))]

    # ---- (a) per-op
    Ba = bufs()
    Ba[0]["h"].copy_(h0)

    def step_a():
        h = Ba[0]["h"]
        for l in range(L):
            b, w = Ba[l], rep.w[l]
            ext.layernorm_forward_cuda(h, norm1[l], b["xn"], EPS)
            qkv = ext.gemm_forward_cuda(b["xn"], *w["qkv"], 8)
            attention(qkv, l, b["attn"])
            o = ext.gemm_forward_cuda(b["attn"], *w["o"], 8)
            torch.add(o, h, out=b["hm"])
            ext.layernorm_forward_cuda(b["hm"], norm2[l], b["xn2"], EPS)
            gu = ext.gemm_forward_cuda(b["xn2"], *w["gate_up"], 8)
            ext.silu_and_mul(b["act"], gu)
            dn = ext.gemm_forward_cuda(b["act"], *w["down"], 8)
            torch.add(dn, b["hm"], out=Ba[l + 1]["h"])
            h = Ba[l + 1]["h"]
        return h

    # ---- (b) three programs per layer + torch.add
    Bb = bufs()
    Bb[0]["h"].copy_(h0)
    plan_b = []
    for l in range(L):
        b, w = Bb[l], rep.w[l]
        p1, p2, p3 = DecodeProgram(), DecodeProgram(), DecodeProgram()
        p1.layernorm_forward_cuda(b["h"], norm1[l], b["xn"], EPS)
        b["qkv"] = p1.gemm_forward_cuda(b["xn"], *w["qkv"], 8)
        b["o"] = p2.gemm_forward_cuda(b["attn"], *w["o"], 8)
        p3.layernorm_forward_cuda(b["hm"], norm2[l], b["xn2"], EPS)
        b["gu"] = p3.gemm_forward_cuda(b["xn2"], *w["gate_up"], 8)
        p3.silu_and_mul(b["act"], b["gu"])
        b["down"] = p3.gemm_forward_cuda(b["act"], *w["down"], 8)
        for p in (p1, p2, p3):
            p.build()
            assert p.fused, "(b): a program did not fuse"
        plan_b.append((p1, p2, p3))

    def step_b():
        for l in range(L):
            b = Bb[l]
            p1, p2, p3 = plan_b[l]
            p1.run()
            attention(b["qkv"], l, b["attn"])
            p2.run()
            torch.add(b["o"], b["h"], out=b["hm"])
            p3.run()
            torch.add(b["down"], b["hm"], out=Bb[l + 1]["h"])
        return Bb[L]["h"]

    # ---- (c) attention-to-attention programs with the adds fused
    Bc = bufs()
    Bc[0]["h"].copy_(h0)
    p0 = DecodeProgram()
    p0.layernorm_forward_cuda(Bc[0]["h"], norm1[0], Bc[0]["xn"], EPS)
    Bc[0]["qkv"] = p0.gemm_forward_cuda(Bc[0]["xn"], *rep.w[0]["qkv"], 8)
    p0.build()
    assert p0.fused, "(c): the first program did not fuse"
    plan_c = [p0]
    for l in range(L):
        b, w = Bc[l], rep.w[l]
        p = DecodeProgram()
        b["o"] = p.gemm_forward_cuda(b["attn"], *w["o"], 8)
        p.add(b["o"], b["h"], out=b["hm"])
        p.layernorm_forward_cuda(b["hm"], norm2[l], b["xn2"], EPS)
        b["gu"] = p.gemm_forward_cuda(b["xn2"], *w["gate_up"], 8)
        p.silu_and_mul(b["act"], b["gu"])
        b["down"] = p.gemm_forward_cuda(b["act"], *w["down"], 8)
        p.add(b["down"], b["hm"], out=Bc[l + 1]["h"])
        if l + 1 < L:
            nb = Bc[l + 1]
            p.layernorm_forward_cuda(nb["h"], norm1[l + 1], nb["xn"], EPS)
            nb["qkv"] = p.gemm_forward_cuda(nb["xn"], *rep.w[l + 1]["qkv"], 8)
        p.build()
        assert p.fused and p.kernel_ops == (4 if l + 1 < L else 3), "(c): a segment did not fuse"
        plan_c.append(p)

    def step_c():
        plan_c[0].run()
        for l in range(L):
            attention(Bc[l]["qkv"], l, Bc[l]["attn"])
            plan_c[l + 1].run()
        return Bc[L]["h"]

    def step_attn():
        for l in range(L):
            attention(Bc[l]["qkv"], l, Bc[l]["attn"])

    graphs = {}
    for name, fn in (("a_per_op", step_a), ("b_three_programs_per_layer", step_b), ("c_fused_adds", step_c),
                     ("attention_stand_in", step_attn)):
        graphs[name], _ = bench.capture(torch, fn)

    # ---- self-checks (after one replay of each graph on identical inputs)
    for gph in graphs.values():
        gph.replay()
    torch.cuda.synchronize()
    ident_out = torch.equal(Bb[L]["h"], Bc[L]["h"])
    last = L - 1
    ident_last = all(torch.equal(Bb[last][k], Bc[last][k]) for k in ("h", "xn", "qkv", "attn", "o", "hm", "xn2", "gu",
                                                                        "act", "down"))
    ident_all_layers = all(torch.equal(Bb[l]["hm"], Bc[l]["hm"]) and torch.equal(Bb[l + 1]["h"], Bc[l + 1]["h"])
                           for l in range(L))
    first_diff = None                      # (layer, buffer) where (b) and (c) first differ, in step order
    for l in range(L):
        for k in ("h", "xn", "qkv", "attn", "o", "hm", "xn2", "gu", "act", "down"):
            if first_diff is None and not torch.equal(Bb[l][k], Bc[l][k]):
                first_diff = [l, k, float((Bb[l][k].float() - Bc[l][k].float()).abs().max())]
    b = Bc[last]
    lw = rep.w[last]
    gu_ref = torch.matmul(b["xn2"].float(), ext.dequantize_weights_cuda(*lw["gate_up"]).float())
    act_ref = F.silu(gu_ref[:, :I]) * gu_ref[:, I:]
    dn_ref = torch.matmul(b["act"].float(), ext.dequantize_weights_cuda(*lw["down"]).float())
    d_act = float((b["act"].float() - act_ref).abs().max())
    d_dn = float((b["down"].float() - dn_ref).abs().max())
    rms_act, rms_dn = float(act_ref.pow(2).mean().sqrt()), float(dn_ref.pow(2).mean().sqrt())
    adds_exact = torch.equal(Bc[L]["h"], torch.add(b["down"], b["hm"])) and torch.equal(b["hm"], torch.add(b["o"], b["h"]))
    d_a_vs_b = float((Ba[L]["h"].float() - Bb[L]["h"].float()).abs().max())
    checks = {"c_output_bit_identical_to_b": ident_out, "first_difference_b_vs_c": first_diff, "c_last_layer_buffers_bit_identical_to_b": ident_last,
              "c_every_layer_residual_stream_bit_identical_to_b": ident_all_layers,
              "last_layer_act_max_abs_diff_vs_torch": round(d_act, 6),
              "last_layer_down_max_abs_diff_vs_torch": round(d_dn, 6), "last_layer_adds_exact": adds_exact,
              "last_layer_consistent": bool(torch.isfinite(Bc[L]["h"]).all()) and d_act <= 0.03 * rms_act + 0.03
              and d_dn <= 0.03 * rms_dn + 0.03 and adds_exact,
              "a_output_max_abs_diff_vs_b": round(d_a_vs_b, 6), "output_rms": round(float(Bc[L]["h"].float().pow(2).mean().sqrt()), 4)}

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
    bytes_step = sum(bench.linear_bytes(K, N, 1) for _, K, N in bench.LINEARS) * L
    attn_ms = med["attention_stand_in"]
    table = {}
    for name in ("a_per_op", "b_three_programs_per_layer", "c_fused_adds"):
        ms = med[name]
        table[name] = {"ms_per_step": round(ms, 4), "tok_s": round(1e3 / ms, 1),
                       "ms_without_attention": round(ms - attn_ms, 4), "tok_s_without_attention": round(1e3 / (ms - attn_ms), 1),
                       "gbs_without_attention": round(bytes_step / (ms - attn_ms) / 1e6, 1),
                       "rounds_ms": [round(t, 4) for t in times[name]]}
    table["c_vs_b"] = round(med["b_three_programs_per_layer"] / med["c_fused_adds"], 3)
    print(json.dumps({"tool": "layer_decode_bench", "workload": "Llama-3-8B decode bs=1, 32 layers with residual adds, "
                      "g128, seeded random weights; attention = SDPA stand-in over a fixed 1024-position KV cache",
                      "card": torch.cuda.get_device_name(dev), "power_limit_w": _power_limit_w(0),
                      "clocks_during_timing": clocks, "steps": a.steps, "warmup": a.warmup, "rounds": a.rounds,
                      "alg_bytes_per_step": bytes_step, "attention_stand_in_ms": round(attn_ms, 4), "attention_backend": a.attention,
                      "launches_per_step_besides_attention": {"a_per_op": 9 * L, "b_three_programs_per_layer": 5 * L,
                                                              "c_fused_adds": 1 + L},
                      "variants": table, "checks": checks}), flush=True)


if __name__ == "__main__":
    main()
