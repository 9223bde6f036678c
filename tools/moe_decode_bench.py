#!/usr/bin/env python
"""Sparse-MoE decode programs on the Mixtral-8x7B decode step of bench.py's Mixtral leg: one JSON line.

The step is the leg's: 32 layers of RMSNorm -> qkv 4096x6144 -> o 4096x4096 -> RMSNorm -> sparse-MoE block (8 experts,
top-2, I = 14336, g128), the same seeded weights and input (bench.py:mixtral_leg).  It is timed two ways:
  * as a decode program (DecodeProgram.sparse_moe per layer: one persistent kernel, 4 kernel ops per layer),
  * as the per-op CUDA graph of the leg's call sequence with PDL on (13 launches per layer),
and reports ms/step, tok/s and GB/s over the active bytes (bench.py's accounting: the two selected experts per layer),
the per-op phase timestamps of the MoE ops (knob 3 = 2, first 8 layers: source polled, staged, routing published,
units, finish) and the last layer's self-consistency check (routing against its own logits, output against torch on
our dequantised experts).  The card name, its power limit and the SM clock during the timed program replays are
recorded in the same run.

    python tools/moe_decode_bench.py [--steps 30] [--warmup 5] [--layers 32]
"""
import argparse
import ctypes
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (shapes, byte accounting, graph capture, timing and the clock sampler of the bench)
from tools.batched_decode_bench import DATASHEET_GBS, _power_limit_w  # noqa: E402


def _weights(torch, dev, layers):
    """bench.py:mixtral_leg's weights and input, drawn in the same order from the same seed."""
    E, H, I, QKV, G = 8, bench.HIDDEN, bench.INTER, 6144, bench.GROUP
    g = torch.Generator(device=dev).manual_seed(4242)

    def lin(K, N):
        return (torch.randint(-2**31, 2**31 - 1, (K, N // 8), dtype=torch.int32, device=dev, generator=g),
                ((torch.rand((K // G, N), device=dev, generator=g) * 0.5 + 0.75) / (6.1 * K**0.5)).half(),
                torch.randint(-2**31, 2**31 - 1, (K // G, N // 8), dtype=torch.int32, device=dev, generator=g))

    def stacked(K, N):
        return (torch.randint(-2**31, 2**31 - 1, (E, K, N // 8), dtype=torch.int32, device=dev, generator=g),
                ((torch.rand((E, K // G, N), device=dev, generator=g) * 0.5 + 0.75) / (6.1 * K**0.5)).half(),
                torch.randint(-2**31, 2**31 - 1, (E, K // G, N // 8), dtype=torch.int32, device=dev, generator=g))

    ws = [dict(qkv=lin(H, QKV), o=lin(H, H), w13=stacked(H, 2 * I), w2=stacked(I, H),
               router=(torch.randn((H, E), device=dev, generator=g) * 0.05).half()) for _ in range(layers)]
    h0 = torch.randn((1, H), device=dev, dtype=torch.float16, generator=g)
    return ws, h0


def _phases(lib, layers):
    """knob 3 = 2 stamps of the last run: [op][cta][slot] ns (first 32 kernel ops = 8 layers x [qkv, o, gate|up, down]).
    Median over the 8 recorded CTAs, averaged over the recorded layers."""
    import numpy as np

    buf = np.zeros(32 * 8 * 8, dtype=np.uint64)
    prev = lib.b200awq_get_knob(3)
    lib.b200awq_set_knob(3, 2)
    try:
        assert lib.b200awq_debug_read(buf.ctypes.data_as(ctypes.c_void_p), buf.nbytes) == 0
    finally:
        lib.b200awq_set_knob(3, prev)
    t = buf.reshape(32, 8, 8).astype(np.int64)
    out = {}
    for j, name in enumerate(["qkv", "o", "moe_gate_up", "moe_down"]):
        rows = []
        for op in range(j, min(4 * layers, 32), 4):
            s = t[op]
            if (s[:, :7] == 0).any():
                continue
            r = [np.median(s[:, 1] - s[:, 0]), np.median(s[:, 2] - s[:, 1]), np.median(s[:, 5] - s[:, 2]),
                 np.median(s[:, 6] - s[:, 5]), np.median(s[:, 6] - s[:, 0])]
            if name == "moe_gate_up":
                r.append(np.median(s[:, 7] - s[:, 2]))      # staged -> routing published
                r.append(np.median(s[:, 3] - s[:, 2]))      # staged -> first expert chunk landed (warp 0)
            rows.append(r)
        if rows:
            r = np.mean(np.array(rows), axis=0) / 1e3
            d = {"poll_us": round(r[0], 2), "stage_us": round(r[1], 2), "units_us": round(r[2], 2),
                 "finish_us": round(r[3], 2), "op_us": round(r[4], 2)}
            if name == "moe_gate_up":
                d["routing_us"] = round(r[5], 2)
                d["first_expert_chunk_us"] = round(r[6], 2)
            out[name] = d
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--layers", type=int, default=32)
    a = ap.parse_args()

    import torch

    import awq_ext
    from autoawq_b200 import ext
    from autoawq_b200._cabi import lib
    from autoawq_b200.program import DecodeProgram

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    E, H, I, topk, QKV, G = 8, bench.HIDDEN, bench.INTER, 2, 6144, bench.GROUP
    ws, h0 = _weights(torch, dev, a.layers)
    nw = torch.ones(H, dtype=torch.float16, device=dev)

    # ---- per-op CUDA graph (PDL on), the leg's call sequence
    xn = torch.empty((1, H), dtype=torch.float16, device=dev)
    tw = torch.empty((1, topk), dtype=torch.float32, device=dev)
    tid = torch.empty((1, topk), dtype=torch.int32, device=dev)
    src = torch.empty((1, topk), dtype=torch.int32, device=dev)
    s_ids = torch.empty((topk + E * 15,), dtype=torch.int32, device=dev)
    e_ids = torch.empty((topk + E,), dtype=torch.int32, device=dev)
    npost = torch.empty((1,), dtype=torch.int32, device=dev)
    act = torch.empty((1, topk, I), dtype=torch.float16, device=dev)

    def step():
        h = h0
        for w in ws:
            awq_ext.layernorm_forward_cuda(h, nw, xn, 1e-5)
            qkv = awq_ext.gemm_forward_cuda(xn, *w["qkv"], 8)
            o = awq_ext.gemm_forward_cuda(qkv[:, :H], *w["o"], 8)
            awq_ext.layernorm_forward_cuda(o, nw, xn, 1e-5)
            logits = torch.matmul(xn, w["router"]).float()
            awq_ext.topk_softmax(tw, tid, src, logits)
            s_ids.fill_(topk)
            awq_ext.moe_alig_block_size(tid, E, 16, s_ids, e_ids, npost)
            gu = awq_ext.grouped_gemm_forward(xn.view(1, 1, H), *w["w13"], tw, s_ids, e_ids, npost, False, 8)
            awq_ext.silu_and_mul(act, gu)
            out = awq_ext.grouped_gemm_forward(act, *w["w2"], tw, s_ids, e_ids, npost, True, 8)
            h = torch.sum(out, dim=1)
        return h

    pdl_was = ext.get_knob(4)
    ext.set_knob(4, 1)
    g_ops, _ = bench.capture(torch, step)
    ms_ops = bench.timed(torch, g_ops.replay, a.steps, a.warmup) / a.steps * 1e3
    ext.set_knob(4, pdl_was)
    del g_ops
    torch.cuda.empty_cache()

    # ---- the decode program (the router weight is the nn.Linear weight [E, H] = the leg's [H, E] transposed)
    prog = DecodeProgram()
    h_in = h0.clone()
    h = h_in
    last = None
    for w in ws:
        xa = torch.empty((1, H), dtype=torch.float16, device=dev)
        prog.layernorm_forward_cuda(h, nw, xa, 1e-5)
        qkv = prog.gemm_forward_cuda(xa, *w["qkv"], 8)
        o = prog.gemm_forward_cuda(qkv[:, :H], *w["o"], 8)
        xb = torch.empty((1, H), dtype=torch.float16, device=dev)
        prog.layernorm_forward_cuda(o, nw, xb, 1e-5)
        h = prog.sparse_moe(xb, w["router"].t().contiguous(), w["w13"], w["w2"], topk)
        last = (xb, w)
    t_build = time.time()
    prog.build()
    t_build = time.time() - t_build
    res = {"program_kind": prog.kind, "program_kernel_ops": prog.kernel_ops, "program_build_s": round(t_build, 1)}
    sampler = bench.ClockSampler(0)
    sampler.start()
    t0 = t1 = None
    if prog.fused:
        g, _ = bench.capture(torch, prog.run)
        t0 = time.time()
        ms = bench.timed(torch, g.replay, a.steps, a.warmup) / a.steps * 1e3
        t1 = time.time()
        del g
    else:
        ms = bench.timed(torch, prog.run, a.steps, a.warmup) / a.steps * 1e3
    clocks = sampler.stop(t0, t1) if t0 is not None else None
    wb = lambda K, N: K * N // 2 + (K // G) * N * 2 + (K // G) * N // 2  # noqa: E731
    active = a.layers * (wb(H, QKV) + wb(H, H) + topk * (wb(H, 2 * I) + wb(I, H)))
    res.update({"program_ms": round(ms, 4), "program_tok_s": round(1e3 / ms, 1),
                "program_gbs_over_active": round(active / ms / 1e6, 1),
                "program_frac_of_datasheet": round(active / ms / 1e6 / DATASHEET_GBS, 4),
                "per_op_graph_ms": round(ms_ops, 4), "per_op_graph_tok_s": round(1e3 / ms_ops, 1),
                "per_op_graph_gbs_over_active": round(active / ms_ops / 1e6, 1),
                "program_vs_per_op_graph": round(ms_ops / ms, 3), "active_gb_per_step": round(active / 1e9, 3)})
    if prog.fused:
        lib.b200awq_set_knob(3, 2)
        try:
            prog.run()
            torch.cuda.synchronize()
        finally:
            lib.b200awq_set_knob(3, 0)
        res["phases_first_8_layers"] = _phases(lib, a.layers)
    # ---- the last layer against its own inputs (bench.py's Mixtral-leg check)
    prog.run()
    torch.cuda.synchronize()
    b = prog.moe_buffers(a.layers - 1)
    xb, wl = last
    probs = torch.softmax(torch.matmul(xb, wl["router"]).float(), dim=-1)
    want = sorted(int(v) for v in torch.topk(probs, topk, dim=-1).indices.flatten().tolist())
    got = [int(v) for v in b["topk_ids"].flatten().tolist()]
    ref = torch.zeros((1, H), dtype=torch.float32, device=dev)
    for k, e in enumerate(got):
        w13 = ext.dequantize_weights_cuda(wl["w13"][0][e], wl["w13"][1][e], wl["w13"][2][e], 0, 0, 0, False)
        w2 = ext.dequantize_weights_cuda(wl["w2"][0][e], wl["w2"][1][e], wl["w2"][2][e], 0, 0, 0, False)
        gu = torch.matmul(xb.float(), w13.float())
        a_k = (torch.nn.functional.silu(gu[:, :I]) * gu[:, I:]).half().float()
        ref += b["topk_weights"][0, k] * torch.matmul(a_k, w2.float()).half().float()
    out = b["out"].float()
    rms = float(ref.pow(2).mean().sqrt())
    diff = float((out - ref).abs().max())
    res["last_layer_check"] = {"experts": sorted(got), "routing_matches_its_logits": sorted(got) == want,
                               "moe_max_abs_diff_vs_torch": round(diff, 5), "output_rms": round(rms, 4),
                               "consistent": bool(torch.isfinite(out).all()) and sorted(got) == want
                               and diff <= 0.03 * rms + 0.02}
    prog.close()
    print(json.dumps({"tool": "moe_decode_bench", "workload": f"bench.py Mixtral-8x7B decode step ({a.layers} layers, "
                      "E = 8, top-2, g128, seeded random weights), bs = 1", "card": torch.cuda.get_device_name(dev),
                      "power_limit_w": _power_limit_w(0), "clocks_during_program_replays": clocks, "steps": a.steps,
                      "warmup": a.warmup, "datasheet_gbs": DATASHEET_GBS, "result": res}), flush=True)


if __name__ == "__main__":
    main()
