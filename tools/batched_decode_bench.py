#!/usr/bin/env python
"""Batched decode programs on the Llama-3-8B decode chain of bench.py: one JSON line.

For M in {1, 2, 4, 8} token rows per step (a fused block built for batch size M) it times
  * the decode program created with DecodeProgram(max_tokens=M) (csrc/program_batch.cuh for M > 1), or reports "per-op"
    where the sequence does not fuse,
  * the per-op CUDA graph of the same step (PDL on, as bench.py runs it),
and reports tok/s (= M / step time), algorithmic GB/s (bench.py's byte accounting) and its fraction of the 3.35 TB/s
H100 SXM data sheet, a last-layer check against torch (bench.py's), the per-token bit identity against M = 1 stream
programs on each token's row, and per-op phase timestamps of the fused kernel (knob 3 = 2: source rows polled,
activations staged, units done, outputs published; median over the first 8 CTAs, per linear of the layer).
The card name, its power limit and the SM clock during the timed program replays are recorded in the same run.

    python tools/batched_decode_bench.py [--steps 30] [--warmup 5] [--tokens 1,2,4,8] [--identity-tokens 8]
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

import bench  # noqa: E402  (shapes, byte accounting, seeded weights, graph capture and timing of the bench)

DATASHEET_GBS = 3350.0


def _power_limit_w(index):
    try:
        import pynvml as nv

        nv.nvmlInit()
        return round(nv.nvmlDeviceGetEnforcedPowerLimit(nv.nvmlDeviceGetHandleByIndex(index)) / 1000.0, 1)
    except Exception:  # noqa: BLE001
        pass
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(index)],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:  # noqa: BLE001
        return None


def _set_rows(rep, M, h):
    """Point the replica's step buffers at M token rows (the weights stay)."""
    torch = rep.torch
    rep.M = M
    rep.xn = torch.empty((M, bench.HIDDEN), dtype=torch.float16, device=rep.dev)
    rep.act = torch.empty((M, bench.INTER), dtype=torch.float16, device=rep.dev)
    rep.h = h.clone()


def _last_layer_check(rep, y):
    """bench.py's check: the stored act and the step's output against torch on the last layer's own inputs."""
    torch = rep.torch
    torch.cuda.synchronize()
    xn, act, yt = rep.xn.float(), rep.act.float(), y.float()
    lw = rep.w[-1]
    gu = torch.matmul(xn, rep.ext.dequantize_weights_cuda(*lw["gate_up"]).float())
    act_ref = torch.nn.functional.silu(gu[:, :bench.INTER]) * gu[:, bench.INTER:]
    y_ref = torch.matmul(act, rep.ext.dequantize_weights_cuda(*lw["down"]).float())
    d_act, d_y = float((act - act_ref).abs().max()), float((yt - y_ref).abs().max())
    rms_act, rms_y = float(act_ref.pow(2).mean().sqrt()), float(y_ref.pow(2).mean().sqrt())
    return {"act_max_abs_diff": round(d_act, 6), "output_max_abs_diff": round(d_y, 6),
            "consistent": bool(torch.isfinite(yt).all()) and d_act <= 0.03 * rms_act + 0.03 and d_y <= 0.03 * rms_y + 0.03}


def _phases(lib, n_layers_ops=32):
    """knob 3 = 2 stamps of the last run: [op][cta][slot] ns, slots 0 begin, 1 source polled, 2 staged, 3 first chunk
    landed, 4 warp 0 done, 5 all warps done, 6 published.  Median over the 8 recorded CTAs, averaged per linear of a layer."""
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
    for li, (name, _, _) in enumerate(bench.LINEARS):
        rows = []
        for op in range(li, min(n_layers_ops, 32), 4):
            s = t[op]
            if (s[:, :7] == 0).any():
                continue
            rows.append([np.median(s[:, 1] - s[:, 0]), np.median(s[:, 2] - s[:, 1]), np.median(s[:, 5] - s[:, 2]),
                         np.median(s[:, 6] - s[:, 5]), np.median(s[:, 6] - s[:, 0])])
        if rows:
            r = np.mean(np.array(rows), axis=0) / 1e3
            out[name] = {"poll_us": round(r[0], 2), "stage_us": round(r[1], 2), "units_us": round(r[2], 2),
                         "finish_us": round(r[3], 2), "op_us": round(r[4], 2)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--tokens", default="1,2,4,8")
    ap.add_argument("--identity-tokens", type=int, default=8, help="tokens per M checked against M = 1 programs")
    a = ap.parse_args()

    import torch

    from autoawq_b200._cabi import lib
    from autoawq_b200.program import DecodeProgram

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    Ms = [int(x) for x in a.tokens.split(",")]
    rep = bench.Replica(dev, max(Ms), seed=0)
    h_all = rep.h.clone()
    rep.ext.set_knob(4, 1)     # the per-op graph runs with PDL, as in bench.py
    sampler = bench.ClockSampler(0)
    sampler.start()
    t_lo = t_hi = None
    res = {}
    for M in Ms:
        _set_rows(rep, M, h_all[:M])
        bytes_step = sum(bench.linear_bytes(K, N, M) for _, K, N in bench.LINEARS) * rep.layers
        g_ops, out_ops = bench.capture(torch, lambda: rep.step(rep.h))
        ms_ops = bench.timed(torch, g_ops.replay, a.steps, a.warmup) / a.steps * 1e3
        del g_ops, out_ops
        row = {"per_op_graph_ms": round(ms_ops, 4), "per_op_graph_tok_s": round(M / ms_ops * 1e3, 1),
               "per_op_graph_gbs": round(bytes_step / ms_ops / 1e6, 1)}
        prog = DecodeProgram(max_tokens=M)
        y = rep.step(rep.h, api=prog)
        prog.build()
        row["program_kind"] = prog.kind
        if prog.fused:
            g, _ = bench.capture(torch, prog.run)
            t0 = time.time()
            ms = bench.timed(torch, g.replay, a.steps, a.warmup) / a.steps * 1e3
            t1 = time.time()
            t_lo = t0 if t_lo is None else t_lo
            t_hi = t1
            gbs = bytes_step / ms / 1e6
            row.update({"program_ms": round(ms, 4), "program_tok_s": round(M / ms * 1e3, 1), "program_gbs": round(gbs, 1),
                        "program_frac_of_datasheet": round(gbs / DATASHEET_GBS, 4),
                        "program_vs_per_op_graph": round(ms_ops / ms, 3)})
            row["last_layer_check"] = _last_layer_check(rep, y)
            # per-op phases: one more (untimed) run with the stamps on
            lib.b200awq_set_knob(3, 2)
            try:
                prog.run()
                torch.cuda.synchronize()
            finally:
                lib.b200awq_set_knob(3, 0)
            row["phases_first_8_layers"] = _phases(lib)
            del g
            if M > 1:
                # token m of the batched run against an M = 1 stream program on row m alone (same inputs, same weights)
                y_b, act_b = y.clone(), rep.act.clone()
                prog.close()
                rep.ext.set_knob(14, 2)
                same = True
                try:
                    for m in range(min(M, a.identity_tokens)):
                        _set_rows(rep, 1, h_all[m:m + 1])
                        p1 = DecodeProgram()
                        y1 = rep.step(rep.h, api=p1)
                        p1.build()
                        p1.run()
                        torch.cuda.synchronize()
                        same = same and torch.equal(y1, y_b[m:m + 1]) and torch.equal(rep.act, act_b[m:m + 1])
                        p1.close()
                finally:
                    rep.ext.set_knob(14, 0)
                row["tokens_bit_identical_to_m1_program"] = bool(same)
        else:
            row["program_ms"] = "per-op"
            row["program_tok_s"] = "per-op"
        prog.close()
        res[str(M)] = row
        torch.cuda.empty_cache()
    clocks = sampler.stop(t_lo, t_hi) if t_lo is not None else None
    print(json.dumps({"tool": "batched_decode_bench", "workload": "bench.py Llama-3-8B decode chain (32 layers, g128, "
                      "seeded random weights), M token rows per step", "card": torch.cuda.get_device_name(dev),
                      "power_limit_w": _power_limit_w(0), "clocks_during_program_replays": clocks, "steps": a.steps,
                      "warmup": a.warmup, "datasheet_gbs": DATASHEET_GBS, "by_tokens": res}), flush=True)


if __name__ == "__main__":
    main()
