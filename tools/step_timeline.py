#!/usr/bin/env python
"""Where the time of bench.py's decode step goes: per-op phase timeline and timed variants of the one-launch step.

The step is bench.py's own: `bench.Replica` (same seeds, shapes and weights) recorded once into a DecodeProgram, which
runs the Llama-3-8B bs = 1 step (32 layers x [RMSNorm, qkv, o, RMSNorm, gate|up, SiLU*mul, down]) as one stream
kernel launch.  One run prints one JSON line with three parts:

  timeline  the program run with knob 3 = 2, stamps read back with b200awq_debug_read (g_prog_dbg: the first 8 CTAs,
            the first 32 kernel ops = 8 layers).  Per op type (qkv / o / gate|up / down) and phase, the median over
            (layer, CTA) samples of the phase time, and the median over layers of its max - min across the 8 CTAs, in us:
              poll         [1] - [0]  waiting for the source row (the grid-wide hand-off) / reading the input
              staging      [2] - [1]  RMSNorm and the B-fragment store of the activations
              first_chunk  [3] - [2]  until consumer warp 0's first ring stage has landed
              units        [5] - [3]  the unit loop of all warps (up to the post-loop barrier)
              publish      [6] - [5]  reduction of the warps' partial sums and the hand-off stores
              op           [6] - [0]
  timings   every variant (--variant NAME=KNOB:VALUE,...: library knobs set while its CUDA graph is captured) replayed
            alternately, `rounds` x `steps` replays each after warm-up; median and range of ms/step, GB/s over the
            step's algorithmic bytes (bench.linear_bytes: 3.63 GB)
  record    card name, power limit, and the SM clock sampled during the timed replays

    python tools/step_timeline.py [--steps 30] [--warmup 5] [--rounds 5] [--variant off=8:-1 --variant l2_16mb=8:16 ...]
"""
import argparse
import ctypes
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (shapes, byte accounting, seeded weights, graph capture and timing of the bench)
from tools.batched_decode_bench import _power_limit_w  # noqa: E402

OP_TYPES = ("qkv", "o", "gate_up", "down")   # kernel op i of the bench step is OP_TYPES[i % 4]
PHASES = (("poll", 0, 1), ("staging", 1, 2), ("first_chunk", 2, 3), ("units", 3, 5), ("publish", 5, 6), ("op", 0, 6))
DBG_OPS, DBG_CTAS, DBG_SLOTS = 32, 8, 8


def parse_variant(s):
    name, _, spec = s.partition("=")
    knobs = {}
    for kv in filter(None, spec.split(",")):
        k, v = kv.split(":")
        knobs[int(k)] = int(v)
    return name, knobs


def timeline(torch, ext, prog, runs):
    """Stamps of `runs` program runs (knob 3 = 2), reduced per op type and phase."""
    import numpy as np

    from autoawq_b200._cabi import check, lib

    buf = np.zeros(DBG_OPS * DBG_CTAS * DBG_SLOTS, dtype=np.uint64)
    was = ext.get_knob(3)
    samples = {t: {p[0]: [] for p in PHASES} for t in OP_TYPES}
    spreads = {t: {p[0]: [] for p in PHASES} for t in OP_TYPES}
    try:
        ext.set_knob(3, 2)
        for _ in range(runs):
            prog.run()
            torch.cuda.synchronize()
            check(lib.b200awq_debug_read(buf.ctypes.data_as(ctypes.c_void_p), buf.nbytes), "b200awq_debug_read")
            st = buf.reshape(DBG_OPS, DBG_CTAS, DBG_SLOTS).astype(np.int64)
            for op in range(DBG_OPS):
                t = OP_TYPES[op % 4]
                for name, a, b in PHASES:
                    d = (st[op, :, b] - st[op, :, a]) / 1e3
                    samples[t][name].extend(d.tolist())
                    spreads[t][name].append(float(d.max() - d.min()))
    finally:
        ext.set_knob(3, was)
    med = lambda v: float(np.median(v)) if v else None  # noqa: E731
    return {t: {name: {"median_us": round(med(samples[t][name]), 3), "cta_spread_us": round(med(spreads[t][name]), 3)}
                for name, _, _ in PHASES} for t in OP_TYPES}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--timeline-runs", type=int, default=5, help="program runs whose stamps are pooled")
    ap.add_argument("--variant", action="append", default=[],
                    help="NAME=KNOB:VALUE[,KNOB:VALUE...] (repeatable); default: one variant with the library defaults")
    a = ap.parse_args()
    variants = [parse_variant(v) for v in a.variant] or [("default", {})]

    import torch

    from autoawq_b200.program import DecodeProgram

    if not torch.cuda.is_available():
        raise SystemExit("step_timeline.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    rep = bench.Replica(dev, 1, seed=0)
    ext = rep.ext
    ext.set_knob(4, 1)     # bench.py's default (--pdl 1)
    prog = DecodeProgram()
    rep.step(rep.h, api=prog)
    prog.build()
    if not prog.fused:
        raise SystemExit("the bench step did not build as one fused program")
    alg_bytes = sum(bench.linear_bytes(K, N, 1) for _, K, N in bench.LINEARS) * rep.layers

    for _ in range(a.warmup):
        prog.run()
    torch.cuda.synchronize()
    tl = timeline(torch, ext, prog, a.timeline_runs)

    graphs = {}
    for name, knobs in variants:
        was = {k: ext.get_knob(k) for k in knobs}
        try:
            for k, v in knobs.items():
                ext.set_knob(k, v)
            graphs[name], _ = bench.capture(torch, prog.run)
        finally:
            for k, v in was.items():
                ext.set_knob(k, v)
    for g in graphs.values():
        for _ in range(a.warmup):
            g.replay()
    torch.cuda.synchronize()
    sampler = bench.ClockSampler(0)
    sampler.start()
    times = {k: [] for k in graphs}
    t0 = time.time()
    for _ in range(a.rounds):
        for name, g in graphs.items():
            times[name].append(bench.timed(torch, g.replay, a.steps, 0) / a.steps * 1e3)
    t1 = time.time()
    clocks = sampler.stop(t0, t1)
    table = {}
    for name, knobs in variants:
        v = sorted(times[name])
        ms = v[len(v) // 2]
        table[name] = {"knobs": {str(k): x for k, x in knobs.items()}, "ms_per_step": round(ms, 4),
                       "ms_range": [round(v[0], 4), round(v[-1], 4)], "gb_s": round(alg_bytes / (ms * 1e-3) / 1e9, 1),
                       "tok_s": round(1e3 / ms, 1)}
    print(json.dumps({"tool": "step_timeline", "workload": "bench.py decode step (Llama-3-8B W4A16 g128, bs=1, "
                      f"{rep.layers} layers) as one decode-program launch", "alg_bytes": alg_bytes,
                      "card": torch.cuda.get_device_name(dev), "power_limit_w": _power_limit_w(0),
                      "clocks_during_timing": clocks, "steps": a.steps, "warmup": a.warmup, "rounds": a.rounds,
                      "timeline_us": tl, "timings": table}), flush=True)
    for t in OP_TYPES:
        print(f"{t:8s} " + "  ".join(f"{n} {tl[t][n]['median_us']:7.2f} ({tl[t][n]['cta_spread_us']:5.2f})"
                                     for n, _, _ in PHASES), file=sys.stderr)


if __name__ == "__main__":
    main()
