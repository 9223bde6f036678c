#!/usr/bin/env python
"""grouped_gemm_forward at prefill sizes, Mixtral-8x7B shapes (E = 8, top-2, 4096 -> 28672 gate|up, 14336 -> 4096 down,
g128, seeded random weights): which kernel should serve which token count.

For T in {16 .. 4096} tokens and two routings (a random router; fully skewed: every token on experts 0 and 1) it times
  * the reference's apply_moe_weights sequence over awq_ext (moe.py:45-91: moe_alig_block_size, gate|up grouped GEMM,
    silu_and_mul, down grouped GEMM with the routing weights, sum over the top-k), and
  * the gate|up and the down call alone,
under knob 12 = 0 (default routing), 1 (the decode-sized kernels: the ring GEMV where its workspace fits, else the
register-staged kernel), 2 (register-staged) and 3 (the grouped wgmma kernel), and the dense gemm_forward_cuda at
M = T * topk / E rows on one expert's weights.  TFLOP/s is 2 * T * topk * K * N over the call's time.

Measurement: `--layers` layers of distinct weights visited in turn (one layer's experts are 705 MB, far beyond the
50 MB L2), a warm-up pass per variant, `--rounds` rounds in which the variants alternate, CUDA events around each
variant's pass; medians with the [min, max] over rounds.  Card, power limit, SM clock and throttle reasons are read
(never set) in the same run.  Before anything is printed, the outputs under knob 12 = 3 are checked against knob 12 = 2
with the tolerance of tests/test_gpu_moe.py.

    python tools/moe_prefill_bench.py [--tokens 16,32,...] [--rounds 5] [--layers 2] [--out result.json]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (the clock sampler of the bench)
from tools.batched_decode_bench import _power_limit_w  # noqa: E402

E, TOPK, H, I, G = 8, 2, 4096, 14336, 128
VARIANTS = {"default": 0, "decode-kernels": 1, "staged": 2, "wgmma": 3}
RTOL, WR = 2.0**-10, 2.0**-11


def _stacked(torch, dev, g, K, N):
    return (torch.randint(-2**31, 2**31 - 1, (E, K, N // 8), dtype=torch.int32, device=dev, generator=g),
            ((torch.rand((E, K // G, N), device=dev, generator=g) * 0.5 + 0.75) / (6.1 * K**0.5)).half(),
            torch.randint(-2**31, 2**31 - 1, (E, K // G, N // 8), dtype=torch.int32, device=dev, generator=g))


def _routing(torch, dev, g, T, skewed):
    if skewed:
        return torch.tensor([[0, 1]], dtype=torch.int32, device=dev).repeat(T, 1)
    logits = torch.randn((T, E), device=dev, generator=g)
    return torch.topk(logits, TOPK, dim=-1).indices.to(torch.int32)


def _median_range(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", default="16,32,64,128,256,512,1024,4096")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--layers", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()

    import torch

    import awq_ext
    from autoawq_b200 import ext

    if not torch.cuda.is_available():
        raise SystemExit("moe_prefill_bench needs a CUDA device: there is nothing to time without one")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    gen = torch.Generator(device=dev).manual_seed(777)
    layers = [dict(w13=_stacked(torch, dev, gen, H, 2 * I), w2=_stacked(torch, dev, gen, I, H)) for _ in range(a.layers)]

    def align(tid):
        s_ids = torch.empty((tid.numel() + E * 15,), dtype=torch.int32, device=dev)
        e_ids = torch.empty((tid.numel() + E,), dtype=torch.int32, device=dev)
        npost = torch.empty((1,), dtype=torch.int32, device=dev)
        s_ids.fill_(tid.numel())
        awq_ext.moe_alig_block_size(tid, E, 16, s_ids, e_ids, npost)
        return s_ids, e_ids, npost

    def gate_up(w, x, tw, tabs):
        return awq_ext.grouped_gemm_forward(x.view(x.shape[0], 1, H), *w["w13"], tw, *tabs, False, 8)

    def down(w, act, tw, tabs):
        return awq_ext.grouped_gemm_forward(act, *w["w2"], tw, *tabs, True, 8)

    def sequence(w, x, tw, tid):
        tabs = align(tid)
        gu = gate_up(w, x, tw, tabs)
        act = torch.empty(gu.shape[:-1] + (I,), dtype=x.dtype, device=dev)
        awq_ext.silu_and_mul(act, gu)
        return torch.sum(down(w, act, tw, tabs), dim=1)

    def one_pass(fn):
        """ms per layer of one pass over the layers."""
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for w in layers:
            fn(w)
        t1.record()
        t1.synchronize()
        return t0.elapsed_time(t1) / len(layers)

    def alternate(fns):
        """{name: [ms per layer, one per round]}: a warm-up pass each, then rounds in which the variants alternate."""
        for name, fn in fns.items():
            ext.set_knob(12, VARIANTS.get(name, 0))
            one_pass(fn)
        out = {name: [] for name in fns}
        for _ in range(a.rounds):
            for name, fn in fns.items():
                ext.set_knob(12, VARIANTS.get(name, 0))
                out[name].append(one_pass(fn))
        ext.set_knob(12, 0)
        return out

    def check(T, x, tw, tid, tabs, act):
        """knob 12 = 3 against knob 12 = 2 on layer 0, both calls: |a - b| <= 2 (RTOL |b| + WR |x| . |W| w) + 1e-6."""
        w = layers[0]
        res = {}
        for name, call, xin, (qw, sc, qz), per_slot, mul in (
                ("gate_up", lambda: gate_up(w, x, tw, tabs), x.view(T, 1, H), w["w13"], False, False),
                ("down", lambda: down(w, act, tw, tabs), act, w["w2"], True, True)):
            ext.set_knob(12, VARIANTS["wgmma"])
            y_new = call()
            ext.set_knob(12, VARIANTS["staged"])
            y_old = call()
            ext.set_knob(12, 0)
            ok = True
            worst = 0.0
            for e in range(E):
                t, k = torch.nonzero(tid == e, as_tuple=True)
                if t.numel() == 0:
                    continue
                w_abs = ext.dequantize_weights_cuda(qw[e], sc[e], qz[e]).abs().float()
                budget = xin[t, k if per_slot else 0].abs().float() @ w_abs
                if mul:
                    budget = budget * tw[t, k][:, None]
                p, q = y_new[t, k].float(), y_old[t, k].float()
                excess = (p - q).abs() - (2 * RTOL * q.abs() + 2 * WR * budget + 1e-6)
                ok = ok and bool((excess <= 0).all()) and bool(torch.isfinite(p).all())
                worst = max(worst, float((p - q).abs().max()))
            res[name] = {"within_tolerance": ok, "max_abs_diff": worst}
        return res

    sampler = bench.ClockSampler(0)
    sampler.start()
    t_begin = time.time()
    rows = []
    all_ok = True
    for skewed in (False, True):
        for T in [int(v) for v in a.tokens.split(",")]:
            x = torch.randn((T, H), device=dev, generator=gen).half()
            tid = _routing(torch, dev, gen, T, skewed)
            tw = torch.rand((T, TOPK), device=dev, generator=gen) + 0.1
            tw = (tw / tw.sum(dim=-1, keepdim=True)).contiguous()
            tabs = align(tid)
            act = (torch.randn((T, TOPK, I), device=dev, generator=gen) * 0.5).half()
            chk = check(T, x, tw, tid, tabs, act)
            all_ok = all_ok and all(c["within_tolerance"] for c in chk.values())
            row = {"T": T, "routing": "skewed (2 experts)" if skewed else "random router", "self_check": chk}
            for what, fn_of, flop in (
                    ("sequence", lambda: (lambda w: sequence(w, x, tw, tid)), None),
                    ("gate_up", lambda: (lambda w: gate_up(w, x, tw, tabs)), 2.0 * T * TOPK * H * 2 * I),
                    ("down", lambda: (lambda w: down(w, act, tw, tabs)), 2.0 * T * TOPK * I * H)):
                ms = alternate({name: fn_of() for name in VARIANTS})
                row[what] = {}
                for name, xs in ms.items():
                    r = _median_range(xs)
                    row[what][name] = {"ms": {k: round(v, 4) for k, v in r.items()}}
                    if flop is not None:
                        row[what][name]["tflops"] = round(flop / (r["median"] * 1e-3) / 1e12, 2)
            # dense GEMM of the same shapes at the average run length, one expert's weights per layer visit
            M = max(1, T * TOPK // E)
            xd, ad = x[:1].expand(M, H).contiguous(), act[:1, 0].expand(M, I).contiguous()
            dense = alternate({
                "dense_gate_up": lambda w: [ext.gemm_forward_cuda(xd, w["w13"][0][e], w["w13"][1][e], w["w13"][2][e])
                                            for e in range(E)],
                "dense_down": lambda w: [ext.gemm_forward_cuda(ad, w["w2"][0][e], w["w2"][1][e], w["w2"][2][e])
                                         for e in range(E)]})
            for name, K_, N_ in (("dense_gate_up", H, 2 * I), ("dense_down", I, H)):
                r = _median_range(dense[name])     # E calls of M rows each per layer visit
                row[name] = {"M": M, "ms_for_E_calls": {k: round(v, 4) for k, v in r.items()},
                             "tflops": round(2.0 * M * E * K_ * N_ / (r["median"] * 1e-3) / 1e12, 2)}
            rows.append(row)
    t_end = time.time()
    clocks = sampler.stop(t_begin, t_end)
    if not all_ok:
        bad = [(r["T"], r["routing"], r["self_check"]) for r in rows
               if not all(c["within_tolerance"] for c in r["self_check"].values())]
        raise SystemExit(f"self-check failed (knob 12 = 3 against knob 12 = 2), nothing reported: {bad}")

    res = {"tool": "moe_prefill_bench", "workload": "Mixtral-8x7B sparse-MoE block, E = 8, top-2, g128, seeded random "
           f"weights, {a.layers} layers of distinct weights", "card": torch.cuda.get_device_name(dev),
           "power_limit_w": _power_limit_w(0), "clocks_during_sweep": clocks, "rounds": a.rounds, "rows": rows}
    print(json.dumps(res), flush=True)
    hdr = ("| T | routing | call | default ms | decode-kernels ms | staged ms | wgmma ms [min, max] | wgmma TFLOP/s | "
           "dense TFLOP/s |")
    print(hdr)
    print("|" + "---|" * (hdr.count("|") - 1))
    for r in rows:
        for what in ("sequence", "gate_up", "down"):
            c = r[what]
            wg = c["wgmma"]["ms"]
            print(f"| {r['T']} | {r['routing']} | {what} | {c['default']['ms']['median']:.3f} | "
                  f"{c['decode-kernels']['ms']['median']:.3f} | {c['staged']['ms']['median']:.3f} | "
                  f"{wg['median']:.3f} [{wg['min']:.3f}, {wg['max']:.3f}] | {c['wgmma'].get('tflops', '')} | "
                  f"{r['dense_' + what]['tflops'] if what != 'sequence' else ''} |")
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
