#!/usr/bin/env python
"""Multi-token decode steps of Llama-3-8B (B sequences x T new tokens each), three ways: one JSON line.

  Llama-3-8B: 32 layers, hidden 4096, 32 q / 8 kv heads of 128, intermediate 14336, RMSNorm eps 1e-5, RoPE theta
  500000.  Per segment: h = o(attn) + x; hn = norm2(h); act = silu(gate) up of gate|up(hn); x' = down(act) + h;
  xn' = norm1(x'); qkv'; then RoPE on q and k and k, v appended to the cache.  The step's tokens sit at positions
  P .. P + T - 1 of a 2048-position cache (P = 1023 by default).

  (a) T sequential one-token steps (programs of M = B rows, rope_kv_cache folded), the position advanced in between;
  (b) one T-token step of programs with M = B T rows that end at the raw qkv, the reference's RoPE.forward(xq, xk, P, T)
      and WindowedCache.update_kv (oracle/_ref, loaded through tests/_refload.py) between them;
  (c) one T-token step with rope_kv_cache(..., seq_len=T) folded into the qkv finish (DESIGN.md 3.5n).

g128 seeded random weights (bench.py's scale recipe).  The attention is a stand-in, F.scaled_dot_product_attention on
torch's math backend over cache[:, :P + T] with a causal mask over the new tokens, outside every program.  Each variant
is one CUDA graph; the graphs are replayed alternately (rounds x steps after warm-up) and the median round is reported
in ms per step and per token, with (c) over a single one-token step of one sequence ((a) at B = T = 1).  Card, power
limit and SM clock are read in the same run.

Self-checks: (c)'s last-layer q and cache rows bit-identical to ext.rope_kv_cache(seq_len=T) on (c)'s own qkv; (c)'s
step output within tolerance of (b)'s.

    python tools/multi_token_decode_bench.py [--steps 10] [--warmup 3] [--rounds 5] [--pos 1023] [--configs 1x1 1x2 ..]
"""
import argparse
import gc
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402  (graph capture, timing and the clock sampler of the bench)
from tools.batched_decode_bench import _power_limit_w  # noqa: E402

CACHE, GROUP, EPS, THETA = 2048, 128, 1e-5, 500000.0
LAYERS, HID, NH, KV, D, INTER = 32, 4096, 32, 8, 128, 14336
CONFIGS = ["1x1", "1x2", "1x4", "2x2"]          # B x T


def make_weights(torch, dev):
    g = torch.Generator(device=dev).manual_seed(0)
    wbytes = 0

    def linear(K, N):
        nonlocal wbytes
        qw = torch.randint(-2**31, 2**31 - 1, (K, N // 8), dtype=torch.int32, device=dev, generator=g)
        qz = torch.randint(-2**31, 2**31 - 1, (K // GROUP, N // 8), dtype=torch.int32, device=dev, generator=g)
        s = ((torch.rand((K // GROUP, N), device=dev, generator=g) * 0.5 + 0.75) / (6.1 * K**0.5)).half()
        wbytes += qw.numel() * 4 + qz.numel() * 4 + s.numel() * 2
        return qw, s, qz

    w = [{"o": linear(NH * D, HID), "gu": linear(HID, 2 * INTER), "down": linear(INTER, HID),
          "qkv": linear(HID, (NH + 2 * KV) * D)} for _ in range(LAYERS)]
    norms = [((1 + 0.1 * torch.randn(HID, generator=g, device=dev)).half(),
              (1 + 0.1 * torch.randn(HID, generator=g, device=dev)).half()) for _ in range(LAYERS)]
    return w, norms, wbytes, g


def run_config(B, T, a, W):
    import torch
    import torch.nn.functional as F
    from torch.nn.attention import SDPBackend, sdpa_kernel

    from autoawq_b200 import ext
    from autoawq_b200.program import DecodeProgram
    from awq.modules.fused.attn import RoPE
    from awq.modules.fused.cache import WindowedCache

    dev = torch.device("cuda", 0)
    f16 = torch.float16
    w, norms, wbytes, g = W
    P, QD = a.pos, NH * D
    rope = RoPE(D, CACHE, dev, THETA)
    freqs = rope.freqs_cis
    k0 = [torch.randn((B, CACHE, KV, D), generator=g, device=dev, dtype=f16) for _ in range(LAYERS)]
    v0 = [torch.randn((B, CACHE, KV, D), generator=g, device=dev, dtype=f16) for _ in range(LAYERS)]
    x0 = torch.randn((B * T, HID), generator=g, device=dev, dtype=f16)

    def bufs(M):
        e = lambda n: torch.empty((M, n), dtype=f16, device=dev)  # noqa: E731
        out = []
        for l in range(LAYERS):
            c = WindowedCache(B, NH, KV, D, CACHE, dev)
            c.k.copy_(k0[l])
            c.v.copy_(v0[l])
            out.append(dict(x=e(HID), xn=e(HID), attn=e(QD), h=e(HID), hn=e(HID), act=e(INTER),
                            q=torch.empty((M, NH, D), dtype=f16, device=dev), cache=c))
        return out + [dict(x=e(HID), xn=e(HID))]

    def attention(b, p, n):
        """n new tokens per sequence at positions p .. p + n - 1, causal over them."""
        k = b["cache"].k[:, : p + n].transpose(1, 2)
        v = b["cache"].v[:, : p + n].transpose(1, 2)
        q = b["q"].view(B, n, NH, D).transpose(1, 2)
        mask = torch.ones((n, p + n), dtype=torch.bool, device=dev).tril(p)
        with sdpa_kernel([SDPBackend.MATH]):
            o = F.scaled_dot_product_attention(q, k, v, attn_mask=mask, enable_gqa=True)
        b["attn"].copy_(o.transpose(1, 2).reshape(B * n, QD))

    def rope_ref(b):
        x = b["qkv"].view(B, T, NH + 2 * KV, D)
        rq, rk = rope.forward(x[:, :, :NH], x[:, :, NH:NH + KV], P, T)
        b["cache"].update_kv(values_store=x[:, :, NH + KV:], keys_store=rk, batch_size=B, start_pos=P, seqlen=T)
        b["q"].copy_(rq.reshape(B * T, NH, D))

    def programs(Bs, M, pos, fold, seq_len):
        def lin(p, x, l, k):
            return p.gemm_forward_cuda(x, *w[l][k], 8)

        def head(p, l):
            Bs[l]["qkv"] = lin(p, Bs[l]["xn"], l, "qkv")
            if fold:
                p.rope_kv_cache(Bs[l]["qkv"], freqs, pos, Bs[l]["cache"].k, Bs[l]["cache"].v, NH, KV,
                                q_out=Bs[l]["q"], seq_len=seq_len)

        p0 = DecodeProgram(max_tokens=M)
        p0.layernorm_forward_cuda(Bs[0]["x"], norms[0][0], Bs[0]["xn"], EPS)
        head(p0, 0)
        progs = [p0]
        for l in range(LAYERS):
            b, nb = Bs[l], Bs[l + 1]
            p = DecodeProgram(max_tokens=M)
            b["o"] = lin(p, b["attn"], l, "o")
            p.add(b["o"], b["x"], out=b["h"])
            p.layernorm_forward_cuda(b["h"], norms[l][1], b["hn"], EPS)
            b["gu"] = lin(p, b["hn"], l, "gu")
            p.silu_and_mul(b["act"], b["gu"])
            b["down"] = lin(p, b["act"], l, "down")
            p.add(b["down"], b["h"], out=nb["x"])
            if l + 1 < LAYERS:
                p.layernorm_forward_cuda(nb["x"], norms[l + 1][0], nb["xn"], EPS)
                head(p, l + 1)
            progs.append(p)
        for p in progs:
            p.build()
            assert p.fused, "a segment program did not fuse"
        return progs

    pos_a = torch.tensor([P], dtype=torch.int32, device=dev)
    pos_c = torch.tensor([P], dtype=torch.int32, device=dev)
    Ba, Bb, Bc = bufs(B), bufs(B * T), bufs(B * T)
    Ba[0]["x"].copy_(x0.view(B, T, HID)[:, 0])
    Bb[0]["x"].copy_(x0)
    Bc[0]["x"].copy_(x0)
    progs_a = programs(Ba, B, pos_a, True, None)
    progs_b = programs(Bb, B * T, None, False, None)
    progs_c = programs(Bc, B * T, pos_c, True, T)

    def step_a():
        for t in range(T):
            pos_a.fill_(P + t)
            progs_a[0].run()
            for l in range(LAYERS):
                attention(Ba[l], P + t, 1)
                progs_a[l + 1].run()
        pos_a.fill_(P)

    def step_b():
        progs_b[0].run()
        for l in range(LAYERS):
            rope_ref(Bb[l])
            attention(Bb[l], P, T)
            progs_b[l + 1].run()

    def step_c():
        progs_c[0].run()
        for l in range(LAYERS):
            attention(Bc[l], P, T)
            progs_c[l + 1].run()

    graphs = {}
    with torch.no_grad():
        for vname, fn in (("a_sequential_one_token_steps", step_a), ("b_rope_in_torch_between_programs", step_b),
                          ("c_rope_folded", step_c)):
            graphs[vname], _ = bench.capture(torch, fn)

    for gph in graphs.values():
        gph.replay()
    torch.cuda.synchronize()
    last = Bc[LAYERS - 1]
    rk, rv = k0[LAYERS - 1].clone(), v0[LAYERS - 1].clone()
    rq = ext.rope_kv_cache(last["qkv"], freqs, pos_c, rk, rv, NH, KV, seq_len=T)
    torch.cuda.synchronize()
    d_out = float((Bc[LAYERS]["x"].float() - Bb[LAYERS]["x"].float()).abs().max())
    rms = float(Bb[LAYERS]["x"].float().pow(2).mean().sqrt())
    chk = {"c_last_layer_q_and_cache_bit_identical_to_standalone_op": torch.equal(rq, last["q"]) and
           torch.equal(rk, last["cache"].k) and torch.equal(rv, last["cache"].v),
           "c_output_max_abs_diff_vs_b": round(d_out, 5), "output_rms": round(rms, 4),
           "c_output_consistent_with_b": bool(torch.isfinite(Bc[LAYERS]["x"]).all()) and d_out <= 0.05 * rms + 0.05}

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
    table = {k: {"ms_per_step": round(med[k], 4), "ms_per_token": round(med[k] / (B * T), 4),
                 "rounds_ms": [round(t, 4) for t in times[k]]} for k in graphs}
    out = {"B": B, "T": T, "weight_bytes": wbytes, "clocks_during_timing": clocks, "variants": table, "checks": chk,
           "b_over_c": round(med["b_rope_in_torch_between_programs"] / med["c_rope_folded"], 3),
           "a_over_c": round(med["a_sequential_one_token_steps"] / med["c_rope_folded"], 3)}
    del graphs, progs_a, progs_b, progs_c, Ba, Bb, Bc
    gc.collect()
    torch.cuda.empty_cache()
    return out, med


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--pos", type=int, default=1023, help="position of the step's first token")
    ap.add_argument("--configs", nargs="*", default=CONFIGS, help="B x T pairs, e.g. 1x4 2x2")
    a = ap.parse_args()

    import torch

    from _refload import load_reference

    if load_reference(shim=True) is None:
        raise SystemExit("the reference package (oracle/_ref) is missing: run __graft_entry__.build() first")
    torch.cuda.set_device(0)
    W = make_weights(torch, torch.device("cuda", 0))
    res, single = {}, None
    for c in a.configs:
        B, T = (int(v) for v in c.split("x"))
        res[c], med = run_config(B, T, a, W)
        if (B, T) == (1, 1):
            single = med["a_sequential_one_token_steps"]
    if single is not None:
        for c, r in res.items():
            r["c_over_single_one_token_step"] = round(r["variants"]["c_rope_folded"]["ms_per_step"] / single, 3)
    print(json.dumps({"tool": "multi_token_decode_bench", "model": "Llama-3-8B shapes", "workload":
                      f"B x T new tokens at positions {a.pos}.. of a {CACHE}-position cache, RoPE theta {THETA:g}, "
                      "g128 seeded random weights; attention = SDPA math-backend stand-in with a causal mask over the "
                      "new tokens", "card": torch.cuda.get_device_name(0), "power_limit_w": _power_limit_w(0),
                      "steps": a.steps, "warmup": a.warmup, "rounds": a.rounds, "configs": res}), flush=True)


if __name__ == "__main__":
    main()
