#!/usr/bin/env python
"""Decode step (bs = 1) of two StableLM models (partial rotary), each two ways: one JSON line.

  StableLM-2-1.6B: 24 layers, hidden 2048, 32 q / 32 kv heads of 64, rotary dim 16 (partial_rotary_factor 0.25),
      intermediate 5632, a qkv bias.
  StableLM-3B-4E1T: 32 layers, hidden 2560, 32 q / 32 kv heads of 80, rotary dim 20 (partial_rotary_factor 0.25),
      intermediate 6912, no bias.
  Both: RoPE theta 10000, nn.LayerNorm (with bias) eps 1e-5.  Per segment (StableLmFuser's LlamaLikeBlock):
  h = o(attn) + x; hn = LN2(h); act = silu(gate) up of gate|up(hn); x' = down(act) + h; xn' = LN1(x'); qkv'; then the
  first R columns of each q / k head rotated, the rest passed through, and k, v appended to the cache.  The shapes run
  are printed with the result.

  (a) programs ending at the raw qkv (the LayerNorms folded), with the reference's RoPE(R).forward on the rotated
      slices, torch.cat with the untouched tails and WindowedCache.update_kv (oracle/_ref, loaded through
      tests/_refload.py) between them;
  (b) one program per attention-to-attention segment, rope_kv_cache(..., head_dim=D) folded into the qkv finish
      (DESIGN.md 3.5m).

g128 seeded random weights (bench.py's scale recipe).  The attention is a stand-in, F.scaled_dot_product_attention on
torch's math backend over cache[:, :P + 1] from the rotated q, outside every program and timed alone.  Each variant is
one CUDA graph; the graphs are replayed alternately (rounds x steps after warm-up), the median round is reported with
ms / step, tok/s and GB/s over the step's algorithmic bytes (packed weights, scales, zeros and biases once, the KV rows
the attention reads).  Card, power limit and SM clock are read in the same run.

Self-checks: (b)'s last-layer q and cache rows bit-identical to ext.rope_kv_cache on (b)'s own qkv; (b)'s step output
within tolerance of (a)'s.

    python tools/stablelm_decode_bench.py [--steps 20] [--warmup 3] [--rounds 5] [--pos 1023]
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

CACHE, GROUP, EPS, THETA = 2048, 128, 1e-5, 10000.0
MODELS = {
    "stablelm-2-1.6b": dict(layers=24, hidden=2048, heads=32, kv=32, head_dim=64, rotary_dim=16, inter=5632,
                            qkv_bias=True),
    "stablelm-3b-4e1t": dict(layers=32, hidden=2560, heads=32, kv=32, head_dim=80, rotary_dim=20, inter=6912,
                             qkv_bias=False),
}


def run_model(name, cfg, a):
    import torch
    import torch.nn.functional as F
    from torch.nn.attention import SDPBackend, sdpa_kernel

    from autoawq_b200 import ext
    from autoawq_b200.program import DecodeProgram
    from awq.modules.fused.attn import RoPE
    from awq.modules.fused.cache import WindowedCache

    dev = torch.device("cuda", 0)
    f16 = torch.float16
    H, I, L, P = cfg["hidden"], cfg["inter"], cfg["layers"], a.pos
    NH, KV, D, R = cfg["heads"], cfg["kv"], cfg["head_dim"], cfg["rotary_dim"]
    QD, NQKV = NH * D, (NH + 2 * KV) * D
    g = torch.Generator(device=dev).manual_seed(0)
    wbytes = 0

    def linear(K, N, bias=False):
        nonlocal wbytes
        qw = torch.randint(-2**31, 2**31 - 1, (K, N // 8), dtype=torch.int32, device=dev, generator=g)
        qz = torch.randint(-2**31, 2**31 - 1, (K // GROUP, N // 8), dtype=torch.int32, device=dev, generator=g)
        s = ((torch.rand((K // GROUP, N), device=dev, generator=g) * 0.5 + 0.75) / (6.1 * K**0.5)).half()
        b = (0.02 * torch.randn(N, device=dev, generator=g)).half() if bias else None
        wbytes += qw.numel() * 4 + qz.numel() * 4 + s.numel() * 2 + (b.numel() * 2 if b is not None else 0)
        return qw, s, qz, b

    def norm():
        return ((1 + 0.1 * torch.randn(H, generator=g, device=dev)).half(),
                (0.05 * torch.randn(H, generator=g, device=dev)).half())

    w = [{"o": linear(QD, H), "gu": linear(H, 2 * I), "down": linear(I, H), "qkv": linear(H, NQKV, cfg["qkv_bias"])}
         for _ in range(L)]
    n1 = [norm() for _ in range(L)]
    n2 = [norm() for _ in range(L)]
    rope = RoPE(R, CACHE, dev, THETA)
    freqs = rope.freqs_cis
    k0 = [torch.randn((1, CACHE, KV, D), generator=g, device=dev, dtype=f16) for _ in range(L)]
    v0 = [torch.randn((1, CACHE, KV, D), generator=g, device=dev, dtype=f16) for _ in range(L)]
    x0 = torch.randn((1, H), generator=g, device=dev, dtype=f16)
    pos = torch.tensor([P], dtype=torch.int32, device=dev)

    def bufs():
        e = lambda n: torch.empty((1, n), dtype=f16, device=dev)  # noqa: E731
        B = []
        for l in range(L):
            c = WindowedCache(1, NH, KV, D, CACHE, dev)
            c.k.copy_(k0[l])
            c.v.copy_(v0[l])
            B.append(dict(x=e(H), xn=e(H), attn=e(QD), h=e(H), hn=e(H), act=e(I),
                          q=torch.empty((1, NH, D), dtype=f16, device=dev), cache=c))
        return B + [dict(x=e(H), xn=e(H))]

    def lin(p, x, l, k):
        qw, s, qz, b = w[l][k]
        return p.gemm_forward_cuda(x, qw, s, qz, 8, bias=b)

    def attention(b):
        k = b["cache"].k[:, : P + 1].transpose(1, 2)
        v = b["cache"].v[:, : P + 1].transpose(1, 2)
        with sdpa_kernel([SDPBackend.MATH]):
            o = F.scaled_dot_product_attention(b["q"].reshape(1, NH, 1, D), k, v, enable_gqa=True)
        b["attn"].copy_(o.reshape(1, QD))

    def rope_ref(b):
        """RoPE(R).forward on the rotated slices, the tails concatenated back, update_kv."""
        x = b["qkv"].view(1, 1, NH + 2 * KV, D)
        xq, xk = x[:, :, :NH], x[:, :, NH:NH + KV]
        rq, rk = rope.forward(xq[..., :R], xk[..., :R], P, 1)
        k = torch.cat((rk, xk[..., R:]), -1)
        b["cache"].update_kv(values_store=x[:, :, NH + KV:], keys_store=k, batch_size=1, start_pos=P, seqlen=1)
        b["q"].copy_(torch.cat((rq, xq[..., R:]), -1).reshape(1, NH, D))

    def programs(B, fold):
        """[LN1, qkv(, rope)], then per layer [o + x, LN2, gate|up, silu, down + h, LN1', qkv'(, rope')]."""
        def head(p, l):
            B[l]["qkv"] = lin(p, B[l]["xn"], l, "qkv")
            if fold:
                p.rope_kv_cache(B[l]["qkv"], freqs, pos, B[l]["cache"].k, B[l]["cache"].v, NH, KV, q_out=B[l]["q"],
                                head_dim=D)

        p0 = DecodeProgram()
        p0.layer_norm(B[0]["x"], *n1[0], B[0]["xn"], EPS)
        head(p0, 0)
        progs = [p0]
        for l in range(L):
            b, nb = B[l], B[l + 1]
            p = DecodeProgram()
            b["o"] = lin(p, b["attn"], l, "o")
            p.add(b["o"], b["x"], out=b["h"])
            p.layer_norm(b["h"], *n2[l], b["hn"], EPS)
            b["gu"] = lin(p, b["hn"], l, "gu")
            p.silu_and_mul(b["act"], b["gu"])
            b["down"] = lin(p, b["act"], l, "down")
            p.add(b["down"], b["h"], out=nb["x"])
            if l + 1 < L:
                p.layer_norm(nb["x"], *n1[l + 1], nb["xn"], EPS)
                head(p, l + 1)
            progs.append(p)
        for p in progs:
            p.build()
            assert p.fused, "a segment program did not fuse"
        return progs

    Ba, Bb = bufs(), bufs()
    for B in (Ba, Bb):
        B[0]["x"].copy_(x0)
    progs_a, progs_b = programs(Ba, False), programs(Bb, True)

    def step_a():
        progs_a[0].run()
        for l in range(L):
            rope_ref(Ba[l])
            attention(Ba[l])
            progs_a[l + 1].run()
        return Ba[L]["x"]

    def step_b():
        progs_b[0].run()
        for l in range(L):
            attention(Bb[l])
            progs_b[l + 1].run()
        return Bb[L]["x"]

    def step_attn():
        for l in range(L):
            attention(Bb[l])

    graphs = {}
    with torch.no_grad():
        for vname, fn in (("a_programs_plus_reference_rope", step_a), ("b_one_program_per_segment", step_b),
                          ("attention_stand_in", step_attn)):
            graphs[vname], _ = bench.capture(torch, fn)

    # ---- self-checks after one replay of each graph on identical inputs (the caches were written at the same position)
    for gph in graphs.values():
        gph.replay()
    torch.cuda.synchronize()
    last = Bb[L - 1]
    rk, rv = k0[L - 1].clone(), v0[L - 1].clone()
    rq = ext.rope_kv_cache(last["qkv"], freqs, pos, rk, rv, NH, KV, head_dim=D)
    torch.cuda.synchronize()
    d_out = float((Bb[L]["x"].float() - Ba[L]["x"].float()).abs().max())
    rms = float(Ba[L]["x"].float().pow(2).mean().sqrt())
    chk = {"b_last_layer_q_and_cache_bit_identical_to_standalone_op": torch.equal(rq, last["q"]) and
           torch.equal(rk, last["cache"].k) and torch.equal(rv, last["cache"].v),
           "b_output_max_abs_diff_vs_a": round(d_out, 5), "output_rms": round(rms, 4),
           "b_output_consistent_with_a": bool(torch.isfinite(Bb[L]["x"]).all()) and d_out <= 0.05 * rms + 0.05}

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
    for vname in ("a_programs_plus_reference_rope", "b_one_program_per_segment"):
        ms = med[vname]
        table[vname] = {"ms_per_step": round(ms, 4), "tok_s": round(1e3 / ms, 1), "gb_s": round(step_bytes / ms / 1e6, 1),
                        "ms_without_attention": round(ms - med["attention_stand_in"], 4),
                        "rounds_ms": [round(t, 4) for t in times[vname]]}
    table["a_vs_b"] = round(med["a_programs_plus_reference_rope"] / med["b_one_program_per_segment"], 3)
    table["saved_ms_per_layer"] = round((med["a_programs_plus_reference_rope"] - med["b_one_program_per_segment"]) / L, 5)
    out = {"model": name, "shapes": cfg, "step_bytes": step_bytes, "attention_stand_in_ms": round(med["attention_stand_in"], 4),
           "clocks_during_timing": clocks, "variants": table, "checks": chk}
    del graphs, progs_a, progs_b, Ba, Bb, w
    gc.collect()
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--pos", type=int, default=1023, help="the fixed decode position P (attention reads P + 1 rows)")
    ap.add_argument("--models", nargs="*", default=list(MODELS))
    a = ap.parse_args()

    import torch

    from _refload import load_reference

    if load_reference(shim=True) is None:
        raise SystemExit("the reference package (oracle/_ref) is missing: run __graft_entry__.build() first")
    torch.cuda.set_device(0)
    res = {n: run_model(n, MODELS[n], a) for n in a.models}
    print(json.dumps({"tool": "stablelm_decode_bench", "workload": f"decode bs=1, position {a.pos} of a {CACHE}-position "
                      f"cache, RoPE theta {THETA:g}, g128 seeded random weights; attention = SDPA math-backend stand-in "
                      "over cache[:, :P + 1]", "card": torch.cuda.get_device_name(0),
                      "power_limit_w": _power_limit_w(0), "steps": a.steps, "warmup": a.warmup, "rounds": a.rounds,
                      "models": res}), flush=True)


if __name__ == "__main__":
    main()
