#!/usr/bin/env python
"""Llama-3-8B decode step (bs = 1, 32 layers) with the residual adds AND real RoPE + KV-cache append, two ways: one
JSON line.

Per layer: xn = norm1(h); qkv = xn Wqkv; q, k = RoPE(q, k) at position P; cache[P] = k, v; attn = ATTENTION STAND-IN;
o = attn Wo; hm = o + h; xn2 = norm2(hm); gu = xn2 Wgu; act = silu(gate) up; down = act Wd; h' = down + hm
(awq/modules/fused/attn.py:243-267, block.py:117-118).

The attention is a stand-in: F.scaled_dot_product_attention over cache[:, :P + 1] (GQA, 8 KV heads) from the rotated q,
on torch's math backend (reproducible from run to run), with P fixed (1023 in a 2048-position WindowedCache).  It stays outside every program (DESIGN.md 7) and is timed on its own.

  (c) 33 attention-to-attention programs (the adds fused, tools/layer_decode_bench.py's (c)), plus the reference's
      RoPE.forward and WindowedCache.update_kv (oracle/_ref, loaded through tests/_refload.py) between them;
  (d) the same 33 programs with DecodeProgram.rope_kv_cache recorded after qkv: RoPE and the cache append run in the
      qkv linear's finish (DESIGN.md 3.5f).

Each variant is captured in one CUDA graph; the graphs are replayed alternately (rounds x steps after warm-up) and the
median round is reported.  Card, power limit and SM clock are read in the same run.  Self-checks: (d)'s last-layer q
and cache rows bit-identical to the stand-alone op (ext.rope_kv_cache) on (d)'s own qkv, and within one fp16 ulp of
RoPE.forward on it (bit-identical at bs = 1, DESIGN.md 3.5f); (d)'s output within tolerance of (c)'s.  The two are not
bit-identical: the fused qkv linear is packed in mode 2, which puts a column in another MMA row than mode 0.

    python tools/rope_decode_bench.py [--steps 30] [--warmup 5] [--rounds 5] [--pos 1023]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402  (shapes, byte accounting, seeded weights, graph capture and timing of the bench)
from tools.batched_decode_bench import _power_limit_w  # noqa: E402

HEADS, KV_HEADS, HEAD_DIM, CACHE = 32, 8, 128, 2048
THETA = 500000.0
EPS = 1e-5


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--pos", type=int, default=1023, help="the fixed decode position P (attention reads P + 1 rows)")
    a = ap.parse_args()

    import torch
    import torch.nn.functional as F
    from torch.nn.attention import SDPBackend, sdpa_kernel

    from _refload import load_reference
    from autoawq_b200.program import DecodeProgram

    if load_reference(shim=True) is None:
        raise SystemExit("the reference package (oracle/_ref) is missing: run __graft_entry__.build() first")
    from awq.modules.fused.attn import RoPE
    from awq.modules.fused.cache import WindowedCache

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    rep = bench.Replica(dev, 1, seed=0)
    ext, H, I, L = rep.ext, bench.HIDDEN, bench.INTER, rep.layers
    P = a.pos
    f16 = torch.float16
    g = torch.Generator(device=dev).manual_seed(1)
    norm1 = [(1 + 0.1 * torch.randn(H, generator=g, device=dev)).half() for _ in range(L)]
    norm2 = [(1 + 0.1 * torch.randn(H, generator=g, device=dev)).half() for _ in range(L)]
    rope = RoPE(HEAD_DIM, CACHE, dev, THETA)
    cache0 = [(torch.randn((1, CACHE, KV_HEADS, HEAD_DIM), generator=g, device=dev, dtype=f16),
               torch.randn((1, CACHE, KV_HEADS, HEAD_DIM), generator=g, device=dev, dtype=f16)) for _ in range(L)]
    h0 = rep.h.clone()

    def caches():
        out = []
        for k, v in cache0:
            c = WindowedCache(1, HEADS, KV_HEADS, HEAD_DIM, CACHE, dev)
            c.k.copy_(k)
            c.v.copy_(v)
            out.append(c)
        return out

    def attention(q, c, out):
        """The stand-in: q [1, 32, 128] over the first P + 1 rows of cache c, into out [1, H]."""
        k = c.k[:, : P + 1].transpose(1, 2)
        v = c.v[:, : P + 1].transpose(1, 2)
        with sdpa_kernel([SDPBackend.MATH]):
            o = F.scaled_dot_product_attention(q.reshape(1, HEADS, 1, HEAD_DIM), k, v, enable_gqa=True)
        out.copy_(o.reshape(1, H))

    def bufs():
        e = lambda n: torch.empty((1, n), dtype=f16, device=dev)  # noqa: E731
        return [dict(h=e(H), xn=e(H), attn=e(H), hm=e(H), xn2=e(H), act=e(I), q=e(H)) for _ in range(L)] + [dict(h=e(H))]

    def programs(B, C, pos=None):
        """[norm1, qkv(, rope)], then per layer [o + h, norm2, gate|up, silu, down + hm, norm1', qkv'(, rope')]."""
        def head(p, l):
            B[l]["qkv"] = p.gemm_forward_cuda(B[l]["xn"], *rep.w[l]["qkv"], 8)
            if pos is not None:
                p.rope_kv_cache(B[l]["qkv"], rope.freqs_cis, pos, C[l].k, C[l].v, HEADS, KV_HEADS, q_out=B[l]["q"])

        p0 = DecodeProgram()
        p0.layernorm_forward_cuda(B[0]["h"], norm1[0], B[0]["xn"], EPS)
        head(p0, 0)
        plan = [p0]
        for l in range(L):
            b, w = B[l], rep.w[l]
            p = DecodeProgram()
            b["o"] = p.gemm_forward_cuda(b["attn"], *w["o"], 8)
            p.add(b["o"], b["h"], out=b["hm"])
            p.layernorm_forward_cuda(b["hm"], norm2[l], b["xn2"], EPS)
            b["gu"] = p.gemm_forward_cuda(b["xn2"], *w["gate_up"], 8)
            p.silu_and_mul(b["act"], b["gu"])
            b["down"] = p.gemm_forward_cuda(b["act"], *w["down"], 8)
            p.add(b["down"], b["hm"], out=B[l + 1]["h"])
            if l + 1 < L:
                p.layernorm_forward_cuda(B[l + 1]["h"], norm1[l + 1], B[l + 1]["xn"], EPS)
                head(p, l + 1)
            plan.append(p)
        for p in plan:
            p.build()
            assert p.fused, "a segment program did not fuse"
        return plan

    # ---- (c) programs + the reference's RoPE.forward and WindowedCache.update_kv
    Bc, Cc = bufs(), caches()
    Bc[0]["h"].copy_(h0)
    plan_c = programs(Bc, Cc)

    def rope_ref(l):
        xqkv = Bc[l]["qkv"].view(1, 1, HEADS + 2 * KV_HEADS, HEAD_DIM)
        xq, xk = rope.forward(xqkv[:, :, :HEADS], xqkv[:, :, HEADS:HEADS + KV_HEADS], P, 1)
        Cc[l].update_kv(values_store=xqkv[:, :, HEADS + KV_HEADS:], keys_store=xk, batch_size=1, start_pos=P, seqlen=1)
        Bc[l]["q"].copy_(xq.reshape(1, H))

    def step_c():
        plan_c[0].run()
        for l in range(L):
            rope_ref(l)
            attention(Bc[l]["q"], Cc[l], Bc[l]["attn"])
            plan_c[l + 1].run()
        return Bc[L]["h"]

    # ---- (d) programs with RoPE + cache append fused into the qkv finish
    Bd, Cd = bufs(), caches()
    Bd[0]["h"].copy_(h0)
    pos = torch.tensor([P], dtype=torch.int32, device=dev)
    plan_d = programs(Bd, Cd, pos)
    assert all(p.kernel_ops == q.kernel_ops for p, q in zip(plan_c, plan_d))

    def step_d():
        plan_d[0].run()
        for l in range(L):
            attention(Bd[l]["q"], Cd[l], Bd[l]["attn"])
            plan_d[l + 1].run()
        return Bd[L]["h"]

    def step_attn():
        for l in range(L):
            attention(Bd[l]["q"], Cd[l], Bd[l]["attn"])

    graphs = {}
    for name, fn in (("c_programs_plus_reference_rope", step_c), ("d_rope_fused", step_d),
                     ("attention_stand_in", step_attn)):
        graphs[name], _ = bench.capture(torch, fn)

    # ---- self-checks (after one replay of each graph on identical inputs)
    for gph in graphs.values():
        gph.replay()
    torch.cuda.synchronize()
    last = L - 1
    rk, rv = Cd[last].k.clone(), Cd[last].v.clone()
    rq = ext.rope_kv_cache(Bd[last]["qkv"], rope.freqs_cis, pos, rk, rv, HEADS, KV_HEADS)
    xqkv = Bd[last]["qkv"].view(1, 1, HEADS + 2 * KV_HEADS, HEAD_DIM)
    xq, xk = rope.forward(xqkv[:, :, :HEADS], xqkv[:, :, HEADS:HEADS + KV_HEADS], P, 1)
    torch.cuda.synchronize()

    def ulps(x, y):
        ix, iy = x.reshape(-1).view(torch.int16).int(), y.reshape(-1).view(torch.int16).int()
        return int(torch.where((ix < 0) == (iy < 0), (ix - iy).abs(), torch.full_like(ix, 1 << 16)).max())

    d_out = float((Bd[L]["h"].float() - Bc[L]["h"].float()).abs().max())
    rms = float(Bc[L]["h"].float().pow(2).mean().sqrt())
    checks = {"d_last_layer_rope_bit_identical_to_standalone_op": torch.equal(rq.reshape(1, H), Bd[last]["q"]) and
              torch.equal(rk, Cd[last].k) and torch.equal(rv, Cd[last].v),
              "d_last_layer_q_max_ulps_vs_reference_rope": ulps(Bd[last]["q"], xq),
              "d_last_layer_k_row_max_ulps_vs_reference_rope": ulps(Cd[last].k[:, P], xk),
              "d_cache_rows_other_than_P_untouched": all(torch.equal(Cd[l].k[:, :P], cache0[l][0][:, :P]) and
                                                         torch.equal(Cd[l].v[:, P + 1:], cache0[l][1][:, P + 1:])
                                                         for l in range(L)),
              "d_output_max_abs_diff_vs_c": round(d_out, 5), "output_rms": round(rms, 4),
              "d_output_consistent_with_c": bool(torch.isfinite(Bd[L]["h"]).all()) and d_out <= 0.05 * rms + 0.05}

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
    table = {}
    for name in ("c_programs_plus_reference_rope", "d_rope_fused"):
        ms = med[name]
        table[name] = {"ms_per_step": round(ms, 4), "tok_s": round(1e3 / ms, 1),
                       "ms_without_attention": round(ms - attn_ms, 4), "rounds_ms": [round(t, 4) for t in times[name]]}
    table["c_vs_d"] = round(med["c_programs_plus_reference_rope"] / med["d_rope_fused"], 3)
    table["saved_ms_per_layer"] = round((med["c_programs_plus_reference_rope"] - med["d_rope_fused"]) / L, 5)
    print(json.dumps({"tool": "rope_decode_bench", "workload": f"Llama-3-8B decode bs=1, 32 layers with residual adds, "
                      f"RoPE (theta {THETA:g}) and KV-cache append at position {P} of a {CACHE}-position cache, g128, "
                      "seeded random weights; attention = SDPA math-backend stand-in over cache[:, :P + 1]",
                      "card": torch.cuda.get_device_name(dev), "power_limit_w": _power_limit_w(0),
                      "clocks_during_timing": clocks, "steps": a.steps, "warmup": a.warmup, "rounds": a.rounds,
                      "attention_stand_in_ms": round(attn_ms, 4), "variants": table, "checks": checks}), flush=True)


if __name__ == "__main__":
    main()
