#!/usr/bin/env python
"""Qwen3-8B decode step (bs = 1, 36 layers) with the residual adds, Qwen3's q / k norm and real RoPE + KV-cache append,
two ways: one JSON line.

Per layer: xn = norm1(h); qkv = xn Wqkv; q, k = q_norm(q), k_norm(k) (per head); q, k = RoPE(q, k) at position P;
cache[P] = k, v; attn = ATTENTION STAND-IN; o = attn Wo; hm = o + h; xn2 = norm2(hm); gu = xn2 Wgu;
act = silu(gate) up; down = act Wd; h' = down + hm.  Shapes: hidden 4096, 32 q / 8 kv heads of 128, intermediate
12288, RoPE theta 1e6, g128, seeded random weights (bench.py's scale recipe).

The attention is a stand-in: F.scaled_dot_product_attention over cache[:, :P + 1] (GQA) from the rotated q, on torch's
math backend, with P fixed (1023 in a 2048-position WindowedCache).  It stays outside every program and is timed alone.

  (c) 37 attention-to-attention programs (the adds fused), plus transformers' Qwen3RMSNorm (q_norm, k_norm), the
      reference's RoPE.forward and WindowedCache.update_kv (oracle/_ref, through tests/_refload.py) between them;
  (d) the same 37 programs with DecodeProgram.rope_kv_cache(..., q_norm=, k_norm=) recorded after qkv: the norms, the
      rotation and the cache append run in the qkv linear's finish (DESIGN.md 3.5g).

Each variant is captured in one CUDA graph; the graphs are replayed alternately (rounds x steps after warm-up) and the
median round is reported.  Card, power limit and SM clock are read in the same run.

publish phase: one layer's segment program run with knob 3 = 2 (per-op stamps of the first 8 CTAs, program_stream.cuh),
once with the q / k norm fold and once with plain ROPE_KV on the same weights; the qkv op's publish phase ([6] - [5]:
the finish, with the norm fold's cross-CTA exchange) per CTA, median over runs and CTAs, in us.

Self-checks: (d)'s last-layer q and cache rows bit-identical to the stand-alone op on (d)'s own qkv, within 2 fp16 ulps
of the reference chain on it; (d)'s output within tolerance of (c)'s (the fused qkv linear is packed in mode 2, which
puts a column in another MMA row than mode 0: not bit-identical).

    python tools/qwen3_decode_bench.py [--steps 30] [--warmup 5] [--rounds 5] [--pos 1023] [--stamp-runs 20]
"""
import argparse
import ctypes
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402  (graph capture, timing and the clock sampler of the bench)
from tools.batched_decode_bench import _power_limit_w  # noqa: E402

HIDDEN, INTER, LAYERS, HEADS, KV_HEADS, HEAD_DIM, CACHE, GROUP = 4096, 12288, 36, 32, 8, 128, 2048, 128
THETA = 1e6
EPS = 1e-6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--pos", type=int, default=1023, help="the fixed decode position P (attention reads P + 1 rows)")
    ap.add_argument("--stamp-runs", type=int, default=20)
    a = ap.parse_args()

    import numpy as np
    import torch
    import torch.nn.functional as F
    from torch.nn.attention import SDPBackend, sdpa_kernel
    from transformers.models.qwen3.modeling_qwen3 import Qwen3RMSNorm

    from _refload import load_reference
    from autoawq_b200 import ext
    from autoawq_b200._cabi import check, lib
    from autoawq_b200.program import DecodeProgram

    if load_reference(shim=True) is None:
        raise SystemExit("the reference package (oracle/_ref) is missing: run __graft_entry__.build() first")
    from awq.modules.fused.attn import RoPE
    from awq.modules.fused.cache import WindowedCache

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    H, I, L, D, P = HIDDEN, INTER, LAYERS, HEAD_DIM, a.pos
    QD = HEADS * D
    f16 = torch.float16
    g = torch.Generator(device=dev).manual_seed(0)

    def linear(K, N):
        qw = torch.randint(-2**31, 2**31 - 1, (K, N // 8), dtype=torch.int32, device=dev, generator=g)
        qz = torch.randint(-2**31, 2**31 - 1, (K // GROUP, N // 8), dtype=torch.int32, device=dev, generator=g)
        s = (torch.rand((K // GROUP, N), device=dev, generator=g) * 0.5 + 0.75) / (6.1 * K**0.5)
        return qw, s.half(), qz

    w = [dict(qkv=linear(H, (HEADS + 2 * KV_HEADS) * D), o=linear(QD, H), gate_up=linear(H, 2 * I), down=linear(I, H))
         for _ in range(L)]
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
    rope = RoPE(D, CACHE, dev, THETA)
    cache0 = [(torch.randn((1, CACHE, KV_HEADS, D), generator=g, device=dev, dtype=f16),
               torch.randn((1, CACHE, KV_HEADS, D), generator=g, device=dev, dtype=f16)) for _ in range(L)]
    h0 = torch.randn((1, H), generator=g, device=dev, dtype=f16)

    def caches():
        out = []
        for k, v in cache0:
            c = WindowedCache(1, HEADS, KV_HEADS, D, CACHE, dev)
            c.k.copy_(k)
            c.v.copy_(v)
            out.append(c)
        return out

    def attention(q, c, out):
        k = c.k[:, : P + 1].transpose(1, 2)
        v = c.v[:, : P + 1].transpose(1, 2)
        with sdpa_kernel([SDPBackend.MATH]):
            o = F.scaled_dot_product_attention(q.reshape(1, HEADS, 1, D), k, v, enable_gqa=True)
        out.copy_(o.reshape(1, QD))

    def bufs():
        e = lambda n: torch.empty((1, n), dtype=f16, device=dev)  # noqa: E731
        return [dict(h=e(H), xn=e(H), attn=e(QD), hm=e(H), xn2=e(H), act=e(I), q=e(QD)) for _ in range(L)] + [dict(h=e(H))]

    def head(p, B, C, l, pos, norms):
        B[l]["qkv"] = p.gemm_forward_cuda(B[l]["xn"], *w[l]["qkv"], 8)
        if pos is not None:
            qn, kn = qk_norms[l] if norms else (None, None)
            p.rope_kv_cache(B[l]["qkv"], rope.freqs_cis, pos, C[l].k, C[l].v, HEADS, KV_HEADS, q_out=B[l]["q"],
                            q_norm=qn, k_norm=kn)

    def segment(p, B, C, l, pos, norms=True):
        b = B[l]
        b["o"] = p.gemm_forward_cuda(b["attn"], *w[l]["o"], 8)
        p.add(b["o"], b["h"], out=b["hm"])
        p.layernorm_forward_cuda(b["hm"], norm2[l], b["xn2"], EPS)
        b["gu"] = p.gemm_forward_cuda(b["xn2"], *w[l]["gate_up"], 8)
        p.silu_and_mul(b["act"], b["gu"])
        b["down"] = p.gemm_forward_cuda(b["act"], *w[l]["down"], 8)
        p.add(b["down"], b["hm"], out=B[l + 1]["h"])
        if l + 1 < L:
            p.layernorm_forward_cuda(B[l + 1]["h"], norm1[l + 1], B[l + 1]["xn"], EPS)
            head(p, B, C, l + 1, pos, norms)

    def programs(B, C, pos=None):
        """[norm1, qkv(, qk-norm-rope)], then per layer [o + h, norm2, gate|up, silu, down + hm, norm1', qkv'(, ..')]."""
        p0 = DecodeProgram()
        p0.layernorm_forward_cuda(B[0]["h"], norm1[0], B[0]["xn"], EPS)
        head(p0, B, C, 0, pos, True)
        plan = [p0]
        for l in range(L):
            p = DecodeProgram()
            segment(p, B, C, l, pos)
            plan.append(p)
        for p in plan:
            p.build()
            assert p.fused, "a segment program did not fuse"
        return plan

    # ---- (c) programs + Qwen3RMSNorm, the reference's RoPE.forward and WindowedCache.update_kv
    Bc, Cc = bufs(), caches()
    Bc[0]["h"].copy_(h0)
    plan_c = programs(Bc, Cc)
    NQ = HEADS + 2 * KV_HEADS

    def ref_chain(qkv, l, C):
        xqkv = qkv.view(1, 1, NQ, D)
        qn, kn = qk_norms[l]
        xq, xk = rope.forward(qn(xqkv[:, :, :HEADS]), kn(xqkv[:, :, HEADS:HEADS + KV_HEADS]), P, 1)
        C.update_kv(values_store=xqkv[:, :, HEADS + KV_HEADS:], keys_store=xk, batch_size=1, start_pos=P, seqlen=1)
        return xq, xk

    def step_c():
        plan_c[0].run()
        for l in range(L):
            with torch.no_grad():
                xq, _ = ref_chain(Bc[l]["qkv"], l, Cc[l])
            Bc[l]["q"].copy_(xq.reshape(1, QD))
            attention(Bc[l]["q"], Cc[l], Bc[l]["attn"])
            plan_c[l + 1].run()
        return Bc[L]["h"]

    # ---- (d) programs with the q / k norm, RoPE and the cache append fused into the qkv finish
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
    for name, fn in (("c_programs_plus_torch_qknorm_rope", step_c), ("d_qknorm_rope_fused", step_d),
                     ("attention_stand_in", step_attn)):
        graphs[name], _ = bench.capture(torch, fn)

    # ---- self-checks (after one replay of each graph on identical inputs)
    for gph in graphs.values():
        gph.replay()
    torch.cuda.synchronize()
    last = L - 1
    rk, rv = Cd[last].k.clone(), Cd[last].v.clone()
    qn, kn = qk_norms[last]
    rq = ext.rope_kv_cache(Bd[last]["qkv"], rope.freqs_cis, pos, rk, rv, HEADS, KV_HEADS, q_norm=qn, k_norm=kn)
    chk = caches()[last]
    with torch.no_grad():
        xq, xk = ref_chain(Bd[last]["qkv"], last, chk)
    torch.cuda.synchronize()

    def ulps(x, y):
        ix, iy = x.reshape(-1).view(torch.int16).int(), y.reshape(-1).view(torch.int16).int()
        return torch.where((ix < 0) == (iy < 0), (ix - iy).abs(), torch.full_like(ix, 1 << 16))

    uq, uk = ulps(Bd[last]["q"], xq), ulps(Cd[last].k[:, P], xk)
    d_out = float((Bd[L]["h"].float() - Bc[L]["h"].float()).abs().max())
    rms = float(Bc[L]["h"].float().pow(2).mean().sqrt())
    checks = {"d_last_layer_bit_identical_to_standalone_op": torch.equal(rq.reshape(1, QD), Bd[last]["q"]) and
              torch.equal(rk, Cd[last].k) and torch.equal(rv, Cd[last].v),
              "d_last_layer_qk_max_ulps_vs_reference_chain": int(max(uq.max(), uk.max())),
              "d_last_layer_qk_elements_differing_from_reference_chain": int((uq > 0).sum() + (uk > 0).sum()),
              "d_output_max_abs_diff_vs_c": round(d_out, 5), "output_rms": round(rms, 4),
              "d_output_consistent_with_c": bool(torch.isfinite(Bd[L]["h"]).all()) and d_out <= 0.05 * rms + 0.05}

    # ---- publish phase of the qkv op (kernel op 3 of a segment program) with the norm fold and with plain RoPE
    def publish_us(norms):
        B, C = bufs(), caches()
        for b in B:
            for t in b.values():
                t.normal_()
        p = DecodeProgram()
        segment(p, B, C, 0, pos, norms)
        p.build()
        assert p.fused and p.kernel_ops == 4
        buf = np.zeros(32 * 8 * 8, dtype=np.uint64)
        vals = []
        was = ext.get_knob(3)
        try:
            ext.set_knob(3, 2)
            for _ in range(a.stamp_runs):
                p.run()
                torch.cuda.synchronize()
                check(lib.b200awq_debug_read(buf.ctypes.data_as(ctypes.c_void_p), buf.nbytes), "b200awq_debug_read")
                st = buf.reshape(32, 8, 8).astype(np.int64)
                vals.extend(((st[3, :, 6] - st[3, :, 5]) / 1e3).tolist())
        finally:
            ext.set_knob(3, was)
        return {"median_us": round(float(np.median(vals)), 3), "max_us": round(float(np.max(vals)), 3)}

    publish = {"qkv_publish_with_qk_norm_fold": publish_us(True), "qkv_publish_with_plain_rope": publish_us(False)}

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
    for name in ("c_programs_plus_torch_qknorm_rope", "d_qknorm_rope_fused"):
        ms = med[name]
        table[name] = {"ms_per_step": round(ms, 4), "tok_s": round(1e3 / ms, 1),
                       "ms_without_attention": round(ms - attn_ms, 4), "rounds_ms": [round(t, 4) for t in times[name]]}
    table["c_vs_d"] = round(med["c_programs_plus_torch_qknorm_rope"] / med["d_qknorm_rope_fused"], 3)
    table["saved_ms_per_layer"] = round((med["c_programs_plus_torch_qknorm_rope"] - med["d_qknorm_rope_fused"]) / L, 5)
    print(json.dumps({"tool": "qwen3_decode_bench", "workload": f"Qwen3-8B decode bs=1, {L} layers with residual adds, "
                      f"q / k norm, RoPE (theta {THETA:g}) and KV-cache append at position {P} of a {CACHE}-position "
                      "cache, g128, seeded random weights; attention = SDPA math-backend stand-in over cache[:, :P + 1]",
                      "card": torch.cuda.get_device_name(dev), "power_limit_w": _power_limit_w(0),
                      "clocks_during_timing": clocks, "steps": a.steps, "warmup": a.warmup, "rounds": a.rounds,
                      "attention_stand_in_ms": round(attn_ms, 4), "variants": table, "publish_phase": publish,
                      "checks": checks}), flush=True)


if __name__ == "__main__":
    main()
