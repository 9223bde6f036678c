#!/usr/bin/env python
"""Decode steps whose rotary positions differ from their cache rows, two ways: one JSON line.

  qwen2.5-vl-7b: a Qwen2.5-VL-7B text step at B = 1 (language model: 28 layers, hidden 3584, 28 q / 4 kv heads of 128,
      intermediate 18944, qkv bias, RMSNorm eps 1e-6, rope_theta 1e6).  The token sits at cache row P and rotates at
      M-RoPE position P + delta (all three components equal, as for every text token after the prompt).
  qwen2.5-vl-3b: the same step at Qwen2.5-VL-3B's shapes (36 layers, hidden 2048, 16 q / 2 kv heads, intermediate
      11008).
  llama-3-8b: Llama-3-8B (32 layers, hidden 4096, 32 q / 8 kv heads of 128, intermediate 14336, eps 1e-5, theta 5e5),
      B = 4 left-padded sequences (pads 0 / 3 / 17 / 250) at T = 1 and T = 2 new tokens, and B = 2 (pads 0 / 250) at
      T = 2: cache rows P .. P + T - 1 in lockstep, rotary positions P + t - pad_b (transformers'
      attention_mask.cumsum(-1) - 1).
  Per segment: h = o(attn) + x; hn = norm2(h); act = silu(gate) up of gate|up(hn); x' = down(act) + h; xn' = norm1(x');
  qkv'; then RoPE on q and k at the rotary positions and k, v written to cache rows P .. P + T - 1 (2048 rows, P = 1023).

  (a) programs end at the raw qkv; transformers' rotation between them (Qwen2.5-VL: Qwen2_5_VLRotaryEmbedding and
      apply_multimodal_rotary_pos_emb with mrope_section [16, 24, 24] on 3-D position ids; Llama: LlamaRotaryEmbedding
      and apply_rotary_pos_emb on per-sequence position ids) and the cache write in torch;
  (b) rope_kv_cache(..., rope_offset=) folded into the qkv finish (DESIGN.md 3.5o): one program per segment.

g128 seeded random weights (bench.py's scale recipe).  The attention is a stand-in, F.scaled_dot_product_attention on
torch's math backend over cache[:, :P + T] with a causal mask over the new tokens and the pad rows of each sequence
masked, outside every program.  Each variant is one CUDA graph; the graphs are replayed alternately (rounds x steps after
warm-up) and the median round is reported in ms per step.  A program the stream kernels cannot run replays per op in
both variants (listed under programs_replayed_per_op).  Card, power limit and SM clock are read in the same run.

Self-checks: (b)'s last-layer q and cache rows bit-identical to ext.rope_kv_cache(rope_offset=) on (b)'s own qkv; (b)'s
step output within tolerance of (a)'s.

    python tools/rope_offset_decode_bench.py [--steps 10] [--warmup 3] [--rounds 5] [--pos 1023] [--configs ...]
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

CACHE, GROUP = 2048, 128
MODELS = {
    "qwen2.5-vl-7b": dict(layers=28, hid=3584, nh=28, kv=4, d=128, inter=18944, bias=True, eps=1e-6, theta=1e6),
    "qwen2.5-vl-3b": dict(layers=36, hid=2048, nh=16, kv=2, d=128, inter=11008, bias=True, eps=1e-6, theta=1e6),
    "llama-3-8b": dict(layers=32, hid=4096, nh=32, kv=8, d=128, inter=14336, bias=False, eps=1e-5, theta=5e5),
}
# config -> (model, B, T, per-sequence offsets of the rotary position from the cache row)
CONFIGS = {
    "qwen2.5-vl-7b/1x1": ("qwen2.5-vl-7b", 1, 1, [-389]),
    "qwen2.5-vl-3b/1x1": ("qwen2.5-vl-3b", 1, 1, [-389]),
    "llama-3-8b/4x1": ("llama-3-8b", 4, 1, [0, -3, -17, -250]),
    "llama-3-8b/4x2": ("llama-3-8b", 4, 2, [0, -3, -17, -250]),   # (M = 8: replays per op, DESIGN.md 3.5o)
    "llama-3-8b/2x2": ("llama-3-8b", 2, 2, [0, -250]),
}
MROPE_SECTION = [16, 24, 24]


def make_weights(torch, dev, m):
    g = torch.Generator(device=dev).manual_seed(0)
    wbytes = 0

    def linear(K, N):
        nonlocal wbytes
        qw = torch.randint(-2**31, 2**31 - 1, (K, N // 8), dtype=torch.int32, device=dev, generator=g)
        qz = torch.randint(-2**31, 2**31 - 1, (K // GROUP, N // 8), dtype=torch.int32, device=dev, generator=g)
        s = ((torch.rand((K // GROUP, N), device=dev, generator=g) * 0.5 + 0.75) / (6.1 * K**0.5)).half()
        wbytes += qw.numel() * 4 + qz.numel() * 4 + s.numel() * 2
        return qw, s, qz

    N = (m["nh"] + 2 * m["kv"]) * m["d"]
    w = [{"o": linear(m["nh"] * m["d"], m["hid"]), "gu": linear(m["hid"], 2 * m["inter"]),
          "down": linear(m["inter"], m["hid"]), "qkv": linear(m["hid"], N),
          "bias": (0.1 * torch.randn(N, generator=g, device=dev)).half() if m["bias"] else None}
         for _ in range(m["layers"])]
    norms = [((1 + 0.1 * torch.randn(m["hid"], generator=g, device=dev)).half(),
              (1 + 0.1 * torch.randn(m["hid"], generator=g, device=dev)).half()) for _ in range(m["layers"])]
    return w, norms, wbytes, g


def torch_rotation(torch, name, m, dev):
    """(cos, sin, apply) of transformers' rotary for the model: cos / sin from its rotary embedding at `positions`
    ([B, T] long), apply(q, k, cos, sin) on [B, heads, T, D] tensors."""
    if name.startswith("qwen2.5-vl"):
        from transformers import Qwen2_5_VLConfig
        from transformers.models.qwen2_5_vl.modeling_qwen2_5_vl import (Qwen2_5_VLRotaryEmbedding,
                                                                        apply_multimodal_rotary_pos_emb)

        cfg = Qwen2_5_VLConfig(text_config=dict(hidden_size=m["hid"], num_attention_heads=m["nh"],
                                                num_key_value_heads=m["kv"], max_position_embeddings=32768,
                                                rope_theta=m["theta"],
                                                rope_scaling={"type": "mrope", "mrope_section": MROPE_SECTION}))
        rot = Qwen2_5_VLRotaryEmbedding(cfg.text_config, device=dev)
        cs = lambda x, pos: rot(x, pos[None].expand(3, -1, -1))  # noqa: E731  (text tokens: 3 equal components)
        return cs, lambda q, k, c, s: apply_multimodal_rotary_pos_emb(q, k, c, s, MROPE_SECTION)
    from transformers import LlamaConfig
    from transformers.models.llama.modeling_llama import LlamaRotaryEmbedding, apply_rotary_pos_emb

    cfg = LlamaConfig(hidden_size=m["hid"], num_attention_heads=m["nh"], num_key_value_heads=m["kv"],
                      max_position_embeddings=8192, rope_theta=m["theta"])
    rot = LlamaRotaryEmbedding(cfg, device=dev)
    return rot, apply_rotary_pos_emb


def rotary_table(torch, m, dev):
    """RoPE.precompute_freqs_cis's table (awq/modules/fused/attn.py) at the model's theta: cos / sin of fp32 angles."""
    d = m["d"]
    inv = 1.0 / (m["theta"] ** (torch.arange(0, d, 2, device=dev)[: d // 2].float() / d))
    return torch.polar(torch.ones((CACHE, d // 2), device=dev), torch.outer(torch.arange(CACHE, device=dev).float(), inv))


def run_config(cname, a, W):
    import torch
    import torch.nn.functional as F
    from torch.nn.attention import SDPBackend, sdpa_kernel

    from autoawq_b200 import ext
    from autoawq_b200.program import DecodeProgram

    name, B, T, offs = CONFIGS[cname]
    m = MODELS[name]
    L, HID, NH, KV, D, INTER, EPS = m["layers"], m["hid"], m["nh"], m["kv"], m["d"], m["inter"], m["eps"]
    dev = torch.device("cuda", 0)
    f16 = torch.float16
    w, norms, wbytes, g = W
    P, QD, M = a.pos, NH * D, B * T
    freqs = rotary_table(torch, m, dev)
    cos_sin, apply = torch_rotation(torch, name, m, dev)
    off = torch.tensor(offs, dtype=torch.int32, device=dev)
    rot_pos = (torch.arange(T, device=dev)[None] + P + off[:, None].long())                      # [B, T]
    pad = [max(0, -o) for o in offs] if name.startswith("llama") else [0] * B
    keep = torch.ones((B, 1, T, P + T), dtype=torch.bool, device=dev).tril(P)
    for b, n in enumerate(pad):
        keep[b, :, :, :n] = False                                                                 # the pad rows
    k0 = [torch.randn((B, CACHE, KV, D), generator=g, device=dev, dtype=f16) for _ in range(L)]
    v0 = [torch.randn((B, CACHE, KV, D), generator=g, device=dev, dtype=f16) for _ in range(L)]
    x0 = torch.randn((M, HID), generator=g, device=dev, dtype=f16)

    def bufs():
        e = lambda n: torch.empty((M, n), dtype=f16, device=dev)  # noqa: E731
        out = [dict(x=e(HID), xn=e(HID), attn=e(QD), h=e(HID), hn=e(HID), act=e(INTER), k=k0[l].clone(),
                    v=v0[l].clone(), q=torch.empty((M, NH, D), dtype=f16, device=dev)) for l in range(L)]
        return out + [dict(x=e(HID), xn=e(HID))]

    def attention(b):
        k, v = b["k"][:, : P + T].transpose(1, 2), b["v"][:, : P + T].transpose(1, 2)
        q = b["q"].view(B, T, NH, D).transpose(1, 2)
        with sdpa_kernel([SDPBackend.MATH]):
            o = F.scaled_dot_product_attention(q, k, v, attn_mask=keep, enable_gqa=True)
        b["attn"].copy_(o.transpose(1, 2).reshape(M, QD))

    def rope_torch(b):
        x = b["qkv"].view(B, T, NH + 2 * KV, D).transpose(1, 2)
        cos, sin = cos_sin(x, rot_pos)
        rq, rk = apply(x[:, :NH], x[:, NH:NH + KV], cos, sin)
        b["q"].copy_(rq.transpose(1, 2).reshape(M, NH, D))
        b["k"][:, P:P + T].copy_(rk.transpose(1, 2))
        b["v"][:, P:P + T].copy_(x[:, NH + KV:].transpose(1, 2))

    def programs(Bs, pos, fold):
        def lin(p, x, l, k, bias=None):
            return p.gemm_forward_cuda(x, *w[l][k], 8, bias=bias)

        def head(p, l):
            Bs[l]["qkv"] = lin(p, Bs[l]["xn"], l, "qkv", w[l]["bias"])
            if fold:
                p.rope_kv_cache(Bs[l]["qkv"], freqs, pos, Bs[l]["k"], Bs[l]["v"], NH, KV, q_out=Bs[l]["q"],
                                seq_len=T, rope_offset=off)

        p0 = DecodeProgram(max_tokens=M)
        p0.layernorm_forward_cuda(Bs[0]["x"], norms[0][0], Bs[0]["xn"], EPS)
        head(p0, 0)
        progs = [p0]
        for l in range(L):
            b, nb = Bs[l], Bs[l + 1]
            p = DecodeProgram(max_tokens=M)
            b["o"] = lin(p, b["attn"], l, "o")
            p.add(b["o"], b["x"], out=b["h"])
            p.layernorm_forward_cuda(b["h"], norms[l][1], b["hn"], EPS)
            b["gu"] = lin(p, b["hn"], l, "gu")
            p.silu_and_mul(b["act"], b["gu"])
            b["down"] = lin(p, b["act"], l, "down")
            p.add(b["down"], b["h"], out=nb["x"])
            if l + 1 < L:
                p.layernorm_forward_cuda(nb["x"], norms[l + 1][0], nb["xn"], EPS)
                head(p, l + 1)
            progs.append(p)
        for p in progs:
            p.build()
        return progs

    pos = torch.tensor([P], dtype=torch.int32, device=dev)
    Ba, Bb = bufs(), bufs()
    Ba[0]["x"].copy_(x0)
    Bb[0]["x"].copy_(x0)
    progs_a, progs_b = programs(Ba, None, False), programs(Bb, pos, True)

    def step_a():
        progs_a[0].run()
        for l in range(L):
            rope_torch(Ba[l])
            attention(Ba[l])
            progs_a[l + 1].run()

    def step_b():
        progs_b[0].run()
        for l in range(L):
            attention(Bb[l])
            progs_b[l + 1].run()

    graphs = {}
    with torch.no_grad():
        for vname, fn in (("a_rope_in_torch_between_programs", step_a), ("b_rope_offset_folded", step_b)):
            graphs[vname], _ = bench.capture(torch, fn)
    for gph in graphs.values():
        gph.replay()
    torch.cuda.synchronize()
    last = Bb[L - 1]
    rk, rv = k0[L - 1].clone(), v0[L - 1].clone()
    rq = ext.rope_kv_cache(last["qkv"], freqs, pos, rk, rv, NH, KV, seq_len=T, rope_offset=off)
    torch.cuda.synchronize()
    d_out = float((Bb[L]["x"].float() - Ba[L]["x"].float()).abs().max())
    rms = float(Ba[L]["x"].float().pow(2).mean().sqrt())
    chk = {"b_last_layer_q_and_cache_bit_identical_to_standalone_op": torch.equal(rq, last["q"]) and
           torch.equal(rk, last["k"]) and torch.equal(rv, last["v"]),
           "b_output_max_abs_diff_vs_a": round(d_out, 5), "output_rms": round(rms, 4),
           "b_output_consistent_with_a": bool(torch.isfinite(Bb[L]["x"]).all()) and d_out <= 0.05 * rms + 0.05}

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
    ma, mb = med["a_rope_in_torch_between_programs"], med["b_rope_offset_folded"]
    unfused = {k: [i for i, p in enumerate(ps) if not p.fused] for k, ps in (("a", progs_a), ("b", progs_b))}
    out = {"model": name, "B": B, "T": T, "rot_offsets": offs, "layers": L, "weight_bytes": wbytes,
           "programs_per_step": len(progs_b), "programs_replayed_per_op": unfused,
           "clocks_during_timing": clocks, "checks": chk, "a_over_b": round(ma / mb, 3),
           "saved_us_per_layer": round((ma - mb) * 1e3 / L, 2),
           "variants": {k: {"ms_per_step": round(med[k], 4), "rounds_ms": [round(t, 4) for t in times[k]]}
                        for k in graphs}}
    del graphs, progs_a, progs_b, Ba, Bb
    gc.collect()
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--pos", type=int, default=1023, help="cache row of the step's first token")
    ap.add_argument("--configs", nargs="*", default=list(CONFIGS), choices=list(CONFIGS))
    a = ap.parse_args()

    import torch

    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    res, weights = {}, {}
    for c in a.configs:
        name = CONFIGS[c][0]
        if name not in weights:
            weights.clear()
            gc.collect()
            torch.cuda.empty_cache()
            weights[name] = make_weights(torch, dev, MODELS[name])
        res[c] = run_config(c, a, weights[name])
    print(json.dumps({"tool": "rope_offset_decode_bench", "workload":
                      f"cache rows {a.pos}.. of a {CACHE}-row cache, rotary positions offset per sequence, g128 "
                      "seeded random weights; attention = SDPA math-backend stand-in (causal over the new tokens, "
                      "pad rows masked)", "card": torch.cuda.get_device_name(0), "power_limit_w": _power_limit_w(0),
                      "steps": a.steps, "warmup": a.warmup, "rounds": a.rounds, "configs": res}), flush=True)


if __name__ == "__main__":
    main()
