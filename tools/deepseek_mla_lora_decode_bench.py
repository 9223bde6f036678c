#!/usr/bin/env python
"""DeepSeek-V3 dense-layer decode step at bs = 1 with the q LoRA MLA glue (seeded random AWQ weights, g128), the glue
left to torch or folded into the decode programs.

`--layers` dense layers at DeepSeek-V3's shapes (hidden 7168, intermediate 18432, 128 heads, Dn 128, Dr 64, Dv 128,
C 512, Cq 1536), each with its own weights, so the step streams them from HBM (about 290 MB of W4 weights per layer).
A yarn-scaled rotary table (V3's rope parameters: theta 1e4, factor 40, original 4096, beta 32 / 1, mscale =
mscale_all_dim = 1) and per layer a KV cache of 2048 positions written at position P = 1023.  Attention is an SDPA
stand-in over cache[:, :P + 1] with the model's softmax scale (192^-0.5 mscale^2), the same in both arms; its output is
the next layer's o_proj input.

Arms, each one CUDA graph of the whole step, rounds alternated, medians reported:
  (c) the programs ending at the fused q_a_proj | kv_a_proj_with_mqa linear, plus the q LoRA glue per op: split,
      q_a_layernorm and kv_a_layernorm (transformers' RMSNorm arithmetic), q_b_proj and kv_b_proj (ext's W4A16 GEMV),
      splits, rotary (apply_rotary_pos_emb_interleave; apply_rotary_emb with --style 0), expand, cat and the cache
      writes;
  (d) the programs with mla_k_rope, q_a_layernorm, q_b_proj, mla_q_rope, kv_a_layernorm, kv_b_proj and mla_kv_cache
      recorded in them.
Self-checks: (d) is one launch per layer, no abort record, and (d)'s last layer's q row and cache rows equal the
stand-alone ops (ext.mla_k_rope / mla_q_rope / mla_kv_cache) run on (d)'s own recorded rows.  Prints one JSON line with
the card's name and power limit."""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from autoawq_b200 import ext  # noqa: E402
from autoawq_b200.program import DecodeProgram  # noqa: E402

H, INTER, G = 7168, 18432, 128
NH, DN, DR, DV, C, CQ = 128, 128, 64, 128, 512, 1536
W = DN + DR
N_QA, N_QB, N_KV = CQ + C + DR, NH * W, NH * (DN + DV)
S_CACHE, P, EPS = 2048, 1023, 1e-6
YARN = dict(rope_type="yarn", rope_theta=10000.0, factor=40.0, original_max_position_embeddings=4096, beta_fast=32.0,
            beta_slow=1.0, mscale=1.0, mscale_all_dim=1.0)


def rotary_tables(dev):
    """(freqs_cis complex64 [S, Dr/2], (cos, sin) f32 [S, Dr]) of V3's yarn rotary embedding, attention_scaling applied"""
    from transformers import DeepseekV3Config
    from transformers.models.deepseek_v3.modeling_deepseek_v3 import DeepseekV3RotaryEmbedding

    cfg = DeepseekV3Config(hidden_size=H, num_attention_heads=NH, q_lora_rank=CQ, kv_lora_rank=C, qk_nope_head_dim=DN,
                           qk_rope_head_dim=DR, v_head_dim=DV, max_position_embeddings=163840, rope_parameters=YARN)
    rot = DeepseekV3RotaryEmbedding(cfg, device=dev)
    f = torch.outer(torch.arange(S_CACHE, device=dev).float(), rot.inv_freq.float())
    emb = torch.cat((f, f), dim=-1)
    s = rot.attention_scaling
    return torch.polar(torch.full_like(f, s), f), (emb.cos() * s, emb.sin() * s)


def card():
    """the card's name, power limit and maximum SM clock as nvidia-smi reports them (a query only)"""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "not reported"
    except (OSError, subprocess.SubprocessError):
        return "not reported"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=6)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--style", type=int, default=1, choices=[0, 1])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    style = a.style
    cis, cs = rotary_tables(dev)
    freqs = cis if style == 0 else cs
    mscale = 0.1 * YARN["mscale_all_dim"] * math.log(YARN["factor"]) + 1.0
    scale = W ** -0.5 * mscale * mscale

    def lin(K, N):
        return (torch.randint(-2**31, 2**31 - 1, (K, N // 8), dtype=torch.int32, device=dev, generator=gen),
                ((torch.rand((K // G, N), device=dev, generator=gen) * 0.5 + 0.75) / (6.1 * K**0.5)).half(),
                torch.randint(-2**31, 2**31 - 1, (K // G, N // 8), dtype=torch.int32, device=dev, generator=gen))

    def norm_w(n=H):
        return (1 + 0.1 * torch.randn(n, device=dev, generator=gen)).half()

    layers = []
    for li in range(a.layers + 1):     # (+1: the last program ends with the MLA chain of the layer after the stack)
        L = dict(wqa=lin(H, N_QA), wqb=lin(CQ, N_QB), wkvb=lin(C, N_KV), n1=norm_w(), nq=norm_w(CQ), nkv=norm_w(C),
                 attn=torch.randn((1, NH * DV), device=dev, generator=gen).half())
        if li < a.layers:
            L.update(wo=lin(NH * DV, H), n2=norm_w(), gu=lin(H, 2 * INTER), down=lin(INTER, H))
        layers.append(L)
    h0 = torch.randn((1, H), device=dev, generator=gen).half()
    pos = torch.tensor([P], dtype=torch.int32, device=dev)
    pos_l = pos.long()

    def rms(x, w):
        v32 = x.float()
        return w * (v32 * torch.rsqrt(v32.pow(2).mean(-1, keepdim=True) + EPS)).half()

    def torch_glue(qa, L, k_cache, v_cache, q_out):
        """transformers' DeepseekV2Attention / DeepseekV3Attention with a q LoRA after q_a_proj | kv_a_proj_with_mqa"""
        from transformers.models.deepseek_v2.modeling_deepseek_v2 import apply_rotary_emb
        from transformers.models.deepseek_v3.modeling_deepseek_v3 import apply_rotary_pos_emb_interleave

        q_a, c_kv, k_pe = torch.split(qa, [CQ, C, DR], dim=-1)
        q = ext.linear_forward("gemm", rms(q_a, L["nq"]), *L["wqb"], G).view(1, 1, NH, W).transpose(1, 2)
        q_nope, q_pe = torch.split(q, [DN, DR], dim=-1)
        kv = ext.linear_forward("gemm", rms(c_kv, L["nkv"]), *L["wkvb"], G).view(1, 1, NH, DN + DV).transpose(1, 2)
        k_nope, v = torch.split(kv, [DN, DV], dim=-1)
        k_pe = k_pe.reshape(1, 1, 1, DR)
        if style == 0:
            q_pe, k_pe = apply_rotary_emb(q_pe, k_pe, cis.index_select(0, pos_l)[None])
        else:
            cos, sin = (t.index_select(0, pos_l)[None].half() for t in cs)
            q_pe, k_pe = apply_rotary_pos_emb_interleave(q_pe, k_pe, cos, sin)
        k_pe = k_pe.expand(*k_nope.shape[:-1], -1)
        q_out.copy_(torch.cat((q_nope, q_pe), dim=-1)[:, :, 0])
        k_cache.index_copy_(1, pos_l, torch.cat((k_nope, k_pe), dim=-1).transpose(1, 2))
        v_cache.index_copy_(1, pos_l, v.transpose(1, 2))

    def build(fold):
        """one step: per layer [program, (c: torch glue), SDPA]; returns the programs, the step functions and the last
        layer's recorded rows / outputs"""
        progs, steps, h = [], [], h0
        last = None
        for li in range(a.layers):
            L, Ln = layers[li], layers[li + 1]
            hm, xn2, h2, xn = (torch.empty((1, H), dtype=torch.float16, device=dev) for _ in range(4))
            act = torch.empty((1, INTER), dtype=torch.float16, device=dev)
            k_cache = torch.zeros((1, S_CACHE, NH, W), dtype=torch.float16, device=dev)
            v_cache = torch.zeros((1, S_CACHE, NH, DV), dtype=torch.float16, device=dev)
            p = DecodeProgram()
            o = p.gemm_forward_cuda(L["attn"], *L["wo"], 8)
            p.add(o, h, out=hm)
            p.layernorm_forward_cuda(hm, L["n2"], xn2, EPS)
            gu = p.gemm_forward_cuda(xn2, *L["gu"], 8)
            p.silu_and_mul(act, gu)
            mo = p.gemm_forward_cuda(act, *L["down"], 8)
            p.add(mo, hm, out=h2)
            p.layernorm_forward_cuda(h2, Ln["n1"], xn, EPS)
            qa = p.gemm_forward_cuda(xn, *Ln["wqa"], 8)
            if fold:
                qan = torch.empty((1, CQ), dtype=torch.float16, device=dev)
                ckv = torch.empty((1, C), dtype=torch.float16, device=dev)
                p.mla_k_rope(qa, freqs, pos, k_cache, NH, DN, DR, C, CQ, style)
                p.layernorm_forward_cuda(qa[:, :CQ], Ln["nq"], qan, EPS)
                qb = p.gemm_forward_cuda(qan, *Ln["wqb"], 8)
                q_out = p.mla_q_rope(qb, freqs, pos, S_CACHE, NH, DN, DR, style)
                p.layernorm_forward_cuda(qa[:, CQ:CQ + C], Ln["nkv"], ckv, EPS)
                kv = p.gemm_forward_cuda(ckv, *Ln["wkvb"], 8)
                p.mla_kv_cache(kv, pos, k_cache, v_cache, NH, DN, DV)
                last = dict(qa=qa, qb=qb, kv=kv, q_out=q_out, k_cache=k_cache, v_cache=v_cache)
            else:
                q_out = torch.empty((1, NH, W), dtype=torch.float16, device=dev)
            p.build()
            progs.append(p)

            def step(p=p, qa=qa, Ln=Ln, q_out=q_out, k_cache=k_cache, v_cache=v_cache):
                p.run()
                if not fold:
                    torch_glue(qa, Ln, k_cache, v_cache, q_out)
                qh = q_out.view(1, NH, 1, W)
                kk = k_cache[:, :P + 1].transpose(1, 2)
                vv = v_cache[:, :P + 1].transpose(1, 2)
                Ln["attn"].copy_(F.scaled_dot_product_attention(qh, kk, vv, scale=scale).reshape(1, NH * DV))
            steps.append(step)
            h = h2
        return progs, steps, last

    pc, sc, _ = build(False)
    pd, sd, last = build(True)
    assert all(p.fused for p in pc), "(c): the programs fuse"
    assert all(p.fused and p.launches_per_run == 1 and p.kernel_ops == 6 for p in pd), "(d): one launch per layer"

    def graph(steps):
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        g = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s):
            for st in steps:
                st()
            torch.cuda.synchronize()
            with torch.cuda.graph(g, stream=s):
                for st in steps:
                    st()
        torch.cuda.current_stream().wait_stream(s)
        return g

    gc, gd = graph(sc), graph(sd)

    def timed(g):
        st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        g.replay()
        st.record()
        for _ in range(a.steps):
            g.replay()
        en.record()
        torch.cuda.synchronize()
        return st.elapsed_time(en) / a.steps

    tc, td = [], []
    for _ in range(a.rounds):
        tc.append(timed(gc))
        td.append(timed(gd))
    rec = DecodeProgram.abort_record()
    assert rec[3] == 0, f"abort record {rec}"
    k2, v2 = torch.zeros_like(last["k_cache"]), torch.zeros_like(last["v_cache"])
    ext.mla_k_rope(last["qa"], freqs, pos, k2, NH, DN, DR, C, CQ, style)
    q2 = ext.mla_q_rope(last["qb"], freqs, pos, S_CACHE, NH, DN, DR, style)
    ext.mla_kv_cache(last["kv"], pos, k2, v2, NH, DN, DV)
    torch.cuda.synchronize()
    assert torch.equal(q2, last["q_out"]), "(d) last layer's q row"
    assert torch.equal(k2[0, P], last["k_cache"][0, P]) and torch.equal(v2[0, P], last["v_cache"][0, P]), "(d) cache rows"
    props = torch.cuda.get_device_properties(dev)
    mc, md = statistics.median(tc), statistics.median(td)
    print(json.dumps(dict(workload=f"DeepSeek-V3 dense decode bs=1, {a.layers} layers, q LoRA MLA glue + SDPA stand-in "
                                   f"over {P + 1} positions, rotary style {style}",
                          gpu=props.name, card=card(), torch_glue_ms=round(mc, 4), folded_ms=round(md, 4),
                          saved_per_layer_us=round((mc - md) * 1000 / a.layers, 2), speedup=round(mc / md, 3),
                          torch_glue_rounds=[round(t, 4) for t in tc], folded_rounds=[round(t, 4) for t in td],
                          self_checks="pass")))


if __name__ == "__main__":
    main()
