#!/usr/bin/env python
"""DeepSeek-V2-Lite decode step at bs = 1 with the MLA glue (seeded random AWQ weights, g128): the programs of
tools/deepseek_moe_decode_bench.py plus everything between them and attention, with the glue left to torch or folded
into the programs.

27 layers as in deepseek_moe_decode_bench.py (layer 0 dense and replayed per op in both arms, layers 1..26
DeepSeek-MoE), with kv_b_proj (512 -> 16 x 256) real W4A16 weights, a yarn-scaled rotary table (V2-Lite's rope
parameters: theta 1e4, factor 40, original 4096, mscale = mscale_all_dim = 0.707) and per layer a KV cache of 2048
positions written at position P = 1023.  Attention is an SDPA stand-in over cache[:, :P + 1] with the model's softmax
scale (192^-0.5 mscale^2), the same in both arms; its output is the next layer's o_proj input.

Arms, each one CUDA graph of the whole step, rounds alternated, medians reported:
  (c) the programs as today (ending at the q_proj | kv_a_proj_with_mqa linear) plus the torch MLA glue: split, kv_a_layernorm
      (transformers' RMSNorm arithmetic), kv_b_proj (ext's W4A16 GEMV), split, rotary (transformers' apply_rotary_emb, or
      apply_rotary_pos_emb_interleave with --sigmoid), expand, cat and the cache writes;
  (d) the programs with mla_rope, kv_a_layernorm (an RMSNorm on the c_kv slice), kv_b_proj and mla_kv_cache recorded in
      them.
Self-checks: (d) is one launch per MoE layer, no abort record, and (d)'s last layer's q row and cache rows equal the
stand-alone ops (ext.mla_rope / ext.mla_kv_cache) run on (d)'s own recorded q|kv_a and kv_b rows.  --sigmoid switches to
Moonlight's routing (as deepseek_moe_decode_bench.py) and rotary style 1 (DeepSeek-V3's interleaved rotation).  Prints
one JSON line."""
import argparse
import json
import math
import os
import statistics
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from autoawq_b200 import ext  # noqa: E402
from autoawq_b200.program import DecodeProgram  # noqa: E402

H, G, E, K_TOP, I, I_S, DENSE_I = 2048, 128, 64, 6, 1408, 2816, 10944
NH, DN, DR, DV, C = 16, 128, 64, 128, 512
W = DN + DR
N_QKVA, N_KV = NH * W + C + DR, NH * (DN + DV)
S_CACHE, P = 2048, 1023
YARN = dict(rope_type="yarn", rope_theta=10000.0, factor=40.0, original_max_position_embeddings=4096, beta_fast=32.0,
            beta_slow=1.0, mscale=0.707, mscale_all_dim=0.707)


def rotary_tables(dev):
    """(freqs_cis complex64 [S, Dr/2], (cos, sin) f32 [S, Dr]) of V2-Lite's yarn rotary embedding"""
    from transformers import DeepseekV2Config
    from transformers.models.deepseek_v2.modeling_deepseek_v2 import DeepseekV2RotaryEmbedding

    cfg = DeepseekV2Config(hidden_size=H, num_attention_heads=NH, q_lora_rank=None, kv_lora_rank=C, qk_nope_head_dim=DN,
                           qk_rope_head_dim=DR, v_head_dim=DV, max_position_embeddings=163840, rope_parameters=YARN)
    rot = DeepseekV2RotaryEmbedding(cfg, device=dev)
    cis = rot(torch.zeros(1, device=dev), torch.arange(S_CACHE, device=dev)[None])[0]
    f = torch.outer(torch.arange(S_CACHE, device=dev).float(), rot.inv_freq.float())
    emb = torch.cat((f, f), dim=-1)
    return cis, (emb.cos() * rot.attention_scaling, emb.sin() * rot.attention_scaling)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=27)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--sigmoid", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    style = 1 if a.sigmoid else 0
    cis, cs = rotary_tables(dev)
    freqs = cis if style == 0 else cs
    mscale = 0.1 * YARN["mscale_all_dim"] * math.log(YARN["factor"]) + 1.0
    scale = W ** -0.5 * mscale * mscale

    def lin(K, N, lead=(), g=G):
        return (torch.randint(-2**31, 2**31 - 1, lead + (K, N // 8), dtype=torch.int32, device=dev, generator=gen),
                ((torch.rand(lead + (K // g, N), device=dev, generator=gen) * 0.5 + 0.75) / (6.1 * K**0.5)).half(),
                torch.randint(-2**31, 2**31 - 1, lead + (K // g, N // 8), dtype=torch.int32, device=dev, generator=gen))

    def norm_w(n=H):
        return (1 + 0.1 * torch.randn(n, device=dev, generator=gen)).half()

    routing = dict(scoring="softmax")
    if a.sigmoid:
        routing = dict(scoring="sigmoid", n_group=1, topk_group=1, norm_topk_prob=True, routed_scaling_factor=2.446)
    layers = []
    for li in range(a.layers + 1):     # (+1: the last program ends with the MLA chain of the layer after the stack)
        L = dict(wo=lin(NH * DV, H), wqkva=lin(H, N_QKVA), wkvb=lin(C, N_KV), n1=norm_w(), n2=norm_w(), nkv=norm_w(C),
                 attn=torch.randn((1, NH * DV), device=dev, generator=gen).half())
        if li == 0:
            L.update(gu=lin(H, 2 * DENSE_I, g=64), down=lin(DENSE_I, H, g=64))
        elif li < a.layers:
            L.update(gate=(torch.randn((E, H), device=dev, generator=gen) * 0.05).half(), w1=lin(H, 2 * I, (E,)),
                     w2=lin(I, H, (E,)), shared=(lin(H, 2 * I_S), lin(I_S, H)),
                     bias=(torch.randn(E, device=dev, generator=gen) * 0.05).float())
        layers.append(L)
    h0 = torch.randn((1, H), device=dev, generator=gen).half()
    pos = torch.tensor([P], dtype=torch.int32, device=dev)
    pos_l = pos.long()

    def torch_glue(qkva, L, k_cache, v_cache, q_out):
        """transformers' DeepseekV2Attention / DeepseekV3Attention between the projections and attention"""
        from transformers.models.deepseek_v2.modeling_deepseek_v2 import apply_rotary_emb
        from transformers.models.deepseek_v3.modeling_deepseek_v3 import apply_rotary_pos_emb_interleave

        q = qkva[:, :NH * W].view(1, 1, NH, W).transpose(1, 2)
        q_nope, q_pe = torch.split(q, [DN, DR], dim=-1)
        c_kv, k_pe = torch.split(qkva[:, NH * W:], [C, DR], dim=-1)
        v32 = c_kv.float()
        c_kv = L["nkv"] * (v32 * torch.rsqrt(v32.pow(2).mean(-1, keepdim=True) + 1e-6)).half()
        kv = ext.linear_forward("gemm", c_kv, *L["wkvb"], G).view(1, 1, NH, DN + DV).transpose(1, 2)
        k_nope, v = torch.split(kv, [DN, DV], dim=-1)
        k_pe = k_pe.view(1, 1, 1, DR)
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
        """one step: per layer [program, (c: torch glue), SDPA]; returns the programs, the step function and the
        last layer's recorded rows / outputs"""
        progs, steps, h = [], [], h0
        last = None
        for li in range(a.layers):
            L, Ln = layers[li], layers[li + 1]
            hm, xn2, h2, xn = (torch.empty((1, H), dtype=torch.float16, device=dev) for _ in range(4))
            k_cache = torch.zeros((1, S_CACHE, NH, W), dtype=torch.float16, device=dev)
            v_cache = torch.zeros((1, S_CACHE, NH, DV), dtype=torch.float16, device=dev)
            p = DecodeProgram()
            o = p.gemm_forward_cuda(L["attn"], *L["wo"], 8)
            p.add(o, h, out=hm)
            p.layernorm_forward_cuda(hm, L["n2"], xn2, 1e-6)
            if li == 0:
                gu = p.gemm_forward_cuda(xn2, *L["gu"], 8)
                act = torch.empty((1, DENSE_I), dtype=torch.float16, device=dev)
                p.silu_and_mul(act, gu)
                mo = p.gemm_forward_cuda(act, *L["down"], 8)
            else:
                kw = dict(routing)
                if a.sigmoid:
                    kw["e_score_correction_bias"] = L["bias"]
                mo = p.deepseek_moe(xn2, L["gate"], L["w1"], L["w2"], K_TOP, L["shared"], **kw)
            p.add(mo, hm, out=h2)
            p.layernorm_forward_cuda(h2, Ln["n1"], xn, 1e-6)
            qkva = p.gemm_forward_cuda(xn, *Ln["wqkva"], 8)
            if fold:
                ckv = torch.empty((1, C), dtype=torch.float16, device=dev)
                q_out = p.mla_rope(qkva, freqs, pos, k_cache, NH, DN, DR, C, style)
                p.layernorm_forward_cuda(qkva[:, NH * W:NH * W + C], Ln["nkv"], ckv, 1e-6)
                kv = p.gemm_forward_cuda(ckv, *Ln["wkvb"], 8)
                p.mla_kv_cache(kv, pos, k_cache, v_cache, NH, DN, DV)
                last = dict(qkva=qkva, kv=kv, q_out=q_out, k_cache=k_cache, v_cache=v_cache)
            else:
                q_out = torch.empty((1, NH, W), dtype=torch.float16, device=dev)
            p.build()
            progs.append(p)

            def step(p=p, qkva=qkva, Ln=Ln, q_out=q_out, k_cache=k_cache, v_cache=v_cache):
                p.run()
                if not fold:
                    torch_glue(qkva, Ln, k_cache, v_cache, q_out)
                qh = q_out.view(1, NH, 1, W)
                kk = k_cache[:, :P + 1].transpose(1, 2)
                vv = v_cache[:, :P + 1].transpose(1, 2)
                Ln["attn"].copy_(F.scaled_dot_product_attention(qh, kk, vv, scale=scale).reshape(1, NH * DV))
            steps.append(step)
            h = h2
        return progs, steps, last

    pc, sc, _ = build(False)
    pd, sd, last = build(True)
    assert all(p.fused and p.launches_per_run == 1 for p in pd[1:]), "(d): one launch per MoE layer"

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
    q2 = ext.mla_rope(last["qkva"], freqs, pos, k2, NH, DN, DR, C, style)
    ext.mla_kv_cache(last["kv"], pos, k2, v2, NH, DN, DV)
    torch.cuda.synchronize()
    assert torch.equal(q2, last["q_out"]), "(d) last layer's q row"
    assert torch.equal(k2[0, P], last["k_cache"][0, P]) and torch.equal(v2[0, P], last["v_cache"][0, P]), "(d) cache rows"
    props = torch.cuda.get_device_properties(dev)
    mc, md = statistics.median(tc), statistics.median(td)
    print(json.dumps(dict(workload=f"DeepSeek-V2-Lite decode bs=1, {a.layers} layers, MLA glue + SDPA stand-in over "
                                   f"{P + 1} positions, {routing['scoring']} routing, rotary style {style}",
                          gpu=props.name, torch_glue_ms=round(mc, 4), folded_ms=round(md, 4),
                          saved_per_layer_us=round((mc - md) * 1000 / a.layers, 2), speedup=round(mc / md, 3),
                          torch_glue_rounds=[round(t, 4) for t in tc], folded_rounds=[round(t, 4) for t in td],
                          self_checks="pass")))


if __name__ == "__main__":
    main()
