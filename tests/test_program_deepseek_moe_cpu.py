"""Host logic of DEEPSEEK_MOE blocks in stream decode programs, checked without a GPU: b200awq_deepseek_moe_plan at
DeepSeek-V2-Lite / Moonlight shapes and every envelope rejection, the ctypes descriptor and op constant against the
header, the folding of a trailing residual add, the register / spill budget of stream_deepseek_moe_kernel, the SASS of
the pre-existing entries against a given revision, the numpy routing oracle (which the GPU tests hold the kernel to)
against transformers' own route_tokens_to_experts, and the shared-expert loader against packing.stack_deepseek_experts."""
import ctypes
import types

import numpy as np
import pytest

from _fake_ops import add, buf, plan
from _toolchain import entries, header_constants, header_layout, mirror_layout, needs_nvcc, sass_compare
from autoawq_b200 import _cabi
from autoawq_b200._cabi import lib


def route_oracle(logits, top_k, scoring, bias=None, n_group=1, topk_group=1, norm=False, rsf=1.0):
    """DeepSeek routing of one token's fp32 logits in numpy fp32: (ids in slot order, fp32 weights).  Ties go to the
    lower expert / group (stable sorts), as the kernel breaks them."""
    l = np.asarray(logits, dtype=np.float32)
    E = l.size
    f32 = np.float32
    if scoring == "softmax":
        e = np.exp(l - l.max()).astype(f32)
        p = (e / e.sum(dtype=f32)).astype(f32)
        ids = np.argsort(-p, kind="stable")[:top_k]
        return ids, (p[ids] * f32(rsf)).astype(f32)
    s = (f32(1) / (f32(1) + np.exp(-l))).astype(f32)
    c = (s + np.asarray(bias, dtype=f32)).astype(f32)
    if topk_group < n_group:
        grp = c.reshape(n_group, E // n_group)
        top2 = -np.sort(-grp, axis=1)[:, :2]
        gs = (top2[:, 0] + top2[:, 1]).astype(f32)
        keep = np.zeros(n_group, dtype=bool)
        keep[np.argsort(-gs, kind="stable")[:topk_group]] = True
        c = np.where(np.repeat(keep, E // n_group), c, f32(0)).astype(f32)
    ids = np.argsort(-c, kind="stable")[:top_k]
    w = s[ids].astype(f32)
    if norm:
        den = f32(0)
        for v in w:
            den = f32(den + v)
        w = (w / f32(den + f32(1e-20))).astype(f32)
    return ids, (w * f32(rsf)).astype(f32)


def _plan(E, k, H, I, I_s, G, sms=132):
    out = (ctypes.c_int * 8)()
    return lib.b200awq_deepseek_moe_plan(E, k, H, I, I_s, G, sms, out), list(out)


@pytest.mark.parametrize("k,E", [(6, 64)])      # DeepSeek-V2-Lite and Moonlight-16B-A3B: E 64, top-6
def test_plan_v2_lite_moonlight(k, E):
    rc, p = _plan(E, k, 2048, 1408, 2816, 128)
    assert rc == 0
    sets_a = (k * 2 * 1408 + 2 * 2816) // 16
    assert sets_a == 1408 and p[1] == sets_a and p[3] == 11          # 11 gate|up sets per CTA on 132 SMs
    assert p[4] == (k * 1408 + 2816) // 128 == 88                   # K' = 11264
    assert p[5] == 1408 // 128 and p[6] == 1 * (k + 2)              # one set per CTA: 6 slot rows + 2 shared rows
    assert p[7] <= 227 * 1024


@pytest.mark.parametrize("args,rc", [
    ((129, 8, 2048, 768, 1536, 128), 2),            # E > 128
    ((128, 9, 2048, 768, 1536, 128), 2),            # top_k > 8
    ((64, 6, 2048, 1408, 2816 + 128, 128), 2),      # I_s not a multiple of I
    ((64, 6, 2048, 1408, 2816, 96), 2),             # group size outside the stream format
    ((64, 8, 2048, 4096, 4 * 4096, 32), 2),         # K' / UK = (8 x 4096 + 16384) / 32 = 1536 > 1024
    ((64, 8, 2048, 1408, 8 * 1408, 128), 0),        # K' = 22528: 176 units, 45 KB of activations
    ((64, 6, 2048, 1408, 0, 128), 1), ((0, 1, 2048, 768, 768, 128), 1), ((4, 5, 2048, 768, 768, 128), 1),
    ((128, 8, 2048, 768, 768, 64), 0), ((64, 6, 1024, 512, 1024, 64), 0)])
def test_plan_envelope(args, rc):
    assert _plan(*args)[0] == rc


def test_plan_partial_row_limit():
    # 4096 / 16 = 256 sets over 132 CTAs: 2 per CTA x (8 + 4) rows = 24 <= 32; with 30 SMs 9 x 12 > 32
    assert _plan(64, 8, 4096, 512, 2048, 128)[0] == 0
    assert _plan(64, 8, 4096, 512, 2048, 128, sms=30)[0] == 2


def _desc(E=64, k=6, H=2048, I=1408, I_s=2816, G=128, scoring=1, n_group=1, topk_group=1):
    """A DEEPSEEK_MOE descriptor with placeholder addresses (the plan makes no CUDA call and reads no tensor)."""
    d = _cabi.DeepseekMoe()
    m = d.moe
    m.E, m.top_k, m.renormalize, m.group_size, m.H, m.I, m.block_size = E, k, 0, G, H, I, 16
    m.sorted_len = k + E * 15
    m.gate_weight = buf(E * H * 2)
    m.w1_qweight, m.w1_scales, m.w1_qzeros = buf(E * H * I), buf(E * H // G * 2 * I * 2), buf(E * H // G * I)
    m.w2_qweight, m.w2_scales, m.w2_qzeros = buf(E * I * H // 2), buf(E * I // G * H * 2), buf(E * I // G * H // 2)
    for f, n in (("logits", E * 4), ("topk_weights", k * 4), ("topk_ids", k * 4), ("token_expert_indices", k * 4),
                 ("sorted_ids", m.sorted_len * 4), ("expert_ids", (k + E) * 4), ("num_tokens_post_pad", 4),
                 ("gate_up", (k * 2 * I + 2 * I_s) * 2), ("act", (k * I + I_s) * 2), ("down", k * H * 2)):
        setattr(m, f, buf(n))
    d.scoring, d.n_group, d.topk_group, d.norm_topk_prob, d.routed_scaling_factor = scoring, n_group, topk_group, 1, 2.5
    d.I_s = I_s
    d.bias = buf(E * 4)
    d.ws1_qweight, d.ws1_scales, d.ws1_qzeros = buf(H * I_s), buf(H // G * 2 * I_s * 2), buf(H // G * I_s)
    d.ws2_qweight, d.ws2_scales, d.ws2_qzeros = buf(I_s * H // 2), buf(I_s // G * H * 2), buf(I_s // G * H // 2)
    d.shared_out = buf(H * 2)
    return d


def _ops(d, with_add=False):
    H = d.moe.H
    ops = [dict(kind=_cabi.OP_DEEPSEEK_MOE, M=1, K=H, N=H, x=buf(H * 2), y=buf(H * 2), weight=ctypes.addressof(d))]
    if with_add:
        ops.append(add(ops[0]["y"], buf(H * 2), H))
    return ops


@pytest.mark.parametrize("with_add", [False, True])
def test_trailing_add_folds_into_down(with_add):
    d = _desc()
    assert plan(_ops(d, with_add)) == (0, 2)               # gate|up (with the routing and the shared expert), down (+ the add)


@pytest.mark.parametrize("field,value", [("scoring", 2), ("n_group", 0), ("n_group", 5), ("topk_group", 0),
                                         ("topk_group", 9), ("I_s", 100), ("bias", None), ("shared_out", None),
                                         ("ws2_qzeros", None)])
def test_bad_descriptor_is_einval(field, value):
    d = _desc(n_group=8, topk_group=4)
    setattr(d, field, value)
    assert plan(_ops(d))[0] == 1


def test_softmax_needs_no_bias():
    d = _desc(scoring=0)
    d.bias = None
    assert plan(_ops(d))[0] == 0


def test_layout_and_op_constant_match_header():
    assert header_layout(_cabi.DeepseekMoe, "b200awq_deepseek_moe_t") == mirror_layout(_cabi.DeepseekMoe)
    assert header_constants("B200AWQ_OP_DEEPSEEK_MOE") == (_cabi.OP_DEEPSEEK_MOE,)


@needs_nvcc
def test_entry_register_and_spill_budget():
    """stream_deepseek_moe_kernel (288 threads, one CTA per SM) fits the register file.  It spills at most 8 bytes: two
    per-op values (the thread index and the CTA's first set) stored before the unit loop and reloaded around it, never
    inside it; the other MoE entries spill nothing (test_program_qwen3moe_cpu.py)."""
    found = entries("program.cu", "stream_deepseek_moe_kernel")
    assert found
    regs, stack, st, ld = next(iter(found.values()))
    assert regs * (32 + 32 * 8) <= 65536 and st <= 8 and stack <= 8, (regs, st, ld, stack)


@needs_nvcc
def test_existing_entries_sass_unchanged():
    """With B200AWQ_SASS_BASE set to a git revision (the commit before this op), every entry both trees have compiles
    to the same SASS (tools/sass_unchanged.py): the DeepSeek code sits behind SP_DEEPSEEK and its own side table.
    Unset, the test is skipped."""
    res = sass_compare()
    assert res, "no entry to compare"
    assert all(res.values()), [n for n, same in res.items() if not same]


def _hf_moe(version, E, k, n_group, topk_group, norm, rsf):
    """transformers' DeepseekV2Moe / DeepseekV3MoE route_tokens_to_experts on a config-only instance (no weights)."""
    import torch

    if version == 2:
        from transformers.models.deepseek_v2.modeling_deepseek_v2 import DeepseekV2Moe as Cls
        blk = Cls.__new__(Cls)
        torch.nn.Module.__init__(blk)
        blk.routed_scaling_factor, blk.topk_method, blk.num_group, blk.top_k, blk.topk_group = rsf, "greedy", 1, k, 1
        return blk
    from transformers.models.deepseek_v3.modeling_deepseek_v3 import DeepseekV3MoE as Cls
    blk = Cls.__new__(Cls)
    torch.nn.Module.__init__(blk)
    blk.n_routed_experts, blk.n_group, blk.topk_group, blk.norm_topk_prob = E, n_group, topk_group, norm
    blk.routed_scaling_factor, blk.top_k = rsf, k
    blk.gate = types.SimpleNamespace(e_score_correction_bias=None)
    return blk


@pytest.mark.parametrize("version,E,k,n_group,topk_group,norm,rsf", [
    (2, 64, 6, 1, 1, False, 1.0), (2, 64, 6, 1, 1, False, 16.0),          # V2-Lite greedy
    (3, 64, 6, 1, 1, True, 2.446), (3, 64, 6, 1, 1, False, 2.446),        # Moonlight
    (3, 128, 8, 8, 4, True, 2.5), (3, 128, 8, 8, 4, False, 1.0), (3, 64, 4, 4, 2, True, 1.0)])
def test_routing_oracle_matches_transformers(version, E, k, n_group, topk_group, norm, rsf):
    import torch

    blk = _hf_moe(version, E, k, n_group, topk_group, norm, rsf)
    rng = np.random.default_rng(E * k + n_group + int(rsf * 10))
    for t in range(20):
        logits = (rng.standard_normal(E) * 2).astype(np.float32)
        bias = (rng.standard_normal(E) * 0.3).astype(np.float32) if version == 3 else None
        if version == 3:
            blk.gate.e_score_correction_bias = torch.from_numpy(bias)
            ids_t, w_t = blk.route_tokens_to_experts(torch.from_numpy(logits)[None])
        else:
            ids_t, w_t = blk.route_tokens_to_experts(torch.from_numpy(logits)[None, None])
        ids, w = route_oracle(logits, k, "softmax" if version == 2 else "sigmoid", bias, n_group, topk_group, norm, rsf)
        order = np.argsort(ids)
        ref_ids, ref_w = ids_t[0].numpy(), w_t[0].numpy()
        ro = np.argsort(ref_ids)
        assert (ids[order] == ref_ids[ro]).all(), t
        assert np.allclose(w[order], ref_w[ro], rtol=4 * 2**-23, atol=0), t


def test_load_shared_expert_matches_stack_deepseek_experts(tmp_path):
    """A two-shard checkpoint of a DeepSeek-V3-shaped block: the stacked experts and the shared expert read from the
    shards equal packing.stack_deepseek_experts on the same modules, routing config included."""
    import json

    import torch
    from safetensors.torch import save_file

    from autoawq_b200 import packing
    from autoawq_b200.loader import load_shared_expert, load_stacked_experts

    E, H, I, I_s, G = 4, 256, 128, 256, 64
    gen = torch.Generator().manual_seed(0)

    def lin(K, N):
        return types.SimpleNamespace(
            qweight=torch.randint(-2**31, 2**31 - 1, (K, N // 8), dtype=torch.int32, generator=gen),
            scales=torch.rand((K // G, N), generator=gen).half(),
            qzeros=torch.randint(-2**31, 2**31 - 1, (K // G, N // 8), dtype=torch.int32, generator=gen))

    def mlp(i):
        return types.SimpleNamespace(gate_proj=lin(H, i), up_proj=lin(H, i), down_proj=lin(i, H))

    experts = [mlp(I) for _ in range(E)]
    shared = mlp(I_s)
    bias = torch.randn(E)
    block = types.SimpleNamespace(gate=types.SimpleNamespace(weight=torch.randn(E, H).half(), e_score_correction_bias=bias),
                                  experts=experts, shared_experts=shared, top_k=2, n_group=2, topk_group=1,
                                  norm_topk_prob=True, routed_scaling_factor=2.5)
    prefix = "model.layers.1.mlp"
    shards, wmap = [{}, {}], {}
    mods = [(f"experts.{e}", ex) for e, ex in enumerate(experts)] + [("shared_experts", shared)]
    for j, (name, mod) in enumerate(mods):
        for proj in ("gate_proj", "up_proj", "down_proj"):
            for t in ("qweight", "scales", "qzeros"):
                key = f"{prefix}.{name}.{proj}.{t}"
                s = (j + len(proj)) % 2
                shards[s][key] = getattr(getattr(mod, proj), t)
                wmap[key] = f"model-{s}.safetensors"
    for s in range(2):
        save_file(shards[s], str(tmp_path / f"model-{s}.safetensors"))
    (tmp_path / "model.safetensors.index.json").write_text(json.dumps({"weight_map": wmap}))
    w1, w2 = load_stacked_experts(str(tmp_path), prefix, E, "cpu")
    ws1, ws2 = load_shared_expert(str(tmp_path), prefix, "cpu")
    gw, r1, r2, k, rshared, routing = packing.stack_deepseek_experts(block)
    assert k == 2 and torch.equal(gw, block.gate.weight)
    assert routing == dict(scoring="sigmoid", e_score_correction_bias=routing["e_score_correction_bias"], n_group=2,
                           topk_group=1, norm_topk_prob=True, routed_scaling_factor=2.5)
    assert torch.equal(routing["e_score_correction_bias"], bias)
    for a, b in zip(w1 + w2 + ws1 + ws2, r1 + r2 + rshared[0] + rshared[1]):
        assert a.dtype == b.dtype and torch.equal(a, b)
    with pytest.raises(KeyError):
        load_shared_expert(str(tmp_path), "model.layers.2.mlp", "cpu")
