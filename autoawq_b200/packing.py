"""Host-side producers of the three packed formats (torch, any device), vectorised.

These mirror what the reference's `from_linear` class methods emit (awq/modules/linear/gemm.py:171-251,
gemv.py:78-153, gemv_fast.py:26-65,120-181) so a model quantised by the reference's AwqQuantizer can be
packed without the O(K) Python loops.  Verified bit-for-bit against the reference's own outputs
(tests/golden/packers.npz) in tests/test_packing.py.
"""
from __future__ import annotations

import torch

PACK_NUM = 8
# nibble i of a GEMM-layout word <- column 8c + AWQ_ORDER[i]  (awq/utils/packing_utils.py:4)
AWQ_ORDER = (0, 2, 4, 6, 1, 3, 5, 7)
AWQ_REVERSE_ORDER = (0, 4, 1, 5, 2, 6, 3, 7)


def calculate_zeros_width(in_features: int, group_size: int = 128, pack_num: int = 8) -> int:
    """Padded width (int32 words) of a GEMV-layout zeros row (gemv.py:12-24)."""
    if group_size >= 128:
        mult = 1
    elif group_size == 64:
        mult = 2
    elif group_size == 32:
        mult = 4
    else:
        raise NotImplementedError
    base = (in_features // group_size + pack_num - 1) // pack_num
    return (base + mult - 1) // mult * mult


def _pack_words(vals: torch.Tensor, nibble_of_col) -> torch.Tensor:
    """[R, 8C] ints in 0..15 -> [R, C] int32; column j of each octet goes to nibble nibble_of_col[j]."""
    R, C8 = vals.shape
    v = vals.to(torch.int64).reshape(R, C8 // PACK_NUM, PACK_NUM) & 0xF
    shifts = torch.tensor([4 * nibble_of_col[j] for j in range(PACK_NUM)], dtype=torch.int64, device=vals.device)
    words = (v << shifts).sum(dim=-1)  # disjoint bit fields: sum == or
    words = torch.where(words >= 2**31, words - 2**32, words)
    return words.to(torch.int32)


def pack_gemm_words(vals: torch.Tensor) -> torch.Tensor:
    return _pack_words(vals, AWQ_REVERSE_ORDER)


def pack_seq_words(vals: torch.Tensor) -> torch.Tensor:
    return _pack_words(vals, tuple(range(PACK_NUM)))


def unpack_gemm_words(words: torch.Tensor) -> torch.Tensor:
    """[R, C] int32 (GEMM interleave) -> [R, 8C] uint8 in natural column order."""
    shifts = torch.tensor([4 * r for r in AWQ_REVERSE_ORDER], dtype=torch.int32, device=words.device)
    v = (words.unsqueeze(-1) >> shifts) & 0xF
    return v.reshape(words.shape[0], -1).to(torch.uint8)


def quantize_to_int(weight_nk: torch.Tensor, scales_ng: torch.Tensor, zeros_ng: torch.Tensor, group_size: int):
    """round((W + z*s) / s) per group, the integer recovery `from_linear` performs (gemm.py:196-203):
    W [N, K] (already pseudo-quantised), scales / zeros [N, K/G] -> ints [N, K] (no clamp, as the reference)."""
    N, K = weight_nk.shape
    s = scales_ng.to(torch.float16).repeat_interleave(group_size, dim=1)  # fp16 scales, as stored
    sz = (zeros_ng * scales_ng).repeat_interleave(group_size, dim=1)
    return torch.round((weight_nk + sz) / s).to(torch.int32)


def pack_gemm(intweight_nk: torch.Tensor, zeros_ng: torch.Tensor, scales_ng: torch.Tensor):
    """-> qweight [K, N/8] i32, qzeros [K/G, N/8] i32, scales [K/G, N] f16 (checkpoint default `version="gemm"`)."""
    qweight = pack_gemm_words(intweight_nk.t().contiguous())
    qzeros = pack_gemm_words(zeros_ng.t().contiguous().to(torch.int32))
    return qweight, qzeros, scales_ng.t().contiguous().to(torch.float16)


def pack_gemv(intweight_nk: torch.Tensor, zeros_ng: torch.Tensor, scales_ng: torch.Tensor, group_size: int):
    """-> qweight [N, K/8] i32 (sequential nibbles), qzeros [N, zw] i32, scales [N, 8 zw] f16 (zero padded)."""
    N, K = intweight_nk.shape
    zw = calculate_zeros_width(K, group_size)
    ng = K // group_size
    qweight = pack_seq_words(intweight_nk)
    z = torch.zeros((N, zw * PACK_NUM), dtype=torch.int32, device=intweight_nk.device)
    z[:, :ng] = zeros_ng.to(torch.int32)
    s = torch.zeros((N, zw * PACK_NUM), dtype=torch.float16, device=intweight_nk.device)
    s[:, :ng] = scales_ng.to(torch.float16)
    return qweight, pack_seq_words(z), s


def _fast_kperm(device) -> torch.Tensor:
    a = torch.arange(32, device=device).reshape(4, 4, 2).permute(1, 0, 2).reshape(32)
    return a.reshape(4, 4, 2).permute(0, 2, 1).reshape(32)


def pack_gemv_fast_weight(intweight_nk: torch.Tensor, interleave: int = 4, kstride: int = 64) -> torch.Tensor:
    """ints [N, K] -> int16 [N/4, K] (gemv_fast.py:26-65)."""
    N, K = intweight_nk.shape
    w = intweight_nk.to(torch.int32).reshape(N, K // 32, 32)[:, :, _fast_kperm(intweight_nk.device)].reshape(N, K)
    w = w.reshape(N // interleave, interleave, K // kstride, kstride).permute(0, 2, 1, 3).contiguous()
    w = w.reshape(N // interleave, K // kstride, kstride, interleave)
    packed = w[..., 0] | (w[..., 1] << 4) | (w[..., 2] << 8) | (w[..., 3] << 12)
    packed = torch.where(packed >= 2**15, packed - 2**16, packed)
    return packed.reshape(N // interleave, K).to(torch.int16)


def pack_gemv_fast(intweight_nk, zeros_ng, scales_ng, group_size: int):
    """-> qweight i16 [N/4, K], scales f16 [8 zw, N], scaled zeros f16 [8 zw, N] = -(s * z) (gemv_fast.py:146-181)."""
    N, K = intweight_nk.shape
    zw = calculate_zeros_width(K, group_size)
    ng = K // group_size
    qs = torch.zeros((N, zw * PACK_NUM), dtype=torch.float16, device=intweight_nk.device)
    qs[:, :ng] = scales_ng.to(torch.float16)
    qz = torch.zeros_like(qs)
    qz[:, :ng] = -(qs[:, :ng] * zeros_ng.to(torch.float32)).to(torch.float16)
    return pack_gemv_fast_weight(intweight_nk), qs.t().contiguous(), qz.t().contiguous()


def stack_experts(block):
    """(gate_weight, w1, w2, top_k, norm_topk_prob) of a transformers-4.5x-shaped MoE block (Qwen3MoeSparseMoeBlock:
    `.gate` nn.Linear, `.experts[e].{gate,up,down}_proj` with qweight / scales / qzeros, `.top_k`, `.norm_topk_prob`),
    in the form DecodeProgram.qwen3_moe takes: w1 = (qweight, scales, qzeros) of [gate | up] concatenated along N and
    stacked over the experts ([E, H, 2I/8], [E, H/G, 2I], [E, H/G, 2I/8]), w2 = the stacked down_proj tensors (the
    concatenation and torch.stack of the reference's Mixtral fuser, awq/models/mixtral.py:131-151)."""
    experts = list(block.experts)

    def cat(a, b):
        return torch.cat((a, b), dim=1)

    w1 = tuple(torch.stack([cat(getattr(e.gate_proj, t), getattr(e.up_proj, t)) for e in experts], dim=0)
               for t in ("qweight", "scales", "qzeros"))
    w2 = tuple(torch.stack([getattr(e.down_proj, t) for e in experts], dim=0) for t in ("qweight", "scales", "qzeros"))
    return (block.gate.weight.detach().contiguous(), w1, w2, int(block.top_k),
            bool(getattr(block, "norm_topk_prob", True)))


def stack_deepseek_experts(block):
    """(gate_weight, w1, w2, top_k, shared, routing) of a DeepSeek-V2 / V3 MoE block in the layout the reference
    quantises (awq/models/deepseek_v2.py, deepseek_v3.py: `.gate` with `.weight` and, for V3, `.e_score_correction_bias`,
    `.experts[e].{gate,up,down}_proj` and `.shared_experts.{gate,up,down}_proj` with qweight / scales / qzeros, and the
    routing config `top_k`, `routed_scaling_factor`, `n_group` (or V2's `num_group`), `topk_group`, `norm_topk_prob`),
    in the form DecodeProgram.deepseek_moe takes: prog.deepseek_moe(x, gate_weight, w1, w2, top_k, shared, **routing).
    w1 / w2 as stack_experts; shared = ((qweight, scales, qzeros) of [gate | up] along N, those of down).  A gate with
    e_score_correction_bias scores with sigmoid (V3), one without with softmax (V2 greedy)."""
    gate_weight, w1, w2, top_k, _ = stack_experts(block)
    sh = block.shared_experts

    def cat(t):
        return torch.cat((getattr(sh.gate_proj, t), getattr(sh.up_proj, t)), dim=1).contiguous()

    shared = (tuple(cat(t) for t in ("qweight", "scales", "qzeros")),
              tuple(getattr(sh.down_proj, t).contiguous() for t in ("qweight", "scales", "qzeros")))
    bias = getattr(block.gate, "e_score_correction_bias", None)
    n_group = int(getattr(block, "n_group", getattr(block, "num_group", 1)) or 1)
    routing = dict(scoring="sigmoid" if bias is not None else "softmax",
                   e_score_correction_bias=None if bias is None else bias.detach().float().contiguous(),
                   n_group=n_group if bias is not None else 1,
                   topk_group=int(getattr(block, "topk_group", 1) or 1) if bias is not None else 1,
                   norm_topk_prob=bool(getattr(block, "norm_topk_prob", False)),
                   routed_scaling_factor=float(getattr(block, "routed_scaling_factor", 1.0)))
    return gate_weight, w1, w2, top_k, shared, routing


def fuse_mla_input(attn):
    """(qweight, scales, qzeros, bias) of the fused q_proj | kv_a_proj_with_mqa linear of a transformers
    DeepseekV2Attention / DeepseekV3Attention without a q LoRA whose two projections are WQLinear_GEMM modules: both read
    the hidden state, so one GEMM-layout linear with N = H (Dn + Dr) + C + Dr gives the row [q | c_kv | k_pe] that
    DecodeProgram.mla_rope takes (loader.fuse_columns' concatenation along N).  bias is None when neither projection
    has one."""
    from .loader import fuse_columns
    from .shard import PackedGemm

    if getattr(attn, "q_lora_rank", None) is not None:
        raise ValueError("fuse_mla_input: the attention has a q LoRA (q_a_proj / q_b_proj); only q_proj is supported")
    parts = [PackedGemm(m.qweight, m.qzeros, m.scales, getattr(m, "bias", None))
             for m in (attn.q_proj, attn.kv_a_proj_with_mqa)]
    f = fuse_columns(parts)
    return f.qweight, f.scales, f.qzeros, f.bias


def fuse_mla_lora_input(attn):
    """(qweight, scales, qzeros, bias) of the fused q_a_proj | kv_a_proj_with_mqa linear of a transformers
    DeepseekV2Attention / DeepseekV3Attention WITH a q LoRA (q_lora_rank set) whose two projections are WQLinear_GEMM
    modules: both read the hidden state, so one GEMM-layout linear with N = Cq + C + Dr gives the row [q_a | c_kv | k_pe]
    that DecodeProgram.mla_k_rope takes (loader.fuse_columns' concatenation along N).  bias is None when neither
    projection has one."""
    from .loader import fuse_columns
    from .shard import PackedGemm

    if getattr(attn, "q_lora_rank", None) is None:
        raise ValueError("fuse_mla_lora_input: the attention has no q LoRA; use fuse_mla_input")
    parts = [PackedGemm(m.qweight, m.qzeros, m.scales, getattr(m, "bias", None))
             for m in (attn.q_a_proj, attn.kv_a_proj_with_mqa)]
    f = fuse_columns(parts)
    return f.qweight, f.scales, f.qzeros, f.bias
