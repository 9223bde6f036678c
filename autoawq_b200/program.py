"""Decode programs: record the awq_ext-facing operator calls of one decode step, run them as ONE persistent
kernel (csrc/program.cu, C ABI b200awq_program_*).

The recorder exposes the same call names and argument order as `awq_ext` (`layernorm_forward_cuda`,
`gemm_forward_cuda`, `silu_and_mul` - call sites awq/modules/fused/norm.py:33-36, fused/mlp.py:41-55,
fused/moe.py:76), so the code that drives a fused block (awq/modules/fused/block.py:117-170) can be pointed at
a `DecodeProgram` once, and `run()` replays it every token:

    prog = DecodeProgram()
    prog.layernorm_forward_cuda(h, w_norm, xn, eps)      # buffers are captured by address: refill h in place
    qkv = prog.gemm_forward_cuda(xn, qweight, scales, qzeros, 8)
    ...
    prog.build()
    prog.run()                               # one memset + one kernel on torch's current stream

If the sequence does not fit the fused kernel (M != 1, unsupported shape, aliasing) `build()` keeps the op list and
`run()` issues the per-op entry points instead - still the CUDA path, `prog.fused` tells which.

A fused block built for batch size B (every call has B rows) is fused when the program is created with
`DecodeProgram(max_tokens=B)`, B <= 8: one persistent kernel then runs all B tokens (csrc/program_batch.cuh), each
bit-identical to an M = 1 program on that token's row.  Without it, M > 1 replays the per-op kernels as before.

`sparse_moe(x, gate_weight, w1, w2, top_k)` records a whole Mixtral sparse-MoE block (FusedSparseMoeBlock.forward);
at M = 1 the stream kernel runs it as two kernel ops with the routing computed inside (DESIGN.md 3.5d), otherwise
`run()` replays apply_moe_weights' sequence through ext.  `moe_buffers(i)` returns the block's routing and intermediates.

`qwen3_moe(x, gate_weight, w1, w2, top_k, norm_topk_prob)` records a Qwen3-MoE expert block with the arithmetic of
transformers' Qwen3MoeSparseMoeBlock (fp16 routing weights, the experts combined in ascending id with fp16 adds); at
M = 1 the stream kernel runs it as two kernel ops with the router logits exchanged across the grid (DESIGN.md 3.5h).
`packing.stack_experts(block)` gives its arguments from a loaded block.

`deepseek_moe(x, gate_weight, w1, w2, top_k, shared, scoring, ...)` records a DeepSeek-V2 / V3 expert block
(transformers' DeepseekV2Moe / DeepseekV3MoE over WQLinear_GEMM experts): fp32 router logits, softmax or sigmoid routing
with expert groups and the correction bias, fp32 weights, the routed experts combined in ascending id, and the dense
shared expert added last; at M = 1 the stream kernel runs it as two kernel ops with the shared expert's weights
streamed while the router logits are exchanged (DESIGN.md 3.5i).  `packing.stack_deepseek_experts(block)` gives its
arguments from a loaded block.

`add(a, b)` records the decoder block's residual add (`h = hidden_states + attn_output`, awq/modules/fused/block.py:
50-52,117-118).  It adds no kernel op: it folds into the epilogue of the linear (or sparse_moe) recorded just before it,
so a layer splits only at attention - [o + h_in -> h, norm2(h), gate|up, silu, down + h -> out, norm1'(out), qkv'] is one
program (DESIGN.md 3.5e).  Outside the folding rule `run()` replays per op, with `torch.add` for the adds.

`scaled_add(residual, y, a)` records the depth-scaled residual add of MiniCPM / MiniCPM3 (a = scale_depth /
sqrt(num_hidden_layers)) and Granite (a = residual_multiplier): out = residual + y * a with torch's rounding,
fp16(r + fp16(y a)) with a in fp32.  It folds where add folds, with y the whole output of the linear recorded just
before (DESIGN.md 3.5p), so a MiniCPM / Granite segment [o, scaled_add, norm2, gate|up, silu, down, scaled_add,
norm1', qkv', rope_kv_cache] is one launch, and a MiniCPM3 segment (the same MLP, then the q-LoRA MLA chain below) too.
Per op it replays torch.mul then torch.add.  The embedding and logit scales and Granite's attention_multiplier (the
softmax scale) stay with the caller.

`rope_kv_cache(qkv, freqs_cis, pos, k_cache, v_cache, n_heads, n_kv_heads)` records the start of the attention block
(RoPE.forward on q and k, WindowedCache.update_kv of k and v: awq/modules/fused/attn.py:243-267).  It adds no kernel
op either: it folds into the finish of the qkv linear recorded just before it, so the segment ends with q rotated and
the cache row written, and attention reads them directly (DESIGN.md 3.5f).  `pos` is a device int32 tensor: advance it
in place between runs (or graph replays).  With `q_norm=` / `k_norm=` (Qwen3's Qwen3RMSNorm modules) it also applies
Qwen3's per-head q / k norm first, still inside the qkv linear's finish (DESIGN.md 3.5g).

A step of T tokens per sequence (speculative verification of a T-token draft, multi-token prediction, a prompt
continued in chunks) records the same segment with M = B T rows, in the reference's order (xqkv viewed as [B, T, N]):
o + x -> h, norm2(h), gate|up, silu, down + h -> out, norm1'(out), qkv', `rope_kv_cache(..., seq_len=T)`.  Row
m = b T + t is token t of sequence b at position *pos + t, written to cache entry b; attention (with the causal mask
over the new tokens) stays the caller's, between programs.  `DecodeProgram(max_tokens=B T)` runs the segment as one
launch (B T <= 8; DESIGN.md 3.5n); advance `pos` by T per step.

When a sequence's rotary position differs from its cache row (a left-padded batch: `rope_offset = -pad`; a Qwen2-VL /
Qwen2.5-VL text step: the M-RoPE delta of each sequence), `rope_kv_cache(..., rope_offset=off)` takes a device int32
tensor of B per-sequence offsets: row m = b T + t is written to cache row *pos + t of entry b and rotated at *pos + t
+ off[b].  It folds wherever the op without offsets folds (DESIGN.md 3.5o); rewrite `off` in place between runs, like
`pos`.

`mla_rope(qkva, freqs, pos, k_cache, ...)` and `mla_kv_cache(kv, pos, k_cache, v_cache, ...)` record the glue of
DeepSeek-V2 / V3 multi-head latent attention (transformers' DeepseekV2Attention / DeepseekV3Attention, no q LoRA) in
transformers' order: the fused q_proj | kv_a_proj_with_mqa linear (packing.fuse_mla_input), mla_rope, kv_a_layernorm as
an RMSNorm on the c_kv slice of that linear's output, kv_b_proj, mla_kv_cache.  Each folds into the finish of the linear
recorded just before it, so at M = 1 a DeepSeek segment runs as one launch from one attention call to the next
(DESIGN.md 3.5j).

With a q LoRA (DeepSeek-V2 / V2.5 / V3, MiniCPM3) the order is: the fused q_a_proj | kv_a_proj_with_mqa linear
(packing.fuse_mla_lora_input), `mla_k_rope`, q_a_layernorm as an RMSNorm on the q_a slice of that linear's output,
q_b_proj, `mla_q_rope`, kv_a_layernorm on its c_kv slice, kv_b_proj, mla_kv_cache.  At M = 1 the chain is three
kernel ops of one launch (DESIGN.md 3.5k).

`layer_norm(x, weight, bias, out, eps)` records an nn.LayerNorm (bias None: transformers' CohereLayerNorm) and
`gelu(out, x, approximate)` an F.gelu ("tanh" or "none").  At M = 1 the LayerNorm runs in the staging of every linear
that reads its output, as layernorm_forward_cuda's RMSNorm does, and the GELU in the finish of the linear recorded just
before it (DESIGN.md 3.5l).  Programs built with max_tokens > 1 replay them per op.  The recording order of one segment,
from one attention call to the next:

  * Command-R (CohereBlock, parallel residual): o + x -> h, gate|up(xn) (gate and up concatenated along N, as
    packing.fuse_qkv concatenates q, k and v), silu_and_mul, down + h -> x', layer_norm(x') -> xn' (no bias), qkv',
    rope_kv_cache.  xn and xn' may be one buffer.
  * StarCoder2 (LlamaLikeBlock): o + x -> h, layer_norm(h), c_fc, gelu("tanh"), c_proj + h -> x', layer_norm(x'), qkv',
    rope_kv_cache.  Every linear has a bias.
  * MPT (MPTBlock): the StarCoder2 order with gelu("none"), no biases and no rope_kv_cache: ALiBi stays in the caller's
    attention, so the segment ends at Wqkv.
  * StableLM (StableLmFuser's LlamaLikeBlock with partial_rotary_factor): o + x -> h, layer_norm(h)
    (post_attention_layernorm, with bias), gate|up (concatenated along N), silu_and_mul, down + h -> x', layer_norm(x')
    (next input_layernorm), qkv' (with its bias on StableLM-2), rope_kv_cache(..., head_dim=D) with freqs_cis the
    table of the R = D x partial_rotary_factor rotated columns.  Four kernel ops, one launch at M = 1 (DESIGN.md 3.5m).
"""
from __future__ import annotations

import ctypes
import math

import torch

from . import _cabi, ext
from ._cabi import B200AwqError, Op, check, lib


# the recorded MLA ops: kind -> op constant (the stand-alone entry is b200awq_<kind>)
_MLA_OPS = {"mla_rope": _cabi.OP_MLA_ROPE, "mla_kv": _cabi.OP_MLA_KV, "mla_k_rope": _cabi.OP_MLA_K_ROPE,
            "mla_q_rope": _cabi.OP_MLA_Q_ROPE}


class DecodeProgram:
    def __init__(self, max_tokens: int = 1):
        if not 1 <= int(max_tokens) <= 8:
            raise B200AwqError("b200awq: max_tokens must be in 1..8")
        self.max_tokens = int(max_tokens)  # > 1: build() may fuse a sequence recorded with up to this many rows per op
        self._ops: list = []          # (kind, dict of tensors / scalars)
        self._keep: list = []         # every tensor named by an op stays alive with the program
        self._handle = None
        self._built = False
        self._dev = None
        self.calibration = None       # kept for callers that record it: there is one kernel, nothing is calibrated

    # ------------------------------------------------------------------ recording (awq_ext call names)
    def _dev_of(self, t: torch.Tensor):
        ext._require_cuda(t)
        if self._dev is None:
            self._dev = t.device
        elif t.device != self._dev:
            raise B200AwqError("b200awq: a decode program lives on one device")

    def _no_more(self):
        if self._built:
            raise B200AwqError("b200awq: program already built")

    def layernorm_forward_cuda(self, x, weight, out, eps):
        """x may also be rows of a wider tensor (unit stride, one row pitch: kv_a_layernorm on the c_kv slice of
        M > 1 q_proj | kv_a_proj_with_mqa rows).  Such a source has its pitch recorded (ldx); the fused kernels stage
        contiguous rows only, so a program with one replays per op."""
        self._no_more()
        self._dev_of(x)
        if x.dtype != torch.float16 or weight.dtype != torch.float16 or out.dtype != torch.float16:
            raise B200AwqError("b200awq: rmsnorm expects float16 tensors")
        hidden = x.shape[-1]
        ldx = 0
        if not x.is_contiguous():
            x2 = x.reshape(-1, hidden) if x.stride(-1) == 1 else None
            if x2 is None or x2.data_ptr() != x.data_ptr() or x2.stride(-1) != 1:
                raise B200AwqError("b200awq: program rmsnorm expects contiguous rows at one row pitch")
            x, ldx = x2, x2.stride(0)
        if not out.is_contiguous() or not weight.is_contiguous():
            raise B200AwqError("b200awq: program rmsnorm expects contiguous tensors")
        self._ops.append(("rmsnorm", dict(x=x, weight=weight, out=out, eps=float(eps), rows=x.numel() // hidden,
                                          hidden=hidden, ldx=ldx)))
        self._keep += [x, weight, out]

    def silu_and_mul(self, out, gate_up):
        self._no_more()
        self._dev_of(out)
        d = out.shape[-1]
        if gate_up.shape[-1] != 2 * d or not gate_up.is_contiguous() or not out.is_contiguous():
            raise B200AwqError("b200awq: silu_and_mul expects contiguous [.., 2d] -> [.., d]")
        self._ops.append(("silu", dict(out=out, gate_up=gate_up, rows=out.numel() // d, d=d)))
        self._keep += [out, gate_up]

    def layer_norm(self, x, weight, bias, out, eps):
        """ext.layer_norm recorded: out = LayerNorm(x) over the last dimension (bias may be None).  x, weight, bias and
        out are contiguous float16 tensors, captured by address."""
        self._no_more()
        self._dev_of(x)
        hidden = x.shape[-1]
        for t in (x, weight, bias, out):
            if t is None:
                continue
            if t.device != self._dev:
                raise B200AwqError("b200awq: a decode program lives on one device")
            if t.dtype != torch.float16 or not t.is_contiguous():
                raise B200AwqError("b200awq: layer_norm expects contiguous float16 tensors")
        if weight.shape != (hidden,) or (bias is not None and bias.shape != (hidden,)) or out.numel() != x.numel():
            raise B200AwqError(f"b200awq: layer_norm expects weight / bias [{hidden}] and out shaped like x")
        self._ops.append(("layer_norm", dict(x=x, weight=weight, bias=bias, out=out, eps=float(eps),
                                             rows=x.numel() // hidden, hidden=hidden)))
        self._keep += [t for t in (x, weight, bias, out) if t is not None]

    def gelu(self, out, x, approximate="none"):
        """ext.gelu recorded: out = F.gelu(x, approximate) ("tanh" or "none") on contiguous float16 tensors of one
        shape.  Fused when x is the whole output of the linear recorded just before it."""
        self._no_more()
        self._dev_of(x)
        if approximate not in ("none", "tanh"):
            raise B200AwqError(f"b200awq: gelu approximate must be 'none' or 'tanh', got {approximate!r}")
        if out.device != self._dev:
            raise B200AwqError("b200awq: a decode program lives on one device")
        if (x.dtype != torch.float16 or out.dtype != torch.float16 or x.shape != out.shape or not x.is_contiguous()
                or not out.is_contiguous()):
            raise B200AwqError("b200awq: gelu expects contiguous float16 tensors of one shape")
        n = x.shape[-1]
        self._ops.append(("gelu", dict(x=x, out=out, approximate=approximate, rows=x.numel() // n, n=n)))
        self._keep += [x, out]

    def gemm_forward_cuda(self, x, qweight, scales, qzeros, split_k_iters=8, bias=None):
        self._no_more()
        self._dev_of(x)
        ext._check_w(qweight, torch.int32, "qweight")
        ext._check_w(scales, torch.float16, "scales")
        ext._check_w(qzeros, torch.int32, "qzeros")
        K, N = qweight.shape[0], qweight.shape[1] * 8
        G = K // scales.shape[0]
        x2 = ext._x2d(x, K)
        if x2.data_ptr() != x.data_ptr():
            raise B200AwqError("b200awq: program inputs must be 16-byte aligned rows with unit stride (no copies "
                               "can be recorded)")
        M = x2.shape[0]
        y = torch.empty((M, N), dtype=torch.float16, device=x.device)
        self._ops.append(("linear", dict(x=x2, qweight=qweight, scales=scales, qzeros=qzeros, bias=bias, y=y, M=M, K=K,
                                         N=N, G=G, ldx=x2.stride(0) if M > 1 else K)))
        self._keep += [x, x2, qweight, scales, qzeros, y] + ([bias] if bias is not None else [])
        return y.reshape(x.shape[:-1] + (N,))

    def add(self, a, b, out=None):
        """out = a + b (fp16, torch's rounding).  `out` is allocated like gemm_forward_cuda's y when not given and
        returned.  Fused when one operand is the whole output of the linear / sparse_moe recorded just before and the
        other is a buffer nothing in the program writes, or the output of an op at most four kernel ops back (DESIGN.md
        3.5e states the rule for the rows such a residual is read from)."""
        out, M, K = self._add_operands(a, b, out, "add")
        self._ops.append(("add", dict(a=a, b=b, out=out, M=M, K=K)))
        self._keep += [a, b, out]
        return out

    def scaled_add(self, residual, y, multiplier, out=None):
        """out = residual + y * multiplier with torch's rounding on float16 tensors: fp16(r + fp16(y a)), the product in
        fp32 with a = float32(multiplier).  The depth-scaled residual add of MiniCPM / MiniCPM3 (a = scale_depth /
        sqrt(num_hidden_layers)) and Granite (a = residual_multiplier).  Tensors and `out` as add.  Fused as add is,
        with y (not residual) the whole output of the linear recorded just before; after a sparse_moe / qwen3_moe /
        deepseek_moe, or anywhere add would not fold, run() replays torch.mul then torch.add (DESIGN.md 3.5p)."""
        mul = float(multiplier)
        if not math.isfinite(ctypes.c_float(mul).value):        # (the op carries it as a float32)
            raise B200AwqError(f"b200awq: scaled_add needs a finite multiplier, got {multiplier!r}")
        out, M, K = self._add_operands(residual, y, out, "scaled_add")
        scaled = torch.empty_like(y)                  # y * multiplier, the per-op replay's first result
        self._ops.append(("scaled_add", dict(a=residual, b=y, out=out, M=M, K=K, mul=mul, scaled=scaled)))
        self._keep += [residual, y, out, scaled]
        return out

    def _add_operands(self, a, b, out, name):
        """add's / scaled_add's checks: contiguous float16 tensors of one shape on the program's device.  Returns out
        (allocated like gemm_forward_cuda's y when None), M and K."""
        self._no_more()
        self._dev_of(a)
        for t in (a, b) + ((out,) if out is not None else ()):
            if t.device != self._dev:
                raise B200AwqError("b200awq: a decode program lives on one device")
            if t.dtype != torch.float16 or not t.is_contiguous():
                raise B200AwqError(f"b200awq: {name} expects contiguous float16 tensors")
        if a.shape != b.shape or (out is not None and out.shape != a.shape):
            raise B200AwqError(f"b200awq: {name} expects equal shapes, got {tuple(a.shape)} and {tuple(b.shape)}")
        K = a.shape[-1]
        M = a.numel() // K
        if out is None:
            out = torch.empty((M, K), dtype=torch.float16, device=a.device).reshape(a.shape)
        return out, M, K

    def rope_kv_cache(self, qkv, freqs_cis, pos, k_cache, v_cache, n_heads, n_kv_heads, q_out=None, q_norm=None,
                      k_norm=None, head_dim=None, seq_len=None, rope_offset=None):
        """RoPE.forward(xq, xk, start_pos = *pos, seqlen = 1) + cache.update_kv(xv, xk) on the fused qkv output (q heads,
        then k heads, then v heads, as get_attention_shapes slices it): writes q_out [M, H, D] (allocated when not given,
        and returned) and row *pos of k_cache / v_cache batch entries 0..M-1, nothing when *pos is outside the cache or
        freqs_cis.  freqs_cis: the RoPE module's complex64 [S_f, D/2] table (any rope_theta / scaling it was built with
        applies as is).  q_norm / k_norm: Qwen3's two Qwen3RMSNorm modules (.weight fp16 [D], .variance_epsilon), both
        or neither; with them q and k heads are normalised per head before the rotation (ext.rope_kv_cache), and the
        fused kernel exchanges the heads' sums of squares across CTAs (DESIGN.md 3.5g).  head_dim: D when it is wider
        than the table's rotary dim R = 2 freqs_cis.shape[1] (partial rotary, StableLM: freqs_cis = RoPE(R, ..)'s
        table); columns [R, D) of each q / k head pass through unchanged, still inside the qkv linear's finish
        (DESIGN.md 3.5m).  ALiBi is not this op: the caller keeps that step.

        seq_len: T tokens per sequence (None or 1: one, as above): RoPE.forward(xq, xk, start_pos = *pos, seqlen = T)
        and update_kv of rows *pos .. *pos + T - 1.  qkv is the step's [B, T, N] (the reference's xqkv view) or [B T, N]
        output; row m = b T + t writes q_out row m and cache entry b at position *pos + t, and the caches need B
        entries.  A program built with max_tokens >= B T folds it into the qkv linear's finish as well (DESIGN.md
        3.5n); advance pos by T between runs.

        rope_offset: a device int32 tensor of B per-sequence rotary offsets (None: none): row m = b T + t keeps cache
        row *pos + t of entry b and is rotated at *pos + t + rope_offset[b] (ext.rope_kv_cache).  It folds wherever
        the op without offsets folds (DESIGN.md 3.5o) and is read at every run: rewrite it in place between runs, as
        pos."""
        self._no_more()
        self._dev_of(qkv)
        H = int(n_heads)
        if freqs_cis.dtype == torch.complex64:
            freqs_cis = torch.view_as_real(freqs_cis)
        if freqs_cis.dtype != torch.float32 or freqs_cis.dim() != 3:
            raise B200AwqError("b200awq: freqs_cis must be RoPE.freqs_cis (complex64 [S, D/2]) or its real view")
        D, _ = ext._rope_dims(freqs_cis, head_dim)
        M = qkv.numel() // qkv.shape[-1] if qkv.shape[-1] else 0
        if q_out is None:
            q_out = torch.empty((M, H, D), dtype=torch.float16, device=qkv.device)
        for t in (freqs_cis, pos, k_cache, v_cache, q_out):
            if t.device != self._dev:
                raise B200AwqError("b200awq: a decode program lives on one device")
        T = ext._seq_len(seq_len)
        desc, q2, M = ext.rope_descriptor(qkv, freqs_cis, pos, k_cache, v_cache, H, n_kv_heads, q_out, head_dim, T)
        if q2.data_ptr() != qkv.data_ptr():
            raise B200AwqError("b200awq: rope_kv_cache records qkv by address: pass its rows as they are")
        qdesc, norm_w = ext.qk_norm_descriptor(desc, q_norm, k_norm, self._dev)
        odesc = ext.rope_offset_descriptor(desc, qdesc, rope_offset, M // T, self._dev)
        self._ops.append(("rope", dict(qkv=q2, freqs=freqs_cis, pos=pos, k_cache=k_cache, v_cache=v_cache, q_out=q_out,
                                       H=H, KV=desc.n_kv_heads, M=M, N=q2.shape[1], T=T,
                                       ldx=q2.stride(0) if M > 1 else q2.shape[1], desc=desc, qdesc=qdesc,
                                       odesc=odesc)))
        self._keep += [qkv, q2, freqs_cis, pos, k_cache, v_cache, q_out] + norm_w
        if odesc is not None:
            self._keep.append(rope_offset)
        return q_out

    def mla_rope(self, qkva, freqs, pos, k_cache, n_heads, nope_dim, rope_dim, kv_lora_rank, style, q_out=None):
        """ext.mla_rope recorded on the fused q_proj | kv_a_proj_with_mqa output qkva [.., H (Dn + Dr) + C + Dr]:
        q_out [M, H, Dn + Dr] = [q_nope | rotated q_pe] (allocated when not given, and returned) and k_cache[m, *pos, h,
        Dn:] = the rotated k_pe for every head.  style 0 (DeepSeek-V2): freqs = the complex64 freqs_cis [S_f, Dr/2] of
        DeepseekV2RotaryEmbedding (or its f32 real view); style 1 (DeepSeek-V3 / Moonlight, rope_interleave): freqs = the
        f32 (cos, sin) pair [S_f, Dr] of DeepseekV3RotaryEmbedding.  The row keeps its values: record kv_a_layernorm as
        layernorm_forward_cuda on qkva[..., H (Dn + Dr): H (Dn + Dr) + C] next.
        The table is read by address when it already is the contiguous [S_f, Dr/2, 2] f32 layout (a contiguous
        freqs_cis, or its real view).  Otherwise - the (cos, sin) pair of style 1, or a non-contiguous freqs_cis such as
        the rotary module's own output - it is copied here, and the program keeps that snapshot: after the caller's
        table changes (a regrown rotary cache), record the program again.  k_cache needs a batch entry per token row,
        q_out M x H x (Dn + Dr) elements."""
        self._no_more()
        self._dev_of(qkva)
        H, Dn, Dr, C = int(n_heads), int(nope_dim), int(rope_dim), int(kv_lora_rank)
        row = ext._rows(qkva, H * (Dn + Dr) + C + Dr, "qkva")
        if row.data_ptr() != qkva.data_ptr():
            raise B200AwqError("b200awq: mla_rope records qkva by address: pass its rows as they are")
        M = row.shape[0]
        if q_out is None:
            q_out = torch.empty((M, H, Dn + Dr), dtype=torch.float16, device=qkva.device)
        f = ext._mla_freqs(freqs, Dr, int(style))
        for t in (f, pos, k_cache, q_out):
            if t.device != self._dev:
                raise B200AwqError("b200awq: a decode program lives on one device")
        desc = ext.mla_descriptor(pos, f, k_cache, None, q_out, M, H, Dn, Dr, 0, C, style)
        self._ops.append(("mla_rope", dict(row=row, M=M, N=row.shape[1], ldx=row.stride(0) if M > 1 else row.shape[1],
                                           desc=desc)))
        self._keep += [qkva, row, f, pos, k_cache, q_out]
        return q_out

    def mla_kv_cache(self, kv, pos, k_cache, v_cache, n_heads, nope_dim, v_dim):
        """ext.mla_kv_cache recorded on kv_b_proj's output kv [.., H (Dn + Dv)]: k_cache[m, *pos, h, :Dn] = k_nope,
        v_cache[m, *pos, h, :Dv] = v.  k_cache may be mla_rope's (the two write disjoint columns of its rows); both
        caches need a batch entry per token row."""
        self._no_more()
        self._dev_of(kv)
        H, Dn, Dv = int(n_heads), int(nope_dim), int(v_dim)
        row = ext._rows(kv, H * (Dn + Dv), "kv")
        if row.data_ptr() != kv.data_ptr():
            raise B200AwqError("b200awq: mla_kv_cache records kv by address: pass its rows as they are")
        for t in (pos, k_cache, v_cache):
            if t.device != self._dev:
                raise B200AwqError("b200awq: a decode program lives on one device")
        M = row.shape[0]
        desc = ext.mla_descriptor(pos, None, k_cache, v_cache, None, M, H, Dn, k_cache.shape[-1] - Dn, Dv, 0, 0)
        self._ops.append(("mla_kv", dict(row=row, M=M, N=row.shape[1], ldx=row.stride(0) if M > 1 else row.shape[1],
                                         desc=desc)))
        self._keep += [kv, row, pos, k_cache, v_cache]

    def mla_k_rope(self, qkva, freqs, pos, k_cache, n_heads, nope_dim, rope_dim, kv_lora_rank, q_lora_rank, style):
        """ext.mla_k_rope recorded on the fused q_a_proj | kv_a_proj_with_mqa output qkva [.., Cq + C + Dr]:
        k_cache[m, *pos, h, Dn:] = the rotated k_pe for every head.  freqs and style as mla_rope (the same table rules).
        The row keeps its values: record q_a_layernorm as layernorm_forward_cuda on qkva[..., :Cq] next, then q_b_proj
        and mla_q_rope, then kv_a_layernorm on qkva[..., Cq:Cq + C].  k_cache needs a batch entry per token row."""
        self._no_more()
        self._dev_of(qkva)
        H, Dn, Dr, C, Cq = int(n_heads), int(nope_dim), int(rope_dim), int(kv_lora_rank), int(q_lora_rank)
        row = ext._rows(qkva, Cq + C + Dr, "qkva")
        if row.data_ptr() != qkva.data_ptr():
            raise B200AwqError("b200awq: mla_k_rope records qkva by address: pass its rows as they are")
        M = row.shape[0]
        f = ext._mla_freqs(freqs, Dr, int(style))
        for t in (f, pos, k_cache):
            if t.device != self._dev:
                raise B200AwqError("b200awq: a decode program lives on one device")
        desc = ext.mla_descriptor(pos, f, k_cache, None, None, M, H, Dn, Dr, 0, C, style)
        self._ops.append(("mla_k_rope", dict(row=row, M=M, N=row.shape[1], pre=(Cq + C,),
                                             ldx=row.stride(0) if M > 1 else row.shape[1], desc=desc)))
        self._keep += [qkva, row, f, pos, k_cache]

    def mla_q_rope(self, q, freqs, pos, cache_len, n_heads, nope_dim, rope_dim, style, q_out=None):
        """ext.mla_q_rope recorded on q_b_proj's output q [.., H (Dn + Dr)]: q_out [M, H, Dn + Dr] = [q_nope | rotated
        q_pe] (allocated when not given, and returned).  cache_len: the caches' S, which bounds the position as it does
        for mla_k_rope.  freqs and style as mla_rope; q_out needs M x H x (Dn + Dr) elements."""
        self._no_more()
        self._dev_of(q)
        H, Dn, Dr = int(n_heads), int(nope_dim), int(rope_dim)
        row = ext._rows(q, H * (Dn + Dr), "q")
        if row.data_ptr() != q.data_ptr():
            raise B200AwqError("b200awq: mla_q_rope records q by address: pass its rows as they are")
        M = row.shape[0]
        if q_out is None:
            q_out = torch.empty((M, H, Dn + Dr), dtype=torch.float16, device=q.device)
        f = ext._mla_freqs(freqs, Dr, int(style))
        for t in (f, pos, q_out):
            if t.device != self._dev:
                raise B200AwqError("b200awq: a decode program lives on one device")
        desc = ext.mla_descriptor(pos, f, None, None, q_out, M, H, Dn, Dr, 0, 0, style, cache_len=cache_len)
        self._ops.append(("mla_q_rope", dict(row=row, M=M, N=row.shape[1], ldx=row.stride(0) if M > 1 else row.shape[1],
                                             desc=desc)))
        self._keep += [q, row, f, pos, q_out]
        return q_out

    @staticmethod
    def _stacked(w, name):
        if hasattr(w, "qweight"):
            return w.qweight, w.scales, w.qzeros
        if isinstance(w, (tuple, list)) and len(w) == 3:
            return tuple(w)
        raise B200AwqError(f"b200awq: {name} must have .qweight/.scales/.qzeros or be a 3-tuple")

    def sparse_moe(self, x, gate_weight, w1, w2, top_k, renormalize=True):
        """FusedSparseMoeBlock.forward (awq/modules/fused/moe.py:26-89) on the normed rows x [.., H]: router matmul,
        topk_softmax, optional renormalisation, moe_alig_block_size, grouped gate|up, SiLU*mul, grouped down x routing
        weight, sum over the slots.  gate_weight: the router's nn.Linear weight [E, H] fp16 (no bias); w1 / w2: the
        stacked GEMM-layout experts of awq/models/mixtral.py:129-151 ([E, H, 2I/8] / [E, I, H/8] qweight).  Returns
        out [M, H] fp16; the routing and the intermediate tensors are the program's (moe_buffers)."""
        return self._moe(x, gate_weight, w1, w2, top_k, renormalize, False)

    def qwen3_moe(self, x, gate_weight, w1, w2, top_k, norm_topk_prob=True):
        """Qwen3MoeSparseMoeBlock.forward (transformers 4.5x) on the normed rows x [.., H], arguments as sparse_moe
        (packing.stack_experts makes them from a block): logits = fp16(x Wg^T), p = softmax_fp32(logits), top_k (ties to
        the lower expert), w = p_k / sum p_k in fp32 when norm_topk_prob, w16 = fp16(w); then per selected expert in
        ascending id a = fp16(fp16(silu(g)) u), y = fp16(W2 a), c = fp16(y w16), out = fp16(out + c) from 0.  E <= 128
        and top_k <= 8 fuse at M = 1.  moe_buffers(i) holds topk_weights as fp16 w16 and down as the per-slot c."""
        return self._moe(x, gate_weight, w1, w2, top_k, norm_topk_prob, True)

    def deepseek_moe(self, x, gate_weight, w1, w2, top_k, shared, scoring, e_score_correction_bias=None, n_group=1,
                     topk_group=1, norm_topk_prob=False, routed_scaling_factor=1.0):
        """DeepseekV2Moe / DeepseekV3MoE.forward (transformers 5.5) over WQLinear_GEMM experts on the normed rows
        x [.., H]; gate_weight, w1, w2, top_k as qwen3_moe; shared = (ws1, ws2): the shared expert's [gate | up] and down
        as (qweight, scales, qzeros) GEMM-layout tensors (2-D, or stacked with E = 1), intermediate size I_s.
        l = fp32(x) fp32(Wg)^T.  scoring "softmax" (V2 greedy): p = softmax_fp32(l), top_k (ties to the lower expert),
        w = p_k * routed_scaling_factor.  scoring "sigmoid" (V3 noaux_tc): s = sigmoid(l), c = s + e_score_correction_bias
        (fp32 [E]); groups of E / n_group experts score their two largest c, the topk_group best stay and every other c
        becomes 0.0; top_k of the masked c; w = s_k, / (sum + 1e-20) when norm_topk_prob, * routed_scaling_factor.  Then
        per selected expert in ascending id a = fp16(fp16(silu(g)) u), y = fp16(W2 a), c = fp16(fp32(y) w),
        r = fp16(r + c) from 0; y_s = the shared MLP with the same rounding; out = fp16(r + y_s).  E <= 128, top_k <= 8
        and I_s a multiple of I fuse at M = 1.  moe_buffers(i) holds logits as fp32 [M, E], topk_weights as the fp32 w,
        gate_up / act with the shared expert's columns after the slots' ([M, top_k 2I + 2 I_s] / [M, top_k I + I_s]),
        down as the per-slot c and shared_out as y_s."""
        if scoring not in ("softmax", "sigmoid"):
            raise B200AwqError(f"b200awq: scoring must be 'softmax' or 'sigmoid', got {scoring!r}")
        ws1 = tuple(t.reshape(t.shape[-2:]) for t in self._stacked(shared[0], "shared gate|up"))
        ws2 = tuple(t.reshape(t.shape[-2:]) for t in self._stacked(shared[1], "shared down"))
        return self._moe(x, gate_weight, w1, w2, top_k, bool(norm_topk_prob), False,
                         ds=dict(ws1=ws1, ws2=ws2, scoring=scoring, bias=e_score_correction_bias, n_group=int(n_group),
                                 topk_group=int(topk_group), rsf=float(routed_scaling_factor)))

    def _moe(self, x, gate_weight, w1, w2, top_k, renormalize, hf, ds=None):
        self._no_more()
        self._dev_of(x)
        q1, s1, z1 = self._stacked(w1, "w1")
        q2, s2, z2 = self._stacked(w2, "w2")
        for t, dt, n in ((q1, torch.int32, "w1.qweight"), (s1, torch.float16, "w1.scales"), (z1, torch.int32, "w1.qzeros"),
                         (q2, torch.int32, "w2.qweight"), (s2, torch.float16, "w2.scales"), (z2, torch.int32, "w2.qzeros")):
            ext._require_cuda(t)
            if t.dim() != 3 or t.dtype != dt or not t.is_contiguous():
                raise B200AwqError(f"b200awq: {n} must be a contiguous stacked [E, ..] {dt} tensor")
        E, H, I = q1.shape[0], q1.shape[1], q1.shape[2] * 4
        G = H // s1.shape[1]
        top_k = int(top_k)
        if gate_weight.dtype != torch.float16 or tuple(gate_weight.shape) != (E, H) or not gate_weight.is_contiguous():
            raise B200AwqError(f"b200awq: gate_weight must be a contiguous [E={E}, H={H}] float16 tensor")
        if tuple(q2.shape) != (E, I, H // 8) or I // s2.shape[1] != G or not 1 <= top_k <= E:
            raise B200AwqError("b200awq: w1 / w2 / top_k do not describe one sparse-MoE block")
        if x.dtype != torch.float16 or x.shape[-1] != H or not x.is_contiguous():
            raise B200AwqError(f"b200awq: sparse_moe expects contiguous float16 rows [.., {H}]")
        M = x.numel() // H
        dev, f16, i32 = x.device, torch.float16, torch.int32
        I_s = 0
        if ds is not None:
            (sq1, ss1, sz1), (sq2, ss2, sz2) = ds["ws1"], ds["ws2"]
            I_s = sq1.shape[1] * 4
            for t, dt in ((sq1, torch.int32), (ss1, f16), (sz1, torch.int32), (sq2, torch.int32), (ss2, f16),
                          (sz2, torch.int32)):
                ext._require_cuda(t)
                if t.dtype != dt or not t.is_contiguous():
                    raise B200AwqError("b200awq: shared expert tensors must be contiguous GEMM-layout int32 / float16")
            if (tuple(sq1.shape) != (H, 2 * I_s // 8) or tuple(sq2.shape) != (I_s, H // 8) or H // ss1.shape[0] != G
                    or I_s // ss2.shape[0] != G):
                raise B200AwqError("b200awq: shared does not describe the block's shared expert")
            if not 1 <= ds["topk_group"] <= ds["n_group"] or E % ds["n_group"] != 0:
                raise B200AwqError("b200awq: need E % n_group == 0 and 1 <= topk_group <= n_group")
            if ds["scoring"] == "sigmoid":
                bias = ds["bias"]
                if bias is None or bias.dtype != torch.float32 or tuple(bias.shape) != (E,) or not bias.is_contiguous():
                    raise B200AwqError(f"b200awq: sigmoid scoring needs e_score_correction_bias, float32 [{E}]")
                ext._require_cuda(bias)
        block = 16                                      # moe_align_block_size's block at moe.py:54-56
        b = dict(logits=torch.empty((M, E), dtype=f16 if ds is None else torch.float32, device=dev),
                 topk_weights=torch.empty((M, top_k), dtype=f16 if hf else torch.float32, device=dev),
                 topk_ids=torch.empty((M, top_k), dtype=i32, device=dev),
                 token_expert_indices=torch.empty((M, top_k), dtype=i32, device=dev),
                 sorted_ids=torch.empty((M * top_k + E * (block - 1),), dtype=i32, device=dev),
                 expert_ids=torch.empty((M * top_k + E,), dtype=i32, device=dev),
                 num_tokens_post_pad=torch.empty((1,), dtype=i32, device=dev),
                 gate_up=torch.empty((M, top_k, 2 * I) if ds is None else (M, top_k * 2 * I + 2 * I_s), dtype=f16, device=dev),
                 act=torch.empty((M, top_k, I) if ds is None else (M, top_k * I + I_s), dtype=f16, device=dev),
                 down=torch.empty((M, top_k, H), dtype=f16, device=dev))
        if ds is not None:
            b["shared_out"] = torch.empty((M, H), dtype=f16, device=dev)
        out = torch.empty((M, H), dtype=f16, device=dev)
        raw_w = torch.empty((M, top_k), dtype=torch.float32, device=dev)    # topk_softmax's output (replay)
        d = _cabi.Moe()
        d.E, d.top_k, d.renormalize, d.group_size, d.H, d.I = E, top_k, 1 if renormalize else 0, G, H, I
        d.block_size, d.sorted_len = block, b["sorted_ids"].numel()
        d.gate_weight = gate_weight.data_ptr()
        d.w1_qweight, d.w1_scales, d.w1_qzeros = q1.data_ptr(), s1.data_ptr(), z1.data_ptr()
        d.w2_qweight, d.w2_scales, d.w2_qzeros = q2.data_ptr(), s2.data_ptr(), z2.data_ptr()
        for k, t in b.items():
            if k != "shared_out":
                setattr(d, k, t.data_ptr())
        if ds is not None:
            dd = _cabi.DeepseekMoe()
            dd.moe = d
            dd.scoring = 0 if ds["scoring"] == "softmax" else 1
            dd.n_group, dd.topk_group, dd.norm_topk_prob = ds["n_group"], ds["topk_group"], 1 if renormalize else 0
            dd.routed_scaling_factor, dd.I_s = ds["rsf"], I_s
            dd.bias = ds["bias"].data_ptr() if ds["scoring"] == "sigmoid" else None
            dd.ws1_qweight, dd.ws1_scales, dd.ws1_qzeros = (t.data_ptr() for t in ds["ws1"])
            dd.ws2_qweight, dd.ws2_scales, dd.ws2_qzeros = (t.data_ptr() for t in ds["ws2"])
            dd.shared_out = b["shared_out"].data_ptr()
            d = dd
            ds = dict(ds, I_s=I_s, G=G)
            self._keep += list(ds["ws1"]) + list(ds["ws2"]) + ([ds["bias"]] if ds["scoring"] == "sigmoid" else [])
        x2 = x.reshape(M, H)
        self._ops.append(("moe", dict(x=x2, gate_weight=gate_weight, w1=(q1, s1, z1), w2=(q2, s2, z2), top_k=top_k,
                                      renormalize=bool(renormalize), E=E, H=H, I=I, M=M, out=out, raw_w=raw_w,
                                      buffers=b, desc=d, hf=bool(hf), ds=ds)))
        self._keep += [x, x2, gate_weight, q1, s1, z1, q2, s2, z2, out, raw_w] + list(b.values())
        return out.reshape(x.shape)

    def moe_buffers(self, i: int = 0) -> dict:
        """The tensors the i-th recorded sparse_moe / qwen3_moe op (counted together, in recording order) owns (read-only views): logits [M, E] f16, topk_weights [M, top_k]
        f32 (after the renormalisation), topk_ids / token_expert_indices [M, top_k] i32, sorted_ids / expert_ids /
        num_tokens_post_pad (moe_alig_block_size), gate_up [M, top_k, 2I], act [M, top_k, I], down [M, top_k, H] (per-slot
        down outputs x routing weight) and out [M, H].  For a qwen3_moe op topk_weights is the fp16 w16 [M, top_k] and
        down holds the per-slot fp16(fp16(y) * w16).  A deepseek_moe op's are listed in deepseek_moe (with shared_out,
        y_s [M, H]).  A run overwrites them; the program reads none of them, so writing into them changes nothing but
        what the caller reads back."""
        o = [o for kind, o in self._ops if kind == "moe"][i]
        return dict(o["buffers"], out=o["out"])

    @staticmethod
    def _moe_replay(o) -> None:
        """apply_moe_weights' sequence (awq/modules/fused/moe.py:45-89) through ext, into the op's own buffers."""
        b, M, H = o["buffers"], o["M"], o["H"]
        torch.matmul(o["x"], o["gate_weight"].t(), out=b["logits"])
        ext.topk_softmax(o["raw_w"], b["topk_ids"], b["token_expert_indices"], b["logits"].float())
        if o["renormalize"]:
            torch.div(o["raw_w"], o["raw_w"].sum(dim=-1, keepdim=True), out=b["topk_weights"])
        else:
            b["topk_weights"].copy_(o["raw_w"])
        b["sorted_ids"].fill_(b["topk_ids"].numel())
        ext.moe_alig_block_size(b["topk_ids"], o["E"], 16, b["sorted_ids"], b["expert_ids"], b["num_tokens_post_pad"])
        gu = ext.grouped_gemm_forward(o["x"].view(M, 1, H), *o["w1"], b["topk_weights"], b["sorted_ids"], b["expert_ids"],
                                      b["num_tokens_post_pad"], False, 8)
        b["gate_up"].copy_(gu)
        ext.silu_and_mul(b["act"], b["gate_up"])
        dn = ext.grouped_gemm_forward(b["act"], *o["w2"], b["topk_weights"], b["sorted_ids"], b["expert_ids"],
                                      b["num_tokens_post_pad"], True, 8)
        b["down"].copy_(dn)
        torch.sum(b["down"], dim=1, out=o["out"])

    @staticmethod
    def _qwen3_moe_replay(o) -> None:
        """qwen3_moe's arithmetic through ext and torch, into the op's own buffers (no host synchronisation)."""
        b, M, H, I, k = o["buffers"], o["M"], o["H"], o["I"], o["top_k"]
        raw = o["raw_w"]
        torch.matmul(o["x"], o["gate_weight"].t(), out=b["logits"])
        ext.topk_softmax(raw, b["topk_ids"], b["token_expert_indices"], b["logits"].float())
        if o["renormalize"]:
            torch.div(raw, raw.sum(dim=-1, keepdim=True), out=raw)
        b["topk_weights"].copy_(raw)                    # .half()
        b["sorted_ids"].fill_(b["topk_ids"].numel())
        ext.moe_alig_block_size(b["topk_ids"], o["E"], 16, b["sorted_ids"], b["expert_ids"], b["num_tokens_post_pad"])
        gu = ext.grouped_gemm_forward(o["x"].view(M, 1, H), *o["w1"], raw, b["sorted_ids"], b["expert_ids"],
                                      b["num_tokens_post_pad"], False, 8)
        b["gate_up"].copy_(gu)
        torch.mul(torch.nn.functional.silu(b["gate_up"][..., :I]), b["gate_up"][..., I:], out=b["act"])
        dn = ext.grouped_gemm_forward(b["act"], *o["w2"], raw, b["sorted_ids"], b["expert_ids"],
                                      b["num_tokens_post_pad"], False, 8)
        torch.mul(dn, b["topk_weights"].unsqueeze(-1), out=b["down"])
        order = torch.sort(b["topk_ids"], dim=-1).indices          # index_add_ per expert, ascending
        slots = torch.gather(b["down"], 1, order.unsqueeze(-1).expand(M, k, H))
        o["out"].zero_()
        for j in range(k):
            o["out"].add_(slots[:, j])

    @staticmethod
    def _deepseek_moe_replay(o) -> None:
        """deepseek_moe's arithmetic through ext and torch, into the op's own buffers (no host synchronisation)."""
        b, M, H, I, k, E, ds = o["buffers"], o["M"], o["H"], o["I"], o["top_k"], o["E"], o["ds"]
        I_s, G = ds["I_s"], ds["G"]
        F = torch.nn.functional
        torch.matmul(o["x"].float(), o["gate_weight"].float().t(), out=b["logits"])
        if ds["scoring"] == "softmax":
            w, ids = torch.topk(b["logits"].softmax(dim=-1), k, dim=-1)
            w = w * ds["rsf"]
        else:
            s = b["logits"].sigmoid()
            c = s + ds["bias"]
            if ds["topk_group"] < ds["n_group"]:
                gs = c.view(M, ds["n_group"], -1).topk(2, dim=-1)[0].sum(dim=-1)
                gidx = torch.topk(gs, ds["topk_group"], dim=-1)[1]
                gmask = torch.zeros_like(gs).scatter_(1, gidx, 1).bool()
                c = c.masked_fill(~gmask.unsqueeze(-1).expand(M, ds["n_group"], E // ds["n_group"]).reshape(M, E), 0.0)
            ids = torch.topk(c, k, dim=-1)[1]
            w = s.gather(1, ids)
            if o["renormalize"]:
                w = w / (w.sum(dim=-1, keepdim=True) + 1e-20)
            w = w * ds["rsf"]
        b["topk_weights"].copy_(w)
        b["topk_ids"].copy_(ids)
        b["token_expert_indices"].copy_(torch.arange(k, device=ids.device, dtype=torch.int32) * M +
                                        torch.arange(M, device=ids.device, dtype=torch.int32).unsqueeze(1))
        b["sorted_ids"].fill_(b["topk_ids"].numel())
        ext.moe_alig_block_size(b["topk_ids"], E, 16, b["sorted_ids"], b["expert_ids"], b["num_tokens_post_pad"])
        tw = b["topk_weights"]
        gu = ext.grouped_gemm_forward(o["x"].view(M, 1, H), *o["w1"], tw, b["sorted_ids"], b["expert_ids"],
                                      b["num_tokens_post_pad"], False, 8)
        gus = ext.linear_forward("gemm", o["x"], *ds["ws1"], G)
        b["gate_up"][:, :k * 2 * I].copy_(gu.view(M, k * 2 * I))
        b["gate_up"][:, k * 2 * I:].copy_(gus)
        act = torch.mul(F.silu(gu[..., :I]), gu[..., I:])
        act_s = torch.mul(F.silu(gus[:, :I_s]), gus[:, I_s:])
        b["act"][:, :k * I].copy_(act.view(M, k * I))
        b["act"][:, k * I:].copy_(act_s)
        dn = ext.grouped_gemm_forward(act, *o["w2"], tw, b["sorted_ids"], b["expert_ids"], b["num_tokens_post_pad"],
                                      False, 8)
        b["down"].copy_(dn.float() * tw.unsqueeze(-1))                # .to(fp16)
        ext.linear_forward("gemm", act_s, *ds["ws2"], G, out=b["shared_out"])
        order = torch.sort(b["topk_ids"], dim=-1).indices             # index_add_ per expert, ascending
        slots = torch.gather(b["down"], 1, order.unsqueeze(-1).expand(M, k, H))
        o["out"].zero_()
        for j in range(k):
            o["out"].add_(slots[:, j])
        o["out"].add_(b["shared_out"])

    # ------------------------------------------------------------------ build / run
    def _c_ops(self):
        arr = (Op * len(self._ops))()
        for i, (kind, o) in enumerate(self._ops):
            c = arr[i]
            if kind == "rmsnorm":
                c.kind, c.M, c.K, c.eps, c.ldx = _cabi.OP_RMSNORM, o["rows"], o["hidden"], o["eps"], o["ldx"]
                c.x, c.weight, c.y = o["x"].data_ptr(), o["weight"].data_ptr(), o["out"].data_ptr()
            elif kind == "silu":
                c.kind, c.M, c.K = _cabi.OP_SILU_AND_MUL, o["rows"], o["d"]
                c.x, c.y = o["gate_up"].data_ptr(), o["out"].data_ptr()
            elif kind == "layer_norm":
                c.kind, c.M, c.K, c.eps = _cabi.OP_LAYER_NORM, o["rows"], o["hidden"], o["eps"]
                c.x, c.weight, c.y = o["x"].data_ptr(), o["weight"].data_ptr(), o["out"].data_ptr()
                c.bias = o["bias"].data_ptr() if o["bias"] is not None else None
            elif kind == "gelu":
                c.kind = _cabi.OP_GELU_TANH if o["approximate"] == "tanh" else _cabi.OP_GELU
                c.M, c.K, c.x, c.y = o["rows"], o["n"], o["x"].data_ptr(), o["out"].data_ptr()
            elif kind == "add":
                c.kind, c.M, c.K = _cabi.OP_ADD, o["M"], o["K"]
                c.x, c.weight, c.y = o["a"].data_ptr(), o["b"].data_ptr(), o["out"].data_ptr()
            elif kind == "scaled_add":                       # x: the residual, weight: the scaled operand
                c.kind, c.M, c.K, c.eps = _cabi.OP_SCALED_ADD, o["M"], o["K"], o["mul"]
                c.x, c.weight, c.y = o["a"].data_ptr(), o["b"].data_ptr(), o["out"].data_ptr()
            elif kind == "moe":
                c.kind, c.M, c.K, c.N = (_cabi.OP_DEEPSEEK_MOE if o["ds"] is not None else
                                         _cabi.OP_QWEN3_MOE if o["hf"] else _cabi.OP_SPARSE_MOE), o["M"], o["H"], o["H"]
                c.x, c.y, c.weight = o["x"].data_ptr(), o["out"].data_ptr(), ctypes.addressof(o["desc"])
            elif kind == "rope" and o["odesc"] is not None:   # kind 19, K = T
                c.kind, c.M, c.N, c.ldx, c.K = _cabi.OP_ROPE_KV_OFFSET, o["M"], o["N"], o["ldx"], o["T"]
                c.x, c.weight = o["qkv"].data_ptr(), ctypes.addressof(o["odesc"])
            elif kind == "rope":
                qk, seq = o["qdesc"] is not None, o["T"] > 1     # (seq: kinds 17 / 18, with K = T)
                c.kind = ((_cabi.OP_QK_NORM_ROPE_KV_SEQ if seq else _cabi.OP_QK_NORM_ROPE_KV) if qk else
                          (_cabi.OP_ROPE_KV_SEQ if seq else _cabi.OP_ROPE_KV))
                c.M, c.N, c.ldx, c.K = o["M"], o["N"], o["ldx"], o["T"] if seq else 0
                c.x, c.weight = o["qkv"].data_ptr(), ctypes.addressof(o["qdesc"] if qk else o["desc"])
            elif kind in _MLA_OPS:
                c.kind, c.M, c.N, c.ldx = _MLA_OPS[kind], o["M"], o["N"], o["ldx"]
                c.x, c.weight = o["row"].data_ptr(), ctypes.addressof(o["desc"])
            else:
                c.kind, c.M, c.K, c.N, c.group_size, c.ldx = _cabi.OP_LINEAR_GEMM, o["M"], o["K"], o["N"], o["G"], o["ldx"]
                c.x, c.qweight, c.scales, c.qzeros = (o["x"].data_ptr(), o["qweight"].data_ptr(), o["scales"].data_ptr(),
                                                      o["qzeros"].data_ptr())
                c.bias = o["bias"].data_ptr() if o["bias"] is not None else None
                c.y = o["y"].data_ptr()
        return arr

    def build(self) -> "DecodeProgram":
        """Fold the recorded calls into a fused program: one-time re-layout of the weights into the stream format and
        the output-stationary kernel (csrc/program_stream.cuh; csrc/program_batch.cuh for M > 1 rows per op,
        max_tokens >= M).  A sequence outside the kernel's envelope, or any sequence under knob 14 = 1, keeps the op
        list: `run()` then replays it per op."""
        self._no_more()
        if not self._ops:
            raise B200AwqError("b200awq: empty program")
        arr = self._c_ops()
        handle = ctypes.c_void_p()
        with ext._DeviceGuard(self._dev):
            if self.max_tokens > 1:
                code = lib.b200awq_program_create_batched(arr, len(self._ops), self.max_tokens, ctypes.byref(handle))
            else:
                code = lib.b200awq_program_create(arr, len(self._ops), ctypes.byref(handle))
        if code != _cabi.EUNSUPPORTED:
            check(code, "b200awq_program_create")
            self._handle = handle         # otherwise None: per-op replay (still the CUDA path)
        self._built = True
        return self

    @property
    def fused(self) -> bool:
        return self._handle is not None

    @property
    def kind(self) -> str:
        """"stream" (re-laid-out weights, output-stationary kernel) or "per-op"."""
        return "per-op" if self._handle is None else "stream"

    @property
    def tokens(self) -> int:
        """Token rows per run (M of the recorded ops, the rows of a norm, silu_and_mul, layer_norm or gelu; 0 before
        anything was recorded)."""
        if self._handle is not None:
            return lib.b200awq_program_tokens(self._handle)
        for kind, o in self._ops:
            return o["M"] if kind in ("linear", "moe", "add", "scaled_add", "rope") or kind in _MLA_OPS else o["rows"]
        return 0

    @property
    def kernel_ops(self) -> int:
        """Ops of the fused kernel: one per linear, two per sparse_moe / qwen3_moe / deepseek_moe (gate|up with the routing, down), none per add,
        scaled_add, rope_kv_cache, mla_rope, mla_kv_cache, mla_k_rope, mla_q_rope or gelu (they fold into their producer's epilogue)
        and none per layernorm_forward_cuda, silu_and_mul or layer_norm (they fold into their consumers' staging); 0
        per-op."""
        return lib.b200awq_program_num_ops(self._handle) if self._handle is not None else 0

    @property
    def launches_per_run(self) -> int:
        """Kernels launched by one run(): 1 when fused (adds and rope_kv_cache included); per op, one per recorded
        call, 6 per sparse_moe, 15 + top_k per qwen3_moe (17 + top_k with norm_topk_prob), 34 + top_k per softmax
        deepseek_moe (sigmoid: 36 + top_k, + 6 with expert groups, + 3 with norm_topk_prob), one torch.add launch per add,
        two (torch.mul, torch.add) per scaled_add and one b200awq_rope_kv (or b200awq_qk_norm_rope_kv) launch per rope_kv_cache, one b200awq_mla_rope / b200awq_mla_kv
        / b200awq_mla_k_rope / b200awq_mla_q_rope launch per mla_rope / mla_kv_cache / mla_k_rope / mla_q_rope, one
        b200awq_layer_norm / b200awq_gelu launch per layer_norm / gelu.  Per op these count the ext / torch calls of the replay: a torch call may launch more than one
        kernel (torch.sort, torch.gather), so the kernel count can be higher."""
        def per_op(kind, o):
            if kind == "scaled_add":
                return 2
            if kind != "moe":
                return 1
            ds = o["ds"]
            if ds is not None:
                if ds["scoring"] == "softmax":
                    return 34 + o["top_k"]
                return (36 + o["top_k"] + (6 if ds["topk_group"] < ds["n_group"] else 0) +
                        (3 if o["renormalize"] else 0))
            return 6 if not o["hf"] else 15 + o["top_k"] + (2 if o["renormalize"] else 0)
        return 1 if self.fused else sum(per_op(kind, o) for kind, o in self._ops)

    def run(self) -> None:
        if not self._built:
            raise B200AwqError("b200awq: build() the program first")
        dev = self._dev
        if self._handle is not None:
            with ext._DeviceGuard(dev):
                code = lib.b200awq_program_run(self._handle, None, 0, ext._stream(dev))
            check(code, "b200awq_program_run")
            return
        for kind, o in self._ops:
            if kind == "rmsnorm":
                ext.layernorm_forward_cuda(o["x"], o["weight"], o["out"], o["eps"])
            elif kind == "silu":
                ext.silu_and_mul(o["out"], o["gate_up"])
            elif kind == "layer_norm":
                ext.layer_norm(o["x"], o["weight"], o["bias"], o["out"], o["eps"])
            elif kind == "gelu":
                ext.gelu(o["out"], o["x"], o["approximate"])
            elif kind == "moe" and o["ds"] is not None:
                self._deepseek_moe_replay(o)
            elif kind == "moe" and o["hf"]:
                self._qwen3_moe_replay(o)
            elif kind == "moe":
                self._moe_replay(o)
            elif kind == "add":
                torch.add(o["a"], o["b"], out=o["out"])
            elif kind == "scaled_add":
                torch.mul(o["b"], o["mul"], out=o["scaled"])
                torch.add(o["a"], o["scaled"], out=o["out"])
            elif kind == "rope":
                with ext._DeviceGuard(dev):
                    code, name = ext.rope_kv_call(o["qkv"].data_ptr(), o["ldx"], o["desc"], o["qdesc"], o["M"], o["T"],
                                                  ext._stream(dev), o["odesc"])
                check(code, name)
            elif kind in _MLA_OPS:
                ext._mla_call(getattr(lib, "b200awq_" + kind), o["row"], o["desc"], o["M"], "b200awq_" + kind,
                              *o.get("pre", ()))
            else:
                ext.linear_forward("gemm", o["x"], o["qweight"], o["scales"], o["qzeros"], o["G"], o["bias"], out=o["y"])

    @staticmethod
    def abort_record():
        """(code, op, cta, aborted) of the last fused run on this device: the kernel's spin loops give up after 0.5 s
        instead of hanging the GPU and record which wait failed (csrc/program.cu).  Synchronises the device."""
        import numpy as np

        prev = lib.b200awq_get_knob(3)
        lib.b200awq_set_knob(3, 3)
        buf = np.zeros(4, dtype=np.int32)
        try:
            check(lib.b200awq_debug_read(buf.ctypes.data_as(ctypes.c_void_p), buf.nbytes), "b200awq_debug_read")
        finally:
            lib.b200awq_set_knob(3, prev)
        return tuple(int(v) for v in buf)

    def close(self) -> None:
        if self._handle is not None:
            lib.b200awq_program_destroy(self._handle)
            self._handle = None
            self._built = False

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
