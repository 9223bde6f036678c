"""Torch-facing operator layer: the functions the reference imports from `awq_ext` / `awq_v2_ext`
(call sites: awq/modules/linear/gemm.py:51-58, gemv.py:168-180, gemv_fast.py:192-205,
awq/modules/fused/norm.py:33-36, moe.py:76), implemented on the C ABI of libb200awq.so.

torch is plumbing only: device memory (caching allocator), the current stream, dtype/shape checks.
Every function launches on torch's current stream, never synchronises and is CUDA-graph capturable
once the per-(device, stream) workspace exists (first call on that stream allocates it).
"""
from __future__ import annotations

import torch

from . import _cabi
from ._cabi import B200AwqError, check, lib

__all__ = [
    "gemm_forward_cuda", "dequantize_weights_cuda", "gemv_forward_cuda", "gemmv2_forward_cuda",
    "gemv_forward_cuda_decode", "gemm_forward_cuda_prefill", "layernorm_forward_cuda", "silu_and_mul",
    "layer_norm", "gelu",
    "topk_softmax", "moe_alig_block_size", "grouped_gemm_forward",
    "linear_forward", "stream_pack", "stream_pack_rotary", "rope_kv_cache", "rope_descriptor", "qk_norm_descriptor",
    "rope_offset_descriptor",
    "mla_descriptor", "mla_rope", "mla_kv_cache", "mla_k_rope", "mla_q_rope",
    "set_knob", "get_knob",
    "B200AwqError",
]

_WS: dict = {}
_WS_MIN = 16 << 20
_WS_TICKETS = 16384          # kTicketBytes (csrc/kernels.h); tests/test_host_cpu.py checks it against the ABI


def _require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise B200AwqError("b200awq: tensors must live on a CUDA device (there is no CPU path)")


def _workspace(dev: torch.device, stream_ptr: int, need: int) -> torch.Tensor:
    key = (dev.index, stream_ptr)
    ws = _WS.get(key)
    if ws is None or ws.numel() < need:
        ws = torch.zeros(max(need, _WS_MIN), dtype=torch.uint8, device=dev)
        _WS[key] = ws
    return ws


def _stream(dev: torch.device) -> int:
    return torch.cuda.current_stream(dev).cuda_stream


class _DeviceGuard:
    """Launch on the tensor's device even when it is not the current one (accelerate places layers
    on several GPUs; the reference's Triton path does the same guard, awq/modules/triton/gemm.py:23-27)."""

    __slots__ = ("dev", "prev")

    def __init__(self, dev: torch.device):
        self.dev, self.prev = dev.index, None

    def __enter__(self):
        cur = torch.cuda.current_device()
        if cur != self.dev:
            self.prev = cur
            torch.cuda.set_device(self.dev)

    def __exit__(self, *exc):
        if self.prev is not None:
            torch.cuda.set_device(self.prev)


def _x2d(x: torch.Tensor, K: int) -> torch.Tensor:
    if x.dtype != torch.float16:
        raise B200AwqError(f"b200awq: activations must be float16, got {x.dtype}")
    if x.shape[-1] != K:
        raise B200AwqError(f"b200awq: activation feature dim {x.shape[-1]} != in_features {K}")
    x2 = x.reshape(-1, K)
    if x2.stride(-1) != 1 or (x2.shape[0] > 1 and (x2.stride(0) < K or x2.stride(0) % 8 != 0)) \
            or x2.data_ptr() % 16 != 0:
        x2 = x2.contiguous()  # TMA needs 16-byte aligned rows
    return x2


def _check_w(t: torch.Tensor, dtype, name: str):
    if t.dtype != dtype or not t.is_contiguous():
        raise B200AwqError(f"b200awq: {name} must be contiguous {dtype}, got {t.dtype} contiguous={t.is_contiguous()}")


_LAYOUT = {
    "gemm": (lib.b200awq_gemm_forward, torch.int32),
    "gemv": (lib.b200awq_gemv_forward, torch.int32),
    "fast": (lib.b200awq_fast_forward, torch.int16),
}
# validated weight triples: id(qweight) -> (weakref to qweight, data_ptrs, K, N, device).  A decode loop calls the
# same 160 linears every token: dtype / contiguity / device checks and the pointer reads are done once per tensor
# (the weakref guards against id() reuse after the tensor died; in-place updates keep the pointers valid).
_WCACHE: dict = {}
_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)
_cur_device = getattr(torch._C, "_cuda_getDevice", None)


def _weights(layout: str, qweight, scales, qzeros):
    import weakref

    key = (id(qweight), id(scales), id(qzeros))
    hit = _WCACHE.get(key)
    if hit is not None:
        refs = hit[7]
        # ids are only unique among LIVE objects: every one of the three must still be the tensor that was validated
        if refs[0]() is qweight and refs[1]() is scales and refs[2]() is qzeros and hit[1] == qweight.data_ptr():
            return hit
    _require_cuda(qweight, scales, qzeros)
    wdt = _LAYOUT[layout][1]
    if layout == "gemm":
        K, N = qweight.shape[0], qweight.shape[1] * 8
    elif layout == "gemv":
        N, K = qweight.shape[0], qweight.shape[1] * 8
    else:
        N, K = qweight.shape[0] * 4, qweight.shape[1]
    _check_w(qweight, wdt, "qweight")
    _check_w(scales, torch.float16, "scales")
    _check_w(qzeros, torch.float16 if layout == "fast" else torch.int32, "qzeros")
    if scales.device != qweight.device or qzeros.device != qweight.device:
        raise B200AwqError("b200awq: qweight / scales / qzeros must live on one device")
    refs = (weakref.ref(qweight), weakref.ref(scales), weakref.ref(qzeros))
    ent = (refs[0], qweight.data_ptr(), scales.data_ptr(), qzeros.data_ptr(), K, N, qweight.device, refs)
    if len(_WCACHE) > 16384:
        _WCACHE.clear()
    _WCACHE[key] = ent
    return ent


def linear_forward(layout: str, x, qweight, scales, qzeros, group_size: int, bias=None, out=None) -> torch.Tensor:
    """Y = X . deq(W) (+ bias) for layout in {"gemm", "gemv", "fast"}; returns [M, N] fp16 (written into `out`
    when given: a contiguous [M, N] fp16 tensor).  The hot call of an eager decode loop (160 per token): weights are
    validated once per tensor, no context-manager object, no extra ABI call (b200awq_workspace_bytes is
    16384 + min(M, 128) * N * 8, restated here)."""
    try:
        fn = _LAYOUT[layout][0]
    except KeyError:
        raise ValueError(layout) from None
    _, p_qw, p_sc, p_qz, K, N, dev, _refs = _weights(layout, qweight, scales, qzeros)
    if not x.is_cuda or (bias is not None and not bias.is_cuda):
        raise B200AwqError("b200awq: tensors must live on a CUDA device (there is no CPU path)")
    x2 = _x2d(x, K)
    M = x2.shape[0]
    if x2.device != dev:
        raise B200AwqError(f"b200awq: activations on {x2.device}, weights on {dev}")
    if out is None:
        y = torch.empty((M, N), dtype=torch.float16, device=dev)
    else:
        y = out
        if y.dtype != torch.float16 or not y.is_contiguous() or y.numel() != M * N or y.device != dev:
            raise B200AwqError("b200awq: `out` must be a contiguous float16 [M, N] tensor on the input's device")
    if M == 0:
        return y
    G = K if group_size in (-1, 0) else int(group_size)
    di = dev.index
    cur = _cur_device() if _cur_device is not None else torch.cuda.current_device()
    if cur != di:
        torch.cuda.set_device(di)
    try:
        st = _raw_stream(di) if _raw_stream is not None else torch.cuda.current_stream(dev).cuda_stream
        need = _WS_TICKETS + (M if M < 128 else 128) * N * 8
        ws = _WS.get((di, st))
        if ws is None or ws.numel() < need:
            ws = _workspace(dev, st, need)
        code = fn(x2.data_ptr(), x2.stride(0) if M > 1 else K, p_qw, p_sc, p_qz,
                  bias.data_ptr() if bias is not None else None, y.data_ptr(), M, K, N, G,
                  ws.data_ptr(), ws.numel(), st)
    finally:
        if cur != di:
            torch.cuda.set_device(cur)
    if code != 0:
        check(code, f"b200awq_{layout}_forward(M={M}, K={K}, N={N}, G={G})")
    return y


# ----------------------------------------------------------------------------- awq_ext surface
def gemm_forward_cuda(x, qweight, scales, qzeros, split_k_iters=8):
    """awq_ext.gemm_forward_cuda (gemm.py:56-58): x [M, K] f16, GEMM layout -> [M, N] f16.
    `split_k_iters` is a legacy hint of the reference kernels; accepted and ignored."""
    K = qweight.shape[0]
    G = K // scales.shape[0]
    out = linear_forward("gemm", x, qweight, scales, qzeros, G)
    return out.reshape(x.shape[:-1] + (out.shape[-1],))


def dequantize_weights_cuda(qweight, scales, qzeros, split_k_iters=0, thx=0, thy=0, dbg=False):
    """awq_ext.dequantize_weights_cuda (gemm.py:51-53, tests/test_dequantization.py:41-49) -> [K, N] f16."""
    _require_cuda(qweight, scales, qzeros)
    _check_w(qweight, torch.int32, "qweight")
    _check_w(scales, torch.float16, "scales")
    _check_w(qzeros, torch.int32, "qzeros")
    K, N = qweight.shape[0], qweight.shape[1] * 8
    G = K // scales.shape[0]
    dev = qweight.device
    out = torch.empty((K, N), dtype=torch.float16, device=dev)
    with _DeviceGuard(dev):
        code = lib.b200awq_dequantize_gemm(qweight.data_ptr(), scales.data_ptr(), qzeros.data_ptr(), out.data_ptr(),
                                           K, N, G, _stream(dev))
    check(code, f"b200awq_dequantize_gemm(K={K}, N={N}, G={G})")
    return out


def gemv_forward_cuda(x, qweight, scales, qzeros, group_size):
    """awq_ext.gemv_forward_cuda (gemv.py:177-180): GEMV layout, M <= 8."""
    out = linear_forward("gemv", x, qweight, scales, qzeros, group_size)
    return out.reshape(x.shape[:-1] + (out.shape[-1],))


def gemmv2_forward_cuda(x, qweight, scales, qzeros, group_size, split_k_iters=8):
    """awq_ext.gemmv2_forward_cuda (gemv.py:168-176): GEMV layout, M > 8."""
    out = linear_forward("gemv", x, qweight, scales, qzeros, group_size)
    return out.reshape(x.shape[:-1] + (out.shape[-1],))


def layernorm_forward_cuda(x, weight, out, eps):
    """awq_ext.layernorm_forward_cuda (fused/norm.py:33-36): RMSNorm written into `out`."""
    _require_cuda(x, weight, out)
    if x.dtype != torch.float16 or weight.dtype != torch.float16 or out.dtype != torch.float16:
        raise B200AwqError("b200awq: rmsnorm expects float16 tensors")
    hidden = x.shape[-1]
    xc = x if x.is_contiguous() else x.contiguous()
    if not out.is_contiguous():
        raise B200AwqError("b200awq: rmsnorm output must be contiguous")
    rows = xc.numel() // hidden
    with _DeviceGuard(x.device):
        code = lib.b200awq_rmsnorm(xc.data_ptr(), weight.data_ptr(), out.data_ptr(), rows, hidden, float(eps),
                                   _stream(x.device))
    check(code, "b200awq_rmsnorm")


def silu_and_mul(out, gate_up):
    """awq_ext.silu_and_mul (fused/moe.py:76): out[.., d] = silu(gate_up[.., :d]) * gate_up[.., d:]."""
    _require_cuda(out, gate_up)
    d = out.shape[-1]
    if gate_up.shape[-1] != 2 * d or not gate_up.is_contiguous() or not out.is_contiguous():
        raise B200AwqError("b200awq: silu_and_mul expects contiguous [.., 2d] -> [.., d]")
    rows = out.numel() // d
    with _DeviceGuard(out.device):
        code = lib.b200awq_silu_and_mul(gate_up.data_ptr(), out.data_ptr(), rows, d, _stream(out.device))
    check(code, "b200awq_silu_and_mul")


def layer_norm(x, weight, bias, out, eps):
    """nn.LayerNorm / F.layer_norm over the last dimension of fp16 x, written into `out` (transformers' CohereLayerNorm
    with bias=None), in the fixed summation order of include/b200awq.h (b200awq_layer_norm): mean, then the centred
    variance in a second pass, fp32 math, rounded once.  hidden % 8 == 0 and 16-byte aligned tensors."""
    _require_cuda(x, weight, bias, out)
    for t, n in ((x, "x"), (weight, "weight"), (bias, "bias"), (out, "out")):
        if t is not None and t.dtype != torch.float16:
            raise B200AwqError(f"b200awq: layer_norm expects float16 tensors ({n} is {t.dtype})")
    hidden = x.shape[-1]
    if weight.shape != (hidden,) or (bias is not None and bias.shape != (hidden,)):
        raise B200AwqError(f"b200awq: layer_norm weight / bias must be [{hidden}]")
    if not weight.is_contiguous() or (bias is not None and not bias.is_contiguous()):
        raise B200AwqError("b200awq: layer_norm weight / bias must be contiguous")
    xc = x if x.is_contiguous() else x.contiguous()
    rows = xc.numel() // hidden if hidden else 0
    if not out.is_contiguous() or out.numel() != rows * hidden:
        raise B200AwqError("b200awq: layer_norm output must be contiguous with x's shape")
    with _DeviceGuard(x.device):
        code = lib.b200awq_layer_norm(xc.data_ptr(), hidden, weight.data_ptr(),
                                      bias.data_ptr() if bias is not None else None, out.data_ptr(), rows, hidden,
                                      float(eps), _stream(x.device))
    check(code, "b200awq_layer_norm")


_GELU_APPROX = {"none": 0, "tanh": 1}


def gelu(out, x, approximate="none"):
    """out = F.gelu(x, approximate=approximate) on fp16 tensors ("tanh": gelu_pytorch_tanh / GELUTanh, StarCoder2;
    "none": the exact erf form, MPT and Falcon), in torch's CUDA formulas with fp32 math, rounded once."""
    _require_cuda(out, x)
    if approximate not in _GELU_APPROX:
        raise B200AwqError(f"b200awq: gelu approximate must be 'none' or 'tanh', got {approximate!r}")
    if x.dtype != torch.float16 or out.dtype != torch.float16:
        raise B200AwqError("b200awq: gelu expects float16 tensors")
    if x.shape != out.shape or not x.is_contiguous() or not out.is_contiguous():
        raise B200AwqError("b200awq: gelu expects contiguous tensors of one shape")
    n = x.shape[-1] if x.dim() else 1
    rows = x.numel() // n if n else 0
    if rows == 0:
        return
    with _DeviceGuard(out.device):
        code = lib.b200awq_gelu(x.data_ptr(), out.data_ptr(), rows, n, _GELU_APPROX[approximate], _stream(out.device))
    check(code, "b200awq_gelu")


def _rope_dims(freqs, head_dim):
    """(D, R) of a rotary table [S_f, R/2] (complex64) or [S_f, R/2, 2] (f32) and the head_dim argument (None: D = R)."""
    R = 2 * (freqs.shape[1] if freqs.dtype == torch.complex64 else freqs.shape[-2])
    D = R if head_dim is None else int(head_dim)
    if D < R or D % 2:
        raise B200AwqError(f"b200awq: head_dim {D} must be even and at least the table's rotary dim {R}")
    return D, R


def _seq_len(seq_len):
    """T of a rope_kv_cache call: None means 1 (one token per sequence)."""
    T = 1 if seq_len is None else int(seq_len)
    if T < 1:
        raise B200AwqError(f"b200awq: seq_len must be at least 1, got {T}")
    return T


def rope_descriptor(qkv, freqs, pos, k_cache, v_cache, n_heads, n_kv_heads, q_out, head_dim=None, seq_len=None):
    """Checks the tensors of one RoPE + KV-cache append and returns (b200awq_rope_t, qkv as [M, N], M).

    qkv [.., (H + 2 KV) D] f16 (rows at a unit stride, any row pitch); freqs: the fp32 [S_f, R/2, 2] real view of
    RoPE(R, ..).freqs_cis (awq/modules/fused/attn.py:29-43) or the complex64 [S_f, R/2] table itself; pos: a device
    int32 tensor of one element; k_cache / v_cache: WindowedCache's contiguous-row f16 [B >= M, S, KV, D]
    (cache.py:5-31); q_out: contiguous f16 with M H D elements.  n_kv_heads = 0 means n_heads, as WindowedCache sizes
    it.  head_dim: D (None: R, full rotary); when larger than R, only the first R columns of each q / k head are
    rotated (partial rotary, StableLM) and the rest pass through.  seq_len: T tokens per sequence (None: 1); M must be
    a multiple of T and the caches need B >= M / T entries."""
    _require_cuda(qkv, freqs, pos, k_cache, v_cache, q_out)
    T = _seq_len(seq_len)
    H = int(n_heads)
    KV = int(n_kv_heads) or H
    if freqs.dtype == torch.complex64:
        freqs = torch.view_as_real(freqs)
    if freqs.dtype != torch.float32 or freqs.dim() != 3 or freqs.shape[-1] != 2 or not freqs.is_contiguous():
        raise B200AwqError("b200awq: freqs must be RoPE.freqs_cis (complex64 [S, R/2]) or its contiguous real view")
    D, R = _rope_dims(freqs, head_dim)
    N = (H + 2 * KV) * D
    if qkv.dtype != torch.float16 or qkv.shape[-1] != N:
        raise B200AwqError(f"b200awq: qkv must be float16 [.., (n_heads + 2 n_kv_heads) head_dim = {N}]")
    q2 = qkv.reshape(-1, N)
    if q2.stride(-1) != 1:
        raise B200AwqError("b200awq: qkv rows must have a unit stride")
    M = q2.shape[0]
    if M % T:
        raise B200AwqError(f"b200awq: {M} qkv rows are not a whole number of sequences of seq_len {T}")
    for name, c in (("k_cache", k_cache), ("v_cache", v_cache)):
        if c.dtype != torch.float16 or c.dim() != 4 or tuple(c.shape[2:]) != (KV, D) or c.shape[0] < M // T:
            raise B200AwqError(f"b200awq: {name} must be float16 [B >= {M // T}, S, {KV}, {D}]")
        if c.stride(3) != 1 or c.stride(2) != D or c.stride(1) != KV * D:
            raise B200AwqError(f"b200awq: {name} must have contiguous [S, KV, D] entries")
    if k_cache.shape[1] != v_cache.shape[1] or k_cache.stride(0) != v_cache.stride(0):
        raise B200AwqError("b200awq: k_cache and v_cache must have the same shape and strides")
    if pos.dtype != torch.int32 or pos.numel() != 1:
        raise B200AwqError("b200awq: pos must be a device int32 tensor with one element")
    if q_out.dtype != torch.float16 or not q_out.is_contiguous() or q_out.numel() != M * H * D:
        raise B200AwqError(f"b200awq: q_out must be a contiguous float16 tensor of {M} x {H} x {D} elements")
    r = _cabi.Rope()
    r.n_heads, r.n_kv_heads, r.head_dim, r.rotary_dim = H, KV, D, R if R < D else 0
    r.cache_len, r.freqs_len = k_cache.shape[1], freqs.shape[0]
    r.cache_batch_stride = k_cache.stride(0)
    r.pos, r.freqs, r.q_out = pos.data_ptr(), freqs.data_ptr(), q_out.data_ptr()
    r.k_cache, r.v_cache = k_cache.data_ptr(), v_cache.data_ptr()
    return r, q2, M


def qk_norm_descriptor(rope, q_norm, k_norm, device):
    """b200awq_qk_norm_rope_t around a b200awq_rope_t from Qwen3's two Qwen3RMSNorm modules (or None when both are None).
    Each module needs .weight (float16 [D] on `device`) and .variance_epsilon; the two epsilons must be equal.  Returns
    (descriptor or None, the tensors it names)."""
    if q_norm is None and k_norm is None:
        return None, []
    if q_norm is None or k_norm is None:
        raise B200AwqError("b200awq: give both q_norm and k_norm, or neither")
    D = rope.head_dim
    if rope.rotary_dim not in (0, D):
        raise B200AwqError("b200awq: q_norm / k_norm need full rotary (head_dim = 2 freqs.shape[1])")
    ws = []
    for name, n in (("q_norm", q_norm), ("k_norm", k_norm)):
        w = getattr(n, "weight", None)
        if not isinstance(w, torch.Tensor) or not hasattr(n, "variance_epsilon"):
            raise B200AwqError(f"b200awq: {name} must be a Qwen3RMSNorm (.weight, .variance_epsilon)")
        w = w.detach()
        if w.dtype != torch.float16 or tuple(w.shape) != (D,) or not w.is_contiguous() or w.device != device:
            raise B200AwqError(f"b200awq: {name}.weight must be a contiguous float16 [{D}] tensor on {device}")
        ws.append(w)
    eps = float(q_norm.variance_epsilon)
    if float(k_norm.variance_epsilon) != eps:
        raise B200AwqError("b200awq: q_norm and k_norm must have the same variance_epsilon")
    d = _cabi.QkNormRope()
    d.rope = rope
    d.q_norm_weight, d.k_norm_weight, d.eps = ws[0].data_ptr(), ws[1].data_ptr(), eps
    return d, ws


def rope_offset_descriptor(desc, qdesc, rope_offset, B, device):
    """b200awq_rope_offset_t around a b200awq_rope_t (and the b200awq_qk_norm_rope_t of q / k norm, or None) with the
    per-sequence rotary offsets rope_offset: a contiguous int32 tensor of B elements on `device` (None: returns None,
    the op without offsets)."""
    if rope_offset is None:
        return None
    if (not isinstance(rope_offset, torch.Tensor) or rope_offset.dtype != torch.int32 or rope_offset.numel() != B
            or not rope_offset.is_contiguous() or rope_offset.device != device):
        raise B200AwqError(f"b200awq: rope_offset must be a contiguous int32 tensor of B = {B} elements on {device}")
    d = _cabi.RopeOffset()
    if qdesc is not None:
        d.qk = qdesc
    else:
        d.qk.rope = desc
    d.rot_offset = rope_offset.data_ptr()
    return d


def rope_kv_cache(qkv, freqs_cis, pos, k_cache, v_cache, n_heads, n_kv_heads, q_out=None, q_norm=None, k_norm=None,
                  head_dim=None, seq_len=None, rope_offset=None):
    """RoPE.forward on q and k of the fused qkv output and WindowedCache.update_kv of k and v at position *pos
    (awq/modules/fused/attn.py:243-267): writes q_out [M, H, D] and the row `pos` of cache batch entries 0..M-1, nothing
    else (nothing at all when pos is outside the cache or the frequency table).  pos is read on the device: a captured
    CUDA graph replays at the position stored there.  Returns q_out (allocated when not given).

    q_norm / k_norm: Qwen3's two Qwen3RMSNorm modules (attn.py:250-253), both or neither.  With them every q head and
    every k head is normalised per token before the rotation (b200awq_qk_norm_rope_kv; the head's sum of squares in the
    fixed order of include/b200awq.h); v heads are not.  They need full rotary.

    head_dim: D when the heads are wider than the table's rotary dim R = 2 freqs_cis.shape[1] (StableLM's
    partial_rotary_factor, freqs_cis = RoPE(R, ..).freqs_cis): columns [0, R) of each q / k head are rotated, columns
    [R, D) are copied unchanged into q_out and k_cache.  None: D = R.

    seq_len: T tokens per sequence at consecutive positions (RoPE.forward(xq, xk, start_pos = *pos, seqlen = T) and
    update_kv of rows *pos .. *pos + T - 1; None or 1: one token, as above).  qkv is then the reference's xqkv view
    [B, T, N] or its rows [B T, N]; row m = b T + t is token t of sequence b at position *pos + t and writes q_out row m
    and cache entry b (the caches need B entries).  A row whose position is outside the cache or the table writes
    nothing; the rest of the step still does (b200awq_rope_kv_seq).

    rope_offset: a device int32 tensor of B = M / T per-sequence rotary offsets (None: none).  Row m = b T + t keeps
    cache row *pos + t of entry b and is rotated at *pos + t + rope_offset[b] (b200awq_rope_kv_offset): -pad_b for a
    left-padded batch, rope_deltas[b] for a Qwen2-VL / Qwen2.5-VL text step.  A row writes nothing unless both its
    cache row and its rotary position are in range.  The offsets are read on the device, as pos is."""
    H = int(n_heads)
    T = _seq_len(seq_len)
    D, _ = _rope_dims(freqs_cis, head_dim)
    if q_out is None:
        M = qkv.numel() // qkv.shape[-1] if qkv.shape[-1] else 0
        q_out = torch.empty((M, H, D), dtype=torch.float16, device=qkv.device)
    r, q2, M = rope_descriptor(qkv, freqs_cis, pos, k_cache, v_cache, H, n_kv_heads, q_out, head_dim, T)
    qd, _ = qk_norm_descriptor(r, q_norm, k_norm, qkv.device)
    od = rope_offset_descriptor(r, qd, rope_offset, M // T, qkv.device)
    ld = q2.stride(0) if M > 1 else q2.shape[1]
    with _DeviceGuard(qkv.device):
        code, name = rope_kv_call(q2.data_ptr(), ld, r, qd, M, T, _stream(qkv.device), od)
    check(code, f"{name}(M={M}, T={T}, H={H}, KV={r.n_kv_heads}, D={D})")
    return q_out


def rope_kv_call(qkv_ptr, ld, desc, qdesc, M, T, stream, odesc=None):
    """The C entry of one RoPE + KV-cache append: b200awq_rope_kv (qdesc None) or b200awq_qk_norm_rope_kv, their
    _seq forms for T > 1, and b200awq_rope_kv_offset for any of them with rotary offsets (odesc, which embeds desc /
    qdesc).  Returns (code, entry name)."""
    if odesc is not None:
        return lib.b200awq_rope_kv_offset(qkv_ptr, ld, odesc, M, T, stream), "b200awq_rope_kv_offset"
    name = ("b200awq_rope_kv" if qdesc is None else "b200awq_qk_norm_rope_kv") + ("_seq" if T > 1 else "")
    args = (qkv_ptr, ld, desc if qdesc is None else qdesc, M) + ((T,) if T > 1 else ())
    return getattr(lib, name)(*args, stream), name


def _rows(x, N, name):
    if x.dtype != torch.float16 or x.shape[-1] != N:
        raise B200AwqError(f"b200awq: {name} must be float16 [.., {N}]")
    x2 = x.reshape(-1, N)
    if x2.stride(-1) != 1:
        raise B200AwqError(f"b200awq: {name} rows must have a unit stride")
    return x2


def _mla_freqs(freqs, rope_dim, style):
    """The [S_f, Dr/2, 2] f32 (cos, sin) table of b200awq_mla_t.  style 0: DeepseekV2RotaryEmbedding's complex64
    freqs_cis [S_f, Dr/2] or its f32 real view.  style 1: a (cos, sin) pair of f32 [S_f, Dr] tensors as
    DeepseekV3RotaryEmbedding returns them (attention_scaling applied, before the cast to the activations' dtype); their
    halves repeat, so the first Dr/2 columns are taken (a new tensor)."""
    if style == 0:
        if isinstance(freqs, torch.Tensor) and freqs.dtype == torch.complex64:
            freqs = torch.view_as_real(freqs)
        if (not isinstance(freqs, torch.Tensor) or freqs.dtype != torch.float32 or freqs.dim() != 3
                or tuple(freqs.shape[1:]) != (rope_dim // 2, 2)):
            raise B200AwqError(f"b200awq: style 0 freqs must be freqs_cis (complex64 [S, {rope_dim // 2}]) or its "
                               "real view")
        return freqs.contiguous()          # (the rotary module's table is a transposed product: a copy then)
    if isinstance(freqs, torch.Tensor) and freqs.dtype == torch.float32 and freqs.dim() == 3:
        t = freqs                                   # already the descriptor's table
    else:
        cos, sin = freqs
        if cos.dtype != torch.float32 or sin.shape != cos.shape or cos.shape[-1] != rope_dim:
            raise B200AwqError(f"b200awq: style 1 freqs must be the f32 (cos, sin) pair [S, {rope_dim}]")
        h = rope_dim // 2
        t = torch.stack((cos.reshape(-1, rope_dim)[:, :h], sin.reshape(-1, rope_dim)[:, :h]), dim=-1).contiguous()
    if tuple(t.shape[1:]) != (rope_dim // 2, 2) or not t.is_contiguous():
        raise B200AwqError(f"b200awq: style 1 freqs must be [S, {rope_dim // 2}, 2] f32")
    return t


def mla_descriptor(pos, freqs, k_cache, v_cache, q_out, M, n_heads, nope_dim, rope_dim, v_dim, kv_lora_rank, style,
                   cache_len=None):
    """Checks the tensors of the MLA glue for M token rows and returns the b200awq_mla_t.  freqs: the [S_f, Dr/2, 2] f32
    table (_mla_freqs) or None (MLA_KV); k_cache f16 [B >= M, S, H, Dn + Dr] with contiguous [S, H, Dn + Dr] entries;
    v_cache f16 [B >= M, S, H, >= Dv] (padded heads allowed: the head stride is its last dimension) with contiguous
    entries, or None (MLA_ROPE); q_out contiguous f16 [M, H, Dn + Dr] (any shape of M H (Dn + Dr) elements ending in
    [H, Dn + Dr]) or None (MLA_KV); pos a device int32 tensor of one element.  k_cache may be None for MLA_Q_ROPE, which
    writes no cache: cache_len then gives the cache's S, which still bounds the position.  The kernels write batch
    entry m and q_out row m for every m < M, so every size is checked against M before a pointer is taken."""
    H, Dn, Dr, Dv, C, M = int(n_heads), int(nope_dim), int(rope_dim), int(v_dim), int(kv_lora_rank), int(M)
    W = Dn + Dr
    d = _cabi.Mla()
    d.n_heads, d.nope_dim, d.rope_dim, d.v_dim, d.kv_lora_rank, d.style = H, Dn, Dr, Dv, C, int(style)
    if pos.dtype != torch.int32 or pos.numel() != 1:
        raise B200AwqError("b200awq: pos must be a device int32 tensor with one element")
    if k_cache is None:
        if cache_len is None or int(cache_len) <= 0 or v_cache is not None:
            raise B200AwqError("b200awq: without k_cache, give the cache length (and no v_cache)")
    elif (k_cache.dtype != torch.float16 or k_cache.dim() != 4 or tuple(k_cache.shape[2:]) != (H, W)
            or k_cache.stride(3) != 1 or k_cache.stride(2) != W or k_cache.stride(1) != H * W):
        raise B200AwqError(f"b200awq: k_cache must be float16 [B, S, {H}, {W}] with contiguous [S, H, D] entries")
    elif k_cache.shape[0] < M:
        raise B200AwqError(f"b200awq: k_cache has {k_cache.shape[0]} batch entries for {M} token rows")
    if v_cache is not None:
        if (v_cache.dtype != torch.float16 or v_cache.dim() != 4 or v_cache.shape[2] != H or v_cache.shape[3] < Dv
                or v_cache.stride(3) != 1 or v_cache.stride(2) != v_cache.shape[3]
                or v_cache.stride(1) != H * v_cache.shape[3] or v_cache.shape[1] != k_cache.shape[1]):
            raise B200AwqError(f"b200awq: v_cache must be float16 [B, S, {H}, >= {Dv}] with contiguous entries and "
                               "k_cache's S")
        if v_cache.shape[0] < M:
            raise B200AwqError(f"b200awq: v_cache has {v_cache.shape[0]} batch entries for {M} token rows")
    if q_out is not None and (q_out.dtype != torch.float16 or not q_out.is_contiguous()
                              or tuple(q_out.shape[-2:]) != (H, W) or q_out.numel() != M * H * W):
        raise B200AwqError(f"b200awq: q_out must be a contiguous float16 [{M}, {H}, {W}] tensor")
    _require_cuda(pos, k_cache, v_cache, freqs, q_out)
    d.pos = pos.data_ptr()
    if k_cache is None:
        d.cache_len = int(cache_len)
    else:
        d.cache_len, d.k_batch_stride, d.k_cache = k_cache.shape[1], k_cache.stride(0), k_cache.data_ptr()
    if v_cache is not None:
        d.v_batch_stride, d.v_head_stride, d.v_cache = v_cache.stride(0), v_cache.shape[3], v_cache.data_ptr()
    if freqs is not None:
        d.freqs_len, d.freqs = freqs.shape[0], freqs.data_ptr()
    if q_out is not None:
        d.q_out = q_out.data_ptr()
    return d


def _mla_call(fn, row2, d, M, name, *pre):
    """fn(row, ld, *pre, desc, M, stream); pre: b200awq_mla_k_rope's k_pe column."""
    ld = row2.stride(0) if M > 1 else row2.shape[1]
    with _DeviceGuard(row2.device):
        code = fn(row2.data_ptr(), ld, *pre, d, M, _stream(row2.device))
    check(code, f"{name}(M={M}, H={d.n_heads}, Dn={d.nope_dim}, Dr={d.rope_dim})")


def mla_rope(qkva, freqs, pos, k_cache, n_heads, nope_dim, rope_dim, kv_lora_rank, style, q_out=None):
    """The glue of transformers' DeepseekV2Attention / DeepseekV3Attention (no q LoRA) after the fused
    q_proj | kv_a_proj_with_mqa linear: qkva [.., H (Dn + Dr) + C + Dr] f16 = [q | c_kv | k_pe].  Writes q_out
    [M, H, Dn + Dr] = [q_nope | rotated q_pe] per head (allocated when not given, and returned) and k_cache[m, *pos, h,
    Dn:] = the rotated k_pe for every head h, for token rows m < M <= 8; nothing when *pos is outside the cache or the
    table.  style 0: V2's apply_rotary_emb, freqs = freqs_cis; style 1: V3's apply_rotary_pos_emb_interleave, freqs =
    the (cos, sin) pair (include/b200awq.h states both arithmetics).  c_kv is left to kv_a_layernorm."""
    H, Dn, Dr, C = int(n_heads), int(nope_dim), int(rope_dim), int(kv_lora_rank)
    row2 = _rows(qkva, H * (Dn + Dr) + C + Dr, "qkva")
    M = row2.shape[0]
    if q_out is None:
        q_out = torch.empty((M, H, Dn + Dr), dtype=torch.float16, device=qkva.device)
    f = _mla_freqs(freqs, Dr, int(style))
    d = mla_descriptor(pos, f, k_cache, None, q_out, M, H, Dn, Dr, 0, C, style)
    _require_cuda(qkva)
    _mla_call(lib.b200awq_mla_rope, row2, d, M, "b200awq_mla_rope")
    return q_out


def mla_kv_cache(kv, pos, k_cache, v_cache, n_heads, nope_dim, v_dim):
    """kv_b_proj's output kv [.., H (Dn + Dv)] f16 (per head [k_nope | v]) into the caches at position *pos:
    k_cache[m, *pos, h, :Dn] = k_nope, v_cache[m, *pos, h, :Dv] = v, for token rows m < M <= 8; nothing when *pos is
    outside the cache.  k_cache [B, S, H, Dn + Dr] fixes Dr; v_cache [B, S, H, >= Dv]."""
    H, Dn, Dv = int(n_heads), int(nope_dim), int(v_dim)
    row2 = _rows(kv, H * (Dn + Dv), "kv")
    M = row2.shape[0]
    Dr = k_cache.shape[-1] - Dn
    d = mla_descriptor(pos, None, k_cache, v_cache, None, M, H, Dn, Dr, Dv, 0, 0)
    _require_cuda(kv)
    _mla_call(lib.b200awq_mla_kv, row2, d, M, "b200awq_mla_kv")


def mla_k_rope(qkva, freqs, pos, k_cache, n_heads, nope_dim, rope_dim, kv_lora_rank, q_lora_rank, style):
    """MLA with a q LoRA (DeepseekV2Attention / DeepseekV3Attention with q_lora_rank set), after the fused
    q_a_proj | kv_a_proj_with_mqa linear: qkva [.., Cq + C + Dr] f16 = [q_a | c_kv | k_pe].  Writes k_cache[m, *pos, h,
    Dn:] = the rotated k_pe for every head h, for token rows m < M <= 8; nothing when *pos is outside the cache or the
    table.  freqs and style as mla_rope.  q_a and c_kv are left to q_a_layernorm and kv_a_layernorm."""
    H, Dn, Dr, C, Cq = int(n_heads), int(nope_dim), int(rope_dim), int(kv_lora_rank), int(q_lora_rank)
    row2 = _rows(qkva, Cq + C + Dr, "qkva")
    M = row2.shape[0]
    f = _mla_freqs(freqs, Dr, int(style))
    d = mla_descriptor(pos, f, k_cache, None, None, M, H, Dn, Dr, 0, C, style)
    _require_cuda(qkva)
    _mla_call(lib.b200awq_mla_k_rope, row2, d, M, "b200awq_mla_k_rope", Cq + C)


def mla_q_rope(q, freqs, pos, cache_len, n_heads, nope_dim, rope_dim, style, q_out=None):
    """MLA with a q LoRA, after q_b_proj: q [.., H (Dn + Dr)] f16.  Writes q_out [M, H, Dn + Dr] = [q_nope | rotated
    q_pe] per head (allocated when not given, and returned), for token rows m < M <= 8; nothing when *pos is outside
    [0, min(cache_len, table rows)), the rule mla_k_rope writes the cache by.  freqs and style as mla_rope."""
    H, Dn, Dr = int(n_heads), int(nope_dim), int(rope_dim)
    row2 = _rows(q, H * (Dn + Dr), "q")
    M = row2.shape[0]
    if q_out is None:
        q_out = torch.empty((M, H, Dn + Dr), dtype=torch.float16, device=q.device)
    f = _mla_freqs(freqs, Dr, int(style))
    d = mla_descriptor(pos, f, None, None, q_out, M, H, Dn, Dr, 0, 0, style, cache_len=cache_len)
    _require_cuda(q)
    _mla_call(lib.b200awq_mla_q_rope, row2, d, M, "b200awq_mla_q_rope")
    return q_out


# ------------------------------------------------------------------------------------ MoE (awq_ext surface)
def topk_softmax(topk_weights, topk_ids, token_expert_indicies, gating_output):
    """awq_ext.topk_softmax (fused/moe.py:162-167): fills the three output tensors [M, topk] from gating_output
    [M, E] f32 (softmax over experts, top-k, not renormalised)."""
    _require_cuda(topk_weights, topk_ids, token_expert_indicies, gating_output)
    if gating_output.dtype != torch.float32 or topk_weights.dtype != torch.float32 \
            or topk_ids.dtype != torch.int32 or token_expert_indicies.dtype != torch.int32:
        raise B200AwqError("b200awq: topk_softmax expects f32 gating / weights and i32 index tensors")
    g = gating_output if gating_output.is_contiguous() else gating_output.contiguous()
    for t in (topk_weights, topk_ids, token_expert_indicies):
        if not t.is_contiguous():
            raise B200AwqError("b200awq: topk_softmax outputs must be contiguous")
    M, E = g.shape
    topk = topk_weights.shape[-1]
    with _DeviceGuard(g.device):
        code = lib.b200awq_topk_softmax(g.data_ptr(), topk_weights.data_ptr(), topk_ids.data_ptr(),
                                        token_expert_indicies.data_ptr(), M, E, topk, _stream(g.device))
    check(code, f"b200awq_topk_softmax(M={M}, E={E}, topk={topk})")


def moe_alig_block_size(topk_ids, num_experts, block_size, sorted_token_ids, expert_ids, num_tokens_post_pad):
    """awq_ext.moe_alig_block_size (sic; fused/moe.py:131-133): fills sorted_token_ids, expert_ids,
    num_tokens_post_pad from topk_ids [M, topk] i32."""
    _require_cuda(topk_ids, sorted_token_ids, expert_ids, num_tokens_post_pad)
    for t in (topk_ids, sorted_token_ids, expert_ids, num_tokens_post_pad):
        if t.dtype != torch.int32 or not t.is_contiguous():
            raise B200AwqError("b200awq: moe_alig_block_size expects contiguous int32 tensors")
    numel = topk_ids.numel()
    if sorted_token_ids.numel() < numel + num_experts * (block_size - 1) or expert_ids.numel() < numel + num_experts:
        raise B200AwqError("b200awq: moe_alig_block_size output tensors are too small")
    with _DeviceGuard(topk_ids.device):
        code = lib.b200awq_moe_align_block_size(topk_ids.data_ptr(), numel, int(num_experts), int(block_size),
                                                sorted_token_ids.data_ptr(), expert_ids.data_ptr(),
                                                num_tokens_post_pad.data_ptr(), _stream(topk_ids.device))
    check(code, "b200awq_moe_align_block_size")


def grouped_gemm_forward(x, qweight, scales, qzeros, topk_weights, sorted_token_ids, expert_ids,
                         num_tokens_post_padded, mul_weights, split_k_iters=8):
    """awq_ext.grouped_gemm_forward (fused/moe.py:60-89): x [T, 1 or topk, K] f16, stacked expert weights
    qweight [E, K, N/8] / scales [E, K/G, N] / qzeros [E, K/G, N/8] -> [T, topk, N] f16."""
    _require_cuda(x, qweight, scales, qzeros, topk_weights, sorted_token_ids, expert_ids, num_tokens_post_padded)
    _check_w(qweight, torch.int32, "qweight")
    _check_w(scales, torch.float16, "scales")
    _check_w(qzeros, torch.int32, "qzeros")
    if x.dim() != 3 or x.dtype != torch.float16:
        raise B200AwqError("b200awq: grouped_gemm_forward expects x [T, 1 or topk, K] float16")
    if topk_weights.dtype != torch.float32 or not topk_weights.is_contiguous():
        raise B200AwqError("b200awq: topk_weights must be contiguous float32")
    E, K, N = qweight.shape[0], qweight.shape[1], qweight.shape[2] * 8
    G = K // scales.shape[1]
    T, topk = topk_weights.shape
    xc = x if x.is_contiguous() else x.contiguous()
    if xc.shape[0] != T or xc.shape[1] not in (1, topk) or xc.shape[2] != K:
        raise B200AwqError(f"b200awq: x {tuple(x.shape)} does not match T={T}, topk={topk}, K={K}")
    y = torch.empty((T, topk, N), dtype=torch.float16, device=x.device)
    with _DeviceGuard(x.device):
        st = _stream(x.device)
        slen = sorted_token_ids.numel()
        # decode-sized calls get the split-K scratch of the persistent kernel (8 rows of fp32 per 8 sorted slots);
        # beyond 64 MB of scratch the library's workspace-free grouped kernel runs instead
        need = 16384 + slen * N * 4
        ws = _workspace(x.device, st, need) if need <= (64 << 20) else None
        code = lib.b200awq_grouped_gemm_forward(
            xc.data_ptr(), int(xc.shape[1]), qweight.data_ptr(), scales.data_ptr(), qzeros.data_ptr(),
            topk_weights.data_ptr(), sorted_token_ids.data_ptr(), expert_ids.data_ptr(),
            num_tokens_post_padded.data_ptr(), y.data_ptr(), T, topk, slen, E, K, N, G,
            1 if mul_weights else 0, 16, ws.data_ptr() if ws is not None else None,
            ws.numel() if ws is not None else 0, st)
    check(code, f"b200awq_grouped_gemm_forward(T={T}, topk={topk}, E={E}, K={K}, N={N}, G={G})")
    return y


# ---------------------------------------------------------------------------- awq_v2_ext surface
def _fast_group_size(K: int, rows: int) -> int:
    from .packing import calculate_zeros_width

    for g in (128, 64, 32):
        if K % g == 0 and calculate_zeros_width(K, g) * 8 == rows:
            return g
    raise B200AwqError(f"b200awq: cannot infer group size from scales rows={rows}, K={K}")


def gemv_forward_cuda_decode(x, qweight, scales, szeros, m, n, k, group_size):
    """awq_v2_ext.gemv_forward_cuda_decode (gemv_fast.py:192-201): x [B, 1, K] -> [B, 1, N]."""
    out = linear_forward("fast", x, qweight, scales, szeros, group_size)
    return out.reshape(x.shape[:-1] + (out.shape[-1],))


def gemm_forward_cuda_prefill(x, qweight, scales, szeros):
    """awq_v2_ext.gemm_forward_cuda_prefill (gemv_fast.py:203-205): x [B, S, K] -> [B, S, N]."""
    K = qweight.shape[1]
    out = linear_forward("fast", x, qweight, scales, szeros, _fast_group_size(K, scales.shape[0]))
    return out.reshape(x.shape[:-1] + (out.shape[-1],))


def stream_pack(qweight, scales, qzeros, mode: int = 0) -> torch.Tensor:
    """One-time re-layout of a GEMM-layout linear into the stream format the decode-program kernel reads
    (include/b200awq.h; the post_init-style hook, cf. awq/modules/linear/exllama.py:66-79).  Returns a uint8 tensor."""
    _require_cuda(qweight, scales, qzeros)
    _check_w(qweight, torch.int32, "qweight")
    _check_w(scales, torch.float16, "scales")
    _check_w(qzeros, torch.int32, "qzeros")
    K, N = qweight.shape[0], qweight.shape[1] * 8
    G = K // scales.shape[0]
    nbytes = lib.b200awq_stream_bytes(K, N, G)
    if nbytes == 0:
        raise B200AwqError(f"b200awq: no stream format for K={K}, N={N}, G={G}")
    out = torch.empty(nbytes, dtype=torch.uint8, device=qweight.device)
    with _DeviceGuard(qweight.device):
        code = lib.b200awq_stream_pack(qweight.data_ptr(), scales.data_ptr(), qzeros.data_ptr(), out.data_ptr(), K, N, G,
                                       int(mode), _stream(qweight.device))
    check(code, f"b200awq_stream_pack(K={K}, N={N}, G={G}, mode={mode})")
    return out


def stream_pack_rotary(qweight, scales, qzeros, head_dim: int, rotary_dim=None) -> torch.Tensor:
    """The stream format in mode 2 (include/b200awq.h): RoPE's column pairs of every head share a lane - (i, i + D/2)
    for full rotary, (i, i + R/2) and the pass-through pairs after column R for rotary_dim R < D (None: R = D).
    What a decode program packs a qkv linear into when a ROPE_KV op folds into its finish."""
    _require_cuda(qweight, scales, qzeros)
    _check_w(qweight, torch.int32, "qweight")
    _check_w(scales, torch.float16, "scales")
    _check_w(qzeros, torch.int32, "qzeros")
    K, N = qweight.shape[0], qweight.shape[1] * 8
    G = K // scales.shape[0]
    nbytes = lib.b200awq_stream_bytes(K, N, G)
    if nbytes == 0:
        raise B200AwqError(f"b200awq: no stream format for K={K}, N={N}, G={G}")
    out = torch.empty(nbytes, dtype=torch.uint8, device=qweight.device)
    with _DeviceGuard(qweight.device):
        code = lib.b200awq_stream_pack_partial_rotary(qweight.data_ptr(), scales.data_ptr(), qzeros.data_ptr(),
                                                      out.data_ptr(), K, N, G, int(head_dim),
                                                      int(rotary_dim or head_dim), _stream(qweight.device))
    check(code, f"b200awq_stream_pack_partial_rotary(K={K}, N={N}, G={G}, head_dim={head_dim}, "
                f"rotary_dim={rotary_dim})")
    return out


def set_knob(key: int, value: int) -> None:
    check(lib.b200awq_set_knob(key, value), "b200awq_set_knob")


def get_knob(key: int) -> int:
    return lib.b200awq_get_knob(key)
