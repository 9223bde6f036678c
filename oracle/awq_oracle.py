"""CPU oracle for the AWQ W4A16 linear path.  TEST INFRASTRUCTURE ONLY.

This file is a numpy restatement of the reference's algorithm for the hot path
(casper-hansen/AutoAWQ @ 88e4c76).  It is the checker, never the product: only
``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import it.  Nothing under ``autoawq_b200/``,
``awq_ext/`` or ``awq_v2_ext/`` imports it, and those packages raise when the
CUDA library is missing instead of falling back to this code.

Parity pinning: every function below is checked against outputs of the real
reference (imported from an upstream checkout, oracle/reference.py) by
``tests/golden/make_golden.py``; the resulting vectors are committed under
``tests/golden/*.npz`` and re-checked by ``tests/test_oracle_golden.py`` on every
run.  The one known-answer recipe the reference's own tests hold for this path
(``tests/test_dequantization.py:10-58``: raw int32 words + randn scales, K=4096,
N=1792, g=128, dequant allclose rtol=1e-4) is mirrored in those fixtures.
GEMM/GEMV *outputs* are unpinned by the reference (no test, SURVEY.md section 8c); for
them the oracle is the fp64 contraction of the bit-exact dequantised weights.

Reference map (file:line in the reference checkout):
  AWQ_ORDER / AWQ_REVERSE_ORDER ........ awq/utils/packing_utils.py:4-5
  unpack_gemm, dequantize_gemm ......... awq/utils/packing_utils.py:8-43,87-102
  pack_gemm ............................ awq/modules/linear/gemm.py:194-249
  calculate_zeros_width ................ awq/modules/linear/gemv.py:12-24
  pack_gemv ............................ awq/modules/linear/gemv.py:96-153
  pack_gemv_fast ....................... awq/modules/linear/gemv_fast.py:26-65,146-181
  quantize_rtn ......................... awq/quantize/quantizer.py:74-109
  wqlinear_forward (naive CPU branch) .. awq/modules/linear/gemm.py:71-86
"""
from __future__ import annotations

import numpy as np

# nibble i of a GEMM-layout word holds column 8c + AWQ_ORDER[i]   (packing_utils.py:4)
AWQ_ORDER = (0, 2, 4, 6, 1, 3, 5, 7)
# column 8c + j sits at nibble AWQ_REVERSE_ORDER[j]                 (packing_utils.py:5)
AWQ_REVERSE_ORDER = (0, 4, 1, 5, 2, 6, 3, 7)
PACK = 8  # 4-bit values per int32

_GEMM_SHIFTS = np.array([4 * r for r in AWQ_REVERSE_ORDER], dtype=np.uint32)  # per column j
_SEQ_SHIFTS = np.arange(0, 32, 4, dtype=np.uint32)


# --------------------------------------------------------------------------- GEMM layout
def unpack_gemm(words: np.ndarray) -> np.ndarray:
    """[R, C] int32 (GEMM interleave) -> [R, 8C] uint8 nibbles in natural column order.

    Equivalent to unpack_awq + reverse_awq_order + (& 0xF)  (packing_utils.py:8-43,94-95).
    """
    w = np.ascontiguousarray(words).view(np.uint32)
    out = (w[:, :, None] >> _GEMM_SHIFTS[None, None, :]) & np.uint32(0xF)
    return out.reshape(w.shape[0], -1).astype(np.uint8)


def pack_gemm_words(vals: np.ndarray) -> np.ndarray:
    """[R, 8C] ints in 0..15 -> [R, C] int32 with the AWQ interleave (gemm.py:220-228)."""
    v = np.asarray(vals).astype(np.uint32)
    assert v.shape[1] % PACK == 0
    v = v.reshape(v.shape[0], -1, PACK)
    words = np.zeros(v.shape[:2], dtype=np.uint32)
    for j in range(PACK):
        words |= (v[:, :, j] & np.uint32(0xF)) << np.uint32(4 * AWQ_REVERSE_ORDER[j])
    return words.view(np.int32)


def dequantize_gemm(qweight, qzeros, scales, group_size: int) -> np.ndarray:
    """GEMM-layout dequant, bit-exact restatement of packing_utils.py:87-102.

    W[k, n] = fp16( (nib(k, n) - znib(k // G, n)) * S[k // G, n] ): the integer
    difference is exact, the product is rounded once (RN-even) to fp16.
    """
    iw = unpack_gemm(qweight).astype(np.int8)
    iz = unpack_gemm(qzeros).astype(np.int8)
    s = np.asarray(scales, dtype=np.float16)
    K = iw.shape[0]
    if group_size == -1:
        group_size = K
    assert K % group_size == 0 and iz.shape[0] == K // group_size
    diff = (iw - np.repeat(iz, group_size, axis=0)).astype(np.float16)  # exact: |d| <= 15
    return diff * np.repeat(s, group_size, axis=0)  # one fp16 rounding


def pack_gemm(intweight_kn, zeros_gn):
    """Canonical ints -> (qweight [K, N/8], qzeros [K/G, N/8]) in GEMM layout."""
    return pack_gemm_words(intweight_kn), pack_gemm_words(zeros_gn)


# --------------------------------------------------------------------------- GEMV layout
def calculate_zeros_width(in_features: int, group_size: int = 128, pack_num: int = 8) -> int:
    """Restates gemv.py:12-24 (width in int32 words of the padded zeros row)."""
    if group_size >= 128:
        mult = 1
    elif group_size == 64:
        mult = 2
    elif group_size == 32:
        mult = 4
    else:
        raise NotImplementedError(f"group_size {group_size}")
    base = -(-(in_features // group_size) // pack_num)
    return -(-base // mult) * mult


def pack_gemv(intweight_kn, zeros_gn, scales_gn, group_size: int):
    """Canonical ints -> GEMV layout (gemv.py:96-153).

    qweight [N, K/8] int32, nibble i <- k = 8c + i; qzeros [N, zw] int32, nibble i <- group
    8c' + i (zero padded); scales [N, 8 zw] fp16 (zero padded).
    """
    iw = np.asarray(intweight_kn).astype(np.uint32).T  # [N, K]
    N, K = iw.shape
    G = K if group_size == -1 else group_size
    zw = calculate_zeros_width(K, G)
    qweight = np.zeros((N, K // PACK), dtype=np.uint32)
    iw = iw.reshape(N, K // PACK, PACK)
    for i in range(PACK):
        qweight |= (iw[:, :, i] & np.uint32(0xF)) << _SEQ_SHIFTS[i]
    z = np.zeros((N, zw * PACK), dtype=np.uint32)
    z[:, : K // G] = np.asarray(zeros_gn).astype(np.uint32).T
    z = z.reshape(N, zw, PACK)
    qzeros = np.zeros((N, zw), dtype=np.uint32)
    for i in range(PACK):
        qzeros |= (z[:, :, i] & np.uint32(0xF)) << _SEQ_SHIFTS[i]
    s = np.zeros((N, zw * PACK), dtype=np.float16)
    s[:, : K // G] = np.asarray(scales_gn, dtype=np.float16).T
    return qweight.view(np.int32), qzeros.view(np.int32), s


def unpack_seq(words: np.ndarray) -> np.ndarray:
    """[R, C] int32 sequential nibbles -> [R, 8C] uint8."""
    w = np.ascontiguousarray(words).view(np.uint32)
    out = (w[:, :, None] >> _SEQ_SHIFTS[None, None, :]) & np.uint32(0xF)
    return out.reshape(w.shape[0], -1).astype(np.uint8)


def dequantize_gemv(qweight, qzeros, scales, group_size: int) -> np.ndarray:
    """GEMV-layout dequant -> W [K, N] fp16, same arithmetic as dequantize_gemm."""
    iw = unpack_seq(qweight).astype(np.int8)  # [N, K]
    N, K = iw.shape
    G = K if group_size == -1 else group_size
    ng = K // G
    iz = unpack_seq(qzeros).astype(np.int8)[:, :ng]
    s = np.asarray(scales, dtype=np.float16)[:, :ng]
    diff = (iw - np.repeat(iz, G, axis=1)).astype(np.float16)
    return np.ascontiguousarray((diff * np.repeat(s, G, axis=1)).T)


# ----------------------------------------------------------------------- GEMVFast layout
def _fast_kperm() -> np.ndarray:
    """Position p of a 32-k block holds original k = perm[p]  (gemv_fast.py:31-40)."""
    a = np.arange(32).reshape(4, 4, 2).transpose(1, 0, 2).reshape(32)  # 0,1,8,9,16,17,24,25,...
    a = a.reshape(4, 4, 2).transpose(0, 2, 1).reshape(32)  # per 8: 0,2,4,6,1,3,5,7
    return a


FAST_KPERM = _fast_kperm()


def pack_gemv_fast_weight(intweight_kn, interleave: int = 4, kstride: int = 64) -> np.ndarray:
    """Canonical ints [K, N] -> int16 [N/4, K]  (pack_intweight, gemv_fast.py:26-65).

    After the 32-wide k permutation, rows are taken four at a time; inside every 64-k block the
    four rows' 64 values each are laid out row after row (256 values) and every four consecutive
    values are packed into one int16, nibble r' <- value 4j + r'.
    """
    w = np.asarray(intweight_kn).astype(np.uint16).T  # [N, K]
    N, K = w.shape
    assert N % interleave == 0 and K % kstride == 0 and K % 32 == 0
    w = w.reshape(N, K // 32, 32)[:, :, FAST_KPERM].reshape(N, K)
    w = w.reshape(N // interleave, interleave, K // kstride, kstride).transpose(0, 2, 1, 3)
    w = w.reshape(N // interleave, K // kstride, kstride, interleave)
    packed = w[..., 0] | (w[..., 1] << 4) | (w[..., 2] << 8) | (w[..., 3] << 12)
    return packed.reshape(N // interleave, K).astype(np.uint16).view(np.int16)


def unpack_gemv_fast_weight(qweight_i16, interleave: int = 4, kstride: int = 64) -> np.ndarray:
    """Inverse of pack_gemv_fast_weight -> canonical ints [K, N] uint8."""
    q = np.ascontiguousarray(qweight_i16).view(np.uint16)
    N4, K = q.shape
    N = N4 * interleave
    v = np.stack([(q >> (4 * r)) & 0xF for r in range(interleave)], axis=-1)  # [N/4, K, 4]
    v = v.reshape(N4, K // kstride, kstride * interleave)  # flat = r*64 + kk
    v = v.reshape(N4, K // kstride, interleave, kstride).transpose(0, 2, 1, 3).reshape(N, K)
    inv = np.argsort(FAST_KPERM)
    v = v.reshape(N, K // 32, 32)[:, :, inv].reshape(N, K)
    return np.ascontiguousarray(v.T).astype(np.uint8)


def pack_gemv_fast(intweight_kn, zeros_gn, scales_gn, group_size: int):
    """-> (qweight int16 [N/4, K], scales fp16 [8zw, N], scaled_zeros fp16 [8zw, N]).

    scaled_zeros = fp16(-(S * Z)) computed in fp32 (gemv_fast.py:175-181).
    """
    K, N = np.asarray(intweight_kn).shape
    G = K if group_size == -1 else group_size
    zw = calculate_zeros_width(K, G)
    s = np.zeros((zw * PACK, N), dtype=np.float16)
    s[: K // G] = np.asarray(scales_gn, dtype=np.float16)
    sz = np.zeros((zw * PACK, N), dtype=np.float16)
    sz[: K // G] = (-(s[: K // G].astype(np.float32) * np.asarray(zeros_gn).astype(np.float32))).astype(
        np.float16
    )
    return pack_gemv_fast_weight(intweight_kn), s, sz


def dequantize_gemv_fast_f64(qweight_i16, scales, scaled_zeros, group_size: int) -> np.ndarray:
    """GEMVFast weights as real numbers: W = q * S + SZ in fp64 (no intermediate rounding).

    The awq_v2_ext kernels are absent from the reference tree (parity unpinned); this is the
    mathematical value the stored tensors encode.
    """
    iw = unpack_gemv_fast_weight(qweight_i16).astype(np.float64)  # [K, N]
    K = iw.shape[0]
    G = K if group_size == -1 else group_size
    ng = K // G
    s = np.repeat(np.asarray(scales)[:ng].astype(np.float64), G, axis=0)
    sz = np.repeat(np.asarray(scaled_zeros)[:ng].astype(np.float64), G, axis=0)
    return iw * s + sz


# --------------------------------------------------------------------- quantiser semantics
def quantize_rtn(w_nk: np.ndarray, group_size: int):
    """Zero-point round-to-nearest group quantisation (quantizer.py:74-109).

    Returns (intweight [K, N] uint8, zeros [K/G, N] uint8, scales [K/G, N] fp16) such that the
    stored fp16 scales are the ones used to derive the integers (as from_linear re-derives them).
    """
    w = np.asarray(w_nk, dtype=np.float32)
    N, K = w.shape
    G = K if group_size == -1 else group_size
    g = w.reshape(N, K // G, G)
    mx, mn = g.max(axis=2), g.min(axis=2)
    s = (np.maximum(mx - mn, 1e-5) / 15.0).astype(np.float16)
    s32 = s.astype(np.float32)
    z = np.clip(-np.round(mn / s32), 0, 15)
    q = np.clip(np.round(g / s32[:, :, None]) + z[:, :, None], 0, 15)
    iw = q.reshape(N, K).T.astype(np.uint8)
    return np.ascontiguousarray(iw), np.ascontiguousarray(z.T.astype(np.uint8)), np.ascontiguousarray(s.T)


# ------------------------------------------------------------------------------- forward
def gemm_f64(x, w_kn) -> np.ndarray:
    """fp64 contraction Y = X . W of fp16 activations with bit-exact dequantised weights."""
    return np.asarray(x, dtype=np.float64) @ np.asarray(w_kn, dtype=np.float64)


def wqlinear_forward(x, qweight, qzeros, scales, group_size: int, bias=None) -> np.ndarray:
    """WQLinear_GEMM.forward through the naive branch (gemm.py:71-86, 253-287), fp16 result.

    dequantise -> matmul with wide accumulation -> one rounding to fp16 -> fp16 bias add.
    """
    w = dequantize_gemm(qweight, qzeros, scales, group_size)
    x16 = np.asarray(x, dtype=np.float16)
    y = gemm_f64(x16.reshape(-1, x16.shape[-1]), w).astype(np.float16)
    if bias is not None:
        y = y + np.asarray(bias, dtype=np.float16)
    return y.reshape(x16.shape[:-1] + (w.shape[1],))


def rmsnorm_f64(x, weight, eps: float) -> np.ndarray:
    """x * rsqrt(mean(x^2) + eps) * w in fp64 (what awq/modules/fused/norm.py:19-38 asks of
    awq_ext.layernorm_forward_cuda; unpinned in the reference)."""
    x = np.asarray(x, dtype=np.float64)
    var = (x * x).mean(axis=-1, keepdims=True)
    return x / np.sqrt(var + eps) * np.asarray(weight, dtype=np.float64)


# ----------------------------------------------------------------------- synthetic inputs
def make_case(K: int, N: int, group_size: int, seed: int, raw: bool = False):
    """Deterministic packed test case.

    raw=False: canonical ints U{0..15}, zeros U{0..15}, scales |N(0,1)|*0.01 + 1e-3 (SURVEY 8d).
    raw=True : the reference test's recipe (tests/test_dequantization.py:15-38): full-range int32
               words for qweight/qzeros and randn fp16 scales.
    Returns dict with canonical (intweight, zeros, scales) and GEMM-layout (qweight, qzeros).
    """
    rng = np.random.default_rng(seed)
    G = K if group_size == -1 else group_size
    if raw:
        qweight = rng.integers(-(2**31), 2**31 - 1, size=(K, N // PACK), dtype=np.int64).astype(np.int32)
        qzeros = rng.integers(-(2**31), 2**31 - 1, size=(K // G, N // PACK), dtype=np.int64).astype(np.int32)
        scales = rng.standard_normal((K // G, N)).astype(np.float16)
        iw, iz = unpack_gemm(qweight), unpack_gemm(qzeros)
    else:
        iw = rng.integers(0, 16, size=(K, N), dtype=np.uint8)
        iz = rng.integers(0, 16, size=(K // G, N), dtype=np.uint8)
        scales = (np.abs(rng.standard_normal((K // G, N))) * 0.01 + 1e-3).astype(np.float16)
        qweight, qzeros = pack_gemm(iw, iz)
    return dict(intweight=iw, zeros=iz, scales=scales, qweight=qweight, qzeros=qzeros, group_size=G)


# ------------------------------------------------------------------------------------- MoE (SURVEY 8f #2)
# The reference's MoE kernels live in the un-vendored `autoawq-kernels` package (vLLM lineage); what is restated
# here is the contract its call sites define (awq/modules/fused/moe.py:45-171) - parity unpinned by the reference.
def topk_softmax(gating_output, topk: int):
    """awq_ext.topk_softmax as fused_topk uses it (moe.py:137-171): softmax over the experts in fp32, the `topk`
    largest probabilities per token (ties -> lower expert index), NOT renormalised (fused_topk does that itself).
    Returns (topk_weights [M, topk] f32, topk_ids [M, topk] i32, token_expert_indices [M, topk] i32 = k * M + m)."""
    g = np.asarray(gating_output, dtype=np.float32)
    M, E = g.shape
    e = np.exp((g - g.max(axis=1, keepdims=True)).astype(np.float64))
    p = (e / e.sum(axis=1, keepdims=True)).astype(np.float32)
    ids = np.zeros((M, topk), dtype=np.int32)
    w = np.zeros((M, topk), dtype=np.float32)
    work = p.copy()
    for k in range(topk):
        j = work.argmax(axis=1)  # first maximum = lowest index
        ids[:, k] = j
        w[:, k] = p[np.arange(M), j]
        work[np.arange(M), j] = -1.0
    src = (np.arange(topk, dtype=np.int32)[None, :] * M + np.arange(M, dtype=np.int32)[:, None]).astype(np.int32)
    return w, ids, src


def moe_align_block_size(topk_ids, block_size: int, num_experts: int):
    """moe_align_block_size (moe.py:92-134, including its worked example): flattened slot indices grouped by expert in
    ascending slot order, each expert's run padded with the sentinel `numel` to a multiple of block_size.
    Returns (sorted_ids [numel + E*(block_size-1)] i32, expert_ids [numel + E] i32 (one per block; unused tail left
    at -1 here, uninitialised in the reference), num_tokens_post_padded int)."""
    flat = np.asarray(topk_ids, dtype=np.int64).reshape(-1)
    numel = flat.size
    sorted_ids = np.full(numel + num_experts * (block_size - 1), numel, dtype=np.int32)
    expert_ids = np.full(numel + num_experts, -1, dtype=np.int32)
    pos = 0
    blk = 0
    for e in range(num_experts):
        idx = np.nonzero(flat == e)[0]
        if idx.size == 0:
            continue
        padded = -(-idx.size // block_size) * block_size
        sorted_ids[pos:pos + idx.size] = idx
        expert_ids[blk:blk + padded // block_size] = e
        pos += padded
        blk += padded // block_size
    return sorted_ids, expert_ids, pos


def grouped_gemm_f64(x, w_ekn, topk_weights, sorted_ids, expert_ids, num_post_padded: int, mul_weights: bool,
                     block_size: int = 16):
    """awq_ext.grouped_gemm_forward as apply_moe_weights calls it (moe.py:60-89): for every real slot id in the
    sorted list, out[id // topk, id % topk, :] = x_row(id) . W[expert of its block] (* topk_weights.flat[id] when
    mul_weights), x_row(id) = x[id // topk, 0] for x [T, 1, K] and x.reshape(-1, K)[id] for x [T, topk, K].
    `w_ekn` = dequantised expert weights [E, K, N] (dequantize_gemm per expert).  fp64; rows of slots that are
    never listed stay zero."""
    x = np.asarray(x)
    T, topk = np.asarray(topk_weights).shape
    K = x.shape[-1]
    N = w_ekn.shape[-1]
    xr = x.reshape(-1, K).astype(np.float64)
    per_slot = x.shape[1] != 1
    out = np.zeros((T * topk, N), dtype=np.float64)
    tw = np.asarray(topk_weights, dtype=np.float64).reshape(-1)
    for s in range(num_post_padded):
        i = int(sorted_ids[s])
        if i >= T * topk:
            continue
        e = int(expert_ids[s // block_size])
        row = xr[i if per_slot else i // topk]
        y = row @ w_ekn[e].astype(np.float64)
        out[i] = y * tw[i] if mul_weights else y
    return out.reshape(T, topk, N)
