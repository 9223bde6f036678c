// RoPE + KV-cache append of one decode step (B200AWQ_OP_ROPE_KV, include/b200awq.h): the per-pair step shared by the
// stand-alone kernel (aux.cu) and the finish of the decode-program kernels that fold it into a qkv linear
// (program_stream_body.inc / program_batch_body.inc under SP_ROPE).
//
// Reference: awq/modules/fused/attn.py:53-86 (RoPE.forward: q and k viewed as complex pairs (x[i], x[i + D/2]), times
// freqs_cis[pos, i] in fp32, rounded back with .type_as) and awq/modules/fused/cache.py:41-46 (update_kv).
#pragma once
#include <cuda_fp16.h>

#include "../../include/b200awq.h"

namespace b200awq {

// R, the rotated columns of a q / k head (b200awq_rope_t.rotary_dim; 0 means D)
__host__ __device__ __forceinline__ int rope_rotary_dim(const b200awq_rope_t& r) {
  return r.rotary_dim != 0 ? r.rotary_dim : r.head_dim;
}

// The column map of a head (include/b200awq.h, b200awq_rope_t): pair p < D/2 of a head of D columns whose first R are
// rotated -> its columns (lo, hi) within the head.  p < R/2: the rotated pair (p, p + R/2); p >= R/2: the pass-through
// pair (R + q, R + q + (D - R)/2) with q = p - R/2.  R = D gives (p, p + D/2).  The stand-alone kernel, the mode-2
// packer and the mode-2 finishes (program_stream.cuh: sp_cols_rot) all pair columns through this one definition.
__host__ __device__ __forceinline__ void rope_cols(int D, int R, int p, int& lo, int& hi) {
  const int hr = R >> 1;
  if (p < hr) {
    lo = p;
    hi = p + hr;
  } else {
    lo = p + hr;
    hi = lo + ((D - R) >> 1);
  }
}

// One pair of token row m, written to q_out row m and to cache entry e at cache row pos, rotated with freqs row rot:
// columns lo = h D + i and hi = h D + j of head h, paired by rope_cols.  a, b: the fp16 qkv values.  A q / k pair with
// i < R/2 is rotated; every other pair (the pass-through columns, a v head) is copied.  (rope_row_pos gives e, pos and
// rot: e = m and rot = pos for a step of one token per sequence without a rotary offset.)
// The rotation is torch's complex<float> product (c10 complex operator*=: re = a c - b s, im = a s + b c) with the
// contraction nvcc gives it there, re = fma(a, c, -(b s)) and im = fma(b, c, a s); explicit intrinsics keep -fmad from
// changing it.  Torch's loops for other shapes differ in a few elements by one fp16 ulp (DESIGN.md 3.5f;
// tests/test_gpu_program_rope.py compares against RoPE.forward with that bound).
__device__ __forceinline__ void rope_pair(const b200awq_rope_t& r, int pos, int rot, int m, int e, int lo, int hi,
                                          __half a, __half b) {
  const int D = r.head_dim, hr = rope_rotary_dim(r) >> 1;
  const int h = lo / D, i = lo - h * D, j = hi - h * D;
  const int H = r.n_heads, KV = r.n_kv_heads;
  if (h >= H + KV) {   // v head: unrotated
    __half* v = static_cast<__half*>(r.v_cache) + (size_t)e * r.cache_batch_stride + ((size_t)pos * KV + (h - H - KV)) * D;
    v[i] = a;
    v[j] = b;
    return;
  }
  __half* dst = h < H ? static_cast<__half*>(r.q_out) + ((size_t)m * H + h) * D
                      : static_cast<__half*>(r.k_cache) + (size_t)e * r.cache_batch_stride + ((size_t)pos * KV + (h - H)) * D;
  if (i >= hr) {       // pass-through pair
    dst[i] = a;
    dst[j] = b;
    return;
  }
  const float2 cs = reinterpret_cast<const float2*>(r.freqs)[(size_t)rot * hr + i];
  const float fa = __half2float(a), fb = __half2float(b);
  const float re = __fmaf_rn(fa, cs.x, -__fmul_rn(fb, cs.y));
  const float im = __fmaf_rn(fb, cs.x, __fmul_rn(fa, cs.y));
  dst[i] = __float2half_rn(re);
  dst[j] = __float2half_rn(im);
}

// Token row m of a step of T tokens per sequence (T = 1: one token, B200AWQ_OP_ROPE_KV): row m = b T + t is token t of
// sequence b, so its cache entry is e = b, its cache row p = p0 + t (p0 = *r.pos) and its rotary row rot = p + off[b]
// (off: B200AWQ_OP_ROPE_KV_OFFSET's per-sequence rotary offsets; null: rot = p).  Returns p, or -1 when p is outside the
// cache or rot outside the frequency table (then the row writes nothing; the other rows of the step still do).
__device__ __forceinline__ int rope_row_pos(const b200awq_rope_t& r, int p0, int T, const int32_t* off, int m, int& e,
                                            int& rot) {
  e = m / T;
  const long long p = (long long)p0 + (m - e * T), q = off != nullptr ? p + off[e] : p;
  rot = static_cast<int>(q);
  return (p >= 0 && p < r.cache_len && q >= 0 && q < r.freqs_len) ? static_cast<int>(p) : -1;
}

// ---- Qwen3 q_norm / k_norm in front of the rotation (B200AWQ_OP_QK_NORM_ROPE_KV).  The sum of squares of a head is
// taken in one fixed order, written only here, so the stand-alone kernel (aux.cu) and the decode-program finish
// (SP_QKNORM), whose sets of one head may sit on different CTAs, produce the same bits:
//   set t (t < D / 16) of a head holds the pairs (8 t + g, 8 t + g + D / 2), g = 0..7, one per lane of an aligned
//   group of 8 lanes; qk_set_partial is the set's partial, qk_head_sum the head total over the sets in ascending t.

// s_g = a^2 + b^2 (fp16 squares are exact in fp32: contraction cannot change it), xor butterfly over the 8 lanes of
// the group (offsets 4, 2, 1): every lane of the group returns the same bits.  All 8 lanes must call it together.
__device__ __forceinline__ float qk_set_partial(__half a, __half b) {
  const unsigned mask = 0xffu << (threadIdx.x & 24);
  const float fa = __half2float(a), fb = __half2float(b);
  float s = __fadd_rn(__fmul_rn(fa, fa), __fmul_rn(fb, fb));
  s = __fadd_rn(s, __shfl_xor_sync(mask, s, 4));
  s = __fadd_rn(s, __shfl_xor_sync(mask, s, 2));
  s = __fadd_rn(s, __shfl_xor_sync(mask, s, 1));
  return s;
}

// the head total: partial(t) for t = 0 .. nsets - 1, summed in ascending t in fp32
template <typename Partial>
__device__ __forceinline__ float qk_head_sum(int nsets, Partial&& partial) {
  float s = 0.f;
  for (int t = 0; t < nsets; ++t) s = __fadd_rn(s, partial(t));
  return s;
}

// Qwen3RMSNorm.forward on one pair of fp16 values (column col = h D + i of token row m, partner col + D / 2; full
// rotary only) of a q or k head with total sum of squares ss, then rope_pair on the result (cache entry e, cache row
// pos, freqs row rot):
//   r = rsqrtf(ss * inv_d + eps), x' = fp16(w * fp16(x * r))   (hidden_states * torch.rsqrt(variance + eps), .to(fp16),
//   weight * it: transformers' Qwen3RMSNorm)
// inv_d = fp32(1 / D), rounded on the host: torch.mean scales its sum by that factor, and ss * inv_d == ss / D for a
// power-of-two D.  (A device division would also pull its slow-path subroutine into the stream kernels, whose call
// convention costs the 8-warp kernel a spill.)
__device__ __forceinline__ void qk_norm_rope_pair(const b200awq_qk_norm_rope_t& q, float inv_d, int pos, int rot, int m,
                                                  int e, int col, __half a, __half b, float ss) {
  const int D = q.rope.head_dim, h = col / D, i = col - h * D;
  const __half* w = static_cast<const __half*>(h < q.rope.n_heads ? q.q_norm_weight : q.k_norm_weight);
  const float r = rsqrtf(__fadd_rn(__fmul_rn(ss, inv_d), q.eps));
  const __half na = __float2half_rn(__fmul_rn(__half2float(a), r));
  const __half nb = __float2half_rn(__fmul_rn(__half2float(b), r));
  const __half wa = __float2half_rn(__fmul_rn(__half2float(w[i]), __half2float(na)));
  const __half wb = __float2half_rn(__fmul_rn(__half2float(w[i + (D >> 1)]), __half2float(nb)));
  rope_pair(q.rope, pos, rot, m, e, col, col + (D >> 1), wa, wb);
}

// ---- MLA (B200AWQ_OP_MLA_ROPE / _MLA_KV / _MLA_K_ROPE / _MLA_Q_ROPE, include/b200awq.h): the per-pair / per-column
// steps shared by the stand-alone kernels (aux.cu) and the finish of the decode-program kernels that fold them
// (program_stream_body.inc under SP_MLA / SP_MLA_LORA).
// Reference: transformers 5.5 DeepseekV2Attention.forward (apply_rotary_emb) and DeepseekV3Attention.forward
// (apply_rotary_pos_emb_interleave).

// the position of this step, or -1 when it is outside the cache (MLA_ROPE: or the frequency table; MLA_KV reads none)
__device__ __forceinline__ int mla_pos(const b200awq_mla_t& d, bool rope) {
  const int p = *d.pos;
  return (p >= 0 && p < d.cache_len && (!rope || p < d.freqs_len)) ? p : -1;
}

// Rotary pair i (a = x[2i], b = x[2i + 1]) of a rope slice of Dr elements: the two results and their places in the
// rotated slice.  Style 0 is the complex<float> product of apply_rotary_emb with rope_pair's contraction, back at the
// interleaved places 2i, 2i + 1.  Style 1 is apply_rotary_pos_emb_interleave's fp16 tensor arithmetic: cos / sin cast
// to fp16, every product and the sum rounded to fp16 (each an exact fp32 value rounded once, as torch's half kernels
// compute them), de-interleaved to i, i + Dr/2.
struct MlaRot {
  int j0, j1;
  __half o0, o1;
};
__device__ __forceinline__ MlaRot mla_rotate(const b200awq_mla_t& d, int pos, int i, __half a, __half b) {
  const int half = d.rope_dim >> 1;
  const float2 cs = reinterpret_cast<const float2*>(d.freqs)[(size_t)pos * half + i];
  const float fa = __half2float(a), fb = __half2float(b);
  MlaRot r;
  if (d.style == 0) {
    r.j0 = 2 * i;
    r.j1 = 2 * i + 1;
    r.o0 = __float2half_rn(__fmaf_rn(fa, cs.x, -__fmul_rn(fb, cs.y)));
    r.o1 = __float2half_rn(__fmaf_rn(fb, cs.x, __fmul_rn(fa, cs.y)));
    return r;
  }
  const float c = __half2float(__float2half_rn(cs.x)), s = __half2float(__float2half_rn(cs.y));
  auto h = [](float v) { return __half2float(__float2half_rn(v)); };
  r.j0 = i;
  r.j1 = i + half;
  r.o0 = __float2half_rn(__fadd_rn(h(__fmul_rn(fa, c)), h(__fmul_rn(-fb, s))));
  r.o1 = __float2half_rn(__fadd_rn(h(__fmul_rn(fb, c)), h(__fmul_rn(fa, s))));
  return r;
}

// Columns (col, col + 1) of token row m's q row [H (Dn + Dr), per head [nope | pe]] (col even, col < H (Dn + Dr); a, b
// their values): q_nope copied, q_pe rotated into q_out.  MLA_ROPE's q part and all of MLA_Q_ROPE.
__device__ __forceinline__ void mla_q_pair(const b200awq_mla_t& d, int pos, int m, int col, __half a, __half b) {
  const int W = d.nope_dim + d.rope_dim, H = d.n_heads;
  const int h = col / W, i = col - h * W;
  __half* q = static_cast<__half*>(d.q_out) + ((size_t)m * H + h) * W;
  if (i < d.nope_dim) {
    q[i] = a;
    q[i + 1] = b;
  } else {
    const MlaRot r = mla_rotate(d, pos, (i - d.nope_dim) >> 1, a, b);
    q[d.nope_dim + r.j0] = r.o0;
    q[d.nope_dim + r.j1] = r.o1;
  }
}

// Elements (kp, kp + 1) of token row m's k_pe (kp even; a, b their values): rotated into the k rows of all H heads at
// position pos.  MLA_ROPE's k part and all of MLA_K_ROPE.
__device__ __forceinline__ void mla_k_pair(const b200awq_mla_t& d, int pos, int m, int kp, __half a, __half b) {
  const int W = d.nope_dim + d.rope_dim, H = d.n_heads, qn = H * W;
  const MlaRot r = mla_rotate(d, pos, kp >> 1, a, b);
  __half* k = static_cast<__half*>(d.k_cache) + (size_t)m * d.k_batch_stride + (size_t)pos * qn + d.nope_dim;
  for (int h = 0; h < H; ++h) {
    k[(size_t)h * W + r.j0] = r.o0;
    k[(size_t)h * W + r.j1] = r.o1;
  }
}

// MLA_ROPE on columns (col, col + 1) of token row m's q_proj | kv_a_proj_with_mqa row (col even; a, b their values):
// q_nope copied and q_pe rotated into q_out, c_kv nothing, k_pe rotated into the k rows of all H heads at position pos
__device__ __forceinline__ void mla_rope_pair(const b200awq_mla_t& d, int pos, int m, int col, __half a, __half b) {
  const int qn = d.n_heads * (d.nope_dim + d.rope_dim);
  if (col < qn) {
    mla_q_pair(d, pos, m, col, a, b);
    return;
  }
  const int kp = col - qn - d.kv_lora_rank;
  if (kp < 0) return;
  mla_k_pair(d, pos, m, kp, a, b);
}

// The mode-3 finish of an op with a q LoRA MLA op folded in (kind 3: MLA_K_ROPE on a row of N columns whose last Dr are
// k_pe; kind 4: MLA_Q_ROPE), on columns (col, col + 1) of token row m
__device__ __forceinline__ void mla_lora_pair(const b200awq_mla_t& d, int kind, int pos, int m, int N, int col, __half a,
                                              __half b) {
  if (kind == 4) {
    mla_q_pair(d, pos, m, col, a, b);
    return;
  }
  const int kp = col - (N - d.rope_dim);
  if (kp >= 0) mla_k_pair(d, pos, m, kp, a, b);
}

// MLA_KV on column col of token row m's kv_b_proj row (value x): k_nope into k_cache, v into v_cache, at position pos
__device__ __forceinline__ void mla_kv_col(const b200awq_mla_t& d, int pos, int m, int col, __half x) {
  const int W = d.nope_dim + d.v_dim, h = col / W, i = col - h * W, H = d.n_heads;
  if (i < d.nope_dim)
    static_cast<__half*>(d.k_cache)[(size_t)m * d.k_batch_stride + ((size_t)pos * H + h) * (d.nope_dim + d.rope_dim) + i] = x;
  else
    static_cast<__half*>(d.v_cache)[(size_t)m * d.v_batch_stride + ((size_t)pos * H + h) * d.v_head_stride + i - d.nope_dim] = x;
}

}  // namespace b200awq
