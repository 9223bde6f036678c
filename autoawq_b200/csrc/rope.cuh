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

// One pair (column h D + i and h D + D/2 + i, i < D/2) of token row m; `col` = h D + i.  a, b: the fp16 qkv values.
// The rotation is torch's complex<float> product (c10 complex operator*=: re = a c - b s, im = a s + b c) with the
// contraction nvcc gives it there, re = fma(a, c, -(b s)) and im = fma(b, c, a s); explicit intrinsics keep -fmad from
// changing it.  Torch's loops for other shapes differ in a few elements by one fp16 ulp (DESIGN.md 3.5f;
// tests/test_gpu_program_rope.py compares against RoPE.forward with that bound).
__device__ __forceinline__ void rope_pair(const b200awq_rope_t& r, int pos, int m, int col, __half a, __half b) {
  const int D = r.head_dim, half = D >> 1;
  const int h = col / D, i = col - h * D;
  const int H = r.n_heads, KV = r.n_kv_heads;
  if (h >= H + KV) {   // v head: unrotated
    __half* v = static_cast<__half*>(r.v_cache) + (size_t)m * r.cache_batch_stride + ((size_t)pos * KV + (h - H - KV)) * D;
    v[i] = a;
    v[i + half] = b;
    return;
  }
  const float2 cs = reinterpret_cast<const float2*>(r.freqs)[(size_t)pos * half + i];
  const float fa = __half2float(a), fb = __half2float(b);
  const float re = __fmaf_rn(fa, cs.x, -__fmul_rn(fb, cs.y));
  const float im = __fmaf_rn(fb, cs.x, __fmul_rn(fa, cs.y));
  __half* dst = h < H ? static_cast<__half*>(r.q_out) + ((size_t)m * H + h) * D
                      : static_cast<__half*>(r.k_cache) + (size_t)m * r.cache_batch_stride + ((size_t)pos * KV + (h - H)) * D;
  dst[i] = __float2half_rn(re);
  dst[i + half] = __float2half_rn(im);
}

// the position of this step, or -1 when it is outside the cache / the frequency table (then nothing is written)
__device__ __forceinline__ int rope_pos(const b200awq_rope_t& r) {
  const int p = *r.pos;
  return (p >= 0 && p < r.cache_len && p < r.freqs_len) ? p : -1;
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

// Qwen3RMSNorm.forward on one pair of fp16 values (column col = h D + i of token row m, partner col + D / 2) of a q
// or k head with total sum of squares ss, then rope_pair on the result:
//   r = rsqrtf(ss * inv_d + eps), x' = fp16(w * fp16(x * r))   (hidden_states * torch.rsqrt(variance + eps), .to(fp16),
//   weight * it: transformers' Qwen3RMSNorm)
// inv_d = fp32(1 / D), rounded on the host: torch.mean scales its sum by that factor, and ss * inv_d == ss / D for a
// power-of-two D.  (A device division would also pull its slow-path subroutine into the stream kernels, whose call
// convention costs the 8-warp kernel a spill.)
__device__ __forceinline__ void qk_norm_rope_pair(const b200awq_qk_norm_rope_t& q, float inv_d, int pos, int m, int col,
                                                  __half a, __half b, float ss) {
  const int D = q.rope.head_dim, h = col / D, i = col - h * D;
  const __half* w = static_cast<const __half*>(h < q.rope.n_heads ? q.q_norm_weight : q.k_norm_weight);
  const float r = rsqrtf(__fadd_rn(__fmul_rn(ss, inv_d), q.eps));
  const __half na = __float2half_rn(__fmul_rn(__half2float(a), r));
  const __half nb = __float2half_rn(__fmul_rn(__half2float(b), r));
  const __half wa = __float2half_rn(__fmul_rn(__half2float(w[i]), __half2float(na)));
  const __half wb = __float2half_rn(__fmul_rn(__half2float(w[i + (D >> 1)]), __half2float(nb)));
  rope_pair(q.rope, pos, m, col, wa, wb);
}

}  // namespace b200awq
