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

}  // namespace b200awq
