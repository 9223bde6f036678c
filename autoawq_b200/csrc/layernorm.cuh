// LayerNorm and GELU (B200AWQ_OP_LAYER_NORM / _GELU / _GELU_TANH, include/b200awq.h): the arithmetic shared by the
// stand-alone kernels (aux.cu) and the decode-program kernel that folds them (program_stream_body.inc under
// SP_LAYERNORM: the LayerNorm in a linear's staging, the GELU in its finish).  Every step is an explicit IEEE fp32
// operation, so -fmad cannot contract the two callers differently and they agree bit for bit.
#pragma once
#include <cuda_fp16.h>

namespace b200awq {

// the pair (v0, v1) of a chunk into the running sum of x: s + (v0 + v1)
__device__ __forceinline__ float ln_sum_pair(float s, __half2 v) {
  const float2 f = __half22float2(v);
  return __fadd_rn(s, __fadd_rn(f.x, f.y));
}
// the pair into the running centred sum of squares: s + (d0 d0 + d1 d1), d = x - mean
__device__ __forceinline__ float ln_sq_pair(float s, __half2 v, float mean) {
  const float2 f = __half22float2(v);
  const float d0 = __fsub_rn(f.x, mean), d1 = __fsub_rn(f.y, mean);
  return __fadd_rn(s, __fadd_rn(__fmul_rn(d0, d0), __fmul_rn(d1, d1)));
}
__device__ __forceinline__ float ln_mean(float s1, int K) { return __fdiv_rn(s1, static_cast<float>(K)); }
__device__ __forceinline__ float ln_rstd(float s2, int K, float eps) {
  return rsqrtf(__fadd_rn(__fdiv_rn(s2, static_cast<float>(K)), eps));
}
// fp16(((x - mean) r) w [+ b]); has_b: the LayerNorm has a bias
__device__ __forceinline__ __half ln_apply(float x, float mean, float r, float w, float b, bool has_b) {
  const float v = __fmul_rn(__fmul_rn(__fsub_rn(x, mean), r), w);
  return __float2half_rn(has_b ? __fadd_rn(v, b) : v);
}

// torch's GELU formulas on an fp16 value (aten GeluCUDAKernelImpl, opmath float): kind 1 = exact (erf), 2 = tanh
// (the tanh form's kappa x^3 + x is the fma nvcc makes of torch's expression)
__device__ __forceinline__ float gelu_f32(float x, int kind) {
  if (kind == 2) {
    constexpr float kBeta = static_cast<float>(1.41421356237309504880 * 1.12837916709551257390 * 0.5);
    constexpr float kKappa = 0.044715f;
    const float inner = __fmul_rn(kBeta, __fmaf_rn(kKappa, __fmul_rn(__fmul_rn(x, x), x), x));
    return __fmul_rn(__fmul_rn(0.5f, x), __fadd_rn(1.f, tanhf(inner)));
  }
  constexpr float kAlpha = static_cast<float>(0.70710678118654752440);
  return __fmul_rn(__fmul_rn(x, 0.5f), __fadd_rn(1.f, erff(__fmul_rn(x, kAlpha))));
}
__device__ __forceinline__ __half gelu_h(__half x, int kind) { return __float2half_rn(gelu_f32(__half2float(x), kind)); }

}  // namespace b200awq
