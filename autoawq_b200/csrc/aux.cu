// Glue kernels the reference's fused modules call through awq_ext (SURVEY.md 8f #1, #2):
//   rmsnorm       <- awq_ext.layernorm_forward_cuda   (awq/modules/fused/norm.py:33-36)
//   silu_and_mul  <- awq_ext.silu_and_mul             (awq/modules/fused/moe.py:76)
//   layer_norm / gelu <- nn.LayerNorm (CohereLayerNorm without a bias) and F.gelu of the LayerNorm blocks
//                    (Command-R, StarCoder2, MPT)
//   rope_kv       <- RoPE.forward + WindowedCache.update_kv (awq/modules/fused/attn.py:53-86,243-267)
//   mla_rope / mla_kv <- the glue of transformers' DeepseekV2Attention / DeepseekV3Attention between the projections
//                    and attention (rotary, head split, cache write); mla_k_rope / mla_q_rope: the same with a q LoRA
// fp16 in/out, fp32 math.  Bandwidth-trivial (KBs per decode step); kept simple.
#include "common.cuh"
#include "kernels.h"
#include "layernorm.cuh"
#include "rope.cuh"

namespace b200awq {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// one CTA per row
__global__ void __launch_bounds__(256)
    rmsnorm_kernel(const __half* __restrict__ x, const __half* __restrict__ w, __half* __restrict__ out, int hidden,
                   float eps) {
  __shared__ float wsum[8];
  pdl_trigger();
  pdl_wait();
  const __half* xr = x + (int64_t)blockIdx.x * hidden;
  __half* orow = out + (int64_t)blockIdx.x * hidden;
  float ss = 0.f;
  const bool vec = (hidden % 8) == 0 && (reinterpret_cast<uintptr_t>(xr) % 16) == 0;
  if (vec) {
    for (int i = threadIdx.x * 8; i < hidden; i += blockDim.x * 8) {
      uint4 v = *reinterpret_cast<const uint4*>(xr + i);
      const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float2 f = __half22float2(h[j]);
        ss += f.x * f.x + f.y * f.y;
      }
    }
  } else {
    for (int i = threadIdx.x; i < hidden; i += blockDim.x) {
      float f = __half2float(xr[i]);
      ss += f * f;
    }
  }
  ss = warp_sum(ss);
  if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) tot += (i < (blockDim.x >> 5)) ? wsum[i] : 0.f;
  const float rs = rsqrtf(tot / static_cast<float>(hidden) + eps);
  for (int i = threadIdx.x; i < hidden; i += blockDim.x) {
    float f = __half2float(xr[i]) * rs * __half2float(w[i]);
    orow[i] = __float2half_rn(f);
  }
}

__global__ void __launch_bounds__(256)
    silu_mul_kernel(const __half* __restrict__ gu, __half* __restrict__ out, int rows, int d) {
  pdl_trigger();
  pdl_wait();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)rows * d) return;
  const int r = static_cast<int>(i / d), j = static_cast<int>(i % d);
  const float g = __half2float(gu[(int64_t)r * 2 * d + j]);
  const float u = __half2float(gu[(int64_t)r * 2 * d + d + j]);
  out[i] = __float2half_rn(g / (1.f + __expf(-g)) * u);
}

// one thread per (token row, head, column pair of rope.cuh's rope_cols); rope.cuh has the arithmetic.  T tokens per
// sequence: token row m writes cache entry m / T at position *pos + m % T, rotated at that position plus off[m / T]
// (off null: plus 0; rope_row_pos)
__global__ void __launch_bounds__(256)
    rope_kv_kernel(const __half* __restrict__ qkv, int64_t ldqkv, b200awq_rope_t r, int M, int T,
                   const int32_t* __restrict__ off) {
  pdl_trigger();
  pdl_wait();
  const int half = r.head_dim >> 1, heads = r.n_heads + 2 * r.n_kv_heads;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)M * heads * half) return;
  const int m = static_cast<int>(i / ((int64_t)heads * half));
  int e, rot;
  const int pos = rope_row_pos(r, *r.pos, T, off, m, e, rot);
  if (pos < 0) return;
  const int p = static_cast<int>(i - (int64_t)m * heads * half), h = p / half;
  int lo, hi;
  rope_cols(r.head_dim, rope_rotary_dim(r), p - h * half, lo, hi);
  lo += h * r.head_dim;
  hi += h * r.head_dim;
  const __half* row = qkv + m * ldqkv;
  rope_pair(r, pos, rot, m, e, lo, hi, row[lo], row[hi]);
}

// one CTA per (token row, head), one thread per pair (a strided loop past 256 pairs); rope.cuh has the arithmetic and
// the summation order of the head's sum of squares (set partials into shared memory, then summed in set order).  T and
// off as rope_kv_kernel
__global__ void __launch_bounds__(256)
    qk_norm_rope_kv_kernel(const __half* __restrict__ qkv, int64_t ldqkv, b200awq_qk_norm_rope_t q, float inv_d,
                           int M, int T, const int32_t* __restrict__ off) {
  extern __shared__ float qk_part[];   // [D / 16] set partials of this head
  pdl_trigger();
  pdl_wait();
  const b200awq_rope_t& r = q.rope;
  const int D = r.head_dim, half = D >> 1, heads = r.n_heads + 2 * r.n_kv_heads;
  const int m = static_cast<int>(blockIdx.x / heads), h = static_cast<int>(blockIdx.x - (unsigned)m * heads);
  if (m >= M) return;
  int e, rot;
  const int pos = rope_row_pos(r, *r.pos, T, off, m, e, rot);
  if (pos < 0) return;
  const __half* row = qkv + (int64_t)m * ldqkv + (int64_t)h * D;
  const int c0 = h * D;
  if (h >= r.n_heads + r.n_kv_heads) {   // v head: not normalised
    for (int p = threadIdx.x; p < half; p += blockDim.x)
      rope_pair(r, pos, rot, m, e, c0 + p, c0 + p + half, row[p], row[p + half]);
    return;
  }
  for (int p = threadIdx.x; p < half; p += blockDim.x) {   // blockDim % 8 == 0: a set's 8 lanes run together
    const float s = qk_set_partial(row[p], row[p + half]);
    if ((p & 7) == 0) qk_part[p >> 3] = s;
  }
  __syncthreads();
  const float ss = qk_head_sum(D >> 4, [&](int t) { return qk_part[t]; });
  for (int p = threadIdx.x; p < half; p += blockDim.x)
    qk_norm_rope_pair(q, inv_d, pos, rot, m, e, c0 + p, row[p], row[p + half], ss);
}

int qk_norm_validate(const b200awq_qk_norm_rope_t* q, int64_t ldqkv) {
  if (q == nullptr) return B200AWQ_EINVAL;
  const int v = rope_validate(&q->rope, ldqkv);
  if (v != B200AWQ_OK) return v;
  if (q->q_norm_weight == nullptr || q->k_norm_weight == nullptr) return B200AWQ_EINVAL;
  return B200AWQ_OK;
}

cudaError_t qk_norm_rope_kv(const void* qkv, int64_t ldqkv, const b200awq_qk_norm_rope_t& q, int M, int T,
                            const int32_t* off, cudaStream_t st) {
  const int half = q.rope.head_dim / 2, heads = q.rope.n_heads + 2 * q.rope.n_kv_heads;
  const int threads = half < 256 ? half : 256;
  return launch_kernel(qk_norm_rope_kv_kernel, dim3(static_cast<unsigned>((int64_t)M * heads)), dim3(threads),
                       (size_t)(q.rope.head_dim / 16) * sizeof(float), st, reinterpret_cast<const __half*>(qkv), ldqkv, q,
                       1.f / static_cast<float>(q.rope.head_dim), M, T, off);
}

int rope_validate(const b200awq_rope_t* r, int64_t ldqkv) {
  if (r == nullptr || r->pos == nullptr || r->freqs == nullptr || r->q_out == nullptr || r->k_cache == nullptr ||
      r->v_cache == nullptr)
    return B200AWQ_EINVAL;
  if (r->n_heads <= 0 || r->n_kv_heads <= 0 || r->head_dim <= 0 || (r->head_dim % 2) != 0 || r->cache_len <= 0 ||
      r->rotary_dim < 0 || (r->rotary_dim % 2) != 0 || r->rotary_dim > r->head_dim || r->freqs_len <= 0 ||
      r->cache_batch_stride < (int64_t)r->cache_len * r->n_kv_heads * r->head_dim ||
      ldqkv < (int64_t)(r->n_heads + 2 * r->n_kv_heads) * r->head_dim)
    return B200AWQ_EINVAL;
  return B200AWQ_OK;
}

cudaError_t rope_kv(const void* qkv, int64_t ldqkv, const b200awq_rope_t& r, int M, int T, const int32_t* off,
                    cudaStream_t st) {
  const int64_t n = (int64_t)M * (r.n_heads + 2 * r.n_kv_heads) * (r.head_dim / 2);
  return launch_kernel(rope_kv_kernel, dim3(static_cast<unsigned>((n + 255) / 256)), dim3(256), 0, st,
                       reinterpret_cast<const __half*>(qkv), ldqkv, r, M, T, off);
}

// one thread per (token row, column pair) of the q_proj | kv_a_proj_with_mqa row; rope.cuh has the arithmetic
__global__ void __launch_bounds__(256)
    mla_rope_kernel(const __half* __restrict__ row, int64_t ld, b200awq_mla_t d, int M) {
  pdl_trigger();
  pdl_wait();
  const int pos = mla_pos(d, true);
  const int pairs = (d.n_heads * (d.nope_dim + d.rope_dim) + d.kv_lora_rank + d.rope_dim) >> 1;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (pos < 0 || i >= (int64_t)M * pairs) return;
  const int m = static_cast<int>(i / pairs), c = 2 * static_cast<int>(i - (int64_t)m * pairs);
  const __half* r = row + m * ld;
  mla_rope_pair(d, pos, m, c, r[c], r[c + 1]);
}

// one thread per (token row, column) of the kv_b_proj row
__global__ void __launch_bounds__(256)
    mla_kv_kernel(const __half* __restrict__ row, int64_t ld, b200awq_mla_t d, int M) {
  pdl_trigger();
  pdl_wait();
  const int pos = mla_pos(d, false);
  const int n = d.n_heads * (d.nope_dim + d.v_dim);
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (pos < 0 || i >= (int64_t)M * n) return;
  const int m = static_cast<int>(i / n), c = static_cast<int>(i - (int64_t)m * n);
  mla_kv_col(d, pos, m, c, row[m * ld + c]);
}

// one thread per (token row, k_pe pair); kpe points at k_pe of token row 0
__global__ void __launch_bounds__(256)
    mla_k_rope_kernel(const __half* __restrict__ kpe, int64_t ld, b200awq_mla_t d, int M) {
  pdl_trigger();
  pdl_wait();
  const int pos = mla_pos(d, true);
  const int pairs = d.rope_dim >> 1;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (pos < 0 || i >= (int64_t)M * pairs) return;
  const int m = static_cast<int>(i / pairs), c = 2 * static_cast<int>(i - (int64_t)m * pairs);
  const __half* r = kpe + m * ld;
  mla_k_pair(d, pos, m, c, r[c], r[c + 1]);
}

// one thread per (token row, column pair) of the q_b_proj row
__global__ void __launch_bounds__(256)
    mla_q_rope_kernel(const __half* __restrict__ row, int64_t ld, b200awq_mla_t d, int M) {
  pdl_trigger();
  pdl_wait();
  const int pos = mla_pos(d, true);
  const int pairs = (d.n_heads * (d.nope_dim + d.rope_dim)) >> 1;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (pos < 0 || i >= (int64_t)M * pairs) return;
  const int m = static_cast<int>(i / pairs), c = 2 * static_cast<int>(i - (int64_t)m * pairs);
  const __half* r = row + m * ld;
  mla_q_pair(d, pos, m, c, r[c], r[c + 1]);
}

// kind: the op (B200AWQ_OP_MLA_*).  Every op reads pos and the head geometry and bounds the position by cache_len; the
// rotations (MLA_ROPE, MLA_K_ROPE, MLA_Q_ROPE) read freqs and style; MLA_ROPE and MLA_Q_ROPE write q_out; MLA_ROPE,
// MLA_K_ROPE and MLA_KV write k_cache (with its geometry); MLA_ROPE and MLA_K_ROPE read C (the row's width), MLA_KV
// v_cache and its geometry
int mla_validate(const b200awq_mla_t* d, int kind) {
  const bool rot = kind != B200AWQ_OP_MLA_KV, q = kind == B200AWQ_OP_MLA_ROPE || kind == B200AWQ_OP_MLA_Q_ROPE;
  const bool k = kind != B200AWQ_OP_MLA_Q_ROPE;
  if (d == nullptr || d->pos == nullptr || (k && d->k_cache == nullptr)) return B200AWQ_EINVAL;
  if (d->n_heads <= 0 || d->nope_dim <= 0 || d->rope_dim <= 0 || (d->rope_dim % 2) != 0 || d->cache_len <= 0 ||
      (k && d->k_batch_stride < (int64_t)d->cache_len * d->n_heads * (d->nope_dim + d->rope_dim)))
    return B200AWQ_EINVAL;
  if (rot)
    return (q && d->q_out == nullptr) || d->freqs == nullptr || (k && d->kv_lora_rank <= 0) ||
                   (d->style != 0 && d->style != 1) || d->freqs_len <= 0
               ? B200AWQ_EINVAL
               : B200AWQ_OK;
  return d->v_cache == nullptr || d->v_dim <= 0 || d->v_head_stride < d->v_dim ||
                 d->v_batch_stride < (int64_t)d->cache_len * d->n_heads * d->v_head_stride
             ? B200AWQ_EINVAL
             : B200AWQ_OK;
}

cudaError_t mla_rope(const void* row, int64_t ld, const b200awq_mla_t& d, int M, cudaStream_t st) {
  const int64_t n = (int64_t)M * ((d.n_heads * (d.nope_dim + d.rope_dim) + d.kv_lora_rank + d.rope_dim) / 2);
  return launch_kernel(mla_rope_kernel, dim3(static_cast<unsigned>((n + 255) / 256)), dim3(256), 0, st,
                       reinterpret_cast<const __half*>(row), ld, d, M);
}

cudaError_t mla_kv(const void* row, int64_t ld, const b200awq_mla_t& d, int M, cudaStream_t st) {
  const int64_t n = (int64_t)M * d.n_heads * (d.nope_dim + d.v_dim);
  return launch_kernel(mla_kv_kernel, dim3(static_cast<unsigned>((n + 255) / 256)), dim3(256), 0, st,
                       reinterpret_cast<const __half*>(row), ld, d, M);
}

cudaError_t mla_k_rope(const void* row, int64_t ld, int64_t k_pe_col, const b200awq_mla_t& d, int M, cudaStream_t st) {
  const int64_t n = (int64_t)M * (d.rope_dim / 2);
  return launch_kernel(mla_k_rope_kernel, dim3(static_cast<unsigned>((n + 255) / 256)), dim3(256), 0, st,
                       reinterpret_cast<const __half*>(row) + k_pe_col, ld, d, M);
}

cudaError_t mla_q_rope(const void* row, int64_t ld, const b200awq_mla_t& d, int M, cudaStream_t st) {
  const int64_t n = (int64_t)M * ((d.n_heads * (d.nope_dim + d.rope_dim)) / 2);
  return launch_kernel(mla_q_rope_kernel, dim3(static_cast<unsigned>((n + 255) / 256)), dim3(256), 0, st,
                       reinterpret_cast<const __half*>(row), ld, d, M);
}

// one CTA of 256 threads per row; thread t takes the chunks of 8 columns at 8 t + 2048 p (the order b200awq.h states,
// which the decode program's LayerNorm staging reproduces: layernorm.cuh has the arithmetic)
__global__ void __launch_bounds__(256)
    layer_norm_kernel(const __half* __restrict__ x, int64_t ldx, const __half* __restrict__ w,
                      const __half* __restrict__ b, __half* __restrict__ out, int K, float eps) {
  __shared__ float wsum[2][8];
  pdl_trigger();
  pdl_wait();
  const __half* xr = x + (int64_t)blockIdx.x * ldx;
  __half* orow = out + (int64_t)blockIdx.x * K;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float s = 0.f;
  for (int c = threadIdx.x * 8; c < K; c += 2048) {
    const uint4 v = *reinterpret_cast<const uint4*>(xr + c);
#pragma unroll
    for (int q = 0; q < 4; ++q) s = ln_sum_pair(s, u32_as_h2((&v.x)[q]));
  }
  s = warp_sum(s);
  if (lane == 0) wsum[0][warp] = s;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) tot = __fadd_rn(tot, wsum[0][i]);
  const float mean = ln_mean(tot, K);
  s = 0.f;
  for (int c = threadIdx.x * 8; c < K; c += 2048) {
    const uint4 v = *reinterpret_cast<const uint4*>(xr + c);
#pragma unroll
    for (int q = 0; q < 4; ++q) s = ln_sq_pair(s, u32_as_h2((&v.x)[q]), mean);
  }
  s = warp_sum(s);
  if (lane == 0) wsum[1][warp] = s;
  __syncthreads();
  tot = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) tot = __fadd_rn(tot, wsum[1][i]);
  const float r = ln_rstd(tot, K, eps);
  for (int c = threadIdx.x * 8; c < K; c += 2048) {
    const uint4 v = *reinterpret_cast<const uint4*>(xr + c);
    const uint4 wv = __ldg(reinterpret_cast<const uint4*>(w + c));
    uint4 bv = make_uint4(0u, 0u, 0u, 0u);
    if (b != nullptr) bv = __ldg(reinterpret_cast<const uint4*>(b + c));
    uint4 o;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float2 a = __half22float2(u32_as_h2((&v.x)[q])), wq = __half22float2(u32_as_h2((&wv.x)[q]));
      const float2 bq = __half22float2(u32_as_h2((&bv.x)[q]));
      (&o.x)[q] = h2_as_u32(__halves2half2(ln_apply(a.x, mean, r, wq.x, bq.x, b != nullptr),
                                           ln_apply(a.y, mean, r, wq.y, bq.y, b != nullptr)));
    }
    *reinterpret_cast<uint4*>(orow + c) = o;
  }
}

// one thread per element; kind 1 = exact, 2 = tanh (layernorm.cuh)
__global__ void __launch_bounds__(256) gelu_kernel(const __half* __restrict__ x, __half* __restrict__ out, int64_t n,
                                                   int kind) {
  pdl_trigger();
  pdl_wait();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = gelu_h(x[i], kind);
}

cudaError_t layer_norm(const void* x, int64_t ldx, const void* w, const void* b, void* out, int rows, int hidden,
                       float eps, cudaStream_t st) {
  return launch_kernel(layer_norm_kernel, dim3(rows), dim3(256), 0, st, reinterpret_cast<const __half*>(x), ldx,
                       reinterpret_cast<const __half*>(w), reinterpret_cast<const __half*>(b),
                       reinterpret_cast<__half*>(out), hidden, eps);
}
cudaError_t gelu(const void* x, void* out, int64_t n, int approximate, cudaStream_t st) {
  return launch_kernel(gelu_kernel, dim3(static_cast<unsigned>((n + 255) / 256)), dim3(256), 0, st,
                       reinterpret_cast<const __half*>(x), reinterpret_cast<__half*>(out), n, approximate ? 2 : 1);
}

cudaError_t rmsnorm(const void* x, const void* w, void* out, int rows, int hidden, float eps, cudaStream_t st) {
  return launch_kernel(rmsnorm_kernel, dim3(rows), dim3(256), 0, st, reinterpret_cast<const __half*>(x),
                       reinterpret_cast<const __half*>(w), reinterpret_cast<__half*>(out), hidden, eps);
}
cudaError_t silu_and_mul(const void* gate_up, void* out, int rows, int d, cudaStream_t st) {
  const int64_t n = (int64_t)rows * d;
  return launch_kernel(silu_mul_kernel, dim3(static_cast<unsigned>((n + 255) / 256)), dim3(256), 0, st,
                       reinterpret_cast<const __half*>(gate_up), reinterpret_cast<__half*>(out), rows, d);
}

}  // namespace b200awq
