// MoE operators the reference's FusedSparseMoeBlock calls through awq_ext (SURVEY.md 8f #2):
//   topk_softmax          <- awq_ext.topk_softmax          (awq/modules/fused/moe.py:137-171, fused_topk)
//   moe_align_block_size  <- awq_ext.moe_alig_block_size   (moe.py:92-134; the misspelling is the real name)
//   grouped_gemm          <- awq_ext.grouped_gemm_forward  (moe.py:60-89): W4A16 GEMM over stacked expert weights
//                            qweight [E, K, N/8] (awq/models/mixtral.py:129-158), rows gathered / scattered through
//                            the sorted slot list, optional multiplication by the routing weight.
// The reference's kernels for these live in the un-vendored autoawq-kernels package (vLLM lineage); the contract
// implemented here is the one its call sites and docstrings define (the test oracle restates it).
//
// grouped_gemm, decode-sized and fallback kernel (bs = 1: two slots, two experts).  Eight sorted slots
// (half a 16-slot block: one expert) ride through mma.sync.m16n8k16 as the n = 8 dimension, exactly like the M <= 8
// GEMV (gemv.cu): one CTA = 256 output columns x 8 slots, streaming the expert's K rows in chunks of 512 with
// register-staged 128-bit loads.  HBM-bound at decode (each active expert's weights are read once per half-block).
// Prefill-sized token counts run the grouped wgmma kernel instead (moe_tc_kernel, gemm_tc.cu), which reads an expert's
// weights once per 32 - 128 slots.
#include "common.cuh"
#include "gemv_tile.cuh"
#include "kernels.h"

namespace b200awq {

// ------------------------------------------------------------------------------------------- topk_softmax
// one warp per token
__global__ void __launch_bounds__(128)
    topk_softmax_kernel(const float* __restrict__ gating, float* __restrict__ topk_w, int* __restrict__ topk_ids,
                        int* __restrict__ src_rows, int M, int E, int topk) {
  extern __shared__ float ts_smem[];   // [4 warps][E]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m = blockIdx.x * 4 + warp;
  pdl_wait();      // the gating logits come from the predecessor kernel (PDL launches may start early)
  pdl_trigger();
  if (m >= M) return;
  float* p = ts_smem + (size_t)warp * E;
  const float* g = gating + (int64_t)m * E;
  float mx = -INFINITY;
  for (int e = lane; e < E; e += 32) mx = fmaxf(mx, g[e]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
  for (int e = lane; e < E; e += 32) {
    const float v = expf(g[e] - mx);
    p[e] = v;
    sum += v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float inv = 1.f / sum;
  __syncwarp();
  for (int k = 0; k < topk; ++k) {
    float best = -1.f;
    int bi = 0x7fffffff;
    for (int e = lane; e < E; e += 32) {
      const float v = p[e];
      if (v > best) {   // strided ascending scan: the first maximum a lane meets is its lowest index
        best = v;
        bi = e;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > best || (ov == best && oi < bi)) {
        best = ov;
        bi = oi;
      }
    }
    if (lane == 0) {
      topk_w[(int64_t)m * topk + k] = best * inv;
      topk_ids[(int64_t)m * topk + k] = bi;
      src_rows[(int64_t)m * topk + k] = k * M + m;
      if (bi < E) p[bi] = -2.f;   // taken (a row of NaNs selects nothing: bi stays at its sentinel)
    }
    __syncwarp();
  }
}

cudaError_t topk_softmax(const float* gating, float* topk_w, int* topk_ids, int* src_rows, int M, int E, int topk,
                         cudaStream_t st) {
  if (M == 0) return cudaSuccess;
  const size_t smem = (size_t)4 * E * sizeof(float);
  if (smem > (size_t)200 * 1024) return cudaErrorNotSupported;
  if (smem > (size_t)48 * 1024) {   // beyond the default dynamic shared memory limit (E > 3072)
    cudaError_t e = cudaFuncSetAttribute(topk_softmax_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  return launch_kernel(topk_softmax_kernel, dim3((M + 3) / 4), dim3(128), smem, st, gating, topk_w, topk_ids, src_rows,
                       M, E, topk);
}

// ------------------------------------------------------------------------------------ moe_align_block_size
// One CTA; thread e owns expert e: counts its slots, the padded runs are laid out in expert order, then the thread
// writes its slots in ascending order (the order the reference's docstring example shows) and pads with `numel`.
__global__ void __launch_bounds__(1024)
    moe_align_kernel(const int* __restrict__ topk_ids, int numel, int num_experts, int block_size,
                     int* __restrict__ sorted_ids, int* __restrict__ expert_ids, int* __restrict__ num_post_pad) {
  extern __shared__ int ma_smem[];   // [E] padded counts -> run offsets
  const int e = threadIdx.x;
  pdl_wait();      // topk_ids are written by the predecessor (topk_softmax)
  pdl_trigger();
  int cnt = 0;
  if (e < num_experts)
    for (int i = 0; i < numel; ++i) cnt += (topk_ids[i] == e);
  const int padded = (cnt + block_size - 1) / block_size * block_size;
  if (e < num_experts) ma_smem[e] = padded;
  __syncthreads();
  if (e >= num_experts) return;
  int off = 0;
  for (int j = 0; j < e; ++j) off += ma_smem[j];
  if (e == num_experts - 1) *num_post_pad = off + padded;
  int pos = off;
  for (int i = 0; i < numel; ++i)
    if (topk_ids[i] == e) sorted_ids[pos++] = i;
  for (; pos < off + padded; ++pos) sorted_ids[pos] = numel;
  for (int b = 0; b < padded / block_size; ++b) expert_ids[off / block_size + b] = e;
}

cudaError_t moe_align_block_size(const int* topk_ids, int numel, int num_experts, int block_size, int* sorted_ids,
                                 int* expert_ids, int* num_post_pad, cudaStream_t st) {
  if (num_experts > 1024) return cudaErrorNotSupported;
  const int threads = ((num_experts + 31) / 32) * 32;
  return launch_kernel(moe_align_kernel, dim3(1), dim3(threads), (size_t)num_experts * sizeof(int), st, topk_ids, numel,
                       num_experts, block_size, sorted_ids, expert_ids, num_post_pad);
}

// ------------------------------------------------------------------------------------------- grouped GEMM
constexpr int kMoeRW = 64;                       // rows per warp and chunk (divides every AWQ group size >= 64)
constexpr int kMoeKC = kGvWarps * kMoeRW;        // 512 rows per chunk
constexpr int kMoeMT = 8;                        // slots per CTA (half a 16-slot block)

__global__ void __launch_bounds__(kGvWarps * 32, 2)
    moe_grouped_kernel(const __half* __restrict__ x, int x_per_slot, const int32_t* __restrict__ qweight,
                       const __half* __restrict__ scales, const int32_t* __restrict__ qzeros,
                       const float* __restrict__ topk_w, const int* __restrict__ sorted_ids,
                       const int* __restrict__ expert_ids, const int* __restrict__ num_post_pad, __half* __restrict__ y,
                       int n_slots, int topk, int K, int N, int G, int mul_weights, int block_size) {
  constexpr int MT = kMoeMT, RW = kMoeRW, NB = RW / 16;
  extern __shared__ __align__(16) float moe_dyn[];
  float (*red)[MT][kGvRedStride] = reinterpret_cast<float (*)[MT][kGvRedStride]>(moe_dyn);
  float (*xsum_s)[MT] = reinterpret_cast<float (*)[MT]>(moe_dyn + kGvWarps * MT * kGvRedStride);
  int* s_id = reinterpret_cast<int*>(moe_dyn + kGvWarps * MT * kGvRedStride + kGvWarps * MT);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, tig = lane & 3;
  const int hb = blockIdx.y;                       // half-block: sorted slots hb*8 .. hb*8+7
  pdl_wait();      // routing data and activations come from predecessor kernels; nothing is read before this
  pdl_trigger();
  if (hb * MT >= *num_post_pad) return;
  if (tid < MT) {
    const int id = sorted_ids[hb * MT + tid];
    s_id[tid] = id < n_slots ? id : -1;
  }
  __syncthreads();
  bool any = false;
#pragma unroll
  for (int m = 0; m < MT; ++m) any = any || s_id[m] >= 0;
  if (!any) return;                                // pure padding
  const int e = expert_ids[(hb * MT) / block_size];
  const int NW = N >> 3;
  const int32_t* qw = qweight + (int64_t)e * K * NW;
  const __half* sc = scales + (int64_t)e * (K / G) * N;
  const int32_t* qz = qzeros + (int64_t)e * (K / G) * NW;

  const int n_base = blockIdx.x * kGvTN;
  const int wc = (n_base >> 3) + 4 * g;
  const bool col_ok = wc < NW;
  const int my_id = s_id[g];
  const bool tok_ok = my_id >= 0;
  const __half* xrow = x + (int64_t)(tok_ok ? (x_per_slot ? my_id : my_id / topk) : 0) * K;

  const int c = tid;
  const int n = n_base + c;
  const int j = c & 7;
  const bool kindB = ((j >> 1) & 1) != 0;
  const int zshift = 4 * ((j >> 1) + 4 * (j & 1));
  const int pc = gv_pos(c);
  float val[MT];
#pragma unroll
  for (int m = 0; m < MT; ++m) val[m] = 0.f;

  for (int k0 = 0; k0 < K; k0 += kMoeKC) {
    const int wrow = k0 + warp * RW;
    uint4 q[2][4];
    uint2 xb[2];
    auto issue = [&](int slot, int b) {
      const int kr = wrow + 16 * b + 4 * tig;
      const int32_t* src = qw + (int64_t)kr * NW + wc;
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        q[slot][r] = make_uint4(0, 0, 0, 0);
        if (col_ok) q[slot][r] = ldg_stream_u4(src + (int64_t)r * NW);
      }
      xb[slot] = make_uint2(0, 0);
      if (tok_ok) xb[slot] = *reinterpret_cast<const uint2*>(xrow + kr);
    };
    issue(0, 0);
    issue(1, 1);
    float acc[4][4][4];
    float xs_acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int w = 0; w < 4; ++w)
#pragma unroll
      for (int t = 0; t < 4; ++t)
#pragma unroll
        for (int r = 0; r < 4; ++r) acc[w][t][r] = 0.f;
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      const int sl = b & 1;
      constexpr uint32_t MA = 0x000f000fu, MB = 0x00f000f0u, MG = 0x64006400u, ONES = 0x3C003C00u;
      mma_16816(xs_acc, ONES, ONES, ONES, ONES, xb[sl].x, xb[sl].y);
#pragma unroll
      for (int w = 0; w < 4; ++w) {
        const uint32_t wa = (&q[sl][0].x)[w], wb = (&q[sl][1].x)[w], wc_ = (&q[sl][2].x)[w], wd = (&q[sl][3].x)[w];
        const uint32_t lo01 = __byte_perm(wa, wb, 0x5410), hi01 = __byte_perm(wa, wb, 0x7632);
        const uint32_t lo23 = __byte_perm(wc_, wd, 0x5410), hi23 = __byte_perm(wc_, wd, 0x7632);
        const uint32_t lo01s = lo01 >> 8, hi01s = hi01 >> 8, lo23s = lo23 >> 8, hi23s = hi23 >> 8;
        mma_16816(acc[w][0], lop3_and_or(lo01, MA, MG), lop3_and_or(hi01, MA, MG), lop3_and_or(lo23, MA, MG),
                  lop3_and_or(hi23, MA, MG), xb[sl].x, xb[sl].y);
        mma_16816(acc[w][1], lop3_and_or(lo01, MB, MG), lop3_and_or(hi01, MB, MG), lop3_and_or(lo23, MB, MG),
                  lop3_and_or(hi23, MB, MG), xb[sl].x, xb[sl].y);
        mma_16816(acc[w][2], lop3_and_or(lo01s, MA, MG), lop3_and_or(hi01s, MA, MG), lop3_and_or(lo23s, MA, MG),
                  lop3_and_or(hi23s, MA, MG), xb[sl].x, xb[sl].y);
        mma_16816(acc[w][3], lop3_and_or(lo01s, MB, MG), lop3_and_or(hi01s, MB, MG), lop3_and_or(lo23s, MB, MG),
                  lop3_and_or(hi23s, MB, MG), xb[sl].x, xb[sl].y);
      }
      if (b + 2 < NB) issue(sl, b + 2);
    }
    // raw per-warp sums -> shared memory, then thread c folds column n_base + c (as gemv_gemm_layout_kernel)
    __syncthreads();   // the previous chunk's fold is done reading `red`
#pragma unroll
    for (int w = 0; w < 4; ++w)
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const int p2 = gv_pos(32 * g + 8 * w + 2 * t);
        *reinterpret_cast<float2*>(&red[warp][2 * tig][p2]) = make_float2(acc[w][t][0], acc[w][t][2]);
        *reinterpret_cast<float2*>(&red[warp][2 * tig + 1][p2]) = make_float2(acc[w][t][1], acc[w][t][3]);
      }
    if (g == 0) {
      xsum_s[warp][2 * tig] = xs_acc[0];
      xsum_s[warp][2 * tig + 1] = xs_acc[1];
    }
    __syncthreads();
    if (n < N) {
      int w = 0;
#pragma unroll 1
      while (w < kGvWarps) {
        const int krow = k0 + w * RW;
        const int gabs = krow / G;
        float s = __half2float(__ldg(sc + (int64_t)gabs * N + n));
        const float z = static_cast<float>((static_cast<uint32_t>(__ldg(qz + (int64_t)gabs * NW + (n >> 3))) >> zshift) & 0xFu);
        const float zoff = kindB ? 1024.f + 16.f * z : 1024.f + z;
        if (kindB) s *= 0.0625f;
        float S[MT], X[MT];
#pragma unroll
        for (int m = 0; m < MT; ++m) S[m] = X[m] = 0.f;
        const int gend = (gabs + 1) * G;
        for (; w < kGvWarps && k0 + w * RW < gend; ++w) {
#pragma unroll
          for (int m = 0; m < MT; ++m) {
            S[m] += red[w][m][pc];
            X[m] += xsum_s[w][m];
          }
        }
#pragma unroll
        for (int m = 0; m < MT; ++m) val[m] += s * (S[m] - zoff * X[m]);
      }
    }
  }
  if (n < N) {
#pragma unroll
    for (int m = 0; m < MT; ++m) {
      const int id = s_id[m];
      if (id >= 0) {
        const float v = mul_weights ? val[m] * topk_w[id] : val[m];
        y[(int64_t)id * N + n] = __float2half_rn(v);
      }
    }
  }
}

bool moe_grouped_supported(int K, int N, int G) {
  return K > 0 && N > 0 && G > 0 && (K % kMoeKC) == 0 && (N % 32) == 0 && (G % kMoeRW) == 0 && (K % G) == 0;
}

cudaError_t moe_grouped_gemm(const void* x, int x_per_slot, const int32_t* qweight, const void* scales,
                             const int32_t* qzeros, const float* topk_w, const int* sorted_ids, const int* expert_ids,
                             const int* num_post_pad, void* y, int n_slots, int topk, int sorted_len, int K, int N, int G,
                             int mul_weights, int block_size, cudaStream_t st) {
  if (!moe_grouped_supported(K, N, G) || (block_size % kMoeMT) != 0) return cudaErrorNotSupported;
  const int hbs = sorted_len / kMoeMT;
  if (hbs == 0 || n_slots == 0) return cudaSuccess;
  if (hbs > 65535) return cudaErrorNotSupported;
  constexpr size_t smem = (size_t)(kGvWarps * kMoeMT * kGvRedStride + kGvWarps * kMoeMT + kMoeMT) * sizeof(float);
  cudaError_t e = cudaFuncSetAttribute(moe_grouped_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  return launch_kernel(moe_grouped_kernel, dim3((N + kGvTN - 1) / kGvTN, hbs), dim3(kGvWarps * 32), smem, st,
                       reinterpret_cast<const __half*>(x), x_per_slot, qweight, reinterpret_cast<const __half*>(scales),
                       qzeros, topk_w, sorted_ids, expert_ids, num_post_pad, reinterpret_cast<__half*>(y), n_slots, topk,
                       K, N, G, mul_weights, block_size);
}

}  // namespace b200awq
