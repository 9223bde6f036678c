// Decode program, batched stream variant: the stream kernel of program_stream.cuh for a decode step of M = 2 .. 8
// tokens (a fused block recorded with batch size M: every op has M rows).
//
// Why: the unit of work is an mma.m16n8k16 whose B operand has 8 token columns, and the M = 1 kernel uses column 0
// only.  The weight stream, which sets the step time, is the same for any M <= 8: extra tokens cost staging (M source
// rows instead of one), fold work (each lane folds the two token columns it already holds) and stores - no weight
// bytes.  Everything else is the M = 1 protocol: the stream format and its re-layout, the producer warp and its 1-D
// bulk-copy ring across op boundaries, the output-stationary CTA partition, the tagged (fp16 | tag) hand-off words
// polled with ld.relaxed.gpu (M rows per op, one tag per (run, op)), the ProgWatch watchdog and its abort record.
//
// Bit identity with M = 1: the kernel keeps the cut of stream_program_kernel<8, 4> - 8 consumer warps, the same
// unit-to-warp split, units folded and summed in the same order, the warps' partial sums reduced in the same fixed
// order - and an MMA column does not depend on the other columns.  The RMSNorm of every row follows aux.cu's
// rmsnorm_kernel (thread -> k mapping and summation order).  So token m of a batched run is bit-identical to an M = 1
// stream program run on row m alone.
//
// Shared memory: ring (8 warps x spw stages) + partial sums [sets per CTA][8 warps][MT][16] + unit sums [K / UK][MT] +
// activations [K / 16][MT][8 words] (token stride MT, a compile-time constant: the unit loop's addressing folds).  The
// host picks the deepest ring (<= 4 stages per warp) that fits 227 KB.
//
// Included by program.cu after program_stream.cuh (one translation unit: shares the watchdog / debug symbols).
#pragma once

namespace b200awq {

constexpr int kSbWarps = 8;   // consumer warps (the cut of stream_program_kernel<8, 4>)
constexpr int kSbGR = 4;      // units in flight per warp
constexpr int kSbMaxStages = 4;
// the kernel instance (MT) that runs M >= 2 tokens (M = 1 is stream_program_kernel: sizes with one row, not sb_mt(1))
__host__ __device__ constexpr int sb_mt(int M) { return M <= 2 ? 2 : (M <= 4 ? 4 : 8); }

// bytes of shared memory in front of the activations; every part is a multiple of 16 bytes
__host__ __device__ constexpr size_t sb_part_bytes(int lmax, int M) { return (size_t)lmax * kSbWarps * M * 16 * 4; }
__host__ __device__ constexpr size_t sb_xsum_bytes(int nu_max, int M) { return ((size_t)nu_max * M * 4 + 15) & ~(size_t)15; }
__host__ __device__ constexpr size_t sb_fixed_smem(int spw, int lmax, int M, int nu_max) {
  return (size_t)kSbWarps * spw * kSpStageBytes + sb_part_bytes(lmax, M) + sb_xsum_bytes(nu_max, M) +
         (size_t)2 * kSbWarps * spw * 8 + 2 * 128 + 512;
}

// One unit times the activations of the tokens this lane's accumulators hold: columns n = 2 tig (d0 / d2) and
// n = 2 tig + 1 (d1 / d3).  Arithmetic of sp_units, per token: t[i][0] = (lo, hi) of token 2 tig, t[i][1] of 2 tig + 1.
template <int F, int NUQ, int MT>
__device__ __forceinline__ void sb_units(const uint8_t* __restrict__ st, int UB, const uint32_t* __restrict__ xs,
                                         const float* __restrict__ xsum, const int (&ju)[NUQ], int lane, int M,
                                         float (&tlo)[NUQ][2], float (&thi)[NUQ][2]) {
  constexpr uint32_t MA = 0x000f000fu, MB = 0x00f000f0u, MG = 0x64006400u;
  const int g = lane >> 2, tig = lane & 3;
  const bool xl = g < M;                       // lane group g supplies token g (column n = g of the B operand)
  uint32_t wq[NUQ][F];
#pragma unroll
  for (int i = 0; i < NUQ; ++i) {
    const uint8_t* up = st + (size_t)i * UB;
    if constexpr (F >= 4) {
#pragma unroll
      for (int qd = 0; qd < F / 4; ++qd) {
        const uint4 q = *reinterpret_cast<const uint4*>(up + qd * 512 + lane * 16);
        wq[i][qd * 4 + 0] = q.x;
        wq[i][qd * 4 + 1] = q.y;
        wq[i][qd * 4 + 2] = q.z;
        wq[i][qd * 4 + 3] = q.w;
      }
    } else {
      const uint2 q = *reinterpret_cast<const uint2*>(up + lane * 8);
      wq[i][0] = q.x;
      wq[i][1] = q.y;
    }
  }
  float acc[NUQ][2][4];
#pragma unroll
  for (int i = 0; i < NUQ; ++i)
#pragma unroll
    for (int c = 0; c < 2; ++c) acc[i][c][0] = acc[i][c][1] = acc[i][c][2] = acc[i][c][3] = 0.f;
#pragma unroll
  for (int f = 0; f < F; ++f) {
#pragma unroll
    for (int i = 0; i < NUQ; ++i) {
      uint2 xb = make_uint2(0u, 0u);
      if (xl) xb = *reinterpret_cast<const uint2*>(xs + (((size_t)ju[i] * F + f) * MT + g) * 8 + tig * 2);
      const uint32_t w = wq[i][f], w8 = w >> 8;
      mma_16816(acc[i][f & 1], lop3_and_or(w, MA, MG), lop3_and_or(w, MB, MG), lop3_and_or(w8, MA, MG),
                lop3_and_or(w8, MB, MG), xb.x, xb.y);
    }
  }
  const int m0 = 2 * tig, m1 = 2 * tig + 1;
#pragma unroll
  for (int i = 0; i < NUQ; ++i) {
    const uint8_t* ax = st + (size_t)i * UB + F * 128;
    const float2 sc = __half22float2(u32_as_h2(*reinterpret_cast<const uint32_t*>(ax + 4 * g)));
    const uint32_t zb = ax[32 + g];
    // (branch-free: a lane whose tokens are >= MT reads a valid slot and its results are never stored)
    const float X0 = xsum[ju[i] * MT + (m0 & (MT - 1))];
    const float X1 = xsum[ju[i] * MT + (m1 & (MT - 1))];
    const float s_lo0 = acc[i][0][0] + acc[i][1][0], s_hi0 = acc[i][0][2] + acc[i][1][2];
    const float s_lo1 = acc[i][0][1] + acc[i][1][1], s_hi1 = acc[i][0][3] + acc[i][1][3];
    tlo[i][0] = sc.x * (s_lo0 - (1024.f + static_cast<float>(zb & 0xFu)) * X0);
    thi[i][0] = (sc.y * 0.0625f) * (s_hi0 - (1024.f + 16.f * static_cast<float>(zb >> 4)) * X0);
    tlo[i][1] = sc.x * (s_lo1 - (1024.f + static_cast<float>(zb & 0xFu)) * X1);
    thi[i][1] = (sc.y * 0.0625f) * (s_hi1 - (1024.f + 16.f * static_cast<float>(zb >> 4)) * X1);
  }
}

// sp_chunk for the batched unit: apply(t_lo[2], t_hi[2]) once per unit, in unit order
template <int F, int GR, int MT, typename Apply>
__device__ __forceinline__ void sb_chunk(const uint8_t* __restrict__ st, int UB, int n, const uint32_t* __restrict__ xs,
                                         const float* __restrict__ xsum, int j, int NU, int lane, int M, Apply&& apply) {
  int i = 0;
  for (; i + GR <= n; i += GR) {
    int ju[GR];
#pragma unroll
    for (int q = 0; q < GR; ++q) {
      ju[q] = j + i + q;
      if (ju[q] >= NU) ju[q] -= NU;
    }
    float a[GR][2], b[GR][2];
    sb_units<F, GR, MT>(st + (size_t)i * UB, UB, xs, xsum, ju, lane, M, a, b);
#pragma unroll
    for (int q = 0; q < GR; ++q) apply(a[q], b[q]);
  }
  for (; i < n; ++i) {
    int ju[1] = {j + i >= NU ? j + i - NU : j + i};
    float a[1][2], b[1][2];
    sb_units<F, 1, MT>(st + (size_t)i * UB, UB, xs, xsum, ju, lane, M, a, b);
    apply(a[0], b[0]);
  }
}

// MT in {2, 4, 8}: the token stride of the shared-memory arrays; the host launches sb_mt(M).  Lanes whose token
// column is >= M feed zeros and nothing is stored for them.  spw = ring stages per consumer warp, lmax = 16-column
// sets one CTA may own in one op, nu_max = units along K of the longest op (shared-memory sizes chosen by the host).
template <int MT>
__global__ void __launch_bounds__(32 + kSbWarps * 32, 1)
    stream_batch_kernel(const SpOp* __restrict__ ops, const uint32_t* __restrict__ cta_all, int n_ops,
                        uint32_t* __restrict__ rows, int row_stride, int* __restrict__ state, int M, int spw, int lmax,
                        int nu_max, int dbg) {
  // a cooperative launch never carries the PDL attribute (then this is a no-op); the tag state the body reads first is
  // written by the previous run of this program
  pdl_wait();
#include "program_batch_body.inc"
}

// batched programs with residual adds (SpRes, program_stream.cuh): the same body plus the residual steps of the finish
template <int MT>
__global__ void __launch_bounds__(32 + kSbWarps * 32, 1)
    stream_batch_residual_kernel(const SpOp* __restrict__ ops, const uint32_t* __restrict__ cta_all, int n_ops,
                                 uint32_t* __restrict__ rows, int row_stride, int* __restrict__ state, int M, int spw,
                                 int lmax, int nu_max, int dbg, const SpRes* __restrict__ res) {
  // a cooperative launch never carries the PDL attribute (then this is a no-op); the tag state the body reads first is
  // written by the previous run of this program
  pdl_wait();
#define SP_RESIDUAL 1
#include "program_batch_body.inc"
#undef SP_RESIDUAL
}

// batched programs with a ROPE_KV or ROPE_KV_SEQ op (SpRopeSeq, program_stream.cuh): the residual kernel plus RoPE +
// cache append in a mode-2 finish (token row m = b T + t writes cache entry b at position *pos + t; T = 1: entry m)
template <int MT>
__global__ void __launch_bounds__(32 + kSbWarps * 32, 1)
    stream_batch_rope_kernel(const SpOp* __restrict__ ops, const uint32_t* __restrict__ cta_all, int n_ops,
                             uint32_t* __restrict__ rows, int row_stride, int* __restrict__ state, int M, int spw,
                             int lmax, int nu_max, int dbg, const SpRes* __restrict__ res,
                             const SpRopeSeq* __restrict__ rope) {
  pdl_wait();
#define SP_RESIDUAL 1
#define SP_ROPE 1
#include "program_batch_body.inc"
#undef SP_ROPE
#undef SP_RESIDUAL
}

// batched programs with a QK_NORM_ROPE_KV op (SpQkNorm, program_stream.cuh): the rope kernel plus the two-phase q / k
// norm of the mode-2 finish (token row m publishes and polls its own partials)
template <int MT>
__global__ void __launch_bounds__(32 + kSbWarps * 32, 1)
    stream_batch_qknorm_kernel(const SpOp* __restrict__ ops, const uint32_t* __restrict__ cta_all, int n_ops,
                               uint32_t* __restrict__ rows, int row_stride, int* __restrict__ state, int M, int spw,
                               int lmax, int nu_max, int dbg, const SpRes* __restrict__ res,
                               const SpRopeSeq* __restrict__ rope, const SpQkNorm* __restrict__ qkn) {
  pdl_wait();
#define SP_RESIDUAL 1
#define SP_ROPE 1
#define SP_QKNORM 1
#include "program_batch_body.inc"
#undef SP_QKNORM
#undef SP_ROPE
#undef SP_RESIDUAL
}

}  // namespace b200awq
