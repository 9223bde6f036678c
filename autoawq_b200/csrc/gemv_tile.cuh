// Device-side pieces shared by the persistent TMA-ring GEMV (gemv.cu) and the decode-program kernel
// (program.cu): tile geometry, the mma.sync tile product on raw (1024 + c*q) codes, the per-group fold and the
// split-K push / finalise helpers.  See gemv.cu for the derivation of the fragment construction.
#pragma once
#include "common.cuh"

namespace b200awq {

__device__ __forceinline__ void mma_16816(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                          uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

__device__ __forceinline__ void named_bar_sync_gv(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

constexpr int kGvTN = 256;       // columns per CTA (one warp width)
constexpr int kGvWarps = 8;      // warps per CTA, each on its own contiguous RW rows
constexpr int kGvRedStride = kGvTN + 32;  // +4 floats per 32 columns: conflict-free float2 stores, 16-B aligned octets

__device__ __forceinline__ int gv_pos(int c) { return c + ((c >> 5) << 2); }

constexpr int kV3TileRows = 64;
constexpr int kV3TileCols = 256;
constexpr int kV3TileBytes = kV3TileRows * 128;               // 8 KB of packed weights
constexpr int kV3ScaleBytes = kV3TileCols * 2;                // 512 B
constexpr int kV3ZeroBytes = kV3TileCols / 8 * 4;             // 128 B
constexpr int kV3AuxBytes = kV3ScaleBytes + kV3ZeroBytes;     // 640 B of group constants per stage
constexpr int kV3Warps = 8;                                   // consumer warps
constexpr int kV3Threads = 32 + kV3Warps * 32;                // producer warp + consumers

template <int MT, int SPW>
struct V3Smem {
  // bytes in flight are what buys bandwidth (HBM latency under load is several us): SPW 8 KB stages per
  // consumer warp, as many as the 227 KB of shared memory allow next to the reduction buffers (and, for
  // M <= 2, the staged activations)
  static constexpr int kStagesPerWarp = SPW;
  static constexpr int kStages = kV3Warps * kStagesPerWarp;
  static constexpr int red_floats = kV3Warps * MT * kGvRedStride;    // per-warp raw sums [MT][288]; at the end of a
                                                                     // run the same area carries the warp's column sums
  static constexpr size_t bytes = (size_t)kStages * (kV3TileBytes + kV3AuxBytes) + (size_t)red_floats * 4 +
                                  2 * kStages * 8 + 128;
};

// Shared by the warp-level (NT = 32) and CTA-level (NT = 256) pushes: add `cols` [MT][256] (shared memory,
// summed over `nsrc` sources `src_stride` floats apart) into the fp32 workspace (relaxed REDs).
// Output scatter of the grouped (MoE) variant: token m of the CTA's job goes to row ids[m] of y (ids in shared
// memory, -1 = padding slot), optionally scaled by the routing weight tw[ids[m]].  ids == nullptr: row m, as is.
struct V3Scatter {
  const int* ids = nullptr;
  const float* tw = nullptr;
};
template <int MT, int NT>
__device__ __forceinline__ void v3_add_cols(float* cols, int nsrc, int src_stride, int cb, int t,
                                            float* __restrict__ acc_ws, int M, int N, V3Scatter sc = V3Scatter()) {
  const int n_base = cb * kV3TileCols;
#pragma unroll
  for (int m = 0; m < MT; ++m) {
    if (m < M && (sc.ids == nullptr || sc.ids[m] >= 0)) {   // padding slots carry exact zeros: nothing to add
      for (int c = t; c < kV3TileCols; c += NT) {
        float v = 0.f;
        for (int sidx = 0; sidx < nsrc; ++sidx) {
          v += cols[sidx * src_stride + m * kV3TileCols + c];
          cols[sidx * src_stride + m * kV3TileCols + c] = 0.f;
        }
        red_add_f32(&acc_ws[(int64_t)m * N + n_base + c], v);
      }
    }
  }
}
// The last contributor of column block `cb` rounds to fp16 (+ bias) and restores the zeros.
template <int MT, int NT>
__device__ __forceinline__ void v3_finalize(int cb, int t, const __half* __restrict__ bias, __half* __restrict__ y,
                                            float* __restrict__ acc_ws, int* __restrict__ tickets, int M, int N,
                                            V3Scatter sc = V3Scatter()) {
  const int n_base = cb * kV3TileCols;
#pragma unroll
  for (int m = 0; m < MT; ++m) {
    if (m < M) {
      int row = m;
      float mulw = 1.f;
      if (sc.ids != nullptr) {
        row = sc.ids[m];
        if (row < 0) continue;   // padding slot: nothing was added for it
        if (sc.tw != nullptr) mulw = sc.tw[row];
      }
      for (int c = t; c < kV3TileCols; c += NT) {
        const int n = n_base + c;
        float* p = &acc_ws[(int64_t)m * N + n];
        float v = ld_relaxed_f32(p);
        *p = 0.f;
        if (bias != nullptr) v += __half2float(bias[n]);
        if (sc.ids != nullptr) v *= mulw;
        y[(int64_t)row * N + n] = __float2half_rn(v);
      }
    }
  }
  if (t == 0) tickets[cb] = 0;
}
// ---------------------------------------------------------------------------------- packed split-K epilogue
// One 64-bit word per (token, column) carries the partial sums AND how many tiles have contributed (the decode
// program's hand-off word, csrc/program.cu):  word = tiles << 48 | sum of (round(v * 2^24) + tiles * 2^39).
// Every contributor does ONE atom.add.u64 WITH RETURN: the one whose add completes the tile count holds the complete
// sum (old + own), rounds it to fp16 (+ bias), stores y and writes the zero back.  One L2 round trip instead of three
// (REDs -> ticket -> read back), no tickets, and - integer addition is associative - the result no longer depends on
// the order in which CTAs arrive: the per-op GEMV is bit-reproducible.  Needs K / 64 < 256 tiles per column and
// |partial| < tiles * 32768 (fp16 outputs beyond that are inf anyway); resolution 2^-24 = one fp16 subnormal step.
constexpr float kV3FixScale = 16777216.0f;
__device__ __forceinline__ unsigned long long v3_pack(float v, int ntl) {
  long long f = __float2ll_rn(v * kV3FixScale);
  const long long lim = ((long long)ntl << 39) - 1;
  f = f > lim ? lim : (f < -lim ? -lim : f);
  return ((unsigned long long)ntl << 48) + (unsigned long long)(((long long)ntl << 39) + f);
}
__device__ __forceinline__ unsigned long long atom_add_u64(unsigned long long* p, unsigned long long v) {
  unsigned long long old;
  asm volatile("atom.relaxed.gpu.global.add.u64 %0, [%1], %2;" : "=l"(old) : "l"(p), "l"(v) : "memory");
  return old;
}
template <int MT, int NT>
__device__ __forceinline__ void v3_atom_cols(float* cols, int nsrc, int src_stride, int cb, int ntl, int TPC, int t,
                                             const __half* __restrict__ bias, __half* __restrict__ y,
                                             unsigned long long* __restrict__ ws64, int M, int N,
                                             V3Scatter sc = V3Scatter()) {
  const int n_base = cb * kV3TileCols;
  const long long off = (long long)TPC << 39;
#pragma unroll
  for (int m = 0; m < MT; ++m) {
    if (m < M && (sc.ids == nullptr || sc.ids[m] >= 0)) {
      int row = m;
      float mulw = 1.f;
      if (sc.ids != nullptr) {
        row = sc.ids[m];
        if (sc.tw != nullptr) mulw = sc.tw[row];
      }
      for (int c = t; c < kV3TileCols; c += NT) {
        float v = 0.f;
        for (int sidx = 0; sidx < nsrc; ++sidx) {
          v += cols[sidx * src_stride + m * kV3TileCols + c];
          cols[sidx * src_stride + m * kV3TileCols + c] = 0.f;
        }
        const int n = n_base + c;
        unsigned long long* p = ws64 + (int64_t)m * N + n;
        const unsigned long long mine = v3_pack(v, ntl);
        const unsigned long long old = atom_add_u64(p, mine);
        if ((int)(old >> 48) + ntl == TPC) {           // this add completed the column: finalise it
          const unsigned long long tot = old + mine;
          float r = __ll2float_rn((long long)(tot & 0xFFFFFFFFFFFFull) - off) * (1.0f / kV3FixScale);
          *p = 0ull;                                     // (the next launch touches the workspace after its PDL wait)
          if (bias != nullptr) r += __half2float(bias[n]);
          if (sc.ids != nullptr) r *= mulw;
          y[(int64_t)row * N + n] = __float2half_rn(r);
        }
      }
    }
  }
}

// Warp-level push (a warp's run crossed a column block; rare).
template <int MT>
__device__ __forceinline__ bool v3_push_warp(float* cols, int cb, int ntl, int TPC, int lane,
                                             const __half* __restrict__ bias, __half* __restrict__ y,
                                             float* __restrict__ acc_ws, int* __restrict__ tickets, int M, int N,
                                             V3Scatter sc = V3Scatter()) {
  v3_add_cols<MT, 32>(cols, 1, 0, cb, lane, acc_ws, M, N, sc);
  __syncwarp();
  int last = 0;
  if (lane == 0) last = (atom_add_acq_rel(&tickets[cb], ntl) + ntl == TPC);
  last = __shfl_sync(0xffffffffu, last, 0);
  if (last) v3_finalize<MT, 32>(cb, lane, bias, y, acc_ws, tickets, M, N, sc);
  return last != 0;
}

// One 64-row x 256-column tile (8 KB, 128B-swizzled rows of 32 words) times the activations of <= 8 tokens:
// acc[w][tt] += raw codes of word w / nibble pair tt, xs_acc += sum_k x_k (ones-row MMA).  xcur[bb] = the lane's
// B fragments of k16-block bb.
__device__ __forceinline__ void v3_tile_mma(const uint8_t* st, int g, int tig, const uint32_t (&xcur)[4][2],
                                            float (&acc)[4][4][4], float (&xs_acc)[4]) {
#pragma unroll
  for (int bb = 0; bb < 4; ++bb) {
    // fragments from the swizzled tile: rows (2tig, 2tig+1, 2tig+8, 2tig+9) of block bb, 16-byte chunk g
    const int r0 = 16 * bb + 2 * tig;
    const uint4 qa = *reinterpret_cast<const uint4*>(st + (r0 + 0) * 128 + ((g ^ ((r0 + 0) & 7)) << 4));
    const uint4 qb = *reinterpret_cast<const uint4*>(st + (r0 + 1) * 128 + ((g ^ ((r0 + 1) & 7)) << 4));
    const uint4 qc = *reinterpret_cast<const uint4*>(st + (r0 + 8) * 128 + ((g ^ ((r0 + 8) & 7)) << 4));
    const uint4 qd = *reinterpret_cast<const uint4*>(st + (r0 + 9) * 128 + ((g ^ ((r0 + 9) & 7)) << 4));
    constexpr uint32_t MA = 0x000f000fu, MB = 0x00f000f0u, MG = 0x64006400u, ONES = 0x3C003C00u;
    const uint32_t xb0 = xcur[bb][0], xb1 = xcur[bb][1];
    mma_16816(xs_acc, ONES, ONES, ONES, ONES, xb0, xb1);
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      const uint32_t wa = (&qa.x)[w], wb = (&qb.x)[w], wc_ = (&qc.x)[w], wd = (&qd.x)[w];
      const uint32_t lo01 = __byte_perm(wa, wb, 0x5410), hi01 = __byte_perm(wa, wb, 0x7632);
      const uint32_t lo23 = __byte_perm(wc_, wd, 0x5410), hi23 = __byte_perm(wc_, wd, 0x7632);
      const uint32_t lo01s = lo01 >> 8, hi01s = hi01 >> 8, lo23s = lo23 >> 8, hi23s = hi23 >> 8;
      mma_16816(acc[w][0], lop3_and_or(lo01, MA, MG), lop3_and_or(hi01, MA, MG), lop3_and_or(lo23, MA, MG),
                lop3_and_or(hi23, MA, MG), xb0, xb1);
      mma_16816(acc[w][1], lop3_and_or(lo01, MB, MG), lop3_and_or(hi01, MB, MG), lop3_and_or(lo23, MB, MG),
                lop3_and_or(hi23, MB, MG), xb0, xb1);
      mma_16816(acc[w][2], lop3_and_or(lo01s, MA, MG), lop3_and_or(hi01s, MA, MG), lop3_and_or(lo23s, MA, MG),
                lop3_and_or(hi23s, MA, MG), xb0, xb1);
      mma_16816(acc[w][3], lop3_and_or(lo01s, MB, MG), lop3_and_or(hi01s, MB, MG), lop3_and_or(lo23s, MB, MG),
                lop3_and_or(hi23s, MB, MG), xb0, xb1);
    }
  }
}

// End of a quantisation group (or of the warp's run): raw sums -> per-warp staging, lane l folds word-column l
// (scales: one LDS.128, zeros: one LDS.32 from the stage's group constants `sa`) into the warp's column sums.
template <int MT>
__device__ __forceinline__ void v3_fold(const uint8_t* sa, float* my_red, float* my_col, int lane, int g, int tig,
                                        const float (&acc)[4][4][4], const float (&xs_acc)[4]) {
  // raw sums -> this warp's staging area (conflict-free float2 stores), then lane l folds word-column l
#pragma unroll
  for (int w = 0; w < 4; ++w)
#pragma unroll
    for (int tt = 0; tt < 4; ++tt) {
      const int pc = gv_pos(32 * g + 8 * w + 2 * tt);
      if (2 * tig < MT)
        *reinterpret_cast<float2*>(&my_red[(2 * tig) * kGvRedStride + pc]) = make_float2(acc[w][tt][0], acc[w][tt][2]);
      if (2 * tig + 1 < MT)
        *reinterpret_cast<float2*>(&my_red[(2 * tig + 1) * kGvRedStride + pc]) =
            make_float2(acc[w][tt][1], acc[w][tt][3]);
    }
  // sum_k x_k per token: d0 / d1 of the ones-row MMA live in the tig lanes of every g; take g = 0
  float X[MT];
#pragma unroll
  for (int m = 0; m < MT; ++m) {
    const float v = (m & 1) ? xs_acc[1] : xs_acc[0];
    X[m] = __shfl_sync(0xffffffffu, v, m >> 1);  // lane (g = 0, tig = m / 2)
  }
  __syncwarp();
  {
    const uint4 sc4 = *reinterpret_cast<const uint4*>(sa + lane * 16);            // 8 scales
    const uint32_t zw = *reinterpret_cast<const uint32_t*>(sa + kV3ScaleBytes + lane * 4);
    const __half2* sc2 = reinterpret_cast<const __half2*>(&sc4);
    float sc[8], zoff[8];
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const float2 f = __half22float2(sc2[jj]);
      sc[2 * jj] = f.x;
      sc[2 * jj + 1] = f.y;
    }
#pragma unroll
    for (int jc = 0; jc < 8; ++jc) {
      const int zshift = 4 * ((jc >> 1) + 4 * (jc & 1));  // 4 * AWQ_REVERSE_ORDER[jc]
      const float z = static_cast<float>((zw >> zshift) & 0xFu);
      const bool kindB = ((jc >> 1) & 1) != 0;
      zoff[jc] = kindB ? 1024.f + 16.f * z : 1024.f + z;
      if (kindB) sc[jc] *= 0.0625f;
    }
    const int pc0 = gv_pos(8 * lane);  // 8 consecutive floats (never straddles a pad)
#pragma unroll
    for (int m = 0; m < MT; ++m) {
      const float4 s0 = *reinterpret_cast<const float4*>(&my_red[m * kGvRedStride + pc0]);
      const float4 s1 = *reinterpret_cast<const float4*>(&my_red[m * kGvRedStride + pc0 + 4]);
      float4* c0 = reinterpret_cast<float4*>(&my_col[m * kV3TileCols + 8 * lane]);
      float4 a0 = c0[0], a1 = c0[1];
      a0.x += sc[0] * (s0.x - zoff[0] * X[m]);
      a0.y += sc[1] * (s0.y - zoff[1] * X[m]);
      a0.z += sc[2] * (s0.z - zoff[2] * X[m]);
      a0.w += sc[3] * (s0.w - zoff[3] * X[m]);
      a1.x += sc[4] * (s1.x - zoff[4] * X[m]);
      a1.y += sc[5] * (s1.y - zoff[5] * X[m]);
      a1.z += sc[6] * (s1.z - zoff[6] * X[m]);
      a1.w += sc[7] * (s1.w - zoff[7] * X[m]);
      c0[0] = a0;
      c0[1] = a1;
    }
  }
}

// As v3_fold, but the folded column sums stay in REGISTERS: lane l owns word-column l = 8 columns x MT tokens
// (ycol[m][j]).  The per-warp column accumulators in shared memory cost 8 KB x MT per CTA - with MT = 8 that left room
// for ONE ring stage per warp and the M = 8 GEMV ran about twice as slow as M = 1; in registers every MT gets at
// least two stages.
template <int MT>
__device__ __forceinline__ void v3_fold_reg(const uint8_t* sa, float* my_red, float (&ycol)[MT][8], int lane, int g, int tig,
                                            const float (&acc)[4][4][4], const float (&xs_acc)[4]) {
#pragma unroll
  for (int w = 0; w < 4; ++w)
#pragma unroll
    for (int tt = 0; tt < 4; ++tt) {
      const int pc = gv_pos(32 * g + 8 * w + 2 * tt);
      if (2 * tig < MT)
        *reinterpret_cast<float2*>(&my_red[(2 * tig) * kGvRedStride + pc]) = make_float2(acc[w][tt][0], acc[w][tt][2]);
      if (2 * tig + 1 < MT)
        *reinterpret_cast<float2*>(&my_red[(2 * tig + 1) * kGvRedStride + pc]) =
            make_float2(acc[w][tt][1], acc[w][tt][3]);
    }
  float X[MT];
#pragma unroll
  for (int m = 0; m < MT; ++m) {
    const float v = (m & 1) ? xs_acc[1] : xs_acc[0];
    X[m] = __shfl_sync(0xffffffffu, v, m >> 1);
  }
  __syncwarp();
  const uint4 sc4 = *reinterpret_cast<const uint4*>(sa + lane * 16);
  const uint32_t zw = *reinterpret_cast<const uint32_t*>(sa + kV3ScaleBytes + lane * 4);
  const __half2* sc2 = reinterpret_cast<const __half2*>(&sc4);
  float sc[8], zoff[8];
#pragma unroll
  for (int jj = 0; jj < 4; ++jj) {
    const float2 f = __half22float2(sc2[jj]);
    sc[2 * jj] = f.x;
    sc[2 * jj + 1] = f.y;
  }
#pragma unroll
  for (int jc = 0; jc < 8; ++jc) {
    const int zshift = 4 * ((jc >> 1) + 4 * (jc & 1));
    const float z = static_cast<float>((zw >> zshift) & 0xFu);
    const bool kindB = ((jc >> 1) & 1) != 0;
    zoff[jc] = kindB ? 1024.f + 16.f * z : 1024.f + z;
    if (kindB) sc[jc] *= 0.0625f;
  }
  const int pc0 = gv_pos(8 * lane);
#pragma unroll
  for (int m = 0; m < MT; ++m) {
    const float4 s0 = *reinterpret_cast<const float4*>(&my_red[m * kGvRedStride + pc0]);
    const float4 s1 = *reinterpret_cast<const float4*>(&my_red[m * kGvRedStride + pc0 + 4]);
    ycol[m][0] += sc[0] * (s0.x - zoff[0] * X[m]);
    ycol[m][1] += sc[1] * (s0.y - zoff[1] * X[m]);
    ycol[m][2] += sc[2] * (s0.z - zoff[2] * X[m]);
    ycol[m][3] += sc[3] * (s0.w - zoff[3] * X[m]);
    ycol[m][4] += sc[4] * (s1.x - zoff[4] * X[m]);
    ycol[m][5] += sc[5] * (s1.y - zoff[5] * X[m]);
    ycol[m][6] += sc[6] * (s1.z - zoff[6] * X[m]);
    ycol[m][7] += sc[7] * (s1.w - zoff[7] * X[m]);
  }
  __syncwarp();   // the staging area may be rewritten (next fold, or the warp's column-sum dump)
}
// Dump the warp's column sums into its staging area as [MT][256] (the layout v3_add_cols / v3_push_warp read) and
// clear them.
template <int MT>
__device__ __forceinline__ void v3_dump_cols(float* my_red, float (&ycol)[MT][8], int lane) {
#pragma unroll
  for (int m = 0; m < MT; ++m) {
    *reinterpret_cast<float4*>(&my_red[m * kV3TileCols + 8 * lane]) = make_float4(ycol[m][0], ycol[m][1], ycol[m][2], ycol[m][3]);
    *reinterpret_cast<float4*>(&my_red[m * kV3TileCols + 8 * lane + 4]) =
        make_float4(ycol[m][4], ycol[m][5], ycol[m][6], ycol[m][7]);
#pragma unroll
    for (int j = 0; j < 8; ++j) ycol[m][j] = 0.f;
  }
  __syncwarp();
}

}  // namespace b200awq
