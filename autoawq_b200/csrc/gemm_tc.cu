// Tensor-core path (M > 4 tokens): Y[M, N] = X[M, K] . deq(W), fp16 x fp16 -> fp32 on the warpgroup MMA (wgmma, sm_90a).
//
// Orientation ("swap-AB"): the MMA's M dimension is the OUTPUT-FEATURE axis n (128 per tile = two warpgroups of
// m64), the MMA's N dimension is the token axis (BT = 16..128 per tile).
//   A operand = W^T tile [128 n x 64 k]  - produced IN-KERNEL: producer warps read packed int4 words, dequantise in
//               registers (bit-exact with the dequant kernel) and store fp16 into shared memory in the 128B-swizzled
//               canonical layout (MN-major for the GEMM layout, whose words hold 8 consecutive n of one k; K-major for
//               the GEMV / GEMVFast layouts, whose words hold consecutive k of one n).
//   B operand = X tile [BT tokens x 64 k], K-major, 128B swizzle, loaded by TMA (cp.async.bulk.tensor.2d).
//   D         = [128 n x BT tokens] fp32 in the registers of two consumer warpgroups (64 n each), which also run the
//               epilogue (+bias -> fp16 -> global, or the split-K reduction).
// Warp roles (512 threads): warpgroups 0-1 = MMA + epilogue, warpgroups 2-3 = dequant producers; producer warp 0 also
// issues the activation TMA and the L2 prefetch of the packed weights.
// Pipeline: NS smem stages, one "full" mbarrier per stage (8 producer-warp arrivals + 1 TMA expect_tx), one "empty"
// mbarrier per stage (8 consumer-warp arrivals once the wgmma reading the stage has retired).
// Persistent CTAs walk (n_tile, m_tile, k_split) work items.  Split-K (only for M <= 256 and fewer tiles than SMs, where
// the problem is HBM-bound and every SM must stream weights) reduces through fp32 atomics into the caller's zeroed
// workspace; the last CTA of a tile rounds to fp16 and restores the zeros.
#include <cuda.h>

#include <mutex>
#include <unordered_map>

#include "common.cuh"
#include "kernels.h"

namespace b200awq {

constexpr int kTileN = 128;  // output features per tile (two m64 warpgroups)
constexpr int kBK = 64;      // k per pipeline stage (one 128B swizzle row of fp16)
constexpr int kAStageBytes = kTileN * kBK * 2;  // 16 KB
constexpr uint32_t kAHalfBytes = 64 * kBK * 2;  // the 64 output features of one consumer warpgroup (either layout)

struct TcParams {
  const int32_t* qweight;
  const __half* scales;
  const int32_t* qzeros;  // FAST layout: scaled zeros (fp16) reinterpret
  const __half* bias;
  __half* y;
  float* acc_ws;
  int* tickets;
  int M, K, N, G;
  int zw;          // GEMV layout: zeros width
  int n_tiles, m_tiles, ksplit;
  int has_tmq;     // GEMM layout: a tensor map over qweight is available for L2 prefetch
  int g_shift;     // log2(G) when G is a power of two, else 31 (G == K: one group) - no integer division on device
  int dbg;         // small-M kernel: record phase timestamps (knob 3 == 9)
};

// Accumulators live in registers (BT / 2 fp32 per consumer thread): BT <= 128 keeps them next to the loop's addresses
// within the 128 registers a thread of a 512-thread CTA may use.
template <int BT>
struct TcCfg {
  static constexpr int kXStageBytes = BT * kBK * 2;
  static constexpr int kStageBytes = kAStageBytes + kXStageBytes;
  static constexpr int kStages = BT >= 128 ? 6 : 8;
  static constexpr size_t kSmemBytes = (size_t)kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(kSmemBytes <= 232448, "shared memory per CTA");
};

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// A-operand descriptor of one consumer warpgroup's 64 output features at smem address `a` (see the loaders' layouts):
// MN-major SW128 (GEMM layout): 8-k groups 1024 B apart; K-major SW128: 8-row groups 1024 B apart.  k16 steps advance the
// start address by 2048 B (MN-major: two 8-k groups) or 32 B (K-major: inside the swizzled 128-byte row).
template <bool kMnMajorA>
__device__ __forceinline__ uint64_t tc_desc_a(uint32_t a) {
  return kMnMajorA ? gmma_desc(a, 8192, 1024) : gmma_desc(a, 16, 1024);
}
template <bool kMnMajorA>
__host__ __device__ constexpr uint32_t tc_a_k16_step() { return kMnMajorA ? (2048u >> 4) : (32u >> 4); }

// Issues the four k16 MMAs of one 64-k stage for one warpgroup (no commit).
template <int BT, bool kMnMajorA>
__device__ __forceinline__ void tc_mma_stage(float (&acc)[BT / 2], uint32_t a_addr, uint32_t x_addr) {
  const uint64_t da = tc_desc_a<kMnMajorA>(a_addr);
  const uint64_t db = gmma_desc(x_addr, 16, 1024);
#pragma unroll
  for (int k16 = 0; k16 < kBK / 16; ++k16)
    wgmma_f16<BT, kMnMajorA ? 1 : 0>(acc, da + (uint64_t)(k16 * tc_a_k16_step<kMnMajorA>()), db + (uint64_t)(k16 * (32 >> 4)));
}

// ------------------------------------------------------------------------------- A-tile producers
// 256 or 512 producer threads.  load() issues the global loads of one k-step (packed words plus,
// when the quantisation group changes, the group's zeros / scales) ONE STEP AHEAD of store(), which
// dequantises from registers and writes the swizzled fp16 tile: no global latency on the critical path.

// GEMM layout: thread dt owns word column c = dt % 16 (8 n) and rows kk = dt/16 + 16 j, j = 0..3.
// NG = quantisation groups per 64-row k-step: 1 for G >= 64, 2 for G == 32 (rows < 32 / >= 32).  Keeping the
// slot small (9 registers for NG = 1) is what allows a 6-deep register prefetch ring.
template <int NG>
struct GemmLayoutLoaderT {
  static constexpr int kThreads = 256;
  static constexpr int kDepth = NG == 1 ? 6 : 4;
  uint32_t q[4];
  uint32_t zq[NG];
  uint4 sc[NG];
  __device__ __forceinline__ void init() {
#pragma unroll
    for (int h = 0; h < NG; ++h) { zq[h] = 0; sc[h] = make_uint4(0, 0, 0, 0); }
  }
  __device__ __forceinline__ void load(const TcParams& p, int nt, int k0, int dt) {
    // 32-bit word offsets (K * N/8 < 2^32 for every real shape) keep the address arithmetic to a few
    // instructions per load; the first version spent ~90 instructions per k-step on 64-bit multiplies.
    const uint32_t NW = (uint32_t)p.N >> 3;
    const uint32_t c = dt & 15, rb = dt >> 4;
    const uint32_t wc = (uint32_t)nt * 16 + c;
    const bool ok = wc < NW;
    const uint32_t row0 = ((uint32_t)k0 + rb) * NW + wc;
    const uint32_t row16 = 16u * NW;
    const int32_t* src = p.qweight + row0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      q[j] = 0u;
      if (ok) q[j] = ldg_stream_u1(src + j * row16);
    }
#pragma unroll
    for (int h = 0; h < NG; ++h) {
      const int g = (k0 + (int)rb + 32 * h) >> p.g_shift;   // G is a power of two, or the single group G == K
      if (ok) {
        const uint32_t goff = (uint32_t)g * NW + wc;
        zq[h] = static_cast<uint32_t>(__ldg(p.qzeros + goff));
        sc[h] = __ldg(reinterpret_cast<const uint4*>(p.scales) + goff);  // 8 halves per word column
      }
    }
  }
  __device__ __forceinline__ void store(const TcParams& p, int nt, int k0, int dt, uint32_t a_stage) const {
    const int c = dt & 15, rb = dt >> 4;
    // columns past N keep q = 0, zeros = 0, scales = 0 from init(): they dequantise to exact zeros
    ZeroPairs zp[NG];
#pragma unroll
    for (int h = 0; h < NG; ++h) zp[h] = awq_zero_pairs(zq[h]);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int h = NG == 1 ? 0 : (j >> 1);
      const uint4 o = awq_dequant_word(q[j], zp[h], sc[h]);
      // MN-major SW128: (n/64)*8192 + (k/8)*1024 + (k%8)*128 + (((n%64)/8) ^ (k%8))*16 ; k = rb + 16 j
      const uint32_t off = (uint32_t)(c >> 3) * 8192u + (uint32_t)(2 * j + (rb >> 3)) * 1024u +
                           (uint32_t)(rb & 7) * 128u + (uint32_t)(((c & 7) ^ (rb & 7)) << 4);
      sts_u4(a_stage + off, o);
    }
  }
};

// GEMV layout: thread dt owns k-word cw = dt % 8 (8 consecutive k) and rows n = dt/8 + 32 j, j = 0..3.
struct GemvLayoutLoader {
  static constexpr int kThreads = 256;
  static constexpr int kDepth = 4;
  uint32_t q[4];
  uint32_t zs[4];  // per row: fp16 scale in the low half, zero-point (0..15) in the high half
  __device__ __forceinline__ void init() { zs[0] = zs[1] = zs[2] = zs[3] = 0; }
  __device__ __forceinline__ void load(const TcParams& p, int nt, int k0, int dt) {
    const int KW = p.K >> 3;
    const int cw = dt & 7, rb = dt >> 3;
    const int g = (k0 + cw * 8) >> p.g_shift;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = nt * kTileN + rb + 32 * j;
      q[j] = 0u;
      if (n < p.N) {
        q[j] = ldg_stream_u1(p.qweight + (int64_t)n * KW + (k0 >> 3) + cw);
        const uint32_t s = __half_as_ushort(__ldg(p.scales + (int64_t)n * (p.zw * 8) + g));
        const uint32_t zword = static_cast<uint32_t>(__ldg(p.qzeros + (int64_t)n * p.zw + (g >> 3)));
        zs[j] = s | (((zword >> (4 * (g & 7))) & 0xFu) << 16);
      }
    }
  }
  __device__ __forceinline__ void store(const TcParams& p, int nt, int k0, int dt, uint32_t a_stage) const {
    const int cw = dt & 7, rb = dt >> 3;
    const __half2 r16 = __float2half2_rn(0.0625f);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int nl = rb + 32 * j;
      const int n = nt * kTileN + nl;
      uint4 o = make_uint4(0, 0, 0, 0);
      if (n < p.N) {
        const float zf = static_cast<float>(zs[j] >> 16);
        const __half2 zA = __float2half2_rn(1024.f + zf);   // exact
        const __half2 zB = __float2half2_rn(-(64.f + zf));  // exact
        const __half2 s2 = __half2half2(__ushort_as_half(static_cast<unsigned short>(zs[j] & 0xffffu)));
        RawPairs r = awq_raw_pairs(q[j]);
        // pairs (k0,k4) (k1,k5) (k2,k6) (k3,k7)
        const uint32_t d0 = h2_as_u32(__hmul2(__hsub2(u32_as_h2(r.p[0]), zA), s2));
        const uint32_t d1 = h2_as_u32(__hmul2(__hfma2(u32_as_h2(r.p[1]), r16, zB), s2));
        const uint32_t d2 = h2_as_u32(__hmul2(__hsub2(u32_as_h2(r.p[2]), zA), s2));
        const uint32_t d3 = h2_as_u32(__hmul2(__hfma2(u32_as_h2(r.p[3]), r16, zB), s2));
        o.x = __byte_perm(d0, d1, 0x5410);  // (k0, k1)
        o.y = __byte_perm(d2, d3, 0x5410);  // (k2, k3)
        o.z = __byte_perm(d0, d1, 0x7632);  // (k4, k5)
        o.w = __byte_perm(d2, d3, 0x7632);  // (k6, k7)
      }
      // K-major SW128: row n * 128 B, 16-byte chunk (k/8) ^ (n % 8)
      const uint32_t off = (uint32_t)nl * 128u + (uint32_t)((cw ^ (nl & 7)) << 4);
      sts_u4(a_stage + off, o);
    }
  }
};

// GEMVFast layout: thread dt owns row n = dt/2 of the tile and the 32-k half h = dt%2 of the step.
struct FastLayoutLoader {
  static constexpr int kThreads = 256;
  static constexpr int kDepth = 4;
  uint4 q;
  uint32_t ss;  // scale (low half) | scaled zero (high half)
  __device__ __forceinline__ void init() { ss = 0; }
  __device__ __forceinline__ void load(const TcParams& p, int nt, int k0, int dt) {
    const int n = nt * kTileN + (dt >> 1), h = dt & 1;
    q = make_uint4(0, 0, 0, 0);
    const int g = (k0 + 32 * h) >> p.g_shift;
    if (n < p.N) {
      // 64-k block k0/64 of row group n/4 starts at int16 offset k0; run (n%4) * 16; half h * 8
      q = ldg_stream_u4(reinterpret_cast<const int16_t*>(p.qweight) + (int64_t)(n >> 2) * p.K + (int64_t)k0 +
                        (n & 3) * 16 + h * 8);
      const __half* sz_ptr = reinterpret_cast<const __half*>(p.qzeros);
      ss = static_cast<uint32_t>(__half_as_ushort(__ldg(p.scales + (int64_t)g * p.N + n))) |
           (static_cast<uint32_t>(__half_as_ushort(__ldg(sz_ptr + (int64_t)g * p.N + n))) << 16);
    }
  }
  __device__ __forceinline__ void store(const TcParams& p, int nt, int k0, int dt, uint32_t a_stage) const {
    const int nl = dt >> 1, h = dt & 1;
    const bool ok = nt * kTileN + nl < p.N;
    const __half2 r16 = __float2half2_rn(0.0625f);
    const __half2 m1024 = __float2half2_rn(1024.f), m64 = __float2half2_rn(-64.f);
    const __half2 s2 = __half2half2(__ushort_as_half(static_cast<unsigned short>(ss & 0xffffu)));
    const __half2 z2 = __half2half2(__ushort_as_half(static_cast<unsigned short>(ss >> 16)));
    const uint32_t w[4] = {q.x, q.y, q.z, q.w};
    uint32_t d[4][4];  // [word u][r'] : pair (k, k+1), k = 32h + 2u + 8r'
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      RawPairs r = awq_raw_pairs(w[u]);
      d[u][0] = h2_as_u32(__hfma2(__hsub2(u32_as_h2(r.p[0]), m1024), s2, z2));
      d[u][1] = h2_as_u32(__hfma2(__hfma2(u32_as_h2(r.p[1]), r16, m64), s2, z2));
      d[u][2] = h2_as_u32(__hfma2(__hsub2(u32_as_h2(r.p[2]), m1024), s2, z2));
      d[u][3] = h2_as_u32(__hfma2(__hfma2(u32_as_h2(r.p[3]), r16, m64), s2, z2));
    }
#pragma unroll
    for (int rp = 0; rp < 4; ++rp) {
      uint4 o = make_uint4(d[0][rp], d[1][rp], d[2][rp], d[3][rp]);  // k = 32h + 8rp + 0..7
      if (!ok) o = make_uint4(0, 0, 0, 0);
      const int cc = 4 * h + rp;
      const uint32_t off = (uint32_t)nl * 128u + (uint32_t)((cc ^ (nl & 7)) << 4);
      sts_u4(a_stage + off, o);
    }
  }
};

template <int LAYOUT>
struct LoaderOf;
template <> struct LoaderOf<0> { using T = GemmLayoutLoaderT<1>; };  // GEMM layout, G >= 64
template <> struct LoaderOf<3> { using T = GemmLayoutLoaderT<2>; };  // GEMM layout, G == 32
template <> struct LoaderOf<1> { using T = GemvLayoutLoader; };
template <> struct LoaderOf<2> { using T = FastLayoutLoader; };

// --------------------------------------------------------------------------------------- kernel
// warpgroups 0-1: consumers (wgmma on 64 output features each, accumulators in registers, epilogue); warpgroups 2-3: the
// dequant producers (8 warps).  The producers' register ring runs ahead across tile boundaries, so the epilogue of one
// tile overlaps the production of the next tile's first stages.
constexpr int kTcThreads = 512;

template <int BT, int LAYOUT>
__global__ void __launch_bounds__(kTcThreads, 1)
    gemm_tc_kernel(const __grid_constant__ CUtensorMap tmx, const __grid_constant__ CUtensorMap tmq,
                   const TcParams p) {
  using Cfg = TcCfg<BT>;
  constexpr int NS = Cfg::kStages;
  constexpr bool kMnMajorA = (LAYOUT == 0 || LAYOUT == 3);
  static_assert(LoaderOf<LAYOUT>::T::kThreads == 256, "two producer warpgroups");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* a_base = smem;                                  // NS x 16 KB
  uint8_t* x_base = smem + (size_t)NS * kAStageBytes;      // NS x BT*128 B
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)NS * Cfg::kStageBytes);
  uint64_t* full = bars;            // [NS]
  uint64_t* empty = bars + NS;      // [NS]
  int* s_flag = reinterpret_cast<int*>(bars + 2 * NS);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  pdl_trigger();

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmx);
    for (int s = 0; s < NS; ++s) {
      mbar_init(&full[s], 8 + 1);  // one elected arrival per producer warp + the TMA expect_tx
      mbar_init(&empty[s], 8);     // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();

  const int KS = p.K / kBK;  // k-steps in total
  const int n_work = p.n_tiles * p.m_tiles * p.ksplit;

  if (warp < 8) {
    // ================================================================= consumers: wgmma + epilogue (2 warpgroups)
    const int wg = warp >> 2;
    const int et = threadIdx.x;  // 0..255
    const uint32_t a_s = smem_u32(a_base) + (uint32_t)wg * kAHalfBytes;
    const uint32_t x_s = smem_u32(x_base);
    pdl_wait();  // outputs / workspace may alias memory the predecessor still uses
    int stage = 0;
    uint32_t phase = 0;
    for (int w = blockIdx.x; w < n_work; w += gridDim.x) {
      const int ks = w % p.ksplit;
      const int mt = (w / p.ksplit) % p.m_tiles;
      const int nt = w / (p.ksplit * p.m_tiles);
      const int s_begin = (int)((int64_t)KS * ks / p.ksplit), s_end = (int)((int64_t)KS * (ks + 1) / p.ksplit);
      float acc[BT / 2];
#pragma unroll
      for (int i = 0; i < BT / 2; ++i) acc[i] = 0.f;
      // one group of MMAs in flight: a stage is released once the group after it has been issued
      int prev = -1;
      for (int s = s_begin; s < s_end; ++s) {
        mbar_wait(&full[stage], phase);
        wgmma_fence();
        tc_mma_stage<BT, kMnMajorA>(acc, a_s + (uint32_t)stage * kAStageBytes, x_s + (uint32_t)stage * Cfg::kXStageBytes);
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
        prev = stage;
        if (++stage == NS) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);

      // accumulator element i of this thread: feature n_a (+8 when i & 2), token m_a + 8 (i / 4) + (i & 1)
      const int n_a = nt * kTileN + wg * 64 + (warp & 3) * 16 + (lane >> 2);
      const int m0 = mt * BT;
      const int m_a = m0 + 2 * (lane & 3);
      const float bias_a = (p.bias != nullptr && n_a < p.N) ? __half2float(p.bias[n_a]) : 0.f;
      const float bias_b = (p.bias != nullptr && n_a + 8 < p.N) ? __half2float(p.bias[n_a + 8]) : 0.f;
#pragma unroll
      for (int i = 0; i < BT / 2; ++i) {
        const int n = n_a + ((i & 2) ? 8 : 0);
        const int m = m_a + 8 * (i >> 2) + (i & 1);
        if (n < p.N && m < p.M) {
          if (p.ksplit == 1)
            p.y[(int64_t)m * p.N + n] = __float2half_rn(acc[i] + ((i & 2) ? bias_b : bias_a));
          else
            atomicAdd(&p.acc_ws[(int64_t)m * p.N + n], acc[i]);
        }
      }
      if (p.ksplit > 1) {
        __threadfence();
        named_bar_sync(1, 256);
        if (et == 0) {
          const int prev_t = atomicAdd(&p.tickets[nt * p.m_tiles + mt], 1);
          *s_flag = (prev_t == p.ksplit - 1);
        }
        named_bar_sync(1, 256);
        const bool last = *s_flag != 0;
        named_bar_sync(1, 256);  // everyone has read the flag before a later item rewrites it
        if (last) {
          __threadfence();
          // thread et finalises feature (et % 128) for the tokens of its half of every 32-token batch; 16 tokens per L2
          // round trip (loads first, then the stores), not one round trip per token
          const int n = nt * kTileN + (et & 127);
          const float bias_v = (p.bias != nullptr && n < p.N) ? __half2float(p.bias[n]) : 0.f;
          if (n < p.N) {
            for (int j0 = 16 * (et >> 7); j0 < BT && m0 + j0 < p.M; j0 += 32) {
              float f[16];
#pragma unroll
              for (int j = 0; j < 16; ++j) {
                const int m = m0 + j0 + j;
                f[j] = m < p.M ? ld_relaxed_f32(&p.acc_ws[(int64_t)m * p.N + n]) : 0.f;
              }
#pragma unroll
              for (int j = 0; j < 16; ++j) {
                const int m = m0 + j0 + j;
                if (m < p.M) {
                  p.acc_ws[(int64_t)m * p.N + n] = 0.f;
                  p.y[(int64_t)m * p.N + n] = __float2half_rn(f[j] + bias_v);
                }
              }
            }
          }
          if (et == 0) p.tickets[nt * p.m_tiles + mt] = 0;
        }
      }
    }
  } else {
    // ================================================================= dequant producers (8 warps)
    // Global loads run kPrefetch k-steps ahead of the dequantisation (register ring): a k-step is only a few hundred
    // MMA cycles, well below the DRAM / L2 latency a 1-deep prefetch would expose every step.
    constexpr int kPrefetch = LoaderOf<LAYOUT>::T::kDepth;
    const int dt = threadIdx.x - 256;  // 0..255
    const int pw = dt >> 5;            // producer warp; warp 0 also issues the activation TMA and the L2 prefetch
    const bool leader = pw == 0 && elect_one();
    const uint32_t a_base_s = smem_u32(a_base);
    typename LoaderOf<LAYOUT>::T ring[kPrefetch];
    // The (work item, k-step) sequence of this CTA is ONE stream: the load cursor runs kPrefetch steps ahead
    // of the store cursor straight through tile boundaries, so the ring never drains between tiles.
    struct Cursor {
      int w, s, s_end, nt, mt;
      bool valid;
    };
    auto set_range = [&](Cursor& c) {
      const int ks = c.w % p.ksplit;
      c.nt = c.w / (p.ksplit * p.m_tiles);
      c.mt = (c.w / p.ksplit) % p.m_tiles;
      c.s = (int)((int64_t)KS * ks / p.ksplit);
      c.s_end = (int)((int64_t)KS * (ks + 1) / p.ksplit);
    };
    auto advance = [&](Cursor& c) {
      if (++c.s == c.s_end) {
        c.w += gridDim.x;
        c.valid = c.w < n_work;
        if (c.valid) set_range(c);
      }
    };
    Cursor L, S, P;
    L.w = S.w = P.w = blockIdx.x;
    L.valid = S.valid = blockIdx.x < n_work;
    if (L.valid) { set_range(L); set_range(S); set_range(P); }
    // GEMM layout: pull the packed weights of the next kL2Ahead k-steps from HBM into L2 (TMA prefetch, no smem
    // destination) so that the register prefetch only has to cover L2 latency.  Weights do not depend on the
    // predecessor kernel: this starts before the PDL wait.
    constexpr int kL2Ahead = 16;
    P.valid = kMnMajorA && p.has_tmq && pw == 0 && L.valid;
    for (int i = 0; i < kL2Ahead && P.valid; ++i) {
      if (leader) tma_prefetch_l2_2d(&tmq, P.nt * 16, P.s * kBK);
      advance(P);
    }
#pragma unroll
    for (int d = 0; d < kPrefetch; ++d) {
      ring[d].init();
      if (L.valid) {
        ring[d].load(p, L.nt, L.s * kBK, dt);
        advance(L);
      }
    }
    if (pw == 0) pdl_wait();  // the activations are the predecessor's output
    int stage = 0;
    uint32_t phase = 0;
    while (S.valid) {
#pragma unroll
      for (int d = 0; d < kPrefetch; ++d) {
        if (S.valid) {
          mbar_wait(&empty[stage], phase ^ 1);
          if (leader) {
            mbar_arrive_expect_tx(&full[stage], Cfg::kXStageBytes);
            tma_load_2d(x_base + (size_t)stage * Cfg::kXStageBytes, &tmx, &full[stage], S.s * kBK, S.mt * BT);
            if (P.valid) tma_prefetch_l2_2d(&tmq, P.nt * 16, P.s * kBK);
          }
          if (P.valid) advance(P);
          ring[d].store(p, S.nt, S.s * kBK, dt, a_base_s + (uint32_t)stage * kAStageBytes);
          fence_proxy_async_smem();   // every writer: generic-proxy stores -> visible to the tensor core
          __syncwarp();
          if (lane == 0) mbar_arrive(&full[stage]);  // 8 arrivals per stage instead of 256
          if (++stage == NS) { stage = 0; phase ^= 1; }
          advance(S);
          if (L.valid) {
            ring[d].load(p, L.nt, L.s * kBK, dt);
            advance(L);
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------ small-M kernel (TMA-staged packed weights)
// M <= 128 on the GEMM layout is HBM-bound; the kernel above is latency-bound there (its producers pull the packed
// words L2 -> registers through a shallow register ring whatever the token count).  This variant keeps the MMA /
// descriptor / epilogue machinery and changes what bounds it:
//   * the packed weights arrive by TMA in a deep shared-memory ring, one stage = a PAIR of k-steps (128 rows x 16 words
//     = 8 KB, plus the rows' group constants: 256 B of scales + 64 B of zeros per group), 11-14 stages = 96-123 KB in
//     flight per SM independent of registers, issued by a dedicated warp that never waits for activations (weights do
//     not depend on the predecessor kernel);
//   * 8 producer warps dequantise both k-steps of every stage (conflict-free LDS, the exact arithmetic of the dequant
//     kernel: the A tile is bit-identical) into the A stages; the activation tiles have their own ring and TMA warp
//     (they come from L2, with its latency under load);
//   * work is cut into CONTIGUOUS RANGES of the linearised (n-tile, k-step pair) sequence, one range per SM: every SM
//     streams the same number of bytes whatever N / 128 is.  A range crosses at most a few n-tiles = segments; a
//     segment that holds a whole K column stores fp16 directly, a partial one adds fp32 into the caller's zeroed
//     workspace and bumps the tile's ticket by its number of k-step pairs; the contributor that completes K rounds,
//     adds the bias, restores zeros.  Wherever N / 128 <= SM count (and from 64 tokens on) the ranges are tile-aligned
//     instead: gemm_tcq_grid.
//   * knob 22 = optional HBM -> L2 prefetch ahead of the ring.
template <int BT>
struct TcqCfg {
  static constexpr int kNS = 4;                                            // A stages (producers -> MMA)
  static constexpr int kNX = BT <= 16 ? 16 : (BT <= 64 ? 8 : 4);           // X stages (TMA -> MMA), own ring
  static constexpr int kNQ = BT <= 32 ? 14 : 11;                           // packed-weight stages (TMA -> producers)
  static constexpr int kXStageBytes = BT * kBK * 2;
  static constexpr int kQRows = 2 * kBK;                                   // rows per packed stage: two k-steps
  static constexpr int kQTileBytes = 16 * 4 * kQRows;                      // 128 rows x 16 words = 8 KB
  static constexpr int kQStageBytes = kQTileBytes + 2 * 256 + 2 * 64 + 128;   // up to 2 groups of constants; 128-B multiple
  static constexpr int kThreads = 256 + 256 + 64;   // 2 consumer warpgroups, 8 producer warps, Q-TMA warp, X-TMA warp
  static constexpr size_t kSmemBytes = (size_t)kNS * kAStageBytes + (size_t)kNX * kXStageBytes +
                                       (size_t)kNQ * kQStageBytes + 1024 /*align slack*/ + 1024 /*barriers*/;
  static_assert(kQStageBytes % 128 == 0, "TMA destination alignment");
  static_assert(kSmemBytes <= 232448, "shared memory per CTA");
};

__device__ __forceinline__ uint32_t lds_u1(uint32_t saddr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(saddr) : "memory");
  return v;
}
__device__ __forceinline__ uint4 lds_u4(uint32_t saddr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(saddr) : "memory");
  return v;
}

// Phase timestamps (globaltimer, ns) of the last small-M launch, 8 per CTA, written only when knob 3 == 9 (TcParams::dbg):
// [0] entry, [1] setup done (barriers), [2] first packed stage landed, [3] producers done, [4] MMA issue done,
// [5] last accumulator complete, [6] epilogue done (incl. finalisation), [7] number of segments.
__device__ unsigned long long g_tcq_dbg[256 * 8];
__device__ __forceinline__ unsigned long long tcq_timer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
cudaError_t gemm_tcq_debug_read(void* dst, size_t bytes) {
  return cudaMemcpyFromSymbol(dst, g_tcq_dbg, bytes < sizeof(g_tcq_dbg) ? bytes : sizeof(g_tcq_dbg));
}

// Work unit = a PAIR of k-steps (128 rows of one 128-column tile); p.K % 128 == 0.
template <int BT>
__global__ void __launch_bounds__(TcqCfg<BT>::kThreads, 1)
    gemm_tcq_kernel(const __grid_constant__ CUtensorMap tmx, const __grid_constant__ CUtensorMap tmq, const TcParams p) {
  using Cfg = TcqCfg<BT>;
  constexpr int NS = Cfg::kNS, NX = Cfg::kNX, NQ = Cfg::kNQ;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* a_base = smem;                                              // NS x 16 KB
  uint8_t* x_base = a_base + (size_t)NS * kAStageBytes;                // NX x BT*128 B
  uint8_t* q_base = x_base + (size_t)NX * Cfg::kXStageBytes;           // NQ x kQStageBytes
  uint64_t* bars = reinterpret_cast<uint64_t*>(q_base + (size_t)NQ * Cfg::kQStageBytes);
  uint64_t* full = bars;                     // [NS]  8 producer warps
  uint64_t* empty = full + NS;               // [NS]  8 consumer warps
  uint64_t* xfull = empty + NS;              // [NX]  expect_tx of the activation tile
  uint64_t* xempty = xfull + NX;             // [NX]  8 consumer warps
  uint64_t* qfull = xempty + NX;             // [NQ]  expect_tx of the packed stage
  uint64_t* qempty = qfull + NQ;             // [NQ]  8 producer warps
  int* s_flag = reinterpret_cast<int*>(qempty + NQ);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  pdl_trigger();
  const bool dbg = (p.dbg & 1) != 0 && blockIdx.x < 256;
  unsigned long long* dbg_row = g_tcq_dbg + blockIdx.x * 8;
  if (dbg && threadIdx.x == 0) dbg_row[0] = tcq_timer();

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmx);
    tma_prefetch_desc(&tmq);
    for (int s = 0; s < NS; ++s) {
      mbar_init(&full[s], 8);
      mbar_init(&empty[s], 8);
    }
    for (int s = 0; s < NX; ++s) {
      mbar_init(&xfull[s], 1);
      mbar_init(&xempty[s], 8);
    }
    for (int s = 0; s < NQ; ++s) {
      mbar_init(&qfull[s], 1);
      mbar_init(&qempty[s], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();
  if (dbg && threadIdx.x == 0) dbg_row[1] = tcq_timer();

  // this CTA's contiguous range of the linearised (n-tile, k-step pair) sequence
  const int KP = p.K / Cfg::kQRows;   // k-step pairs per tile
  const long long T = (long long)p.n_tiles * KP;
  const int t_begin = (int)(T * (long long)blockIdx.x / (long long)gridDim.x);
  const int t_end = (int)(T * (long long)(blockIdx.x + 1) / (long long)gridDim.x);
  constexpr int kQWarp = 16, kXWarp = 17;
  // groups of constants per packed stage: G = 64 -> one per k-step; G >= 128 (or one group per row) -> one per pair
  const int ng = p.g_shift == 6 ? 2 : 1;

  if (warp == kQWarp) {
    // ================================================================= Q-TMA: packed weights + group constants
    // (the whole warp walks the loop, one elected lane issues: uniform operands, no per-instruction retry loops)
    const bool leader = elect_one();
    const uint32_t NW = (uint32_t)p.N >> 3;
    const uint32_t tx = (uint32_t)Cfg::kQTileBytes + (uint32_t)ng * 320u;
    const int pf_ahead = p.ksplit;   // (field reused by this kernel: L2 prefetch distance in pairs)
    int qs = 0;
    uint32_t qph = 0;
    for (int t = t_begin; t < t_end;) {
      const int nt = t / KP, d0 = t - nt * KP;
      const int d1 = (KP - d0 < t_end - t) ? KP : d0 + (t_end - t);
      for (int d = d0; d < d1; ++d) {
        mbar_wait(&qempty[qs], qph ^ 1);
        uint8_t* dst = q_base + (size_t)qs * Cfg::kQStageBytes;
        const uint32_t g = (uint32_t)(d * Cfg::kQRows) >> p.g_shift;
        if (leader) {
          // optional HBM -> L2 prefetch of the pair pf_ahead positions further down this CTA's range (knob 22)
          if (pf_ahead > 0) {
            const int tp = t + (d - d0) + pf_ahead;
            if (tp < t_end) {
              const int ntp = tp / KP;
              tma_prefetch_l2_2d(&tmq, ntp * 16, (tp - ntp * KP) * Cfg::kQRows);
            }
          }
          mbar_arrive_expect_tx(&qfull[qs], tx);
          tma_load_2d(dst, &tmq, &qfull[qs], nt * 16, d * Cfg::kQRows);
          for (int h = 0; h < ng; ++h) {
            bulk_load_1d(dst + Cfg::kQTileBytes + h * 256, p.scales + (size_t)(g + h) * p.N + (size_t)nt * kTileN, 256,
                         &qfull[qs]);
            bulk_load_1d(dst + Cfg::kQTileBytes + 512 + h * 64, p.qzeros + (size_t)(g + h) * NW + (size_t)nt * 16, 64,
                         &qfull[qs]);
          }
        }
        __syncwarp();
        if (++qs == NQ) { qs = 0; qph ^= 1; }
      }
      t += d1 - d0;
    }
  } else if (warp == kXWarp) {
    // ================================================================= X-TMA: activation tiles, own ring
    const bool leader = elect_one();
    pdl_wait();  // the activations are the predecessor's output
    int xs = 0;
    uint32_t xph = 0;
    for (int t = t_begin; t < t_end;) {
      const int nt = t / KP, d0 = t - nt * KP;
      const int d1 = (KP - d0 < t_end - t) ? KP : d0 + (t_end - t);
      for (int s = 2 * d0; s < 2 * d1; ++s) {
        mbar_wait(&xempty[xs], xph ^ 1);
        if (leader) {
          mbar_arrive_expect_tx(&xfull[xs], Cfg::kXStageBytes);
          tma_load_2d(x_base + (size_t)xs * Cfg::kXStageBytes, &tmx, &xfull[xs], s * kBK, 0);
        }
        __syncwarp();
        if (++xs == NX) { xs = 0; xph ^= 1; }
      }
      t += d1 - d0;
    }
  } else if (warp < 8) {
    // ================================================================= consumers: wgmma + epilogue (2 warpgroups)
    const int wg = warp >> 2;
    const int et = threadIdx.x;  // 0..255
    const uint32_t a_s = smem_u32(a_base) + (uint32_t)wg * kAHalfBytes;
    const uint32_t x_s = smem_u32(x_base);
    pdl_wait();  // outputs / workspace may alias memory the predecessor still uses
    int stage = 0, xs = 0;
    uint32_t phase = 0, xph = 0;
    int it = 0;
    for (int t = t_begin; t < t_end; ++it) {
      const int nt = t / KP, d0 = t - nt * KP;
      const int d1 = (KP - d0 < t_end - t) ? KP : d0 + (t_end - t);
      const bool whole = (d0 == 0 && d1 == KP);
      float acc[BT / 2];
#pragma unroll
      for (int i = 0; i < BT / 2; ++i) acc[i] = 0.f;
      int prev = -1, prev_x = -1;
      for (int s = 2 * d0; s < 2 * d1; ++s) {
        mbar_wait(&xfull[xs], xph);
        mbar_wait(&full[stage], phase);
        wgmma_fence();
        tc_mma_stage<BT, true>(acc, a_s + (uint32_t)stage * kAStageBytes, x_s + (uint32_t)xs * Cfg::kXStageBytes);
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && lane == 0) {
          mbar_arrive(&empty[prev]);
          mbar_arrive(&xempty[prev_x]);
        }
        prev = stage;
        prev_x = xs;
        if (++stage == NS) { stage = 0; phase ^= 1; }
        if (++xs == NX) { xs = 0; xph ^= 1; }
      }
      wgmma_wait<0>();
      if (prev >= 0 && lane == 0) {
        mbar_arrive(&empty[prev]);
        mbar_arrive(&xempty[prev_x]);
      }
      if (dbg && et == 0) dbg_row[5] = tcq_timer();

      // accumulator element i of this thread: feature n_a (+8 when i & 2), token m_a + 8 (i / 4) + (i & 1)
      const int n_a = nt * kTileN + wg * 64 + (warp & 3) * 16 + (lane >> 2);   // N % 128 == 0: always in range
      const int m_a = 2 * (lane & 3);
      const float bias_a = p.bias != nullptr ? __half2float(p.bias[n_a]) : 0.f;
      const float bias_b = p.bias != nullptr ? __half2float(p.bias[n_a + 8]) : 0.f;
#pragma unroll
      for (int i = 0; i < BT / 2; ++i) {
        const int n = n_a + ((i & 2) ? 8 : 0);
        const int m = m_a + 8 * (i >> 2) + (i & 1);
        if (m < p.M) {
          if (whole)
            p.y[(int64_t)m * p.N + n] = __float2half_rn(acc[i] + ((i & 2) ? bias_b : bias_a));
          else
            red_add_f32(&p.acc_ws[(int64_t)m * p.N + n], acc[i]);
        }
      }
      if (!whole) {
        // relaxed REDs -> CTA-scope barrier -> one acq_rel ticket (release is cumulative over what the barrier ordered)
        named_bar_sync(1, 256);
        if (et == 0) {
          const int prev_t = atom_add_acq_rel(&p.tickets[nt], d1 - d0);
          *s_flag = (prev_t + (d1 - d0) == KP);
        }
        named_bar_sync(1, 256);
        const bool last = *s_flag != 0;
        named_bar_sync(1, 256);  // everyone has read the flag before a later segment rewrites it
        if (last) {
          // thread et finalises feature (et % 128) for its half of every 32-token batch; all loads of a batch of 16
          // tokens are in flight before the first store (one L2 round trip per batch, not one per token)
          const int n = nt * kTileN + (et & 127);
          const float bias_v = p.bias != nullptr ? __half2float(p.bias[n]) : 0.f;
          for (int m0 = 16 * (et >> 7); m0 < p.M; m0 += 32) {
            float f[16];
#pragma unroll
            for (int j = 0; j < 16; ++j)
              f[j] = (m0 + j < p.M) ? ld_relaxed_f32(&p.acc_ws[(int64_t)(m0 + j) * p.N + n]) : 0.f;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
              if (m0 + j < p.M) {
                p.acc_ws[(int64_t)(m0 + j) * p.N + n] = 0.f;
                p.y[(int64_t)(m0 + j) * p.N + n] = __float2half_rn(f[j] + bias_v);
              }
            }
          }
          if (et == 0) p.tickets[nt] = 0;
        }
      }
      t += d1 - d0;
    }
    if (dbg && et == 0) { dbg_row[4] = tcq_timer(); dbg_row[6] = dbg_row[4]; dbg_row[7] = (unsigned long long)it; }
  } else {
    // ================================================================= dequant producers (8 warps)
    // Each packed stage holds two k-steps: rows 0..63 go to one A stage, rows 64..127 to the next.  Both halves' words
    // are read from shared memory before the first store, so the LDS latency overlaps the first half's dequantisation.
    const int dt = threadIdx.x - 256;  // 0..255
    const uint32_t a_base_s = smem_u32(a_base);
    const uint32_t q_base_s = smem_u32(q_base);
    const uint32_t c = dt & 15, rb = dt >> 4;
    using L = GemmLayoutLoaderT<1>;
    auto fetch = [&](L& r, uint32_t qa, uint32_t h) {
      const uint32_t q_off = (h * kBK + rb) * 64u + c * 4u;                        // rows 64 h + rb + 16 j, word column c
      const uint32_t gh = ng == 2 ? h : 0u;                                       // which group of constants
#pragma unroll
      for (int j = 0; j < 4; ++j) r.q[j] = lds_u1(qa + q_off + (uint32_t)j * 1024u);
      r.sc[0] = lds_u4(qa + Cfg::kQTileBytes + gh * 256u + c * 16u);              // 8 scales of word column c
      r.zq[0] = lds_u1(qa + Cfg::kQTileBytes + 512u + gh * 64u + c * 4u);         // its 8 zero-points
    };
    const int npairs = t_end - t_begin;
    int qs = 0, stage = 0;
    uint32_t qph = 0, phase = 0;
    for (int i = 0; i < npairs; ++i) {
      mbar_wait(&qfull[qs], qph);
      if (dbg && dt == 0 && i == 0) dbg_row[2] = tcq_timer();
      const uint32_t qa = q_base_s + (uint32_t)qs * Cfg::kQStageBytes;
      L hw[2];
      fetch(hw[0], qa, 0u);
      fetch(hw[1], qa, 1u);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        mbar_wait(&empty[stage], phase ^ 1);
        if (!(p.dbg & 2)) hw[h].store(p, 0, 0, dt, a_base_s + (uint32_t)stage * kAStageBytes);   // (knob 20)
        if (!(p.dbg & 4)) fence_proxy_async_smem();   // every writer: generic-proxy stores -> visible to the tensor core
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(&full[stage]);
          if (h == 1) mbar_arrive(&qempty[qs]);   // after the stores that consumed the stage's words (data dependence)
        }
        if (++stage == NS) { stage = 0; phase ^= 1; }
      }
      if (++qs == NQ) { qs = 0; qph ^= 1; }
    }
    if (dbg && dt == 0) dbg_row[3] = tcq_timer();
  }
}

// ------------------------------------------------------------ grouped (MoE) kernel: one launch over all experts' runs
// grouped_gemm_forward at prefill sizes: gemm_tc_kernel's tile, pipeline and MMA loop over stacked GEMM-layout experts.
//   * tile = 128 output features x BT sorted slots of ONE expert; the expert only moves the three weight base pointers
//     of the A-tile loader, so the A stage stays bit-identical to the dequant kernel;
//   * the X stage is a GATHER: row j of a tile is slot sorted_ids[pos0 + j], whose activations are x[id / topk] or
//     x[id] - no tensor map describes that.  Each of the 256 producer threads copies the 16-byte chunk (dt % 8) of rows
//     dt / 8 + 32 i with cp.async straight into the 128B-swizzled K-major layout the TMA would have written (the XOR is
//     applied to the destination address), zero-filling padding slots and rows past the run, and arrives on the
//     stage's `full` barrier through cp.async.mbarrier.arrive.noinc: full = 8 warp arrivals (A tile) + 256 (X rows);
//   * the work list is built ON THE DEVICE, so routing may change between replays of a captured graph: after
//     griddepcontrol.wait every CTA scans expert_ids[0 .. num_post_pad / block_size) into the list of runs (maximal
//     sequences of blocks of one expert) in shared memory; moe_tc_tile() then enumerates (run, n-tile, token tile) with
//     the token tile fastest - CTAs resident together share an expert's 128-column weight slab in L2 - and a grid
//     stride.  A token tile never crosses a run; the last one of a run is partial; experts without tokens have no run;
//   * the epilogue scatters: token column j goes to y[id], times topk_weights[id] in fp32 when asked (one rounding).
// No split-K and no workspace: calls with fewer tiles than SMs belong to the decode-sized kernels (see the routing).
constexpr int kMoeTcMaxRuns = 256;   // = the largest E routed here: moe_align_block_size writes one run per used expert
constexpr size_t kMoeTcTableBytes = (size_t)(2 * kMoeTcMaxRuns + 4) * sizeof(int);   // run_blk[257], run_e[256], n_runs

struct MoeTcParams {
  const __half* x;
  const int32_t* qweight;
  const __half* scales;
  const int32_t* qzeros;
  const float* topk_w;   // nullptr: outputs are not multiplied by the routing weight
  const int* sorted_ids;
  const int* expert_ids;
  const int* num_post_pad;
  __half* y;
  int n_slots, topk, x_per_slot;
  int E, K, N, groups, g_shift;
  int block_size, max_blocks;   // blocks the sorted_ids buffer holds: the scan never trusts *num_post_pad beyond it
};

struct MoeTcTile {
  int expert, pos0, rows, nt;   // expert, first sorted position, rows (<= BT), 128-column tile
};
struct MoeTcCursor {
  int run, base;                // tiles that precede `run`
};

// Tile w of the fixed order (run, n-tile, token tile), walking `c` forward from the previous query (w never
// decreases).  run_blk[r] .. run_blk[r + 1] are the blocks of run r; a run whose expert is out of range has no tiles.
// The kernel's three warp roles and b200awq_moe_tc_plan all enumerate through this one function.
__host__ __device__ inline bool moe_tc_tile(const int* run_blk, const int* run_e, int n_runs, int E, int block_size,
                                            int n_tiles, int BT, int w, MoeTcCursor& c, MoeTcTile& t) {
  for (; c.run < n_runs; ++c.run) {
    const int e = run_e[c.run];
    const int rows = (e >= 0 && e < E) ? (run_blk[c.run + 1] - run_blk[c.run]) * block_size : 0;
    const int tt = (rows + BT - 1) / BT;
    if (w < c.base + tt * n_tiles) {
      const int local = w - c.base;
      const int ti = local % tt;
      t.expert = e;
      t.nt = local / tt;
      t.pos0 = run_blk[c.run] * block_size + ti * BT;
      t.rows = rows - ti * BT < BT ? rows - ti * BT : BT;
      return true;
    }
    c.base += tt * n_tiles;
  }
  return false;
}

template <int BT, int NG>
__global__ void __launch_bounds__(kTcThreads, 1) moe_tc_kernel(const MoeTcParams p) {
  using Cfg = TcCfg<BT>;
  using Loader = GemmLayoutLoaderT<NG>;
  constexpr int NS = Cfg::kStages;
  constexpr int kRowsPerThread = BT / 32;   // gathered rows per producer thread and k-step
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* a_base = smem;                                  // NS x 16 KB
  uint8_t* x_base = smem + (size_t)NS * kAStageBytes;      // NS x BT*128 B
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)NS * Cfg::kStageBytes);
  uint64_t* full = bars;            // [NS]
  uint64_t* empty = bars + NS;      // [NS]
  int* run_blk = reinterpret_cast<int*>(smem + (size_t)NS * Cfg::kStageBytes + 256);   // [kMoeTcMaxRuns + 1]
  int* run_e = run_blk + kMoeTcMaxRuns + 1;                                            // [kMoeTcMaxRuns]
  int* s_runs = run_e + kMoeTcMaxRuns;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  pdl_trigger();
  if (threadIdx.x == 0) {
    for (int s = 0; s < NS; ++s) {
      mbar_init(&full[s], 8 + 256);  // one elected arrival per producer warp + every producer thread's gathered rows
      mbar_init(&empty[s], 8);       // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  // The routing tables decide WHICH weights are read, and they, the activations and y belong to predecessor kernels:
  // nothing is loaded before the wait.
  pdl_wait();
  if (warp == 0) {
    int nblk = *p.num_post_pad / p.block_size;
    nblk = nblk < p.max_blocks ? nblk : p.max_blocks;
    int n = 0;   // runs found so far
    for (int i0 = 0; i0 < nblk; i0 += 32) {
      const int i = i0 + lane;
      const int e = i < nblk ? p.expert_ids[i] : -1;
      const bool start = i < nblk && (i == 0 || p.expert_ids[i - 1] != e);
      const uint32_t m = __ballot_sync(0xffffffffu, start);
      const int r = n + __popc(m & ((1u << lane) - 1u));
      if (start && r <= kMoeTcMaxRuns) {
        run_blk[r] = i;
        if (r < kMoeTcMaxRuns) run_e[r] = e;
      }
      n += __popc(m);
    }
    if (lane == 0) {
      if (n <= kMoeTcMaxRuns) run_blk[n] = nblk;
      *s_runs = n < kMoeTcMaxRuns ? n : kMoeTcMaxRuns;
    }
  }
  __syncthreads();

  const int n_runs = *s_runs;
  const int n_tiles = (p.N + kTileN - 1) / kTileN;
  const int KS = p.K / kBK;
  auto locate = [&](int w, MoeTcCursor& c, MoeTcTile& t) {
    return moe_tc_tile(run_blk, run_e, n_runs, p.E, p.block_size, n_tiles, BT, w, c, t);
  };

  if (warp < 8) {
    // ================================================================= consumers: wgmma + scatter (2 warpgroups)
    const int wg = warp >> 2;
    const uint32_t a_s = smem_u32(a_base) + (uint32_t)wg * kAHalfBytes;
    const uint32_t x_s = smem_u32(x_base);
    int stage = 0;
    uint32_t phase = 0;
    MoeTcCursor cur{0, 0};
    MoeTcTile t;
    for (int w = blockIdx.x; locate(w, cur, t); w += gridDim.x) {
      float acc[BT / 2];
#pragma unroll
      for (int i = 0; i < BT / 2; ++i) acc[i] = 0.f;
      int prev = -1;
      for (int s = 0; s < KS; ++s) {
        mbar_wait(&full[stage], phase);
        fence_proxy_async_smem();   // the gathered rows are generic-proxy writes that completed asynchronously
        wgmma_fence();
        tc_mma_stage<BT, true>(acc, a_s + (uint32_t)stage * kAStageBytes, x_s + (uint32_t)stage * Cfg::kXStageBytes);
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
        prev = stage;
        if (++stage == NS) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);

      // accumulator elements 4 j + b (feature n_a) and 4 j + 2 + b (feature n_a + 8): tile row 8 j + 2 (lane % 4) + b
      const int n_a = t.nt * kTileN + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
      for (int j = 0; j < BT / 8; ++j) {
#pragma unroll
        for (int b = 0; b < 2; ++b) {
          const int m = 8 * j + 2 * (lane & 3) + b;
          if (m >= t.rows) continue;
          const int id = p.sorted_ids[t.pos0 + m];
          if ((unsigned)id >= (unsigned)p.n_slots) continue;   // padding
          const float v0 = p.topk_w != nullptr ? acc[4 * j + b] * p.topk_w[id] : acc[4 * j + b];
          const float v1 = p.topk_w != nullptr ? acc[4 * j + 2 + b] * p.topk_w[id] : acc[4 * j + 2 + b];
          __half* dst = p.y + (int64_t)id * p.N;
          if (n_a < p.N) dst[n_a] = __float2half_rn(v0);
          if (n_a + 8 < p.N) dst[n_a + 8] = __float2half_rn(v1);
        }
      }
    }
  } else {
    // ================================================================= producers: dequant + activation gather (8 warps)
    // As in gemm_tc_kernel the (tile, k-step) sequence of the CTA is one stream and the packed words run kPrefetch
    // k-steps ahead of the dequantisation in a register ring, straight through tile boundaries.
    constexpr int kPrefetch = Loader::kDepth;
    const int dt = threadIdx.x - 256;  // 0..255
    const uint32_t a_base_s = smem_u32(a_base);
    const uint32_t x_base_s = smem_u32(x_base);
    Loader ring[kPrefetch];
    struct Cursor {
      int w, s;
      bool valid;
      MoeTcCursor c;
      MoeTcTile t;
    };
    auto advance = [&](Cursor& c) {   // true when it entered a new tile
      if (++c.s < KS) return false;
      c.s = 0;
      c.w += gridDim.x;
      c.valid = locate(c.w, c.c, c.t);
      return c.valid;
    };
    // load cursor: the loader reads qweight / scales / qzeros / N / g_shift of a dense layer = this tile's expert
    TcParams lp;
    lp.N = p.N;
    lp.g_shift = p.g_shift;
    const int64_t NW = p.N >> 3;
    auto set_expert = [&](int e) {
      lp.qweight = p.qweight + (int64_t)e * p.K * NW;
      lp.scales = p.scales + (int64_t)e * p.groups * p.N;
      lp.qzeros = p.qzeros + (int64_t)e * p.groups * NW;
    };
    // store cursor: source row of each gathered tile row (-1: padding slot or past the run, zero-filled)
    int xrow[kRowsPerThread];
    auto set_rows = [&](const MoeTcTile& t) {
#pragma unroll
      for (int i = 0; i < kRowsPerThread; ++i) {
        const int j = (dt >> 3) + 32 * i;
        xrow[i] = -1;
        if (j < t.rows) {
          const int id = p.sorted_ids[t.pos0 + j];
          if ((unsigned)id < (unsigned)p.n_slots) xrow[i] = p.x_per_slot ? id : id / p.topk;
        }
      }
    };
    Cursor L, S;
    L.w = S.w = blockIdx.x;
    L.s = S.s = 0;
    L.c = S.c = MoeTcCursor{0, 0};
    L.valid = S.valid = locate(L.w, L.c, L.t);
    S.t = L.t;
    if (L.valid) {
      set_expert(L.t.expert);
      set_rows(S.t);
    }
#pragma unroll
    for (int d = 0; d < kPrefetch; ++d) {
      ring[d].init();
      if (L.valid) {
        ring[d].load(lp, L.t.nt, L.s * kBK, dt);
        if (advance(L)) set_expert(L.t.expert);
      }
    }
    int stage = 0;
    uint32_t phase = 0;
    while (S.valid) {
#pragma unroll
      for (int d = 0; d < kPrefetch; ++d) {
        if (S.valid) {
          mbar_wait(&empty[stage], phase ^ 1);
          // K-major SW128: tile row j at j * 128 B, 16-byte chunk c at (c ^ (j % 8)); j % 8 == (dt / 8) % 8 for every i
          const uint32_t x_dst = x_base_s + (uint32_t)stage * Cfg::kXStageBytes + (uint32_t)(dt >> 3) * 128u +
                                 (uint32_t)(((dt & 7) ^ ((dt >> 3) & 7)) << 4);
          const __half* x_src = p.x + S.s * kBK + (dt & 7) * 8;
#pragma unroll
          for (int i = 0; i < kRowsPerThread; ++i) {
            const bool ok = xrow[i] >= 0;
            cp_async_16(x_dst + (uint32_t)i * 4096u, x_src + (int64_t)(ok ? xrow[i] : 0) * p.K, ok ? 16u : 0u);
          }
          cp_async_mbar_arrive_noinc(&full[stage]);
          ring[d].store(lp, 0, 0, dt, a_base_s + (uint32_t)stage * kAStageBytes);
          fence_proxy_async_smem();   // every writer: generic-proxy stores -> visible to the tensor core
          __syncwarp();
          if (lane == 0) mbar_arrive(&full[stage]);
          if (++stage == NS) { stage = 0; phase ^= 1; }
          if (advance(S)) set_rows(S.t);
          if (L.valid) {
            ring[d].load(lp, L.t.nt, L.s * kBK, dt);
            if (advance(L)) set_expert(L.t.expert);
          }
        }
      }
    }
  }
}

// -------------------------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(f);
  });
  return fn;
}

struct TmapKey {
  const void* ptr;
  uint64_t inner, outer, pitch;
  uint32_t bi, bo;
  int kind;  // bit 0: element type, bit 1: 128B swizzle
  bool operator==(const TmapKey& o) const {
    return ptr == o.ptr && inner == o.inner && outer == o.outer && pitch == o.pitch && bi == o.bi && bo == o.bo &&
           kind == o.kind;
  }
};
struct TmapKeyHash {
  size_t operator()(const TmapKey& k) const {
    size_t h = reinterpret_cast<size_t>(k.ptr);
    h ^= (size_t)k.inner * 0x9E3779B97F4A7C15ull + (size_t)k.outer * 1315423911u + (size_t)k.pitch * 2654435761u +
         (size_t)k.bi * 31u + (size_t)k.bo * 131u + (size_t)k.kind;
    return h;
  }
};

cudaError_t make_tmap_2d(const void* ptr, int elem_kind, uint64_t inner, uint64_t outer, uint64_t pitch_bytes,
                         uint32_t box_inner, uint32_t box_outer, CUtensorMap* out, bool swizzle128) {
  static std::mutex mu;
  static std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> cache;
  TmapKey key{ptr, inner, outer, pitch_bytes, box_inner, box_outer, elem_kind | (swizzle128 ? 2 : 0)};
  {
    std::lock_guard<std::mutex> lk(mu);
    auto it = cache.find(key);
    if (it != cache.end()) {
      *out = it->second;
      return cudaSuccess;
    }
  }
  EncodeTiledFn enc = get_encode_fn();
  if (enc == nullptr) return cudaErrorNotSupported;
  cuuint64_t dims[2] = {(cuuint64_t)inner, (cuuint64_t)outer};
  cuuint64_t strides[1] = {(cuuint64_t)pitch_bytes};
  cuuint32_t box[2] = {(cuuint32_t)box_inner, (cuuint32_t)box_outer};
  cuuint32_t estr[2] = {1, 1};
  const CUtensorMapDataType dt = elem_kind == 0 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_INT32;
  CUresult r = enc(out, dt, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return cudaErrorInvalidValue;
  std::lock_guard<std::mutex> lk(mu);
  if (cache.size() > 8192) cache.clear();
  cache.emplace(key, *out);
  return cudaSuccess;
}

// X[M, K] fp16 (row pitch ld elements) -> box {64 k, BT rows}
static cudaError_t make_x_tmap(const void* x, int64_t ld, int M, int K, int BT, CUtensorMap* out) {
  return make_tmap_2d(x, 0, (uint64_t)K, (uint64_t)M, (uint64_t)ld * 2, kBK, (uint32_t)BT, out);
}

static int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = B200AWQ_SM_COUNT_FALLBACK;
  }
  return n;
}

template <int BT, int LAYOUT>
static cudaError_t launch_tc(const CUtensorMap& tm, const CUtensorMap& tmq, const TcParams& p, cudaStream_t st) {
  using Cfg = TcCfg<BT>;
  auto kern = gemm_tc_kernel<BT, LAYOUT>;
  static bool attr_set[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !attr_set[dev]) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::kSmemBytes);
    if (e != cudaSuccess) return e;
    if (dev >= 0 && dev < 64) attr_set[dev] = true;
  }
  const int n_work = p.n_tiles * p.m_tiles * p.ksplit;
  const int grid = n_work < sm_count() ? n_work : sm_count();
  return launch_kernel(kern, dim3(grid), dim3(kTcThreads), Cfg::kSmemBytes, st, tm, tmq, p);
}

template <int LAYOUT>
static cudaError_t dispatch_bt(int BT, const CUtensorMap& tm, const CUtensorMap& tmq, const TcParams& p,
                               cudaStream_t st) {
  switch (BT) {
    case 32: return launch_tc<32, LAYOUT>(tm, tmq, p, st);
    case 64: return launch_tc<64, LAYOUT>(tm, tmq, p, st);
    default: return launch_tc<128, LAYOUT>(tm, tmq, p, st);
  }
}

// Grid of the small-M kernel = how the linearised (n-tile, k-step pair) sequence is cut (CTA b owns the pairs
// [T b / grid, T (b + 1) / grid), T = n_tiles * KP).  mode = knob 21.
int gemm_tcq_grid(int n_tiles, int KP, int M, int sms, int mode) {
  const long long T = (long long)n_tiles * KP;
  long long grid = T / 2;   // balanced ranges: every CTA streams the same bytes; at least 2 pairs per CTA
  if (grid < 1) grid = 1;
  if (grid > sms) grid = sms;
  // Tile-aligned ranges (knob 21: 1 = never, 2 = always): a range that never straddles an n-tile has ONE segment, and a
  // range that is a whole tile stores fp16 directly - no fp32 REDs, no ticket, no read-back (M * 128 REDs per segment,
  // M / 16 L2 round trips per finalised tile).
  if (mode != 1) {
    long long g = 0;
    if (n_tiles <= sms) {
      // every tile is cut into ks ranges (boundaries b * KP / ks never cross a tile since the grid is a multiple of
      // n_tiles); ks = 1 stores whole tiles directly: no fp32 reduction at all.
      int ks = sms / n_tiles;
      if (ks > KP / 2) ks = KP / 2;
      if (ks < 1) ks = 1;
      g = (long long)n_tiles * ks;
    } else if (mode == 2 || M >= 64) {
      // more tiles than SMs: whole tiles per CTA when they divide evenly (224 tiles -> 112 CTAs x 2); below 64 tokens
      // the balanced cut (every SM streams, the split-K traffic is small) is kept
      const int tpc = (n_tiles + sms - 1) / sms;
      if (n_tiles % tpc == 0) g = n_tiles / tpc;
    }
    if (g > 0) grid = g;
  }
  return (int)grid;
}

template <int BT>
static cudaError_t launch_tcq(const CUtensorMap& tm, const CUtensorMap& tmq, const TcParams& p, cudaStream_t st) {
  using Cfg = TcqCfg<BT>;
  auto kern = gemm_tcq_kernel<BT>;
  static bool attr_set[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !attr_set[dev]) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::kSmemBytes);
    if (e != cudaSuccess) return e;
    if (dev >= 0 && dev < 64) attr_set[dev] = true;
  }
  const int grid = gemm_tcq_grid(p.n_tiles, p.K / Cfg::kQRows, p.M, sm_count(), knob(21));
  return launch_kernel(kern, dim3((unsigned)grid), dim3(Cfg::kThreads), Cfg::kSmemBytes, st, tm, tmq, p);
}

// Small-M path (M <= kTcqMaxM, GEMM layout, G >= 64, N % 128 == 0): see gemm_tcq_kernel.  The fp32 split-K scratch is
// the caller's workspace: M * N floats fit the documented min(M, 128) * N * 8 bytes.
constexpr int kTcqMaxM = 128;
bool gemm_tcq_shape_ok(int M, int K, int N, int G) {
  return M >= 1 && M <= kTcqMaxM && G >= 64 && (K % 128) == 0 && (N % kTileN) == 0 && N / kTileN <= 4096;
}
bool gemm_tcq_applicable(const GemmArgs& a, const float* acc_ws, const int* tickets) {
  if (knob(19) == 1) return false;
  if (!gemm_tcq_shape_ok(a.M, a.K, a.N, a.G)) return false;
  if (acc_ws == nullptr || tickets == nullptr) return false;
  if (((reinterpret_cast<uintptr_t>(a.qweight) | reinterpret_cast<uintptr_t>(a.scales) |
        reinterpret_cast<uintptr_t>(a.qzeros)) & 15) != 0)
    return false;
  return true;
}

static int zeros_width_tc(int K, int G) {
  const int mult = G >= 128 ? 1 : (G == 64 ? 2 : 4);
  int base = ((K / G) + 7) / 8;
  return ((base + mult - 1) / mult) * mult;
}

cudaError_t gemm_tc(const GemmArgs& a, int layout, float* acc_ws, int* tickets, cudaStream_t st) {
  if (a.K % kBK != 0 || a.G % 32 != 0) return cudaErrorNotSupported;
  const bool g_pow2 = (a.G & (a.G - 1)) == 0;
  if (!g_pow2 && a.G != a.K) return cudaErrorNotSupported;  // AWQ group sizes: 32 / 64 / 128 / whole row
  if ((reinterpret_cast<uintptr_t>(a.x) & 15) != 0 || (a.ldx % 8) != 0) return cudaErrorMisalignedAddress;
  const int BT = a.M <= 32 ? 32 : (a.M <= 64 ? 64 : 128);
  TcParams p;
  p.qweight = a.qweight;
  p.scales = reinterpret_cast<const __half*>(a.scales);
  p.qzeros = a.qzeros;
  p.bias = reinterpret_cast<const __half*>(a.bias);
  p.y = reinterpret_cast<__half*>(a.y);
  p.acc_ws = acc_ws;
  p.tickets = tickets;
  p.M = a.M; p.K = a.K; p.N = a.N; p.G = a.G;
  p.dbg = 0;
  p.zw = zeros_width_tc(a.K, a.G);
  p.g_shift = 31;
  if (g_pow2) {
    p.g_shift = 0;
    while ((1 << p.g_shift) < a.G) ++p.g_shift;
  }
  p.n_tiles = (a.N + kTileN - 1) / kTileN;
  if (layout == 0 && gemm_tcq_applicable(a, acc_ws, tickets)) {
    const int BQ = a.M <= 16 ? 16 : (a.M <= 32 ? 32 : (a.M <= 64 ? 64 : 128));
    CUtensorMap tmxq, tmwq;
    p.m_tiles = 1;
    p.ksplit = knob(22);   // small-M kernel: L2 prefetch distance in k-step pairs (0 = off)
    p.has_tmq = 1;
    p.dbg = (knob(3) == 9 ? 1 : 0) | ((knob(20) & 3) << 1);   // knob 20: producer timing experiments (results invalid)
    cudaError_t eq = make_x_tmap(a.x, a.ldx, a.M, a.K, BQ, &tmxq);
    if (eq == cudaSuccess)
      eq = make_tmap_2d(a.qweight, 1, (uint64_t)(a.N / 8), (uint64_t)a.K, (uint64_t)(a.N / 8) * 4, 16, 2 * kBK, &tmwq, false);
    if (eq == cudaSuccess) {
      switch (BQ) {
        case 16: return launch_tcq<16>(tmxq, tmwq, p, st);
        case 32: return launch_tcq<32>(tmxq, tmwq, p, st);
        case 64: return launch_tcq<64>(tmxq, tmwq, p, st);
        default: return launch_tcq<128>(tmxq, tmwq, p, st);
      }
    }
    // a tensor map that cannot be encoded: fall through to the register-staged kernel
  }
  p.m_tiles = (a.M + BT - 1) / BT;
  const int KS = a.K / kBK;
  int ksplit = 1;
  const int tiles = p.n_tiles * p.m_tiles;
  // fp32 partial sums: the workspace holds min(M, kMaxSplitM) * N 8-byte words = room for 2 * kMaxSplitM token rows
  if (a.M <= 2 * kMaxSplitM && acc_ws != nullptr && tickets != nullptr && tiles < sm_count() && tiles <= 4096) {
    ksplit = sm_count() / tiles;
    if (ksplit < 1) ksplit = 1;
    while (ksplit > 1 && KS / ksplit < 4) --ksplit;  // at least 4 k-steps per slice
  }
  // Above 64 tokens the reduction is no longer free (M * 128 fp32 REDs per CTA, M / 16 L2 round trips for the
  // finaliser) against the k-steps it takes off the critical path - split only when it pays.  The cost model (0.15 per
  // token vs 0.5 per k-step saved) was carried over from the kernel's earlier tuning and not re-measured on H100.
  if (a.M > 64 && ksplit > 1 && (float)(KS - KS / ksplit) * 0.5f < 0.15f * (float)a.M) ksplit = 1;
  const int forced = knob(1);
  if (forced > 0 && a.M <= 2 * kMaxSplitM && acc_ws != nullptr && tickets != nullptr) ksplit = forced > KS ? KS : forced;
  p.ksplit = ksplit;
  CUtensorMap tm, tmq;
  cudaError_t e = make_x_tmap(a.x, a.ldx, a.M, a.K, BT, &tm);
  if (e != cudaSuccess) return e;
  tmq = tm;
  p.has_tmq = 0;
  if (layout == 0 && (a.N % 4) == 0 && (reinterpret_cast<uintptr_t>(a.qweight) & 15) == 0 && (a.N / 8) % 4 == 0) {
    // qweight [K, N/8] int32 -> box {16 words = one 128-column tile, 64 rows}; only used for L2 prefetch
    if (make_tmap_2d(a.qweight, 1, (uint64_t)(a.N / 8), (uint64_t)a.K, (uint64_t)(a.N / 8) * 4, 16, kBK, &tmq, false) ==
        cudaSuccess)
      p.has_tmq = 1;
  }
  switch (layout) {
    case 0: return a.G >= 64 ? dispatch_bt<0>(BT, tm, tmq, p, st) : dispatch_bt<3>(BT, tm, tmq, p, st);
    case 1: return dispatch_bt<1>(BT, tm, tmq, p, st);
    default: return dispatch_bt<2>(BT, tm, tmq, p, st);
  }
}

// ----------------------------------------------------------------------------- grouped (MoE) kernel, host side
bool moe_tc_supported(int K, int N, int G, int block_size, int E) {
  const bool g_ok = G == K || (G >= 32 && (G & (G - 1)) == 0);
  return K > 0 && N > 0 && (K % kBK) == 0 && (N % 8) == 0 && g_ok && (K % G) == 0 && block_size > 0 &&
         (block_size % 16) == 0 && E >= 1 && E <= kMoeTcMaxRuns;
}

// Token tile from the average run: a tile wider than the runs multiplies zeros.  The host never sees the per-expert
// counts (they live on the device and must not be read back).
int moe_tc_token_tile(int n_slots, int E) {
  const int avg = n_slots / E;
  return avg < 48 ? 32 : (avg < 96 ? 64 : 128);
}

template <int BT, int NG>
static cudaError_t launch_moe_tc(const MoeTcParams& p, cudaStream_t st) {
  constexpr size_t smem = TcCfg<BT>::kSmemBytes + kMoeTcTableBytes;
  static_assert(smem <= 232448, "shared memory per CTA");
  auto kern = moe_tc_kernel<BT, NG>;
  static bool attr_set[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !attr_set[dev]) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    if (dev >= 0 && dev < 64) attr_set[dev] = true;
  }
  // the tile count is only known on the device; a run of b blocks has at most b * ceil(block_size / BT) token tiles
  const int64_t bound = (int64_t)((p.N + kTileN - 1) / kTileN) * p.max_blocks * ((p.block_size + BT - 1) / BT);
  const int grid = bound < sm_count() ? (int)bound : sm_count();
  return launch_kernel(kern, dim3(grid), dim3(kTcThreads), smem, st, p);
}

cudaError_t moe_tc_gemm(const void* x, int x_per_slot, const int32_t* qweight, const void* scales, const int32_t* qzeros,
                        const float* topk_w, const int* sorted_ids, const int* expert_ids, const int* num_post_pad,
                        void* y, int n_slots, int topk, int sorted_len, int E, int K, int N, int G, int block_size,
                        int BT, cudaStream_t st) {
  if (!moe_tc_supported(K, N, G, block_size, E)) return cudaErrorNotSupported;
  if (((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(scales)) & 15) != 0) return cudaErrorMisalignedAddress;
  MoeTcParams p;
  p.x = reinterpret_cast<const __half*>(x);
  p.qweight = qweight;
  p.scales = reinterpret_cast<const __half*>(scales);
  p.qzeros = qzeros;
  p.topk_w = topk_w;
  p.sorted_ids = sorted_ids;
  p.expert_ids = expert_ids;
  p.num_post_pad = num_post_pad;
  p.y = reinterpret_cast<__half*>(y);
  p.n_slots = n_slots; p.topk = topk; p.x_per_slot = x_per_slot;
  p.E = E; p.K = K; p.N = N; p.groups = K / G;
  p.g_shift = 31;
  if ((G & (G - 1)) == 0) {   // else G == K: one group
    p.g_shift = 0;
    while ((1 << p.g_shift) < G) ++p.g_shift;
  }
  p.block_size = block_size;
  p.max_blocks = sorted_len / block_size;
  if (p.max_blocks == 0 || n_slots == 0) return cudaSuccess;
  const bool ng2 = G == 32;   // two quantisation groups per 64-row k-step
  switch (BT) {
    case 32: return ng2 ? launch_moe_tc<32, 2>(p, st) : launch_moe_tc<32, 1>(p, st);
    case 64: return ng2 ? launch_moe_tc<64, 2>(p, st) : launch_moe_tc<64, 1>(p, st);
    case 128: return ng2 ? launch_moe_tc<128, 2>(p, st) : launch_moe_tc<128, 1>(p, st);
    default: return cudaErrorInvalidValue;
  }
}

// The kernel's tile list for a host copy of expert_ids: the same run list (built sequentially here, by one warp's
// ballots there) walked by the same moe_tc_tile().
int moe_tc_plan(const int32_t* expert_ids, int n_blocks, int block_size, int E, int N, int BT, int32_t* tiles_out,
                int max_tiles) {
  int run_blk[kMoeTcMaxRuns + 1], run_e[kMoeTcMaxRuns];
  int n = 0;
  for (int i = 0; i < n_blocks; ++i) {
    if (i > 0 && expert_ids[i - 1] == expert_ids[i]) continue;
    if (n <= kMoeTcMaxRuns) run_blk[n] = i;
    if (n < kMoeTcMaxRuns) run_e[n] = expert_ids[i];
    ++n;
  }
  if (n <= kMoeTcMaxRuns) run_blk[n] = n_blocks;
  const int n_runs = n < kMoeTcMaxRuns ? n : kMoeTcMaxRuns;
  MoeTcCursor c{0, 0};
  MoeTcTile t;
  int w = 0;
  for (; moe_tc_tile(run_blk, run_e, n_runs, E, block_size, (N + kTileN - 1) / kTileN, BT, w, c, t); ++w) {
    if (w < max_tiles) {
      tiles_out[4 * w + 0] = t.expert;
      tiles_out[4 * w + 1] = t.pos0;
      tiles_out[4 * w + 2] = t.rows;
      tiles_out[4 * w + 3] = t.nt;
    }
  }
  return w;
}

}  // namespace b200awq
