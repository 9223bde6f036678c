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
// Bit identity with M = 1: the kernel keeps the cut of stream_program_kernel<8, 4, 4> - 8 consumer warps, the same
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

constexpr int kSbWarps = 8;   // consumer warps (the cut of stream_program_kernel<8, 4, 4>)
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
  constexpr int NW = kSbWarps, GR = kSbGR;
  extern __shared__ __align__(1024) uint8_t sb_smem[];
  const int NS = NW * spw;
  uint8_t* ring = sb_smem;
  float* part = reinterpret_cast<float*>(sb_smem + (size_t)NS * kSpStageBytes);   // [lmax][8 warps][MT][16]
  float* xsum = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(part) + sb_part_bytes(lmax, MT));   // [NU][MT]
  uint64_t* full = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(xsum) + sb_xsum_bytes(nu_max, MT));
  uint64_t* empty = full + NS;
  SpOp* sdesc = reinterpret_cast<SpOp*>(empty + NS);        // [2] op descriptors, prefetched one op ahead
  int* misc = reinterpret_cast<int*>(sdesc + 2);
  float* wsum = reinterpret_cast<float*>(misc);             // [MT][8] per-warp sums of squares of every row
  int* wfirst = misc + 64;                                  // [NW] first local set each warp touched (-1: none)
  int* wlast = misc + 64 + NW;                              // [NW]
  uint32_t* scta = reinterpret_cast<uint32_t*>(misc + 64 + 2 * NW);   // [2][2] this CTA's unit range
  int* staged_op = misc + 68 + 2 * NW;
  static_assert((69 + 2 * NW) * 4 <= 512 && MT <= 8, "misc area");
  uint32_t* xs = reinterpret_cast<uint32_t*>(sb_smem + sb_fixed_smem(spw, lmax, MT, nu_max));   // [K / 16][MT][8 words]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nblk = gridDim.x, bid = blockIdx.x;
  // a cooperative launch never carries the PDL attribute (then this is a no-op); the tag state below is written by
  // the previous run of this program
  pdl_wait();
  const int base = state[0];

  if (tid == 0) {
    for (int s = 0; s < NS; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 1);
    }
    fence_mbar_init();
    *staged_op = -1;
  }
  if (warp == 1) {
    reinterpret_cast<uint32_t*>(sdesc)[lane] = reinterpret_cast<const uint32_t*>(ops)[lane];
    if (lane < 2) scta[lane] = cta_all[bid + lane];
  }
  __syncthreads();

  if (warp == 0) {
    // ============================================================ producer: the weight stream of ALL ops
    // as in stream_program_kernel (ungated, no L2 prefetch cursor: the defaults there)
    const int w = lane < NW ? lane : 0;
    bool active = lane < NW;
    struct Run {
      uint32_t u, ub;
      int UB, ups;
      const uint8_t* src;
    };
    auto fetch = [&](int op, Run& r) {
      r.u = r.ub = 0;
      r.UB = r.ups = 1;
      r.src = nullptr;
      if (op < n_ops && lane < NW) {
        const uint32_t u0 = cta_all[(size_t)op * (nblk + 1) + bid], u1 = cta_all[(size_t)op * (nblk + 1) + bid + 1];
        const uint32_t nu = u1 - u0;
        r.u = u0 + (uint32_t)((uint64_t)nu * w / NW);
        r.ub = u0 + (uint32_t)((uint64_t)nu * (w + 1) / NW);
        r.UB = ops[op].unit_bytes;
        r.ups = ops[op].ups;
        r.src = ops[op].wstream;
      }
    };
    Run cur, nxt;
    int op = 0;
    fetch(0, cur);
    fetch(1, nxt);
    int stage_i = 0;
    uint32_t ph = 0;
    ProgWatch wd;
    for (;;) {
      while (active && cur.u >= cur.ub) {
        if (++op >= n_ops) {
          active = false;
          break;
        }
        cur = nxt;
        fetch(op + 1, nxt);
      }
      if (!__any_sync(0xffffffffu, active)) break;
      bool issued = false;
      if (active) {
        const int stage = w * spw + stage_i;
        if (mbar_test_wait(&empty[stage], ph ^ 1)) {
          const int n = (int)(cur.ub - cur.u) < cur.ups ? (int)(cur.ub - cur.u) : cur.ups;
          mbar_arrive_expect_tx(&full[stage], (uint32_t)(n * cur.UB));
          bulk_load_1d(ring + (size_t)stage * kSpStageBytes, cur.src + (size_t)cur.u * cur.UB, (uint32_t)(n * cur.UB),
                       &full[stage]);
          cur.u += (uint32_t)cur.ups;
          if (++stage_i == spw) { stage_i = 0; ph ^= 1; }
          issued = true;
        }
      }
      if (!__any_sync(0xffffffffu, issued)) {
        if (__any_sync(0xffffffffu, wd.tick(kWEmpty, op))) break;   // watchdog (warp-uniform): never hang the GPU
        __nanosleep(32);
      }
    }
  } else {
    // ================================================================ consumers
    const int cw = warp - 1;
    const int ct = tid - 32;
    const int g = lane >> 2, tig = lane & 3;
    const int m0 = 2 * tig, m1 = 2 * tig + 1;   // tokens of this lane's accumulators (d0 / d2 and d1 / d3)
    int stage_i = 0;
    uint32_t ph = 0;

    for (int op = 0; op < n_ops; ++op) {
      const SpOp* o = sdesc + (op & 1);
      const int K = o->K, N = o->N, NU = o->NU, F = o->F, UB = o->unit_bytes, ups = o->ups, mode = o->mode;
      const uint32_t u0 = scta[(op & 1) * 2], u1 = scta[(op & 1) * 2 + 1];
      const uint32_t nu = u1 - u0;
      const uint32_t ua = u0 + (uint32_t)((uint64_t)nu * cw / NW), ub = u0 + (uint32_t)((uint64_t)nu * (cw + 1) / NW);
      const int set0 = (int)(u0 / NU);
      const __half* bias = o->bias;
      __half* y = o->y;
      __half* act_out = o->act_out;
      SP_STAMP(0);

      // ---- stage M rows: per row exactly the M = 1 staging (thread t: 8 consecutive k per pass, k = 2048 pass + 8 t;
      //      sums of squares in the order of aux.cu's rmsnorm_kernel).  The (row, pass) items are taken in batches of
      //      4 so that four loads are in flight before the first tag is looked at.
      {
        const int uk_shift = o->uk_shift;
        const int seg = (1 << uk_shift) >> 3;
        const bool from_row = o->src_op >= 0;
        const uint32_t* row0 = from_row ? rows + (size_t)(o->src_op % kSpRows) * M * row_stride + o->src_off : nullptr;
        const uint32_t want = from_row ? sp_tag(base, o->src_op) : 0u;
        const __half* src = o->src;
        const int64_t ldx = o->ldx;
        const bool norm = o->prologue == kProRmsnorm;
        const __half* nw = o->norm_w;
        const int cb_first = cw * 256;
        const int P = cb_first < K ? (K - cb_first + kSpStagePass - 1) / kSpStagePass : 0;   // passes per row
        const int items = P * M;
        auto frag_ptr = [&](int c, int m) { return xs + ((size_t)(c >> 4) * MT + m) * 8 + ((c >> 3) & 1); };
        auto unit_sums = [&](int c, int m, bool ok, const uint32_t (&h)[4]) {
          float sx = 0.f;
          if (ok) {
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const float2 f = __half22float2(u32_as_h2(h[q]));
              sx += f.x + f.y;
            }
          }
          for (int d = 1; d < seg; d <<= 1) sx += __shfl_xor_sync(0xffffffffu, sx, d);
          if (ok && (lane & (seg - 1)) == 0) xsum[(c >> uk_shift) * MT + m] = sx;
        };
        float ss = 0.f;
        for (int q0 = 0; q0 < items; q0 += 4) {       // warp-uniform trip counts
          uint4 v0[4], v1[4];
#pragma unroll
          for (int b = 0; b < 4; ++b) {
            const int q = q0 + b, m = q / (P > 0 ? P : 1), c = cb_first + (q - m * P) * kSpStagePass + lane * 8;
            if (q < items && c < K) {
              if (from_row) {
                v0[b] = ld_relaxed_u4(row0 + (size_t)m * row_stride + c);
                v1[b] = ld_relaxed_u4(row0 + (size_t)m * row_stride + c + 4);
              } else {
                v0[b] = ldg_stream_u4(src + m * ldx + c);
              }
            }
          }
#pragma unroll
          for (int b = 0; b < 4; ++b) {
            const int q = q0 + b;
            if (q >= items) break;                                       // warp-uniform
            const int m = q / P, p = q - m * P;
            const int c = cb_first + p * kSpStagePass + lane * 8;
            const bool ok = c < K;
            uint32_t h[4] = {0u, 0u, 0u, 0u};
            if (ok) {
              if (from_row) {
                const uint32_t* row = row0 + (size_t)m * row_stride;
                ProgWatch wd;
                for (;;) {
                  const uint4 a = v0[b], d = v1[b];
                  if ((a.x >> 16) == want && (a.y >> 16) == want && (a.z >> 16) == want && (a.w >> 16) == want &&
                      (d.x >> 16) == want && (d.y >> 16) == want && (d.z >> 16) == want && (d.w >> 16) == want)
                    break;
                  if (wd.tick(kWCopy, op)) break;
                  v0[b] = ld_relaxed_u4(row + c);
                  v1[b] = ld_relaxed_u4(row + c + 4);
                }
                h[0] = (v0[b].x & 0xffffu) | (v0[b].y << 16);
                h[1] = (v0[b].z & 0xffffu) | (v0[b].w << 16);
                h[2] = (v1[b].x & 0xffffu) | (v1[b].y << 16);
                h[3] = (v1[b].z & 0xffffu) | (v1[b].w << 16);
              } else {
                h[0] = v0[b].x; h[1] = v0[b].y; h[2] = v0[b].z; h[3] = v0[b].w;
              }
              uint32_t* dst = frag_ptr(c, m);
#pragma unroll
              for (int k = 0; k < 4; ++k) {
                dst[2 * k] = h[k];
                const float2 f = __half22float2(u32_as_h2(h[k]));
                ss += f.x * f.x + f.y * f.y;
              }
            }
            if (!norm) unit_sums(c, m, ok, h);
            if (p == P - 1) {                                            // row m done: this warp's sum of squares
              if (norm) {
                const float sw = prog_warp_sum(ss);
                if (lane == 0) wsum[m * 8 + cw] = sw;
              }
              ss = 0.f;
            }
          }
        }
        if (cb_first >= K && norm && lane == 0)                          // a warp without k of its own
          for (int m = 0; m < M; ++m) wsum[m * 8 + cw] = 0.f;
        SP_STAMP(1);
        if (norm) {
          named_bar_sync_gv(1, NW * 32);
          __half* xout = o->xout;
          int xlo = 0, xhi = 0;
          if (xout != nullptr) {
            const int u8 = K >> 3;
            xlo = (int)((int64_t)u8 * bid / nblk) << 3;
            xhi = (int)((int64_t)u8 * (bid + 1) / nblk) << 3;
          }
          for (int q = 0; q < items; ++q) {
            const int m = q / P, p = q - m * P;
            const int c = cb_first + p * kSpStagePass + lane * 8;
            const bool ok = c < K;
            float tot = 0.f;
#pragma unroll
            for (int i = 0; i < kSpStageWarps; ++i) tot += wsum[m * 8 + i];
            const float rs = rsqrtf(tot / static_cast<float>(K) + o->eps);
            uint32_t h[4] = {0u, 0u, 0u, 0u};
            if (ok) {
              uint32_t* dst = frag_ptr(c, m);
              const uint4 wv = __ldg(reinterpret_cast<const uint4*>(nw + c));
#pragma unroll
              for (int k = 0; k < 4; ++k) {
                const float2 a = __half22float2(u32_as_h2(dst[2 * k]));
                const float2 wk = __half22float2(u32_as_h2((&wv.x)[k]));
                h[k] = h2_as_u32(__halves2half2(__float2half_rn(a.x * rs * wk.x), __float2half_rn(a.y * rs * wk.y)));
                dst[2 * k] = h[k];
              }
              if (c >= xlo && c < xhi)
                *reinterpret_cast<uint4*>(xout + (size_t)m * K + c) = make_uint4(h[0], h[1], h[2], h[3]);
            }
            unit_sums(c, m, ok, h);
          }
        }
        named_bar_sync_gv(1, NW * 32);
      }
      if (ct == 0) st_release_cta_smem(staged_op, op);
      SP_STAMP(2);
      if (cw == 0 && op + 1 < n_ops) {
        SpOp* dn = sdesc + ((op + 1) & 1);
        if (lane < 8) cp_async_16(reinterpret_cast<uint8_t*>(dn) + lane * 16, reinterpret_cast<const uint8_t*>(ops + op + 1) + lane * 16);
        else if (lane < 10)
          cp_async_4(scta + ((op + 1) & 1) * 2 + (lane - 8), cta_all + (size_t)(op + 1) * (nblk + 1) + bid + (lane - 8));
      }

      // ---- this warp's run of units: the split and fold order of the M = 1 kernel, two tokens per lane
      {
        int s_cur = (int)(ua / NU), j = (int)(ua - (uint32_t)s_cur * NU);
        float ylo0 = 0.f, yhi0 = 0.f, ylo1 = 0.f, yhi1 = 0.f;
        int first_ls = -1, last_ls = -1;
        auto flush = [&]() {
          const int ls = s_cur - set0;
          float* p = part + ((size_t)ls * NW + cw) * MT * 16;
          if (m0 < M) {
            p[m0 * 16 + g] = ylo0;
            p[m0 * 16 + g + 8] = yhi0;
          }
          if (m1 < M) {
            p[m1 * 16 + g] = ylo1;
            p[m1 * 16 + g + 8] = yhi1;
          }
          if (first_ls < 0) first_ls = ls;
          last_ls = ls;
          ylo0 = yhi0 = ylo1 = yhi1 = 0.f;
        };
        for (uint32_t u = ua; u < ub; u += ups) {
          const int n = (int)(ub - u) < ups ? (int)(ub - u) : ups;
          const int stage = cw * spw + stage_i;
          prog_mbar_wait(&full[stage], ph, kWFull, op);
          if (u == ua) SP_STAMP(3);
          const uint8_t* st = ring + (size_t)stage * kSpStageBytes;
          auto apply = [&](const float (&t_lo)[2], const float (&t_hi)[2]) {
            ylo0 += t_lo[0];
            yhi0 += t_hi[0];
            ylo1 += t_lo[1];
            yhi1 += t_hi[1];
            if (++j == NU) {
              flush();
              j = 0;
              ++s_cur;
            }
          };
          const int j0 = j;
          if (F == 8) sb_chunk<8, GR, MT>(st, UB, n, xs, xsum, j0, NU, lane, M, apply);
          else if (F == 4) sb_chunk<4, GR, MT>(st, UB, n, xs, xsum, j0, NU, lane, M, apply);
          else sb_chunk<2, GR, MT>(st, UB, n, xs, xsum, j0, NU, lane, M, apply);
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty[stage]);
          if (++stage_i == spw) { stage_i = 0; ph ^= 1; }
        }
        if (j != 0 && ua < ub) flush();
        if (lane == 0) {
          wfirst[cw] = first_ls;
          wlast[cw] = last_ls;
        }
      }
      SP_STAMP(4);
      if (cw == 0) cp_async_wait_all();
      named_bar_sync_gv(1, NW * 32);
      SP_STAMP(5);

      // ---- finish: per token, the warps' partial sums in a fixed order, publish (fp16 | tag) into the token's row
      {
        const int nsets = nu == 0 ? 0 : (int)((u1 - 1) / NU) - set0 + 1;
        const uint32_t tagw = sp_tag(base, op) << 16;
        uint32_t* out_rows = rows + (size_t)(op % kSpRows) * M * row_stride;
        const int per_set = 8 * M;
        for (int t = ct; t < nsets * per_set; t += NW * 32) {
          const int ls = t / per_set, r = t - ls * per_set, m = r >> 3, gg = r & 7;
          float lo = 0.f, hi = 0.f;
#pragma unroll
          for (int w = 0; w < NW; ++w) {
            if (wfirst[w] >= 0 && wfirst[w] <= ls && ls <= wlast[w]) {
              const float* p = part + (((size_t)ls * NW + w) * MT + m) * 16;
              lo += p[gg];
              hi += p[gg + 8];
            }
          }
          int clo, chi;
          sp_cols(mode, N, set0 + ls, gg, clo, chi);
          if (bias != nullptr) {
            lo += __half2float(bias[clo]);
            hi += __half2float(bias[chi]);
          }
          const __half hlo = __float2half_rn(lo), hhi = __float2half_rn(hi);
          uint32_t* out_row = out_rows + (size_t)m * row_stride;
          if (mode == 0) {
            st_relaxed_u32(out_row + clo, tagw | __half_as_ushort(hlo));
            st_relaxed_u32(out_row + chi, tagw | __half_as_ushort(hhi));
          } else {
            const float gf = __half2float(hlo), uf = __half2float(hhi);
            const __half a = __float2half_rn(gf / (1.f + __expf(-gf)) * uf);
            st_relaxed_u32(out_row + clo, tagw | __half_as_ushort(a));
            if (act_out != nullptr) act_out[(size_t)m * (N >> 1) + clo] = a;
          }
          y[(size_t)m * N + clo] = hlo;
          y[(size_t)m * N + chi] = hhi;
        }
      }
      SP_STAMP(6);
    }
  }

  __syncthreads();
  if (tid == 0) {
    __threadfence();
    if (atomicAdd(&state[1], 1) == nblk - 1) {
      state[1] = 0;
      state[0] = (base + n_ops) % 65535;
    }
  }
}

}  // namespace b200awq
