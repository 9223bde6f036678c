// Shared device helpers for the H100 (sm_90a) AWQ W4A16 kernels.
// Raw PTX wrappers only: mbarrier, TMA (cp.async.bulk[.tensor]), wgmma (warpgroup MMA, descriptors),
// int4 -> fp16 unpack tricks.  No CUTLASS/CuTe, no torch.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200awq {

#ifndef B200AWQ_SM_COUNT_FALLBACK
#define B200AWQ_SM_COUNT_FALLBACK 132
#endif

// ------------------------------------------------------------------------------------ misc
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// streaming 128-bit global load, read-only path, do not keep in L1
__device__ __forceinline__ uint4 ldg_stream_u4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ uint2 ldg_stream_u2(const void* p) {
  uint2 r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
  return r;
}
__device__ __forceinline__ uint32_t ldg_stream_u1(const void* p) {
  uint32_t r;
  asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(r) : "l"(p));
  return r;
}
// L2-only (coherent across SMs) loads for split-K partials written by other CTAs
__device__ __forceinline__ float4 ldcg_f4(const void* p) {
  float4 r;
  asm volatile("ld.global.cg.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ float ldcg_f1(const void* p) {
  float r;
  asm volatile("ld.global.cg.f32 %0, [%1];" : "=f"(r) : "l"(p));
  return r;
}

// Split-K hand-off without sequentially-consistent fences (__threadfence() = fence.sc.gpu = MEMBAR.SC.GPU +
// L1 invalidate, microseconds in the GEMV tail): contributors add with relaxed REDs, synchronise
// on a CTA barrier, ONE thread bumps the ticket with acq_rel at gpu scope (release is cumulative over what the
// barrier ordered before it); the thread that sees the final count acquires, and the barrier after it orders
// the rest of the CTA.
__device__ __forceinline__ void red_add_f32(float* p, float v) {
  asm volatile("red.relaxed.gpu.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}
__device__ __forceinline__ int atom_add_acq_rel(int* p, int v) {
  int old;
  asm volatile("atom.acq_rel.gpu.global.add.s32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(v) : "memory");
  return old;
}
// Cross-CTA completion counters of the decode-program kernel: producers of a result release-add after a CTA
// barrier, consumers poll with an acquiring load (then a CTA barrier orders the rest of the CTA).
__device__ __forceinline__ void red_release_add_s32(int* p, int v) {
  asm volatile("red.release.gpu.global.add.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ int ld_acquire_s32(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint4 ldcg_u4(const void* p) {
  uint4 r;
  asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
  return r;
}
__device__ __forceinline__ float ld_relaxed_f32(const float* p) {
  float v;
  asm volatile("ld.relaxed.gpu.global.f32 %0, [%1];" : "=f"(v) : "l"(p) : "memory");
  return v;
}

// Programmatic dependent launch (PDL): a kernel launched with the programmatic-stream-serialization
// attribute may start while its predecessor is still running.  pdl_trigger() lets OUR successor start
// early; pdl_wait() blocks until the predecessor grid has completed and its writes are visible - it must
// precede every access to memory the predecessor may write (activations, workspace, outputs).  Loads of
// the packed weights (never written on the stream) are issued BEFORE pdl_wait(): consecutive linears
// then stream weights back to back.  Both are no-ops for a normally launched kernel.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

__device__ __forceinline__ void sts_u4(uint32_t saddr, const uint4& v) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(saddr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// ----------------------------------------------------------------------- int4 -> fp16 unpack
// (a & b) | c in one LOP3
__device__ __forceinline__ uint32_t lop3_and_or(uint32_t a, uint32_t b, uint32_t c) {
  uint32_t d;
  asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  return d;
}
__device__ __forceinline__ __half2 u32_as_h2(uint32_t v) { return *reinterpret_cast<__half2*>(&v); }
__device__ __forceinline__ uint32_t h2_as_u32(__half2 v) { return *reinterpret_cast<uint32_t*>(&v); }

// f32 += f16 * f16 (exact product, single fp32 rounding).  sm_90 has no mixed-precision FMA: both fp16 operands are
// widened (exact) and multiplied in fp32 - an fp16 x fp16 product has at most 22 significant bits, so it is exact there.
__device__ __forceinline__ float fhfma(uint16_t a, uint16_t b, float c) {
  return fmaf(__half2float(__ushort_as_half(a)), __half2float(__ushort_as_half(b)), c);
}
__device__ __forceinline__ uint16_t lo16(uint32_t v) { return static_cast<uint16_t>(v & 0xffffu); }
__device__ __forceinline__ uint16_t hi16(uint32_t v) { return static_cast<uint16_t>(v >> 16); }

// One AWQ GEMM-layout word holds 8 output columns of one k.  Pair t = columns (2t, 2t+1) sits in
// bits [4t, 4t+4) of the low / high half-word.  raw pairs as fp16 bit patterns:
//   kind A (t = 0, 2): 0x6400 | q        = 1024 + q
//   kind B (t = 1, 3): 0x6400 | (q << 4) = 1024 + 16 q
struct RawPairs {
  uint32_t p[4];
};
__device__ __forceinline__ RawPairs awq_raw_pairs(uint32_t w) {
  RawPairs r;
  const uint32_t w8 = w >> 8;
  r.p[0] = lop3_and_or(w, 0x000f000fu, 0x64006400u);
  r.p[1] = lop3_and_or(w, 0x00f000f0u, 0x64006400u);
  r.p[2] = lop3_and_or(w8, 0x000f000fu, 0x64006400u);
  r.p[3] = lop3_and_or(w8, 0x00f000f0u, 0x64006400u);
  return r;
}
// Zero-point operands for exact (q - z): kind A uses HSUB2 with (1024 + z); kind B uses
// HFMA2(raw, 1/16, -(64 + z)).  Both results are exact small integers in fp16.
struct ZeroPairs {
  __half2 z[4];
};
__device__ __forceinline__ ZeroPairs awq_zero_pairs(uint32_t zw) {
  RawPairs r = awq_raw_pairs(zw);
  ZeroPairs z;
  const __half2 m16 = __float2half2_rn(-0.0625f);
  z.z[0] = u32_as_h2(r.p[0]);
  z.z[1] = __hmul2(u32_as_h2(r.p[1]), m16);  // -(64 + z), exact
  z.z[2] = u32_as_h2(r.p[2]);
  z.z[3] = __hmul2(u32_as_h2(r.p[3]), m16);
  return z;
}
// Bit-exact dequant of one word: out[t] = fp16((q - z) * s) for column pair t, natural column order.
__device__ __forceinline__ uint4 awq_dequant_word(uint32_t w, const ZeroPairs& z, const uint4& s) {
  RawPairs r = awq_raw_pairs(w);
  const __half2 r16 = __float2half2_rn(0.0625f);
  __half2 d0 = __hsub2(u32_as_h2(r.p[0]), z.z[0]);
  __half2 d1 = __hfma2(u32_as_h2(r.p[1]), r16, z.z[1]);
  __half2 d2 = __hsub2(u32_as_h2(r.p[2]), z.z[2]);
  __half2 d3 = __hfma2(u32_as_h2(r.p[3]), r16, z.z[3]);
  uint4 o;
  o.x = h2_as_u32(__hmul2(d0, u32_as_h2(s.x)));
  o.y = h2_as_u32(__hmul2(d1, u32_as_h2(s.y)));
  o.z = h2_as_u32(__hmul2(d2, u32_as_h2(s.z)));
  o.w = h2_as_u32(__hmul2(d3, u32_as_h2(s.w)));
  return o;
}

// ---------------------------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// non-blocking probe (try_wait may suspend the calling thread for a system-dependent time; a warp whose lanes poll
// DIFFERENT barriers must not let one lane's suspension stall the others: see the converged producer loops)
__device__ __forceinline__ bool mbar_test_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// generic-proxy smem writes -> visible to the async proxy (TMA / wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---------------------------------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}
// 2-D tiled load global -> smem, completion on mbarrier (bytes)
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const void* tmap, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// L2 prefetch of a 2-D tile (no shared-memory destination, no completion tracking)
__device__ __forceinline__ void tma_prefetch_l2_2d(const void* tmap, int c0, int c1) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global [%0, {%1, %2}];" ::"l"(tmap), "r"(c0), "r"(c1) : "memory");
}
// L2 prefetch hint for one 128-byte line (a hint: dropped, not faulted, if the address cannot be translated)
__device__ __forceinline__ void prefetch_l2_line(const void* gsrc) {
  asm volatile("prefetch.global.L2 [%0];" ::"l"(gsrc) : "memory");
}
// L2 prefetch of a contiguous range (size % 16 == 0), no completion tracking
__device__ __forceinline__ void bulk_prefetch_l2(const void* gsrc, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(gsrc), "r"(bytes) : "memory");
}
// 1-D bulk copy global -> smem (no tensor map), completion on mbarrier (bytes); size % 16 == 0
__device__ __forceinline__ void bulk_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
      ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
// 16-byte asynchronous copy global -> smem through L2 only (cp.async, not bulk: per-thread addresses, so the rows of a
// gather may come from anywhere); src_bytes = 0 reads nothing and zero-fills the destination
__device__ __forceinline__ void cp_async_16(uint32_t saddr, const void* gsrc, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(saddr), "l"(gsrc), "r"(src_bytes) : "memory");
}
// One arrival on the mbarrier once every cp.async this thread has issued so far has landed.  .noinc: the arrival is
// part of the count the barrier was initialised with.  The copies are generic-proxy writes: a reader in the async
// proxy (wgmma) fences (fence_proxy_async_smem) after its wait on the barrier.
__device__ __forceinline__ void cp_async_mbar_arrive_noinc(uint64_t* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// L2 cache policies (createpolicy) for the .L2::cache_hint forms below: evict_first for data that is dead once it has
// been read, evict_last for data that must stay in L2 until it is read
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ void bulk_prefetch_l2_hint(const void* gsrc, uint32_t bytes, uint64_t policy) {
  asm volatile("cp.async.bulk.prefetch.L2.global.L2::cache_hint [%0], %1, %2;" ::"l"(gsrc), "r"(bytes), "l"(policy)
               : "memory");
}
__device__ __forceinline__ void bulk_load_1d_hint(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar,
                                                  uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
      ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
      : "memory");
}

// -------------------------------------------------------------------------------------- wgmma
// Warpgroup MMA (sm_90a): four consecutive warps, aligned to a multiple of four, issue one D[64 x N] (+)= A[64 x 16] .
// B[16 x N] together; A and B are read from shared memory through matrix descriptors, D lives in the 128 threads'
// registers.  Accumulator fragment of m64nNk16 (fp32): thread t of the warpgroup (warp w = t / 32, lane l) holds
// d[4 j + r] = D[16 w + l / 4 + 8 (r / 2)][8 j + 2 (l % 4) + (r % 2)].
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// GMMA shared-memory matrix descriptor (sm_90): start>>4 [0,14) | LBO>>4 [16,30) | SBO>>4 [32,46) | base offset [49,52)
// (0: every stage is 1024-byte aligned) | layout type [62,64) (1 = SWIZZLE_128B).  128B-swizzled canonical layouts of
// 16-bit elements: K-major = rows of 64 k (128 B), SBO = stride between 8-row groups; MN-major = 64-element rows along
// MN per k, LBO = stride between 64-element MN blocks, SBO = stride between 8-k groups.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// D (fp32, registers) += A (fp16, smem desc) . B (fp16, smem desc); TA = 1: A is MN-major, 0: K-major; B K-major.
template <int TA>
__device__ __forceinline__ void wgmma_m64n16k16(float (&d)[8], uint64_t da, uint64_t db) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, "
      "%8, %9, 1, 1, 1, %10, 0;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(da), "l"(db), "n"(TA)
      : "memory");
}
template <int TA>
__device__ __forceinline__ void wgmma_m64n32k16(float (&d)[16], uint64_t da, uint64_t db) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "%16, %17, 1, 1, 1, %18, 0;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "n"(TA)
      : "memory");
}
template <int TA>
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[32], uint64_t da, uint64_t db) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, 1, 1, 1, %34, 0;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "n"(TA)
      : "memory");
}
template <int TA>
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t da, uint64_t db) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, 1, 1, 1, %66, 0;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "n"(TA)
      : "memory");
}

template <int N, int TA>
__device__ __forceinline__ void wgmma_f16(float (&d)[N / 2], uint64_t da, uint64_t db) {
  static_assert(N == 16 || N == 32 || N == 64 || N == 128, "token tile");
  if constexpr (N == 16) wgmma_m64n16k16<TA>(d, da, db);
  else if constexpr (N == 32) wgmma_m64n32k16<TA>(d, da, db);
  else if constexpr (N == 64) wgmma_m64n64k16<TA>(d, da, db);
  else wgmma_m64n128k16<TA>(d, da, db);
}

}  // namespace b200awq
