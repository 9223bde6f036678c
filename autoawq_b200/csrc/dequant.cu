// awq_ext.dequantize_weights_cuda replacement: W[K, N] fp16 = (q - z) * s, GEMM layout, bit-exact with
// awq/utils/packing_utils.py:87-102 (exact integer difference, one RN rounding of the product).
// Pure streaming kernel: reads K*N/2 bytes, writes 2*K*N bytes.
#include "common.cuh"
#include "kernels.h"

namespace b200awq {

// Thread = ONE packed word column x ROWS consecutive k-rows of one quantisation group (scales / zeros fetched once).
// Consecutive lanes take consecutive words, so every warp-level load reads 128 contiguous bytes and every warp-level
// store writes 512 contiguous bytes (32 lanes x 16 B): full sectors both ways.  (A thread that owns 4 adjacent words
// instead makes each of its four 16-byte stores hit half of a 32-byte sector.)  ROWS independent
// loads are in flight per thread before the first store.
// (plain write-back stores: the reference's caller hands W straight to torch.matmul, gemm.py:50-54, and whatever part
// of the result is still in L2 - 50 MB on H100, against 33 MB for a 4096 x 4096 W - is read from there)

template <int ROWS>
__global__ void __launch_bounds__(256)
    dequant_gemm_kernel(const int32_t* __restrict__ qweight, const __half* __restrict__ scales,
                        const int32_t* __restrict__ qzeros, __half* __restrict__ out, int K, int N, int G) {
  pdl_trigger();
  pdl_wait();
  const int NW = N >> 3;
  const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int wc = static_cast<int>(gid % NW);
  const int64_t rb = gid / NW;
  const int64_t r0l = rb * ROWS;
  if (r0l >= K) return;
  const int r0 = static_cast<int>(r0l);
  const int g = r0 / G;      // ROWS divides G: the whole run lies in one group
  const ZeroPairs zp = awq_zero_pairs(static_cast<uint32_t>(__ldg(qzeros + (int64_t)g * NW + wc)));
  const uint4 sc = __ldg(reinterpret_cast<const uint4*>(scales + (int64_t)g * N + wc * 8));
  uint32_t q[ROWS];
#pragma unroll
  for (int i = 0; i < ROWS; ++i) q[i] = (r0 + i < K) ? ldg_stream_u1(qweight + (int64_t)(r0 + i) * NW + wc) : 0u;
#pragma unroll
  for (int i = 0; i < ROWS; ++i)
    if (r0 + i < K) *reinterpret_cast<uint4*>(out + (int64_t)(r0 + i) * N + wc * 8) = awq_dequant_word(q[i], zp, sc);
}

cudaError_t dequantize_gemm(const int32_t* qweight, const void* scales, const int32_t* qzeros, void* out, int K,
                            int N, int G, cudaStream_t st) {
  const int NW = N / 8;
  const int rows = (G % 16) == 0 ? 16 : ((G % 8) == 0 ? 8 : 1);
  const int64_t threads = (int64_t)NW * ((K + rows - 1) / rows);
  const int blocks = static_cast<int>((threads + 255) / 256);
  const __half* s = reinterpret_cast<const __half*>(scales);
  __half* o = reinterpret_cast<__half*>(out);
  const dim3 grid(blocks), block(256);
  if (rows == 16) return launch_kernel(dequant_gemm_kernel<16>, grid, block, 0, st, qweight, s, qzeros, o, K, N, G);
  if (rows == 8) return launch_kernel(dequant_gemm_kernel<8>, grid, block, 0, st, qweight, s, qzeros, o, K, N, G);
  return launch_kernel(dequant_gemm_kernel<1>, grid, block, 0, st, qweight, s, qzeros, o, K, N, G);
}

}  // namespace b200awq
