/* b200awq.h - C ABI of the H100 (sm_90a) AWQ W4A16 linear path.
 *
 * This is the drop-in boundary: a plain C shared library (libb200awq.so) whose entry points are what a
 * replacement for the reference's `awq_ext` / `awq_v2_ext` pybind modules binds.  No torch types: device
 * pointers, sizes, a CUDA stream.  All pointers are DEVICE pointers unless stated; fp16 tensors are passed
 * as `const void*` (IEEE binary16).  Every function launches asynchronously on `stream`, never
 * synchronises, never allocates (CUDA-graph capturable) and returns 0 on success or a B200AWQ_E* code
 * (b200awq_error_string() explains it; `cudaGetLastError` state is folded into B200AWQ_ECUDA).
 *
 * Reference interface each entry point replaces (file:line under casper-hansen/AutoAWQ @ 88e4c76):
 *   b200awq_dequantize_gemm ...... awq_ext.dequantize_weights_cuda  awq/modules/linear/gemm.py:51-53,100-102
 *                                                                   tests/test_dequantization.py:40-49
 *   b200awq_gemm_forward ......... awq_ext.gemm_forward_cuda        awq/modules/linear/gemm.py:56-58
 *                                   (+ the dequant+matmul branch)   awq/modules/linear/gemm.py:50-54
 *   b200awq_gemv_forward ......... awq_ext.gemv_forward_cuda        awq/modules/linear/gemv.py:177-180
 *                                   awq_ext.gemmv2_forward_cuda     awq/modules/linear/gemv.py:168-176
 *   b200awq_fast_forward ......... awq_v2_ext.gemv_forward_cuda_decode   awq/modules/linear/gemv_fast.py:192-201
 *                                   awq_v2_ext.gemm_forward_cuda_prefill  awq/modules/linear/gemv_fast.py:203-205
 *   b200awq_rmsnorm .............. awq_ext.layernorm_forward_cuda   awq/modules/fused/norm.py:33-36
 *   b200awq_silu_and_mul ......... awq_ext.silu_and_mul             awq/modules/fused/moe.py:76
 *   b200awq_rope_kv .............. RoPE.forward + WindowedCache.update_kv   awq/modules/fused/attn.py:53-86,243-267
 *   b200awq_qk_norm_rope_kv ...... q_norm / k_norm (Qwen3RMSNorm), then as b200awq_rope_kv   attn.py:250-253
 *
 * Tensor layouts (SURVEY.md Appendix A):
 *   GEMM  : qweight [K, N/8] i32 (AWQ interleave), qzeros [K/G, N/8] i32, scales [K/G, N] f16
 *   GEMV  : qweight [N, K/8] i32 (sequential),     qzeros [N, zw] i32,    scales [N, 8*zw] f16
 *   FAST  : qweight [N/4, K] i16,                  szeros [8*zw, N] f16 (= -z*s), scales [8*zw, N] f16
 */
#ifndef B200AWQ_H_
#define B200AWQ_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200AWQ_ABI_VERSION 1

typedef void* b200awq_stream_t; /* cudaStream_t */

enum {
  B200AWQ_OK = 0,
  B200AWQ_EINVAL = 1,      /* bad shape / null pointer / misaligned pointer */
  B200AWQ_EUNSUPPORTED = 2,/* shape outside the implemented envelope (e.g. K % 64 != 0 on the tensor-core path) */
  B200AWQ_EWORKSPACE = 3,  /* workspace missing or too small */
  B200AWQ_ECUDA = 4,       /* a CUDA runtime / driver call failed */
  B200AWQ_EARCH = 5        /* device is not sm_90 */
};

int b200awq_abi_version(void);
const char* b200awq_error_string(int code);
/* last CUDA error text seen by this library on the calling thread ("" if none) */
const char* b200awq_last_cuda_error(void);

/* Bytes of scratch the forward entry points may need for (M, K, N): 16 KB of tickets + min(M, 128) * N 64-bit words
 * (split-K partials: packed fixed-point sum + tile count per element for the M <= 8 GEMV, fp32 sums of up to 256 token
 * rows otherwise).
 * The caller allocates once (zero-initialised!) and passes it to every call; the library restores the
 * all-zero ticket state before each kernel exits, so one buffer serves any number of calls on one stream. */
size_t b200awq_workspace_bytes(int M, int K, int N);

/* W[K, N] f16 = (nibble - zero_nibble) * scale, bit-exact with awq/utils/packing_utils.py:87-102. */
int b200awq_dequantize_gemm(const int32_t* qweight, const void* scales, const int32_t* qzeros, void* out_f16,
                            int K, int N, int group_size, b200awq_stream_t stream);

/* Y[M, N] f16 = X[M, K] f16 . deq(W) (+ bias[N] f16 if non-null), GEMM layout.  ldx = row pitch of X in
 * elements (>= K).  M <= 4 runs the persistent tensor-core GEMV (M <= 8 where the small-M kernel does not apply),
 * 5 <= M <= 128 the small-M wgmma kernel with TMA-staged packed weights, larger M the wgmma GEMM. */
int b200awq_gemm_forward(const void* x, int64_t ldx, const int32_t* qweight, const void* scales,
                         const int32_t* qzeros, const void* bias, void* y, int M, int K, int N, int group_size,
                         void* workspace, size_t workspace_bytes, b200awq_stream_t stream);

/* Same contraction on the GEMV layout (WQLinear_GEMV buffers). */
int b200awq_gemv_forward(const void* x, int64_t ldx, const int32_t* qweight, const void* scales,
                         const int32_t* qzeros, const void* bias, void* y, int M, int K, int N, int group_size,
                         void* workspace, size_t workspace_bytes, b200awq_stream_t stream);

/* Same contraction on the GEMVFast layout (WQLinear_GEMVFast buffers; W = q*s + szeros). */
int b200awq_fast_forward(const void* x, int64_t ldx, const int16_t* qweight, const void* scales,
                         const void* scaled_zeros, const void* bias, void* y, int M, int K, int N, int group_size,
                         void* workspace, size_t workspace_bytes, b200awq_stream_t stream);

/* out[r, :] = x[r, :] * rsqrt(mean(x[r, :]^2) + eps) * weight   (fp32 math, fp16 in/out; out may alias x) */
int b200awq_rmsnorm(const void* x, const void* weight, void* out, int rows, int hidden, float eps,
                    b200awq_stream_t stream);

/* out[r, j] = silu(gate_up[r, j]) * gate_up[r, d + j], j < d  (fp32 math, fp16 in/out) */
int b200awq_silu_and_mul(const void* gate_up, void* out, int rows, int d, b200awq_stream_t stream);

/* LayerNorm (nn.LayerNorm / F.layer_norm on fp16 rows; transformers' CohereLayerNorm when bias is null): for row r of
 * x (pitch ldx elements, >= hidden) into the contiguous out[r, :], K = hidden, fp32 math:
 *   mean = S1 / K                                    S1 = sum of x in the order below
 *   var  = S2 / K                                    S2 = sum of (x - mean)^2 in the same order (a second pass over the
 *                                                    row, not E[x^2] - mean^2: rows whose mean is large against their
 *                                                    spread would cancel in that form)
 *   r    = rsqrtf(var + eps)
 *   out  = fp16(((x - mean) * r) * w [+ b])          rounded once; no bias add when bias is null
 * Every operation is one IEEE fp32 operation (no contraction); r is the device's rsqrtf.  Summation order (both sums):
 * thread t < 256 takes the chunks of 8 consecutive columns c = 8 t + 2048 p, p = 0, 1, ...; within a chunk the pairs
 * (c + 2q, c + 2q + 1), q = 0..3, in order: s = s + (v0 + v1) for S1, s = s + (d0 d0 + d1 d1) for S2 (d = x - mean);
 * the 32 lanes of warp w = t / 32 are summed with the xor butterfly at offsets 16, 8, 4, 2, 1; the 8 warp totals are
 * added to 0 in ascending w.  Requires hidden % 8 == 0, ldx % 8 == 0 and 16-byte aligned x, weight, bias and out
 * (else B200AWQ_EUNSUPPORTED); out must not overlap x. */
int b200awq_layer_norm(const void* x, int64_t ldx, const void* weight, const void* bias, void* out, int rows,
                       int hidden, float eps, b200awq_stream_t stream);

/* GELU, elementwise over rows x n contiguous fp16 values, fp32 math, rounded once (torch's CUDA formulas):
 *   approximate = 1 (F.gelu(x, approximate="tanh"), gelu_pytorch_tanh):
 *       fp16(0.5 x (1 + tanhf(kBeta fma(0.044715, x^3, x)))),  kBeta = fp32(sqrt(2 / pi)), x^3 = (x x) x
 *   approximate = 0 (F.gelu): fp16((0.5 x) (1 + erff(x fp32(sqrt(1/2)))))
 * out may not partially overlap x (out == x is fine). */
int b200awq_gelu(const void* x, void* out, int rows, int n, int approximate, b200awq_stream_t stream);

/* ---- MoE (awq/modules/fused/moe.py:45-171; Mixtral: awq/models/mixtral.py:129-158) ------------------------------
 * b200awq_topk_softmax ............ awq_ext.topk_softmax        moe.py:162-167 (fused_topk)
 * b200awq_moe_align_block_size .... awq_ext.moe_alig_block_size moe.py:131-133
 * b200awq_grouped_gemm_forward .... awq_ext.grouped_gemm_forward moe.py:60-89
 *
 * topk_softmax: softmax over the E experts (fp32), the topk largest probabilities per token (ties: lower expert),
 * not renormalised; token_expert_indices[m, k] = k * M + m.
 * moe_align_block_size: flattened slot indices (token * topk + k) grouped by expert in ascending order, every
 * expert's run padded with `numel` to a multiple of block_size; expert_ids[b] = expert of block b;
 * *num_tokens_post_pad = total padded length.  sorted_ids holds numel + E * (block_size - 1) entries, expert_ids
 * numel + E.
 * grouped_gemm_forward: y [T * topk, N] f16; for every real slot id in sorted_ids[0 .. *num_tokens_post_pad),
 * y[id] = x_row(id) . deq(W[expert_ids[pos / block_size]]) (* topk_weights[id] if mul_weights), x_row(id) = x[id /
 * topk] when x_rows_per_token == 1 (x [T, 1, K]) and x[id] when x_rows_per_token == topk (x [T, topk, K]).
 * qweight [E, K, N/8], scales [E, K/G, N], qzeros [E, K/G, N/8] (stacked GEMM layout).  block_size is 16 at the
 * reference's call site (moe.py:54-56) and must be a multiple of 8 here.  Three kernels:
 *   - prefill-sized calls, T * topk >= 20 * E (an average of 20 slots per expert), with K % 64 == 0, G a power of two
 *     >= 32 or G == K, block_size % 16 == 0, E <= 256, x and scales 16-byte aligned: the grouped tensor-core kernel
 *     (wgmma), one tile per 128 output columns x 32 / 64 / 128 sorted slots of one expert.  It builds its tile list on
 *     the device from expert_ids, which must list every expert's blocks contiguously (as moe_align_block_size
 *     writes them); no workspace, no host read-back, CUDA-graph capturable with routing that changes between replays.
 *   - otherwise, with a workspace of b200awq_workspace_bytes(sorted_len, K, N) bytes (zero-initialised, left zero;
 *     the per-op workspace serves) and N % 256 == 0, K % 64 == 0, G in {64, 128, K}: the persistent TMA-ring GEMV, one
 *     job per 8 sorted slots (the decode case);
 *   - otherwise a register-staged grouped kernel (K % 512 == 0, N % 32 == 0, G % 64 == 0), else B200AWQ_EUNSUPPORTED.
 * Knob 12 = 2 forces the third kernel, 3 the first wherever its shape conditions hold, 1 excludes the first. */
int b200awq_topk_softmax(const float* gating_output, float* topk_weights, int32_t* topk_ids,
                         int32_t* token_expert_indices, int M, int E, int topk, b200awq_stream_t stream);
int b200awq_moe_align_block_size(const int32_t* topk_ids, int numel, int num_experts, int block_size,
                                 int32_t* sorted_ids, int32_t* expert_ids, int32_t* num_tokens_post_pad,
                                 b200awq_stream_t stream);
int b200awq_grouped_gemm_forward(const void* x, int x_rows_per_token, const int32_t* qweight, const void* scales,
                                 const int32_t* qzeros, const float* topk_weights, const int32_t* sorted_ids,
                                 const int32_t* expert_ids, const int32_t* num_tokens_post_pad, void* y, int T, int topk,
                                 int sorted_len, int E, int K, int N, int group_size, int mul_weights, int block_size,
                                 void* workspace, size_t workspace_bytes, b200awq_stream_t stream);

/* Host-side tile list of the grouped tensor-core kernel (no GPU needed, no CUDA call): for a HOST copy of the first
 * n_blocks = num_tokens_post_pad / block_size entries of expert_ids, the tiles in the kernel's order, 4 ints each:
 * {expert, first sorted position, rows (<= BT), 128-column tile}.  Token tiles of one (expert, column tile) are
 * adjacent; CTA b of a grid of min(*n_tiles, sm_count) CTAs runs tiles b, b + grid, ...  At most max_tiles tiles are
 * written; *n_tiles is the full count.  BT in {32, 64, 128}; block_size % 16 == 0 and E <= 256 as the kernel. */
int b200awq_moe_tc_plan(const int32_t* expert_ids_host, int n_blocks, int block_size, int E, int N, int BT, int sm_count,
                        int32_t* tiles_out, int max_tiles, int* n_tiles);

/* Host-side plan of the small-M tensor-core kernel (no GPU needed): for a GEMM-layout call of this shape on a device with
 * `sm_count` SMs, *grid = number of CTAs and *pairs_per_tile = K / 128; CTA b owns the contiguous range
 * [T b / grid, T (b + 1) / grid) of the linearised (128-column tile, 128-row pair) sequence, T = (N / 128) * (K / 128).
 * `mode` as knob 21.  B200AWQ_EUNSUPPORTED when the shape is outside that kernel's envelope
 * (M <= 128, G >= 64, K % 128 == 0, N % 128 == 0). */
int b200awq_tcq_plan(int M, int K, int N, int group_size, int sm_count, int mode, int* grid, int* pairs_per_tile);

/* Tuning / debug knobs (process-global; used by the micro-benchmarks and layout self-tests).
 *   key 0: GEMV rows per warp override: 32 / 64 / 128 (0 = heuristic)
 *   key 1: tensor-core path split-K override (0 = heuristic)
 *   key 2: M threshold at or below which the GEMV kernels are used (default 8; the GEMM-layout entry point lowers it to 4
 *          wherever the small-M tensor-core kernel of key 19 applies: over the Llama-3-8B linears it is faster from 5
 *          tokens on, measured on H100)
 *   key 3: 1 = the persistent GEMV records per-CTA phase timestamps (read with b200awq_debug_read);
 *          2 = the decode-program kernel records per-op phase timestamps of its first 8 CTAs / 32 ops
 *          (b200awq_debug_read then returns [op][cta][8] uint64 ns: op begin, source row complete, activations
 *          staged, first chunk landed, warp 0 done, all warps done, outputs published, routing published);
 *          3 = b200awq_debug_read returns the decode-program kernel's abort record instead: int32 [0..3] = {code, op,
 *          CTA, aborted} of the first wait that exceeded 0.5 s (every spin loop of that kernel gives up rather than
 *          hang the GPU), then per CTA 10 ints = (code << 16 | op) of the wait each warp abandoned;
 *          9 = the small-M tensor-core kernel (9 <= M <= 128, GEMM layout) records per-CTA phase timestamps
 *          (b200awq_debug_read returns [cta][8] uint64 ns: entry, setup done, first packed stage landed, producers
 *          done, MMA issuer done, last accumulator drained, epilogue done, number of segments)
 *   key 4: 1 = launch every kernel with the programmatic-dependent-launch attribute (the kernels issue
 *          their weight loads before griddepcontrol.wait, so consecutive linears overlap); default 0
 *   key 5: 1 = disable the persistent TMA-ring GEMV (use the register-staged GEMV for every M <= 8 shape)
 *   key 6: 1 = enable the learned next-weight L2 prefetch (the M <= 8 path remembers which weight tensor
 *          followed which in the call sequence and prefetches the successor's packed weights into L2 at the
 *          tail of each kernel); default 0
 *   key 7: 1 = stage the activations in shared memory in the persistent GEMV (M <= 2); default 0
 *   key 8: persistent GEMV L2-prefetch distance + 1 in tiles (0 / 1 = off, the default)
 *   key 9: persistent GEMV ring stages per consumer warp for M = 1 (1 / 2; 0 = default 3); the M = 1 decode program
 *          runs 12 consumer warps when this is 12 (default 8; any other value, 16 included, means 8: a 16-warp CTA
 *          spills on sm_90)
 *   key 10: decode program gate: 0 = ungated (the default: 1.93 vs 1.98 ms per Llama-3-8B step with 2 = gated one op
 *           ahead, H100 at 400 W), n > 0 = weight loads at most n - 1 ops ahead of the staging
 *   key 12: grouped_gemm_forward kernel choice: 1 = never the grouped tensor-core kernel (the decode-sized kernels at
 *           every token count); 2 = always the register-staged grouped kernel; 3 = the grouped tensor-core kernel
 *           wherever its shape conditions hold, whatever the token count
 *   key 18: 1 = the persistent GEMV uses round 1's split-K epilogue (fp32 REDs, tickets, read-back) also at M = 1,
 *           instead of the packed one (one returning 64-bit atomic per element; bit-reproducible)
 *   key 17: 1 = b200awq_comm_all_reduce uses the flag protocol (push, fence, flag, wait, reduce) instead of the default
 *           LL protocol (8-byte words carrying {2 x fp16, call number}: one NVLink hop, no fences)
 *   key 16: decode-program watchdog in seconds (0 = the default 0.5 s): every spin of the program kernels gives up
 *           after this long; raise it under compute-sanitizer / a debugger, where kernels run orders of magnitude slower
 *   key 15: 1 = wrap every launching entry point in an NVTX range named after it (profiler timelines); default 0
 *   key 19: 1 = never use the small-M kernel with TMA-staged packed weights (gemm_tcq_kernel; default: every GEMM-layout
 *           call with 5 <= M <= 128 (M above key 2's threshold), G >= 64, K % 128 == 0, N % 128 == 0 runs it)
 *   key 20: small-M kernel timing experiments (outputs are WRONG while set): bit 0 = producers skip the dequantisation and
 *           the shared-memory stores, bit 1 = producers skip the generic->async proxy fence (the MMA loop itself has
 *           no experiment switch: a runtime condition around wgmma would change its code)
 *   key 21: small-M kernel work cut: 0 = tile-aligned ranges when N / 128 <= SM count (or from 64 tokens on), balanced
 *           (n-tile, k-step pair) ranges otherwise; 1 = always balanced; 2 = tile-aligned whenever possible
 *   key 22: small-M kernel: HBM -> L2 prefetch distance in k-step pairs ahead of the shared-memory ring (0 = off, default)
 *   key 14: decode programs (read at b200awq_program_create): 1 = do not fuse: create returns B200AWQ_EUNSUPPORTED for
 *           any sequence that folds (folding errors are still reported as such) and the caller replays per op, the
 *           reference the fused kernels are held to; any other value = fuse when the sequence fits the kernels
 */
int b200awq_set_knob(int key, int value);
int b200awq_get_knob(int key);
/* Copies the phase timestamps of the last persistent-GEMV launch (knob 3) to HOST memory: per CTA 8 x uint64 ns
 * (globaltimer): [0] kernel entry, [1] after the PDL wait, [2] first tile landed, [3] consumer warp 0 done,
 * [4] all consumer warps done, [5] partial sums added (REDs issued), [6] tickets bumped, [7] finalisation done.
 * Synchronises the device. */
int b200awq_debug_read(void* host_dst, size_t bytes);

/* ---------------------------------------------------------------------------------------------------------
 * Decode programs: the chain of operator calls of one decode step (M = 1), recorded once and executed by ONE
 * persistent kernel whose weight stream runs across op boundaries (csrc/program.cu).  The op list is exactly
 * the sequence of calls the reference's fused block makes through awq_ext (awq/modules/fused/block.py:117-170,
 * awq/modules/fused/mlp.py:41-55): RMSNorm -> linear -> ... -> SiLU*mul -> linear.  After a run every buffer
 * named by the ops holds what the per-op entry points above would have left there.
 *
 *   RMSNORM       : x = input row [K], weight [K], y = output [K], eps           (K = hidden); M > 1 rows at
 *                   pitch ldx (0 or K: contiguous; any other pitch, e.g. the c_kv slice of MLA rows, is
 *                   B200AWQ_EUNSUPPORTED: the caller replays per op)
 *   SILU_AND_MUL  : x = gate|up [2K], y = output [K]                             (K = d)
 *   LINEAR_GEMM   : as b200awq_gemm_forward (GEMM layout)
 * b200awq_program_create returns B200AWQ_EUNSUPPORTED when the sequence does not fit the fused kernel (M != 1,
 * a shape outside the stream format's or the kernel's envelope, a glue op whose output no later linear reads,
 * aliasing the kernel's ordering cannot honour); the caller then issues the ops one by one.  Pointers are captured,
 * not copied: the tensors must stay alive and in place for the life of the program.  Create / destroy allocate and
 * copy (not capturable); run only enqueues a memset + one kernel on `stream` (capturable).  A program is not
 * re-entrant: one run in flight at a time.
 *
 *   SPARSE_MOE    : a whole sparse-MoE block (awq/modules/fused/moe.py:26-89, FusedSparseMoeBlock.forward):
 *                   x = normed input row [H], y = output [H], K = H, weight = a b200awq_moe_t descriptor; the op's
 *                   result is sum_k fp16(w_k * down_k(silu_mul(gate_up_k(x)))) over the top_k routed experts.
 *     Folding: two kernel ops.  (1) gate|up with a routing prologue: every CTA computes the router logits (fp32 dots,
 *     rounded to fp16 like nn.Linear), softmax and top-k with topk_softmax's arithmetic (ties: lower expert) and the
 *     optional fp32 renormalisation from its staged row, then streams the top_k selected experts' gate|up slices with
 *     SiLU*mul fused (top_k x I activation words, slot-major).  (2) down with K' = top_k I: unit j of a set reads slot
 *     j / (I / 128)'s expert; each slot's fp32 sum is multiplied by its routing weight and rounded to fp16 (as
 *     grouped_gemm_forward(mul_weights) does), the slots are summed in fp32 in slot order and rounded once (torch.sum).
 *     After a run every buffer of the descriptor holds what the per-op sequence (gate matmul, topk_softmax,
 *     renormalisation, moe_alig_block_size, grouped_gemm_forward, silu_and_mul, grouped_gemm_forward(mul_weights),
 *     sum) would leave there; routing tensors for M = 1.
 *     Envelope (else B200AWQ_EUNSUPPORTED, the caller replays per op): M = 1, knob 14 != 1, E <= 64, top_k <= 8, the
 *     per-expert shapes in the stream format, at most 32 16-column sets of the gate|up op and 32 (set, slot) partial
 *     rows of the down op per CTA, and the activations of the longest K (top_k I for down) in shared memory next to the
 *     8-warp x 4-stage weight ring (b200awq_moe_plan below says which).
 *     Memory: the program keeps a stream-format copy of every expert of both stacked tensors (about the size of the
 *     packed checkpoint again: ~24 GB for Mixtral-8x7B's 32 layers).
 *
 *   ADD           : the decoder block's residual add (awq/modules/fused/block.py:50-52,117-118): y[M, K] = x + weight,
 *                   elementwise fp16 with torch's rounding, fp16(float(x) + float(weight)); x, weight, y = M contiguous
 *                   rows of K (null: B200AWQ_EINVAL; K % 8 != 0 or a pointer not 16-byte aligned: B200AWQ_EUNSUPPORTED).
 *     Folding: an ADD adds no kernel op.  It folds into the epilogue of the kernel op that produced one operand, which
 *     must be the op recorded immediately before it (a linear, or the down op of a SPARSE_MOE) and whose whole output
 *     (all M rows x N, N = K) that operand is.  The other operand, the residual, is either a buffer no op of the program
 *     writes, or the output of an older op j of the program at most 4 kernel ops back (its published row).  Ops j + 4,
 *     j + 8, ... publish into that row again; for the first of them after the producer i, k, some op in (i, k] must
 *     stage the whole published row of an op >= i that has at least 16 columns per SM, so that no CTA can overwrite a
 *     residual word before every CTA has read it (tests/test_stream_residual_model.py; b200awq_program_plan below).  The producer's
 *     hand-off row then carries the sum: later ops that read the ADD's output read the sum, and a later op that reads
 *     the producer's raw output is rejected.  Both the producer's y and the ADD's y are stored.  Everything else is
 *     B200AWQ_EUNSUPPORTED and the caller replays per op: an ADD after a glue op or another ADD, after a gate|up whose
 *     output only SiLU*mul reads, with both operands external, in place, with a residual out of the window or one the
 *     program overwrites.  M = 1 runs 8 consumer warps x 4 stages (knob 9 ignored); M > 1 the batched kernel.
 *
 *   ROPE_KV       : the start of the attention block (awq/modules/fused/attn.py:243-267): rotate q and k of the fused
 *                   qkv output with RoPE.forward and write k and v into the WindowedCache row update_kv writes.
 *                   x = qkv [M, (H + 2 KV) D] f16 at row pitch ldx, weight = a b200awq_rope_t descriptor (below), M, and
 *                   N = (H + 2 KV) D.  As b200awq_rope_kv.
 *     Folding: a ROPE_KV adds no kernel op.  It folds into the finish of the linear recorded immediately before it, whose
 *     whole output must be its qkv: that linear is re-laid-out in stream mode 2 (rotary pairs, below), so the thread that
 *     finishes column i < R/2 of a head also holds column i + R/2 and rotates the pair in registers (a pass-through pair
 *     is copied).  Partial rotary (rotary_dim < D) folds like full rotary, at M = 1 and at max_tokens > 1.  The
 *     linear's y and published row keep the raw qkv values.  B200AWQ_EUNSUPPORTED (the caller replays per op) when the op before it is
 *     not a plain linear (a glue op, an ADD, a gate|up whose product SiLU*mul reads, a SPARSE_MOE) or already carries an
 *     ADD, when N != (H + 2 KV) D or D % 16 != 0, or when any other op of the program reads or writes q_out or the
 *     caches.
 *
 *   QK_NORM_ROPE_KV : ROPE_KV preceded by the per-head RMSNorm of q and k that Qwen3's attention applies
 *                   (Qwen3RMSNorm q_norm / k_norm, awq/modules/fused/attn.py:250-253).  x, M, N as ROPE_KV, weight = a
 *                   b200awq_qk_norm_rope_t descriptor (below).  As b200awq_qk_norm_rope_kv.
 *     Folding: exactly ROPE_KV's rules and rejections (on the embedded descriptor), plus B200AWQ_EINVAL for a null norm
 *     weight and B200AWQ_EUNSUPPORTED for one that is not 16-byte aligned or that an op of the program writes, or for
 *     partial rotary (rotary_dim not 0 or D).  A head's
 *     sums of squares span sets that other CTAs may finish: every CTA publishes the partials of its sets into a buffer
 *     the program owns, then waits for all partials of each q / k head it finishes (DESIGN.md 3.5g).
 *
 *   QWEN3_MOE     : a Qwen3-MoE expert block as transformers' Qwen3MoeSparseMoeBlock computes it (one token row),
 *                   x, y, K and weight as SPARSE_MOE (renormalize = norm_topk_prob).  Arithmetic:
 *                   logits = fp16(x Wg^T); p = softmax_fp32(logits) (topk_softmax's arithmetic); top_k, ties to the lower
 *                   expert; w = p_k / sum p_k in fp32 when renormalize; w16 = fp16(w).  Then for each selected expert in
 *                   ASCENDING EXPERT ID: a = fp16(fp16(silu(g)) * u) of its gate|up, y = fp16(W2 a), c = fp16(y * w16),
 *                   out = fp16(out + c) from out = 0.  The descriptor's buffers hold what SPARSE_MOE's do, except
 *                   topk_weights, which holds the fp16 w16 [top_k] (the pointer is reinterpreted), and down, which holds
 *                   the per-slot c.
 *     Folding: two kernel ops, as SPARSE_MOE.  The router logits are computed once across the grid (CTA c computes the
 *     logits e = c mod grid) and exchanged through tagged words the program owns; every CTA then runs the routing from
 *     all E logits (DESIGN.md 3.5h).  Envelope (else B200AWQ_EUNSUPPORTED): SPARSE_MOE's with E <= 128
 *     (b200awq_qwen3_moe_plan below).  An ADD right after it folds into its down op.
 *
 *   DEEPSEEK_MOE  : a DeepSeek-MoE expert block as transformers' DeepseekV2Moe / DeepseekV3MoE computes it over
 *                   WQLinear_GEMM experts (one token row): routed experts plus one dense shared expert every token runs.
 *                   x, y, K as SPARSE_MOE; weight = a b200awq_deepseek_moe_t descriptor (below).  Arithmetic:
 *                   l = fp32(x) . fp32(Wg)^T, kept in fp32.
 *                   scoring 0 (softmax, V2 "greedy"): p = softmax_fp32(l); the top_k largest p (ties to the lower
 *                     expert); w = p_k * routed_scaling_factor.
 *                   scoring 1 (sigmoid, V3 "noaux_tc"): s = sigmoid(l), c = s + bias; each of the n_group groups of
 *                     E / n_group consecutive experts scores the sum of its two largest c; the topk_group best groups
 *                     stay (ties to the lower group) and every other c becomes 0.0; the top_k largest masked c (ties to
 *                     the lower expert); w = s_k, w = w / (sum w + 1e-20) when norm_topk_prob, w = w * routed_scaling_factor,
 *                     all in fp32.
 *                   Routed experts in ASCENDING EXPERT ID: a = fp16(fp16(silu(g)) * u), y = fp16(W2 a),
 *                   c = fp16(fp32(y) * w), r = fp16(r + c) from r = 0.  Shared expert (gate|up concatenated along N):
 *                   a_s = fp16(fp16(silu(g_s)) * u_s), y_s = fp16(W2s a_s).  y = fp16(r + y_s).
 *                   The embedded descriptor's buffers hold what QWEN3_MOE's do, except: logits holds the fp32 l [E]
 *                   and topk_weights the fp32 w [top_k] (pointers reinterpreted / as declared), gate_up holds
 *                   [top_k 2I + 2 I_s] (the slots, then the shared gate|up) and act [top_k I + I_s] (the slots, then a_s);
 *                   down holds the per-slot c.  renormalize is ignored (norm_topk_prob below).
 *     Folding: two kernel ops.  gate|up has top_k 2I + 2 I_s columns, the shared sets after the slots; their weights do
 *     not depend on the routing, so the producer streams them while the router logits are exchanged.  down reads
 *     K' = top_k I + I_s (the shared expert concatenated along K after the slots) and keeps the shared expert's sum in
 *     a partial row of its own.  Logit exchange as QWEN3_MOE, with the unrounded fp32 logits (DESIGN.md 3.5i).
 *     Envelope (else B200AWQ_EUNSUPPORTED): M = 1, E <= 128, top_k <= 8, the shapes of b200awq_deepseek_moe_plan below.
 *     A program that mixes SPARSE_MOE, QWEN3_MOE and DEEPSEEK_MOE blocks replays per op.  An ADD right after it folds
 *     into its down op.
 *
 *   MLA_ROPE      : the start of DeepSeek-V2 / V3 multi-head latent attention without a q LoRA, on the fused
 *                   q_proj | kv_a_proj_with_mqa output row [q (H (Dn + Dr)) | c_kv (C) | k_pe (Dr)]: x = that row [M, N]
 *                   at row pitch ldx, N = H (Dn + Dr) + C + Dr, weight = a b200awq_mla_t descriptor (below).  As
 *                   b200awq_mla_rope.
 *   MLA_KV        : the kv_b_proj output [M, H (Dn + Dv)] into the cache: x, ldx, weight as MLA_ROPE, N = H (Dn + Dv).
 *                   As b200awq_mla_kv.
 *     Folding: neither adds a kernel op.  Each folds into the finish of the linear recorded immediately before it, whose
 *     whole output must be its row.  The linear before an MLA_ROPE is re-laid-out in stream
 *     mode 3 (adjacent pairs, below), so the thread that finishes column 2i also holds 2i + 1 and rotates the pair in
 *     registers; its y and published row keep the raw values, so kv_a_layernorm is the RMSNORM op recorded on the c_kv
 *     slice of that y (a source inside the previous op's output).  B200AWQ_EUNSUPPORTED (the caller replays per op) when
 *     M != 1, the op before is not a plain linear, N does not match the descriptor, Dn, Dr, Dv or C is not a
 *     multiple of 16, or any other op reads or writes q_out or the caches or writes pos / freqs; the MLA_ROPE and MLA_KV
 *     ops of one layer may share k_cache (they write disjoint columns).  A program with MLA ops runs the DeepSeek-MoE
 *     kernel's configuration (a program that also holds SPARSE_MOE or QWEN3_MOE blocks replays per op).
 *
 *   MLA_K_ROPE    : MLA with a q LoRA (DeepSeek-V2 / V2.5 / V3, MiniCPM3), on the fused q_a_proj | kv_a_proj_with_mqa
 *                   output row [q_a (Cq) | c_kv (C) | k_pe (Dr)]: x = that row [M, N] at pitch ldx, Cq = N - C - Dr > 0,
 *                   weight = a b200awq_mla_t.  Writes only k_cache (q_out may be null).  As b200awq_mla_k_rope with
 *                   k_pe_col = N - Dr.
 *   MLA_Q_ROPE    : the q_b_proj output [M, H (Dn + Dr)] into q_out = [q_nope | rotated q_pe]: x, ldx, weight as above,
 *                   N = H (Dn + Dr).  Writes only q_out (k_cache may be null).  As b200awq_mla_q_rope.
 *     Folding: as MLA_ROPE, each into the finish of the linear recorded immediately before it, packed in mode 3.  The
 *     chain [q_a|kv_a, MLA_K_ROPE, RMSNORM(q_a slice), q_b, MLA_Q_ROPE, RMSNORM(c_kv slice), kv_b, MLA_KV] is three
 *     kernel ops; kv_b stages the c_kv slice of the row two ops back.  The rejections of MLA_ROPE apply, Cq must be a
 *     multiple of 16, two k rotations may not share a k_cache, and a program may not mix MLA_ROPE with these ops.
 *
 *   LAYER_NORM    : as b200awq_layer_norm: x = input row [K] at pitch ldx, weight [K], bias = [K] or null, y = output
 *                   [K], eps (Command-R's CohereLayerNorm without a bias; StarCoder2's and MPT's nn.LayerNorm).
 *     Folding: as RMSNORM, into the staging of every later linear that reads its output (a published row, a slice of
 *     one, or an external buffer); the first such linear stores y.  Its staging sums x while it stages, takes the
 *     centred sum of squares from the staged row after a CTA barrier and normalises in place: the stand-alone order
 *     above, bit for bit.
 *   GELU / GELU_TANH : as b200awq_gelu with approximate 0 / 1: x = the input [K], y = output [K] (MPT and Falcon use
 *                   GELU; StarCoder2 GELU_TANH).
 *     Folding: into the finish of the plain linear recorded immediately before it, whose whole output must be x (as
 *     an ADD folds): the linear's row publishes fp16(gelu(y)), its y and the op's y are both stored, and the next
 *     linear copies the published row.  The linear keeps mode-0 packing.
 *     Both fold at M = 1 only.  B200AWQ_EUNSUPPORTED (the caller replays per op) for any program created with
 *     max_tokens > 1, a program that also holds MoE, QK_NORM_ROPE_KV or MLA ops, a GELU after anything but a plain
 *     linear (a glue op, an ADD, a ROPE_KV or MLA finish, a MoE block, a linear that already carries an ADD or a GELU),
 *     a GELU in place or on part of the linear's output, a later read of that linear's raw y, and a SiLU*mul of a GELU's
 *     output.
 *
 *   ROPE_KV_SEQ / QK_NORM_ROPE_KV_SEQ : ROPE_KV / QK_NORM_ROPE_KV for a step of T tokens per sequence (speculative
 *                   verification, multi-token prediction, a prompt continued in chunks): the record of kind 6 / 7 with
 *                   K = T (1 <= T, M % T == 0).  Row m = b T + t of x is token t of sequence b at position *pos + t; it
 *                   writes q_out row m and cache entry b.  As b200awq_rope_kv_seq / b200awq_qk_norm_rope_kv_seq.
 *     Folding: the rules and rejections of kind 6 / 7 on the embedded descriptor, with the cache extent of the hazard
 *     checks taken over B = M / T entries.  B200AWQ_EINVAL for T < 1 or M % T != 0.  T = 1 folds exactly as kind 6 / 7.
 *     T > 1 means M > 1, so it folds only in a program created with max_tokens >= M, in the segments where ROPE_KV
 *     folds at M > 1 (RMSNorm staging, residual adds, partial rotary, q / k norm); with LAYER_NORM, GELU, MLA or MoE
 *     ops the program replays per op (B200AWQ_EUNSUPPORTED), as it does for ROPE_KV at M > 1.
 *
 *   ROPE_KV_OFFSET : ROPE_KV_SEQ / QK_NORM_ROPE_KV_SEQ with a per-sequence rotary offset (left-padded batches, the text
 *                   steps of Qwen2-VL / Qwen2.5-VL): x, M, N as kind 17 / 18, K = T (1 <= T, M % T == 0), weight = a
 *                   b200awq_rope_offset_t descriptor (below; null norm weights: no q / k norm).  Row m = b T + t writes
 *                   cache row *pos + t of entry b, rotated at that row plus rot_offset[b].  As b200awq_rope_kv_offset.
 *     Folding: wherever kind 17 / 18 fold (at M = 1 in every program where kind 6 / 7 fold), under their rules and
 *     rejections on the embedded descriptor, plus B200AWQ_EINVAL for a null rot_offset.  rot_offset is a read like
 *     pos: B200AWQ_EUNSUPPORTED when an op of the program writes any of its B = M / T entries.
 *
 *   SCALED_ADD    : the depth-scaled residual add of MiniCPM / MiniCPM3 (h = residual + h * scale_depth /
 *                   sqrt(num_hidden_layers)) and Granite (h = residual + h * residual_multiplier): x = the residual,
 *                   weight = the scaled operand, y = the output, all M contiguous rows of K; eps = the multiplier a
 *                   (float32).  y = fp16(float(x) + float(fp16(float(weight) * a))): torch's rounding of
 *                   `residual + hidden * a` on float16 tensors with a Python scalar a (an fp32 opmath multiply, rounded
 *                   to fp16, then the fp16 add).  A non-finite a, a null pointer or K <= 0: B200AWQ_EINVAL; K % 8 != 0
 *                   or a pointer not 16-byte aligned: B200AWQ_EUNSUPPORTED.
 *     Folding: ADD's rules and rejections, with the operands fixed: weight must be the whole output of the linear
 *     recorded immediately before it, x the residual (an external buffer, or a row published at most 4 kernel ops
 *     back).  It adds no kernel op; the producer's row carries the sum.  B200AWQ_EUNSUPPORTED (the caller replays per op)
 *     also after a MoE block's down op, and when the operands are swapped. */
enum { B200AWQ_OP_RMSNORM = 1, B200AWQ_OP_LINEAR_GEMM = 2, B200AWQ_OP_SILU_AND_MUL = 3, B200AWQ_OP_SPARSE_MOE = 4,
       B200AWQ_OP_ADD = 5, B200AWQ_OP_ROPE_KV = 6, B200AWQ_OP_QK_NORM_ROPE_KV = 7, B200AWQ_OP_QWEN3_MOE = 8,
       B200AWQ_OP_DEEPSEEK_MOE = 9, B200AWQ_OP_MLA_ROPE = 10, B200AWQ_OP_MLA_KV = 11, B200AWQ_OP_MLA_K_ROPE = 12,
       B200AWQ_OP_MLA_Q_ROPE = 13, B200AWQ_OP_LAYER_NORM = 14, B200AWQ_OP_GELU = 15, B200AWQ_OP_GELU_TANH = 16,
       B200AWQ_OP_ROPE_KV_SEQ = 17, B200AWQ_OP_QK_NORM_ROPE_KV_SEQ = 18, B200AWQ_OP_ROPE_KV_OFFSET = 19,
       B200AWQ_OP_SCALED_ADD = 20 };

typedef struct b200awq_op {
  int32_t kind;
  int32_t M, K, N, group_size;
  float eps;
  int64_t ldx;
  const void* x;
  const void* qweight;
  const void* scales;
  const void* qzeros;
  const void* bias;
  const void* weight;
  void* y;
} b200awq_op_t;

/* SPARSE_MOE descriptor (b200awq_op_t.weight points at it; the program copies it at creation, the tensors it names
 * are captured by address).  Stacked GEMM-layout experts as awq/models/mixtral.py:129-151 builds them. */
typedef struct b200awq_moe {
  int32_t E, top_k, renormalize, group_size;
  int32_t H, I;                 /* hidden size, expert intermediate size */
  int32_t block_size;           /* moe_alig_block_size block (16 at the reference's call site) */
  int32_t sorted_len;           /* entries of sorted_ids: >= top_k * M + E * (block_size - 1) */
  const void* gate_weight;      /* router nn.Linear weight [E, H] f16, no bias */
  const int32_t* w1_qweight;    /* gate|up [E, H, 2I/8] */
  const void* w1_scales;        /* [E, H/G, 2I] f16 */
  const int32_t* w1_qzeros;     /* [E, H/G, 2I/8] */
  const int32_t* w2_qweight;    /* down [E, I, H/8] */
  const void* w2_scales;        /* [E, I/G, H] f16 */
  const int32_t* w2_qzeros;     /* [E, I/G, H/8] */
  /* outputs, as the per-op sequence leaves them (M = 1) */
  void* logits;                 /* [E] f16 */
  float* topk_weights;          /* [top_k] f32, after the renormalisation */
  int32_t* topk_ids;            /* [top_k] */
  int32_t* token_expert_indices;/* [top_k] */
  int32_t* sorted_ids;          /* [sorted_len] (entries past the padded runs = top_k) */
  int32_t* expert_ids;          /* [>= top_k + E] */
  int32_t* num_tokens_post_pad; /* [1] */
  void* gate_up;                /* [top_k, 2I] f16 */
  void* act;                    /* [top_k, I] f16 */
  void* down;                   /* [top_k, H] f16: per-slot down outputs x routing weight */
} b200awq_moe_t;

/* Host-side plan of one SPARSE_MOE block in an M = 1 stream program on a device with `sm_count` SMs (no GPU needed).
 * out8 = {kernel ops (2), gate|up 16-column sets (top_k 2I / 16), gate|up units per slot segment, most gate|up sets one
 * CTA owns, down units per set (top_k I / min(G, 128)), down units per slot segment, most (set, slot) partial rows one
 * CTA keeps in the down op, dynamic shared memory of the kernel for this block alone}.  B200AWQ_EUNSUPPORTED outside the
 * envelope above, B200AWQ_EINVAL for bad arguments. */
int b200awq_moe_plan(int E, int top_k, int H, int I, int group_size, int sm_count, int* out8);
/* The same plan for one QWEN3_MOE block: the same out8 layout and envelope, with E <= 128. */
int b200awq_qwen3_moe_plan(int E, int top_k, int H, int I, int group_size, int sm_count, int* out8);

/* DEEPSEEK_MOE descriptor (b200awq_op_t.weight points at it; copied at creation, tensors captured by address). */
typedef struct b200awq_deepseek_moe {
  b200awq_moe_t moe;            /* routed experts, router weight and the per-op buffers (see DEEPSEEK_MOE above) */
  int32_t scoring;              /* 0: softmax (DeepSeek-V2), 1: sigmoid with e_score_correction_bias (DeepSeek-V3) */
  int32_t n_group, topk_group;  /* expert groups (sigmoid): E % n_group == 0, E / n_group >= 2 unless n_group == 1 */
  int32_t norm_topk_prob;       /* sigmoid: normalise the selected weights */
  float routed_scaling_factor;
  int32_t I_s;                  /* shared expert intermediate size (n_shared_experts x moe_intermediate_size) */
  const float* bias;            /* e_score_correction_bias [E] f32 (sigmoid; null for softmax) */
  const int32_t* ws1_qweight;   /* shared gate|up [H, 2 I_s / 8] (gate | up along N) */
  const void* ws1_scales;       /* [H/G, 2 I_s] f16 */
  const int32_t* ws1_qzeros;    /* [H/G, 2 I_s / 8] */
  const int32_t* ws2_qweight;   /* shared down [I_s, H/8] */
  const void* ws2_scales;       /* [I_s/G, H] f16 */
  const int32_t* ws2_qzeros;    /* [I_s/G, H/8] */
  void* shared_out;             /* y_s [H] f16 */
} b200awq_deepseek_moe_t;

/* Plan of one DEEPSEEK_MOE block, out8 as b200awq_moe_plan's with: [1] gate|up sets (top_k 2I + 2 I_s) / 16, [4] down
 * units per set K' / min(G, 128) with K' = top_k I + I_s, [6] partial rows (top_k + I_s / I per set: the shared expert
 * runs as I_s / I more slots).  Envelope (else B200AWQ_EUNSUPPORTED): E <= 128, top_k <= 8, I_s a multiple of I (DeepSeek's
 * n_shared_experts x moe_intermediate_size), the expert and the shared shapes in the stream format, at most 32 gate|up
 * sets and 32 partial rows per CTA, K' / min(G, 128) <= 1024, H / min(G, 128) <= 896 and the activations of K' in
 * shared memory.  The routing arguments are checked at program creation (B200AWQ_EINVAL): scoring 0 or 1, a bias for
 * sigmoid, n_group >= 1 dividing E with E / n_group >= 2 unless n_group == 1, 1 <= topk_group <= n_group. */
int b200awq_deepseek_moe_plan(int E, int top_k, int H, int I, int I_s, int group_size, int sm_count, int* out8);

/* RoPE + KV-cache append of one decode step (awq/modules/fused/attn.py:53-86 RoPE.forward, cache.py:41-46
 * WindowedCache.update_kv), with partial rotary (StableLM's partial_rotary_factor): only the first R = rotary_dim
 * columns of a q / k head are rotated, the other D - R pass through.  For token row m < M, head h < H + 2 KV and
 * rotated pair i < R/2, with a = qkv[m, h D + i], b = qkv[m, h D + R/2 + i], (c, s) = freqs[pos, i]:
 *   q head (h < H):   q_out[m, h, i] = fp16(fma(a, c, -(b s))), q_out[m, h, i + R/2] = fp16(fma(b, c, a s))
 *   k head:           the same rotation into k_cache[m, pos, h - H, .]
 * and every column R <= j < D of a q / k head, and every column of a v head, is copied unchanged into q_out,
 * k_cache[m, pos, h - H, j] or v_cache[m, pos, h - H - KV, j].  R = D (rotary_dim 0) is full rotary.
 * (the fp32 complex product of RoPE.forward with the FMA contraction torch's CUDA kernel uses, then .type_as(fp16);
 * torch's loops for some shapes round a few elements differently, within one fp16 ulp of this).
 * Nothing else is written; when *pos is outside [0, min(cache_len, freqs_len)) nothing at all.  The kernel reads *pos
 * on the device, so a captured CUDA graph replays at whatever position the caller stored there.
 * Column pairs: the kernels handle a head as D/2 column pairs; pair p < R/2 is the rotated pair (p, p + R/2), and pair
 * p >= R/2 with q = p - R/2 is the pass-through pair (R + q, R + q + (D - R)/2) (v heads: the same pairs, copied).
 * For R = D that is (p, p + D/2).  Stream mode 2 lays a qkv linear out in these pairs (below). */
typedef struct b200awq_rope {
  int32_t n_heads, n_kv_heads, head_dim; /* H, KV, D (D % 2 == 0) */
  int32_t cache_len;                     /* S: positions of the cache */
  int32_t freqs_len;                     /* S_f: rows of freqs */
  int32_t rotary_dim;                    /* R: rotated columns per q / k head, even, 2 <= R <= D; 0 means D */
  int64_t cache_batch_stride;            /* elements between two batch entries of k_cache / v_cache (>= S KV D) */
  const int32_t* pos;                    /* device int32[1]: the position written (start_pos) */
  const float* freqs;                    /* [S_f, R/2, 2] f32 (cos, sin): torch.view_as_real(RoPE(R, ..).freqs_cis) */
  void* q_out;                           /* [M, H, D] f16 */
  void* k_cache;                         /* [B >= M, S, KV, D] f16 */
  void* v_cache;                         /* [B >= M, S, KV, D] f16 */
} b200awq_rope_t;
/* ldqkv: row pitch of qkv in elements (>= (H + 2 KV) D).  `rope` is a host pointer, read at the call.
 * B200AWQ_EINVAL for an odd, negative or larger-than-D rotary_dim. */
int b200awq_rope_kv(const void* qkv, int64_t ldqkv, const b200awq_rope_t* rope, int M, b200awq_stream_t stream);

/* Qwen3's q_norm / k_norm, then RoPE + KV-cache append (awq/modules/fused/attn.py:250-253, then as b200awq_rope_kv).
 * For token row m and q or k head h (weight w = q_norm_weight for q heads, k_norm_weight for k heads, both [D] f16):
 *   r     = rsqrtf(ss * fp32(1/D) + eps)  with ss the head's sum of squares in the fixed order below (fp32);
 *                                         fp32(1/D) is torch.mean's scale (ss / D exactly for a power-of-two D)
 *   x'_i  = fp16(w_i * fp16(x_i * r))      (Qwen3RMSNorm.forward on fp16 input)
 * then the rotation and stores of b200awq_rope_kv on x'.  v heads are not normalised.  Summation order: set t of a head
 * (t < D/16) holds the pairs (8 t + g, 8 t + g + D/2), g < 8; s_g = a_g^2 + b_g^2; the set partial is the xor
 * butterfly of the 8 s_g at offsets 4, 2, 1; the head total is the sum of the D/16 set partials in ascending t.
 * Requires D % 16 == 0 and full rotary (rope.rotary_dim 0 or D; else B200AWQ_EUNSUPPORTED).  Nothing is written when
 * *pos is outside [0, min(cache_len, freqs_len)). */
typedef struct b200awq_qk_norm_rope {
  b200awq_rope_t rope;
  const void* q_norm_weight;             /* [D] f16 */
  const void* k_norm_weight;             /* [D] f16 */
  float eps;                             /* variance_epsilon, shared by both norms */
  int32_t pad_;
} b200awq_qk_norm_rope_t;
int b200awq_qk_norm_rope_kv(const void* qkv, int64_t ldqkv, const b200awq_qk_norm_rope_t* desc, int M,
                            b200awq_stream_t stream);

/* b200awq_rope_kv / b200awq_qk_norm_rope_kv for a step of T tokens per sequence at consecutive positions
 * (RoPE.forward(xq, xk, start_pos, seqlen = T) and WindowedCache.update_kv over start_pos .. start_pos + T - 1 for
 * each of B = M / T sequences; speculative verification, multi-token prediction, a prompt continued in chunks, prefill
 * at *pos = 0).  Row m = b T + t of qkv is token t of sequence b at position p = *pos + t: it gets exactly the
 * rotation, copies and norm b200awq_rope_kv / b200awq_qk_norm_rope_kv give one row at p, written to q_out[m] and to
 * k_cache / v_cache entry b, row p (so the caches need B entries).  A row whose p is outside [0, min(cache_len,
 * freqs_len)) writes nothing, not even its q_out row; the other rows of the step still write.  Any M (a prefill of T up
 * to cache_len tokens included).  T = 1 is b200awq_rope_kv / b200awq_qk_norm_rope_kv.  The descriptors are the same;
 * B200AWQ_EINVAL for T < 1 or M % T != 0, otherwise the return codes of those entries. */
int b200awq_rope_kv_seq(const void* qkv, int64_t ldqkv, const b200awq_rope_t* rope, int M, int T,
                        b200awq_stream_t stream);
int b200awq_qk_norm_rope_kv_seq(const void* qkv, int64_t ldqkv, const b200awq_qk_norm_rope_t* desc, int M, int T,
                                b200awq_stream_t stream);

/* b200awq_rope_kv_seq / b200awq_qk_norm_rope_kv_seq with a per-sequence rotary offset: the rotary position differs from
 * the cache row.  Row m = b T + t of qkv has cache row p = *pos + t in entry b (as b200awq_rope_kv_seq) and rotary
 * position r = p + rot_offset[b].  It gets exactly the arithmetic those entries give one row rotated with freqs[r]
 * (partial rotary, the copied v and, when the norm weights are set, Qwen3's q / k norm), written to q_out[m] and to row
 * p of cache entry b.  A row writes nothing, not even its q_out row, unless 0 <= p < cache_len and 0 <= r < freqs_len;
 * the other rows of the step still write.  Uses:
 *   - a left-padded batch (transformers' position_ids = attention_mask.cumsum(-1) - 1): rot_offset[b] = -pad_b, the
 *     cache rows staying in lockstep across the batch;
 *   - a text step of Qwen2-VL / Qwen2.5-VL, whose M-RoPE components are equal for a text token, so the rotation is
 *     plain rotate-half RoPE at p + rope_deltas[b].
 * rot_offset is read on the device at every call, as *pos is: a captured CUDA graph uses what the caller last stored
 * there.  All-zero offsets give the results of b200awq_rope_kv_seq / b200awq_qk_norm_rope_kv_seq byte for byte.
 * B200AWQ_EINVAL for a null desc or rot_offset, T < 1 or M % T != 0, otherwise the return codes of
 * b200awq_rope_kv_seq (both norm weights null) or b200awq_qk_norm_rope_kv_seq (B200AWQ_EINVAL for one null weight,
 * B200AWQ_EUNSUPPORTED for q / k norm with partial rotary or D % 16 != 0). */
typedef struct b200awq_rope_offset {
  b200awq_qk_norm_rope_t qk;             /* the rotation; q_norm_weight = k_norm_weight = null: no q / k norm */
  const int32_t* rot_offset;             /* device int32[B = M / T]: rotary position minus cache row, per sequence */
} b200awq_rope_offset_t;
int b200awq_rope_kv_offset(const void* qkv, int64_t ldqkv, const b200awq_rope_offset_t* desc, int M, int T,
                           b200awq_stream_t stream);

/* MLA (DeepSeek-V2 / V3 multi-head latent attention, no q LoRA): the glue between the fused q_proj | kv_a_proj_with_mqa
 * linear and attention, in transformers' arithmetic (DeepseekV2Attention.forward, DeepseekV3Attention.forward with
 * rope_interleave), for token rows m < M <= 8 writing cache batch entry m at position p = *pos.  Rotary pairs are adjacent
 * elements (a, b) = (x[2i], x[2i + 1]) with (c, s) = freqs[p, i], i < Dr/2:
 *   style 0 (V2, apply_rotary_emb's complex64 product):  out[2i] = fp16(fma(a, c, -(b s))), out[2i + 1] = fp16(fma(b, c, a s))
 *   style 1 (V3, apply_rotary_pos_emb_interleave in fp16, with c16 = fp16(c), s16 = fp16(s)):
 *            out[i] = fp16(fp16(a c16) + fp16(-b s16)),  out[i + Dr/2] = fp16(fp16(b c16) + fp16(a s16))
 * b200awq_mla_rope on the row [q (H (Dn + Dr), per head [nope | pe]) | c_kv (C) | k_pe (Dr)]:
 *   q_out[m, h, :Dn] = q_nope, q_out[m, h, Dn:] = rotate(q_pe), k_cache[m, p, h, Dn:] = rotate(k_pe) for every h;
 *   c_kv is not written anywhere (kv_a_layernorm reads it from the row).
 * b200awq_mla_kv on the kv_b_proj row [H (Dn + Dv)], per head [k_nope | v]:
 *   k_cache[m, p, h, :Dn] = k_nope, v_cache[m, p, h, :Dv] = v.
 * Nothing is written when *pos is outside [0, min(cache_len, freqs_len)) (b200awq_mla_kv: outside [0, cache_len); it
 * reads neither freqs nor q_out, style, C; b200awq_mla_rope reads neither v_cache nor its geometry, Dv).  *pos is read on
 * the device, so a captured CUDA graph replays at whatever position the caller stored there. */
typedef struct b200awq_mla {
  int32_t n_heads, nope_dim, rope_dim, v_dim, kv_lora_rank; /* H, Dn, Dr (even), Dv, C */
  int32_t style;                         /* 0: V2 (interleaved output), 1: V3 (de-interleaved, fp16 arithmetic) */
  int32_t cache_len;                     /* S: positions of the caches */
  int32_t freqs_len;                     /* S_f: rows of freqs */
  int64_t k_batch_stride;                /* elements between two batch entries of k_cache (>= S H (Dn + Dr)) */
  int64_t v_batch_stride;                /* elements between two batch entries of v_cache (>= S H v_head_stride) */
  int32_t v_head_stride;                 /* elements between two heads of one v_cache row (>= Dv; e.g. Dn + Dr) */
  int32_t pad_;
  const int32_t* pos;                    /* device int32[1]: the position written */
  const float* freqs;                    /* [S_f, Dr/2, 2] f32 (cos, sin); style 0: view_as_real(freqs_cis) */
  void* q_out;                           /* [M, H, Dn + Dr] f16 */
  void* k_cache;                         /* [B >= M, S, H, Dn + Dr] f16 */
  void* v_cache;                         /* [B >= M, S, H, v_head_stride] f16 */
} b200awq_mla_t;
/* ld: row pitch of `row` in elements.  `desc` is a host pointer, read at the call. */
int b200awq_mla_rope(const void* row, int64_t ld, const b200awq_mla_t* desc, int M, b200awq_stream_t stream);
int b200awq_mla_kv(const void* row, int64_t ld, const b200awq_mla_t* desc, int M, b200awq_stream_t stream);
/* MLA with a q LoRA (q = q_b_proj(q_a_layernorm(q_a_proj(h)))): the rotation split in two, same arithmetic and position
 * rule as b200awq_mla_rope.
 * b200awq_mla_k_rope on a row whose columns [k_pe_col, k_pe_col + Dr) are k_pe (k_pe_col = Cq + C for the fused
 *   q_a_proj | kv_a_proj_with_mqa row [q_a | c_kv | k_pe]): k_cache[m, p, h, Dn:] = rotate(k_pe) for every h.  Reads
 *   neither q_out nor v_cache; C only as the op's row width in a program.
 * b200awq_mla_q_rope on the q_b_proj row [H (Dn + Dr), per head [nope | pe]]: q_out[m, h, :Dn] = q_nope,
 *   q_out[m, h, Dn:] = rotate(q_pe).  Reads neither k_cache (cache_len still bounds the position) nor v_cache, C. */
int b200awq_mla_k_rope(const void* row, int64_t ld, int64_t k_pe_col, const b200awq_mla_t* desc, int M,
                       b200awq_stream_t stream);
int b200awq_mla_q_rope(const void* row, int64_t ld, const b200awq_mla_t* desc, int M, b200awq_stream_t stream);

typedef struct b200awq_program* b200awq_program_t;

int b200awq_program_create(const b200awq_op_t* ops, int n_ops, b200awq_program_t* out);
/* Host-side plan (no GPU, no CUDA call): the folding rules of b200awq_program_create_batched alone, for a device with
 * `sm_count` SMs and an in-program residual window of `residual_window` kernel ops (<= 0: the library's, 4).  B200AWQ_OK
 * with *kernel_ops = the fused kernel ops when the sequence folds (create may still replay per op: the stream kernels'
 * shape and shared-memory envelope are checked at creation), B200AWQ_EUNSUPPORTED / B200AWQ_EINVAL as create returns
 * them for the folding. */
int b200awq_program_plan(const b200awq_op_t* ops, int n_ops, int max_tokens, int sm_count, int residual_window,
                         int* kernel_ops);
/* Batched decode programs: the same op list recorded with M token rows per op (a fused block built for batch size M:
 * RMSNorm / SiLU*mul over M contiguous rows, linears with M rows at pitch ldx), 1 <= max_tokens <= 8 (else
 * B200AWQ_EINVAL).  Every op must have the same M <= max_tokens, else B200AWQ_EUNSUPPORTED.  M = 1 behaves exactly like
 * b200awq_program_create.  One persistent kernel stages the M rows and uses M token columns of its MMAs, so
 * every token is bit-identical to an M = 1 stream program run on that row alone.  A linear that reads a previous op's
 * output must read it at that op's row pitch (ldx == N of the producer; a column offset is fine); an external source
 * needs 16-byte aligned rows and ldx % 8 == 0.  The activations of M rows of the longest K must fit shared memory
 * next to the weight ring: Llama-3-8B shapes (K up to 14336) fuse up to M = 4.  The program owns its hand-off rows
 * (4 x M rows of the widest output). */
int b200awq_program_create_batched(const b200awq_op_t* ops, int n_ops, int max_tokens, b200awq_program_t* out);
/* token rows per run (M of the recorded ops); 0 for a null handle */
int b200awq_program_tokens(b200awq_program_t prog);
/* 0: null handle; 2: a program - at creation every linear of the program was re-laid-out once into the stream format
 * (below), the kernel partitions the work output-stationary and hands activations from op to op as tagged fp16 words
 * (csrc/program_stream.cuh).  1 (the split-K kernel on the checkpoint layout of earlier versions) is no longer
 * returned. */
int b200awq_program_kind(b200awq_program_t prog);
/* number of fused kernel ops (= linear ops, two per SPARSE_MOE / QWEN3_MOE / DEEPSEEK_MOE op) of the program; 0 for a null handle */
int b200awq_program_num_ops(b200awq_program_t prog);
/* workspace / workspace_bytes: accepted and ignored (null is fine); the program owns its hand-off rows */
int b200awq_program_run(b200awq_program_t prog, void* workspace, size_t workspace_bytes, b200awq_stream_t stream);
int b200awq_program_destroy(b200awq_program_t prog);

/* ---------------------------------------------------------------------------------------------------------
 * One-shot all-reduce over NVLink peer memory (csrc/comm.cu; SURVEY 8e: the reference has no collective at all -
 * multi-GPU there is accelerate layer placement, awq/models/base.py:527-535).  For the tensor-parallel decode path:
 * the fp16 partial outputs of a row-parallel linear (o_proj / down_proj split along K) are summed across the GPUs
 * of one box in ONE kernel launch per call: push into every rank's inbox (P2P stores), flag, wait, reduce in rank
 * order (bit-identical results on all ranks).  One process per GPU: create -> exchange the 64-byte IPC handles by
 * any means (autoawq_b200/comm.py uses torch.distributed.all_gather_object) -> open -> all_reduce any number of
 * times (asynchronous on `stream`, CUDA-graph capturable: the call counter lives on the device).  n % 8 == 0,
 * n <= max_elems (larger messages: use NCCL), world <= 8, y 16-byte aligned; in place.  b200awq_comm_error
 * synchronises and returns B200AWQ_ECUDA if a wait ever timed out (2 s: dead peer). */
typedef struct b200awq_comm* b200awq_comm_t;
int b200awq_comm_create(int rank, int world, int max_elems, b200awq_comm_t* out);
int b200awq_comm_ipc_handle(b200awq_comm_t comm, void* out_64_bytes);
int b200awq_comm_open(b200awq_comm_t comm, const void* handles_world_x_64_bytes);
int b200awq_comm_all_reduce(b200awq_comm_t comm, void* y_f16, int n, b200awq_stream_t stream);
int b200awq_comm_error(b200awq_comm_t comm);
int b200awq_comm_destroy(b200awq_comm_t comm);

/* ---------------------------------------------------------------------------------------------------------
 * Stream format: the one-time, load-time re-layout of a GEMM-layout linear that the decode-program kernel
 * streams (SURVEY 8f #4; the reference's precedent for a post-load re-layout is WQLinear_Exllama.post_init,
 * awq/modules/linear/exllama.py:66-79; the checkpoint format and the module API stay the reference's).  Layout:
 * oracle/stream_format.py (numpy restatement, bit-compared with this entry point in the tests).  Columns are taken
 * in sets of 16, K in units of min(G, 128) rows; a unit is contiguous (fragments in mma.m16n8k16 A-operand order +
 * the unit's scales / zeros), the buffer is set-major, so any partition of the work is a contiguous byte range.
 * mode 0: set s = columns 16 s .. 16 s + 15; mode 1 (a fused gate|up linear): gate column j and up column j share
 * a lane, so SiLU*mul happens in the producer; mode 2 (a qkv linear followed by ROPE_KV, b200awq_stream_pack_rotary):
 * set s of head h = s / (D / 16) holds the column pairs p = 8 t + g (t = s % (D / 16)) of b200awq_rope_t's pairing,
 * lo = h D + p, hi = lo + D/2 for full rotary (R = D), so RoPE's rotation partners share a lane (requires D % 16 == 0
 * and N % D == 0; R even, 2 <= R <= D, with no alignment: a set may hold rotated and pass-through pairs); mode 3 (a q_proj | kv_a_proj_with_mqa linear
 * followed by MLA_ROPE, MLA_K_ROPE or MLA_Q_ROPE, adjacent pairs): set s pairs column 16 s + 2 g with 16 s + 2 g + 1, so MLA's interleaved rotation
 * partners share a lane (b200awq_stream_pack with mode 3).  Requires N % 16 == 0, K % 128 == 0, G in
 * {32, 64} or G % 128 == 0.  b200awq_stream_bytes returns 0 for unsupported shapes; the byte count is the same for
 * every mode. */
size_t b200awq_stream_bytes(int K, int N, int group_size);
int b200awq_stream_pack(const int32_t* qweight, const void* scales, const int32_t* qzeros, void* out, int K, int N,
                        int group_size, int mode, b200awq_stream_t stream);
int b200awq_stream_pack_rotary(const int32_t* qweight, const void* scales, const int32_t* qzeros, void* out, int K,
                               int N, int group_size, int head_dim, b200awq_stream_t stream);
/* Mode 2 for partial rotary: rotary_dim R (even, 2 <= R <= head_dim; 0 means head_dim).  b200awq_stream_pack_rotary is
 * this with R = head_dim. */
int b200awq_stream_pack_partial_rotary(const int32_t* qweight, const void* scales, const int32_t* qzeros, void* out,
                                       int K, int N, int group_size, int head_dim, int rotary_dim,
                                       b200awq_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* B200AWQ_H_ */
