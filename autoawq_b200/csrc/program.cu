// Decode program: the chain of operator calls of a decode step (RMSNorm -> W4A16 linear -> ... -> SiLU*mul -> linear,
// sparse-MoE blocks, residual adds) recorded once and executed by ONE persistent kernel launch.
//
// Why: a stand-alone GEMV launch spends microseconds outside the weight stream - launch + ring fill (the first tile
// lands after the loaded HBM latency), the split-K tail, the ticket round trip - and HBM idles through every one of
// those gaps, 128 times per decode step.  The packed weights never depend on the activations, so the producer warp of
// every CTA walks the WHOLE op list and keeps its shared-memory ring full across op boundaries.
//
// This file is the host side of the stream kernels (program_stream.cuh: M = 1, with or without MoE blocks, residual
// adds, ROPE_KV and QK_NORM_ROPE_KV ops; program_batch.cuh: M = 2..8) plus what those kernels share:
//   * program_create folds the recorded calls into a FoldedProgram: one ProgOp per kernel op (a linear, the glue op
//     that feeds it as an activation prologue, what is folded into its finish) and one MoeBlock per MoE op, and
//     enforces the hazard rules the kernels' ordering relies on;
//   * stream_build re-lays out every linear once into the stream format, builds the kernels' op table, chooses the
//     kernel (ProgKernel) and uploads the side tables it takes; a sequence outside the kernels' envelope is not fused
//     (B200AWQ_EUNSUPPORTED: the caller replays it per op);
//   * program_run launches that kernel; the Program owns every device buffer and frees it when deleted;
//   * the watchdog of every spin loop (ProgWatch, g_prog_abort) and the per-op phase timestamps (g_prog_dbg).
//
// Reference call sequence this replaces: awq/modules/fused/block.py:117-170 (norm -> qkv -> ... -> o -> norm ->
// mlp) with awq/modules/fused/mlp.py:41-55 (gate/up GEMM, silu*mul, down GEMM), each a separate awq_ext call.
#include <algorithm>
#include <array>
#include <cmath>
#include <cstring>
#include <utility>
#include <vector>

#include "../../include/b200awq.h"
#include "common.cuh"
#include "gemv_tile.cuh"
#include "kernels.h"
#include "layernorm.cuh"
#include "rope.cuh"

namespace b200awq {

enum { kProCopy = 0, kProRmsnorm = 1, kProSilu = 2, kProLayernorm = 3 };

// knob 3 = 2: per-op phase timestamps (globaltimer ns) of the first 8 CTAs for the first 32 kernel ops; the slots are
// listed in program_stream.cuh (SP_STAMP)
__device__ unsigned long long g_prog_dbg[32 * 8 * 8];
__device__ __forceinline__ unsigned long long prog_timer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
cudaError_t program_debug_read(void* dst, size_t bytes) {
  return cudaMemcpyFromSymbol(dst, g_prog_dbg, bytes < sizeof(g_prog_dbg) ? bytes : sizeof(g_prog_dbg));
}

__device__ __forceinline__ float prog_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Watchdog for every spin in the program kernels: a lost completion must never hang the GPU.  The first wait that
// exceeds the limit records {code, op, CTA, 1} in g_prog_abort and every spin loop bails out once that is set: the
// kernel terminates (with garbage results) and the host reads the record with b200awq_debug_read under knob 3 = 3.
// [0..3] = first record; [4 + cta * 10 + warp] = (code << 16 | op) of the wait each warp abandoned (0 = none)
__device__ int g_prog_abort[4 + 256 * 10];
cudaError_t program_abort_read(void* dst, size_t bytes) {
  return cudaMemcpyFromSymbol(dst, g_prog_abort, bytes < sizeof(g_prog_abort) ? bytes : sizeof(g_prog_abort));
}
cudaError_t program_abort_clear(cudaStream_t st) {
  void* p = nullptr;
  cudaError_t e = cudaGetSymbolAddress(&p, g_prog_abort);
  return e != cudaSuccess ? e : cudaMemsetAsync(p, 0, sizeof(g_prog_abort), st);
}
// watchdog limit in ns (default 0.5 s; knob 16 = seconds, for runs under compute-sanitizer / cuda-gdb where a kernel
// is orders of magnitude slower and a healthy wait would be mistaken for a lost completion)
__device__ unsigned long long g_prog_watch_ns = 500000000ull;
cudaError_t program_set_watchdog_seconds(int seconds) {
  const unsigned long long ns = seconds > 0 ? (unsigned long long)seconds * 1000000000ull : 500000000ull;
  return cudaMemcpyToSymbol(g_prog_watch_ns, &ns, sizeof(ns));
}
struct ProgWatch {
  unsigned long long t_start = 0;
  int spins = 0;
  // returns true when the caller must give up
  __device__ __forceinline__ bool tick(int code, int op) {
    if ((++spins & 255) == 0) {
      if (*reinterpret_cast<volatile int*>(&g_prog_abort[3]) != 0) {
        if (blockIdx.x < 256 && g_prog_abort[4 + blockIdx.x * 10 + (threadIdx.x >> 5)] == 0)
          g_prog_abort[4 + blockIdx.x * 10 + (threadIdx.x >> 5)] = (code << 16) | (op & 0xffff);
        return true;
      }
      const unsigned long long now = prog_timer();
      if (t_start == 0) t_start = now;
      else if (now - t_start > g_prog_watch_ns) {
        if (atomicCAS(&g_prog_abort[3], 0, 1) == 0) {
          g_prog_abort[0] = code;
          g_prog_abort[1] = op;
          g_prog_abort[2] = blockIdx.x;
        }
        if (blockIdx.x < 256 && g_prog_abort[4 + blockIdx.x * 10 + (threadIdx.x >> 5)] == 0)
          g_prog_abort[4 + blockIdx.x * 10 + (threadIdx.x >> 5)] = (code << 16) | (op & 0xffff);
        return true;
      }
    }
    return false;
  }
};
// wait codes of the abort record (the values are what b200awq_debug_read reports: they stay fixed)
enum { kWEmpty = 3 /* producer: a free ring stage */, kWFull = 4 /* consumer: a landed ring stage */,
       kWCopy = 10 /* staging: the source row's tagged words */, kWRoute = 13 /* producer: a MoE block's routing */,
       kWResidual = 14 /* finish: the tagged row of a residual add's source op */,
       kWQkNorm = 15 /* finish: a q / k head's tagged sum-of-squares partials (QK_NORM_ROPE_KV) */,
       kWLogit = 16 /* routing: a QWEN3_MOE / DEEPSEEK_MOE block's tagged router logits, published across the grid */ };
// returns false when the wait was abandoned (abort): the caller must not touch the barrier's stage any more
__device__ __forceinline__ bool prog_mbar_wait(uint64_t* bar, uint32_t parity, int code, int op) {
  ProgWatch wd;
  while (!mbar_try_wait(bar, parity))
    if (wd.tick(code, op)) return false;
  return true;
}

}  // namespace b200awq
#include "program_stream.cuh"
#include "program_batch.cuh"
namespace b200awq {

// ------------------------------------------------------------------------------------------------ host side
// One kernel op of a folded program (program_create): a linear, the activation prologue that feeds it and what is
// folded into its finish.  stream_build turns the ops into the kernels' SpOp table and side tables.
struct ProgOp {
  const __half* scales = nullptr;
  const int32_t* qzeros = nullptr;
  const __half* bias = nullptr;
  __half* y = nullptr;           // what the op's row publishes (an ADD folded in swaps the linear's y for its output)
  const __half* src = nullptr;   // external source (fp16, global) when !src_prev: COPY x, RMSNORM row, SILU gate|up
  const __half* norm_w = nullptr;   // RMSNORM / LAYER_NORM weight [K]
  const __half* ln_b = nullptr;     // LAYER_NORM bias [K], or null
  __half* xout = nullptr;        // where the recorded glue op wanted its result, or null
  int src_off = 0;               // src_prev: first column of the previous op's output this op reads
  int src_prev = 0;              // 1: the source is the previous op's output
  int K = 0, N = 0, G = 0;
  int prologue = kProCopy;
  float eps = 0.f;
  int ext_dep = -1;              // >= 0: the external source was written by that (older) op of this program
  const int32_t* qw_src = nullptr;   // the checkpoint-format qweight (re-laid-out by stream_build)
  int src_ld = 0;                // row pitch of src in elements (M > 1)
  int stage_row = -1;            // the op whose WHOLE published row this op's staging waits for, or -1
  int moe = 0, mi = -1;          // 1: the gate|up op of MoE block `mi`, 2: its down op (0: a plain linear)
  // an ADD folded into the finish (raw_y != null): raw_y is the linear's own output, still stored; the residual is the
  // published row of the older op res_op, or res_ext, which no op of the program writes; res_mul: a SCALED_ADD's
  // multiplier (the linear's output is scaled before the add), NaN for an ADD
  const void* raw_y = nullptr;
  const void* res_ext = nullptr;
  int res_op = -1;
  float res_mul = NAN;
  // a ROPE_KV folded into the finish (qkr.rope.head_dim != 0); a QK_NORM_ROPE_KV also sets qkr's norm weights;
  // rope_T: tokens per sequence (ROPE_KV_SEQ / QK_NORM_ROPE_KV_SEQ / ROPE_KV_OFFSET: the op's K; 1 for ROPE_KV);
  // rot_offset: a ROPE_KV_OFFSET's per-sequence rotary offsets (null for the other kinds)
  b200awq_qk_norm_rope_t qkr = {};
  int rope_T = 1;
  const int32_t* rot_offset = nullptr;
  // an MLA_ROPE (mla_kind 1), MLA_KV (2), MLA_K_ROPE (3) or MLA_Q_ROPE (4) folded into the finish
  b200awq_mla_t mla = {};
  int mla_kind = 0;
  // a GELU (1) or GELU_TANH (2) folded into the finish: y is the GELU's output (the row publishes it), raw_y the
  // linear's own, still stored (res_op / res_ext stay unset: no residual)
  int gelu = 0;
};

// One MoE op of a folded program (two kernel ops): kind is B200AWQ_OP_SPARSE_MOE, _QWEN3_MOE or _DEEPSEEK_MOE, ds.moe
// the block's descriptor; the DeepSeek fields of ds are zero for the other kinds.
struct MoeBlock {
  int kind;
  b200awq_deepseek_moe_t ds;
  // What the block touches while the kernel runs, as (address, bytes): the kMoeWrites buffers it writes, then the
  // router weight and the correction bias it only reads.  A DEEPSEEK_MOE block's gate_up and act include the shared
  // expert and its logits are fp32.  (null, 0) overlaps nothing.
  static constexpr int kMoeWrites = 11;
  std::array<std::pair<const void*, size_t>, 13> extents(int M) const {
    const b200awq_moe_t& m = ds.moe;
    const bool dsk = kind == B200AWQ_OP_DEEPSEEK_MOE;
    return {{{m.gate_up, ((size_t)m.top_k * 2 * m.I + 2 * (size_t)ds.I_s) * 2},
             {m.act, ((size_t)m.top_k * m.I + ds.I_s) * 2},
             {m.down, (size_t)m.top_k * m.H * 2},
             {m.logits, (size_t)m.E * (dsk ? 4 : 2)},
             {m.topk_weights, (size_t)m.top_k * M * 4},
             {m.topk_ids, (size_t)m.top_k * M * 4},
             {m.token_expert_indices, (size_t)m.top_k * M * 4},
             {m.sorted_ids, (size_t)m.sorted_len * 4},
             {m.expert_ids, (size_t)(m.top_k * M + m.E) * 4},
             {m.num_tokens_post_pad, 4},
             {ds.shared_out, dsk ? (size_t)m.H * 2 : 0},
             {m.gate_weight, (size_t)m.E * m.H * 2},
             {ds.bias, ds.bias != nullptr ? (size_t)m.E * 4 : 0}}};
  }
};

// A folded program: its kernel ops and the MoE blocks they refer to
struct FoldedProgram {
  std::vector<ProgOp> table;
  std::vector<MoeBlock> moes;
};

// The kernel entry that runs a program (chosen by stream_build).  M = 1: the plain kernel (8 or 12 consumer warps,
// knob 9) or the 8-warp kernel of the program's features; M > 1: the batched kernels at MT = sb_mt(M).  Side tables:
// the M = 1 kernels from kKernMoe on take SpMoe (null without MoE blocks), from kKernResidual on SpRes, from kKernRope on
// SpRope, kKernLayerNorm SpLn (and none of the later tables), from kKernQkNorm on SpQkNorm, kKernDeepseekMoe, kKernMla and kKernMlaLora SpDsk, and the last two SpMla; the
// batched ones take SpRes from kKernBatchResidual2 on, SpRopeSeq from kKernBatchRope2 on, SpQkNorm from kKernBatchQkNorm2
// on.  The Qwen3-MoE, DeepSeek-MoE and MLA kernels take every table, with empty entries where an op has no add,
// rotation or norm.
enum ProgKernel {
  kKernPlain, kKernMoe, kKernResidual, kKernRope, kKernLayerNorm, kKernQkNorm, kKernQwen3Moe, kKernDeepseekMoe, kKernMla, kKernMlaLora,
  kKernBatch2, kKernBatch4, kKernBatch8, kKernBatchResidual2, kKernBatchResidual4, kKernBatchResidual8,
  kKernBatchRope2, kKernBatchRope4, kKernBatchRope8, kKernBatchQkNorm2, kKernBatchQkNorm4, kKernBatchQkNorm8
};

struct Program {
  int n_ops = 0;
  int M = 0;
  ProgKernel kernel = kKernPlain;
  size_t xs_bytes = 0;
  int device = 0;
  // re-laid-out weights, per-op CTA partition, hand-off rows, tag state (program_stream.cuh)
  SpOp* d_sp_ops = nullptr;
  uint8_t* d_stream = nullptr;
  uint32_t* d_cta = nullptr;
  uint32_t* d_rows = nullptr;
  int* d_state = nullptr;
  int row_stride = 0;
  size_t stream_bytes = 0;
  // batched stream variant (M > 1, program_batch.cuh): ring stages per warp, sets per CTA, units along K (smem sizes)
  int sb_spw = 0, sb_lmax = 0, sb_nu_max = 0;
  // M = 1 stream kernels (program_stream.cuh): ring stages per warp with 8 / 12 consumer warps (sp_pick_spw); the
  // device's L2 size (the run-ahead window, knob 8)
  int sp_spw8 = 0, sp_spw12 = 0;
  int l2_bytes = 0;
  // side tables, null where the kernel does not take them (ProgKernel): one SpMoe per MoE block, with the published
  // router logits of QWEN3_MOE / DEEPSEEK_MOE blocks ([E] words per block); one SpDsk per DEEPSEEK_MOE block; one
  // SpRes, SpRope and SpQkNorm per kernel op, with the published set partials of QK_NORM_ROPE_KV ops
  SpMoe* d_moe = nullptr;
  unsigned long long* d_xlog = nullptr;
  SpDsk* d_dsk = nullptr;
  SpRes* d_res = nullptr;
  SpRope* d_rope = nullptr;
  SpRopeSeq* d_rope_seq = nullptr;   // (the batched kernels' table in place of SpRope)
  SpQkNorm* d_qkn = nullptr;
  unsigned long long* d_qkn_part = nullptr;
  SpMla* d_mla = nullptr;
  SpLn* d_ln = nullptr;

  Program() = default;
  Program(const Program&) = delete;
  Program& operator=(const Program&) = delete;
  ~Program() {
    for (void* d : std::initializer_list<void*>{d_sp_ops, d_stream, d_cta, d_rows, d_state, d_moe, d_xlog, d_dsk, d_res,
                                                d_rope, d_rope_seq, d_qkn, d_qkn_part, d_mla, d_ln})
      cudaFree(d);
  }
};

// Envelope and partition of a sparse-MoE block in an M = 1 stream program (host only, see b200awq_moe_plan); e_max:
// the experts the block's routing handles (kSpMoeEMax for SPARSE_MOE, kSpQwenEMax for QWEN3_MOE)
static int moe_plan_e(int e_max, int E, int topk, int H, int I, int G, int grid, int* out8) {
  if (E <= 0 || topk <= 0 || topk > E || H <= 0 || I <= 0 || G <= 0 || grid <= 0 || out8 == nullptr)
    return B200AWQ_EINVAL;
  if (E > e_max || topk > kSpMoeKMax) return B200AWQ_EUNSUPPORTED;
  if (!stream_format_supported(H, 2 * I, G, 1) || !stream_format_supported(I, H, G, 0)) return B200AWQ_EUNSUPPORTED;
  const int UK = G < 128 ? G : 128;
  const int sets_a = topk * (2 * I / 16), nu_a = H / UK;
  const int nu_b1 = I / UK, sets_b = H / 16;
  const int lmax_a = (sets_a + grid - 1) / grid;
  const int lmax_b = (sets_b + grid - 1) / grid * topk;     // partial rows: (set, slot)
  if (H / UK > kSpXsumMax || topk * nu_b1 > kSpXsumMax) return B200AWQ_EUNSUPPORTED;
  if (lmax_a > kSpLMax || lmax_b > kSpLMax) return B200AWQ_EUNSUPPORTED;
  const int kmax = H > topk * I ? H : topk * I;
  const size_t smem = sp_fixed_smem(8, 4, true) + (size_t)kmax * 2;   // (at the minimum ring depth)
  if (smem > (size_t)227 * 1024) return B200AWQ_EUNSUPPORTED;
  out8[0] = 2;                         // kernel ops
  out8[1] = sets_a;                    // gate|up: 16-column sets (top_k slots x 2I / 16)
  out8[2] = (2 * I / 16) * nu_a;       // gate|up: units per slot segment
  out8[3] = lmax_a;                    // gate|up: most sets one CTA owns
  out8[4] = topk * nu_b1;              // down: units per set (K' = top_k * I)
  out8[5] = nu_b1;                     // down: units per slot segment
  out8[6] = lmax_b;                    // down: most (set, slot) partial rows one CTA keeps
  out8[7] = (int)smem;                 // dynamic shared memory of the kernel for this block alone
  return B200AWQ_OK;
}
int moe_plan(int E, int topk, int H, int I, int G, int grid, int* out8) {
  return moe_plan_e(kSpMoeEMax, E, topk, H, I, G, grid, out8);
}
int qwen3_moe_plan(int E, int topk, int H, int I, int G, int grid, int* out8) {
  return moe_plan_e(kSpQwenEMax, E, topk, H, I, G, grid, out8);
}
// A DEEPSEEK_MOE block (SpDsk in program_stream.cuh): the QWEN3_MOE plan of the routed experts; the shared expert
// (I_s = nsh I) widens gate|up by 2 I_s / 16 sets and down by I_s / UK units and nsh partial rows per set
int deepseek_moe_plan(int E, int topk, int H, int I, int I_s, int G, int grid, int* out8) {
  if (I_s <= 0 || out8 == nullptr) return B200AWQ_EINVAL;
  const int rc = moe_plan_e(kSpQwenEMax, E, topk, H, I, G, grid, out8);
  if (rc != B200AWQ_OK) return rc;
  if ((I_s % I) != 0) return B200AWQ_EUNSUPPORTED;
  if (!stream_format_supported(H, 2 * I_s, G, 1) || !stream_format_supported(I_s, H, G, 0)) return B200AWQ_EUNSUPPORTED;
  const int UK = G < 128 ? G : 128;
  const int sets_a = (topk * 2 * I + 2 * I_s) / 16, kp = topk * I + I_s, sets_b = H / 16;
  const int lmax_a = (sets_a + grid - 1) / grid, lmax_b = (sets_b + grid - 1) / grid * (topk + I_s / I);
  // (the routing keeps E weights in the tail of the gate|up op's xsum: H / UK + kSpQwenEMax of its entries)
  if (kp / UK > kSpXsumMax || H / UK + kSpQwenEMax > kSpXsumMax || lmax_a > kSpLMax || lmax_b > kSpLMax)
    return B200AWQ_EUNSUPPORTED;
  const size_t smem = sp_fixed_smem(8, 4, true) + (size_t)(H > kp ? H : kp) * 2;
  if (smem > (size_t)227 * 1024) return B200AWQ_EUNSUPPORTED;
  out8[1] = sets_a;
  out8[3] = lmax_a;
  out8[4] = kp / UK;
  out8[6] = lmax_b;
  out8[7] = (int)smem;
  return B200AWQ_OK;
}

size_t stream_format_bytes(int K, int N, int G) {
  if (K <= 0 || N <= 0 || G <= 0) return 0;
  const int UK = G < 128 ? G : 128;
  return (size_t)(N / 16) * (K / UK) * ((size_t)(UK / 16) * 128 + kSpAux);
}
bool stream_format_supported(int K, int N, int G, int mode) {
  if (K <= 0 || N <= 0 || G <= 0 || (K % G) != 0 || (N % 16) != 0 || (K % 128) != 0) return false;
  if (!(G == 32 || G == 64 || (G % 128) == 0)) return false;
  if (mode == 1 && ((N / 2) % 8) != 0) return false;
  return mode == 0 || mode == 1 || mode == 3;
}
static int prog_sm_count();   // device SM count (defined below)

// The deepest ring (stages per consumer warp, at most kSpMaxStages) of an M = 1 stream kernel with nw consumer warps
// that fits 227 KB next to the program's activations (xs_bytes).  A program stream_build accepts gets at least 4 stages
// at 8 warps and 3 at 12.
static int sp_pick_spw(int nw, bool moe, size_t xs_bytes) {
  int spw = kSpMaxStages;
  while (spw > 1 && sp_fixed_smem(nw, spw, moe) + xs_bytes > (size_t)227 * 1024) --spw;
  return spw;
}

cudaError_t stream_pack_rotary(const int32_t* qweight, const void* scales, const int32_t* qzeros, void* out, int K, int N,
                               int G, int head_dim, int rotary_dim, cudaStream_t st) {
  if (!stream_format_supported(K, N, G, 0) || head_dim <= 0 || (head_dim % 16) != 0 || (N % head_dim) != 0 ||
      rotary_dim < 2 || (rotary_dim % 2) != 0 || rotary_dim > head_dim)
    return cudaErrorNotSupported;
  const int UK = G < 128 ? G : 128;
  const int64_t total = (int64_t)(N / 16) * (K / UK) * ((UK / 16) * 32 + 12);
  const int cap = prog_sm_count() * 16;
  const int blocks = (int)((total + 255) / 256 < cap ? (total + 255) / 256 : cap);
  stream_pack_rotary_kernel<<<blocks, 256, 0, st>>>(qweight, static_cast<const __half*>(scales), qzeros,
                                                    static_cast<uint8_t*>(out), K, N, G, head_dim, rotary_dim);
  return cudaGetLastError();
}

cudaError_t stream_pack(const int32_t* qweight, const void* scales, const int32_t* qzeros, void* out, int K, int N, int G,
                        int mode, cudaStream_t st) {
  if (!stream_format_supported(K, N, G, mode)) return cudaErrorNotSupported;
  const int UK = G < 128 ? G : 128;
  const int64_t total = (int64_t)(N / 16) * (K / UK) * ((UK / 16) * 32 + 12);
  const int cap = prog_sm_count() * 16;
  const int blocks = (int)((total + 255) / 256 < cap ? (total + 255) / 256 : cap);
  if (mode == 3)   // (a kernel of its own: stream_pack_kernel keeps its code)
    stream_pack_pairs_kernel<<<blocks, 256, 0, st>>>(qweight, static_cast<const __half*>(scales), qzeros,
                                                     static_cast<uint8_t*>(out), K, N, G);
  else
    stream_pack_kernel<<<blocks, 256, 0, st>>>(qweight, static_cast<const __half*>(scales), qzeros,
                                               static_cast<uint8_t*>(out), K, N, G, mode);
  return cudaGetLastError();
}

// Allocates *d and copies h into it (an empty h leaves *d null)
template <typename T>
static cudaError_t upload(T** d, const std::vector<T>& h) {
  if (h.empty()) return cudaSuccess;
  const cudaError_t e = cudaMalloc(d, h.size() * sizeof(T));
  return e != cudaSuccess ? e : cudaMemcpy(*d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice);
}

// Builds the stream kernels' program from the folded one, for pr->M token rows (M > 1: the batched kernel of
// program_batch.cuh), and chooses the kernel that runs it.  Returns false when the sequence is outside their envelope.
// *err != cudaSuccess reports a CUDA failure; what was allocated by then is pr's to free.
// MoE blocks (`moe` != 0, M = 1 only): the gate|up op is a mode-1 op over top_k slots of 2I columns, the down op reads
// its published row (K' = top_k I); both stream E per-expert slices packed back to back.
// ROPE_KV ops (`qkr.rope.head_dim` != 0): packed in mode 2, the finish rotates / appends (SpRope).
// QK_NORM_ROPE_KV ops: as ROPE_KV, and `qkr` carries the norm weights (q_norm_weight != null: SpQkNorm).
// MLA_ROPE ops (`mla_kind` 1): packed in mode 3, the finish rotates / stores (SpMla); MLA_KV (2): mode 0, the finish
// stores the cache columns.  Such a program runs stream_mla_kernel, whose MoE blocks are DEEPSEEK_MOE blocks.
// MLA_K_ROPE / MLA_Q_ROPE (3 / 4): packed in mode 3, on stream_mla_lora_kernel (the same, plus their finishes).
// LAYER_NORM prologues (kProLayernorm) and GELU finishes (`gelu` != 0, mode 0): stream_layernorm_kernel (SpLn).
static bool stream_build(Program* pr, const FoldedProgram& f, int grid, cudaError_t* err) {
  *err = cudaSuccess;
  const std::vector<ProgOp>& table = f.table;
  const int n = static_cast<int>(table.size()), M = pr->M;
  if (n >= 60000) return false;
  const bool has_moe = !f.moes.empty();
  if (has_moe && M != 1) return false;
  // a QWEN3_MOE (DEEPSEEK_MOE) program runs stream_qwen3moe_kernel (stream_deepseek_moe_kernel), whose MoE blocks are
  // all of that kind
  const int mkind = has_moe ? f.moes[0].kind : B200AWQ_OP_SPARSE_MOE;
  // MLA ops run on stream_mla_kernel, whose MoE blocks are DEEPSEEK_MOE blocks
  for (const ProgOp& p : table)
    if (p.mla_kind != 0 && has_moe && mkind != B200AWQ_OP_DEEPSEEK_MOE) return false;
  for (const MoeBlock& b : f.moes)
    if (b.kind != mkind) return false;
  std::vector<int> plan_a(f.moes.size() * 8);
  for (size_t b = 0; b < f.moes.size(); ++b) {
    const b200awq_moe_t& m = f.moes[b].ds.moe;
    const int rc = mkind == B200AWQ_OP_DEEPSEEK_MOE
                       ? deepseek_moe_plan(m.E, m.top_k, m.H, m.I, f.moes[b].ds.I_s, m.group_size, grid, &plan_a[b * 8])
                       : (mkind == B200AWQ_OP_QWEN3_MOE ? qwen3_moe_plan : moe_plan)(m.E, m.top_k, m.H, m.I, m.group_size,
                                                                                   grid, &plan_a[b * 8]);
    if (rc != B200AWQ_OK) return false;
  }
  // creation is a load-time step (not capturable): whatever produced the checkpoint tensors on any stream is done
  // before the re-layout reads them
  if ((*err = cudaDeviceSynchronize()) != cudaSuccess) return false;
  std::vector<SpOp> ops(n);
  std::vector<int> mode(n, 0);
  // producer-side SiLU*mul: a SILU prologue whose source is the whole output of the previous linear
  for (int i = 0; i < n; ++i)
    if (table[i].prologue == kProSilu) {
      if (i == 0 || !table[i].src_prev || table[i].src_off != 0 || table[i - 1].N != 2 * table[i].K) {
        // a later consumer of an already fused gate|up output (ext_dep) is fine, anything else is not
        const int j = table[i].ext_dep;
        if (!(j >= 0 && mode[j] == 1 && table[i].src == table[j].y && table[j].N == 2 * table[i].K)) return false;
      } else {
        mode[i - 1] = 1;
      }
    }
  // bytes of one expert's slice of a MoE op's stream copy (256-byte aligned)
  auto expert_bytes = [&](int i) {
    const b200awq_moe_t& m = f.moes[table[i].mi].ds.moe;
    const size_t b = table[i].moe == 1 ? stream_format_bytes(m.H, 2 * m.I, m.group_size)
                                       : stream_format_bytes(m.I, m.H, m.group_size);
    return (b + 255) & ~(size_t)255;
  };
  // bytes of the shared expert's stream copy of a DEEPSEEK_MOE op (in front of its expert slices; 0 otherwise)
  auto shared_bytes = [&](int i) {
    const MoeBlock& blk = f.moes[table[i].mi];
    if (blk.kind != B200AWQ_OP_DEEPSEEK_MOE) return (size_t)0;
    const b200awq_moe_t& m = blk.ds.moe;
    const size_t b = table[i].moe == 1 ? stream_format_bytes(m.H, 2 * blk.ds.I_s, m.group_size)
                                       : stream_format_bytes(blk.ds.I_s, m.H, m.group_size);
    return (b + 255) & ~(size_t)255;
  };
  for (int i = 0; i < n; ++i)
    if (table[i].moe == 1) mode[i] = 1;
  bool has_rope = false, has_qkn = false, has_res = false, has_mla = false, has_lora = false;
  for (int i = 0; i < n; ++i) {
    if (table[i].qkr.rope.head_dim != 0) {
      if (mode[i] != 0) return false;   // (program_create rejects a gate|up producer already)
      mode[i] = 2;
      has_rope = true;
    }
    has_qkn = has_qkn || table[i].qkr.q_norm_weight != nullptr;
    if (table[i].mla_kind != 0) {
      if (mode[i] != 0) return false;
      if (table[i].mla_kind != 2) mode[i] = 3;
      has_mla = true;
      has_lora = has_lora || table[i].mla_kind >= 3;
    }
  }
  if (has_mla && M != 1) return false;   // (program_create rejects it already)
  // residual adds and GELUs: the producer and an in-program residual must publish plain columns (a mode-1 row holds
  // SiLU*mul)
  bool has_ln = false;
  for (int i = 0; i < n; ++i) {
    if (table[i].raw_y != nullptr) {
      if (mode[i] == 1 || (table[i].res_op >= 0 && mode[table[i].res_op] == 1)) return false;
      has_res = has_res || table[i].gelu == 0;
    }
    has_ln = has_ln || table[i].gelu != 0 || table[i].prologue == kProLayernorm;
  }
  // LAYER_NORM / GELU run on stream_layernorm_kernel only (program_create rejects the rest already)
  if (has_ln && (M != 1 || has_moe || has_qkn || has_mla)) return false;
  // the kernel: the first of these the program needs (has_qkn implies has_rope; QWEN3_MOE and DEEPSEEK_MOE blocks only
  // exist at M = 1)
  const int mt = sb_mt(M) == 2 ? 0 : (sb_mt(M) == 4 ? 1 : 2);
  const ProgKernel kern =
      M > 1 ? ProgKernel((has_qkn ? kKernBatchQkNorm2 : has_rope ? kKernBatchRope2 : has_res ? kKernBatchResidual2
                                                                                             : kKernBatch2) + mt)
      : has_ln                           ? kKernLayerNorm
      : has_lora                         ? kKernMlaLora
      : has_mla                          ? kKernMla
      : mkind == B200AWQ_OP_DEEPSEEK_MOE ? kKernDeepseekMoe
      : mkind == B200AWQ_OP_QWEN3_MOE    ? kKernQwen3Moe
      : has_qkn                          ? kKernQkNorm
      : has_rope                         ? kKernRope
      : has_res                          ? kKernResidual
      : has_moe                          ? kKernMoe
                                         : kKernPlain;
  size_t wbytes = 0, max_cols = 0;
  int max_K = 0, lmax = 0, nu_max = 0;
  std::vector<size_t> woff(n);
  for (int i = 0; i < n; ++i) {
    const ProgOp& p = table[i];
    if (p.moe != 0) {   // envelope checked by moe_plan (per-expert shapes, sets and partial rows per CTA)
      woff[i] = wbytes;
      wbytes += shared_bytes(i) + (size_t)f.moes[p.mi].ds.moe.E * expert_bytes(i);
    } else {
      if (!stream_format_supported(p.K, p.N, p.G, mode[i] == 2 ? 0 : mode[i])) return false;
      const int UK = p.G < 128 ? p.G : 128;
      if (p.K / UK > kSpXsumMax) return false;
      if (M == 1 && (p.N / 16 + grid - 1) / grid > kSpLMax) return false;
      lmax = std::max(lmax, (p.N / 16 + grid - 1) / grid);
      nu_max = std::max(nu_max, p.K / UK);
      woff[i] = wbytes;
      wbytes += (stream_format_bytes(p.K, p.N, p.G) + 255) & ~(size_t)255;
    }
    max_cols = std::max(max_cols, (size_t)(mode[i] == 1 ? p.N / 2 : p.N));
    max_K = std::max(max_K, p.K);
  }
  if (M == 1) {
    // the envelope: a ring of 4 stages at 8 warps (the MoE / residual / rope kernels, behind the routing area) or 3 at
    // 12 must fit; the program then runs the deepest ring its activations leave room for
    const bool moe_k = kern != kKernPlain;
    if (moe_k && sp_fixed_smem(8, 4, true) + (size_t)max_K * 2 > (size_t)227 * 1024) return false;
    if (!moe_k && sp_fixed_smem(12, 3, false) + (size_t)max_K * 2 > (size_t)227 * 1024) return false;
    pr->sp_spw8 = sp_pick_spw(8, moe_k, (size_t)max_K * 2);
    pr->sp_spw12 = moe_k ? 0 : sp_pick_spw(12, false, (size_t)max_K * 2);
  } else {
    // the batched kernel: the deepest ring (<= 4 stages per warp) that leaves room for M rows of activations
    int spw = kSbMaxStages;
    while (spw > 0 && sb_fixed_smem(spw, lmax, sb_mt(M), nu_max) + (size_t)max_K * sb_mt(M) * 2 > (size_t)227 * 1024) --spw;
    if (spw == 0) return false;
    pr->sb_spw = spw;
    pr->sb_lmax = lmax;
    pr->sb_nu_max = nu_max;
  }
  for (int i = 0; i < n; ++i) {
    const ProgOp& p = table[i];
    SpOp& o = ops[i];
    std::memset(&o, 0, sizeof(o));
    o.bias = p.bias;
    o.y = p.raw_y != nullptr ? static_cast<__half*>(const_cast<void*>(p.raw_y)) : p.y;
    o.K = p.K;
    o.N = p.N;
    const int UK = p.G < 128 ? p.G : 128;
    o.uk_shift = UK == 32 ? 5 : (UK == 64 ? 6 : 7);
    o.F = UK / 16;
    o.NU = p.K / UK;
    o.unit_bytes = o.F * 128 + kSpAux;
    o.ups = kSpStageBytes / o.unit_bytes;
    o.mode = mode[i];
    o.eps = p.eps;
    o.norm_w = p.norm_w;
    o.src_op = -1;
    if (p.prologue == kProSilu) {
      // the SiLU*mul itself runs in the producer (mode 1); this op copies the published product
      const int j = p.src_prev ? i - 1 : p.ext_dep;
      if (i - j >= kSpRows) return false;
      o.prologue = kProCopy;
      o.src_op = j;
      o.src_off = 0;
      if (p.xout != nullptr) ops[j].act_out = p.xout;
    } else {
      o.prologue = p.prologue;
      o.xout = p.prologue == kProRmsnorm || p.prologue == kProLayernorm ? p.xout : nullptr;
      if (p.prologue == kProCopy && p.xout != nullptr) return false;
      int j = -1;
      if (p.src_prev) j = i - 1;
      else if (p.ext_dep >= 0) j = p.ext_dep;
      if (j >= 0) {
        if (mode[j] == 1 || i - j >= kSpRows) return false;   // raw gate|up columns of a fused producer / row recycled
        const uintptr_t y0 = reinterpret_cast<uintptr_t>(table[j].y), s0 = reinterpret_cast<uintptr_t>(p.src);
        if (s0 < y0 || s0 + (size_t)p.K * 2 > y0 + (size_t)table[j].N * 2 || ((s0 - y0) & 7) != 0) return false;
        if (M > 1 && p.src_ld != table[j].N) return false;   // row m of the source must be row m of the producer
        o.src_op = j;
        o.src_off = static_cast<int>((s0 - y0) / 2);
      } else {
        o.src = p.src;
        if ((reinterpret_cast<uintptr_t>(p.src) & 7) != 0) return false;
        if (M > 1 && ((reinterpret_cast<uintptr_t>(p.src) & 15) != 0 || (p.src_ld % 8) != 0)) return false;
        o.ldx = p.src_ld;
      }
    }
    if (p.gelu != 0) o.act_out = p.y;   // the GELU's output (o.y is the linear's raw y)
    if (p.moe != 0) {
      o.moe = p.moe;
      o.moe_i = p.mi;
      if (o.moe == 2) {
        // the down op stages the gate|up op's published SiLU*mul row (top_k x I words, slot-major); the recorded
        // activation tensor is written as a side effect of that op
        if (i == 0 || table[i - 1].moe != 1 || table[i - 1].mi != p.mi) return false;
        o.prologue = kProCopy;
        o.src = nullptr;
        o.src_op = i - 1;
        o.src_off = 0;
        ops[i - 1].act_out = const_cast<__half*>(p.src);
      }
    }
  }
  // CTA partition: whole 16-column sets, as even as the set count allows
  std::vector<uint32_t> cta((size_t)n * (grid + 1));
  for (int i = 0; i < n; ++i) {
    const int64_t S = table[i].N / 16;
    for (int c = 0; c <= grid; ++c) cta[(size_t)i * (grid + 1) + c] = (uint32_t)((S * c / grid) * ops[i].NU);
  }
  pr->row_stride = (int)((max_cols + 63) & ~(size_t)63);
  cudaError_t e = cudaMalloc(&pr->d_stream, wbytes);
  if (e == cudaSuccess) e = upload(&pr->d_cta, cta);
  // M hand-off rows per op and the tag state, zero (no run's tag) until the first run
  if (e == cudaSuccess) e = upload(&pr->d_rows, std::vector<uint32_t>((size_t)kSpRows * M * pr->row_stride));
  if (e == cudaSuccess) e = upload(&pr->d_state, std::vector<int>(2));
  for (int i = 0; i < n && e == cudaSuccess; ++i) {
    ops[i].wstream = pr->d_stream + woff[i];
    ops[i].cta_begin = pr->d_cta + (size_t)i * (grid + 1);
    if (table[i].moe != 0) {
      // one stream copy per expert slice of the stacked tensors ([E, K, N/8], [E, K/G, N], [E, K/G, N/8])
      const MoeBlock& blk = f.moes[table[i].mi];
      const b200awq_moe_t& m = blk.ds.moe;
      const bool gu = table[i].moe == 1;
      const int K = gu ? m.H : m.I, N = gu ? 2 * m.I : m.H, G = m.group_size;
      const int32_t* qw = table[i].qw_src;
      const size_t shb = shared_bytes(i);
      for (int x = 0; x < m.E && e == cudaSuccess; ++x)
        e = stream_pack(qw + (size_t)x * K * (N / 8), table[i].scales + (size_t)x * (K / G) * N,
                        table[i].qzeros + (size_t)x * (K / G) * (N / 8),
                        pr->d_stream + woff[i] + shb + (size_t)x * expert_bytes(i), K, N, G, mode[i], nullptr);
      if (shb != 0 && e == cudaSuccess) {   // DEEPSEEK_MOE: the shared expert's copy, first
        const b200awq_deepseek_moe_t& d = blk.ds;
        e = stream_pack(gu ? d.ws1_qweight : d.ws2_qweight, gu ? d.ws1_scales : d.ws2_scales,
                        gu ? d.ws1_qzeros : d.ws2_qzeros, pr->d_stream + woff[i], gu ? m.H : d.I_s, gu ? 2 * d.I_s : m.H,
                        G, mode[i], nullptr);
      }
      continue;
    }
    if (mode[i] == 2)
      e = stream_pack_rotary(table[i].qw_src, table[i].scales, table[i].qzeros, pr->d_stream + woff[i], table[i].K,
                             table[i].N, table[i].G, table[i].qkr.rope.head_dim, rope_rotary_dim(table[i].qkr.rope),
                             nullptr);
    else
      e = stream_pack(table[i].qw_src, table[i].scales, table[i].qzeros, pr->d_stream + woff[i], table[i].K, table[i].N,
                      table[i].G, mode[i], nullptr);
  }
  if (e == cudaSuccess && has_moe) {
    // QWEN3_MOE / DEEPSEEK_MOE blocks: [E] logit words each, zero (no run's tag) until the first run
    size_t xwords = 0;
    for (const MoeBlock& b : f.moes) xwords += b.kind != B200AWQ_OP_SPARSE_MOE ? (size_t)b.ds.moe.E : 0;
    e = upload(&pr->d_xlog, std::vector<unsigned long long>(xwords));
    size_t xoff = 0;
    std::vector<SpMoe> md(f.moes.size());
    std::vector<SpDsk> dd(f.moes.size());
    for (size_t b = 0; b < f.moes.size(); ++b) {
      const b200awq_moe_t& m = f.moes[b].ds.moe;
      SpMoe& d = md[b];
      d.gate_w = static_cast<const __half*>(m.gate_weight);
      d.logits = static_cast<__half*>(m.logits);
      d.topk_w = m.topk_weights;
      d.topk_ids = m.topk_ids;
      d.tok_idx = m.token_expert_indices;
      d.sorted_ids = m.sorted_ids;
      d.expert_ids = m.expert_ids;
      d.npost = m.num_tokens_post_pad;
      d.down = static_cast<__half*>(m.down);
      d.E = m.E;
      d.topk = m.top_k;
      d.renorm = m.renormalize != 0;
      d.block_size = m.block_size;
      d.sorted_len = m.sorted_len;
      d.seg_a = plan_a[b * 8 + 2];
      d.seg_b = plan_a[b * 8 + 5];
      d.I = m.I;
      if (f.moes[b].kind != B200AWQ_OP_SPARSE_MOE) {
        d.xlog = pr->d_xlog + xoff;
        xoff += (size_t)m.E;
      }
      const b200awq_deepseek_moe_t& s = f.moes[b].ds;
      SpDsk& x = dd[b];
      x.bias = s.bias;
      x.shared_out = static_cast<__half*>(s.shared_out);
      x.scoring = s.scoring;
      x.n_group = s.n_group;
      x.topk_group = s.topk_group;
      x.norm = s.norm_topk_prob != 0;
      x.rsf = s.routed_scaling_factor;
      x.nsh = s.I_s / m.I;
    }
    for (int i = 0; i < n; ++i)
      if (table[i].moe != 0) {
        (table[i].moe == 1 ? md[table[i].mi].eb_a : md[table[i].mi].eb_b) = (long long)expert_bytes(i);
        (table[i].moe == 1 ? dd[table[i].mi].shb_a : dd[table[i].mi].shb_b) = (long long)shared_bytes(i);
      }
    if (e == cudaSuccess) e = upload(&pr->d_moe, md);
    if (e == cudaSuccess && (kern == kKernDeepseekMoe || kern == kKernMla || kern == kKernMlaLora))
      e = upload(&pr->d_dsk, dd);
  }
  // the side tables the kernel takes (ProgKernel)
  const bool takes_res = (kern >= kKernResidual && kern <= kKernMlaLora) || kern >= kKernBatchResidual2;
  const bool takes_rope = (kern >= kKernRope && kern <= kKernMlaLora) || kern >= kKernBatchRope2;
  const bool takes_qkn = (kern >= kKernQkNorm && kern <= kKernMlaLora) || kern >= kKernBatchQkNorm2;
  if (e == cudaSuccess && takes_res) {
    std::vector<SpRes> rd(n);
    for (int i = 0; i < n; ++i) {
      rd[i].op = table[i].res_op;
      if (table[i].raw_y == nullptr || table[i].gelu != 0) continue;
      rd[i].out = table[i].y;                       // the ADD's output (the op's y was swapped for it)
      rd[i].ext = static_cast<const __half*>(table[i].res_ext);
      rd[i].mul = table[i].res_mul;
    }
    e = upload(&pr->d_res, rd);
  }
  if (e == cudaSuccess && takes_rope && M == 1) {
    std::vector<SpRope> rp(n);
    for (int i = 0; i < n; ++i) {
      rp[i].r = table[i].qkr.rope;   // (head_dim 0: no rotation)
      rp[i].rot_offset = table[i].rot_offset;
    }
    e = upload(&pr->d_rope, rp);
  } else if (e == cudaSuccess && takes_rope) {
    std::vector<SpRopeSeq> rp(n);
    for (int i = 0; i < n; ++i) {
      rp[i].r = table[i].qkr.rope;
      rp[i].rot_offset = table[i].rot_offset;
      rp[i].T = table[i].rope_T;
    }
    e = upload(&pr->d_rope_seq, rp);
  }
  if (e == cudaSuccess && takes_qkn) {
    // the partials of op i live at [M][N_i / 16] words from its offset; zero tags are never a run's (sp_tag >= 1)
    size_t words = 0;
    for (const ProgOp& p : table) words += p.qkr.q_norm_weight != nullptr ? (size_t)M * (p.N / 16) : 0;
    e = upload(&pr->d_qkn_part, std::vector<unsigned long long>(words));
    std::vector<SpQkNorm> qd(n);
    size_t off = 0;
    for (int i = 0; i < n; ++i) {
      if (table[i].qkr.q_norm_weight == nullptr) continue;
      qd[i].q = table[i].qkr;
      qd[i].part = pr->d_qkn_part + off;
      qd[i].inv_d = 1.f / static_cast<float>(table[i].qkr.rope.head_dim);
      qd[i].rot_offset = table[i].rot_offset;
      off += (size_t)M * (table[i].N / 16);
    }
    if (e == cudaSuccess) e = upload(&pr->d_qkn, qd);
  }
  if (e == cudaSuccess && (kern == kKernMla || kern == kKernMlaLora)) {
    std::vector<SpMla> ml(n);
    for (int i = 0; i < n; ++i) {
      ml[i].d = table[i].mla;
      ml[i].kind = table[i].mla_kind;
      const int s = table[i].stage_row;
      if (s >= 0 && table[s].mla_kind == 1 && ops[i].src_op == s) ml[i].wait_words = table[s].N;
      // stream_mla_lora_kernel polls the previous op's row (program_create: a slice of a K_ROPE row)
      if (kern == kKernMlaLora && s == i - 1 && ops[i].src_op >= 0 && table[ops[i].src_op].mla_kind == 3)
        ml[i].wait_words = table[s].N;
    }
    e = upload(&pr->d_mla, ml);
  }
  if (e == cudaSuccess && kern == kKernLayerNorm) {
    std::vector<SpLn> ln(n);
    for (int i = 0; i < n; ++i) {
      ln[i].bias = table[i].prologue == kProLayernorm ? table[i].ln_b : nullptr;
      ln[i].gelu = table[i].gelu;
    }
    e = upload(&pr->d_ln, ln);
  }
  if (e == cudaSuccess) e = upload(&pr->d_sp_ops, ops);
  // the kernel may use all 227 KB of shared memory (the plain one at both warp counts: knob 9 is read at run time)
  static const void* const entry[] = {
      (const void*)stream_program_kernel<8, 4>, (const void*)stream_moe_kernel, (const void*)stream_residual_kernel,
      (const void*)stream_rope_kernel, (const void*)stream_layernorm_kernel, (const void*)stream_qknorm_kernel,
      (const void*)stream_qwen3moe_kernel,
      (const void*)stream_deepseek_moe_kernel, (const void*)stream_mla_kernel, (const void*)stream_mla_lora_kernel,
      (const void*)stream_batch_kernel<2>, (const void*)stream_batch_kernel<4>,
      (const void*)stream_batch_kernel<8>, (const void*)stream_batch_residual_kernel<2>,
      (const void*)stream_batch_residual_kernel<4>, (const void*)stream_batch_residual_kernel<8>,
      (const void*)stream_batch_rope_kernel<2>, (const void*)stream_batch_rope_kernel<4>,
      (const void*)stream_batch_rope_kernel<8>, (const void*)stream_batch_qknorm_kernel<2>,
      (const void*)stream_batch_qknorm_kernel<4>, (const void*)stream_batch_qknorm_kernel<8>};
  static_assert(sizeof(entry) / sizeof(entry[0]) == kKernBatchQkNorm8 + 1, "one entry per ProgKernel");
  if (e == cudaSuccess) e = cudaFuncSetAttribute(entry[kern], cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
  if (e == cudaSuccess && kern == kKernPlain)
    e = cudaFuncSetAttribute(stream_program_kernel<12, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&pr->l2_bytes, cudaDevAttrL2CacheSize, pr->device);
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  pr->kernel = kern;
  pr->stream_bytes = wbytes;
  pr->xs_bytes = (size_t)max_K * (M == 1 ? 1 : sb_mt(M)) * 2;   // M = 1: one row (stream_program_kernel)
  *err = e;
  return e == cudaSuccess;
}

static int prog_sm_count() {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess ||
      cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
    n = B200AWQ_SM_COUNT_FALLBACK;
  return n;
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
static bool overlaps(const void* a, size_t na, const void* b, size_t nb) {
  const uintptr_t a0 = reinterpret_cast<uintptr_t>(a), b0 = reinterpret_cast<uintptr_t>(b);
  return a0 < b0 + nb && b0 < a0 + na;
}

// Folds the recorded call sequence into linear ops with an activation prologue.  Returns a B200AWQ_* code;
// *cuda_err carries the CUDA error behind B200AWQ_ECUDA.
//
// Hazard rules (the kernels order ops only through the hand-off rows the ops publish; the fp16 outputs and the glue
// outputs in the recorded buffers are stored on the side, by the CTAs that own them, while later ops run):
//   * a glue op (RMSNorm / SiLU*mul) is executed as the prologue of every later linear that reads its output
//     buffer; that buffer is written as a side effect, nobody inside the kernel may READ it;
//   * a source inside the previous op's output is read from that op's published row (src_prev); any other
//     overlap with the previous op's output is rejected; a source written by an older op (ext_dep) is read from that
//     op's row as well (stream_build);
//   * a linear must not write (y) what it reads (src) or what its own prologue publishes (xout);
//   * a buffer that a pending glue record depends on must not be overwritten before the record's last use.
// Every op has the same M <= max_tokens rows (M > 1: the batched stream kernel only); extents below cover all M rows.
int program_create(const b200awq_op_t* ops_in, int n_in, int max_tokens, Program** out, cudaError_t* cuda_err,
                   ProgramPlan* plan) {
  *cuda_err = cudaSuccess;
  *out = nullptr;
  if (ops_in == nullptr || n_in <= 0 || max_tokens < 1 || max_tokens > 8) return B200AWQ_EINVAL;
  // A MoE op folds as two linears: gate|up (x [H] -> the recorded gate_up [top_k, 2I], N = top_k 2I) and down (the
  // recorded activations [top_k, I] -> y [H], K = top_k I); a DEEPSEEK_MOE op's shared expert widens both by I_s.  The
  // hazard rules below then see every buffer they touch.  Only the stream kernel runs them (M = 1; stream_build checks
  // the envelope); otherwise the caller replays per op.
  FoldedProgram f;
  std::vector<ProgOp>& table = f.table;
  std::vector<MoeBlock>& moes = f.moes;
  std::vector<b200awq_op_t> xops;
  std::vector<std::pair<int, int>> xmoe;   // per entry of xops: ProgOp::moe and ProgOp::mi
  for (int i = 0; i < n_in; ++i) {
    const b200awq_op_t& op = ops_in[i];
    if (op.kind != B200AWQ_OP_SPARSE_MOE && op.kind != B200AWQ_OP_QWEN3_MOE && op.kind != B200AWQ_OP_DEEPSEEK_MOE) {
      xops.push_back(op);
      xmoe.emplace_back(0, -1);
      continue;
    }
    const bool ds = op.kind == B200AWQ_OP_DEEPSEEK_MOE;
    const b200awq_deepseek_moe_t* dd = ds ? static_cast<const b200awq_deepseek_moe_t*>(op.weight) : nullptr;
    const b200awq_moe_t* m = ds ? (dd != nullptr ? &dd->moe : nullptr) : static_cast<const b200awq_moe_t*>(op.weight);
    if (m == nullptr || op.x == nullptr || op.y == nullptr || m->gate_weight == nullptr || m->w1_qweight == nullptr ||
        m->w1_scales == nullptr || m->w1_qzeros == nullptr || m->w2_qweight == nullptr || m->w2_scales == nullptr ||
        m->w2_qzeros == nullptr || m->logits == nullptr || m->topk_weights == nullptr || m->topk_ids == nullptr ||
        m->token_expert_indices == nullptr || m->sorted_ids == nullptr || m->expert_ids == nullptr ||
        m->num_tokens_post_pad == nullptr || m->gate_up == nullptr || m->act == nullptr || m->down == nullptr)
      return B200AWQ_EINVAL;
    if (m->E <= 0 || m->top_k <= 0 || m->top_k > m->E || m->H <= 0 || m->H != op.K || m->I <= 0 || m->group_size <= 0 ||
        (m->H % m->group_size) != 0 || (m->I % m->group_size) != 0 || m->block_size <= 0 ||
        m->sorted_len < m->top_k * op.M + m->E * (m->block_size - 1))
      return B200AWQ_EINVAL;
    int I_s = 0;
    if (ds) {
      if (dd->ws1_qweight == nullptr || dd->ws1_scales == nullptr || dd->ws1_qzeros == nullptr ||
          dd->ws2_qweight == nullptr || dd->ws2_scales == nullptr || dd->ws2_qzeros == nullptr ||
          dd->shared_out == nullptr || (dd->scoring == 1 && dd->bias == nullptr))
        return B200AWQ_EINVAL;
      if (dd->I_s <= 0 || (dd->I_s % m->group_size) != 0 || (dd->scoring != 0 && dd->scoring != 1) || dd->n_group <= 0 ||
          (m->E % dd->n_group) != 0 || dd->topk_group <= 0 || dd->topk_group > dd->n_group ||
          (dd->n_group > 1 && m->E / dd->n_group < 2))
        return B200AWQ_EINVAL;
      I_s = dd->I_s;
    }
    if (op.M != 1) return B200AWQ_EUNSUPPORTED;
    const int mi = static_cast<int>(moes.size());
    moes.push_back(MoeBlock{op.kind, {}});
    if (ds) moes.back().ds = *dd;
    else moes.back().ds.moe = *m;
    b200awq_op_t a;
    std::memset(&a, 0, sizeof(a));
    a.kind = B200AWQ_OP_LINEAR_GEMM;
    a.M = op.M;
    a.group_size = m->group_size;
    b200awq_op_t b = a;
    a.K = m->H;
    a.N = m->top_k * 2 * m->I + 2 * I_s;
    a.ldx = a.K;
    a.x = op.x;
    a.qweight = m->w1_qweight;
    a.scales = m->w1_scales;
    a.qzeros = m->w1_qzeros;
    a.y = m->gate_up;
    b.K = m->top_k * m->I + I_s;
    b.N = m->H;
    b.ldx = b.K;
    b.x = m->act;
    b.qweight = m->w2_qweight;
    b.scales = m->w2_scales;
    b.qzeros = m->w2_qzeros;
    b.y = op.y;
    xops.push_back(a);
    xmoe.emplace_back(1, mi);
    xops.push_back(b);
    xmoe.emplace_back(2, mi);
  }
  const b200awq_op_t* ops = xops.data();
  const int n = static_cast<int>(xops.size());
  struct Glue {
    int kind;
    const void* src;
    const void* w;
    const void* b;   // LAYER_NORM bias, or null
    void* out;
    int width;
    float eps;
    bool used;
    bool live;
  };
  std::vector<Glue> glues;
  // plan: the folding alone, for `plan->grid` SMs and residual window `plan->window`, without any CUDA call
  const int grid = plan != nullptr ? plan->grid : prog_sm_count();
  const int res_window = plan != nullptr && plan->window > 0 ? plan->window : kSpResWindow;
  int M = -1;
  // extents in bytes: M contiguous fp16 rows of `width`; an op's source (M rows at pitch src_ld, gate|up for SiLU*mul)
  // and output; a glue record's output and source
  auto rows_bytes = [&](int width) { return (size_t)(M > 0 ? M : 1) * width * 2; };
  auto src_bytes = [&](const ProgOp& p) {
    return ((size_t)(M - 1) * p.src_ld + (size_t)(p.prologue == kProSilu ? 2 : 1) * p.K) * 2;
  };
  auto y_bytes = [&](const ProgOp& p) { return rows_bytes(p.N); };
  auto glue_out_bytes = [&](const Glue& gl) { return rows_bytes(gl.width); };
  auto glue_src_bytes = [&](const Glue& gl) { return rows_bytes((gl.kind == kProSilu ? 2 : 1) * gl.width); };
  // a write over something a live glue record (other than `keep`) still needs ends that record; false: the record was
  // never used, so it would never run
  auto glue_write = [&](const void* p, size_t bytes, const Glue* keep) {
    for (Glue& gl : glues)
      if (gl.live && &gl != keep &&
          (overlaps(gl.out, glue_out_bytes(gl), p, bytes) || overlaps(gl.src, glue_src_bytes(gl), p, bytes))) {
        if (!gl.used) return false;
        gl.live = false;
      }
    return true;
  };
  // a read of a linear's raw output after an ADD was folded into it: its row carries the sum, not y
  auto reads_raw_y = [&](const void* p, size_t bytes) {
    for (const ProgOp& t : table)
      if (t.raw_y != nullptr && overlaps(t.raw_y, y_bytes(t), p, bytes)) return true;
    return false;
  };
  for (int i = 0; i < n; ++i) {
    const b200awq_op_t& op = ops[i];
    if (M < 0) M = op.M;
    if (op.M != M) return B200AWQ_EUNSUPPORTED;
    if (op.kind == B200AWQ_OP_ROPE_KV || op.kind == B200AWQ_OP_QK_NORM_ROPE_KV || op.kind == B200AWQ_OP_ROPE_KV_SEQ ||
        op.kind == B200AWQ_OP_QK_NORM_ROPE_KV_SEQ || op.kind == B200AWQ_OP_ROPE_KV_OFFSET) {
      // RoPE + cache append, folded into the finish of the linear recorded just before it (whose whole output is qkv);
      // QK_NORM_ROPE_KV: the same op on its embedded descriptor, with q / k normalised first.  The _SEQ kinds: T = op.K
      // tokens per sequence (M = B T rows; T > 1 needs M > 1, so only the batched kernels see it).  ROPE_KV_OFFSET: the
      // _SEQ kind its embedded descriptor's norm weights name (both null: no norm), with per-sequence rotary offsets
      const b200awq_rope_offset_t* od =
          op.kind == B200AWQ_OP_ROPE_KV_OFFSET ? static_cast<const b200awq_rope_offset_t*>(op.weight) : nullptr;
      if (op.kind == B200AWQ_OP_ROPE_KV_OFFSET && (od == nullptr || od->rot_offset == nullptr)) return B200AWQ_EINVAL;
      const bool qkn = op.kind == B200AWQ_OP_QK_NORM_ROPE_KV || op.kind == B200AWQ_OP_QK_NORM_ROPE_KV_SEQ ||
                       (od != nullptr && (od->qk.q_norm_weight != nullptr || od->qk.k_norm_weight != nullptr));
      const bool seq = op.kind == B200AWQ_OP_ROPE_KV_SEQ || op.kind == B200AWQ_OP_QK_NORM_ROPE_KV_SEQ || od != nullptr;
      const int T = seq ? op.K : 1;
      if (T < 1 || (M % T) != 0) return B200AWQ_EINVAL;
      const b200awq_qk_norm_rope_t* qd =
          od != nullptr ? &od->qk : qkn ? static_cast<const b200awq_qk_norm_rope_t*>(op.weight) : nullptr;
      const b200awq_rope_t* r = qd != nullptr ? &qd->rope : qkn ? nullptr : static_cast<const b200awq_rope_t*>(op.weight);
      if (op.x == nullptr) return B200AWQ_EINVAL;
      const int v = rope_validate(r, M > 1 ? op.ldx : INT64_MAX);   // (one row: no pitch; N is checked below)
      if (v != B200AWQ_OK) return v;
      if (qkn && (qd->q_norm_weight == nullptr || qd->k_norm_weight == nullptr)) return B200AWQ_EINVAL;
      if (qkn && (!aligned16(qd->q_norm_weight) || !aligned16(qd->k_norm_weight))) return B200AWQ_EUNSUPPORTED;
      const int D = r->head_dim;
      if (qkn && rope_rotary_dim(*r) != D) return B200AWQ_EUNSUPPORTED;   // q / k norm: full rotary only
      if (op.N != (r->n_heads + 2 * r->n_kv_heads) * D || (D % 16) != 0) return B200AWQ_EUNSUPPORTED;
      // (an ADD or a glue op in between: the op before is not a linear; a MoE block's ops are not plain linears)
      if (i == 0 || ops[i - 1].kind != B200AWQ_OP_LINEAR_GEMM || table.empty() || table.back().moe != 0)
        return B200AWQ_EUNSUPPORTED;
      ProgOp& pv = table.back();
      if (op.x != pv.y || op.N != pv.N || (M > 1 && op.ldx != op.N)) return B200AWQ_EUNSUPPORTED;
      if (qkn) pv.qkr = *qd;
      else pv.qkr.rope = *r;
      pv.rope_T = T;
      pv.rot_offset = od != nullptr ? od->rot_offset : nullptr;
      continue;
    }
    if (op.kind == B200AWQ_OP_MLA_ROPE || op.kind == B200AWQ_OP_MLA_KV || op.kind == B200AWQ_OP_MLA_K_ROPE ||
        op.kind == B200AWQ_OP_MLA_Q_ROPE) {
      // MLA's rotation / cache stores, folded into the finish of the linear recorded just before it (whose whole output
      // is the op's row): q_proj | kv_a_proj_with_mqa for MLA_ROPE, kv_b_proj for MLA_KV; with a q LoRA,
      // q_a_proj | kv_a_proj_with_mqa for MLA_K_ROPE and q_b_proj for MLA_Q_ROPE
      const bool mrope = op.kind == B200AWQ_OP_MLA_ROPE, krope = op.kind == B200AWQ_OP_MLA_K_ROPE;
      const bool qrope = op.kind == B200AWQ_OP_MLA_Q_ROPE;
      const b200awq_mla_t* d = static_cast<const b200awq_mla_t*>(op.weight);
      if (op.x == nullptr) return B200AWQ_EINVAL;
      const int v = mla_validate(d, op.kind);
      if (v != B200AWQ_OK) return v;
      if (M != 1) return B200AWQ_EUNSUPPORTED;
      if ((d->nope_dim % 16) != 0 || (d->rope_dim % 16) != 0 ||
          (mrope || krope ? d->kv_lora_rank : qrope ? 0 : d->v_dim) % 16 != 0)
        return B200AWQ_EUNSUPPORTED;
      const int64_t qn = (int64_t)d->n_heads * (d->nope_dim + d->rope_dim);
      if (krope) {   // [q_a (Cq) | c_kv | k_pe]: Cq = N - C - Dr
        const int64_t cq = (int64_t)op.N - d->kv_lora_rank - d->rope_dim;
        if (cq <= 0 || (cq % 16) != 0) return B200AWQ_EUNSUPPORTED;
      } else {
        const int64_t want = mrope ? qn + d->kv_lora_rank + d->rope_dim
                                   : qrope ? qn : (int64_t)d->n_heads * (d->nope_dim + d->v_dim);
        if (op.N != want) return B200AWQ_EUNSUPPORTED;
      }
      if (i == 0 || ops[i - 1].kind != B200AWQ_OP_LINEAR_GEMM || table.empty() || table.back().moe != 0)
        return B200AWQ_EUNSUPPORTED;
      ProgOp& pv = table.back();
      if (op.x != pv.y || op.N != pv.N) return B200AWQ_EUNSUPPORTED;
      pv.mla = *d;
      pv.mla_kind = mrope ? 1 : krope ? 3 : qrope ? 4 : 2;
      continue;
    }
    if (op.kind == B200AWQ_OP_ADD || op.kind == B200AWQ_OP_SCALED_ADD) {
      // y = x + weight, folded into the epilogue of the op recorded just before it (a linear / a MoE block's down);
      // SCALED_ADD: y = x + fp16(weight * eps), weight the producer's output (a linear's only)
      const bool scaled = op.kind == B200AWQ_OP_SCALED_ADD;
      if (op.x == nullptr || op.weight == nullptr || op.y == nullptr || op.K <= 0) return B200AWQ_EINVAL;
      if (scaled && !std::isfinite(op.eps)) return B200AWQ_EINVAL;
      if ((op.K % 8) != 0 || !aligned16(op.x) || !aligned16(op.weight) || !aligned16(op.y)) return B200AWQ_EUNSUPPORTED;
      const size_t bytes = rows_bytes(op.K);
      if (overlaps(op.y, bytes, op.x, bytes) || overlaps(op.y, bytes, op.weight, bytes)) return B200AWQ_EUNSUPPORTED;
      if (i == 0 || ops[i - 1].kind != B200AWQ_OP_LINEAR_GEMM || table.empty()) return B200AWQ_EUNSUPPORTED;
      ProgOp& pv = table.back();
      if (scaled && pv.moe != 0) return B200AWQ_EUNSUPPORTED;
      const void* r;                 // the residual: the operand that is not the producer's whole output
      if (op.weight == pv.y) r = op.x;
      else if (op.x == pv.y && !scaled) r = op.weight;
      else return B200AWQ_EUNSUPPORTED;  // neither operand is the producer's output (both external), or swapped scaled
      if (op.K != pv.N || overlaps(r, bytes, pv.y, bytes)) return B200AWQ_EUNSUPPORTED;
      // in-program residual: the newest op that wrote any of it must have published exactly it, kSpResWindow ops back
      int res_op = -1;
      for (int j = static_cast<int>(table.size()) - 2; j >= 0 && res_op < 0; --j) {
        const bool hit = overlaps(table[j].y, y_bytes(table[j]), r, bytes) ||
                         (table[j].raw_y != nullptr && overlaps(table[j].raw_y, y_bytes(table[j]), r, bytes));
        if (!hit) continue;
        if (r != table[j].y || table[j].N != op.K) return B200AWQ_EUNSUPPORTED;
        if (static_cast<int>(table.size()) - 1 - j > res_window) return B200AWQ_EUNSUPPORTED;
        res_op = j;
      }
      for (const Glue& gl : glues)   // a glue output is written by CTA slices, never published as a row
        if (overlaps(gl.out, glue_out_bytes(gl), r, bytes)) return B200AWQ_EUNSUPPORTED;
      // the output must not overlap what the producer reads (other CTAs may still be staging it) or publishes
      if (overlaps(op.y, bytes, pv.src, src_bytes(pv)) || (pv.xout != nullptr && overlaps(op.y, bytes, pv.xout, rows_bytes(pv.K))))
        return B200AWQ_EUNSUPPORTED;
      if (!glue_write(op.y, bytes, nullptr)) return B200AWQ_EUNSUPPORTED;
      pv.raw_y = pv.y;
      pv.res_op = res_op;
      pv.res_ext = res_op < 0 ? r : nullptr;
      if (scaled) pv.res_mul = op.eps;
      pv.y = static_cast<__half*>(op.y);   // the producer's row now publishes the sum
      continue;
    }
    if (op.kind == B200AWQ_OP_GELU || op.kind == B200AWQ_OP_GELU_TANH) {
      // y = gelu(x), folded into the finish of the linear recorded just before it, whose whole output x must be (as an
      // ADD folds: that linear's row then publishes the GELU's output, its raw y is stored on the side)
      if (op.x == nullptr || op.y == nullptr || op.K <= 0) return B200AWQ_EINVAL;
      if ((op.K % 8) != 0 || !aligned16(op.x) || !aligned16(op.y)) return B200AWQ_EUNSUPPORTED;
      if (M != 1 || max_tokens > 1) return B200AWQ_EUNSUPPORTED;   // batched programs replay per op
      const size_t bytes = rows_bytes(op.K);
      if (overlaps(op.y, bytes, op.x, bytes)) return B200AWQ_EUNSUPPORTED;   // in place
      // (an ADD, a glue op or a ROPE_KV / MLA op in between: the op before is not a linear; a MoE block's ops are not
      // plain linears; a linear carrying an ADD or a GELU already has raw_y)
      if (i == 0 || ops[i - 1].kind != B200AWQ_OP_LINEAR_GEMM || table.empty()) return B200AWQ_EUNSUPPORTED;
      ProgOp& pv = table.back();
      if (pv.moe != 0 || pv.raw_y != nullptr || op.x != pv.y || op.K != pv.N) return B200AWQ_EUNSUPPORTED;
      // the output must not overlap what the producer reads (other CTAs may still be staging it) or publishes
      if (overlaps(op.y, bytes, pv.src, src_bytes(pv)) || (pv.xout != nullptr && overlaps(op.y, bytes, pv.xout, rows_bytes(pv.K))))
        return B200AWQ_EUNSUPPORTED;
      if (!glue_write(op.y, bytes, nullptr)) return B200AWQ_EUNSUPPORTED;
      pv.raw_y = pv.y;
      pv.gelu = op.kind == B200AWQ_OP_GELU ? 1 : 2;
      pv.y = static_cast<__half*>(op.y);   // the producer's row now publishes the GELU's output
      continue;
    }
    if (op.kind == B200AWQ_OP_RMSNORM || op.kind == B200AWQ_OP_SILU_AND_MUL || op.kind == B200AWQ_OP_LAYER_NORM) {
      const bool ln = op.kind == B200AWQ_OP_LAYER_NORM;
      if (op.x == nullptr || op.y == nullptr || op.K <= 0) return B200AWQ_EINVAL;
      if (op.kind != B200AWQ_OP_SILU_AND_MUL && op.weight == nullptr) return B200AWQ_EINVAL;
      // an RMSNORM over rows of a wider tensor (ldx > K): the kernels stage contiguous rows only
      if (op.kind != B200AWQ_OP_SILU_AND_MUL && M > 1 && op.ldx != 0 && op.ldx != op.K) return B200AWQ_EUNSUPPORTED;
      if ((op.K % 8) != 0 || !aligned16(op.x) || !aligned16(op.y) || (op.weight != nullptr && !aligned16(op.weight)))
        return B200AWQ_EUNSUPPORTED;
      if (ln && (M != 1 || max_tokens > 1 || (op.bias != nullptr && !aligned16(op.bias)))) return B200AWQ_EUNSUPPORTED;
      const size_t in_bytes = (size_t)M * (op.kind == B200AWQ_OP_SILU_AND_MUL ? 2 : 1) * op.K * 2;
      if (overlaps(op.y, rows_bytes(op.K), op.x, in_bytes)) return B200AWQ_EUNSUPPORTED;  // in-place glue op
      if (!glue_write(op.y, rows_bytes(op.K), nullptr)) return B200AWQ_EUNSUPPORTED;
      if (reads_raw_y(op.x, in_bytes)) return B200AWQ_EUNSUPPORTED;
      // its input must not be a buffer only CTA 0 publishes
      for (const Glue& gl : glues)
        if (overlaps(gl.out, glue_out_bytes(gl), op.x, in_bytes)) return B200AWQ_EUNSUPPORTED;
      // a SiLU*mul of a GELU's output: its producer would have to be a mode-1 gate|up
      if (op.kind == B200AWQ_OP_SILU_AND_MUL)
        for (const ProgOp& t : table)
          if (t.gelu != 0 && overlaps(t.y, y_bytes(t), op.x, in_bytes)) return B200AWQ_EUNSUPPORTED;
      glues.push_back(Glue{op.kind == B200AWQ_OP_RMSNORM ? kProRmsnorm : ln ? kProLayernorm : kProSilu, op.x, op.weight,
                           ln ? op.bias : nullptr, op.y, op.K, op.eps, false, true});
      continue;
    }
    if (op.kind != B200AWQ_OP_LINEAR_GEMM) return B200AWQ_EINVAL;
    if (op.x == nullptr || op.qweight == nullptr || op.scales == nullptr || op.qzeros == nullptr || op.y == nullptr ||
        op.K <= 0 || op.N <= 0 || op.group_size <= 0 || (op.K % op.group_size) != 0)
      return B200AWQ_EINVAL;
    if (M < 1 || M > max_tokens) return B200AWQ_EUNSUPPORTED;
    if (M > 1 && op.ldx < op.K) return B200AWQ_EINVAL;
    ProgOp p;
    p.qw_src = static_cast<const int32_t*>(op.qweight);
    p.scales = static_cast<const __half*>(op.scales);
    p.qzeros = static_cast<const int32_t*>(op.qzeros);
    p.bias = static_cast<const __half*>(op.bias);
    p.y = static_cast<__half*>(op.y);
    p.K = op.K;
    p.N = op.N;
    p.G = op.group_size;
    p.moe = xmoe[i].first;
    p.mi = xmoe[i].second;
    Glue* hit = nullptr;
    for (Glue& gl : glues)
      if (gl.live && gl.out == op.x && gl.width == op.K) hit = &gl;
    if (hit != nullptr) {
      p.prologue = hit->kind;
      p.src = static_cast<const __half*>(hit->src);
      p.norm_w = static_cast<const __half*>(hit->w);
      p.ln_b = static_cast<const __half*>(hit->b);
      p.xout = hit->used ? nullptr : static_cast<__half*>(hit->out);   // published once, by its first consumer
      p.eps = hit->eps;
      p.src_ld = (hit->kind == kProSilu ? 2 : 1) * op.K;   // glue buffers are contiguous rows
      hit->used = true;
      if (M > 1 && op.ldx != op.K) return B200AWQ_EUNSUPPORTED;
    } else {
      p.prologue = kProCopy;
      p.src = static_cast<const __half*>(op.x);
      p.src_ld = M > 1 ? static_cast<int>(op.ldx) : op.K;
      if (!aligned16(op.x)) return B200AWQ_EUNSUPPORTED;
      for (const Glue& gl : glues)   // reading a buffer only CTA 0 publishes (a dead or mismatching record)
        if (overlaps(gl.out, glue_out_bytes(gl), op.x, src_bytes(p))) return B200AWQ_EUNSUPPORTED;
    }
    // the source's M rows (row pitch src_ld), this op's output (M rows of N)
    const size_t sb = src_bytes(p), yb = y_bytes(p);
    if (overlaps(p.y, yb, p.src, sb) || reads_raw_y(p.src, sb)) return B200AWQ_EUNSUPPORTED;
    if (p.xout != nullptr && overlaps(p.xout, rows_bytes(op.K), p.y, yb)) return B200AWQ_EUNSUPPORTED;
    if (!table.empty()) {
      // the previous op's fp16 output reaches memory only while THIS op stages its activations: a source inside it
      // is taken from the previous op's fp32 accumulators instead (same values), anything else touching it is a race
      const ProgOp& pv = table.back();
      const uintptr_t y0 = reinterpret_cast<uintptr_t>(pv.y), s0 = reinterpret_cast<uintptr_t>(p.src);
      if (s0 >= y0 && s0 + sb <= y0 + y_bytes(pv)) {
        if (((s0 - y0) & 15) != 0) return B200AWQ_EUNSUPPORTED;
        p.src_prev = 1;
        p.src_off = static_cast<int>((s0 - y0) / 2);
      } else if (overlaps(pv.y, y_bytes(pv), p.src, sb)) {
        return B200AWQ_EUNSUPPORTED;
      } else {
        // a source written by an older op of this program: wait for that op's duty-warp stores
        for (int j = static_cast<int>(table.size()) - 2; j >= 0; --j)
          if (overlaps(table[j].y, y_bytes(table[j]), p.src, sb)) {
            p.ext_dep = j;
            break;
          }
      }
      if (p.xout != nullptr && overlaps(p.xout, rows_bytes(op.K), pv.y, y_bytes(pv))) return B200AWQ_EUNSUPPORTED;
    }
    if (!glue_write(p.y, yb, hit)) return B200AWQ_EUNSUPPORTED;
    // a staging wait on the whole row of op s waits for every CTA that owns columns of s
    const int s = p.src_prev ? static_cast<int>(table.size()) - 1 : p.ext_dep;
    const size_t width = (size_t)(p.prologue == kProSilu ? 2 : 1) * op.K;
    p.stage_row = s >= 0 && p.src == table[s].y && width == (size_t)table[s].N ? s : -1;
    // a slice of an MLA_ROPE producer's row: stream_mla_kernel stages it after the whole row (SpMla::wait_words)
    if (s >= 0 && table[s].mla_kind == 1 && p.prologue != kProSilu) p.stage_row = s;
    // a slice of an MLA_K_ROPE producer's row (q_b's q_a slice, or kv_b's c_kv slice two ops back):
    // stream_mla_lora_kernel first polls one word of every set of the previous op's row (SpMla::wait_words), which
    // shows what staging that whole row shows
    if (s >= 0 && table[s].mla_kind == 3 && p.prologue != kProSilu && p.stage_row < 0 && table.back().moe == 0)
      p.stage_row = static_cast<int>(table.size()) - 1;
    table.push_back(p);
  }
  for (const Glue& gl : glues)
    if (!gl.used) return B200AWQ_EUNSUPPORTED;   // a glue op nobody consumes would never run
  if (table.empty()) return B200AWQ_EUNSUPPORTED;
  const int nt = static_cast<int>(table.size());
  // LAYER_NORM / GELU ops run on stream_layernorm_kernel, which has no MoE, q / k norm or MLA steps (no model mixes them)
  bool has_ln = false, has_other = !moes.empty();
  for (const ProgOp& t : table) {
    has_ln = has_ln || t.prologue == kProLayernorm || t.gelu != 0;
    has_other = has_other || t.qkr.q_norm_weight != nullptr || t.mla_kind != 0;
  }
  if (has_ln && has_other) return B200AWQ_EUNSUPPORTED;
  for (const ProgOp& t : table) {
    // an external residual is read at the finish of its op, any time during the run: nothing of the program may write it
    if (t.res_ext == nullptr) continue;
    const size_t eb = y_bytes(t);
    for (const ProgOp& o : table)
      if (overlaps(o.y, y_bytes(o), t.res_ext, eb) || (o.raw_y != nullptr && overlaps(o.raw_y, y_bytes(o), t.res_ext, eb)))
        return B200AWQ_EUNSUPPORTED;
    for (const Glue& gl : glues)
      if (overlaps(gl.out, glue_out_bytes(gl), t.res_ext, eb)) return B200AWQ_EUNSUPPORTED;
    for (const MoeBlock& b : moes) {
      const auto x = b.extents(M);
      for (int k = 0; k < MoeBlock::kMoeWrites; ++k)
        if (overlaps(x[k].first, x[k].second, t.res_ext, eb)) return B200AWQ_EUNSUPPORTED;
    }
  }
  // ROPE_KV: the rotated q and the appended cache rows are written in a finish, while other CTAs run later ops.  No
  // other op of the program may read or write them, nor write the position / frequency table the finish reads; the
  // producer must not be a gate|up whose product a SiLU*mul reads (its row would hold silu(gate) * up).
  // QK_NORM_ROPE_KV: its two norm weights are reads like the position and the frequency table; ROPE_KV_OFFSET: its B
  // rotary offsets too.  (the caches and the offsets: B = M / T entries)
  auto rope_outs = [&](const ProgOp& p) {
    const b200awq_rope_t& r = p.qkr.rope;
    const size_t cache =
        ((size_t)(M / p.rope_T - 1) * r.cache_batch_stride + (size_t)r.cache_len * r.n_kv_heads * r.head_dim) * 2;
    return std::array<std::pair<const void*, size_t>, 3>{
        {{r.q_out, (size_t)M * r.n_heads * r.head_dim * 2}, {r.k_cache, cache}, {r.v_cache, cache}}};
  };
  for (int ri = 0; ri < nt; ++ri) {
    const b200awq_qk_norm_rope_t& q = table[ri].qkr;
    const b200awq_rope_t& r = q.rope;
    if (r.head_dim == 0) continue;
    const auto outs = rope_outs(table[ri]);
    const size_t wn = q.q_norm_weight != nullptr ? (size_t)r.head_dim * 2 : 0;   // (null, 0: overlaps nothing)
    const size_t ob = table[ri].rot_offset != nullptr ? (size_t)(M / table[ri].rope_T) * 4 : 0;
    const std::pair<const void*, size_t> ins[5] = {{r.pos, 4}, {r.freqs, (size_t)r.freqs_len * rope_rotary_dim(r) * 4},
                                                   {q.q_norm_weight, wn}, {q.k_norm_weight, wn},
                                                   {table[ri].rot_offset, ob}};
    auto hits_out = [&](const void* p, size_t b) {
      for (const auto& o : outs)
        if (overlaps(o.first, o.second, p, b)) return true;
      return false;
    };
    auto hits_any = [&](const void* p, size_t b) {
      if (hits_out(p, b)) return true;
      for (const auto& in : ins)
        if (overlaps(in.first, in.second, p, b)) return true;
      return false;
    };
    if (overlaps(outs[0].first, outs[0].second, outs[1].first, outs[1].second) ||
        overlaps(outs[0].first, outs[0].second, outs[2].first, outs[2].second) ||
        overlaps(outs[1].first, outs[1].second, outs[2].first, outs[2].second))
      return B200AWQ_EUNSUPPORTED;
    for (int j = 0; j < nt; ++j) {
      const ProgOp& o = table[j];
      if (hits_any(o.y, y_bytes(o)) || (o.raw_y != nullptr && hits_any(o.raw_y, y_bytes(o))) ||
          (o.src != nullptr && hits_out(o.src, src_bytes(o))) || (o.res_ext != nullptr && hits_out(o.res_ext, y_bytes(o))))
        return B200AWQ_EUNSUPPORTED;
      if (o.prologue == kProSilu && overlaps(o.src, src_bytes(o), table[ri].y, y_bytes(table[ri])))
        return B200AWQ_EUNSUPPORTED;   // a SiLU*mul of the qkv output: the producer would be a mode-1 gate|up
      if (j != ri && o.qkr.rope.head_dim != 0)   // another ROPE_KV: its outputs are writes, its inputs reads
        for (const auto& w : rope_outs(o))
          if (hits_any(w.first, w.second)) return B200AWQ_EUNSUPPORTED;
    }
    for (const Glue& gl : glues)
      if (hits_any(gl.out, glue_out_bytes(gl)) || hits_out(gl.src, glue_src_bytes(gl))) return B200AWQ_EUNSUPPORTED;
    for (const MoeBlock& b : moes) {
      const auto x = b.extents(M);
      for (int k = 0; k < (int)x.size(); ++k)
        if (k < MoeBlock::kMoeWrites ? hits_any(x[k].first, x[k].second) : hits_out(x[k].first, x[k].second))
          return B200AWQ_EUNSUPPORTED;
    }
  }
  // MLA ops: the same rule as ROPE_KV for q_out, the caches, pos and (the rotations) freqs, against every op, glue
  // record, MoE block and ROPE_KV op.  A k rotation (MLA_ROPE, MLA_K_ROPE) and an MLA_KV may share k_cache: with the same
  // geometry they write disjoint columns of its rows (k_pe, k_nope); two k rotations may not.  q LoRA ops (MLA_K_ROPE,
  // MLA_Q_ROPE) and MLA_ROPE ops do not mix in one program (their kernels poll different rows, SpMla::wait_words).
  bool has_mla_rope = false, has_mla_lora = false;
  for (const ProgOp& p : table) {
    has_mla_rope = has_mla_rope || p.mla_kind == 1;
    has_mla_lora = has_mla_lora || p.mla_kind >= 3;
  }
  if (has_mla_rope && has_mla_lora) return B200AWQ_EUNSUPPORTED;
  auto mla_outs = [&](const ProgOp& p) {
    const b200awq_mla_t& d = p.mla;
    const bool q = p.mla_kind == 1 || p.mla_kind == 4, k = p.mla_kind != 4, v = p.mla_kind == 2;
    const size_t kb = ((size_t)(M - 1) * d.k_batch_stride + (size_t)d.cache_len * d.n_heads * (d.nope_dim + d.rope_dim)) * 2;
    const size_t vb = ((size_t)(M - 1) * d.v_batch_stride + (size_t)d.cache_len * d.n_heads * d.v_head_stride) * 2;
    return std::array<std::pair<const void*, size_t>, 3>{
        {{q ? d.q_out : nullptr, q ? (size_t)M * d.n_heads * (d.nope_dim + d.rope_dim) * 2 : 0},
         {k ? d.k_cache : nullptr, k ? kb : 0},
         {v ? d.v_cache : nullptr, v ? vb : 0}}};
  };
  auto shares_k = [&](const ProgOp& a, const ProgOp& b) {
    const b200awq_mla_t &x = a.mla, &y = b.mla;
    return (a.mla_kind == 2) != (b.mla_kind == 2) && x.k_cache == y.k_cache && x.n_heads == y.n_heads &&
           x.nope_dim == y.nope_dim && x.rope_dim == y.rope_dim && x.cache_len == y.cache_len &&
           x.k_batch_stride == y.k_batch_stride;
  };
  for (int ri = 0; ri < nt; ++ri) {
    const ProgOp& mp = table[ri];
    if (mp.mla_kind == 0) continue;
    const b200awq_mla_t& d = mp.mla;
    const auto outs = mla_outs(mp);
    const std::pair<const void*, size_t> ins[2] = {
        {d.pos, 4}, {mp.mla_kind != 2 ? d.freqs : nullptr, mp.mla_kind != 2 ? (size_t)d.freqs_len * d.rope_dim * 4 : 0}};
    auto hits_out = [&](const void* p, size_t b) {
      for (const auto& o : outs)
        if (overlaps(o.first, o.second, p, b)) return true;
      return false;
    };
    // (skip: the one output of this op the other write may overlap, or -1)
    auto hits_any = [&](const void* p, size_t b, int skip = -1) {
      for (int k = 0; k < 3; ++k)
        if (k != skip && overlaps(outs[k].first, outs[k].second, p, b)) return true;
      for (const auto& in : ins)
        if (overlaps(in.first, in.second, p, b)) return true;
      return false;
    };
    for (int a = 0; a < 3; ++a)
      for (int b = a + 1; b < 3; ++b)
        if (overlaps(outs[a].first, outs[a].second, outs[b].first, outs[b].second)) return B200AWQ_EUNSUPPORTED;
    for (int j = 0; j < nt; ++j) {
      const ProgOp& o = table[j];
      if (hits_any(o.y, y_bytes(o)) || (o.raw_y != nullptr && hits_any(o.raw_y, y_bytes(o))) ||
          (o.src != nullptr && hits_out(o.src, src_bytes(o))) || (o.res_ext != nullptr && hits_out(o.res_ext, y_bytes(o))))
        return B200AWQ_EUNSUPPORTED;
      if (o.qkr.rope.head_dim != 0) {   // a ROPE_KV: its outputs are writes, its inputs reads
        const b200awq_qk_norm_rope_t& q = o.qkr;
        for (const auto& w : rope_outs(o))
          if (hits_any(w.first, w.second)) return B200AWQ_EUNSUPPORTED;
        const size_t wn = q.q_norm_weight != nullptr ? (size_t)q.rope.head_dim * 2 : 0;
        const size_t ob = o.rot_offset != nullptr ? (size_t)(M / o.rope_T) * 4 : 0;
        if (hits_out(q.rope.pos, 4) || hits_out(q.rope.freqs, (size_t)q.rope.freqs_len * rope_rotary_dim(q.rope) * 4) ||
            hits_out(q.q_norm_weight, wn) || hits_out(q.k_norm_weight, wn) || hits_out(o.rot_offset, ob))
          return B200AWQ_EUNSUPPORTED;
      }
      if (j != ri && o.mla_kind != 0) {   // another MLA op: its outputs are writes (its reads: its own pass of this loop)
        const auto w = mla_outs(o);
        for (int k = 0; k < 3; ++k)
          if (hits_any(w[k].first, w[k].second, k == 1 && shares_k(mp, o) ? 1 : -1)) return B200AWQ_EUNSUPPORTED;
      }
    }
    for (const Glue& gl : glues)
      if (hits_any(gl.out, glue_out_bytes(gl)) || hits_out(gl.src, glue_src_bytes(gl))) return B200AWQ_EUNSUPPORTED;
    for (const MoeBlock& b : moes) {
      const auto x = b.extents(M);
      for (int k = 0; k < (int)x.size(); ++k)
        if (k < MoeBlock::kMoeWrites ? hits_any(x[k].first, x[k].second) : hits_out(x[k].first, x[k].second))
          return B200AWQ_EUNSUPPORTED;
    }
  }
  for (int i = 0; i < nt; ++i) {
    // An in-program residual (row j % 4) is read in op i's finish, by the CTA that published those columns in op j (same
    // width, same partition).  Ops j + 4, j + 8, ... publish into that row again.  Op i itself (i = j + 4) only rewrites
    // the words each thread has just read; the next one after i, op k, may overwrite them only once every CTA has
    // finished op i: some op in (i, k] must stage the WHOLE row of an op >= i that every CTA owns columns of (a wait on a
    // slice of a row, or on a narrow op, waits for a few CTAs only).  tests/test_stream_residual_model.py replays random
    // programs through this rule (b200awq_program_plan).
    const int j = table[i].res_op;
    if (j < 0) continue;
    int k = j + kSpRows;
    while (k <= i) k += kSpRows;
    if (k >= nt) continue;
    int reach = -1;
    for (int m = i + 1; m <= k; ++m) {
      const int s = table[m].stage_row;
      if (s >= 0 && table[s].N / 16 >= grid) reach = std::max(reach, s);
    }
    if (reach < i) return B200AWQ_EUNSUPPORTED;
  }
  if (plan != nullptr) {
    plan->kernel_ops = nt;
    return B200AWQ_OK;
  }

  if (knob(14) == 1) return B200AWQ_EUNSUPPORTED;   // knob 14 = 1: do not fuse (the caller replays per op)

  Program* pr = new Program();
  pr->n_ops = nt;
  pr->M = M;
  cudaError_t e = cudaGetDevice(&pr->device);
  if (e == cudaSuccess && stream_build(pr, f, grid, &e)) {
    *out = pr;
    return B200AWQ_OK;
  }
  delete pr;
  if (e != cudaSuccess) {
    *cuda_err = e;
    return B200AWQ_ECUDA;
  }
  return B200AWQ_EUNSUPPORTED;
}

int program_m(const Program* p) { return p->M; }
int program_num_ops(const Program* p) { return p->n_ops; }

size_t program_stream_bytes(const Program* p) { return p->stream_bytes; }

cudaError_t program_run(Program* p, cudaStream_t st) {
  cudaError_t e = program_abort_clear(st);
  if (e != cudaSuccess) return e;
  const ProgKernel k = p->kernel;
  // knob 9: consumer warps of the plain M = 1 kernel: 8 (4 units in flight; the default) or 12 (2 units), each with the
  // ring depth chosen at creation (at least 4 / 3 stages).  No 16-warp variant: 17 warps put 5 on one of the SM's four
  // register-file partitions, which caps a thread at 96 registers on sm_90 and spills the unit loop.  Every other
  // kernel runs 8 warps; a batched one the ring depth chosen at creation, at MT = the smallest of 2 / 4 / 8 >= M.
  const int nw = k == kKernPlain && knob(9) == 12 ? 12 : 8;
  const int spw = nw == 8 ? p->sp_spw8 : p->sp_spw12;
  const int grid = prog_sm_count();
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(32 + nw * 32);
  cfg.dynamicSmemBytes = p->xs_bytes + (p->M > 1 ? sb_fixed_smem(p->sb_spw, p->sb_lmax, sb_mt(p->M), p->sb_nu_max)
                                                 : sp_fixed_smem(nw, spw, k != kKernPlain));
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;   // all CTAs co-resident: the hand-off polls are grid-wide waits
  attr[0].val.cooperative = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  int l2_ahead = 0, gate_ahead = 0;
  if (p->M == 1) {
    // knob 8: the HBM -> L2 run-ahead window of the weight stream, grid-wide, in MB, at most the device's L2 (<= 0:
    // off, the default).  The producer advances its prefetch cursor only while it has no ring stage to fill - during op
    // hand-offs and tails - and each of its grid x nw lanes keeps at most window / (grid x nw) bytes ahead of its ring.
    // Off is the default: on the bench step no window beat it by more than its run-to-run spread (H100 SXM, DESIGN
    // 3.5b: 8 and 16 MB within 0.5 %, 32 MB 4 % slower).
    const size_t window = knob(8) <= 0 ? 0 : std::min((size_t)knob(8) << 20, (size_t)p->l2_bytes);
    l2_ahead = (int)(window / ((size_t)grid * nw));
    // knob 10: ops ahead of the consumers' staging for which shared-memory loads may already be issued (0 = ungated,
    // the default: a gate of 2 measured 1.5-2 % slower on the bench step, DESIGN 3.5b; n > 0: at most n - 1 ops ahead,
    // 1 = strictly gated)
    gate_ahead = knob(10) <= 0 ? 1 << 20 : knob(10) - 1;
  }
  auto batch = [&](auto kern, auto... side) {
    return cudaLaunchKernelEx(&cfg, kern, p->d_sp_ops, p->d_cta, p->n_ops, p->d_rows, p->row_stride, p->d_state, p->M,
                              p->sb_spw, p->sb_lmax, p->sb_nu_max, knob(3), side...);
  };
  auto stream = [&](auto kern, auto... side) {   // (d_moe: null without MoE blocks)
    return cudaLaunchKernelEx(&cfg, kern, p->d_sp_ops, p->d_cta, p->n_ops, p->d_rows, p->row_stride, p->d_state, spw,
                              knob(3), l2_ahead, gate_ahead, p->d_moe, side...);
  };
  switch (k) {
    case kKernPlain: return nw == 8 ? stream(stream_program_kernel<8, 4>) : stream(stream_program_kernel<12, 2>);
    case kKernMoe: return stream(stream_moe_kernel);
    case kKernResidual: return stream(stream_residual_kernel, p->d_res);
    case kKernRope: return stream(stream_rope_kernel, p->d_res, p->d_rope);
    case kKernLayerNorm: return stream(stream_layernorm_kernel, p->d_res, p->d_rope, p->d_ln);
    case kKernQkNorm: return stream(stream_qknorm_kernel, p->d_res, p->d_rope, p->d_qkn);
    case kKernQwen3Moe: return stream(stream_qwen3moe_kernel, p->d_res, p->d_rope, p->d_qkn);
    case kKernDeepseekMoe: return stream(stream_deepseek_moe_kernel, p->d_res, p->d_rope, p->d_qkn, p->d_dsk);
    case kKernMla: return stream(stream_mla_kernel, p->d_res, p->d_rope, p->d_qkn, p->d_dsk, p->d_mla);
    case kKernMlaLora: return stream(stream_mla_lora_kernel, p->d_res, p->d_rope, p->d_qkn, p->d_dsk, p->d_mla);
    case kKernBatch2: return batch(stream_batch_kernel<2>);
    case kKernBatch4: return batch(stream_batch_kernel<4>);
    case kKernBatch8: return batch(stream_batch_kernel<8>);
    case kKernBatchResidual2: return batch(stream_batch_residual_kernel<2>, p->d_res);
    case kKernBatchResidual4: return batch(stream_batch_residual_kernel<4>, p->d_res);
    case kKernBatchResidual8: return batch(stream_batch_residual_kernel<8>, p->d_res);
    case kKernBatchRope2: return batch(stream_batch_rope_kernel<2>, p->d_res, p->d_rope_seq);
    case kKernBatchRope4: return batch(stream_batch_rope_kernel<4>, p->d_res, p->d_rope_seq);
    case kKernBatchRope8: return batch(stream_batch_rope_kernel<8>, p->d_res, p->d_rope_seq);
    case kKernBatchQkNorm2: return batch(stream_batch_qknorm_kernel<2>, p->d_res, p->d_rope_seq, p->d_qkn);
    case kKernBatchQkNorm4: return batch(stream_batch_qknorm_kernel<4>, p->d_res, p->d_rope_seq, p->d_qkn);
    case kKernBatchQkNorm8: return batch(stream_batch_qknorm_kernel<8>, p->d_res, p->d_rope_seq, p->d_qkn);
  }
  return cudaErrorInvalidValue;   // (not reached: stream_build sets one of the above)
}

void program_destroy(Program* p) { delete p; }

}  // namespace b200awq
