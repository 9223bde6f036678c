// Decode program: the chain of operator calls of a decode step (RMSNorm -> W4A16 linear -> ... -> SiLU*mul -> linear,
// sparse-MoE blocks, residual adds) recorded once and executed by ONE persistent kernel launch.
//
// Why: a stand-alone GEMV launch spends microseconds outside the weight stream - launch + ring fill (the first tile
// lands after the loaded HBM latency), the split-K tail, the ticket round trip - and HBM idles through every one of
// those gaps, 128 times per decode step.  The packed weights never depend on the activations, so the producer warp of
// every CTA walks the WHOLE op list and keeps its shared-memory ring full across op boundaries.
//
// This file is the host side of the stream kernels (program_stream.cuh: M = 1, with or without sparse-MoE blocks and
// residual adds; program_batch.cuh: M = 2..8) plus what those kernels share:
//   * program_create folds the recorded calls into a table of linears, each with the glue op that feeds it as an
//     activation prologue, and enforces the hazard rules the kernels' ordering relies on;
//   * stream_build re-lays out every linear once into the stream format and builds the kernels' op table; a
//     sequence outside their envelope is not fused (B200AWQ_EUNSUPPORTED: the caller replays it per op);
//   * program_run launches the kernel that matches the program;
//   * the watchdog of every spin loop (ProgWatch, g_prog_abort) and the per-op phase timestamps (g_prog_dbg).
//
// Reference call sequence this replaces: awq/modules/fused/block.py:117-170 (norm -> qkv -> ... -> o -> norm ->
// mlp) with awq/modules/fused/mlp.py:41-55 (gate/up GEMM, silu*mul, down GEMM), each a separate awq_ext call.
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../include/b200awq.h"
#include "common.cuh"
#include "gemv_tile.cuh"
#include "kernels.h"
#include "rope.cuh"

namespace b200awq {

enum { kProCopy = 0, kProRmsnorm = 1, kProSilu = 2 };

// One entry of the fold table program_create builds (host only): a linear and the activation prologue that feeds it.
// stream_build turns the table into the kernels' SpOp table.
struct ProgOp {
  const __half* scales;
  const int32_t* qzeros;
  const __half* bias;
  __half* y;
  const __half* src;      // external source (fp16, global) when !src_prev: COPY x, RMSNORM row, SILU gate|up
  const __half* norm_w;   // RMSNORM weight [K]
  __half* xout;           // where the recorded glue op wanted its result, or null
  int src_off;            // src_prev: first column of the previous op's output this op reads
  int src_prev;           // 1: the source is the previous op's output
  int K, N, G;
  int prologue;
  float eps;
  int ext_dep;            // >= 0: the external source was written by that (older) op of this program
  const int32_t* qw_src;  // the checkpoint-format qweight (re-laid-out by stream_build)
  int src_ld;             // row pitch of src in elements (M > 1)
};

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
struct Program {
  int n_ops = 0;
  int M = 0;
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
  // sparse-MoE blocks (stream_moe_kernel): their descriptors
  SpMoe* d_moe = nullptr;
  int n_moe = 0;
  unsigned long long* d_xlog = nullptr;   // QWEN3_MOE blocks: their published router logits ([E] words per block)
  bool qwen3 = false;                      // QWEN3_MOE blocks: stream_qwen3moe_kernel
  SpDsk* d_dsk = nullptr;                  // DEEPSEEK_MOE blocks (stream_deepseek_moe_kernel): one SpDsk per block
  // residual adds (stream_residual_kernel / stream_batch_residual_kernel): one SpRes per kernel op, null without adds
  SpRes* d_res = nullptr;
  // ROPE_KV ops (stream_rope_kernel / stream_batch_rope_kernel): one SpRope per kernel op, null without them (d_res is
  // then allocated too, empty where there is no add: the rope kernels are the residual kernels plus the rope steps)
  SpRope* d_rope = nullptr;
  // QK_NORM_ROPE_KV ops (stream_qknorm_kernel / stream_batch_qknorm_kernel): one SpQkNorm per kernel op and the published
  // set partials of their heads, null without them (d_res and d_rope are then allocated too)
  SpQkNorm* d_qkn = nullptr;
  unsigned long long* d_qkn_part = nullptr;
};

// An ADD folded into table entry i (program_create): the entry's y is swapped for the ADD's output (what its row
// publishes, so the hazard rules resolve later readers to the row); raw_y is the linear's own output, still stored
struct ResFold {
  const void* raw_y = nullptr;   // null: no ADD folded into this entry
  const void* ext = nullptr;     // external residual (no op of the program writes it)
  int op = -1;                   // >= 0: the residual is that older entry's published row
};

// One SPARSE_MOE op as the folding sees it: two table entries (gate|up, down) and the recorded descriptor
struct MoeFold {
  int kind = 0;        // 0: plain linear, 1: gate|up of block `mi`, 2: its down
  int mi = -1;
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
  return mode == 0 || mode == 1;
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
                               int G, int head_dim, cudaStream_t st) {
  if (!stream_format_supported(K, N, G, 0) || head_dim <= 0 || (head_dim % 16) != 0 || (N % head_dim) != 0)
    return cudaErrorNotSupported;
  const int UK = G < 128 ? G : 128;
  const int64_t total = (int64_t)(N / 16) * (K / UK) * ((UK / 16) * 32 + 12);
  const int cap = prog_sm_count() * 16;
  const int blocks = (int)((total + 255) / 256 < cap ? (total + 255) / 256 : cap);
  stream_pack_rotary_kernel<<<blocks, 256, 0, st>>>(qweight, static_cast<const __half*>(scales), qzeros,
                                                    static_cast<uint8_t*>(out), K, N, G, head_dim);
  return cudaGetLastError();
}

cudaError_t stream_pack(const int32_t* qweight, const void* scales, const int32_t* qzeros, void* out, int K, int N, int G,
                        int mode, cudaStream_t st) {
  if (!stream_format_supported(K, N, G, mode)) return cudaErrorNotSupported;
  const int UK = G < 128 ? G : 128;
  const int64_t total = (int64_t)(N / 16) * (K / UK) * ((UK / 16) * 32 + 12);
  const int cap = prog_sm_count() * 16;
  const int blocks = (int)((total + 255) / 256 < cap ? (total + 255) / 256 : cap);
  stream_pack_kernel<<<blocks, 256, 0, st>>>(qweight, static_cast<const __half*>(scales), qzeros,
                                             static_cast<uint8_t*>(out), K, N, G, mode);
  return cudaGetLastError();
}

// Builds the stream kernels' program from the folded op table, for M token rows (M > 1: the batched kernel of
// program_batch.cuh).  Returns false when the sequence is outside their envelope.  *err != cudaSuccess reports a CUDA
// failure.
// Sparse-MoE blocks (`fold[i].kind` != 0, M = 1 only): the gate|up entry is a mode-1 op over top_k slots of 2I
// columns, the down entry reads its published row (K' = top_k I); both stream E per-expert slices packed back to back.
// ROPE_KV ops (`ropes[i].head_dim` != 0): entry i is packed in mode 2 and its finish rotates / appends (SpRope).
// QK_NORM_ROPE_KV ops: as ROPE_KV, and `qkns[i]` carries the norm weights (q_norm_weight != null: SpQkNorm).
static bool stream_build(Program* pr, const std::vector<ProgOp>& table, int grid, int M, cudaError_t* err,
                         const std::vector<MoeFold>& fold, const std::vector<b200awq_moe_t>& moes,
                         const std::vector<ResFold>& res, const std::vector<b200awq_rope_t>& ropes,
                         const std::vector<b200awq_qk_norm_rope_t>& qkns, const std::vector<int>& moe_hf,
                         const std::vector<b200awq_deepseek_moe_t>& dsks) {
  *err = cudaSuccess;
  const int n = static_cast<int>(table.size());
  if (n >= 60000) return false;
  const bool has_moe = !moes.empty();
  if (has_moe && M != 1) return false;
  // moe_hf: 0 SPARSE_MOE, 1 QWEN3_MOE, 2 DEEPSEEK_MOE.  A QWEN3_MOE (DEEPSEEK_MOE) program runs stream_qwen3moe_kernel
  // (stream_deepseek_moe_kernel), whose MoE blocks are all of that kind
  const int mkind = moe_hf.empty() ? 0 : moe_hf[0];
  if (std::find_if(moe_hf.begin(), moe_hf.end(), [&](int k) { return k != mkind; }) != moe_hf.end()) return false;
  const bool has_hf = mkind != 0, has_ds = mkind == 2;
  std::vector<int> plan_a(moes.size() * 8);
  for (size_t b = 0; b < moes.size(); ++b) {
    const b200awq_moe_t& m = moes[b];
    const int rc = moe_hf[b] == 2 ? deepseek_moe_plan(m.E, m.top_k, m.H, m.I, dsks[b].I_s, m.group_size, grid, &plan_a[b * 8])
                                  : (moe_hf[b] ? qwen3_moe_plan : moe_plan)(m.E, m.top_k, m.H, m.I, m.group_size, grid,
                                                                             &plan_a[b * 8]);
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
  auto moe_kind = [&](int i) { return fold.empty() ? 0 : fold[i].kind; };
  // bytes of one expert's slice of a MoE entry's stream copy (256-byte aligned)
  auto expert_bytes = [&](int i) {
    const b200awq_moe_t& m = moes[fold[i].mi];
    const size_t b = moe_kind(i) == 1 ? stream_format_bytes(m.H, 2 * m.I, m.group_size)
                                      : stream_format_bytes(m.I, m.H, m.group_size);
    return (b + 255) & ~(size_t)255;
  };
  // bytes of the shared expert's stream copy of a DEEPSEEK_MOE entry (in front of its expert slices; 0 otherwise)
  auto shared_bytes = [&](int i) {
    if (moe_hf[fold[i].mi] != 2) return (size_t)0;
    const b200awq_moe_t& m = moes[fold[i].mi];
    const int I_s = dsks[fold[i].mi].I_s;
    const size_t b = moe_kind(i) == 1 ? stream_format_bytes(m.H, 2 * I_s, m.group_size)
                                      : stream_format_bytes(I_s, m.H, m.group_size);
    return (b + 255) & ~(size_t)255;
  };
  for (int i = 0; i < n; ++i)
    if (moe_kind(i) == 1) mode[i] = 1;
  bool has_rope = false;
  for (int i = 0; i < n && !ropes.empty(); ++i)
    if (ropes[i].head_dim != 0) {
      if (mode[i] != 0) return false;   // (program_create rejects a gate|up producer already)
      mode[i] = 2;
      has_rope = true;
    }
  // residual adds: the producer and an in-program residual must publish plain columns (a mode-1 row holds SiLU*mul)
  bool has_res = false;
  for (int i = 0; i < n && !res.empty(); ++i)
    if (res[i].raw_y != nullptr) {
      if (mode[i] == 1 || (res[i].op >= 0 && mode[res[i].op] == 1)) return false;
      has_res = true;
    }
  size_t wbytes = 0, max_cols = 0;
  int max_K = 0, lmax = 0, nu_max = 0;
  std::vector<size_t> woff(n);
  for (int i = 0; i < n; ++i) {
    const ProgOp& p = table[i];
    if (moe_kind(i) != 0) {   // envelope checked by moe_plan (per-expert shapes, sets and partial rows per CTA)
      woff[i] = wbytes;
      wbytes += shared_bytes(i) + (size_t)moes[fold[i].mi].E * expert_bytes(i);
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
    const bool moe_k = has_moe || has_res || has_rope;
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
    o.y = (!res.empty() && res[i].raw_y != nullptr) ? static_cast<__half*>(const_cast<void*>(res[i].raw_y)) : p.y;
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
      o.xout = p.prologue == kProRmsnorm ? p.xout : nullptr;
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
    if (moe_kind(i) != 0) {
      o.moe = moe_kind(i);
      o.moe_i = fold[i].mi;
      if (o.moe == 2) {
        // the down entry stages the gate|up entry's published SiLU*mul row (top_k x I words, slot-major); the recorded
        // activation tensor is written as a side effect of that entry
        if (i == 0 || moe_kind(i - 1) != 1 || fold[i - 1].mi != fold[i].mi) return false;
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
  if (e == cudaSuccess) e = cudaMalloc(&pr->d_sp_ops, (size_t)n * sizeof(SpOp));
  if (e == cudaSuccess) e = cudaMalloc(&pr->d_cta, cta.size() * sizeof(uint32_t));
  const size_t row_bytes = (size_t)kSpRows * M * pr->row_stride * sizeof(uint32_t);   // M hand-off rows per op
  if (e == cudaSuccess) e = cudaMalloc(&pr->d_rows, row_bytes);
  if (e == cudaSuccess) e = cudaMalloc(&pr->d_state, 2 * sizeof(int));
  if (e == cudaSuccess) e = cudaMemset(pr->d_rows, 0, row_bytes);
  if (e == cudaSuccess) e = cudaMemset(pr->d_state, 0, 2 * sizeof(int));
  for (int i = 0; i < n && e == cudaSuccess; ++i) {
    ops[i].wstream = pr->d_stream + woff[i];
    ops[i].cta_begin = pr->d_cta + (size_t)i * (grid + 1);
    if (moe_kind(i) != 0) {
      // one stream copy per expert slice of the stacked tensors ([E, K, N/8], [E, K/G, N], [E, K/G, N/8])
      const b200awq_moe_t& m = moes[fold[i].mi];
      const int K = moe_kind(i) == 1 ? m.H : m.I, N = moe_kind(i) == 1 ? 2 * m.I : m.H, G = m.group_size;
      const int32_t* qw = static_cast<const int32_t*>(table[i].qw_src);
      const size_t shb = shared_bytes(i);
      for (int x = 0; x < m.E && e == cudaSuccess; ++x)
        e = stream_pack(qw + (size_t)x * K * (N / 8), table[i].scales + (size_t)x * (K / G) * N,
                        table[i].qzeros + (size_t)x * (K / G) * (N / 8),
                        pr->d_stream + woff[i] + shb + (size_t)x * expert_bytes(i), K, N, G, mode[i], nullptr);
      if (shb != 0 && e == cudaSuccess) {   // DEEPSEEK_MOE: the shared expert's copy, first
        const b200awq_deepseek_moe_t& d = dsks[fold[i].mi];
        const bool gu = moe_kind(i) == 1;
        e = stream_pack(gu ? d.ws1_qweight : d.ws2_qweight, gu ? d.ws1_scales : d.ws2_scales,
                        gu ? d.ws1_qzeros : d.ws2_qzeros, pr->d_stream + woff[i], gu ? m.H : d.I_s, gu ? 2 * d.I_s : m.H,
                        G, mode[i], nullptr);
      }
      continue;
    }
    if (mode[i] == 2)
      e = stream_pack_rotary(table[i].qw_src, table[i].scales, table[i].qzeros, pr->d_stream + woff[i], table[i].K,
                             table[i].N, table[i].G, ropes[i].head_dim, nullptr);
    else
      e = stream_pack(table[i].qw_src, table[i].scales, table[i].qzeros, pr->d_stream + woff[i], table[i].K, table[i].N,
                      table[i].G, mode[i], nullptr);
  }
  if (e == cudaSuccess && has_moe) {
    // QWEN3_MOE blocks: [E] logit words each, zero (no run's tag) until the first run
    size_t xwords = 0;
    for (size_t b = 0; b < moes.size(); ++b) xwords += moe_hf[b] ? (size_t)moes[b].E : 0;
    if (xwords > 0) e = cudaMalloc(&pr->d_xlog, xwords * sizeof(unsigned long long));
    if (e == cudaSuccess && xwords > 0) e = cudaMemset(pr->d_xlog, 0, xwords * sizeof(unsigned long long));
    size_t xoff = 0;
    std::vector<SpMoe> md(moes.size());
    for (size_t b = 0; b < moes.size(); ++b) {
      const b200awq_moe_t& m = moes[b];
      SpMoe& d = md[b];
      std::memset(&d, 0, sizeof(d));
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
      if (moe_hf[b]) {
        d.xlog = pr->d_xlog + xoff;
        xoff += (size_t)m.E;
      }
      for (int i = 0; i < n; ++i)
        if (moe_kind(i) != 0 && fold[i].mi == (int)b) (moe_kind(i) == 1 ? d.eb_a : d.eb_b) = (long long)expert_bytes(i);
    }
    if (e == cudaSuccess) e = cudaMalloc(&pr->d_moe, md.size() * sizeof(SpMoe));
    if (e == cudaSuccess) e = cudaMemcpy(pr->d_moe, md.data(), md.size() * sizeof(SpMoe), cudaMemcpyHostToDevice);
    pr->n_moe = static_cast<int>(md.size());
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(stream_moe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                               (int)(227 * 1024));
    if (e == cudaSuccess && has_ds) {
      std::vector<SpDsk> dd(moes.size());
      for (size_t b = 0; b < moes.size(); ++b) {
        const b200awq_deepseek_moe_t& d = dsks[b];
        SpDsk& x = dd[b];
        std::memset(&x, 0, sizeof(x));
        x.bias = d.bias;
        x.shared_out = static_cast<__half*>(d.shared_out);
        x.scoring = d.scoring;
        x.n_group = d.n_group;
        x.topk_group = d.topk_group;
        x.norm = d.norm_topk_prob != 0;
        x.rsf = d.routed_scaling_factor;
        x.nsh = d.I_s / d.moe.I;
        for (int i = 0; i < n; ++i)
          if (moe_kind(i) != 0 && fold[i].mi == (int)b) (moe_kind(i) == 1 ? x.shb_a : x.shb_b) = (long long)shared_bytes(i);
      }
      e = cudaMalloc(&pr->d_dsk, dd.size() * sizeof(SpDsk));
      if (e == cudaSuccess) e = cudaMemcpy(pr->d_dsk, dd.data(), dd.size() * sizeof(SpDsk), cudaMemcpyHostToDevice);
      if (e == cudaSuccess)
        e = cudaFuncSetAttribute(stream_deepseek_moe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
    }
  }
  if (e == cudaSuccess && (has_res || has_rope || has_hf)) {
    std::vector<SpRes> rd(n);
    for (int i = 0; i < n; ++i) {
      std::memset(&rd[i], 0, sizeof(SpRes));
      rd[i].op = -1;
      if (res.empty() || res[i].raw_y == nullptr) continue;
      rd[i].out = table[i].y;                       // the ADD's output (the entry's y was swapped for it)
      rd[i].op = res[i].op;
      rd[i].ext = static_cast<const __half*>(res[i].ext);
    }
    e = cudaMalloc(&pr->d_res, (size_t)n * sizeof(SpRes));
    if (e == cudaSuccess) e = cudaMemcpy(pr->d_res, rd.data(), (size_t)n * sizeof(SpRes), cudaMemcpyHostToDevice);
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(stream_residual_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(stream_batch_residual_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(stream_batch_residual_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(stream_batch_residual_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
  }
  bool has_qkn = false;
  for (int i = 0; i < n && !qkns.empty(); ++i) has_qkn = has_qkn || qkns[i].q_norm_weight != nullptr;
  if (e == cudaSuccess && (has_qkn || has_hf)) {
    // the partials of op i live at [M][N_i / 16] words from its offset; zero tags are never a run's (sp_tag >= 1)
    std::vector<SpQkNorm> qd(n);
    size_t words = 0;
    for (int i = 0; i < n; ++i)
      if (qkns[i].q_norm_weight != nullptr) words += (size_t)M * (table[i].N / 16);
    if (words > 0) e = cudaMalloc(&pr->d_qkn_part, words * sizeof(unsigned long long));
    if (e == cudaSuccess && words > 0) e = cudaMemset(pr->d_qkn_part, 0, words * sizeof(unsigned long long));
    size_t off = 0;
    for (int i = 0; i < n; ++i) {
      std::memset(&qd[i], 0, sizeof(SpQkNorm));
      if (qkns[i].q_norm_weight == nullptr) continue;
      qd[i].q = qkns[i];
      qd[i].part = pr->d_qkn_part + off;
      qd[i].inv_d = 1.f / static_cast<float>(qkns[i].rope.head_dim);
      off += (size_t)M * (table[i].N / 16);
    }
    if (e == cudaSuccess) e = cudaMalloc(&pr->d_qkn, (size_t)n * sizeof(SpQkNorm));
    if (e == cudaSuccess) e = cudaMemcpy(pr->d_qkn, qd.data(), (size_t)n * sizeof(SpQkNorm), cudaMemcpyHostToDevice);
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(stream_qknorm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(stream_batch_qknorm_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(stream_batch_qknorm_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(stream_batch_qknorm_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
  }
  if (e == cudaSuccess && (has_rope || has_hf)) {
    std::vector<SpRope> rp(n);
    for (int i = 0; i < n; ++i) rp[i].r = ropes[i];   // (head_dim 0: no rotation)
    e = cudaMalloc(&pr->d_rope, (size_t)n * sizeof(SpRope));
    if (e == cudaSuccess) e = cudaMemcpy(pr->d_rope, rp.data(), (size_t)n * sizeof(SpRope), cudaMemcpyHostToDevice);
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(stream_rope_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(stream_batch_rope_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(stream_batch_rope_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(stream_batch_rope_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
  }
  if (e == cudaSuccess) e = cudaMemcpy(pr->d_sp_ops, ops.data(), (size_t)n * sizeof(SpOp), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(pr->d_cta, cta.data(), cta.size() * sizeof(uint32_t), cudaMemcpyHostToDevice);
  if (e == cudaSuccess && has_hf)
    e = cudaFuncSetAttribute(stream_qwen3moe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(stream_program_kernel<8, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(stream_program_kernel<12, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&pr->l2_bytes, cudaDevAttrL2CacheSize, pr->device);
  if (e == cudaSuccess && M > 1) {
    e = cudaFuncSetAttribute(stream_batch_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(stream_batch_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(stream_batch_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
  }
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    cudaFree(pr->d_stream);
    cudaFree(pr->d_sp_ops);
    cudaFree(pr->d_cta);
    cudaFree(pr->d_rows);
    cudaFree(pr->d_state);
    cudaFree(pr->d_moe);
    cudaFree(pr->d_xlog);
    cudaFree(pr->d_dsk);
    cudaFree(pr->d_res);
    cudaFree(pr->d_rope);
    cudaFree(pr->d_qkn);
    cudaFree(pr->d_qkn_part);
    pr->d_res = nullptr;
    pr->d_rope = nullptr;
    pr->d_qkn = nullptr;
    pr->d_qkn_part = nullptr;
    pr->d_stream = nullptr;
    pr->d_sp_ops = nullptr;
    pr->d_cta = nullptr;
    pr->d_rows = nullptr;
    pr->d_state = nullptr;
    pr->d_moe = nullptr;
    pr->d_xlog = nullptr;
    pr->d_dsk = nullptr;
    pr->n_moe = 0;
    *err = e;
    return false;
  }
  pr->stream_bytes = wbytes;
  pr->qwen3 = has_hf;
  pr->xs_bytes = (size_t)max_K * (M == 1 ? 1 : sb_mt(M)) * 2;   // M = 1: one row (stream_program_kernel)
  return true;
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
  // A SPARSE_MOE or QWEN3_MOE op folds as two linears: gate|up (x [H] -> the recorded gate_up [top_k, 2I], N = top_k 2I) and down
  // (the recorded activations [top_k, I] -> y [H], K = top_k I); the hazard rules below then see every buffer they touch.
  // Only the stream kernel runs them (M = 1; stream_build checks the envelope); otherwise the caller replays per op.
  std::vector<b200awq_op_t> xops;
  std::vector<MoeFold> xfold;
  std::vector<b200awq_moe_t> moes;
  std::vector<int> moe_hf;       // per block: 1 for QWEN3_MOE (the same folding, Qwen3-MoE's routing and finishes),
                                 // 2 for DEEPSEEK_MOE (plus the shared expert: gate|up N and down K grow by it)
  std::vector<b200awq_deepseek_moe_t> dsks;   // per block: DEEPSEEK_MOE's descriptor (zero for the other kinds)
  for (int i = 0; i < n_in; ++i) {
    const b200awq_op_t& op = ops_in[i];
    if (op.kind != B200AWQ_OP_SPARSE_MOE && op.kind != B200AWQ_OP_QWEN3_MOE && op.kind != B200AWQ_OP_DEEPSEEK_MOE) {
      xops.push_back(op);
      xfold.push_back(MoeFold{});
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
    moes.push_back(*m);
    moe_hf.push_back(ds ? 2 : (op.kind == B200AWQ_OP_QWEN3_MOE ? 1 : 0));
    dsks.emplace_back();
    if (ds) dsks.back() = *dd;
    else std::memset(&dsks.back(), 0, sizeof(b200awq_deepseek_moe_t));
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
    xfold.push_back(MoeFold{1, mi});
    xops.push_back(b);
    xfold.push_back(MoeFold{2, mi});
  }
  const b200awq_op_t* ops = xops.data();
  const int n = static_cast<int>(xops.size());
  std::vector<MoeFold> fold;     // per table entry
  std::vector<ProgOp> table;
  struct Glue {
    int kind;
    const void* src;
    const void* w;
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
  std::vector<int> stage_row;    // per table entry: the op whose WHOLE published row its staging waits for, or -1
  int M = -1;
  std::vector<ResFold> res;     // per table entry: the ADD folded into it, if any
  std::vector<std::pair<const void*, size_t>> ext_res;   // external residuals: no op of the program may write them
  std::vector<b200awq_rope_t> ropes;   // per table entry: the ROPE_KV folded into it (head_dim == 0: none)
  std::vector<int> rope_ops;           // table entries that carry one
  std::vector<b200awq_qk_norm_rope_t> qkns;   // per table entry: a QK_NORM_ROPE_KV's descriptor (q_norm_weight == null:
                                              // none, or a plain ROPE_KV)
  for (int i = 0; i < n; ++i) {
    const b200awq_op_t& op = ops[i];
    if (M < 0) M = op.M;
    if (op.M != M) return B200AWQ_EUNSUPPORTED;
    auto rows_bytes = [&](int width) { return (size_t)(M > 0 ? M : 1) * width * 2; };   // M contiguous fp16 rows
    // a read of a linear's raw output after an ADD was folded into it: its row carries the sum, not y
    auto reads_raw_y = [&](const void* p, size_t bytes) {
      for (size_t j = 0; j < table.size(); ++j)
        if (res[j].raw_y != nullptr && overlaps(res[j].raw_y, rows_bytes(table[j].N), p, bytes)) return true;
      return false;
    };
    if (op.kind == B200AWQ_OP_ROPE_KV || op.kind == B200AWQ_OP_QK_NORM_ROPE_KV) {
      // RoPE + cache append, folded into the finish of the linear recorded just before it (whose whole output is qkv);
      // QK_NORM_ROPE_KV: the same op on its embedded descriptor, with q / k normalised first
      const bool qkn = op.kind == B200AWQ_OP_QK_NORM_ROPE_KV;
      const b200awq_qk_norm_rope_t* qd = qkn ? static_cast<const b200awq_qk_norm_rope_t*>(op.weight) : nullptr;
      const b200awq_rope_t* r = qkn ? (qd != nullptr ? &qd->rope : nullptr) : static_cast<const b200awq_rope_t*>(op.weight);
      if (op.x == nullptr) return B200AWQ_EINVAL;
      const int v = rope_validate(r, M > 1 ? op.ldx : INT64_MAX);   // (one row: no pitch; N is checked below)
      if (v != B200AWQ_OK) return v;
      if (qkn && (qd->q_norm_weight == nullptr || qd->k_norm_weight == nullptr)) return B200AWQ_EINVAL;
      if (qkn && (!aligned16(qd->q_norm_weight) || !aligned16(qd->k_norm_weight))) return B200AWQ_EUNSUPPORTED;
      const int D = r->head_dim;
      if (op.N != (r->n_heads + 2 * r->n_kv_heads) * D || (D % 16) != 0) return B200AWQ_EUNSUPPORTED;
      // (an ADD or a glue op in between: the op before is not a linear; a SPARSE_MOE's entries are not plain linears)
      if (i == 0 || ops[i - 1].kind != B200AWQ_OP_LINEAR_GEMM || table.empty() || fold.back().kind != 0)
        return B200AWQ_EUNSUPPORTED;
      const ProgOp& pv = table.back();
      if (op.x != pv.y || op.N != pv.N || (M > 1 && op.ldx != op.N)) return B200AWQ_EUNSUPPORTED;
      ropes.back() = *r;
      if (qkn) qkns.back() = *qd;
      rope_ops.push_back(static_cast<int>(table.size()) - 1);
      continue;
    }
    if (op.kind == B200AWQ_OP_ADD) {
      // y = x + weight, folded into the epilogue of the op recorded just before it (a linear / a MoE block's down)
      if (op.x == nullptr || op.weight == nullptr || op.y == nullptr || op.K <= 0) return B200AWQ_EINVAL;
      if ((op.K % 8) != 0 || !aligned16(op.x) || !aligned16(op.weight) || !aligned16(op.y)) return B200AWQ_EUNSUPPORTED;
      const size_t bytes = rows_bytes(op.K);
      if (overlaps(op.y, bytes, op.x, bytes) || overlaps(op.y, bytes, op.weight, bytes)) return B200AWQ_EUNSUPPORTED;
      if (i == 0 || ops[i - 1].kind != B200AWQ_OP_LINEAR_GEMM || table.empty()) return B200AWQ_EUNSUPPORTED;
      ProgOp& pv = table.back();
      const void* r;                 // the residual: the operand that is not the producer's whole output
      if (op.x == pv.y) r = op.weight;
      else if (op.weight == pv.y) r = op.x;
      else return B200AWQ_EUNSUPPORTED;  // neither operand is the producer's output (both external)
      if (op.K != pv.N || overlaps(r, bytes, pv.y, bytes)) return B200AWQ_EUNSUPPORTED;
      ResFold rf;
      rf.raw_y = pv.y;
      // in-program residual: the newest op that wrote any of it must have published exactly it, kSpResWindow ops back
      for (int j = static_cast<int>(table.size()) - 2; j >= 0 && rf.op < 0; --j) {
        const bool hit = overlaps(table[j].y, rows_bytes(table[j].N), r, bytes) ||
                         (res[j].raw_y != nullptr && overlaps(res[j].raw_y, rows_bytes(table[j].N), r, bytes));
        if (!hit) continue;
        if (r != table[j].y || table[j].N != op.K) return B200AWQ_EUNSUPPORTED;
        if (static_cast<int>(table.size()) - 1 - j > res_window) return B200AWQ_EUNSUPPORTED;
        rf.op = j;
      }
      for (const Glue& gl : glues)   // a glue output is written by CTA slices, never published as a row
        if (overlaps(gl.out, rows_bytes(gl.width), r, bytes)) return B200AWQ_EUNSUPPORTED;
      if (rf.op < 0) {
        rf.ext = r;
        ext_res.emplace_back(r, bytes);
      }
      // the output must not overlap what the producer reads (other CTAs may still be staging it) or publishes
      const size_t pv_src = ((size_t)(M - 1) * pv.src_ld + (size_t)(pv.prologue == kProSilu ? 2 : 1) * pv.K) * 2;
      if (overlaps(op.y, bytes, pv.src, pv_src) || (pv.xout != nullptr && overlaps(op.y, bytes, pv.xout, rows_bytes(pv.K))))
        return B200AWQ_EUNSUPPORTED;
      for (Glue& gl : glues)         // writing the output over something a live glue record still needs ends that record
        if (gl.live && (overlaps(gl.out, rows_bytes(gl.width), op.y, bytes) ||
                        overlaps(gl.src, rows_bytes((gl.kind == kProSilu ? 2 : 1) * gl.width), op.y, bytes))) {
          if (!gl.used) return B200AWQ_EUNSUPPORTED;
          gl.live = false;
        }
      pv.y = static_cast<__half*>(op.y);   // the producer's row now publishes the sum
      res.back() = rf;
      continue;
    }
    if (op.kind == B200AWQ_OP_RMSNORM || op.kind == B200AWQ_OP_SILU_AND_MUL) {
      if (op.x == nullptr || op.y == nullptr || op.K <= 0) return B200AWQ_EINVAL;
      if (op.kind == B200AWQ_OP_RMSNORM && op.weight == nullptr) return B200AWQ_EINVAL;
      if ((op.K % 8) != 0 || !aligned16(op.x) || !aligned16(op.y) || (op.weight != nullptr && !aligned16(op.weight)))
        return B200AWQ_EUNSUPPORTED;
      const size_t in_bytes = (size_t)M * (op.kind == B200AWQ_OP_SILU_AND_MUL ? 2 : 1) * op.K * 2;
      if (overlaps(op.y, rows_bytes(op.K), op.x, in_bytes)) return B200AWQ_EUNSUPPORTED;  // in-place glue op
      for (Glue& gl : glues)
        if (gl.live && (overlaps(gl.out, rows_bytes(gl.width), op.y, rows_bytes(op.K)) ||
                        overlaps(gl.src, rows_bytes((gl.kind == kProSilu ? 2 : 1) * gl.width), op.y, rows_bytes(op.K)))) {
          if (!gl.used) return B200AWQ_EUNSUPPORTED;
          gl.live = false;
        }
      if (reads_raw_y(op.x, in_bytes)) return B200AWQ_EUNSUPPORTED;
      // its input must not be a buffer only CTA 0 publishes
      for (const Glue& gl : glues)
        if (overlaps(gl.out, rows_bytes(gl.width), op.x, in_bytes)) return B200AWQ_EUNSUPPORTED;
      glues.push_back(Glue{op.kind == B200AWQ_OP_RMSNORM ? kProRmsnorm : kProSilu, op.x, op.weight, op.y, op.K, op.eps,
                           false, true});
      continue;
    }
    if (op.kind != B200AWQ_OP_LINEAR_GEMM) return B200AWQ_EINVAL;
    if (op.x == nullptr || op.qweight == nullptr || op.scales == nullptr || op.qzeros == nullptr || op.y == nullptr ||
        op.K <= 0 || op.N <= 0 || op.group_size <= 0 || (op.K % op.group_size) != 0)
      return B200AWQ_EINVAL;
    if (M < 1 || M > max_tokens) return B200AWQ_EUNSUPPORTED;
    if (M > 1 && op.ldx < op.K) return B200AWQ_EINVAL;
    ProgOp p;
    std::memset(&p, 0, sizeof(p));
    p.ext_dep = -1;
    p.qw_src = static_cast<const int32_t*>(op.qweight);
    p.scales = static_cast<const __half*>(op.scales);
    p.qzeros = static_cast<const int32_t*>(op.qzeros);
    p.bias = static_cast<const __half*>(op.bias);
    p.y = static_cast<__half*>(op.y);
    p.K = op.K;
    p.N = op.N;
    p.G = op.group_size;
    Glue* hit = nullptr;
    for (Glue& gl : glues)
      if (gl.live && gl.out == op.x && gl.width == op.K) hit = &gl;
    if (hit != nullptr) {
      p.prologue = hit->kind;
      p.src = static_cast<const __half*>(hit->src);
      p.norm_w = static_cast<const __half*>(hit->w);
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
        if (overlaps(gl.out, rows_bytes(gl.width), op.x, ((size_t)(M - 1) * p.src_ld + op.K) * 2)) return B200AWQ_EUNSUPPORTED;
    }
    // the source's M rows (row pitch src_ld), this op's output (M rows of N)
    const size_t src_bytes = ((size_t)(M - 1) * p.src_ld + (size_t)(p.prologue == kProSilu ? 2 : 1) * op.K) * 2;
    const size_t y_bytes = rows_bytes(op.N);
    if (overlaps(p.y, y_bytes, p.src, src_bytes) || reads_raw_y(p.src, src_bytes)) return B200AWQ_EUNSUPPORTED;
    if (p.xout != nullptr && overlaps(p.xout, rows_bytes(op.K), p.y, y_bytes)) return B200AWQ_EUNSUPPORTED;
    if (!table.empty()) {
      // the previous op's fp16 output reaches memory only while THIS op stages its activations: a source inside it
      // is taken from the previous op's fp32 accumulators instead (same values), anything else touching it is a race
      const ProgOp& pv = table.back();
      const uintptr_t y0 = reinterpret_cast<uintptr_t>(pv.y), s0 = reinterpret_cast<uintptr_t>(p.src);
      if (s0 >= y0 && s0 + src_bytes <= y0 + rows_bytes(pv.N)) {
        if (((s0 - y0) & 15) != 0) return B200AWQ_EUNSUPPORTED;
        p.src_prev = 1;
        p.src_off = static_cast<int>((s0 - y0) / 2);
      } else if (overlaps(pv.y, rows_bytes(pv.N), p.src, src_bytes)) {
        return B200AWQ_EUNSUPPORTED;
      } else {
        // a source written by an older op of this program: wait for that op's duty-warp stores
        for (int j = static_cast<int>(table.size()) - 2; j >= 0; --j)
          if (overlaps(table[j].y, rows_bytes(table[j].N), p.src, src_bytes)) {
            p.ext_dep = j;
            break;
          }
      }
      if (p.xout != nullptr && overlaps(p.xout, rows_bytes(op.K), pv.y, rows_bytes(pv.N))) return B200AWQ_EUNSUPPORTED;
    }
    // writing y over something a live glue record still needs ends that record
    for (Glue& gl : glues)
      if (gl.live && &gl != hit &&
          (overlaps(gl.out, rows_bytes(gl.width), p.y, y_bytes) ||
           overlaps(gl.src, rows_bytes((gl.kind == kProSilu ? 2 : 1) * gl.width), p.y, y_bytes))) {
        if (!gl.used) return B200AWQ_EUNSUPPORTED;
        gl.live = false;
      }
    {
      // a staging wait on the whole row of op s waits for every CTA that owns columns of s
      const int s = p.src_prev ? static_cast<int>(table.size()) - 1 : p.ext_dep;
      const size_t width = (size_t)(p.prologue == kProSilu ? 2 : 1) * op.K;
      stage_row.push_back(s >= 0 && p.src == table[s].y && width == (size_t)table[s].N ? s : -1);
    }
    table.push_back(p);
    fold.push_back(xfold[i]);
    res.emplace_back();
    ropes.emplace_back();
    std::memset(&ropes.back(), 0, sizeof(b200awq_rope_t));
    qkns.emplace_back();
    std::memset(&qkns.back(), 0, sizeof(b200awq_qk_norm_rope_t));
  }
  for (const Glue& gl : glues)
    if (!gl.used) return B200AWQ_EUNSUPPORTED;   // a glue op nobody consumes would never run
  if (table.empty()) return B200AWQ_EUNSUPPORTED;
  const int nt = static_cast<int>(table.size());
  for (const auto& er : ext_res) {
    // an external residual is read at the finish of its op, any time during the run: nothing of the program may write it
    for (int j = 0; j < nt; ++j)
      if (overlaps(table[j].y, (size_t)M * table[j].N * 2, er.first, er.second) ||
          (res[j].raw_y != nullptr && overlaps(res[j].raw_y, (size_t)M * table[j].N * 2, er.first, er.second)))
        return B200AWQ_EUNSUPPORTED;
    for (const Glue& gl : glues)
      if (overlaps(gl.out, (size_t)M * gl.width * 2, er.first, er.second)) return B200AWQ_EUNSUPPORTED;
    for (const b200awq_moe_t& m : moes)
      if (overlaps(m.gate_up, (size_t)m.top_k * 2 * m.I * 2, er.first, er.second) ||
          overlaps(m.act, (size_t)m.top_k * m.I * 2, er.first, er.second) ||
          overlaps(m.down, (size_t)m.top_k * m.H * 2, er.first, er.second) ||
          overlaps(m.logits, (size_t)m.E * 2, er.first, er.second) ||
          overlaps(m.topk_weights, (size_t)m.top_k * M * 4, er.first, er.second) ||
          overlaps(m.topk_ids, (size_t)m.top_k * M * 4, er.first, er.second) ||
          overlaps(m.token_expert_indices, (size_t)m.top_k * M * 4, er.first, er.second) ||
          overlaps(m.sorted_ids, (size_t)m.sorted_len * 4, er.first, er.second) ||
          overlaps(m.expert_ids, (size_t)(m.top_k * M + m.E) * 4, er.first, er.second) ||
          overlaps(m.num_tokens_post_pad, 4, er.first, er.second))
        return B200AWQ_EUNSUPPORTED;
    for (const b200awq_deepseek_moe_t& d : dsks)   // (zero for other blocks: overlaps nothing)
      if (overlaps(d.moe.gate_up, (size_t)(d.moe.top_k * 2 * d.moe.I + 2 * d.I_s) * 2, er.first, er.second) ||
          overlaps(d.moe.act, (size_t)(d.moe.top_k * d.moe.I + d.I_s) * 2, er.first, er.second) ||
          overlaps(d.moe.logits, (size_t)d.moe.E * 4, er.first, er.second) ||
          overlaps(d.shared_out, (size_t)d.moe.H * 2, er.first, er.second))
        return B200AWQ_EUNSUPPORTED;
  }
  // ROPE_KV: the rotated q and the appended cache rows are written in a finish, while other CTAs run later ops.  No
  // other op of the program may read or write them, nor write the position / frequency table the finish reads; the
  // producer must not be a gate|up whose product a SiLU*mul reads (its row would hold silu(gate) * up).
  // QK_NORM_ROPE_KV: its two norm weights are reads like the position and the frequency table.
  for (int ri : rope_ops) {
    const b200awq_rope_t& r = ropes[ri];
    const size_t cache = ((size_t)(M - 1) * r.cache_batch_stride + (size_t)r.cache_len * r.n_kv_heads * r.head_dim) * 2;
    const std::pair<const void*, size_t> outs[3] = {{r.q_out, (size_t)M * r.n_heads * r.head_dim * 2},
                                                    {r.k_cache, cache}, {r.v_cache, cache}};
    const size_t wn = qkns[ri].q_norm_weight != nullptr ? (size_t)r.head_dim * 2 : 0;   // (null, 0: overlaps nothing)
    const std::pair<const void*, size_t> ins[4] = {{r.pos, 4}, {r.freqs, (size_t)r.freqs_len * r.head_dim * 4},
                                                   {qkns[ri].q_norm_weight, wn}, {qkns[ri].k_norm_weight, wn}};
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
      const size_t src_bytes = ((size_t)(M - 1) * table[j].src_ld + (size_t)(table[j].prologue == kProSilu ? 2 : 1) * table[j].K) * 2;
      if (hits_any(table[j].y, (size_t)M * table[j].N * 2) ||
          (res[j].raw_y != nullptr && hits_any(res[j].raw_y, (size_t)M * table[j].N * 2)) ||
          (table[j].src != nullptr && hits_out(table[j].src, src_bytes)) ||
          (res[j].ext != nullptr && hits_out(res[j].ext, (size_t)M * table[j].N * 2)))
        return B200AWQ_EUNSUPPORTED;
      if (table[j].prologue == kProSilu && overlaps(table[j].src, src_bytes, table[ri].y, (size_t)M * table[ri].N * 2))
        return B200AWQ_EUNSUPPORTED;   // a SiLU*mul of the qkv output: the producer would be a mode-1 gate|up
      if (j != ri && ropes[j].head_dim != 0) {   // another ROPE_KV: its outputs are writes, its inputs reads
        const b200awq_rope_t& o = ropes[j];
        const size_t oc = ((size_t)(M - 1) * o.cache_batch_stride + (size_t)o.cache_len * o.n_kv_heads * o.head_dim) * 2;
        if (hits_any(o.q_out, (size_t)M * o.n_heads * o.head_dim * 2) || hits_any(o.k_cache, oc) || hits_any(o.v_cache, oc))
          return B200AWQ_EUNSUPPORTED;
      }
    }
    for (const Glue& gl : glues)
      if (hits_any(gl.out, (size_t)M * gl.width * 2) || hits_out(gl.src, (size_t)M * (gl.kind == kProSilu ? 2 : 1) * gl.width * 2))
        return B200AWQ_EUNSUPPORTED;
    for (const b200awq_moe_t& m : moes)
      if (hits_any(m.gate_up, (size_t)m.top_k * 2 * m.I * 2) || hits_any(m.act, (size_t)m.top_k * m.I * 2) ||
          hits_any(m.down, (size_t)m.top_k * m.H * 2) || hits_any(m.logits, (size_t)m.E * 2) ||
          hits_any(m.topk_weights, (size_t)m.top_k * M * 4) || hits_any(m.topk_ids, (size_t)m.top_k * M * 4) ||
          hits_any(m.token_expert_indices, (size_t)m.top_k * M * 4) || hits_any(m.sorted_ids, (size_t)m.sorted_len * 4) ||
          hits_any(m.expert_ids, (size_t)(m.top_k * M + m.E) * 4) || hits_any(m.num_tokens_post_pad, 4) ||
          hits_out(m.gate_weight, (size_t)m.E * m.H * 2))
        return B200AWQ_EUNSUPPORTED;
    for (const b200awq_deepseek_moe_t& d : dsks)
      if (hits_any(d.moe.gate_up, (size_t)(d.moe.top_k * 2 * d.moe.I + 2 * d.I_s) * 2) ||
          hits_any(d.moe.act, (size_t)(d.moe.top_k * d.moe.I + d.I_s) * 2) || hits_any(d.moe.logits, (size_t)d.moe.E * 4) ||
          hits_any(d.shared_out, (size_t)d.moe.H * 2) || hits_out(d.bias, d.bias != nullptr ? (size_t)d.moe.E * 4 : 0))
        return B200AWQ_EUNSUPPORTED;
  }
  for (int i = 0; i < nt; ++i) {
    // An in-program residual (row j % 4) is read in op i's finish, by the CTA that published those columns in op j (same
    // width, same partition).  Ops j + 4, j + 8, ... publish into that row again.  Op i itself (i = j + 4) only rewrites
    // the words each thread has just read; the next one after i, op k, may overwrite them only once every CTA has
    // finished op i: some op in (i, k] must stage the WHOLE row of an op >= i that every CTA owns columns of (a wait on a
    // slice of a row, or on a narrow op, waits for a few CTAs only).  tests/test_stream_residual_model.py replays random
    // programs through this rule (b200awq_program_plan).
    const int j = res[i].op;
    if (j < 0) continue;
    int k = j + kSpRows;
    while (k <= i) k += kSpRows;
    if (k >= nt) continue;
    int reach = -1;
    for (int m = i + 1; m <= k; ++m) {
      const int s = stage_row[m];
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
  if (e == cudaSuccess && stream_build(pr, table, grid, M, &e, fold, moes, res, ropes, qkns, moe_hf, dsks)) {
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
  if (p->M > 1) {
    // batched stream variant: 8 consumer warps, the ring depth chosen at creation, MT = the smallest of 2 / 4 / 8 >= M
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(prog_sm_count());
    cfg.blockDim = dim3(32 + kSbWarps * 32);
    cfg.dynamicSmemBytes = sb_fixed_smem(p->sb_spw, p->sb_lmax, sb_mt(p->M), p->sb_nu_max) + p->xs_bytes;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeCooperative;   // all CTAs co-resident: the hand-off polls are grid-wide waits
    attr[0].val.cooperative = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    const SpOp* sops = p->d_sp_ops;
    const uint32_t* cta = p->d_cta;
    if (p->d_qkn != nullptr) {   // a QK_NORM_ROPE_KV op: the rope kernel plus the two-phase q / k norm
      auto nk = sb_mt(p->M) == 2 ? stream_batch_qknorm_kernel<2>
                                 : (sb_mt(p->M) == 4 ? stream_batch_qknorm_kernel<4> : stream_batch_qknorm_kernel<8>);
      const SpRes* rd = p->d_res;
      const SpRope* qd = p->d_rope;
      const SpQkNorm* nd = p->d_qkn;
      return cudaLaunchKernelEx(&cfg, nk, sops, cta, p->n_ops, p->d_rows, p->row_stride, p->d_state, p->M, p->sb_spw,
                                p->sb_lmax, p->sb_nu_max, knob(3), rd, qd, nd);
    }
    if (p->d_rope != nullptr) {  // a ROPE_KV op: the residual kernel plus the rope steps of a mode-2 finish
      auto qk = sb_mt(p->M) == 2 ? stream_batch_rope_kernel<2>
                                 : (sb_mt(p->M) == 4 ? stream_batch_rope_kernel<4> : stream_batch_rope_kernel<8>);
      const SpRes* rd = p->d_res;
      const SpRope* qd = p->d_rope;
      return cudaLaunchKernelEx(&cfg, qk, sops, cta, p->n_ops, p->d_rows, p->row_stride, p->d_state, p->M, p->sb_spw,
                                p->sb_lmax, p->sb_nu_max, knob(3), rd, qd);
    }
    if (p->d_res != nullptr) {   // residual adds: the same kernel with the residual steps in its finish
      auto rk = sb_mt(p->M) == 2 ? stream_batch_residual_kernel<2>
                                 : (sb_mt(p->M) == 4 ? stream_batch_residual_kernel<4> : stream_batch_residual_kernel<8>);
      const SpRes* rd = p->d_res;
      return cudaLaunchKernelEx(&cfg, rk, sops, cta, p->n_ops, p->d_rows, p->row_stride, p->d_state, p->M, p->sb_spw,
                                p->sb_lmax, p->sb_nu_max, knob(3), rd);
    }
    auto kern = sb_mt(p->M) == 2 ? stream_batch_kernel<2> : (sb_mt(p->M) == 4 ? stream_batch_kernel<4> : stream_batch_kernel<8>);
    return cudaLaunchKernelEx(&cfg, kern, sops, cta, p->n_ops, p->d_rows, p->row_stride, p->d_state, p->M, p->sb_spw,
                              p->sb_lmax, p->sb_nu_max, knob(3));
  }
  // knob 9: consumer warps of the stream kernel: 8 (4 units in flight; the default) or 12 (2 units), each with the ring
  // depth chosen at creation (at least 4 / 3 stages).  No 16-warp variant: 17 warps put 5 on one of the SM's four
  // register-file partitions, which caps a thread at 96 registers on sm_90 and spills the unit loop.  The MoE, residual
  // and rope kernels always run 8 warps.
  const bool moe_k = p->d_rope != nullptr || p->d_res != nullptr || p->n_moe > 0;
  const int nw = knob(9) == 12 && !moe_k ? 12 : 8;
  const int spw = nw == 8 ? p->sp_spw8 : p->sp_spw12;
  const int grid = prog_sm_count();
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(32 + nw * 32);
  cfg.dynamicSmemBytes = sp_fixed_smem(nw, spw, moe_k) + p->xs_bytes;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;   // all CTAs co-resident: the hand-off polls are grid-wide waits
  attr[0].val.cooperative = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  const SpOp* sops = p->d_sp_ops;
  const uint32_t* cta = p->d_cta;
  // knob 8: the HBM -> L2 run-ahead window of the weight stream, grid-wide, in MB, at most the device's L2 (<= 0: off,
  // the default).  The producer advances its prefetch cursor only while it has no ring stage to fill - during op
  // hand-offs and tails - and each of its grid x nw lanes keeps at most window / (grid x nw) bytes ahead of its ring.
  // Off is the default: on the bench step no window beat it by more than its run-to-run spread (H100 SXM, DESIGN
  // 3.5b: 8 and 16 MB within 0.5 %, 32 MB 4 % slower).
  const size_t window = knob(8) <= 0 ? 0 : std::min((size_t)knob(8) << 20, (size_t)p->l2_bytes);
  const int l2_ahead = (int)(window / ((size_t)grid * nw));
  // knob 10: ops ahead of the consumers' staging for which shared-memory loads may already be issued (0 = ungated,
  // the default: a gate of 2 measured 1.5-2 % slower on the bench step, DESIGN 3.5b; n > 0: at most n - 1 ops ahead,
  // 1 = strictly gated)
  const int gate_ahead = knob(10) <= 0 ? 1 << 20 : knob(10) - 1;
  const SpMoe* no_moe = nullptr;
  if (p->d_dsk != nullptr) {    // programs with DEEPSEEK_MOE blocks (every side table allocated)
    const SpMoe* md = p->d_moe;
    const SpRes* rd = p->d_res;
    const SpRope* qd = p->d_rope;
    const SpQkNorm* nd = p->d_qkn;
    const SpDsk* dd = p->d_dsk;
    return cudaLaunchKernelEx(&cfg, stream_deepseek_moe_kernel, sops, cta, p->n_ops, p->d_rows, p->row_stride,
                              p->d_state, spw, knob(3), l2_ahead, gate_ahead, md, rd, qd, nd, dd);
  }
  if (p->qwen3) {    // programs with QWEN3_MOE blocks (every side table allocated)
    const SpMoe* md = p->d_moe;
    const SpRes* rd = p->d_res;
    const SpRope* qd = p->d_rope;
    const SpQkNorm* nd = p->d_qkn;
    return cudaLaunchKernelEx(&cfg, stream_qwen3moe_kernel, sops, cta, p->n_ops, p->d_rows, p->row_stride, p->d_state,
                              spw, knob(3), l2_ahead, gate_ahead, md, rd, qd, nd);
  }
  if (p->d_qkn != nullptr) {    // programs with a QK_NORM_ROPE_KV op (with or without other ROPE_KV ops, adds, MoE blocks)
    const SpMoe* md = p->d_moe;
    const SpRes* rd = p->d_res;
    const SpRope* qd = p->d_rope;
    const SpQkNorm* nd = p->d_qkn;
    return cudaLaunchKernelEx(&cfg, stream_qknorm_kernel, sops, cta, p->n_ops, p->d_rows, p->row_stride, p->d_state, spw,
                              knob(3), l2_ahead, gate_ahead, md, rd, qd, nd);
  }
  if (p->d_rope != nullptr) {   // programs with a ROPE_KV op (with or without adds / sparse-MoE blocks)
    const SpMoe* md = p->d_moe;
    const SpRes* rd = p->d_res;
    const SpRope* qd = p->d_rope;
    return cudaLaunchKernelEx(&cfg, stream_rope_kernel, sops, cta, p->n_ops, p->d_rows, p->row_stride, p->d_state, spw,
                              knob(3), l2_ahead, gate_ahead, md, rd, qd);
  }
  if (p->d_res != nullptr) {   // programs with residual adds (with or without sparse-MoE blocks)
    const SpMoe* md = p->d_moe;
    const SpRes* rd = p->d_res;
    return cudaLaunchKernelEx(&cfg, stream_residual_kernel, sops, cta, p->n_ops, p->d_rows, p->row_stride, p->d_state,
                              spw, knob(3), l2_ahead, gate_ahead, md, rd);
  }
  if (p->n_moe > 0) {   // programs with sparse-MoE blocks: the MOE instantiation
    const SpMoe* md = p->d_moe;
    return cudaLaunchKernelEx(&cfg, stream_moe_kernel, sops, cta, p->n_ops, p->d_rows, p->row_stride, p->d_state, spw,
                              knob(3), l2_ahead, gate_ahead, md);
  }
  if (nw == 8)
    return cudaLaunchKernelEx(&cfg, stream_program_kernel<8, 4>, sops, cta, p->n_ops, p->d_rows, p->row_stride,
                              p->d_state, spw, knob(3), l2_ahead, gate_ahead, no_moe);
  return cudaLaunchKernelEx(&cfg, stream_program_kernel<12, 2>, sops, cta, p->n_ops, p->d_rows, p->row_stride,
                            p->d_state, spw, knob(3), l2_ahead, gate_ahead, no_moe);
}

void program_destroy(Program* p) {
  if (p == nullptr) return;
  cudaFree(p->d_sp_ops);
  cudaFree(p->d_stream);
  cudaFree(p->d_cta);
  cudaFree(p->d_rows);
  cudaFree(p->d_state);
  cudaFree(p->d_moe);
  cudaFree(p->d_xlog);
  cudaFree(p->d_dsk);
  cudaFree(p->d_res);
  cudaFree(p->d_rope);
  cudaFree(p->d_qkn);
  cudaFree(p->d_qkn_part);
  delete p;
}

}  // namespace b200awq
