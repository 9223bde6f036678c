// Internal launcher interface between the C-ABI layer (cabi.cu) and the kernel translation units.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

struct b200awq_op;
struct b200awq_rope;
struct b200awq_qk_norm_rope;
struct b200awq_mla;

namespace b200awq {

struct GemmArgs {
  const void* x;        // [M, ldx] fp16
  int64_t ldx;
  const int32_t* qweight;
  const void* scales;
  const int32_t* qzeros;
  const void* bias;     // [N] fp16 or nullptr
  void* y;              // [M, N] fp16
  int M, K, N, G;
};

struct FastArgs {
  const void* x;
  int64_t ldx;
  const int16_t* qweight;  // [N/4, K]
  const void* scales;      // [8 zw, N]
  const void* szeros;      // [8 zw, N] = -z*s
  const void* bias;
  void* y;
  int M, K, N, G;
};

// workspace carve-up (see b200awq_workspace_bytes): tickets first, fp32 accumulators after
constexpr size_t kTicketBytes = 16384;  // 4096 int tickets
constexpr int kMaxSplitM = 128;         // rows of 8-byte scratch kept for split-K (= 256 rows of fp32 partial sums)

// knobs (cabi.cu)
int knob(int key);

// Kernel launch with the optional PDL attribute (knob 4).
template <typename... KArgs, typename... Args>
inline cudaError_t launch_kernel(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                 Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  if (knob(4) != 0) {
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
  }
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

cudaError_t dequantize_gemm(const int32_t* qweight, const void* scales, const int32_t* qzeros, void* out, int K,
                            int N, int G, cudaStream_t st);

// 2-D tiled tensor map over a row-major matrix (cached by address + shape; weights are static, activations
// recycle a few buffers).  elem_kind: 0 = fp16, 1 = int32.  128B swizzle, zero fill out of bounds.
cudaError_t make_tmap_2d(const void* ptr, int elem_kind, uint64_t inner, uint64_t outer, uint64_t pitch_bytes,
                         uint32_t box_inner, uint32_t box_outer, CUtensorMap* out, bool swizzle128 = true);

bool gemv_gemm_layout_supported(const GemmArgs& a);
bool gemv_v3_supported(const GemmArgs& a);
cudaError_t gemv_v3(const GemmArgs& a, float* acc_ws, int* tickets, cudaStream_t st);
cudaError_t gemv_v3_debug_read(void* dst, size_t bytes);
cudaError_t gemv_gemm_layout(const GemmArgs& a, float* acc_ws, int* tickets, cudaStream_t st);
cudaError_t gemv_gemv_layout(const GemmArgs& a, cudaStream_t st);
cudaError_t gemv_fast_layout(const FastArgs& a, cudaStream_t st);

// tensor-core path; layout: 0 = GEMM, 1 = GEMV, 2 = FAST (qweight/qzeros reinterpretations documented in gemm_tc.cu)
cudaError_t gemm_tc(const GemmArgs& a, int layout, float* acc_ws, int* tickets, cudaStream_t st);
// true when gemm_tc(layout 0) would run the small-M kernel (TMA-staged packed weights) for these arguments
bool gemm_tcq_applicable(const GemmArgs& a, const float* acc_ws, const int* tickets);
bool gemm_tcq_shape_ok(int M, int K, int N, int G);                       // the kernel's shape envelope
int gemm_tcq_grid(int n_tiles, int KP, int M, int sms, int mode);         // its work cut (host logic, CPU-testable)
cudaError_t gemm_tcq_debug_read(void* dst, size_t bytes);   // phase timestamps of the last small-M launch (knob 3 == 9)

// grouped (MoE) tensor-core kernel (gemm_tc.cu): the prefill-size path of grouped_gemm_forward.  BT = token tile (32 /
// 64 / 128); x_per_slot and the routing tables as moe_grouped_gemm; topk_w == nullptr: no routing-weight multiply.
bool moe_tc_supported(int K, int N, int G, int block_size, int E);        // the kernel's envelope
int moe_tc_token_tile(int n_slots, int E);                                // BT the routing picks
cudaError_t moe_tc_gemm(const void* x, int x_per_slot, const int32_t* qweight, const void* scales, const int32_t* qzeros,
                        const float* topk_w, const int* sorted_ids, const int* expert_ids, const int* num_post_pad,
                        void* y, int n_slots, int topk, int sorted_len, int E, int K, int N, int G, int block_size,
                        int BT, cudaStream_t st);
// its tile list for a HOST copy of expert_ids (host logic, CPU-testable): 4 ints per tile, returns the tile count
int moe_tc_plan(const int32_t* expert_ids, int n_blocks, int block_size, int E, int N, int BT, int32_t* tiles_out,
                int max_tiles);

// decode program (program.cu)
struct Program;
// plan (b200awq_program_plan): fold only, for `grid` SMs and a residual window (<= 0: the library's); no CUDA call
struct ProgramPlan {
  int grid, window, kernel_ops;
};
int program_create(const struct ::b200awq_op* ops, int n, int max_tokens, Program** out, cudaError_t* cuda_err,
                   ProgramPlan* plan = nullptr);
int program_m(const Program* p);
int program_num_ops(const Program* p);
int moe_plan(int E, int topk, int H, int I, int G, int grid, int* out8);   // host only (b200awq_moe_plan)
int qwen3_moe_plan(int E, int topk, int H, int I, int G, int grid, int* out8);   // host only (b200awq_qwen3_moe_plan)
int deepseek_moe_plan(int E, int topk, int H, int I, int I_s, int G, int grid, int* out8);   // (b200awq_deepseek_moe_plan)
cudaError_t program_run(Program* p, cudaStream_t st);
size_t program_stream_bytes(const Program* p);
// stream format (program_stream.cuh; oracle/stream_format.py): one-time re-layout of a GEMM-layout linear
size_t stream_format_bytes(int K, int N, int G);
bool stream_format_supported(int K, int N, int G, int mode);
cudaError_t stream_pack(const int32_t* qweight, const void* scales, const int32_t* qzeros, void* out, int K, int N, int G,
                        int mode, cudaStream_t st);
void program_destroy(Program* p);
cudaError_t program_debug_read(void* dst, size_t bytes);
cudaError_t program_abort_read(void* dst, size_t bytes);
cudaError_t stream_debug_read(void* dst, size_t bytes);
cudaError_t program_set_watchdog_seconds(int seconds);

// grouped persistent GEMV (gemv.cu): the decode-size path of grouped_gemm_forward
bool gemv_v3_moe_supported(int K, int N, int G, int hbs);
cudaError_t gemv_v3_moe(const void* x, int x_per_slot, const int32_t* qweight, const void* scales, const int32_t* qzeros,
                        const float* topk_w, const int* sorted_ids, const int* expert_ids, const int* num_post_pad,
                        void* y, int n_slots, int topk, int hbs, int E, int K, int N, int G, int block_size,
                        float* acc_ws, int* tickets, cudaStream_t st);

// MoE (moe.cu)
cudaError_t topk_softmax(const float* gating, float* topk_w, int* topk_ids, int* src_rows, int M, int E, int topk,
                         cudaStream_t st);
cudaError_t moe_align_block_size(const int* topk_ids, int numel, int num_experts, int block_size, int* sorted_ids,
                                 int* expert_ids, int* num_post_pad, cudaStream_t st);
bool moe_grouped_supported(int K, int N, int G);
cudaError_t moe_grouped_gemm(const void* x, int x_per_slot, const int32_t* qweight, const void* scales,
                             const int32_t* qzeros, const float* topk_w, const int* sorted_ids, const int* expert_ids,
                             const int* num_post_pad, void* y, int n_slots, int topk, int sorted_len, int K, int N, int G,
                             int mul_weights, int block_size, cudaStream_t st);

// one-shot all-reduce over peer memory (comm.cu)
struct Comm;
int comm_create(int rank, int world, int max_elems, Comm** out, cudaError_t* err);
cudaError_t comm_ipc_handle(Comm* c, void* out64);
cudaError_t comm_open(Comm* c, const void* handles);
cudaError_t comm_all_reduce(Comm* c, void* y, int n, cudaStream_t st);
bool comm_ready(const Comm* c);
int comm_max_elems(const Comm* c);
cudaError_t comm_error_flag(Comm* c, int* out);
void comm_destroy(Comm* c);

cudaError_t rmsnorm(const void* x, const void* w, void* out, int rows, int hidden, float eps, cudaStream_t st);
cudaError_t silu_and_mul(const void* gate_up, void* out, int rows, int d, cudaStream_t st);
cudaError_t layer_norm(const void* x, int64_t ldx, const void* w, const void* b, void* out, int rows, int hidden,
                       float eps, cudaStream_t st);
cudaError_t gelu(const void* x, void* out, int64_t n, int approximate, cudaStream_t st);
// B200AWQ_OK, or the code b200awq_rope_kv returns for a bad descriptor / qkv pitch (host only)
int rope_validate(const struct ::b200awq_rope* r, int64_t ldqkv);
// T tokens per sequence (M % T == 0): token row m writes cache entry m / T at position *pos + m % T (T = 1: entry m),
// rotated at that position plus off[m / T] (off: device int32[M / T] rotary offsets; null: none)
cudaError_t rope_kv(const void* qkv, int64_t ldqkv, const struct ::b200awq_rope& r, int M, int T, const int32_t* off,
                    cudaStream_t st);
// B200AWQ_OK, or the code b200awq_qk_norm_rope_kv returns for a bad descriptor / qkv pitch (host only; D % 16 is
// checked by the callers)
int qk_norm_validate(const struct ::b200awq_qk_norm_rope* q, int64_t ldqkv);
cudaError_t qk_norm_rope_kv(const void* qkv, int64_t ldqkv, const struct ::b200awq_qk_norm_rope& q, int M, int T,
                            const int32_t* off, cudaStream_t st);
cudaError_t stream_pack_rotary(const int32_t* qweight, const void* scales, const int32_t* qzeros, void* out, int K, int N,
                               int G, int head_dim, int rotary_dim, cudaStream_t st);
// B200AWQ_OK, or the code the stand-alone op of kind (B200AWQ_OP_MLA_*) returns for a bad descriptor (host only)
int mla_validate(const struct ::b200awq_mla* d, int kind);
cudaError_t mla_rope(const void* row, int64_t ld, const struct ::b200awq_mla& d, int M, cudaStream_t st);
cudaError_t mla_kv(const void* row, int64_t ld, const struct ::b200awq_mla& d, int M, cudaStream_t st);
cudaError_t mla_k_rope(const void* row, int64_t ld, int64_t k_pe_col, const struct ::b200awq_mla& d, int M,
                       cudaStream_t st);
cudaError_t mla_q_rope(const void* row, int64_t ld, const struct ::b200awq_mla& d, int M, cudaStream_t st);

}  // namespace b200awq
