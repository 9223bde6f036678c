// Decode program kernel (program.cu is its host side): a persistent kernel built around a ONE-TIME RE-LAYOUT of the
// packed weights (the "stream format", restated in numpy in oracle/stream_format.py; the reference's precedent for
// a post-load re-layout is awq/modules/linear/exllama.py:66-79) so that the grid-wide hand-off between two
// dependent linears shrinks to "store, poll".
//
// Why: with the checkpoint's GEMM layout [K, N/8] a DRAM-efficient tile is >= 128 bytes = 256 columns wide, so
// N = 4096 has only 16 column blocks for 132 CTAs: split-K with a fan-in of ~8 CTAs per column block is forced, and its
// cost - ~100 k 64-bit REDs per op into L2, every CTA polling 64-bit sums, a reclamation protocol for the accumulator
// rows - is comparable to the op's own weight streaming.  In the stream format ANY partition is contiguous in memory, so the work is
// cut OUTPUT-STATIONARY: a CTA owns whole 16-column sets (all of K), its 8 consumer warps split the CTA's units
// (set, 128 rows of K) evenly, partial sums meet in shared memory, and the CTA publishes FINISHED fp16 outputs:
//   * no cross-CTA reduction, no atomics, no fixed-point packing, nothing to zero or reclaim, no duty warp;
//   * the hand-off word is (fp16 value | 16-bit tag): one plain 32-bit store by the owner, polled by the consumers
//     with ld.relaxed.gpu - a word is valid when its tag equals the tag of (run, op), so buffers never need
//     clearing and a run is bit-reproducible (fixed summation order);
//   * every CTA reads the whole activation row (K x 4 bytes from L2), RMSNorm needs no second grid-wide pass;
//   * SiLU*mul is fused into the PRODUCER: the stream format of a gate|up linear pairs gate column j and up
//     column j in one lane, so the consumer of `down` polls d words instead of 2 d.
// The weight stream itself is as before: a producer warp keeps a shared-memory ring of bulk copies
// (cp.async.bulk, plain 1-D: every warp's byte range is contiguous) full ACROSS op boundaries.
//
// Included by program.cu (one translation unit: shares the watchdog / debug symbols).
#pragma once

namespace b200awq {

constexpr int kSpMaxWarps = 16;                   // consumer warps at most (the kernel is a template over the count)
constexpr int kSpStageWarps = 8;                  // warps that stage the activations (thread -> k mapping of aux.cu's
                                                  // rmsnorm_kernel: 256 threads x 8 consecutive k per pass)
constexpr int kSpStagePass = kSpStageWarps * 32 * 8;   // k covered by one staging pass
constexpr int kSpStageBytes = 4288;               // 4 units of G >= 128 (4 x 1072), 7 of G = 64, 14 of G = 32
constexpr int kSpAux = 48;                        // group constants per unit: 32 B scales + 8 B zeros + 8 B pad
constexpr int kSpLMax = 32;                       // 16-column sets one CTA may touch in one op
constexpr int kSpRows = 4;                        // hand-off rows in rotation (op i publishes into row i % 4)
constexpr int kSpXsumMax = 1024;                  // units along K (K / UK) an op may have

struct __align__(128) SpOp {
  const uint8_t* wstream;      // stream-format weights
  const uint32_t* cta_begin;   // [grid + 1] first unit of every CTA (unit = set * NU + j)
  const __half* bias;
  __half* y;                   // fp16 output of the per-op path (every buffer holds the same values after a run)
  const __half* src;           // source in plain global memory (src_op < 0)
  const __half* norm_w;        // RMSNorm weight [K]
  __half* xout;                // RMSNorm prologue: where the recorded norm wanted its output, or null
  __half* act_out;             // mode 1: where the recorded SiLU*mul wanted its output, or null
  int K, N;
  int uk_shift, F, NU, unit_bytes, ups;
  int mode;                    // 0: plain sets, 1: gate|up pairs (publishes silu(gate) * up, N / 2 columns)
  int prologue;                // kProCopy / kProRmsnorm
  int src_op, src_off;         // >= 0: the source is op src_op's published row, from column src_off
  float eps;
  int ldx;                     // row pitch (elements) of `src` when a batched program stages several rows
  int moe;                     // MoE kernel only: 0 plain op, 1 a MoE block's gate|up (routing prologue), 2 its down
  int moe_i;                   // index of the block's SpMoe
  int pad_[1];
};
static_assert(sizeof(SpOp) == 128, "SpOp layout");

// Sparse-MoE block (stream_moe_kernel): one block = two kernel ops.
//   gate|up (moe = 1): K = H, N = top_k * 2I: the top_k selected experts' gate|up linears side by side, slot-major
//     (set s of the op = set s % (I / 8) of slot s / (I / 8)'s expert, mode 1: publishes top_k x I SiLU*mul words);
//   down (moe = 2): K = top_k * I (the published row unchanged), N = H: unit j of a set reads slot j / (I / UK)'s
//     expert; every CTA keeps one partial row per (set, slot) and publishes sum_k fp16(w_k * slot_k) directly.
// A unit u of either op lives in segment q = u / seg (seg = units per slot: (I / 8) * (H / UK) for gate|up, I / UK
// for down): slot q % top_k, unit (q / top_k) * seg + u % seg of the expert's stream copy.  A bulk copy never crosses
// a segment (the consumers cut their chunks the same way).
constexpr int kSpMoeEMax = 64;                    // experts
constexpr int kSpMoeKMax = 8;                     // top_k
constexpr int kSpMoeSmem = 512;                   // logits [64] f32, weights [8] f32, ids [8] i32, routed op
// QWEN3_MOE blocks (stream_qwen3moe_kernel, whose MoE blocks are all of this kind): up to 128 experts.  The logits are
// not staged in shared memory: CTA c computes the logits e = c mod grid and publishes each as one 64-bit word
// (tag << 32 | f32 bits of the fp16 value) into xlog[e]; warp 0 of every CTA then polls all E words into registers (lane l: experts l, l + 32, l + 64, l + 96) and runs the routing.
// Every CTA publishes before it polls and all CTAs are co-resident (cooperative launch); each word has one writer per
// run, under the run's tag of the op, so nothing is reset.  The routing area keeps its size: its logit slots hold the
// slots' ascending-expert order (m_ord) instead, which the down finish sums in.
constexpr int kSpQwenEMax = 128;
// Finishes of a QWEN3_MOE block (transformers' Qwen3MoeSparseMoeBlock): gate|up publishes fp16(fp16(silu(g)) * u);
// down rounds each slot's sum to fp16(y), takes c = fp16(y * w16) and adds the slots in ascending expert id with an
// fp16 rounding after every add (index_add_ per expert).
struct SpMoe {
  const __half* gate_w;        // router weight [E, H] fp16
  __half* logits;              // [E] fp16 (what nn.Linear returns)
  float* topk_w;               // [top_k] (renormalised when renorm)
  int* topk_ids;               // [top_k]
  int* tok_idx;                // [top_k] token_expert_indices (k * M + m = k)
  int* sorted_ids;             // [sorted_len] moe_align_block_size outputs
  int* expert_ids;
  int* npost;
  __half* down;                // [top_k, H] per-slot down outputs x routing weight
  long long eb_a, eb_b;        // bytes per expert slice of the gate|up / down stream copies
  int E, topk, renorm, block_size, sorted_len;
  int seg_a, seg_b, I;
  unsigned long long* xlog;    // QWEN3_MOE: [E] published logits of this block (program-owned; topk_w then points at
                               // fp16 weights), else null
};

// DEEPSEEK_MOE blocks (stream_deepseek_moe_kernel, whose MoE blocks are all of this kind): the QWEN3_MOE folding and
// logit exchange (xlog, fp32 logits unrounded) plus one shared expert per block, in a side table indexed like SpMoe
// (SpMoe keeps its layout, so the other MoE entries compile as before).  The shared expert's intermediate size is
// I_s = nsh I (DeepSeek's n_shared_experts x moe_intermediate_size), so it runs as nsh more slots of the block's
// segment length: after the top_k routed slots, in the shared expert's own stream copy (shb bytes, 256-byte aligned,
// in front of the E expert slices).
//   gate|up (K = H, N = top_k 2I + 2 I_s): segments q < top_k are routed slots, q >= top_k the shared expert's
//     (unit u - top_k seg_a of its copy).  They need no routing: the producer issues them before the routed-op word is
//     released, while the router logits are exchanged.
//   down (K' = top_k I + I_s, N = H): a set has top_k + nsh partial rows of seg_b units; rows top_k.. read the shared
//     copy (unit set I_s / UK + (row - top_k) seg_b + j).  The finish sums the shared rows in fp32 and rounds them on
//     their own to y_s before adding it to the routed sum.
struct SpDsk {
  const float* bias;           // e_score_correction_bias [E] (sigmoid), else null
  __half* shared_out;          // y_s [H]
  long long shb_a, shb_b;      // bytes of the shared gate|up / down stream copies (in front of the expert slices)
  int scoring, n_group, topk_group, norm;
  float rsf;                   // routed_scaling_factor
  int nsh;                     // I_s / I
};

// Shared memory of the M = 1 stream kernels:
//   sdesc [2] SpOp (256 B) | misc (256 B) | MoE routing area (SpMoeSmem, MOE kernels only) |
//   part [kSpLMax][nw][16] f32 | xsum [kSpXsumMax] f32 | ring [spw][nw] stages | full / empty barriers [spw * nw] each |
//   xs (the activations, K fp16)
// spw = ring stages per consumer warp: the host picks the deepest ring that fits next to the program's activations
// (sp_pick_spw in program.cu); at the minimum depth the layout is as large as with the fixed ring before.  Everything
// in front of the ring sits at a compile-time offset: a base that depends on the program costs registers the kernels
// do not have (9 warps cap a thread at 168, 13 at 128; sizing part and xsum from the program spills 24 / 60 bytes in
// the 8-warp kernel).  Every part is a multiple of 16 bytes.
constexpr int kSpMaxStages = 8;                   // ring stages per warp at most (227 KB allows 6 at 8 warps)
constexpr int kSpMoeOff = 512;                    // the routing area (behind sdesc and misc)
__host__ __device__ constexpr size_t sp_ring_off(int nw, bool moe) {
  return kSpMoeOff + (moe ? kSpMoeSmem : 0) + (size_t)kSpLMax * nw * 16 * 4 + (size_t)kSpXsumMax * 4;
}
// bytes in front of the activations (xs)
__host__ __device__ constexpr size_t sp_fixed_smem(int nw, int spw, bool moe) {
  return sp_ring_off(nw, moe) + (size_t)nw * spw * (kSpStageBytes + 2 * 8);
}
static_assert(sp_fixed_smem(8, 4, false) % 16 == 0 && sp_fixed_smem(12, 3, true) % 16 == 0,
              "xs must stay 16-byte aligned");

__device__ __forceinline__ uint4 ld_relaxed_u4(const void* p) {
  uint4 r;
  asm volatile("ld.relaxed.gpu.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
  return r;
}
__device__ __forceinline__ void st_relaxed_u32(void* p, uint32_t v) {
  asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void st_release_cta_smem(int* p, int v) {
  asm volatile("st.release.cta.shared.s32 [%0], %1;" ::"r"(smem_u32(p)), "r"(v) : "memory");
}
__device__ __forceinline__ int ld_acquire_cta_smem(const int* p) {
  int v;
  asm volatile("ld.acquire.cta.shared.s32 %0, [%1];" : "=r"(v) : "r"(smem_u32(p)) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t sp_tag(int base, int op) { return (uint32_t)((base + op) % 65535 + 1); }

// Residual add folded into an op's finish (B200AWQ_OP_ADD; stream_residual_kernel / stream_batch_residual_kernel): one
// entry per kernel op in a side table (SpOp has no room left).  out == null: the op has no residual.  Otherwise the op
// publishes fp16(fp16(sum [+ bias]) + residual) into its hand-off row and stores it to `out`, and still stores the raw
// fp16(sum [+ bias]) to its y.  The residual of column c, token row m is ext[m N + c] (a buffer no op of the program
// writes: ready at launch) when op < 0, else the tagged word of op `op`'s published row (kSpResWindow ops back at most).
// A SCALED_ADD (mul not NaN) adds fp16(y * mul) instead of y, with the multiply in fp32 (torch's `r + y * a`).
constexpr int kSpResWindow = 4;                   // largest producer - residual distance in kernel ops (program_create;
                                                  // tests/test_stream_residual_model.py derives it)
struct SpRes {
  const __half* ext;
  __half* out;
  int op;
  float mul;   // SCALED_ADD's multiplier (finite); NaN for an ADD, which adds y itself
};
static_assert(sizeof(SpRes) == 24 && offsetof(SpRes, mul) == 20, "SpRes layout (sp_res_mul)");
// res[op].mul, read where the finish uses it by a volatile load that also forms the address: neither the multiplier nor
// a pointer to it is hoisted into a register across the finish loop (the LayerNorm and q / k norm entries have none to
// spare; their register counts are asserted by the CPU tests)
__device__ __forceinline__ float sp_res_mul(const SpRes* res, int op) {
  float v;
  asm volatile("{\n\t.reg .u64 a;\n\tmad.wide.s32 a, %2, 24, %1;\n\tld.global.nc.f32 %0, [a+20];\n\t}"
               : "=f"(v) : "l"(res), "r"(op));
  return v;
}
// the linear's operand of the residual add: y for an ADD (mul NaN), fp16(y * mul) for a SCALED_ADD
__device__ __forceinline__ float sp_res_y(float mul, __half y) {
  return mul == mul ? __half2float(__float2half_rn(__half2float(y) * mul)) : __half2float(y);
}
__device__ __forceinline__ uint32_t ld_relaxed_u32(const void* p) {
  uint32_t r;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(r) : "l"(p) : "memory");
  return r;
}
// the residual of column c (token row m of M) for op `op`: external, or polled from the source op's tagged row
__device__ __forceinline__ float sp_residual(const SpRes& r, const uint32_t* rows, int row_stride, int M, int m, int N,
                                             int c, int base, int op) {
  if (r.op < 0) return __half2float(r.ext[(size_t)m * N + c]);
  const uint32_t* p = rows + ((size_t)(r.op % kSpRows) * M + m) * row_stride + c;
  const uint32_t want = sp_tag(base, r.op);
  uint32_t v = ld_relaxed_u32(p);
  if ((v >> 16) != want) {
    ProgWatch wd;
    do {
      if (wd.tick(kWResidual, op)) break;
      v = ld_relaxed_u32(p);
    } while ((v >> 16) != want);
  }
  return __half2float(__ushort_as_half((unsigned short)(v & 0xffffu)));
}

// ROPE_KV folded into a qkv linear's finish (stream_rope_kernel / stream_batch_rope_kernel): one entry per kernel op in a
// side table, like SpRes.  The op is packed in mode 2 (sp_cols_rot with r.head_dim and r's rotary dim); r.head_dim == 0
// on every other op.  The descriptor is the recorded b200awq_rope_t (rope.cuh does the arithmetic); rot_offset: a
// ROPE_KV_OFFSET's per-sequence rotary offsets (null for every other op).
struct SpRope {
  b200awq_rope_t r;
  const int32_t* rot_offset;
};
// The batched kernels' entry (stream_batch_rope_kernel / stream_batch_qknorm_kernel): SpRope's descriptor and T, the
// tokens per sequence of the op (B200AWQ_OP_ROPE_KV_SEQ's b200awq_op_t.K; 1 for ROPE_KV): token row m = b T + t writes
// cache entry b at position *r.pos + t (rope.cuh: rope_row_pos).  A table of its own: the M = 1 kernels only run T = 1.
// rot_offset as SpRope.
struct SpRopeSeq {
  b200awq_rope_t r;
  const int32_t* rot_offset;
  int T;
  int pad_;
};

// The rotary row of cache row p in the M = 1 finish (one sequence): p plus the offset behind the op's side-table field
// `field` (SpRope::rot_offset, SpQkNorm::rot_offset; null: none).  The finish derives it again for every pair instead of
// carrying it from the range check: carried through the pair loop it costs the M = 1 kernels, already at 168
// registers, a spill; derived here every M = 1 entry keeps the registers and spills it had without offsets.
__device__ __forceinline__ int sp_rot_row(const int32_t* const* field, int p) {
  const int32_t* o = *field;
  return o != nullptr ? p + *o : p;
}

// QK_NORM_ROPE_KV folded into a qkv linear's finish (stream_qknorm_kernel / stream_batch_qknorm_kernel): one entry per
// kernel op in a side table next to SpRope (whose descriptor is the embedded b200awq_rope_t); part == null on every op
// without it.  A head's D / 16 sets can sit on different CTAs, so the finish runs in two phases: (a) every CTA publishes
// the sum-of-squares partial of each of its q / k sets (rope.cuh: qk_set_partial) as one 64-bit word
// (tag << 32 | float bits) into part[m * N / 16 + set]; (b) for each q / k pair it finishes it polls all partials of the
// pair's head in set order (its own included), sums them (qk_head_sum), normalises, rotates and appends.  Every CTA
// publishes before it waits and all CTAs are co-resident (cooperative launch), so no CTA waits on a waiting one.  Each
// word is written once per run, under the run's tag of the op: nothing needs resetting.
struct SpQkNorm {
  b200awq_qk_norm_rope_t q;
  unsigned long long* part;    // [M][N / 16] published set partials of this op (program-owned)
  const int32_t* rot_offset;   // SpRope::rot_offset again: phase (b) reads it from here (sp_qk_finish)
  float inv_d;                 // fp32(1 / head_dim), rounded on the host (rope.cuh: qk_norm_rope_pair)
  int pad_;
};
__device__ __forceinline__ void st_relaxed_u64(void* p, unsigned long long v) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_relaxed_u64(const void* p) {
  unsigned long long r;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(r) : "l"(p) : "memory");
  return r;
}
// a 64-bit word (tag << 32 | f32 bits) published by another CTA, waited for under the op's tag; `code` names the wait
// in the abort record (QK_NORM_ROPE_KV's set partials, QWEN3_MOE's router logits)
__device__ __forceinline__ float sp_tagged_f32(const unsigned long long* p, uint32_t tag, int code, int op) {
  unsigned long long v = ld_relaxed_u64(p);
  if ((uint32_t)(v >> 32) != tag) {
    ProgWatch wd;
    do {
      if (wd.tick(code, op)) break;
      v = ld_relaxed_u64(p);
    } while ((uint32_t)(v >> 32) != tag);
  }
  return __uint_as_float((uint32_t)v);
}
// phase (b): the published partial of one set
__device__ __forceinline__ float sp_qk_partial(const unsigned long long* p, uint32_t tag, int op) {
  return sp_tagged_f32(p, tag, kWQkNorm, op);
}

// set -> original columns (oracle/stream_format.py:set_columns)
__device__ __forceinline__ void sp_cols(int mode, int N, int s, int g, int& lo, int& hi) {
  if (mode == 0) {
    lo = 16 * s + g;
    hi = lo + 8;
  } else {
    lo = 8 * s + g;
    hi = (N >> 1) + lo;
  }
}

// mode 2 (a qkv linear whose ROPE_KV folds into its finish): set s of head h = s / (D / 16) holds the head's column
// pairs p = 8 t + g (t = s % (D / 16)) of rope.cuh's rope_cols with R rotated columns (lo = h D + p, hi = lo + D / 2
// for R = D), so one lane finishes both columns of a rotation
__device__ __forceinline__ void sp_cols_rot(int D, int R, int s, int g, int& lo, int& hi) {
  const int per_head = D >> 4, h = s / per_head, t = s - h * per_head;
  rope_cols(D, R, 8 * t + g, lo, hi);
  lo += h * D;
  hi += h * D;
}

// mode 3 (a q_proj | kv_a_proj_with_mqa linear whose MLA_ROPE folds into its finish): set s holds the adjacent pairs
// lo = 16 s + 2 g, hi = lo + 1, so one lane finishes both elements of an interleaved rotary pair
__device__ __forceinline__ void sp_cols_pairs(int s, int g, int& lo, int& hi) {
  lo = 16 * s + 2 * g;
  hi = lo + 1;
}

// MLA_ROPE / MLA_KV folded into a linear's finish (stream_mla_kernel): one entry per kernel op in a side table, like
// SpRope.  kind 1: the op is packed in mode 3 and its finish runs rope.cuh's mla_rope_pair on every pair; kind 2: a
// mode-0 kv_b_proj op whose finish stores every column with mla_kv_col; kind 0 on every other op.
// wait_words > 0: the op stages a slice of an MLA_ROPE producer's row (kv_a_layernorm of c_kv, kv_b_proj's prologue) and
// first waits for one word of every 16-column set of that row (wait_words columns): each is published by the set's owner
// after it finished every earlier op, as a whole-row staging shows, so program_create's residual rule may count this
// staging as one (ProgOp::stage_row).
// stream_mla_lora_kernel adds kind 3 (MLA_K_ROPE: mode 3, k_pe of the row rotated into k_cache) and kind 4 (MLA_Q_ROPE:
// mode 3, the row rotated into q_out); there wait_words polls the previous op's row (wait_words = its N), which covers
// kv_b_proj staging the c_kv slice of the K_ROPE row two ops back.
struct SpMla {
  b200awq_mla_t d;
  int kind;
  int wait_words;
};

// LAYER_NORM / GELU / GELU_TANH folded into a linear (stream_layernorm_kernel): one entry per kernel op in a side table,
// like SpRope.  bias: the LayerNorm bias of the op's staging prologue (prologue kProLayernorm; null without one);
// gelu: 1 (exact) or 2 (tanh) when the op's mode-0 finish publishes fp16(gelu(y)) and stores it to act_out, else 0.
struct SpLn {
  const __half* bias;
  int gelu;
  int pad_;
};

// phase (b) of a QK_NORM_ROPE_KV finish (SpQkNorm above), shared by the M = 1 and the batched body: item t of this
// thread (t = ct, ct + nthr, ... < nsets * per_set; per_set = 8 M) is lane group t % 8 of token row (t % per_set) / 8 of
// local set t / per_set, whose fp16 pair phase (a) kept in part[(ls * kst + m) * 16 + g] / [.. + 8].  T >= 1 (the
// batched body): p0 = *pos and T tokens per sequence, each row's entry, cache row and rotary row from rope.cuh's
// rope_row_pos (a row out of range writes nothing); T = 0 (the M = 1 body): p0 is the step's cache row, already checked
// with its rotary row (sp_rot_row), entry m.
__device__ __forceinline__ void sp_qk_finish(const SpQkNorm* __restrict__ qn, int p0, int T, const float* part, int kst,
                                          int ct, int nthr, int nsets, int per_set, int set0, int N, uint32_t tag, int op) {
  const b200awq_rope_t& rp = qn->q.rope;
  const int per_head = rp.head_dim >> 4, hqk = rp.n_heads + rp.n_kv_heads;
  for (int t = ct; t < nsets * per_set; t += nthr) {
    const int ls = t / per_set, r = t - ls * per_set, m = r >> 3, gg = r & 7, hd = (set0 + ls) / per_head;
    const float* keep = part + ((size_t)ls * kst + m) * 16;
    int clo, chi;
    sp_cols_rot(rp.head_dim, rp.head_dim, set0 + ls, gg, clo, chi);   // (full rotary: program_create checks it)
    const __half a = __float2half_rn(keep[gg]), b = __float2half_rn(keep[gg + 8]);
    int e = m, rpos = p0, rot;
    if (T == 0) rot = sp_rot_row(&qn->rot_offset, p0);
    else if ((rpos = rope_row_pos(rp, p0, T, qn->rot_offset, m, e, rot)) < 0) continue;
    if (hd >= hqk) {   // v head: not normalised, only appended
      rope_pair(rp, rpos, rot, m, e, clo, chi, a, b);
      continue;
    }
    const unsigned long long* hp = qn->part + (size_t)m * (N >> 4) + (size_t)hd * per_head;
    const float ss = qk_head_sum(per_head, [&](int u) { return sp_qk_partial(hp + u, tag, op); });
    qk_norm_rope_pair(qn->q, qn->inv_d, rpos, rot, m, e, clo, a, b, ss);
  }
}

// ------------------------------------------------------------------------------------------ re-layout kernel
// One thread per output word / per group-constant slot; run once per linear at program creation.  cols(s, g, lo, hi)
// maps set s, lane group g to its two original columns.
template <typename Cols>
__device__ __forceinline__ void sp_pack(const int32_t* __restrict__ qweight, const __half* __restrict__ scales,
                                        const int32_t* __restrict__ qzeros, uint8_t* __restrict__ out, int K, int N,
                                        int G, Cols cols) {
  const int UK = G < 128 ? G : 128, F = UK >> 4, NU = K / UK, UB = F * 128 + kSpAux;
  const int NW = N >> 3;
  const int wpu = F * 32 + 12;   // 32-bit slots per unit: fragment words + 8 scale pairs + 2 zero words + 2 pad
  const int64_t total = (int64_t)(N >> 4) * NU * wpu;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int slot = (int)(i % wpu);
    const int64_t unit = i / wpu;
    const int j = (int)(unit % NU), s = (int)(unit / NU);
    uint8_t* ub = out + unit * UB;
    auto nib = [&](int k, int col) -> uint32_t {
      const uint32_t w = (uint32_t)qweight[(int64_t)k * NW + (col >> 3)];
      const int jj = col & 7;
      return (w >> (4 * ((jj >> 1) + 4 * (jj & 1)))) & 0xFu;   // 4 * AWQ_REVERSE_ORDER[jj]
    };
    if (slot < F * 32) {
      int f, lane;
      if (F >= 4) {          // [quad][lane][4]
        const int quad = slot >> 7, r = slot & 127;
        lane = r >> 2;
        f = quad * 4 + (r & 3);
      } else {               // [lane][2]
        lane = slot >> 1;
        f = slot & 1;
      }
      const int g = lane >> 2, tig = lane & 3;
      int lo, hi;
      cols(s, g, lo, hi);
      const int k0 = j * UK + 16 * f + 2 * tig;
      const uint32_t w = nib(k0, lo) | nib(k0, hi) << 4 | nib(k0 + 8, lo) << 8 | nib(k0 + 8, hi) << 12 |
                         nib(k0 + 1, lo) << 16 | nib(k0 + 1, hi) << 20 | nib(k0 + 9, lo) << 24 | nib(k0 + 9, hi) << 28;
      reinterpret_cast<uint32_t*>(ub)[slot] = w;
    } else {
      const int a = slot - F * 32;      // 0..7 scale pairs, 8..9 zero words, 10..11 pad
      const int grp = (j * UK) / G;
      uint32_t v = 0;
      if (a < 8) {
        int lo, hi;
        cols(s, a, lo, hi);
        const __half sl = scales[(int64_t)grp * N + lo], sh = scales[(int64_t)grp * N + hi];
        v = (uint32_t)__half_as_ushort(sl) | (uint32_t)__half_as_ushort(sh) << 16;
      } else if (a < 10) {
        for (int b = 0; b < 4; ++b) {
          const int g = (a - 8) * 4 + b;
          int lo, hi;
          cols(s, g, lo, hi);
          auto znib = [&](int col) -> uint32_t {
            const uint32_t w = (uint32_t)qzeros[(int64_t)grp * NW + (col >> 3)];
            const int jj = col & 7;
            return (w >> (4 * ((jj >> 1) + 4 * (jj & 1)))) & 0xFu;
          };
          v |= (znib(lo) | znib(hi) << 4) << (8 * b);
        }
      }
      reinterpret_cast<uint32_t*>(ub + F * 128)[a] = v;
    }
  }
}

__global__ void __launch_bounds__(256)
    stream_pack_kernel(const int32_t* __restrict__ qweight, const __half* __restrict__ scales,
                       const int32_t* __restrict__ qzeros, uint8_t* __restrict__ out, int K, int N, int G, int mode) {
  sp_pack(qweight, scales, qzeros, out, K, N, G,
          [=](int s, int g, int& lo, int& hi) { sp_cols(mode, N, s, g, lo, hi); });
}
__global__ void __launch_bounds__(256)
    stream_pack_rotary_kernel(const int32_t* __restrict__ qweight, const __half* __restrict__ scales,
                              const int32_t* __restrict__ qzeros, uint8_t* __restrict__ out, int K, int N, int G,
                              int head_dim, int rotary_dim) {
  pdl_wait();   // (launched without the PDL attribute: a no-op, kept so the kernel stays safe under one)
  sp_pack(qweight, scales, qzeros, out, K, N, G,
          [=](int s, int g, int& lo, int& hi) { sp_cols_rot(head_dim, rotary_dim, s, g, lo, hi); });
}

__global__ void __launch_bounds__(256)
    stream_pack_pairs_kernel(const int32_t* __restrict__ qweight, const __half* __restrict__ scales,
                             const int32_t* __restrict__ qzeros, uint8_t* __restrict__ out, int K, int N, int G) {
  pdl_wait();   // (launched without the PDL attribute: a no-op, kept so the kernel stays safe under one)
  sp_pack(qweight, scales, qzeros, out, K, N, G, [=](int s, int g, int& lo, int& hi) { sp_cols_pairs(s, g, lo, hi); });
}

// ------------------------------------------------------------------------------------------ the kernel
// One unit (one 16-column set, UK = 16 F rows of K) times the activations, folded with the unit's group constants:
// returns the unit's contribution to the lo / hi column of lane group g (token 0).
//   raw sums:  S = sum_k x_k (1024 + c q)   (mma.sync on the raw codes, two accumulator chains: even / odd fragments)
//   fold:      s (S - (1024 + c z) X) / c   with X = sum_k x_k of the unit   (csrc/gemv_tile.cuh:v3_fold)
// NU units in flight per call (sp_units<F, NU>): a single unit is one long dependency chain (LDS -> unpack -> 4
// chained HMMA -> fold, a few hundred cycles) and a warp has nothing else to overlap it with: unit-at-a-time the
// kernel is bound by that latency, not by the tensor pipe.  Four units interleaved give eight independent chains per
// warp.
template <int F, int NUQ>
__device__ __forceinline__ void sp_units(const uint8_t* __restrict__ st, int UB, const uint32_t* __restrict__ xs,
                                         const float* __restrict__ xsum, const int (&ju)[NUQ], int lane, bool xl,
                                         float (&tlo)[NUQ], float (&thi)[NUQ]) {
  constexpr uint32_t MA = 0x000f000fu, MB = 0x00f000f0u, MG = 0x64006400u;
  const int g = lane >> 2, tig = lane & 3;
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
      if (xl) xb = *reinterpret_cast<const uint2*>(xs + ((size_t)ju[i] * F + f) * 8 + tig * 2);
      const uint32_t w = wq[i][f], w8 = w >> 8;
      mma_16816(acc[i][f & 1], lop3_and_or(w, MA, MG), lop3_and_or(w, MB, MG), lop3_and_or(w8, MA, MG),
                lop3_and_or(w8, MB, MG), xb.x, xb.y);
    }
  }
#pragma unroll
  for (int i = 0; i < NUQ; ++i) {
    const uint8_t* ax = st + (size_t)i * UB + F * 128;
    const float2 sc = __half22float2(u32_as_h2(*reinterpret_cast<const uint32_t*>(ax + 4 * g)));
    const uint32_t zb = ax[32 + g];
    const float X = xsum[ju[i]];
    const float s_lo = acc[i][0][0] + acc[i][1][0], s_hi = acc[i][0][2] + acc[i][1][2];
    tlo[i] = sc.x * (s_lo - (1024.f + static_cast<float>(zb & 0xFu)) * X);
    thi[i] = (sc.y * 0.0625f) * (s_hi - (1024.f + 16.f * static_cast<float>(zb >> 4)) * X);
  }
}

// a chunk of n units starting at unit j (within its set): apply(t_lo, t_hi) is called once per unit, in unit order
// (so the sums do not depend on how the chunk was cut into groups of four)
template <int F, int GR, typename Apply>
__device__ __forceinline__ void sp_chunk(const uint8_t* __restrict__ st, int UB, int n, const uint32_t* __restrict__ xs,
                                         const float* __restrict__ xsum, int j, int NU, int lane, bool xl, Apply&& apply) {
  int i = 0;
  for (; i + GR <= n; i += GR) {
    int ju[GR];
#pragma unroll
    for (int q = 0; q < GR; ++q) {
      ju[q] = j + i + q;
      if (ju[q] >= NU) ju[q] -= NU;      // the chunk may run across a set boundary (at most one: NU >= units per chunk)
    }
    float a[GR], b[GR];
    sp_units<F, GR>(st + (size_t)i * UB, UB, xs, xsum, ju, lane, xl, a, b);
#pragma unroll
    for (int q = 0; q < GR; ++q) apply(a[q], b[q]);
  }
  for (; i < n; ++i) {
    int ju[1] = {j + i >= NU ? j + i - NU : j + i};
    float a[1], b[1];
    sp_units<F, 1>(st + (size_t)i * UB, UB, xs, xsum, ju, lane, xl, a, b);
    apply(a[0], b[0]);
  }
}

// debug stamps (knob 3 = 2), per op and CTA (first 8 CTAs, first 32 ops):
// [0] op begin, [1] source row complete (poll over), [2] activations staged, [3] warp 0's first chunk landed,
// [4] warp 0 finished its units, [5] all warps finished, [6] outputs published, [7] routing published (the gate|up op
// of a MoE block; 0 for other ops)
// knob 3 = 8: per-WARP stamps of the first 8 CTAs / 16 ops: g_sp_dbg[op][cta][warp][slot], slots: 0 op begin, 1 own
// polls done, 2 staged (past the barrier), 3 first chunk landed, 4 own units done, 5 past the post-loop barrier,
// 6 own finish stores issued.  (A timer read right after bar.sync captures the ARRIVAL: the barrier blocks at the next
// instruction that touches barrier-protected state - hence the shared-memory read in front of slots 2 and 5.)
__device__ unsigned long long g_sp_dbg[16 * 8 * 8 * 8];
cudaError_t stream_debug_read(void* dst, size_t bytes) {
  return cudaMemcpyFromSymbol(dst, g_sp_dbg, bytes < sizeof(g_sp_dbg) ? bytes : sizeof(g_sp_dbg));
}
#define SP_WSTAMP(slot)                                                                                          \
  do {                                                                                                           \
    if (dbg == 8 && blockIdx.x < 8 && op < 16) {                                                                 \
      __syncwarp();                                                                                              \
      if (lane == 0) g_sp_dbg[((op * 8 + blockIdx.x) * 8 + cw) * 8 + (slot)] = prog_timer();                    \
    }                                                                                                            \
  } while (0)
#define SP_TOUCH_SMEM()                                                                      \
  do {                                                                                       \
    if (dbg == 8) {                                                                          \
      int tv_;                                                                               \
      asm volatile("ld.volatile.shared.s32 %0, [%1];" : "=r"(tv_) : "r"(smem_u32(wfirst)) : "memory"); \
      if (tv_ == 0x7fffffff) __trap();                                                       \
    }                                                                                        \
  } while (0)
#define SP_STAMP(slot)                                                                                       \
  do {                                                                                                       \
    if (dbg == 2 && ct == 0 && blockIdx.x < 8 && op < 32) g_prog_dbg[(op * 8 + blockIdx.x) * 8 + (slot)] = prog_timer(); \
  } while (0)

__device__ __forceinline__ void cp_async_16(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_4(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// MOE kernel: the routing area in shared memory, right behind the fixed part
struct SpMoeSmem {
  float* m_logit;      // [64] widened fp16 logits (QWEN3_MOE: int [8] ascending-expert order of the slots)
  float* m_w;          // [8] routing weights
  int* m_ids;          // [8] expert of each slot
  int* routed_op;      // last gate|up op whose routing is in m_w / m_ids (release / acquire at CTA scope)
};
__device__ __forceinline__ SpMoeSmem sp_moe_smem(uint8_t* area) {
  SpMoeSmem s;
  s.m_logit = reinterpret_cast<float*>(area);
  s.m_w = s.m_logit + kSpMoeEMax;
  s.m_ids = reinterpret_cast<int*>(s.m_w + kSpMoeKMax);
  s.routed_op = s.m_ids + kSpMoeKMax;
  return s;
}

// The kernel body is program_stream_body.inc: stream_program_kernel<NW, GR> (MOE = false; `moe` unused) and
// stream_moe_kernel (programs with sparse-MoE blocks, SpMoe above) include it.  Every MoE-only step sits behind
// `if constexpr (MOE)`: stream_program_kernel is the plain kernel, instruction for instruction.
// (MOE is only ever false here; it is a template parameter rather than a local constant because a local constant,
// unlike the parameter, changes the register assignment ptxas makes for this kernel)
// spw: ring stages per consumer warp (sp_fixed_smem above)
template <int NW, int GR, bool MOE = false>
__global__ void __launch_bounds__(32 + NW * 32, 1)
    stream_program_kernel(const SpOp* __restrict__ ops, const uint32_t* __restrict__ cta_all, int n_ops,
                          uint32_t* __restrict__ rows, int row_stride, int* __restrict__ state, int spw, int dbg,
                          int l2_ahead, int gate_ahead, const SpMoe* __restrict__ moe) {
#include "program_stream_body.inc"
}

// programs with sparse-MoE blocks: 8 consumer warps
__global__ void __launch_bounds__(32 + 8 * 32, 1)
    stream_moe_kernel(const SpOp* __restrict__ ops, const uint32_t* __restrict__ cta_all, int n_ops,
                      uint32_t* __restrict__ rows, int row_stride, int* __restrict__ state, int spw, int dbg,
                      int l2_ahead, int gate_ahead, const SpMoe* __restrict__ moe) {
  constexpr int NW = 8, GR = 4;
  constexpr bool MOE = true;
  pdl_wait();   // nothing is read before the predecessor is done, should it ever be launched with PDL (a no-op under
                // the cooperative launch of program_run)
#include "program_stream_body.inc"
}

// M = 1 programs with residual adds (SpRes above), with or without sparse-MoE blocks: the MoE instantiation plus the
// residual steps of the finish, which only SP_RESIDUAL compiles in (the kernels above do not see them at all)
__global__ void __launch_bounds__(32 + 8 * 32, 1)
    stream_residual_kernel(const SpOp* __restrict__ ops, const uint32_t* __restrict__ cta_all, int n_ops,
                           uint32_t* __restrict__ rows, int row_stride, int* __restrict__ state, int spw, int dbg,
                           int l2_ahead, int gate_ahead, const SpMoe* __restrict__ moe, const SpRes* __restrict__ res) {
  constexpr int NW = 8, GR = 4;
  constexpr bool MOE = true;
  pdl_wait();
#define SP_RESIDUAL 1
#include "program_stream_body.inc"
#undef SP_RESIDUAL
}

// M = 1 programs with a ROPE_KV op (SpRope above), with or without residual adds and sparse-MoE blocks: the residual
// kernel plus the rotation / cache stores of a mode-2 finish, which only SP_ROPE compiles in
__global__ void __launch_bounds__(32 + 8 * 32, 1)
    stream_rope_kernel(const SpOp* __restrict__ ops, const uint32_t* __restrict__ cta_all, int n_ops,
                       uint32_t* __restrict__ rows, int row_stride, int* __restrict__ state, int spw, int dbg,
                       int l2_ahead, int gate_ahead, const SpMoe* __restrict__ moe, const SpRes* __restrict__ res,
                       const SpRope* __restrict__ rope) {
  constexpr int NW = 8, GR = 4;
  constexpr bool MOE = true;
  pdl_wait();
#define SP_RESIDUAL 1
#define SP_ROPE 1
#include "program_stream_body.inc"
#undef SP_ROPE
#undef SP_RESIDUAL
}

// M = 1 programs with a QK_NORM_ROPE_KV op (SpQkNorm above): the rope kernel plus the two-phase q / k norm of the
// mode-2 finish, which only SP_QKNORM compiles in (programs with plain ROPE_KV ops only keep stream_rope_kernel)
__global__ void __launch_bounds__(32 + 8 * 32, 1)
    stream_qknorm_kernel(const SpOp* __restrict__ ops, const uint32_t* __restrict__ cta_all, int n_ops,
                         uint32_t* __restrict__ rows, int row_stride, int* __restrict__ state, int spw, int dbg,
                         int l2_ahead, int gate_ahead, const SpMoe* __restrict__ moe, const SpRes* __restrict__ res,
                         const SpRope* __restrict__ rope, const SpQkNorm* __restrict__ qkn) {
  constexpr int NW = 8, GR = 4;
  constexpr bool MOE = true;
  pdl_wait();
#define SP_RESIDUAL 1
#define SP_ROPE 1
#define SP_QKNORM 1
#include "program_stream_body.inc"
#undef SP_QKNORM
#undef SP_ROPE
#undef SP_RESIDUAL
}

// M = 1 programs with QWEN3_MOE blocks (with or without residual adds, ROPE_KV and QK_NORM_ROPE_KV ops): the qknorm
// kernel with the Qwen3-MoE routing and finishes, which only SP_QWEN3 compiles in.  Every MoE block of such a program
// is a QWEN3_MOE block (program_create replays a program that mixes them with SPARSE_MOE per op).  It takes every side
// table (ProgKernel in program.cu), with empty entries where an op has no add, rotation or norm.
__global__ void __launch_bounds__(32 + 8 * 32, 1)
    stream_qwen3moe_kernel(const SpOp* __restrict__ ops, const uint32_t* __restrict__ cta_all, int n_ops,
                           uint32_t* __restrict__ rows, int row_stride, int* __restrict__ state, int spw, int dbg,
                           int l2_ahead, int gate_ahead, const SpMoe* __restrict__ moe, const SpRes* __restrict__ res,
                           const SpRope* __restrict__ rope, const SpQkNorm* __restrict__ qkn) {
  constexpr int NW = 8, GR = 4;
  constexpr bool MOE = true;
  pdl_wait();
#define SP_RESIDUAL 1
#define SP_ROPE 1
#define SP_QKNORM 1
#define SP_QWEN3 1
#include "program_stream_body.inc"
#undef SP_QWEN3
#undef SP_QKNORM
#undef SP_ROPE
#undef SP_RESIDUAL
}

// M = 1 programs with DEEPSEEK_MOE blocks (SpDsk above; with or without residual adds, ROPE_KV and QK_NORM_ROPE_KV
// ops): the Qwen3-MoE kernel with DeepSeek's routing, the shared expert and its finishes, which only SP_DEEPSEEK
// compiles in.  Every MoE block of such a program is a DEEPSEEK_MOE block.
__global__ void __launch_bounds__(32 + 8 * 32, 1)
    stream_deepseek_moe_kernel(const SpOp* __restrict__ ops, const uint32_t* __restrict__ cta_all, int n_ops,
                               uint32_t* __restrict__ rows, int row_stride, int* __restrict__ state, int spw, int dbg,
                               int l2_ahead, int gate_ahead, const SpMoe* __restrict__ moe, const SpRes* __restrict__ res,
                               const SpRope* __restrict__ rope, const SpQkNorm* __restrict__ qkn,
                               const SpDsk* __restrict__ dsk) {
  constexpr int NW = 8, GR = 4;
  constexpr bool MOE = true;
  pdl_wait();
#define SP_RESIDUAL 1
#define SP_ROPE 1
#define SP_QKNORM 1
#define SP_QWEN3 1
#define SP_DEEPSEEK 1
#include "program_stream_body.inc"
#undef SP_DEEPSEEK
#undef SP_QWEN3
#undef SP_QKNORM
#undef SP_ROPE
#undef SP_RESIDUAL
}

// M = 1 programs with MLA_ROPE / MLA_KV ops (SpMla above), with or without DEEPSEEK_MOE blocks (a DeepSeek segment, or
// its dense first layer): the DeepSeek-MoE kernel plus the mode-3 rotation and the q / k / v stores of the finish, which
// only SP_MLA compiles in.  Every rotated pair lives in one lane: no cross-CTA exchange.
__global__ void __launch_bounds__(32 + 8 * 32, 1)
    stream_mla_kernel(const SpOp* __restrict__ ops, const uint32_t* __restrict__ cta_all, int n_ops,
                      uint32_t* __restrict__ rows, int row_stride, int* __restrict__ state, int spw, int dbg,
                      int l2_ahead, int gate_ahead, const SpMoe* __restrict__ moe, const SpRes* __restrict__ res,
                      const SpRope* __restrict__ rope, const SpQkNorm* __restrict__ qkn, const SpDsk* __restrict__ dsk,
                      const SpMla* __restrict__ mla) {
  constexpr int NW = 8, GR = 4;
  constexpr bool MOE = true;
  pdl_wait();
#define SP_RESIDUAL 1
#define SP_ROPE 1
#define SP_QKNORM 1
#define SP_QWEN3 1
#define SP_DEEPSEEK 1
#define SP_MLA 1
#include "program_stream_body.inc"
#undef SP_MLA
#undef SP_DEEPSEEK
#undef SP_QWEN3
#undef SP_QKNORM
#undef SP_ROPE
#undef SP_RESIDUAL
}

// M = 1 programs with MLA_K_ROPE / MLA_Q_ROPE ops (MLA with a q LoRA; SpMla kinds 3 / 4), with or without DEEPSEEK_MOE
// blocks: stream_mla_kernel plus SP_MLA_LORA.  The mode-3 finish runs rope.cuh's mla_lora_pair (k_pe of the fused
// q_a | kv_a row into every head's k row, or q_b's row into q_out), and an op that stages a slice of a K_ROPE op's row
// first polls one word of every set of the PREVIOUS op's row (SpMla::wait_words; kv_b's source is two ops back).
__global__ void __launch_bounds__(32 + 8 * 32, 1)
    stream_mla_lora_kernel(const SpOp* __restrict__ ops, const uint32_t* __restrict__ cta_all, int n_ops,
                           uint32_t* __restrict__ rows, int row_stride, int* __restrict__ state, int spw, int dbg,
                           int l2_ahead, int gate_ahead, const SpMoe* __restrict__ moe, const SpRes* __restrict__ res,
                           const SpRope* __restrict__ rope, const SpQkNorm* __restrict__ qkn,
                           const SpDsk* __restrict__ dsk, const SpMla* __restrict__ mla) {
  constexpr int NW = 8, GR = 4;
  constexpr bool MOE = true;
  pdl_wait();
#define SP_RESIDUAL 1
#define SP_ROPE 1
#define SP_QKNORM 1
#define SP_QWEN3 1
#define SP_DEEPSEEK 1
#define SP_MLA 1
#define SP_MLA_LORA 1
#include "program_stream_body.inc"
#undef SP_MLA_LORA
#undef SP_MLA
#undef SP_DEEPSEEK
#undef SP_QWEN3
#undef SP_QKNORM
#undef SP_ROPE
#undef SP_RESIDUAL
}

// M = 1 programs with LAYER_NORM / GELU / GELU_TANH ops (SpLn above; Command-R, StarCoder2 and MPT blocks), with or
// without residual adds and ROPE_KV ops: stream_rope_kernel plus SP_LAYERNORM, which compiles in the LayerNorm staging
// (sum of x while staging, the centred sum of squares from the staged row after a CTA barrier, then the normalisation in
// place) and the GELU of a mode-0 finish.  Neither crosses CTAs.  A program with these ops has no MoE, q / k norm or
// MLA op (program_create).
__global__ void __launch_bounds__(32 + 8 * 32, 1)
    stream_layernorm_kernel(const SpOp* __restrict__ ops, const uint32_t* __restrict__ cta_all, int n_ops,
                            uint32_t* __restrict__ rows, int row_stride, int* __restrict__ state, int spw, int dbg,
                            int l2_ahead, int gate_ahead, const SpMoe* __restrict__ moe, const SpRes* __restrict__ res,
                            const SpRope* __restrict__ rope, const SpLn* __restrict__ lnt) {
  constexpr int NW = 8, GR = 4;
  constexpr bool MOE = true;
  pdl_wait();
#define SP_RESIDUAL 1
#define SP_ROPE 1
#define SP_LAYERNORM 1
#include "program_stream_body.inc"
#undef SP_LAYERNORM
#undef SP_ROPE
#undef SP_RESIDUAL
}

}  // namespace b200awq
