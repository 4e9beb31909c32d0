// b2m_internal.h -- declarations shared by the kernel translation units and the C-ABI layer.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace b2m {

enum : int { ACT_NONE = 0, ACT_SILU = 1, ACT_RELU = 2, ACT_GELU = 3 };
enum : int { EPI_ACT16 = 0, EPI_LINEAR_F32 = 1 };

// router kinds (which reference routing function is restated)
enum : int {
  ROUTER_MIXTRAL = 0,          // moe_infinity/models/mixtral.py:48-54
  ROUTER_DEEPSEEK_GREEDY = 1,  // modeling_deepseek.py:467-483,508-512
  ROUTER_DEEPSEEK_GROUP = 2,   // modeling_deepseek.py:484-505
  ROUTER_SWITCH_TOP1 = 3,      // HF 4.x SwitchTransformersTop1Router (switch_transformers.py:76)
  ROUTER_DEEPSEEK_V3 = 4,      // modeling_deepseek_v3/modeling_deepseek.py:466-527 (sigmoid, noaux_tc)
  ROUTER_QWEN_MOE = 5,         // transformers Qwen2MoeTopKRouter / Qwen3MoeTopKRouter (model-dtype logits, fp32 weights)
  ROUTER_LLAMA4 = 6,           // transformers Llama4Router (top-k of model-dtype logits, rounded sigmoid weights scale the inputs)
};
// combine kinds (which reference combine loop is restated)
enum : int {
  COMBINE_MIXTRAL = 0,   // mixtral.py:96-101 (weights in model dtype, product and += rounded to model dtype)
  COMBINE_DEEPSEEK = 1,  // deepseek.py:123-128 (+133-136 shared experts); fp32 weights
  COMBINE_SWITCH = 2,    // switch_transformers.py:99-109
  COMBINE_FP32 = 3,      // fast path: fp32 accumulate, single rounding
  COMBINE_QWEN = 4,      // Qwen2MoeExperts + Qwen2MoeSparseMoeBlock: product and += rounded, fp32 weights; gated shared expert
  COMBINE_QWEN_GATE = 5, // the first phase of a Qwen2 combine, launched ahead of it on the shared-expert stream: out[t] =
                         // sigmoid(x[t] . shared_gate_w) in the model dtype (x [T,H], shared_gate_w [H], out [T], 16-bit)
  COMBINE_LLAMA4 = 6,    // Llama4TextMoe: unweighted fp32 sum of the rounded expert outputs, rounded once, + rounded shared
};

// Where a tensor-core GEMM's A operand (the weight tile) comes from: GemmParams::a_src, the kernels' AS template parameter
enum : int { AS_BF16 = 0,   // bf16 tile in shared memory, read by the wgmma itself
             AS_PK12 = 1,   // bf16 tile or 12-bit packed record (weight_pack.cuh), decoded into register fragments
             AS_FP8 = 2,    // e4m3 tile + 128x128 block scales (fp8_weights.cuh), dequantised into register fragments
             AS_INT4 = 3,   // 4-bit code tile + per-128-input scale / zero point (int4_weights.cuh), dequantised likewise
             AS_FP8_ROW = 4 };  // e4m3 tile as AS_FP8 + one fp32 scale per weight row (fp8_weights.cuh)

struct GemmParams {
  const int* offsets;   // [E+1] first permuted row of each expert
  const int* slot_of;   // [E]   HBM slot of each expert of this layer (-1: not resident -> skipped)
  int E;
  int M;                // weight rows per expert
  int K;                // reduction length
  int ksplit;           // split-K factor (EPI_LINEAR_F32 only)
  int stream_k;         // with ksplit > 1: ignore the factor and give every CTA an equal, contiguous share of all
                        // (tile, k-block) units; a CTA red.adds one partial per tile segment it crosses
  int epi;              // EPI_*
  int act;              // ACT_*
  int mimic;            // replay the reference's per-op rounding to the model dtype
  void* out;
  int ld_out;
  int single_n;         // >= 0: one expert (E must be 1) with single_n rows in slot single_slot; offsets/slot_of unused
  int single_slot;
  int pdl_edge;         // launch with a programmatic edge (prologue overlaps the predecessor's tail; waits before any global access)
  int early_a;          // launched with a programmatic edge: weight tiles may be fetched before the predecessor finishes
  int dual_m;           // DUAL kernel, EPI_LINEAR_F32: A1 = rows m0+128.. of the same matrix (two m-tiles share a token tile)
  // bias experts (NLLB / FSGPT, expert_module.cpp:88-92,124-128): bias[m] of the expert in slot s lives at
  // bias_base + s * bias_slot_elems + bias_off (16-bit elements of the model dtype); null = no bias.  Needs ksplit == 1.
  const void* bias_base;
  size_t bias_slot_elems;
  size_t bias_off;
  // ---- expert-parallel "direct" mode (ep_rows > 0; csrc/ep.cu header): the token operand is this rank's peer-written receive
  // area itself.  Every local expert owns a region of ep_rows = nranks*cap rows (its worst case); the source ranks claim rows
  // in it from the front with (remote) atomics on ep_cnt[local expert], so the rows of an expert are contiguous and the tile
  // width follows the actual count -- no regroup kernel, no host involvement.
  int m_rows;                // 0 = 128; else weight rows per tile (A maps carry that box), see gemm_body
  int ep_l2pf;               // direct mode: k-blocks of every expected weight tile to prefetch into L2 before the flag wait
  int ep_rows;               // 0 = off; else rows per expert region
  int ep_first;              // first global expert id owned by this rank
  int ep_el;                 // experts per rank
  int* ep_cnt;               // [ep_el] rows claimed in each local expert's region (cleared by the down GEMM's last CTA)
  int ep_nranks;
  int ep_wait;               // (kept for diagnostics) 1 = gate/up GEMM, the launch that actually has to wait for the peers
  const int* ep_flag;        // [nranks] this rank's receive flags
  const int* ep_epoch;       // local epoch word the flags must reach
  float* ep_zero;            // fp32 accumulator of the down projection, cleared once the flags have been seen
  size_t ep_zero_elems;
  int ep_signal;             // 1: when the whole grid has finished, publish *ep_done_epoch + 1 to every peer (down GEMM)
  int* ep_done_ctr;          // CTA arrival counter (0 between launches)
  int* ep_done_epoch;        // local epoch word of the return direction
  int* ep_peer_done_flag[16];  // peer r's done_flag[nranks] (this rank writes entry [rank])
  int ep_rank;
  unsigned long long* tl;    // optional timeline slots of this launch: [0] first CTA start, [1] peers' flags seen, [2] last CTA end (ns)
  // ---- packed weights (weight_pack.cuh; bf16, 16..64-token tiles, single 128-row m-tiles).  pk_ok[slot] bit b set: matrix b
  // of the slot has a current packed copy, read instead of the bf16 arena.  A0 / A1 of this GEMM are matrices pk_bit0 / pk_bit1.
  const int* pk_ok;          // null = bf16 only
  int pk_bit0, pk_bit1;
  const uint8_t* pk_a0;      // packed A0 / A1 of slot 0: records in (m-tile, k-block) order, pk_slot_bytes apart
  const uint8_t* pk_a1;
  size_t pk_slot_bytes;
  // packing request (host side, read by launch_grouped_gemm_tc before it launches the GEMM): pack the matrices of these slots
  const int* pack_slots;     // host array, pack_n entries; null / 0 = nothing to pack
  int pack_n;
  int pack_nmat;             // matrices per slot
  const uint8_t* pack_src;   // bf16 arena
  size_t pack_src_slot_bytes;
  size_t pack_src_off[3];    // byte offset of matrix b inside a bf16 slot ...
  size_t pack_dst_off[3];    // ... and of its packed copy inside a packed slot
  int pack_rows[3], pack_cols[3];
  uint8_t* pack_dst;         // packed arena (pk_slot_bytes per slot)
  int* pack_ok;              // = pk_ok, writable
  // ---- quantised weights (AS_FP8, AS_FP8_ROW, AS_INT4): the A maps are uint8 maps over the quantised matrices, and grid0 / grid1 are
  // the side grids of A0 / A1 in slot 0, grid_slot_bytes apart: fp32 block scales [M / 128][K / 128] or row scales [M]
  // (fp8_weights.cuh), or tile-major group words, one uint32 per row and 128 k (int4_weights.cuh)
  const uint8_t* grid0;
  const uint8_t* grid1;
  size_t grid_slot_bytes;
  int a_src;                 // AS_*: how the GEMM reads its A operand (read by the launcher, which picks the kernel)
};

// packed copy of a rows x cols K-major bf16 matrix (weight_pack.cuh); 0 when its shape does not divide into tiles
inline size_t packed_matrix_bytes(int rows, int cols) {
  if (rows % 128 || cols % 64) return 0;
  return (size_t)(rows / 128) * (size_t)(cols / 64) * (128 + 12288);
}

cudaError_t launch_grouped_gemm_tc(int dtype, int nt, bool dual, const CUtensorMap& a0, const CUtensorMap& a1,
                                   const CUtensorMap& b, const GemmParams& p, int grid, cudaStream_t st);
cudaError_t launch_grouped_gemm_tc_mc2(int dtype, bool dual, const CUtensorMap& a0h, const CUtensorMap& a1h,
                                       const CUtensorMap& b, const GemmParams& p, int grid, cudaStream_t st);
cudaError_t launch_grouped_gemm_simt(int dtype, const void* arena, size_t slot_elems, size_t offA0, size_t offA1,
                                     const void* B, int ldb, const GemmParams& p, bool dual, cudaStream_t st);
// fused expert FFN (decode regime): gate/up + SwiGLU phase on the first `up_ctas` CTAs, grid barrier (gbar: 2 ints, zero
// initialised), down phase on all `grid` CTAs.  `dn.early_a` must be 1 (its weights stream before the barrier).
cudaError_t launch_fused_ffn(int dtype, int nt, const CUtensorMap& gate, const CUtensorMap& upm, const CUtensorMap& b_up,
                             const CUtensorMap& down, const CUtensorMap& b_down, const GemmParams& up, const GemmParams& dn,
                             int grid, int up_ctas, int* gbar, cudaStream_t st);
// fp32 experts (dtype int 1): CUDA-core fp32 FMA kernel, f32_path.cu.  Offsets/slot sizes in fp32 elements.
cudaError_t launch_grouped_gemm_f32(const void* arena, size_t slot_elems, size_t offA0, size_t offA1, const void* B,
                                    int ldb, const GemmParams& p, bool dual, int num_sms, cudaStream_t st);

// ---- expert-parallel dispatch helpers (ep.cu) ----------------------------------------------
struct EpParams {
  int nranks, rank, E, H, cap;      // cap = rows per peer in the fixed-capacity exchange buffers
  int inline_counts;                // 1: buffers are [nranks][cap+1][H]; the extra last row carries counts[E] (int32)
  const int* offsets;               // in: routing offsets[E+1] (pack) ; out: regrouped offsets (regroup)
  int* offsets_rw;                  // same buffer, writable (regroup)
  int* offsets_src;                 // [E+1] source-side copy kept for unpack
  int* send_counts;                 // [E] this rank's per-expert row counts
  const int* recv_counts;           // [nranks][E] all ranks' counts
  void* xp;                         // workspace rows (pack: in, regroup: out)
  void* send_rows;                  // [nranks][cap][H]
  const void* recv_rows;            // [nranks][cap][H]
  void* ret_rows;                   // [nranks][cap][H]
  const void* back_rows;            // [nranks][cap][H]
  float* y;                         // fp32 expert outputs
  int* dest_of;                     // [nranks*cap] workspace row of each received slot (-1: empty)
  float* y_zero;
  size_t y_zero_elems;
  // ---- peer-to-peer mode (p2p = 1): rows are stored straight into the peers' buffers over NVLink and completion is
  // signalled with release/acquire flags in peer memory; no collective library call in the layer.
  int p2p;
  void* peer_recv[16];        // peer r's receive area  [nranks][cap+1][H]   (peer-mapped via CUDA IPC)
  void* peer_back[16];        // peer r's return area   [nranks][cap+1][H]
  int* peer_recv_flag[16];    // peer r's recv_flag[nranks]
  int* peer_back_flag[16];    // peer r's back_flag[nranks]
  int* local_recv_flag;       // this rank's recv_flag[nranks]
  int* local_back_flag;
  int* epoch;                 // local: [0] dispatches issued, [1] returns issued
  int* done_ctr;              // local: [0] CTAs finished in dispatch kernel, [1] in return kernel
  // ---- direct mode (direct = 1): receive slots are [nranks][cap] rows (no counts row); every slot carries a tag; the owners'
  // fp32 outputs are read in place by the source ranks' combine kernels (peer loads), no return kernel
  int direct;
  int region_rows;            // direct mode: rows per expert region = nranks*cap
  int* peer_cnt[16];          // peer r's row counters cnt[E/nranks] (direct mode: sources claim rows with remote atomics)
  int* local_cnt;
  float* peer_y[16];          // peer r's fp32 outputs y[nranks*cap][H]
  float* local_y;
};
cudaError_t launch_ep_pack(const EpParams& p, int max_rows, cudaStream_t st);
cudaError_t launch_ep_regroup(const EpParams& p, cudaStream_t st);
cudaError_t launch_ep_ungroup(const EpParams& p, int dtype, cudaStream_t st);
cudaError_t launch_ep_unpack(const EpParams& p, int dtype, int max_rows, cudaStream_t st);

// ---- routing / permutation / combine (route.cu) -----------------------------------------
struct RouteParams {
  // inputs
  const void* x;             // [T,H] model dtype
  const void* gate_w;        // [E,H] router weight (model dtype for Mixtral, any of bf16/f16/f32 otherwise) or null
  const void* logits;        // optional precomputed router logits/scores [T,E]
  int logits_dtype;          // DT_* of `logits`
  int logits_are_scores;     // 1: `logits` already holds fp32 softmax scores (DeepSeek parity tests)
  int gate_dtype;            // DT_* of gate_w
  int T, H, E, k;
  int dtype;                 // model dtype
  int router;                // ROUTER_*
  int n_group, topk_group, norm_topk_prob;
  float routed_scaling_factor;
  const float* gate_bias;    // ROUTER_DEEPSEEK_V3: the layer's e_score_correction_bias [E] fp32 (required)
  int seq_len, expert_capacity;   // Switch only
  // outputs (workspace)
  float* scores;             // [T,E] fp32 softmax probabilities (optional, may be null)
  void* logits_out;          // [T,E] router logits in their natural dtype (optional)
  int* topk_idx;             // [T,k]
  float* topk_w;             // [T,k]
  int* row_of;               // [T,k] permuted row of (t,j); -1 if dropped
  int* perm_token;           // [T*k] source token of each permuted row
  int* counts;               // [E]
  int* offsets;              // [E+1]
  int* chunk_counts;         // [ceil(T/32), E]
  void* xp;                  // [T*k, H] gathered activations
  float* y_zero;             // optional fp32 buffer to clear (split-K accumulator), y_zero_elems floats
  size_t y_zero_elems;
  int* ticket;               // small-T path: CTA arrival counter (0 between launches)
  int* err_flag;             // sticky device error word (bit0: a mask row had more than k experts, bit1: an input-permutation
                             // entry >= H)
  const uint16_t* input_perm;  // null, or the layer's [E][H] table (b2m_set_input_perm): column c of a gathered row of expert e
                               // is x[t][input_perm[e * H + c]]
  int rows_by_gate;          // with offsets_early: the last gate/top-k CTA also publishes row_of / perm_token, and the permute
                             // kernel only copies rows (no redundant ranking in each of its CTAs)
  int offsets_early;         // small-T path: the last gate/top-k CTA already publishes counts/offsets (so the gate/up GEMM can
                             // start fetching weights while the permute kernel is still gathering rows)
  int pdl_edge;              // ep_fused: launch with a programmatic edge behind the previous layer's combine (the kernel waits before any access)
  int ep_fused;              // ep_dispatch in direct mode with T <= #SMs: the gate/top-k kernel also permutes + dispatches (one launch)
  int* ready;                // ep_fused: word the last gate/top-k CTA releases (value = local dispatch epoch + 1) once the row maps are out
  int ep_dispatch;           // 1 (T <= 256 only): gathered rows go straight to the owning ranks' buffers (ep)
  EpParams ep;
  unsigned long long* tl;    // optional timeline slots: [0] gate/top-k start, [1] its end, [2] permute start, [3] permute end
  int scale_rows;            // Llama 4: the gathered row of pair i is round(x[t] * topk_w[i]) (written by this routing call)
  int logits_model_dtype;    // the router's logits are rounded to the model dtype (its gate is an nn.Linear in that dtype)
};
cudaError_t launch_route(const RouteParams& p, cudaStream_t st);
// look-ahead: top-k of the NEXT layer's router (p.gate_w = its weight; DeepSeek-V3: p.gate_bias = its bias) on this layer's
// input p.x -> counts_out[E] += 1 per selected (token, expert); counts_out must be zero.  T <= 256.
cudaError_t launch_lookahead_counts(const RouteParams& p, int* counts_out, cudaStream_t st);
// routing from a caller-supplied dense mask (reference compat: ExpertDispatcher::SetInputs + per-expert gather,
// core/parallel/expert_dispatcher.h:66-70, expert_dispatcher.cpp:274-285)
cudaError_t launch_route_from_mask(const RouteParams& p, const uint8_t* mask /*[T,E]*/, cudaStream_t st);

struct CombineParams {
  const float* y;          // [rows, H] fp32 expert outputs (permuted row order)
  const float* y_shared;   // [T, H] fp32 shared-expert output or null
  const void* x;           // [T,H] (Switch pass-through; the COMBINE_QWEN_GATE input) or null
  const int* topk_idx;     // [T,k]
  const float* topk_w;     // [T,k]
  const int* row_of;       // [T,k]
  void* out;               // [T,H] model dtype
  int T, H, k, dtype, mode;
  int ep_collect;          // 1: expert outputs are read from the peer-written return area (model dtype rows)
  int ep_early;            // direct mode: programmatic edge behind the down GEMM, no grid-completion wait (flags guard the data)
  EpParams ep;
  unsigned long long* tl;  // optional timeline slots: [0] start, [1] owners' flags seen, [2] end
  const uint16_t* shared_gate;  // Qwen2-MoE: [T] model-dtype sigmoid(shared_expert_gate(x)) scaling y_shared (COMBINE_QWEN_GATE)
  const void* shared_gate_w;    // COMBINE_QWEN_GATE: the layer's [H] shared_expert_gate.weight (model dtype)
  int unweighted;               // Llama 4 (COMBINE_LLAMA4, or COMBINE_FP32): expert outputs summed without weights, + y_shared
};
cudaError_t launch_combine(const CombineParams& p, cudaStream_t st);
cudaError_t launch_combine_f32(const CombineParams& p, cudaStream_t st);

// ---- device-side activation tracer / predictor (tracer.cu; SURVEY §8f N1) ----------------------------------------------
struct TraceParams {
  int L, E, k;
  int layer;
  int seq_len;             // tokens per sequence in this call (rows b*seq_len .. of the routing result belong to sequence b)
  int seq_slot0;           // first sequence slot of this call
  int capacity, persistent;
  const int* topk_idx;     // [num_seqs*seq_len, k] routing result of the call (workspace)
  float* seq;              // [max_seqs][L][E] per-sequence trace matrices
  float* lib;              // [capacity][L][E] trace library
  int* access;             // [capacity]
  float* pred;             // [max_seqs][L][E] decayed prediction of the last call
  float* hint;             // [L][E] sum of the predictions of the call's sequences (zeroed by the caller)
  int* winner;             // [max_seqs] library entry chosen for each sequence
};
cudaError_t launch_trace_update_predict(const TraceParams& p, int num_seqs, cudaStream_t st);
cudaError_t launch_trace_finish(const TraceParams& p, int seq_slot, cudaStream_t st);

// fp32 [rows,H] -> model dtype [rows,H] (compat path: per-expert outputs handed back to Python)
cudaError_t launch_cast_rows(const float* y, void* out, size_t n, int dtype, cudaStream_t st);

}  // namespace b2m
