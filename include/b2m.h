/* b2m.h -- C ABI of the H100-native MoE expert dispatch/offload engine (libb2m.so).
 *
 * Drop-in boundary for the ONE hot path of EfficientMoE/MoE-Infinity named in BASELINE.json:
 * router softmax/top-k -> token permute -> grouped expert GEMM -> unpermute/combine, plus the HBM expert
 * cache and prefetch scheduler that stage expert weights from pinned host DRAM.
 *
 * The reference binds this path through pybind11 (core/python/py_archer_prefetch.cpp:10-92, module
 * `moe_infinity.ops.prefetch.prefetch_op`): classes `expert_dispatcher` (:84-92) and `prefetch_handle`
 * (:11-80).  Every entry point below names the reference interface it replaces.  All pointers are plain
 * device/host addresses; no C++/torch types cross the boundary.  Every function returns 0 on success or a
 * negative B2M_E* code; b2m_last_error() gives the message.  Nothing aborts the process
 * (reference: DLOG_FATAL -> abort(), core/base/logging.cc:172-174).
 *
 * Threading: one caller thread per context, non re-entrant (same as the reference's ExpertDispatcher,
 * which shares hidden_states_/pending_ across a dispatch).  Hot calls are asynchronous on the caller's CUDA
 * stream; when every expert of the model is HBM resident no call synchronises with the host.
 */
#ifndef B2M_H_
#define B2M_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2M_VERSION 1

/* status codes */
#define B2M_OK 0
#define B2M_EINVAL (-1)    /* bad argument */
#define B2M_ECUDA (-2)     /* CUDA runtime/driver error (message has the CUDA string) */
#define B2M_ENOMEM (-3)    /* no evictable HBM slot / allocation failure */
#define B2M_ESTATE (-4)    /* call not valid in this state (e.g. expert not registered) */
#define B2M_EUNSUPPORTED (-5)
#define B2M_EIO (-6)       /* disk tier: open/read failed or a file is shorter than its index entry */

/* dtype ints == reference core/parallel/expert_module.h:20-23 */
#define B2M_DTYPE_BF16 0
#define B2M_DTYPE_F32 1
#define B2M_DTYPE_F16 2
#define B2M_DTYPE_FP8_E4M3 3 /* not supported as a model dtype (B2M_EUNSUPPORTED): fp8 experts are a weight format of a
                                bf16 context, B2M_WEIGHTS_FP8_E4M3_B128 of b2m_ctx_create_ex */

/* expert-type ints == reference core/parallel/expert_module.h:13-18 */
#define B2M_EXPERT_SWITCH_DENSE_ACT_DENSE 0       /* wi, wo; ReLU            (expert_module.cpp:24-35)  */
#define B2M_EXPERT_SWITCH_DENSE_GATED_ACT_DENSE 1 /* wi_0, wi_1, wo; GELU    (:54-59)                   */
#define B2M_EXPERT_NLLB_MOE_DENSE_ACT_DENSE 2     /* fc1, fc1_bias, fc2, fc2_bias; ReLU (:79-129)        */
#define B2M_EXPERT_FSGPT_MOE_DENSE_ACT_DENSE 3    /* fc1, fc1_bias, fc2, fc2_bias; ReLU (:79-129)        */
#define B2M_EXPERT_MIXTRAL_MOE_DENSE_ACT_DENSE 4  /* w1, w2, w3; SiLU        (:147-175)                 */
#define B2M_EXPERT_DEEPSEEK_MOE_DENSE_ACT_DENSE 5 /* gate, up, down; SiLU    (:193-203)                 */

/* router kinds: which reference routing function the fused top-k kernel restates */
#define B2M_ROUTER_MIXTRAL 0         /* moe_infinity/models/mixtral.py:48-54                              */
#define B2M_ROUTER_DEEPSEEK_GREEDY 1 /* models/modeling_deepseek/modeling_deepseek.py:467-483,508-512     */
#define B2M_ROUTER_DEEPSEEK_GROUP 2  /* modeling_deepseek.py:484-505 (group_limited_greedy)               */
#define B2M_ROUTER_SWITCH_TOP1 3     /* HF 4.x SwitchTransformersTop1Router (switch_transformers.py:76)   */
/* DeepSeek-V3 MoEGate, topk_method "noaux_tc", scoring_func "sigmoid"
 * (models/modeling_deepseek_v3/modeling_deepseek.py:466-527, built by models/deepseek.py:23-27).  Per token:
 *   1. s = sigmoid(fp32 logits)                           (no softmax; 1 / (1 + exp(-x)) with an IEEE division)
 *   2. choice[e] = s[e] + bias[e]                          bias = the layer's fp32 [E] e_score_correction_bias (b2m_set_gate_bias)
 *   3. group score = top1 + top2 of the group's choices    (n_group groups of E / n_group experts); the topk_group best
 *                                                          groups are kept
 *   4. choices outside the kept groups become 0.0          (masked_fill(~mask, 0.0), not -inf: with negative biases a
 *                                                          masked expert can win)
 *   5. top_k experts by choice; their weights are the UNBIASED s
 *   6. if top_k > 1 and norm_topk_prob: w /= (sum of the k weights, in selection order) + 1e-20; then ALWAYS
 *      w *= routed_scaling_factor
 * Ties at every stage (groups and experts) go to the lowest index.  Limits (b2m_ctx_create_ex, B2M_EINVAL otherwise):
 * 1 <= n_group <= 32, E % n_group == 0, E / n_group >= 2, 1 <= topk_group <= n_group.
 * router_in_kind: 0 = fused fp32 gate (B2M_WS_LOGITS holds fp32 logits), 1 = logits of any supported dtype (sigmoid
 * applied here), 2 = fp32 sigmoid scores used as given.  B2M_WS_SCORES holds the unbiased sigmoid scores.  A routing call
 * on a layer whose bias was never set returns B2M_ESTATE (whatever router_in_kind).  The combine is the DeepSeek one
 * (models/deepseek.py:115-137). */
#define B2M_ROUTER_DEEPSEEK_V3 4
/* Qwen2-MoE / Qwen3-MoE router (transformers Qwen2MoeTopKRouter, Qwen3MoeTopKRouter: identical).  Per token:
 *   1. logits in the model dtype                           (F.linear in bf16/f16: the fp32 dot is rounded to the model dtype)
 *   2. p = fp32 softmax of the logits
 *   3. top_k experts by p                                  ties go to the lowest index
 *   4. if norm_topk_prob: w /= (sum of the k weights, in selection order), for every k (k = 1 gives 1.0); no epsilon
 *   5. the weights stay fp32 and are never scaled
 * Accepted by b2m_ctx_create_ex (B2M_EINVAL with a message otherwise) only with expert_type
 * B2M_EXPERT_DEEPSEEK_MOE_DENSE_ACT_DENSE (gate|up|down, the HF tensor order), dtype bf16 or f16, n_group = topk_group = 1
 * and routed_scaling_factor = 1.0; every weight format works with its own restrictions.  The router weight is an nn.Linear
 * of the model, so gate_dtype is normally the model dtype; B2M_WS_LOGITS holds model-dtype logits, as for Mixtral.
 * Combine (Qwen2MoeExperts + Qwen2MoeSparseMoeBlock), per element, experts in ascending id (index_add_ order):
 *   acc = 0;  acc = round(acc + round(round(y) * w))       y: fp32 expert output, w: fp32 weight, round: to the model dtype
 * shared_inter > 0 makes it a Qwen2-MoE layer with a GATED shared expert (b2m_set_shared_gate):
 *   g = round(sigmoid(round(x . shared_expert_gate)))       (B2M_WS_SHARED_GATE; the sigmoid is PyTorch's CUDA formula)
 *   out = round(acc + round(g * round(s)))                  s: fp32 shared-expert output (B2M_WS_Y_SHARED)
 * With B2M_NUMERICS_FP32: acc += w * y, then acc += g * s, rounded once.  A forward or combine of a layer with shared experts
 * and no gate returns B2M_ESTATE.  The expert-parallel entry points return B2M_EUNSUPPORTED on such a context. */
#define B2M_ROUTER_QWEN_MOE 5
/* Llama 4 router (transformers Llama4Router + Llama4TextMoe).  Per token:
 *   1. logits in the model dtype                           (F.linear in bf16/f16: the fp32 dot is rounded to the model dtype)
 *   2. top_k experts by the logits themselves              ties go to the lowest index (not by sigmoid values: two logits
 *                                                          can share one fp32 sigmoid)
 *   3. w = round(sigmoid(logit)) for each chosen expert    fp32 sigmoid (PyTorch's CUDA formula), rounded to the model dtype
 *                                                          and stored as fp32 in B2M_WS_TOPK_W; B2M_WS_SCORES holds the
 *                                                          unrounded fp32 sigmoid of every logit
 *   4. the input row of (t, e) is round(x[t] * w)          elementwise: the routing weight scales the expert's INPUT, so
 *                                                          B2M_WS_XP rows hold scaled activations
 * Accepted by b2m_ctx_create_ex (B2M_EINVAL with a message naming llama4 otherwise) only with expert_type
 * B2M_EXPERT_DEEPSEEK_MOE_DENSE_ACT_DENSE (gate|up|down), dtype bf16 or f16, n_group = topk_group = 1,
 * routed_scaling_factor = 1.0, norm_topk_prob = 0 and shared_inter > 0 (every Llama 4 MoE layer has its ungated shared
 * expert); every weight format works with its own restrictions.  gate_dtype is normally the model dtype; B2M_WS_LOGITS
 * holds model-dtype logits.
 * Combine (Llama4TextMoe.forward: routed_out.reshape(k, T, H).sum(0), then shared_expert(x).add_), per element:
 *   r = round(sum of round(y_e) over the chosen experts)   fp32 sum in ascending expert id, rounded ONCE
 *   out = round(r + round(s))                               s: fp32 shared-expert output (B2M_WS_Y_SHARED)
 * With B2M_NUMERICS_FP32: out = round(sum of y_e + s).  The weights are not applied after the experts.
 * router_in_kind 2 (scores given), b2m_set_input_perm and the expert-parallel entry points return B2M_EUNSUPPORTED on
 * such a context.  b2m_route_from_mask keeps weight 1: its gathered rows are the unscaled inputs. */
#define B2M_ROUTER_LLAMA4 6

/* numerics of epilogue + combine */
#define B2M_NUMERICS_REFERENCE 0 /* replay the reference's per-ATen-op rounding to the model dtype */
#define B2M_NUMERICS_FP32 1      /* keep fp32 until the single final rounding (fewer roundings)    */

/* on-demand cache accounting */
#define B2M_CACHE_REFERENCE 0 /* byte budget charged exactly like cache_sizes_ in core/parallel/expert_dispatcher.cpp:228,257,266:
                                 every dispatched expert (hit or miss) costs one expert, an eviction refunds one, a miss evicts
                                 exactly one victim iff the budget is used up */
#define B2M_CACHE_SLOTS 1     /* evict only when no physical HBM slot is free (hits are not charged) */
#define B2M_CACHE_ACTIVATION_AWARE 2 /* the "activation-aware expert cache" the reference specifies but never wires in
                                 (moe_infinity/memory/expert_priority_score.py:84-172: layer-distance decay x activation
                                 frequency; expert_cache.py:95-167): the victim is the resident expert with the largest
                                 EXPECTED time to its next use = layers until its layer runs again (decode visits layers in
                                 order) + L * (1/f - 1), f = moving average of "activated in a step" (cfg.freq_alpha).
                                 Physical slots are the budget.  Measured against B2M_CACHE_REFERENCE by tools/policy_sim.py */

typedef struct b2m_ctx b2m_ctx;

typedef struct b2m_config {
  int32_t struct_size;      /* = sizeof(b2m_config) */
  int32_t device;           /* CUDA device ordinal */
  int32_t num_layers;       /* absolute layer count L (DeepSeek counts its dense layer 0 too;
                               reference: expert_dispatcher(E, L, ...) model_offload.py:471-477) */
  int32_t num_experts;      /* routed experts per layer E (<= 256) */
  int32_t hidden;           /* H (multiple of 8) */
  int32_t inter;            /* I of a routed expert (multiple of 8) */
  int32_t top_k;            /* <= 8 */
  int32_t dtype;            /* B2M_DTYPE_BF16 | B2M_DTYPE_F16 */
  int32_t expert_type;      /* B2M_EXPERT_* */
  int32_t router;           /* B2M_ROUTER_* */
  int32_t numerics;         /* B2M_NUMERICS_* */
  int32_t max_tokens;       /* workspace capacity: largest T of one forward call */
  int32_t num_slots;        /* HBM expert slots; 0 = derive from device_memory_ratio */
  int32_t shared_inter;     /* DeepSeek shared experts: I_shared = moe_intermediate * n_shared; 0 = none */
  int32_t n_group;          /* DeepSeek group-limited routing */
  int32_t topk_group;
  int32_t norm_topk_prob;
  int32_t expert_capacity;  /* Switch */
  float routed_scaling_factor;
  int32_t gate_dtype;       /* dtype of the router weight handed to b2m_set_gate */
  double device_memory_ratio; /* reference: prefetch_handle(prefix, ratio) / DeviceMemoryPool::SetMemoryRatio
                                 (core/memory/memory_pool.cpp:150-158): slots = ratio * total HBM / expert bytes */
  int32_t max_inflight_prefetch; /* concurrent prefetch copies on the side stream (default 2) */
  int32_t h2d_chunk_bytes;  /* H2D copy granularity in bytes (0 = whole expert in one cudaMemcpyAsync) */
  int32_t gemm_impl;        /* 0 = wgmma tensor cores (product); 1 = CUDA-core cross-check kernel (bring-up only);
                               2 = wgmma tensor cores reading the bf16 slots only.
                               With 0, the decode GEMMs (<= 64-token tiles) of an all-resident, single-rank bf16 context read the
                               routed experts from a lossless 12-bit packed copy beside the bf16 slots (0.76 of their bytes,
                               csrc/weight_pack.cuh; results are bit-identical), allocated by the first eager forward that packs if 2 GiB of
                               device memory stay free.  A slot is packed by the second eager forward of its layer after
                               b2m_make_resident(flags & 2), b2m_expert_dev_ptr or a host->device staging (the first one runs as
                               without the copy); forwards captured into a graph before that read it as bf16.  2 never allocates the copy (frees that HBM). */
  int32_t cache_policy;     /* B2M_CACHE_* : on-demand budget accounting */
  int32_t lookahead_prefetch; /* 1 | 2 (offload mode, T <= 256): every routing call also applies the NEXT layer's router weight
                               (b2m_set_gate) to this layer's input and reads the predicted expert counts back with this
                               layer's own counts (same synchronisation); predicted experts that are not resident are staged
                               on the prefetch stream while this layer computes -- the router-logit driven prefetch of the
                               north star; replaces expert_predictor.predict + prefetch_experts (expert_prefetcher.py:42-59)
                               for callers that do not supply their own hints.  1 = only from layers that staged nothing
                               on demand (the link is idle) and only while the scheduler's own measured accuracy (prefetched
                               experts used before eviction) stays >= 90 % -- otherwise it suspends itself for 256 layer calls
                               and probes again; 2 = always (costs bandwidth when the link is saturated) */
  float freq_alpha;         /* B2M_CACHE_ACTIVATION_AWARE: weight of the newest step in the activation average (0 = 0.25) */
} b2m_config;

/* cache / traffic counters; columns mirror the reference's per-node counters exported by get_hit_rate
 * (core/model/model_topology.cpp:253-263, archer_prefetch_handle.cpp:281-297) */
typedef struct b2m_stats {
  uint64_t dispatches;        /* expert invocations (layer,expert with >=1 token) seen by the cache */
  uint64_t hits;              /* resident at dispatch */
  uint64_t misses;            /* fetched on demand */
  uint64_t prefetch_issued;
  uint64_t prefetch_useful;   /* prefetched expert later dispatched before eviction */
  uint64_t evictions;
  uint64_t h2d_bytes;
  uint64_t host_syncs;        /* stream synchronisations forced by on-demand routing readback */
  uint64_t kernel_launches;   /* kernels of this library launched so far */
  uint64_t resident;          /* experts currently in HBM */
  uint64_t slots;             /* total HBM slots */
  uint64_t slot_bytes;
} b2m_stats;

const char* b2m_last_error(const b2m_ctx* ctx); /* ctx may be NULL: last error of a failed b2m_ctx_create */
int b2m_version(void);

/* replaces: prefetch_handle(prefix, ratio) + expert_dispatcher(E, L, dtype, expert_type, num_threads)
 * construction (py_archer_prefetch.cpp:12,85; core/prefetch/archer_prefetch_handle.cpp:18-64;
 * core/parallel/expert_dispatcher.cpp:22-109) */
int b2m_ctx_create(const b2m_config* cfg, b2m_ctx** out);
int b2m_ctx_destroy(b2m_ctx* ctx);

/* Storage format of the routed experts' weights (b2m_ctx_create_ex) */
#define B2M_WEIGHTS_MODEL_DTYPE 0   /* cfg.dtype, as b2m_ctx_create */
#define B2M_WEIGHTS_FP8_E4M3_B128 1 /* FP8 E4M3 matrices with one fp32 scale per 128x128 block (DeepSeek-V3 / Qwen3-MoE FP8
                                       checkpoints).  Each routed matrix (nn.Linear [out,in], row-major) is float8_e4m3fn with
                                       a row-major fp32 scale grid s[out/128][in/128]; the scale multiplies.  The experts
                                       compute exactly what the bf16 engine computes on
                                         W[r][c] = bf16(fp32(w_q[r][c]) * s[r/128][c/128])
                                       -- one fp32 multiply rounded to nearest-even, then one rounding to bf16 (torch:
                                       `(w_q.float() * s_expanded).to(torch.bfloat16)`); the GEMMs dequantise inside the
                                       kernel, so results are bit-identical to a bf16 context holding those W.
                                       Expert blob (b2m_register_expert, b2m_expert_dev_ptr): the three e4m3 matrices in the
                                       model's tensor order (Mixtral w1|w2|w3, DeepSeek gate|up|down), then their three scale
                                       grids in the same order, zero-padded to a multiple of 16 bytes (b2m_stats.slot_bytes).
                                       Activations, outputs, workspaces and the router stay bf16; DeepSeek shared experts
                                       stay bf16 (b2m_register_shared is unchanged).  Restrictions, each refused by
                                       b2m_ctx_create_ex with B2M_EUNSUPPORTED and a message: cfg.dtype bf16; expert types
                                       Mixtral (4) and DeepSeek (5); hidden and inter multiples of 128; gemm_impl 0 or 2 (the
                                       12-bit packed copy of gemm_impl 0 is never made).  The expert-parallel entry points
                                       return B2M_EUNSUPPORTED on such a context. */
/* (2 and 3 are not weight formats: B2M_EINVAL) */
#define B2M_WEIGHTS_INT4_G128 4     /* 4-bit integer matrices with a bf16 scale and a 4-bit zero point per 128 inputs (W4A16,
                                       asymmetric group quantisation).  Each routed matrix (nn.Linear [out,in], row-major) is
                                       codes q[r][c] in 0..15, scales s[r][c/128] (bf16) and zero points z[r][c/128] in 0..15.
                                       The experts compute exactly what the bf16 engine computes on
                                         W[r][c] = bf16(s[r][c/128] * (q[r][c] - z[r][c/128]))
                                       -- the product is exact in fp32 and is rounded once to nearest-even, subnormals kept
                                       (torch: `(s_expanded.float() * (q.float() - z_expanded.float())).to(torch.bfloat16)`);
                                       the GEMMs dequantise inside the kernel, so results are bit-identical to a bf16 context
                                       holding those W.
                                       Expert blob (b2m_register_expert, b2m_expert_dev_ptr), 3*H*I/2 + 3*(H*I/128)*4 bytes,
                                       no padding: (1) the three code matrices in the model's tensor order (Mixtral w1|w2|w3,
                                       DeepSeek gate|up|down), each [rows][cols/2] bytes, byte c/2 holding column c in its low
                                       nibble (c even) or its high nibble (c odd); (2) their three group grids in the same
                                       order, one uint32 per (row r, group g = c/128): bits 0..15 the bf16 bits of s, bits
                                       16..19 z, the other bits ignored; the grid is tile-major, the word of (r, g) at index
                                       ((r/128) * (cols/128) + g) * 128 + r%128.  Activations, outputs, workspaces and the
                                       router stay bf16; DeepSeek shared experts stay bf16.  Restrictions (B2M_EUNSUPPORTED
                                       with a message) and the expert-parallel refusal: as B2M_WEIGHTS_FP8_E4M3_B128. */
/* (5 is not a weight format: B2M_EINVAL) */
#define B2M_WEIGHTS_INT4_G128_F16 6 /* B2M_WEIGHTS_INT4_G128 with fp16 scales and f16 activations: the format of AWQ and GPTQ
                                       4-bit checkpoints (group size 128).  Each routed matrix is codes q[r][c] in 0..15,
                                       scales s[r][c/128] (fp16) and zero points z[r][c/128] in 0..15.  The experts compute
                                       exactly what the f16 engine computes on
                                         W[r][c] = f16(s[r][c/128] * (q[r][c] - z[r][c/128]))
                                       -- the product is exact in fp32 and is rounded once to nearest-even, subnormals kept,
                                       overflow to +-Inf (torch: `(s_expanded.float() * (q.float() -
                                       z_expanded.float())).to(torch.float16)`); this is the value AWQ's and GPTQ's own
                                       dequantisation produces.  Expert blob: byte for byte the layout of
                                       B2M_WEIGHTS_INT4_G128 (same size and offsets), except that bits 0..15 of each group word
                                       are the fp16 bits of s.  Activations, outputs, workspaces and the router are f16;
                                       DeepSeek shared experts stay f16.  Restrictions, each refused by b2m_ctx_create_ex with
                                       B2M_EUNSUPPORTED and a message: cfg.dtype f16; expert types Mixtral (4) and DeepSeek
                                       (5); hidden and inter multiples of 128; gemm_impl 0 or 2.  The expert-parallel entry
                                       points return B2M_EUNSUPPORTED on such a context. */
#define B2M_WEIGHTS_FP8_E4M3_ROW 7  /* FP8 E4M3 matrices with one fp32 scale per output channel (Llama 4 Maverick FP8 and other
                                       fbgemm FP8 checkpoints; a per-tensor scale is this format with the scalar repeated).
                                       Each routed matrix (nn.Linear [out,in], row-major) is float8_e4m3fn with an fp32 scale
                                       vector s[out]; the scale multiplies.  The experts compute exactly what the bf16 engine
                                       computes on
                                         W[r][c] = bf16(fp32(w_q[r][c]) * s[r])
                                       -- one fp32 multiply rounded to nearest-even, then one rounding to bf16 (torch:
                                       `(w_q.float() * s[:, None]).to(torch.bfloat16)`); the GEMMs dequantise inside the
                                       kernel, so results are bit-identical to a bf16 context holding those W.
                                       Expert blob, 3*H*I + 4*(2*I + H) bytes rounded up to a multiple of 16: the three e4m3
                                       matrices in the model's tensor order (Mixtral w1|w2|w3, DeepSeek gate|up|down), then
                                       their three scale vectors in the same order (lengths I, H, I for Mixtral; I, I, H for
                                       gate|up|down), zero-padded.  Activations, outputs, workspaces, the router and the shared
                                       experts stay bf16.  Restrictions (B2M_EUNSUPPORTED with a message) and the
                                       expert-parallel refusal: as B2M_WEIGHTS_FP8_E4M3_B128. */
/* b2m_ctx_create with the routed experts stored in `weight_format` (B2M_WEIGHTS_*; any other value: B2M_EINVAL) */
int b2m_ctx_create_ex(const b2m_config* cfg, int weight_format, b2m_ctx** out);
/* B2M_WEIGHTS_INT4_G128_F16 only: act-order GPTQ (desc_act).  `dev_perm` is a borrowed device table uint16 [E][H] (like the
 * gate weight): column j of every row the routing kernels gather for expert e is x[t][dev_perm[e * H + j]], so expert e's
 * gate/up matrices are stored with their input columns in that order (W[:, P], whose 128-column groups are then contiguous;
 * the down projection's permutation is applied to the stored matrices at load time and needs no table).  NULL returns the
 * layer to natural order.  The table is read by every routing call of the layer (b2m_moe_forward, b2m_route,
 * b2m_route_from_mask); a captured graph keeps the pointer it was captured with and reads the table's contents at replay.
 * B2M_WS_XP and B2M_WS_HMID rows of such a layer hold permuted activations.  An entry >= H reads as 0 and sets a bit of the
 * sticky device error word (B2M_EINVAL from b2m_check_errors / b2m_expert_outputs); nothing faults.  B2M_EUNSUPPORTED on a
 * context of any other weight format, B2M_EINVAL for a layer out of range. */
int b2m_set_input_perm(b2m_ctx* ctx, int layer, const uint16_t* dev_perm);

/* replaces: prefetch_handle.offload/register + set_topology for an expert stage + expert_dispatcher.register_expert
 * (core/parallel/expert_dispatcher.cpp:160-173; blob layout core/model/model_topology.cpp:429-431:
 * tensors concatenated in tensor_ids order -- Mixtral w1|w2|w3, DeepSeek gate|up|down, Switch wi|wo, gated Switch
 * wi_0|wi_1|wo, NLLB/FSGPT fc1|fc1_bias|fc2|fc2_bias -- packed without the reference's 4 KiB padding between tensors).
 * `host_blob` must stay valid (and should be pinned, see b2m_host_pin) for the life of the context; may be NULL
 * for an expert that only ever lives in HBM (then it is never evicted). */
int b2m_register_expert(b2m_ctx* ctx, int layer, int expert, const void* host_blob, size_t bytes);
int b2m_register_shared(b2m_ctx* ctx, int layer, const void* host_blob, size_t bytes); /* deepseek.py:39-45 */
/* router weight [E,H] on the device, dtype cfg.gate_dtype (mixtral.py:30 `self.gate`; MoEGate.weight) */
int b2m_set_gate(b2m_ctx* ctx, int layer, const void* dev_gate_weight);
/* B2M_ROUTER_DEEPSEEK_V3 only: the layer's e_score_correction_bias, fp32 [E] on the device (MoEGate.e_score_correction_bias,
 * modeling_deepseek.py:455-458).  Borrowed like the gate weight: it must stay valid, and is read by every routing call of
 * the layer (and by the look-ahead prediction made from the layer before it).  B2M_EINVAL for a layer out of range, a null
 * pointer, or a context whose router is not B2M_ROUTER_DEEPSEEK_V3. */
int b2m_set_gate_bias(b2m_ctx* ctx, int layer, const float* dev_bias);
/* B2M_ROUTER_QWEN_MOE with shared experts (Qwen2-MoE) only: the layer's shared_expert_gate.weight, [H] in the model dtype on
 * the device.  Borrowed like the gate weight: it must stay valid, and is read by every forward or combine of the layer (a
 * captured graph reads its contents at replay).  B2M_EINVAL for a layer out of range, a null pointer, a context whose router
 * is not B2M_ROUTER_QWEN_MOE, or a context without shared experts. */
int b2m_set_shared_gate(b2m_ctx* ctx, int layer, const void* dev_w);

/* replaces: HostMemoryPool / cudaHostAlloc per node (core/memory/memory_pool.cpp:29-83) */
int b2m_host_pin(b2m_ctx* ctx, void* host_ptr, size_t bytes);
int b2m_host_unpin(b2m_ctx* ctx, void* host_ptr);

/* replaces: Node::SetDevice(cuda) at init for resident experts (core/model/model_topology.cpp:53-136).
 * flags: 1 = pin in HBM (never evict), 2 = do not copy (caller fills the slot on the device, see b2m_expert_dev_ptr) */
int b2m_make_resident(b2m_ctx* ctx, int layer, int expert, int flags, void* stream);
int b2m_expert_dev_ptr(b2m_ctx* ctx, int layer, int expert, void** dev_ptr); /* NULL if not resident */
int b2m_shared_dev_ptr(b2m_ctx* ctx, int layer, void** dev_ptr);

/* THE hot call.  replaces Sync*MoeBlock.forward steps A-G (SURVEY §3.2): mixtral.py:46-101,
 * deepseek.py:53-136, switch_transformers.py:76-109 + expert_executor.dispatch_local (expert_executor.py:32-58)
 * + ExpertDispatcher fetch/exec/output threads (expert_dispatcher.cpp:191-450).
 *   x            [T,H] device, model dtype
 *   router_in    optional [T,E] device: precomputed router logits (router_in_kind=1, dtype router_in_dtype) or
 *                fp32 softmax scores (router_in_kind=2); NULL (kind 0) = compute the gate from b2m_set_gate weights
 *   seq_len      Switch only (capacity is per batch row); otherwise ignored
 *   out          [T,H] device, model dtype
 * Asynchronous on `stream` (a cudaStream_t).  Host-synchronises only when an activated expert is not resident. */
int b2m_moe_forward(b2m_ctx* ctx, int layer, const void* x, const void* router_in, int router_in_kind,
                    int router_in_dtype, int T, int seq_len, void* out, void* stream);

/* Staged entry points (same kernels; used by the reference-compat executor and by tests) */
int b2m_route(b2m_ctx* ctx, int layer, const void* x, const void* router_in, int router_in_kind, int router_in_dtype,
              int T, int seq_len, void* stream);
/* replaces ExpertDispatcher::SetInputs + per-expert boolean-mask gather (expert_dispatcher.h:66-70,
 * expert_dispatcher.cpp:274-285): routing taken from a dense uint8 mask [T,E].  Every weight is 1 (B2M_ROUTER_LLAMA4:
 * the gathered rows are the unscaled inputs) */
int b2m_route_from_mask(b2m_ctx* ctx, int layer, const void* x, const uint8_t* mask, int T, void* stream);
/* replaces EnqueueExpert*n + GPUFetchFunc/GPUExecFunc (expert_dispatcher.cpp:111-395) for the routed tokens
 * currently in the workspace: residency (on demand fetch + eviction) and both grouped GEMMs */
int b2m_run_experts(b2m_ctx* ctx, int layer, int T, void* stream);
/* same, restricted to phases: bit0 = residency + gate/up GEMM (K3), bit1 = down GEMM (K4); used by bench.py to
 * time the dominant kernel on its own stream with CUDA events */
int b2m_run_experts_ex(b2m_ctx* ctx, int layer, int T, int phases, void* stream);
int b2m_combine(b2m_ctx* ctx, int layer, const void* x, int T, void* out, void* stream);
/* replaces OutputFunc/Wait (expert_dispatcher.cpp:397-450): expert outputs in the model dtype, rows grouped by
 * ascending expert id, ascending token order inside an expert; `offsets_host` (E+1 ints) may be NULL */
int b2m_expert_outputs(b2m_ctx* ctx, int T, void* out_rows, int* offsets_host, void* stream);
/* synchronises `stream` and reports (then clears) the sticky device error word; B2M_EINVAL when a mask handed to
 * b2m_route_from_mask had a row with more than top_k experts (the reference would run them all: expert_dispatcher.cpp:274-285),
 * or when a table set with b2m_set_input_perm held an entry >= H */
int b2m_check_errors(b2m_ctx* ctx, void* stream);

/* workspace access for tests / EP plumbing (device pointers owned by the context) */
#define B2M_WS_TOPK_IDX 0   /* int32 [T,k]  (descending score; -1 = dropped) */
#define B2M_WS_TOPK_W 1     /* fp32  [T,k] */
#define B2M_WS_ROW_OF 2     /* int32 [T,k]  permuted row of (t,j) */
#define B2M_WS_PERM_TOKEN 3 /* int32 [T*k]  source token of each permuted row */
#define B2M_WS_COUNTS 4     /* int32 [E] */
#define B2M_WS_OFFSETS 5    /* int32 [E+1] */
#define B2M_WS_XP 6         /* dtype [T*k,H] (B2M_ROUTER_LLAMA4: round(x[t] * w) per row) */
#define B2M_WS_HMID 7       /* dtype [T*k,I] */
#define B2M_WS_Y 8          /* fp32  [T*k,H] */
#define B2M_WS_SCORES 9     /* fp32  [T,E] softmax probabilities (B2M_ROUTER_DEEPSEEK_V3: unbiased sigmoid scores;
                               B2M_ROUTER_LLAMA4: sigmoid of every logit, unrounded) */
#define B2M_WS_LOGITS 10    /* router logits computed by the fused gate: model dtype (Mixtral, Qwen, Llama 4) or fp32 */
#define B2M_WS_SHARED_GATE 11 /* dtype [T]   B2M_ROUTER_QWEN_MOE with shared experts: sigmoid(shared_expert_gate(x)), rounded
                                 (B2M_ESTATE on other contexts) */
#define B2M_WS_Y_SHARED 12  /* fp32  [T,H] shared-expert output (B2M_ESTATE on a context without shared experts) */
int b2m_ws_ptr(b2m_ctx* ctx, int which, void** dev_ptr);

/* replaces prefetch_handle.replace_cache_candidates(ids) (archer_prefetch_handle.cpp:195-205,
 * task_scheduler.h:66-79): new protected set; queued-but-not-started prefetches are dropped */
int b2m_replace_cache_candidates(b2m_ctx* ctx, int n, const int32_t* layer_expert_pairs);
/* replaces prefetch_handle.enqueue_prefetch(id, gpu) (archer_prefetch_handle.cpp:206-218,
 * task_scheduler.cpp:82-118,451-561): async H2D on the side stream, evict-to-fit, dedup */
int b2m_enqueue_prefetch(b2m_ctx* ctx, int layer, int expert);
/* one call = ExpertPrefetcher.prefetch_experts (moe_infinity/memory/expert_prefetcher.py:42-59):
 * pairs sorted by descending score by the caller or not -- sorted here; protected set replaced, then enqueued */
int b2m_prefetch_hint(b2m_ctx* ctx, int n, const int32_t* layer_expert_pairs, const float* scores);
int b2m_prefetch_pump(b2m_ctx* ctx);   /* retire finished copies, start queued ones (called by every hot call) */
int b2m_prefetch_drain(b2m_ctx* ctx);  /* block until the side stream is idle */
/* replaces expert_dispatcher.clear_expert_cache_counts() (expert_dispatcher.cpp:175-185) */
int b2m_clear_expert_cache_counts(b2m_ctx* ctx);
int b2m_is_resident(b2m_ctx* ctx, int layer, int expert);  /* 1/0, <0 error (get_node_device) */
int b2m_stats_get(b2m_ctx* ctx, b2m_stats* out);
/* activated experts of the last b2m_run_experts/b2m_moe_forward that had to read counts back (offload mode):
 * counts_host[E]; returns B2M_ESTATE if the last call ran sync-free */
int b2m_last_counts(b2m_ctx* ctx, int32_t* counts_host);
/* with cfg.lookahead_prefetch: per-expert token counts the NEXT layer's router predicted from the last call's input
 * (look_host[E]); B2M_ESTATE if the last call made no prediction */
int b2m_last_lookahead(b2m_ctx* ctx, int32_t* look_host);

/* ---- expert parallel (BASELINE config 5): one process per GPU, rank r owns experts [r*E/N, (r+1)*E/N).
 * The reference has no live collective (README.md:18; dead code modeling_deepseek.py:657-721); these helpers
 * replace its `.to(device)` token moves (expert_dispatcher.cpp:283-285,403-405) around a fixed-capacity
 * all-to-all (cap = rows per peer, >= T_local*top_k).  Buffers are caller-owned device memory:
 *   send_rows/recv_rows/ret_rows/back_rows [nranks][cap][H] model dtype; send_counts [E]; recv_counts [nranks][E].
 *   Passing NULL for send_counts / recv_counts selects the inline layout: all four row buffers are
 *   [nranks][cap+1][H] and the extra last row of every peer segment carries counts[E] (int32, needs 4E <= 2H),
 *   so one all-to-all moves rows and counts together.
 * A context with B2M_NUMERICS_FP32 is refused with B2M_EUNSUPPORTED by these four and by b2m_ep_p2p_init (so the
 * peer-to-peer calls below never run on it): the rows come back in the model dtype, so each expert output would be rounded
 * once more than on one GPU, where the fp32 combine reads it unrounded, and the result would depend on the exchange mode
 * (the peer-to-peer direct mode reads the owners' fp32 outputs in place).
 * Call order per layer: b2m_route -> b2m_ep_pack -> (exchange counts+rows) -> b2m_ep_regroup -> b2m_run_experts(T_total)
 *   -> b2m_ep_ungroup -> (exchange back) -> b2m_ep_unpack -> b2m_combine. */
int b2m_ep_pack(b2m_ctx* ctx, int nranks, int rank, int cap, int T_local, void* send_rows, int32_t* send_counts,
                void* stream);
int b2m_ep_regroup(b2m_ctx* ctx, int nranks, int rank, int cap, int T_total, const void* recv_rows,
                   const int32_t* recv_counts, void* stream);
int b2m_ep_ungroup(b2m_ctx* ctx, int nranks, int rank, int cap, void* ret_rows, void* stream);
int b2m_ep_unpack(b2m_ctx* ctx, int nranks, int rank, int cap, int T_local, const void* back_rows, void* stream);

/* Peer-to-peer variant of the same exchange: no collective library call inside the layer.  Each rank allocates its
 * receive/return areas + flag words (b2m_ep_p2p_init returns a 64-byte CUDA IPC handle), the host side exchanges the
 * handles once (any transport) and maps the peers with b2m_ep_p2p_open.  Per layer:
 *   b2m_route -> b2m_ep_p2p_dispatch (stores rows + counts straight into the owners' buffers over NVLink, then
 *   publishes an epoch flag with st.release.sys) -> b2m_ep_p2p_regroup (ld.acquire.sys wait, regroup) ->
 *   b2m_run_experts(T_total) -> b2m_ep_p2p_return (outputs stored into the source ranks' buffers + flag) ->
 *   b2m_ep_p2p_collect (wait, unpack) -> b2m_combine.  Every rank must issue the same sequence of calls. */
int b2m_ep_p2p_init(b2m_ctx* ctx, int nranks, int rank, int cap, void* ipc_handle_out64);
int b2m_ep_p2p_open(b2m_ctx* ctx, int peer, const void* ipc_handle64);
int b2m_ep_p2p_dispatch(b2m_ctx* ctx, int T_local, void* stream);
int b2m_ep_p2p_regroup(b2m_ctx* ctx, int T_total, void* stream);
int b2m_ep_p2p_return(b2m_ctx* ctx, void* stream);
int b2m_ep_p2p_collect(b2m_ctx* ctx, int T_local, void* stream);
/* fused variants (T_local <= 256): b2m_ep_p2p_route = b2m_route + b2m_ep_p2p_dispatch in the same two kernels (the
 * permute kernel stores each gathered row straight into its owner's buffer); b2m_ep_p2p_combine = b2m_ep_p2p_collect +
 * b2m_combine in one kernel (the combine kernel reads the returned rows in place). */
int b2m_ep_p2p_route(b2m_ctx* ctx, int layer, const void* x, const void* router_in, int router_in_kind,
                     int router_in_dtype, int T_local, void* stream);
int b2m_ep_p2p_combine(b2m_ctx* ctx, int layer, const void* x, int T_local, void* out, void* stream);
/* the whole expert-parallel layer in one call (T_local <= 256).  With <= 8 experts per rank it runs in FIVE kernels: the
 * permute kernel stores rows + per-slot expert tags into the owners' receive areas, the owners' gate/up GEMM reads its
 * token tile straight from that area (no regroup kernel; weights stream while the tokens are still in flight), the down
 * GEMM's last CTA publishes "done", and the source's combine kernel reads the owners' fp32 outputs in place over NVLink
 * (no return kernel).  Otherwise = b2m_ep_p2p_route -> regroup -> b2m_run_experts -> return -> b2m_ep_p2p_combine. */
int b2m_ep_p2p_layer(b2m_ctx* ctx, int layer, const void* x, const void* router_in, int router_in_kind,
                     int router_in_dtype, int T_local, void* out, void* stream);

/* ---- device-side activation tracer / predictor (SURVEY §8f N1).  Replaces ExpertTracer.update_entry / find_most_similar
 * (moe_infinity/memory/expert_tracer.py:78-125: two device syncs per sequence per layer in the reference) and
 * ExpertPredictor.predict (expert_predictor.py:17-35) with ONE kernel per layer call and no host round trip; the trace
 * library (load_trace, :40-52) and the per-sequence matrices live on the device.
 *   b2m_trace_init        capacity = library entries (ArcherConfig.trace_capacity), max_seqs = concurrent sequences
 *   b2m_trace_load        load_trace: n entries [n][L][E] fp32 from the host (persistent entries, never replaced)
 *   b2m_trace_reset_seq   create_entry: zero the sequence's matrix
 *   b2m_trace_update_predict  after a routing call of num_seqs*seq_len tokens (sequence-major rows): update every sequence's
 *                         matrix at `layer`, pick its nearest library trace, write the decayed prediction, and add it to the
 *                         call's hint matrix [L][E] (the scores ExpertPrefetcher.prefetch_experts sorts).  Asynchronous.
 *                         In offload mode the hint matrix rides back with the next per-layer count read-back and feeds
 *                         the prefetch scheduler (b2m_prefetch_hint semantics) when auto_prefetch != 0.
 *   b2m_trace_finish_seq  finish_entry (:61-76): store the sequence's matrix in the library
 *   b2m_trace_read        what: 0 sequence matrix, 1 last prediction of a sequence, 2 hint matrix, 3 library entry (all [L][E]
 *                         fp32), 4 access counts (int32 [capacity] written as-is), 5 winner index of a sequence (1 int32);
 *                         synchronises the device (tests, get_trace / save_trace persistence) */
int b2m_trace_init(b2m_ctx* ctx, int capacity, int max_seqs, int auto_prefetch);
int b2m_trace_load(b2m_ctx* ctx, int n, const float* lib_host);
int b2m_trace_reset_seq(b2m_ctx* ctx, int seq_slot, void* stream);
int b2m_trace_update_predict(b2m_ctx* ctx, int layer, int seq_slot0, int num_seqs, int seq_len, void* stream);
int b2m_trace_finish_seq(b2m_ctx* ctx, int seq_slot, void* stream);
int b2m_trace_read(b2m_ctx* ctx, int what, int index, void* host_out);

/* diagnostics (B2M_TIMELINE=1 in the environment): device-side nanosecond timestamps of the kernels of b2m_ep_p2p_layer's
 * direct mode, 16 words per layer: [0,1] gate/top-k first start / last end, [2,3] permute+dispatch, [4,5,6] gate/up GEMM
 * start / peers' flags seen / end, [8,10] down GEMM start / end (after "done" is published), [12,13,14] combine start /
 * owners' flags seen / end.  Synchronises the device. */
int b2m_timeline_read(b2m_ctx* ctx, unsigned long long* host_out, int n_layers);

/* ---- disk tier (SURVEY §8f N3): reader of the reference's on-disk tensor store, `<prefix>/archer_index` +
 * `<prefix>/archer_param_<n>` (archer_tensor_index.cpp:101-132, archer_tensor_handle.cpp:53-86).  Replaces
 * ArcherTensorHandle::ReadTensor (archer_tensor_handle.cpp:189-201) -> ArcherPrioAioHandle::Read
 * (archer_prio_aio_handle.cpp:37-70): there a synchronous call served by ONE worker thread in 1 MiB preads, with
 * high-priority requests overtaking low-priority ones between blocks (Schedule, :123-169).  Here: asynchronous tickets, a
 * pool of worker threads, the same two-level priority at block granularity, O_DIRECT for 4096-aligned blocks and buffered
 * reads for the rest (and on file systems without O_DIRECT).  Host code only: usable without a GPU.
 *   b2m_store_open        num_threads <= 0: 8; block_bytes <= 0: 4 MiB; flags: B2M_STORE_NO_ODIRECT
 *   b2m_store_tensor      index entry of a tensor id (any out pointer may be NULL)
 *   b2m_store_blob_bytes  size of the concatenation of tensors `ids` (the expert blob, model_topology.cpp:429-431)
 *   b2m_store_read_async  read the tensors back to back (exact sizes, no alignment padding) into dst
 *   b2m_store_read_range_async  bytes [blob_off, blob_off+len) of that concatenation into dst (one staging chunk)
 *   b2m_store_poll        1 done, 0 pending, B2M_EIO failed (the ticket stays valid)
 *   b2m_store_wait        blocks until the request is complete and retires the ticket; B2M_EIO with a message on failure
 *   b2m_store_stats       out4 = {bytes read, O_DIRECT blocks, buffered blocks, requests}
 *   b2m_store_close       serves what is queued, joins the workers, closes the files */
#define B2M_STORE_NO_ODIRECT 1
typedef struct b2m_store b2m_store;
int b2m_store_open(const char* prefix, int num_threads, int block_bytes, int flags, b2m_store** out);
int b2m_store_close(b2m_store* store);
const char* b2m_store_last_error(b2m_store* store);
int b2m_store_count(b2m_store* store);
int b2m_store_tensor(b2m_store* store, uint32_t id, uint32_t* file_id, int64_t* offset, uint64_t* nbytes);
int b2m_store_blob_bytes(b2m_store* store, const uint32_t* ids, int n, uint64_t* total);
int b2m_store_read_async(b2m_store* store, const uint32_t* ids, int n, void* dst, uint64_t dst_bytes, int high_prio,
                         uint64_t* ticket);
int b2m_store_read_range_async(b2m_store* store, const uint32_t* ids, int n, uint64_t blob_off, uint64_t len, void* dst,
                               int high_prio, uint64_t* ticket);
int b2m_store_poll(b2m_store* store, uint64_t ticket);
int b2m_store_wait(b2m_store* store, uint64_t ticket);
int b2m_store_stats(b2m_store* store, uint64_t out4[4]);
/* An expert whose weights stay on the store (host DRAM smaller than the model): a miss reads the blob chunk by chunk into a
 * small pinned staging ring and copies each chunk to its HBM slot while the next ones are being read (the reference stages
 * disk -> pinned host -> device one whole tensor at a time, archer_tensor_handle.cpp:189-201 + model_topology.cpp:150-185).
 * `ids` are the expert's tensor ids in blob order (the list register_expert receives, model_offload.py:851-853); their sizes
 * must add up to the expert's blob size.  The store must outlive the context.  Chunk size: B2M_DISK_CHUNK_BYTES in the
 * environment at context creation (default 32 MiB). */
int b2m_register_expert_on_store(b2m_ctx* ctx, int layer, int expert, b2m_store* store, const uint32_t* ids, int n);

#ifdef __cplusplus
}
#endif
#endif /* B2M_H_ */
