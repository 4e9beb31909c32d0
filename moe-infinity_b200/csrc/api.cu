// api.cu -- C-ABI entry points (include/b2m.h), context, HBM expert cache and prefetch scheduler.
//
// Host-side design:
//  * one arena of fixed-size expert slots in HBM (blob layout == the reference's host blob, so staging an expert
//    is one contiguous H2D copy); three 3-D TMA tensor maps {K, rows, slot} describe every slot at once;
//  * device table slot_of[L][E] tells the grouped GEMM which slot holds which expert; it is re-uploaded in
//    stream order only when the mapping of that layer changed;
//  * when every expert fits (num_slots >= L*E) the hot call is sync-free and CUDA-graph capturable;
//  * otherwise ("offload mode") the per-expert token counts are read back once per layer -- the same
//    synchronisation the reference performs (expert_executor.py:34-39) -- misses are staged on a fetch stream,
//    predicted experts on a prefetch stream, and the compute stream waits on per-expert events only.
//  Cache policy (explicit; SURVEY §9 Q4): evict the resident, unpinned, not-in-use expert with the smallest
//  in-cache visit count (core/parallel/expert_dispatcher.cpp:243-258), skipping protected prefetch candidates
//  unless nothing else is evictable (core/prefetch/task_scheduler.cpp:288-296).
#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <mutex>
#include <new>
#include <string>
#include <unordered_set>
#include <vector>

#include <cudaTypedefs.h>

#include "../../include/b2m.h"
#include "b2m_internal.h"
#include "fp8_weights.cuh"
#include "int4_weights.cuh"

using namespace b2m;

namespace {

constexpr int NT_LIST[5] = {16, 32, 64, 128, 256};
constexpr int EVENT_RING = 64;
constexpr int STAGE_RING = 8;

std::string g_create_error;

// ---- run-time switches: read ONCE per process, here and nowhere else in this file.  The alternative to every default
// stays selectable for A/B measurement (DESIGN.md §6).
struct Switches {
  bool nt256, pdl, early_k3, rows_by_gate, pdl_k3, early_a, streamk, ep_early_combine, ep_direct, ep_mrows, timeline, fused_ffn;
  int ep_l2pf_mb;
  long long nt256_min_avg;
  static bool off(const char* n) { const char* v = getenv(n); return v && v[0] == '0'; }   // default on
  static bool on(const char* n) { const char* v = getenv(n); return v && v[0] == '1'; }    // default off
  Switches()
      : nt256(!off("B2M_NT256")),                 // 256-token tiles for the down projection in the tensor-bound regime
        pdl(on("B2M_PDL")),                       // programmatic dependent launch on every decode kernel
        early_k3(!off("B2M_EARLY_K3")),           // gate/up GEMM prefetches weights under the permute kernel
        rows_by_gate(!off("B2M_ROWS_BY_GATE")),   // the last gate/top-k CTA publishes the row maps
        pdl_k3(on("B2M_PDL_K3")),
        early_a(!off("B2M_EARLY_A")),             // down GEMM prefetches weights under the gate/up GEMM's tail
        streamk(!off("B2M_STREAMK")),             // stream-K partition of the split-K down GEMM
        ep_early_combine(!off("B2M_EP_EARLY_COMBINE")),
        ep_mrows(!off("B2M_EP_MROWS")),
        ep_l2pf_mb(getenv("B2M_EP_L2PF_MB") ? atoi(getenv("B2M_EP_L2PF_MB")) : 0),   // L2 prefetch of gate/up weights behind programmatic edges: opt-in
        ep_direct(!off("B2M_EP_DIRECT")),         // four-launch expert-parallel layer
        timeline(on("B2M_TIMELINE")),             // device timestamps of the expert-parallel layer (diagnostics)
        fused_ffn(on("B2M_FUSED_FFN")),           // (only in -DB2M_ENABLE_FUSED_FFN builds) gate/up + down GEMMs in one persistent kernel
                                                  // (it keeps the side-stream shared-expert GEMMs off the SMs) -> opt-in
        nt256_min_avg(getenv("B2M_NT256_MIN_AVG") ? atoll(getenv("B2M_NT256_MIN_AVG")) : 256) {}
};
const Switches& sw() {
  static const Switches s;
  return s;
}

struct ExpertShape {
  int H = 0, I = 0;
  bool dual = true;
  int act = ACT_SILU;
  size_t off_gate = 0, off_up = 0, off_down = 0, bytes = 0;
  bool has_bias = false;          // fc1 | fc1_bias | fc2 | fc2_bias (NLLB / FSGPT)
  size_t off_bias1 = 0, off_bias2 = 0;
  int bits = 16;                  // bits per stored weight
  size_t grid_gate = 0, grid_up = 0, grid_down = 0;   // quantised formats: byte offsets of the matrices' side grids
};

// How routed experts are stored: one row per B2M_WEIGHTS_* value.  A quantised format's header (fp8_weights.cuh,
// int4_weights.cuh) defines its blob and decode; gemm_body in grouped_gemm.cu decodes it for its A source.
struct WeightFormat {
  int id;                               // B2M_WEIGHTS_*
  const char* name;                     // in messages
  int act_dtype;                        // the model dtype (activations) the format needs; -1 = any
  int bits;                             // bits per stored weight; 0 = the model dtype's
  size_t (*grid_bytes)(int rows, int cols);   // bytes of the side grid (block scales / row scales / group words) of a
                                              // rows x cols matrix; null = none
  int hi_multiple;                      // hidden and inter must be multiples of this
  int a_src;                            // AS_*: how the tensor-core GEMMs read the weights
};
const WeightFormat WEIGHT_FORMATS[] = {
    {B2M_WEIGHTS_MODEL_DTYPE, "model-dtype", -1, 0, nullptr, 1, AS_BF16},
    {B2M_WEIGHTS_FP8_E4M3_B128, "fp8", B2M_DTYPE_BF16, 8, f8::scale_grid_bytes, f8::BLOCK, AS_FP8},
    {B2M_WEIGHTS_FP8_E4M3_ROW, "fp8 (row scales)", B2M_DTYPE_BF16, 8, f8::row_scale_bytes, f8::BLOCK, AS_FP8_ROW},
    {B2M_WEIGHTS_INT4_G128, "int4", B2M_DTYPE_BF16, 4, i4::grid_bytes, i4::GROUP, AS_INT4},
    {B2M_WEIGHTS_INT4_G128_F16, "int4 (fp16 scales)", B2M_DTYPE_F16, 4, i4::grid_bytes, i4::GROUP, AS_INT4},
};

// How a router kind constrains the configuration and changes the host logic around its routing math (route.cu): one row
// per B2M_ROUTER_* value.  ROUTER_DEEPSEEK_GROUP's group rule is checked at launch (route_args_ok), not here.
enum : int { GROUPS_ANY = 0,   // n_group / topk_group are ignored
             GROUPS_NONE = 1,  // no group-limited routing: n_group == topk_group == 1
             GROUPS_V3 = 2 };  // noaux_tc: n_group in 1..32 divides E, E / n_group >= 2, topk_group in 1..n_group
struct RouterKind {
  int id;                     // B2M_ROUTER_*
  const char* name;           // in messages
  bool model_dtype_logits;    // the gate is an nn.Linear in the model dtype: logits are rounded to it (RouteParams)
  bool gate_up_down;          // experts are gate|up|down (expert_type 5) ...
  bool dtype16;               // ... in a bf16 or f16 model dtype
  int groups;                 // GROUPS_*
  bool unscaled;              // routed_scaling_factor must be 1
  bool unnormalised;          // norm_topk_prob must be 0
  bool needs_shared;          // every layer has a shared expert: shared_inter > 0
  bool top1;                  // top_k must be 1
  bool gate_bias;             // a per-layer correction bias (b2m_set_gate_bias), required to route and to look ahead
  bool shared_gate;           // a per-layer shared-expert gate (b2m_set_shared_gate)
  bool scales_inputs;         // the weights scale the gathered expert inputs and the combine sums unweighted; the router
                              // ranks logits, so no scores as router input, and no input permutation
  bool capacity;              // a capacity pass after top-k: seq_len divides T, extra routing launches, no early gate/up GEMM
                              // and no direct-mode expert parallelism
  bool ep;                    // expert parallelism is available
  int combine, combine_fp32;  // COMBINE_* under B2M_NUMERICS_REFERENCE / B2M_NUMERICS_FP32
};
const RouterKind ROUTERS[] = {
    // id, name, model_dtype_logits, gate_up_down, dtype16, groups, unscaled, unnormalised, needs_shared, top1, gate_bias,
    // shared_gate, scales_inputs, capacity, ep, combine, combine_fp32
    {B2M_ROUTER_MIXTRAL,        "mixtral",     true,  false, false, GROUPS_ANY,  false, false, false, false, false, false, false, false, true,  COMBINE_MIXTRAL,  COMBINE_FP32},
    {B2M_ROUTER_DEEPSEEK_GREEDY, "greedy",     false, false, false, GROUPS_ANY,  false, false, false, false, false, false, false, false, true,  COMBINE_DEEPSEEK, COMBINE_FP32},
    {B2M_ROUTER_DEEPSEEK_GROUP, "group",       false, false, false, GROUPS_ANY,  false, false, false, false, false, false, false, false, true,  COMBINE_DEEPSEEK, COMBINE_FP32},
    {B2M_ROUTER_SWITCH_TOP1,    "switch",      false, false, false, GROUPS_ANY,  false, false, false, true,  false, false, false, true,  true,  COMBINE_SWITCH,   COMBINE_SWITCH},
    {B2M_ROUTER_DEEPSEEK_V3,    "deepseek_v3", false, false, false, GROUPS_V3,   false, false, false, false, true,  false, false, false, true,  COMBINE_DEEPSEEK, COMBINE_FP32},
    {B2M_ROUTER_QWEN_MOE,       "qwen_moe",    true,  true,  true,  GROUPS_NONE, true,  false, false, false, false, true,  false, false, false, COMBINE_QWEN,     COMBINE_FP32},
    {B2M_ROUTER_LLAMA4,         "llama4",      true,  true,  true,  GROUPS_NONE, true,  true,  true,  false, false, false, true,  false, false, COMBINE_LLAMA4,   COMBINE_FP32},
};
// the names of the router kinds that have a feature, for the message that refuses it to the others
std::string routers_with(bool RouterKind::*has) {
  std::string s;
  for (const RouterKind& r : ROUTERS)
    if (r.*has) s += (s.empty() ? "" : " or ") + std::string(r.name);
  return s;
}

struct Arena {
  uint8_t* base = nullptr;
  size_t slot_bytes = 0;
  int nslots = 0;
  bool owned = false;
  ExpertShape shape;
  CUtensorMap tm_gate, tm_up, tm_down;
  CUtensorMap tm_gate_h, tm_up_h, tm_down_h;   // 64-row boxes for the 2-CTA multicast kernels (each CTA fetches half a tile)
};

enum ExpertState : int { ST_UNREGISTERED = 0, ST_HOST = 1, ST_LOADING = 2, ST_RESIDENT = 3 };

struct Expert {
  const uint8_t* host = nullptr;
  b2m_store* store = nullptr;   // disk tier: the blob stays on the store (b2m_register_expert_on_store); tensor ids in blob order
  std::vector<uint32_t> ids;
  bool backed() const { return host != nullptr || store != nullptr; }   // can be evicted and staged again
  int state = ST_UNREGISTERED;
  int slot = -1;
  bool pinned = false;
  bool prefetched_unused = false;
  int visits = 0;               // incache_visit_count (model_topology.h:75-91)
  float freq = 0.5f;            // B2M_CACHE_ACTIVATION_AWARE: moving average of "activated in a step"
  uint64_t total_visits = 0;
  cudaEvent_t ready = nullptr;  // H2D complete
  bool ready_pending = false;   // compute stream has not yet been ordered after `ready`
};

struct Slot {
  int owner = -1;
  int last_use_ev = -1;  // index into the event ring
};

}  // namespace

struct b2m_ctx {
  b2m_config cfg;
  std::string err;
  int num_sms = 132;
  size_t total_mem = 0;
  PFN_cuTensorMapEncodeTiled_v12000 encode = nullptr;

  Arena arena;         // routed experts
  Arena shared_arena;  // DeepSeek shared experts: slot == layer, always resident
  std::vector<uint8_t> shared_registered;
  std::vector<Expert> experts;  // [L*E], id = layer*E + expert
  std::vector<Slot> slots;
  std::vector<int> free_slots;
  bool offload = false;

  // device tables
  int* d_slot_of = nullptr;  // [L*E]
  std::vector<int> h_slot_of;
  std::vector<uint8_t> row_dirty;
  int* h_stage = nullptr;  // pinned [STAGE_RING][E]
  int stage_pos = 0;
  std::vector<const void*> gate_w;  // per layer device pointers
  std::vector<const float*> gate_bias;  // RouterKind::gate_bias: per layer e_score_correction_bias [E] (device, borrowed)
  std::vector<const uint16_t*> input_perm;  // B2M_WEIGHTS_INT4_G128_F16: per layer [E][H] gather table (device, borrowed) or null
  std::vector<const void*> shared_gate_w;   // RouterKind::shared_gate: per layer [H] shared_expert_gate.weight

  // workspace
  int cap_T = 0, cap_R = 0;
  int* d_topk_idx = nullptr;
  float* d_topk_w = nullptr;
  int* d_row_of = nullptr;
  int* d_perm_token = nullptr;
  int* d_counts = nullptr;
  int* d_offsets = nullptr;
  int* d_chunk_counts = nullptr;
  float* d_scores = nullptr;
  void* d_logits = nullptr;
  void* d_xp = nullptr;
  void* d_hmid = nullptr;
  float* d_y = nullptr;
  void* d_hmid_s = nullptr;
  float* d_y_s = nullptr;
  void* d_shared_gate = nullptr;   // Qwen2-MoE: [T] model-dtype gate values of the shared expert
  int* h_counts = nullptr;  // pinned [E+1]
  bool last_counts_valid = false;
  CUtensorMap tm_xp[5], tm_hmid[5], tm_hmid_s[5];

  // streams / events
  cudaStream_t fetch_stream = nullptr, prefetch_stream = nullptr;
  cudaStream_t shared_stream = nullptr;          // DeepSeek shared experts run here, concurrently with the routing kernels
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  bool shared_in_flight = false;                 // b2m_moe_forward already launched this call's shared-expert GEMMs
  cudaEvent_t ev_ring[EVENT_RING] = {nullptr};
  // disk tier staging: pinned chunks that take a store-backed expert from the reader to the copy engine (see issue_copy)
  static constexpr int DISK_RING = 3;
  uint8_t* disk_bounce[DISK_RING] = {nullptr};
  cudaEvent_t disk_ev[DISK_RING] = {nullptr};
  bool disk_ev_pending[DISK_RING] = {false};
  size_t disk_chunk = 32u << 20;
  uint64_t disk_bytes = 0;
  int ev_pos = 0;

  // prefetch scheduler
  std::unordered_set<int> protected_set;
  std::deque<int> pending;
  std::vector<int> inflight;
  std::vector<int> last_active;

  int cur_ksplit = 1, cur_nt = 16, cur_nt_dn = 16, cur_T = 0;   // token-tile widths of the up (K3) and down (K4) GEMMs
  const WeightFormat* wf = nullptr;   // how the routed experts are stored
  const RouterKind* rk = nullptr;     // how they are routed
  bool ep_mode = false;       // experts of other ranks are simply absent (never an error)
  // 12-bit packed copy of the routed arena (weight_pack.cuh; same slot index), read by the decode GEMMs.  Allocated by the first
  // eager forward that packs, if the device keeps PK_RESERVE free beside it.  d_ok[slot]: bit b = matrix b (gate, up, down)
  // of the slot has a current packed copy.  A slot is stale from the moment a caller may write it (its device flag is cleared
  // in stream order then) until an eager forward of its layer packs it: the second one after the write, so the forward that
  // directly follows a weight load runs exactly as it would without the packed copy (no allocation, no extra device work).
  struct Packed {
    int state = 0;              // 0 = not allocated yet, 1 = allocated, -1 = not available in this context
    uint8_t* base = nullptr;
    int* d_ok = nullptr;
    size_t slot_bytes = 0;
    size_t off[3] = {0, 0, 0};  // packed gate, up, down inside a packed slot
    std::vector<uint8_t> dirty; // [nslots] PK_WRITTEN / PK_SEEN (one eager forward since the write) / 0 = packed or never
  } pk;
  // device-side tracer / predictor (b2m_trace_*)
  struct Trace {
    int capacity = 0, max_seqs = 0, persistent = 0, auto_prefetch = 0;
    float *seq = nullptr, *lib = nullptr, *pred = nullptr, *hint = nullptr;
    int *access = nullptr, *winner = nullptr;
    float* h_hint = nullptr;      // pinned [L][E]: the hint matrix rides back with the per-layer count read-back
    bool hint_pending = false;
    int hint_layer = 0;
  } tr;
  unsigned long long* tl_next = nullptr;   // timeline slots of the layer call in progress
  unsigned long long* d_tl = nullptr;   // B2M_TIMELINE=1: [L][16] device timestamps of the expert-parallel layer's kernels
  bool ep_direct_next = false;   // the routing / combine call in progress belongs to b2m_ep_p2p_layer's direct mode
  bool ep_fused_last = false;    // ... and its routing call was the fused gate/top-k + dispatch kernel
  int ep_inline = 0;          // exchange buffers carry the counts in an extra row per peer
  // peer-to-peer exchange (CUDA IPC mapped buffers of the other ranks)
  struct P2P {
    int nranks = 0, rank = 0, cap = 0;
    uint8_t* base = nullptr;            // own allocation: [recv area][back area][flags]
    size_t area_bytes = 0;
    uint8_t* peer_base[16] = {nullptr};
    int* local_ctr = nullptr;           // [0..1] epoch, [2..3] done counters, [4..19] slot counters of the fused dispatch
    // direct mode regions inside the allocation (after the two exchange areas and the flags): row counters cnt[E/nranks] (int),
    // receive rows [E/nranks][nranks*cap][H] (model dtype), outputs y [E/nranks][nranks*cap][H] (fp32)
    size_t cnt_off = 0, drecv_off = 0, y_off = 0;
    CUtensorMap tm_recv[5];             // the direct receive area as the token operand of the gate/up GEMM: [E*cap rows][H]
    void* d_hmid = nullptr;             // direct mode intermediate [E*cap rows][I] (local, same row indexing as the receive area)
    CUtensorMap tm_hmid[5];
    int m_rows = 0;                     // weight rows per gate/up tile in direct mode (0 = not planned yet), see plan_ep_m_rows
    CUtensorMap tm_gate_r, tm_up_r;     // gate/up weight maps with a box of m_rows rows
  } p2p;
  int* d_offsets_src = nullptr;  // [E+1]
  int* d_ticket = nullptr;       // CTA arrival counter of the small-T gate/top-k kernel
  int* d_gbar = nullptr;         // [2] grid barrier of the fused expert-FFN kernel (arrival counter, generation)
  int* d_err = nullptr;          // sticky device error word (RouteParams::err_flag)
  int* h_err = nullptr;          // pinned readback of d_err
  bool k3_early_ok = false;      // offsets of the current routing were published before the permute kernel
  int* d_dest_of = nullptr;      // [cap_R]
  // on-demand budget in expert units, accounted exactly as the reference's cache_sizes_[gpu] (expert_dispatcher.cpp:228,
  // 257,266): -1 for EVERY dispatched expert (hit or miss -- the reference subtracts byte_size unconditionally), +1 per
  // on-demand eviction; a miss evicts exactly one victim iff budget < 1.  Physical slots remain the hard limit.
  long long budget_units = 0;
  int cur_layer = 0;             // layer of the dispatch in progress / last dispatched (next-use distance of the activation-aware policy)
  // look-ahead prefetch governor: on a link-bound path a wrong prefetch costs a whole expert of bandwidth, so the scheduler
  // watches its own accuracy (prefetched experts used before eviction vs evicted unused) and suspends itself when it is low
  unsigned pf_win_useful = 0, pf_win_wasted = 0;
  long long pf_suspended_until = 0;   // in on-demand layer calls (stats.host_syncs)
  int* d_look = nullptr;         // [E] look-ahead counts: next layer's router applied to this layer's input
  int* h_look = nullptr;         // pinned [E]
  bool look_pending = false;     // the last routing call launched the look-ahead kernel
  bool last_look_valid = false;
  b2m_stats stats;
};

namespace {

int fail(b2m_ctx* c, int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  if (c) c->err = buf; else g_create_error = buf;
  return code;
}

#define CK(c, call)                                                                                   \
  do {                                                                                                \
    cudaError_t _e = (call);                                                                          \
    if (_e != cudaSuccess)                                                                            \
      return fail((c), B2M_ECUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

// Slot layout of one expert: its matrices in the model's tensor order, H * I * bits / 8 bytes each, then (quantised formats)
// the side grid of each matrix, grid_bytes(rows, cols), in the same order; rounded up to 16 B so that TMA strides stay
// multiples of 16 B.  For the quantised formats this is f8::expert_blob_bytes, f8::row_expert_blob_bytes and
// i4::expert_blob_bytes.
bool make_shape(int expert_type, int H, int I, int bits, size_t (*grid_bytes)(int, int), ExpertShape* s) {
  const size_t m = (size_t)H * I * bits / 8, esize = bits / 8;
  s->H = H;
  s->I = I;
  s->bits = bits;
  switch (expert_type) {
    case B2M_EXPERT_MIXTRAL_MOE_DENSE_ACT_DENSE:  // w1 | w2 | w3  (expert_module.cpp:139-145)
      s->dual = true; s->act = ACT_SILU; s->off_gate = 0; s->off_down = m; s->off_up = 2 * m; s->bytes = 3 * m;
      break;
    case B2M_EXPERT_DEEPSEEK_MOE_DENSE_ACT_DENSE:  // gate | up | down  (:185-191)
      s->dual = true; s->act = ACT_SILU; s->off_gate = 0; s->off_up = m; s->off_down = 2 * m; s->bytes = 3 * m;
      break;
    case B2M_EXPERT_SWITCH_DENSE_GATED_ACT_DENSE:  // wi_0 | wi_1 | wo  (:45-52)
      s->dual = true; s->act = ACT_GELU; s->off_gate = 0; s->off_up = m; s->off_down = 2 * m; s->bytes = 3 * m;
      break;
    case B2M_EXPERT_SWITCH_DENSE_ACT_DENSE:  // wi | wo  (:17-23)
      s->dual = false; s->act = ACT_RELU; s->off_gate = 0; s->off_up = 0; s->off_down = m; s->bytes = 2 * m;
      break;
    case B2M_EXPERT_NLLB_MOE_DENSE_ACT_DENSE:   // fc1 | fc1_bias | fc2 | fc2_bias  (:70-77; forward :88-92)
    case B2M_EXPERT_FSGPT_MOE_DENSE_ACT_DENSE:  // same binding (:104-111; forward :124-128, ReLU as well)
      s->dual = false; s->act = ACT_RELU; s->has_bias = true;
      s->off_gate = 0; s->off_up = 0; s->off_bias1 = m; s->off_down = m + (size_t)I * esize;
      s->off_bias2 = s->off_down + m; s->bytes = s->off_bias2 + (size_t)H * esize;   // H, I multiples of 8: all 16-B aligned
      break;
    default:
      return false;
  }
  if (grid_bytes) {
    // matrix j of the blob starts at j * m; the grids follow the matrices in that order (gate / up [I x H], down [H x I])
    const size_t g_in = grid_bytes(I, H), g_dn = grid_bytes(H, I);
    const size_t j_dn = s->off_down / m;
    auto grid_of = [&](size_t off) {
      size_t o = 3 * m;
      for (size_t j = 0; j < off / m; ++j) o += j == j_dn ? g_dn : g_in;
      return o;
    };
    s->grid_gate = grid_of(s->off_gate);
    s->grid_up = grid_of(s->off_up);
    s->grid_down = grid_of(s->off_down);
    s->bytes += 2 * g_in + g_dn;
  }
  s->bytes = (s->bytes + 15) & ~(size_t)15;
  return true;
}

// A K-major tensor map over `bits`-bit values: 16-bit values in the model dtype, narrower ones as uint8 bytes.  One k-row of
// the GEMM's 64-wide k-block spans 64 * bits / 8 bytes (128, 64 or 32), and that span is the swizzle.
int encode_map(b2m_ctx* c, CUtensorMap* tm, int bits, void* base, int rank, const uint64_t* dims,
               const uint64_t* strides_bytes /*rank-1*/, const uint32_t* box) {
  cuuint64_t gdim[3];
  cuuint64_t gstr[2];
  cuuint32_t b[3], es[3];
  for (int i = 0; i < rank; ++i) { gdim[i] = dims[i]; b[i] = box[i]; es[i] = 1; }
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  const CUtensorMapDataType dt = bits < 16 ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                               : c->cfg.dtype == B2M_DTYPE_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  const int span = 64 * bits / 8;
  const CUtensorMapSwizzle swz = span == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : span == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B;
  CUresult r = c->encode(tm, dt, (cuuint32_t)rank, base, gdim, gstr, b, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(c, B2M_ECUDA, "cuTensorMapEncodeTiled failed (CUresult %d)", (int)r);
  return B2M_OK;
}

int build_arena_maps_box(b2m_ctx* c, Arena* a, uint32_t box_rows, CUtensorMap* g, CUtensorMap* u, CUtensorMap* d);
int build_arena_maps(b2m_ctx* c, Arena* a) {
  int r = build_arena_maps_box(c, a, 128, &a->tm_gate, &a->tm_up, &a->tm_down);
  if (r) return r;
  return build_arena_maps_box(c, a, 64, &a->tm_gate_h, &a->tm_up_h, &a->tm_down_h);
}
int build_arena_maps_box(b2m_ctx* c, Arena* a, uint32_t box_rows, CUtensorMap* tg, CUtensorMap* tu, CUtensorMap* td) {
  const ExpertShape& s = a->shape;
  const uint64_t es = s.bits < 16 ? 1 : 2;                                          // bytes per map element (encode_map)
  const uint64_t rH = (uint64_t)s.H * s.bits / 8, rI = (uint64_t)s.I * s.bits / 8;   // bytes per row of K = H / K = I
  const uint32_t box[3] = {(uint32_t)(64 * s.bits / 8 / es), box_rows, 1};          // one k-row of a 64-wide k-block
  {
    const uint64_t dims[3] = {rH / es, (uint64_t)s.I, (uint64_t)a->nslots};
    const uint64_t str[2] = {rH, (uint64_t)a->slot_bytes};
    int r = encode_map(c, tg, s.bits, a->base + s.off_gate, 3, dims, str, box);
    if (r) return r;
    r = encode_map(c, tu, s.bits, a->base + s.off_up, 3, dims, str, box);
    if (r) return r;
  }
  {
    const uint64_t dims[3] = {rI / es, (uint64_t)s.H, (uint64_t)a->nslots};
    const uint64_t str[2] = {rI, (uint64_t)a->slot_bytes};
    int r = encode_map(c, td, s.bits, a->base + s.off_down, 3, dims, str, box);
    if (r) return r;
  }
  return B2M_OK;
}

int build_act_map(b2m_ctx* c, CUtensorMap* tm, void* base, int K, int rows, int nt) {
  const uint64_t dims[2] = {(uint64_t)K, (uint64_t)rows};
  const uint64_t str[1] = {(uint64_t)K * 2};
  const uint32_t box[2] = {64, (uint32_t)nt};
  return encode_map(c, tm, 16, base, 2, dims, str, box);
}

int nt_index(int nt) { return nt == 16 ? 0 : nt == 32 ? 1 : nt == 64 ? 2 : nt == 128 ? 3 : 4; }

int pick_nt(int T) {
  for (int i = 0; i < 4; ++i)
    if (T <= NT_LIST[i]) return NT_LIST[i];
  return 128;
}
// tensor-bound regime: 256-token tiles when the average expert sees at least one full tile
// (B2M_NT256=0 disables): a weight tile read once serves twice the tokens.  Down projection only (see plan_gemm).
int pick_nt_model(const b2m_config& f, int T) {
  const long long avg = (long long)T * f.top_k / f.num_experts;
  if (sw().nt256 && avg >= sw().nt256_min_avg && f.hidden >= 256) return 256;
  return pick_nt(T);
}

// split-K for the down projection: enough tiles for ~6 waves, every split non-empty and >= 4 k-blocks
int pick_ksplit(const b2m_ctx* c, int T, int M, int K, int E, int k, int nt) {
  const int kblocks = (K + 63) / 64;
  const long long rows = (long long)T * k;
  const int active = (int)std::min<long long>(E, std::max<long long>(1, rows));
  const long long n_tiles = std::max<long long>(1, (rows / std::max(1, active) + nt - 1) / nt);
  const long long tiles = (long long)active * ((M + 127) / 128) * n_tiles;
  int ks = (int)std::min<long long>(8, (6LL * c->num_sms + tiles - 1) / tiles);
  ks = std::max(1, std::min(ks, kblocks / 4 > 0 ? kblocks / 4 : 1));
  while (ks > 1) {
    const int per = (kblocks + ks - 1) / ks;
    if ((ks - 1) * per < kblocks) break;
    --ks;
  }
  return ks;
}

cudaEvent_t next_ring_event(b2m_ctx* c, int* idx) {
  *idx = c->ev_pos;
  cudaEvent_t e = c->ev_ring[c->ev_pos];
  c->ev_pos = (c->ev_pos + 1) % EVENT_RING;
  return e;
}

// ---------------- packed weights ----------------
constexpr size_t PK_RESERVE = 2ull << 30;   // device memory left free beside the packed copy
enum : uint8_t { PK_SEEN = 1, PK_WRITTEN = 2 };
size_t pk_matrix_rows(const ExpertShape& s, int m) { return m == 2 ? s.H : (m == 1 && !s.dual) ? 0 : s.I; }
size_t pk_matrix_cols(const ExpertShape& s, int m) { return m == 2 ? s.I : s.H; }
// contexts whose routed experts the decode GEMMs may read from a packed copy: all resident, bf16 tensor cores (gemm_impl 0),
// one rank
bool pk_eligible(const b2m_ctx* c) {
  return c->cfg.gemm_impl == 0 && !c->offload && c->cfg.dtype == B2M_DTYPE_BF16 && !c->ep_mode &&
         c->pk.slot_bytes > 0;
}
// slot `slot` may be written by the caller from now on (on stream st): its packed copy is stale
int pk_invalidate(b2m_ctx* c, int slot, cudaStream_t st) {
  if (slot < 0 || c->pk.dirty.empty()) return B2M_OK;
  c->pk.dirty[slot] = PK_WRITTEN;
  if (c->pk.d_ok) CK(c, cudaMemsetAsync(c->pk.d_ok + slot, 0, sizeof(int), st));
  return B2M_OK;
}
// the stale resident slots of `layer` that this eager call's gate/up GEMM launch packs (those seen by an earlier eager forward
// since they were written); none while the stream is captured (their flags stay 0, the graph reads them as bf16)
int pk_collect(b2m_ctx* c, int layer, cudaStream_t st, std::vector<int>* out) {
  out->clear();
  if (!pk_eligible(c) || c->pk.state < 0) return B2M_OK;
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(st, &cs) != cudaSuccess) cudaGetLastError();
  if (cs != cudaStreamCaptureStatusNone) return B2M_OK;
  const int E = c->cfg.num_experts;
  for (int e = 0; e < E; ++e) {
    const int slot = c->experts[(size_t)layer * E + e].slot;
    if (slot < 0 || !c->pk.dirty[slot]) continue;
    if (c->pk.dirty[slot] == PK_WRITTEN) c->pk.dirty[slot] = PK_SEEN;
    else out->push_back(slot);
  }
  if (out->empty()) return B2M_OK;
  if (c->pk.state == 0) {
    c->pk.state = -1;
    const size_t bytes = (size_t)c->arena.nslots * c->pk.slot_bytes;
    size_t fr = 0, tot = 0;
    CK(c, cudaMemGetInfo(&fr, &tot));
    if (fr < bytes + PK_RESERVE + sizeof(int) * c->arena.nslots) { out->clear(); return B2M_OK; }
    if (cudaMalloc((void**)&c->pk.base, bytes) != cudaSuccess) { cudaGetLastError(); out->clear(); return B2M_OK; }
    CK(c, cudaMalloc((void**)&c->pk.d_ok, sizeof(int) * c->arena.nslots));
    CK(c, cudaMemsetAsync(c->pk.d_ok, 0, sizeof(int) * c->arena.nslots, st));
    c->pk.state = 1;
  }
  for (int slot : *out) c->pk.dirty[slot] = 0;
  return B2M_OK;
}

// ---------------- cache policy ----------------
int pick_victim(b2m_ctx* c, const std::vector<int>& in_use, bool allow_protected) {
  const int L = c->cfg.num_layers, E = c->cfg.num_experts;
  int best = -1, best_visits = INT32_MAX;
  // expert-major scan, strict '<' : same tie order as expert_dispatcher.cpp:233-252
  for (int e = 0; e < E; ++e) {
    for (int l = 0; l < L; ++l) {
      const int id = l * E + e;
      const Expert& x = c->experts[id];
      if (x.state != ST_RESIDENT || x.pinned || !x.backed()) continue;
      if (!allow_protected && c->protected_set.count(id)) continue;
      if (std::find(in_use.begin(), in_use.end(), id) != in_use.end()) continue;
      if (x.visits < best_visits) { best = id; best_visits = x.visits; }
    }
  }
  return best;
}

// B2M_CACHE_ACTIVATION_AWARE: expected time (in layer visits) to the next use of expert (l, e) seen from layer `cur`:
// layers until l runs again (decode visits layers in order; the layer in progress comes back after a full cycle) plus
// L * (1/f - 1) for the steps it is expected to sit out.  float32 throughout (oracle/policy_oracle.py mirrors it).
inline float next_use_score(int l, int cur, int L, float freq) {
  int d = (l - cur) % L;
  if (d <= 0) d += L;
  const float f = freq < 0.02f ? 0.02f : freq;
  return (float)d + (float)L * (1.0f / f - 1.0f);
}
int pick_victim_next_use(b2m_ctx* c, const std::vector<int>& in_use, bool allow_protected, float* score_out = nullptr) {
  const int L = c->cfg.num_layers, E = c->cfg.num_experts;
  int best = -1;
  float best_s = -1.0f;
  for (int l = 0; l < L; ++l) {            // layer-major scan, strict '>' : first maximum wins
    for (int e = 0; e < E; ++e) {
      const int id = l * E + e;
      const Expert& x = c->experts[id];
      if (x.state != ST_RESIDENT || x.pinned || !x.backed()) continue;
      if (!allow_protected && c->protected_set.count(id)) continue;
      if (std::find(in_use.begin(), in_use.end(), id) != in_use.end()) continue;
      const float s = next_use_score(l, c->cur_layer, L, x.freq);
      if (s > best_s) { best = id; best_s = s; }
    }
  }
  if (score_out) *score_out = best_s;
  return best;
}
int pick_victim_policy(b2m_ctx* c, const std::vector<int>& in_use, bool allow_protected) {
  return c->cfg.cache_policy == B2M_CACHE_ACTIVATION_AWARE ? pick_victim_next_use(c, in_use, allow_protected)
                                                            : pick_victim(c, in_use, allow_protected);
}

void evict(b2m_ctx* c, int id) {
  Expert& x = c->experts[id];
  const int slot = x.slot;
  x.state = ST_HOST;
  x.slot = -1;
  if (x.prefetched_unused) c->pf_win_wasted++;
  x.prefetched_unused = false;
  c->slots[slot].owner = -1;
  c->h_slot_of[id] = -1;
  c->row_dirty[id / c->cfg.num_experts] = 1;
  c->free_slots.push_back(slot);
  c->stats.evictions++;
}

int acquire_slot(b2m_ctx* c, const std::vector<int>& in_use, bool prefetch) {
  if (c->free_slots.empty()) {
    int v = pick_victim_policy(c, in_use, false);
    if (v < 0 && !prefetch) v = pick_victim_policy(c, in_use, true);   // overflow: on-demand beats protection
    if (v < 0) return -1;
    evict(c, v);
  }
  const int s = c->free_slots.back();
  c->free_slots.pop_back();
  return s;
}

// On-demand miss, the reference's way (GPUFetchFunc, expert_dispatcher.cpp:227-258): if the byte budget is used up
// (cache_sizes_ < byte_size) evict exactly ONE victim -- even while the budget arithmetic and the physical slots
// disagree (the reference charges hits too, see budget_units) -- then stage.  cfg.cache_policy == B2M_CACHE_SLOTS skips
// the budget test and evicts only when no physical slot is free.
int acquire_slot_on_demand(b2m_ctx* c, const std::vector<int>& in_use) {
  const bool ref_acct = c->cfg.cache_policy == B2M_CACHE_REFERENCE;
  if (c->free_slots.empty() || (ref_acct && c->budget_units < 1)) {
    int v = pick_victim_policy(c, in_use, false);
    if (v < 0) v = pick_victim_policy(c, in_use, true);   // overflow: on-demand beats protection
    if (v >= 0) {
      evict(c, v);
      c->budget_units += 1;                        // cache_sizes_ += evict_node->byte_size (:257)
    } else if (c->free_slots.empty()) {
      return -1;                                   // nothing evictable in this wave
    }                                              // (reference: assert(evict_node != nullptr); a free slot lets us go on)
  }
  const int s = c->free_slots.back();
  c->free_slots.pop_back();
  return s;
}

// Disk tier: stage a store-backed expert into its HBM slot.  The blob is cut into chunks; up to DISK_RING - 1 chunk reads are
// in flight at the reader (many threads, O_DIRECT) while the previous chunk is on its way to the device, so the disk, the
// staging memory and the host->device link work at the same time.  The host thread blocks for the reads (as the reference's
// ReadTensor does, archer_tensor_handle.cpp:189-201) but not for the copies.  A staging chunk is reused once the copy that
// read it has completed (event per chunk).
int copy_from_store(b2m_ctx* c, Expert& x, uint8_t* dst, cudaStream_t st, bool on_demand) {
  const size_t bytes = c->arena.shape.bytes;
  const size_t chunk = c->disk_chunk;
  const int nchunks = (int)((bytes + chunk - 1) / chunk);
  for (int b = 0; b < b2m_ctx::DISK_RING; ++b) {
    if (!c->disk_bounce[b]) CK(c, cudaHostAlloc((void**)&c->disk_bounce[b], chunk, cudaHostAllocDefault));
    if (!c->disk_ev[b]) CK(c, cudaEventCreateWithFlags(&c->disk_ev[b], cudaEventDisableTiming));
  }
  uint64_t tk[b2m_ctx::DISK_RING] = {0};
  bool tk_live[b2m_ctx::DISK_RING] = {false};
  int rc = B2M_OK;
  auto submit = [&](int ci) -> int {
    const int b = ci % b2m_ctx::DISK_RING;
    if (c->disk_ev_pending[b]) {
      CK(c, cudaEventSynchronize(c->disk_ev[b]));
      c->disk_ev_pending[b] = false;
    }
    const size_t off = (size_t)ci * chunk;
    int r = b2m_store_read_range_async(x.store, x.ids.data(), (int)x.ids.size(), off, std::min(chunk, bytes - off), c->disk_bounce[b],
                                       on_demand ? 1 : 0, &tk[b]);
    if (r) return fail(c, r, "disk tier: %s", b2m_store_last_error(x.store));
    tk_live[b] = true;
    return B2M_OK;
  };
  const int ahead = b2m_ctx::DISK_RING - 1;
  for (int ci = 0; ci < std::min(ahead, nchunks) && !rc; ++ci) rc = submit(ci);
  for (int ci = 0; ci < nchunks && !rc; ++ci) {
    const int b = ci % b2m_ctx::DISK_RING;
    const size_t off = (size_t)ci * chunk;
    const int r = b2m_store_wait(x.store, tk[b]);
    tk_live[b] = false;
    if (r) { rc = fail(c, r, "disk tier: %s", b2m_store_last_error(x.store)); break; }
    cudaError_t e = cudaMemcpyAsync(dst + off, c->disk_bounce[b], std::min(chunk, bytes - off), cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaEventRecord(c->disk_ev[b], st);
    if (e != cudaSuccess) { rc = fail(c, B2M_ECUDA, "disk tier copy: %s", cudaGetErrorString(e)); break; }
    c->disk_ev_pending[b] = true;
    if (ci + ahead < nchunks) rc = submit(ci + ahead);
  }
  for (int b = 0; b < b2m_ctx::DISK_RING; ++b)   // error path: no reader thread may still write into the staging ring
    if (tk_live[b]) b2m_store_wait(x.store, tk[b]);
  if (rc) return rc;
  c->stats.h2d_bytes += bytes;
  c->disk_bytes += bytes;
  return B2M_OK;
}

int issue_copy(b2m_ctx* c, int id, int slot, cudaStream_t st, bool do_copy) {
  Expert& x = c->experts[id];
  Slot& sl = c->slots[slot];
  if (sl.last_use_ev >= 0) CK(c, cudaStreamWaitEvent(st, c->ev_ring[sl.last_use_ev], 0));
  uint8_t* dst = c->arena.base + (size_t)slot * c->arena.slot_bytes;
  if (do_copy && x.host) {
    const size_t bytes = c->arena.shape.bytes;
    const size_t chunk = c->cfg.h2d_chunk_bytes > 0 ? (size_t)c->cfg.h2d_chunk_bytes : bytes;
    for (size_t off = 0; off < bytes; off += chunk)
      CK(c, cudaMemcpyAsync(dst + off, x.host + off, std::min(chunk, bytes - off), cudaMemcpyHostToDevice, st));
    c->stats.h2d_bytes += bytes;
  } else if (do_copy) {
    int r = copy_from_store(c, x, dst, st, st != c->prefetch_stream);
    if (r) { c->free_slots.push_back(slot); return r; }   // the expert stays on the store; its slot goes back
  }
  int r = pk_invalidate(c, slot, st);
  if (r) return r;
  if (!x.ready) CK(c, cudaEventCreateWithFlags(&x.ready, cudaEventDisableTiming));
  CK(c, cudaEventRecord(x.ready, st));
  x.ready_pending = true;
  x.state = ST_LOADING;
  x.slot = slot;
  sl.owner = id;
  c->h_slot_of[id] = slot;
  c->row_dirty[id / c->cfg.num_experts] = 1;
  return B2M_OK;
}

int pump(b2m_ctx* c) {
  // retire finished prefetches
  for (size_t i = 0; i < c->inflight.size();) {
    Expert& x = c->experts[c->inflight[i]];
    bool done = x.state != ST_LOADING;
    if (!done) {
      cudaError_t q = cudaEventQuery(x.ready);
      if (q == cudaSuccess) { x.state = ST_RESIDENT; done = true; }
      else if (q != cudaErrorNotReady) return fail(c, B2M_ECUDA, "cudaEventQuery: %s", cudaGetErrorString(q));
    }
    if (done) { c->inflight[i] = c->inflight.back(); c->inflight.pop_back(); } else ++i;
  }
  const int max_if = c->cfg.max_inflight_prefetch > 0 ? c->cfg.max_inflight_prefetch : 2;
  while ((int)c->inflight.size() < max_if && !c->pending.empty()) {
    const int id = c->pending.front();
    c->pending.pop_front();
    Expert& x = c->experts[id];
    if (x.state != ST_HOST) continue;
    const int slot = acquire_slot(c, c->last_active, true);
    if (slot < 0) { c->pending.clear(); break; }   // nothing evictable without hurting protected experts
    int r = issue_copy(c, id, slot, c->prefetch_stream, true);
    if (r) return r;
    x.prefetched_unused = true;
    c->inflight.push_back(id);
    c->stats.prefetch_issued++;
  }
  return B2M_OK;
}

int upload_row_if_dirty(b2m_ctx* c, int layer, cudaStream_t st) {
  if (!c->row_dirty[layer]) return B2M_OK;
  {
    // a dirty row while the stream is being captured would bake a copy from the reused pinned staging ring into the graph:
    // every replay would then upload whatever the ring holds at that time
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(st, &cs) != cudaSuccess) cudaGetLastError();   // (legacy stream beside a capture: not ours to judge)
    else if (cs != cudaStreamCaptureStatusNone)
      return fail(c, B2M_ESTATE, "layer %d's expert->slot row changed and the stream is capturing: run the step once eagerly "
                  "(all experts of the graph resident) before capturing it", layer);
  }
  const int E = c->cfg.num_experts;
  int* stage = c->h_stage + (size_t)c->stage_pos * E;
  c->stage_pos = (c->stage_pos + 1) % STAGE_RING;
  memcpy(stage, &c->h_slot_of[(size_t)layer * E], sizeof(int) * E);
  CK(c, cudaMemcpyAsync(c->d_slot_of + (size_t)layer * E, stage, sizeof(int) * E, cudaMemcpyHostToDevice, st));
  c->row_dirty[layer] = 0;
  return B2M_OK;
}

int check_layer(b2m_ctx* c, int layer) {
  if (!c) return B2M_EINVAL;
  if (layer < 0 || layer >= c->cfg.num_layers) return fail(c, B2M_EINVAL, "layer %d out of range", layer);
  return B2M_OK;
}

RouteParams base_route_params(b2m_ctx* c, int layer, const void* x, int T, int seq_len) {
  RouteParams p;
  memset(&p, 0, sizeof p);
  const b2m_config& f = c->cfg;
  p.x = x;
  p.gate_w = c->gate_w[layer];
  p.gate_dtype = f.gate_dtype;
  p.T = T; p.H = f.hidden; p.E = f.num_experts; p.k = f.top_k;
  p.dtype = f.dtype;
  p.router = f.router;
  p.logits_model_dtype = c->rk->model_dtype_logits;
  p.n_group = f.n_group; p.topk_group = f.topk_group; p.norm_topk_prob = f.norm_topk_prob;
  p.routed_scaling_factor = f.routed_scaling_factor;
  p.gate_bias = c->gate_bias[layer];
  p.seq_len = seq_len > 0 ? seq_len : T;
  p.expert_capacity = f.expert_capacity;
  p.scores = c->d_scores;
  p.logits_out = f.dtype == B2M_DTYPE_F32 ? nullptr : c->d_logits;
  p.topk_idx = c->d_topk_idx; p.topk_w = c->d_topk_w; p.row_of = c->d_row_of; p.perm_token = c->d_perm_token;
  p.counts = c->d_counts; p.offsets = c->d_offsets; p.chunk_counts = c->d_chunk_counts;
  p.xp = c->d_xp;
  p.ticket = c->d_ticket;
  p.err_flag = c->d_err;
  p.input_perm = c->input_perm[layer];
  return p;
}

void plan_gemm(b2m_ctx* c, int T) {
  c->cur_T = T;
  c->cur_nt_dn = pick_nt_model(c->cfg, T);
  // gate/up GEMM: at most 128-token tiles -- its two accumulators (gate and up) of a 256-token tile would need 256 fp32
  // registers per thread of a wgmma warpgroup
  c->cur_nt = pick_nt(T);
  c->cur_ksplit = pick_ksplit(c, T, c->cfg.hidden, c->cfg.inter, c->cfg.num_experts, c->cfg.top_k, c->cur_nt_dn);
  if (c->arena.shape.has_bias) c->cur_ksplit = 1;   // `+ fc2_bias` is applied once, in the epilogue of the whole-K product
  if (c->cfg.dtype == B2M_DTYPE_F32) c->cur_ksplit = 1;   // CUDA-core fp32 path: whole-K tiles
}

// same switch as b2m_common.cuh:pdl_enabled() (that header is device code; this file also builds against the host emulation)
bool pdl_enabled() { return sw().pdl; }


int route_launch_count(int T, const RouterKind& rk, bool fused_gate) {
  if (T == 0) return 0;
  if (T <= 256) return 2;
  return (rk.capacity ? 5 : 3) + (fused_gate ? 1 : 0);
}

// scores as router input: a router that ranks its logits cannot take them
int refuse_scores(b2m_ctx* c, int kind) {
  if (kind == 2 && c->rk->scales_inputs)
    return fail(c, B2M_EUNSUPPORTED, "%s router: takes logits (router_in_kind 0 or 1), not scores: it ranks the logits", c->rk->name);
  return B2M_OK;
}

}  // namespace

// =====================================================================================
extern "C" {

const char* b2m_last_error(const b2m_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }
int b2m_version(void) { return B2M_VERSION; }

int b2m_ctx_create(const b2m_config* cfg, b2m_ctx** out) { return b2m_ctx_create_ex(cfg, B2M_WEIGHTS_MODEL_DTYPE, out); }

int b2m_ctx_create_ex(const b2m_config* cfg, int weight_format, b2m_ctx** out) {
  if (!cfg || !out) return fail(nullptr, B2M_EINVAL, "null argument");
  if (cfg->struct_size != (int)sizeof(b2m_config))
    return fail(nullptr, B2M_EINVAL, "b2m_config size mismatch (%d vs %d)", cfg->struct_size, (int)sizeof(b2m_config));
  const WeightFormat* wf = nullptr;
  for (const WeightFormat& f : WEIGHT_FORMATS)
    if (f.id == weight_format) wf = &f;
  if (!wf) return fail(nullptr, B2M_EINVAL, "unknown weight format %d", weight_format);
  if (cfg->dtype == B2M_DTYPE_FP8_E4M3)
    return fail(nullptr, B2M_EUNSUPPORTED, "dtype %d (fp8): the reference's own torch::matmul has no Float8 kernel; bf16, f16 and f32 experts are supported", cfg->dtype);
  if (cfg->dtype != B2M_DTYPE_BF16 && cfg->dtype != B2M_DTYPE_F16 && cfg->dtype != B2M_DTYPE_F32) return fail(nullptr, B2M_EINVAL, "bad dtype");
  const size_t esize = cfg->dtype == B2M_DTYPE_F32 ? 4 : 2;
  if (cfg->num_layers < 1 || cfg->num_experts < 1 || cfg->num_experts > 256 || cfg->top_k < 1 || cfg->top_k > 8 ||
      cfg->top_k > cfg->num_experts || cfg->hidden < 64 || cfg->inter < 64 || cfg->hidden % 8 || cfg->inter % 8 ||
      cfg->max_tokens < 1)
    return fail(nullptr, B2M_EINVAL, "bad model dimensions");
  ExpertShape shape;
  if (!make_shape(cfg->expert_type, cfg->hidden, cfg->inter, wf->bits ? wf->bits : 8 * (int)esize, wf->grid_bytes, &shape))
    return fail(nullptr, B2M_EUNSUPPORTED, "expert_type %d is unknown (expert_module.h:13-18 defines 0..5)", cfg->expert_type);
  if (wf->a_src != AS_BF16) {   // a quantised format: three matrices per expert, decoded inside the tensor-core GEMMs
    if (cfg->dtype != wf->act_dtype)
      return fail(nullptr, B2M_EUNSUPPORTED, "%s weights need %s activations (model dtype), got dtype %d", wf->name,
                  wf->act_dtype == B2M_DTYPE_BF16 ? "bf16" : "f16", cfg->dtype);
    if (cfg->expert_type != B2M_EXPERT_MIXTRAL_MOE_DENSE_ACT_DENSE && cfg->expert_type != B2M_EXPERT_DEEPSEEK_MOE_DENSE_ACT_DENSE)
      return fail(nullptr, B2M_EUNSUPPORTED, "%s weights support Mixtral (4) and DeepSeek (5) experts, got expert_type %d",
                  wf->name, cfg->expert_type);
    if (cfg->hidden % wf->hi_multiple || cfg->inter % wf->hi_multiple)
      return fail(nullptr, B2M_EUNSUPPORTED, "%s weights need hidden and inter to be multiples of %d (scale blocks or groups, "
                  "128-row tiles), got %d / %d", wf->name, wf->hi_multiple, cfg->hidden, cfg->inter);
    if (cfg->gemm_impl == 1)
      return fail(nullptr, B2M_EUNSUPPORTED, "%s weights run on the tensor-core GEMMs only (gemm_impl 1 is the bf16 cross-check kernel)",
                  wf->name);
  }
  const RouterKind* rk = nullptr;
  for (const RouterKind& r : ROUTERS)
    if (r.id == cfg->router) rk = &r;
  if (!rk) return fail(nullptr, B2M_EINVAL, "bad router kind");
  if (rk->gate_up_down && cfg->expert_type != B2M_EXPERT_DEEPSEEK_MOE_DENSE_ACT_DENSE)
    return fail(nullptr, B2M_EINVAL, "%s router: experts are gate|up|down (expert_type %d), got expert_type %d", rk->name,
                B2M_EXPERT_DEEPSEEK_MOE_DENSE_ACT_DENSE, cfg->expert_type);
  if (rk->dtype16 && cfg->dtype != B2M_DTYPE_BF16 && cfg->dtype != B2M_DTYPE_F16)
    return fail(nullptr, B2M_EINVAL, "%s router: the model dtype must be bf16 or f16, got dtype %d", rk->name, cfg->dtype);
  if (rk->groups == GROUPS_NONE && (cfg->n_group != 1 || cfg->topk_group != 1))
    return fail(nullptr, B2M_EINVAL, "%s router: no group-limited routing (n_group=%d, topk_group=%d must be 1)", rk->name,
                cfg->n_group, cfg->topk_group);
  if (rk->groups == GROUPS_V3) {
    if (cfg->n_group < 1 || cfg->n_group > 32 || cfg->num_experts % cfg->n_group)
      return fail(nullptr, B2M_EINVAL, "%s router: n_group=%d must be in 1..32 and divide num_experts=%d", rk->name,
                  cfg->n_group, cfg->num_experts);
    if (cfg->num_experts / cfg->n_group < 2)
      return fail(nullptr, B2M_EINVAL, "%s router: a group needs at least 2 experts (top-2 group score), got %d", rk->name,
                  cfg->num_experts / cfg->n_group);
    if (cfg->topk_group < 1 || cfg->topk_group > cfg->n_group)
      return fail(nullptr, B2M_EINVAL, "%s router: topk_group=%d must be in 1..n_group=%d", rk->name, cfg->topk_group,
                  cfg->n_group);
  }
  if (rk->unscaled && cfg->routed_scaling_factor != 1.0f)
    return fail(nullptr, B2M_EINVAL, "%s router: weights are not scaled (routed_scaling_factor=%g must be 1.0)", rk->name,
                (double)cfg->routed_scaling_factor);
  if (rk->unnormalised && cfg->norm_topk_prob)
    return fail(nullptr, B2M_EINVAL, "%s router: weights are not normalised (norm_topk_prob=%d must be 0)", rk->name,
                cfg->norm_topk_prob);
  if (rk->needs_shared && cfg->shared_inter <= 0)
    return fail(nullptr, B2M_EINVAL, "%s router: every MoE layer has a shared expert (shared_inter=%d must be > 0)", rk->name,
                cfg->shared_inter);
  if (rk->top1 && cfg->top_k != 1) return fail(nullptr, B2M_EINVAL, "%s router needs top_k=1", rk->name);
  if (cfg->cache_policy < B2M_CACHE_REFERENCE || cfg->cache_policy > B2M_CACHE_ACTIVATION_AWARE) return fail(nullptr, B2M_EINVAL, "bad cache_policy");
  if (cfg->freq_alpha < 0.f || cfg->freq_alpha > 1.f) return fail(nullptr, B2M_EINVAL, "freq_alpha must be in [0,1]");

  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return fail(nullptr, B2M_ECUDA, "no CUDA device: %s -- this library has no CPU fallback", cudaGetErrorString(e));
  if (cfg->device < 0 || cfg->device >= ndev) return fail(nullptr, B2M_EINVAL, "device %d out of range", cfg->device);

  b2m_ctx* c = new (std::nothrow) b2m_ctx();
  if (!c) return fail(nullptr, B2M_ENOMEM, "out of host memory");
  c->cfg = *cfg;
  c->wf = wf;
  c->rk = rk;
  memset(&c->stats, 0, sizeof c->stats);
#define CKC(call)                                                                                     \
  do {                                                                                                \
    cudaError_t _e = (call);                                                                          \
    if (_e != cudaSuccess) {                                                                          \
      fail(nullptr, B2M_ECUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__); \
      b2m_ctx_destroy(c);                                                                             \
      return B2M_ECUDA;                                                                               \
    }                                                                                                 \
  } while (0)
  CKC(cudaSetDevice(cfg->device));
  cudaDeviceProp prop;
  CKC(cudaGetDeviceProperties(&prop, cfg->device));
  if (prop.major != 9 || prop.minor != 0) {
    fail(nullptr, B2M_EUNSUPPORTED, "device sm_%d%d: this library is built for sm_90a (H100) only", prop.major, prop.minor);
    b2m_ctx_destroy(c);
    return B2M_EUNSUPPORTED;
  }
  c->num_sms = prop.multiProcessorCount;
  c->total_mem = prop.totalGlobalMem;
  {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    CKC(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
    if (!fn || qres != cudaDriverEntryPointSuccess) {
      fail(nullptr, B2M_ECUDA, "cuTensorMapEncodeTiled not available in this driver");
      b2m_ctx_destroy(c);
      return B2M_ECUDA;
    }
    c->encode = (PFN_cuTensorMapEncodeTiled_v12000)fn;
  }
  const int L = cfg->num_layers, E = cfg->num_experts, H = cfg->hidden, I = cfg->inter, k = cfg->top_k;
  // ---- HBM slot arena: budget = ratio * total / expert bytes (memory_pool.cpp:150-158; expert_dispatcher.cpp:52-54)
  c->arena.shape = shape;
  c->arena.slot_bytes = shape.bytes;
  long long nslots = cfg->num_slots;
  if (nslots <= 0) {
    const double ratio = cfg->device_memory_ratio > 0 ? cfg->device_memory_ratio : 0.9;
    nslots = (long long)(ratio * (double)c->total_mem / (double)shape.bytes);
  }
  nslots = std::max<long long>(1, std::min<long long>(nslots, (long long)L * E));
  c->arena.nslots = (int)nslots;
  c->offload = nslots < (long long)L * E;
  CKC(cudaMalloc((void**)&c->arena.base, (size_t)nslots * shape.bytes));
  c->arena.owned = true;
  for (int m = 0; m < 3 && wf->a_src == AS_BF16; ++m) {   // (a quantised context has no 12-bit packed copy: pk.slot_bytes stays 0)
    c->pk.off[m] = c->pk.slot_bytes;
    c->pk.slot_bytes += packed_matrix_bytes((int)pk_matrix_rows(shape, m), (int)pk_matrix_cols(shape, m));
  }
  c->pk.dirty.assign((size_t)nslots, PK_WRITTEN);
  const bool tc = cfg->dtype != B2M_DTYPE_F32;   // fp32 experts run on the CUDA-core path (f32_path.cu): no TMA maps
  int r = tc ? build_arena_maps(c, &c->arena) : B2M_OK;
  if (r) { g_create_error = c->err; b2m_ctx_destroy(c); return r; }
  if (cfg->shared_inter > 0) {
    ExpertShape ss;
    make_shape(B2M_EXPERT_DEEPSEEK_MOE_DENSE_ACT_DENSE, H, cfg->shared_inter, 8 * (int)esize, nullptr, &ss);
    c->shared_arena.shape = ss;
    c->shared_arena.slot_bytes = ss.bytes;
    c->shared_arena.nslots = L;
    CKC(cudaMalloc((void**)&c->shared_arena.base, (size_t)L * ss.bytes));
    c->shared_arena.owned = true;
    r = tc ? build_arena_maps(c, &c->shared_arena) : B2M_OK;
    if (r) { g_create_error = c->err; b2m_ctx_destroy(c); return r; }
    c->shared_registered.assign(L, 0);
  }
  c->experts.assign((size_t)L * E, Expert());
  c->slots.assign((size_t)nslots, Slot());
  for (int s = (int)nslots - 1; s >= 0; --s) c->free_slots.push_back(s);
  c->h_slot_of.assign((size_t)L * E, -1);
  c->row_dirty.assign(L, 1);
  c->gate_w.assign(L, nullptr);
  c->gate_bias.assign(L, nullptr);
  c->input_perm.assign(L, nullptr);
  c->shared_gate_w.assign(L, nullptr);
  CKC(cudaMalloc((void**)&c->d_slot_of, sizeof(int) * L * E));
  CKC(cudaMemset(c->d_slot_of, 0xff, sizeof(int) * L * E));
  CKC(cudaHostAlloc((void**)&c->h_stage, sizeof(int) * STAGE_RING * E, cudaHostAllocDefault));
  CKC(cudaHostAlloc((void**)&c->h_counts, sizeof(int) * (E + 1), cudaHostAllocDefault));
  // ---- workspace
  const int T = cfg->max_tokens;
  const size_t R = (size_t)T * k;
  c->cap_T = T;
  c->cap_R = (int)R;
  CKC(cudaMalloc((void**)&c->d_topk_idx, sizeof(int) * R));
  CKC(cudaMalloc((void**)&c->d_topk_w, sizeof(float) * R));
  CKC(cudaMalloc((void**)&c->d_row_of, sizeof(int) * R));
  CKC(cudaMalloc((void**)&c->d_perm_token, sizeof(int) * R));
  CKC(cudaMalloc((void**)&c->d_counts, sizeof(int) * E));
  CKC(cudaMalloc((void**)&c->d_offsets, sizeof(int) * (E + 1)));
  CKC(cudaMemset(c->d_offsets, 0, sizeof(int) * (E + 1)));
  CKC(cudaMalloc((void**)&c->d_offsets_src, sizeof(int) * (E + 1)));
  CKC(cudaMalloc((void**)&c->d_ticket, 2 * sizeof(int)));       // [0] CTA arrival counter, [1] "row maps published" word (ep_fused)
  CKC(cudaMemset(c->d_ticket, 0, 2 * sizeof(int)));
  CKC(cudaMalloc((void**)&c->d_gbar, 2 * sizeof(int)));
  CKC(cudaMemset(c->d_gbar, 0, 2 * sizeof(int)));
  CKC(cudaMalloc((void**)&c->d_err, sizeof(int)));
  CKC(cudaMemset(c->d_err, 0, sizeof(int)));
  CKC(cudaHostAlloc((void**)&c->h_err, sizeof(int), cudaHostAllocDefault));
  CKC(cudaMalloc((void**)&c->d_look, sizeof(int) * E));
  CKC(cudaMemset(c->d_look, 0, sizeof(int) * E));
  CKC(cudaHostAlloc((void**)&c->h_look, sizeof(int) * E, cudaHostAllocDefault));
  CKC(cudaMalloc((void**)&c->d_dest_of, sizeof(int) * R));
  CKC(cudaMalloc((void**)&c->d_chunk_counts, sizeof(int) * ((size_t)(T + 31) / 32) * E));
  CKC(cudaMalloc((void**)&c->d_scores, sizeof(float) * (size_t)T * E));
  CKC(cudaMalloc((void**)&c->d_logits, sizeof(float) * (size_t)T * E));
  CKC(cudaMalloc(&c->d_xp, R * H * esize));
  CKC(cudaMalloc(&c->d_hmid, R * I * esize));
  CKC(cudaMalloc((void**)&c->d_y, R * H * sizeof(float)));
  CKC(cudaMemset(c->d_xp, 0, R * H * esize));
  CKC(cudaMemset(c->d_hmid, 0, R * I * esize));
  if (cfg->shared_inter > 0) {
    CKC(cudaMalloc(&c->d_hmid_s, (size_t)T * cfg->shared_inter * esize));
    CKC(cudaMemset(c->d_hmid_s, 0, (size_t)T * cfg->shared_inter * esize));
    CKC(cudaMalloc((void**)&c->d_y_s, (size_t)T * H * sizeof(float)));
    if (rk->shared_gate) CKC(cudaMalloc(&c->d_shared_gate, (size_t)T * esize));
  }
  for (int i = 0; tc && i < 5; ++i) {
    r = build_act_map(c, &c->tm_xp[i], c->d_xp, H, (int)R, NT_LIST[i]);
    if (!r) r = build_act_map(c, &c->tm_hmid[i], c->d_hmid, I, (int)R, NT_LIST[i]);
    if (!r && cfg->shared_inter > 0) r = build_act_map(c, &c->tm_hmid_s[i], c->d_hmid_s, cfg->shared_inter, T, NT_LIST[i]);
    if (r) { g_create_error = c->err; b2m_ctx_destroy(c); return r; }
  }
  int lo = 0, hi = 0;
  CKC(cudaDeviceGetStreamPriorityRange(&lo, &hi));
  CKC(cudaStreamCreateWithPriority(&c->fetch_stream, cudaStreamNonBlocking, hi));
  CKC(cudaStreamCreateWithPriority(&c->prefetch_stream, cudaStreamNonBlocking, lo));
  for (int i = 0; i < EVENT_RING; ++i) CKC(cudaEventCreateWithFlags(&c->ev_ring[i], cudaEventDisableTiming));
  if (const char* e = getenv("B2M_DISK_CHUNK_BYTES")) {   // disk tier staging chunk (a multiple of 4096 keeps the reads O_DIRECT-aligned)
    const long long v = atoll(e);
    if (v >= 4096) c->disk_chunk = ((size_t)v + 4095) & ~(size_t)4095;
  }
  CKC(cudaStreamCreateWithFlags(&c->shared_stream, cudaStreamNonBlocking));
  CKC(cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming));
  CKC(cudaEventCreateWithFlags(&c->ev_join, cudaEventDisableTiming));
  c->stats.slots = (uint64_t)nslots;
  c->stats.slot_bytes = shape.bytes;
  c->budget_units = nslots;
#undef CKC
  *out = c;
  return B2M_OK;
}

int b2m_ctx_destroy(b2m_ctx* c) {
  if (!c) return B2M_OK;
  cudaDeviceSynchronize();
  if (c->arena.owned && c->arena.base) cudaFree(c->arena.base);
  if (c->shared_arena.owned && c->shared_arena.base) cudaFree(c->shared_arena.base);
  if (c->pk.base) cudaFree(c->pk.base);
  if (c->pk.d_ok) cudaFree(c->pk.d_ok);
  void* bufs[] = {c->d_slot_of, c->d_topk_idx, c->d_topk_w, c->d_row_of, c->d_perm_token, c->d_counts, c->d_offsets,
                  c->d_chunk_counts, c->d_offsets_src, c->d_ticket, c->d_gbar, c->d_err, c->d_look, c->d_tl, c->d_dest_of, c->d_scores, c->d_logits, c->d_xp, c->d_hmid, c->d_y, c->d_hmid_s, c->d_y_s, c->d_shared_gate};
  for (void* b : bufs) if (b) cudaFree(b);
  for (int r = 0; r < c->p2p.nranks; ++r)
    if (c->p2p.peer_base[r] && r != c->p2p.rank) cudaIpcCloseMemHandle(c->p2p.peer_base[r]);
  if (c->p2p.base) cudaFree(c->p2p.base);
  if (c->p2p.d_hmid) cudaFree(c->p2p.d_hmid);
  if (c->p2p.local_ctr) cudaFree(c->p2p.local_ctr);
  if (c->h_stage) cudaFreeHost(c->h_stage);
  if (c->h_counts) cudaFreeHost(c->h_counts);
  if (c->h_err) cudaFreeHost(c->h_err);
  if (c->h_look) cudaFreeHost(c->h_look);
  {
    void* tb[] = {c->tr.seq, c->tr.lib, c->tr.pred, c->tr.hint, c->tr.access, c->tr.winner};
    for (void* b : tb) if (b) cudaFree(b);
    if (c->tr.h_hint) cudaFreeHost(c->tr.h_hint);
  }
  for (auto& x : c->experts) if (x.ready) cudaEventDestroy(x.ready);
  if (c->fetch_stream) cudaStreamDestroy(c->fetch_stream);
  if (c->prefetch_stream) cudaStreamDestroy(c->prefetch_stream);
  if (c->shared_stream) cudaStreamDestroy(c->shared_stream);
  if (c->ev_fork) cudaEventDestroy(c->ev_fork);
  if (c->ev_join) cudaEventDestroy(c->ev_join);
  for (int i = 0; i < EVENT_RING; ++i) if (c->ev_ring[i]) cudaEventDestroy(c->ev_ring[i]);
  for (int b = 0; b < b2m_ctx::DISK_RING; ++b) {
    if (c->disk_bounce[b]) cudaFreeHost(c->disk_bounce[b]);
    if (c->disk_ev[b]) cudaEventDestroy(c->disk_ev[b]);
  }
  delete c;
  return B2M_OK;
}

int b2m_register_expert(b2m_ctx* c, int layer, int expert, const void* host_blob, size_t bytes) {
  int r = check_layer(c, layer);
  if (r) return r;
  if (expert < 0 || expert >= c->cfg.num_experts) return fail(c, B2M_EINVAL, "expert %d out of range", expert);
  if (host_blob && bytes != c->arena.shape.bytes)
    return fail(c, B2M_EINVAL, "expert blob is %zu bytes, expected %zu", bytes, c->arena.shape.bytes);
  Expert& x = c->experts[(size_t)layer * c->cfg.num_experts + expert];
  x.host = reinterpret_cast<const uint8_t*>(host_blob);
  x.store = nullptr;
  x.ids.clear();
  if (x.state == ST_UNREGISTERED) x.state = ST_HOST;
  return B2M_OK;
}

int b2m_register_expert_on_store(b2m_ctx* c, int layer, int expert, b2m_store* store, const uint32_t* ids, int n) {
  int r = check_layer(c, layer);
  if (r) return r;
  if (expert < 0 || expert >= c->cfg.num_experts) return fail(c, B2M_EINVAL, "expert %d out of range", expert);
  if (!store || !ids || n < 1) return fail(c, B2M_EINVAL, "b2m_register_expert_on_store needs a store and the expert's tensor ids");
  uint64_t total = 0;
  r = b2m_store_blob_bytes(store, ids, n, &total);
  if (r) return fail(c, r, "disk tier: %s", b2m_store_last_error(store));
  if (total != c->arena.shape.bytes)
    return fail(c, B2M_EINVAL, "the expert's tensors hold %llu bytes on the store, expected %zu", (unsigned long long)total,
                c->arena.shape.bytes);
  Expert& x = c->experts[(size_t)layer * c->cfg.num_experts + expert];
  x.host = nullptr;
  x.store = store;
  x.ids.assign(ids, ids + n);
  if (x.state == ST_UNREGISTERED) x.state = ST_HOST;
  return B2M_OK;
}

int b2m_register_shared(b2m_ctx* c, int layer, const void* host_blob, size_t bytes) {
  int r = check_layer(c, layer);
  if (r) return r;
  if (c->cfg.shared_inter <= 0) return fail(c, B2M_ESTATE, "context has no shared experts");
  if (host_blob) {
    if (bytes != c->shared_arena.shape.bytes)
      return fail(c, B2M_EINVAL, "shared blob is %zu bytes, expected %zu", bytes, c->shared_arena.shape.bytes);
    CK(c, cudaMemcpy(c->shared_arena.base + (size_t)layer * c->shared_arena.slot_bytes, host_blob, bytes, cudaMemcpyHostToDevice));
  }
  c->shared_registered[layer] = 1;
  return B2M_OK;
}

int b2m_set_gate(b2m_ctx* c, int layer, const void* dev_gate_weight) {
  int r = check_layer(c, layer);
  if (r) return r;
  c->gate_w[layer] = dev_gate_weight;
  return B2M_OK;
}

int b2m_set_gate_bias(b2m_ctx* c, int layer, const float* dev_bias) {
  int r = check_layer(c, layer);
  if (r) return r;
  if (!c->rk->gate_bias)
    return fail(c, B2M_EINVAL, "b2m_set_gate_bias: only a %s router has a correction bias, this context's router is %s",
                routers_with(&RouterKind::gate_bias).c_str(), c->rk->name);
  if (!dev_bias) return fail(c, B2M_EINVAL, "b2m_set_gate_bias: dev_bias is null");
  c->gate_bias[layer] = dev_bias;
  return B2M_OK;
}

int b2m_set_shared_gate(b2m_ctx* c, int layer, const void* dev_w) {
  int r = check_layer(c, layer);
  if (r) return r;
  if (!c->rk->shared_gate)
    return fail(c, B2M_EINVAL, "b2m_set_shared_gate: only a %s router has a shared-expert gate, this context's router is %s",
                routers_with(&RouterKind::shared_gate).c_str(), c->rk->name);
  if (c->cfg.shared_inter <= 0) return fail(c, B2M_EINVAL, "b2m_set_shared_gate: the context has no shared experts (shared_inter = 0)");
  if (!dev_w) return fail(c, B2M_EINVAL, "b2m_set_shared_gate: dev_w is null");
  c->shared_gate_w[layer] = dev_w;
  return B2M_OK;
}

int b2m_set_input_perm(b2m_ctx* c, int layer, const uint16_t* dev_perm) {
  int r = check_layer(c, layer);
  if (r) return r;
  if (c->rk->scales_inputs)
    return fail(c, B2M_EUNSUPPORTED, "b2m_set_input_perm: input permutations are not available with the %s router", c->rk->name);
  if (c->wf->id != B2M_WEIGHTS_INT4_G128_F16)
    return fail(c, B2M_EUNSUPPORTED, "b2m_set_input_perm: input permutations (act-order GPTQ) need a B2M_WEIGHTS_INT4_G128_F16 "
                "context");
  c->input_perm[layer] = dev_perm;
  return B2M_OK;
}

int b2m_host_pin(b2m_ctx* c, void* host_ptr, size_t bytes) {
  if (!c || !host_ptr) return B2M_EINVAL;
  CK(c, cudaHostRegister(host_ptr, bytes, cudaHostRegisterDefault));
  return B2M_OK;
}
int b2m_host_unpin(b2m_ctx* c, void* host_ptr) {
  if (!c || !host_ptr) return B2M_EINVAL;
  CK(c, cudaHostUnregister(host_ptr));
  return B2M_OK;
}

int b2m_make_resident(b2m_ctx* c, int layer, int expert, int flags, void* stream) {
  int r = check_layer(c, layer);
  if (r) return r;
  if (expert < 0 || expert >= c->cfg.num_experts) return fail(c, B2M_EINVAL, "expert %d out of range", expert);
  const int id = layer * c->cfg.num_experts + expert;
  Expert& x = c->experts[id];
  const bool no_copy = (flags & 2) != 0;
  if (x.state == ST_UNREGISTERED) {
    if (!no_copy) return fail(c, B2M_ESTATE, "expert (%d,%d) is not registered", layer, expert);
    x.state = ST_HOST;
  }
  if (x.state == ST_HOST) {
    if (!no_copy && !x.backed()) return fail(c, B2M_ESTATE, "expert (%d,%d) has no host blob", layer, expert);
    std::vector<int> none;
    const int slot = acquire_slot(c, none, false);
    if (slot < 0) return fail(c, B2M_ENOMEM, "no evictable HBM slot for expert (%d,%d)", layer, expert);
    r = issue_copy(c, id, slot, c->fetch_stream, !no_copy);
    if (r) return r;
    c->budget_units -= 1;   // the expert occupies budget like one staged by a dispatch
  }
  if (x.state == ST_LOADING) {
    CK(c, cudaEventSynchronize(x.ready));
    x.state = ST_RESIDENT;
    x.ready_pending = false;
  }
  if (flags & 1) x.pinned = true;
  if (!x.backed()) x.pinned = true;
  if (no_copy) return pk_invalidate(c, x.slot, (cudaStream_t)stream);   // the caller fills the slot next
  return B2M_OK;
}

int b2m_expert_dev_ptr(b2m_ctx* c, int layer, int expert, void** dev_ptr) {
  int r = check_layer(c, layer);
  if (r) return r;
  if (expert < 0 || expert >= c->cfg.num_experts || !dev_ptr) return fail(c, B2M_EINVAL, "bad argument");
  const Expert& x = c->experts[(size_t)layer * c->cfg.num_experts + expert];
  *dev_ptr = x.slot >= 0 ? c->arena.base + (size_t)x.slot * c->arena.slot_bytes : nullptr;
  return pk_invalidate(c, x.slot, 0);   // a writable view: the slot may change before the next forward
}

int b2m_shared_dev_ptr(b2m_ctx* c, int layer, void** dev_ptr) {
  int r = check_layer(c, layer);
  if (r) return r;
  if (c->cfg.shared_inter <= 0 || !dev_ptr) return fail(c, B2M_ESTATE, "context has no shared experts");
  *dev_ptr = c->shared_arena.base + (size_t)layer * c->shared_arena.slot_bytes;
  return B2M_OK;
}

int b2m_ws_ptr(b2m_ctx* c, int which, void** p) {
  if (!c || !p) return B2M_EINVAL;
  switch (which) {
    case B2M_WS_TOPK_IDX: *p = c->d_topk_idx; break;
    case B2M_WS_TOPK_W: *p = c->d_topk_w; break;
    case B2M_WS_ROW_OF: *p = c->d_row_of; break;
    case B2M_WS_PERM_TOKEN: *p = c->d_perm_token; break;
    case B2M_WS_COUNTS: *p = c->d_counts; break;
    case B2M_WS_OFFSETS: *p = c->d_offsets; break;
    case B2M_WS_XP: *p = c->d_xp; break;
    case B2M_WS_HMID: *p = c->d_hmid; break;
    case B2M_WS_Y: *p = c->d_y; break;
    case B2M_WS_SCORES: *p = c->d_scores; break;
    case B2M_WS_LOGITS: *p = c->d_logits; break;
    case B2M_WS_SHARED_GATE:
      if (!c->d_shared_gate) return fail(c, B2M_ESTATE, "workspace %d: the context has no gated shared expert", which);
      *p = c->d_shared_gate;
      break;
    case B2M_WS_Y_SHARED:
      if (!c->d_y_s) return fail(c, B2M_ESTATE, "workspace %d: the context has no shared experts", which);
      *p = c->d_y_s;
      break;
    default: return fail(c, B2M_EINVAL, "unknown workspace id %d", which);
  }
  return B2M_OK;
}

// ------------------------------------------------------------------------------------
static EpParams ep_p2p_params(b2m_ctx* c);
static EpParams ep_p2p_params_direct(b2m_ctx* c);
static int route_impl(b2m_ctx* c, int layer, const void* x, const void* router_in, int kind, int in_dtype, int T,
                      int seq_len, void* stream, bool ep_dispatch);

int b2m_route(b2m_ctx* c, int layer, const void* x, const void* router_in, int kind, int in_dtype, int T, int seq_len,
              void* stream) {
  return route_impl(c, layer, x, router_in, kind, in_dtype, T, seq_len, stream, false);
}

static int route_impl(b2m_ctx* c, int layer, const void* x, const void* router_in, int kind, int in_dtype, int T,
                      int seq_len, void* stream, bool ep_dispatch) {
  int r = check_layer(c, layer);
  if (r) return r;
  if (T < 0 || T > c->cap_T) return fail(c, B2M_EINVAL, "T=%d exceeds workspace capacity %d", T, c->cap_T);
  if (!x && T > 0) return fail(c, B2M_EINVAL, "x is null");
  cudaStream_t st = (cudaStream_t)stream;
  RouteParams p = base_route_params(c, layer, x, T, seq_len);
  if (kind == 0) {
    if (c->cfg.dtype == B2M_DTYPE_F32)
      return fail(c, B2M_EUNSUPPORTED, "fp32 contexts take router logits / scores (or a mask): the fused gate kernel reads 16-bit activations");
    if (!p.gate_w) return fail(c, B2M_ESTATE, "layer %d has no gate weight (b2m_set_gate) and no router input", layer);
  } else {
    // no tokens, nothing to read: an expert-parallel rank with an empty batch hands over an empty (null) router input
    if (!router_in && T > 0) return fail(c, B2M_EINVAL, "router_in is null");
    p.logits = router_in;
    p.logits_dtype = in_dtype;
    p.logits_are_scores = (kind == 2);
    if (kind == 2 && in_dtype != B2M_DTYPE_F32) return fail(c, B2M_EINVAL, "scores must be fp32");
    r = refuse_scores(c, kind);
    if (r) return r;
  }
  p.scale_rows = c->rk->scales_inputs;   // the routing weight scales the expert's input row
  if (c->rk->capacity && (p.seq_len <= 0 || T % p.seq_len))
    return fail(c, B2M_EINVAL, "T=%d is not a multiple of seq_len=%d", T, p.seq_len);
  if (c->rk->gate_bias && !p.gate_bias)
    return fail(c, B2M_ESTATE, "layer %d has no correction bias (b2m_set_gate_bias)", layer);
  plan_gemm(c, T);
  if (c->cur_ksplit > 1) { p.y_zero = c->d_y; p.y_zero_elems = (size_t)T * c->cfg.top_k * c->cfg.hidden; }
  // small batches, all experts resident: let the last gate/top-k CTA publish the offsets so that the gate/up GEMM can be
  // launched with a programmatic edge behind the permute kernel and stream weights while rows are still being gathered
  const bool k3_early = sw().early_k3;
  // Not with B2M_PDL=1: with a programmatic edge on EVERY kernel the permute kernel may start before the gate/top-k kernel
  // has finished, so a GEMM that reads offsets/slot_of before its own griddepcontrol.wait could see the previous layer's
  // tables.  Pre-wait reads may only touch data older than the predecessor's own launch.
  c->k3_early_ok = k3_early && !pdl_enabled() && T >= 1 && T <= 256 && !c->rk->capacity && !ep_dispatch &&
                   !c->offload && !c->ep_mode && c->cfg.gemm_impl != 1;
  p.offsets_early = c->k3_early_ok ? 1 : 0;
  const bool rows_by_gate = sw().rows_by_gate;
  p.rows_by_gate = (c->k3_early_ok && rows_by_gate) ? 1 : 0;
  if (ep_dispatch) {
    if (T > 256 || T < 1) return fail(c, B2M_EINVAL, "fused route+dispatch handles 1..256 tokens per rank (got %d)", T);
    p.ep_dispatch = 1;
    p.tl = c->tl_next;
    p.ep = c->ep_direct_next ? ep_p2p_params_direct(c) : ep_p2p_params(c);
    if (c->ep_direct_next && sw().ep_l2pf_mb > 0 && !pdl_enabled()) p.pdl_edge = 1;   // lets the gate/up GEMM's CTAs arrive (and prefetch) early
    if (c->ep_direct_next) p.ep_fused = 1;   // one launch: gate/top-k + row claim (remote atomics) + row stores + signal
    p.y_zero = nullptr;        // the regroup kernel (direct mode: the owner's gate/up GEMM) clears the accumulator
  }
  CK(c, launch_route(p, st));
  c->stats.kernel_launches += route_launch_count(T, *c->rk, kind == 0) - (p.ep_fused ? 1 : 0);
  c->ep_fused_last = p.ep_fused != 0;
  c->last_counts_valid = false;
  // router-logit driven prefetch: the next layer's router applied to THIS layer's input predicts which experts the next
  // layer will want; the counts ride back with this layer's own counts (b2m_run_experts reads both in one synchronisation).
  // DeepSeek-V3 predicts with the next layer's bias too (top-k of raw logits is not its choice); no bias, no prediction.
  c->look_pending = false;
  const int nxt = (layer + 1) % c->cfg.num_layers;
  if (c->cfg.lookahead_prefetch && c->offload && !c->ep_mode && T >= 1 && T <= 256 && c->cfg.dtype != B2M_DTYPE_F32 &&
      c->cfg.num_layers > 1 && c->gate_w[nxt] && (!c->rk->gate_bias || c->gate_bias[nxt])) {
    RouteParams q = p;
    q.gate_w = c->gate_w[nxt];
    q.gate_bias = c->gate_bias[nxt];
    q.logits = nullptr;
    CK(c, cudaMemsetAsync(c->d_look, 0, sizeof(int) * c->cfg.num_experts, st));
    CK(c, launch_lookahead_counts(q, c->d_look, st));
    c->stats.kernel_launches += 1;
    c->look_pending = true;
  }
  return B2M_OK;
}

int b2m_route_from_mask(b2m_ctx* c, int layer, const void* x, const uint8_t* mask, int T, void* stream) {
  int r = check_layer(c, layer);
  if (r) return r;
  if (T < 0 || T > c->cap_T) return fail(c, B2M_EINVAL, "T=%d exceeds workspace capacity %d", T, c->cap_T);
  cudaStream_t st = (cudaStream_t)stream;
  RouteParams p = base_route_params(c, layer, x, T, T);
  p.scores = nullptr;
  p.logits_out = nullptr;
  c->k3_early_ok = false;
  plan_gemm(c, T);
  if (c->cur_ksplit > 1) { p.y_zero = c->d_y; p.y_zero_elems = (size_t)T * c->cfg.top_k * c->cfg.hidden; }
  CK(c, launch_route_from_mask(p, mask, st));
  c->stats.kernel_launches += T == 0 ? 0 : (T <= 256 ? 2 : 4);
  c->last_counts_valid = false;
  return B2M_OK;
}

static int launch_expert_gemms(b2m_ctx* c, Arena& a, const GemmParams& base, const CUtensorMap& tm_b_up,
                               const CUtensorMap& tm_b_down, const void* b_up, int ldb_up, const void* b_down,
                               void* hmid, float* y, int nt, int nt_dn, int ksplit, cudaStream_t st, int phases = 3,
                               int T_hint = -1) {
  // several token tiles per expert are likely: tensor-bound regime
  const bool T_hint_large = (T_hint >= 0 ? T_hint : c->cur_T) > 128;
  const b2m_config& f = c->cfg;
  const ExpertShape& s = a.shape;
  GemmParams up = base;
  up.M = s.I; up.K = s.H; up.ksplit = 1; up.epi = EPI_ACT16; up.act = s.act;
  up.mimic = f.numerics == B2M_NUMERICS_REFERENCE; up.out = hmid; up.ld_out = s.I;
  GemmParams dn = base;
  dn.M = s.H; dn.K = s.I; dn.ksplit = ksplit; dn.epi = EPI_LINEAR_F32; dn.act = ACT_NONE; dn.mimic = 0;
  dn.out = y; dn.ld_out = s.H;
  const size_t esz = f.dtype == B2M_DTYPE_F32 ? 4 : 2;
  if (s.has_bias) {
    up.bias_base = dn.bias_base = a.base;
    up.bias_slot_elems = dn.bias_slot_elems = a.slot_bytes / esz;
    up.bias_off = s.off_bias1 / esz;
    dn.bias_off = s.off_bias2 / esz;
    dn.ksplit = 1;
    dn.mimic = up.mimic;     // round(matmul) + bias -> round happens here; the combine's rounding is then the identity
  }
  if (f.dtype == B2M_DTYPE_F32) {
    // fp32 experts: CUDA-core fp32 FMA path (f32_path.cu); whole-K tiles, fp32 intermediate
    const size_t slot_elems = a.slot_bytes / 4;
    dn.ksplit = 1;
    if (phases & 1)
      CK(c, launch_grouped_gemm_f32(a.base, slot_elems, s.off_gate / 4, s.off_up / 4, b_up, ldb_up, up, s.dual, c->num_sms, st));
    if (phases & 2)
      CK(c, launch_grouped_gemm_f32(a.base, slot_elems, s.off_down / 4, s.off_down / 4, b_down, s.I, dn, false, c->num_sms, st));
  } else if (f.gemm_impl == 1) {
    const size_t slot_elems = a.slot_bytes / 2;
    if (phases & 1)
      CK(c, launch_grouped_gemm_simt(f.dtype, a.base, slot_elems, s.off_gate / 2, s.off_up / 2, b_up, ldb_up, up, s.dual, st));
    dn.ksplit = 1;
    if (phases & 2)
      CK(c, launch_grouped_gemm_simt(f.dtype, a.base, slot_elems, s.off_down / 2, s.off_down / 2, b_down, s.I, dn, false, st));
  } else {
    // tensor-bound regime (several 128-token tiles per expert): a 2-CTA cluster variant that multicasts the weight tiles is
    // compiled only with -DB2M_ENABLE_MC2 (then selected with B2M_MC2=1), not part of the default library (L2 already
    // de-duplicates the two CTAs' requests)
#ifdef B2M_ENABLE_MC2
    static const bool mc2_on = getenv("B2M_MC2") && getenv("B2M_MC2")[0] == '1';
    const bool mc2 = mc2_on && nt == 128 && T_hint_large;
#else
    const bool mc2 = false;
#endif
    // packed weights (decode-sized tiles of the routed experts); this call's gate/up launch first packs the stale slots it
    // was handed (base.pack_slots), the down launch never packs
    dn.pack_n = 0;
    if (&a == &c->arena && c->wf->a_src != AS_BF16) {   // (shared experts are always in the model dtype)
      up.a_src = dn.a_src = c->wf->a_src;
      up.grid0 = a.base + s.grid_gate;
      up.grid1 = a.base + s.grid_up;
      dn.grid0 = dn.grid1 = a.base + s.grid_down;
      up.grid_slot_bytes = dn.grid_slot_bytes = a.slot_bytes;
    }
    if (&a == &c->arena && c->pk.state == 1) {
      up.pk_ok = dn.pk_ok = c->pk.d_ok;
      up.pk_slot_bytes = dn.pk_slot_bytes = c->pk.slot_bytes;
      up.pk_bit0 = 0; up.pk_bit1 = 1;
      up.pk_a0 = c->pk.base + c->pk.off[0];
      up.pk_a1 = c->pk.base + c->pk.off[1];
      dn.pk_bit0 = dn.pk_bit1 = 2;
      dn.pk_a0 = dn.pk_a1 = c->pk.base + c->pk.off[2];
      up.pack_ok = c->pk.d_ok;
      up.pack_dst = c->pk.base;
      up.pack_src = a.base;
      up.pack_src_slot_bytes = a.slot_bytes;
      up.pack_nmat = 3;
      const size_t src_off[3] = {s.off_gate, s.off_up, s.off_down};
      for (int m = 0; m < 3; ++m) {
        up.pack_src_off[m] = src_off[m];
        up.pack_dst_off[m] = c->pk.off[m];
        up.pack_rows[m] = (int)pk_matrix_rows(s, m);
        up.pack_cols[m] = (int)pk_matrix_cols(s, m);
      }
    } else {
      up.pack_n = 0;
    }
    if (up.pack_n > 0) c->stats.kernel_launches += 2;   // pack + publish flags
    const bool pdl_k3 = sw().pdl_k3;
    up.pdl_edge = (pdl_k3 && !T_hint_large) ? 1 : 0;
    up.early_a = (c->k3_early_ok && &a == &c->arena && phases == 3) ? 1 : 0;   // routed experts right behind the permute kernel
    // decode regime, routed experts, both phases in one call: ONE persistent kernel (gate/up phase, grid barrier, down phase)
    // -- the down GEMM's set-up and first pipeline fill no longer sit on the critical path between two kernels
#ifdef B2M_ENABLE_FUSED_FFN
    if (sw().fused_ffn && phases == 3 && !T_hint_large && !mc2 && &a == &c->arena && s.dual && nt == nt_dn && nt <= 128 &&
        !pdl_enabled()) {
      dn.dual_m = 0;
      dn.early_a = 1;
      dn.stream_k = (sw().streamk && dn.ksplit > 1) ? 1 : 0;
      CK(c, launch_fused_ffn(f.dtype, nt, a.tm_gate, a.tm_up, tm_b_up, a.tm_down, tm_b_down, up, dn, c->num_sms, c->num_sms,
                             c->d_gbar, st));
      c->stats.kernel_launches += 1;
      return B2M_OK;
    }
#endif
    if (phases & 1) {
#ifdef B2M_ENABLE_MC2
      if (mc2) CK(c, launch_grouped_gemm_tc_mc2(f.dtype, s.dual, a.tm_gate_h, a.tm_up_h, tm_b_up, up, c->num_sms, st));
      else
#endif
      CK(c, launch_grouped_gemm_tc(f.dtype, nt, s.dual, a.tm_gate, a.tm_up, tm_b_up, up, c->num_sms, st));
    }
    if (phases & 2) {
      // prefill-sized token tiles: pair two m-tiles of the down matrix on one token tile (dual_m) -> 1.33x the
      // FLOP per operand byte; decode keeps single tiles (finer split-K balance, HBM bound anyway).  256-token tiles already
      // share each weight tile between twice the tokens, and a paired 256-token tile has no room in the registers.
      const bool pair = nt_dn == 128 && s.H >= 256 && T_hint_large;
      dn.dual_m = pair ? 1 : 0;
      // decode: let the down projection start under the tail of the gate/up GEMM and prefetch its first weight tiles
      // B2M_EARLY_A=0 disables
      const bool early_a = sw().early_a;
      dn.early_a = (early_a && !pdl_enabled() && (phases & 1) && f.gemm_impl != 1 && !T_hint_large) ? 1 : 0;
      // split-K at decode: equal contiguous shares of all (tile, k-block) units per CTA instead of a fixed factor, so no
      // SM is left with an extra slice in the last wave (B2M_STREAMK=0: fixed factor)
      const bool streamk = sw().streamk;
      dn.stream_k = (streamk && dn.ksplit > 1 && !(mc2 && nt_dn == 128)) ? 1 : 0;
#ifdef B2M_ENABLE_MC2
      if (mc2 && nt_dn == 128) CK(c, launch_grouped_gemm_tc_mc2(f.dtype, pair, a.tm_down_h, a.tm_down_h, tm_b_down, dn, c->num_sms, st));
      else
#endif
      CK(c, launch_grouped_gemm_tc(f.dtype, nt_dn, pair, a.tm_down, a.tm_down, tm_b_down, dn, c->num_sms, st));
    }
  }
  c->stats.kernel_launches += ((phases & 1) ? 1 : 0) + ((phases & 2) ? 1 : 0);
  return B2M_OK;
}

int b2m_run_experts(b2m_ctx* c, int layer, int T, void* stream) { return b2m_run_experts_ex(c, layer, T, 3, stream); }

int b2m_run_experts_ex(b2m_ctx* c, int layer, int T, int phases, void* stream) {
  int r = check_layer(c, layer);
  if (r) return r;
  if (T != c->cur_T) return fail(c, B2M_ESTATE, "b2m_run_experts(T=%d) does not follow a routing call with the same T (%d)", T, c->cur_T);
  if (T == 0) return B2M_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int E = c->cfg.num_experts;
  r = pump(c);
  if (r) return r;
  std::vector<int> active;
  const bool do_residency = (phases & 1) != 0;
  // expert-parallel contexts hold only this rank's experts, all resident: never the on-demand path
  const bool on_demand = c->offload && !c->ep_mode;
  if (!do_residency) {
    active = c->last_active;
  } else if (on_demand) {
    // on-demand path: read the per-expert counts back (the reference's .cpu() in dispatch_local)
    CK(c, cudaMemcpyAsync(c->h_counts, c->d_counts, sizeof(int) * E, cudaMemcpyDeviceToHost, st));
    c->last_look_valid = false;
    if (c->look_pending) CK(c, cudaMemcpyAsync(c->h_look, c->d_look, sizeof(int) * E, cudaMemcpyDeviceToHost, st));
    CK(c, cudaStreamSynchronize(st));
    c->stats.host_syncs++;
    c->last_counts_valid = true;
    c->last_look_valid = c->look_pending;
    c->look_pending = false;
    c->cur_layer = layer;
    if (c->tr.hint_pending && c->tr.auto_prefetch) {
      // the device predictor's score matrix arrived with this read-back: ExpertPrefetcher.prefetch_experts on the host side
      // (expert_prefetcher.py:42-59: layers >= the predicting layer, score > 0, descending) -> protected set + prefetch queue
      c->tr.hint_pending = false;
      const int Ln = c->cfg.num_layers;
      std::vector<int32_t> pairs;
      std::vector<float> scores;
      for (int l = c->tr.hint_layer; l < Ln; ++l)
        for (int e = 0; e < E; ++e) {
          const float sc = c->tr.h_hint[(size_t)l * E + e];
          if (sc > 0.f && !(l == layer && c->h_counts[e] > 0)) { pairs.push_back(l); pairs.push_back(e); scores.push_back(sc); }
        }
      if (!scores.empty()) {
        for (int e = 0; e < E; ++e)                    // this layer's activated experts are in use from now on: never a prefetch victim
          if (c->h_counts[e] > 0) c->last_active.push_back(layer * E + e);
        int rr = b2m_prefetch_hint(c, (int)scores.size(), pairs.data(), scores.data());
        if (rr) return rr;
      }
    }
    const float alpha = c->cfg.freq_alpha > 0.f ? c->cfg.freq_alpha : 0.25f;
    for (int e = 0; e < E; ++e) {
      Expert& x = c->experts[(size_t)layer * E + e];
      if (c->h_counts[e] > 0) active.push_back(layer * E + e);
      x.freq = (1.0f - alpha) * x.freq + (c->h_counts[e] > 0 ? alpha : 0.0f);
    }
    if (c->last_look_valid) {
      // the predicted experts of the next layer must not be evicted to make room for this layer's misses
      const int nxt = (layer + 1) % c->cfg.num_layers;
      c->protected_set.clear();
      for (int e = 0; e < E; ++e)
        if (c->h_look[e] > 0) c->protected_set.insert(nxt * E + e);
    }
  } else {
    for (int e = 0; e < E; ++e)
      if (!c->ep_mode || c->experts[(size_t)layer * E + e].state != ST_UNREGISTERED) active.push_back(layer * E + e);
  }
  // ---- residency + launch, in waves.  Normally one wave holds every activated expert.  When the HBM budget is
  // smaller than one layer's active set (reference: experts run one at a time, a single slot suffices) the set is
  // split: a wave is staged, its GEMMs are launched against a slot row that names only that wave, then the next.
  GemmParams base;
  memset(&base, 0, sizeof base);
  base.offsets = c->d_offsets;
  base.slot_of = c->d_slot_of + (size_t)layer * E;
  base.E = E;
  base.single_n = -1;
  const int ni = nt_index(c->cur_nt), nd = nt_index(c->cur_nt_dn);
  if (!do_residency) {
    r = upload_row_if_dirty(c, layer, st);
    if (r) return r;
    return launch_expert_gemms(c, c->arena, base, c->tm_xp[ni], c->tm_hmid[nd], c->d_xp, c->cfg.hidden, c->d_hmid,
                               c->d_hmid, c->d_y, c->cur_nt, c->cur_nt_dn, c->cur_ksplit, st, phases);
  }
  for (int id : active)
    if (c->experts[id].state == ST_UNREGISTERED)
      return fail(c, B2M_ESTATE, "expert (%d,%d) was never registered", id / E, id % E);
  std::vector<int> remaining = active, wave;
  int waves = 0;
  int demand_copies = 0;   // experts this call had to stage on demand
  while (!remaining.empty()) {
    wave.clear();
    for (int id : remaining) {
      Expert& x = c->experts[id];
      const bool resident = x.state == ST_RESIDENT || x.state == ST_LOADING;
      if (!resident) {
        if (!x.backed()) return fail(c, B2M_ESTATE, "expert (%d,%d) is neither resident nor backed by a host blob", id / E, id % E);
        if (c->ep_mode) return fail(c, B2M_ESTATE, "expert-parallel mode needs every local expert resident: (%d,%d) is not", id / E, id % E);
        // never evict an expert this call still has to run (reference: those nodes hold their mutex, :239)
        const int slot = on_demand ? acquire_slot_on_demand(c, remaining) : acquire_slot(c, remaining, false);
        if (slot < 0) continue;                               // no room in this wave: stays in `remaining`
        if (on_demand) c->stats.misses++;
        ++demand_copies;
        r = issue_copy(c, id, slot, c->fetch_stream, true);
        if (r) return r;
      } else if (on_demand) {
        c->stats.hits++;
        if (x.prefetched_unused) { c->stats.prefetch_useful++; c->pf_win_useful++; x.prefetched_unused = false; }
      }
      if (on_demand) {
        c->stats.dispatches++;
        x.visits += 1;            // incache_visit_count += 1 for every dispatched expert (expert_dispatcher.cpp:264)
        x.total_visits += 1;
        c->budget_units -= 1;     // cache_sizes_ -= byte_size for every dispatched expert, hit or miss (:266)
      }
      wave.push_back(id);
    }
    if (wave.empty())
      return fail(c, B2M_ENOMEM, "no evictable HBM slot: %d experts active, %d slots", (int)active.size(), c->arena.nslots);
    for (int id : wave) {
      Expert& x = c->experts[id];
      if (x.ready_pending) {
        CK(c, cudaStreamWaitEvent(st, x.ready, 0));
        x.ready_pending = false;
      }
      if (x.state == ST_LOADING) x.state = ST_RESIDENT;   // every later use is stream-ordered after the wait above
    }
    const bool whole = wave.size() == active.size();
    if (!whole && phases != 3) return fail(c, B2M_ESTATE, "phase-split launches need the whole active set resident");
    std::vector<int> pack;
    if (whole) {
      r = upload_row_if_dirty(c, layer, st);
      if (r) return r;
      if (phases & 1) {   // the gate/up launch packs
        r = pk_collect(c, layer, st, &pack);
        if (r) return r;
      }
    } else {
      // partial wave: the device row names only this wave's experts (others -1 => their tiles are skipped)
      if (waves > 0 && waves % (STAGE_RING - 1) == 0) CK(c, cudaStreamSynchronize(st));   // staging ring would wrap
      int* stage = c->h_stage + (size_t)c->stage_pos * E;
      c->stage_pos = (c->stage_pos + 1) % STAGE_RING;
      for (int e = 0; e < E; ++e) stage[e] = -1;
      for (int id : wave) stage[id % E] = c->experts[id].slot;
      CK(c, cudaMemcpyAsync(c->d_slot_of + (size_t)layer * E, stage, sizeof(int) * E, cudaMemcpyHostToDevice, st));
      c->row_dirty[layer] = 1;   // the true mapping is re-uploaded by the next whole-wave call
    }
    GemmParams wave_base = base;
    wave_base.pack_slots = pack.data();
    wave_base.pack_n = (int)pack.size();
    r = launch_expert_gemms(c, c->arena, wave_base, c->tm_xp[ni], c->tm_hmid[nd], c->d_xp, c->cfg.hidden, c->d_hmid,
                            c->d_hmid, c->d_y, c->cur_nt, c->cur_nt_dn, c->cur_ksplit, st, phases);
    if (r) return r;
    if (on_demand) {
      int evi;
      cudaEvent_t ev = next_ring_event(c, &evi);
      CK(c, cudaEventRecord(ev, st));
      for (int id : wave) c->slots[c->experts[id].slot].last_use_ev = evi;
    }
    ++waves;
    remaining.erase(std::remove_if(remaining.begin(), remaining.end(),
                                   [&](int id) { return std::find(wave.begin(), wave.end(), id) != wave.end(); }),
                    remaining.end());
  }
  c->last_active = wave;   // experts of the last wave are still being read by kernels in flight
  // When the host->device link is saturated by on-demand copies a prefetch cannot save time, only bytes -- and a wrong
  // prediction costs a whole expert (352 MB for Mixtral), so ~80 % accurate predictions lose against the same cache
  // without prefetching.  So (lookahead_prefetch = 1)
  // predictions are staged only from layers that staged nothing on demand, i.e. into link time that is otherwise idle;
  // lookahead_prefetch = 2 prefetches unconditionally (sparse-miss regimes, ablations).
  if (c->cfg.lookahead_prefetch == 1 && c->pf_win_useful + c->pf_win_wasted >= 16) {
    // governor (mode 1 only): below 90 % accuracy prefetching loses on a saturated link -> suspend for 256 layer calls, then probe again
    if (c->pf_win_useful * 10 < (c->pf_win_useful + c->pf_win_wasted) * 9) c->pf_suspended_until = (long long)c->stats.host_syncs + 256;
    c->pf_win_useful = c->pf_win_wasted = 0;
  }
  const bool pf_suspended = c->cfg.lookahead_prefetch == 1 && (long long)c->stats.host_syncs < c->pf_suspended_until;
  if (on_demand && c->last_look_valid && !pf_suspended && (demand_copies == 0 || c->cfg.lookahead_prefetch >= 2)) {
    // stage the next layer's predicted experts while this layer computes: most-wanted first; a prediction only displaces
    // an expert whose own next use is expected at least a few layer visits later than the next layer
    const int nxt = (layer + 1) % c->cfg.num_layers;
    std::vector<int> order;
    for (int e = 0; e < E; ++e)
      if (c->h_look[e] > 0 && c->experts[(size_t)nxt * E + e].state == ST_HOST && c->experts[(size_t)nxt * E + e].backed()) order.push_back(e);
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return c->h_look[a] > c->h_look[b]; });
    r = pump(c);   // retire finished copies first
    if (r) return r;
    const int max_if = c->cfg.max_inflight_prefetch > 0 ? c->cfg.max_inflight_prefetch : 2;
    for (int e : order) {
      if ((int)c->inflight.size() >= max_if) break;
      const int id = nxt * E + e;
      int slot = -1;
      if (!c->free_slots.empty()) {
        slot = c->free_slots.back();
        c->free_slots.pop_back();
      } else {
        float vs = 0.f;
        const int v = c->cfg.cache_policy == B2M_CACHE_ACTIVATION_AWARE ? pick_victim_next_use(c, c->last_active, false, &vs)
                                                                         : pick_victim(c, c->last_active, false);
        if (v < 0 || (c->cfg.cache_policy == B2M_CACHE_ACTIVATION_AWARE && vs < 2.5f)) break;   // never trade away an expert that is itself expected within the next two layer visits
        evict(c, v);
        slot = c->free_slots.back();
        c->free_slots.pop_back();
      }
      r = issue_copy(c, id, slot, c->prefetch_stream, true);
      if (r) return r;
      c->experts[id].prefetched_unused = true;
      c->inflight.push_back(id);
      c->stats.prefetch_issued++;
    }
  }
  return B2M_OK;
}

static int run_shared(b2m_ctx* c, int layer, const void* x, int T, cudaStream_t st) {
  if (!c->shared_registered[layer]) return fail(c, B2M_ESTATE, "shared expert of layer %d not registered", layer);
  if (c->d_shared_gate) {
    // Qwen2-MoE: the gate values depend on x only, so they are computed here, ahead of the shared GEMMs on the same stream
    if (!c->shared_gate_w[layer]) return fail(c, B2M_ESTATE, "layer %d has no shared-expert gate (b2m_set_shared_gate)", layer);
    CombineParams g;
    memset(&g, 0, sizeof g);
    g.mode = COMBINE_QWEN_GATE;
    g.x = x;
    g.shared_gate_w = c->shared_gate_w[layer];
    g.out = c->d_shared_gate;
    g.T = T; g.H = c->cfg.hidden; g.k = c->cfg.top_k; g.dtype = c->cfg.dtype;
    CK(c, launch_combine(g, st));
    c->stats.kernel_launches += 1;
  }
  const int nt = pick_nt(T);
  const int ks = pick_ksplit(c, T, c->cfg.hidden, c->cfg.shared_inter, 1, 1, nt);
  CUtensorMap tm_x;
  memset(&tm_x, 0, sizeof tm_x);
  int r = c->cfg.dtype == B2M_DTYPE_F32 ? B2M_OK : build_act_map(c, &tm_x, const_cast<void*>(x), c->cfg.hidden, T, nt);
  if (r) return r;
  if (ks > 1 && c->cfg.dtype != B2M_DTYPE_F32) CK(c, cudaMemsetAsync(c->d_y_s, 0, (size_t)T * c->cfg.hidden * sizeof(float), st));
  GemmParams base;
  memset(&base, 0, sizeof base);
  base.E = 1;
  base.single_n = T;
  base.single_slot = layer;
  return launch_expert_gemms(c, c->shared_arena, base, tm_x, c->tm_hmid_s[nt_index(nt)], x, c->cfg.hidden, c->d_hmid_s,
                             c->d_hmid_s, c->d_y_s, nt, nt, ks, st, 3, T);
}

static int combine_impl(b2m_ctx* c, int layer, const void* x, int T, void* out, void* stream, bool ep_collect);

int b2m_combine(b2m_ctx* c, int layer, const void* x, int T, void* out, void* stream) {
  return combine_impl(c, layer, x, T, out, stream, false);
}

static int combine_impl(b2m_ctx* c, int layer, const void* x, int T, void* out, void* stream, bool ep_collect) {
  int r = check_layer(c, layer);
  if (r) return r;
  if (T < 0 || T > c->cap_T) return fail(c, B2M_EINVAL, "T=%d exceeds workspace capacity %d", T, c->cap_T);
  if (T == 0) return B2M_OK;
  if (!out) return fail(c, B2M_EINVAL, "out is null");
  cudaStream_t st = (cudaStream_t)stream;
  const b2m_config& f = c->cfg;
  CombineParams p;
  memset(&p, 0, sizeof p);
  p.y = c->d_y;
  p.x = x;
  p.topk_idx = c->d_topk_idx; p.topk_w = c->d_topk_w; p.row_of = c->d_row_of;
  p.out = out;
  p.T = T; p.H = f.hidden; p.k = f.top_k; p.dtype = f.dtype;
  p.mode = f.numerics == B2M_NUMERICS_FP32 ? c->rk->combine_fp32 : c->rk->combine;
  p.unweighted = c->rk->scales_inputs;   // the weights scaled the expert inputs (COMBINE_LLAMA4 or COMBINE_FP32)
  if (f.shared_inter > 0) {
    if (c->shared_in_flight) {
      // launched by b2m_moe_forward on the side stream at the start of the call: join it
      CK(c, cudaStreamWaitEvent(st, c->ev_join, 0));
      c->shared_in_flight = false;
    } else {
      r = run_shared(c, layer, x, T, st);
      if (r) return r;
    }
    p.y_shared = c->d_y_s;
    p.shared_gate = reinterpret_cast<const uint16_t*>(c->d_shared_gate);
  }
  if (ep_collect) {
    p.ep_collect = 1;
    p.ep = c->ep_direct_next ? ep_p2p_params_direct(c) : ep_p2p_params(c);
    const bool early_combine = sw().ep_early_combine;
    p.ep_early = (c->ep_direct_next && early_combine && !pdl_enabled() && f.shared_inter == 0) ? 1 : 0;
    if (c->tl_next) p.tl = c->tl_next + 12;
  }
  CK(c, launch_combine(p, st));
  c->stats.kernel_launches += 1;
  return B2M_OK;
}

int b2m_moe_forward(b2m_ctx* c, int layer, const void* x, const void* router_in, int kind, int in_dtype, int T,
                    int seq_len, void* out, void* stream) {
  int r = check_layer(c, layer);
  if (r) return r;
  r = refuse_scores(c, kind);   // before the shared expert is launched
  if (r) return r;
  if (c->cfg.shared_inter > 0 && T > 0 && T <= c->cap_T && x) {
    // the shared experts (deepseek.py:133-136) depend on x only: fork them onto a side stream so that their two GEMM
    // launches overlap the gate / top-k / permute kernels of the routed path; b2m_combine joins
    cudaStream_t st = (cudaStream_t)stream;
    CK(c, cudaEventRecord(c->ev_fork, st));
    CK(c, cudaStreamWaitEvent(c->shared_stream, c->ev_fork, 0));
    r = run_shared(c, layer, x, T, c->shared_stream);
    if (r) return r;
    CK(c, cudaEventRecord(c->ev_join, c->shared_stream));
    c->shared_in_flight = true;
  }
  r = b2m_route(c, layer, x, router_in, kind, in_dtype, T, seq_len, stream);
  if (!r) r = b2m_run_experts(c, layer, T, stream);
  if (r) {
    if (c->shared_in_flight) { cudaStreamWaitEvent((cudaStream_t)stream, c->ev_join, 0); c->shared_in_flight = false; }
    return r;
  }
  return b2m_combine(c, layer, x, T, out, stream);
}

// B2M_EINVAL naming what each bit of the (already cleared) sticky device error word reports
static int fail_err_word(b2m_ctx* c, int bits) {
  std::string what;
  if (bits & 1) what += "a router-mask row names more experts than top_k (rows would be dropped)";
  if (bits & 2) what += std::string(what.empty() ? "" : "; ") + "an input-permutation entry (b2m_set_input_perm) is >= hidden (read as 0)";
  return fail(c, B2M_EINVAL, "device error word %d: %s", bits, what.c_str());
}

int b2m_expert_outputs(b2m_ctx* c, int T, void* out_rows, int* offsets_host, void* stream) {
  if (!c) return B2M_EINVAL;
  if (T < 0 || T > c->cap_T) return fail(c, B2M_EINVAL, "T=%d exceeds workspace capacity %d", T, c->cap_T);
  if (T != c->cur_T) return fail(c, B2M_ESTATE, "b2m_expert_outputs(T=%d) does not follow a routing call with the same T (%d)", T, c->cur_T);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t n = (size_t)T * c->cfg.top_k * c->cfg.hidden;
  if (out_rows && T > 0) {
    CK(c, launch_cast_rows(c->d_y, out_rows, n, c->cfg.dtype, st));
    c->stats.kernel_launches += 1;
  }
  if (offsets_host) {
    CK(c, cudaMemcpyAsync(offsets_host, c->d_offsets, sizeof(int) * (c->cfg.num_experts + 1), cudaMemcpyDeviceToHost, st));
    CK(c, cudaMemcpyAsync(c->h_err, c->d_err, sizeof(int), cudaMemcpyDeviceToHost, st));
    CK(c, cudaStreamSynchronize(st));
    if (*c->h_err) {
      const int bits = *c->h_err;
      CK(c, cudaMemsetAsync(c->d_err, 0, sizeof(int), st));
      return fail_err_word(c, bits);
    }
  }
  return B2M_OK;
}

int b2m_check_errors(b2m_ctx* c, void* stream) {
  if (!c) return B2M_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  CK(c, cudaMemcpyAsync(c->h_err, c->d_err, sizeof(int), cudaMemcpyDeviceToHost, st));
  CK(c, cudaStreamSynchronize(st));
  if (*c->h_err) {
    const int bits = *c->h_err;
    CK(c, cudaMemsetAsync(c->d_err, 0, sizeof(int), st));
return fail_err_word(c, bits);
  }
  return B2M_OK;
}

// ------------------------------------------------------------------------------------
int b2m_replace_cache_candidates(b2m_ctx* c, int n, const int32_t* pairs) {
  if (!c || (n > 0 && !pairs)) return B2M_EINVAL;
  const int L = c->cfg.num_layers, E = c->cfg.num_experts;
  c->protected_set.clear();
  for (int i = 0; i < n; ++i) {
    const int l = pairs[2 * i], e = pairs[2 * i + 1];
    if (l < 0 || l >= L || e < 0 || e >= E) return fail(c, B2M_EINVAL, "candidate (%d,%d) out of range", l, e);
    c->protected_set.insert(l * E + e);
  }
  c->pending.clear();   // ArcherTaskPool::ReplaceCacheCandidates clears queued prefetches (task_scheduler.h:76-78)
  return B2M_OK;
}

int b2m_enqueue_prefetch(b2m_ctx* c, int layer, int expert) {
  int r = check_layer(c, layer);
  if (r) return r;
  if (expert < 0 || expert >= c->cfg.num_experts) return fail(c, B2M_EINVAL, "expert %d out of range", expert);
  const int id = layer * c->cfg.num_experts + expert;
  Expert& x = c->experts[id];
  if (x.state == ST_UNREGISTERED || !x.backed()) return fail(c, B2M_ESTATE, "expert (%d,%d) has no host blob", layer, expert);
  if (x.state == ST_HOST && std::find(c->pending.begin(), c->pending.end(), id) == c->pending.end())
    c->pending.push_back(id);   // dedupe (task_scheduler.cpp:86-104)
  return pump(c);
}

int b2m_prefetch_hint(b2m_ctx* c, int n, const int32_t* pairs, const float* scores) {
  if (!c || (n > 0 && (!pairs || !scores))) return B2M_EINVAL;
  std::vector<int> order(n);
  for (int i = 0; i < n; ++i) order[i] = i;
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return scores[a] > scores[b]; });
  std::vector<int32_t> sorted(2 * (size_t)n);
  for (int i = 0; i < n; ++i) { sorted[2 * i] = pairs[2 * order[i]]; sorted[2 * i + 1] = pairs[2 * order[i] + 1]; }
  int r = b2m_replace_cache_candidates(c, n, sorted.data());
  if (r) return r;
  for (int i = 0; i < n; ++i) {
    const int id = sorted[2 * i] * c->cfg.num_experts + sorted[2 * i + 1];
    Expert& x = c->experts[id];
    if (x.state == ST_HOST && x.backed()) c->pending.push_back(id);
  }
  return pump(c);
}

int b2m_prefetch_pump(b2m_ctx* c) { return c ? pump(c) : B2M_EINVAL; }

int b2m_prefetch_drain(b2m_ctx* c) {
  if (!c) return B2M_EINVAL;
  for (int guard = 0; guard < 1 << 20; ++guard) {
    CK(c, cudaStreamSynchronize(c->prefetch_stream));
    CK(c, cudaStreamSynchronize(c->fetch_stream));
    int r = pump(c);
    if (r) return r;
    if (c->inflight.empty() && c->pending.empty()) break;
  }
  return B2M_OK;
}

int b2m_clear_expert_cache_counts(b2m_ctx* c) {
  if (!c) return B2M_EINVAL;
  for (auto& x : c->experts) x.visits = 0;
  return B2M_OK;
}

int b2m_is_resident(b2m_ctx* c, int layer, int expert) {
  int r = check_layer(c, layer);
  if (r) return r;
  if (expert < 0 || expert >= c->cfg.num_experts) return fail(c, B2M_EINVAL, "expert %d out of range", expert);
  const Expert& x = c->experts[(size_t)layer * c->cfg.num_experts + expert];
  return (x.state == ST_RESIDENT || x.state == ST_LOADING) ? 1 : 0;
}

int b2m_stats_get(b2m_ctx* c, b2m_stats* out) {
  if (!c || !out) return B2M_EINVAL;
  uint64_t res = 0;
  for (auto& x : c->experts) res += (x.state == ST_RESIDENT || x.state == ST_LOADING) ? 1 : 0;
  c->stats.resident = res;
  *out = c->stats;
  return B2M_OK;
}

int b2m_last_lookahead(b2m_ctx* c, int32_t* look_host) {
  if (!c || !look_host) return B2M_EINVAL;
  if (!c->last_look_valid) return fail(c, B2M_ESTATE, "the last call made no look-ahead prediction (cfg.lookahead_prefetch, offload mode, T <= 256, next layer's gate set)");
  memcpy(look_host, c->h_look, sizeof(int) * c->cfg.num_experts);
  return B2M_OK;
}

int b2m_last_counts(b2m_ctx* c, int32_t* counts_host) {
  if (!c || !counts_host) return B2M_EINVAL;
  if (!c->last_counts_valid) return fail(c, B2M_ESTATE, "last call ran sync-free; counts were not read back");
  memcpy(counts_host, c->h_counts, sizeof(int) * c->cfg.num_experts);
  return B2M_OK;
}

// ------------------------------------------------------------------------------------ expert parallel
static EpParams ep_base(b2m_ctx* c, int nranks, int rank, int cap) {
  EpParams p;
  memset(&p, 0, sizeof p);
  p.nranks = nranks; p.rank = rank; p.E = c->cfg.num_experts; p.H = c->cfg.hidden; p.cap = cap;
  p.offsets = c->d_offsets; p.offsets_rw = c->d_offsets; p.offsets_src = c->d_offsets_src;
  p.xp = c->d_xp; p.y = c->d_y; p.dest_of = c->d_dest_of;
  return p;
}
static int ep_check(b2m_ctx* c, int nranks, int rank, int cap) {
  if (!c) return B2M_EINVAL;
  if (c->cfg.dtype == B2M_DTYPE_F32) return fail(c, B2M_EUNSUPPORTED, "expert parallel exchange handles 16-bit models");
  // the buffer exchange returns expert outputs in the model dtype, the single-GPU fp32 combine reads them unrounded (and
  // the peer-to-peer direct mode reads the owners' fp32 outputs): the result would depend on the exchange mode
  if (c->cfg.numerics == B2M_NUMERICS_FP32)
    return fail(c, B2M_EUNSUPPORTED, "expert parallelism is not available with fp32 numerics (B2M_NUMERICS_FP32): the "
                "exchange returns expert outputs rounded to the model dtype");
  if (c->wf->a_src != AS_BF16) return fail(c, B2M_EUNSUPPORTED, "expert parallelism is not available with %s weights", c->wf->name);
  if (!c->rk->ep) return fail(c, B2M_EUNSUPPORTED, "expert parallelism is not available with the %s router", c->rk->name);
  if (nranks < 2 || nranks > 16 || rank < 0 || rank >= nranks || c->cfg.num_experts % nranks || cap < 1)
    return fail(c, B2M_EINVAL, "bad expert-parallel geometry (nranks=%d rank=%d cap=%d E=%d)", nranks, rank, cap, c->cfg.num_experts);
  if ((long long)nranks * cap > c->cap_R)
    return fail(c, B2M_EINVAL, "workspace too small for EP: nranks*cap=%d rows > %d (create the context with max_tokens >= nranks*T_local)", nranks * cap, c->cap_R);
  return B2M_OK;
}

int b2m_ep_pack(b2m_ctx* c, int nranks, int rank, int cap, int T_local, void* send_rows, int32_t* send_counts, void* stream) {
  if (c) c->k3_early_ok = false;
  int r = ep_check(c, nranks, rank, cap);
  if (r) return r;
  if (T_local * c->cfg.top_k > cap) return fail(c, B2M_EINVAL, "cap=%d < T_local*top_k=%d", cap, T_local * c->cfg.top_k);
  EpParams p = ep_base(c, nranks, rank, cap);
  p.send_rows = send_rows;
  p.send_counts = send_counts;
  p.inline_counts = send_counts == nullptr;   // counts ride in the row buffers ([nranks][cap+1][H])
  c->ep_inline = p.inline_counts;
  CK(c, launch_ep_pack(p, T_local * c->cfg.top_k, (cudaStream_t)stream));
  c->stats.kernel_launches += 1;
  c->ep_mode = true;
  return B2M_OK;
}

int b2m_ep_regroup(b2m_ctx* c, int nranks, int rank, int cap, int T_total, const void* recv_rows, const int32_t* recv_counts, void* stream) {
  if (c) c->k3_early_ok = false;
  int r = ep_check(c, nranks, rank, cap);
  if (r) return r;
  if (T_total < 1 || T_total > c->cap_T) return fail(c, B2M_EINVAL, "T_total=%d exceeds workspace capacity %d", T_total, c->cap_T);
  EpParams p = ep_base(c, nranks, rank, cap);
  p.recv_rows = recv_rows;
  p.recv_counts = recv_counts;
  p.inline_counts = recv_counts == nullptr;
  c->ep_inline = p.inline_counts;
  // plan the local GEMMs for the rows this rank may receive
  c->cur_T = T_total;
  c->cur_nt = c->cur_nt_dn = pick_nt(T_total);
  c->cur_ksplit = pick_ksplit(c, T_total, c->cfg.hidden, c->cfg.inter, c->cfg.num_experts / nranks, c->cfg.top_k, c->cur_nt);
  if (c->cur_ksplit > 1) { p.y_zero = c->d_y; p.y_zero_elems = (size_t)nranks * cap * c->cfg.hidden; }
  CK(c, launch_ep_regroup(p, (cudaStream_t)stream));
  c->stats.kernel_launches += 1;
  c->ep_mode = true;
  return B2M_OK;
}

int b2m_ep_ungroup(b2m_ctx* c, int nranks, int rank, int cap, void* ret_rows, void* stream) {
  int r = ep_check(c, nranks, rank, cap);
  if (r) return r;
  EpParams p = ep_base(c, nranks, rank, cap);
  p.ret_rows = ret_rows;
  p.inline_counts = c->ep_inline;
  CK(c, launch_ep_ungroup(p, c->cfg.dtype, (cudaStream_t)stream));
  c->stats.kernel_launches += 1;
  return B2M_OK;
}

int b2m_ep_unpack(b2m_ctx* c, int nranks, int rank, int cap, int T_local, const void* back_rows, void* stream) {
  int r = ep_check(c, nranks, rank, cap);
  if (r) return r;
  if (T_local < 0 || T_local * c->cfg.top_k > cap) return fail(c, B2M_EINVAL, "T_local=%d: T_local*top_k exceeds cap=%d", T_local, cap);
  EpParams p = ep_base(c, nranks, rank, cap);
  p.back_rows = back_rows;
  p.inline_counts = c->ep_inline;
  CK(c, launch_ep_unpack(p, c->cfg.dtype, T_local * c->cfg.top_k, (cudaStream_t)stream));
  c->stats.kernel_launches += 1;
  return B2M_OK;
}

// ---- peer-to-peer exchange: rows go straight into the peers' buffers over NVLink, no collective call ----
static size_t p2p_area_bytes(const b2m_ctx* c, int nranks, int cap) {
  return (size_t)nranks * (cap + 1) * c->cfg.hidden * 2;
}
static EpParams ep_p2p_params(b2m_ctx* c) {
  const b2m_ctx::P2P& q = c->p2p;
  EpParams p = ep_base(c, q.nranks, q.rank, q.cap);
  p.inline_counts = 1;
  p.p2p = 1;
  for (int r = 0; r < q.nranks; ++r) {
    p.peer_recv[r] = q.peer_base[r];
    p.peer_back[r] = q.peer_base[r] + q.area_bytes;
    p.peer_recv_flag[r] = reinterpret_cast<int*>(q.peer_base[r] + 2 * q.area_bytes);
    p.peer_back_flag[r] = p.peer_recv_flag[r] + 16;
  }
  p.local_recv_flag = reinterpret_cast<int*>(q.base + 2 * q.area_bytes);
  p.local_back_flag = p.local_recv_flag + 16;
  p.recv_rows = q.base;
  p.back_rows = q.base + q.area_bytes;
  p.epoch = q.local_ctr;
  p.done_ctr = q.local_ctr + 2;
  for (int r = 0; r < q.nranks; ++r) {
    p.peer_cnt[r] = reinterpret_cast<int*>(q.peer_base[r] + q.cnt_off);
    p.peer_y[r] = reinterpret_cast<float*>(q.peer_base[r] + q.y_off);
  }
  p.local_cnt = reinterpret_cast<int*>(q.base + q.cnt_off);
  p.local_y = reinterpret_cast<float*>(q.base + q.y_off);
  p.region_rows = q.nranks * q.cap;
  return p;
}
// direct mode: [nranks][cap] receive slots without a counts row, per-slot tags, outputs read in place by the sources
static EpParams ep_p2p_params_direct(b2m_ctx* c) {
  EpParams p = ep_p2p_params(c);
  p.inline_counts = 0;
  p.direct = 1;
  const b2m_ctx::P2P& q = c->p2p;
  for (int r = 0; r < q.nranks; ++r) p.peer_recv[r] = q.peer_base[r] + q.drecv_off;   // per-expert regions, not per-source segments
  p.recv_rows = q.base + q.drecv_off;
  return p;
}

int b2m_ep_p2p_init(b2m_ctx* c, int nranks, int rank, int cap, void* ipc_handle_out64) {
  int r = ep_check(c, nranks, rank, cap);
  if (r) return r;
  if (!ipc_handle_out64) return fail(c, B2M_EINVAL, "null handle buffer");
  if (c->p2p.base) return fail(c, B2M_ESTATE, "peer-to-peer exchange already initialised");
  if (4 * c->cfg.num_experts > 2 * c->cfg.hidden) return fail(c, B2M_EINVAL, "inline counts need 4*E <= 2*H");
  b2m_ctx::P2P& q = c->p2p;
  q.nranks = nranks; q.rank = rank; q.cap = cap;
  q.area_bytes = p2p_area_bytes(c, nranks, cap);
  const size_t drows = (size_t)(c->cfg.num_experts / nranks) * nranks * cap;   // = E*cap: one region of nranks*cap rows per local expert
  q.cnt_off = (2 * q.area_bytes + 32 * sizeof(int) + 255) & ~(size_t)255;
  q.drecv_off = (q.cnt_off + 256 * sizeof(int) + 255) & ~(size_t)255;
  q.y_off = (q.drecv_off + drows * c->cfg.hidden * 2 + 255) & ~(size_t)255;
  const size_t total = q.y_off + drows * c->cfg.hidden * sizeof(float);
  CK(c, cudaMalloc((void**)&q.base, total));
  CK(c, cudaMemset(q.base, 0, total));
  CK(c, cudaMalloc(&q.d_hmid, drows * c->cfg.inter * 2));
  CK(c, cudaMemset(q.d_hmid, 0, drows * c->cfg.inter * 2));
  for (int i = 0; i < 5; ++i) {
    int rr = build_act_map(c, &q.tm_recv[i], q.base + q.drecv_off, c->cfg.hidden, (int)drows, NT_LIST[i]);
    if (!rr) rr = build_act_map(c, &q.tm_hmid[i], q.d_hmid, c->cfg.inter, (int)drows, NT_LIST[i]);
    if (rr) return rr;
  }
  CK(c, cudaMalloc((void**)&q.local_ctr, 20 * sizeof(int)));
  CK(c, cudaMemset(q.local_ctr, 0, 20 * sizeof(int)));
  CK(c, cudaDeviceSynchronize());
  cudaIpcMemHandle_t h;
  CK(c, cudaIpcGetMemHandle(&h, q.base));
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  memcpy(ipc_handle_out64, &h, 64);
  q.peer_base[rank] = q.base;
  return B2M_OK;
}

int b2m_ep_p2p_open(b2m_ctx* c, int peer, const void* ipc_handle64) {
  if (!c || !ipc_handle64) return B2M_EINVAL;
  b2m_ctx::P2P& q = c->p2p;
  if (!q.base) return fail(c, B2M_ESTATE, "call b2m_ep_p2p_init first");
  if (peer < 0 || peer >= q.nranks) return fail(c, B2M_EINVAL, "peer %d out of range", peer);
  if (peer == q.rank) return B2M_OK;
  cudaIpcMemHandle_t h;
  memcpy(&h, ipc_handle64, 64);
  void* ptr = nullptr;
  CK(c, cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
  q.peer_base[peer] = reinterpret_cast<uint8_t*>(ptr);
  return B2M_OK;
}

static int p2p_ready(b2m_ctx* c) {
  if (!c) return B2M_EINVAL;
  if (!c->p2p.base) return fail(c, B2M_ESTATE, "peer-to-peer exchange not initialised");
  for (int r = 0; r < c->p2p.nranks; ++r)
    if (!c->p2p.peer_base[r]) return fail(c, B2M_ESTATE, "peer %d buffer not opened (b2m_ep_p2p_open)", r);
  return B2M_OK;
}

int b2m_ep_p2p_dispatch(b2m_ctx* c, int T_local, void* stream) {
  if (c) c->k3_early_ok = false;
  int r = p2p_ready(c);
  if (r) return r;
  if (T_local * c->cfg.top_k > c->p2p.cap) return fail(c, B2M_EINVAL, "cap=%d < T_local*top_k", c->p2p.cap);
  EpParams p = ep_p2p_params(c);
  CK(c, launch_ep_pack(p, T_local * c->cfg.top_k, (cudaStream_t)stream));
  c->stats.kernel_launches += 1;
  c->ep_mode = true;
  c->ep_inline = 1;
  return B2M_OK;
}

int b2m_ep_p2p_route(b2m_ctx* c, int layer, const void* x, const void* router_in, int kind, int in_dtype, int T_local,
                     void* stream) {
  int r = p2p_ready(c);
  if (r) return r;
  if (T_local * c->cfg.top_k > c->p2p.cap) return fail(c, B2M_EINVAL, "cap=%d < T_local*top_k", c->p2p.cap);
  r = route_impl(c, layer, x, router_in, kind, in_dtype, T_local, 0, stream, true);
  if (r) return r;
  c->ep_mode = true;
  c->ep_inline = 1;
  return B2M_OK;
}

int b2m_ep_p2p_combine(b2m_ctx* c, int layer, const void* x, int T_local, void* out, void* stream) {
  int r = p2p_ready(c);
  if (r) return r;
  if (T_local < 0 || T_local * c->cfg.top_k > c->p2p.cap) return fail(c, B2M_EINVAL, "T_local=%d: T_local*top_k exceeds cap=%d", T_local, c->p2p.cap);
  return combine_impl(c, layer, x, T_local, out, stream, true);
}

// One expert-parallel MoE layer in FIVE kernels (was seven): gate/top-k -> permute that stores rows + slot tags into the
// owners' receive areas -> gate/up GEMM reading its token tile straight from the receive area (weights stream from the
// first cycle, only the token tiles wait for the peers' flags) -> down GEMM whose last CTA publishes "done" -> combine
// that waits for the owners and reads their fp32 outputs in place over NVLink.  Falls back to the seven-kernel sequence
// when a rank owns many experts (every local expert's GEMM spans all receive slots: fine for <= 8 experts per rank).
int b2m_ep_p2p_layer(b2m_ctx* c, int layer, const void* x, const void* router_in, int kind, int in_dtype, int T_local,
                     void* out, void* stream) {
  int r = p2p_ready(c);
  if (r) return r;
  r = check_layer(c, layer);
  if (r) return r;
  b2m_ctx::P2P& q = c->p2p;
  const b2m_config& f = c->cfg;
  if (T_local < 1 || T_local * f.top_k > q.cap) return fail(c, B2M_EINVAL, "T_local=%d: T_local*top_k exceeds cap=%d", T_local, q.cap);
  if (!out) return fail(c, B2M_EINVAL, "out is null");
  const int El = f.num_experts / q.nranks, R = q.nranks * q.cap, T_total = q.nranks * T_local;
  const bool direct_on = sw().ep_direct;
  // direct mode: the fused route+dispatch kernel needs every CTA resident (T_local <= #SMs)
  const bool direct = direct_on && T_local <= c->num_sms && f.gemm_impl != 1 && f.shared_inter == 0 &&
                      !c->rk->capacity && f.dtype != B2M_DTYPE_F32;
  cudaStream_t st = (cudaStream_t)stream;
  if (!direct) {
    r = b2m_ep_p2p_route(c, layer, x, router_in, kind, in_dtype, T_local, stream);
    if (!r) r = b2m_ep_p2p_regroup(c, T_total, stream);
    if (!r) r = b2m_run_experts(c, layer, T_total, stream);
    if (!r) r = b2m_ep_p2p_return(c, stream);
    if (!r) r = b2m_ep_p2p_combine(c, layer, x, T_local, out, stream);
    return r;
  }
  const bool timeline = sw().timeline;
  unsigned long long* tl = nullptr;
  if (timeline) {
    if (!c->d_tl) {
      // [L][16] slots + one more row holding the reset pattern (device-to-device copies are capturable in a CUDA graph);
      // starts are atomicMin'ed (-> all ones), ends atomicMax'ed (-> zero): slots 0, 2, 4, 8, 12 are starts
      CK(c, cudaMalloc((void**)&c->d_tl, sizeof(unsigned long long) * 16 * (f.num_layers + 1)));
      CK(c, cudaMemset(c->d_tl, 0, sizeof(unsigned long long) * 16 * (f.num_layers + 1)));
      static const unsigned long long init[16] = {~0ull, 0, ~0ull, 0, ~0ull, 0, 0, 0, ~0ull, 0, 0, 0, ~0ull, 0, 0, 0};
      CK(c, cudaMemcpy(c->d_tl + (size_t)16 * f.num_layers, init, sizeof init, cudaMemcpyHostToDevice));
    }
    tl = c->d_tl + (size_t)layer * 16;
    CK(c, cudaMemcpyAsync(tl, c->d_tl + (size_t)16 * f.num_layers, 16 * sizeof(unsigned long long), cudaMemcpyDeviceToDevice, st));
  }
  c->tl_next = tl;
  c->ep_direct_next = true;
  r = route_impl(c, layer, x, router_in, kind, in_dtype, T_local, 0, stream, true);
  c->ep_direct_next = false;
  if (r) { c->tl_next = nullptr; return r; }
  c->ep_mode = true;
  c->ep_inline = 0;
  for (int e = q.rank * El; e < (q.rank + 1) * El; ++e) {
    const Expert& ex = c->experts[(size_t)layer * f.num_experts + e];
    if (ex.state != ST_RESIDENT && ex.state != ST_LOADING)
      return fail(c, B2M_ESTATE, "expert-parallel mode needs every local expert resident: (%d,%d) is not", layer, e);
  }
  r = upload_row_if_dirty(c, layer, st);
  if (r) return r;
  // ---- plan: token tiles sized for the expected rows per expert (an expert with more rows simply takes several tiles: the
  // tile list is built on the device from the row counters)
  const int nt = pick_nt(std::max(1, (2 * T_total * f.top_k + f.num_experts - 1) / f.num_experts));
  c->cur_T = T_total;
  c->cur_nt = c->cur_nt_dn = nt;
  const ExpertShape& s = c->arena.shape;
  int ks = 1;
  if (!s.has_bias) {
    const int kblocks = (s.I + 63) / 64;
    const long long tiles = (long long)std::min(El, T_total * f.top_k) * ((s.H + 127) / 128);
    ks = (int)std::min<long long>(8, (6LL * c->num_sms + tiles - 1) / tiles);
    ks = std::max(1, std::min(ks, kblocks / 4 > 0 ? kblocks / 4 : 1));
  }
  c->cur_ksplit = ks;
  EpParams ep = ep_p2p_params_direct(c);
  GemmParams base;
  memset(&base, 0, sizeof base);
  base.slot_of = c->d_slot_of + (size_t)layer * f.num_experts;
  base.E = f.num_experts;
  base.single_n = -1;
  base.ep_rows = R;
  base.ep_first = q.rank * El;
  base.ep_el = El;
  base.ep_cnt = ep.local_cnt;
  base.ep_nranks = q.nranks;
  base.ep_rank = q.rank;
  base.ep_flag = ep.local_recv_flag;
  base.ep_epoch = ep.epoch;
  GemmParams up = base;
  up.M = s.I; up.K = s.H; up.ksplit = 1; up.epi = EPI_ACT16; up.act = s.act;
  up.mimic = f.numerics == B2M_NUMERICS_REFERENCE; up.out = c->p2p.d_hmid; up.ld_out = s.I;
  up.ep_wait = 1;
  up.ep_zero = ks > 1 ? ep.local_y : nullptr;
  up.ep_zero_elems = (size_t)El * R * s.H;
  GemmParams dn = base;
  dn.M = s.H; dn.K = s.I; dn.ksplit = ks; dn.epi = EPI_LINEAR_F32; dn.act = ACT_NONE; dn.mimic = 0;
  dn.out = ep.local_y; dn.ld_out = s.H;
  dn.stream_k = ks > 1 ? 1 : 0;
  dn.early_a = pdl_enabled() ? 0 : 1;        // weights of the down projection are prefetched under the gate/up GEMM's tail
  dn.ep_signal = 1;
  dn.ep_done_ctr = ep.done_ctr + 1;
  dn.ep_done_epoch = ep.epoch + 1;
  for (int p2 = 0; p2 < q.nranks; ++p2) dn.ep_peer_done_flag[p2] = ep.peer_back_flag[p2];
  if (s.has_bias) {
    up.bias_base = dn.bias_base = c->arena.base;
    up.bias_slot_elems = dn.bias_slot_elems = c->arena.slot_bytes / 2;
    up.bias_off = s.off_bias1 / 2;
    dn.bias_off = s.off_bias2 / 2;
    dn.mimic = up.mimic;
  }
  const int ni = nt_index(nt);
  if (tl) { up.tl = tl + 4; dn.tl = tl + 8; }
  // The tile list is static here, so the grid can be sized to it: with 448 tiles (4 experts x 112) on 132 CTAs the last
  // tiles of an uneven last round run alone, limited by what one SM can ingest; 112 CTAs x 4 tiles each finish together.
  // Weight rows per tile: 128-row tiles cut I = 14336 into 112 tiles per expert, which leaves 20 of 132 SMs idle when a rank
  // owns one expert (N = 8) and a 128-row tile is bound by what one SM ingests.  Tiles of
  // m_rows = roundup8(El*I / (SMs * rounds)) rows (112 -> 128 tiles per expert) put every SM to work; the MMA stays M = 128.
  if (!q.m_rows) {
    q.m_rows = 128;
    if (sw().ep_mrows && s.dual) {
      const long long rows_total = (long long)El * s.I;
      const long long rounds = (rows_total + 128LL * c->num_sms - 1) / (128LL * c->num_sms);
      int mr = (int)((rows_total + c->num_sms * rounds - 1) / (c->num_sms * rounds));
      mr = std::min(128, (mr + 7) & ~7);
      while (mr < 128 && (long long)El * ((s.I + mr - 1) / mr) > c->num_sms * rounds) mr += 8;
      if (mr >= 64 && mr < 128) {
        CUtensorMap unused;
        r = build_arena_maps_box(c, &c->arena, (uint32_t)mr, &q.tm_gate_r, &q.tm_up_r, &unused);
        if (r) return r;
        q.m_rows = mr;
      }
    }
  }
  {
    // L2 prefetch budget (MB, both GEMMs) spread over the tiles each kernel expects to own: k-blocks per tile
    const double up_kb_bytes = (double)El * ((s.I + q.m_rows - 1) / q.m_rows) * (s.dual ? 2 : 1) * q.m_rows * 128.0;
    up.ep_l2pf = !pdl_enabled() ? std::max(0, (int)(sw().ep_l2pf_mb * 1e6 / up_kb_bytes)) : 0;
    if (up.ep_l2pf > 0) up.pdl_edge = 1;   // resident behind the routing kernel (which has an edge behind the previous combine)
  }
  const bool mrows = q.m_rows < 128 && !sw().fused_ffn;   // (the opt-in fused kernel keeps the 128-row maps)
  if (mrows) up.m_rows = q.m_rows;
  const int up_tiles = std::min(El, T_total * f.top_k) * ((s.I + q.m_rows - 1) / q.m_rows);   // expected: every local expert active, one token tile
  const int up_rounds = (up_tiles + c->num_sms - 1) / c->num_sms;
  const int up_grid = std::max(1, std::min(c->num_sms, (up_tiles + up_rounds - 1) / up_rounds));
#ifdef B2M_ENABLE_FUSED_FFN
  if (sw().fused_ffn && s.dual && nt <= 128 && !pdl_enabled()) {
    dn.early_a = 1;
    CK(c, launch_fused_ffn(f.dtype, nt, c->arena.tm_gate, c->arena.tm_up, q.tm_recv[ni], c->arena.tm_down, q.tm_hmid[ni], up, dn,
                           c->num_sms, up_grid, c->d_gbar, st));
    c->stats.kernel_launches += 1;
  } else
#endif
  {
    CK(c, launch_grouped_gemm_tc(f.dtype, nt, s.dual, mrows ? q.tm_gate_r : c->arena.tm_gate, mrows ? q.tm_up_r : c->arena.tm_up,
                                 q.tm_recv[ni], up, up_grid, st));
    CK(c, launch_grouped_gemm_tc(f.dtype, nt, false, c->arena.tm_down, c->arena.tm_down, q.tm_hmid[ni], dn, c->num_sms, st));
    c->stats.kernel_launches += 2;
  }
  // ---- combine at the source: wait for the owners' "done", read their outputs in place
  c->ep_direct_next = true;
  r = combine_impl(c, layer, x, T_local, out, stream, true);
  c->ep_direct_next = false;
  c->tl_next = nullptr;
  return r;
}

// ------------------------------------------------------------------------------------ device-side tracer / predictor
static TraceParams trace_params(b2m_ctx* c) {
  TraceParams p;
  memset(&p, 0, sizeof p);
  p.L = c->cfg.num_layers; p.E = c->cfg.num_experts; p.k = c->cfg.top_k;
  p.capacity = c->tr.capacity; p.persistent = c->tr.persistent;
  p.topk_idx = c->d_topk_idx;
  p.seq = c->tr.seq; p.lib = c->tr.lib; p.access = c->tr.access; p.pred = c->tr.pred; p.hint = c->tr.hint; p.winner = c->tr.winner;
  return p;
}

int b2m_trace_init(b2m_ctx* c, int capacity, int max_seqs, int auto_prefetch) {
  if (!c) return B2M_EINVAL;
  if (c->tr.lib) return fail(c, B2M_ESTATE, "tracer already initialised");
  const int L = c->cfg.num_layers, E = c->cfg.num_experts;
  if (capacity < 1 || max_seqs < 1 || (long long)L * E > 8192) return fail(c, B2M_EINVAL, "bad tracer geometry (capacity=%d max_seqs=%d L*E=%d)", capacity, max_seqs, L * E);
  const size_t m = (size_t)L * E * sizeof(float);
  CK(c, cudaMalloc((void**)&c->tr.lib, m * capacity));
  CK(c, cudaMemset(c->tr.lib, 0, m * capacity));
  CK(c, cudaMalloc((void**)&c->tr.seq, m * max_seqs));
  CK(c, cudaMemset(c->tr.seq, 0, m * max_seqs));
  CK(c, cudaMalloc((void**)&c->tr.pred, m * max_seqs));
  CK(c, cudaMemset(c->tr.pred, 0, m * max_seqs));
  CK(c, cudaMalloc((void**)&c->tr.hint, m));
  CK(c, cudaMemset(c->tr.hint, 0, m));
  CK(c, cudaMalloc((void**)&c->tr.access, sizeof(int) * capacity));
  CK(c, cudaMemset(c->tr.access, 0, sizeof(int) * capacity));
  CK(c, cudaMalloc((void**)&c->tr.winner, sizeof(int) * max_seqs));
  CK(c, cudaMemset(c->tr.winner, 0, sizeof(int) * max_seqs));
  CK(c, cudaHostAlloc((void**)&c->tr.h_hint, m, cudaHostAllocDefault));
  c->tr.capacity = capacity; c->tr.max_seqs = max_seqs; c->tr.auto_prefetch = auto_prefetch;
  return B2M_OK;
}

int b2m_trace_load(b2m_ctx* c, int n, const float* lib_host) {
  if (!c || !lib_host) return B2M_EINVAL;
  if (!c->tr.lib) return fail(c, B2M_ESTATE, "call b2m_trace_init first");
  if (n < 0 || n > c->tr.capacity) return fail(c, B2M_EINVAL, "loaded trace capacity %d must be less than or equal to capacity %d", n, c->tr.capacity);
  CK(c, cudaMemcpy(c->tr.lib, lib_host, (size_t)n * c->cfg.num_layers * c->cfg.num_experts * sizeof(float), cudaMemcpyHostToDevice));
  c->tr.persistent = n;
  return B2M_OK;
}

int b2m_trace_reset_seq(b2m_ctx* c, int seq_slot, void* stream) {
  if (!c) return B2M_EINVAL;
  if (!c->tr.lib) return fail(c, B2M_ESTATE, "call b2m_trace_init first");
  if (seq_slot < 0 || seq_slot >= c->tr.max_seqs) return fail(c, B2M_EINVAL, "sequence slot %d out of range", seq_slot);
  const size_t m = (size_t)c->cfg.num_layers * c->cfg.num_experts;
  CK(c, cudaMemsetAsync(c->tr.seq + m * seq_slot, 0, m * sizeof(float), (cudaStream_t)stream));
  return B2M_OK;
}

int b2m_trace_update_predict(b2m_ctx* c, int layer, int seq_slot0, int num_seqs, int seq_len, void* stream) {
  int r = check_layer(c, layer);
  if (r) return r;
  if (!c->tr.lib) return fail(c, B2M_ESTATE, "call b2m_trace_init first");
  if (num_seqs < 1 || seq_len < 1 || seq_slot0 < 0 || seq_slot0 + num_seqs > c->tr.max_seqs)
    return fail(c, B2M_EINVAL, "sequences [%d, %d) out of range (max_seqs=%d)", seq_slot0, seq_slot0 + num_seqs, c->tr.max_seqs);
  if (num_seqs * seq_len != c->cur_T) return fail(c, B2M_ESTATE, "num_seqs*seq_len=%d does not match the last routing call (T=%d)", num_seqs * seq_len, c->cur_T);
  cudaStream_t st = (cudaStream_t)stream;
  TraceParams p = trace_params(c);
  p.layer = layer; p.seq_len = seq_len; p.seq_slot0 = seq_slot0;
  const size_t m = (size_t)c->cfg.num_layers * c->cfg.num_experts * sizeof(float);
  CK(c, cudaMemsetAsync(c->tr.hint, 0, m, st));
  CK(c, launch_trace_update_predict(p, num_seqs, st));
  c->stats.kernel_launches += 1;
  if (c->tr.auto_prefetch && c->offload && !c->ep_mode) {
    CK(c, cudaMemcpyAsync(c->tr.h_hint, c->tr.hint, m, cudaMemcpyDeviceToHost, st));   // consumed after the next count read-back
    c->tr.hint_pending = true;
    c->tr.hint_layer = layer;
  }
  return B2M_OK;
}

int b2m_trace_finish_seq(b2m_ctx* c, int seq_slot, void* stream) {
  if (!c) return B2M_EINVAL;
  if (!c->tr.lib) return fail(c, B2M_ESTATE, "call b2m_trace_init first");
  if (seq_slot < 0 || seq_slot >= c->tr.max_seqs) return fail(c, B2M_EINVAL, "sequence slot %d out of range", seq_slot);
  TraceParams p = trace_params(c);
  CK(c, launch_trace_finish(p, seq_slot, (cudaStream_t)stream));
  c->stats.kernel_launches += 1;
  return B2M_OK;
}

int b2m_trace_read(b2m_ctx* c, int what, int index, void* host_out) {
  if (!c || !host_out) return B2M_EINVAL;
  if (!c->tr.lib) return fail(c, B2M_ESTATE, "call b2m_trace_init first");
  const size_t m = (size_t)c->cfg.num_layers * c->cfg.num_experts;
  CK(c, cudaDeviceSynchronize());
  switch (what) {
    case 0: case 1:
      if (index < 0 || index >= c->tr.max_seqs) return fail(c, B2M_EINVAL, "sequence slot %d out of range", index);
      CK(c, cudaMemcpy(host_out, (what == 0 ? c->tr.seq : c->tr.pred) + m * index, m * sizeof(float), cudaMemcpyDeviceToHost));
      break;
    case 2: CK(c, cudaMemcpy(host_out, c->tr.hint, m * sizeof(float), cudaMemcpyDeviceToHost)); break;
    case 3:
      if (index < 0 || index >= c->tr.capacity) return fail(c, B2M_EINVAL, "library entry %d out of range", index);
      CK(c, cudaMemcpy(host_out, c->tr.lib + m * index, m * sizeof(float), cudaMemcpyDeviceToHost));
      break;
    case 4: CK(c, cudaMemcpy(host_out, c->tr.access, sizeof(int) * c->tr.capacity, cudaMemcpyDeviceToHost)); break;
    case 5:
      if (index < 0 || index >= c->tr.max_seqs) return fail(c, B2M_EINVAL, "sequence slot %d out of range", index);
      CK(c, cudaMemcpy(host_out, c->tr.winner + index, sizeof(int), cudaMemcpyDeviceToHost));
      break;
    default: return fail(c, B2M_EINVAL, "unknown trace item %d", what);
  }
  return B2M_OK;
}

int b2m_timeline_read(b2m_ctx* c, unsigned long long* host_out, int n_layers) {
  if (!c || !host_out) return B2M_EINVAL;
  if (!c->d_tl) return fail(c, B2M_ESTATE, "no timeline recorded (B2M_TIMELINE=1 and b2m_ep_p2p_layer)");
  if (n_layers < 1 || n_layers > c->cfg.num_layers) return fail(c, B2M_EINVAL, "n_layers out of range");
  CK(c, cudaDeviceSynchronize());
  CK(c, cudaMemcpy(host_out, c->d_tl, sizeof(unsigned long long) * 16 * n_layers, cudaMemcpyDeviceToHost));
  return B2M_OK;
}

int b2m_ep_p2p_regroup(b2m_ctx* c, int T_total, void* stream) {
  if (c) c->k3_early_ok = false;
  int r = p2p_ready(c);
  if (r) return r;
  if (T_total < 1 || T_total > c->cap_T) return fail(c, B2M_EINVAL, "T_total=%d exceeds workspace capacity %d", T_total, c->cap_T);
  EpParams p = ep_p2p_params(c);
  c->cur_T = T_total;
  c->cur_nt = c->cur_nt_dn = pick_nt(T_total);
  c->cur_ksplit = pick_ksplit(c, T_total, c->cfg.hidden, c->cfg.inter, c->cfg.num_experts / c->p2p.nranks, c->cfg.top_k, c->cur_nt);
  if (c->cur_ksplit > 1) { p.y_zero = c->d_y; p.y_zero_elems = (size_t)c->p2p.nranks * c->p2p.cap * c->cfg.hidden; }
  CK(c, launch_ep_regroup(p, (cudaStream_t)stream));
  c->stats.kernel_launches += 1;
  c->ep_mode = true;
  return B2M_OK;
}

int b2m_ep_p2p_return(b2m_ctx* c, void* stream) {
  int r = p2p_ready(c);
  if (r) return r;
  EpParams p = ep_p2p_params(c);
  CK(c, launch_ep_ungroup(p, c->cfg.dtype, (cudaStream_t)stream));
  c->stats.kernel_launches += 1;
  return B2M_OK;
}

int b2m_ep_p2p_collect(b2m_ctx* c, int T_local, void* stream) {
  int r = p2p_ready(c);
  if (r) return r;
  if (T_local < 0 || T_local * c->cfg.top_k > c->p2p.cap) return fail(c, B2M_EINVAL, "T_local=%d: T_local*top_k exceeds cap=%d", T_local, c->p2p.cap);
  EpParams p = ep_p2p_params(c);
  CK(c, launch_ep_unpack(p, c->cfg.dtype, T_local * c->cfg.top_k, (cudaStream_t)stream));
  c->stats.kernel_launches += 1;
  return B2M_OK;
}

}  // extern "C"
