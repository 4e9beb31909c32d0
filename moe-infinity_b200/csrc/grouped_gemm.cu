// grouped_gemm.cu -- K3/K4: grouped (per-expert segmented) expert GEMMs on Hopper wgmma tensor cores.
//
// Replaces the per-expert ATen loop of the reference, core/parallel/expert_module.cpp:171-175 (Mixtral),
// :200-203 (DeepSeek), :31-35 (Switch): `matmul(act(matmul(x, w1^T)) * matmul(x, w3^T), w2^T)` issued as
// 3 cuBLAS GEMMs + 2 elementwise kernels per expert from C++ worker threads
// (core/parallel/expert_dispatcher.cpp:309-395).
//
// Design (decode-first, "swap-AB"): the expert weight matrix [M rows, K] (nn.Linear layout, K-major) is the
// wgmma *A* operand (128 rows per tile = two m64 halves, streamed once from HBM by TMA), the expert's tokens
// [n_e, K] are the *B* operand (N = NT in {16,32,64,128,256} tokens).  D[128, NT] accumulates in registers.
// One persistent CTA per SM walks a device-side tile list derived from the per-expert token offsets the
// routing kernel produced -- no host sync.  Roles: warpgroup 0 = TMA producer (one lane); consumer warpgroups
// 1 and 2 each own one 64-row half of the tile (all NT columns): they issue its wgmmas out of the shared-memory ring and
// run the epilogue (activation -> global) from their registers while the producer already fills the ring for the
// next tile.
//   DUAL  = gate and up projections share the token tile and are fused with act(g)*u in the epilogue.
//   !DUAL = single projection: activation epilogue (Switch wi + ReLU) or linear fp32 output
//           (down projection), optionally split-K with fp32 red.add.
#include <string.h>

#include <algorithm>
#include <type_traits>

#include "b2m_common.cuh"
#include "b2m_internal.h"
#include "ep_device.cuh"
#include "tile_walker.cuh"
#include "fp8_weights.cuh"
#include "int4_weights.cuh"
#include "weight_pack.cuh"

namespace b2m {

constexpr int BLOCK_M = 128;   // weight rows per tile
constexpr int BLOCK_K = 64;    // 64 x 16-bit = 128 B = one SWIZZLE_128B row
constexpr int MMA_K = 16;
constexpr int A_TILE_BYTES = BLOCK_M * BLOCK_K * 2;  // 16 KiB
constexpr int MAX_E = 256;
constexpr int SMEM_BUDGET = 216 * 1024;   // of the 227 KiB a block may use on sm_90; the rest holds barriers and tile tables

template <int NT, bool DUAL, int AS = AS_BF16>
struct GemmCfg {
  static constexpr int A_BYTES = (AS == AS_FP8 || AS == AS_FP8_ROW) ? f8::TILE_BYTES : AS == AS_INT4 ? i4::TILE_BYTES : A_TILE_BYTES;   // one A tile of a stage
  static constexpr int B_TILE_BYTES = NT * BLOCK_K * 2;
  static constexpr int STAGE_BYTES = (DUAL ? 2 : 1) * A_BYTES + B_TILE_BYTES;
  static constexpr int STAGES_RAW = SMEM_BUDGET / STAGE_BYTES;
  static constexpr int STAGES = STAGES_RAW > 10 ? 10 : STAGES_RAW;
  // a consumer warpgroup holds a 64 x NT fp32 accumulator (NT/2 registers per thread, twice for DUAL): a DUAL 256-token
  // tile (256 accumulator registers per thread) does not exist
  static constexpr int ACC_REGS = NT / 2;
  static constexpr int CONSUMERS = 2;     // warpgroups: one per 64-row half of the tile
  static constexpr int THREADS = 128 * (1 + CONSUMERS);
  // setmaxnreg split of the CTA's registers: the block is launched with LAUNCH_REGS per thread (what __launch_bounds__ leaves
  // for one block of THREADS per SM, rounded down to the allocation granule of 8); setmaxnreg only moves registers inside
  // that allocation, so the producer warpgroup (one issuing lane) drops to 40 and the consumers take what it frees (a
  // request beyond the allocation would never be granted).  launch_tc checks LAUNCH_REGS against the compiled kernel.
  static constexpr int LAUNCH_REGS = (65536 / THREADS) & ~7;
  // (the packed-weight producer also walks record addresses: 48 keeps it free of spills)
  static constexpr int PRODUCER_REGS = AS == AS_PK12 ? 48 : 40;
  static constexpr int CONSUMER_REGS_RAW = (LAUNCH_REGS * THREADS - 128 * PRODUCER_REGS) / (128 * CONSUMERS);
  static constexpr int CONSUMER_REGS = (CONSUMER_REGS_RAW > 240 ? 240 : CONSUMER_REGS_RAW) & ~7;
  static_assert(PRODUCER_REGS * 128 + CONSUMER_REGS * 128 * CONSUMERS <= LAUNCH_REGS * THREADS, "register split too large");
  static_assert(CONSUMER_REGS >= LAUNCH_REGS, "setmaxnreg.inc must not lower the consumers' count");
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/ +
                                    (MAX_E + 1) * 4 * 2 /*tile_start, offsets*/ + MAX_E * 4 * 3 /*slots, region counts, packed flags*/;
  static_assert(!(DUAL && NT > 128), "DUAL tiles are at most 128 tokens wide");
  static_assert(STAGES >= 2, "need >=2 stages");
  static_assert(SMEM_BYTES <= 227 * 1024, "over the sm_90 shared-memory limit");
  static_assert(wp::REC_BYTES <= A_TILE_BYTES && wp::ROWS == BLOCK_M && wp::COLS == BLOCK_K, "a packed record fills an A slot of the stage");
  static_assert(f8::ROWS == BLOCK_M && f8::COLS == BLOCK_K && A_BYTES % 1024 == 0, "an fp8 tile keeps the stage's 1024-B alignment");
  static_assert(i4::ROWS == BLOCK_M && i4::COLS == BLOCK_K && i4::GROUP == 2 * BLOCK_K, "an int4 tile is one k-block, a group two");
};

__device__ __forceinline__ float act_apply(float x, int act) {
  if (act == ACT_SILU) return x / (1.0f + expf(-x));
  if (act == ACT_RELU) return fmaxf(x, 0.0f);
  if (act == ACT_GELU) return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
  return x;
}

// the four k16 steps of one 64-wide k-block for a 64 x W accumulator
template <int W, int DT>
__device__ __forceinline__ void wgmma_kblock(float (&d)[W / 2], uint64_t da, uint64_t db, bool first) {
#pragma unroll
  for (int k = 0; k < BLOCK_K / MMA_K; ++k) {
    const uint64_t koff = (uint64_t)((k * MMA_K * 2) >> 4);   // advance the start address inside the SW128 atom
    const uint32_t acc = (!first || k > 0) ? 1u : 0u;
    if constexpr (W == 16) wgmma_m64n16k16<DT>(d, da + koff, db + koff, acc);
    else if constexpr (W == 32) wgmma_m64n32k16<DT>(d, da + koff, db + koff, acc);
    else if constexpr (W == 64) wgmma_m64n64k16<DT>(d, da + koff, db + koff, acc);
    else if constexpr (W == 128) wgmma_m64n128k16<DT>(d, da + koff, db + koff, acc);
    else wgmma_m64n256k16<DT>(d, da + koff, db + koff, acc);
  }
}

// expert-parallel direct mode: wait (one thread) until every source rank has published this layer's epoch, i.e. its rows
// and tags have landed in this rank's receive area.  Called by every thread that goes on to read peer-written data with
// ordinary loads (the acquire orders that thread's own later reads); the TMA producer adds a generic->async proxy fence.
__device__ __forceinline__ int ep_gemm_wait(const GemmParams& p) {
  const int want = *reinterpret_cast<const volatile int*>(p.ep_epoch);
  for (int r = 0; r < p.ep_nranks; ++r)
    while (ld_acquire_sys(p.ep_flag + r) < want) __nanosleep(32);
  return want;
}

// How a phase waits for the data its token operand depends on
enum : int { DEP_PDL = 0,     // griddepcontrol.wait: the predecessor kernel in the stream (stand-alone launches)
             DEP_GRID = 1 };  // fused gate/up + down kernel: every CTA of THIS grid has finished the gate/up phase
struct GridBar {
  int* word;   // [0] arrival counter, [1] generation (bumped by the last arriver)
  int gen;     // generation observed at kernel start
};
__device__ __forceinline__ void grid_bar_wait(const GridBar& g) {
  int v;
  do {
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(g.word + 1) : "memory");
    if (v == g.gen) __nanosleep(20);
  } while (v == g.gen);
}

// One grouped GEMM over the device-side tile list: a TMA producer and the wgmma consumer warpgroups over a shared-memory ring.
// Used as the whole body of grouped_gemm_tc_kernel and, twice, by fused_ffn_kernel (gate/up phase, grid barrier, down phase).
// `ctas` = how many CTAs of the grid take tiles of this phase.  REGSPLIT: rebalance registers between producer and consumers
// (once per kernel: the two-phase fused kernel keeps the even split).
// PK (bf16, NT <= 64, MC == 1, no dual_m / m_rows / expert-parallel regions): a weight matrix whose packed copy is current
// (p.pk_ok) streams as 12-bit records (weight_pack.cuh) with one bulk copy per (tile, k-block); the consumers decode their A
// fragments into registers and issue register-A wgmmas.  Other matrices take the bf16 TMA path.
// FP8 (AS_FP8: bf16, MC == 1, no m_rows / expert-parallel regions; every tile width): the A maps are uint8 maps over e4m3
// matrices; the producer loads 8-KiB e4m3 tiles and the consumers dequantise their fragments with the tile's block scale
// (fp8_weights.cuh) into the same register-A wgmmas, over the same tile walk and launch plan as the bf16 engine.
// FP8_ROW (AS_FP8_ROW: as FP8, with one scale per weight row): each consumer thread loads the scales of its two rows once per
// tile and dequantises every k-block with them.
// INT4 (AS_INT4: same restrictions and plan as FP8, but bf16 or f16 -- the group scales are of the activations' type): the A
// maps are uint8 maps over the 4-bit code matrices (32-byte rows); the producer loads 4-KiB code tiles and the consumers
// dequantise their fragments with the group words of their rows (int4_weights.cuh), read from the tile-major group grids
// one k-block ahead.
template <int NT, bool DUAL, int DT, int MC, bool REGSPLIT = true, int AS = AS_BF16>
__device__ __forceinline__ void gemm_body(const CUtensorMap& tmA0, const CUtensorMap& tmA1, const CUtensorMap& tmB,
                                          const GemmParams& p, uint8_t* smem, int dep_mode, const GridBar& gbar, int ctas) {
  using Cfg = GemmCfg<NT, DUAL, AS>;
  constexpr bool PK = AS == AS_PK12, F8 = AS == AS_FP8 || AS == AS_FP8_ROW, F8R = AS == AS_FP8_ROW, I4 = AS == AS_INT4;
  constexpr int A_BYTES = Cfg::A_BYTES;
  // carve shared memory: [stages | barriers | tile tables]
  uint8_t* stage_base = smem;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::STAGES * Cfg::STAGE_BYTES);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + Cfg::STAGES;
  int* tile_start = reinterpret_cast<int*>(empty_bar + Cfg::STAGES);
  int* offs = tile_start + (MAX_E + 1);
  int* slots = offs + (MAX_E + 1);
  int* cnts = slots + MAX_E;           // direct mode: rows per expert region
  int* pkf = cnts + MAX_E;             // PK: pk_ok of each expert's slot
  static_assert(!PK || (MC == 1 && DT == DT_BF16 && NT <= 64), "packed weights: bf16 decode-sized tiles");
  static_assert(!F8 || (MC == 1 && DT == DT_BF16), "fp8 weights: bf16 activations, single-CTA tiles");
  static_assert(!I4 || (MC == 1 && (DT == DT_BF16 || DT == DT_F16)), "int4 weights: 16-bit activations, single-CTA tiles");

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int E = p.E;
  const int kblocks = (p.K + BLOCK_K - 1) / BLOCK_K;
  // dual_m: the two A tiles are rows [m0, m0+128) and [m0+128, m0+256) of the SAME matrix sharing one token tile
  // (doubles the arithmetic intensity of the down projection at prefill; the kernel is L2->SM operand-bandwidth bound)
  // m_rows (EP region mode, MC == 1): weight rows a tile really covers (a multiple of 8, <= 128; the A tensor maps carry a box of
  // that many rows).  The MMA still runs M = 128; the tail rows of the stage hold stale bytes and their accumulator rows are
  // dropped in the epilogue.  Lets the host cut I rows into as many tiles as there are SMs (14336 / 112 = 128 <= 132).
  const int m_rows = (MC == 1 && !p.dual_m && p.m_rows > 0) ? p.m_rows : BLOCK_M;
  const int m_step = (DUAL && p.dual_m) ? 2 * BLOCK_M : m_rows;
  const int m_tiles = (p.M + m_step - 1) / m_step;

  // ---- per-phase setup ------------------------------------------------------------
  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA0);
    if (DUAL) tma_prefetch_desc(&tmA1);
    tma_prefetch_desc(&tmB);
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < Cfg::STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      // a stage is free when every consumer warpgroup -- with multicast operands: of every CTA of the cluster -- consumed it
      mbar_init(&empty_bar[s], Cfg::CONSUMERS * MC);
    }
    fence_barrier_init();
  }
  // Expert parallel (direct mode): this kernel's CTAs are resident while the routing kernel is still exchanging rows with the peers
  // and the previous layer's combine waits for its owners, so HBM idles at the start of every layer.
  // Each CTA asks the TMA unit to pull the first ep_l2pf k-blocks of the weight tiles it will most likely own (one token tile
  // per local expert: tile = le * m_tiles + m) into L2.  A hint only: a wrong guess costs bandwidth, never correctness.  The slot
  // table is older than any predecessor in the stream.
  if (p.ep_l2pf > 0 && p.ep_rows > 0 && warp == 0 && lane == 0 && (int)blockIdx.x < ctas && MC == 1) {
    const int npf = p.ep_l2pf < kblocks ? p.ep_l2pf : kblocks;
    for (int tile = blockIdx.x; tile < p.ep_el * m_tiles; tile += ctas) {
      const int slot = p.slot_of[p.ep_first + tile / m_tiles];
      const int m0 = (tile % m_tiles) * m_step;
      if (slot < 0) continue;
      for (int kb = 0; kb < npf; ++kb) {
        tma_prefetch_3d(&tmA0, kb * BLOCK_K, m0, slot);
        if (DUAL) tma_prefetch_3d(&tmA1, kb * BLOCK_K, m0, slot);
      }
    }
  }
  // everything above is on-chip; from here on we touch memory earlier kernels produced.  In early_a mode (down projection
  // launched with a programmatic edge behind the gate/up GEMM) only the token-tile loads depend on the predecessor: the
  // producer prefetches weight tiles first and waits later; the routing tables read below are older than the predecessor.
  if (!p.early_a && dep_mode == DEP_PDL) pdl_wait();
  if (p.pdl_edge && dep_mode == DEP_PDL) pdl_launch();
  if (p.single_n >= 0) {
    if (threadIdx.x == 0) { offs[0] = 0; offs[1] = p.single_n; slots[0] = p.single_slot; }
  } else if (p.ep_rows > 0) {
    // direct mode: local expert le owns rows [le*ep_rows, le*ep_rows + cnt[le]) of the receive area; the counts are final
    // once every source rank has published this layer's flag
    if (threadIdx.x == 0) {
      ep_gemm_wait(p);
      fence_proxy_async_global();          // this thread is also the TMA producer: its later bulk loads read the peers' rows
      if (p.tl && p.ep_wait) tl_max(p.tl + 1);
    }
    __syncthreads();
    for (int i = threadIdx.x; i <= E; i += Cfg::THREADS) {
      int le = i - p.ep_first;
      le = le < 0 ? 0 : (le > p.ep_el ? p.ep_el : le);
      offs[i] = le * p.ep_rows;
    }
    for (int i = threadIdx.x; i < E; i += Cfg::THREADS) {
      slots[i] = p.slot_of[i];
      const int le = i - p.ep_first;
      cnts[i] = (le >= 0 && le < p.ep_el) ? __ldcg(p.ep_cnt + le) : 0;
    }
  } else {
    for (int i = threadIdx.x; i <= E; i += Cfg::THREADS) offs[i] = p.offsets[i];
    for (int i = threadIdx.x; i < E; i += Cfg::THREADS) slots[i] = p.slot_of[i];
  }
  __syncthreads();
  if constexpr (PK) {
    for (int i = threadIdx.x; i < E; i += Cfg::THREADS) pkf[i] = slots[i] >= 0 ? p.pk_ok[slots[i]] : 0;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int e = 0; e < E; ++e) {
      tile_start[e] = acc;
      const int n_e = p.ep_rows > 0 ? cnts[e] : offs[e + 1] - offs[e];
      if (n_e > 0 && slots[e] >= 0) acc += m_tiles * (((n_e + NT - 1) / NT + MC - 1) / MC) * (p.stream_k ? 1 : p.ksplit);
    }
    tile_start[E] = acc;
  }
  __syncthreads();
  const int crank = MC > 1 ? (int)cluster_ctarank() : 0;
  if (MC > 1) cluster_sync_all();   // peers' barriers are initialised before any multicast targets them

  TileWalker walker{tile_start, offs, slots, E, NT, p.stream_k ? 1 : p.ksplit, kblocks, 0, m_step, MC, crank, 0, 0, 0,
                    p.ep_rows > 0 ? cnts : nullptr};
  if (MC == 1 && p.stream_k) {
    const long long units = (long long)tile_start[E] * kblocks;
    walker.stream = 1;
    walker.u_cur = (int)blockIdx.x < ctas ? (int)(units * blockIdx.x / ctas) : 0;
    walker.u_end = (int)blockIdx.x < ctas ? (int)(units * (blockIdx.x + 1) / ctas) : 0;
  }
  TileInfo t;
  // tiles are dealt to clusters; in the fused kernel a phase may use fewer CTAs than the grid has (ctas): the rest take none
  const int tile_stride = ctas / MC;
  const int tile0 = (int)blockIdx.x < ctas ? (int)blockIdx.x / MC : 0x3fffffff;

  if (warp < 4) {
    if constexpr (REGSPLIT) setmaxnreg_dec<Cfg::PRODUCER_REGS>();
    // ===================== TMA producer (one lane) =====================
    if (warp == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      bool waited = !p.early_a;
      int npend = 0, pend_stage[Cfg::STAGES], pend_kb[Cfg::STAGES], pend_row[Cfg::STAGES];
      for (int tile = tile0; walker.get(tile, t); tile += tile_stride) {
        // packed records stream only when every A matrix of the tile has a current packed copy (the consumers decide the same)
        const bool pk0 = PK && ((pkf[t.e] >> p.pk_bit0) & 1) && (!DUAL || ((pkf[t.e] >> p.pk_bit1) & 1));
        // packed records of this tile's k-blocks: (m-tile, k-block) order inside the slot's copy of the matrix
        const uint8_t* rec = pk0 ? p.pk_a0 + (size_t)t.slot * p.pk_slot_bytes + (size_t)(t.m0 / BLOCK_M) * kblocks * wp::REC_BYTES
                                 : nullptr;
        for (int kb = t.kb_begin; kb < t.kb_end; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sA0 = stage_base + stage * Cfg::STAGE_BYTES;
          uint8_t* sA1 = sA0 + A_BYTES;
          uint8_t* sB = sA0 + (DUAL ? 2 : 1) * A_BYTES;
          const int a_bytes = I4 ? m_rows * i4::ROW_BYTES : m_rows * BLOCK_K * (F8 ? 1 : 2);
          mbar_arrive_expect_tx(&full_bar[stage], (DUAL ? 2 : 1) * (pk0 ? wp::REC_BYTES : a_bytes) + Cfg::B_TILE_BYTES);
          // decode: weights are streamed exactly once -> evict-first.  Several n-tiles per expert (prefill): the same
          // weight tile is re-read by every n-tile -> keep it in L2.  Tokens are re-read by every m-tile: keep.
          const uint64_t wh = ((p.ep_rows > 0 ? cnts[t.e] : offs[t.e + 1] - offs[t.e]) <= NT) ? CACHE_EVICT_FIRST : CACHE_EVICT_NORMAL;
          if (MC == 1) {
            if (pk0) {
              bulk_load(&full_bar[stage], sA0, rec + (size_t)kb * wp::REC_BYTES, wp::REC_BYTES, wh);
              if (DUAL) bulk_load(&full_bar[stage], sA1, rec + (p.pk_a1 - p.pk_a0) + (size_t)kb * wp::REC_BYTES, wp::REC_BYTES, wh);
            } else {
              // (k coordinate of the A maps: int4 maps count bytes, two codes each)
              tma_load_3d(&tmA0, &full_bar[stage], sA0, I4 ? kb * i4::ROW_BYTES : kb * BLOCK_K, t.m0, t.slot, wh);
              if (DUAL)
                tma_load_3d(&tmA1, &full_bar[stage], sA1, I4 ? kb * i4::ROW_BYTES : kb * BLOCK_K, t.m0 + (p.dual_m ? BLOCK_M : 0),
                            t.slot, wh);
            }
          } else {
            // 2-CTA multicast: the cluster's CTAs work on the same weight tiles and adjacent token tiles; each CTA fetches
            // HALF of every weight tile (64 rows; tmA* carry 64-row boxes) and multicasts it into both CTAs' stages, so
            // a CTA pulls 16+16 KB instead of 32+16 KB per k-block from L2
            const int half = crank * (BLOCK_M / 2);          // rows this CTA fetches
            const int hoff = crank * (A_TILE_BYTES / 2);     // where they sit inside the 128-row stage tile
            tma_load_3d_mc(&tmA0, &full_bar[stage], sA0 + hoff, kb * BLOCK_K, t.m0 + half, t.slot, (uint16_t)0x3, wh);
            if (DUAL)
              tma_load_3d_mc(&tmA1, &full_bar[stage], sA1 + hoff, kb * BLOCK_K,
                             t.m0 + (p.dual_m ? BLOCK_M : 0) + half, t.slot, (uint16_t)0x3, wh);
          }
          if (!waited) {
            // weight tiles of the first pipeline fill are in flight before the predecessor has finished; their token
            // tiles follow once it has
            pend_stage[npend] = stage; pend_kb[npend] = kb; pend_row[npend] = t.row0;
            if (++npend == Cfg::STAGES) {
              if (dep_mode == DEP_PDL) pdl_wait(); else { grid_bar_wait(gbar); fence_proxy_async_global(); }
              for (int i = 0; i < npend; ++i)
                tma_load_2d(&tmB, &full_bar[pend_stage[i]], stage_base + pend_stage[i] * Cfg::STAGE_BYTES + (DUAL ? 2 : 1) * A_BYTES,
                            pend_kb[i] * BLOCK_K, pend_row[i], CACHE_EVICT_LAST);
              waited = true;
            }
          } else {
            tma_load_2d(&tmB, &full_bar[stage], sB, kb * BLOCK_K, t.row0, CACHE_EVICT_LAST);
          }
          if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
        }
      }
      if (!waited) {   // fewer work items than pipeline stages
        if (dep_mode == DEP_PDL) pdl_wait(); else { grid_bar_wait(gbar); fence_proxy_async_global(); }
        for (int i = 0; i < npend; ++i)
          tma_load_2d(&tmB, &full_bar[pend_stage[i]], stage_base + pend_stage[i] * Cfg::STAGE_BYTES + (DUAL ? 2 : 1) * A_BYTES,
                      pend_kb[i] * BLOCK_K, pend_row[i], CACHE_EVICT_LAST);
      }
    }
  } else {
    if constexpr (REGSPLIT) setmaxnreg_inc<Cfg::CONSUMER_REGS>();
    // ===================== consumer warpgroups: wgmma + epilogue =====================
    if (p.early_a && dep_mode == DEP_PDL) pdl_wait();
    const int ct = threadIdx.x - 128;    // thread index among all consumers
    if (p.ep_rows > 0 && p.ep_zero) {
      // clear the down projection's accumulator: safe now -- a source rank publishes this layer's flag only after its
      // combine of the previous layer has finished reading the previous outputs
      float4* z = reinterpret_cast<float4*>(p.ep_zero);
      const size_t n4 = p.ep_zero_elems / 4;
      const int et = Cfg::CONSUMERS * 128;
      for (size_t i = (size_t)blockIdx.x * et + ct; i < n4; i += (size_t)gridDim.x * et)
        z[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    const int mh = ct >> 7;                  // consumer warpgroup = row half of the tile
    const bool signaller = (ct & 127) == 0;  // releases ring stages for its warpgroup
    const int ra = mh * 64 + ((ct & 127) >> 5) * 16 + (lane >> 2);   // tile rows of this thread: ra, ra + 8
    const int cb = (lane & 3) * 2;                                   // token columns: cb + 8j + {0, 1}
    float acc0[Cfg::ACC_REGS];
    float acc1[DUAL ? Cfg::ACC_REGS : 1];
    int stage = 0;
    uint32_t phase = 0;
    auto release = [&](int s) {
      if (!signaller) return;
      if (MC == 1) mbar_arrive(&empty_bar[s]);
      else for (int c = 0; c < MC; ++c) mbar_arrive_cluster(&empty_bar[s], (uint32_t)c);   // the peer multicasts into it too
    };
    // PK / F8: decoded A fragments, double-buffered -- the wgmmas of the k-block in flight still read one buffer while the next
    // k-block is decoded into the other (wgmma_wait<1> retires the older one).  The fp8 DUAL 128-token tile keeps ONE buffer:
    // beside its 128 accumulator registers a second one spills.  Its decode then waits for the previous k-block's wgmmas; the
    // other consumer warpgroup's wgmmas keep the tensor cores busy meanwhile (this width only runs at prefill).
    constexpr int FRAG_BUFS = ((F8 || I4) && DUAL && NT == 128) ? 1 : 2;
    uint32_t fa0[FRAG_BUFS][16], fa1[FRAG_BUFS][16];   // (unused without PK / F8 / I4)
    for (int tile = tile0; walker.get(tile, t); tile += tile_stride) {
      int prev = -1;
      auto next_stage = [&]() {
        wgmma_commit();
        wgmma_fence_regs(acc0);
        if (DUAL) wgmma_fence_regs(acc1);
        wgmma_wait<1>();                 // the previous k-block's wgmmas have read their operands: that stage may be refilled
        if (prev >= 0) release(prev);
        prev = stage;
        if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
      };
      // one k-block, A from the bf16 tile in shared memory
      auto kblock_smem = [&](int kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t a0 = smem_u32(stage_base + stage * Cfg::STAGE_BYTES) + mh * (64 * BLOCK_K * 2);
        const uint32_t b = smem_u32(stage_base + stage * Cfg::STAGE_BYTES + (DUAL ? 2 : 1) * A_BYTES);
        wgmma_fence_regs(acc0);
        if (DUAL) wgmma_fence_regs(acc1);
        wgmma_fence();
        wgmma_kblock<NT, DT>(acc0, make_kmajor_sw128_desc(a0), make_kmajor_sw128_desc(b), kb == t.kb_begin);
        if constexpr (DUAL) wgmma_kblock<NT, DT>(acc1, make_kmajor_sw128_desc(a0 + A_BYTES), make_kmajor_sw128_desc(b), kb == t.kb_begin);
        next_stage();
      };
      // FP8: block scales of this tile's A0 / A1 rows (dual_m: A1 is the next 128-row tile of the same matrix, clamped to the
      // matrix -- a tile past its end holds TMA's zero fill and its rows are dropped).  One fp32 per 128 k, loaded one k-block
      // ahead of its use.
      const float* sc0 = nullptr;
      const float* sc1 = nullptr;
      float sn0 = 0.f, sn1 = 0.f;
      if constexpr (F8 && !F8R) {
        const int kbs = p.K / f8::BLOCK, mt = t.m0 / BLOCK_M, mts = p.M / BLOCK_M;
        sc0 = reinterpret_cast<const float*>(p.grid0 + (size_t)t.slot * p.grid_slot_bytes) + (size_t)mt * kbs;
        sc1 = DUAL ? reinterpret_cast<const float*>(p.grid1 + (size_t)t.slot * p.grid_slot_bytes) +
                         (size_t)(p.dual_m && mt + 1 < mts ? mt + 1 : mt) * kbs
                   : sc0;
        sn0 = __ldg(sc0 + t.kb_begin / 2);
        if (DUAL) sn1 = __ldg(sc1 + t.kb_begin / 2);
      }
      // INT4: group words of this thread's rows ra, ra + 8 in A0 / A1 (tile-major grids: the 128 rows of a tile's group are
      // contiguous; dual_m as for FP8).  One word per row and 128 k, loaded one k-block ahead of its use.
      struct I4Groups {
        const uint32_t* w[2];   // A0 / A1: word of row ra in group 0 of the tile
        uint32_t cur[2][2];     // [A0 / A1][row ra / ra + 8]: words of the k-block being decoded ...
        uint32_t nxt[2][2];     // ... and of the next one
        __device__ __forceinline__ void load(int kb) {
          const int g = kb / 2;
#pragma unroll
          for (int a = 0; a < (DUAL ? 2 : 1); ++a) {
            nxt[a][0] = __ldg(w[a] + g * BLOCK_M);
            nxt[a][1] = __ldg(w[a] + g * BLOCK_M + 8);
          }
        }
      };
      struct NoGroups {};
      std::conditional_t<I4, I4Groups, NoGroups> grp;
      if constexpr (I4) {
        const int gs = p.K / i4::GROUP, mt = t.m0 / BLOCK_M, mts = p.M / BLOCK_M;
        grp.w[0] = reinterpret_cast<const uint32_t*>(p.grid0 + (size_t)t.slot * p.grid_slot_bytes) + (size_t)mt * gs * BLOCK_M + ra;
        grp.w[1] = DUAL ? reinterpret_cast<const uint32_t*>(p.grid1 + (size_t)t.slot * p.grid_slot_bytes) +
                              (size_t)(p.dual_m && mt + 1 < mts ? mt + 1 : mt) * gs * BLOCK_M + ra
                        : grp.w[0];
        grp.load(t.kb_begin);
      }
      // FP8_ROW: scales of this thread's rows ra, ra + 8 in A0 / A1 (dual_m as for FP8; a row past the matrix -- TMA zero fill,
      // dropped in the epilogue -- gets 0), loaded once per tile
      float rs[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
      if constexpr (F8R) {
        const float* r0 = reinterpret_cast<const float*>(p.grid0 + (size_t)t.slot * p.grid_slot_bytes);
        const float* r1 = reinterpret_cast<const float*>(p.grid1 + (size_t)t.slot * p.grid_slot_bytes);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int m = t.m0 + ra + 8 * h, m1 = m + (p.dual_m ? BLOCK_M : 0);
          rs[0][h] = m < p.M ? __ldg(r0 + m) : 0.f;
          if (DUAL) rs[1][h] = m1 < p.M ? __ldg(r1 + m1) : 0.f;
        }
      }
      // one k-block, A decoded from packed records / dequantised from e4m3 into fragment buffer BUF (compile time)
      auto kblock_packed = [&](int kb, auto BUF) {
        constexpr int bf = decltype(BUF)::value;
        float s0 = 0.f, s1 = 0.f;
        if constexpr (F8 && !F8R) {
          s0 = sn0;
          s1 = sn1;
          if (kb + 1 < t.kb_end) {
            sn0 = __ldg(sc0 + (kb + 1) / 2);
            if (DUAL) sn1 = __ldg(sc1 + (kb + 1) / 2);
          }
        }
        if constexpr (I4) {
#pragma unroll
          for (int a = 0; a < 2; ++a) { grp.cur[a][0] = grp.nxt[a][0]; grp.cur[a][1] = grp.nxt[a][1]; }
          if (kb + 1 < t.kb_end) grp.load(kb + 1);
        }
        mbar_wait(&full_bar[stage], phase);
        if constexpr (FRAG_BUFS == 1) wgmma_wait<0>();   // the previous k-block's wgmmas have read the fragments
        const uint8_t* sa = stage_base + stage * Cfg::STAGE_BYTES;
        if constexpr (F8R) {
          f8::decode_lane(sa, ct, rs[0][0], rs[0][1], fa0[bf]);
          if constexpr (DUAL) f8::decode_lane(sa + A_BYTES, ct, rs[1][0], rs[1][1], fa1[bf]);
        } else if constexpr (F8) {
          f8::decode_lane(sa, ct, s0, fa0[bf]);
          if constexpr (DUAL) f8::decode_lane(sa + A_BYTES, ct, s1, fa1[bf]);
        } else if constexpr (I4) {
          i4::decode_lane<typename Half16<DT>::T>(sa, ct, grp.cur[0][0], grp.cur[0][1], fa0[bf]);
          if constexpr (DUAL) i4::decode_lane<typename Half16<DT>::T>(sa + A_BYTES, ct, grp.cur[1][0], grp.cur[1][1], fa1[bf]);
        } else {
          wp::decode_lane(sa, ct, fa0[bf]);
          if constexpr (DUAL) wp::decode_lane(sa + A_BYTES, ct, fa1[bf]);
        }
        const uint64_t db = make_kmajor_sw128_desc(smem_u32(sa + (DUAL ? 2 : 1) * A_BYTES));
        wgmma_fence_regs(acc0);
        if (DUAL) wgmma_fence_regs(acc1);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / MMA_K; ++k) {
          const uint64_t koff = (uint64_t)((k * MMA_K * 2) >> 4);
          const uint32_t acc = (kb != t.kb_begin || k > 0) ? 1u : 0u;
          wgmma_rs<NT, DT>(acc0, fa0[bf][4 * k], fa0[bf][4 * k + 1], fa0[bf][4 * k + 2], fa0[bf][4 * k + 3], db + koff, acc);
          if constexpr (DUAL)
            wgmma_rs<NT, DT>(acc1, fa1[bf][4 * k], fa1[bf][4 * k + 1], fa1[bf][4 * k + 2], fa1[bf][4 * k + 3], db + koff, acc);
        }
        next_stage();
      };
      // a tile streams packed records when every A matrix it reads has a current packed copy (the producer decides the same)
      bool packed = F8 || I4;
      if constexpr (PK) packed = ((pkf[t.e] >> p.pk_bit0) & 1) && (!DUAL || ((pkf[t.e] >> p.pk_bit1) & 1));
      if (!packed) {
        if constexpr (!F8 && !I4)
          for (int kb = t.kb_begin; kb < t.kb_end; ++kb) kblock_smem(kb);
      } else if constexpr (PK || F8 || I4) {
        for (int kb = t.kb_begin; kb < t.kb_end; ++kb) {
          kblock_packed(kb, std::integral_constant<int, 0>{});
          if (++kb >= t.kb_end) break;
          kblock_packed(kb, std::integral_constant<int, FRAG_BUFS - 1>{});
        }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc0);
      if (DUAL) wgmma_fence_regs(acc1);
      if (prev >= 0) release(prev);

      float bias0[2] = {0.f, 0.f}, bias1[2] = {0.f, 0.f};   // bias experts: one value per weight row
      bool row_ok[2], row2_ok[2];
      int mrow[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = ra + 8 * h;
        mrow[h] = t.m0 + r;
        row_ok[h] = mrow[h] < p.M && r < m_rows;
        row2_ok[h] = DUAL && mrow[h] + BLOCK_M < p.M;   // dual_m: second accumulator = rows m0+128..m0+255
        if (p.bias_base) {
          const uint16_t* bp = reinterpret_cast<const uint16_t*>(p.bias_base) + (size_t)t.slot * p.bias_slot_elems + p.bias_off;
          if (row_ok[h]) bias0[h] = Half16<DT>::to_f(bp[mrow[h]]);
          if (row2_ok[h]) bias1[h] = Half16<DT>::to_f(bp[mrow[h] + BLOCK_M]);
        }
      }
#pragma unroll
      for (int j = 0; j < NT / 8; ++j) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int h = i >> 1;
          const int c = cb + 8 * j + (i & 1);
          if (c >= t.ncols) continue;
          const int m = mrow[h];
          if (p.epi == EPI_LINEAR_F32) {
            float* dst = reinterpret_cast<float*>(p.out) + (size_t)(t.row0 + c) * p.ld_out + m;
            if (row_ok[h]) {
              float v = acc0[4 * j + i];
              if (p.bias_base) v = p.mimic ? round_dt<DT>(round_dt<DT>(v) + bias0[h]) : v + bias0[h];   // matmul, then `+ bias`
              if (p.ksplit > 1) atomicAdd(dst, v); else *dst = v;
            }
            if (DUAL && row2_ok[h]) {
              float v = acc1[DUAL ? 4 * j + i : 0];
              if (p.bias_base) v = p.mimic ? round_dt<DT>(round_dt<DT>(v) + bias1[h]) : v + bias1[h];
              if (p.ksplit > 1) atomicAdd(dst + BLOCK_M, v); else dst[BLOCK_M] = v;
            }
          } else if (row_ok[h]) {
            float g = acc0[4 * j + i];
            float hv;
            if (DUAL) {
              float u = acc1[DUAL ? 4 * j + i : 0];
              if (p.mimic) {   // reference rounding chain: each ATen op rounds to the model dtype
                g = round_dt<DT>(g);
                u = round_dt<DT>(u);
                hv = round_dt<DT>(act_apply(g, p.act)) * u;
              } else {
                hv = act_apply(g, p.act) * u;
              }
            } else {
              if (p.mimic) g = round_dt<DT>(g);
              if (p.bias_base) { g += bias0[h]; if (p.mimic) g = round_dt<DT>(g); }
              hv = act_apply(g, p.act);
            }
            reinterpret_cast<uint16_t*>(p.out)[(size_t)(t.row0 + c) * p.ld_out + m] = Half16<DT>::from_f(hv);
          }
        }
      }
    }
  }

  // ---- end of the phase: every role of this CTA is done with the ring and the barriers
  __syncthreads();
}

// after the last phase of a kernel: timeline and the expert-parallel "done" signal
template <int MC>
__device__ __forceinline__ void gemm_finish(const GemmParams& p) {
  if (p.tl && threadIdx.x == 0) tl_max(p.tl + 2);
  if (p.ep_signal && threadIdx.x == 0) {
    // the CTA's output stores / reductions (all threads, ordered before this point by the barrier that ended the phase) become
    // visible system-wide with ONE fence (fences are cumulative); the last CTA of the grid then tells the source ranks, whose
    // combine kernels read the rows in place over NVLink
    __threadfence_system();
    if (atomicAdd(p.ep_done_ctr, 1) == (int)gridDim.x - 1) {
      *p.ep_done_ctr = 0;
      for (int le = 0; le < p.ep_el; ++le) p.ep_cnt[le] = 0;   // every CTA has read the counts: regions are free for the next layer
      const int e = *p.ep_done_epoch + 1;
      *p.ep_done_epoch = e;
      __threadfence_system();   // the other CTAs' fenced outputs and the counter reset happen-before the flags; the flag stores
      for (int r = 0; r < p.ep_nranks; ++r) st_relaxed_sys(p.ep_peer_done_flag[r] + p.ep_rank, e);   // themselves go out back to back
    }
  }
  if (MC > 1) cluster_sync_all();   // no CTA leaves while a peer may still multicast into or arrive on its shared memory
}

__device__ __forceinline__ uint8_t* smem_aligned(uint8_t* raw) {
  return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(raw) + 1023) & ~uintptr_t(1023));
}

template <int NT, bool DUAL, int DT, int MC, int AS>
__device__ __forceinline__ void tc_kernel_body(const CUtensorMap& tmA0, const CUtensorMap& tmA1, const CUtensorMap& tmB,
                                               const GemmParams& p, uint8_t* smem_raw) {
  uint8_t* smem = smem_aligned(smem_raw);
  if (p.tl && threadIdx.x == 0) tl_min(p.tl);
  // pdl_edge: this grid may be resident long before its predecessor finishes (expert parallel: the gate/up GEMM arrives behind the
  // routing kernel to prefetch weights into L2).  Its successor reads state the predecessor publishes (dispatch epoch, row
  // counters) in ITS prologue, so it must not be released before this grid has passed its own wait: gemm_body triggers then.
  if (!p.pdl_edge) pdl_launch();
  GridBar nobar{nullptr, 0};
  gemm_body<NT, DUAL, DT, MC, true, AS>(tmA0, tmA1, tmB, p, smem, DEP_PDL, nobar, (int)gridDim.x);
  gemm_finish<MC>(p);
}

template <int NT, bool DUAL, int DT, int MC, int AS>
__global__ void __launch_bounds__((GemmCfg<NT, DUAL, AS>::THREADS), 1)
grouped_gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
                       const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  tc_kernel_body<NT, DUAL, DT, MC, AS>(tmA0, tmA1, tmB, p, smem_raw);
}

// The same GEMM for row-scaled fp8 experts (AS_FP8_ROW: bf16, MC == 1) under a name of its own, so that profiles and the
// library's SASS tell the two fp8 formats' kernels apart.
template <int NT, bool DUAL>
__global__ void __launch_bounds__((GemmCfg<NT, DUAL, AS_FP8_ROW>::THREADS), 1)
grouped_gemm_fp8_row_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
                            const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  tc_kernel_body<NT, DUAL, DT_BF16, 1, AS_FP8_ROW>(tmA0, tmA1, tmB, p, smem_raw);
}

#ifdef B2M_ENABLE_FUSED_FFN
// (Experiment, NOT part of the default library: a persistent barrier kernel keeps the side-stream shared-expert GEMMs off the
// SMs.  Build with -DB2M_ENABLE_FUSED_FFN and run with B2M_FUSED_FFN=1.)
// Fused expert FFN for the HBM-bound (decode) regime: gate/up GEMM + SwiGLU, grid-wide barrier, down GEMM in ONE persistent
// kernel.  What it removes from every layer: a kernel boundary on the critical path -- the down GEMM's CTAs could only become
// resident when the gate/up CTAs had left their SMs (both want all shared memory), so its barrier set-up, tile tables and
// first pipeline fill were exposed.  Here the
// CTA keeps its resources, re-arms its barriers, starts streaming the down projection's weights at once and only its token
// tiles wait for the grid barrier.  Needs every CTA resident (persistent grid <= #SMs, one CTA per SM: true by construction)
// and no second barrier-kernel running beside it.
template <int NT, int DT>
__global__ void __launch_bounds__((GemmCfg<NT, true>::THREADS), 1)
fused_ffn_kernel(const __grid_constant__ CUtensorMap tmGate, const __grid_constant__ CUtensorMap tmUp,
                 const __grid_constant__ CUtensorMap tmBup, const __grid_constant__ CUtensorMap tmDown,
                 const __grid_constant__ CUtensorMap tmBdn, const GemmParams up, const GemmParams dn, int* gbar_word,
                 int up_ctas) {
  using CfgU = GemmCfg<NT, true>;
  using CfgD = GemmCfg<NT, false>;
  static_assert(CfgU::THREADS == CfgD::THREADS, "both phases run on the same block");
  extern __shared__ uint8_t smem_raw[];
  __shared__ int s_gen;
  uint8_t* smem = smem_aligned(smem_raw);
  if (up.tl && threadIdx.x == 0) tl_min(up.tl);
  pdl_launch();
  if (threadIdx.x == 0) s_gen = *reinterpret_cast<volatile int*>(gbar_word + 1);   // moves only after every CTA of this grid arrived
  __syncthreads();
  GridBar gb{gbar_word, s_gen};
  gemm_body<NT, true, DT, 1, false>(tmGate, tmUp, tmBup, up, smem, DEP_PDL, gb, up_ctas);
  if (threadIdx.x == 0) {
    if (up.tl) tl_max(up.tl + 2);
    if (dn.tl) tl_min(dn.tl);
    __threadfence();                       // this CTA's intermediate rows (all threads, ordered by the barrier that ended the phase)
    if (atomicAdd(gbar_word, 1) == (int)gridDim.x - 1) {
      gbar_word[0] = 0;
      __threadfence();
      asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(gbar_word + 1), "r"(gb.gen + 1) : "memory");
    }
  }
  gemm_body<NT, false, DT, 1, false>(tmDown, tmDown, tmBdn, dn, smem, DEP_GRID, gb, (int)gridDim.x);
  gemm_finish<1>(dn);
}

#endif  // B2M_ENABLE_FUSED_FFN

// --------------------------------------------------------------------------------------
// Plain CUDA-core grouped GEMM with identical semantics (debug / bring-up cross-check only;
// selected with B2M_GEMM_IMPL=simt).  One warp per output element.
// --------------------------------------------------------------------------------------
template <int DT>
__global__ void grouped_gemm_simt_kernel(const uint16_t* __restrict__ arena, size_t slot_elems, size_t offA0,
                                         size_t offA1, const uint16_t* __restrict__ B, int ldb, GemmParams p,
                                         int dual) {
  const bool single = p.single_n >= 0;
  const int total_rows = single ? p.single_n : p.offsets[p.E];
  const long long nout = (long long)total_rows * p.M;
  const int warps_per_block = blockDim.x >> 5;
  const int lane = threadIdx.x & 31;
  for (long long o = (long long)blockIdx.x * warps_per_block + (threadIdx.x >> 5); o < nout;
       o += (long long)gridDim.x * warps_per_block) {
    const int row = (int)(o / p.M);
    const int m = (int)(o % p.M);
    int e = 0;
    if (!single) while (e + 1 < p.E && row >= p.offsets[e + 1]) ++e;
    const int slot = single ? p.single_slot : p.slot_of[e];
    if (slot < 0) continue;
    const uint16_t* a0 = arena + (size_t)slot * slot_elems + offA0 + (size_t)m * p.K;
    const uint16_t* a1 = arena + (size_t)slot * slot_elems + offA1 + (size_t)m * p.K;
    const uint16_t* b = B + (size_t)row * ldb;
    float s0 = 0.f, s1 = 0.f;
    for (int k = lane; k < p.K; k += 32) {
      const float x = Half16<DT>::to_f(b[k]);
      s0 += Half16<DT>::to_f(a0[k]) * x;
      if (dual) s1 += Half16<DT>::to_f(a1[k]) * x;
    }
    for (int d = 16; d; d >>= 1) {
      s0 += __shfl_xor_sync(0xffffffffu, s0, d);
      s1 += __shfl_xor_sync(0xffffffffu, s1, d);
    }
    if (lane == 0) {
      float bias = 0.f;
      if (p.bias_base)
        bias = Half16<DT>::to_f(reinterpret_cast<const uint16_t*>(p.bias_base)[(size_t)slot * p.bias_slot_elems + p.bias_off + m]);
      if (p.epi == EPI_LINEAR_F32) {
        if (p.bias_base) s0 = p.mimic ? round_dt<DT>(round_dt<DT>(s0) + bias) : s0 + bias;
        reinterpret_cast<float*>(p.out)[(size_t)row * p.ld_out + m] = s0;
      } else {
        float g = s0, h;
        if (dual) {
          float u = s1;
          if (p.mimic) { g = round_dt<DT>(g); u = round_dt<DT>(u); h = round_dt<DT>(act_apply(g, p.act)) * u; }
          else h = act_apply(g, p.act) * u;
        } else {
          if (p.mimic) g = round_dt<DT>(g);
          if (p.bias_base) { g += bias; if (p.mimic) g = round_dt<DT>(g); }
          h = act_apply(g, p.act);
        }
        reinterpret_cast<uint16_t*>(p.out)[(size_t)row * p.ld_out + m] = Half16<DT>::from_f(h);
      }
    }
  }
}

// --------------------------------------------------------------------------------------
// host launchers
// --------------------------------------------------------------------------------------
template <int NT, bool DUAL, int DT, int MC, int AS>
static auto tc_kernel() {
  if constexpr (AS == AS_FP8_ROW) {
    static_assert(DT == DT_BF16 && MC == 1, "row-scaled fp8 weights: bf16 activations, single-CTA tiles");
    return grouped_gemm_fp8_row_kernel<NT, DUAL>;
  } else {
    return grouped_gemm_tc_kernel<NT, DUAL, DT, MC, AS>;
  }
}

template <int NT, bool DUAL, int DT, int MC = 1, int AS = AS_BF16>
static cudaError_t launch_tc(const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& b, const GemmParams& p,
                             int grid, cudaStream_t st) {
  using Cfg = GemmCfg<NT, DUAL, AS>;
  auto kern = tc_kernel<NT, DUAL, DT, MC, AS>();
  static bool attr_done = false;   // per-instantiation
  if (!attr_done) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
    if (e != cudaSuccess) return e;
    // the consumers' setmaxnreg.inc is granted from the registers the block was launched with: a kernel compiled to fewer
    // registers per thread than the split assumes would wait forever -> refuse to launch it
    cudaFuncAttributes fa;
    e = cudaFuncGetAttributes(&fa, kern);
    if (e != cudaSuccess) return e;
    if (fa.numRegs != Cfg::LAUNCH_REGS) return cudaErrorInvalidConfiguration;
    attr_done = true;
  }
  if (MC > 1) grid -= grid % MC;
  return launch_cluster(kern, dim3(grid), dim3(Cfg::THREADS), (size_t)Cfg::SMEM_BYTES, st, MC, p.early_a != 0 || p.pdl_edge != 0, a0, a1, b, p);
}

#ifdef B2M_ENABLE_FUSED_FFN
template <int NT, int DT>
static cudaError_t launch_fused(const CUtensorMap& g, const CUtensorMap& u, const CUtensorMap& bup, const CUtensorMap& d,
                                const CUtensorMap& bdn, const GemmParams& up, const GemmParams& dn, int grid, int up_ctas,
                                int* gbar, cudaStream_t st) {
  using CfgU = GemmCfg<NT, true>;
  using CfgD = GemmCfg<NT, false>;
  constexpr int SMEM = CfgU::SMEM_BYTES > CfgD::SMEM_BYTES ? CfgU::SMEM_BYTES : CfgD::SMEM_BYTES;
  auto kern = fused_ffn_kernel<NT, DT>;
  static bool attr_done = false;   // per-instantiation
  if (!attr_done) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    if (e != cudaSuccess) return e;
    attr_done = true;
  }
  return launch_cluster(kern, dim3(grid), dim3(CfgU::THREADS), (size_t)SMEM, st, 1, up.early_a != 0 || up.pdl_edge != 0, g, u, bup, d,
                        bdn, up, dn, gbar, up_ctas);
}

// gate/up + SwiGLU and down projection of the routed experts in one persistent kernel (decode regime: nt <= 128, dual gate/up)
cudaError_t launch_fused_ffn(int dtype, int nt, const CUtensorMap& g, const CUtensorMap& u, const CUtensorMap& bup,
                             const CUtensorMap& d, const CUtensorMap& bdn, const GemmParams& up, const GemmParams& dn, int grid,
                             int up_ctas, int* gbar, cudaStream_t st) {
  if (up.E > MAX_E || grid < 1 || up_ctas < 1 || up_ctas > grid || !gbar) return cudaErrorInvalidValue;
#define B2M_FCASE(N)                                                                                         \
  case N:                                                                                                    \
    return dtype == DT_BF16 ? launch_fused<N, DT_BF16>(g, u, bup, d, bdn, up, dn, grid, up_ctas, gbar, st)   \
                            : launch_fused<N, DT_F16>(g, u, bup, d, bdn, up, dn, grid, up_ctas, gbar, st);
  if (dtype != DT_BF16 && dtype != DT_F16) return cudaErrorInvalidValue;
  switch (nt) {
    B2M_FCASE(16)
    B2M_FCASE(32)
    B2M_FCASE(64)
    B2M_FCASE(128)
    default:
      return cudaErrorInvalidValue;
  }
#undef B2M_FCASE
}

#endif  // B2M_ENABLE_FUSED_FFN

// one kernel per token-tile width for the A source AS (256-token tiles: single projections only, GemmCfg; packed records:
// decode-sized tiles only)
template <int DT, int AS>
static cudaError_t launch_nt(int nt, bool dual, const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& b,
                             const GemmParams& p, int grid, cudaStream_t st) {
  switch (nt) {
    case 16: return dual ? launch_tc<16, true, DT, 1, AS>(a0, a1, b, p, grid, st) : launch_tc<16, false, DT, 1, AS>(a0, a1, b, p, grid, st);
    case 32: return dual ? launch_tc<32, true, DT, 1, AS>(a0, a1, b, p, grid, st) : launch_tc<32, false, DT, 1, AS>(a0, a1, b, p, grid, st);
    case 64: return dual ? launch_tc<64, true, DT, 1, AS>(a0, a1, b, p, grid, st) : launch_tc<64, false, DT, 1, AS>(a0, a1, b, p, grid, st);
  }
  if constexpr (AS != AS_PK12) {
    switch (nt) {
      case 128: return dual ? launch_tc<128, true, DT, 1, AS>(a0, a1, b, p, grid, st) : launch_tc<128, false, DT, 1, AS>(a0, a1, b, p, grid, st);
      case 256: return dual ? cudaErrorInvalidValue : launch_tc<256, false, DT, 1, AS>(a0, a1, b, p, grid, st);
    }
  }
  return cudaErrorInvalidValue;
}

#ifdef B2M_ENABLE_MC2
// 2-CTA multicast variant (prefill: NT = 128, several token tiles per expert); a0/a1 must be the 64-row-box maps.
// Not instantiated in the default build (-DB2M_ENABLE_MC2 brings it back).
cudaError_t launch_grouped_gemm_tc_mc2(int dtype, bool dual, const CUtensorMap& a0h, const CUtensorMap& a1h,
                                       const CUtensorMap& b, const GemmParams& p, int grid, cudaStream_t st) {
  if (p.E > MAX_E) return cudaErrorInvalidValue;
  if (dtype == DT_BF16)
    return dual ? launch_tc<128, true, DT_BF16, 2>(a0h, a1h, b, p, grid, st) : launch_tc<128, false, DT_BF16, 2>(a0h, a1h, b, p, grid, st);
  if (dtype == DT_F16)
    return dual ? launch_tc<128, true, DT_F16, 2>(a0h, a1h, b, p, grid, st) : launch_tc<128, false, DT_F16, 2>(a0h, a1h, b, p, grid, st);
  return cudaErrorInvalidValue;
}
#endif

// --------------------------------------------------------------------------------------
// packing: bf16 slot arena -> 12-bit packed copy (weight_pack.cuh).  One CTA of LANES threads codes one tile at a time, thread L
// the values of consumer lane L; a tile that cannot be coded marks its matrix bad (pk_ok bit 8 + matrix), and the finish kernel
// then publishes pk_ok[slot] = the matrices whose every tile was coded.
// --------------------------------------------------------------------------------------
struct PackArgs {
  const uint8_t* src;
  size_t src_slot_bytes;
  uint8_t* dst;
  size_t dst_slot_bytes;
  size_t src_off[3], dst_off[3];
  int cols[3], kblocks[3];
  long long tiles_before[4];   // prefix sums of the tiles of matrices 0..2 of one slot
  int* ok;
  int n;
  int slots[MAX_E];
};

__global__ void __launch_bounds__(wp::LANES) pack_weights_kernel(const __grid_constant__ PackArgs a) {
  __shared__ int s_max, s_special, s_np;
  __shared__ uint32_t s_patch[wp::MAX_PATCH];
  const int L = threadIdx.x;
  const long long per_slot = a.tiles_before[3];
  for (long long tile = blockIdx.x; tile < per_slot * a.n; tile += gridDim.x) {
    const int slot = a.slots[tile / per_slot];
    long long r = tile % per_slot;
    const int m = r < a.tiles_before[1] ? 0 : r < a.tiles_before[2] ? 1 : 2;
    r -= a.tiles_before[m];
    const int mt = (int)(r / a.kblocks[m]), kb = (int)(r % a.kblocks[m]);
    const uint16_t* src = reinterpret_cast<const uint16_t*>(a.src + (size_t)slot * a.src_slot_bytes + a.src_off[m]) +
                          (size_t)mt * wp::ROWS * a.cols[m] + (size_t)kb * wp::COLS;
    uint8_t* rec = a.dst + (size_t)slot * a.dst_slot_bytes + a.dst_off[m] + (size_t)r * wp::REC_BYTES;
    if (L == 0) { s_max = 0; s_special = 0; s_np = 0; }
    uint16_t u[wp::VALS];
    int me = 0;
    bool special = false;
#pragma unroll
    for (int v = 0; v < wp::VALS; v += 2) {   // values v, v + 1 are adjacent columns of one row
      int row, col;
      wp::lane_coord(L, v, &row, &col);
      const uint32_t two = *reinterpret_cast<const uint32_t*>(src + (size_t)row * a.cols[m] + col);
      u[v] = (uint16_t)two;
      u[v + 1] = (uint16_t)(two >> 16);
    }
#pragma unroll
    for (int v = 0; v < wp::VALS; ++v) {
      const int e = wp::bf16_exp(u[v]);
      special |= e == 255;
      me = e > me ? e : me;
    }
    me = __reduce_max_sync(0xffffffffu, me);
    special = __any_sync(0xffffffffu, special);
    __syncthreads();
    if ((L & 31) == 0) {
      atomicMax(&s_max, me);
      if (special) s_special = 1;
    }
    __syncthreads();
    const int base = wp::window_base(s_max);
    uint16_t pre[wp::VALS];
#pragma unroll
    for (int v = 0; v < wp::VALS; ++v)
      if (!wp::to_pre(u[v], base, &pre[v])) {
        const int i = atomicAdd(&s_np, 1);
        if (i < wp::MAX_PATCH) s_patch[i] = (uint32_t)(L * wp::VALS + v) | ((uint32_t)u[v] << 16);
      }
    __syncthreads();
    const int np = s_np;
    const bool ok = !s_special && base <= wp::MAX_BASE && np <= wp::MAX_PATCH;
    if (ok) {
      uint32_t w[12];
      wp::pack_lane(pre, w);
#pragma unroll
      for (int c = 0; c < 3; ++c)
        *reinterpret_cast<uint4*>(rec + wp::body_word_offset(L, 4 * c)) = make_uint4(w[4 * c], w[4 * c + 1], w[4 * c + 2], w[4 * c + 3]);
    }
    if (L < wp::HDR_BYTES / 4) {
      const int i = L - 4;
      const uint32_t hw = L == 0 ? wp::header_word0(ok ? base : 0, ok ? np : 0, !ok) : (ok && i >= 0 && i < np) ? s_patch[i] : 0u;
      reinterpret_cast<uint32_t*>(rec)[L] = hw;
    }
    if (!ok && L == 0) atomicOr(a.ok + slot, 1 << (8 + m));
    __syncthreads();   // the tile's shared state is reset by the next iteration
  }
}

__global__ void pack_finish_kernel(const __grid_constant__ PackArgs a, int mats) {
  for (int i = threadIdx.x; i < a.n; i += blockDim.x) {
    int* f = a.ok + a.slots[i];
    *f = mats & ~(*f >> 8);
  }
}

static cudaError_t launch_pack(const GemmParams& p, cudaStream_t st) {
  if (p.pack_n > MAX_E || !p.pack_ok || !p.pack_dst || !p.pack_src) return cudaErrorInvalidValue;
  PackArgs a;
  memset(&a, 0, sizeof a);
  a.src = p.pack_src;
  a.src_slot_bytes = p.pack_src_slot_bytes;
  a.dst = p.pack_dst;
  a.dst_slot_bytes = p.pk_slot_bytes;
  a.ok = p.pack_ok;
  a.n = p.pack_n;
  int mats = 0;
  for (int m = 0; m < 3; ++m) {
    const int rows = m < p.pack_nmat ? p.pack_rows[m] : 0, cols = m < p.pack_nmat ? p.pack_cols[m] : 0;
    const bool on = packed_matrix_bytes(rows, cols) > 0 && rows > 0;
    a.src_off[m] = p.pack_src_off[m];
    a.dst_off[m] = p.pack_dst_off[m];
    a.cols[m] = cols;
    a.kblocks[m] = on ? cols / wp::COLS : 1;
    a.tiles_before[m + 1] = a.tiles_before[m] + (on ? (long long)(rows / wp::ROWS) * (cols / wp::COLS) : 0);
    if (on) mats |= 1 << m;
  }
  for (int i = 0; i < p.pack_n; ++i) a.slots[i] = p.pack_slots[i];
  const long long tiles = a.tiles_before[3] * a.n;
  if (tiles == 0) return cudaSuccess;
  pack_weights_kernel<<<(unsigned)std::min<long long>(tiles, (long long)H100_SMS * 8), wp::LANES, 0, st>>>(a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  pack_finish_kernel<<<1, 256, 0, st>>>(a, mats);
  return cudaGetLastError();
}

cudaError_t launch_grouped_gemm_tc(int dtype, int nt, bool dual, const CUtensorMap& a0, const CUtensorMap& a1,
                                   const CUtensorMap& b, const GemmParams& p, int grid, cudaStream_t st) {
  if (p.E > MAX_E) return cudaErrorInvalidValue;
  if (p.pack_n > 0) {
    // pack first, then run this GEMM as a plain stream-ordered launch: its prologue reads the flags the packing just wrote
    cudaError_t e = launch_pack(p, st);
    if (e != cudaSuccess) return e;
    GemmParams q = p;
    q.pack_n = 0;
    q.early_a = 0;
    q.pdl_edge = 0;
    return launch_grouped_gemm_tc(dtype, nt, dual, a0, a1, b, q, grid, st);
  }
  // packed weights: decode-sized tiles only (at prefill the GEMM is tensor-bound and keeps the shared-memory A operand)
  const bool pk = p.pk_ok && nt <= 64 && !p.dual_m && p.m_rows == 0 && p.ep_rows == 0;
  if (dtype == DT_BF16) {
    switch (p.a_src) {
      case AS_BF16: return pk ? launch_nt<DT_BF16, AS_PK12>(nt, dual, a0, a1, b, p, grid, st)
                              : launch_nt<DT_BF16, AS_BF16>(nt, dual, a0, a1, b, p, grid, st);
      case AS_FP8: return launch_nt<DT_BF16, AS_FP8>(nt, dual, a0, a1, b, p, grid, st);
      case AS_FP8_ROW: return launch_nt<DT_BF16, AS_FP8_ROW>(nt, dual, a0, a1, b, p, grid, st);
      case AS_INT4: return launch_nt<DT_BF16, AS_INT4>(nt, dual, a0, a1, b, p, grid, st);
    }
  } else if (dtype == DT_F16) {   // (no packed copy, no fp8 weights)
    switch (p.a_src) {
      case AS_BF16: return launch_nt<DT_F16, AS_BF16>(nt, dual, a0, a1, b, p, grid, st);
      case AS_INT4: return launch_nt<DT_F16, AS_INT4>(nt, dual, a0, a1, b, p, grid, st);
    }
  }
  return cudaErrorInvalidValue;
}

cudaError_t launch_grouped_gemm_simt(int dtype, const void* arena, size_t slot_elems, size_t offA0, size_t offA1,
                                     const void* B, int ldb, const GemmParams& p, bool dual, cudaStream_t st) {
  const int grid = H100_SMS * 8;   // grid-stride loop
  if (dtype == DT_BF16)
    grouped_gemm_simt_kernel<DT_BF16><<<grid, 256, 0, st>>>((const uint16_t*)arena, slot_elems, offA0, offA1,
                                                             (const uint16_t*)B, ldb, p, dual ? 1 : 0);
  else if (dtype == DT_F16)
    grouped_gemm_simt_kernel<DT_F16><<<grid, 256, 0, st>>>((const uint16_t*)arena, slot_elems, offA0, offA1,
                                                            (const uint16_t*)B, ldb, p, dual ? 1 : 0);
  else
    return cudaErrorInvalidValue;
  return cudaGetLastError();
}

}  // namespace b2m
