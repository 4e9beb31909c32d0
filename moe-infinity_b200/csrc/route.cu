// route.cu -- K0/K1/K2/K5: router gate, fused softmax+top-k, token index sort/permute, weighted combine.
//
// Replaces, with zero host synchronisation:
//   * moe_infinity/models/mixtral.py:46-65        gate GEMM, softmax, topk, renorm, dense [T,E] mask build
//   * modeling_deepseek.py:463-512 + deepseek.py:76-91   MoEGate and its mask build
//   * modeling_deepseek_v3/modeling_deepseek.py:466-527  DeepSeek-V3 MoEGate (sigmoid, correction bias, noaux_tc)
//   * distributed/expert_executor.py:34-44         per-expert token counts (.cpu() sync in the reference)
//   * core/parallel/expert_dispatcher.cpp:274-285  per-expert boolean-mask gather (nonzero + index_select)
//   * mixtral.py:96-101 / deepseek.py:123-136 / switch_transformers.py:99-109   per-expert masked combine
// Instead of dense masks the kernels emit: top-k ids/weights, per-expert counts + offsets, a stable
// (ascending token order inside each expert, the reference's gather order) permutation, and the gathered
// activation rows, written with 16-byte vector stores.
#include "b2m_common.cuh"
#include "b2m_internal.h"
#include "ep_device.cuh"

namespace b2m {

constexpr int RT_THREADS = 256;
constexpr int RT_WARPS = RT_THREADS / 32;
constexpr int CHUNK = 32;                      // tokens per ranking chunk (one warp, lane == token)
constexpr int TOK_PER_BLOCK = CHUNK * RT_WARPS;  // 256
constexpr int MAX_K = 8;
constexpr int MAX_PL = 8;                      // experts per lane  -> E <= 256
constexpr int FUSED_MAX_T = TOK_PER_BLOCK;     // single-CTA fused path

__device__ __forceinline__ float load_as_float(const void* p, size_t i, int dt) {
  if (dt == DT_F32) return reinterpret_cast<const float*>(p)[i];
  const uint16_t b = reinterpret_cast<const uint16_t*>(p)[i];
  return dt == DT_BF16 ? Half16<DT_BF16>::to_f(b) : Half16<DT_F16>::to_f(b);
}
// bytes of one hidden row of the model dtype (fp32 models: 4-byte elements; rows stay multiples of 16 B since H % 8 == 0)
__device__ __forceinline__ size_t row_bytes(const RouteParams& p) { return (size_t)p.H * (p.dtype == DT_F32 ? 4 : 2); }
__device__ __forceinline__ float round_to(float f, int dt) {
  if (dt == DT_BF16) return round_dt<DT_BF16>(f);
  if (dt == DT_F16) return round_dt<DT_F16>(f);
  return f;
}

// (value desc, index asc) arg-max across the warp; every lane returns the winner.
__device__ __forceinline__ void warp_argmax(float& v, int& i) {
#pragma unroll
  for (int d = 16; d; d >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, d);
    const int oi = __shfl_xor_sync(0xffffffffu, i, d);
    if (ov > v || (ov == v && oi < i)) { v = ov; i = oi; }
  }
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int d = 16; d; d >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, d));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int d = 16; d; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  return v;
}

// --------------------------------------------------------------------------------------
// K0: router gate.  logits[e] = <x[t], Wg[e]> with fp32 accumulation, 16-byte vector loads.
// p.logits_model_dtype (Mixtral, mixtral.py:46; Qwen2-MoE / Qwen3-MoE, Qwen2MoeTopKRouter; Llama 4, Llama4Router, which
// ranks those logits directly): nn.Linear in model dtype -> result rounded to the model dtype.
// DeepSeek/Switch: fp32 linear on upcast operands (modeling_deepseek.py:467-471).
// --------------------------------------------------------------------------------------
__device__ __forceinline__ void unpack8(const uint4& v, int dt, float (&f)[8]) {
  const uint16_t* s = reinterpret_cast<const uint16_t*>(&v);
#pragma unroll
  for (int j = 0; j < 8; ++j) f[j] = dt == DT_BF16 ? Half16<DT_BF16>::to_f(s[j]) : Half16<DT_F16>::to_f(s[j]);
}
// one warp: dot product of x[t] (model dtype) with gate row e (gate dtype); result in every lane
__device__ float gate_dot_warp(const RouteParams& p, int t, int e) {
  const int lane = threadIdx.x & 31;
  const uint16_t* x = reinterpret_cast<const uint16_t*>(p.x) + (size_t)t * p.H;
  float acc = 0.f;
  if (p.gate_dtype == DT_F32) {
    const float* w = reinterpret_cast<const float*>(p.gate_w) + (size_t)e * p.H;
#pragma unroll 16
    for (int h = lane * 8; h < p.H; h += 256) {
      const uint4 xv = *reinterpret_cast<const uint4*>(x + h);
      const float4 w0 = *reinterpret_cast<const float4*>(w + h), w1 = *reinterpret_cast<const float4*>(w + h + 4);
      float xf[8];
      unpack8(xv, p.dtype, xf);
      acc = fmaf(xf[0], w0.x, acc); acc = fmaf(xf[1], w0.y, acc); acc = fmaf(xf[2], w0.z, acc); acc = fmaf(xf[3], w0.w, acc);
      acc = fmaf(xf[4], w1.x, acc); acc = fmaf(xf[5], w1.y, acc); acc = fmaf(xf[6], w1.z, acc); acc = fmaf(xf[7], w1.w, acc);
    }
  } else {
    const uint16_t* w = reinterpret_cast<const uint16_t*>(p.gate_w) + (size_t)e * p.H;
#pragma unroll 16
    for (int h = lane * 8; h < p.H; h += 256) {
      const uint4 xv = *reinterpret_cast<const uint4*>(x + h);
      const uint4 wv = *reinterpret_cast<const uint4*>(w + h);
      float xf[8], wf[8];
      unpack8(xv, p.dtype, xf);
      unpack8(wv, p.gate_dtype, wf);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc = fmaf(xf[j], wf[j], acc);
    }
  }
  acc = warp_sum(acc);
  return round_to(acc, p.logits_model_dtype ? p.dtype : DT_F32);
}
// One warp, one token, experts [e0, e0+8): x is loaded once per 8-element chunk and reused for all 8 rows
// (16-byte loads of both operands).  out[i] (i < 8) valid in every lane.  No predicates inside the loop (expert
// indices beyond E are clamped to a valid row and their results ignored) so that all 17 loads of an iteration
// are in flight together -- with per-expert `if`s the compiler serialised them: 64 dependent DRAM round trips.
template <bool WF32>
__device__ __forceinline__ void gate_dot8_impl(const RouteParams& p, int t, int e0, float (&out)[8]) {
  const int lane = threadIdx.x & 31;
  const uint16_t* x = reinterpret_cast<const uint16_t*>(p.x) + (size_t)t * p.H;
  const size_t wsz = WF32 ? 4 : 2;
  const char* wrow[8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
    wrow[i] = reinterpret_cast<const char*>(p.gate_w) + (size_t)min(e0 + i, p.E - 1) * p.H * wsz;
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
#pragma unroll 2
  for (int h = lane * 8; h < p.H; h += 256) {
    float xf[8];
    unpack8(*reinterpret_cast<const uint4*>(x + h), p.dtype, xf);
    float wf[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (WF32) {
        const float4 a = *reinterpret_cast<const float4*>(wrow[i] + (size_t)h * 4);
        const float4 b = *reinterpret_cast<const float4*>(wrow[i] + (size_t)h * 4 + 16);
        wf[i][0] = a.x; wf[i][1] = a.y; wf[i][2] = a.z; wf[i][3] = a.w;
        wf[i][4] = b.x; wf[i][5] = b.y; wf[i][6] = b.z; wf[i][7] = b.w;
      } else {
        unpack8(*reinterpret_cast<const uint4*>(wrow[i] + (size_t)h * 2), p.gate_dtype, wf[i]);
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[i] = fmaf(xf[j], wf[i][j], acc[i]);
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float v = warp_sum(acc[i]);
    out[i] = round_to(v, p.logits_model_dtype ? p.dtype : DT_F32);
  }
}
__device__ __forceinline__ void gate_dot8_warp(const RouteParams& p, int t, int e0, float (&out)[8]) {
  if (p.gate_dtype == DT_F32) gate_dot8_impl<true>(p, t, e0, out);
  else gate_dot8_impl<false>(p, t, e0, out);
}

// Large-T gate (prefill): a small fp32 GEMM logits[T,E] = x[T,H] . Wg[E,H]^T on the CUDA cores (fp32 FMA: the expert
// indices derived from it must match the reference's fp32 linear, so no reduced-precision tensor-core inputs).
// A CTA owns 32 tokens (8 warps x GATE_TW) and walks (8-expert group, 256-element slice of H) chunks of the gate matrix:
// each chunk (8 KB fp32 / 4 KB 16-bit) is staged ONCE per CTA in shared memory by cp.async (3-deep ring, one
// __syncthreads per chunk) and used by all 8 warps for GATE_TW x 8 x 8 FMAs per lane.  Reading the gate rows per token
// straight from L2 instead moves 2 GB of L2 traffic per DeepSeek-V2-Lite layer at T=4096, and a register-only variant
// with 4-8 tokens per warp stays L2-bound.  Expert groups are split over blockIdx.y
// when the token blocks alone would not fill the GPU.
constexpr int GATE_TW = 4;
constexpr int GATE_TOK_PER_CTA = 8 * GATE_TW;
constexpr int GATE_RING = 3;
__device__ __forceinline__ void cp_async_16(void* smem_dst, const void* gsrc, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

template <int WDT, int XDT>
__device__ __forceinline__ void gate_logits_impl(const RouteParams& p, uint4* ring /*[GATE_RING][WF32 ? 512 : 256]*/) {
  constexpr bool WF32 = WDT == DT_F32;
  constexpr int PIECES = WF32 ? 512 : 256;                 // 16-byte pieces per chunk
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int ngroups = (p.E + 7) / 8;
  const int nh = (p.H + 255) / 256;
  const int t0 = blockIdx.x * GATE_TOK_PER_CTA + warp * GATE_TW;
  // this CTA's expert groups: blockIdx.y, blockIdx.y + gridDim.y, ...
  const int npass = (ngroups - (int)blockIdx.y + (int)gridDim.y - 1) / (int)gridDim.y;
  const int nchunks = npass * nh;
  const uint16_t* xrow[GATE_TW];
#pragma unroll
  for (int q = 0; q < GATE_TW; ++q)
    xrow[q] = reinterpret_cast<const uint16_t*>(p.x) + (size_t)min(t0 + q, p.T - 1) * p.H;   // clamped: no predicates on addresses
  const bool hvalid_all = (p.H % 256) == 0;

  auto issue = [&](int c) {   // stage chunk c = (pass c / nh, slice c % nh) into ring slot c % GATE_RING
    if (c < nchunks) {
      const int e0 = ((int)blockIdx.y + (c / nh) * (int)gridDim.y) * 8;
      const int h0 = (c % nh) * 256;
      uint4* dst = ring + (size_t)(c % GATE_RING) * PIECES;
      for (int pc = threadIdx.x; pc < PIECES; pc += 256) {
        int i, l, half = 0;
        if (WF32) { i = pc >> 6; l = (pc & 63) >> 1; half = pc & 1; } else { i = pc >> 5; l = pc & 31; }
        const int h = h0 + l * 8;
        const bool ok = h < p.H;
        const char* src = reinterpret_cast<const char*>(p.gate_w) +
                          ((size_t)min(e0 + i, p.E - 1) * p.H + (ok ? h : 0)) * (WF32 ? 4 : 2) + half * 16;
        // fp32: [i][half][lane] so that the 32 lanes of a warp read 512 contiguous bytes (no bank conflicts)
        cp_async_16(dst + (WF32 ? ((i * 2 + half) * 32 + l) : (i * 32 + l)), src, ok ? 16 : 0);
      }
    }
    cp_async_commit();
  };

  issue(0);
  issue(1);
  float acc[GATE_TW][8];
  uint4 xnext[GATE_TW];
#pragma unroll
  for (int q = 0; q < GATE_TW; ++q)
    xnext[q] = (lane * 8 < p.H) ? *reinterpret_cast<const uint4*>(xrow[q] + lane * 8) : make_uint4(0u, 0u, 0u, 0u);
  for (int c = 0; c < nchunks; ++c) {
    const int hc = c % nh;
    if (hc == 0) {
#pragma unroll
      for (int q = 0; q < GATE_TW; ++q)
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[q][i] = 0.f;
    }
    // token slices are requested one chunk ahead (their L2 latency hides under this chunk's FMAs)
    uint4 xv[GATE_TW];
#pragma unroll
    for (int q = 0; q < GATE_TW; ++q) xv[q] = xnext[q];
    {
      const int hn = ((c + 1) % nh) * 256 + lane * 8;
      if (c + 1 < nchunks) {
#pragma unroll
        for (int q = 0; q < GATE_TW; ++q)
          xnext[q] = (hvalid_all || hn < p.H) ? *reinterpret_cast<const uint4*>(xrow[q] + hn) : make_uint4(0u, 0u, 0u, 0u);
      }
    }
    cp_async_wait<1>();        // chunk c has landed (chunk c+1 may still be in flight)
    __syncthreads();           // ... for every thread's pieces; and every warp is done with chunk c-1
    issue(c + 2);              // refills the slot chunk c-1 used
    float xf[GATE_TW][8];
#pragma unroll
    for (int q = 0; q < GATE_TW; ++q) unpack8(xv[q], XDT, xf[q]);      // compile-time dtype: one shift per element
    const uint4* w = ring + (size_t)(c % GATE_RING) * PIECES;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float wf[8];
      if (WF32) {
        const uint4 a = w[(i * 2) * 32 + lane], b = w[(i * 2 + 1) * 32 + lane];
        wf[0] = __uint_as_float(a.x); wf[1] = __uint_as_float(a.y); wf[2] = __uint_as_float(a.z); wf[3] = __uint_as_float(a.w);
        wf[4] = __uint_as_float(b.x); wf[5] = __uint_as_float(b.y); wf[6] = __uint_as_float(b.z); wf[7] = __uint_as_float(b.w);
      } else {
        unpack8(w[i * 32 + lane], WDT, wf);
      }
#pragma unroll
      for (int q = 0; q < GATE_TW; ++q)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[q][i] = fmaf(xf[q][j], wf[j], acc[q][i]);
    }
    if (hc == nh - 1) {
      const int e0 = ((int)blockIdx.y + (c / nh) * (int)gridDim.y) * 8;
#pragma unroll
      for (int q = 0; q < GATE_TW; ++q) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float v = warp_sum(acc[q][i]);
          const int t = t0 + q;
          if (lane == 0 && t < p.T && e0 + i < p.E) {
            if (p.logits_model_dtype)
              reinterpret_cast<uint16_t*>(p.logits_out)[(size_t)t * p.E + e0 + i] =
                  p.dtype == DT_BF16 ? Half16<DT_BF16>::from_f(v) : Half16<DT_F16>::from_f(v);
            else
              reinterpret_cast<float*>(p.logits_out)[(size_t)t * p.E + e0 + i] = v;
          }
        }
      }
    }
  }
  cp_async_wait<0>();
}
__global__ void __launch_bounds__(256, 2) gate_logits_kernel(const RouteParams p) {
  __shared__ __align__(16) uint4 ring[GATE_RING * 512];
  if (p.dtype == DT_BF16) {
    if (p.gate_dtype == DT_F32) gate_logits_impl<DT_F32, DT_BF16>(p, ring);
    else if (p.gate_dtype == DT_BF16) gate_logits_impl<DT_BF16, DT_BF16>(p, ring);
    else gate_logits_impl<DT_F16, DT_BF16>(p, ring);
  } else {
    if (p.gate_dtype == DT_F32) gate_logits_impl<DT_F32, DT_F16>(p, ring);
    else if (p.gate_dtype == DT_BF16) gate_logits_impl<DT_BF16, DT_F16>(p, ring);
    else gate_logits_impl<DT_F16, DT_F16>(p, ring);
  }
}

// --------------------------------------------------------------------------------------
// DeepSeek-V3 noaux_tc selection (modeling_deepseek_v3/modeling_deepseek.py:483-513) for one token, one warp, lane owns
// experts lane + 32*i.  s = unbiased sigmoid scores, bias = the layer's e_score_correction_bias [E].
//   choice = s + bias; group score = top1 + top2 of the group's choices; the topk_group best groups are kept; choices
//   outside them become 0.0 (masked_fill, not -inf); k rounds of arg-max over the choices.  Ties -> lowest index.
// Leaves winner j (selection order) in s_scr[MAX_K + j] (int bits) and its UNBIASED score in s_scr[j].
// Used by the routing kernels and by the look-ahead predictor.
// --------------------------------------------------------------------------------------
__device__ __forceinline__ void v3_select_warp(const RouteParams& p, const float (&s)[MAX_PL], const float* __restrict__ bias,
                                               float* s_scr /*[E] smem scratch*/) {
  const int lane = threadIdx.x & 31;
  const int E = p.E;
  const int gsz = E / p.n_group;
  float c[MAX_PL];
#pragma unroll
  for (int i = 0; i < MAX_PL; ++i) {
    const int e = lane + 32 * i;
    c[i] = e < E ? __fadd_rn(s[i], bias[e]) : -INFINITY;
    if (e < E) s_scr[e] = c[i];
  }
  __syncwarp();
  // group score: sum of the two largest choices of the group (topk(2).sum(); duplicates count twice)
  float gsc = -INFINITY;
  if (lane < p.n_group) {
    float t1 = -INFINITY, t2 = -INFINITY;
    for (int j = 0; j < gsz; ++j) {
      const float cv = s_scr[lane * gsz + j];
      if (cv > t1) { t2 = t1; t1 = cv; } else if (cv > t2) { t2 = cv; }
    }
    gsc = __fadd_rn(t1, t2);
  }
  uint32_t allowed = 0;
  for (int r = 0; r < p.topk_group; ++r) {
    float bv = lane < p.n_group ? gsc : -INFINITY;
    int bi = lane < p.n_group ? lane : 0x7fffffff;
    warp_argmax(bv, bi);
    allowed |= 1u << bi;
    if (lane == bi) gsc = -INFINITY;
  }
#pragma unroll
  for (int i = 0; i < MAX_PL; ++i) {
    const int e = lane + 32 * i;
    if (e < E && !((allowed >> (e / gsz)) & 1u)) c[i] = 0.0f;   // masked_fill(~score_mask, 0.0)
  }
  __syncwarp();   // s_scr is reused for the winners below
  uint32_t taken = 0;
#pragma unroll 1
  for (int j = 0; j < p.k; ++j) {
    float bv = -INFINITY, sw = 0.f;   // sw: the candidate's unbiased score travels with it (gather(scores, topk_idx))
    int bi = 0x7fffffff;
#pragma unroll
    for (int i = 0; i < MAX_PL; ++i) {
      const int e = lane + 32 * i;
      if (e < E && !((taken >> i) & 1u) && (c[i] > bv || bi == 0x7fffffff)) { bv = c[i]; bi = e; sw = s[i]; }
    }
#pragma unroll
    for (int d = 16; d; d >>= 1) {   // warp_argmax carrying sw
      const float ov = __shfl_xor_sync(0xffffffffu, bv, d);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, d);
      const float os = __shfl_xor_sync(0xffffffffu, sw, d);
      if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; sw = os; }
    }
    if ((bi & 31) == lane) taken |= 1u << (bi >> 5);
    if (lane == 0) {
      s_scr[j] = sw;
      s_scr[MAX_K + j] = __int_as_float(bi);
    }
  }
  __syncwarp();
}

// sigmoid exactly as PyTorch's CUDA kernel computes it in fp32: 1 / (1 + exp(-x)), IEEE division
__device__ __forceinline__ float sigmoid_ref(float x) { return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x))); }

// DeepSeek-V3 gate for one token: sigmoid (unless scores come in), selection, weights (modeling_deepseek.py:475-526)
// (inlined: a call would copy the kernel's RouteParams to a 1.2 KB stack frame to pass it by reference)
__device__ __forceinline__ void route_token_v3(const RouteParams& p, int t, const float* s_in, bool in_are_scores,
                                               float* s_scr, int* out_idx, float* out_w) {
  const int lane = threadIdx.x & 31;
  const int E = p.E;
  float s[MAX_PL];
#pragma unroll
  for (int i = 0; i < MAX_PL; ++i) {
    const int e = lane + 32 * i;
    s[i] = e < E ? (in_are_scores ? s_in[e] : sigmoid_ref(s_in[e])) : 0.f;
    if (p.scores && e < E) p.scores[(size_t)t * E + e] = s[i];
  }
  v3_select_warp(p, s, p.gate_bias, s_scr);
  // weights: unbiased scores, normalised by their sum in selection order (k > 1 and norm_topk_prob), then ALWAYS scaled
  float denom = 0.f;
  for (int j = 0; j < p.k; ++j) denom = __fadd_rn(denom, s_scr[j]);
  if (lane < p.k) {
    float w = s_scr[lane];
    if (p.k > 1 && p.norm_topk_prob) w = __fdiv_rn(w, __fadd_rn(denom, 1e-20f));
    out_idx[lane] = __float_as_int(s_scr[MAX_K + lane]);
    out_w[lane] = __fmul_rn(w, p.routed_scaling_factor);
  }
  __syncwarp();
}

// Llama 4 pieces of K1, kept out of line so that the other routers' code around them is not rearranged (the routing
// kernels are instruction-cache cold every launch): the fp32 sigmoid of every logit (B2M_WS_SCORES, one warp, logits in
// shared memory) and the weight of a chosen logit, round(sigmoid(l)) in the model dtype (Llama4Router).
__device__ __noinline__ void llama4_scores(const float* s_in, float* scores_row, int E) {
  for (int e = threadIdx.x & 31; e < E; e += 32) scores_row[e] = sigmoid_ref(s_in[e]);
}
__device__ __noinline__ float llama4_weight(float logit, int dtype) { return round_to(sigmoid_ref(logit), dtype); }

// --------------------------------------------------------------------------------------
// K1: softmax + top-k (+renorm) for one token (one warp, lane owns experts lane, lane+32, ...)
// --------------------------------------------------------------------------------------
__device__ void route_token_warp(const RouteParams& p, int t, const float* s_in /*[E] logits or scores (smem)*/,
                                 bool in_are_scores, float* s_scr /*[E] smem scratch*/, int* out_idx, float* out_w) {
  if (p.router == ROUTER_DEEPSEEK_V3) {
    route_token_v3(p, t, s_in, in_are_scores, s_scr, out_idx, out_w);
    return;
  }
  const int lane = threadIdx.x & 31;
  const int E = p.E;
  float v[MAX_PL];
  // --- softmax in fp32: exp(x - max) / sum  (F.softmax(dtype=float), mixtral.py:48; modeling_deepseek.py:473)
  float m = -INFINITY;
#pragma unroll
  for (int i = 0; i < MAX_PL; ++i) {
    const int e = lane + 32 * i;
    v[i] = e < E ? s_in[e] : -INFINITY;
    m = fmaxf(m, v[i]);
  }
  // Llama 4 selects on the logits themselves (Llama4Router: torch.topk(router_logits)), so there is no softmax
  if (!in_are_scores && p.router != ROUTER_LLAMA4) {
    m = warp_max(m);
    float z = 0.f;
#pragma unroll
    for (int i = 0; i < MAX_PL; ++i) {
      const int e = lane + 32 * i;
      v[i] = e < E ? expf(v[i] - m) : 0.f;
      z += v[i];
    }
    z = warp_sum(z);
#pragma unroll
    for (int i = 0; i < MAX_PL; ++i) v[i] = __fdiv_rn(v[i], z);
  }
  if (p.scores && p.router == ROUTER_LLAMA4) {
    llama4_scores(s_in, p.scores + (size_t)t * E, E);
  } else if (p.scores) {
#pragma unroll
    for (int i = 0; i < MAX_PL; ++i) {
      const int e = lane + 32 * i;
      if (e < E) p.scores[(size_t)t * E + e] = v[i];
    }
  }
  if (p.router == ROUTER_SWITCH_TOP1) {
    // router_probs are cast to the input dtype before argmax/max (HF 4.x Top1Router._compute_router_probabilities)
#pragma unroll
    for (int i = 0; i < MAX_PL; ++i) v[i] = round_to(v[i], p.dtype);
  }
  if (p.router == ROUTER_DEEPSEEK_GROUP) {
    // modeling_deepseek.py:484-505: keep the topk_group groups with the largest max score, zero the rest
    const int gsz = E / p.n_group;
#pragma unroll
    for (int i = 0; i < MAX_PL; ++i) {
      const int e = lane + 32 * i;
      if (e < E) s_scr[e] = v[i];
    }
    __syncwarp();
    float gmax = -INFINITY;
    if (lane < p.n_group)
      for (int j = 0; j < gsz; ++j) gmax = fmaxf(gmax, s_scr[lane * gsz + j]);
    uint32_t allowed = 0;
    for (int r = 0; r < p.topk_group; ++r) {
      float bv = gmax;
      int bi = lane < p.n_group ? lane : 0x7fffffff;
      if (lane >= p.n_group) bv = -INFINITY;
      warp_argmax(bv, bi);
      allowed |= 1u << bi;
      if (lane == bi) gmax = -INFINITY;
    }
#pragma unroll
    for (int i = 0; i < MAX_PL; ++i) {
      const int e = lane + 32 * i;
      if (e < E && !((allowed >> (e / gsz)) & 1u)) v[i] = 0.0f;   // masked_fill(~score_mask, 0.0)
    }
    __syncwarp();
  }
  // --- top-k, ties -> lowest expert index.  The k selection rounds are a real loop (winners parked in shared
  // scratch) rather than 8x8 unrolled code: the kernel is launch/latency bound and instruction-cache cold every launch.
  uint32_t taken = 0;
  float denom = 0.f;
  __syncwarp();
#pragma unroll 1
  for (int j = 0; j < p.k; ++j) {
    float bv = -INFINITY;
    int bi = 0x7fffffff;
#pragma unroll
    for (int i = 0; i < MAX_PL; ++i) {
      const int e = lane + 32 * i;
      if (e < E && !((taken >> i) & 1u) && (v[i] > bv || bi == 0x7fffffff)) { bv = v[i]; bi = e; }
    }
    warp_argmax(bv, bi);
    if ((bi & 31) == lane) taken |= 1u << (bi >> 5);
    denom = __fadd_rn(denom, bv);
    if (lane == 0) {
      s_scr[j] = bv;
      s_scr[MAX_K + j] = __int_as_float(bi);
    }
  }
  __syncwarp();
  // --- weights
  if (lane < p.k) {
    const float sv = s_scr[lane];
    float w;
    if (p.router == ROUTER_MIXTRAL) {
      w = round_to(__fdiv_rn(sv, denom), p.dtype);                       // mixtral.py:52-54
    } else if (p.router == ROUTER_SWITCH_TOP1) {
      w = sv;
    } else if (p.router == ROUTER_QWEN_MOE) {
      // Qwen2MoeTopKRouter: fp32 weights, divided by their sum (selection order) for every k, no epsilon, no scaling
      w = p.norm_topk_prob ? __fdiv_rn(sv, denom) : sv;
    } else if (p.router == ROUTER_LLAMA4) {
      // Llama4Router: sigmoid(router_scores.float()).to(model dtype) of the chosen logit; it scales the expert's input rows
      w = llama4_weight(sv, p.dtype);
    } else if (p.k > 1 && p.norm_topk_prob) {
      w = __fdiv_rn(sv, __fadd_rn(denom, 1e-20f));                        // modeling_deepseek.py:508-510
    } else {
      w = __fmul_rn(sv, p.routed_scaling_factor);                        // :512
    }
    out_idx[lane] = __float_as_int(s_scr[MAX_K + lane]);
    out_w[lane] = w;
  }
  __syncwarp();
}

// lane == token: does this lane's token route to expert e ?
__device__ __forceinline__ bool lane_has(const int (&idx)[MAX_K], int k, int e) {
  bool h = false;
#pragma unroll
  for (int j = 0; j < MAX_K; ++j) h |= (j < k && idx[j] == e);
  return h;
}

// Per-chunk per-expert counts (lane == token).  counts_out[e] for e in [0,E)
__device__ void chunk_count_warp(const int* topk_idx, int t0, int T, int k, int E, int* counts_out) {
  const int lane = threadIdx.x & 31;
  const int t = t0 + lane;
  int idx[MAX_K];
#pragma unroll
  for (int j = 0; j < MAX_K; ++j) idx[j] = (t < T && j < k) ? topk_idx[(size_t)t * k + j] : -1;
  for (int e0 = 0; e0 < E; e0 += 32) {
    int mine = 0;
    for (int ee = 0; ee < 32 && e0 + ee < E; ++ee) {
      const uint32_t b = __ballot_sync(0xffffffffu, lane_has(idx, k, e0 + ee));
      if (lane == ee) mine = __popc(b);
    }
    if (e0 + lane < E) counts_out[e0 + lane] = mine;
  }
}

// Destination rows for the tokens of one chunk (lane == token), stable inside each expert.
// base_of(e) = first permuted row available to this chunk for expert e.
template <class BaseFn>
__device__ void chunk_rank_warp(const RouteParams& p, int t0, BaseFn base_of, int* s_rows /*[CHUNK*k] smem*/,
                                const int* idx_src = nullptr, bool write_global = true) {
  const int lane = threadIdx.x & 31;
  const int t = t0 + lane;
  const int k = p.k;
  if (!idx_src) idx_src = p.topk_idx;
  int idx[MAX_K];
#pragma unroll
  for (int j = 0; j < MAX_K; ++j) idx[j] = (t < p.T && j < k) ? idx_src[(size_t)t * k + j] : -1;
  int dest[MAX_K];
#pragma unroll
  for (int j = 0; j < MAX_K; ++j) dest[j] = -1;
  for (int e = 0; e < p.E; ++e) {
    const bool h = lane_has(idx, k, e);
    const uint32_t b = __ballot_sync(0xffffffffu, h);
    if (b == 0) continue;
    if (h) {
      const int row = base_of(e) + __popc(b & ((1u << lane) - 1u));
#pragma unroll
      for (int j = 0; j < MAX_K; ++j)
        if (j < k && idx[j] == e) dest[j] = row;
    }
  }
#pragma unroll
  for (int j = 0; j < MAX_K; ++j) {
    if (j < k) {
      if (s_rows) s_rows[lane * k + j] = dest[j];
      if (t < p.T && write_global) {
        p.row_of[(size_t)t * k + j] = dest[j];
        if (dest[j] >= 0) p.perm_token[dest[j]] = t;
      }
    }
  }
}

// Expert-strided variants for the last gate/top-k CTA: the (chunk, expert subset) tasks are spread over all warps of
// the CTA instead of one warp walking all E experts of a chunk (64 dependent ballots for DeepSeek).
__device__ __forceinline__ void chunk_count_strided(const int* idx_src, int t0, int T, int k, int E, int* counts_out,
                                                    int e_begin, int e_step) {
  const int lane = threadIdx.x & 31;
  const int t = t0 + lane;
  int idx[MAX_K];
#pragma unroll
  for (int j = 0; j < MAX_K; ++j) idx[j] = (t < T && j < k) ? idx_src[(size_t)t * k + j] : -1;
  for (int e = e_begin; e < E; e += e_step) {
    const uint32_t b = __ballot_sync(0xffffffffu, lane_has(idx, k, e));
    if (lane == 0) counts_out[e] = __popc(b);
  }
}
template <class BaseFn>
__device__ __forceinline__ void chunk_rank_strided(const RouteParams& p, int t0, BaseFn base_of, const int* idx_src,
                                                   int e_begin, int e_step) {
  const int lane = threadIdx.x & 31;
  const int t = t0 + lane;
  const int k = p.k;
  int idx[MAX_K];
#pragma unroll
  for (int j = 0; j < MAX_K; ++j) idx[j] = (t < p.T && j < k) ? idx_src[(size_t)t * k + j] : -1;
  for (int e = e_begin; e < p.E; e += e_step) {
    const bool h = lane_has(idx, k, e);
    const uint32_t b = __ballot_sync(0xffffffffu, h);
    if (h) {
      const int row = base_of(e) + __popc(b & ((1u << lane) - 1u));
#pragma unroll
      for (int j = 0; j < MAX_K; ++j)
        if (j < k && idx[j] == e) p.row_of[(size_t)t * k + j] = row;
      p.perm_token[row] = t;
    }
  }
}

// Gather of one 16-bit row through an input permutation (b2m_set_input_perm): dst[c] = src[perm[c]], 8 table entries per
// 16-byte load, 8 independent 2-byte loads of the source row (L1-resident after the first touch), one 16-byte store; threads
// tid, tid + nthr, ... of the caller share the row.  An entry >= H reads as 0 and sets bit 1 of the sticky error word
// (b2m_check_errors); nothing outside src is read.  Not inlined: the routing kernels are instruction-cache cold every
// launch, and layers without a table should not fetch this code (scalar arguments: no RouteParams copy for the call).
__device__ __noinline__ void gather_row_perm(const uint16_t* __restrict__ src, const uint16_t* __restrict__ perm,
                                             uint4* __restrict__ dst, int H, int tid, int nthr, int* err_flag) {
  bool bad = false;
  for (int v = tid; v < H / 8; v += nthr) {
    const uint4 iv = reinterpret_cast<const uint4*>(perm)[v];
    const uint16_t* ix = reinterpret_cast<const uint16_t*>(&iv);
    uint4 o;
    uint16_t* os = reinterpret_cast<uint16_t*>(&o);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const bool ok = ix[j] < H;
      bad |= !ok;
      os[j] = ok ? src[ix[j]] : (uint16_t)0;
    }
    dst[v] = o;
  }
  if (bad && err_flag) atomicOr(err_flag, 2);
}

// Llama 4 gather of one 16-bit row scaled by its routing weight: dst[c] = round(x[c] * w) (the product of two 16-bit
// values is exact in fp32, so one __fmul_rn and one rounding to the model dtype), 16-byte loads and stores; threads tid,
// tid + nthr, ... of the caller share the row.  Not inlined, for the same reason as gather_row_perm.
__device__ __noinline__ void scale_row(const uint4* __restrict__ src, uint4* __restrict__ dst, int nvec, float w, int dtype,
                                       int tid, int nthr) {
  for (int v = tid; v < nvec; v += nthr) {
    float f[8];
    unpack8(src[v], dtype, f);
    uint4 o;
    uint16_t* os = reinterpret_cast<uint16_t*>(&o);
#pragma unroll
    for (int j = 0; j < 8; ++j)
      os[j] = dtype == DT_BF16 ? Half16<DT_BF16>::from_f(__fmul_rn(f[j], w)) : Half16<DT_F16>::from_f(__fmul_rn(f[j], w));
    dst[v] = o;
  }
}

// Copy one activation row x[t] -> dst with 16-byte vectors, NTHR threads (a warp or the whole CTA; `tid` = this thread's
// index among them).  e = the expert of the row: a layer with an input permutation gathers column c from x[t][perm[e][c]]
// instead (gather_row_perm; 16-bit models only).  pair = the row's (token, choice) index t * k + j: a Llama 4 routing call
// (p.scale_rows) scales the row by topk_w[pair] (scale_row).
template <int NTHR>
__device__ __forceinline__ void copy_row(const RouteParams& p, int t, int e, int pair, void* dst_row, int tid) {
  const size_t rb = row_bytes(p);
  const int vec_per_row = (int)(rb / 16);   // uint4 = 8 x 16-bit (4 x fp32)
  const uint4* src = reinterpret_cast<const uint4*>(reinterpret_cast<const uint8_t*>(p.x) + (size_t)t * rb);
  uint4* dst = reinterpret_cast<uint4*>(dst_row);
  if (p.input_perm) {
    gather_row_perm(reinterpret_cast<const uint16_t*>(src), p.input_perm + (size_t)e * p.H, dst, p.H, tid, NTHR, p.err_flag);
    return;
  }
  if (p.scale_rows) {
    scale_row(src, dst, vec_per_row, p.topk_w[pair], p.dtype, tid, NTHR);
    return;
  }
  int v = tid;
  if (NTHR == 32) {
    for (; v + 96 < vec_per_row; v += 128) {   // 4 independent 16 B loads in flight per lane
      const uint4 a = src[v], b = src[v + 32], c = src[v + 64], d = src[v + 96];
      dst[v] = a; dst[v + 32] = b; dst[v + 64] = c; dst[v + 96] = d;
    }
  }
  for (; v < vec_per_row; v += NTHR) dst[v] = src[v];
}

// Copy gathered rows x[t] -> xp[row], one warp per row; `npairs` (token,slot) pairs starting at token t0.
__device__ void copy_rows_block(const RouteParams& p, int t0, int npairs, const int* s_rows, int warp0, int nwarps) {
  const int lane = threadIdx.x & 31;
  const int warp = (threadIdx.x >> 5) - warp0;
  const size_t rb = row_bytes(p);
  for (int i = warp; i < npairs; i += nwarps) {
    const int row = s_rows[i];
    const int t = t0 + i / p.k;
    if (row < 0 || t >= p.T) continue;
    const int e = p.input_perm ? p.topk_idx[(size_t)t0 * p.k + i] : 0;
    copy_row<32>(p, t, e, t0 * p.k + i, reinterpret_cast<uint8_t*>(p.xp) + (size_t)row * rb, lane);
  }
}

// --------------------------------------------------------------------------------------
// Multi-CTA path (large T): route -> scan -> permute
// --------------------------------------------------------------------------------------
__global__ void __launch_bounds__(RT_THREADS) route_topk_kernel(const RouteParams p) {
  __shared__ float s_logits[RT_WARPS][MAX_PL * 32];
  __shared__ float s_scr[RT_WARPS][MAX_PL * 32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tb = blockIdx.x * CHUNK;   // one 32-token ranking chunk per block: T/32 blocks keep every SM busy
  for (int i = warp; i < CHUNK; i += RT_WARPS) {
    const int t = tb + i;
    if (t >= p.T) break;
    // large-T path: logits/scores always come from memory (caller-supplied, or written by gate_logits_kernel)
    for (int e = lane; e < p.E; e += 32) s_logits[warp][e] = load_as_float(p.logits, (size_t)t * p.E + e, p.logits_dtype);
    const bool scores_in = p.logits_are_scores != 0;
    __syncwarp();
    if (p.logits_out && !scores_in) {
      for (int e = lane; e < p.E; e += 32) {
        const float lv = s_logits[warp][e];
        if (p.logits_model_dtype) {
          reinterpret_cast<uint16_t*>(p.logits_out)[(size_t)t * p.E + e] =
              p.dtype == DT_BF16 ? Half16<DT_BF16>::from_f(lv) : Half16<DT_F16>::from_f(lv);
        } else {
          reinterpret_cast<float*>(p.logits_out)[(size_t)t * p.E + e] = lv;
        }
      }
    }
    route_token_warp(p, t, s_logits[warp], scores_in, s_scr[warp], p.topk_idx + (size_t)t * p.k,
                     p.topk_w + (size_t)t * p.k);
    __syncwarp();
  }
  if (p.router == ROUTER_SWITCH_TOP1) return;   // capacity pass + counts run in a separate kernel
  __threadfence_block();
  __syncthreads();
  // per-chunk counts
  if (warp == 0 && tb < p.T) chunk_count_warp(p.topk_idx, tb, p.T, p.k, p.E, p.chunk_counts + (size_t)blockIdx.x * p.E);
}

// Switch capacity (cumsum priority <= capacity, per batch row), then per-chunk counts.  One block per batch row.
__global__ void __launch_bounds__(RT_THREADS) switch_capacity_kernel(const RouteParams p) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.x;
  const int S = p.seq_len;
  // warp w handles experts w, w+8, ...; walks the row in token order
  for (int e = warp; e < p.E; e += RT_WARPS) {
    int running = 0;
    for (int s0 = 0; s0 < S; s0 += 32) {
      const int s = s0 + lane;
      const int t = b * S + s;
      const int raw = s < S ? p.topk_idx[t] : -1;
      const bool h = s < S && (raw >= 0 ? raw : -(raw + 2)) == e;
      const uint32_t m = __ballot_sync(0xffffffffu, h);
      if (h) {
        const int prio = running + __popc(m & ((1u << lane) - 1u)) + 1;   // cumsum is 1-based
        if (prio > p.expert_capacity) p.topk_idx[t] = -(e + 2);           // dropped: passes through unchanged
      }
      running += __popc(m);
    }
  }
}
__global__ void __launch_bounds__(RT_THREADS) chunk_count_kernel(const RouteParams p) {
  const int warp = threadIdx.x >> 5;
  const int chunk = blockIdx.x * RT_WARPS + warp;
  const int t0 = chunk * CHUNK;
  if (t0 < p.T) chunk_count_warp(p.topk_idx, t0, p.T, p.k, p.E, p.chunk_counts + (size_t)chunk * p.E);
}

// dense mask -> per-token expert list (ascending expert id, -1 padded), weights = 1
__global__ void __launch_bounds__(RT_THREADS) mask_to_topk_kernel(const RouteParams p, const uint8_t* __restrict__ mask) {
  const int t = blockIdx.x * RT_THREADS + threadIdx.x;
  if (t >= p.T) return;
  int n = 0, nset = 0;
  for (int e = 0; e < p.E; ++e) {
    if (!mask[(size_t)t * p.E + e]) continue;
    ++nset;
    if (n < p.k) {
      p.topk_idx[(size_t)t * p.k + n] = e;
      p.topk_w[(size_t)t * p.k + n] = 1.0f;
      ++n;
    }
  }
  // more experts per token than the context's top_k: rows would be dropped silently -> raise the sticky error flag
  // (reported as B2M_EINVAL by the next call that synchronises: b2m_expert_outputs / b2m_check_errors)
  if (nset > p.k && p.err_flag) atomicOr(p.err_flag, 1);
  for (; n < p.k; ++n) {
    p.topk_idx[(size_t)t * p.k + n] = -1;
    p.topk_w[(size_t)t * p.k + n] = 0.0f;
  }
}

// exclusive scan: chunk_counts[c][e] -> first row of (chunk c, expert e) relative to the expert start;
// counts[e], offsets[e].  Single block, thread == expert.
__global__ void __launch_bounds__(256) route_scan_kernel(const RouteParams p, int nchunks) {
  __shared__ int s_tot[MAX_PL * 32];
  const int e = threadIdx.x;
  if (e < p.E) {
    int run = 0;
    int c = 0;
    for (; c + 8 <= nchunks; c += 8) {
      int v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) v[u] = p.chunk_counts[(size_t)(c + u) * p.E + e];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        p.chunk_counts[(size_t)(c + u) * p.E + e] = run;
        run += v[u];
      }
    }
    for (; c < nchunks; ++c) {
      const int v = p.chunk_counts[(size_t)c * p.E + e];
      p.chunk_counts[(size_t)c * p.E + e] = run;
      run += v;
    }
    s_tot[e] = run;
    p.counts[e] = run;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int i = 0; i < p.E; ++i) {
      p.offsets[i] = acc;
      acc += s_tot[i];
    }
    p.offsets[p.E] = acc;
  }
}

// one block per chunk of 32 tokens: warp 0 ranks the chunk, then all warps copy its rows
__global__ void __launch_bounds__(RT_THREADS) route_permute_kernel(const RouteParams p) {
  __shared__ int s_rows[CHUNK * MAX_K];
  const int warp = threadIdx.x >> 5;
  const int chunk = blockIdx.x;
  const int t0 = chunk * CHUNK;
  if (warp == 0 && t0 < p.T) {
    const int* cb = p.chunk_counts + (size_t)chunk * p.E;
    chunk_rank_warp(p, t0, [&](int e) { return p.offsets[e] + cb[e]; }, s_rows);
  }
  __syncthreads();
  if (t0 < p.T) copy_rows_block(p, t0, CHUNK * p.k, s_rows, 0, RT_WARPS);
  // clear the split-K accumulator (grid-stride over the whole grid)
  if (p.y_zero) {
    float4* z = reinterpret_cast<float4*>(p.y_zero);
    const size_t n4 = p.y_zero_elems / 4;
    for (size_t i = (size_t)blockIdx.x * RT_THREADS + threadIdx.x; i < n4; i += (size_t)gridDim.x * RT_THREADS)
      z[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// --------------------------------------------------------------------------------------
// Small-T path (decode, T <= 256): two launches, both multi-CTA.
//   gate_topk_small_kernel : one CTA per token -- the E gate dot products are spread over the CTA's warps,
//                            warp 0 then does softmax + top-k (+renorm).
//   permute_small_kernel   : every CTA redundantly ranks the (tiny) routing table in shared memory, CTA 0
//                            publishes counts/offsets/row maps, and the gathered rows are copied one row per CTA
//                            with 16-byte vectors.
// --------------------------------------------------------------------------------------
__global__ void __launch_bounds__(RT_THREADS) gate_topk_small_kernel(const RouteParams p) {
  __shared__ float s_logits[MAX_PL * 32];
  __shared__ float s_scr[MAX_PL * 32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t = blockIdx.x;
  pdl_launch();
  pdl_wait();
  if (p.tl && threadIdx.x == 0) tl_min(p.tl);
  bool scores_in = false;
  if (p.logits) {
    for (int e = threadIdx.x; e < p.E; e += RT_THREADS) s_logits[e] = load_as_float(p.logits, (size_t)t * p.E + e, p.logits_dtype);
    scores_in = p.logits_are_scores != 0;
  } else {
    if (p.E >= 8 * RT_WARPS) {
      // many experts (DeepSeek): every warp takes 8 experts per pass and reads the token row once per pass
      for (int e0 = warp * 8; e0 < p.E; e0 += 8 * RT_WARPS) {
        float v[8];
        gate_dot8_warp(p, t, e0, v);
#pragma unroll
        for (int i = 0; i < 8; ++i)
          if (lane == 0 && e0 + i < p.E) s_logits[e0 + i] = v[i];
      }
    } else {
      for (int e = warp; e < p.E; e += RT_WARPS) {
        const float v = gate_dot_warp(p, t, e);
        if (lane == 0) s_logits[e] = v;
      }
    }
  }
  __syncthreads();
  if (warp == 0) {
    if (p.logits_out && !scores_in) {
      for (int e = lane; e < p.E; e += 32) {
        const float lv = s_logits[e];
        if (p.logits_model_dtype)
          reinterpret_cast<uint16_t*>(p.logits_out)[(size_t)t * p.E + e] =
              p.dtype == DT_BF16 ? Half16<DT_BF16>::from_f(lv) : Half16<DT_F16>::from_f(lv);
        else
          reinterpret_cast<float*>(p.logits_out)[(size_t)t * p.E + e] = lv;
      }
    }
    route_token_warp(p, t, s_logits, scores_in, s_scr, p.topk_idx + (size_t)t * p.k, p.topk_w + (size_t)t * p.k);
    if (p.tl && lane == 0) tl_max(p.tl + 1);
  }
  if (p.ep_fused) {
    // ---- expert parallel, direct mode: this kernel is also the permute + dispatch kernel.  Rows need no global ranking
    // (every row is processed independently by the owner and found again through row_of): each (token, choice) claims the
    // next free row of its expert's region at the owner with an atomic on the OWNER's counter (a remote atomic over NVLink
    // for peers) and stores its row there -- the owner sees each expert's rows contiguous, exactly as many as there are.
    __shared__ int s_dst_rank[MAX_K], s_dst_row[MAX_K];
    __syncthreads();
    if (warp == 0 && lane < p.k) {
      const int El = p.E / p.ep.nranks;
      const int e = p.topk_idx[(size_t)t * p.k + lane];
      int r = -1, pos = -1, le = 0;
      if (e >= 0) {
        r = e / El;
        le = e - r * El;
        pos = atomicAdd(p.ep.peer_cnt[r] + le, 1);
      }
      p.row_of[(size_t)t * p.k + lane] = pos;            // row inside the expert's region at the owner (the combine's key)
      s_dst_rank[lane] = r;
      s_dst_row[lane] = le * p.ep.region_rows + pos;
    }
    __syncthreads();
    const int vec_per_row = p.H / 8;
    const uint4* src = reinterpret_cast<const uint4*>(reinterpret_cast<const uint16_t*>(p.x) + (size_t)t * p.H);
    for (int j = 0; j < p.k; ++j) {
      if (s_dst_rank[j] < 0) continue;
      uint4* dst = reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(p.ep.peer_recv[s_dst_rank[j]]) + (size_t)s_dst_row[j] * p.H);
      for (int v = threadIdx.x; v < vec_per_row; v += RT_THREADS) dst[v] = src[v];
    }
    p2p_signal(p.ep, 0);
    if (p.tl && threadIdx.x == 0) tl_max(p.tl + 3);
    return;
  }
  if (!p.offsets_early) return;
  // ---- the last CTA to finish publishes counts[E] / offsets[E+1] for the whole batch: the grouped GEMM only needs these
  // (not the gathered rows) to start streaming weights, so it can overlap the permute kernel
  __shared__ int s_last;
  __shared__ int s_idx2[FUSED_MAX_T * MAX_K];
  __shared__ int s_cnt2[RT_WARPS][MAX_PL * 32];
  __shared__ int s_tot2[MAX_PL * 32];
  __shared__ int s_off2[MAX_PL * 32 + 1];
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    s_last = (atomicAdd(p.ticket, 1) == (int)gridDim.x - 1);
  }
  __syncthreads();
  if (!s_last) return;
  const int npairs = p.T * p.k;
  if (s_last) {
    __threadfence();
    const int nchunks = (p.T + CHUNK - 1) / CHUNK;
    for (int i = threadIdx.x; i < npairs; i += RT_THREADS) s_idx2[i] = __ldcg(p.topk_idx + i);   // other CTAs' results: L2
    __syncthreads();
    for (int task = warp; task < nchunks * RT_WARPS; task += RT_WARPS)   // (chunk, expert subset) tasks over all warps
      chunk_count_strided(s_idx2, (task / RT_WARPS) * CHUNK, p.T, p.k, p.E, s_cnt2[task / RT_WARPS], task % RT_WARPS, RT_WARPS);
    __syncthreads();
    if (threadIdx.x < p.E) {
      int run = 0;
      for (int c = 0; c < nchunks; ++c) { const int v = s_cnt2[c][threadIdx.x]; s_cnt2[c][threadIdx.x] = run; run += v; }   // -> exclusive chunk bases
      s_tot2[threadIdx.x] = run;
      p.counts[threadIdx.x] = run;
    }
    __syncthreads();
    if (warp == 0) {
      int v[MAX_PL], run = 0;
#pragma unroll
      for (int i = 0; i < MAX_PL; ++i) {
        const int e = lane * MAX_PL + i;
        v[i] = e < p.E ? s_tot2[e] : 0;
        run += v[i];
      }
      int incl = run;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int o = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += o;
      }
      int base = incl - run;
#pragma unroll
      for (int i = 0; i < MAX_PL; ++i) {
        const int e = lane * MAX_PL + i;
        if (e < p.E) { p.offsets[e] = base; s_off2[e] = base; }
        base += v[i];
      }
      if (lane == 31) { p.offsets[p.E] = incl; s_off2[p.E] = incl; }
      if (lane == 0) *p.ticket = 0;
    }
    if (p.rows_by_gate) {
      // publish the row maps as well (stable ascending-token order inside each expert): the permute kernel then only copies
      __syncthreads();
      for (int task = warp; task < nchunks * RT_WARPS; task += RT_WARPS) {
        const int* cb = s_cnt2[task / RT_WARPS];
        chunk_rank_strided(p, (task / RT_WARPS) * CHUNK, [&](int e) { return s_off2[e] + cb[e]; }, s_idx2, task % RT_WARPS, RT_WARPS);
      }
    }
  }
}

__global__ void __launch_bounds__(RT_THREADS) permute_small_kernel(const RouteParams p) {
  __shared__ int s_idx[FUSED_MAX_T * MAX_K];
  __shared__ int s_cnt[RT_WARPS][MAX_PL * 32];   // per-chunk counts -> exclusive bases
  __shared__ int s_off[MAX_PL * 32 + 1];
  __shared__ int s_tot[MAX_PL * 32];
  __shared__ int s_rows[FUSED_MAX_T * MAX_K];    // destination row of (t, j), index t*k + j
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nchunks = (p.T + CHUNK - 1) / CHUNK;
  const int npairs = p.T * p.k;
  pdl_launch();
  pdl_wait();
  if (p.tl && threadIdx.x == 0) tl_min(p.tl + 2);
  if (p.rows_by_gate) {
    // the gate/top-k kernel already published counts, offsets and the row maps: this kernel is a pure row copy
    const size_t rb = row_bytes(p);
    for (int i = blockIdx.x; i < npairs; i += gridDim.x) {
      const int row = p.row_of[i];
      if (row < 0) continue;
      const int e = p.input_perm ? p.topk_idx[i] : 0;
      copy_row<RT_THREADS>(p, i / p.k, e, i, reinterpret_cast<uint8_t*>(p.xp) + (size_t)row * rb, threadIdx.x);
    }
    if (p.y_zero) {
      float4* z = reinterpret_cast<float4*>(p.y_zero);
      const size_t n4 = p.y_zero_elems / 4;
      for (size_t i = (size_t)blockIdx.x * RT_THREADS + threadIdx.x; i < n4; i += (size_t)gridDim.x * RT_THREADS)
        z[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    return;
  }
  for (int i = threadIdx.x; i < npairs; i += RT_THREADS) s_idx[i] = p.topk_idx[i];
  __syncthreads();
  if (p.router == ROUTER_SWITCH_TOP1) {
    // capacity (cumsum priority <= capacity, per batch row): dropped tokens get expert -1
    const int S = p.seq_len;
    const int B = p.T / S;
    for (int pe = warp; pe < B * p.E; pe += RT_WARPS) {
      const int b = pe / p.E, e = pe % p.E;
      int running = 0;
      for (int s0 = 0; s0 < S; s0 += 32) {
        const int sidx = s0 + lane;
        const int t = b * S + sidx;
        // dropped entries are stored as -(e+2): the pass is idempotent, so CTAs that read indices another CTA
        // has already rewritten reach the same result
        const int raw = sidx < S ? s_idx[t] : -1;
        const bool h = sidx < S && (raw >= 0 ? raw : -(raw + 2)) == e;
        const uint32_t m = __ballot_sync(0xffffffffu, h);
        if (h && running + __popc(m & ((1u << lane) - 1u)) + 1 > p.expert_capacity) s_idx[t] = -(e + 2);
        running += __popc(m);
      }
    }
    __syncthreads();
    if (blockIdx.x == 0)
      for (int i = threadIdx.x; i < npairs; i += RT_THREADS) p.topk_idx[i] = s_idx[i];
  }
  if (warp < nchunks) chunk_count_warp(s_idx, warp * CHUNK, p.T, p.k, p.E, s_cnt[warp]);
  __syncthreads();
  if (threadIdx.x < p.E) {
    const int e = threadIdx.x;
    int run = 0;
    for (int c = 0; c < nchunks; ++c) { const int v = s_cnt[c][e]; s_cnt[c][e] = run; run += v; }
    s_tot[e] = run;
  }
  __syncthreads();
  if (warp == 0) {
    // exclusive scan of the per-expert totals by one warp (E <= 256: 8 per lane)
    int v[MAX_PL], run = 0;
#pragma unroll
    for (int i = 0; i < MAX_PL; ++i) {
      const int e = lane * MAX_PL + i;
      v[i] = e < p.E ? s_tot[e] : 0;
      run += v[i];
    }
    int incl = run;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int o = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += o;
    }
    int base = incl - run;
#pragma unroll
    for (int i = 0; i < MAX_PL; ++i) {
      const int e = lane * MAX_PL + i;
      if (e < p.E) s_off[e] = base;
      base += v[i];
    }
    const int total = __shfl_sync(0xffffffffu, incl, 31);
    if (lane == 0) s_off[p.E] = total;
  }
  __syncthreads();
  if (blockIdx.x == 0) {
    for (int e = threadIdx.x; e <= p.E; e += RT_THREADS) {   // E may equal the block size: stride loop, not tid <= E
      if (!p.offsets_early) {   // otherwise the gate/top-k kernel published them (and the GEMM may be reading them now)
        p.offsets[e] = s_off[e];
        if (e < p.E) p.counts[e] = s_tot[e];
      }
      if (p.ep_dispatch) p.ep.offsets_src[e] = s_off[e];
    }
  }
  if (p.ep_dispatch && blockIdx.x == 0 && p.ep.inline_counts) {
    // counts ride in the extra last row of every peer segment
    for (int i = threadIdx.x; i < p.ep.nranks * p.E; i += RT_THREADS) {
      const int r = i / p.E, e = i - r * p.E;
      reinterpret_cast<int*>(ep_send_row(p.ep, r, p.ep.cap))[e] = s_tot[e];
    }
  }
  if (warp < nchunks) {
    const int* cb = s_cnt[warp];
    chunk_rank_warp(p, warp * CHUNK, [&](int e) { return s_off[e] + cb[e]; }, s_rows + warp * CHUNK * p.k, s_idx,
                    blockIdx.x == 0);
  }
  __syncthreads();
  // gather: CTA b copies rows b, b+grid, ...; the whole CTA moves one row (H*2 bytes) with 16 B vectors
  const size_t rb = row_bytes(p);
  for (int i = blockIdx.x; i < npairs; i += gridDim.x) {
    const int row = s_rows[i];
    if (row < 0) continue;
    const int t = i / p.k;
    void* dst;
    if (p.ep_dispatch) {
      // expert-parallel: the row goes to the rank that owns its expert (peer memory over NVLink, or the send buffer)
      const int El = p.E / p.ep.nranks;
      const int e = s_idx[i];
      const int r = e / El;
      dst = ep_send_row(p.ep, r, row - s_off[r * El]);
    } else {
      dst = reinterpret_cast<uint8_t*>(p.xp) + (size_t)row * rb;
    }
    copy_row<RT_THREADS>(p, t, s_idx[i], i, dst, threadIdx.x);
  }
  if (p.ep_dispatch && p.ep.p2p) p2p_signal(p.ep, 0);
  if (p.tl && threadIdx.x == 0) tl_max(p.tl + 3);
  if (p.y_zero) {
    float4* z = reinterpret_cast<float4*>(p.y_zero);
    const size_t n4 = p.y_zero_elems / 4;
    for (size_t i = (size_t)blockIdx.x * RT_THREADS + threadIdx.x; i < n4; i += (size_t)gridDim.x * RT_THREADS)
      z[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

static bool route_args_ok(const RouteParams& p);

// Look-ahead routing (cfg.lookahead_prefetch): one CTA per token applies the NEXT layer's router weight (p.gate_w) to this
// layer's input row and counts its top-k choice per expert.  softmax is monotonic, so top-k of the logits is the top-k of
// the scores (ties -> lowest index, like every routing kernel here); weights are not needed for a prefetch hint.
// DeepSeek-V3: the bias and the group rule change the order, so the next layer's full V3 selection runs (p.gate_bias =
// that layer's bias).  Mixtral / Qwen: top-k of the logits rounded to the model dtype, as their routers rank them.
__global__ void __launch_bounds__(RT_THREADS) lookahead_counts_kernel(const RouteParams p, int* __restrict__ counts_out) {
  __shared__ float s_logits[MAX_PL * 32];
  __shared__ float s_scr[MAX_PL * 32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t = blockIdx.x;
  for (int e = warp; e < p.E; e += RT_WARPS) {
    const float v = gate_dot_warp(p, t, e);
    if (lane == 0) s_logits[e] = v;
  }
  __syncthreads();
  if (warp == 0 && p.router == ROUTER_DEEPSEEK_V3) {
    float s[MAX_PL];
#pragma unroll
    for (int i = 0; i < MAX_PL; ++i) {
      const int e = lane + 32 * i;
      s[i] = e < p.E ? sigmoid_ref(s_logits[e]) : 0.f;
    }
    v3_select_warp(p, s, p.gate_bias, s_scr);
    if (lane < p.k) atomicAdd(counts_out + __float_as_int(s_scr[MAX_K + lane]), 1);
  } else if (warp == 0) {
    for (int j = 0; j < p.k; ++j) {
      float best = -INFINITY;
      int bi = 0x7fffffff;
      for (int e = lane; e < p.E; e += 32) {
        const float v = s_logits[e];
        if (v > best) { best = v; bi = e; }       // ascending e within a lane: first maximum kept
      }
      warp_argmax(best, bi);
      if (bi >= p.E) break;
      if (lane == 0) { atomicAdd(counts_out + bi, 1); s_logits[bi] = -INFINITY; }
      __syncwarp();
    }
  }
}

cudaError_t launch_lookahead_counts(const RouteParams& p, int* counts_out, cudaStream_t st) {
  if (!route_args_ok(p) || !p.gate_w || !p.x || !counts_out || p.T < 1 || p.T > FUSED_MAX_T || p.dtype == DT_F32 ||
      (p.router == ROUTER_DEEPSEEK_V3 && !p.gate_bias))
    return cudaErrorInvalidValue;
  lookahead_counts_kernel<<<p.T, RT_THREADS, 0, st>>>(p, counts_out);
  return cudaGetLastError();
}

static int small_permute_grid(const RouteParams& p) {
  const int pairs = p.T * p.k;
  return pairs < 1 ? 1 : (pairs > 128 ? 128 : pairs);
}

static bool route_args_ok(const RouteParams& p) {
  return p.E >= 1 && p.E <= MAX_PL * 32 && p.k >= 1 && p.k <= MAX_K && p.k <= p.E && p.H % 8 == 0 && p.T >= 0 &&
         (p.router != ROUTER_DEEPSEEK_GROUP || (p.n_group >= 1 && p.n_group <= 32 && p.E % p.n_group == 0 &&
                                                 p.topk_group >= 1 && p.topk_group <= p.n_group)) &&
         (p.router != ROUTER_DEEPSEEK_V3 || (p.n_group >= 1 && p.n_group <= 32 && p.E % p.n_group == 0 &&
                                              p.E / p.n_group >= 2 && p.topk_group >= 1 && p.topk_group <= p.n_group)) &&
         (p.router != ROUTER_SWITCH_TOP1 || (p.k == 1 && p.seq_len > 0 && p.T % p.seq_len == 0));
}

cudaError_t launch_route(const RouteParams& p, cudaStream_t st) {
  if (!route_args_ok(p)) return cudaErrorInvalidValue;
  if (p.router == ROUTER_DEEPSEEK_V3 && !p.gate_bias) return cudaErrorInvalidValue;   // the V3 gate always has a bias
  if (p.dtype == DT_F32 && (!p.logits || p.ep_dispatch)) return cudaErrorInvalidValue;   // fp32 models: router logits/scores come in
  if (p.T == 0) return cudaMemsetAsync(p.offsets, 0, sizeof(int) * (p.E + 1), st);
  if (p.T <= FUSED_MAX_T) {
    cudaError_t e = launch_cluster(gate_topk_small_kernel, dim3(p.T), dim3(RT_THREADS), 0, st, 1, p.ep_fused && p.pdl_edge, p);
    if (e != cudaSuccess || p.ep_fused) return e;      // ep_fused: that kernel also permuted and dispatched the rows
    return launch_pdl(permute_small_kernel, dim3(small_permute_grid(p)), dim3(RT_THREADS), 0, st, p);
  }
  const int nblocks = (p.T + TOK_PER_BLOCK - 1) / TOK_PER_BLOCK;
  const int nchunks = (p.T + CHUNK - 1) / CHUNK;
  RouteParams q = p;
  if (!p.logits) {
    if (!p.logits_out) return cudaErrorInvalidValue;
    {
      const int ngroups = (p.E + 7) / 8;
      const int nblocks = (p.T + GATE_TOK_PER_CTA - 1) / GATE_TOK_PER_CTA;
      // expert groups are split over blockIdx.y so that (rounds of resident CTAs) x (chunks per CTA) is smallest;
      // 2 CTAs fit per SM.  Ties -> fewer splits (each split re-reads the token rows).
      const long long slots = 2LL * H100_SMS;
      int gsplit = 1;
      long long best = -1;
      for (int g = 1; g <= ngroups; ++g) {
        const long long cost = (((long long)nblocks * g + slots - 1) / slots) * ((ngroups + g - 1) / g);
        if (best < 0 || cost < best) { best = cost; gsplit = g; }
      }
      gate_logits_kernel<<<dim3(nblocks, gsplit), 256, 0, st>>>(p);
    }
    q.logits = p.logits_out;
    q.logits_dtype = p.logits_model_dtype ? p.dtype : DT_F32;
    q.logits_are_scores = 0;
    q.logits_out = nullptr;
  }
  route_topk_kernel<<<nchunks, RT_THREADS, 0, st>>>(q);
  if (p.router == ROUTER_SWITCH_TOP1) {
    switch_capacity_kernel<<<p.T / p.seq_len, RT_THREADS, 0, st>>>(p);
    chunk_count_kernel<<<nblocks, RT_THREADS, 0, st>>>(p);
  }
  route_scan_kernel<<<1, 256, 0, st>>>(p, nchunks);
  route_permute_kernel<<<nchunks, RT_THREADS, 0, st>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_route_from_mask(const RouteParams& p, const uint8_t* mask, cudaStream_t st) {
  if (!route_args_ok(p) || mask == nullptr) return cudaErrorInvalidValue;
  if (p.T == 0) return cudaMemsetAsync(p.offsets, 0, sizeof(int) * (p.E + 1), st);
  if (p.T <= FUSED_MAX_T) {
    mask_to_topk_kernel<<<(p.T + RT_THREADS - 1) / RT_THREADS, RT_THREADS, 0, st>>>(p, mask);
    RouteParams q = p;
    q.router = ROUTER_MIXTRAL;   // routing decisions already taken: no capacity pass
    return launch_pdl(permute_small_kernel, dim3(small_permute_grid(q)), dim3(RT_THREADS), 0, st, q);
  }
  const int nblocks = (p.T + TOK_PER_BLOCK - 1) / TOK_PER_BLOCK;
  const int nchunks = (p.T + CHUNK - 1) / CHUNK;
  mask_to_topk_kernel<<<(p.T + RT_THREADS - 1) / RT_THREADS, RT_THREADS, 0, st>>>(p, mask);
  chunk_count_kernel<<<nblocks, RT_THREADS, 0, st>>>(p);
  route_scan_kernel<<<1, 256, 0, st>>>(p, nchunks);
  route_permute_kernel<<<nchunks, RT_THREADS, 0, st>>>(p);
  return cudaGetLastError();
}

// --------------------------------------------------------------------------------------
// K5: un-permute + weighted combine.  One warp-group of lanes shares a token's (row, weight) list by
// warp shuffle; every lane owns 8 consecutive hidden elements (2 x 16 B fp32 loads per expert row,
// one 16 B store).  Experts are applied in ascending expert id (the oracle's fixed order).
// RULE: which combine arithmetic the instantiation compiles (launch_combine picks it):
//   RULE_PLAIN   COMBINE_MIXTRAL / DEEPSEEK / SWITCH / FP32, and the expert-parallel collect path;
//   RULE_QWEN    Qwen2-MoE / Qwen3-MoE layers (COMBINE_QWEN, or COMBINE_FP32 with a gated shared expert);
//   RULE_LLAMA4  Llama 4 layers (COMBINE_LLAMA4, or COMBINE_FP32): the routing weights already scaled the expert inputs, so
//                the expert outputs are summed without weights -- routed_out.reshape(k, T, H).sum(dim=0) on the model dtype
//                accumulates round(y) in fp32 and rounds once -- and out = shared_expert(x).add_(that sum):
//                round(r + round(s)).  COMBINE_FP32: round(sum of y + s).  Experts in ascending id, as in the dense HF
//                sum (its unselected experts add exact zeros).  No weights are loaded and there is no collect path.
// Each branch on RULE is decided at compile time, so the plain and Qwen instantiations compile exactly the code they had
// before the Qwen and Llama 4 rules existed.
// --------------------------------------------------------------------------------------
constexpr int CB_THREADS = 256;
enum : int { RULE_PLAIN = 0, RULE_QWEN = 1, RULE_LLAMA4 = 2 };

template <int DT, int RULE>
__global__ void __launch_bounds__(CB_THREADS) combine_kernel(const CombineParams p) {
  constexpr bool WEIGHTED = RULE != RULE_LLAMA4;   // also: may collect expert-parallel outputs
  const int t = blockIdx.x;
  const int lane = threadIdx.x & 31;
  const int k = p.k;
  pdl_launch();
  // expert parallel, direct mode: launched with a programmatic edge behind the down GEMM and NOT waiting for that grid to
  // drain -- everything it reads from earlier kernels is older than the GEMMs (routing tables) and the expert outputs are
  // guarded by the owners' "done" flags (this rank's own included), so its CTAs are resident and polling when "done" lands
  if (!(WEIGHTED && p.ep_collect && p.ep.direct && p.ep_early)) pdl_wait();
  if (p.tl && threadIdx.x == 0) tl_min(p.tl);
  // each warp loads the token's routing list into lanes 0..k-1 and sorts it by expert id via shuffles
  int my_e = 0x7fffffff, my_row = -1;
  float my_w = 0.f;
  if (lane < k) {
    my_e = p.topk_idx[(size_t)t * k + lane];
    if (WEIGHTED) my_w = p.topk_w[(size_t)t * k + lane];
    my_row = p.row_of[(size_t)t * k + lane];
    if (my_e < 0 || my_row < 0) { my_e = 0x7ffffff0 + lane; my_row = -1; }
  }
  int rank = 0;
  for (int j = 0; j < k; ++j) {
    const int oe = __shfl_sync(0xffffffffu, my_e, j);
    rank += (oe < my_e) ? 1 : 0;
  }
  int rows[MAX_K];
  float ws[MAX_K];
  const uint16_t* src16[MAX_K];
  const float* srcf[MAX_K];
  int my_owner = 0;
  if (WEIGHTED && p.ep_collect) {
    if (p.ep.p2p) p2p_wait(p.ep, 1, (p.ep.direct && p.ep_early) ? 0 : -1);   // return rows landed (direct mode: the owners' GEMMs are done)
    if (p.tl && threadIdx.x == 0) tl_max(p.tl + 1);
    if (lane < k && my_row >= 0) {
      // permuted row -> (owner rank, position in that rank's segment of this rank's return area)
      const int El = p.ep.E / p.ep.nranks;
      const int r = my_e / El;
      const int stride = p.ep.inline_counts ? p.ep.cap + 1 : p.ep.cap;
      my_owner = r;
      my_row = p.ep.direct ? (my_e - r * El) * p.ep.region_rows + my_row     // row_of = row inside the expert's region at the owner
                           : r * stride + (my_row - p.ep.offsets_src[r * El]);
    }
  }
#pragma unroll
  for (int r = 0; r < MAX_K; ++r) {
    rows[r] = -1;
    ws[r] = 0.f;
    src16[r] = nullptr;
    srcf[r] = nullptr;
    if (r < k) {
      const uint32_t who = __ballot_sync(0xffffffffu, lane < k && rank == r);
      const int src = __ffs(who) - 1;
      rows[r] = __shfl_sync(0xffffffffu, my_row, src);
      if (WEIGHTED) ws[r] = __shfl_sync(0xffffffffu, my_w, src);
      const int owner = __shfl_sync(0xffffffffu, my_owner, src);
      if (WEIGHTED && p.ep_collect && rows[r] >= 0) {
        if (p.ep.direct) srcf[r] = p.ep.peer_y[owner] + (size_t)rows[r] * p.H;   // the owner's fp32 outputs, read over NVLink
        else src16[r] = reinterpret_cast<const uint16_t*>(p.ep.back_rows) + (size_t)rows[r] * p.H;
      }
    }
  }
  const int H = p.H;
  for (int h = (blockIdx.y * CB_THREADS + threadIdx.x) * 8; h < H; h += gridDim.y * CB_THREADS * 8) {
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    bool any = false;
    // expert rows are fetched four at a time (invalid rows read row 0 and are ignored): up to 4 independent requests
    // in flight instead of one dependent round trip per expert, at 32 registers
#pragma unroll
    for (int r0 = 0; r0 < MAX_K; r0 += 4) {
      if (r0 >= k) break;
      float yk[4][8];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int r = r0 + q;
        if (r < k) {
          const bool ok = rows[r] >= 0;
          if (WEIGHTED && p.ep_collect && p.ep.direct) {
            const float4* src = reinterpret_cast<const float4*>((ok ? srcf[r] : p.ep.local_y) + h);
            const float4 a = src[0], b = src[1];
            yk[q][0] = a.x; yk[q][1] = a.y; yk[q][2] = a.z; yk[q][3] = a.w;
            yk[q][4] = b.x; yk[q][5] = b.y; yk[q][6] = b.z; yk[q][7] = b.w;
          } else if (WEIGHTED && p.ep_collect) {
            const uint16_t* sp = ok ? src16[r] : reinterpret_cast<const uint16_t*>(p.ep.back_rows);
            const uint4 v = *reinterpret_cast<const uint4*>(sp + h);
            const uint16_t* vs = reinterpret_cast<const uint16_t*>(&v);
#pragma unroll
            for (int i = 0; i < 8; ++i) yk[q][i] = Half16<DT>::to_f(vs[i]);
          } else {
            const float4* src = reinterpret_cast<const float4*>(p.y + (size_t)(ok ? rows[r] : 0) * H + h);
            const float4 a = src[0], b = src[1];
            yk[q][0] = a.x; yk[q][1] = a.y; yk[q][2] = a.z; yk[q][3] = a.w;
            yk[q][4] = b.x; yk[q][5] = b.y; yk[q][6] = b.z; yk[q][7] = b.w;
          }
        }
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int r = r0 + q;
        if (r < k && rows[r] >= 0) {
          const float (&y)[8] = yk[q];
          const float w = ws[r];
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            if (RULE == RULE_LLAMA4) {
              acc[i] = __fadd_rn(acc[i], p.mode == COMBINE_FP32 ? y[i] : round_dt<DT>(y[i]));
            } else if (p.mode == COMBINE_FP32) {
              acc[i] = fmaf(y[i], w, acc[i]);
            } else if (p.mode == COMBINE_MIXTRAL) {
              // out (model dtype) * weight (model dtype) -> rounded; final += -> rounded  (mixtral.py:98-101)
              const float prod = round_dt<DT>(__fmul_rn(round_dt<DT>(y[i]), w));
              acc[i] = any ? round_dt<DT>(__fadd_rn(acc[i], prod)) : prod;
            } else if (p.mode == COMBINE_DEEPSEEK) {
              // out (model dtype) * weight (fp32) -> fp32; final(model dtype) += fp32 -> rounded (deepseek.py:125-128)
              const float prod = __fmul_rn(round_dt<DT>(y[i]), w);
              acc[i] = round_dt<DT>(__fadd_rn(acc[i], prod));
            } else if (RULE == RULE_QWEN) {   // COMBINE_QWEN
              // Qwen2MoeExperts: index_add_(final (model dtype, zeros), (out (model dtype) * weight (fp32)).to(model dtype)):
              // the product is rounded, then every add is rounded
              const float prod = round_dt<DT>(__fmul_rn(round_dt<DT>(y[i]), w));
              acc[i] = round_dt<DT>(__fadd_rn(acc[i], prod));
            } else {  // COMBINE_SWITCH: next_states[idx] = out (switch_transformers.py:99-101)
              acc[i] = round_dt<DT>(y[i]);
            }
          }
          any = true;
        }
      }
    }
    if (WEIGHTED && p.mode == COMBINE_SWITCH) {
      // dropped tokens keep their input; hidden = router_probs * next_states (switch_transformers.py:81,109)
      const uint4 xv = *reinterpret_cast<const uint4*>(reinterpret_cast<const uint16_t*>(p.x) + (size_t)t * H + h);
      const uint16_t* xs = reinterpret_cast<const uint16_t*>(&xv);
      const float prob = p.topk_w[(size_t)t * k];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float nxt = any ? acc[i] : Half16<DT>::to_f(xs[i]);
        acc[i] = __fmul_rn(prob, nxt);
      }
    }
    if (p.y_shared) {
      const float4* src = reinterpret_cast<const float4*>(p.y_shared + (size_t)t * H + h);
      const float4 a = src[0], b = src[1];
      const float s[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
      if (RULE == RULE_QWEN) {
        // Qwen2MoeSparseMoeBlock: out + sigmoid(shared_expert_gate(x)) * shared_expert(x), every op in the model dtype;
        // g = that sigmoid, already rounded (shared_gate_kernel)
        const float g = Half16<DT>::to_f(p.shared_gate[t]);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          if (p.mode == COMBINE_FP32) acc[i] = fmaf(g, s[i], acc[i]);
          else acc[i] = round_dt<DT>(__fadd_rn(acc[i], round_dt<DT>(__fmul_rn(g, round_dt<DT>(s[i])))));
        }
      } else if (RULE == RULE_LLAMA4) {
#pragma unroll
        for (int i = 0; i < 8; ++i)
          acc[i] = p.mode == COMBINE_FP32 ? __fadd_rn(acc[i], s[i]) : __fadd_rn(round_dt<DT>(acc[i]), round_dt<DT>(s[i]));
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          if (p.mode == COMBINE_FP32) acc[i] += s[i];
          else acc[i] = round_dt<DT>(__fadd_rn(acc[i], round_dt<DT>(s[i])));   // final + shared_experts(identity), deepseek.py:133-136
        }
      }
    }
    uint4 o;
    uint16_t* os = reinterpret_cast<uint16_t*>(&o);
#pragma unroll
    for (int i = 0; i < 8; ++i) os[i] = Half16<DT>::from_f(acc[i]);
    *reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(p.out) + (size_t)t * H + h) = o;
  }
  if (p.tl && threadIdx.x == 0) tl_max(p.tl + 2);
}

static cudaError_t launch_shared_gate(const CombineParams& p, cudaStream_t st);

template <int DT>
static cudaError_t launch_combine_rule(int rule, dim3 grid, bool early, const CombineParams& p, cudaStream_t st) {
  void (*kernel)(const CombineParams) = rule == RULE_LLAMA4 ? combine_kernel<DT, RULE_LLAMA4>
                                        : rule == RULE_QWEN ? combine_kernel<DT, RULE_QWEN>
                                                            : combine_kernel<DT, RULE_PLAIN>;
  return launch_cluster(kernel, grid, dim3(CB_THREADS), 0, st, 1, early, p);
}

cudaError_t launch_combine(const CombineParams& p, cudaStream_t st) {
  if (p.T == 0) return cudaSuccess;
  if (p.mode == COMBINE_QWEN_GATE) return launch_shared_gate(p, st);
  if (p.k > MAX_K || p.H % 8 != 0) return cudaErrorInvalidValue;
  int gy = (p.H + CB_THREADS * 8 - 1) / (CB_THREADS * 8);
  dim3 grid(p.T, gy);
  if (p.dtype == DT_F32) return launch_combine_f32(p, st);
  const int rule = (p.unweighted || p.mode == COMBINE_LLAMA4) ? RULE_LLAMA4
                   : (p.mode == COMBINE_QWEN || p.shared_gate) ? RULE_QWEN : RULE_PLAIN;
  if (rule == RULE_LLAMA4 && (!p.unweighted || (p.mode != COMBINE_LLAMA4 && p.mode != COMBINE_FP32) || !p.y_shared ||
                              p.ep_collect || p.shared_gate))
    return cudaErrorInvalidValue;
  if (rule == RULE_QWEN && (p.ep_collect || (p.y_shared && !p.shared_gate))) return cudaErrorInvalidValue;
  const bool early = rule == RULE_PLAIN && p.ep_collect && p.ep.direct && p.ep_early;
  if (p.dtype == DT_BF16) return launch_combine_rule<DT_BF16>(rule, grid, early, p, st);
  if (p.dtype == DT_F16) return launch_combine_rule<DT_F16>(rule, grid, early, p, st);
  return cudaErrorInvalidValue;
}

// --------------------------------------------------------------------------------------
// Qwen2-MoE shared-expert gate: g[t] = sigmoid(shared_expert_gate(x[t])) with every op in the model dtype (an nn.Linear(H, 1)
// without bias, then F.sigmoid): the dot is accumulated in fp32 and rounded, the sigmoid is PyTorch's CUDA formula on that
// value (sigmoid_ref, as the V3 router) and is rounded again.  One warp per token, 16-byte loads of both operands.  It
// depends on x only: launch_combine runs it as the COMBINE_QWEN_GATE phase, which the caller issues on the shared-expert
// stream beside the routing kernels; the combine proper reads g.
// --------------------------------------------------------------------------------------
template <int DT>
__global__ void __launch_bounds__(256) shared_gate_kernel(const uint16_t* __restrict__ x, const uint16_t* __restrict__ w,
                                                          uint16_t* __restrict__ out, int T, int H) {
  const int lane = threadIdx.x & 31;
  const int t = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (t >= T) return;
  const uint16_t* xr = x + (size_t)t * H;
  float acc = 0.f;
  for (int h = lane * 8; h < H; h += 256) {
    float xf[8], wf[8];
    unpack8(*reinterpret_cast<const uint4*>(xr + h), DT, xf);
    unpack8(*reinterpret_cast<const uint4*>(w + h), DT, wf);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc = fmaf(xf[j], wf[j], acc);
  }
  acc = warp_sum(acc);
  if (lane == 0) out[t] = Half16<DT>::from_f(round_dt<DT>(sigmoid_ref(round_dt<DT>(acc))));
}

static cudaError_t launch_shared_gate(const CombineParams& p, cudaStream_t st) {
  const int T = p.T, H = p.H;
  if (T < 0 || H % 8 || !p.x || !p.shared_gate_w || !p.out) return cudaErrorInvalidValue;
  const dim3 grid((T + 7) / 8);
  const uint16_t* xs = reinterpret_cast<const uint16_t*>(p.x);
  const uint16_t* ws = reinterpret_cast<const uint16_t*>(p.shared_gate_w);
  uint16_t* o = reinterpret_cast<uint16_t*>(p.out);
  const int dtype = p.dtype;
  if (dtype == DT_BF16) shared_gate_kernel<DT_BF16><<<grid, 256, 0, st>>>(xs, ws, o, T, H);
  else if (dtype == DT_F16) shared_gate_kernel<DT_F16><<<grid, 256, 0, st>>>(xs, ws, o, T, H);
  else return cudaErrorInvalidValue;
  return cudaGetLastError();
}

template <int DT>
__global__ void cast_rows_kernel(const float* __restrict__ y, uint16_t* __restrict__ out, size_t n) {
  for (size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 8; i < n; i += (size_t)gridDim.x * blockDim.x * 8) {
    const float4 a = *reinterpret_cast<const float4*>(y + i), b = *reinterpret_cast<const float4*>(y + i + 4);
    const float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    uint4 o;
    uint16_t* os = reinterpret_cast<uint16_t*>(&o);
#pragma unroll
    for (int j = 0; j < 8; ++j) os[j] = Half16<DT>::from_f(v[j]);
    *reinterpret_cast<uint4*>(out + i) = o;
  }
}

cudaError_t launch_cast_rows(const float* y, void* out, size_t n, int dtype, cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  if (n % 8) return cudaErrorInvalidValue;
  const int blocks = (int)((n / 8 + 255) / 256 < H100_SMS * 8 ? (n / 8 + 255) / 256 : H100_SMS * 8);
  if (dtype == DT_F32) return cudaMemcpyAsync(out, y, n * sizeof(float), cudaMemcpyDeviceToDevice, st);
  if (dtype == DT_BF16) cast_rows_kernel<DT_BF16><<<blocks, 256, 0, st>>>(y, (uint16_t*)out, n);
  else if (dtype == DT_F16) cast_rows_kernel<DT_F16><<<blocks, 256, 0, st>>>(y, (uint16_t*)out, n);
  else return cudaErrorInvalidValue;
  return cudaGetLastError();
}

}  // namespace b2m
