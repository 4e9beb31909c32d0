// ep.cu -- expert-parallel token dispatch helpers (BASELINE config 5: experts sharded over the GPUs of one box).
//
// The reference has no live collective (SURVEY §2.2): "multi-GPU" there is one process moving token rows with
// `.to(device)` (core/parallel/expert_dispatcher.cpp:283-285, :403-405).  Here one process per GPU owns a
// contiguous block of experts (rank r: experts [r*El, (r+1)*El)); because the routing kernel already sorts the
// gathered rows by expert id, a rank's outgoing rows are contiguous.  Exchange = fixed-capacity all-to-all
// (capacity C = T_local*k rows per peer, so no host ever needs the counts):
//   pack     : Xp segment of each destination rank -> send[r][0..n_r) ; send_counts[r][le]
//   (all-to-all of counts and rows: NCCL via torch.distributed, or peer copies)
//   regroup  : recv[s][c] rows -> workspace Xp grouped by local expert (expert-major, then source rank, then
//              source order); offsets[E+1] over GLOBAL expert ids (zero rows for experts of other ranks)
//   ungroup  : fp32 expert outputs Y -> ret[s][c] rows in the model dtype (what the reference's OutputFunc returns)
//   unpack   : back[r][i] rows -> fp32 Y at the source rank's permuted row positions, ready for the combine kernel
#include "b2m_common.cuh"
#include "b2m_internal.h"
#include "ep_device.cuh"

namespace b2m {

constexpr int EP_THREADS = 256;
constexpr int EP_MAX_RANKS = 16;
constexpr int EP_MAX_EL = 128;   // experts per rank (E <= 256, >= 2 ranks)

__device__ __forceinline__ void copy_row16(const uint16_t* src, uint16_t* dst, int H) {
  const uint4* s = reinterpret_cast<const uint4*>(src);
  uint4* d = reinterpret_cast<uint4*>(dst);
  for (int v = threadIdx.x; v < H / 8; v += EP_THREADS) d[v] = s[v];
}


// grid: one CTA per permuted row (grid-stride); CTA 0 also publishes counts and the source-side offsets copy
__global__ void __launch_bounds__(EP_THREADS) ep_pack_kernel(EpParams p) {
  __shared__ int s_start[EP_MAX_RANKS + 1];
  const int El = p.E / p.nranks;
  pdl_launch();
  pdl_wait();
  if (threadIdx.x <= p.nranks) s_start[threadIdx.x] = p.offsets[threadIdx.x * El];
  __syncthreads();
  const int stride = p.inline_counts ? p.cap + 1 : p.cap;   // rows per peer segment
  if (blockIdx.x == 0) {
    for (int e = threadIdx.x; e <= p.E; e += EP_THREADS) p.offsets_src[e] = p.offsets[e];
    if (p.send_counts)
      for (int e = threadIdx.x; e < p.E; e += EP_THREADS) p.send_counts[e] = p.offsets[e + 1] - p.offsets[e];
    if (p.inline_counts)   // the counts ride in the extra last row of every peer segment: one collective less
      for (int i = threadIdx.x; i < p.nranks * p.E; i += EP_THREADS) {
        const int r = i / p.E, e = i - r * p.E;
        uint16_t* seg = p.p2p ? reinterpret_cast<uint16_t*>(p.peer_recv[r]) + (size_t)p.rank * stride * p.H
                              : reinterpret_cast<uint16_t*>(p.send_rows) + (size_t)r * stride * p.H;
        reinterpret_cast<int*>(seg + (size_t)p.cap * p.H)[e] = p.offsets[e + 1] - p.offsets[e];
      }
  }
  const int total = s_start[p.nranks];
  for (int i = blockIdx.x; i < total; i += gridDim.x) {
    int r = 0;
    while (i >= s_start[r + 1]) ++r;
    const int pos = i - s_start[r];
    if (pos < p.cap) {
      uint16_t* seg = p.p2p ? reinterpret_cast<uint16_t*>(p.peer_recv[r]) + (size_t)p.rank * stride * p.H
                            : reinterpret_cast<uint16_t*>(p.send_rows) + (size_t)r * stride * p.H;
      copy_row16(reinterpret_cast<const uint16_t*>(p.xp) + (size_t)i * p.H, seg + (size_t)pos * p.H, p.H);
    }
  }
  if (p.p2p) p2p_signal(p, 0);
}

// grid-stride over (source rank s, slot c); every CTA rebuilds the small prefix tables in shared memory
__global__ void __launch_bounds__(EP_THREADS) ep_regroup_kernel(EpParams p) {
  __shared__ int s_cnt[EP_MAX_RANKS][EP_MAX_EL];   // recv_counts[s][le]
  __shared__ int s_pre[EP_MAX_RANKS][EP_MAX_EL];   // exclusive prefix over le inside source s
  __shared__ int s_src[EP_MAX_RANKS][EP_MAX_EL];   // rows of sources < s for expert le
  __shared__ int s_off[EP_MAX_EL + 1];             // first workspace row of local expert le
  __shared__ int s_tot[EP_MAX_RANKS];
  const int N = p.nranks, El = p.E / p.nranks;
  const int stride = p.inline_counts ? p.cap + 1 : p.cap;
  pdl_launch();
  pdl_wait();
  if (p.p2p) p2p_wait(p, 0);
  for (int i = threadIdx.x; i < N * El; i += EP_THREADS) {
    const int s = i / El, le = i % El;
    const int* cnt = p.inline_counts
        ? reinterpret_cast<const int*>(reinterpret_cast<const uint16_t*>(p.recv_rows) + ((size_t)s * stride + p.cap) * p.H)
        : p.recv_counts + (size_t)s * p.E;
    s_cnt[s][le] = cnt[p.rank * El + le];
  }
  __syncthreads();
  if (threadIdx.x < N) {
    int run = 0;
    for (int le = 0; le < El; ++le) { s_pre[threadIdx.x][le] = run; run += s_cnt[threadIdx.x][le]; }
    s_tot[threadIdx.x] = min(run, p.cap);
  }
  if (threadIdx.x < El) {
    int run = 0;
    for (int s = 0; s < N; ++s) { s_src[s][threadIdx.x] = run; run += s_cnt[s][threadIdx.x]; }
    s_off[threadIdx.x] = run;   // total of expert le (turned into an exclusive prefix below)
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int le = 0; le < El; ++le) { const int v = s_off[le]; s_off[le] = acc; acc += v; }
    s_off[El] = acc;
  }
  __syncthreads();
  if (blockIdx.x == 0) {
    // offsets over global expert ids: experts of lower ranks have no rows here, higher ranks neither
    for (int e = threadIdx.x; e <= p.E; e += EP_THREADS) {
      const int le = e - p.rank * El;
      p.offsets_rw[e] = le <= 0 ? 0 : (le >= El ? s_off[El] : s_off[le]);
    }
  }
  const int slots = N * p.cap;
  for (int i = blockIdx.x; i < slots; i += gridDim.x) {
    const int s = i / p.cap, c = i - s * p.cap;
    int dest = -1;
    if (c < s_tot[s]) {
      int le = 0;
      while (le + 1 < El && c >= s_pre[s][le + 1]) ++le;
      dest = s_off[le] + s_src[s][le] + (c - s_pre[s][le]);
      copy_row16(reinterpret_cast<const uint16_t*>(p.recv_rows) + ((size_t)s * stride + c) * p.H,
                 reinterpret_cast<uint16_t*>(p.xp) + (size_t)dest * p.H, p.H);
    }
    if (threadIdx.x == 0) p.dest_of[i] = dest;
  }
  if (p.y_zero) {
    float4* z = reinterpret_cast<float4*>(p.y_zero);
    const size_t n4 = p.y_zero_elems / 4;
    for (size_t i = (size_t)blockIdx.x * EP_THREADS + threadIdx.x; i < n4; i += (size_t)gridDim.x * EP_THREADS)
      z[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

template <int DT>
__global__ void __launch_bounds__(EP_THREADS) ep_ungroup_kernel(EpParams p) {
  const int slots = p.nranks * p.cap;
  pdl_launch();
  pdl_wait();
  for (int i = blockIdx.x; i < slots; i += gridDim.x) {
    const int dest = p.dest_of[i];
    if (dest < 0) continue;
    const float* src = p.y + (size_t)dest * p.H;
    const int stride = p.inline_counts ? p.cap + 1 : p.cap;
    const int src_rank = i / p.cap, c = i % p.cap;
    uint16_t* dst = p.p2p ? reinterpret_cast<uint16_t*>(p.peer_back[src_rank]) + ((size_t)p.rank * stride + c) * p.H
                          : reinterpret_cast<uint16_t*>(p.ret_rows) + ((size_t)src_rank * stride + c) * p.H;
    for (int v = threadIdx.x * 8; v < p.H; v += EP_THREADS * 8) {
      const float4 a = *reinterpret_cast<const float4*>(src + v), b = *reinterpret_cast<const float4*>(src + v + 4);
      const float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
      uint4 o;
      uint16_t* os = reinterpret_cast<uint16_t*>(&o);
#pragma unroll
      for (int j = 0; j < 8; ++j) os[j] = Half16<DT>::from_f(f[j]);
      *reinterpret_cast<uint4*>(dst + v) = o;
    }
  }
  if (p.p2p) p2p_signal(p, 1);
}

template <int DT>
__global__ void __launch_bounds__(EP_THREADS) ep_unpack_kernel(EpParams p) {
  __shared__ int s_start[EP_MAX_RANKS + 1];
  const int El = p.E / p.nranks;
  pdl_launch();
  pdl_wait();
  if (p.p2p) p2p_wait(p, 1);
  if (threadIdx.x <= p.nranks) s_start[threadIdx.x] = p.offsets_src[threadIdx.x * El];
  __syncthreads();
  const int total = s_start[p.nranks];
  for (int i = blockIdx.x; i < total; i += gridDim.x) {
    int r = 0;
    while (i >= s_start[r + 1]) ++r;
    const int pos = i - s_start[r];
    if (pos >= p.cap) continue;
    const int stride = p.inline_counts ? p.cap + 1 : p.cap;
    const uint16_t* src = reinterpret_cast<const uint16_t*>(p.back_rows) + ((size_t)r * stride + pos) * p.H;
    float* dst = p.y + (size_t)i * p.H;
    for (int v = threadIdx.x * 8; v < p.H; v += EP_THREADS * 8) {
      const uint4 x = *reinterpret_cast<const uint4*>(src + v);
      const uint16_t* xs = reinterpret_cast<const uint16_t*>(&x);
      float4 a, b;
      a.x = Half16<DT>::to_f(xs[0]); a.y = Half16<DT>::to_f(xs[1]); a.z = Half16<DT>::to_f(xs[2]); a.w = Half16<DT>::to_f(xs[3]);
      b.x = Half16<DT>::to_f(xs[4]); b.y = Half16<DT>::to_f(xs[5]); b.z = Half16<DT>::to_f(xs[6]); b.w = Half16<DT>::to_f(xs[7]);
      *reinterpret_cast<float4*>(dst + v) = a;
      *reinterpret_cast<float4*>(dst + v + 4) = b;
    }
  }
}

static bool ep_ok(const EpParams& p) {
  return p.nranks >= 1 && p.nranks <= EP_MAX_RANKS && p.E % p.nranks == 0 && p.E / p.nranks <= EP_MAX_EL &&
         p.rank >= 0 && p.rank < p.nranks && p.cap >= 1 && p.H % 8 == 0 && (!p.inline_counts || p.E * 4 <= p.H * 2);
}
static int ep_grid(int rows) { return rows < 1 ? 1 : (rows > H100_SMS * 4 ? H100_SMS * 4 : rows); }

cudaError_t launch_ep_pack(const EpParams& p, int max_rows, cudaStream_t st) {
  if (!ep_ok(p)) return cudaErrorInvalidValue;
  return launch_pdl(ep_pack_kernel, dim3(ep_grid(max_rows)), dim3(EP_THREADS), 0, st, p);
}
cudaError_t launch_ep_regroup(const EpParams& p, cudaStream_t st) {
  if (!ep_ok(p)) return cudaErrorInvalidValue;
  return launch_pdl(ep_regroup_kernel, dim3(ep_grid(p.nranks * p.cap)), dim3(EP_THREADS), 0, st, p);
}
cudaError_t launch_ep_ungroup(const EpParams& p, int dtype, cudaStream_t st) {
  if (!ep_ok(p)) return cudaErrorInvalidValue;
  if (dtype == DT_BF16) return launch_pdl(ep_ungroup_kernel<DT_BF16>, dim3(ep_grid(p.nranks * p.cap)), dim3(EP_THREADS), 0, st, p);
  if (dtype == DT_F16) return launch_pdl(ep_ungroup_kernel<DT_F16>, dim3(ep_grid(p.nranks * p.cap)), dim3(EP_THREADS), 0, st, p);
  return cudaErrorInvalidValue;
}
cudaError_t launch_ep_unpack(const EpParams& p, int dtype, int max_rows, cudaStream_t st) {
  if (!ep_ok(p)) return cudaErrorInvalidValue;
  if (dtype == DT_BF16) return launch_pdl(ep_unpack_kernel<DT_BF16>, dim3(ep_grid(max_rows)), dim3(EP_THREADS), 0, st, p);
  if (dtype == DT_F16) return launch_pdl(ep_unpack_kernel<DT_F16>, dim3(ep_grid(max_rows)), dim3(EP_THREADS), 0, st, p);
  return cudaErrorInvalidValue;
}

}  // namespace b2m
