// ep_device.cuh -- device helpers of the peer-to-peer expert-parallel exchange (shared by ep.cu and route.cu).
#pragma once
#include "b2m_common.cuh"
#include "b2m_internal.h"

namespace b2m {

__device__ __forceinline__ void st_release_sys(int* p, int v) {
  asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// Flag store of a release SEQUENCE: the caller has issued one __threadfence_system() after its last payload store; the flag
// stores to the N peers are then relaxed, so they leave back to back.  (N st.release.sys in a row cost N NVLink round trips:
// each one is a system fence that waits for the previous peer's flag store to be acknowledged.)
__device__ __forceinline__ void st_relaxed_sys(int* p, int v) {
  asm volatile("st.relaxed.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ int ld_acquire_sys(const int* p) {
  int v;
  asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// Every CTA calls this after its last store to peer memory; the last CTA to arrive publishes epoch to all peers.
__device__ __forceinline__ void p2p_signal(const EpParams& p, int which /*0 dispatch, 1 return*/) {
  __syncthreads();                 // every thread's peer stores are ordered before thread 0's fence (CTA-scope barrier) ...
  if (threadIdx.x != 0) return;
  __threadfence_system();          // ... which makes them visible system-wide (fences are cumulative): one fence per CTA
  if (atomicAdd(p.done_ctr + which, 1) != (int)gridDim.x - 1) return;
  p.done_ctr[which] = 0;
  const int e = p.epoch[which] + 1;
  p.epoch[which] = e;
  __threadfence_system();          // last arriver: the other CTAs' (fenced) stores happen-before the flags (fence cumulativity)
  for (int r = 0; r < p.nranks; ++r) st_relaxed_sys((which ? p.peer_back_flag[r] : p.peer_recv_flag[r]) + p.rank, e);
}
// Wait until every source rank's flag reached this rank's own epoch (all ranks issue the same number of exchanges).
__device__ __forceinline__ void p2p_wait(const EpParams& p, int which, int epoch_word = -1) {
  if (threadIdx.x < p.nranks) {
    // epoch_word: which local epoch the flags must reach.  Direct mode's combine starts before this rank's own down GEMM has
    // bumped epoch[1], so it compares the "done" flags with epoch[0] (this layer's dispatch count, final since the routing
    // kernel finished): every layer call issues exactly one dispatch and one "done", so the two counters agree.
    const int want = *reinterpret_cast<volatile int*>(p.epoch + (epoch_word < 0 ? which : epoch_word));
    const int* f = (which ? p.local_back_flag : p.local_recv_flag) + threadIdx.x;
    while (ld_acquire_sys(f) < want) __nanosleep(64);
  }
  __syncthreads();
}

// destination of row `pos` of the segment this rank sends to rank r (dispatch direction)
__device__ __forceinline__ uint16_t* ep_send_row(const EpParams& p, int r, int pos) {
  const int stride = p.inline_counts ? p.cap + 1 : p.cap;
  uint16_t* seg = p.p2p ? reinterpret_cast<uint16_t*>(p.peer_recv[r]) + (size_t)p.rank * stride * p.H
                        : reinterpret_cast<uint16_t*>(p.send_rows) + (size_t)r * stride * p.H;
  return seg + (size_t)pos * p.H;
}

}  // namespace b2m
