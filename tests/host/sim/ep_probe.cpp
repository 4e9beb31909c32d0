// TEST INFRASTRUCTURE ONLY: records the geometry of every expert-parallel exchange launch that csrc/api.cu makes in the
// host simulation, and refuses what the real launchers refuse (ep.cu's ep_ok) without launching.  Linked by
// tests/test_ep_loopback_cases.py into its own copy of the host simulation with `-Wl,--wrap` on the four exchange
// launchers: api.cu's calls land here, are checked and recorded, and go on to the simulation's own launchers
// (fake_kernels.cpp) unchanged.
#include <cstdint>
#include <cstring>
#include <mutex>
#include <vector>

#include "b2m_internal.h"

namespace {
std::mutex g_mu;
std::vector<int64_t> g_seen;   // per launch: kind (0 pack, 1 regroup, 2 ungroup, 3 unpack), nranks, rank, cap, inline, y_zero

bool ep_ok(const b2m::EpParams& p) {
  return p.nranks >= 1 && p.nranks <= 16 && p.E % p.nranks == 0 && p.E / p.nranks <= 128 && p.rank >= 0 &&
         p.rank < p.nranks && p.cap >= 1 && p.H % 8 == 0 && (!p.inline_counts || p.E * 4 <= p.H * 2);
}
bool record(int kind, const b2m::EpParams& p) {
  if (!ep_ok(p)) return false;
  std::lock_guard<std::mutex> lk(g_mu);
  const int64_t v[6] = {kind, p.nranks, p.rank, p.cap, p.inline_counts, p.y_zero ? (int64_t)p.y_zero_elems : 0};
  g_seen.insert(g_seen.end(), v, v + 6);
  return true;
}
}  // namespace

extern "C" {
cudaError_t __real__ZN3b2m14launch_ep_packERKNS_8EpParamsEiP11CUstream_st(const b2m::EpParams&, int, cudaStream_t);
cudaError_t __real__ZN3b2m17launch_ep_regroupERKNS_8EpParamsEP11CUstream_st(const b2m::EpParams&, cudaStream_t);
cudaError_t __real__ZN3b2m17launch_ep_ungroupERKNS_8EpParamsEiP11CUstream_st(const b2m::EpParams&, int, cudaStream_t);
cudaError_t __real__ZN3b2m16launch_ep_unpackERKNS_8EpParamsEiiP11CUstream_st(const b2m::EpParams&, int, int, cudaStream_t);

cudaError_t __wrap__ZN3b2m14launch_ep_packERKNS_8EpParamsEiP11CUstream_st(const b2m::EpParams& p, int rows, cudaStream_t st) {
  if (!record(0, p)) return cudaErrorInvalidValue;
  return __real__ZN3b2m14launch_ep_packERKNS_8EpParamsEiP11CUstream_st(p, rows, st);
}
cudaError_t __wrap__ZN3b2m17launch_ep_regroupERKNS_8EpParamsEP11CUstream_st(const b2m::EpParams& p, cudaStream_t st) {
  if (!record(1, p)) return cudaErrorInvalidValue;
  return __real__ZN3b2m17launch_ep_regroupERKNS_8EpParamsEP11CUstream_st(p, st);
}
cudaError_t __wrap__ZN3b2m17launch_ep_ungroupERKNS_8EpParamsEiP11CUstream_st(const b2m::EpParams& p, int dt, cudaStream_t st) {
  if (!record(2, p)) return cudaErrorInvalidValue;
  return __real__ZN3b2m17launch_ep_ungroupERKNS_8EpParamsEiP11CUstream_st(p, dt, st);
}
cudaError_t __wrap__ZN3b2m16launch_ep_unpackERKNS_8EpParamsEiiP11CUstream_st(const b2m::EpParams& p, int dt, int rows,
                                                                            cudaStream_t st) {
  if (!record(3, p)) return cudaErrorInvalidValue;
  return __real__ZN3b2m16launch_ep_unpackERKNS_8EpParamsEiiP11CUstream_st(p, dt, rows, st);
}

// copy up to `cap` recorded values (six per launch) into `out`, clear the record; returns how many values were recorded
size_t b2m_probe_take_ep(int64_t* out, size_t cap) {
  std::lock_guard<std::mutex> lk(g_mu);
  const size_t n = g_seen.size();
  if (out) std::memcpy(out, g_seen.data(), sizeof(int64_t) * (n < cap ? n : cap));
  g_seen.clear();
  return n;
}
}
