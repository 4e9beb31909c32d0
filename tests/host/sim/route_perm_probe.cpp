// TEST INFRASTRUCTURE ONLY: records the input-permutation table (RouteParams::input_perm) of every routing launch that
// csrc/api.cu makes in the host simulation.  Linked by tests/test_host_sim_act_order.py into its own copy of the host
// simulation with `-Wl,--wrap` on the two routing launchers: api.cu's calls land here, are recorded, and go on to the
// simulation's own launchers (fake_kernels.cpp) unchanged.
#include <cstdint>
#include <cstring>
#include <mutex>
#include <vector>

#include "b2m_internal.h"

namespace {
std::mutex g_mu;
std::vector<uintptr_t> g_seen;   // input_perm of each launch, in launch order (0 = no table)
void record(const b2m::RouteParams& p) {
  std::lock_guard<std::mutex> lk(g_mu);
  g_seen.push_back(reinterpret_cast<uintptr_t>(p.input_perm));
}
}  // namespace

extern "C" {
cudaError_t __real__ZN3b2m12launch_routeERKNS_11RouteParamsEP11CUstream_st(const b2m::RouteParams&, cudaStream_t);
cudaError_t __real__ZN3b2m22launch_route_from_maskERKNS_11RouteParamsEPKhP11CUstream_st(const b2m::RouteParams&,
                                                                                         const uint8_t*, cudaStream_t);

cudaError_t __wrap__ZN3b2m12launch_routeERKNS_11RouteParamsEP11CUstream_st(const b2m::RouteParams& p, cudaStream_t st) {
  record(p);
  return __real__ZN3b2m12launch_routeERKNS_11RouteParamsEP11CUstream_st(p, st);
}
cudaError_t __wrap__ZN3b2m22launch_route_from_maskERKNS_11RouteParamsEPKhP11CUstream_st(const b2m::RouteParams& p,
                                                                                         const uint8_t* mask, cudaStream_t st) {
  record(p);
  return __real__ZN3b2m22launch_route_from_maskERKNS_11RouteParamsEPKhP11CUstream_st(p, mask, st);
}

// copy up to `cap` recorded tables into `out`, clear the record; returns how many launches were recorded
size_t b2m_probe_take_perms(uintptr_t* out, size_t cap) {
  std::lock_guard<std::mutex> lk(g_mu);
  const size_t n = g_seen.size();
  if (out) std::memcpy(out, g_seen.data(), sizeof(uintptr_t) * (n < cap ? n : cap));
  g_seen.clear();
  return n;
}
}
