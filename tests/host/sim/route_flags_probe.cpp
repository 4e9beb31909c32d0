// TEST INFRASTRUCTURE ONLY: records RouteParams::scale_rows and RouteParams::logits_model_dtype of every b2m_route launch
// that csrc/api.cu makes in the host simulation.  Linked by tests/test_host_sim_router_table.py into its own copy of the
// host simulation with `-Wl,--wrap` on the routing launcher: api.cu's calls land here, are recorded, and go on to the
// simulation's own launcher (fake_kernels.cpp) unchanged.
#include <cstdint>
#include <cstring>
#include <mutex>
#include <vector>

#include "b2m_internal.h"

namespace {
std::mutex g_mu;
std::vector<int32_t> g_seen;   // per launch, in launch order: scale_rows, logits_model_dtype
}  // namespace

extern "C" {
cudaError_t __real__ZN3b2m12launch_routeERKNS_11RouteParamsEP11CUstream_st(const b2m::RouteParams&, cudaStream_t);

cudaError_t __wrap__ZN3b2m12launch_routeERKNS_11RouteParamsEP11CUstream_st(const b2m::RouteParams& p, cudaStream_t st) {
  {
    std::lock_guard<std::mutex> lk(g_mu);
    g_seen.push_back(p.scale_rows);
    g_seen.push_back(p.logits_model_dtype);
  }
  return __real__ZN3b2m12launch_routeERKNS_11RouteParamsEP11CUstream_st(p, st);
}

// copy up to `cap` recorded values (two per launch) into `out`, clear the record; returns how many values were recorded
size_t b2m_probe_take_route_flags(int32_t* out, size_t cap) {
  std::lock_guard<std::mutex> lk(g_mu);
  const size_t n = g_seen.size();
  if (out) std::memcpy(out, g_seen.data(), sizeof(int32_t) * (n < cap ? n : cap));
  g_seen.clear();
  return n;
}
}
