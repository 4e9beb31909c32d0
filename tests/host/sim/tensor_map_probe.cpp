// TEST INFRASTRUCTURE ONLY: records the arguments of every tensor map csrc/api.cu encodes in the host simulation.  Linked by
// tests/test_weight_format_maps.py into its own copy of the host simulation with `-Wl,--wrap=cudaGetDriverEntryPoint`:
// api.cu's request for cuTensorMapEncodeTiled lands here and gets the recorder, which passes every call on to the
// simulation's own encoder (fake_cudart.cpp) and records the maps that encoder accepts.
#include <cuda.h>
#include <cuda_runtime_api.h>

#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>

namespace {
using EncodeFn = decltype(&cuTensorMapEncodeTiled);
EncodeFn g_encode = nullptr;
std::mutex g_mu;
std::string g_maps;   // one line per encoded map

CUresult record_encode(CUtensorMap* tm, CUtensorMapDataType dt, cuuint32_t rank, void* base, const cuuint64_t* dims,
                       const cuuint64_t* strides, const cuuint32_t* box, const cuuint32_t* es, CUtensorMapInterleave il,
                       CUtensorMapSwizzle swz, CUtensorMapL2promotion l2, CUtensorMapFloatOOBfill oob) {
  const CUresult r = g_encode(tm, dt, rank, base, dims, strides, box, es, il, swz, l2, oob);
  if (r != CUDA_SUCCESS) return r;
  std::string line = "dt=" + std::to_string((int)dt) + " swz=" + std::to_string((int)swz) +
                     " base=" + std::to_string(reinterpret_cast<uintptr_t>(base));
  const char* sep = " dims=";
  for (cuuint32_t i = 0; i < rank; ++i, sep = ",") line += sep + std::to_string(dims[i]);
  sep = " strides=";
  for (cuuint32_t i = 0; i + 1 < rank; ++i, sep = ",") line += sep + std::to_string(strides[i]);
  sep = " box=";
  for (cuuint32_t i = 0; i < rank; ++i, sep = ",") line += sep + std::to_string(box[i]);
  std::lock_guard<std::mutex> lk(g_mu);
  g_maps += line + "\n";
  return r;
}
}  // namespace

extern "C" {
cudaError_t __real_cudaGetDriverEntryPoint(const char*, void**, unsigned long long, cudaDriverEntryPointQueryResult*);

cudaError_t __wrap_cudaGetDriverEntryPoint(const char* name, void** fn, unsigned long long flags,
                                           cudaDriverEntryPointQueryResult* q) {
  const cudaError_t e = __real_cudaGetDriverEntryPoint(name, fn, flags, q);
  if (e == cudaSuccess && *fn && std::strcmp(name, "cuTensorMapEncodeTiled") == 0) {
    g_encode = reinterpret_cast<EncodeFn>(*fn);
    *fn = reinterpret_cast<void*>(&record_encode);
  }
  return e;
}

// hand the record of the maps encoded so far to the test and clear it; returns the bytes the full record needs
size_t b2m_probe_take_maps(char* buf, size_t cap) {
  std::lock_guard<std::mutex> lk(g_mu);
  const size_t n = g_maps.size();
  if (buf && cap) {
    const size_t m = n < cap - 1 ? n : cap - 1;
    std::memcpy(buf, g_maps.data(), m);
    buf[m] = 0;
  }
  g_maps.clear();
  return n;
}
}
