// TEST INFRASTRUCTURE ONLY: a host emulation of the few CUDA runtime entry points csrc/api.cu uses, so that the C-ABI
// layer's HOST logic (context set-up, HBM slot cache, eviction policy, wave splitting, prefetch queue, launch planning,
// error handling) can be executed by the CPU test-suite without a GPU.  "Device" memory is host memory, copies are
// memcpy, streams and events complete immediately.  Linked only into tests/host/_build/libb2m_hostsim.so
// (tests/host/sim/build_sim.py); the product library links the real runtime and refuses to run without a GPU.
#include <cuda.h>
#include <cuda_runtime_api.h>

#include <atomic>
#include <cstdlib>
#include <cstring>

namespace {
std::atomic<long long> g_h2d_bytes{0}, g_d2h_bytes{0}, g_copies{0}, g_allocs{0}, g_frees{0}, g_alloc_bytes{0};
long long g_total_mem = 8LL << 30;
CUresult fake_encode_tiled(CUtensorMap* tm, CUtensorMapDataType, cuuint32_t rank, void* base, const cuuint64_t* dims,
                           const cuuint64_t* strides, const cuuint32_t* box, const cuuint32_t*, CUtensorMapInterleave,
                           CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill) {
  // the same argument checks the driver applies to the maps api.cu builds (16-byte base/stride alignment, box <= 256)
  if (!tm || !base || rank < 2 || rank > 5) return CUDA_ERROR_INVALID_VALUE;
  if (reinterpret_cast<uintptr_t>(base) % 16) return CUDA_ERROR_INVALID_VALUE;
  for (cuuint32_t i = 0; i + 1 < rank; ++i)
    if (strides[i] % 16) return CUDA_ERROR_INVALID_VALUE;
  for (cuuint32_t i = 0; i < rank; ++i)
    if (box[i] == 0 || box[i] > 256 || dims[i] == 0) return CUDA_ERROR_INVALID_VALUE;
  std::memset(tm, 0, sizeof *tm);
  std::memcpy(tm, &base, sizeof base);
  return CUDA_SUCCESS;
}
}  // namespace

extern "C" {
// statistics for the tests
long long b2m_sim_h2d_bytes() { return g_h2d_bytes; }
long long b2m_sim_d2h_bytes() { return g_d2h_bytes; }
long long b2m_sim_live_allocs() { return g_allocs - g_frees; }
void b2m_sim_set_total_mem(long long b) { g_total_mem = b; }

void** __cudaRegisterFatBinary(void*) { static void* h; return &h; }
void __cudaRegisterFatBinaryEnd(void**) {}
void __cudaUnregisterFatBinary(void**) {}

cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return cudaSuccess; }
cudaError_t cudaSetDevice(int) { return cudaSuccess; }
cudaError_t cudaGetDeviceProperties_v2(cudaDeviceProp* p, int) {
  std::memset(p, 0, sizeof *p);
  std::strcpy(p->name, "simulated H100 (host)");
  p->major = 9; p->minor = 0; p->multiProcessorCount = 132; p->totalGlobalMem = (size_t)g_total_mem;
  p->sharedMemPerBlockOptin = 227 * 1024;
  return cudaSuccess;
}
cudaError_t cudaMemGetInfo(size_t* f, size_t* t) { *f = *t = (size_t)g_total_mem; return cudaSuccess; }
const char* cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : "simulated CUDA error"; }
cudaError_t cudaGetLastError() { return cudaSuccess; }
cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
cudaError_t cudaDeviceGetStreamPriorityRange(int* lo, int* hi) { *lo = 0; *hi = -5; return cudaSuccess; }

cudaError_t cudaMalloc(void** p, size_t n) {
  void* q = nullptr;
  if (posix_memalign(&q, 1024, n ? n : 1)) return cudaErrorMemoryAllocation;
  std::memset(q, 0xCD, n);   // poison: anything read before it was written shows up
  *p = q; ++g_allocs; g_alloc_bytes += (long long)n;
  return cudaSuccess;
}
cudaError_t cudaFree(void* p) { if (p) { free(p); ++g_frees; } return cudaSuccess; }
cudaError_t cudaHostAlloc(void** p, size_t n, unsigned) {
  void* q = nullptr;
  if (posix_memalign(&q, 4096, n ? n : 1)) return cudaErrorMemoryAllocation;
  *p = q; ++g_allocs;
  return cudaSuccess;
}
cudaError_t cudaFreeHost(void* p) { if (p) { free(p); ++g_frees; } return cudaSuccess; }
cudaError_t cudaHostRegister(void*, size_t, unsigned) { return cudaSuccess; }
cudaError_t cudaHostUnregister(void*) { return cudaSuccess; }

static cudaError_t do_copy(void* d, const void* s, size_t n, cudaMemcpyKind k) {
  if (n) std::memcpy(d, s, n);
  ++g_copies;
  if (k == cudaMemcpyHostToDevice) g_h2d_bytes += (long long)n;
  if (k == cudaMemcpyDeviceToHost) g_d2h_bytes += (long long)n;
  return cudaSuccess;
}
cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind k) { return do_copy(d, s, n, k); }
cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind k, cudaStream_t) { return do_copy(d, s, n, k); }
cudaError_t cudaMemset(void* d, int v, size_t n) { std::memset(d, v, n); return cudaSuccess; }
cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t) { std::memset(d, v, n); return cudaSuccess; }

cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = reinterpret_cast<cudaStream_t>(malloc(8)); return cudaSuccess; }
cudaError_t cudaStreamCreateWithPriority(cudaStream_t* s, unsigned, int) { *s = reinterpret_cast<cudaStream_t>(malloc(8)); return cudaSuccess; }
cudaError_t cudaStreamDestroy(cudaStream_t s) { free(s); return cudaSuccess; }
cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
// test hook: pretend every stream is (not) being captured
static int g_fake_capturing = 0;
extern "C" void fake_set_capturing(int on) { g_fake_capturing = on; }
cudaError_t cudaStreamIsCapturing(cudaStream_t, cudaStreamCaptureStatus* s) {
  *s = g_fake_capturing ? cudaStreamCaptureStatusActive : cudaStreamCaptureStatusNone;
  return cudaSuccess;
}
cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return cudaSuccess; }
cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { *e = reinterpret_cast<cudaEvent_t>(malloc(8)); return cudaSuccess; }
cudaError_t cudaEventDestroy(cudaEvent_t e) { free(e); return cudaSuccess; }
cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t) { return cudaSuccess; }
cudaError_t cudaEventQuery(cudaEvent_t) { return cudaSuccess; }          // everything "submitted" has already run
cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }

// CUDA IPC: off by default (the real failure mode of a locked-down container); b2m_sim_enable_ipc(1) turns on an
// in-process emulation -- a handle is the pointer itself -- so that several "ranks" can live in one test process
static int g_ipc_on = 0;
extern "C" void b2m_sim_enable_ipc(int on) { g_ipc_on = on; }
cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_t* h, void* p) {
  if (!g_ipc_on) return cudaErrorNotSupported;
  std::memset(h, 0, sizeof *h);
  std::memcpy(h, &p, sizeof p);
  return cudaSuccess;
}
cudaError_t cudaIpcOpenMemHandle(void** p, cudaIpcMemHandle_t h, unsigned) {
  if (!g_ipc_on) return cudaErrorNotSupported;
  std::memcpy(p, &h, sizeof *p);
  return cudaSuccess;
}
cudaError_t cudaIpcCloseMemHandle(void*) { return g_ipc_on ? cudaSuccess : cudaErrorNotSupported; }

cudaError_t cudaGetDriverEntryPoint(const char* name, void** fn, unsigned long long, cudaDriverEntryPointQueryResult* q) {
  if (std::strcmp(name, "cuTensorMapEncodeTiled") == 0) {
    *fn = reinterpret_cast<void*>(&fake_encode_tiled);
    if (q) *q = cudaDriverEntryPointSuccess;
    return cudaSuccess;
  }
  *fn = nullptr;
  if (q) *q = cudaDriverEntryPointSymbolNotFound;
  return cudaSuccess;
}
}  // extern "C"
