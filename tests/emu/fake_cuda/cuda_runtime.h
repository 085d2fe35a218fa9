// fake_cuda/cuda_runtime.h — a host-only stand-in for the CUDA runtime, for compiling the LIBRARY's own .cu files
// (host code included) into libcozo_gpu_emu.so with g++ (tests/emu/build_emu_lib.py; TEST INFRASTRUCTURE ONLY).
// Device memory is host memory, streams are synchronous, events are wall-clock stamps, a kernel launch is
// emu::launch_dyn (cuda_emu.hpp: one OS thread per CUDA thread, blocks one after the other).  The "device" reports
// itself as sm_90 with a handful of SMs so that persistent grids stay small.  Nothing under cozo_b200/ includes this.
#pragma once
#include "../cuda_emu.hpp"

#include <string.h>

#include <chrono>
#include <cstdlib>
#include <tuple>

typedef int cudaError_t;
enum : int {
  cudaSuccess = 0,
  cudaErrorInvalidValue = 1,
  cudaErrorMemoryAllocation = 2,
  cudaErrorNotSupported = 801,
  cudaErrorLaunchFailure = 719,
};
typedef struct emu_stream_st* cudaStream_t;
struct emu_event_st {
  std::chrono::steady_clock::time_point t;
};
typedef emu_event_st* cudaEvent_t;
enum cudaMemcpyKind { cudaMemcpyHostToHost = 0, cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3, cudaMemcpyDefault = 4 };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
enum : unsigned { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2, cudaIpcMemLazyEnablePeerAccess = 1 };
struct cudaIpcMemHandle_t {
  char reserved[64];
};
struct cudaFuncAttributes {
  size_t sharedSizeBytes = 0;
  int numRegs = 0;
  int maxThreadsPerBlock = 1024;
};
struct cudaDeviceProp {
  char name[64];
  int major, minor, multiProcessorCount;
  size_t sharedMemPerBlockOptin, totalGlobalMem;
};

namespace emu {
inline thread_local cudaError_t t_last_error = cudaSuccess;
inline constexpr size_t kSmemOptin = 232448;  // 227 KB, the H100 opt-in limit: the host code sizes tiles against it
inline int sm_count() {
  const char* e = getenv("COZO_EMU_SM_COUNT");
  return e && *e ? atoi(e) : 4;
}
}  // namespace emu

inline const char* cudaGetErrorString(cudaError_t e) {
  switch (e) {
    case cudaSuccess: return "no error";
    case cudaErrorInvalidValue: return "invalid argument";
    case cudaErrorMemoryAllocation: return "out of memory";
    case cudaErrorNotSupported: return "operation not supported (CPU emulation)";
    default: return "emulated CUDA error";
  }
}
inline cudaError_t cudaGetLastError() {
  cudaError_t e = emu::t_last_error;
  emu::t_last_error = cudaSuccess;
  return e;
}
inline cudaError_t cudaGetDeviceCount(int* c) { *c = 1; return cudaSuccess; }
inline cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp* p, int) {
  memset(p, 0, sizeof(*p));
  strcpy(p->name, "CPU SIMT emulator (reports sm_90)");
  p->major = 9;
  p->minor = 0;
  p->multiProcessorCount = emu::sm_count();
  p->sharedMemPerBlockOptin = emu::kSmemOptin;
  p->totalGlobalMem = (size_t)8 << 30;
  return cudaSuccess;
}
inline cudaError_t cudaMemGetInfo(size_t* free_b, size_t* total_b) {
  *free_b = (size_t)256 << 20;  // small on purpose: chunked paths (sssp_chunks) really chunk
  *total_b = (size_t)8 << 30;
  return cudaSuccess;
}
// exact-size allocations so that AddressSanitizer sees an out-of-bounds access of a kernel; 128-byte aligned like cudaMalloc
template <class T>
inline cudaError_t cudaMalloc(T** p, size_t bytes) {
  void* q = nullptr;
  if (posix_memalign(&q, 256, bytes ? bytes : 1) != 0) {
    *p = nullptr;
    return cudaErrorMemoryAllocation;
  }
  memset(q, 0xA5, bytes);  // device memory is NOT zero-initialised: make reads of uninitialised memory visible
  *p = static_cast<T*>(q);
  return cudaSuccess;
}
inline cudaError_t cudaFree(void* p) { free(p); return cudaSuccess; }
inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { if (n) memmove(d, s, n); return cudaSuccess; }
inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind k, cudaStream_t = nullptr) { return cudaMemcpy(d, s, n, k); }
inline cudaError_t cudaMemcpy2D(void* d, size_t dpitch, const void* s, size_t spitch, size_t width, size_t height, cudaMemcpyKind) {
  for (size_t r = 0; r < height; ++r) memmove((char*)d + r * dpitch, (const char*)s + r * spitch, width);
  return cudaSuccess;
}
inline cudaError_t cudaMemset(void* p, int v, size_t n) { if (n) memset(p, v, n); return cudaSuccess; }
inline cudaError_t cudaMemsetAsync(void* p, int v, size_t n, cudaStream_t = nullptr) { return cudaMemset(p, v, n); }
inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = reinterpret_cast<cudaStream_t>(new int(0)); return cudaSuccess; }
inline cudaError_t cudaStreamDestroy(cudaStream_t s) { delete reinterpret_cast<int*>(s); return cudaSuccess; }
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = new emu_event_st(); return cudaSuccess; }
inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { return cudaEventCreate(e); }
inline cudaError_t cudaEventDestroy(cudaEvent_t e) { delete e; return cudaSuccess; }
inline cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t = nullptr) { e->t = std::chrono::steady_clock::now(); return cudaSuccess; }
inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return cudaSuccess; }
inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t a, cudaEvent_t b) {
  *ms = std::chrono::duration<float, std::milli>(b->t - a->t).count();
  return cudaSuccess;
}
inline cudaError_t cudaLaunchHostFunc(cudaStream_t, void (*fn)(void*), void* user) { fn(user); return cudaSuccess; }
template <class F> inline cudaError_t cudaFuncSetAttribute(F, cudaFuncAttribute, int bytes) {
  return bytes >= 0 && (size_t)bytes <= emu::kSmemOptin ? cudaSuccess : cudaErrorInvalidValue;
}
template <class F> inline cudaError_t cudaFuncGetAttributes(cudaFuncAttributes* a, F) { *a = cudaFuncAttributes(); return cudaSuccess; }
template <class F> inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int* n, F, int threads, size_t smem) {
  size_t by_smem = smem ? emu::kSmemOptin / smem : 16, by_threads = (size_t)2048 / (size_t)(threads > 0 ? threads : 1);
  *n = (int)std::min<size_t>(std::min(by_smem, by_threads), 4);
  return cudaSuccess;
}
// "IPC": the ranks of an emulated group are threads of one process, so a handle is just the pointer
inline cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_t* h, void* p) { memset(h, 0, sizeof(*h)); memcpy(h->reserved, &p, sizeof(p)); return cudaSuccess; }
inline cudaError_t cudaIpcOpenMemHandle(void** p, cudaIpcMemHandle_t h, unsigned) { memcpy(p, h.reserved, sizeof(*p)); return cudaSuccess; }
inline cudaError_t cudaIpcCloseMemHandle(void*) { return cudaSuccess; }

namespace emu {
// dynamic shared memory of the running launch (`extern __shared__` declarations are rewritten to read this)
inline thread_local uint8_t* t_dyn_smem = nullptr;
inline unsigned bx(unsigned b) { return b; }
inline unsigned bx(const emu_dim3& b) { return b.x * b.y * b.z; }
// kernel<<<grid, block, smem, stream>>>(args)  ->  emu::launch_k(grid, block, smem, "kernel", kernel, args)  (below)
template <class G, class B, class Body>
inline void launch_dyn(G grid, B block, size_t smem, Body body, const char* name) {
  const unsigned threads = bx(block);
  if (threads == 0 || threads > 1024 || smem > kSmemOptin) {
    t_last_error = cudaErrorInvalidValue;
    return;
  }
  const emu_dim3 g(grid);
  if (g.x == 0 || g.y == 0 || g.z == 0 || g.x > 2147483647u || g.y > 65535u || g.z > 65535u) {
    t_last_error = cudaErrorInvalidValue;  // a zero-sized or over-sized grid is a launch error on the device too
    return;
  }
  void* buf = nullptr;
  if (posix_memalign(&buf, 1024, smem ? smem : 16) != 0) {
    t_last_error = cudaErrorMemoryAllocation;
    return;
  }
  memset(buf, 0xC3, smem);  // shared memory is not initialised either
  uint8_t* sm = static_cast<uint8_t*>(buf);
  const char* to = getenv("COZO_EMU_LAUNCH_TIMEOUT_S");
  launch(g, threads, [&, sm] {
    t_dyn_smem = sm;
    Body b = body;  // every thread runs its own copy of the argument pack, like kernel parameters
    b();
  }, to && *to ? atof(to) : 300.0, name);
  free(buf);
}
// kernel<<<grid, block, smem, stream>>>(args): the argument expressions are evaluated ONCE, here on the launching thread,
// and the kernel sees by-value copies (kernel parameters) — never copies of host objects the expressions mention
template <class G, class B, class K, class... A>
inline void launch_k(G grid, B block, size_t smem, const char* name, K kernel, A... args) {
  auto pack = std::make_tuple(args...);
  launch_dyn(grid, block, smem, [kernel, pack]() mutable { std::apply(kernel, pack); }, name);
}
}  // namespace emu
