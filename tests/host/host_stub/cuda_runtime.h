// TEST VEHICLE ONLY (g++, no CUDA): just enough of the CUDA execution model to run the kernels of bucket_affine.cuh
// on the CPU.  Per-thread kernels run one emulated thread at a time (the test sets threadIdx / blockIdx); kernels that
// synchronise or shuffle run one CTA at a time with one OS thread per CUDA thread, __syncthreads and the warp shuffles
// being barriers + an exchange buffer supplied by the test (stub_syncthreads / stub_shfl, host_kernel_test.cpp).
// Nothing in the product build includes this file: nvcc resolves <cuda_runtime.h> to the real header.
#pragma once
#ifdef __CUDACC__
#error "host_stub/cuda_runtime.h is for the g++ test build only"
#endif
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__
#define __launch_bounds__(...)
#define __shared__ static

struct Dim3Stub { unsigned x = 0, y = 0, z = 0; };
inline thread_local Dim3Stub threadIdx, blockIdx, blockDim, gridDim;
struct dim3 {   // launch grids (the emulated launches take x and y)
  unsigned x, y, z;
  dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
struct uint2 { unsigned x, y; };
inline uint2 make_uint2(unsigned x, unsigned y) { return uint2{x, y}; }
typedef void* cudaStream_t;
// just enough of the runtime API for the host orchestration of poly_host.cuh / qap_sparse.cuh / msm_host.cuh (device
// memory = heap; launches and copies are synchronous, so events order nothing)
typedef int cudaError_t;
constexpr cudaError_t cudaSuccess = 0;
typedef void* cudaEvent_t;
constexpr unsigned cudaEventDisableTiming = 2;
inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { static char token; *e = &token; return 0; }
inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t = nullptr) { return 0; }
inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return 0; }
inline cudaError_t cudaEventDestroy(cudaEvent_t) { return 0; }
inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned = 0) { return 0; }
enum cudaMemcpyKind { cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice };
inline cudaError_t cudaMalloc(void** p, size_t b) { *p = std::malloc(b ? b : 1); return *p ? 0 : 2; }
template <class T> inline cudaError_t cudaMalloc(T** p, size_t b) { return cudaMalloc(reinterpret_cast<void**>(p), b); }
inline cudaError_t cudaFree(void* p) { std::free(p); return 0; }
inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t b, cudaMemcpyKind, cudaStream_t) { std::memmove(d, s, b); return 0; }
inline cudaError_t cudaMemcpy(void* d, const void* s, size_t b, cudaMemcpyKind) { std::memmove(d, s, b); return 0; }
inline cudaError_t cudaMemsetAsync(void* d, int v, size_t b, cudaStream_t) { std::memset(d, v, b); return 0; }
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return 0; }
inline cudaError_t cudaGetLastError() { return 0; }

[[noreturn]] inline void stub_abort(const char* what) { std::fprintf(stderr, "host stub: %s is not emulated\n", what); std::abort(); }
// provided by the test translation unit (CTA-at-a-time emulation); mode 0 = idx, 1 = up, 2 = down
void stub_syncthreads();
uint32_t stub_shfl(uint32_t v, int arg, int mode, int width);
inline void __syncthreads() { stub_syncthreads(); }
inline uint32_t __shfl_sync(unsigned, uint32_t v, int lane, int width = 32) { return stub_shfl(v, lane, 0, width); }
inline uint32_t __shfl_up_sync(unsigned, uint32_t v, unsigned d, int width = 32) { return stub_shfl(v, (int)d, 1, width); }
inline uint32_t __shfl_down_sync(unsigned, uint32_t v, unsigned d, int width = 32) { return stub_shfl(v, (int)d, 2, width); }
inline unsigned long long __shfl_up_sync(unsigned m, unsigned long long v, unsigned d, int width = 32) {
  uint32_t lo = __shfl_up_sync(m, (uint32_t)v, d, width), hi = __shfl_up_sync(m, (uint32_t)(v >> 32), d, width);
  return ((unsigned long long)hi << 32) | lo;
}
unsigned stub_ballot(int pred);
void stub_syncwarp();   // warp barrier in CTA emulation, no-op otherwise
inline unsigned __ballot_sync(unsigned, int pred) { return stub_ballot(pred); }
inline int __ffs(int v) { return __builtin_ffs(v); }
inline int __popc(unsigned v) { return __builtin_popcount(v); }
inline int __clz(int v) { return v ? __builtin_clz((unsigned)v) : 32; }
template <class T> inline T atomicAdd(T* p, T v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
template <class T> inline T atomicOr(T* p, T v) { return __atomic_fetch_or(p, v, __ATOMIC_SEQ_CST); }
template <class T> inline T atomicMax(T* p, T v) {
  T o = __atomic_load_n(p, __ATOMIC_SEQ_CST);
  while (v > o && !__atomic_compare_exchange_n(p, &o, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
  return o;
}
