// Host emulation of the CUDA subset used by the SIMT sources of iaf_b200 (TEST INFRASTRUCTURE ONLY).
//
// Purpose: the build container has no GPU, so `-m "not gpu"` tests compile iaf_capi.cu, iaf_pack.cu, iaf_simt.cu and
// iaf_bwd.cu with g++ against this header (-DIAF_EMU) into tests/emu/_build/libiaf_emu.so and drive the SAME C ABI with
// numpy buffers standing in for device memory.  That executes the kernels' real index arithmetic, shared-memory
// staging, barriers and reductions (one CUDA thread = one std::thread, one block at a time) and checks them against
// the oracle before any GPU time is spent.  It is not a product path: nothing under iaf_b200/ can load this library,
// it has no tensor-core path, and it is orders of magnitude slower than anything useful.
//
// Covered: __global__/__device__ qualifiers, threadIdx/blockIdx/blockDim/gridDim, static and dynamic shared memory,
// __syncthreads (std::barrier; a thread that returns early drops out of the barrier as on the device), __threadfence,
// atomicAdd, __ldg/__ldcg, float4, and the handful of runtime calls iaf_capi.cu makes (malloc/memset/memcpy as host
// operations, streams and events as no-ops).  Not covered on purpose: warp shuffles, inline PTX, wgmma/TMA.
#pragma once
#include <atomic>
#include <barrier>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <thread>
#include <vector>
#include <algorithm>
#if defined(__SANITIZE_ADDRESS__)
#include <sanitizer/asan_interface.h>
#endif

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __launch_bounds__(...)
#define __grid_constant__
#define __restrict__
#define __align__(n) alignas(n)
#define __shared__ static

struct uint3 { unsigned x, y, z; };
struct dim3 {
  unsigned x, y, z;
  dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
struct alignas(16) float4 { float x, y, z, w; };
struct alignas(8) float2 { float x, y; };
static inline float4 make_float4(float x, float y, float z, float w) { return float4{x, y, z, w}; }

namespace emu {
inline thread_local uint3 t_threadIdx, t_blockIdx;
inline dim3 g_blockDim, g_gridDim;
inline unsigned char* g_dyn_smem = nullptr;
inline thread_local std::barrier<>* t_bar = nullptr;
}  // namespace emu
#define threadIdx (emu::t_threadIdx)
#define blockIdx (emu::t_blockIdx)
#define blockDim (emu::g_blockDim)
#define gridDim (emu::g_gridDim)

#define IAF_DYN_SMEM(type, name) type* name = reinterpret_cast<type*>(emu::g_dyn_smem)
// cp.async: the emulated copy completes at once (a superset of the device's ordering guarantees after wait + barrier)
static inline void iaf_cp_async4(float* dst, const float* src, bool valid) { *dst = valid ? *src : 0.f; }
static inline void iaf_cp_async_commit() {}
template <int N> static inline void iaf_cp_async_wait() {}

static inline void __syncthreads() { emu::t_bar->arrive_and_wait(); }
static inline void __threadfence() { std::atomic_thread_fence(std::memory_order_seq_cst); }
static inline unsigned atomicAdd(unsigned* p, unsigned v) { return std::atomic_ref<unsigned>(*p).fetch_add(v); }
static inline float atomicAdd(float* p, float v) { return std::atomic_ref<float>(*p).fetch_add(v); }
static inline unsigned __umulhi(unsigned a, unsigned b) { return (unsigned)(((unsigned long long)a * b) >> 32); }
template <class T> static inline T __ldg(const T* p) { return *p; }
template <class T> static inline T __ldcg(const T* p) { return *reinterpret_cast<const volatile T*>(p); }
using std::max;
using std::min;

// ---- runtime ----
typedef int cudaError_t;
typedef void* cudaStream_t;
typedef void* cudaEvent_t;
enum { cudaSuccess = 0, cudaErrorMemoryAllocation = 2, cudaErrorInvalidValue = 1 };
enum { cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3 };
enum { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2 };
struct cudaDeviceProp { int major, minor, multiProcessorCount; };

template <class T> static inline cudaError_t cudaMalloc(T** p, size_t n) {
  *p = reinterpret_cast<T*>(std::aligned_alloc(256, (n + 255) / 256 * 256));
  return *p ? cudaSuccess : cudaErrorMemoryAllocation;
}
static inline cudaError_t cudaFree(void* p) { std::free(p); return cudaSuccess; }
static inline cudaError_t cudaMemset(void* p, int v, size_t n) { std::memset(p, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemsetAsync(void* p, int v, size_t n, cudaStream_t) { std::memset(p, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, int, cudaStream_t) { std::memcpy(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline const char* cudaGetErrorName(cudaError_t) { return "emu"; }
static inline const char* cudaGetErrorString(cudaError_t) { return "host emulation"; }
static inline cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
static inline cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return cudaSuccess; }
static inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp* p, int) { p->major = 10; p->minor = 0; p->multiProcessorCount = 4; return cudaSuccess; }
static inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = reinterpret_cast<void*>(1); return cudaSuccess; }
static inline cudaError_t cudaStreamDestroy(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return cudaSuccess; }
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { *e = reinterpret_cast<void*>(1); return cudaSuccess; }
static inline cudaError_t cudaEventDestroy(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t) { return cudaSuccess; }
template <class F> static inline cudaError_t cudaFuncSetAttribute(F, int, int) { return cudaSuccess; }

namespace emu {
// run one grid: blocks one after another (static / dynamic shared memory is one CTA's at a time), the threads of a block as
// std::threads.  The threads are created once per launch and walk the blocks together: a fresh barrier per block serves
// __syncthreads (a thread that returns early drops out of it, as on the device), a second reusable one marks the block
// boundary.
template <class K, class... A>
inline void launch(K kernel, dim3 grid, dim3 block, size_t smem, const A&... args) {
  g_blockDim = block;
  g_gridDim = grid;
  const unsigned nthreads = block.x * block.y * block.z;
  const size_t nblocks = (size_t)grid.x * grid.y * grid.z;
  std::vector<unsigned char> dyn(smem + 512);
  g_dyn_smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(dyn.data()) + 255) / 256 * 256);
#if defined(__SANITIZE_ADDRESS__)
  // under AddressSanitizer the bytes past the requested dynamic shared memory are poisoned: an out-of-range smem index
  // in a kernel is reported instead of landing in the allocation's slack
  ASAN_POISON_MEMORY_REGION(g_dyn_smem + smem, (size_t)(dyn.data() + dyn.size() - (g_dyn_smem + smem)));
  struct Unpoison {
    void* p; size_t n;
    ~Unpoison() { ASAN_UNPOISON_MEMORY_REGION(p, n); }
  } unpoison{g_dyn_smem + smem, (size_t)(dyn.data() + dyn.size() - (g_dyn_smem + smem))};
#endif
  std::vector<std::unique_ptr<std::barrier<>>> bars;
  bars.reserve(nblocks);
  for (size_t b = 0; b < nblocks; ++b) bars.emplace_back(new std::barrier<>((std::ptrdiff_t)nthreads));
  std::barrier<> boundary((std::ptrdiff_t)nthreads);
  std::vector<std::thread> th;
  th.reserve(nthreads);
  for (unsigned t = 0; t < nthreads; ++t) {
    th.emplace_back([&, t]() {
      t_threadIdx = uint3{t % block.x, (t / block.x) % block.y, t / (block.x * block.y)};
      for (size_t b = 0; b < nblocks; ++b) {
        t_blockIdx = uint3{(unsigned)(b % grid.x), (unsigned)((b / grid.x) % grid.y), (unsigned)(b / ((size_t)grid.x * grid.y))};
        t_bar = bars[b].get();
        kernel(args...);
        bars[b]->arrive_and_drop();  // an exited thread no longer takes part in this block's __syncthreads
        boundary.arrive_and_wait();  // nobody enters the next block while this one still uses the shared memory
      }
    });
  }
  for (auto& x : th) x.join();
}
}  // namespace emu
#define IAF_LAUNCH(kernel, grid, block, smem, stream, ...) emu::launch(kernel, dim3(grid), dim3(block), (size_t)(smem), __VA_ARGS__)
