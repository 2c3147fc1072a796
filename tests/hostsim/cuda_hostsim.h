// TEST INFRASTRUCTURE ONLY -- never part of the product library.
//
// A tiny single-threaded emulation of the CUDA execution model, so that the *same* .cu sources
// that nvcc compiles for sm_90a (every kernel except the wgmma/TMA ones) can also be compiled
// by g++ and exercised by the CPU test-suite in a container that has no GPU:
//   * a kernel launch runs the blocks of the grid one after another;
//   * the threads of a block are ucontext fibers; __syncthreads() yields to the scheduler, which
//     resumes every live fiber once per barrier phase (= lock-step at barriers);
//   * warp shuffles are emulated with an exchange buffer + two barrier phases (all warps of the
//     block must execute the same shuffle sequence, which holds for the kernels in this repo);
//   * __shared__ becomes static storage (blocks are sequential), dynamic shared memory a global
//     buffer; cudaMalloc/cudaMemcpy/... map to malloc/memcpy; streams and events are no-ops.
// The library built this way (tests/hostsim/build.py -> libdfvo_hostsim.so) exports the same
// C-ABI as the product, is loaded only by tests/, and exists to validate indexing / layout /
// orchestration logic before GPU time is spent.  It is NOT a fallback: the product loader
// (df-vo_b200/b200/native.py) refuses to run without the nvcc-built library and a CUDA device.
#pragma once
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <ucontext.h>
#include <algorithm>
#include <functional>
#include <vector>

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __restrict__
#define __launch_bounds__(...)
#define __shared__ static
#define __constant__ static
#define __grid_constant__
#define __align__(n) __attribute__((aligned(n)))

struct dim3 {
  unsigned x, y, z;
  dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
struct uint3_ { unsigned x, y, z; };
struct uint4 { unsigned x, y, z, w; };
struct float4 { float x, y, z, w; };
inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { uint4 r = {x, y, z, w}; return r; }
extern uint3_ threadIdx, blockIdx;
extern dim3 blockDim, gridDim;
extern unsigned char* hostsim_dyn_smem;

typedef int cudaError_t;
typedef void* cudaStream_t;
typedef void* cudaEvent_t;
enum { cudaSuccess = 0, cudaErrorMemoryAllocation = 2 };
enum cudaMemcpyKind { cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice, cudaMemcpyDefault };
inline const char* cudaGetErrorString(cudaError_t) { return "hostsim"; }
inline cudaError_t cudaGetLastError() { return 0; }
inline cudaError_t cudaMalloc(void** p, size_t n) { *p = calloc(n ? n : 1, 1); return *p ? 0 : 2; }
inline cudaError_t cudaFree(void* p) { free(p); return 0; }
inline cudaError_t cudaMemset(void* p, int v, size_t n) { memset(p, v, n); return 0; }
inline cudaError_t cudaMemsetAsync(void* p, int v, size_t n, cudaStream_t) { memset(p, v, n); return 0; }
inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { memcpy(d, s, n); return 0; }
inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t) { memcpy(d, s, n); return 0; }
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return 0; }
inline cudaError_t cudaDeviceSynchronize() { return 0; }
inline cudaError_t cudaSetDevice(int) { return 0; }
inline cudaError_t cudaGetDevice(int* d) { *d = 0; return 0; }

// ---- bf16 ------------------------------------------------------------------------------
struct __nv_bfloat16 { uint16_t x; };
inline __nv_bfloat16 __float2bfloat16_rn(float f) {
  uint32_t u; memcpy(&u, &f, 4);
  __nv_bfloat16 r;
  if ((u & 0x7fffffffu) > 0x7f800000u) { r.x = 0x7fff; return r; }
  u += 0x7fffu + ((u >> 16) & 1u);
  r.x = (uint16_t)(u >> 16);
  return r;
}
inline float __bfloat162float(__nv_bfloat16 b) { uint32_t u = (uint32_t)b.x << 16; float f; memcpy(&f, &u, 4); return f; }

// ---- intrinsics ------------------------------------------------------------------------
template <typename T> inline T __ldg(const T* p) { return *p; }
inline float __fdividef(float a, float b) { return a / b; }
inline float __expf(float a) { return expf(a); }
inline float fminf_(float a, float b) { return a < b ? a : b; }
inline int __float2int_rd(float a) { return (int)floorf(a); }
inline float __fmaf_rn(float a, float b, float c) { return fmaf(a, b, c); }
inline float __fmul_rn(float a, float b) { volatile float r = a * b; return r; }
inline float __fadd_rn(float a, float b) { volatile float r = a + b; return r; }
inline float __fsub_rn(float a, float b) { volatile float r = a - b; return r; }
inline float __fdiv_rn(float a, float b) { volatile float r = a / b; return r; }
inline float __fsqrt_rn(float a) { return sqrtf(a); }
inline double __dmul_rn(double a, double b) { volatile double r = a * b; return r; }
inline double __dadd_rn(double a, double b) { volatile double r = a + b; return r; }
inline double __dsub_rn(double a, double b) { volatile double r = a - b; return r; }
inline double __ddiv_rn(double a, double b) { volatile double r = a / b; return r; }
inline double __fma_rn(double a, double b, double c) { return fma(a, b, c); }
inline int __popc(unsigned v) { return __builtin_popcount(v); }
inline int __ffs(int v) { return __builtin_ffs(v); }
inline int __clz(int v) { return v ? __builtin_clz((unsigned)v) : 32; }
inline double rsqrt(double x) { return 1.0 / sqrt(x); }
inline unsigned __float_as_uint(float f) { unsigned u; memcpy(&u, &f, 4); return u; }
inline float __uint_as_float(unsigned u) { float f; memcpy(&f, &u, 4); return f; }

namespace hostsim {
void yield_barrier();                       // __syncthreads
void launch(dim3 grid, dim3 block, size_t smem, const std::function<void()>& body);
unsigned long long shfl_u64(unsigned long long v, int src_lane_in_warp);
}
#define __syncthreads() hostsim::yield_barrier()
#define __syncwarp(...) ((void)0)

template <typename T> inline T hostsim_shfl(T v, int src) {
  static_assert(sizeof(T) <= 8, "shfl");
  unsigned long long u = 0; memcpy(&u, &v, sizeof(T));
  u = hostsim::shfl_u64(u, src);
  T r; memcpy(&r, &u, sizeof(T)); return r;
}
inline int hostsim_lane() { return (int)((threadIdx.x + blockDim.x * (threadIdx.y + blockDim.y * threadIdx.z)) & 31); }
template <typename T> inline T __shfl_xor_sync(unsigned, T v, int m) { return hostsim_shfl(v, hostsim_lane() ^ m); }
template <typename T> inline T __shfl_down_sync(unsigned, T v, int d) { int s = hostsim_lane() + d; return hostsim_shfl(v, s > 31 ? hostsim_lane() : s); }
template <typename T> inline T __shfl_up_sync(unsigned, T v, int d) { int s = hostsim_lane() - d; return hostsim_shfl(v, s < 0 ? hostsim_lane() : s); }
template <typename T> inline T __shfl_sync(unsigned, T v, int s) { return hostsim_shfl(v, s & 31); }
inline unsigned __ballot_sync(unsigned, int pred) {
  unsigned r = 0;
  for (int l = 0; l < 32; ++l) { unsigned b = hostsim_shfl<unsigned>(pred ? 1u : 0u, l); r |= (b << l); }
  return r;
}

// atomics (single OS thread -> plain ops)
template <typename T> inline T atomicAdd(T* p, T v) { T o = *p; *p = o + v; return o; }
template <typename T> inline T atomicMax(T* p, T v) { T o = *p; if (v > o) *p = v; return o; }
template <typename T> inline T atomicMin(T* p, T v) { T o = *p; if (v < o) *p = v; return o; }
inline unsigned atomicInc(unsigned* p, unsigned lim) { unsigned o = *p; *p = (o >= lim) ? 0 : o + 1; return o; }
template <typename T> inline T atomicExch(T* p, T v) { T o = *p; *p = v; return o; }
template <typename T> inline T atomicCAS(T* p, T c, T v) { T o = *p; if (o == c) *p = v; return o; }
inline void __threadfence() {}

// dynamic shared memory: kernels declare it through DFVO_DYN_SMEM(type, name)
#define DFVO_DYN_SMEM(type, name) type* name = reinterpret_cast<type*>(hostsim_dyn_smem)
#include <atomic>
namespace dfvo { extern std::atomic<long long> g_launch_count; }
#define DFVO_LAUNCH(kern, grid, block, smem, stream, ...) \
  do { ++dfvo::g_launch_count; hostsim::launch((grid), (block), (smem), [&]() { kern(__VA_ARGS__); }); } while (0)
