// Shared helpers for the dfvo_b200 CUDA library (sm_90a only).
#pragma once
#include "launch.cuh"
#ifndef DFVO_HOSTSIM
#include <cuda_bf16.h>
#endif
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#define DFVO_OK 0
#define DFVO_EINVAL (-1)
#define DFVO_ECUDA (-2)
#define DFVO_ESHAPE (-3)
#define DFVO_ENOMEM (-4)
#define DFVO_ESTATE (-5)

#if defined(__CUDACC__)
#define DFVO_HD __host__ __device__ __forceinline__
#define DFVO_D __device__ __forceinline__
#define DFVO_HD_NOINLINE __host__ __device__ __noinline__
#else
#define DFVO_HD inline
#define DFVO_D inline
#define DFVO_HD_NOINLINE inline
#endif

namespace dfvo {

void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what, const char* file, int line);

#define DFVO_CUDA(expr)                                                          \
  do {                                                                           \
    cudaError_t _e = (expr);                                                     \
    if (_e != cudaSuccess) return dfvo::cuda_fail(_e, #expr, __FILE__, __LINE__); \
  } while (0)

#define DFVO_CHECK_LAUNCH() DFVO_CUDA(cudaGetLastError())

#define DFVO_REQUIRE(cond, code, ...)      \
  do {                                     \
    if (!(cond)) {                         \
      dfvo::set_error(__VA_ARGS__);        \
      return (code);                       \
    }                                      \
  } while (0)

// NHWC view with explicit strides (in elements).  Channel stride is 1.
template <typename T>
struct Ten {
  T* p;
  int N, H, W, C;
  long long sN, sH, sW;
  DFVO_HD T* at(int n, int y, int x) const {
    return p + n * sN + y * sH + x * sW;
  }
};

template <typename T>
inline Ten<T> make_ten(T* p, int N, int H, int W, int C, int pitch) {
  Ten<T> t;
  t.p = p; t.N = N; t.H = H; t.W = W; t.C = C;
  t.sW = pitch; t.sH = (long long)W * pitch; t.sN = (long long)H * W * pitch;
  return t;
}

template <typename T>
inline Ten<const T> cten(const Ten<T>& t) {
  Ten<const T> c;
  c.p = t.p; c.N = t.N; c.H = t.H; c.W = t.W; c.C = t.C; c.sN = t.sN; c.sH = t.sH; c.sW = t.sW;
  return c;
}

enum Act { ACT_NONE = 0, ACT_LEAKY = 1, ACT_RELU = 2, ACT_ELU = 3, ACT_SIGMOID = 4 };

DFVO_D float apply_act(float v, int act) {
  switch (act) {
    case ACT_LEAKY: return v > 0.f ? v : 0.1f * v;
    case ACT_RELU: return v > 0.f ? v : 0.f;
    case ACT_ELU: return v > 0.f ? v : expm1f(v);
    case ACT_SIGMOID: return 1.f / (1.f + expf(-v));
    default: return v;
  }
}

DFVO_D float to_f(float v) { return v; }
DFVO_D float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename T> DFVO_D T from_f(float v);
template <> DFVO_D float from_f<float>(float v) { return v; }
template <> DFVO_D __nv_bfloat16 from_f<__nv_bfloat16>(float v) {
  return __float2bfloat16_rn(v);
}

// fp32 -> tf32 grid (10-bit mantissa), round to nearest, ties away from zero: cvt.rna.tf32.f32 on the device, its bit-level
// equivalent in the CPU test build
DFVO_D float rna_tf32(float v) {
#if defined(__CUDA_ARCH__)
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
  return __uint_as_float(r);
#else
  uint32_t u;
  memcpy(&u, &v, 4);
  if ((u & 0x7f800000u) != 0x7f800000u) u = (u + 0x1000u) & 0xffffe000u;
  memcpy(&v, &u, 4);
  return v;
#endif
}

inline int cdiv(int a, int b) { return (a + b - 1) / b; }

}  // namespace dfvo
