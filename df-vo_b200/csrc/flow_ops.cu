// Memory-bound kernels of the LiteFlowNet path: image prep / resizes, depthwise deconv, backward
// warp, 49-channel correlation, Regularization prep + tail, final flow upsample and the
// forward-backward consistency map.  Reference lines are cited per kernel; layouts are NHWC.
#include <stdlib.h>
#include "ops.h"

namespace dfvo {

// ---------------------------------------------------------------------------------------------
// bilinear helpers (torch upsample_bilinear2d semantics)
// ---------------------------------------------------------------------------------------------
struct Lerp { int i0, i1; float l0, l1; };

DFVO_D Lerp lerp_coord(int dst, int in_size, int out_size, int align_corners) {
  Lerp r;
  float src;
  if (align_corners) {
    float scale = out_size > 1 ? (float)(in_size - 1) / (float)(out_size - 1) : 0.f;
    src = scale * (float)dst;
  } else {
    float scale = (float)in_size / (float)out_size;
    src = scale * ((float)dst + 0.5f) - 0.5f;
    if (src < 0.f) src = 0.f;
  }
  r.i0 = (int)src;
  if (r.i0 > in_size - 1) r.i0 = in_size - 1;
  r.i1 = r.i0 + ((r.i0 < in_size - 1) ? 1 : 0);
  r.l1 = src - (float)r.i0;
  r.l0 = 1.f - r.l1;
  return r;
}

// deep_models.py:160-163 (img/255 in float64 -> float32) + lite_flow.py:72-76 (bilinear, AC=True)
__global__ void k_prep_image_u8(const uint8_t* __restrict__ img, int H0, int W0, Ten<float> out, int n) {
  int x = blockIdx.x * blockDim.x + threadIdx.x;
  int y = blockIdx.y;
  if (x >= out.W) return;
  Lerp ly = lerp_coord(y, H0, out.H, 1), lx = lerp_coord(x, W0, out.W, 1);
  float* o = out.at(n, y, x);
  for (int c = 0; c < 3; ++c) {
    float v00 = (float)((double)img[((size_t)ly.i0 * W0 + lx.i0) * 3 + c] / 255.0);
    float v01 = (float)((double)img[((size_t)ly.i0 * W0 + lx.i1) * 3 + c] / 255.0);
    float v10 = (float)((double)img[((size_t)ly.i1 * W0 + lx.i0) * 3 + c] / 255.0);
    float v11 = (float)((double)img[((size_t)ly.i1 * W0 + lx.i1) * 3 + c] / 255.0);
    o[c] = ly.l0 * (lx.l0 * v00 + lx.l1 * v01) + ly.l1 * (lx.l0 * v10 + lx.l1 * v11);
  }
  for (int c = 3; c < out.C; ++c) o[c] = 0.f;
}

int prep_image_u8(const uint8_t* img, int H0, int W0, Ten<float> out, int n, cudaStream_t s) {
  dim3 block(128), grid(cdiv(out.W, 128), out.H);
  DFVO_LAUNCH(k_prep_image_u8, grid, block, 0, s, img, H0, W0, out, n);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

__global__ void k_resize_bilinear_f32(Ten<const float> in, Ten<float> out, int ac) {
  int x = blockIdx.x * blockDim.x + threadIdx.x;
  int y = blockIdx.y, n = blockIdx.z;
  if (x >= out.W) return;
  Lerp ly = lerp_coord(y, in.H, out.H, ac), lx = lerp_coord(x, in.W, out.W, ac);
  const float* p00 = in.at(n, ly.i0, lx.i0);
  const float* p01 = in.at(n, ly.i0, lx.i1);
  const float* p10 = in.at(n, ly.i1, lx.i0);
  const float* p11 = in.at(n, ly.i1, lx.i1);
  float* o = out.at(n, y, x);
  for (int c = 0; c < in.C; ++c)
    o[c] = ly.l0 * (lx.l0 * p00[c] + lx.l1 * p01[c]) + ly.l1 * (lx.l0 * p10[c] + lx.l1 * p11[c]);
  for (int c = in.C; c < out.C; ++c) o[c] = 0.f;
}

int resize_bilinear_f32(Ten<const float> in, Ten<float> out, int align_corners, cudaStream_t s) {
  dim3 block(128), grid(cdiv(out.W, 128), out.H, out.N);
  DFVO_LAUNCH(k_resize_bilinear_f32, grid, block, 0, s, in, out, align_corners);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

// ---------------------------------------------------------------------------------------------
// Row-unroll of the 3-channel input for the 7x7 stem (lite_flow_net.py:39-42): out[n,y,x, dx*3+c] =
// img[n, y, x+dx-3, c] (zero outside), channels 21..31 zero.  The 7x7x3 convolution then is a 7x1
// convolution over 32 channels, which the wgmma kernel can run (its K granularity is 16 channels).
// ---------------------------------------------------------------------------------------------
template <typename T>
__global__ void k_im2row7(Ten<const float> img, Ten<T> out) {
  int x = blockIdx.x * blockDim.x + threadIdx.x;
  int y = blockIdx.y, n = blockIdx.z;
  if (x >= out.W) return;
  T* o = out.at(n, y, x);
#pragma unroll
  for (int dx = 0; dx < 7; ++dx) {
    const int xx = x + dx - 3;
    const bool in = xx >= 0 && xx < img.W;
    const float* p = img.at(n, y, in ? xx : 0);
#pragma unroll
    for (int c = 0; c < 3; ++c) o[dx * 3 + c] = from_f<T>(in ? p[c] : 0.f);
  }
  for (int c = 21; c < out.C; ++c) o[c] = from_f<T>(0.f);
}

template <typename T>
int im2row7(Ten<const float> img, Ten<T> out, cudaStream_t s) {
  DFVO_REQUIRE(out.C >= 21 && out.H == img.H && out.W == img.W, DFVO_ESHAPE, "im2row7 shapes");
  auto k = k_im2row7<T>;
  DFVO_LAUNCH(k, dim3(cdiv(out.W, 128), out.H, out.N), dim3(128), 0, s, img, out);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}
template int im2row7<float>(Ten<const float>, Ten<float>, cudaStream_t);
template int im2row7<bf16>(Ten<const float>, Ten<bf16>, cudaStream_t);

// ---------------------------------------------------------------------------------------------
// Column-padded 8-channel copy of the 3-channel input for the 7x7 stem: out[n, y, x + 3, 0..2] = img[n, y, x, 0..2],
// channels 3..7 and the 3 + 5 pad columns of every row stay zero (they are never written; the arena zero-fills).
// With 16 bytes per pixel, the 64 consecutive elements starting at padded column x are the 8 pixels x-3 .. x+4 of that
// row -- the horizontal window of the stem -- so a tensor map with a 16-byte pixel stride and a 64-element innermost
// dimension (overlapping boxes) lets TMA deliver the row-unrolled operand without materialising it.
// ---------------------------------------------------------------------------------------------
template <typename T>
__global__ void k_pad_image8(Ten<const float> img, Ten<T> out) {
  int x = blockIdx.x * blockDim.x + threadIdx.x;
  int y = blockIdx.y, n = blockIdx.z;
  if (x >= img.W) return;
  const float* p = img.at(n, y, x);
  T* o = out.at(n, y, x + 3);
  o[0] = from_f<T>(p[0]); o[1] = from_f<T>(p[1]); o[2] = from_f<T>(p[2]);
}

template <typename T>
int pad_image8(Ten<const float> img, Ten<T> out, cudaStream_t s) {
  DFVO_REQUIRE(out.C == 8 && out.H == img.H && out.W == img.W + 8 && out.sW == 8, DFVO_ESHAPE, "pad_image8 shapes");
  auto k = k_pad_image8<T>;
  DFVO_LAUNCH(k, dim3(cdiv(img.W, 128), img.H, img.N), dim3(128), 0, s, img, out);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}
template int pad_image8<float>(Ten<const float>, Ten<float>, cudaStream_t);
template int pad_image8<bf16>(Ten<const float>, Ten<bf16>, cudaStream_t);

// ---------------------------------------------------------------------------------------------
// depthwise ConvTranspose2d(k=4, s=2, p=1, groups=C, bias=False)  (lite_flow_net.py:109,117)
// out[oy] += in[iy] * w[ky] with oy = 2*iy - 1 + ky
// ---------------------------------------------------------------------------------------------
template <typename T>
__global__ void k_deconv4x4s2_dw(Ten<const T> in, const float* __restrict__ w, Ten<T> out) {
  int c = threadIdx.x % out.C, xi = threadIdx.x / out.C;
  int px_per_block = blockDim.x / out.C;
  int x = blockIdx.x * px_per_block + xi;
  int y = blockIdx.y, n = blockIdx.z;
  if (xi >= px_per_block || x >= out.W) return;
  float acc = 0.f;
  if (c < in.C) {
    int ky0 = (y + 1) & 1, kx0 = (x + 1) & 1;
    for (int a = 0; a < 2; ++a) {
      int ky = ky0 + 2 * a;
      int iy = (y + 1 - ky) / 2;
      if ((y + 1 - ky) < 0 || iy >= in.H) continue;
      for (int b = 0; b < 2; ++b) {
        int kx = kx0 + 2 * b;
        int ix = (x + 1 - kx) / 2;
        if ((x + 1 - kx) < 0 || ix >= in.W) continue;
        acc += to_f(in.at(n, iy, ix)[c]) * w[c * 16 + ky * 4 + kx];
      }
    }
  }
  out.at(n, y, x)[c] = from_f<T>(acc);
}

// bf16 fast path: one thread per (output pixel, 8 channels), 128-bit loads / stores; same tap order as the generic kernel
__global__ void k_deconv4x4s2_dw_bf16v(Ten<const bf16> in, const float* __restrict__ w, Ten<bf16> out, int groups) {
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)out.N * out.H * out.W * groups;
  if (gid >= total) return;
  const int g = (int)(gid % groups);
  long long p = gid / groups;
  const int x = (int)(p % out.W); p /= out.W;
  const int y = (int)(p % out.H);
  const int n = (int)(p / out.H);
  const int c0 = g * 8;
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  const int ky0 = (y + 1) & 1, kx0 = (x + 1) & 1;
  for (int a = 0; a < 2; ++a) {
    const int ky = ky0 + 2 * a;
    const int iy = (y + 1 - ky) / 2;
    if ((y + 1 - ky) < 0 || iy >= in.H) continue;
    for (int b = 0; b < 2; ++b) {
      const int kx = kx0 + 2 * b;
      const int ix = (x + 1 - kx) / 2;
      if ((x + 1 - kx) < 0 || ix >= in.W) continue;
      const uint4 v = *reinterpret_cast<const uint4*>(in.at(n, iy, ix) + c0);
      const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = c0 + j;
        if (c < in.C) {
          const float f = (j & 1) ? __uint_as_float(u[j >> 1] & 0xffff0000u) : __uint_as_float(u[j >> 1] << 16);
          acc[j] += f * w[c * 16 + ky * 4 + kx];
        }
      }
    }
  }
  uint32_t o[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const bf16 lo = __float2bfloat16_rn(acc[2 * j]), hi = __float2bfloat16_rn(acc[2 * j + 1]);
    o[j] = (uint32_t)(*reinterpret_cast<const uint16_t*>(&lo)) | ((uint32_t)(*reinterpret_cast<const uint16_t*>(&hi)) << 16);
  }
  *reinterpret_cast<uint4*>(out.at(n, y, x) + c0) = make_uint4(o[0], o[1], o[2], o[3]);
}

template <typename T> struct DeconvFast { static bool launch(Ten<const T>, const float*, Ten<T>, cudaStream_t) { return false; } };
template <> struct DeconvFast<bf16> {
  static bool launch(Ten<const bf16> in, const float* w, Ten<bf16> out, cudaStream_t s) {
    const bool ok = out.C % 8 == 0 && ((uintptr_t)in.p & 15) == 0 && ((uintptr_t)out.p & 15) == 0 && in.sW % 8 == 0 && out.sW % 8 == 0 &&
                    in.sH % 8 == 0 && out.sH % 8 == 0 && in.sN % 8 == 0 && out.sN % 8 == 0 && in.sW >= out.C;
    if (!ok) return false;
    const int groups = out.C / 8;
    const long long total = (long long)out.N * out.H * out.W * groups;
    DFVO_LAUNCH(k_deconv4x4s2_dw_bf16v, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, s, in, w, out, groups);
    return true;
  }
};

template <typename T>
int deconv4x4s2_dw(Ten<const T> in, const float* w, Ten<T> out, cudaStream_t s) {
  DFVO_REQUIRE(out.H == 2 * in.H && out.W == 2 * in.W && out.C <= 256, DFVO_ESHAPE, "deconv4x4s2 shape");
  if (DeconvFast<T>::launch(in, w, out, s)) {
    DFVO_CHECK_LAUNCH();
    return DFVO_OK;
  }
  int ppb = 256 / out.C;
  if (ppb < 1) ppb = 1;
  dim3 block(ppb * out.C), grid(cdiv(out.W, ppb), out.H, out.N);
  auto k = k_deconv4x4s2_dw<T>;
  DFVO_LAUNCH(k, grid, block, 0, s, in, w, out);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}
template int deconv4x4s2_dw<float>(Ten<const float>, const float*, Ten<float>, cudaStream_t);
template int deconv4x4s2_dw<bf16>(Ten<const bf16>, const float*, Ten<bf16>, cudaStream_t);

// ---------------------------------------------------------------------------------------------
// Backward warp: bilinear gather, zeros padding, pixel coords (x+fx*scale, y+fy*scale)
// (lite_flow_net.py:10-28 under the pinned align_corners=True semantics)
// ---------------------------------------------------------------------------------------------
struct Bil { int x0, y0; float w00, w01, w10, w11; };   // weights already zeroed when out of bounds

DFVO_D Bil bilinear_zeros(float px, float py, int W, int H) {
  Bil b;
  float fx0 = floorf(px), fy0 = floorf(py);
  b.x0 = (int)fx0; b.y0 = (int)fy0;
  float wx1 = px - fx0, wy1 = py - fy0, wx0 = 1.f - wx1, wy0 = 1.f - wy1;
  bool xin0 = b.x0 >= 0 && b.x0 <= W - 1, xin1 = b.x0 + 1 >= 0 && b.x0 + 1 <= W - 1;
  bool yin0 = b.y0 >= 0 && b.y0 <= H - 1, yin1 = b.y0 + 1 >= 0 && b.y0 + 1 <= H - 1;
  // non-finite coordinates sample nothing
  bool fin = (px == px) && (py == py) && fabsf(px) < 1e9f && fabsf(py) < 1e9f;
  b.w00 = (fin && xin0 && yin0) ? wx0 * wy0 : 0.f;
  b.w01 = (fin && xin1 && yin0) ? wx1 * wy0 : 0.f;
  b.w10 = (fin && xin0 && yin1) ? wx0 * wy1 : 0.f;
  b.w11 = (fin && xin1 && yin1) ? wx1 * wy1 : 0.f;
  if (!fin) { b.x0 = 0; b.y0 = 0; }
  return b;
}

template <typename T>
__global__ void k_warp_bilinear(Ten<const T> in, Ten<const float> flow, float scale, int nxor, Ten<T> out) {
  // one thread per (pixel, channel); channel fastest so neighbouring lanes read neighbouring bytes
  int C = out.C;
  long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long npix = (long long)out.N * out.H * out.W;
  if (gid >= npix * C) return;
  int c = (int)(gid % C);
  long long p = gid / C;
  int x = (int)(p % out.W);
  int y = (int)((p / out.W) % out.H);
  int n = (int)(p / ((long long)out.W * out.H));
  const float* f = flow.at(n, y, x);
  float px = (float)x + f[0] * scale, py = (float)y + f[1] * scale;
  Bil b = bilinear_zeros(px, py, in.W, in.H);
  float v = 0.f;
  const int ns = n ^ nxor;
  if (c < in.C) {
    if (b.w00 != 0.f) v += to_f(in.at(ns, b.y0, b.x0)[c]) * b.w00;
    if (b.w01 != 0.f) v += to_f(in.at(ns, b.y0, b.x0 + 1)[c]) * b.w01;
    if (b.w10 != 0.f) v += to_f(in.at(ns, b.y0 + 1, b.x0)[c]) * b.w10;
    if (b.w11 != 0.f) v += to_f(in.at(ns, b.y0 + 1, b.x0 + 1)[c]) * b.w11;
  }
  out.at(n, y, x)[c] = from_f<T>(v);
}

// vectorised variant: one thread per (pixel, 16-byte channel group); used when C and the strides allow it
template <typename T>
__global__ void k_warp_bilinear_vec(Ten<const T> in, Ten<const float> flow, float scale, int nxor, Ten<T> out) {
  constexpr int VEC = 16 / sizeof(T);
  const int groups = out.C / VEC;
  long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long npix = (long long)out.N * out.H * out.W;
  if (gid >= npix * groups) return;
  const int g = (int)(gid % groups);
  long long p = gid / groups;
  const int x = (int)(p % out.W), y = (int)((p / out.W) % out.H), n = (int)(p / ((long long)out.W * out.H));
  const float* f = flow.at(n, y, x);
  const float px = (float)x + f[0] * scale, py = (float)y + f[1] * scale;
  const Bil b = bilinear_zeros(px, py, in.W, in.H);
  const int ns = n ^ nxor;
  float acc[VEC];
#pragma unroll
  for (int j = 0; j < VEC; ++j) acc[j] = 0.f;
  const float wts[4] = {b.w00, b.w01, b.w10, b.w11};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (wts[k] == 0.f) continue;
    const T* src = in.at(ns, b.y0 + (k >> 1), b.x0 + (k & 1)) + g * VEC;
    const uint4 v = *reinterpret_cast<const uint4*>(src);
    const uint32_t w4[4] = {v.x, v.y, v.z, v.w};
    if (sizeof(T) == 4) {
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[j] += __uint_as_float(w4[j]) * wts[k];
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        acc[2 * j] += __uint_as_float(w4[j] << 16) * wts[k];
        acc[2 * j + 1] += __uint_as_float(w4[j] & 0xffff0000u) * wts[k];
      }
    }
  }
  uint32_t o4[4];
  if (sizeof(T) == 4) {
#pragma unroll
    for (int j = 0; j < 4; ++j) o4[j] = __float_as_uint(acc[j]);
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint32_t lo = __float_as_uint(to_f(from_f<T>(acc[2 * j]))) >> 16;
      const uint32_t hi = __float_as_uint(to_f(from_f<T>(acc[2 * j + 1]))) & 0xffff0000u;
      o4[j] = lo | hi;
    }
  }
  uint4 ov; ov.x = o4[0]; ov.y = o4[1]; ov.z = o4[2]; ov.w = o4[3];
  *reinterpret_cast<uint4*>(out.at(n, y, x) + g * VEC) = ov;
}

template <typename T>
int warp_bilinear(Ten<const T> in, Ten<const float> flow, float scale, int in_nxor, Ten<T> out, cudaStream_t s) {
  constexpr int VEC = 16 / sizeof(T);
  const bool vec_ok = out.C % VEC == 0 && in.C >= out.C && in.sW % VEC == 0 && in.sH % VEC == 0 && in.sN % VEC == 0 &&
                      out.sW % VEC == 0 && out.sH % VEC == 0 && out.sN % VEC == 0 &&
                      (reinterpret_cast<uintptr_t>(in.p) & 15) == 0 && (reinterpret_cast<uintptr_t>(out.p) & 15) == 0;
  if (vec_ok) {
    long long total = (long long)out.N * out.H * out.W * (out.C / VEC);
    auto k = k_warp_bilinear_vec<T>;
    DFVO_LAUNCH(k, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, s, in, flow, scale, in_nxor, out);
    DFVO_CHECK_LAUNCH();
    return DFVO_OK;
  }
  long long total = (long long)out.N * out.H * out.W * out.C;
  dim3 block(256), grid((unsigned)((total + 255) / 256));
  auto k = k_warp_bilinear<T>;
  DFVO_LAUNCH(k, grid, block, 0, s, in, flow, scale, in_nxor, out);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}
template int warp_bilinear<float>(Ten<const float>, Ten<const float>, float, int, Ten<float>, cudaStream_t);
template int warp_bilinear<bf16>(Ten<const bf16>, Ten<const float>, float, int, Ten<bf16>, cudaStream_t);

// ---------------------------------------------------------------------------------------------
// 49-channel correlation (correlation.py:38-106).  Output pixel (y,x) reads first at (y*s, x*s)
// and second at (y*s + dy*s, x*s + dx*s), dy,dx in [-3,3], zero outside; result / C; optional
// LeakyReLU(0.1) (lite_flow_net.py:145-149).  For s=2 only even pixels are ever touched.
// Tile: 32x4 output pixels per 128-thread block; the second feature map's (4+6)x(32+6) patch is
// staged in shared memory 16 words (16 floats / 32 bf16) of channels at a time with a 20-word
// pixel pitch (conflict-free 128-bit reads); each thread keeps its 49 accumulators in registers.
// ---------------------------------------------------------------------------------------------
#define CORR_TW 32
#define CORR_TH 4
#define CORR_PW (CORR_TW + 6)
#define CORR_PH (CORR_TH + 6)
#define CORR_PITCH 20

template <typename T> struct CorrVec;
template <> struct CorrVec<float> { enum { CK = 16 }; };
template <> struct CorrVec<bf16> { enum { CK = 32 }; };

DFVO_D void corr_unpack(const uint32_t* w, float* f, float) {
  for (int i = 0; i < 4; ++i) f[i] = __uint_as_float(w[i]);
}
DFVO_D int corr_unpack_n(float) { return 4; }
DFVO_D void corr_unpack8(const uint32_t* w, float* f) {     // 4 words of bf16x2 -> 8 floats
  for (int i = 0; i < 4; ++i) {
    f[2 * i] = __uint_as_float(w[i] << 16);
    f[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
  }
}

template <typename T>
__global__ void __launch_bounds__(CORR_TW* CORR_TH)
k_correlation49(Ten<const T> f1, Ten<const T> f2, int f2_nxor, int stride, int leaky, Ten<T> out) {
  constexpr int CK = CorrVec<T>::CK;          // channels per 16-word chunk
  constexpr int EPW = CK / 16;                // elements per 32-bit word (1 or 2)
  __shared__ __align__(16) uint32_t patch[CORR_PH * CORR_PW * CORR_PITCH];
  const int tx = threadIdx.x % CORR_TW, ty = threadIdx.x / CORR_TW;
  const int x0 = blockIdx.x * CORR_TW, y0 = blockIdx.y * CORR_TH, n = blockIdx.z;
  const int ox = x0 + tx, oy = y0 + ty;
  const bool active = ox < out.W && oy < out.H;
  const int C = f1.C;
  float acc[49];
#pragma unroll
  for (int i = 0; i < 49; ++i) acc[i] = 0.f;

  for (int c0 = 0; c0 < C; c0 += CK) {
    __syncthreads();
    // stage second-map patch: pixel (py,px) of the patch <-> source ((y0+py-3)*s, (x0+px-3)*s)
    for (int i = threadIdx.x; i < CORR_PH * CORR_PW * 4; i += blockDim.x) {
      int q = i & 3, pp = i >> 2;
      int px = pp % CORR_PW, py = pp / CORR_PW;
      int sy = (y0 + py - 3) * stride, sx = (x0 + px - 3) * stride;
      uint32_t wv[4] = {0u, 0u, 0u, 0u};
      if (sy >= 0 && sy < f2.H && sx >= 0 && sx < f2.W) {
        const T* src = f2.at(n ^ f2_nxor, sy, sx) + c0 + q * 4 * EPW;
        for (int j = 0; j < 4; ++j) {
          if (EPW == 1) {
            int c = c0 + q * 4 + j;
            wv[j] = (c < C) ? __float_as_uint(to_f(src[j])) : 0u;
          } else {
            int c = c0 + (q * 4 + j) * 2;
            uint32_t lo = 0u, hi = 0u;
            if (c < C) lo = __float_as_uint(to_f(src[2 * j])) >> 16;
            if (c + 1 < C) hi = __float_as_uint(to_f(src[2 * j + 1])) & 0xffff0000u;
            wv[j] = lo | hi;
          }
        }
      }
      uint32_t* dst = &patch[pp * CORR_PITCH + q * 4];
      dst[0] = wv[0]; dst[1] = wv[1]; dst[2] = wv[2]; dst[3] = wv[3];
    }
    __syncthreads();
    if (!active) continue;
    // this thread's first-map chunk
    float a[CK];
    {
      const T* src = f1.at(n, oy * stride, ox * stride) + c0;
      for (int j = 0; j < CK; ++j) a[j] = (c0 + j < C) ? to_f(src[j]) : 0.f;
    }
#pragma unroll
    for (int dy = 0; dy < 7; ++dy) {
#pragma unroll
      for (int dx = 0; dx < 7; ++dx) {
        const uint32_t* pw = &patch[((ty + dy) * CORR_PW + tx + dx) * CORR_PITCH];
        float sum = 0.f;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          uint32_t wv[4] = {pw[q * 4], pw[q * 4 + 1], pw[q * 4 + 2], pw[q * 4 + 3]};
          if (EPW == 1) {
            for (int j = 0; j < 4; ++j) sum += a[q * 4 + j] * __uint_as_float(wv[j]);
          } else {
            float b[8];
            corr_unpack8(wv, b);
            for (int j = 0; j < 8; ++j) sum += a[q * 8 + j] * b[j];
          }
        }
        acc[dy * 7 + dx] += sum;
      }
    }
  }
  if (!active) return;
  T* o = out.at(n, oy, ox);
  const float inv = 1.f / (float)C;
#pragma unroll
  for (int i = 0; i < 49; ++i) {
    float v = acc[i] * inv;
    if (leaky) v = v > 0.f ? v : 0.1f * v;
    o[i] = from_f<T>(v);
  }
  for (int i = 49; i < out.C; ++i) o[i] = from_f<T>(0.f);
}

// bf16 fast path (channel count a multiple of 32, 16-byte aligned pixels): 16x4 output pixels x 7 displacement rows per
// 448-thread block -- thread (pixel, dy) keeps 7 accumulators -- with 128-bit global loads for both operands.  Seven
// times the threads per pixel of the generic kernel and no scalar loads: the coarse pyramid levels (a dozen blocks) are
// latency-bound, so the work per thread is what sets their run time.  Same per-displacement summation order as the
// generic kernel (bit-identical results).
#define CORRV_TW 16
#define CORRV_TH 4
#define CORRV_PW (CORRV_TW + 6)
#define CORRV_PH (CORRV_TH + 6)
__global__ void __launch_bounds__(CORRV_TW* CORRV_TH * 7)
k_correlation49_bf16v(Ten<const bf16> f1, Ten<const bf16> f2, int f2_nxor, int stride, int leaky, Ten<bf16> out) {
  __shared__ __align__(16) uint32_t patch[CORRV_PH * CORRV_PW * CORR_PITCH];
  const int p = threadIdx.x % (CORRV_TW * CORRV_TH), dy = threadIdx.x / (CORRV_TW * CORRV_TH);
  const int tx = p % CORRV_TW, ty = p / CORRV_TW;
  const int x0 = blockIdx.x * CORRV_TW, y0 = blockIdx.y * CORRV_TH, n = blockIdx.z;
  const int ox = x0 + tx, oy = y0 + ty;
  const bool active = ox < out.W && oy < out.H;
  const int C = f1.C;
  float acc[7];
#pragma unroll
  for (int i = 0; i < 7; ++i) acc[i] = 0.f;
  for (int c0 = 0; c0 < C; c0 += 32) {
    __syncthreads();
    for (int i = threadIdx.x; i < CORRV_PH * CORRV_PW * 4; i += CORRV_TW * CORRV_TH * 7) {
      const int q = i & 3, pp = i >> 2;
      const int sy = (y0 + pp / CORRV_PW - 3) * stride, sx = (x0 + pp % CORRV_PW - 3) * stride;
      uint4 v; v.x = v.y = v.z = v.w = 0u;
      if (sy >= 0 && sy < f2.H && sx >= 0 && sx < f2.W) v = *reinterpret_cast<const uint4*>(f2.at(n ^ f2_nxor, sy, sx) + c0 + q * 8);
      *reinterpret_cast<uint4*>(&patch[pp * CORR_PITCH + q * 4]) = v;
    }
    __syncthreads();
    if (!active) continue;
    float a[32];
    {
      const bf16* src = f1.at(n, oy * stride, ox * stride) + c0;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const uint4 v = *reinterpret_cast<const uint4*>(src + q * 8);
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
        corr_unpack8(w, a + q * 8);
      }
    }
#pragma unroll
    for (int dx = 0; dx < 7; ++dx) {
      const uint32_t* pw = &patch[((ty + dy) * CORRV_PW + tx + dx) * CORR_PITCH];
      float sum = 0.f;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const uint4 v = *reinterpret_cast<const uint4*>(pw + q * 4);
        const uint32_t wv[4] = {v.x, v.y, v.z, v.w};
        float b[8];
        corr_unpack8(wv, b);
#pragma unroll
        for (int j = 0; j < 8; ++j) sum += a[q * 8 + j] * b[j];
      }
      acc[dx] += sum;
    }
  }
  if (!active) return;
  bf16* o = out.at(n, oy, ox) + dy * 7;
  const float inv = 1.f / (float)C;
#pragma unroll
  for (int i = 0; i < 7; ++i) {
    float v = acc[i] * inv;
    if (leaky) v = v > 0.f ? v : 0.1f * v;
    o[i] = __float2bfloat16_rn(v);
  }
  if (dy == 6) for (int i = 49; i < out.C; ++i) out.at(n, oy, ox)[i] = __float2bfloat16_rn(0.f);
}

template <typename T> struct CorrFast { static bool launch(Ten<const T>, Ten<const T>, int, int, int, Ten<T>, cudaStream_t) { return false; } };
template <> struct CorrFast<bf16> {
  static bool launch(Ten<const bf16> f1, Ten<const bf16> f2, int f2_nxor, int stride, int leaky, Ten<bf16> out, cudaStream_t s) {
    const bool ok = f1.C % 32 == 0 && ((uintptr_t)f1.p & 15) == 0 && ((uintptr_t)f2.p & 15) == 0 && f1.sW % 8 == 0 && f2.sW % 8 == 0 &&
                    f1.sH % 8 == 0 && f2.sH % 8 == 0 && f1.sN % 8 == 0 && f2.sN % 8 == 0;
    if (!ok) return false;
    dim3 block(CORRV_TW * CORRV_TH * 7), grid(cdiv(out.W, CORRV_TW), cdiv(out.H, CORRV_TH), out.N);
    DFVO_LAUNCH(k_correlation49_bf16v, grid, block, 0, s, f1, f2, f2_nxor, stride, leaky, out);
    return true;
  }
};

template <typename T>
int correlation49(Ten<const T> f1, Ten<const T> f2, int f2_nxor, int stride, int leaky, Ten<T> out, cudaStream_t s) {
  DFVO_REQUIRE(stride == 1 || stride == 2, DFVO_EINVAL, "correlation stride must be 1 or 2");
  DFVO_REQUIRE(out.H == (f1.H + stride - 1) / stride && out.W == (f1.W + stride - 1) / stride &&
                   out.C >= 49 && f1.C == f2.C && f1.H == f2.H && f1.W == f2.W,
               DFVO_ESHAPE, "correlation shapes");
  if (CorrFast<T>::launch(f1, f2, f2_nxor, stride, leaky, out, s)) {
    DFVO_CHECK_LAUNCH();
    return DFVO_OK;
  }
  dim3 block(CORR_TW * CORR_TH), grid(cdiv(out.W, CORR_TW), cdiv(out.H, CORR_TH), out.N);
  auto k = k_correlation49<T>;
  DFVO_LAUNCH(k, grid, block, 0, s, f1, f2, f2_nxor, stride, leaky, out);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}
template int correlation49<float>(Ten<const float>, Ten<const float>, int, int, int, Ten<float>, cudaStream_t);
template int correlation49<bf16>(Ten<const bf16>, Ten<const bf16>, int, int, int, Ten<bf16>, cudaStream_t);

// ---------------------------------------------------------------------------------------------
// 2-channel flow head: 32x8 output pixels per 256-thread block; the (8+k-1)x(32+k-1) input patch (32 bf16
// channels, 20-word pixel pitch = conflict-free 128-bit reads) and the k*k*32*2 fp32 weights live in shared memory.
// ---------------------------------------------------------------------------------------------
#define FH_TW 32
#define FH_TH 8
template <int K>
__global__ void __launch_bounds__(FH_TW* FH_TH)
k_flow_head(Ten<const bf16> in, const float* __restrict__ w, float b0, float b1, Ten<const float> res, int has_res, Ten<float> out) {
  constexpr int PW = FH_TW + K - 1, PH = FH_TH + K - 1, R = K / 2;
  DFVO_DYN_SMEM(uint32_t, smem);
  uint32_t* patch = smem;                                   // [PH*PW][20] words
  float* ws = reinterpret_cast<float*>(smem + PH * PW * 20);  // [K*K][32][2]
  const int tx = threadIdx.x % FH_TW, ty = threadIdx.x / FH_TW;
  const int x0 = blockIdx.x * FH_TW, y0 = blockIdx.y * FH_TH, n = blockIdx.z;
  for (int i = threadIdx.x; i < K * K * 64; i += FH_TW * FH_TH) ws[i] = w[i];
  for (int i = threadIdx.x; i < PH * PW * 4; i += FH_TW * FH_TH) {
    const int q = i & 3, pp = i >> 2;
    const int sx = x0 + pp % PW - R, sy = y0 + pp / PW - R;
    uint4 v; v.x = v.y = v.z = v.w = 0u;
    if (sx >= 0 && sx < in.W && sy >= 0 && sy < in.H) v = *reinterpret_cast<const uint4*>(in.at(n, sy, sx) + q * 8);
    uint32_t* d = patch + pp * 20 + q * 4;
    d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
  }
  __syncthreads();
  const int ox = x0 + tx, oy = y0 + ty;
  float a0 = 0.f, a1 = 0.f;
#pragma unroll 1
  for (int ky = 0; ky < K; ++ky) {
#pragma unroll
    for (int kx = 0; kx < K; ++kx) {
      const uint32_t* pw = patch + ((ty + ky) * PW + tx + kx) * 20;
      const float* wt = ws + (ky * K + kx) * 64;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const uint4 v = *reinterpret_cast<const uint4*>(pw + q * 4);
        const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float f0 = __uint_as_float(u[j] << 16), f1 = __uint_as_float(u[j] & 0xffff0000u);
          const float4 wv = *reinterpret_cast<const float4*>(wt + (q * 8 + 2 * j) * 2);   // (c,0) (c,1) (c+1,0) (c+1,1)
          a0 += f0 * wv.x + f1 * wv.z;
          a1 += f0 * wv.y + f1 * wv.w;
        }
      }
    }
  }
  if (ox >= out.W || oy >= out.H) return;
  float* o = out.at(n, oy, ox);
  float r0 = 0.f, r1 = 0.f;
  if (has_res) { const float* r = res.at(n, oy, ox); r0 = r[0]; r1 = r[1]; }
  o[0] = a0 + b0 + r0;
  o[1] = a1 + b1 + r1;
}


#ifndef DFVO_HOSTSIM
// Register-blocked variant for the device: a thread owns EIGHT output rows of one column, so an input pixel chunk is read from
// shared memory once per kx and feeds up to 7 x 8 (ky, output row) pairs, and a weight vector once per tap for eight outputs; the
// weights of the two output channels (w[c][0], w[c][1]) are adjacent in shared memory, so one 128-bit load feeds both channels'
// FMAs.  The first kernel above issues 20 LDS.128 per 64 FFMA (shared-memory bound); this one ~0.1 LDS per FMA.  Patch layout: [channel chunk q][row][pixel] x 16 B, so the lanes of a warp (consecutive pixels) read
// consecutive 16-byte words: conflict-free.  Block = 4 warps = 32 columns x 32 rows of outputs.
#define FH8_TW 32
#define FH8_RPT 8
#define FH8_WY 4
__device__ __forceinline__ void fh_ffma2(float2& acc, float f, float w0, float w1) {
  acc.x = fmaf(f, w0, acc.x);
  acc.y = fmaf(f, w1, acc.y);
}
template <int K>
__global__ void __launch_bounds__(32 * FH8_WY, 2)
k_flow_head8(Ten<const bf16> in, const float* __restrict__ w, float b0, float b1, Ten<const float> res, int has_res, Ten<float> out) {
  constexpr int TH = FH8_RPT * FH8_WY, PW = FH8_TW + K - 1, PH = TH + K - 1, R = K / 2, NI = FH8_RPT + K - 1;
  DFVO_DYN_SMEM(uint4, smem4);
  uint4* patch = smem4;                                                    // [4][PH][PW]
  float* ws = reinterpret_cast<float*>(smem4 + 4 * PH * PW);               // [K*K][32][2]
  const int tid = threadIdx.x, lane = tid & 31, wy = tid >> 5;
  const int x0 = blockIdx.x * FH8_TW, y0 = blockIdx.y * TH, n = blockIdx.z;
  for (int i = tid; i < K * K * 64; i += 32 * FH8_WY) ws[i] = w[i];
  for (int i = tid; i < PH * PW * 4; i += 32 * FH8_WY) {
    const int q = i & 3, pp = i >> 2;
    const int py = pp / PW, px = pp - py * PW;
    const int sx = x0 + px - R, sy = y0 + py - R;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (sx >= 0 && sx < in.W && sy >= 0 && sy < in.H) v = *reinterpret_cast<const uint4*>(in.at(n, sy, sx) + q * 8);
    patch[(q * PH + py) * PW + px] = v;
  }
  __syncthreads();
  float2 acc[FH8_RPT];
#pragma unroll
  for (int r = 0; r < FH8_RPT; ++r) acc[r] = make_float2(0.f, 0.f);
#pragma unroll 1
  for (int kx = 0; kx < K; ++kx) {
#pragma unroll 1
    for (int q = 0; q < 4; ++q) {
      const uint4* col = patch + (q * PH + wy * FH8_RPT) * PW + lane + kx;
#pragma unroll
      for (int half = 0; half < 2; ++half) {                               // four channels at a time: 4 x NI unpacked floats live
        float f[NI][4];
#pragma unroll
        for (int i = 0; i < NI; ++i) {
          const uint4 v = col[i * PW];
          const uint32_t u0 = half ? v.z : v.x, u1 = half ? v.w : v.y;
          f[i][0] = __uint_as_float(u0 << 16); f[i][1] = __uint_as_float(u0 & 0xffff0000u);
          f[i][2] = __uint_as_float(u1 << 16); f[i][3] = __uint_as_float(u1 & 0xffff0000u);
        }
#pragma unroll
        for (int ky = 0; ky < K; ++ky) {
          // channels q*8 + half*4 + {0..3}: (c,0) (c,1) pairs = 8 floats = 2 x 128-bit loads (broadcast)
          const float4* wp = reinterpret_cast<const float4*>(ws + (ky * K + kx) * 64 + (q * 8 + half * 4) * 2);
          const float4 w01 = wp[0], w23 = wp[1];
#pragma unroll
          for (int r = 0; r < FH8_RPT; ++r) {
            fh_ffma2(acc[r], f[r + ky][0], w01.x, w01.y);
            fh_ffma2(acc[r], f[r + ky][1], w01.z, w01.w);
            fh_ffma2(acc[r], f[r + ky][2], w23.x, w23.y);
            fh_ffma2(acc[r], f[r + ky][3], w23.z, w23.w);
          }
        }
      }
    }
  }
  const int ox = x0 + lane;
  if (ox >= out.W) return;
#pragma unroll
  for (int r = 0; r < FH8_RPT; ++r) {
    const int oy = y0 + wy * FH8_RPT + r;
    if (oy >= out.H) break;
    const float a0 = acc[r].x, a1 = acc[r].y;
    float r0 = 0.f, r1 = 0.f;
    if (has_res) { const float* rr = res.at(n, oy, ox); r0 = rr[0]; r1 = rr[1]; }
    float* o = out.at(n, oy, ox);
    o[0] = a0 + b0 + r0;
    o[1] = a1 + b1 + r1;
  }
}
#endif

int flow_head(Ten<const bf16> in, const float* w, float bias0, float bias1, int k, Ten<const float> residual, Ten<float> out,
              cudaStream_t s) {
  DFVO_REQUIRE(in.C == 32 && (k == 3 || k == 5 || k == 7) && in.H == out.H && in.W == out.W && in.sW % 8 == 0 &&
                   (reinterpret_cast<uintptr_t>(in.p) & 15) == 0, DFVO_ESHAPE, "flow_head shapes");
  const float hb[2] = {bias0, bias1};
  const int has_res = residual.p != nullptr;
#ifndef DFVO_HOSTSIM
  {
    // big maps: the register-blocked kernel (DFVO_FLOW_HEAD8=0 keeps the first one; small maps stay on it -- fewer, fuller blocks).
    // The choice depends on the size of ONE image, not on the batch: a pair gives the same bits alone and inside a batch.
    static int use8 = -1;
    if (use8 < 0) { const char* e = getenv("DFVO_FLOW_HEAD8"); use8 = !(e && atoi(e) == 0); }
    if (use8 && (long long)out.H * out.W >= 20000) {
      static bool attr8 = false;
      if (!attr8) {
        cudaFuncSetAttribute(k_flow_head8<7>, cudaFuncAttributeMaxDynamicSharedMemorySize, 112 * 1024);
        cudaFuncSetAttribute(k_flow_head8<5>, cudaFuncAttributeMaxDynamicSharedMemorySize, 112 * 1024);
        cudaFuncSetAttribute(k_flow_head8<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, 112 * 1024);
        attr8 = true;
      }
      const int TH = FH8_RPT * FH8_WY;
      dim3 grid8(cdiv(out.W, FH8_TW), cdiv(out.H, TH), out.N), block8(32 * FH8_WY);
      const size_t smem8 = (size_t)4 * (TH + k - 1) * (FH8_TW + k - 1) * 16 + (size_t)k * k * 64 * 4;
      if (k == 7) { auto kn = k_flow_head8<7>; DFVO_LAUNCH(kn, grid8, block8, smem8, s, in, w, hb[0], hb[1], residual, has_res, out); }
      else if (k == 5) { auto kn = k_flow_head8<5>; DFVO_LAUNCH(kn, grid8, block8, smem8, s, in, w, hb[0], hb[1], residual, has_res, out); }
      else { auto kn = k_flow_head8<3>; DFVO_LAUNCH(kn, grid8, block8, smem8, s, in, w, hb[0], hb[1], residual, has_res, out); }
      DFVO_CHECK_LAUNCH();
      return DFVO_OK;
    }
  }
#endif
  dim3 grid(cdiv(out.W, FH_TW), cdiv(out.H, FH_TH), out.N), block(FH_TW * FH_TH);
  const size_t smem = ((size_t)(FH_TH + k - 1) * (FH_TW + k - 1) * 20 + (size_t)k * k * 64) * 4;
#ifndef DFVO_HOSTSIM
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(k_flow_head<7>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024);
    cudaFuncSetAttribute(k_flow_head<5>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024);
    cudaFuncSetAttribute(k_flow_head<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024);
    attr = true;
  }
#endif
  if (k == 7) { auto kn = k_flow_head<7>; DFVO_LAUNCH(kn, grid, block, smem, s, in, w, hb[0], hb[1], residual, has_res, out); }
  else if (k == 5) { auto kn = k_flow_head<5>; DFVO_LAUNCH(kn, grid, block, smem, s, in, w, hb[0], hb[1], residual, has_res, out); }
  else { auto kn = k_flow_head<3>; DFVO_LAUNCH(kn, grid, block, smem, s, in, w, hb[0], hb[1], residual, has_res, out); }
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

// ---------------------------------------------------------------------------------------------
// flow mean (lite_flow_net.py:257: tensorFlow.view(N,2,-1).mean(2))  -- one block per n
// ---------------------------------------------------------------------------------------------
#define FM_BLOCKS 64
__global__ void k_flow_mean_partial(Ten<const float> flow, double* __restrict__ partial) {
  __shared__ double sx[256], sy[256];
  const int n = blockIdx.y;
  const int npix = flow.H * flow.W;
  double ax = 0.0, ay = 0.0;
  for (int p = blockIdx.x * 256 + threadIdx.x; p < npix; p += FM_BLOCKS * 256) {
    const float* f = flow.at(n, p / flow.W, p % flow.W);
    ax += (double)f[0]; ay += (double)f[1];
  }
  sx[threadIdx.x] = ax; sy[threadIdx.x] = ay;
  __syncthreads();
  for (int off = 128; off > 0; off >>= 1) {
    if ((int)threadIdx.x < off) { sx[threadIdx.x] += sx[threadIdx.x + off]; sy[threadIdx.x] += sy[threadIdx.x + off]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) { partial[(n * FM_BLOCKS + blockIdx.x) * 2] = sx[0]; partial[(n * FM_BLOCKS + blockIdx.x) * 2 + 1] = sy[0]; }
}

__global__ void k_flow_mean_final(const double* __restrict__ partial, int npix, float* __restrict__ mean) {
  const int n = blockIdx.x;
  if (threadIdx.x < 2) {
    double a = 0.0;
    for (int b = 0; b < FM_BLOCKS; ++b) a += partial[(n * FM_BLOCKS + b) * 2 + threadIdx.x];     // fixed order: deterministic
    mean[n * 2 + threadIdx.x] = (float)(a / (double)npix);
  }
}

int flow_mean(Ten<const float> flow, float* mean, cudaStream_t s) {
  // the partial sums live behind the means: caller's buffer holds [N*2 floats | pad | N*FM_BLOCKS*2 doubles]
  double* partial = reinterpret_cast<double*>(mean + ((flow.N * 2 + 3) & ~3));
  DFVO_LAUNCH(k_flow_mean_partial, dim3(FM_BLOCKS, flow.N), dim3(256), 0, s, flow, partial);
  DFVO_LAUNCH(k_flow_mean_final, dim3(flow.N), dim3(32), 0, s, (const double*)partial, flow.H * flow.W, mean);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

// ---------------------------------------------------------------------------------------------
// Regularization prep (lite_flow_net.py:244-257)
// ---------------------------------------------------------------------------------------------
template <typename T>
__global__ void k_reg_prep(Ten<const float> img1, Ten<const float> img2, int nxor, Ten<const float> flow,
                           const float* __restrict__ mean, float scale, Ten<T> out) {
  int x = blockIdx.x * blockDim.x + threadIdx.x;
  int y = blockIdx.y, n = blockIdx.z;
  if (x >= out.W) return;
  const float* f = flow.at(n, y, x);
  float px = (float)x + f[0] * scale, py = (float)y + f[1] * scale;
  Bil b = bilinear_zeros(px, py, img2.W, img2.H);
  const float* a = img1.at(n, y, x);
  float ss = 0.f;
  for (int c = 0; c < 3; ++c) {
    float v = 0.f;
    if (b.w00 != 0.f) v += img2.at(n ^ nxor, b.y0, b.x0)[c] * b.w00;
    if (b.w01 != 0.f) v += img2.at(n ^ nxor, b.y0, b.x0 + 1)[c] * b.w01;
    if (b.w10 != 0.f) v += img2.at(n ^ nxor, b.y0 + 1, b.x0)[c] * b.w10;
    if (b.w11 != 0.f) v += img2.at(n ^ nxor, b.y0 + 1, b.x0 + 1)[c] * b.w11;
    float d = a[c] - v;
    ss += d * d;
  }
  T* o = out.at(n, y, x);
  o[0] = from_f<T>(sqrtf(ss + 1e-6f));
  o[1] = from_f<T>(f[0] - mean[n * 2 + 0]);
  o[2] = from_f<T>(f[1] - mean[n * 2 + 1]);
  for (int c = 3; c < out.C; ++c) o[c] = from_f<T>(0.f);
}

template <typename T>
int reg_prep(Ten<const float> img1, Ten<const float> img2, int img2_nxor, Ten<const float> flow, const float* mean,
             float scale, Ten<T> out, cudaStream_t s) {
  dim3 block(128), grid(cdiv(out.W, 128), out.H, out.N);
  auto k = k_reg_prep<T>;
  DFVO_LAUNCH(k, grid, block, 0, s, img1, img2, img2_nxor, flow, mean, scale, out);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}
template int reg_prep<float>(Ten<const float>, Ten<const float>, int, Ten<const float>, const float*, float, Ten<float>, cudaStream_t);
template int reg_prep<bf16>(Ten<const float>, Ten<const float>, int, Ten<const float>, const float*, float, Ten<bf16>, cudaStream_t);

// ---------------------------------------------------------------------------------------------
// Regularization tail (lite_flow_net.py:258-264).  dist channel j <-> unfold offset
// (j / k - k/2, j % k - k/2) (torch.nn.functional.unfold ordering), zero padding.
// ---------------------------------------------------------------------------------------------
template <typename T>
__global__ void k_reg_tail(Ten<const T> dist, Ten<const float> flow, int k, const float* __restrict__ wx,
                           const float* __restrict__ wy, float bx, float by, Ten<float> out) {
  int x = blockIdx.x * blockDim.x + threadIdx.x;
  int y = blockIdx.y, n = blockIdx.z;
  if (x >= out.W) return;
  const int cd = k * k, r = k / 2;
  const T* d = dist.at(n, y, x);
  float m = -3.4e38f;
  for (int j = 0; j < cd; ++j) {
    float v = to_f(d[j]);
    float nv = -(v * v);
    m = nv > m ? nv : m;
  }
  float se = 0.f, ax = 0.f, ay = 0.f;
  for (int j = 0; j < cd; ++j) {
    float v = to_f(d[j]);
    float e = expf(-(v * v) - m);
    se += e;
    int yy = y + j / k - r, xx = x + j % k - r;
    if (yy >= 0 && yy < flow.H && xx >= 0 && xx < flow.W) {
      const float* f = flow.at(n, yy, xx);
      ax += wx[j] * (e * f[0]);
      ay += wy[j] * (e * f[1]);
    }
  }
  float inv = 1.f / se;
  float* o = out.at(n, y, x);
  o[0] = (ax + bx) * inv;
  o[1] = (ay + by) * inv;
}

// bf16 fast path: the k*k distances of a pixel are fetched once with 128-bit loads and kept in registers for both passes
template <int K>
__global__ void __launch_bounds__(128)
k_reg_tail_bf16v(Ten<const bf16> dist, Ten<const float> flow, const float* __restrict__ wx, const float* __restrict__ wy, float bx,
                 float by, Ten<float> out) {
  constexpr int CD = K * K, NV = (CD + 7) / 8, R = K / 2;
  int x = blockIdx.x * blockDim.x + threadIdx.x;
  int y = blockIdx.y, n = blockIdx.z;
  if (x >= out.W) return;
  const bf16* d = dist.at(n, y, x);
  float v[NV * 8];
#pragma unroll
  for (int q = 0; q < NV; ++q) {
    const uint4 u4 = *reinterpret_cast<const uint4*>(d + q * 8);
    const uint32_t u[4] = {u4.x, u4.y, u4.z, u4.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) { v[q * 8 + 2 * j] = __uint_as_float(u[j] << 16); v[q * 8 + 2 * j + 1] = __uint_as_float(u[j] & 0xffff0000u); }
  }
  float m = -3.4e38f;
#pragma unroll
  for (int j = 0; j < CD; ++j) {
    const float nv = -(v[j] * v[j]);
    m = nv > m ? nv : m;
  }
  float se = 0.f, ax = 0.f, ay = 0.f;
#pragma unroll
  for (int j = 0; j < CD; ++j) {
    const float e = expf(-(v[j] * v[j]) - m);
    se += e;
    const int yy = y + j / K - R, xx = x + j % K - R;
    if (yy >= 0 && yy < flow.H && xx >= 0 && xx < flow.W) {
      const float* f = flow.at(n, yy, xx);
      ax += wx[j] * (e * f[0]);
      ay += wy[j] * (e * f[1]);
    }
  }
  const float inv = 1.f / se;
  float* o = out.at(n, y, x);
  o[0] = (ax + bx) * inv;
  o[1] = (ay + by) * inv;
}

template <typename T> struct RegTailFast {
  static bool launch(Ten<const T>, Ten<const float>, int, const float*, const float*, float, float, Ten<float>, cudaStream_t) { return false; }
};
template <> struct RegTailFast<bf16> {
  static bool launch(Ten<const bf16> dist, Ten<const float> flow, int k, const float* wx, const float* wy, float bx, float by,
                     Ten<float> out, cudaStream_t s) {
    const int nv8 = (k * k + 7) / 8 * 8;
    const bool ok = (k == 3 || k == 5 || k == 7) && ((uintptr_t)dist.p & 15) == 0 && dist.sW % 8 == 0 && dist.sH % 8 == 0 && dist.sN % 8 == 0 &&
                    dist.sW >= nv8 && flow.sW == 2 && ((uintptr_t)flow.p & 7) == 0;
    if (!ok) return false;
    dim3 block(128), grid(cdiv(out.W, 128), out.H, out.N);
    if (k == 3) DFVO_LAUNCH(k_reg_tail_bf16v<3>, grid, block, 0, s, dist, flow, wx, wy, bx, by, out);
    else if (k == 5) DFVO_LAUNCH(k_reg_tail_bf16v<5>, grid, block, 0, s, dist, flow, wx, wy, bx, by, out);
    else DFVO_LAUNCH(k_reg_tail_bf16v<7>, grid, block, 0, s, dist, flow, wx, wy, bx, by, out);
    return true;
  }
};

template <typename T>
int reg_tail(Ten<const T> dist, Ten<const float> flow, int k, const float* wx, const float* wy, float bx,
             float by, Ten<float> out, cudaStream_t s) {
  if (RegTailFast<T>::launch(dist, flow, k, wx, wy, bx, by, out, s)) {
    DFVO_CHECK_LAUNCH();
    return DFVO_OK;
  }
  dim3 block(128), grid(cdiv(out.W, 128), out.H, out.N);
  auto kk = k_reg_tail<T>;
  DFVO_LAUNCH(kk, grid, block, 0, s, dist, flow, k, wx, wy, bx, by, out);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}
template int reg_tail<float>(Ten<const float>, Ten<const float>, int, const float*, const float*, float, float, Ten<float>, cudaStream_t);
template int reg_tail<bf16>(Ten<const bf16>, Ten<const float>, int, const float*, const float*, float, float, Ten<float>, cudaStream_t);

// ---------------------------------------------------------------------------------------------
// flows[1]*mul -> bilinear(AC=True) to HxW -> *(W/w, H/h)   (lite_flow_net.py:322-324, deep_flow.py:107-129)
// ---------------------------------------------------------------------------------------------
__global__ void k_flow_upsample_final(Ten<const float> flow, float mul, int H, int W, float rw, float rh,
                                      float* __restrict__ out) {
  int x = blockIdx.x * blockDim.x + threadIdx.x;
  int y = blockIdx.y, n = blockIdx.z;
  if (x >= W) return;
  Lerp ly = lerp_coord(y, flow.H, H, 1), lx = lerp_coord(x, flow.W, W, 1);
  const float* p00 = flow.at(n, ly.i0, lx.i0);
  const float* p01 = flow.at(n, ly.i0, lx.i1);
  const float* p10 = flow.at(n, ly.i1, lx.i0);
  const float* p11 = flow.at(n, ly.i1, lx.i1);
  for (int c = 0; c < 2; ++c) {
    float v = ly.l0 * (lx.l0 * (p00[c] * mul) + lx.l1 * (p01[c] * mul)) +
              ly.l1 * (lx.l0 * (p10[c] * mul) + lx.l1 * (p11[c] * mul));
    out[(((size_t)n * 2 + c) * H + y) * W + x] = v * (c == 0 ? rw : rh);
  }
}

int flow_upsample_final(Ten<const float> flow, float mul, int H, int W, float* out, cudaStream_t s) {
  float rw = (float)((double)W / (double)flow.W), rh = (float)((double)H / (double)flow.H);
  dim3 block(128), grid(cdiv(W, 128), H, flow.N);
  DFVO_LAUNCH(k_flow_upsample_final, grid, block, 0, s, flow, mul, H, W, rw, rh, out);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

// ---------------------------------------------------------------------------------------------
// forward-backward consistency (layers.py:213-229 FlowToPix normalisation, deep_flow.py:171-196).
// Keeps the reference's normalise -> un-normalise arithmetic so coordinates round the same way.
// ---------------------------------------------------------------------------------------------
__global__ void k_fb_consistency(const float* __restrict__ fwd, const float* __restrict__ bwd, int H, int W,
                                 float* __restrict__ diff, long long pair_stride) {
  int x = blockIdx.x * blockDim.x + threadIdx.x;
  int y = blockIdx.y;
  if (x >= W) return;
  size_t hw = (size_t)H * W, i = (size_t)y * W + x;
  fwd += blockIdx.z * pair_stride; bwd += blockIdx.z * pair_stride; diff += blockIdx.z * hw;
  float fx = fwd[i], fy = fwd[hw + i];
  float gx = (((float)x + fx) / (float)(W - 1) - 0.5f) * 2.f;
  float gy = (((float)y + fy) / (float)(H - 1) - 0.5f) * 2.f;
  float px = ((gx + 1.f) / 2.f) * (float)(W - 1);
  float py = ((gy + 1.f) / 2.f) * (float)(H - 1);
  Bil b = bilinear_zeros(px, py, W, H);
  float wx = 0.f, wy = 0.f;
  if (b.w00 != 0.f) { size_t j = (size_t)b.y0 * W + b.x0; wx += -bwd[j] * b.w00; wy += -bwd[hw + j] * b.w00; }
  if (b.w01 != 0.f) { size_t j = (size_t)b.y0 * W + b.x0 + 1; wx += -bwd[j] * b.w01; wy += -bwd[hw + j] * b.w01; }
  if (b.w10 != 0.f) { size_t j = (size_t)(b.y0 + 1) * W + b.x0; wx += -bwd[j] * b.w10; wy += -bwd[hw + j] * b.w10; }
  if (b.w11 != 0.f) { size_t j = (size_t)(b.y0 + 1) * W + b.x0 + 1; wx += -bwd[j] * b.w11; wy += -bwd[hw + j] * b.w11; }
  float dx = fx - wx, dy = fy - wy;
  diff[i] = sqrtf(dx * dx + dy * dy);
}

// n pairs in one launch: pair p reads fwd + p * pair_stride, bwd + p * pair_stride ([2,H,W] planes each), writes diff + p * H * W
int fb_consistency(const float* fwd, const float* bwd, int H, int W, float* diff, cudaStream_t s, int n, long long pair_stride) {
  dim3 block(128), grid(cdiv(W, 128), H, n);
  DFVO_LAUNCH(k_fb_consistency, grid, block, 0, s, fwd, bwd, H, W, diff, pair_stride);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

// ---------------------------------------------------------------------------------------------
// layout / dtype helpers
// ---------------------------------------------------------------------------------------------
template <typename TI, typename TO>
__global__ void k_convert_copy(Ten<const TI> in, Ten<TO> out) {
  long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long total = (long long)out.N * out.H * out.W * out.C;
  if (gid >= total) return;
  int c = (int)(gid % out.C);
  long long p = gid / out.C;
  int x = (int)(p % out.W), y = (int)((p / out.W) % out.H), n = (int)(p / ((long long)out.W * out.H));
  float v = c < in.C ? to_f(in.at(n, y, x)[c]) : 0.f;
  out.at(n, y, x)[c] = from_f<TO>(v);
}

template <typename TI, typename TO>
int convert_copy(Ten<const TI> in, Ten<TO> out, cudaStream_t s) {
  long long total = (long long)out.N * out.H * out.W * out.C;
  auto k = k_convert_copy<TI, TO>;
  DFVO_LAUNCH(k, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, s, in, out);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}
template int convert_copy<float, bf16>(Ten<const float>, Ten<bf16>, cudaStream_t);
template int convert_copy<bf16, float>(Ten<const bf16>, Ten<float>, cudaStream_t);
template int convert_copy<float, float>(Ten<const float>, Ten<float>, cudaStream_t);
template int convert_copy<bf16, bf16>(Ten<const bf16>, Ten<bf16>, cudaStream_t);

__global__ void k_nchw_to_nhwc_f32(const float* __restrict__ in, int C, Ten<float> out) {
  long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long total = (long long)out.N * out.H * out.W * out.C;
  if (gid >= total) return;
  int c = (int)(gid % out.C);
  long long p = gid / out.C;
  int x = (int)(p % out.W), y = (int)((p / out.W) % out.H), n = (int)(p / ((long long)out.W * out.H));
  out.at(n, y, x)[c] = c < C ? in[(((size_t)n * C + c) * out.H + y) * out.W + x] : 0.f;
}

int nchw_to_nhwc_f32(const float* in, int N, int C, int H, int W, Ten<float> out, cudaStream_t s) {
  long long total = (long long)N * H * W * out.C;
  DFVO_LAUNCH(k_nchw_to_nhwc_f32, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, s, in, C, out);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

template <typename T>
__global__ void k_nhwc_to_nchw(Ten<const T> in, float* __restrict__ out) {
  long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long total = (long long)in.N * in.H * in.W * in.C;
  if (gid >= total) return;
  int x = (int)(gid % in.W);
  long long r = gid / in.W;
  int y = (int)(r % in.H); r /= in.H;
  int c = (int)(r % in.C);
  int n = (int)(r / in.C);
  out[gid] = to_f(in.at(n, y, x)[c]);
}

template <typename T>
int nhwc_to_nchw(Ten<const T> in, float* out, cudaStream_t s) {
  long long total = (long long)in.N * in.H * in.W * in.C;
  auto k = k_nhwc_to_nchw<T>;
  DFVO_LAUNCH(k, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, s, in, out);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}
template int nhwc_to_nchw<float>(Ten<const float>, float*, cudaStream_t);
template int nhwc_to_nchw<bf16>(Ten<const bf16>, float*, cudaStream_t);

}  // namespace dfvo
