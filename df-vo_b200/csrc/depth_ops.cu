// Small kernels of the monodepth2 path: input normalisation, ResNet max-pool, decoder
// upsample+concat+reflection-pad, disparity->depth, and the depth post-processing of dfvo.py:314-319.
#include "ops.h"

namespace dfvo {

template <typename T>
__global__ void k_normalize_nchw_to_nhwc(const float* __restrict__ in, int C, float mean, float inv_std_is_div, Ten<T> out) {
  long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long total = (long long)out.N * out.H * out.W * out.C;
  if (gid >= total) return;
  int c = (int)(gid % out.C);
  long long p = gid / out.C;
  int x = (int)(p % out.W), y = (int)((p / out.W) % out.H), n = (int)(p / ((long long)out.W * out.H));
  float v = 0.f;
  if (c < C) v = (in[(((size_t)n * C + c) * out.H + y) * out.W + x] - mean) / inv_std_is_div;   // (x - 0.45) / 0.225
  out.at(n, y, x)[c] = from_f<T>(v);
}

template <typename T>
int normalize_nchw_to_nhwc(const float* in, int N, int C, int H, int W, float mean, float std, Ten<T> out, cudaStream_t s) {
  long long total = (long long)N * H * W * out.C;
  auto k = k_normalize_nchw_to_nhwc<T>;
  DFVO_LAUNCH(k, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, s, in, C, mean, std, out);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}
template int normalize_nchw_to_nhwc<float>(const float*, int, int, int, int, float, float, Ten<float>, cudaStream_t);
template int normalize_nchw_to_nhwc<bf16>(const float*, int, int, int, int, float, float, Ten<bf16>, cudaStream_t);

template <typename T>
__global__ void k_maxpool3x3s2(Ten<const T> in, Ten<T> out) {
  long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long total = (long long)out.N * out.H * out.W * out.C;
  if (gid >= total) return;
  int c = (int)(gid % out.C);
  long long p = gid / out.C;
  int x = (int)(p % out.W), y = (int)((p / out.W) % out.H), n = (int)(p / ((long long)out.W * out.H));
  float m = -3.4e38f;
  for (int dy = -1; dy <= 1; ++dy)
    for (int dx = -1; dx <= 1; ++dx) {
      int iy = 2 * y + dy, ix = 2 * x + dx;
      if (iy < 0 || iy >= in.H || ix < 0 || ix >= in.W) continue;
      float v = to_f(in.at(n, iy, ix)[c]);
      m = v > m ? v : m;
    }
  out.at(n, y, x)[c] = from_f<T>(m);
}

template <typename T>
int maxpool3x3s2(Ten<const T> in, Ten<T> out, cudaStream_t s) {
  DFVO_REQUIRE(out.H == (in.H + 2 - 3) / 2 + 1 && out.W == (in.W + 2 - 3) / 2 + 1 && out.C == in.C, DFVO_ESHAPE, "maxpool shape");
  long long total = (long long)out.N * out.H * out.W * out.C;
  auto k = k_maxpool3x3s2<T>;
  DFVO_LAUNCH(k, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, s, in, out);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}
template int maxpool3x3s2<float>(Ten<const float>, Ten<float>, cudaStream_t);
template int maxpool3x3s2<bf16>(Ten<const bf16>, Ten<bf16>, cudaStream_t);

template <typename T>
__global__ void k_upcat_reflect(Ten<const T> lo, int up, Ten<const T> skip, int has_skip, Ten<T> out) {
  long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long total = (long long)out.N * out.H * out.W * out.C;
  if (gid >= total) return;
  int c = (int)(gid % out.C);
  long long p = gid / out.C;
  int x = (int)(p % out.W), y = (int)((p / out.W) % out.H), n = (int)(p / ((long long)out.W * out.H));
  const int h = out.H - 2, w = out.W - 2;            // un-padded size
  int yy = y - 1, xx = x - 1;
  if (yy < 0) yy = -yy;
  if (yy >= h) yy = 2 * (h - 1) - yy;
  if (xx < 0) xx = -xx;
  if (xx >= w) xx = 2 * (w - 1) - xx;
  float v = 0.f;
  if (c < lo.C) v = to_f(lo.at(n, yy / up, xx / up)[c]);
  else if (has_skip && c - lo.C < skip.C) v = to_f(skip.at(n, yy, xx)[c - lo.C]);
  out.at(n, y, x)[c] = from_f<T>(v);
}

template <typename T>
int upcat_reflect(Ten<const T> lo, int up, Ten<const T> skip, Ten<T> out, cudaStream_t s) {
  const int has_skip = skip.p != nullptr;
  DFVO_REQUIRE((up == 1 || up == 2) && out.H == lo.H * up + 2 && out.W == lo.W * up + 2 &&
                   out.C >= lo.C + (has_skip ? skip.C : 0) && (!has_skip || (skip.H == lo.H * up && skip.W == lo.W * up)),
               DFVO_ESHAPE, "upcat_reflect shapes");
  long long total = (long long)out.N * out.H * out.W * out.C;
  auto k = k_upcat_reflect<T>;
  DFVO_LAUNCH(k, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, s, lo, up, skip, has_skip, out);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}
template int upcat_reflect<float>(Ten<const float>, int, Ten<const float>, Ten<float>, cudaStream_t);
template int upcat_reflect<bf16>(Ten<const bf16>, int, Ten<const bf16>, Ten<bf16>, cudaStream_t);

__global__ void k_disp_to_depth(const float* __restrict__ disp, int n, float min_disp, float max_disp, float baseline,
                                float* __restrict__ depth) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float scaled = min_disp + (max_disp - min_disp) * disp[i];      // layers.py:21-24
  depth[i] = (1.f / scaled) * baseline;                           // monodepth2.py:115,138
}

int disp_to_depth(const float* disp, int n, float min_depth, float max_depth, float baseline, float* depth, cudaStream_t s) {
  DFVO_LAUNCH(k_disp_to_depth, dim3(cdiv(n, 256)), dim3(256), 0, s, disp, n, 1.f / max_depth, 1.f / min_depth, baseline, depth);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

// PoseDecoder.forward after net.3 (pose_decoder.py: out.mean(3).mean(2), 0.01 * view(-1, 2, 1, 6), frame 0), then
// transformation_from_parameters(axisangle, translation, invert=True) (layers.py:28-94) and pose[:, :3, 3] *= baseline
// (monodepth2.py:117-118), all in float32 in the torch operation order.  One block: thread (c, y) averages row y of channel c
// over x, then thread c averages its rows, then thread 0 builds the matrix.
#define POSE_HEAD_MAXH 64
__global__ void k_pose_head(const float* __restrict__ out12, int h, int w, int pitch, float baseline, float* __restrict__ pose) {
  __shared__ float rowmean[6 * POSE_HEAD_MAXH];
  __shared__ float p6[6];
  for (int t = threadIdx.x; t < 6 * h; t += blockDim.x) {
    const int c = t / h, y = t - c * h;
    float s = 0.f;
    for (int x = 0; x < w; ++x) s += out12[((size_t)y * w + x) * pitch + c];
    rowmean[t] = s / (float)w;
  }
  __syncthreads();
  if (threadIdx.x < 6) {
    float s = 0.f;
    for (int y = 0; y < h; ++y) s += rowmean[threadIdx.x * h + y];
    p6[threadIdx.x] = 0.01f * (s / (float)h);
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  // rot_from_axisangle (layers.py:63-94)
  const float vx = p6[0], vy = p6[1], vz = p6[2];
  const float angle = sqrtf(vx * vx + vy * vy + vz * vz);
  const float x = vx / (angle + 1e-7f), y = vy / (angle + 1e-7f), z = vz / (angle + 1e-7f);
  const float ca = cosf(angle), sa = sinf(angle), C = 1.f - ca;
  const float xs = x * sa, ys = y * sa, zs = z * sa;
  const float xC = x * C, yC = y * C, zC = z * C;
  const float xyC = x * yC, yzC = y * zC, zxC = z * xC;
  const float R[3][3] = {{x * xC + ca, xyC - zs, zxC + ys}, {xyC + zs, y * yC + ca, yzC - xs}, {zxC - ys, yzC + xs, z * zC + ca}};
  // invert: M = R^T @ translation(-t)
  const float t[3] = {-p6[3], -p6[4], -p6[5]};
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) pose[4 * i + j] = R[j][i];
    pose[4 * i + 3] = (R[0][i] * t[0] + R[1][i] * t[1] + R[2][i] * t[2]) * baseline;
  }
  pose[12] = 0.f; pose[13] = 0.f; pose[14] = 0.f; pose[15] = 1.f;
}

int pose_head(const float* out12, int h, int w, int pitch, float baseline_multiplier, float* pose_out, cudaStream_t s) {
  DFVO_REQUIRE(h >= 1 && h <= POSE_HEAD_MAXH && w >= 1 && pitch >= 12, DFVO_ESHAPE, "pose_head: %dx%d map (at most %d rows)", h, w, POSE_HEAD_MAXH);
  DFVO_LAUNCH(k_pose_head, dim3(1), dim3(128), 0, s, out12, h, w, pitch, baseline_multiplier, pose_out);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

// cv2.resize(..., INTER_NEAREST) (OpenCV resizeNN): inv_scale = W / w, ifx = 1 / inv_scale,
// sx = min(floor(dx * ifx), w - 1), all in double -- note 1/(W/w) is not bit-identical to w/W
__global__ void k_depth_post(const float* __restrict__ depth, int h, int w, int H, int W, int y0, int y1, int x0, int x1,
                             float min_depth, float max_depth, float* __restrict__ raw_out, float* __restrict__ depth_out) {
  int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= W) return;
  const double ify = 1.0 / ((double)H / (double)h), ifx = 1.0 / ((double)W / (double)w);
  int sy = (int)floor((double)y * ify), sx = (int)floor((double)x * ifx);
  sy = sy < h - 1 ? sy : h - 1; sx = sx < w - 1 ? sx : w - 1;
  float d = depth[(size_t)sy * w + sx];
  if (raw_out) raw_out[(size_t)y * W + x] = d;
  bool keep = y >= y0 && y < y1 && x >= x0 && x < x1 && d < max_depth && d > min_depth;     // utils.py:104-113
  depth_out[(size_t)y * W + x] = keep ? d : 0.f;
}

int depth_post(const float* depth, int h, int w, int H, int W, double cy0, double cy1, double cx0, double cx1, float min_depth,
               float max_depth, float* raw_out, float* depth_out, cudaStream_t s) {
  // int(h*crop): Python float64 multiply then truncation (utils.py:103-104); the fractions cross the ABI as doubles
  int y0 = (int)((double)H * cy0), y1 = (int)((double)H * cy1);
  int x0 = (int)((double)W * cx0), x1 = (int)((double)W * cx1);
  DFVO_LAUNCH(k_depth_post, dim3(cdiv(W, 128), H), dim3(128), 0, s, depth, h, w, H, W, y0, y1, x0, x1, min_depth, max_depth, raw_out,
              depth_out);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

// ---------------------------------------------------------------------------------------------
// PIL-exact antialiased resize of an 8-bit HWC image (Pillow libImaging/Resample.c, 8bpc path): horizontal
// pass to a uint8 intermediate, vertical pass, both with 22-bit fixed-point coefficients and the same
// rounding (start at 1 << 21, arithmetic shift, clamp).  The vertical pass also emits the network feed tensor
// float32 NCHW = uint8 / 255 (transforms.ToTensor, deep_models.py:198).
// ---------------------------------------------------------------------------------------------
DFVO_D uint8_t clip8_fixed(int v) {
  v >>= 22;
  return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

__global__ void k_resample_h_u8(const uint8_t* __restrict__ img, int H, int W, const int32_t* __restrict__ bounds,
                                const int32_t* __restrict__ kk, int ksize, int out_w, uint8_t* __restrict__ tmp) {
  int xx = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (xx >= out_w) return;
  const int xmin = bounds[2 * xx], n = bounds[2 * xx + 1];
  int s0 = 1 << 21, s1 = 1 << 21, s2 = 1 << 21;
  const uint8_t* row = img + ((size_t)y * W + xmin) * 3;
  const int32_t* k = kk + (size_t)xx * ksize;
  for (int x = 0; x < n; ++x) {
    const int c = k[x];
    s0 += (int)row[3 * x] * c; s1 += (int)row[3 * x + 1] * c; s2 += (int)row[3 * x + 2] * c;
  }
  uint8_t* o = tmp + ((size_t)y * out_w + xx) * 3;
  o[0] = clip8_fixed(s0); o[1] = clip8_fixed(s1); o[2] = clip8_fixed(s2);
}

__global__ void k_resample_v_u8(const uint8_t* __restrict__ tmp, int W, const int32_t* __restrict__ bounds,
                                const int32_t* __restrict__ kk, int ksize, int out_h, uint8_t* __restrict__ out_u8,
                                float* __restrict__ out_nchw) {
  int x = blockIdx.x * blockDim.x + threadIdx.x, yy = blockIdx.y;
  if (x >= W) return;
  const int ymin = bounds[2 * yy], n = bounds[2 * yy + 1];
  int s0 = 1 << 21, s1 = 1 << 21, s2 = 1 << 21;
  const int32_t* k = kk + (size_t)yy * ksize;
  for (int y = 0; y < n; ++y) {
    const uint8_t* p = tmp + ((size_t)(ymin + y) * W + x) * 3;
    const int c = k[y];
    s0 += (int)p[0] * c; s1 += (int)p[1] * c; s2 += (int)p[2] * c;
  }
  const uint8_t v[3] = {clip8_fixed(s0), clip8_fixed(s1), clip8_fixed(s2)};
  if (out_u8) { uint8_t* o = out_u8 + ((size_t)yy * W + x) * 3; o[0] = v[0]; o[1] = v[1]; o[2] = v[2]; }
  if (out_nchw)
    for (int c = 0; c < 3; ++c) out_nchw[((size_t)c * out_h + yy) * W + x] = (float)v[c] / 255.0f;
}

int lanczos_resize_u8(const uint8_t* img, int H, int W, const int32_t* bounds_h, const int32_t* kk_h, int ksize_h,
                      const int32_t* bounds_v, const int32_t* kk_v, int ksize_v, int out_h, int out_w, uint8_t* tmp,
                      uint8_t* out_u8, float* out_nchw, cudaStream_t s) {
  DFVO_LAUNCH(k_resample_h_u8, dim3(cdiv(out_w, 128), H), dim3(128), 0, s, img, H, W, bounds_h, kk_h, ksize_h, out_w, tmp);
  DFVO_LAUNCH(k_resample_v_u8, dim3(cdiv(out_w, 128), out_h), dim3(128), 0, s, (const uint8_t*)tmp, out_w, bounds_v, kk_v, ksize_v,
              out_h, out_u8, out_nchw);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

}  // namespace dfvo
