// Per-pixel geometry layers of the reference (libs/geometry): Backprojection (backprojection.py:45-63), Transformation3D
// (transformation3d.py:21-31), Projection (projection.py:31-52), their composition Reprojection (reprojection.py:37-56)
// and RigidFlow (rigid_flow.py:38-58 = Reprojection + PixToFlow, layers.py:252-266).  All float32 like the torch layers,
// one thread per pixel, in the operation order of the torch matmuls (row dot products accumulated left to right) so that
// the results agree with the layers to float32 round-off.  HBM-bound: 4 B read + 8..16 B written per pixel.
#include "ops.h"

namespace dfvo {

struct GeomP { float T[16]; float K[12]; float iK[9]; float eps; int normalized; };

// points[c][i], c = 0..3: inv_K[:3,:3] @ (x, y, 1) * depth, 1
__global__ void k_backproject(const float* __restrict__ depth, int H, int W, GeomP p, float* __restrict__ points) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= W) return;
  const size_t i = (size_t)y * W + x, hw = (size_t)H * W;
  const float fx = (float)x, fy = (float)y, d = depth[i];
  points[i] = d * (p.iK[0] * fx + p.iK[1] * fy + p.iK[2]);
  points[hw + i] = d * (p.iK[3] * fx + p.iK[4] * fy + p.iK[5]);
  points[2 * hw + i] = d * (p.iK[6] * fx + p.iK[7] * fy + p.iK[8]);
  points[3 * hw + i] = 1.f;
}

// out[r][i] = sum_c T[r][c] * in[c][i]   (4 x 4 @ 4 x n)
__global__ void k_transform3d(const float* __restrict__ in, size_t n, GeomP p, float* __restrict__ out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float a = in[i], b = in[n + i], c = in[2 * n + i], d = in[3 * n + i];
#pragma unroll
  for (int r = 0; r < 4; ++r) out[(size_t)r * n + i] = p.T[4 * r] * a + p.T[4 * r + 1] * b + p.T[4 * r + 2] * c + p.T[4 * r + 3] * d;
}

DFVO_D void project_point(const GeomP& p, float a, float b, float c, float d, int H, int W, float* ox, float* oy) {
  const float ux = p.K[0] * a + p.K[1] * b + p.K[2] * c + p.K[3] * d;
  const float uy = p.K[4] * a + p.K[5] * b + p.K[6] * c + p.K[7] * d;
  const float uw = p.K[8] * a + p.K[9] * b + p.K[10] * c + p.K[11] * d + p.eps;
  float x = ux / uw, y = uy / uw;
  if (p.normalized) {                       // xy[...,0] /= W-1; xy[...,1] /= H-1; xy = (xy - 0.5) * 2
    x = (x / (float)(W - 1) - 0.5f) * 2.f;
    y = (y / (float)(H - 1) - 0.5f) * 2.f;
  }
  *ox = x; *oy = y;
}

// xy[y][x][0..1] = K[:3,:] @ points / (w + eps) [normalised]
__global__ void k_project(const float* __restrict__ points, int H, int W, GeomP p, float* __restrict__ xy) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= W) return;
  const size_t i = (size_t)y * W + x, hw = (size_t)H * W;
  float ox, oy;
  project_point(p, points[i], points[hw + i], points[2 * hw + i], points[3 * hw + i], H, W, &ox, &oy);
  xy[2 * i] = ox; xy[2 * i + 1] = oy;
}

// q = T @ (inv_K[:3,:3] @ (x, y, 1) * d, 1): Backprojection + Transformation3D of one pixel
DFVO_D void backproject_transform(const GeomP& p, float d, float fx, float fy, float q[4]) {
  const float X = d * (p.iK[0] * fx + p.iK[1] * fy + p.iK[2]);
  const float Y = d * (p.iK[3] * fx + p.iK[4] * fy + p.iK[5]);
  const float Z = d * (p.iK[6] * fx + p.iK[7] * fy + p.iK[8]);
#pragma unroll
  for (int r = 0; r < 4; ++r) q[r] = p.T[4 * r] * X + p.T[4 * r + 1] * Y + p.T[4 * r + 2] * Z + p.T[4 * r + 3] * 1.f;
}

// mode 0: xy [H][W][2] (Reprojection);  mode 1: planar flow [2][H][W] = xy - pixel grid (RigidFlow)
__global__ void k_reproject(const float* __restrict__ depth, int H, int W, GeomP p, int mode, float* __restrict__ out) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= W) return;
  const size_t i = (size_t)y * W + x, hw = (size_t)H * W;
  const float fx = (float)x, fy = (float)y;
  float q[4];
  backproject_transform(p, depth[i], fx, fy, q);
  float ox, oy;
  project_point(p, q[0], q[1], q[2], q[3], H, W, &ox, &oy);
  if (mode == 0) { out[2 * i] = ox; out[2 * i + 1] = oy; }
  else { out[i] = ox - fx; out[hw + i] = oy - fy; }
}

// DepthConsistency.compute (depth_consistency.py:69-163) in one pass per pixel of the current frame:
//   reproj_xy  = Reprojection(depth_cur, T, K, inv_K) (normalised, eps 1e-7)
//   warp       = grid_sample(depth_ref, reproj_xy, padding_mode="border", align_corners=True) (torch 1.1 semantics)
//   reproj     = row 2 of T[:3] @ cam_points
//   depth_diff = clamp(|warp - reproj| / reproj, 0, 1)
// The bilinear weights and the tap order are those of torch's grid_sampler_2d.  clamp keeps a NaN (0/0) and maps a negative
// ratio (reproj < 0, behind the camera) to 0, like torch.clamp.  T is the device fp32 4x4 of the PoseNet.
__global__ void k_depth_consistency(const float* __restrict__ depth_cur, const float* __restrict__ depth_ref, int H, int W, GeomP p,
                                    const float* __restrict__ T, float* __restrict__ out) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= W) return;
#pragma unroll
  for (int k = 0; k < 16; ++k) p.T[k] = __ldg(T + k);
  const size_t i = (size_t)y * W + x;
  float q[4];
  backproject_transform(p, depth_cur[i], (float)x, (float)y, q);
  float gx, gy;
  project_point(p, q[0], q[1], q[2], q[3], H, W, &gx, &gy);
  // grid_sampler_unnormalize (align_corners) + clip_coordinates (border)
  float ix = ((gx + 1.f) / 2.f) * (float)(W - 1), iy = ((gy + 1.f) / 2.f) * (float)(H - 1);
  ix = fminf((float)(W - 1), fmaxf(ix, 0.f));
  iy = fminf((float)(H - 1), fmaxf(iy, 0.f));
  const float x0f = floorf(ix), y0f = floorf(iy);
  const int x0 = (int)x0f, y0 = (int)y0f, x1 = x0 + 1, y1 = y0 + 1;
  const float nw = ((float)x1 - ix) * ((float)y1 - iy), ne = (ix - (float)x0) * ((float)y1 - iy);
  const float sw = ((float)x1 - ix) * (iy - (float)y0), se = (ix - (float)x0) * (iy - (float)y0);
  float warp = 0.f;
  const bool xin1 = x1 < W, yin1 = y1 < H;                         // x0, y0 are inside after the border clip
  warp += depth_ref[(size_t)y0 * W + x0] * nw;
  if (xin1) warp += depth_ref[(size_t)y0 * W + x1] * ne;
  if (yin1) warp += depth_ref[(size_t)y1 * W + x0] * sw;
  if (xin1 && yin1) warp += depth_ref[(size_t)y1 * W + x1] * se;
  const float reproj = q[2];
  float r = fabsf(warp - reproj) / reproj;
  if (r < 0.f) r = 0.f;                                            // comparisons are false for NaN: it stays NaN
  else if (r > 1.f) r = 1.f;
  out[i] = r;
}

static void geom_params(const double* T16, const double* K12, const double* iK9, float eps, int normalized, GeomP* p) {
  for (int i = 0; i < 16; ++i) p->T[i] = T16 ? (float)T16[i] : (i % 5 == 0 ? 1.f : 0.f);
  for (int i = 0; i < 12; ++i) p->K[i] = K12 ? (float)K12[i] : 0.f;
  for (int i = 0; i < 9; ++i) p->iK[i] = iK9 ? (float)iK9[i] : 0.f;
  p->eps = eps; p->normalized = normalized;
}

int geom_backproject(const float* depth, int H, int W, const double* iK9, float* points, cudaStream_t s) {
  GeomP p; geom_params(nullptr, nullptr, iK9, 0.f, 0, &p);
  DFVO_LAUNCH(k_backproject, dim3(cdiv(W, 128), H), dim3(128), 0, s, depth, H, W, p, points);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

int geom_transform3d(const float* in, size_t n, const double* T16, float* out, cudaStream_t s) {
  GeomP p; geom_params(T16, nullptr, nullptr, 0.f, 0, &p);
  DFVO_LAUNCH(k_transform3d, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, s, in, n, p, out);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

int geom_project(const float* points, int H, int W, const double* K12, float eps, int normalized, float* xy, cudaStream_t s) {
  GeomP p; geom_params(nullptr, K12, nullptr, eps, normalized, &p);
  DFVO_LAUNCH(k_project, dim3(cdiv(W, 128), H), dim3(128), 0, s, points, H, W, p, xy);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

int geom_reproject(const float* depth, int H, int W, const double* T16, const double* K12, const double* iK9, float eps, int normalized,
                   int mode, float* out, cudaStream_t s) {
  GeomP p; geom_params(T16, K12, iK9, eps, normalized, &p);
  DFVO_LAUNCH(k_reproject, dim3(cdiv(W, 128), H), dim3(128), 0, s, depth, H, W, p, mode, out);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

int geom_depth_consistency(const float* depth_cur, const float* depth_ref, int H, int W, const float* T, const float* K9, const float* iK9,
                           float* out, cudaStream_t s) {
  GeomP p;
  geom_params(nullptr, nullptr, nullptr, 1e-7f, 1, &p);               // Projection(eps=1e-7), normalised (reprojection.py:33-56)
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) { p.K[4 * r + c] = K9[3 * r + c]; p.iK[3 * r + c] = iK9[3 * r + c]; }
  DFVO_LAUNCH(k_depth_consistency, dim3(cdiv(W, 128), H), dim3(128), 0, s, depth_cur, depth_ref, H, W, p, T, out);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

}  // namespace dfvo
