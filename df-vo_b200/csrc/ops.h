// Internal C++ interface of the dfvo_b200 kernels (one declaration per launcher).
// All tensors are device memory, NHWC with explicit strides (common.cuh::Ten); every launcher
// enqueues on the caller's stream and returns DFVO_OK or a negative error code.
#pragma once
#include "common.cuh"

namespace dfvo {

typedef __nv_bfloat16 bf16;

// ---- image / flow plumbing (flow_ops.cu) -------------------------------------------------
// u8 HWC [H0,W0,3] -> float(/255) -> bilinear(align_corners=True) to [th,tw] -> out[n] (pitch>=3).
// (deep_models.py:160-163 + lite_flow.py:72-76).  If norm_mean/std given: (v-mean)/std after resize.
int prep_image_u8(const uint8_t* img, int H0, int W0, Ten<float> out, int n, cudaStream_t s);
// generic bilinear resize of float NHWC (C<=4), align_corners flag (lite_flow_net.py:307-309)
int resize_bilinear_f32(Ten<const float> in, Ten<float> out, int align_corners, cudaStream_t s);
// out[n,y,x,dx*3+c] = img[n,y,x+dx-3,c], zero padded, channels >= 21 zero (stem 7x7 -> 7x1 over 32 channels)
template <typename T>
int im2row7(Ten<const float> img, Ten<T> out, cudaStream_t s);
// out[n, y, x+3, 0..2] = img[n, y, x, 0..2] into a zero-initialised [N, H, W+8, 8] buffer (overlapping-window stem operand)
template <typename T>
int pad_image8(Ten<const float> img, Ten<T> out, cudaStream_t s);
// depthwise ConvTranspose2d k4 s2 p1, no bias (lite_flow_net.py:109,117); w = [C][4][4] float
template <typename T>
int deconv4x4s2_dw(Ten<const T> in, const float* w, Ten<T> out, cudaStream_t s);
// Backward warp (lite_flow_net.py:10-28): out = bilinear(in at (x,y) + flow*scale), zeros outside
// in_nxor: the source is read at batch index (n ^ in_nxor) -- "second image" addressing, see liteflownet.cu
template <typename T>
int warp_bilinear(Ten<const T> in, Ten<const float> flow, float scale, int in_nxor, Ten<T> out, cudaStream_t s);
// 49-channel correlation + fused LeakyReLU(0.1) (correlation.py:38-106, lite_flow_net.py:145-149)
template <typename T>
int correlation49(Ten<const T> f1, Ten<const T> f2, int f2_nxor, int stride, int leaky, Ten<T> out, cudaStream_t s);
// Backward warp + correlation + LeakyReLU of a Matching unit in one call (corr_mma.cu): second operand = feat2[n ^ feat2_nxor]
// warped by flow * scale (flow.p == nullptr: no warp).  bf16 on the device: one tensor-core kernel (mma.sync banded GEMM, warp
// fused into the operand staging); otherwise warp_bilinear into warp_scratch + correlation49.
template <typename T>
int correlation49_warped(Ten<const T> first, Ten<const T> feat2, int feat2_nxor, Ten<const float> flow, float scale, int stride, int leaky,
                         Ten<T> warp_scratch, Ten<T> out, cudaStream_t s);
// per-(n,c) spatial mean of a 2-channel float field (lite_flow_net.py:257) -> mean[n*2+c].  `mean` must have
// room for flow_mean_buffer_floats(N) floats (the means followed by the per-block partial sums).
int flow_mean(Ten<const float> flow, float* mean, cudaStream_t s);
inline size_t flow_mean_buffer_floats(int N) { return (size_t)((N * 2 + 3) & ~3) + (size_t)N * 64 * 2 * 2; }
// Regularization input prep (lite_flow_net.py:244-257): out[...,0]=sqrt(sum((img1-warp(img2))^2)+1e-6),
// out[...,1:3] = flow - mean, remaining channels of out (up to out.C) zero.
template <typename T>
int reg_prep(Ten<const float> img1, Ten<const float> img2, int img2_nxor, Ten<const float> flow, const float* mean,
             float scale, Ten<T> out, cudaStream_t s);
// Regularization tail (lite_flow_net.py:258-264): dist -> exp(-(d^2)-max) weights, weighted local flow
// average through ScaleX/ScaleY (1x1 convs, weights wx/wy[cd], biases bx/by) / sum of weights.
template <typename T>
int reg_tail(Ten<const T> dist, Ten<const float> flow, int k, const float* wx, const float* wy,
             float bx, float by, Ten<float> out, cudaStream_t s);
// flows[1] * 10 -> bilinear(align_corners=True) to [H,W] -> * (W/w, H/h); planar [n][2][H][W] out
// (lite_flow_net.py:322-324, deep_flow.py:107-129)
int flow_upsample_final(Ten<const float> flow, float mul, int H, int W, float* out_planar, cudaStream_t s);
// forward-backward consistency (layers.py:213-229, deep_flow.py:171-196); planar [2][H][W] inputs
int fb_consistency(const float* flow_fwd, const float* flow_bwd, int H, int W, float* diff, cudaStream_t s, int n = 1, long long pair_stride = 0);
// converts / layout helpers (used by stage-level parity entry points)
template <typename TI, typename TO>
int convert_copy(Ten<const TI> in, Ten<TO> out, cudaStream_t s);          // NHWC -> NHWC (C=min)
int nchw_to_nhwc_f32(const float* in, int N, int C, int H, int W, Ten<float> out, cudaStream_t s);
template <typename T>
int nhwc_to_nchw(Ten<const T> in, float* out, cudaStream_t s);

// ---- CUDA-core convolution (conv_direct.cu) -------------------------------------------------
struct ConvDirect {
  int Cin, Cout, kh, kw, stride, pad_y, pad_x;
  int reflect;            // 0: zero padding, 1: reflection padding (layers.py:127-128)
  int act;                // Act
  const float* w;         // [kh*kw*Cin][Cout_pitch] fp32, k = (ky*kw+kx)*Cin + ci
  int w_pitch;            // Cout rounded up to 4
  const float* bias;      // [Cout] or nullptr
};
template <typename TI, typename TO>
int conv_direct(const ConvDirect& c, Ten<const TI> in, Ten<TO> out, Ten<const TO> residual,
                cudaStream_t s);

// 2-channel flow head (lite_flow_net.py:128,178): k x k conv (k = 3, 5, 7; 'same' zero padding) over 32 bf16 channels
// -> 2 fp32 channels + bias + optional fp32 residual.  w = [k*k][32][2] fp32.  CUDA cores: with N = 2 the tensor-core
// tile would be 87 % padding and its 49 taps make it L2-bound.
int flow_head(Ten<const __nv_bfloat16> in, const float* w, float bias0, float bias1, int k, Ten<const float> residual,
              Ten<float> out, cudaStream_t s);

// ---- wgmma implicit-GEMM convolution (conv_tc.cu) ---------------------------------------------
struct ConvTcSource {
  const void* p;          // NHWC view (channel slice allowed) of bf16 (esize 2) or float (esize 4, read as tf32) elements
  int C;                  // channels in this source (multiple of 16; zero-padded by the producer)
  long long sN, sH, sW;   // strides in elements
};
struct ConvTc {
  int N, H, W;            // output spatial size (stride 1)
  int inH, inW;           // input spatial size; 0 = same as output (zero padding through TMA OOB fill).  When
                          // the input is pre-padded (reflection padding) use inH = H + kh - 1 and tap offsets >= 0
  int nsrc;               // 1..3 virtual-concat sources
  ConvTcSource src[3];
  int stride;             // 1, or 2 (then nsrc == 1, even input size; taps address the 2x2 pixel phases through a
                          // 5-D tensor map (pitch+C, W/2, 2, H/2, N) -- see conv_tc.cu)
  int ntaps;              // kh*kw
  int8_t dy[49], dx[49];  // tap offsets in INPUT pixels (already include -pad): iy = oy*stride + dy
  int esize;              // operand element size: 2 = bf16, 4 = fp32 storage read as tf32
  int round_out_tf32;     // esize 4: round the stored fp32 activations to tf32 (cvt.rna) so the next conv's operand is unbiased
  const void* w;          // packed [ntaps][Cout_pad][Ktot] (bf16 or tf32-rounded float), Ktot = sum(src[i].C)
  int Cout_pad;           // multiple of 16
  int Cout;               // real output channels written
  const float* bias;      // [Cout_pad] fp32
  int act;
  int out_f32;            // 0: bf16 output, 1: float output
  void* out;              // NHWC, pointer already offset to the first output channel
  long long oN, oH, oW;   // output strides (elements of the output type)
  const void* residual;   // optional, same type/strides family as out
  long long rN, rH, rW;
  int zero_pad_to;        // if > Cout: also write zeros to channels [Cout, zero_pad_to)
  double flops;           // algorithmic FLOPs of this launch (2*MAC, real channels), for the roofline report
};
// profiling hooks (bench.py roofline): CUDA-event timing of every conv_tc launch while enabled
void conv_tc_profile_enable(int on);
void conv_tc_profile_read(double* ms, long long* launches, double* flops);
int conv_tc(const ConvTc& c, cudaStream_t s);
// Layer chains (conv_chain.cu): between begin and end, consecutive eligible conv_tc() calls on stream s are collected and issued
// as ONE persistent cooperative launch with grid-wide barriers between the layers.  ONLY conv_tc() calls may be made inside the
// scope (collected layers run at conv_chain_end).  `bar`: CHAIN_BAR_WORDS zero-initialised device words owned by the caller, one
// block per chain site (launches that can be in flight together must not share it).  No-op in the CPU test build.
#define CHAIN_BAR_WORDS 16
void conv_chain_begin(cudaStream_t s, unsigned* bar);
int conv_chain_end();
bool conv_chain_take(const ConvTc& c, cudaStream_t s, int* rc);
int conv_chain_set_enabled(int on);      // returns the previous setting; applies to chain scopes opened afterwards
// tile shape chooser shared with tests
void conv_tc_tile_shape(int H, int W, int* tw, int* th);

// ---- monodepth2 helpers (depth_ops.cu) ----------------------------------------------------------------
// NCHW float image -> NHWC T with (x - mean) / std  (resnet_encoder.py:89)
template <typename T>
int normalize_nchw_to_nhwc(const float* in, int N, int C, int H, int W, float mean, float std, Ten<T> out, cudaStream_t s);
// MaxPool2d(kernel 3, stride 2, padding 1)  (torchvision ResNet)
template <typename T>
int maxpool3x3s2(Ten<const T> in, Ten<T> out, cudaStream_t s);
// out[(up*h + 2) x (up*w + 2)] = ReflectionPad2d(1)( cat( nearest_upsample(lo, up), skip ) )  (depth_decoder.py:54-60,
// layers.py:121-136,347-350).  skip may be empty (p == nullptr).  up is 1 or 2.
template <typename T>
int upcat_reflect(Ten<const T> lo, int up, Ten<const T> skip, Ten<T> out, cudaStream_t s);
// sigmoid disparity -> depth (layers.py:16-25, monodepth2.py:111-138): depth = baseline / (min_disp + (max_disp-min_disp)*disp)
int disp_to_depth(const float* disp, int n, float min_depth, float max_depth, float baseline, float* depth, cudaStream_t s);
// PoseDecoder tail + transformation_from_parameters(invert=True) (pose_decoder.py, layers.py:28-94, monodepth2.py:102-119):
// out12 [h][w][pitch] fp32 (channels 0..11 of net.3) -> spatial mean, x 0.01, frame 0's axis-angle / translation, 4x4 pose with
// the translation times baseline_multiplier -> pose_out (device fp32 [4][4])
int pose_head(const float* out12, int h, int w, int pitch, float baseline_multiplier, float* pose_out, cudaStream_t s);
// cv2.resize(INTER_NEAREST) to (W,H) + preprocess_depth (dfvo.py:314-319, utils.py:89-114)
int depth_post(const float* depth, int h, int w, int H, int W, double crop_y0, double crop_y1, double crop_x0, double crop_x1,
               float min_depth, float max_depth, float* raw_out, float* depth_out, cudaStream_t s);

// PIL-exact LANCZOS resize of a uint8 HWC image (tables from b200/lanczos.py); tmp = uint8 [H][out_w][3]
int lanczos_resize_u8(const uint8_t* img, int H, int W, const int32_t* bounds_h, const int32_t* kk_h, int ksize_h,
                      const int32_t* bounds_v, const int32_t* kk_v, int ksize_v, int out_h, int out_w, uint8_t* tmp,
                      uint8_t* out_u8, float* out_nchw, cudaStream_t s);

// ---- keypoint selection (select.cu) -------------------------------------------------------------
int local_bestn(const float* diff, const float* depth_diff, int H, int W, int rows, int cols, int n_best,
                float thre, float depth_thre, int N_total, int32_t* idx_out, int32_t* cell_counts,
                int32_t* status, cudaStream_t s);
int bestn(const float* diff, int H, int W, int N, int32_t* idx_out, void* workspace, size_t ws_bytes,
          cudaStream_t s);
size_t bestn_workspace_bytes(int H, int W);
// opt_rigid_flow_kp 'uniform' sampling per cell (kp_selection.py:277-284); output format of local_bestn
int uniform_cells(const float* rigid_diff, const float* flow_diff, int H, int W, int rows, int cols, int n_best, float rigid_thre,
                  float flow_thre, int32_t* idx_out, int32_t* cell_counts, cudaStream_t s);
// |RigidFlow(depth, T, K) - flow| per pixel (E_tracker.py:666-691); T_host = row-major 3x4 (or 4x4) float64 on the host
int rigid_flow_diff(const float* depth, const float* flow, int H, int W, const double* T_host, double fx, double fy, double cx, double cy,
                    float* out, cudaStream_t s);
int gather_depth(const float* depth, int H, int W, const double* kp, int n, float* out, cudaStream_t s);
// np.mean(np.linalg.norm(kp_ref - kp_cur, axis=1)) bit for bit; status (local_bestn's, nullable) supplies good / n on the device.
// out [3] = {good, n, mean}
int flow_mean(const double* kp_ref, const double* kp_cur, int n, const int32_t* status, double* out, cudaStream_t s);

// ---- geometry layers (geometry.cu): libs/geometry/{backprojection,transformation3d,projection,reprojection,rigid_flow}.py ----
// host matrices are row-major float64 (cast to float32 like torch.from_numpy(..).float()); points are planar [4][H*W]
int geom_backproject(const float* depth, int H, int W, const double* iK9, float* points, cudaStream_t s);
int geom_transform3d(const float* in, size_t n, const double* T16, float* out, cudaStream_t s);
int geom_project(const float* points, int H, int W, const double* K12, float eps, int normalized, float* xy, cudaStream_t s);
// mode 0: xy [H][W][2] (Reprojection.forward);  mode 1: planar flow [2][H][W] (RigidFlow.forward)
int geom_reproject(const float* depth, int H, int W, const double* T16, const double* K12, const double* iK9, float eps, int normalized,
                   int mode, float* out, cudaStream_t s);
// DepthConsistency.compute (depth_consistency.py:69-163): depth_diff [H][W] of depth_cur / depth_ref [H][W] under the device fp32
// pose T [4][4]; K9 / iK9 host float32 3x3 row-major
int geom_depth_consistency(const float* depth_cur, const float* depth_ref, int H, int W, const float* T, const float* K9, const float* iK9,
                           float* out, cudaStream_t s);
// idx: [ncells*n_best] slots (cell-major); cell_counts may be null (all slots valid, e.g. bestN with ncells=1)
int gather_keypoints(const int32_t* idx, const int32_t* cell_counts, int ncells, int n_best, const float* flow_fwd, int H, int W,
                     double* kp1, double* kp2, int32_t* n_out, cudaStream_t s);

}  // namespace dfvo
