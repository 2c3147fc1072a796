/* dfvo_b200 -- C ABI of the H100-native DF-VO tracking hot path (libdfvo_b200.so).
 *
 * This is the drop-in boundary of SURVEY.md section 8(b): the reference is pure Python and has no
 * FFI of its own, so every entry point below names the reference *Python* interface it replaces
 * (file:line under the DF-VO repository) -- the `libs.*` mirror under df-vo_b200/libs binds these
 * through ctypes (see INTEGRATION.md).
 *
 * Conventions
 *   - return 0 on success, negative DFVO_E* on failure; dfvo_last_error() gives a message
 *     (thread-local).  Nothing throws across the boundary.
 *   - every pointer is caller-owned DEVICE memory unless the name ends in `_host`;
 *   - work is enqueued on the caller's CUDA stream (`stream` is a cudaStream_t passed as void*)
 *     and is asynchronous: outputs are valid after the caller synchronises that stream;
 *   - a handle owns packed weights, workspaces and plans; it is not thread-safe (one per device /
 *     stream of work).
 */
#ifndef DFVO_B200_H_
#define DFVO_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DFVO_OK 0
#define DFVO_EINVAL (-1)
#define DFVO_ECUDA (-2)
#define DFVO_ESHAPE (-3)
#define DFVO_ENOMEM (-4)
#define DFVO_ESTATE (-5)

#define DFVO_NET_LITEFLOWNET 0
#define DFVO_NET_MONODEPTH2 1
#define DFVO_NET_POSENET 2     /* pose_encoder.pth (encoder.* keys) + pose.pth (net.0 .. net.3) */

#define DFVO_PREC_FP32 0 /* every conv on CUDA cores in fp32 (parity mode)            */
#define DFVO_PREC_BF16 1 /* bf16 activations, wgmma tensor-core convs, fp32 accum     */
#define DFVO_PREC_TF32 2 /* fp32 activations, wgmma tf32 convs, fp32 accum            */

#define DFVO_ACT_NONE 0
#define DFVO_ACT_LEAKY 1 /* LeakyReLU(0.1) */
#define DFVO_ACT_RELU 2
#define DFVO_ACT_ELU 3
#define DFVO_ACT_SIGMOID 4

typedef struct dfvo_ctx dfvo_ctx;

const char* dfvo_last_error(void);
const char* dfvo_version(void);
/* 1 if this library was built by nvcc for sm_90a, 0 for the CPU test build (tests/hostsim). */
int dfvo_is_device_build(void);

/* instrumentation for bench.py: number of kernel launches issued by this library so far (process-wide), and
 * CUDA-event timing of the tensor-core conv launches while enabled (sum of durations in ms, launch count, and
 * algorithmic FLOPs = 2*MAC over real channels). */
long long dfvo_launch_count(void);
void dfvo_profile_enable(int on);
void dfvo_profile_read(double* tc_ms, long long* tc_launches, double* tc_flops);
/* Layer chains (csrc/conv_chain.cu): consecutive stride-1 convolutions of a network unit as ONE cooperative launch.  Off by default
 * (measured: fewer launches and a shorter single-stream conv time, but less overlap between the frame pipeline's streams, DESIGN.md
 * 4.4); env DFVO_CONV_CHAIN=1 or this call turn it on for networks created afterwards.  Returns the previous setting. */
int dfvo_set_conv_chain(int on);

int dfvo_create(dfvo_ctx** out, int device);
int dfvo_destroy(dfvo_ctx* ctx);

/* ---- weights --------------------------------------------------------------------------------
 * Replaces torch.load + load_state_dict: LiteFlow.initialize_network_model (lite_flow.py:31-53)
 * Monodepth2DepthNet.initialize_network_model (monodepth2.py:29-71) and Monodepth2PoseNet.initialize_network_model
 * (pose/monodepth2/monodepth2.py:31-84).  `key` is the reference
 * state-dict key (e.g. "moduleFeatures.moduleOne.0.weight", "encoder.layer1.0.conv1.weight",
 * "decoder.0.conv.conv.weight"); data_host is fp32, C-contiguous. */
int dfvo_load_weight(dfvo_ctx* ctx, int net, const char* key, const float* data_host,
                     const int64_t* shape, int ndim);

/* ---- LiteFlowNet: DeepModel.forward_flow (deep_models.py:144-182) ------------------------------
 * Build the plan for `pairs` image pairs of height x width uint8 RGB frames. */
int dfvo_liteflow_build(dfvo_ctx* ctx, int height, int width, int pairs, int precision);
/* imgs: 2*pairs device pointers (host array of device pointers) to HWC uint8 frames ordered
 * [ref0, cur0, ref1, cur1, ...]; n_imgs must equal 2*pairs of the built plan.  Outputs (any may be NULL): flow_fwd / flow_bwd
 * [pairs][2][H][W] fp32 (= flows[(ref,cur)], flows[(cur,ref)]), flow_diff [pairs][H][W] fp32
 * (= flows[(ref,cur,'diff')], deep_flow.py:171-196). */
int dfvo_liteflow_forward(dfvo_ctx* ctx, const uint8_t* const* imgs_host_array, int n_imgs, float* flow_fwd,
                          float* flow_bwd, float* flow_diff, void* stream);
/* parity helper: regularised flow of pyramid level (2..6), NHWC [2*pairs][h][w][2] fp32 */
int dfvo_liteflow_level_flow(dfvo_ctx* ctx, int level, float* out);
int dfvo_liteflow_geometry(dfvo_ctx* ctx, int* net_h, int* net_w, int* batch);

/* ---- monodepth2: DeepModel.forward_depth (deep_models.py:184-206) -------------------------------------
 * feed size = checkpoint 'height'/'width' (monodepth2.py:70-71); (min_depth, max_depth, baseline) are the
 * dataset constants of monodepth2.py:73-88 (kitti: 0.1, 100, 5.4). */
int dfvo_monodepth2_build(dfvo_ctx* ctx, int feed_h, int feed_w, int precision, float min_depth,
                          float max_depth, float baseline);
/* img: float [1,3,feed_h,feed_w] in [0,1] (the PIL-LANCZOS-resized ToTensor image, deep_models.py:195-201);
 * depth_out [feed_h,feed_w] fp32 = Monodepth2DepthNet.inference_depth (monodepth2.py:121-139). */
int dfvo_monodepth2_forward(dfvo_ctx* ctx, const float* img, float* depth_out, void* stream);
/* ---- monodepth2 PoseNet: DeepModel.forward_pose (deep_models.py:208-230) -------------------------------------------------
 * ResnetEncoder(18, False, 2) + PoseDecoder (pose/monodepth2/monodepth2.py:44-119, pose_decoder.py) from the DFVO_NET_POSENET
 * weights.  The feed size is the DEPTH network's (deep_models.py:220: self.depth.feed_width/height); baseline_multiplier is
 * stereo_baseline_multiplier (monodepth2.py:77-84: 5.4 for kitti / robotcar, 1 otherwise). */
int dfvo_posenet_build(dfvo_ctx* ctx, int feed_h, int feed_w, int precision, float baseline_multiplier);
/* feed_ref / feed_cur: float [1,3,feed_h,feed_w] in [0,1] (the feeds of dfvo_lanczos_resize_u8, concatenated [ref, cur] as in
 * deep_models.py:218-226); pose_out: device fp32 [4][4] row-major = inference_pose(...)[0]: transformation_from_parameters(
 * axisangle, translation, invert=True) (layers.py:28-94) with the translation times baseline_multiplier (monodepth2.py:102-119). */
int dfvo_posenet_forward(dfvo_ctx* ctx, const float* feed_ref, const float* feed_cur, float* pose_out, void* stream);
/* ---- batched monodepth2 / PoseNet: one forward over `batch` independent images (e.g. one frame of each of several sequences) --
 * Every layer runs once over N = batch; entry i of the output equals what a batch-1 runner gives for entry i's feed(s), bit for
 * bit.  dfvo_monodepth2_build / dfvo_posenet_build are these with batch = 1 (they replace any runner of the same network). */
int dfvo_monodepth2_build_batch(dfvo_ctx* ctx, int feed_h, int feed_w, int batch, int precision, float min_depth, float max_depth,
                                float baseline);
/* feeds_host_array: n device pointers (host array of device pointers, as dfvo_liteflow_forward's imgs) to float [1,3,feed_h,feed_w]
 * feeds; each entry may point anywhere.  n must equal the built batch (else DFVO_ESHAPE).  depth_out [n][feed_h][feed_w] fp32. */
int dfvo_monodepth2_forward_batch(dfvo_ctx* ctx, const float* const* feeds_host_array, int n, float* depth_out, void* stream);
int dfvo_posenet_build_batch(dfvo_ctx* ctx, int feed_h, int feed_w, int batch, int precision, float baseline_multiplier);
/* feeds_host_array: 2n device pointers [ref0, cur0, ref1, cur1, ...] to float [1,3,feed_h,feed_w] feeds; n must equal the built
 * batch (else DFVO_ESHAPE).  pose_out: device fp32 [n][4][4], entry i = dfvo_posenet_forward(ref_i, cur_i). */
int dfvo_posenet_forward_batch(dfvo_ctx* ctx, const float* const* feeds_host_array, int n, float* pose_out, void* stream);
/* DepthConsistency.compute (depth_consistency.py:31-163): depth_diff [H,W] = clamp(|warp - reproj| / reproj, 0, 1) where reproj is
 * the depth of depth_cur's points under T and warp = grid_sample(depth_ref, Reprojection(depth_cur, T, K, inv_K),
 * padding_mode="border", align_corners=True).  depth_cur / depth_ref: the [H,W] NEAREST-resized raw depths (not range-clamped);
 * T: DEVICE fp32 [4][4] (dfvo_posenet_forward's pose_out, ref_data['deep_pose']); K_host / inv_K_host: float32 3x3 row-major
 * (cam_intrinsics.mat / inv_mat cast to float32).  A 0/0 ratio stays NaN (it fails the selection's `< thre` test). */
int dfvo_depth_consistency(const float* depth_cur, const float* depth_ref, int H, int W, const float* T, const float* K_host,
                           const float* inv_K_host, float* depth_diff, void* stream);
/* PIL.Image.resize((out_w,out_h), LANCZOS) + transforms.ToTensor (deep_models.py:195-198) on the device,
 * bit-exact with Pillow's 8-bit path.  img uint8 [H,W,3]; bounds_* [out][2] / kk_* [out][ksize] int32 are the
 * fixed-point filter tables of b200/lanczos.py (device memory); tmp uint8 [H][out_w][3]; out_u8 [out_h][out_w][3]
 * and/or out_nchw float32 [3][out_h][out_w] (= uint8/255). */
int dfvo_lanczos_resize_u8(const uint8_t* img, int H, int W, const int32_t* bounds_h, const int32_t* kk_h,
                           int ksize_h, const int32_t* bounds_v, const int32_t* kk_v, int ksize_v, int out_h,
                           int out_w, uint8_t* tmp, uint8_t* out_u8, float* out_nchw, void* stream);
/* cv2.resize(raw_depth, (W,H), INTER_NEAREST) + utils.preprocess_depth (dfvo.py:314-319, utils.py:89-114):
 * depth [h,w] -> raw_out [H,W] (may be NULL), depth_out [H,W]; crop = [[y0,y1],[x0,x1]] normalised. */
int dfvo_depth_post(const float* depth, int h, int w, int H, int W, double crop_y0, double crop_y1,
                    double crop_x0, double crop_x1, float min_depth, float max_depth, float* raw_out,
                    float* depth_out, void* stream);

/* ---- stage-level entry points (parity tests; NCHW fp32 at the boundary like the reference) -----
 * FunctionCorrelation (correlation.py:400-402) [+ LeakyReLU if leaky]: first/second [B,C,H,W]
 * -> out [B,49,ceil(H/s),ceil(W/s)].  precision selects the fp32 or bf16 kernel. */
int dfvo_correlation(const float* first, const float* second, float* out, int B, int C, int H, int W,
                     int stride, int leaky, int precision, void* stream);
/* The correlation kernel of the product path on its own layout (BASELINE configs[2] bench): first/second/out are NHWC
 * bf16 device tensors, first/second [B][H][W][Cpitch] (C real channels, Cpitch % 8 == 0), out [B][ceil(H/s)][ceil(W/s)][64]
 * (49 real channels, the rest zero).  second_nxor: the second operand of batch entry n is read at index n ^ second_nxor
 * (1 = the "other image of the pair" addressing LiteFlowNet's level 6 uses, 0 = plain). */
int dfvo_correlation_nhwc_bf16(const void* first, const void* second, void* out, int B, int C, int Cpitch, int H, int W,
                               int stride, int leaky, int second_nxor, void* stream);
/* Backward (lite_flow_net.py:10-28): input [B,C,H,W], flow [B,2,H,W] (already scaled) -> [B,C,H,W] */
int dfvo_backward_warp(const float* input, const float* flow, float* out, int B, int C, int H, int W,
                       int precision, void* stream);
/* FlowToPix + forward_backward_consistency (layers.py:213-229, deep_flow.py:171-196):
 * flow_fwd / flow_bwd [2,H,W] -> diff [H,W] */
int dfvo_fb_consistency(const float* flow_fwd, const float* flow_bwd, float* diff, int H, int W,
                        void* stream);
/* the same over a batch (deep_flow.py:171-196 takes [N,2,H,W]): flow_fwd / flow_bwd [n_pairs,2,H,W] -> diff [n_pairs,H,W], one launch */
int dfvo_fb_consistency_batch(const float* flow_fwd, const float* flow_bwd, float* diff, int n_pairs, int H, int W,
                              void* stream);
/* torch.nn.Conv2d (+ activation): x [B,Cin,H,W], w_host [Cout,Cin,kh,kw], bias_host [Cout] or NULL
 * -> y [B,Cout,Ho,Wo].  precision DFVO_PREC_BF16 / DFVO_PREC_TF32 run the wgmma kernels (bf16 operands /
 * fp32 operands read as tf32; stride 1, or stride 2 on even sizes with 'same' padding). */
int dfvo_conv2d(const float* x, const float* w_host, const float* bias_host, float* y, int B, int Cin,
                int H, int W, int Cout, int kh, int kw, int stride, int pad_y, int pad_x, int reflect,
                int act, int precision, void* stream);

/* ---- correspondence selection (libs/matching) -----------------------------------------------------
 * local_bestN, score_method 'flow' (kp_selection.py:74-200; KeypointSampler.kp_selection,
 * keypoint_sampler.py:76-143).  flow_diff [H,W] fp32; depth_diff optional [H,W] (NULL = depth consistency
 * off).  num_bestN = cfg.kp_selection.local_bestN.num_bestN (per-cell quota = floor(N/(rows*cols))).
 * idx_out [rows*cols*quota] int32: per-cell slots, selected linear pixel indices (y*W+x) ascending, -1
 * padded.  cell_counts [rows*cols].  status[0]=good_kp_found, [1]=#selected, [2]=#(diff<thre), [3]=#cells
 * with >=1 keypoint.  The selected SET equals np.argpartition's; order is canonical (SURVEY H2). */
int dfvo_local_bestn(const float* flow_diff, const float* depth_diff, int H, int W, int rows, int cols,
                     int num_bestN, float thre, float depth_thre, int32_t* idx_out, int32_t* cell_counts,
                     int32_t* status, void* stream);
/* local_bestN, score_method 'flow_ratio' (kp_selection.py:135-160,192-199): ratio_out [H,W] fp32 = flow_diff / ||flow_fwd||, the
 * norm sqrt(fx*fx + fy*fy) rounded step by step like NumPy's float32 np.linalg.norm, so ratio_out is bit-equal to the
 * reference's fb_flow_mask (0/0 = NaN, x/0 = inf; neither passes `< thre`).  The cells select on the ratio with the depth mask as
 * in dfvo_local_bestn; status[2] counts the RAW flow_diff < thre (the "case 1" early-out, kp_selection.py:121-125).  Outputs as
 * dfvo_local_bestn. */
int dfvo_local_bestn_flow_ratio(const float* flow_diff, const float* flow_fwd, const float* depth_diff, int H, int W, int rows,
                                int cols, int num_bestN, float thre, float depth_thre, float* ratio_out, int32_t* idx_out,
                                int32_t* cell_counts, int32_t* status, void* stream);
/* bestN_flow_kp (kp_selection.py:33-71): N smallest of the whole map, ascending linear index. */
size_t dfvo_bestn_workspace_bytes(int H, int W);
int dfvo_bestn(const float* flow_diff, int H, int W, int N, int32_t* idx_out, void* workspace,
               size_t workspace_bytes, void* stream);
/* kp1 = (x,y), kp2 = kp1 + flow_fwd[:,y,x] as float64 [n,2] (keypoint_sampler.py:101-104); compacts the
 * slots of dfvo_local_bestn (cell_counts != NULL) or takes all ncells*quota entries (bestN: ncells=1).  Also serves
 * sampled_kp (kp_selection.py:327-378): idx = the constant uniform list of generate_kp_samples (keypoint_sampler.py:52-74) as
 * full-image linear indices, cell_counts NULL, ncells 1. */
int dfvo_gather_keypoints(const int32_t* idx, const int32_t* cell_counts, int ncells, int quota,
                          const float* flow_fwd, int H, int W, double* kp1, double* kp2, int32_t* n_out,
                          void* stream);

/* ---- rigid-flow keypoints (SURVEY 8f rank 1; EssTracker.kp_selection_good_depth, E_tracker.py:645-705) --------------------
 * rigid_flow_diff [H,W] = | RigidFlow(raw_depth, T, K) - flow_fwd | (rigid_flow.py:38-60, float32): raw_depth [H,W] and
 * flow_fwd [2,H,W] device fp32; T_host = the 4x4 (row-major, first 12 entries used) float64 pose on the HOST. */
int dfvo_rigid_flow_diff(const float* raw_depth, const float* flow_fwd, int H, int W, const double* T_host, double fx, double fy,
                         double cx, double cy, float* rigid_flow_diff, void* stream);
/* opt_rigid_flow_kp (kp_selection.py:203-324), 'uniform' list: per cell every step-th pixel (row-major) that passes both masks.
 * Same output format as dfvo_local_bestn.  The 'best' list is dfvo_local_bestn with (score map, threshold) = (flow_diff,
 * optical_flow_thre) and (second mask map, threshold) = (rigid_flow_diff, rigid_flow_thre), or swapped for score_method
 * 'rigid_flow'. */
int dfvo_uniform_cells(const float* rigid_flow_diff, const float* flow_diff, int H, int W, int rows, int cols, int num_bestN,
                       float rigid_flow_thre, float optical_flow_thre, int32_t* idx_out, int32_t* cell_counts, void* stream);

/* ---- geometry layers (libs/geometry; float32 like the torch modules; matrices are row-major float64 on the HOST) ----------
 * Backprojection.forward (backprojection.py:45-63): depth [H,W] -> points [4][H*W] = (inv_K[:3,:3] @ (x,y,1)) * depth, 1. */
int dfvo_backproject(const float* depth, int H, int W, const double* inv_K9_host, float* points, void* stream);
/* Transformation3D.forward (transformation3d.py:21-31): out [4][n] = T (4x4) @ points [4][n]. */
int dfvo_transform3d(const float* points, long long n, const double* T16_host, float* out, void* stream);
/* Projection.forward (projection.py:31-52): points [4][H*W] -> xy [H][W][2] = (K[:3,:] @ p)[:2] / ((K[:3,:] @ p)[2] + eps),
 * normalized != 0: x/(W-1), y/(H-1), then (xy-0.5)*2.  K12 = the 3x4 matrix K[:3,:]. */
int dfvo_project(const float* points, int H, int W, const double* K12_host, float eps, int normalized, float* xy, void* stream);
/* Reprojection.forward (reprojection.py:37-56) fused: depth [H,W] -> xy [H][W][2]. */
int dfvo_reproject(const float* depth, int H, int W, const double* T16_host, const double* K12_host, const double* inv_K9_host,
                   float eps, int normalized, float* xy, void* stream);
/* RigidFlow.forward (rigid_flow.py:38-58; PixToFlow layers.py:252-266): depth [H,W] -> flow [2][H][W] = reprojected pixel - pixel. */
int dfvo_rigid_flow(const float* depth, int H, int W, const double* T16_host, const double* K12_host, const double* inv_K9_host,
                    float* flow, void* stream);

/* depth[int(kp_y), int(kp_x)] for n keypoints (ops_3d.py:29, pnp_tracker.py:72-73); 0 outside the image. */
int dfvo_gather_depth(const float* depth, int H, int W, const double* kp, int n, float* out, void* stream);

/* ---- pose solvers (libs/tracker, FP64) ------------------------------------------------------------------
 * 5-point minimal solver (inside cv2.findEssentialMat, E_tracker.py:231): M problems, x1/x2 [M][5][2]
 * normalised image points -> E [M][10][9] (row-major, x2^T E x1 = 0, Frobenius-normalised), n [M]. */
int dfvo_five_point(const double* x1, const double* x2, int M, double* E, int32_t* n, void* stream);
/* Sampson inlier counts of M models over N normalised correspondences (BASELINE config #4). */
int dfvo_score_hypotheses(const double* E, int M, const double* x1, const double* x2, int N, double thr2,
                          int32_t* counts, void* stream);
/* R repeats of cv2.findEssentialMat(p1[perm_r], p2[perm_r], focal=fx, pp=(cx,cy), RANSAC, prob, threshold)
 * (E_tracker.py:223-286) + the GRIC-E score of each repeat's winner (gric.py).  p1 = kp_cur, p2 = kp_ref
 * [N][2] pixels; perm [R][N] int32 = the host np.random.shuffle permutations (NULL: identity); subsets
 * [max_iters][5] int32 = OpenCV's subset stream for this N (b200/cvrng.py).  Outputs per repeat: E_out
 * [R][9], mask_out [R][N] uint8 in ORIGINAL point order, info [R][4] = {inliers, iterations run, winning
 * iteration, winning candidate}, gric [R]. */
size_t dfvo_essential_workspace_bytes(int N, int R, int max_iters);
int dfvo_essential_ransac(const double* p1, const double* p2, int N, const int32_t* perm, int R,
                          const int32_t* subsets, int max_iters, double fx, double fy, double cx, double cy,
                          double threshold, double prob, void* workspace, size_t workspace_bytes,
                          double* E_out, uint8_t* mask_out, int32_t* info, double* gric, void* stream);
/* OpenCV's RANSAC subset stream (cv::RNG((uint64)-1) + getSubset, ptsetreg.cpp): the model_points-tuples
 * findEssentialMat / solvePnPRansac draw for `count` correspondences depend only on `count`.  HOST function:
 * out_host [n_subsets][model_points] int32. */
int dfvo_cv_subset_stream_host(int count, int model_points, int n_subsets, int32_t* out_host);
/* The scale fit of find_scale_from_depth (E_tracker.py:618-641): RANSACRegressor(LinearRegression(fit_intercept=False),
 * min_samples, max_trials, stop_probability, residual_threshold).fit(ratio[:, None], ones).estimator_.coef_[0, 0], with the sampling
 * drawn from NumPy's global MT19937 exactly as scikit-learn draws it.  ratio [n] float64 (device).  io (device, DFVO_TAIL_SCALE_IO
 * doubles, offsets DFVO_TAIL_* below): in: the generator state at DFVO_TAIL_MT as 625 uint32 (key[624], pos --
 * np.random.get_state()[1:3]); out: scale, status 1 (ok) / -1 (no consensus: the reference raises ValueError), trials, inliers,
 * and the advanced generator state for np.random.set_state().  perm_scratch: device [n] int32. */
int dfvo_scale_ransac(const double* ratio, int n, int min_samples, int max_trials, double stop_prob, double threshold,
                      double* io, int32_t* perm_scratch, void* stream);
/* Offsets (in doubles) of the packed result of dfvo_essential_tail: res holds DFVO_TAIL_EGRIC + 5 R doubles.  Its prefix
 * [0, DFVO_TAIL_SCALE_IO) is the io block of dfvo_scale_ransac. */
enum {
  DFVO_TAIL_SCALE = 0,         /* scale of the regressor */
  DFVO_TAIL_STATUS = 1,        /* 1 fitted, -1 no consensus, -2 fewer than 11 ratios, -3 pose rejected (scale recovery not run) */
  DFVO_TAIL_TRIALS = 2,        /* regressor trials */
  DFVO_TAIL_INLIERS = 3,       /* regressor inliers */
  DFVO_TAIL_MT = 4,            /* MT19937 state as 625 uint32 (key[624], pos) in DFVO_TAIL_MT_DOUBLES doubles */
  DFVO_TAIL_MT_DOUBLES = 313,
  DFVO_TAIL_SCALE_IO = 317,    /* size of the dfvo_scale_ransac io block */
  DFVO_TAIL_BEST = 317,        /* best repeat (-1: none) */
  DFVO_TAIL_VALID = 318,       /* validity vote */
  DFVO_TAIL_HGRIC = 319,       /* H_gric (0 for flow validity) */
  DFVO_TAIL_CHEIR = 320,       /* cheirality count of recoverPose on the best E */
  DFVO_TAIL_NVALID = 321,      /* valid depth ratios */
  DFVO_TAIL_GATE = 322,        /* 1: the pose stands and |t| != 0, scale recovery runs */
  DFVO_TAIL_RT = 323,          /* R (row-major) then t of recoverPose: 12 doubles */
  DFVO_TAIL_EGRIC = 335        /* [R] E_gric (flow validity: per-repeat cheirality counts), then info [R][4] */
};
/* Everything of the hybrid tracker between "the essential-matrix repeats are done" and "pose and scale are known" in one enqueue, no
 * host round trip (dfvo.py:165-193): the best repeat, cv2.recoverPose on its E (E_tracker.py:292-300), the validity vote, the
 * cheirality gate and -- when the pose stands and |t| != 0 -- find_scale_from_depth (:571-643): triangulation of the normalised
 * keypoints with inv([R|t]), CNN depth at int(kp_cur), last-writer-wins per pixel, depth ratios in row-major pixel order,
 * RANSACRegressor with NumPy's generator state (dfvo_scale_ransac).  E [R][9], info [R][4], gric [R]: outputs of
 * dfvo_essential_ransac.  The validity method follows h_gric:
 *   - h_gric != NULL (GRIC, E_tracker.py:270-290): h_gric [1] is the GRIC of dfvo_homography_ransac (the caller makes the stream wait
 *     for it); the best repeat is the first with the most inliers, the vote is H_gric > E_gric [R].
 *   - h_gric == NULL (flow, E_tracker.py:182-186,249-257,289-300; called only when the dfvo_flow_mean gate passed): gric is not read.
 *     Every repeat's cv2.recoverPose(E_r, kp_cur[perm_r], kp_ref[perm_r]) count cnt_r (a count, so independent of the permutation);
 *     the best repeat is the first with inliers_r > best AND cnt_r > 0.05 N, the vote sum(cnt_r > 0.1 N) > R / 2.
 * depth [H][W] float32 (pre-processed, dfvo_depth_post), or NULL: pose only -- no scale recovery, [0, DFVO_TAIL_SCALE_IO) untouched.
 * res (device, DFVO_TAIL_EGRIC + 5 R doubles, offsets above): in: the generator state at DFVO_TAIL_MT; out: everything else and the
 * advanced generator state.  N <= 4096, R <= 32. */
size_t dfvo_essential_tail_workspace_bytes(int N);
int dfvo_essential_tail(const double* E, const int32_t* info, const double* gric, int R, const double* kp_cur, const double* kp_ref, int N,
                        double fx, double fy, double cx, double cy, const double* h_gric, const float* depth, int H, int W,
                        int min_samples, int max_trials, double stop_prob, double threshold, void* workspace, size_t workspace_bytes,
                        double* res, uint8_t* pose_mask, int32_t* pose_info, void* stream);
/* The flow-magnitude gate of the E-tracker (E_tracker.py:182-185): np.mean(np.linalg.norm(kp_ref - kp_cur, axis=1)), bit-equal to
 * NumPy (rounded products and sums, NumPy's pairwise summation order).  kp [n][2] float64 (device).  status: NULL, or the device
 * status of dfvo_local_bestn ({good, n, ...}), which then supplies the count -- so the selection's one status read also carries
 * the mean.  out (device, 3 doubles) = {good (1 without status), n, mean}.  n <= 65536. */
int dfvo_flow_mean(const double* kp_ref, const double* kp_cur, int n, const int32_t* status, double* out, void* stream);
/* First half of the fused PnP tracker (pnp_tracker.py:45-94): keep the pairs whose kp_cur lies inside the H x W image, read the
 * reference depth [H][W] float32 at int(kp_ref), keep 0 != d, min_depth < d < max_depth, compact in order and unproject:
 * obj [m][3] = (inv(K) [u v 1]^T) d with NumPy's rounding, img [m][2] = kp_cur.  iK_host: inv(K) as np.linalg.inv gives it, row-major
 * [9] in HOST memory (its off-diagonal zeros are checked).  count (device, 1 int32) = m. */
int dfvo_pnp_filter(const double* kp_ref, const double* kp_cur, int n, const float* depth, int H, int W, double min_depth,
                    double max_depth, const double* iK_host, double* obj, double* img, int32_t* count, void* stream);
/* Offsets (in doubles) of the packed result of dfvo_pnp_tail: res holds DFVO_PNP_INFO + 4 R doubles. */
enum {
  DFVO_PNP_BEST = 0,           /* best repeat (-1: none) */
  DFVO_PNP_INLIERS = 1,        /* its RANSAC inliers */
  DFVO_PNP_RVEC = 2,           /* its rvec [3] */
  DFVO_PNP_TVEC = 5,           /* its tvec [3] */
  DFVO_PNP_INFO = 8            /* info [R][4] of dfvo_pnp_ransac */
};
/* Second half: dfvo_pnp_ransac on the filtered points (N = m >= 5, perm = the host's R shuffles of arange(m), subsets =
 * dfvo_cv_subset_stream_host(m, 5, iters)) and the best repeat (found && inliers > best, first maximum; pnp_tracker.py:108-110).
 * res (device, DFVO_PNP_INFO + 4 R doubles, offsets above). */
size_t dfvo_pnp_tail_workspace_bytes(int N, int R, int iters);
int dfvo_pnp_tail(const double* obj, const double* img, int N, const int32_t* perm, int R, const int32_t* subsets, int iters,
                  double fx, double fy, double cx, double cy, double threshold, double prob, void* workspace,
                  size_t workspace_bytes, double* res, void* stream);
/* cv::triangulatePoints([I|0], T_21[:3], x1, x2) followed by X2 = T_21[:3] X / X_w (ops_3d.py:44-67): x1, x2
 * [N][2] normalised (float64), T21 [12] row-major 3x4 -> depth2 [N] = z of the point in view 2. */
int dfvo_triangulate_depth(const double* x1, const double* x2, int N, const double* T21, double* depth2, void* stream);
/* ops_3d.triangulation(kp1, kp2, T_1w, T_2w) (ops_3d.py:44-67) for two general views: x1, x2 [N][2] normalised float64, T1w / T2w
 * [12] = the 3x4 matrices (device memory) -> X, X1, X2 [3][N] (world / view-1 / view-2 coordinates; any may be NULL). */
int dfvo_triangulate_points(const double* x1, const double* x2, int N, const double* T1w, const double* T2w, double* X, double* X1,
                            double* X2, void* stream);
/* cv2.recoverPose(E, p1, p2, focal, pp) (E_tracker.py:292-295): Rt_out[12] = R row-major then t, mask [N],
 * info[5] = {cheirality count, counts of the four (R,t) candidates}. */
int dfvo_recover_pose(const double* E, const double* p1, const double* p2, int N, double focal, double cx,
                      double cy, double* Rt_out, uint8_t* mask_out, int32_t* info, void* stream);

/* cv2.findHomography(p1, p2, RANSAC, ransacReprojThreshold=threshold, maxIters=max_iters, confidence=prob) followed by the
 * GRIC score of the result (E_tracker.py:199-215, gric.py:40-132): p1 = kp_cur, p2 = kp_ref [N][2] float64 pixels.
 * H_out [9] row-major (H[8] = 1), mask_out [N] uint8 = RANSAC inliers, info [4] = {found, inliers, iterations run, winning
 * iteration}, gric [1] = calc_GRIC(compute_homography_residual(H, p1, p2), 0.8, N, 'HMat'). */
size_t dfvo_homography_workspace_bytes(int N, int max_iters);
int dfvo_homography_ransac(const double* p1, const double* p2, int N, int max_iters, double threshold, double prob,
                           void* workspace, size_t workspace_bytes, double* H_out, uint8_t* mask_out, int32_t* info,
                           double* gric, void* stream);
/* R repeats of cv2.solvePnPRansac(obj[perm_r], img[perm_r], K, None, iterationsCount=iters, reprojectionError=threshold,
 * confidence=prob, flags=SOLVEPNP_ITERATIVE) (pnp_tracker.py:86-112).  obj [N][3] = unprojected reference keypoints
 * (ops_3d.py:70-94), img [N][2] pixels, float64; perm [R][N] int32 = the host np.random.shuffle permutations (NULL:
 * identity); subsets [iters][5] int32 = dfvo_cv_subset_stream_host(N, 5, iters).  Per repeat: rt_out [R][6] = rvec, tvec
 * of the final least-squares pose over the RANSAC inliers; info [R][4] = {found, RANSAC inliers, iterations run, winning
 * iteration}.  The caller ranks repeats by the inlier count (pnp_tracker.py:108-110). */
size_t dfvo_pnp_workspace_bytes(int N, int R, int iters);
int dfvo_pnp_ransac(const double* obj, const double* img, int N, const int32_t* perm, int R, const int32_t* subsets,
                    int iters, double fx, double fy, double cx, double cy, double threshold, double prob,
                    void* workspace, size_t workspace_bytes, double* rt_out, int32_t* info, void* stream);
/* Stage entry for parity tests: the minimal solver inside solvePnPRansac -- cv2.solvePnP(obj5, img5, K, None,
 * flags=SOLVEPNP_EPNP) -- on M independent 5-point samples.  obj [M*5][3], img [M*5][2] float64 on the device ->
 * rt [M][12] = R (row-major), t; ok [M].  coop: 1 = lane-cooperative kernel (one warp per sample), 0 = one thread per sample,
 * -1 = what dfvo_pnp_ransac uses (cooperative unless env DFVO_PNP_COOP=0). */
int dfvo_epnp_minimal(const double* obj, const double* img, int M, double fx, double fy, double cx, double cy, int coop,
                      double* rt, int32_t* ok, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DFVO_B200_H_ */
