// Pose-solver launchers (ransac.cu).
#pragma once
#include "../../include/dfvo_b200.h"
#include "common.cuh"

namespace dfvo {

// stage: M independent 5-point problems; x1/x2 [M][5][2] normalised; E [M][10][9], n [M]
int five_point(const double* x1, const double* x2, int M, double* E, int32_t* n, cudaStream_t s);
// stage: Sampson inlier counts of M models over N normalised correspondences (BASELINE config #4)
int score_hypotheses(const double* E, int M, const double* x1, const double* x2, int N, double thr2, int32_t* counts,
                     cudaStream_t s);
size_t essential_workspace_bytes(int N, int R, int max_iters);
// R repeats of cv2.findEssentialMat(p1[perm_r], p2[perm_r], focal=fx, pp=(cx,cy), RANSAC, prob, threshold) + GRIC-E.
// perm [R][N] (may be null = identity), subsets [max_iters][5] = OpenCV's subset stream for this N.
// outputs per repeat: E_out [R][9], mask_out [R][N] (ORIGINAL point order), info [R][4] = {inliers, iterations,
// best iteration, best candidate}, gric [R].
int essential_ransac(const double* p1, const double* p2, int N, const int32_t* perm, int R, const int32_t* subsets, int max_iters,
                     double fx, double fy, double cx, double cy, double threshold, double prob, void* workspace, size_t ws_bytes,
                     double* E_out, uint8_t* mask_out, int32_t* info, double* gric, cudaStream_t s);
// cv2.recoverPose(E, p1, p2, focal, pp): Rt_out[12] = R (row-major) then t; mask [N]; info[5] = {count, c0..c3}
int recover_pose(const double* E, const double* p1, const double* p2, int N, double focal, double cx, double cy, double* Rt_out,
                 uint8_t* mask_out, int32_t* info, cudaStream_t s);

// R repeats of cv2.solvePnPRansac (pnp.cu): rt_out [R][6] = rvec, tvec; info [R][4] = {found, inliers, iterations, best iteration}
size_t pnp_workspace_bytes(int N, int R, int iters);
int pnp_ransac(const double* obj, const double* img, int N, const int32_t* perm, int R, const int32_t* subsets, int iters, double fx,
               double fy, double cx, double cy, double threshold, double prob, void* workspace, size_t ws_bytes, double* rt_out,
               int32_t* info, cudaStream_t s);

// sklearn RANSACRegressor scale fit on the device, walking NumPy's MT19937 stream (ransac.cu::k_scale_ransac).  io: device
// [DFVO_TAIL_SCALE_IO] doubles = {scale, status, trials, inliers} + key[624], pos as uint32; perm_scratch: device [n] int32
int scale_ransac(const double* ratio, int n, int min_samples, int max_trials, double stop_prob, double thr, double* io, int32_t* perm_scratch,
                 cudaStream_t s);

// fused tail of the E-tracker after essential_ransac (ransac.cu): best repeat -> recoverPose -> validity vote / cheirality gate ->
// depth ratios -> scale regressor, no host round trip.  res: device [DFVO_TAIL_EGRIC + 5 R] doubles (DFVO_TAIL_* of dfvo_b200.h), the
// host generator's MT19937 state at DFVO_TAIL_MT on entry.  h_gric: device [1] GRIC of the homography model (the caller orders the
// stream after it), or nullptr for e_tracker.validity.method 'flow' (gric unused).  depth == nullptr: no scale recovery.
size_t essential_tail_workspace_bytes(int N);
int essential_tail(const double* E, const int32_t* info, const double* gric, int R, const double* kp_cur, const double* kp_ref, int N,
                   double fx, double fy, double cx, double cy, const double* h_gric, const float* depth, int H, int W, int min_samples,
                   int max_trials, double stop_prob, double thr, void* workspace, size_t ws_bytes, double* res, uint8_t* pose_mask,
                   int32_t* pose_info, cudaStream_t s);

// fused PnP tracker (pnp.cu): in-image / depth-range filter + order-preserving compaction + unprojection -> obj [m][3], img [m][2],
// count [1] = m; iK = inv(K) row-major [9] (host memory)
int pnp_filter(const double* kp_ref, const double* kp_cur, int n, const float* depth, int H, int W, double min_depth, double max_depth,
               const double* iK, double* obj, double* img, int32_t* count, cudaStream_t s);
// pnp_ransac + best repeat: res [DFVO_PNP_INFO + 4 R] (DFVO_PNP_* of dfvo_b200.h)
size_t pnp_tail_workspace_bytes(int N, int R, int iters);
int pnp_tail(const double* obj, const double* img, int N, const int32_t* perm, int R, const int32_t* subsets, int iters, double fx, double fy,
             double cx, double cy, double threshold, double prob, void* workspace, size_t ws_bytes, double* res, cudaStream_t s);

// stage entry: EPnP (cv2.solvePnP(flags=SOLVEPNP_EPNP) as solvePnPRansac's minimal solver uses it) on M independent 5-point
// samples; coop: 1 = lane-cooperative kernel, 0 = one thread per sample, -1 = the default of the build
int epnp_minimal(const double* obj, const double* img, int M, double fx, double fy, double cx, double cy, int coop, double* rt,
                 int32_t* ok, cudaStream_t s);

// cv2.findHomography(p1, p2, RANSAC, threshold, maxIters, confidence) + GRIC-H (homog.cu)
size_t homography_workspace_bytes(int N, int max_iters);
int homography_ransac(const double* p1, const double* p2, int N, int max_iters, double threshold, double prob, void* workspace, size_t ws_bytes,
                      double* H_out, uint8_t* mask_out, int32_t* info, double* gric, cudaStream_t s);

// ops_3d.triangulation(kp1n, kp2n, eye(4), T_21) -> z of X2 per point (ops_3d.py:44-67)
int triangulate_depth(const double* x1, const double* x2, int N, const double* T21, double* depth2, cudaStream_t s);
// ops_3d.triangulation for two general views: T1w/T2w device [12] (rows of the 3x4 matrices), outputs [3][N] (nullable)
int triangulate_points(const double* x1, const double* x2, int N, const double* T1w, const double* T2w, double* Xw, double* X1, double* X2,
                       cudaStream_t s);

}  // namespace dfvo
