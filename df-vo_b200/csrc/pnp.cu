// PnP RANSAC on the device: R repeats of
//   cv2.solvePnPRansac(objectPoints[perm_r], imagePoints[perm_r], K, None, iterationsCount, reprojectionError,
//                      confidence 0.99, flags=SOLVEPNP_ITERATIVE)                      (pnp_tracker.py:86-112)
// Structure of OpenCV's routine (calib3d solvepnp.cpp / ptsetreg.cpp; SURVEY.md Appendix C, black-box validated):
//   * points are converted to float32 first (both arrays) -- restated here by rounding the inputs through float;
//   * RANSACPointSetRegistrator(modelPoints = 5, threshold, confidence, maxIters): the SAME subset stream as
//     findEssentialMat (cv::RNG(-1), ransac.cu / dfvo_cv_subset_stream_host), minimal solver = EPnP on the 5 points,
//     error = squared reprojection distance (float), inlier iff err <= thr^2, accept iff good > max(best, 4),
//     niters = RANSACUpdateNumIters(confidence, (N - good) / N, 5, niters);
//   * final pose = solvePnP(ITERATIVE) on the inliers of the best model: the least-squares minimum of the reprojection
//     error.  OpenCV reaches it by Levenberg-Marquardt from a DLT start, this file by Gauss-Newton/LM from the RANSAC
//     model; both stop at the same minimum (the tests state the tolerance).
// EPnP follows Lepetit, Moreno-Noguer, Fua, "EPnP: An Accurate O(n) Solution to the PnP Problem" (IJCV 2009) in the
// formulation OpenCV ships (control points from the PCA of the object points, 12x12 M^T M null space, the three
// beta approximations N = 1..3 + five Gauss-Newton steps each, absolute orientation by Horn/Arun, best reprojection
// error wins).  All arithmetic FP64; one thread per minimal sample (the 12x12 Jacobi eigen-solve dominates).
#include <stdlib.h>
#include "ransac.h"
#include "smallmat.cuh"

namespace dfvo {

struct PnpState { int niters, best_good, best_iter, it; };

namespace epnp {

// One-sided (Hestenes) Jacobi SVD in the formulation of cv::SVD (modules/core lapack.cpp, JacobiSVDImpl_<double>, restated
// from the published algorithm): A [M][N] (M >= N) is held transposed (At: N rows of length M), row pairs (i, j) are
// rotated until orthogonal (|p| <= eps sqrt(ab), eps = 10 DBL_EPSILON), W[i] = |At row i|, rows sorted by descending
// W, rows normalised.  Ut[i] = i-th left singular vector, Vt[i] = i-th right singular vector.  The ORDER of the
// operations is what fixes the signs of the vectors and the basis inside (near-)degenerate singular subspaces --
// EPnP's control points and null-space vectors inherit both, so the minimal-sample poses only agree with OpenCV's
// to round-off if the decomposition is walked the same way.
template <int M, int N>
DFVO_HD void ocv_svd(const double A[M][N], double W[N], double Ut[N][M], double Vt[N][N]) {
  const double eps = 2.220446049250313e-16 * 10;
  for (int i = 0; i < N; ++i) {
    double sd = 0;
    for (int k = 0; k < M; ++k) { const double t = A[k][i]; Ut[i][k] = t; sd += t * t; }
    W[i] = sd;
    for (int k = 0; k < N; ++k) Vt[i][k] = (i == k) ? 1.0 : 0.0;
  }
  const int max_iter = M > 30 ? M : 30;
  for (int iter = 0; iter < max_iter; ++iter) {
    bool changed = false;
    for (int i = 0; i < N - 1; ++i)
      for (int j = i + 1; j < N; ++j) {
        double a = W[i], p = 0, b = W[j];
        for (int k = 0; k < M; ++k) p += Ut[i][k] * Ut[j][k];
        if (fabs(p) <= eps * sqrt(a * b)) continue;
        p *= 2;
        const double beta = a - b, gamma = hypot(p, beta);
        double c, s;
        if (beta < 0) {
          const double delta = (gamma - beta) * 0.5;
          s = sqrt(delta / gamma);
          c = p / (gamma * s * 2);
        } else {
          c = sqrt((gamma + beta) / (gamma * 2));
          s = p / (gamma * c * 2);
        }
        a = b = 0;
        for (int k = 0; k < M; ++k) {
          const double t0 = c * Ut[i][k] + s * Ut[j][k], t1 = -s * Ut[i][k] + c * Ut[j][k];
          Ut[i][k] = t0; Ut[j][k] = t1;
          a += t0 * t0; b += t1 * t1;
        }
        W[i] = a; W[j] = b;
        changed = true;
        for (int k = 0; k < N; ++k) {
          const double t0 = c * Vt[i][k] + s * Vt[j][k], t1 = -s * Vt[i][k] + c * Vt[j][k];
          Vt[i][k] = t0; Vt[j][k] = t1;
        }
      }
    if (!changed) break;
  }
  for (int i = 0; i < N; ++i) {
    double sd = 0;
    for (int k = 0; k < M; ++k) sd += Ut[i][k] * Ut[i][k];
    W[i] = sqrt(sd);
  }
  for (int i = 0; i < N - 1; ++i) {
    int j = i;
    for (int k = i + 1; k < N; ++k) if (W[j] < W[k]) j = k;
    if (i != j) {
      double t = W[i]; W[i] = W[j]; W[j] = t;
      for (int k = 0; k < M; ++k) { t = Ut[i][k]; Ut[i][k] = Ut[j][k]; Ut[j][k] = t; }
      for (int k = 0; k < N; ++k) { t = Vt[i][k]; Vt[i][k] = Vt[j][k]; Vt[j][k] = t; }
    }
  }
  for (int i = 0; i < N; ++i) {
    const double s = W[i] > 2.2250738585072014e-308 ? 1.0 / W[i] : 0.0;      // (OpenCV re-draws a random direction for an
    for (int k = 0; k < M; ++k) Ut[i][k] *= s;                                 //  exactly zero singular value; not needed here)
  }
}

// least squares  min |A x - b|  as cv::solve(A, b, x, DECOMP_SVD): x = sum_i (u_i . b / w_i) v_i over w_i > 2 DBL_EPSILON sum(w)
template <int M, int N>
DFVO_HD void lstsq(const double A[M][N], const double b[M], double x[N]) {
  double W[N], Ut[N][M], Vt[N][N];
  ocv_svd<M, N>(A, W, Ut, Vt);
  double thr = 0;
  for (int i = 0; i < N; ++i) thr += W[i];
  thr *= 2.220446049250313e-16 * 2;
  for (int i = 0; i < N; ++i) x[i] = 0;
  for (int i = 0; i < N; ++i) {
    if (!(W[i] > thr)) continue;
    double c = 0;
    for (int k = 0; k < M; ++k) c += Ut[i][k] * b[k];
    c /= W[i];
    for (int k = 0; k < N; ++k) x[k] += c * Vt[i][k];
  }
}

// the 12 x 12 instance lives in one non-inlined function (local-memory arrays, rolled loops)
DFVO_HD_NOINLINE void svd12(const double A[12][12], double W[12], double Ut[12][12], double Vt[12][12]) {
  ocv_svd<12, 12>(A, W, Ut, Vt);
}

struct Ctx {
  int n;
  double pw[5][3], uv[5][2], al[5][4], cws[4][3];
  double fu, fv, uc, vc;
  double v[4][12];                       // null-space basis, v[0] = smallest eigenvalue
};

// camera-frame control points for a beta vector, sign fix, absolute orientation; returns the mean reprojection error
DFVO_HD double r_and_t(const Ctx& c, const double betas[4], double R[3][3], double t[3]) {
  double ccs[4][3];
  for (int i = 0; i < 4; ++i)
    for (int k = 0; k < 3; ++k) {
      double s = 0;
      for (int j = 0; j < 4; ++j) s += betas[j] * c.v[j][3 * i + k];
      ccs[i][k] = s;
    }
  double pcs[5][3];
  for (int p = 0; p < c.n; ++p)
    for (int k = 0; k < 3; ++k) pcs[p][k] = c.al[p][0] * ccs[0][k] + c.al[p][1] * ccs[1][k] + c.al[p][2] * ccs[2][k] + c.al[p][3] * ccs[3][k];
  if (pcs[0][2] < 0.0)
    for (int p = 0; p < c.n; ++p) for (int k = 0; k < 3; ++k) pcs[p][k] = -pcs[p][k];
  double pc0[3] = {0, 0, 0}, pw0[3] = {0, 0, 0};
  for (int p = 0; p < c.n; ++p) for (int k = 0; k < 3; ++k) { pc0[k] += pcs[p][k]; pw0[k] += c.pw[p][k]; }
  for (int k = 0; k < 3; ++k) { pc0[k] /= c.n; pw0[k] /= c.n; }
  double ABt[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
  for (int p = 0; p < c.n; ++p)
    for (int j = 0; j < 3; ++j)
      for (int k = 0; k < 3; ++k) ABt[j][k] += (pcs[p][j] - pc0[j]) * (c.pw[p][k] - pw0[k]);
  // R = U V^T from the SVD of ABt; a reflection (det < 0) is repaired by negating the last row, as OpenCV's EPnP does
  {
    double W[3], Ut[3][3], Vt[3][3];
    ocv_svd<3, 3>(ABt, W, Ut, Vt);
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) R[i][j] = Ut[0][i] * Vt[0][j] + Ut[1][i] * Vt[1][j] + Ut[2][i] * Vt[2][j];
    if (sm::det3(R) < 0) { R[2][0] = -R[2][0]; R[2][1] = -R[2][1]; R[2][2] = -R[2][2]; }
  }
  for (int k = 0; k < 3; ++k) t[k] = pc0[k] - (R[k][0] * pw0[0] + R[k][1] * pw0[1] + R[k][2] * pw0[2]);
  double err = 0;
  for (int p = 0; p < c.n; ++p) {
    const double X = R[0][0] * c.pw[p][0] + R[0][1] * c.pw[p][1] + R[0][2] * c.pw[p][2] + t[0];
    const double Y = R[1][0] * c.pw[p][0] + R[1][1] * c.pw[p][1] + R[1][2] * c.pw[p][2] + t[1];
    const double iZ = 1.0 / (R[2][0] * c.pw[p][0] + R[2][1] * c.pw[p][1] + R[2][2] * c.pw[p][2] + t[2]);
    const double du = c.uc + c.fu * X * iZ - c.uv[p][0], dv = c.vc + c.fv * Y * iZ - c.uv[p][1];
    err += sqrt(du * du + dv * dv);
  }
  return err / c.n;
}

DFVO_HD void gauss_newton(const double L[6][10], const double rho[6], double b[4]) {
  for (int it = 0; it < 5; ++it) {
    double A[6][4], r[6], x[4];
    for (int i = 0; i < 6; ++i) {
      const double* l = L[i];
      A[i][0] = 2 * l[0] * b[0] + l[1] * b[1] + l[3] * b[2] + l[6] * b[3];
      A[i][1] = l[1] * b[0] + 2 * l[2] * b[1] + l[4] * b[2] + l[7] * b[3];
      A[i][2] = l[3] * b[0] + l[4] * b[1] + 2 * l[5] * b[2] + l[8] * b[3];
      A[i][3] = l[6] * b[0] + l[7] * b[1] + l[8] * b[2] + 2 * l[9] * b[3];
      r[i] = rho[i] - (l[0] * b[0] * b[0] + l[1] * b[0] * b[1] + l[2] * b[1] * b[1] + l[3] * b[0] * b[2] + l[4] * b[1] * b[2] +
                       l[5] * b[2] * b[2] + l[6] * b[0] * b[3] + l[7] * b[1] * b[3] + l[8] * b[2] * b[3] + l[9] * b[3] * b[3]);
    }
    lstsq<6, 4>(A, r, x);
    for (int k = 0; k < 4; ++k) b[k] += x[k];
  }
}

// ---- the stages of EPnP, shared by the one-thread driver (solve) and the lane-cooperative one (solve_coop) ----------------------
// control points (centroid + principal directions scaled by sqrt(eigenvalue / n)) and barycentric coordinates
DFVO_HD bool prepare(Ctx& c, int n, const double pw[][3], const double uv[][2], double fu, double fv, double uc, double vc) {
  c.n = n; c.fu = fu; c.fv = fv; c.uc = uc; c.vc = vc;
  for (int p = 0; p < n; ++p) { for (int k = 0; k < 3; ++k) c.pw[p][k] = pw[p][k]; c.uv[p][0] = uv[p][0]; c.uv[p][1] = uv[p][1]; }
  for (int k = 0; k < 3; ++k) { double s = 0; for (int p = 0; p < n; ++p) s += pw[p][k]; c.cws[0][k] = s / n; }
  {
    double C[3][3], W[3], Ut[3][3], Vt[3][3];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) { double a = 0; for (int p = 0; p < n; ++p) a += (pw[p][i] - c.cws[0][i]) * (pw[p][j] - c.cws[0][j]); C[i][j] = a; }
    ocv_svd<3, 3>(C, W, Ut, Vt);                              // singular values descending, Ut rows = principal directions
    for (int i = 1; i < 4; ++i) {
      const double k = sqrt(W[i - 1] / n);
      for (int j = 0; j < 3; ++j) c.cws[i][j] = c.cws[0][j] + k * Ut[i - 1][j];
    }
  }
  double cc[3][3];
  for (int i = 0; i < 3; ++i) for (int j = 1; j < 4; ++j) cc[i][j - 1] = c.cws[j][i] - c.cws[0][i];
  const double det = sm::det3(cc);
  if (!(fabs(det) > 1e-300)) return false;
  double ci[3][3];
  ci[0][0] = (cc[1][1] * cc[2][2] - cc[1][2] * cc[2][1]) / det; ci[0][1] = (cc[0][2] * cc[2][1] - cc[0][1] * cc[2][2]) / det; ci[0][2] = (cc[0][1] * cc[1][2] - cc[0][2] * cc[1][1]) / det;
  ci[1][0] = (cc[1][2] * cc[2][0] - cc[1][0] * cc[2][2]) / det; ci[1][1] = (cc[0][0] * cc[2][2] - cc[0][2] * cc[2][0]) / det; ci[1][2] = (cc[0][2] * cc[1][0] - cc[0][0] * cc[1][2]) / det;
  ci[2][0] = (cc[1][0] * cc[2][1] - cc[1][1] * cc[2][0]) / det; ci[2][1] = (cc[0][1] * cc[2][0] - cc[0][0] * cc[2][1]) / det; ci[2][2] = (cc[0][0] * cc[1][1] - cc[0][1] * cc[1][0]) / det;
  for (int p = 0; p < n; ++p) {
    double d[3] = {pw[p][0] - c.cws[0][0], pw[p][1] - c.cws[0][1], pw[p][2] - c.cws[0][2]};
    for (int j = 0; j < 3; ++j) c.al[p][1 + j] = ci[j][0] * d[0] + ci[j][1] * d[1] + ci[j][2] * d[2];
    c.al[p][0] = 1.0 - c.al[p][1] - c.al[p][2] - c.al[p][3];
  }
  return true;
}

// row i of M^T M (12 x 12), accumulated over the points in the same order as the full matrix
DFVO_HD void mtm_row(const Ctx& c, int i, double row[12]) {
  for (int j = 0; j < 12; ++j) row[j] = 0;
  for (int p = 0; p < c.n; ++p) {
    double m1[12], m2[12];
    for (int j = 0; j < 4; ++j) {
      m1[3 * j] = c.al[p][j] * c.fu; m1[3 * j + 1] = 0.0;                m1[3 * j + 2] = c.al[p][j] * (c.uc - c.uv[p][0]);
      m2[3 * j] = 0.0;               m2[3 * j + 1] = c.al[p][j] * c.fv;  m2[3 * j + 2] = c.al[p][j] * (c.vc - c.uv[p][1]);
    }
    for (int j = 0; j < 12; ++j) row[j] += m1[i] * m1[j] + m2[i] * m2[j];
  }
}

// L (6 x 10) and rho from the null-space vectors c.v
DFVO_HD void build_L(const Ctx& c, double L[6][10], double rho[6]) {
  const int pa[6] = {0, 0, 0, 1, 1, 2}, pb[6] = {1, 2, 3, 2, 3, 3};
  double dv[4][6][3];
  for (int k = 0; k < 4; ++k)
    for (int i = 0; i < 6; ++i)
      for (int j = 0; j < 3; ++j) dv[k][i][j] = c.v[k][3 * pa[i] + j] - c.v[k][3 * pb[i] + j];
  auto dot = [&](int a, int b, int i) { return dv[a][i][0] * dv[b][i][0] + dv[a][i][1] * dv[b][i][1] + dv[a][i][2] * dv[b][i][2]; };
  for (int i = 0; i < 6; ++i) {
    L[i][0] = dot(0, 0, i); L[i][1] = 2 * dot(0, 1, i); L[i][2] = dot(1, 1, i); L[i][3] = 2 * dot(0, 2, i); L[i][4] = 2 * dot(1, 2, i);
    L[i][5] = dot(2, 2, i); L[i][6] = 2 * dot(0, 3, i); L[i][7] = 2 * dot(1, 3, i); L[i][8] = 2 * dot(2, 3, i); L[i][9] = dot(3, 3, i);
    double s = 0;
    for (int j = 0; j < 3; ++j) { const double d = c.cws[pa[i]][j] - c.cws[pb[i]][j]; s += d * d; }
    rho[i] = s;
  }
}

// the three beta approximations (N = 1, 2, 3); false when the start is not finite
DFVO_HD bool initial_betas(int approx, const double L[6][10], const double rho[6], double b[4]) {
  b[0] = b[1] = b[2] = b[3] = 0;
  if (approx == 1) {                       // betas10 columns {B11, B12, B13, B14}
    double A[6][4], x[4];
    for (int i = 0; i < 6; ++i) { A[i][0] = L[i][0]; A[i][1] = L[i][1]; A[i][2] = L[i][3]; A[i][3] = L[i][6]; }
    lstsq<6, 4>(A, rho, x);
    if (x[0] < 0) { b[0] = sqrt(-x[0]); b[1] = -x[1] / b[0]; b[2] = -x[2] / b[0]; b[3] = -x[3] / b[0]; }
    else { b[0] = sqrt(x[0]); b[1] = x[1] / b[0]; b[2] = x[2] / b[0]; b[3] = x[3] / b[0]; }
  } else if (approx == 2) {                // {B11, B12, B22}
    double A[6][3], x[3];
    for (int i = 0; i < 6; ++i) { A[i][0] = L[i][0]; A[i][1] = L[i][1]; A[i][2] = L[i][2]; }
    lstsq<6, 3>(A, rho, x);
    if (x[0] < 0) { b[0] = sqrt(-x[0]); b[1] = x[2] < 0 ? sqrt(-x[2]) : 0.0; }
    else { b[0] = sqrt(x[0]); b[1] = x[2] > 0 ? sqrt(x[2]) : 0.0; }
    if (x[1] < 0) b[0] = -b[0];
  } else {                                 // {B11, B12, B22, B13, B23}
    double A[6][5], x[5];
    for (int i = 0; i < 6; ++i) { A[i][0] = L[i][0]; A[i][1] = L[i][1]; A[i][2] = L[i][2]; A[i][3] = L[i][3]; A[i][4] = L[i][4]; }
    lstsq<6, 5>(A, rho, x);
    if (x[0] < 0) { b[0] = sqrt(-x[0]); b[1] = x[2] < 0 ? sqrt(-x[2]) : 0.0; }
    else { b[0] = sqrt(x[0]); b[1] = x[2] > 0 ? sqrt(x[2]) : 0.0; }
    if (x[1] < 0) b[0] = -b[0];
    b[2] = x[3] / b[0];
  }
  return (b[0] == b[0]) && (fabs(b[0]) < 1e300);
}

// EPnP on n <= 5 points.  pw: object points, uv: pixels.  Returns false for a degenerate configuration.
DFVO_HD bool solve(int n, const double pw[][3], const double uv[][2], double fu, double fv, double uc, double vc, double R[3][3],
                   double t[3]) {
  Ctx c;
  if (!prepare(c, n, pw, uv, fu, fv, uc, vc)) return false;
  // ---- M^T M (12 x 12) and its four smallest eigenvectors
  {
    double MtM[12][12], W[12], Ut[12][12], Vt[12][12];
    for (int i = 0; i < 12; ++i) mtm_row(c, i, MtM[i]);
    svd12(MtM, W, Ut, Vt);
    for (int k = 0; k < 4; ++k) for (int i = 0; i < 12; ++i) c.v[k][i] = Ut[11 - k][i];      // smallest singular values last
  }
  double L[6][10], rho[6];
  build_L(c, L, rho);
  // ---- three beta approximations, Gauss-Newton, keep the smallest reprojection error
  double best = 1e300;
  for (int approx = 1; approx <= 3; ++approx) {
    double b[4];
    if (!initial_betas(approx, L, rho, b)) continue;
    gauss_newton(L, rho, b);
    double Rc[3][3], tc[3];
    const double e = r_and_t(c, b, Rc, tc);
    if (e == e && e < best) {
      best = e;
      for (int i = 0; i < 3; ++i) { t[i] = tc[i]; for (int j = 0; j < 3; ++j) R[i][j] = Rc[i][j]; }
    }
  }
  return best < 1e300;
}

// ------------------------------------------------------------------------------------------------
// Lane-cooperative EPnP: one warp per minimal sample.
//   * the 12 x 12 one-sided Jacobi SVD -- 55 % of the one-thread solve -- keeps ONE COLUMN of Ut / Vt per lane (lanes 12..31 carry
//     zeros): the row-pair dot product and the two row norms are butterfly sums (every lane ends with the same bits, so the
//     skip / rotate decision is warp-uniform), the rotation is two FMAs per lane.  The PAIR ORDER is the sequential cyclic order of
//     cv::SVD (it fixes the signs and the basis inside the rank-deficient null space, see ocv_svd); what differs from the
//     one-thread path is round-off only: the order of the 12 additions inside a dot product, and the rotation (c, s) evaluated with
//     two reciprocal square roots instead of hypot + 2 divisions + 2 square roots (the dependent FP64 chain that dominates a pair:
//     a version that keeps the division / sqrt chain and packs two samples per warp is slower than the one-thread kernel --
//     the two halves diverge on every skipped pair);
//   * control points / barycentric coordinates / L / rho are recomputed redundantly by every lane (no communication);
//   * the three beta approximations + Gauss-Newton + absolute orientation run on lanes 0, 1, 2 in parallel; the winner (first
//     strictly smaller reprojection error, as in the sequential loop) is broadcast.
// Control flow around the shuffles is warp-uniform, so the CPU emulation build runs it unchanged with one warp per block.
struct CoopSm { double u[12][32], v[12][32], w[12][32]; };      // one private column slot per lane (lanes 16..31 mirror 0..15)
#define EP_FULL 0xffffffffu
DFVO_D double grp_sum(double x) {                // lanes 0..15 (lanes 16..31 mirror them)
  x += __shfl_xor_sync(EP_FULL, x, 8); x += __shfl_xor_sync(EP_FULL, x, 4);
  x += __shfl_xor_sync(EP_FULL, x, 2); x += __shfl_xor_sync(EP_FULL, x, 1);
  return x;
}

// arow: row gl of the symmetric A (= this lane's column of At); vout[k]: this lane's element of null vector k (Ut[11 - k][gl])
DFVO_D void svd12_coop(const double arow[12], CoopSm& sm, int lane, double vout[4]) {
  const int gl = lane & 15;
  const double eps = 2.220446049250313e-16 * 10, eps2 = eps * eps;
  for (int i = 0; i < 12; ++i) {
    const double t = gl < 12 ? arow[i] : 0.0;
    sm.u[i][lane] = t;
    sm.v[i][lane] = (i == gl) ? 1.0 : 0.0;
    sm.w[i][lane] = grp_sum(t * t);
  }
  for (int iter = 0; iter < 30; ++iter) {
    bool changed = false;
    for (int i = 0; i < 11; ++i)
      for (int j = i + 1; j < 12; ++j) {
        const double ui = sm.u[i][lane], uj = sm.u[j][lane];
        const double a = sm.w[i][lane], b = sm.w[j][lane];
        double p = grp_sum(ui * uj);
        if (p * p <= eps2 * (a * b)) continue;                    // |p| <= eps sqrt(a b)
        p *= 2;
        // gamma = hypot(p, beta);  beta < 0: s = sqrt((gamma - beta) / (2 gamma)), c = p / (2 gamma s)
        //                          else:     c = sqrt((gamma + beta) / (2 gamma)), s = p / (2 gamma c)
        const double beta = a - b, g2 = p * p + beta * beta;
        const double rg = rsqrt(g2), gamma = g2 * rg;             // 1 / gamma, gamma
        const double q = 0.5 * (gamma + fabs(beta)) * rg;          // the larger of c^2, s^2  (in [0.5, 1])
        const double rq = rsqrt(q), big = q * rq, small_ = 0.5 * p * rg * rq;
        const double c = beta < 0 ? small_ : big, s = beta < 0 ? big : small_;
        const double t0 = c * ui + s * uj, t1 = -s * ui + c * uj;
        sm.u[i][lane] = t0; sm.u[j][lane] = t1;
        double a2 = t0 * t0, b2 = t1 * t1;                       // two independent butterflies in flight
        a2 += __shfl_xor_sync(EP_FULL, a2, 8); b2 += __shfl_xor_sync(EP_FULL, b2, 8);
        a2 += __shfl_xor_sync(EP_FULL, a2, 4); b2 += __shfl_xor_sync(EP_FULL, b2, 4);
        a2 += __shfl_xor_sync(EP_FULL, a2, 2); b2 += __shfl_xor_sync(EP_FULL, b2, 2);
        a2 += __shfl_xor_sync(EP_FULL, a2, 1); b2 += __shfl_xor_sync(EP_FULL, b2, 1);
        sm.w[i][lane] = a2; sm.w[j][lane] = b2;
        changed = true;
        const double vi = sm.v[i][lane], vj = sm.v[j][lane];
        sm.v[i][lane] = c * vi + s * vj; sm.v[j][lane] = -s * vi + c * vj;
      }
    if (!changed) break;                                          // warp-uniform
  }
  double W[12];
  int perm[12];
  for (int i = 0; i < 12; ++i) { const double t = sm.u[i][lane]; W[i] = sqrt(grp_sum(t * t)); perm[i] = i; }
  for (int i = 0; i < 11; ++i) {                                 // the selection sort of ocv_svd, on a row permutation
    int j = i;
    for (int k = i + 1; k < 12; ++k) if (W[j] < W[k]) j = k;
    if (i != j) { const double t = W[i]; W[i] = W[j]; W[j] = t; const int q = perm[i]; perm[i] = perm[j]; perm[j] = q; }
  }
  for (int k = 0; k < 4; ++k) {
    const double sc = W[11 - k] > 2.2250738585072014e-308 ? 1.0 / W[11 - k] : 0.0;
    vout[k] = sm.u[perm[11 - k]][lane] * sc;
  }
}

// every lane of the warp passes the same sample; R, t, return value are warp-uniform
DFVO_D bool solve_coop(const double pw[][3], const double uv[][2], double fu, double fv, double uc, double vc, CoopSm& sm, int lane,
                       double R[3][3], double t[3]) {
  const int gl = lane & 15;
  Ctx c;
  bool good = prepare(c, 5, pw, uv, fu, fv, uc, vc);
  if (!good)                                                    // degenerate sample: keep walking (uniform shuffles), report failure
    for (int p = 0; p < 5; ++p) for (int j = 0; j < 4; ++j) c.al[p][j] = 0.25;
  double row[12], vout[4];
  mtm_row(c, gl < 12 ? gl : 0, row);
  svd12_coop(row, sm, lane, vout);
  for (int k = 0; k < 4; ++k)
    for (int i = 0; i < 12; ++i) c.v[k][i] = __shfl_sync(EP_FULL, vout[k], i);
  double L[6][10], rho[6];
  build_L(c, L, rho);
  double e = 1e300, Rc[3][3], tc[3];
  for (int i = 0; i < 3; ++i) { tc[i] = 0; for (int j = 0; j < 3; ++j) Rc[i][j] = 0; }
  if (lane < 3) {
    double b[4];
    if (initial_betas(lane + 1, L, rho, b)) {
      gauss_newton(L, rho, b);
      const double ee = r_and_t(c, b, Rc, tc);
      if (ee == ee) e = ee;
    }
  }
  double best = 1e300;
  int win = 0;
  for (int a = 0; a < 3; ++a) {
    const double ea = __shfl_sync(EP_FULL, e, a);
    if (ea < best) { best = ea; win = a; }
  }
  for (int i = 0; i < 3; ++i) {
    t[i] = __shfl_sync(EP_FULL, tc[i], win);
    for (int j = 0; j < 3; ++j) R[i][j] = __shfl_sync(EP_FULL, Rc[i][j], win);
  }
  return good && best < 1e300;
}

}  // namespace epnp

// ------------------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------------------
// float32-rounded, permuted copies of the points: objp [R][N][3], imgp [R][N][2]
__global__ void k_pnp_prepare(const double* __restrict__ obj, const double* __restrict__ img, const int32_t* __restrict__ perm, int N,
                              double* __restrict__ objp, double* __restrict__ imgp, PnpState* st, int iters) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x, r = blockIdx.y;
  if (i == 0) { st[r].niters = iters; st[r].best_good = -1; st[r].best_iter = -1; st[r].it = 0; }
  if (i >= N) return;
  const int src = perm ? perm[(size_t)r * N + i] : i;
  const size_t o = (size_t)r * N + i;
  for (int k = 0; k < 3; ++k) objp[o * 3 + k] = (double)(float)obj[3 * src + k];
  for (int k = 0; k < 2; ++k) imgp[o * 2 + k] = (double)(float)img[2 * src + k];
}

// one thread per (iteration, repeat): EPnP on the sample -> hyp [R][iters][12] (R row-major, t), ok [R][iters]
__global__ void k_pnp_hypotheses(const double* __restrict__ objp, const double* __restrict__ imgp, const int32_t* __restrict__ subsets,
                                 int N, int iters, double fx, double fy, double cx, double cy, double* __restrict__ hyp,
                                 int32_t* __restrict__ ok) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x, r = blockIdx.y;
  if (i >= iters) return;
  double pw[5][3], uv[5][2];
  for (int k = 0; k < 5; ++k) {
    const size_t o = (size_t)r * N + (subsets ? subsets[i * 5 + k] : i * 5 + k);
    for (int j = 0; j < 3; ++j) pw[k][j] = objp[o * 3 + j];
    uv[k][0] = imgp[o * 2]; uv[k][1] = imgp[o * 2 + 1];
  }
  // solvePnP(SOLVEPNP_EPNP) first maps the pixels to normalised coordinates (cv::undistortPoints without distortion:
  // (u - cx) * (1 / fx), stored as float32 because the RANSAC's points are float32) and runs EPnP with an identity
  // camera matrix
  const double ifx = 1.0 / fx, ify = 1.0 / fy;
  for (int k = 0; k < 5; ++k) { uv[k][0] = (double)(float)((uv[k][0] - cx) * ifx); uv[k][1] = (double)(float)((uv[k][1] - cy) * ify); }
  double Rm[3][3], t[3];
  const bool good = epnp::solve(5, pw, uv, 1.0, 1.0, 0.0, 0.0, Rm, t);
  const size_t h = (size_t)r * iters + i;
  ok[h] = good ? 1 : 0;
  if (good) {
    for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) hyp[h * 12 + 3 * a + b] = Rm[a][b];
    for (int a = 0; a < 3; ++a) hyp[h * 12 + 9 + a] = t[a];
  }
}

// one minimal sample per warp, epnp::solve_coop
#ifdef DFVO_HOSTSIM
#define PNP_COOP_WARPS 1            // the CPU emulation treats a shuffle as a block-wide rendezvous: one warp per block
#else
#define PNP_COOP_WARPS 4
#endif
__global__ void __launch_bounds__(32 * PNP_COOP_WARPS)
k_pnp_hypotheses_coop(const double* __restrict__ objp, const double* __restrict__ imgp, const int32_t* __restrict__ subsets, int N,
                      int iters, double fx, double fy, double cx, double cy, double* __restrict__ hyp, int32_t* __restrict__ ok) {
  __shared__ epnp::CoopSm sm[PNP_COOP_WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, r = blockIdx.y;
  const int i = blockIdx.x * PNP_COOP_WARPS + warp;
  if (i >= iters) return;                                    // whole warps leave: the shuffles below stay warp-complete
  double pw[5][3], uv[5][2];
  const double ifx = 1.0 / fx, ify = 1.0 / fy;
  for (int k = 0; k < 5; ++k) {
    const size_t o = (size_t)r * N + (subsets ? subsets[i * 5 + k] : i * 5 + k);
    for (int j = 0; j < 3; ++j) pw[k][j] = objp[o * 3 + j];
    uv[k][0] = (double)(float)((imgp[o * 2] - cx) * ifx); uv[k][1] = (double)(float)((imgp[o * 2 + 1] - cy) * ify);   // see k_pnp_hypotheses
  }
  double Rm[3][3], t[3];
  const bool good = epnp::solve_coop(pw, uv, 1.0, 1.0, 0.0, 0.0, sm[warp], lane, Rm, t);
  if (lane == 0) {
    const size_t h = (size_t)r * iters + i;
    ok[h] = good ? 1 : 0;
    if (good) {
      for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) hyp[h * 12 + 3 * a + b] = Rm[a][b];
      for (int a = 0; a < 3; ++a) hyp[h * 12 + 9 + a] = t[a];
    }
  }
}

// DFVO_PNP_COOP=0 selects the one-thread-per-sample kernel; read per call so tests can compare the two paths
static bool pnp_coop_enabled() {
  const char* e = getenv("DFVO_PNP_COOP");
  return !(e && atoi(e) == 0);
}

static int pnp_hypotheses(const double* objp, const double* imgp, const int32_t* subsets, int N, int R, int iters, double fx, double fy,
                          double cx, double cy, double* hyp, int32_t* ok, int coop, cudaStream_t s) {
  if (coop < 0) coop = pnp_coop_enabled() ? 1 : 0;
  if (coop) {
    DFVO_LAUNCH(k_pnp_hypotheses_coop, dim3(cdiv(iters, PNP_COOP_WARPS), R), dim3(32 * PNP_COOP_WARPS), 0, s, objp, imgp, subsets, N, iters,
                fx, fy, cx, cy, hyp, ok);
  } else {
    DFVO_LAUNCH(k_pnp_hypotheses, dim3(cdiv(iters, 32), R), dim3(32), 0, s, objp, imgp, subsets, N, iters, fx, fy, cx, cy, hyp, ok);
  }
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

// stage entry (dfvo_epnp_minimal): M independent 5-point samples, obj [M*5][3], img [M*5][2] (device, FP64) -> rt [M][12], ok [M]
int epnp_minimal(const double* obj, const double* img, int M, double fx, double fy, double cx, double cy, int coop, double* rt,
                 int32_t* ok, cudaStream_t s) {
  DFVO_REQUIRE(obj && img && rt && ok && M >= 1, DFVO_EINVAL, "epnp_minimal args");
  return pnp_hypotheses(obj, img, nullptr, 5 * M, 1, M, fx, fy, cx, cy, rt, ok, coop, s);
}

DFVO_D bool pnp_inlier(const double* __restrict__ h, const double* __restrict__ X, const double* __restrict__ u, double fx, double fy,
                       double cx, double cy, float thr2) {
  const double x = h[0] * X[0] + h[1] * X[1] + h[2] * X[2] + h[9];
  const double y = h[3] * X[0] + h[4] * X[1] + h[5] * X[2] + h[10];
  const double z = h[6] * X[0] + h[7] * X[1] + h[8] * X[2] + h[11];
  const double iz = z != 0.0 ? 1.0 / z : 1.0;                   // cv::projectPoints: z = z ? 1/z : 1
  // OpenCV evaluates the error on float32 projections / image points (solvepnp.cpp PnPRansacCallback::computeError)
  const float du = (float)((x * iz) * fx + cx) - (float)u[0], dv = (float)((y * iz) * fy + cy) - (float)u[1];
  return du * du + dv * dv <= thr2;
}

// one warp per (iteration, repeat): inlier count of the hypothesis
__global__ void __launch_bounds__(256)
k_pnp_score(const double* __restrict__ hyp, const int32_t* __restrict__ ok, const double* __restrict__ objp,
            const double* __restrict__ imgp, int N, int iters, double fx, double fy, double cx, double cy, float thr2,
            int32_t* __restrict__ counts) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, r = blockIdx.y;
  if (w >= iters) return;
  const size_t h = (size_t)r * iters + w;
  int c = 0;
  if (ok[h]) {
    double m[12];
    for (int q = 0; q < 12; ++q) m[q] = hyp[h * 12 + q];
    const double* X = objp + (size_t)r * N * 3;
    const double* u = imgp + (size_t)r * N * 2;
    for (int j = lane; j < N; j += 32) c += pnp_inlier(m, X + 3 * j, u + 2 * j, fx, fy, cx, cy, thr2) ? 1 : 0;
  }
  for (int off = 16; off > 0; off >>= 1) c += __shfl_xor_sync(0xffffffffu, c, off);
  if (lane == 0) counts[h] = c;
}

DFVO_HD int pnp_update_num_iters(double p, double ep, int model_points, int max_iters) {
  // cv::RANSACUpdateNumIters (ptsetreg.cpp)
  p = p < 0 ? 0 : (p > 1 ? 1 : p);
  ep = ep < 0 ? 0 : (ep > 1 ? 1 : ep);
  double num = 1.0 - p;
  if (num < 2.2250738585072014e-308) num = 2.2250738585072014e-308;
  double denom = 1.0 - pow(1.0 - ep, (double)model_points);
  if (denom < 2.2250738585072014e-308) return 0;
  num = log(num);
  denom = log(denom);
  if (denom >= 0 || -num >= max_iters * (-denom)) return max_iters;
  return (int)rint(num / denom);
}

// sequential acceptance rule of RANSACPointSetRegistrator::run, one thread per repeat
__global__ void k_pnp_replay(const int32_t* __restrict__ ok, const int32_t* __restrict__ counts, int N, int iters, double prob,
                             PnpState* st, int R) {
  const int r = threadIdx.x + blockIdx.x * blockDim.x;
  if (r >= R) return;
  PnpState s = st[r];
  int it = 0;
  while (it < s.niters && it < iters) {
    const size_t h = (size_t)r * iters + it;
    if (ok[h]) {
      const int good = counts[h];
      const int lim = s.best_good > 4 ? s.best_good : 4;
      if (good > lim) {
        s.best_good = good; s.best_iter = it;
        s.niters = pnp_update_num_iters(prob, (double)(N - good) / (double)N, 5, s.niters);
      }
    }
    ++it;
  }
  s.it = it;
  st[r] = s;
}

// one block per repeat: least-squares pose over the inliers of the best model (Gauss-Newton with Levenberg damping on
// the left-multiplied rotation increment), then rvec = log(R).  out: rt [R][6], info [R][4] = {ok, inliers, iterations,
// best iteration}
__global__ void __launch_bounds__(256)
k_pnp_refine(const double* __restrict__ hyp, const PnpState* __restrict__ st, const double* __restrict__ objp,
             const double* __restrict__ imgp, int N, int iters, double fx, double fy, double cx, double cy, float thr2,
             double* __restrict__ rt_out, int32_t* __restrict__ info, uint8_t* __restrict__ inl) {
  __shared__ double red[256];
  __shared__ double part[8][27];
  __shared__ double pose[12], trial[12], acc[28];
  __shared__ double lambda, cur_cost;
  __shared__ int stop;
  const int r = blockIdx.x, t = threadIdx.x;
  const PnpState s = st[r];
  if (s.best_iter < 0) {
    if (t == 0) {
      for (int k = 0; k < 6; ++k) rt_out[r * 6 + k] = 0.0;
      info[r * 4 + 0] = 0; info[r * 4 + 1] = 0; info[r * 4 + 2] = s.it; info[r * 4 + 3] = -1;
    }
    return;
  }
  const double* X = objp + (size_t)r * N * 3;
  const double* u = imgp + (size_t)r * N * 2;
  uint8_t* mask = inl + (size_t)r * N;
  if (t < 12) pose[t] = hyp[((size_t)r * iters + s.best_iter) * 12 + t];
  __syncthreads();
  for (int j = t; j < N; j += 256) mask[j] = pnp_inlier(pose, X + 3 * j, u + 2 * j, fx, fy, cx, cy, thr2) ? 1 : 0;
  if (t == 0) { lambda = 1e-3; stop = 0; cur_cost = -1.0; }
  __syncthreads();

  auto reduce = [&](double v) {             // block sum, result in red[0]
    red[t] = v;
    __syncthreads();
    for (int off = 128; off > 0; off >>= 1) { if (t < off) red[t] += red[t + off]; __syncthreads(); }
    const double out = red[0];
    __syncthreads();
    return out;
  };
  auto cost_of = [&](const double* P) {
    double c = 0;
    for (int j = t; j < N; j += 256) {
      if (!mask[j]) continue;
      const double* Xj = X + 3 * j;
      const double x = P[0] * Xj[0] + P[1] * Xj[1] + P[2] * Xj[2] + P[9], y = P[3] * Xj[0] + P[4] * Xj[1] + P[5] * Xj[2] + P[10];
      const double z = P[6] * Xj[0] + P[7] * Xj[1] + P[8] * Xj[2] + P[11];
      const double du = fx * x / z + cx - u[2 * j], dv = fy * y / z + cy - u[2 * j + 1];
      c += du * du + dv * dv;
    }
    return reduce(c);
  };
  {
    const double c0 = cost_of(pose);
    if (t == 0) cur_cost = c0;
    __syncthreads();
  }
  for (int iter = 0; iter < 60; ++iter) {
    // normal equations  J^T J d = -J^T e  with d = (dw, dt):  Xc' = (I + [dw]x) Xc + dt
    double a[27];
    for (int k = 0; k < 27; ++k) a[k] = 0.0;
    for (int j = t; j < N; j += 256) {
      if (!mask[j]) continue;
      const double* Xj = X + 3 * j;
      const double x = pose[0] * Xj[0] + pose[1] * Xj[1] + pose[2] * Xj[2] + pose[9];
      const double y = pose[3] * Xj[0] + pose[4] * Xj[1] + pose[5] * Xj[2] + pose[10];
      const double z = pose[6] * Xj[0] + pose[7] * Xj[1] + pose[8] * Xj[2] + pose[11];
      const double iz = 1.0 / z;
      const double eu = fx * x * iz + cx - u[2 * j], ev = fy * y * iz + cy - u[2 * j + 1];
      // d(u)/d(Xc) = fx [1/z, 0, -x/z^2];  d(Xc)/d(dw) = -[Xc]x;  d(Xc)/d(dt) = I
      const double gu[3] = {fx * iz, 0.0, -fx * x * iz * iz}, gv[3] = {0.0, fy * iz, -fy * y * iz * iz};
      double ju[6], jv[6];
      ju[0] = gu[2] * y - gu[1] * z; ju[1] = gu[0] * z - gu[2] * x; ju[2] = gu[1] * x - gu[0] * y;      // (g x Xc)^T ... = g . (-[Xc]x)
      jv[0] = gv[2] * y - gv[1] * z; jv[1] = gv[0] * z - gv[2] * x; jv[2] = gv[1] * x - gv[0] * y;
      for (int k = 0; k < 3; ++k) { ju[3 + k] = gu[k]; jv[3 + k] = gv[k]; }
      int q = 0;
      for (int i = 0; i < 6; ++i)
        for (int k = i; k < 6; ++k) a[q++] += ju[i] * ju[k] + jv[i] * jv[k];
      for (int i = 0; i < 6; ++i) a[21 + i] += ju[i] * eu + jv[i] * ev;
    }
    for (int k = 0; k < 27; ++k) {                   // warp sums, then the 8 warp partials
      double v = a[k];
      for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
      if ((t & 31) == 0) part[t >> 5][k] = v;
    }
    __syncthreads();
    if (t < 27) { double v = 0; for (int w8 = 0; w8 < 8; ++w8) v += part[w8][t]; acc[t] = v; }
    __syncthreads();
    if (t == 0) {
      double Hm[6][6], g[6];
      int q = 0;
      for (int i = 0; i < 6; ++i) for (int k = i; k < 6; ++k) { Hm[i][k] = acc[q]; Hm[k][i] = acc[q]; ++q; }
      for (int i = 0; i < 6; ++i) { g[i] = -acc[21 + i]; Hm[i][i] *= (1.0 + lambda); }
      // Cholesky solve
      double Lc[6][6];
      bool pd = true;
      for (int i = 0; i < 6 && pd; ++i)
        for (int k = 0; k <= i; ++k) {
          double sum = Hm[i][k];
          for (int m = 0; m < k; ++m) sum -= Lc[i][m] * Lc[k][m];
          if (i == k) { if (sum <= 0) { pd = false; break; } Lc[i][i] = sqrt(sum); }
          else Lc[i][k] = sum / Lc[k][k];
        }
      double d[6] = {0, 0, 0, 0, 0, 0};
      if (pd) {
        double yv[6];
        for (int i = 0; i < 6; ++i) { double sum = g[i]; for (int m = 0; m < i; ++m) sum -= Lc[i][m] * yv[m]; yv[i] = sum / Lc[i][i]; }
        for (int i = 5; i >= 0; --i) { double sum = yv[i]; for (int m = i + 1; m < 6; ++m) sum -= Lc[m][i] * d[m]; d[i] = sum / Lc[i][i]; }
      }
      // trial pose: R' = exp([dw]x) R, t' = exp([dw]x) t + dt
      const double th = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
      double E[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
      if (th > 0) {
        const double kx = d[0] / th, ky = d[1] / th, kz = d[2] / th, c = cos(th), sn = sin(th), v = 1 - c;
        E[0][0] = c + kx * kx * v; E[0][1] = kx * ky * v - kz * sn; E[0][2] = kx * kz * v + ky * sn;
        E[1][0] = ky * kx * v + kz * sn; E[1][1] = c + ky * ky * v; E[1][2] = ky * kz * v - kx * sn;
        E[2][0] = kz * kx * v - ky * sn; E[2][1] = kz * ky * v + kx * sn; E[2][2] = c + kz * kz * v;
      }
      for (int i = 0; i < 3; ++i) {
        for (int k = 0; k < 3; ++k) trial[3 * i + k] = E[i][0] * pose[k] + E[i][1] * pose[3 + k] + E[i][2] * pose[6 + k];
        trial[9 + i] = E[i][0] * pose[9] + E[i][1] * pose[10] + E[i][2] * pose[11] + d[3 + i];
      }
      acc[27] = pd ? sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2] + d[3] * d[3] + d[4] * d[4] + d[5] * d[5]) : -1.0;
    }
    __syncthreads();
    const double c1 = cost_of(trial);
    if (t == 0) {
      const double step = acc[27];
      if (step >= 0 && c1 <= cur_cost) {
        for (int k = 0; k < 12; ++k) pose[k] = trial[k];
        const double rel = (cur_cost - c1) <= 1e-14 * (cur_cost > 1e-300 ? cur_cost : 1e-300);
        cur_cost = c1;
        lambda = lambda * 0.1 > 1e-12 ? lambda * 0.1 : 1e-12;
        if (step < 1e-13 || rel) stop = 1;
      } else {
        lambda *= 10.0;
        if (lambda > 1e12) stop = 1;
      }
    }
    __syncthreads();
    if (stop) break;
  }
  if (t == 0) {
    // rvec = log(R)  (cv::Rodrigues, matrix -> vector)
    const double* P = pose;
    const double rx = P[7] - P[5], ry = P[2] - P[6], rz = P[3] - P[1];
    const double sn = 0.5 * sqrt(rx * rx + ry * ry + rz * rz);
    double c = 0.5 * (P[0] + P[4] + P[8] - 1.0);
    c = c > 1.0 ? 1.0 : (c < -1.0 ? -1.0 : c);
    const double theta = acos(c);
    double rv[3];
    if (sn < 1e-5) {
      if (c > 0) { rv[0] = rv[1] = rv[2] = 0.0; }
      else {
        double tx = sqrt(fmax((P[0] + 1) * 0.5, 0.0)), ty = sqrt(fmax((P[4] + 1) * 0.5, 0.0)) * (P[1] < 0 ? -1.0 : 1.0);
        double tz = sqrt(fmax((P[8] + 1) * 0.5, 0.0)) * (P[2] < 0 ? -1.0 : 1.0);
        if (fabs(tx) < fabs(ty) && fabs(tx) < fabs(tz) && (P[5] > 0) != (ty * tz > 0)) tz = -tz;
        const double nn = theta / sqrt(tx * tx + ty * ty + tz * tz);
        rv[0] = tx * nn; rv[1] = ty * nn; rv[2] = tz * nn;
      }
    } else {
      const double vth = 0.5 / sn * theta;
      rv[0] = rx * vth; rv[1] = ry * vth; rv[2] = rz * vth;
    }
    for (int k = 0; k < 3; ++k) { rt_out[r * 6 + k] = rv[k]; rt_out[r * 6 + 3 + k] = pose[9 + k]; }
    info[r * 4 + 0] = 1; info[r * 4 + 1] = s.best_good; info[r * 4 + 2] = s.it; info[r * 4 + 3] = s.best_iter;
  }
}

size_t pnp_workspace_bytes(int N, int R, int iters) {
  size_t b = 0;
  b += (size_t)R * N * 5 * 8;                    // permuted object / image points
  b += (size_t)R * iters * 12 * 8;               // hypotheses
  b += (size_t)R * iters * 4 * 2;                // ok, counts
  b += (size_t)R * N;                            // inlier masks
  b += (size_t)R * sizeof(PnpState);
  return b + 2048;
}

int pnp_ransac(const double* obj, const double* img, int N, const int32_t* perm, int R, const int32_t* subsets, int iters, double fx,
               double fy, double cx, double cy, double threshold, double prob, void* workspace, size_t ws_bytes, double* rt_out,
               int32_t* info, cudaStream_t s) {
  DFVO_REQUIRE(obj && img && subsets && rt_out && info && N >= 5 && R >= 1 && R <= 32 && iters >= 1, DFVO_EINVAL, "pnp_ransac args (N=%d R=%d)", N, R);
  DFVO_REQUIRE(ws_bytes >= pnp_workspace_bytes(N, R, iters), DFVO_EINVAL, "pnp_ransac workspace too small");
  uint8_t* w = reinterpret_cast<uint8_t*>(workspace);
  auto take = [&](size_t bytes) { uint8_t* p = w; w += (bytes + 127) & ~(size_t)127; return p; };
  double* objp = (double*)take((size_t)R * N * 3 * 8);
  double* imgp = (double*)take((size_t)R * N * 2 * 8);
  double* hyp = (double*)take((size_t)R * iters * 12 * 8);
  int32_t* ok = (int32_t*)take((size_t)R * iters * 4);
  int32_t* counts = (int32_t*)take((size_t)R * iters * 4);
  uint8_t* inl = (uint8_t*)take((size_t)R * N);
  PnpState* st = (PnpState*)take((size_t)R * sizeof(PnpState));
  const float thr2 = (float)(threshold * threshold);
  DFVO_LAUNCH(k_pnp_prepare, dim3(cdiv(N, 128), R), dim3(128), 0, s, obj, img, perm, N, objp, imgp, st, iters);
  { int rc = pnp_hypotheses(objp, imgp, subsets, N, R, iters, fx, fy, cx, cy, hyp, ok, -1, s); if (rc) return rc; }
  DFVO_LAUNCH(k_pnp_score, dim3(cdiv(iters * 32, 256), R), dim3(256), 0, s, hyp, ok, objp, imgp, N, iters, fx, fy, cx, cy, thr2, counts);
  DFVO_LAUNCH(k_pnp_replay, dim3(1), dim3(32), 0, s, ok, counts, N, iters, prob, st, R);
  DFVO_LAUNCH(k_pnp_refine, dim3(R), dim3(256), 0, s, hyp, st, objp, imgp, N, iters, fx, fy, cx, cy, thr2, rt_out, info, inl);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

}  // namespace dfvo
