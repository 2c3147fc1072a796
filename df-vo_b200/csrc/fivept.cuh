// Nister five-point essential-matrix minimal solver in FP64, written as __host__ __device__ code so
// the very same source is exercised by the CPU test-suite (tests/hostsim) and by the CUDA RANSAC.
//
// Replaces the minimal solver inside cv2.findEssentialMat (E_tracker.py:231-239; OpenCV calib3d
// five-point.cpp, SURVEY Appendix C): epipolar constraints -> 4-D null space -> ten cubic constraints
// (det E = 0, 2 E E^T E - tr(E E^T) E = 0) in the monomials of (x,y,z) -> Gauss-Jordan -> 3x3
// polynomial matrix B(z) -> degree-10 polynomial -> real roots -> (x,y) back-substitution ->
// E = xX + yY + zZ + W, Frobenius-normalised.  Differences from OpenCV that do not change the solution
// set: the null space comes from Householder QR instead of a Jacobi SVD (any basis spans the same
// space) and (x,y) from cross products instead of SVD::solveZ.  Roots come from the same
// Durand-Kerner iteration OpenCV's solvePoly uses; candidates are emitted in root-index order.
#pragma once
#include "common.cuh"

namespace dfvo {
namespace fivept {

// monomial orders: deg<=1: [x,y,z,1]; deg<=2: [x2,xy,xz,x,y2,yz,y,z2,z,1];
// deg<=3 (Nister): [x3,y3,x2y,xy2,x2z,x2,y2z,y2,xyz,xy | xz2,xz,x,yz2,yz,y,z3,z2,z,1]
DFVO_HD int m11(int a, int b) {
  const int t[4][4] = {{0, 1, 2, 3}, {1, 4, 5, 6}, {2, 5, 7, 8}, {3, 6, 8, 9}};
  return t[a][b];
}
DFVO_HD int m21(int a, int b) {
  const int t[10][4] = {{0, 2, 4, 5}, {2, 3, 8, 9}, {4, 8, 10, 11}, {5, 9, 11, 12}, {3, 1, 6, 7},
                        {8, 6, 13, 14}, {9, 7, 14, 15}, {10, 13, 16, 17}, {11, 14, 17, 18}, {12, 15, 18, 19}};
  return t[a][b];
}

// c(deg2) += a(deg1) * b(deg1)
DFVO_HD void mul11_acc(const double* a, const double* b, double* c, double s) {
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) c[m11(i, j)] += s * a[i] * b[j];
}
// c(deg3) += a(deg2) * b(deg1)
DFVO_HD void mul21_acc(const double* a, const double* b, double* c, double s) {
  for (int i = 0; i < 10; ++i)
    for (int j = 0; j < 4; ++j) c[m21(i, j)] += s * a[i] * b[j];
}

// Null space of the 5x9 epipolar matrix: last four columns of the full Q of Householder QR of Q^T.
// basis[k][9], k = 0..3 (X, Y, Z, W); returns false if rank deficient beyond recovery.
DFVO_HD bool null_space(const double* x1, const double* x2, double basis[4][9]) {
  double A[9][5];   // Q^T: column i is the constraint of point i
  for (int i = 0; i < 5; ++i) {
    const double u1 = x1[2 * i], v1 = x1[2 * i + 1], u2 = x2[2 * i], v2 = x2[2 * i + 1];
    // x2^T E x1 = 0, E row-major
    A[0][i] = u2 * u1; A[1][i] = u2 * v1; A[2][i] = u2;
    A[3][i] = v2 * u1; A[4][i] = v2 * v1; A[5][i] = v2;
    A[6][i] = u1;      A[7][i] = v1;      A[8][i] = 1.0;
  }
  double V[5][9];    // Householder vectors
  double beta[5];
  for (int k = 0; k < 5; ++k) {
    double norm2 = 0.0;
    for (int r = k; r < 9; ++r) norm2 += A[r][k] * A[r][k];
    const double norm = sqrt(norm2);
    for (int r = 0; r < 9; ++r) V[k][r] = 0.0;
    if (norm == 0.0) { beta[k] = 0.0; continue; }
    const double alpha = A[k][k] > 0 ? -norm : norm;
    for (int r = k; r < 9; ++r) V[k][r] = A[r][k];
    V[k][k] -= alpha;
    double vn2 = 0.0;
    for (int r = k; r < 9; ++r) vn2 += V[k][r] * V[k][r];
    beta[k] = vn2 > 0.0 ? 2.0 / vn2 : 0.0;
    for (int c = k; c < 5; ++c) {
      double dot = 0.0;
      for (int r = k; r < 9; ++r) dot += V[k][r] * A[r][c];
      dot *= beta[k];
      for (int r = k; r < 9; ++r) A[r][c] -= dot * V[k][r];
    }
  }
  // Q e_j = H1 H2 ... H5 e_j for j = 5..8
  for (int j = 0; j < 4; ++j) {
    double q[9];
    for (int r = 0; r < 9; ++r) q[r] = (r == 5 + j) ? 1.0 : 0.0;
    for (int k = 4; k >= 0; --k) {
      double dot = 0.0;
      for (int r = k; r < 9; ++r) dot += V[k][r] * q[r];
      dot *= beta[k];
      for (int r = k; r < 9; ++r) q[r] -= dot * V[k][r];
    }
    for (int r = 0; r < 9; ++r) basis[j][r] = q[r];
  }
  return true;
}

// The ten cubic constraints, one row at a time (Nister monomial order).  constraint_prep: E[i][j] as degree-1 polynomials,
// E E^T (degree 2) and its trace; constraint_row(r): r = 0 -> det E, r = 1 + 3i + j -> entry (i,j) of 2 E E^T E - tr(E E^T) E.
DFVO_HD void constraint_prep(const double basis[4][9], double E[9][4], double EEt[9][10], double tr[10]) {
  // E[i][j] as a degree-1 polynomial: coefficients [x,y,z,1] = basis[0..3][3i+j]
  for (int e = 0; e < 9; ++e)
    for (int k = 0; k < 4; ++k) E[e][k] = basis[k][e];
  // EEt = E E^T (symmetric, deg 2); trace
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double* d = EEt[3 * i + j];
      for (int m = 0; m < 10; ++m) d[m] = 0.0;
      for (int k = 0; k < 3; ++k) mul11_acc(E[3 * i + k], E[3 * j + k], d, 1.0);
    }
  for (int m = 0; m < 10; ++m) tr[m] = EEt[0][m] + EEt[4][m] + EEt[8][m];
}

DFVO_HD void constraint_row(const double E[9][4], const double EEt[9][10], const double tr[10], int r, double* row) {
  for (int c = 0; c < 20; ++c) row[c] = 0.0;
  if (r == 0) {
    // det(E) = e0(e4 e8 - e5 e7) - e1(e3 e8 - e5 e6) + e2(e3 e7 - e4 e6)
    double t[10];
    const int a[3] = {0, 1, 2}, p[3][2] = {{4, 8}, {3, 8}, {3, 7}}, q[3][2] = {{5, 7}, {5, 6}, {4, 6}};
    const double sg[3] = {1.0, -1.0, 1.0};
    for (int k = 0; k < 3; ++k) {
      for (int i = 0; i < 10; ++i) t[i] = 0.0;
      mul11_acc(E[p[k][0]], E[p[k][1]], t, 1.0);
      mul11_acc(E[q[k][0]], E[q[k][1]], t, -1.0);
      mul21_acc(t, E[a[k]], row, sg[k]);
    }
    return;
  }
  // 2 EEt E - tr E = 0  <=>  (EEt - 0.5 tr I) E = 0
  const int i = (r - 1) / 3, j = (r - 1) % 3;
  for (int k = 0; k < 3; ++k) {
    double L[10];
    for (int m = 0; m < 10; ++m) L[m] = EEt[3 * i + k][m] - (i == k ? 0.5 * tr[m] : 0.0);
    mul21_acc(L, E[3 * k + j], row, 1.0);
  }
}

// Build the 10x20 constraint matrix (Nister monomial order).
DFVO_HD void constraint_matrix(const double basis[4][9], double M[10][20]) {
  double E[9][4], EEt[9][10], tr[10];
  constraint_prep(basis, E, EEt, tr);
  for (int r = 0; r < 10; ++r) constraint_row(E, EEt, tr, r, M[r]);
}

// Gauss-Jordan with partial pivoting on the left 10x10 block; false if singular.
DFVO_HD bool gauss_jordan(double M[10][20]) {
  for (int c = 0; c < 10; ++c) {
    int piv = c;
    double best = fabs(M[c][c]);
    for (int r = c + 1; r < 10; ++r) {
      double v = fabs(M[r][c]);
      if (v > best) { best = v; piv = r; }
    }
    if (best < 1e-300) return false;
    if (piv != c)
      for (int k = 0; k < 20; ++k) { double t = M[c][k]; M[c][k] = M[piv][k]; M[piv][k] = t; }
    const double inv = 1.0 / M[c][c];
    for (int k = c; k < 20; ++k) M[c][k] *= inv;
    for (int r = 0; r < 10; ++r) {
      if (r == c) continue;
      const double f = M[r][c];
      if (f == 0.0) continue;
      for (int k = c; k < 20; ++k) M[r][k] -= f * M[c][k];
    }
  }
  return true;
}

// polynomials in z stored ascending (p[0] = constant)
DFVO_HD void pmul(const double* a, int da, const double* b, int db, double* c) {
  for (int i = 0; i <= da + db; ++i) c[i] = 0.0;
  for (int i = 0; i <= da; ++i)
    for (int j = 0; j <= db; ++j) c[i + j] += a[i] * b[j];
}

// B rows from the eliminated matrix; det B(z) -> c[0..10] ascending.  bx,by: [3][4], b1: [3][5] ascending.
// `right` points at the first right-hand-side column of row 0, rows are `stride` doubles apart.
DFVO_HD void build_poly_rows(const double* right, int stride, double bx[3][4], double by[3][4], double b1[3][5], double c[11]) {
  for (int i = 0; i < 3; ++i) {
    const double* r1 = right + (4 + 2 * i) * stride;
    const double* r2 = right + (5 + 2 * i) * stride;
    // r = [x z2, x z, x, y z2, y z, y, z3, z2, z, 1];  row = r1 - z * r2
    bx[i][0] = r1[2];            bx[i][1] = r1[1] - r2[2]; bx[i][2] = r1[0] - r2[1]; bx[i][3] = -r2[0];
    by[i][0] = r1[5];            by[i][1] = r1[4] - r2[5]; by[i][2] = r1[3] - r2[4]; by[i][3] = -r2[3];
    b1[i][0] = r1[9];            b1[i][1] = r1[8] - r2[9]; b1[i][2] = r1[7] - r2[8]; b1[i][3] = r1[6] - r2[7];
    b1[i][4] = -r2[6];
  }
  for (int k = 0; k <= 10; ++k) c[k] = 0.0;
  // det = bx0 (by1 b12 - by2 b11) - by0 (bx1 b12 - bx2 b11) + b10 (bx1 by2 - bx2 by1)
  double t7a[8], t7b[8], t6a[7], t6b[7], t10[11];
  pmul(by[1], 3, b1[2], 4, t7a); pmul(by[2], 3, b1[1], 4, t7b);
  for (int k = 0; k < 8; ++k) t7a[k] -= t7b[k];
  pmul(bx[0], 3, t7a, 7, t10);
  for (int k = 0; k <= 10; ++k) c[k] += t10[k];
  pmul(bx[1], 3, b1[2], 4, t7a); pmul(bx[2], 3, b1[1], 4, t7b);
  for (int k = 0; k < 8; ++k) t7a[k] -= t7b[k];
  pmul(by[0], 3, t7a, 7, t10);
  for (int k = 0; k <= 10; ++k) c[k] -= t10[k];
  pmul(bx[1], 3, by[2], 3, t6a); pmul(bx[2], 3, by[1], 3, t6b);
  for (int k = 0; k < 7; ++k) t6a[k] -= t6b[k];
  pmul(b1[0], 4, t6a, 6, t10);
  for (int k = 0; k <= 10; ++k) c[k] += t10[k];
}

DFVO_HD void build_poly(const double M[10][20], double bx[3][4], double by[3][4], double b1[3][5], double c[11]) {
  build_poly_rows(&M[0][10], 20, bx, by, b1, c);
}

// Durand-Kerner (the iteration of cv::solvePoly): roots of c[0..n] (ascending).  re/im: [n].
// cv::solvePoly stops only at exact stagnation (max_diff <= 0), i.e. it normally runs all of its 1000
// iterations.  The iteration converges quadratically at simple roots (linearly, ratio 1/2, at double roots):
// once the largest correction is below 1e-13 of the root scale -- or has stopped contracting at the
// round-off floor (eps for simple roots, eps^(1/m) for an m-fold root) -- the roots are stationary at
// round-off level: same roots, same index order; the real ones are Newton-polished by the caller.
// N is a compile-time degree so that roots and coefficients live in registers on the device.
struct DkStop {
  double prev = 1e300;
  int stall = 0;
  DFVO_HD bool done(double max_diff, double rmax) {
    if (max_diff <= 1e-13 * rmax) return true;
    if (!(max_diff == max_diff)) return true;       // NaN guard
    if (max_diff >= 0.25 * prev) {                  // no longer contracting quadratically
      if (max_diff <= 1e-9 * rmax) return true;
      if (max_diff <= 1e-4 * rmax && ++stall >= 8) return true;
    } else {
      stall = 0;
    }
    prev = max_diff;
    return false;
  }
};

template <int N>
DFVO_HD_NOINLINE int durand_kerner_fixed(const double* c_in, double* re_out, double* im_out, int max_iters) {
  double c[N + 1], re[N], im[N];
#pragma unroll
  for (int k = 0; k <= N; ++k) c[k] = c_in[k];
  {
    double pr = 1.0, pi = 0.0;                       // initial guesses p = (1,0) * (1,1)^i
#pragma unroll
    for (int i = 0; i < N; ++i) {
      re[i] = pr; im[i] = pi;
      const double nr = pr - pi, ni = pr + pi;
      pr = nr; pi = ni;
    }
  }
  DkStop stop;
  int iter = 0;
  for (; iter < max_iters; ++iter) {
    double max_diff = 0.0;
#pragma unroll
    for (int i = 0; i < N; ++i) {
      const double xr = re[i], xi = im[i];
      double nr = c[N], ni = 0.0, dr = c[N], di = 0.0;
#pragma unroll
      for (int j = 0; j < N; ++j) {
        const double tr = nr * xr - ni * xi + c[N - j - 1], ti = nr * xi + ni * xr;   // num = num * p + c[n-j-1]
        nr = tr; ni = ti;
        if (j != i) {
          const double er = xr - re[j], ei = xi - im[j];
          const bool nz = (er != 0.0 || ei != 0.0);
          const double ur = dr * er - di * ei, ui = dr * ei + di * er;
          dr = nz ? ur : dr; di = nz ? ui : di;
        }
      }
      const double den = dr * dr + di * di;
      double qr = 0.0, qi = 0.0;
      if (den > 0.0) { qr = (nr * dr + ni * di) / den; qi = (ni * dr - nr * di) / den; }   // num /= denom
      re[i] = xr - qr; im[i] = xi - qi;
      const double ad = sqrt(qr * qr + qi * qi);
      if (ad > max_diff) max_diff = ad;
    }
    double rmax = 0.0;
#pragma unroll
    for (int i = 0; i < N; ++i) { const double a = fabs(re[i]) + fabs(im[i]); if (a > rmax) rmax = a; }
    if (stop.done(max_diff, rmax)) break;
  }
#pragma unroll
  for (int i = 0; i < N; ++i) { re_out[i] = re[i]; im_out[i] = im[i]; }
#ifdef DFVO_DK_STATS
  DFVO_DK_STATS(iter);
#endif
  return iter;
}

// run-time degree (n < 10 only when the leading coefficients vanish)
DFVO_HD int durand_kerner(const double* c, int n, double* re, double* im, int max_iters) {
  if (n == 10) return durand_kerner_fixed<10>(c, re, im, max_iters);
  double pr = 1.0, pi = 0.0;
  for (int i = 0; i < n; ++i) {
    re[i] = pr; im[i] = pi;
    const double nr = pr - pi, ni = pr + pi;
    pr = nr; pi = ni;
  }
  DkStop stop;
  int iter = 0;
  for (; iter < max_iters; ++iter) {
    double max_diff = 0.0;
    for (int i = 0; i < n; ++i) {
      const double xr = re[i], xi = im[i];
      double nr = c[n], ni = 0.0, dr = c[n], di = 0.0;
      for (int j = 0; j < n; ++j) {
        const double tr = nr * xr - ni * xi + c[n - j - 1], ti = nr * xi + ni * xr;
        nr = tr; ni = ti;
        if (j != i) {
          const double er = xr - re[j], ei = xi - im[j];
          if (er != 0.0 || ei != 0.0) {
            const double ur = dr * er - di * ei, ui = dr * ei + di * er;
            dr = ur; di = ui;
          }
        }
      }
      const double den = dr * dr + di * di;
      double qr = 0.0, qi = 0.0;
      if (den > 0.0) { qr = (nr * dr + ni * di) / den; qi = (ni * dr - nr * di) / den; }
      re[i] = xr - qr; im[i] = xi - qi;
      const double ad = sqrt(qr * qr + qi * qi);
      if (ad > max_diff) max_diff = ad;
    }
    double rmax = 0.0;
    for (int i = 0; i < n; ++i) { const double a = fabs(re[i]) + fabs(im[i]); if (a > rmax) rmax = a; }
    if (stop.done(max_diff, rmax)) break;
  }
  return iter;
}

// Nister-order monomials of (x,y,z) and their partial derivatives
DFVO_HD void monomials(double x, double y, double z, double m[20], double dx[20], double dy[20], double dz[20]) {
  const double v[20][3] = {{3, 0, 0}, {0, 3, 0}, {2, 1, 0}, {1, 2, 0}, {2, 0, 1}, {2, 0, 0}, {0, 2, 1}, {0, 2, 0}, {1, 1, 1}, {1, 1, 0},
                           {1, 0, 2}, {1, 0, 1}, {1, 0, 0}, {0, 1, 2}, {0, 1, 1}, {0, 1, 0}, {0, 0, 3}, {0, 0, 2}, {0, 0, 1}, {0, 0, 0}};
  double px[4] = {1, x, x * x, x * x * x}, py[4] = {1, y, y * y, y * y * y}, pz[4] = {1, z, z * z, z * z * z};
  for (int k = 0; k < 20; ++k) {
    const int a = (int)v[k][0], b = (int)v[k][1], c = (int)v[k][2];
    m[k] = px[a] * py[b] * pz[c];
    dx[k] = a ? a * px[a - 1] * py[b] * pz[c] : 0.0;
    dy[k] = b ? b * px[a] * py[b - 1] * pz[c] : 0.0;
    dz[k] = c ? c * px[a] * py[b] * pz[c - 1] : 0.0;
  }
}

// Gauss-Newton polish of (x,y,z) on the ten cubic constraints M0 * monomials = 0.
DFVO_HD void refine(const double M0[10][20], double* x, double* y, double* z) {
  for (int it = 0; it < 3; ++it) {
    double m[20], dx[20], dy[20], dz[20];
    monomials(*x, *y, *z, m, dx, dy, dz);
    double JtJ[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}}, Jtr[3] = {0, 0, 0}, rr = 0.0;
    for (int r = 0; r < 10; ++r) {
      double f = 0, j0 = 0, j1 = 0, j2 = 0;
      for (int k = 0; k < 20; ++k) { f += M0[r][k] * m[k]; j0 += M0[r][k] * dx[k]; j1 += M0[r][k] * dy[k]; j2 += M0[r][k] * dz[k]; }
      const double j[3] = {j0, j1, j2};
      for (int a = 0; a < 3; ++a) { Jtr[a] += j[a] * f; for (int b = 0; b < 3; ++b) JtJ[a][b] += j[a] * j[b]; }
      rr += f * f;
    }
    if (rr == 0.0) return;
    // solve JtJ d = Jtr (3x3, Cramer)
    const double det = JtJ[0][0] * (JtJ[1][1] * JtJ[2][2] - JtJ[1][2] * JtJ[2][1]) - JtJ[0][1] * (JtJ[1][0] * JtJ[2][2] - JtJ[1][2] * JtJ[2][0]) +
                       JtJ[0][2] * (JtJ[1][0] * JtJ[2][1] - JtJ[1][1] * JtJ[2][0]);
    if (!(fabs(det) > 1e-300)) return;
    double d[3];
    for (int c = 0; c < 3; ++c) {
      double A[3][3];
      for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) A[a][b] = (b == c) ? Jtr[a] : JtJ[a][b];
      d[c] = (A[0][0] * (A[1][1] * A[2][2] - A[1][2] * A[2][1]) - A[0][1] * (A[1][0] * A[2][2] - A[1][2] * A[2][0]) +
              A[0][2] * (A[1][0] * A[2][1] - A[1][1] * A[2][0])) / det;
    }
    const double nx = *x - d[0], ny = *y - d[1], nz = *z - d[2];
    if (!(nx == nx) || !(ny == ny) || !(nz == nz)) return;
    // accept only if the residual does not grow
    double m2[20], t0[20], t1[20], t2[20], rr2 = 0.0;
    monomials(nx, ny, nz, m2, t0, t1, t2);
    for (int r = 0; r < 10; ++r) { double f = 0; for (int k = 0; k < 20; ++k) f += M0[r][k] * m2[k]; rr2 += f * f; }
    if (!(rr2 <= rr)) return;
    *x = nx; *y = ny; *z = nz;
  }
}

// One real root z of the degree-n polynomial -> the essential matrix of that solution (row-major, Frobenius-normalised);
// false if the root is complex / degenerate (the cases OpenCV skips).
DFVO_HD bool candidate_from_root(double zr, double zi, const double* c, int n, const double bx[3][4], const double by[3][4],
                                 const double b1[3][5], const double M0[10][20], const double basis[4][9], double* E) {
  if (!(fabs(zi) <= 1e-10) || !(zr == zr)) return false;
  double z = zr;
  // polish the real root with two Newton steps on the real polynomial
  for (int it = 0; it < 2; ++it) {
    double p = c[n], dp = 0.0;
    for (int k = n - 1; k >= 0; --k) { dp = dp * z + p; p = p * z + c[k]; }
    if (dp != 0.0) { double zn = z - p / dp; if (zn == zn && fabs(zn - z) < 1e-3 * (1.0 + fabs(z))) z = zn; }
  }
  const double z2 = z * z, z3 = z2 * z, z4 = z3 * z;
  double B[3][3];
  for (int j = 0; j < 3; ++j) {
    B[j][0] = bx[j][0] + bx[j][1] * z + bx[j][2] * z2 + bx[j][3] * z3;
    B[j][1] = by[j][0] + by[j][1] * z + by[j][2] * z2 + by[j][3] * z3;
    B[j][2] = b1[j][0] + b1[j][1] * z + b1[j][2] * z2 + b1[j][3] * z3 + b1[j][4] * z4;
  }
  // null vector of B: best of the three row cross products
  double best[3] = {0, 0, 0}, bn = -1.0;
  for (int a = 0; a < 3; ++a) {
    const int r0 = a, r1 = (a + 1) % 3;
    const double v0 = B[r0][1] * B[r1][2] - B[r0][2] * B[r1][1];
    const double v1 = B[r0][2] * B[r1][0] - B[r0][0] * B[r1][2];
    const double v2 = B[r0][0] * B[r1][1] - B[r0][1] * B[r1][0];
    const double nn = v0 * v0 + v1 * v1 + v2 * v2;
    if (nn > bn) { bn = nn; best[0] = v0; best[1] = v1; best[2] = v2; }
  }
  if (!(bn > 0.0)) return false;
  const double nrm = sqrt(bn);
  if (fabs(best[2]) < 1e-10 * nrm) return false;          // OpenCV: |xy1(2)| < 1e-10 on the unit null vector
  double x = best[0] / best[2], y = best[1] / best[2];
  refine(M0, &x, &y, &z);
  double fro = 0.0;
  for (int e = 0; e < 9; ++e) {
    E[e] = x * basis[0][e] + y * basis[1][e] + z * basis[2][e] + basis[3][e];
    fro += E[e] * E[e];
  }
  fro = sqrt(fro);
  if (!(fro > 0.0) || !(fro == fro)) return false;
  for (int e = 0; e < 9; ++e) E[e] /= fro;
  return true;
}

// Full solve.  x1, x2: 5 normalised points each ([5][2]).  E_out: up to 10 row-major 3x3 (x2^T E x1 = 0).
// Kept out of line: inlined into a kernel body, nvcc 12.9's optimiser for sm_90a produces wrong candidates for most
// samples (tests/test_gpu_depth_pose.py::test_five_point_vs_cv2; -G builds and the out-of-line call are correct).
static DFVO_HD_NOINLINE int solve(const double* x1, const double* x2, double* E_out) {
  double basis[4][9];
  if (!null_space(x1, x2, basis)) return 0;
  double M[10][20], M0[10][20];
  constraint_matrix(basis, M);
  for (int r = 0; r < 10; ++r) for (int k = 0; k < 20; ++k) M0[r][k] = M[r][k];
  if (!gauss_jordan(M)) return 0;
  double bx[3][4], by[3][4], b1[3][5], c[11];
  build_poly(M, bx, by, b1, c);
  // effective degree
  double cmax = 0.0;
  for (int k = 0; k <= 10; ++k) { double v = fabs(c[k]); if (v > cmax) cmax = v; }
  if (!(cmax > 0.0) || !(cmax == cmax) || cmax > 1e300) return 0;
  int n = 10;
  while (n > 0 && fabs(c[n]) <= 1e-14 * cmax) --n;
  if (n < 1) return 0;
  double re[10], im[10];
  durand_kerner(c, n, re, im, 160);
  int count = 0;
  for (int i = 0; i < n; ++i)
    if (candidate_from_root(re[i], im[i], c, n, bx, by, b1, M0, basis, E_out + 9 * count)) ++count;
  return count;
}


// =================================================================================================================
// Warp-cooperative variant: ten lanes per minimal sample (three samples per warp; lanes 30, 31 ride along idle).
// Same algorithm and the same per-element operation order as solve() above for the null space, the constraint rows, the
// Gauss-Jordan elimination (lane r owns row r; pivot search, row swap and pivot-row broadcast through shuffles) and the
// candidate extraction (lane i owns root i).  The Durand-Kerner sweep keeps OpenCV's Gauss-Seidel semantics -- root i is
// corrected with the already corrected roots j < i and the old roots j > i -- as a wavefront: every lane evaluates its Horner
// numerator and the old-root part of its denominator in parallel, then the ten corrections are finalised in index order, each
// broadcast to the lanes behind it.  Only the multiplication order inside the denominator product differs from solve()
// (old-root factors first), i.e. round-off of the correction, not the iteration: same roots, same index order.
// One thread per sample takes ~450 us for a single solve (a dependent chain of ~10^5 FP64 operations); ten lanes cut the
// chain by the width of the sweep and of the per-root refinement.
// Control flow is uniform across the warp (finished groups keep shuffling, masked), so full-mask shuffles are legal and the
// CPU emulation of the test build -- which needs every thread of a block to execute the same shuffle sequence -- runs it too.
// =================================================================================================================
#if defined(__CUDACC__) || defined(DFVO_HOSTSIM)
struct CoopShared {
  double M0[10][20];      // original constraint rows (the refinement's residuals)
  double R[10][10];       // right-hand halves of the eliminated rows
};

DFVO_D double coop_shfl(double v, int src) { return __shfl_sync(0xffffffffu, v, src); }

// l: lane inside the group (0..9 active, >= 10 idle), gbase: warp lane of the group's lane 0, live: this group has a sample.
// Every lane must pass the points of ITS group's sample (idle lanes: any valid sample).  Returns the candidate count of the
// group; E_out [10][9] receives them in root-index order (written by the owning lanes).
DFVO_D int solve_coop(const double* x1, const double* x2, CoopShared* sm, int l, int gbase, bool live, double* E_out) {
  const bool act = l < 10;
  double basis[4][9];
  bool ok = null_space(x1, x2, basis) && live;
  double row[20];
  {
    double E[9][4], EEt[9][10], tr[10];
    constraint_prep(basis, E, EEt, tr);
    constraint_row(E, EEt, tr, act ? l : 0, row);
  }
  if (act) for (int k = 0; k < 20; ++k) sm->M0[l][k] = row[k];
  // ---- Gauss-Jordan with partial pivoting, lane r = physical row r
  for (int c = 0; c < 10; ++c) {
    const double mine = fabs(row[c]);
    int piv = c;
    double best = coop_shfl(mine, gbase + c);
    for (int r = c + 1; r < 10; ++r) {
      const double v = coop_shfl(mine, gbase + r);
      if (v > best) { best = v; piv = r; }
    }
    if (best < 1e-300) ok = false;
    // swap rows c <-> piv (no-op when piv == c), columns c..19
    const int partner = gbase + (l == c ? piv : (l == piv ? c : (act ? l : 0)));
    for (int k = 0; k < 20; ++k) {
      const double o = coop_shfl(row[k], partner);
      if (k >= c && act) row[k] = o;
    }
    if (l == c) {
      const double inv = 1.0 / row[c];
      for (int k = c; k < 20; ++k) row[k] *= inv;
    }
    const double f = row[c];
    for (int k = c; k < 20; ++k) {
      const double pk = coop_shfl(row[k], gbase + c);
      if (act && l != c && f != 0.0) row[k] -= f * pk;
    }
  }
  if (act) for (int k = 0; k < 10; ++k) sm->R[l][k] = row[10 + k];
#ifdef DFVO_HOSTSIM
  __syncthreads();          // the emulation runs a block's threads as fibers: only a barrier orders the shared-memory hand-over
#else
  __syncwarp();
#endif
  double bx[3][4], by[3][4], b1[3][5], c[11];
  build_poly_rows(&sm->R[0][0], 10, bx, by, b1, c);
  double cmax = 0.0;
  for (int k = 0; k <= 10; ++k) { double v = fabs(c[k]); if (v > cmax) cmax = v; }
  if (!(cmax > 0.0) || !(cmax == cmax) || cmax > 1e300) ok = false;
  int n = 10;
  while (n > 0 && fabs(c[n]) <= 1e-14 * cmax) --n;
  if (n < 1) { ok = false; n = 1; }
  // ---- Durand-Kerner wavefront
  double zr, zi;
  {
    double pr = 1.0, pi = 0.0;                       // initial guesses p = (1,0) * (1,1)^i
    for (int i = 0; i < (act ? l : 0); ++i) { const double nr = pr - pi, ni = pr + pi; pr = nr; pi = ni; }
    zr = pr; zi = pi;
  }
  const bool root = act && l < n;
  DkStop stop;
  bool done = !ok;
  for (int iter = 0; iter < 160; ++iter) {
    // any group of the warp still iterating?
    const int d0 = __shfl_sync(0xffffffffu, (int)done, 0), d1 = __shfl_sync(0xffffffffu, (int)done, 10), d2 = __shfl_sync(0xffffffffu, (int)done, 20);
    if (d0 && d1 && d2) break;
    const double xr = zr, xi = zi;
    // Horner numerator of the own root and the old-root factors j > l of the denominator
    double nr = c[n], ni = 0.0, dr = c[n], di = 0.0;
    for (int j = 0; j < 10; ++j) {
      const double orj = coop_shfl(zr, gbase + j), oij = coop_shfl(zi, gbase + j);
      if (j < n) {
        const double tr = nr * xr - ni * xi + c[n - j - 1], ti = nr * xi + ni * xr;   // num = num * p + c[n-j-1]
        nr = tr; ni = ti;
        if (j > l) {
          const double er = xr - orj, ei = xi - oij;
          if (er != 0.0 || ei != 0.0) { const double ur = dr * er - di * ei, ui = dr * ei + di * er; dr = ur; di = ui; }
        }
      }
    }
    // corrections in index order; the new root i reaches the lanes behind it
    double ad = 0.0;
    for (int i = 0; i < 10; ++i) {
      if (l == i && root) {
        const double den = dr * dr + di * di;
        double qr = 0.0, qi = 0.0;
        if (den > 0.0) { qr = (nr * dr + ni * di) / den; qi = (ni * dr - nr * di) / den; }   // num /= denom
        if (!done) { zr = xr - qr; zi = xi - qi; }
        ad = sqrt(qr * qr + qi * qi);
      }
      const double nzr = coop_shfl(zr, gbase + i), nzi = coop_shfl(zi, gbase + i);
      if (root && l > i && i < n) {
        const double er = xr - nzr, ei = xi - nzi;
        if (er != 0.0 || ei != 0.0) { const double ur = dr * er - di * ei, ui = dr * ei + di * er; dr = ur; di = ui; }
      }
    }
    double max_diff = 0.0, rmax = 0.0;
    const double mag = fabs(zr) + fabs(zi);
    for (int j = 0; j < 10; ++j) {
      const double a = coop_shfl(ad, gbase + j), m = coop_shfl(mag, gbase + j);
      if (j < n) { if (a > max_diff) max_diff = a; if (m > rmax) rmax = m; }
    }
    if (!done && stop.done(max_diff, rmax)) done = true;
  }
  // ---- one candidate per real root, emitted in root-index order
  double Ec[9];
  const bool have = ok && root && candidate_from_root(zr, zi, c, n, bx, by, b1, sm->M0, basis, Ec);
  const unsigned bal = __ballot_sync(0xffffffffu, have ? 1 : 0);
  const unsigned grp = (bal >> gbase) & 0x3ffu;
  if (have) {
    const int pos = __popc(grp & ((1u << l) - 1u));
    for (int e = 0; e < 9; ++e) E_out[9 * pos + e] = Ec[e];
  }
  return __popc(grp);
}
#endif

}  // namespace fivept
}  // namespace dfvo
