// Essential-matrix RANSAC on the device, reproducing cv2.findEssentialMat + cv2.recoverPose as the
// reference calls them (E_tracker.py:223-296; OpenCV calib3d ptsetreg.cpp / five-point.cpp, SURVEY
// Appendix C): "parallel-evaluate / sequential-replay".
//   1. the 5-point subsets OpenCV would draw depend only on N (its RNG is re-seeded per call); the
//      host supplies that table (b200/cvrng.py) and the permutations drawn from the host np.random;
//   2. k_hypotheses: one thread per (repeat, iteration) solves the 5-point problem (fivept.cuh, FP64);
//   3. k_score: one warp per candidate counts Sampson inliers over all N correspondences (FP64);
//   4. k_replay: one thread per repeat walks the iterations in order applying OpenCV's acceptance rule
//      (strict >, first-found wins) and adaptive iteration count, i.e. finds the candidate OpenCV
//      would return and where it would stop;
//   5. k_finalize: inlier mask + GRIC-E residual sum (gric.py:14-37,94-132) of each repeat's winner;
//   6. k_recover_pose_vote / _pick: decomposeEssentialMat + 4 x triangulation + cheirality vote.
// All arithmetic is FP64 (inlier decisions are threshold tests, SURVEY H1).
#include <stdlib.h>

#include "fivept.cuh"
#include "ops.h"
#include "ransac.h"
#include "smallmat.cuh"

namespace dfvo {

// ---------------------------------------------------------------------------------------------
// stage kernels
// ---------------------------------------------------------------------------------------------
__global__ void k_five_point(const double* __restrict__ x1, const double* __restrict__ x2, int M, double* __restrict__ E,
                             int32_t* __restrict__ n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  double a[10], b[10], e[90];
  for (int k = 0; k < 10; ++k) { a[k] = x1[i * 10 + k]; b[k] = x2[i * 10 + k]; }
  int c = fivept::solve(a, b, e);
  n[i] = c;
  for (int k = 0; k < 90; ++k) E[(size_t)i * 90 + k] = k < 9 * c ? e[k] : 0.0;
}

int five_point(const double* x1, const double* x2, int M, double* E, int32_t* n, cudaStream_t s) {
  DFVO_LAUNCH(k_five_point, dim3(cdiv(M, 64)), dim3(64), 0, s, x1, x2, M, E, n);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

DFVO_D double sampson(const double* E, double u1, double v1, double u2, double v2) {
  // EMEstimatorCallback::computeError: x2^T E x1 squared over the four gradient terms
  const double a0 = E[0] * u1 + E[1] * v1 + E[2];
  const double a1 = E[3] * u1 + E[4] * v1 + E[5];
  const double a2 = E[6] * u1 + E[7] * v1 + E[8];
  const double b0 = E[0] * u2 + E[3] * v2 + E[6];
  const double b1 = E[1] * u2 + E[4] * v2 + E[7];
  const double x2tEx1 = u2 * a0 + v2 * a1 + a2;
  return x2tEx1 * x2tEx1 / (a0 * a0 + a1 * a1 + b0 * b0 + b1 * b1);
}

// one warp per candidate; counts[m] = #{ i : sampson(E_m, x1_i, x2_i) <= thr2 }.  perm (optional) maps
// slot -> original point index per repeat (repeat = m / cand_per_repeat).
__global__ void __launch_bounds__(256)
k_score(const double* __restrict__ E, const int32_t* __restrict__ valid, int M, const double* __restrict__ x1,
        const double* __restrict__ x2, int N, double thr2, int32_t* __restrict__ counts) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= M) return;
  if (valid && !valid[warp]) { if (lane == 0) counts[warp] = 0; return; }
  double e[9];
  for (int k = 0; k < 9; ++k) e[k] = E[(size_t)warp * 9 + k];
  int c = 0;
  for (int i = lane; i < N; i += 32) {
    double err = sampson(e, x1[2 * i], x1[2 * i + 1], x2[2 * i], x2[2 * i + 1]);
    c += (err <= thr2) ? 1 : 0;
  }
  for (int off = 16; off > 0; off >>= 1) c += __shfl_xor_sync(0xffffffffu, c, off);
  if (lane == 0) counts[warp] = c;
}

int score_hypotheses(const double* E, int M, const double* x1, const double* x2, int N, double thr2, int32_t* counts,
                     cudaStream_t s) {
  DFVO_LAUNCH(k_score, dim3(cdiv(M * 32, 256)), dim3(256), 0, s, E, (const int32_t*)nullptr, M, x1, x2, N, thr2, counts);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

// ---------------------------------------------------------------------------------------------
// fused pipeline
// ---------------------------------------------------------------------------------------------
struct EssState {          // one per repeat, device memory
  int32_t niters, best_good, best_iter, best_cand, it, done, evaluated, pad;
};

// x1n/x2n [R][N][2]: normalised AND permuted points of each repeat
__global__ void k_normalize_perm(const double* __restrict__ p1, const double* __restrict__ p2, const int32_t* __restrict__ perm,
                                 int N, double focal, double cx, double cy, double* __restrict__ x1n, double* __restrict__ x2n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x, r = blockIdx.y;
  if (i >= N) return;
  int src = perm ? perm[(size_t)r * N + i] : i;
  size_t o = ((size_t)r * N + i) * 2;
  x1n[o] = (p1[2 * src] - cx) / focal; x1n[o + 1] = (p1[2 * src + 1] - cy) / focal;
  x2n[o] = (p2[2 * src] - cx) / focal; x2n[o + 1] = (p2[2 * src + 1] - cy) / focal;
}

__global__ void k_ess_init(EssState* st, int R, int max_iters) {
  int r = threadIdx.x;
  if (r < R) { st[r].niters = max_iters; st[r].best_good = -1; st[r].best_iter = -1; st[r].best_cand = -1; st[r].it = 0; st[r].done = 0; st[r].evaluated = 0; }
}

__global__ void k_hypotheses(const double* __restrict__ x1n, const double* __restrict__ x2n, const int32_t* __restrict__ subsets,
                             int N, int i0, int i1, const EssState* __restrict__ st, double* __restrict__ Ecand,
                             int32_t* __restrict__ ncand, int max_iters) {
  int i = i0 + blockIdx.x * blockDim.x + threadIdx.x, r = blockIdx.y;
  if (i >= i1) return;
  if (st[r].done) return;
  double a[10], b[10], e[90];
  for (int k = 0; k < 5; ++k) {
    int s = subsets[i * 5 + k];
    size_t o = ((size_t)r * N + s) * 2;
    a[2 * k] = x1n[o]; a[2 * k + 1] = x1n[o + 1];
    b[2 * k] = x2n[o]; b[2 * k + 1] = x2n[o + 1];
  }
  int c = fivept::solve(a, b, e);
  size_t h = (size_t)r * max_iters + i;
  ncand[h] = c;
  for (int k = 0; k < 9 * c; ++k) Ecand[h * 90 + k] = e[k];
}

// Warp-cooperative hypothesis generation (fivept::solve_coop): ten lanes per minimal sample, three samples per warp.
#ifdef DFVO_HOSTSIM
#define HYP_WARPS 1          // the CPU emulation pays per shuffle and per thread of the block
#else
#define HYP_WARPS 4
#endif
__global__ void __launch_bounds__(HYP_WARPS * 32)
k_hypotheses_coop(const double* __restrict__ x1n, const double* __restrict__ x2n, const int32_t* __restrict__ subsets, int N, int i0, int i1,
                  const EssState* __restrict__ st, double* __restrict__ Ecand, int32_t* __restrict__ ncand, int max_iters) {
  __shared__ fivept::CoopShared sm[HYP_WARPS * 3];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, r = blockIdx.y;
  if (st[r].done) return;                                  // uniform per block
  int g = lane / 10, l = lane - 10 * g;
  if (g == 3) { g = 2; l += 10; }                           // lanes 30, 31 ride along with the third group
  int i = i0 + (blockIdx.x * HYP_WARPS + warp) * 3 + g;
  const bool live = i < i1;
  if (!live) i = i1 - 1;                                    // duplicate work on a valid sample, results discarded
  double a[10], b[10];
  for (int k = 0; k < 5; ++k) {
    const int s = subsets[i * 5 + k];
    const size_t o = ((size_t)r * N + s) * 2;
    a[2 * k] = x1n[o]; a[2 * k + 1] = x1n[o + 1];
    b[2 * k] = x2n[o]; b[2 * k + 1] = x2n[o + 1];
  }
  const size_t h = (size_t)r * max_iters + i;
  // dead groups write nowhere: E_out is only dereferenced by lanes whose candidate exists (live is folded into `ok`)
  const int c = fivept::solve_coop(a, b, &sm[warp * 3 + g], l, 10 * g, live, Ecand + h * 90);
  if (live && l == 0) ncand[h] = c;
}

__global__ void __launch_bounds__(256)
k_score_round(const double* __restrict__ Ecand, const int32_t* __restrict__ ncand, const double* __restrict__ x1n,
              const double* __restrict__ x2n, int N, int i0, int i1, double thr2, const EssState* __restrict__ st,
              int32_t* __restrict__ counts, int max_iters) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, r = blockIdx.y;
  const int i = i0 + w / 10, k = w % 10;
  if (i >= i1) return;
  if (st[r].done) return;
  size_t h = (size_t)r * max_iters + i;
  if (k >= ncand[h]) return;
  double e[9];
  for (int q = 0; q < 9; ++q) e[q] = Ecand[h * 90 + 9 * k + q];
  const double* a = x1n + (size_t)r * N * 2;
  const double* b = x2n + (size_t)r * N * 2;
  int c = 0;
  for (int j = lane; j < N; j += 32) c += (sampson(e, a[2 * j], a[2 * j + 1], b[2 * j], b[2 * j + 1]) <= thr2) ? 1 : 0;
  for (int off = 16; off > 0; off >>= 1) c += __shfl_xor_sync(0xffffffffu, c, off);
  if (lane == 0) counts[h * 10 + k] = c;
}

DFVO_HD int ransac_update_num_iters(double p, double ep, int model_points, int max_iters) {
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
  double q = num / denom;
  return (int)rint(q);           // cvRound: round half to even
}

__global__ void k_replay(const int32_t* __restrict__ ncand, const int32_t* __restrict__ counts, int N, int i1, double prob,
                         EssState* st, int max_iters, int R) {
  int r = threadIdx.x + blockIdx.x * blockDim.x;
  if (r >= R) return;
  EssState s = st[r];
  if (s.done) return;
  int it = s.it;
  while (it < s.niters && it < i1) {
    size_t h = (size_t)r * max_iters + it;
    int nc = ncand[h];
    for (int k = 0; k < nc; ++k) {
      int good = counts[h * 10 + k];
      int lim = s.best_good > 4 ? s.best_good : 4;
      if (good > lim) {
        s.best_good = good; s.best_iter = it; s.best_cand = k;
        s.niters = ransac_update_num_iters(prob, (double)(N - good) / (double)N, 5, s.niters);
      }
    }
    ++it;
  }
  s.it = it;
  s.evaluated = i1;
  if (it >= s.niters) s.done = 1;
  st[r] = s;
}

// Warp version of k_replay (one warp per repeat): the acceptance rule is sequential only through the running best, so each lane
// loads one iteration's candidate counts (max and its first index) -- 32 iterations per round trip to memory instead of one --
// and the warp then applies, in iteration order, only the iterations that beat the running best (a handful).  Same state
// transitions as k_replay: within an iteration the first candidate with the largest count wins, and niters after several
// improvements equals RANSACUpdateNumIters of the last one (it only ever shrinks with the inlier ratio).
__global__ void __launch_bounds__(32)
k_replay_warp(const int32_t* __restrict__ ncand, const int32_t* __restrict__ counts, int N, int i1, double prob, EssState* st, int max_iters) {
  const int r = blockIdx.x, lane = threadIdx.x;
  EssState s = st[r];
  if (s.done) return;
  int it = s.it;
  while (it < s.niters && it < i1) {
    const int mine = it + lane;
    int m = -1, mk = -1;
    if (mine < i1) {
      const size_t h = (size_t)r * max_iters + mine;
      const int nc = ncand[h];
      for (int k = 0; k < nc; ++k) { const int g = counts[h * 10 + k]; if (g > m) { m = g; mk = k; } }
    }
    int from = 0;                                             // lanes below `from` are settled
    while (true) {
      const int lim = s.best_good > 4 ? s.best_good : 4;
      const int upto = (s.niters < i1 ? s.niters : i1) - it;   // iterations of this batch that OpenCV would still run
      const unsigned cand = __ballot_sync(0xffffffffu, lane >= from && lane < upto && m > lim);
      if (!cand) break;
      const int j = __ffs(cand) - 1;
      const int good = __shfl_sync(0xffffffffu, m, j), k = __shfl_sync(0xffffffffu, mk, j);
      // within the winning iteration candidates are visited in order: the first one that beats the running best may be an earlier,
      // smaller one -- but every later strictly larger one replaces it, so the iteration ends on its maximum (first occurrence)
      s.best_good = good; s.best_iter = it + j; s.best_cand = k;
      s.niters = ransac_update_num_iters(prob, (double)(N - good) / (double)N, 5, s.niters);
      from = j + 1;
    }
    const int upto = (s.niters < i1 ? s.niters : i1) - it;
    it += upto < 32 ? (upto > 0 ? upto : 0) : 32;
    if (upto <= 0) break;
  }
  if (lane == 0) {
    s.it = it;
    s.evaluated = i1;
    if (it >= s.niters) s.done = 1;
    st[r] = s;
  }
}

// mask of the winner in ORIGINAL point order (E_tracker.py:278-285 un-permutes), GRIC-E (gric.py), counts.
// out per repeat: E[9], info[4] = {inlier count, iterations, best_iter, best_cand}, gric
__global__ void __launch_bounds__(256)
k_finalize(const double* __restrict__ Ecand, const EssState* __restrict__ st, const double* __restrict__ x1n,
           const double* __restrict__ x2n, const int32_t* __restrict__ perm, const double* __restrict__ p1,
           const double* __restrict__ p2, int N, double thr2, double fx, double fy, double cx, double cy, int max_iters,
           double* __restrict__ E_out, uint8_t* __restrict__ mask_out, int32_t* __restrict__ info, double* __restrict__ gric) {
  __shared__ double red[256];
  const int r = blockIdx.x, t = threadIdx.x;
  const EssState s = st[r];
  double e[9];
  const bool have = s.best_iter >= 0;
  if (have) for (int q = 0; q < 9; ++q) e[q] = Ecand[((size_t)r * max_iters + s.best_iter) * 90 + 9 * s.best_cand + q];
  else for (int q = 0; q < 9; ++q) e[q] = 0.0;
  // F = K^-T E K^-1 (E_tracker.py:261-262); K = [[fx,0,cx],[0,fy,cy],[0,0,1]]
  double F[9];
  {
    // K^-1 = [[1/fx,0,-cx/fx],[0,1/fy,-cy/fy],[0,0,1]]
    const double ki[9] = {1.0 / fx, 0.0, -cx / fx, 0.0, 1.0 / fy, -cy / fy, 0.0, 0.0, 1.0};
    double T[9];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { double a = 0; for (int k = 0; k < 3; ++k) a += e[3 * i + k] * ki[3 * k + j]; T[3 * i + j] = a; }
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { double a = 0; for (int k = 0; k < 3; ++k) a += ki[3 * k + i] * T[3 * k + j]; F[3 * i + j] = a; }
  }
  const double* a = x1n + (size_t)r * N * 2;
  const double* b = x2n + (size_t)r * N * 2;
  double gsum = 0.0;
  const double sigmasq1 = 1.0 / (0.8 * 0.8), lam3RD = 2.0 * (4 - 3);
  for (int j = t; j < N; j += 256) {
    int src = perm ? perm[(size_t)r * N + j] : j;
    bool inl = have && (sampson(e, a[2 * j], a[2 * j + 1], b[2 * j], b[2 * j + 1]) <= thr2);
    mask_out[(size_t)r * N + src] = inl ? 1 : 0;
    // compute_fundamental_residual(F, kp1=points1, kp2=points2) on pixel coordinates (gric.py:14-37)
    const double u1 = p1[2 * src], v1 = p1[2 * src + 1], u2 = p2[2 * src], v2 = p2[2 * src + 1];
    const double f0 = F[0] * u1 + F[1] * v1 + F[2], f1 = F[3] * u1 + F[4] * v1 + F[5], f2 = F[6] * u1 + F[7] * v1 + F[8];
    const double g0 = F[0] * u2 + F[3] * v2 + F[6], g1 = F[1] * u2 + F[4] * v2 + F[7];
    const double m = u2 * f0 + v2 * f1 + f2;
    const double res = m * m / (f0 * f0 + f1 * f1 + g0 * g0 + g1 * g1);
    const double tmp = res * sigmasq1;
    gsum += (tmp <= lam3RD) ? tmp : lam3RD;
  }
  red[t] = gsum;
  __syncthreads();
  for (int off = 128; off > 0; off >>= 1) { if (t < off) red[t] += red[t + off]; __syncthreads(); }
  if (t == 0) {
    // calc_GRIC(res, 0.8, n, 'EMat'): sum + n*D*log(R) + K*log(R*n), R=4, D=3, K=5
    gric[r] = red[0] + (double)N * 3.0 * log(4.0) + 5.0 * log(4.0 * (double)N);
    for (int q = 0; q < 9; ++q) E_out[r * 9 + q] = e[q];
    info[r * 4 + 0] = have ? s.best_good : 0; info[r * 4 + 1] = s.it; info[r * 4 + 2] = s.best_iter; info[r * 4 + 3] = s.best_cand;
  }
}

size_t essential_workspace_bytes(int N, int R, int max_iters) {
  size_t b = 0;
  b += (size_t)R * N * 2 * 8 * 2;                 // x1n, x2n
  b += (size_t)R * max_iters * 90 * 8;            // candidates
  b += (size_t)R * max_iters * 4;                 // ncand
  b += (size_t)R * max_iters * 10 * 4;            // counts
  b += (size_t)R * sizeof(EssState);
  return b + 1024;
}

int essential_ransac(const double* p1, const double* p2, int N, const int32_t* perm, int R, const int32_t* subsets, int max_iters,
                     double fx, double fy, double cx, double cy, double threshold, double prob, void* workspace, size_t ws_bytes,
                     double* E_out, uint8_t* mask_out, int32_t* info, double* gric, cudaStream_t s) {
  DFVO_REQUIRE(N >= 5 && R >= 1 && R <= 32 && max_iters >= 1, DFVO_EINVAL, "essential_ransac args (N=%d R=%d)", N, R);
  DFVO_REQUIRE(ws_bytes >= essential_workspace_bytes(N, R, max_iters), DFVO_EINVAL, "essential_ransac workspace too small");
  uint8_t* w = reinterpret_cast<uint8_t*>(workspace);
  auto take = [&](size_t bytes) { uint8_t* p = w; w += (bytes + 127) & ~(size_t)127; return p; };
  double* x1n = (double*)take((size_t)R * N * 2 * 8);
  double* x2n = (double*)take((size_t)R * N * 2 * 8);
  double* Ecand = (double*)take((size_t)R * max_iters * 90 * 8);
  int32_t* ncand = (int32_t*)take((size_t)R * max_iters * 4);
  int32_t* counts = (int32_t*)take((size_t)R * max_iters * 10 * 4);
  EssState* st = (EssState*)take((size_t)R * sizeof(EssState));
  const double focal = fx;                                    // findEssentialMat(focal=fx, pp) (E_tracker.py:231-239)
  const double thr = threshold / focal, thr2 = thr * thr;
  DFVO_LAUNCH(k_normalize_perm, dim3(cdiv(N, 128), R), dim3(128), 0, s, p1, p2, perm, N, focal, cx, cy, x1n, x2n);
  DFVO_LAUNCH(k_ess_init, dim3(1), dim3(32), 0, s, st, R, max_iters);
  // rounds: most scenes stop within the first few dozen iterations; later rounds early-exit on st.done
  const int bounds[4] = {0, 48 < max_iters ? 48 : max_iters, 256 < max_iters ? 256 : max_iters, max_iters};
  for (int rd = 0; rd < 3; ++rd) {
    const int i0 = bounds[rd], i1 = bounds[rd + 1];
    if (i1 <= i0) continue;
    // DFVO_HYP_COOP=0 selects the one-thread-per-sample solver (read per call so a test can compare the two paths)
    const char* e_coop = getenv("DFVO_HYP_COOP");
    const int coop = !(e_coop && atoi(e_coop) == 0);
    if (coop)
      DFVO_LAUNCH(k_hypotheses_coop, dim3(cdiv(i1 - i0, HYP_WARPS * 3), R), dim3(HYP_WARPS * 32), 0, s, x1n, x2n, subsets, N, i0, i1, st, Ecand,
                  ncand, max_iters);
    else
      DFVO_LAUNCH(k_hypotheses, dim3(cdiv(i1 - i0, 32), R), dim3(32), 0, s, x1n, x2n, subsets, N, i0, i1, st, Ecand, ncand, max_iters);
    DFVO_LAUNCH(k_score_round, dim3(cdiv((i1 - i0) * 10 * 32, 256), R), dim3(256), 0, s, Ecand, ncand, x1n, x2n, N, i0, i1, thr2, st,
                counts, max_iters);
    DFVO_LAUNCH(k_replay_warp, dim3(R), dim3(32), 0, s, ncand, counts, N, i1, prob, st, max_iters);
  }
  DFVO_LAUNCH(k_finalize, dim3(R), dim3(256), 0, s, Ecand, st, x1n, x2n, perm, p1, p2, N, thr2, fx, fy, cx, cy, max_iters, E_out,
              mask_out, info, gric);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

// ---------------------------------------------------------------------------------------------
// cv2.recoverPose(E, points1, points2, focal, pp)  (E_tracker.py:292-295; five-point.cpp)
// decomposeEssentialMat, then every point is triangulated (4x4 DLT, smallest singular vector as in
// cv::triangulatePoints) against the four (R,t) candidates; cheirality masks in OpenCV's order; first
// maximum wins.  out: Rt[12] (R row-major then t), info[5] = {best count, c0..c3}.
// ---------------------------------------------------------------------------------------------
DFVO_D void triangulate_dlt(const double P1[3][4], double u0, double v0, double u1, double v1, double X[4]) {
  // rows of A (cvTriangulatePoints): x*P[2] - P[0], y*P[2] - P[1] for view 0 = [I|0] and view 1 = P1
  double A[4][4] = {{-1.0, 0.0, u0, 0.0}, {0.0, -1.0, v0, 0.0}, {0, 0, 0, 0}, {0, 0, 0, 0}};
  for (int k = 0; k < 4; ++k) { A[2][k] = u1 * P1[2][k] - P1[0][k]; A[3][k] = v1 * P1[2][k] - P1[1][k]; }
  double AtA[4][4], V[4][4], w[4];
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) { double a = 0; for (int k = 0; k < 4; ++k) a += A[k][i] * A[k][j]; AtA[i][j] = a; }
  sm::jacobi_eig<4>(AtA, V, w);
  int m = 0;
  for (int i = 1; i < 4; ++i) if (w[i] < w[m]) m = i;
  for (int i = 0; i < 4; ++i) X[i] = V[i][m];
}

// decomposeEssentialMat: R candidates U W Vt / U W^T Vt and t = U[:,2]
DFVO_D void decompose_essential(const double* __restrict__ Eptr, double R[2][3][3], double tv[3]) {
  double E[3][3], U[3][3], s[3], Vt[3][3];
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) E[i][j] = Eptr[3 * i + j];
  sm::svd3_rank2(E, U, s, Vt);
  if (sm::det3(U) < 0) for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) U[i][j] = -U[i][j];
  if (sm::det3(Vt) < 0) for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) Vt[i][j] = -Vt[i][j];
  const double W[3][3] = {{0, 1, 0}, {-1, 0, 0}, {0, 0, 1}};
  for (int which = 0; which < 2; ++which) {
    double T[3][3];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) {
      double a = 0;
      for (int k = 0; k < 3; ++k) a += U[i][k] * (which == 0 ? W[k][j] : W[j][k]);
      T[i][j] = a;
    }
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) {
      double a = 0;
      for (int k = 0; k < 3; ++k) a += T[i][k] * Vt[k][j];
      R[which][i][j] = a;
    }
  }
  for (int i = 0; i < 3; ++i) tv[i] = U[i][2];
}

// Cheirality test of point j under candidate k (recoverPose's triangulate + depth checks).
DFVO_D bool cheirality_ok(const double (*sR)[3][3], const double* st, int k, const double* __restrict__ p1, const double* __restrict__ p2,
                          int j, double focal, double cx, double cy, double dist) {
  const double u0 = (p1[2 * j] - cx) / focal, v0 = (p1[2 * j + 1] - cy) / focal;
  const double u1 = (p2[2 * j] - cx) / focal, v1 = (p2[2 * j + 1] - cy) / focal;
  double P[3][4];
  const double sg = k < 2 ? 1.0 : -1.0;
  for (int a = 0; a < 3; ++a) { for (int b = 0; b < 3; ++b) P[a][b] = sR[k & 1][a][b]; P[a][3] = sg * st[a]; }
  double X[4];
  triangulate_dlt(P, u0, v0, u1, v1, X);
  bool m = (X[2] * X[3]) > 0;
  const double x = X[0] / X[3], y = X[1] / X[3], z = X[2] / X[3];
  m = m && (z < dist);
  const double z2 = P[2][0] * x + P[2][1] * y + P[2][2] * z + P[2][3];
  return m && (z2 > 0) && (z2 < dist);
}

// Pass 1: one thread per (point, candidate) -- the 4 candidates of a point sit in adjacent lanes.  Every block
// repeats the (tiny) decomposition instead of waiting for a producer kernel.  mask_out[j] receives the 4-bit
// candidate field, info[1+k] the cheirality count of candidate k (atomics; info zeroed by the caller).
__global__ void __launch_bounds__(256)
k_recover_pose_vote(const double* __restrict__ Eptr, const double* __restrict__ p1, const double* __restrict__ p2, int N, double focal,
                    double cx, double cy, double dist, uint8_t* __restrict__ mask_out, int32_t* __restrict__ info) {
  __shared__ double sR[2][3][3], st[3];
  __shared__ int cnt[4];
  const int t = threadIdx.x;
  if (t == 0) decompose_essential(Eptr, sR, st);
  if (t < 4) cnt[t] = 0;
  __syncthreads();
  const int g = blockIdx.x * 256 + t, j = g >> 2, k = g & 3;
  const bool m = j < N && cheirality_ok(sR, st, k, p1, p2, j, focal, cx, cy, dist);
  const unsigned ballot = __ballot_sync(0xffffffffu, m);
  const int lane = t & 31;
  if (j < N && k == 0) mask_out[j] = (uint8_t)((ballot >> lane) & 0xfu);
  if (lane < 4) {                                  // lane k sums candidate k over the warp's 8 points
    const int c = __popc(ballot & (0x11111111u << lane));
    if (c) atomicAdd(&cnt[lane], c);
  }
  __syncthreads();
  if (t < 4 && cnt[t]) atomicAdd(&info[1 + t], cnt[t]);
}

// Pass 2: first maximum wins (OpenCV's order); resolve the bit-field to the winner's mask; block 0 writes R|t.
__global__ void __launch_bounds__(256)
k_recover_pose_pick(const double* __restrict__ Eptr, int N, double* __restrict__ Rt_out, uint8_t* __restrict__ mask_out,
                    int32_t* __restrict__ info) {
  int b = 0;
  for (int k = 1; k < 4; ++k) if (info[1 + k] > info[1 + b]) b = k;
  const int j = blockIdx.x * 256 + threadIdx.x;
  if (j < N) mask_out[j] = (mask_out[j] >> b) & 1u;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    double R[2][3][3], tv[3];
    decompose_essential(Eptr, R, tv);
    for (int a = 0; a < 3; ++a) for (int q = 0; q < 3; ++q) Rt_out[3 * a + q] = R[b & 1][a][q];
    for (int a = 0; a < 3; ++a) Rt_out[9 + a] = (b < 2 ? 1.0 : -1.0) * tv[a];
    info[0] = info[1 + b];
  }
}

__global__ void k_triangulate_depth(const double* __restrict__ x1, const double* __restrict__ x2, int N, const double* __restrict__ T21,
                                    double* __restrict__ depth2) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  double P[3][4];
  for (int a = 0; a < 3; ++a) for (int b = 0; b < 4; ++b) P[a][b] = T21[4 * a + b];
  double X[4];
  triangulate_dlt(P, x1[2 * i], x1[2 * i + 1], x2[2 * i], x2[2 * i + 1], X);
  const double x = X[0] / X[3], y = X[1] / X[3], z = X[2] / X[3];           // X /= X[3]  (ops_3d.py:64)
  depth2[i] = P[2][0] * x + P[2][1] * y + P[2][2] * z + P[2][3];             // X2 = T_2w[:3] @ X
}

// ops_3d.triangulation (ops_3d.py:44-67) for two general views: cv2.triangulatePoints(T_1w[:3], T_2w[:3], kp1, kp2) (the same 4x4 DLT,
// smallest singular vector), X /= X[3], X1 = T_1w[:3] @ X, X2 = T_2w[:3] @ X.  Outputs are [3][N] (any may be null).
__global__ void k_triangulate_points(const double* __restrict__ x1, const double* __restrict__ x2, int N, const double* __restrict__ T1w,
                                     const double* __restrict__ T2w, double* __restrict__ Xw, double* __restrict__ X1, double* __restrict__ X2) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  double P0[3][4], P1[3][4];
  for (int a = 0; a < 3; ++a) for (int b = 0; b < 4; ++b) { P0[a][b] = T1w[4 * a + b]; P1[a][b] = T2w[4 * a + b]; }
  const double u0 = x1[2 * i], v0 = x1[2 * i + 1], u1 = x2[2 * i], v1 = x2[2 * i + 1];
  double A[4][4];
  for (int k = 0; k < 4; ++k) {
    A[0][k] = u0 * P0[2][k] - P0[0][k]; A[1][k] = v0 * P0[2][k] - P0[1][k];
    A[2][k] = u1 * P1[2][k] - P1[0][k]; A[3][k] = v1 * P1[2][k] - P1[1][k];
  }
  double AtA[4][4], V[4][4], w[4];
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) { double a = 0; for (int k = 0; k < 4; ++k) a += A[k][r] * A[k][c]; AtA[r][c] = a; }
  sm::jacobi_eig<4>(AtA, V, w);
  int m = 0;
  for (int r = 1; r < 4; ++r) if (w[r] < w[m]) m = r;
  const double X[4] = {V[0][m] / V[3][m], V[1][m] / V[3][m], V[2][m] / V[3][m], 1.0};
  for (int a = 0; a < 3; ++a) {
    if (Xw) Xw[(size_t)a * N + i] = X[a];
    if (X1) X1[(size_t)a * N + i] = P0[a][0] * X[0] + P0[a][1] * X[1] + P0[a][2] * X[2] + P0[a][3];
    if (X2) X2[(size_t)a * N + i] = P1[a][0] * X[0] + P1[a][1] * X[1] + P1[a][2] * X[2] + P1[a][3];
  }
}

int triangulate_points(const double* x1, const double* x2, int N, const double* T1w, const double* T2w, double* Xw, double* X1, double* X2,
                       cudaStream_t s) {
  DFVO_LAUNCH(k_triangulate_points, dim3(cdiv(N, 128)), dim3(128), 0, s, x1, x2, N, T1w, T2w, Xw, X1, X2);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

int triangulate_depth(const double* x1, const double* x2, int N, const double* T21, double* depth2, cudaStream_t s) {
  DFVO_LAUNCH(k_triangulate_depth, dim3(cdiv(N, 128)), dim3(128), 0, s, x1, x2, N, T21, depth2);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

int recover_pose(const double* E, const double* p1, const double* p2, int N, double focal, double cx, double cy, double* Rt_out,
                 uint8_t* mask_out, int32_t* info, cudaStream_t s) {
  DFVO_CUDA(cudaMemsetAsync(info, 0, 5 * sizeof(int32_t), s));
  DFVO_LAUNCH(k_recover_pose_vote, dim3(cdiv(4 * N, 256)), dim3(256), 0, s, E, p1, p2, N, focal, cx, cy, 50.0, mask_out, info);
  DFVO_LAUNCH(k_recover_pose_pick, dim3(cdiv(N, 256)), dim3(256), 0, s, E, N, Rt_out, mask_out, info);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

// ------------------------------------------------------------------------------------------------
// Scale recovery: sklearn.linear_model.RANSACRegressor(LinearRegression(fit_intercept=False), min_samples, max_trials, stop_probability,
// residual_threshold).fit(ratio[:, None], ones) -> estimator_.coef_[0, 0]   (E_tracker.py:618-641), on the device, INCLUDING the host's
// random stream: the regressor draws its samples from NumPy's global MT19937 (sample_without_replacement -> RandomState.randint /
// permutation), and the reference's later shuffles continue from wherever it stopped -- so the kernel takes the generator's state
// (key[624], pos), walks it exactly as NumPy does (32-bit draws, masked rejection: random_interval / buffered_bounded_masked_uint32)
// and hands the advanced state back.  One block: thread 0 owns the generator and the accept / max_trials logic (sklearn's
// _ransac.py loop), the block evaluates the residuals |1 - s x| <= threshold of a trial in parallel.
// Arithmetic follows the NumPy expressions operation by operation (no FMA contraction) except the two long dot products of the
// final refit, which NumPy hands to BLAS (order of additions unspecified): the scale agrees to ~1e-15 relative.
// io (doubles): [0] scale, [1] status (1 ok, -1 no consensus), [2] trials run, [3] inliers of the best model, then key/pos as
// 625 uint32 starting at io + 4.
// ------------------------------------------------------------------------------------------------
struct Mt { uint32_t* key; int pos; };
DFVO_D void mt_regen(uint32_t* mt) {
  const uint32_t UP = 0x80000000u, LO = 0x7fffffffu, A = 0x9908b0dfu;
  int kk = 0;
  for (; kk < 624 - 397; ++kk) { const uint32_t y = (mt[kk] & UP) | (mt[kk + 1] & LO); mt[kk] = mt[kk + 397] ^ (y >> 1) ^ ((y & 1u) ? A : 0u); }
  for (; kk < 623; ++kk) { const uint32_t y = (mt[kk] & UP) | (mt[kk + 1] & LO); mt[kk] = mt[kk + (397 - 624)] ^ (y >> 1) ^ ((y & 1u) ? A : 0u); }
  const uint32_t y = (mt[623] & UP) | (mt[0] & LO);
  mt[623] = mt[396] ^ (y >> 1) ^ ((y & 1u) ? A : 0u);
}
DFVO_D uint32_t mt_next(Mt& g) {
  if (g.pos >= 624) { mt_regen(g.key); g.pos = 0; }
  uint32_t y = g.key[g.pos++];
  y ^= (y >> 11); y ^= (y << 7) & 0x9d2c5680u; y ^= (y << 15) & 0xefc60000u; y ^= (y >> 18);
  return y;
}
// numpy random_interval(max) / bounded masked uint32: uniform integer in [0, max]
DFVO_D uint32_t mt_interval(Mt& g, uint32_t max) {
  if (max == 0) return 0;
  uint32_t mask = max;
  mask |= mask >> 1; mask |= mask >> 2; mask |= mask >> 4; mask |= mask >> 8; mask |= mask >> 16;
  uint32_t v;
  do { v = mt_next(g) & mask; } while (v > max);
  return v;
}

#define SR_THREADS 256
#define SR_MAX_SAMPLES 16
__global__ void __launch_bounds__(SR_THREADS)
k_scale_ransac(const double* __restrict__ x, int n, int min_samples, int max_trials_in, double stop_prob, double thr, double* __restrict__ io,
               int32_t* __restrict__ perm_scratch, const double* __restrict__ n_dev, const double* __restrict__ gate) {
  // fused E-tracker tail: the sample count and the go / no-go decision live on the device (no generator draw when the gate is closed
  // or fewer than 11 depth ratios are valid, exactly where the reference does not call the regressor: E_tracker.py:617-643)
  if (gate != nullptr) {
    if (*gate == 0.0) {
      if (threadIdx.x == 0) { io[DFVO_TAIL_SCALE] = -1.0; io[DFVO_TAIL_STATUS] = -3.0; io[DFVO_TAIL_TRIALS] = 0.0; io[DFVO_TAIL_INLIERS] = 0.0; }
      return;
    }
    n = (int)*n_dev;
    if (n <= 10) {
      if (threadIdx.x == 0) { io[DFVO_TAIL_SCALE] = -1.0; io[DFVO_TAIL_STATUS] = -2.0; io[DFVO_TAIL_TRIALS] = 0.0; io[DFVO_TAIL_INLIERS] = 0.0; }
      return;
    }
  }
  __shared__ uint32_t key[624];
  __shared__ int idx[SR_MAX_SAMPLES];
  __shared__ int part_i[SR_THREADS / 32], part_nz[SR_THREADS / 32];
  __shared__ double part_d[2][SR_THREADS / 32];
  __shared__ double s_best_sh;
  __shared__ int go;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  uint32_t* st = reinterpret_cast<uint32_t*>(io + DFVO_TAIL_MT);
  for (int i = t; i < 624; i += SR_THREADS) key[i] = st[i];
  __syncthreads();
  Mt g; g.key = key; g.pos = (int)st[624];
  double max_trials = (double)max_trials_in;
  int n_trials = 0, n_best = 1, have = 0;
  double score_best = -1e300, s_best = 0.0;
  const double ratio = n > 0 ? (double)min_samples / (double)n : 1.0;
  while (true) {
    if (t == 0) {
      go = ((double)n_trials < max_trials) ? 1 : 0;
      if (go) {
        // sklearn.utils.random.sample_without_replacement(n, min_samples, method='auto') of scikit-learn 1.9 (hostmath.py docstring)
        if (ratio > 0.01 && ratio < 0.99) {                       // rng.permutation(n)[:k]: arange + legacy shuffle
          for (int i = 0; i < n; ++i) perm_scratch[i] = i;
          for (int i = n - 1; i >= 1; --i) {
            const int j = (int)mt_interval(g, (uint32_t)i);
            const int tmp = perm_scratch[i]; perm_scratch[i] = perm_scratch[j]; perm_scratch[j] = tmp;
          }
          for (int i = 0; i < min_samples; ++i) idx[i] = perm_scratch[i];
        } else if (ratio < 0.2) {                                 // tracking selection: rng.randint(n) until unseen
          for (int i = 0; i < min_samples; ++i) {
            int j;
            bool dup;
            do {
              j = (int)mt_interval(g, (uint32_t)(n - 1));
              dup = false;
              for (int q = 0; q < i; ++q) dup = dup || idx[q] == j;
            } while (dup);
            idx[i] = j;
          }
        } else {                                                  // reservoir sampling
          for (int i = 0; i < min_samples; ++i) idx[i] = i;
          for (int i = min_samples; i < n; ++i) {
            const int j = (int)mt_interval(g, (uint32_t)i);
            if (j < min_samples) idx[j] = i;
          }
        }
      }
    }
    __syncthreads();
    if (!go) break;
    ++n_trials;
    // LinearRegression(fit_intercept=False) on the sample: s = dot(x, y) / dot(x, x), y = 1
    double num = 0.0, den = 0.0;
    for (int i = 0; i < min_samples; ++i) { const double xi = x[idx[i]]; num = __dadd_rn(num, xi); den = __dadd_rn(den, __dmul_rn(xi, xi)); }
    const double s = den != 0.0 ? num / den : 0.0;
    int cnt = 0, nz = 0;
    for (int i = t; i < n; i += SR_THREADS) {
      const double r = __dsub_rn(1.0, __dmul_rn(s, x[i]));
      if (fabs(r) <= thr) { ++cnt; nz |= (r != 0.0) ? 1 : 0; }
    }
    for (int off = 16; off > 0; off >>= 1) { cnt += __shfl_xor_sync(0xffffffffu, cnt, off); nz |= __shfl_xor_sync(0xffffffffu, nz, off); }
    if (lane == 0) { part_i[warp] = cnt; part_nz[warp] = nz; }
    __syncthreads();
    int n_inl = 0, any_nz = 0;
    for (int w8 = 0; w8 < SR_THREADS / 32; ++w8) { n_inl += part_i[w8]; any_nz |= part_nz[w8]; }
    __syncthreads();                                              // part_* are rewritten by the next trial
    // _ransac.py: fewer inliers -> next; equal inliers and worse score -> next (score = r2 of the constant target: 1 if exact, else 0)
    if (n_inl < n_best) continue;
    const double score = any_nz ? 0.0 : 1.0;
    if (n_inl == n_best && score < score_best) continue;
    n_best = n_inl; score_best = score; s_best = s; have = 1;
    {
      const double eps = 2.220446049250313e-16;
      const double w = (double)n_best / (double)n;
      const double nom = fmax(eps, 1.0 - stop_prob), denom = fmax(eps, 1.0 - pow(w, (double)min_samples));
      double dyn;
      if (nom == 1.0) dyn = 0.0;
      else if (denom == 1.0) dyn = 1e300;
      else dyn = fabs(ceil(log(nom) / log(denom)));
      if (dyn < max_trials) max_trials = dyn;
    }
  }
  // final refit on the best consensus set
  double sx = 0.0, sxx = 0.0;
  int cnt = 0;
  if (have)
    for (int i = t; i < n; i += SR_THREADS) {
      const double xi = x[i];
      if (fabs(__dsub_rn(1.0, __dmul_rn(s_best, xi))) <= thr) { sx += xi; sxx += xi * xi; ++cnt; }
    }
  for (int off = 16; off > 0; off >>= 1) {
    sx += __shfl_xor_sync(0xffffffffu, sx, off); sxx += __shfl_xor_sync(0xffffffffu, sxx, off); cnt += __shfl_xor_sync(0xffffffffu, cnt, off);
  }
  if (lane == 0) { part_d[0][warp] = sx; part_d[1][warp] = sxx; part_i[warp] = cnt; }
  __syncthreads();
  if (t == 0) {
    double a = 0, b = 0; int c = 0;
    for (int w8 = 0; w8 < SR_THREADS / 32; ++w8) { a += part_d[0][w8]; b += part_d[1][w8]; c += part_i[w8]; }
    io[DFVO_TAIL_SCALE] = (have && b != 0.0) ? a / b : 0.0;
    io[DFVO_TAIL_STATUS] = have ? 1.0 : -1.0;
    io[DFVO_TAIL_TRIALS] = (double)n_trials;
    io[DFVO_TAIL_INLIERS] = (double)c;
    (void)s_best_sh;
  }
  __syncthreads();
  for (int i = t; i < 624; i += SR_THREADS) st[i] = key[i];
  if (t == 0) st[624] = (uint32_t)g.pos;
}

int scale_ransac(const double* ratio, int n, int min_samples, int max_trials, double stop_prob, double thr, double* io, int32_t* perm_scratch,
                 cudaStream_t s) {
  DFVO_REQUIRE(ratio && io && perm_scratch && n >= 1 && min_samples >= 1 && min_samples <= SR_MAX_SAMPLES && min_samples <= n && max_trials >= 0,
               DFVO_EINVAL, "scale_ransac args (n=%d min_samples=%d)", n, min_samples);
  DFVO_LAUNCH(k_scale_ransac, dim3(1), dim3(SR_THREADS), 0, s, ratio, n, min_samples, max_trials, stop_prob, thr, io, perm_scratch,
              (const double*)nullptr, (const double*)nullptr);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

// ------------------------------------------------------------------------------------------------
// Fused tail of the E-tracker (E_tracker.py:182-186,249-300 + dfvo.py:165-193 + E_tracker.py:476-507,571-643): everything between
// "the five RANSAC repeats are done" and "the host knows pose and scale" without a host round trip.  The validity method decides the
// pick: GRIC (h_gric != nullptr) or the flow magnitude (h_gric == nullptr; the caller took the gate mean flow > thre before it drew
// the shuffles).
//   k_recover_pose_counts  flow only: every repeat's recoverPose count (a count over all points, so the permutation drops out)
//   k_track_pick           GRIC: first repeat with the most inliers (E_tracker.py:278-281), its E, the per-repeat numbers as doubles
//   k_track_pick_flow      flow: first repeat with more inliers AND count > 0.05 n, the vote sum(count > 0.1 n) > R / 2
//   recover_pose           cv2.recoverPose on the best E (kernels above)
//   k_track_gate           GRIC: majority vote H_gric > E_gric (:286-290); cheirality > 0.1 n (:299-300), |t| != 0 (dfvo.py:182)
//                          -> gate; T_21 = inv([R|t])
//   k_scale_chain          find_scale_from_depth up to the regressor: normalise, triangulate, CNN depth at int(kp_cur),
//                          last-writer-wins per pixel, ratios in row-major pixel order (ops_3d.py:15-41, E_tracker.py:598-616)
//   k_scale_ransac         the regressor with the host generator's MT19937 state (above), gated
// res layout: DFVO_TAIL_* (include/dfvo_b200.h).
// ------------------------------------------------------------------------------------------------
// every repeat's four candidate counts in one launch: grid (cdiv(4N, 256), R), counts [R][4] zeroed by the caller
__global__ void __launch_bounds__(256)
k_recover_pose_counts(const double* __restrict__ E, const double* __restrict__ p1, const double* __restrict__ p2, int N, double focal,
                      double cx, double cy, double dist, int32_t* __restrict__ counts) {
  __shared__ double sR[2][3][3], st[3];
  __shared__ int cnt[4];
  const int t = threadIdx.x, r = blockIdx.y;
  if (t == 0) decompose_essential(E + 9 * r, sR, st);
  if (t < 4) cnt[t] = 0;
  __syncthreads();
  const int g = blockIdx.x * 256 + t, j = g >> 2, k = g & 3;
  const bool m = j < N && cheirality_ok(sR, st, k, p1, p2, j, focal, cx, cy, dist);
  const unsigned ballot = __ballot_sync(0xffffffffu, m);
  const int lane = t & 31;
  if (lane < 4) {
    const int c = __popc(ballot & (0x11111111u << lane));
    if (c) atomicAdd(&cnt[lane], c);
  }
  __syncthreads();
  if (t < 4 && cnt[t]) atomicAdd(&counts[4 * r + t], cnt[t]);
}

// what both pick rules store: the best repeat, info [R][4] as doubles, the best E (any finite E keeps the kernels benign when none)
DFVO_D void track_pick_store(const int32_t* __restrict__ info, const double* __restrict__ E, int R, int best, double* __restrict__ res,
                             double* __restrict__ E_best) {
  res[DFVO_TAIL_BEST] = (double)best;
  for (int q = 0; q < 4 * R; ++q) res[DFVO_TAIL_EGRIC + R + q] = (double)info[q];
  for (int q = 0; q < 9; ++q) E_best[q] = best >= 0 ? E[9 * best + q] : ((q % 4 == 0 && q < 8) ? 1.0 : 0.0);
}

__global__ void k_track_pick(const int32_t* __restrict__ info, const double* __restrict__ gric, const double* __restrict__ E, int R,
                             double* __restrict__ res, double* __restrict__ E_best) {
  if (threadIdx.x != 0) return;
  int best = -1, cnt = 0;
  for (int r = 0; r < R; ++r) {
    if (info[4 * r] > cnt) { best = r; cnt = info[4 * r]; }
    res[DFVO_TAIL_EGRIC + r] = gric[r];
  }
  track_pick_store(info, E, R, best, res, E_best);
}

__global__ void k_track_pick_flow(const int32_t* __restrict__ info, const int32_t* __restrict__ counts, const double* __restrict__ E, int R,
                                  int n, double* __restrict__ res, double* __restrict__ E_best) {
  if (threadIdx.x != 0) return;
  int best = -1, best_inl = 0, votes = 0;
  for (int r = 0; r < R; ++r) {
    int b = 0;                                                         // recoverPose keeps the first candidate with the most points
    for (int k = 1; k < 4; ++k) if (counts[4 * r + k] > counts[4 * r + b]) b = k;
    const int c = counts[4 * r + b];
    votes += ((double)c > (double)n * 0.1) ? 1 : 0;
    if (info[4 * r] > best_inl && (double)c > (double)n * 0.05) { best = r; best_inl = info[4 * r]; }
    res[DFVO_TAIL_EGRIC + r] = (double)c;
  }
  res[DFVO_TAIL_VALID] = ((double)votes > (double)R / 2.0) ? 1.0 : 0.0;
  track_pick_store(info, E, R, best, res, E_best);
}

// h_gric == nullptr: the vote is the one k_track_pick_flow wrote
__global__ void k_track_gate(double* __restrict__ res, const int32_t* __restrict__ pinfo, const double* __restrict__ h_gric, int R, int n,
                             double* __restrict__ T21) {
  if (threadIdx.x != 0) return;
  const double hg = h_gric != nullptr ? h_gric[0] : 0.0;
  if (h_gric != nullptr) {
    int votes = 0;
    for (int r = 0; r < R; ++r) votes += (hg > res[DFVO_TAIL_EGRIC + r]) ? 1 : 0;
    res[DFVO_TAIL_VALID] = ((double)votes > (double)R / 2.0) ? 1.0 : 0.0;
  }
  const bool valid = res[DFVO_TAIL_VALID] != 0.0;
  const int best = (int)res[DFVO_TAIL_BEST], cheir = best >= 0 ? pinfo[0] : 0;
  const double* Rt = res + DFVO_TAIL_RT;
  const bool pose_ok = valid && best >= 0 && (double)cheir > (double)n * 0.1;
  const double tn = Rt[9] * Rt[9] + Rt[10] * Rt[10] + Rt[11] * Rt[11];
  res[DFVO_TAIL_HGRIC] = hg; res[DFVO_TAIL_CHEIR] = (double)cheir; res[DFVO_TAIL_GATE] = (pose_ok && tn != 0.0) ? 1.0 : 0.0;
  res[DFVO_TAIL_NVALID] = 0.0;
  // T_21 = inv([R | t]) = [R^T | -R^T t], rows 0..2
  for (int a = 0; a < 3; ++a) {
    double tt = 0;
    for (int b = 0; b < 3; ++b) { T21[4 * a + b] = Rt[3 * b + a]; tt += Rt[3 * b + a] * Rt[9 + b]; }
    T21[4 * a + 3] = -tt;
  }
}

#define SC_THREADS 1024
#define SC_MAX 4096
// per keypoint (many blocks): normalise, triangulate, CNN depth at int(kp_cur), sort key (pixel index, then LAST keypoint first)
__global__ void __launch_bounds__(128)
k_scale_points(const double* __restrict__ kp_ref, const double* __restrict__ kp_cur, int n, double fx, double fy, double cx, double cy,
               const double* __restrict__ T21, const float* __restrict__ depth, int H, int W, const double* __restrict__ res,
               double* __restrict__ zbuf, double* __restrict__ dbuf, unsigned long long* __restrict__ keys) {
  if (res[DFVO_TAIL_GATE] == 0.0) return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double Pm[3][4];
  for (int a = 0; a < 3; ++a) for (int b = 0; b < 4; ++b) Pm[a][b] = T21[4 * a + b];
  // normalised coordinates as the host computes them: (kp - [cx, cy]) / [fx, fy]
  const double u0 = (kp_ref[2 * i] - cx) / fx, v0 = (kp_ref[2 * i + 1] - cy) / fy;
  const double u1 = (kp_cur[2 * i] - cx) / fx, v1 = (kp_cur[2 * i + 1] - cy) / fy;
  double X[4];
  triangulate_dlt(Pm, u0, v0, u1, v1, X);
  const double x = X[0] / X[3], y = X[1] / X[3], z = X[2] / X[3];
  zbuf[i] = Pm[2][0] * x + Pm[2][1] * y + Pm[2][2] * z + Pm[2][3];
  const int px = (int)kp_cur[2 * i], py = (int)kp_cur[2 * i + 1];                    // truncation toward zero (ops_3d.py:35-37)
  unsigned long long k = ~0ull;
  if (px >= 0 && px < W && py >= 0 && py < H) {
    const unsigned lin = (unsigned)py * (unsigned)W + (unsigned)px;
    dbuf[i] = (double)depth[lin];
    k = ((unsigned long long)lin << 32) | (unsigned long long)(0xffffffffu - (unsigned)i);   // equal pixels: the LAST keypoint sorts first
  }
  keys[i] = k;
}

// one block: sort the keys, keep the first entry of every pixel, compact the usable ratios in pixel order
__global__ void __launch_bounds__(SC_THREADS)
k_scale_chain(const unsigned long long* __restrict__ keys, int n, double* __restrict__ res, const double* __restrict__ zbuf,
              const double* __restrict__ dbuf, double* __restrict__ ratio) {
  __shared__ unsigned long long key[SC_MAX];
  __shared__ int wsum[SC_THREADS / 32];
  __shared__ int total_s;
  if (res[DFVO_TAIL_GATE] == 0.0) return;
  const int t = threadIdx.x;
  int P = 1; while (P < n) P <<= 1;
  for (int i = t; i < P; i += SC_THREADS) key[i] = i < n ? keys[i] : ~0ull;
  __syncthreads();
  // bitonic sort, ascending
  for (int size = 2; size <= P; size <<= 1)
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = t; i < P; i += SC_THREADS) {
        const int j = i ^ stride;
        if (j > i) {
          const bool up = (i & size) == 0;
          const unsigned long long a = key[i], b = key[j];
          if ((a > b) == up) { key[i] = b; key[j] = a; }
        }
      }
      __syncthreads();
    }
  // heads of the runs with a usable ratio, compacted in order: thread t owns the slots [t * per, (t + 1) * per)
  const int per = P / SC_THREADS > 0 ? P / SC_THREADS : 1;
  const int j0 = t * per;
  int cnt = 0;
  double rloc[SC_MAX / SC_THREADS];
  for (int q = 0; q < per; ++q) {
    const int j = j0 + q;
    if (j >= P) break;
    const unsigned long long k = key[j];
    if (k == ~0ull) continue;
    if (j > 0 && (key[j - 1] >> 32) == (k >> 32)) continue;                  // an earlier keypoint of the same pixel: overwritten
    const int i = (int)(0xffffffffu - (unsigned)(k & 0xffffffffu));
    double zt = zbuf[i];
    zt = zt < 0 ? 0.0 : zt;
    const double dp = dbuf[i];
    if (dp > 0 && zt > 0) rloc[cnt++] = zt / dp;
  }
  int incl = cnt;
  for (int off = 1; off < 32; off <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, off); if ((t & 31) >= off) incl += v; }
  if ((t & 31) == 31) wsum[t >> 5] = incl;
  __syncthreads();
  if (t == 0) { int a = 0; for (int w8 = 0; w8 < SC_THREADS / 32; ++w8) { const int v = wsum[w8]; wsum[w8] = a; a += v; } total_s = a; }
  __syncthreads();
  const int base = wsum[t >> 5] + incl - cnt;
  for (int q = 0; q < cnt; ++q) ratio[base + q] = rloc[q];
  if (t == 0) res[DFVO_TAIL_NVALID] = (double)total_s;
}

#define TAIL_MAX_R 32
size_t essential_tail_workspace_bytes(int N) {
  return (size_t)N * 8 * 4 + (size_t)N * 4 + 9 * 8 + 12 * 8 + (size_t)TAIL_MAX_R * 16 + 1024;
}

int essential_tail(const double* E, const int32_t* info, const double* gric, int R, const double* kp_cur, const double* kp_ref, int N,
                   double fx, double fy, double cx, double cy, const double* h_gric, const float* depth, int H, int W, int min_samples,
                   int max_trials, double stop_prob, double thr, void* workspace, size_t ws_bytes, double* res, uint8_t* pose_mask,
                   int32_t* pose_info, cudaStream_t s) {
  DFVO_REQUIRE(E && info && (gric || !h_gric) && kp_cur && kp_ref && workspace && res && pose_mask && pose_info, DFVO_EINVAL,
               "essential_tail args");
  DFVO_REQUIRE(R >= 1 && R <= TAIL_MAX_R && N >= 1 && N <= SC_MAX && min_samples >= 1 && min_samples <= SR_MAX_SAMPLES, DFVO_EINVAL,
               "essential_tail: R=%d N=%d", R, N);
  DFVO_REQUIRE(ws_bytes >= essential_tail_workspace_bytes(N), DFVO_EINVAL, "essential_tail workspace too small");
  uint8_t* w = reinterpret_cast<uint8_t*>(workspace);
  auto take = [&](size_t bytes) { uint8_t* p = w; w += (bytes + 127) & ~(size_t)127; return p; };
  double* zbuf = (double*)take((size_t)N * 8);
  double* dbuf = (double*)take((size_t)N * 8);
  double* ratio = (double*)take((size_t)N * 8);
  int32_t* perm = (int32_t*)take((size_t)N * 4);
  unsigned long long* keys = (unsigned long long*)take((size_t)N * 8);
  double* E_best = (double*)take(9 * 8);
  double* T21 = (double*)take(12 * 8);
  int32_t* counts = (int32_t*)take((size_t)TAIL_MAX_R * 16);
  if (h_gric != nullptr) {
    DFVO_LAUNCH(k_track_pick, dim3(1), dim3(32), 0, s, info, gric, E, R, res, E_best);
  } else {
    DFVO_CUDA(cudaMemsetAsync(counts, 0, (size_t)R * 16, s));
    DFVO_LAUNCH(k_recover_pose_counts, dim3(cdiv(4 * N, 256), R), dim3(256), 0, s, E, kp_cur, kp_ref, N, fx, cx, cy, 50.0, counts);
    DFVO_LAUNCH(k_track_pick_flow, dim3(1), dim3(32), 0, s, info, (const int32_t*)counts, E, R, N, res, E_best);
  }
  DFVO_CUDA(cudaMemsetAsync(pose_info, 0, 5 * sizeof(int32_t), s));
  DFVO_LAUNCH(k_recover_pose_vote, dim3(cdiv(4 * N, 256)), dim3(256), 0, s, (const double*)E_best, kp_cur, kp_ref, N, fx, cx, cy, 50.0, pose_mask, pose_info);
  DFVO_LAUNCH(k_recover_pose_pick, dim3(cdiv(N, 256)), dim3(256), 0, s, (const double*)E_best, N, res + DFVO_TAIL_RT, pose_mask, pose_info);
  DFVO_LAUNCH(k_track_gate, dim3(1), dim3(32), 0, s, res, (const int32_t*)pose_info, h_gric, R, N, T21);
  if (depth != nullptr) {
    DFVO_LAUNCH(k_scale_points, dim3(cdiv(N, 128)), dim3(128), 0, s, kp_ref, kp_cur, N, fx, fy, cx, cy, (const double*)T21, depth, H, W,
                (const double*)res, zbuf, dbuf, keys);
    DFVO_LAUNCH(k_scale_chain, dim3(1), dim3(SC_THREADS), 0, s, (const unsigned long long*)keys, N, res, (const double*)zbuf, (const double*)dbuf, ratio);
    DFVO_LAUNCH(k_scale_ransac, dim3(1), dim3(SR_THREADS), 0, s, (const double*)ratio, N, min_samples, max_trials, stop_prob, thr, res, perm,
                (const double*)(res + DFVO_TAIL_NVALID), (const double*)(res + DFVO_TAIL_GATE));
  }
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

}  // namespace dfvo
