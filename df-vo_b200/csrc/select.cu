// Correspondence selection on the device (kp_selection.py:33-200).
//
// local_bestN: the image is cut into rows x cols cells with the reference's slice quirk
// ([y0, y1) with y1 = int(h/rows*(r+1)) - 1, kp_selection.py:129-133); inside each cell the
// n_best pixels with the smallest forward-backward inconsistency among those below the threshold
// are kept.  The reference uses np.argpartition, whose order inside the first k is
// implementation-defined, so the contract is the *set*; this kernel emits it in canonical order
// (cell-major, ascending linear pixel index) and breaks ties at the k-th value by smaller index.
// Exact selection = 4-pass radix select over the fp32 bit pattern (values are >= 0, so the
// unsigned bit pattern is order-preserving) + ordered compaction.  One 256-thread block per cell.
//
// bestN: the same radix select over the whole map (kp_selection.py:33-71).
//
// score_method 'flow_ratio' (kp_selection.py:135-160,192-199): the same selection on the ratio map flow_diff / |flow|, which
// k_flow_ratio writes while it counts the raw flow_diff < thre of the "case 1" early-out.
#include "ops.h"

namespace dfvo {

#define SEL_THREADS 256

DFVO_D uint32_t sel_key(float v) {
  // order-preserving map of a float to uint32 (handles the negative range too, although the
  // inconsistency map is a norm); NaN sorts last.
  uint32_t u = __float_as_uint(v);
  if (v != v) return 0xffffffffu;
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// block-wide exclusive scan of one int per thread (SEL_THREADS threads); returns exclusive prefix,
// *total gets the block sum.  Uses shared scratch of SEL_THREADS ints.
DFVO_D int block_exclusive_scan(int v, int* scratch, int* total) {
  const int t = threadIdx.x;
  scratch[t] = v;
  __syncthreads();
  for (int off = 1; off < SEL_THREADS; off <<= 1) {
    int add = (t >= off) ? scratch[t - off] : 0;
    __syncthreads();
    scratch[t] += add;
    __syncthreads();
  }
  int incl = scratch[t];
  *total = scratch[SEL_THREADS - 1];
  __syncthreads();
  return incl - v;
}

struct CellGeom { int y0, y1, x0, x1; };

DFVO_D CellGeom cell_geom(int cell, int H, int W, int rows, int cols) {
  // int(h / num_row * row): true division in float64 then truncation (kp_selection.py:129-130)
  CellGeom g;
  int r = cell / cols, c = cell % cols;
  g.y0 = (int)((double)H / (double)rows * (double)r);
  g.x0 = (int)((double)W / (double)cols * (double)c);
  g.y1 = (int)((double)H / (double)rows * (double)(r + 1)) - 1;
  g.x1 = (int)((double)W / (double)cols * (double)(c + 1)) - 1;
  return g;
}

__global__ void __launch_bounds__(SEL_THREADS)
k_local_bestn(const float* __restrict__ diff, const float* __restrict__ depth_diff, int H, int W, int rows, int cols,
              int n_best, float thre, float depth_thre, int32_t* __restrict__ idx_out, int32_t* __restrict__ cell_counts) {
  __shared__ int hist[256];
  __shared__ int scratch[SEL_THREADS];
  __shared__ uint32_t s_prefix;
  __shared__ int s_remaining, s_nvalid;
  const int cell = blockIdx.x;
  const CellGeom g = cell_geom(cell, H, W, rows, cols);
  const int ch = g.y1 - g.y0, cw = g.x1 - g.x0;
  const int npx = (ch > 0 && cw > 0) ? ch * cw : 0;
  const int t = threadIdx.x;

  auto valid_key = [&](int i, uint32_t* key) -> bool {
    int y = g.y0 + i / cw, x = g.x0 + i % cw;
    float v = diff[(size_t)y * W + x];
    bool ok = v < thre;
    if (ok && depth_diff) ok = depth_diff[(size_t)y * W + x] < depth_thre;
    *key = sel_key(v);
    return ok;
  };

  // ---- count candidates ----
  int cnt = 0;
  for (int i = t; i < npx; i += SEL_THREADS) { uint32_t k; cnt += valid_key(i, &k) ? 1 : 0; }
  int total;
  block_exclusive_scan(cnt, scratch, &total);
  if (t == 0) s_nvalid = total;
  __syncthreads();
  const int nvalid = s_nvalid;
  const int k = nvalid < n_best ? nvalid : n_best;       // num_to_pick (kp_selection.py:156)
  if (t == 0) cell_counts[cell] = k;
  for (int i = t; i < n_best; i += SEL_THREADS) idx_out[cell * n_best + i] = -1;
  if (k == 0) return;

  // ---- radix select: key of the k-th smallest candidate ----
  if (t == 0) { s_prefix = 0u; s_remaining = k; }
  __syncthreads();
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    const uint32_t mask_hi = pass == 0 ? 0u : (0xffffffffu << (shift + 8));
    hist[t] = 0;
    __syncthreads();
    const uint32_t prefix = s_prefix;
    for (int i = t; i < npx; i += SEL_THREADS) {
      uint32_t key;
      if (valid_key(i, &key) && (key & mask_hi) == prefix) atomicAdd(&hist[(key >> shift) & 0xff], 1);
    }
    __syncthreads();
    if (t == 0) {
      int rem = s_remaining, b = 0;
      while (b < 255 && hist[b] < rem) { rem -= hist[b]; ++b; }
      s_remaining = rem;                      // rank of the k-th inside bucket b
      s_prefix = prefix | ((uint32_t)b << shift);
    }
    __syncthreads();
  }
  const uint32_t kth = s_prefix;
  const int need_eq = s_remaining;             // how many keys == kth are taken (smallest indices first)

  // ---- ordered compaction (ascending linear index) ----
  int base_less = 0, base_eq = 0;
  for (int c0 = 0; c0 < npx; c0 += SEL_THREADS) {
    const int i = c0 + t;
    uint32_t key = 0; bool ok = false;
    if (i < npx) ok = valid_key(i, &key);
    const int is_less = (ok && key < kth) ? 1 : 0;
    const int is_eq = (ok && key == kth) ? 1 : 0;
    int tot_less, tot_eq;
    const int pl = block_exclusive_scan(is_less, scratch, &tot_less);
    const int pe = block_exclusive_scan(is_eq, scratch, &tot_eq);
    const int eq_rank = base_eq + pe;
    if (is_less || (is_eq && eq_rank < need_eq)) {
      const int eq_before = eq_rank < need_eq ? eq_rank : need_eq;
      const int pos = base_less + pl + eq_before;
      const int y = g.y0 + i / cw, x = g.x0 + i % cw;
      idx_out[cell * n_best + pos] = y * W + x;
    }
    base_less += tot_less; base_eq += tot_eq;
  }
}

// ------------------------------------------------------------------------------------------------
// 'uniform' keypoints of opt_rigid_flow_kp (kp_selection.py:203-324, :277-284): inside each cell the pixels that pass both
// masks (rigid-flow inconsistency < rigid_thre, forward-backward inconsistency < flow_thre) are enumerated in row-major
// order of the cell slice (np.where), and every step-th of them is kept: step = int(n / k), k = min(n_best, n), positions
// 0, step, 2 step, ... (the first k).  One 256-thread block per cell; each thread owns a contiguous run of the cell's
// row-major order so that ranks come from one exclusive scan.  idx_out [cells * n_best] (-1 padded), cell_counts [cells].
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SEL_THREADS)
k_uniform_cells(const float* __restrict__ rigid_diff, const float* __restrict__ flow_diff, int H, int W, int rows, int cols, int n_best,
                float rigid_thre, float flow_thre, int32_t* __restrict__ idx_out, int32_t* __restrict__ cell_counts) {
  __shared__ int scratch[SEL_THREADS];
  const int cell = blockIdx.x;
  const CellGeom g = cell_geom(cell, H, W, rows, cols);
  const int ch = g.y1 - g.y0, cw = g.x1 - g.x0;
  const int npx = (ch > 0 && cw > 0) ? ch * cw : 0;
  const int t = threadIdx.x;
  const int chunk = (npx + SEL_THREADS - 1) / SEL_THREADS;
  const int i0 = t * chunk < npx ? t * chunk : npx, i1 = i0 + chunk < npx ? i0 + chunk : npx;
  auto valid = [&](int i) -> bool {
    const size_t o = (size_t)(g.y0 + i / cw) * W + (g.x0 + i % cw);
    return rigid_diff[o] < rigid_thre && flow_diff[o] < flow_thre;
  };
  int cnt = 0;
  for (int i = i0; i < i1; ++i) cnt += valid(i) ? 1 : 0;
  int n;
  int rank = block_exclusive_scan(cnt, scratch, &n);
  const int k = n < n_best ? n : n_best;
  if (t == 0) cell_counts[cell] = k;
  for (int i = t; i < n_best; i += SEL_THREADS) idx_out[cell * n_best + i] = -1;
  __syncthreads();
  if (k == 0) return;
  const int step = n / k;
  for (int i = i0; i < i1; ++i) {
    if (!valid(i)) continue;
    if (rank % step == 0 && rank / step < k) idx_out[cell * n_best + rank / step] = (g.y0 + i / cw) * W + (g.x0 + i % cw);
    ++rank;
  }
}

int uniform_cells(const float* rigid_diff, const float* flow_diff, int H, int W, int rows, int cols, int n_best, float rigid_thre,
                  float flow_thre, int32_t* idx_out, int32_t* cell_counts, cudaStream_t s) {
  DFVO_REQUIRE(rows > 0 && cols > 0 && n_best > 0 && rows * cols <= 65535, DFVO_EINVAL, "uniform_cells args");
  DFVO_LAUNCH(k_uniform_cells, dim3(rows * cols), dim3(SEL_THREADS), 0, s, rigid_diff, flow_diff, H, W, rows, cols, n_best, rigid_thre,
              flow_thre, idx_out, cell_counts);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

// ------------------------------------------------------------------------------------------------
// Rigid-flow inconsistency map (E_tracker.py:666-691): the RigidFlow layer (backproject the reference depth with K^-1,
// transform by T, project with K, subtract the pixel grid; rigid_flow.py / backprojection.py / projection.py, float32,
// eps = 1e-7 in the perspective division) and the norm of its difference to the optical flow, fused per pixel.
// T, Kinv rows: float32 copies of the float64 inputs (torch.from_numpy(..).float()).
// ------------------------------------------------------------------------------------------------
struct RigidP { float T[12]; float ik[9]; float fx, fy, cx, cy; };

__global__ void k_rigid_flow_diff(const float* __restrict__ depth, const float* __restrict__ flow, int H, int W, RigidP p,
                                  float* __restrict__ out) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= W) return;
  const size_t i = (size_t)y * W + x, hw = (size_t)H * W;
  const float fxp = (float)x, fyp = (float)y, d = depth[i];
  // points = inv_K[:3,:3] @ (x, y, 1); points *= depth
  const float X = d * (p.ik[0] * fxp + p.ik[1] * fyp + p.ik[2]);
  const float Y = d * (p.ik[3] * fxp + p.ik[4] * fyp + p.ik[5]);
  const float Z = d * (p.ik[6] * fxp + p.ik[7] * fyp + p.ik[8]);
  // T @ (X, Y, Z, 1)
  const float qx = p.T[0] * X + p.T[1] * Y + p.T[2] * Z + p.T[3];
  const float qy = p.T[4] * X + p.T[5] * Y + p.T[6] * Z + p.T[7];
  const float qz = p.T[8] * X + p.T[9] * Y + p.T[10] * Z + p.T[11];
  // K[:3,:] @ q ; xy = uv / (w + eps)
  const float ux = p.fx * qx + p.cx * qz, uy = p.fy * qy + p.cy * qz, uw = qz + 1e-7f;
  const float rx = ux / uw - fxp, ry = uy / uw - fyp;
  const float dx = rx - flow[i], dy = ry - flow[hw + i];
  out[i] = sqrtf(dx * dx + dy * dy);
}

int rigid_flow_diff(const float* depth, const float* flow, int H, int W, const double* T_host, double fx, double fy, double cx, double cy,
                    float* out, cudaStream_t s) {
  RigidP p;
  for (int i = 0; i < 12; ++i) p.T[i] = (float)T_host[i];
  // inverse of [[fx,0,cx],[0,fy,cy],[0,0,1]] in float64 (Intrinsics.inv_mat = np.linalg.inv), then float32
  const double ik[9] = {1.0 / fx, 0.0, -cx / fx, 0.0, 1.0 / fy, -cy / fy, 0.0, 0.0, 1.0};
  for (int i = 0; i < 9; ++i) p.ik[i] = (float)ik[i];
  p.fx = (float)fx; p.fy = (float)fy; p.cx = (float)cx; p.cy = (float)cy;
  DFVO_LAUNCH(k_rigid_flow_diff, dim3(cdiv(W, 128), H), dim3(128), 0, s, depth, flow, H, W, p, out);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

__global__ void k_count_below(const float* __restrict__ diff, int n, float thre, int32_t* __restrict__ out) {
  __shared__ int scratch[SEL_THREADS];
  int c = 0;
  for (int i = blockIdx.x * SEL_THREADS + threadIdx.x; i < n; i += gridDim.x * SEL_THREADS) c += diff[i] < thre ? 1 : 0;
  int total;
  block_exclusive_scan(c, scratch, &total);
  if (threadIdx.x == 0 && total) atomicAdd(out, total);
}

// status[0] = good_kp_found, status[1] = number of selected keypoints, status[2] = #(diff < thre),
// status[3] = number of non-empty cells
__global__ void k_local_bestn_status(const int32_t* __restrict__ cell_counts, int ncells, int N_total, int32_t* __restrict__ status) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  int sel = 0, nonempty = 0;
  for (int i = 0; i < ncells; ++i) { sel += cell_counts[i]; nonempty += cell_counts[i] != 0; }
  int good = 1;
  if ((double)status[2] < (double)N_total * 0.1) good = 0;        // kp_selection.py:121-125
  if ((double)nonempty < (double)ncells * 0.1) good = 0;          // kp_selection.py:175-179
  status[0] = good; status[1] = good ? sel : 0; status[3] = nonempty;
}

// local_bestN's score map for score_method 'flow_ratio' (kp_selection.py:146-149,193-197): ratio = flow_diff / ||flow||, the norm
// as NumPy computes np.linalg.norm(axis=3) in float32 -- sqrt(fx*fx + fy*fy) with every operation rounded on its own (no FMA) --
// so the map is bit-equal to the reference's fb_flow_mask; 0/0 gives NaN and x/0 inf, and neither passes `< thre`.  The same pass
// counts the RAW flow_diff < thre into *count: the "case 1" early-out (kp_selection.py:121-125) tests flow_diff, not the ratio.
__global__ void k_flow_ratio(const float* __restrict__ diff, const float* __restrict__ flow, int n, float thre, float* __restrict__ ratio,
                             int32_t* __restrict__ count) {
  __shared__ int scratch[SEL_THREADS];
  int c = 0;
  for (int i = blockIdx.x * SEL_THREADS + threadIdx.x; i < n; i += gridDim.x * SEL_THREADS) {
    const float d = diff[i], fx = flow[i], fy = flow[(size_t)n + i];
    const float nrm = __fsqrt_rn(__fadd_rn(__fmul_rn(fx, fx), __fmul_rn(fy, fy)));
    ratio[i] = __fdiv_rn(d, nrm);
    c += d < thre ? 1 : 0;
  }
  int total;
  block_exclusive_scan(c, scratch, &total);
  if (threadIdx.x == 0 && total) atomicAdd(count, total);
}

// count_map: the map whose `< thre` count is status[2] (case 1); nullptr when the caller has already zeroed the status and
// counted into status[2] itself.  score: the map the cells select on.
int local_bestn(const float* count_map, const float* score, const float* depth_diff, int H, int W, int rows, int cols, int n_best,
                float thre, float depth_thre, int N_total, int32_t* idx_out, int32_t* cell_counts, int32_t* status, cudaStream_t s) {
  DFVO_REQUIRE(rows > 0 && cols > 0 && n_best > 0 && rows * cols <= 65535, DFVO_EINVAL, "local_bestn args");
  if (count_map) {
    DFVO_CUDA(cudaMemsetAsync(status, 0, 4 * sizeof(int32_t), s));
    DFVO_LAUNCH(k_count_below, dim3(132), dim3(SEL_THREADS), 0, s, count_map, H * W, thre, status + 2);
    DFVO_CHECK_LAUNCH();
  }
  DFVO_LAUNCH(k_local_bestn, dim3(rows * cols), dim3(SEL_THREADS), 0, s, score, depth_diff, H, W, rows, cols, n_best, thre,
              depth_thre, idx_out, cell_counts);
  DFVO_CHECK_LAUNCH();
  DFVO_LAUNCH(k_local_bestn_status, dim3(1), dim3(32), 0, s, cell_counts, rows * cols, N_total, status);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

int local_bestn_flow_ratio(const float* flow_diff, const float* flow_fwd, const float* depth_diff, int H, int W, int rows, int cols,
                           int n_best, float thre, float depth_thre, int N_total, float* ratio_out, int32_t* idx_out, int32_t* cell_counts,
                           int32_t* status, cudaStream_t s) {
  DFVO_REQUIRE(rows > 0 && cols > 0 && n_best > 0 && rows * cols <= 65535, DFVO_EINVAL, "local_bestn_flow_ratio args");
  const int n = H * W;
  DFVO_CUDA(cudaMemsetAsync(status, 0, 4 * sizeof(int32_t), s));
  const int blocks = cdiv(n, SEL_THREADS) < 1056 ? cdiv(n, SEL_THREADS) : 1056;
  DFVO_LAUNCH(k_flow_ratio, dim3(blocks), dim3(SEL_THREADS), 0, s, flow_diff, flow_fwd, n, thre, ratio_out, status + 2);
  DFVO_CHECK_LAUNCH();
  return local_bestn(nullptr, ratio_out, depth_diff, H, W, rows, cols, n_best, thre, depth_thre, N_total, idx_out, cell_counts, status, s);
}

// ------------------------------------------------------------------------------------------------
// bestN over the whole map.  workspace: [0..255] histogram, [256] prefix, [257] remaining,
// [258 .. 258+2*nblocks) per-block (less, equal) counts, then their exclusive prefixes.
// ------------------------------------------------------------------------------------------------
#define BESTN_CHUNK 4096

__global__ void k_bestn_init(uint32_t* ws, int N) {
  for (int i = threadIdx.x; i < 256; i += blockDim.x) ws[i] = 0u;
  if (threadIdx.x == 0) { ws[256] = 0u; ws[257] = (uint32_t)N; }
}

__global__ void k_bestn_hist(const float* __restrict__ diff, int n, int pass, uint32_t* ws) {
  __shared__ int hist[256];
  const int shift = 24 - 8 * pass;
  const uint32_t mask_hi = pass == 0 ? 0u : (0xffffffffu << (shift + 8));
  const uint32_t prefix = ws[256];
  hist[threadIdx.x] = 0;
  __syncthreads();
  for (int i = blockIdx.x * SEL_THREADS + threadIdx.x; i < n; i += gridDim.x * SEL_THREADS) {
    uint32_t key = sel_key(diff[i]);
    if ((key & mask_hi) == prefix) atomicAdd(&hist[(key >> shift) & 0xff], 1);
  }
  __syncthreads();
  if (hist[threadIdx.x]) atomicAdd(&ws[threadIdx.x], (uint32_t)hist[threadIdx.x]);
}

__global__ void k_bestn_pick(int pass, uint32_t* ws) {
  if (threadIdx.x == 0) {
    const int shift = 24 - 8 * pass;
    uint32_t rem = ws[257];
    int b = 0;
    while (b < 255 && ws[b] < rem) { rem -= ws[b]; ++b; }
    ws[257] = rem;
    ws[256] |= (uint32_t)b << shift;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 256; i += blockDim.x) ws[i] = 0u;
}

__global__ void k_bestn_count(const float* __restrict__ diff, int n, uint32_t* ws) {
  __shared__ int scratch[SEL_THREADS];
  const uint32_t kth = ws[256];
  const int c0 = blockIdx.x * BESTN_CHUNK;
  int less = 0, eq = 0;
  for (int i = c0 + threadIdx.x; i < c0 + BESTN_CHUNK && i < n; i += SEL_THREADS) {
    uint32_t key = sel_key(diff[i]);
    less += key < kth; eq += key == kth;
  }
  int tl, te;
  block_exclusive_scan(less, scratch, &tl);
  block_exclusive_scan(eq, scratch, &te);
  if (threadIdx.x == 0) { ws[258 + 2 * blockIdx.x] = (uint32_t)tl; ws[258 + 2 * blockIdx.x + 1] = (uint32_t)te; }
}

__global__ void k_bestn_scan(int nblocks, uint32_t* ws) {
  if (threadIdx.x != 0) return;
  uint32_t al = 0, ae = 0;
  uint32_t* cnt = ws + 258;
  uint32_t* pre = ws + 258 + 2 * nblocks;
  for (int b = 0; b < nblocks; ++b) {
    pre[2 * b] = al; pre[2 * b + 1] = ae;
    al += cnt[2 * b]; ae += cnt[2 * b + 1];
  }
}

__global__ void k_bestn_write(const float* __restrict__ diff, int n, int nblocks, const uint32_t* __restrict__ ws,
                              int32_t* __restrict__ idx_out) {
  __shared__ int scratch[SEL_THREADS];
  const uint32_t kth = ws[256];
  const int need_eq = (int)ws[257];
  const uint32_t* pre = ws + 258 + 2 * nblocks;
  int base_less = (int)pre[2 * blockIdx.x], base_eq = (int)pre[2 * blockIdx.x + 1];
  const int c0 = blockIdx.x * BESTN_CHUNK;
  for (int j = 0; j < BESTN_CHUNK; j += SEL_THREADS) {
    const int i = c0 + j + threadIdx.x;
    uint32_t key = 0; bool in = i < n && (c0 + j + (int)threadIdx.x) < c0 + BESTN_CHUNK;
    if (in) key = sel_key(diff[i]);
    const int is_less = in && key < kth, is_eq = in && key == kth;
    int tl, te;
    const int pl = block_exclusive_scan(is_less, scratch, &tl);
    const int pe = block_exclusive_scan(is_eq, scratch, &te);
    const int eq_rank = base_eq + pe;
    if (is_less || (is_eq && eq_rank < need_eq)) {
      // global position in ascending-index order: all selected entries before i
      const int eq_before = eq_rank < need_eq ? eq_rank : need_eq;
      idx_out[base_less + pl + eq_before] = i;
    }
    base_less += tl; base_eq += te;
  }
}

size_t bestn_workspace_bytes(int H, int W) {
  int nblocks = cdiv(H * W, BESTN_CHUNK);
  return (size_t)(258 + 4 * nblocks) * sizeof(uint32_t);
}

int bestn(const float* diff, int H, int W, int N, int32_t* idx_out, void* workspace, size_t ws_bytes, cudaStream_t s) {
  const int n = H * W;
  DFVO_REQUIRE(N > 0 && N <= n, DFVO_EINVAL, "bestn: N out of range");
  DFVO_REQUIRE(ws_bytes >= bestn_workspace_bytes(H, W), DFVO_EINVAL, "bestn: workspace too small");
  uint32_t* ws = reinterpret_cast<uint32_t*>(workspace);
  const int nblocks = cdiv(n, BESTN_CHUNK);
  DFVO_LAUNCH(k_bestn_init, dim3(1), dim3(256), 0, s, ws, N);
  for (int pass = 0; pass < 4; ++pass) {
    DFVO_LAUNCH(k_bestn_hist, dim3(132), dim3(SEL_THREADS), 0, s, diff, n, pass, ws);
    DFVO_LAUNCH(k_bestn_pick, dim3(1), dim3(256), 0, s, pass, ws);
  }
  DFVO_LAUNCH(k_bestn_count, dim3(nblocks), dim3(SEL_THREADS), 0, s, diff, n, ws);
  DFVO_LAUNCH(k_bestn_scan, dim3(1), dim3(32), 0, s, nblocks, ws);
  DFVO_LAUNCH(k_bestn_write, dim3(nblocks), dim3(SEL_THREADS), 0, s, diff, n, nblocks, (const uint32_t*)ws, idx_out);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

// ------------------------------------------------------------------------------------------------
// keypoint gather (keypoint_sampler.py:101-104 + kp_selection.py:181-190): compact the per-cell slots
// into kp1 = (x, y) float64 and kp2 = kp1 + forward flow (float32 promoted to float64).
// ------------------------------------------------------------------------------------------------
__global__ void k_gather_keypoints(const int32_t* __restrict__ idx, const int32_t* __restrict__ cell_counts, int ncells, int n_best,
                                   const float* __restrict__ flow, int H, int W, double* __restrict__ kp1,
                                   double* __restrict__ kp2, int32_t* __restrict__ n_out) {
  DFVO_DYN_SMEM(int, prefix);
  if (threadIdx.x == 0) {
    int a = 0;
    for (int c = 0; c < ncells; ++c) { prefix[c] = a; a += cell_counts ? cell_counts[c] : n_best; }
    prefix[ncells] = a;
    if (n_out) *n_out = a;
  }
  __syncthreads();
  for (int slot = threadIdx.x; slot < ncells * n_best; slot += blockDim.x) {
    int c = slot / n_best, j = slot % n_best;
    int cnt = cell_counts ? cell_counts[c] : n_best;
    if (j >= cnt) continue;
    int lin = idx[slot];
    int y = lin / W, x = lin % W;
    int o = prefix[c] + j;
    kp1[2 * o] = (double)x; kp1[2 * o + 1] = (double)y;
    kp2[2 * o] = (double)x + (double)flow[(size_t)y * W + x];
    kp2[2 * o + 1] = (double)y + (double)flow[(size_t)H * W + (size_t)y * W + x];
  }
}

// depth at int(kp) (truncation toward zero, like kp.astype(int) at ops_3d.py:29 / pnp_tracker.py:72); 0 if outside
__global__ void k_gather_depth(const float* __restrict__ depth, int H, int W, const double* __restrict__ kp, int n,
                               float* __restrict__ out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int x = (int)kp[2 * i], y = (int)kp[2 * i + 1];
  out[i] = (x >= 0 && x < W && y >= 0 && y < H) ? depth[(size_t)y * W + x] : 0.f;
}

int gather_depth(const float* depth, int H, int W, const double* kp, int n, float* out, cudaStream_t s) {
  DFVO_LAUNCH(k_gather_depth, dim3(cdiv(n, 128)), dim3(128), 0, s, depth, H, W, kp, n, out);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

// ------------------------------------------------------------------------------------------------
// Flow-magnitude validity (E_tracker.py:182-185): np.mean(np.linalg.norm(kp_ref - kp_cur, axis=1)) bit for bit.  The norm of a row
// is sqrt(dx*dx + dy*dy) with every operation rounded (no FMA); the mean is NumPy's pairwise sum (pairwise_sum in
// loops_utils.h.src: blocks of <= 128 elements summed with 8 accumulators, larger ranges split at n/2 rounded down to a multiple
// of 8) divided by n.  One block: the blocks of the recursion ("leaves") are summed in parallel, thread 0 adds them up in the
// recursion's order.  Leaves hold 64..128 elements, so FM_MAX_LEAVES covers n <= FM_MAX_N.
// ------------------------------------------------------------------------------------------------
#define FM_THREADS 256
#define FM_MAX_LEAVES 1200
#define FM_MAX_N 65536

DFVO_D double kp_disp(const double* __restrict__ a, const double* __restrict__ b, int i) {
  const double dx = __dsub_rn(a[2 * i], b[2 * i]), dy = __dsub_rn(a[2 * i + 1], b[2 * i + 1]);
  return sqrt(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)));
}

// pairwise_sum's base case on [lo, lo + n), n <= 128
DFVO_D double pw_leaf(const double* __restrict__ a, const double* __restrict__ b, int lo, int n) {
  if (n < 8) {
    double r = 0.0;
    for (int i = 0; i < n; ++i) r = __dadd_rn(r, kp_disp(a, b, lo + i));
    return r;
  }
  double r[8];
  for (int j = 0; j < 8; ++j) r[j] = kp_disp(a, b, lo + j);
  int i = 8;
  for (; i < n - (n % 8); i += 8)
    for (int j = 0; j < 8; ++j) r[j] = __dadd_rn(r[j], kp_disp(a, b, lo + i + j));
  double res = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])), __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
  for (; i < n; ++i) res = __dadd_rn(res, kp_disp(a, b, lo + i));
  return res;
}

// the leaves of pairwise_sum(lo, n) in recursion order
DFVO_D void pw_leaves(int lo, int n, int* leaf_lo, int* leaf_n, int* count) {
  if (n <= 128) { leaf_lo[*count] = lo; leaf_n[*count] = n; ++*count; return; }
  int n2 = n / 2;
  n2 -= n2 % 8;
  pw_leaves(lo, n2, leaf_lo, leaf_n, count);
  pw_leaves(lo + n2, n - n2, leaf_lo, leaf_n, count);
}

DFVO_D double pw_combine(int n, const double* leaf_sum, int* next) {
  if (n <= 128) return leaf_sum[(*next)++];
  int n2 = n / 2;
  n2 -= n2 % 8;
  const double l = pw_combine(n2, leaf_sum, next);
  return __dadd_rn(l, pw_combine(n - n2, leaf_sum, next));
}

__global__ void __launch_bounds__(FM_THREADS)
k_flow_mean(const double* __restrict__ kp_ref, const double* __restrict__ kp_cur, int n_in, const int32_t* __restrict__ status,
            double* __restrict__ out) {
  __shared__ int leaf_lo[FM_MAX_LEAVES], leaf_n[FM_MAX_LEAVES];
  __shared__ double leaf_sum[FM_MAX_LEAVES];
  __shared__ int nleaves;
  const int t = threadIdx.x;
  const int good = status ? status[0] : 1;
  int n = status ? status[1] : n_in;
  n = n < 0 ? 0 : (n > FM_MAX_N ? FM_MAX_N : n);
  if (t == 0) { nleaves = 0; pw_leaves(0, n, leaf_lo, leaf_n, &nleaves); }
  __syncthreads();
  for (int l = t; l < nleaves; l += FM_THREADS) leaf_sum[l] = pw_leaf(kp_ref, kp_cur, leaf_lo[l], leaf_n[l]);
  __syncthreads();
  if (t == 0) {
    int next = 0;
    const double sum = pw_combine(n, leaf_sum, &next);
    out[0] = (double)good;
    out[1] = (double)n;
    out[2] = n > 0 ? sum / (double)n : 0.0;
  }
}

int flow_mean(const double* kp_ref, const double* kp_cur, int n, const int32_t* status, double* out, cudaStream_t s) {
  DFVO_REQUIRE(status != nullptr || (n >= 0 && n <= FM_MAX_N), DFVO_EINVAL, "flow_mean: n=%d (max %d)", n, FM_MAX_N);
  DFVO_LAUNCH(k_flow_mean, dim3(1), dim3(FM_THREADS), 0, s, kp_ref, kp_cur, n, status, out);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

int gather_keypoints(const int32_t* idx, const int32_t* cell_counts, int ncells, int n_best, const float* flow, int H, int W,
                     double* kp1, double* kp2, int32_t* n_out, cudaStream_t s) {
  DFVO_REQUIRE(ncells > 0 && ncells <= 8192, DFVO_EINVAL, "gather_keypoints: ncells");
  DFVO_LAUNCH(k_gather_keypoints, dim3(1), dim3(256), (size_t)(ncells + 1) * sizeof(int), s, idx, cell_counts, ncells, n_best, flow, H,
              W, kp1, kp2, n_out);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

}  // namespace dfvo
