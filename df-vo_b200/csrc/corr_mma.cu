// 49-channel correlation of LiteFlowNet's Matching units (lite_flow_net.py:132-152: Backward warp of the second feature map,
// FunctionCorrelation correlation.py:38-106, LeakyReLU) as ONE kernel on the tensor cores.
//
//   out[n, (dy+3)*7 + (dx+3), y, x] = leaky( 1/C * sum_c first[n, c, y*s, x*s] * second[n, c, (y+dy)*s, (x+dx)*s] ),  dy, dx in [-3, 3]
//   second = Backward(feat2[n ^ nxor], flow * scale)   (bilinear, zeros outside; lite_flow_net.py:10-28), or feat2 itself at level 6.
//
// Formulation: a block owns 16 x 8 output pixels.  For one output row (16 pixels = M) and one displacement row dy, the products
// with the 22 (-> 24) second-map pixels of patch row (y + dy) are a [16 x C] x [C x 24] GEMM on mma.sync.m16n8k16 (bf16, fp32
// accumulate); the 7 wanted displacements are the diagonal band dx = column - pixel of the [16 x 24] result, and in the mma.sync
// accumulator layout every register has a FIXED (row, column), so the band is picked with compile-time-known predicates.
// (the warp-level MMA's fixed fragment layout is what lets the band be selected in registers; a warpgroup MMA would read the
// 64-row operand once per displacement row for no gain at this size.)  The tensor
// cores do 24/7 = 3.4x the useful FLOPs, which is irrelevant at 1.2 GFLOP per launch; what matters is that a pixel of the second map
// is read from shared memory 7 times (once per dy) instead of 49 times, and no scalar FMA is issued at all.
// Fusions: the Backward warp is evaluated while staging the patch (no warped copy of the feature map in HBM -- and at the stride-2
// levels only the even pixels the correlation touches are warped at all: 1/4 of the old warp kernel's work), the 1/C scale and the
// LeakyReLU in the band extraction, and the output tile goes out as full 128-byte rows.
// Operands are staged with 16-byte chunks XOR-swizzled by the pixel index (ldmatrix reads 8 pixels x 16 B: conflict-free).
#include "ops.h"

namespace dfvo {

#ifndef DFVO_HOSTSIM
#define CM_TW 16
#define CM_TH 8
#define CM_PW 24            // patch columns: 16 + 6 used, padded to three n8 tiles
#define CM_PH (CM_TH + 6)
#define CM_THREADS 256

__device__ __forceinline__ uint32_t cm_smem(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void cm_ldsm4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void cm_ldsm2(uint32_t addr, uint32_t& r0, uint32_t& r1) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0, %1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(addr));
}
__device__ __forceinline__ void cm_mma(float* c, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
// byte offset of 16-byte chunk `ch` of pixel `px` in a [pixels][pitch] tile (pitch a multiple of 128 B)
__device__ __forceinline__ uint32_t cm_off(int px, int ch, int pitch) { return (uint32_t)px * (uint32_t)pitch + (uint32_t)(((ch & ~7) | ((ch ^ px) & 7)) << 4); }

// Single-slice variant (C <= 64): displacement rows outermost, 12 accumulators live -> 48 registers, three blocks per SM.
__global__ void __launch_bounds__(CM_THREADS)
k_corr_mma1(Ten<const bf16> f1, Ten<const bf16> f2, int f2_nxor, const float* __restrict__ flow, long long fN, long long fH, long long fW,
           float scale, int stride, int leaky, Ten<bf16> out, int pitch) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t* s_f1 = smem;                                              // [128 px][pitch]
  uint8_t* s_p = s_f1 + (size_t)CM_TW * CM_TH * pitch;               // [14 * 24 px][pitch]
  uint8_t* s_out = s_p + (size_t)CM_PH * CM_PW * pitch;              // [128 px][128 B]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int x0 = blockIdx.x * CM_TW, y0 = blockIdx.y * CM_TH, n = blockIdx.z;
  const int C = f1.C, nch = C >> 3;                                  // 16-byte chunks per pixel
  // ---- stage the first map's tile (pixels sampled with the stride)
  for (int i = tid; i < CM_TW * CM_TH * nch; i += CM_THREADS) {
    const int m = i / nch, ch = i - m * nch;
    const int ox = x0 + (m & 15), oy = y0 + (m >> 4);
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (ox < out.W && oy < out.H) v = *reinterpret_cast<const uint4*>(f1.at(n, oy * stride, ox * stride) + ch * 8);
    *reinterpret_cast<uint4*>(s_f1 + cm_off(m, ch, pitch)) = v;
  }
  // ---- stage the second map's patch: plain copy, or the Backward warp evaluated here
  const int n2 = n ^ f2_nxor;
  for (int i = tid; i < CM_PH * CM_PW * nch; i += CM_THREADS) {
    const int q = i / nch, ch = i - q * nch;
    const int pj = q / CM_PW, pi = q - pj * CM_PW;
    const int sx = (x0 + pi - 3) * stride, sy = (y0 + pj - 3) * stride;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (pi < CM_TW + 6 && sx >= 0 && sx < f2.W && sy >= 0 && sy < f2.H) {
      if (flow == nullptr) {
        v = *reinterpret_cast<const uint4*>(f2.at(n2, sy, sx) + ch * 8);
      } else {
        // Backward (lite_flow_net.py:10-28): bilinear sample at (x, y) + flow * scale, zeros outside; same arithmetic as
        // flow_ops.cu::k_warp_bilinear_vec (fp32 blend, round to bf16)
        const float* fl = flow + n * fN + (long long)sy * fH + (long long)sx * fW;
        const float px = (float)sx + fl[0] * scale, py = (float)sy + fl[1] * scale;
        const float fx0 = floorf(px), fy0 = floorf(py);
        const int ix = (int)fx0, iy = (int)fy0;
        const float wx1 = px - fx0, wy1 = py - fy0, wx0 = 1.f - wx1, wy0 = 1.f - wy1;
        const bool fin = (px == px) && (py == py) && fabsf(px) < 1e9f && fabsf(py) < 1e9f;      // non-finite coordinates sample nothing
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int xx = ix + (k & 1), yy = iy + (k >> 1);
          const float wgt = ((k & 1) ? wx1 : wx0) * ((k >> 1) ? wy1 : wy0);
          if (!fin || xx < 0 || xx > f2.W - 1 || yy < 0 || yy > f2.H - 1 || wgt == 0.f) continue;
          const uint4 t = *reinterpret_cast<const uint4*>(f2.at(n2, yy, xx) + ch * 8);
          const uint32_t w4[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            acc[2 * j] += __uint_as_float(w4[j] << 16) * wgt;
            acc[2 * j + 1] += __uint_as_float(w4[j] & 0xffff0000u) * wgt;
          }
        }
        uint32_t o4[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const __nv_bfloat162 h = __floats2bfloat162_rn(acc[2 * j], acc[2 * j + 1]);
          o4[j] = *reinterpret_cast<const uint32_t*>(&h);
        }
        v = make_uint4(o4[0], o4[1], o4[2], o4[3]);
      }
    }
    *reinterpret_cast<uint4*>(s_p + cm_off(q, ch, pitch)) = v;
  }
  // zero the pad channels 49..63 of the output staging once
  for (int i = tid; i < CM_TW * CM_TH * 2; i += CM_THREADS) {
    // channels 48..63 of pixel i/2 = chunks 6, 7; channel 48 is rewritten below
    *reinterpret_cast<uint4*>(s_out + (size_t)(i >> 1) * 128 + 96 + (i & 1) * 16) = make_uint4(0u, 0u, 0u, 0u);
  }
  __syncthreads();
  // ---- banded GEMMs: warp w = output row w of the tile
  const uint32_t f1_base = cm_smem(s_f1), p_base = cm_smem(s_p);
  const float inv = 1.f / (float)C;
  const int arow = warp * CM_TW + (lane & 7) + ((lane >> 3) & 1) * 8;          // A: pixel of this lane's ldmatrix row
  const int akc = lane >> 4;                                                  //    k-chunk within the k16 step
  const int brow4 = (lane & 7) + ((lane >> 4) & 1) * 8, bkc = (lane >> 3) & 1; // B x4: two n8 tiles;  B x2 uses lanes 0..15
  const int g = lane >> 2, tq = lane & 3;
  __nv_bfloat16* so = reinterpret_cast<__nv_bfloat16*>(s_out);
#pragma unroll 1
  for (int dy = 0; dy < 7; ++dy) {
    float acc[3][4];
#pragma unroll
    for (int t = 0; t < 3; ++t) { acc[t][0] = acc[t][1] = acc[t][2] = acc[t][3] = 0.f; }
    const int prow = (warp + dy) * CM_PW;                                       // patch row of this output row and displacement
    for (int ks = 0; ks < (C >> 4); ++ks) {
      uint32_t a0, a1, a2, a3, b0, b1, b2, b3, b4, b5;
      cm_ldsm4(f1_base + cm_off(arow, 2 * ks + akc, pitch), a0, a1, a2, a3);
      cm_ldsm4(p_base + cm_off(prow + brow4, 2 * ks + bkc, pitch), b0, b1, b2, b3);       // columns 0..15
      cm_ldsm2(p_base + cm_off(prow + 16 + (lane & 7), 2 * ks + bkc, pitch), b4, b5);      // columns 16..23
      cm_mma(acc[0], a0, a1, a2, a3, b0, b1);
      cm_mma(acc[1], a0, a1, a2, a3, b2, b3);
      cm_mma(acc[2], a0, a1, a2, a3, b4, b5);
    }
    // band extraction: accumulator e of tile t sits at (row, col) = (g + 8 * (e >> 1), 8 * t + 2 * tq + (e & 1)); dx = col - row
#pragma unroll
    for (int t = 0; t < 3; ++t) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int row = g + 8 * (e >> 1), col = 8 * t + 2 * tq + (e & 1);
        const int dx = col - row;
        if (dx >= 0 && dx < 7) {
          float v = acc[t][e] * inv;
          if (leaky) v = v > 0.f ? v : 0.1f * v;
          so[(warp * CM_TW + row) * 64 + dy * 7 + dx] = __float2bfloat16_rn(v);
        }
      }
    }
  }
  __syncthreads();
  // ---- write the tile: 128 pixels x 128 bytes
  for (int i = tid; i < CM_TW * CM_TH * 8; i += CM_THREADS) {
    const int m = i >> 3, ch = i & 7;
    const int ox = x0 + (m & 15), oy = y0 + (m >> 4);
    if (ox < out.W && oy < out.H) *reinterpret_cast<uint4*>(out.at(n, oy, ox) + ch * 8) = *reinterpret_cast<const uint4*>(s_out + (size_t)m * 128 + ch * 16);
  }
}

__global__ void __launch_bounds__(CM_THREADS, 2)
k_corr_mma(Ten<const bf16> f1, Ten<const bf16> f2, int f2_nxor, const float* __restrict__ flow, long long fN, long long fH, long long fW,
           float scale, int stride, int leaky, Ten<bf16> out) {
  // Channels are walked in slices of 64 (one 128-byte swizzle row per pixel): the tile of the first map, the patch of the second and
  // the output staging take 75 KB whatever C is, so two to three blocks share an SM; the 7 x 3 accumulator tiles of all
  // displacement rows stay in registers across the slices.
  constexpr int pitch = 128;
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t* s_f1 = smem;                                              // [128 px][128 B]
  uint8_t* s_p = s_f1 + (size_t)CM_TW * CM_TH * pitch;               // [14 * 24 px][128 B]
  uint8_t* s_out = s_p + (size_t)CM_PH * CM_PW * pitch;              // [128 px][128 B]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int x0 = blockIdx.x * CM_TW, y0 = blockIdx.y * CM_TH, n = blockIdx.z;
  const int C = f1.C;
  const int n2 = n ^ f2_nxor;
  const uint32_t f1_base = cm_smem(s_f1), p_base = cm_smem(s_p);
  const int arow = warp * CM_TW + (lane & 7) + ((lane >> 3) & 1) * 8;          // A: pixel of this lane's ldmatrix row
  const int akc = lane >> 4;                                                  //    k-chunk within the k16 step
  const int brow4 = (lane & 7) + ((lane >> 4) & 1) * 8, bkc = (lane >> 3) & 1; // B x4: two n8 tiles;  B x2 uses lanes 0..15
  float acc[7][3][4];
#pragma unroll
  for (int dy = 0; dy < 7; ++dy)
#pragma unroll
    for (int t = 0; t < 3; ++t) { acc[dy][t][0] = acc[dy][t][1] = acc[dy][t][2] = acc[dy][t][3] = 0.f; }
  // zero the pad channels 49..63 of the output staging once (channel 48 is rewritten by the band extraction)
  for (int i = tid; i < CM_TW * CM_TH * 2; i += CM_THREADS)
    *reinterpret_cast<uint4*>(s_out + (size_t)(i >> 1) * 128 + 96 + (i & 1) * 16) = make_uint4(0u, 0u, 0u, 0u);

#pragma unroll 1
  for (int c0 = 0; c0 < C; c0 += 64) {
    const int cs = min(64, C - c0), nch = cs >> 3;                   // channels / 16-byte chunks of this slice
    if (c0) __syncthreads();                                         // the previous slice's fragments have been read
    // ---- stage the first map's tile (pixels sampled with the stride)
    for (int i = tid; i < CM_TW * CM_TH * nch; i += CM_THREADS) {
      const int m = i / nch, ch = i - m * nch;
      const int ox = x0 + (m & 15), oy = y0 + (m >> 4);
      uint4 v = make_uint4(0u, 0u, 0u, 0u);
      if (ox < out.W && oy < out.H) v = *reinterpret_cast<const uint4*>(f1.at(n, oy * stride, ox * stride) + c0 + ch * 8);
      *reinterpret_cast<uint4*>(s_f1 + cm_off(m, ch, pitch)) = v;
    }
    // ---- stage the second map's patch: plain copy, or the Backward warp evaluated here
    for (int i = tid; i < CM_PH * CM_PW * nch; i += CM_THREADS) {
      const int q = i / nch, ch = i - q * nch;
      const int pj = q / CM_PW, pi = q - pj * CM_PW;
      const int sx = (x0 + pi - 3) * stride, sy = (y0 + pj - 3) * stride;
      uint4 v = make_uint4(0u, 0u, 0u, 0u);
      if (pi < CM_TW + 6 && sx >= 0 && sx < f2.W && sy >= 0 && sy < f2.H) {
        if (flow == nullptr) {
          v = *reinterpret_cast<const uint4*>(f2.at(n2, sy, sx) + c0 + ch * 8);
        } else {
          // Backward (lite_flow_net.py:10-28): bilinear sample at (x, y) + flow * scale, zeros outside; same arithmetic as
          // flow_ops.cu::k_warp_bilinear_vec (fp32 blend, round to bf16)
          const float* fl = flow + n * fN + (long long)sy * fH + (long long)sx * fW;
          const float px = (float)sx + fl[0] * scale, py = (float)sy + fl[1] * scale;
          const float fx0 = floorf(px), fy0 = floorf(py);
          const int ix = (int)fx0, iy = (int)fy0;
          const float wx1 = px - fx0, wy1 = py - fy0, wx0 = 1.f - wx1, wy0 = 1.f - wy1;
          const bool fin = (px == px) && (py == py) && fabsf(px) < 1e9f && fabsf(py) < 1e9f;      // non-finite coordinates sample nothing
          float w8[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) w8[j] = 0.f;
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int xx = ix + (k & 1), yy = iy + (k >> 1);
            const float wgt = ((k & 1) ? wx1 : wx0) * ((k >> 1) ? wy1 : wy0);
            if (!fin || xx < 0 || xx > f2.W - 1 || yy < 0 || yy > f2.H - 1 || wgt == 0.f) continue;
            const uint4 t = *reinterpret_cast<const uint4*>(f2.at(n2, yy, xx) + c0 + ch * 8);
            const uint32_t w4[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              w8[2 * j] += __uint_as_float(w4[j] << 16) * wgt;
              w8[2 * j + 1] += __uint_as_float(w4[j] & 0xffff0000u) * wgt;
            }
          }
          uint32_t o4[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const __nv_bfloat162 h = __floats2bfloat162_rn(w8[2 * j], w8[2 * j + 1]);
            o4[j] = *reinterpret_cast<const uint32_t*>(&h);
          }
          v = make_uint4(o4[0], o4[1], o4[2], o4[3]);
        }
      }
      *reinterpret_cast<uint4*>(s_p + cm_off(q, ch, pitch)) = v;
    }
    __syncthreads();
    // ---- banded GEMMs: warp w = output row w of the tile; the A fragments of a k16 step serve all seven displacement rows
    for (int ks = 0; ks < (cs >> 4); ++ks) {
      uint32_t a0, a1, a2, a3;
      cm_ldsm4(f1_base + cm_off(arow, 2 * ks + akc, pitch), a0, a1, a2, a3);
#pragma unroll
      for (int dy = 0; dy < 7; ++dy) {
        const int prow = (warp + dy) * CM_PW;                                     // patch row of this output row and displacement
        uint32_t b0, b1, b2, b3, b4, b5;
        cm_ldsm4(p_base + cm_off(prow + brow4, 2 * ks + bkc, pitch), b0, b1, b2, b3);       // columns 0..15
        cm_ldsm2(p_base + cm_off(prow + 16 + (lane & 7), 2 * ks + bkc, pitch), b4, b5);      // columns 16..23
        cm_mma(acc[dy][0], a0, a1, a2, a3, b0, b1);
        cm_mma(acc[dy][1], a0, a1, a2, a3, b2, b3);
        cm_mma(acc[dy][2], a0, a1, a2, a3, b4, b5);
      }
    }
  }
  // ---- band extraction: accumulator e of tile t sits at (row, col) = (g + 8 * (e >> 1), 8 * t + 2 * tq + (e & 1)); dx = col - row
  const float inv = 1.f / (float)C;
  const int g = lane >> 2, tq = lane & 3;
  __nv_bfloat16* so = reinterpret_cast<__nv_bfloat16*>(s_out);
#pragma unroll
  for (int dy = 0; dy < 7; ++dy)
#pragma unroll
    for (int t = 0; t < 3; ++t)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int row = g + 8 * (e >> 1), col = 8 * t + 2 * tq + (e & 1);
        const int dx = col - row;
        if (dx >= 0 && dx < 7) {
          float v = acc[dy][t][e] * inv;
          if (leaky) v = v > 0.f ? v : 0.1f * v;
          so[(warp * CM_TW + row) * 64 + dy * 7 + dx] = __float2bfloat16_rn(v);
        }
      }
  __syncthreads();
  // ---- write the tile: 128 pixels x 128 bytes
  for (int i = tid; i < CM_TW * CM_TH * 8; i += CM_THREADS) {
    const int m = i >> 3, ch = i & 7;
    const int ox = x0 + (m & 15), oy = y0 + (m >> 4);
    if (ox < out.W && oy < out.H) *reinterpret_cast<uint4*>(out.at(n, oy, ox) + ch * 8) = *reinterpret_cast<const uint4*>(s_out + (size_t)m * 128 + ch * 16);
  }
}

static bool corr_mma_ok(Ten<const bf16> f1, Ten<const bf16> f2, Ten<bf16> out) {
  static int on = -1;
  if (on < 0) { const char* e = getenv("DFVO_CORR_MMA"); on = !(e && atoi(e) == 0); }
  return on && f1.C % 16 == 0 && out.C == 64 && out.sW == 64 && ((uintptr_t)f1.p & 15) == 0 && ((uintptr_t)f2.p & 15) == 0 &&
         ((uintptr_t)out.p & 15) == 0 && f1.sW % 8 == 0 && f2.sW % 8 == 0 && f1.sH % 8 == 0 && f2.sH % 8 == 0 && f1.sN % 8 == 0 && f2.sN % 8 == 0 &&
         out.sH % 8 == 0 && out.sN % 8 == 0;
}
#endif  // !DFVO_HOSTSIM

// first: [N,H,W,C]; feat2: the map the second operand comes from (batch entry n ^ feat2_nxor); flow (may be null): [N,H,W,2] fp32
// displacement field applied to feat2 (Backward warp with `scale`); warp_scratch: [N,H,W,C] buffer for the un-fused fallback.
template <typename T>
int correlation49_warped(Ten<const T> first, Ten<const T> feat2, int feat2_nxor, Ten<const float> flow, float scale, int stride, int leaky,
                         Ten<T> warp_scratch, Ten<T> out, cudaStream_t s) {
  const bool has_flow = flow.p != nullptr;
  if (has_flow) {
    int rc = warp_bilinear<T>(feat2, flow, scale, feat2_nxor, warp_scratch, s);
    if (rc) return rc;
    return correlation49<T>(first, cten(warp_scratch), 0, stride, leaky, out, s);
  }
  return correlation49<T>(first, feat2, feat2_nxor, stride, leaky, out, s);
}

#ifndef DFVO_HOSTSIM
template <>
int correlation49_warped<bf16>(Ten<const bf16> first, Ten<const bf16> feat2, int feat2_nxor, Ten<const float> flow, float scale, int stride, int leaky,
                               Ten<bf16> warp_scratch, Ten<bf16> out, cudaStream_t s) {
  DFVO_REQUIRE(stride == 1 || stride == 2, DFVO_EINVAL, "correlation stride must be 1 or 2");
  DFVO_REQUIRE(out.H == (first.H + stride - 1) / stride && out.W == (first.W + stride - 1) / stride && out.C >= 49 && first.C == feat2.C &&
                   first.H == feat2.H && first.W == feat2.W,
               DFVO_ESHAPE, "correlation shapes");
  const bool has_flow = flow.p != nullptr;
  if (!corr_mma_ok(first, feat2, out)) {
    if (has_flow) {
      int rc = warp_bilinear<bf16>(feat2, flow, scale, feat2_nxor, warp_scratch, s);
      if (rc) return rc;
      return correlation49<bf16>(first, cten(warp_scratch), 0, stride, leaky, out, s);
    }
    return correlation49<bf16>(first, feat2, feat2_nxor, stride, leaky, out, s);
  }
  const size_t smem = (size_t)(CM_TW * CM_TH + CM_PH * CM_PW) * 128 + (size_t)CM_TW * CM_TH * 128;
  static bool attr_set = false;
  if (!attr_set) {
    DFVO_CUDA(cudaFuncSetAttribute(k_corr_mma, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    DFVO_CUDA(cudaFuncSetAttribute(k_corr_mma1, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr_set = true;
  }
  dim3 grid(cdiv(out.W, CM_TW), cdiv(out.H, CM_TH), out.N);
  ++g_launch_count;
  if (first.C <= 64)
    k_corr_mma1<<<grid, CM_THREADS, smem, s>>>(first, feat2, feat2_nxor, has_flow ? flow.p : nullptr, flow.sN, flow.sH, flow.sW, scale, stride, leaky, out, 128);
  else
    k_corr_mma<<<grid, CM_THREADS, smem, s>>>(first, feat2, feat2_nxor, has_flow ? flow.p : nullptr, flow.sN, flow.sH, flow.sW, scale, stride, leaky, out);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}
#endif

template int correlation49_warped<float>(Ten<const float>, Ten<const float>, int, Ten<const float>, float, int, int, Ten<float>, Ten<float>, cudaStream_t);
#ifdef DFVO_HOSTSIM
template int correlation49_warped<bf16>(Ten<const bf16>, Ten<const bf16>, int, Ten<const float>, float, int, int, Ten<bf16>, Ten<bf16>, cudaStream_t);
#endif

}  // namespace dfvo
