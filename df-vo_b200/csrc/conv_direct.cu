// CUDA-core implicit-GEMM convolution (fp32 accumulate), NHWC, any kernel size / stride, zero or
// reflection padding, fused bias + activation + residual.  Used for the layers the wgmma kernel
// does not cover (3-channel 7x7 stems, stride-2 convs, 1-channel heads) and for the all-fp32
// "exact" mode the parity tests use.  Restates torch.nn.Conv2d as used at lite_flow_net.py:39-75
// and resnet_encoder.py / layers.py:121-136 (ReflectionPad2d(1) + 3x3).
//
// Tiling: 64 output pixels x 64 output channels per 256-thread block, K = kh*kw*Cin consumed 16
// at a time through shared memory; each thread owns a 4x4 register tile.
#include "ops.h"

namespace dfvo {

#define CD_BM 64
#define CD_BN 64
#define CD_BK 16

DFVO_D int reflect_idx(int i, int n) {
  if (i < 0) i = -i;
  if (i >= n) i = 2 * (n - 1) - i;
  return i;
}

template <typename TI, typename TO>
__global__ void __launch_bounds__(256)
k_conv_direct(ConvDirect c, Ten<const TI> in, Ten<TO> out, Ten<const TO> res, int has_res) {
  __shared__ float As[CD_BK][CD_BM + 4];
  __shared__ float Bs[CD_BK][CD_BN + 4];
  const int tid = threadIdx.x;
  const int tn = tid % 16, tm = tid / 16;          // 16x16 threads, 4x4 outputs each
  const long long npix = (long long)out.N * out.H * out.W;
  const long long p0 = (long long)blockIdx.x * CD_BM;
  const int n0 = blockIdx.y * CD_BN;
  const int K = c.kh * c.kw * c.Cin;

  // A-load assignment: thread loads 4 consecutive k for one pixel
  const int a_px = tid / 4, a_k4 = (tid % 4) * 4;
  long long ap = p0 + a_px;
  const bool a_valid = ap < npix;
  int an = 0, ay = 0, ax = 0;
  if (a_valid) {
    ax = (int)(ap % out.W);
    ay = (int)((ap / out.W) % out.H);
    an = (int)(ap / ((long long)out.W * out.H));
  }
  // B-load assignment: thread loads 4 consecutive couts for one k
  const int b_k = tid / 16, b_n4 = (tid % 16) * 4;

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < K; k0 += CD_BK) {
    // ---- stage A (gathered input patch values) ----
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int k = k0 + a_k4 + j;
      float v = 0.f;
      if (a_valid && k < K) {
        int tap = k / c.Cin, ci = k - tap * c.Cin;
        int ky = tap / c.kw, kx = tap - ky * c.kw;
        int iy = ay * c.stride + ky - c.pad_y, ix = ax * c.stride + kx - c.pad_x;
        if (c.reflect) {
          iy = reflect_idx(iy, in.H); ix = reflect_idx(ix, in.W);
          v = to_f(in.at(an, iy, ix)[ci]);
        } else if (iy >= 0 && iy < in.H && ix >= 0 && ix < in.W) {
          v = to_f(in.at(an, iy, ix)[ci]);
        }
      }
      As[a_k4 + j][a_px] = v;
    }
    // ---- stage B (weights) ----
    {
      int k = k0 + b_k;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        int co = n0 + b_n4 + j;
        Bs[b_k][b_n4 + j] = (k < K && co < c.Cout) ? c.w[(size_t)k * c.w_pitch + co] : 0.f;
      }
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < CD_BK; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[kk][tm * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Bs[kk][tn * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] += a[i] * b[j];
    }
    __syncthreads();
  }

  // ---- epilogue ----
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    long long p = p0 + tm * 4 + i;
    if (p >= npix) continue;
    int x = (int)(p % out.W), y = (int)((p / out.W) % out.H), n = (int)(p / ((long long)out.W * out.H));
    TO* o = out.at(n, y, x);
    const TO* r = has_res ? res.at(n, y, x) : nullptr;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int co = n0 + tn * 4 + j;
      if (co >= c.Cout) continue;
      float v = acc[i][j] + (c.bias ? c.bias[co] : 0.f);
      if (has_res) v += to_f(r[co]);
      o[co] = from_f<TO>(apply_act(v, c.act));
    }
  }
}

template <typename TI, typename TO>
int conv_direct(const ConvDirect& c, Ten<const TI> in, Ten<TO> out, Ten<const TO> residual, cudaStream_t s) {
  DFVO_REQUIRE(in.C >= c.Cin && out.C >= c.Cout, DFVO_ESHAPE, "conv_direct channels (in %d>=%d, out %d>=%d)",
               in.C, c.Cin, out.C, c.Cout);
  int eh = (in.H + 2 * c.pad_y - c.kh) / c.stride + 1, ew = (in.W + 2 * c.pad_x - c.kw) / c.stride + 1;
  DFVO_REQUIRE(eh == out.H && ew == out.W && in.N == out.N, DFVO_ESHAPE,
               "conv_direct spatial: expect %dx%d got %dx%d", eh, ew, out.H, out.W);
  long long npix = (long long)out.N * out.H * out.W;
  dim3 grid((unsigned)((npix + CD_BM - 1) / CD_BM), cdiv(c.Cout, CD_BN));
  auto k = k_conv_direct<TI, TO>;
  int has_res = residual.p != nullptr;
  DFVO_LAUNCH(k, grid, dim3(256), 0, s, c, in, out, residual, has_res);
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

template int conv_direct<float, float>(const ConvDirect&, Ten<const float>, Ten<float>, Ten<const float>, cudaStream_t);
template int conv_direct<bf16, bf16>(const ConvDirect&, Ten<const bf16>, Ten<bf16>, Ten<const bf16>, cudaStream_t);
template int conv_direct<float, bf16>(const ConvDirect&, Ten<const float>, Ten<bf16>, Ten<const bf16>, cudaStream_t);
template int conv_direct<bf16, float>(const ConvDirect&, Ten<const bf16>, Ten<float>, Ten<const float>, cudaStream_t);

}  // namespace dfvo
