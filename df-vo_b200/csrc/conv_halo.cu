// Halo-resident wgmma implicit-GEMM convolution for sm_90a (stride 1, rectangular kh x kw tap set, up to 3 virtually
// concatenated NHWC bf16 / fp32 sources, fused bias + activation + residual epilogue).
//
// Why a second kernel: conv_tc.cu loads one shifted A box per tap, so a 3x3 layer pulls every input pixel nine times and the
// full weight set once per 128 output pixels through L2 -> SM, and L2 bandwidth bounds such a layer well below the tensor rate.
// Here
//   * the A operand of a tile is ONE TMA box per 64-channel chunk: the (8S + kw - 1) x (16 + kh - 1) pixel halo
//     of the tile, 128 B per pixel, SWIZZLE_128B.  Every tap of the kh x kw window is the same shared-memory
//     data addressed through a wgmma descriptor whose start is shifted by (ky * halo_w + kx) pixels and whose
//     stride-byte-offset is one halo row: the 8-row groups of the K-major operand are the tile's pixel rows.
//     A 3x3 layer reads each input pixel 1.27x (S = 2) instead of 9x;
//   * one CTA owns S sub-tiles of 8 x 16 pixels (M = 128 each) that share every B (weight) stage, so the
//     weights cross L2 -> SM once per 128*S pixels;
//   * A and B have their own mbarrier rings and producer warps (a B slot is freed per tap, an A slot per chunk).
// Warp roles: 0 = A producer (TMA), 1 = B producer (TMA), 2-3 idle; warpgroups 1 and 2 = consumers (wgmma for pixel rows 0-7 / 8-15
// of every sub-tile, accumulators in registers, then the epilogue).  tc_ptx.cuh::halo_tile_mma is the MMA loop.
// Restates torch.nn.Conv2d(stride=1) + LeakyReLU/ELU/ReLU as used at lite_flow_net.py:98-240 and
// depth_decoder.py / torchvision BasicBlock (BN folded by the weight packer), like conv_tc.cu.
#include "tc_ptx.cuh"

#ifndef DFVO_HOSTSIM
#include <cuda.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

namespace dfvo {

struct ConvHaloK {
  int N, H, W, tiles_x, tiles_y, n_blocks, ntiles;
  int nsrc, srcC[3];
  int kh, kw, dy0, dx0;          // input pixel of tap (ky,kx) for output (y,x): (y + dy0 + ky, x + dx0 + kx)
  int HW, HH;                    // halo box, pixels
  int a_stages, b_stages, a_stage_bytes;
  int Cout, Cout_pad, act, out_f32, zero_pad_to;
  int chunk;                     // channels per 128-byte operand row: 64 (bf16) or 32 (fp32 read as tf32)
  int esize, round_tf32;
  const float* bias;
  void* out; long long oN, oH, oW;
  const void* res; long long rN, rH, rW;
};

#define HALO_THREADS 384
#define HALO_TH 16

template <int S, int BN, int TF32>
__global__ void __launch_bounds__(HALO_THREADS, 1)
k_conv_halo(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
            const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB,
            const __grid_constant__ ConvHaloK p) {
  using namespace tc;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;                 // SWIZZLE_128B pattern repeats every 1024 B
  uint8_t* base_ptr = smem_raw + (base - raw);
  const uint32_t b_stage_bytes = (uint32_t)BN * 128u;
  const uint32_t a_base = base;
  const uint32_t b_base = base + (uint32_t)p.a_stages * (uint32_t)p.a_stage_bytes;
  // [A ring][B ring][barriers: a_full[A], a_empty[A], b_full[B], b_empty[B]][bias]
  const uint32_t bar_base = b_base + (uint32_t)p.b_stages * b_stage_bytes;
  TcRing ra{a_base, (uint32_t)p.a_stage_bytes, bar_base, bar_base + 8u * (uint32_t)p.a_stages, p.a_stages, 0, 0u};
  TcRing rb{b_base, b_stage_bytes, bar_base + 16u * (uint32_t)p.a_stages, bar_base + 16u * (uint32_t)p.a_stages + 8u * (uint32_t)p.b_stages,
            p.b_stages, 0, 0u};
  float* bias_s = reinterpret_cast<float*>(base_ptr + (bar_base - base) + 16u * (uint32_t)(p.a_stages + p.b_stages));

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  pdl_trigger();

  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tmA0); prefetch_tmap(&tmB);
    for (int s = 0; s < p.a_stages; ++s) { mbar_init(ra.full0 + 8u * s, 1); mbar_init(ra.empty0 + 8u * s, 2); }
    for (int s = 0; s < p.b_stages; ++s) { mbar_init(rb.full0 + 8u * s, 1); mbar_init(rb.empty0 + 8u * s, 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int ntaps = p.kh * p.kw;
  pdl_wait();                                  // from here on: activations of the previous kernel / our output buffers

  if (warp == 0) {
    // ===================================== A producer: one halo box per (tile, source, 64-channel chunk)
    const uint32_t a_bytes = (uint32_t)p.HW * (uint32_t)p.HH * 128u;
    for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
      int t = tile;
      const int tx = t % p.tiles_x; t /= p.tiles_x;
      const int ty = t % p.tiles_y; t /= p.tiles_y;
      const int n = t % p.N;
      const int x0 = tx * 8 * S + p.dx0, y0 = ty * HALO_TH + p.dy0;
      for (int s = 0; s < p.nsrc; ++s) {
        const CUtensorMap* tm = s == 0 ? &tmA0 : (s == 1 ? &tmA1 : &tmA2);
        for (int c0 = 0; c0 < p.srcC[s]; c0 += p.chunk) {
          mbar_wait(ra.empty(), ra.ph ^ 1u);
          if (elect_one()) {
            mbar_expect_tx(ra.full(), a_bytes);
            tma_load_4d(ra.slot(), tm, ra.full(), c0, x0, y0, n);
          }
          __syncwarp();
          ra.next();
        }
      }
    }
  } else if (warp == 1) {
    // ===================================== B producer: one weight box per (tile, chunk, tap)
    for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
      const int nb = tile / (p.tiles_x * p.tiles_y * p.N);
      int kofs = 0;
      for (int s = 0; s < p.nsrc; ++s) {
        for (int c0 = 0; c0 < p.srcC[s]; c0 += p.chunk) {
          for (int tap = 0; tap < ntaps; ++tap) {
            mbar_wait(rb.empty(), rb.ph ^ 1u);
            if (elect_one()) {
              mbar_expect_tx(rb.full(), b_stage_bytes);
              tma_load_3d(rb.slot(), &tmB, rb.full(), kofs + c0, nb * BN, tap);
            }
            __syncwarp();
            rb.next();
          }
        }
        kofs += p.srcC[s];
      }
    }
  } else if (warp >= 4) {
    // ============================ two consumer warpgroups: MMA + epilogue ============================
    const int ct = threadIdx.x - 128, wg = ct >> 7;
    // bias staging belongs to the consumers (the producers start on the barrier-init sync instead of waiting for a global load)
    for (int i = ct; i < p.Cout_pad; i += 256) bias_s[i] = p.bias ? p.bias[i] : 0.f;
    asm volatile("bar.sync 1, 256;" ::: "memory");
    TcEpi ep; ep.Cout = p.Cout; ep.zero_pad_to = p.zero_pad_to; ep.act = p.act; ep.out_f32 = p.out_f32; ep.round_tf32 = p.round_tf32; ep.out = p.out; ep.res = p.res;
    float acc[S][BN / 2];
    for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
      halo_tile_mma<S, BN, TF32>(acc, ra, rb, p.nsrc, p.srcC, p.chunk, p.esize, p.kh, p.kw, p.HW, wg, (ct & 127) == 0);
      int t = tile;
      const int tx = t % p.tiles_x; t /= p.tiles_x;
      const int ty = t % p.tiles_y; t /= p.tiles_y;
      const int n = t % p.N; const int nb = t / p.N;
      halo_tile_store<S, BN>(acc, ep, bias_s, nb * BN, n, tx * 8 * S, ty * HALO_TH, p.W, p.H, p.oN, p.oH, p.oW, p.rN, p.rH, p.rW, wg,
                             (ct >> 5) & 3, lane);
    }
  }
}

// =============================================================================================
//                                        host side
// =============================================================================================
static int env_int(const char* name, int dflt) {
  const char* v = getenv(name);
  return v ? atoi(v) : dflt;
}

static bool rect_taps(const ConvTc& c, int* kh, int* kw, int* dy0, int* dx0) {
  // taps must enumerate a full kh x kw rectangle in row-major order (what fill_taps produces)
  int ymin = 127, ymax = -128, xmin = 127, xmax = -128;
  for (int t = 0; t < c.ntaps; ++t) {
    if (c.dy[t] < ymin) ymin = c.dy[t];
    if (c.dy[t] > ymax) ymax = c.dy[t];
    if (c.dx[t] < xmin) xmin = c.dx[t];
    if (c.dx[t] > xmax) xmax = c.dx[t];
  }
  const int h = ymax - ymin + 1, w = xmax - xmin + 1;
  if (h * w != c.ntaps) return false;
  for (int t = 0; t < c.ntaps; ++t)
    if (c.dy[t] != ymin + t / w || c.dx[t] != xmin + t % w) return false;
  *kh = h; *kw = w; *dy0 = ymin; *dx0 = xmin;
  return true;
}

struct HaloCfg { int S, block_n, a_stages, b_stages, a_stage_bytes; size_t smem; double cost; };

// shared memory: A ring + B ring + barriers + bias (+ 1 KB alignment slack)
static bool halo_fit(int S, int bn, int kh, int kw, int Cout_pad, HaloCfg* out) {
  const int HW = 8 * S + kw - 1, HH = HALO_TH + kh - 1;
  if (HW > 256 || HH > 256) return false;
  const int a_stage = (HW * HH * 128 + 1023) & ~1023;
  const int b_stage = bn * 128;
  const size_t fixed = 1024 + 8 * 64 + (size_t)Cout_pad * 4;      // alignment slack, <= 30 barriers, bias
  const size_t budget = 220 * 1024;
  int a_stages = 2, b_stages = 2;
  if (fixed + (size_t)a_stages * a_stage + (size_t)b_stages * b_stage > budget) return false;
  // a B slot lives for one tap (S MMAs per K step), an A slot for a whole chunk (kh*kw taps): two A slots already cover the
  // TMA latency, so the B ring grows first (up to 8 slots in flight), then a third A slot, then B up to 12
  while (b_stages < 8 && fixed + (size_t)a_stages * a_stage + (size_t)(b_stages + 1) * b_stage <= budget) ++b_stages;
  while (a_stages < 3 && fixed + (size_t)(a_stages + 1) * a_stage + (size_t)b_stages * b_stage <= budget) ++a_stages;
  while (b_stages < 12 && fixed + (size_t)a_stages * a_stage + (size_t)(b_stages + 1) * b_stage <= budget) ++b_stages;
  out->S = S; out->block_n = bn; out->a_stages = a_stages; out->b_stages = b_stages; out->a_stage_bytes = a_stage;
  out->smem = fixed + (size_t)a_stages * a_stage + (size_t)b_stages * b_stage;
  return true;
}

// Pick (S, block_n): minimise  waves x max(MMA time, L2->SM time)  per tile + a fixed per-tile overhead.  An estimate from the
// H100 SXM data sheet, not a measurement: per K=16 step of the 128-pixel sub-tile, MMA time = max(block_n, 32 + block_n / 2) clk
// (tensor rate of ~2048 bf16 MACs / clk / SM vs shared-memory operand reads at 128 B / clk); L2 -> SM ~25 B/clk per SM when every
// SM streams (~3.3 KB / clk for the chip), up to ~5x that for a lone CTA.  block_n is one of the wgmma shapes 16 .. 256 and
// S * block_n <= 256 keeps the accumulators of a consumer thread at <= 128 registers.
static bool halo_choose(const ConvTc& c, int kh, int kw, HaloCfg* best) {
  int ktot16 = 0, kbytes = 0;                       // 32-byte K steps and bytes per pixel over all sources
  const int es = c.esize == 4 ? 4 : 2;
  for (int s = 0; s < c.nsrc; ++s) { ktot16 += (c.src[s].C * es + 31) / 32; kbytes += c.src[s].C * es; }
  const int nsm = tc_num_sms();
  const int fS = env_int("DFVO_HALO_S", 0), fN = env_int("DFVO_HALO_BN", 0);
  bool found = false;
  for (int S = 1; S <= 4; S <<= 1) {
    if (fS && S != fS) continue;
    for (int bn = 16; bn <= 256 && bn <= c.Cout_pad; bn <<= 1) {
      if (c.Cout_pad % bn || S * bn > 256) continue;
      if (fN && bn != fN) continue;
      HaloCfg h;
      if (!halo_fit(S, bn, kh, kw, c.Cout_pad, &h)) continue;
      const long long tiles = (long long)cdiv(c.W, 8 * S) * cdiv(c.H, HALO_TH) * c.N * (c.Cout_pad / bn);
      const long long waves = (tiles + nsm - 1) / nsm;
      const int active = (int)(tiles < nsm ? tiles : nsm);
      const double mma = (double)ktot16 * kh * kw * S * ((bn > 32 + bn / 2.0) ? bn : 32 + bn / 2.0);
      const double bytes = (double)(8 * S + kw - 1) * (HALO_TH + kh - 1) * kbytes + (double)kh * kw * bn * kbytes;
      double bw = 3300.0 / active; if (bw > 128.0) bw = 128.0;
      const double l2 = bytes / bw;
      const double epi = (double)S * bn * 10.0;                 // ~epilogue clk per tile (not overlapped with the MMAs)
      const double tile = (mma > l2 ? mma : l2) + epi;
      h.cost = (double)waves * (tile + 1500.0) + 4000.0;        // per-tile pipeline bubble, per-launch prologue
      if (!found || h.cost < best->cost) { *best = h; found = true; }
    }
  }
  return found;
}

bool conv_halo_supported(const ConvTc& c) {
  if (env_int("DFVO_CONV_HALO", 1) == 0) return false;
  if (c.stride == 2) return false;
  int kh, kw, dy0, dx0;
  if (!rect_taps(c, &kh, &kw, &dy0, &dx0)) return false;
  HaloCfg h;
  return halo_choose(c, kh, kw, &h);
}

template <int S, int BN, int TF32>
static int launch_halo(const CUtensorMap* tmA, const CUtensorMap& tmB, const ConvHaloK& k, int grid, size_t smem, cudaStream_t s) {
  static bool attr_set = false;
  if (!attr_set) {
    DFVO_CUDA(cudaFuncSetAttribute(k_conv_halo<S, BN, TF32>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_set = true;
  }
  cudaLaunchConfig_t cfg; cudaLaunchAttribute attr;
  tc_launch_config(&cfg, &attr, grid, HALO_THREADS, smem, s);
  DFVO_CUDA(cudaLaunchKernelEx(&cfg, k_conv_halo<S, BN, TF32>, tmA[0], tmA[1], tmA[2], tmB, k));
  return DFVO_OK;
}

template <int TF32>
static int launch_halo_t(int S, int bn, const CUtensorMap* tmA, const CUtensorMap& tmB, const ConvHaloK& k, int grid, size_t smem,
                         cudaStream_t s) {
#define DFVO_HALO_CASE(SS, NN) if (S == SS && bn == NN) return launch_halo<SS, NN, TF32>(tmA, tmB, k, grid, smem, s);
  DFVO_HALO_CASE(1, 16) DFVO_HALO_CASE(1, 32) DFVO_HALO_CASE(1, 64) DFVO_HALO_CASE(1, 128) DFVO_HALO_CASE(1, 256)
  DFVO_HALO_CASE(2, 16) DFVO_HALO_CASE(2, 32) DFVO_HALO_CASE(2, 64) DFVO_HALO_CASE(2, 128)
  DFVO_HALO_CASE(4, 16) DFVO_HALO_CASE(4, 32) DFVO_HALO_CASE(4, 64)
#undef DFVO_HALO_CASE
  DFVO_REQUIRE(false, DFVO_EINVAL, "conv_halo: no kernel for S %d block_n %d", S, bn);
}

int conv_halo(const ConvTc& c, cudaStream_t s) {
  DFVO_REQUIRE(c.nsrc >= 1 && c.nsrc <= 3 && c.ntaps >= 1 && c.ntaps <= 49, DFVO_EINVAL, "conv_halo: nsrc/ntaps");
  DFVO_REQUIRE(c.Cout_pad % 16 == 0 && c.Cout_pad >= 16, DFVO_EINVAL, "conv_halo: Cout_pad %d must be a multiple of 16", c.Cout_pad);
  ConvHaloK k;
  memset(&k, 0, sizeof(k));
  DFVO_REQUIRE(rect_taps(c, &k.kh, &k.kw, &k.dy0, &k.dx0), DFVO_EINVAL, "conv_halo: taps are not a rectangle");
  HaloCfg h;
  DFVO_REQUIRE(halo_choose(c, k.kh, k.kw, &h), DFVO_EINVAL, "conv_halo: no tile configuration fits");
  const int S = h.S, bn = h.block_n;
  k.N = c.N; k.H = c.H; k.W = c.W;
  k.tiles_x = cdiv(c.W, 8 * S); k.tiles_y = cdiv(c.H, HALO_TH);
  k.n_blocks = c.Cout_pad / bn;
  k.ntiles = k.tiles_x * k.tiles_y * c.N * k.n_blocks;
  k.HW = 8 * S + k.kw - 1; k.HH = HALO_TH + k.kh - 1;
  k.a_stages = h.a_stages; k.b_stages = h.b_stages; k.a_stage_bytes = h.a_stage_bytes;
  k.nsrc = c.nsrc;
  const int es = c.esize == 4 ? 4 : 2;
  k.esize = es; k.chunk = 128 / es; k.round_tf32 = c.round_out_tf32;
  int ktot = 0;
  for (int i = 0; i < c.nsrc; ++i) {
    DFVO_REQUIRE(c.src[i].C % 16 == 0 && c.src[i].C > 0, DFVO_EINVAL, "conv_halo: source %d channels %d not a multiple of 16", i, c.src[i].C);
    DFVO_REQUIRE(((uintptr_t)c.src[i].p & 15) == 0 && (c.src[i].sW * es) % 16 == 0 && (c.src[i].sH * es) % 16 == 0 && (c.src[i].sN * es) % 16 == 0,
                 DFVO_EINVAL, "conv_halo: source %d not 16-byte aligned/strided", i);
    k.srcC[i] = c.src[i].C; ktot += c.src[i].C;
  }
  k.Cout = c.Cout; k.Cout_pad = c.Cout_pad; k.act = c.act; k.out_f32 = c.out_f32;
  k.zero_pad_to = c.zero_pad_to > c.Cout ? c.zero_pad_to : c.Cout;
  k.bias = c.bias; k.out = c.out; k.oN = c.oN; k.oH = c.oH; k.oW = c.oW;
  k.res = c.residual; k.rN = c.rN; k.rH = c.rH; k.rW = c.rW;

  CUtensorMap tmA[3], tmB;
  for (int i = 0; i < 3; ++i) {
    const ConvTcSource& src = c.src[i < c.nsrc ? i : 0];
    const int inW = c.inW > 0 ? c.inW : c.W, inH = c.inH > 0 ? c.inH : c.H;
    unsigned long long dims[4] = {(unsigned long long)src.C, (unsigned long long)inW, (unsigned long long)inH, (unsigned long long)c.N};
    unsigned long long str[3] = {(unsigned long long)src.sW * es, (unsigned long long)src.sH * es, (unsigned long long)src.sN * es};
    unsigned box[4] = {(unsigned)k.chunk, (unsigned)k.HW, (unsigned)k.HH, 1};
    int rc = tc_encode_map(&tmA[i], src.p, 4, dims, str, box, es);
    if (rc) return rc;
  }
  {
    unsigned long long dims[3] = {(unsigned long long)ktot, (unsigned long long)c.Cout_pad, (unsigned long long)c.ntaps};
    unsigned long long str[2] = {(unsigned long long)ktot * es, (unsigned long long)ktot * es * (unsigned long long)c.Cout_pad};
    unsigned box[3] = {(unsigned)k.chunk, (unsigned)bn, 1};
    int rc = tc_encode_map(&tmB, c.w, 3, dims, str, box, es);
    if (rc) return rc;
  }
  const int grid = k.ntiles < tc_num_sms() ? k.ntiles : tc_num_sms();
  ++g_launch_count;
  TcProf pr;
  const bool prof = tc_prof_begin(s, &pr);
  const int rc = es == 4 ? launch_halo_t<1>(S, bn, tmA, tmB, k, grid, h.smem, s) : launch_halo_t<0>(S, bn, tmA, tmB, k, grid, h.smem, s);
  if (rc) return rc;
  if (prof) {
    char d[256];
    snprintf(d, sizeof(d), "halo%s N%d %dx%d k%dx%d src[%d,%d,%d] cout%d/%d bn%d S%d stages%d/%d grid%d tiles%d gflop %.3f", es == 4 ? "-tf32" : "", c.N, c.H, c.W,
             k.kh, k.kw, c.src[0].C, c.nsrc > 1 ? c.src[1].C : 0, c.nsrc > 2 ? c.src[2].C : 0, c.Cout, c.Cout_pad, bn,
             S, k.a_stages, k.b_stages, grid, k.ntiles, c.flops * 1e-9);
    tc_prof_end(s, pr, c.flops, d);
  }
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

}  // namespace dfvo
#endif  // !DFVO_HOSTSIM
