// Layer-chain convolution kernel: up to CHAIN_MAXL consecutive stride-1 convolutions of one network module (LiteFlowNet Matching /
// Subpixel / Regularization main stacks, lite_flow_net.py:98-240) in ONE persistent cooperative launch, with a grid-wide barrier
// between layers instead of a kernel boundary.
//
// Why: the coarse pyramid levels are chains of tiny layers (11x38 ... 44x152 pixels, 1 tile per CTA) whose few microseconds of
// work on the SM are small next to the fixed cost of a launch of their own (grid launch, ~200 KB shared-memory set-up, completion
// and flush).  Inside a chain a layer boundary is one release/acquire counter in global memory, and the weight stream of the next
// layer is prefetched across it (the B producer never waits for the barrier).
//
// Same tile machinery as conv_halo.cu (halo-resident A operand, shifted wgmma descriptors per tap, S sub-tiles share B, warp roles
// A-producer / B-producer / two consumer warpgroups: tc_ptx.cuh::halo_tile_mma + halo_tile_store); the ring geometry (slot sizes,
// stage counts) is fixed per chain, everything else (window, channels, block_n, activation, output) is per layer.
// Memory-model notes: a layer's outputs are written with generic-proxy stores by the consumer warps of all CTAs and read by the next
// layer's TMA loads (async proxy) of other CTAs.  Writers: st.global, fence.proxy.async, __threadfence, then ONE red.release.gpu per CTA.
// Reader (the A producer's elected lane): ld.acquire.gpu spin until all CTAs arrived, fence.proxy.async, then the TMA loads.
// All CTAs must be co-resident: the launcher uses a cooperative launch with grid <= #SMs (1 CTA per SM by shared memory).
#include "tc_ptx.cuh"

#ifndef DFVO_HOSTSIM
#include <cuda.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

namespace dfvo {

#define CHAIN_MAXL 12
#define CHAIN_THREADS 384
#define CHAIN_TH 16

struct ChainL {
  int N, H, W, tiles_x, tiles_y, n_blocks, ntiles;
  int nsrc, srcC[3];
  int kh, kw, dy0, dx0, HW, HH;
  int block_n;
  int Cout, Cout_pad, act, out_f32, zero_pad_to;
  const float* bias;
  void* out; long long oN, oH, oW;
  const void* res; long long rN, rH, rW;
};

struct alignas(64) ChainArgs {
  CUtensorMap tmA[CHAIN_MAXL][3];
  CUtensorMap tmB[CHAIN_MAXL];
  ChainL L[CHAIN_MAXL];
  int nlayers, a_stages, b_stages, a_stage_bytes, b_stage_bytes, bias_cap, pad0, pad1;
  unsigned* bar;            // [nlayers] arrival counters, zeroed by the launcher
  unsigned* err;            // set if a barrier wait gave up (watchdog)
};

__device__ __forceinline__ void chain_arrive(unsigned* ctr) {
  asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(ctr) : "memory");
}
__device__ __forceinline__ bool chain_wait(const unsigned* ctr, unsigned target) {
  for (unsigned spins = 0; spins < (1u << 24); ++spins) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory");
    if (v >= target) return true;
    __nanosleep(32);
  }
  return false;
}

// the tiles of one layer for one consumer warpgroup (block_n is a template parameter of the wgmma shape)
template <int S, int BN>
__device__ __noinline__ void chain_layer(const ChainL& p, TcRing& ra, TcRing& rb, const TcEpi& ep, const float* bias_s, int wg, int wq,
                                            int lane, bool leader) {
  float acc[S][BN / 2];
  for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
    halo_tile_mma<S, BN, 0>(acc, ra, rb, p.nsrc, p.srcC, 64, 2, p.kh, p.kw, p.HW, wg, leader);
    int t = tile;
    const int tx = t % p.tiles_x; t /= p.tiles_x;
    const int ty = t % p.tiles_y; t /= p.tiles_y;
    const int n = t % p.N; const int nb = t / p.N;
    halo_tile_store<S, BN>(acc, ep, bias_s, nb * BN, n, tx * 8 * S, ty * CHAIN_TH, p.W, p.H, p.oN, p.oH, p.oW, p.rN, p.rH, p.rW, wg, wq, lane);
  }
}

template <int S>
__global__ void __launch_bounds__(CHAIN_THREADS, 1)
k_conv_chain(const __grid_constant__ ChainArgs P) {
  using namespace tc;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* base_ptr = smem_raw + (base - raw);
  const uint32_t a_base = base;
  const uint32_t b_base = base + (uint32_t)P.a_stages * (uint32_t)P.a_stage_bytes;
  const uint32_t bar_base = b_base + (uint32_t)P.b_stages * (uint32_t)P.b_stage_bytes;
  TcRing ra{a_base, (uint32_t)P.a_stage_bytes, bar_base, bar_base + 8u * (uint32_t)P.a_stages, P.a_stages, 0, 0u};
  TcRing rb{b_base, (uint32_t)P.b_stage_bytes, bar_base + 16u * (uint32_t)P.a_stages, bar_base + 16u * (uint32_t)P.a_stages + 8u * (uint32_t)P.b_stages,
            P.b_stages, 0, 0u};
  float* bias_s = reinterpret_cast<float*>(base_ptr + (bar_base - base) + 16u * (uint32_t)(P.a_stages + P.b_stages));

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 0 && lane == 0) {
    for (int l = 0; l < P.nlayers; ++l) { prefetch_tmap(&P.tmA[l][0]); prefetch_tmap(&P.tmB[l]); }
    for (int s = 0; s < P.a_stages; ++s) { mbar_init(ra.full0 + 8u * s, 1); mbar_init(ra.empty0 + 8u * s, 2); }
    for (int s = 0; s < P.b_stages; ++s) { mbar_init(rb.full0 + 8u * s, 1); mbar_init(rb.empty0 + 8u * s, 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 0) {
    // ===================================== A producer ===================================================================
    for (int l = 0; l < P.nlayers; ++l) {
      const ChainL& p = P.L[l];
      if (l > 0) {                                            // every CTA has written its part of layer l-1
        if (elect_one()) {
          if (!chain_wait(P.bar + (l - 1), gridDim.x)) *P.err = 1u;
          asm volatile("fence.proxy.async;" ::: "memory");
        }
        __syncwarp();
      }
      const uint32_t a_bytes = (uint32_t)p.HW * (uint32_t)p.HH * 128u;
      for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
        int t = tile;
        const int tx = t % p.tiles_x; t /= p.tiles_x;
        const int ty = t % p.tiles_y; t /= p.tiles_y;
        const int n = t % p.N;
        const int x0 = tx * 8 * S + p.dx0, y0 = ty * CHAIN_TH + p.dy0;
        for (int s = 0; s < p.nsrc; ++s) {
          const CUtensorMap* tm = &P.tmA[l][s];
          for (int c0 = 0; c0 < p.srcC[s]; c0 += 64) {
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
    }
  } else if (warp == 1) {
    // ===================================== B producer: weights are constants -- runs ahead across layer boundaries ========
    for (int l = 0; l < P.nlayers; ++l) {
      const ChainL& p = P.L[l];
      const int ntaps = p.kh * p.kw;
      const uint32_t b_bytes = (uint32_t)p.block_n * 128u;
      for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
        const int nb = tile / (p.tiles_x * p.tiles_y * p.N);
        int kofs = 0;
        for (int s = 0; s < p.nsrc; ++s) {
          for (int c0 = 0; c0 < p.srcC[s]; c0 += 64) {
            for (int tap = 0; tap < ntaps; ++tap) {
              mbar_wait(rb.empty(), rb.ph ^ 1u);
              if (elect_one()) {
                mbar_expect_tx(rb.full(), b_bytes);
                tma_load_3d(rb.slot(), &P.tmB[l], rb.full(), kofs + c0, nb * p.block_n, tap);
              }
              __syncwarp();
              rb.next();
            }
          }
          kofs += p.srcC[s];
        }
      }
    }
  } else if (warp >= 4) {
    // ============================ two consumer warpgroups: MMA + epilogue ================================================
    const int ct = threadIdx.x - 128, wg = ct >> 7, wq = (ct >> 5) & 3;
    const bool leader = (ct & 127) == 0;
    for (int l = 0; l < P.nlayers; ++l) {
      const ChainL& p = P.L[l];
      // bias of this layer (the previous layer's tiles of this CTA are finished: its arrival below came after them)
      asm volatile("bar.sync 1, 256;" ::: "memory");
      for (int i = ct; i < p.Cout_pad; i += 256) bias_s[i] = p.bias ? p.bias[i] : 0.f;
      asm volatile("bar.sync 1, 256;" ::: "memory");
      if (l > 0 && p.res != nullptr) {                        // the residual may come from an earlier layer of this chain: acquire it
        if (lane == 0 && !chain_wait(P.bar + (l - 1), gridDim.x)) *P.err = 1u;
        __syncwarp();
      }
      TcEpi ep; ep.Cout = p.Cout; ep.zero_pad_to = p.zero_pad_to; ep.act = p.act; ep.out_f32 = p.out_f32; ep.round_tf32 = 0; ep.out = p.out; ep.res = p.res;
      switch (p.block_n) {
        case 16: chain_layer<S, 16>(p, ra, rb, ep, bias_s, wg, wq, lane, leader); break;
        case 32: chain_layer<S, 32>(p, ra, rb, ep, bias_s, wg, wq, lane, leader); break;
        case 64: chain_layer<S, 64>(p, ra, rb, ep, bias_s, wg, wq, lane, leader); break;
        case 128: if (S <= 2) chain_layer<S, (S <= 2 ? 128 : 16)>(p, ra, rb, ep, bias_s, wg, wq, lane, leader); break;
        default: if (S == 1) chain_layer<S, (S == 1 ? 256 : 16)>(p, ra, rb, ep, bias_s, wg, wq, lane, leader); break;
      }
      // this CTA's share of layer l is in global memory: publish it to the other CTAs' TMA loads
      if (l + 1 < P.nlayers) {
        asm volatile("fence.proxy.async;" ::: "memory");
        __threadfence();
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (ct == 0) chain_arrive(P.bar + l);
      }
    }
  }
}

// =====================================================================================================================
//                                               host side
// =====================================================================================================================
static int chain_env(const char* name, int dflt) {
  const char* v = getenv(name);
  return v ? atoi(v) : dflt;
}

static bool chain_rect(const ConvTc& c, int* kh, int* kw, int* dy0, int* dx0) {
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

bool conv_chain_eligible(const ConvTc& c) {
  if (c.stride == 2 || c.esize == 4 || c.nsrc < 1 || c.nsrc > 3) return false;
  // DFVO_CHAIN_MAX_PIXELS: only layers up to this many output pixels join chains (a chain is a cooperative launch -- all its CTAs must be
  // resident at once -- which costs concurrency with the other streams of the frame pipeline; the big levels gain little from chaining)
  static long long max_px = -1;
  if (max_px < 0) max_px = chain_env("DFVO_CHAIN_MAX_PIXELS", 1 << 30);
  if ((long long)c.N * c.H * c.W > max_px) return false;
  int kh, kw, dy0, dx0;
  if (!chain_rect(c, &kh, &kw, &dy0, &dx0)) return false;
  for (int i = 0; i < c.nsrc; ++i)
    if (c.src[i].C % 16 || ((uintptr_t)c.src[i].p & 15) || (c.src[i].sW * 2) % 16 || (c.src[i].sH * 2) % 16 || (c.src[i].sN * 2) % 16) return false;
  return c.Cout_pad % 16 == 0 && c.Cout_pad <= 256;
}

// per-K16-step clocks of one M = 128 MMA with N = bn: the larger of the tensor rate and the shared-memory operand reads (the
// estimate conv_halo.cu's halo_choose uses)
static double chain_mma_clk(int bn) { return bn > 32 + 0.5 * bn ? (double)bn : 32 + 0.5 * bn; }

int conv_chain_launch(const std::vector<ConvTc>& layers, unsigned* bar, cudaStream_t s) {
  const int n = (int)layers.size();
  DFVO_REQUIRE(n >= 1 && n <= CHAIN_MAXL, DFVO_EINVAL, "conv_chain: %d layers", n);
  const int nsm = tc_num_sms();
  // ---- common sub-tile count S and per-layer block_n from the cost model
  int bestS = 1; double bestCost = -1.0;
  int bn_for[3][CHAIN_MAXL];
  for (int si = 0; si < 3; ++si) {
    const int S = 1 << si;
    double cost = 0.0;
    bool okS = true;
    for (int l = 0; l < n && okS; ++l) {
      const ConvTc& c = layers[l];
      int kh, kw, dy0, dx0;
      chain_rect(c, &kh, &kw, &dy0, &dx0);
      int k16 = 0;
      for (int i = 0; i < c.nsrc; ++i) k16 += (c.src[i].C + 15) / 16;
      double bl = -1.0; int bbn = 0;
      for (int bn = 16; bn <= c.Cout_pad && bn <= 256; bn <<= 1) {         // the wgmma shapes 16 .. 256
        if (c.Cout_pad % bn || S * bn > 256) continue;
        const long long tiles = (long long)cdiv(c.W, 8 * S) * cdiv(c.H, CHAIN_TH) * c.N * (c.Cout_pad / bn);
        const long long waves = (tiles + nsm - 1) / nsm;
        const double mma = (double)k16 * kh * kw * S * chain_mma_clk(bn);
        const double epi = (double)S * bn * 4.0;
        const double t = (double)waves * ((mma > epi ? mma : epi) + 1200.0);
        if (bl < 0 || t < bl) { bl = t; bbn = bn; }
      }
      if (bbn == 0) okS = false;
      bn_for[si][l] = bbn;
      cost += bl + 3000.0;
    }
    if (okS && (bestCost < 0 || cost < bestCost)) { bestCost = cost; bestS = S; }
  }
  const int fS = chain_env("DFVO_CHAIN_S", 0);
  if (fS == 1 || fS == 2 || fS == 4) bestS = fS;
  const int si = bestS == 1 ? 0 : (bestS == 2 ? 1 : 2);
  static ChainArgs A;                     // 8.5 KB of kernel parameters; filled per launch (single host thread per context)
  memset(&A, 0, sizeof(A));
  A.nlayers = n;
  int a_stage = 0, b_stage = 0, cout_max = 0, grid = 1;
  double flops = 0.0;
  for (int l = 0; l < n; ++l) {
    const ConvTc& c = layers[l];
    ChainL& k = A.L[l];
    chain_rect(c, &k.kh, &k.kw, &k.dy0, &k.dx0);
    k.N = c.N; k.H = c.H; k.W = c.W; k.block_n = bn_for[si][l];
    DFVO_REQUIRE(k.block_n > 0, DFVO_EINVAL, "conv_chain: no block_n for layer %d", l);
    k.tiles_x = cdiv(c.W, 8 * bestS); k.tiles_y = cdiv(c.H, CHAIN_TH);
    k.n_blocks = c.Cout_pad / k.block_n;
    k.ntiles = k.tiles_x * k.tiles_y * c.N * k.n_blocks;
    k.HW = 8 * bestS + k.kw - 1; k.HH = CHAIN_TH + k.kh - 1;
    k.nsrc = c.nsrc;
    int ktot = 0;
    for (int i = 0; i < c.nsrc; ++i) { k.srcC[i] = c.src[i].C; ktot += c.src[i].C; }
    k.Cout = c.Cout; k.Cout_pad = c.Cout_pad; k.act = c.act; k.out_f32 = c.out_f32;
    k.zero_pad_to = c.zero_pad_to > c.Cout ? c.zero_pad_to : c.Cout;
    k.bias = c.bias; k.out = c.out; k.oN = c.oN; k.oH = c.oH; k.oW = c.oW;
    k.res = c.residual; k.rN = c.rN; k.rH = c.rH; k.rW = c.rW;
    const int as = (k.HW * k.HH * 128 + 1023) & ~1023;
    if (as > a_stage) a_stage = as;
    if (k.block_n * 128 > b_stage) b_stage = k.block_n * 128;
    if (c.Cout_pad > cout_max) cout_max = c.Cout_pad;
    if (k.ntiles > grid) grid = k.ntiles;
    flops += c.flops;
    for (int i = 0; i < 3; ++i) {
      const ConvTcSource& src = c.src[i < c.nsrc ? i : 0];
      const int inW = c.inW > 0 ? c.inW : c.W, inH = c.inH > 0 ? c.inH : c.H;
      unsigned long long dims[4] = {(unsigned long long)src.C, (unsigned long long)inW, (unsigned long long)inH, (unsigned long long)c.N};
      unsigned long long str[3] = {(unsigned long long)src.sW * 2, (unsigned long long)src.sH * 2, (unsigned long long)src.sN * 2};
      unsigned box[4] = {64, (unsigned)k.HW, (unsigned)k.HH, 1};
      int rc = tc_encode_map(&A.tmA[l][i], src.p, 4, dims, str, box, 2);
      if (rc) return rc;
    }
    {
      unsigned long long dims[3] = {(unsigned long long)ktot, (unsigned long long)c.Cout_pad, (unsigned long long)c.ntaps};
      unsigned long long str[2] = {(unsigned long long)ktot * 2, (unsigned long long)ktot * 2 * (unsigned long long)c.Cout_pad};
      unsigned box[3] = {64, (unsigned)k.block_n, 1};
      int rc = tc_encode_map(&A.tmB[l], c.w, 3, dims, str, box, 2);
      if (rc) return rc;
    }
  }
  if (grid > nsm) grid = nsm;
  // ring geometry common to the chain
  const size_t fixed = 1024 + 8 * 64 + (size_t)cout_max * 4;
  const size_t budget = 220 * 1024;
  int a_stages = 2, b_stages = 2;
  DFVO_REQUIRE(fixed + 2 * (size_t)a_stage + 2 * (size_t)b_stage <= budget, DFVO_EINVAL, "conv_chain: tiles do not fit in shared memory");
  while (b_stages < 8 && fixed + (size_t)a_stages * a_stage + (size_t)(b_stages + 1) * b_stage <= budget) ++b_stages;
  while (a_stages < 3 && fixed + (size_t)(a_stages + 1) * a_stage + (size_t)b_stages * b_stage <= budget) ++a_stages;
  while (b_stages < 12 && fixed + (size_t)a_stages * a_stage + (size_t)(b_stages + 1) * b_stage <= budget) ++b_stages;
  A.a_stages = a_stages; A.b_stages = b_stages; A.a_stage_bytes = a_stage; A.b_stage_bytes = b_stage;
  A.bias_cap = cout_max;
  const size_t smem = fixed + (size_t)a_stages * a_stage + (size_t)b_stages * b_stage;
  // arrival counters: CHAIN_BAR_WORDS words owned by the caller (one block per chain site of a network, so launches that may be in
  // flight together -- other engines, other graphs -- never share counters); word [CHAIN_MAXL] collects the watchdog flag
  A.bar = bar;
  A.err = bar + CHAIN_MAXL;
  DFVO_CUDA(cudaMemsetAsync(A.bar, 0, CHAIN_MAXL * sizeof(unsigned), s));
  static bool attr_set = false;
  if (!attr_set) {
    DFVO_CUDA(cudaFuncSetAttribute(k_conv_chain<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    DFVO_CUDA(cudaFuncSetAttribute(k_conv_chain<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    DFVO_CUDA(cudaFuncSetAttribute(k_conv_chain<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_set = true;
  }
  ++g_launch_count;
  TcProf pr;
  const bool prof = tc_prof_begin(s, &pr);
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cudaLaunchAttribute attr;
  cfg.gridDim = dim3(grid); cfg.blockDim = dim3(CHAIN_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = s;
  attr.id = cudaLaunchAttributeCooperative;
  attr.val.cooperative = 1;
  cfg.attrs = &attr; cfg.numAttrs = 1;
  if (bestS == 1) DFVO_CUDA(cudaLaunchKernelEx(&cfg, k_conv_chain<1>, A));
  else if (bestS == 2) DFVO_CUDA(cudaLaunchKernelEx(&cfg, k_conv_chain<2>, A));
  else DFVO_CUDA(cudaLaunchKernelEx(&cfg, k_conv_chain<4>, A));
  if (prof) {
    char d[256];
    const ConvTc& c0 = layers[0];
    snprintf(d, sizeof(d), "chain x%d N%d %dx%d S%d stages%d/%d grid%d first k%dx%d cin%d cout%d ... last cout%d gflop %.3f", n, c0.N, c0.H, c0.W, bestS,
             a_stages, b_stages, grid, A.L[0].kh, A.L[0].kw, c0.src[0].C, c0.Cout, layers[n - 1].Cout, flops * 1e-9);
    tc_prof_end(s, pr, flops, d);
  }
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

// ---- recorder: conv_tc() hands eligible layers to the open chain instead of launching them ---------------------------------
struct ChainRec { bool open = false; cudaStream_t s = nullptr; unsigned* bar = nullptr; std::vector<ConvTc> layers; };
static thread_local ChainRec g_rec;

static int g_chain_on = -1;
static int chain_enabled() {
  if (g_chain_on < 0) g_chain_on = chain_env("DFVO_CONV_CHAIN", 0);
  return g_chain_on;
}
int conv_chain_set_enabled(int on) { const int prev = chain_enabled(); g_chain_on = on ? 1 : 0; return prev; }

int conv_tc_single(const ConvTc& c, cudaStream_t s);

int conv_chain_flush() {
  ChainRec& r = g_rec;
  if (r.layers.empty()) return DFVO_OK;
  std::vector<ConvTc> ls;
  ls.swap(r.layers);
  if (ls.size() == 1) return conv_tc_single(ls[0], r.s);
  return conv_chain_launch(ls, r.bar, r.s);
}

void conv_chain_begin(cudaStream_t s, unsigned* bar) {
  if (!chain_enabled() || bar == nullptr) return;
  g_rec.open = true; g_rec.s = s; g_rec.bar = bar; g_rec.layers.clear();
}

int conv_chain_end() {
  if (!g_rec.open) return DFVO_OK;
  g_rec.open = false;
  return conv_chain_flush();
}

// called by conv_tc(): true if the layer was taken by the open chain
bool conv_chain_take(const ConvTc& c, cudaStream_t s, int* rc) {
  ChainRec& r = g_rec;
  *rc = DFVO_OK;
  if (!r.open) return false;
  if (s != r.s || !conv_chain_eligible(c)) { *rc = conv_chain_flush(); return false; }
  if ((int)r.layers.size() == CHAIN_MAXL) { *rc = conv_chain_flush(); if (*rc) return true; }
  if (!r.layers.empty() && (r.layers[0].N != c.N)) { *rc = conv_chain_flush(); if (*rc) return true; }
  r.layers.push_back(c);
  return true;
}

}  // namespace dfvo
#else
#include <vector>
namespace dfvo {
// CPU test build: no chains, every layer runs through the per-layer emulation
void conv_chain_begin(cudaStream_t, unsigned*) {}
int conv_chain_end() { return DFVO_OK; }
bool conv_chain_take(const ConvTc&, cudaStream_t, int* rc) { *rc = DFVO_OK; return false; }
int conv_chain_set_enabled(int) { return 0; }
}  // namespace dfvo
#endif
