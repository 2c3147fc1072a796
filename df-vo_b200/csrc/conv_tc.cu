// wgmma implicit-GEMM convolution for sm_90a (stride 1 or 2, arbitrary tap set, up to 3 virtually
// concatenated NHWC bf16 / fp32 sources, fused bias + activation + residual epilogue).
//
// GEMM view:  D[128 pixels, BLOCK_N couts] += sum over (tap, source, 64-channel chunk) of
//             A[128 pixels, 64 ch] * B[BLOCK_N couts, 64 ch]^T        (bf16 x bf16 -> fp32 in registers)
//   * A tile = one TMA 4-D box {64 ch, tw, th, 1} of the NHWC source at pixel offset (dx,dy) of the
//     tap: the box lands in shared memory as 128 rows x 128 B, K-major, 128-B swizzled -- exactly
//     the canonical wgmma operand layout, so there is no im2col pass; out-of-image rows/columns
//     (the convolution's zero padding) and channels beyond the source's C are zero-filled by TMA.
//   * B tile = TMA 3-D box {64 k, BLOCK_N, 1 tap} of the packed weights [tap][Cout_pad][Ktot].
//   * warp 0 = TMA producer (warps 1-3 idle); warpgroups 1 and 2 = consumers: each issues wgmma for
//     64 of the 128 pixel rows (accumulators in registers) and runs the bias/act/residual epilogue.
//   * persistent CTAs, static round-robin tile schedule, mbarrier full/empty smem ring.
// Restates torch.nn.Conv2d(stride=1) + LeakyReLU/ELU/ReLU as used at lite_flow_net.py:98-240 and
// depth_decoder.py / torchvision BasicBlock (BN folded by the weight packer).
#include "tc_ptx.cuh"

#ifndef DFVO_HOSTSIM
#include <cuda.h>
#endif
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <utility>
#include <vector>

namespace dfvo {

void conv_tc_tile_shape(int H, int W, int* tw, int* th) {
  // 128 pixels per tile as tw x th (powers of two); minimise padded area, prefer wide tiles.
  long long best = -1;
  int bw = 128, bh = 1;
  for (int w = 128; w >= 1; w >>= 1) {
    int h = 128 / w;
    long long area = (long long)cdiv(W, w) * w * (long long)cdiv(H, h) * h;
    if (best < 0 || area < best) { best = area; bw = w; bh = h; }
  }
  *tw = bw; *th = bh;
}

struct ConvTcK {
  int N, H, W, tw, th, tiles_x, tiles_y, n_blocks, ntiles;
  int nsrc, srcC[3];
  int ntaps;
  int8_t dy[49], dx[49];        // stride 1: input offsets; stride 2: offsets in units of double-pixels (floor((k-pad)/2))
  int8_t py[49], px[49];        // stride 2: pixel phase of the tap inside the 2x2 cell
  int stride, src_pitch;        // src_pitch (elements) = channel offset of the odd pixel inside a double-pixel
  int block_n, stages;
  int Cout, Cout_pad, act, out_f32, zero_pad_to;
  int chunk, esize, round_tf32;   // channels per 128-byte operand row (64 bf16 / 32 tf32), operand element size
  const float* bias;
  void* out; long long oN, oH, oW;
  const void* res; long long rN, rH, rW;
};

#ifndef DFVO_HOSTSIM
// =============================================================================================
//                                       device side
// =============================================================================================
#define TC_THREADS 384
#define TC_A_BYTES 16384

template <int BN, int TF32>
__global__ void __launch_bounds__(TC_THREADS, 1)
k_conv_tc(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
          const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB,
          const __grid_constant__ ConvTcK p) {
  using namespace tc;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;                 // SWIZZLE_128B needs 1024-B alignment
  uint8_t* base_ptr = smem_raw + (base - raw);
  const uint32_t stage_bytes = TC_A_BYTES + (uint32_t)BN * 128u;
  const uint32_t bar_base = base + (uint32_t)p.stages * stage_bytes;    // 8-byte aligned
  // barrier layout: full[stages], empty[stages]
  auto full_bar = [&](int s) { return bar_base + 8u * (uint32_t)s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (uint32_t)(p.stages + s); };
  float* bias_s = reinterpret_cast<float*>(base_ptr + (size_t)p.stages * stage_bytes + 8u * (2 * p.stages) + 64);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  pdl_trigger();

  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tmA0); prefetch_tmap(&tmB);
    for (int s = 0; s < p.stages; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();                                  // from here on: activations of the previous kernel / our output buffers

  if (warp == 0) {
    // ===================================== TMA producer =====================================
    // whole warp walks the loop, one elected lane issues (see tc_ptx.cuh::elect_one)
    int stage = 0; uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
      int t = tile;
      const int tx = t % p.tiles_x; t /= p.tiles_x;
      const int ty = t % p.tiles_y; t /= p.tiles_y;
      const int n = t % p.N; const int nb = t / p.N;
      const int x0 = tx * p.tw, y0 = ty * p.th;
      for (int tap = 0; tap < p.ntaps; ++tap) {
        int kofs = 0;
        for (int s = 0; s < p.nsrc; ++s) {
          const CUtensorMap* tm = s == 0 ? &tmA0 : (s == 1 ? &tmA1 : &tmA2);
          for (int c0 = 0; c0 < p.srcC[s]; c0 += p.chunk) {
            mbar_wait(empty_bar(stage), phase ^ 1u);
            if (elect_one()) {
              const uint32_t sa = base + (uint32_t)stage * stage_bytes;
              mbar_expect_tx(full_bar(stage), stage_bytes);
              if (p.stride == 2)
                tma_load_5d(sa, tm, full_bar(stage), c0 + p.px[tap] * p.src_pitch, x0 + p.dx[tap], p.py[tap], y0 + p.dy[tap], n);
              else
                tma_load_4d(sa, tm, full_bar(stage), c0, x0 + p.dx[tap], y0 + p.dy[tap], n);
              tma_load_3d(sa + TC_A_BYTES, &tmB, full_bar(stage), kofs + c0, nb * BN, tap);
            }
            __syncwarp();
            if (++stage == p.stages) { stage = 0; phase ^= 1u; }
          }
          kofs += p.srcC[s];
        }
      }
    }
  } else if (warp >= 4) {
    // ============================ two consumer warpgroups: MMA + epilogue ============================
    // warpgroup wg owns rows [64 wg, 64 wg + 64) of the 128-pixel tile: its A operand starts 64 rows = 8 KB into the A box.
    const int ct = threadIdx.x - 128, wg = ct >> 7, wq = (ct >> 5) & 3;
    const bool leader = (ct & 127) == 0;
    for (int i = ct; i < p.Cout_pad; i += 256) bias_s[i] = p.bias ? p.bias[i] : 0.f;
    asm volatile("bar.sync 1, 256;" ::: "memory");
    TcEpi ep; ep.Cout = p.Cout; ep.zero_pad_to = p.zero_pad_to; ep.act = p.act; ep.out_f32 = p.out_f32; ep.round_tf32 = p.round_tf32; ep.out = p.out; ep.res = p.res;
    int stage = 0; uint32_t phase = 0;
    float acc[BN / 2];
    for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
      uint32_t fresh = 0;
      int pend = -1;
      for (int tap = 0; tap < p.ntaps; ++tap) {
        for (int s = 0; s < p.nsrc; ++s) {
          for (int c0 = 0; c0 < p.srcC[s]; c0 += p.chunk) {
            mbar_wait(full_bar(stage), phase);
            wgmma_fence();
            const uint32_t sa = base + (uint32_t)stage * stage_bytes;
            const int rem = p.srcC[s] - c0;
            const int nks = ((rem >= p.chunk ? p.chunk : rem) * p.esize) >> 5;       // 32-byte K steps with real channels
            float (&acc1)[1][BN / 2] = reinterpret_cast<float (&)[1][BN / 2]>(acc);
            const uint32_t at = sa + (uint32_t)wg * 8192u, bt = sa + TC_A_BYTES;   // the same K-step walk as one halo tap, S = 1
            switch (nks) {
              case 4: halo_tap_mma<1, BN, TF32, 4>(acc1, at, bt, 1024u, fresh); break;
              case 3: halo_tap_mma<1, BN, TF32, 3>(acc1, at, bt, 1024u, fresh); break;
              case 2: halo_tap_mma<1, BN, TF32, 2>(acc1, at, bt, 1024u, fresh); break;
              default: halo_tap_mma<1, BN, TF32, 1>(acc1, at, bt, 1024u, fresh); break;
            }
            wgmma_commit();
            wgmma_wait<1>();                                                          // the previous stage's MMAs are done
            if (pend >= 0 && leader) mbar_arrive(empty_bar(pend));
            pend = stage;
            fresh = 1u;
            if (++stage == p.stages) { stage = 0; phase ^= 1u; }
          }
        }
      }
      wgmma_wait<0>();
      if (leader) mbar_arrive(empty_bar(pend));

      int t = tile;
      const int tx = t % p.tiles_x; t /= p.tiles_x;
      const int ty = t % p.tiles_y; t /= p.tiles_y;
      const int n = t % p.N; const int nb = t / p.N;
      // accumulator pair (4 j + 2 h, +1) = tile row 64 wg + 16 wq + lane / 4 + 8 h, channels nb * BN + 8 j + 2 (lane % 4) + {0, 1}
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = 64 * wg + 16 * wq + (lane >> 2) + 8 * h;
        const int x = tx * p.tw + (row % p.tw), y = ty * p.th + (row / p.tw);
        if (x >= p.W || y >= p.H) continue;
        const long long opix = n * p.oN + y * p.oH + x * p.oW, rpix = n * p.rN + y * p.rH + x * p.rW;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j)
          tc_store2(ep, bias_s, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], nb * BN + 8 * j + 2 * (lane & 3), opix, rpix);
      }
    }
  }
}

// =============================================================================================
//                                        host side
// =============================================================================================
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = (PFN_encodeTiled)p;
  }
  return fn;
}

int tc_encode_map(void* map, const void* ptr, int rank, const unsigned long long* dims_, const unsigned long long* strides_, const unsigned* box_,
                  int esize, int swizzle_bytes) {
  cuuint64_t dims[5], str[5];
  cuuint32_t box[5];
  for (int i = 0; i < rank; ++i) { dims[i] = dims_[i]; box[i] = box_[i]; if (i < rank - 1) str[i] = strides_[i]; }
  CUtensorMap* m = reinterpret_cast<CUtensorMap*>(map);
  const cuuint64_t* strides_bytes = str;
  PFN_encodeTiled enc = get_encode();
  DFVO_REQUIRE(enc != nullptr, DFVO_ECUDA, "cuTensorMapEncodeTiled entry point unavailable");
  cuuint32_t es[5] = {1, 1, 1, 1, 1};
  CUresult r = enc(m, esize == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(ptr), dims, strides_bytes, box, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B : (swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B),
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  DFVO_REQUIRE(r == CUDA_SUCCESS, DFVO_ECUDA, "cuTensorMapEncodeTiled failed: %d (rank %d dims %llu %llu %llu box %u %u %u)", (int)r,
               rank, (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)dims[2], box[0], box[1], box[2]);
  return DFVO_OK;
}

struct ConvTcPlanImpl {
  CUtensorMap tmA[3], tmB;
  ConvTcK k;
  int grid;
  size_t smem;
};

static int g_num_sms = 0;
void tc_launch_config(cudaLaunchConfig_t* cfg, cudaLaunchAttribute* attr, int grid, int block, size_t smem, cudaStream_t s) {
  static int pdl = -1;
  if (pdl < 0) { const char* e = getenv("DFVO_PDL"); pdl = !(e && atoi(e) == 0); }
  memset(cfg, 0, sizeof(*cfg));
  cfg->gridDim = dim3(grid); cfg->blockDim = dim3(block); cfg->dynamicSmemBytes = smem; cfg->stream = s;
  attr->id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr->val.programmaticStreamSerializationAllowed = 1;
  cfg->attrs = attr; cfg->numAttrs = pdl ? 1 : 0;
}
int tc_num_sms() {
  if (!g_num_sms) {
    int dev = 0; cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
    if (g_num_sms <= 0) g_num_sms = 132;
  }
  return g_num_sms;
}
static int encode_map(CUtensorMap* m, const void* ptr, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes, const cuuint32_t* box,
                      int esize) {
  unsigned long long d[5], st[5]; unsigned b[5];
  for (int i = 0; i < rank; ++i) { d[i] = dims[i]; b[i] = box[i]; if (i < rank - 1) st[i] = strides_bytes[i]; }
  return tc_encode_map(m, ptr, rank, d, st, b, esize, 128);
}

static int build_plan(const ConvTc& c, ConvTcPlanImpl* pl) {
  DFVO_REQUIRE(c.nsrc >= 1 && c.nsrc <= 3 && c.ntaps >= 1 && c.ntaps <= 49, DFVO_EINVAL, "conv_tc: nsrc/ntaps");
  DFVO_REQUIRE(c.Cout_pad % 16 == 0 && c.Cout_pad >= 16, DFVO_EINVAL, "conv_tc: Cout_pad %d must be a multiple of 16", c.Cout_pad);
  ConvTcK& k = pl->k;
  memset(&k, 0, sizeof(k));
  k.N = c.N; k.H = c.H; k.W = c.W;
  conv_tc_tile_shape(c.H, c.W, &k.tw, &k.th);
  k.tiles_x = cdiv(c.W, k.tw); k.tiles_y = cdiv(c.H, k.th);
  // N tile: the widest wgmma shape (256, 128, 64, 32, 16) that divides Cout_pad
  k.block_n = 256;
  while (c.Cout_pad % k.block_n) k.block_n >>= 1;
  k.n_blocks = c.Cout_pad / k.block_n;
  k.ntiles = k.tiles_x * k.tiles_y * c.N * k.n_blocks;
  k.nsrc = c.nsrc; k.ntaps = c.ntaps;
  const int es = c.esize == 4 ? 4 : 2;
  k.esize = es; k.chunk = 128 / es; k.round_tf32 = c.round_out_tf32;
  int ktot = 0;
  for (int s = 0; s < c.nsrc; ++s) {
    DFVO_REQUIRE(c.src[s].C % 16 == 0 && c.src[s].C > 0, DFVO_EINVAL, "conv_tc: source %d channels %d not a multiple of 16", s, c.src[s].C);
    DFVO_REQUIRE(((uintptr_t)c.src[s].p & 15) == 0 && (c.src[s].sW * es) % 16 == 0 && (c.src[s].sH * es) % 16 == 0 && (c.src[s].sN * es) % 16 == 0,
                 DFVO_EINVAL, "conv_tc: source %d not 16-byte aligned/strided", s);
    k.srcC[s] = c.src[s].C; ktot += c.src[s].C;
  }
  k.stride = c.stride == 2 ? 2 : 1;
  if (k.stride == 2) {
    const int inH = c.inH > 0 ? c.inH : 2 * c.H, inW = c.inW > 0 ? c.inW : 2 * c.W;
    DFVO_REQUIRE(c.nsrc == 1 && inH % 2 == 0 && inW % 2 == 0 && inH == 2 * c.H && inW == 2 * c.W, DFVO_EINVAL,
                 "conv_tc stride 2: needs one source and even input size = 2x output");
    DFVO_REQUIRE(c.src[0].sH == (long long)inW * c.src[0].sW, DFVO_EINVAL, "conv_tc stride 2: rows must be contiguous");
    k.src_pitch = (int)c.src[0].sW;
    for (int t = 0; t < c.ntaps; ++t) {
      const int oy = c.dy[t], ox = c.dx[t];                 // input-pixel offsets
      k.py[t] = (int8_t)(((oy % 2) + 2) % 2); k.dy[t] = (int8_t)((oy - k.py[t]) / 2);
      k.px[t] = (int8_t)(((ox % 2) + 2) % 2); k.dx[t] = (int8_t)((ox - k.px[t]) / 2);
    }
  } else {
    memcpy(k.dy, c.dy, sizeof(k.dy)); memcpy(k.dx, c.dx, sizeof(k.dx));
  }
  k.Cout = c.Cout; k.Cout_pad = c.Cout_pad; k.act = c.act; k.out_f32 = c.out_f32;
  k.zero_pad_to = c.zero_pad_to > c.Cout ? c.zero_pad_to : c.Cout;
  k.bias = c.bias; k.out = c.out; k.oN = c.oN; k.oH = c.oH; k.oW = c.oW;
  k.res = c.residual; k.rN = c.rN; k.rH = c.rH; k.rW = c.rW;
  const size_t stage_bytes = TC_A_BYTES + (size_t)k.block_n * 128;
  const size_t fixed = 1024 /*align slack*/ + 8 * 64 /*barriers*/ + 64 + (size_t)c.Cout_pad * 4 /*bias*/;
  int stages = (int)((200 * 1024 - fixed) / stage_bytes);
  if (stages > 8) stages = 8;
  DFVO_REQUIRE(stages >= 2, DFVO_EINVAL, "conv_tc: tile does not fit in shared memory");
  k.stages = stages;
  pl->smem = fixed + (size_t)stages * stage_bytes;
  pl->grid = k.ntiles < tc_num_sms() ? k.ntiles : tc_num_sms();
  // tensor maps
  for (int s = 0; s < 3; ++s) {
    const ConvTcSource& src = c.src[s < c.nsrc ? s : 0];
    if (k.stride == 2) {
      // view [N][H/2][2][W/2][pitch+C]: a double-pixel holds the even pixel's channels at [0,C) and the odd pixel's
      // at [pitch, pitch+C); (py, px) of a tap select the phase, the box walks W/2 x H/2 cells of the output tile
      const int inW2 = c.W, inH2 = c.H;
      cuuint64_t dims[5] = {(cuuint64_t)(src.sW + src.C), (cuuint64_t)inW2, 2, (cuuint64_t)inH2, (cuuint64_t)c.N};
      cuuint64_t str[4] = {(cuuint64_t)src.sW * 2 * es, (cuuint64_t)src.sH * es, (cuuint64_t)src.sH * 2 * es, (cuuint64_t)src.sN * es};
      cuuint32_t box[5] = {(cuuint32_t)k.chunk, (cuuint32_t)k.tw, 1, (cuuint32_t)k.th, 1};
      int rc = encode_map(&pl->tmA[s], src.p, 5, dims, str, box, es);
      if (rc) return rc;
      continue;
    }
    const int inW = c.inW > 0 ? c.inW : c.W, inH = c.inH > 0 ? c.inH : c.H;
    cuuint64_t dims[4] = {(cuuint64_t)src.C, (cuuint64_t)inW, (cuuint64_t)inH, (cuuint64_t)c.N};
    cuuint64_t str[3] = {(cuuint64_t)src.sW * es, (cuuint64_t)src.sH * es, (cuuint64_t)src.sN * es};
    cuuint32_t box[4] = {(cuuint32_t)k.chunk, (cuuint32_t)k.tw, (cuuint32_t)k.th, 1};
    int rc = encode_map(&pl->tmA[s], src.p, 4, dims, str, box, es);
    if (rc) return rc;
  }
  {
    cuuint64_t dims[3] = {(cuuint64_t)ktot, (cuuint64_t)c.Cout_pad, (cuuint64_t)c.ntaps};
    cuuint64_t str[2] = {(cuuint64_t)ktot * es, (cuuint64_t)ktot * es * (cuuint64_t)c.Cout_pad};
    cuuint32_t box[3] = {(cuuint32_t)k.chunk, (cuuint32_t)k.block_n, 1};
    int rc = encode_map(&pl->tmB, c.w, 3, dims, str, box, es);
    if (rc) return rc;
  }
  return DFVO_OK;
}

std::atomic<long long> g_launch_count{0};
int g_tc_prof_on = 0;
static double g_prof_flops = 0.0;
static std::vector<std::pair<cudaEvent_t, cudaEvent_t>> g_prof_events;
static std::vector<std::string> g_prof_desc;      // per-launch layer description (DFVO_TC_TRACE=1 prints them with their times)

void conv_tc_profile_enable(int on) {
  g_tc_prof_on = on;
  if (on) {
    for (auto& e : g_prof_events) { cudaEventDestroy(e.first); cudaEventDestroy(e.second); }
    g_prof_events.clear();
    g_prof_desc.clear();
    g_prof_flops = 0.0;
  }
}

void conv_tc_profile_read(double* ms, long long* launches, double* flops) {
  double tot = 0.0;
  const bool trace = getenv("DFVO_TC_TRACE") != nullptr;
  for (size_t i = 0; i < g_prof_events.size(); ++i) {
    auto& e = g_prof_events[i];
    cudaEventSynchronize(e.second);
    float t = 0.f;
    if (cudaEventElapsedTime(&t, e.first, e.second) == cudaSuccess) tot += t;
    if (trace && i < g_prof_desc.size()) fprintf(stderr, "conv_tc %4zu %8.2f us  %s\n", i, t * 1e3, g_prof_desc[i].c_str());
  }
  *ms = tot; *launches = (long long)g_prof_events.size(); *flops = g_prof_flops;
}

bool tc_prof_begin(cudaStream_t s, TcProf* p) {
  if (!g_tc_prof_on) return false;
  cudaEventCreate(&p->e0); cudaEventCreate(&p->e1); cudaEventRecord(p->e0, s);
  return true;
}
void tc_prof_end(cudaStream_t s, const TcProf& p, double flops, const char* desc) {
  cudaEventRecord(p.e1, s);
  g_prof_events.push_back({p.e0, p.e1});
  g_prof_flops += flops;
  g_prof_desc.push_back(desc);
}

int conv_tc_single(const ConvTc& c, cudaStream_t s);
int conv_tc(const ConvTc& c, cudaStream_t s) {
  int rc = DFVO_OK;
  if (conv_chain_take(c, s, &rc)) return rc;              // deferred into the open layer chain (conv_chain.cu)
  if (rc) return rc;
  return conv_tc_single(c, s);
}

template <int BN, int TF32>
static int launch_tc(const ConvTcPlanImpl& pl, cudaStream_t s) {
  static bool attr_set = false;
  if (!attr_set) {
    DFVO_CUDA(cudaFuncSetAttribute(k_conv_tc<BN, TF32>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_set = true;
  }
  cudaLaunchConfig_t cfg; cudaLaunchAttribute attr;
  tc_launch_config(&cfg, &attr, pl.grid, TC_THREADS, pl.smem, s);
  DFVO_CUDA(cudaLaunchKernelEx(&cfg, k_conv_tc<BN, TF32>, pl.tmA[0], pl.tmA[1], pl.tmA[2], pl.tmB, pl.k));
  return DFVO_OK;
}

int conv_tc_single(const ConvTc& c, cudaStream_t s) {
  if (conv_halo_supported(c)) return conv_halo(c, s);
  ConvTcPlanImpl pl;
  int rc = build_plan(c, &pl);
  if (rc) return rc;
  ++g_launch_count;
  TcProf pr;
  const bool prof = tc_prof_begin(s, &pr);
  const int tf32 = pl.k.esize == 4;
  switch (pl.k.block_n) {
    case 256: rc = tf32 ? launch_tc<256, 1>(pl, s) : launch_tc<256, 0>(pl, s); break;
    case 128: rc = tf32 ? launch_tc<128, 1>(pl, s) : launch_tc<128, 0>(pl, s); break;
    case 64: rc = tf32 ? launch_tc<64, 1>(pl, s) : launch_tc<64, 0>(pl, s); break;
    case 32: rc = tf32 ? launch_tc<32, 1>(pl, s) : launch_tc<32, 0>(pl, s); break;
    default: rc = tf32 ? launch_tc<16, 1>(pl, s) : launch_tc<16, 0>(pl, s); break;
  }
  if (rc) return rc;
  if (prof) {
    char d[256];
    snprintf(d, sizeof(d), "tap  N%d %dx%d s%d taps%d src[%d,%d,%d] cout%d/%d bn%d tile%dx%d stages%d grid%d tiles%d gflop %.3f", c.N, c.H, c.W,
             pl.k.stride, c.ntaps, c.src[0].C, c.nsrc > 1 ? c.src[1].C : 0, c.nsrc > 2 ? c.src[2].C : 0, c.Cout, c.Cout_pad, pl.k.block_n,
             pl.k.tw, pl.k.th, pl.k.stages, pl.grid, pl.k.ntiles, c.flops * 1e-9);
    tc_prof_end(s, pr, c.flops, d);
  }
  DFVO_CHECK_LAUNCH();
  return DFVO_OK;
}

#else  // DFVO_HOSTSIM ---------------------------------------------------------------------------
// CPU test build only: consumes the SAME ConvTc description and packed weights as the device
// kernel and applies the same TMA semantics (zero fill outside the image / beyond a source's C,
// virtual concat of sources, tap offsets), so the layer wiring and the weight packer can be
// validated without a GPU.  Never compiled into the product library.
std::atomic<long long> g_launch_count{0};
void conv_tc_profile_enable(int) {}
void conv_tc_profile_read(double* ms, long long* launches, double* flops) { *ms = 0; *launches = 0; *flops = 0; }
int conv_tc(const ConvTc& c, cudaStream_t) {
  int ktot = 0;
  for (int s = 0; s < c.nsrc; ++s) ktot += c.src[s].C;
  int zp = c.zero_pad_to > c.Cout ? c.zero_pad_to : c.Cout;
  std::vector<float> acc(c.Cout_pad);
  for (int n = 0; n < c.N; ++n)
    for (int y = 0; y < c.H; ++y)
      for (int x = 0; x < c.W; ++x) {
        for (int co = 0; co < c.Cout_pad; ++co) acc[co] = 0.f;
        for (int t = 0; t < c.ntaps; ++t) {
          const int st = c.stride == 2 ? 2 : 1;
          int iy = y * st + c.dy[t], ix = x * st + c.dx[t];
          const int inW = c.inW > 0 ? c.inW : c.W * st, inH = c.inH > 0 ? c.inH : c.H * st;
          if (iy < 0 || iy >= inH || ix < 0 || ix >= inW) continue;
          int kofs = 0;
          for (int s = 0; s < c.nsrc; ++s) {
            const size_t eoff = n * c.src[s].sN + iy * c.src[s].sH + ix * c.src[s].sW;
            for (int ci = 0; ci < c.src[s].C; ++ci) {
              const float av = c.esize == 4 ? ((const float*)c.src[s].p)[eoff + ci] : __bfloat162float(((const bf16*)c.src[s].p)[eoff + ci]);
              if (av == 0.f) continue;
              const size_t woff = ((size_t)t * c.Cout_pad) * ktot + kofs + ci;
              for (int co = 0; co < c.Cout_pad; ++co)
                acc[co] += av * (c.esize == 4 ? ((const float*)c.w)[woff + (size_t)co * ktot] : __bfloat162float(((const bf16*)c.w)[woff + (size_t)co * ktot]));
            }
            kofs += c.src[s].C;
          }
        }
        for (int co = 0; co < zp; ++co) {
          float v = 0.f;
          if (co < c.Cout) {
            v = acc[co] + (c.bias ? c.bias[co] : 0.f);
            if (c.residual) {
              if (c.out_f32) v += ((const float*)c.residual)[n * c.rN + y * c.rH + x * c.rW + co];
              else v += __bfloat162float(((const bf16*)c.residual)[n * c.rN + y * c.rH + x * c.rW + co]);
            }
            v = apply_act(v, c.act);
          }
          if (c.out_f32) ((float*)c.out)[n * c.oN + y * c.oH + x * c.oW + co] = v;
          else ((bf16*)c.out)[n * c.oN + y * c.oH + x * c.oW + co] = __float2bfloat16_rn(v);
        }
      }
  return DFVO_OK;
}
#endif

}  // namespace dfvo
