// C-ABI glue (include/dfvo_b200.h).  No torch types, no exceptions across the boundary.
#include "../../include/dfvo_b200.h"

#include <stdlib.h>
#include <string.h>

#include <map>
#include <new>
#include <vector>

#include "liteflownet.h"
#include "monodepth2.h"
#include "net_common.h"
#include "ransac.h"

namespace dfvo { const char* last_error(); }

using namespace dfvo;

// ---- CUDA-graph replay of a network forward ------------------------------------------------------------------
// A forward pass is a fixed sequence of ~100-200 small launches whose arguments depend only on the caller's buffer
// pointers.  The first call with a given pointer set runs eagerly (lazy module loading, function attributes), the
// second is stream-captured and instantiated, later ones are one cudaGraphLaunch: the host enqueue cost drops from
// ~0.5 ms to tens of microseconds and the launch gaps between dependent kernels shrink.  Only on a capturable stream
// (not the legacy default stream) and never while the per-launch profiler is on.  DFVO_GRAPHS=0 disables.
#ifndef DFVO_HOSTSIM
namespace dfvo { extern int g_tc_prof_on; }
struct GraphEntry { int seen = 0; cudaGraphExec_t exec = nullptr; long long launches = 0; };
struct GraphCache {
  std::map<std::vector<uintptr_t>, GraphEntry> m;
  ~GraphCache() { for (auto& kv : m) if (kv.second.exec) cudaGraphExecDestroy(kv.second.exec); }
  void clear() { for (auto& kv : m) if (kv.second.exec) cudaGraphExecDestroy(kv.second.exec); m.clear(); }
};

template <typename F>
static int run_graphed(GraphCache& gc, const std::vector<uintptr_t>& key, cudaStream_t s, F body) {
  static int enabled = -1;
  if (enabled < 0) { const char* e = getenv("DFVO_GRAPHS"); enabled = !(e && atoi(e) == 0); }
  if (!enabled || dfvo::g_tc_prof_on || s == nullptr || s == cudaStreamLegacy) return body();
  auto it = gc.m.find(key);
  if (it == gc.m.end()) {
    if (gc.m.size() >= 64) return body();                 // bounded cache: unusual callers stay eager
    it = gc.m.emplace(key, GraphEntry()).first;
  }
  GraphEntry& e = it->second;
  if (e.exec) {
    DFVO_CUDA(cudaGraphLaunch(e.exec, s));
    dfvo::g_launch_count += e.launches;
    return DFVO_OK;
  }
  if (e.seen < 0 || e.seen++ == 0) return body();
  const long long l0 = dfvo::g_launch_count.load();
  if (cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal) != cudaSuccess) { cudaGetLastError(); e.seen = -1; return body(); }
  const int rc = body();
  cudaGraph_t g = nullptr;
  const cudaError_t ce = cudaStreamEndCapture(s, &g);
  if (rc != DFVO_OK || ce != cudaSuccess || !g) {
    if (g) cudaGraphDestroy(g);
    cudaGetLastError();
    e.seen = -1;                                           // not capturable: stay eager for this pointer set
    dfvo::g_launch_count = l0;
    return body();
  }
  e.launches = dfvo::g_launch_count.load() - l0;
  const cudaError_t ie = cudaGraphInstantiate(&e.exec, g, 0);
  cudaGraphDestroy(g);
  if (ie != cudaSuccess) { cudaGetLastError(); e.exec = nullptr; e.seen = -1; dfvo::g_launch_count = l0; return body(); }
  DFVO_CUDA(cudaGraphLaunch(e.exec, s));
  return DFVO_OK;
}

#else   // CPU test build: no graphs, every forward runs eagerly
struct GraphCache { void clear() {} };
template <typename F>
static int run_graphed(GraphCache&, const std::vector<uintptr_t>&, cudaStream_t, F body) { return body(); }
#endif

struct dfvo_ctx {
  int device = 0;
  WeightStore weights[3];
  LiteFlowNetBase* lfn = nullptr;
  Monodepth2Base* mono = nullptr;
  PoseNetBase* pose = nullptr;
  GraphCache flow_graphs, depth_graphs, pose_graphs;
};

#define API_BEGIN try {
#define API_END                                                     \
  } catch (const std::bad_alloc&) {                                 \
    dfvo::set_error("host allocation failed");                      \
    return DFVO_ENOMEM;                                             \
  } catch (...) {                                                   \
    dfvo::set_error("unexpected C++ exception");                    \
    return DFVO_EINVAL;                                             \
  }

template <typename T>
static int stage_correlation(const float* first, const float* second, float* out, int B, int C, int H, int W, int stride,
                             int leaky, cudaStream_t s) {
  Arena a;
  const int Cp = (C + 15) / 16 * 16;
  const int Ho = (H + stride - 1) / stride, Wo = (W + stride - 1) / stride;
  float* f32a = a.alloc_t<float>((size_t)B * H * W * Cp);
  float* f32b = a.alloc_t<float>((size_t)B * H * W * Cp);
  T* ta = a.alloc_t<T>((size_t)B * H * W * Cp);
  T* tb = a.alloc_t<T>((size_t)B * H * W * Cp);
  T* to = a.alloc_t<T>((size_t)B * Ho * Wo * 64);
  if (!f32a || !f32b || !ta || !tb || !to) return DFVO_ENOMEM;
  Ten<float> A = make_ten<float>(f32a, B, H, W, Cp, Cp), Bn = make_ten<float>(f32b, B, H, W, Cp, Cp);
  int rc;
  if ((rc = nchw_to_nhwc_f32(first, B, C, H, W, A, s))) return rc;
  if ((rc = nchw_to_nhwc_f32(second, B, C, H, W, Bn, s))) return rc;
  Ten<T> TA = make_ten<T>(ta, B, H, W, C, Cp), TB = make_ten<T>(tb, B, H, W, C, Cp);
  Ten<float> Ac = A, Bc = Bn; Ac.C = C; Bc.C = C;
  if ((rc = convert_copy<float, T>(cten(Ac), TA, s))) return rc;
  if ((rc = convert_copy<float, T>(cten(Bc), TB, s))) return rc;
  Ten<T> TO = make_ten<T>(to, B, Ho, Wo, 64, 64);
  {
    Ten<const float> noflow; memset(&noflow, 0, sizeof(noflow));
    Ten<T> noscratch; memset(&noscratch, 0, sizeof(noscratch));
    if ((rc = correlation49_warped<T>(cten(TA), cten(TB), 0, noflow, 0.f, stride, leaky, noscratch, TO, s))) return rc;
  }
  Ten<T> TO49 = TO; TO49.C = 49;
  if ((rc = nhwc_to_nchw<T>(cten(TO49), out, s))) return rc;
  DFVO_CUDA(cudaStreamSynchronize(s));
  return DFVO_OK;
}

template <typename T>
static int stage_warp(const float* input, const float* flow, float* out, int B, int C, int H, int W, cudaStream_t s) {
  Arena a;
  float* f32 = a.alloc_t<float>((size_t)B * H * W * C);
  float* fl = a.alloc_t<float>((size_t)B * H * W * 2);
  T* ti = a.alloc_t<T>((size_t)B * H * W * C);
  T* to = a.alloc_t<T>((size_t)B * H * W * C);
  if (!f32 || !fl || !ti || !to) return DFVO_ENOMEM;
  int rc;
  Ten<float> I = make_ten<float>(f32, B, H, W, C, C), Fl = make_ten<float>(fl, B, H, W, 2, 2);
  if ((rc = nchw_to_nhwc_f32(input, B, C, H, W, I, s))) return rc;
  if ((rc = nchw_to_nhwc_f32(flow, B, 2, H, W, Fl, s))) return rc;
  Ten<T> TI = make_ten<T>(ti, B, H, W, C, C), TO = make_ten<T>(to, B, H, W, C, C);
  if ((rc = convert_copy<float, T>(cten(I), TI, s))) return rc;
  if ((rc = warp_bilinear<T>(cten(TI), cten(Fl), 1.0f, 0, TO, s))) return rc;
  if ((rc = nhwc_to_nchw<T>(cten(TO), out, s))) return rc;
  DFVO_CUDA(cudaStreamSynchronize(s));
  return DFVO_OK;
}

template <typename T>
static int stage_conv(const float* x, const HostTensor& w, const HostTensor* b, float* y, int B, int Cin, int H, int W, int Cout,
                      int kh, int kw, int stride, int pad_y, int pad_x, int reflect, int act, cudaStream_t s, bool tf32 = false) {
  Arena a;
  const bool is_bf16 = sizeof(T) == 2 || tf32;          // "tensor-core layer": bf16 operands, or fp32 operands read as tf32
  const int Cp = (Cin + 15) / 16 * 16, Cop = (Cout + 15) / 16 * 16;
  const int Ho = (H + 2 * pad_y - kh) / stride + 1, Wo = (W + 2 * pad_x - kw) / stride + 1;
  ConvLayer L;
  int rc;
  if ((rc = build_conv_layer(a, w, b, {{Cin, Cp}}, stride, pad_y, pad_x, reflect, is_bf16, !is_bf16, nullptr, nullptr, &L, sizeof(T) == 2 ? 2 : 4))) return rc;
  float* f32 = a.alloc_t<float>((size_t)B * H * W * Cp);
  T* ti = a.alloc_t<T>((size_t)B * H * W * Cp);
  T* to = a.alloc_t<T>((size_t)B * Ho * Wo * Cop);
  if (!f32 || !ti || !to) return DFVO_ENOMEM;
  Ten<float> I = make_ten<float>(f32, B, H, W, Cp, Cp);
  if ((rc = nchw_to_nhwc_f32(x, B, Cin, H, W, I, s))) return rc;
  Ten<T> TI = make_ten<T>(ti, B, H, W, Cp, Cp);
  if ((rc = convert_copy<float, T>(cten(I), TI, s))) return rc;
  Ten<T> TO = make_ten<T>(to, B, Ho, Wo, Cout, Cop);
  Ten<const T> none; memset(&none, 0, sizeof(none));
  if ((rc = run_conv<T>(L, cten(TI), TO, act, none, 0, s))) return rc;
  if ((rc = nhwc_to_nchw<T>(cten(TO), y, s))) return rc;
  DFVO_CUDA(cudaStreamSynchronize(s));
  return DFVO_OK;
}

extern "C" {

const char* dfvo_last_error(void) { return dfvo::last_error(); }
const char* dfvo_version(void) { return "dfvo_b200 0.1 (sm_90a)"; }
int dfvo_is_device_build(void) {
#ifdef DFVO_HOSTSIM
  return 0;
#else
  return 1;
#endif
}

long long dfvo_launch_count(void) { return dfvo::g_launch_count.load(); }
int dfvo_set_conv_chain(int on) { return dfvo::conv_chain_set_enabled(on); }
void dfvo_profile_enable(int on) { dfvo::conv_tc_profile_enable(on); }
void dfvo_profile_read(double* tc_ms, long long* tc_launches, double* tc_flops) { dfvo::conv_tc_profile_read(tc_ms, tc_launches, tc_flops); }

int dfvo_create(dfvo_ctx** out, int device) {
  API_BEGIN
  DFVO_REQUIRE(out != nullptr, DFVO_EINVAL, "dfvo_create: null out");
  DFVO_CUDA(cudaSetDevice(device));
  *out = new dfvo_ctx();
  (*out)->device = device;
  return DFVO_OK;
  API_END
}

int dfvo_destroy(dfvo_ctx* ctx) {
  API_BEGIN
  if (!ctx) return DFVO_OK;
  delete ctx->lfn;
  delete ctx->mono;
  delete ctx->pose;
  delete ctx;
  return DFVO_OK;
  API_END
}

int dfvo_load_weight(dfvo_ctx* ctx, int net, const char* key, const float* data, const int64_t* shape, int ndim) {
  API_BEGIN
  DFVO_REQUIRE(ctx && key && data && net >= 0 && net <= DFVO_NET_POSENET && ndim >= 0 && ndim <= 4, DFVO_EINVAL, "dfvo_load_weight args");
  HostTensor t;
  size_t n = 1;
  for (int i = 0; i < ndim; ++i) { t.shape.push_back(shape[i]); n *= (size_t)shape[i]; }
  t.data.assign(data, data + n);
  ctx->weights[net][key] = std::move(t);
  return DFVO_OK;
  API_END
}

int dfvo_liteflow_build(dfvo_ctx* ctx, int height, int width, int pairs, int precision) {
  API_BEGIN
  DFVO_REQUIRE(ctx && pairs >= 1 && precision >= 0 && precision <= 2, DFVO_EINVAL, "dfvo_liteflow_build args");
  DFVO_CUDA(cudaSetDevice(ctx->device));
  delete ctx->lfn;
  ctx->lfn = nullptr;
  ctx->flow_graphs.clear();
  return liteflownet_create(ctx->weights[DFVO_NET_LITEFLOWNET], height, width, pairs, precision, &ctx->lfn);
  API_END
}

int dfvo_liteflow_forward(dfvo_ctx* ctx, const uint8_t* const* imgs, int n_imgs, float* flow_fwd, float* flow_bwd, float* flow_diff,
                          void* stream) {
  API_BEGIN
  DFVO_REQUIRE(ctx && ctx->lfn && imgs, DFVO_ESTATE, "dfvo_liteflow_forward: call dfvo_liteflow_build first");
  {
    int th, tw, B;
    ctx->lfn->geometry(&th, &tw, &B);
    DFVO_REQUIRE(n_imgs == B, DFVO_EINVAL, "dfvo_liteflow_forward: %d images given, the plan was built for %d (2 per pair)", n_imgs, B);
    for (int i = 0; i < n_imgs; ++i) DFVO_REQUIRE(imgs[i] != nullptr, DFVO_EINVAL, "dfvo_liteflow_forward: image %d is null", i);
  }
  // only the body -- the part that touches nothing but the runner's own buffers -- is replayed as a graph, so there is
  // one graph per network no matter which frame / output buffers the caller cycles through
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ctx->lfn->ingest(imgs, st);
  if (rc) return rc;
  rc = run_graphed(ctx->flow_graphs, std::vector<uintptr_t>(), st, [&]() { return ctx->lfn->body(st); });
  if (rc) return rc;
  return ctx->lfn->emit(flow_fwd, flow_bwd, flow_diff, st);
  API_END
}

int dfvo_liteflow_level_flow(dfvo_ctx* ctx, int level, float* out) {
  API_BEGIN
  DFVO_REQUIRE(ctx && ctx->lfn && out, DFVO_ESTATE, "dfvo_liteflow_level_flow: no plan");
  return ctx->lfn->debug_level_flow(level, 0, out);
  API_END
}

int dfvo_liteflow_geometry(dfvo_ctx* ctx, int* net_h, int* net_w, int* batch) {
  API_BEGIN
  DFVO_REQUIRE(ctx && ctx->lfn, DFVO_ESTATE, "dfvo_liteflow_geometry: no plan");
  ctx->lfn->geometry(net_h, net_w, batch);
  return DFVO_OK;
  API_END
}

// ------------------------------------------------------------------------------------------------
// stage-level entry points: NCHW fp32 at the boundary, converted to the internal NHWC layout here
// ------------------------------------------------------------------------------------------------

int dfvo_correlation(const float* first, const float* second, float* out, int B, int C, int H, int W, int stride, int leaky,
                     int precision, void* stream) {
  API_BEGIN
  DFVO_REQUIRE(first && second && out && B > 0 && C > 0 && H > 0 && W > 0, DFVO_EINVAL, "dfvo_correlation args");
  if (precision == DFVO_PREC_FP32) return stage_correlation<float>(first, second, out, B, C, H, W, stride, leaky, (cudaStream_t)stream);
  return stage_correlation<bf16>(first, second, out, B, C, H, W, stride, leaky, (cudaStream_t)stream);
  API_END
}


int dfvo_correlation_nhwc_bf16(const void* first, const void* second, void* out, int B, int C, int Cpitch, int H, int W, int stride,
                               int leaky, int second_nxor, void* stream) {
  API_BEGIN
  DFVO_REQUIRE(first && second && out && B > 0 && C > 0 && Cpitch >= C && Cpitch % 8 == 0 && H > 0 && W > 0 && (stride == 1 || stride == 2),
               DFVO_EINVAL, "dfvo_correlation_nhwc_bf16 args");
  const int Ho = (H + stride - 1) / stride, Wo = (W + stride - 1) / stride;
  Ten<bf16> A = make_ten<bf16>((bf16*)const_cast<void*>(first), B, H, W, C, Cpitch);
  Ten<bf16> Bn = make_ten<bf16>((bf16*)const_cast<void*>(second), B, H, W, C, Cpitch);
  Ten<bf16> O = make_ten<bf16>((bf16*)out, B, Ho, Wo, 64, 64);
  Ten<const float> noflow; memset(&noflow, 0, sizeof(noflow));
  Ten<bf16> noscratch; memset(&noscratch, 0, sizeof(noscratch));
  return correlation49_warped<bf16>(cten(A), cten(Bn), second_nxor, noflow, 0.f, stride, leaky, noscratch, O, (cudaStream_t)stream);
  API_END
}

int dfvo_backward_warp(const float* input, const float* flow, float* out, int B, int C, int H, int W, int precision, void* stream) {
  API_BEGIN
  DFVO_REQUIRE(input && flow && out && B > 0 && C > 0 && H > 0 && W > 0, DFVO_EINVAL, "dfvo_backward_warp args");
  if (precision == DFVO_PREC_FP32) return stage_warp<float>(input, flow, out, B, C, H, W, (cudaStream_t)stream);
  return stage_warp<bf16>(input, flow, out, B, C, H, W, (cudaStream_t)stream);
  API_END
}

int dfvo_fb_consistency(const float* flow_fwd, const float* flow_bwd, float* diff, int H, int W, void* stream) {
  API_BEGIN
  DFVO_REQUIRE(flow_fwd && flow_bwd && diff && H > 1 && W > 1, DFVO_EINVAL, "dfvo_fb_consistency args");
  return fb_consistency(flow_fwd, flow_bwd, H, W, diff, (cudaStream_t)stream);
  API_END
}

int dfvo_fb_consistency_batch(const float* flow_fwd, const float* flow_bwd, float* diff, int n_pairs, int H, int W, void* stream) {
  API_BEGIN
  DFVO_REQUIRE(flow_fwd && flow_bwd && diff && n_pairs > 0 && n_pairs <= 65535 && H > 1 && W > 1, DFVO_EINVAL, "dfvo_fb_consistency_batch args");
  return fb_consistency(flow_fwd, flow_bwd, H, W, diff, (cudaStream_t)stream, n_pairs, (long long)2 * H * W);
  API_END
}


int dfvo_conv2d(const float* x, const float* w_host, const float* bias_host, float* y, int B, int Cin, int H, int W, int Cout, int kh,
                int kw, int stride, int pad_y, int pad_x, int reflect, int act, int precision, void* stream) {
  API_BEGIN
  DFVO_REQUIRE(x && w_host && y && B > 0 && Cin > 0 && Cout > 0, DFVO_EINVAL, "dfvo_conv2d args");
  HostTensor w, b;
  w.shape = {Cout, Cin, kh, kw};
  w.data.assign(w_host, w_host + (size_t)Cout * Cin * kh * kw);
  if (bias_host) { b.shape = {Cout}; b.data.assign(bias_host, bias_host + Cout); }
  if (precision == DFVO_PREC_FP32)
    return stage_conv<float>(x, w, bias_host ? &b : nullptr, y, B, Cin, H, W, Cout, kh, kw, stride, pad_y, pad_x, reflect, act, (cudaStream_t)stream);
  DFVO_REQUIRE((stride == 1 || (stride == 2 && H % 2 == 0 && W % 2 == 0 && kh % 2 == 1 && pad_y == kh / 2 && pad_x == kw / 2)) && !reflect,
               DFVO_EINVAL, "dfvo_conv2d: the tensor-core path needs stride 1, or stride 2 on even sizes with 'same' padding; zero padding");
  if (precision == DFVO_PREC_TF32)
    return stage_conv<float>(x, w, bias_host ? &b : nullptr, y, B, Cin, H, W, Cout, kh, kw, stride, pad_y, pad_x, reflect, act, (cudaStream_t)stream, true);
  return stage_conv<bf16>(x, w, bias_host ? &b : nullptr, y, B, Cin, H, W, Cout, kh, kw, stride, pad_y, pad_x, reflect, act, (cudaStream_t)stream);
  API_END
}

int dfvo_monodepth2_build(dfvo_ctx* ctx, int feed_h, int feed_w, int precision, float min_depth, float max_depth, float baseline) {
  API_BEGIN
  DFVO_REQUIRE(ctx && precision >= 0 && precision <= 2, DFVO_EINVAL, "dfvo_monodepth2_build args");
  DFVO_CUDA(cudaSetDevice(ctx->device));
  delete ctx->mono;
  ctx->mono = nullptr;
  ctx->depth_graphs.clear();
  return monodepth2_create(ctx->weights[DFVO_NET_MONODEPTH2], feed_h, feed_w, precision, min_depth, max_depth, baseline, &ctx->mono);
  API_END
}

int dfvo_monodepth2_forward(dfvo_ctx* ctx, const float* img, float* depth_out, void* stream) {
  API_BEGIN
  DFVO_REQUIRE(ctx && ctx->mono && img && depth_out, DFVO_ESTATE, "dfvo_monodepth2_forward: call dfvo_monodepth2_build first");
  std::vector<uintptr_t> key = {(uintptr_t)img, (uintptr_t)depth_out};
  return run_graphed(ctx->depth_graphs, key, (cudaStream_t)stream, [&]() { return ctx->mono->run(img, depth_out, (cudaStream_t)stream); });
  API_END
}

int dfvo_posenet_build(dfvo_ctx* ctx, int feed_h, int feed_w, int precision, float baseline_multiplier) {
  API_BEGIN
  DFVO_REQUIRE(ctx && precision >= 0 && precision <= 2, DFVO_EINVAL, "dfvo_posenet_build args");
  DFVO_CUDA(cudaSetDevice(ctx->device));
  delete ctx->pose;
  ctx->pose = nullptr;
  ctx->pose_graphs.clear();
  return posenet_create(ctx->weights[DFVO_NET_POSENET], feed_h, feed_w, precision, baseline_multiplier, &ctx->pose);
  API_END
}

int dfvo_posenet_forward(dfvo_ctx* ctx, const float* feed_ref, const float* feed_cur, float* pose_out, void* stream) {
  API_BEGIN
  DFVO_REQUIRE(ctx && ctx->pose && feed_ref && feed_cur && pose_out, DFVO_ESTATE, "dfvo_posenet_forward: call dfvo_posenet_build first");
  std::vector<uintptr_t> key = {(uintptr_t)feed_ref, (uintptr_t)feed_cur, (uintptr_t)pose_out};
  return run_graphed(ctx->pose_graphs, key, (cudaStream_t)stream, [&]() { return ctx->pose->run(feed_ref, feed_cur, pose_out, (cudaStream_t)stream); });
  API_END
}

int dfvo_depth_consistency(const float* depth_cur, const float* depth_ref, int H, int W, const float* T, const float* K_host,
                           const float* inv_K_host, float* depth_diff, void* stream) {
  API_BEGIN
  DFVO_REQUIRE(depth_cur && depth_ref && T && K_host && inv_K_host && depth_diff && H > 1 && W > 1, DFVO_EINVAL, "dfvo_depth_consistency args");
  return geom_depth_consistency(depth_cur, depth_ref, H, W, T, K_host, inv_K_host, depth_diff, (cudaStream_t)stream);
  API_END
}

int dfvo_depth_post(const float* depth, int h, int w, int H, int W, double crop_y0, double crop_y1, double crop_x0, double crop_x1,
                    float min_depth, float max_depth, float* raw_out, float* depth_out, void* stream) {
  API_BEGIN
  DFVO_REQUIRE(depth && depth_out && h > 0 && w > 0 && H > 0 && W > 0, DFVO_EINVAL, "dfvo_depth_post args");
  return depth_post(depth, h, w, H, W, crop_y0, crop_y1, crop_x0, crop_x1, min_depth, max_depth, raw_out, depth_out, (cudaStream_t)stream);
  API_END
}

int dfvo_lanczos_resize_u8(const uint8_t* img, int H, int W, const int32_t* bounds_h, const int32_t* kk_h, int ksize_h,
                           const int32_t* bounds_v, const int32_t* kk_v, int ksize_v, int out_h, int out_w, uint8_t* tmp, uint8_t* out_u8,
                           float* out_nchw, void* stream) {
  API_BEGIN
  DFVO_REQUIRE(img && bounds_h && kk_h && bounds_v && kk_v && tmp && (out_u8 || out_nchw), DFVO_EINVAL, "dfvo_lanczos_resize_u8 args");
  return lanczos_resize_u8(img, H, W, bounds_h, kk_h, ksize_h, bounds_v, kk_v, ksize_v, out_h, out_w, tmp, out_u8, out_nchw,
                           (cudaStream_t)stream);
  API_END
}

int dfvo_local_bestn(const float* flow_diff, const float* depth_diff, int H, int W, int rows, int cols, int num_bestN, float thre,
                     float depth_thre, int32_t* idx_out, int32_t* cell_counts, int32_t* status, void* stream) {
  API_BEGIN
  DFVO_REQUIRE(flow_diff && idx_out && cell_counts && status && H > 0 && W > 0 && rows > 0 && cols > 0, DFVO_EINVAL, "dfvo_local_bestn args");
  int quota = num_bestN / (rows * cols);
  DFVO_REQUIRE(quota > 0, DFVO_EINVAL, "dfvo_local_bestn: num_bestN < rows*cols");
  return local_bestn(flow_diff, depth_diff, H, W, rows, cols, quota, thre, depth_thre, num_bestN, idx_out, cell_counts, status,
                     (cudaStream_t)stream);
  API_END
}

int dfvo_rigid_flow_diff(const float* raw_depth, const float* flow_fwd, int H, int W, const double* T_host, double fx, double fy, double cx,
                         double cy, float* out, void* stream) {
  API_BEGIN
  DFVO_REQUIRE(raw_depth && flow_fwd && T_host && out && H > 0 && W > 0, DFVO_EINVAL, "dfvo_rigid_flow_diff args");
  return rigid_flow_diff(raw_depth, flow_fwd, H, W, T_host, fx, fy, cx, cy, out, (cudaStream_t)stream);
  API_END
}

int dfvo_uniform_cells(const float* rigid_diff, const float* flow_diff, int H, int W, int rows, int cols, int num_bestN, float rigid_thre,
                       float flow_thre, int32_t* idx_out, int32_t* cell_counts, void* stream) {
  API_BEGIN
  DFVO_REQUIRE(rigid_diff && flow_diff && idx_out && cell_counts && H > 0 && W > 0 && rows > 0 && cols > 0, DFVO_EINVAL, "dfvo_uniform_cells args");
  const int quota = num_bestN / (rows * cols);
  DFVO_REQUIRE(quota > 0, DFVO_EINVAL, "dfvo_uniform_cells: num_bestN < rows*cols");
  return uniform_cells(rigid_diff, flow_diff, H, W, rows, cols, quota, rigid_thre, flow_thre, idx_out, cell_counts, (cudaStream_t)stream);
  API_END
}

size_t dfvo_bestn_workspace_bytes(int H, int W) { return bestn_workspace_bytes(H, W); }

int dfvo_bestn(const float* flow_diff, int H, int W, int N, int32_t* idx_out, void* workspace, size_t workspace_bytes, void* stream) {
  API_BEGIN
  DFVO_REQUIRE(flow_diff && idx_out && workspace, DFVO_EINVAL, "dfvo_bestn args");
  return bestn(flow_diff, H, W, N, idx_out, workspace, workspace_bytes, (cudaStream_t)stream);
  API_END
}

int dfvo_gather_keypoints(const int32_t* idx, const int32_t* cell_counts, int ncells, int quota, const float* flow_fwd, int H, int W,
                          double* kp1, double* kp2, int32_t* n_out, void* stream) {
  API_BEGIN
  DFVO_REQUIRE(idx && flow_fwd && kp1 && kp2, DFVO_EINVAL, "dfvo_gather_keypoints args");
  return gather_keypoints(idx, cell_counts, ncells, quota, flow_fwd, H, W, kp1, kp2, n_out, (cudaStream_t)stream);
  API_END
}

int dfvo_gather_depth(const float* depth, int H, int W, const double* kp, int n, float* out, void* stream) {
  API_BEGIN
  DFVO_REQUIRE(depth && kp && out && n > 0, DFVO_EINVAL, "dfvo_gather_depth args");
  return gather_depth(depth, H, W, kp, n, out, (cudaStream_t)stream);
  API_END
}

int dfvo_backproject(const float* depth, int H, int W, const double* iK9, float* points, void* stream) {
  API_BEGIN
  DFVO_REQUIRE(depth && iK9 && points && H > 0 && W > 0, DFVO_EINVAL, "dfvo_backproject args");
  return geom_backproject(depth, H, W, iK9, points, (cudaStream_t)stream);
  API_END
}

int dfvo_transform3d(const float* points, long long n, const double* T16, float* out, void* stream) {
  API_BEGIN
  DFVO_REQUIRE(points && T16 && out && n > 0, DFVO_EINVAL, "dfvo_transform3d args");
  return geom_transform3d(points, (size_t)n, T16, out, (cudaStream_t)stream);
  API_END
}

int dfvo_project(const float* points, int H, int W, const double* K12, float eps, int normalized, float* xy, void* stream) {
  API_BEGIN
  DFVO_REQUIRE(points && K12 && xy && H > 1 && W > 1, DFVO_EINVAL, "dfvo_project args");
  return geom_project(points, H, W, K12, eps, normalized, xy, (cudaStream_t)stream);
  API_END
}

int dfvo_reproject(const float* depth, int H, int W, const double* T16, const double* K12, const double* iK9, float eps, int normalized,
                   float* xy, void* stream) {
  API_BEGIN
  DFVO_REQUIRE(depth && T16 && K12 && iK9 && xy && H > 1 && W > 1, DFVO_EINVAL, "dfvo_reproject args");
  return geom_reproject(depth, H, W, T16, K12, iK9, eps, normalized, 0, xy, (cudaStream_t)stream);
  API_END
}

int dfvo_rigid_flow(const float* depth, int H, int W, const double* T16, const double* K12, const double* iK9, float* flow, void* stream) {
  API_BEGIN
  DFVO_REQUIRE(depth && T16 && K12 && iK9 && flow && H > 1 && W > 1, DFVO_EINVAL, "dfvo_rigid_flow args");
  return geom_reproject(depth, H, W, T16, K12, iK9, 1e-7f, 0, 1, flow, (cudaStream_t)stream);
  API_END
}

int dfvo_five_point(const double* x1, const double* x2, int M, double* E, int32_t* n, void* stream) {
  API_BEGIN
  DFVO_REQUIRE(x1 && x2 && E && n && M > 0, DFVO_EINVAL, "dfvo_five_point args");
  return five_point(x1, x2, M, E, n, (cudaStream_t)stream);
  API_END
}

int dfvo_score_hypotheses(const double* E, int M, const double* x1, const double* x2, int N, double thr2, int32_t* counts,
                          void* stream) {
  API_BEGIN
  DFVO_REQUIRE(E && x1 && x2 && counts && M > 0 && N > 0, DFVO_EINVAL, "dfvo_score_hypotheses args");
  return score_hypotheses(E, M, x1, x2, N, thr2, counts, (cudaStream_t)stream);
  API_END
}

size_t dfvo_essential_workspace_bytes(int N, int R, int max_iters) { return essential_workspace_bytes(N, R, max_iters); }

int dfvo_essential_ransac(const double* p1, const double* p2, int N, const int32_t* perm, int R, const int32_t* subsets, int max_iters,
                          double fx, double fy, double cx, double cy, double threshold, double prob, void* workspace,
                          size_t workspace_bytes, double* E_out, uint8_t* mask_out, int32_t* info, double* gric, void* stream) {
  API_BEGIN
  DFVO_REQUIRE(p1 && p2 && subsets && workspace && E_out && mask_out && info && gric, DFVO_EINVAL, "dfvo_essential_ransac args");
  return essential_ransac(p1, p2, N, perm, R, subsets, max_iters, fx, fy, cx, cy, threshold, prob, workspace, workspace_bytes, E_out,
                          mask_out, info, gric, (cudaStream_t)stream);
  API_END
}

int dfvo_cv_subset_stream_host(int count, int model_points, int n_subsets, int32_t* out) {
  API_BEGIN
  DFVO_REQUIRE(out && count >= model_points && model_points > 0 && model_points <= 16 && n_subsets > 0, DFVO_EINVAL, "dfvo_cv_subset_stream_host args");
  uint64_t state = 0xFFFFFFFFFFFFFFFFull;                       // cv::RNG((uint64)-1)
  for (int s = 0; s < n_subsets; ++s) {
    int32_t* idx = out + (size_t)s * model_points;
    for (int i = 0; i < model_points;) {
      state = (uint64_t)(uint32_t)state * 4164903690u + (uint32_t)(state >> 32);   // cv::RNG::next
      int v = (int)((uint32_t)state % (uint32_t)count);         // uniform(0, count)
      bool dup = false;
      for (int j = 0; j < i; ++j) dup = dup || idx[j] == v;
      if (dup) continue;
      idx[i++] = v;
    }
  }
  return DFVO_OK;
  API_END
}

int dfvo_triangulate_depth(const double* x1, const double* x2, int N, const double* T21, double* depth2, void* stream) {
  API_BEGIN
  DFVO_REQUIRE(x1 && x2 && T21 && depth2 && N > 0, DFVO_EINVAL, "dfvo_triangulate_depth args");
  return triangulate_depth(x1, x2, N, T21, depth2, (cudaStream_t)stream);
  API_END
}

int dfvo_triangulate_points(const double* x1, const double* x2, int N, const double* T1w, const double* T2w, double* X, double* X1, double* X2,
                            void* stream) {
  API_BEGIN
  DFVO_REQUIRE(x1 && x2 && T1w && T2w && N > 0, DFVO_EINVAL, "dfvo_triangulate_points args");
  return triangulate_points(x1, x2, N, T1w, T2w, X, X1, X2, (cudaStream_t)stream);
  API_END
}

int dfvo_recover_pose(const double* E, const double* p1, const double* p2, int N, double focal, double cx, double cy, double* Rt_out,
                      uint8_t* mask_out, int32_t* info, void* stream) {
  API_BEGIN
  DFVO_REQUIRE(E && p1 && p2 && Rt_out && mask_out && info && N > 0, DFVO_EINVAL, "dfvo_recover_pose args");
  return recover_pose(E, p1, p2, N, focal, cx, cy, Rt_out, mask_out, info, (cudaStream_t)stream);
  API_END
}

size_t dfvo_homography_workspace_bytes(int N, int max_iters) { return homography_workspace_bytes(N, max_iters); }

int dfvo_homography_ransac(const double* p1, const double* p2, int N, int max_iters, double threshold, double prob, void* workspace,
                           size_t workspace_bytes, double* H_out, uint8_t* mask_out, int32_t* info, double* gric, void* stream) {
  API_BEGIN
  DFVO_REQUIRE(workspace != nullptr, DFVO_EINVAL, "dfvo_homography_ransac: null workspace");
  return homography_ransac(p1, p2, N, max_iters, threshold, prob, workspace, workspace_bytes, H_out, mask_out, info, gric,
                           (cudaStream_t)stream);
  API_END
}

size_t dfvo_pnp_workspace_bytes(int N, int R, int iters) { return pnp_workspace_bytes(N, R, iters); }

int dfvo_pnp_ransac(const double* obj, const double* img, int N, const int32_t* perm, int R, const int32_t* subsets, int iters,
                    double fx, double fy, double cx, double cy, double threshold, double prob, void* workspace,
                    size_t workspace_bytes, double* rt_out, int32_t* info, void* stream) {
  API_BEGIN
  DFVO_REQUIRE(workspace != nullptr, DFVO_EINVAL, "dfvo_pnp_ransac: null workspace");
  return pnp_ransac(obj, img, N, perm, R, subsets, iters, fx, fy, cx, cy, threshold, prob, workspace, workspace_bytes, rt_out, info,
                    (cudaStream_t)stream);
  API_END
}

int dfvo_scale_ransac(const double* ratio, int n, int min_samples, int max_trials, double stop_prob, double threshold, double* io,
                      int32_t* perm_scratch, void* stream) {
  API_BEGIN
  return scale_ransac(ratio, n, min_samples, max_trials, stop_prob, threshold, io, perm_scratch, (cudaStream_t)stream);
  API_END
}

size_t dfvo_essential_tail_workspace_bytes(int N) { return essential_tail_workspace_bytes(N); }
int dfvo_essential_tail(const double* E, const int32_t* info, const double* gric, int R, const double* kp_cur, const double* kp_ref, int N,
                        double fx, double fy, double cx, double cy, const double* h_gric, const float* depth, int H, int W,
                        int min_samples, int max_trials, double stop_prob, double threshold, void* workspace, size_t workspace_bytes,
                        double* res, uint8_t* pose_mask, int32_t* pose_info, void* stream) {
  API_BEGIN
  return essential_tail(E, info, gric, R, kp_cur, kp_ref, N, fx, fy, cx, cy, h_gric, depth, H, W, min_samples, max_trials, stop_prob, threshold,
                        workspace, workspace_bytes, res, pose_mask, pose_info, (cudaStream_t)stream);
  API_END
}

int dfvo_flow_mean(const double* kp_ref, const double* kp_cur, int n, const int32_t* status, double* out, void* stream) {
  API_BEGIN
  DFVO_REQUIRE(kp_ref && kp_cur && out, DFVO_EINVAL, "dfvo_flow_mean args");
  return flow_mean(kp_ref, kp_cur, n, status, out, (cudaStream_t)stream);
  API_END
}

int dfvo_pnp_filter(const double* kp_ref, const double* kp_cur, int n, const float* depth, int H, int W, double min_depth, double max_depth,
                    const double* iK_host, double* obj, double* img, int32_t* count, void* stream) {
  API_BEGIN
  return pnp_filter(kp_ref, kp_cur, n, depth, H, W, min_depth, max_depth, iK_host, obj, img, count, (cudaStream_t)stream);
  API_END
}

size_t dfvo_pnp_tail_workspace_bytes(int N, int R, int iters) { return pnp_tail_workspace_bytes(N, R, iters); }
int dfvo_pnp_tail(const double* obj, const double* img, int N, const int32_t* perm, int R, const int32_t* subsets, int iters, double fx,
                  double fy, double cx, double cy, double threshold, double prob, void* workspace, size_t workspace_bytes, double* res,
                  void* stream) {
  API_BEGIN
  DFVO_REQUIRE(workspace != nullptr, DFVO_EINVAL, "dfvo_pnp_tail: null workspace");
  return pnp_tail(obj, img, N, perm, R, subsets, iters, fx, fy, cx, cy, threshold, prob, workspace, workspace_bytes, res, (cudaStream_t)stream);
  API_END
}

int dfvo_epnp_minimal(const double* obj, const double* img, int M, double fx, double fy, double cx, double cy, int coop, double* rt,
                      int32_t* ok, void* stream) {
  API_BEGIN
  return epnp_minimal(obj, img, M, fx, fy, cx, cy, coop, rt, ok, (cudaStream_t)stream);
  API_END
}

}  // extern "C"
