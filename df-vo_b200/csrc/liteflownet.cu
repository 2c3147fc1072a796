// LiteFlowNet forward + backward flow for P image pairs, device-resident from uint8 frames to the
// [2,H,W] flows and the forward-backward consistency map.
// Restates LiteFlow.inference_flow / inference (lite_flow.py:55-148), DeepFlow.get_target_size /
// resize_dense_flow / forward_backward_consistency (deep_flow.py:89-129,171-196) and
// LiteFlowNet.forward with its Features / Matching / Subpixel / Regularization modules
// (lite_flow_net.py:35-325).  Differences in *how* (not what):
//   * the reference stacks (img1,img2) and (img2,img1) and runs Features on all four images; the two
//     unique images are encoded once here and the "second" operand is addressed as batch index n^1;
//   * activations are NHWC; concatenations are channel slots of one buffer that producers write into
//     directly (no torch.cat copies); small channel groups are zero-padded to 16;
//   * T = float: every conv on the CUDA-core kernel (parity mode);  T = bf16: stride-1 convs with
//     >=16 input channels on the wgmma kernel, the rest on the CUDA-core kernel.
#include "liteflownet.h"

#include <stdlib.h>
#include <string.h>

namespace dfvo {

static const int kFeatC[7] = {0, 32, 32, 64, 96, 128, 192};
static const int kKLast[7] = {0, 0, 7, 5, 5, 3, 3};
static const float kBackward[7] = {0.f, 0.f, 10.f, 5.f, 2.5f, 1.25f, 0.625f};

// DeepFlow.get_target_size (deep_flow.py:89-105), operation for operation in float64: the reference
// shadows h,w with the candidate arrays, so it minimises |h_i*(1/w_j) - h_j/w_j|; the diagonal is zero
// only up to one rounding, hence floor multiples of 32 for 376x1241 but ceil multiples for 192x640.
void liteflow_target_size(int h, int w, int* th, int* tw) {
  const double hh[2] = {32.0 * (h / 32), 32.0 * (h / 32 + 1)};
  const double ww[2] = {32.0 * (w / 32), 32.0 * (w / 32 + 1)};
  int best = 0;
  double bestv = 0.0;
  for (int i = 0; i < 2; ++i)
    for (int j = 0; j < 2; ++j) {
      volatile double inv = 1.0 / ww[j];
      volatile double prod = hh[i] * inv;
      volatile double quot = hh[j] / ww[j];
      double r = prod - quot;
      if (r < 0) r = -r;
      if ((i == 0 && j == 0) || r < bestv) { bestv = r; best = i * 2 + j; }
    }
  *th = (int)hh[best / 2];
  *tw = (int)ww[best % 2];
}

template <typename T> struct IsBf16 { enum { v = 0 }; };
template <> struct IsBf16<bf16> { enum { v = 1 }; };

template <typename T>
struct LfnImpl : public LiteFlowNetBase {
  Arena arena;
  bool tf32 = false;          // T = float only: convs on wgmma tf32 (DFVO_PREC_TF32) instead of the CUDA-core kernel
  int H0 = 0, W0 = 0, th = 0, tw = 0, B = 0, P = 0;
  int lh[7], lw[7];
  // weights
  ConvLayer fOne, fTwo0, fTwo2, fTwo4, fThr0, fThr2, fFou0, fFou2, fFiv0, fSix0;
  struct Lvl {
    ConvLayer mFeat, mMain0, mMain2, mMain4, mMain6;
    float* upflow = nullptr; float* upcorr = nullptr;
    ConvLayer sFeat, sMain0, sMain2, sMain4, sMain6;
    ConvLayer rFeat, rMain[6], rDist0, rDist1;
    float* wx = nullptr; float* wy = nullptr; float bx = 0.f, by = 0.f;
  } lv[7];
  // buffers
  float* img[7];              // [B,h,w,4] fp32 pyramid (img[1] = network input)
  bool stem_window = false;
  T* imgpad = nullptr;
  T *f1buf, *rowbuf, *t2a, *t2b, *feat2, *t3a, *t4a;
  T* subcat[7]; int subC[7];
  T *mfeat, *warpbuf, *corr, *corrU, *b128a, *b128b, *b64a, *b64b, *b32a, *b32b, *d0, *d1, *regcat;
  float *flow_up, *flow_m, *flow_s, *flow_r[7], *meanbuf;
  unsigned* chain_bars = nullptr;   // arrival counters of the layer chains: one block per chain site of the forward pass
  int chain_site = 0;
  unsigned* next_chain() { return (IsBf16<T>::v && chain_bars && chain_site < 64) ? chain_bars + (chain_site++) * CHAIN_BAR_WORDS : nullptr; }
  float* out_planar = nullptr;   // [B][2][H0][W0]

  ~LfnImpl() override {}

  Ten<T> view(T* p, int L, int C, int pitch) { return make_ten<T>(p, B, lh[L], lw[L], C, pitch); }
  Ten<const T> cview(const T* p, int L, int C, int pitch) {
    Ten<const T> t; Ten<T> a = make_ten<T>(const_cast<T*>(p), B, lh[L], lw[L], C, pitch);
    t.p = a.p; t.N = a.N; t.H = a.H; t.W = a.W; t.C = a.C; t.sN = a.sN; t.sH = a.sH; t.sW = a.sW;
    return t;
  }
  Ten<float> fview(float* p, int L, int C, int pitch) { return make_ten<float>(p, B, lh[L], lw[L], C, pitch); }
  Ten<const float> cfview(const float* p, int L, int C, int pitch) {
    Ten<const float> t; Ten<float> a = make_ten<float>(const_cast<float*>(p), B, lh[L], lw[L], C, pitch);
    t.p = a.p; t.N = a.N; t.H = a.H; t.W = a.W; t.C = a.C; t.sN = a.sN; t.sH = a.sH; t.sW = a.sW;
    return t;
  }

  int conv_layer(const WeightStore& ws, const std::string& name, const std::vector<Seg>& segs, int stride, int pad_y,
                 int pad_x, bool tc_ok, ConvLayer* L) {
    const HostTensor* w = find_weight(ws, name + ".weight");
    const HostTensor* b = find_weight(ws, name + ".bias");
    DFVO_REQUIRE(w != nullptr, DFVO_ESTATE, "missing weight %s.weight", name.c_str());
    const bool want_tc = (IsBf16<T>::v || tf32) && tc_ok;
    // fp32 / tf32 modes keep the CUDA-core weights as well (2-channel heads, debugging)
    return build_conv_layer(arena, *w, b, segs, stride, pad_y, pad_x, 0, want_tc, !want_tc || !IsBf16<T>::v, nullptr, nullptr, L,
                            IsBf16<T>::v ? 2 : 4);
  }
  int raw_weight(const WeightStore& ws, const std::string& key, size_t n, float** out) {
    const HostTensor* w = find_weight(ws, key);
    DFVO_REQUIRE(w != nullptr && w->data.size() == n, DFVO_ESTATE, "missing/odd weight %s", key.c_str());
    *out = arena.alloc_t<float>(n);
    if (!*out) return DFVO_ENOMEM;
    DFVO_CUDA(cudaMemcpy(*out, w->data.data(), n * 4, cudaMemcpyHostToDevice));
    return DFVO_OK;
  }

#define TRY(x) do { int _rc = (x); if (_rc) return _rc; } while (0)

  int build(const WeightStore& ws, int H0_, int W0_, int pairs) {
    H0 = H0_; W0 = W0_; P = pairs; B = 2 * pairs;
    liteflow_target_size(H0, W0, &th, &tw);
    DFVO_REQUIRE(th >= 64 && tw >= 64, DFVO_ESHAPE, "image %dx%d too small for LiteFlowNet", H0, W0);
    for (int L = 1; L <= 6; ++L) { lh[L] = th >> (L - 1); lw[L] = tw >> (L - 1); }
    // ---------------- weights ----------------
    const std::string F = "moduleFeatures.";
    if (IsBf16<T>::v || tf32) {
      // stem on tensor cores: 7x7x3 -> 7x1 over a horizontal window of pixels.
      //   window mode (default): K = 64 = 8 pixels x 8 channels read straight from the column-padded image through an
      //     overlapping-box tensor map (flow_ops.cu::pad_image8), w'[co][px*8+c][ky] = w[co][c][ky][px], px < 7, c < 3;
      //   row-unroll mode (DFVO_STEM_WINDOW=0): K = 32 over the materialised [.., 7*3 -> 32] buffer (im2row7).
      const HostTensor* w7 = find_weight(ws, F + "moduleOne.0.weight");
      const HostTensor* b7 = find_weight(ws, F + "moduleOne.0.bias");
      DFVO_REQUIRE(w7 && w7->shape.size() == 4 && w7->shape[1] == 3 && w7->shape[2] == 7 && w7->shape[3] == 7, DFVO_ESTATE, "moduleOne weight");
      const char* env = getenv("DFVO_STEM_WINDOW");
      stem_window = IsBf16<T>::v && !(env && atoi(env) == 0);          // the 64-element window needs 2-byte elements (128-byte box rows)
      const int kk = stem_window ? 64 : 21, cs = stem_window ? 8 : 3;
      HostTensor wr;
      wr.shape = {w7->shape[0], kk, 7, 1};
      wr.data.assign((size_t)w7->shape[0] * kk * 7, 0.f);
      for (int co = 0; co < (int)w7->shape[0]; ++co)
        for (int c = 0; c < 3; ++c)
          for (int ky = 0; ky < 7; ++ky)
            for (int dx = 0; dx < 7; ++dx)
              wr.data[((size_t)co * kk + dx * cs + c) * 7 + ky] = w7->data[(((size_t)co * 3 + c) * 7 + ky) * 7 + dx];
      if (stem_window) {
        TRY(build_conv_layer(arena, wr, b7, {{64, 64}}, 1, 3, 0, 0, true, false, nullptr, nullptr, &fOne));
        fOne.Cin_ref = 21;                       // algorithmic FLOPs of the layer: 7 x 7 x 3 real taps per output channel
      } else {
        TRY(build_conv_layer(arena, wr, b7, {{21, 32}}, 1, 3, 0, 0, true, false, nullptr, nullptr, &fOne, IsBf16<T>::v ? 2 : 4));
      }
    } else {
      TRY(conv_layer(ws, F + "moduleOne.0", {{3, 3}}, 1, 3, 3, false, &fOne));
    }
    TRY(conv_layer(ws, F + "moduleTwo.0", {{32, 32}}, 2, 1, 1, true, &fTwo0));
    TRY(conv_layer(ws, F + "moduleTwo.2", {{32, 32}}, 1, 1, 1, true, &fTwo2));
    TRY(conv_layer(ws, F + "moduleTwo.4", {{32, 32}}, 1, 1, 1, true, &fTwo4));
    TRY(conv_layer(ws, F + "moduleThr.0", {{32, 32}}, 2, 1, 1, true, &fThr0));
    TRY(conv_layer(ws, F + "moduleThr.2", {{64, 64}}, 1, 1, 1, true, &fThr2));
    TRY(conv_layer(ws, F + "moduleFou.0", {{64, 64}}, 2, 1, 1, true, &fFou0));
    TRY(conv_layer(ws, F + "moduleFou.2", {{96, 96}}, 1, 1, 1, true, &fFou2));
    TRY(conv_layer(ws, F + "moduleFiv.0", {{96, 96}}, 2, 1, 1, true, &fFiv0));
    TRY(conv_layer(ws, F + "moduleSix.0", {{128, 128}}, 2, 1, 1, true, &fSix0));
    for (int L = 2; L <= 6; ++L) {
      Lvl& v = lv[L];
      const int k = L - 2, kl = kKLast[L], C = (L == 2) ? 64 : kFeatC[L];
      char buf[64];
      snprintf(buf, sizeof(buf), "moduleMatching.%d.", k); std::string M = buf;
      snprintf(buf, sizeof(buf), "moduleSubpixel.%d.", k); std::string S = buf;
      snprintf(buf, sizeof(buf), "moduleRegularization.%d.", k); std::string R = buf;
      if (L == 2) {
        TRY(conv_layer(ws, M + "moduleFeat.0", {{32, 32}}, 1, 0, 0, true, &v.mFeat));
        TRY(conv_layer(ws, S + "moduleFeat.0", {{32, 32}}, 1, 0, 0, true, &v.sFeat));
      }
      if (L != 6) TRY(raw_weight(ws, M + "moduleUpflow.weight", 2 * 16, &v.upflow));
      if (L < 4) TRY(raw_weight(ws, M + "moduleUpcorr.weight", 49 * 16, &v.upcorr));
      TRY(conv_layer(ws, M + "moduleMain.0", {{49, 64}}, 1, 1, 1, true, &v.mMain0));
      TRY(conv_layer(ws, M + "moduleMain.2", {{128, 128}}, 1, 1, 1, true, &v.mMain2));
      TRY(conv_layer(ws, M + "moduleMain.4", {{64, 64}}, 1, 1, 1, true, &v.mMain4));
      TRY(conv_layer(ws, M + "moduleMain.6", {{32, 32}}, 1, kl / 2, kl / 2, true, &v.mMain6));
      TRY(conv_layer(ws, S + "moduleMain.0", {{C, C}, {C, C}, {2, 16}}, 1, 1, 1, true, &v.sMain0));
      TRY(conv_layer(ws, S + "moduleMain.2", {{128, 128}}, 1, 1, 1, true, &v.sMain2));
      TRY(conv_layer(ws, S + "moduleMain.4", {{64, 64}}, 1, 1, 1, true, &v.sMain4));
      TRY(conv_layer(ws, S + "moduleMain.6", {{32, 32}}, 1, kl / 2, kl / 2, true, &v.sMain6));
      const int RF = (L < 5) ? 128 : kFeatC[L];
      if (L < 5) TRY(conv_layer(ws, R + "moduleFeat.0", {{kFeatC[L], kFeatC[L]}}, 1, 0, 0, true, &v.rFeat));
      TRY(conv_layer(ws, R + "moduleMain.0", {{3, 16}, {RF, RF}}, 1, 1, 1, true, &v.rMain[0]));
      TRY(conv_layer(ws, R + "moduleMain.2", {{128, 128}}, 1, 1, 1, true, &v.rMain[1]));
      TRY(conv_layer(ws, R + "moduleMain.4", {{128, 128}}, 1, 1, 1, true, &v.rMain[2]));
      TRY(conv_layer(ws, R + "moduleMain.6", {{64, 64}}, 1, 1, 1, true, &v.rMain[3]));
      TRY(conv_layer(ws, R + "moduleMain.8", {{64, 64}}, 1, 1, 1, true, &v.rMain[4]));
      TRY(conv_layer(ws, R + "moduleMain.10", {{32, 32}}, 1, 1, 1, true, &v.rMain[5]));
      const int cd = kl * kl, cdp = (cd + 15) / 16 * 16;
      if (L >= 5) {
        TRY(conv_layer(ws, R + "moduleDist.0", {{32, 32}}, 1, kl / 2, kl / 2, true, &v.rDist0));
      } else {
        TRY(conv_layer(ws, R + "moduleDist.0", {{32, 32}}, 1, kl / 2, 0, true, &v.rDist0));
        TRY(conv_layer(ws, R + "moduleDist.1", {{cd, cdp}}, 1, 0, kl / 2, true, &v.rDist1));
      }
      TRY(raw_weight(ws, R + "moduleScaleX.weight", cd, &v.wx));
      TRY(raw_weight(ws, R + "moduleScaleY.weight", cd, &v.wy));
      const HostTensor* bx = find_weight(ws, R + "moduleScaleX.bias");
      const HostTensor* by = find_weight(ws, R + "moduleScaleY.bias");
      DFVO_REQUIRE(bx && by, DFVO_ESTATE, "missing ScaleX/Y bias");
      v.bx = bx->data[0]; v.by = by->data[0];
    }
    // ---------------- buffers ----------------
    auto px = [&](int L) { return (size_t)B * lh[L] * lw[L]; };
    for (int L = 1; L <= 6; ++L) { img[L] = arena.alloc_t<float>(px(L) * 4); if (!img[L]) return DFVO_ENOMEM; }
#define ALLOC(ptr, type, count) do { ptr = arena.alloc_t<type>(count); if (!ptr) return DFVO_ENOMEM; } while (0)
    ALLOC(f1buf, T, px(1) * 32);
    ALLOC(rowbuf, T, ((IsBf16<T>::v || tf32) && !stem_window) ? px(1) * 32 : 64);
    ALLOC(imgpad, T, (IsBf16<T>::v && stem_window) ? (size_t)B * lh[1] * (lw[1] + 8) * 8 + 64 : 64);
    ALLOC(t2a, T, px(2) * 32); ALLOC(t2b, T, px(2) * 32); ALLOC(feat2, T, px(2) * 32);
    ALLOC(t3a, T, px(3) * 64); ALLOC(t4a, T, px(4) * 96);
    subcat[1] = nullptr; subC[1] = 0;
    for (int L = 2; L <= 6; ++L) {
      int C = (L == 2) ? 64 : kFeatC[L];
      subC[L] = 2 * C + 16;
      ALLOC(subcat[L], T, px(L) * subC[L]);
    }
    ALLOC(mfeat, T, px(2) * 64);
    {  // warp scratch: max over levels of px*C
      size_t m = 0;
      for (int L = 2; L <= 6; ++L) { size_t v = px(L) * ((L == 2) ? 64 : kFeatC[L]); if (v > m) m = v; }
      ALLOC(warpbuf, T, m);
    }
    {  // correlation output (stride 1 at L4 is the largest) and its upsampled version
      size_t m = 0;
      for (int L = 2; L <= 6; ++L) { int s = L >= 4 ? 1 : 2; size_t v = (size_t)B * (lh[L] / s) * (lw[L] / s) * 64; if (v > m) m = v; }
      ALLOC(corr, T, m);
      ALLOC(corrU, T, px(2) * 64);
    }
    ALLOC(b128a, T, px(2) * 128); ALLOC(b128b, T, px(2) * 128);
    ALLOC(b64a, T, px(2) * 64); ALLOC(b64b, T, px(2) * 64);
    ALLOC(b32a, T, px(2) * 32); ALLOC(b32b, T, px(2) * 32);
    ALLOC(d0, T, px(2) * 64); ALLOC(d1, T, px(2) * 64);
    {
      size_t m = px(2) * 144;
      for (int L = 5; L <= 6; ++L) { size_t v = px(L) * (16 + kFeatC[L]); if (v > m) m = v; }
      ALLOC(regcat, T, m);
    }
    ALLOC(flow_up, float, px(2) * 2); ALLOC(flow_m, float, px(2) * 2); ALLOC(flow_s, float, px(2) * 2);
    for (int L = 2; L <= 6; ++L) ALLOC(flow_r[L], float, px(L) * 2);
    ALLOC(meanbuf, float, flow_mean_buffer_floats(B));
    ALLOC(out_planar, float, (size_t)B * 2 * H0 * W0);
    ALLOC(chain_bars, unsigned, 64 * CHAIN_BAR_WORDS);
    return DFVO_OK;
  }

  // ------------------------------------------------------------------------------------------
  // the only launches that read caller memory: uint8 frames -> normalised, resized network input
  int ingest(const uint8_t* const* imgs_u8, cudaStream_t s) override {
    Ten<float> i1 = fview(img[1], 1, 4, 4);
    for (int b = 0; b < B; ++b) TRY(prep_image_u8(imgs_u8[b], H0, W0, i1, b, s));
    return DFVO_OK;
  }

  int features(cudaStream_t s) {
    for (int L = 2; L <= 6; ++L) TRY(resize_bilinear_f32(cfview(img[L - 1], L - 1, 3, 4), fview(img[L], L, 4, 4), 0, s));
    Ten<const T> none; memset(&none, 0, sizeof(none));
    // level 1: 7x7 3->32.  bf16: row-unroll + wgmma 7x1 conv;  fp32: CUDA-core kernel on the float image
    if (IsBf16<T>::v && stem_window) {
      Ten<T> pad = make_ten<T>(imgpad, B, lh[1], lw[1] + 8, 8, 8);
      TRY(pad_image8<T>(cfview(img[1], 1, 3, 4), pad, s));
      // window view: pixel x of the view starts at padded column x (= image column x - 3) and spans 64 elements
      Ten<const T> win; win.p = imgpad; win.N = B; win.H = lh[1]; win.W = lw[1]; win.C = 64;
      win.sW = 8; win.sH = (long long)(lw[1] + 8) * 8; win.sN = (long long)lh[1] * (lw[1] + 8) * 8;
      TRY(run_conv<T>(fOne, win, view(f1buf, 1, 32, 32), ACT_LEAKY, none, 0, s));
    } else if (IsBf16<T>::v || tf32) {
      TRY(im2row7<T>(cfview(img[1], 1, 3, 4), view(rowbuf, 1, 32, 32), s));
      TRY(run_conv<T>(fOne, cview(rowbuf, 1, 32, 32), view(f1buf, 1, 32, 32), ACT_LEAKY, none, 0, s));
    } else {
      ConvDirect d; d.Cin = 3; d.Cout = 32; d.kh = 7; d.kw = 7; d.stride = 1; d.pad_y = 3; d.pad_x = 3; d.reflect = 0;
      d.act = ACT_LEAKY; d.w = fOne.w_direct; d.w_pitch = fOne.w_pitch; d.bias = fOne.bias;
      DFVO_REQUIRE(fOne.w_direct, DFVO_ESTATE, "moduleOne weights");
      TRY((conv_direct<float, T>(d, cfview(img[1], 1, 3, 4), view(f1buf, 1, 32, 32), none, s)));
    }
    ChainScope chain(s, next_chain());          // consecutive stride-1 layers of the pyramid become one launch
    TRY(run_conv<T>(fTwo0, cview(f1buf, 1, 32, 32), view(t2a, 2, 32, 32), ACT_LEAKY, none, 0, s));
    TRY(run_conv<T>(fTwo2, cview(t2a, 2, 32, 32), view(t2b, 2, 32, 32), ACT_LEAKY, none, 0, s));
    TRY(run_conv<T>(fTwo4, cview(t2b, 2, 32, 32), view(feat2, 2, 32, 32), ACT_LEAKY, none, 0, s));
    TRY(run_conv<T>(fThr0, cview(feat2, 2, 32, 32), view(t3a, 3, 64, 64), ACT_LEAKY, none, 0, s));
    TRY(run_conv<T>(fThr2, cview(t3a, 3, 64, 64), view(subcat[3], 3, 64, subC[3]), ACT_LEAKY, none, 0, s));
    TRY(run_conv<T>(fFou0, cview(subcat[3], 3, 64, subC[3]), view(t4a, 4, 96, 96), ACT_LEAKY, none, 0, s));
    TRY(run_conv<T>(fFou2, cview(t4a, 4, 96, 96), view(subcat[4], 4, 96, subC[4]), ACT_LEAKY, none, 0, s));
    TRY(run_conv<T>(fFiv0, cview(subcat[4], 4, 96, subC[4]), view(subcat[5], 5, 128, subC[5]), ACT_LEAKY, none, 0, s));
    TRY(run_conv<T>(fSix0, cview(subcat[5], 5, 128, subC[5]), view(subcat[6], 6, 192, subC[6]), ACT_LEAKY, none, 0, s));
    return chain.end();
  }

  int level(int L, const float* flow_prev, cudaStream_t s) {
    Lvl& v = lv[L];
    const int C = (L == 2) ? 64 : kFeatC[L];
    const int kl = kKLast[L];
    const float dbl = kBackward[L];
    Ten<const T> none; memset(&none, 0, sizeof(none));
    Ten<const float> fnone; memset(&fnone, 0, sizeof(fnone));
    // ------------------------------ Matching (lite_flow_net.py:132-152) ----------------------
    Ten<const T> f1m;
    if (L == 2) {
      TRY(run_conv<T>(v.mFeat, cview(feat2, 2, 32, 32), view(mfeat, 2, 64, 64), ACT_LEAKY, none, 0, s));
      f1m = cview(mfeat, 2, 64, 64);
    } else {
      f1m = cview(subcat[L], L, C, subC[L]);
    }
    const int cs = (L >= 4) ? 1 : 2;
    Ten<T> corr_o = make_ten<T>(corr, B, lh[L] / cs, lw[L] / cs, 64, 64);
    if (flow_prev) {
      Ten<const float> fp = cfview(flow_prev, L + 1, 2, 2);
      TRY(deconv4x4s2_dw<float>(fp, v.upflow, fview(flow_up, L, 2, 2), s));
      TRY(correlation49_warped<T>(f1m, f1m, 1, cfview(flow_up, L, 2, 2), dbl, cs, 1, view(warpbuf, L, C, C), corr_o, s));
    } else {
      TRY(correlation49_warped<T>(f1m, f1m, 1, fnone, 0.f, cs, 1, view(warpbuf, L, C, C), corr_o, s));
    }
    Ten<const T> cin;
    if (L < 4) {
      Ten<const T> ci; ci.p = corr; ci.N = B; ci.H = lh[L] / cs; ci.W = lw[L] / cs; ci.C = 49;
      ci.sW = 64; ci.sH = (long long)ci.W * 64; ci.sN = (long long)ci.H * ci.W * 64;
      TRY(deconv4x4s2_dw<T>(ci, v.upcorr, view(corrU, L, 64, 64), s));
      cin = cview(corrU, L, 64, 64);
    } else {
      cin = cview(corr, L, 64, 64);
    }
    {
      ChainScope chain(s, next_chain());
      TRY(run_conv<T>(v.mMain0, cin, view(b128a, L, 128, 128), ACT_LEAKY, none, 0, s));
      TRY(run_conv<T>(v.mMain2, cview(b128a, L, 128, 128), view(b64a, L, 64, 64), ACT_LEAKY, none, 0, s));
      TRY(run_conv<T>(v.mMain4, cview(b64a, L, 64, 64), view(b32a, L, 32, 32), ACT_LEAKY, none, 0, s));
      TRY(chain.end());
    }
    TRY(run_conv_f32out<T>(v.mMain6, cview(b32a, L, 32, 32), fview(flow_m, L, 2, 2), ACT_NONE,
                           flow_prev ? cfview(flow_up, L, 2, 2) : fnone, s));
    // ------------------------------ Subpixel (lite_flow_net.py:182-190) -----------------------
    if (L == 2) TRY(run_conv<T>(v.sFeat, cview(feat2, 2, 32, 32), view(subcat[2], 2, 64, subC[2]), ACT_LEAKY, none, 0, s));
    TRY(warp_bilinear<T>(cview(subcat[L], L, C, subC[L]), cfview(flow_m, L, 2, 2), dbl, 1, view(subcat[L] + C, L, C, subC[L]), s));
    TRY((convert_copy<float, T>(cfview(flow_m, L, 2, 2), view(subcat[L] + 2 * C, L, 16, subC[L]), s)));
    {
      ChainScope chain(s, next_chain());
      TRY(run_conv<T>(v.sMain0, cview(subcat[L], L, subC[L], subC[L]), view(b128a, L, 128, 128), ACT_LEAKY, none, 0, s));
      TRY(run_conv<T>(v.sMain2, cview(b128a, L, 128, 128), view(b64a, L, 64, 64), ACT_LEAKY, none, 0, s));
      TRY(run_conv<T>(v.sMain4, cview(b64a, L, 64, 64), view(b32a, L, 32, 32), ACT_LEAKY, none, 0, s));
      TRY(chain.end());
    }
    TRY(run_conv_f32out<T>(v.sMain6, cview(b32a, L, 32, 32), fview(flow_s, L, 2, 2), ACT_NONE, cfview(flow_m, L, 2, 2), s));
    // ------------------------------ Regularization (lite_flow_net.py:243-264) ------------------
    const int RF = (L < 5) ? 128 : kFeatC[L];
    const int RC = 16 + RF;
    TRY(flow_mean(cfview(flow_s, L, 2, 2), meanbuf, s));
    TRY(reg_prep<T>(cfview(img[L], L, 3, 4), cfview(img[L], L, 3, 4), 1, cfview(flow_s, L, 2, 2), meanbuf, dbl,
                    view(regcat, L, 16, RC), s));
    if (L >= 5) TRY((convert_copy<T, T>(cview(subcat[L], L, RF, subC[L]), view(regcat + 16, L, RF, RC), s)));
    ChainScope chain(s, next_chain());            // rFeat, the six main layers and the distance conv(s): one launch
    if (L < 5) {
      Ten<const T> rf = (L == 2) ? cview(feat2, 2, 32, 32) : cview(subcat[L], L, kFeatC[L], subC[L]);
      TRY(run_conv<T>(v.rFeat, rf, view(regcat + 16, L, 128, RC), ACT_LEAKY, none, 0, s));
    }
    TRY(run_conv<T>(v.rMain[0], cview(regcat, L, RC, RC), view(b128a, L, 128, 128), ACT_LEAKY, none, 0, s));
    TRY(run_conv<T>(v.rMain[1], cview(b128a, L, 128, 128), view(b128b, L, 128, 128), ACT_LEAKY, none, 0, s));
    TRY(run_conv<T>(v.rMain[2], cview(b128b, L, 128, 128), view(b64a, L, 64, 64), ACT_LEAKY, none, 0, s));
    TRY(run_conv<T>(v.rMain[3], cview(b64a, L, 64, 64), view(b64b, L, 64, 64), ACT_LEAKY, none, 0, s));
    TRY(run_conv<T>(v.rMain[4], cview(b64b, L, 64, 64), view(b32a, L, 32, 32), ACT_LEAKY, none, 0, s));
    TRY(run_conv<T>(v.rMain[5], cview(b32a, L, 32, 32), view(b32b, L, 32, 32), ACT_LEAKY, none, 0, s));
    const int cd = kl * kl, cdp = (cd + 15) / 16 * 16;
    const T* dist;
    if (L >= 5) {
      TRY(run_conv<T>(v.rDist0, cview(b32b, L, 32, 32), view(d0, L, cd, cdp), ACT_NONE, none, 0, s));
      dist = d0;
    } else {
      TRY(run_conv<T>(v.rDist0, cview(b32b, L, 32, 32), view(d0, L, cd, cdp), ACT_NONE, none, cdp, s));
      TRY(run_conv<T>(v.rDist1, cview(d0, L, cdp, cdp), view(d1, L, cd, cdp), ACT_NONE, none, 0, s));
      dist = d1;
    }
    TRY(chain.end());
    TRY(reg_tail<T>(cview(dist, L, cd, cdp), cfview(flow_s, L, 2, 2), kl, v.wx, v.wy, v.bx, v.by, fview(flow_r[L], L, 2, 2), s));
    return DFVO_OK;
  }

  // everything between the ingest and the emit: touches only buffers this object owns, so it is one fixed launch
  // sequence (replayed as a CUDA graph by the C-ABI layer)
  int body(cudaStream_t s) override {
    chain_site = 0;
    TRY(features(s));
    const float* prev = nullptr;
    for (int L = 6; L >= 2; --L) {
      TRY(level(L, prev, s));
      prev = flow_r[L];
    }
    // flows[1] = flow * 20 * 0.5^1 (lite_flow_net.py:322-324), then resize_dense_flow (deep_flow.py:107-129)
    TRY(flow_upsample_final(cfview(flow_r[2], 2, 2, 2), 10.0f, H0, W0, out_planar, s));
    return DFVO_OK;
  }

  // the only launches that write caller memory: consistency map + copies of the two flows
  int emit(float* flow_fwd, float* flow_bwd, float* flow_diff, cudaStream_t s) override {
    const size_t plane2 = (size_t)2 * H0 * W0;
    // all pairs in one launch: pair p's forward / backward flows sit at out_planar + (2p, 2p + 1) * plane2
    if (flow_diff) TRY(fb_consistency(out_planar, out_planar + plane2, H0, W0, flow_diff, s, P, (long long)(2 * plane2)));
    for (int p = 0; p < P; ++p) {
      const float* f = out_planar + (size_t)(2 * p) * plane2;
      const float* b = out_planar + (size_t)(2 * p + 1) * plane2;
      if (flow_fwd) DFVO_CUDA(cudaMemcpyAsync(flow_fwd + p * plane2, f, plane2 * 4, cudaMemcpyDeviceToDevice, s));
      if (flow_bwd) DFVO_CUDA(cudaMemcpyAsync(flow_bwd + p * plane2, b, plane2 * 4, cudaMemcpyDeviceToDevice, s));
    }
    return DFVO_OK;
  }

  int run(const uint8_t* const* imgs_u8, float* flow_fwd, float* flow_bwd, float* flow_diff, cudaStream_t s) override {
    TRY(ingest(imgs_u8, s));
    TRY(body(s));
    return emit(flow_fwd, flow_bwd, flow_diff, s);
  }

  int debug_level_flow(int L, int which, float* out_nhwc2) override {
    // parity tests: copy a level's regularised flow (which=0) [B,h,w,2] to caller memory
    DFVO_REQUIRE(L >= 2 && L <= 6 && which == 0, DFVO_EINVAL, "debug_level_flow args");
    DFVO_CUDA(cudaMemcpy(out_nhwc2, flow_r[L], (size_t)B * lh[L] * lw[L] * 2 * 4, cudaMemcpyDeviceToDevice));
    return DFVO_OK;
  }
  void geometry(int* th_, int* tw_, int* B_) override { *th_ = th; *tw_ = tw; *B_ = B; }
  size_t bytes() override { return arena.total(); }
};

int liteflownet_create(const WeightStore& ws, int H0, int W0, int pairs, int precision, LiteFlowNetBase** out) {
  *out = nullptr;
  if (precision == 0 || precision == 2) {
    auto* p = new LfnImpl<float>();
    p->tf32 = precision == 2;
    int rc = p->build(ws, H0, W0, pairs);
    if (rc) { delete p; return rc; }
    *out = p;
  } else {
    auto* p = new LfnImpl<bf16>();
    int rc = p->build(ws, H0, W0, pairs);
    if (rc) { delete p; return rc; }
    *out = p;
  }
  return DFVO_OK;
}

}  // namespace dfvo
