// monodepth2 depth inference on the device.  Restates Monodepth2DepthNet.inference(_depth)
// (monodepth2.py:91-139), ResnetEncoder.forward (resnet_encoder.py:87-98, torchvision ResNet-18
// BasicBlocks, eval-mode BatchNorm folded into the conv weights), DepthDecoder.forward
// (depth_decoder.py:50-65) with Conv3x3 = ReflectionPad2d(1) + 3x3 conv (layers.py:121-136), ELU
// ConvBlocks (layers.py:106-118), nearest x2 upsampling (layers.py:347-350), sigmoid disparity and
// disp_to_depth (layers.py:16-25).  Only the scale-0 head is evaluated: depth_scales == [0] at
// inference (deep_depth.py:32), the other three heads never influence the output.
//
// Layout/plan: NHWC; every 3x3 decoder conv reads a reflection-padded buffer produced by one fused
// "nearest-upsample + concat skip + reflect-pad" kernel, so the convs are plain valid convs and run on
// the wgmma kernel (T = bf16) or the CUDA-core kernel (T = float, parity mode; stride-2 / 3-channel /
// 1-channel layers in both modes).
#include <stdlib.h>
#include "monodepth2.h"

#include <math.h>
#include <string.h>

namespace dfvo {

template <typename T> struct IsBf16m { enum { v = 0 }; };
template <> struct IsBf16m<bf16> { enum { v = 1 }; };

template <typename T>
struct MonoImpl : public Monodepth2Base {
  Arena arena;
  bool tf32 = false;          // T = float only: wgmma tf32 convs (DFVO_PREC_TF32)
  int h = 0, w = 0;
  float min_depth = 0.1f, max_depth = 100.f, baseline = 5.4f;
  ConvLayer conv1;
  ConvLayer conv1_tc;          // bf16: the 7x7 stride-2 stem on the tensor cores (see stem_tc_layer)
  bool stem_tc = false;
  T* imgpad = nullptr;        // [h][w+8][8] column-padded normalised image (zero borders / pad channels)
  struct Block { ConvLayer c1, c2, down; bool has_down = false; int stride = 1; } blk[4][2];
  ConvLayer up[10], disp0;
  // buffers
  T* x0;                      // normalised input NHWC (C=3, pitch 4)
  T* f[5];                    // encoder features
  int fh[5], fw[5], fc[5];
  T *pool, *tA, *tB, *tD;     // scratch at layer resolution
  T* padbuf;                  // reflection-padded conv input scratch
  T *dA, *dB;                 // decoder activations
  float* disp;
  unsigned* chain_bars = nullptr;     // arrival counters of the encoder's layer chain

  Ten<T> tv(T* p, int H, int W, int C, int pitch) { return make_ten<T>(p, 1, H, W, C, pitch); }
  Ten<const T> ctv(const T* p, int H, int W, int C, int pitch) { return cten(make_ten<T>(const_cast<T*>(p), 1, H, W, C, pitch)); }

#define TRYM(x) do { int _rc = (x); if (_rc) return _rc; } while (0)

  int bn_conv(const WeightStore& ws, const std::string& conv, const std::string& bn, int cin, int stride, int pad, bool tc_ok,
              ConvLayer* L) {
    const HostTensor* wgt = find_weight(ws, conv + ".weight");
    const HostTensor* g = find_weight(ws, bn + ".weight");
    const HostTensor* b = find_weight(ws, bn + ".bias");
    const HostTensor* m = find_weight(ws, bn + ".running_mean");
    const HostTensor* v = find_weight(ws, bn + ".running_var");
    DFVO_REQUIRE(wgt && g && b && m && v, DFVO_ESTATE, "missing weights for %s / %s", conv.c_str(), bn.c_str());
    const int cout = (int)wgt->shape[0];
    std::vector<float> scale(cout), shift(cout);
    for (int c = 0; c < cout; ++c) {
      scale[c] = g->data[c] / sqrtf(v->data[c] + 1e-5f);            // BatchNorm2d eps (torchvision default)
      shift[c] = b->data[c] - m->data[c] * scale[c];
    }
    const int cp = cin == 3 ? 3 : cin;
    const bool want_tc = (IsBf16m<T>::v || tf32) && tc_ok;
    return build_conv_layer(arena, *wgt, nullptr, {{cin, cp}}, stride, pad, pad, 0, want_tc, !want_tc || !IsBf16m<T>::v, scale.data(), shift.data(), L,
                            IsBf16m<T>::v ? 2 : 4);
  }
  // The stem (resnet_encoder.py:87-98: conv1 7x7 s2 p3 + bn1 + relu) as a stride-1 tensor-core convolution:
  //   * columns: output pixel x needs input columns 2x-3 .. 2x+3 = padded columns 2x .. 2x+6: a 64-element window (8 pixels x 8
  //     channels, the 8th pixel and channels 3..7 carry zero weights) starting at padded column 2x -- an overlapping-box view
  //     with a pixel stride of 2 padded pixels (32 B), exactly LiteFlowNet's window stem with a doubled stride;
  //   * rows: output row y needs input rows 2y-3 .. 2y+3.  Split the rows by parity (two views E, O of the same buffer with a row
  //     stride of two image rows): rows 2y+{-2,0,2} = E[y-1], E[y], E[y+1] (ky = 1, 3, 5) and rows 2y+{-3,-1,1,3} = O[y-2 .. y+1]
  //     (ky = 0, 2, 4, 6) -- a 4 x 1 window (dy = -2 .. 1) over the two sources, E's dy = -2 tap carrying zero weights.
  // 8 K-steps x 4 taps of N = 64 MMAs per 128 outputs instead of 147 x 64 scalar FMAs per output; zero padding by TMA out-of-bounds
  // fill (rows) and the zero borders of the padded image (columns).
  int stem_tc_layer(const WeightStore& ws) {
    const HostTensor* wgt = find_weight(ws, "encoder.conv1.weight");
    const HostTensor* g = find_weight(ws, "encoder.bn1.weight");
    const HostTensor* b = find_weight(ws, "encoder.bn1.bias");
    const HostTensor* m = find_weight(ws, "encoder.bn1.running_mean");
    const HostTensor* v = find_weight(ws, "encoder.bn1.running_var");
    DFVO_REQUIRE(wgt && g && b && m && v && wgt->shape.size() == 4 && wgt->shape[0] == 64 && wgt->shape[1] == 3 && wgt->shape[2] == 7 && wgt->shape[3] == 7,
                 DFVO_ESTATE, "encoder.conv1 / bn1 weights");
    std::vector<float> scale(64), shift(64);
    for (int c = 0; c < 64; ++c) {
      scale[c] = g->data[c] / sqrtf(v->data[c] + 1e-5f);
      shift[c] = b->data[c] - m->data[c] * scale[c];
    }
    HostTensor wr;
    wr.shape = {64, 128, 4, 1};
    wr.data.assign((size_t)64 * 128 * 4, 0.f);
    for (int co = 0; co < 64; ++co)
      for (int c = 0; c < 3; ++c)
        for (int ky = 0; ky < 7; ++ky)
          for (int dx = 0; dx < 7; ++dx) {
            const int src = (ky & 1) ? 0 : 1;                         // odd ky -> even input rows (E), even ky -> odd rows (O)
            const int kyy = (ky & 1) ? (ky + 1) / 2 : ky / 2;         // E: ky = 2 kyy - 1;  O: ky = 2 kyy
            wr.data[((size_t)co * 128 + src * 64 + dx * 8 + c) * 4 + kyy] = wgt->data[(((size_t)co * 3 + c) * 7 + ky) * 7 + dx];
          }
    return build_conv_layer(arena, wr, nullptr, {{64, 64}, {64, 64}}, 1, 2, 0, 0, true, false, scale.data(), shift.data(), &conv1_tc, 2);
  }

  int plain_conv(const WeightStore& ws, const std::string& name, int cin, bool tc_ok, ConvLayer* L) {
    const HostTensor* wgt = find_weight(ws, name + ".weight");
    const HostTensor* b = find_weight(ws, name + ".bias");
    DFVO_REQUIRE(wgt && b, DFVO_ESTATE, "missing weights for %s", name.c_str());
    const bool want_tc = (IsBf16m<T>::v || tf32) && tc_ok;
    // input is pre-padded by upcat_reflect -> the conv itself has no padding
    return build_conv_layer(arena, *wgt, b, {{cin, cin}}, 1, 0, 0, 0, want_tc, !want_tc || !IsBf16m<T>::v, nullptr, nullptr, L, IsBf16m<T>::v ? 2 : 4);
  }

  int build(const WeightStore& ws, int feed_h, int feed_w, float mind, float maxd, float base) {
    h = feed_h; w = feed_w; min_depth = mind; max_depth = maxd; baseline = base;
    // >= 64: the decoder reflection-pads the 1/32-resolution map by one pixel, which needs at least two rows and columns
    // (torch.nn.ReflectionPad2d refuses a 1-pixel map the same way)
    DFVO_REQUIRE(h % 32 == 0 && w % 32 == 0 && h >= 64 && w >= 64, DFVO_ESHAPE, "monodepth2 feed size must be a multiple of 32 and at least 64x64 (got %dx%d)", h, w);
    TRYM(bn_conv(ws, "encoder.conv1", "encoder.bn1", 3, 2, 3, false, &conv1));
    {
      const char* e = getenv("DFVO_MONO_STEM_TC");
      stem_tc = IsBf16m<T>::v && !(e && atoi(e) == 0);
      if (stem_tc) TRYM(stem_tc_layer(ws));
    }
    const int chans[4] = {64, 128, 256, 512};
    int cin = 64;
    for (int li = 0; li < 4; ++li) {
      for (int b = 0; b < 2; ++b) {
        char pre[64];
        snprintf(pre, sizeof(pre), "encoder.layer%d.%d.", li + 1, b);
        Block& B = blk[li][b];
        B.stride = (li > 0 && b == 0) ? 2 : 1;
        const int ci = b == 0 ? cin : chans[li];
        TRYM(bn_conv(ws, std::string(pre) + "conv1", std::string(pre) + "bn1", ci, B.stride, 1, true, &B.c1));
        TRYM(bn_conv(ws, std::string(pre) + "conv2", std::string(pre) + "bn2", chans[li], 1, 1, true, &B.c2));
        B.has_down = find_weight(ws, std::string(pre) + "downsample.0.weight") != nullptr;
        if (B.has_down) TRYM(bn_conv(ws, std::string(pre) + "downsample.0", std::string(pre) + "downsample.1", ci, B.stride, 0, true, &B.down));
      }
      cin = chans[li];
    }
    const int enc[5] = {64, 64, 128, 256, 512}, dec[5] = {16, 32, 64, 128, 256};
    int idx = 0;
    for (int i = 4; i >= 0; --i) {
      const int ci0 = (i == 4) ? enc[4] : dec[i + 1];
      char nm[64];
      snprintf(nm, sizeof(nm), "decoder.%d.conv.conv", idx);
      TRYM(plain_conv(ws, nm, ci0, true, &up[idx])); ++idx;
      const int ci1 = dec[i] + (i > 0 ? enc[i - 1] : 0);
      snprintf(nm, sizeof(nm), "decoder.%d.conv.conv", idx);
      TRYM(plain_conv(ws, nm, ci1, true, &up[idx])); ++idx;
    }
    TRYM(plain_conv(ws, "decoder.10.conv", 16, true, &disp0));      // bf16: tensor-core kernel with N padded 1 -> 16
    // ---------------- buffers ----------------
    fh[0] = h / 2; fw[0] = w / 2; fc[0] = 64;
    for (int i = 1; i < 5; ++i) { fh[i] = h >> (i + 1); fw[i] = w >> (i + 1); fc[i] = enc[i]; }
#define ALLOCM(ptr, type, count) do { ptr = arena.alloc_t<type>(count); if (!ptr) return DFVO_ENOMEM; } while (0)
    ALLOCM(x0, T, (size_t)h * w * 4);
    ALLOCM(imgpad, T, stem_tc ? (size_t)h * (w + 8) * 8 + 64 : 64);
    for (int i = 0; i < 5; ++i) ALLOCM(f[i], T, (size_t)fh[i] * fw[i] * fc[i]);
    const size_t big = (size_t)fh[1] * fw[1] * 64;      // largest BasicBlock tensor (layer1)
    ALLOCM(pool, T, big); ALLOCM(tA, T, big); ALLOCM(tB, T, big); ALLOCM(tD, T, big);
    // largest padded decoder input: i=1 stage (h/2+2)x(w/2+2)x96 vs i=0: (h+2)x(w+2)x16, i=2: (h/4+2)(w/4+2)x128 ...
    size_t pmax = 0;
    for (int i = 4; i >= 0; --i) {
      const int hh = h >> (i + 1), ww = w >> (i + 1);
      const int ci0 = (i == 4) ? enc[4] : dec[i + 1];
      const int ci1 = dec[i] + (i > 0 ? enc[i - 1] : 0);
      size_t a = (size_t)(hh + 2) * (ww + 2) * ci0, b2 = (size_t)(2 * hh + 2) * (2 * ww + 2) * ci1;
      if (a > pmax) pmax = a;
      if (b2 > pmax) pmax = b2;
    }
    { size_t d = (size_t)(h + 2) * (w + 2) * 16; if (d > pmax) pmax = d; }
    ALLOCM(padbuf, T, pmax);
    ALLOCM(dA, T, (size_t)h * w * 16 + (size_t)(h / 2) * (w / 2) * 32); ALLOCM(dB, T, (size_t)h * w * 16 + (size_t)(h / 2) * (w / 2) * 32);
    ALLOCM(disp, float, (size_t)h * w);
    ALLOCM(chain_bars, unsigned, 4 * CHAIN_BAR_WORDS);
    return DFVO_OK;
  }

  int basic_block(Block& B, const T* in, int ih, int iw, int ic, T* out, int oc, cudaStream_t s) {
    const int oh = ih / B.stride, ow = iw / B.stride;
    Ten<const T> none; memset(&none, 0, sizeof(none));
    TRYM(run_conv<T>(B.c1, ctv(in, ih, iw, ic, ic), tv(tA, oh, ow, oc, oc), ACT_RELU, none, 0, s));
    const T* idt = in;
    if (B.has_down) {
      TRYM(run_conv<T>(B.down, ctv(in, ih, iw, ic, ic), tv(tD, oh, ow, oc, oc), ACT_NONE, none, 0, s));
      idt = tD;
    }
    // out = relu(bn2(conv2(.)) + identity)   (torchvision BasicBlock.forward)
    TRYM(run_conv<T>(B.c2, ctv(tA, oh, ow, oc, oc), tv(out, oh, ow, oc, oc), ACT_RELU, ctv(idt, oh, ow, oc, oc), 0, s));
    return DFVO_OK;
  }

  int run(const float* img, float* depth_out, cudaStream_t s) override {
    Ten<const T> none; memset(&none, 0, sizeof(none));
    if (stem_tc) {
      const long long row = (long long)(w + 8) * 8;
      Ten<T> pv; pv.p = imgpad + 3 * 8; pv.N = 1; pv.H = h; pv.W = w; pv.C = 3; pv.sW = 8; pv.sH = row; pv.sN = (long long)h * row;
      TRYM(normalize_nchw_to_nhwc<T>(img, 1, 3, h, w, 0.45f, 0.225f, pv, s));          // borders / pad channels stay zero
      Ten<const T> eo[2];
      for (int par = 0; par < 2; ++par) {
        Ten<const T>& v = eo[par];
        v.p = imgpad + par * row; v.N = 1; v.H = h / 2; v.W = w / 2; v.C = 64; v.sW = 16; v.sH = 2 * row; v.sN = (long long)h * row;
      }
      TRYM(run_conv_multi<T>(conv1_tc, eo, 2, tv(f[0], fh[0], fw[0], 64, 64), ACT_RELU, 2.0 * fh[0] * fw[0] * 64.0 * 147.0, s));
    } else {
      TRYM(normalize_nchw_to_nhwc<T>(img, 1, 3, h, w, 0.45f, 0.225f, tv(x0, h, w, 4, 4), s));
      ConvDirect d = {3, 64, 7, 7, 2, 3, 3, 0, ACT_RELU, conv1.w_direct, conv1.w_pitch, conv1.bias};
      TRYM((conv_direct<T, T>(d, ctv(x0, h, w, 3, 4), tv(f[0], fh[0], fw[0], 64, 64), none, s)));
    }
    TRYM(maxpool3x3s2<T>(ctv(f[0], fh[0], fw[0], 64, 64), tv(pool, fh[1], fw[1], 64, 64), s));
    const T* cur = pool;
    int ch = fh[1], cw = fw[1], cc = 64;
    {
      // the encoder is convolutions only: consecutive stride-1 layers (c1 -> c2 of a block, and on into the next block) form chains
      ChainScope chain(s, IsBf16m<T>::v ? chain_bars : nullptr);
      for (int li = 0; li < 4; ++li) {
        const int oc = fc[li + 1];
        TRYM(basic_block(blk[li][0], cur, ch, cw, cc, tB, oc, s));
        ch /= blk[li][0].stride; cw /= blk[li][0].stride; cc = oc;
        TRYM(basic_block(blk[li][1], tB, ch, cw, cc, f[li + 1], oc, s));
        cur = f[li + 1];
      }
      TRYM(chain.end());
    }
    // ---------------- decoder (depth_decoder.py:50-65) ----------------
    const int dec[5] = {16, 32, 64, 128, 256};
    const T* x = f[4];
    int xh = fh[4], xw = fw[4], xc = fc[4];
    int idx = 0;
    for (int i = 4; i >= 0; --i) {
      // upconv(i,0): ConvBlock on x
      TRYM(upcat_reflect<T>(ctv(x, xh, xw, xc, xc), 1, none, tv(padbuf, xh + 2, xw + 2, xc, xc), s));
      TRYM(run_conv<T>(up[idx], ctv(padbuf, xh + 2, xw + 2, xc, xc), tv(dA, xh, xw, dec[i], dec[i]), ACT_ELU, none, 0, s));
      ++idx;
      // upsample x2, concat skip, upconv(i,1)
      const int sc = i > 0 ? fc[i - 1] : 0;
      Ten<const T> skip = none;
      if (i > 0) skip = ctv(f[i - 1], fh[i - 1], fw[i - 1], sc, sc);
      const int nh = 2 * xh, nw = 2 * xw, ncat = dec[i] + sc;
      TRYM(upcat_reflect<T>(ctv(dA, xh, xw, dec[i], dec[i]), 2, skip, tv(padbuf, nh + 2, nw + 2, ncat, ncat), s));
      TRYM(run_conv<T>(up[idx], ctv(padbuf, nh + 2, nw + 2, ncat, ncat), tv(dB, nh, nw, dec[i], dec[i]), ACT_ELU, none, 0, s));
      ++idx;
      x = dB; xh = nh; xw = nw; xc = dec[i];
      // swap scratch so the next stage does not overwrite its own input
      T* t = dA; dA = dB; dB = t;
      x = dA;
    }
    // dispconv scale 0: Conv3x3 (reflect) + sigmoid, 16 -> 1
    TRYM(upcat_reflect<T>(ctv(x, xh, xw, 16, 16), 1, none, tv(padbuf, xh + 2, xw + 2, 16, 16), s));
    {
      Ten<const float> fnone; memset(&fnone, 0, sizeof(fnone));
      TRYM(run_conv_f32out<T>(disp0, ctv(padbuf, xh + 2, xw + 2, 16, 16), make_ten<float>(disp, 1, h, w, 1, 1), ACT_SIGMOID, fnone, s));
    }
    TRYM(disp_to_depth(disp, h * w, min_depth, max_depth, baseline, depth_out, s));
    return DFVO_OK;
  }
  void geometry(int* hh, int* ww) override { *hh = h; *ww = w; }
  size_t bytes() override { return arena.total(); }
};

int monodepth2_create(const WeightStore& ws, int feed_h, int feed_w, int precision, float min_depth, float max_depth,
                      float baseline, Monodepth2Base** out) {
  *out = nullptr;
  if (precision == 0 || precision == 2) {
    auto* p = new MonoImpl<float>();
    p->tf32 = precision == 2;
    int rc = p->build(ws, feed_h, feed_w, min_depth, max_depth, baseline);
    if (rc) { delete p; return rc; }
    *out = p;
  } else {
    auto* p = new MonoImpl<bf16>();
    int rc = p->build(ws, feed_h, feed_w, min_depth, max_depth, baseline);
    if (rc) { delete p; return rc; }
    *out = p;
  }
  return DFVO_OK;
}

}  // namespace dfvo
