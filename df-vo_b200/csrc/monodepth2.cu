// monodepth2 depth and pose inference on the device.
//
// Depth: restates Monodepth2DepthNet.inference(_depth) (monodepth2.py:91-139), ResnetEncoder.forward
// (resnet_encoder.py:87-98, torchvision ResNet-18 BasicBlocks, eval-mode BatchNorm folded into the conv weights),
// DepthDecoder.forward (depth_decoder.py:50-65) with Conv3x3 = ReflectionPad2d(1) + 3x3 conv (layers.py:121-136), ELU
// ConvBlocks (layers.py:106-118), nearest x2 upsampling (layers.py:347-350), sigmoid disparity and disp_to_depth
// (layers.py:16-25).  Only the scale-0 head is evaluated: depth_scales == [0] at inference (deep_depth.py:32), the other
// three heads never influence the output.
//
// Pose: restates Monodepth2PoseNet.inference_pose (pose/monodepth2/monodepth2.py:86-119): ResnetEncoder(18, False, 2) over
// the [ref, cur] channel concatenation, PoseDecoder.forward (pose_decoder.py) and transformation_from_parameters(invert=True)
// (depth/monodepth2/layers.py:28-94), translation times stereo_baseline_multiplier.  The encoder is the depth network's
// (Resnet18Encoder below) with a 6-channel stem.
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

#define TRYM(x) do { int _rc = (x); if (_rc) return _rc; } while (0)
#define ALLOCM(ptr, type, count) do { ptr = arena.alloc_t<type>(count); if (!ptr) return DFVO_ENOMEM; } while (0)

template <typename T>
static Ten<T> tv(T* p, int H, int W, int C, int pitch) { return make_ten<T>(p, 1, H, W, C, pitch); }
template <typename T>
static Ten<const T> ctv(const T* p, int H, int W, int C, int pitch) { return cten(make_ten<T>(const_cast<T*>(p), 1, H, W, C, pitch)); }

// conv + eval-mode BatchNorm folded into the weights (torchvision BasicBlock / stem)
template <typename T>
static int bn_conv(Arena& arena, bool tf32, const WeightStore& ws, const std::string& conv, const std::string& bn, int cin, int stride,
                   int pad, bool tc_ok, ConvLayer* L) {
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
  const bool want_tc = (IsBf16m<T>::v || tf32) && tc_ok;
  return build_conv_layer(arena, *wgt, nullptr, {{cin, cin}}, stride, pad, pad, 0, want_tc, !want_tc || !IsBf16m<T>::v, scale.data(), shift.data(), L,
                          IsBf16m<T>::v ? 2 : 4);
}

// conv + bias; `pad` zero padding (the depth decoder's inputs are pre-padded by upcat_reflect and use pad 0)
template <typename T>
static int plain_conv(Arena& arena, bool tf32, const WeightStore& ws, const std::string& name, int cin, int pad, ConvLayer* L) {
  const HostTensor* wgt = find_weight(ws, name + ".weight");
  const HostTensor* b = find_weight(ws, name + ".bias");
  DFVO_REQUIRE(wgt && b, DFVO_ESTATE, "missing weights for %s", name.c_str());
  const bool want_tc = IsBf16m<T>::v || tf32;
  return build_conv_layer(arena, *wgt, b, {{cin, cin}}, 1, pad, pad, 0, want_tc, !want_tc || !IsBf16m<T>::v, nullptr, nullptr, L, IsBf16m<T>::v ? 2 : 4);
}

// ResnetEncoder.forward (resnet_encoder.py:87-98) over `cin` input channels: 3 for the depth network, 6 for the PoseNet
// (ResnetEncoder(18, False, 2): the two feeds concatenated on channels).  The feeds are normalised straight into channel slots
// 3i .. 3i+2 of the stem's input, so the concatenation is never materialised.
template <typename T>
struct Resnet18Encoder {
  bool tf32 = false;          // T = float only: wgmma tf32 convs (DFVO_PREC_TF32)
  int h = 0, w = 0, cin = 3;
  ConvLayer conv1;
  ConvLayer conv1_tc;          // bf16: the 7x7 stride-2 stem on the tensor cores (see stem_tc_layer)
  bool stem_tc = false;
  T* imgpad = nullptr;        // [h][w+8][8] column-padded normalised image (zero borders / pad channels)
  struct Block { ConvLayer c1, c2, down; bool has_down = false; int stride = 1; } blk[4][2];
  T* x0;                      // normalised input NHWC (cin channels, pitch xpitch())
  T* f[5];                    // encoder features
  int fh[5], fw[5], fc[5];
  T *pool, *tA, *tB, *tD;     // scratch at layer resolution
  unsigned* chain_bars = nullptr;     // arrival counters of the encoder's layer chain

  int xpitch() const { return cin == 3 ? 4 : 8; }

  // The stem (resnet_encoder.py:87-98: conv1 7x7 s2 p3 + bn1 + relu) as a stride-1 tensor-core convolution:
  //   * columns: output pixel x needs input columns 2x-3 .. 2x+3 = padded columns 2x .. 2x+6: a 64-element window (8 pixels x 8
  //     channels, the 8th pixel and channels cin..7 carry zero weights) starting at padded column 2x -- an overlapping-box view
  //     with a pixel stride of 2 padded pixels (32 B), exactly LiteFlowNet's window stem with a doubled stride;
  //   * rows: output row y needs input rows 2y-3 .. 2y+3.  Split the rows by parity (two views E, O of the same buffer with a row
  //     stride of two image rows): rows 2y+{-2,0,2} = E[y-1], E[y], E[y+1] (ky = 1, 3, 5) and rows 2y+{-3,-1,1,3} = O[y-2 .. y+1]
  //     (ky = 0, 2, 4, 6) -- a 4 x 1 window (dy = -2 .. 1) over the two sources, E's dy = -2 tap carrying zero weights.
  // 8 K-steps x 4 taps of N = 64 MMAs per 128 outputs instead of 49 cin x 64 scalar FMAs per output; zero padding by TMA
  // out-of-bounds fill (rows) and the zero borders of the padded image (columns).
  int stem_tc_layer(Arena& arena, const WeightStore& ws) {
    const HostTensor* wgt = find_weight(ws, "encoder.conv1.weight");
    const HostTensor* g = find_weight(ws, "encoder.bn1.weight");
    const HostTensor* b = find_weight(ws, "encoder.bn1.bias");
    const HostTensor* m = find_weight(ws, "encoder.bn1.running_mean");
    const HostTensor* v = find_weight(ws, "encoder.bn1.running_var");
    DFVO_REQUIRE(wgt && g && b && m && v && wgt->shape.size() == 4 && wgt->shape[0] == 64 && wgt->shape[1] == cin && wgt->shape[2] == 7 && wgt->shape[3] == 7,
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
      for (int c = 0; c < cin; ++c)
        for (int ky = 0; ky < 7; ++ky)
          for (int dx = 0; dx < 7; ++dx) {
            const int src = (ky & 1) ? 0 : 1;                         // odd ky -> even input rows (E), even ky -> odd rows (O)
            const int kyy = (ky & 1) ? (ky + 1) / 2 : ky / 2;         // E: ky = 2 kyy - 1;  O: ky = 2 kyy
            wr.data[((size_t)co * 128 + src * 64 + dx * 8 + c) * 4 + kyy] = wgt->data[(((size_t)co * cin + c) * 7 + ky) * 7 + dx];
          }
    return build_conv_layer(arena, wr, nullptr, {{64, 64}, {64, 64}}, 1, 2, 0, 0, true, false, scale.data(), shift.data(), &conv1_tc, 2);
  }

  int build_layers(Arena& arena, const WeightStore& ws, int feed_h, int feed_w, int in_ch) {
    h = feed_h; w = feed_w; cin = in_ch;
    TRYM(bn_conv<T>(arena, tf32, ws, "encoder.conv1", "encoder.bn1", cin, 2, 3, false, &conv1));
    {
      const char* e = getenv("DFVO_MONO_STEM_TC");
      stem_tc = IsBf16m<T>::v && !(e && atoi(e) == 0);
      if (stem_tc) TRYM(stem_tc_layer(arena, ws));
    }
    const int chans[4] = {64, 128, 256, 512};
    int ci0 = 64;
    for (int li = 0; li < 4; ++li) {
      for (int b = 0; b < 2; ++b) {
        char pre[64];
        snprintf(pre, sizeof(pre), "encoder.layer%d.%d.", li + 1, b);
        Block& B = blk[li][b];
        B.stride = (li > 0 && b == 0) ? 2 : 1;
        const int ci = b == 0 ? ci0 : chans[li];
        TRYM(bn_conv<T>(arena, tf32, ws, std::string(pre) + "conv1", std::string(pre) + "bn1", ci, B.stride, 1, true, &B.c1));
        TRYM(bn_conv<T>(arena, tf32, ws, std::string(pre) + "conv2", std::string(pre) + "bn2", chans[li], 1, 1, true, &B.c2));
        B.has_down = find_weight(ws, std::string(pre) + "downsample.0.weight") != nullptr;
        if (B.has_down)
          TRYM(bn_conv<T>(arena, tf32, ws, std::string(pre) + "downsample.0", std::string(pre) + "downsample.1", ci, B.stride, 0, true, &B.down));
      }
      ci0 = chans[li];
    }
    const int enc[5] = {64, 64, 128, 256, 512};
    fh[0] = h / 2; fw[0] = w / 2; fc[0] = 64;
    for (int i = 1; i < 5; ++i) { fh[i] = h >> (i + 1); fw[i] = w >> (i + 1); fc[i] = enc[i]; }
    return DFVO_OK;
  }

  int alloc_buffers(Arena& arena) {
    ALLOCM(x0, T, (size_t)h * w * xpitch());
    ALLOCM(imgpad, T, stem_tc ? (size_t)h * (w + 8) * 8 + 64 : 64);
    for (int i = 0; i < 5; ++i) ALLOCM(f[i], T, (size_t)fh[i] * fw[i] * fc[i]);
    const size_t big = (size_t)fh[1] * fw[1] * 64;      // largest BasicBlock tensor (layer1)
    ALLOCM(pool, T, big); ALLOCM(tA, T, big); ALLOCM(tB, T, big); ALLOCM(tD, T, big);
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

  // imgs: cin / 3 float NCHW [3,h,w] feeds in [0,1]; fills f[0..4]
  int run(const float* const* imgs, cudaStream_t s) {
    Ten<const T> none; memset(&none, 0, sizeof(none));
    if (stem_tc) {
      const long long row = (long long)(w + 8) * 8;
      for (int i = 0; i < cin / 3; ++i) {
        Ten<T> pv; pv.p = imgpad + 3 * 8 + 3 * i; pv.N = 1; pv.H = h; pv.W = w; pv.C = 3; pv.sW = 8; pv.sH = row; pv.sN = (long long)h * row;
        TRYM(normalize_nchw_to_nhwc<T>(imgs[i], 1, 3, h, w, 0.45f, 0.225f, pv, s));          // borders / pad channels stay zero
      }
      Ten<const T> eo[2];
      for (int par = 0; par < 2; ++par) {
        Ten<const T>& v = eo[par];
        v.p = imgpad + par * row; v.N = 1; v.H = h / 2; v.W = w / 2; v.C = 64; v.sW = 16; v.sH = 2 * row; v.sN = (long long)h * row;
      }
      TRYM(run_conv_multi<T>(conv1_tc, eo, 2, tv(f[0], fh[0], fw[0], 64, 64), ACT_RELU, 2.0 * fh[0] * fw[0] * 64.0 * (49.0 * cin), s));
    } else {
      for (int i = 0; i < cin / 3; ++i)
        TRYM(normalize_nchw_to_nhwc<T>(imgs[i], 1, 3, h, w, 0.45f, 0.225f, tv(x0 + 3 * i, h, w, 3, xpitch()), s));
      ConvDirect d = {cin, 64, 7, 7, 2, 3, 3, 0, ACT_RELU, conv1.w_direct, conv1.w_pitch, conv1.bias};
      TRYM((conv_direct<T, T>(d, ctv(x0, h, w, cin, xpitch()), tv(f[0], fh[0], fw[0], 64, 64), none, s)));
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
    return DFVO_OK;
  }
};

template <typename T>
struct MonoImpl : public Monodepth2Base {
  Arena arena;
  bool tf32 = false;          // T = float only: wgmma tf32 convs (DFVO_PREC_TF32)
  int h = 0, w = 0;
  float min_depth = 0.1f, max_depth = 100.f, baseline = 5.4f;
  Resnet18Encoder<T> enc;
  ConvLayer up[10], disp0;
  // buffers
  T* padbuf;                  // reflection-padded conv input scratch
  T *dA, *dB;                 // decoder activations
  float* disp;

  int build(const WeightStore& ws, int feed_h, int feed_w, float mind, float maxd, float base) {
    h = feed_h; w = feed_w; min_depth = mind; max_depth = maxd; baseline = base;
    // >= 64: the decoder reflection-pads the 1/32-resolution map by one pixel, which needs at least two rows and columns
    // (torch.nn.ReflectionPad2d refuses a 1-pixel map the same way)
    DFVO_REQUIRE(h % 32 == 0 && w % 32 == 0 && h >= 64 && w >= 64, DFVO_ESHAPE, "monodepth2 feed size must be a multiple of 32 and at least 64x64 (got %dx%d)", h, w);
    enc.tf32 = tf32;
    TRYM(enc.build_layers(arena, ws, h, w, 3));
    const int encc[5] = {64, 64, 128, 256, 512}, dec[5] = {16, 32, 64, 128, 256};
    int idx = 0;
    for (int i = 4; i >= 0; --i) {
      const int ci0 = (i == 4) ? encc[4] : dec[i + 1];
      char nm[64];
      snprintf(nm, sizeof(nm), "decoder.%d.conv.conv", idx);
      TRYM(plain_conv<T>(arena, tf32, ws, nm, ci0, 0, &up[idx])); ++idx;
      const int ci1 = dec[i] + (i > 0 ? encc[i - 1] : 0);
      snprintf(nm, sizeof(nm), "decoder.%d.conv.conv", idx);
      TRYM(plain_conv<T>(arena, tf32, ws, nm, ci1, 0, &up[idx])); ++idx;
    }
    TRYM(plain_conv<T>(arena, tf32, ws, "decoder.10.conv", 16, 0, &disp0));      // bf16: tensor-core kernel with N padded 1 -> 16
    // ---------------- buffers ----------------
    TRYM(enc.alloc_buffers(arena));
    // largest padded decoder input: i=1 stage (h/2+2)x(w/2+2)x96 vs i=0: (h+2)x(w+2)x16, i=2: (h/4+2)(w/4+2)x128 ...
    size_t pmax = 0;
    for (int i = 4; i >= 0; --i) {
      const int hh = h >> (i + 1), ww = w >> (i + 1);
      const int ci0 = (i == 4) ? encc[4] : dec[i + 1];
      const int ci1 = dec[i] + (i > 0 ? encc[i - 1] : 0);
      size_t a = (size_t)(hh + 2) * (ww + 2) * ci0, b2 = (size_t)(2 * hh + 2) * (2 * ww + 2) * ci1;
      if (a > pmax) pmax = a;
      if (b2 > pmax) pmax = b2;
    }
    { size_t d = (size_t)(h + 2) * (w + 2) * 16; if (d > pmax) pmax = d; }
    ALLOCM(padbuf, T, pmax);
    ALLOCM(dA, T, (size_t)h * w * 16 + (size_t)(h / 2) * (w / 2) * 32); ALLOCM(dB, T, (size_t)h * w * 16 + (size_t)(h / 2) * (w / 2) * 32);
    ALLOCM(disp, float, (size_t)h * w);
    ALLOCM(enc.chain_bars, unsigned, 4 * CHAIN_BAR_WORDS);
    return DFVO_OK;
  }

  int run(const float* img, float* depth_out, cudaStream_t s) override {
    Ten<const T> none; memset(&none, 0, sizeof(none));
    TRYM(enc.run(&img, s));
    // ---------------- decoder (depth_decoder.py:50-65) ----------------
    const int dec[5] = {16, 32, 64, 128, 256};
    T* const* f = enc.f;
    const int *fh = enc.fh, *fw = enc.fw, *fc = enc.fc;
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

// PoseDecoder (pose_decoder.py, num_input_features 1, num_frames_to_predict_for 2): net.0 squeeze 1x1 512 -> 256 + ReLU,
// net.1 / net.2 3x3 (zero pad 1) 256 -> 256 + ReLU, net.3 1x1 256 -> 12; all at 1/32 resolution on the encoder's conv kernels.
// net.3 writes fp32 (N padded 12 -> 16, like the disparity head) and pose_head does the rest of the network in fp32.
template <typename T>
struct PoseImpl : public PoseNetBase {
  Arena arena;
  bool tf32 = false;
  int h = 0, w = 0, hh = 0, ww = 0;
  float baseline = 1.f;
  Resnet18Encoder<T> enc;
  ConvLayer squeeze, pose0, pose1, pose2;
  T *dA, *dB;
  float* out12;               // [hh][ww][16] fp32, channels 0..11 real

  int build(const WeightStore& ws, int feed_h, int feed_w, float base) {
    h = feed_h; w = feed_w; baseline = base;
    DFVO_REQUIRE(h % 32 == 0 && w % 32 == 0 && h >= 64 && w >= 64, DFVO_ESHAPE, "PoseNet feed size must be a multiple of 32 and at least 64x64 (got %dx%d)", h, w);
    enc.tf32 = tf32;
    TRYM(enc.build_layers(arena, ws, h, w, 6));
    TRYM(plain_conv<T>(arena, tf32, ws, "net.0", 512, 0, &squeeze));
    TRYM(plain_conv<T>(arena, tf32, ws, "net.1", 256, 1, &pose0));
    TRYM(plain_conv<T>(arena, tf32, ws, "net.2", 256, 1, &pose1));
    TRYM(plain_conv<T>(arena, tf32, ws, "net.3", 256, 0, &pose2));
    DFVO_REQUIRE(squeeze.Cout == 256 && pose0.Cout == 256 && pose1.Cout == 256 && pose2.Cout == 12 && pose0.kh == 3 && pose1.kh == 3 &&
                 squeeze.kh == 1 && pose2.kh == 1, DFVO_ESTATE, "PoseDecoder weights (net.0 .. net.3) have unexpected shapes");
    TRYM(enc.alloc_buffers(arena));
    hh = enc.fh[4]; ww = enc.fw[4];
    ALLOCM(dA, T, (size_t)hh * ww * 256); ALLOCM(dB, T, (size_t)hh * ww * 256);
    ALLOCM(out12, float, (size_t)hh * ww * 16);
    ALLOCM(enc.chain_bars, unsigned, 4 * CHAIN_BAR_WORDS);
    return DFVO_OK;
  }

  int run(const float* feed_ref, const float* feed_cur, float* pose_out, cudaStream_t s) override {
    Ten<const T> none; memset(&none, 0, sizeof(none));
    const float* imgs[2] = {feed_ref, feed_cur};                  // torch.cat([ref, cur], 1) (deep_models.py:222-226)
    TRYM(enc.run(imgs, s));
    TRYM(run_conv<T>(squeeze, ctv(enc.f[4], hh, ww, 512, 512), tv(dA, hh, ww, 256, 256), ACT_RELU, none, 0, s));
    TRYM(run_conv<T>(pose0, ctv(dA, hh, ww, 256, 256), tv(dB, hh, ww, 256, 256), ACT_RELU, none, 0, s));
    TRYM(run_conv<T>(pose1, ctv(dB, hh, ww, 256, 256), tv(dA, hh, ww, 256, 256), ACT_RELU, none, 0, s));
    Ten<const float> fnone; memset(&fnone, 0, sizeof(fnone));
    TRYM(run_conv_f32out<T>(pose2, ctv(dA, hh, ww, 256, 256), make_ten<float>(out12, 1, hh, ww, 12, 16), ACT_NONE, fnone, s));
    return pose_head(out12, hh, ww, 16, baseline, pose_out, s);
  }
  void geometry(int* ph, int* pw) override { *ph = h; *pw = w; }
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

int posenet_create(const WeightStore& ws, int feed_h, int feed_w, int precision, float baseline_multiplier, PoseNetBase** out) {
  *out = nullptr;
  if (precision == 0 || precision == 2) {
    auto* p = new PoseImpl<float>();
    p->tf32 = precision == 2;
    int rc = p->build(ws, feed_h, feed_w, baseline_multiplier);
    if (rc) { delete p; return rc; }
    *out = p;
  } else {
    auto* p = new PoseImpl<bf16>();
    int rc = p->build(ws, feed_h, feed_w, baseline_multiplier);
    if (rc) { delete p; return rc; }
    *out = p;
  }
  return DFVO_OK;
}

}  // namespace dfvo
