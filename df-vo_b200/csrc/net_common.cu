#include "net_common.h"

#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

namespace dfvo {

// ---- error plumbing (thread-local last-error string, SURVEY 8b: never throw across the boundary)
static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* last_error() { return g_err; }
int cuda_fail(cudaError_t e, const char* what, const char* file, int line) {
  set_error("CUDA error %d (%s) at %s:%d: %s", (int)e, cudaGetErrorString(e), file, line, what);
  return DFVO_ECUDA;
}

void* Arena::alloc(size_t bytes) {
  bytes = (bytes + 255) & ~(size_t)255;
  if (bytes == 0) bytes = 256;
  void* p = nullptr;
  if (cudaMalloc(&p, bytes) != cudaSuccess || !p) {
    set_error("cudaMalloc(%zu) failed", bytes);
    return nullptr;
  }
  cudaMemset(p, 0, bytes);
  chunks_.push_back(p);
  total_ += bytes;
  return p;
}
void Arena::release() {
  for (void* p : chunks_) cudaFree(p);
  chunks_.clear();
  total_ = 0;
}

const HostTensor* find_weight(const WeightStore& ws, const std::string& key) {
  auto it = ws.find(key);
  return it == ws.end() ? nullptr : &it->second;
}

// fp32 -> tf32 grid (10-bit mantissa), round to nearest, ties away from zero (= cvt.rna.tf32.f32); the tensor core reads
// the upper 19 bits of an fp32 operand, so pre-rounded weights make its truncation a no-op
static float f2tf32(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  if ((u & 0x7f800000u) == 0x7f800000u) return f;
  u = (u + 0x1000u) & 0xffffe000u;
  memcpy(&f, &u, 4);
  return f;
}

static uint16_t f2bf(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return 0x7fff;
  u += 0x7fffu + ((u >> 16) & 1u);
  return (uint16_t)(u >> 16);
}

int build_conv_layer(Arena& arena, const HostTensor& w, const HostTensor* bias, const std::vector<Seg>& segs,
                     int stride, int pad_y, int pad_x, int reflect, bool want_tc, bool want_direct,
                     const float* scale, const float* shift, ConvLayer* L, int tc_esize) {
  DFVO_REQUIRE(w.shape.size() == 4, DFVO_ESHAPE, "conv weight must be 4-D");
  const int Cout = (int)w.shape[0], Cin = (int)w.shape[1], kh = (int)w.shape[2], kw = (int)w.shape[3];
  int real = 0, ktot = 0;
  for (const Seg& sg : segs) { real += sg.real; ktot += sg.padded; }
  DFVO_REQUIRE(real == Cin, DFVO_ESHAPE, "conv segments cover %d channels, weight has %d", real, Cin);
  L->Cin_ref = Cin; L->Cout = Cout; L->kh = kh; L->kw = kw; L->stride = stride;
  L->pad_y = pad_y; L->pad_x = pad_x; L->reflect = reflect; L->Ktot = ktot;
  L->Cout_pad = (Cout + 15) / 16 * 16;
  L->tc = want_tc;
  L->tc_esize = tc_esize;
  // padded-k -> reference channel (or -1)
  std::vector<int> kmap(ktot, -1);
  {
    int kb = 0, rb = 0;
    for (const Seg& sg : segs) {
      for (int c = 0; c < sg.real; ++c) kmap[kb + c] = rb + c;
      kb += sg.padded; rb += sg.real;
    }
  }
  auto W = [&](int co, int ci, int ky, int kx) {
    float v = w.data[(((size_t)co * Cin + ci) * kh + ky) * kw + kx];
    return scale ? v * scale[co] : v;
  };
  // bias
  {
    std::vector<float> b(L->Cout_pad, 0.f);
    for (int co = 0; co < Cout; ++co) {
      float v = bias ? bias->data[co] : 0.f;
      if (scale) v *= scale[co];
      if (shift) v += shift[co];
      b[co] = v;
    }
    for (int co = 0; co < 4 && co < Cout; ++co) L->bias_h[co] = b[co];
    L->bias = arena.alloc_t<float>(L->Cout_pad);
    if (!L->bias) return DFVO_ENOMEM;
    DFVO_CUDA(cudaMemcpy(L->bias, b.data(), b.size() * 4, cudaMemcpyHostToDevice));
  }
  if (want_direct) {
    L->w_pitch = (Cout + 3) / 4 * 4;
    std::vector<float> h((size_t)kh * kw * ktot * L->w_pitch, 0.f);
    for (int ky = 0; ky < kh; ++ky)
      for (int kx = 0; kx < kw; ++kx)
        for (int k = 0; k < ktot; ++k) {
          if (kmap[k] < 0) continue;
          float* dst = &h[(((size_t)ky * kw + kx) * ktot + k) * L->w_pitch];
          for (int co = 0; co < Cout; ++co) dst[co] = W(co, kmap[k], ky, kx);
        }
    L->w_direct = arena.alloc_t<float>(h.size());
    if (!L->w_direct) return DFVO_ENOMEM;
    DFVO_CUDA(cudaMemcpy(L->w_direct, h.data(), h.size() * 4, cudaMemcpyHostToDevice));
  }
  if (want_tc && Cout == 2 && stride == 1 && kh == kw && ktot == 32) {
    std::vector<float> h((size_t)kh * kw * ktot * 2, 0.f);
    for (int ky = 0; ky < kh; ++ky)
      for (int kx = 0; kx < kw; ++kx)
        for (int k = 0; k < ktot; ++k)
          if (kmap[k] >= 0)
            for (int co = 0; co < 2; ++co) h[((((size_t)ky * kw + kx) * ktot) + k) * 2 + co] = W(co, kmap[k], ky, kx);
    L->w_head = arena.alloc_t<float>(h.size());
    if (!L->w_head) return DFVO_ENOMEM;
    DFVO_CUDA(cudaMemcpy(L->w_head, h.data(), h.size() * 4, cudaMemcpyHostToDevice));
  }
  if (want_tc && tc_esize == 4) {
    DFVO_REQUIRE((stride == 1 || stride == 2) && !reflect && ktot % 16 == 0, DFVO_EINVAL, "tc conv needs stride 1|2, zero pad, K %% 16 == 0");
    std::vector<float> h((size_t)kh * kw * L->Cout_pad * ktot, 0.f);
    for (int ky = 0; ky < kh; ++ky)
      for (int kx = 0; kx < kw; ++kx)
        for (int co = 0; co < Cout; ++co) {
          float* dst = &h[(((size_t)ky * kw + kx) * L->Cout_pad + co) * ktot];
          for (int k = 0; k < ktot; ++k)
            if (kmap[k] >= 0) dst[k] = f2tf32(W(co, kmap[k], ky, kx));
        }
    L->w_tc = arena.alloc(h.size() * 4);
    if (!L->w_tc) return DFVO_ENOMEM;
    DFVO_CUDA(cudaMemcpy(L->w_tc, h.data(), h.size() * 4, cudaMemcpyHostToDevice));
  } else if (want_tc) {
    DFVO_REQUIRE((stride == 1 || stride == 2) && !reflect && ktot % 16 == 0, DFVO_EINVAL, "tc conv needs stride 1|2, zero pad, K %% 16 == 0");
    std::vector<uint16_t> h((size_t)kh * kw * L->Cout_pad * ktot, 0);
    for (int ky = 0; ky < kh; ++ky)
      for (int kx = 0; kx < kw; ++kx)
        for (int co = 0; co < Cout; ++co) {
          uint16_t* dst = &h[(((size_t)ky * kw + kx) * L->Cout_pad + co) * ktot];
          for (int k = 0; k < ktot; ++k)
            if (kmap[k] >= 0) dst[k] = f2bf(W(co, kmap[k], ky, kx));
        }
    L->w_tc = arena.alloc(h.size() * 2);
    if (!L->w_tc) return DFVO_ENOMEM;
    DFVO_CUDA(cudaMemcpy(L->w_tc, h.data(), h.size() * 2, cudaMemcpyHostToDevice));
  }
  return DFVO_OK;
}

static void fill_taps(const ConvLayer& L, ConvTc* c) {
  c->ntaps = L.kh * L.kw;
  for (int ky = 0; ky < L.kh; ++ky)
    for (int kx = 0; kx < L.kw; ++kx) {
      c->dy[ky * L.kw + kx] = (int8_t)(ky - L.pad_y);
      c->dx[ky * L.kw + kx] = (int8_t)(kx - L.pad_x);
    }
}

static ConvDirect to_direct(const ConvLayer& L, int act) {
  ConvDirect d;
  d.Cin = L.Ktot; d.Cout = L.Cout; d.kh = L.kh; d.kw = L.kw; d.stride = L.stride;
  d.pad_y = L.pad_y; d.pad_x = L.pad_x; d.reflect = L.reflect; d.act = act;
  d.w = L.w_direct; d.w_pitch = L.w_pitch; d.bias = L.bias;
  return d;
}

// common description of a tensor-core launch for either operand type
template <typename T, typename TO>
static int launch_tc(const ConvLayer& L, Ten<const T> in, Ten<TO> out, int act, Ten<const TO> residual, int zero_pad_to, int round_out,
                     cudaStream_t s) {
  DFVO_REQUIRE(in.C == L.Ktot, DFVO_ESHAPE, "tc conv: input view has %d channels, layer expects %d", in.C, L.Ktot);
  DFVO_REQUIRE((int)sizeof(T) == L.tc_esize, DFVO_ESTATE, "tc conv: layer packed for %d-byte operands, input has %d", L.tc_esize, (int)sizeof(T));
  ConvTc c;
  memset(&c, 0, sizeof(c));
  c.N = in.N; c.H = out.H; c.W = out.W; c.inH = in.H; c.inW = in.W; c.stride = L.stride;
  if (L.stride == 2) {
    DFVO_REQUIRE(in.H == 2 * out.H && in.W == 2 * out.W, DFVO_ESHAPE, "tc conv stride 2: in %dx%d out %dx%d", in.H, in.W, out.H, out.W);
  } else {
    DFVO_REQUIRE(in.H == out.H + L.kh - 1 - 2 * L.pad_y && in.W == out.W + L.kw - 1 - 2 * L.pad_x, DFVO_ESHAPE,
                 "tc conv: in %dx%d out %dx%d k %dx%d pad %d,%d", in.H, in.W, out.H, out.W, L.kh, L.kw, L.pad_y, L.pad_x);
  }
  c.nsrc = 1;
  c.src[0].p = in.p; c.src[0].C = in.C; c.src[0].sN = in.sN; c.src[0].sH = in.sH; c.src[0].sW = in.sW;
  fill_taps(L, &c);
  c.esize = L.tc_esize; c.round_out_tf32 = round_out;
  c.w = L.w_tc; c.Cout_pad = L.Cout_pad; c.Cout = L.Cout; c.bias = L.bias; c.act = act; c.out_f32 = sizeof(TO) == 4;
  c.out = out.p; c.oN = out.sN; c.oH = out.sH; c.oW = out.sW;
  c.residual = residual.p; c.rN = residual.sN; c.rH = residual.sH; c.rW = residual.sW;
  c.zero_pad_to = zero_pad_to;
  c.flops = 2.0 * (double)in.N * out.H * out.W * (double)L.Cout * L.Cin_ref * L.kh * L.kw;
  return conv_tc(c, s);
}

template <typename T>
int run_conv_multi(const ConvLayer& L, const Ten<const T>* ins, int nin, Ten<T> out, int act, double flops, cudaStream_t s) {
  DFVO_REQUIRE(L.tc && nin >= 1 && nin <= 3 && L.stride == 1 && (int)sizeof(T) == L.tc_esize, DFVO_ESTATE, "run_conv_multi: tensor-core stride-1 layers only");
  ConvTc c;
  memset(&c, 0, sizeof(c));
  int ktot = 0;
  for (int i = 0; i < nin; ++i) {
    DFVO_REQUIRE(ins[i].N == ins[0].N && ins[i].H == ins[0].H && ins[i].W == ins[0].W, DFVO_ESHAPE, "run_conv_multi: source %d shape", i);
    c.src[i].p = ins[i].p; c.src[i].C = ins[i].C; c.src[i].sN = ins[i].sN; c.src[i].sH = ins[i].sH; c.src[i].sW = ins[i].sW;
    ktot += ins[i].C;
  }
  DFVO_REQUIRE(ktot == L.Ktot, DFVO_ESHAPE, "run_conv_multi: sources carry %d channels, layer expects %d", ktot, L.Ktot);
  c.N = ins[0].N; c.H = out.H; c.W = out.W; c.inH = ins[0].H; c.inW = ins[0].W; c.stride = 1; c.nsrc = nin;
  fill_taps(L, &c);
  c.esize = L.tc_esize; c.round_out_tf32 = sizeof(T) == 4;
  c.w = L.w_tc; c.Cout_pad = L.Cout_pad; c.Cout = L.Cout; c.bias = L.bias; c.act = act; c.out_f32 = sizeof(T) == 4;
  c.out = out.p; c.oN = out.sN; c.oH = out.sH; c.oW = out.sW;
  c.flops = flops > 0 ? flops : 2.0 * (double)c.N * out.H * out.W * (double)L.Cout * L.Cin_ref * L.kh * L.kw;
  return conv_tc(c, s);
}
template int run_conv_multi<bf16>(const ConvLayer&, const Ten<const bf16>*, int, Ten<bf16>, int, double, cudaStream_t);
template int run_conv_multi<float>(const ConvLayer&, const Ten<const float>*, int, Ten<float>, int, double, cudaStream_t);

template <>
int run_conv<float>(const ConvLayer& L, Ten<const float> in, Ten<float> out, int act, Ten<const float> residual,
                    int zero_pad_to, cudaStream_t s) {
  // tf32 mode: fp32 activations, wgmma tf32; stored activations are rounded to tf32 (the next conv's operand)
  if (L.tc && L.tc_esize == 4) return launch_tc<float, float>(L, in, out, act, residual, zero_pad_to, 1, s);
  DFVO_REQUIRE(L.w_direct, DFVO_ESTATE, "conv layer has no fp32 weights");
  // pad channels of fp32 buffers are zero from allocation and never written; nothing to do for zero_pad_to
  (void)zero_pad_to;
  return conv_direct<float, float>(to_direct(L, act), in, out, residual, s);
}

template <>
int run_conv<bf16>(const ConvLayer& L, Ten<const bf16> in, Ten<bf16> out, int act, Ten<const bf16> residual,
                   int zero_pad_to, cudaStream_t s) {
  if (!L.tc) {
    DFVO_REQUIRE(L.w_direct, DFVO_ESTATE, "conv layer has no direct weights");
    return conv_direct<bf16, bf16>(to_direct(L, act), in, out, residual, s);
  }
  return launch_tc<bf16, bf16>(L, in, out, act, residual, zero_pad_to, 0, s);
}

template <>
int run_conv_f32out<float>(const ConvLayer& L, Ten<const float> in, Ten<float> out, int act,
                           Ten<const float> residual, cudaStream_t s) {
  return conv_direct<float, float>(to_direct(L, act), in, out, residual, s);
}

template <>
int run_conv_f32out<bf16>(const ConvLayer& L, Ten<const bf16> in, Ten<float> out, int act, Ten<const float> residual,
                          cudaStream_t s) {
  if (!L.tc) return conv_direct<bf16, float>(to_direct(L, act), in, out, residual, s);
  // 2-channel flow heads: dedicated CUDA-core kernel; the tensor-core kernel (N padded to 16) serves the other
  // float-output layers (monodepth2's disparity head)
  // (49 taps of N = 16 MMAs are issue / barrier bound, so the tensor-core route is opt-in: DFVO_HEAD_TC=1)
  static int head_tc = -1;
  if (head_tc < 0) { const char* e = getenv("DFVO_HEAD_TC"); head_tc = (e && atoi(e) == 1); }
  const bool big = (long long)in.N * in.H * in.W >= 100000;
  if (L.w_head && !(head_tc && big) && act == ACT_NONE && in.C == 32 && (L.kh == 3 || L.kh == 5 || L.kh == 7) &&
      L.pad_y == L.kh / 2 && L.pad_x == L.kw / 2)
    return flow_head(in, L.w_head, L.bias_h[0], L.bias_h[1], L.kh, residual, out, s);
  return launch_tc<bf16, float>(L, in, out, act, residual, 0, 0, s);
}

}  // namespace dfvo
