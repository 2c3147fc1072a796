// TEST INFRASTRUCTURE ONLY: extern "C" entry points that call the library's internal dfvo:: launchers directly, so the test suite
// can drive each kernel with views, strides and descriptor features the product C ABI (include/dfvo_b200.h) never exposes.
// Built twice by tests/kernels/build.py: with nvcc against the product libdfvo_b200.so, and with g++ -DDFVO_HOSTSIM against the
// CPU emulation library.  Never loaded by the product.
//
// Every tensor crosses the boundary as a ProbeTen: a raw pointer (device memory, or host memory in the emulation build) and an
// NHWC view with element strides.  ProbeConv is a flat mirror of dfvo::ConvTc, copied field by field, so a layout change of
// ConvTc breaks this file's compile instead of silently shifting what the tests set.
#include <string.h>

#include <vector>

#include "net_common.h"
#include "ops.h"

using dfvo::bf16;
using dfvo::Ten;

extern "C" {

struct ProbeTen {
  void* p;
  int N, H, W, C;
  long long sN, sH, sW;
};

struct ProbeConv {
  int N, H, W, inH, inW;
  int nsrc;
  ProbeTen src[3];           // p, C, sN, sH, sW
  int stride, ntaps;
  int dy[49], dx[49];
  int esize, round_out_tf32;
  const void* w;
  int Cout_pad, Cout;
  const float* bias;
  int act, out_f32;
  ProbeTen out;              // p, sN, sH, sW
  ProbeTen residual;         // p (nullptr: none), sN, sH, sW
  int zero_pad_to;
};

}  // extern "C"

template <typename T>
static Ten<T> ten(const ProbeTen* t) {
  Ten<T> r;
  memset(&r, 0, sizeof(r));
  if (!t) return r;
  r.p = reinterpret_cast<T*>(t->p);
  r.N = t->N; r.H = t->H; r.W = t->W; r.C = t->C;
  r.sN = t->sN; r.sH = t->sH; r.sW = t->sW;
  return r;
}

static dfvo::ConvTc to_conv(const ProbeConv& d) {
  dfvo::ConvTc c;
  memset(&c, 0, sizeof(c));
  c.N = d.N; c.H = d.H; c.W = d.W; c.inH = d.inH; c.inW = d.inW;
  c.nsrc = d.nsrc;
  for (int i = 0; i < 3; ++i) {
    c.src[i].p = d.src[i].p; c.src[i].C = d.src[i].C;
    c.src[i].sN = d.src[i].sN; c.src[i].sH = d.src[i].sH; c.src[i].sW = d.src[i].sW;
  }
  c.stride = d.stride; c.ntaps = d.ntaps;
  for (int t = 0; t < 49; ++t) { c.dy[t] = (int8_t)d.dy[t]; c.dx[t] = (int8_t)d.dx[t]; }
  c.esize = d.esize; c.round_out_tf32 = d.round_out_tf32;
  c.w = d.w; c.Cout_pad = d.Cout_pad; c.Cout = d.Cout; c.bias = d.bias; c.act = d.act; c.out_f32 = d.out_f32;
  c.out = d.out.p; c.oN = d.out.sN; c.oH = d.out.sH; c.oW = d.out.sW;
  c.residual = d.residual.p; c.rN = d.residual.sN; c.rH = d.residual.sH; c.rW = d.residual.sW;
  c.zero_pad_to = d.zero_pad_to;
  c.flops = 2.0 * d.N * d.H * d.W * (double)d.Cout * d.ntaps * (d.src[0].C + (d.nsrc > 1 ? d.src[1].C : 0) + (d.nsrc > 2 ? d.src[2].C : 0));
  return c;
}

static cudaStream_t strm(void* s) { return reinterpret_cast<cudaStream_t>(s); }

extern "C" {

int probe_is_device_build(void) {
#ifdef DFVO_HOSTSIM
  return 0;
#else
  return 1;
#endif
}

const char* dfvo_last_error(void);          // the library's C ABI (include/dfvo_b200.h)
const char* probe_last_error(void) { return dfvo_last_error(); }

int probe_struct_sizes(int* ten, int* conv) {
  *ten = (int)sizeof(ProbeTen);
  *conv = (int)sizeof(ProbeConv);
  return 0;
}

// ---- convolutions ------------------------------------------------------------------------------------------------
int probe_conv_tc(const ProbeConv* d, void* s) { return dfvo::conv_tc(to_conv(*d), strm(s)); }

// the descriptors issued one after the other inside one conv_chain scope with chains enabled (bar: CHAIN_BAR_WORDS zeroed words)
int probe_conv_chain(const ProbeConv* ds, int n, unsigned* bar, void* s) {
  const int prev = dfvo::conv_chain_set_enabled(1);
  dfvo::conv_chain_begin(strm(s), bar);
  int rc = 0;
  for (int i = 0; i < n && rc == 0; ++i) rc = dfvo::conv_tc(to_conv(ds[i]), strm(s));
  const int rc2 = dfvo::conv_chain_end();
  dfvo::conv_chain_set_enabled(prev);
  return rc ? rc : rc2;
}

// build_conv_layer (reference weight [Cout][Cin][kh][kw] on the host, Seg list as (real, padded) pairs, optional BN scale / shift)
// and run it: mode 0 = run_conv_multi over `nin` sources, mode 1 = run_conv (one source, residual, zero_pad_to).
// esize 2: bf16 views, 4: fp32 views (tf32 tensor-core layer).
int probe_conv_layer(const float* w, int Cout, int Cin, int kh, int kw, const float* bias, const int* segs, int nseg, int pad_y,
                     int pad_x, const float* scale, const float* shift, int esize, int mode, const ProbeTen* ins, int nin,
                     const ProbeTen* out, int act, const ProbeTen* residual, int zero_pad_to, void* s) {
  dfvo::Arena arena;
  dfvo::HostTensor hw;
  hw.shape = {Cout, Cin, kh, kw};
  hw.data.assign(w, w + (size_t)Cout * Cin * kh * kw);
  dfvo::HostTensor hb;
  if (bias) { hb.shape = {Cout}; hb.data.assign(bias, bias + Cout); }
  std::vector<dfvo::Seg> sg;
  for (int i = 0; i < nseg; ++i) sg.push_back({segs[2 * i], segs[2 * i + 1]});
  dfvo::ConvLayer L;
  int rc = dfvo::build_conv_layer(arena, hw, bias ? &hb : nullptr, sg, 1, pad_y, pad_x, 0, true, false, scale, shift, &L, esize);
  if (rc) return rc;
  if (esize == 2) {
    if (mode == 0) {
      Ten<const bf16> v[3];
      for (int i = 0; i < nin && i < 3; ++i) v[i] = dfvo::cten(ten<bf16>(&ins[i]));
      rc = dfvo::run_conv_multi<bf16>(L, v, nin, ten<bf16>(out), act, 0.0, strm(s));
    } else {
      rc = dfvo::run_conv<bf16>(L, dfvo::cten(ten<bf16>(&ins[0])), ten<bf16>(out), act, dfvo::cten(ten<bf16>(residual)), zero_pad_to, strm(s));
    }
  } else {
    if (mode == 0) {
      Ten<const float> v[3];
      for (int i = 0; i < nin && i < 3; ++i) v[i] = dfvo::cten(ten<float>(&ins[i]));
      rc = dfvo::run_conv_multi<float>(L, v, nin, ten<float>(out), act, 0.0, strm(s));
    } else {
      rc = dfvo::run_conv<float>(L, dfvo::cten(ten<float>(&ins[0])), ten<float>(out), act, dfvo::cten(ten<float>(residual)), zero_pad_to, strm(s));
    }
  }
  // the arena's weights must outlive the launch
  cudaStreamSynchronize(strm(s));
  return rc;
}

// ---- LiteFlowNet flow kernels ---------------------------------------------------------------------------------------
int probe_correlation49_warped(int bf, const ProbeTen* first, const ProbeTen* feat2, int nxor, const ProbeTen* flow, float scale,
                               int stride, int leaky, const ProbeTen* scratch, const ProbeTen* out, void* s) {
  if (bf)
    return dfvo::correlation49_warped<bf16>(dfvo::cten(ten<bf16>(first)), dfvo::cten(ten<bf16>(feat2)), nxor, dfvo::cten(ten<float>(flow)),
                                            scale, stride, leaky, ten<bf16>(scratch), ten<bf16>(out), strm(s));
  return dfvo::correlation49_warped<float>(dfvo::cten(ten<float>(first)), dfvo::cten(ten<float>(feat2)), nxor, dfvo::cten(ten<float>(flow)),
                                           scale, stride, leaky, ten<float>(scratch), ten<float>(out), strm(s));
}

int probe_warp_bilinear(int bf, const ProbeTen* in, const ProbeTen* flow, float scale, int nxor, const ProbeTen* out, void* s) {
  if (bf) return dfvo::warp_bilinear<bf16>(dfvo::cten(ten<bf16>(in)), dfvo::cten(ten<float>(flow)), scale, nxor, ten<bf16>(out), strm(s));
  return dfvo::warp_bilinear<float>(dfvo::cten(ten<float>(in)), dfvo::cten(ten<float>(flow)), scale, nxor, ten<float>(out), strm(s));
}

int probe_deconv4x4s2_dw(int bf, const ProbeTen* in, const float* w, const ProbeTen* out, void* s) {
  if (bf) return dfvo::deconv4x4s2_dw<bf16>(dfvo::cten(ten<bf16>(in)), w, ten<bf16>(out), strm(s));
  return dfvo::deconv4x4s2_dw<float>(dfvo::cten(ten<float>(in)), w, ten<float>(out), strm(s));
}

int probe_flow_head(const ProbeTen* in, const float* w, float b0, float b1, int k, const ProbeTen* residual, const ProbeTen* out, void* s) {
  return dfvo::flow_head(dfvo::cten(ten<bf16>(in)), w, b0, b1, k, dfvo::cten(ten<float>(residual)), ten<float>(out), strm(s));
}

int probe_flow_mean(const ProbeTen* flow, float* mean, void* s) { return dfvo::flow_mean(dfvo::cten(ten<float>(flow)), mean, strm(s)); }

long long probe_flow_mean_buffer_floats(int N) { return (long long)dfvo::flow_mean_buffer_floats(N); }

int probe_reg_prep(int bf, const ProbeTen* img1, const ProbeTen* img2, int nxor, const ProbeTen* flow, const float* mean, float scale,
                   const ProbeTen* out, void* s) {
  if (bf)
    return dfvo::reg_prep<bf16>(dfvo::cten(ten<float>(img1)), dfvo::cten(ten<float>(img2)), nxor, dfvo::cten(ten<float>(flow)), mean, scale,
                                ten<bf16>(out), strm(s));
  return dfvo::reg_prep<float>(dfvo::cten(ten<float>(img1)), dfvo::cten(ten<float>(img2)), nxor, dfvo::cten(ten<float>(flow)), mean, scale,
                               ten<float>(out), strm(s));
}

int probe_reg_tail(int bf, const ProbeTen* dist, const ProbeTen* flow, int k, const float* wx, const float* wy, float bx, float by,
                   const ProbeTen* out, void* s) {
  if (bf)
    return dfvo::reg_tail<bf16>(dfvo::cten(ten<bf16>(dist)), dfvo::cten(ten<float>(flow)), k, wx, wy, bx, by, ten<float>(out), strm(s));
  return dfvo::reg_tail<float>(dfvo::cten(ten<float>(dist)), dfvo::cten(ten<float>(flow)), k, wx, wy, bx, by, ten<float>(out), strm(s));
}

int probe_flow_upsample_final(const ProbeTen* flow, float mul, int H, int W, float* out, void* s) {
  return dfvo::flow_upsample_final(dfvo::cten(ten<float>(flow)), mul, H, W, out, strm(s));
}

// ---- monodepth2 helpers ---------------------------------------------------------------------------------------------
int probe_maxpool3x3s2(const ProbeTen* in, const ProbeTen* out, void* s) {
  return dfvo::maxpool3x3s2<bf16>(dfvo::cten(ten<bf16>(in)), ten<bf16>(out), strm(s));
}

int probe_upcat_reflect(const ProbeTen* lo, int up, const ProbeTen* skip, const ProbeTen* out, void* s) {
  return dfvo::upcat_reflect<bf16>(dfvo::cten(ten<bf16>(lo)), up, dfvo::cten(ten<bf16>(skip)), ten<bf16>(out), strm(s));
}

}  // extern "C"
