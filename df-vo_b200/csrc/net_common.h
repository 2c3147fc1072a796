// Host-side plumbing shared by the two network runners: weight store (reference state-dict key
// -> fp32 host array), device arena, conv-layer packing for the two conv backends.
#pragma once
#include <stdarg.h>

#include <map>
#include <string>
#include <vector>

#include "ops.h"

namespace dfvo {

// Per-layer observation hook of the network runners: called right after a runner has enqueued the launch that produces a tensor,
// with the view that launch wrote (esize: 2 = bf16, 4 = fp32 elements) and a stable name that maps to the reference state-dict
// keys.  The callee may synchronise `s` and read the view; the next launch overwrites reused scratch.  Unset (fn == nullptr) it
// costs one host-side pointer test per layer and changes no launch.
struct LayerTap {
  void (*fn)(void* user, const char* name, int esize, const void* p, int N, int H, int W, int C, long long sN, long long sH, long long sW,
             cudaStream_t s) = nullptr;
  void* user = nullptr;

  template <typename T>
  void operator()(cudaStream_t s, const Ten<T>& v, const char* fmt, ...) const {
    if (!fn) return;
    char name[64];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(name, sizeof(name), fmt, ap);
    va_end(ap);
    fn(user, name, (int)sizeof(T), (const void*)v.p, v.N, v.H, v.W, v.C, v.sN, v.sH, v.sW, s);
  }
};

struct HostTensor {
  std::vector<int64_t> shape;
  std::vector<float> data;
};
typedef std::map<std::string, HostTensor> WeightStore;

// Simple bump allocator over cudaMalloc'd chunks; everything is freed with the owner.
class Arena {
 public:
  ~Arena() { release(); }
  void* alloc(size_t bytes);                 // 256-byte aligned, zero-initialised; nullptr on failure
  template <typename T> T* alloc_t(size_t n) { return reinterpret_cast<T*>(alloc(n * sizeof(T))); }
  void release();
  size_t total() const { return total_; }

 private:
  std::vector<void*> chunks_;
  size_t total_ = 0;
};

// One input segment of a (possibly concatenated) conv input: `real` reference channels stored in a
// slot of `padded` channels (padded % 16 == 0); pad channels carry zero weights.
struct Seg { int real, padded; };

struct ConvLayer {
  int Cin_ref = 0, Cout = 0, kh = 0, kw = 0, stride = 1, pad_y = 0, pad_x = 0, reflect = 0;
  int Ktot = 0;            // sum of padded segment sizes == channel count of the input view
  int Cout_pad = 0;        // multiple of 16
  float* w_direct = nullptr;   // device [kh*kw*Ktot][w_pitch] fp32
  int w_pitch = 0;
  void* w_tc = nullptr;        // device [kh*kw][Cout_pad][Ktot] bf16 (tc_esize 2) or tf32-rounded float (tc_esize 4), if tc requested
  int tc_esize = 2;
  float* w_head = nullptr;     // device [kh*kw][Ktot][2] fp32, only for 2-channel heads (flow_head kernel)
  float* bias = nullptr;       // device [Cout_pad] fp32 (zero padded; zeros if the conv has no bias)
  float bias_h[4] = {0.f, 0.f, 0.f, 0.f};   // host copy of the first biases (kernel arguments of the head kernel)
  bool tc = false;
};

// Build a layer from reference tensors `w` [Cout][Cin_ref][kh][kw] (+ optional bias [Cout]).
// `scale`/`shift` (optional, per Cout) fold an eval-mode BatchNorm: y = conv*scale + shift.
int build_conv_layer(Arena& arena, const HostTensor& w, const HostTensor* bias, const std::vector<Seg>& segs,
                     int stride, int pad_y, int pad_x, int reflect, bool want_tc, bool want_direct,
                     const float* scale, const float* shift, ConvLayer* out, int tc_esize = 2);

template <typename T>
int run_conv(const ConvLayer& L, Ten<const T> in, Ten<T> out, int act, Ten<const T> residual, int zero_pad_to,
             cudaStream_t s);
// the same over nin <= 3 virtual-concat sources (views of equal N, H, W; channels in the layer's segment order); the input views may
// be smaller / larger than "same" padding implies (asymmetric windows): anything outside them reads as zero.  flops: algorithmic
// FLOPs of the launch for the roofline report (0 = derive from the layer).  Tensor-core layers only.
template <typename T>
int run_conv_multi(const ConvLayer& L, const Ten<const T>* ins, int nin, Ten<T> out, int act, double flops, cudaStream_t s);
// flow head: T input, float output (+ float residual)
template <typename T>
int run_conv_f32out(const ConvLayer& L, Ten<const T> in, Ten<float> out, int act, Ten<const float> residual,
                    cudaStream_t s);

const HostTensor* find_weight(const WeightStore& ws, const std::string& key);

// RAII scope of a layer chain (ops.h::conv_chain_begin): the run_conv calls inside are issued as one launch at end() / scope exit.
struct ChainScope {
  bool open;
  ChainScope(cudaStream_t s, unsigned* bar) : open(bar != nullptr) { if (open) conv_chain_begin(s, bar); }
  int end() { if (!open) return DFVO_OK; open = false; return conv_chain_end(); }
  ~ChainScope() { if (open) conv_chain_end(); }
};

}  // namespace dfvo
