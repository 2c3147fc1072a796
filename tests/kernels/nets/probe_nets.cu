// TEST INFRASTRUCTURE ONLY: extern "C" entry points that run the monodepth2 depth runner and the PoseNet runner (monodepth2.h)
// eagerly with a per-layer tap (net_common.h::LayerTap) installed, so the test suite can check each layer of the product plan on its
// own.  Built twice by tests/kernels/nets/build.py: with nvcc against the product libdfvo_b200.so, and with g++ -DDFVO_HOSTSIM
// against the CPU emulation library.  Never loaded by the product.
#include <stdio.h>
#include <string.h>

#include <string>
#include <vector>

#include "monodepth2.h"
#include "net_common.h"

// Every tapped view is copied, right after the launch that wrote it, into host storage owned here: the span
// (N-1) sN + (H-1) sH + (W-1) sW + C elements from the view's first element.  The records live until the next run.
namespace {
struct TapRecord {
  std::string name;
  int esize, N, H, W, C;
  long long sN, sH, sW;
  std::vector<char> bytes;
};
std::vector<TapRecord> g_taps;
int g_tap_rc = 0;

void tap_copy(void*, const char* name, int esize, const void* p, int N, int H, int W, int C, long long sN, long long sH, long long sW,
              cudaStream_t s) {
  TapRecord r;
  r.name = name; r.esize = esize; r.N = N; r.H = H; r.W = W; r.C = C; r.sN = sN; r.sH = sH; r.sW = sW;
  const long long span = (long long)(N - 1) * sN + (long long)(H - 1) * sH + (long long)(W - 1) * sW + C;
  r.bytes.resize((size_t)span * esize);
  cudaError_t e = cudaStreamSynchronize(s);
  if (e == cudaSuccess) e = cudaMemcpy(r.bytes.data(), p, r.bytes.size(), cudaMemcpyDeviceToHost);
  if (e != cudaSuccess && !g_tap_rc) g_tap_rc = dfvo::cuda_fail(e, name, __FILE__, __LINE__);
  g_taps.push_back(std::move(r));
}

// nw (key, ndim, shape, fp32 host data) triples -> a probe-owned WeightStore
dfvo::WeightStore weight_store(int nw, const char* const* keys, const int* ndims, const long long* shapes, const float* const* data) {
  dfvo::WeightStore ws;
  for (int i = 0, o = 0; i < nw; o += ndims[i], ++i) {
    dfvo::HostTensor& t = ws[keys[i]];
    size_t n = 1;
    for (int d = 0; d < ndims[i]; ++d) { t.shape.push_back(shapes[o + d]); n *= (size_t)shapes[o + d]; }
    t.data.assign(data[i], data[i] + n);
  }
  return ws;
}

template <typename Net>
int run_tapped(Net* net, int rc, int tap, const float* const* feeds, int batch, float* out, cudaStream_t s) {
  g_taps.clear();
  g_tap_rc = 0;
  if (rc) return rc;
  if (tap) {
    dfvo::LayerTap t;
    t.fn = tap_copy;
    net->set_tap(t);
  }
  rc = net->run_batch(feeds, batch, out, s);
  if (!rc) rc = g_tap_rc;
  cudaStreamSynchronize(s);
  delete net;
  return rc;
}
}  // namespace

extern "C" {

int nets_is_device_build(void) {
#ifdef DFVO_HOSTSIM
  return 0;
#else
  return 1;
#endif
}

const char* dfvo_last_error(void);          // the library's C ABI (include/dfvo_b200.h)
const char* nets_last_error(void) { return dfvo_last_error(); }

// monodepth2_create + one eager run_batch on stream s; tap != 0 records every layer (nets_tap_*)
int nets_monodepth2_run(int nw, const char* const* keys, const int* ndims, const long long* shapes, const float* const* data, int feed_h,
                         int feed_w, int batch, int precision, float min_depth, float max_depth, float baseline, const float* const* feeds,
                         float* depth_out, int tap, void* s) {
  dfvo::Monodepth2Base* net = nullptr;
  const int rc = dfvo::monodepth2_create(weight_store(nw, keys, ndims, shapes, data), feed_h, feed_w, batch, precision, min_depth, max_depth,
                                         baseline, &net);
  return run_tapped(net, rc, tap, feeds, batch, depth_out, reinterpret_cast<cudaStream_t>(s));
}

// posenet_create + one eager run_batch (feeds: 2 * batch pointers [ref0, cur0, ref1, cur1, ...])
int nets_posenet_run(int nw, const char* const* keys, const int* ndims, const long long* shapes, const float* const* data, int feed_h,
                      int feed_w, int batch, int precision, float baseline_multiplier, const float* const* feeds, float* pose_out, int tap,
                      void* s) {
  dfvo::PoseNetBase* net = nullptr;
  const int rc = dfvo::posenet_create(weight_store(nw, keys, ndims, shapes, data), feed_h, feed_w, batch, precision, baseline_multiplier, &net);
  return run_tapped(net, rc, tap, feeds, batch, pose_out, reinterpret_cast<cudaStream_t>(s));
}

int nets_tap_count(void) { return (int)g_taps.size(); }

// name (NUL-terminated, at most name_len bytes), element size, dims {N, H, W, C}, strides {sN, sH, sW}, span in elements
int nets_tap_info(int i, char* name, int name_len, int* esize, int* dims, long long* strides, long long* span) {
  if (i < 0 || i >= (int)g_taps.size() || name_len < 1) return DFVO_EINVAL;
  const TapRecord& r = g_taps[i];
  snprintf(name, name_len, "%s", r.name.c_str());
  *esize = r.esize;
  dims[0] = r.N; dims[1] = r.H; dims[2] = r.W; dims[3] = r.C;
  strides[0] = r.sN; strides[1] = r.sH; strides[2] = r.sW;
  *span = (long long)r.bytes.size() / r.esize;
  return 0;
}

// the record's span (nets_tap_info) into host memory dst
int nets_tap_copy(int i, void* dst) {
  if (i < 0 || i >= (int)g_taps.size()) return DFVO_EINVAL;
  memcpy(dst, g_taps[i].bytes.data(), g_taps[i].bytes.size());
  return 0;
}

}  // extern "C"
