// LiteFlowNet runner interface (implementation: liteflownet.cu).
#pragma once
#include "net_common.h"

namespace dfvo {

struct LiteFlowNetBase {
  virtual ~LiteFlowNetBase() {}
  // imgs_u8: 2*pairs device pointers to HWC uint8 frames ordered [ref0, cur0, ref1, cur1, ...].
  // Outputs (device, may be null): flow_fwd/flow_bwd [pairs][2][H][W], flow_diff [pairs][H][W].
  virtual int run(const uint8_t* const* imgs_u8, float* flow_fwd, float* flow_bwd, float* flow_diff, cudaStream_t s) = 0;
  // run() = ingest (reads the caller's frames) + body (own buffers only: a fixed launch sequence) + emit (writes the
  // caller's outputs)
  virtual int ingest(const uint8_t* const* imgs_u8, cudaStream_t s) = 0;
  virtual int body(cudaStream_t s) = 0;
  virtual int emit(float* flow_fwd, float* flow_bwd, float* flow_diff, cudaStream_t s) = 0;
  virtual int debug_level_flow(int level, int which, float* out_nhwc2) = 0;
  virtual void geometry(int* th, int* tw, int* B) = 0;
  virtual size_t bytes() = 0;
};

void liteflow_target_size(int h, int w, int* th, int* tw);

// precision: 0 = fp32 everywhere (CUDA-core convs), 1 = bf16 activations + wgmma convs
int liteflownet_create(const WeightStore& ws, int H0, int W0, int pairs, int precision, LiteFlowNetBase** out);

}  // namespace dfvo
