// monodepth2 depth runner (ResNet-18 encoder + skip decoder) and PoseNet runner (the same encoder with a 6-channel stem +
// PoseDecoder) (implementation: monodepth2.cu).
#pragma once
#include "net_common.h"

namespace dfvo {

struct Monodepth2Base {
  virtual ~Monodepth2Base() {}
  // img: float NCHW [1,3,h,w] in [0,1] (the LANCZOS-resized feed image, deep_models.py:195-201);
  // depth_out: [h,w] fp32 = Monodepth2DepthNet.inference_depth (monodepth2.py:121-139)
  virtual int run(const float* img_nchw, float* depth_out, cudaStream_t s) = 0;
  virtual void geometry(int* h, int* w) = 0;
  virtual size_t bytes() = 0;
};

int monodepth2_create(const WeightStore& ws, int feed_h, int feed_w, int precision, float min_depth, float max_depth,
                      float baseline, Monodepth2Base** out);

struct PoseNetBase {
  virtual ~PoseNetBase() {}
  // feed_ref / feed_cur: float NCHW [1,3,h,w] in [0,1] (the depth network's feeds, deep_models.py:218-226);
  // pose_out: device fp32 4x4 row-major = Monodepth2PoseNet.inference_pose([ref, cur])[0] (pose/monodepth2/monodepth2.py:102-119)
  virtual int run(const float* feed_ref, const float* feed_cur, float* pose_out, cudaStream_t s) = 0;
  virtual void geometry(int* h, int* w) = 0;
  virtual size_t bytes() = 0;
};

int posenet_create(const WeightStore& ws, int feed_h, int feed_w, int precision, float baseline_multiplier, PoseNetBase** out);

}  // namespace dfvo
