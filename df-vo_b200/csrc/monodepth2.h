// monodepth2 depth runner (ResNet-18 encoder + skip decoder) and PoseNet runner (the same encoder with a 6-channel stem +
// PoseDecoder) (implementation: monodepth2.cu).  Both are built for a batch of B images: every layer runs once over N = B.
#pragma once
#include "net_common.h"

namespace dfvo {

struct Monodepth2Base {
  virtual ~Monodepth2Base() {}
  // imgs: n == batch() device pointers to float NCHW [1,3,h,w] feeds in [0,1] (the LANCZOS-resized feed images,
  // deep_models.py:195-201); depth_out: [n][h][w] fp32 = Monodepth2DepthNet.inference_depth (monodepth2.py:121-139) per image
  virtual int run_batch(const float* const* imgs, int n, float* depth_out, cudaStream_t s) = 0;
  int run(const float* img_nchw, float* depth_out, cudaStream_t s) { return run_batch(&img_nchw, 1, depth_out, s); }
  // per-layer hook (net_common.h::LayerTap) of the following run_batch calls: x0 | imgpad, enc.stem, enc.pool,
  // enc.layer{1..4}.{0,1}.{conv1,down,out}, dec.{0..10}.pad, dec.{0..9}.conv, disp, depth
  virtual void set_tap(LayerTap t) = 0;
  virtual void geometry(int* h, int* w) = 0;
  virtual int batch() = 0;
  virtual size_t bytes() = 0;
};

int monodepth2_create(const WeightStore& ws, int feed_h, int feed_w, int batch, int precision, float min_depth, float max_depth,
                      float baseline, Monodepth2Base** out);

struct PoseNetBase {
  virtual ~PoseNetBase() {}
  // feeds: 2n device pointers [ref0, cur0, ref1, cur1, ...] to float NCHW [1,3,h,w] feeds in [0,1] (the depth network's feeds,
  // deep_models.py:218-226), n == batch(); pose_out: device fp32 [n][4][4] row-major, entry i =
  // Monodepth2PoseNet.inference_pose([ref_i, cur_i])[0] (pose/monodepth2/monodepth2.py:102-119)
  virtual int run_batch(const float* const* feeds, int n, float* pose_out, cudaStream_t s) = 0;
  int run(const float* feed_ref, const float* feed_cur, float* pose_out, cudaStream_t s) {
    const float* feeds[2] = {feed_ref, feed_cur};
    return run_batch(feeds, 1, pose_out, s);
  }
  // per-layer hook of the following run_batch calls: the encoder's taps (Monodepth2Base::set_tap), pose.net0 .. pose.net2,
  // pose.out12, pose
  virtual void set_tap(LayerTap t) = 0;
  virtual void geometry(int* h, int* w) = 0;
  virtual int batch() = 0;
  virtual size_t bytes() = 0;
};

int posenet_create(const WeightStore& ws, int feed_h, int feed_w, int batch, int precision, float baseline_multiplier, PoseNetBase** out);

}  // namespace dfvo
