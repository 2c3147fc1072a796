"""``DeepModel`` facade with the reference's interface (libs/deep_models/deep_models.py:25-350), backed by
the dfvo_b200 CUDA library: LiteFlowNet forward+backward flow with the forward-backward consistency map,
monodepth2 single-view depth and the monodepth2 PoseNet (deep_pose).  Inference only -- the online-finetuning half of the
reference class (``setup_train``, ``finetune``, ``save_model``) is outside the hot path (SURVEY.md section 2, rows 1/6) and
raises ``NotImplementedError``.
"""
import os

import numpy as np

from b200 import native, runtime, tracking


def _load_state_dict(path):
    """Checkpoint IO (torch.load, lite_flow.py:45 / monodepth2.py:47-55) -> {key: float32 ndarray}."""
    import torch
    sd = torch.load(path, map_location="cpu", weights_only=False)
    out = {}
    for k, v in sd.items():
        out[k] = v.detach().float().numpy() if hasattr(v, "detach") else v
    return out


def _same_image(a, b):
    a = np.asarray(a)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a, b)


class _FlowHandle:
    """What the driver / tools read on ``deep_models.flow`` (SURVEY 8b 'attributes read on sub-objects')."""
    flow_scales = [1]
    enable_finetune = False
    half_flow = False


class _DepthHandle:
    enable_finetune = False
    depth_scales = [0]


class DeepModel:
    def __init__(self, cfg):
        self.cfg = cfg
        self.finetune_cfg = cfg.online_finetune
        self.precision = native.PREC_NAMES[os.environ.get("DFVO_B200_PRECISION", "bf16")]          # bf16 | tf32 | fp32
        self.engine = tracking.default_engine(cfg.image.height, cfg.image.width)
        self.rt = self.engine.rt
        # The driver asks for the depth of the current image first and for the flow of (previous, current) afterwards
        # (dfvo.py:299-333), with host work (cv2.resize, preprocess_depth) in between.  forward_depth therefore also enqueues the flow
        # network of (image of the previous forward_depth call, this image) on a side stream; forward_flow hands that result out when
        # -- and only when -- it is called with exactly those two images (compared byte for byte), and computes afresh otherwise.
        # Same kernels, same results; the flow network just runs while the host is busy.  DFVO_LIBS_SPECULATE=0 turns it off.
        self.speculate = os.environ.get("DFVO_LIBS_SPECULATE", "1") != "0"
        self._prev = None            # (host copy, device buffer) of the image of the last forward_depth call
        self._spec = None            # (ref host copy, cur host copy, (fwd, bwd, diff), event) of the speculative flow
        self._flow_stream = None

    # ------------------------------------------------------------------ setup (deep_models.py:38-117)
    def initialize_models(self):
        assert not self.finetune_cfg.enable, "dfvo_b200 is inference-only (online_finetune.enable must be False)"
        self.flow = self.initialize_deep_flow_model()
        if self.cfg.depth.depth_src is None:
            assert self.cfg.depth.deep_depth.pretrained_model is not None, "No precomputed depths nor pretrained depth model"
            self.depth = self.initialize_deep_depth_model()
        if self.cfg.deep_pose.enable:
            self.pose = self.initialize_deep_pose_model()

    def initialize_deep_pose_model(self):
        """deep_models.py:104-117 / pose/monodepth2/monodepth2.py:31-84: pose_encoder.pth (the encoder's keys only) + pose.pth, at
        the depth network's feed size."""
        assert self.cfg.depth.depth_src is None, "the PoseNet reads the depth network's feed size (deep_models.py:220)"
        wdir = self.cfg.deep_pose.pretrained_model
        print("==> Initialize Pose-CNN with [{}]".format(wdir))
        enc = _load_state_dict(os.path.join(wdir, "pose_encoder.pth"))
        dec = _load_state_dict(os.path.join(wdir, "pose.pth"))
        self.engine.build_pose(enc, dec, precision=self.precision, dataset=self.cfg.dataset)
        h = _DepthHandle()
        h.stereo_baseline_multiplier = tracking.pose_baseline_multiplier(self.cfg.dataset)
        return h

    def initialize_deep_flow_model(self):
        assert self.cfg.deep_flow.network == "liteflow", "Invalid flow network [{}] is provided.".format(self.cfg.deep_flow.network)
        path = self.cfg.deep_flow.flow_net_weight
        assert path is not None, "No LiteFlowNet pretrained model is provided."
        print("==> Initialize LiteFlowNet with [{}]: ".format(path))
        self.engine.build_flow(_load_state_dict(path), pairs=1, precision=self.precision)
        return _FlowHandle()

    def initialize_deep_depth_model(self):
        assert self.cfg.depth.deep_depth.network == "monodepth2", "Invalid depth network"
        wdir = self.cfg.depth.deep_depth.pretrained_model
        print("==> Initialize Depth-CNN with [{}]".format(wdir))
        enc = _load_state_dict(os.path.join(wdir, "encoder.pth"))
        dec = _load_state_dict(os.path.join(wdir, "depth.pth"))
        self.engine.build_depth(enc, dec, precision=self.precision, dataset=self.cfg.dataset)
        h = _DepthHandle()
        h.feed_height, h.feed_width = self.engine.feed_h, self.engine.feed_w          # monodepth2.py:70-71
        c = tracking.depth_constants(self.cfg.dataset)
        h.min_depth, h.max_depth, h.stereo_baseline_multiplier = c["min_depth"], c["max_depth"], c["baseline"]
        return h

    def setup_train(self):
        raise NotImplementedError("online finetuning is outside the dfvo_b200 hot path (SURVEY.md section 8f rank 4)")

    # ------------------------------------------------------------------ inference
    def forward_flow(self, in_cur_data, in_ref_data, forward_backward):
        """deep_models.py:144-182.  Values are device-backed arrays (``tracking.DevArray``): [2,H,W] flows
        and the [H,W,1] inconsistency map; they convert to NumPy on demand."""
        assert forward_backward, "dfvo_b200 always computes forward+backward flow (deep_flow.forward_backward: True)"
        H, W = self.engine.H, self.engine.W
        spec, self._spec = self._spec, None
        if spec is not None and _same_image(in_ref_data["img"], spec[0]) and _same_image(in_cur_data["img"], spec[1]):
            fwd, bwd, diff = spec[2]
            self.rt.wait_event(spec[3])                       # the caller's stream continues after the speculative flow network
        else:
            if spec is not None:
                self.rt.wait_event(spec[3])                   # the engine's flow buffers are about to be rewritten
            ref = self.rt.from_host(np.ascontiguousarray(in_ref_data["img"], np.uint8))
            cur = self.rt.from_host(np.ascontiguousarray(in_cur_data["img"], np.uint8))
            fwd, bwd, diff = self.engine.flow([ref, cur])
        src_id, tgt_id = in_ref_data["id"], in_cur_data["id"]
        return {
            (src_id, tgt_id): tracking.DevArray(fwd, (2, H, W)),
            (tgt_id, src_id): tracking.DevArray(bwd, (2, H, W)),
            (src_id, tgt_id, "diff"): tracking.DevArray(diff, (H, W, 1)),
        }

    def forward_depth(self, imgs):
        """deep_models.py:184-206.  The PIL LANCZOS resize to the feed size + ToTensor run on the device,
        bit-identical to Pillow's 8-bit path (b200/lanczos.py, csrc/depth_ops.cu).  Returns float32
        [feed_h, feed_w] on the host because the driver hands it to cv2.resize (dfvo.py:314-317)."""
        host = np.ascontiguousarray(imgs[0], np.uint8)
        img = self.rt.from_host(host)
        if self.speculate and self.engine.flow_ready:
            if self._spec is not None:                        # an unclaimed speculation: let it finish before its buffers are reused
                self.rt.wait_event(self._spec[3])
                self._spec = None
            keep = host.copy()
            if self._prev is not None and self._prev[0].shape == keep.shape:
                if self._flow_stream is None:
                    self._flow_stream = self.rt.new_stream()
                fork = self.rt.record_event()                 # the uploads above are ordered before the side stream's work
                with self.rt.on_stream(self._flow_stream):
                    self.rt.wait_event(fork)
                    res = self.engine.flow([self._prev[1], img])
                    ev = self.rt.record_event()
                self._spec = (self._prev[0], keep, res, ev)
            self._prev = (keep, img)
        out = self.engine.depth(self.engine.depth_feed(img))
        return out.numpy()

    def forward_pose(self, imgs):
        """deep_models.py:208-230: [ref, cur] uint8 images -> float32 [4,4] pose (relative pose from cur to ref).  The feeds are
        the device LANCZOS resize of forward_depth (deep_models.py:218-221 resize to the depth network's feed size)."""
        if not hasattr(self, "_pose_feeds"):
            shape = (1, 3, self.engine.feed_h, self.engine.feed_w)
            self._pose_feeds = [self.rt.empty(shape, np.float32), self.rt.empty(shape, np.float32)]
            self._pose_prev = None                            # host copy of the last call's cur image (its feed is _pose_feeds[1])
        ref, cur = (np.ascontiguousarray(im, np.uint8) for im in imgs)
        if self._pose_prev is not None and _same_image(ref, self._pose_prev):
            self._pose_feeds.reverse()                        # the driver's ref is the previous call's cur: reuse its feed
        else:
            self.engine.depth_feed(self.rt.from_host(ref), out=self._pose_feeds[0])
        self.engine.depth_feed(self.rt.from_host(cur), out=self._pose_feeds[1])
        self._pose_prev = cur.copy()
        return self.engine.pose(*self._pose_feeds).numpy().astype(np.float32)

    def finetune(self, *a, **k):
        raise NotImplementedError("online finetuning is outside the dfvo_b200 hot path")

    def save_model(self):
        raise NotImplementedError("online finetuning is outside the dfvo_b200 hot path")
