"""Generate the goldens of the PoseNet depth-consistency branch (deep_pose.enable + kp_selection.depth_consistency.enable) by
running the REFERENCE ITSELF (a DF-VO checkout named by DFVO_REFERENCE_ROOT, imported under oracle/shims.py) with the helpers of
oracle/gen_golden.py:

    python -m oracle.gen_golden_depth_consistency

writes tests/golden/depth_consistency.npz:
  pose_*        DeepModel.forward_pose([ref, cur]) (deep_models.py:208-230) with seeded synthetic PoseNet weights at a 64x192 depth
                feed, plus the LANCZOS feeds it used and the pose parameters before transformation_from_parameters
  dc{0,1}_*     DepthConsistency.compute (depth_consistency.py:153-163) on synthetic depths: case 0 sends pixels out of the image
                and behind the camera (negative ratios), case 1 has a zero z-translation so zero-depth pixels give 0/0 = NaN
  sel_*         KeypointSampler.kp_selection (local_bestN, score 'flow') with the depth mask of selection_depth_diff

    python -m oracle.gen_golden_depth_consistency driver

writes tests/golden/dfvo_driver_depthcons_188x620.npz: the unmodified driver (DFVO.main) with deep_pose and
kp_selection.depth_consistency enabled on the synthetic sequence of oracle/seqdata.py, forward_pose patched to analytic_deep_pose.
"""
import os
import tempfile

import cv2
import numpy as np
import torch

from . import pose_consistency, shims, synth


def _gg():
    from . import gen_golden
    return gen_golden


H_IMG, W_IMG, FEED_H, FEED_W = 70, 150, 64, 192


def save_pose_weights(tmp):
    d = os.path.join(tmp, "pose")
    os.makedirs(d, exist_ok=True)
    enc, dec = synth.posenet_weights()
    mod = shims.import_reference("libs.deep_models.depth.monodepth2.resnet_encoder")
    full = {k: v.clone() for k, v in mod.ResnetEncoder(18, False, 2).state_dict().items()}     # fc.* / num_batches_tracked
    for k, v in enc.items():
        full[k] = torch.from_numpy(v)
    full["unused.weight"] = torch.zeros(3)                       # a key the encoder does not have: filtered out on load
    torch.save(full, os.path.join(d, "pose_encoder.pth"))
    torch.save({k: torch.from_numpy(v) for k, v in dec.items()}, os.path.join(d, "pose.pth"))
    return d


def gen_pose():
    gg = _gg()
    shims.patch_reference_correlation(gg.nets.correlation)
    dm = shims.import_reference("libs.deep_models.deep_models")
    with tempfile.TemporaryDirectory() as tmp:
        cfg = gg.build_cfg(H_IMG, W_IMG, **{"deep_flow.flow_net_weight": gg.save_weights(tmp),
                                            "depth.deep_depth.pretrained_model": gg.save_depth_weights(tmp, FEED_H, FEED_W),
                                            "deep_pose.enable": True, "deep_pose.pretrained_model": save_pose_weights(tmp)})
        model = dm.DeepModel(cfg)
        model.initialize_models()
        ref, cur = synth.value_noise_image(H_IMG, W_IMG, 1), synth.value_noise_image(H_IMG, W_IMG, 2)
        with torch.no_grad():
            pose = model.forward_pose([ref, cur])
            import PIL.Image as pil
            from torchvision import transforms
            feeds = [transforms.ToTensor()(pil.fromarray(im).resize((FEED_W, FEED_H), pil.LANCZOS)).unsqueeze(0) for im in (ref, cur)]
            feats = model.pose.encoder(torch.cat(feeds, 1))
            aa, t = model.pose.pose_decoder([feats])
        mult = model.pose.stereo_baseline_multiplier
    return dict(pose=pose, pose_feed_ref=feeds[0][0].numpy(), pose_feed_cur=feeds[1][0].numpy(), pose_axisangle=aa[0, 0, 0].numpy(),
                pose_translation=t[0, 0, 0].numpy(), pose_multiplier=np.array(mult), pose_feed_hw=np.array([FEED_H, FEED_W]))


def consistency_case(case, h=60, w=90):
    """Synthetic (depth_cur, depth_ref, pose, [cx, cy, fx, fy]) of DepthConsistency case 0 / 1."""
    rs = np.random.RandomState(40 + case)
    K = synth.kitti_intrinsics(h, w)
    smooth = lambda: cv2.resize(rs.uniform(0.3, 20.0, (6, 9)), (w, h), interpolation=cv2.INTER_CUBIC).clip(0.3, 30).astype(np.float32)
    cur, ref = smooth(), smooth()                                           # CNN depths are smooth away from their edges
    cur[rs.rand(h, w) < 0.05] = 0.0                                        # zero-depth pixels (NEAREST-resized raw depth)
    ref[rs.rand(h, w) < 0.05] = 0.0
    rvec = np.array([0.01, -0.03, 0.005])
    t = np.array([0.4, -0.1, -1.5]) if case == 0 else np.array([0.3, 0.05, 0.0])
    if case == 1:
        ref[:, -2:] = 0.0                  # zero-depth points project to the far right: warp = 0 = reproj there -> NaN
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = synth.rodrigues(rvec), t
    return cur, ref, T.astype(np.float32), K


def gen_consistency():
    dcm = shims.import_reference("libs.matching.depth_consistency")
    cam = shims.import_reference("libs.geometry.camera_modules")
    out = {}
    for case in (0, 1):
        cur, ref, T, K = consistency_case(case)
        h, w = cur.shape
        cfg = _gg().build_cfg(h, w)
        dc = dcm.DepthConsistency(cfg, cam.Intrinsics(K))
        cd, rd = {"id": 1, "raw_depth": cur}, {"id": 0, "raw_depth": ref, "deep_pose": T}
        with torch.no_grad():
            dc.compute(cd, rd)
        out["dc%d_depth_diff" % case] = rd["depth_diff"]
        out["dc%d_K" % case] = np.asarray(K, np.float64)
    return out


def gen_selection():
    ks = shims.import_reference("libs.matching.keypoint_sampler")
    out = {}
    fr = synth.analytic_frame(seed=21, h=376, w=1241)
    cfg = _gg().build_cfg(376, 1241, **{"kp_selection.depth_consistency.enable": True})
    for name, thre in (("a", 0.05), ("b", 0.02)):
        cfg.kp_selection.depth_consistency.thre = thre
        sampler = ks.KeypointSampler(cfg)
        o = sampler.kp_selection({"depth": fr["depth"]}, {"flow": fr["flow_fwd"], "flow_diff": fr["flow_diff"],
                                                          "depth_diff": pose_consistency.selection_depth_diff(376, 1241)})
        kp1 = o["kp1_best"][0]
        out["sel_%s_thre" % name] = np.array(thre)
        out["sel_%s_idx_sorted" % name] = np.sort((kp1[:, 1] * 1241 + kp1[:, 0]).astype(np.int64))
    return out


DRIVER_CFG = {"deep_pose.enable": True, "kp_selection.depth_consistency.enable": True}
POSE_BIAS = np.array([0.004, -0.006, 0.003])       # rad: the mask then removes a visible share of the pixels


def analytic_deep_pose(t, h, w, K):
    """What the patched forward_pose returns at frame t: the analytic motion of the sequence plus a small fixed rotation bias,
    float32 4x4 (the PoseNet's output type)."""
    from . import seqdata
    f = seqdata.frame_inputs(t, h, w, K, seqdata.MODES[t % len(seqdata.MODES)])
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = synth.rodrigues(np.asarray(f["rvec"], np.float64) + POSE_BIAS), np.asarray(f["t"], np.float64).reshape(3)
    return T.astype(np.float32)


def gen_driver():
    """gen_golden.gen_dfvo_driver with the depth-consistency branch; asserts the trajectory differs from the unmasked driver golden
    (so the mask changed the keypoint sets of at least one frame)."""
    gg = _gg()
    dm = shims.import_reference("libs.deep_models.deep_models")
    h, w = 188, 620
    orig = getattr(dm.DeepModel, "forward_pose")

    def forward_pose(self, imgs):
        return analytic_deep_pose(self._t, h, w, self._K)
    from . import seqdata
    orig_patch = seqdata.patch_deep_model

    def patch(DeepModel, h_, w_, K):
        orig_patch(DeepModel, h_, w_, K)
        DeepModel._K = K
        DeepModel.forward_pose = forward_pose
    seqdata.patch_deep_model = patch
    try:
        gg.gen_dfvo_driver(DRIVER_CFG, "dfvo_driver_depthcons_188x620")
    finally:
        seqdata.patch_deep_model = orig_patch
        dm.DeepModel.forward_pose = orig
    a = np.load(os.path.join(gg.GOLDEN_DIR, "dfvo_driver_depthcons_188x620.npz"))["poses"]
    b = np.load(os.path.join(gg.GOLDEN_DIR, "dfvo_driver_188x620.npz"))["poses"]
    assert np.abs(a - b).max() > 1e-6, "the depth mask did not change any frame's keypoints"
    print("max |pose difference| vs the unmasked driver: %.3g" % np.abs(a - b).max())


if __name__ == "__main__":
    import sys
    if sys.argv[1:] == ["driver"]:
        gen_driver()
        sys.exit(0)
    res = {}
    res.update(gen_pose())
    res.update(gen_consistency())
    res.update(gen_selection())
    _gg().save("depth_consistency", **res)
