"""GPU: the PoseNet (dfvo_posenet_*) and the depth-consistency mask (dfvo_depth_consistency) on the H100 against the reference
goldens (tests/golden/depth_consistency.npz) and, at 376x1241 with a 192x640 feed, against the oracle restatements
(oracle/pose_consistency.py), and FramePipeline's branch in every execution mode."""
import os

import numpy as np
import pytest
import torch

from b200 import native
from oracle import pose_consistency, synth
import depth_consistency_cases as dc

pytestmark = pytest.mark.gpu

# relative bars on the six pose parameters (max |error| / max |reference|), measured on one H100 80GB HBM3
BARS = {native.PREC_FP32: 1e-4, native.PREC_TF32: 5e-3, native.PREC_BF16: 5e-2}


@pytest.mark.parametrize("prec", [native.PREC_FP32, native.PREC_TF32, native.PREC_BF16])
def test_posenet_vs_reference_golden(dev_lib, prec):
    g = dc.golden()
    mult = float(g["pose_multiplier"])
    pose = dc.posenet(dev_lib, dc.CudaMem(), g["pose_feed_ref"], g["pose_feed_cur"], prec, mult)
    aa, t = dc.pose_parameters_of(pose, mult)
    ea = np.abs(aa - g["pose_axisangle"]).max() / np.abs(g["pose_axisangle"]).max()
    et = np.abs(t - g["pose_translation"]).max() / np.abs(g["pose_translation"]).max()
    print("precision %d: axis-angle rel %.2e, translation rel %.2e" % (prec, ea, et))
    assert ea < BARS[prec] and et < BARS[prec]


def test_posenet_fullsize_and_mask_flips(dev_lib):
    """192x640 feed: fp32 pose vs the oracle; the share of mask pixels that flip between the fp32-mode and bf16-mode pose at
    376x1241 is reported (selection is chaotic, so the bound is on the pose)."""
    rs = np.random.RandomState(5)
    fr, fc = [rs.uniform(0, 1, (3, 192, 640)).astype(np.float32) for _ in range(2)]
    want = dc.oracle_pose(fr, fc, 5.4)
    p32 = dc.posenet(dev_lib, dc.CudaMem(), fr, fc, native.PREC_FP32, 5.4)
    pbf = dc.posenet(dev_lib, dc.CudaMem(), fr, fc, native.PREC_BF16, 5.4)
    a0, t0 = dc.pose_parameters_of(want, 5.4)
    a1, t1 = dc.pose_parameters_of(p32, 5.4)
    assert np.abs(a1 - a0).max() < 1e-4 * np.abs(a0).max() and np.abs(t1 - t0).max() < 1e-4 * np.abs(t0).max()
    H, W = 376, 1241
    K = synth.kitti_intrinsics(H, W)
    depth = synth.scene_depth(H, W, K, 3).astype(np.float32)
    m32 = dc.depth_consistency(dev_lib, dc.CudaMem(), depth, depth, p32, K) < 0.05
    mbf = dc.depth_consistency(dev_lib, dc.CudaMem(), depth, depth, pbf, K) < 0.05
    print("mask flips fp32 vs bf16 pose: %.4f %%" % (100.0 * (m32 != mbf).mean()))


def test_depth_consistency_golden_and_fullsize(dev_lib):
    g = dc.golden()
    from oracle import gen_golden_depth_consistency as gen
    for case in (0, 1):
        cur, ref, T, K = gen.consistency_case(case)
        dc.compare_depth_diff(dc.depth_consistency(dev_lib, dc.CudaMem(), cur, ref, T, K), g["dc%d_depth_diff" % case])
    H, W = 376, 1241
    K = synth.kitti_intrinsics(H, W)
    cur, ref = synth.scene_depth(H, W, K, 1).astype(np.float32), synth.scene_depth(H, W, K, 2).astype(np.float32)
    T = np.eye(4, dtype=np.float32)
    T[:3, :3], T[:3, 3] = synth.rodrigues(np.array([0.002, 0.01, -0.001])), [0.05, -0.02, 0.9]
    cx, cy, fx, fy = K
    Km = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float64)
    want = pose_consistency.depth_consistency(cur, ref, T, Km, np.linalg.inv(Km))
    got = dc.depth_consistency(dev_lib, dc.CudaMem(), cur, ref, T, K)
    n = dc.compare_depth_diff(got, want)
    print("376x1241: %d pixels within 5e-4 of the threshold" % n)


def test_masked_local_bestn_vs_reference_golden(dev_lib):
    g = dc.golden()
    fr = synth.analytic_frame(seed=21, h=376, w=1241)
    dd = pose_consistency.selection_depth_diff(376, 1241)
    for name in ("a", "b"):
        idx = dc.select_with_mask(dev_lib, dc.CudaMem(), fr["flow_diff"][..., 0], dd, float(g["sel_%s_thre" % name]))
        assert np.array_equal(idx, g["sel_%s_idx_sorted" % name])


def test_mirror_forward_pose_and_depth_consistency(dev_lib, tmp_path):
    """The libs mirror: DeepModel.initialize_models (pose_encoder.pth with keys the encoder does not have, pose.pth) and
    forward_pose against the reference's DeepModel.forward_pose golden in fp32 mode, on consecutive calls (the second reuses the
    first call's cur feed as its ref); DepthConsistency.compute against the kernel."""
    import dropin_cases as dcase
    from b200 import runtime as rt_mod, tracking
    from oracle import gen_golden_depth_consistency as gen, nets
    g = dc.golden()
    rt_mod.set_runtime(rt_mod.CudaRuntime(0))
    tracking._default_engine = None
    dcase.fresh_libs()
    import libs.deep_models.deep_models as dm
    from libs.geometry.camera_modules import Intrinsics
    from libs.matching.depth_consistency import DepthConsistency
    enc, dec = synth.monodepth2_weights(4869, gen.FEED_H, gen.FEED_W)
    penc, pdec = synth.posenet_weights()
    (tmp_path / "depth").mkdir(); (tmp_path / "pose").mkdir()
    torch.save(nets.to_torch(synth.liteflownet_weights()), str(tmp_path / "lfn.pth"))
    torch.save(nets.to_torch(enc), str(tmp_path / "depth" / "encoder.pth"))
    torch.save(nets.to_torch(dec), str(tmp_path / "depth" / "depth.pth"))
    torch.save(dict(nets.to_torch(penc), **{"unused.weight": torch.zeros(3), "encoder.fc.weight": torch.zeros(1000, 512)}),
               str(tmp_path / "pose" / "pose_encoder.pth"))
    torch.save(nets.to_torch(pdec), str(tmp_path / "pose" / "pose.pth"))
    cfg = dcase.make_cfg(gen.H_IMG, gen.W_IMG, gen.DRIVER_CFG)
    cfg.deep_flow.flow_net_weight = str(tmp_path / "lfn.pth")
    cfg.depth.deep_depth.pretrained_model = str(tmp_path / "depth")
    cfg.deep_pose.pretrained_model = str(tmp_path / "pose")
    old = os.environ.get("DFVO_B200_PRECISION")
    os.environ["DFVO_B200_PRECISION"] = "fp32"
    try:
        model = dm.DeepModel(cfg)
        model.initialize_models()
    finally:
        os.environ.pop("DFVO_B200_PRECISION") if old is None else os.environ.__setitem__("DFVO_B200_PRECISION", old)
    ref, cur = synth.value_noise_image(gen.H_IMG, gen.W_IMG, 1), synth.value_noise_image(gen.H_IMG, gen.W_IMG, 2)
    third = synth.value_noise_image(gen.H_IMG, gen.W_IMG, 3)
    p0 = model.forward_pose([third, ref])
    pose = model.forward_pose([ref, cur])                      # ref is the previous call's cur: its feed is reused
    assert pose.dtype == np.float32 and pose.shape == (4, 4)
    assert np.abs(pose - g["pose"]).max() < 1e-5 and np.abs(p0 - pose).max() > 1e-6
    cur_d, ref_d, T, K = gen.consistency_case(0)
    tracking.default_engine(cur_d.shape[0], cur_d.shape[1])
    cd, rd = {"id": 1, "raw_depth": cur_d}, {"id": 0, "raw_depth": ref_d, "deep_pose": T}
    DepthConsistency(cfg, Intrinsics(K)).compute(cd, rd)
    out = np.asarray(rd["depth_diff"])
    want = dc.depth_consistency(dev_lib, dc.CudaMem(), cur_d, ref_d, T, K)
    assert np.array_equal(np.isnan(out), np.isnan(want)) and np.array_equal(np.nan_to_num(out), np.nan_to_num(want))


def test_pipeline_posenet_modes_bit_identical(dev_lib):
    """FramePipeline with the branch on and the real PoseNet (seeded synthetic weights; analytic flows injected so the selection
    finds keypoints): the per-frame feeds, the PoseNet on the depth stream after the reference frame's feed, and the mask give
    bit-identical poses in every execution mode."""
    import tracking_modes_cases as tm
    from b200 import config, pipeline, runtime as rt_mod
    from oracle import seqdata
    rt = rt_mod.CudaRuntime(0)
    rt_mod.set_runtime(rt)
    h, w, n = 188, 620, 6
    K = synth.kitti_intrinsics(h, w)
    lfn = synth.liteflownet_weights()
    enc, dec = synth.monodepth2_weights(4869, 64, 192)
    penc, pdec = synth.posenet_weights()
    frames = [synth.value_noise_image(h, w, 100 + i) for i in range(n)]

    def inject(p, st):
        if st.fwd is not None:
            f = seqdata.frame_inputs(st.id, h, w, K, seqdata.MODES[st.id % len(seqdata.MODES)])
            st.fwd.upload(f["fwd"][None]); st.bwd.upload(f["bwd"][None]); st.diff.upload(f["diff"][None, :, :, 0])

    def run(mode, on=True):
        cfg = config.default_cfg(h, w)
        cfg.deep_pose.enable = on
        cfg.kp_selection.depth_consistency.enable = on
        np.random.seed(4869)
        p = pipeline.FramePipeline(K, h, w, cfg=cfg, runtime=rt, inject=inject, **tm.MODES[mode])
        p.load_weights(lfn, enc, dec, penc, pdec)
        for im in frames:
            p.step(im)
        if p.overlap:
            p.flush()
        p.close()
        return np.stack([p.poses[i] for i in range(n)])

    base = run("in_order")
    for mode in ("overlap", "inflight2", "inflight3", "pipelined", "tracker_thread"):
        assert np.array_equal(run(mode), base), mode
    print("max |pose difference| with the branch off: %.3g" % np.abs(run("in_order", on=False) - base).max())
