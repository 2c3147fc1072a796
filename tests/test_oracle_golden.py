"""CPU: the oracle restatements (oracle/nets.py, oracle/vo.py) against golden vectors produced by
the reference itself (oracle/gen_golden.py, run against a DF-VO checkout named by DFVO_REFERENCE_ROOT).  This is what pins the oracle (SURVEY 8c: the reference ships no tests of its own)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import nets, synth, vo
from util import img_to_tensor

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load(name):
    return np.load(os.path.join(G, name + ".npz"))


def test_correlation_vs_reference_kernel_text():
    g = load("correlation")
    i = 0
    while "case%d_shape" % i in g.files:
        B, C, H, W, s = g["case%d_shape" % i]
        rs = np.random.RandomState(100 + i)
        a = rs.standard_normal((B, C, H, W)).astype(np.float32)
        b = rs.standard_normal((B, C, H, W)).astype(np.float32)
        mine = nets.correlation(torch.from_numpy(a), torch.from_numpy(b), int(s)).numpy()
        assert mine.shape == g["case%d_out" % i].shape
        assert np.abs(mine - g["case%d_out" % i]).max() < 1e-6
        i += 1
    assert i >= 4


def test_warp_fb_target_size():
    g = load("warp_fb")
    w = nets.backward_warp(torch.from_numpy(g["warp_x"]), torch.from_numpy(g["warp_flow"])).numpy()
    assert np.abs(w - g["warp_out"]).max() < 2e-5
    d = nets.fb_consistency(torch.from_numpy(g["fb_fwd"]), torch.from_numpy(g["fb_bwd"])).numpy()
    assert np.abs(d - g["fb_diff"]).max() < 2e-5
    sizes = [(376, 1241), (370, 1226), (192, 640), (70, 150)]
    assert [tuple(x) for x in g["target_sizes"]] == [nets.get_target_size(*s) for s in sizes]
    assert nets.get_target_size(376, 1241) == (352, 1216)       # SURVEY Appendix D #1


def test_liteflownet_module():
    g = load("liteflownet_64x128")
    p = nets.to_torch(synth.liteflownet_weights())
    H, W = 64, 128
    a = torch.cat([img_to_tensor(synth.value_noise_image(H, W, 1)), img_to_tensor(synth.value_noise_image(H, W, 2))])
    b = torch.cat([a[1:2], a[0:1]])
    with torch.no_grad():
        out = nets.liteflownet_forward(p, a, b)
    for i in range(1, 6):
        assert np.abs(out[i].numpy() - g["flow%d" % i]).max() < 1e-5, i
    assert np.abs(g["flow1"]).max() > 1.0      # the synthetic net produces non-trivial flow


def test_deep_model_facade():
    g = load("deep_models_70x150")
    H, W = 70, 150
    p = nets.to_torch(synth.liteflownet_weights())
    ref, cur = synth.value_noise_image(H, W, 1), synth.value_noise_image(H, W, 2)
    with torch.no_grad():
        o = nets.liteflow_inference_flow(p, img_to_tensor(ref), img_to_tensor(cur))
    assert np.abs(o["forward"][0].numpy() - g["flow_fwd"]).max() < 2e-5
    assert np.abs(o["backward"][0].numpy() - g["flow_bwd"]).max() < 2e-5
    assert np.abs(o["flow_diff"][0].numpy() - g["flow_diff"]).max() < 5e-5
    fh, fw = g["feed_hw"]
    enc, dec = synth.monodepth2_weights(4869, int(fh), int(fw))
    enc = {k: v for k, v in nets.to_torch(enc).items() if not isinstance(v, int)}
    with torch.no_grad():
        d = nets.monodepth2_inference_depth(enc, nets.to_torch(dec), torch.from_numpy(g["depth_feed"]).unsqueeze(0))
    assert np.abs(d[0, 0].numpy() - g["depth"]).max() < 1e-4 * np.abs(g["depth"]).max()


SEL_CASES = {"easy": dict(seed=21), "outliers": dict(seed=22, outlier_frac=0.3, diff_sigma=0.12),
             "sparse": dict(seed=23, diff_sigma=2.0), "toofew": dict(seed=24, diff_sigma=60.0)}


@pytest.mark.parametrize("name", list(SEL_CASES))
def test_selection_sets(name):
    g = load("selection_376x1241")
    fr = synth.analytic_frame(h=376, w=1241, **SEL_CASES[name])
    good, sel = vo.local_bestn_indices(fr["flow_diff"])
    assert good == bool(g[name + "_local_bestN_good"])
    if good:
        lin = np.sort(np.concatenate(sel))
        assert np.array_equal(lin, g[name + "_local_bestN_idx_sorted"])
        kp1, kp2 = vo.keypoints_from_indices([lin], fr["flow_fwd"], 1241)
        assert np.array_equal(kp2, g[name + "_local_bestN_kp2_of_sorted"])
    lin = vo.bestn_indices(fr["flow_diff"])
    assert np.array_equal(lin, g[name + "_bestN_idx_sorted"])


TRK_CASES = {"out00": dict(seed=31, outlier_frac=0.0), "out30": dict(seed=32, outlier_frac=0.3),
             "out60": dict(seed=33, outlier_frac=0.6), "still": dict(seed=34, outlier_frac=0.1, zero_motion=True)}


@pytest.mark.parametrize("name", list(TRK_CASES))
def test_trackers_vs_reference(name):
    """oracle/vo.py orchestration (same cv2 / sklearn calls, same RNG consumption) == reference classes."""
    g = load("trackers_2000")
    K = synth.kitti_intrinsics()
    kp_ref, kp_cur, info = synth.correspondences(n=2000, **TRK_CASES[name])
    np.random.seed(4869)
    r = vo.compute_pose_2d2d(kp_ref, kp_cur, K)
    pose = np.eye(4); pose[:3, :3] = r["R"]; pose[:3, 3:] = r["t"]
    assert np.array_equal(pose, g[name + "_pose"])
    assert np.array_equal(r["inliers"], g[name + "_inliers"])
    depth = info["depth"].astype(np.float32)
    depth_proc = (depth * ((depth < 50) & (depth > 0))).astype(np.float64)
    if np.linalg.norm(r["t"]) != 0:
        s = vo.find_scale_from_depth(kp_ref, kp_cur, np.linalg.inv(pose), depth_proc, K)
        assert s == float(g[name + "_scale"])
    else:
        assert np.isnan(g[name + "_scale"])
    ppose, kp1, kp2, _ = vo.compute_pose_3d2d(kp_ref, kp_cur, depth_proc, K)
    assert np.allclose(ppose, g[name + "_pnp_pose"], atol=1e-12)
    assert kp1.shape[0] == int(g[name + "_pnp_nkp"])
    assert np.random.randint(0, 2 ** 31 - 1) == int(g[name + "_rng_after"])      # RNG stream position (H8)


def _rigid_case(name):
    import synthdata
    kw = {"clean": dict(seed=51), "outliers": dict(seed=52, outlier_frac=0.3, diff_sigma=0.12)}[name]
    fr = synthdata.analytic_frame(h=376, w=1241, **kw)
    depth_proc = (fr["depth"] * ((fr["depth"] < 50) & (fr["depth"] > 0))).astype(np.float64)
    good, cells = vo.local_bestn_indices(fr["flow_diff"])
    kp1, kp2 = vo.keypoints_from_indices([np.sort(np.concatenate(cells))], fr["flow_fwd"], 1241)
    return fr, depth_proc, kp1, kp2


@pytest.mark.parametrize("name", ["clean", "outliers"])
@pytest.mark.parametrize("kp_src", ["kp_best", "kp_depth"])
def test_rigid_flow_kp_iterative_scale_vs_reference(name, kp_src):
    """SURVEY 8f rank 1: oracle restatement of kp_selection_good_depth / opt_rigid_flow_kp / scale_recovery_iterative
    against the reference classes (golden rigid_flow_kp_376x1241.npz): scale, RNG position, uniform keypoints, the
    rigid-flow inconsistency map (sampled), the 'best' index set of compute_rigid_flow_kp."""
    g = np.load(os.path.join(G, "rigid_flow_kp_376x1241.npz"))
    K = synth.kitti_intrinsics(376, 1241)
    fr, depth_proc, kp1, kp2 = _rigid_case(name)
    key = "%s_%s" % (name, kp_src)
    np.random.seed(4869)
    r = vo.compute_pose_2d2d(kp1, kp2, K)
    E = np.eye(4); E[:3, :3] = r["R"]; E[:3, 3:] = r["t"]
    assert np.abs(E - g[key + "_E_pose"]).max() < 1e-12
    o = vo.scale_recovery_iterative(kp1, kp2, E, depth_proc, fr["depth"], fr["flow_fwd"], fr["flow_diff"], K, 0, kp_src=kp_src)
    assert abs(o["scale"] - float(g[key + "_scale"])) < 1e-12
    assert int(np.random.randint(0, 2 ** 31 - 1)) == int(g[key + "_rng_after"])
    if kp_src == "kp_best":
        assert np.abs(o["rigid_flow_pose"] - g[key + "_rigid_flow_pose"]).max() < 1e-12
        assert np.abs(o["rigid_flow_diff"][::9, ::9] - g[key + "_rigid_flow_diff_s9"]).max() < 1e-4      # torch float32 kernels may differ per CPU
        assert np.array_equal(o["kp1_uniform"].astype(np.int32), g[key + "_kp1_uniform"])
        assert np.array_equal(o["kp2_uniform"].astype(np.float32), g[key + "_kp2_uniform"])
        # compute_rigid_flow_kp with the hybrid pose (E_tracker.py:421-440; e_tracker.iterative_kp.score_method)
        hyb = E.copy(); hyb[:3, 3] *= o["scale"]
        rd = vo.rigid_flow_diff(fr["depth"], fr["flow_fwd"], np.linalg.inv(hyb), K)
        assert np.abs(rd[::9, ::9] - g[key + "_rigid_flow_diff_hyb_s9"]).max() < 1e-4
        best, uniform = vo.opt_rigid_flow_kp(rd, fr["flow_diff"][:, :, 0], score_method="opt_flow")
        assert np.array_equal(np.sort(np.concatenate(best)), g[key + "_best_idx_sorted"])
        ku, _ = vo.keypoints_from_indices(uniform, fr["flow_fwd"], 1241)
        assert np.array_equal(ku.astype(np.int32), g[key + "_kp1_uniform_hyb"])
