"""Shared by the CPU (host-emulation) and GPU tests of the correspondence-selection ablations: local best-N with score_method
flow_ratio, global best-N and uniformly sampled keypoints (ablation_correspondences_best_n.yml, ablation_correspondences_uniform.yml)
-- the class-level checks against the reference KeypointSampler's goldens and the driver-golden harness."""
import os

import numpy as np

import tracking_modes_cases as tm
from oracle import gen_golden_correspondences as ggc, seqdata

G = tm.G
H, W = ggc.H, ggc.W
CASES = ggc.CORRESPONDENCE_CASES
DRIVER_CFGS = {"uniform": ggc.UNIFORM_CFG, "bestn": ggc.BESTN_CFG, "flowratio": ggc.FLOWRATIO_CFG}
# the E-tracker on local best-N, scale recovery on the sampled list: the stepwise E branch with a separate scale set
MIXED_CFG = {"kp_selection.sampled_kp.enable": True, "scale_recovery.kp_src": "kp_list"}


def golden():
    return np.load(os.path.join(G, "correspondences_376x1241.npz"))


def upload_frame(rt, fr):
    fwd = rt.from_host(np.ascontiguousarray(fr["flow_fwd"][None], np.float32))
    diff = rt.from_host(np.ascontiguousarray(fr["flow_diff"][None, :, :, 0], np.float32))
    dd = rt.from_host(fr["depth_diff"]) if "depth_diff" in fr else None
    return fwd, diff, dd


def sorted_idx(kp1):
    return np.sort((kp1[:, 1] * W + kp1[:, 0]).astype(np.int64))


def check_flow_ratio(eng, name):
    """Engine.select_local_bestn(score_method='flow_ratio'): the ratio map bit-equal to the reference's fb_flow_mask (NaN / inf in
    the same places), good_kp_found and the selected set equal to the reference's."""
    g = golden()
    fr = ggc.correspondence_frame(**CASES[name])
    fwd, diff, dd = upload_frame(eng.rt, fr)
    good, n, kp1, _ = eng.select_local_bestn(diff, fwd, 10, 10, 2000, 0.1, depth_diff_buf=dd, depth_thre=ggc.DEPTH_THRE,
                                             score_method="flow_ratio")
    assert good == bool(g[name + "_ratio_good"]), name
    if not good:
        return
    m = eng.flow_ratio_map.numpy().reshape(H, W)
    assert np.array_equal(np.flatnonzero(np.isnan(m)), g[name + "_ratio_nan_idx"]), name
    assert np.array_equal(np.flatnonzero(np.isinf(m)), g[name + "_ratio_inf_idx"]), name
    win = m[ggc.WINDOW]
    want = g[name + "_ratio_window"]
    assert np.array_equal(np.isnan(win), np.isnan(want.view(np.float32))), name
    assert np.array_equal(win.view(np.uint32)[~np.isnan(win)], want[~np.isnan(win)]), name
    assert ggc.ratio_digest(m) == str(g[name + "_ratio_sha"]), name
    assert np.array_equal(sorted_idx(kp1.numpy()[:n]), g[name + "_ratio_idx_sorted"]), name


def check_flow_ratio_case1_counts_raw_diff(eng):
    """The case-1 early-out counts the raw flow_diff < thre: a frame whose raw differences pass but whose ratios all fail (tiny
    flow) is good by case 1, and then fails case 2 (no cell has a keypoint) -- so status[2] is the raw count."""
    fr = ggc.correspondence_frame(**CASES["easy"])
    fr["flow_fwd"][:] = 1e-12
    fwd, diff, _ = upload_frame(eng.rt, fr)
    good, n, _, _ = eng.select_local_bestn(diff, fwd, 10, 10, 2000, 0.1, score_method="flow_ratio")
    assert not good and n == 0
    key = (10, 10, 20)
    st = eng._sel[key]["st"].numpy()
    assert st[2] == int((fr["flow_diff"][:, :, 0] < np.float32(0.1)).sum()) and st[3] == 0


def check_bestn(eng, name):
    fr = ggc.correspondence_frame(**CASES[name])
    fwd, diff, _ = upload_frame(eng.rt, fr)
    good, n, kp1, _ = eng.select_bestn(diff, fwd, 2000)
    assert good and n == 2000
    assert np.array_equal(sorted_idx(kp1.numpy()[:n]), golden()[name + "_bestN_idx_sorted"]), name
    lin = (kp1.numpy()[:n, 1] * W + kp1.numpy()[:n, 0]).astype(np.int64)
    assert np.all(np.diff(lin) > 0), "best-N is emitted in ascending pixel index"


def check_sampled(eng):
    """Engine.sampled_keypoints and the mirror's sampled_kp bit-equal to the reference's kp1_list / kp2_list."""
    import dropin_cases as dc
    from b200 import config, tracking
    g = golden()
    fr = ggc.correspondence_frame(**CASES["easy"])
    fwd, _, _ = upload_frame(eng.rt, fr)
    tracking._default_engine = eng
    dc.fresh_libs()
    from libs.matching import keypoint_sampler, kp_selection
    for name, (crop, num_kp) in ggc.SAMPLED_SETTINGS.items():
        k1, k2, n = eng.sampled_keypoints(fwd, crop, num_kp)
        assert n == num_kp
        assert np.array_equal(k1.numpy(), g["kp1_list_" + name][0]), name
        assert np.array_equal(k2.numpy(), g["kp2_list_" + name][0]), name
        cfg = config.default_cfg(H, W)
        cfg.crop.flow_crop = crop
        cfg.kp_selection.sampled_kp = config.AttrDict(enable=True, num_kp=num_kp)
        ks = keypoint_sampler.KeypointSampler(cfg)
        o = kp_selection.sampled_kp(None, None, {"flow": tracking.DevArray(fwd, (2, H, W))}, ks.kps["uniform"], cfg, {})
        assert o["kp1_list"].dtype == np.float64 and o["kp1_list"].shape == (1, num_kp, 2)
        assert np.array_equal(o["kp1_list"], g["kp1_list_" + name]), name
        assert np.array_equal(o["kp2_list"], g["kp2_list_" + name]), name


def pipeline_cfg(kind, h, w):
    import dropin_cases as dc
    return dc.make_cfg(h, w, DRIVER_CFGS.get(kind, MIXED_CFG if kind == "mixed" else None))


def driver_golden(kind):
    """The driver golden of `kind`; 'mixed' has none and uses the flow_ratio one for the sequence (the same in every golden)."""
    return np.load(os.path.join(G, "dfvo_driver_%s_188x620.npz" % (kind if kind in DRIVER_CFGS else "flowratio")))


def run_pipeline(kind, mode, runtime=None):
    """The injected pipeline (analytic flow / depth of the driver golden's sequence) -> (poses [n,4,4], per-frame branch, pipeline)."""
    g = driver_golden(kind)
    h, w = [int(v) for v in g["hw"]]
    n = g["poses"].shape[0]
    np.random.seed(4869)
    p = tm.injected_pipeline_class()(list(g["K"]), h, w, cfg=pipeline_cfg(kind, h, w), runtime=runtime, **tm.MODES[mode])
    for _ in range(n):
        p.step(None)
    if p.overlap:
        p.flush()
    p.close()
    return np.stack([p.poses[i] for i in range(n)]), [p.modes[i] for i in range(n)], p


def run_mirror_driver(kind, runtime):
    """The reference driver's call sequence over the libs mirror (analytic network outputs) -> (poses, per-frame branch)."""
    import dropin_cases as dc
    import synthdata
    import vo_driver
    from b200 import runtime as rt_mod, tracking
    rt_mod.set_runtime(runtime)
    tracking._default_engine = None
    dc.fresh_libs()
    import libs.deep_models.deep_models as dm
    g = driver_golden(kind)
    h, w = [int(v) for v in g["hw"]]
    n = g["poses"].shape[0]
    K = synthdata.kitti_intrinsics(h, w)
    cfg = pipeline_cfg(kind, h, w)
    seqdata.patch_deep_model(dm.DeepModel, h, w, K)
    tracking.default_engine(h, w)
    frames = [synthdata.value_noise_image(h, w, 100 + i) for i in range(n)]
    np.random.seed(cfg.seed)
    drv = vo_driver.SequenceDriver(cfg, K, frames)
    orig = drv.infer

    def infer():
        drv.deep_models._t = drv.cur["id"]
        orig()
    drv.infer = infer
    poses = drv.run()
    return poses, [drv.modes.get(i) for i in range(n)]


REFUSED = [{"kp_selection.local_bestN.score_method": "flow_depth"},
           {"kp_selection.local_bestN.enable": False},                                   # no selector at all
           {"e_tracker.kp_src": "kp_list"},                                             # sampled_kp is off
           {"scale_recovery.kp_src": "kp_list"},
           {"pnp_tracker.kp_src": "kp_list"},
           {"tracking_method": "PnP", "pnp_tracker.kp_src": "kp_list"},
           {"kp_selection.local_bestN.enable": False, "kp_selection.sampled_kp.enable": True},   # kp_best named, not produced
           {"kp_selection.local_bestN.enable": False, "kp_selection.bestN.enable": True, "e_tracker.kp_src": "kp_list"},
           {"kp_selection.sampled_kp.enable": True, "kp_selection.rigid_flow_kp.enable": True, "scale_recovery.method": "iterative",
            "scale_recovery.kp_src": "kp_list"}]                                          # iterative scale on another set than E's
