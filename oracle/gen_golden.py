"""Generate tests/golden/*.npz by running the REFERENCE ITSELF (a DF-VO checkout named by DFVO_REFERENCE_ROOT, imported
under oracle/shims.py) on seeded synthetic inputs.

    python -m oracle.gen_golden [name ...]

Only *outputs* (and tiny inputs) are stored; weights / frames / correspondences are regenerated
from seeds by oracle/synth.py on both sides.  Every file records the library versions that produced
it (SURVEY 8c) and the pinned ``align_corners`` choice (H3).
"""
import os
import sys
import tempfile

import numpy as np
import torch

from . import nets, ref_corr_emul, shims, synth

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def versions():
    import cv2
    import sklearn
    return dict(cv2=cv2.__version__, sklearn=sklearn.__version__, numpy=np.__version__, torch=torch.__version__,
                align_corners=str(shims.ALIGN_CORNERS_PINNED), reference="Huangying-Zhan/DF-VO @ 50e6ffa")


def save(name, **arrays):
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    meta = {"meta_" + k: np.array(v) for k, v in versions().items()}
    path = os.path.join(GOLDEN_DIR, name + ".npz")
    np.savez_compressed(path, **arrays, **meta)
    print("wrote %s (%.1f KB)" % (path, os.path.getsize(path) / 1024))


def build_cfg(h, w, **over):
    """The reference's own default configuration (options/examples/default_configuration.yml) via its
    ConfigLoader, with the image size / visualisation overrides the tests use."""
    conf = shims.import_reference("libs.general.configuration")
    cfg = conf.ConfigLoader().merge_cfg([os.path.join(shims.REFERENCE_ROOT, "options/examples/default_configuration.yml")])
    cfg.image.height, cfg.image.width = h, w
    cfg.visualization.enable = False
    cfg.directory.gt_pose_dir = None
    cfg.no_confirm = True
    for k, v in over.items():
        node = cfg
        parts = k.split(".")
        for p in parts[:-1]:
            node = node[p]
        node[parts[-1]] = v
    return cfg


def save_weights(tmp):
    lfn = os.path.join(tmp, "lfn.pth")
    torch.save(nets.to_torch(synth.liteflownet_weights()), lfn)
    return lfn


def save_depth_weights(tmp, feed_h, feed_w):
    d = os.path.join(tmp, "depth_%dx%d" % (feed_h, feed_w))
    os.makedirs(d, exist_ok=True)
    enc, dec = synth.monodepth2_weights(4869, feed_h, feed_w)
    mod = shims.import_reference("libs.deep_models.depth.monodepth2.resnet_encoder")
    full = mod.ResnetEncoder(18, False).state_dict()          # supplies fc.* / num_batches_tracked entries
    full = {k: v.clone() for k, v in full.items()}
    for k, v in nets.to_torch(enc).items():
        full[k] = v
    torch.save(full, os.path.join(d, "encoder.pth"))
    torch.save(nets.to_torch(dec), os.path.join(d, "depth.pth"))
    return d


# ---------------------------------------------------------------------------------------------
def gen_correlation():
    """Reference CUDA kernel text executed under emulation (oracle/ref_corr_emul.py)."""
    out = {}
    for i, (B, C, H, W, s) in enumerate([(2, 64, 5, 7, 1), (1, 32, 9, 11, 2), (1, 192, 4, 6, 1), (2, 96, 6, 8, 2)]):
        rs = np.random.RandomState(100 + i)
        a = rs.standard_normal((B, C, H, W)).astype(np.float32)
        b = rs.standard_normal((B, C, H, W)).astype(np.float32)
        out["case%d_shape" % i] = np.array([B, C, H, W, s])
        out["case%d_out" % i] = ref_corr_emul.reference_correlation(a, b, s)
    save("correlation", **out)


def gen_warp_fb():
    lfn = shims.import_reference("libs.deep_models.flow.lite_flow_net.lite_flow_net")
    df = shims.import_reference("libs.deep_models.flow.deep_flow")
    layers = shims.import_reference("libs.deep_models.depth.monodepth2.layers")
    rs = np.random.RandomState(7)
    x = rs.standard_normal((2, 8, 12, 20)).astype(np.float32)
    flow = (rs.standard_normal((2, 2, 12, 20)) * 3).astype(np.float32)
    lfn.Backward_tensorGrid.clear()
    warped = lfn.Backward(torch.from_numpy(x), torch.from_numpy(flow)).numpy()
    H, W = 24, 40
    fwd = (rs.standard_normal((1, 2, H, W)) * 3).astype(np.float32)
    bwd = (-fwd + rs.standard_normal((1, 2, H, W)) * 0.2).astype(np.float32)
    d = df.DeepFlow(H, W)
    px = layers.FlowToPix(1, H, W)(torch.from_numpy(fwd))
    diff = d.forward_backward_consistency(torch.from_numpy(fwd), torch.from_numpy(bwd), px).detach().numpy()
    ts = np.array([d.get_target_size(376, 1241), d.get_target_size(370, 1226), d.get_target_size(192, 640),
                   d.get_target_size(70, 150)])
    save("warp_fb", warp_x=x, warp_flow=flow, warp_out=warped, fb_fwd=fwd, fb_bwd=bwd, fb_diff=diff, target_sizes=ts)


def gen_liteflownet():
    shims.patch_reference_correlation(nets.correlation)
    lfn = shims.import_reference("libs.deep_models.flow.lite_flow_net.lite_flow_net")
    lfn.Backward_tensorGrid.clear()
    model = lfn.LiteFlowNet().eval()
    model.load_state_dict(nets.to_torch(synth.liteflownet_weights()))
    H, W = 64, 128
    a = torch.cat([_img(H, W, 1), _img(H, W, 2)])
    b = torch.cat([_img(H, W, 2), _img(H, W, 1)])
    with torch.no_grad():
        out = model([a, b])
    save("liteflownet_64x128", **{"flow%d" % i: v.numpy() for i, v in out.items()})


def _img(H, W, seed):
    return torch.from_numpy(np.transpose(synth.value_noise_image(H, W, seed) / 255, (2, 0, 1))).unsqueeze(0).float()


def gen_deep_models():
    """DeepModel.forward_flow / forward_depth through the reference facade (deep_models.py)."""
    shims.patch_reference_correlation(nets.correlation)
    lfn = shims.import_reference("libs.deep_models.flow.lite_flow_net.lite_flow_net")
    lfn.Backward_tensorGrid.clear()
    dm = shims.import_reference("libs.deep_models.deep_models")
    H, W, fh, fw = 70, 150, 64, 96
    with tempfile.TemporaryDirectory() as tmp:
        cfg = build_cfg(H, W, **{"deep_flow.flow_net_weight": save_weights(tmp),
                                 "depth.deep_depth.pretrained_model": save_depth_weights(tmp, fh, fw)})
        model = dm.DeepModel(cfg)
        model.initialize_models()
        ref = {"img": synth.value_noise_image(H, W, 1), "id": 0}
        cur = {"img": synth.value_noise_image(H, W, 2), "id": 1}
        with torch.no_grad():
            flows = model.forward_flow(cur, ref, forward_backward=True)
            depth = model.forward_depth([cur["img"]])
        # the LANCZOS-resized network input the reference fed (deep_models.py:195-201), for staged parity
        import PIL.Image as pil
        from torchvision import transforms
        feed = transforms.ToTensor()(pil.fromarray(cur["img"]).resize((fw, fh), pil.LANCZOS)).numpy()
    save("deep_models_70x150", flow_fwd=flows[(0, 1)], flow_bwd=flows[(1, 0)], flow_diff=flows[(0, 1, "diff")],
         depth=depth, depth_feed=feed, feed_hw=np.array([fh, fw]))


def gen_selection():
    ks = shims.import_reference("libs.matching.keypoint_sampler")
    out = {}
    cases = {"easy": dict(seed=21), "outliers": dict(seed=22, outlier_frac=0.3, diff_sigma=0.12),
             "sparse": dict(seed=23, diff_sigma=2.0), "toofew": dict(seed=24, diff_sigma=60.0)}
    for name, kw in cases.items():
        fr = synth.analytic_frame(h=376, w=1241, **kw)
        for method in ("local_bestN", "bestN"):
            cfg = build_cfg(376, 1241)
            cfg.kp_selection.local_bestN.enable = method == "local_bestN"
            cfg.kp_selection.bestN.enable = method == "bestN"
            sampler = ks.KeypointSampler(cfg)
            cur = {"depth": fr["depth"]}
            ref = {"flow": fr["flow_fwd"], "flow_diff": fr["flow_diff"]}
            o = sampler.kp_selection(cur, ref)
            key = "%s_%s" % (name, method)
            out[key + "_good"] = np.array(o["good_kp_found"])
            if o["good_kp_found"] and isinstance(o["kp1_best"], np.ndarray):
                kp1 = o["kp1_best"][0]
                lin = (kp1[:, 1] * 1241 + kp1[:, 0]).astype(np.int64)
                out[key + "_idx_sorted"] = np.sort(lin)
                out[key + "_kp2_of_sorted"] = o["kp2_best"][0][np.argsort(lin)]
    save("selection_376x1241", **out)


def _tracker_objs(h, w):
    cfg = build_cfg(h, w)
    cam = shims.import_reference("libs.geometry.camera_modules")
    timer = shims.import_reference("libs.general.timer")
    trk = shims.import_reference("libs.tracker")
    K = cam.Intrinsics(synth.kitti_intrinsics(h, w))
    return cfg, trk.EssTracker(cfg, K, timer.Timer()), trk.PnpTracker(cfg, K), cam


def gen_trackers():
    h, w = 376, 1241
    cfg, ess, pnp, cam = _tracker_objs(h, w)
    out = {}
    cases = {"out00": dict(seed=31, outlier_frac=0.0), "out30": dict(seed=32, outlier_frac=0.3),
             "out60": dict(seed=33, outlier_frac=0.6), "still": dict(seed=34, outlier_frac=0.1, zero_motion=True)}
    for name, kw in cases.items():
        kp_ref, kp_cur, info = synth.correspondences(n=2000, **kw)
        np.random.seed(4869)                                       # run.py:81-84
        r = ess.compute_pose_2d2d(kp_ref, kp_cur, True)
        out[name + "_pose"] = r["pose"].pose.copy()
        out[name + "_inliers"] = r["inliers"].copy()
        # scale recovery with the same RNG stream position the driver would have (dfvo.py:184)
        depth = info["depth"].astype(np.float32)
        depth_proc = depth * ((depth < 50) & (depth > 0))
        if np.linalg.norm(r["pose"].t) != 0:
            s = ess.find_scale_from_depth(kp_ref, kp_cur, r["pose"].inv_pose, depth_proc.astype(np.float64))
        else:
            s = np.nan
        out[name + "_scale"] = np.array(s)
        po = pnp.compute_pose_3d2d(kp_ref, kp_cur, depth_proc.astype(np.float64), True)
        out[name + "_pnp_pose"] = po["pose"].pose.copy()
        out[name + "_pnp_nkp"] = np.array(po["kp1"].shape[0])
        out[name + "_rng_after"] = np.array(np.random.randint(0, 2 ** 31 - 1))   # RNG position check
    save("trackers_2000", **out)


def gen_cv_solvers():
    """Raw third-party solver outputs the replays / CUDA solvers are pinned to."""
    import cv2
    out = {}
    K = synth.kitti_intrinsics()
    cx, cy, fx, fy = K
    for name, kw in {"out00": dict(seed=41, outlier_frac=0.0), "out30": dict(seed=42, outlier_frac=0.3),
                     "out60": dict(seed=43, outlier_frac=0.6)}.items():
        kp_ref, kp_cur, info = synth.correspondences(n=2000, **kw)
        E, mask = cv2.findEssentialMat(kp_cur, kp_ref, focal=fx, pp=(cx, cy), method=cv2.RANSAC, prob=0.99, threshold=0.2)
        cnt, R, t, pmask = cv2.recoverPose(E, kp_cur, kp_ref, focal=fx, pp=(cx, cy))
        out[name + "_E"] = E; out[name + "_mask"] = mask[:, 0]
        out[name + "_R"] = R; out[name + "_t"] = t; out[name + "_cheir"] = np.array(cnt); out[name + "_pmask"] = pmask[:, 0]
    # 5-point minimal solver: all real solutions stacked (SURVEY C.1)
    rs = np.random.RandomState(5)
    kp_ref, kp_cur, _ = synth.correspondences(seed=44, n=400, outlier_frac=0.0)
    sols, subsets = [], []
    for i in range(40):
        idx = rs.choice(400, 5, replace=False)
        E5, _ = cv2.findEssentialMat(kp_cur[idx], kp_ref[idx], focal=fx, pp=(cx, cy), method=cv2.RANSAC, prob=0.99, threshold=0.2)
        E5 = np.zeros((0, 3)) if E5 is None else E5
        sols.append(np.concatenate([E5, np.full((30 - E5.shape[0], 3), np.nan)]))
        subsets.append(idx)
    out["five_point_subsets"] = np.array(subsets); out["five_point_solutions"] = np.array(sols)
    save("cv_solvers", **out)


ITERATIVE_CFG = {"kp_selection.rigid_flow_kp.enable": True, "scale_recovery.method": "iterative"}      # ablation_scale_iterative.yml


def gen_dfvo_driver_iter():
    """gen_dfvo_driver with rigid-flow keypoints + iterative scale recovery (SURVEY 8f rank 1; kitti_*_extend.yml)."""
    gen_dfvo_driver(ITERATIVE_CFG, "dfvo_driver_iter_188x620")


def gen_dfvo_driver(extra_cfg=None, name="dfvo_driver_188x620"):
    """The UNMODIFIED reference driver (libs/dfvo.py main loop) on a synthetic sequence with analytic
    network outputs injected at DeepModel.forward_flow / forward_depth; trackers, selection, GRIC, scale
    recovery and PnP fallback are the reference's own.  Poses are the golden for the drop-in test."""
    from . import seqdata
    h, w, n = 188, 620, 7
    with tempfile.TemporaryDirectory() as tmp:
        K = seqdata.write_sequence(os.path.join(tmp, "seqs"), n, h, w)
        cfg = build_cfg(h, w, **{"directory.img_seq_dir": os.path.join(tmp, "seqs"), "directory.result_dir": os.path.join(tmp, "res"),
                                 "image.ext": "png", "seq": "00", **(extra_cfg or {})})
        os.makedirs(cfg.directory.result_dir, exist_ok=True)
        dm = shims.import_reference("libs.deep_models.deep_models")
        seqdata.patch_deep_model(dm.DeepModel, h, w, K)
        ks = shims.import_reference("libs.matching.keypoint_sampler")
        seqdata.patch_canonical_kp_order(ks.KeypointSampler)        # order of an unordered set only (SURVEY H2)
        dfvo = shims.import_reference("libs.dfvo")
        np.random.seed(cfg.seed)                                    # apis/run.py:81-84
        torch.manual_seed(cfg.seed)
        poses = seqdata.run_driver(dfvo, cfg, n)
    save(name, poses=poses, K=np.array(K), hw=np.array([h, w]))


def gen_rigid_flow_kp():
    """SURVEY 8f rank 1: EssTracker.kp_selection_good_depth (RigidFlow layer + opt_rigid_flow_kp), compute_rigid_flow_kp
    and scale_recovery_iterative of the reference, with rigid_flow_kp enabled (kitti_*_extend.yml / ablation_scale_iterative.yml)."""
    h, w = 376, 1241
    cam = shims.import_reference("libs.geometry.camera_modules")
    timer = shims.import_reference("libs.general.timer")
    trk = shims.import_reference("libs.tracker")
    ks = shims.import_reference("libs.matching.keypoint_sampler")
    out = {}
    cases = {"clean": dict(seed=51), "outliers": dict(seed=52, outlier_frac=0.3, diff_sigma=0.12)}
    for kp_src in ("kp_best", "kp_depth"):
        for name, kw in cases.items():
            cfg = build_cfg(h, w, **{"kp_selection.rigid_flow_kp.enable": True, "scale_recovery.method": "iterative",
                                     "scale_recovery.kp_src": kp_src})
            K = cam.Intrinsics(synth.kitti_intrinsics(h, w))
            ess = trk.EssTracker(cfg, K, timer.Timer())
            fr = synth.analytic_frame(h=h, w=w, **kw)
            depth_proc = fr["depth"] * ((fr["depth"] < 50) & (fr["depth"] > 0))
            cur = {"depth": depth_proc.astype(np.float64), "raw_depth": fr["depth"]}
            ref = {"flow": fr["flow_fwd"], "flow_diff": fr["flow_diff"], "raw_depth": fr["depth"], "depth": depth_proc.astype(np.float64)}
            sampler = ks.KeypointSampler(cfg)
            o = sampler.kp_selection(cur, ref)
            lin = (o["kp1_best"][0][:, 1] * w + o["kp1_best"][0][:, 0]).astype(np.int64)
            order = np.argsort(lin)                                    # canonical order (SURVEY H2)
            ref["kp_best"], cur["kp_best"] = o["kp1_best"][0][order], o["kp2_best"][0][order]
            np.random.seed(4869)
            r = ess.compute_pose_2d2d(ref["kp_best"], cur["kp_best"], True)
            E_pose = r["pose"]
            key = "%s_%s" % (name, kp_src)
            out[key + "_E_pose"] = E_pose.pose.copy()
            so = ess.scale_recovery(cur, ref, E_pose, False)
            out[key + "_scale"] = np.array(so["scale"])
            out[key + "_prev_scale"] = np.array(ess.prev_scale)
            out[key + "_rng_after"] = np.array(np.random.randint(0, 2 ** 31 - 1))
            if kp_src == "kp_best":
                # the maps / keypoint sets of the LAST iteration (pose scaled by the converged scale)
                out[key + "_rigid_flow_pose"] = ref["rigid_flow_pose"].pose.copy()
                out[key + "_rigid_flow_diff_s9"] = ref["rigid_flow_diff"][::9, ::9, 0].astype(np.float32)     # every 9th pixel
                out[key + "_kp1_uniform"] = so["ref_kp_depth"].astype(np.int32)       # integer pixel grid
                out[key + "_kp2_uniform"] = so["cur_kp_depth"].astype(np.float32)     # kp1 + float32 flow
                # compute_rigid_flow_kp with the hybrid pose (dfvo.py:195-200): best + uniform sets
                hyb = cam.SE3(E_pose.pose.copy())
                hyb.t = E_pose.t * so["scale"]
                ess.compute_rigid_flow_kp(cur, ref, hyb)
                k1 = ref["kp_depth"]
                lin = (k1[:, 1] * w + k1[:, 0]).astype(np.int64)
                out[key + "_best_idx_sorted"] = np.sort(lin)
                out[key + "_kp1_uniform_hyb"] = ref["kp_depth_uniform"].astype(np.int32)
                out[key + "_rigid_flow_diff_hyb_s9"] = ref["rigid_flow_diff"][::9, ::9, 0].astype(np.float32)
    save("rigid_flow_kp_376x1241", **out)


GENERATORS = {
    "correlation": gen_correlation, "warp_fb": gen_warp_fb, "liteflownet": gen_liteflownet,
    "deep_models": gen_deep_models, "selection": gen_selection, "trackers": gen_trackers,
    "cv_solvers": gen_cv_solvers, "dfvo_driver": gen_dfvo_driver, "rigid_flow_kp": gen_rigid_flow_kp,
    "dfvo_driver_iter": gen_dfvo_driver_iter,
}

if __name__ == "__main__":
    names = sys.argv[1:] or list(GENERATORS)
    for n in names:
        print("== generating", n)
        GENERATORS[n]()
