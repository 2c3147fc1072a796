"""Precision-mode parity measurements at the BASELINE sizes (376x1241 frames, 352x1216 flow-net input, 192x640 depth feed):
device networks in every precision mode against the CPU oracle (torch fp32), and what the difference does downstream --
bits of the `flow_diff < 0.1` mask, members of the local_bestN keypoint set, the recovered pose.

Used by tests/test_gpu_parity_fullsize.py (asserts the bounds, writes the table to $DFVO_REPORT_DIR/parity_fullsize.json) and by
`bench.py --config parity` (prints the same table).  The oracle is the checker only.

End-to-end chain.  There are no trained weights offline, and a random-weight LiteFlowNet has no forward-backward-consistent
pixels (the oracle's own `flow_diff` is > 0.1 px almost everywhere), so "net -> mask -> keypoints -> pose" cannot be closed
on the networks' raw output.  `chain_case` therefore transplants the precision error FIELD of the real network at full size
(device flow in mode p minus oracle flow, forward and backward: its true magnitude, spatial structure and correlation with
image content) onto a consistent synthetic scene: rigid flow of the analytic KITTI-like scene + its exact inverse flow +
a smooth model-error field that puts the consistency map in the regime a trained network produces (a sizeable fraction of
pixels on either side of the 0.1 px threshold).  Reference arm: oracle consistency map -> oracle local_bestN -> cv2
E-tracker.  Device arm: device consistency kernel -> device selection -> device E-tracker, on flow + error field of mode p.
"""
import ctypes
import json
import os

import numpy as np

import synthdata

H, W = 376, 1241
FEED_H, FEED_W = 192, 640


def _dptr(t):
    return ctypes.c_void_p(t.data_ptr())


def device_flow(lib, ref, cur, prec, weights, h=H, w=W):
    import torch
    from b200 import native
    ctx = native.Context(lib)
    ctx.load_weights(native.NET_LITEFLOWNET, weights)
    ctx.liteflow_build(h, w, 1, prec)
    d_ref, d_cur = torch.from_numpy(ref).cuda(), torch.from_numpy(cur).cuda()
    fwd = torch.zeros((2, h, w), dtype=torch.float32, device="cuda")
    bwd = torch.zeros_like(fwd)
    diff = torch.zeros((h, w), dtype=torch.float32, device="cuda")
    ctx.liteflow_forward([d_ref.data_ptr(), d_cur.data_ptr()], _dptr(fwd), _dptr(bwd), _dptr(diff))
    torch.cuda.synchronize()
    out = fwd.cpu().numpy(), bwd.cpu().numpy(), diff.cpu().numpy()
    ctx.close()
    return out


def device_depth(lib, feed, prec, enc, dec):
    import torch
    from b200 import native
    ctx = native.Context(lib)
    ctx.load_weights(native.NET_MONODEPTH2, enc)
    ctx.load_weights(native.NET_MONODEPTH2, dec)
    ctx.monodepth2_build(feed.shape[2], feed.shape[3], prec)
    x = torch.from_numpy(feed).cuda()
    out = torch.zeros((feed.shape[2], feed.shape[3]), dtype=torch.float32, device="cuda")
    ctx.monodepth2_forward(_dptr(x), _dptr(out))
    torch.cuda.synchronize()
    r = out.cpu().numpy()
    ctx.close()
    return r


_ORACLE = {}


def oracle_flow(seed_a=11, seed_b=12):
    """Oracle LiteFlowNet at 376x1241 on two value-noise frames (a few seconds of CPU); cached per process."""
    import torch
    from oracle import nets
    key = ("flow", seed_a, seed_b)
    if key not in _ORACLE:
        ref, cur = synthdata.value_noise_image(H, W, seed_a), synthdata.value_noise_image(H, W, seed_b)
        w = synthdata.liteflownet_weights()
        to_t = lambda im: torch.from_numpy(np.transpose(im / 255, (2, 0, 1))).unsqueeze(0).float()
        with torch.no_grad():
            o = nets.liteflow_inference_flow(nets.to_torch(w), to_t(ref), to_t(cur))
        _ORACLE[key] = dict(ref=ref, cur=cur, weights=w, fwd=o["forward"][0].numpy(), bwd=o["backward"][0].numpy(),
                            diff=o["flow_diff"][0, :, :, 0].numpy())
    return _ORACLE[key]


def oracle_depth(seed=21):
    import torch
    from oracle import nets
    key = ("depth", seed)
    if key not in _ORACLE:
        enc, dec = synthdata.monodepth2_weights(4869, FEED_H, FEED_W)
        img = synthdata.value_noise_image(H, W, seed)
        import PIL.Image as pil
        feed = np.ascontiguousarray(np.transpose(np.asarray(pil.fromarray(img).resize((FEED_W, FEED_H), pil.LANCZOS), np.float32) / 255, (2, 0, 1))[None])
        with torch.no_grad():
            d = nets.monodepth2_inference_depth({k: v for k, v in nets.to_torch(enc).items() if not isinstance(v, int)},
                                                nets.to_torch(dec), torch.from_numpy(feed))[0, 0].numpy()
        _ORACLE[key] = dict(enc=enc, dec=dec, feed=feed, depth=d)
    return _ORACLE[key]


def flow_metrics(dev, orc, thre=0.1):
    """dev = (fwd, bwd, diff) of the device, orc = oracle dict."""
    f, b, d = dev
    epe_f = np.sqrt(((f - orc["fwd"]) ** 2).sum(0))
    epe_b = np.sqrt(((b - orc["bwd"]) ** 2).sum(0))
    dd = np.abs(d - orc["diff"])
    m_dev, m_orc = d < thre, orc["diff"] < thre
    mag = np.sqrt((orc["fwd"] ** 2).sum(0))
    return dict(epe_mean=float(epe_f.mean()), epe_p99=float(np.percentile(epe_f, 99)), epe_max=float(epe_f.max()),
                epe_bwd_mean=float(epe_b.mean()), flow_mag_mean=float(mag.mean()),
                diff_abs_err_mean=float(dd.mean()), diff_abs_err_max=float(dd.max()),
                mask_flip_frac=float((m_dev != m_orc).mean()), mask_density_oracle=float(m_orc.mean()), mask_density_device=float(m_dev.mean()))


def inverse_flow(fwd, iters=12):
    """bwd(y) with y = x + fwd(x)  =>  bwd(y) = -fwd(x); fixed point x <- y - fwd(x) with bilinear sampling (scipy)."""
    from scipy.ndimage import map_coordinates
    h, w = fwd.shape[1:]
    ys, xs = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing="ij")
    px, py = xs.copy(), ys.copy()
    for _ in range(iters):
        fx = map_coordinates(fwd[0], [py, px], order=1, mode="nearest")
        fy = map_coordinates(fwd[1], [py, px], order=1, mode="nearest")
        px, py = xs - fx, ys - fy
    fx = map_coordinates(fwd[0], [py, px], order=1, mode="nearest")
    fy = map_coordinates(fwd[1], [py, px], order=1, mode="nearest")
    return np.stack([-fx, -fy], 0)


def smooth_field(seed, sigma, grid=12):
    """Smooth 2-channel error field: coarse N(0, sigma) grid, bicubically upsampled (correlation length ~ `grid` px)."""
    import cv2
    rs = np.random.RandomState(seed)
    g = rs.standard_normal((2, H // grid + 3, W // grid + 3)) * sigma
    return np.stack([cv2.resize(g[c], (W, H), interpolation=cv2.INTER_CUBIC) for c in range(2)], 0)


def chain_scene(seed=71, model_err=0.045):
    """Consistent scene + model-error fields (shared by every arm)."""
    K = synthdata.kitti_intrinsics(H, W)
    depth = synthdata.scene_depth(H, W, K, seed)
    rvec, t = synthdata.default_motion(np.random.RandomState(seed))
    R = synthdata.rodrigues(rvec)
    f0 = synthdata.rigid_flow(depth, K, R, t)
    b0 = inverse_flow(f0)
    F = (f0 + smooth_field(seed + 1, model_err)).astype(np.float32)
    B = (b0 + smooth_field(seed + 2, model_err)).astype(np.float32)
    return dict(K=K, R=R, t=t, fwd=F, bwd=B)


def pose_delta(Ra, ta, Rb, tb):
    dR = Ra.T @ Rb
    ang = float(np.arccos(np.clip((np.trace(dR) - 1) / 2, -1, 1)))
    na, nb = np.linalg.norm(ta), np.linalg.norm(tb)
    dt = float(np.linalg.norm(ta / na - tb / nb)) if na > 0 and nb > 0 else float(na != nb)
    return ang, dt


def chain_reference(scene):
    """Oracle arm: torch consistency map -> oracle local_bestN -> cv2 E-tracker (vo.compute_pose_2d2d)."""
    import torch
    from oracle import nets, vo
    with torch.no_grad():
        diff = nets.fb_consistency(torch.from_numpy(scene["fwd"][None]), torch.from_numpy(scene["bwd"][None]))[0, :, :, 0].numpy()
    good, cells = vo.local_bestn_indices(diff)
    assert good, "chain scene: the oracle finds too few consistent pixels"
    kp1, kp2 = vo.keypoints_from_indices(cells, scene["fwd"], W)
    np.random.seed(4869)
    r = vo.compute_pose_2d2d(kp1, kp2, scene["K"])
    return dict(diff=diff, idx=np.concatenate(cells), pose=r, kp1=kp1, kp2=kp2)


def chain_device(engine, scene, dfwd, dbwd):
    """Device arm: flows + precision error field -> dfvo_fb_consistency -> dfvo_local_bestn -> device E-tracker."""
    from b200 import tracking
    rt = engine.rt
    F = rt.from_host(np.ascontiguousarray((scene["fwd"] + dfwd).astype(np.float32))[None])
    B = rt.from_host(np.ascontiguousarray((scene["bwd"] + dbwd).astype(np.float32))[None])
    D = rt.empty((1, H, W), np.float32)
    engine.lib.check(engine.lib.dfvo_fb_consistency(F.ptr, B.ptr, D.ptr, H, W, rt.stream_ptr()))
    good, n, k1, k2 = engine.select_local_bestn(D, F, 10, 10, 2000, 0.1)
    assert good
    kp1, kp2 = k1.numpy()[:n], k2.numpy()[:n]
    np.random.seed(4869)
    r = tracking.compute_pose_2d2d(engine, kp1, kp2, scene["K"], kp_ref_buf=k1, kp_cur_buf=k2)
    idx = (kp1[:, 1] * W + kp1[:, 0]).astype(np.int64)
    return dict(diff=D.numpy()[0], idx=idx, pose=r)


def gt_error(scene, pose):
    """Error of a recovered (cur -> ref, unit translation) pose against the scene's true motion (ref -> cur: R, t)."""
    Rt, tt = scene["R"].T, -scene["R"].T @ np.asarray(scene["t"], np.float64).reshape(3, 1)
    return pose_delta(Rt, tt, pose["R"], pose["t"])


def chain_metrics(dev, ref, scene=None, thre=0.1):
    a, b = set(dev["idx"].tolist()), set(ref["idx"].tolist())
    ang, dt = pose_delta(ref["pose"]["R"], ref["pose"]["t"], dev["pose"]["R"], dev["pose"]["t"])
    extra = {}
    if scene is not None:
        (ra, ta), (rb, tb) = gt_error(scene, ref["pose"]), gt_error(scene, dev["pose"])
        extra = dict(gt_rot_err_ref=ra, gt_tdir_err_ref=ta, gt_rot_err_dev=rb, gt_tdir_err_dev=tb)
    return dict(**extra, mask_flip_frac=float(((dev["diff"] < thre) != (ref["diff"] < thre)).mean()), mask_density=float((ref["diff"] < thre).mean()),
                kp_ref=len(b), kp_dev=len(a), kp_changed_frac=float(len(b - a) / max(1, len(b))),
                pose_rot_rad=ang, pose_tdir=dt, inliers_ref=int(ref["pose"]["inliers"].sum()), inliers_dev=int(dev["pose"]["inliers"].sum()))


def precision_modes():
    from b200 import native
    return [("fp32", native.PREC_FP32), ("tf32", native.PREC_TF32), ("bf16", native.PREC_BF16)]


CHAIN_SEEDS = (71, 83, 97)


def _mean_rows(rows):
    return {k: float(np.mean([r[k] for r in rows])) for k in rows[0]}


def measure_all(lib, engine, modes=None, seeds=CHAIN_SEEDS):
    """The whole table: {mode: {flow: .., depth: .., chain: ..}} + the chain on identical inputs ('exact_inputs');
    chain rows are means over `seeds` scenes (per-scene rows under chain_scenes)."""
    orc, od = oracle_flow(), oracle_depth()
    scenes = [chain_scene(s) for s in seeds]
    refs = [chain_reference(sc) for sc in scenes]
    ex = [chain_metrics(chain_device(engine, sc, 0.0, 0.0), rf, sc) for sc, rf in zip(scenes, refs)]
    out = {"exact_inputs": dict(chain=_mean_rows(ex), chain_scenes=ex)}
    for name, prec in (modes or precision_modes()):
        dev = device_flow(lib, orc["ref"], orc["cur"], prec, orc["weights"])
        row = dict(flow=flow_metrics(dev, orc))
        d = device_depth(lib, od["feed"], prec, od["enc"], od["dec"])
        rel = np.abs(d - od["depth"]) / od["depth"]
        row["depth"] = dict(rel_err_mean=float(rel.mean()), rel_err_max=float(rel.max()))
        ch = [chain_metrics(chain_device(engine, sc, dev[0] - orc["fwd"], dev[1] - orc["bwd"]), rf, sc) for sc, rf in zip(scenes, refs)]
        row["chain"], row["chain_scenes"] = _mean_rows(ch), ch
        out[name] = row
    return out


def write_report(table, name="parity_fullsize.json"):
    """Writes the table as JSON into the directory DFVO_REPORT_DIR names; nothing is written when it is unset (the test prints
    the table either way), so a test run leaves the source tree as it found it."""
    d = os.environ.get("DFVO_REPORT_DIR")
    if not d:
        return
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, name), "w") as f:
        json.dump(table, f, indent=1, sort_keys=True)
