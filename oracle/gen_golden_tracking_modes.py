"""Generate the goldens of the reference's tracker ablations by running the REFERENCE ITSELF (a DF-VO checkout named by
DFVO_REFERENCE_ROOT, imported under oracle/shims.py), with the helpers of oracle/gen_golden.py:

    python -m oracle.gen_golden_tracking_modes [name ...]

  dfvo_driver_pnp           the unmodified driver with tracking_method PnP (ablation_tracker_pnp.yml)
  dfvo_driver_flowsel       ... with e_tracker.validity.method flow, thre 5 (ablation_model_sel_flow.yml)
  dfvo_driver_flowsel_gate  ... the same at thre 8, where the sequence's still frame closes the gate
  tracking_modes            class-level EssTracker (flow) / PnpTracker results on seeded scenes (tracking_mode_scene)
"""
import sys

import numpy as np

from . import shims, synth


def _gg():
    from . import gen_golden                  # the reference-facing helpers; importing them needs torch and the oracle nets
    return gen_golden


PNP_CFG = {"tracking_method": "PnP"}                                                                # ablation_tracker_pnp.yml
FLOWSEL_CFG = {"e_tracker.validity.method": "flow", "e_tracker.validity.thre": 5}                  # ablation_model_sel_flow.yml


def gen_dfvo_driver_pnp():
    """gen_dfvo_driver with PnP-only tracking."""
    _gg().gen_dfvo_driver(PNP_CFG, "dfvo_driver_pnp_188x620")


def gen_dfvo_driver_flowsel():
    """gen_dfvo_driver with the E-tracker's flow-magnitude model selection."""
    _gg().gen_dfvo_driver(FLOWSEL_CFG, "dfvo_driver_flowsel_188x620")


def gen_dfvo_driver_flowsel_gate():
    """gen_dfvo_driver with the flow-magnitude check at thre 8: the sequence's still frame (mean flow ~7.3 px) then closes the gate
    (no shuffle, PnP fallback) while the others pass it -- thre 5 passes every frame of this sequence."""
    _gg().gen_dfvo_driver(dict(FLOWSEL_CFG, **{"e_tracker.validity.thre": 8}), "dfvo_driver_flowsel_gate_188x620")


def tracking_mode_scene(seed, t_scale=1.0, r_scale=1.0, n=2000, outlier_frac=0.3, noise=0.05, h=376, w=1241):
    """synth.correspondences with the translation / rotation vector scaled: both at 0 is a still camera (mean flow far below the
    gate); a tiny translation with noisy flow makes every repeat's recoverPose count fall under 0.05 n, so the flow-mode rule
    rejects repeats that have more RANSAC inliers.  Returns (kp_ref, kp_cur, depth)."""
    rs = np.random.RandomState(seed)
    K = synth.kitti_intrinsics(h, w)
    depth = synth.scene_depth(h, w, K, seed + 1)
    rvec, t = synth.default_motion(rs)
    flow = synth.rigid_flow(depth, K, synth.rodrigues(rvec * r_scale), t * t_scale)
    ys, xs = rs.randint(0, h, n), rs.randint(0, w, n)
    kp_ref = np.stack([xs, ys], 1).astype(np.float64)
    kp_cur = kp_ref + flow[:, ys, xs].T + rs.standard_normal((n, 2)) * noise
    nout = int(round(outlier_frac * n))
    if nout:
        idx = rs.permutation(n)[:nout]
        kp_cur[idx] = kp_ref[idx] + rs.uniform(-30, 30, (nout, 2))
    return kp_ref, kp_cur, depth


TRACKING_MODE_CASES = {"moving": dict(seed=71), "outliers": dict(seed=72, outlier_frac=0.6),
                       "still": dict(seed=73, t_scale=0.0, r_scale=0.0, outlier_frac=0.0),
                       "cheirality": dict(seed=61, t_scale=0.001, outlier_frac=0.0, noise=0.3)}


def gen_tracking_modes():
    """Class-level goldens of the reference EssTracker with validity.method 'flow' (thre 5) and of PnpTracker on seeded scenes:
    pose, inlier mask / kept keypoint count, and the global generator's position afterwards (state pos + the next draw)."""
    h, w = 376, 1241
    cfg = _gg().build_cfg(h, w, **FLOWSEL_CFG)
    cam = shims.import_reference("libs.geometry.camera_modules")
    timer = shims.import_reference("libs.general.timer")
    trk = shims.import_reference("libs.tracker")
    K = cam.Intrinsics(synth.kitti_intrinsics(h, w))
    ess, pnp = trk.EssTracker(cfg, K, timer.Timer()), trk.PnpTracker(cfg, K)
    out = {}
    for name, kw in TRACKING_MODE_CASES.items():
        kp_ref, kp_cur, depth = tracking_mode_scene(**kw)
        out[name + "_flow_mean"] = np.array(np.mean(np.linalg.norm(kp_ref - kp_cur, axis=1)))
        np.random.seed(4869)
        r = ess.compute_pose_2d2d(kp_ref, kp_cur, True)
        out[name + "_E_pose"] = r["pose"].pose.copy()
        out[name + "_E_inliers"] = r["inliers"].copy()
        out[name + "_E_rng_pos"] = np.array(np.random.get_state()[2])
        out[name + "_E_rng_after"] = np.array(np.random.randint(0, 2 ** 31 - 1))
        depth_proc = (depth * ((depth < 50) & (depth > 0))).astype(np.float32).astype(np.float64)
        np.random.seed(4869)
        po = pnp.compute_pose_3d2d(kp_ref, kp_cur, depth_proc, True)
        out[name + "_pnp_pose"] = po["pose"].pose.copy()
        out[name + "_pnp_nkp"] = np.array(po["kp1"].shape[0])
        out[name + "_pnp_rng_pos"] = np.array(np.random.get_state()[2])
        out[name + "_pnp_rng_after"] = np.array(np.random.randint(0, 2 ** 31 - 1))
    _gg().save("tracking_modes_2000", **out)


GENERATORS = {"dfvo_driver_pnp": gen_dfvo_driver_pnp, "dfvo_driver_flowsel": gen_dfvo_driver_flowsel,
              "dfvo_driver_flowsel_gate": gen_dfvo_driver_flowsel_gate, "tracking_modes": gen_tracking_modes}

if __name__ == "__main__":
    for n in sys.argv[1:] or list(GENERATORS):
        print("== generating", n)
        GENERATORS[n]()
