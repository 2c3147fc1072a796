"""TEST INFRASTRUCTURE: the per-frame call sequence of the reference driver (libs/dfvo.py), hybrid tracking, restated as a
small loop so that the drop-in tests can run without a DF-VO checkout (and therefore without libs/dfvo.py itself)
does not exist.  It touches the `libs.*` mirror only through the calls the real driver makes, in the same order:

    DFVO.setup            dfvo.py:60-92    Dataset -> trackers -> KeypointSampler -> DeepModel(cfg).initialize_models()
    deep_model_inference  dfvo.py:299-345  forward_depth -> cv2.resize NEAREST -> preprocess_depth -> forward_flow -> .copy()
    tracking              dfvo.py:121-262  kp_selection / update_kp_data -> compute_pose_2d2d -> scale_recovery ->
                                           [compute_rigid_flow_kp -> 2nd pass] -> PnP fallback -> update_global_pose
    update_data           dfvo.py:264-287

With the unmodified driver available (CPU container) test_dropin_driver.py runs the real file; the golden trajectories were
produced by the real file too.  `hooks` lets a test observe / replace network outputs the way oracle/seqdata.py does for the
real driver."""
import copy

import cv2
import numpy as np

from oracle import vo


class SequenceDriver:
    def __init__(self, cfg, K, frames, hooks=None):
        from libs.deep_models.deep_models import DeepModel
        from libs.geometry.camera_modules import SE3, Intrinsics
        from libs.matching.keypoint_sampler import KeypointSampler
        from libs.tracker import EssTracker, PnpTracker
        self.SE3 = SE3
        self.cfg, self.frames, self.hooks = cfg, frames, hooks or {}
        cam = Intrinsics(K)
        self.e_tracker = EssTracker(cfg, cam, None)
        self.pnp_tracker = PnpTracker(cfg, cam)
        self.kp_sampler = KeypointSampler(cfg)
        self.deep_models = DeepModel(cfg)
        self.deep_models.initialize_models()
        self.ref, self.cur = {}, {}
        self.global_poses = {}
        self.modes = {}
        self.stage = 0

    # dfvo.py:299-345
    def infer(self):
        c, cur, ref = self.cfg, self.cur, self.ref
        raw = self.deep_models.forward_depth(imgs=[cur["img"]])
        if "depth" in self.hooks:
            raw = self.hooks["depth"](cur["id"], raw)
        raw = cv2.resize(raw, (c.image.width, c.image.height), interpolation=cv2.INTER_NEAREST)
        cur["raw_depth"] = raw
        cur["depth"] = vo.preprocess_depth(raw, c.crop.depth_crop, [c.depth.min_depth, c.depth.max_depth])      # utils.py:89-114
        if self.stage >= 1:
            flows = self.deep_models.forward_flow(cur, ref, forward_backward=c.deep_flow.forward_backward)
            if "flow" in self.hooks:
                self.hooks["flow"](cur["id"], ref["id"], flows)
            ref["flow"] = flows[(ref["id"], cur["id"])].copy()
            cur["flow"] = flows[(cur["id"], ref["id"])].copy()
            ref["flow_diff"] = flows[(ref["id"], cur["id"], "diff")].copy()

    def chain(self, pose):                                                      # update_global_pose, dfvo.py:109-119
        g = self.cur["pose"]
        g.t = g.R @ pose.t + g.t
        g.R = g.R @ pose.R
        self.global_poses[self.cur["id"]] = copy.deepcopy(g)

    # dfvo.py:121-262, tracking_method == 'hybrid'
    def track(self):
        c, cur, ref, SE3 = self.cfg, self.cur, self.ref, self.SE3
        if self.stage == 0:
            cur["pose"] = SE3()
            ref["motion"] = SE3()
            self.global_poses[cur["id"]] = copy.deepcopy(cur["pose"])
            return
        sel = self.kp_sampler.kp_selection(cur, ref)
        if sel["good_kp_found"]:
            self.kp_sampler.update_kp_data(cur, ref, sel)
        hybrid, E_pose = SE3(), SE3()
        if not sel["good_kp_found"]:
            self.modes[cur["id"]] = "const"
            self.chain(ref["motion"])
            return
        out = self.e_tracker.compute_pose_2d2d(ref[c.e_tracker.kp_src], cur[c.e_tracker.kp_src], not c.e_tracker.iterative_kp.enable)
        E_pose = out["pose"]
        hybrid.R = E_pose.R
        ref["inliers"] = out["inliers"]
        scale = None
        self.modes[cur["id"]] = "E"
        if np.linalg.norm(E_pose.t) != 0:
            so = self.e_tracker.scale_recovery(cur, ref, E_pose, False)
            scale = so["scale"]
            if c.scale_recovery.kp_src == "kp_depth":
                cur["kp_depth"], ref["kp_depth"], cur["rigid_flow_mask"] = so["cur_kp_depth"], so["ref_kp_depth"], so["rigid_flow_mask"]
            if scale != -1:
                hybrid.t = E_pose.t * scale
        if np.linalg.norm(E_pose.t) != 0 and c.e_tracker.iterative_kp.enable:
            self.e_tracker.compute_rigid_flow_kp(cur, ref, hybrid)
            out = self.e_tracker.compute_pose_2d2d(ref[c.e_tracker.iterative_kp.kp_src], cur[c.e_tracker.iterative_kp.kp_src], True)
            E_pose = out["pose"]
            hybrid.R = E_pose.R
            ref["inliers"] = out["inliers"]
            if np.linalg.norm(E_pose.t) != 0 and c.scale_recovery.iterative_kp.enable:
                so = self.e_tracker.scale_recovery(cur, ref, E_pose, True)
                scale = so["scale"]
                if scale != -1:
                    hybrid.t = E_pose.t * scale
            else:
                hybrid.t = E_pose.t * scale
        if np.linalg.norm(E_pose.t) == 0 or scale == -1:
            pn = self.pnp_tracker.compute_pose_3d2d(ref[c.pnp_tracker.kp_src], cur[c.pnp_tracker.kp_src], ref["depth"],
                                                    not c.pnp_tracker.iterative_kp.enable)
            if c.pnp_tracker.iterative_kp.enable:
                self.pnp_tracker.compute_rigid_flow_kp(cur, ref, pn["pose"])
                pn = self.pnp_tracker.compute_pose_3d2d(ref[c.pnp_tracker.iterative_kp.kp_src], cur[c.pnp_tracker.iterative_kp.kp_src],
                                                        ref["depth"], True)
            hybrid = pn["pose"]
            self.modes[cur["id"]] = "PnP"
        ref["pose"] = copy.deepcopy(hybrid)
        ref["motion"] = copy.deepcopy(hybrid)
        self.chain(ref["pose"])

    def run(self):
        for i, img in enumerate(self.frames):
            self.cur["id"], self.cur["timestamp"], self.cur["img"] = i, i, img
            self.infer()
            self.track()
            for k in self.cur:                                                  # update_data, dfvo.py:264-287
                self.ref[k] = self.cur[k]
            self.ref["flow"] = None
            self.cur["flow"] = None
            self.ref["flow_diff"] = None
            self.stage += 1
        return np.stack([self.global_poses[i].pose for i in range(len(self.frames))])
