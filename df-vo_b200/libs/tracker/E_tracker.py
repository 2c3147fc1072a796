"""``EssTracker`` with the reference's interface (libs/tracker/E_tracker.py:129-705) on the dfvo_b200
kernels: five repeated essential-matrix RANSACs (replaying OpenCV's sampling sequence), GRIC or flow-magnitude
model selection, pose recovery, and scale recovery from triangulated-vs-CNN depth."""
import copy

import numpy as np

from b200 import tracking
from libs.geometry.camera_modules import SE3


def get_E_from_pose(pose):
    """E_tracker.py:102-127: E = [t]x R with t normalised."""
    R = pose.R
    t = pose.t / np.linalg.norm(pose.t)
    tx = np.array([[0, -t[2, 0], t[1, 0]], [t[2, 0], 0, -t[0, 0]], [-t[1, 0], t[0, 0], 0]])
    return tx @ R


class EssTracker:
    def __init__(self, cfg, cam_intrinsics, timers):
        self.cfg = cfg
        self.prev_scale = 0
        self.prev_pose = SE3()
        self.cam_intrinsics = cam_intrinsics
        self.timers = timers
        assert cfg.e_tracker.validity.method in ("GRIC", "flow"), "dfvo_b200 implements e_tracker.validity.method GRIC and flow"
        self.K = [float(cam_intrinsics.cx), float(cam_intrinsics.cy), float(cam_intrinsics.fx), float(cam_intrinsics.fy)]

    def compute_pose_2d2d(self, kp_ref, kp_cur, is_iterative):
        """E_tracker.py:154-307 -> {'pose': SE3 (cur -> ref, unit translation or identity), 'inliers': bool[N]}."""
        repeat = self.cfg.e_tracker.ransac.repeat if is_iterative else 3                 # :179
        r = tracking.compute_pose_2d2d(tracking.default_engine(), np.ascontiguousarray(kp_ref, np.float64),
                                       np.ascontiguousarray(kp_cur, np.float64), self.K, repeat=repeat,
                                       reproj_thre=self.cfg.e_tracker.ransac.reproj_thre, validity=self.cfg.e_tracker.validity.method,
                                       flow_thre=self.cfg.e_tracker.validity.get("thre"))
        pose = SE3()
        pose.R = r["R"]
        pose.t = r["t"]
        return {"pose": pose, "inliers": r["inliers"]}

    def scale_recovery(self, cur_data, ref_data, E_pose, is_iterative):
        """E_tracker.py:442-474."""
        outputs = {}
        if self.cfg.scale_recovery.method == "simple":
            scale = self.scale_recovery_simple(cur_data, ref_data, E_pose, is_iterative)
        elif self.cfg.scale_recovery.method == "iterative":
            it = self.scale_recovery_iterative(cur_data, ref_data, E_pose)
            scale = it["scale"]
            outputs["cur_kp_depth"], outputs["ref_kp_depth"], outputs["rigid_flow_mask"] = it["cur_kp"], it["ref_kp"], it["rigid_flow_mask"]
        else:
            assert False, "Wrong scale recovery method [{}] used.".format(self.cfg.scale_recovery.method)
        outputs["scale"] = scale
        return outputs

    def scale_recovery_simple(self, cur_data, ref_data, E_pose, is_iterative):
        """E_tracker.py:476-507."""
        src = self.cfg.scale_recovery.iterative_kp.kp_src if is_iterative else self.cfg.scale_recovery.kp_src
        return self.find_scale_from_depth(ref_data[src], cur_data[src], E_pose.inv_pose, cur_data["depth"])

    def find_scale_from_depth(self, kp1, kp2, T_21, depth2):
        """E_tracker.py:571-643."""
        c = self.cfg.scale_recovery.ransac
        assert c.method == "depth_ratio", "dfvo_b200 implements scale_recovery.ransac.method depth_ratio (the default)"
        return tracking.find_scale_from_depth(tracking.default_engine(), np.asarray(kp1, np.float64), np.asarray(kp2, np.float64),
                                              np.asarray(T_21, np.float64), np.asarray(depth2), self.K, c.min_samples,
                                              c.max_trials, c.stop_prob, c.thre)

    # ---- rigid-flow keypoints / iterative scale recovery (SURVEY 8f rank 1) ------------------------------------------
    def _dev(self, eng, arr, shape):
        """Device buffer of a per-frame map: the DeepModel mirror hands out device-backed arrays (tracking.DevArray); a plain
        ndarray (e.g. the driver's resized raw depth) is uploaded."""
        if isinstance(arr, tracking.DevArray):
            return arr.dev
        return eng.rt.from_host(np.ascontiguousarray(np.asarray(arr, np.float32).reshape(shape)))

    def kp_selection_good_depth(self, cur_data, ref_data, rigid_kp_score_method):
        """E_tracker.py:645-705: RigidFlow layer + optical-rigid flow difference + opt_rigid_flow_kp, on the device."""
        outputs = {}
        if not self.cfg.kp_selection.rigid_flow_kp.enable:
            return outputs
        h, w = np.shape(cur_data["depth"])
        eng = tracking.default_engine(h, w)
        rk = self.cfg.kp_selection.rigid_flow_kp
        o = eng.rigid_flow_keypoints(self._dev(eng, ref_data["raw_depth"], (h, w)), self._dev(eng, ref_data["flow"], (1, 2, h, w)),
                                     self._dev(eng, ref_data["flow_diff"], (1, h, w)), ref_data["rigid_flow_pose"].pose, self.K,
                                     rk.num_row, rk.num_col, rk.num_bestN, float(rk.rigid_flow_thre), float(rk.optical_flow_thre),
                                     rigid_kp_score_method)
        mask = tracking.DevArray(o["rigid_flow_diff"], (h, w))
        ref_data["rigid_flow_diff"] = tracking.DevArray(o["rigid_flow_diff"], (h, w, 1))
        outputs.update(kp1_depth=o["kp1_best"][None], kp2_depth=o["kp2_best"][None], kp1_depth_uniform=o["kp1_uniform"][None],
                       kp2_depth_uniform=o["kp2_uniform"][None], rigid_flow_mask=mask)
        return outputs

    def compute_rigid_flow_kp(self, cur_data, ref_data, pose):
        """E_tracker.py:421-440."""
        rigid_pose = copy.deepcopy(pose)
        ref_data["rigid_flow_pose"] = SE3(rigid_pose.inv_pose)
        k = self.kp_selection_good_depth(cur_data, ref_data, self.cfg.e_tracker.iterative_kp.score_method)
        ref_data["kp_depth"], cur_data["kp_depth"] = k["kp1_depth"][0], k["kp2_depth"][0]
        ref_data["kp_depth_uniform"], cur_data["kp_depth_uniform"] = k["kp1_depth_uniform"][0], k["kp2_depth_uniform"][0]
        cur_data["rigid_flow_mask"] = k["rigid_flow_mask"]

    def scale_recovery_iterative(self, cur_data, ref_data, E_pose):
        """E_tracker.py:509-569."""
        outputs = {}
        scale, delta = self.prev_scale, 0.001
        for _ in range(5):
            rigid_flow_pose = copy.deepcopy(E_pose)
            rigid_flow_pose.t *= scale
            ref_data["rigid_flow_pose"] = SE3(rigid_flow_pose.inv_pose)
            k = self.kp_selection_good_depth(cur_data, ref_data, self.cfg.scale_recovery.iterative_kp.score_method)
            ref_data["kp_depth"], cur_data["kp_depth"] = k["kp1_depth_uniform"][0], k["kp2_depth_uniform"][0]
            cur_data["rigid_flow_mask"] = k["rigid_flow_mask"]
            cur_kp, ref_kp = cur_data[self.cfg.scale_recovery.kp_src], ref_data[self.cfg.scale_recovery.kp_src]
            new_scale = self.find_scale_from_depth(ref_kp, cur_kp, E_pose.inv_pose, cur_data["depth"])
            delta_scale = np.abs(new_scale - scale)
            scale = new_scale
            self.prev_scale = new_scale
            outputs.update(scale=scale, cur_kp=cur_data["kp_depth"], ref_kp=ref_data["kp_depth"], rigid_flow_mask=cur_data["rigid_flow_mask"])
            if delta_scale < delta:
                return outputs
        return outputs
