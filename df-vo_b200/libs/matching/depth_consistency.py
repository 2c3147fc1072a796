"""``DepthConsistency`` (libs/matching/depth_consistency.py) on the device: the PoseNet depth-consistency map of
kp_selection.depth_consistency, one fused kernel (csrc/geometry.cu: k_depth_consistency)."""
import numpy as np

from b200 import runtime, tracking


class DepthConsistency:
    def __init__(self, cfg, cam_intrinsics):
        self.cfg = cfg
        self.cam_intrinsics = cam_intrinsics

    def compute(self, cur_data, ref_data):
        """depth_consistency.py:153-163: sets ``ref_data['depth_diff']`` [H,W] (a device-backed ``DevArray``) from the raw depths of
        both frames and ``ref_data['deep_pose']`` (float32 4x4)."""
        eng = tracking.default_engine()
        rt = runtime.get()

        def dev(x):
            return x.dev if isinstance(x, tracking.DevArray) else rt.from_host(np.ascontiguousarray(x, np.float32))

        T = rt.from_host(np.ascontiguousarray(ref_data["deep_pose"], np.float32).reshape(4, 4))
        out = eng.depth_consistency(dev(cur_data["raw_depth"]), dev(ref_data["raw_depth"]), T, self.cam_intrinsics.mat,
                                    self.cam_intrinsics.inv_mat)
        ref_data["depth_diff"] = tracking.DevArray(out, (eng.H, eng.W))
