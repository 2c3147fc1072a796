"""CPU (host-emulation build): the depth-consistency branch (deep_pose + kp_selection.depth_consistency) end to end against the
unmodified reference driver's golden (tests/golden/dfvo_driver_depthcons_188x620.npz, oracle/gen_golden_depth_consistency.py):
the libs mirror through the driver's call sequence and FramePipeline in every execution mode, with the PoseNet's output replaced by
the golden's analytic pose."""
import os
import sys

import numpy as np
import pytest

import tracking_modes_cases as tm
from oracle import gen_golden_depth_consistency as gen

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim"))

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GOLDEN = os.path.join(G, "dfvo_driver_depthcons_188x620.npz")


def check(poses):
    g = np.load(GOLDEN)
    for t in range(poses.shape[0]):
        want = g["poses"][t]
        dR = poses[t][:3, :3].T @ want[:3, :3]
        ang = np.arccos(np.clip((np.trace(dR) - 1) / 2, -1, 1))
        dt = np.linalg.norm(poses[t][:3, 3] - want[:3, 3])
        assert ang < 1e-6 and dt < 1e-6 * max(1.0, np.linalg.norm(want[:3, 3])), (t, ang, dt)


def run_mirror(runtime):
    """tests/vo_driver.py's call sequence plus dfvo.py:84 (DepthConsistency), :338-345 (forward_pose) and :142-143 (compute)."""
    import dropin_cases as dc
    import synthdata
    import vo_driver
    from b200 import runtime as rt_mod, tracking
    from oracle import seqdata
    rt_mod.set_runtime(runtime)
    tracking._default_engine = None
    dc.fresh_libs()
    import libs.deep_models.deep_models as dm
    from libs.geometry.camera_modules import Intrinsics
    from libs.matching.depth_consistency import DepthConsistency
    g = np.load(GOLDEN)
    h, w = [int(v) for v in g["hw"]]
    n = g["poses"].shape[0]
    K = synthdata.kitti_intrinsics(h, w)
    cfg = dc.make_cfg(h, w, gen.DRIVER_CFG)
    seqdata.patch_deep_model(dm.DeepModel, h, w, K)
    dm.DeepModel.forward_pose = lambda self, imgs: gen.analytic_deep_pose(self._t, h, w, K)
    tracking.default_engine(h, w)

    class Driver(vo_driver.SequenceDriver):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            self.dc = DepthConsistency(cfg, Intrinsics(K))

        def infer(self):
            self.deep_models._t = self.cur["id"]
            super().infer()
            if self.stage >= 1:
                self.ref["deep_pose"] = self.deep_models.forward_pose([self.ref["img"], self.cur["img"]])

        def track(self):
            if self.stage >= 1:
                self.dc.compute(self.cur, self.ref)
            super().track()

    frames = [synthdata.value_noise_image(h, w, 100 + i) for i in range(n)]
    np.random.seed(cfg.seed)
    drv = Driver(cfg, K, frames)
    poses = drv.run()
    return poses, np.random.get_state()[2]


def injected_class():
    from b200 import pipeline  # noqa: F401

    class Injected(tm.injected_pipeline_class()):
        def infer(self, img, fid):
            st = super().infer(img, fid)
            if fid > 0:
                st.deep_pose = self._buf("dpose%d" % self.slot(fid), (4, 4), np.float32).upload(gen.analytic_deep_pose(fid, self.H, self.W, self.K))
            return st
    return Injected


def run_pipeline(mode, runtime):
    from b200 import config
    g = np.load(GOLDEN)
    h, w = [int(v) for v in g["hw"]]
    n = g["poses"].shape[0]
    cfg = config.default_cfg(h, w)
    cfg.deep_pose.enable = True
    cfg.kp_selection.depth_consistency.enable = True
    np.random.seed(4869)
    p = injected_class()(list(g["K"]), h, w, cfg=cfg, runtime=runtime, **tm.MODES[mode])
    for _ in range(n):
        p.step(None)
    if p.overlap:
        p.flush()
    p.close()
    return np.stack([p.poses[i] for i in range(n)]), np.random.get_state()[2]


def test_mirror_driver_matches_reference_driver(hostsim_lib):
    from runtime import HostsimRuntime
    poses, _ = run_mirror(HostsimRuntime(hostsim_lib))
    check(poses)


def test_pipeline_matches_reference_driver_in_every_mode(hostsim_lib):
    from runtime import HostsimRuntime
    from b200 import runtime as rt_mod
    rt = HostsimRuntime(hostsim_lib)
    rt_mod.set_runtime(rt)
    base, pos = run_pipeline("in_order", rt)
    check(base)
    _, mirror_pos = run_mirror(rt)
    assert pos == mirror_pos                                   # same generator position as the mirror driver
    for mode in ("overlap", "inflight2", "inflight3", "pipelined", "tracker_thread"):
        rt_mod.set_runtime(rt)
        poses, p2 = run_pipeline(mode, rt)
        assert np.array_equal(poses, base) and p2 == pos, mode


def test_pipeline_refuses_depth_consistency_without_deep_pose(hostsim_lib):
    import dropin_cases as dc
    from runtime import HostsimRuntime
    from b200 import pipeline, runtime as rt_mod
    rt = HostsimRuntime(hostsim_lib)
    rt_mod.set_runtime(rt)
    with pytest.raises(ValueError):
        pipeline.FramePipeline([60, 40, 100, 100], 80, 120, cfg=dc.make_cfg(80, 120, {"kp_selection.depth_consistency.enable": True}),
                               runtime=rt)
