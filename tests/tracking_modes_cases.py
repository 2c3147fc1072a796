"""Shared by the CPU (host-emulation) and GPU tests of the PnP-only and flow-validity tracking configurations
(ablation_tracker_pnp.yml, ablation_model_sel_flow.yml): golden scenes, the class-level checks and the pipeline harness."""
import os

import numpy as np

from oracle import gen_golden_tracking_modes as ggt, seqdata, synth

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = ggt.TRACKING_MODE_CASES
FLOW_THRE = 5.0
H, W = 376, 1241


def golden():
    return np.load(os.path.join(G, "tracking_modes_2000.npz"))


def scene(name):
    return ggt.tracking_mode_scene(**CASES[name])


def rng_position():
    """(state pos, next draw) of the global generator, as the goldens store it (the draw advances the generator)."""
    pos = np.random.get_state()[2]
    return pos, np.random.randint(0, 2 ** 31 - 1)


def flow_cfg():
    from b200 import config
    cfg = config.default_cfg(H, W)
    cfg.e_tracker.validity = config.AttrDict(method="flow", thre=FLOW_THRE)
    return cfg


def check_ess_flow(eng, name):
    """The mirror's EssTracker (validity 'flow') on a golden scene: pose 1e-12, inlier mask equal, generator position equal."""
    from libs.geometry.camera_modules import Intrinsics
    from libs.tracker.E_tracker import EssTracker
    from b200 import tracking
    g = golden()
    kp_ref, kp_cur, _ = scene(name)
    tracking._default_engine = eng
    ess = EssTracker(flow_cfg(), Intrinsics(synth.kitti_intrinsics(H, W)), None)
    np.random.seed(4869)
    r = ess.compute_pose_2d2d(kp_ref, kp_cur, True)
    pos, after = rng_position()
    assert np.abs(r["pose"].pose - g[name + "_E_pose"]).max() < 1e-12, name
    assert np.array_equal(r["inliers"], g[name + "_E_inliers"]), name
    assert pos == int(g[name + "_E_rng_pos"]) and after == int(g[name + "_E_rng_after"]), name


def check_pnp_tail(eng, name):
    """Engine.pnp_tail_launch/_finish (the fused PnP tracker) on a golden scene against the reference PnpTracker: pose, kept
    keypoints, generator position; and bit-equal to the stepwise host-filter path (tracking.compute_pose_3d2d)."""
    from b200 import config, tracking
    g = golden()
    kp_ref, kp_cur, depth = scene(name)
    depth_proc = (depth * ((depth < 50) & (depth > 0))).astype(np.float32)
    K = synth.kitti_intrinsics(H, W)
    c = config.default_cfg(H, W)
    rt = eng.rt
    kb1, kb2, db = rt.from_host(kp_ref), rt.from_host(kp_cur), rt.from_host(depth_proc)
    np.random.seed(4869)
    tok = eng.pnp_tail_launch(kb1, kb2, kp_ref.shape[0], db, K, c.depth.min_depth, c.depth.max_depth, np.random)
    pose, _, m = eng.pnp_tail_finish(tok)
    pos, after = rng_position()
    # the device solvePnPRansac refines with its own Levenberg-Marquardt, so it meets OpenCV's pose to the tolerance of
    # tests/pnp_cases.py (observed ~1e-7), not to 1e-12; against the stepwise device path below it is bit-exact
    want = g[name + "_pnp_pose"]
    dR = pose[:3, :3].T @ want[:3, :3]
    ang = np.arccos(np.clip((np.trace(dR) - 1) / 2, -1, 1))
    assert ang < 1e-4 and np.linalg.norm(pose[:3, 3] - want[:3, 3]) < 1e-3, name
    assert m == int(g[name + "_pnp_nkp"]), name
    assert pos == int(g[name + "_pnp_rng_pos"]) and after == int(g[name + "_pnp_rng_after"]), name
    # the stepwise path: host filter + compute_pose_3d2d
    d = depth_proc[kp_ref[:, 1].astype(int), kp_ref[:, 0].astype(int)].astype(np.float64)
    keep = (kp_cur[:, 0] >= 0) & (kp_cur[:, 0] < W) & (kp_cur[:, 1] >= 0) & (kp_cur[:, 1] < H)
    keep &= (d != 0) & (d < c.depth.max_depth) & (d > c.depth.min_depth)
    np.random.seed(4869)
    want, _ = tracking.compute_pose_3d2d(eng, kp_ref[keep], kp_cur[keep], d[keep], K)
    assert np.array_equal(pose, want), name
    assert np.random.get_state()[2] == pos


def check_flow_mean(eng, name):
    """dfvo_flow_mean == np.mean(np.linalg.norm(kp_ref - kp_cur, axis=1)) bit for bit, and on the expected side of the gate."""
    kp_ref, kp_cur, _ = scene(name)
    rt = eng.rt
    m = eng.flow_mean(rt.from_host(kp_ref), rt.from_host(kp_cur), kp_ref.shape[0])
    want = np.mean(np.linalg.norm(kp_ref - kp_cur, axis=1))
    assert m == want, (name, m, want)
    assert m == float(golden()[name + "_flow_mean"])
    return m


def check_flow_mean_sizes(eng, sizes=(1, 7, 8, 9, 127, 128, 129, 255, 256, 1000, 2000, 4097)):
    rs = np.random.RandomState(3)
    rt = eng.rt
    for n in sizes:
        a, b = rs.uniform(0, 1241, (n, 2)), rs.uniform(0, 1241, (n, 2)) + rs.standard_normal((n, 2)) * 3
        m = eng.flow_mean(rt.from_host(a), rt.from_host(b), n)
        assert m == np.mean(np.linalg.norm(a - b, axis=1)), n


DRIVER_CFGS = {"pnp": {"tracking_method": "PnP"}, "flowsel": {"e_tracker.validity.method": "flow", "e_tracker.validity.thre": 5},
               "flowsel_gate": {"e_tracker.validity.method": "flow", "e_tracker.validity.thre": 8}}   # thre 8 closes the gate once


def pipeline_cfg(kind, h, w):
    from b200 import config
    cfg = config.default_cfg(h, w)
    if kind == "pnp":
        cfg.tracking_method = "PnP"
    elif kind.startswith("flowsel"):
        cfg.e_tracker.validity = config.AttrDict(method="flow", thre=DRIVER_CFGS[kind]["e_tracker.validity.thre"])
    return cfg


def injected_pipeline_class():
    """FramePipeline whose infer() feeds the analytic network outputs of the driver golden's sequence (oracle/seqdata.py)."""
    from b200 import pipeline

    class Injected(pipeline.FramePipeline):
        def infer(self, img, fid):
            h, w, K = self.H, self.W, self.K
            f = seqdata.frame_inputs(fid, h, w, K, seqdata.MODES[fid % len(seqdata.MODES)])
            st = pipeline.FrameState()
            st.id = fid
            slot = self.slot(fid)
            st.raw_depth = self._buf("raw%d" % slot, (h, w), np.float32)
            st.depth = self._buf("dep%d" % slot, (h, w), np.float32)
            d = self._buf("dsrc", (h, w), np.float32).upload(f["depth"])
            self.eng.depth_post(d, self.cfg.crop.depth_crop, 0.0, 50.0, st.raw_depth, st.depth)
            if not self.eng.flow_ready:
                self.eng.flow_fwd = self.rt.empty((1, 2, h, w), np.float32)
                self.eng.flow_bwd = self.rt.empty((1, 2, h, w), np.float32)
                self.eng.flow_diff = self.rt.empty((1, h, w), np.float32)
                self.eng.flow_ready = True
            st.fwd, st.bwd, st.diff = self.flow_slot(slot)
            st.fwd.upload(f["fwd"][None]); st.bwd.upload(f["bwd"][None]); st.diff.upload(f["diff"][None, :, :, 0])
            return st
    return Injected


MODES = {"in_order": dict(), "overlap": dict(overlap=True), "inflight2": dict(overlap=True, inflight=2),
         "inflight3": dict(overlap=True, inflight=3), "pipelined": dict(overlap=True, inflight=3, pipelined=True),
         "tracker_thread": dict(overlap=True, inflight=2, tracker_thread=True)}


def run_pipeline(kind, mode, runtime=None, n=None):
    """Runs the injected pipeline over the driver golden's sequence -> (global poses [n,4,4], per-frame branch, pipeline)."""
    g = np.load(os.path.join(G, "dfvo_driver_%s_188x620.npz" % kind))
    h, w = [int(v) for v in g["hw"]]
    K = list(g["K"])
    n = n or g["poses"].shape[0]
    np.random.seed(4869)
    p = injected_pipeline_class()(K, h, w, cfg=pipeline_cfg(kind, h, w), runtime=runtime, **MODES[mode])
    for _ in range(n):
        p.step(None)
    if p.overlap:
        p.flush()
    p.close()
    return np.stack([p.poses[i] for i in range(n)]), [p.modes[i] for i in range(n)], p


def check_against_driver_golden(kind, poses):
    g = np.load(os.path.join(G, "dfvo_driver_%s_188x620.npz" % kind))
    for t in range(poses.shape[0]):
        want = g["poses"][t]
        dR = poses[t][:3, :3].T @ want[:3, :3]
        ang = np.arccos(np.clip((np.trace(dR) - 1) / 2, -1, 1))
        dt = np.linalg.norm(poses[t][:3, 3] - want[:3, 3])
        assert ang < 1e-6 and dt < 1e-6 * max(1.0, np.linalg.norm(want[:3, 3])), (kind, t, ang, dt)


def pnp_sequence_driver_class():
    """tests/vo_driver.py's SequenceDriver with dfvo.py:121-262 for tracking_method 'PnP': selection as in hybrid mode, E_pose stays
    identity so the PnP tracker runs on every frame with good keypoints (the `or` of dfvo.py:227 never reads `scale`)."""
    import copy
    import vo_driver

    class PnPSequenceDriver(vo_driver.SequenceDriver):
        def track(self):
            c, cur, ref, SE3 = self.cfg, self.cur, self.ref, self.SE3
            if self.stage == 0:
                return super().track()
            sel = self.kp_sampler.kp_selection(cur, ref)
            if not sel["good_kp_found"]:
                self.modes[cur["id"]] = "const"
                self.chain(ref["motion"])
                return
            self.kp_sampler.update_kp_data(cur, ref, sel)
            pn = self.pnp_tracker.compute_pose_3d2d(ref[c.pnp_tracker.kp_src], cur[c.pnp_tracker.kp_src], ref["depth"],
                                                    not c.pnp_tracker.iterative_kp.enable)
            self.modes[cur["id"]] = "PnP"
            ref["pose"] = copy.deepcopy(pn["pose"])
            ref["motion"] = copy.deepcopy(pn["pose"])
            self.chain(ref["pose"])
    return PnPSequenceDriver


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
    g = np.load(os.path.join(G, "dfvo_driver_%s_188x620.npz" % kind))
    h, w = [int(v) for v in g["hw"]]
    n = g["poses"].shape[0]
    K = synthdata.kitti_intrinsics(h, w)
    cfg = dc.make_cfg(h, w, DRIVER_CFGS[kind])
    seqdata.patch_deep_model(dm.DeepModel, h, w, K)
    tracking.default_engine(h, w)
    frames = [synthdata.value_noise_image(h, w, 100 + i) for i in range(n)]
    np.random.seed(cfg.seed)
    cls = pnp_sequence_driver_class() if kind == "pnp" else vo_driver.SequenceDriver
    drv = cls(cfg, K, frames)
    orig = drv.infer

    def infer():
        drv.deep_models._t = drv.cur["id"]
        orig()
    drv.infer = infer
    poses = drv.run()
    return poses, [drv.modes.get(i) for i in range(n)]
