"""CPU (host-emulation build): several sequences on one GPU.

* The batched monodepth2 / PoseNet runners (dfvo_*_build_batch / *_forward_batch) give, entry by entry, the bits of a batch-1
  runner on the same feed.
* multiseq.SequenceBatch gives every sequence exactly the poses and tracker branches of an independent FramePipeline on the same
  frames, in order and in overlap mode, for the tracking configurations the pipeline accepts; a slot fed the golden sequence
  reproduces the unmodified reference driver's trajectory; idle slots and reset behave like separate pipelines.
"""
import os
import sys

import numpy as np
import pytest

from oracle import seqdata, synth
from util import hptr

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim"))

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FH, FW = 64, 96                      # test_hostsim.py's monodepth2 feed size (deep_models_70x150.npz)
PRECS = {"fp32": 0, "bf16": 1, "tf32": 2}


def _feeds(n):
    return [np.random.RandomState(100 + i).uniform(0, 1, (1, 3, FH, FW)).astype(np.float32) for i in range(n)]


_single = {}


def _single_outputs(lib, prec):
    """Batch-1 depth of feeds 0..2 and batch-1 poses of the pairs (0,1), (1,2), (2,0)."""
    from b200 import native
    if prec not in _single:
        f = _feeds(3)
        enc, dec = synth.monodepth2_weights(4869, FH, FW)
        penc, pdec = synth.posenet_weights()
        ctx = native.Context(lib)
        ctx.load_weights(native.NET_MONODEPTH2, enc); ctx.load_weights(native.NET_MONODEPTH2, dec)
        ctx.load_weights(native.NET_POSENET, {k: v for k, v in penc.items() if k.startswith("encoder.")})
        ctx.load_weights(native.NET_POSENET, pdec)
        ctx.monodepth2_build(FH, FW, PRECS[prec])
        ctx.posenet_build(FH, FW, PRECS[prec], 5.4)
        depth, pose = [], []
        for i in range(3):
            d = np.zeros((FH, FW), np.float32)
            ctx.monodepth2_forward(hptr(f[i]), hptr(d))
            p = np.zeros((4, 4), np.float32)
            ctx.posenet_forward(hptr(f[i]), hptr(f[(i + 1) % 3]), hptr(p))
            depth.append(d); pose.append(p)
        _single[prec] = (f, depth, pose, enc, dec, penc, pdec)
    return _single[prec]


@pytest.mark.parametrize("prec", ["fp32", "tf32", "bf16"])
@pytest.mark.parametrize("B", [1, 2, 3])
def test_batched_depth_and_pose_equal_batch_one(hostsim_lib, B, prec):
    from b200 import native
    f, depth, pose, enc, dec, penc, pdec = _single_outputs(hostsim_lib, prec)
    ctx = native.Context(hostsim_lib)
    ctx.load_weights(native.NET_MONODEPTH2, enc); ctx.load_weights(native.NET_MONODEPTH2, dec)
    ctx.load_weights(native.NET_POSENET, {k: v for k, v in penc.items() if k.startswith("encoder.")})
    ctx.load_weights(native.NET_POSENET, pdec)
    ctx.monodepth2_build_batch(FH, FW, B, PRECS[prec])
    ctx.posenet_build_batch(FH, FW, B, PRECS[prec], 5.4)
    order = [2, 0, 1][:B]                                     # entry i reads feed order[i]: not the feeds' own order
    d = np.zeros((B, FH, FW), np.float32)
    ctx.monodepth2_forward_batch([f[i].ctypes.data for i in order], hptr(d))
    p = np.zeros((B, 4, 4), np.float32)
    ctx.posenet_forward_batch([a for i in order for a in (f[i].ctypes.data, f[(i + 1) % 3].ctypes.data)], hptr(p))
    for b, i in enumerate(order):
        assert np.array_equal(d[b], depth[i]), (b, i)
        assert np.array_equal(p[b], pose[i]), (b, i)
    assert np.all(np.isfinite(d)) and d.max() > 0
    # the batch is part of the plan: a forward over another number of entries is refused with DFVO_ESHAPE
    with pytest.raises(native.DfvoError, match="error -3: .*built for %d" % B):
        ctx.monodepth2_forward_batch([f[0].ctypes.data] * (B + 1), hptr(np.zeros((B + 1, FH, FW), np.float32)))
    with pytest.raises(native.DfvoError, match="error -3: .*built for %d" % B):
        ctx.posenet_forward_batch([f[0].ctypes.data] * (2 * B + 2), hptr(np.zeros((B + 1, 4, 4), np.float32)))


# ---------------------------------------------------------------------------------------------------------------------------
# SequenceBatch vs independent FramePipelines on analytic network outputs
# ---------------------------------------------------------------------------------------------------------------------------
# (each tracked frame costs seconds in the CPU emulation, so the sequences are short: every one has at least two tracked frames)
_golden = np.load(os.path.join(G, "dfvo_driver_188x620.npz"))
H, W = [int(v) for v in _golden["hw"]]
K0 = [float(v) for v in _golden["K"]]
N = _golden["poses"].shape[0]
# three sequences of analytic frames (seqdata.MODES: frame 3 is the still frame that forces the PnP fallback, 5 the blind one)
ORDERS = [[2, 3, 4], [6, 5, 1], [4, 0, 2]]
KS = [K0, [K0[0] + 2.0, K0[1] - 1.0, K0[2] * 1.01, K0[3] * 1.01], [K0[0] - 3.0, K0[1] + 2.0, K0[2] * 0.98, K0[3] * 0.98]]
SEEDS = [4869, 4876, 4883]
_inputs, _indep = {}, {}


def _frame(idx):
    if idx not in _inputs:
        _inputs[idx] = seqdata.frame_inputs(idx, H, W, K0, seqdata.MODES[idx % len(seqdata.MODES)])
    return _inputs[idx]


def _write_analytic(eng, st, f, scratch):
    """The analytic network outputs of a frame into its buffers (depth through the device post-processing, as
    test_pipeline_hostsim.py does it)."""
    eng.depth_post(scratch.upload(f["depth"]), [[0.3, 1], [0, 1]], 0.0, 50.0, st.raw_depth, st.depth)
    if st.fwd is not None:
        st.fwd.upload(f["fwd"][None]); st.bwd.upload(f["bwd"][None]); st.diff.upload(f["diff"][None, :, :, 0])


def _hostsim_rt(lib):
    from runtime import HostsimRuntime
    from b200 import runtime as rt_mod
    rt = HostsimRuntime(lib)
    rt_mod.set_runtime(rt)
    return rt


def _cfg(name):
    from b200 import config
    cfg = config.default_cfg(H, W)
    if name == "pnp":
        cfg.tracking_method = "PnP"
    elif name == "iterative":
        cfg.kp_selection.rigid_flow_kp.enable = True
        cfg.scale_recovery.method = "iterative"
    elif name == "flow_validity":
        cfg.e_tracker.validity.method = "flow"
        cfg.e_tracker.validity.thre = 5.0
    return cfg


def _analytic_batch(rt, cfg, Ks, overlap, frames_of, seeds):
    """A SequenceBatch whose network forwards are replaced by the analytic outputs of the frame each slot receives: the batched
    buffers and their per-sequence views, buffer slots, references, streams and trackers are the product's (LiteFlowNet at
    188x620 in the CPU emulation would take minutes per step; the batched networks have their own tests above and on the GPU).
    frames_of[s]: the analytic frame indices of sequence s, in the order its frames arrive."""
    from b200 import multiseq
    scratch = rt.empty((H, W), np.float32)

    class Analytic(multiseq.SequenceBatch):
        def load_weights(self):                               # the batched buffers only: no network is built
            self.eng.feed_h, self.eng.feed_w = 64, 96
            self._alloc_buffers()

        def _networks(self, curs, refs, out):
            for s, st in enumerate(curs):
                if st is not None:
                    _write_analytic(self.eng, st, _frame(self.frames_of[s][st.id]), scratch)

    b = Analytic(Ks, H, W, cfg=cfg, overlap=overlap, runtime=rt, rngs=[np.random.RandomState(v) for v in seeds])
    b.frames_of = [list(f) for f in frames_of]
    b.load_weights()
    return b


def _independent(rt, cfg_name, K, frames, seed):
    """(poses, modes) of an in-order FramePipeline fed the analytic frames `frames` (cached: the same run serves several tests)."""
    key = (cfg_name, tuple(K), tuple(frames), seed)
    if key in _indep:
        return _indep[key]
    from b200 import pipeline
    scratch = rt.empty((H, W), np.float32)

    class Injected(pipeline.FramePipeline):
        def infer(self, img, fid):
            st = pipeline.FrameState()
            st.id = fid
            slot = self.slot(fid)
            st.raw_depth = self._buf("raw%d" % slot, (H, W), np.float32)
            st.depth = self._buf("dep%d" % slot, (H, W), np.float32)
            if self.ref is not None:
                st.fwd = self._buf("ffwd%d" % slot, (1, 2, H, W), np.float32)
                st.bwd = self._buf("fbwd%d" % slot, (1, 2, H, W), np.float32)
                st.diff = self._buf("fdif%d" % slot, (1, H, W), np.float32)
            _write_analytic(self.eng, st, _frame(frames[fid]), scratch)
            return st

    p = Injected(K, H, W, cfg=_cfg(cfg_name), runtime=rt, rng=np.random.RandomState(seed))
    for _ in frames:
        p.step(None)
    _indep[key] = (dict(p.poses), dict(p.modes))
    return _indep[key]


def _run(b, schedule, overlap):
    """schedule: per step, per slot: True (a frame) / False (idle).  Returns the S-pose lists of step (and flush)."""
    dummy = np.zeros((H, W, 3), np.uint8)
    out = [b.step([dummy if a else None for a in row]) for row in schedule]
    if overlap:
        out.append(b.flush())
    return out


def _assert_same(poses_a, modes_a, poses_b, modes_b):
    assert sorted(poses_a) == sorted(poses_b)
    for f in poses_b:
        assert np.array_equal(poses_a[f], poses_b[f]), f
    assert modes_a == modes_b


@pytest.mark.parametrize("cfg_name", ["default", "pnp", "iterative", "flow_validity"])
@pytest.mark.parametrize("overlap", [False, True])
def test_sequence_batch_equals_independent_pipelines(hostsim_lib, overlap, cfg_name):
    rt = _hostsim_rt(hostsim_lib)
    b = _analytic_batch(rt, _cfg(cfg_name), KS, overlap, ORDERS, SEEDS)
    n = len(ORDERS[0])
    res = _run(b, [[True] * 3] * n, overlap)
    if overlap:                                               # step t returns the poses of step t-1, flush() the last ones
        assert res[0] == [None] * 3
        res = res[1:]
    modes = set()
    for s in range(3):
        for t in range(n):
            assert np.array_equal(res[t][s], b.poses[s][t]), (t, s)
        poses, m = _independent(rt, cfg_name, KS[s], ORDERS[s], SEEDS[s])
        _assert_same(b.poses[s], b.modes[s], poses, m)
        modes |= set(m.values())
    if cfg_name == "default":
        assert {"E", "PnP"} <= modes                          # the still frame forces the PnP fallback


def test_golden_slot_reproduces_reference_driver(hostsim_lib):
    """Slot 1 carries the golden sequence with RandomState(4869) (= the driver's np.random.seed(4869)) while slots 0 and 2 carry
    two-frame sequences and then idle: slot 1's trajectory is the unmodified driver's, to test_pipeline_hostsim.py's tolerance."""
    rt = _hostsim_rt(hostsim_lib)
    b = _analytic_batch(rt, _cfg("default"), [KS[1], K0, KS[2]], False, [ORDERS[1], list(range(N)), ORDERS[2]], [1, 4869, 2])
    _run(b, [[t < 2, True, t < 2] for t in range(N)], False)
    assert sorted(b.poses[0]) == [0, 1] and sorted(b.poses[2]) == [0, 1]
    for t in range(N):
        pose, want = b.poses[1][t], _golden["poses"][t]
        dR = pose[:3, :3].T @ want[:3, :3]
        ang = np.arccos(np.clip((np.trace(dR) - 1) / 2, -1, 1))
        dt = np.linalg.norm(pose[:3, 3] - want[:3, 3])
        assert ang < 1e-6 and dt < 1e-6 * max(1.0, np.linalg.norm(want[:3, 3])), (t, ang, dt)


@pytest.mark.parametrize("overlap", [False, True])
def test_idle_slots_and_reset(hostsim_lib, overlap):
    """Slot 0 idles in steps 1 and 4; slot 1 runs two frames, is reset to a new sequence (other K, generator and frames) and
    runs three more; slot 2 starts in step 2 and idles in step 3.  Every sequence's poses and branches equal an independent
    pipeline's on the frames it received, and reset returns the finished sequence's poses."""
    rt = _hostsim_rt(hostsim_lib)
    new1 = [0, 3, 6]
    b = _analytic_batch(rt, _cfg("default"), KS, overlap, ORDERS, SEEDS)
    got = _run(b, [[True, True, False], [False, True, False]], False)       # (overlap: the second step returns the first's poses)
    assert got[1][2] is None and (got[1][0] is None) != overlap
    old = b.reset(1, K=KS[2], rng=np.random.RandomState(99))
    b.frames_of[1] = new1
    poses, _ = _independent(rt, "default", KS[1], ORDERS[1][:2], SEEDS[1])
    assert sorted(old) == [0, 1] and all(np.array_equal(old[f], poses[f]) for f in poses)
    _run(b, [[True, True, True], [True, True, False], [False, True, True]], overlap)
    for s, (K, frames, seed) in enumerate([(KS[0], ORDERS[0], SEEDS[0]), (KS[2], new1, 99), (KS[2], ORDERS[2][:2], SEEDS[2])]):
        _assert_same(b.poses[s], b.modes[s], *_independent(rt, "default", K, frames, seed))


def test_bad_input_raises(hostsim_lib):
    from b200 import multiseq
    rt = _hostsim_rt(hostsim_lib)
    b = _analytic_batch(rt, _cfg("default"), KS, False, ORDERS, SEEDS)
    ok = np.zeros((H, W, 3), np.uint8)
    with pytest.raises(ValueError, match="3 sequences"):
        b.step([ok, ok])
    with pytest.raises(ValueError, match="shape"):
        b.step([ok, np.zeros((H, W + 1, 3), np.uint8), None])
    for bad in (3, -1):
        with pytest.raises(IndexError):
            b.reset(bad)
    with pytest.raises(ValueError):
        multiseq.SequenceBatch([], H, W, runtime=rt)
    with pytest.raises(ValueError, match="generators"):
        multiseq.SequenceBatch(KS, H, W, runtime=rt, rngs=[np.random.RandomState(0)])
    assert b.stage == 0 and b._nframes == [0, 0, 0]               # rejected steps advance nothing
