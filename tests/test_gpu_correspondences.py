"""GPU: the correspondence-selection ablations on the device -- local best-N scored by flow_ratio, global best-N and uniformly
sampled keypoints against the reference KeypointSampler's goldens, FramePipeline in every execution mode against the in-order
pipeline and the unmodified driver's goldens, and the uniform path's device->host reads."""
import numpy as np
import pytest

import correspondences_cases as cc
import tracking_modes_cases as tm
from b200 import runtime as rt_mod, tracking

pytestmark = pytest.mark.gpu
KINDS = list(cc.DRIVER_CFGS)


@pytest.fixture
def rt(dev_lib):
    r = rt_mod.CudaRuntime(0)
    rt_mod.set_runtime(r)
    return r


@pytest.fixture
def eng(rt):
    return tracking.Engine(cc.H, cc.W, rt)


@pytest.mark.parametrize("name", list(cc.CASES))
def test_flow_ratio_matches_reference(eng, name):
    cc.check_flow_ratio(eng, name)


def test_flow_ratio_case1_counts_raw_flow_diff(eng):
    cc.check_flow_ratio_case1_counts_raw_diff(eng)


@pytest.mark.parametrize("name", ["easy", "zero_patch"])
def test_bestn_matches_reference(eng, name):
    cc.check_bestn(eng, name)


def test_sampled_keypoints_match_reference(eng):
    cc.check_sampled(eng)


@pytest.mark.parametrize("kind", KINDS + ["mixed"])
def test_pipeline_modes_equal_in_order(rt, kind):
    ref, ref_modes, _ = cc.run_pipeline(kind, "in_order", runtime=rt)
    if kind != "mixed":
        tm.check_against_driver_golden(kind, ref)
    for mode in tm.MODES:
        if mode == "in_order":
            continue
        poses, modes, _ = cc.run_pipeline(kind, mode, runtime=rt)
        rt.torch.cuda.synchronize()
        assert np.array_equal(poses, ref), (kind, mode)
        assert modes == ref_modes, (kind, mode, modes, ref_modes)


def test_uniform_path_reads_no_dense_map(rt):
    """Per tracked frame of the uniform configuration no device->host read is as large as one [H, W] map: the keypoints are
    gathered on the device and the tracker reads only its packed results."""
    g = cc.driver_golden("uniform")
    h, w = [int(v) for v in g["hw"]]
    np.random.seed(4869)
    p = tm.injected_pipeline_class()(list(g["K"]), h, w, cfg=cc.pipeline_cfg("uniform", h, w), runtime=rt)
    sizes = []
    orig = rt.to_host

    def to_host(buf):
        sizes.append(int(buf.size))
        return orig(buf)
    for t in range(g["poses"].shape[0]):
        cur = p.infer(None, t)
        p.stage += 1
        rt.torch.cuda.synchronize()
        rt.to_host = to_host
        try:
            p._advance(cur, p.ref)
        finally:
            rt.to_host = orig
        p.ref = cur
    assert sizes and max(sizes) < h * w, sizes
    tm.check_against_driver_golden("uniform", np.stack([p.poses[i] for i in range(g["poses"].shape[0])]))
