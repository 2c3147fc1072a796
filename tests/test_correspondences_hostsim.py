"""CPU (host-emulation build): the correspondence-selection ablations -- local best-N scored by flow_ratio, global best-N and
uniformly sampled keypoints -- against the reference KeypointSampler's goldens, and the libs mirror / FramePipeline / SequenceBatch
against the unmodified driver's goldens."""
import os
import sys

import numpy as np
import pytest

import correspondences_cases as cc
import tracking_modes_cases as tm

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim"))

KINDS = list(cc.DRIVER_CFGS)


@pytest.fixture
def rt(hostsim_lib):
    from runtime import HostsimRuntime
    from b200 import runtime as rt_mod
    r = HostsimRuntime(hostsim_lib)
    rt_mod.set_runtime(r)
    return r


@pytest.fixture
def eng(rt):
    from b200 import tracking
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


@pytest.mark.parametrize("kind", KINDS)
def test_mirror_driver_matches_reference_driver(rt, kind):
    poses, _ = cc.run_mirror_driver(kind, rt)
    tm.check_against_driver_golden(kind, poses)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("mode", ["in_order", "pipelined", "tracker_thread"])
def test_pipeline_matches_reference_driver(rt, kind, mode):
    """FramePipeline: the driver golden, and the same per-frame branch as the mirror driver."""
    poses, modes, _ = cc.run_pipeline(kind, mode, runtime=rt)
    tm.check_against_driver_golden(kind, poses)
    _, mirror_modes = cc.run_mirror_driver(kind, rt)
    assert modes[1:] == mirror_modes[1:], (modes, mirror_modes)


def test_mixed_sources_run_stepwise_and_match_mirror(rt, monkeypatch):
    """E-tracker on local best-N, scale recovery on the sampled list: every E frame goes through track_stepwise with the scale set
    passed separately, and the poses and branches match the mirror driver's."""
    from b200 import pipeline
    calls = {"stepwise": 0, "fused": 0}
    stepwise, fused = pipeline.FramePipeline.track_stepwise, pipeline.FramePipeline.track_fused_launch

    def spy_stepwise(self, *a, **k):
        calls["stepwise"] += 1
        assert a[5] is not None, "the scale set is passed separately"
        return stepwise(self, *a, **k)

    def spy_fused(self, *a, **k):
        calls["fused"] += 1
        return fused(self, *a, **k)
    monkeypatch.setattr(pipeline.FramePipeline, "track_stepwise", spy_stepwise)
    monkeypatch.setattr(pipeline.FramePipeline, "track_fused_launch", spy_fused)
    poses, modes, _ = cc.run_pipeline("mixed", "in_order", runtime=rt)
    assert calls["fused"] == 0 and calls["stepwise"] == sum(m in ("E", "PnP") for m in modes[1:])
    want, want_modes = cc.run_mirror_driver("mixed", rt)
    assert modes[1:] == want_modes[1:], (modes, want_modes)
    for t in range(poses.shape[0]):
        assert np.abs(poses[t] - want[t]).max() < 1e-6 * max(1.0, np.linalg.norm(want[t][:3, 3])), t


def test_sequence_batch_uniform_equals_pipelines(hostsim_lib, monkeypatch):
    """SequenceBatch of the uniform configuration: every slot gets exactly the poses and branches of an independent pipeline
    (test_multiseq_hostsim.py's harness, with the uniform configuration)."""
    import test_multiseq_hostsim as ms
    monkeypatch.setattr(ms, "_cfg", lambda name: cc.pipeline_cfg("uniform", ms.H, ms.W))
    rt = ms._hostsim_rt(hostsim_lib)
    b = ms._analytic_batch(rt, ms._cfg("uniform"), ms.KS, False, ms.ORDERS, ms.SEEDS)
    ms._run(b, [[True] * 3] * len(ms.ORDERS[0]), False)
    for s in range(3):
        poses, modes = ms._independent(rt, "uniform-correspondences", ms.KS[s], ms.ORDERS[s], ms.SEEDS[s])
        ms._assert_same(b.poses[s], b.modes[s], poses, modes)


@pytest.mark.parametrize("over", cc.REFUSED)
def test_pipeline_refuses_unproduced_sources_and_unknown_scores(rt, over):
    import dropin_cases as dc
    from b200 import pipeline
    with pytest.raises(ValueError):
        pipeline.FramePipeline([60, 40, 100, 100], 80, 120, cfg=dc.make_cfg(80, 120, over), runtime=rt)


@pytest.mark.parametrize("over", [cc.MIXED_CFG, cc.DRIVER_CFGS["flowratio"], cc.DRIVER_CFGS["uniform"], cc.DRIVER_CFGS["bestn"],
                                  dict(cc.DRIVER_CFGS["uniform"], tracking_method="PnP")])
def test_pipeline_accepts_the_correspondence_configurations(rt, over):
    import dropin_cases as dc
    from b200 import pipeline
    pipeline.FramePipeline([60, 40, 100, 100], 80, 120, cfg=dc.make_cfg(80, 120, over), runtime=rt)
