"""CPU (host-emulation build): the PnP-only and flow-validity tracking configurations of the reference (ablation_tracker_pnp.yml,
ablation_model_sel_flow.yml) -- the two device tails against class-level goldens of the reference trackers, the flow gate's mean
bit-equal to NumPy, and the libs mirror / FramePipeline against the unmodified driver's goldens."""
import os
import sys

import numpy as np
import pytest

import tracking_modes_cases as tm

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim"))


@pytest.fixture
def eng(hostsim_lib):
    from runtime import HostsimRuntime
    from b200 import runtime as rt_mod, tracking
    rt = HostsimRuntime(hostsim_lib)
    rt_mod.set_runtime(rt)
    return tracking.Engine(tm.H, tm.W, rt)


@pytest.mark.parametrize("name", list(tm.CASES))
def test_flow_tail_matches_reference_ess_tracker(eng, name):
    import dropin_cases as dc
    dc.fresh_libs()
    tm.check_ess_flow(eng, name)


@pytest.mark.parametrize("name", list(tm.CASES))
def test_pnp_tail_matches_reference_pnp_tracker(eng, name):
    tm.check_pnp_tail(eng, name)


def test_flow_gate_mean_bit_equal_both_sides(eng):
    means = {name: tm.check_flow_mean(eng, name) for name in tm.CASES}
    assert means["still"] <= tm.FLOW_THRE < means["moving"]
    tm.check_flow_mean_sizes(eng)


def test_flow_gate_mean_rides_on_selection_status(eng):
    """select_local_bestn(with_flow_mean=True): good / n / mean from one packed read, the mean bit-equal to NumPy."""
    from oracle import synth
    fr = synth.analytic_frame(h=tm.H, w=tm.W, seed=21)
    rt = eng.rt
    fwd = rt.from_host(np.ascontiguousarray(fr["flow_fwd"][None], np.float32))
    diff = rt.from_host(np.ascontiguousarray(fr["flow_diff"][None, :, :, 0], np.float32))
    good, n, kp1, kp2, mean = eng.select_local_bestn(diff, fwd, 10, 10, 2000, 0.1, with_flow_mean=True)
    good0, n0, _, _ = eng.select_local_bestn(diff, fwd, 10, 10, 2000, 0.1)
    assert good == good0 and n == n0 and n > 100
    assert mean == np.mean(np.linalg.norm(kp1.numpy()[:n] - kp2.numpy()[:n], axis=1))


@pytest.mark.parametrize("kind", ["pnp", "flowsel", "flowsel_gate"])
def test_mirror_driver_matches_reference_driver(hostsim_lib, kind):
    from runtime import HostsimRuntime
    poses, modes = tm.run_mirror_driver(kind, HostsimRuntime(hostsim_lib))
    tm.check_against_driver_golden(kind, poses)
    if kind == "pnp":
        assert set(modes[1:]) <= {"PnP", "const"} and "PnP" in modes


@pytest.mark.parametrize("kind", ["pnp", "flowsel", "flowsel_gate"])
@pytest.mark.parametrize("mode", ["in_order", "pipelined", "tracker_thread"])
def test_pipeline_matches_reference_driver(hostsim_lib, kind, mode):
    """FramePipeline under both configurations: the driver golden, and the same per-frame branch as the mirror driver."""
    from runtime import HostsimRuntime
    from b200 import runtime as rt_mod
    rt = HostsimRuntime(hostsim_lib)
    rt_mod.set_runtime(rt)
    poses, modes, p = tm.run_pipeline(kind, mode, runtime=rt)
    tm.check_against_driver_golden(kind, poses)
    _, mirror_modes = tm.run_mirror_driver(kind, rt)
    assert modes[1:] == mirror_modes[1:], (modes, mirror_modes)


def test_pipeline_stepwise_path_matches_fused(hostsim_lib, monkeypatch):
    """DFVO_FUSED_TAIL=0 (host-orchestrated trackers) gives the same branches in both configurations and the same pose bits for
    PnP-only; with the E branch the scale differs at the 1e-12 level, as between the GRIC fused tail and its stepwise path."""
    from runtime import HostsimRuntime
    from b200 import runtime as rt_mod
    rt = HostsimRuntime(hostsim_lib)
    rt_mod.set_runtime(rt)
    for kind in ("pnp", "flowsel"):
        a, ma, _ = tm.run_pipeline(kind, "in_order", runtime=rt)
        monkeypatch.setenv("DFVO_FUSED_TAIL", "0")
        b, mb, _ = tm.run_pipeline(kind, "in_order", runtime=rt)
        monkeypatch.delenv("DFVO_FUSED_TAIL")
        assert ma == mb, kind
        assert np.array_equal(a, b) if kind == "pnp" else np.abs(a - b).max() < 1e-9, kind


@pytest.mark.parametrize("bad", [{"tracking_method": "deep_pose"}, {"e_tracker.validity.method": "homo_ratio"}])
def test_pipeline_rejects_unsupported_configurations(hostsim_lib, bad):
    import dropin_cases as dc
    from runtime import HostsimRuntime
    from b200 import pipeline, runtime as rt_mod
    rt = HostsimRuntime(hostsim_lib)
    rt_mod.set_runtime(rt)
    with pytest.raises(ValueError):
        pipeline.FramePipeline([60, 40, 100, 100], 80, 120, cfg=dc.make_cfg(80, 120, bad), runtime=rt)
