"""GPU: the PnP-only and flow-validity tracking configurations (ablation_tracker_pnp.yml, ablation_model_sel_flow.yml) on the
device -- the two fused tracker tails against the reference trackers' goldens, FramePipeline in every execution mode against the
in-order pipeline and the unmodified driver's goldens, and the device->host read budget of the tails."""
import numpy as np
import pytest

import tracking_modes_cases as tm
from b200 import runtime as rt_mod, tracking

pytestmark = pytest.mark.gpu


@pytest.fixture
def eng(dev_lib):
    rt = rt_mod.CudaRuntime(0)
    rt_mod.set_runtime(rt)
    return tracking.Engine(tm.H, tm.W, rt)


@pytest.mark.parametrize("name", list(tm.CASES))
def test_flow_tail_matches_reference_ess_tracker(eng, name):
    import dropin_cases as dc
    dc.fresh_libs()
    tm.check_ess_flow(eng, name)


@pytest.mark.parametrize("name", list(tm.CASES))
def test_pnp_tail_matches_reference_and_stepwise(eng, name):
    tm.check_pnp_tail(eng, name)


def test_flow_gate_mean_bit_equal(eng):
    means = {name: tm.check_flow_mean(eng, name) for name in tm.CASES}
    assert means["still"] <= tm.FLOW_THRE < means["moving"]
    tm.check_flow_mean_sizes(eng)


@pytest.mark.parametrize("kind", ["pnp", "flowsel", "flowsel_gate"])
def test_pipeline_modes_equal_in_order(dev_lib, kind):
    rt = rt_mod.CudaRuntime(0)
    rt_mod.set_runtime(rt)
    ref, ref_modes, _ = tm.run_pipeline(kind, "in_order", runtime=rt)
    tm.check_against_driver_golden(kind, ref)
    for mode in tm.MODES:
        if mode == "in_order":
            continue
        poses, modes, _ = tm.run_pipeline(kind, mode, runtime=rt)
        rt.torch.cuda.synchronize()
        assert np.array_equal(poses, ref), (kind, mode)
        assert modes == ref_modes, (kind, mode, modes, ref_modes)


def test_fused_pnp_equals_stepwise_pipeline_pnp(dev_lib, monkeypatch):
    """PnP-only FramePipeline: the fused tail (default) and FramePipeline.pnp (DFVO_FUSED_TAIL=0) give the same pose bits and leave
    the generator in the same state."""
    rt = rt_mod.CudaRuntime(0)
    rt_mod.set_runtime(rt)
    a, ma, _ = tm.run_pipeline("pnp", "in_order", runtime=rt)
    st_a = np.random.get_state()
    monkeypatch.setenv("DFVO_FUSED_TAIL", "0")
    b, mb, _ = tm.run_pipeline("pnp", "in_order", runtime=rt)
    st_b = np.random.get_state()
    assert np.array_equal(a, b) and ma == mb
    assert st_a[2] == st_b[2] and np.array_equal(st_a[1], st_b[1])


class _CountReads:
    """Counts the runtime's device->host reads (Buf.numpy goes through runtime.to_host)."""

    def __init__(self, rt):
        self.rt, self.n = rt, 0
        self.orig = rt.to_host

    def __enter__(self):
        def to_host(buf):
            self.n += 1
            return self.orig(buf)
        self.rt.to_host = to_host
        return self

    def __exit__(self, *a):
        self.rt.to_host = self.orig


@pytest.mark.parametrize("kind", ["pnp", "flowsel", "flowsel_gate"])
def test_tracker_read_budget(dev_lib, kind):
    """Per tracked frame: the selection's one status read (which in flow mode also carries the gate's mean), then PnP-only: one
    read of the filtered count + one packed read; flow validity with the E pose accepted: one packed read."""
    rt = rt_mod.CudaRuntime(0)
    rt_mod.set_runtime(rt)
    g = np.load(tm.G + "/dfvo_driver_%s_188x620.npz" % kind)
    h, w = [int(v) for v in g["hw"]]
    np.random.seed(4869)
    p = tm.injected_pipeline_class()(list(g["K"]), h, w, cfg=tm.pipeline_cfg(kind, h, w), runtime=rt)
    per_frame = []
    for t in range(g["poses"].shape[0]):
        cur = p.infer(None, t)
        p.stage += 1
        rt.torch.cuda.synchronize()
        with _CountReads(rt) as c:
            p._advance(cur, p.ref)
        per_frame.append((p.modes[t], p.last.get("scale"), c.n))
        p.ref = cur
    checked = 0
    for mode, scale, n in per_frame[1:]:
        if kind == "pnp" and mode == "PnP":
            assert n == 3, per_frame
            checked += 1
        if kind.startswith("flowsel") and mode == "E":
            assert n == 2, per_frame
            checked += 1
    assert checked > 0, per_frame
