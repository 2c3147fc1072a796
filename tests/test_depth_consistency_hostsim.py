"""CPU: the PoseNet (dfvo_posenet_*), the depth-consistency kernel (dfvo_depth_consistency) and the masked local_bestN through the
emulation build, and the oracle restatements (oracle/pose_consistency.py), against the goldens the reference produced
(tests/golden/depth_consistency.npz, oracle/gen_golden_depth_consistency.py)."""
import numpy as np
import pytest

from b200 import native
from oracle import pose_consistency, synth
import depth_consistency_cases as dc


def test_oracle_restatements_match_reference_golden():
    g = dc.golden()
    mult = float(g["pose_multiplier"])
    pose = dc.oracle_pose(g["pose_feed_ref"], g["pose_feed_cur"], mult)
    assert np.abs(pose - g["pose"]).max() < 1e-6
    for case in (0, 1):
        cur, ref, T, K = pose_consistency_case(case)
        got = pose_consistency.depth_consistency(cur, ref, T, *intrinsics(K))
        dc.compare_depth_diff(got, g["dc%d_depth_diff" % case])


def pose_consistency_case(case):
    from oracle import gen_golden_depth_consistency as gen
    return gen.consistency_case(case)


def intrinsics(K):
    cx, cy, fx, fy = K
    Km = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float64)
    return Km, np.linalg.inv(Km)


def test_posenet_fp32_vs_reference_golden(hostsim_lib):
    g = dc.golden()
    mult = float(g["pose_multiplier"])
    pose = dc.posenet(hostsim_lib, dc.HostMem(), g["pose_feed_ref"], g["pose_feed_cur"], native.PREC_FP32, mult)
    assert np.abs(pose - g["pose"]).max() < 1e-6, np.abs(pose - g["pose"]).max()
    aa, t = dc.pose_parameters_of(pose, mult)
    assert np.abs(aa - g["pose_axisangle"]).max() < 1e-4 * np.abs(g["pose_axisangle"]).max()
    assert np.abs(t - g["pose_translation"]).max() < 1e-4 * np.abs(g["pose_translation"]).max()


@pytest.mark.parametrize("prec", [native.PREC_BF16, native.PREC_TF32])
def test_posenet_tensor_core_plumbing(hostsim_lib, prec):
    """bf16 / tf32 wiring (6-channel tensor-core stem in bf16, 1/32-resolution decoder on the tensor-core kernel): within the
    rounding distance of the operands of the reference pose."""
    g = dc.golden()
    mult = float(g["pose_multiplier"])
    pose = dc.posenet(hostsim_lib, dc.HostMem(), g["pose_feed_ref"], g["pose_feed_cur"], prec, mult)
    aa, t = dc.pose_parameters_of(pose, mult)
    bar = 5e-2 if prec == native.PREC_BF16 else 5e-3
    assert np.abs(aa - g["pose_axisangle"]).max() < bar * np.abs(g["pose_axisangle"]).max()
    assert np.abs(t - g["pose_translation"]).max() < bar * np.abs(g["pose_translation"]).max()


def test_posenet_rejects_a_three_channel_stem(hostsim_lib):
    enc, dec = synth.posenet_weights()
    enc = dict(enc, **{"encoder.conv1.weight": enc["encoder.conv1.weight"][:, :3].copy()})
    with pytest.raises(native.DfvoError):
        dc.posenet(hostsim_lib, dc.HostMem(), np.zeros((3, 64, 64), np.float32), np.zeros((3, 64, 64), np.float32),
                   native.PREC_FP32, 1.0, enc, dec)


@pytest.mark.parametrize("case", [0, 1])
def test_depth_consistency_vs_reference_golden(hostsim_lib, case):
    g = dc.golden()
    cur, ref, T, K = pose_consistency_case(case)
    got = dc.depth_consistency(hostsim_lib, dc.HostMem(), cur, ref, T, K)
    want = g["dc%d_depth_diff" % case]
    nborder = dc.compare_depth_diff(got, want)
    print("case %d: %d pixels within 5e-4 of the threshold" % (case, nborder))
    if case == 0:
        assert (want == 0).sum() > 0 and (want == 1).sum() > 0       # negative ratios clamp to 0; out-of-image / large ratios to 1
    else:
        assert np.isnan(want).sum() > 0                               # 0/0: fails the `< thre` test like in torch


def test_masked_local_bestn_vs_reference_golden(hostsim_lib):
    g = dc.golden()
    fr = synth.analytic_frame(seed=21, h=376, w=1241)
    dd = pose_consistency.selection_depth_diff(376, 1241)
    for name in ("a", "b"):
        idx = dc.select_with_mask(hostsim_lib, dc.HostMem(), fr["flow_diff"][..., 0], dd, float(g["sel_%s_thre" % name]))
        assert np.array_equal(idx, g["sel_%s_idx_sorted" % name])
    assert not np.array_equal(g["sel_a_idx_sorted"], g["sel_b_idx_sorted"])
