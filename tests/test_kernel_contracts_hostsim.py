"""The kernel contracts of test_gpu_conv_contract.py and test_gpu_flow_kernels.py at reduced shapes on the host-emulation build
of the probe (tests/kernels/probe.cu compiled with -DDFVO_HOSTSIM): the descriptor features, views, strides and poison checks run
on a machine without a GPU.  Only what the emulation implements runs here -- no halo variants, chains, tensor-core correlation or
register-blocked flow head, and the emulated conv does not round its fp32 output to tf32, so the tf32-grid check is device-only.
Same references and tolerances as the GPU modules."""
import pytest

import kernel_probe as kp
import test_gpu_conv_contract as cc
import test_gpu_flow_kernels as fk


@pytest.fixture(scope="module")
def probe(hostsim_lib):
    p = kp.load_hostsim()
    assert not p.is_device
    return p


def _shrink(c, H, W):
    s = dict(c, N=2, H=H, W=W)
    if c["inHW"]:
        s["inHW"] = (H - 1, W + 1, 2, 3)
    return s


@pytest.mark.parametrize("name", [c["name"] for c in cc.CASES])
def test_conv_descriptor_hostsim(probe, name):
    c = _shrink(cc.BY_NAME[name], 11, 19)
    cc.run_case(probe, c, 2)


def test_conv_stem_overlapping_windows_hostsim(probe):
    cc.stem_case(probe, 32, 48)


@pytest.mark.parametrize("mode", [0, 1], ids=["run_conv_multi", "run_conv"])
@pytest.mark.parametrize("esize", [2, 4], ids=["bf16", "tf32"])
def test_conv_layer_packer_hostsim(probe, esize, mode):
    cc.packer_case(probe, esize, mode, H=9, W=21)


# ---- flow kernels and monodepth2 helpers (test_gpu_flow_kernels.py) at reduced shapes -------------------------------------------
@pytest.mark.parametrize("C,stride,pitch", [(64, 2, 64), (32, 1, 72), (48, 1, 72)])
def test_correlation_warped_hostsim(probe, C, stride, pitch):
    fk.corr_case(probe, C, 13, 29, stride, 2.5, out_pitch=pitch)


@pytest.mark.parametrize("with_res", [0, 1])
@pytest.mark.parametrize("k", [3, 5, 7])
def test_flow_head_hostsim(probe, k, with_res):
    fk.flow_head_case(probe, 11, 38, k, with_res)


@pytest.mark.parametrize("bf", [1, 0], ids=["bf16", "fp32"])
def test_flow_mean_reg_prep_hostsim(probe, bf):
    fk.reg_prep_case(probe, 13, 29, bf)


@pytest.mark.parametrize("k", [3, 5, 7])
@pytest.mark.parametrize("variant", ["bf16v", "bf16_generic", "fp32"])
def test_reg_tail_hostsim(probe, k, variant):
    cd = k * k
    pitch = 64 if variant == "bf16v" else (cd + 1 if (cd + 1) % 8 else cd + 2)
    fk.reg_tail_case(probe, 13, 29, k, variant != "fp32", pitch)


def test_deconv4x4s2_dw_hostsim(probe):
    fk.deconv_case(probe, 2, 7, 11, 49, 64, 64, 64, 1)
    fk.deconv_case(probe, 2, 7, 11, 12, 12, 12, 16, 1)
    fk.deconv_case(probe, 2, 7, 11, 2, 2, 2, 2, 0)


@pytest.mark.parametrize("bf", [1, 0], ids=["bf16", "fp32"])
@pytest.mark.parametrize("C", [64, 6])
def test_warp_bilinear_hostsim(probe, bf, C):
    fk.warp_case(probe, 2, 13, 29, C, bf, 2 * C + 16, C)


def test_flow_upsample_final_hostsim(probe):
    fk.upsample_case(probe, 11, 38, 24, 77)


def test_monodepth2_helpers_hostsim(probe):
    fk.maxpool_case(probe, 1, 15, 21, 16)
    for up in (1, 2):
        for skip in (0, 1):
            fk.upcat_case(probe, up, skip, h=5, w=7, C=8, Cs=8)
