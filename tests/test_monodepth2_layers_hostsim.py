"""The layer-by-layer checks of test_gpu_monodepth2_layers.py on the host-emulation build of the network probe, at reduced shapes, so the
tap, the references and the bars run on a machine without a GPU.  Same references and bars as the GPU module.  The emulated
tensor-core convolution does not round its fp32 outputs to tf32, so in tf32 mode only the stem's output (conv_direct, whose
rounding the emulation reproduces) is held to the tf32 grid here; the grid check of every tensor-core operand is device-only."""
import pytest

import test_gpu_monodepth2_layers as ml


@pytest.fixture(scope="module")
def probe(hostsim_lib):
    p = ml.load_hostsim()
    assert not p.is_device
    return p


SHAPES = [(64, 64, 2), (64, 128, 1)]


@pytest.mark.parametrize("h,w,B", SHAPES, ids=["%dx%d_B%d" % s for s in SHAPES])
@pytest.mark.parametrize("prec", ["fp32", "bf16", "tf32"])
@pytest.mark.parametrize("net", ["depth", "pose"])
def test_layers_hostsim(hostsim_lib, probe, monkeypatch, net, prec, h, w, B):
    ml.check_network(probe, hostsim_lib, monkeypatch, net, prec, h, w, B)
