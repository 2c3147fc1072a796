"""Every (S, block_n) variant of the halo-resident conv kernel, forced through DFVO_HALO_S / DFVO_HALO_BN: the cost model picks
only some of them for the LiteFlowNet layers, so each compiled variant gets its own check against an fp64 convolution (bf16 and
tf32 operands), and the per-launch trace confirms that the forced configuration is the one that ran."""
import ctypes

import pytest

from test_gpu_stage_ops import _tc_conv_check

pytestmark = pytest.mark.gpu

# the kernel's dispatch table (conv_halo.cu launch_halo_t)
HALO_VARIANTS = [(1, 16), (1, 32), (1, 64), (2, 16), (2, 32), (4, 16)]

# B, Cin, H, W, Cout, kh, kw, pad_y, pad_x, act: a partial last K chunk (80 = 64 + 16 bf16 / 32 + 32 + 16 tf32 channels), a
# partial second tile row, a last x-tile that runs past the image for S = 2 and 4, and Cout divisible by every block_n
CASE = (2, 80, 20, 72, 64, 3, 3, 1, 1, 1)


@pytest.mark.parametrize("prec", [1, 2])
@pytest.mark.parametrize("S,bn", HALO_VARIANTS)
def test_halo_forced_variant(dev_lib, monkeypatch, capfd, S, bn, prec):
    monkeypatch.setenv("DFVO_HALO_S", str(S))
    monkeypatch.setenv("DFVO_HALO_BN", str(bn))
    monkeypatch.setenv("DFVO_TC_TRACE", "1")
    dev_lib.dfvo_profile_enable(1)
    try:
        _tc_conv_check(dev_lib, CASE, prec)
        ms, n, fl = ctypes.c_double(), ctypes.c_longlong(), ctypes.c_double()
        dev_lib.dfvo_profile_read(ctypes.byref(ms), ctypes.byref(n), ctypes.byref(fl))
    finally:
        dev_lib.dfvo_profile_enable(0)
    err = capfd.readouterr().err
    assert n.value == 1 and "halo" in err and " bn%d S%d " % (bn, S) in err, err
