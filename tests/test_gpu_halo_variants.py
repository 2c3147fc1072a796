"""Every kernel of the halo conv dispatch table (conv_halo.cu launch_halo_t), forced through DFVO_HALO_S / DFVO_HALO_BN /
DFVO_HALO_CTAS: one and two resident CTAs per SM.  Each is checked against an fp64 convolution (bf16 and tf32 operands), and the
per-launch trace confirms that the forced configuration ran.  Two CTAs per SM change only which SM runs a tile and how deep the
rings are, not the K order of an output element, so their outputs must equal the one-CTA kernel's bit for bit, also on a shape
where every CTA walks many tiles."""
import ctypes

import numpy as np
import pytest
import torch

from test_gpu_stage_ops import _tc_conv_check

pytestmark = pytest.mark.gpu

# (S, block_n, CTAs per SM)
HALO_KERNELS = [(1, 16, 1), (1, 32, 1), (1, 64, 1), (2, 16, 1), (2, 32, 1), (4, 16, 1),
                (1, 16, 2), (1, 32, 2), (1, 64, 2), (2, 16, 2), (2, 32, 2)]

# B, Cin, H, W, Cout, kh, kw, pad_y, pad_x, act: a partial last K chunk, a partial second tile row, a last x-tile past the
# image for S = 2 and 4, Cout divisible by every block_n
CASE = (2, 80, 20, 72, 64, 3, 3, 1, 1, 1)
# 512 to 2048 tiles: each persistent CTA runs several, so the rings wrap across tiles
MANY_TILES = (2, 80, 64, 256, 64, 3, 3, 1, 1, 1)


def _force(monkeypatch, S, bn, ctas):
    monkeypatch.setenv("DFVO_HALO_S", str(S))
    monkeypatch.setenv("DFVO_HALO_BN", str(bn))
    monkeypatch.setenv("DFVO_HALO_CTAS", str(ctas))


def _trace(dev_lib, capfd, fn):
    dev_lib.dfvo_profile_enable(1)
    try:
        r = fn()
        ms, n, fl = ctypes.c_double(), ctypes.c_longlong(), ctypes.c_double()
        dev_lib.dfvo_profile_read(ctypes.byref(ms), ctypes.byref(n), ctypes.byref(fl))
    finally:
        dev_lib.dfvo_profile_enable(0)
    return r, n.value, capfd.readouterr().err


@pytest.mark.parametrize("prec", [1, 2])
@pytest.mark.parametrize("S,bn,ctas", HALO_KERNELS)
def test_halo_kernel_forced(dev_lib, monkeypatch, capfd, S, bn, ctas, prec):
    _force(monkeypatch, S, bn, ctas)
    monkeypatch.setenv("DFVO_TC_TRACE", "1")
    _, n, err = _trace(dev_lib, capfd, lambda: _tc_conv_check(dev_lib, CASE, prec))
    assert n == 1 and "halo" in err and " bn%d S%d " % (bn, S) in err and " ctas%d " % ctas in err, err


def _conv(dev_lib, case, prec):
    B, Cin, H, W, Cout, kh, kw, py, px, act = case
    rs = np.random.RandomState(7)
    x = torch.from_numpy(rs.standard_normal((B, Cin, H, W)).astype(np.float32)).cuda()
    w = (rs.standard_normal((Cout, Cin, kh, kw)) / np.sqrt(Cin * kh * kw)).astype(np.float32)
    b = (rs.standard_normal(Cout) * 0.1).astype(np.float32)
    out = torch.full((B, Cout, H, W), float("nan"), dtype=torch.float32, device="cuda")
    dev_lib.check(dev_lib.dfvo_conv2d(ctypes.c_void_p(x.data_ptr()), w.ctypes.data_as(ctypes.c_void_p), b.ctypes.data_as(ctypes.c_void_p),
                                      ctypes.c_void_p(out.data_ptr()), B, Cin, H, W, Cout, kh, kw, 1, py, px, 0, act, prec, None))
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize("prec", [1, 2])
@pytest.mark.parametrize("S,bn", sorted({(S, bn) for S, bn, ctas in HALO_KERNELS if ctas == 2}))
def test_two_ctas_bit_equal(dev_lib, monkeypatch, capfd, S, bn, prec):
    monkeypatch.setenv("DFVO_TC_TRACE", "1")
    outs = []
    for ctas in (1, 2):
        _force(monkeypatch, S, bn, ctas)
        y, n, err = _trace(dev_lib, capfd, lambda: _conv(dev_lib, MANY_TILES, prec))
        assert n == 1 and " bn%d S%d " % (bn, S) in err and " ctas%d " % ctas in err, err
        outs.append(y)
    assert np.isfinite(outs[0]).all()
    assert np.array_equal(outs[0].view(np.uint32), outs[1].view(np.uint32))
