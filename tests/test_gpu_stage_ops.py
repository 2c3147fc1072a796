"""GPU parity of the stage-level C-ABI entry points against the CPU oracle (oracle/nets.py).

Tolerances (floating point, SURVEY 8a / H4):
  * fp32 kernels vs fp32 oracle: 2e-5 abs on O(1) data (summation order only);
  * bf16/wgmma kernels vs an fp32 oracle evaluated on bf16-rounded operands: 1e-2 relative
    (fp32 accumulation, outputs rounded to bf16).
"""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import nets
from util import bf16_round, dptr

pytestmark = pytest.mark.gpu


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize("B,C,H,W,s", [(2, 192, 11, 38, 1), (2, 128, 22, 76, 1), (2, 96, 44, 152, 1),
                                       (2, 64, 88, 304, 2), (2, 64, 176, 608, 2), (1, 64, 35, 51, 2), (1, 32, 9, 13, 1)])
@pytest.mark.parametrize("prec", [0, 1])
def test_correlation(dev_lib, B, C, H, W, s, prec):
    rs = np.random.RandomState(C + H)
    a = rs.standard_normal((B, C, H, W)).astype(np.float32)
    b = rs.standard_normal((B, C, H, W)).astype(np.float32)
    if prec == 1:
        a, b = bf16_round(a), bf16_round(b)
    ref = F.leaky_relu(nets.correlation(torch.from_numpy(a), torch.from_numpy(b), s), 0.1).numpy()
    da, db = cu(a), cu(b)
    out = torch.zeros(ref.shape, dtype=torch.float32, device="cuda")
    dev_lib.check(dev_lib.dfvo_correlation(dptr(da), dptr(db), dptr(out), B, C, H, W, s, 1, prec, None))
    torch.cuda.synchronize()
    err = np.abs(out.cpu().numpy() - ref)
    if prec == 0:
        assert err.max() < 2e-5
    else:
        assert (err <= 1e-2 * np.abs(ref) + 2e-3).all(), err.max()


def test_correlation_fb_config3_batched(dev_lib):
    """BASELINE configs[2]: 64 independent frame pairs (128 maps after fwd/bwd stacking) through the correlation at the
    level-3 shape (C=64, 88x304, stride 2) and the consistency map at 376x1241.  Size-independent checks: batch entries
    are independent (entry i of the batched call == the same pair run alone, bit for bit), sampled entries match the
    oracle, and correlation is linear in its first argument."""
    rs = np.random.RandomState(64)
    B, C, H, W, s = 128, 64, 88, 304, 2
    a = bf16_round(rs.standard_normal((B, C, H, W)).astype(np.float32))
    b = bf16_round(rs.standard_normal((B, C, H, W)).astype(np.float32))
    da, db = cu(a), cu(b)
    out = torch.zeros((B, 49, H // s, W // s), dtype=torch.float32, device="cuda")
    dev_lib.check(dev_lib.dfvo_correlation(dptr(da), dptr(db), dptr(out), B, C, H, W, s, 0, 1, None))
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    for i in (0, 77, 127):
        ref = nets.correlation(torch.from_numpy(a[i:i + 1]), torch.from_numpy(b[i:i + 1]), s).numpy()
        assert (np.abs(got[i:i + 1] - ref) <= 1e-2 * np.abs(ref) + 2e-3).all()
        one = torch.zeros((1, 49, H // s, W // s), dtype=torch.float32, device="cuda")
        dai, dbi = cu(a[i:i + 1]), cu(b[i:i + 1])
        dev_lib.check(dev_lib.dfvo_correlation(dptr(dai), dptr(dbi), dptr(one), 1, C, H, W, s, 0, 1, None))
        torch.cuda.synchronize()
        assert np.array_equal(one.cpu().numpy()[0], got[i])
    # linearity in the first argument (exact in exact arithmetic; bf16 outputs -> 2 ulp of bf16)
    a2 = bf16_round(2.0 * a[:2])
    d2 = cu(a2)
    out2 = torch.zeros((2, 49, H // s, W // s), dtype=torch.float32, device="cuda")
    dev_lib.check(dev_lib.dfvo_correlation(dptr(d2), dptr(db), dptr(out2), 2, C, H, W, s, 0, 1, None))
    torch.cuda.synchronize()
    assert np.array_equal(out2.cpu().numpy(), 2.0 * got[:2])        # scaling by 2 is exact in binary floating point
    # consistency map, 64 pairs one after the other: |fwd + warp(bwd)| is zero for exactly opposite constant flows
    Hf, Wf = 376, 1241
    fwd = torch.full((2, Hf, Wf), 1.5, dtype=torch.float32, device="cuda")
    bwd = -fwd
    diff = torch.zeros((Hf, Wf), dtype=torch.float32, device="cuda")
    for _ in range(64):
        dev_lib.check(dev_lib.dfvo_fb_consistency(dptr(fwd), dptr(bwd), dptr(diff), Hf, Wf, None))
    torch.cuda.synchronize()
    d = diff.cpu().numpy()
    assert np.abs(d[:-3, :-3]).max() < 1e-5        # interior: fwd + bwd(p + fwd) = 0 (the right / bottom borders warp out of the image)


@pytest.mark.parametrize("prec", [0, 1])
def test_backward_warp(dev_lib, prec):
    rs = np.random.RandomState(3)
    B, C, H, W = 2, 64, 44, 152
    x = rs.standard_normal((B, C, H, W)).astype(np.float32)
    flow = (rs.standard_normal((B, 2, H, W)) * 6).astype(np.float32)
    flow[0, :, :3, :3] = 1e4          # far out of bounds -> zeros
    if prec == 1:
        x = bf16_round(x)
    ref = nets.backward_warp(torch.from_numpy(x), torch.from_numpy(flow)).numpy()
    dx, df = cu(x), cu(flow)
    out = torch.zeros_like(dx)
    dev_lib.check(dev_lib.dfvo_backward_warp(dptr(dx), dptr(df), dptr(out), B, C, H, W, prec, None))
    torch.cuda.synchronize()
    err = np.abs(out.cpu().numpy() - ref)
    assert err.max() < (2e-5 if prec == 0 else 2e-2)


def test_fb_consistency(dev_lib):
    rs = np.random.RandomState(5)
    H, W = 376, 1241
    fwd = (rs.standard_normal((1, 2, H, W)) * 4).astype(np.float32)
    bwd = (-fwd + rs.standard_normal((1, 2, H, W)) * 0.1).astype(np.float32)
    ref = nets.fb_consistency(torch.from_numpy(fwd), torch.from_numpy(bwd))[0, :, :, 0].numpy()
    dfw, dbw = cu(fwd[0]), cu(bwd[0])
    out = torch.zeros((H, W), dtype=torch.float32, device="cuda")
    dev_lib.check(dev_lib.dfvo_fb_consistency(dptr(dfw), dptr(dbw), dptr(out), H, W, None))
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    err = np.abs(got - ref)
    assert err.max() < 1e-4
    # mask agreement at the reference threshold (kp_selection.thre = 0.1) is reported, not asserted bit-exact
    flips = ((got < 0.1) != (ref < 0.1)).mean()
    assert flips < 1e-4
    # batched entry: three pairs in one launch == the single-pair call on each
    f3 = np.concatenate([fwd, fwd[:, :, ::-1].copy(), fwd * 0.5]).astype(np.float32)
    b3 = np.concatenate([bwd, bwd[:, :, ::-1].copy(), bwd * 0.5]).astype(np.float32)
    df3, db3 = cu(f3), cu(b3)
    out3 = torch.zeros((3, H, W), dtype=torch.float32, device="cuda")
    dev_lib.check(dev_lib.dfvo_fb_consistency_batch(dptr(df3), dptr(db3), dptr(out3), 3, H, W, None))
    for p in range(3):
        one = torch.zeros((H, W), dtype=torch.float32, device="cuda")
        dev_lib.check(dev_lib.dfvo_fb_consistency(dptr(df3[p]), dptr(db3[p]), dptr(one), H, W, None))
        assert torch.equal(one, out3[p])


CONV_CASES = [
    # B, Cin, H, W, Cout, kh, kw, stride, pad_y, pad_x, act
    (2, 3, 40, 72, 32, 7, 7, 1, 3, 3, 1),
    (2, 32, 40, 72, 32, 3, 3, 2, 1, 1, 1),
    (1, 64, 22, 38, 96, 3, 3, 2, 1, 1, 1),
    (2, 32, 33, 47, 2, 7, 7, 1, 3, 3, 0),
    (1, 16, 24, 40, 1, 3, 3, 1, 1, 1, 4),
]


@pytest.mark.parametrize("case", CONV_CASES)
def test_conv2d_fp32(dev_lib, case):
    B, Cin, H, W, Cout, kh, kw, st, py, px, act = case
    rs = np.random.RandomState(Cin * 7 + Cout)
    x = rs.standard_normal((B, Cin, H, W)).astype(np.float32)
    w = (rs.standard_normal((Cout, Cin, kh, kw)) / np.sqrt(Cin * kh * kw)).astype(np.float32)
    b = rs.standard_normal(Cout).astype(np.float32) * 0.1
    y = F.conv2d(torch.from_numpy(x), torch.from_numpy(w), torch.from_numpy(b), stride=st, padding=(py, px))
    y = {0: lambda t: t, 1: lambda t: F.leaky_relu(t, 0.1), 4: torch.sigmoid}[act](y).numpy()
    dx = cu(x)
    out = torch.zeros(y.shape, dtype=torch.float32, device="cuda")
    dev_lib.check(dev_lib.dfvo_conv2d(dptr(dx), w.ctypes.data_as(ctypes.c_void_p), b.ctypes.data_as(ctypes.c_void_p),
                                      dptr(out), B, Cin, H, W, Cout, kh, kw, st, py, px, 0, act, 0, None))
    torch.cuda.synchronize()
    assert np.abs(out.cpu().numpy() - y).max() < 3e-5


def test_conv2d_fp32_reflect(dev_lib):
    rs = np.random.RandomState(11)
    B, Cin, H, W, Cout = 1, 48, 12, 40, 32
    x = rs.standard_normal((B, Cin, H, W)).astype(np.float32)
    w = (rs.standard_normal((Cout, Cin, 3, 3)) / np.sqrt(Cin * 9)).astype(np.float32)
    b = rs.standard_normal(Cout).astype(np.float32) * 0.1
    y = F.elu(F.conv2d(F.pad(torch.from_numpy(x), (1, 1, 1, 1), mode="reflect"), torch.from_numpy(w), torch.from_numpy(b))).numpy()
    dx = cu(x)
    out = torch.zeros(y.shape, dtype=torch.float32, device="cuda")
    dev_lib.check(dev_lib.dfvo_conv2d(dptr(dx), w.ctypes.data_as(ctypes.c_void_p), b.ctypes.data_as(ctypes.c_void_p),
                                      dptr(out), B, Cin, H, W, Cout, 3, 3, 1, 1, 1, 1, 3, 0, None))
    torch.cuda.synchronize()
    assert np.abs(out.cpu().numpy() - y).max() < 3e-5


TC_CASES = [
    # B, Cin, H, W, Cout, kh, kw, pad_y, pad_x, act  -- the LiteFlowNet layer shapes (small spatial)
    (2, 128, 16, 64, 128, 3, 3, 1, 1, 1),      # single full tile row group
    (2, 64, 44, 152, 32, 3, 3, 1, 1, 1),
    (2, 49, 22, 76, 128, 3, 3, 1, 1, 1),       # Cin padded 49 -> 64
    (1, 130, 44, 152, 128, 3, 3, 1, 1, 1),     # Cin 130 -> 144 (partial last K chunk)
    (1, 386, 11, 38, 128, 3, 3, 1, 1, 1),      # many K chunks, tiny image, tile wider than image
    (2, 32, 40, 72, 2, 7, 7, 3, 3, 0),         # flow head: 49 taps, Cout 2 -> 16
    (1, 32, 22, 76, 49, 7, 1, 3, 0, 0),        # separable dist conv (7x1)
    (1, 49, 22, 76, 49, 1, 7, 0, 3, 0),        # (1x7), Cin 49 -> 64
    (1, 32, 24, 40, 64, 1, 1, 0, 0, 1),        # 1x1
    (1, 96, 24, 40, 192, 3, 3, 1, 1, 1),       # N = 192
    (1, 256, 6, 20, 512, 3, 3, 1, 1, 2),       # N blocks (512 = 4 x 128), relu
    (3, 16, 9, 130, 16, 3, 3, 1, 1, 3),        # odd sizes, elu, minimum channels
]

# the level-2 layers that carry 69 % of the frame's FLOPs (176x608x2, multi-wave persistent CTAs, S = 2 / 4 sub-tiles)
TC_BIG_CASES = [
    (2, 128, 176, 608, 128, 3, 3, 1, 1, 1),    # S = 2, block_n 128, 836 tiles over the persistent CTAs
    (2, 130, 176, 608, 128, 3, 3, 1, 1, 1),    # Subpixel Main.0: 144-channel input with a partial last chunk
    (2, 128, 176, 608, 64, 3, 3, 1, 1, 1),     # S = 4, block_n 64
    (2, 64, 176, 608, 32, 3, 3, 1, 1, 1),      # S = 4, block_n 32
    (2, 32, 176, 608, 64, 1, 1, 0, 0, 1),      # 1x1, store-bound
    (2, 32, 176, 608, 49, 7, 1, 3, 0, 0),      # distance conv 7x1 -> 49 (zero-padded to 64)
]

TC_S2_CASES = [
    # B, Cin, H, W, Cout, k, pad, act -- stride-2 convs (5-D tensor map over the 2x2 pixel phases)
    (2, 32, 64, 96, 32, 3, 1, 1), (2, 64, 44, 152, 96, 3, 1, 1), (1, 128, 22, 76, 192, 3, 1, 1),
    (1, 64, 48, 160, 128, 1, 0, 0), (1, 256, 12, 40, 512, 3, 1, 2), (2, 32, 352, 1216, 32, 3, 1, 1),
]


@pytest.mark.parametrize("case", TC_S2_CASES)
def test_conv2d_tcgen05_stride2(dev_lib, case):
    B, Cin, H, W, Cout, k, pad, act = case
    rs = np.random.RandomState(Cin + 7 * Cout + k)
    x = bf16_round(rs.standard_normal((B, Cin, H, W)).astype(np.float32))
    w = bf16_round((rs.standard_normal((Cout, Cin, k, k)) / np.sqrt(Cin * k * k)).astype(np.float32))
    b = (rs.standard_normal(Cout) * 0.1).astype(np.float32)
    y = F.conv2d(torch.from_numpy(x), torch.from_numpy(w), torch.from_numpy(b), stride=2, padding=pad)
    y = {0: lambda t: t, 1: lambda t: F.leaky_relu(t, 0.1), 2: F.relu}[act](y).numpy()
    dx = cu(x)
    out = torch.zeros(y.shape, dtype=torch.float32, device="cuda")
    dev_lib.check(dev_lib.dfvo_conv2d(dptr(dx), w.ctypes.data_as(ctypes.c_void_p), b.ctypes.data_as(ctypes.c_void_p),
                                      dptr(out), B, Cin, H, W, Cout, k, k, 2, pad, pad, 0, act, 1, None))
    torch.cuda.synchronize()
    err = np.abs(out.cpu().numpy() - y)
    assert (err <= 8e-3 * np.abs(y) + 4e-3).all(), err.max()



def tf32_round(x):
    """Round float32 to the 10-bit-mantissa tf32 grid (round to nearest, ties away: cvt.rna.tf32.f32)."""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    u = ((u + 0x1000) & 0xFFFFE000).astype(np.uint32)
    return u.view(np.float32)


def _tc_conv_check(dev_lib, case, prec, stride=1):
    """wgmma conv (prec 1: bf16 operands; prec 2: fp32 operands read as tf32) vs an fp64 convolution of the
    operands rounded to the tensor core's input format.  Tolerances: bf16 output rounding 2^-9; tf32 mode stores fp32
    rounded to tf32 (2^-11) and the activations are rounded once more on the way in."""
    B, Cin, H, W, Cout, kh, kw, py, px, act = case
    rs = np.random.RandomState(Cin + 13 * Cout + kh)
    rnd = bf16_round if prec == 1 else tf32_round
    x = rnd(rs.standard_normal((B, Cin, H, W)).astype(np.float32))
    w = rnd((rs.standard_normal((Cout, Cin, kh, kw)) / np.sqrt(Cin * kh * kw)).astype(np.float32))
    b = (rs.standard_normal(Cout) * 0.1).astype(np.float32)
    y = F.conv2d(torch.from_numpy(x).double(), torch.from_numpy(w).double(), torch.from_numpy(b).double(), stride=stride, padding=(py, px))
    y = {0: lambda t: t, 1: lambda t: F.leaky_relu(t, 0.1), 2: F.relu, 3: F.elu}[act](y).float().numpy()
    dx = cu(x)
    out = torch.zeros(y.shape, dtype=torch.float32, device="cuda")
    dev_lib.check(dev_lib.dfvo_conv2d(dptr(dx), w.ctypes.data_as(ctypes.c_void_p), b.ctypes.data_as(ctypes.c_void_p),
                                      dptr(out), B, Cin, H, W, Cout, kh, kw, stride, py, px, 0, act, prec, None))
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    err = np.abs(got - y)
    tol = (8e-3 * np.abs(y) + 4e-3) if prec == 1 else (1e-3 * np.abs(y) + 5e-4)
    assert (err <= tol).all(), "max err %g at %s (ref %g got %g)" % (
        err.max(), np.unravel_index(err.argmax(), err.shape), y.flat[err.argmax()], got.flat[err.argmax()])


@pytest.mark.parametrize("prec", [1, 2])
@pytest.mark.parametrize("case", TC_CASES)
def test_conv2d_tcgen05(dev_lib, case, prec):
    _tc_conv_check(dev_lib, case, prec)


@pytest.mark.parametrize("prec", [1, 2])
@pytest.mark.parametrize("case", TC_BIG_CASES)
def test_conv2d_tcgen05_level2_shapes(dev_lib, case, prec):
    _tc_conv_check(dev_lib, case, prec)


@pytest.mark.parametrize("case", [(2, 32, 64, 96, 32, 3, 3, 1, 1, 1), (1, 128, 22, 76, 192, 3, 3, 1, 1, 1), (2, 32, 352, 1216, 32, 3, 3, 1, 1, 1)])
def test_conv2d_tcgen05_stride2_tf32(dev_lib, case):
    _tc_conv_check(dev_lib, case, 2, stride=2)
