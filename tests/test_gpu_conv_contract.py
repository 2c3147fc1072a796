"""The tensor-core convolution descriptor (ops.h::ConvTc) feature by feature, on every kernel that implements it.

Each case is one feature of the descriptor at a LiteFlowNet / monodepth2 layer shape: virtual-concat sources that are channel
slices of wider buffers, outputs into a channel slot of a wider buffer, Cout < Cout_pad with and without zero_pad_to, bf16 and
fp32 residuals, fp32 output with a sigmoid (disparity head), pre-padded and asymmetric input windows, overlapping-window
sources (the monodepth2 stem), tf32 operands.  A case runs on the halo kernel with the cost model's configuration, on every
compiled (S, block_n) halo variant (DFVO_HALO_S / DFVO_HALO_BN), on the per-tap kernel (DFVO_CONV_HALO=0) and inside a layer
chain; the DFVO_TC_TRACE line of each launch says which one ran.

Poison: source buffers are NaN outside each view (other channels of the pitch, pixels outside a sub-window), the padded rows of
the packed weights and of the bias are NaN, and outputs start as a NaN sentinel bit pattern.  So a kernel that reads outside a
view or lets a padded Cout row reach a stored channel produces a non-finite output, and one that writes outside its view
changes a sentinel.

Reference: fp64 `F.conv2d` (on the device of the probe) of the operands the tensor core sees -- bf16 values, or fp32 rounded to
tf32 with cvt.rna -- then the epilogue in its order, act(conv + bias + residual).  Tolerance, from the arithmetic:

    |got - ref| <= u_out * |ref| + 2^-20 * (sum |x||w| + |bias| + |residual|)

  * u_out = 2^-8 for a bf16 output (round to nearest, 8 significant bits), 2^-10 for the tf32-rounded fp32 output, and 2^-10
    for the plain fp32 output of the disparity head (its error is the fp32 accumulation below, bounded generously);
  * sum |x||w| is a second fp64 conv of |x| with |w|: the products are exact in fp32, so the only error is the fp32
    accumulation of K <= 2600 terms.  With the independent random operands used here the partial sums random-walk: the k-th
    addition rounds with an error of ~2^-24 * sqrt(k) * s (s = typical |x w|), and these independent errors add up to
    ~2^-24 * s * K / sqrt(2), while sum |x||w| ~ 0.8 * K * s -- about 2^-24 relative, independent of K.  2^-20 leaves a 16x
    margin over that estimate (it is not the worst-case K * 2^-24 bound, which adversarial signs would need); the bias and
    residual are added once in fp32 (2^-24 relative);
  * every activation used (LeakyReLU, ReLU, ELU, sigmoid) is 1-Lipschitz, so the pre-activation bound carries through it.
Channels [Cout, zero_pad_to) must be exactly 0; channels from max(Cout, zero_pad_to) on must keep the sentinel.  In tf32 mode
every stored value must lie on the tf32 grid (low 13 mantissa bits zero).
"""
import ctypes

import pytest
import torch
import torch.nn.functional as F

import kernel_probe as kp

pytestmark = pytest.mark.gpu

ACT_NONE, ACT_LEAKY, ACT_RELU, ACT_ELU, ACT_SIGMOID = 0, 1, 2, 3, 4
_ACT = {ACT_NONE: lambda t: t, ACT_LEAKY: lambda t: F.leaky_relu(t, 0.1), ACT_RELU: F.relu, ACT_ELU: F.elu, ACT_SIGMOID: torch.sigmoid}
HALO_VARIANTS = [(1, 16), (1, 32), (1, 64), (2, 16), (2, 32), (4, 16)]


def case(name, N, H, W, srcs, Cout, kh=3, kw=3, pad=None, Cout_pad=None, zp=0, out=None, res=None, out_f32=0, act=ACT_LEAKY,
         inHW=None, prepad=False):
    """srcs: [(C, pitch, channel offset, buffer key)] -- sources with one key are views of one buffer; out / res: (pitch, offset)
    of the output / residual buffer; inHW: input window (inH, inW, pixel offset y, x inside an (H, W) + margin buffer)."""
    pad = (kh // 2, kw // 2) if pad is None else pad
    Cout_pad = (Cout + 15) // 16 * 16 if Cout_pad is None else Cout_pad
    return dict(name=name, N=N, H=H, W=W, srcs=srcs, Cout=Cout, kh=kh, kw=kw, pad=pad, Cout_pad=Cout_pad, zp=zp,
                out=out or (Cout_pad, 0), res=res, out_f32=out_f32, act=act, inHW=inHW, prepad=prepad)


# LiteFlowNet at 376x1241 runs its pyramid at 352x1216: levels 2..6 are 176x608, 88x304, 44x152, 22x76, 11x38
CASES = [
    # Subpixel subcat at level 3: [feat 64 | warped 64 | flow 16] = three views of one pitch-144 buffer, two pairs
    case("subcat3", 4, 88, 304, [(64, 144, 0, "a"), (64, 144, 64, "a"), (16, 144, 128, "a")], 128),
    # Regularization regcat at level 4 = [16 | 128] from two buffers (the 128 a slice of a pitch-160 one), output into channel
    # slot 32 of a pitch-192 buffer
    case("regcat4_slot", 2, 44, 152, [(16, 16, 0, "a"), (128, 160, 16, "b")], 128, out=(192, 32)),
    # rDist0 / rDist1 of level 2: 7x1 and 1x7, Cout 49 in a 64 slot, with and without zero_pad_to
    case("rdist0_zp", 2, 176, 608, [(32, 32, 0, "a")], 49, kh=7, kw=1, zp=64, act=ACT_NONE),
    case("rdist1_nozp", 2, 176, 608, [(64, 64, 0, "a")], 49, kh=1, kw=7, act=ACT_NONE, out=(64, 0)),
    # Cout < zero_pad_to < pitch: channels [49, 56) must become 0 and [56, 64) must keep the sentinel
    case("rdist0_zp56", 2, 176, 608, [(32, 32, 0, "a")], 49, kh=7, kw=1, zp=56, act=ACT_NONE, out=(64, 0)),
    # BasicBlock conv2: bf16 residual with its own strides (a slice of a pitch-160 buffer), ReLU after the sum
    case("residual5", 4, 22, 76, [(128, 128, 0, "a")], 128, res=(160, 16), act=ACT_RELU),
    # disparity head: fp32 output + fp32 residual, sigmoid, N padded 1 -> 16, ragged size
    case("disp_f32_sigmoid", 1, 37, 83, [(16, 16, 0, "a")], 1, out=(1, 0), res=(1, 0), out_f32=1, act=ACT_SIGMOID),
    # monodepth2 decoder: input pre-padded by reflection (inH = H + 2, pad 0), ragged size
    case("prepadded", 2, 45, 70, [(32, 32, 0, "a")], 16, pad=(0, 0), prepad=True, act=ACT_ELU),
    # asymmetric windows: the input window is one row shorter and one column wider than "same" padding implies, and sits
    # inside a larger NaN-poisoned buffer
    case("window", 2, 30, 61, [(48, 64, 0, "a")], 64, inHW=(29, 62, 2, 3)),
]
# the stride-1 bf16 cases that also run inside a layer chain (the chain takes 1..256-wide Cout_pad, bf16, stride 1)
CHAIN_CASES = ["subcat3", "regcat4_slot", "rdist0_zp", "rdist0_zp56", "rdist1_nozp", "residual5"]
BY_NAME = {c["name"]: c for c in CASES}


def _rnd(t, esize):
    return kp.bf16_rt(t) if esize == 2 else kp.tf32_rna(t)


def build(probe, c, esize, seed=0):
    """Allocate the poisoned operands of case c, return (descriptor, reference pieces, buffers to check)."""
    dev = probe.device
    g = torch.Generator(device="cpu").manual_seed(seed)
    dt = torch.bfloat16 if esize == 2 else torch.float32
    N, H, W, kh, kw = c["N"], c["H"], c["W"], c["kh"], c["kw"]
    py, px = c["pad"]
    if c["inHW"]:
        inH, inW, oy, ox = c["inHW"]
        bH, bW = inH + oy + 2, inW + ox + 2
    elif c["prepad"]:
        inH, inW, oy, ox = H + kh - 1, W + kw - 1, 0, 0
        bH, bW = inH, inW
    else:
        inH, inW, oy, ox = H, W, 0, 0
        bH, bW = H, W
    bufs, views = {}, []
    for (C, pitch, off, key) in c["srcs"]:
        if key not in bufs:
            bufs[key] = kp.Buf(N * bH * bW * pitch, dt, dev)
        v = bufs[key].view(N, inH, inW, C, sW=pitch, sH=bW * pitch, sN=bH * bW * pitch, off=(oy * bW + ox) * pitch + off)
        views.append(v)
    xs = []
    for v in views:
        if c["prepad"]:
            core = torch.randn(N, v.C, H, W, generator=g)
            x = F.pad(core, (kw // 2, kw // 2, kh // 2, kh // 2), mode="reflect")
        else:
            x = torch.randn(N, v.C, inH, inW, generator=g)
        x = _rnd(x.float(), esize).to(dev)
        v.t.copy_(x.permute(0, 2, 3, 1).to(dt))
        xs.append(x.double())
    x64 = torch.cat(xs, 1)
    K, Cout, Cp = x64.shape[1], c["Cout"], c["Cout_pad"]
    w = _rnd((torch.randn(Cout, K, kh, kw, generator=g) / (K * kh * kw) ** 0.5).float(), esize).to(dev)
    wp = torch.full((kh * kw, Cp, K), float("nan"), dtype=torch.float32, device=dev)     # padded Cout rows poisoned
    wp[:, :Cout, :] = w.permute(2, 3, 0, 1).reshape(kh * kw, Cout, K)
    wp = wp.to(dt).contiguous()
    bias = torch.full((Cp,), float("nan"), dtype=torch.float32, device=dev)
    bias[:Cout] = (torch.randn(Cout, generator=g) * 0.1).to(dev)
    out_dt = torch.float32 if (c["out_f32"] or esize == 4) else torch.bfloat16
    opitch, ooff = c["out"]
    oC = max(Cout, c["zp"])
    ob = kp.Buf(N * H * W * opitch, out_dt, dev, sentinel=True)
    ov = ob.view(N, H, W, oC, sW=opitch, off=ooff)
    rv = None
    if c["res"]:
        rpitch, roff = c["res"]
        rb = kp.Buf(N * H * W * rpitch, out_dt, dev)
        rv = rb.view(N, H, W, Cout, sW=rpitch, off=roff)
        r = torch.randn(N, H, W, Cout, generator=g).to(dev)
        rv.t.copy_(r.to(out_dt))
    d = kp.Conv()
    d.N, d.H, d.W = N, H, W
    d.inH, d.inW = (inH, inW) if (c["inHW"] or c["prepad"]) else (0, 0)
    d.nsrc = len(views)
    for i, v in enumerate(views):
        d.src[i] = v.ten
    d.stride, d.ntaps = 1, kh * kw
    dy0, dx0 = (0, 0) if c["prepad"] else (-py, -px)
    for t in range(kh * kw):
        d.dy[t], d.dx[t] = dy0 + t // kw, dx0 + t % kw
    d.esize, d.round_out_tf32 = esize, int(esize == 4)
    d.w, d.Cout_pad, d.Cout, d.bias = wp.data_ptr(), Cp, Cout, bias.data_ptr()
    d.act, d.out_f32 = c["act"], int(out_dt == torch.float32)
    d.out = ov.ten
    if rv is not None:
        d.residual = rv.ten
    d.zero_pad_to = c["zp"]
    keep = dict(wp=wp, bias=bias, bufs=bufs, res=rv)     # the allocations the descriptor points to must outlive it
    ref = dict(x64=x64, w64=w.double(), bias=bias[:Cout].double(), res=None if rv is None else rv.nchw64(), dy0=dy0, dx0=dx0,
               inH=inH, inW=inW)
    return d, ref, ob, ov, keep


def reference(c, ref):
    N, H, W, kh, kw = c["N"], c["H"], c["W"], c["kh"], c["kw"]
    dy0, dx0, inH, inW = ref["dy0"], ref["dx0"], ref["inH"], ref["inW"]
    padding = (-dx0, W - 1 + dx0 + kw - 1 - (inW - 1), -dy0, H - 1 + dy0 + kh - 1 - (inH - 1))     # negative = crop

    def conv(x, w):
        return F.conv2d(F.pad(x, padding), w)

    z = conv(ref["x64"], ref["w64"]) + ref["bias"].view(1, -1, 1, 1)
    mag = conv(ref["x64"].abs(), ref["w64"].abs()) + ref["bias"].abs().view(1, -1, 1, 1)
    if ref["res"] is not None:
        z = z + ref["res"]
        mag = mag + ref["res"].abs()
    return _ACT[c["act"]](z), mag


def check(c, esize, ref, ob, ov):
    """Values, exact zeros in [Cout, zero_pad_to), untouched sentinels, tf32 grid."""
    y, mag = reference(c, ref)
    Cout = c["Cout"]
    got = ov.t.double().permute(0, 3, 1, 2)
    gv = got[:, :Cout]
    assert torch.isfinite(gv).all(), "%s: %d non-finite outputs (a read outside a view?)" % (c["name"], int((~torch.isfinite(gv)).sum()))
    u_out = 2.0 ** -8 if (esize == 2 and not c["out_f32"]) else 2.0 ** -10
    tol = u_out * y.abs() + 2.0 ** -20 * mag
    err = (gv - y).abs()
    bad = err > tol
    assert not bad.any(), "%s: %d outside the bound, worst err %g (tol %g) at %s" % (
        c["name"], int(bad.sum()), float(err.max()), float(tol.flatten()[int((err - tol).argmax())]),
        [int(i) for i in torch.nonzero(bad)[0]])
    if c["zp"] > Cout:
        assert (got[:, Cout:c["zp"]] == 0).all(), "%s: channels [Cout, zero_pad_to) not zero" % c["name"]
    n = ob.untouched_outside([ov])
    assert n == 0, "%s: %d elements outside the output view were written" % (c["name"], n)
    if esize == 4:
        bits = ov.t.contiguous().view(torch.int32)
        assert ((bits & 0x1FFF) == 0).all(), "%s: stored fp32 values are not on the tf32 grid" % c["name"]


def run_case(probe, c, esize):
    d, ref, ob, ov, keep = build(probe, c, esize)
    probe("probe_conv_tc", d, None)
    check(c, esize, ref, ob, ov)
    return ov.t.clone()


# ------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def probe(dev_lib):
    p = kp.load_device()
    assert p.is_device
    return p


def _traced(dev_lib, monkeypatch, capfd, fn):
    """Run fn() with per-launch profiling and return the DFVO_TC_TRACE lines it printed."""
    monkeypatch.setenv("DFVO_TC_TRACE", "1")
    capfd.readouterr()
    dev_lib.dfvo_profile_enable(1)
    try:
        r = fn()
        ms, n, fl = ctypes.c_double(), ctypes.c_longlong(), ctypes.c_double()
        dev_lib.dfvo_profile_read(ctypes.byref(ms), ctypes.byref(n), ctypes.byref(fl))
    finally:
        dev_lib.dfvo_profile_enable(0)
    lines = [ln for ln in capfd.readouterr().err.splitlines() if ln.startswith("conv_tc ")]
    assert len(lines) == n.value
    return r, lines


def test_probe_shares_the_product_library(dev_lib, probe):
    """The probe's launches go through the one mapped copy of libdfvo_b200.so (its launch counter moves)."""
    c = BY_NAME["residual5"]
    before = dev_lib.dfvo_launch_count()
    run_case(probe, c, 2)
    assert dev_lib.dfvo_launch_count() == before + 1


@pytest.mark.parametrize("esize", [2, 4], ids=["bf16", "tf32"])
@pytest.mark.parametrize("name", [c["name"] for c in CASES])
def test_conv_default_config(dev_lib, probe, monkeypatch, capfd, name, esize):
    _, lines = _traced(dev_lib, monkeypatch, capfd, lambda: run_case(probe, BY_NAME[name], esize))
    assert len(lines) == 1 and " halo" in lines[0], lines


@pytest.mark.parametrize("esize", [2, 4], ids=["bf16", "tf32"])
@pytest.mark.parametrize("name", [c["name"] for c in CASES])
def test_conv_per_tap_kernel(dev_lib, probe, monkeypatch, capfd, name, esize):
    monkeypatch.setenv("DFVO_CONV_HALO", "0")
    _, lines = _traced(dev_lib, monkeypatch, capfd, lambda: run_case(probe, BY_NAME[name], esize))
    assert len(lines) == 1 and " tap " in lines[0], lines


@pytest.mark.parametrize("esize", [2, 4], ids=["bf16", "tf32"])
@pytest.mark.parametrize("S,bn", HALO_VARIANTS)
@pytest.mark.parametrize("name", ["subcat3", "regcat4_slot", "rdist0_zp", "rdist0_zp56", "residual5", "window"])
def test_conv_halo_variant(dev_lib, probe, monkeypatch, capfd, name, S, bn, esize):
    monkeypatch.setenv("DFVO_HALO_S", str(S))
    monkeypatch.setenv("DFVO_HALO_BN", str(bn))
    _, lines = _traced(dev_lib, monkeypatch, capfd, lambda: run_case(probe, BY_NAME[name], esize))
    assert len(lines) == 1 and " halo" in lines[0] and " bn%d S%d " % (bn, S) in lines[0], lines


def test_conv_chain_bit_exact(dev_lib, probe, monkeypatch, capfd):
    """The stride-1 bf16 cases inside one chain scope: each layer twice (into two output buffers) so the chain has work to fuse;
    both copies must equal the separate launch bit for bit."""
    taken = []
    for name in CHAIN_CASES:
        c = BY_NAME[name]
        d1, ref, ob1, ov1, k1 = build(probe, c, 2)
        probe("probe_conv_tc", d1, None)
        check(c, 2, ref, ob1, ov1)
        single = ov1.t.clone()
        ob1.flat.view(torch.int16).fill_(kp.SENTINEL[torch.bfloat16])
        d2, _, ob2, ov2, k2 = build(probe, c, 2)            # same seed: the same operands in fresh buffers
        bar = torch.zeros(16, dtype=torch.int32, device="cuda")
        arr = (kp.Conv * 2)(d1, d2)
        _, lines = _traced(dev_lib, monkeypatch, capfd, lambda: probe("probe_conv_chain", arr, 2, bar, None))
        assert torch.equal(ov1.t.view(torch.int16), single.view(torch.int16)), name
        assert torch.equal(ov2.t.view(torch.int16), single.view(torch.int16)), name
        assert ob1.untouched_outside([ov1]) == 0 and ob2.untouched_outside([ov2]) == 0, name
        if len(lines) == 1 and lines[0].split()[4] == "chain":
            taken.append(name)
    print("chained:", taken)
    assert taken, "no case ran as a chain"


# ---- the product packer: build_conv_layer with a Seg list and a folded BatchNorm, run through run_conv_multi / run_conv ----------
def packer_case(probe, esize, mode, H=44, W=152):
    """Regularization-style input [flow 2 of 16 | dist 49 of 64] through build_conv_layer (Seg list, BN scale / shift) and
    run_conv_multi (mode 0, two sources) or, for one source, run_conv with a residual and zero_pad_to (mode 1)."""
    dev = probe.device
    g = torch.Generator(device="cpu").manual_seed(7)
    dt = torch.bfloat16 if esize == 2 else torch.float32
    N = 2
    segs = [(2, 16), (49, 64)] if mode == 0 else [(49, 64)]
    Cout, kh, kw = 40, 3, 3
    Cin = sum(r for r, _ in segs)
    wref = torch.randn(Cout, Cin, kh, kw, generator=g) / (Cin * 9) ** 0.5
    bref = torch.randn(Cout, generator=g) * 0.1
    scale = torch.rand(Cout, generator=g) + 0.5
    shift = torch.randn(Cout, generator=g) * 0.1
    views, xs = [], []
    for (real, padded) in segs:
        b = kp.Buf(N * H * W * padded, dt, dev)
        v = b.view(N, H, W, padded)
        x = _rnd(torch.randn(N, real, H, W, generator=g), esize)
        full = torch.zeros(N, padded, H, W)
        full[:, :real] = x                                   # pad channels are zero (written by the producer)
        v.t.copy_(full.permute(0, 2, 3, 1).to(dev).to(dt))
        views.append(v)
        xs.append(x.double())
    zp = 48 if mode == 1 else 0
    ob = kp.Buf(N * H * W * 64, dt, dev, sentinel=True)
    ov = ob.view(N, H, W, max(Cout, zp), sW=64)
    rv, rarg = None, None
    if mode == 1:
        rb = kp.Buf(N * H * W * 48, dt, dev)
        rv = rb.view(N, H, W, Cout, sW=48)
        rv.t.copy_(torch.randn(N, H, W, Cout, generator=g).to(dev).to(dt))
        rarg = rv
    segs_c = (ctypes.c_int * (2 * len(segs)))(*[v for s in segs for v in s])
    ins = (kp.Ten * len(views))(*[v.ten for v in views])
    wc, bc, sc, shc = (t.float().contiguous().numpy() for t in (wref, bref, scale, shift))
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    probe("probe_conv_layer", P(wc), Cout, Cin, kh, kw, P(bc), segs_c, len(segs), 1, 1, P(sc), P(shc), esize, mode, ins, len(views),
          ov, ACT_LEAKY, rarg, zp, None)
    # reference: the layer as the network defines it, conv -> BN (eval) -> (+ residual) -> act, on the packer's rounded weights
    wfold = _rnd((wref * scale.view(-1, 1, 1, 1)).float(), esize).double().to(dev)
    bfold = (bref * scale + shift).double().to(dev)
    x64 = torch.cat(xs, 1).to(dev)
    z = F.conv2d(x64, wfold, bfold, padding=1)
    mag = F.conv2d(x64.abs(), wfold.abs(), bfold.abs(), padding=1)
    if rv is not None:
        z, mag = z + rv.nchw64(), mag + rv.nchw64().abs()
    y = F.leaky_relu(z, 0.1)
    got = ov.t.double().permute(0, 3, 1, 2)
    u_out = 2.0 ** -8 if esize == 2 else 2.0 ** -10
    err = (got[:, :Cout] - y).abs()
    assert torch.isfinite(got[:, :Cout]).all()
    assert (err <= u_out * y.abs() + 2.0 ** -20 * mag).all(), float(err.max())
    if zp:
        assert (got[:, Cout:zp] == 0).all()
    assert ob.untouched_outside([ov]) == 0


@pytest.mark.parametrize("mode", [0, 1], ids=["run_conv_multi", "run_conv"])
@pytest.mark.parametrize("esize", [2, 4], ids=["bf16", "tf32"])
def test_conv_layer_packer(probe, esize, mode):
    packer_case(probe, esize, mode)


# ---- overlapping-window sources: the monodepth2 stem (monodepth2.cu stem_tc_layer / run) ----------------------------------------
def stem_rearrange(w7):
    """encoder.conv1's 7x7 stride-2 weight [64][3][7][7] -> the 4x1 stride-1 weight [64][128][4][1] over the two row-parity views,
    by the packing rule of monodepth2.cu stem_tc_layer: input channel src * 64 + dx * 8 + c, tap kyy; odd ky read the even rows
    (src 0, ky = 2 kyy - 1), even ky the odd rows (src 1, ky = 2 kyy)."""
    wr = torch.zeros(w7.shape[0], 128, 4, 1, dtype=w7.dtype)
    for ky in range(7):
        src, kyy = (0, (ky + 1) // 2) if ky & 1 else (1, ky // 2)
        for dx in range(7):
            for c in range(3):
                wr[:, src * 64 + dx * 8 + c, kyy, 0] = w7[:, c, ky, dx]
    return wr


def stem_case(probe, h, w, seed=11):
    """The normalised image sits in a zero-initialised [h][w + 8][8] buffer at column offset 3 (pad_image8 / normalize); each
    row-parity view reads 64 channels (8 padded columns x 8) per pixel with a pixel stride of 16 elements, so consecutive pixels
    overlap (sW < C).  The rearranged weight goes through the product packer (build_conv_layer with the BatchNorm scale / shift,
    Seg list [64 | 64], pad_y 2) and run_conv_multi; the result must equal ReLU(BN(7x7 stride-2 pad-3 conv)) of the image."""
    dev = probe.device
    g = torch.Generator(device="cpu").manual_seed(seed)
    row = (w + 8) * 8
    b = kp.Buf(h * row + 64, torch.bfloat16, dev)            # the 64-element tail stays NaN: nothing may read past the rows
    b.flat[:h * row].zero_()
    img = ((torch.rand(1, 3, h, w, generator=g) - 0.45) / 0.225).to(torch.bfloat16)
    b.view(1, h, w, 3, sW=8, sH=row, sN=h * row, off=3 * 8).t.copy_(img.permute(0, 2, 3, 1).to(dev))
    views = [b.view(1, h // 2, w // 2, 64, sW=16, sH=2 * row, sN=h * row, off=par * row) for par in (0, 1)]
    w7 = torch.randn(64, 3, 7, 7, generator=g) / 147 ** 0.5
    scale = torch.rand(64, generator=g) + 0.5
    shift = torch.randn(64, generator=g) * 0.1
    ob = kp.Buf(h // 2 * (w // 2) * 80, torch.bfloat16, dev, sentinel=True)
    ov = ob.view(1, h // 2, w // 2, 64, sW=80, off=16)
    segs = (ctypes.c_int * 4)(64, 64, 64, 64)
    ins = (kp.Ten * 2)(*[v.ten for v in views])
    wr, sc, sh = (t.float().contiguous().numpy() for t in (stem_rearrange(w7), scale, shift))
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    probe("probe_conv_layer", P(wr), 64, 128, 4, 1, None, segs, 2, 2, 0, P(sc), P(sh), 2, 0, ins, 2, ov, ACT_RELU, None, 0, None)
    # reference: the packer rounds W * scale to bf16; the rearrangement is a permutation, so round the 7x7 weight the same way
    wfold = kp.bf16_rt((w7 * scale.view(-1, 1, 1, 1)).float()).double().to(dev)
    x = img.double().to(dev)
    z = F.conv2d(x, wfold, shift.double().to(dev), stride=2, padding=3)
    mag = F.conv2d(x.abs(), wfold.abs(), shift.double().abs().to(dev), stride=2, padding=3)
    y = F.relu(z)
    got = ov.t.double().permute(0, 3, 1, 2)
    assert torch.isfinite(got).all(), "non-finite stem outputs"
    err = (got - y).abs()
    assert (err <= 2.0 ** -8 * y.abs() + 2.0 ** -20 * mag).all(), "stem: max err %g" % float(err.max())
    assert ob.untouched_outside([ov]) == 0


STEM_CONFIGS = ["default", "per_tap"] + ["halo_S%d_bn%d" % v for v in HALO_VARIANTS]


@pytest.mark.parametrize("config", STEM_CONFIGS)
def test_conv_stem_overlapping_windows(dev_lib, probe, monkeypatch, capfd, config):
    """At the KITTI feed size of monodepth2 (192 x 640 -> 96 x 320)."""
    if config == "per_tap":
        monkeypatch.setenv("DFVO_CONV_HALO", "0")
    elif config != "default":
        S, bn = (int(t[1:]) if t[0] == "S" else int(t[2:]) for t in config.split("_")[1:])
        monkeypatch.setenv("DFVO_HALO_S", str(S))
        monkeypatch.setenv("DFVO_HALO_BN", str(bn))
    _, lines = _traced(dev_lib, monkeypatch, capfd, lambda: stem_case(probe, 192, 640))
    assert len(lines) == 1, lines
    if config == "per_tap":
        assert " tap " in lines[0], lines
    else:
        assert " halo" in lines[0] and "src[64,64,0]" in lines[0], lines
        if config != "default":
            assert " bn%d S%d " % (bn, S) in lines[0], lines
