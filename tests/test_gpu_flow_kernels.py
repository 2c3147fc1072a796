"""LiteFlowNet's flow kernels (flow_ops.cu, corr_mma.cu) and monodepth2's helpers (depth_ops.cu) one at a time, against fp64
references, on every dispatch variant -- reached through the views' strides and sizes, and confirmed by the kernel names that
torch.profiler records.

Tolerances and where they come from:
  * correlation49_warped<bf16> (Backward warp fused into the tensor-core correlation, or warp_bilinear + the CUDA-core
    correlation): reference = fp64 warp, rounded to bf16, fp64 correlation / C, LeakyReLU.
        |got - ref| <= 2^-8 |ref| + 2^-7 sum_c |a_c b_c| / C
    2^-8: the bf16 output.  2^-7 sum|ab|/C: the kernel blends the warp in fp32 before rounding to bf16, so a warped element can
    land one bf16 ulp (<= 2^-7 relative) from the fp64-then-bf16 value; fp32 accumulation adds ~2^-24 sqrt(C), far below.
    Flows are multiples of 1/64 so x + f * scale is exact in fp32 and no floor() can move under FMA contraction.
  * flow_head (k x k conv, 32 bf16 channels -> 2 fp32): fp32 FMA accumulation of k*k*32 exact products:
        |got - ref| <= 2^-20 (sum |x||w| + |b| + |r|).
  * flow_mean accumulates in double and rounds once: 2^-23 relative to the mean plus the fp32 subtraction; reg_prep's
    distance channel is an fp32 bilinear blend + sum of squares + sqrt: 2^-18 relative to the scale of its terms.
  * reg_tail: the lite_flow_net.py:258-264 formula; fp32 exp and sums over <= 49 terms: 2^-16 relative to the weighted mean's
    scale (sum |w f| e / sum e), plus 2^-21 max(d^2) relative: the exponent -(d^2) - max is formed in fp32, so it carries an
    absolute rounding error of ~2^-23 d^2, which exp turns into that relative error of the weights.
  * deconv4x4s2_dw, warp_bilinear, flow_upsample_final: four fp32 products per output (2^-21 relative to sum |terms|), then
    the output rounding (2^-8 for bf16); flow_upsample_final also forms its source coordinates in fp32 like torch, which moves
    a bilinear weight by up to 2^-23 (h + w).
  * maxpool3x3s2, upcat_reflect: pure data movement -- bit-exact against torch on the same bf16 values.
"""
import pytest
import torch
import torch.nn.functional as F

import kernel_probe as kp

pytestmark = pytest.mark.gpu

LEVELS = {2: (176, 608), 3: (88, 304), 4: (44, 152), 5: (22, 76), 6: (11, 38)}
SCALE = {2: 10.0, 3: 5.0, 4: 2.5, 5: 1.25, 6: 0.625}


@pytest.fixture(scope="module")
def probe(dev_lib):
    p = kp.load_device()
    assert p.is_device
    return p


def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _run(probe, call, out, want=(), reject=()):
    """Launch `call` once; the caller checks the values it left in `out` (a Buf).  On the device, also confirm the dispatch path:
    the call is relaunched under torch.profiler (kp.kernel_names), every name in `want` must appear and none in `reject`, and
    the relaunch must reproduce the first launch's output bit for bit (the kernels are deterministic)."""
    call()
    if probe.device != "cuda":
        return
    first = out.flat.clone()
    names = kp.kernel_names(call, want)
    bits = kp.INT_VIEW[out.dtype]
    assert torch.equal(out.flat.view(bits), first.view(bits)), "a relaunch changed the output"
    for w in want:
        assert any(w in n for n in names), (w, names)
    for r in reject:
        assert not any(r in n for n in names), (r, names)


# ---- references ------------------------------------------------------------------------------------------------------------
def warp_ref(src, flow, scale, nxor=0):
    """Backward warp in fp64 (lite_flow_net.py:10-28, zeros outside, non-finite coordinates sample nothing).
    src [N,H,W,C] float64, flow [N,H,W,2] float32 -> [N,H,W,C] float64; batch entry n reads src[n ^ nxor]."""
    N, H, W, C = src.shape
    dev = src.device
    ys, xs = torch.meshgrid(torch.arange(H, device=dev), torch.arange(W, device=dev), indexing="ij")
    # x + f * scale in fp32, as the kernels do (exact for the flows used here)
    px = (xs.float() + flow[..., 0] * scale).double()
    py = (ys.float() + flow[..., 1] * scale).double()
    fin = torch.isfinite(px) & torch.isfinite(py) & (px.abs() < 1e9) & (py.abs() < 1e9)
    px, py = torch.where(fin, px, 0.0), torch.where(fin, py, 0.0)
    x0, y0 = torch.floor(px), torch.floor(py)
    wx1, wy1 = px - x0, py - y0
    nidx = (torch.arange(N, device=dev) ^ nxor).view(N, 1, 1).expand(N, H, W)
    out = torch.zeros_like(src)
    for ddy in (0, 1):
        for ddx in (0, 1):
            xx, yy = x0 + ddx, y0 + ddy
            wgt = (wx1 if ddx else 1 - wx1) * (wy1 if ddy else 1 - wy1)
            ok = fin & (xx >= 0) & (xx <= W - 1) & (yy >= 0) & (yy <= H - 1)
            v = src[nidx, yy.clamp(0, H - 1).long(), xx.clamp(0, W - 1).long()]
            out += torch.where(ok, wgt, 0.0).unsqueeze(-1) * v
    return out


def corr_ref(a, b, stride):
    """49-channel correlation / C (correlation.py:38-106) of a and b [N,H,W,C] float64 -> ([N,oH,oW,49], sum|ab|/C)."""
    C = a.shape[-1]
    a, b = a[:, ::stride, ::stride], b[:, ::stride, ::stride]
    oH, oW = a.shape[1], a.shape[2]
    bp = F.pad(b, (0, 0, 3, 3, 3, 3))
    out = torch.empty(a.shape[:3] + (49,), dtype=torch.float64, device=a.device)
    mag = torch.empty_like(out)
    for dy in range(7):
        for dx in range(7):
            p = a * bp[:, dy:dy + oH, dx:dx + oW]
            out[..., dy * 7 + dx] = p.sum(-1) / C
            mag[..., dy * 7 + dx] = p.abs().sum(-1) / C
    return out, mag


def _flow(N, H, W, g, span):
    """Random multiples of 1/64 in [-span, span] with the special regions the kernels must get right."""
    f = torch.round((torch.rand(N, H, W, 2, generator=g) * 2 - 1) * span * 64) / 64
    f[:, :H // 6, :W // 6] = torch.round(f[:, :H // 6, :W // 6])                    # integer flows: one bilinear weight of 1
    f[:, -3:, :, 1] = 0.5                                                            # last rows: partial weights past the border
    f[:, :, -3:, 0] = 0.75
    f[:, :2, W // 3:W // 3 + 8, 1] = -0.25                                           # first rows: partial weights above the image
    f[0, H // 2, W // 2:W // 2 + 5] = 1e4                                            # far outside
    f[0, H // 2 + 1, W // 2, 0] = float("nan")
    f[-1, H // 3, W // 3, 1] = float("inf")
    f[-1, H // 3, W // 3 + 1, 0] = float("-inf")
    return f


# ---- correlation49_warped ---------------------------------------------------------------------------------------------------
def corr_case(probe, C, H, W, stride, scale, out_pitch=64, N=2, seed=0, want=(), reject=()):
    """Called as liteflownet.cu's Matching unit does: first and feat2 are the same channel-slice view of one feature buffer
    (pitch C + 16, the rest NaN), nxor = 1 (each image of a pair correlates with the other one warped by its flow)."""
    dev = probe.device
    g = _gen(seed + C + H)
    fb = kp.Buf(N * H * W * (C + 16), torch.bfloat16, dev)
    fv = fb.view(N, H, W, C, sW=C + 16)
    feat = torch.randn(N, H, W, C, generator=g).to(torch.bfloat16)
    fv.t.copy_(feat.to(dev))
    span = 4.0 / scale * 8
    flow = _flow(N, H, W, g, span).to(dev)
    flb = kp.Buf(N * H * W * 2, torch.float32, dev)
    flv = flb.view(N, H, W, 2)
    flv.t.copy_(flow)
    sb = kp.Buf(N * H * W * C, torch.bfloat16, dev)
    sv = sb.view(N, H, W, C)
    oH, oW = (H + stride - 1) // stride, (W + stride - 1) // stride
    ob = kp.Buf(N * oH * oW * out_pitch, torch.bfloat16, dev, sentinel=True)
    ov = ob.view(N, oH, oW, 64, sW=out_pitch)
    _run(probe, lambda: probe("probe_correlation49_warped", 1, fv, fv, 1, flv, float(scale), stride, 1, sv, ov, None), ob, want, reject)
    f64 = feat.double().to(dev)
    warped = kp.bf16_rt(warp_ref(f64, flow, scale, nxor=1))
    ref, mag = corr_ref(f64, warped, stride)
    ref = F.leaky_relu(ref, 0.1)
    got = ov.t.double()
    assert torch.isfinite(got).all()
    err = (got[..., :49] - ref).abs()
    tol = 2.0 ** -8 * ref.abs() + 2.0 ** -7 * mag
    assert (err <= tol).all(), "max err %g over %d elements" % (float(err.max()), int((err > tol).sum()))
    assert (got[..., 49:] == 0).all(), "pad channels 49..63 not zero"
    assert ob.untouched_outside([ov]) == 0


CORR_SHAPES = [(64, 2, 2), (64, 3, 2), (96, 4, 1), (128, 5, 1), (192, 6, 1)]


@pytest.mark.parametrize("C,level,stride", CORR_SHAPES)
def test_correlation_warped_mma(probe, C, level, stride):
    H, W = LEVELS[level]
    corr_case(probe, C, H, W, stride, SCALE[level], want=("k_corr_mma1" if C <= 64 else "k_corr_mma(",), reject=("k_correlation49",))


@pytest.mark.parametrize("C,level,stride", [(64, 3, 2), (128, 5, 1), (48, 5, 1), (48, 3, 2)])
def test_correlation_warped_fallback(probe, C, level, stride):
    """An output pitch of 72 fails corr_mma_ok: warp_bilinear + k_correlation49_bf16v, or generic k_correlation49 for C = 48."""
    H, W = LEVELS[level]
    if C % 32 == 0:
        want, reject = ("k_warp_bilinear", "k_correlation49_bf16v"), ("k_corr_mma",)
    else:
        want, reject = ("k_warp_bilinear", "k_correlation49<"), ("k_corr_mma", "k_correlation49_bf16v")
    corr_case(probe, C, H, W, stride, SCALE[level], out_pitch=72, want=want, reject=reject)


def test_correlation_warped_mma1_ragged(probe):
    corr_case(probe, 32, 37, 101, 1, 2.5, N=4, want=("k_corr_mma1",))


# ---- flow_head ---------------------------------------------------------------------------------------------------------------
def flow_head_case(probe, H, W, k, with_res, N=2, seed=1, want=(), reject=()):
    dev = probe.device
    g = _gen(seed + k + H)
    ib = kp.Buf(N * H * W * 64, torch.bfloat16, dev)
    iv = ib.view(N, H, W, 32, sW=64)                                  # a channel slice: channels 32..63 NaN
    x = torch.randn(N, H, W, 32, generator=g).to(torch.bfloat16)
    iv.t.copy_(x.to(dev))
    w = (torch.randn(k, k, 32, 2, generator=g) / (32 * k * k) ** 0.5).float().to(dev).contiguous()
    b0, b1 = 0.125, -0.375
    rv = None
    if with_res:
        rb = kp.Buf(N * H * W * 4, torch.float32, dev)
        rv = rb.view(N, H, W, 2, sW=4)
        rv.t.copy_(torch.randn(N, H, W, 2, generator=g).to(dev))
    ob = kp.Buf(N * H * W * 4, torch.float32, dev, sentinel=True)
    ov = ob.view(N, H, W, 2, sW=4)
    call = lambda: probe("probe_flow_head", iv, w, b0, b1, k, rv, ov, None)
    _run(probe, call, ob, want, reject)
    x64 = x.double().to(dev).permute(0, 3, 1, 2)
    w64 = w.double().permute(3, 2, 0, 1)                              # [2][32][k][k]
    b64 = torch.tensor([b0, b1], dtype=torch.float64, device=dev)
    ref = F.conv2d(x64, w64, b64, padding=k // 2)
    mag = F.conv2d(x64.abs(), w64.abs(), b64.abs(), padding=k // 2)
    if rv is not None:
        ref, mag = ref + rv.nchw64(), mag + rv.nchw64().abs()
    got = ov.t.double().permute(0, 3, 1, 2)
    err = (got - ref).abs()
    assert torch.isfinite(got).all()
    assert (err <= 2.0 ** -20 * mag).all(), float(err.max())
    assert ob.untouched_outside([ov]) == 0


@pytest.mark.parametrize("with_res", [0, 1])
@pytest.mark.parametrize("k", [3, 5, 7])
@pytest.mark.parametrize("H,W", [(176, 608), (88, 304), (70, 301), (44, 152), (11, 38)])
def test_flow_head(probe, H, W, k, with_res):
    if H * W >= 20000:
        flow_head_case(probe, H, W, k, with_res, want=("k_flow_head8<%d>" % k,))
    else:
        flow_head_case(probe, H, W, k, with_res, want=("k_flow_head<%d>" % k,), reject=("k_flow_head8",))


# ---- flow_mean + reg_prep ---------------------------------------------------------------------------------------------------
def reg_prep_case(probe, H, W, bf, N=4, seed=2):
    """Regularization input (lite_flow_net.py:244-257) with nxor pairing: img2 of pair entry n is image n ^ 1."""
    dev = probe.device
    g = _gen(seed + H)
    scale = 1.25
    imgs = []
    for _ in range(2):
        b = kp.Buf(N * H * W * 4, torch.float32, dev)
        v = b.view(N, H, W, 3, sW=4)
        v.t.copy_(torch.rand(N, H, W, 3, generator=g).to(dev))
        imgs.append(v)
    flow = _flow(N, H, W, g, 6.0)
    flow[~torch.isfinite(flow)] = 0.0                                   # the mean of a non-finite field is not a contract
    flow[flow.abs() > 100] = 3.0
    flow = flow + 2.5                                                   # a mean far from zero
    fb = kp.Buf(N * H * W * 2, torch.float32, dev)
    fv = fb.view(N, H, W, 2)
    fv.t.copy_(flow.to(dev))
    mean = torch.zeros(int(probe.lib.probe_flow_mean_buffer_floats(N)), dtype=torch.float32, device=dev)
    probe("probe_flow_mean", fv, mean, None)
    dt = torch.bfloat16 if bf else torch.float32
    ob = kp.Buf(N * H * W * 16, dt, dev, sentinel=True)
    ov = ob.view(N, H, W, 8, sW=16)
    probe("probe_reg_prep", int(bf), imgs[0], imgs[1], 1, fv, mean, float(scale), ov, None)
    f64 = fv.t.double()
    mref = f64.mean(dim=(1, 2))                                         # [N, 2]
    got_mean = mean[:2 * N].double().view(N, 2)
    assert ((got_mean - mref).abs() <= 2.0 ** -23 * mref.abs() + 1e-12).all(), (got_mean, mref)
    i1, i2 = imgs[0].t.double(), imgs[1].t.double()
    warped = warp_ref(i2, fv.t, scale, nxor=1)
    dist = torch.sqrt(((i1 - warped) ** 2).sum(-1) + 1e-6)
    got = ov.t.double()
    u = 2.0 ** -8 if bf else 0.0
    assert ((got[..., 0] - dist).abs() <= u * dist + 2.0 ** -18 * (1 + dist)).all(), float((got[..., 0] - dist).abs().max())
    dflow = f64 - got_mean.view(N, 1, 1, 2)
    assert ((got[..., 1:3] - dflow).abs() <= u * dflow.abs() + 2.0 ** -22 * (f64.abs() + got_mean.abs().view(N, 1, 1, 2))).all()
    assert (got[..., 3:] == 0).all()
    assert ob.untouched_outside([ov]) == 0


@pytest.mark.parametrize("bf", [1, 0], ids=["bf16", "fp32"])
@pytest.mark.parametrize("H,W", [(176, 608), (37, 101)])
def test_flow_mean_reg_prep(probe, H, W, bf):
    reg_prep_case(probe, H, W, bf)


# ---- reg_tail ------------------------------------------------------------------------------------------------------------------
def reg_tail_case(probe, H, W, k, bf, pitch, N=2, seed=3, want=(), reject=()):
    dev = probe.device
    g = _gen(seed + k + pitch)
    cd = k * k
    dt = torch.bfloat16 if bf else torch.float32
    db = kp.Buf(N * H * W * pitch, dt, dev)
    dv = db.view(N, H, W, cd, sW=pitch)
    # the vector kernel loads the channels past cd up to the next multiple of 8 with the distances: they stay NaN and must be ignored
    d = torch.rand(N, H, W, cd, generator=g) * 3
    d[:, :H // 4] += 12.0                      # exp(-d^2) underflows in fp32 without the max subtraction (d^2 > 104)
    dv.t.copy_(d.to(dev).to(dt))
    fb = kp.Buf(N * H * W * 2, torch.float32, dev)
    fv = fb.view(N, H, W, 2)
    fv.t.copy_((torch.randn(N, H, W, 2, generator=g) * 4).to(dev))
    wx = torch.randn(cd, generator=g).float().to(dev)
    wy = torch.randn(cd, generator=g).float().to(dev)
    bx, by = 0.25, -0.5
    ob = kp.Buf(N * H * W * 2, torch.float32, dev, sentinel=True)
    ov = ob.view(N, H, W, 2)
    call = lambda: probe("probe_reg_tail", int(bf), dv, fv, k, wx, wy, bx, by, ov, None)
    _run(probe, call, ob, want, reject)
    # lite_flow_net.py:258-264: dist -> -(d^2) -> exp(x - max) -> weights; ScaleX/ScaleY (1x1 convs over unfold(flow)) / sum
    d64 = dv.t.double()
    e = torch.exp(-(d64 ** 2) - (-(d64 ** 2)).max(-1, keepdim=True).values)
    f64 = fv.t.double().permute(0, 3, 1, 2)
    unf = F.unfold(f64, k, padding=k // 2).view(N, 2, cd, H, W).permute(0, 3, 4, 1, 2)     # [N,H,W,2,cd]; zero padded
    ax = (wx.double() * e * unf[..., 0, :]).sum(-1) + bx
    ay = (wy.double() * e * unf[..., 1, :]).sum(-1) + by
    se = e.sum(-1)
    ref = torch.stack([ax / se, ay / se], -1)
    scl = torch.stack([((wx.double().abs() * e * unf[..., 0, :].abs()).sum(-1) + abs(bx)) / se,
                       ((wy.double().abs() * e * unf[..., 1, :].abs()).sum(-1) + abs(by)) / se], -1)
    got = ov.t.double()
    assert torch.isfinite(got).all()
    err = (got - ref).abs()
    dmax2 = (d64 ** 2).max(-1).values.unsqueeze(-1)
    tol = (2.0 ** -16 + 2.0 ** -21 * dmax2) * scl
    assert (err <= tol).all(), float((err / tol).max())
    assert ob.untouched_outside([ov]) == 0


@pytest.mark.parametrize("k", [3, 5, 7])
@pytest.mark.parametrize("variant", ["bf16v", "bf16_generic", "fp32"])
def test_reg_tail(probe, k, variant):
    H, W = LEVELS[3] if k == 7 else (37, 101)
    cd = k * k
    bf = variant != "fp32"
    pitch = 64 if variant == "bf16v" else (cd + 1 if (cd + 1) % 8 else cd + 2)
    if variant == "bf16v":
        reg_tail_case(probe, H, W, k, bf, pitch, want=("k_reg_tail_bf16v<%d>" % k,))
    else:
        reg_tail_case(probe, H, W, k, bf, pitch, want=("k_reg_tail<",), reject=("k_reg_tail_bf16v",))


# ---- deconv4x4s2_dw --------------------------------------------------------------------------------------------------------------
def deconv_case(probe, N, h, w, C_in, in_pitch, C_out, out_pitch, bf, seed=4, want=(), reject=()):
    dev = probe.device
    g = _gen(seed + C_in)
    dt = torch.bfloat16 if bf else torch.float32
    ib = kp.Buf(N * h * w * in_pitch, dt, dev)
    iv = ib.view(N, h, w, C_in, sW=in_pitch)
    # channels past C_in (the upcorr input's 49..63) stay NaN: the vector path loads them and must ignore them
    x = torch.randn(N, h, w, C_in, generator=g).to(dt)
    iv.t.copy_(x.to(dev))
    wt = torch.randn(C_in, 4, 4, generator=g).float().to(dev).contiguous()
    wfull = torch.zeros(max(C_in, C_out), 4, 4, device=dev)
    wfull[:C_in] = wt
    ob = kp.Buf(N * 2 * h * 2 * w * out_pitch, dt, dev, sentinel=True)
    ov = ob.view(N, 2 * h, 2 * w, C_out, sW=out_pitch)
    call = lambda: probe("probe_deconv4x4s2_dw", int(bf), iv, wfull.contiguous(), ov, None)
    _run(probe, call, ob, want, reject)
    x64 = x.double().to(dev).permute(0, 3, 1, 2)
    w64 = wt.double().unsqueeze(1)                                     # [C][1][4][4]
    ref = F.conv_transpose2d(x64, w64, stride=2, padding=1, groups=C_in)
    mag = F.conv_transpose2d(x64.abs(), w64.abs(), stride=2, padding=1, groups=C_in)
    got = ov.t.double().permute(0, 3, 1, 2)
    u = 2.0 ** -8 if bf else 0.0
    assert torch.isfinite(got).all()
    assert ((got[:, :C_in] - ref).abs() <= u * ref.abs() + 2.0 ** -21 * mag).all()
    assert (got[:, C_in:] == 0).all()
    assert ob.untouched_outside([ov]) == 0


@pytest.mark.parametrize("kind", ["upcorr", "bf16_generic", "upflow"])
def test_deconv4x4s2_dw(probe, kind):
    h, w = LEVELS[4]
    if kind == "upcorr":        # correlation 49 of a pitch-64 view -> 64-channel output, 8-channel vector path
        deconv_case(probe, 2, h, w, 49, 64, 64, 64, 1, want=("k_deconv4x4s2_dw_bf16v",))
    elif kind == "bf16_generic":
        deconv_case(probe, 2, 23, 37, 12, 12, 12, 16, 1, want=("k_deconv4x4s2_dw<",), reject=("bf16v",))
    else:                       # 2-channel float flow
        deconv_case(probe, 2, h, w, 2, 2, 2, 2, 0, want=("k_deconv4x4s2_dw<",))


# ---- warp_bilinear -------------------------------------------------------------------------------------------------------------
def warp_case(probe, N, H, W, C, bf, pitch, slot_off, seed=5, want=(), reject=()):
    """Writes into channel slot [slot_off, slot_off + C) of a pitch-`pitch` buffer, as liteflownet.cu writes subcat + C; the
    source is read at batch n ^ 1."""
    dev = probe.device
    g = _gen(seed + C)
    dt = torch.bfloat16 if bf else torch.float32
    ib = kp.Buf(N * H * W * (C + 8), dt, dev)
    iv = ib.view(N, H, W, C, sW=C + 8)
    x = torch.randn(N, H, W, C, generator=g).to(dt)
    iv.t.copy_(x.to(dev))
    flow = _flow(N, H, W, g, 6.0).to(dev)
    fb = kp.Buf(N * H * W * 2, torch.float32, dev)
    fv = fb.view(N, H, W, 2)
    fv.t.copy_(flow)
    ob = kp.Buf(N * H * W * pitch, dt, dev, sentinel=True)
    ov = ob.view(N, H, W, C, sW=pitch, off=slot_off)
    call = lambda: probe("probe_warp_bilinear", int(bf), iv, fv, 2.5, 1, ov, None)
    _run(probe, call, ob, want, reject)
    ref = warp_ref(x.double().to(dev), flow, 2.5, nxor=1)
    mag = warp_ref(x.double().abs().to(dev), flow, 2.5, nxor=1)
    got = ov.t.double()
    u = 2.0 ** -8 if bf else 0.0
    assert torch.isfinite(got).all()
    assert ((got - ref).abs() <= u * ref.abs() + 2.0 ** -21 * mag).all(), float((got - ref).abs().max())
    assert ob.untouched_outside([ov]) == 0


@pytest.mark.parametrize("bf", [1, 0], ids=["bf16", "fp32"])
@pytest.mark.parametrize("vec", [1, 0], ids=["vec", "scalar"])
def test_warp_bilinear(probe, bf, vec):
    C = 64 if vec else 6
    if vec:
        warp_case(probe, 2, 44, 152, C, bf, 2 * C + 16, C, want=("k_warp_bilinear_vec",))
    else:
        warp_case(probe, 2, 44, 152, C, bf, 2 * C + 16, C, want=("k_warp_bilinear<",), reject=("k_warp_bilinear_vec",))


# ---- flow_upsample_final -----------------------------------------------------------------------------------------------------
def upsample_case(probe, h, w, H, W, N=2, seed=6):
    dev = probe.device
    g = _gen(seed)
    fb = kp.Buf(N * h * w * 4, torch.float32, dev)
    fv = fb.view(N, h, w, 2, sW=4)
    fv.t.copy_((torch.randn(N, h, w, 2, generator=g) * 3).to(dev))
    out = torch.full((N, 2, H, W), float("nan"), dtype=torch.float32, device=dev)
    probe("probe_flow_upsample_final", fv, 10.0, H, W, out, None)
    f64 = fv.nchw64() * 10.0
    ref = F.interpolate(f64, size=(H, W), mode="bilinear", align_corners=True)
    ratio = torch.tensor([W / w, H / h], dtype=torch.float64, device=dev).view(1, 2, 1, 1)
    ref = ref * ratio
    mag = F.interpolate(f64.abs(), size=(H, W), mode="bilinear", align_corners=True) * ratio
    err = (out.double() - ref).abs()
    assert torch.isfinite(out).all()
    # the source coordinate (h - 1) / (H - 1) * y is formed in fp32 as torch does: its rounding (<= 2^-23 h) moves a lerp weight
    # by that much, times the difference of two neighbouring samples (<= 2 max |flow| * ratio)
    coord = 2.0 ** -22 * (h + w) * 2 * f64.abs().amax(dim=(2, 3), keepdim=True) * ratio
    assert (err <= 2.0 ** -20 * mag + coord).all(), float(err.max())


def test_flow_upsample_final(probe):
    upsample_case(probe, 176, 608, 376, 1241)


# ---- monodepth2 helpers: bit-exact ---------------------------------------------------------------------------------------------
def maxpool_case(probe, N, H, W, C, seed=7):
    dev = probe.device
    g = _gen(seed)
    ib = kp.Buf(N * H * W * C, torch.bfloat16, dev)
    iv = ib.view(N, H, W, C)
    x = (torch.randn(N, H, W, C, generator=g) - 2.0).to(torch.bfloat16)          # mostly negative: the padding must be -inf
    iv.t.copy_(x.to(dev))
    oH, oW = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    ob = kp.Buf(N * oH * oW * C, torch.bfloat16, dev, sentinel=True)
    ov = ob.view(N, oH, oW, C)
    probe("probe_maxpool3x3s2", iv, ov, None)
    ref = F.max_pool2d(x.float().permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1).to(torch.bfloat16).to(dev)
    assert torch.equal(ov.t.view(torch.int16), ref.view(torch.int16))


@pytest.mark.parametrize("H,W", [(188, 620), (33, 47)])
def test_maxpool3x3s2(probe, H, W):
    maxpool_case(probe, 1, H, W, 64)


def upcat_case(probe, up, with_skip, h=11, w=19, C=24, Cs=16, N=1, seed=8):
    dev = probe.device
    g = _gen(seed + up)
    lb = kp.Buf(N * h * w * C, torch.bfloat16, dev)
    lv = lb.view(N, h, w, C)
    lo = torch.randn(N, h, w, C, generator=g).to(torch.bfloat16)
    lv.t.copy_(lo.to(dev))
    sv, skip = None, None
    if with_skip:
        sb = kp.Buf(N * up * h * up * w * Cs, torch.bfloat16, dev)
        sv = sb.view(N, up * h, up * w, Cs)
        skip = torch.randn(N, up * h, up * w, Cs, generator=g).to(torch.bfloat16)
        sv.t.copy_(skip.to(dev))
    oC = C + (Cs if with_skip else 0)
    ob = kp.Buf(N * (up * h + 2) * (up * w + 2) * oC, torch.bfloat16, dev, sentinel=True)
    ov = ob.view(N, up * h + 2, up * w + 2, oC)
    probe("probe_upcat_reflect", lv, up, sv, ov, None)
    x = lo.float().permute(0, 3, 1, 2)
    if up == 2:
        x = F.interpolate(x, scale_factor=2, mode="nearest")
    if with_skip:
        x = torch.cat([x, skip.float().permute(0, 3, 1, 2)], 1)
    ref = F.pad(x, (1, 1, 1, 1), mode="reflect").permute(0, 2, 3, 1).to(torch.bfloat16).to(dev)
    assert torch.equal(ov.t.view(torch.int16), ref.view(torch.int16))


@pytest.mark.parametrize("with_skip", [0, 1])
@pytest.mark.parametrize("up", [1, 2])
def test_upcat_reflect(probe, up, with_skip):
    upcat_case(probe, up, with_skip)
