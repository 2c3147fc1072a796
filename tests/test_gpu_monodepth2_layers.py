"""The monodepth2 depth runner and the PoseNet runner layer by layer, against fp64 references, as the product plans them.

The network probe (tests/kernels/nets/probe_nets.cu) builds each runner with monodepth2_create / posenet_create and runs it eagerly with a LayerTap
installed (monodepth2.h set_tap): every tensor the runner produces is copied back right after its launch.  Each layer is then
checked against an fp64 torch evaluation of that layer alone, whose input is the device's own tapped input, so errors do not
compound from layer to layer and the bars stay tight.  Per network (depth, PoseNet), precision (fp32, tf32, bf16, and bf16 with
DFVO_MONO_STEM_TC=0) and (feed_h, feed_w, B):

  * plan: the tap names equal the plan the architecture implies (a skipped layer fails here, not as a numeric drift);
  * normalisation: bit-exact against fp32 (x - 0.45) / 0.225 rounded to the storage type, the PoseNet's ref / cur feeds in
    channel slots 0-2 / 3-5; pad channels and the borders of the tensor-core stem's column-padded image exactly 0;
  * max-pool and upcat_reflect: bit-exact against F.max_pool2d(., 3, 2, 1) and F.pad(cat(nearest x2 (lo), skip), reflect);
  * every convolution (stem, BasicBlock convs with their residual, downsample, decoder convs, disparity head, PoseDecoder): the
    eval-mode BatchNorm folded as build_conv_layer does it (scale = g / sqrtf(v + 1e-5f), w * scale and b - m * scale in fp32),
    the weight rounded as the layer's path rounds it (bf16 RNE or tf32 RNA on the tensor cores, none on conv_direct's fp32
    weights), then fp64 act(conv + bias + residual).  Bar, as derived in test_gpu_conv_contract.py:

        |got - ref| <= u_out * |ref| + 2^-20 * (sum |x||w| + |bias| + |residual|)

    with one change for the tensor-core layers: their accumulation term is 2^-18 instead of 2^-20.  The contract test's 2^-20
    rests on rounding errors that cancel like a random walk, as conv_direct's round-to-nearest FMAs do (fp32 mode stays below
    half its bar).  The wgmma accumulator instead aligns the addends of each MMA to the largest and truncates, so its errors
    share a sign; where a layer's sum cancels deeply (|ref| ~ 1e-3 sum |x||w|, layer3 / layer4 of the tf32 encoder) they reach
    2^-19.1 sum |x||w| on an H100, which the tf32 output bar 2^-10 |ref| does not cover.  2^-18 holds twice that.
    u_out = 2^-8 for bf16 outputs, 2^-10 for fp32 outputs of the tensor cores (tf32-rounded, or the plain fp32 of the disparity
    head / net.3 in bf16 mode, as in the contract test) and of the tf32-rounded stem, 2^-23 for conv_direct's fp32 outputs.  A
    conv_direct fp32 output adds the error of its activation, which the fp32 accumulation term does not cover: ELU's expm1f (at
    most 1 ulp, 2^-22 relative with a binade edge) and the sigmoid 1 / (1 + expf(-v)) (expf's 2 ulp become <= 2^-22 relative,
    plus one add and one division: 2^-21).  In fp32 mode this bar is tight enough to catch weight-packing and BatchNorm-fold
    mistakes a bf16 bar hides;
  * tf32 grid: in tf32 mode every tapped tensor a tf32 tensor-core layer reads has its low 13 mantissa bits zero -- the wgmma
    kernels read fp32 operands as they are, so an off-grid operand would be truncated, not rounded;
  * disp_to_depth: within 4 fp32 ulp of fp64 baseline / (min_disp + (max_disp - min_disp) * disp) (depth_ops.cu is built with
    FMA contraction, so bit-exact is the wrong bar);
  * pose_head: fp64 restatement from the tapped net.3 output (fp32, pitch 16): mean over W then H, x 0.01, rot_from_axisangle,
    the inversion R^T, -R^T t and the translation times the baseline multiplier.  Bar: the kernel sums w values per row and h row
    means in fp32, then divides twice and scales, so each of the six parameters is within
        d_c = 0.01 * (w + h + 4) * 2^-24 * mean |out12[..., c]|
    of the fp64 value.  The rotation entries are a few fp32 operations on values <= 1 plus cosf / sinf (at most 2 ulp): 2^-20
    absolute covers their rounding, and R moves by at most 2 |dv| for a parameter error dv: E_R = 2^-20 + 4 max(d_0..2).  The
    translation column is b * sum_j R_ji (-t_j): E_T = b * (3 E_R |t|max + 3 max(d_3..5) + 12 * 2^-24 |t|max) + 2^-24 |T|.  The
    parameters are ~1e-2 and a wrong row count, pitch (12 vs 16), a missing transpose or the baseline on one component move an
    entry by 1e-4 or more, far outside these bars (~1e-6);
  * end-to-end tie: the probe's final depth / pose equal dfvo_monodepth2_forward_batch / dfvo_posenet_forward_batch (the product
    C ABI, CUDA-graphed) on the same weights and feeds bit for bit, so the tapped eager run is the product's computation;
  * non-degeneracy: at least 20 % of every conv layer's outputs are non-zero, and the disparity lies in (0.02, 0.98) for at least
    90 % of the pixels, so no layer passes by being constant.
The B = 3 case feeds three different images from separate allocations, so a wrong per-entry stride cannot line up by accident; the
64x64 feed is the smallest accepted, its 1/32 map is 2x2 (the reflection pad's edge case).  Each run prints, per layer, the worst
err / bar, so later changes can see their margin.
"""
import ctypes
import importlib.util
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import kernel_probe as kp
import synthdata as synth

pytestmark = pytest.mark.gpu

PRECISION = {"fp32": 0, "bf16": 1, "tf32": 2, "bf16_stem_direct": 1}
MIN_DEPTH, MAX_DEPTH, BASELINE, POSE_BASELINE = 0.1, 100.0, 5.4, 5.4
ACT_NONE, ACT_RELU, ACT_ELU, ACT_SIGMOID = 0, 2, 3, 4
_ACT = {ACT_NONE: lambda t: t, ACT_RELU: F.relu, ACT_ELU: F.elu, ACT_SIGMOID: torch.sigmoid}
# conv_direct fp32 output: relative error of the activation itself (see the module docstring)
_ACT_ERR = {ACT_NONE: 0.0, ACT_RELU: 0.0, ACT_ELU: 2.0 ** -22, ACT_SIGMOID: 2.0 ** -21}
U = 2.0 ** -24
# decoder stage k's upcat_reflect: (lo tap, upsampling, skip tap)
UPCAT = {0: ("enc.layer4.1.out", 1, None), 1: ("dec.0.conv", 2, "enc.layer3.1.out"), 2: ("dec.1.conv", 1, None),
         3: ("dec.2.conv", 2, "enc.layer2.1.out"), 4: ("dec.3.conv", 1, None), 5: ("dec.4.conv", 2, "enc.layer1.1.out"),
         6: ("dec.5.conv", 1, None), 7: ("dec.6.conv", 2, "enc.stem"), 8: ("dec.7.conv", 1, None), 9: ("dec.8.conv", 2, None),
         10: ("dec.9.conv", 1, None)}


def weights(net):
    if net == "depth":
        enc, dec = synth.monodepth2_weights(4869, 192, 640)
    else:
        enc, dec = synth.posenet_weights()
        enc = {k: v for k, v in enc.items() if k.startswith("encoder.")}
    return {k: v for d in (enc, dec) for k, v in d.items() if hasattr(v, "shape")}


def feeds(net, h, w, B, dev):
    """B entries (2B images for the PoseNet, [ref0, cur0, ref1, cur1, ...]) of textured [1, 3, h, w] feeds in [0, 1], every image its
    own allocation (allocated in reverse order, with spacers, so the addresses are unrelated to the entry index)."""
    n = B * (2 if net == "pose" else 1)
    out, spacers = [None] * n, []
    for i in reversed(range(n)):
        img = synth.value_noise_image(h, w, 31 + 7 * i)
        out[i] = torch.from_numpy(np.ascontiguousarray(np.transpose(img / 255.0, (2, 0, 1))[None])).float().to(dev)
        spacers.append(torch.empty(4096 * (i + 1), device=dev))
    return out


def plan(net, stem_tc):
    names = ["imgpad" if stem_tc else "x0", "enc.stem", "enc.pool"]
    for li in range(1, 5):
        for b in range(2):
            p = "enc.layer%d.%d." % (li, b)
            names += [p + "conv1"] + ([p + "down"] if li > 1 and b == 0 else []) + [p + "out"]
    if net == "depth":
        for k in range(10):
            names += ["dec.%d.pad" % k, "dec.%d.conv" % k]
        names += ["dec.10.pad", "disp", "depth"]
    else:
        names += ["pose.net0", "pose.net1", "pose.net2", "pose.out12", "pose"]
    return names


def conv_layers(net, prec, stem_tc):
    """(output tap, input tap, weight key, BatchNorm prefix | None, stride, pad, act, residual tap | None, tensor-core path)"""
    tc = prec != "fp32"
    L = [("enc.stem", "stem", "encoder.conv1", "encoder.bn1", 2, 3, ACT_RELU, None, stem_tc)]
    prev = "enc.pool"
    for li in range(1, 5):
        for b in range(2):
            p, k = "enc.layer%d.%d." % (li, b), "encoder.layer%d.%d." % (li, b)
            s = 2 if li > 1 and b == 0 else 1
            L.append((p + "conv1", prev, k + "conv1", k + "bn1", s, 1, ACT_RELU, None, tc))
            res = prev
            if li > 1 and b == 0:
                L.append((p + "down", prev, k + "downsample.0", k + "downsample.1", 2, 0, ACT_NONE, None, tc))
                res = p + "down"
            L.append((p + "out", p + "conv1", k + "conv2", k + "bn2", 1, 1, ACT_RELU, res, tc))
            prev = p + "out"
    bf = prec.startswith("bf16")
    if net == "depth":
        for k in range(10):
            L.append(("dec.%d.conv" % k, "dec.%d.pad" % k, "decoder.%d.conv.conv" % k, None, 1, 0, ACT_ELU, None, tc))
        L.append(("disp", "dec.10.pad", "decoder.10.conv", None, 1, 0, ACT_SIGMOID, None, bf))     # fp32 output: conv_direct in fp32 / tf32
    else:
        L.append(("pose.net0", prev, "net.0", None, 1, 0, ACT_RELU, None, tc))
        L.append(("pose.net1", "pose.net0", "net.1", None, 1, 1, ACT_RELU, None, tc))
        L.append(("pose.net2", "pose.net1", "net.2", None, 1, 1, ACT_RELU, None, tc))
        L.append(("pose.out12", "pose.net2", "net.3", None, 1, 0, ACT_NONE, None, bf))
    return L


def nchw(t, dev):
    return t.to(dev).double().permute(0, 3, 1, 2)


def on_tf32_grid(t):
    return bool(((t.float().contiguous().view(torch.int32) & 0x1FFF) == 0).all())


def fold(W, key, bn):
    """build_conv_layer's fold in fp32: (weight * scale, bias * scale + shift), scale = g / sqrtf(v + 1e-5f), shift = b - m * scale."""
    w = torch.from_numpy(W[key + ".weight"])
    if bn is None:
        return w, torch.from_numpy(W[key + ".bias"])
    g, b, m, v = (torch.from_numpy(W[bn + s]) for s in (".weight", ".bias", ".running_mean", ".running_var"))
    scale = g / torch.sqrt(v + torch.tensor(1e-5, dtype=torch.float32))
    return w * scale.view(-1, 1, 1, 1), b - m * scale


def check_conv(T, W, prec, layer, h, w, cin, dev):
    """One convolution against fp64; returns max err / bar."""
    out, inp, key, bn, stride, pad, act, res, tc = layer
    wf, bias = fold(W, key, bn)
    if tc:
        wf = kp.bf16_rt(wf) if prec.startswith("bf16") else kp.tf32_rna(wf)
    wf, bias = wf.double().to(dev), bias.double().to(dev)
    if inp == "stem":
        x = nchw(T["imgpad"][:, :, 3:3 + w, :cin], dev) if "imgpad" in T else nchw(T["x0"][..., :cin], dev)
    else:
        x = nchw(T[inp], dev)[:, :wf.shape[1]]
    z = F.conv2d(x, wf, bias, stride=stride, padding=pad)
    mag = F.conv2d(x.abs(), wf.abs(), bias.abs(), stride=stride, padding=pad)
    if res is not None:
        r = nchw(T[res], dev)
        z, mag = z + r, mag + r.abs()
    y = _ACT[act](z)
    got_t = T[out]
    got = nchw(got_t, dev)[:, :wf.shape[0]]
    assert got.shape == y.shape, "%s: tapped %s, reference %s" % (out, tuple(got.shape), tuple(y.shape))
    assert torch.isfinite(got).all(), "%s: non-finite outputs" % out
    if got_t.dtype == torch.bfloat16:
        u_out = 2.0 ** -8
    elif tc or (prec == "tf32" and out == "enc.stem"):
        u_out = 2.0 ** -10
    else:
        u_out = 2.0 ** -23 + _ACT_ERR[act]
    bar = u_out * y.abs() + (2.0 ** -18 if tc else 2.0 ** -20) * mag
    err = (got - y).abs()
    q = err / bar
    ratio = float(q.max())
    bad = err > bar
    i = int(q.argmax())
    assert not bad.any(), "%s: %d of %d outputs outside the bar, worst err / bar %.3g (err %g, ref %g, sum |x||w| %g at %s)" % (
        out, int(bad.sum()), bad.numel(), ratio, float(err.flatten()[i]), float(y.flatten()[i]), float(mag.flatten()[i]),
        list(np.unravel_index(i, tuple(err.shape))))
    nz = float((got != 0).double().mean())
    assert nz >= 0.2, "%s: only %.1f %% of the outputs are non-zero (degenerate layer)" % (out, 100 * nz)
    return ratio


def check_normalisation(T, fds, net, B, h, w):
    per = 2 if net == "pose" else 1
    cin = 3 * per
    dt = T["enc.stem"].dtype
    mean, std = torch.tensor(0.45, dtype=torch.float32), torch.tensor(0.225, dtype=torch.float32)
    want = torch.cat([((f.cpu() - mean) / std) for f in fds], 1).view(B, cin, h, w).permute(0, 2, 3, 1).to(dt).float()
    if "imgpad" in T:
        t = T["imgpad"].float()
        assert tuple(t.shape) == (B, h, w + 8, 8), tuple(t.shape)
        got, inside = t[:, :, 3:3 + w, :cin], torch.zeros(t.shape, dtype=torch.bool)
        inside[:, :, 3:3 + w, :cin] = True
        assert (t[~inside] == 0).all(), "imgpad: a border column or pad channel is not 0"
    else:
        t = T["x0"].float()
        assert tuple(t.shape) == (B, h, w, 4 if cin == 3 else 8), tuple(t.shape)
        got = t[..., :cin]
        assert (t[..., cin:] == 0).all(), "x0: a pad channel is not 0"
    assert torch.equal(got, want), "normalised feeds differ from (x - 0.45) / 0.225 at %d elements" % int((got != want).sum())


def check_pool_upcat(T, net, dev):
    stem = nchw(T["enc.stem"], dev)
    assert torch.equal(nchw(T["enc.pool"], dev), F.max_pool2d(stem, 3, 2, 1)), "enc.pool != max_pool2d(enc.stem, 3, 2, 1)"
    if net != "depth":
        return
    for k, (lo, up, skip) in UPCAT.items():
        x = nchw(T[lo], dev)
        if up == 2:
            x = F.interpolate(x, scale_factor=2, mode="nearest")
        if skip is not None:
            x = torch.cat([x, nchw(T[skip], dev)], 1)
        want = F.pad(x, (1, 1, 1, 1), mode="reflect")
        got = nchw(T["dec.%d.pad" % k], dev)
        assert got.shape == want.shape and torch.equal(got, want), "dec.%d.pad != reflect-pad(cat(upsample(%s), %s))" % (k, lo, skip)


def check_depth(T):
    disp, depth = T["disp"].double(), T["depth"]
    min_disp = np.float32(1.0) / np.float32(MAX_DEPTH)
    max_disp = np.float32(1.0) / np.float32(MIN_DEPTH)
    ref = float(np.float32(BASELINE)) / (float(min_disp) + (float(max_disp) - float(min_disp)) * disp)
    ulp = torch.from_numpy(np.spacing(np.abs(ref.numpy().astype(np.float32)))).double()
    err = (depth.double() - ref).abs()
    assert (err <= 4 * ulp).all(), "disp_to_depth: worst error %.3g ulp" % float((err / ulp).max())
    inside = float(((T["disp"] > 0.02) & (T["disp"] < 0.98)).double().mean())
    assert inside >= 0.9, "disparity saturated: only %.1f %% of the pixels in (0.02, 0.98)" % (100 * inside)
    return float((err / ulp).max())


def rot_from_axisangle(v):
    angle = np.linalg.norm(v)
    x, y, z = v / (angle + 1e-7)
    ca, sa = np.cos(angle), np.sin(angle)
    C = 1 - ca
    return np.array([[x * x * C + ca, x * y * C - z * sa, z * x * C + y * sa],
                     [x * y * C + z * sa, y * y * C + ca, y * z * C - x * sa],
                     [z * x * C - y * sa, y * z * C + x * sa, z * z * C + ca]])


def pose_reference(out12, baseline):
    """fp64 pose_head of one entry's [hh, ww, 12] map -> (4x4 pose, |R| bar, |t| bar)"""
    hh, ww = out12.shape[:2]
    x = out12[..., :6].astype(np.float64)
    p = 0.01 * x.mean(1).mean(0)
    d = 0.01 * (ww + hh + 4) * U * np.abs(x).mean((0, 1))
    R = rot_from_axisangle(p[:3])
    M = np.eye(4)
    M[:3, :3] = R.T
    M[:3, 3] = R.T @ (-p[3:]) * baseline
    tmax = np.abs(p[3:]).max()
    e_r = 2.0 ** -20 + 4 * d[:3].max()
    e_t = baseline * (3 * e_r * tmax + 3 * d[3:].max() + 12 * U * tmax) + U * np.abs(M[:3, 3]).max()
    return M, e_r, e_t


def check_pose(T, B):
    out12, pose = T["pose.out12"].numpy(), T["pose"].numpy().reshape(B, 4, 4)
    worst = 0.0
    for b in range(B):
        M, e_r, e_t = pose_reference(out12[b], POSE_BASELINE)
        got = pose[b].astype(np.float64)
        assert np.array_equal(got[3], [0, 0, 0, 1]), got[3]
        er, et = np.abs(got[:3, :3] - M[:3, :3]).max(), np.abs(got[:3, 3] - M[:3, 3]).max()
        assert er <= e_r and et <= e_t, "entry %d pose_head: rotation err %.3g (bar %.3g), translation err %.3g (bar %.3g)" % (
            b, er, e_r, et, e_t)
        worst = max(worst, er / e_r, et / e_t)
    return worst


class NetProbe:
    """ctypes bindings of the network probe library (tests/kernels/nets/probe_nets.cu)."""

    def __init__(self, path, device):
        self.lib = ctypes.CDLL(path)
        self.device = device
        self.lib.nets_last_error.restype = ctypes.c_char_p
        self.is_device = bool(self.lib.nets_is_device_build())

    def run(self, entry, weights, *args):
        """nets_monodepth2_run / nets_posenet_run with the state dict `weights` ({key: float32 array}) as (key, ndim, shape, data)
        arrays, then the entry's remaining arguments (torch tensors as their addresses, floats as C floats)."""
        items = [(k, np.ascontiguousarray(v, dtype=np.float32)) for k, v in weights.items()]
        n = len(items)
        keys = (ctypes.c_char_p * n)(*[k.encode() for k, _ in items])
        ndims = (ctypes.c_int * n)(*[a.ndim for _, a in items])
        shapes = (ctypes.c_longlong * sum(a.ndim for _, a in items))(*[d for _, a in items for d in a.shape])
        data = (ctypes.c_void_p * n)(*[a.ctypes.data for _, a in items])
        conv = [ctypes.c_void_p(a.data_ptr()) if isinstance(a, torch.Tensor) else ctypes.c_float(a) if isinstance(a, float) else a
                for a in args]
        rc = getattr(self.lib, entry)(n, keys, ndims, shapes, data, *conv)
        if rc != 0:
            msg = self.lib.nets_last_error()
            raise RuntimeError("%s failed (%d): %s" % (entry, rc, msg.decode() if msg else "?"))
        if self.device == "cuda":
            torch.cuda.synchronize()

    def taps(self):
        """The views the last run recorded, in launch order: [(name, [N, H, W, C] host tensor)]."""
        out = []
        for i in range(self.lib.nets_tap_count()):
            name = ctypes.create_string_buffer(64)
            esize, span = ctypes.c_int(), ctypes.c_longlong()
            dims, strides = (ctypes.c_int * 4)(), (ctypes.c_longlong * 3)()
            assert self.lib.nets_tap_info(i, name, 64, ctypes.byref(esize), dims, strides, ctypes.byref(span)) == 0
            flat = torch.empty(span.value, dtype=torch.bfloat16 if esize.value == 2 else torch.float32)
            assert self.lib.nets_tap_copy(i, ctypes.c_void_p(flat.data_ptr())) == 0
            out.append((name.value.decode(), torch.as_strided(flat, tuple(dims), tuple(strides) + (1,))))
        return out


def _nets_build():
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "kernels", "nets", "build.py")
    spec = importlib.util.spec_from_file_location("_probe_nets_build", path)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def load_device():
    """The network probe linked against the product library (load the product first: one copy of it must be mapped)."""
    return NetProbe(_nets_build().build_device(), "cuda")


def load_hostsim():
    return NetProbe(_nets_build().build_hostsim(), "cpu")


def run_probe(probe, net, prec, h, w, B, fds, out):
    W = weights(net)
    ptrs = (ctypes.c_void_p * len(fds))(*[f.data_ptr() for f in fds])
    if net == "depth":
        probe.run("nets_monodepth2_run", W, h, w, B, PRECISION[prec], MIN_DEPTH, MAX_DEPTH, BASELINE, ptrs, out, 1, None)
    else:
        probe.run("nets_posenet_run", W, h, w, B, PRECISION[prec], POSE_BASELINE, ptrs, out, 1, None)
    return W, probe.taps()


def run_product(lib, net, prec, h, w, B, fds, dev):
    """The same network through the product C ABI (dfvo_*_build_batch / *_forward_batch)."""
    from b200 import native
    W = weights(net)
    ctx = native.Context(lib)
    if net == "depth":
        ctx.load_weights(native.NET_MONODEPTH2, W)
        ctx.monodepth2_build_batch(h, w, B, PRECISION[prec], MIN_DEPTH, MAX_DEPTH, BASELINE)
        out = torch.zeros((B, h, w), device=dev)
        ctx.monodepth2_forward_batch([f.data_ptr() for f in fds], out.data_ptr())
    else:
        ctx.load_weights(native.NET_POSENET, W)
        ctx.posenet_build_batch(h, w, B, PRECISION[prec], POSE_BASELINE)
        out = torch.zeros((B, 4, 4), device=dev)
        ctx.posenet_forward_batch([f.data_ptr() for f in fds], out.data_ptr())
    if dev == "cuda":
        torch.cuda.synchronize()
    ctx.close()
    return out.cpu()


def check_network(probe, lib, monkeypatch, net, prec, h, w, B):
    """Run the tapped network and every check of the module docstring; returns {layer: worst err / bar}."""
    dev = probe.device
    if prec == "bf16_stem_direct":
        monkeypatch.setenv("DFVO_MONO_STEM_TC", "0")
    else:
        monkeypatch.delenv("DFVO_MONO_STEM_TC", raising=False)
    stem_tc = prec in ("bf16",)
    fds = feeds(net, h, w, B, dev)
    out = torch.full((B, h, w) if net == "depth" else (B, 4, 4), float("nan"), device=dev)
    W, taps = run_probe(probe, net, prec, h, w, B, fds, out)
    names = [n for n, _ in taps]
    assert names == plan(net, stem_tc), "tapped layers differ from the plan: %s" % names
    T = dict(taps)
    for n, t in taps:
        assert t.shape[0] == B, "%s: batch %d" % (n, t.shape[0])
    check_normalisation(T, fds, net, B, h, w)
    check_pool_upcat(T, net, dev)
    layers = conv_layers(net, prec, stem_tc)
    if prec == "tf32":
        # the stem is conv_direct, whose tf32 rounding the emulation reproduces; the emulated tensor-core layers do not round
        assert on_tf32_grid(T["enc.stem"]), "tf32 mode: the stem's output is not on the tf32 grid"
    if prec == "tf32" and probe.is_device:
        for layer in layers:
            if layer[8]:
                assert on_tf32_grid(T[layer[1]]), "tf32 mode: %s, the input of the tf32 tensor-core layer %s, is not on the tf32 grid" % (
                    layer[1], layer[0])
    report = {}
    cin = 6 if net == "pose" else 3
    for layer in layers:
        report[layer[0]] = check_conv(T, W, prec, layer, h, w, cin, dev)
    if net == "depth":
        report["depth (ulp / 4)"] = check_depth(T) / 4
    else:
        report["pose_head"] = check_pose(T, B)
    final = T["depth"][..., 0] if net == "depth" else T["pose"].reshape(B, 4, 4)
    assert torch.equal(out.cpu().view(torch.int32), final.contiguous().view(torch.int32)), "the tap of the output differs from the output"
    prod = run_product(lib, net, prec, h, w, B, fds, dev)
    assert torch.equal(prod.view(torch.int32), out.cpu().view(torch.int32)), (
        "the probe's eager run and the product's batched forward differ at %d elements" % int((prod != out.cpu()).sum()))
    print("\n%s %s %dx%d B=%d: worst err / bar per layer" % (net, prec, h, w, B))
    for k, v in report.items():
        print("  %-22s %.3f" % (k, v))
    print("  max %.3f" % max(report.values()))
    return report


# ------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def probe(dev_lib):
    p = load_device()
    assert p.is_device
    return p


SHAPES = [(192, 640, 1), (192, 640, 3), (64, 64, 2), (128, 416, 1)]


@pytest.mark.parametrize("h,w,B", SHAPES, ids=["%dx%d_B%d" % s for s in SHAPES])
@pytest.mark.parametrize("prec", ["fp32", "tf32", "bf16", "bf16_stem_direct"])
@pytest.mark.parametrize("net", ["depth", "pose"])
def test_layers(dev_lib, probe, monkeypatch, net, prec, h, w, B):
    check_network(probe, dev_lib, monkeypatch, net, prec, h, w, B)
