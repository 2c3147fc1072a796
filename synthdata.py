"""Seeded synthetic inputs shared by golden generation, tests and bench (SURVEY.md 8d).

Everything is produced from ``np.random.RandomState(seed)`` with a fixed draw order, so the
machine that generates goldens and every machine that tests regenerate bit-identical weights / frames / correspondences
and only small *outputs* need to be committed under ``tests/golden/``.

Weight dictionaries use the reference's own state-dict key names
(``lite_flow_net.py:35-271`` -> ``moduleFeatures.moduleOne.0.weight`` ...;
``resnet_encoder.py:68-98`` / ``depth_decoder.py:30-47`` -> ``encoder.layer1.0.conv1.weight``,
``decoder.0.conv.conv.weight`` ...), so the same dict loads into the reference modules
(golden generation) and into the CUDA weight packer.
"""
import math

import numpy as np

# ----------------------------------------------------------------------------------------
# LiteFlowNet parameter shapes (lite_flow_net.py:35-271)
# ----------------------------------------------------------------------------------------
LFN_LEVELS = [2, 3, 4, 5, 6]                      # ModuleList index k <-> level LFN_LEVELS[k]
LFN_FEAT_CH = {1: 32, 2: 32, 3: 64, 4: 96, 5: 128, 6: 192}
LFN_KLAST = {2: 7, 3: 5, 4: 5, 5: 3, 6: 3}          # last-conv / unfold kernel per level
LFN_SUB_CIN = {2: 130, 3: 130, 4: 194, 5: 258, 6: 386}
LFN_REG_CIN = {2: 131, 3: 131, 4: 131, 5: 131, 6: 195}
LFN_DIST_CH = {2: 49, 3: 25, 4: 25, 5: 9, 6: 9}
LFN_BACKWARD = {2: 10.0, 3: 5.0, 4: 2.5, 5: 1.25, 6: 0.625}


def liteflownet_shapes():
    """Ordered {key: shape} for every LiteFlowNet parameter."""
    s = {}

    def conv(name, cout, cin, kh, kw=None, bias=True):
        s[name + ".weight"] = (cout, cin, kh, kh if kw is None else kw)
        if bias:
            s[name + ".bias"] = (cout,)

    f = "moduleFeatures."
    conv(f + "moduleOne.0", 32, 3, 7)
    conv(f + "moduleTwo.0", 32, 32, 3)
    conv(f + "moduleTwo.2", 32, 32, 3)
    conv(f + "moduleTwo.4", 32, 32, 3)
    conv(f + "moduleThr.0", 64, 32, 3)
    conv(f + "moduleThr.2", 64, 64, 3)
    conv(f + "moduleFou.0", 96, 64, 3)
    conv(f + "moduleFou.2", 96, 96, 3)
    conv(f + "moduleFiv.0", 128, 96, 3)
    conv(f + "moduleSix.0", 192, 128, 3)
    for k, lv in enumerate(LFN_LEVELS):
        m = "moduleMatching.%d." % k
        if lv == 2:
            conv(m + "moduleFeat.0", 64, 32, 1)
        if lv != 6:
            s[m + "moduleUpflow.weight"] = (2, 1, 4, 4)      # ConvTranspose2d groups=2
        if lv < 4:
            s[m + "moduleUpcorr.weight"] = (49, 1, 4, 4)     # ConvTranspose2d groups=49
        conv(m + "moduleMain.0", 128, 49, 3)
        conv(m + "moduleMain.2", 64, 128, 3)
        conv(m + "moduleMain.4", 32, 64, 3)
        conv(m + "moduleMain.6", 2, 32, LFN_KLAST[lv])
    for k, lv in enumerate(LFN_LEVELS):
        m = "moduleSubpixel.%d." % k
        if lv == 2:
            conv(m + "moduleFeat.0", 64, 32, 1)
        conv(m + "moduleMain.0", 128, LFN_SUB_CIN[lv], 3)
        conv(m + "moduleMain.2", 64, 128, 3)
        conv(m + "moduleMain.4", 32, 64, 3)
        conv(m + "moduleMain.6", 2, 32, LFN_KLAST[lv])
    for k, lv in enumerate(LFN_LEVELS):
        m = "moduleRegularization.%d." % k
        if lv < 5:
            conv(m + "moduleFeat.0", 128, LFN_FEAT_CH[lv], 1)
        conv(m + "moduleMain.0", 128, LFN_REG_CIN[lv], 3)
        conv(m + "moduleMain.2", 128, 128, 3)
        conv(m + "moduleMain.4", 64, 128, 3)
        conv(m + "moduleMain.6", 64, 64, 3)
        conv(m + "moduleMain.8", 32, 64, 3)
        conv(m + "moduleMain.10", 32, 32, 3)
        kd, cd = LFN_KLAST[lv], LFN_DIST_CH[lv]
        if lv >= 5:
            conv(m + "moduleDist.0", cd, 32, kd)
        else:
            conv(m + "moduleDist.0", cd, 32, kd, 1)
            conv(m + "moduleDist.1", cd, cd, 1, kd)
        conv(m + "moduleScaleX", 1, cd, 1)
        conv(m + "moduleScaleY", 1, cd, 1)
    return s


def _fill(shapes, seed, bias_std=0.02, gain=math.sqrt(2.0), scale_overrides=None):
    rs = np.random.RandomState(seed)
    out = {}
    for name, shp in shapes.items():
        if name.endswith(".weight") and len(shp) == 4:
            fan_in = shp[1] * shp[2] * shp[3]
            std = gain / math.sqrt(fan_in)
            if scale_overrides:
                for pat, sc in scale_overrides.items():
                    if pat in name:
                        std *= sc
            out[name] = (rs.standard_normal(shp) * std).astype(np.float32)
            if "moduleScale" in name:      # trained nets: ~identity weighting of the local average
                out[name] = (1.0 + 0.1 * out[name] / std).astype(np.float32)
        elif name.endswith(".bias"):
            out[name] = (rs.standard_normal(shp) * bias_std).astype(np.float32)
        elif name.endswith("running_var"):
            out[name] = rs.uniform(0.5, 1.5, shp).astype(np.float32)
        elif name.endswith("running_mean"):
            out[name] = (rs.standard_normal(shp) * 0.1).astype(np.float32)
        elif name.endswith("bn_weight"):
            out[name] = rs.uniform(0.5, 1.5, shp).astype(np.float32)
        else:
            raise KeyError(name)
    return out


def liteflownet_weights(seed=4869):
    """Kaiming-scaled (the reference's own init, ``lite_flow_net.py:273-279``) but with small
    non-zero biases so bias handling is exercised.  The flow heads are damped and the
    ScaleX/ScaleY 1x1 convs set near one so synthetic flows are a few pixels: large enough to
    exercise the warps, small enough that they do not all sample out of bounds."""
    return _fill(liteflownet_shapes(), seed,
                 scale_overrides={"moduleMain.6": 0.5, "moduleDist": 0.5})


# ----------------------------------------------------------------------------------------
# monodepth2 ResNet-18 encoder + depth decoder (resnet_encoder.py:68-98, depth_decoder.py:17-65)
# ----------------------------------------------------------------------------------------
def monodepth2_shapes():
    enc, dec = {}, {}

    def bn(d, name, c):
        d[name + ".weight"] = ("bn_weight", (c,))
        d[name + ".bias"] = ("bias", (c,))
        d[name + ".running_mean"] = ("running_mean", (c,))
        d[name + ".running_var"] = ("running_var", (c,))

    enc["encoder.conv1.weight"] = ("weight", (64, 3, 7, 7))
    bn(enc, "encoder.bn1", 64)
    cin = 64
    for li, cout in zip([1, 2, 3, 4], [64, 128, 256, 512]):
        for b in range(2):
            p = "encoder.layer%d.%d." % (li, b)
            enc[p + "conv1.weight"] = ("weight", (cout, cin if b == 0 else cout, 3, 3))
            bn(enc, p + "bn1", cout)
            enc[p + "conv2.weight"] = ("weight", (cout, cout, 3, 3))
            bn(enc, p + "bn2", cout)
            if b == 0 and li > 1:
                enc[p + "downsample.0.weight"] = ("weight", (cout, cin, 1, 1))
                bn(enc, p + "downsample.1", cout)
        cin = cout
    num_ch_enc = [64, 64, 128, 256, 512]
    num_ch_dec = [16, 32, 64, 128, 256]
    idx = 0
    for i in range(4, -1, -1):
        ci = num_ch_enc[-1] if i == 4 else num_ch_dec[i + 1]
        dec["decoder.%d.conv.conv.weight" % idx] = ("weight", (num_ch_dec[i], ci, 3, 3))
        dec["decoder.%d.conv.conv.bias" % idx] = ("bias", (num_ch_dec[i],))
        idx += 1
        ci = num_ch_dec[i] + (num_ch_enc[i - 1] if i > 0 else 0)
        dec["decoder.%d.conv.conv.weight" % idx] = ("weight", (num_ch_dec[i], ci, 3, 3))
        dec["decoder.%d.conv.conv.bias" % idx] = ("bias", (num_ch_dec[i],))
        idx += 1
    for s_ in range(4):
        dec["decoder.%d.conv.weight" % idx] = ("weight", (1, num_ch_dec[s_], 3, 3))
        dec["decoder.%d.conv.bias" % idx] = ("bias", (1,))
        idx += 1
    return enc, dec


def monodepth2_weights(seed=4869, height=192, width=640):
    """Returns (encoder_dict, decoder_dict).  ``encoder_dict`` additionally carries the
    ``height``/``width`` entries the reference reads the feed size from (monodepth2.py:70-71)."""
    enc_s, dec_s = monodepth2_shapes()
    rs = np.random.RandomState(seed)

    def fill(spec):
        out = {}
        for name, (kind, shp) in spec.items():
            if kind == "weight":
                fan_in = shp[1] * shp[2] * shp[3]
                out[name] = (rs.standard_normal(shp) * math.sqrt(2.0 / fan_in)).astype(np.float32)
            elif kind == "bias":
                out[name] = (rs.standard_normal(shp) * 0.05).astype(np.float32)
            elif kind == "running_mean":
                out[name] = (rs.standard_normal(shp) * 0.1).astype(np.float32)
            elif kind == "running_var":
                out[name] = rs.uniform(0.5, 1.5, shp).astype(np.float32)
            elif kind == "bn_weight":
                out[name] = rs.uniform(0.5, 1.0, shp).astype(np.float32)
        return out

    enc = fill(enc_s)
    dec = fill(dec_s)
    enc["height"] = height
    enc["width"] = width
    return enc, dec


def posenet_weights(seed=5171):
    """monodepth2 PoseNet: ResnetEncoder(18, False, 2) (6-channel stem) + PoseDecoder(num_ch_enc, 1, 2) (pose_decoder.py:
    net.0 squeeze 1x1 512->256, net.1 / net.2 3x3 256->256, net.3 1x1 256->12), Kaiming-scaled like monodepth2_weights.
    Returns (pose_encoder_dict, pose_decoder_dict)."""
    enc_s, _ = monodepth2_shapes()
    enc_s["encoder.conv1.weight"] = ("weight", (64, 6, 7, 7))
    dec_s = {"net.0.weight": ("weight", (256, 512, 1, 1)), "net.0.bias": ("bias", (256,)),
             "net.1.weight": ("weight", (256, 256, 3, 3)), "net.1.bias": ("bias", (256,)),
             "net.2.weight": ("weight", (256, 256, 3, 3)), "net.2.bias": ("bias", (256,)),
             "net.3.weight": ("weight", (12, 256, 1, 1)), "net.3.bias": ("bias", (12,))}
    rs = np.random.RandomState(seed)
    out = []
    for spec in (enc_s, dec_s):
        d = {}
        for name, (kind, shp) in spec.items():
            if kind == "weight":
                d[name] = (rs.standard_normal(shp) * math.sqrt(2.0 / (shp[1] * shp[2] * shp[3]))).astype(np.float32)
            elif kind == "bias":
                d[name] = (rs.standard_normal(shp) * 0.05).astype(np.float32)
            elif kind == "running_mean":
                d[name] = (rs.standard_normal(shp) * 0.1).astype(np.float32)
            elif kind == "running_var":
                d[name] = rs.uniform(0.5, 1.5, shp).astype(np.float32)
            else:
                d[name] = rs.uniform(0.5, 1.0, shp).astype(np.float32)
        out.append(d)
    return out[0], out[1]


# ----------------------------------------------------------------------------------------
# Frames, camera, flow / depth / correspondences
# ----------------------------------------------------------------------------------------
def kitti_intrinsics(h=376, w=1241):
    """[cx, cy, fx, fy] scaled the way ``utils.load_kitti_odom_intrinsics`` does
    (utils.py:240-262) from the KITTI odometry seq-00 calibration."""
    return [607.1928 / 1226.0 * w, 185.2157 / 370.0 * h, 718.856 / 1226.0 * w, 718.856 / 370.0 * h]


def value_noise_image(h, w, seed, octaves=5):
    """Multi-octave value noise, RGB uint8 [h, w, 3] -- textured so the nets see structure."""
    rs = np.random.RandomState(seed)
    img = np.zeros((h, w, 3), np.float64)
    amp, tot = 1.0, 0.0
    for o in range(octaves):
        gh, gw = 3 * 2 ** o + 2, 8 * 2 ** o + 2
        g = rs.uniform(0, 1, (gh, gw, 3))
        ys = np.linspace(0, gh - 1.001, h)
        xs = np.linspace(0, gw - 1.001, w)
        y0, x0 = ys.astype(int), xs.astype(int)
        fy, fx = (ys - y0)[:, None, None], (xs - x0)[None, :, None]
        a = g[y0][:, x0] * (1 - fx) + g[y0][:, x0 + 1] * fx
        b = g[y0 + 1][:, x0] * (1 - fx) + g[y0 + 1][:, x0 + 1] * fx
        img += amp * (a * (1 - fy) + b * fy)
        tot += amp
        amp *= 0.55
    return np.clip(img / tot * 255.0, 0, 255).astype(np.uint8)


def scene_depth(h, w, K, seed):
    """Ground plane (camera height 1.65 m) below the horizon + fronto-parallel blocks above."""
    rs = np.random.RandomState(seed)
    cx, cy, fx, fy = K
    v = np.arange(h, dtype=np.float64)[:, None] + np.zeros((1, w))
    depth = np.full((h, w), 60.0)
    below = v > cy + 4
    depth[below] = np.minimum(60.0, 1.65 * fy / (v[below] - cy))
    nblk = 12
    edges = np.linspace(0, w, nblk + 1).astype(int)
    for i in range(nblk):
        d = rs.uniform(15, 60)
        top = int(rs.uniform(0.05, 0.35) * h)
        region = depth[top:int(cy) + 4, edges[i]:edges[i + 1]]
        depth[top:int(cy) + 4, edges[i]:edges[i + 1]] = np.minimum(region, d)
    return depth


def rodrigues(rvec):
    th = np.linalg.norm(rvec)
    if th < 1e-12:
        return np.eye(3)
    k = np.asarray(rvec, np.float64) / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + math.sin(th) * Kx + (1 - math.cos(th)) * Kx @ Kx


def rigid_flow(depth, K, R, t):
    """Flow ref->cur for points X_cur = R X_ref + t (pixel units, [2,h,w] float64)."""
    h, w = depth.shape
    cx, cy, fx, fy = K
    u, v = np.meshgrid(np.arange(w, dtype=np.float64), np.arange(h, dtype=np.float64))
    X = np.stack([(u - cx) / fx * depth, (v - cy) / fy * depth, depth], 0).reshape(3, -1)
    Y = R @ X + np.asarray(t, np.float64).reshape(3, 1)
    u2 = fx * Y[0] / Y[2] + cx
    v2 = fy * Y[1] / Y[2] + cy
    return np.stack([u2.reshape(h, w) - u, v2.reshape(h, w) - v], 0)


def default_motion(rs=None):
    rvec = np.array([1e-3, 1.2e-2, -5e-4])
    t = np.array([0.02, -0.01, -0.9])
    if rs is not None:
        rvec = rvec + rs.standard_normal(3) * 2e-3
        t = t + rs.standard_normal(3) * np.array([0.02, 0.01, 0.1])
    return rvec, t


def analytic_frame(seed, h=376, w=1241, outlier_frac=0.0, flow_noise=0.05, diff_sigma=0.08,
                   zero_motion=False):
    """Stage inputs for selection / RANSAC tests (SURVEY 8d): analytic rigid flow + noise,
    |N(0, sigma)| forward-backward inconsistency, optional gross outliers.

    Returns dict with float32 ``flow_fwd`` [2,h,w], ``flow_bwd`` [2,h,w], ``flow_diff`` [h,w,1],
    float32 ``depth`` [h,w] (of the *current* view, approximated by the ref depth), K, R, t.
    """
    rs = np.random.RandomState(seed)
    K = kitti_intrinsics(h, w)
    depth = scene_depth(h, w, K, seed + 1)
    rvec, t = default_motion(rs)
    if zero_motion:
        t = t * 0.0
    R = rodrigues(rvec)
    flow = rigid_flow(depth, K, R, t) + rs.standard_normal((2, h, w)) * flow_noise
    diff = np.abs(rs.standard_normal((h, w)) * diff_sigma)
    if outlier_frac > 0:
        m = rs.uniform(0, 1, (h, w)) < outlier_frac
        bad = rs.uniform(-30, 30, (2, h, w))
        flow = np.where(m[None], bad, flow)
    return {
        "flow_fwd": flow.astype(np.float32),
        "flow_bwd": (-flow).astype(np.float32),
        "flow_diff": diff.astype(np.float32)[..., None],
        "depth": depth.astype(np.float32),
        "K": K, "R": R, "t": t, "rvec": rvec,
    }


def correspondences(seed, n=2000, outlier_frac=0.3, noise=0.05, h=376, w=1241, zero_motion=False):
    """[n,2] float64 (kp_ref, kp_cur) pairs from the analytic scene; used by RANSAC tests."""
    rs = np.random.RandomState(seed)
    K = kitti_intrinsics(h, w)
    depth = scene_depth(h, w, K, seed + 1)
    rvec, t = default_motion(rs)
    if zero_motion:
        t = t * 0.0
    R = rodrigues(rvec)
    flow = rigid_flow(depth, K, R, t)
    ys = rs.randint(0, h, n)
    xs = rs.randint(0, w, n)
    kp_ref = np.stack([xs, ys], 1).astype(np.float64)
    kp_cur = kp_ref + flow[:, ys, xs].T + rs.standard_normal((n, 2)) * noise
    nout = int(round(outlier_frac * n))
    if nout:
        idx = rs.permutation(n)[:nout]
        kp_cur[idx] = kp_ref[idx] + rs.uniform(-30, 30, (nout, 2))
    return kp_ref, kp_cur, dict(K=K, R=R, t=t, depth=depth)


# ----------------------------------------------------------------------------------------
# per-frame analytic network outputs of the synthetic drive (driver golden, bench)
# ----------------------------------------------------------------------------------------
def frame_inputs(t, h, w, K, mode="normal", outlier_frac=0.0):
    """Analytic network outputs for the pair (t-1, t): forward/backward flow [2,h,w] f32, inconsistency
    [h,w,1] f32 and the CNN depth [h,w] f32 of frame t.  mode 'still' has zero translation (forces the
    GRIC check to prefer the homography -> PnP fallback); 'blind' has no consistent flow at all.
    outlier_frac > 0 replaces that fraction of the flow vectors by U(-30, 30) px without touching the
    inconsistency map (SURVEY 8d: the E-RANSAC then needs ~28 / ~410 iterations at 0.3 / 0.6)."""
    rs = np.random.RandomState(1000 + t)
    depth = scene_depth(h, w, K, 7).astype(np.float32) * np.float32(1.0 + 0.05 * np.sin(t))
    rvec, tr = default_motion(rs)
    if mode == "still":
        tr = tr * 0.0
    flow = rigid_flow(depth.astype(np.float64), K, rodrigues(rvec), tr) + rs.standard_normal((2, h, w)) * 0.05
    diff = np.abs(rs.standard_normal((h, w)) * (0.08 if mode != "blind" else 50.0))
    if outlier_frac > 0:
        ro = np.random.RandomState(5000 + t)
        m = ro.uniform(0, 1, (h, w)) < outlier_frac
        flow = np.where(m[None], ro.uniform(-30, 30, (2, h, w)), flow)
    return dict(fwd=flow.astype(np.float32), bwd=(-flow).astype(np.float32), diff=diff.astype(np.float32)[..., None],
                depth=depth, rvec=rvec, t=tr)


SEQUENCE_MODES = ["normal", "normal", "normal", "still", "normal", "blind", "normal"]      # frame t uses MODES[t]
