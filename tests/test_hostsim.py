"""CPU: the library's own .cu sources compiled for the host against an emulation of the CUDA execution
model (tests/hostsim) -- validates kernel indexing, layouts, weight packing and the network / RANSAC
orchestration against the oracle and the reference-generated goldens before GPU time is spent.
(The wgmma kernels themselves cannot run here; its host emulation consumes the same ConvTc description and
packed weights, so the bf16 plumbing is covered, the PTX is covered by tests/test_gpu_*.py.)"""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from b200 import native
from oracle import cvreplay, nets, synth, vo
from util import bf16_round, hptr, img_to_tensor

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.mark.parametrize("B,C,H,W,s,prec", [(1, 64, 9, 13, 1, 0), (2, 32, 11, 14, 2, 0), (1, 96, 8, 36, 1, 1)])
def test_correlation(hostsim_lib, B, C, H, W, s, prec):
    rs = np.random.RandomState(C)
    a = rs.standard_normal((B, C, H, W)).astype(np.float32)
    b = rs.standard_normal((B, C, H, W)).astype(np.float32)
    if prec:
        a, b = bf16_round(a), bf16_round(b)
    ref = F.leaky_relu(nets.correlation(torch.from_numpy(a), torch.from_numpy(b), s), 0.1).numpy()
    out = np.zeros_like(ref)
    hostsim_lib.check(hostsim_lib.dfvo_correlation(hptr(a), hptr(b), hptr(out), B, C, H, W, s, 1, prec, None))
    assert np.abs(out - ref).max() < (1e-5 if prec == 0 else 1e-2)


def test_warp_and_fb(hostsim_lib):
    g = np.load(os.path.join(G, "warp_fb.npz"))
    x, fl = np.ascontiguousarray(g["warp_x"]), np.ascontiguousarray(g["warp_flow"])
    out = np.zeros_like(x)
    hostsim_lib.check(hostsim_lib.dfvo_backward_warp(hptr(x), hptr(fl), hptr(out), *x.shape, 0, None))
    assert np.abs(out - g["warp_out"]).max() < 2e-5              # vs the reference's own Backward()
    fwd, bwd = np.ascontiguousarray(g["fb_fwd"][0]), np.ascontiguousarray(g["fb_bwd"][0])
    d = np.zeros(fwd.shape[1:], np.float32)
    hostsim_lib.check(hostsim_lib.dfvo_fb_consistency(hptr(fwd), hptr(bwd), hptr(d), fwd.shape[1], fwd.shape[2], None))
    assert np.abs(d - g["fb_diff"][0, :, :, 0]).max() < 2e-5      # vs DeepFlow.forward_backward_consistency
    f2, b2 = np.ascontiguousarray(np.stack([fwd, bwd])), np.ascontiguousarray(np.stack([bwd, fwd]))
    d2 = np.zeros((2,) + fwd.shape[1:], np.float32)
    hostsim_lib.check(hostsim_lib.dfvo_fb_consistency_batch(hptr(f2), hptr(b2), hptr(d2), 2, fwd.shape[1], fwd.shape[2], None))
    assert np.array_equal(d2[0], d)


@pytest.mark.parametrize("case", [(1, 3, 12, 20, 8, 7, 7, 1, 3, 3, 0, 1, 0), (1, 16, 9, 14, 24, 3, 3, 2, 1, 1, 0, 2, 0),
                                  (1, 16, 8, 12, 8, 3, 3, 1, 1, 1, 1, 3, 0), (1, 49, 7, 20, 20, 3, 3, 1, 1, 1, 0, 1, 1),
                                  (1, 32, 6, 18, 2, 5, 5, 1, 2, 2, 0, 0, 1), (2, 32, 8, 12, 48, 3, 3, 2, 1, 1, 0, 1, 1),
                                  (1, 64, 6, 10, 32, 1, 1, 2, 0, 0, 0, 0, 1)])
def test_conv2d(hostsim_lib, case):
    B, Cin, H, W, Cout, kh, kw, st, py, px, refl, act, prec = case
    rs = np.random.RandomState(Cin + Cout)
    x = rs.standard_normal((B, Cin, H, W)).astype(np.float32)
    w = (rs.standard_normal((Cout, Cin, kh, kw)) / np.sqrt(Cin * kh * kw)).astype(np.float32)
    b = (rs.standard_normal(Cout) * 0.1).astype(np.float32)
    if prec:
        x, w = bf16_round(x), bf16_round(w)
    xin = F.pad(torch.from_numpy(x), (px, px, py, py), mode="reflect") if refl else torch.from_numpy(x)
    y = F.conv2d(xin, torch.from_numpy(w), torch.from_numpy(b), stride=st, padding=(0, 0) if refl else (py, px))
    y = {0: lambda t: t, 1: lambda t: F.leaky_relu(t, 0.1), 2: F.relu, 3: F.elu}[act](y).numpy()
    out = np.zeros_like(y)
    hostsim_lib.check(hostsim_lib.dfvo_conv2d(hptr(x), hptr(w), hptr(b), hptr(out), B, Cin, H, W, Cout, kh, kw, st, py, px, refl,
                                              act, prec, None))
    assert np.abs(out - y).max() < (2e-5 if prec == 0 else 1.5e-2)


def test_liteflownet_pipeline_vs_reference_golden(hostsim_lib):
    """Whole flow path (uint8 frames -> flows + consistency map) in fp32 mode against the golden produced
    by the reference's DeepModel.forward_flow (tests/golden/deep_models_70x150.npz)."""
    g = np.load(os.path.join(G, "deep_models_70x150.npz"))
    H, W = 70, 150
    ref, cur = synth.value_noise_image(H, W, 1), synth.value_noise_image(H, W, 2)
    ctx = native.Context(hostsim_lib)
    ctx.load_weights(native.NET_LITEFLOWNET, synth.liteflownet_weights())
    ctx.liteflow_build(H, W, 1, native.PREC_FP32)
    assert ctx.liteflow_geometry() == (64, 128, 2)
    fwd, bwd, diff = np.zeros((2, H, W), np.float32), np.zeros((2, H, W), np.float32), np.zeros((H, W), np.float32)
    ctx.liteflow_forward([ref.ctypes.data, cur.ctypes.data], hptr(fwd), hptr(bwd), hptr(diff))
    assert np.abs(fwd - g["flow_fwd"]).max() < 5e-5 and np.abs(bwd - g["flow_bwd"]).max() < 5e-5
    assert np.abs(diff - g["flow_diff"][:, :, 0]).max() < 2e-4
    assert np.abs(g["flow_fwd"]).max() > 1.0


def test_liteflownet_bf16_plumbing(hostsim_lib):
    H, W = 64, 128
    ref, cur = synth.value_noise_image(H, W, 1), synth.value_noise_image(H, W, 2)
    w = synth.liteflownet_weights()
    with torch.no_grad():
        o = nets.liteflow_inference_flow(nets.to_torch(w), img_to_tensor(ref), img_to_tensor(cur))
    ctx = native.Context(hostsim_lib)
    ctx.load_weights(native.NET_LITEFLOWNET, w)
    ctx.liteflow_build(H, W, 1, native.PREC_BF16)
    fwd, bwd, diff = np.zeros((2, H, W), np.float32), np.zeros((2, H, W), np.float32), np.zeros((H, W), np.float32)
    ctx.liteflow_forward([ref.ctypes.data, cur.ctypes.data], hptr(fwd), hptr(bwd), hptr(diff))
    epe = np.sqrt(((fwd - o["forward"][0].numpy()) ** 2).sum(0))
    assert epe.mean() < 0.05 and epe.max() < 0.5


def test_tf32_mode_plumbing(hostsim_lib):
    """DFVO_PREC_TF32 wiring (fp32 activations, layers packed for 4-byte tensor-core operands, im2row stem, CUDA-core heads):
    in the CPU emulation the wgmma tf32 convs are exact fp32 arithmetic on tf32-rounded weights, so both networks must
    land within tf32 weight-rounding distance of the reference goldens."""
    g = np.load(os.path.join(G, "deep_models_70x150.npz"))
    H, W = 70, 150
    ref, cur = synth.value_noise_image(H, W, 1), synth.value_noise_image(H, W, 2)
    ctx = native.Context(hostsim_lib)
    ctx.load_weights(native.NET_LITEFLOWNET, synth.liteflownet_weights())
    ctx.liteflow_build(H, W, 1, native.PREC_TF32)
    fwd, bwd, diff = np.zeros((2, H, W), np.float32), np.zeros((2, H, W), np.float32), np.zeros((H, W), np.float32)
    ctx.liteflow_forward([ref.ctypes.data, cur.ctypes.data], hptr(fwd), hptr(bwd), hptr(diff))
    epe = np.sqrt(((fwd - g["flow_fwd"]) ** 2).sum(0))
    assert epe.mean() < 5e-3 and epe.max() < 5e-2, (epe.mean(), epe.max())
    fh, fw = [int(x) for x in g["feed_hw"]]
    enc, dec = synth.monodepth2_weights(4869, fh, fw)
    ctx.load_weights(native.NET_MONODEPTH2, enc); ctx.load_weights(native.NET_MONODEPTH2, dec)
    ctx.monodepth2_build(fh, fw, native.PREC_TF32)
    out = np.zeros((fh, fw), np.float32)
    ctx.monodepth2_forward(hptr(np.ascontiguousarray(g["depth_feed"][None])), hptr(out))
    assert (np.abs(out - g["depth"]) / g["depth"]).max() < 2e-3


def test_liteflownet_two_pairs_batched(hostsim_lib):
    """The batched many-pairs mode (BASELINE configs[2] / SURVEY 8e pair-level sharding): two independent frame pairs in one
    forward (batch of 4 images, 'second image' = n ^ 1 inside each pair) give, pair by pair, exactly what each pair gives
    alone -- same kernels, same per-image arithmetic."""
    H, W = 64, 128
    imgs = [synth.value_noise_image(H, W, s) for s in (1, 2, 3, 4)]
    w = synth.liteflownet_weights()

    def run(pairs, frames):
        ctx = native.Context(hostsim_lib)
        ctx.load_weights(native.NET_LITEFLOWNET, w)
        ctx.liteflow_build(H, W, pairs, native.PREC_BF16)
        fwd, bwd = np.zeros((pairs, 2, H, W), np.float32), np.zeros((pairs, 2, H, W), np.float32)
        diff = np.zeros((pairs, H, W), np.float32)
        ctx.liteflow_forward([f.ctypes.data for f in frames], hptr(fwd), hptr(bwd), hptr(diff))
        ctx.close()
        return fwd, bwd, diff

    f2, b2, d2 = run(2, imgs)
    for p in (1,):                                      # the second pair (batch indices 2, 3) is the non-trivial one
        f1, b1, d1 = run(1, imgs[2 * p:2 * p + 2])
        assert np.array_equal(f2[p], f1[0]) and np.array_equal(b2[p], b1[0]) and np.array_equal(d2[p], d1[0]), p
    assert np.abs(f2[0] - f2[1]).max() > 1e-3          # the two pairs really are different problems


def test_monodepth2_vs_reference_golden(hostsim_lib):
    g = np.load(os.path.join(G, "deep_models_70x150.npz"))
    fh, fw = [int(x) for x in g["feed_hw"]]
    enc, dec = synth.monodepth2_weights(4869, fh, fw)
    ctx = native.Context(hostsim_lib)
    ctx.load_weights(native.NET_MONODEPTH2, enc); ctx.load_weights(native.NET_MONODEPTH2, dec)
    ctx.monodepth2_build(fh, fw, native.PREC_FP32)
    out = np.zeros((fh, fw), np.float32)
    ctx.monodepth2_forward(hptr(np.ascontiguousarray(g["depth_feed"][None])), hptr(out))
    assert (np.abs(out - g["depth"]) / g["depth"]).max() < 2e-5


def test_monodepth2_bf16_stem_on_tensor_core_path(hostsim_lib):
    """bf16 mode: the 7x7 stride-2 stem as a 4x1 window conv over the two row-parity views of the column-padded image
    (monodepth2.cu::stem_tc_layer; weight packing, views and taps are host logic, the MMAs are emulated) vs the reference golden."""
    g = np.load(os.path.join(G, "deep_models_70x150.npz"))
    fh, fw = [int(x) for x in g["feed_hw"]]
    enc, dec = synth.monodepth2_weights(4869, fh, fw)
    ctx = native.Context(hostsim_lib)
    ctx.load_weights(native.NET_MONODEPTH2, enc); ctx.load_weights(native.NET_MONODEPTH2, dec)
    ctx.monodepth2_build(fh, fw, native.PREC_BF16)
    out = np.zeros((fh, fw), np.float32)
    ctx.monodepth2_forward(hptr(np.ascontiguousarray(g["depth_feed"][None])), hptr(out))
    rel = np.abs(out - g["depth"]) / g["depth"]
    assert rel.max() < 3e-2 and rel.mean() < 3e-3, (rel.max(), rel.mean())


def test_selection_vs_reference_golden(hostsim_lib):
    g = np.load(os.path.join(G, "selection_376x1241.npz"))
    H, W = 376, 1241
    fr = synth.analytic_frame(h=H, w=W, seed=22, outlier_frac=0.3, diff_sigma=0.12)
    diff = np.ascontiguousarray(fr["flow_diff"][..., 0])
    idx, cc, st = np.zeros(2000, np.int32), np.zeros(100, np.int32), np.zeros(4, np.int32)
    hostsim_lib.check(hostsim_lib.dfvo_local_bestn(hptr(diff), None, H, W, 10, 10, 2000, 0.1, 0.05, hptr(idx), hptr(cc), hptr(st), None))
    assert st[0] == 1 and np.array_equal(np.sort(idx[idx >= 0]), g["outliers_local_bestN_idx_sorted"])


def test_five_point_and_essential_ransac_vs_cv2(hostsim_lib):
    g = np.load(os.path.join(G, "cv_solvers.npz"))
    cx, cy, fx, fy = synth.kitti_intrinsics()
    N, MI = 2000, 1000
    kp_ref, kp_cur, _ = synth.correspondences(n=N, seed=42, outlier_frac=0.3)
    subsets = np.zeros((MI, 5), np.int32)
    hostsim_lib.check(hostsim_lib.dfvo_cv_subset_stream_host(N, 5, MI, hptr(subsets)))
    assert np.array_equal(subsets, cvreplay.subset_stream(N, 5, MI))
    ws = np.zeros(hostsim_lib.dfvo_essential_workspace_bytes(N, 1, MI), np.uint8)
    E, mask, info, gric = np.zeros((1, 9)), np.zeros((1, N), np.uint8), np.zeros((1, 4), np.int32), np.zeros(1)
    p1, p2 = np.ascontiguousarray(kp_cur), np.ascontiguousarray(kp_ref)
    hostsim_lib.check(hostsim_lib.dfvo_essential_ransac(hptr(p1), hptr(p2), N, None, 1, hptr(subsets), MI, fx, fy, cx, cy, 0.2, 0.99,
                                                        hptr(ws), ws.size, hptr(E), hptr(mask), hptr(info), hptr(gric), None))
    Eref = g["out30_E"]
    assert min(np.abs(E[0].reshape(3, 3) - Eref).max(), np.abs(E[0].reshape(3, 3) + Eref).max()) < 1e-10
    assert np.array_equal(mask[0], g["out30_mask"]) and info[0, 1] == 28          # same stopping iteration as cv2
    Rt, pm, pi = np.zeros(12), np.zeros(N, np.uint8), np.zeros(5, np.int32)
    hostsim_lib.check(hostsim_lib.dfvo_recover_pose(hptr(np.ascontiguousarray(Eref)), hptr(p1), hptr(p2), N, fx, cx, cy, hptr(Rt),
                                                    hptr(pm), hptr(pi), None))
    assert pi[0] == int(g["out30_cheir"]) and np.abs(Rt[:9].reshape(3, 3) - g["out30_R"]).max() < 1e-12
    assert np.array_equal(pm, (g["out30_pmask"] > 0).astype(np.uint8))


def test_tracker_orchestration_vs_reference_classes(hostsim_lib):
    """b200.tracking.compute_pose_2d2d / find_scale_from_depth == reference EssTracker (golden)."""
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim"))
    from runtime import HostsimRuntime
    from b200 import runtime as rt_mod, tracking
    rt_mod.set_runtime(HostsimRuntime(hostsim_lib))
    eng = tracking.Engine(376, 1241)
    g = np.load(os.path.join(G, "trackers_2000.npz"))
    K = synth.kitti_intrinsics()
    for name, kw in {"out30": dict(seed=32, outlier_frac=0.3), "still": dict(seed=34, outlier_frac=0.1, zero_motion=True)}.items():
        kp_ref, kp_cur, info = synth.correspondences(n=2000, **kw)
        np.random.seed(4869)
        r = tracking.compute_pose_2d2d(eng, kp_ref, kp_cur, K)
        pose = np.eye(4); pose[:3, :3] = r["R"]; pose[:3, 3:] = r["t"]
        assert np.abs(pose - g[name + "_pose"]).max() < 1e-10
        assert np.array_equal(r["inliers"], g[name + "_inliers"])
        if np.linalg.norm(r["t"]) != 0:
            depth = info["depth"].astype(np.float32)
            dp = (depth * ((depth < 50) & (depth > 0))).astype(np.float64)
            s = tracking.find_scale_from_depth(eng, kp_ref, kp_cur, np.linalg.inv(pose), dp, K)
            assert abs(s - float(g[name + "_scale"])) < 1e-10


def test_lanczos_feed_bit_exact_with_pil(hostsim_lib):
    """deep_models.py:195-198: the device resize (run here in emulation) equals PIL.Image.resize(LANCZOS)
    + ToTensor bit for bit."""
    import PIL.Image as pil
    from b200 import lanczos
    for (H, W, oh, ow, seed) in [(376, 1241, 192, 640, 1), (70, 150, 64, 96, 2), (100, 300, 128, 416, 3)]:
        rs = np.random.RandomState(seed)
        img = synth.value_noise_image(H, W, seed) if seed != 2 else rs.randint(0, 256, (H, W, 3)).astype(np.uint8)
        ref = np.asarray(pil.fromarray(img).resize((ow, oh), pil.LANCZOS))
        bh, kh, ksh = lanczos.coeffs(W, ow)
        bv, kv, ksv = lanczos.coeffs(H, oh)
        tmp, out, f = np.zeros((H, ow, 3), np.uint8), np.zeros((oh, ow, 3), np.uint8), np.zeros((3, oh, ow), np.float32)
        hostsim_lib.check(hostsim_lib.dfvo_lanczos_resize_u8(hptr(img), H, W, hptr(bh), hptr(kh), ksh, hptr(bv), hptr(kv), ksv, oh, ow,
                                                              hptr(tmp), hptr(out), hptr(f), None))
        assert np.array_equal(out, ref)
        assert np.array_equal(f, np.transpose(ref, (2, 0, 1)).astype(np.float32) / np.float32(255))
