"""Checks of the PoseNet and the depth-consistency mask through the C ABI, shared by the CPU emulation tests
(test_depth_consistency_hostsim.py) and the GPU tests (test_gpu_depth_consistency.py).  `mem` moves arrays in and out of the
library's memory space: `mem.put(ndarray) -> buffer`, `mem.get(buffer) -> ndarray`, `mem.ptr(buffer)`."""
import os

import numpy as np
import torch

from b200 import native
from oracle import nets, pose_consistency, synth

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def golden():
    return np.load(os.path.join(G, "depth_consistency.npz"))


class HostMem:
    def put(self, a):
        return np.ascontiguousarray(a)

    def get(self, b):
        return np.array(b)

    def ptr(self, b):
        import ctypes
        return b.ctypes.data_as(ctypes.c_void_p)


class CudaMem:
    def put(self, a):
        return torch.from_numpy(np.ascontiguousarray(a)).cuda()

    def get(self, b):
        torch.cuda.synchronize()
        return b.cpu().numpy()

    def ptr(self, b):
        import ctypes
        return ctypes.c_void_p(b.data_ptr())


def posenet(lib, mem, feed_ref, feed_cur, precision, multiplier, enc=None, dec=None):
    """dfvo_posenet_forward of two [3,h,w] feeds -> float32 [4,4]."""
    if enc is None:
        enc, dec = synth.posenet_weights()
    h, w = feed_ref.shape[-2:]
    ctx = native.Context(lib)
    ctx.load_weights(native.NET_POSENET, enc)
    ctx.load_weights(native.NET_POSENET, dec)
    ctx.posenet_build(h, w, precision, multiplier)
    a, b = mem.put(np.asarray(feed_ref, np.float32)[None]), mem.put(np.asarray(feed_cur, np.float32)[None])
    out = mem.put(np.zeros((4, 4), np.float32))
    ctx.posenet_forward(mem.ptr(a), mem.ptr(b), mem.ptr(out), None)
    r = mem.get(out)
    ctx.close()
    return r


def pose_parameters_of(T, multiplier):
    """(axis-angle, translation) that transformation_from_parameters(invert=True) and the multiplier turned into T."""
    R = T[:3, :3].astype(np.float64).T
    t = -(R @ (T[:3, 3].astype(np.float64) / multiplier))
    angle = np.arccos(np.clip((np.trace(R) - 1) / 2, -1, 1))
    axis = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]]) / (2 * np.sin(angle))
    return axis * angle, t


def depth_consistency(lib, mem, cur, ref, T, K):
    """dfvo_depth_consistency with K = [cx, cy, fx, fy] (float64 mat / inv_mat cast to float32 like the reference)."""
    cx, cy, fx, fy = K
    Km = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float64)
    K32 = np.ascontiguousarray(Km, np.float32)
    iK32 = np.ascontiguousarray(np.linalg.inv(Km), np.float32)
    H, W = cur.shape
    c, r, t = mem.put(np.asarray(cur, np.float32)), mem.put(np.asarray(ref, np.float32)), mem.put(np.asarray(T, np.float32))
    out = mem.put(np.full((H, W), -7.0, np.float32))
    lib.check(lib.dfvo_depth_consistency(mem.ptr(c), mem.ptr(r), H, W, mem.ptr(t), K32.ctypes.data_as(__import__("ctypes").c_void_p),
                                         iK32.ctypes.data_as(__import__("ctypes").c_void_p), mem.ptr(out), None))
    return mem.get(out)


def compare_depth_diff(got, want, thre=0.05, tol=1e-6, tol_max=5e-4):
    """NaN exactly where the reference has NaN; values within `tol` on at least 90 % of the pixels and within `tol_max` everywhere
    (the rest sample the reference depth across a jump, where the last-bit differences of torch's sgemm accumulation order in
    the projected coordinates are multiplied by the depth gradient); the `< thre` mask bit-equal except where
    |want - thre| < tol_max.  Returns the number of such borderline pixels."""
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan)
    d = np.abs(got[~nan] - want[~nan])
    assert (d <= tol).mean() >= 0.9 and d.max() <= tol_max, ((d <= tol).mean(), d.max())
    border = np.abs(want - thre) < tol_max
    assert np.array_equal((got < thre)[~border], (want < thre)[~border])
    return int(border.sum())


def select_with_mask(lib, mem, flow_diff, depth_diff, depth_thre, num_bestN=2000, thre=0.1):
    """dfvo_local_bestn with the depth mask -> sorted selected linear indices."""
    H, W = flow_diff.shape
    fd, dd = mem.put(np.asarray(flow_diff, np.float32)), mem.put(np.asarray(depth_diff, np.float32))
    idx, cc, st = mem.put(np.zeros(num_bestN, np.int32)), mem.put(np.zeros(100, np.int32)), mem.put(np.zeros(4, np.int32))
    lib.check(lib.dfvo_local_bestn(mem.ptr(fd), mem.ptr(dd), H, W, 10, 10, num_bestN, thre, depth_thre, mem.ptr(idx), mem.ptr(cc),
                                   mem.ptr(st), None))
    i = mem.get(idx)
    assert mem.get(st)[0] == 1
    return np.sort(i[i >= 0]).astype(np.int64)


def oracle_pose(feed_ref, feed_cur, multiplier):
    enc, dec = synth.posenet_weights()
    return pose_consistency.posenet_inference_pose(nets.to_torch(enc), nets.to_torch(dec), torch.from_numpy(feed_ref)[None],
                                                   torch.from_numpy(feed_cur)[None], multiplier)
