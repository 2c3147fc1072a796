"""CPU restatements of the monodepth2 PoseNet and of DepthConsistency in torch, pinned to the reference by
tests/golden/depth_consistency.npz (oracle/gen_golden_depth_consistency.py) and used as the full-size reference of the GPU tests.

  posenet_inference_pose  Monodepth2PoseNet.inference_pose (pose/monodepth2/monodepth2.py:86-119, pose_decoder.py,
                          depth/monodepth2/layers.py:28-94)
  depth_consistency       DepthConsistency.compute (depth_consistency.py:31-163)
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import nets


def selection_depth_diff(h, w, seed=31):
    """Seeded depth_diff map for the masked local_bestN goldens: uniform in [0, 0.1) with a NaN block (a 0/0 region)."""
    rs = np.random.RandomState(seed)
    dd = rs.uniform(0.0, 0.1, (h, w)).astype(np.float32)
    dd[h // 4:h // 4 + 40, w // 5:w // 5 + 200] = np.nan
    return dd


def pose_parameters(enc, dec, feed_ref, feed_cur):
    """ResnetEncoder(18, False, 2) + PoseDecoder on [1,3,h,w] feeds -> (axisangle [3], translation [3]) of frame 0."""
    x = torch.cat([feed_ref, feed_cur], 1)
    f = nets.resnet18_encoder(enc, x)[-1]
    out = F.relu(F.conv2d(f, dec["net.0.weight"], dec["net.0.bias"]))
    out = F.relu(F.conv2d(out, dec["net.1.weight"], dec["net.1.bias"], padding=1))
    out = F.relu(F.conv2d(out, dec["net.2.weight"], dec["net.2.bias"], padding=1))
    out = F.conv2d(out, dec["net.3.weight"], dec["net.3.bias"])
    out = 0.01 * out.mean(3).mean(2).view(-1, 2, 1, 6)
    return out[0, 0, 0, :3], out[0, 0, 0, 3:]


def transformation_from_parameters(axisangle, translation, baseline=1.0):
    """transformation_from_parameters(axisangle, translation, invert=True) (layers.py:28-94) and the baseline multiplier
    (monodepth2.py:117-118) -> float32 [4,4] tensor."""
    vec = axisangle.reshape(1, 1, 3)
    angle = torch.norm(vec, 2, 2, True)
    axis = vec / (angle + 1e-7)
    ca, sa = torch.cos(angle), torch.sin(angle)
    C = 1 - ca
    x, y, z = axis[..., 0], axis[..., 1], axis[..., 2]
    xs, ys, zs = x * sa[..., 0], y * sa[..., 0], z * sa[..., 0]
    xC, yC, zC = x * C[..., 0], y * C[..., 0], z * C[..., 0]
    xyC, yzC, zxC = x * yC, y * zC, z * xC
    ca = ca[..., 0]
    R = torch.zeros(4, 4)
    R[0, 0], R[0, 1], R[0, 2] = (x * xC + ca)[0, 0], (xyC - zs)[0, 0], (zxC + ys)[0, 0]
    R[1, 0], R[1, 1], R[1, 2] = (xyC + zs)[0, 0], (y * yC + ca)[0, 0], (yzC - xs)[0, 0]
    R[2, 0], R[2, 1], R[2, 2] = (zxC - ys)[0, 0], (yzC + xs)[0, 0], (z * zC + ca)[0, 0]
    R[3, 3] = 1
    T = torch.eye(4)
    T[:3, 3] = -translation.reshape(3)
    M = torch.matmul(R.t(), T)
    M[:3, 3] *= baseline
    return M


def posenet_inference_pose(enc, dec, feed_ref, feed_cur, baseline=1.0):
    """Monodepth2PoseNet.inference_pose([ref, cur]) -> float32 [4,4] numpy."""
    with torch.no_grad():
        aa, t = pose_parameters(enc, dec, feed_ref, feed_cur)
        return transformation_from_parameters(aa, t, baseline).numpy()


def depth_consistency(depth_cur, depth_ref, T, K, inv_K):
    """DepthConsistency.compute: [H,W] raw depths, float32 4x4 pose, float64 3x3 K / inv_K -> depth_diff [H,W] float32
    (clamp(|warp - reproj| / reproj, 0, 1), grid_sample border padding with align_corners=True)."""
    H, W = depth_cur.shape
    K4, iK4 = np.eye(4), np.eye(4)
    K4[:3, :3], iK4[:3, :3] = K, inv_K
    K4 = torch.from_numpy(K4).float()
    iK4 = torch.from_numpy(iK4).float()
    T = torch.from_numpy(np.asarray(T, np.float32))
    d = torch.from_numpy(np.ascontiguousarray(depth_cur, np.float32)).view(1, -1)
    ys, xs = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    pix = torch.from_numpy(np.stack([xs.reshape(-1), ys.reshape(-1), np.ones(H * W)]).astype(np.float32))
    cam = torch.cat([d * torch.matmul(iK4[:3, :3], pix), torch.ones(1, H * W)], 0)          # Backprojection
    q = torch.matmul(T, cam)                                                                  # Transformation3D
    p2 = torch.matmul(K4[:3, :], q)                                                           # Projection
    xy = (p2[:2] / (p2[2:3] + 1e-7)).view(2, H, W).permute(1, 2, 0).clone()
    xy[..., 0] /= W - 1
    xy[..., 1] /= H - 1
    xy = (xy - 0.5) * 2
    ref = torch.from_numpy(np.ascontiguousarray(depth_ref, np.float32)).view(1, 1, H, W)
    warp = F.grid_sample(ref, xy[None], padding_mode="border", align_corners=True)[0, 0]
    reproj = torch.matmul(T[:3, :], cam)[2].view(H, W)
    return ((warp - reproj).abs() / reproj).clamp(0, 1).numpy()
