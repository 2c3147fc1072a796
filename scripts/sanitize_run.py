"""Small pass over every kernel family of the hot path, meant to run under compute-sanitizer (memcheck / racecheck / synccheck):
LiteFlowNet (per-layer and chained convs, fused warp+correlation), monodepth2, consistency, selection, E / H / PnP RANSAC, and a
short two-sequence multiseq.SequenceBatch run (batched monodepth2, PoseNet and LiteFlowNet).
No oracle here -- the parity tests do the checking; this run only has to be clean.  Usage (on a GPU):
  compute-sanitizer --tool memcheck python scripts/sanitize_run.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "df-vo_b200"))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from b200 import native, runtime as rt_mod, tracking      # noqa: E402
from oracle import synth                                   # noqa: E402  (seeded synthetic weights / frames only)
import synthdata                                           # noqa: E402


def main():
    rt = rt_mod.CudaRuntime(0)
    rt_mod.set_runtime(rt)
    H, W = 128, 416
    K = synthdata.kitti_intrinsics(H, W)
    for chain in (0, 1):
        rt.lib.dfvo_set_conv_chain(chain)
        eng = tracking.Engine(H, W, rt)
        eng.build_flow(synth.liteflownet_weights(), precision=native.PREC_BF16)
        enc, dec = synth.monodepth2_weights(4869, 64, 96)
        eng.build_depth(enc, dec, precision=native.PREC_BF16)
        ref, cur = synth.value_noise_image(H, W, 1), synth.value_noise_image(H, W, 2)
        fwd, bwd, diff = eng.flow([rt.from_host(ref), rt.from_host(cur)])
        feed = np.random.RandomState(0).uniform(0, 1, (1, 3, 64, 96)).astype(np.float32)
        d = eng.depth(rt.from_host(feed)).numpy()
        assert np.isfinite(fwd.numpy()).all() and np.isfinite(d).all()
        print("nets ok (chains %d)" % chain, flush=True)
    rt.lib.dfvo_set_conv_chain(0)
    # two sequences on one GPU: batched monodepth2 / PoseNet / LiteFlowNet (S = 2), one sequence idle for a step
    from b200 import config, multiseq
    cfg = config.default_cfg(H, W)
    cfg.deep_pose.enable = cfg.kp_selection.depth_consistency.enable = True
    penc, pdec = synth.posenet_weights()
    for overlap in (False, True):
        b = multiseq.SequenceBatch([K, K], H, W, cfg=cfg, overlap=overlap, runtime=rt)
        b.load_weights(synth.liteflownet_weights(), *synth.monodepth2_weights(4869, 64, 96), penc, pdec)
        imgs = [synth.value_noise_image(H, W, 10 + i) for i in range(4)]
        for row in ([imgs[0], imgs[1]], [imgs[2], None], [imgs[3], imgs[2]]):
            b.step(row)
        b.flush()
        rt.sync()
        print("SequenceBatch ok (overlap %d): frames tracked %s" % (overlap, [len(p) for p in b.poses]), flush=True)
    eng = tracking.Engine(376, 1241, rt)              # the synthetic correspondences / depths are KITTI-sized
    for seed, outl, still in [(31, 0.0, False), (33, 0.6, False), (34, 0.1, True)]:
        kp_ref, kp_cur, info = synthdata.correspondences(n=600, seed=seed, outlier_frac=outl, zero_motion=still)
        np.random.seed(4869)
        r = tracking.compute_pose_2d2d(eng, kp_ref, kp_cur, synthdata.kitti_intrinsics())
        depth = np.clip(info["depth"], 0, 49).astype(np.float64)
        ki = kp_ref.astype(int)
        ok = (ki[:, 0] >= 0) & (ki[:, 0] < depth.shape[1]) & (ki[:, 1] >= 0) & (ki[:, 1] < depth.shape[0])
        dd = depth[ki[ok, 1], ki[ok, 0]]
        keep = dd > 0
        T, ninl = tracking.compute_pose_3d2d(eng, kp_ref[ok][keep], kp_cur[ok][keep], dd[keep], synthdata.kitti_intrinsics())
        # the fused device-side tail (recoverPose, vote, depth ratios incl. the block sort, scale RANSAC with the MT19937 stream)
        n = kp_ref.shape[0]
        np.random.seed(4869)
        perms = [np.random.permutation(n) for _ in range(5)]
        b_ref, b_cur = rt.from_host(kp_ref), rt.from_host(kp_cur)
        b_depth = rt.from_host(np.ascontiguousarray(depth, np.float32))
        h = eng.homography_launch(b_cur, b_ref, n)
        w = eng.essential_launch(b_cur, b_ref, n, perms, synthdata.kitti_intrinsics(), threshold=0.2)
        o = eng.essential_tail(w, h, b_cur, b_ref, n, synthdata.kitti_intrinsics(), b_depth, np.random)
        print("trackers ok (outliers %.1f still %d): E inliers %d, PnP inliers %d, fused tail: valid %s scale %.4f status %d" %
              (outl, still, int(r["inliers"].sum()), ninl, o["valid"], o["scale"], o["scale_status"]), flush=True)
    print("sanitize_run done")


if __name__ == "__main__":
    main()
