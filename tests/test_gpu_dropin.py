"""GPU: the drop-in boundary on real hardware (SURVEY 8b), without a DF-VO checkout: tests/vo_driver.py replays the call
sequence of libs/dfvo.py against the UN-PATCHED mirror -- DeepModel.initialize_models (torch.load of checkpoints written
with torch.save) -> forward_depth / forward_flow (device-backed arrays) -> KeypointSampler -> EssTracker / PnpTracker.

Two things are checked: (1) what the two networks return through the facade equals the CPU oracle on the same frames;
(2) with the analytic frame inputs copied over those outputs (random-weight networks give no usable flow) the trajectory
equals the golden of the unmodified reference driver (E-tracker, PnP-fallback and constant-motion frames)."""
import os

import numpy as np
import pytest
import torch

import dropin_cases as dc
import synthdata
from oracle import nets
from util import img_to_tensor

pytestmark = pytest.mark.gpu
FEED_H, FEED_W = 96, 320


def _checkpoints(tmp):
    lfn = os.path.join(tmp, "lfn.pth")
    torch.save(nets.to_torch(synthdata.liteflownet_weights()), lfn)
    d = os.path.join(tmp, "depth")
    os.makedirs(d, exist_ok=True)
    enc, dec = synthdata.monodepth2_weights(4869, FEED_H, FEED_W)
    torch.save(nets.to_torch(enc), os.path.join(d, "encoder.pth"))      # carries 'height' / 'width' like monodepth2's encoder.pth
    torch.save(nets.to_torch(dec), os.path.join(d, "depth.pth"))
    return lfn, d, enc, dec


@pytest.mark.parametrize("golden,extra,prec", [("dfvo_driver_188x620.npz", None, "bf16"), ("dfvo_driver_188x620.npz", None, "fp32"),
                                               ("dfvo_driver_iter_188x620.npz", dc.ITERATIVE, "bf16")])
def test_driver_sequence_on_device(dev_lib, tmp_path, monkeypatch, golden, extra, prec):
    from b200 import runtime as rt_mod, tracking
    monkeypatch.setenv("DFVO_B200_PRECISION", prec)
    rt_mod.set_runtime(rt_mod.CudaRuntime(0))
    tracking._default_engine = None
    dc.fresh_libs()
    import vo_driver
    g = np.load(os.path.join(dc.G, golden))
    h, w = [int(v) for v in g["hw"]]
    n = g["poses"].shape[0]
    lfn, ddir, enc, dec = _checkpoints(str(tmp_path))
    cfg = dc.make_cfg(h, w, extra, **{"deep_flow.flow_net_weight": lfn, "depth.deep_depth.pretrained_model": ddir})
    K = synthdata.kitti_intrinsics(h, w)
    assert np.allclose(K, g["K"])
    frames = [synthdata.value_noise_image(h, w, 100 + i) for i in range(n)]
    seen = {}
    np.random.seed(cfg.seed)
    drv = vo_driver.SequenceDriver(cfg, K, frames, dc.analytic_hooks(h, w, K, seen))
    assert drv.deep_models.depth.feed_height == FEED_H and drv.deep_models.depth.feed_width == FEED_W
    poses = drv.run()
    dc.check_poses(poses, g["poses"])
    assert set(drv.modes.values()) >= {"E", "PnP", "const"}
    # (1) the facade's real network outputs vs the CPU oracle (frames 1 and 2)
    tol_flow, tol_depth = (2e-4, 2e-5) if prec == "fp32" else (0.06, 5e-2)
    p_flow = nets.to_torch(synthdata.liteflownet_weights())
    p_enc = {k: v for k, v in nets.to_torch(enc).items() if not isinstance(v, int)}
    import PIL.Image as pil
    for fid in (1, 2):
        with torch.no_grad():
            o = nets.liteflow_inference_flow(p_flow, img_to_tensor(frames[fid - 1]), img_to_tensor(frames[fid]))
            feed = np.transpose(np.asarray(pil.fromarray(frames[fid]).resize((FEED_W, FEED_H), pil.LANCZOS), np.float32) / 255, (2, 0, 1))[None]
            dref = nets.monodepth2_inference_depth(p_enc, nets.to_torch(dec), torch.from_numpy(np.ascontiguousarray(feed)))[0, 0].numpy()
        got = seen["flow"][(fid,)]
        epe = np.sqrt(((got - o["forward"][0].numpy()) ** 2).sum(0))
        assert got.shape == (2, h, w) and (epe.max() < tol_flow if prec == "fp32" else epe.mean() < tol_flow), (prec, epe.mean(), epe.max())
        dd = seen["flow"][(fid, "diff")]
        assert dd.shape == (h, w, 1)
        d = seen["depth"][fid]
        assert d.shape == (FEED_H, FEED_W) and d.dtype == np.float32
        assert (np.abs(d - dref) / dref).max() < tol_depth, (prec, (np.abs(d - dref) / dref).max())
