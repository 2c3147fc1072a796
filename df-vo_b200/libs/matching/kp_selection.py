"""Correspondence selection with the reference's function signatures (libs/matching/kp_selection.py).
The selection itself runs in the CUDA kernels of csrc/select.cu; these wrappers only marshal the data
dictionaries.  Keypoints come back in canonical order (cell-major, ascending pixel index): the reference's
order inside a cell is whatever ``np.argpartition`` produced (implementation-defined, SURVEY H2)."""
import numpy as np

from b200 import runtime, tracking


def _dev(x, dtype):
    """Device buffer of ``x`` (DevArray -> its buffer, ndarray -> upload)."""
    if isinstance(x, tracking.DevArray):
        return x.dev
    return runtime.get().from_host(np.ascontiguousarray(x, dtype))


def _finish(outputs, good, n, kp1, kp2, ref_data):
    if not good:
        print("Cannot find enough good keypoints!")
        outputs["good_kp_found"] = False
        outputs["kp1_best"], outputs["kp2_best"] = {}, {}
        return outputs
    outputs["kp1_best"] = kp1.numpy()[:n][None]
    outputs["kp2_best"] = kp2.numpy()[:n][None]
    fd = ref_data["flow_diff"]
    h, w = fd.shape[0], fd.shape[1]
    outputs["fb_flow_mask"] = tracking.DevArray(fd.dev, (h, w)) if isinstance(fd, tracking.DevArray) else np.asarray(fd)[:, :, 0]
    return outputs


def local_bestN(kp1, kp2, ref_data, cfg, outputs):
    """kp_selection.py:74-200 (score_method 'flow'); ``kp1``/``kp2`` (the dense grids of the reference) are
    accepted for signature compatibility and ignored -- the kernel derives them from the flow."""
    b = cfg.kp_selection.local_bestN
    assert b.score_method == "flow", "dfvo_b200 implements local_bestN score_method 'flow' (the default)"
    eng = tracking.default_engine()
    fd = ref_data["flow_diff"]
    assert (fd.shape[0], fd.shape[1]) == (eng.H, eng.W)
    dc = cfg.kp_selection.depth_consistency
    dd = _dev(ref_data["depth_diff"], np.float32) if dc.enable else None          # kp_selection.py:118-148
    good, n, k1, k2 = eng.select_local_bestn(_dev(fd, np.float32), _dev(ref_data["flow"], np.float32), b.num_row, b.num_col,
                                             b.num_bestN, b.thre, dd, float(dc.thre) if dc.enable else 0.05)
    return _finish(outputs, good, n, k1, k2, ref_data)


def bestN_flow_kp(kp1, kp2, ref_data, cfg, outputs):
    """kp_selection.py:33-71."""
    eng = tracking.default_engine()
    good, n, k1, k2 = eng.select_bestn(_dev(ref_data["flow_diff"], np.float32), _dev(ref_data["flow"], np.float32),
                                       cfg.kp_selection.bestN.num_bestN)
    return _finish(outputs, good, n, k1, k2, ref_data)


def sampled_kp(kp1, kp2, ref_data, kp_list, cfg, outputs):
    """kp_selection.py:327-378: uniform sub-sampling of the (cropped) dense grid -- a pure gather."""
    flow = np.asarray(ref_data["flow"])
    _, h, w = flow.shape
    y0, y1 = [int(v * h) for v in cfg.crop.flow_crop[0]]
    x0, x1 = [int(v * w) for v in cfg.crop.flow_crop[1]]
    ys, xs = np.meshgrid(np.arange(y0, y1), np.arange(x0, x1), indexing="ij")
    ys, xs = ys.reshape(-1)[kp_list], xs.reshape(-1)[kp_list]
    k1 = np.stack([xs, ys], 1).astype(np.float64)
    k2 = k1 + np.stack([flow[0, ys, xs], flow[1, ys, xs]], 1).astype(np.float64)
    outputs["kp1_list"], outputs["kp2_list"] = k1[None], k2[None]
    return outputs


def opt_rigid_flow_kp(kp1, kp2, ref_data, cfg, outputs, score_method):
    """kp_selection.py:203-324: per cell the 'uniform' list (every step-th pixel that passes both masks) and the 'best' list
    (n_best smallest ``score_method`` scores among them) from ``ref_data['rigid_flow_diff']`` [H,W,1] and
    ``ref_data['flow_diff']`` [H,W,1]; ``kp1``/``kp2`` (the reference's dense grids) are ignored -- the kernels derive the
    keypoints from ``ref_data['flow']``.  Runs on the device (csrc/select.cu: k_uniform_cells, k_local_bestn)."""
    assert score_method in ("opt_flow", "rigid_flow"), score_method
    rk = cfg.kp_selection.rigid_flow_kp
    eng = tracking.default_engine()
    h, w = eng.H, eng.W
    rmap = ref_data["rigid_flow_diff"]
    rbuf = rmap.dev if isinstance(rmap, tracking.DevArray) else runtime.get().from_host(np.ascontiguousarray(np.asarray(rmap, np.float32).reshape(h, w)))
    o = eng.opt_rigid_flow_select(rbuf, _dev(ref_data["flow"], np.float32), _dev(ref_data["flow_diff"], np.float32), rk.num_row, rk.num_col,
                                  rk.num_bestN, float(rk.rigid_flow_thre), float(rk.optical_flow_thre), score_method)
    outputs["kp1_depth"], outputs["kp2_depth"] = o["kp1_best"][None], o["kp2_best"][None]
    outputs["kp1_depth_uniform"], outputs["kp2_depth_uniform"] = o["kp1_uniform"][None], o["kp2_uniform"][None]
    outputs["rigid_flow_mask"] = tracking.DevArray(rbuf, (h, w))
    return outputs
