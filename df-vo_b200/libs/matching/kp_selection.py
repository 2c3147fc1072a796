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


def _finish(outputs, good, n, kp1, kp2, ref_data, mask=None):
    if not good:
        print("Cannot find enough good keypoints!")
        outputs["good_kp_found"] = False
        outputs["kp1_best"], outputs["kp2_best"] = {}, {}
        return outputs
    outputs["kp1_best"] = kp1.numpy()[:n][None]
    outputs["kp2_best"] = kp2.numpy()[:n][None]
    fd = ref_data["flow_diff"]
    h, w = fd.shape[0], fd.shape[1]
    if mask is not None:
        outputs["fb_flow_mask"] = tracking.DevArray(mask, (h, w))
    else:
        outputs["fb_flow_mask"] = tracking.DevArray(fd.dev, (h, w)) if isinstance(fd, tracking.DevArray) else np.asarray(fd)[:, :, 0]
    return outputs


def local_bestN(kp1, kp2, ref_data, cfg, outputs):
    """kp_selection.py:74-200 (score_method 'flow' or 'flow_ratio'); ``kp1``/``kp2`` (the dense grids of the reference) are
    accepted for signature compatibility and ignored -- the kernel derives them from the flow.  With 'flow_ratio' the
    ``fb_flow_mask`` output is the device ratio map flow_diff / |flow| (the engine's buffer, rewritten by its next selection)."""
    b = cfg.kp_selection.local_bestN
    assert b.score_method in ("flow", "flow_ratio"), "dfvo_b200 implements local_bestN score_method 'flow' and 'flow_ratio'"
    eng = tracking.default_engine()
    fd = ref_data["flow_diff"]
    assert (fd.shape[0], fd.shape[1]) == (eng.H, eng.W)
    dc = cfg.kp_selection.depth_consistency
    dd = _dev(ref_data["depth_diff"], np.float32) if dc.enable else None          # kp_selection.py:118-148
    good, n, k1, k2 = eng.select_local_bestn(_dev(fd, np.float32), _dev(ref_data["flow"], np.float32), b.num_row, b.num_col,
                                             b.num_bestN, b.thre, dd, float(dc.thre) if dc.enable else 0.05,
                                             score_method=b.score_method)
    mask = eng.flow_ratio_map if b.score_method == "flow_ratio" else None
    return _finish(outputs, good, n, k1, k2, ref_data, mask)


def bestN_flow_kp(kp1, kp2, ref_data, cfg, outputs):
    """kp_selection.py:33-71."""
    eng = tracking.default_engine()
    good, n, k1, k2 = eng.select_bestn(_dev(ref_data["flow_diff"], np.float32), _dev(ref_data["flow"], np.float32),
                                       cfg.kp_selection.bestN.num_bestN)
    return _finish(outputs, good, n, k1, k2, ref_data)


def sampled_kp(kp1, kp2, ref_data, kp_list, cfg, outputs):
    """kp_selection.py:327-378: the (cropped) dense grid at the indices ``kp_list`` -- a gather on the device-resident flow
    (Engine.sampled_keypoints); only the float64 [1, N, 2] keypoints come back to the host."""
    eng = tracking.default_engine()
    k1, k2, n = eng.sampled_keypoints(_dev(ref_data["flow"], np.float32), cfg.crop.flow_crop, len(kp_list), kp_list=kp_list)
    outputs["kp1_list"], outputs["kp2_list"] = k1.numpy()[:n][None], k2.numpy()[:n][None]
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
