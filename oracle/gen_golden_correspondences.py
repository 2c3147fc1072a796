"""Generate the goldens of the reference's correspondence-selection ablations by running the REFERENCE ITSELF (a DF-VO checkout
named by DFVO_REFERENCE_ROOT, imported under oracle/shims.py), with the helpers of oracle/gen_golden.py:

    python -m oracle.gen_golden_correspondences [name ...]

  correspondences               class-level KeypointSampler results on seeded analytic frames (correspondence_frame): local
                                best-N with score_method flow_ratio (ratio map, index sets, good_kp_found; with and without the
                                depth-consistency mask), global best-N, and sampled_kp's kp1_list / kp2_list for two (flow_crop,
                                num_kp) settings
  dfvo_driver_uniform           the unmodified driver with ablation_correspondences_uniform.yml's settings
  dfvo_driver_bestn             ... with ablation_correspondences_best_n.yml's settings
  dfvo_driver_flowratio         ... with local best-N and score_method flow_ratio
"""
import hashlib
import sys

import numpy as np

from . import shims, synth


def _gg():
    from . import gen_golden                  # the reference-facing helpers; importing them needs torch and the oracle nets
    return gen_golden


UNIFORM_CFG = {"kp_selection.local_bestN.enable": False, "kp_selection.sampled_kp.enable": True,   # ablation_correspondences_uniform.yml
               "kp_selection.sampled_kp.num_kp": 2000, "e_tracker.kp_src": "kp_list", "scale_recovery.kp_src": "kp_list",
               "pnp_tracker.kp_src": "kp_list"}
BESTN_CFG = {"kp_selection.local_bestN.enable": False, "kp_selection.bestN.enable": True,          # ablation_correspondences_best_n.yml
             "kp_selection.bestN.num_bestN": 2000}
FLOWRATIO_CFG = {"kp_selection.local_bestN.score_method": "flow_ratio"}

H, W = 376, 1241
ZERO_PATCH = (slice(100, 140), slice(300, 380))          # flow_fwd = 0 there; flow_diff = 0 in its top half: 0/0 = NaN, x/0 = inf
WINDOW = (slice(90, 150), slice(290, 390))               # the ratio map's bits stored verbatim around the patch
DEPTH_THRE = 0.05

# name -> analytic_frame arguments + what to add: "zero_patch" (NaN / inf ratios), "depth" (a depth-difference map, masked selection)
CORRESPONDENCE_CASES = {"easy": dict(seed=21), "zero_patch": dict(seed=25, zero_patch=True), "depth": dict(seed=26, depth=True),
                        "toofew": dict(seed=24, diff_sigma=600.0)}
SAMPLED_SETTINGS = {"full2000": ([[0, 1], [0, 1]], 2000), "crop777": ([[0.3, 0.9], [0.1, 0.95]], 777)}


def correspondence_frame(seed, zero_patch=False, depth=False, **kw):
    """synth.analytic_frame at 376x1241, optionally with a zero-flow patch and a seeded |N(0, 0.05)| depth-difference map."""
    fr = synth.analytic_frame(h=H, w=W, seed=seed, **kw)
    if zero_patch:
        fr["flow_fwd"][:, ZERO_PATCH[0], ZERO_PATCH[1]] = 0.0
        fr["flow_diff"][100:120, ZERO_PATCH[1], 0] = 0.0
    if depth:
        fr["depth_diff"] = np.abs(np.random.RandomState(seed + 100).standard_normal((H, W)) * 0.05).astype(np.float32)
    return fr


def ratio_digest(m):
    """SHA-256 of a float32 map's bits with every NaN written as 0x7fc00000 (NaN payloads are platform-specific)."""
    b = np.ascontiguousarray(m, np.float32).view(np.uint32).copy()
    b[np.isnan(m)] = 0x7FC00000
    return hashlib.sha256(b.tobytes()).hexdigest()


def gen_correspondences():
    """Class-level goldens of the reference KeypointSampler.  Per case: <case>_ratio_{sha,nan_idx,inf_idx,window} (the flow_ratio
    fb_flow_mask: digest, NaN / inf linear indices, bits of WINDOW), <case>_ratio_good and <case>_ratio_idx_sorted (local best-N,
    flow_ratio), <case>_bestN_idx_sorted; and kp1_list_<setting> / kp2_list_<setting> of sampled_kp on the 'easy' frame."""
    ks = shims.import_reference("libs.matching.keypoint_sampler")
    gg = _gg()
    out = {}
    for name, kw in CORRESPONDENCE_CASES.items():
        fr = correspondence_frame(**kw)
        ref = {"flow": fr["flow_fwd"], "flow_diff": fr["flow_diff"], "depth": fr["depth"]}
        cur = {"depth": fr["depth"]}
        cfg = gg.build_cfg(H, W, **FLOWRATIO_CFG)
        if "depth_diff" in fr:
            cfg.kp_selection.depth_consistency.enable = True
            cfg.kp_selection.depth_consistency.thre = DEPTH_THRE
            ref["depth_diff"] = fr["depth_diff"]
        o = ks.KeypointSampler(cfg).kp_selection(cur, ref)
        out[name + "_ratio_good"] = np.array(o["good_kp_found"])
        if o["good_kp_found"]:
            kp1 = o["kp1_best"][0]
            out[name + "_ratio_idx_sorted"] = np.sort((kp1[:, 1] * W + kp1[:, 0]).astype(np.int64))
            m = o["fb_flow_mask"]
            out[name + "_ratio_sha"] = np.array(ratio_digest(m))
            out[name + "_ratio_nan_idx"] = np.flatnonzero(np.isnan(m))
            out[name + "_ratio_inf_idx"] = np.flatnonzero(np.isinf(m))
            out[name + "_ratio_window"] = np.ascontiguousarray(m[WINDOW], np.float32).view(np.uint32)
        cfg = gg.build_cfg(H, W, **BESTN_CFG)
        o = ks.KeypointSampler(cfg).kp_selection(cur, ref)
        kp1 = o["kp1_best"][0]
        out[name + "_bestN_idx_sorted"] = np.sort((kp1[:, 1] * W + kp1[:, 0]).astype(np.int64))
    fr = correspondence_frame(**CORRESPONDENCE_CASES["easy"])
    for name, (crop, num_kp) in SAMPLED_SETTINGS.items():
        cfg = gg.build_cfg(H, W, **UNIFORM_CFG)
        cfg.crop.flow_crop = crop
        cfg.kp_selection.sampled_kp.num_kp = num_kp
        o = ks.KeypointSampler(cfg).kp_selection({"depth": fr["depth"]}, {"flow": fr["flow_fwd"], "depth": fr["depth"]})
        out["kp1_list_" + name], out["kp2_list_" + name] = o["kp1_list"], o["kp2_list"]
    gg.save("correspondences_376x1241", **out)


def gen_dfvo_driver_uniform():
    """gen_dfvo_driver with uniformly sampled keypoints for the E-tracker, scale recovery and PnP."""
    _gg().gen_dfvo_driver(UNIFORM_CFG, "dfvo_driver_uniform_188x620")


def _pixel_order_patch(orig):
    """seqdata.patch_canonical_kp_order, and then, when global best-N produced kp_best, kp_best reordered by ascending pixel index:
    the order the device's best-N emits (np.argpartition's order over the whole map is implementation-defined).  Local best-N
    keeps the cell-major canonical order; the sampled list is deterministic and never reordered."""
    def patch(KeypointSampler):
        orig(KeypointSampler)
        inner = KeypointSampler.update_kp_data

        def update_kp_data(self, cur_data, ref_data, kp_sel_outputs):
            inner(self, cur_data, ref_data, kp_sel_outputs)
            sel = self.cfg.kp_selection
            if not sel.local_bestN.enable and sel.bestN.enable and hasattr(ref_data.get("kp_best"), "shape"):
                w = cur_data["depth"].shape[1]
                kp = ref_data["kp_best"]
                o = np.argsort(kp[:, 1].astype(int) * w + kp[:, 0].astype(int), kind="stable")
                ref_data["kp_best"], cur_data["kp_best"] = ref_data["kp_best"][o], cur_data["kp_best"][o]
        KeypointSampler.update_kp_data = update_kp_data
    return patch


def gen_dfvo_driver_bestn():
    """gen_dfvo_driver with global best-N, kp_best in ascending pixel index (_pixel_order_patch)."""
    from . import seqdata
    orig = seqdata.patch_canonical_kp_order
    seqdata.patch_canonical_kp_order = _pixel_order_patch(orig)
    try:
        _gg().gen_dfvo_driver(BESTN_CFG, "dfvo_driver_bestn_188x620")
    finally:
        seqdata.patch_canonical_kp_order = orig


def gen_dfvo_driver_flowratio():
    """gen_dfvo_driver with local best-N scored by flow_diff / |flow|."""
    _gg().gen_dfvo_driver(FLOWRATIO_CFG, "dfvo_driver_flowratio_188x620")


GENERATORS = {"correspondences": gen_correspondences, "dfvo_driver_uniform": gen_dfvo_driver_uniform,
              "dfvo_driver_bestn": gen_dfvo_driver_bestn, "dfvo_driver_flowratio": gen_dfvo_driver_flowratio}

if __name__ == "__main__":
    for n in sys.argv[1:] or list(GENERATORS):
        print("== generating", n)
        GENERATORS[n]()
