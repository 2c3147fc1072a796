"""Throughput of FramePipeline under the tracking configurations the device runs: hybrid with GRIC model selection (the
default), hybrid with the flow-magnitude check (ablation_model_sel_flow.yml: e_tracker.validity.method flow, thre 5), PnP-only
(ablation_tracker_pnp.yml: tracking_method PnP), and the correspondence-selection ablations: uniformly sampled keypoints
(ablation_correspondences_uniform.yml), global best-N (ablation_correspondences_best_n.yml) and local best-N with
score_method flow_ratio.  Same frames, analytic flow / depth injection and default execution mode as
bench.py (376x1241, three network engines in flight, pipelined tracker).  Prints one JSON line per configuration: frames/s and
the tracker's host milliseconds per frame (enqueue + read, including its device waits) by branch.

    python scripts/track_modes.py [--steps 200] [--warmup 20]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "df-vo_b200"))

import numpy as np  # noqa: E402

import bench  # noqa: E402  (frame cycle and sizes only)

CONFIGS = {"hybrid/GRIC": {}, "hybrid/flow": {"e_tracker.validity": dict(method="flow", thre=5)}, "PnP": {"tracking_method": "PnP"},
           "uniform": {"kp_selection.local_bestN.enable": False, "kp_selection.sampled_kp.enable": True, "e_tracker.kp_src": "kp_list",
                       "scale_recovery.kp_src": "kp_list", "pnp_tracker.kp_src": "kp_list"},
           "bestN": {"kp_selection.local_bestN.enable": False, "kp_selection.bestN.enable": True},
           "local_bestN/flow_ratio": {"kp_selection.local_bestN.score_method": "flow_ratio"}}


def configure(cfg, over):
    """Sets the dotted keys of `over` in `cfg` (dict values become config nodes)."""
    from b200 import config
    for k, v in over.items():
        node = cfg
        *path, last = k.split(".")
        for part in path:
            node = node[part]
        node[last] = config.AttrDict(v) if isinstance(v, dict) else v
    return cfg


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    import torch
    import synthdata as synth
    from b200 import config, native, pipeline, runtime as rt_mod
    H, W, N = bench.H, bench.W, bench.N_DISTINCT
    rt = rt_mod.CudaRuntime(0)
    rt_mod.set_runtime(rt)
    K, frames, analytic = bench.make_inputs(0)
    d_frames = [rt.from_host(f) for f in frames]
    d_fwd = [rt.from_host(a["fwd"][None]) for a in analytic]
    d_bwd = [rt.from_host(a["bwd"][None]) for a in analytic]
    d_diff = [rt.from_host(a["diff"][None, :, :, 0]) for a in analytic]
    d_depth = [rt.from_host(a["depth"]) for a in analytic]
    enc, dec = synth.monodepth2_weights(4869, bench.FEED_H, bench.FEED_W)
    flow_w = synth.liteflownet_weights()

    def inject(pipe, st):                                   # bench.py's hook: analytic flow / depth over the network outputs
        slot = st.id % N
        if st.fwd is not None:
            st.fwd.t.copy_(d_fwd[slot].t); st.bwd.t.copy_(d_bwd[slot].t); st.diff.t.copy_(d_diff[slot].t)
        with pipe.depth_stream(st.id):
            tmp = pipe._buf("dsrc%d" % pipe.slot(st.id), (H, W), np.float32)
            tmp.t.copy_(d_depth[slot].t)
            pipe.eng.depth_post(tmp, pipe.cfg.crop.depth_crop, 0.0, 50.0, st.raw_depth, st.depth)

    for name, over in CONFIGS.items():
        cfg = configure(config.default_cfg(H, W), over)
        np.random.seed(4869)
        p = pipeline.FramePipeline(K, H, W, cfg=cfg, precision=native.PREC_BF16, runtime=rt, overlap=True, inflight=3, inject=inject,
                                   pipelined=True)
        p.load_weights(flow_w, enc, dec)
        for _ in range(args.warmup):
            p.step(d_frames[p.stage % N])
        torch.cuda.synchronize()
        first = p.stage
        t0 = time.perf_counter()
        for _ in range(args.steps):
            p.step(d_frames[p.stage % N])
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        p.flush()
        torch.cuda.synchronize()
        by_branch = {}
        for fid, ms in p.track_ms.items():
            if fid >= first:
                by_branch.setdefault(p.modes.get(fid), []).append(ms)
        print(json.dumps({"config": name, "frames_per_s": round(args.steps / dt, 2), "steps": args.steps,
                          "tracker_ms_per_frame": {str(k): round(float(np.mean(v)), 3) for k, v in by_branch.items()},
                          "frames_by_branch": {str(k): len(v) for k, v in by_branch.items()}, "device": torch.cuda.get_device_name(0)}))
        p.close()


if __name__ == "__main__":
    main()
