"""Several sequences on one GPU: aggregate frames/s of multiseq.SequenceBatch (one batched forward of each network per step, then
the S trackers) against S independent FramePipelines stepped round-robin in one process on their own streams, for S in
{1, 2, 4, 8} at 376x1241 in bf16.  Both run in overlap mode (networks of step t beside the trackers of step t-1, the
FramePipeline's overlap=True, inflight=1).  Inputs are bench.py's: seeded random weights, its synthetic frame cycle, and analytic
flows / depths copied over the network outputs on the device through the inject hooks; sequence s starts s frames into the cycle.

Also reported per S: the host ms per step spent in the S trackers of the batch, and the device ms per step of the batch's
networks alone (the same step without trackers), so a host-bound S shows; and the card's name and power limit, read in the same
run.  Prints one JSON line (and writes it to --out if given).  Usage (on a GPU):
  python scripts/multi_seq.py --steps 60 --warmup 10 --out /tmp/multi_seq.json"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "df-vo_b200"))

import bench                                                   # noqa: E402  (frame cycle, sizes)
import synthdata as synth                                      # noqa: E402


def card():
    import torch
    out = dict(name=torch.cuda.get_device_name(0), power_limit_w=None)
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True,
                           text=True, timeout=30)
        out["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except Exception as e:                                     # reported, not guessed
        out["power_limit_w"] = "unavailable: %s" % e
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--sizes", default="1,2,4,8")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from b200 import multiseq, native, pipeline, runtime as rt_mod
    assert torch.cuda.is_available(), "multi_seq.py measures on a CUDA device"
    rt = rt_mod.CudaRuntime(0)
    rt_mod.set_runtime(rt)
    H, W, ND = bench.H, bench.W, bench.N_DISTINCT
    enc, dec = synth.monodepth2_weights(4869, bench.FEED_H, bench.FEED_W)
    flow_w = synth.liteflownet_weights()
    K, frames, analytic = bench.make_inputs(0)
    d_frames = [rt.from_host(f) for f in frames]
    d_fwd = [rt.from_host(a["fwd"][None]) for a in analytic]
    d_bwd = [rt.from_host(a["bwd"][None]) for a in analytic]
    d_diff = [rt.from_host(a["diff"][None, :, :, 0]) for a in analytic]
    d_depth = [rt.from_host(a["depth"]) for a in analytic]
    cyc = lambda s, fid: (fid + s) % ND                        # frame of the cycle sequence s shows at its frame fid

    def put(st, k, eng, cfg, tmp):
        if st.fwd is not None:
            st.fwd.t.copy_(d_fwd[k].t); st.bwd.t.copy_(d_bwd[k].t); st.diff.t.copy_(d_diff[k].t)
        tmp.t.copy_(d_depth[k].t)
        eng.depth_post(tmp, cfg.crop.depth_crop, 0.0, 50.0, st.raw_depth, st.depth)

    def make_batch(S):
        tmp = [rt.empty((H, W), np.float32) for _ in range(S)]

        def inject(b, s, st):
            put(st, cyc(s, st.id), b.eng, b.cfg, tmp[s])
        b = multiseq.SequenceBatch([K] * S, H, W, precision=native.PREC_BF16, overlap=True, inject=inject, runtime=rt,
                                   rngs=[np.random.RandomState(4869 + s) for s in range(S)])
        b.load_weights(flow_w, enc, dec)
        return b

    def make_pipes(S):
        pipes = []
        for s in range(S):
            tmp = rt.empty((H, W), np.float32)

            def inject(p, st, s=s, tmp=tmp):
                with p.depth_stream(st.id):                    # ordered after the depth network's own post-processing (bench.py)
                    put(st, cyc(s, st.id), p.eng, p.cfg, tmp)
            p = pipeline.FramePipeline(K, H, W, precision=native.PREC_BF16, runtime=rt, overlap=True, inflight=1, inject=inject,
                                       rng=np.random.RandomState(4869 + s))
            p.load_weights(flow_w, enc, dec)
            pipes.append(p)
        return pipes

    def timed(step_fn, streams, n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for t in range(n):
            step_fn(t)
        cs = torch.cuda.current_stream()
        for sx in streams:
            cs.wait_stream(sx)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    rows = []
    for S in [int(v) for v in args.sizes.split(",")]:
        b = make_batch(S)
        frame = lambda s, t: d_frames[cyc(s, t)]
        step_b = lambda t: b.step([frame(s, b._nframes[s]) for s in range(S)])
        for t in range(args.warmup):
            step_b(t)
        b.track_ms.clear()
        ms_b = timed(step_b, [b.s_net, b.s_trk], args.steps)
        trk_ms = float(np.mean(b.track_ms))
        # the batch's networks alone: the same step without the trackers
        with rt.on_stream(b.s_net):
            def nets(t):
                b._infer([frame(s, b._nframes[s]) for s in range(S)])
                b.stage += 1
            ms_n = timed(nets, [b.s_net], args.steps)
        del b
        pipes = make_pipes(S)

        def step_rr(t):
            for s, p in enumerate(pipes):
                p.step(frame(s, p.stage))
        for t in range(args.warmup):
            step_rr(t)
        ms_rr = timed(step_rr, [x for p in pipes for x in p.s_nets + p.s_depths + [p.s_trk]], args.steps)
        del pipes
        torch.cuda.empty_cache()
        row = dict(S=S, batch_fps=S * args.steps / (ms_b / 1e3), round_robin_fps=S * args.steps / (ms_rr / 1e3),
                   batch_step_ms=ms_b / args.steps, round_robin_step_ms=ms_rr / args.steps,
                   batch_tracker_host_ms_per_step=trk_ms, batch_network_device_ms_per_step=ms_n / args.steps)
        row["batch_over_round_robin"] = row["batch_fps"] / row["round_robin_fps"]
        rows.append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)
    res = dict(metric="aggregate VO frames/s, S sequences at %dx%d, bf16, overlap mode" % (H, W), steps=args.steps, warmup=args.warmup,
               card=card(), results=rows)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
