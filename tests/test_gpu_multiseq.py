"""GPU: several sequences on one H100.

* The batched monodepth2 and PoseNet runners at the KITTI feed size 192x640, B in {1, 2, 4}, in fp32, tf32 and bf16: every entry
  has the bits of a batch-1 runner on the same feed(s).
* multiseq.SequenceBatch with S = 4 sequences at 376x1241, the real networks (seeded synthetic weights) and the PoseNet depth
  consistency on: each sequence's network outputs (flows, depths, PoseNet depth-consistency maps) and poses equal those of an
  independent FramePipeline on the same frames, bit for bit, in order and in overlap mode.
"""
import numpy as np
import pytest

import synthdata as synth

pytestmark = pytest.mark.gpu

FH, FW = 192, 640


@pytest.mark.parametrize("prec", [0, 1, 2])
def test_batched_depth_and_pose_bit_equal_to_batch_one(dev_lib, prec):
    import torch
    from b200 import native
    enc, dec = synth.monodepth2_weights(4869, FH, FW)
    penc, pdec = synth.posenet_weights()
    penc = {k: v for k, v in penc.items() if k.startswith("encoder.")}
    g = torch.Generator().manual_seed(7)
    feeds = [torch.rand((1, 3, FH, FW), generator=g).cuda() for _ in range(5)]
    stream = torch.cuda.current_stream().cuda_stream

    def ctx_for():
        c = native.Context(dev_lib)
        c.load_weights(native.NET_MONODEPTH2, enc); c.load_weights(native.NET_MONODEPTH2, dec)
        c.load_weights(native.NET_POSENET, penc); c.load_weights(native.NET_POSENET, pdec)
        return c

    one = ctx_for()
    one.monodepth2_build(FH, FW, prec)
    one.posenet_build(FH, FW, prec, 5.4)
    d1, p1 = [], []
    for i in range(4):
        d = torch.empty((FH, FW), device="cuda")
        p = torch.empty((4, 4), device="cuda")
        for _ in range(3):                                     # eager, captured and replayed graph: all the same bits
            one.monodepth2_forward(feeds[i].data_ptr(), d.data_ptr(), stream)
            one.posenet_forward(feeds[i + 1].data_ptr(), feeds[i].data_ptr(), p.data_ptr(), stream)
        d1.append(d.cpu().numpy()); p1.append(p.cpu().numpy())
    for B in (1, 2, 4):
        c = ctx_for()
        c.monodepth2_build_batch(FH, FW, B, prec)
        c.posenet_build_batch(FH, FW, B, prec, 5.4)
        order = [3, 1, 0, 2][:B]
        d = torch.empty((B, FH, FW), device="cuda")
        p = torch.empty((B, 4, 4), device="cuda")
        for _ in range(3):
            c.monodepth2_forward_batch([feeds[i].data_ptr() for i in order], d.data_ptr(), stream)
            c.posenet_forward_batch([a for i in order for a in (feeds[i + 1].data_ptr(), feeds[i].data_ptr())], p.data_ptr(), stream)
        d, p = d.cpu().numpy(), p.cpu().numpy()
        for b, i in enumerate(order):
            assert np.array_equal(d[b], d1[i]), (prec, B, b)
            assert np.array_equal(p[b], p1[i]), (prec, B, b)
        c.close()
    assert all(np.isfinite(x).all() for x in d1 + p1)


def test_sequence_batch_matches_independent_pipelines(dev_lib):
    import torch
    from b200 import config, multiseq, pipeline, runtime as rt_mod
    from oracle import seqdata
    rt = rt_mod.CudaRuntime(0)
    rt_mod.set_runtime(rt)
    H, W, S, n = 376, 1241, 4, 5
    K0 = synth.kitti_intrinsics(H, W)
    Ks = [[K0[0] + s, K0[1] - s, K0[2] * (1 + 0.01 * s), K0[3] * (1 + 0.01 * s)] for s in range(S)]
    lfn = synth.liteflownet_weights()
    enc, dec = synth.monodepth2_weights(4869, FH, FW)
    penc, pdec = synth.posenet_weights()
    frames = [[synth.value_noise_image(H, W, 1000 * s + i) for i in range(n)] for s in range(S)]
    order = [[(i + 2 * s) % 7 for i in range(n)] for s in range(S)]
    analytic = {}

    def flows(s, fid):
        k = (s, fid)
        if k not in analytic:
            j = order[s][fid]
            f = seqdata.frame_inputs(j, H, W, Ks[s], seqdata.MODES[j % len(seqdata.MODES)])
            analytic[k] = [rt.from_host(f["fwd"][None]), rt.from_host(f["bwd"][None]), rt.from_host(f["diff"][None, :, :, 0])]
        return analytic[k]

    def cfg():
        c = config.default_cfg(H, W)
        c.deep_pose.enable = True
        c.kp_selection.depth_consistency.enable = True
        return c

    def capture(rec, s, st):
        """Record the frame's flows, then put analytic flows over them (so the selection finds keypoints)."""
        if st.fwd is not None:
            rec[(s, st.id, "fwd")], rec[(s, st.id, "diff")] = st.fwd.clone(), st.diff.clone()
            for dst, src in zip((st.fwd, st.bwd, st.diff), flows(s, st.id)):
                dst.t.copy_(src.t)

    def capture_depth(rec, s, st):
        rec[(s, st.id, "depth")] = st.depth.clone()
        if st.deep_pose is not None:
            rec[(s, st.id, "pose")] = st.deep_pose.clone()

    def host(rec):
        torch.cuda.synchronize()
        return {k: v.numpy() for k, v in rec.items()}

    def run_batch(overlap):
        rec = {}

        def inject(b, s, st):
            capture_depth(rec, s, st)
            capture(rec, s, st)
        b = multiseq.SequenceBatch(Ks, H, W, cfg=cfg(), overlap=overlap, inject=inject, runtime=rt)
        b.load_weights(lfn, enc, dec, penc, pdec)
        steps = [b.step([frames[s][i] for s in range(S)]) for i in range(n)]
        if overlap:
            steps.append(b.flush())
        rec = host(rec)
        dd = [b.seqs[s]._bufs["ddiff"].numpy() for s in range(S)]
        return steps, [dict(p) for p in b.poses], [dict(m) for m in b.modes], rec, dd

    def run_single(s, overlap):
        rec = {}

        def inject(p, st):
            with p.depth_stream(st.id):                         # after the frame's depth network, post-processing and PoseNet
                capture_depth(rec, s, st)
            capture(rec, s, st)
        p = pipeline.FramePipeline(Ks[s], H, W, cfg=cfg(), runtime=rt, rng=np.random.RandomState(4869), overlap=overlap, inject=inject)
        p.load_weights(lfn, enc, dec, penc, pdec)
        for i in range(n):
            p.step(frames[s][i])
        if overlap:
            p.flush()
        rec = host(rec)
        return dict(p.poses), dict(p.modes), rec, p._bufs["ddiff"].numpy()

    for overlap in (False, True):
        steps, poses, modes, rec, dd = run_batch(overlap)
        if overlap:
            assert steps[0] == [None] * S
            steps = steps[1:]
        for s in range(S):
            ps, ms, rs, ds = run_single(s, overlap)
            assert sorted(ps) == list(range(n)) and ms == modes[s], (overlap, s)
            for i in range(n):
                assert np.array_equal(poses[s][i], ps[i]) and np.array_equal(steps[i][s], ps[i]), (overlap, s, i)
            keys = [k for k in rs if k[0] == s]
            assert len(keys) == 4 * (n - 1) + 1
            for k in keys:
                assert np.array_equal(rec[k], rs[k]), (overlap, k)
            assert np.array_equal(dd[s], ds, equal_nan=True), (overlap, s)      # the last frame's depth-consistency map
