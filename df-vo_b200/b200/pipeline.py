"""Device-resident DF-VO frame pipeline: uint8 frame in, 4x4 pose out.

The same per-frame algorithm as the reference driver's ``deep_model_inference`` + ``tracking``
(dfvo.py:121-262,299-345, hybrid tracking, default configuration; also ``tracking_method: PnP`` and the E-tracker's
``validity.method: flow``) but organised for the GPU:
everything from the uploaded frame to the keypoints / RANSAC scores / triangulated depths stays in HBM;
the host only draws the RNG-dependent permutations, takes the small decisions the reference takes on the
host (GRIC vote, cheirality threshold, sentinels) and chains the pose.  Per frame the host receives a few
kilobytes (keypoints, masks, scores) instead of the reference's ~9.8 MB of dense maps
(deep_models.py:178-181,205).

This is the object ``bench.py`` times; ``df-vo_b200/libs`` exposes the same kernels behind the reference's
class API for the unmodified driver.
"""
import os
import time

import numpy as np

from . import config as cfg_mod
from . import hostmath, native, tracking
from . import runtime as rt_mod


class FrameState:
    """Device buffers of one frame: image, depths and (for every frame but the first) the flows of the pair
    (previous frame -> this frame).  `ready` = event recorded after the frame's networks (two-stream mode)."""
    __slots__ = ("id", "img", "depth", "raw_depth", "fwd", "bwd", "diff", "ready", "img_ready", "feed", "feed_ready", "deep_pose")

    def __init__(self):
        self.fwd = self.bwd = self.diff = self.ready = self.img_ready = None
        self.feed = self.feed_ready = self.deep_pose = None


class _ForkJoin:
    """`with` block whose launches go to `side`, ordered after everything already on the current stream; the join event
    is left in ``owner._depth_done`` for the step to wait on."""

    def __init__(self, rt, side, owner):
        self.rt, self.side, self.owner = rt, side, owner

    def __enter__(self):
        fork = self.rt.record_event()
        self.ctx = self.rt.on_stream(self.side)
        self.ctx.__enter__()
        self.rt.wait_event(fork)

    def __exit__(self, *a):
        self.owner._depth_done = self.rt.record_event()
        return self.ctx.__exit__(*a)


class FramePipeline:
    def __init__(self, K, height=376, width=1241, cfg=None, precision=native.PREC_BF16, runtime=None, rng=np.random,
                 overlap=False, engine=None, inflight=1, inject=None, tracker_thread=False, pipelined=False):
        """K = [cx, cy, fx, fy].

        inject: optional ``callable(pipeline, frame_state)`` run by ``infer`` right after the two networks of a frame were
        enqueued (on the frame's network stream).  Without trained weights a benchmark / test uses it to copy analytic
        flow / depth over the network outputs on the device; it is the one official hook for that -- nothing else of the
        pipeline needs replacing.

        overlap=False: ``step(img)`` returns the pose of ``img`` (one stream, in order).
        overlap=True : two CUDA streams; ``step(img)`` enqueues the networks of ``img`` and then tracks the
        PREVIOUS frame while the GPU runs them, returning the previous frame's pose (``None`` on the first
        call); ``flush()`` tracks the last frame.  Same arithmetic, same RNG order, same poses -- frames only
        depend on each other through the reference image / depth, which are triple-buffered here.
        inflight=2 (overlap mode only): a second, independent network engine, so the networks of two consecutive frames run
        concurrently (their small-grid phases fill each other's idle SMs) and tracking lags by two frames: ``step``
        returns the pose of frame t-2, ``flush()`` the remaining ones (a list).  Same poses again.
        pipelined=True (overlap mode only): the tracker of a frame is split into its enqueue half and its read half
        (track_launch / track_finish): ``step(t)`` enqueues the networks of frame t, then reads the result of the tracker enqueued by
        the previous step, then enqueues the tracker of frame t-inflight and returns WITHOUT waiting for it -- the tracker's kernels
        (~1 ms of dependent small launches) run while the caller fetches the next frame and the next step enqueues its networks.  ``step`` then returns the pose of
        frame t-inflight-1 (``self.lag`` steps behind) and ``flush()`` the remaining ones.  Same arithmetic, generator order and poses.
        tracker_thread=True (overlap mode only): the tracker runs on its own host thread (one frame at a time, in frame order, so
        the RNG stream and the poses are unchanged).  ``step(img)`` enqueues the networks of ``img``, hands the frame to the tracker
        thread and then waits for the pose of frame t-inflight, which that thread has been working on meanwhile: the host work
        of enqueueing a frame and the tracker's device waits overlap instead of adding up."""
        self.cfg = cfg or cfg_mod.default_cfg(height, width)
        self.tracking_method = self.cfg.get("tracking_method", "hybrid")
        self.validity = self.cfg.e_tracker.validity.method
        if self.tracking_method not in ("hybrid", "PnP"):
            raise ValueError("FramePipeline implements tracking_method 'hybrid' and 'PnP', not %r" % (self.tracking_method,))
        if self.validity not in ("GRIC", "flow"):
            raise ValueError("FramePipeline implements e_tracker.validity.method 'GRIC' and 'flow', not %r" % (self.validity,))
        # kp_selection.depth_consistency (dfvo.py:84,142-143,338-345): the PoseNet of (ref, cur) masks the selection
        self.depth_consistency = bool(self.cfg.kp_selection.depth_consistency.enable)
        if self.depth_consistency and not self.cfg.deep_pose.enable:
            raise ValueError("kp_selection.depth_consistency needs deep_pose.enable (the PoseNet gives its pose, dfvo.py:338-345)")
        self.kp_src = self._keypoint_routing(self.cfg, self.tracking_method)
        self.K = [float(v) for v in K]
        self.H, self.W = height, width
        self.rt = runtime or rt_mod.get()
        self.eng = engine or tracking.Engine(height, width, self.rt)      # `engine`: share built networks with another pipeline
        self.precision = precision
        self.rng = rng
        self.inject = inject
        self.ref = None
        self.stage = 0
        self.global_pose = np.eye(4)
        self.motion = np.eye(4)
        self.poses = {}
        self.track_ms = {}
        self.modes = {}              # frame id -> branch taken by the tracker ('E', 'PnP', 'const'; None for the first frame)
        self.last = {}
        self._bufs = {}
        self.overlap = bool(overlap)
        self.inflight = int(inflight) if self.overlap else 1
        assert self.inflight in (1, 2, 3)
        # buffer slots: a frame's buffers serve its own tracker and, as reference, the next frame's; the pipelined mode finishes a
        # tracker AFTER the next frame's networks were enqueued, which needs one slot more
        self.nslots = (self.inflight + 2 + (1 if (pipelined and not tracker_thread) else 0)) if self.overlap else 2
        self.fused_tail = os.environ.get("DFVO_FUSED_TAIL", "1") != "0"     # device-side tail of the E branch (track_fused)
        self.pipelined = bool(pipelined) and self.overlap and not tracker_thread
        self._tok = None             # pipelined mode: (frame state, token of track_launch, host ms so far) of the tracker in flight
        self.lag = (self.inflight + (1 if self.pipelined else 0)) if self.overlap else 0     # step(t) returns the pose of frame t - lag
        self.tracker_thread = bool(tracker_thread) and self.overlap
        self._thr = None
        self.pending = []            # overlap mode: frames whose networks are enqueued but which are not tracked yet
        self.trk_ref = None          # overlap mode: the tracker's reference frame (self.ref is the networks')
        self.engs = [self.eng] + [tracking.Engine(height, width, self.rt) for _ in range(self.inflight - 1)]
        if self.overlap:
            self.s_nets = [self.rt.new_stream() for _ in self.engs]      # LiteFlowNet (per engine)
            self.s_depths = [self.rt.new_stream() for _ in self.engs]    # monodepth2: independent of the flow network, its small
            self.s_net, self.s_depth = self.s_nets[0], self.s_depths[0]  # launches fill the SMs LiteFlowNet's coarse levels leave idle
            self.s_trk = self.rt.new_stream(high_priority=True)

    @staticmethod
    def _keypoint_routing(c, tracking_method):
        """Which keypoint set each consumer reads (dfvo.py:165-250): {'e', 'scale', 'pnp'} -> 'kp_best' / 'kp_list'.  kp_best comes
        from local best-N (or global best-N when only bestN.enable), kp_list from sampled_kp (keypoint_sampler.py:76-163).  A source
        no enabled selector produces is refused here; the reference would raise KeyError on the second frame."""
        sel = c.kp_selection
        if sel.local_bestN.enable and sel.local_bestN.score_method not in ("flow", "flow_ratio"):
            raise ValueError("FramePipeline implements local_bestN score_method 'flow' and 'flow_ratio', not %r"
                             % (sel.local_bestN.score_method,))
        produced = set()
        if sel.local_bestN.enable or sel.bestN.get("enable", False):
            produced.add("kp_best")
        if sel.get("sampled_kp", {}).get("enable", False):
            produced.add("kp_list")
        src = dict(pnp=c.pnp_tracker.get("kp_src", "kp_best"))
        if tracking_method == "hybrid":
            src["e"] = c.e_tracker.get("kp_src", "kp_best")
            s_src = c.scale_recovery.get("kp_src", "kp_best")
            if c.scale_recovery.method == "iterative":
                # iterative scale recovery takes kp_depth from its own rigid-flow selection, or else the E-tracker's set
                if s_src not in ("kp_depth", src["e"]):
                    raise ValueError("iterative scale recovery on kp_src %r needs the E-tracker's set (%r) or kp_depth" % (s_src, src["e"]))
                s_src = src["e"]
            src["scale"] = s_src
        for who, name in sorted(src.items()):
            if name not in produced:
                raise ValueError("%s kp_src %r: no enabled keypoint selector produces it (enabled: %s)"
                                 % ({"e": "e_tracker", "scale": "scale_recovery", "pnp": "pnp_tracker"}[who], name,
                                    ", ".join(sorted(produced)) or "none"))
        return src

    # ------------------------------------------------------------------ setup
    def load_weights(self, flow_weights, depth_enc, depth_dec, pose_enc=None, pose_dec=None):
        """pose_enc / pose_dec: pose_encoder.pth / pose.pth, needed (and only used) with kp_selection.depth_consistency."""
        if self.depth_consistency and (pose_enc is None or pose_dec is None):
            raise ValueError("kp_selection.depth_consistency needs the PoseNet weights (pose_enc, pose_dec)")
        for e in self.engs:
            e.build_flow(flow_weights, pairs=1, precision=self.precision)
            e.build_depth(depth_enc, depth_dec, precision=self.precision, dataset=self.cfg.dataset)
            if self.depth_consistency:
                e.build_pose(pose_enc, pose_dec, precision=self.precision, dataset=self.cfg.dataset)

    def engine_for(self, fid):
        """The network engine of frame `fid` (tracking always uses engine 0's solvers)."""
        return self.engs[fid % len(self.engs)]

    def slot(self, fid):
        """Buffer slot of frame `fid` (images / depths / flows are multi-buffered so a reference frame stays valid)."""
        return fid % self.nslots

    def _buf(self, name, shape, dtype, cap0=None):
        """Named device buffer, grow-only: allocated for a capacity (`cap0` rows if given) and handed out as an exactly-shaped
        view, so per-frame keypoint counts never reallocate."""
        shape = tuple(int(d) for d in shape)
        n = int(np.prod(shape)) if shape else 1
        b = self._bufs.get(name)
        if b is None or b.size < n or b.dtype != np.dtype(dtype):
            cap = n
            if cap0 is not None and shape:
                rows = int(cap0)
                while rows < shape[0]:
                    rows *= 2
                cap = rows * (n // max(shape[0], 1))
            b = self._bufs[name] = self.rt.empty((max(cap, 1),), dtype)
        return b.view(shape)

    # ------------------------------------------------------------------ per-frame stages
    def depth_feed_host(self, img):
        """deep_models.py:195-198 as the reference does it on the host (PIL LANCZOS + ToTensor).  The pipeline
        uses the bit-identical device version (Engine.depth_feed); this one serves tests / comparisons."""
        import PIL.Image as pil
        im = pil.fromarray(img).resize((self.eng.feed_w, self.eng.feed_h), pil.LANCZOS)
        return np.ascontiguousarray(np.transpose(np.asarray(im, np.uint8), (2, 0, 1))[None].astype(np.float32) / np.float32(255))

    def infer(self, img, fid):
        """Upload + both networks for one new frame; returns its FrameState (device buffers).  `img`: uint8 HWC frame as a
        host ndarray, a pinned host tensor (asynchronous H2D) or an already device-resident ``runtime.Buf``."""
        st = FrameState()
        st.id = fid
        # multi-buffer images / depths / flows so the previous frame's stay valid as 'ref'
        slot = self.slot(fid)
        eng = self.engine_for(fid)
        if isinstance(img, rt_mod.Buf):
            st.img = img
        else:
            st.img = self._buf("img%d" % slot, (self.H, self.W, 3), np.uint8).upload(img)
        self.mark_image_ready(st)
        st.raw_depth = self._buf("raw%d" % slot, (self.H, self.W), np.float32)
        st.depth = self._buf("dep%d" % slot, (self.H, self.W), np.float32)
        with self.depth_stream(fid):
            if self.depth_consistency:
                # the frame keeps its feed: the next frame's PoseNet reads it as the reference image (deep_models.py:218-226)
                st.feed = eng.depth_feed(st.img, out=self._buf("feed%d" % slot, (1, 3, eng.feed_h, eng.feed_w), np.float32))
                if self.overlap:
                    st.feed_ready = self.rt.record_event()
                d = eng.depth(st.feed)
                if self.ref is not None:
                    self.pose_cnn(eng, st, slot)
            else:
                d = eng.depth(eng.depth_feed(st.img))                    # LANCZOS resize + ToTensor on the device
            c = self.cfg
            eng.depth_post(d, c.crop.depth_crop, float(c.depth.min_depth), float(c.depth.max_depth), st.raw_depth, st.depth)
        if self.ref is not None:
            self.wait_reference_image()
            st.fwd, st.bwd, st.diff = self.flow_slot(slot)
            eng.flow([self.ref.img, st.img], out=(st.fwd, st.bwd, st.diff))
        if self.inject is not None:
            self.inject(self, st)
        return st

    def pose_cnn(self, eng, st, slot):
        """ref_data['deep_pose'] = forward_pose([ref, cur]) (dfvo.py:338-345) on the frame's depth stream, after the reference
        frame's feed (another engine's stream with inflight > 1) is ready.  The pose stays on the device."""
        if self.overlap and self.ref.feed_ready is not None:
            self.rt.wait_event(self.ref.feed_ready)
        st.deep_pose = eng.pose(self.ref.feed, st.feed, out=self._buf("dpose%d" % slot, (4, 4), np.float32))

    def mark_image_ready(self, st):
        """Called by infer() right after the frame's image is on the device (its upload was enqueued on this frame's
        network stream); with two engines the next frame's flow network, on the other stream, waits for it."""
        if self.overlap and self.inflight > 1:
            st.img_ready = self.rt.record_event()

    def wait_reference_image(self):
        if self.overlap and self.inflight > 1 and self.ref is not None and self.ref.img_ready is not None:
            self.rt.wait_event(self.ref.img_ready)

    def depth_stream(self, fid=None):
        """Context for the depth network of the frame being inferred: in overlap mode a side stream forked from the
        network stream (after the image upload) and joined back into it by ``step`` -- monodepth2 and LiteFlowNet share
        only the input image; in-order mode: the current stream."""
        import contextlib
        if not self.overlap:
            return contextlib.nullcontext()
        fid = self.stage - 1 if fid is None else fid                   # the frame being inferred
        return _ForkJoin(self.rt, self.s_depths[fid % len(self.engs)], self)

    def flow_slot(self, slot):
        """The (fwd, bwd, diff) output buffers of buffer slot `slot`."""
        e = self.eng
        return (self._buf("ffwd%d" % slot, e.flow_fwd.shape, np.float32), self._buf("fbwd%d" % slot, e.flow_bwd.shape, np.float32),
                self._buf("fdif%d" % slot, e.flow_diff.shape, np.float32))

    def track(self, cur, ref=None):
        """dfvo.py:121-262 (tracking_method hybrid or PnP).  Returns the relative pose cur -> ref as a 4x4."""
        return self.track_finish(self.track_launch(cur, ref))

    def track_launch(self, cur, ref=None):
        """First half of `track`: everything up to the last enqueue.  Returns a token for `track_finish`.  On the fused E branch the
        tracker's kernels are still running when this returns (the caller may do other host work -- e.g. enqueue the next frame's
        networks -- before it finishes the frame); every other branch is finished here and the token just carries the pose."""
        c, eng, K = self.cfg, self.eng, self.K
        ref = ref or self.ref
        fwd = cur.fwd if cur.fwd is not None else eng.flow_fwd          # (subclasses may leave the flows in the engine's buffers)
        diff = cur.diff if cur.diff is not None else eng.flow_diff
        # flow validity on the fused path: the gate's mean flow magnitude of the E-tracker's set (riding on the selection's status read
        # for local best-N)
        want_mean = self.tracking_method == "hybrid" and self.validity == "flow" and self.fused_tail
        sets, good, flow_mean = self.select(cur, ref, fwd, diff, want_mean)
        self.last = dict(good=good, n=sets[self.kp_src["e" if self.tracking_method == "hybrid" else "pnp"]][2] if good else 0, mode="const")
        if not good:
            return dict(pose=self.motion.copy())                          # constant motion (dfvo.py:157-161)
        pnp_kp = sets[self.kp_src["pnp"]]
        if self.tracking_method == "PnP":                                 # E_pose stays identity: PnP on every frame (dfvo.py:224-250)
            kp1_buf, kp2_buf, n = pnp_kp
            self.last["mode"] = "PnP"
            if self.fused_tail and n <= eng.TAIL_MAX_N:
                return dict(pnp=self.pnp_fused_launch(kp1_buf, kp2_buf, n, ref))
            return dict(pose=self.pnp(kp1_buf.numpy()[:n], kp2_buf.numpy()[:n], kp1_buf, n, ref))
        kp1_buf, kp2_buf, n = sets[self.kp_src["e"]]
        iterative = c.scale_recovery.method == "iterative"
        same_scale = self.kp_src["scale"] == self.kp_src["e"]
        if not iterative and same_scale and 10 < n <= eng.TAIL_MAX_N and self.fused_tail:
            return self.track_fused_launch(cur, ref, kp1_buf, kp2_buf, n, flow_mean, pnp_kp)
        return dict(pose=self.track_stepwise(cur, ref, kp1_buf, kp2_buf, n, None if same_scale else sets[self.kp_src["scale"]], pnp_kp))

    def select(self, cur, ref, fwd, diff, want_mean=False):
        """KeypointSampler.kp_selection (keypoint_sampler.py:76-143, dfvo.py:140-150) on the device: the keypoint sets the
        configuration enables -> ({'kp_best' / 'kp_list': (kp1, kp2, n)}, good_kp_found, flow mean).  good_kp_found comes from local
        best-N only (best-N and sampled_kp never fail); when it is False no other set is gathered.  want_mean: also the mean flow
        magnitude of the E-tracker's set (None otherwise)."""
        c, eng, K = self.cfg, self.eng, self.K
        sel = c.kp_selection
        b = sel.local_bestN
        e_src = self.kp_src.get("e")
        sets, good, flow_mean = {}, True, None
        if b.enable:
            dd, dthre = None, 0.05
            if self.depth_consistency:                                    # DepthConsistency.compute (dfvo.py:142-143)
                cx, cy, fx, fy = K
                Km = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]])
                dd = eng.depth_consistency(cur.raw_depth, ref.raw_depth, cur.deep_pose, Km, np.linalg.inv(Km),
                                           out=self._buf("ddiff", (self.H, self.W), np.float32))
                dthre = float(c.kp_selection.depth_consistency.thre)
            mean_here = want_mean and e_src == "kp_best"
            r = eng.select_local_bestn(diff, fwd, b.num_row, b.num_col, b.num_bestN, b.thre, depth_diff_buf=dd, depth_thre=dthre,
                                       with_flow_mean=mean_here, score_method=b.score_method)
            good = r[0]
            sets["kp_best"] = (r[2], r[3], r[1])
            if mean_here:
                flow_mean = r[4]
        elif sel.bestN.get("enable", False):
            _, n, kp1_buf, kp2_buf = eng.select_bestn(diff, fwd, sel.bestN.num_bestN)
            sets["kp_best"] = (kp1_buf, kp2_buf, n)
            if want_mean and e_src == "kp_best":
                flow_mean = eng.flow_mean(kp1_buf, kp2_buf, n)
        sk = sel.get("sampled_kp", {})
        if good and sk.get("enable", False):
            sets["kp_list"] = eng.sampled_keypoints(fwd, c.crop.flow_crop, sk.num_kp)
            if want_mean and e_src == "kp_list":
                flow_mean = eng.flow_mean(sets["kp_list"][0], sets["kp_list"][1], sets["kp_list"][2])
        return sets, good, flow_mean

    def track_finish(self, tok):
        """Second half of `track`: the relative pose cur -> ref (4x4)."""
        if "pose" in tok:
            return tok["pose"]
        if "pnp" in tok:
            return self.pnp_fused_finish(tok["pnp"])
        return self.track_fused_finish(tok)

    def track_stepwise(self, cur, ref, kp1_buf, kp2_buf, n, scale_kp=None, pnp_kp=None):
        """The E branch with the host in the loop after every stage (iterative scale recovery, tiny / huge keypoint sets,
        DFVO_FUSED_TAIL=0, or a scale recovery on another keypoint set than the E-tracker's).  scale_kp / pnp_kp: (kp1, kp2, n) of
        the scale recovery's / PnP tracker's set when it is not the E-tracker's (scale_recovery.kp_src, pnp_tracker.kp_src)."""
        c, eng, K = self.cfg, self.eng, self.K
        iterative = c.scale_recovery.method == "iterative"
        kp_ref = kp1_buf.numpy()[:n]
        kp_cur = kp2_buf.numpy()[:n]
        if scale_kp is not None:
            s1, s2, sn = scale_kp
            s_ref, s_cur, s_buf = s1.numpy()[:sn], s2.numpy()[:sn], s2
        else:
            s_ref, s_cur, s_buf, sn = kp_ref, kp_cur, kp2_buf, n
        # ---- E-tracker (dfvo.py:165-193).  The homography vote runs on a host worker thread; the pose-dependent device
        # work of the scale recovery (triangulation, depth gather) is issued before the vote is joined.
        r = tracking.compute_pose_2d2d(eng, kp_ref, kp_cur, K, repeat=c.e_tracker.ransac.repeat,
                                       reproj_thre=c.e_tracker.ransac.reproj_thre, rng=self.rng,
                                       kp_ref_buf=kp1_buf, kp_cur_buf=kp2_buf, defer_validity=True, validity=self.validity,
                                       flow_thre=c.e_tracker.validity.get("thre"))
        prep = None
        if np.linalg.norm(r["t"]) != 0 and not iterative:
            E_spec = np.eye(4)
            E_spec[:3, :3], E_spec[:3, 3:] = r["R"], r["t"]
            prep = self.scale_prepare(s_ref, s_cur, s_buf, np.linalg.inv(E_spec), cur.depth, sn)
        tracking.resolve_validity(r)
        E_pose = np.eye(4)
        E_pose[:3, :3], E_pose[:3, 3:] = r["R"], r["t"]
        hybrid = np.eye(4)
        hybrid[:3, :3] = r["R"]
        scale = None
        self.last.update(valid=r["valid"], inliers=r["inliers"], mode="E")
        if np.linalg.norm(E_pose[:3, 3]) != 0:
            scale = self.scale_iterative(cur, ref, kp_ref, kp_cur, E_pose) if iterative else self.scale_finish(prep)
            if scale != -1:
                hybrid[:3, 3] = E_pose[:3, 3] * scale
        self.last["scale"] = scale
        # ---- PnP fallback (dfvo.py:225-250)
        if np.linalg.norm(E_pose[:3, 3]) == 0 or scale == -1:
            if pnp_kp is None or pnp_kp[0] is kp1_buf:
                hybrid = self.pnp(kp_ref, kp_cur, kp1_buf, n, ref)
            else:
                p1, p2, pn = pnp_kp
                hybrid = self.pnp(p1.numpy()[:pn], p2.numpy()[:pn], p1, pn, ref)
            self.last["mode"] = "PnP"
        return hybrid

    def _pnp_on(self, pnp_kp, ref):
        """PnP tracker (the fallback) on the set (kp1, kp2, n) of pnp_tracker.kp_src."""
        p1, p2, pn = pnp_kp
        return self.pnp(p1.numpy()[:pn], p2.numpy()[:pn], p1, pn, ref)

    def track_fused_launch(self, cur, ref, kp1_buf, kp2_buf, n, flow_mean=None, pnp_kp=None):
        """The E branch of `track` with the device-side tail (tracking.Engine.essential_tail): after the keypoint count is known the
        host draws the five shuffles, enqueues the homography model, the essential-matrix repeats and the fused tail, and reads ONE
        packed result -- instead of eleven small reads with host arithmetic in between (keypoints, RANSAC info, GRIC, mask, pose,
        cheirality, triangulated depths, CNN depths, H-GRIC, scale).  Same decisions, same generator stream; the host copies of the
        keypoints are fetched only when the PnP fallback needs them.
        flow_mean (e_tracker.validity.method 'flow', E_tracker.py:182-186,249-257): the mean flow magnitude the selection read
        returned.  A closed gate draws no shuffle and leaves E_pose at identity, so the PnP fallback runs; otherwise the tail uses
        the flow-mode validity and no homography is launched.  pnp_kp: (kp1, kp2, n) of the PnP fallback's set (default: this one)."""
        c, eng, K = self.cfg, self.eng, self.K
        pnp_kp = pnp_kp or (kp1_buf, kp2_buf, n)
        if flow_mean is not None:
            self.last["flow_mean"] = flow_mean
            if not flow_mean > c.e_tracker.validity.thre:
                self.last.update(valid=False, inliers=np.ones(n, bool), mode="PnP", scale=None)
                return dict(pose=self._pnp_on(pnp_kp, ref))
        rs = c.scale_recovery.ransac
        perms = tracking.shuffles(self.rng, n, c.e_tracker.ransac.repeat)
        h = eng.homography_launch(kp2_buf, kp1_buf, n) if flow_mean is None else None
        w = eng.essential_launch(kp2_buf, kp1_buf, n, perms, K, threshold=c.e_tracker.ransac.reproj_thre)
        tail = eng.essential_tail_launch(w, h, kp2_buf, kp1_buf, n, K, cur.depth, self.rng, rs.min_samples, rs.max_trials, rs.stop_prob, rs.thre)
        return dict(tail=tail, w=w, ref=ref, kp1_buf=kp1_buf, kp2_buf=kp2_buf, n=n, last=self.last, pnp_kp=pnp_kp)

    def pnp_fused_launch(self, kp1_buf, kp2_buf, n, ref=None):
        """PnP tracker on the device keypoints (Engine.pnp_tail_launch): filter + unprojection, one read of the filtered count, the
        shuffles, the solver repeats; pnp_fused_finish reads the packed result.  Same pose bits and generator stream as `pnp`."""
        c = self.cfg
        ref = ref or self.ref
        pr = c.pnp_tracker.ransac
        return self.eng.pnp_tail_launch(kp1_buf, kp2_buf, n, ref.depth, self.K, c.depth.min_depth, c.depth.max_depth, self.rng,
                                        repeat=pr.repeat, iters=pr.iter, reproj_thre=pr.reproj_thre)

    def pnp_fused_finish(self, tok):
        pose, _, _ = self.eng.pnp_tail_finish(tok)
        return pose

    def track_fused_finish(self, tok):
        eng = self.eng
        w, ref, kp1_buf, kp2_buf, n = tok["w"], tok["ref"], tok["kp1_buf"], tok["kp2_buf"], tok["n"]
        self.last = tok["last"]
        o = eng.essential_tail_finish(tok["tail"])
        self.last.update(valid=o["valid"], inliers=None, inlier_handle=(w, o["best"]), mode="E", scale=None)
        hybrid = np.eye(4)
        hybrid[:3, :3] = o["R"]
        t = o["t"]
        scale = None
        if np.linalg.norm(t) != 0:
            scale = o["scale"]
            if scale != -1:
                hybrid[:3, 3] = t[:, 0] * scale
        self.last["scale"] = scale
        if np.linalg.norm(t) == 0 or scale == -1:                    # PnP fallback (dfvo.py:225-250)
            hybrid = self._pnp_on(tok.get("pnp_kp") or (kp1_buf, kp2_buf, n), ref)
            self.last["mode"] = "PnP"
        return hybrid

    def last_inliers(self):
        """Inlier mask of the last E-tracked frame (bool [n]); read from the device on demand in the fused path."""
        if self.last.get("inliers") is not None:
            return self.last["inliers"]
        hw = self.last.get("inlier_handle")
        if hw is None or hw[1] < 0:
            return None
        return hw[0]["mask"].numpy()[hw[1]].astype(bool)

    def scale_prepare(self, kp_ref, kp_cur, kp_cur_buf, T_21, depth_buf, n):
        """E_tracker.py:476-507,571-616: device triangulation + device gather of the CNN depth at the keypoints ->
        (depth ratios, number of valid ones).  Consumes no host RNG."""
        cx, cy, fx, fy = self.K
        k1 = self._buf("k1n", (n, 2), np.float64, self.eng.kp_capacity).upload((kp_ref - np.array([cx, cy])) / np.array([fx, fy]))
        k2 = self._buf("k2n", (n, 2), np.float64, self.eng.kp_capacity).upload((kp_cur - np.array([cx, cy])) / np.array([fx, fy]))
        z = self.eng.triangulate_depth(k1, k2, n, T_21)
        dk = self._buf("dkp", (n,), np.float32, self.eng.kp_capacity)
        self.rt.lib.check(self.rt.lib.dfvo_gather_depth(depth_buf.ptr, self.H, self.W, kp_cur_buf.ptr, n, dk.ptr, self.rt.stream_ptr()))
        return hostmath.last_writer_depth_ratio_sparse(kp_cur, z, dk.numpy(), self.H, self.W)

    def scale_finish(self, prep):
        """E_tracker.py:617-643: the 1-parameter RANSAC, on the device with the host generator's MT19937 state (Engine.ransac_scale)."""
        c = self.cfg.scale_recovery.ransac
        ratio, nvalid = prep
        if nvalid > 10:
            return self.eng.ransac_scale(ratio, c.min_samples, c.max_trials, c.stop_prob, c.thre, self.rng)
        return -1

    def scale_iterative(self, cur, ref, kp_ref, kp_cur, E_pose):
        """E_tracker.py:509-569 with kp_selection.rigid_flow_kp (SURVEY 8f rank 1): rigid-flow keypoint selection on the
        device each round; the depth ratios / scale RANSAC as in the simple method."""
        c = self.cfg
        rk = c.kp_selection.rigid_flow_kp
        T_21 = np.linalg.inv(E_pose)

        def select(T, score_method):
            return self.eng.rigid_flow_keypoints(ref.raw_depth, cur.fwd, cur.diff, T, self.K, rk.num_row, rk.num_col, rk.num_bestN,
                                                 float(rk.rigid_flow_thre), float(rk.optical_flow_thre), score_method, want_best=False)

        def find_scale(k_ref, k_cur):
            k2 = self._buf("kcur_it", (k_cur.shape[0], 2), np.float64, self.eng.kp_capacity).upload(k_cur)
            return self.scale_finish(self.scale_prepare(k_ref, k_cur, k2, T_21, cur.depth, k_cur.shape[0]))

        o = tracking.scale_recovery_iterative(select, find_scale, E_pose, getattr(self, "prev_scale", 0), (kp_ref, kp_cur),
                                              kp_src=c.scale_recovery.kp_src, score_method=c.scale_recovery.iterative_kp.score_method)
        self.prev_scale = o["scale"]
        self.last["rigid_flow_mask"] = o["rigid_flow_mask"]
        return o["scale"]

    def scale_recovery(self, kp_ref, kp_cur, kp_cur_buf, T_21, depth_buf, n):
        """E_tracker.py:476-507,571-643 in one call (scale_prepare + scale_finish)."""
        return self.scale_finish(self.scale_prepare(kp_ref, kp_cur, kp_cur_buf, T_21, depth_buf, n))

    def pnp(self, kp_ref, kp_cur, kp_ref_buf, n, ref=None):
        """pnp_tracker.py:45-125: keypoint filtering on the host arrays the tracker already holds, the reference depth
        at the keypoints gathered on the device, the five solvePnPRansac repeats + refits on the device (csrc/pnp.cu)."""
        c = self.cfg
        ref = ref or self.ref
        dk = self._buf("dkp", (n,), np.float32, self.eng.kp_capacity)
        self.rt.lib.check(self.rt.lib.dfvo_gather_depth(ref.depth.ptr, self.H, self.W, kp_ref_buf.ptr, n, dk.ptr, self.rt.stream_ptr()))
        d_all = dk.numpy().astype(np.float64)
        keep = (kp_cur[:, 0] >= 0) & (kp_cur[:, 0] < self.W) & (kp_cur[:, 1] >= 0) & (kp_cur[:, 1] < self.H)
        kp1, kp2, d = kp_ref[keep], kp_cur[keep], d_all[keep]
        keep = (d != 0) & (d < c.depth.max_depth) & (d > c.depth.min_depth)
        kp1, kp2, d = kp1[keep], kp2[keep], d[keep]
        pose, _ = tracking.compute_pose_3d2d(self.eng, kp1, kp2, d, self.K, repeat=c.pnp_tracker.ransac.repeat,
                                             iters=c.pnp_tracker.ransac.iter, reproj_thre=c.pnp_tracker.ransac.reproj_thre,
                                             rng=self.rng)
        return pose

    # ------------------------------------------------------------------ driver step
    def advance(self, cur, ref):
        """Track the FrameState `cur` against `ref` (None: `cur` starts the sequence), chain the global pose and record
        ``poses[cur.id]`` / ``modes[cur.id]``; returns the global pose.  For callers that run the networks themselves and only
        use this pipeline as the tracker of one sequence (multiseq.SequenceBatch); runs on the current stream."""
        return self._advance(cur, ref)

    def _advance(self, cur, ref):
        """Track `cur` against `ref` and chain the global pose (dfvo.py:358-403 loop body)."""
        return self._advance_finish(self._advance_launch(cur, ref))

    def _advance_launch(self, cur, ref):
        if ref is None:
            return (cur, None, 0.0)
        t0 = time.perf_counter()
        tok = self.track_launch(cur, ref)
        return (cur, tok, (time.perf_counter() - t0) * 1e3)

    def _advance_finish(self, launched):
        cur, tok, ms0 = launched
        fid = cur.id
        if tok is None:
            self.global_pose = np.eye(4)
            self.motion = np.eye(4)
        else:
            t0 = time.perf_counter()
            rel = self.track_finish(tok)
            self.track_ms[fid] = ms0 + (time.perf_counter() - t0) * 1e3      # host time of the tracker path (includes its device waits)
            self.motion = rel.copy()
            # update_global_pose (dfvo.py:109-119): t_w += R_w t ; R_w = R_w R
            self.global_pose[:3, 3:] = self.global_pose[:3, :3] @ rel[:3, 3:] + self.global_pose[:3, 3:]
            self.global_pose[:3, :3] = self.global_pose[:3, :3] @ rel[:3, :3]
        self.poses[fid] = self.global_pose.copy()
        self.modes[fid] = self.last.get("mode") if tok is not None else None
        return self.poses[fid]

    def step(self, img):
        """One VO frame.  In-order mode: returns the global pose (4x4) after this frame.  Overlap mode: returns the
        pose of the previous frame (None on the first call); see __init__."""
        fid = self.stage
        self.stage += 1
        if not self.overlap:
            cur = self.infer(img, fid)
            pose = self._advance(cur, self.ref)
            self.ref = cur
            return pose
        pose = None
        with self.rt.on_stream(self.s_nets[fid % len(self.engs)]):
            self._depth_done = None
            with self.rt.nvtx("dfvo.infer"):
                cur = self.infer(img, fid)                  # uses self.ref (previous image) for the flow pair
            if self._depth_done is not None:                # join the depth side stream
                self.rt.wait_event(self._depth_done)
            cur.ready = self.rt.record_event()
        self.ref = cur
        if self.tracker_thread:
            return self._hand_over(cur)
        if self.pipelined:
            if self._tok is not None:                            # the tracker enqueued by the previous step ran while the
                pose = self._finish_inflight()                  # networks above were being enqueued
            self.pending.append(cur)
            if len(self.pending) > self.inflight:
                self._launch_oldest()
            return pose
        pose = self._track_oldest() if len(self.pending) >= self.inflight else None
        self.pending.append(cur)
        return pose

    def _launch_oldest(self):
        nxt = self.pending.pop(0)
        with self.rt.on_stream(self.s_trk), self.rt.nvtx("dfvo.track_launch"):
            self.rt.wait_event(nxt.ready)
            self._tok = self._advance_launch(nxt, self.trk_ref)
        self.trk_ref = nxt

    def _finish_inflight(self):
        launched, self._tok = self._tok, None
        with self.rt.on_stream(self.s_trk), self.rt.nvtx("dfvo.track_finish"):
            return self._advance_finish(launched)

    # ---- tracker thread -------------------------------------------------------------------------------------------------
    def _start_tracker_thread(self):
        import queue
        import threading
        self._q = queue.Queue()
        self._cv = threading.Condition()
        self._tracked = -1           # id of the last frame whose pose is in self.poses
        self._thr_exc = None

        def loop():
            if getattr(self.rt, "is_device", True) and hasattr(self.rt, "torch"):
                self.rt.torch.cuda.set_device(self.rt.device)
            while True:
                st = self._q.get()
                if st is None:
                    return
                try:
                    with self.rt.on_stream(self.s_trk):
                        self.rt.wait_event(st.ready)
                        self._advance(st, self.trk_ref)
                    self.trk_ref = st
                except BaseException as e:          # surfaced by the next step() / flush() on the caller's thread
                    self._thr_exc = e
                with self._cv:
                    self._tracked = st.id
                    self._cv.notify_all()
                if self._thr_exc is not None:
                    return
        self._thr = threading.Thread(target=loop, name="dfvo-tracker", daemon=True)
        self._thr.start()

    def _wait_tracked(self, fid):
        with self._cv:
            while self._tracked < fid and self._thr_exc is None:
                self._cv.wait(0.5)
        if self._thr_exc is not None:
            e, self._thr_exc = self._thr_exc, None
            raise e

    def _hand_over(self, cur):
        """tracker_thread mode: queue `cur` for tracking, return the pose of frame cur.id - inflight (the buffers are
        inflight + 2 deep, so the networks may run exactly that far ahead of the tracker)."""
        if self._thr is None:
            self._start_tracker_thread()
        self._q.put(cur)
        back = cur.id - self.inflight
        if back < 0:
            return None
        self._wait_tracked(back)
        return self.poses[back]

    def close(self):
        """Stops the tracker thread (tracker_thread mode); the pipeline can be used again afterwards."""
        if self._thr is not None:
            self._q.put(None)
            self._thr.join(timeout=30)
            self._thr = None

    def _track_oldest(self):
        nxt = self.pending.pop(0)
        with self.rt.on_stream(self.s_trk), self.rt.nvtx("dfvo.track"):
            self.rt.wait_event(nxt.ready)
            pose = self._advance(nxt, self.trk_ref)
        self.trk_ref = nxt
        return pose

    def flush(self):
        """Overlap mode: track the frames whose networks are still in flight; returns the last pose for inflight=1 (None if
        there is none), the list of remaining poses for inflight=2."""
        poses = []
        if self.pipelined:
            if self._tok is not None:
                poses.append(self._finish_inflight())
            while self.pending:
                self._launch_oldest()
                poses.append(self._finish_inflight())
            return poses
        if self.tracker_thread:
            last = self.stage - 1
            if self._thr is not None and last >= 0:
                self._wait_tracked(last)
                poses = [self.poses[f] for f in range(max(last - self.inflight + 1, 0), last + 1)]
        while self.overlap and self.pending:
            poses.append(self._track_oldest())
        if self.inflight > 1:
            return poses
        return poses[-1] if poses else None
