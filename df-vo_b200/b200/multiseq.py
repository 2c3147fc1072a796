"""Several independent image sequences on one GPU.

:class:`SequenceBatch` tracks S sequences of the same frame size and configuration (the sequences of an evaluation, the cameras
of a rig) in one process.  Per step it runs each network ONCE over all S frames -- LiteFlowNet over S pairs, monodepth2 over S
feeds and (with kp_selection.depth_consistency) the PoseNet over S feed pairs -- so the coarse pyramid levels, which leave most
SMs idle for one image, get S times the work per launch.  Then it runs each sequence's tracker, which is a
:class:`pipeline.FramePipeline` of its own used through :meth:`FramePipeline.advance`: every tracking configuration the pipeline
accepts works here, with the same arithmetic and generator stream, so a sequence gives exactly the poses an independent
FramePipeline gives on the same frames.
"""
import time

import numpy as np

from . import config as cfg_mod
from . import native, tracking
from . import runtime as rt_mod
from .pipeline import FramePipeline, FrameState


class SequenceBatch:
    def __init__(self, Ks, height, width, cfg=None, precision=native.PREC_BF16, rngs=None, overlap=False, inject=None, runtime=None):
        """Ks: one K = [cx, cy, fx, fy] per sequence (S = len(Ks)).  rngs: one generator per sequence (the host draws of its
        tracker), default ``np.random.RandomState(cfg.seed)`` each.

        overlap=False: ``step(imgs)`` returns the poses of `imgs`.  overlap=True: the networks of step t run on a network stream
        while the trackers of step t-1 run on a high-priority tracker stream; ``step`` returns the poses of step t-1 (all None on
        the first call) and ``flush()`` the last ones -- as ``FramePipeline(overlap=True, inflight=1)``.

        inject: optional ``callable(batch, s, frame_state)`` run after the networks of a step were enqueued, once per sequence
        `s` that has a frame in the step (on the network stream): the hook through which tests and benchmarks replace network
        outputs by analytic ones, as FramePipeline's ``inject``."""
        self.S = len(Ks)
        if self.S < 1:
            raise ValueError("SequenceBatch needs at least one sequence")
        self.cfg = cfg or cfg_mod.default_cfg(height, width)
        self.H, self.W = int(height), int(width)
        self.rt = runtime or rt_mod.get()
        self.precision = precision
        self.overlap = bool(overlap)
        self.inject = inject
        if rngs is None:
            rngs = [np.random.RandomState(self.cfg.seed) for _ in range(self.S)]
        if len(rngs) != self.S:
            raise ValueError("SequenceBatch: %d generators for %d sequences" % (len(rngs), self.S))
        self.eng = tracking.Engine(self.H, self.W, self.rt)         # the batched networks
        # frame buffers per sequence: a frame serves its own tracker and, as reference, the next frame's networks and tracker;
        # in overlap mode the networks of a new frame run while the tracker of the previous one still reads its reference
        self.nslots = 3 if self.overlap else 2
        # batched network outputs (flows, PoseNet poses) are read only by the trackers of their own step
        self.nout = 2 if self.overlap else 1
        self.seqs = [None] * self.S          # per-sequence trackers
        self._net_ref = [None] * self.S      # (FrameState, slot) of the last frame whose networks were enqueued
        self._trk_ref = [None] * self.S      # (FrameState, slot) of the last tracked frame
        self._nframes = [0] * self.S
        for s in range(self.S):
            self._start(s, Ks[s], rngs[s])
        self.depth_consistency = self.seqs[0].depth_consistency
        self.stage = 0
        self.pending = []                    # overlap mode: (s, (FrameState, slot)) of the last step: networks enqueued, not tracked
        self._ready = None
        self.track_ms = []                   # host ms per step spent in the S trackers (includes their device waits)
        if self.overlap:
            self.s_net = self.rt.new_stream()
            self.s_trk = self.rt.new_stream(high_priority=True)

    def _start(self, s, K, rng):
        self.seqs[s] = FramePipeline(K, self.H, self.W, cfg=self.cfg, precision=self.precision, runtime=self.rt, rng=rng,
                                     engine=tracking.Engine(self.H, self.W, self.rt))
        self._net_ref[s] = self._trk_ref[s] = None
        self._nframes[s] = 0

    @property
    def poses(self):
        """poses[s]: {frame index within sequence s: 4x4 global pose}, as FramePipeline.poses."""
        return [p.poses for p in self.seqs]

    @property
    def modes(self):
        """modes[s]: {frame index: tracker branch ('E', 'PnP', 'const'; None for the first frame)}, as FramePipeline.modes."""
        return [p.modes for p in self.seqs]

    # ------------------------------------------------------------------ setup
    def load_weights(self, flow_weights, depth_enc, depth_dec, pose_enc=None, pose_dec=None):
        """As FramePipeline.load_weights; builds LiteFlowNet for S pairs, monodepth2 and (depth consistency) the PoseNet for
        batches of S."""
        if self.depth_consistency and (pose_enc is None or pose_dec is None):
            raise ValueError("kp_selection.depth_consistency needs the PoseNet weights (pose_enc, pose_dec)")
        e = self.eng
        e.build_flow(flow_weights, pairs=self.S, precision=self.precision)
        e.build_depth(depth_enc, depth_dec, precision=self.precision, dataset=self.cfg.dataset, batch=self.S)
        if self.depth_consistency:
            e.build_pose(pose_enc, pose_dec, precision=self.precision, dataset=self.cfg.dataset, batch=self.S)
        self._alloc_buffers()

    def _alloc_buffers(self):
        """Per-sequence frame buffers (nslots batched arrays, one entry per sequence) and the batched network outputs."""
        S, H, W, rt = self.S, self.H, self.W, self.rt
        fh, fw = self.eng.feed_h, self.eng.feed_w
        mk = lambda shape, dt: [rt.empty((S,) + shape, dt) for _ in range(self.nslots)]
        self._img, self._feed = mk((H, W, 3), np.uint8), mk((3, fh, fw), np.float32)
        self._raw, self._dep = mk((H, W), np.float32), mk((H, W), np.float32)
        self._blank_img = rt.zeros((H, W, 3), np.uint8)             # network input of a sequence without any frame yet
        self._blank_feed = rt.zeros((1, 3, fh, fw), np.float32)
        self._flow = [(rt.empty((S, 2, H, W), np.float32), rt.empty((S, 2, H, W), np.float32), rt.empty((S, H, W), np.float32))
                      for _ in range(self.nout)]
        self._dpose = [rt.empty((S, 4, 4), np.float32) for _ in range(self.nout)] if self.depth_consistency else None

    # ------------------------------------------------------------------ per step
    def _check(self, imgs):
        if len(imgs) != self.S:
            raise ValueError("SequenceBatch.step: %d frames given for %d sequences" % (len(imgs), self.S))
        for s, img in enumerate(imgs):
            if img is not None and tuple(img.shape) != (self.H, self.W, 3):
                raise ValueError("SequenceBatch.step: frame of sequence %d has shape %s, expected (%d, %d, 3)"
                                 % (s, tuple(img.shape), self.H, self.W))

    def _free_slot(self, s):
        """Buffer slot for the next frame of sequence s: the step's own slot unless a frame still needed lives there."""
        busy = {r[1] for r in (self._net_ref[s], self._trk_ref[s]) if r is not None}
        k = self.stage % self.nslots
        return k if k not in busy else min(set(range(self.nslots)) - busy)

    def _infer(self, imgs):
        """Upload and the per-frame buffers (views into the batched ones), the networks, the inject hook; returns
        [(FrameState, slot) or None] per sequence."""
        S, e, HW = self.S, self.eng, self.H * self.W
        fh, fw = e.feed_h, e.feed_w
        out = self.stage % self.nout
        fwd_b, bwd_b, diff_b = self._flow[out]
        refs = [r[0] if r is not None else None for r in self._net_ref]
        curs = [None] * S
        for s, img in enumerate(imgs):
            if img is None:
                continue
            k = self._free_slot(s)
            st = FrameState()
            st.id = self._nframes[s]
            self._nframes[s] += 1
            st.img = img if isinstance(img, rt_mod.Buf) else self._img[k].view((self.H, self.W, 3), s * HW * 3).upload(img)
            st.feed = self._feed[k].view((1, 3, fh, fw), s * 3 * fh * fw)
            st.raw_depth = self._raw[k].view((self.H, self.W), s * HW)
            st.depth = self._dep[k].view((self.H, self.W), s * HW)
            if refs[s] is not None:
                st.fwd, st.bwd = fwd_b.view((1, 2, self.H, self.W), s * 2 * HW), bwd_b.view((1, 2, self.H, self.W), s * 2 * HW)
                st.diff = diff_b.view((1, self.H, self.W), s * HW)
                if self.depth_consistency:
                    st.deep_pose = self._dpose[out].view((4, 4), s * 16)
            curs[s] = (st, k)
        self._networks([c[0] if c else None for c in curs], refs, out)
        for s in range(S):
            if curs[s]:
                if self.inject is not None:
                    self.inject(self, s, curs[s][0])
                self._net_ref[s] = curs[s]
        return curs

    def _networks(self, curs, refs, out):
        """The step's networks, each one forward over all S: feeds, monodepth2 + depth post-processing, the PoseNet of (ref, cur)
        feeds (depth consistency) and LiteFlowNet of (ref, cur) images, into the buffers of the FrameStates `curs` (None: idle).
        A sequence without a frame or without a reference is fed a stand-in and its output entry is ignored."""
        S, e, c = self.S, self.eng, self.cfg
        fh, fw = e.feed_h, e.feed_w
        for s in range(S):
            if curs[s]:
                e.depth_feed(curs[s].img, out=curs[s].feed)             # LANCZOS resize + ToTensor on the device
        d = e.depth_batch([curs[s].feed if curs[s] else (refs[s].feed if refs[s] else self._blank_feed) for s in range(S)])
        for s in range(S):
            if curs[s]:
                e.depth_post(d.view((fh, fw), s * fh * fw), c.crop.depth_crop, float(c.depth.min_depth), float(c.depth.max_depth),
                             curs[s].raw_depth, curs[s].depth)
        paired = [bool(curs[s] and refs[s]) for s in range(S)]
        if not any(paired):
            return
        stand_in = [(curs[s] or refs[s]) for s in range(S)]
        if self.depth_consistency:
            feeds = [(refs[s].feed, curs[s].feed) if paired[s] else ((stand_in[s].feed if stand_in[s] else self._blank_feed),) * 2
                     for s in range(S)]
            e.pose_batch([f[0] for f in feeds], [f[1] for f in feeds], out=self._dpose[out])
        imgs = []
        for s in range(S):
            imgs += [refs[s].img, curs[s].img] if paired[s] else [stand_in[s].img if stand_in[s] else self._blank_img] * 2
        e.flow(imgs, out=self._flow[out])

    def _track(self, s, cur):
        """Tracker of sequence s on the frame (FrameState, slot) `cur` (current stream); returns its global pose."""
        ref = self._trk_ref[s]
        pose = self.seqs[s].advance(cur[0], ref[0] if ref is not None else None)
        self._trk_ref[s] = cur
        return pose

    def _track_pending(self):
        poses = [None] * self.S
        if not self.pending:
            return poses
        t0 = time.perf_counter()
        with self.rt.on_stream(self.s_trk):
            self.rt.wait_event(self._ready)
            for s, cur in self.pending:
                poses[s] = self._track(s, cur)
        self.track_ms.append((time.perf_counter() - t0) * 1e3)
        self.pending = []
        return poses

    def step(self, imgs):
        """One frame of each sequence: ``imgs[s]`` is a uint8 HWC frame (host array, pinned host tensor or device ``runtime.Buf``)
        or None for a sequence that is idle this step (its buffers, reference frame, generator and pose do not advance).
        Returns S global poses (None for an idle sequence; in overlap mode the poses of the previous step)."""
        self._check(imgs)
        if not self.overlap:
            curs = self._infer(imgs)
            self.stage += 1
            poses = [None] * self.S
            t0 = time.perf_counter()
            for s in range(self.S):
                if curs[s]:
                    poses[s] = self._track(s, curs[s])
            self.track_ms.append((time.perf_counter() - t0) * 1e3)
            return poses
        with self.rt.on_stream(self.s_net):
            curs = self._infer(imgs)
            ready = self.rt.record_event()
        self.stage += 1
        poses = self._track_pending()                 # the trackers of the previous step, while the networks above run
        self.pending = [(s, curs[s]) for s in range(self.S) if curs[s]]
        self._ready = ready
        return poses

    def flush(self):
        """Overlap mode: track the frames of the last step; returns their S poses (None where a sequence had no frame)."""
        return self._track_pending()

    def reset(self, s, K=None, rng=None):
        """Start a new sequence in slot s (intrinsics K, default the slot's current ones; generator rng, default a fresh
        ``RandomState(cfg.seed)``).  In overlap mode the slot's last frame is tracked first.  Returns the finished sequence's
        poses ({frame index: 4x4 global pose})."""
        if not isinstance(s, (int, np.integer)) or not 0 <= s < self.S:
            raise IndexError("SequenceBatch.reset: slot %r out of range for %d sequences" % (s, self.S))
        mine = [p for p in self.pending if p[0] == s]
        if mine:
            with self.rt.on_stream(self.s_trk):
                self.rt.wait_event(self._ready)
                self._track(s, mine[0][1])
            self.pending = [p for p in self.pending if p[0] != s]
        old = self.seqs[s]
        self._start(s, old.K if K is None else K, np.random.RandomState(self.cfg.seed) if rng is None else rng)
        return old.poses
