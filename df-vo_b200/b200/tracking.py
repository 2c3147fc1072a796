"""Device-side building blocks of one DF-VO tracking step, shared by the reference-API mirror
(``df-vo_b200/libs``) and the device-resident pipeline (``b200/pipeline.py``).

Every numeric step is a call into the C ABI (``include/dfvo_b200.h``); this module only owns buffers,
the order of calls and the few host-side decisions the reference makes on the host as well (RNG draws,
majority vote, sentinels).  There is no CPU implementation of the kernels here.
"""
import collections
import ctypes

import numpy as np

from . import hostmath, native
from . import runtime as rt_mod

KITTI_DEPTH = dict(min_depth=0.1, max_depth=100.0, baseline=5.4)      # monodepth2.py:73-77
TUM_DEPTH = dict(min_depth=0.1, max_depth=10.0, baseline=1.0)         # monodepth2.py:78-81


def depth_constants(dataset):
    return TUM_DEPTH if "tum" in dataset else KITTI_DEPTH


def pose_baseline_multiplier(dataset):
    """Monodepth2PoseNet.stereo_baseline_multiplier (pose/monodepth2/monodepth2.py:77-84)."""
    return 5.4 if ("kitti" in dataset or "robotcar" in dataset) else 1.0


def shuffles(rng, n, repeat):
    """The reference's per-repeat shuffles (E_tracker.py:225-226, pnp_tracker.py:90-95): `repeat` permutations of arange(n), each
    drawn by rng.shuffle in turn, so the generator advances exactly as in the reference."""
    perms = []
    for _ in range(repeat):
        order = np.arange(0, n, 1)
        rng.shuffle(order)
        perms.append(order)
    return perms


def _mt_state_in(rng, block, who):
    """Write `rng`'s MT19937 state into the result block (host float64 array) at DFVO_TAIL_MT; returns the state."""
    st = rng.get_state()
    if st[0] != "MT19937":
        raise TypeError("%s needs a legacy MT19937 generator (np.random / np.random.RandomState)" % who)
    u = block[native.DFVO_TAIL_MT:native.DFVO_TAIL_SCALE_IO].view(np.uint32)
    u[:624] = st[1]
    u[624] = st[2]
    return st


def _mt_state_out(rng, block, st):
    """Install the advanced MT19937 state the device left in the result block into `rng` (`st`: the state written at launch)."""
    u = block[native.DFVO_TAIL_MT:native.DFVO_TAIL_SCALE_IO].view(np.uint32)
    rng.set_state(("MT19937", u[:624].copy(), int(u[624]), st[3], st[4]))


class Engine:
    """One ``dfvo_ctx`` + its buffers for a fixed image size."""

    def __init__(self, height, width, runtime=None):
        self.rt = runtime or rt_mod.get()
        self.lib = self.rt.lib
        self.ctx = native.Context(self.lib, getattr(self.rt, "device_index", 0))     # the dfvo_ctx lives on the runtime's device
        self.H, self.W = int(height), int(width)
        self.flow_ready = False
        self.depth_ready = False
        self.pose_ready = False
        # Workspaces are allocated once per configuration for a CAPACITY of keypoints (grown geometrically if a frame ever
        # exceeds it) and handed out as exactly-shaped views: with local_bestN the keypoint count changes almost every
        # frame, and a per-count cache would grow without bound and put cudaMalloc into the tracked region.
        self._subsets = collections.OrderedDict()    # (N, iters) -> device table of OpenCV's subset stream; LRU-bounded
        self._subsets_cap = 256
        self._ess_ws, self._h_ws, self._pnp_ws = {}, {}, {}
        self._sel, self._bsel, self._rf = {}, {}, {}
        self.kp_capacity = 2048

    # ------------------------------------------------------------------ networks
    def build_flow(self, weights, pairs=1, precision=native.PREC_BF16):
        self.ctx.load_weights(native.NET_LITEFLOWNET, weights)
        self.ctx.liteflow_build(self.H, self.W, pairs, precision)
        self.pairs = pairs
        self.flow_fwd = self.rt.empty((pairs, 2, self.H, self.W), np.float32)
        self.flow_bwd = self.rt.empty((pairs, 2, self.H, self.W), np.float32)
        self.flow_diff = self.rt.empty((pairs, self.H, self.W), np.float32)
        self.flow_ready = True

    def build_depth(self, enc, dec, precision=native.PREC_BF16, dataset="kitti_odom"):
        self.ctx.load_weights(native.NET_MONODEPTH2, enc)
        self.ctx.load_weights(native.NET_MONODEPTH2, dec)
        self.feed_h, self.feed_w = int(enc["height"]), int(enc["width"])
        c = depth_constants(dataset)
        self.ctx.monodepth2_build(self.feed_h, self.feed_w, precision, c["min_depth"], c["max_depth"], c["baseline"])
        self.depth_out = self.rt.empty((self.feed_h, self.feed_w), np.float32)
        self.depth_ready = True

    def build_pose(self, enc, dec, precision=native.PREC_BF16, dataset="kitti_odom"):
        """Monodepth2PoseNet (pose/monodepth2/monodepth2.py:31-84) at the depth network's feed size (deep_models.py:220), so
        build_depth first.  ``enc``: pose_encoder.pth (only its ``encoder.*`` keys are used), ``dec``: pose.pth."""
        assert self.depth_ready, "build_depth first: the PoseNet reads the depth network's feeds"
        self.ctx.load_weights(native.NET_POSENET, {k: v for k, v in enc.items() if k.startswith("encoder.")})
        self.ctx.load_weights(native.NET_POSENET, dec)
        self.ctx.posenet_build(self.feed_h, self.feed_w, precision, pose_baseline_multiplier(dataset))
        self.pose_out = self.rt.empty((4, 4), np.float32)
        self.pose_ready = True

    def pose(self, feed_ref, feed_cur, out=None):
        """Monodepth2PoseNet.inference_pose of the depth feeds [ref, cur] (deep_models.py:208-230) -> device fp32 [4,4]."""
        assert self.pose_ready, "build_pose first"
        out = out or self.pose_out
        self.ctx.posenet_forward(feed_ref.ptr, feed_cur.ptr, out.ptr, self.rt.stream_ptr())
        return out

    def depth_consistency(self, depth_cur, depth_ref, T_buf, K_mat, inv_K_mat, out=None):
        """DepthConsistency.compute (depth_consistency.py:31-163): [H,W] raw depths of the current / reference frame and the
        device fp32 4x4 pose -> depth_diff [H,W] (device).  K_mat / inv_K_mat: the 3x3 float64 intrinsics, cast to float32 like
        the reference."""
        if out is None:
            if getattr(self, "_dc_out", None) is None:
                self._dc_out = self.rt.empty((self.H, self.W), np.float32)
            out = self._dc_out
        K32 = np.ascontiguousarray(np.asarray(K_mat, np.float64)[:3, :3], np.float32)
        iK32 = np.ascontiguousarray(np.asarray(inv_K_mat, np.float64)[:3, :3], np.float32)
        self.lib.check(self.lib.dfvo_depth_consistency(depth_cur.ptr, depth_ref.ptr, self.H, self.W, T_buf.ptr,
                                                       K32.ctypes.data_as(ctypes.c_void_p), iK32.ctypes.data_as(ctypes.c_void_p),
                                                       out.ptr, self.rt.stream_ptr()))
        return out

    def flow(self, img_bufs, out=None):
        """img_bufs: 2*pairs uint8 HWC device buffers [ref0, cur0, ...] -> (fwd, bwd, diff) buffers
        (`out` or the engine's own)."""
        assert self.flow_ready, "build_flow first"
        ptrs = [b.ptr.value for b in img_bufs]
        fwd, bwd, diff = out or (self.flow_fwd, self.flow_bwd, self.flow_diff)
        self.ctx.liteflow_forward(ptrs, fwd.ptr, bwd.ptr, diff.ptr, self.rt.stream_ptr())
        return fwd, bwd, diff

    def depth_feed(self, img_buf, out=None):
        """deep_models.py:195-198 on the device: PIL-exact LANCZOS resize of the uint8 HWC frame to the feed size +
        ToTensor -> float32 [1,3,feed_h,feed_w] (csrc/depth_ops.cu, tables from b200/lanczos.py)."""
        from . import lanczos
        H, W = img_buf.shape[0], img_buf.shape[1]
        key = (H, W, self.feed_h, self.feed_w)
        if getattr(self, "_lz_key", None) != key:
            bh, kh, ksh = lanczos.coeffs(W, self.feed_w)
            bv, kv, ksv = lanczos.coeffs(H, self.feed_h)
            self._lz = dict(bh=self.rt.from_host(bh), kh=self.rt.from_host(kh), ksh=ksh, bv=self.rt.from_host(bv),
                            kv=self.rt.from_host(kv), ksv=ksv, tmp=self.rt.empty((H, self.feed_w, 3), np.uint8),
                            feed=self.rt.empty((1, 3, self.feed_h, self.feed_w), np.float32))
            self._lz_key = key
        z = self._lz
        out = out or z["feed"]
        self.lib.check(self.lib.dfvo_lanczos_resize_u8(img_buf.ptr, H, W, z["bh"].ptr, z["kh"].ptr, z["ksh"], z["bv"].ptr, z["kv"].ptr,
                                                       z["ksv"], self.feed_h, self.feed_w, z["tmp"].ptr, None, out.ptr,
                                                       self.rt.stream_ptr()))
        return out

    def depth(self, feed_buf, out=None):
        """feed_buf: float32 [1,3,feed_h,feed_w] device buffer -> depth [feed_h, feed_w]."""
        assert self.depth_ready, "build_depth first"
        out = out or self.depth_out
        self.ctx.monodepth2_forward(feed_buf.ptr, out.ptr, self.rt.stream_ptr())
        return out

    def depth_post(self, depth_buf, crop, min_depth, max_depth, raw_out=None, out=None):
        raw_out = raw_out or self.rt.empty((self.H, self.W), np.float32)
        out = out or self.rt.empty((self.H, self.W), np.float32)
        h, w = depth_buf.shape[-2:]
        self.lib.check(self.lib.dfvo_depth_post(depth_buf.ptr, h, w, self.H, self.W, crop[0][0], crop[0][1], crop[1][0],
                                                crop[1][1], min_depth, max_depth, raw_out.ptr, out.ptr, self.rt.stream_ptr()))
        return raw_out, out

    # ------------------------------------------------------------------ selection
    def select_local_bestn(self, diff_buf, flow_fwd_buf, rows, cols, num_bestN, thre, depth_diff_buf=None, depth_thre=0.05,
                           with_flow_mean=False):
        """local_bestN (kp_selection.py:74-200) + keypoint gather.  Returns (good, n, kp1, kp2, mask-less)
        with kp buffers float64 [num_bestN, 2] (first n rows valid).  One small D2H (status).
        with_flow_mean: the same single read also carries the mean flow magnitude of the selection (the E-tracker's 'flow'
        validity gate, dfvo_flow_mean), appended as a fifth element."""
        quota = num_bestN // (rows * cols)
        key = (rows, cols, quota)
        if key not in self._sel:
            self._sel[key] = dict(idx=self.rt.empty((rows * cols * quota,), np.int32), cc=self.rt.empty((rows * cols,), np.int32),
                                  st=self.rt.empty((4,), np.int32), kp1=self.rt.empty((rows * cols * quota, 2), np.float64),
                                  kp2=self.rt.empty((rows * cols * quota, 2), np.float64), n=self.rt.empty((1,), np.int32))
        s = self._sel[key]
        st = self.rt.stream_ptr()
        self.lib.check(self.lib.dfvo_local_bestn(diff_buf.ptr, depth_diff_buf.ptr if depth_diff_buf else None, self.H, self.W,
                                                 rows, cols, num_bestN, thre, depth_thre, s["idx"].ptr, s["cc"].ptr, s["st"].ptr, st))
        self.lib.check(self.lib.dfvo_gather_keypoints(s["idx"].ptr, s["cc"].ptr, rows * cols, quota, flow_fwd_buf.ptr, self.H,
                                                      self.W, s["kp1"].ptr, s["kp2"].ptr, s["n"].ptr, st))
        if with_flow_mean:                                        # the mean flow magnitude travels with the status (one read)
            if "fm" not in s:
                s["fm"] = self.rt.empty((3,), np.float64)
            self.lib.check(self.lib.dfvo_flow_mean(s["kp1"].ptr, s["kp2"].ptr, 0, s["st"].ptr, s["fm"].ptr, st))
            o = s["fm"].numpy()
            return bool(o[0]), int(o[1]), s["kp1"], s["kp2"], float(o[2])
        status = s["st"].numpy()
        return bool(status[0]), int(status[1]), s["kp1"], s["kp2"]

    def flow_mean(self, kp_ref_buf, kp_cur_buf, n):
        """np.mean(np.linalg.norm(kp_ref - kp_cur, axis=1)) of n device keypoint pairs, bit-equal to NumPy (E_tracker.py:184)."""
        if not hasattr(self, "_fm"):
            self._fm = self.rt.empty((3,), np.float64)
        self.lib.check(self.lib.dfvo_flow_mean(kp_ref_buf.ptr, kp_cur_buf.ptr, int(n), None, self._fm.ptr, self.rt.stream_ptr()))
        return float(self._fm.numpy()[2])

    def select_bestn(self, diff_buf, flow_fwd_buf, N):
        """bestN_flow_kp (kp_selection.py:33-71)."""
        if N not in self._bsel:
            nb = int(self.lib.dfvo_bestn_workspace_bytes(self.H, self.W))
            self._bsel[N] = dict(idx=self.rt.empty((N,), np.int32), ws=self.rt.empty((nb,), np.uint8),
                                 kp1=self.rt.empty((N, 2), np.float64), kp2=self.rt.empty((N, 2), np.float64))
        s = self._bsel[N]
        st = self.rt.stream_ptr()
        self.lib.check(self.lib.dfvo_bestn(diff_buf.ptr, self.H, self.W, N, s["idx"].ptr, s["ws"].ptr, s["ws"].shape[0], st))
        self.lib.check(self.lib.dfvo_gather_keypoints(s["idx"].ptr, None, 1, N, flow_fwd_buf.ptr, self.H, self.W, s["kp1"].ptr,
                                                      s["kp2"].ptr, None, st))
        return True, N, s["kp1"], s["kp2"]

    def rigid_flow_keypoints(self, raw_depth_buf, flow_fwd_buf, flow_diff_buf, T, K, rows=10, cols=10, num_bestN=2000, rigid_thre=5.0,
                             flow_thre=0.1, score_method="opt_flow", want_best=True):
        """``EssTracker.kp_selection_good_depth`` (E_tracker.py:645-705) on the device: rigid-flow inconsistency map of the
        reference depth under pose ``T`` (4x4, float64), then ``opt_rigid_flow_kp`` (kp_selection.py:203-324): the
        'uniform' list per cell and (optionally) the 'best' set by ``score_method``.  Returns dict with the device map
        ``rigid_flow_diff`` [H,W] and host float64 keypoints kp1/kp2_uniform [n,2], kp1/kp2_best [m,2] (canonical order:
        cell-major; uniform in the reference's own order, best ascending by pixel index inside a cell)."""
        cx, cy, fx, fy = K
        r = self._rf_buffers(rows, cols, num_bestN // (rows * cols))
        Th = np.ascontiguousarray(np.asarray(T, np.float64).reshape(-1)[:16])
        self.lib.check(self.lib.dfvo_rigid_flow_diff(raw_depth_buf.ptr, flow_fwd_buf.ptr, self.H, self.W, Th.ctypes.data_as(ctypes.c_void_p),
                                                     fx, fy, cx, cy, r["map"].ptr, self.rt.stream_ptr()))
        return self.opt_rigid_flow_select(r["map"], flow_fwd_buf, flow_diff_buf, rows, cols, num_bestN, rigid_thre, flow_thre,
                                          score_method, want_best)

    def _rf_buffers(self, rows, cols, quota):
        key = (rows, cols, quota)
        if key not in self._rf:
            cells = rows * cols
            mk = lambda: dict(idx=self.rt.empty((cells * quota,), np.int32), cc=self.rt.empty((cells,), np.int32),
                              kp1=self.rt.empty((cells * quota, 2), np.float64), kp2=self.rt.empty((cells * quota, 2), np.float64),
                              n=self.rt.empty((1,), np.int32))
            self._rf[key] = dict(map=self.rt.empty((self.H, self.W), np.float32), u=mk(), b=mk(), st=self.rt.empty((4,), np.int32))
        return self._rf[key]

    def opt_rigid_flow_select(self, rigid_map_buf, flow_fwd_buf, flow_diff_buf, rows=10, cols=10, num_bestN=2000, rigid_thre=5.0,
                              flow_thre=0.1, score_method="opt_flow", want_best=True):
        """``opt_rigid_flow_kp`` (kp_selection.py:203-324) on a given rigid-flow inconsistency map [H,W] (device)."""
        quota = num_bestN // (rows * cols)
        cells = rows * cols
        r = self._rf_buffers(rows, cols, quota)
        st = self.rt.stream_ptr()
        u = r["u"]
        self.lib.check(self.lib.dfvo_uniform_cells(rigid_map_buf.ptr, flow_diff_buf.ptr, self.H, self.W, rows, cols, num_bestN, rigid_thre,
                                                   flow_thre, u["idx"].ptr, u["cc"].ptr, st))
        self.lib.check(self.lib.dfvo_gather_keypoints(u["idx"].ptr, u["cc"].ptr, cells, quota, flow_fwd_buf.ptr, self.H, self.W,
                                                      u["kp1"].ptr, u["kp2"].ptr, u["n"].ptr, st))
        out = dict(rigid_flow_diff=rigid_map_buf)
        if want_best:
            b = r["b"]
            if score_method == "rigid_flow":                      # score = rigid-flow inconsistency (kp_selection.py:266-269)
                args = (rigid_map_buf.ptr, flow_diff_buf.ptr, rigid_thre, flow_thre)
            else:
                args = (flow_diff_buf.ptr, rigid_map_buf.ptr, flow_thre, rigid_thre)
            self.lib.check(self.lib.dfvo_local_bestn(args[0], args[1], self.H, self.W, rows, cols, num_bestN, args[2], args[3],
                                                     b["idx"].ptr, b["cc"].ptr, r["st"].ptr, st))
            self.lib.check(self.lib.dfvo_gather_keypoints(b["idx"].ptr, b["cc"].ptr, cells, quota, flow_fwd_buf.ptr, self.H, self.W,
                                                          b["kp1"].ptr, b["kp2"].ptr, b["n"].ptr, st))
            nb = int(b["n"].numpy()[0])
            assert nb != 0, "sampling threshold is too small."       # kp_selection.py:298
            out["kp1_best"], out["kp2_best"] = b["kp1"].numpy()[:nb], b["kp2"].numpy()[:nb]
        nu = int(u["n"].numpy()[0])
        assert nu != 0, "sampling threshold is too small."          # kp_selection.py:306
        out["kp1_uniform"], out["kp2_uniform"] = u["kp1"].numpy()[:nu], u["kp2"].numpy()[:nu]
        return out

    # ------------------------------------------------------------------ pose
    def _subset_table(self, n, max_iters=1000):
        key = (n, max_iters)
        t = self._subsets.get(key)
        if t is None:
            host = np.zeros((max_iters, 5), np.int32)
            self.lib.check(self.lib.dfvo_cv_subset_stream_host(n, 5, max_iters, host.ctypes.data_as(ctypes.c_void_p)))
            while len(self._subsets) >= self._subsets_cap:          # recycle the least recently used table (no allocation)
                _, t = self._subsets.popitem(last=False)
                t = t.view((max_iters, 5)) if t.size >= max_iters * 5 else None
            t = t.upload(host) if t is not None else self.rt.from_host(host)
            self._subsets[key] = t
        else:
            self._subsets.move_to_end(key)
        return t

    def _capacity(self, n):
        """Keypoint capacity covering n: the configured one, doubled until it fits."""
        cap = self.kp_capacity
        while cap < n:
            cap *= 2
        return cap

    def essential_launch(self, kp_cur_buf, kp_ref_buf, n, perms, K, threshold=0.2, prob=0.99, max_iters=1000):
        """Enqueue R = len(perms) repeats of findEssentialMat(kp_cur[perm], kp_ref[perm]) + GRIC-E
        (E_tracker.py:223-286).  Returns a handle for :meth:`essential_result`."""
        cx, cy, fx, fy = K
        R = len(perms)
        key = (R, max_iters)
        c = self._ess_ws.get(key)
        if c is None or c["cap"] < n:
            cap = self._capacity(n)
            nb = int(self.lib.dfvo_essential_workspace_bytes(cap, R, max_iters))
            c = self._ess_ws[key] = dict(cap=cap, ws=self.rt.empty((nb,), np.uint8), E=self.rt.empty((R, 9), np.float64),
                                         mask_c=self.rt.empty((R * cap,), np.uint8), info=self.rt.empty((R, 4), np.int32),
                                         gric=self.rt.empty((R,), np.float64), perm_c=self.rt.empty((R * cap,), np.int32),
                                         Rt=self.rt.empty((12,), np.float64), pmask_c=self.rt.empty((cap,), np.uint8),
                                         pinfo=self.rt.empty((5,), np.int32))
        w = dict(c)
        w["mask"], w["perm"], w["pmask"] = c["mask_c"].view((R, n)), c["perm_c"].view((R, n)), c["pmask_c"].view((n,))
        w["perm"].upload(np.asarray(perms, np.int32))
        self.lib.check(self.lib.dfvo_essential_ransac(kp_cur_buf.ptr, kp_ref_buf.ptr, n, w["perm"].ptr, R,
                                                      self._subset_table(n, max_iters).ptr, max_iters, fx, fy, cx, cy, threshold,
                                                      prob, w["ws"].ptr, w["ws"].shape[0], w["E"].ptr, w["mask"].ptr,
                                                      w["info"].ptr, w["gric"].ptr, self.rt.stream_ptr()))
        return w

    TAIL_MAX_N = 4096

    def essential_tail(self, w, h, kp_cur_buf, kp_ref_buf, n, K, depth_buf, rng, min_samples=3, max_trials=100, stop_prob=0.99, thre=0.1):
        """Everything between the essential-matrix repeats and "pose and scale known" in one enqueue and ONE device->host read
        (dfvo_essential_tail): best repeat, recoverPose, the validity vote, the cheirality gate, the depth ratios and the scale
        regressor (with `rng`'s MT19937 state; the advanced state is installed back).  `h`: the homography handle for GRIC validity,
        or None for e_tracker.validity.method 'flow' (the caller took the flow gate before drawing the shuffles of `w`).
        `depth_buf` None: pose only (no scale recovery, `rng` untouched).  Returns a dict with R, t (identity / zero when the pose is
        rejected, as compute_pose_2d2d + resolve_validity give them), valid, cheirality, best, E_gric (flow: the per-repeat
        cheirality counts), H_gric (flow: 0), ransac_info, scale (-1 when not recovered), scale_status, and `w` for a lazy inlier
        mask.  = essential_tail_launch + essential_tail_finish; between the two `rng` must not be used (its state travels with the
        launch)."""
        return self.essential_tail_finish(self.essential_tail_launch(w, h, kp_cur_buf, kp_ref_buf, n, K, depth_buf, rng, min_samples,
                                                                     max_trials, stop_prob, thre))

    def essential_tail_launch(self, w, h, kp_cur_buf, kp_ref_buf, n, K, depth_buf, rng, min_samples=3, max_trials=100, stop_prob=0.99, thre=0.1):
        cx, cy, fx, fy = K
        R = w["info"].shape[0]
        cap = w["cap"]
        c = getattr(self, "_tail", None)
        if c is None or c["cap"] < cap or c["R"] != R:
            nb = int(self.lib.dfvo_essential_tail_workspace_bytes(cap))
            size = native.tail_result_doubles(R)
            c = self._tail = dict(cap=cap, R=R, ws=self.rt.empty((nb,), np.uint8), res=self.rt.empty((size,), np.float64),
                                  host=np.zeros(size, np.float64))
        st = _mt_state_in(rng, c["host"], "essential_tail")
        c["res"].upload(c["host"])
        gric = h_gric = None                                        # flow validity: no homography
        if h is not None:
            self.rt.wait_event(h["done"])                           # order this stream after the homography side stream
            gric, h_gric = w["gric"].ptr, h["gric"].ptr
        self.lib.check(self.lib.dfvo_essential_tail(w["E"].ptr, w["info"].ptr, gric, R, kp_cur_buf.ptr, kp_ref_buf.ptr, n, fx, fy, cx, cy,
                                                    h_gric, depth_buf.ptr if depth_buf is not None else None, self.H, self.W,
                                                    int(min_samples), int(max_trials), float(stop_prob), float(thre), c["ws"].ptr,
                                                    c["ws"].shape[0], c["res"].ptr, w["pmask"].ptr, w["pinfo"].ptr, self.rt.stream_ptr()))
        return dict(c=c, w=w, n=n, R=R, rng=rng, st=st)

    def essential_tail_finish(self, tok):
        c, w, n, R, rng, st = tok["c"], tok["w"], tok["n"], tok["R"], tok["rng"], tok["st"]
        o = c["res"].numpy()                                        # the one synchronising read
        _mt_state_out(rng, o, st)
        best, valid, cheir = int(o[native.DFVO_TAIL_BEST]), bool(o[native.DFVO_TAIL_VALID]), int(o[native.DFVO_TAIL_CHEIR])
        status, e0, rt0 = o[native.DFVO_TAIL_STATUS], native.DFVO_TAIL_EGRIC, native.DFVO_TAIL_RT
        out = dict(R=np.eye(3), t=np.zeros((3, 1)), valid=valid, cheirality=0, best=best, H_gric=float(o[native.DFVO_TAIL_HGRIC]),
                   E_gric=o[e0:e0 + R].copy(), ransac_info=o[e0 + R:e0 + 5 * R].reshape(R, 4).astype(np.int32), scale=-1,
                   scale_status=int(status), n_ratios=int(o[native.DFVO_TAIL_NVALID]), handle=w)
        if valid and best >= 0 and cheir > n * 0.1:
            out["R"], out["t"], out["cheirality"] = o[rt0:rt0 + 9].reshape(3, 3).copy(), o[rt0 + 9:rt0 + 12].reshape(3, 1).copy(), cheir
        if status == -1:
            raise ValueError("RANSAC could not find a valid consensus set")
        if status == 1:
            out["scale"] = float(o[native.DFVO_TAIL_SCALE])
        return out

    def pnp_tail_launch(self, kp_ref_buf, kp_cur_buf, n, depth_buf, K, min_depth, max_depth, rng, repeat=5, iters=100, reproj_thre=1.0,
                        prob=0.99):
        """``PnpTracker.compute_pose_3d2d`` (pnp_tracker.py:45-125) on device keypoints: dfvo_pnp_filter (in-image filter, reference depth
        at int(kp_ref), depth range, ordered compaction, unprojection), ONE read of the filtered count m, the host's `repeat` shuffles of
        arange(m) (drawn even when m <= 4, as the reference does), then dfvo_pnp_tail (the solvePnPRansac repeats and the best one).
        Finish with :meth:`pnp_tail_finish` (one packed read)."""
        cx, cy, fx, fy = K
        if not hasattr(self, "_pf") or self._pf["cap"] < n:
            cap = self._capacity(n)
            self._pf = dict(cap=cap, obj=self.rt.empty((cap * 3,), np.float64), img=self.rt.empty((cap * 2,), np.float64),
                            m=self.rt.empty((1,), np.int32))
        f = self._pf
        iK = np.ascontiguousarray(np.linalg.inv(np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1.0]])))    # as compute_pose_3d2d unprojects
        self.lib.check(self.lib.dfvo_pnp_filter(kp_ref_buf.ptr, kp_cur_buf.ptr, n, depth_buf.ptr, self.H, self.W, float(min_depth),
                                                float(max_depth), iK.ctypes.data_as(ctypes.c_void_p), f["obj"].ptr, f["img"].ptr,
                                                f["m"].ptr, self.rt.stream_ptr()))
        m = int(f["m"].numpy()[0])                                        # the one read before the solver
        perms = shuffles(rng, m, repeat)                                  # pnp_tracker.py:90-95
        if m <= 4:                                                        # pnp_tracker.py:97: no solver, identity
            return dict(m=m, res=None)
        key = (repeat, iters)
        c = self._pnp_ws.get(("tail",) + key)
        if c is None or c["cap"] < m:
            cap = self._capacity(m)
            nb = int(self.lib.dfvo_pnp_tail_workspace_bytes(cap, repeat, iters))
            c = self._pnp_ws[("tail",) + key] = dict(cap=cap, ws=self.rt.empty((nb,), np.uint8), perm_c=self.rt.empty((repeat * cap,), np.int32),
                                                     res=self.rt.empty((native.pnp_result_doubles(repeat),), np.float64))
        perm = c["perm_c"].view((repeat, m)).upload(np.asarray(perms, np.int32))
        self.lib.check(self.lib.dfvo_pnp_tail(f["obj"].ptr, f["img"].ptr, m, perm.ptr, repeat, self._subset_table(m, iters).ptr, iters,
                                              fx, fy, cx, cy, float(reproj_thre), prob, c["ws"].ptr, c["ws"].shape[0], c["res"].ptr,
                                              self.rt.stream_ptr()))
        return dict(m=m, res=c["res"])

    def pnp_tail_finish(self, tok):
        """-> (4x4 pose current -> reference, winning inlier count, filtered count).  The pose is assembled exactly as
        :func:`compute_pose_3d2d` does it (hostmath.rodrigues, np.linalg.inv), so both paths give the same bits."""
        pose = np.eye(4)
        best_inl = 0
        if tok["res"] is not None:
            o = tok["res"].numpy()                                        # the one packed read
            if o[native.DFVO_PNP_BEST] >= 0:
                best_inl = int(o[native.DFVO_PNP_INLIERS])
                pose[:3, :3] = hostmath.rodrigues(o[native.DFVO_PNP_RVEC:native.DFVO_PNP_RVEC + 3].copy())
                pose[:3, 3] = o[native.DFVO_PNP_TVEC:native.DFVO_PNP_TVEC + 3]
        return np.linalg.inv(pose), best_inl, tok["m"]

    def recover_pose(self, w, best, kp_cur_buf, kp_ref_buf, n, K):
        """cv2.recoverPose(best_E, kp_cur, kp_ref, focal=fx, pp) (E_tracker.py:292-295)."""
        cx, cy, fx, fy = K
        e_ptr = ctypes.c_void_p(w["E"].ptr.value + best * 9 * 8)
        self.lib.check(self.lib.dfvo_recover_pose(e_ptr, kp_cur_buf.ptr, kp_ref_buf.ptr, n, fx, cx, cy, w["Rt"].ptr,
                                                  w["pmask"].ptr, w["pinfo"].ptr, self.rt.stream_ptr()))
        return w["Rt"].numpy(), int(w["pinfo"].numpy()[0])

    def homography_launch(self, kp_cur_buf, kp_ref_buf, n, threshold=1.0, prob=0.99, max_iters=2000):
        """Enqueue cv2.findHomography(kp_cur, kp_ref, RANSAC, confidence, ransacReprojThreshold) + GRIC-H
        (E_tracker.py:199-215) on the device (csrc/homog.cu); returns the buffers (H [9], mask [n], info [4], gric [1])."""
        c = self._h_ws.get(max_iters)
        if c is None or c["cap"] < n:
            cap = self._capacity(n)
            nb = int(self.lib.dfvo_homography_workspace_bytes(cap, max_iters))
            c = self._h_ws[max_iters] = dict(cap=cap, ws=self.rt.empty((nb,), np.uint8), H=self.rt.empty((9,), np.float64),
                                             mask_c=self.rt.empty((cap,), np.uint8), info=self.rt.empty((4,), np.int32),
                                             gric=self.rt.empty((1,), np.float64))
        w = dict(c)
        w["mask"] = c["mask_c"].view((n,))
        # forked onto a side stream so it runs beside the essential-matrix RANSAC (both are short chains of small kernels);
        # whoever reads the result waits on w["done"] first (resolve_validity)
        if not hasattr(self, "_h_stream"):
            self._h_stream = self.rt.new_stream(high_priority=True)
        fork = self.rt.record_event()
        with self.rt.on_stream(self._h_stream):
            self.rt.wait_event(fork)
            self.lib.check(self.lib.dfvo_homography_ransac(kp_cur_buf.ptr, kp_ref_buf.ptr, n, max_iters, float(threshold), prob, w["ws"].ptr,
                                                           w["ws"].shape[0], w["H"].ptr, w["mask"].ptr, w["info"].ptr, w["gric"].ptr,
                                                           self.rt.stream_ptr()))
            w["done"] = self.rt.record_event()
        w["rt"] = self.rt
        return w

    def pnp_ransac(self, XYZ, kp2, perms, K, iters=100, reproj_thre=1.0, prob=0.99):
        """len(perms) repeats of cv2.solvePnPRansac(XYZ[perm], kp2[perm], K, None, iterationsCount=iters,
        reprojectionError=reproj_thre) on the device (pnp_tracker.py:86-112; csrc/pnp.cu).  XYZ [n,3], kp2 [n,2] float64
        host arrays.  Returns (rt [R,6] = rvec|tvec, info [R,4] = found, inliers, iterations, winning iteration)."""
        cx, cy, fx, fy = K
        n, R = XYZ.shape[0], len(perms)
        key = (R, iters)
        c = self._pnp_ws.get(key)
        if c is None or c["cap"] < n:
            cap = self._capacity(n)
            nb = int(self.lib.dfvo_pnp_workspace_bytes(cap, R, iters))
            c = self._pnp_ws[key] = dict(cap=cap, ws=self.rt.empty((nb,), np.uint8), obj_c=self.rt.empty((cap * 3,), np.float64),
                                         img_c=self.rt.empty((cap * 2,), np.float64), perm_c=self.rt.empty((R * cap,), np.int32),
                                         rt=self.rt.empty((R, 6), np.float64), info=self.rt.empty((R, 4), np.int32))
        w = dict(c)
        w["obj"], w["img"], w["perm"] = c["obj_c"].view((n, 3)), c["img_c"].view((n, 2)), c["perm_c"].view((R, n))
        w["obj"].upload(XYZ); w["img"].upload(kp2); w["perm"].upload(np.asarray(perms, np.int32))
        self.lib.check(self.lib.dfvo_pnp_ransac(w["obj"].ptr, w["img"].ptr, n, w["perm"].ptr, R, self._subset_table(n, iters).ptr,
                                                iters, fx, fy, cx, cy, float(reproj_thre), prob, w["ws"].ptr, w["ws"].shape[0],
                                                w["rt"].ptr, w["info"].ptr, self.rt.stream_ptr()))
        return w["rt"].numpy(), w["info"].numpy()

    def ransac_scale(self, ratio, min_samples=3, max_trials=100, stop_prob=0.99, thre=0.1, rng=np.random):
        """The scale fit of find_scale_from_depth (E_tracker.py:618-641, sklearn RANSACRegressor through the origin) on the device
        (csrc/ransac.cu::k_scale_ransac).  The regressor samples from NumPy's global generator; the kernel receives that generator's
        MT19937 state, draws exactly what scikit-learn would draw, and the advanced state is installed back into ``rng`` -- the
        shuffles of the next frame continue from the same position as in the reference.  Raises ValueError like sklearn when no
        consensus set exists."""
        ratio = np.ascontiguousarray(ratio, np.float64).reshape(-1)
        n = ratio.shape[0]
        io_h = np.zeros(native.DFVO_TAIL_SCALE_IO, np.float64)
        st = _mt_state_in(rng, io_h, "ransac_scale")
        cap = self._capacity(n)
        if not hasattr(self, "_sr") or self._sr["x"].size < cap:
            self._sr = dict(x=self.rt.empty((cap,), np.float64), io=self.rt.empty((native.DFVO_TAIL_SCALE_IO,), np.float64),
                            perm=self.rt.empty((cap,), np.int32))
        w = self._sr
        w["x"].view((n,)).upload(ratio)
        w["io"].upload(io_h)
        self.lib.check(self.lib.dfvo_scale_ransac(w["x"].ptr, n, int(min_samples), int(max_trials), float(stop_prob), float(thre), w["io"].ptr,
                                                  w["perm"].ptr, self.rt.stream_ptr()))
        out = w["io"].numpy()
        _mt_state_out(rng, out, st)
        if out[native.DFVO_TAIL_STATUS] < 0:
            raise ValueError("RANSAC could not find a valid consensus set")
        return float(out[native.DFVO_TAIL_SCALE])

    def triangulate_depth(self, kp1n_buf, kp2n_buf, n, T21):
        if not hasattr(self, "_tri") or self._tri["z"].shape[0] < n:
            self._tri = dict(z=self.rt.empty((max(n, 2048),), np.float64), T=self.rt.empty((12,), np.float64))
        t = self._tri
        t["T"].upload(np.asarray(T21, np.float64)[:3].reshape(-1))
        self.lib.check(self.lib.dfvo_triangulate_depth(kp1n_buf.ptr, kp2n_buf.ptr, n, t["T"].ptr, t["z"].ptr, self.rt.stream_ptr()))
        return t["z"].numpy()[:n]


# ---------------------------------------------------------------------------------------------
# host-level orchestration of the E-tracker (E_tracker.py:154-307)
# ---------------------------------------------------------------------------------------------
def compute_pose_2d2d(engine, kp_ref, kp_cur, K, repeat=5, reproj_thre=0.2, rng=np.random, kp_ref_buf=None, kp_cur_buf=None,
                      defer_validity=False, validity="GRIC", flow_thre=None):
    """Same contract as ``EssTracker.compute_pose_2d2d`` with the GRIC validity check, or (validity='flow') the flow-magnitude
    check with threshold `flow_thre`.
    kp_ref/kp_cur: float64 [N,2] host arrays (device copies optional).  Everything numeric runs on the device: the
    homography model + GRIC-H (csrc/homog.cu), the five essential-matrix RANSAC repeats + GRIC-E (ransac.cu) and
    recoverPose; the host draws the shuffles, takes the majority vote and the cheirality decision.
    Returns dict(R, t, inliers, valid, cheirality).

    GRIC, defer_validity=True: R, t are the pose *as if* the E-model is valid and the caller must call
    :func:`resolve_validity` (which resets them to identity / zero when GRIC prefers the homography) before using them
    for a decision; lets a caller issue pose-dependent device work before it reads the vote.  Results are identical.

    flow (E_tracker.py:182-186,249-257,289-300): the gate mean |kp_ref - kp_cur| > thre is NumPy's own expression on the host
    arrays; a closed gate draws no shuffle and leaves the pose at identity.  Otherwise the repeats, the per-repeat recoverPose
    counts, the flow-mode best-E rule, the vote and the final recoverPose run on the device (essential_ransac + the essential tail
    without scale recovery) and are read once."""
    n = kp_ref.shape[0]
    R, t = np.eye(3), np.zeros((3, 1))
    out = dict(R=R, t=t, inliers=np.ones(n, bool), valid=False, cheirality=0)
    if validity == "flow":
        out["flow_mean"] = np.mean(np.linalg.norm(kp_ref - kp_cur, axis=1))
        if not out["flow_mean"] > flow_thre:
            return out
    elif n <= 10:                                                   # E_tracker.py:196,216-217
        return out
    perms = shuffles(rng, n, repeat)                                # host RNG consumption identical to the reference
    rt = engine.rt
    kp_cur_buf = kp_cur_buf or rt.from_host(kp_cur)
    kp_ref_buf = kp_ref_buf or rt.from_host(kp_ref)
    if validity == "flow":
        w = engine.essential_launch(kp_cur_buf, kp_ref_buf, n, perms, K, threshold=reproj_thre)
        o = engine.essential_tail(w, None, kp_cur_buf, kp_ref_buf, n, K, None, rng)
        out.update(valid=o["valid"], cheirality=o["cheirality"], R=o["R"], t=o["t"], ransac_info=o["ransac_info"],
                   cheirality_counts=o["E_gric"])
        if o["best"] >= 0:
            out["inliers"] = w["mask"].numpy()[o["best"]].astype(bool)
        return out
    h = engine.homography_launch(kp_cur_buf, kp_ref_buf, n)         # homography model (E_tracker.py:199-215)
    w = engine.essential_launch(kp_cur_buf, kp_ref_buf, n, perms, K, threshold=reproj_thre)
    info = w["info"].numpy()
    gric = w["gric"].numpy()
    best, best_cnt = -1, 0
    for r in range(repeat):
        if info[r, 0] > best_cnt:                                   # strict '>' keeps the first maximum (:278-281)
            best, best_cnt = r, int(info[r, 0])
    out["E_gric"], out["ransac_info"] = gric, info
    if best >= 0:
        out["inliers"] = w["mask"].numpy()[best].astype(bool)
        # recoverPose before the validity vote is read (a wasted ~30 us of device time when the vote fails)
        Rt, cheir = engine.recover_pose(w, best, kp_cur_buf, kp_ref_buf, n, K)
        out["cheirality"] = cheir
        if cheir > n * 0.1:                                         # :299-300
            out["R"], out["t"] = Rt[:9].reshape(3, 3).copy(), Rt[9:].reshape(3, 1).copy()
    out["_vote"] = (h, gric, repeat, best)
    if not defer_validity:
        resolve_validity(out)
    return out


def resolve_validity(out):
    """Read GRIC-H and apply the majority vote H_gric > E_gric (E_tracker.py:270,286-290)."""
    vote = out.pop("_vote", None)
    if vote is None:
        return out
    h, gric, repeat, best = vote
    h["rt"].wait_event(h["done"])                                   # join the homography side stream
    H_gric = float(h["gric"].numpy()[0])
    num_valid = sum(int(H_gric > gric[r]) for r in range(repeat))
    out["valid"] = num_valid > repeat / 2
    out["H_gric"] = H_gric
    if not (out["valid"] and best >= 0):
        out["R"], out["t"], out["cheirality"] = np.eye(3), np.zeros((3, 1)), 0
    return out


def compute_pose_3d2d(engine, kp1, kp2, d, K, repeat=5, iters=100, reproj_thre=1.0, rng=np.random):
    """The solver part of ``PnpTracker.compute_pose_3d2d`` (pnp_tracker.py:80-118) for keypoints already filtered by the
    caller: kp1 [n,2] reference pixels with depths d [n], kp2 [n,2] current pixels.  Unprojection (ops_3d.py:70-94),
    one host shuffle per repeat (same RNG consumption as the reference), the RANSACs + refits on the device, best
    repeat by inlier count (strict '>', first maximum).  Returns the 4x4 pose current -> reference (the inverse of
    solvePnP's, pnp_tracker.py:113-118) and the winning inlier count."""
    cx, cy, fx, fy = K
    n = kp1.shape[0]
    Kmat = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1.0]])
    XYZ = (np.linalg.inv(Kmat) @ np.concatenate([kp1, np.ones((n, 1))], 1).T).T * np.asarray(d, np.float64)[:, None]
    perms = shuffles(rng, n, repeat)
    pose = np.eye(4)
    best_inl = 0
    if n > 4:                                                       # pnp_tracker.py:97
        rt, info = engine.pnp_ransac(XYZ, np.ascontiguousarray(kp2, np.float64), perms, K, iters, reproj_thre)
        best = -1
        for r in range(repeat):
            if info[r, 0] and info[r, 1] > best_inl:
                best, best_inl = r, int(info[r, 1])
        if best >= 0:
            pose[:3, :3] = hostmath.rodrigues(rt[best, :3])
            pose[:3, 3] = rt[best, 3:]
    return np.linalg.inv(pose), best_inl


def find_scale_from_depth(engine, kp1, kp2, T_21, depth2, K, min_samples=3, max_trials=100, stop_prob=0.99, thre=0.1,
                          rng=np.random):
    """``EssTracker.find_scale_from_depth`` (E_tracker.py:571-643): triangulation on the device, the
    scale RANSAC (which consumes the host generator's stream) on the device too (Engine.ransac_scale)."""
    cx, cy, fx, fy = K
    n = kp1.shape[0]
    k1 = (kp1 - np.array([cx, cy])) / np.array([fx, fy])
    k2 = (kp2 - np.array([cx, cy])) / np.array([fx, fy])
    z = engine.triangulate_depth(engine.rt.from_host(k1), engine.rt.from_host(k2), n, T_21)
    ratio, nvalid = hostmath.last_writer_depth_ratio(kp2, z, depth2)
    if nvalid > 10:
        return engine.ransac_scale(ratio, min_samples, max_trials, stop_prob, thre, rng)
    return -1


def scale_recovery_iterative(select, find_scale, E_pose, prev_scale, kp_best, kp_src="kp_best", score_method="rigid_flow"):
    """``EssTracker.scale_recovery_iterative`` (E_tracker.py:509-569).  ``select(T, score_method)`` = the rigid-flow keypoint
    selection under pose T (Engine.rigid_flow_keypoints bound to the frame's buffers), ``find_scale(kp_ref, kp_cur)`` =
    find_scale_from_depth on the frame, ``kp_best`` = (kp_ref, kp_cur) of the best-N selection.  Up to five rounds; stops when
    the scale moves by less than 0.001.  Returns dict(scale, cur_kp, ref_kp, rigid_flow_mask) -- the last round's."""
    scale, delta = prev_scale, 0.001
    out = {}
    for _ in range(5):
        P = np.array(E_pose, np.float64)
        P[:3, 3] = P[:3, 3] * scale                               # rigid_flow_pose.t *= scale (:535)
        sel = select(np.linalg.inv(P), score_method)              # ref_data['rigid_flow_pose'] = SE3(inv) (:537)
        ref_kp, cur_kp = (sel["kp1_uniform"], sel["kp2_uniform"]) if kp_src == "kp_depth" else kp_best
        new_scale = find_scale(ref_kp, cur_kp)
        d = abs(new_scale - scale)
        scale = new_scale
        out = dict(scale=scale, cur_kp=sel["kp2_uniform"], ref_kp=sel["kp1_uniform"], rigid_flow_mask=sel["rigid_flow_diff"])
        if d < delta:
            break
    return out


# ---------------------------------------------------------------------------------------------
# process-wide default engine (the libs mirror's DeepModel / trackers share one dfvo_ctx)
# ---------------------------------------------------------------------------------------------
_default_engine = None


def default_engine(height=None, width=None):
    global _default_engine
    if _default_engine is None or (height is not None and (_default_engine.H, _default_engine.W) != (height, width)):
        if height is None:
            raise native.DfvoError("no dfvo_b200 engine yet: construct libs.deep_models.DeepModel (or tracking.Engine) first")
        _default_engine = Engine(height, width)
    return _default_engine


class DevArray:
    """A device-resident array that behaves enough like ``numpy.ndarray`` for the reference driver
    (``.copy()``, ``.shape``, indexing, ``np.asarray``) while the hot path keeps using ``.dev``.
    Host materialisation happens lazily, once, and only if somebody (e.g. the visualiser) asks."""

    def __init__(self, dev, shape=None, view=None):
        self.dev = dev
        self.shape = tuple(shape if shape is not None else dev.shape)
        self.dtype = dev.dtype
        self.ndim = len(self.shape)
        self._view = view            # optional callable applied to the host copy (e.g. reshape)
        self._host = None

    def copy(self):
        """A snapshot, like ``ndarray.copy()``: the engine reuses its flow / mask buffers every frame, and the driver keeps
        copies across frames (dfvo.py:329-332; ``update_data`` moves ``fb_flow_mask`` / ``rigid_flow_mask`` into ``ref_data``).
        If the host copy already exists it is the snapshot; else a device-side clone (ordered after the producer kernel)."""
        if self._host is not None:
            c = DevArray(self.dev, self.shape, self._view)
            c._host = self._host.copy()
            return c
        return DevArray(self.dev.clone(), self.shape, self._view)

    def __array__(self, dtype=None, copy=None):
        if self._host is None:
            h = self.dev.numpy()
            self._host = (self._view(h) if self._view else h).reshape(self.shape)
        return self._host if dtype is None else self._host.astype(dtype)

    def __getitem__(self, k):
        return np.asarray(self)[k]

    def __len__(self):
        return self.shape[0]
