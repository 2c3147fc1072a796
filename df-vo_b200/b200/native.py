"""ctypes binding of the C ABI declared in ``include/dfvo_b200.h``.

The product entry point is :func:`load`: it loads the nvcc-built ``libdfvo_b200.so`` (building it
in-tree first if the sources are newer) and **fails loudly** when the library is missing, is not
a device build, or no CUDA device is visible.  There is no CPU fallback.

``Lib`` itself only describes the ABI; the CPU test-suite instantiates it on the host-emulation
build (``tests/hostsim``) to exercise the same entry points with host memory.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.normpath(os.path.join(_HERE, "..", "csrc"))
LIB_PATH = os.path.join(CSRC, "libdfvo_b200.so")

PREC_FP32, PREC_BF16, PREC_TF32 = 0, 1, 2
PREC_NAMES = {"fp32": PREC_FP32, "bf16": PREC_BF16, "tf32": PREC_TF32}
NET_LITEFLOWNET, NET_MONODEPTH2, NET_POSENET = 0, 1, 2
ACT_NONE, ACT_LEAKY, ACT_RELU, ACT_ELU, ACT_SIGMOID = 0, 1, 2, 3, 4

# offsets (in doubles) of the packed results of dfvo_essential_tail / dfvo_scale_ransac and dfvo_pnp_tail (the DFVO_TAIL_* and
# DFVO_PNP_* enums of include/dfvo_b200.h)
DFVO_TAIL_SCALE, DFVO_TAIL_STATUS, DFVO_TAIL_TRIALS, DFVO_TAIL_INLIERS = 0, 1, 2, 3
DFVO_TAIL_MT, DFVO_TAIL_MT_DOUBLES, DFVO_TAIL_SCALE_IO = 4, 313, 317
DFVO_TAIL_BEST, DFVO_TAIL_VALID, DFVO_TAIL_HGRIC, DFVO_TAIL_CHEIR, DFVO_TAIL_NVALID, DFVO_TAIL_GATE = 317, 318, 319, 320, 321, 322
DFVO_TAIL_RT, DFVO_TAIL_EGRIC = 323, 335
DFVO_PNP_BEST, DFVO_PNP_INLIERS, DFVO_PNP_RVEC, DFVO_PNP_TVEC, DFVO_PNP_INFO = 0, 1, 2, 5, 8


def tail_result_doubles(R):
    """Length of dfvo_essential_tail's res for R repeats."""
    return DFVO_TAIL_EGRIC + 5 * R


def pnp_result_doubles(R):
    """Length of dfvo_pnp_tail's res for R repeats."""
    return DFVO_PNP_INFO + 4 * R

c_int, c_void_p, c_char_p, c_float, c_double = (ctypes.c_int, ctypes.c_void_p, ctypes.c_char_p,
                                               ctypes.c_float, ctypes.c_double)
c_size_t = ctypes.c_size_t

# name -> (restype, argtypes); one row per symbol of include/dfvo_b200.h
SIGNATURES = {
    "dfvo_last_error": (c_char_p, []),
    "dfvo_version": (c_char_p, []),
    "dfvo_is_device_build": (c_int, []),
    "dfvo_launch_count": (ctypes.c_longlong, []),
    "dfvo_set_conv_chain": (c_int, [c_int]),
    "dfvo_profile_enable": (None, [c_int]),
    "dfvo_profile_read": (None, [ctypes.POINTER(c_double), ctypes.POINTER(ctypes.c_longlong), ctypes.POINTER(c_double)]),
    "dfvo_create": (c_int, [ctypes.POINTER(c_void_p), c_int]),
    "dfvo_destroy": (c_int, [c_void_p]),
    "dfvo_load_weight": (c_int, [c_void_p, c_int, c_char_p, c_void_p, ctypes.POINTER(ctypes.c_int64), c_int]),
    "dfvo_liteflow_build": (c_int, [c_void_p, c_int, c_int, c_int, c_int]),
    "dfvo_liteflow_forward": (c_int, [c_void_p, ctypes.POINTER(c_void_p), c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "dfvo_liteflow_level_flow": (c_int, [c_void_p, c_int, c_void_p]),
    "dfvo_liteflow_geometry": (c_int, [c_void_p, ctypes.POINTER(c_int), ctypes.POINTER(c_int), ctypes.POINTER(c_int)]),
    "dfvo_correlation": (c_int, [c_void_p, c_void_p, c_void_p] + [c_int] * 7 + [c_void_p]),
    "dfvo_correlation_nhwc_bf16": (c_int, [c_void_p, c_void_p, c_void_p] + [c_int] * 8 + [c_void_p]),
    "dfvo_backproject": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "dfvo_transform3d": (c_int, [c_void_p, ctypes.c_longlong, c_void_p, c_void_p, c_void_p]),
    "dfvo_project": (c_int, [c_void_p, c_int, c_int, c_void_p, c_float, c_int, c_void_p, c_void_p]),
    "dfvo_reproject": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_float, c_int, c_void_p, c_void_p]),
    "dfvo_rigid_flow": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "dfvo_backward_warp": (c_int, [c_void_p, c_void_p, c_void_p] + [c_int] * 5 + [c_void_p]),
    "dfvo_fb_consistency": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "dfvo_fb_consistency_batch": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "dfvo_conv2d": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p] + [c_int] * 13 + [c_void_p]),
    "dfvo_local_bestn": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_float,
                                 c_void_p, c_void_p, c_void_p, c_void_p]),
    "dfvo_rigid_flow_diff": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_double, c_double, c_double, c_double, c_void_p, c_void_p]),
    "dfvo_uniform_cells": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_float, c_void_p, c_void_p, c_void_p]),
    "dfvo_bestn_workspace_bytes": (c_size_t, [c_int, c_int]),
    "dfvo_bestn": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    "dfvo_gather_keypoints": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p,
                                      c_void_p, c_void_p]),
    "dfvo_monodepth2_build": (c_int, [c_void_p, c_int, c_int, c_int, c_float, c_float, c_float]),
    "dfvo_monodepth2_forward": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p]),
    "dfvo_posenet_build": (c_int, [c_void_p, c_int, c_int, c_int, c_float]),
    "dfvo_posenet_forward": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "dfvo_depth_consistency": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "dfvo_lanczos_resize_u8": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int,
                                       c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "dfvo_depth_post": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_double, c_double, c_double, c_double, c_float, c_float,
                                c_void_p, c_void_p, c_void_p]),
    "dfvo_gather_depth": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p]),
    "dfvo_five_point": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "dfvo_score_hypotheses": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_double, c_void_p, c_void_p]),
    "dfvo_essential_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "dfvo_essential_ransac": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_double, c_double,
                                      c_double, c_double, c_double, c_double, c_void_p, c_size_t, c_void_p, c_void_p,
                                      c_void_p, c_void_p, c_void_p]),
    "dfvo_homography_workspace_bytes": (c_size_t, [c_int, c_int]),
    "dfvo_homography_ransac": (c_int, [c_void_p, c_void_p, c_int, c_int, c_double, c_double, c_void_p, c_size_t, c_void_p, c_void_p,
                                       c_void_p, c_void_p, c_void_p]),
    "dfvo_pnp_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "dfvo_pnp_ransac": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_double, c_double, c_double,
                                c_double, c_double, c_double, c_void_p, c_size_t, c_void_p, c_void_p, c_void_p]),
    "dfvo_scale_ransac": (c_int, [c_void_p, c_int, c_int, c_int, c_double, c_double, c_void_p, c_void_p, c_void_p]),
    "dfvo_essential_tail_workspace_bytes": (c_size_t, [c_int]),
    "dfvo_essential_tail": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_double, c_double, c_double, c_double,
                                    c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_double, c_double, c_void_p, c_size_t, c_void_p, c_void_p,
                                    c_void_p, c_void_p]),
    "dfvo_flow_mean": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "dfvo_pnp_filter": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_double, c_double, c_void_p, c_void_p, c_void_p,
                                c_void_p, c_void_p]),
    "dfvo_pnp_tail_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "dfvo_pnp_tail": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_double, c_double, c_double, c_double,
                              c_double, c_double, c_void_p, c_size_t, c_void_p, c_void_p]),
    "dfvo_epnp_minimal": (c_int, [c_void_p, c_void_p, c_int, c_double, c_double, c_double, c_double, c_int, c_void_p, c_void_p, c_void_p]),
    "dfvo_cv_subset_stream_host": (c_int, [c_int, c_int, c_int, c_void_p]),
    "dfvo_triangulate_depth": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "dfvo_triangulate_points": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "dfvo_recover_pose": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_double, c_double, c_double, c_void_p, c_void_p,
                                  c_void_p, c_void_p]),
}


class DfvoError(RuntimeError):
    pass


class Lib:
    """Thin typed wrapper around one loaded shared library."""

    def __init__(self, path):
        if not os.path.exists(path):
            raise DfvoError("dfvo_b200 native library not found: %s" % path)
        self.path = path
        self.cdll = ctypes.CDLL(path)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(self.cdll, name)            # AttributeError if the symbol is missing
            fn.restype = res
            fn.argtypes = args

    def check(self, rc):
        if rc != 0:
            msg = self.cdll.dfvo_last_error()
            raise DfvoError("dfvo_b200 error %d: %s" % (rc, msg.decode() if msg else "?"))

    def __getattr__(self, name):
        return getattr(self.cdll, name)


class Context:
    """RAII handle (``dfvo_ctx``) plus convenience wrappers.  ``ptr(x)`` must return the raw
    address of array-like ``x`` in the memory space the library computes in (torch CUDA tensors
    for the product, numpy arrays for the host-emulation test build)."""

    def __init__(self, lib, device=0):
        self.lib = lib
        self.h = c_void_p()
        lib.check(lib.dfvo_create(ctypes.byref(self.h), device))

    def close(self):
        if self.h:
            self.lib.dfvo_destroy(self.h)
            self.h = c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def load_weights(self, net, weights):
        """weights: {reference state-dict key: float32 numpy array (host)}"""
        import numpy as np
        for k, v in weights.items():
            if not hasattr(v, "shape"):
                continue                      # e.g. encoder.pth's 'height' / 'width' entries
            a = np.ascontiguousarray(v, dtype=np.float32)
            shape = (ctypes.c_int64 * max(a.ndim, 1))(*a.shape)
            self.lib.check(self.lib.dfvo_load_weight(self.h, net, k.encode(), a.ctypes.data_as(c_void_p),
                                                     shape, a.ndim))

    def liteflow_build(self, height, width, pairs=1, precision=PREC_BF16):
        self.lib.check(self.lib.dfvo_liteflow_build(self.h, height, width, pairs, precision))

    def monodepth2_build(self, feed_h, feed_w, precision=PREC_BF16, min_depth=0.1, max_depth=100.0, baseline=5.4):
        self.lib.check(self.lib.dfvo_monodepth2_build(self.h, feed_h, feed_w, precision, min_depth, max_depth, baseline))

    def monodepth2_forward(self, img, depth_out, stream=0):
        self.lib.check(self.lib.dfvo_monodepth2_forward(self.h, img, depth_out, stream))

    def posenet_build(self, feed_h, feed_w, precision=PREC_BF16, baseline_multiplier=5.4):
        self.lib.check(self.lib.dfvo_posenet_build(self.h, feed_h, feed_w, precision, baseline_multiplier))

    def posenet_forward(self, feed_ref, feed_cur, pose_out, stream=0):
        self.lib.check(self.lib.dfvo_posenet_forward(self.h, feed_ref, feed_cur, pose_out, stream))

    def liteflow_geometry(self):
        a, b, c = c_int(), c_int(), c_int()
        self.lib.check(self.lib.dfvo_liteflow_geometry(self.h, ctypes.byref(a), ctypes.byref(b), ctypes.byref(c)))
        return a.value, b.value, c.value

    def liteflow_forward(self, img_ptrs, flow_fwd, flow_bwd, flow_diff, stream=0):
        arr = (c_void_p * len(img_ptrs))(*img_ptrs)
        self.lib.check(self.lib.dfvo_liteflow_forward(self.h, arr, len(img_ptrs), flow_fwd, flow_bwd, flow_diff, stream))


_lib = None


def load(build_if_needed=True):
    """Load the device library or raise.  Never returns a CPU implementation."""
    global _lib
    if _lib is not None:
        return _lib
    if build_if_needed and not os.path.exists(LIB_PATH):
        import importlib.util
        spec = importlib.util.spec_from_file_location("_dfvo_build", os.path.join(CSRC, "build.py"))
        m = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(m)
        m.build()
    lib = Lib(LIB_PATH)
    if lib.dfvo_is_device_build() != 1:
        raise DfvoError("%s is not a device (nvcc, sm_90a) build" % LIB_PATH)
    _lib = lib
    return lib


def require_cuda():
    import torch
    if not torch.cuda.is_available():
        raise DfvoError("dfvo_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
