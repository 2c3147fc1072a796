"""Import shims that let the UNMODIFIED reference (a DF-VO checkout named by ``DFVO_REFERENCE_ROOT``) run on a
CPU-only machine with current library versions.  Used only by ``oracle/gen_golden.py`` (golden-vector generation)
and ``oracle/ref_corr_emul.py`` -- never at test or bench time.

Each shim corresponds to one row of SURVEY.md Appendix B:

  * ``cupy``, ``easydict``, ``matplotlib``, ``colour_demosaicing``, ``g2o`` are absent -> stubs
  * ``np.int`` was removed in NumPy 1.24                                   -> ``np.int = int``
  * sklearn ``RANSACRegressor(base_estimator=...)`` was renamed            -> kwarg adapter
  * ``grid_sample`` default ``align_corners`` flipped in torch 1.3; the reference was written
    for torch 1.1 (= ``align_corners=True``)                               -> explicit True
  * ``.cuda()`` / ``torch.device('cuda')`` without a GPU                    -> identity / cpu
  * ``correlation.FunctionCorrelation`` has no CPU path (correlation.py:335-336)
                                                                           -> oracle restatement
"""
import importlib
import os
import sys
import types

import numpy as np
import torch

REFERENCE_ROOT = os.environ.get("DFVO_REFERENCE_ROOT", "")
ALIGN_CORNERS_PINNED = True  # torch-1.1 semantics the reference was written for (SURVEY H3)

_installed = False


class _EasyDict(dict):
    """Minimal attribute-dict standing in for the absent ``easydict`` package."""

    def __init__(self, d=None, **kw):
        super().__init__()
        d = dict(d or {}, **kw)
        for k, v in d.items():
            self[k] = v

    @classmethod
    def _wrap(cls, v):
        if isinstance(v, dict) and not isinstance(v, cls):
            return cls(v)
        if isinstance(v, (list, tuple)):
            return type(v)(cls._wrap(x) for x in v)
        return v

    def __setitem__(self, k, v):
        super().__setitem__(k, self._wrap(v))

    def __setattr__(self, k, v):
        self[k] = v

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k)


def _stub(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


class _AnyAttr(types.ModuleType):
    """Stub package: any attribute access yields a no-op callable (only visualisation and
    dataset-IO code touches these modules; none of it runs during golden generation)."""
    __path__ = []

    def __getattr__(self, k):
        if k.startswith("__"):
            raise AttributeError(k)
        return lambda *a, **kw: None


def _install_stub_finder(prefixes):
    import importlib.abc
    import importlib.machinery

    class Finder(importlib.abc.MetaPathFinder, importlib.abc.Loader):
        def find_spec(self, name, path=None, target=None):
            if name.split(".")[0] in prefixes:
                return importlib.machinery.ModuleSpec(name, self, is_package=True)
            return None

        def create_module(self, spec):
            return _AnyAttr(spec.name)

        def exec_module(self, module):
            pass

    sys.meta_path.insert(0, Finder())


def install():
    """Install all shims and put the reference on ``sys.path``.  Idempotent."""
    global _installed
    if _installed:
        return
    _installed = True

    # --- absent third-party modules --------------------------------------------------
    cupy = _stub("cupy")
    cupy.util = types.SimpleNamespace(memoize=lambda **kw: (lambda f: f))
    cupy.cuda = types.SimpleNamespace(compile_with_cache=None)
    _stub("easydict", EasyDict=_EasyDict)
    _install_stub_finder(("matplotlib", "colour_demosaicing", "g2o"))

    # --- numpy / sklearn API drift -----------------------------------------------------
    if not hasattr(np, "int"):
        np.int = int
    from sklearn import linear_model

    _RR = linear_model.RANSACRegressor
    if not getattr(_RR, "_dfvo_shim", False):
        class _RRShim(_RR):
            _dfvo_shim = True

            def __init__(self, base_estimator=None, **kw):
                if base_estimator is not None:
                    kw["estimator"] = base_estimator
                super().__init__(**kw)

            @classmethod
            def _get_param_names(cls):
                return _RR._get_param_names()

        linear_model.RANSACRegressor = _RRShim

    # --- CUDA-less torch -----------------------------------------------------------------
    if not torch.cuda.is_available():
        torch.Tensor.cuda = lambda self, *a, **k: self
        torch.nn.Module.cuda = lambda self, *a, **k: self
        _to_t, _to_m = torch.Tensor.to, torch.nn.Module.to

        def _cpuify(args, kw):
            def fix(x):
                if isinstance(x, torch.device) and x.type == "cuda":
                    return torch.device("cpu")
                if isinstance(x, str) and x.startswith("cuda"):
                    return "cpu"
                return x
            return tuple(fix(a) for a in args), {k: fix(v) for k, v in kw.items()}

        def t_to(self, *a, **k):
            a, k = _cpuify(a, k)
            return _to_t(self, *a, **k)

        def m_to(self, *a, **k):
            a, k = _cpuify(a, k)
            return _to_m(self, *a, **k)

        torch.Tensor.to = t_to
        torch.nn.Module.to = m_to
        _load = torch.load

        def load(f, *a, **k):
            k["map_location"] = "cpu"
            k.setdefault("weights_only", False)
            return _load(f, **k)

        torch.load = load
        # correlation.py:7-9 reads the current CUDA stream at import time
        torch.cuda.current_stream = lambda *a, **k: types.SimpleNamespace(cuda_stream=0)

    # --- grid_sample: make the torch-1.1 default explicit ---------------------------------
    import torch.nn.functional as F

    if not getattr(F.grid_sample, "_dfvo_shim", False):
        _gs = F.grid_sample

        def grid_sample(input, grid, mode="bilinear", padding_mode="zeros", align_corners=None):
            if align_corners is None:
                align_corners = ALIGN_CORNERS_PINNED
            return _gs(input, grid, mode=mode, padding_mode=padding_mode,
                       align_corners=align_corners)

        grid_sample._dfvo_shim = True
        F.grid_sample = grid_sample
        torch.nn.functional.grid_sample = grid_sample

    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)


def import_reference(module):
    """Import ``module`` (e.g. ``libs.tracker.E_tracker``) from the reference tree."""
    install()
    # the product ships its own ``libs`` package; make sure the reference one wins here
    for k in [k for k in sys.modules if k == "libs" or k.startswith("libs.")]:
        m = sys.modules[k]
        f = getattr(m, "__file__", "") or ""
        if not f.startswith(REFERENCE_ROOT):
            del sys.modules[k]
    return importlib.import_module(module)


def patch_reference_correlation(fn):
    """Give the reference LiteFlowNet a CPU correlation (it has none).  ``fn(first, second,
    stride)`` is the oracle restatement, itself pinned against an emulation of the reference
    CUDA kernel text (``oracle/ref_corr_emul.py``)."""
    corr = import_reference("libs.deep_models.flow.lite_flow_net.correlation")
    corr.FunctionCorrelation = lambda tensorFirst, tensorSecond, intStride: fn(
        tensorFirst, tensorSecond, intStride)
    return corr
