"""CPU: tests/vo_driver.py -- the reference driver's call sequence restated for machines without a DF-VO checkout (libs/dfvo.py
is not part of this repository) -- reproduces the goldens the UNMODIFIED driver produced (tests/golden/dfvo_driver_*.npz), so the GPU drop-in test
(test_gpu_dropin.py) is anchored on the reference's own output.  Kernels run in the host-emulation build; the two networks
are replaced by the analytic frame inputs here (their emulation takes minutes) and run for real in the GPU test."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "tests", "golden")


def _run_sequence(hostsim_lib, golden, extra):
    sys.path.insert(0, os.path.join(ROOT, "tests", "hostsim"))
    from runtime import HostsimRuntime
    import dropin_cases as dc
    import synthdata
    from b200 import runtime as rt_mod, tracking
    from oracle import seqdata
    rt_mod.set_runtime(HostsimRuntime(hostsim_lib))
    tracking._default_engine = None
    dc.fresh_libs()
    import libs.deep_models.deep_models as dm
    import vo_driver
    g = np.load(os.path.join(G, golden))
    h, w = [int(v) for v in g["hw"]]
    n = g["poses"].shape[0]
    K = synthdata.kitti_intrinsics(h, w)
    cfg = dc.make_cfg(h, w, extra)
    seqdata.patch_deep_model(dm.DeepModel, h, w, K)          # the networks are far too slow in the CPU emulation
    tracking.default_engine(h, w)                            # (the patched initialize_models builds no engine)
    frames = [synthdata.value_noise_image(h, w, 100 + i) for i in range(n)]
    np.random.seed(cfg.seed)
    drv = vo_driver.SequenceDriver(cfg, K, frames)
    orig = drv.infer

    def infer():
        drv.deep_models._t = drv.cur["id"]
        orig()
    drv.infer = infer
    dc.check_poses(drv.run(), g["poses"])


def test_vendored_sequence_matches_reference_golden(hostsim_lib):
    _run_sequence(hostsim_lib, "dfvo_driver_188x620.npz", None)


def test_vendored_sequence_iterative_matches_reference_golden(hostsim_lib):
    import dropin_cases as dc
    _run_sequence(hostsim_lib, "dfvo_driver_iter_188x620.npz", dc.ITERATIVE)
