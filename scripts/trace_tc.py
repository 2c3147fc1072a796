"""Per-layer CUDA-event times of every tensor-core conv launch of one frame (development aid).
Run with DFVO_TC_TRACE=1; the table goes to stderr."""
import ctypes, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "df-vo_b200")); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
import synthdata as synth
from b200 import native, pipeline, runtime as rt_mod

H, W = 376, 1241
rt = rt_mod.CudaRuntime(0); rt_mod.set_runtime(rt)
lib = rt.lib
K = synth.kitti_intrinsics(H, W)
pipe = pipeline.FramePipeline(K, H, W, precision=native.PREC_BF16, runtime=rt)
enc, dec = synth.monodepth2_weights(4869, 192, 640)
pipe.load_weights(synth.liteflownet_weights(), enc, dec)
frames = [synth.value_noise_image(H, W, i) for i in range(3)]
st = None
for i in range(4):
    cur = pipe.infer(frames[i % 3], i); pipe.ref = cur
torch.cuda.synchronize()
lib.dfvo_profile_enable(1)
cur = pipe.infer(frames[1], 4)
torch.cuda.synchronize()
ms, n, fl = ctypes.c_double(), ctypes.c_longlong(), ctypes.c_double()
lib.dfvo_profile_read(ctypes.byref(ms), ctypes.byref(n), ctypes.byref(fl))
print("conv_tc: %d launches, %.3f ms, %.1f GFLOP -> %.1f TFLOP/s" % (n.value, ms.value, fl.value / 1e9, fl.value / ms.value / 1e9))
