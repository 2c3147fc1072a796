"""Drive single tensor-core conv launches (LiteFlowNet level-2 shapes) for ncu."""
import sys, os, ctypes
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "df-vo_b200")); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
from b200 import native
from util import dptr
lib = native.load()
shapes = [(2, 128, 176, 608, 128, 3, 3, 1, 1), (2, 32, 176, 608, 128, 1, 1, 0, 0), (2, 128, 176, 608, 64, 3, 3, 1, 1),
          (2, 32, 176, 608, 64, 1, 1, 0, 0), (2, 64, 176, 608, 128, 3, 3, 1, 1), (2, 64, 176, 608, 32, 3, 3, 1, 1)]
if len(sys.argv) > 1:
    shapes = [shapes[int(a)] for a in sys.argv[1:]]
for (B, Cin, H, W, Cout, kh, kw, py, px) in shapes:
    rs = np.random.RandomState(0)
    x = torch.from_numpy(rs.standard_normal((B, Cin, H, W)).astype(np.float32)).cuda()
    w = (rs.standard_normal((Cout, Cin, kh, kw)) / np.sqrt(Cin * kh * kw)).astype(np.float32)
    b = np.zeros(Cout, np.float32)
    y = torch.zeros((B, Cout, H, W), device="cuda")
    for it in range(2):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        lib.check(lib.dfvo_conv2d(dptr(x), w.ctypes.data_as(ctypes.c_void_p), b.ctypes.data_as(ctypes.c_void_p), dptr(y),
                                  B, Cin, H, W, Cout, kh, kw, 1, py, px, 0, 1, 1, None))
        e1.record(); torch.cuda.synchronize()
    print((B, Cin, H, W, Cout, kh, kw), "stage call %.3f ms (includes layout conversions + weight packing)" % e0.elapsed_time(e1), flush=True)
