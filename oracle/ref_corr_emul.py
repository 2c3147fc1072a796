"""Run the REFERENCE's own correlation CUDA kernels on the CPU, from the source text where it
lies (``libs/deep_models/flow/lite_flow_net/correlation.py:11-106`` of the checkout), to pin
the oracle restatement ``oracle.nets.correlation`` (needs
a checkout named by ``DFVO_REFERENCE_ROOT``); products go to ``oracle/_ref/`` (git-ignored).

How: the reference keeps its kernels as CUDA-C strings and specialises them per tensor shape
with its own pure-Python ``cupy_kernel`` substitution (correlation.py:238-274).  We call that
function unchanged, wrap the resulting text in a tiny CUDA-execution-model emulation
(``blockIdx``/``threadIdx`` variables, one OpenMP thread per CUDA thread of a block,
``__syncthreads`` = ``omp barrier``, ``__shared__`` = one static buffer per block; blocks run
one after another), compile with gcc and launch with the reference's own grid/block shapes
(correlation.py:298-333).

One deliberate addition: the reference kernel re-zeroes ``sum[ch_off]`` for the next output
channel without a barrier after thread 0's serial reduction (correlation.py:72-104), relying on
warp lock-step.  The emulation inserts a barrier there, which is the lock-step behaviour.
"""
import ctypes
import hashlib
import math
import os
import subprocess

import numpy as np

from . import shims

_REF_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")

_HARNESS = r"""
#include <omp.h>
#include <string.h>
typedef struct { int x, y, z; } dim3_t;
static dim3_t blockIdx, blockDim;
static __thread dim3_t threadIdx;
static char patch_data_char[1 << 16];
static float sum[32];
#define __global__
#define SYNC_%(sync)s
#ifdef SYNC_ON
#define __syncthreads() _Pragma("omp barrier")
#else
#define __syncthreads()
#endif
%(kernel)s
void launch(int gx, int gy, int gz, int bx, const int n, const float* a, const float* b, float* c) {
  blockDim.x = bx; blockDim.y = 1; blockDim.z = 1;
  for (int z = 0; z < gz; ++z) for (int y = 0; y < gy; ++y) for (int x = 0; x < gx; ++x) {
    blockIdx.x = x; blockIdx.y = y; blockIdx.z = z;
    #pragma omp parallel num_threads(bx)
    {
      threadIdx.x = omp_get_thread_num(); threadIdx.y = 0; threadIdx.z = 0;
      CALL
    }
  }
}
"""


def _compile(kernel_text, name, sync, call):
    os.makedirs(_REF_DIR, exist_ok=True)
    text = kernel_text.replace('extern "C"', "")
    text = text.replace("extern __shared__ char patch_data_char[];", "")
    text = text.replace("__shared__ float sum[32];", "")
    text = text.replace("sum[ch_off] = 0;", '_Pragma("omp barrier") sum[ch_off] = 0;')
    src = (_HARNESS % {"kernel": text, "sync": "ON" if sync else "OFF"}).replace("CALL", call)
    tag = hashlib.sha1(src.encode()).hexdigest()[:12]
    so = os.path.join(_REF_DIR, "%s_%s.so" % (name, tag))
    if not os.path.exists(so):
        c = os.path.join(_REF_DIR, "%s_%s.c" % (name, tag))
        with open(c, "w") as f:
            f.write(src)
        subprocess.check_call(["gcc", "-O1", "-fopenmp", "-shared", "-fPIC", "-o", so, c])
    lib = ctypes.CDLL(so)
    lib.launch.argtypes = [ctypes.c_int] * 5 + [ctypes.c_void_p] * 3
    return lib


class _T:
    """Just enough of a tensor for the reference's ``cupy_kernel`` (uses .size()/.stride())."""

    def __init__(self, shape):
        self.shape = tuple(shape)

    def size(self):
        return self.shape

    def stride(self):
        st, acc = [], 1
        for d in reversed(self.shape):
            st.append(acc)
            acc *= d
        return tuple(reversed(st))


def reference_correlation(first, second, stride):
    """first/second: float32 numpy [B,C,H,W] -> [B,49,ceil(H/s),ceil(W/s)] computed by the
    reference kernels (rearrange x2 + updateOutput) under emulation."""
    corr = shims.import_reference("libs.deep_models.flow.lite_flow_net.correlation")
    first = np.ascontiguousarray(first, np.float32)
    second = np.ascontiguousarray(second, np.float32)
    B, C, H, W = first.shape
    s = int(stride)
    rb_shape = (B, H + 6 * s, W + 6 * s, C)                       # correlation.py:283-284
    rbot0 = np.zeros(rb_shape, np.float32)
    rbot1 = np.zeros(rb_shape, np.float32)
    out = np.zeros((B, 49, int(math.ceil(H / s)), int(math.ceil(W / s))), np.float32)  # :294

    def ptr(a):
        return a.ctypes.data_as(ctypes.c_void_p)

    for inp, rb in ((first, rbot0), (second, rbot1)):              # correlation.py:296-319
        k = corr.cupy_kernel("kernel_Correlation_rearrange",
                             {"intStride": s, "input": _T(inp.shape), "output": _T(rb.shape)})
        lib = _compile(k, "rearrange", False, "kernel_Correlation_rearrange(n, a, c);")
        n = H * W
        lib.launch(int((n + 16 - 1) / 16), C, B, 16, n, ptr(inp), None, ptr(rb))
    k = corr.cupy_kernel("kernel_Correlation_updateOutput",        # correlation.py:321-333
                         {"intStride": s, "rbot0": _T(rbot0.shape), "rbot1": _T(rbot1.shape),
                          "top": _T(out.shape)})
    lib = _compile(k, "update", True, "kernel_Correlation_updateOutput(n, a, b, c);")
    n = out.shape[1] * out.shape[2] * out.shape[3]
    lib.launch(out.shape[3], out.shape[2], out.shape[0], 32, n, ptr(rbot0), ptr(rbot1), ptr(out))
    return out
