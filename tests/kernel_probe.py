"""ctypes bindings of the kernel probe library (tests/kernels/probe.cu) and the buffer helpers its tests share.

Tensors are torch tensors: CUDA tensors with the device build, CPU tensors with the host-emulation build (whose "device
pointers" are host pointers).  A `Buf` is one flat allocation; a `View` is an NHWC window into it with explicit element strides,
which is how the kernels see every operand.  Buffers start out poisoned -- NaN in sources (a kernel that reads outside its view
produces a non-finite value), a NaN *sentinel bit pattern* in outputs (a kernel that writes outside its view changes it)."""
import ctypes
import importlib.util
import os

import torch

HERE = os.path.dirname(os.path.abspath(__file__))

# NaN payloads no kernel computes (computed NaNs are the canonical 0x7FC0 / 0x7FFF patterns)
SENTINEL = {torch.bfloat16: 0x7FA5, torch.float32: 0x7FA0DEAD}
INT_VIEW = {torch.bfloat16: torch.int16, torch.float32: torch.int32}


class Ten(ctypes.Structure):
    _fields_ = [("p", ctypes.c_void_p), ("N", ctypes.c_int), ("H", ctypes.c_int), ("W", ctypes.c_int), ("C", ctypes.c_int),
                ("sN", ctypes.c_longlong), ("sH", ctypes.c_longlong), ("sW", ctypes.c_longlong)]


class Conv(ctypes.Structure):
    """Mirror of probe.cu::ProbeConv (itself a flat mirror of dfvo::ConvTc)."""
    _fields_ = [("N", ctypes.c_int), ("H", ctypes.c_int), ("W", ctypes.c_int), ("inH", ctypes.c_int), ("inW", ctypes.c_int),
                ("nsrc", ctypes.c_int), ("src", Ten * 3), ("stride", ctypes.c_int), ("ntaps", ctypes.c_int),
                ("dy", ctypes.c_int * 49), ("dx", ctypes.c_int * 49), ("esize", ctypes.c_int), ("round_out_tf32", ctypes.c_int),
                ("w", ctypes.c_void_p), ("Cout_pad", ctypes.c_int), ("Cout", ctypes.c_int), ("bias", ctypes.c_void_p),
                ("act", ctypes.c_int), ("out_f32", ctypes.c_int), ("out", Ten), ("residual", Ten), ("zero_pad_to", ctypes.c_int)]


class View:
    def __init__(self, buf, off, N, H, W, C, sN, sH, sW):
        self.buf, self.off = buf, off
        self.N, self.H, self.W, self.C, self.sN, self.sH, self.sW = N, H, W, C, sN, sH, sW

    @property
    def t(self):
        """The view's elements as an [N, H, W, C] strided torch tensor (writes go to the buffer)."""
        return torch.as_strided(self.buf.flat, (self.N, self.H, self.W, self.C), (self.sN, self.sH, self.sW, 1), self.off)

    @property
    def ten(self):
        return Ten(self.buf.flat.data_ptr() + self.off * self.buf.flat.element_size(), self.N, self.H, self.W, self.C,
                   self.sN, self.sH, self.sW)

    def nchw64(self):
        return self.t.permute(0, 3, 1, 2).double()


class Buf:
    def __init__(self, n, dtype, device, sentinel=False):
        self.dtype = dtype
        self.flat = torch.full((n,), float("nan"), dtype=dtype, device=device)
        if sentinel:
            self.flat.view(INT_VIEW[dtype]).fill_(SENTINEL[dtype])

    def view(self, N, H, W, C, sW=None, sH=None, sN=None, off=0):
        sW = C if sW is None else sW
        sH = W * sW if sH is None else sH
        sN = H * sH if sN is None else sN
        assert off + (N - 1) * sN + (H - 1) * sH + (W - 1) * sW + C <= self.flat.numel(), "view past the end of its buffer"
        return View(self, off, N, H, W, C, sN, sH, sW)

    def untouched_outside(self, views):
        """Number of elements outside every view that no longer hold the sentinel bit pattern (0 = nothing was written there)."""
        inside = torch.zeros(self.flat.shape, dtype=torch.bool, device=self.flat.device)
        for v in views:
            torch.as_strided(inside, (v.N, v.H, v.W, v.C), (v.sN, v.sH, v.sW, 1), v.off).fill_(True)
        bits = self.flat.view(INT_VIEW[self.dtype])
        bad = (~inside) & (bits != SENTINEL[self.dtype])
        return int(bad.sum().item())


def bf16_rt(x):
    return x.to(torch.bfloat16).to(x.dtype)


def tf32_rna(x):
    """fp32 -> tf32 grid, round to nearest, ties away from zero (cvt.rna.tf32.f32)."""
    x = x.float().contiguous()
    u = x.view(torch.int32).to(torch.int64)
    u = ((u + 0x1000) & 0xFFFFE000)
    u = torch.where(u >= 2 ** 31, u - 2 ** 32, u).to(torch.int32)
    return u.view(torch.float32)


class Probe:
    def __init__(self, path, device):
        self.lib = ctypes.CDLL(path)
        self.device = device
        self.lib.probe_last_error.restype = ctypes.c_char_p
        self.lib.probe_flow_mean_buffer_floats.restype = ctypes.c_longlong
        a, b = ctypes.c_int(), ctypes.c_int()
        self.lib.probe_struct_sizes(ctypes.byref(a), ctypes.byref(b))
        assert (a.value, b.value) == (ctypes.sizeof(Ten), ctypes.sizeof(Conv)), "probe.cu structs and kernel_probe.py disagree"

    @property
    def is_device(self):
        return bool(self.lib.probe_is_device_build())

    def sync(self):
        if self.device == "cuda":
            torch.cuda.synchronize()

    def __call__(self, name, *args):
        conv = []
        for a in args:
            if isinstance(a, View):
                a = ctypes.byref(a.ten)
            elif isinstance(a, (Ten, Conv)):
                a = ctypes.byref(a)
            elif isinstance(a, torch.Tensor):
                a = ctypes.c_void_p(a.data_ptr())
            elif isinstance(a, float):
                a = ctypes.c_float(a)
            conv.append(a)
        rc = getattr(self.lib, name)(*conv)
        if rc != 0:
            msg = self.lib.probe_last_error()
            raise RuntimeError("%s failed (%d): %s" % (name, rc, msg.decode() if msg else "?"))
        self.sync()


def _build_module():
    spec = importlib.util.spec_from_file_location("_probe_build", os.path.join(HERE, "kernels", "build.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def load_device():
    """The probe linked against the product library (load the product first: one copy of it must be mapped)."""
    return Probe(_build_module().build_device(), "cuda")


def load_hostsim():
    return Probe(_build_module().build_hostsim(), "cpu")


def kernel_names(fn, want=()):
    """Run fn() under torch.profiler (CUDA activity) and return the names of the kernels it launched.  CUPTI can drop activity
    records (most often in a profiler's first cycles), so the collection -- only the collection, never a value check -- is
    repeated, up to three times, until every name in `want` has been seen; fn must be safe to relaunch."""
    from torch.profiler import ProfilerActivity, profile
    names = set()
    for _ in range(3):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
        if all(any(w in n for n in names) for w in want):
            break
    return names
