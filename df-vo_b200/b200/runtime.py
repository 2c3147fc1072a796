"""Device memory / stream plumbing for the host side (PyTorch is used for exactly this: allocation,
H2D/D2H copies, streams -- never for arithmetic on the hot path).

``get()`` returns the process-wide runtime.  The product runtime is :class:`CudaRuntime`; it refuses
to exist without a CUDA device.  The CPU test-suite injects the host-emulation runtime from
``tests/hostsim`` with :func:`set_runtime` so the very same host logic (libs mirror, pipeline) can be
exercised without a GPU -- that object lives in the test tree, not here.
"""
import ctypes
import os

import numpy as np

from . import native


class Buf:
    """A typed device buffer: ``ptr`` (ctypes void*), ``shape``, ``dtype`` (numpy dtype)."""

    __slots__ = ("t", "shape", "dtype", "rt")

    def __init__(self, t, shape, dtype, rt):
        self.t, self.shape, self.dtype, self.rt = t, tuple(shape), np.dtype(dtype), rt

    @property
    def ptr(self):
        return self.rt.ptr_of(self.t)

    def numpy(self):
        """Blocking copy to a new host array."""
        return self.rt.to_host(self)

    def upload(self, arr):
        self.rt.upload(self, arr)
        return self

    def view(self, shape, offset=0):
        """A Buf over prod(shape) elements of this buffer starting at element `offset` (no copy): capacity-allocated workspaces
        hand out exactly-shaped views so a changing keypoint count never reallocates, and one entry of a batched output
        (e.g. ``flow_fwd.view((1, 2, H, W), i * 2 * H * W)``) is handed out as a buffer of its own."""
        if not offset:
            return self.rt.view(self, shape)
        n = int(np.prod(shape)) if len(shape) else 1
        if offset < 0 or offset + n > self.size:
            raise ValueError("view of %d elements at offset %d exceeds a buffer of %d" % (n, offset, self.size))
        # the runtime's view takes the leading elements: hand it the (contiguous) tail that starts at `offset`
        tail = Buf(self.t.reshape(-1)[offset:], (self.size - offset,), self.dtype, self.rt)
        return self.rt.view(tail, shape)

    def clone(self):
        """Device-side copy (same stream as the producer: ordered after it)."""
        return self.rt.clone(self)

    @property
    def size(self):
        n = 1
        for d in self.shape:
            n *= int(d)
        return n


_TORCH_DTYPES = None


def _torch_dtype(dt):
    global _TORCH_DTYPES
    import torch
    if _TORCH_DTYPES is None:
        _TORCH_DTYPES = {np.dtype(np.float32): torch.float32, np.dtype(np.float64): torch.float64,
                         np.dtype(np.int32): torch.int32, np.dtype(np.uint8): torch.uint8,
                         np.dtype(np.int64): torch.int64}
    return _TORCH_DTYPES[np.dtype(dt)]


class CudaRuntime:
    """torch.cuda-backed runtime of the product."""

    is_device = True

    def __init__(self, device=0):
        import torch
        native.require_cuda()
        self.torch = torch
        self.device = torch.device("cuda", device)
        self.device_index = int(device)
        torch.cuda.set_device(self.device)
        self.lib = native.load()
        self.stream = None          # None -> torch's current stream (0 = legacy default is never used implicitly)

    def stream_ptr(self):
        return ctypes.c_void_p(self.torch.cuda.current_stream(self.device).cuda_stream)

    def empty(self, shape, dtype):
        t = self.torch.empty(tuple(shape), dtype=_torch_dtype(dtype), device=self.device)
        return Buf(t, shape, dtype, self)

    def zeros(self, shape, dtype):
        t = self.torch.zeros(tuple(shape), dtype=_torch_dtype(dtype), device=self.device)
        return Buf(t, shape, dtype, self)

    def from_host(self, arr):
        arr = np.ascontiguousarray(arr)
        t = self.torch.from_numpy(arr).to(self.device, non_blocking=False)
        return Buf(t, arr.shape, arr.dtype, self)

    PINNED_STAGE_MAX = 1 << 20

    def nvtx(self, name):
        """NVTX range around a pipeline stage when DFVO_NVTX=1 (for `ncu --nvtx` / Nsight timelines); a null context otherwise."""
        import contextlib
        if not getattr(self, "_nvtx_on", None):
            if getattr(self, "_nvtx_on", None) is None:
                self._nvtx_on = os.environ.get("DFVO_NVTX", "0") == "1"
            if not self._nvtx_on:
                return contextlib.nullcontext()
        return self.torch.cuda.nvtx.range(name)

    def upload(self, buf, arr):
        torch = self.torch
        if torch.is_tensor(arr):                      # e.g. a pinned host tensor: asynchronous H2D on the current stream
            buf.t.copy_(arr.reshape(buf.shape), non_blocking=True)
            return
        a = np.ascontiguousarray(arr, dtype=buf.dtype).reshape(buf.shape)
        nbytes = a.nbytes
        if nbytes == 0 or nbytes > self.PINNED_STAGE_MAX or not buf.t.is_contiguous():
            buf.t.copy_(torch.from_numpy(a))
            return
        # Small host arrays (shuffles, generator state, poses) go through a pinned staging buffer and an asynchronous copy: a copy
        # from pageable memory blocks the host until everything queued before it on the stream has run (measured: 0.3 ms per
        # tracker launch).  Staging buffers come from a small pool per size class and are reused only after the copy out of them
        # has executed (an event per buffer); the pool is bounded, so neither pinned allocations (~1 ms each) nor memory grow
        # with the number of destinations.
        if not hasattr(self, "_stage_pool"):
            import threading
            self._stage_pool, self._stage_lock, self._stage_made = {}, threading.Lock(), {}
        cap = 4096
        while cap < nbytes:
            cap *= 2
        # take a free staging buffer OUT of the pool while it is in use (the tracker-thread mode uploads from two host threads)
        ent = None
        with self._stage_lock:
            pool = self._stage_pool.setdefault(cap, [])
            for i, cand in enumerate(pool):
                if cand[1] is None or cand[1].query():
                    ent = pool.pop(i)
                    break
            if ent is None and self._stage_made.get(cap, 0) >= 8 and pool:
                ent = pool.pop(0)                        # all busy: take the oldest and wait for its copy below
            if ent is None:
                self._stage_made[cap] = self._stage_made.get(cap, 0) + 1
        if ent is None:
            ent = [torch.empty((cap,), dtype=torch.uint8, pin_memory=True), None]
        elif ent[1] is not None:
            ent[1].synchronize()
        host = ent[0][:nbytes]
        host.numpy().view(a.dtype).reshape(a.shape)[...] = a
        buf.t.view(torch.uint8).reshape(-1)[:nbytes].copy_(host, non_blocking=True)
        e = torch.cuda.Event()
        e.record(torch.cuda.current_stream(self.device))
        ent[1] = e
        with self._stage_lock:
            self._stage_pool[cap].append(ent)

    def to_host(self, buf):
        return buf.t.cpu().numpy()

    def view(self, buf, shape):
        n = int(np.prod(shape)) if len(shape) else 1
        return Buf(buf.t.reshape(-1)[:n].view(tuple(shape)), shape, buf.dtype, self)

    def clone(self, buf):
        return Buf(buf.t.clone(), buf.shape, buf.dtype, self)

    def ptr_of(self, t):
        return ctypes.c_void_p(t.data_ptr())

    def sync(self):
        self.torch.cuda.current_stream(self.device).synchronize()

    # ---- streams / events (the two-stream frame pipeline: networks of frame t+1 overlap the tracker of frame t)
    def new_stream(self, high_priority=False):
        return self.torch.cuda.Stream(device=self.device, priority=-1 if high_priority else 0)

    def on_stream(self, stream):
        """Context manager: every launch / copy inside is enqueued on `stream`."""
        return self.torch.cuda.stream(stream)

    def record_event(self):
        ev = self.torch.cuda.Event()
        ev.record(self.torch.cuda.current_stream(self.device))
        return ev

    def wait_event(self, ev):
        self.torch.cuda.current_stream(self.device).wait_event(ev)

    def pinned(self, shape, dtype):
        return self.torch.empty(tuple(shape), dtype=_torch_dtype(dtype)).pin_memory()


_runtime = None


def set_runtime(rt):
    global _runtime
    _runtime = rt


def get():
    global _runtime
    if _runtime is None:
        _runtime = CudaRuntime()
    return _runtime
