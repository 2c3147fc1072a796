"""TEST INFRASTRUCTURE ONLY: build the kernel probe library (tests/kernels/probe.cu) twice.

    python tests/kernels/build.py [--force]

* device: nvcc for sm_90a with the product's own NVCC_FLAGS, linked against the product libdfvo_b200.so (rpath $ORIGIN-relative),
  so the probe's launches run the very kernels the product ships -> tests/kernels/_build/libdfvo_probe.so;
* hostsim: g++ -DDFVO_HOSTSIM against the CPU emulation library of tests/hostsim -> tests/kernels/_build/libdfvo_probe_hostsim.so.

Outputs are git-ignored; a content stamp skips rebuilds."""
import hashlib
import importlib.util
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "df-vo_b200", "csrc")
HOSTSIM = os.path.join(ROOT, "tests", "hostsim")
OUTDIR = os.path.join(HERE, "_build")
DEVICE_OUT = os.path.join(OUTDIR, "libdfvo_probe.so")
HOSTSIM_OUT = os.path.join(OUTDIR, "libdfvo_probe_hostsim.so")


def _load(path, name):
    spec = importlib.util.spec_from_file_location(name, path)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def _digest(extra):
    h = hashlib.sha1()
    for d in (CSRC, HERE):
        for f in sorted(os.listdir(d)):
            if f.endswith((".cu", ".cuh", ".h")):
                h.update(open(os.path.join(d, f), "rb").read())
    h.update(" ".join(extra).encode())
    return h.hexdigest()


def _fresh(out, dig):
    stamp = out + ".stamp"
    return os.path.exists(out) and os.path.exists(stamp) and open(stamp).read() == dig


def _run(cmd):
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if p.returncode != 0:
        sys.stderr.write(p.stdout)
        raise RuntimeError("probe build failed: %s" % " ".join(cmd))


def build_device(force=False):
    """nvcc -> libdfvo_probe.so, linked against (and built after) the product library."""
    prod = _load(os.path.join(CSRC, "build.py"), "_dfvo_build")
    lib = prod.build()
    flags = [f for f in prod.NVCC_FLAGS if f not in ("-Xptxas", "-v")]
    dig = _digest(flags)
    if not force and _fresh(DEVICE_OUT, dig):
        return DEVICE_OUT
    os.makedirs(OUTDIR, exist_ok=True)
    rpath = "$ORIGIN/" + os.path.relpath(os.path.dirname(lib), OUTDIR)
    _run(["nvcc"] + flags + ["-shared", "-I", CSRC, os.path.join(HERE, "probe.cu"), "-o", DEVICE_OUT,
                             "-L", os.path.dirname(lib), "-l:" + os.path.basename(lib), "-Xlinker", "-rpath," + rpath, "-lcudart"])
    with open(DEVICE_OUT + ".stamp", "w") as f:
        f.write(dig)
    return DEVICE_OUT


def build_hostsim(force=False):
    """g++ -DDFVO_HOSTSIM -> libdfvo_probe_hostsim.so, linked against the emulation library of tests/hostsim."""
    lib = _load(os.path.join(HOSTSIM, "build.py"), "_hostsim_build").build()
    flags = ["-O2", "-g", "-std=c++17", "-fPIC", "-DDFVO_HOSTSIM", "-I", HOSTSIM, "-I", CSRC, "-Wno-unused-value"]
    h = hashlib.sha1(_digest(flags).encode())
    h.update(open(os.path.join(HOSTSIM, "cuda_hostsim.h"), "rb").read())
    dig = h.hexdigest()
    if not force and _fresh(HOSTSIM_OUT, dig):
        return HOSTSIM_OUT
    os.makedirs(OUTDIR, exist_ok=True)
    rpath = "$ORIGIN/" + os.path.relpath(os.path.dirname(lib), OUTDIR)
    _run(["g++"] + flags + ["-shared", "-x", "c++", os.path.join(HERE, "probe.cu"), "-x", "none", "-o", HOSTSIM_OUT,
                            "-L", os.path.dirname(lib), "-l:" + os.path.basename(lib), "-Wl,-rpath," + rpath])
    with open(HOSTSIM_OUT + ".stamp", "w") as f:
        f.write(dig)
    return HOSTSIM_OUT


def build(force=False):
    return build_device(force), build_hostsim(force)


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
