"""TEST INFRASTRUCTURE ONLY: build the network-runner probe library (tests/kernels/nets/probe_nets.cu) twice.

    python tests/kernels/nets/build.py [--force]

* device: nvcc for sm_90a with the product's own NVCC_FLAGS, linked against the product libdfvo_b200.so ->
  tests/kernels/_build/libdfvo_probe_nets.so;
* hostsim: g++ -DDFVO_HOSTSIM against the CPU emulation library of tests/hostsim -> tests/kernels/_build/libdfvo_probe_nets_hostsim.so.

Same recipe and output directory as the kernel probe (tests/kernels/build.py), whose helpers it uses.  Outputs are git-ignored;
a content stamp skips rebuilds."""
import hashlib
import importlib.util
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "probe_nets.cu")


def _load(path, name):
    spec = importlib.util.spec_from_file_location(name, path)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


K = _load(os.path.join(os.path.dirname(HERE), "build.py"), "_probe_build")
DEVICE_OUT = os.path.join(K.OUTDIR, "libdfvo_probe_nets.so")
HOSTSIM_OUT = os.path.join(K.OUTDIR, "libdfvo_probe_nets_hostsim.so")


def _digest(extra):
    h = hashlib.sha1()
    for f in sorted(os.listdir(K.CSRC)):
        if f.endswith((".cu", ".cuh", ".h")):
            h.update(open(os.path.join(K.CSRC, f), "rb").read())
    h.update(open(SRC, "rb").read())
    h.update(" ".join(extra).encode())
    return h.hexdigest()


def _stamp(out, dig):
    with open(out + ".stamp", "w") as f:
        f.write(dig)


def build_device(force=False):
    prod = K._load(os.path.join(K.CSRC, "build.py"), "_dfvo_build")
    lib = prod.build()
    flags = [f for f in prod.NVCC_FLAGS if f not in ("-Xptxas", "-v")]
    dig = _digest(flags)
    if not force and K._fresh(DEVICE_OUT, dig):
        return DEVICE_OUT
    os.makedirs(K.OUTDIR, exist_ok=True)
    rpath = "$ORIGIN/" + os.path.relpath(os.path.dirname(lib), K.OUTDIR)
    K._run(["nvcc"] + flags + ["-shared", "-I", K.CSRC, SRC, "-o", DEVICE_OUT,
                               "-L", os.path.dirname(lib), "-l:" + os.path.basename(lib), "-Xlinker", "-rpath," + rpath, "-lcudart"])
    _stamp(DEVICE_OUT, dig)
    return DEVICE_OUT


def build_hostsim(force=False):
    lib = K._load(os.path.join(K.HOSTSIM, "build.py"), "_hostsim_build").build()
    flags = ["-O2", "-g", "-std=c++17", "-fPIC", "-DDFVO_HOSTSIM", "-I", K.HOSTSIM, "-I", K.CSRC, "-Wno-unused-value"]
    h = hashlib.sha1(_digest(flags).encode())
    h.update(open(os.path.join(K.HOSTSIM, "cuda_hostsim.h"), "rb").read())
    dig = h.hexdigest()
    if not force and K._fresh(HOSTSIM_OUT, dig):
        return HOSTSIM_OUT
    os.makedirs(K.OUTDIR, exist_ok=True)
    rpath = "$ORIGIN/" + os.path.relpath(os.path.dirname(lib), K.OUTDIR)
    K._run(["g++"] + flags + ["-shared", "-x", "c++", SRC, "-x", "none", "-o", HOSTSIM_OUT,
                              "-L", os.path.dirname(lib), "-l:" + os.path.basename(lib), "-Wl,-rpath," + rpath])
    _stamp(HOSTSIM_OUT, dig)
    return HOSTSIM_OUT


def build(force=False):
    return build_device(force), build_hostsim(force)


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
