"""Build libdfvo_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python df-vo_b200/csrc/build.py [--force]

The .so stays next to the sources (git-ignored).
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SOURCES = ["capi.cu", "net_common.cu", "flow_ops.cu", "conv_direct.cu", "conv_tc.cu", "conv_halo.cu", "conv_chain.cu", "liteflownet.cu", "select.cu", "ransac.cu", "pnp.cu", "homog.cu", "depth_ops.cu", "monodepth2.cu", "geometry.cu", "corr_mma.cu"]
NO_FMA = {"ransac.cu", "pnp.cu", "homog.cu"}
OUT = os.path.join(HERE, "libdfvo_b200.so")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v"]


def _digest():
    h = hashlib.sha1()
    for f in sorted(os.listdir(HERE)):
        if f.endswith((".cu", ".cuh", ".h")):
            h.update(open(os.path.join(HERE, f), "rb").read())
    h.update(open(os.path.join(HERE, "..", "..", "include", "dfvo_b200.h"), "rb").read())
    h.update(" ".join(NVCC_FLAGS + SOURCES).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    stamp = OUT + ".stamp"
    dig = _digest()
    if not force and os.path.exists(OUT) and os.path.exists(stamp) and open(stamp).read() == dig:
        return OUT
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(HERE, "_obj_" + src.replace(".cu", ".o"))
        objs.append(obj)
        # the FP64 pose solvers make threshold decisions that were validated without FMA contraction
        extra = ["-fmad=false"] if src in NO_FMA else []
        cmd = ["nvcc"] + NVCC_FLAGS + extra + ["-c", os.path.join(HERE, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    for src, p in procs:
        out, _ = p.communicate()
        log.append("==== %s ====\n%s" % (src, out))
        if p.returncode != 0:
            sys.stderr.write(out)
            raise RuntimeError("nvcc failed on %s" % src)
    with open(os.path.join(HERE, "build.log"), "w") as f:
        f.write("\n".join(log))
    if verbose:
        print("\n".join(log))
    subprocess.check_call(["nvcc", "-shared", "-o", OUT] + objs + ["-lcudart"])
    for o in objs:
        os.remove(o)
    with open(stamp, "w") as f:
        f.write(dig)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
