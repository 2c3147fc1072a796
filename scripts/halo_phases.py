"""Per-phase clocks of a k_conv_halo tile (development aid): where a tile's time goes, per shape and tile configuration.

    python scripts/halo_phases.py OUT_DIR [--shapes SUBSTR ...] [--configs default|all] [--build-only | --lib SO]

Builds a second copy of the library into OUT_DIR with -DDFVO_HALO_STAMPS (the product library in df-vo_b200/csrc is not
touched): the leader thread of each consumer warpgroup then records clock64() at fixed points of every tile it runs
(tc_ptx.cuh, DFVO_HALO_STAMP).  Runs the scripts/conv_shapes.py shapes through that copy, each with the configuration the
library picks and, with --configs all, with every (S, block_n, CTAs per SM) forced through DFVO_HALO_S / _BN / _CTAS, and
writes OUT_DIR/halo_phases.json: per shape and configuration the median and p90 clocks per tile of

    a_first   waiting for the tile's first A halo (tile start -> first A slot full)
    mma       the MMA loop (first A slot full -> last wgmma retired), split into
      b_wait    waiting for B (weight) slots to fill
      a_wait    waiting for the later chunks' A slots
      issue     the rest: issuing and retiring the wgmma groups
    epilogue  last wgmma retired -> the tile's outputs stored
    gap       epilogue end -> the next tile's start (same warpgroup)
    tile      tile start -> epilogue end

plus the launch time from CUDA events (of the stamped build, so slightly above the product's).  The card name, power limit
and max SM clock are recorded from nvidia-smi in the same run."""
import argparse
import ctypes
import importlib.util
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "df-vo_b200")); sys.path.insert(0, os.path.join(ROOT, "scripts"))
import numpy as np

CSRC = os.path.join(ROOT, "df-vo_b200", "csrc")
VARIANTS = [(1, 16, 1), (1, 32, 1), (1, 64, 1), (2, 16, 1), (2, 32, 1), (4, 16, 1),
            (1, 16, 2), (1, 32, 2), (1, 64, 2), (2, 16, 2), (2, 32, 2)]          # conv_halo.cu launch_halo_t
PHASES = ["a_first", "mma", "b_wait", "a_wait", "issue", "epilogue", "gap", "tile"]


def build(out_dir):
    """The library's sources and flags (csrc/build.py) plus -DDFVO_HALO_STAMPS, linked into OUT_DIR."""
    spec = importlib.util.spec_from_file_location("_dfvo_build", os.path.join(CSRC, "build.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    obj_dir = os.path.join(out_dir, "obj")
    os.makedirs(obj_dir, exist_ok=True)
    procs, objs = [], []
    for src in m.SOURCES:
        obj = os.path.join(obj_dir, src.replace(".cu", ".o"))
        objs.append(obj)
        extra = ["-fmad=false"] if src in m.NO_FMA else []
        cmd = ["nvcc"] + m.NVCC_FLAGS + extra + ["-DDFVO_HALO_STAMPS", "-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    for src, p in procs:
        out, _ = p.communicate()
        log.append("==== %s ====\n%s" % (src, out))
        if p.returncode != 0:
            sys.stderr.write(out)
            raise RuntimeError("nvcc failed on %s" % src)
    with open(os.path.join(out_dir, "build.log"), "w") as f:
        f.write("\n".join(log))
    lib = os.path.join(out_dir, "libdfvo_b200_stamps.so")
    subprocess.check_call(["nvcc", "-shared", "-o", lib] + objs + ["-lcudart"])
    return lib


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return "nvidia-smi unavailable: %s" % e


def read_stamps(lib):
    dims = (ctypes.c_int * 3)()
    lib.dfvo_halo_stamps_read(None, dims)
    ctas, tiles, n = dims
    buf = np.zeros((ctas, 2, tiles + 1, n), np.uint64)
    if lib.dfvo_halo_stamps_read(buf.ctypes.data_as(ctypes.c_void_p), dims) != 0:
        raise RuntimeError("dfvo_halo_stamps_read failed")
    return buf[:, :, :tiles].astype(np.int64)


def phases(st):
    """Per-tile phase clocks from a [CTA][warpgroup][tile][slot] stamp array (slots: tc_ptx.cuh, DFVO_HALO_STAMPS)."""
    t0, t1, aw, bw, t4, t5 = (st[..., k] for k in range(6))
    done = (t0 != 0) & (t5 != 0)
    nxt = np.zeros_like(t0)
    nxt[..., :-1] = t0[..., 1:]
    per = {
        "a_first": t1 - t0, "mma": t4 - t1, "b_wait": bw, "a_wait": aw - (t1 - t0),
        "issue": (t4 - t1) - bw - (aw - (t1 - t0)), "epilogue": t5 - t4, "tile": t5 - t0,
    }
    res = {}
    for k, v in per.items():
        x = v[done]
        res[k] = dict(median=float(np.median(x)), p90=float(np.percentile(x, 90))) if x.size else None
    g = (nxt - t5)[done & (nxt != 0)]
    res["gap"] = dict(median=float(np.median(g)), p90=float(np.percentile(g, 90))) if g.size else None
    res["tiles"] = int(done.sum())
    return res


def run(args, lib_path):
    import torch
    import conv_shapes
    from b200 import native
    assert torch.cuda.is_available(), "halo_phases.py measures on a CUDA device"
    lib = native.Lib(lib_path)
    native._lib = lib
    info = card()
    print(info, flush=True)
    rows = []
    for name, case in conv_shapes.SHAPES.items():
        if args.shapes and not any(s in name for s in args.shapes):
            continue
        B, Cin, H, W, Cout, kh, kw, py, px, act = case
        rs = np.random.RandomState(Cin + 13 * Cout + kh)
        x = torch.from_numpy(rs.standard_normal((B, Cin, H, W)).astype(np.float32)).cuda()
        w = (rs.standard_normal((Cout, Cin, kh, kw)) / np.sqrt(Cin * kh * kw)).astype(np.float32)
        b = (rs.standard_normal(Cout) * 0.1).astype(np.float32)
        out = torch.zeros((B, Cout, H, W), dtype=torch.float32, device="cuda")

        def conv():
            lib.check(lib.dfvo_conv2d(ctypes.c_void_p(x.data_ptr()), w.ctypes.data_as(ctypes.c_void_p), b.ctypes.data_as(ctypes.c_void_p),
                                      ctypes.c_void_p(out.data_ptr()), B, Cin, H, W, Cout, kh, kw, 1, py, px, 0, act,
                                      native.PREC_BF16, None))
        cout_pad = (Cout + 15) // 16 * 16
        configs = [None] + ([v for v in VARIANTS if cout_pad % v[1] == 0] if args.configs == "all" else [])
        for cfg in configs:
            for k, v in zip(("DFVO_HALO_S", "DFVO_HALO_BN", "DFVO_HALO_CTAS"), cfg or (None, None, None)):
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = str(v)
            conv(); conv()
            torch.cuda.synchronize()
            read_stamps(lib)                                  # zero the buffer
            lib.dfvo_profile_enable(1)
            conv()
            torch.cuda.synchronize()
            ms, n, _, lines = conv_shapes.read_profile(lib)
            lib.dfvo_profile_enable(0)
            st = read_stamps(lib)
            m = conv_shapes.DESC.search(lines[-1]) if lines else None
            if not (m and "halo" in lines[-1]):
                print("%-18s %-12s not a halo launch, skipped" % (name, cfg), flush=True)
                continue
            bn, S = int(m.group(1)), int(m.group(2))
            ctas = int(lines[-1].split(" ctas")[1].split()[0])
            if cfg and (S, bn, ctas) != cfg:
                print("%-18s %-12s does not fit (library chose S%d bn%d ctas%d), skipped" % (name, cfg, S, bn, ctas), flush=True)
                continue
            ph = phases(st)
            row = dict(name=name, case=list(case), S=S, block_n=bn, ctas=ctas, default=cfg is None, us=ms / n * 1e3,
                       grid=int(m.group(5)), ntiles=int(m.group(6)), phases=ph)
            rows.append(row)
            print("%-18s S%d bn%-2d ctas%d %s %8.1f us  " % (name, S, bn, ctas, "*" if cfg is None else " ", row["us"]) +
                  "  ".join("%s %6.0f" % (k, ph[k]["median"]) for k in PHASES if ph.get(k)), flush=True)
        for k in ("DFVO_HALO_S", "DFVO_HALO_BN", "DFVO_HALO_CTAS"):
            os.environ.pop(k, None)
        del x, out
        torch.cuda.empty_cache()
    with open(os.path.join(args.out_dir, "halo_phases.json"), "w") as f:
        json.dump(dict(device=info, units="clk (clock64, SM clock) per tile", rows=rows), f, indent=1)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--shapes", nargs="*", help="only shapes whose name contains one of these")
    ap.add_argument("--configs", choices=["default", "all"], default="default")
    ap.add_argument("--build-only", action="store_true", help="build the stamped library into OUT_DIR and stop")
    ap.add_argument("--lib", help="a stamped library built earlier with --build-only")
    args = ap.parse_args()
    os.makedirs(args.out_dir, exist_ok=True)
    lib = args.lib or build(args.out_dir)
    if not args.build_only:
        run(args, lib)
