"""Per-shape times of the halo-resident tensor-core convolution at the LiteFlowNet level-2 / level-3 layer shapes (batch 2:
the 3x3 layers of both levels and the level-2 1x1 and 7x1 layers), through dfvo_conv2d (bf16 operands, fp32 accumulate).

    python scripts/conv_shapes.py OUT_DIR [--iters 50] [--save-outputs DIR] [--compare DIR_A DIR_B]

For every shape: CUDA events around each conv kernel launch (the library's per-launch profile), summed over --iters launches
after a warm-up; ms per launch, TFLOP/s, the tile configuration the library chose (S, block_n, stages, grid, tiles) and the
bytes one tile moves L2 -> SM by the tile model (A: one (8S + kw - 1) x (16 + kh - 1) pixel halo box per 64-channel chunk;
B: kh * kw weight boxes of block_n x 128 B per chunk).  OUT_DIR/conv_shapes.json holds the table and a SHA-256 of every
output.  --save-outputs writes each output as .npy; --compare prints the max abs difference of two such directories."""
import argparse
import ctypes
import hashlib
import json
import os
import re
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "df-vo_b200"))
import numpy as np

# B, Cin, H, W, Cout, kh, kw, pad_y, pad_x, act
SHAPES = {
    # tests/test_gpu_stage_ops.py TC_BIG_CASES: level 2 (176 x 608)
    "L2 128->128 3x3": (2, 128, 176, 608, 128, 3, 3, 1, 1, 1),
    "L2 130->128 3x3": (2, 130, 176, 608, 128, 3, 3, 1, 1, 1),
    "L2 128->64 3x3": (2, 128, 176, 608, 64, 3, 3, 1, 1, 1),
    "L2 64->32 3x3": (2, 64, 176, 608, 32, 3, 3, 1, 1, 1),
    "L2 32->64 1x1": (2, 32, 176, 608, 64, 1, 1, 0, 0, 1),
    "L2 32->49 7x1": (2, 32, 176, 608, 49, 7, 1, 3, 0, 0),
    # the other level-2 3x3 layers of Matching / Subpixel / Regularization
    "L2 49->128 3x3": (2, 49, 176, 608, 128, 3, 3, 1, 1, 1),
    "L2 144->128 3x3": (2, 144, 176, 608, 128, 3, 3, 1, 1, 1),
    "L2 64->64 3x3": (2, 64, 176, 608, 64, 3, 3, 1, 1, 1),
    "L2 32->32 3x3": (2, 32, 176, 608, 32, 3, 3, 1, 1, 1),
    # level 3 (88 x 304)
    "L3 49->128 3x3": (2, 49, 88, 304, 128, 3, 3, 1, 1, 1),
    "L3 144->128 3x3": (2, 144, 88, 304, 128, 3, 3, 1, 1, 1),
    "L3 128->128 3x3": (2, 128, 88, 304, 128, 3, 3, 1, 1, 1),
    "L3 128->64 3x3": (2, 128, 88, 304, 64, 3, 3, 1, 1, 1),
    "L3 64->64 3x3": (2, 64, 88, 304, 64, 3, 3, 1, 1, 1),
    "L3 64->32 3x3": (2, 64, 88, 304, 32, 3, 3, 1, 1, 1),
    "L3 32->32 3x3": (2, 32, 88, 304, 32, 3, 3, 1, 1, 1),
}

DESC = re.compile(r"bn(\d+) S(\d+) stages(\d+)/(\d+) grid(\d+) tiles(\d+)")


def fname(name):
    return re.sub(r"[^A-Za-z0-9]+", "_", name).strip("_")


def tile_bytes(case, S, bn):
    B, Cin, H, W, Cout, kh, kw = case[:7]
    chunks = (((Cin + 15) // 16 * 16) * 2 + 127) // 128
    a = (8 * S + kw - 1) * (16 + kh - 1) * 128 * chunks
    b = kh * kw * bn * 128 * chunks
    return a, b


def read_profile(lib):
    """Summed event time and launch count since dfvo_profile_enable(1), plus the per-launch descriptions the library prints
    to stderr when DFVO_TC_TRACE is set."""
    prev = os.environ.get("DFVO_TC_TRACE")
    os.environ["DFVO_TC_TRACE"] = "1"
    sys.stderr.flush()
    saved = os.dup(2)
    with tempfile.TemporaryFile(mode="w+") as f:
        os.dup2(f.fileno(), 2)
        try:
            ms, n, fl = ctypes.c_double(), ctypes.c_longlong(), ctypes.c_double()
            lib.dfvo_profile_read(ctypes.byref(ms), ctypes.byref(n), ctypes.byref(fl))
        finally:
            os.dup2(saved, 2); os.close(saved)
        f.seek(0)
        lines = f.read().splitlines()
    if prev is None:
        del os.environ["DFVO_TC_TRACE"]
    else:
        os.environ["DFVO_TC_TRACE"] = prev
    return ms.value, n.value, fl.value, lines


def run(args):
    import torch
    from b200 import native
    assert torch.cuda.is_available(), "conv_shapes.py measures on a CUDA device"
    lib = native.load()
    os.makedirs(args.out_dir, exist_ok=True)
    if args.save_outputs:
        os.makedirs(args.save_outputs, exist_ok=True)
    rows = []
    for name, case in SHAPES.items():
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
        for _ in range(5):
            conv()
        torch.cuda.synchronize()
        lib.dfvo_profile_enable(1)
        for _ in range(args.iters):
            conv()
        torch.cuda.synchronize()
        ms, n, flops, lines = read_profile(lib)
        lib.dfvo_profile_enable(0)
        assert n == args.iters, "%s: %d profiled launches for %d calls" % (name, n, args.iters)
        m = DESC.search(lines[-1]) if lines else None
        assert m and "halo" in lines[-1], "%s: not a halo launch: %s" % (name, lines[-1:] or "no trace")
        bn, S, ast, bst, grid, tiles = (int(g) for g in m.groups())
        a_bytes, b_bytes = tile_bytes(case, S, bn)
        y = out.cpu().numpy()
        if args.save_outputs:
            np.save(os.path.join(args.save_outputs, fname(name) + ".npy"), y)
        row = dict(name=name, case=list(case), ms=ms / n, tflops=flops / (ms / 1e3) / 1e12, gflop=flops / n / 1e9, S=S, block_n=bn,
                   a_stages=ast, b_stages=bst, grid=grid, tiles=tiles, tile_a_bytes=a_bytes, tile_b_bytes=b_bytes,
                   b_share=b_bytes / (a_bytes + b_bytes), sha256=hashlib.sha256(y.tobytes()).hexdigest())
        rows.append(row)
        print("%-18s %8.3f ms %7.1f TFLOP/s  S%d bn%-3d stages %d/%-2d grid %3d tiles %5d  A %6d B %6d B/tile (B %.0f %%)" % (
            name, row["ms"], row["tflops"], S, bn, ast, bst, grid, tiles, a_bytes, b_bytes, 100 * row["b_share"]), flush=True)
        del x, out
        torch.cuda.empty_cache()
    dev = torch.cuda.get_device_name(0)
    with open(os.path.join(args.out_dir, "conv_shapes.json"), "w") as f:
        json.dump(dict(device=dev, iters=args.iters, shapes=rows), f, indent=1)
    print("total %.3f ms over %d shapes on %s" % (sum(r["ms"] for r in rows), len(rows), dev))


def compare(a, b):
    worst = 0.0
    for name in SHAPES:
        x, y = (np.load(os.path.join(d, fname(name) + ".npy")) for d in (a, b))
        d = float(np.abs(x.astype(np.float64) - y).max()) if x.shape == y.shape else float("inf")
        print("%-18s max abs diff %g" % (name, d))
        worst = max(worst, d)
    print("max abs diff over all shapes: %g" % worst)
    return worst


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir", nargs="?")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--save-outputs", metavar="DIR")
    ap.add_argument("--compare", nargs=2, metavar="DIR")
    args = ap.parse_args()
    if args.compare:
        sys.exit(0 if compare(*args.compare) == 0 else 1)
    if not args.out_dir:
        ap.error("OUT_DIR is required")
    run(args)
