"""Where the one-pass blur->sobel kernel's time goes: interior tiles against tiles that touch an image border.

    python tools/blur_sobel_attrib.py [--lib NAME=PATH ...] [--reps 3] [--iters 30] [--out FILE.json]

k_blur_sobel_tma covers 224 columns x 128 sobel rows per CTA.  A tile is "interior" when every blurred window it
needs lies inside the image (the test the kernel made per CTA before it decided the path per warp and per lane);
every other tile holds a frame border.  This times gs_b200_blur_sobel_batch(r=5) with CUDA events at large shapes
whose border shares differ, and fits

    time = a * (interior tiles) + b * (border tiles)

by least squares.  b/a is what a border tile costs relative to an interior one.  Several builds of the library
(--lib, default: this tree's) are loaded side by side and timed alternately, each shape warmed first; the median
and spread over --reps runs are reported per build.  Needs a CUDA device; writes only the --out file.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R = 5
STRIDE, TH = 224, 128                       # box.cu: BS_STRIDE, BX_TH
SHAPES = [(256, 4096, 4096), (256, 4064, 4096), (64, 8064, 8192), (1024, 1920, 1080)]   # (frames, w, h)


def tile_counts(w, h, r=R):
    """(interior, border) tiles per frame, with the kernel's old per-CTA interior test"""
    tx, ty = (w + STRIDE - 1) // STRIDE, (h + TH - 1) // TH
    xb = np.arange(tx) * STRIDE - 16
    y0 = np.arange(ty) * TH
    ix = (xb + 8 - r >= 0) & (xb + 8 + 240 - 1 + r <= w - 1)
    iy = (y0 - 1 - r >= 0) & (y0 + TH + r <= h - 1)
    interior = int(ix.sum()) * int(iy.sum())
    return interior, tx * ty - interior


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return dict(zip(q.split(","), [s.strip() for s in out[0].split(",")])) if out else None
    except (OSError, subprocess.SubprocessError):
        return None


def load(path):
    lib = C.CDLL(path)
    fn = lib.gs_b200_blur_sobel_batch
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_uint, C.c_uint, C.c_uint, C.c_uint, C.c_void_p]
    lib.gs_b200_set_device.argtypes = [C.c_int]
    lib.gs_b200_set_device(0)
    return fn


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=[], metavar="NAME=PATH",
                    help="a build of libgrayskull_b200.so to time (repeatable)")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--out")
    a = ap.parse_args()
    libs = [s.split("=", 1) for s in a.lib] or [["tree", os.path.join(ROOT, "grayskull_b200", "libgrayskull_b200.so")]]

    import torch
    assert torch.cuda.is_available(), "needs a CUDA device"
    fns = {name: load(os.path.abspath(path)) for name, path in libs}
    stream = torch.cuda.current_stream().cuda_stream
    res = {"gpu_before": gpu_info(), "radius": R, "reps": a.reps, "iters": a.iters, "shapes": []}
    for n, w, h in SHAPES:
        g = torch.Generator(device="cuda").manual_seed(w * h + n)
        src = torch.randint(0, 256, (n, h, w), dtype=torch.uint8, device="cuda", generator=g)
        dst = torch.zeros_like(src)

        def call(fn):
            rc = fn(dst.data_ptr(), src.data_ptr(), w, h, n, R, stream)
            assert rc == 0, rc

        for fn in fns.values():                      # warm every build at this shape
            for _ in range(3):
                call(fn)
        torch.cuda.synchronize()
        ms = {name: [] for name in fns}
        for _ in range(a.reps):
            for name, fn in fns.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.iters):
                    call(fn)
                e1.record()
                e1.synchronize()
                ms[name].append(e0.elapsed_time(e1) / a.iters)
        interior, border = tile_counts(w, h)
        row = {"frames": n, "w": w, "h": h, "interior_tiles": interior * n, "border_tiles": border * n,
               "border_share": border / (interior + border), "builds": {}}
        for name, v in ms.items():
            med = statistics.median(v)
            row["builds"][name] = {"ms": v, "ms_median": med, "spread_pct": 100 * (max(v) - min(v)) / med,
                                   "mpix_s": n * w * h / med / 1e3}
        res["shapes"].append(row)
        print("%4d x %dx%d  border %4.1f%%  " % (n, w, h, 100 * row["border_share"]) +
              "  ".join("%s %.3f ms (%.0f Mpix/s, spread %.2f%%)" % (k, b["ms_median"], b["mpix_s"], b["spread_pct"])
                        for k, b in row["builds"].items()), flush=True)
        del src, dst
        torch.cuda.empty_cache()
    res["gpu_after"] = gpu_info()
    A = np.array([[s["interior_tiles"], s["border_tiles"]] for s in res["shapes"]], dtype=np.float64)
    res["fit"] = {}
    for name in fns:
        t = np.array([s["builds"][name]["ms_median"] for s in res["shapes"]])
        (ca, cb), *_ = np.linalg.lstsq(A, t, rcond=None)
        resid = t - A @ np.array([ca, cb])
        res["fit"][name] = {"a_us_per_tile": ca * 1e3, "b_us_per_tile": cb * 1e3, "b_over_a": cb / ca,
                            "max_rel_residual": float(np.max(np.abs(resid) / t))}
        print("%s: a = %.4f us, b = %.4f us per tile, b/a = %.3f (max residual %.2f%%)" %
              (name, ca * 1e3, cb * 1e3, cb / ca, 100 * res["fit"][name]["max_rel_residual"]))
    print("gpu:", res["gpu_before"], "->", res["gpu_after"])
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    sys.exit(main())
