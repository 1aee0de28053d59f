"""The one-pass blur->sobel kernel against the card's practical copy ceiling, in one run on one card.

    python tools/blur_sobel_attrib.py [--lib NAME=PATH ...] [--reps 5] [--iters 20] [--out FILE.json]

Prints the card's name, power limit and SM clocks, then, each in ms and GB/s (CUDA events, warmed first):
  * copy    device-to-device torch copy_ of the c2 batch (256 x 4096^2 u8): the practical HBM ceiling of a
            1:1 read:write stream, the figure the kernels below are set against;
  * sobel   gs_b200_sobel_batch at c2's shape;
  * fused   gs_b200_blur_sobel_batch, r=5, at c2's shape, at c5's (1024 x 1920x1080) and on one 4096^2 frame,
            whose 16 MB in and 16 MB out stay in the 50 MB L2 across the back-to-back calls.
Every kernel moves 1 B read + 1 B written per pixel, so GB/s = 2 * pixels / time for all of them.  The fused rows
also give the time per 256 x 110 tile: the L2-resident frame's against c2's tells whether the kernel waits on its
tile loads from HBM (well below c2's) or is bound by issuing its instructions (about equal).  One frame is only about
1.5 waves of resident CTAs, so that comparison is approximate.  Several builds of the library (--lib, default: this
tree's) are loaded side by side and timed alternately, --reps times; the median and the spread (max - min over the
median) are reported per build.  Needs a CUDA device; writes only the --out file.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R = 5
C2, C5, L2 = (256, 4096, 4096), (1024, 1920, 1080), (1, 4096, 4096)     # (frames, w, h)
TW, TH = 256, 110                                                      # the fused kernel's tile


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
    for fn in (lib.gs_b200_blur_sobel_batch, lib.gs_b200_sobel_batch):
        fn.restype = C.c_int
    lib.gs_b200_blur_sobel_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint, C.c_uint, C.c_uint, C.c_uint, C.c_void_p]
    lib.gs_b200_sobel_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint, C.c_uint, C.c_uint, C.c_void_p]
    lib.gs_b200_set_device.argtypes = [C.c_int]
    lib.gs_b200_set_device(0)
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=[], metavar="NAME=PATH",
                    help="a build of libgrayskull_b200.so to time (repeatable)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out")
    a = ap.parse_args()
    libs = [s.split("=", 1) for s in a.lib] or [["tree", os.path.join(ROOT, "grayskull_b200", "libgrayskull_b200.so")]]

    import torch
    assert torch.cuda.is_available(), "needs a CUDA device"
    builds = {name: load(os.path.abspath(path)) for name, path in libs}
    stream = torch.cuda.current_stream().cuda_stream
    res = {"gpu_before": gpu_info(), "device": torch.cuda.get_device_name(0), "radius": R, "reps": a.reps,
           "iters": a.iters, "rows": []}
    print("gpu:", res["gpu_before"], flush=True)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        # the device sleeps while the host queues the calls, so that the short L2-resident ones run back to back
        torch.cuda._sleep(4_000_000)
        e0.record()
        for _ in range(a.iters):
            fn()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) / a.iters

    def row(label, shape, fns):
        """fns: {build name: callable}; alternated, each warmed by one untimed batch (the clocks ramp up from idle)"""
        n, w, h = shape
        for fn in fns.values():
            timed(fn)
        ms = {name: [] for name in fns}
        for _ in range(a.reps):
            for name, fn in fns.items():
                ms[name].append(timed(fn))
        out = {"what": label, "frames": n, "w": w, "h": h, "builds": {}}
        tiles = n * -(-w // TW) * -(-h // TH)
        for name, v in ms.items():
            med = statistics.median(v)
            out["builds"][name] = {"ms": v, "ms_median": med, "spread_pct": 100 * (max(v) - min(v)) / med,
                                   "GB_s": 2 * n * w * h / med / 1e6, "us_per_tile": 1e3 * med / tiles}
        res["rows"].append(out)
        print("%-6s %4d x %dx%d  " % (label, n, w, h) +
              "  ".join("%s %.4f ms %.0f GB/s (spread %.2f%%)" % (k, b["ms_median"], b["GB_s"], b["spread_pct"]) +
                        (" %.4f us/tile" % b["us_per_tile"] if label == "fused" else "")
                        for k, b in out["builds"].items()), flush=True)
        return out

    def check(rc):
        assert rc == 0, rc

    for shape in (C2, C5, L2):
        n, w, h = shape
        g = torch.Generator(device="cuda").manual_seed(w * h + n)
        src = torch.randint(0, 256, (n, h, w), dtype=torch.uint8, device="cuda", generator=g)
        dst = torch.zeros_like(src)
        if shape == C2:
            row("copy", shape, {"torch": lambda: dst.copy_(src)})
            row("sobel", shape, {name: (lambda lib=lib: check(lib.gs_b200_sobel_batch(
                dst.data_ptr(), src.data_ptr(), w, h, n, stream))) for name, lib in builds.items()})
        row("fused", shape, {name: (lambda lib=lib: check(lib.gs_b200_blur_sobel_batch(
            dst.data_ptr(), src.data_ptr(), w, h, n, R, stream))) for name, lib in builds.items()})
        del src, dst
        torch.cuda.empty_cache()
    res["gpu_after"] = gpu_info()
    copy_gbs = res["rows"][0]["builds"]["torch"]["GB_s"]
    for r in res["rows"][1:]:
        for name, b in r["builds"].items():
            b["of_copy"] = b["GB_s"] / copy_gbs
            print("%-6s %dx%d %s: %.3f of the copy rate" % (r["what"], r["w"], r["h"], name, b["of_copy"]))
    print("gpu:", res["gpu_after"])
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    sys.exit(main())
