"""The colour conversions (include/grayskull_color.h) on one GPU: one JSON line per call and workload.

    python tools/color_bench.py [--reps 20] [--warmup 3] [--workloads 1080p,4k]

Workloads: 256 frames of 1920x1080 ("1080p") and 64 frames of 4096x4096 ("4k"), seeded uniform random pixels.  For
each, the three forms of the library (RGBA -> gray, RGB -> gray, gray -> RGBA) and, for context, what a torch user
writes today for RGBA -> gray: the demo's expression in float32 and in float64, as eager elementwise ops on the RGBA
tensor.  Each line has the median time per call over `reps` calls timed one by one with CUDA events after `warmup`
calls, the algorithmic bytes per pixel (RGBA -> gray 4 + 1, RGB -> gray 3 + 1, gray -> RGBA 1 + 4; the torch lines
are charged the same 5, not what their intermediates move), GB/s on those bytes, and the share of the H100 SXM data
sheet's 3.35 TB/s HBM3 that is; the card's name and power limit are read in the same run.  Every library output is
checked bit-exact against the model (numpy float64 in the demo's order, then floor, as a table of all 2^24 triples)
on the timed inputs, and the torch lines report how many pixels differ from it.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HBM_BYTES_PER_S = 3.35e12
WORKLOADS = {"1080p": (1920, 1080, 256), "4k": (4096, 4096, 64)}


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = "unknown"
    return name, out


def model_table():
    """the demo's gray of every (r, g, b), by index (r << 16) | (g << 8) | b"""
    i = np.arange(1 << 24, dtype=np.uint32)
    v = np.multiply(0.299, (i >> 16).astype(np.uint8), dtype=np.float64)
    v = v + np.multiply(0.587, ((i >> 8) & 255).astype(np.uint8), dtype=np.float64)
    v = v + np.multiply(0.114, (i & 255).astype(np.uint8), dtype=np.float64)
    return np.floor(v).astype(np.uint8)


def median_time(fn, reps, warmup):
    """median seconds of one fn() over `reps` calls, each between its own pair of CUDA events"""
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / 1e3)
    return float(np.median(times)), float(min(times)), float(max(times))


def mismatches(gray, rgb, table):
    """pixels of gray (flat uint8) that differ from the model's gray of rgb (flat pixels x >= 3 channels)"""
    import torch
    bad, step = 0, 1 << 26
    for i in range(0, gray.numel(), step):
        p = rgb[i:i + step].to(torch.int64)
        bad += int((gray[i:i + step] != table[(p[:, 0] << 16) | (p[:, 1] << 8) | p[:, 2]]).sum())
    return bad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--workloads", default="1080p,4k")
    args = ap.parse_args()
    import torch
    from grayskull_b200 import color
    assert torch.cuda.is_available(), "the benchmark needs a CUDA device"
    lib = color.lib()
    name, power = card()
    table = torch.from_numpy(model_table()).cuda()
    for wl in args.workloads.split(","):
        w, h, n = WORKLOADS[wl]
        pixels = w * h * n
        gen = torch.Generator(device="cuda").manual_seed(1)
        rgba = torch.randint(0, 256, (pixels, 4), dtype=torch.uint8, device="cuda", generator=gen)
        gray = torch.empty(pixels, dtype=torch.uint8, device="cuda")
        s = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)   # noqa: E731

        def line(form, bpp, t, **extra):
            rec = {"workload": wl, "w": w, "h": h, "frames": n, "form": form, "median_ms": round(t[0] * 1e3, 4),
                   "min_ms": round(t[1] * 1e3, 4), "max_ms": round(t[2] * 1e3, 4), "reps": args.reps,
                   "bytes_per_pixel": bpp, "GB_per_s": round(bpp * pixels / t[0] / 1e9, 1),
                   "fraction_of_3.35TB_s": round(bpp * pixels / t[0] / HBM_BYTES_PER_S, 3),
                   "card": name, "power_limit": power}
            rec.update(extra)
            print(json.dumps(rec), flush=True)

        def rc(v):
            color.check(v, "benchmark call")

        gray.fill_(0)
        t = median_time(lambda: rc(lib.gs_b200_rgb_to_gray_batch(gray.data_ptr(), rgba.data_ptr(), w, h, n, 4, s())),
                        args.reps, args.warmup)
        bad = mismatches(gray, rgba, table)
        assert bad == 0, "RGBA -> gray: %d pixels differ from the model" % bad
        line("rgba_to_gray", 5, t, bit_exact=True)

        rgb = rgba[:, :3].contiguous()
        gray.fill_(0)
        t = median_time(lambda: rc(lib.gs_b200_rgb_to_gray_batch(gray.data_ptr(), rgb.data_ptr(), w, h, n, 3, s())),
                        args.reps, args.warmup)
        bad = mismatches(gray, rgb, table)
        assert bad == 0, "RGB -> gray: %d pixels differ from the model" % bad
        line("rgb_to_gray", 4, t, bit_exact=True)
        del rgb

        out = torch.empty_like(rgba)
        t = median_time(lambda: rc(lib.gs_b200_gray_to_rgba_batch(out.data_ptr(), gray.data_ptr(), w, h, n, s())),
                        args.reps, args.warmup)
        ok = all(torch.equal(out[:, k], gray) for k in range(3)) and bool((out[:, 3] == 255).all())
        assert ok, "gray -> RGBA differs from (g, g, g, 255)"
        line("gray_to_rgba", 5, t, bit_exact=True)
        del out

        # what a torch user writes today, on the same RGBA tensor
        for dt, label in ((torch.float32, "torch_float32"), (torch.float64, "torch_float64")):
            def expr():
                v = 0.299 * rgba[:, 0].to(dt) + 0.587 * rgba[:, 1].to(dt)
                v = v + 0.114 * rgba[:, 2].to(dt)
                return v.floor_().to(torch.uint8)
            t = median_time(expr, args.reps, args.warmup)
            got = expr()
            line(label, 5, t, mismatches=mismatches(got, rgba, table))
            del got
        del rgba, gray
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
