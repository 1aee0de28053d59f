"""Region-of-interest kernels (include/grayskull_b200_roi.h) on one GPU: one JSON line per workload.

    python tools/roi_bench.py [--iters 20] [--warmup 3]

Workloads, one on each side of the copy / gather choice and the detector use case between them:
  crop       a 2048^2 region at an odd offset (1027, 513) of 256 frames of 4096^2: the copy kernel; torch's strided
             copy dst.copy_(src[:, y:y+h, x:x+w]) of the same region is timed in the same run as the yardstick
  nn_whole   whole-frame nearest resize 4096^2 -> 1024^2 over the same 256 frames: the gather kernel
  chips_nn / chips_bl
             face-chip extraction: 256 frames of 1920x1080, 64 seeded regions per frame with sides 24..400 and seeded
             counts 0..64, each to 64 x 64 in nearest / bilinear mode (region lists on the device)
Each line has the kernel time per call from CUDA events, output Mpixels/s, GB/s over compulsory bytes (the output
plus the distinct source bytes the index formulas touch, computed here on the host from the regions) and that rate's
share of the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s), with the card's name and power limit read in the run.
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


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = "unknown"
    return name, out


def timed(fn, iters, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters / 1e3


def axis_nn(dim, src_dim):
    return np.unique(((np.arange(dim, dtype=np.int64) * src_dim) & 0xFFFFFFFF) // dim)


def axis_bl(dim, src_dim):
    """the taps gs_resize's fp32 formula touches on one axis (numpy float32 rounds each step like the kernel)"""
    i = np.arange(dim, dtype=np.float32)
    s = ((i + np.float32(0.5)) * np.float32(src_dim)) / np.float32(dim) - np.float32(0.5)
    s = np.maximum(np.float32(0), np.minimum(s, np.float32(src_dim) - np.float32(1)))
    i0 = s.astype(np.int64)
    return np.unique(np.concatenate([i0, np.minimum(i0 + 1, src_dim - 1)]))


def line(name, secs, out_px, compulsory, gpu, extra=None):
    d = {"workload": name, "kernel_ms": round(secs * 1e3, 4), "mpix_per_s": round(out_px / secs / 1e6, 1),
         "compulsory_bytes": int(compulsory), "gb_per_s": round(compulsory / secs / 1e9, 1),
         "hbm_share": round(compulsory / secs / HBM_BYTES_PER_S, 3), "gpu": gpu[0], "power_limit": gpu[1]}
    d.update(extra or {})
    print(json.dumps(d), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    import grayskull_b200 as g
    from grayskull_b200 import roi
    assert torch.cuda.is_available(), "roi_bench needs a CUDA device"
    g.lib().gs_b200_set_device(0)
    gpu = card()
    launches = g.lib().gs_b200_launch_count

    # ---- 256 frames of 4096^2: crop (copy kernel) and whole-frame nearest (gather kernel)
    n, w = 256, 4096
    src = torch.randint(0, 256, (n, w, w), dtype=torch.uint8, device="cuda")
    x, y, cw = 1027, 513, 2048
    out = torch.empty((n, cw, cw), dtype=torch.uint8, device="cuda")
    ref = torch.empty_like(out)
    k0 = launches()
    roi.crop_resize_batch(src, (x, y, cw, cw), cw, cw, roi.NEAREST, out=out)
    assert launches() - k0 == 1
    t_ours = timed(lambda: roi.crop_resize_batch(src, (x, y, cw, cw), cw, cw, roi.NEAREST, out=out), args.iters, args.warmup)
    t_torch = timed(lambda: ref.copy_(src[:, y:y + cw, x:x + cw]), args.iters, args.warmup)
    assert torch.equal(out, ref)
    comp = 2 * n * cw * cw
    line("crop", t_ours, n * cw * cw, comp, gpu, {"path": "k_roi_copy", "torch_copy_ms": round(t_torch * 1e3, 4),
                                                  "torch_copy_gb_per_s": round(comp / t_torch / 1e9, 1)})
    dw = 1024
    out = torch.empty((n, dw, dw), dtype=torch.uint8, device="cuda")
    t = timed(lambda: roi.crop_resize_batch(src, (0, 0, w, w), dw, dw, roi.NEAREST, out=out), args.iters, args.warmup)
    assert torch.equal(out, src[:, ::4, ::4])
    comp = n * dw * dw + n * len(axis_nn(dw, w)) ** 2
    line("nn_whole", t, n * dw * dw, comp, gpu, {"path": "k_roi_gather<0>"})
    del src, out, ref
    torch.cuda.empty_cache()

    # ---- face chips: 256 frames of 1920x1080, 64 regions each, to 64 x 64
    n, fw, fh, mr, d = 256, 1920, 1080, 64, 64
    rng = np.random.default_rng(7)
    side_w, side_h = rng.integers(24, 401, (n, mr)), rng.integers(24, 401, (n, mr))
    rects = np.zeros((n, mr, 4), np.int64)
    rects[..., 2], rects[..., 3] = side_w, side_h
    rects[..., 0] = rng.integers(0, fw - side_w + 1)
    rects[..., 1] = rng.integers(0, fh - side_h + 1)
    counts = rng.integers(0, mr + 1, n)
    src = torch.randint(0, 256, (n, fh, fw), dtype=torch.uint8, device="cuda")
    R = torch.from_numpy(rects.astype(np.int32)).cuda()
    N = torch.from_numpy(counts.astype(np.int32)).cuda()
    out = torch.empty((n, mr, d, d), dtype=torch.uint8, device="cuda")
    slots = int(counts.sum())
    for mode, name, axis in ((roi.NEAREST, "chips_nn", axis_nn), (roi.BILINEAR, "chips_bl", axis_bl)):
        touched = 0
        mask = np.zeros((fh, fw), bool)
        for f in range(n):
            mask[:] = False
            for k in range(counts[f]):
                rx, ry, rw, rh = (int(v) for v in rects[f, k])
                mask[np.ix_(ry + axis(d, rh), rx + axis(d, rw))] = True
            touched += int(mask.sum())
        t = timed(lambda: roi.rois_resize_batch(src, R, N, d, d, mode, out=out), args.iters, args.warmup)
        line(name, t, slots * d * d, slots * d * d + touched, gpu,
             {"path": "k_roi_gather<%d>" % mode, "slots": slots, "frames": n})


if __name__ == "__main__":
    main()
