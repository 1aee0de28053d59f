"""The annotated-picture calls (include/grayskull_draw.h) on one GPU: one JSON line per workload.

    python tools/draw_bench.py [--iters 20] [--warmup 3] [--frames 256] [--cpu-frames 2]

Workloads on 256 frames of 1920x1080:
  blobs        the records gs_b200_blobs_batch finds in a thresholded natural frame (nblobs 4096)
  blobs_rings  4096 nested boxes per frame (rings and holes): the coverage cost must not follow the boxes' areas
  keypoints    gs_b200_fast_batch at cap 5000, threshold 20, then the crosses of the top 100
  rects        100 seeded rects per frame
  matches      a 320x240 template beside each frame, 300 matches with seeded distances, top 15
Each line has the draw call's time per batch from CUDA events (the detector that made the lists is not timed), the
compulsory bytes (2 B/pixel for the same-size calls: read the frame, write it; the orb canvas writes
(tw + w) * max(th, h) and reads the frame), that bound's time at the H100 SXM data sheet's 3.35 TB/s HBM3 and the
share of it reached, the card's name and power limit read in the same run, and -- for context -- the reference CLI's
time per frame for the same verb on one host core (oracle/_ref/nanomagick_cpu, when it was built; its whole verb,
detector included, on a 1920x1080 PGM).
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
HBM_BYTES_PER_S = 3.35e12
W, H = 1920, 1080


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


def cpu_verb(args, frame, runs):
    """seconds per frame of `nanomagick_cpu <args> in.pgm out.pgm` on one host core, or None without it"""
    exe = os.path.join(ROOT, "oracle", "_ref", "nanomagick_cpu")
    if not os.path.exists(exe) or runs == 0:
        return None
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "in.pgm")
        with open(src, "wb") as f:
            f.write(b"P5\n%d %d\n255\n" % (frame.shape[1], frame.shape[0]) + frame.tobytes())
        cmd = ["taskset", "-c", "0"] if os.path.exists("/usr/bin/taskset") else []
        t0 = time.perf_counter()
        for _ in range(runs):
            subprocess.run(cmd + [exe] + args + [src, os.path.join(d, "out.pgm")], capture_output=True, timeout=600)
        return (time.perf_counter() - t0) / runs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--cpu-frames", type=int, default=2)
    a = ap.parse_args()
    import torch
    import _libs as L
    import grayskull_b200 as g
    from grayskull_b200 import api, draw
    assert torch.cuda.is_available(), "draw_bench needs a CUDA device"
    g.lib().gs_b200_set_device(0)
    name, power = card()
    n = a.frames
    rng = np.random.default_rng(0)
    nat = L.natural_like(W, H, 1)
    src = torch.from_numpy(nat).cuda().expand(n, H, W).contiguous()
    binary = torch.from_numpy(np.where(nat > 150, 255, 0).astype(np.uint8)).cuda().expand(n, H, W).contiguous()
    out = torch.empty_like(src)
    rows = []

    def row(workload, fn, bytes_, cpu_args=None, cpu_frame=None, **extra):
        t = timed(fn, a.iters, a.warmup)
        bound = bytes_ / HBM_BYTES_PER_S
        r = dict(workload=workload, frames=n, w=W, h=H, ms_per_batch=round(t * 1e3, 4),
                 gb_per_s=round(bytes_ / t / 1e9, 1), hbm_bound_ms=round(bound * 1e3, 4),
                 share_of_hbm_bound=round(bound / t, 3), device=name, power_limit=power, **extra)
        cpu = cpu_verb(cpu_args, cpu_frame, a.cpu_frames) if cpu_args else None
        r["nanomagick_cpu_ms_per_frame"] = None if cpu is None else round(cpu * 1e3, 2)
        rows.append(r)
        print(json.dumps(r), flush=True)

    same = 2.0 * n * W * H
    # blobs of a thresholded natural frame
    _, blobs, bcount = api.blobs_batch(binary, 4096)
    nb = int(bcount[0])
    row("blobs", lambda: draw.draw_blobs_batch(binary, blobs, bcount, out), same, ["blobs", "4096"],
        np.where(nat > 150, 255, 0).astype(np.uint8), blobs_per_frame=nb)
    # rings: 4096 nested boxes per frame
    k = 4096
    ring = np.zeros((k, 8), np.int32)
    i = np.arange(k)
    ring[:, 2] = (i * 3) % 500
    ring[:, 3] = (i * 5) % 500
    ring[:, 4] = W - 2 * ring[:, 2]
    ring[:, 5] = H - 2 * ring[:, 3]
    rings = torch.from_numpy(ring).cuda().expand(n, k, 8).contiguous()
    rcount = torch.full((n,), k, dtype=torch.int32, device="cuda")
    row("blobs_rings", lambda: draw.draw_blobs_batch(binary, rings, rcount, out), same, boxes_per_frame=k)
    # FAST at 5000, top 100
    _, kps, kcount = api.fast_batch(src, 5000, 20)
    row("keypoints", lambda: draw.draw_keypoints_batch(src, kps, kcount, 100, out), same, ["keypoints", "100", "20"],
        nat, keypoints_per_frame=int(kcount[0]), top=100)
    # 100 rects
    rr = np.stack([rng.integers(0, W - 100, (n, 100)), rng.integers(0, H - 100, (n, 100)),
                   rng.integers(24, 400, (n, 100)), rng.integers(24, 400, (n, 100))], -1).astype(np.int32)
    rects = torch.from_numpy(rr).cuda()
    rcnt = torch.full((n,), 100, dtype=torch.int32, device="cuda")
    small = np.ascontiguousarray(nat[:480, :640])
    row("rects", lambda: draw.draw_rects_batch(src, rects, rcnt, out), same, ["faces", "1"], small, rects_per_frame=100)
    # matches: 300 with top 15 beside a 320x240 template
    tw, th = 320, 240
    tpl = torch.from_numpy(np.ascontiguousarray(nat[100:100 + th, 200:200 + tw])).cuda()
    k1 = np.zeros((1, 2500, 12), np.int32)
    k1[0, :, 0], k1[0, :, 1] = rng.integers(0, tw, 2500), rng.integers(0, th, 2500)
    k2 = np.zeros((n, 2500, 12), np.int32)
    k2[:, :, 0], k2[:, :, 1] = rng.integers(0, W, (n, 2500)), rng.integers(0, H, (n, 2500))
    m = np.stack([rng.integers(0, 2500, (n, 300)), rng.integers(0, 2500, (n, 300)), rng.integers(20, 60, (n, 300))],
                 -1).astype(np.int32)
    k1t, k2t, mt = (torch.from_numpy(x).cuda() for x in (k1, k2, m))
    mc = torch.full((n,), 300, dtype=torch.int32, device="cuda")
    canvas = torch.empty((n, max(th, H), tw + W), dtype=torch.uint8, device="cuda")
    row("matches", lambda: draw.draw_matches_batch(src, tpl, k1t, k2t, mt, mc, 15, canvas),
        float(n) * ((tw + W) * max(th, H) + W * H), None, matches_per_frame=300, top=15, template=[tw, th])
    # a device-to-device copy of the same bytes, for the same-size calls' yardstick
    row("d2d_copy", lambda: out.copy_(src), same)


if __name__ == "__main__":
    main()
