"""Pyramid ORB (include/grayskull_b200_pyramid.h) on one GPU: one JSON line per workload.

    python tools/orb_pyramid_bench.py [--workload fhd|vga|all] [--steps 10] [--warmup 2] [--check 3] [--cpu-frames 2]

Workloads (nkps 2500, threshold 20, 3 levels: the reference CLI's orb verb parameters):
  fhd   1024 frames of 1920x1080 blurred noise (bench.py c3's inputs: torch.randint, then gs_blur r = 3)
  vga   256 frames of 640x480 of the same kind (the size the reference CLI's faces verb caps itself at; the template
        and the scene of its orb verb both fit its 1 MiB buffer there)
Each line has the time per batch from CUDA events (mean and best of --steps), level-0 Mpixels/s, the library's launches
per call (gs_b200_launch_count), the per-kernel split of one call under torch.profiler, the card's name and power limit
read in the run, the outputs of the last timed call checked bit for bit against the test suite's restatement on
--check sampled frames, and that restatement's time per frame on one host core (C oracle) for --cpu-frames frames.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time
from collections import defaultdict

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
WORKLOADS = {"fhd": (1920, 1080, 1024), "vga": (640, 480, 256)}
NKPS, THRESH, LEVELS = 2500, 20, 3


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = "unknown"
    return name, out


def run(wl, steps, warmup, check, cpu_frames):
    import torch
    from torch.profiler import ProfilerActivity, profile
    import grayskull_b200 as g
    from grayskull_b200 import api, pyramid
    import _libs as L
    import test_orb_pyramid as T

    w, h, n = WORKLOADS[wl]
    g.lib().gs_b200_set_device(0)
    gen = torch.Generator(device="cuda").manual_seed(3)
    noise = torch.randint(0, 256, (n, h, w), dtype=torch.uint8, device="cuda", generator=gen)
    src = api.blur_batch(noise, 3)
    del noise
    sizes = pyramid.level_sizes(w, h, LEVELS)
    nmaps = sum(a * b for a, b in sizes) * n
    maps0 = torch.zeros(nmaps, dtype=torch.uint8, device="cuda")
    sm = torch.empty_like(maps0)
    pyr = torch.empty(sum(a * b for a, b in sizes[1:]) * n, dtype=torch.uint8, device="cuda")
    kps = torch.empty((n, NKPS, 12), dtype=torch.int32, device="cuda")
    counts = torch.empty(n, dtype=torch.int32, device="cuda")
    lp = pyramid.lib()
    s = torch.cuda.current_stream()

    def call():
        sm.copy_(maps0)          # the score maps start zeroed every call, as a fresh buffer would
        rc = lp.gs_b200_orb_pyramid_batch(src.data_ptr(), w, h, n, LEVELS, pyr.data_ptr(), sm.data_ptr(),
                                          kps.data_ptr(), counts.data_ptr(), NKPS, THRESH, C.c_void_p(s.cuda_stream))
        assert rc == 0, g.lib().gs_b200_last_error()

    for _ in range(warmup):
        call()
    torch.cuda.synchronize()
    times = []
    l0 = g.lib().gs_b200_launch_count()
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        call()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    launches = (g.lib().gs_b200_launch_count() - l0) / steps
    got_counts, got_kps = counts.cpu().numpy(), kps.cpu().numpy()
    got_pyr, got_sm = pyr.cpu().numpy(), sm.cpu().numpy()
    # the score-map reset (a torch copy) is inside the events: time it alone and report the call without it
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        sm.copy_(maps0)
    e1.record()
    e1.synchronize()
    reset_ms = e0.elapsed_time(e1) / steps
    call_ms = [t - reset_ms for t in times]

    # the last timed call's outputs against the restatement on sampled frames
    Od = L.oracle()
    rng = np.random.default_rng(0)
    sample = sorted(set([0, n - 1] + [int(v) for v in rng.integers(0, n, max(check - 2, 0))]))[:max(check, 1)]
    starts = np.cumsum([0] + [a * b * n for a, b in sizes])
    pstarts = np.cumsum([0] + [a * b * n for a, b in sizes[1:]])
    ok = True
    for f in sample:
        a = src[f].cpu().numpy()
        want = T.expected(Od, a[None], NKPS, THRESH, LEVELS, np.zeros(nmaps // n, np.uint8))
        ok &= int(got_counts[f]) == len(want[0][0])
        ok &= got_kps[f].view(np.uint8).reshape(-1)[:len(want[0][0]) * 48].tobytes() == want[0][0].tobytes()
        for lv, (lw, lh) in enumerate(sizes):
            ok &= np.array_equal(got_sm[starts[lv] + f * lw * lh:starts[lv] + (f + 1) * lw * lh],
                                 want[2][starts[lv] // n:starts[lv] // n + lw * lh])
            if lv:
                ok &= np.array_equal(got_pyr[pstarts[lv - 1] + f * lw * lh:pstarts[lv - 1] + (f + 1) * lw * lh],
                                     want[1][pstarts[lv - 1] // n:pstarts[lv - 1] // n + lw * lh])

    # the host restatement (C oracle, one core) on a few frames
    cpu_s = []
    for f in sample[:cpu_frames]:
        a = src[f].cpu().numpy()
        buf = np.zeros(T.layout(w, h, LEVELS)[3], np.uint8)
        t0 = time.perf_counter()
        T.pyramid_orb(Od, a, NKPS, THRESH, buf, LEVELS)
        cpu_s.append(time.perf_counter() - t0)

    # per-kernel split of one call
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    split = defaultdict(float)
    for e in prof.events():
        if e.device_type.name == "CUDA":
            split[e.name.split("(")[0].replace("void ", "")[:60]] += e.device_time_total / 1e3
    split = dict(sorted(((k, round(v, 3)) for k, v in split.items()), key=lambda kv: -kv[1]))

    name, power = card()
    mean, best = float(np.mean(call_ms)), float(np.min(call_ms))
    return {"workload": "%s: pyramid ORB nkps=%d t=%d levels=%d, %dx%d blurred noise, batch %d" % (
                wl, NKPS, THRESH, LEVELS, w, h, n),
            "ms_per_batch_mean": round(mean, 3), "ms_per_batch_best": round(best, 3),
            "level0_mpix_per_s": round(w * h * n / (mean * 1e-3) / 1e6, 1),
            "launches_per_call": launches, "levels_run": len(sizes),
            "mean_keypoints_per_frame": float(got_counts.mean()),
            "checked_frames": sample, "bit_exact": bool(ok),
            "host_restatement_ms_per_frame_one_core": round(1e3 * float(np.mean(cpu_s)), 1) if cpu_s else None,
            "host_cores": os.cpu_count(),
            "profile_ms_per_kernel": split, "score_map_reset_ms_excluded": round(reset_ms, 3),
            "card": name, "power_limit": power}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="all", choices=["fhd", "vga", "all"])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--check", type=int, default=3)
    ap.add_argument("--cpu-frames", type=int, default=2)
    args = ap.parse_args()
    for wl in (["fhd", "vga"] if args.workload == "all" else [args.workload]):
        print(json.dumps(run(wl, args.steps, args.warmup, args.check, args.cpu_frames)), flush=True)


if __name__ == "__main__":
    main()
