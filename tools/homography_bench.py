"""Time gs_b200_find_homography_batch (libgrayskull_homography.so) with CUDA events, against the Python model on one
core.

    python tools/homography_bench.py [--reps 20] [--out results.json]

  (a) 1024 frames of 300 synthetic correspondences each, half of them outliers, at 1024 and 4096 hypotheses
  (b) the orb verb's lists for 64 frames of 1920x1080 (bench.py's c3 size; the tests' textured natural_like frames):
      a 320x240 crop of each scene as the template, pyramid ORB (2500 keypoints, threshold 20, 3 levels) and match_orb
      (300 matches, distance 60) on the device, then 1024 hypotheses
  (c) the Python model of tests/test_homography.py on the host, one core, per frame of (a) at 1024 hypotheses

Each device figure is the median over --reps timed calls after 3 warm-up calls.  Tests per second count one
(hypothesis, correspondence) score each.  The FP64 share is a bound, not a reached rate: the 20 double operations of
one score (11 multiplies, 9 adds) times the tests, over the call time, over the data sheet's 34 TFLOP/s of non-tensor
FP64 for an H100 SXM at 700 W; the solves and the refit are not counted.  The card's name and power limit are read in
the same run.  Nothing is written inside the repository unless --out points there.
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

os.environ.setdefault("OMP_NUM_THREADS", "1")
os.environ.setdefault("OPENBLAS_NUM_THREADS", "1")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402

FP64_PEAK = 34e12
OPS_PER_TEST = 20


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except Exception as e:  # the figures still stand; say what could not be read
        import torch
        return torch.cuda.get_device_name(0), "unknown (%s)" % e


def timed(fn, reps):
    import torch
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times)), float(min(times)), float(max(times))


def synthetic(n, m, seed):
    """n frames of m correspondences on random similarity-plus-perspective maps, half of them moved off the map"""
    rng = np.random.default_rng(seed)
    x, y = rng.integers(0, 640, (n, m)), rng.integers(0, 480, (n, m))
    a, th = rng.uniform(0.8, 1.2, (n, 1)), rng.uniform(-0.4, 0.4, (n, 1))
    tx, ty = rng.uniform(50, 300, (n, 1)), rng.uniform(50, 300, (n, 1))
    g, h = rng.uniform(-1e-4, 1e-4, (n, 1)), rng.uniform(-1e-4, 1e-4, (n, 1))
    w = g * x + h * y + 1
    X = np.rint((a * np.cos(th) * x - a * np.sin(th) * y + tx) / w)
    Y = np.rint((a * np.sin(th) * x + a * np.cos(th) * y + ty) / w)
    bad = rng.random((n, m)) < 0.5
    X[bad], Y[bad] = rng.integers(0, 1200, bad.sum()), rng.integers(0, 1000, bad.sum())
    kp1, kp2 = np.zeros((n, m, 12), np.int32), np.zeros((n, m, 12), np.int32)
    kp1[..., 0], kp1[..., 1], kp2[..., 0], kp2[..., 1] = x, y, np.maximum(X, 0), np.maximum(Y, 0)
    mt = np.zeros((n, m, 3), np.int32)
    mt[..., 0] = mt[..., 1] = np.arange(m)
    return kp1, kp2, mt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--model-frames", type=int, default=4)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    from grayskull_b200 import api, homography, pyramid
    name, power = card()
    res = {"card": name, "power_limit": power, "rows": []}
    n, m = 1024, 300
    kp1, kp2, mt = synthetic(n, m, 1)
    d = lambda a: torch.from_numpy(a).cuda()   # noqa: E731
    k1, k2, mm = d(kp1), d(kp2), d(mt)
    cnt = torch.full((n,), m, dtype=torch.int32, device="cuda")
    for hyp in (1024, 4096):
        med, lo, hi = timed(lambda: homography.find_homography_batch(k1, cnt, k2, cnt, mm, cnt, hyp, 0, 3.0), args.reps)
        tests = n * m * hyp
        res["rows"].append({"workload": "1024 x 300 synthetic, 50 %% outliers, %d hypotheses" % hyp, "ms": med,
                            "ms_min": lo, "ms_max": hi, "tests_per_s": tests / (med * 1e-3),
                            "fp64_share_bound": tests * OPS_PER_TEST / (med * 1e-3) / FP64_PEAK})
    # (b) the orb verb's lists at c3 size
    nc, W, Hh = 64, 1920, 1080
    import _libs as L
    scenes = torch.from_numpy(np.stack([L.natural_like(W, Hh, 100 + f) for f in range(nc)])).cuda()
    tpl = scenes[:, 400:640, 800:1120].contiguous()
    tk, tc, _, _ = pyramid.orb_pyramid_batch(tpl, 2500, 20)
    sk, sc, _, _ = pyramid.orb_pyramid_batch(scenes, 2500, 20)
    om, oc = api.match_orb_batch(tk, tc, sk, sc, 300, 60.0)
    med, lo, hi = timed(lambda: homography.find_homography_batch(tk, tc, sk, sc, om, oc, 1024, 0, 3.0), args.reps)
    tests = int(oc.sum()) * 1024
    _, inl, _ = homography.find_homography_batch(tk, tc, sk, sc, om, oc, 1024, 0, 3.0)
    res["rows"].append({"workload": "orb verb lists, 64 frames of 1920x1080, 320x240 templates, 1024 hypotheses",
                        "matches_mean": float(oc.float().mean()), "inliers_mean": float(inl.float().mean()),
                        "ms": med, "ms_min": lo, "ms_max": hi, "tests_per_s": tests / (med * 1e-3),
                        "fp64_share_bound": tests * OPS_PER_TEST / (med * 1e-3) / FP64_PEAK})
    # (c) the model on one host core
    import test_homography as T
    KP, MATCH = T.KP, T.MATCH
    t0 = time.perf_counter()
    for f in range(args.model_frames):
        k1n = np.ascontiguousarray(kp1[f]).view(KP).reshape(m)
        k2n = np.ascontiguousarray(kp2[f]).view(KP).reshape(m)
        idx, P = T.correspondences(k1n, m, k2n, m, np.ascontiguousarray(mt[f]).view(MATCH).reshape(m))
        T.model_frame(idx, P, f, 1024, 0, 3.0)
    res["model_s_per_frame"] = (time.perf_counter() - t0) / args.model_frames
    print(json.dumps(res, indent=1))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)
    assert all(math.isfinite(r["ms"]) for r in res["rows"])


if __name__ == "__main__":
    main()
