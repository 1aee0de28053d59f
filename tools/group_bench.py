"""Time gs_b200_group_rects_batch (libgrayskull_group.so) with CUDA events, against the numpy model on one core.

    python tools/group_bench.py [--reps 20] [--model-frames 32] [--out results.json]

  (a) the detector's lists for 256 c4 frames: 3840x2160 blurred noise (gs_blur r=3 of uniform u8, as bench.py's c4),
      frontalface with scale factor 1.1, scales 1..4, step 2 and max_rects 65536; grouped with K = 3, eps = 0.2
  (b) 64 frames of 65536 synthetic clustered records (2048 clusters of 32 jittered windows each, in random order);
      grouped with K = 3, eps = 0.2
  (c) the numpy model of tests/test_group.py on the host, one core, over the first --model-frames lists of (a); the
      figure for 256 frames is that time scaled by 256 / --model-frames, and the copy of the lists to the host is not
      counted

Each device figure is the median over --reps timed calls after 3 warm-up calls, with the minimum and maximum beside it.
The card's name and power limit are read in the same run.  Nothing is written inside the repository unless --out
points there.
"""
import argparse
import json
import os
import subprocess
import sys
import time

os.environ.setdefault("OMP_NUM_THREADS", "1")
os.environ.setdefault("OPENBLAS_NUM_THREADS", "1")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402


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
    return {"median_ms": float(np.median(times)), "min_ms": min(times), "max_ms": max(times), "reps": reps}


def grouping(rects, counts, k, eps):
    """a zero-argument call of the device grouping on preallocated outputs and workspace"""
    import ctypes as C
    import torch
    from grayskull_b200 import group
    n, stride = rects.shape[0], rects.shape[1]
    out = torch.empty((n, stride, 4), dtype=torch.int32, device="cuda")
    weights = torch.empty((n, stride), dtype=torch.int32, device="cuda")
    oc = torch.empty((n,), dtype=torch.int32, device="cuda")
    wb = group.work_bytes(stride, n)
    work = torch.empty(wb, dtype=torch.uint8, device="cuda")
    lib = group.lib()

    def call():
        group.check(lib.gs_b200_group_rects_batch(rects.data_ptr(), None if counts is None else counts.data_ptr(),
                                                  stride, n, k, eps, out.data_ptr(), weights.data_ptr(), oc.data_ptr(),
                                                  stride, work.data_ptr(), wb,
                                                  C.c_void_p(torch.cuda.current_stream().cuda_stream)), "bench")
    return call, oc


def synthetic(n, stride, seed):
    rng = np.random.default_rng(seed)
    per = 32
    nc = stride // per
    cx = rng.integers(0, 60000, (n, nc, 1))
    cy = rng.integers(0, 60000, (n, nc, 1))
    cs = rng.integers(24, 200, (n, nc, 1))
    d = (rng.integers(-100, 101, (n, nc, per)) * cs) // 1000
    x = cx + (rng.integers(-100, 101, (n, nc, per)) * cs) // 1000
    y = cy + (rng.integers(-100, 101, (n, nc, per)) * cs) // 1000
    r = np.stack([x, y, cs + d, cs + d], -1).reshape(n, stride, 4)
    for f in range(n):
        r[f] = r[f][rng.permutation(stride)]
    return r.astype(np.uint32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--model-frames", type=int, default=32)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import grayskull_b200 as g
    from grayskull_b200 import api
    from test_group import model_frame
    g.lib().gs_b200_set_device(0)
    name, power = card()
    res = {"card": name, "power_limit": power, "k": 3, "eps": 0.2}

    # (a) the detector's lists for 256 c4 frames
    n, h, w = 256, 2160, 3840
    cas = g.load_cascade()
    gen = torch.Generator(device="cuda").manual_seed(0)
    noise = torch.randint(0, 256, (n, h, w), dtype=torch.uint8, device="cuda", generator=gen)
    src = api.blur_batch(noise, 3)
    del noise
    ii = api.integral_batch(src)
    del src
    rects, counts = api.lbp_detect_batch(cas, ii, 65536, 1.1, 1.0, 4.0, 2)
    del ii
    torch.cuda.synchronize()
    cn = counts.cpu().numpy()
    call, oc = grouping(rects, counts, 3, 0.2)
    res["a_c4_lists"] = dict(timed(call, args.reps), frames=n, windows_total=int(cn.sum()), windows_max=int(cn.max()),
                             groups_total=int(oc.cpu().numpy().sum()))
    print("(a) 256 c4 frames: %s" % res["a_c4_lists"], flush=True)

    # (c) the numpy model on one core over the first frames of (a)
    rn = rects.cpu().numpy().view(np.uint32)
    m = min(args.model_frames, n)
    t0 = time.perf_counter()
    for f in range(m):
        model_frame(np.ascontiguousarray(rn[f, :cn[f]]).view(g.RECT_DTYPE).reshape(-1), 3, 0.2, 65536)
    dt = time.perf_counter() - t0
    res["c_numpy_model"] = {"frames_timed": m, "ms_per_frame": 1e3 * dt / m, "ms_for_256_frames": 1e3 * dt / m * 256}
    print("(c) numpy model: %s" % res["c_numpy_model"], flush=True)
    del rects, counts, call, oc
    torch.cuda.empty_cache()

    # (b) 64 frames of 65536 synthetic clustered records
    r = torch.from_numpy(synthetic(64, 65536, 1).view(np.int32)).cuda()
    call, oc = grouping(r, None, 3, 0.2)
    res["b_synthetic_65536"] = dict(timed(call, max(3, args.reps // 4)), frames=64, records_per_frame=65536,
                                    groups_total=int(oc.cpu().numpy().sum()))
    print("(b) 64 x 65536 synthetic: %s" % res["b_synthetic_65536"], flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
