"""Time blur r=5, blur->sobel r=5 and ORB extraction on one batch of more than 65535 frames (default 65536 frames of
272 x 64), where the dispatchers must split the batch into frame groups to stay on their tiled kernels.

    python tools/batch_limits_bench.py [--frames 65536] [--ops blur,blur_sobel,orb] [--lib path/to/libgrayskull_b200.so]

--lib times another build of the library (say, of an earlier commit) in the same way.  Prints one JSON line: the GPU,
its power limit, and per op the median of --reps timed calls (CUDA events, after a warm-up call) with the kernels the
call launched (torch.profiler, in a separate untimed call)."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=65536)
    ap.add_argument("--w", type=int, default=272)
    ap.add_argument("--h", type=int, default=64)
    ap.add_argument("--ops", default="blur,blur_sobel,orb")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--lib", default=None)
    a = ap.parse_args()
    import numpy as np
    import torch
    from grayskull_b200 import _lib
    if a.lib:
        _lib.LIB_PATH = os.path.abspath(a.lib)
    lib = _lib.lib()
    assert torch.cuda.is_available(), "needs a CUDA device"
    lib.gs_b200_set_device(0)
    from _gpu import traced
    n, w, h = a.frames, a.w, a.h
    rng = np.random.default_rng(0)
    base = torch.from_numpy(rng.integers(0, 256, (7, h, w), dtype=np.uint8)).cuda()
    src = base[torch.arange(n, device="cuda") % 7].contiguous()
    dst = torch.empty_like(src)
    nk = 64
    kps = torch.empty((n, nk, 48), dtype=torch.uint8, device="cuda")
    counts = torch.empty(n, dtype=torch.int32, device="cuda")
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    calls = {
        "blur": lambda: lib.gs_b200_blur_batch(dst.data_ptr(), src.data_ptr(), w, h, n, 5, s),
        "blur_sobel": lambda: lib.gs_b200_blur_sobel_batch(dst.data_ptr(), src.data_ptr(), w, h, n, 5, s),
        "orb": lambda: lib.gs_b200_orb_extract_batch(src.data_ptr(), w, h, n, dst.data_ptr(), kps.data_ptr(),
                                                     counts.data_ptr(), nk, 20, s),
    }
    out = {"frames": n, "w": w, "h": h, "lib": a.lib or "tree"}
    try:
        out["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                    capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out["gpu"] = torch.cuda.get_device_name(0)
    for op in a.ops.split(","):
        fn = calls[op]
        _lib.check(fn(), op)                                  # warm-up: workspace, tables, modules
        torch.cuda.synchronize()
        times = []
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            _lib.check(fn(), op)
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1))
        _, seen = traced(fn)
        out[op] = {"median_ms": round(sorted(times)[len(times) // 2], 3), "min_ms": round(min(times), 3),
                   "kernels": sorted(seen)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
