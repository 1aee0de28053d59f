"""Contour tracing throughput on the device: every blob of 256 frames of 1920x1080 natural_like frames thresholded at
128 (gs_threshold: > 128 -> 255), gs_b200_blobs_batch with 1000 records per frame, then the wasm demo's start for every
blob record (gs_b200_blob_contour_starts_batch) and the trace of all of them (gs_b200_trace_contours_batch).

Prints one JSON line: blob contours/s and walk steps/s of starts + trace (CUDA events over --reps calls), the kernel
time of each call, and the GPU's name and power limit.  Walk steps are counted by the contour oracle
(tools/contour_oracle.c), which also checks the device's records, ends and visited maps on --check frames.  When oracle/_ref/libgs_ref.so is
present, the reference gs_trace_contour runs on one host core over the same lists, on the walks that end (those the
device reports as returned or open; the reference never leaves the others), for its contours/s and steps/s.

    python tools/bench_contour.py [--frames 256] [--reps 10] [--check 8]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def gpu_identity():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.TimeoutExpired):
        q = "unknown"
    return name, q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--check", type=int, default=8)
    ap.add_argument("--nblobs", type=int, default=1000)
    a = ap.parse_args()

    import torch
    import _libs as L
    import grayskull_b200 as g
    from grayskull_b200 import api, contour
    import contour_oracle

    assert torch.cuda.is_available(), "bench_contour needs a CUDA device"
    g.lib().gs_b200_set_device(0)
    w, h, n, nb = 1920, 1080, a.frames, a.nblobs
    frames = np.stack([np.where(L.natural_like(w, h, 100 + f) > 128, 255, 0).astype(np.uint8) for f in range(n)])
    src = torch.from_numpy(frames).cuda()
    labels, blobs, counts = api.blobs_batch(src, nb)
    cl = contour.lib()
    cons = torch.zeros((n, nb, 7), dtype=torch.int32, device="cuda")
    ends = torch.empty((n, nb), dtype=torch.uint8, device="cuda")
    vis = torch.zeros_like(src)
    wb = cl.gs_b200_trace_contours_work_bytes(w, h, n)
    work = torch.empty(wb, dtype=torch.uint8, device="cuda")
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: C.c_void_p(t.data_ptr())   # noqa: E731

    def starts():
        contour.check(cl.gs_b200_blob_contour_starts_batch(p(labels), w, h, n, p(blobs), p(counts), nb, p(cons), s))

    def trace():
        contour.check(cl.gs_b200_trace_contours_batch(p(src), p(vis), w, h, n, p(cons), p(counts), nb, p(ends), p(work),
                                                      wb, s))

    def timed(fn):
        fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / a.reps / 1e3

    t_starts = timed(starts)
    t_trace = timed(trace)
    # one clean pass for the outputs
    vis.zero_()
    starts()
    trace()
    torch.cuda.synchronize()
    hc = counts.cpu().numpy().astype(np.int64)
    got = cons.cpu().numpy().view(np.uint32).view(contour.CONTOUR_DTYPE).reshape(n, nb)
    got_e, got_v = ends.cpu().numpy(), vis.cpu().numpy()

    O = contour_oracle.load()
    steps, by_end = 0, np.zeros(3, np.int64)
    for f in range(n):
        k = int(hc[f])
        rec = got[f][:k].copy()
        rec["bx"] = rec["by"] = rec["bw"] = rec["bh"] = rec["length"] = 0
        v = np.zeros((h, w), np.uint8)
        e = np.zeros(k, np.uint8)
        steps += O.gso_trace_contours(L.ptr(frames[f]), L.ptr(v), w, h, L.ptr(rec), k, L.ptr(e))
        by_end += np.bincount(got_e[f][:k], minlength=3)[:3]
        if f < a.check:
            assert rec.tobytes() == got[f][:k].tobytes(), "frame %d: records differ from the oracle" % f
            assert np.array_equal(e, got_e[f][:k]) and np.array_equal(v, got_v[f]), "frame %d differs" % f
    contours_n = int(hc.sum())
    t = t_starts + t_trace
    name, limit = gpu_identity()
    out = {"metric": "blob_contours", "gpu": name, "power_limit_max_sm_clock": limit, "frames": n, "w": w, "h": h,
           "contours": contours_n, "ends_returned_open_cycle": by_end.tolist(), "walk_steps": int(steps),
           "starts_ms": round(t_starts * 1e3, 3), "trace_ms": round(t_trace * 1e3, 3),
           "contours_per_s": round(contours_n / t), "steps_per_s": round(steps / t), "checked_frames": min(a.check, n)}
    if L.have_ref():
        R = L.ref()
        R.gs_trace_contour.restype = None
        R.gs_trace_contour.argtypes = [L.Image, L.Image, C.c_void_p]
        ref_n, ref_steps, ref_t = 0, 0, 0.0
        for f in range(n):
            k = int(hc[f])
            ok = np.flatnonzero(got_e[f][:k] != contour.CYCLE)
            rec = got[f][ok].copy()
            v = np.zeros((h, w), np.uint8)
            ev = np.zeros(len(ok), np.uint8)
            ref_steps += O.gso_trace_contours(L.ptr(frames[f]), L.ptr(v), w, h, L.ptr(rec.copy()), len(ok), L.ptr(ev))
            v[:] = 0
            img = L.img(frames[f])
            vi = L.img(v)
            t0 = time.perf_counter()
            for i in range(len(ok)):
                R.gs_trace_contour(img, vi, rec[i:i + 1].ctypes.data)
            ref_t += time.perf_counter() - t0
            ref_n += len(ok)
        out.update({"ref_cpu_contours": ref_n, "ref_cpu_steps": int(ref_steps), "ref_cpu_s": round(ref_t, 3),
                    "ref_cpu_contours_per_s": round(ref_n / ref_t) if ref_t else None,
                    "ref_cpu_steps_per_s": round(ref_steps / ref_t) if ref_t else None})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
