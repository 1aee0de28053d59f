"""The largest-blob pick and batched blob corners (include/grayskull_corners.h) on one GPU: one JSON line per workload.

    python tools/corners_bench.py [--reps 10] [--warmup 2] [--workloads w1,w2,w3] [--out FILE]

Workloads, all seeded and synthetic:
  w1  scanner: 256 frames of 2048x2048, each a noisy bright quadrilateral over about 70 % of a dark noisy frame, taken
      through blur 1 / Otsu + 10 / blobs(1000) as gsb_magick's scan stage does.  Timed: the new pick + corners calls,
      the path they replace (D2H of the counts and records, the pick on the host, n H2D copies of the picks and n
      gs_b200_blob_corners launches, as the scan stage did), and the whole scan chain through the perspective warp.
  w2  ArUco-like: 256 frames of 1024x1024 with 150 records each, squares of mixed sizes plus one frame-sized
      background record.  Timed: the corners of every record.
  w3  many records: 64 frames of 512x512 checkerboard-like content (a 1-px checkerboard with 3 % of its pixels
      flipped), gs_blobs' list at its 65534 cap.  Timed: the corners of every record.
Each timing is the median over `reps` runs after `warmup` runs, the old and new paths alternated run by run; device
work is timed with CUDA events, and the old path (which waits on the host in the middle) with a host clock between
device synchronisations.  For w1 and w2 the line also has the bytes the corners must read (the used records' boxes
clipped to the frame, 1 byte of img and 2 of labels per pixel, computed from the records on the host) and the time
those bytes take at the H100 SXM data sheet's 3.35 TB/s, named hbm_floor_ms.  The outputs of the old and new paths are
compared on the timed inputs (w3: on its first and last frames, as the old path is one launch per record).  The card's
name and power limit are read in the same run.
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


def _s():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def event_ms(fn):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def host_ms(fn):
    import torch
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3


def alternate(paths, reps, warmup):
    """{name: (timer, fn)} run in turn `warmup` times, then `reps` times timed -> {name: median ms}"""
    for _ in range(warmup):
        for timer, fn in paths.values():
            fn()
    import torch
    torch.cuda.synchronize()
    times = {k: [] for k in paths}
    for _ in range(reps):
        for k, (timer, fn) in paths.items():
            times[k].append(timer(fn))
    return {k: float(np.median(v)) for k, v in times.items()}


def box_bytes(blobs, counts, w, h):
    """1 + 2 bytes for every pixel of every used record's box clipped to the frame (the reference's 32-bit ends)"""
    b = blobs.astype(np.int64)                                    # (n, stride, 8) record words
    bx, by, bw, bh = b[..., 2], b[..., 3], b[..., 4], b[..., 5]
    xe, ye = (bx + bw) & 0xFFFFFFFF, (by + bh) & 0xFFFFFFFF
    cw = np.where((xe < bx) | (bx >= w), 0, np.minimum(xe, w) - bx)
    ch = np.where((ye < by) | (by >= h), 0, np.minimum(ye, h) - by)
    used = np.arange(blobs.shape[1])[None, :] < np.minimum(counts, blobs.shape[1])[:, None]
    return int((cw * ch * used).sum()) * 3


def scanner_frames(n, w, h, seed):
    """noisy dark frames with a noisy bright quadrilateral over about 70 % of each"""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    frames = torch.randint(0, 70, (n, h, w), dtype=torch.uint8, device="cuda", generator=g)
    yy = torch.arange(h, device="cuda", dtype=torch.float32).view(1, h, 1)
    xx = torch.arange(w, device="cuda", dtype=torch.float32).view(1, 1, w)
    j = (torch.rand((n, 4, 2), device="cuda", generator=g) - 0.5) * 0.08
    base = torch.tensor([[0.08, 0.08], [0.92, 0.06], [0.93, 0.92], [0.07, 0.93]], device="cuda")
    q = (base + j) * torch.tensor([w, h], device="cuda", dtype=torch.float32)
    inside = torch.ones((n, h, w), dtype=torch.bool, device="cuda")
    for i in range(4):
        x0, y0 = q[:, i, 0].view(n, 1, 1), q[:, i, 1].view(n, 1, 1)
        x1, y1 = q[:, (i + 1) % 4, 0].view(n, 1, 1), q[:, (i + 1) % 4, 1].view(n, 1, 1)
        inside &= (x1 - x0) * (yy - y0) - (y1 - y0) * (xx - x0) >= 0
    bright = torch.randint(170, 256, (n, h, w), dtype=torch.uint8, device="cuda", generator=g)
    return torch.where(inside, bright, frames)


_pinned = {}


def old_corners(G, bin_, labels, blobs, counts, corners, pick):
    """the scan stage's former path: records to the host, the pick there, one copy and one launch per frame (the
    pinned host buffers are allocated once, outside the timing)"""
    import torch
    n, h, w = bin_.shape
    nb = blobs.shape[1]
    if not _pinned:
        _pinned.update(hc=torch.empty(n, dtype=torch.int32, pin_memory=True),
                       hb=torch.empty((n, nb, 8), dtype=torch.int32, pin_memory=True),
                       hp=torch.zeros((n, 8), dtype=torch.int32, pin_memory=True))
    hc, hb, hp = _pinned["hc"], _pinned["hb"], _pinned["hp"]
    lib = G.lib()
    s = _s()
    assert lib.gs_b200_memcpy_d2h(hc.data_ptr(), counts.data_ptr(), 4 * n, s) == 0
    assert lib.gs_b200_memcpy_d2h(hb.data_ptr(), blobs.data_ptr(), 32 * nb * n, s) == 0
    torch.cuda.current_stream().synchronize()
    c, area = hc.numpy(), hb.numpy()[:, :, 1].view(np.uint32).astype(np.int64)
    # the scan loop's strict >, first record on ties: argmax over the used records (the others masked below 0)
    area = np.where(np.arange(nb)[None, :] < c[:, None], area, -1)
    largest = area.argmax(1)
    hp.numpy()[c > 0] = hb.numpy()[np.arange(n), largest][c > 0]
    for f in range(n):
        fb = w * h * f
        assert lib.gs_b200_memcpy_h2d(pick.data_ptr() + 32 * f, hp.data_ptr() + 32 * f, 32, s) == 0
        assert lib.gs_b200_blob_corners(bin_.data_ptr() + fb, w, h, labels.data_ptr() + 2 * fb,
                                        pick.data_ptr() + 32 * f, corners.data_ptr() + 32 * f, s) == 0
    return hp


def w1(args, G, K):
    import torch
    n, w, h = 256, 2048, 2048
    src = scanner_frames(n, w, h, 1)
    bin_ = G.blur_batch(src, 1)
    th = torch.empty(n, dtype=torch.uint8, device="cuda")
    lib = G.lib()
    assert lib.gs_b200_otsu_threshold_batch(th.data_ptr(), None, bin_.data_ptr(), w, h, n, _s()) == 0
    assert lib.gs_b200_threshold_each_batch(bin_.data_ptr(), w, h, n, th.data_ptr(), 10, _s()) == 0
    labels, blobs, counts = G.blobs_batch(bin_, 1000)
    pick = torch.empty((n, 1, 8), dtype=torch.int32, device="cuda")
    new_c = torch.empty((n, 1, 4, 2), dtype=torch.int32, device="cuda")
    old_c = torch.empty_like(new_c)
    old_pick = torch.empty_like(pick)
    kl = K.lib()

    def new():
        assert kl.gs_b200_largest_blob_batch(blobs.data_ptr(), counts.data_ptr(), 1000, n, 0, pick.data_ptr(), None,
                                             _s()) == 0
        assert kl.gs_b200_blob_corners_batch(bin_.data_ptr(), w, h, n, labels.data_ptr(), pick.data_ptr(), None, 1,
                                             new_c.data_ptr(), _s()) == 0

    out = torch.empty((n, 1000, 800), dtype=torch.uint8, device="cuda")

    def chain():
        b = G.blur_batch(src, 1)
        assert lib.gs_b200_otsu_threshold_batch(th.data_ptr(), None, b.data_ptr(), w, h, n, _s()) == 0
        assert lib.gs_b200_threshold_each_batch(b.data_ptr(), w, h, n, th.data_ptr(), 10, _s()) == 0
        lb, bl, ct = G.blobs_batch(b, 1000)
        pk, _ = K.largest_blob_batch(bl, ct, 0)
        cs = K.blob_corners_batch(b, lb, pk)
        G.perspective_correct_batch(src, 800, 1000, cs.view(n, 4, 2), out=out)

    t = alternate({"new": (event_ms, new), "old": (host_ms, lambda: old_corners(G, bin_, labels, blobs, counts,
                                                                                   old_c, old_pick)),
                   "chain": (event_ms, chain)}, args.reps, args.warmup)
    same = bool(torch.equal(new_c, old_c)) and bool(torch.equal(pick, old_pick))
    nbytes = box_bytes(pick.cpu().numpy().view(np.uint32), np.ones(n, np.int64), w, h)
    hc = counts.cpu().numpy()
    return {"workload": "w1 scanner", "frames": n, "w": w, "h": h, "records_per_frame_mean": float(hc.mean()),
            "new_ms": t["new"], "new_launches": 4, "old_ms": t["old"],
            "old_launches": n, "old_copies": 2 + n, "old_host_syncs": 1, "speedup": t["old"] / t["new"],
            "chain_ms": t["chain"], "box_bytes": nbytes, "hbm_floor_ms": nbytes / HBM_BYTES_PER_S * 1e3,
            "new_share_of_hbm_floor": nbytes / HBM_BYTES_PER_S * 1e3 / t["new"], "outputs_equal": same}


def w2_inputs(n, w, h, stride, seed):
    rng = np.random.default_rng(seed)
    frames = ((rng.random((n, h, w)) < 0.02) * 140).astype(np.uint8)
    labels = (frames > 0).astype(np.uint16)
    blobs = np.zeros((n, stride, 8), np.uint32)
    for f in range(n):
        blobs[f, 0] = (1, w * h, 0, 0, w, h, w // 2, h // 2)
        for k in range(1, stride):
            s = int(rng.choice([3, 6, 12, 24, 48, 96, 200]))
            x, y = int(rng.integers(0, w - s)), int(rng.integers(0, h - s))
            frames[f, y:y + s, x:x + s] = 255
            frames[f, y + s // 3, x:x + s] = 90
            labels[f, y:y + s, x:x + s] = k + 1
            blobs[f, k] = (k + 1, s * s, x, y, s, s, x + s // 2, y + s // 2)
    return frames, labels, blobs


def per_record_old(G, img, labels, blobs, counts, frames_idx):
    """gs_b200_blob_corners once per record of the listed frames -> {f: (used, 4, 2) points}"""
    import torch
    n, h, w = img.shape
    stride = blobs.shape[1]
    out = torch.empty((n, stride, 4, 2), dtype=torch.int32, device="cuda")
    hc = counts.cpu().numpy() if counts is not None else np.full(n, stride)
    for f in frames_idx:
        fb = w * h * f
        for k in range(min(int(hc[f]), stride)):
            assert G.lib().gs_b200_blob_corners(img.data_ptr() + fb, w, h, labels.data_ptr() + 2 * fb,
                                                blobs.data_ptr() + 32 * (f * stride + k),
                                                out.data_ptr() + 32 * (f * stride + k), _s()) == 0
    torch.cuda.synchronize()
    return {f: out[f, :min(int(hc[f]), stride)] for f in frames_idx}


def records_workload(args, G, K, name, img, labels, blobs, counts, check_frames, with_bytes):
    import torch
    n, h, w = img.shape
    stride = blobs.shape[1]
    got = torch.empty((n, stride, 4, 2), dtype=torch.int32, device="cuda")
    kl = K.lib()
    cp = None if counts is None else counts.data_ptr()

    def new():
        assert kl.gs_b200_blob_corners_batch(img.data_ptr(), w, h, n, labels.data_ptr(), blobs.data_ptr(), cp, stride,
                                             got.data_ptr(), _s()) == 0

    t = alternate({"new": (event_ms, new)}, args.reps, args.warmup)
    old = per_record_old(G, img, labels, blobs, counts, check_frames)
    same = all(bool(torch.equal(got[f, :len(v)], v)) for f, v in old.items())
    hc = counts.cpu().numpy() if counts is not None else np.full(n, stride)
    line = {"workload": name, "frames": n, "w": w, "h": h, "stride": stride, "records": int(np.minimum(hc, stride).sum()),
            "new_ms": t["new"], "new_launches": 3, "old_launches_would_be": int(np.minimum(hc, stride).sum()),
            "outputs_equal_on_frames": check_frames if len(check_frames) < n else "all", "outputs_equal": same}
    if with_bytes:
        nb = box_bytes(blobs.cpu().numpy().view(np.uint32), hc, w, h)
        line.update({"box_bytes": nb, "hbm_floor_ms": nb / HBM_BYTES_PER_S * 1e3,
                     "new_share_of_hbm_floor": nb / HBM_BYTES_PER_S * 1e3 / t["new"]})
    return line


def w2(args, G, K):
    import torch
    n, w, h, stride = 256, 1024, 1024, 150
    frames, labels, blobs = w2_inputs(n, w, h, stride, 2)
    img = torch.from_numpy(frames).cuda()
    lab = torch.from_numpy(labels.view(np.int16)).cuda()
    bl = torch.from_numpy(blobs.view(np.int32)).cuda()
    return records_workload(args, G, K, "w2 aruco-like", img, lab, bl, None, list(range(n)), True)


def w3(args, G, K):
    import torch
    n, w, h = 64, 512, 512
    rng = np.random.default_rng(3)
    board = (np.indices((h, w)).sum(0) % 2).astype(bool)
    frames = np.stack([(board ^ (rng.random((h, w)) < 0.03)) * 255 for _ in range(n)]).astype(np.uint8)
    img = torch.from_numpy(frames).cuda()
    labels, blobs, counts = G.blobs_batch(img, 65534)
    return records_workload(args, G, K, "w3 many records", img, labels, blobs, counts, [0, n - 1], False)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--workloads", default="w1,w2,w3")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("corners_bench needs a CUDA device")
    import grayskull_b200 as g
    from grayskull_b200 import api as G, corners as K
    g.lib().gs_b200_set_device(0)
    name, power = card()
    lines = []
    for wl in args.workloads.split(","):
        line = {"w1": w1, "w2": w2, "w3": w3}[wl](args, G, K)
        line.update({"gpu": name, "power_limit": power, "reps": args.reps, "warmup": args.warmup})
        print(json.dumps(line), flush=True)
        lines.append(line)
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(json.dumps(x) for x in lines) + "\n")


if __name__ == "__main__":
    main()
