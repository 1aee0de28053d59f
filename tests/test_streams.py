"""Every batch entry point runs on the caller's stream and only there: ordered behind work already queued on it, with
no hidden wait on the host, correct on two streams at once, on cudaStreamPerThread from two host threads, and inside a
captured CUDA graph.

CASES is the coverage record: one row per batch entry point of include/grayskull_b200.h that takes a gs_b200_stream,
with a tiled and a generic geometry where the host code has both.  A row's spec gives its inputs for a seed, its
outputs, the call on a stream and the oracle's check (tests/_libs.py).  Seed 1 is the real input; seed 2 is the
"poison", the same op's valid inputs for another seed, so a read that is not ordered behind the copy of the real
inputs computes wrong values but never addresses out of bounds.

  * CPU: CASES names every such entry point the header declares; the census of blocking or legacy-stream runtime
    calls each object of the library imports, each with its reason.
  * GPU A: on a non-blocking stream behind a sleep, the real inputs are copied over the poison, the outputs are
    overwritten, the call is made and its outputs cloned.  Right after the call returns neither that stream nor a
    second sleeping stream may have finished, and the clones must be bit-exact.
  * GPU B: every row on two streams at once, at two geometries.
  * GPU C: cudaStreamPerThread from two host threads, ops whose scratch holds values.
  * GPU D: every row captured into a CUDA graph and replayed with new inputs and changed host parameters.
"""
import ctypes as C
import os
import re
import shutil
import subprocess
import threading
import time

import numpy as np
import pytest

import _libs as L
from _gpu import O, frames, lib  # noqa: F401

ROOT = L.ROOT
FILL = 0xA5                          # what the outputs hold before a call
SLEEP_MIN_CYCLES = 40_000_000        # ~20 ms at 1.98 GHz
SLEEP_MAX_CYCLES = 400_000_000       # ~200 ms: the bound on any one sleep
CAPTURE_UNSUPPORTED = 900            # cudaErrorStreamCaptureUnsupported


def _bump(p):
    """the second geometry of a row (part B): one more frame, two more rows"""
    q = dict(p)
    if "n" in q:
        q["n"] += 1
    if "h" in q:
        q["h"] += 2
    return q


def case(cid, fn, **p):
    """a row: id, the entry point it calls, its parameters"""
    return cid, fn, p


CASES = [
    case("blur-tma", "gs_b200_blur_batch", w=272, h=70, n=3, r=3),
    case("blur-ragged", "gs_b200_blur_batch", w=100, h=70, n=3, r=9),
    case("adaptive-tma", "gs_b200_adaptive_threshold_batch", w=272, h=70, n=3, r=3, c=2),
    case("adaptive-ragged", "gs_b200_adaptive_threshold_batch", w=100, h=70, n=3, r=5, c=-1),
    case("sobel-tma", "gs_b200_sobel_batch", w=272, h=41, n=3),
    case("sobel-ragged", "gs_b200_sobel_batch", w=100, h=37, n=3),
    case("blur_sobel-tma", "gs_b200_blur_sobel_batch", w=272, h=70, n=3, r=3),
    case("blur_sobel-staged", "gs_b200_blur_sobel_batch", w=1080, h=40, n=2, r=5),     # WS_STAGE_FUSED
    case("erode-tma", "gs_b200_erode_batch", w=272, h=41, n=3),
    case("erode-ragged", "gs_b200_erode_batch", w=100, h=37, n=3),
    case("dilate-tma", "gs_b200_dilate_batch", w=272, h=41, n=3),
    case("dilate-ragged", "gs_b200_dilate_batch", w=100, h=37, n=3),
    case("erode_n-9", "gs_b200_erode_n_batch", w=272, h=70, n=2, it=9),
    case("erode_n-17", "gs_b200_erode_n_batch", w=272, h=70, n=2, it=17),               # two composed launches
    case("erode_n-ragged", "gs_b200_erode_n_batch", w=100, h=37, n=3, it=3),            # row / column path
    case("dilate_n-9", "gs_b200_dilate_n_batch", w=272, h=70, n=2, it=9),
    case("dilate_n-ragged", "gs_b200_dilate_n_batch", w=100, h=37, n=3, it=4),
    case("resize-tiled", "gs_b200_resize_batch", w=272, h=60, n=3, dw=200, dh=50),
    case("resize-ragged", "gs_b200_resize_batch", w=100, h=37, n=3, dw=37, dh=50),
    case("downsample-vec", "gs_b200_downsample_batch", w=272, h=41, n=3),
    case("downsample-ragged", "gs_b200_downsample_batch", w=100, h=37, n=3),
    case("integral-bands", "gs_b200_integral_batch", w=40, h=17, n=3, env="bands"),
    case("integral-strips", "gs_b200_integral_batch", w=1000, h=37, n=3, env="strips"),
    case("integral-ragged", "gs_b200_integral_batch", w=100, h=37, n=3),
    case("histogram-vec", "gs_b200_histogram_batch", w=272, h=41, n=3),
    case("histogram-ragged", "gs_b200_histogram_batch", w=100, h=37, n=3),
    case("otsu-vec", "gs_b200_otsu_threshold_batch", w=272, h=41, n=3),
    case("otsu-ragged", "gs_b200_otsu_threshold_batch", w=101, h=37, n=3),
    case("threshold-vec", "gs_b200_threshold_batch", w=272, h=41, n=3, t=100),
    case("threshold-ragged", "gs_b200_threshold_batch", w=100, h=37, n=3, t=100),
    case("threshold_each-vec", "gs_b200_threshold_each_batch", w=272, h=41, n=3, offset=10),
    case("threshold_each-ragged", "gs_b200_threshold_each_batch", w=100, h=37, n=3, offset=-20),
    case("filter-3x3", "gs_b200_filter_batch", w=272, h=41, n=3, k="3x3"),
    case("filter-7x5", "gs_b200_filter_batch", w=272, h=41, n=3, k="7x5"),
    case("match_template-packed", "gs_b200_match_template_batch", w=256, h=60, n=3, tw=30, th=24),
    case("match_template-ragged", "gs_b200_match_template_batch", w=101, h=37, n=3, tw=9, th=4),
    case("find_best_match", "gs_b200_find_best_match_batch", w=101, h=37, n=3),
    case("blobs-overflow", "gs_b200_blobs_batch", w=100, h=37, n=3, nb=12),
    case("blob_corners", "gs_b200_blob_corners", w=100, h=37),
    case("perspective-host", "gs_b200_perspective_correct_batch", w=200, h=150, n=3, dw=90, dh=71, per_frame=0),
    case("perspective-per_frame", "gs_b200_perspective_correct_batch", w=200, h=150, n=3, dw=90, dh=71, per_frame=1),
    case("fast-tiled", "gs_b200_fast_batch", w=272, h=60, n=3, t=20),
    case("fast-ragged", "gs_b200_fast_batch", w=101, h=37, n=3, t=10),
    case("orb-tiled", "gs_b200_orb_extract_batch", w=272, h=60, n=3, t=20),
    case("orb-ragged", "gs_b200_orb_extract_batch", w=202, h=60, n=3, t=20),
    case("match_orb", "gs_b200_match_orb_batch", n=3),
    case("lbp-chunked", "gs_b200_lbp_detect_batch", w=136, h=130, n=3, chunk="1"),
    case("lbp-ragged", "gs_b200_lbp_detect_batch", w=130, h=130, n=2),
    case("memcpy_h2d", "gs_b200_memcpy_h2d", bytes=100003),
    case("memcpy_d2h", "gs_b200_memcpy_d2h", bytes=100003),
    case("memset", "gs_b200_memset", bytes=100003),
    case("stream_sync", "gs_b200_stream_sync"),
]

# rows whose call waits by design, with the reason; every other call must return before its stream has run it
WAITS = {"stream_sync": "gs_b200_stream_sync waits for its own stream, and only for it"}

# rows that refuse graph capture by design, with the reason; the rest must capture and replay
NO_CAPTURE = {"filter-7x5": "the generic filter copies its host weights from pageable memory, which a graph would "
                            "capture by pointer; it returns cudaErrorStreamCaptureUnsupported"}

# part C: ops whose workspace holds values only (no tickets, flags or indices a race could turn into a hang)
PER_THREAD = ("otsu-ragged", "filter-7x5", "match_template-packed", "find_best_match", "erode_n-17", "dilate_n-ragged",
              "blur_sobel-staged")


# ---- CPU -----------------------------------------------------------------------------------------------------------
def test_cases_cover_every_stream_entry_point():
    with open(os.path.join(ROOT, "include", "grayskull_b200.h")) as f:
        text = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    declared = set()
    for m in re.finditer(r"\b(gs_b200_\w+)\s*\(([^)]*)\)\s*;", text):
        if "gs_b200_stream" in m.group(2):
            declared.add(m.group(1))
    assert len(declared) >= 29, sorted(declared)
    named = {fn for _, fn, _ in CASES}
    assert declared == named, "header entry points without a row: %s; rows naming no entry point: %s" % (
        sorted(declared - named), sorted(named - declared))
    ids = [cid for cid, _, _ in CASES]
    assert len(ids) == len(set(ids))
    assert set(WAITS) | set(NO_CAPTURE) | set(PER_THREAD) <= set(ids)


# (object, runtime call) pairs that may block the host or use the legacy stream, each with its reason
BLOCKING = {
    ("api.o", "cudaMemcpy"): "single-image calls are synchronous (gs_filter / gs_perspective_correct read device "
                             "parameters back)",
    ("api.o", "cudaStreamCreate"): "single-image calls are synchronous: each host thread's own stream",
    ("api.o", "cudaStreamDestroy"): "single-image calls are synchronous: the thread's stream goes with the thread",
    ("api.o", "cudaStreamSynchronize"): "single-image calls are synchronous",
    ("fast_orb.o", "cudaMalloc"): "the once-per-process trig check on its private stream",
    ("fast_orb.o", "cudaFree"): "the once-per-process trig check on its private stream",
    ("fast_orb.o", "cudaStreamCreateWithFlags"): "the once-per-process trig check on its private stream",
    ("fast_orb.o", "cudaStreamDestroy"): "the once-per-process trig check on its private stream",
    ("fast_orb.o", "cudaStreamSynchronize"): "the once-per-process trig check on its private stream",
    ("lbp.o", "cudaMalloc"): "plan upload: a cache miss allocates the plan's tables",
    ("lbp.o", "cudaFree"): "plan upload: an evicted plan is freed once nobody holds it",
    ("lbp.o", "cudaStreamSynchronize"): "single-image gs_lbp_window stages its tables and waits",
    ("runtime.o", "cudaMalloc"): "workspace growth, and gs_b200_malloc",
    ("runtime.o", "cudaFree"): "workspace growth, and gs_b200_free / gs_b200_image_free",
    ("runtime.o", "cudaStreamSynchronize"): "workspace growth waits for the stream's use of the old arena; "
                                            "plan upload on its private stream; gs_b200_stream_sync",
    ("runtime.o", "cudaStreamCreateWithFlags"): "plan upload: the private non-blocking stream of upload()",
    ("runtime.o", "cudaStreamDestroy"): "plan upload: the private non-blocking stream of upload()",
    ("runtime.o", "cudaMallocHost"): "gs_b200_malloc_host",
    ("runtime.o", "cudaFreeHost"): "gs_b200_free_host",
    ("runtime.o", "cudaMallocManaged"): "gs_b200_alloc",
}
_BLOCKING_RE = re.compile(r"^(cudaMemcpy|cudaMemcpyToSymbol|cudaMemset|cudaMemcpy2D|cudaDeviceSynchronize|"
                          r"cudaStreamSynchronize|cudaEventSynchronize|cudaMalloc\w*|cudaFree\w*|cudaStreamCreate\w*|"
                          r"cudaStreamDestroy)$")


def test_blocking_runtime_calls_census():
    """cudart is linked statically, so each object's undefined symbols show the runtime calls the .so hides"""
    from grayskull_b200 import build
    nm = shutil.which("nm")
    if nm is None:
        pytest.skip("nm not found")
    objs = [os.path.join(build.OBJ, s.replace(".cu", ".o")) for s in build.SOURCES]
    missing = [o for o in objs if not os.path.exists(o)]
    assert not missing, "objects missing (rebuild with `python -m grayskull_b200.build --force`): %s" % missing
    found = set()
    for o in objs:
        out = subprocess.run([nm, "-u", o], capture_output=True, text=True, check=True).stdout
        for line in out.splitlines():
            sym = line.split()[-1]
            if _BLOCKING_RE.match(sym):
                found.add((os.path.basename(o), sym))
    unexplained = sorted(found - set(BLOCKING))
    assert not unexplained, "blocking or legacy-stream runtime calls without a reason: %s" % unexplained
    stale = sorted(set(BLOCKING) - found)
    assert not stale, "reasons for calls the objects no longer make: %s" % stale


# ---- GPU: the rows -------------------------------------------------------------------------------------------------
def _fr(w, h, n, seed):
    """frames; the poison seed reverses their kinds, so no frame of it equals the real one"""
    return frames(w, h, n, 1) if seed == 1 else np.ascontiguousarray(frames(w, h, n, 100 + seed)[::-1])


def _eq(got, want, what):
    assert np.array_equal(got, want), what


class Spec:
    """ins: input arrays for a seed (gen); outs: (nbytes, fill, on_host); call(in_ptrs, out_ptrs, stream) -> rc;
    check(ins, results) with results = the outputs' bytes, then those of the inputs listed in `inplace`"""

    def __init__(self, gen, outs, call, check, host_ins=(), inplace=(), mutate=None, env=None):
        self.gen, self.outs, self.call, self.check = gen, outs, call, check
        self.host_ins, self.inplace, self.mutate, self.env = set(host_ins), tuple(inplace), mutate, env or {}


def out(nbytes, fill=FILL, host=False):
    return nbytes, fill, host


def _spec(fn, p):
    import grayskull_b200 as g
    lib, Od = g.lib(), L.oracle()
    w, h, n = p.get("w"), p.get("h"), p.get("n")
    ff = lambda seed: [_fr(w, h, n, seed)]                                   # noqa: E731

    def frames_check(want_fn, shape=None):
        def check(ins, res):
            got = res[0].reshape(shape or (n, h, w))
            for i in range(n):
                _eq(got[i], want_fn(ins[0][i]), i)
        return check

    if fn in ("gs_b200_blur_batch", "gs_b200_adaptive_threshold_batch"):
        r, c = p["r"], p.get("c")
        if c is None:
            return Spec(ff, [out(n * w * h)], lambda i, o, s: lib.gs_b200_blur_batch(o[0], i[0], w, h, n, r, s),
                        frames_check(lambda a: L.o_blur(Od, a, r)))
        return Spec(ff, [out(n * w * h)],
                    lambda i, o, s: lib.gs_b200_adaptive_threshold_batch(o[0], i[0], w, h, n, r, c, s),
                    frames_check(lambda a: L.o_adaptive(Od, a, r, c)))
    if fn == "gs_b200_sobel_batch":
        return Spec(ff, [out(n * w * h)], lambda i, o, s: lib.gs_b200_sobel_batch(o[0], i[0], w, h, n, s),
                    frames_check(lambda a: L.o_sobel(Od, a, FILL)))
    if fn == "gs_b200_blur_sobel_batch":
        r = p["r"]
        return Spec(ff, [out(n * w * h)], lambda i, o, s: lib.gs_b200_blur_sobel_batch(o[0], i[0], w, h, n, r, s),
                    frames_check(lambda a: L.o_sobel(Od, L.o_blur(Od, a, r), FILL)))
    if fn in ("gs_b200_erode_batch", "gs_b200_dilate_batch", "gs_b200_erode_n_batch", "gs_b200_dilate_n_batch"):
        dil, it = "dilate" in fn, p.get("it")
        f = getattr(lib, fn)

        def want(a):
            for _ in range(it or 1):
                a = L.o_morph(Od, a, dil)
            return a
        if it is None:
            return Spec(ff, [out(n * w * h)], lambda i, o, s: f(o[0], i[0], w, h, n, s), frames_check(want))
        return Spec(ff, [out(n * w * h)], lambda i, o, s: f(o[0], i[0], w, h, n, it, s), frames_check(want))
    if fn == "gs_b200_resize_batch":
        dw, dh = p["dw"], p["dh"]
        return Spec(ff, [out(n * dw * dh)], lambda i, o, s: lib.gs_b200_resize_batch(o[0], dw, dh, i[0], w, h, n, s),
                    frames_check(lambda a: L.o_resize(Od, a, dw, dh), (n, dh, dw)))
    if fn == "gs_b200_downsample_batch":
        return Spec(ff, [out(n * (w // 2) * (h // 2))],
                    lambda i, o, s: lib.gs_b200_downsample_batch(o[0], i[0], w, h, n, s),
                    frames_check(lambda a: L.o_down(Od, a), (n, h // 2, w // 2)))
    if fn == "gs_b200_integral_batch":
        def check(ins, res):
            got = res[0].view(np.uint32).reshape(n, h, w)
            for i in range(n):
                _eq(got[i], L.o_integral(Od, ins[0][i]), i)
        return Spec(ff, [out(4 * n * w * h)], lambda i, o, s: lib.gs_b200_integral_batch(o[0], i[0], w, h, n, s),
                    check, env={"GS_B200_INTEGRAL": p["env"]} if "env" in p else None)
    if fn == "gs_b200_histogram_batch":
        def check(ins, res):
            got = res[0].view(np.uint32).reshape(n, 256)
            for i in range(n):
                _eq(got[i], np.bincount(ins[0][i].ravel(), minlength=256), i)
        return Spec(ff, [out(4 * 256 * n)], lambda i, o, s: lib.gs_b200_histogram_batch(o[0], i[0], w, h, n, s), check)
    if fn == "gs_b200_otsu_threshold_batch":
        def check(ins, res):
            for i in range(n):
                assert res[0][i] == Od.gso_otsu_threshold(L.ptr(ins[0][i]), w, h), i
        return Spec(ff, [out(n)], lambda i, o, s: lib.gs_b200_otsu_threshold_batch(o[0], None, i[0], w, h, n, s), check)
    if fn in ("gs_b200_threshold_batch", "gs_b200_threshold_each_batch"):
        each = fn.endswith("each_batch")

        def gen(seed):
            t = np.random.default_rng(seed).integers(0, 256, n).astype(np.uint8)
            return [_fr(w, h, n, seed)] + ([t] if each else [])

        def check(ins, res):
            got = res[0].reshape(n, h, w)
            for i in range(n):
                want = ins[0][i].copy()
                Od.gso_threshold(L.ptr(want), w, h, (int(ins[1][i]) + p["offset"]) & 255 if each else p["t"])
                _eq(got[i], want, i)
        if each:
            call = lambda i, o, s: lib.gs_b200_threshold_each_batch(i[0], w, h, n, i[1], p["offset"], s)  # noqa: E731
        else:
            call = lambda i, o, s: lib.gs_b200_threshold_batch(i[0], w, h, n, p["t"], s)                  # noqa: E731
        return Spec(gen, [], call, check, inplace=(0,))
    if fn == "gs_b200_filter_batch":
        if p["k"] == "3x3":
            k, norm = L.filter_kernel("sharpen")
        else:
            k = np.random.default_rng(75).integers(-8, 9, (5, 7)).astype(np.int8).view(np.uint8)
            norm = 9
        ks, k0 = np.ascontiguousarray(k), np.ascontiguousarray(k).copy()   # ks: the host weights a call reads

        def check(ins, res):
            got = res[0].reshape(n, h, w)
            for i in range(n):
                want = np.zeros((h, w), np.uint8)
                Od.gso_filter(L.ptr(want), L.ptr(ins[0][i]), w, h, L.ptr(k0), k0.shape[1], k0.shape[0], norm)
                _eq(got[i], want, i)

        def mutate():
            ks[:] = 1
        return Spec(ff, [out(n * w * h)],
                    lambda i, o, s: lib.gs_b200_filter_batch(o[0], i[0], w, h, n, ks.ctypes.data, ks.shape[1], ks.shape[0],
                                                             norm, s), check, mutate=mutate)
    if fn == "gs_b200_match_template_batch":
        tw, th = p["tw"], p["th"]
        rw, rh = w - tw + 1, h - th + 1

        def gen(seed):
            fr = _fr(w, h, n, seed)
            return [fr, np.ascontiguousarray(fr[1, 5 + seed:5 + seed + th, 10 + seed:10 + seed + tw])]

        def check(ins, res):
            got = res[0].reshape(n, rh, rw)
            for i in range(n):
                want = np.zeros((rh, rw), np.uint8)
                Od.gso_match_template(L.ptr(ins[0][i]), w, h, L.ptr(ins[1]), tw, th, L.ptr(want))
                _eq(got[i], want, i)
        return Spec(gen, [out(n * rw * rh)],
                    lambda i, o, s: lib.gs_b200_match_template_batch(o[0], i[0], w, h, n, i[1], tw, th, s), check)
    if fn == "gs_b200_find_best_match_batch":
        px = w * h

        def gen(seed):
            rng = np.random.default_rng(px + seed)
            return [(rng.integers(0, 250, (n, px)) * (rng.random((n, px)) < 0.5)).astype(np.uint8)]

        def check(ins, res):
            got = res[0].view(np.uint32).reshape(n, 2)
            for i in range(n):
                b = Od.gso_find_best_match(L.ptr(np.ascontiguousarray(ins[0][i])), w, h)
                assert tuple(got[i]) == (b % w, b // w), i
        return Spec(gen, [out(8 * n)], lambda i, o, s: lib.gs_b200_find_best_match_batch(o[0], i[0], w, h, n, s), check)
    if fn == "gs_b200_blobs_batch":
        nb = p["nb"]

        def check(ins, res):
            labels = res[0].view(np.uint16).reshape(n, h, w)
            blobs, counts = res[1].view(L.BLOB_DTYPE).reshape(n, nb), res[2].view(np.uint32)
            for i in range(n):
                wl, wb = _o_blobs(Od, ins[0][i], nb)
                assert counts[i] == len(wb) and np.array_equal(labels[i], wl), i
                assert L.blob_fields(blobs[i, :counts[i]]) == L.blob_fields(wb), i
        return Spec(lambda seed: [np.stack([L.binary_like(w, h, 50 * seed + i) for i in range(n)])],
                    [out(2 * n * w * h), out(32 * n * nb), out(4 * n)],
                    lambda i, o, s: lib.gs_b200_blobs_batch(i[0], w, h, n, o[0], o[1], o[2], nb, s), check)
    if fn == "gs_b200_blob_corners":
        def gen(seed):
            a = L.binary_like(w, h, 7 + seed)
            labels, blobs = _o_blobs(Od, a, 300)
            j = int(np.argmax(blobs["area"]))
            return [a, labels, np.ascontiguousarray(blobs[j:j + 1])]

        def check(ins, res):
            want = np.zeros((4, 2), np.uint32)
            Od.gso_blob_corners(L.ptr(ins[0]), w, h, L.ptr(ins[1]), L.ptr(ins[2]), L.ptr(want))
            _eq(res[0].view(np.uint32).reshape(4, 2), want, "corners")
        return Spec(gen, [out(32)], lambda i, o, s: lib.gs_b200_blob_corners(i[0], w, h, i[1], i[2], o[0], s), check)
    if fn == "gs_b200_perspective_correct_batch":
        dw, dh = p["dw"], p["dh"]
        q_host = np.random.default_rng(5).integers(0, 140, (4, 2)).astype(np.uint32)
        q0 = q_host.copy()

        def gen(seed):
            fr = _fr(w, h, n, seed)
            return [fr, np.random.default_rng(5 + seed).integers(0, 140, (n, 4, 2)).astype(np.uint32)] if p["per_frame"] \
                else [fr]

        def check(ins, res):
            got = res[0].reshape(n, dh, dw)
            for i in range(n):
                want = np.empty((dh, dw), np.uint8)
                q = np.ascontiguousarray(ins[1][i]) if p["per_frame"] else q0
                Od.gso_perspective_correct(L.ptr(want), dw, dh, L.ptr(ins[0][i]), w, h, L.ptr(q))
                _eq(got[i], want, i)

        def mutate():
            q_host[:] = 0
        if p["per_frame"]:
            call = lambda i, o, s: lib.gs_b200_perspective_correct_batch(o[0], dw, dh, i[0], w, h, n, i[1], 1, s)  # noqa
        else:
            call = lambda i, o, s: lib.gs_b200_perspective_correct_batch(o[0], dw, dh, i[0], w, h, n,  # noqa: E731
                                                                         q_host.ctypes.data, 0, s)
        return Spec(gen, [out(n * dw * dh)], call, check, mutate=None if p["per_frame"] else mutate)
    if fn in ("gs_b200_fast_batch", "gs_b200_orb_extract_batch"):
        orb, t, nk = "orb" in fn, p["t"], 400
        sm_fill = 0 if orb else FILL

        def gen(seed):
            fr = _fr(w, h, n, seed)
            fr[seed % n] = L.natural_like(w, h, 90 + seed)            # corners in every batch
            return [fr]

        def check(ins, res):
            sm = res[0].reshape(n, h, w)
            kps, counts = res[1].view(np.uint32).reshape(n, nk, 12), res[2].view(np.uint32)
            for i in range(n):
                so = np.full((h, w), sm_fill, np.uint8)
                want = L.o_orb(Od, ins[0][i], so, nk, t) if orb else L.o_fast(Od, ins[0][i], so, nk, t)
                got = np.ascontiguousarray(kps[i, :counts[i]]).view(L.KP_DTYPE).reshape(-1)
                assert got.tobytes() == want.tobytes(), (i, len(got), len(want))
                if not orb:
                    _eq(sm[i], so, i)
            assert counts.sum() > 0
        f = getattr(lib, fn)
        return Spec(gen, [out(n * w * h, sm_fill), out(48 * n * nk), out(4 * n)],
                    lambda i, o, s: f(i[0], w, h, n, o[0], o[1], o[2], nk, t, s), check)
    if fn == "gs_b200_match_orb_batch":
        s1, s2, mm = 130, 90, 150
        md = {"max_distance": 60.0}
        sizes = ((120, 90), (7, 0), (130, 61), (40, 75))

        def gen(seed):
            rng = np.random.default_rng(16 + seed)
            sets = [L.desc_sets(rng, *sizes[(i + seed) % 4]) for i in range(n)]
            k1, k2 = np.zeros((n, s1), L.KP_DTYPE), np.zeros((n, s2), L.KP_DTYPE)
            for i, (a, b) in enumerate(sets):
                k1[i, :len(a)], k2[i, :len(b)] = a, b
            return [k1, k2, np.array([len(a) for a, _ in sets], np.uint32), np.array([len(b) for _, b in sets], np.uint32)]

        def check(ins, res):
            counts, m = res[1].view(np.uint32), res[0].view(np.uint32).reshape(n, mm, 3)
            for i in range(n):
                want = L.o_match(Od, ins[0][i, :ins[2][i]], ins[1][i, :ins[3][i]], mm, 60.0)
                assert counts[i] == len(want) and np.ascontiguousarray(m[i, :counts[i]]).tobytes() == want.tobytes(), i

        def mutate():
            md["max_distance"] = 1.0
        return Spec(gen, [out(12 * n * mm), out(4 * n)],
                    lambda i, o, s: lib.gs_b200_match_orb_batch(i[0], i[2], s1, i[1], i[3], s2, n, o[0], o[1], mm,
                                                                md["max_distance"], s), check, mutate=mutate)
    if fn == "gs_b200_lbp_detect_batch":
        from grayskull_b200._lib import load_cascade
        cas, cas0, mr = load_cascade(), L.HostCascade(), 1000
        lena = np.load(os.path.join(ROOT, "tests", "golden", "lena_golden.npz"))["lena"]      # 128 x 128, faces found

        def gen(seed):
            fr = [np.pad(np.roll(lena, 4 * (i + seed), axis=1), ((0, h - 128), (0, w - 128)), mode="edge")
                  if (i + seed) % 2 else L.natural_like(w, h, 40 + i + 10 * seed) for i in range(n)]
            return [np.stack([L.o_integral(Od, f) for f in fr])]

        def check(ins, res):
            counts, rects = res[1].view(np.uint32), res[0].view(np.uint32).reshape(n, mr, 4)
            for i in range(n):
                want = L.o_detect(Od, cas0, ins[0][i], mr, 1.1, 1.0, 4.0, 2)
                assert np.ascontiguousarray(rects[i, :counts[i]]).tobytes() == want.tobytes(), (i, counts[i], len(want))
            assert counts.sum() > 0

        def mutate():
            cas.arrays["stage_threshold"][:] = 1e9
        return Spec(gen, [out(16 * n * mr), out(4 * n)],
                    lambda i, o, s: lib.gs_b200_lbp_detect_batch(cas.ptr, i[0], w, h, n, o[0], o[1], mr, 1.1, 1.0, 4.0,
                                                                 2, s), check, mutate=mutate,
                    env={"GS_B200_LBP_CHUNK_FRAMES": p["chunk"]} if "chunk" in p else None)
    if fn in ("gs_b200_memcpy_h2d", "gs_b200_memcpy_d2h", "gs_b200_memset"):
        nbytes = p["bytes"]
        gen = lambda seed: [np.random.default_rng(seed).integers(0, 256, nbytes).astype(np.uint8)]  # noqa: E731
        if fn == "gs_b200_memset":
            return Spec(lambda seed: [], [out(nbytes)], lambda i, o, s: lib.gs_b200_memset(o[0], 0x3C, nbytes, s),
                        lambda ins, res: _eq(res[0], np.full(nbytes, 0x3C, np.uint8), "memset"))
        h2d = fn.endswith("h2d")
        return Spec(gen, [out(nbytes, host=not h2d)], lambda i, o, s: getattr(lib, fn)(o[0], i[0], nbytes, s),
                    lambda ins, res: _eq(res[0], ins[0], fn), host_ins=(0,) if h2d else ())
    if fn == "gs_b200_stream_sync":
        return Spec(lambda seed: [], [], lambda i, o, s: lib.gs_b200_stream_sync(s), lambda ins, res: None)
    raise KeyError(fn)


def _o_blobs(Od, a, nb):
    h, w = a.shape
    labels, blobs = np.zeros((h, w), np.uint16), np.zeros(nb, L.BLOB_DTYPE)
    m = Od.gso_blobs(L.ptr(a), w, h, L.ptr(labels), L.ptr(blobs), nb)
    return labels, blobs[:m]


def _bytes(a):
    return np.frombuffer(np.ascontiguousarray(a).tobytes(), np.uint8)


class Run:
    """one row's buffers: every input on the device (or pinned, for a host input) starts as the poison; the real and
    poison inputs wait on the device, so staging either is a device copy on the stream"""

    def __init__(self, fn, p):
        import torch
        self.fn, self.p, self.spec = fn, p, _spec(fn, p)
        self.data = {seed: self.spec.gen(seed) for seed in (1, 2)}
        self.src = {seed: [torch.from_numpy(_bytes(a).copy()).cuda() for a in arrs] for seed, arrs in self.data.items()}
        self.ins = []
        for k, a in enumerate(self.src[2]):
            t = torch.empty(a.numel(), dtype=torch.uint8, pin_memory=True) if k in self.spec.host_ins else torch.empty_like(a)
            t.copy_(a)
            self.ins.append(t)
        self.outs = [torch.empty(nb, dtype=torch.uint8, pin_memory=True) if host else
                     torch.empty(nb, dtype=torch.uint8, device="cuda") for nb, _, host in self.spec.outs]
        torch.cuda.synchronize()

    def call(self, s):
        """the library call on torch stream s (None: cudaStreamPerThread) -> rc"""
        handle = C.c_void_p(2) if s is None else C.c_void_p(s.cuda_stream)
        old = {k: os.environ.get(k) for k in self.spec.env}
        os.environ.update(self.spec.env)
        try:
            return self.spec.call([t.data_ptr() for t in self.ins], [t.data_ptr() for t in self.outs], handle)
        finally:
            for k, v in old.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v

    def stage(self, s, seed):
        """enqueue on s: the inputs of `seed` over the device inputs, the fill over the device outputs (host outputs
        are filled now, on the host)"""
        import torch
        with torch.cuda.stream(s):
            for t, a in zip(self.ins, self.src[seed]):
                t.copy_(a, non_blocking=True)
            for t, (_, fill, host) in zip(self.outs, self.spec.outs):
                t.fill_(fill)

    def results(self):
        return self.outs + [self.ins[k] for k in self.spec.inplace]

    def grab(self, s):
        """enqueue on s: clones of the device results (host results are read after the sync)"""
        import torch
        with torch.cuda.stream(s):
            return [t if not t.is_cuda else t.clone() for t in self.results()]

    def verify(self, got, seed, what=""):
        res = [g.cpu().numpy() for g in got]
        try:
            self.spec.check(self.data[seed], res)
        except AssertionError as e:
            raise AssertionError("%s%s (inputs of seed %d): %s" % (self.fn, what, seed, e)) from None

    def run_sync(self, s, seed=2):
        """one plain call on s, checked: the warm-up (sizes the workspace, builds the LBP plan, the ORB tables)"""
        self.stage(s, seed)
        rc = self.call(s)
        _ok(rc, self.fn)
        s.synchronize()
        self.verify(self.results(), seed, " warm-up")


def _ok(rc, what):
    from grayskull_b200 import _lib
    _lib.check(rc, what)


def _cudart():
    for line in open("/proc/self/maps"):
        path = line.split()[-1]
        if "libcudart.so" in os.path.basename(path):
            rt = C.CDLL(path)
            rt.cudaStreamGetFlags.argtypes = [C.c_void_p, C.POINTER(C.c_uint)]
            return rt
    pytest.fail("libcudart is not loaded in this process")


def _sleep(s, cycles):
    import torch
    with torch.cuda.stream(s):
        torch.cuda._sleep(int(cycles))


def _ids(rows):
    return [pytest.param(fn, p, id=cid) for cid, fn, p in rows]


# ---- GPU A: ordered behind pending work, no hidden waits -----------------------------------------------------------
@pytest.mark.gpu
def test_side_streams_are_non_blocking(lib):
    import torch
    flags = C.c_uint(7)
    s = torch.cuda.Stream()
    assert _cudart().cudaStreamGetFlags(C.c_void_p(s.cuda_stream), C.byref(flags)) == 0
    assert flags.value == 1, "torch.cuda.Stream() is not cudaStreamNonBlocking: the legacy stream would order it"


@pytest.mark.gpu
@pytest.mark.parametrize("fn,p", _ids(CASES))
def test_ordered_and_asynchronous(lib, fn, p, request):
    import torch
    cid = request.node.callspec.id
    run, s, u = Run(fn, p), torch.cuda.Stream(), torch.cuda.Stream()
    run.run_sync(s)
    t0 = time.perf_counter()                     # the host time of a warm call
    _ok(run.call(s), fn)
    host = time.perf_counter() - t0
    s.synchronize()
    cycles = min(max(SLEEP_MIN_CYCLES, 10 * host * 1.98e9), SLEEP_MAX_CYCLES)
    _sleep(u, min(2 * cycles, SLEEP_MAX_CYCLES))   # outlasts s's sleep, so a call that waits for s alone is told apart
    _sleep(s, cycles)
    run.stage(s, 1)
    rc = run.call(s)
    s_done, u_done = s.query(), u.query()
    got = run.grab(s)
    torch.cuda.synchronize()
    _ok(rc, fn)
    if cid in WAITS:
        assert s_done and not u_done, "%s: expected to wait for its stream and only for it" % fn
    else:
        assert not s_done, "%s returned after its stream had drained: it waited for it" % fn
        assert not u_done, "%s returned after another stream had drained: it synchronised the device" % fn
    run.verify(got, 1)


@pytest.mark.gpu
def test_single_image_calls_follow_the_legacy_stream(lib):
    """INTEGRATION.md §5: work queued on the legacy stream is ordered before a single-image call on device memory"""
    import torch
    from grayskull_b200._lib import Image
    Od = L.oracle()
    w, h = 272, 70
    a = _fr(w, h, 1, 1)[0]
    src = torch.zeros((h, w), dtype=torch.uint8, device="cuda")
    dst = torch.zeros_like(src)
    real = torch.from_numpy(a).cuda()
    torch.cuda.synchronize()
    for op in ("blur", "sobel"):
        dst.fill_(FILL)
        src.zero_()
        torch.cuda.synchronize()
        stream = torch.cuda.default_stream()
        _sleep(stream, SLEEP_MIN_CYCLES)
        src.copy_(real)                           # the legacy stream: behind the sleep
        di, si = Image(w, h, dst.data_ptr()), Image(w, h, src.data_ptr())
        if op == "blur":
            lib.gs_blur(di, si, 3)
            want = L.o_blur(Od, a, 3)
        else:
            lib.gs_sobel(di, si)
            want = L.o_sobel(Od, a, FILL)
        _eq(dst.cpu().numpy(), want, op)


# ---- GPU B: two streams at once ------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("head_sleep", [False, True], ids=["interleaved", "nested"])
def test_two_streams_at_once(lib, head_sleep):
    import torch
    s0, s1 = torch.cuda.Stream(), torch.cuda.Stream()
    pairs = [(Run(fn, p), Run(fn, _bump(p))) for cid, fn, p in CASES if cid not in WAITS]
    for r0, r1 in pairs:                         # each stream's workspace sized for its own geometry
        r0.run_sync(s0)
        r1.run_sync(s1)
    if head_sleep:                               # s0's whole sequence runs while s1 is held
        _sleep(s1, SLEEP_MIN_CYCLES)
    got = []
    for r0, r1 in pairs:
        for r, s in ((r0, s0), (r1, s1)):
            r.stage(s, 1)
            _ok(r.call(s), r.fn)
            got.append((r, r.grab(s)))
    torch.cuda.synchronize()
    for k, (r, g) in enumerate(got):
        r.verify(g, 1, " on stream %d" % (k % 2))


# ---- GPU C: cudaStreamPerThread from two host threads ----------------------------------------------------------------
def _long_filter():
    """thread A's long call: a generic 9x9 filter over 64 identical 2048 x 2048 frames (256 MiB)"""
    import torch
    import grayskull_b200 as g
    w = h = 2048
    n = 64
    a = L.natural_like(w, h, 5)
    k = np.random.default_rng(9).integers(-3, 4, (9, 9)).astype(np.int8).view(np.uint8)
    k = np.ascontiguousarray(k)
    src = torch.from_numpy(a).cuda().expand(n, h, w).contiguous()
    dst = torch.empty_like(src)
    want = np.zeros_like(a)
    L.oracle().gso_filter(L.ptr(want), L.ptr(a), w, h, L.ptr(k), 9, 9, 7)
    call = lambda: g.lib().gs_b200_filter_batch(dst.data_ptr(), src.data_ptr(), w, h, n, k.ctypes.data, 9, 9, 7,  # noqa
                                                C.c_void_p(2))
    return call, dst, torch.from_numpy(want).cuda()


@pytest.mark.gpu
def test_stream_per_thread_has_per_thread_scratch(lib):
    import torch
    rows = {cid: (fn, p) for cid, fn, p in CASES}
    runs = {who: [Run(*rows[cid]) for cid in PER_THREAD] for who in "AB"}
    long_call, long_dst, long_want = _long_filter()
    staged = [[_bytes(a) for a in r.data[1]] for r in runs["B"]]
    torch.cuda.synchronize()
    a_returned, errors, got = threading.Event(), [], {}

    def sync():
        _ok(lib.gs_b200_stream_sync(C.c_void_p(2)), "gs_b200_stream_sync")

    def warm(who):
        for r in runs[who]:
            _ok(r.call(None), r.fn)
        if who == "A":
            _ok(long_call(), "long filter")
        sync()

    def thread_a():
        try:
            _ok(long_call(), "long filter")
            a_returned.set()
            sync()
        except BaseException as e:   # noqa: B036
            errors.append(e)
            a_returned.set()

    def thread_b():
        try:
            a_returned.wait(60)
            # nothing on the legacy stream from here on: it would wait for thread A's stream
            for r, host in zip(runs["B"], staged):
                for t, a in zip(r.ins, host):        # the real inputs, on this thread's stream only
                    _ok(lib.gs_b200_memcpy_h2d(t.data_ptr(), a.ctypes.data, a.nbytes, C.c_void_p(2)), "h2d")
                for t, (nb, fill, _) in zip(r.outs, r.spec.outs):
                    _ok(lib.gs_b200_memset(t.data_ptr(), fill, nb, C.c_void_p(2)), "memset")
                _ok(r.call(None), r.fn)
            sync()
            got["B"] = [[t.cpu() for t in r.results()] for r in runs["B"]]
        except BaseException as e:   # noqa: B036
            errors.append(e)

    # warm-ups run one thread after the other, so that no arena grows while the other thread's work runs
    ta = threading.Thread(target=warm, args=("A",))
    ta.start()
    ta.join()
    tb = threading.Thread(target=warm, args=("B",))
    tb.start()
    tb.join()
    long_dst.zero_()
    torch.cuda.synchronize()
    ta, tb = threading.Thread(target=thread_a), threading.Thread(target=thread_b)
    tb.start()
    ta.start()
    ta.join(120)
    tb.join(120)
    assert not ta.is_alive() and not tb.is_alive()
    if errors:
        raise errors[0]
    torch.cuda.synchronize()
    for r, g in zip(runs["B"], got["B"]):
        r.verify(g, 1, " (thread B)")
    bad = [f for f in range(long_dst.shape[0]) if not torch.equal(long_dst[f], long_want)]
    assert not bad, "thread A's filter differs from the oracle in frames %s: its scratch was not its own" % bad


# ---- GPU D: CUDA graph capture -------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("fn,p", _ids([c for c in CASES if c[0] not in WAITS]))
def test_graph_capture_and_replay(lib, fn, p, request):
    import torch
    cid = request.node.callspec.id
    run, s = Run(fn, p), torch.cuda.Stream()
    run.run_sync(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        rc = run.call(s)
    if cid in NO_CAPTURE:
        assert rc == CAPTURE_UNSUPPORTED, (rc, lib.gs_b200_last_error())
        run.run_sync(s, 1)                       # still correct uncaptured
        return
    _ok(rc, fn)
    if run.spec.mutate:
        run.spec.mutate()                        # the graph keeps the values it captured
    for seed in (1, 2):
        run.stage(s, seed)
        with torch.cuda.stream(s):
            g.replay()
        got = run.grab(s)
        s.synchronize()
        run.verify(got, seed, " replay")


@pytest.mark.gpu
def test_workspace_cannot_grow_inside_a_capture(lib):
    """a capture that would need a larger arena fails with a clear error and leaves the arena as it was"""
    import torch
    small, big = Run("gs_b200_otsu_threshold_batch", dict(w=101, h=37, n=2)), \
        Run("gs_b200_otsu_threshold_batch", dict(w=101, h=37, n=64))
    s = torch.cuda.Stream()
    small.run_sync(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        rc = big.call(s)
    assert rc == CAPTURE_UNSUPPORTED, (rc, lib.gs_b200_last_error())
    assert b"capturing" in lib.gs_b200_last_error()
    small.run_sync(s, 1)                         # the old arena still serves the small geometry
    big.run_sync(s, 1)                           # and the next uncaptured call grows it
