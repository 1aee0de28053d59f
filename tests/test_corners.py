"""The largest-blob pick and batched blob corners on the device (include/grayskull_corners.h, libgrayskull_corners.so).

On the CPU a numpy model of both rules is pinned against the compiled reference (oracle/_ref/libgs_ref.so: gs_blobs and
gs_blob_corners; skipped when it was not built) and the oracle's gso_blob_corners, and the companion is checked as a
library.  On the GPU both calls are checked against the model with poisoned outputs and the bytes outside every written
slot, with the kernels each case launched; then past 65535 frames, past 4 GiB and on frames taller than 65535 row
tiles, on the caller's stream, two streams and a CUDA graph, through the scanner chain against the oracle chain, and
through gsb_magick's scan stage on the reference's own scanner images (tests/golden/scan_*_golden.npz).
"""
import ctypes as C
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

import _libs as L
from _gpu import Region, lib, traced, witness, witnessed  # noqa: F401

ROOT = L.ROOT
M32 = 0xFFFFFFFF
INT_MAX, INT_MIN = 2 ** 31 - 1, -2 ** 31
BIG = 1 << 40

# every kernel of libgrayskull_corners.so, and which call launches it
KERNELS = {
    "gsb::k_largest_blob": "pick",
    "gsb::k_corners_small": "corners",
    "gsb::k_corners_tiles": "corners",
    "gsb::k_corners_final": "corners",
}
CORNER_KERNELS = ["gsb::k_corners_small", "gsb::k_corners_tiles", "gsb::k_corners_final"]


# ---- the rules, restated ----------------------------------------------------------------------------------------------
def i32(a):
    a = np.asarray(a, np.int64)
    return ((a + 2 ** 31) % 2 ** 32) - 2 ** 31


def model_corners(img, labels, rec):
    """gs_blob_corners (grayskull.h:404-421) for one record -> (4, 2) uint32 points tl, tr, br, bl.  The loops run
    while y < box.y + box.h and x < box.x + box.w in 32-bit unsigned arithmetic; gs_get gives 0 outside the frame, so
    only the box's part inside it counts; sums and differences are the reference's wrapping ints, with its INT_MAX /
    INT_MIN starting values and strict comparisons (the first pixel in raster order wins a tie)."""
    h, w = img.shape
    bx, by, bw, bh = (int(rec[k]) for k in ("bx", "by", "bw", "bh"))
    out = np.array([[int(rec["cx"]), int(rec["cy"])]] * 4, np.uint32)
    x1, y1 = min((bx + bw) & M32, w), min((by + bh) & M32, h)
    if bx >= x1 or by >= y1:
        return out
    ys, xs = np.nonzero((img[by:y1, bx:x1] >= 128) & (labels[by:y1, bx:x1] == int(rec["label"])))
    if not len(xs):
        return out
    xs, ys = xs.astype(np.int64) + bx, ys.astype(np.int64) + by       # raster order
    s, d = i32(xs + ys), i32(xs - ys)
    picks = [np.where(s < INT_MAX, s, BIG), np.where(d > INT_MIN, d, -BIG), np.where(s > INT_MIN, s, -BIG),
             np.where(d < INT_MAX, d, BIG)]
    for q, v in enumerate(picks):
        i = int(np.argmin(v)) if q in (0, 3) else int(np.argmax(v))
        if abs(int(v[i])) != BIG:
            out[q] = (xs[i], ys[i])
    return out


def model_pick(blobs, count, stride, min_area):
    """nanomagick.c:196-199 / grayskull.c:285-295 over the first min(count, stride) records -> (record, pcount)"""
    c = min(count, stride)
    if c == 0:
        init = np.zeros(1, L.BLOB_DTYPE)[0]
        init["bx"] = init["by"] = M32
        return init, 0
    largest = 0
    for i in range(1, c):
        if blobs[i]["area"] > blobs[largest]["area"]:
            largest = i
    return blobs[largest], int(int(blobs[largest]["area"]) >= min_area)


def rec(label, area, bx, by, bw, bh, cx=0, cy=0):
    r = np.zeros(1, L.BLOB_DTYPE)
    r[0] = (label, area, bx & M32, by & M32, bw & M32, bh & M32, cx, cy)
    return r[0]


def O_corners(a, lab, r):
    c = np.zeros((4, 2), np.uint32)
    rr = np.array([r], L.BLOB_DTYPE)
    L.oracle().gso_blob_corners(L.ptr(a), a.shape[1], a.shape[0], L.ptr(lab), L.ptr(rr), L.ptr(c))
    return c


def R_corners(a, lab, r):
    c = np.zeros((4, 2), np.uint32)
    rr = np.array([r], L.BLOB_DTYPE)
    L.ref().gs_blob_corners(L.img(a), L.ptr(lab), L.ptr(rr), L.ptr(c))
    return c


def R_blobs(a, cap):
    lab = np.zeros(a.shape, np.uint16)
    b = np.zeros(cap, L.BLOB_DTYPE)
    k = L.ref().gs_blobs(L.img(a), L.ptr(lab), L.ptr(b), cap) if L.have_ref() else \
        L.oracle().gso_blobs(L.ptr(a), a.shape[1], a.shape[0], L.ptr(lab), L.ptr(b), cap)
    return lab, b, int(k)


# ---- inputs ------------------------------------------------------------------------------------------------------------
def edge_records(w, h, rng, k=40):
    """boxes past and clipped by the frame, wrapping past 2^32, shared labels, boxes that miss their label, labels that
    do not occur, empty boxes, whole-frame boxes"""
    out = [rec(1, 5, 0, 0, w, h, 3, 4), rec(1, 5, w - 3, h - 2, 50, 40, 7, 9), rec(2, 0, 0, 0, 0, 0, 11, 12),
           rec(2, 1, w - 5, 2, 2 ** 32 - w + 6, 5, 1, 2), rec(3, 1, 1, h - 4, 7, 2 ** 32 - h + 5, 5, 5),
           rec(3, 1, w, 0, 5, h, 9, 9), rec(1, 1, 0, h, w, 3, 8, 8), rec(999, 1, 0, 0, w, h, 6, 6),
           rec(1, 1, 3, 3, 0, 10, 2, 2), rec(2, 1, M32, M32, 2, 2, 1, 1), rec(1, 9, 2, 1, w - 4, h - 2, 0, 0),
           rec(0, 9, 0, 0, w, h, 4, 4)]
    while len(out) < k:
        bx, by = int(rng.integers(0, w + 3)), int(rng.integers(0, h + 3))
        out.append(rec(int(rng.integers(0, 5)), int(rng.integers(0, 50)), bx, by, int(rng.integers(0, w + 5)),
                       int(rng.integers(0, h + 5)), int(rng.integers(0, w)), int(rng.integers(0, h))))
    return out


def labelled_frame(w, h, rng, nlab=4):
    """random pixels around 128 and random labels 0..nlab-1"""
    a = rng.choice(np.array([0, 127, 128, 200, 255], np.uint8), (h, w))
    lab = rng.integers(0, nlab, (h, w)).astype(np.uint16)
    return a, lab


def diagonal_frame(w, h):
    """diagonal lines both ways, where every pixel of a line ties on x - y (or x + y)"""
    a = np.zeros((h, w), np.uint8)
    for i in range(min(w, h)):
        a[i, i] = 255
        a[i, w - 1 - i] = 200
        if i + 3 < w:
            a[i, i + 3] = 130
    return a, (a > 0).astype(np.uint16)


# ---- CPU: the model against the reference ------------------------------------------------------------------------------
def _both(a, lab, r):
    want = model_corners(a, lab, r)
    assert np.array_equal(O_corners(a, lab, r), want), (r, want)
    if L.have_ref():
        assert np.array_equal(R_corners(a, lab, r), want), (r, want)


def test_model_matches_the_reference_on_edge_records():
    rng = np.random.default_rng(1)
    for w, h in ((1, 1), (7, 5), (33, 17), (64, 40)):
        a, lab = labelled_frame(w, h, rng)
        for r in edge_records(w, h, rng):
            _both(a, lab, r)


def test_model_matches_the_reference_on_tie_heavy_shapes():
    for w, h in ((9, 9), (40, 23), (23, 40)):
        a, lab = diagonal_frame(w, h)
        for r in (rec(1, 1, 0, 0, w, h), rec(1, 1, 2, 1, w - 3, h - 2, 4, 4), rec(1, 1, 0, 0, w // 2, h),
                  rec(0, 1, 0, 0, w, h, 5, 6)):
            _both(a, lab, r)
        full = np.full((h, w), 255, np.uint8)
        _both(full, np.ones((h, w), np.uint16), rec(1, 1, 0, 0, w, h))


@pytest.mark.parametrize("cap", [3, 1000, 65534])
def test_model_matches_the_reference_on_gs_blobs_lists(cap):
    """every record of gs_blobs' list, capped at 3, 1000 and 65534 (where a checkerboard runs out of labels)"""
    frames = [np.where(L.natural_like(96, 64, 3) > 128, 255, 0).astype(np.uint8), L.binary_like(80, 60, 2, 0.4)]
    if cap == 65534:
        frames = [((np.indices((400, 400)).sum(0) % 2) * 255).astype(np.uint8)]   # 80000 one-pixel blobs
    for a in frames:
        lab, b, k = R_blobs(a, cap)
        assert k == min(cap, k) and (cap != 65534 or k == 65534)
        idx = range(k) if k <= 1000 else list(range(300)) + list(range(k - 300, k))
        for i in idx:
            want = model_corners(a, lab, b[i])
            assert np.array_equal(O_corners(a, lab, b[i]), want)
            if L.have_ref():
                assert np.array_equal(R_corners(a, lab, b[i]), want), i


def test_pick_rule():
    b = np.zeros(6, L.BLOB_DTYPE)
    b["area"] = [5, 9, 9, 2, 9, 0]
    b["label"] = np.arange(1, 7)
    assert model_pick(b, 6, 6, 0)[0]["label"] == 2          # the first of the tied 9s
    assert model_pick(b, 1, 6, 0)[0]["label"] == 1
    assert model_pick(b, 99, 6, 0)[0]["label"] == 2         # counts above the stride: the stride
    z = np.zeros(3, L.BLOB_DTYPE)
    z["label"] = [7, 8, 9]
    assert model_pick(z, 3, 3, 0) == (z[0], 1)               # all area 0: the first, and it counts at min_area 0
    assert model_pick(z, 3, 3, 100)[1] == 0
    assert model_pick(b, 6, 6, 9)[1] == 1 and model_pick(b, 6, 6, 10)[1] == 0 and model_pick(b, 6, 6, M32)[1] == 0
    init, pc = model_pick(b, 6, 0, 0)                         # stride 0: every list is empty
    assert pc == 0 and init.tobytes() == np.array([(0, 0, M32, M32, 0, 0, 0, 0)], L.BLOB_DTYPE).tobytes()
    if L.have_ref():                                          # gs_blobs initialises every slot to that record
        lab, got, k = R_blobs(np.zeros((4, 4), np.uint8), 2)
        assert k == 0 and got[0].tobytes() == init.tobytes()
        assert np.array_equal(R_corners(np.zeros((4, 4), np.uint8), lab, got[0]), np.zeros((4, 2), np.uint32))


# ---- CPU: the library ------------------------------------------------------------------------------------------------------
HEADER = os.path.join(ROOT, "include", "grayskull_corners.h")


def _declarations():
    txt = open(HEADER).read()
    txt = txt[txt.rindex('extern "C" {'):]
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return {m.group(2): (m.group(1).strip().split("\n")[-1].strip(), [a.strip() for a in m.group(3).split(",") if a.strip() != "void"])
            for m in re.finditer(r"([\w\s\*]+?)\b(gs_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", txt)}


def test_companion_exports_exactly_its_header():
    from grayskull_b200 import build, corners
    build.build()
    declared = sorted(_declarations())
    assert len(declared) == 3 and sorted(corners.SIGNATURES) == declared
    nm = subprocess.run(["nm", "-D", "--defined-only", corners.LIB_PATH], capture_output=True, text=True,
                        check=True).stdout
    assert sorted(ln.split()[-1] for ln in nm.splitlines() if " T " in ln) == declared
    needed = subprocess.run(["readelf", "-d", corners.LIB_PATH], capture_output=True, text=True, check=True).stdout
    assert "libgrayskull_b200" not in needed
    from grayskull_b200 import _lib
    main = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    assert "largest_blob" not in main and "corners_batch" not in main and "corners_last_error" not in main
    assert not any("k_corners" in k or "k_largest_blob" in k for k in L.sass_functions())
    assert corners.lib().gs_b200_corners_last_error() == b"no error"


def test_ctypes_table_matches_the_header():
    from grayskull_b200 import corners
    for name, (ret, args) in _declarations().items():
        res, argtypes = corners.SIGNATURES[name]
        assert (res is C.c_int) == (ret == "int") and (res is C.c_char_p) == ("char" in ret), name
        assert len(argtypes) == len(args), name
        for a, t in zip(args, argtypes):
            want = C.c_void_p if "*" in a or a.startswith("gs_b200_stream") else C.c_uint
            assert t is want, (name, a)


def test_header_compiles_as_c99(tmp_path):
    for first in ("", '#include "grayskull_b200.h"\n', '#include "grayskull_contour.h"\n'):
        src = tmp_path / "t.c"
        src.write_text(first + '#include "grayskull_corners.h"\n'
                       'int main(void) { struct gs_blob b = {0, 0, {0, 0, 1, 1}, {0, 0}};\n'
                       '  return gs_b200_corners_last_error() == 0 && b.area == 2; }\n')
        r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-fsyntax-only",
                            "-I", os.path.join(ROOT, "include"), str(src)], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    assert not re.match(r"grayskull_b200.*\.h$", "grayskull_corners.h")


def _corners_sass():
    from grayskull_b200 import corners
    tool = L.cuda_tool("cuobjdump")
    if tool is None:
        pytest.skip("cuobjdump not found")
    listing = subprocess.run([tool, "-sass", corners.LIB_PATH], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for cubin in re.split(r"^\s*(?=code for sm_\w+\s*$)", listing, flags=re.M)[1:]:
        arch, *parts = re.split(r"^\s*Function : (\S+)\s*$", cubin, flags=re.M)
        for name in L.demangle(parts[0::2]):
            funcs[L.kernel_id(name)] = arch.strip().splitlines()[0]
    return funcs


def test_every_companion_kernel_is_sm90a_and_has_a_row():
    funcs = _corners_sass()
    assert set(funcs) == set(KERNELS)
    assert all(arch == "code for sm_90a" for arch in funcs.values())


def test_launches_go_through_the_companions_helper():
    d = os.path.join(ROOT, "grayskull_b200", "corners")
    text = {f: open(os.path.join(d, f)).read() for f in sorted(os.listdir(d))}
    sites = [(f, m.start()) for f, t in text.items() for m in re.finditer(r"<<<", t)]
    assert len(sites) == 1
    f, at = sites[0]
    assert text[f].rindex("static int launch(", 0, at) < at < text[f].index("cudaGetLastError")
    assert text[f].count("cudaGetLastError") == 1
    from grayskull_b200 import build
    assert not set(build.CORNERS_SOURCES) & set(build.SOURCES)


def test_companion_object_makes_no_blocking_runtime_call():
    from grayskull_b200 import build
    nm = shutil.which("nm")
    if nm is None:
        pytest.skip("nm not found")
    blocking = re.compile(r"^(cudaMemcpy|cudaMemcpyToSymbol|cudaMemset|cudaMemcpy2D|cudaDeviceSynchronize|"
                          r"cudaStreamSynchronize|cudaEventSynchronize|cudaMalloc\w*|cudaFree\w*|cudaStreamCreate\w*|"
                          r"cudaStreamDestroy|cudaMemcpyAsync|cudaMemsetAsync)$")
    for s in build.CORNERS_SOURCES:
        o = os.path.join(build.OBJ, s.replace(".cu", ".o"))
        syms = [ln.split()[-1] for ln in subprocess.run([nm, "-u", o], capture_output=True, text=True,
                                                         check=True).stdout.splitlines()]
        assert "cudaGetLastError" in syms
        assert not [x for x in syms if blocking.match(x)], syms


def test_empty_batch_and_missing_pointer_without_a_gpu():
    code = ("import ctypes as C, sys; sys.path.insert(0, %r); from grayskull_b200 import corners; "
            "L = corners.lib(); P = C.c_void_p(4096); rc = %s; print('rc', rc)")
    calls = {"pick": "L.gs_b200_largest_blob_batch(P, P, 4, %d, 0, %s, P, None)",
             "corners": "L.gs_b200_blob_corners_batch(P, 8, 8, %d, P, P, P, 4, %s, None)"}
    for name, c in calls.items():
        ok = subprocess.run([sys.executable, "-c", code % (ROOT, c % (0, "P"))], capture_output=True, text=True,
                            timeout=120)
        assert ok.returncode == 0 and "rc 0" in ok.stdout, (name, ok.stdout, ok.stderr)
        bad = subprocess.run([sys.executable, "-c", code % (ROOT, c % (2, "None"))], capture_output=True, text=True,
                             timeout=120)
        assert bad.returncode != 0 and "Assertion failed: " in bad.stderr, (name, bad.stderr)
    for empty in ("L.gs_b200_blob_corners_batch(P, 0, 8, 2, P, P, P, 4, P, None)",
                  "L.gs_b200_blob_corners_batch(P, 8, 0, 2, P, P, P, 4, P, None)"):
        bad = subprocess.run([sys.executable, "-c", code % (ROOT, empty)], capture_output=True, text=True, timeout=120)
        assert bad.returncode != 0 and "Assertion failed: w > 0 && h > 0" in bad.stderr, bad.stderr
    # misaligned corners are refused before anything is launched
    mis = "L.gs_b200_blob_corners_batch(P, 8, 8, 2, P, P, P, 4, C.c_void_p(4100), None)"
    r = subprocess.run([sys.executable, "-c", code % (ROOT, mis) + "; print(L.gs_b200_corners_last_error())"],
                       capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "rc 1" in r.stdout and "8-byte aligned" in r.stdout, (r.stdout, r.stderr)


# ---- GPU ---------------------------------------------------------------------------------------------------------------------
def klib():
    from grayskull_b200 import corners
    return corners.lib()


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()


def _s():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


class Case:
    """one corners call: frames (n, h, w), labels (n, h, w) uint16, records (n, stride) and counts (None: all)"""

    def __init__(self, frames, labels, blobs, counts):
        assert blobs.dtype.itemsize == 32
        self.frames, self.labels, self.blobs, self.counts = frames, labels, blobs, counts
        self.n, self.stride = blobs.shape

    def used(self, f):
        return self.stride if self.counts is None else min(int(self.counts[f]), self.stride)

    def buffers(self, off=0):
        self.img = Region(self.frames.nbytes, off, self.frames, seed=1)
        self.lab = Region(self.labels.nbytes, 2 * off, self.labels, seed=2)
        self.rec = Region(self.blobs.nbytes, 4 * (off % 8), self.blobs, seed=3)
        self.out = Region(32 * self.n * self.stride, 8 * off, seed=4)
        self.count_t = None if self.counts is None else _dev(np.asarray(self.counts, np.uint32))
        return self

    def call(self, s=None):
        n, h, w = self.frames.shape
        cp = None if self.count_t is None else self.count_t.data_ptr()
        return klib().gs_b200_blob_corners_batch(self.img.ptr, w, h, n, self.lab.ptr, self.rec.ptr, cp, self.stride,
                                                 self.out.ptr, _s() if s is None else s)

    def expected(self, frames=None):
        want = self.out.before().view(np.uint32).reshape(self.n, self.stride, 4, 2).copy()
        for f in range(self.n) if frames is None else frames:
            for k in range(self.used(f)):
                want[f, k] = model_corners(self.frames[f], self.labels[f], self.blobs[f, k])
        return want

    def check(self, what, frames=None):
        got = self.out.read(what).view(np.uint32).reshape(self.n, self.stride, 4, 2)
        self.img.read(what), self.lab.read(what), self.rec.read(what)
        want = self.expected(frames)
        fs = range(self.n) if frames is None else frames
        for f in fs:
            bad = np.flatnonzero((got[f] != want[f]).any(axis=(1, 2)))
            assert not len(bad), "%s: frame %d record %d: got %s, want %s (%s)" % (
                what, f, bad[0], got[f, bad[0]].tolist(), want[f, bad[0]].tolist(), self.blobs[f, bad[0]])


def mixed_case(w, h, n, stride, seed, counts="random"):
    """random labelled frames with gs_blobs-like records, the edge records and one frame-sized record"""
    rng = np.random.default_rng(seed)
    frames = np.empty((n, h, w), np.uint8)
    labels = np.empty((n, h, w), np.uint16)
    blobs = np.zeros((n, stride), L.BLOB_DTYPE)
    for f in range(n):
        frames[f], labels[f] = labelled_frame(w, h, rng, 6)
        recs = edge_records(w, h, rng, stride)
        for k in range(stride):
            blobs[f, k] = recs[k]
        if stride > 12:
            blobs[f, 12] = rec(int(rng.integers(1, 6)), 1, 0, 0, w, h, 1, 1)
    if counts == "random":
        counts = rng.integers(0, stride + 1, n).astype(np.uint32)
        counts[0] = stride + 3
    return Case(frames, labels, blobs, counts)


SIZES = [(1, 300, 2, 20), (300, 1, 2, 20), (17, 9, 3, 30), (613, 411, 3, 40), (1023, 777, 2, 60)]


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,n,stride", SIZES, ids=["%dx%d" % s[:2] for s in SIZES])
@pytest.mark.parametrize("layout", ["aligned", "offset", "counts-null"])
def test_corners_match_the_model(lib, witness, w, h, n, stride, layout):
    c = mixed_case(w, h, n, stride, seed=w * 7 + h, counts=None if layout == "counts-null" else "random")

    def run():
        c.buffers(off=3 if layout == "offset" else 0)
        rc, seen = traced(lambda: c.call())
        assert rc == 0, klib().gs_b200_corners_last_error()
        c.check("%dx%d %s" % (w, h, layout))
        return seen

    witnessed(witness, run, CORNER_KERNELS, "%dx%d %s" % (w, h, layout))


def w2_case(n, seed, w=1024, h=1024, stride=150):
    """ArUco-like: square marks of mixed sizes on a dark frame, their records, and one frame-sized background record"""
    rng = np.random.default_rng(seed)
    frames = (rng.random((n, h, w)) < 0.02).astype(np.uint8) * 140
    labels = np.zeros((n, h, w), np.uint16)
    blobs = np.zeros((n, stride), L.BLOB_DTYPE)
    for f in range(n):
        blobs[f, 0] = rec(1, w * h, 0, 0, w, h, w // 2, h // 2)
        labels[f][frames[f] > 0] = 1
        for k in range(1, stride):
            s = int(rng.choice([2, 5, 9, 17, 40, 90, 200]))
            x, y = int(rng.integers(0, w - s)), int(rng.integers(0, h - s))
            frames[f, y:y + s, x:x + s] = 255
            frames[f, y + s // 2, x:x + s] = 100
            labels[f, y:y + s, x:x + s] = k + 1
            blobs[f, k] = rec(k + 1, s * s, x, y, s, s, x + s // 2, y + s // 2)
    return Case(frames, labels, blobs, None)


@pytest.mark.gpu
def test_w2_mix_and_one_frame_sized_record(lib, witness):
    c = w2_case(2, seed=3)

    def run():
        c.buffers()
        rc, seen = traced(lambda: c.call())
        assert rc == 0
        c.check("w2 mix")
        return seen

    witnessed(witness, run, CORNER_KERNELS, "w2 mix")
    # one frame-sized record alone, on a bright noisy frame
    rng = np.random.default_rng(4)
    a = np.where(rng.random((1, 2048, 2048)) < 0.9, 255, 0).astype(np.uint8)
    one = Case(a, (a > 0).astype(np.uint16), np.array([[rec(1, 1, 0, 0, 2048, 2048, 9, 9)]], L.BLOB_DTYPE), None)
    one.buffers()
    assert one.call() == 0
    one.check("frame-sized")


@pytest.mark.gpu
def test_65534_records_per_frame(lib, witness):
    """a checkerboard's gs_blobs list at its cap, and records entirely outside the frame"""
    a = ((np.indices((512, 512)).sum(0) % 2) * 255).astype(np.uint8)
    lab, b, k = R_blobs(a, 65534)
    assert k == 65534
    outside = b.copy()
    outside["bx"] = (outside["bx"].astype(np.int64) + 512 + np.arange(65534) % 7).astype(np.uint32)
    both = np.zeros((2, 65534), L.BLOB_DTYPE)                # np.stack would drop the records' 2 padding bytes
    both[0], both[1] = b, outside
    c = Case(np.stack([a, a]), np.stack([lab, lab]), both, np.array([65534, 65534], np.uint32))

    def run():
        c.buffers(off=1)
        rc, seen = traced(lambda: c.call())
        assert rc == 0
        c.check("65534 records")
        return seen

    witnessed(witness, run, CORNER_KERNELS, "65534 records")
    got = c.out.read("again").view(np.uint32).reshape(2, 65534, 4, 2)
    assert (got[1] == np.stack([outside["cx"], outside["cy"]], -1)[:, None, :]).all()


# ---- GPU: the pick -------------------------------------------------------------------------------------------------------
def pick_call(blobs, counts, min_area, pcount=True, off=0):
    n, stride = blobs.shape
    bl = Region(blobs.nbytes, 4 * off, blobs, seed=5) if blobs.size else None
    pk = Region(32 * n, 4 * off, seed=6)
    pc = Region(4 * n, 4 * off, seed=7)
    ct = None if counts is None else _dev(np.asarray(counts, np.uint32))
    rc = klib().gs_b200_largest_blob_batch(bl.ptr if bl else C.c_void_p(4096), None if ct is None else ct.data_ptr(),
                                           stride, n, min_area, pk.ptr, pc.ptr if pcount else None, _s())
    assert rc == 0
    return pk.read("pick"), pc.read("pcount")


def check_pick(blobs, counts, min_area, got_pick, got_pc, pcount=True, before=None):
    n, stride = blobs.shape
    gp = got_pick.view(L.BLOB_DTYPE)
    gc = got_pc.view(np.uint32)
    for f in range(n):
        want, wc = model_pick(blobs[f], stride if counts is None else int(counts[f]), stride, min_area)
        assert gp[f].tobytes() == want.tobytes(), (f, gp[f], want)
        if pcount:
            assert gc[f] == wc, f
    if not pcount:
        assert np.array_equal(got_pc, before)


@pytest.mark.gpu
def test_pick_matches_the_rule(lib, witness):
    rng = np.random.default_rng(8)
    n, stride = 9, 70
    b = np.frombuffer(rng.integers(0, 256, n * stride * 32, dtype=np.uint8).tobytes(), L.BLOB_DTYPE).copy()
    b = b.reshape(n, stride)
    b["area"] = rng.integers(0, 5, (n, stride))               # many ties
    b[1]["area"] = 0
    b[2]["area"] = 7
    b[3, 40]["area"] = 300
    counts = np.array([0, 70, 70, 41, 40, 99, 1, 33, 69], np.uint32)
    for min_area in (0, 3, 4, 100, M32):
        def run():
            (p, c), seen = traced(lambda: pick_call(b, counts, min_area))
            check_pick(b, counts, min_area, p, c)
            return seen

        witnessed(witness, run, ["gsb::k_largest_blob"], "pick min_area %d" % min_area)
    p, c = pick_call(b, None, 0, off=1)
    check_pick(b, None, 0, p, c)
    pc_before = Region(4 * n, 0, seed=7).before()
    p, c = pick_call(b, counts, 0, pcount=False)              # pcount NULL: pick alone, pcount untouched
    check_pick(b, counts, 0, p, c, pcount=False, before=pc_before)
    p, c = pick_call(np.zeros((n, 0), L.BLOB_DTYPE), counts, 0)  # stride 0
    check_pick(np.zeros((n, 0), L.BLOB_DTYPE), counts, 0, p, c)


@pytest.mark.gpu
def test_pick_over_65534_records_and_65536_frames(lib):
    rng = np.random.default_rng(9)
    b = np.zeros((2, 65534), L.BLOB_DTYPE)
    b["area"] = rng.integers(0, 1000, (2, 65534))
    b[0, 65533]["area"] = 5000
    b[1, 17]["area"] = b[1, 60000]["area"] = 5000
    p, c = pick_call(b, None, 100)
    check_pick(b, None, 100, p, c)
    n = 65536 + 7
    b = np.zeros((n, 3), L.BLOB_DTYPE)
    b["area"] = rng.integers(0, 200, (n, 3))
    b["label"] = rng.integers(0, 60000, (n, 3))
    counts = rng.integers(0, 5, n).astype(np.uint32)
    p, c = pick_call(b, counts, 100)
    check_pick(b[-300:], counts[-300:], 100, p[-300 * 32:], c[-300 * 4:])
    check_pick(b[:300], counts[:300], 100, p[:300 * 32], c[:300 * 4])


# ---- GPU: limits -----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_batches_above_the_grid_limit(lib):
    w, h, n, stride = 6, 5, 65536 + 3, 3
    rng = np.random.default_rng(10)
    frames = rng.choice(np.array([0, 200], np.uint8), (n, h, w))
    labels = rng.integers(0, 3, (n, h, w)).astype(np.uint16)
    blobs = np.zeros((n, stride), L.BLOB_DTYPE)
    blobs["label"] = rng.integers(0, 3, (n, stride))
    blobs["bx"], blobs["by"] = rng.integers(0, w, (n, stride)), rng.integers(0, h, (n, stride))
    blobs["bw"], blobs["bh"] = rng.integers(0, w + 1, (n, stride)), rng.integers(0, h + 1, (n, stride))
    blobs["cx"], blobs["cy"] = 77, 88
    counts = rng.integers(0, 5, n).astype(np.uint32)
    c = Case(frames, labels, blobs, counts).buffers()
    assert c.call() == 0
    c.check("65539 frames", frames=list(range(100)) + list(range(n - 100, n)))


@pytest.mark.gpu
def test_frames_past_4_gib_and_taller_than_65535_row_tiles(lib):
    """9 frames of 512 MiB (labels past 8 GiB), the last frame's records past 4 GiB; then a frame of 64 * 65535 + 100
    rows with a record near its bottom and one spanning it"""
    import torch
    w, h, n = 32768, 16384, 9
    img = torch.zeros((n, h, w), dtype=torch.uint8, device="cuda")
    lab = torch.zeros((n, h, w), dtype=torch.int16, device="cuda")
    x0, y0 = w - 300, h - 40
    patch, plab = diagonal_frame(280, 30)
    img[n - 1, y0:y0 + 30, x0:x0 + 280] = torch.from_numpy(patch).cuda()
    lab[n - 1, y0:y0 + 30, x0:x0 + 280] = torch.from_numpy(plab.astype(np.int16)).cuda()
    img[0, 5:9, 5:9] = 255
    lab[0, 5:9, 5:9] = 1
    blobs = np.zeros((n, 2), L.BLOB_DTYPE)
    blobs[:, 0] = rec(1, 1, 0, 0, w, h, 3, 3)
    blobs[:, 1] = rec(1, 1, x0 - 5, y0 - 5, 300, 40, 4, 4)
    out = torch.full((n * 2 * 8,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
    bt = _dev(blobs)
    assert klib().gs_b200_blob_corners_batch(img.data_ptr(), w, h, n, lab.data_ptr(), bt.data_ptr(), None, 2,
                                             out.data_ptr(), _s()) == 0
    got = out.cpu().numpy().view(np.uint32).reshape(n, 2, 4, 2)
    full = np.zeros((h, w), np.uint8)
    flab = np.zeros((h, w), np.uint16)
    full[y0:y0 + 30, x0:x0 + 280], flab[y0:y0 + 30, x0:x0 + 280] = patch, plab
    last = [model_corners(full, flab, blobs[n - 1, k]) for k in range(2)]
    assert np.array_equal(got[n - 1], np.stack(last))
    assert np.array_equal(got[0, 0], [[5, 5], [8, 5], [8, 8], [5, 8]])
    for f in range(1, n - 1):
        assert (got[f, 0] == 3).all() and (got[f, 1] == 4).all()
    del img, lab
    torch.cuda.empty_cache()
    w, h = 5, 64 * 65535 + 100
    a = np.zeros((h, w), np.uint8)
    al = np.zeros((h, w), np.uint16)
    for (y, x) in ((h - 20, 3), (h - 19, 1), (7, 2), (h - 1, 4), (h - 2, 0)):
        a[y, x], al[y, x] = 255, 7
    blobs = np.array([[rec(7, 1, 0, h - 30, w, 30, 1, 1), rec(7, 1, 0, 0, w, h, 2, 2), rec(7, 1, 0, h - 2, 3, 2)]],
                     L.BLOB_DTYPE)
    img, lab = _dev(a), _dev(al)
    out = torch.zeros(24, dtype=torch.int32, device="cuda")
    bt = _dev(blobs)
    assert klib().gs_b200_blob_corners_batch(img.data_ptr(), w, h, 1, lab.data_ptr(), bt.data_ptr(), None, 3,
                                             out.data_ptr(), _s()) == 0
    got = out.cpu().numpy().view(np.uint32).reshape(3, 4, 2)
    for k in range(3):
        assert np.array_equal(got[k], model_corners(a, al, blobs[0, k])), k
    assert got[1].tolist() == [[2, 7], [2, 7], [4, h - 1], [0, h - 2]]


# ---- GPU: streams -------------------------------------------------------------------------------------------------------------
def _sleep(s, cycles):
    import torch
    with torch.cuda.stream(s):
        torch.cuda._sleep(int(cycles))


@pytest.mark.gpu
def test_ordered_behind_a_sleeping_stream_without_a_host_wait(lib):
    import torch
    c = mixed_case(300, 200, 3, 30, seed=21).buffers()
    s, u = torch.cuda.Stream(), torch.cuda.Stream()
    real = _dev(c.frames)
    out0 = torch.from_numpy(c.out.before()).cuda()          # host copies wait for their stream: all made up front
    pk = torch.empty(32 * 3, dtype=torch.uint8, device="cuda")
    with torch.cuda.stream(s):
        c.img.t[c.img.off:c.img.off + c.img.nbytes].zero_()
    assert c.call(C.c_void_p(s.cuda_stream)) == 0      # warm, on zeros
    torch.cuda.synchronize()
    _sleep(u, 400_000_000)
    _sleep(s, 200_000_000)
    with torch.cuda.stream(s):
        c.img.t[c.img.off:c.img.off + c.img.nbytes].copy_(real)
        c.out.t[c.out.off:c.out.off + c.out.nbytes].copy_(out0)
    assert c.call(C.c_void_p(s.cuda_stream)) == 0
    assert klib().gs_b200_largest_blob_batch(c.rec.ptr, c.count_t.data_ptr(), c.stride, 3, 0, pk.data_ptr(), None,
                                             C.c_void_p(s.cuda_stream)) == 0
    s_done, u_done = s.query(), u.query()
    torch.cuda.synchronize()
    assert not s_done and not u_done, "a call waited for its stream or for the device"
    c.check("behind a sleep")


@pytest.mark.gpu
def test_two_streams_at_once(lib):
    import torch
    s0, s1 = torch.cuda.Stream(), torch.cuda.Stream()
    cases = [(mixed_case(300, 200, 3, 30, seed=seed).buffers(), st) for seed, st in ((22, s0), (23, s1), (24, s0),
                                                                                       (25, s1))]
    _sleep(s1, 50_000_000)
    for c, st in cases:
        assert c.call(C.c_void_p(st.cuda_stream)) == 0
    torch.cuda.synchronize()
    for c, _ in cases:
        c.check("two streams")


@pytest.mark.gpu
def test_graph_capture_and_replay_on_new_inputs(lib):
    """pick then corners of the pick, captured once and replayed on two new batches"""
    import torch
    n, stride = 3, 30
    c = mixed_case(300, 200, n, stride, seed=26).buffers()
    pick = torch.empty(n * 8, dtype=torch.int32, device="cuda")
    pcount = torch.empty(n, dtype=torch.int32, device="cuda")
    out = torch.full((n * 8,), -1, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    h, w = c.frames.shape[1:]
    with torch.cuda.graph(g, stream=s):
        assert klib().gs_b200_largest_blob_batch(c.rec.ptr, c.count_t.data_ptr(), stride, n, 10, pick.data_ptr(),
                                                 pcount.data_ptr(), C.c_void_p(s.cuda_stream)) == 0
        assert klib().gs_b200_blob_corners_batch(c.img.ptr, w, h, n, c.lab.ptr, pick.data_ptr(), pcount.data_ptr(),
                                                 1, out.data_ptr(), C.c_void_p(s.cuda_stream)) == 0
    for seed in (31, 32):
        fresh = mixed_case(300, 200, n, stride, seed=seed)
        fresh.blobs["area"] = np.random.default_rng(seed).integers(0, 30, (n, stride))
        with torch.cuda.stream(s):
            c.img.t[c.img.off:c.img.off + c.img.nbytes].copy_(_dev(fresh.frames))
            c.lab.t[c.lab.off:c.lab.off + c.lab.nbytes].copy_(_dev(fresh.labels))
            c.rec.t[c.rec.off:c.rec.off + c.rec.nbytes].copy_(_dev(fresh.blobs))
            c.count_t.copy_(_dev(np.asarray(fresh.counts, np.uint32)))
            out.fill_(-1)
            g.replay()
        s.synchronize()
        got_p = pick.cpu().numpy().view(L.BLOB_DTYPE)
        got_c = pcount.cpu().numpy()
        got = out.cpu().numpy().view(np.uint32).reshape(n, 4, 2)
        for f in range(n):
            want, wc = model_pick(fresh.blobs[f], int(fresh.counts[f]), stride, 10)
            assert got_p[f].tobytes() == want.tobytes() and got_c[f] == wc
            if wc:
                assert np.array_equal(got[f], model_corners(fresh.frames[f], fresh.labels[f], want)), seed
            else:
                assert (got[f] == M32).all()


# ---- GPU: the scanner chain and the CLI -------------------------------------------------------------------------------------
def oracle_scan(a, dw, dh):
    """nanomagick.c:186-210 from the oracle: blur 1, Otsu + 10, blobs(1000), the largest's corners, the warp"""
    Od = L.oracle()
    h, w = a.shape
    t = L.o_blur(Od, a, 1)
    th = Od.gso_otsu_threshold(L.ptr(t), w, h)
    Od.gso_threshold(L.ptr(t), w, h, (th + 10) & 255)      # the verb's uint8_t argument
    lab = np.zeros((h, w), np.uint16)
    b = np.zeros(1000, L.BLOB_DTYPE)
    k = Od.gso_blobs(L.ptr(t), w, h, L.ptr(lab), L.ptr(b), 1000)
    pick, _ = model_pick(b, k, 1000, 0)
    corners = O_corners(t, lab, pick)
    out = np.zeros((dh, dw), np.uint8)
    Od.gso_perspective_correct(L.ptr(out), dw, dh, L.ptr(a), w, h, L.ptr(corners))
    return corners, out


@pytest.mark.gpu
def test_scanner_chain_matches_the_oracle_chain(lib, witness):
    """blobs_batch -> largest_blob_batch -> blob_corners_batch -> perspective_correct_batch, with an all-dark frame"""
    import torch
    from grayskull_b200 import api, corners
    h, w = 480, 640
    frames = []
    for seed in range(3):
        rng = np.random.default_rng(seed)
        a = rng.integers(0, 60, (h, w)).astype(np.uint8)
        yy, xx = np.mgrid[0:h, 0:w]
        q = (xx - 100 - 20 * seed) * 3 + (yy - 60) > 0
        q &= (xx - 560) * 4 - (yy - 40) < 0
        q &= (yy - 440 + seed * 10) < (xx - 100) // 8
        a[q] = rng.integers(190, 250, int(q.sum()))
        frames.append(a)
    frames.append(np.zeros((h, w), np.uint8))
    src = torch.from_numpy(np.stack(frames)).cuda()

    def run():
        def chain():
            blur = api.blur_batch(src, 1)
            th = torch.empty(len(frames), dtype=torch.uint8, device="cuda")
            assert lib.gs_b200_otsu_threshold_batch(th.data_ptr(), None, blur.data_ptr(), w, h, len(frames),
                                                    _s()) == 0
            assert lib.gs_b200_threshold_each_batch(blur.data_ptr(), w, h, len(frames), th.data_ptr(), 10, _s()) == 0
            labels, blobs, counts = api.blobs_batch(blur, 1000)
            pick, pcount = corners.largest_blob_batch(blobs, counts, 0)
            cs = corners.blob_corners_batch(blur, labels, pick)
            return cs, api.perspective_correct_batch(src, 160, 200, cs.reshape(len(frames), 4, 2).contiguous())
        (cs, out), seen = traced(chain)
        cs, out = cs.cpu().numpy().view(np.uint32), out.cpu().numpy()
        for f, a in enumerate(frames):
            wc, wo = oracle_scan(a, 160, 200)
            assert np.array_equal(cs[f, 0], wc), (f, cs[f, 0], wc)
            assert np.array_equal(out[f], wo), f
        assert (cs[-1] == 0).all()
        return seen

    witnessed(witness, run, list(KERNELS), "scanner chain")


def scan_fixture(name):
    """tests/golden/scan_<name>_golden.npz (tools/make_scan_golden.py): the reference's scanner image, the SHA-256 and
    length of its scan verb's output file, and the corners the verb warps from"""
    z = np.load(os.path.join(ROOT, "tests", "golden", "scan_%s_golden.npz" % name))
    return z["frame"], bytes(z["scan_sha256"]), int(z["scan_size"]), z["corners"]


SCAN_IMAGES = ["document", "receipt"]


@pytest.mark.parametrize("name", SCAN_IMAGES)
def test_scan_fixture_matches_the_oracle_chain(name):
    """the oracle's scan chain on the fixture's frame gives the verb's corners and, byte for byte, its output file"""
    import hashlib
    a, digest, size, corners = scan_fixture(name)
    c, out = oracle_scan(a, 800, 1000)
    assert np.array_equal(c, corners)
    data = b"P5\n800 1000\n255\n" + out.tobytes()
    assert len(data) == size and hashlib.sha256(data).digest() == digest


@pytest.mark.gpu
@pytest.mark.parametrize("name", SCAN_IMAGES)
def test_gsb_magick_scan_matches_the_reference_on_its_scanner_images(lib, tmp_path, name):
    """gsb_magick scan:800:1000 writes the verb's output file byte for byte, for each frame of a batch of three, and
    the library chain finds the verb's corners"""
    import hashlib
    import torch
    from grayskull_b200 import api, build, corners
    exe = os.path.join(os.path.dirname(build.LIB), "gsb_magick")
    a, digest, size, want = scan_fixture(name)
    h, w = a.shape
    p = tmp_path / (name + ".pgm")
    p.write_bytes(b"P5\n%d %d\n255\n" % (w, h) + a.tobytes())
    r = subprocess.run([exe, "scan:800:1000", str(tmp_path / (name + "_"))] + [str(p)] * 3, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    for f in range(3):
        data = (tmp_path / ("%s_%04d.pgm" % (name, f))).read_bytes()
        assert len(data) == size and hashlib.sha256(data).digest() == digest, (name, f)
    src = torch.from_numpy(np.stack([a, a[::-1, ::-1].copy()])).cuda()
    t = api.blur_batch(src, 1)
    th = torch.empty(2, dtype=torch.uint8, device="cuda")
    assert lib.gs_b200_otsu_threshold_batch(th.data_ptr(), None, t.data_ptr(), w, h, 2, _s()) == 0
    assert lib.gs_b200_threshold_each_batch(t.data_ptr(), w, h, 2, th.data_ptr(), 10, _s()) == 0
    labels, blobs, counts = api.blobs_batch(t, 1000)
    pick, _ = corners.largest_blob_batch(blobs, counts, 0)
    got = corners.blob_corners_batch(t, labels, pick).cpu().numpy().view(np.uint32)
    assert np.array_equal(got[0, 0], want)
    assert np.array_equal(got[1, 0], oracle_scan(src[1].cpu().numpy(), 8, 8)[0])
