"""Contour tracing on the device (include/grayskull_contour.h, libgrayskull_contour.so): gs_trace_contour over frame
batches, bit-exact, with a defined end (GS_CONTOUR_CYCLE) for walks the reference never leaves, and the wasm demo's
contour start for blob records.

On the CPU the contour oracle's gso_trace_contour (tools/contour_oracle.c) is pinned against the reference's own test
case, the compiled reference
(oracle/_ref/libgs_ref.so, called only on walks the oracle classified as returning or open, so nothing here can hang)
and, for cycling walks, a literal Python walk run past the point where nothing can change any more; the companion
library is checked as a library.  On the GPU every call is checked against the oracle, bytes outside each buffer
included, with a census of the kernels it launched; then on the caller's stream, two streams and a CUDA graph, past
65535 frames and 4 GiB, on the blob chain and through the gsb_magick contour stage.
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
DX = (1, 1, 0, -1, -1, -1, 0, 1)
DY = (0, 1, 1, 1, 0, -1, -1, -1)
RETURNED, OPEN, CYCLE = 0, 1, 2

# every kernel of libgrayskull_contour.so, and which call launches it
KERNELS = {
    "gsb::k_contour_clear": "trace",
    "gsb::k_contour_walk": "trace",
    "gsb::k_contour_mark": "trace",
    "gsb::k_contour_starts": "starts",
}
TRACE_KERNELS = ["gsb::k_contour_clear", "gsb::k_contour_walk", "gsb::k_contour_mark"]


def contour_dtype():
    from grayskull_b200.contour import CONTOUR_DTYPE
    return CONTOUR_DTYPE


# ---- the walk, restated ---------------------------------------------------------------------------------------------
def i32(v):
    v &= M32
    return v - (1 << 32) if v >= 1 << 31 else v


def states(S):
    return 16 * S + 16


def py_walk(img, visited, start, cap):
    """grayskull.h:446-480 as written, stopped after `cap` steps -> (box, length, steps or None when it stopped by
    itself); visited is updated in place"""
    h, w = img.shape
    sx, sy = start
    box = [sx, sy, 1, 1]
    length, p, d, seen = 0, (sx, sy), 7, 0
    for t in range(cap):
        inside = p[0] < w and p[1] < h
        if not (inside and visited[p[1], p[0]]):
            length += 1
        if inside:
            visited[p[1], p[0]] = 255
        nd, q = (d + 1) % 8, None
        for i in range(8):
            dd = (nd + i) % 8
            nx, ny = i32(p[0] + DX[dd]), i32(p[1] + DY[dd])
            if 0 <= nx < i32(w) and 0 <= ny < i32(h) and img[ny, nx] > 128:
                q, d = (nx, ny), (dd + 6) % 8
                break
        if q is None:
            return box, length, None
        p = q
        box[0], box[1] = min(box[0], p[0]), min(box[1], p[1])
        box[2], box[3] = max(box[2], (p[0] - box[0] + 1) & M32), max(box[3], (p[1] - box[1] + 1) & M32)
        if p == (sx, sy):
            if seen:
                return box, length, None
            seen = 1
    return box, length, cap


def brent_match_step(img, start):
    """the step at which Brent's test (saved state at steps 2^j - 1) first sees the saved state again"""
    h, w = img.shape
    p, d, seen = tuple(start), 7, 0
    saved, power, lam, t = (p, d, seen), 1, 0, 0
    while True:
        nd, q = (d + 1) % 8, None
        for i in range(8):
            dd = (nd + i) % 8
            nx, ny = i32(p[0] + DX[dd]), i32(p[1] + DY[dd])
            if 0 <= nx < i32(w) and 0 <= ny < i32(h) and img[ny, nx] > 128:
                q, d = (nx, ny), (dd + 6) % 8
                break
        assert q is not None
        p, t, lam = q, t + 1, lam + 1
        if p == tuple(start):
            assert not seen
            seen = 1
        if (p, d, seen) == saved:
            return t
        if lam == power:
            saved, power, lam = (p, d, seen), power * 2, 0


def O():
    """the contour oracle (tools/contour_oracle.c), compiled on first use into a temporary directory"""
    if os.path.join(ROOT, "tools") not in sys.path:
        sys.path.insert(0, os.path.join(ROOT, "tools"))
    import contour_oracle
    return contour_oracle.load()


def R():
    r = L.ref()
    r.gs_trace_contour.restype = None
    r.gs_trace_contour.argtypes = [L.Image, L.Image, C.c_void_p]
    return r


def records(starts, stride=None, fill=None):
    """contour records with these starts, `stride` slots (the ones past the starts `fill`ed from an rng)"""
    stride = len(starts) if stride is None else stride
    if fill is None:
        rec = np.zeros(stride, contour_dtype())
    else:
        rec = np.frombuffer(fill.integers(0, 256, stride * 28, dtype=np.uint8).tobytes(), contour_dtype()).copy()
    for k, (x, y) in enumerate(starts):
        rec[k]["sx"], rec[k]["sy"] = x & M32, y & M32
    return rec


def o_trace(img, visited, rec):
    """the oracle over a frame's list, in order, on visited (in place) -> (records, ends)"""
    img = np.ascontiguousarray(img)
    rec = rec.copy()
    ends = np.zeros(len(rec), np.uint8)
    if len(rec):
        O().gso_trace_contours(L.ptr(img), L.ptr(visited), img.shape[1], img.shape[0], L.ptr(rec), len(rec),
                               L.ptr(ends))
    return rec, ends


def fields(r):
    return tuple(int(r[k]) for k in ("bx", "by", "bw", "bh", "sx", "sy", "length"))


# ---- CPU: the oracle -------------------------------------------------------------------------------------------------
W = 255
TEST_C = np.array([[0, W, W, W, 0], [0, W, W, W, 0], [0, W, 0, W, W], [0, W, W, W, 0], [0, 0, W, 0, W]], np.uint8)
TEST_C_VISITED = np.array([[0, W, W, W, 0], [0, W, 0, W, 0], [0, W, 0, 0, W], [0, W, 0, W, 0], [0, 0, W, 0, 0]],
                          np.uint8)


def test_reference_case_from_its_test_c():
    """test.c:261-283: length 10, box {1, 0, 4, 5}, and its visited map"""
    v = np.zeros_like(TEST_C)
    rec, ends = o_trace(TEST_C, v, records([(1, 0)]))
    assert fields(rec[0]) == (1, 0, 4, 5, 1, 0, 10) and ends[0] == RETURNED
    assert np.array_equal(v, TEST_C_VISITED)
    if L.have_ref():
        c = records([(1, 0)])
        v2 = np.zeros_like(TEST_C)
        R().gs_trace_contour(L.img(TEST_C), L.img(v2), L.ptr(c))
        assert fields(c[0]) == (1, 0, 4, 5, 1, 0, 10) and np.array_equal(v2, TEST_C_VISITED)


def block7():
    a = np.zeros((7, 7), np.uint8)
    a[2:5, 2:5] = 255
    return a


def test_ends_of_the_7x7_block():
    """a 3x3 block in a 7x7 frame: from its corner the walk returns (in 16 steps), from the background pixel next to
    it and from its centre it never returns, from (0, 0) it is open after 1 step; the cycling walks' outputs are what
    the reference's walk holds once nothing can change any more"""
    a = block7()
    want = {(2, 2): RETURNED, (1, 2): CYCLE, (3, 3): CYCLE, (0, 0): OPEN}
    for start, end in want.items():
        v = np.zeros_like(a)
        rec, ends = o_trace(a, v, records([start]))
        assert ends[0] == end, start
        cap = 2 * states(a.size) + 1
        for steps in (states(a.size) + 1, cap):      # 16wh + 17 steps, and past the closing lap's bound
            pv = np.zeros_like(a)
            box, length, stopped = py_walk(a, pv, start, steps)
            assert (stopped is None) == (end != CYCLE), start
            assert tuple(box) + (length,) == fields(rec[0])[:4] + (fields(rec[0])[6],), (start, steps)
            assert np.array_equal(pv, v), (start, steps)
        if end == RETURNED:
            assert py_walk(a, np.zeros_like(a), start, 16)[2] is None and py_walk(a, np.zeros_like(a), start, 15)[2]


def quirk_frames():
    """two frames of a seeded search in which the box after Brent's match is not yet final: a pixel walked before
    box.x reached its minimum widens the box on the next lap"""
    rng = np.random.default_rng(1)
    out = []
    for it in range(1474):
        w, h = int(rng.integers(5, 24)), int(rng.integers(5, 24))
        a = ((rng.random((h, w)) < rng.uniform(0.3, 0.95)) * 255).astype(np.uint8)
        s = (int(rng.integers(0, w)), int(rng.integers(0, h)))
        if it in (1306, 1473):
            out.append((a, s))
    return out


def test_cycle_box_needs_the_closing_lap():
    for a, s in quirk_frames():
        v = np.zeros_like(a)
        rec, ends = o_trace(a, v, records([s]))
        assert ends[0] == CYCLE
        cap = 2 * states(a.size) + 1
        pv = np.zeros_like(a)
        box, length, _ = py_walk(a, pv, s, cap)
        got = fields(rec[0])
        assert tuple(box) == got[:4] and length == got[6] and np.array_equal(pv, v)
        at_match = py_walk(a, np.zeros_like(a), s, brent_match_step(a, s))[0]
        assert tuple(at_match) != got[:4], "the box is already final at the match: the lap after it is not shown"


def fuzz_frame(rng):
    w, h = int(rng.integers(1, 14)), int(rng.integers(1, 14))
    density = rng.choice([0.15, 0.4, 0.7])
    a = np.where(rng.random((h, w)) < density, rng.choice([129, 255, 200], (h, w)), 0).astype(np.uint8)
    a[rng.random((h, w)) < 0.08] = 128                   # foreground for gs_blobs, background for the walk
    return a


def fuzz_starts(rng, a, k):
    h, w = a.shape
    fg = np.argwhere(a > 128)
    out = []
    for _ in range(k):
        kind = rng.integers(0, 6)
        if kind <= 1 and len(fg):
            y, x = fg[rng.integers(0, len(fg))]
        elif kind == 2:
            x, y = int(rng.choice([0, w - 1])), int(rng.integers(0, h))
        elif kind == 3:
            x, y = int(rng.choice([w, M32, w + 1])), int(rng.choice([0, h - 1, h, M32]))
        else:
            x, y = int(rng.integers(0, w)), int(rng.integers(0, h))
        out.append((int(x), int(y)))
    if k > 1 and rng.random() < 0.3:
        out[-1] = out[0]                                 # a repeated start
    return out


def test_oracle_matches_the_reference_on_thousands_of_walks():
    """random sparse frames, starts on foreground, background, the frame edge and outside it, pixel values 128 and
    129, pre-filled visited maps and lists sharing one visited: returning and open walks against the compiled
    reference byte for byte, cycling walks against the literal walk capped past the closing lap's bound"""
    rng = np.random.default_rng(7)
    walks = {RETURNED: 0, OPEN: 0, CYCLE: 0}
    for it in range(1500):
        a = fuzz_frame(rng)
        v0 = np.where(rng.random(a.shape) < 0.1, rng.integers(1, 256, a.shape), 0).astype(np.uint8) \
            if it % 3 == 0 else np.zeros_like(a)
        starts = fuzz_starts(rng, a, int(rng.integers(1, 4)))
        v = v0.copy()
        rec, ends = o_trace(a, v, records(starts))
        rv = v0.copy()
        for k, s in enumerate(starts):
            walks[int(ends[k])] += 1
            if ends[k] == CYCLE:
                box, length, stopped = py_walk(a, rv, s, 2 * states(a.size) + 1)
                assert stopped is not None and tuple(box) + (length,) == fields(rec[k])[:4] + (fields(rec[k])[6],)
            elif L.have_ref():
                c = records([s])
                R().gs_trace_contour(L.img(a), L.img(rv), L.ptr(c))
                assert c.tobytes() == rec[k:k + 1].tobytes(), (it, k, s, fields(c[0]), fields(rec[k]))
            else:
                box, length, stopped = py_walk(a, rv, s, 2 * states(a.size) + 1)
                assert stopped is None and tuple(box) + (length,) == fields(rec[k])[:4] + (fields(rec[k])[6],)
        assert np.array_equal(rv, v), it
    print("\nwalks by end: %s" % walks)
    assert min(walks.values()) > 100


# ---- CPU: the library --------------------------------------------------------------------------------------------------
def _declared(path):
    txt = open(path).read()
    txt = txt[txt.rindex('extern "C" {'):]
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(gs_[a-z0-9_]+)\s*\(", txt)))


def test_companion_exports_exactly_its_header():
    from grayskull_b200 import build, contour
    build.build()
    declared = _declared(os.path.join(ROOT, "include", "grayskull_contour.h"))
    assert len(declared) == 4 and sorted(contour.SIGNATURES) == declared
    nm = subprocess.run(["nm", "-D", "--defined-only", contour.LIB_PATH], capture_output=True, text=True,
                        check=True).stdout
    assert sorted(ln.split()[-1] for ln in nm.splitlines() if " T " in ln) == declared
    needed = subprocess.run(["readelf", "-d", contour.LIB_PATH], capture_output=True, text=True, check=True).stdout
    assert "libgrayskull_b200" not in needed
    from grayskull_b200 import _lib
    main = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    assert "contour" not in main
    assert not any("k_contour" in k for k in L.sass_functions())
    assert contour.lib().gs_b200_contour_last_error() == b"no error"
    assert contour.lib().gs_b200_trace_contours_work_bytes(1920, 1080, 3) == 16 + 4 * 1920 * 1080 * 3
    assert contour.lib().gs_b200_trace_contours_work_bytes(M32, M32, M32) == (1 << 64) - 1


def test_header_compiles_as_c99(tmp_path):
    for first in ("", '#include "grayskull_b200.h"\n', '#include "grayskull_draw.h"\n'):
        src = tmp_path / "t.c"
        src.write_text(first + '#include "grayskull_contour.h"\n'
                       'int main(void) { struct gs_contour c = {{0, 0, 1, 1}, {0, 0}, GS_CONTOUR_CYCLE};\n'
                       '  return gs_b200_contour_last_error() == 0 && c.length == 2; }\n')
        r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-fsyntax-only",
                            "-I", os.path.join(ROOT, "include"), str(src)], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    assert not re.match(r"grayskull_b200.*\.h$", "grayskull_contour.h")


def test_contour_layout_matches_the_reference():
    assert contour_dtype().itemsize == 28
    if L.have_ref():
        c = records([(3, 4)])
        R().gs_trace_contour(L.img(np.zeros((8, 8), np.uint8)), L.img(np.zeros((8, 8), np.uint8)), L.ptr(c))
        assert fields(c[0]) == (3, 4, 1, 1, 3, 4, 1)


def _contour_sass():
    from grayskull_b200 import contour
    tool = L.cuda_tool("cuobjdump")
    if tool is None:
        pytest.skip("cuobjdump not found")
    listing = subprocess.run([tool, "-sass", contour.LIB_PATH], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for cubin in re.split(r"^\s*(?=code for sm_\w+\s*$)", listing, flags=re.M)[1:]:
        arch, *parts = re.split(r"^\s*Function : (\S+)\s*$", cubin, flags=re.M)
        for name in L.demangle(parts[0::2]):
            funcs[L.kernel_id(name)] = arch.strip().splitlines()[0]
    return funcs


def test_every_companion_kernel_is_sm90a_and_has_a_row():
    funcs = _contour_sass()
    assert set(funcs) == set(KERNELS)
    assert all(arch == "code for sm_90a" for arch in funcs.values())


def test_launches_go_through_the_companions_helper():
    d = os.path.join(ROOT, "grayskull_b200", "contour")
    text = {f: open(os.path.join(d, f)).read() for f in sorted(os.listdir(d))}
    sites = [(f, m.start()) for f, t in text.items() for m in re.finditer(r"<<<", t)]
    assert len(sites) == 1
    f, at = sites[0]
    assert text[f].rindex("static int launch(", 0, at) < at < text[f].index("cudaGetLastError")
    assert text[f].count("cudaGetLastError") == 1
    from grayskull_b200 import build
    assert not set(build.CONTOUR_SOURCES) & set(build.SOURCES)


def test_companion_object_makes_no_blocking_runtime_call():
    from grayskull_b200 import build
    nm = shutil.which("nm")
    if nm is None:
        pytest.skip("nm not found")
    blocking = re.compile(r"^(cudaMemcpy|cudaMemcpyToSymbol|cudaMemset|cudaMemcpy2D|cudaDeviceSynchronize|"
                          r"cudaStreamSynchronize|cudaEventSynchronize|cudaMalloc\w*|cudaFree\w*|cudaStreamCreate\w*|"
                          r"cudaStreamDestroy|cudaMemcpyAsync|cudaMemsetAsync)$")
    for s in build.CONTOUR_SOURCES:
        o = os.path.join(build.OBJ, s.replace(".cu", ".o"))
        syms = [ln.split()[-1] for ln in subprocess.run([nm, "-u", o], capture_output=True, text=True,
                                                         check=True).stdout.splitlines()]
        assert "cudaGetLastError" in syms
        assert not [x for x in syms if blocking.match(x)], syms


def test_empty_batch_and_missing_pointer_without_a_gpu():
    code = ("import ctypes as C, sys; sys.path.insert(0, %r); from grayskull_b200 import contour; "
            "L = contour.lib(); P = C.c_void_p(4096); rc = %s; print('rc', rc)")
    calls = {"trace": "L.gs_b200_trace_contours_batch(P, C.c_void_p(1 << 20), 8, 8, %d, %s, P, 4, P, P, 1 << 20, None)",
             "starts": "L.gs_b200_blob_contour_starts_batch(P, 8, 8, %d, P, P, 4, %s, None)"}
    for name, c in calls.items():
        ok = subprocess.run([sys.executable, "-c", code % (ROOT, c % (0, "P"))], capture_output=True, text=True,
                            timeout=120)
        assert ok.returncode == 0 and "rc 0" in ok.stdout, (name, ok.stdout, ok.stderr)
        bad = subprocess.run([sys.executable, "-c", code % (ROOT, c % (2, "None"))], capture_output=True, text=True,
                             timeout=120)
        assert bad.returncode != 0 and "Assertion failed: " in bad.stderr, (name, bad.stderr)
    empty = "L.gs_b200_trace_contours_batch(P, C.c_void_p(1 << 20), 0, 8, 2, P, P, 4, P, P, 1 << 20, None)"
    bad = subprocess.run([sys.executable, "-c", code % (ROOT, empty)], capture_output=True, text=True, timeout=120)
    assert bad.returncode != 0 and "Assertion failed: w > 0 && h > 0" in bad.stderr, bad.stderr


# ---- GPU ---------------------------------------------------------------------------------------------------------------
def clib():
    from grayskull_b200 import contour
    return contour.lib()


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()


def _s():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def walk_frame(w, h, seed, f):
    """binary blobs with 127 / 128 / 130 pixels, sparse random pixels of 128 / 129 / 255, or the 7x7 block tiled"""
    rng = np.random.default_rng(seed * 1000 + f)
    kind = f % 3
    if kind == 0:
        a = L.binary_like(w, h, seed + f, 0.3)
        a[rng.random((h, w)) < 0.01] = 128
        return a
    if kind == 1:
        return np.where(rng.random((h, w)) < 0.35, rng.choice([128, 129, 255], (h, w)), 0).astype(np.uint8)
    return np.tile(block7(), ((h + 6) // 7, (w + 6) // 7))[:h, :w].copy()


def gen_starts(rng, a, k):
    """boundary, interior, background and out-of-frame starts, and a repeat"""
    h, w = a.shape
    fg = a > 128
    pad = np.pad(fg, 1)
    inner = fg & pad[:-2, 1:-1] & pad[2:, 1:-1] & pad[1:-1, :-2] & pad[1:-1, 2:]
    pools = [np.argwhere(fg & ~inner), np.argwhere(inner), np.argwhere(~fg)]
    out = []
    for i in range(k):
        kind = i % 5 if i < 5 else int(rng.integers(0, 5))
        if kind < 3 and len(pools[kind]):
            y, x = pools[kind][rng.integers(0, len(pools[kind]))]
            out.append((int(x), int(y)))
        elif kind == 3:
            out.append([(w, int(rng.integers(0, h))), (int(rng.integers(0, w)), h), (M32, M32), (M32, 0)][i % 4])
        else:
            out.append((int(rng.integers(0, w)), int(rng.integers(0, h))))
    if k > 2:
        out[-1] = out[0]
    return out


class Case:
    """one trace call on n frames: frames, initial visited maps, per-frame records (stride slots, the ones past the
    starts random) and counts (None: all `stride`)"""

    def __init__(self, frames, visited, recs, counts, stride):
        self.frames, self.visited, self.recs, self.counts, self.stride = frames, visited, recs, counts, stride

    def used(self, f):
        return self.stride if self.counts is None else min(int(self.counts[f]), self.stride)

    def expected(self, ends_before):
        n = len(self.frames)
        recs, vis = [], []
        ends = ends_before.reshape(n, self.stride).copy()
        for f in range(n):
            c = self.used(f)
            v = self.visited[f].copy()
            r, e = o_trace(self.frames[f], v, self.recs[f][:c])
            full = self.recs[f].copy()
            full[:c] = r
            ends[f, :c] = e
            recs.append(full)
            vis.append(v)
        return np.concatenate(recs), ends.reshape(-1), np.stack(vis)

    def buffers(self, off=0, work_frames=None):
        import torch
        n, h, w = self.frames.shape
        self.img = Region(self.frames.nbytes, off, self.frames, seed=1)
        self.vis = Region(self.visited.nbytes, off + 1 if off else 0, self.visited, seed=2)
        self.con = Region(28 * n * self.stride, 4 * off, np.concatenate(self.recs), seed=3)
        self.end = Region(n * self.stride, off + 2 if off else 0, seed=4)
        self.count_t = None if self.counts is None else _dev(np.asarray(self.counts, np.uint32))
        m = n if work_frames is None else work_frames
        # the query leaves 16 bytes for aligning the owner maps: a work pointer off by `off` needs 16 - off of them
        self.work_bytes = clib().gs_b200_trace_contours_work_bytes(w, h, m) - off
        self.work = torch.empty(self.work_bytes + 16, dtype=torch.uint8, device="cuda")
        self.work_off = off
        return self

    def call(self, s=None, ends=True):
        n, h, w = self.frames.shape
        s = _s() if s is None else s
        cp = None if self.count_t is None else self.count_t.data_ptr()
        return clib().gs_b200_trace_contours_batch(self.img.ptr, self.vis.ptr, w, h, n, self.con.ptr, cp, self.stride,
                                                   self.end.ptr if ends else None, self.work.data_ptr() + self.work_off,
                                                   self.work_bytes, s)

    def check(self, what):
        want_c, want_e, want_v = self.expected(self.end.before())
        got_c = self.con.read(what).view(contour_dtype())
        got_e = self.end.read(what)
        got_v = self.vis.read(what).reshape(self.frames.shape)
        self.img.read(what)
        bad = [f for f in range(len(self.frames)) if not np.array_equal(got_v[f], want_v[f])]
        assert not bad, "%s: visited differs in frames %s" % (what, bad[:10])
        if got_c.tobytes() != want_c.tobytes():
            i = int(np.flatnonzero([a.tobytes() != b.tobytes() for a, b in zip(got_c, want_c)])[0])
            pytest.fail("%s: record %d (frame %d): got %s, want %s" % (what, i, i // self.stride, fields(got_c[i]),
                                                                         fields(want_c[i])))
        assert np.array_equal(got_e, want_e), "%s: ends differ at %s" % (what, np.flatnonzero(got_e != want_e)[:10])


def make_case(w, h, n, seed, stride=7, counts="random", prefill=True):
    rng = np.random.default_rng(seed)
    frames = np.stack([walk_frame(w, h, seed, f) for f in range(n)])
    visited = np.zeros_like(frames)
    if prefill:
        visited[1::2] = np.where(rng.random(frames[1::2].shape) < 0.05, rng.integers(1, 256, frames[1::2].shape), 0)
    recs = [records(gen_starts(rng, frames[f], stride), stride) for f in range(n)]
    if counts == "random":
        counts = [int(rng.integers(0, stride + 1)) for _ in range(n)]
        counts[0] = 0
        if n > 1:
            counts[1] = stride + 5                        # above the stride: `stride` records are traced
    return Case(frames, visited, recs, counts, stride)


SIZES = [(1, 300, 3), (300, 1, 3), (7, 7, 4), (612, 816, 3), (640, 480, 3), (1920, 1080, 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,n", SIZES, ids=["%dx%d" % (w, h) for w, h, _ in SIZES])
@pytest.mark.parametrize("layout", ["aligned", "misaligned", "counts-null"])
def test_trace_matches_the_oracle(lib, witness, w, h, n, layout):
    c = make_case(w, h, n, seed=w + 3 * h, counts=None if layout == "counts-null" else "random")

    def run():
        c.buffers(off=3 if layout == "misaligned" else 0)   # fresh inputs: the call updates visited in place
        rc, seen = traced(lambda: c.call())
        assert rc == 0, clib().gs_b200_contour_last_error()
        c.check("%dx%d %s" % (w, h, layout))
        return seen

    witnessed(witness, run, TRACE_KERNELS, "%dx%d %s" % (w, h, layout))


def spiral(w, h):
    """a 1-px square spiral, turns kept one pixel apart, from (0, 0) inwards"""
    a = np.zeros((h, w), np.uint8)
    x = y = d = turns = 0
    a[0, 0] = 255
    dirs = ((1, 0), (0, 1), (-1, 0), (0, -1))
    while turns < 2:
        dx, dy = dirs[d]
        nx, ny, fx, fy = x + dx, y + dy, x + 2 * dx, y + 2 * dy
        if 0 <= nx < w and 0 <= ny < h and not a[ny, nx] and not (0 <= fx < w and 0 <= fy < h and a[fy, fx]):
            x, y, turns = nx, ny, 0
            a[y, x] = 255
        else:
            d, turns = (d + 1) % 4, turns + 1
    return a


@pytest.mark.gpu
def test_long_walks_spiral_and_lines_both_ways(lib):
    """a spiral walked end to end and back (hundreds of thousands of steps) and 1-px lines from either end and the
    middle, next to short walks in the same call"""
    w, h = 640, 480
    sp = spiral(w, h)
    lines = np.zeros((h, w), np.uint8)
    lines[100, 50:600] = 255
    lines[150:450, 320] = 255
    for i in range(200):
        lines[200 + i, 20 + i] = 255
    frames = np.stack([sp, lines])
    starts = [[(0, 0), (1, 0), (5, 5)],
              [(50, 100), (599, 100), (320, 150), (320, 449), (20, 200), (219, 399), (300, 100), (320, 300)]]
    stride = 8
    c = Case(frames, np.zeros_like(frames), [records(s, stride) for s in starts], [3, 8], stride).buffers()
    assert c.call() == 0, clib().gs_b200_contour_last_error()
    c.check("spiral and lines")
    want_c, want_e, _ = c.expected(c.end.before())
    assert int(want_c[0]["length"]) == int((sp > 0).sum()) > w * h // 3


@pytest.mark.gpu
def test_chunked_workspace_matches_one_chunk(lib):
    """one frame per chunk, two, and all frames in one chunk give the same outputs"""
    for frames_per_chunk in (1, 2, 5):
        c = make_case(97, 61, 5, seed=12).buffers(work_frames=frames_per_chunk)
        assert c.call() == 0, clib().gs_b200_contour_last_error()
        c.check("%d frames per chunk" % frames_per_chunk)
    c = make_case(97, 61, 5, seed=12).buffers(off=3, work_frames=1)   # misaligned work: one frame still fits
    assert c.call() == 0, clib().gs_b200_contour_last_error()
    c.check("misaligned work")


@pytest.mark.gpu
def test_overlap_and_short_work_are_refused(lib):
    import torch
    buf = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    lst = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    p, lp = buf.data_ptr(), lst.data_ptr()
    L_ = clib()
    wb = L_.gs_b200_trace_contours_work_bytes(16, 16, 2)
    work = torch.empty(wb, dtype=torch.uint8, device="cuda")
    wp = work.data_ptr()
    assert L_.gs_b200_trace_contours_batch(p, p + 500, 16, 16, 2, lp, None, 2, None, wp, wb, _s()) == 1
    assert L_.gs_b200_trace_contours_batch(p + 500, p, 16, 16, 2, lp, None, 2, None, wp, wb, _s()) == 1
    assert b"InvalidValue" in L_.gs_b200_contour_last_error()
    assert wp % 16 == 0
    assert L_.gs_b200_trace_contours_batch(p, p + 512, 16, 16, 2, lp, None, 2, None, wp, 4 * 256 - 1, _s()) == 1
    assert L_.gs_b200_trace_contours_batch(p, p + 512, 16, 16, 2, lp, None, 2, None, wp + 1, 4 * 256 + 14, _s()) == 1
    assert L_.gs_b200_trace_contours_batch(p, p + 512, 16, 16, 2, lp, None, 2, None, wp + 1, 4 * 256 + 15, _s()) == 0
    assert L_.gs_b200_trace_contours_batch(p, p + 512, 16, 16, 2, lp, None, 2, None, wp, 4 * 256, _s()) == 0
    torch.cuda.synchronize()


# ---- GPU: starts and the blob chain ------------------------------------------------------------------------------------
def start_rule(labels, blob):
    """grayskull.c:303-318 for one record, inside the frame"""
    h, w = labels.shape
    x0, y0, bw, bh = (int(blob[k]) for k in ("bx", "by", "bw", "bh"))
    xe, ye = min((x0 + bw) & M32, w), min((y0 + bh) & M32, h)
    if x0 < xe and y0 < ye:
        hit = np.argwhere(labels[y0:ye, x0:xe] == int(blob["label"]))
        if len(hit):
            return x0 + int(hit[0][1]), y0 + int(hit[0][0])
    return x0, y0


def chain_frames():
    lena = np.ascontiguousarray(np.load(os.path.join(ROOT, "tests", "golden", "lena_golden.npz"))["lena"])
    nat = [L.natural_like(320, 240, s) for s in (1, 2)]
    return [lena] + [np.where(a > 128, 255, 0).astype(np.uint8) for a in nat] + nat


@pytest.mark.gpu
def test_blob_chain_matches_the_oracle(lib, witness):
    """gs_b200_blobs_batch -> starts -> trace, against gso_blobs, the start rule in numpy and gso_trace_contour, on lena
    (whose pixels of exactly 128 are blob foreground but not walk foreground) and thresholded and raw natural frames"""
    import torch
    from grayskull_b200 import api, contour
    nb = 200
    for a in chain_frames():
        h, w = a.shape
        src = torch.from_numpy(np.stack([a, a[::-1].copy()])).cuda()
        labels, blobs, counts = api.blobs_batch(src, nb)

        def run():
            starts, seen = traced(lambda: contour.blob_contour_starts_batch(labels, blobs, counts))
            (cons, ends, vis), seen2 = traced(lambda: contour.trace_contours_batch(src, starts, counts))
            got = contour.to_numpy(cons)
            got_e, got_v = ends.cpu().numpy(), vis.cpu().numpy()
            for f in range(2):
                fa = src[f].cpu().numpy()
                ol = np.zeros((h, w), np.uint16)
                ob = np.zeros(nb, L.BLOB_DTYPE)
                k = L.oracle().gso_blobs(L.ptr(fa), w, h, L.ptr(ol), L.ptr(ob), nb)
                assert int(counts[f]) == k
                st = [start_rule(ol, ob[i]) for i in range(k)]
                assert [(int(r["sx"]), int(r["sy"])) for r in got[f][:k]] == st
                v = np.zeros_like(fa)
                want, we = o_trace(fa, v, records(st, nb)[:k])
                assert got[f][:k].tobytes() == want.tobytes(), f
                assert np.array_equal(got_e[f][:k], we) and np.array_equal(got_v[f], v)
                assert (got[f][k:].view(np.uint32) == 0).all()
            return seen | seen2

        witnessed(witness, run, list(KERNELS), "blob chain %dx%d" % (w, h))
    assert any((np.asarray(a) == 128).any() for a in chain_frames())


# ---- GPU: limits ---------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_batches_above_the_grid_limit(lib):
    """65536 frames in one trace and one starts call"""
    import torch
    w, h, n, stride = 6, 5, 65536, 2
    rng = np.random.default_rng(5)
    frames = np.where(rng.random((n, h, w)) < 0.5, 255, 0).astype(np.uint8)
    recs = [records([(int(rng.integers(0, w)), int(rng.integers(0, h))) for _ in range(stride)], stride)
            for _ in range(n)]
    counts = rng.integers(0, 4, n).astype(np.uint32)
    counts[-1] = 2
    c = Case(frames, np.zeros_like(frames), recs, counts, stride).buffers()
    assert c.call() == 0, clib().gs_b200_contour_last_error()
    c.check("65536 frames")
    # starts: blob records over random labels, the last frame's records used in full
    labels = rng.integers(0, 4, (n, h, w)).astype(np.uint16)
    blobs = np.zeros((n, stride), L.BLOB_DTYPE)
    blobs["label"] = rng.integers(0, 4, (n, stride))
    blobs["bx"], blobs["by"] = rng.integers(0, w, (n, stride)), rng.integers(0, h, (n, stride))
    blobs["bw"], blobs["bh"] = rng.integers(1, w + 1, (n, stride)), rng.integers(1, h + 1, (n, stride))
    con = Region(28 * n * stride, 0, np.zeros(n * stride, contour_dtype()), seed=5)
    lt, bt, ct = _dev(labels), _dev(blobs), _dev(counts)
    assert clib().gs_b200_blob_contour_starts_batch(lt.data_ptr(), w, h, n, bt.data_ptr(), ct.data_ptr(), stride,
                                                    con.ptr, _s()) == 0
    got = con.read("starts").view(contour_dtype()).reshape(n, stride)
    for f in list(range(0, 50)) + list(range(n - 50, n)):
        for b in range(stride):
            want = start_rule(labels[f], blobs[f, b]) if b < min(counts[f], stride) else (0, 0)
            assert (int(got[f, b]["sx"]), int(got[f, b]["sy"])) == want, (f, b)
    assert (got.view(np.uint32).reshape(n, stride, 7)[:, :, [0, 1, 2, 3, 6]] == 0).all()


@pytest.mark.gpu
def test_tall_frame_starts(lib):
    """a blob whose label first appears on a row past 65535 * 8"""
    w, h = 5, 8 * 65535 + 40
    labels = np.zeros((1, h, w), np.uint16)
    labels[0, h - 20, 3] = 7
    labels[0, h - 19, 1] = 7
    blobs = np.zeros((1, 2), L.BLOB_DTYPE)
    blobs[0, 0] = (7, 2, 0, h - 30, w, 25, 0, 0)
    blobs[0, 1] = (9, 2, 1, 3, 2, 2, 0, 0)
    con = Region(56, 0, np.zeros(2, contour_dtype()), seed=6)
    lt, bt = _dev(labels), _dev(blobs)
    assert clib().gs_b200_blob_contour_starts_batch(lt.data_ptr(), w, h, 1, bt.data_ptr(), None, 2, con.ptr, _s()) == 0
    got = con.read("tall").view(contour_dtype())
    assert [(int(r["sx"]), int(r["sy"])) for r in got] == [(3, h - 20), (1, 3)]


@pytest.mark.gpu
def test_frames_past_4_gib(lib):
    """img and visited of 9 frames of 512 MiB: every frame's walk, the last frame's past 4 GiB"""
    import torch
    w, h, n = 32768, 16384 + 8, 9
    img = torch.zeros((n, h, w), dtype=torch.uint8, device="cuda")
    vis = torch.zeros_like(img)
    x0, y0 = w - 9, h - 7
    img[n - 1, y0:y0 + 5, x0:x0 + 5] = torch.from_numpy(TEST_C).cuda()
    img[n - 2, 3:10, 3:10] = torch.from_numpy(block7()).cuda()
    starts = np.zeros((n, 2), contour_dtype())
    for f in range(n):
        starts[f, 0]["sx"], starts[f, 0]["sy"] = 5, 5
        starts[f, 1]["sx"], starts[f, 1]["sy"] = (x0 + 1, y0) if f == n - 1 else (4, 4)
    con = _dev(starts)
    ends = torch.full((n * 2,), 9, dtype=torch.uint8, device="cuda")
    wb = clib().gs_b200_trace_contours_work_bytes(w, h, 1)
    work = torch.empty(wb, dtype=torch.uint8, device="cuda")
    assert clib().gs_b200_trace_contours_batch(img.data_ptr(), vis.data_ptr(), w, h, n, con.data_ptr(), None, 2,
                                               ends.data_ptr(), work.data_ptr(), wb, _s()) == 0
    got = con.cpu().numpy().view(contour_dtype()).reshape(n, 2)
    e = ends.cpu().numpy().reshape(n, 2)
    del work
    for f in range(n):
        fr = img[f, :, :].cpu().numpy() if f >= n - 2 else None
        for k in range(2):
            s = (int(starts[f, k]["sx"]), int(starts[f, k]["sy"]))
            if fr is None:
                assert fields(got[f, k]) == (s[0], s[1], 1, 1, s[0], s[1], 1) and e[f, k] == OPEN, (f, k)
                continue
            # the walk stays within 16 pixels of its start: the oracle on that window, shifted
            ox, oy = max(0, s[0] - 16), max(0, s[1] - 16)
            sub = np.ascontiguousarray(fr[oy:oy + 40, ox:ox + 40])
            v = np.zeros_like(sub)
            prior = records([(5 - ox, 5 - oy)]) if k == 1 and ox <= 5 and oy <= 5 else records([])
            o_trace(sub, v, prior)
            r, oe = o_trace(sub, v, records([(s[0] - ox, s[1] - oy)]))
            want = fields(r[0])
            assert fields(got[f, k]) == (want[0] + ox, want[1] + oy, want[2], want[3], s[0], s[1], want[6]), (f, k)
            assert e[f, k] == oe[0]
    nz = torch.nonzero(vis.view(n, -1).sum(1, dtype=torch.int64)).flatten().cpu().tolist()
    assert nz == list(range(n))
    last = vis[n - 1, y0:y0 + 5, x0:x0 + 5].cpu().numpy()
    assert np.array_equal(last, TEST_C_VISITED)
    assert int(vis[n - 1].sum(dtype=torch.int64)) == 255 * (int((TEST_C_VISITED > 0).sum()) + 1)


# ---- GPU: streams -------------------------------------------------------------------------------------------------------
def _sleep(s, cycles):
    import torch
    with torch.cuda.stream(s):
        torch.cuda._sleep(int(cycles))


def _stage(c, s, frames_dev, vis_dev, recs_dev):
    """the case's inputs copied into its buffers on stream s, behind whatever s holds"""
    import torch
    with torch.cuda.stream(s):
        c.img.t[c.img.off:c.img.off + c.img.nbytes].copy_(frames_dev)
        c.vis.t[c.vis.off:c.vis.off + c.vis.nbytes].copy_(vis_dev)
        c.con.t[c.con.off:c.con.off + c.con.nbytes].copy_(recs_dev)


@pytest.mark.gpu
def test_ordered_behind_a_sleeping_stream_without_a_host_wait(lib):
    import torch
    c = make_case(300, 200, 3, seed=21).buffers()
    s, u = torch.cuda.Stream(), torch.cuda.Stream()
    real = (_dev(c.frames), _dev(c.visited), _dev(np.concatenate(c.recs)))
    _stage(c, s, torch.zeros_like(real[0]), torch.zeros_like(real[1]), real[2])
    assert c.call(C.c_void_p(s.cuda_stream)) == 0      # warm
    torch.cuda.synchronize()
    _sleep(u, 400_000_000)
    _sleep(s, 200_000_000)
    _stage(c, s, *real)
    with torch.cuda.stream(s):
        c.end.t[c.end.off:c.end.off + c.end.nbytes].copy_(torch.from_numpy(c.end.before()).cuda())
    assert c.call(C.c_void_p(s.cuda_stream)) == 0
    s_done, u_done = s.query(), u.query()
    torch.cuda.synchronize()
    assert not s_done and not u_done, "the call waited for its stream or for the device"
    c.check("behind a sleep")


@pytest.mark.gpu
def test_two_streams_at_once(lib):
    import torch
    s0, s1 = torch.cuda.Stream(), torch.cuda.Stream()
    cases = [(make_case(300, 200, 3, seed=seed).buffers(), st) for seed, st in ((22, s0), (23, s1), (24, s0), (25, s1))]
    _sleep(s1, 50_000_000)
    for c, st in cases:
        assert c.call(C.c_void_p(st.cuda_stream)) == 0
    torch.cuda.synchronize()
    for c, _ in cases:
        c.check("two streams")


@pytest.mark.gpu
def test_graph_capture_and_replay_on_new_inputs(lib):
    import torch
    c = make_case(300, 200, 3, seed=26).buffers()
    ends0 = torch.from_numpy(c.end.before()).cuda()
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        assert c.call(C.c_void_p(s.cuda_stream)) == 0
    for seed in (31, 32):
        fresh = make_case(300, 200, 3, seed=seed)
        c.frames, c.visited, c.recs, c.counts = fresh.frames, fresh.visited, fresh.recs, fresh.counts
        with torch.cuda.stream(s):
            c.count_t.copy_(_dev(np.asarray(fresh.counts, np.uint32)))
            c.end.t[c.end.off:c.end.off + c.end.nbytes].copy_(ends0)
        _stage(c, s, _dev(fresh.frames), _dev(fresh.visited), _dev(np.concatenate(fresh.recs)))
        with torch.cuda.stream(s):
            g.replay()
        s.synchronize()
        c.check("replay %d" % seed)


# ---- GPU: the CLI stage -------------------------------------------------------------------------------------------------
def contour_line(f, a, nb):
    """the wasm demo's gs_detect_largest_blob_contour(a, nb) from the oracle, as gsb_magick prints it"""
    h, w = a.shape
    ol = np.zeros((h, w), np.uint16)
    ob = np.zeros(nb, L.BLOB_DTYPE)
    k = L.oracle().gso_blobs(L.ptr(a), w, h, L.ptr(ol), L.ptr(ob), nb)
    if k == 0:
        return "frame %d: no contour" % f
    largest = 0
    for i in range(1, k):
        if ob[i]["area"] > ob[largest]["area"]:
            largest = i
    if ob[largest]["area"] < 100:
        return "frame %d: no contour" % f
    s = start_rule(ol, ob[largest])
    r, e = o_trace(a, np.zeros_like(a), records([s]))
    x = fields(r[0])
    return "frame %d: contour start %d %d box %d %d %d %d length %d end %s" % (
        f, x[4], x[5], x[0], x[1], x[2], x[3], x[6], ("returned", "open", "cycle")[int(e[0])])


@pytest.mark.gpu
def test_gsb_magick_contour_stage_matches_the_oracle_chain(lib, tmp_path):
    from grayskull_b200 import build
    exe = os.path.join(os.path.dirname(build.LIB), "gsb_magick")
    lena = np.ascontiguousarray(np.load(os.path.join(ROOT, "tests", "golden", "lena_golden.npz"))["lena"])
    h, w = lena.shape
    small = np.zeros((h, w), np.uint8)
    small[10:19, 10:19] = 255                                # area 81: below 100
    frames = [lena, np.ascontiguousarray(lena[::-1, ::-1]), np.where(L.natural_like(w, h, 3) > 128, 255, 0),
              L.binary_like(w, h, 4, 0.3), np.zeros((h, w)), small]
    frames = [np.ascontiguousarray(a, dtype=np.uint8) for a in frames]
    ins = []
    for f, a in enumerate(frames):
        p = tmp_path / ("in%d.pgm" % f)
        p.write_bytes(b"P5\n%d %d\n255\n" % (w, h) + a.tobytes())
        ins.append(str(p))
    r = subprocess.run([exe, "contour:50", str(tmp_path / "o_")] + ins, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("frame ")]
    want = [contour_line(f, a, 50) for f, a in enumerate(frames)]
    print("\n" + "\n".join(lines))
    assert lines == want
    assert sum("no contour" in ln for ln in lines) == 2
    for f, a in enumerate(frames):
        data = (tmp_path / ("o_%04d.pgm" % f)).read_bytes()
        assert data.endswith(a.tobytes())
