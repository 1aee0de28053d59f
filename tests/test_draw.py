"""The reference CLI's annotated pictures on the device (include/grayskull_draw.h, libgrayskull_draw.so): the blobs,
keypoints, faces and orb verbs of nanomagick.c, bit-exact.

The pictures are restated here in numpy from the verbs' code (blobs_picture, keypoints_picture, rects_picture,
matches_picture).  On the CPU those restatements are pinned byte for byte against the compiled verb
(oracle/_ref/nanomagick_cpu, when the reference was present at build time), and the companion library is checked as a
library: its exports, its header, its SASS, its one launch site and the runtime calls its object makes.  On the GPU
every call is checked against the restatement, bytes outside dst included, with a census of the kernels it launched;
then on the caller's stream, two streams and a CUDA graph; then the gsb_magick stages against the verb frame by frame.
"""
import ctypes as C
import hashlib
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
POISON = 0xA5

# every kernel of libgrayskull_draw.so, and which call launches it
KERNELS = {
    "gsb::k_draw_copy": "keypoints, rects (not in place)",
    "gsb::k_draw_blobs": "blobs",
    "gsb::k_draw_keypoints": "keypoints",
    "gsb::k_draw_rects": "rects",
    "gsb::k_draw_canvas": "matches",
    "gsb::k_draw_match_lines": "matches",
}


# ---- the verbs, restated ---------------------------------------------------------------------------------------------
def i32(v):
    """an unsigned 32-bit value taken as int, as gcc converts it"""
    v = int(v) & M32
    return v - (1 << 32) if v >= 1 << 31 else v


def blob_spans(boxes, w, h):
    """nanomagick.c:161-167 per record -> the rectangles (ya, yb, xa, xb), inclusive, of the frame it covers: rows
    y1..y2 times columns x1..x2 of linear indices, so x2 == w also covers column 0 one row down; indices >= w*h dropped"""
    out = []
    for x, y, bw, bh in boxes:
        x1, y1 = max(0, i32(int(x) - 2)), max(0, i32(int(y) - 2))
        x2, y2 = min(w, (int(x) + int(bw) + 2) & M32), min(h, (int(y) + int(bh) + 2) & M32)
        if x1 > x2 or y1 > y2:
            continue
        if x1 <= min(x2, w - 1) and y1 <= h - 1:
            out.append((y1, min(y2, h - 1), x1, min(x2, w - 1)))
        if x2 == w and y1 + 1 <= min(y2 + 1, h - 1):
            out.append((y1 + 1, min(y2 + 1, h - 1), 0, 0))
    return out


def blobs_picture(a, boxes):
    """the blobs verb's picture of frame a (h, w) for the records' boxes (x, y, w, h): a 2-D difference array, so the
    cost does not follow the boxes' areas"""
    h, w = a.shape
    d = np.zeros((h + 1, w + 1), np.int64)
    for ya, yb, xa, xb in blob_spans(boxes, w, h):
        d[ya, xa] += 1
        d[ya, xb + 1] -= 1
        d[yb + 1, xa] -= 1
        d[yb + 1, xb + 1] += 1
    cov = np.cumsum(np.cumsum(d, 0), 1)[:h, :w] > 0
    return np.where(a > 128, 255, np.where(cov, 128, 0)).astype(np.uint8)


def blobs_picture_literal(a, boxes):
    """the verb's loops over linear indices, as written (small inputs only)"""
    h, w = a.shape
    out = np.zeros(w * h, np.uint8)
    for x, y, bw, bh in boxes:
        x1, y1 = max(0, i32(int(x) - 2)), max(0, i32(int(y) - 2))
        x2, y2 = min(w, (int(x) + int(bw) + 2) & M32), min(h, (int(y) + int(bh) + 2) & M32)
        for yy in range(y1, y2 + 1):
            for xx in range(x1, x2 + 1):
                i = (yy * w + xx) & M32
                if i < w * h:
                    out[i] = 128
    out[a.reshape(-1) > 128] = 255
    return out.reshape(h, w)


def keypoints_picture(a, xyr, top):
    """nanomagick.c:229-239 for keypoints (x, y, response): a stable sort by descending response, crosses at the first
    top"""
    out = a.copy()
    h, w = a.shape
    order = sorted(range(len(xyr)), key=lambda i: -int(xyr[i][2]))
    for i in order[:min(top, len(xyr))]:
        x, y = int(xyr[i][0]), int(xyr[i][1])
        for d in range(-2, 3):
            for px, py in ((x, (y + d) & M32), ((x + d) & M32, y)):
                if px < w and py < h:
                    out[py, px] = 255
    return out


def _span(out, horizontal, fixed, a, b):
    h, w = out.shape
    lim, other = (w, h) if horizontal else (h, w)
    if not 0 <= fixed < other:
        return
    lo, hi = max(min(a, b), 0), min(max(a, b), lim - 1)
    if lo <= hi:
        if horizontal:
            out[fixed, lo:hi + 1] = 255
        else:
            out[lo:hi + 1, fixed] = 255


def rects_picture(a, rects):
    """nanomagick.c:369-375: four draw_line calls per rect; an axis-aligned draw_line visits every pixel between its
    ends (the unsigned sums taken as int)"""
    out = a.copy()
    for x, y, rw, rh in rects:
        x, y, xw, yh = i32(x), i32(y), i32(int(x) + int(rw)), i32(int(y) + int(rh))
        _span(out, True, y, x, xw)
        _span(out, True, yh, x, xw)
        _span(out, False, x, y, yh)
        _span(out, False, xw, y, yh)
    return out


def draw_line(img, x1, y1, x2, y2):
    """draw_line, nanomagick.c:172-184, as written"""
    h, w = img.shape
    dx, dy = abs(i32(x2) - i32(x1)), abs(i32(y2) - i32(y1))
    sx, sy = (1 if x1 < x2 else -1), (1 if y1 < y2 else -1)
    err, x, y = dx - dy, i32(x1), i32(y1)
    while True:
        if 0 <= x < w and 0 <= y < h:
            img[y, x] = 255
        if x == i32(x2) and y == i32(y2):
            break
        e2 = 2 * err
        if e2 > -dy:
            err -= dy
            x += sx
        if e2 < dx:
            err += dx
            y += sy


def exchange_order(d):
    """nanomagick.c:315-321 on distances d -> the slots in the sorted order (the whole sort, as the verb runs it)"""
    s = list(range(len(d)))
    for i in range(len(s) - 1):
        for j in range(i + 1, len(s)):
            if d[s[j]] < d[s[i]]:
                s[i], s[j] = s[j], s[i]
    return s


def matches_picture(a, tpl, k1, k2, m, top):
    """nanomagick.c:322-343: the side-by-side canvas and the first `top` matches of the exchange sort as lines; k1 /
    k2 arrays of (x, y), m of (idx1, idx2, distance).  Matches whose keypoint is outside its image are skipped."""
    h, w = a.shape
    th, tw = tpl.shape
    out = np.zeros((max(th, h), tw + w), np.uint8)
    out[:th, :tw] = tpl
    out[:h, tw:] = a
    order = exchange_order([int(r[2]) for r in m])
    for s in order[:top]:
        i1, i2 = int(m[s][0]), int(m[s][1])
        if i1 >= len(k1) or i2 >= len(k2):
            continue
        x1, y1 = int(k1[i1][0]), int(k1[i1][1])
        x2, y2 = int(k2[i2][0]), int(k2[i2][1])
        if x1 >= tw or y1 >= th or x2 >= w or y2 >= h:
            continue
        draw_line(out, x1, y1, x2 + tw, y2)
    return out


# ---- inputs ------------------------------------------------------------------------------------------------------------
def _lena():
    return np.ascontiguousarray(np.load(os.path.join(ROOT, "tests", "golden", "lena_golden.npz"))["lena"])


def _pgm(path, a):
    with open(path, "wb") as f:
        f.write(b"P5\n%d %d\n255\n" % (a.shape[1], a.shape[0]) + np.ascontiguousarray(a).tobytes())
    return str(path)


def _read_pgm(path):
    data = open(path, "rb").read()
    m = re.match(rb"P5\s+(\d+)\s+(\d+)\s+255\s", data)
    w, h = int(m.group(1)), int(m.group(2))
    return np.frombuffer(data[m.end():], np.uint8).reshape(h, w)


def _cascade():
    import grayskull_b200
    return grayskull_b200.load_cascade()


def _nanomagick():
    path = os.path.join(ROOT, "oracle", "_ref", "nanomagick_cpu")
    return path if os.path.exists(path) else None


def _blobs(a, nb):
    """gs_blobs of frame a (the oracle) -> records as BLOB_DTYPE"""
    O = L.oracle()
    h, w = a.shape
    labels = np.zeros((h, w), np.uint16)
    b = np.zeros(max(nb, 1), L.BLOB_DTYPE)
    n = O.gso_blobs(L.ptr(a), w, h, L.ptr(labels), L.ptr(b), nb)
    return b[:n]


def _boxes(b):
    return [(int(r["bx"]), int(r["by"]), int(r["bw"]), int(r["bh"])) for r in b]


def verb_frames():
    """lena, a natural frame, a binary one with blobs on the right edge; no foreground in the last 5 rows, where the
    verb would write past its buffer"""
    rng = np.random.default_rng(3)
    fr = {"lena": _lena(), "natural": L.natural_like(200, 150, 4), "binary": L.binary_like(160, 120, 5, 0.3)}
    edge = np.zeros((90, 120), np.uint8)
    edge[10:30, 100:] = 200       # touches the right edge: x2 == w, the wrap
    edge[40:60, 117:119] = 255    # ends one column short of it: x2 == w as well
    edge[70:80, 5:20] = 255
    edge[rng.random(edge.shape) < 0.01] = 255
    fr["edge"] = edge
    for a in fr.values():
        a[-5:] = 0
    return fr


def fast_keypoints(a, t):
    """gs_fast with cap 5000 on a zeroed score map, as the keypoints verb calls it"""
    return L.o_fast(L.oracle(), a, np.zeros_like(a), 5000, t)


def tie_cut(resp):
    """a top n whose cut falls inside a run of equal responses that are not adjacent in the list"""
    s = sorted(resp, reverse=True)
    for n in range(1, len(s)):
        if s[n - 1] == s[n] and sum(1 for r in resp if r == s[n]) >= 3:
            return n
    return None


# ---- CPU: the restatements ---------------------------------------------------------------------------------------------
def test_blob_restatement_is_the_verbs_loop():
    rng = np.random.default_rng(1)
    for trial in range(40):
        w, h = int(rng.integers(1, 30)), int(rng.integers(1, 30))
        a = rng.integers(0, 256, (h, w)).astype(np.uint8)
        boxes = [(int(rng.integers(0, w + 3)), int(rng.integers(0, h + 3)), int(rng.integers(0, w + 2)),
                  int(rng.integers(0, h + 2))) for _ in range(int(rng.integers(0, 6)))]
        boxes += [(w - 1, 0, 1, h), (0, h - 1, w, 1), (M32 - 1, 3, 5, 2), (3, 1 << 31, 2, 2)]
        assert np.array_equal(blobs_picture(a, boxes), blobs_picture_literal(a, boxes)), (trial, boxes)


def test_exchange_sort_is_not_stable_and_its_head_is_final_after_top_passes():
    d = [5, 3, 5, 1, 3, 5, 2, 1]
    full = exchange_order(d)
    assert [d[s] for s in full] == sorted(d)
    assert full != sorted(range(len(d)), key=lambda i: d[i])      # ties come out of list order
    rng = np.random.default_rng(2)
    for _ in range(50):
        d = list(rng.integers(0, 4, int(rng.integers(2, 40))))
        s = list(range(len(d)))
        top = int(rng.integers(1, len(d) + 1))
        for i in range(top):                                       # only the first top outer passes
            for j in range(i + 1, len(s)):
                if d[s[j]] < d[s[i]]:
                    s[i], s[j] = s[j], s[i]
        assert s[:top] == exchange_order(d)[:top]


@pytest.mark.skipif(_nanomagick() is None, reason="oracle/_ref/nanomagick_cpu not built (no reference checkout)")
def test_restatements_match_the_compiled_verbs(tmp_path):
    exe = _nanomagick()

    def verb(*args):
        r = subprocess.run([exe] + [str(x) for x in args], capture_output=True, text=True, timeout=300)
        return r

    checked = 0
    for name, a in verb_frames().items():
        src = _pgm(tmp_path / (name + ".pgm"), a)
        for nb in (3, 1000):
            assert verb("blobs", nb, src, tmp_path / "b.pgm").returncode == 0
            want = blobs_picture(a, _boxes(_blobs(a, nb)))
            assert np.array_equal(_read_pgm(tmp_path / "b.pgm"), want), (name, nb)
            checked += 1
        k = fast_keypoints(a, 20)
        resp = [int(r) for r in k["response"]]
        cut = tie_cut(resp)
        for top in sorted({1, 10, 100, 6000} | ({cut} if cut else set())):
            assert verb("keypoints", top, 20, src, tmp_path / "k.pgm").returncode == 0
            want = keypoints_picture(a, list(zip(k["x"], k["y"], k["response"])), top)
            assert np.array_equal(_read_pgm(tmp_path / "k.pgm"), want), (name, top)
            checked += 1
    # ties straddling the cut, on a frame whose FAST scores tie heavily
    lena = _lena()
    k = fast_keypoints(lena, 20)
    assert tie_cut([int(r) for r in k["response"]]) is not None
    # faces 1 and 2 on lena
    cas = _cascade()
    src = _pgm(tmp_path / "lena.pgm", lena)
    for mn in (1, 2):
        assert verb("faces", mn, src, tmp_path / ("f%d.pgm" % mn)).returncode == 0
        r = L.o_detect(L.oracle(), cas, L.o_integral(L.oracle(), lena), 100, 1.2, 1.0, 4.0, mn)
        assert len(r) > 0
        want = rects_picture(lena, [tuple(int(v) for v in x) for x in r])
        assert np.array_equal(_read_pgm(tmp_path / ("f%d.pgm" % mn)), want), mn
    assert hashlib.md5(open(tmp_path / "f2.pgm", "rb").read()).hexdigest() == "0fdde3c4c3121ebe696b2e9100615e6e"
    # orb: a pair with matches, and one without
    for name, (tpl, scene) in orb_pairs().items():
        out = tmp_path / ("o_%s.pgm" % name)
        r = verb("orb", _pgm(tmp_path / ("t_%s.pgm" % name), tpl), _pgm(tmp_path / ("s_%s.pgm" % name), scene), out)
        want = orb_picture(tpl, scene)
        if want is None:
            assert r.returncode != 0 and not out.exists(), name
        else:
            assert r.returncode == 0 and np.array_equal(_read_pgm(out), want), name
    assert checked >= 16


def orb_pairs():
    lena = _lena()
    return {"lena": (np.ascontiguousarray(lena[20:100, 10:110]), lena),
            "none": (lena, np.full((96, 128), 77, np.uint8))}


def orb_lists(tpl, scene):
    """the orb verb's keypoints of template and scene and its matches (nanomagick.c:299-311, the shared 1 MiB buffer
    included)"""
    Od = L.oracle()
    buf = np.zeros(1024 * 1024, np.uint8)
    kt = L.pyramid_orb(Od, tpl, 2500, 20, buf, 3)
    ks = L.pyramid_orb(Od, scene, 2500, 20, buf, 3)
    return kt, ks, L.o_match(Od, kt, ks, 300, 60.0)


def orb_picture(tpl, scene):
    kt, ks, m = orb_lists(tpl, scene)
    if len(m) == 0:
        return None
    return matches_picture(scene, tpl, list(zip(kt["x"], kt["y"])), list(zip(ks["x"], ks["y"])),
                           list(zip(m["idx1"], m["idx2"], m["distance"])), 15)


# ---- CPU: the library --------------------------------------------------------------------------------------------------
def _declared(path):
    txt = open(path).read()
    txt = txt[txt.rindex('extern "C" {'):]
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(gs_[a-z0-9_]+)\s*\(", txt)))


def test_companion_exports_exactly_its_header():
    from grayskull_b200 import build, draw
    build.build()
    declared = _declared(os.path.join(ROOT, "include", "grayskull_draw.h"))
    assert len(declared) == 5 and sorted(draw.SIGNATURES) == declared
    nm = subprocess.run(["nm", "-D", "--defined-only", draw.LIB_PATH], capture_output=True, text=True, check=True).stdout
    assert sorted(ln.split()[-1] for ln in nm.splitlines() if " T " in ln) == declared
    # not linked against the main library, which neither exports nor holds any of this
    needed = subprocess.run(["readelf", "-d", draw.LIB_PATH], capture_output=True, text=True, check=True).stdout
    assert "libgrayskull_b200" not in needed
    from grayskull_b200 import _lib
    main = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    assert "draw" not in main
    assert not any("k_draw" in k for k in L.sass_functions())
    assert draw.lib().gs_b200_draw_last_error() == b"no error"


def test_header_compiles_as_c99(tmp_path):
    for first in ("", '#include "grayskull_b200.h"\n'):
        src = tmp_path / "t.c"
        src.write_text(first + '#include "grayskull_draw.h"\nint main(void) { return gs_b200_draw_last_error() == 0; }\n')
        r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-fsyntax-only",
                            "-I", os.path.join(ROOT, "include"), str(src)], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    assert not re.match(r"grayskull_b200.*\.h$", "grayskull_draw.h")


def _draw_sass():
    from grayskull_b200 import draw
    tool = L.cuda_tool("cuobjdump")
    if tool is None:
        pytest.skip("cuobjdump not found")
    listing = subprocess.run([tool, "-sass", draw.LIB_PATH], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for cubin in re.split(r"^\s*(?=code for sm_\w+\s*$)", listing, flags=re.M)[1:]:
        arch, *parts = re.split(r"^\s*Function : (\S+)\s*$", cubin, flags=re.M)
        for name in L.demangle(parts[0::2]):
            funcs[L.kernel_id(name)] = arch.strip().splitlines()[0]
    return funcs


def test_every_companion_kernel_is_sm90a_and_has_a_row():
    funcs = _draw_sass()
    assert set(funcs) == set(KERNELS)
    assert all(arch == "code for sm_90a" for arch in funcs.values())


def test_launches_go_through_the_companions_helper():
    d = os.path.join(ROOT, "grayskull_b200", "draw")
    text = {f: open(os.path.join(d, f)).read() for f in sorted(os.listdir(d))}
    sites = [(f, m.start()) for f, t in text.items() for m in re.finditer(r"<<<", t)]
    assert len(sites) == 1
    f, at = sites[0]
    assert text[f].rindex("static int launch(", 0, at) < at < text[f].index("cudaGetLastError")
    assert text[f].count("cudaGetLastError") == 1
    from grayskull_b200 import build
    assert not set(build.DRAW_SOURCES) & set(build.SOURCES)


def test_companion_object_makes_no_blocking_runtime_call():
    from grayskull_b200 import build
    nm = shutil.which("nm")
    if nm is None:
        pytest.skip("nm not found")
    blocking = re.compile(r"^(cudaMemcpy|cudaMemcpyToSymbol|cudaMemset|cudaMemcpy2D|cudaDeviceSynchronize|"
                          r"cudaStreamSynchronize|cudaEventSynchronize|cudaMalloc\w*|cudaFree\w*|cudaStreamCreate\w*|"
                          r"cudaStreamDestroy|cudaMemcpyAsync|cudaMemsetAsync)$")
    for s in build.DRAW_SOURCES:
        o = os.path.join(build.OBJ, s.replace(".cu", ".o"))
        syms = [ln.split()[-1] for ln in subprocess.run([nm, "-u", o], capture_output=True, text=True,
                                                         check=True).stdout.splitlines()]
        assert "cudaGetLastError" in syms
        assert not [x for x in syms if blocking.match(x)], syms


def test_empty_batch_and_missing_pointer_without_a_gpu():
    code = ("import ctypes as C, sys; sys.path.insert(0, %r); from grayskull_b200 import draw; "
            "L = draw.lib(); P = C.c_void_p(4096); rc = %s; print('rc', rc)")
    calls = {"blobs": "L.gs_b200_draw_blobs_batch(P, P, 8, 8, %d, %s, P, 4, None)",
             "keypoints": "L.gs_b200_draw_keypoints_batch(P, P, 8, 8, %d, %s, P, 4, 3, None)",
             "rects": "L.gs_b200_draw_rects_batch(P, P, 8, 8, %d, %s, P, 4, None)",
             "matches": "L.gs_b200_draw_matches_batch(P, P, 8, 8, %d, P, 4, 4, %s, 0, P, 4, P, P, 4, 15, None)"}
    for name, c in calls.items():
        ok = subprocess.run([sys.executable, "-c", code % (ROOT, c % (0, "P"))], capture_output=True, text=True,
                            timeout=120)
        assert ok.returncode == 0 and "rc 0" in ok.stdout, (name, ok.stdout, ok.stderr)
        bad = subprocess.run([sys.executable, "-c", code % (ROOT, c % (2, "None"))], capture_output=True, text=True,
                             timeout=120)
        assert bad.returncode != 0 and "Assertion failed: " in bad.stderr, (name, bad.stderr)


# ---- GPU ---------------------------------------------------------------------------------------------------------------
def dlib():
    from grayskull_b200 import draw
    return draw.lib()


def _kp_records(xyr, stride, rng):
    """keypoint records (x, y, response) in a list of `stride` slots, the slots past them random"""
    k = np.frombuffer(rng.integers(0, 256, stride * 48, dtype=np.uint8).tobytes(), L.KP_DTYPE).copy()
    for i, (x, y, r) in enumerate(xyr):
        k[i]["x"], k[i]["y"], k[i]["response"] = x, y, r
    return k


def _blob_records(boxes, stride, rng):
    b = np.frombuffer(rng.integers(0, 256, stride * 32, dtype=np.uint8).tobytes(), L.BLOB_DTYPE).copy()
    for i, (x, y, bw, bh) in enumerate(boxes):
        b[i]["bx"], b[i]["by"], b[i]["bw"], b[i]["bh"] = x, y, bw, bh
    return b


def _rect_records(rects, stride, rng):
    r = np.frombuffer(rng.integers(0, 256, stride * 16, dtype=np.uint8).tobytes(), L.RECT_DTYPE).copy()
    for i, v in enumerate(rects):
        r[i] = tuple(int(x) & M32 for x in v)
    return r


def _raw(lists):
    """records back to back as bytes (np.concatenate would drop gs_blob's padding and pack it to 30 bytes)"""
    return np.concatenate([np.ascontiguousarray(x).view(np.uint8).reshape(-1) for x in lists])


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).cuda()


def _s():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


class Case:
    """one call on n frames of w x h: frames, per-frame lists (records already padded to the stride) and counts; the
    expected picture per frame comes from the restatement of the records each frame uses"""

    def __init__(self, kind, frames, lists, counts, stride, top=15, tpl=None, k1=None, k2=None):
        self.kind, self.frames, self.lists, self.counts, self.stride, self.top = kind, frames, lists, counts, stride, top
        self.tpl, self.k1, self.k2 = tpl, k1, k2

    def expected(self):
        out = []
        for f, a in enumerate(self.frames):
            c = min(int(self.counts[f]), self.stride)
            rec = self.lists[f][:c]
            if self.kind == "blobs":
                out.append(blobs_picture(a, [(r["bx"], r["by"], r["bw"], r["bh"]) for r in rec]))
            elif self.kind == "keypoints":
                out.append(keypoints_picture(a, list(zip(rec["x"], rec["y"], rec["response"])), self.top))
            elif self.kind == "rects":
                out.append(rects_picture(a, [tuple(r) for r in rec]))
            else:
                k1 = self.k1[0] if len(self.k1) == 1 else self.k1[f]
                out.append(matches_picture(a, self.tpl, list(zip(k1["x"], k1["y"])),
                                           list(zip(self.k2[f]["x"], self.k2[f]["y"])),
                                           [tuple(r) for r in rec], self.top))
        return np.stack(out)

    def out_shape(self):
        n, h, w = self.frames.shape
        if self.kind == "matches":
            th, tw = self.tpl.shape
            return (n, max(th, h), tw + w)
        return (n, h, w)

    def buffers(self, off=0, inplace=False):
        self.src = Region(self.frames.nbytes, off, self.frames, seed=1)
        self.dst = self.src if inplace else Region(int(np.prod(self.out_shape())), off + 1 if off else 0, seed=2)
        lists = _raw(self.lists)
        self.list_t = _dev(lists if lists.size else np.zeros(64, np.uint8))   # stride 0: a list nobody reads
        self.count_t = _dev(np.asarray(self.counts, np.uint32))
        if self.kind == "matches":
            self.tpl_t, self.k1_t, self.k2_t = _dev(self.tpl), _dev(_raw(self.k1)), _dev(_raw(self.k2))
        return self

    def call(self, s=None):
        n, h, w = self.frames.shape
        s = _s() if s is None else s
        D = dlib()
        lp, cp, dp, sp = self.list_t.data_ptr(), self.count_t.data_ptr(), self.dst.ptr, self.src.ptr
        if self.kind == "blobs":
            return D.gs_b200_draw_blobs_batch(dp, sp, w, h, n, lp, cp, self.stride, s)
        if self.kind == "keypoints":
            return D.gs_b200_draw_keypoints_batch(dp, sp, w, h, n, lp, cp, self.stride, self.top, s)
        if self.kind == "rects":
            return D.gs_b200_draw_rects_batch(dp, sp, w, h, n, lp, cp, self.stride, s)
        th, tw = self.tpl.shape
        s1 = 0 if len(self.k1) == 1 else len(self.k1[0])
        return D.gs_b200_draw_matches_batch(dp, sp, w, h, n, self.tpl_t.data_ptr(), tw, th, self.k1_t.data_ptr(), s1,
                                            self.k2_t.data_ptr(), len(self.k2[0]), lp, cp, self.stride, self.top, s)

    def check(self, what):
        got = self.dst.read(what).reshape(self.out_shape())
        want = self.expected()
        bad = [f for f in range(len(want)) if not np.array_equal(got[f], want[f])]
        if bad:
            at = np.argwhere(got[bad[0]] != want[bad[0]])[:8]
            pytest.fail("%s: frames %s differ; frame %d at %s: got %s, want %s" % (
                what, bad[:10], bad[0], at.tolist(), [int(got[bad[0]][tuple(p)]) for p in at],
                [int(want[bad[0]][tuple(p)]) for p in at]))


KINDS = {"blobs": ["gsb::k_draw_blobs"], "keypoints": ["gsb::k_draw_copy", "gsb::k_draw_keypoints"],
         "rects": ["gsb::k_draw_copy", "gsb::k_draw_rects"], "matches": ["gsb::k_draw_canvas", "gsb::k_draw_match_lines"]}


def make_case(kind, w, h, n, seed, stride=None, top=15, counts=None, huge=False):
    rng = np.random.default_rng(seed)
    frames = np.stack([[rng.integers(0, 256, (h, w), dtype=np.uint8), L.natural_like(w, h, seed + f),
                        L.binary_like(w, h, seed + f, 0.3)][f % 3] for f in range(n)])
    stride = 40 if stride is None else stride
    if counts is None:
        counts = [int(rng.integers(0, stride + 1)) for _ in range(n)]
        counts[0] = 0
        if n > 1:
            counts[1] = stride + 7             # above the stride: only `stride` records are used
    lists = []
    for f in range(n):
        k = stride
        if kind == "blobs":
            boxes = [(int(rng.integers(0, w)), int(rng.integers(0, h)), int(rng.integers(1, w // 2 + 2)),
                      int(rng.integers(1, h // 2 + 2))) for _ in range(k)]
            boxes[:4] = [(w - 3, 1, 3, 4), (w - 1, h - 2, 1, 2), (0, 0, w, h), (w - 6, h // 2, 4, 3)][:k]
            if huge:
                boxes[4:8] = [(M32 - 1, 5, 9, 3), (1 << 31, 0, 5, 5), (3, M32 - 2, 4, 9), (M32, M32, 10, 10)]
            lists.append(_blob_records(boxes, stride, rng))
        elif kind == "keypoints":
            xyr = [(int(rng.integers(0, w)), int(rng.integers(0, h)), int(rng.integers(0, 4))) for _ in range(k)]
            xyr[:4] = [(0, 0, 3), (w - 1, h - 1, 3), (1, h - 2, 2), (w - 2, 1, 2)][:k]
            if huge:
                xyr[4:7] = [(M32, 3, 3), (2, M32 - 1, 3), (w + 1, h + 1, 3)]
            lists.append(_kp_records(xyr, stride, rng))
        elif kind == "rects":
            if huge:
                big = [0, 1, w - 1, w, h, 1 << 31, (1 << 31) - 1, M32, M32 - 3, 1 << 30]
                rects = [tuple(int(rng.choice(big)) for _ in range(4)) for _ in range(k)]
            else:
                rects = [(int(rng.integers(0, w + 4)), int(rng.integers(0, h + 4)), int(rng.integers(0, w)),
                          int(rng.integers(0, h))) for _ in range(k)]
            lists.append(_rect_records(rects, stride, rng))
        else:
            pass
    if kind != "matches":
        return Case(kind, frames, lists, counts, stride, top)
    th, tw = int(rng.integers(8, 40)), int(rng.integers(8, 40))
    tpl = rng.integers(0, 256, (th, tw), dtype=np.uint8)
    n1, n2 = 30, 35
    k1 = [_kp_records([(int(rng.integers(0, tw + (2 if huge else 0))), int(rng.integers(0, th)), 0) for _ in range(n1)],
                      n1, rng)]
    if n > 1 and seed % 4 == 1:
        k1 = [_kp_records([(int(rng.integers(0, tw)), int(rng.integers(0, th)), 0) for _ in range(n1)], n1, rng)
              for _ in range(n)]
    k2 = [_kp_records([(int(rng.integers(0, w + (2 if huge else 0))), int(rng.integers(0, h)), 0) for _ in range(n2)],
                      n2, rng) for _ in range(n)]
    for f in range(n):
        m = np.zeros(stride, L.MATCH_DTYPE)
        m["idx1"] = rng.integers(0, n1, stride)
        m["idx2"] = rng.integers(0, n2, stride)
        m["distance"] = rng.integers(0, 5, stride)         # heavy ties, which the exchange sort reorders
        lists.append(m)
    return Case(kind, frames, lists, counts, stride, top, tpl, k1, k2)


CASES = [
    ("blobs", dict(w=70, h=45, n=4, seed=1)),
    ("blobs", dict(w=1030, h=33, n=3, seed=2, huge=True)),             # two column tiles, odd row band
    ("blobs", dict(w=64, h=24, n=2, seed=3, stride=0)),
    ("keypoints", dict(w=61, h=37, n=4, seed=4, top=7)),
    ("keypoints", dict(w=48, h=32, n=3, seed=5, top=0)),
    ("keypoints", dict(w=48, h=32, n=3, seed=6, top=1, huge=True)),
    ("keypoints", dict(w=97, h=40, n=3, seed=7, top=1000)),
    ("keypoints", dict(w=97, h=40, n=2, seed=8, top=9, stride=700)),    # more keypoints than one CTA's pass
    ("rects", dict(w=80, h=50, n=4, seed=9)),
    ("rects", dict(w=80, h=50, n=3, seed=10, huge=True)),
    ("matches", dict(w=60, h=40, n=3, seed=11)),                        # one template list: stride1 == 0
    ("matches", dict(w=60, h=25, n=3, seed=13, top=1)),                 # per-frame template lists, th > h possible
    ("matches", dict(w=50, h=40, n=3, seed=15, top=0)),
    ("matches", dict(w=50, h=40, n=3, seed=17, top=100, huge=True)),
]
CASE_IDS = ["%s-%d" % (k, p["seed"]) for k, p in CASES]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,p", CASES, ids=CASE_IDS)
@pytest.mark.parametrize("layout", ["aligned", "misaligned", "in-place"])
def test_call_matches_restatement(lib, witness, kind, p, layout):
    if layout == "in-place" and kind == "matches":
        pytest.skip("the orb picture is not the frame's size")
    c = make_case(kind, **p).buffers(off=3 if layout == "misaligned" else 0, inplace=layout == "in-place")

    def run():
        rc, seen = traced(lambda: c.call())
        assert rc == 0, dlib().gs_b200_draw_last_error()
        c.check("%s %s" % (kind, layout))
        return seen

    kernels = [k for k in KINDS[kind] if not (layout == "in-place" and k == "gsb::k_draw_copy")
               and not (p.get("top") == 0 and k in ("gsb::k_draw_keypoints", "gsb::k_draw_match_lines"))]
    witnessed(witness, run, kernels, "%s %s" % (kind, layout))


@pytest.mark.gpu
def test_overlap_is_refused(lib):
    import torch
    buf = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    lst = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    p = buf.data_ptr()
    D = dlib()
    assert D.gs_b200_draw_blobs_batch(p + 8, p, 16, 16, 2, lst.data_ptr(), lst.data_ptr(), 1, _s()) == 1
    assert D.gs_b200_draw_rects_batch(p, p + 1, 16, 16, 2, lst.data_ptr(), lst.data_ptr(), 1, _s()) == 1
    assert D.gs_b200_draw_matches_batch(p, p + 100, 16, 16, 1, p + 3000, 4, 4, lst.data_ptr(), 0, lst.data_ptr(), 1,
                                        lst.data_ptr(), lst.data_ptr(), 1, 15, _s()) == 1
    assert D.gs_b200_draw_matches_batch(p, p + 1000, 16, 16, 1, p + 3000, 4, 4, lst.data_ptr(), 0, lst.data_ptr(), 1,
                                        lst.data_ptr(), lst.data_ptr(), 20000, 15, _s()) == 1
    assert b"InvalidValue" in D.gs_b200_draw_last_error()


@pytest.mark.gpu
def test_nested_blobs_at_the_record_limit_cost_what_disjoint_ones_do(lib):
    """65534 nested boxes (rings and holes nest) are drawn exactly, and take about the time of as many small ones"""
    import torch
    w, h, k = 1024, 768, 65534
    rng = np.random.default_rng(4)
    a = L.binary_like(w, h, 9, 0.4)
    nested = [(i % 380, (i * 7) % 380, w - 2 * (i % 380), h - 2 * ((i * 7) % 380)) for i in range(k)]
    small = [(int(rng.integers(0, w - 4)), int(rng.integers(0, h - 4)), 3, 3) for _ in range(k)]
    times = {}
    for name, boxes in (("nested", nested), ("small", small)):
        c = Case("blobs", a[None], [_blob_records(boxes, k, rng)], [k], k).buffers()
        assert c.call() == 0
        c.check(name)
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(20):
            c.call()
        e.record()
        torch.cuda.synchronize()
        times[name] = s.elapsed_time(e) / 20
    area = sum(bw * bh for _, _, bw, bh in nested) / sum(bw * bh for _, _, bw, bh in small)
    print("\nnested %.3f ms, small %.3f ms, area ratio %.0f" % (times["nested"], times["small"], area))
    assert area > 1000 and times["nested"] < 3 * times["small"] + 0.05


@pytest.mark.gpu
@pytest.mark.parametrize("kind", list(KINDS))
def test_batches_above_the_grid_limit_and_tall_frames(lib, kind):
    """65540 frames in one call, and one frame of more than 65535 tiles of 8 rows"""
    for w, h, n in ((8, 3, 65540), (5, 8 * 65535 + 11, 1)):
        rng = np.random.default_rng(n)
        frames = rng.integers(0, 256, (n, h, w), dtype=np.uint8)
        stride = 3
        counts = rng.integers(0, 5, n).astype(np.uint32)
        if kind == "blobs":
            lists = [_blob_records([(int(rng.integers(0, w)), int(rng.integers(0, h)), 3, 2) for _ in range(3)], 3, rng)
                     for _ in range(n)]
            if n == 1:
                lists[-1] = _blob_records([(w - 2, h - 9, 2, 5), (0, 65535 * 8 - 3, w, 6), (1, 2, 1, 1)], 3, rng)
        elif kind == "keypoints":
            lists = [_kp_records([(int(rng.integers(0, w)), int(rng.integers(0, h)), int(rng.integers(0, 3)))
                                  for _ in range(3)], 3, rng) for _ in range(n)]
        elif kind == "rects":
            lists = [_rect_records([(int(rng.integers(0, w)), int(rng.integers(0, h)), 2, int(rng.integers(0, h)))
                                    for _ in range(3)], 3, rng) for _ in range(n)]
        else:
            lists = []
            for _ in range(n):
                m = np.zeros(3, L.MATCH_DTYPE)
                m["idx1"], m["idx2"], m["distance"] = rng.integers(0, 2, 3), 0, rng.integers(0, 3, 3)
                lists.append(m)
        counts[-1] = 3
        if kind == "matches":
            tpl = rng.integers(0, 256, (4, 3), dtype=np.uint8)
            k1 = [_kp_records([(1, 1, 0), (2, 3, 0)], 2, rng)]
            k2 = [_kp_records([(int(rng.integers(0, w)), int(rng.integers(0, h)), 0)], 1, rng) for _ in range(n)]
            c = Case(kind, frames, lists, counts, stride, 2, tpl, k1, k2)
        else:
            c = Case(kind, frames, lists, counts, stride, 2)
        if n > 1:   # the restatement per frame would take minutes: check the distinct frames a sample stands for
            c.buffers()
            assert c.call() == 0, dlib().gs_b200_draw_last_error()
            got = c.dst.read(kind).reshape(c.out_shape())
            for f in list(range(0, 4)) + list(range(65530, n)):
                sub = Case(kind, frames[f:f + 1], [lists[f]], [counts[f]], stride, 2, c.tpl, c.k1,
                           None if c.k2 is None else [c.k2[f]])
                assert np.array_equal(got[f], sub.expected()[0]), (kind, f)
        else:
            c.buffers()
            assert c.call() == 0, dlib().gs_b200_draw_last_error()
            c.check("%s tall" % kind)


@pytest.mark.gpu
def test_copy_past_4_gib(lib):
    """the keypoint call's copy and its crosses in frames past 4 GiB"""
    import torch
    w, h, n = 32768, 16384 + 8, 9          # 4.83 GB
    src = torch.randint(0, 256, (n, h, w), dtype=torch.uint8, device="cuda")
    dst = torch.empty_like(src)
    xyr = [[(5, 5, 1), (w - 1, h - 1, 2), (100, h - 2, 2)] for _ in range(n)]
    kp = _raw([_kp_records(x, 3, np.random.default_rng(f)) for f, x in enumerate(xyr)])
    kps, counts = _dev(kp), _dev(np.full(n, 3, np.uint32))
    assert dlib().gs_b200_draw_keypoints_batch(dst.data_ptr(), src.data_ptr(), w, h, n, kps.data_ptr(),
                                               counts.data_ptr(), 3, 2, _s()) == 0
    want = src.clone()
    for f in range(n):
        for x, y, _ in xyr[f][1:]:
            want[f, max(0, y - 2):y + 3, x] = 255
            want[f, y, max(0, x - 2):x + 3] = 255
    torch.cuda.synchronize()
    assert torch.equal(dst, want)


# ---- GPU: streams -------------------------------------------------------------------------------------------------------
STREAM_CASES = [("blobs", dict(w=300, h=200, n=3, seed=21)), ("keypoints", dict(w=300, h=200, n=3, seed=22)),
                ("rects", dict(w=300, h=200, n=3, seed=23)), ("matches", dict(w=300, h=200, n=3, seed=25))]


def _sleep(s, cycles):
    import torch
    with torch.cuda.stream(s):
        torch.cuda._sleep(int(cycles))


def _stage(c, s, frames_dev):
    """the case's frames (a device tensor) copied into src on stream s, behind whatever s holds; dst poisoned"""
    import torch
    with torch.cuda.stream(s):
        c.src.t[c.src.off:c.src.off + c.src.nbytes].copy_(frames_dev)
        c.dst.t[c.dst.off:c.dst.off + c.dst.nbytes].fill_(POISON)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,p", STREAM_CASES, ids=[k for k, _ in STREAM_CASES])
def test_ordered_behind_a_sleeping_stream_without_a_host_wait(lib, kind, p):
    import torch
    c = make_case(kind, **p).buffers()
    s, u = torch.cuda.Stream(), torch.cuda.Stream()
    real = _dev(c.frames)
    _stage(c, s, torch.zeros_like(real))
    assert c.call(C.c_void_p(s.cuda_stream)) == 0      # warm
    torch.cuda.synchronize()
    _sleep(u, 400_000_000)
    _sleep(s, 200_000_000)
    _stage(c, s, real)
    assert c.call(C.c_void_p(s.cuda_stream)) == 0
    s_done, u_done = s.query(), u.query()
    torch.cuda.synchronize()
    assert not s_done and not u_done, "the call waited for its stream or for the device"
    c.check(kind + " behind a sleep")


@pytest.mark.gpu
def test_two_streams_at_once(lib):
    import torch
    s0, s1 = torch.cuda.Stream(), torch.cuda.Stream()
    cases = [(make_case(k, **dict(p, seed=p["seed"] + off)).buffers(), st)
             for k, p in STREAM_CASES for off, st in ((0, s0), (100, s1))]
    _sleep(s1, 50_000_000)
    for c, st in cases:
        assert c.call(C.c_void_p(st.cuda_stream)) == 0
    torch.cuda.synchronize()
    for c, _ in cases:
        c.check(c.kind + " on two streams")


@pytest.mark.gpu
@pytest.mark.parametrize("kind,p", STREAM_CASES, ids=[k for k, _ in STREAM_CASES])
def test_graph_capture_and_replay_on_new_inputs(lib, kind, p):
    import torch
    c = make_case(kind, **p).buffers()
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        assert c.call(C.c_void_p(s.cuda_stream)) == 0
    for seed in (31, 32):
        fresh = make_case(kind, **dict(p, seed=seed))   # new frames, lists and counts in the captured buffers
        c.frames, c.lists, c.counts = fresh.frames, fresh.lists, fresh.counts
        with torch.cuda.stream(s):
            c.list_t.copy_(_dev(_raw(fresh.lists)))
            c.count_t.copy_(_dev(np.asarray(fresh.counts, np.uint32)))
        _stage(c, s, _dev(fresh.frames))
        with torch.cuda.stream(s):
            g.replay()
        s.synchronize()
        c.check("%s replay %d" % (kind, seed))


# ---- GPU: the CLI stages ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gsb_magick_stages_match_the_verb(lib, tmp_path):
    from grayskull_b200 import build
    exe = os.path.join(os.path.dirname(build.LIB), "gsb_magick")
    ref = _nanomagick()
    lena = _lena()
    frames = [lena, np.ascontiguousarray(lena[:, ::-1]), L.natural_like(128, 128, 2),
              L.binary_like(128, 128, 3, 0.3), np.full((128, 128), 77, np.uint8)]
    for a in frames:
        a[-5:] = 0                          # the blobs verb writes past its buffer for blobs near the bottom
    ins = [_pgm(tmp_path / ("in%d.pgm" % f), a) for f, a in enumerate(frames)]
    tpl = np.ascontiguousarray(lena[20:100, 10:110])
    tp = _pgm(tmp_path / "tpl.pgm", tpl)
    cas = _cascade()
    stages = {"draw-blobs:50": ("blobs", "50"), "draw-blobs:3": ("blobs", "3"),
              "draw-keypoints:100:20": ("keypoints", "100", "20"), "draw-keypoints:7:30": ("keypoints", "7", "30"),
              "faces:1": ("faces", "1"), "faces:2": ("faces", "2"), "draw-orb:" + tp: ("orb", tp)}
    for stage, verb in stages.items():
        prefix = tmp_path / ("o%d_" % abs(hash(stage)))
        r = subprocess.run([exe, stage, str(prefix)] + ins, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, (stage, r.stderr)
        lines = [ln for ln in r.stdout.splitlines() if ln.startswith("frame ")]
        for f, a in enumerate(frames):
            out = tmp_path / ("%s%04d.pgm" % (prefix, f))
            if verb[0] == "blobs":
                want = blobs_picture(a, _boxes(_blobs(a, int(verb[1]))))
            elif verb[0] == "keypoints":
                k = fast_keypoints(a, int(verb[2]))
                want = keypoints_picture(a, list(zip(k["x"], k["y"], k["response"])), int(verb[1]))
            elif verb[0] == "faces":
                rr = L.o_detect(L.oracle(), cas, L.o_integral(L.oracle(), a), 100, 1.2, 1.0, 4.0, int(verb[1]))
                want = rects_picture(a, [tuple(int(v) for v in x) for x in rr])
            else:
                want = orb_picture(tpl, a)
                kt, ks, m = orb_lists(tpl, a)
                assert lines[f] == "frame %d: Template: %u keypoints, Scene: %u keypoints, Matches: %u" % (
                    f, len(kt), len(ks), len(m)), lines
            if want is None:
                assert not out.exists() and ("frame %d: no matches" % f) in r.stderr, (stage, f)
            else:
                assert np.array_equal(_read_pgm(out), want), (stage, f)
            if ref is not None:
                rout = tmp_path / "ref.pgm"
                if rout.exists():
                    rout.unlink()
                rr = subprocess.run([ref] + list(verb) + [ins[f], str(rout)], capture_output=True, text=True, timeout=300)
                if want is None:
                    assert rr.returncode != 0 and not rout.exists(), (stage, f)
                else:
                    assert rr.returncode == 0 and rout.read_bytes() == out.read_bytes(), (stage, f)
                    if verb[0] == "orb":
                        assert lines[f].split(": ", 1)[1] in rr.stdout
    assert any(orb_picture(tpl, a) is None for a in frames) and any(orb_picture(tpl, a) is not None for a in frames)
