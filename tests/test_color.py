"""The wasm demo's colour conversions on the device (include/grayskull_color.h, libgrayskull_color.so): RGB and RGBA
frame batches to gray, bit-exact with examples/wasm/grayskull.js:33-38, and gray back to RGBA (:40-45).

The model is numpy float64 in the demo's order, then floor: numpy rounds every elementwise float64 operation to
nearest and fuses nothing, as JS numbers do.  On the CPU it is pinned against Python's own floats (also IEEE double)
and against the rule's known quirks, and the companion library is checked as a library.  On the GPU every call is
checked against the model from a poisoned dst, bytes outside each buffer included, with a census of the kernels it
launched: all 2^24 (r, g, b) triples in one frame, ragged widths, sub-batch views and byte offsets, past 65535 frames,
4 GiB and 65535 row tiles, on the caller's stream, two streams and a CUDA graph, and through gsb_magick's P6 inputs.
"""
import ctypes as C
import math
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

# every kernel of libgrayskull_color.so, and which call launches it
KERNELS = {
    "gsb::k_rgb_gray_wide": "rgb_to_gray",
    "gsb::k_rgba_gray_wide": "rgb_to_gray",
    "gsb::k_rgb_gray_bytes<3>": "rgb_to_gray",
    "gsb::k_rgb_gray_bytes<4>": "rgb_to_gray",
    "gsb::k_gray_rgba_wide": "gray_to_rgba",
    "gsb::k_gray_rgba_bytes": "gray_to_rgba",
}
CONVERSIONS = [k for k, call in KERNELS.items() if call == "rgb_to_gray"]


# ---- the model -------------------------------------------------------------------------------------------------------
def model(r, g, b):
    """the demo's gray of uint8 arrays: ((0.299 * r) + (0.587 * g)) + (0.114 * b) in float64, then floor"""
    v = np.multiply(0.299, r, dtype=np.float64)
    v = v + np.multiply(0.587, g, dtype=np.float64)
    v = v + np.multiply(0.114, b, dtype=np.float64)
    return np.floor(v).astype(np.uint8)


_cache = {}


def triples():
    """r, g, b of every triple, index (r << 16) | (g << 8) | b"""
    if "rgb" not in _cache:
        i = np.arange(1 << 24, dtype=np.uint32)
        _cache["rgb"] = ((i >> 16).astype(np.uint8), ((i >> 8) & 255).astype(np.uint8), (i & 255).astype(np.uint8))
    return _cache["rgb"]


def lut():
    """the model's gray of every triple, by index (r << 16) | (g << 8) | b"""
    if "lut" not in _cache:
        _cache["lut"] = model(*triples())
    return _cache["lut"]


def expected(px):
    """the model on (..., 3 or 4) uint8 pixels, through the table"""
    px = np.asarray(px)
    idx = (px[..., 0].astype(np.uint32) << 16) | (px[..., 1].astype(np.uint32) << 8) | px[..., 2]
    return lut()[idx]


# ---- CPU: the model --------------------------------------------------------------------------------------------------
def test_model_matches_python_floats():
    """every triple whose 299r + 587g + 114b is a multiple of 1000 (16774 of them), every pure gray and a dense random
    sample: Python's float expression, evaluated left to right, then floor"""
    r, g, b = triples()
    s = 299 * r.astype(np.int64) + 587 * g.astype(np.int64) + 114 * b.astype(np.int64)
    mult = np.flatnonzero(s % 1000 == 0)
    assert len(mult) == 16774
    rng = np.random.default_rng(0)
    pick = np.concatenate([mult, np.arange(256) * 0x010101, rng.integers(0, 1 << 24, 200_000)])
    want = lut()[pick]
    for i, x in zip(pick.tolist(), want.tolist()):
        pr, pg, pb = i >> 16, (i >> 8) & 255, i & 255
        assert math.floor(0.299 * pr + 0.587 * pg + 0.114 * pb) == x, (pr, pg, pb)


def test_model_quirks():
    r, g, b = triples()
    v = np.multiply(0.299, r, dtype=np.float64) + np.multiply(0.587, g, dtype=np.float64)
    v = v + np.multiply(0.114, b, dtype=np.float64)
    assert v.min() == 0.0 and v.max() == 255.0
    s = 299 * r.astype(np.int64) + 587 * g.astype(np.int64) + 114 * b.astype(np.int64)
    low = lut().astype(np.int64) != s // 1000
    assert int(low.sum()) == 3464
    assert (lut().astype(np.int64)[low] == s[low] // 1000 - 1).all() and (s[low] % 1000 == 0).all()
    grays = lut()[np.arange(256) * 0x010101]
    changed = np.flatnonzero(grays != np.arange(256))
    assert len(changed) == 65 and (grays[changed] == changed - 1).all()
    assert list(changed[:5]) == [1, 2, 4, 8, 11]
    known = {(3, 3, 3): 3, (100, 100, 100): 100, (255, 255, 255): 255, (255, 0, 0): 76, (0, 255, 0): 149,
             (0, 0, 255): 29, (10, 20, 30): 18, (200, 100, 50): 124, (1, 1, 1): 0, (8, 8, 8): 7}
    for (pr, pg, pb), x in known.items():
        assert int(lut()[(pr << 16) | (pg << 8) | pb]) == x, (pr, pg, pb)


def test_float32_is_not_the_rule():
    """what a torch user writes in float32 differs from the rule on 3708 triples"""
    r, g, b = triples()
    f = np.float32
    v = (f(0.299) * r.astype(f) + f(0.587) * g.astype(f)) + f(0.114) * b.astype(f)
    assert int((np.floor(v).astype(np.uint8) != lut()).sum()) == 3708


# ---- CPU: the library ------------------------------------------------------------------------------------------------
def _declared(path):
    txt = open(path).read()
    txt = txt[txt.rindex('extern "C" {'):]
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(gs_[a-z0-9_]+)\s*\(", txt)))


def test_companion_exports_exactly_its_header():
    from grayskull_b200 import build, color
    build.build()
    declared = _declared(os.path.join(ROOT, "include", "grayskull_color.h"))
    assert len(declared) == 3 and sorted(color.SIGNATURES) == declared
    nm = subprocess.run(["nm", "-D", "--defined-only", color.LIB_PATH], capture_output=True, text=True,
                        check=True).stdout
    assert sorted(ln.split()[-1] for ln in nm.splitlines() if " T " in ln) == declared
    needed = subprocess.run(["readelf", "-d", color.LIB_PATH], capture_output=True, text=True, check=True).stdout
    assert "libgrayskull_b200" not in needed
    from grayskull_b200 import _lib
    main = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    assert "gray" not in main and "color" not in main
    assert not any("k_rgb_gray" in k or "k_gray_rgba" in k for k in L.sass_functions())
    assert color.lib().gs_b200_color_last_error() == b"no error"
    cli = subprocess.run(["readelf", "-d", os.path.join(os.path.dirname(build.LIB), "gsb_magick")],
                         capture_output=True, text=True, check=True).stdout
    assert "libgrayskull_color.so" in cli


def test_ctypes_table_matches_the_header():
    from grayskull_b200 import color
    txt = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "grayskull_color.h")).read(), flags=re.S)
    ctype = {"uint8_t*": C.c_void_p, "constuint8_t*": C.c_void_p, "unsigned": C.c_uint, "gs_b200_stream": C.c_void_p,
             "int": C.c_int, "constchar*": C.c_char_p}
    decls = re.findall(r"^\s*(int|const char \*)\s*(gs_\w+)\s*\(([^)]*)\)\s*;", txt, flags=re.M)
    assert sorted(d[1] for d in decls) == sorted(color.SIGNATURES)
    for ret, name, args in decls:
        want_args = [] if args.strip() == "void" else \
            [ctype[re.sub(r"\s+", "", re.sub(r"\w+\s*$", "", a.strip()))] for a in args.split(",")]
        res, got_args = color.SIGNATURES[name]
        assert res is ctype[ret.replace(" ", "")] and got_args == want_args, name


def test_header_compiles_as_c99(tmp_path):
    for first in ("", '#include "grayskull_b200.h"\n', '#include "grayskull_contour.h"\n'):
        src = tmp_path / "t.c"
        src.write_text(first + '#include "grayskull_color.h"\n'
                       'int main(void) { return gs_b200_color_last_error() == 0 &&\n'
                       '  gs_b200_rgb_to_gray_batch(0, 0, 1, 1, 0, 3, 0) == 0; }\n')
        r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-fsyntax-only",
                            "-I", os.path.join(ROOT, "include"), str(src)], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    assert not re.match(r"grayskull_b200.*\.h$", "grayskull_color.h")


def _color_sass():
    from grayskull_b200 import color
    tool = L.cuda_tool("cuobjdump")
    if tool is None:
        pytest.skip("cuobjdump not found")
    listing = subprocess.run([tool, "-sass", color.LIB_PATH], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for cubin in re.split(r"^\s*(?=code for sm_\w+\s*$)", listing, flags=re.M)[1:]:
        arch, *parts = re.split(r"^\s*Function : (\S+)\s*$", cubin, flags=re.M)
        for name, body in zip(L.demangle(parts[0::2]), parts[1::2]):
            funcs[L.kernel_id(name)] = (arch.strip().splitlines()[0], body)
    return funcs


def test_every_companion_kernel_is_sm90a_and_has_a_row():
    funcs = _color_sass()
    assert set(funcs) == set(KERNELS)
    assert all(arch == "code for sm_90a" for arch, _ in funcs.values())


def test_conversions_are_unfused_double_without_conversion_instructions():
    """per pixel: three DADDs make the bytes' doubles, three DMULs and two DADDs the sum, one DADD.RM the floor; no
    DFMA, and no I2F.F64 / F2I.F64"""
    funcs = _color_sass()
    for k in CONVERSIONS:
        body = funcs[k][1]
        assert re.search(r"\bDMUL\b", body) and re.search(r"\bDADD\.RM\b", body), k
        assert not re.search(r"\bDFMA\b", body), k
        assert not re.search(r"\b(I2F|F2I)(\.\w+)*\.F64\b", body), k
    wide = funcs["gsb::k_rgba_gray_wide"][1]   # 16 pixels per pass, and one for the head and tail
    assert len(re.findall(r"\bDMUL\b", wide)) == 3 * 16 + 3 and len(re.findall(r"\bDADD\b", wide)) == 6 * 16 + 6


def test_launches_go_through_the_companions_helper():
    d = os.path.join(ROOT, "grayskull_b200", "color")
    text = {f: open(os.path.join(d, f)).read() for f in sorted(os.listdir(d))}
    sites = [(f, m.start()) for f, t in text.items() for m in re.finditer(r"<<<", t)]
    assert len(sites) == 1
    f, at = sites[0]
    assert text[f].rindex("static int launch(", 0, at) < at < text[f].index("cudaGetLastError")
    assert text[f].count("cudaGetLastError") == 1
    from grayskull_b200 import build
    assert not set(build.COLOR_SOURCES) & set(build.SOURCES)


def test_companion_object_makes_no_blocking_runtime_call():
    from grayskull_b200 import build
    nm = shutil.which("nm")
    if nm is None:
        pytest.skip("nm not found")
    blocking = re.compile(r"^(cudaMemcpy|cudaMemcpyToSymbol|cudaMemset|cudaMemcpy2D|cudaDeviceSynchronize|"
                          r"cudaStreamSynchronize|cudaEventSynchronize|cudaMalloc\w*|cudaFree\w*|cudaStreamCreate\w*|"
                          r"cudaStreamDestroy|cudaMemcpyAsync|cudaMemsetAsync)$")
    for s in build.COLOR_SOURCES:
        o = os.path.join(build.OBJ, s.replace(".cu", ".o"))
        syms = [ln.split()[-1] for ln in subprocess.run([nm, "-u", o], capture_output=True, text=True,
                                                         check=True).stdout.splitlines()]
        assert "cudaGetLastError" in syms
        assert not [x for x in syms if blocking.match(x)], syms


def test_empty_batch_bad_channels_and_missing_pointer_without_a_gpu():
    from grayskull_b200 import color
    L_ = color.lib()
    P, Q = 1 << 20, 1 << 24
    assert L_.gs_b200_rgb_to_gray_batch(P, Q, 8, 8, 0, 3, None) == 0
    assert L_.gs_b200_rgb_to_gray_batch(None, None, 0, 0, 0, 7, None) == 0
    assert L_.gs_b200_gray_to_rgba_batch(P, Q, 8, 8, 0, None) == 0
    for ch in (0, 1, 2, 5, 255):
        assert L_.gs_b200_rgb_to_gray_batch(P, Q, 8, 8, 2, ch, None) == 1
        assert b"InvalidValue" in L_.gs_b200_color_last_error() and b"channels" in L_.gs_b200_color_last_error()
    # overlap is refused before anything reaches the device
    assert L_.gs_b200_rgb_to_gray_batch(P + 3 * 64 - 1, P, 8, 8, 1, 3, None) == 1
    assert L_.gs_b200_rgb_to_gray_batch(P - 63, P, 8, 8, 1, 4, None) == 1
    assert L_.gs_b200_gray_to_rgba_batch(P, P + 4 * 64 - 1, 8, 8, 1, None) == 1
    assert L_.gs_b200_gray_to_rgba_batch(P + 63, P, 8, 8, 1, None) == 1
    assert b"overlaps" in L_.gs_b200_color_last_error()
    code = ("import ctypes as C, sys; sys.path.insert(0, %r); from grayskull_b200 import color; "
            "L = color.lib(); P = C.c_void_p(4096); Q = C.c_void_p(1 << 20); rc = %s; print('rc', rc)")
    for call, msg in (("L.gs_b200_rgb_to_gray_batch(None, Q, 8, 8, 2, 3, None)", "dst && src"),
                      ("L.gs_b200_rgb_to_gray_batch(P, None, 8, 8, 2, 4, None)", "dst && src"),
                      ("L.gs_b200_gray_to_rgba_batch(P, None, 8, 8, 1, None)", "dst && src"),
                      ("L.gs_b200_rgb_to_gray_batch(P, Q, 0, 8, 2, 3, None)", "w > 0 && h > 0"),
                      ("L.gs_b200_gray_to_rgba_batch(P, Q, 8, 0, 2, None)", "w > 0 && h > 0")):
        bad = subprocess.run([sys.executable, "-c", code % (ROOT, call)], capture_output=True, text=True, timeout=120)
        assert bad.returncode != 0 and "Assertion failed: " + msg in bad.stderr, (call, bad.stderr)


# ---- GPU -------------------------------------------------------------------------------------------------------------
def clib():
    from grayskull_b200 import color
    return color.lib()


def _s():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def colour_frames(w, h, n, c, seed):
    """random pixels, pure grays (every one a multiple-of-1000 triple) and smooth gradients, frame by frame"""
    rng = np.random.default_rng(seed)
    out = []
    for f in range(n):
        kind = f % 3
        if kind == 0:
            a = rng.integers(0, 256, (h, w, c), dtype=np.uint8)
        elif kind == 1:
            a = np.repeat(rng.integers(0, 256, (h, w, 1), dtype=np.uint8), c, axis=2)
        else:
            y, x = np.mgrid[0:h, 0:w]
            a = np.stack([(x * 7 + y) & 255, (y * 5 + 3 * x) & 255, (x ^ y) & 255, rng.integers(0, 256, (h, w))][:c],
                         axis=2).astype(np.uint8)
        out.append(a)
    return np.stack(out)


def rgb_kernel(src_ptr, dst_ptr, c):
    if (src_ptr - c * dst_ptr) % 16:
        return "gsb::k_rgb_gray_bytes<%d>" % c
    return "gsb::k_rgb_gray_wide" if c == 3 else "gsb::k_rgba_gray_wide"


def rgba_kernel(src_ptr, dst_ptr):
    return "gsb::k_gray_rgba_%s" % ("wide" if (dst_ptr - 4 * src_ptr) % 16 == 0 else "bytes")


# (src byte offset, dst byte offset) by layout: 16-byte aligned; both off, with dst's head peeled before the wide path;
# and an alignment the wide path cannot take
RGB_LAYOUTS = {"aligned": lambda c: (0, 0), "head": lambda c: ((5 * c) % 16, 5), "bytes": lambda c: (1, 0)}
RGBA_LAYOUTS = {"aligned": (0, 0), "head": (5, 4), "bytes": (0, 1)}
GEOMS = [(1, 7, 1), (3, 5, 3), (5, 33, 1), (17, 9, 3), (1081, 13, 3), (4096, 3, 1), (4096, 5, 3)]


def calls_for(layout, n):
    """(first frame, frames) of each call: the whole batch, or frames[1:] and then frames[:1] as views into it"""
    return [(1, n - 1), (0, 1)] if layout == "subbatch" else [(0, n)]


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,n", GEOMS, ids=["%dx%dx%d" % g for g in GEOMS])
@pytest.mark.parametrize("c", [3, 4])
@pytest.mark.parametrize("layout", list(RGB_LAYOUTS) + ["subbatch"])
def test_rgb_to_gray_geometry(lib, witness, w, h, n, c, layout):
    """every frame from a poisoned dst; sub-batch views frames[k:] of an aligned pair of buffers, as a caller slicing
    a batch makes them, run on the wide path"""
    n = max(n, 2) if layout == "subbatch" else n
    frames = colour_frames(w, h, n, c, seed=w * 7 + h + c)
    so, do = RGB_LAYOUTS[layout](c) if layout != "subbatch" else (0, 0)
    kernel = "gsb::k_rgb_gray_bytes<%d>" % c if layout == "bytes" else \
        ("gsb::k_rgb_gray_wide", "gsb::k_rgba_gray_wide")[c - 3]
    what = "%dx%dx%d c%d %s" % (w, h, n, c, layout)

    def run():
        src = Region(frames.nbytes, so, frames, seed=1)
        dst = Region(n * w * h, do, seed=2)
        seen = set()
        for k, m in calls_for(layout, n):
            sp, dp = src.ptr + k * w * h * c, dst.ptr + k * w * h
            assert rgb_kernel(sp, dp, c) == kernel
            rc, got = traced(lambda: clib().gs_b200_rgb_to_gray_batch(dp, sp, w, h, m, c, _s()))
            assert rc == 0, clib().gs_b200_color_last_error()
            seen |= got
        assert np.array_equal(dst.read(what).reshape(n, h, w), expected(frames)), what
        assert np.array_equal(src.read(what + " src"), src.before())
        return seen

    witnessed(witness, run, [kernel], what)


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,n", GEOMS, ids=["%dx%dx%d" % g for g in GEOMS])
@pytest.mark.parametrize("layout", list(RGBA_LAYOUTS) + ["subbatch"])
def test_gray_to_rgba_geometry(lib, witness, w, h, n, layout):
    n = max(n, 2) if layout == "subbatch" else n
    gray = np.random.default_rng(w + h).integers(0, 256, (n, h, w), dtype=np.uint8)
    want = np.stack([gray, gray, gray, np.full_like(gray, 255)], axis=3)
    so, do = RGBA_LAYOUTS[layout] if layout != "subbatch" else (0, 0)
    kernel = "gsb::k_gray_rgba_%s" % ("bytes" if layout == "bytes" else "wide")
    what = "%dx%dx%d %s" % (w, h, n, layout)

    def run():
        src = Region(gray.nbytes, so, gray, seed=3)
        dst = Region(4 * gray.size, do, seed=4)
        seen = set()
        for k, m in calls_for(layout, n):
            sp, dp = src.ptr + k * w * h, dst.ptr + 4 * k * w * h
            assert rgba_kernel(sp, dp) == kernel
            rc, got = traced(lambda: clib().gs_b200_gray_to_rgba_batch(dp, sp, w, h, m, _s()))
            assert rc == 0, clib().gs_b200_color_last_error()
            seen |= got
        assert np.array_equal(dst.read(what).reshape(n, h, w, 4), want), what
        assert np.array_equal(src.read(what + " src"), src.before())
        return seen

    witnessed(witness, run, [kernel], what)


@pytest.mark.gpu
@pytest.mark.parametrize("c", [3, 4])
def test_every_triple(lib, c):
    """one 4096 x 4096 frame holds every (r, g, b) once, pixel i = (i >> 16, (i >> 8) & 255, i & 255), alpha random"""
    r, g, b = triples()
    px = np.stack([r, g, b, np.random.default_rng(9).integers(0, 256, 1 << 24, dtype=np.uint8)][:c], axis=1)
    src = Region(px.nbytes, 0, px, seed=5)
    dst = Region(1 << 24, 0, seed=6)
    assert clib().gs_b200_rgb_to_gray_batch(dst.ptr, src.ptr, 4096, 4096, 1, c, _s()) == 0, \
        clib().gs_b200_color_last_error()
    got = dst.read("every triple c%d" % c)
    bad = np.flatnonzero(got != lut())
    assert not len(bad), "%d triples differ, the first %s: got %d, want %d" % (
        len(bad), [(int(i) >> 16, (int(i) >> 8) & 255, int(i) & 255) for i in bad[:1]], got[bad[0]], lut()[bad[0]])
    assert np.array_equal(src.read("src"), px.reshape(-1))


@pytest.mark.gpu
def test_gray_round_trip_and_the_python_calls(lib):
    """gray -> RGBA -> gray through the torch calls: the model's gray of (v, v, v), which is v at all but 65 levels"""
    import torch
    from grayskull_b200 import color
    levels = torch.arange(256, dtype=torch.uint8, device="cuda").reshape(1, 16, 16).repeat(2, 1, 1).contiguous()
    rgba = color.gray_to_rgba_batch(levels)
    assert rgba.shape == (2, 16, 16, 4)
    back = color.rgb_to_gray_batch(rgba)
    want = lut()[np.arange(256) * 0x010101].reshape(16, 16)
    got = back.cpu().numpy()
    assert np.array_equal(got[0], want) and np.array_equal(got[1], want)
    assert int((got[0].reshape(-1) != np.arange(256)).sum()) == 65
    out = torch.full((2, 16, 16), 7, dtype=torch.uint8, device="cuda")
    assert color.rgb_to_gray_batch(rgba[:, :, :, :3].contiguous(), out=out) is out
    assert np.array_equal(out.cpu().numpy(), got)
    assert np.array_equal(rgba.cpu().numpy(), np.stack([levels.cpu().numpy()] * 3 + [np.full((2, 16, 16), 255)], 3))


# ---- GPU: limits -----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_batches_above_the_grid_limit(lib):
    """70000 frames of 3 x 2, both channel counts and the way back"""
    w, h, n = 3, 2, 70000
    for c in (3, 4):
        frames = colour_frames(w, h, 3, c, seed=c)
        frames = np.concatenate([frames] * (n // 3) + [frames[:n % 3]])
        src, dst = Region(frames.nbytes, 0, frames, seed=7), Region(n * w * h, 0, seed=8)
        assert clib().gs_b200_rgb_to_gray_batch(dst.ptr, src.ptr, w, h, n, c, _s()) == 0
        assert np.array_equal(dst.read("70000 frames c%d" % c).reshape(n, h, w), expected(frames))
    gray = np.random.default_rng(3).integers(0, 256, (n, h, w), dtype=np.uint8)
    src, dst = Region(gray.nbytes, 0, gray, seed=9), Region(4 * gray.size, 0, seed=10)
    assert clib().gs_b200_gray_to_rgba_batch(dst.ptr, src.ptr, w, h, n, _s()) == 0
    got = dst.read("70000 frames rgba").reshape(n, h, w, 4)
    assert np.array_equal(got[..., 0], gray) and (got[..., 1] == gray).all() and (got[..., 3] == 255).all()


@pytest.mark.gpu
def test_tall_frame(lib):
    """one frame of 16 * 65535 + 40 rows"""
    w, h = 3, 16 * 65535 + 40
    for c in (3, 4):
        frames = colour_frames(w, h, 1, c, seed=11)
        src, dst = Region(frames.nbytes, 0, frames, seed=11), Region(w * h, 0, seed=12)
        assert clib().gs_b200_rgb_to_gray_batch(dst.ptr, src.ptr, w, h, 1, c, _s()) == 0
        assert np.array_equal(dst.read("tall c%d" % c).reshape(1, h, w), expected(frames))
    gray = colour_frames(w, h, 1, 1, seed=13)[..., 0]
    src, dst = Region(gray.nbytes, 0, gray, seed=13), Region(4 * gray.size, 0, seed=14)
    assert clib().gs_b200_gray_to_rgba_batch(dst.ptr, src.ptr, w, h, 1, _s()) == 0
    got = dst.read("tall rgba").reshape(1, h, w, 4)
    assert (got[..., 2] == gray).all() and (got[..., 3] == 255).all()


@pytest.mark.gpu
def test_inputs_past_4_gib(lib):
    """five RGBA frames of 16384 x 16384 (5 GiB), checked on the device against the model's table; then those gray
    frames back to 5 GiB of RGBA"""
    import torch
    w, h, n = 16384, 16384, 5
    pixels = w * h * n
    src = torch.randint(0, 256, (pixels, 4), dtype=torch.uint8, device="cuda")
    gray = torch.full((pixels + 16,), 0xA5, dtype=torch.uint8, device="cuda")
    assert clib().gs_b200_rgb_to_gray_batch(gray.data_ptr(), src.data_ptr(), w, h, n, 4, _s()) == 0
    table = torch.from_numpy(lut()).cuda()
    step = 1 << 27
    for i in range(0, pixels, step):
        p = src[i:i + step].to(torch.int64)
        idx = (p[:, 0] << 16) | (p[:, 1] << 8) | p[:, 2]
        assert torch.equal(gray[i:i + step], table[idx]), "pixels from %d differ" % i
    assert (gray[pixels:] == 0xA5).all()
    del src
    rgba = torch.full((pixels * 4 + 16,), 0x5A, dtype=torch.uint8, device="cuda")
    assert clib().gs_b200_gray_to_rgba_batch(rgba.data_ptr(), gray.data_ptr(), w, h, n, _s()) == 0
    for i in range(0, pixels, step):
        q = rgba[4 * i:4 * min(i + step, pixels)].view(-1, 4)
        g = gray[i:min(i + step, pixels)]
        assert torch.equal(q[:, 0], g) and torch.equal(q[:, 1], g) and torch.equal(q[:, 2], g), i
        assert (q[:, 3] == 255).all(), i
    assert (rgba[pixels * 4:] == 0x5A).all()


# ---- GPU: streams ----------------------------------------------------------------------------------------------------
def _sleep(s, cycles):
    import torch
    with torch.cuda.stream(s):
        torch.cuda._sleep(int(cycles))


@pytest.mark.gpu
def test_ordered_behind_a_sleeping_stream_without_a_host_wait(lib):
    import torch
    w, h, n = 640, 480, 3
    frames = colour_frames(w, h, n, 4, seed=21)
    src, dst = Region(frames.nbytes, 0, np.zeros_like(frames), seed=15), Region(n * w * h, 0, seed=16)
    real = torch.from_numpy(frames.reshape(-1)).cuda()
    s, u = torch.cuda.Stream(), torch.cuda.Stream()
    assert clib().gs_b200_rgb_to_gray_batch(dst.ptr, src.ptr, w, h, n, 4, C.c_void_p(s.cuda_stream)) == 0   # warm
    torch.cuda.synchronize()
    _sleep(u, 400_000_000)
    _sleep(s, 200_000_000)
    with torch.cuda.stream(s):
        src.t[:frames.nbytes].copy_(real)
    assert clib().gs_b200_rgb_to_gray_batch(dst.ptr, src.ptr, w, h, n, 4, C.c_void_p(s.cuda_stream)) == 0
    assert clib().gs_b200_gray_to_rgba_batch(src.ptr, dst.ptr, w, h, n, C.c_void_p(s.cuda_stream)) == 0
    s_done, u_done = s.query(), u.query()
    torch.cuda.synchronize()
    assert not s_done and not u_done, "the call waited for its stream or for the device"
    g = dst.read("behind a sleep").reshape(n, h, w)
    assert np.array_equal(g, expected(frames))
    back = src.t[:frames.nbytes].cpu().numpy().reshape(n, h, w, 4)
    assert np.array_equal(back[..., 0], g) and (back[..., 3] == 255).all()


@pytest.mark.gpu
def test_two_streams_at_once(lib):
    import torch
    s0, s1 = torch.cuda.Stream(), torch.cuda.Stream()
    w, h, n = 1081, 301, 3
    cases = []
    for seed, st, c in ((22, s0, 3), (23, s1, 4), (24, s0, 4), (25, s1, 3)):
        frames = colour_frames(w, h, n, c, seed)
        cases.append((frames, Region(frames.nbytes, 0, frames, seed=seed), Region(n * w * h, 0, seed=seed), st, c))
    _sleep(s1, 50_000_000)
    for frames, src, dst, st, c in cases:
        assert clib().gs_b200_rgb_to_gray_batch(dst.ptr, src.ptr, w, h, n, c, C.c_void_p(st.cuda_stream)) == 0
    torch.cuda.synchronize()
    for frames, src, dst, st, c in cases:
        assert np.array_equal(dst.read("two streams").reshape(n, h, w), expected(frames))


@pytest.mark.gpu
def test_graph_capture_and_replay_on_new_inputs(lib):
    import torch
    w, h, n = 1920, 1080, 2
    src = torch.zeros(n * h * w * 3, dtype=torch.uint8, device="cuda")
    gray = torch.zeros(n * h * w, dtype=torch.uint8, device="cuda")
    rgba = torch.zeros(n * h * w * 4, dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        assert clib().gs_b200_rgb_to_gray_batch(gray.data_ptr(), src.data_ptr(), w, h, n, 3,
                                                C.c_void_p(s.cuda_stream)) == 0
        assert clib().gs_b200_gray_to_rgba_batch(rgba.data_ptr(), gray.data_ptr(), w, h, n,
                                                 C.c_void_p(s.cuda_stream)) == 0
    for seed in (31, 32):
        frames = colour_frames(w, h, n, 3, seed)
        with torch.cuda.stream(s):
            src.copy_(torch.from_numpy(frames.reshape(-1)).cuda())
            gray.fill_(0x33)
            rgba.fill_(0x44)
            g.replay()
        s.synchronize()
        want = expected(frames)
        assert np.array_equal(gray.cpu().numpy().reshape(n, h, w), want), seed
        q = rgba.cpu().numpy().reshape(n, h, w, 4)
        assert np.array_equal(q[..., 1], want) and (q[..., 3] == 255).all(), seed


# ---- GPU: gsb_magick's P6 inputs -------------------------------------------------------------------------------------
def _exe():
    from grayskull_b200 import build
    return os.path.join(os.path.dirname(build.LIB), "gsb_magick")


def _read_pgm(path):
    b = open(path, "rb").read()
    hdr = b.split(b"\n", 3)
    ww, hh = map(int, hdr[1].split())
    return np.frombuffer(hdr[3], np.uint8).reshape(hh, ww)


@pytest.mark.gpu
def test_gsb_magick_p6_inputs(lib, tmp_path):
    """P6 inputs through blur:1,threshold:otsu: the model's gray, then the oracle chain; a comment in a header too"""
    O = L.oracle()
    w, h, n = 321, 203, 3
    frames = colour_frames(w, h, n, 3, seed=41)
    ins = []
    for f in range(n):
        p = tmp_path / ("in%d.ppm" % f)
        head = b"P6\n# a comment\n%d %d\n255\n" % (w, h) if f == 1 else b"P6\n%d %d\n255\n" % (w, h)
        p.write_bytes(head + frames[f].tobytes())
        ins.append(str(p))
    r = subprocess.run([_exe(), "blur:1,threshold:otsu", str(tmp_path / "o_")] + ins, capture_output=True, text=True,
                       timeout=300)
    assert r.returncode == 0, r.stderr
    for f in range(n):
        x = L.o_blur(O, np.ascontiguousarray(expected(frames[f])), 1)
        t = O.gso_otsu_threshold(L.ptr(x), w, h)
        x = x.copy()
        O.gso_threshold(L.ptr(x), w, h, t)
        assert np.array_equal(_read_pgm(str(tmp_path / ("o_%04d.pgm" % f))), x), f
    # no stage: the converted frames themselves
    r = subprocess.run([_exe(), "threshold:0", str(tmp_path / "g_"), ins[0]], capture_output=True, text=True,
                       timeout=300)
    assert r.returncode == 0, r.stderr


@pytest.mark.gpu
def test_gsb_magick_refuses_bad_p6_batches(lib, tmp_path):
    w, h = 40, 30
    a = colour_frames(w, h, 1, 3, seed=42)[0]
    files = {
        "good.ppm": b"P6\n%d %d\n255\n" % (w, h) + a.tobytes(),
        "other.ppm": b"P6\n%d %d\n255\n" % (w + 1, h) + np.zeros((h, w + 1, 3), np.uint8).tobytes(),
        "gray.pgm": b"P5\n%d %d\n255\n" % (w, h) + a[..., 0].tobytes(),
        "deep.ppm": b"P6\n%d %d\n65535\n" % (w, h) + np.zeros((h, w, 6), np.uint8).tobytes(),
        "short.ppm": b"P6\n%d %d\n255\n" % (w, h) + a.tobytes()[:-7],
    }
    for name, data in files.items():
        (tmp_path / name).write_bytes(data)
    cases = [(["good.ppm", "gray.pgm"], "gray.pgm is not P6, the batch is P6"),
             (["gray.pgm", "good.ppm"], "good.ppm is P6, the batch is P5"),
             (["good.ppm", "other.ppm"], "other.ppm is 41x30, the batch is 40x30"),
             (["deep.ppm"], "P6 maxval 65535, only 255 is supported"),
             (["good.ppm", "short.ppm"], "short.ppm is truncated: 3593 of 3600 pixel bytes")]
    for ins, msg in cases:
        r = subprocess.run([_exe(), "blur:1", str(tmp_path / "x_")] + [str(tmp_path / i) for i in ins],
                           capture_output=True, text=True, timeout=300)
        assert r.returncode == 1 and msg in r.stderr and "gsb_magick: " in r.stderr, (ins, r.stderr)
    assert not list(tmp_path.glob("x_*"))
