"""Regions of interest on the device (include/grayskull_b200_roi.h): crop, then nearest or bilinear resize, bit-exact
with the reference's gs_crop followed by gs_resize_nn or gs_resize.

gso_crop / gso_resize_nn (tests/_libs.py) restate the reference's two calls in numpy, 32-bit wrapping arithmetic included; the
bilinear half of the composition is the C oracle's gso_resize (tests/_libs.py).  test_dispatch_paths.py has the rows
that pick each region kernel (gsb::k_roi_*) and checks that its launches go through gsb::launch; test_host_logic.py
checks the exports, the binding table and that every kernel is sm_90a, test_streams.py the runtime calls of roi.o.

  * CPU: the copy kernel's SASS moves 16-byte blocks; the restatement equals the reference's gs_crop / gs_resize_nn
    (when oracle/_ref is built), wrap cases included; the host asserts abort with the reference's message and an
    unknown mode is an error.
  * GPU: both entry points against the composition (host regions at TMA-friendly and ragged widths, odd offsets,
    misaligned pointers; device lists with and without counts, untouched slots past the counts, invalid regions,
    a source batch over 4 GiB); LBP detection chained into the region call on the device counts; the CLI's crop
    stage.  test_streams.py runs both entry points on the caller's stream, on two streams at once and in a graph.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import _libs as L
from _calls import POISON
from _libs import M32, composition, gso_crop, gso_resize_nn, roi_valid  # noqa: F401
from grayskull_b200._lib import Rect
from _gpu import O, Region, frames, lib, stream, traced, witness, witnessed  # noqa: F401

ROOT = L.ROOT
NEAREST, BILINEAR = 0, 1
COPY, NN, BL = "gsb::k_roi_copy", "gsb::k_roi_gather<0>", "gsb::k_roi_gather<1>"


def roi_lib():
    from grayskull_b200 import roi
    return roi.lib()


# ---- CPU: the library --------------------------------------------------------------------------------------------------
def test_copy_kernel_moves_16_byte_blocks():
    """the copy kernel loads aligned 16-byte blocks, funnel-shifts them into place and stores 16-byte chunks"""
    sass = L.sass_functions()[COPY]
    assert "LDG.E.128.CONSTANT" in sass and "STG.E.EF.128" in sass and "SHF.R" in sass


# ---- CPU: the restatement against the reference ------------------------------------------------------------------------
def _geometries(rng):
    out = []
    for _ in range(40):
        sw, sh = int(rng.integers(1, 90)), int(rng.integers(1, 60))
        x, y = int(rng.integers(0, sw)), int(rng.integers(0, sh))
        out.append(((sw, sh), (x, y, int(rng.integers(1, sw - x + 1)), int(rng.integers(1, sh - y + 1))),
                   (int(rng.integers(1, 120)), int(rng.integers(1, 80)))))
    # roi.x / roi.y near 2^32: the wrapped assert passes, the first columns / rows read outside the frame
    out.append(((64, 9), (2 ** 32 - 5, 0, 10, 9), (10, 9)))
    out.append(((16, 30), (3, 2 ** 32 - 7, 13, 20), (5, 41)))
    out.append(((70, 2), (2 ** 32 - 60, 2 ** 32 - 1, 100, 3), (33, 7)))
    # one-row frames about 10^5 wide: x * src.w wraps in gs_resize_nn
    out.append(((100_003, 1), (0, 0, 100_003, 1), (99_991, 1)))
    out.append(((120_000, 1), (7, 0, 110_000, 1), (100_000, 2)))
    out.append(((1, 90_001), (0, 0, 1, 90_001), (1, 70_000)))
    return out


@pytest.mark.skipif(not L.have_ref(), reason="oracle/_ref/libgs_ref.so not built (no reference checkout)")
def test_restatement_matches_reference():
    R = L.ref()
    R.gs_crop.argtypes = [L.Image, L.Image, L.Rect]
    R.gs_crop.restype = None
    R.gs_resize_nn.argtypes = [L.Image, L.Image]
    R.gs_resize_nn.restype = None
    rng = np.random.default_rng(11)
    for (sw, sh), roi, (dw, dh) in _geometries(rng):
        a = rng.integers(0, 256, (sh, sw), dtype=np.uint8)
        assert roi_valid(roi, sw, sh)
        c = np.zeros((roi[3], roi[2]), np.uint8)
        R.gs_crop(L.img(c), L.img(a), L.Rect(*roi))
        assert np.array_equal(gso_crop(a, roi), c), (sw, sh, roi)
        d = np.zeros((dh, dw), np.uint8)
        R.gs_resize_nn(L.img(d), L.img(c))
        assert np.array_equal(gso_resize_nn(c, dw, dh), d), (roi, dw, dh)


# ---- CPU: host checks ---------------------------------------------------------------------------------------------------
def _abort_run(call):
    code = ("import ctypes as C, sys; sys.path.insert(0, %r); from grayskull_b200 import roi, _lib; "
            "L = roi.lib(); R = _lib.Rect; P = C.c_void_p(4096); rc = %s; print('rc', rc)" % (ROOT, call))
    return subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120)


CROP_MSG = ("Assertion failed: gs_valid(dst) && gs_valid(src) && roi.x + roi.w <= src.w && roi.y + roi.h <= src.h && "
            "dst.w == roi.w && dst.h == roi.h")


@pytest.mark.parametrize("roi", [(1, 0, 64, 10), (0, 5, 10, 6), (0, 0, 0, 4), (3, 3, 5, 0), (2 ** 32 - 5, 0, 70, 2)],
                         ids=["x-overrun", "y-overrun", "w0", "h0", "wrap-overrun"])
def test_crop_assert_aborts_with_reference_message(roi):
    r = _abort_run("L.gs_b200_crop_resize_batch(P, 8, 8, P, 64, 10, 1, R(%d, %d, %d, %d), 0, None)" % roi)
    assert r.returncode != 0 and "rc" not in r.stdout, (r.stdout, r.stderr)
    assert CROP_MSG in r.stderr, r.stderr


def test_bilinear_assert_aborts_on_empty_output():
    r = _abort_run("L.gs_b200_crop_resize_batch(P, 0, 8, P, 64, 10, 1, R(0, 0, 8, 8), 1, None)")
    assert r.returncode != 0 and "Assertion failed: gs_valid(dst) && gs_valid(src)" in r.stderr, r.stderr
    r = _abort_run("L.gs_b200_rois_resize_batch(P, 8, 0, P, 64, 10, 1, P, None, 1, 1, None)")
    assert r.returncode != 0 and "Assertion failed: dw > 0 && dh > 0" in r.stderr, r.stderr


def test_wrapped_region_passes_and_empty_nearest_writes_nothing():
    """n == 0 launches nothing, so these run without a GPU: the wrapped region passes gs_crop's assert, and a 0 x 8
    nearest output is gs_resize_nn's empty loop"""
    r = _abort_run("L.gs_b200_crop_resize_batch(P, 8, 8, P, 64, 10, 0, R(2 ** 32 - 5, 0, 8, 8), 0, None)")
    assert r.returncode == 0 and "rc 0" in r.stdout, (r.stdout, r.stderr)
    r = _abort_run("L.gs_b200_crop_resize_batch(P, 0, 8, P, 64, 10, 3, R(0, 0, 8, 8), 0, None)")
    assert r.returncode == 0 and "rc 0" in r.stdout, (r.stdout, r.stderr)


def test_unknown_mode_is_an_error():
    from grayskull_b200 import _lib
    lr = roi_lib()
    p = C.c_void_p(4096)
    before = _lib.lib().gs_b200_launch_count()
    assert lr.gs_b200_crop_resize_batch(p, 8, 8, p, 64, 10, 1, _lib.Rect(0, 0, 8, 8), 2, None) == 1
    assert b"cudaErrorInvalidValue" in _lib.lib().gs_b200_last_error()
    assert lr.gs_b200_rois_resize_batch(p, 8, 8, p, 64, 10, 1, p, None, 1, -1, None) == 1
    assert _lib.lib().gs_b200_launch_count() == before


# ---- GPU: host-region entry ---------------------------------------------------------------------------------------------
def _case(cid, sw, sh, roi, dw, dh, mode, kernel, so=0, do=0):
    return pytest.param(dict(sw=sw, sh=sh, roi=roi, dw=dw, dh=dh, mode=mode, kernel=kernel, so=so, do=do), id=cid)


HOST_CASES = [
    # unscaled regions: the copy kernel in either mode, at 16-multiple and ragged widths, odd offsets, any alignment
    _case("crop-tma-nn", 272, 70, (3, 5, 160, 40), 160, 40, NEAREST, COPY),
    _case("crop-tma-bl", 272, 70, (17, 1, 96, 61), 96, 61, BILINEAR, COPY),
    _case("crop-ragged-nn", 101, 37, (13, 7, 77, 29), 77, 29, NEAREST, COPY, so=5, do=3),
    _case("crop-ragged-bl", 101, 37, (1, 0, 99, 37), 99, 37, BILINEAR, COPY, so=1, do=7),
    _case("crop-narrow", 40, 20, (31, 2, 9, 17), 9, 17, NEAREST, COPY, so=3, do=1),
    _case("crop-1px", 19, 5, (18, 4, 1, 1), 1, 1, BILINEAR, COPY, so=9),
    _case("crop-copy-whole", 333, 21, (0, 0, 333, 21), 333, 21, NEAREST, COPY, so=6, do=2),   # gs_copy
    _case("crop-2896", 2900, 3, (4, 0, 2896, 3), 2896, 3, BILINEAR, COPY, so=2, do=5),
    # scaled regions, and unscaled ones past a mode's identity or wrapping: the gather kernel
    _case("nn-up", 272, 70, (7, 3, 50, 31), 64, 64, NEAREST, NN),
    _case("nn-down", 101, 37, (0, 1, 100, 36), 33, 11, NEAREST, NN, so=3, do=1),
    _case("nn-whole", 272, 70, (0, 0, 272, 70), 100, 30, NEAREST, NN),                       # pure gs_resize_nn
    _case("nn-wrap-x", 64, 9, (2 ** 32 - 5, 0, 10, 9), 10, 9, NEAREST, NN),
    _case("nn-wrap-y", 16, 30, (3, 2 ** 32 - 7, 13, 20), 13, 20, NEAREST, NN),
    _case("nn-65537", 65600, 2, (40, 0, 65537, 2), 65537, 2, NEAREST, NN),                    # x * w wraps at scale 1
    _case("nn-row-wrap", 100_003, 1, (0, 0, 100_003, 1), 99_991, 1, NEAREST, NN, do=1),
    _case("bl-up", 272, 70, (7, 3, 50, 31), 64, 64, BILINEAR, BL),
    _case("bl-down", 101, 37, (2, 1, 97, 35), 40, 13, BILINEAR, BL, so=7, do=2),
    _case("bl-chip", 200, 150, (60, 40, 77, 77), 64, 64, BILINEAR, BL, so=1),
    _case("bl-2897", 2900, 3, (3, 0, 2897, 3), 2897, 3, BILINEAR, BL),                         # not the identity
    _case("bl-wrap-x", 64, 9, (2 ** 32 - 5, 0, 10, 9), 31, 4, BILINEAR, BL),
]


def _run_host(lib, c, n, seed):
    import torch  # noqa: F401
    from grayskull_b200 import roi
    lr = roi.lib()
    sw, sh, dw, dh = c["sw"], c["sh"], c["dw"], c["dh"]
    a = frames(sw, sh, n, seed)
    src = Region(a.nbytes, c["so"], a, seed)
    dst = Region(n * dw * dh, c["do"], seed=seed + 1)
    rc, seen = traced(lambda: lr.gs_b200_crop_resize_batch(C.c_void_p(dst.ptr), dw, dh, C.c_void_p(src.ptr), sw, sh, n,
                                                          Rect(*c["roi"]), c["mode"], stream()))
    assert rc == 0, lib.gs_b200_last_error()
    return a, dst.read("dst").reshape(n, dh, dw), seen


@pytest.mark.gpu
@pytest.mark.parametrize("c", HOST_CASES)
@pytest.mark.parametrize("n", [1, 2, 3, 5])
def test_crop_resize_vs_oracle(lib, O, witness, c, n):
    def run():
        a, got, seen = _run_host(lib, c, n, 3 + n)
        for f in range(n):
            want = composition(O, a[f], c["roi"], c["dw"], c["dh"], c["mode"])
            assert np.array_equal(got[f], want), "frame %d: %d of %d bytes differ" % (f, (got[f] != want).sum(), want.size)
        return seen
    witnessed(witness, run, [c["kernel"]], "crop_resize %s n=%d" % (c, n))


@pytest.mark.gpu
@pytest.mark.parametrize("geom", [(272, 70, 100, 30), (640, 480, 64, 64), (101, 37, 300, 90), (200, 150, 200, 150)])
def test_whole_frame_bilinear_equals_resize_batch(lib, geom):
    import torch
    from grayskull_b200 import api, roi
    sw, sh, dw, dh = geom
    src = torch.from_numpy(frames(sw, sh, 3, 21)).cuda()
    want = api.resize_batch(src, dw, dh)
    got = roi.crop_resize_batch(src, (0, 0, sw, sh), dw, dh, roi.BILINEAR)
    torch.cuda.synchronize()
    assert torch.equal(got, want)


# ---- GPU: region lists ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mode", [NEAREST, BILINEAR], ids=["nearest", "bilinear"])
@pytest.mark.parametrize("counts", ["null", "partial"])
@pytest.mark.parametrize("geom", [(200, 150, 48, 40, 0, 0), (131, 97, 37, 23, 3, 5)], ids=["even", "ragged"])
def test_rois_resize_vs_oracle(lib, O, witness, mode, counts, geom):
    import torch
    from grayskull_b200 import roi
    sw, sh, dw, dh, so, do = geom
    n, mr = 4, 8
    rng = np.random.default_rng(sw + 7 * mode)
    a = frames(sw, sh, n, 5)
    rects = L.regions(rng, n, mr, sw, sh, dw, dh)
    cnt = np.array([mr, 3, 0, 5 + 2 * mode], np.uint32) if counts == "partial" else None
    src = Region(a.nbytes, so, a, 1)
    dst = Region(n * mr * dw * dh, do, seed=2)
    R = torch.from_numpy(rects.view(np.int32).reshape(n, mr, 4)).cuda()
    N = torch.from_numpy(cnt.view(np.int32)).cuda() if cnt is not None else None

    def run():
        dst.t.copy_(torch.from_numpy(dst.host))
        rc, seen = traced(lambda: roi.lib().gs_b200_rois_resize_batch(
            C.c_void_p(dst.ptr), dw, dh, C.c_void_p(src.ptr), sw, sh, n, C.c_void_p(R.data_ptr()),
            None if N is None else C.c_void_p(N.data_ptr()), mr, mode, stream()))
        assert rc == 0, lib.gs_b200_last_error()
        got = dst.read("dst").reshape(n, mr, dh, dw)
        before = dst.before().reshape(n, mr, dh, dw)
        for f in range(n):
            for k in range(mr):
                if cnt is not None and k >= cnt[f]:
                    assert np.array_equal(got[f, k], before[f, k]), "slot (%d, %d) past the count changed" % (f, k)
                else:
                    want = composition(O, a[f], tuple(rects[f, k]), dw, dh, mode)
                    assert np.array_equal(got[f, k], want), "slot (%d, %d) %s" % (f, k, rects[f, k])
        return seen
    witnessed(witness, run, [COPY, NN if mode == NEAREST else BL], "rois_resize mode %d %s" % (mode, counts))


@pytest.mark.gpu
def test_rois_in_the_last_frame_of_a_batch_over_4gib(lib, O):
    import torch
    from grayskull_b200 import roi
    sw = sh = 4096
    n = 257                                            # 4 GiB + 16 MiB of frames: the last frame starts past 2^32
    src = torch.empty((n, sh, sw), dtype=torch.uint8, device="cuda")
    last = L.natural_like(sw, sh, 9)
    src[n - 1].copy_(torch.from_numpy(last))
    rects = np.zeros((n, 3), L.RECT_DTYPE)
    rects[n - 1] = [(4001, 17, 64, 64), (1, 3000, 900, 1000), (0, 0, 4096, 4096)]
    cnt = np.zeros(n, np.int32)
    cnt[n - 1] = 3
    R = torch.from_numpy(rects.view(np.int32).reshape(n, 3, 4)).cuda()
    N = torch.from_numpy(cnt).cuda()
    for mode in (NEAREST, BILINEAR):
        out = torch.full((n, 3, 64, 64), POISON, dtype=torch.uint8, device="cuda")
        roi.rois_resize_batch(src, R, N, 64, 64, mode, out=out)
        got = out[n - 1].cpu().numpy()
        for k in range(3):
            assert np.array_equal(got[k], composition(O, last, tuple(rects[n - 1, k]), 64, 64, mode)), (mode, k)
        assert bool((out[: n - 1] == POISON).all()), "slots of frames with count 0 changed"
    del src
    torch.cuda.empty_cache()


# ---- GPU: detection chained into the region call ------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mode", [NEAREST, BILINEAR], ids=["nearest", "bilinear"])
def test_lbp_detect_into_rois(lib, O, mode):
    import torch
    import grayskull_b200 as g
    from grayskull_b200 import api, roi
    lena = np.load(os.path.join(ROOT, "tests", "golden", "lena_golden.npz"))["lena"]
    fr = np.stack([lena, np.ascontiguousarray(lena[:, ::-1]), L.natural_like(128, 128, 4)])
    n, h, w = fr.shape
    cas, hc = g.load_cascade(), L.HostCascade()
    mr = 32
    src = torch.from_numpy(fr).cuda()
    rects, counts = api.lbp_detect_batch(cas, api.integral_batch(src), mr, 1.1, 1.0, 4.0, 2)
    out = torch.full((n, mr, 24, 24), POISON, dtype=torch.uint8, device="cuda")
    roi.rois_resize_batch(src, rects, counts, 24, 24, mode, out=out)
    got = out.cpu().numpy()
    total = 0
    for f in range(n):
        want_rects = L.o_detect(O, hc, L.o_integral(O, fr[f]), mr, 1.1, 1.0, 4.0, 2)
        assert int(counts[f]) == len(want_rects)
        total += len(want_rects)
        for k, r in enumerate(want_rects):
            assert np.array_equal(got[f, k], composition(O, fr[f], tuple(r), 24, 24, mode)), (f, k, r)
        assert (got[f, len(want_rects):] == POISON).all()
    assert total > 0, "no detections: the chain was not exercised"


# ---- GPU: the CLI's crop stage --------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gsb_magick_crop_stage(lib, tmp_path):
    from grayskull_b200 import build
    exe = os.path.join(os.path.dirname(build.LIB), "gsb_magick")
    a = frames(123, 77, 2, 8)
    ins = []
    for f in range(2):
        p = tmp_path / ("in%d.pgm" % f)
        p.write_bytes(b"P5\n123 77\n255\n" + a[f].tobytes())
        ins.append(str(p))
    r = subprocess.run([exe, "crop:17:9:61:40,blur:1,crop:0:3:61:37", str(tmp_path / "out")] + ins,
                       capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    Od = L.oracle()
    for f in range(2):
        want = L.o_blur(Od, gso_crop(a[f], (17, 9, 61, 40)), 1)
        want = gso_crop(want, (0, 3, 61, 37))
        data = (tmp_path / ("out%04d.pgm" % f)).read_bytes()
        assert data.startswith(b"P5\n61 37\n255\n")
        assert np.array_equal(np.frombuffer(data[-61 * 37:], np.uint8).reshape(37, 61), want)
    r = subprocess.run([exe, "crop:100:0:30:5", str(tmp_path / "bad")] + ins, capture_output=True, text=True, timeout=120)
    assert r.returncode != 0 and "invalid crop rectangle" in r.stderr
