"""GPU parity tests: the CUDA path (through the C ABI of libgrayskull_b200.so) against
  * the reference-generated golden fixtures in tests/golden/ (bit-exact),
  * the oracle restatement on the same seeded inputs (bit-exact),
  * size-independent properties / crop checks at BASELINE.json's full sizes.
Bit-exact everywhere; gs_compute_orientation's angle is additionally checked within 1e-5 in the
libdevice trig mode (north_star's stated tolerance).  Needs a CUDA device (-m gpu)."""
import os

import numpy as np
import pytest

import _libs as L
from _gpu import G, O, dev  # noqa: F401

pytestmark = pytest.mark.gpu
GOLD = os.path.join(L.ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def cas():
    import grayskull_b200 as g
    return g.load_cascade()


# ---- single-image gs_* API (host pointers, staged) against the reference's own fixtures ------
def test_golden_lena_single_image_api(G, cas):
    """BASELINE config C1: gs_sobel (and every other op) on testdata/lena.pgm, bit-exact against
    outputs the real reference produced (tools/make_golden.py)."""
    z = np.load(os.path.join(GOLD, "lena_golden.npz"))
    a = z["lena"]
    d = np.zeros_like(a); G.gs_sobel(d, a); assert np.array_equal(d, z["sobel"])
    for r in (1, 5, 9):
        d = np.empty_like(a); G.gs_blur(d, a, r); assert np.array_equal(d, z["blur%d" % r]), r
    d = np.empty_like(a); G.gs_adaptive_threshold(d, a, 15, 5); assert np.array_equal(d, z["adaptive_15_5"])
    d = np.empty_like(a); G.gs_erode(d, a); assert np.array_equal(d, z["erode"])
    d = np.empty_like(a); G.gs_dilate(d, a); assert np.array_equal(d, z["dilate"])
    d = np.empty((64, 128), np.uint8); G.gs_resize(d, a); assert np.array_equal(d, z["resize_128x64"])
    d = np.empty((64, 64), np.uint8); G.gs_downsample(d, a); assert np.array_equal(d, z["downsample"])
    ii = np.empty(a.shape, np.uint32); G.gs_integral(a, ii); assert np.array_equal(ii, z["integral"])
    sm = np.zeros_like(a)
    k = G.gs_fast(a, sm, 5000, 20)
    assert k.tobytes() == z["fast_kps"].tobytes() and np.array_equal(sm, z["fast_scoremap"])
    k = G.gs_orb_extract(a, 500, 20, np.zeros_like(a))
    assert len(k) == len(z["orb_kps"]) == 280
    assert k.tobytes() == z["orb_kps"].tobytes()       # angles and descriptors bit-identical
    r = G.gs_lbp_detect(cas, ii, 1000, 1.1, 1.0, 4.0, 2)
    assert r.tobytes() == z["lbp_rects"].tobytes() and len(r) == 10
    # the individual ORB pieces
    ref_k = z["orb_kps"]
    for i in (0, 7, 100, 279):
        ang = G.gs_compute_orientation(a, int(ref_k[i]["x"]), int(ref_k[i]["y"]), 15)
        assert np.float32(ang).tobytes() == np.float32(ref_k[i]["angle"]).tobytes()
        kp = ref_k[i:i + 1].copy(); kp["descriptor"] = 0
        G.gs_brief_descriptor(a, kp)
        assert kp.tobytes() == ref_k[i:i + 1].tobytes()
    # single windows
    for (x, y, s) in ((54, 52, 1.9487171), (0, 0, 1.0), (100, 100, 1.0), (30, 40, 2.0)):
        got = G.gs_lbp_window(cas, ii, x, y, s)
        want = L.oracle().gso_lbp_window(cas.ptr, L.ptr(ii), 128, 128, x, y, s)
        assert got == want


def test_golden_random_ragged(G, cas):
    """odd sizes (33x29 ... 130x131): generic (non-TMA) kernels, reference-generated fixtures"""
    z = np.load(os.path.join(GOLD, "random_golden.npz"))
    for i, (w, h) in enumerate(z["shapes"]):
        a = z["img%d" % i]; t = "i%d_" % i
        d = np.zeros_like(a); G.gs_sobel(d, a); assert np.array_equal(d, z[t + "sobel"]), (w, h)
        for r in (1, 5, 9):
            d = np.empty_like(a); G.gs_blur(d, a, r); assert np.array_equal(d, z[t + "blur%d" % r]), (w, h, r)
        d = np.empty_like(a); G.gs_adaptive_threshold(d, a, 15, 5); assert np.array_equal(d, z[t + "adaptive_15_5"])
        d = np.empty_like(a); G.gs_erode(d, a); assert np.array_equal(d, z[t + "erode"])
        d = np.empty_like(a); G.gs_dilate(d, a); assert np.array_equal(d, z[t + "dilate"])
        d = np.empty((64, 128), np.uint8); G.gs_resize(d, a); assert np.array_equal(d, z[t + "resize_128x64"])
        d = np.empty((h // 2, w // 2), np.uint8); G.gs_downsample(d, a); assert np.array_equal(d, z[t + "downsample"])
        ii = np.empty(a.shape, np.uint32); G.gs_integral(a, ii); assert np.array_equal(ii, z[t + "integral"])
        sm = np.zeros_like(a)
        k = G.gs_fast(a, sm, 5000, 20)
        assert k.tobytes() == z[t + "fast_kps"].tobytes() and np.array_equal(sm, z[t + "fast_scoremap"]), (w, h)
        k = G.gs_orb_extract(a, 200, 20, np.zeros_like(a))
        assert k.tobytes() == z[t + "orb_kps"].tobytes(), (w, h)
        if t + "lbp_rects" in z.files:
            r = G.gs_lbp_detect(cas, ii, 1000, 1.1, 1.0, 4.0, 2)
            assert r.tobytes() == z[t + "lbp_rects"].tobytes(), (w, h)


def test_sobel_border_untouched(G):
    a = L.natural_like(64, 48, 1)
    d = np.full_like(a, 77); G.gs_sobel(d, a)
    assert (d[0] == 77).all() and (d[-1] == 77).all() and (d[:, 0] == 77).all() and (d[:, -1] == 77).all()
    tiny = np.full((2, 2), 9, np.uint8); d = np.full_like(tiny, 5); G.gs_sobel(d, tiny); assert (d == 5).all()


def test_fast_quirks(G):
    """SURVEY appendix B quirk probes: dark-centre wrap, stale score-map ring, cap in raster order"""
    a = np.full((7, 7), 5, np.uint8); a[3, 3] = 3
    sm = np.zeros((7, 7), np.uint8)
    k = G.gs_fast(a, sm, 10, 20)
    assert len(k) == 1 and sm[3, 3] == 2 and k[0]["response"] == 2
    sm = np.zeros((7, 7), np.uint8); sm[2, 2] = 200
    assert len(G.gs_fast(a, sm, 10, 20)) == 0 and sm[2, 2] == 200
    b = np.full((7, 7), 105, np.uint8); b[3, 3] = 103
    assert len(G.gs_fast(b, np.zeros((7, 7), np.uint8), 10, 20)) == 0
    assert len(G.gs_fast(a, None, 10, 20)) == 0      # invalid score map: writes dropped, reads 0


# ---- batched device API vs oracle on seeded inputs (TMA and generic kernels) -----------------
SHAPES = [(256, 128), (272, 140), (512, 300), (16, 16), (48, 7), (1024, 67), (640, 480), (100, 37), (17, 1), (1, 1)]


@pytest.mark.parametrize("force_generic", [0, 1])
def test_stencils_vs_oracle(G, O, force_generic):
    import grayskull_b200 as g
    g.lib().gs_b200_force_generic(force_generic)
    try:
        rng = np.random.default_rng(7)
        for (w, h) in SHAPES:
            n = 3
            frames = np.stack([rng.integers(0, 256, (h, w)).astype(np.uint8) if i != 1 else L.natural_like(w, h, 3)
                               for i in range(n)])
            src = dev(frames)
            got = G.sobel_batch(src, out=dev(np.full_like(frames, 77))).cpu().numpy()
            for i in range(n):
                assert np.array_equal(got[i], L.o_sobel(O, frames[i], 77)), ("sobel", w, h, i)
            ge, gd = G.erode_batch(src).cpu().numpy(), G.dilate_batch(src).cpu().numpy()
            for i in range(n):
                assert np.array_equal(ge[i], L.o_morph(O, frames[i], 0)), ("erode", w, h, i)
                assert np.array_equal(gd[i], L.o_morph(O, frames[i], 1)), ("dilate", w, h, i)
            for r in (0, 1, 2, 3, 4, 5, 6, 7, 8, 11):
                gb = G.blur_batch(src, r).cpu().numpy()
                c = int(rng.integers(-40, 40))
                ga = G.adaptive_threshold_batch(src, r, c).cpu().numpy()
                for i in range(n):
                    assert np.array_equal(gb[i], L.o_blur(O, frames[i], r)), ("blur", w, h, r, i)
                    assert np.array_equal(ga[i], L.o_adaptive(O, frames[i], r, c)), ("adaptive", w, h, r, c, i)
            if w >= 2 and h >= 2:
                gd = G.downsample_batch(src).cpu().numpy()
                for i in range(n):
                    assert np.array_equal(gd[i], L.o_down(O, frames[i])), ("down", w, h)
            for (dw, dh) in ((w // 2 + 1, h // 2 + 1), (w * 2 + 3, h + 5), (w, h), (7, 3), (max(w // 2, 1), max(h // 2, 1)),
                             (max(w // 2, 1), h + 1)):
                gr = G.resize_batch(src, dw, dh).cpu().numpy()
                for i in range(n):
                    assert np.array_equal(gr[i], L.o_resize(O, frames[i], dw, dh)), ("resize", w, h, dw, dh)
            gi = G.integral_batch(src).cpu().numpy().view(np.uint32)
            for i in range(n):
                assert np.array_equal(gi[i], L.o_integral(O, frames[i])), ("integral", w, h)
    finally:
        g.lib().gs_b200_force_generic(0)


@pytest.mark.parametrize("kernel", ["bands", "strips", "auto"])
def test_integral_single_pass_batches(G, O, kernel):
    """the two single-pass kernels of integral.cu -- chained 16-row bands (round 1) and 1024-column strips walking
    down the frame (round 2; the default once n * strips >= the SM count) -- on ragged heights, 1..8 strips per row (strip
    seams at multiples of 1024 columns), band counts from 1 to 270, all-255 frames (the largest sums)"""
    if kernel != "auto":
        os.environ["GS_B200_INTEGRAL"] = kernel
    try:
        for (w, h, n) in ((3840, 2160, 40), (256, 37, 33), (4096, 100, 40), (8192, 33, 32), (1920, 1080, 80), (8, 16, 160), (40, 17, 150),
                          (1032, 9, 75), (2048, 8, 74), (5000 // 8 * 8, 23, 40), (2048, 19, 300)):
            rng = np.random.default_rng(w + h)
            fr = rng.integers(0, 256, (n, h, w), dtype=np.uint8)
            fr[n - 1] = 255
            got = G.integral_batch(dev(fr)).cpu().numpy().view(np.uint32)
            for i in (0, n // 2, n - 1):
                assert np.array_equal(got[i], L.o_integral(O, fr[i])), (kernel, w, h, n, i)
    finally:
        os.environ.pop("GS_B200_INTEGRAL", None)


def test_blur_constant_and_saturated(G, O):
    """all-255 and all-0 frames: the division must be exact at the extremes for every clipped count"""
    for r in range(1, 8):
        for v in (255, 0, 1, 254):
            a = np.full((2, 80, 272), v, np.uint8)
            assert (G.blur_batch(dev(a), r).cpu().numpy() == v).all(), (r, v)


def test_fast_orb_vs_oracle(G, O):
    rng = np.random.default_rng(11)
    for (w, h, nk, t) in ((320, 240, 300, 20), (161, 97, 50, 10), (640, 360, 1250, 20), (64, 64, 5000, 0), (40, 33, 7, 35)):
        frames = np.stack([L.natural_like(w, h, 20 + i) if i % 2 == 0 else rng.integers(0, 256, (h, w)).astype(np.uint8)
                           for i in range(4)])
        stale = (rng.integers(0, 256, frames.shape) * (rng.random(frames.shape) < 0.02)).astype(np.uint8)
        sm, kps, counts = G.fast_batch(dev(frames), nk, t, scoremap=dev(stale))
        got = G.kps_to_numpy(kps, counts); smh = sm.cpu().numpy()
        for i in range(4):
            so = stale[i].copy()
            want = L.o_fast(O, frames[i], so, nk, t)
            assert np.array_equal(smh[i], so), ("scoremap", w, h, i)
            assert got[i].tobytes() == want.tobytes(), ("fast", w, h, i, len(got[i]), len(want))
        sm, kps, counts = G.orb_extract_batch(dev(frames), nk, t)
        got = G.kps_to_numpy(kps, counts)
        for i in range(4):
            want = L.o_orb(O, frames[i], np.zeros_like(frames[i]), nk, t)
            assert len(got[i]) == len(want), ("orb count", w, h, i)
            assert got[i].tobytes() == want.tobytes(), ("orb", w, h, i)


def test_orb_libdevice_trig_tolerance(G, O):
    """trig mode 1 (CUDA libdevice): angle within 1e-5 of the reference (north_star tolerance)"""
    import grayskull_b200 as g
    a = L.natural_like(320, 240, 5)[None]
    g.lib().gs_b200_set_trig_mode(1)
    try:
        _, kps, counts = G.orb_extract_batch(dev(a), 300, 20)
    finally:
        g.lib().gs_b200_set_trig_mode(0)
    got = G.kps_to_numpy(kps, counts)[0]
    want = L.o_orb(O, a[0], np.zeros_like(a[0]), 300, 20)
    assert len(got) == len(want) > 0
    assert np.array_equal(got["x"], want["x"]) and np.array_equal(got["y"], want["y"])
    assert np.abs(got["angle"] - want["angle"]).max() <= 1e-5


def test_lbp_vs_oracle(G, O, cas):
    rng = np.random.default_rng(13)
    for (w, h) in ((160, 120), (200, 131), (97, 64)):
        frames = np.stack([L.natural_like(w, h, 40 + i) for i in range(3)])
        ii = np.stack([L.o_integral(O, f) for f in frames])
        iid = dev(ii.view(np.int32))
        for (mr, sf, mn, mx, st) in ((1000, 1.1, 1.0, 4.0, 2), (5, 1.2, 1.0, 3.0, 1), (1000, 1.25, 1.5, 2.0, 3)):
            rects, counts = G.lbp_detect_batch(cas, iid, mr, sf, mn, mx, st)
            got = G.rects_to_numpy(rects, counts)
            for i in range(3):
                want = L.o_detect(O, cas, ii[i], mr, sf, mn, mx, st)
                assert got[i].tobytes() == want.tobytes(), ("lbp", w, h, mr, sf, i, len(got[i]), len(want))


def test_lbp_frame_chunks(G, O, cas):
    """k_lbp_scan3 takes big batches through its parity-plane workspace in chunks of frames (1 GiB worth);
    GS_B200_LBP_CHUNK_FRAMES forces small chunks so that a 5-frame batch crosses chunk boundaries (2 + 2 + 1)"""
    w, h, n = 320, 240, 5
    frames = np.stack([L.natural_like(w, h, 60 + i) for i in range(n)])
    ii = np.stack([L.o_integral(O, f) for f in frames])
    iid = dev(ii.view(np.int32))
    os.environ["GS_B200_LBP_CHUNK_FRAMES"] = "2"
    try:
        rects, counts = G.lbp_detect_batch(cas, iid, 1000, 1.1, 1.0, 4.0, 2)
        got = G.rects_to_numpy(rects, counts)
    finally:
        del os.environ["GS_B200_LBP_CHUNK_FRAMES"]
    for i in range(n):
        want = L.o_detect(O, cas, ii[i], 1000, 1.1, 1.0, 4.0, 2)
        assert got[i].tobytes() == want.tobytes(), (i, len(got[i]), len(want))
    assert sum(len(g) for g in got) > 0


# ---- BASELINE.json sizes: crop checks and size-independent properties ------------------------
def _crop_check(full_out, frame, fn, r, rng, ncrops=6, size=160):
    h, w = frame.shape
    spots = [(0, 0), (w - size, 0), (0, h - size), (w - size, h - size)]
    spots += [(int(rng.integers(0, w - size)), int(rng.integers(0, h - size))) for _ in range(ncrops)]
    for (x, y) in spots:
        xa, ya, xb, yb = max(x - r, 0), max(y - r, 0), min(x + size + r, w), min(y + size + r, h)
        sub = np.ascontiguousarray(frame[ya:yb, xa:xb])
        want = fn(sub)
        # rows/cols whose windows stay inside the crop (or touch the true image border) are exact
        ix0, iy0 = (0 if xa == 0 else r), (0 if ya == 0 else r)
        ix1, iy1 = (sub.shape[1] if xb == w else sub.shape[1] - r), (sub.shape[0] if yb == h else sub.shape[0] - r)
        assert np.array_equal(full_out[ya + iy0:ya + iy1, xa + ix0:xa + ix1], want[iy0:iy1, ix0:ix1]), (x, y)


def test_c2_blur_sobel_4096(G, O):
    """config C2 shape (4096x4096, small batch): crops of the GPU output vs the oracle on the crop"""
    import torch
    rng = np.random.default_rng(17)
    torch.manual_seed(1)
    src = torch.randint(0, 256, (3, 4096, 4096), dtype=torch.uint8, device="cuda")
    blur = G.blur_batch(src, 5)
    sob = G.sobel_batch(blur)
    f = src[1].cpu().numpy(); b = blur[1].cpu().numpy(); s = sob[1].cpu().numpy()
    _crop_check(b, f, lambda a: L.o_blur(O, a, 5), 5, rng)
    # sobel: compare interior of crops (border rows/cols of a crop are not written by the oracle)
    for (x, y) in [(0, 0), (4096 - 200, 4096 - 200), (1000, 2000), (3071, 255)]:
        sub = np.ascontiguousarray(b[y:y + 200, x:x + 200])
        assert np.array_equal(s[y + 1:y + 199, x + 1:x + 199], L.o_sobel(O, sub)[1:-1, 1:-1])
    assert (s[0] == 0).all() and (s[:, 0] == 0).all() and (s[-1] == 0).all() and (s[:, -1] == 0).all()
    # idempotence-style property: blur of a constant frame is that constant, at full size
    const = torch.full((1, 4096, 4096), 201, dtype=torch.uint8, device="cuda")
    assert bool((G.blur_batch(const, 5) == 201).all())
    # erode <= src <= dilate pointwise, at full size
    e, d = G.erode_batch(src[:1]), G.dilate_batch(src[:1])
    assert bool((e <= src[:1]).all()) and bool((d >= src[:1]).all())


def test_c3_orb_1080p(G, O):
    """config C3 shape (1920x1080, nkps=1250, t=20; small batch) against the oracle"""
    frames = np.stack([L.natural_like(1920, 1080, 60), np.random.default_rng(3).integers(0, 256, (1080, 1920)).astype(np.uint8)])
    _, kps, counts = G.orb_extract_batch(dev(frames), 1250, 20)
    got = G.kps_to_numpy(kps, counts)
    for i in range(2):
        want = L.o_orb(O, frames[i], np.zeros_like(frames[i]), 1250, 20)
        assert len(got[i]) == len(want)
        assert got[i].tobytes() == want.tobytes(), i


def test_reference_unit_tests_run_on_cuda_path():
    """oracle/_ref/test_overlay is the reference's own test.c, unmodified, compiled in overlay mode against
    libgrayskull_b200.so (oracle/Makefile): its asserts on blur / threshold / histogram / otsu / morph / sobel /
    resize / integral / adaptive threshold / template matching now exercise the CUDA kernels through host-pointer staging."""
    import subprocess
    exe = os.path.join(L.ORACLE_DIR, "_ref", "test_overlay")
    if not os.path.exists(exe):
        pytest.skip("overlay test binary not built (needs the reference tree at build time)")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.returncode, r.stdout[-400:], r.stderr[-400:])


def test_golden_next_rows(G):
    """the 8(f) rows against the reference-generated fixture (tests/golden/next_golden.npz), single-image API"""
    class Impl:
        gs_histogram = staticmethod(G.gs_histogram)
        gs_otsu_threshold = staticmethod(G.gs_otsu_threshold)
        gs_threshold = staticmethod(G.gs_threshold)
        gs_filter = staticmethod(G.gs_filter)
        gs_match_template = staticmethod(G.gs_match_template)
        gs_find_best_match = staticmethod(G.gs_find_best_match)
        gs_match_orb = staticmethod(G.gs_match_orb)

        @staticmethod
        def gs_orb(a, nkps, t):
            return G.gs_orb_extract(a, nkps, t, np.zeros_like(a))

    L.check_next_golden(Impl)


def test_cli_batch_pipeline(G, O, tmp_path):
    """gsb_magick: PGM batch in, device-resident pipeline, PGM batch out -- against the oracle chain
    (the reference Makefile's lena chain plus sobel / filter / resize stages)"""
    import subprocess
    from grayskull_b200 import _lib
    exe = os.path.join(os.path.dirname(_lib.LIB_PATH), "gsb_magick")
    w, h, n = 320, 200, 3
    frames = [L.natural_like(w, h, 90 + f) for f in range(n)]
    paths = []
    for f, a in enumerate(frames):
        pth = tmp_path / ("in%d.pgm" % f)
        pth.write_bytes(b"P5\n%d %d\n255\n" % (w, h) + a.tobytes())
        paths.append(str(pth))

    def read(pth):
        b = open(pth, "rb").read()
        hdr = b.split(b"\n", 3)
        ww, hh = map(int, hdr[1].split())
        return np.frombuffer(hdr[3], np.uint8).reshape(hh, ww)

    r = subprocess.run([exe, "blur:2,threshold:otsu,erode:2,dilate:2", str(tmp_path / "a_")] + paths, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    for f, a in enumerate(frames):
        x = L.o_blur(O, a, 2)
        t = O.gso_otsu_threshold(L.ptr(x), w, h)
        x = x.copy(); O.gso_threshold(L.ptr(x), w, h, t)
        for op in (0, 0, 1, 1):
            x = L.o_morph(O, x, op)
        assert np.array_equal(read(str(tmp_path / ("a_%04d.pgm" % f))), x), f
    r = subprocess.run([exe, "filter:gaussian,sobel,threshold:otsu+10,downsample,resize:100:37,keypoints:50:20", str(tmp_path / "b_")] + paths,
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert r.stdout.count("keypoints") == n
    for f, a in enumerate(frames):
        k, norm = L.filter_kernel("gaussian")
        x = np.zeros_like(a); O.gso_filter(L.ptr(x), L.ptr(a), w, h, L.ptr(k), 3, 3, norm)
        x = L.o_sobel(O, x, 0)
        t = (O.gso_otsu_threshold(L.ptr(x), w, h) + 10) & 255
        x = x.copy(); O.gso_threshold(L.ptr(x), w, h, t)
        x = L.o_resize(O, L.o_down(O, x), 100, 37)
        assert np.array_equal(read(str(tmp_path / ("b_%04d.pgm" % f))), x), f
    # the reference's document scanner (nanomagick.c:186-210) as one device-resident stage, and the blob counter
    rng = np.random.default_rng(5)
    docs = []
    for f in range(2):
        doc = np.full((300, 400), 40, np.int16) + rng.integers(-8, 9, (300, 400))
        yy, xx = np.mgrid[0:300, 0:400]
        inside = (yy > 40 + xx * 0.05 + 7 * f) & (yy < 250 - xx * 0.04) & (xx > 60 + yy * 0.08) & (xx < 340 - yy * 0.03 - 11 * f)
        doc[inside] = 210 + rng.integers(-10, 11, int(inside.sum()))
        docs.append(np.clip(doc, 0, 255).astype(np.uint8))
    dpaths = []
    for f, a in enumerate(docs):
        pth = tmp_path / ("doc%d.pgm" % f)
        pth.write_bytes(b"P5\n400 300\n255\n" + a.tobytes())
        dpaths.append(str(pth))
    r = subprocess.run([exe, "blobs:500,scan:160:200", str(tmp_path / "s_")] + dpaths, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    for f, a in enumerate(docs):
        lab = np.zeros(a.shape, np.uint16); bl = np.zeros(500, L.BLOB_DTYPE)
        assert ("frame %d: %d blobs" % (f, O.gso_blobs(L.ptr(a), 400, 300, L.ptr(lab), L.ptr(bl), 500))) in r.stdout
        x = L.o_blur(O, a, 1)
        t = (O.gso_otsu_threshold(L.ptr(x), 400, 300) + 10) & 255
        x = x.copy(); O.gso_threshold(L.ptr(x), 400, 300, t)
        lab = np.zeros(a.shape, np.uint16); bl = np.zeros(1000, L.BLOB_DTYPE)
        m = O.gso_blobs(L.ptr(x), 400, 300, L.ptr(lab), L.ptr(bl), 1000)
        assert m > 0
        largest = 0
        for i in range(1, m):
            if bl["area"][i] > bl["area"][largest]:
                largest = i
        c = np.zeros((4, 2), np.uint32)
        O.gso_blob_corners(L.ptr(x), 400, 300, L.ptr(lab), L.ptr(bl[largest:largest + 1]), L.ptr(c))
        want = np.empty((200, 160), np.uint8)
        O.gso_perspective_correct(L.ptr(want), 160, 200, L.ptr(a), 400, 300, L.ptr(c))
        assert np.array_equal(read(str(tmp_path / ("s_%04d.pgm" % f))), want), f


def test_reference_cli_overlay_vs_cpu(tmp_path):
    """The reference's own CLI (examples/nanomagick/nanomagick.c, unmodified) built twice by oracle/Makefile: as
    upstream builds it, and in overlay mode against libgrayskull_b200.so.  The command lines of the reference
    Makefile's `testdata` target (on lena from the fixture and synthetic stand-ins for its other images) must
    give the same exit codes, the same stdout and byte-identical PGMs from both."""
    import subprocess
    ref_dir = os.path.join(L.ORACLE_DIR, "_ref")
    exes = {k: os.path.join(ref_dir, "nanomagick_" + k) for k in ("cpu", "overlay")}
    if not all(os.path.exists(e) for e in exes.values()):
        pytest.skip("nanomagick builds not present (need the reference tree at build time)")

    def pgm(path, a):
        path.write_bytes(b"P5\n%d %d\n255\n" % (a.shape[1], a.shape[0]) + a.tobytes())

    lena = np.load(os.path.join(GOLD, "lena_golden.npz"))["lena"]
    pgm(tmp_path / "lena.pgm", lena)
    pgm(tmp_path / "nat.pgm", L.natural_like(320, 240, 11))
    rng = np.random.default_rng(5)
    doc = np.full((300, 400), 40, np.int16) + rng.integers(-8, 9, (300, 400))
    yy, xx = np.mgrid[0:300, 0:400]
    inside = (yy > 40 + xx * 0.05) & (yy < 250 - xx * 0.04) & (xx > 60 + yy * 0.08) & (xx < 340 - yy * 0.03)
    doc[inside] = 210 + rng.integers(-10, 11, int(inside.sum()))
    doc[inside & (yy % 12 < 3) & (xx % 9 < 6)] = 60                     # "text"
    pgm(tmp_path / "doc.pgm", np.clip(doc, 0, 255).astype(np.uint8))
    marks = np.full((240, 320), 200, np.uint8)
    for (y, x) in ((30, 40), (30, 200), (150, 60), (140, 220)):
        marks[y:y + 50, x:x + 50] = 20; marks[y + 10:y + 40, x + 10:x + 40] = 230
    pgm(tmp_path / "marks.pgm", np.clip(marks.astype(np.int16) + rng.integers(-6, 7, marks.shape), 0, 255).astype(np.uint8))

    cmds = [("identify", "{i}lena.pgm"), ("resize 128 64", "{i}lena.pgm {o}r.pgm"), ("crop 32 32 64 64", "{i}lena.pgm {o}c.pgm"),
            ("blur 1", "{i}lena.pgm {o}b1.pgm"), ("blur 9", "{i}lena.pgm {o}b9.pgm"), ("threshold 128", "{o}b1.pgm {o}t128.pgm"),
            ("threshold otsu", "{o}b1.pgm {o}otsu.pgm"), ("adaptive 15 5", "{i}lena.pgm {o}ad.pgm"),
            ("morph erode 2", "{o}otsu.pgm {o}er.pgm"), ("morph dilate 2", "{o}er.pgm {o}di.pgm"), ("sobel", "{i}lena.pgm {o}so.pgm"),
            ("blur 3", "{i}marks.pgm {o}m1.pgm"), ("sobel", "{o}m1.pgm {o}m2.pgm"), ("threshold otsu", "{o}m2.pgm {o}m3.pgm"),
            ("morph dilate 9", "{o}m3.pgm {o}m4.pgm"), ("morph erode 10", "{o}m4.pgm {o}m5.pgm"), ("blobs 150", "{o}m5.pgm {o}m6.pgm"),
            ("scan", "{i}doc.pgm {o}scan.pgm"), ("keypoints 100 20", "{i}nat.pgm {o}kp.pgm"),
            ("orb {o}c.pgm", "{i}lena.pgm {o}orb.pgm"), ("faces 1", "{i}lena.pgm {o}f1.pgm"), ("faces 2", "{i}lena.pgm {o}f2.pgm")]
    outs = {}
    for kind, exe in exes.items():
        od = tmp_path / kind
        od.mkdir()
        log = []
        for verb, files in cmds:
            line = (verb + " " + files).format(i=str(tmp_path) + "/", o=str(od) + "/")
            r = subprocess.run([exe] + line.split(), capture_output=True, timeout=300)
            log.append((verb, r.returncode, r.stdout.replace(str(od).encode(), b"<out>")))
        outs[kind] = (log, {p.name: p.read_bytes() for p in sorted(od.iterdir())})
    (log_c, files_c), (log_o, files_o) = outs["cpu"], outs["overlay"]
    assert log_c == log_o
    assert all(rc == 0 for _, rc, _ in log_c), [(v, rc) for v, rc, _ in log_c if rc]
    assert sorted(files_c) == sorted(files_o) and len(files_c) >= 20
    for name in files_c:
        assert files_c[name] == files_o[name], name
    # the overlay build binds the whole hot path AND the 8(f) rows to the CUDA library: every one of these is an
    # undefined (imported) symbol of the executable, none resolves to the upstream CPU body (gs_cpu_*)
    nm = subprocess.run(["nm", "-D", "--undefined-only", exes["overlay"]], capture_output=True, text=True).stdout
    for sym in ("gs_blur", "gs_sobel", "gs_adaptive_threshold", "gs_erode", "gs_dilate", "gs_resize", "gs_fast", "gs_orb_extract",
                "gs_match_orb", "gs_integral", "gs_lbp_detect", "gs_threshold", "gs_otsu_threshold", "gs_blobs",
                "gs_blob_corners", "gs_perspective_correct"):
        assert (" U " + sym + "\n") in nm, sym


def _o_hist(O, a):
    h = np.zeros(256, np.uint32); O.gso_histogram(L.ptr(a), a.shape[1], a.shape[0], L.ptr(h)); return h


def test_histogram_otsu_threshold_vs_oracle(G, O):
    """gs_histogram / gs_otsu_threshold / gs_threshold (reference grayskull.h:199-229): test.c vectors through the
    single-image API, then bimodal / flat / two-level / noise images incl. ragged sizes (scalar path)"""
    a = np.array([[0, 50, 100], [50, 100, 150], [100, 150, 200]], np.uint8)
    hist = G.gs_histogram(a)
    assert hist[0] == 1 and hist[50] == 2 and hist[100] == 3 and hist[150] == 2 and hist[200] == 1 and hist.sum() == 9
    assert G.gs_threshold(np.array([[50, 150], [75, 200]], np.uint8), 100).tolist() == [[0, 255], [0, 255]]
    assert G.gs_otsu_threshold(np.array([[40, 50, 60], [45, 55, 50], [190, 200, 210]], np.uint8)) == 60
    assert G.gs_otsu_threshold(np.array([[0, 85], [170, 255]], np.uint8)) == 85
    assert G.gs_otsu_threshold(np.full((2, 2), 128, np.uint8)) == 0
    rng = np.random.default_rng(21)
    for a in L.otsu_images(rng) + [L.natural_like(1024, 1024, 5), np.zeros((512, 512), np.uint8)]:
        h, w = a.shape
        assert np.array_equal(G.gs_histogram(a), _o_hist(O, a)), a.shape
        t = O.gso_otsu_threshold(L.ptr(a), w, h)
        assert G.gs_otsu_threshold(a) == t, (a.shape, t)
        for th in (0, 100, 255, int(t)):
            want = a.copy(); O.gso_threshold(L.ptr(want), w, h, th)
            assert np.array_equal(G.gs_threshold(a.copy(), th), want), (a.shape, th)


def test_histogram_otsu_threshold_batches(G, O):
    """device-resident batches: per-frame histograms, Otsu thresholds kept on the device and fed to the
    per-frame threshold (+10 like nanomagick.c:191); 4096^2 frames cross the chunk boundaries"""
    import torch
    rng = np.random.default_rng(22)
    for (w, h, n) in ((640, 480, 9), (1000, 37, 5), (4096, 4096, 3)):
        frames = np.stack([np.clip(rng.normal(60 + 15 * f, 20, (h, w)) * (rng.random((h, w)) < 0.5) +
                                   rng.normal(200 - 10 * f, 15, (h, w)) * (rng.random((h, w)) < 0.4), 0, 255).astype(np.uint8)
                           for f in range(n)])
        if n > 2:
            frames[1] = 77                                   # constant frame: every lane hits one bin
        d = dev(frames)
        hist = G.histogram_batch(d).cpu().numpy().view(np.uint32)
        for f in range(n):
            assert np.array_equal(hist[f], np.bincount(frames[f].ravel(), minlength=256)), (w, h, f)
        th = G.otsu_threshold_batch(d)
        want_t = [O.gso_otsu_from_hist(L.ptr(np.ascontiguousarray(hist[f])), w * h) for f in range(n)]
        assert th.cpu().numpy().tolist() == want_t
        out = G.threshold_batch(d.clone(), th, 10).cpu().numpy()
        for f in range(n):
            assert np.array_equal(out[f], np.where(frames[f] > ((want_t[f] + 10) & 255), 255, 0).astype(np.uint8)), (w, h, f)
        out = G.threshold_batch(d.clone(), 128).cpu().numpy()
        assert np.array_equal(out, np.where(frames > 128, 255, 0).astype(np.uint8))


def test_filter_vs_oracle(G, O):
    """gs_filter (reference grayskull.h:255-266): presets and stress kernels (negative sums with norm > 1, norms
    beyond the magic-multiplier range, even / non-square sizes), widths on and off the 8-px fast path"""
    rng = np.random.default_rng(31)
    for (w, h) in ((64, 48), (640, 480), (8, 1), (33, 17), (1, 1), (250, 40)):
        a = rng.integers(0, 256, (h, w), dtype=np.uint8) if w < 600 else L.natural_like(w, h, 2)
        for name in L.FILTER_KERNELS:
            k, norm = L.filter_kernel(name)
            want = np.zeros_like(a)
            O.gso_filter(L.ptr(want), L.ptr(a), w, h, L.ptr(k), k.shape[1], k.shape[0], norm)
            got = G.gs_filter(np.full_like(a, 7), a, k, norm)
            assert np.array_equal(got, want), (w, h, name)
    # device-resident batch, band boundaries (h not a multiple of the 16-row bands)
    frames = np.stack([L.natural_like(256, 100, 50 + f) for f in range(5)])
    for name in ("sharpen", "emboss", "box", "gaussian", "emboss_norm3", "k5"):
        k, norm = L.filter_kernel(name)
        got = G.filter_batch(dev(frames), k.view(np.int8), norm).cpu().numpy()
        for f in range(5):
            want = np.zeros_like(frames[f])
            O.gso_filter(L.ptr(want), L.ptr(frames[f]), 256, 100, L.ptr(k), k.shape[1], k.shape[0], norm)
            assert np.array_equal(got[f], want), (name, f)


def test_match_template_vs_oracle(G, O):
    """gs_match_template / gs_find_best_match (reference grayskull.h:705-738): test.c vectors, ragged template
    widths (tail mask), template == image, word-aligned and unaligned image widths"""
    import torch
    img = np.array([[0, 0, 0, 0, 0], [0, 100, 150, 200, 0], [0, 125, 175, 225, 0], [0, 110, 160, 210, 0], [0, 0, 0, 0, 0]], np.uint8)
    res = G.gs_match_template(img, np.ascontiguousarray(img[1:4, 1:4]))
    assert G.gs_find_best_match(res) == (1, 1) and res[1, 1] == 255
    s = np.full((4, 4), 50, np.uint8); s[1:3, 1:3] = 255
    assert G.gs_find_best_match(G.gs_match_template(s, np.full((2, 2), 255, np.uint8))) == (1, 1)
    assert G.gs_find_best_match(np.zeros((3, 4), np.uint8)) == (0, 0)
    rng = np.random.default_rng(32)
    for (w, h, tw, th) in ((64, 48, 8, 8), (37, 29, 37, 29), (52, 40, 1, 1), (92, 31, 17, 5), (36, 70, 4, 33), (320, 240, 31, 27),
                           (33, 70, 6, 9), (320, 200, 320, 3)):
        a = L.natural_like(w, h, w + h)
        y0, x0 = int(rng.integers(0, h - th + 1)), int(rng.integers(0, w - tw + 1))
        t = np.clip(a[y0:y0 + th, x0:x0 + tw].astype(np.int16) + rng.integers(-3, 4, (th, tw)), 0, 255).astype(np.uint8)
        for tmpl in (t, rng.integers(0, 256, (th, tw), dtype=np.uint8)):
            want = np.zeros((h - th + 1, w - tw + 1), np.uint8)
            O.gso_match_template(L.ptr(a), w, h, L.ptr(tmpl), tw, th, L.ptr(want))
            got = G.gs_match_template(a, np.ascontiguousarray(tmpl))
            assert np.array_equal(got, want), (w, h, tw, th)
            b = O.gso_find_best_match(L.ptr(want), want.shape[1], want.shape[0])
            assert G.gs_find_best_match(got) == (b % want.shape[1], b // want.shape[1])
    # batch: one template against several frames, best match per frame on the device
    frames = np.stack([L.natural_like(256, 128, 70 + f) for f in range(4)])
    tmpl = np.ascontiguousarray(frames[2, 40:40 + 24, 100:100 + 30])
    r = G.match_template_batch(dev(frames), dev(tmpl))
    best = G.find_best_match_batch(r).cpu().numpy()
    r = r.cpu().numpy()
    for f in range(4):
        want = np.zeros((128 - 24 + 1, 256 - 30 + 1), np.uint8)
        O.gso_match_template(L.ptr(frames[f]), 256, 128, L.ptr(tmpl), 30, 24, L.ptr(want))
        assert np.array_equal(r[f], want), f
        b = O.gso_find_best_match(L.ptr(want), want.shape[1], want.shape[0])
        assert tuple(best[f]) == (b % want.shape[1], b // want.shape[1])
    assert tuple(best[2]) == (100, 40)


def test_match_orb_vs_oracle(G, O):
    """gs_match_orb (reference grayskull.h:680-699): ties, empty sets, caps, max_distance extremes"""
    rng = np.random.default_rng(16)
    for (n1, n2, mm, md) in ((50, 60, 300, 60.0), (300, 257, 40, 60.0), (7, 0, 10, 60.0), (120, 1, 500, 300.0),
                             (90, 33, 500, 10.0), (64, 64, 500, 0.0), (200, 500, 500, 255.5), (1250, 1250, 2500, 60.0),
                             (9, 700, 3, 80.0), (513, 31, 513, 64.5)):
        k1, k2 = L.desc_sets(rng, n1, n2)
        want = L.o_match(O, k1, k2, mm, md)
        got = G.gs_match_orb(k1, k2, mm, md)
        assert got.tobytes() == want.tobytes(), (n1, n2, mm, md, len(got), len(want))
    assert len(G.gs_match_orb(np.zeros(0, L.KP_DTYPE), L.desc_sets(rng, 1, 9)[1], 10, 60.0)) == 0


def test_match_orb_batch_after_extract(G, O):
    """frame pairs: orb_extract_batch output (device resident) fed straight into match_orb_batch"""
    import torch
    w, h, n, nk = 640, 480, 6, 600
    frames = np.stack([L.natural_like(w, h, 40 + (f // 2)) for f in range(n)])
    frames[1::2] = np.roll(frames[1::2], (3, 5), axis=(1, 2))           # odd frames: shifted copies of the even ones
    d = dev(frames)
    _, kps, counts = G.orb_extract_batch(d, nk, 20)
    a, b = kps[0::2].contiguous(), kps[1::2].contiguous()
    ca, cb = counts[0::2].contiguous(), counts[1::2].contiguous()
    m, mc = G.match_orb_batch(a, ca, b, cb, nk, 60.0)
    torch.cuda.synchronize()
    m = m.cpu().numpy(); mc = mc.cpu().numpy()
    ka, kb = G.kps_to_numpy(a, ca), G.kps_to_numpy(b, cb)
    for p in range(n // 2):
        want = L.o_match(O, ka[p], kb[p], nk, 60.0)
        got = np.ascontiguousarray(m[p, :mc[p]]).view(np.uint32).reshape(-1, 3)
        assert mc[p] == len(want) and got.tobytes() == want.tobytes(), p
        assert len(want) > 20                                            # the shifted copy really matches


def test_c4_integral_lbp_2160p(G, O, cas):
    """config C4 shape (3840x2160, sf 1.1, scales 1..4, step 2): window count, integral checksum,
    and full rect-list parity on one frame (the oracle needs a few seconds for it)"""
    import grayskull_b200 as g
    assert G.lbp_window_count(cas, 3840, 2160, 1.1, 1.0, 4.0, 2) == 30016520   # SURVEY 8(d)
    f = L.natural_like(3840, 2160, 77)
    src = dev(f[None])
    ii = G.integral_batch(src)
    iih = ii.cpu().numpy().view(np.uint32)[0]
    want_ii = L.o_integral(O, f)
    assert np.array_equal(iih, want_ii)
    assert int(iih[-1, -1]) == int(f.astype(np.uint64).sum() % (1 << 32))   # checksum of checksums
    rects, counts = G.lbp_detect_batch(cas, ii, 65536, 1.1, 1.0, 4.0, 2)
    got = G.rects_to_numpy(rects, counts)[0]
    want = L.o_detect(O, cas, want_ii, 65536, 1.1, 1.0, 4.0, 2)
    assert got.tobytes() == want.tobytes(), (len(got), len(want))


def test_c5_pipeline_composition(G, O, cas):
    """config C5 shape of work on small frames: blur -> sobel -> ORB and integral + LBP on the sobel
    output, every stage consuming the previous stage's device buffer, against the oracle chain"""
    import torch
    frames = np.stack([L.natural_like(320, 240, 90 + i) for i in range(3)])
    src = dev(frames)
    blur = G.blur_batch(src, 5)
    sob = G.sobel_batch(blur)
    _, kps, kc = G.orb_extract_batch(sob, 300, 20)
    ii = G.integral_batch(sob)
    rects, rc = G.lbp_detect_batch(cas, ii, 1000, 1.1, 1.0, 4.0, 2)
    gk, gr = G.kps_to_numpy(kps, kc), G.rects_to_numpy(rects, rc)
    for i in range(3):
        b = L.o_blur(O, frames[i], 5)
        s = L.o_sobel(O, b)
        assert np.array_equal(sob[i].cpu().numpy(), s)
        assert gk[i].tobytes() == L.o_orb(O, s, np.zeros_like(s), 300, 20).tobytes()
        t = L.o_integral(O, s)
        assert np.array_equal(ii[i].cpu().numpy().view(np.uint32), t)
        assert gr[i].tobytes() == L.o_detect(O, cas, t, 1000, 1.1, 1.0, 4.0, 2).tobytes()


# ---- round 2: sharding over NCCL, re-entrancy, large-batch offsets, ADVICE cases ---------------------------
def test_sharded_pipeline_nccl():
    """SURVEY.md 8(e): one NCCL scatter of uint8 frames from rank 0, the C5 chain on every rank's shard, one
    NCCL gather of sobel maps / keypoints / rects, compared frame by frame with the oracle chain on rank 0
    (tests/shard_worker.py).  World size 2 when the machine has two GPUs, else the same code
    path with a single rank (scatter / gather degenerate to local copies)."""
    import subprocess
    import sys
    import torch
    world = min(2, torch.cuda.device_count())
    port = str(29600 + os.getpid() % 300)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", port, os.path.join(L.ROOT, "tests", "shard_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "SHARD_OK world=%d" % world in r.stdout, r.stdout[-2000:]


def test_single_image_api_is_reentrant(G, O):
    """the reference's gs_* functions are re-entrant (SURVEY.md 8b "Threading"): eight host threads hammer the
    drop-in API with different images and radii concurrently (ctypes releases the GIL inside the calls); every
    result must equal the oracle's -- each thread stages through its own stream and arenas"""
    import threading
    rng = np.random.default_rng(5)
    jobs = []
    for i in range(8):
        h, w = int(rng.integers(90, 400)), int(rng.integers(6, 40)) * 16
        a = rng.integers(0, 256, (h, w)).astype(np.uint8)
        r = int(rng.integers(1, 8))
        jobs.append((a, r, L.o_blur(O, a, r), L.o_sobel(O, a), L.o_integral(O, a)))
    errs = []

    def work(j):
        a, r, wb, ws, wi = jobs[j]
        try:
            for _ in range(25):
                d = np.empty_like(a); G.gs_blur(d, a, r)
                s = np.zeros_like(a); G.gs_sobel(s, a)
                ii = np.empty(a.shape, np.uint32); G.gs_integral(a, ii)
                if not (np.array_equal(d, wb) and np.array_equal(s, ws) and np.array_equal(ii, wi)):
                    errs.append(j)
                    return
        except Exception as e:   # noqa: BLE001
            errs.append((j, repr(e)))

    th = [threading.Thread(target=work, args=(j,)) for j in range(8)]
    [t.start() for t in th]
    [t.join() for t in th]
    assert not errs, errs


def test_last_frame_of_a_large_batch(G, O, cas):
    """offset arithmetic past 4 GiB: frame 271 of a 272-frame 4096x4096 batch (byte offset 4.5 GB) for the
    stencils, and the last frame of a 136-frame UHD integral batch (u32 table offset 4.5 GB)"""
    import torch
    n, h, w = 272, 4096, 4096
    src = torch.zeros((n, h, w), dtype=torch.uint8, device="cuda")
    f = np.random.default_rng(9).integers(0, 256, (h, w)).astype(np.uint8)
    src[n - 1].copy_(dev(f))
    blur = G.blur_batch(src, 5)
    assert bool((blur[: n - 1] == 0).all())
    b = blur[n - 1].cpu().numpy()
    rng = np.random.default_rng(2)
    _crop_check(b, f, lambda a: L.o_blur(O, a, 5), 5, rng)
    del src
    sob = G.sobel_batch(blur)
    s = sob[n - 1].cpu().numpy()
    for (x, y) in [(0, 0), (4096 - 200, 4096 - 200), (1777, 2000)]:
        sub = np.ascontiguousarray(b[y:y + 200, x:x + 200])
        assert np.array_equal(s[y + 1:y + 199, x + 1:x + 199], L.o_sobel(O, sub)[1:-1, 1:-1])
    if hasattr(G, "blur_sobel_batch"):
        src2 = torch.zeros((n, h, w), dtype=torch.uint8, device="cuda")
        src2[n - 1].copy_(dev(f))
        del sob
        fs = G.blur_sobel_batch(src2, 5)
        assert np.array_equal(fs[n - 1].cpu().numpy(), s)
        del src2, fs
    del blur
    torch.cuda.empty_cache()
    n4, h4, w4 = 136, 2160, 3840
    f4 = L.natural_like(w4, h4, 31)
    src4 = torch.zeros((n4, h4, w4), dtype=torch.uint8, device="cuda")
    src4[n4 - 1].copy_(dev(f4))
    ii = G.integral_batch(src4)
    want_ii = L.o_integral(O, f4)
    assert np.array_equal(ii[n4 - 1].cpu().numpy().view(np.uint32), want_ii)
    rects, counts = G.lbp_detect_batch(cas, ii[n4 - 4:], 65536, 1.1, 1.0, 4.0, 2)
    got = G.rects_to_numpy(rects, counts)
    assert got[3].tobytes() == L.o_detect(O, cas, want_ii, 65536, 1.1, 1.0, 4.0, 2).tobytes()
    assert len(got[0]) == 0


def test_fast_huge_threshold_and_foreign_scoremap(G, O):
    """ADVICE r1: thresholds above 255 wrap in the reference's unsigned arithmetic (:496-498) -- the result must not
    depend on which kernel (tiled / per-pixel) runs; a score map shorter than the image must not be read past its end"""
    a = L.natural_like(256, 96, 4)
    for t in (256, 300, 2**31 + 5, 2**32 - 3, 2**32 - 200):
        for force in (0, 1):
            import grayskull_b200 as g
            g.lib().gs_b200_force_generic(force)
            try:
                sm = np.zeros_like(a)
                got = G.gs_fast(a, sm, 500, t)
            finally:
                g.lib().gs_b200_force_generic(0)
            sm2 = np.zeros_like(a)
            want = L.o_fast(O, a, sm2, 500, t)
            assert got.tobytes() == want.tobytes() and np.array_equal(sm, sm2), (t, force)
    sm = np.full((40, 256), 7, np.uint8)               # foreign size: fewer rows than the image
    sm2 = sm.copy()
    got = G.gs_fast(a, sm, 500, 20)
    want = L.o_fast(O, a, sm2, 500, 20)
    assert got.tobytes() == want.tobytes() and np.array_equal(sm, sm2)


def test_orientation_large_radius(G):
    """ADVICE r1: for r > 15 the reference's float moment sums round; the device follows the same fp32 order
    (checked against the compiled reference through golden values generated by tools/make_golden.py)"""
    z = np.load(os.path.join(GOLD, "round2_golden.npz"))
    a = np.ascontiguousarray(z["orient_img"])
    for (x, y, r), want in zip(z["orient_xyr"], z["orient_angle"]):
        got = G.gs_compute_orientation(a, int(x), int(y), int(r))
        assert np.float32(got).tobytes() == np.float32(want).tobytes(), (x, y, r, got, want)


def test_trig_selfcheck_matches_this_libm():
    """the device restates glibc 2.39's sinf / atan2f; on this image (glibc 2.39) the first-use self-check must
    report zero differing samples"""
    import grayskull_b200 as g
    assert g.lib().gs_b200_trig_selfcheck() == 0


WIDE_SHAPES = [(256, 128), (272, 140), (640, 480), (100, 37), (612, 90), (17, 1), (1, 1), (1024, 300), (2048, 67)]


def test_wide_radius_box_vs_oracle_and_reference_goldens(G, O):
    """VERDICT r1 item 6: radii beyond 7 (the reference Makefile's `blur 9`, `adaptive 15 5`) run the
    radius-independent kernel (k_box_wide); r > 120 falls back to the per-pixel kernel.  Against the oracle on
    aligned, ragged and tiny shapes, band / strip seams included, and against reference-generated goldens."""
    rng = np.random.default_rng(11)
    for (w, h) in WIDE_SHAPES:
        frames = np.stack([rng.integers(0, 256, (h, w)).astype(np.uint8), L.natural_like(w, h, 8),
                           np.full((h, w), 255, np.uint8)])
        src = dev(frames)
        for r in (8, 9, 10, 12, 13, 15, 16, 17, 22, 31, 63, 64, 100, 120, 121, 300):   # r mod 4 = 0..3: the four k_box_mid instantiations
            if r > 31 and w * h > 200000:
                continue                       # the oracle's cost grows with r
            gb = G.blur_batch(src, r).cpu().numpy()
            c = int(rng.integers(-60, 60))
            ga = G.adaptive_threshold_batch(src, r, c).cpu().numpy()
            for i in range(3):
                assert np.array_equal(gb[i], L.o_blur(O, frames[i], r)), ("blur", w, h, r, i)
                assert np.array_equal(ga[i], L.o_adaptive(O, frames[i], r, c)), ("adaptive", w, h, r, c, i)
    z = np.load(os.path.join(GOLD, "round2_golden.npz"))
    for tag in z["radius_tags"]:
        a = np.ascontiguousarray(z["radius_img_" + str(tag)])
        for r in z["radii"]:
            r = int(r)
            d = np.empty_like(a); G.gs_blur(d, a, r)
            assert np.array_equal(d, z["blur%d_%s" % (r, tag)]), ("golden blur", tag, r)
            d = np.empty_like(a); G.gs_adaptive_threshold(d, a, r, 5 - r)
            assert np.array_equal(d, z["adaptive%d_%s" % (r, tag)]), ("golden adaptive", tag, r)
    # a tall frame: several row bands per strip (band seams), full-size width
    f = L.natural_like(4096, 1500, 12)
    got = G.blur_batch(dev(f[None]), 15)[0].cpu().numpy()
    rng2 = np.random.default_rng(3)
    _crop_check(got, f, lambda a: L.o_blur(O, a, 15), 15, rng2)


@pytest.mark.parametrize("force_generic", [0, 1])
def test_fused_blur_sobel_vs_oracle_chain(G, O, force_generic):
    """gs_b200_blur_sobel_batch == gs_blur -> gs_sobel bit for bit (VERDICT r1 item 3): every radius of the fused
    kernel (1..7) and the two-kernel fall-back (0, 8, 15; ragged widths), dst pre-filled with 77 so that sobel's
    untouched 1-px frame is checked, widths and heights around the tile seams of this and earlier geometries"""
    import grayskull_b200 as g
    g.lib().gs_b200_force_generic(force_generic)
    try:
        rng = np.random.default_rng(23)
        for (w, h) in [(256, 128), (272, 140), (512, 300), (16, 16), (48, 7), (1024, 67), (640, 480), (100, 37), (17, 1), (3, 3),
                       (2, 9), (464, 259), (240, 34), (224, 33)]:
            frames = np.stack([rng.integers(0, 256, (h, w)).astype(np.uint8), L.natural_like(w, h, 5), np.full((h, w), 255, np.uint8)])
            src = dev(frames)
            for r in (0, 1, 2, 3, 4, 5, 6, 7, 8, 15):
                got = G.blur_sobel_batch(src, r, out=dev(np.full_like(frames, 77))).cpu().numpy()
                for i in range(3):
                    want = L.o_sobel(O, L.o_blur(O, frames[i], r), 77)
                    assert np.array_equal(got[i], want), (w, h, r, i)
    finally:
        g.lib().gs_b200_force_generic(0)
    # full C2 frame size: equality with the two-call chain on the device
    import torch
    torch.manual_seed(4)
    src = torch.randint(0, 256, (3, 4096, 4096), dtype=torch.uint8, device="cuda")
    a = G.blur_sobel_batch(src, 5)
    b = G.sobel_batch(G.blur_batch(src, 5))
    assert bool((a == b).all())


def test_blobs_corners_perspective_vs_reference_goldens_and_oracle(G, O):
    """SURVEY.md 8(f) N4: gs_blobs (labels = the reference's union-find numbering, running out of labels included),
    gs_blob_corners, gs_perspective_correct -- against reference-generated goldens, the oracle on random binary
    images, the batched ABI, and the reference's test.c vector"""
    import torch
    z = np.load(os.path.join(GOLD, "round2_golden.npz"))
    for tag in z["blob_tags"]:
        a = np.ascontiguousarray(z["blob_img_" + str(tag)])
        for nb in (1000, 7, 1):
            labels, blobs = G.gs_blobs(a, nb)
            assert np.array_equal(labels, z["blob_%s_n%d_labels" % (tag, nb)]), (tag, nb)
            assert np.array_equal(np.array(L.blob_fields(blobs), np.int64).reshape(-1, 8), z["blob_%s_n%d_blobs" % (tag, nb)]), (tag, nb)
        key = "blob_%s_corners" % tag
        if key in z.files:
            labels, blobs = G.gs_blobs(a, 1000)
            for j, want in enumerate(z[key]):
                assert np.array_equal(G.gs_blob_corners(a, labels, blobs[j:j + 1]), want), (tag, j)
    src = np.ascontiguousarray(z["persp_src"])
    for qi, q in enumerate(z["persp_quads"]):
        for (dw, dh) in ((160, 100), (33, 47), (1, 1), (2, 5)):
            d = G.gs_perspective_correct(np.empty((dh, dw), np.uint8), src, q)
            assert np.array_equal(d, z["persp_q%d_%dx%d" % (qi, dw, dh)]), (qi, dw, dh)
    # test.c:232-257
    Wv = 255
    a = np.array([[Wv, Wv, 0, 0, Wv, 0], [Wv, 0, 0, Wv, Wv, 0], [0, 0, Wv, Wv, 0, 0], [Wv, Wv, Wv, 0, 0, Wv],
                  [0, Wv, 0, 0, 0, Wv]], np.uint8)
    _, blobs = G.gs_blobs(a, 10)
    assert L.blob_fields(blobs) == [(1, 3, 0, 0, 2, 2, 0, 0), (2, 9, 0, 0, 5, 5, 2, 2), (6, 2, 5, 3, 1, 2, 5, 3)]
    # batched ABI vs the oracle: ragged widths, wide frames (several mask-word chunks per row), label overflow
    rng = np.random.default_rng(31)
    for (w, h, nb) in ((100, 37, 500), (1300, 90, 4000), (640, 480, 3000), (64, 64, 5), (2200, 40, 60000), (33, 200, 2)):
        frames = np.stack([L.binary_like(w, h, 50 + i, density=float(rng.uniform(0.3, 0.7)), smooth=int(rng.integers(0, 5))) for i in range(3)])
        frames[2] = rng.integers(0, 256, (h, w)).astype(np.uint8)
        labels, blobs, counts = G.blobs_batch(dev(frames), nb)
        lab = labels.cpu().numpy().view(np.uint16)
        bl = blobs.cpu().numpy().view(np.uint32)
        cnt = counts.cpu().numpy()
        for i in range(3):
            wl = np.zeros((h, w), np.uint16); wb = np.zeros(nb, L.BLOB_DTYPE)
            m = O.gso_blobs(L.ptr(frames[i]), w, h, L.ptr(wl), L.ptr(wb), nb)
            assert cnt[i] == m, (w, h, nb, i, cnt[i], m)
            assert np.array_equal(lab[i], wl), (w, h, nb, i)
            got = np.ascontiguousarray(bl[i, :m]).view(L.BLOB_DTYPE).reshape(-1)
            assert L.blob_fields(got) == L.blob_fields(wb[:m]), (w, h, nb, i)
    # perspective, batched with device-resident per-frame corners
    frames = np.stack([L.natural_like(200, 150, 70 + i) for i in range(3)])
    quads = rng.integers(0, 230, (3, 4, 2)).astype(np.int32)
    out = G.perspective_correct_batch(dev(frames), 90, 70, torch.from_numpy(quads).cuda()).cpu().numpy()
    for i in range(3):
        want = np.empty((70, 90), np.uint8)
        O.gso_perspective_correct(L.ptr(want), 90, 70, L.ptr(frames[i]), 200, 150, L.ptr(np.ascontiguousarray(quads[i].astype(np.uint32))))
        assert np.array_equal(out[i], want), i


@pytest.mark.parametrize("big", ["0", "1"])
def test_lbp_tile_configs(G, O, cas, big):
    """k_lbp_scan3 runs a scale either as two 512-thread CTAs per SM or (large windows) as one 1024-thread CTA with a
    tile of up to 224 KB; GS_B200_LBP_BIG forces one form for every scale.  Both against the oracle on frames wide and
    tall enough for several tiles per scale, all 15 scales of the 1.1 ladder"""
    w, h = 704, 520
    frames = np.stack([L.natural_like(w, h, 80 + i) for i in range(2)])
    ii = np.stack([L.o_integral(O, f) for f in frames])
    os.environ["GS_B200_LBP_BIG"] = big
    try:
        rects, counts = G.lbp_detect_batch(cas, dev(ii.view(np.int32)), 4000, 1.1, 1.0, 4.0, 2)
        got = G.rects_to_numpy(rects, counts)
    finally:
        del os.environ["GS_B200_LBP_BIG"]
    for i in range(2):
        want = L.o_detect(O, cas, ii[i], 4000, 1.1, 1.0, 4.0, 2)
        assert got[i].tobytes() == want.tobytes(), (big, i, len(got[i]), len(want))
        assert len(want) > 3


def test_resize_full_size_ratios(G, O):
    """gs_resize at BASELINE frame sizes through the staged-tile kernel (ratios up to ~2.8:1, up-scaling, ragged targets),
    the 2:1 dispatch to the downsample kernel and the gather kernel (large ratios), whole frames against the oracle"""
    import torch
    rng = np.random.default_rng(19)
    src = rng.integers(0, 256, (2, 2160, 3840)).astype(np.uint8)
    src[1] = L.natural_like(3840, 2160, 4)
    d = dev(src)
    for (dw, dh) in ((2560, 1440), (1920, 1080), (1500, 2000), (4097, 2161), (3837, 797), (960, 2159), (640, 360), (5000, 300)):
        got = G.resize_batch(d, dw, dh).cpu().numpy()
        for i in range(2):
            assert np.array_equal(got[i], L.o_resize(O, src[i], dw, dh)), (dw, dh, i)
