"""gs_b200_erode_n_batch / gs_b200_dilate_n_batch: `iters` passes of the 3x3 erode / dilate in one call.

The kernels rest on one identity: N passes of the reference's 3x3 op (min / max over the in-image pixels of the
neighbourhood) give the min / max over the in-image pixels of the (2N+1)^2 square, i.e. a clipped row window followed
by a clipped column window.  The CPU tests pin that identity on the oracle (and on the reference build when present)
and check the TMA kernels' SASS; the GPU tests check both dispatch paths bit for bit against iterated gso_morph."""
import os
import re
import subprocess

import numpy as np
import pytest

import _libs as L
from _gpu import G, dev  # noqa: F401

SHAPES = [(1, 1), (7, 1), (1, 7), (2, 2), (5, 3), (17, 9), (33, 40)]   # (w, h)


def o_iter(O, a, dil, iters):
    x = np.ascontiguousarray(a)
    for _ in range(iters):
        d = np.empty_like(x)
        O.gso_morph(L.ptr(d), L.ptr(x), x.shape[1], x.shape[0], dil)
        x = d
    return x


def separable(a, dil, n):
    """clipped row window, then clipped column window"""
    f = np.max if dil else np.min
    h, w = a.shape
    r = np.stack([f(a[:, max(0, x - n):x + n + 1], axis=1) for x in range(w)], axis=1)
    return np.stack([f(r[max(0, y - n):y + n + 1], axis=0) for y in range(h)], axis=0)


def inputs(w, h, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (h, w)).astype(np.uint8),
            (rng.random((h, w)) < 0.3).astype(np.uint8) * 255]


@pytest.mark.parametrize("w,h", SHAPES)
def test_iterated_oracle_is_the_clipped_square(w, h):
    from scipy import ndimage
    O = L.oracle()
    for a in inputs(w, h, w * 100 + h):
        for dil in (0, 1):
            filt = ndimage.maximum_filter if dil else ndimage.minimum_filter
            x = a
            for n in range(1, 13):
                x = o_iter(O, x, dil, 1)
                assert np.array_equal(x, filt(a, size=2 * n + 1, mode="nearest")), (w, h, dil, n)
                assert np.array_equal(x, separable(a, dil, n)), (w, h, dil, n)


@pytest.mark.skipif(not L.have_ref(), reason="reference build (oracle/_ref) not present")
@pytest.mark.parametrize("w,h", SHAPES)
def test_iterated_reference_is_the_clipped_square(w, h):
    R = L.ref()
    for a in inputs(w, h, w * 7 + h):
        for dil, fn in ((0, R.gs_erode), (1, R.gs_dilate)):
            x = a.copy()
            for n in range(1, 13):
                d = np.empty_like(x)
                fn(L.img(d), L.img(x))
                x = d
                assert np.array_equal(x, separable(a, dil, n)), (w, h, dil, n)


def test_morph_tma_sass():
    k = {name: body for name, body in L.sass_functions().items() if "k_morph_tma" in name}
    assert len(k) == 30, sorted(k)                            # N = 2..16, erode and dilate
    for name, body in k.items():
        assert "UTMALDG" in body and "VIMNMX3.U16x2" in body, name
        assert not re.search(r"\bLDG\b", body), name


# ---- GPU -----------------------------------------------------------------------------------------------------------
def run(G, frames, dil, iters, offset=0):
    """frames (n, h, w) through the new entry, dst pre-filled with random bytes; `offset` shifts both bases"""
    import torch
    n, h, w = frames.shape
    size = n * h * w
    rng = np.random.default_rng(iters + w + h)
    sbuf = torch.zeros(size + 16, dtype=torch.uint8, device="cuda")
    dbuf = dev(rng.integers(0, 256, size + 16).astype(np.uint8))
    sbuf[offset:offset + size] = dev(frames.reshape(-1))
    src, out = sbuf[offset:offset + size].view(n, h, w), dbuf[offset:offset + size].view(n, h, w)
    (G.dilate_n_batch if dil else G.erode_n_batch)(src, iters, out=out)
    return out.cpu().numpy()


def check(G, O, w, h, iters_list, offset=0, seed=0):
    rng = np.random.default_rng(seed + w * 1000 + h)
    frames = np.stack([rng.integers(0, 256, (h, w)).astype(np.uint8), L.natural_like(w, h, seed % 17),
                       (rng.random((h, w)) < 0.5).astype(np.uint8) * 255])
    O = L.oracle()
    for dil in (0, 1):
        want, x, done = {}, list(frames), 0          # iterate the oracle once, keeping the counts asked for
        for iters in sorted(set(min(n, max(w, h)) for n in iters_list)):
            x = [o_iter(O, a, dil, iters - done) for a in x]
            done, want[iters] = iters, x
        for iters in iters_list:
            got = run(G, frames, dil, iters, offset)
            for i in range(3):
                assert np.array_equal(got[i], want[min(iters, max(w, h))][i]), (w, h, dil, iters, offset, i)


NS = [0, 1, 2, 3, 4, 5, 7, 8, 9, 10, 15, 16, 17, 31, 100]
A_W = [16, 32, 240, 256, 272, 528, 1920]
B_W = [1, 2, 3, 15, 17, 100, 612]
HS = [1, 2, 3, 5, 16, 17, 31, 33, 127, 128, 129, 161, 300]


def combos(widths):
    """every width, height and N at least once, without the full product"""
    out = []
    for i in range(max(len(widths), len(HS))):
        w, h = widths[i % len(widths)], HS[(3 * i) % len(HS)]
        out.append((w, h, [NS[(i + j) % len(NS)] for j in range(0, len(NS), 3)]))
    covered = {n for _, _, ns in out for n in ns}
    assert covered == set(NS) and {h for _, h, _ in out} == set(HS)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,ns", combos(A_W))
def test_path_a_shapes(G, w, h, ns):
    check(G, L.oracle(), w, h, ns)


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,ns", combos(B_W))
def test_path_b_shapes(G, w, h, ns):
    check(G, L.oracle(), w, h, ns)


@pytest.mark.gpu
@pytest.mark.parametrize("w,h", [(256, 129), (528, 33), (1920, 17)])
def test_path_b_on_tma_shapes(G, w, h):
    import grayskull_b200 as g
    O = L.oracle()
    check(G, O, w, h, [2, 9, 16], offset=1)
    g.lib().gs_b200_force_generic(1)
    try:
        check(G, O, w, h, [2, 3, 9, 16])
    finally:
        g.lib().gs_b200_force_generic(0)


@pytest.mark.gpu
@pytest.mark.parametrize("w,h", [(256, 129), (272, 300), (32, 161)])
def test_composed_tma_passes(G, w, h):
    """17 <= N <= 48 on TMA geometry: TMA passes of at most 16 composed through the workspace, remainders 0, 1 and
    2..15 included; 49 is the first count past them"""
    check(G, L.oracle(), w, h, [17, 18, 31, 32, 33, 47, 48, 49])


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,offset", [(272, 161, 0), (100, 161, 0), (272, 161, 1)])
def test_frames_stay_isolated(G, w, h, offset):
    rng = np.random.default_rng(w + h)
    frames = np.stack([np.zeros((h, w), np.uint8), np.full((h, w), 255, np.uint8),
                       rng.integers(0, 256, (h, w)).astype(np.uint8)])
    O = L.oracle()
    for dil in (0, 1):
        for iters in (2, 9, 16, 17, 33, 100):
            got = run(G, frames, dil, iters, offset)
            assert (got[0] == 0).all() and (got[1] == 255).all(), (dil, iters)
            assert np.array_equal(got[2], o_iter(O, frames[2], dil, min(iters, max(w, h)))), (dil, iters)


@pytest.mark.gpu
@pytest.mark.parametrize("w,h", [(16, 5), (256, 300), (17, 31), (612, 2), (1, 129)])
def test_saturation(G, w, h):
    rng = np.random.default_rng(w * h)
    frames = rng.integers(0, 256, (3, h, w)).astype(np.uint8)
    O = L.oracle()
    for iters in (w, h, max(w, h) + 5, 2 ** 31, 2 ** 32 - 1):
        for dil in (0, 1):
            got = run(G, frames, dil, iters)
            for i in range(3):
                if iters >= max(w, h) - 1:          # the square covers the frame from every pixel
                    v = frames[i].max() if dil else frames[i].min()
                    assert (got[i] == v).all(), (w, h, iters, dil, i)
                else:
                    assert np.array_equal(got[i], o_iter(O, frames[i], dil, iters)), (w, h, iters, dil, i)


@pytest.mark.gpu
def test_launch_count(G):
    import torch
    import grayskull_b200 as g
    lib = g.lib()
    for (w, h, off), per in (((256, 64, 0), {1: 1, 2: 1, 9: 1, 16: 1, 17: 2, 31: 2, 33: 3, 48: 3, 49: 2, 1000: 2}),
                             ((100, 64, 0), {1: 1, 2: 2, 16: 2, 1000: 2}),
                             ((256, 64, 1), {1: 1, 2: 2, 5: 2})):
        for n in (1, 3):
            buf = torch.zeros(n * h * w + 1, dtype=torch.uint8, device="cuda")
            src = buf[off:off + n * h * w].view(n, h, w)
            out = torch.empty_like(src)
            for iters, want in per.items():
                for fn in (G.erode_n_batch, G.dilate_n_batch):
                    before = lib.gs_b200_launch_count()
                    fn(src, iters, out=out)
                    assert lib.gs_b200_launch_count() - before == want, (w, h, off, n, iters)
    torch.cuda.synchronize()


def _cli(tmp_path, chain, frames):
    from grayskull_b200 import _lib
    exe = os.path.join(os.path.dirname(_lib.LIB_PATH), "gsb_magick")
    h, w = frames[0].shape
    paths = []
    for f, a in enumerate(frames):
        p = tmp_path / ("in%d.pgm" % f)
        p.write_bytes(b"P5\n%d %d\n255\n" % (w, h) + a.tobytes())
        paths.append(str(p))
    r = subprocess.run([exe, chain, str(tmp_path / "o_")] + paths, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    outs = []
    for f in range(len(frames)):
        b = (tmp_path / ("o_%04d.pgm" % f)).read_bytes().split(b"\n", 3)
        outs.append(np.frombuffer(b[3], np.uint8).reshape(h, w))
    return r.stdout, outs


@pytest.mark.gpu
def test_cli_aruco_chain(G, tmp_path):
    O = L.oracle()
    w, h = 640, 480
    frames = [L.natural_like(w, h, 40 + f) for f in range(3)]
    stdout, outs = _cli(tmp_path, "blur:3,sobel,threshold:otsu,dilate:9,erode:10,blobs:150", frames)
    lines = [ln for ln in stdout.splitlines() if "blobs" in ln]
    assert len(lines) == 3
    for f, a in enumerate(frames):
        x = np.empty_like(a); O.gso_blur(L.ptr(x), L.ptr(a), w, h, 3)
        s = np.zeros_like(a); O.gso_sobel(L.ptr(s), L.ptr(x), w, h)
        t = O.gso_otsu_threshold(L.ptr(s), w, h)
        O.gso_threshold(L.ptr(s), w, h, t)
        x = o_iter(O, o_iter(O, s, 1, 9), 0, 10)
        assert np.array_equal(outs[f], x), f
        labels = np.zeros((h, w), np.uint16)
        blobs = np.zeros(150, L.BLOB_DTYPE)
        nb = O.gso_blobs(L.ptr(x), w, h, L.ptr(labels), L.ptr(blobs), 150)
        assert lines[f] == "frame %d: %d blobs" % (f, nb), (lines[f], nb)


@pytest.mark.gpu
def test_cli_open_close(G, tmp_path):
    O = L.oracle()
    w, h = 612, 816
    frames = [L.binary_like(w, h, 7 + f) for f in range(2)]
    _, outs = _cli(tmp_path, "dilate:5,erode:5", frames)
    for f, a in enumerate(frames):
        assert np.array_equal(outs[f], o_iter(O, o_iter(O, a, 1, 5), 0, 5)), f


@pytest.mark.gpu
def test_iters_out_of_range_raises(G):
    src = dev(np.zeros((1, 4, 16), np.uint8))
    for fn in (G.erode_n_batch, G.dilate_n_batch):
        for bad in (-1, 2 ** 32):
            with pytest.raises(ValueError):
                fn(src, bad)
