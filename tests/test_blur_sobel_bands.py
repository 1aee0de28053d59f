"""gs_b200_blur_sobel_batch's one-pass kernel with 240-column warps.  Lanes 1..30 of a warp write outputs and lanes 0
and 31 only hand on one blurred pixel each (lane 0 its pixel 7, lane 31 its pixel 0), so CTAs advance 240 columns
and the first CTA's lane 1 sits left of the image at column -8.

The widths 240k + 16m (m = 0..14) put column w-1 in every lane position of the last warp, including lanes 30 and 31;
960k + 240j + 16 leave 1..4 warp-widths of image in the last 960 columns.  The heights put the frame's last rows just
before, on and after the 32-row band and 128-row tile seams, and include frames shorter than 2r+1 rows.  Bit-exact
against the oracle chain gs_blur -> gs_sobel for r = 1..7, with dst pre-filled with random bytes, so the untouched
1-px frame must keep exactly its own values.  The CPU test checks on a model of window_sums that lane 0's pixel 7 and
lane 31's pixel 0 do not depend on the neighbour words those lanes lack."""
import numpy as np
import pytest

import _libs as L


def dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.fixture(scope="module")
def G():
    import torch
    import grayskull_b200 as g
    from grayskull_b200 import api
    assert torch.cuda.is_available()
    g.lib().gs_b200_set_device(0)
    return api


def check_shape(G, O, w, h, seed):
    rng = np.random.default_rng(seed)
    frames = np.stack([rng.integers(0, 256, (h, w)).astype(np.uint8), L.natural_like(w, h, seed % 13)])
    fill = rng.integers(0, 256, frames.shape).astype(np.uint8)
    src = dev(frames)
    for r in range(1, 8):
        got = G.blur_sobel_batch(src, r, out=dev(fill)).cpu().numpy()
        for i in range(len(frames)):
            b = np.empty_like(frames[i])
            O.gso_blur(L.ptr(b), L.ptr(frames[i]), w, h, r)
            want = fill[i].copy()
            O.gso_sobel(L.ptr(want), L.ptr(b), w, h)
            assert np.array_equal(got[i], want), (w, h, r, i)


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 2])
def test_blur_sobel_last_warp_lanes(G, k):
    O = L.oracle()
    for m in range(15):
        check_shape(G, O, 240 * k + 16 * m, 70, 300 * k + m)


@pytest.mark.gpu
@pytest.mark.parametrize("j", [0, 1, 2, 3])
def test_blur_sobel_live_warps_in_last_cta(G, j):
    O = L.oracle()
    for k in (0, 1):
        check_shape(G, O, 960 * k + 240 * j + 16, 45, 400 + 10 * k + j)


@pytest.mark.gpu
@pytest.mark.parametrize("h", [3, 4, 5, 9, 14, 15, 16, 31, 32, 33, 34, 127, 128, 129, 130, 255, 256, 257, 258])
def test_blur_sobel_heights_at_seams(G, h):
    check_shape(G, L.oracle(), 496, h, 500 + h)


def _window_sums(V, R):
    """box.cu window_sums<R> on Python ints, mod 2^32: V = 12 pair words (lo = column 2m, hi = column 2m+1)"""
    M = 0xFFFFFFFF
    odd = R & 1
    NP = R if odd else R + 1
    M0 = (8 - R + 1) // 2 if odd else (8 - R) // 2
    ps = sum(V[M0:M0 + NP]) & M
    T = []
    for p in range(4):
        m = M0 + p
        x16 = ((ps * 0x10001) & M) >> 16
        if odd:
            edge = (V[m - 1] >> 16) | ((V[m + NP] & 0xFFFF) << 16)      # prmt(V[m-1], V[m+NP], 0x5432)
            T.append((x16 * 0x10001 + edge) & M)
        else:
            sub = (V[m + R] >> 16) | ((V[m] & 0xFFFF) << 16)           # prmt(V[m+R], V[m], 0x5432)
            T.append((x16 * 0x10001 - sub) & M)
        if p < 3:
            ps = (ps + V[m + NP] - V[m]) & M
    return T


@pytest.mark.parametrize("R", range(1, 8))
def test_halo_lane_pixels_ignore_missing_words(R):
    """lane 0 has no left neighbour (its V[0..3] are its own column sums) and lane 31 no right one (V[8..11]); the
    pixel each hands on must still be the window sum of the true columns"""
    rng = np.random.default_rng(R)
    top = (2 * R + 1) * 255
    for _ in range(2000):
        s = rng.integers(0, top + 1, 24)                            # true column sums of columns x-8 .. x+15
        true = [int(s[2 * m]) | int(s[2 * m + 1]) << 16 for m in range(12)]
        junk = [int(a) | int(b) << 16 for a, b in rng.integers(0, top + 1, (4, 2))]
        lane0 = _window_sums(junk + true[4:], R)
        assert lane0[3] >> 16 == int(s[15 - R:16 + R].sum()), R    # pixel 7 = column x+7 = index 15
        lane31 = _window_sums(true[:8] + junk, R)
        assert lane31[0] & 0xFFFF == int(s[8 - R:9 + R].sum()), R   # pixel 0 = column x = index 8
