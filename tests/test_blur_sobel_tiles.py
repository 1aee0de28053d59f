"""k_blur_sobel_tma's tile geometry (box.cu): 256 sobel columns x 110 rows per CTA.

A tile's sobel columns are [256 bx, 256 bx + 256), all 32 lanes of a warp row.  Its blurred columns come from 17
16-column strips: warp w walks strips w and w + 8 down the tile's 7 16-row steps, and warps 0..6 make one step each
of strip 16, the strip that holds the tile's right halo.  A strip with a clipped window anywhere takes the per-pixel
count table, so strip 16 is the only clipped strip of a tile whose right neighbour is past the image's last column.

GPU: each shape runs for every r into dst pre-filled with random bytes and must equal the oracle's gso_blur ->
gso_sobel (test_blur_sobel.check):
  * widths 256k + 16m and 256k + 16m + 16, 240 rows: the right edge at the end of every strip of the last tile,
    strip 16 included, on tile rows with clipped (first, last) and full (middle) windows;
  * heights y0 + 8j - 1 + {-1, 0, 1}, y0 = 110 (and 0 for j <= 2): the last tile's bottom edge on either side of
    every 8-row H tile and 16-row step, and heights 110 j + {-1, 0, 1}: one row short of, on and one row past the
    tile seams;
  * 4096 x 240: c2's width, 16 tiles per row, the last of them with only strip 16 clipped;
  * widths 256k x 330 rows: tiles of the middle row whose only clipped strip is strip 16;
  * 16 x 16 and 256 x 110: a single tile."""
import numpy as np
import pytest

from _gpu import G, O  # noqa: F401
from test_blur_sobel import check, check_shape

TW, TH = 256, 110   # sobel columns and rows per tile


def pair(w, h, seed):
    """a random and a 0/255 frame of w x h"""
    rng = np.random.default_rng(seed)
    return np.stack([rng.integers(0, 256, (h, w)), 255 * (rng.random((h, w)) < 0.5)])


@pytest.mark.gpu
@pytest.mark.parametrize("k", range(4))
def test_right_edge_in_every_strip(G, O, k):
    for m in range(16):
        for w in (TW * k + 16 * m, TW * k + 16 * m + 16):
            if w >= 16:
                check(G, O, pair(w, 240, 3000 + w), w)


@pytest.mark.gpu
@pytest.mark.parametrize("j", range(15))
def test_bottom_edge_at_step_seams(G, O, j):
    for y0 in ((0, TH) if j <= 2 else (TH,)):
        for d in (-1, 0, 1):
            h = y0 + 8 * j - 1 + d
            if h >= 3:
                check(G, O, pair(512, h, 4000 + h), h)


@pytest.mark.gpu
@pytest.mark.parametrize("j", [1, 2, 3])
def test_heights_at_tile_seams(G, O, j):
    for d in (-1, 0, 1):
        check_shape(G, O, 528, TH * j + d, 5000 + TH * j + d)


@pytest.mark.gpu
def test_c2_width(G, O):
    check(G, O, pair(4096, 240, 6000), 6001)


@pytest.mark.gpu
@pytest.mark.parametrize("k", [2, 3, 5])
def test_only_strip_16_clipped(G, O, k):
    check_shape(G, O, TW * k, 3 * TH, 7000 + k)


@pytest.mark.gpu
@pytest.mark.parametrize("w,h", [(16, 16), (TW, TH)])
def test_single_tile(G, O, w, h):
    check_shape(G, O, w, h, 8000 + w * h)
