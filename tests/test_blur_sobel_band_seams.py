"""k_blur_sobel_tma's phase-B bands (box.cu): the 110 sobel rows of a tile are split over all 8 warps, 14 rows on warps
0..5 and 13 on warps 6 and 7, so bands start at tile rows 0, 14, 28, 42, 56, 70, 84 and 97.  A band that ends on or
past the image's last sobel row h - 2 takes the clipped walk, and one that starts past it writes nothing.

GPU: for every band seam s, frames whose last sobel row is tile row s - 1, s or s + 1 (the band before the seam ends
there, the band after it has one row, or two rows), in the first tile row (whose band 0 also holds image row 0) and in
the second.  768 columns: the middle tile has no lane on column 0 or w - 1, so it runs the unrolled walk without the
edge stores, and the outer tiles run it with them.  Each shape is bit-exact against the oracle's gso_blur -> gso_sobel
for every r (test_blur_sobel.check)."""
import pytest

from _gpu import G, O  # noqa: F401
from test_blur_sobel import check_shape

TH = 110                                  # sobel rows per tile
SEAMS = [14, 28, 42, 56, 70, 84, 97]      # tile rows where a warp's band starts after another's


@pytest.mark.gpu
@pytest.mark.parametrize("s", SEAMS)
def test_last_row_at_band_seams(G, O, s):
    for y0 in (0, TH):
        for d in (-1, 0, 1):
            h = y0 + s + d + 2            # last sobel row y0 + s + d
            check_shape(G, O, 768, h, 9000 + h)
