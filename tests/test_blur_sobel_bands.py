"""The constant MMA bands of k_blur_sobel_tma (box.cu), built in closed form from one window mask per register.

For band register j of lane (g, t), row = g + 8 (j & 1) and the window mask M = (2^(2R+1) - 1) << (row + 8 - R) has bit
k' set exactly when |k' - 8 - row| <= R.  Byte i of ah[j] is bit 16 (j >> 1) + 4t + i of M, and byte i of av[j] is bit
16 (j >> 1) + 2t + {0, 1, 8, 9}[i] (the H row of k slot 16 (j >> 1) + 4t + i).  A nibble becomes the low bits of four
bytes by * 0x204081.

CPU: that restatement equals the bands written as the window test of each entry (test_blur_sobel._bands, which the
fragment model there checks against the box sums) for every R and lane."""
import pytest

from test_blur_sobel import _bands


def closed_form_bands(R):
    ah, av = [], []
    for lane in range(32):
        g, t = lane >> 2, lane & 3
        a4, v4 = [], []
        for j in range(4):
            m = ((1 << (2 * R + 1)) - 1) << (g + 8 * (j & 1) + 8 - R)
            assert m < 1 << 32
            mh, mv = m >> (16 * (j >> 1) + 4 * t), m >> (16 * (j >> 1) + 2 * t)
            a4.append((mh & 0xF) * 0x204081 & 0x01010101)
            v4.append(((mv & 0x3) | (mv >> 6 & 0xC)) * 0x204081 & 0x01010101)
        ah.append(a4)
        av.append(v4)
    return ah, av


@pytest.mark.parametrize("R", range(1, 8))
def test_closed_form_bands(R):
    assert closed_form_bands(R) == _bands(R)
