"""gs_b200_blur_sobel_batch == gs_blur -> gs_sobel bit for bit, and its one-pass kernel k_blur_sobel_tma<R> (box.cu).

For r = 1..7, w % 16 == 0 and 16-byte aligned bases, a CTA makes 240 sobel columns x 126 sobel rows in two phases:
  A. blur on the tensor cores.  One TMA box loads input columns [xb, xb + 272) and rows [Y - 8, Y + 136), Y = y0 - 1
     the tile's first blurred row.  The warps walk 16-column strips (blurred columns [xb + 8, xb + 264)) down the tile
     in 16-row steps: the horizontal sums H of 8-row tiles with one mma.m16n8k32.u8 each, H = 256 hi + lo, and the
     vertical sums of 16 blurred rows with two more MMAs per 8 columns, whose k slot order follows the register layout
     of the first MMA's result and is baked into a constant 0/1 band.  The lo MMA accumulates onto 0x4B000000, so
     IMAD(hi, 256, lo) is the float 2^23 + S, divided exactly on the FMA pipe.
  B. sobel from the blurred tile: 8 warps of one 16-row band each (the last one 14 rows).  The lanes holding column 0
     or w-1 write seven of their eight bytes, so dst's 1-px frame is kept without being read.
Other radii and geometries run the two per-op kernels through a scratch batch.

GPU: each shape runs for every r into dst pre-filled with random bytes and must equal the oracle's gso_blur ->
gso_sobel, whose expected array keeps the fill in the 1-px frame.  The shape families and what they reach:
  * all 255 and 255/0 stripes: the largest hi byte; near-constant rows or columns whose sums sit on either side of
    multiples of 256: a carry lost between lo and hi;
  * widths 240k + 16m + 16 (40 rows) and 240k + 16m (70 rows): the right edge at the end of every 16-column strip of
    the last tile, and on a tile seam; the second family is kept from the SIMD form's 240-column warps;
  * widths 960k + 240j + 16: 0-7 whole tiles and a last tile of one strip (kept from the SIMD form's 960-column CTAs);
  * widths 224k + 16m (134 rows, 8 rows into the second tile row): right edges at strip ends, kept from 224-column
    tiles;
  * heights y0 + 8j - 1 + {-1, 0, 1}, y0 = 126 (and 0 for j <= 2): the last tile's bottom edge on either side of every
    8-row H tile and 16-row step;
  * heights 3-258 (496 wide): shorter than 2r + 1 rows, around the 16-row steps and 1-6 rows past the tile seams at 126
    and 252, kept from 32-row bands and 128-row tiles; heights 128k + {6, 7, 33, 38, 100, 129} (464 and 656 wide) and
    31-300 (480 and 1024 wide), kept from the 128-row tiles and 32-row bands of earlier forms;
  * 16 x 16 and 48 x 40: a single tile;
  * c5's 16 frames of 1920 x 1080, against the two-kernel chain on the device.
CPU: a numpy model of one step's fragments gives the box sums for every R; the seven kernels' SASS uses IMMA and no
I2F, and reads its input through TMA only (no LDG)."""
import re

import numpy as np
import pytest

import _libs as L
from _gpu import G, O, dev  # noqa: F401

TH = 126   # sobel rows per tile


def check(G, O, frames, seed, radii=range(1, 8)):
    """frames (n, h, w) through blur_sobel_batch into dst pre-filled with random bytes: bit-exact against the oracle
    chain for each r, the untouched 1-px frame included"""
    frames = np.ascontiguousarray(frames, dtype=np.uint8)
    fill = np.random.default_rng(seed).integers(0, 256, frames.shape).astype(np.uint8)
    src = dev(frames)
    for r in radii:
        got = G.blur_sobel_batch(src, r, out=dev(fill)).cpu().numpy()
        for i in range(len(frames)):
            want = L.o_sobel(O, L.o_blur(O, frames[i], r), fill[i])
            assert np.array_equal(got[i], want), (frames.shape, r, i)


def check_shape(G, O, w, h, seed):
    """a random and a natural_like frame of w x h"""
    rng = np.random.default_rng(seed)
    check(G, O, [rng.integers(0, 256, (h, w)), L.natural_like(w, h, seed % 13)], seed + 1)


def stripes(w, h, period):
    x = (np.arange(w) // period) % 2
    y = (np.arange(h) // period) % 2
    return [np.full((h, w), 255, np.uint8), np.broadcast_to(255 * x[None, :], (h, w)),
            np.broadcast_to(255 * y[:, None], (h, w)), 255 * (x[None, :] ^ y[:, None])]


@pytest.mark.gpu
@pytest.mark.parametrize("period", [1, 3, 8, 16])
def test_largest_hi_byte(G, O, period):
    """all 255 gives H = (2R+1) 255 (hi = 14 at R = 7) in every window; stripes give full and empty windows side by
    side, across the 16-column strips and the 8-row tiles"""
    for w, h in ((256, 140), (496, 263)):
        check(G, O, np.stack(stripes(w, h, period)), w + h + period)


@pytest.mark.gpu
@pytest.mark.parametrize("R", range(1, 8))
def test_sums_around_multiples_of_256(G, O, R):
    """rows (and columns) of nearly constant value v, with (2R+1) v on either side of 256 k, so that the horizontal
    sums and the window sums cross lo/hi boundaries by one or two"""
    rng = np.random.default_rng(R)
    n = 2 * R + 1
    levels = sorted({v for k in range(1, 15) for v in (256 * k // n, -(-256 * k // n)) if 0 <= v <= 255})
    w, h = 272, 150
    rows = np.array(levels)[rng.integers(0, len(levels), h)]
    a = np.clip(rows[:, None] + rng.integers(-1, 2, (h, w)), 0, 255)
    cols = np.array(levels)[rng.integers(0, len(levels), w)]
    b = np.clip(cols[None, :] + rng.integers(-1, 2, (h, w)), 0, 255)
    c = np.clip(np.maximum(rows[:, None], cols[None, :]), 0, 255) + np.zeros((h, w), int)
    check(G, O, np.stack([a, b, c]), 7 * R, radii=[R])


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 2])
def test_right_edge_in_every_strip(G, O, k):
    for m in range(15):
        w = 240 * k + 16 * m + 16
        rng = np.random.default_rng(900 + 20 * k + m)
        check(G, O, np.stack([rng.integers(0, 256, (40, w)), 255 * (rng.random((40, w)) < 0.5)]), w)


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 2])
def test_blur_sobel_widths_240k_16m(G, O, k):
    for m in range(15):
        check_shape(G, O, 240 * k + 16 * m, 70, 300 * k + m)


@pytest.mark.gpu
@pytest.mark.parametrize("j", [0, 1, 2, 3])
def test_blur_sobel_widths_960k_240j_16(G, O, j):
    for k in (0, 1):
        check_shape(G, O, 960 * k + 240 * j + 16, 45, 400 + 10 * k + j)


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 2])
def test_blur_sobel_widths_224k_16m(G, O, k):
    for m in range(14):
        check_shape(G, O, 224 * k + 16 * m, 134, 100 * k + m)


@pytest.mark.gpu
@pytest.mark.parametrize("j", range(17))
def test_bottom_edge_at_tile_and_step_seams(G, O, j):
    """the last tile's blurred rows start at y0 - 1 and go in 8-row H tiles and 16-row steps: heights y0 + 8 j - 1
    + {-1, 0, 1} for the last tile's y0 = 126 (and the first tile's for j <= 2)"""
    for y0 in ((0, TH) if j <= 2 else (TH,)):
        for d in (-1, 0, 1):
            h = y0 + 8 * j - 1 + d
            if h < 3:
                continue
            rng = np.random.default_rng(1000 + h)
            check(G, O, np.stack([rng.integers(0, 256, (h, 256)), 255 * (rng.random((h, 256)) < 0.5)]), h)


@pytest.mark.gpu
@pytest.mark.parametrize("h", [3, 4, 5, 9, 14, 15, 16, 31, 32, 33, 34, 127, 128, 129, 130, 255, 256, 257, 258])
def test_blur_sobel_heights_at_seams(G, O, h):
    check_shape(G, O, 496, h, 500 + h)


@pytest.mark.gpu
@pytest.mark.parametrize("w", [464, 656])
def test_blur_sobel_heights_128k_plus(G, O, w):
    for k in (1, 2):
        for dh in (6, 7, 33, 38, 100, 129):
            check_shape(G, O, w, 128 * k + dh, w + 128 * k + dh)


@pytest.mark.gpu
def test_blur_sobel_heights_around_32k(G, O):
    for w in (480, 1024):
        for h in (31, 32, 33, 34, 35, 45, 67, 68, 129, 130, 131, 280, 300):
            check_shape(G, O, w, h, w + h)


@pytest.mark.gpu
@pytest.mark.parametrize("w,h", [(16, 16), (48, 40)])
def test_blur_sobel_single_tile(G, O, w, h):
    check_shape(G, O, w, h, w * h)


@pytest.mark.gpu
def test_blur_sobel_c5_shape_vs_two_kernels(G):
    import torch
    torch.manual_seed(8)
    src = torch.randint(0, 256, (16, 1080, 1920), dtype=torch.uint8, device="cuda")
    for r in range(1, 8):
        got = G.blur_sobel_batch(src, r, out=torch.full_like(src, 77))
        want = G.sobel_batch(G.blur_batch(src, r))
        assert bool((got[:, 1:-1, 1:-1] == want[:, 1:-1, 1:-1]).all()), r
        for edge in (got[:, 0], got[:, -1], got[:, :, 0], got[:, :, -1]):
            assert bool((edge == 77).all()), r


# ---- CPU: the fragment layout of one blur step, and the SASS
def _frag_matrix(regs, rows=16, cols=32):
    """A operand (16 x 32 u8, row-major fragments) from the per-thread registers regs[lane][j]"""
    A = np.zeros((rows, cols), np.int64)
    for lane in range(32):
        g, t = lane >> 2, lane & 3
        for j in range(4):
            for i in range(4):
                A[g + 8 * (j & 1), 16 * (j >> 1) + 4 * t + i] = (regs[lane][j] >> (8 * i)) & 0xFF
    return A


def _bands(R):
    """ah / av as k_blur_sobel_tma builds them, per lane"""
    ah, av = [], []
    for lane in range(32):
        g, t = lane >> 2, lane & 3
        a4, v4 = [], []
        for j in range(4):
            row, kb = g + 8 * (j & 1), 16 * (j >> 1) + 4 * t
            a = v = 0
            for i in range(4):
                k = kb + i
                hrow = (k >> 4) * 16 + ((k >> 1) & 1) * 8 + 2 * ((k >> 2) & 3) + (k & 1)
                a |= int(abs(k - 8 - row) <= R) << (8 * i)
                v |= int(abs(hrow - 8 - row) <= R) << (8 * i)
            a4.append(a)
            v4.append(v)
        ah.append(a4)
        av.append(v4)
    return ah, av


def _prmt(a, b, sel):
    src = [(a >> (8 * i)) & 0xFF for i in range(4)] + [(b >> (8 * i)) & 0xFF for i in range(4)]
    return sum(src[(sel >> (4 * i)) & 7] << (8 * i) for i in range(4))


@pytest.mark.parametrize("R", range(1, 8))
def test_step_fragments_give_box_sums(R):
    """one 16-row step of one strip, lane by lane: horizontal MMA per 8-row tile, the PRMT split into lo / hi operand
    registers, the vertical MMAs with C = 0x4B000000 for lo, and IMAD(hi, 256, lo) = 0x4B000000 + the window sum"""
    rng = np.random.default_rng(R)
    ah, av = _bands(R)
    Ah, Av = _frag_matrix(ah), _frag_matrix(av)
    for img in (rng.integers(0, 256, (32, 32)), np.full((32, 32), 255), 255 * (rng.random((32, 32)) < 0.5)):
        # input rows 0..31 = H rows of pairs u and u+1 (blurred row y of the step = H row y + 8); input columns
        # 0..31 = c0 - 8 .. c0 + 23
        D = []                                                  # D[tile][lane] = 4 s32 results
        for tile in range(4):
            rows = img[8 * tile:8 * tile + 8]                   # N index = row within the tile
            Ht = Ah @ rows.T                                    # 16 output columns x 8 rows
            D.append([[Ht[g, 2 * t], Ht[g, 2 * t + 1], Ht[g + 8, 2 * t], Ht[g + 8, 2 * t + 1]]
                      for g, t in ((lane >> 2, lane & 3) for lane in range(32))])
            assert Ht.max() <= (2 * R + 1) * 255
        ops = []                                                # per pair, per lane: lo0, hi0, lo1, hi1
        for p in range(2):
            P, Q = D[2 * p], D[2 * p + 1]
            per = []
            for lane in range(32):
                o = []
                for hh in range(2):
                    x = _prmt(int(P[lane][2 * hh]), int(P[lane][2 * hh + 1]), 0x5140)
                    y = _prmt(int(Q[lane][2 * hh]), int(Q[lane][2 * hh + 1]), 0x5140)
                    o += [_prmt(x, y, 0x5410), _prmt(x, y, 0x7632)]
                per.append(o)
            ops.append(per)
        for hh in range(2):
            S = {}
            for part in (0, 1):                                 # lo, hi
                B = np.zeros((32, 8), np.int64)                 # k slot x column
                for lane in range(32):
                    g, t = lane >> 2, lane & 3
                    for i in range(4):
                        B[4 * t + i, g] = (ops[0][lane][2 * hh + part] >> (8 * i)) & 0xFF
                        B[16 + 4 * t + i, g] = (ops[1][lane][2 * hh + part] >> (8 * i)) & 0xFF
                S[part] = Av @ B + (0x4B000000 if part == 0 else 0)
            got = (S[1] * 256 + S[0]) & 0xFFFFFFFF
            for y in range(16):
                for n in range(8):
                    col = 8 * hh + n + 8                        # input column of the output column
                    want = img[y + 8 - R:y + 9 + R, col - R:col + R + 1].sum()
                    assert got[y, n] == 0x4B000000 + want, (R, y, n)


def _one_pass_sass():
    fused = {name: body for name, body in L.sass_functions().items() if "k_blur_sobel_tma" in name}
    assert len(fused) == 7, sorted(fused)                     # r = 1..7
    return fused


def test_blur_sobel_sass_uses_tensor_cores():
    """the box sums run on IMMA and the division needs no int -> float conversion"""
    for name, body in _one_pass_sass().items():
        assert re.search(r"\bIMMA\b", body), name
        assert not re.search(r"\bI2F\b", body), name


def test_blur_sobel_sass_reads_only_through_tma():
    """the input comes through TMA only, and dst is never read"""
    for name, body in _one_pass_sass().items():
        assert "UTMALDG" in body, name
        assert not re.search(r"\bLDG\b", body), name
