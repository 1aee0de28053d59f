"""gs_b200_blur_sobel_batch's one-pass kernel with its box sums on the tensor cores.  k_blur_sobel_tma<R> forms the
horizontal sums H of 8-row tiles with one mma.m16n8k32.u8 each, splits H = 256 hi + lo, and forms the vertical sums of
16 blurred rows from lo and hi with two more MMAs per 8 columns; the slot order of those MMAs' k dimension follows the
register layout of the first MMA's result and is baked into a constant 0/1 band (box.cu).

On the GPU, bit-exact against the oracle chain gs_blur -> gs_sobel for r = 1..7 with dst pre-filled with random
bytes:
  * frames that reach the largest hi byte (all 255, and 255/0 stripes across and down the frame);
  * frames whose horizontal sums sit on either side of multiples of 256, where a carry lost between lo and hi shows;
  * widths 240k + 16m, which put the right edge in every 16-column strip of the last tile, and heights on either side
    of every 8-row H tile and 16-row step of the last tile (126 sobel rows per tile, blurred rows from y0 - 1).
On the CPU, a numpy model of one step's fragments checks that the band and slot layout give the box sums for every R,
and the built kernels are checked to use IMMA and no I2F."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import _libs as L

TH = 126   # sobel rows per tile


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


def check_frames(G, O, frames, seed, radii=range(1, 8)):
    frames = np.ascontiguousarray(frames, dtype=np.uint8)
    n, h, w = frames.shape
    fill = np.random.default_rng(seed).integers(0, 256, frames.shape).astype(np.uint8)
    src = dev(frames)
    for r in radii:
        got = G.blur_sobel_batch(src, r, out=dev(fill)).cpu().numpy()
        for i in range(n):
            b = np.empty_like(frames[i])
            O.gso_blur(L.ptr(b), L.ptr(frames[i]), w, h, r)
            want = fill[i].copy()
            O.gso_sobel(L.ptr(want), L.ptr(b), w, h)
            assert np.array_equal(got[i], want), (w, h, r, i)


def stripes(w, h, period):
    x = (np.arange(w) // period) % 2
    y = (np.arange(h) // period) % 2
    return [np.full((h, w), 255, np.uint8), np.broadcast_to(255 * x[None, :], (h, w)),
            np.broadcast_to(255 * y[:, None], (h, w)), 255 * (x[None, :] ^ y[:, None])]


@pytest.mark.gpu
@pytest.mark.parametrize("period", [1, 3, 8, 16])
def test_largest_hi_byte(G, period):
    """all 255 gives H = (2R+1) 255 (hi = 14 at R = 7) in every window; stripes give full and empty windows side by
    side, across the 16-column strips and the 8-row tiles"""
    O = L.oracle()
    for w, h in ((256, 140), (496, 263)):
        check_frames(G, O, np.stack(stripes(w, h, period)), w + h + period)


@pytest.mark.gpu
@pytest.mark.parametrize("R", range(1, 8))
def test_sums_around_multiples_of_256(G, R):
    """rows (and columns) of nearly constant value v, with (2R+1) v on either side of 256 k, so that the horizontal
    sums and the window sums cross lo/hi boundaries by one or two"""
    O = L.oracle()
    rng = np.random.default_rng(R)
    n = 2 * R + 1
    levels = sorted({v for k in range(1, 15) for v in (256 * k // n, -(-256 * k // n)) if 0 <= v <= 255})
    w, h = 272, 150
    rows = np.array(levels)[rng.integers(0, len(levels), h)]
    a = np.clip(rows[:, None] + rng.integers(-1, 2, (h, w)), 0, 255)
    cols = np.array(levels)[rng.integers(0, len(levels), w)]
    b = np.clip(cols[None, :] + rng.integers(-1, 2, (h, w)), 0, 255)
    c = np.clip(np.maximum(rows[:, None], cols[None, :]), 0, 255) + np.zeros((h, w), int)
    check_frames(G, O, np.stack([a, b, c]), 7 * R, radii=[R])


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 2])
def test_right_edge_in_every_strip(G, k):
    O = L.oracle()
    for m in range(15):
        w = 240 * k + 16 * m + 16
        rng = np.random.default_rng(900 + 20 * k + m)
        frames = np.stack([rng.integers(0, 256, (40, w)), 255 * (rng.random((40, w)) < 0.5)])
        check_frames(G, O, frames, w)


@pytest.mark.gpu
@pytest.mark.parametrize("j", range(17))
def test_bottom_edge_at_tile_and_step_seams(G, j):
    """the last tile's blurred rows start at y0 - 1 and go in 8-row H tiles and 16-row steps: heights y0 + 8 j - 1
    + {-1, 0, 1} for the last tile's y0 = 126 (and the first tile's for j <= 2)"""
    O = L.oracle()
    for y0 in ((0, TH) if j <= 2 else (TH,)):
        for d in (-1, 0, 1):
            h = y0 + 8 * j - 1 + d
            if h < 3:
                continue
            rng = np.random.default_rng(1000 + h)
            frames = np.stack([rng.integers(0, 256, (h, 256)), 255 * (rng.random((h, 256)) < 0.5)])
            check_frames(G, O, frames, h)


# ---- CPU: the fragment layout of one blur step
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


def _functions(sass):
    parts = re.split(r"^\s*Function : (\S+)\s*$", sass, flags=re.M)
    return dict(zip(parts[1::2], parts[2::2]))


def test_blur_sobel_sass_uses_tensor_cores():
    """the box sums run on IMMA and the division needs no int -> float conversion"""
    from grayskull_b200 import _lib
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not found")
    out = subprocess.run([tool, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    fused = {name: body for name, body in _functions(out).items() if "k_blur_sobel_tma" in name}
    assert len(fused) == 7, sorted(fused)
    for name, body in fused.items():
        assert re.search(r"\bIMMA\b", body), name
        assert not re.search(r"\bI2F\b", body), name
