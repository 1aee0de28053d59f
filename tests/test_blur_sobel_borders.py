"""gs_b200_blur_sobel_batch's one-pass kernel at the frame borders.  The kernel picks its row loop per warp (only
bands whose blurred rows have clipped row windows take the clipped loop) and its divisors per lane (the lanes of
columns 0 and w-8 divide by clipped column counts inside the unrolled loop), and the lanes holding columns 0 and
w-1 write seven of their eight bytes so that dst's frame is kept without being read.

The widths 224k + 16m (m = 0..13) put column w-1 in every lane position of the last 224-column tile; the heights
128k + {6, 7, 33, 38, 100, 129} make only the first band, only the last band or a partial band of a tile row-clipped;
16x16 and 48x40 are frames of a single tile.  Bit-exact against the oracle chain gs_blur -> gs_sobel for r = 1..7,
with dst pre-filled with random bytes, so the untouched 1-px frame must keep exactly its own values.  The CPU test
checks the built kernels for global loads: the kernel reads its input through TMA only and never reads dst."""
import os
import re
import shutil
import subprocess

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
            for edge in (np.s_[0], np.s_[-1], np.s_[:, 0], np.s_[:, -1]):
                assert np.array_equal(got[i][edge], fill[i][edge]), (w, h, r, i)


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 2])
def test_blur_sobel_last_lane_positions(G, k):
    O = L.oracle()
    for m in range(14):
        check_shape(G, O, 224 * k + 16 * m, 134, 100 * k + m)


@pytest.mark.gpu
@pytest.mark.parametrize("w", [464, 656])
def test_blur_sobel_row_clipped_bands(G, w):
    O = L.oracle()
    for k in (1, 2):
        for dh in (6, 7, 33, 38, 100, 129):
            check_shape(G, O, w, 128 * k + dh, w + 128 * k + dh)


@pytest.mark.gpu
@pytest.mark.parametrize("w,h", [(16, 16), (48, 40)])
def test_blur_sobel_single_tile(G, w, h):
    check_shape(G, L.oracle(), w, h, w * h)


def _functions(sass):
    """{function name: its SASS} of a cuobjdump -sass listing"""
    parts = re.split(r"^\s*Function : (\S+)\s*$", sass, flags=re.M)
    return dict(zip(parts[1::2], parts[2::2]))


def test_blur_sobel_sass_reads_only_through_tma():
    from grayskull_b200 import _lib
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not found")
    out = subprocess.run([tool, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    fused = {name: body for name, body in _functions(out).items() if "k_blur_sobel_tma" in name}
    assert len(fused) == 7, sorted(fused)                     # r = 1..7
    for name, body in fused.items():
        assert "UTMALDG" in body, name
        assert not re.search(r"\bLDG\b", body), name
