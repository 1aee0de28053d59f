"""gs_perspective_correct and gs_blob_corners at large coordinates, against plain numpy models of the reference.

k_perspective (gs_perspective_correct) clamps its source point to (float)sw - 1.0f and (float)sh - 1.0f.  For about
half of all sizes above 2^24 that value rounds past sw - 1, so the first tap can lie one or more pixels past the row;
the reference samples through gs_get, which gives 0 there.  k_blob_corners (gs_blob_corners) keeps each corner as the
minimum of a 64-bit key (value, raster index), the value being x + y, y - x, -(x + y) or x - y; its half of the key has
to keep the order of every int the reference reaches, down to -(2^31 - 1) for pixels with x + y < 2^31.

  * models: model_perspective evaluates reference grayskull.h:423-444 in numpy float32, one IEEE operation at a time in
    the reference's order, gs_get's 0 outside the image included; model_blob_corners is the loop of :404-421 over the
    box, with its 32-bit loop bounds, its strict comparisons and its starting values INT_MAX / INT_MIN.  Neither shares
    code with the C oracle or the kernels.
  * CPU: the models against the reference build (oracle/_ref, when present) and the C oracle on the round-2 goldens,
    random, degenerate, mirrored and crossed quads, sources of 2^24 + 1 ... 2^24 + 7 pixels with quads past their edge,
    hand-built blob records (boxes outside the frame, empty, wrapping past 2^32, a wrong label, ties) and frames of
    2^31 pixels at x + y = INT_MAX.  A table of (float)s - 1.0f around every power of two from 2^12 to 2^31 picks the
    GPU sources.
  * GPU: every output byte against the models from a poisoned dst, with k_perspective / k_blob_corners witnessed.
    Each source sits in an allocation with a nonzero guard after its last frame, as long as any tap a kernel without
    the zero taps could take, so such a tap fails a byte comparison instead of reading outside the allocation.
Measured on one H100 80GB (700 W power limit), torch's peak device allocation and wall time per case:
  2^29 + 3 frames of 2 x 1 -> 2 x 2, per-frame corners       20.9 GB, 7 s
  a row of 2^31 + 384 pixels, 3 frames, 4.3 GB guard          11.8 GB, under 1 s (a column: 7.5 GB)
  blob corners on a row or a column of 2^31 pixels            6.4 GB, under 1 s
  dw = 2^24 + 5, dh = 1 / 2                                   under 1 GB, 19 s / 37 s, mostly the model on the host
The file's GPU tests take 86 to 109 s in all.
"""
import time

import numpy as np
import pytest

import _calls as calls
import _libs as L
from _gpu import G, O, Region, lib, stream, traced, witness, witnessed  # noqa: F401

F32 = np.float32
M32 = 0xFFFFFFFF
INT_MAX, INT_MIN = 2 ** 31 - 1, -2 ** 31
POISON = calls.POISON
SENTINEL = 0xC5             # the guard after a source: nonzero, so a tap read there is never the reference's 0
LABEL_SENTINEL = 0x5A5A
PAT = np.random.default_rng(251).integers(1, 256, 251, dtype=np.uint8)     # periodic content: no zero byte
CHUNK = 1 << 22
needs_ref = pytest.mark.skipif(not L.have_ref(), reason="oracle/_ref not built")
LIBS = [pytest.param("oracle"), pytest.param("reference", marks=needs_ref)]


# ---- the models ------------------------------------------------------------------------------------------------------
def gs_get(src, x, y):
    """reference grayskull.h:143-145 as float32: the pixel, or 0 outside the image"""
    sh, sw = src.shape
    inside = (x < sw) & (y < sh)
    v = src.take(np.where(inside, y * sw + x, 0))
    return np.where(inside, v, 0).astype(F32)


def model_perspective(dst_w, dst_h, src, quad):
    """gs_perspective_correct (reference grayskull.h:423-444) of one frame -> (dst_h, dst_w) uint8.  src: an (h, w)
    uint8 array, or an object with .shape and .take(flat indices); quad: 4 unsigned points tl, tr, br, bl."""
    sh, sw = src.shape
    c = np.asarray(quad, np.uint32).reshape(4, 2).astype(F32)           # (float) of an unsigned: round to nearest
    out = np.empty(dst_w * dst_h, np.uint8)
    with np.errstate(invalid="ignore", divide="ignore"):
        w, h = F32(dst_w) - F32(1), F32(dst_h) - F32(1)                  # 0: x / w is NaN for dst_w == 1
        mx, my = F32(sw) - F32(1), F32(sh) - F32(1)                      # may round past sw - 1 above 2^24
        for k0 in range(0, out.size, CHUNK):
            k = np.arange(k0, min(k0 + CHUNK, out.size), dtype=np.int64)
            u, v = (k % dst_w).astype(F32) / w, (k // dst_w).astype(F32) / h
            omu, omv = F32(1) - u, F32(1) - v
            top_x = c[0, 0] * omu + c[1, 0] * u
            top_y = c[0, 1] * omu + c[1, 1] * u
            bot_x = c[3, 0] * omu + c[2, 0] * u
            bot_y = c[3, 1] * omu + c[2, 1] * u
            src_x = top_x * omv + bot_x * v
            src_y = top_y * omv + bot_y * v
            src_x = np.where(src_x < mx, src_x, mx)                      # GS_MIN(src_x, src.w - 1.0f): NaN -> mx
            src_y = np.where(src_y < my, src_y, my)
            src_x = np.where(F32(0) > src_x, F32(0), src_x)              # GS_MAX(0.0f, .)
            src_y = np.where(F32(0) > src_y, F32(0), src_y)
            sx, sy = src_x.astype(np.int64), src_y.astype(np.int64)      # (unsigned): truncation of values >= 0
            sx1, sy1 = np.minimum(sx + 1, sw - 1), np.minimum(sy + 1, sh - 1)
            dx, dy = src_x - sx.astype(F32), src_y - sy.astype(F32)
            omx, omy = F32(1) - dx, F32(1) - dy
            acc = gs_get(src, sx, sy) * omx * omy
            acc = acc + gs_get(src, sx1, sy) * dx * omy
            acc = acc + gs_get(src, sx, sy1) * omx * dy
            acc = acc + gs_get(src, sx1, sy1) * dx * dy
            assert acc.dtype == F32 and not (acc >= 256).any()
            out[k0:k0 + k.size] = acc.astype(np.int64)                   # (uint8_t): truncation
    return out.reshape(dst_h, dst_w)


def model_blob_corners(img, labels, w, h, blob):
    """gs_blob_corners (reference grayskull.h:404-421) -> (4, 2) uint32 corners tl, tr, br, bl.  img / labels: the
    frame's w * h pixels / labels in any shape; blob: a BLOB_DTYPE record.  Defined while every pixel it takes has
    x + y < 2^31, where the reference's int arithmetic does not overflow."""
    img, labels = np.asarray(img).reshape(-1), np.asarray(labels).reshape(-1)
    bx, by, bw, bh = (int(blob[k]) for k in ("bx", "by", "bw", "bh"))
    out = np.array([[int(blob["cx"]), int(blob["cy"])]] * 4, np.uint32)      # every corner starts at the centroid
    # x from box.x while x < box.x + box.w, the bound a 32-bit sum (y likewise): a box whose end wraps visits nothing.
    # gs_get reads 0 outside the frame, which the < 128 test skips, so only the box's part inside the frame counts.
    xs = np.arange(bx, min((bx + bw) & M32, w), dtype=np.int64)
    ys = np.arange(by, min((by + bh) & M32, h), dtype=np.int64)
    y, x = (a.ravel() for a in np.meshgrid(ys, xs, indexing="ij"))           # raster order
    p = y * w + x
    keep = img[p] >= 128
    keep[keep] = labels[p[keep]] == int(blob["label"])
    x, y = x[keep], y[keep]
    s, d = x + y, x - y
    assert s.size == 0 or s.max() < 2 ** 31, "outside the reference's defined range"
    # running extremes from INT_MAX (minima) / INT_MIN (maxima), replaced only by a strictly better value: the first
    # pixel in raster order with the extreme value, none where only the start value itself is reached
    for k, (val, lowest) in enumerate(((s, True), (d, False), (s, False), (d, True))):     # tl, tr, br, bl
        i = np.flatnonzero(val < INT_MAX if lowest else val > INT_MIN)
        if i.size:
            j = i[np.argmin(val[i])] if lowest else i[np.argmax(val[i])]
            out[k] = x[j], y[j]
    return out


class Periodic:
    """frame f of a batch of sw x sh frames whose byte j, counted over the frames back to back, is PAT[j % 251]; .take()
    reads flat indices of the frame as ndarray.take does"""

    def __init__(self, sw, sh, f=0):
        self.shape, self.base = (sh, sw), f * sw * sh

    def take(self, idx):
        return PAT[(self.base + np.asarray(idx, np.int64)) % PAT.size]


def mx_int(s):
    """(float)s - 1.0f, the reference's clamp for a side of s pixels, as an integer"""
    return int(F32(F32(s) - F32(1)))


def overshoot(s):
    """how far (float)s - 1.0f lies past the last pixel s - 1 (negative: it rounds down)"""
    return mx_int(s) - (s - 1)


def src_guard(sw, sh):
    """bytes of guard after a batch's last frame: (its largest row overshoot + 2) rows and 256 bytes, past anything a
    tap of (mx, my) can reach"""
    return (max(0, overshoot(sh)) + 2) * sw + 256


def guarded(a, guard):
    """a copy of array a followed by `guard` SENTINEL bytes -> (buffer, pointer to the copy)"""
    buf = np.full(a.size + guard, SENTINEL, np.uint8)
    buf[:a.size] = a.reshape(-1)
    return buf, buf.ctypes.data


def c_perspective(which, dst_w, dst_h, src, quad):
    """the C oracle's or the reference's gs_perspective_correct of src (h, w), read from a copy with a guard after it"""
    sh, sw = src.shape
    buf, p = guarded(src, src_guard(sw, sh))
    d = np.full((dst_h, dst_w), POISON, np.uint8)
    q = np.ascontiguousarray(quad, np.uint32)
    if which == "reference":
        L.ref().gs_perspective_correct(L.img(d), L.Image(sw, sh, p), L.ptr(q))
    else:
        L.oracle().gso_perspective_correct(L.ptr(d), dst_w, dst_h, p, sw, sh, L.ptr(q))
    return d


def c_blob_corners(which, img, labels, w, h, rec):
    c = np.zeros((4, 2), np.uint32)
    r = np.ascontiguousarray(np.asarray(rec, L.BLOB_DTYPE).reshape(1))
    if which == "reference":
        L.ref().gs_blob_corners(L.Image(w, h, img.ctypes.data), L.ptr(labels), L.ptr(r), L.ptr(c))
    else:
        L.oracle().gso_blob_corners(L.ptr(img), w, h, L.ptr(labels), L.ptr(r), L.ptr(c))
    return c


def record(label, box, centroid):
    r = np.zeros(1, L.BLOB_DTYPE)
    r["label"] = label
    r["bx"], r["by"], r["bw"], r["bh"] = box
    r["cx"], r["cy"] = centroid
    return r[0]


# ---- CPU: model_perspective ------------------------------------------------------------------------------------------
def test_model_perspective_matches_the_round2_goldens():
    """the reference's own output for five quads at 160 x 100, 33 x 47, 1 x 1 and 2 x 5"""
    z = np.load(L.ROOT + "/tests/golden/round2_golden.npz")
    src = np.ascontiguousarray(z["persp_src"])
    for qi, q in enumerate(z["persp_quads"]):
        for dw, dh in ((160, 100), (33, 47), (1, 1), (2, 5)):
            assert np.array_equal(model_perspective(dw, dh, src, q), z["persp_q%d_%dx%d" % (qi, dw, dh)]), (qi, dw, dh)


def _random_quads(rng, sw, sh):
    inside = rng.integers(0, [sw, sh], (4, 2))
    p = rng.integers(0, max(sw, sh) + 30, 2)
    return {
        "near": rng.integers(0, max(sw, sh) + 30, (4, 2)),
        "any": rng.integers(0, 2 ** 32, (4, 2), dtype=np.uint64),            # corners up to 2^32 - 1
        "top": np.array([[M32, M32], [M32 - 1, 0], [2 ** 31, M32], [0, 2 ** 31 + 1]]),
        "degenerate": np.array([p] * 4),
        "mirrored": inside[[1, 0, 3, 2]],
        "crossed": inside[[0, 2, 1, 3]],
    }


@pytest.mark.parametrize("which", LIBS)
def test_model_perspective_on_random_quads(which):
    """small sources of 1 to 60 pixels a side, dst sizes of 1, 2 and odd ones, quads near the image, anywhere up to
    2^32 - 1, degenerate (four equal corners), mirrored and crossed"""
    rng = np.random.default_rng(2026)
    n = 0
    for i in range(40):
        sw, sh = (int(rng.choice([1, 2, 3, int(rng.integers(1, 61))])) for _ in range(2))
        src = rng.integers(0, 256, (sh, sw), dtype=np.uint8)
        dw, dh = (int(rng.choice([1, 2, 3, 7, 33, int(rng.integers(1, 50))])) for _ in range(2))
        for name, q in _random_quads(rng, sw, sh).items():
            q = np.asarray(q, np.uint64).astype(np.uint32)
            assert np.array_equal(model_perspective(dw, dh, src, q), c_perspective(which, dw, dh, src, q)), \
                (i, name, sw, sh, dw, dh, q.tolist())
            n += 1
    assert n == 240


def edge_quads(sw, sh):
    """quads inside, mirrored, right of, below and far outside (crossed, corners up to 2^32 - 1) a sw x sh source"""
    return {
        "inside": [[0, 0], [sw - 1, 0], [sw - 1, sh - 1], [0, sh - 1]],
        "mirrored": [[sw - 1, 0], [0, 0], [0, sh - 1], [sw - 1, sh - 1]],
        "right": [[sw + 3, 0], [sw + 900, 0], [sw + 900, sh - 1], [sw + 3, sh - 1]],
        "below": [[0, sh + 2], [sw - 1, sh + 2], [sw - 1, sh + 700], [0, sh + 700]],
        "far": [[M32, M32], [M32 - 9, 7], [2 ** 31, M32 - 3], [5, 2 ** 31 + 11]],
    }


EDGE_DSTS = ((7, 5), (1, 4), (6, 1))


@pytest.mark.parametrize("which", LIBS)
@pytest.mark.parametrize("axis", ["wide", "tall"])
@pytest.mark.parametrize("s", range(2 ** 24 + 1, 2 ** 24 + 8))
def test_model_perspective_past_2_24(which, axis, s):
    """sources of s x 3 and 3 x s pixels: where (float)s - 1.0f rounds to s or s + 1, a quad right of or below the
    image (and every quad at dst sizes of 1, through the NaN coordinate) takes its first tap past the source, which
    the reference reads as 0"""
    sw, sh = (s, 3) if axis == "wide" else (3, s)
    src = Periodic(sw, sh)
    a = np.resize(PAT, (sh, sw))                        # Periodic's bytes
    for name, q in edge_quads(sw, sh).items():
        for dw, dh in EDGE_DSTS:
            want = model_perspective(dw, dh, src, q)
            assert np.array_equal(want, c_perspective(which, dw, dh, a, q)), (name, dw, dh)


def test_model_perspective_zero_taps_matter():
    """at 16,777,219 columns a quad right of the image clamps to x = 16,777,220, two past the last pixel: its weighted
    taps are both past the row, so the reference's result is black, where the bytes after the row are not zero"""
    sw, sh = 16_777_219, 3
    assert mx_int(sw) == sw + 1
    want = model_perspective(7, 5, Periodic(sw, sh), edge_quads(sw, sh)["right"])
    assert (want == 0).all() and (PAT > 0).all()


# ---- CPU: which source sizes round past their last pixel -------------------------------------------------------------
def table_sizes():
    """every size within 4 float32 ulps of each power of two from 2^12 to 2^31"""
    out = set()
    for k in range(12, 32):
        u = 2 ** max(0, k - 23)
        out.update(2 ** k + d for d in range(-4 * u, 4 * u + 1))
    return sorted(out)


# (first size, last size) of each memory tier of the GPU cases: 3 frames of 3 x s or s x 3 pixels (about 150 MB), and
# 3 frames of one row or one column of s pixels (about 6.4 GB plus a 4.3 GB guard for the row)
TIERS = {"3 x s": (2 ** 24 + 1, 2 ** 24 + 8), "1 x s": (2 ** 31 + 1, 2 ** 31 + 1024)}


def test_rounding_table():
    """(float)s - 1.0f is exact up to 2^24, rounds past s - 1 for some sizes in every band above it and below it for
    others; the GPU cases take the largest overshoot of each tier at its smallest size, and a size that rounds down"""
    sizes = np.array(table_sizes(), np.int64)
    over = np.array([overshoot(int(s)) for s in sizes])
    assert np.all(over[sizes <= 2 ** 24] == 0)
    for k in range(25, 32):
        band = over[(sizes > 2 ** (k - 1)) & (sizes <= 2 ** k)]
        assert (band > 0).any() and (band < 0).any(), k
    sides = {max(c[0], c[1]) for c in PERSP_SOURCES.values()}
    rows = []
    for tier, (lo, hi) in TIERS.items():
        inside = (sizes >= lo) & (sizes <= hi)
        top = over[inside].max()
        first = int(sizes[inside][np.argmax(over[inside])])
        rows.append((tier, first, top))
        assert first in sides, (tier, first, top)
        assert all(overshoot(s) <= top for s in sides if lo <= s <= hi), tier
    assert rows == [("3 x s", 16_777_219, 2), ("1 x s", 2 ** 31 + 384, 129)]
    assert any(overshoot(s) < 0 for s in sides)


# ---- CPU: model_blob_corners -----------------------------------------------------------------------------------------
def _oracle_blobs(a, nb):
    labels = np.full(a.shape, 0x5555, np.uint16)
    blobs = np.zeros(nb, L.BLOB_DTYPE)
    m = L.oracle().gso_blobs(L.ptr(a), a.shape[1], a.shape[0], L.ptr(labels), L.ptr(blobs), nb)
    return labels, blobs[:m]


def test_model_blob_corners_matches_the_round2_goldens():
    """the reference's corners of the first blobs of each round-2 blob image (labels from the oracle's gs_blobs, which
    test_oracle.py checks against the same goldens)"""
    z = np.load(L.ROOT + "/tests/golden/round2_golden.npz")
    n = 0
    for tag in z["blob_tags"]:
        key = "blob_%s_corners" % tag
        if key not in z.files:
            continue
        a = np.ascontiguousarray(z["blob_img_" + str(tag)])
        labels, blobs = _oracle_blobs(a, 1000)
        for j, want in enumerate(z[key]):
            assert np.array_equal(model_blob_corners(a, labels, a.shape[1], a.shape[0], blobs[j]), want), (tag, j)
            n += 1
    assert n > 50


def small_blob_frame():
    """a 40 x 30 frame with hand-placed labels: label 1 on a diamond (four pixels tied for each corner), its pixels
    at 127 and 128 around the >= 128 test, label 2 beside it and label 1 pixels that are background"""
    w, h = 40, 30
    img, lab = np.zeros((h, w), np.uint8), np.zeros((h, w), np.uint16)
    yy, xx = np.mgrid[:h, :w]
    dia = np.abs(xx - 15) + np.abs(yy - 12) <= 6
    img[dia], lab[dia] = 255, 1
    img[12, 9], img[12, 21] = 127, 128                  # the diamond's left tip is background, its right tip counts
    img[3:6, 30:36], lab[3:6, 30:36] = 200, 2
    img[25:28, 2:5], lab[25:28, 2:5] = 90, 1            # label 1 but background
    lab[20, 30:34] = 1                                   # label 1 on background pixels
    return img, lab


def small_records():
    M = M32
    return {
        "diamond": record(1, (0, 0, 40, 30), (15, 12)),
        "diamond-box": record(1, (9, 6, 13, 13), (15, 12)),
        "label2": record(2, (28, 2, 10, 6), (33, 4)),
        "wrong-label": record(7, (0, 0, 40, 30), (3, 4)),
        "outside": record(1, (41, 31, 5, 5), (3, 4)),
        "outside-x": record(1, (40, 0, 100, 30), (3, 4)),
        "part-outside": record(1, (14, 10, 500, 700), (3, 4)),
        "w0": record(1, (0, 0, 0, 30), (3, 4)),
        "h0": record(1, (0, 0, 40, 0), (3, 4)),
        "x-wraps": record(1, (M - 4, 0, 30, 30), (3, 4)),      # box.x + box.w = 25 after the wrap: nothing visited
        "y-wraps": record(1, (0, M - 2, 40, 25), (3, 4)),
        "both-wrap": record(1, (M, M, 2, 2), (3, 4)),
        "x-end-2^32": record(1, (9, 0, M - 8, 30), (3, 4)),    # box.x + box.w = 2^32 wraps to 0: nothing visited
    }


@pytest.mark.parametrize("which", LIBS)
def test_model_blob_corners_on_hand_built_records(which):
    img, lab = small_blob_frame()
    for name, rec in small_records().items():
        want = model_blob_corners(img, lab, 40, 30, rec)
        assert np.array_equal(want, c_blob_corners(which, img, lab, 40, 30, rec)), name
    # each corner is the first of its tied pixels in raster order: the top tip ends two edges of the diamond (tl and
    # tr), the right tip one (br), and the left tip is background (bl: the pixel below it); a wrapped box keeps the
    # centroid
    assert model_blob_corners(img, lab, 40, 30, small_records()["diamond"]).tolist() == [[15, 6], [15, 6], [21, 12],
                                                                                         [10, 13]]
    assert model_blob_corners(img, lab, 40, 30, small_records()["x-wraps"]).tolist() == [[3, 4]] * 4


@pytest.mark.parametrize("which", LIBS)
def test_model_blob_corners_on_random_records(which):
    """binary frames labelled by the oracle's gs_blobs, each blob's own record and records with shifted, cut and
    wrapping boxes"""
    rng = np.random.default_rng(404)
    for i in range(12):
        w, h = int(rng.integers(5, 90)), int(rng.integers(5, 70))
        a = L.binary_like(w, h, 500 + i, density=float(rng.uniform(0.2, 0.7)), smooth=int(rng.integers(0, 3)))
        labels, blobs = _oracle_blobs(a, 200)
        for b in blobs[:8]:
            recs = [b.copy() for _ in range(4)]
            recs[1]["bx"], recs[1]["bw"] = max(int(b["bx"]) - 3, 0), int(b["bw"]) + 6
            recs[2]["bh"] = max(int(b["bh"]) // 2, 1)
            recs[3]["bx"] = (int(b["bx"]) - 1 - int(rng.integers(0, 5))) & M32
            recs[3]["bw"] = (M32 - int(recs[3]["bx"]) + 1 + int(rng.integers(0, w))) & M32    # end wraps into the frame
            for r in recs:
                want = model_blob_corners(a, labels, w, h, r)
                got = c_blob_corners(which, a, labels, w, h, r)
                assert np.array_equal(want, got), (i, L.blob_fields(np.array([r])))


def int_max_frames():
    """(name, w, h, flat runs (start, stop, value, label), records): a row and a column of 2^31 pixels, where the last
    pixel has x + y = INT_MAX.  Only the runs' pages of the zero frames are ever written."""
    E = 2 ** 31
    return [
        ("row-2^31", E, 1, [(E - 200, E, 255, 1)],
         {"blob": record(1, (E - 300, 0, 300, 1), (E - 100, 0)), "last": record(1, (E - 1, 0, 1, 1), (5, 0))}),
        ("col-2^31", 1, E, [(E - 200, E, 255, 1)],
         {"blob": record(1, (0, E - 300, 1, 300), (0, E - 100)), "last": record(1, (0, E - 1, 1, 1), (0, 5))}),
    ]


def host_frame(w, h, runs):
    img, lab = np.zeros(w * h, np.uint8), np.zeros(w * h, np.uint16)
    for a, b, v, label in runs:
        img[a:b], lab[a:b] = v, label
    return img, lab


@pytest.mark.parametrize("which", LIBS)
def test_model_blob_corners_at_int_max(which):
    """a lone pixel at x + y = INT_MAX keeps tl (and in a row bl, whose x - y is INT_MAX too) at the centroid, as the
    reference's minima start at INT_MAX; in a column its x - y = -INT_MAX still sets tr and bl"""
    for name, w, h, runs, recs in int_max_frames():
        img, lab = host_frame(w, h, runs)
        for rn, rec in recs.items():
            want = model_blob_corners(img, lab, w, h, rec)
            assert np.array_equal(want, c_blob_corners(which, img, lab, w, h, rec)), (name, rn)
        del img, lab
    E = 2 ** 31
    (_, w, h, runs, recs), (_, w2, h2, runs2, recs2) = int_max_frames()
    img, lab = host_frame(w, h, runs)
    assert model_blob_corners(img, lab, w, h, recs["last"]).tolist() == [[5, 0], [E - 1, 0], [E - 1, 0], [5, 0]]
    del img, lab
    img, lab = host_frame(w2, h2, runs2)
    assert model_blob_corners(img, lab, w2, h2, recs2["last"]).tolist() == [[0, 5], [0, E - 1], [0, E - 1], [0, E - 1]]


# ---- GPU: perspective ------------------------------------------------------------------------------------------------
def _room(gb):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < gb * 2 ** 30:
        pytest.skip("needs %.0f GB of free device memory, %.1f GB free (the device is shared)" % (gb, free / 2 ** 30))


def _start():
    import torch
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    return time.perf_counter()


def _report(what, t0):
    import torch
    print("\n%s: %.1f s, torch peak device memory %.2f GB" % (what, time.perf_counter() - t0,
                                                              torch.cuda.max_memory_allocated() / 1e9))


def periodic_device(nbytes, guard):
    """a device buffer of nbytes of the periodic content (Periodic's bytes, frames back to back), then `guard` bytes of
    SENTINEL"""
    import torch
    buf = torch.full((nbytes + guard,), SENTINEL, dtype=torch.uint8, device="cuda")
    chunk = torch.from_numpy(PAT).cuda().repeat(1 << 22)
    for j in range(0, nbytes, chunk.numel()):                 # each chunk starts at a multiple of 251
        k = min(chunk.numel(), nbytes - j)
        buf[j:j + k].copy_(chunk[:k])
    return buf


# (sw, sh, n): sources past 2^24 (2 past their last pixel, and rounding down), one side past 2^31 at the table's
# largest overshoot (129: 2^31 + 512 for a last pixel of 2^31 + 383), as a row and as a column
PERSP_SOURCES = {
    "wide-16777219": (16_777_219, 3, 3),
    "wide-16777217": (16_777_217, 3, 3),
    "tall-16777219": (3, 16_777_219, 3),
    "tall-16777217": (3, 16_777_217, 3),
    "row-2^31+384": (2 ** 31 + 384, 1, 3),
    "col-2^31+384": (1, 2 ** 31 + 384, 3),
}


def run_perspective(lib, witness, what, sw, sh, n, src, calls_, model_src):
    """calls_: [(dw, dh, per_frame, quads)], quads one per frame (per_frame) or one for all; every call's dst checked
    byte for byte against model_perspective from poison, and the bytes around it unchanged"""
    import torch
    qs = [np.ascontiguousarray(np.asarray(q, np.uint32).reshape(-1, 4, 2)) for _, _, _, q in calls_]
    dev_q = [torch.from_numpy(q.view(np.int32)).cuda() if pf else None for q, (_, _, pf, _) in zip(qs, calls_)]
    want = []
    for (dw, dh, pf, _), q in zip(calls_, qs):
        want.append(np.stack([model_perspective(dw, dh, model_src(f), q[f if pf else 0]) for f in range(n)]).ravel())

    def run():
        D = [Region(w.size, 0, np.full(w.size, POISON, np.uint8), i) for i, w in enumerate(want)]

        def launch():
            rc = 0
            for (dw, dh, pf, _), q, dq, d in zip(calls_, qs, dev_q, D):
                c = dq.data_ptr() if pf else L.ptr(q)
                rc |= lib.gs_b200_perspective_correct_batch(d.ptr, dw, dh, src, sw, sh, n, c, pf, stream())
            return rc
        rc, seen = traced(launch)
        assert rc == 0, lib.gs_b200_last_error().decode()
        for (dw, dh, pf, _), d, w in zip(calls_, D, want):
            got = d.read("dst")
            bad = np.flatnonzero(got != w)
            assert not bad.size, "%dx%d per_frame=%d: %d bytes differ, the first at %d: %d, want %d" % (
                dw, dh, pf, bad.size, bad[0], got[bad[0]], w[bad[0]])
        return seen

    witnessed(witness, run, ["gsb::k_perspective"], what)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PERSP_SOURCES))
def test_perspective_large_sources(lib, witness, name):
    """every edge quad as the host quad and, three frames at a time, as per-frame device corners (int32 tensors holding
    the bit patterns of values >= 2^31), at dst sizes 7 x 5, 1 x 4 and 6 x 1"""
    sw, sh, n = PERSP_SOURCES[name]
    _room((n * sw * sh + src_guard(sw, sh)) / 2 ** 30 + 3)
    t0 = _start()
    buf = periodic_device(n * sw * sh, src_guard(sw, sh))
    quads = list(edge_quads(sw, sh).values())
    calls_ = []
    for dw, dh in EDGE_DSTS:
        calls_ += [(dw, dh, 0, [q]) for q in quads]
        calls_ += [(dw, dh, 1, [quads[(r + f) % len(quads)] for f in range(n)]) for r in (0, 3)]
    run_perspective(lib, witness, "perspective %s" % name, sw, sh, n, buf.data_ptr(), calls_,
                    lambda f: Periodic(sw, sh, f))
    del buf
    _report("perspective %s" % name, t0)


@pytest.mark.gpu
@pytest.mark.parametrize("dh", [1, 2])
def test_perspective_dst_wider_than_2_24(lib, witness, dh):
    """dw = 2^24 + 5, where (float)x rounds: rows of 1 (every coordinate NaN) and 2, from 48 x 40 sources"""
    _room(2)
    sw, sh, n, dw = 48, 40, 3, 2 ** 24 + 5
    buf = periodic_device(n * sw * sh, src_guard(sw, sh))
    q0, q1, q2 = [[3, 2], [44, 5], [40, 37], [1, 30]], [[47, 0], [0, 3], [9, 39], [40, 30]], [[0, 0]] * 4
    calls_ = [(dw, dh, 0, [q0]), (dw, dh, 1, [q0, q1, q2])]
    run_perspective(lib, witness, "perspective dw=%d dh=%d" % (dw, dh), sw, sh, n, buf.data_ptr(), calls_,
                    lambda f: Periodic(sw, sh, f))


@pytest.mark.gpu
def test_perspective_single_image_past_2_24(G):
    """the host-array gs_perspective_correct on 16,777,219 x 3 and 16,777,217 x 3 sources, quads right of the image on
    row 0 (a tap past the row stays inside the staged frame)"""
    for sw in (16_777_219, 16_777_217):
        sh = 3
        src = Periodic(sw, sh)
        a = np.resize(PAT, (sh, sw))
        for q in ([[sw + 3, 0], [sw + 900, 0], [sw + 900, 0], [sw + 3, 0]], [[sw - 5, 0], [sw + 9, 0], [sw + 9, 0],
                                                                              [sw - 5, 0]]):
            got = G.gs_perspective_correct(np.full((4, 6), POISON, np.uint8), a, np.array(q, np.uint32))
            assert np.array_equal(got, model_perspective(6, 4, src, q)), (sw, q)


# 2^29 + 3 frames of 2 x 1 -> 2 x 2.  A dst side of 1 makes every source coordinate NaN (x / 0.0f), which clamps to
# (mx, my) whatever the corners, so 2 x 2 is the smallest dst whose pixels read the corners: exactly the four corners'
# x, clamped to the two source pixels.  Frame f's corners and content are those of class f % 7; the seven classes'
# corners pick seven different patterns of the two pixels, and 2^29 = 4 (mod 7), so a frame that takes another
# frame's corners 2^29 frames back gets another pattern.
FRAMES_2_29 = 2 ** 29 + 3


def _classes():
    q = np.zeros((7, 4, 2), np.uint32)
    for c in range(7):
        bits = [(c + 1) >> i & 1 for i in range(4)]
        q[c, :, 0] = [(2 ** 31 + 17 * c) if b else 0 for b in bits]     # >= 2^31 clamps to the last pixel, 1
        q[c, :, 1] = [M32 - c, 0, 5 * c, 2 ** 31]                     # rows clamp to 0
    src = np.array([[10 + 20 * c, 200 - 20 * c] for c in range(7)], np.uint8)
    return q, src


@pytest.mark.gpu
def test_perspective_past_2_29_frames(lib, witness):
    """per-frame corners of frame f at (size_t)f * 8: every frame of 2^29 + 3 against expected[f % 7], on the device"""
    import torch
    _room(26)
    t0 = _start()
    n = FRAMES_2_29
    q, cls = _classes()
    exp = np.stack([model_perspective(2, 2, cls[c].reshape(1, 2), q[c]).ravel() for c in range(7)])
    assert len({e.tobytes() for e in exp}) == 7
    reps = -(-n // 7)
    src = torch.full((2 * n + src_guard(2, 1),), SENTINEL, dtype=torch.uint8, device="cuda")
    src[:2 * n].view(n, 2).copy_(torch.from_numpy(cls).cuda().repeat(reps, 1)[:n])
    corners = torch.from_numpy(q.view(np.int32)).cuda().repeat(reps, 1, 1)[:n]          # 16 GiB
    want = torch.from_numpy(exp).cuda()

    def run():
        dst = torch.full((4 * n + 256,), POISON, dtype=torch.uint8, device="cuda")
        rc, seen = traced(lambda: lib.gs_b200_perspective_correct_batch(dst.data_ptr(), 2, 2, src.data_ptr(), 2, 1, n,
                                                                        corners.data_ptr(), 1, stream()))
        assert rc == 0, lib.gs_b200_last_error().decode()
        assert bool((dst[4 * n:] == POISON).all()), "bytes after the batch changed"
        d = dst[:4 * n].view(n, 4)
        for c in range(7):                                   # the frames of class c, strided: no n-sized temporaries
            bad = (d[c::7] != want[c]).any(1)
            if bool(bad.any()):
                f = c + 7 * int(bad.nonzero()[0, 0])
                raise AssertionError("frame %d (class %d): %s, want %s" % (f, c, d[f].tolist(), exp[c].tolist()))
        del dst, d
        return seen

    witnessed(witness, run, ["gsb::k_perspective"], "perspective %d frames" % n)
    del src, corners
    _report("perspective %d frames" % n, t0)


# ---- GPU: blob corners -----------------------------------------------------------------------------------------------
def straddle_frames():
    """(name, w, h, flat runs, records) of 1-row and 1-column frames 2^30 + 512 long with a blob across 2^30, where
    a bias of 2^30 wrapped, and the frames of int_max_frames()"""
    c, M, E = 2 ** 30, M32, 2 ** 30 + 512
    runs = [(c - 100, c + 101, 255, 1), (c + 101, c + 140, 127, 1), (c + 140, c + 160, 255, 2),
            (c - 140, c - 120, 255, 2)]
    out = []
    for name, w, h in (("row-2^30", E, 1), ("col-2^30", 1, E)):
        box = (lambda x0, bw: (x0, 0, bw, 1)) if h == 1 else (lambda x0, bw: (0, x0, 1, bw))
        cen = (lambda t: (t, 0)) if h == 1 else (lambda t: (0, t))
        out.append((name, w, h, runs, {
            "blob": record(1, box(c - 150, 320), cen(c)),
            "label2": record(2, box(c - 150, 320), cen(1)),
            "part": record(1, box(c - 50, 30), cen(7)),
            "past-frame": record(1, box(c, 2 ** 31), cen(7)),
            "wraps": record(1, box(M - 99, 200), cen(7)),
            "w0": record(1, box(c - 100, 0), cen(7)),
            "wrong-label": record(3, box(c - 150, 320), cen(7)),
        }))
    return out + int_max_frames()


def blob_device_frame(w, h, runs):
    import torch
    img = torch.zeros(w * h + 256, dtype=torch.uint8, device="cuda")
    lab = torch.zeros(w * h + 128, dtype=torch.int16, device="cuda")
    img[w * h:], lab[w * h:] = SENTINEL, LABEL_SENTINEL
    for a, b, v, label in runs:
        img[a:b], lab[a:b] = v, label
    return img, lab


def run_blob_corners(lib, witness, what, w, h, img_ptr, lab_ptr, recs, want):
    import torch
    R = torch.from_numpy(np.ascontiguousarray(np.array(list(recs.values()), L.BLOB_DTYPE)).view(np.uint8)).cuda()

    def run():
        out = torch.full((len(recs) * 8,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
        rc, seen = traced(lambda: max(lib.gs_b200_blob_corners(img_ptr, w, h, lab_ptr, R.data_ptr() + 32 * i,
                                                               out.data_ptr() + 32 * i, stream())
                                      for i in range(len(recs))))
        assert rc == 0, lib.gs_b200_last_error().decode()
        got = out.cpu().numpy().view(np.uint32).reshape(-1, 4, 2)
        for (name, _), g, wnt in zip(recs.items(), got, want):
            assert np.array_equal(g, wnt), (name, g.tolist(), wnt.tolist())
        return seen

    witnessed(witness, run, ["gsb::k_blob_corners"], what)


@pytest.mark.gpu
@pytest.mark.parametrize("case", straddle_frames(), ids=lambda c: c[0])
def test_blob_corners_large_frames(lib, witness, case):
    """hand-built 0 / 255 frames and label maps of a row or a column of 2^30 + 512 and 2^31 pixels, each followed by a
    nonzero guard; every record's corners against model_blob_corners"""
    name, w, h, runs, recs = case
    _room(3 * w * h / 2 ** 30 + 1)
    t0 = _start()
    himg, hlab = host_frame(w, h, runs)
    want = [model_blob_corners(himg, hlab, w, h, r) for r in recs.values()]
    del himg, hlab
    img, lab = blob_device_frame(w, h, runs)
    run_blob_corners(lib, witness, "blob corners %s" % name, w, h, img.data_ptr(), lab.data_ptr(), recs, want)
    del img, lab
    _report("blob corners %s" % name, t0)


@pytest.mark.gpu
def test_blob_corners_small_records(G, lib, witness):
    """the hand-built records of the CPU test through the host-array gs_blob_corners and through gs_b200_blob_corners
    on guarded device copies"""
    import torch
    img, lab = small_blob_frame()
    recs = small_records()
    want = [model_blob_corners(img, lab, 40, 30, r) for r in recs.values()]
    for (name, r), w in zip(recs.items(), want):
        assert np.array_equal(G.gs_blob_corners(img, lab, np.array([r], L.BLOB_DTYPE)), w), name
    dimg = torch.full((img.size + 256,), SENTINEL, dtype=torch.uint8, device="cuda")
    dlab = torch.full((img.size + 128,), LABEL_SENTINEL, dtype=torch.int16, device="cuda")
    dimg[:img.size].copy_(torch.from_numpy(img.ravel()))
    dlab[:img.size].copy_(torch.from_numpy(lab.ravel().view(np.int16)))
    run_blob_corners(lib, witness, "blob corners small records", 40, 30, dimg.data_ptr(), dlab.data_ptr(), recs, want)


@pytest.mark.gpu
def test_scanner_chain(lib, witness):
    """the reference CLI's scanner order on a device-resident batch: gs_b200_blob_corners of each frame's largest blob
    writes the corners gs_b200_perspective_correct_batch(per_frame = 1) reads, against the two models chained"""
    import torch
    n, w, h, dw, dh = 3, 200, 150, 90, 70
    binary = np.stack([L.binary_like(w, h, 60 + f, density=0.45, smooth=3) for f in range(n)])
    gray = np.stack([L.natural_like(w, h, 70 + f) for f in range(n)])
    labs, picks, quads, want = [], [], [], []
    for f in range(n):
        lab, blobs = _oracle_blobs(binary[f], 1000)
        b = blobs[int(np.argmax(blobs["area"]))]                # the largest, the first one on ties
        labs.append(lab)
        picks.append(b)
        quads.append(model_blob_corners(binary[f], lab, w, h, b))
        want.append(model_perspective(dw, dh, gray[f], quads[-1]))
    B, LB, GR = (torch.from_numpy(np.ascontiguousarray(x)).cuda()
                 for x in (binary, np.stack(labs).view(np.int16), gray))
    P = torch.from_numpy(np.ascontiguousarray(np.array(picks, L.BLOB_DTYPE)).view(np.uint8)).cuda()
    want = np.stack(want).ravel()

    def run():
        C = torch.full((n * 8,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
        D = Region(want.size, 0, np.full(want.size, POISON, np.uint8), 5)

        def launch():
            rc = 0
            for f in range(n):
                rc |= lib.gs_b200_blob_corners(B.data_ptr() + f * w * h, w, h, LB.data_ptr() + 2 * f * w * h,
                                               P.data_ptr() + 32 * f, C.data_ptr() + 32 * f, stream())
            return rc | lib.gs_b200_perspective_correct_batch(D.ptr, dw, dh, GR.data_ptr(), w, h, n, C.data_ptr(), 1,
                                                              stream())
        rc, seen = traced(launch)
        assert rc == 0, lib.gs_b200_last_error().decode()
        assert np.array_equal(C.cpu().numpy().view(np.uint32).reshape(n, 4, 2), np.stack(quads))
        assert np.array_equal(D.read("dst"), want)
        return seen

    witnessed(witness, run, ["gsb::k_blob_corners", "gsb::k_perspective"], "scanner chain")
