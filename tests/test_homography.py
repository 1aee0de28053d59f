"""A RANSAC homography per frame from its ORB matches, and the template's outline in the scene, on the device
(include/grayskull_homography.h, libgrayskull_homography.so).

The rule is the header's, restated here as a Python model (model_frame, model_quad): exact integers where the rule is
integer, Python floats (IEEE double, one rounding per operation, no FMA) where it is double, numpy float64 for the
scoring, which is elementwise.  On the CPU the model is pinned against hand-built lists and against the true placement
of a template in a warped scene, and the companion is checked as a library.  On the GPU both calls are checked bit-exact
against the model with poisoned outputs: on the device's own pyramid ORB lists, on synthetic lists with 10-90 %
outliers, at several record strides and hypothesis counts, at byte offsets, without inlier records and past 65535
frames; then on the caller's stream, two streams and a CUDA graph; and through gsb_magick's find stage against the same
chain built from the library calls.
"""
import ctypes as C
import math
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

import _libs as L
from _gpu import Region, lib, traced, witness, witnessed  # noqa: F401

ROOT = L.ROOT
KP, MATCH = L.KP_DTYPE, L.MATCH_DTYPE
M64 = (1 << 64) - 1
GOLDEN = 0x9E3779B97F4A7C15
COORD = 1 << 20
TRIPLES = ((0, 1, 2), (0, 1, 3), (0, 2, 3), (1, 2, 3))

KERNELS = {"gsb::k_find": "find", "gsb::k_quads": "quads"}


# ---- the rule, restated -------------------------------------------------------------------------------------------
def mix(z):
    """splitmix64's finaliser"""
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def sample(seed, f, k, m):
    """rule 2: hypothesis k's four indices among m correspondences of frame f"""
    idx = []
    for j in range(4):
        J = m - 4 + j
        t = ((mix((seed + GOLDEN * ((f << 18) | (k << 2) | j)) & M64) >> 32) * (J + 1)) >> 32
        idx.append(J if t in idx else t)
    return sorted(idx)


def _orient(p, q, r, o):
    return (q[o] - p[o]) * (r[o + 1] - p[o + 1]) - (q[o + 1] - p[o + 1]) * (r[o] - p[o])


def degenerate(pts):
    """rule 3 over four (x, y, X, Y)"""
    for t in TRIPLES:
        ot, os_ = _orient(*[pts[i] for i in t], 0), _orient(*[pts[i] for i in t], 2)
        if ot == 0 or os_ == 0 or (ot > 0) != (os_ > 0):
            return True
    return False


def solve(pts):
    """rule 4 over a list of (x, y, X, Y) -> 9 floats, or None when invalid"""
    m = len(pts)
    cx, cy, CX, CY = (sum(p[i] for p in pts) // m for i in range(4))
    c = [(p[0] - cx, p[1] - cy, p[2] - CX, p[3] - CY) for p in pts]
    kt = max(max(abs(a), abs(b)) for a, b, _, _ in c).bit_length()
    ks = max(max(abs(A), abs(B)) for _, _, A, B in c).bit_length()
    s = [0] * 22
    for a, b, A, B in c:
        R = A * A + B * B
        for q, v in enumerate((a, b, A, B, a * a, a * b, b * b, a * A, b * A, a * B, b * B, a * a * A, a * b * A,
                               b * b * A, a * a * B, a * b * B, b * b * B, a * R, b * R, a * a * R, a * b * R, b * b * R)):
            s[q] += v
    S = [[s[4], s[5], s[0], 0, 0, 0, -s[11], -s[12]], [0, s[6], s[1], 0, 0, 0, -s[12], -s[13]],
         [0, 0, m, 0, 0, 0, -s[7], -s[8]], [0, 0, 0, s[4], s[5], s[0], -s[14], -s[15]],
         [0, 0, 0, 0, s[6], s[1], -s[15], -s[16]], [0, 0, 0, 0, 0, m, -s[9], -s[10]],
         [0, 0, 0, 0, 0, 0, s[19], s[20]], [0, 0, 0, 0, 0, 0, 0, s[21]]]
    V = [s[7], s[8], s[2], s[9], s[10], s[3], -s[17], -s[18]]
    E = [kt, kt, 0, kt, kt, 0, kt + ks, kt + ks]
    A = [[0.0] * 8 for _ in range(8)]
    for p in range(8):
        for q in range(p, 8):
            A[q][p] = math.ldexp(float(S[p][q]), -(E[p] + E[q]))
    r = [math.ldexp(float(V[p]), -(E[p] + ks)) for p in range(8)]
    for j in range(8):
        d = A[j][j]
        for k in range(j):
            d = d - A[j][k] * A[j][k]
        if not (0.0 < d < math.inf):
            return None
        A[j][j] = math.sqrt(d)
        for i in range(j + 1, 8):
            t = A[i][j]
            for k in range(j):
                t = t - A[i][k] * A[j][k]
            A[i][j] = t / A[j][j]
    for i in range(8):
        t = r[i]
        for k in range(i):
            t = t - A[i][k] * r[k]
        r[i] = t / A[i][i]
    for i in range(7, -1, -1):
        t = r[i]
        for k in range(i + 1, 8):
            t = t - A[k][i] * r[k]
        r[i] = t / A[i][i]
    st, up = math.ldexp(1.0, -kt), math.ldexp(1.0, ks)
    G = []
    for row in range(3):
        p, q, cc = r[3 * row], r[3 * row + 1], (r[3 * row + 2] if row < 2 else 1.0)
        P, Q = p * st, q * st
        G += [P, Q, cc - ((P * float(cx)) + (Q * float(cy)))]
    H = [G[j] * up + float(CX) * G[6 + j] for j in range(3)] + [G[3 + j] * up + float(CY) * G[6 + j] for j in range(3)]
    H += G[6:]
    d = H[8]
    if d == 0.0 or not math.isfinite(d):
        return None
    H = [h / d for h in H]
    return H if all(math.isfinite(h) for h in H) else None


def inlier_mask(H, P, threshold):
    """rule 5 for 9 floats H over P (m, 4) int64 -> bool (m,)"""
    x, y, X, Y = (P[:, i].astype(np.float64) for i in range(4))
    with np.errstate(all="ignore"):
        u = (H[0] * x + H[1] * y) + H[2]
        v = (H[3] * x + H[4] * y) + H[5]
        w = (H[6] * x + H[7] * y) + H[8]
        du, dv = u - X * w, v - Y * w
        return (w > 0) & ((du * du + dv * dv) <= (threshold * threshold) * (w * w))


def _counts_many(Hs, P, threshold):
    """inlier counts of many hypotheses (K, 9) over P, in blocks"""
    out = np.zeros(len(Hs), np.int64)
    x, y, X, Y = (P[None, :, i].astype(np.float64) for i in range(4))
    t2 = threshold * threshold
    for k0 in range(0, len(Hs), 2048):
        h = Hs[k0:k0 + 2048, :, None]
        with np.errstate(all="ignore"):
            u = (h[:, 0] * x + h[:, 1] * y) + h[:, 2]
            v = (h[:, 3] * x + h[:, 4] * y) + h[:, 5]
            w = (h[:, 6] * x + h[:, 7] * y) + h[:, 8]
            du, dv = u - X * w, v - Y * w
            out[k0:k0 + 2048] = ((w > 0) & ((du * du + dv * dv) <= t2 * (w * w))).sum(1)
    return out


def correspondences(k1, c1, k2, c2, recs):
    """rule 1: k1, k2 (stride,) KP arrays with used lengths c1, c2; recs (c,) MATCH -> (record indices, P (m, 4))"""
    i1, i2 = recs["idx1"].astype(np.int64), recs["idx2"].astype(np.int64)
    ok = (i1 < c1) & (i2 < c2)
    P = np.zeros((len(recs), 4), np.int64)
    P[ok, 0], P[ok, 1] = k1["x"][i1[ok]], k1["y"][i1[ok]]
    P[ok, 2], P[ok, 3] = k2["x"][i2[ok]], k2["y"][i2[ok]]
    ok &= (P < COORD).all(1)
    return np.flatnonzero(ok), P[ok]


def model_frame(rec_idx, P, f, hypotheses, seed, threshold):
    """rules 2-6 for frame f's correspondences P (m, 4) at record indices rec_idx -> (H 9 floats, inliers, records)"""
    m = len(P)
    none = ([0.0] * 9, 0, np.zeros(0, np.int64))
    if m < 4:
        return none
    rows = [tuple(int(v) for v in p) for p in P]
    Hs = np.full((hypotheses, 9), np.nan)
    for k in range(hypotheses):
        pts = [rows[i] for i in sample(seed, f, k, m)]
        H = None if degenerate(pts) else solve(pts)
        if H is not None:
            Hs[k] = H
    valid = ~np.isnan(Hs[:, 8])
    if not valid.any():
        return none
    counts = np.where(valid, _counts_many(Hs, P, threshold), -1)
    best = int(np.argmax(counts))                                  # the first of the largest: the lowest k
    H, cb = [float(v) for v in Hs[best]], int(counts[best])
    final, count = H, cb
    if cb >= 4:
        inl = inlier_mask(H, P, threshold)
        Hr = solve([rows[i] for i in np.flatnonzero(inl)])
        if Hr is not None:
            cr = int(inlier_mask(Hr, P, threshold).sum())
            if cr >= cb:
                final, count = Hr, cr
    return final, count, rec_idx[inlier_mask(final, P, threshold)]


def model_quad(H, inliers, min_inliers, tw, th, sw, sh):
    """rule 7 -> (corners [(x, y)] * 4, found)"""
    if all(h == 0.0 for h in H) or inliers < min_inliers:
        return [(0, 0)] * 4, 0
    out = []
    for x, y in ((0.0, 0.0), (float(tw - 1), 0.0), (float(tw - 1), float(th - 1)), (0.0, float(th - 1))):
        u = (H[0] * x + H[1] * y) + H[2]
        v = (H[3] * x + H[4] * y) + H[5]
        w = (H[6] * x + H[7] * y) + H[8]
        if not w > 0:
            return [(0, 0)] * 4, 0
        with np.errstate(all="ignore"):
            px, py = float(np.rint(np.float64(u) / w)), float(np.rint(np.float64(v) / w))
        if math.isnan(px) or math.isnan(py):
            return [(0, 0)] * 4, 0
        out.append((int(min(max(px, 0.0), sw - 1)), int(min(max(py, 0.0), sh - 1))))
    return out, 1


def model_batch(k1, n1, k2, n2, mt, mc, hypotheses, seed, threshold, frames=None):
    """the lists (n, stride) as the call reads them -> {f: (H, inliers, inlier record indices)}"""
    fs = range(mt.shape[0]) if frames is None else frames
    out = {}
    for f in fs:
        c = min(int(mc[f]), mt.shape[1])
        idx, P = correspondences(k1[f], min(int(n1[f]), k1.shape[1]), k2[f], min(int(n2[f]), k2.shape[1]), mt[f, :c])
        out[f] = model_frame(idx, P, f, hypotheses, seed, threshold)
    return out


# ---- hand-built lists ------------------------------------------------------------------------------------------------
def lists(pairs, extra=()):
    """[(x, y, X, Y)] -> (k1, k2, recs) of one frame: keypoint i of each list is pair i, record i matches them; extra
    records (idx1, idx2) are appended"""
    k1, k2 = np.zeros(len(pairs), KP), np.zeros(len(pairs), KP)
    for i, (x, y, X, Y) in enumerate(pairs):
        k1[i]["x"], k1[i]["y"], k2[i]["x"], k2[i]["y"] = x, y, X, Y
    recs = np.zeros(len(pairs) + len(extra), MATCH)
    recs["idx1"][:len(pairs)] = recs["idx2"][:len(pairs)] = np.arange(len(pairs))
    for i, (a, b) in enumerate(extra):
        recs[len(pairs) + i] = (a, b, 0)
    return k1, k2, recs


def fit(pairs, hypotheses=64, seed=0, threshold=3.0, extra=(), f=0):
    k1, k2, recs = lists(pairs, extra)
    idx, P = correspondences(k1, len(k1), k2, len(k2), recs)
    return model_frame(idx, P, f, hypotheses, seed, threshold)


def project(Ht, x, y):
    w = Ht[6] * x + Ht[7] * y + Ht[8]
    return (Ht[0] * x + Ht[1] * y + Ht[2]) / w, (Ht[3] * x + Ht[4] * y + Ht[5]) / w


def planted(Ht, n_in, n_out, seed, span=600):
    """n_in correspondences on the map Ht (exact when Ht maps the grid points to integers) and n_out far-off outliers,
    shuffled -> (pairs, the inlier positions)"""
    rng = np.random.default_rng(seed)
    pairs, good = [], set()
    pts = set()
    while len(pts) < n_in:
        pts.add((int(rng.integers(0, span)), int(rng.integers(0, span))))
    for x, y in sorted(pts):
        X, Y = project(Ht, x, y)
        pairs.append((x, y, int(round(X)), int(round(Y))))
    for _ in range(n_out):
        x, y = int(rng.integers(0, span)), int(rng.integers(0, span))
        X, Y = project(Ht, x, y)
        pairs.append((x, y, abs(int(X + rng.choice([-1, 1]) * rng.integers(40, 200))), abs(int(Y + rng.integers(-200, 200)))))
    order = rng.permutation(len(pairs))
    return [pairs[i] for i in order], {int(np.flatnonzero(order == i)[0]) for i in range(n_in)}


def reproj(H, pairs):
    return max(math.hypot(*(np.subtract(project(H, x, y), (X, Y)))) for x, y, X, Y in pairs)


# ---- CPU: the model against hand-built lists -------------------------------------------------------------------------
@pytest.mark.parametrize("name,Ht", [
    ("translation", [1, 0, 37, 0, 1, 12, 0, 0, 1]),
    ("affine", [2, 1, 100, 1, 3, 50, 0, 0, 1]),
    ("projective", None),
])
def test_planted_maps_recover_exactly_the_planted_inliers(name, Ht):
    if Ht is None:
        # a projective map does not land its integer points on integers: the inliers are rounded to the pixel, so
        # the check is the planted set and a fit within the rounding
        Ht = [1.1, 0.05, 20, -0.03, 0.95, 40, 1e-4, 5e-5, 1]
    pairs, good = planted(Ht, 60, 40, seed=len(name))
    H, count, recs = fit(pairs, hypotheses=200)
    assert set(recs.tolist()) == good and count == len(good), name
    exact = name != "projective"
    err = reproj(H, [pairs[i] for i in good])
    assert err < (1e-6 if exact else 0.75), (name, err)
    assert H[8] == 1.0


def test_score_boundary_3_4_5():
    H = [1.0, 0.0, 10.0, 0.0, 1.0, 20.0, 0.0, 0.0, 1.0]
    P = np.array([[0, 0, 13, 24], [5, 5, 18, 29], [5, 5, 18, 30]], np.int64)   # offsets (3, 4), (3, 4), (3, 5)
    assert inlier_mask(H, P, 5.0).tolist() == [True, True, False]
    assert inlier_mask(H, P, 4.999999).tolist() == [False, False, False]
    # w <= 0 is never an inlier, whatever the distance
    assert inlier_mask([1.0, 0, 0, 0, 1.0, 0, 0, 0, -1.0], np.array([[1, 1, 1, 1]]), 1e9).tolist() == [False]


def test_all_degenerate_sets_are_not_found():
    collinear = [(10 * i, 20 * i, 10 * i + 5, 20 * i + 7) for i in range(12)]
    assert fit(collinear)[1] == 0 and fit(collinear)[0] == [0.0] * 9
    # a mirror flips every orientation
    flip = [(x, y, 500 - x, y) for x, y in ((0, 0), (100, 0), (0, 100), (100, 100), (50, 20), (20, 70))]
    assert fit(flip)[1] == 0
    # duplicates of one point
    assert fit([(5, 5, 6, 6)] * 10)[1] == 0
    assert degenerate([(0, 0, 0, 0), (1, 0, 1, 0), (0, 1, 0, 1), (1, 1, 1, 1)]) is False


def test_lowest_k_wins_ties():
    # two translations of 6 points each: the hypotheses drawn from either group alone tie at 6 inliers
    a = [(x, y, x + 100, y) for x, y in ((0, 0), (40, 3), (7, 50), (60, 61), (25, 90), (90, 20))]
    b = [(x + 300, y, x + 300, y + 200) for x, y in ((0, 0), (40, 3), (7, 50), (60, 61), (25, 90), (90, 20))]
    for pairs in (a + b, b + a):
        P = np.array(pairs, np.int64)
        winners = []
        for k in range(400):
            pts = [pairs[i] for i in sample(0, 0, k, len(pairs))]
            H = None if degenerate(pts) else solve(pts)
            if H is not None and inlier_mask(H, P, 3.0).sum() == 6:
                winners.append((k, frozenset(np.flatnonzero(inlier_mask(H, P, 3.0)).tolist())))
        assert {w[1] for w in winners} == {frozenset(range(6)), frozenset(range(6, 12))}
        H, count, recs = fit(pairs, hypotheses=400)
        assert count == 6 and frozenset(recs.tolist()) == winners[0][1]


def test_first_samples_table():
    # splitmix64 seeded 0 gives 0xE220A8397B1DCDAF first: the finaliser of 0 + GOLDEN
    assert mix(GOLDEN) == 0xE220A8397B1DCDAF and mix(0) == 0
    # m = 4 has one sample; (0, 0, 0, 5): j = 0 draws t = hi32(z0) * 2 >> 32 with z0 = mix(GOLDEN * 0) = 0, so 0; j = 1
    # draws from z1 = mix(GOLDEN) (hi32 0xE220A839 * 3 >> 32 = 2); j = 2 from mix(2 GOLDEN), j = 3 from mix(3 GOLDEN)
    assert sample(0, 0, 0, 4) == [0, 1, 2, 3]
    assert ((0xE220A839 * 3) >> 32) == 2
    table = {(0, 0, 0, 5): [0, 1, 2, 4], (0, 0, 1, 10): [0, 1, 2, 6], (7, 3, 2, 300): [15, 121, 198, 216],
             (2 ** 64 - 1, 70000, 65535, 1000): [319, 571, 663, 804]}
    for (seed, f, k, m), want in table.items():
        idx = []
        for j in range(4):                                       # the rule once more, spelled out
            J = m - 4 + j
            zz = (seed + GOLDEN * ((f << 18) | (k << 2) | j)) % 2 ** 64
            zz = ((zz ^ (zz >> 30)) * 0xBF58476D1CE4E5B9) % 2 ** 64
            zz = ((zz ^ (zz >> 27)) * 0x94D049BB133111EB) % 2 ** 64
            zz ^= zz >> 31
            t = (zz >> 32) * (J + 1) // 2 ** 32
            idx.append(J if t in idx else t)
        assert sample(seed, f, k, m) == sorted(idx) == want


def test_skipped_records_and_too_few():
    pairs, good = planted([1, 0, 5, 0, 1, 7, 0, 0, 1], 10, 0, seed=3)
    # keypoints 10 and 11 have a coordinate at 2^20; records 12..14 point past the lists
    k1, k2, recs = lists(pairs + [(COORD, 5, 5, 5), (5, 5, 5, COORD)], extra=[(12, 0), (0, 12), (99, 99)])
    idx, P = correspondences(k1, len(k1), k2, len(k2), recs)
    assert idx.tolist() == list(range(10))
    # a template count of 9 drops the record whose idx1 is 9
    idx, P = correspondences(k1, 9, k2, len(k2), recs)
    assert idx.tolist() == [i for i in range(10) if recs["idx1"][i] != 9]
    H, count, recs_in = model_frame(idx, P, 0, 50, 0, 3.0)
    assert count == 9 and recs_in.tolist() == idx.tolist()
    # m < 4 writes H = 0 and no inliers; m = 4 fits
    H, count, recs_in = fit(pairs[:3])
    assert H == [0.0] * 9 and count == 0 and len(recs_in) == 0
    assert fit(pairs[:4])[1] == 4


def test_a_refit_that_loses_is_not_kept():
    # 8 points on a translation by (100, 50), 5 at +2.9 px in x and 3 at -2.9 px: a hypothesis from the 8 exact points
    # has all 16 inliers, and the refit over them, pulled towards the 5, loses the 3
    rng = np.random.default_rng(5)
    xy = [tuple(int(v) for v in p) for p in rng.choice(400, (16, 2), replace=False)]
    pairs = [(x, y, x + 100, y + 50) for x, y in xy[:8]]
    pairs += [(x, y, x + 103, y + 50) for x, y in xy[8:13]] + [(x, y, x + 97, y + 50) for x, y in xy[13:]]
    P = np.array(pairs, np.int64)
    seen = {"lost": 0, "kept": 0}
    for seed in range(30):
        Hm, count, _ = model_frame(np.arange(16), P, 0, 40, seed, 3.0)
        best, cb = None, -1                                      # the best hypothesis and the refit, by hand
        for k in range(40):
            pts = [pairs[i] for i in sample(seed, 0, k, 16)]
            H = None if degenerate(pts) else solve(pts)
            if H is not None and inlier_mask(H, P, 3.0).sum() > cb:
                best, cb = H, int(inlier_mask(H, P, 3.0).sum())
        Hr = solve([pairs[i] for i in np.flatnonzero(inlier_mask(best, P, 3.0))])
        cr = -1 if Hr is None else int(inlier_mask(Hr, P, 3.0).sum())
        if cr < cb:
            seen["lost"] += 1
            assert Hm == best and count == cb
        else:
            seen["kept"] += 1
            assert Hm == Hr and count == cr
    assert seen["lost"] and seen["kept"], seen


def i128_to_double_by_parts(v):
    """the device's conversion: the top 64 bits with a sticky bit for the rest, converted once, scaled exactly"""
    neg, u = v < 0, abs(v)
    if u < 2 ** 64:
        d = float(u)
    else:
        sh = u.bit_length() - 64
        top = (u >> sh) | (1 if u & ((1 << sh) - 1) else 0)
        d = math.ldexp(float(top), sh)
    return -d if neg else d


def test_int128_to_double_rounds_ties_to_even():
    for base in (2 ** 70, 2 ** 100, 2 ** 112 - 2 ** 59, 2 ** 64, 3 * 2 ** 80):
        ulp = 2 ** (base.bit_length() - 53)
        for v in (base + ulp // 2, base + ulp + ulp // 2, base + ulp // 2 + 1, base + ulp // 2 - 1, base + 1,
                  base - 1, base + ulp - 1):
            for s in (1, -1):
                assert i128_to_double_by_parts(s * v) == float(s * v), hex(v)
    # the two ties of 2^70's ulp 2^18 go to the even neighbour, down and up
    v = 2 ** 70 + 2 ** 17
    assert i128_to_double_by_parts(v) == 2.0 ** 70 and i128_to_double_by_parts(v + 2 ** 18) == 2.0 ** 70 + 2 ** 19
    # converting the halves separately rounds twice: hi * 2^64 + lo lands on the wrong side of a near-tie
    u = 2 ** 64 * (2 ** 53 + 1) + 1                            # hi rounds down to 2^53, the sum is past half an ulp
    assert float(u >> 64) * 2.0 ** 64 + float(u & M64) != float(u) == i128_to_double_by_parts(u)


def test_quads_half_even_clamp_and_w():
    H = [1.0, 0.0, 10.5, 0.0, 1.0, 11.5, 0.0, 0.0, 1.0]
    assert model_quad(H, 10, 10, 5, 4, 100, 100) == ([(10, 12), (14, 12), (14, 14), (10, 14)], 1)
    assert model_quad(H, 9, 10, 5, 4, 100, 100) == ([(0, 0)] * 4, 0)
    assert model_quad([0.0] * 9, 99, 4, 5, 4, 100, 100)[1] == 0
    # clamped to the frame, both sides
    assert model_quad([1.0, 0, -50, 0, 1.0, 95, 0, 0, 1.0], 10, 4, 70, 10, 60, 100)[0] == [(0, 95), (19, 95), (19, 99),
                                                                                         (0, 99)]
    # w <= 0 at a corner: not found
    assert model_quad([1.0, 0, 0, 0, 1.0, 0, -0.01, 0, 1.0], 10, 4, 200, 10, 1000, 1000)[1] == 0
    assert model_quad([1.0, 0, 0, 0, 1.0, 0, -0.01, 0, 1.0], 10, 4, 100, 10, 1000, 1000)[1] == 1   # w = 0.01 at 99


# ---- CPU: the rule on real features ----------------------------------------------------------------------------------
CANVAS = (640, 480)
CROP = (200, 140, 200, 160)                   # x, y, w, h of the template in the canvas
SCENE = (512, 384)
PARALLELOGRAMS = [((60, 40), (571, 70), (40, 423)), ((90, 70), (590, 20), (120, 450)), ((30, 30), (540, 30), (70, 410))]


def _para(tl, tr, bl):
    return np.array([tl, tr, (tr[0] + bl[0] - tl[0], tr[1] + bl[1] - tl[1]), bl], np.uint32)


def accuracy_scene(p, seed=31):
    """the canvas, the template (a crop of it), the scene (the canvas warped from a parallelogram by the reference's
    bilinear quad warp, exactly affine there) and the true template corners in the scene"""
    O = L.oracle()
    canvas = L.natural_like(CANVAS[0], CANVAS[1], seed)
    x0, y0, tw, th = CROP
    tpl = np.ascontiguousarray(canvas[y0:y0 + th, x0:x0 + tw])
    q = _para(*p)
    sw, sh = SCENE
    scene = np.zeros((sh, sw), np.uint8)
    O.gso_perspective_correct(L.ptr(scene), sw, sh, L.ptr(canvas), CANVAS[0], CANVAS[1], L.ptr(q))
    tl, tr, bl = (np.array(v, np.float64) for v in p)
    A = np.stack([(tr - tl) / (sw - 1), (bl - tl) / (sh - 1)], 1)          # scene (x, y) -> canvas - tl
    inv = np.linalg.inv(A)
    truth = [inv @ (np.array([x0 + cx, y0 + cy], np.float64) - tl) for cx, cy in ((0, 0), (tw - 1, 0), (tw - 1, th - 1),
                                                                                   (0, th - 1))]
    return canvas, tpl, scene, np.array(truth)


def orb_lists(tpl, scene):
    """the orb verb's keypoints of template and scene and its matches (its shared 1 MiB buffer included)"""
    Od = L.oracle()
    buf = np.zeros(1024 * 1024, np.uint8)
    kt = L.pyramid_orb(Od, tpl, 2500, 20, buf, 3)
    ks = L.pyramid_orb(Od, scene, 2500, 20, buf, 3)
    return kt, ks, L.o_match(Od, kt, ks, 300, 60.0)


# measured with the model, 1024 hypotheses, seed 0, threshold 3: the largest corner error against the truth is 1.01,
# 0.99 and 1.35 px on the three parallelograms (68 of 76, 55 of 60 and 42 of 47 matches are inliers)
ACCURACY_PX = 3.0


@pytest.mark.parametrize("p", PARALLELOGRAMS)
def test_template_found_where_the_warp_put_it(p):
    _, tpl, scene, truth = accuracy_scene(p)
    kt, ks, mt = orb_lists(tpl, scene)
    idx, P = correspondences(kt, len(kt), ks, len(ks), mt)
    H, count, _ = model_frame(idx, P, 0, 1024, 0, 3.0)
    corners, found = model_quad(H, count, 10, tpl.shape[1], tpl.shape[0], scene.shape[1], scene.shape[0])
    assert found and count >= 10, (count, len(mt))
    err = np.abs(np.array(corners, np.float64) - truth).max()
    assert err <= ACCURACY_PX, (err, corners, truth)


# ---- CPU: the library ------------------------------------------------------------------------------------------------
HEADER = os.path.join(ROOT, "include", "grayskull_homography.h")


def _declarations():
    txt = open(HEADER).read()
    txt = txt[txt.rindex('extern "C" {'):]
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return {m.group(2): (m.group(1).strip().split("\n")[-1].strip(), [a.strip() for a in m.group(3).split(",") if a.strip() != "void"])
            for m in re.finditer(r"([\w\s\*]+?)\b(gs_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", txt)}


def test_companion_exports_exactly_its_header():
    from grayskull_b200 import build, homography
    build.build()
    declared = sorted(_declarations())
    assert len(declared) == 3 and sorted(homography.SIGNATURES) == declared
    nm = subprocess.run(["nm", "-D", "--defined-only", homography.LIB_PATH], capture_output=True, text=True,
                        check=True).stdout
    assert sorted(ln.split()[-1] for ln in nm.splitlines() if " T " in ln) == declared
    needed = subprocess.run(["readelf", "-d", homography.LIB_PATH], capture_output=True, text=True, check=True).stdout
    assert "libgrayskull_b200" not in needed
    assert homography.lib().gs_b200_homography_last_error() == b"no error"


def test_main_library_exports_nothing_of_it():
    from grayskull_b200 import _lib
    main = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True,
                          check=True).stdout
    assert "homography" not in main
    assert not any(k in ("gsb::k_find", "gsb::k_quads") for k in L.sass_functions())


def test_ctypes_table_matches_the_header():
    from grayskull_b200 import homography
    want_of = {"double": C.c_double, "size_t": C.c_size_t}
    for name, (ret, args) in _declarations().items():
        res, argtypes = homography.SIGNATURES[name]
        assert res is {"int": C.c_int}.get(ret, C.c_char_p), name
        assert len(argtypes) == len(args), name
        for a, t in zip(args, argtypes):
            words = [w for w in a.replace("*", " * ").split() if w != "const"]
            kind = " ".join(words[:-1]) if "*" not in a else words[0]
            if "*" in a or kind == "gs_b200_stream":
                want = C.c_void_p
            elif kind == "unsigned long long":
                want = C.c_ulonglong
            else:
                want = want_of.get(kind, C.c_uint)
            assert t is want, (name, a)


def test_header_compiles_as_c99(tmp_path):
    for first in ("", '#include "grayskull_b200.h"\n', '#include "grayskull_group.h"\n'):
        src = tmp_path / "t.c"
        src.write_text(first + '#include "grayskull_homography.h"\n'
                       'int main(void) { struct gs_point p = {0, 0}; struct gs_match m = {0, 0, 0};\n'
                       '  return gs_b200_homography_last_error() == 0 && p.x == 2 && m.idx1 == 1; }\n')
        r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-fsyntax-only",
                            "-I", os.path.join(ROOT, "include"), str(src)], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    assert not re.match(r"grayskull_b200.*\.h$", "grayskull_homography.h")


def test_every_companion_kernel_is_sm90a_and_has_a_row():
    from grayskull_b200 import homography
    tool = L.cuda_tool("cuobjdump")
    if tool is None:
        pytest.skip("cuobjdump not found")
    listing = subprocess.run([tool, "-sass", homography.LIB_PATH], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for cubin in re.split(r"^\s*(?=code for sm_\w+\s*$)", listing, flags=re.M)[1:]:
        arch, *parts = re.split(r"^\s*Function : (\S+)\s*$", cubin, flags=re.M)
        for name in L.demangle(parts[0::2]):
            funcs[L.kernel_id(name)] = arch.strip().splitlines()[0]
    assert set(funcs) == set(KERNELS)
    assert all(arch == "code for sm_90a" for arch in funcs.values())


def test_launches_go_through_the_companions_helper():
    d = os.path.join(ROOT, "grayskull_b200", "homography")
    text = {f: open(os.path.join(d, f)).read() for f in sorted(os.listdir(d))}
    sites = [(f, m.start()) for f, t in text.items() for m in re.finditer(r"<<<", t)]
    assert len(sites) == 1
    f, at = sites[0]
    assert text[f].rindex("static int launch(", 0, at) < at < text[f].index("cudaGetLastError")
    assert text[f].count("cudaGetLastError") == 1
    from grayskull_b200 import build
    assert not set(build.HOMOGRAPHY_SOURCES) & set(build.SOURCES)


def test_companion_object_makes_no_blocking_runtime_call():
    from grayskull_b200 import build
    nm = shutil.which("nm")
    if nm is None:
        pytest.skip("nm not found")
    blocking = re.compile(r"^(cudaMemcpy|cudaMemcpyToSymbol|cudaMemset|cudaMemcpy2D|cudaDeviceSynchronize|"
                          r"cudaStreamSynchronize|cudaEventSynchronize|cudaMalloc\w*|cudaFree\w*|cudaStreamCreate\w*|"
                          r"cudaStreamDestroy|cudaMemcpyAsync|cudaMemsetAsync)$")
    for s in build.HOMOGRAPHY_SOURCES:
        o = os.path.join(build.OBJ, s.replace(".cu", ".o"))
        syms = [ln.split()[-1] for ln in subprocess.run([nm, "-u", o], capture_output=True, text=True,
                                                         check=True).stdout.splitlines()]
        assert "cudaGetLastError" in syms
        assert not [x for x in syms if blocking.match(x)], syms


def _run_py(expr):
    code = ("import ctypes as C, sys; sys.path.insert(0, %r); from grayskull_b200 import homography; "
            "L = homography.lib(); P = C.c_void_p(4096); rc = %s; print('rc', rc); "
            "print(L.gs_b200_homography_last_error())")
    return subprocess.run([sys.executable, "-c", code % (ROOT, expr)], capture_output=True, text=True, timeout=120)


FIND = "L.gs_b200_find_homography_batch(%s, P, 4, P, P, 4, P, P, 4, %d, %s, 0, %s, %s, P, None, None)"
QUADS = "L.gs_b200_homography_quads_batch(%s, P, %d, %s, 5, 5, 9, 9, P, P, None)"


def test_empty_batch_missing_pointer_and_bad_arguments_without_a_gpu():
    for call in (FIND % ("None", 0, "1024", "3.0", "None"), QUADS % ("None", 0, "10")):
        ok = _run_py(call)
        assert ok.returncode == 0 and "rc 0" in ok.stdout, (ok.stdout, ok.stderr)
    for call in (FIND % ("None", 2, "1024", "3.0", "P"), FIND % ("P", 2, "1024", "3.0", "None"),
                 QUADS % ("None", 2, "10")):
        bad = _run_py(call)
        assert bad.returncode != 0 and "Assertion failed: " in bad.stderr, (call, bad.stderr)
    # refused before anything is enqueued
    for thr in ("float('nan')", "-1.0", "0.0", "-0.0", "float('inf')", "-float('inf')"):
        r = _run_py(FIND % ("P", 2, "1024", thr, "P"))
        assert r.returncode == 0 and "rc 1" in r.stdout and "threshold" in r.stdout, (thr, r.stdout, r.stderr)
    for hyp in ("0", "65537", "0xFFFFFFFF"):
        r = _run_py(FIND % ("P", 2, hyp, "3.0", "P"))
        assert r.returncode == 0 and "rc 1" in r.stdout and "hypotheses" in r.stdout, (hyp, r.stdout, r.stderr)
    for mi in ("0", "3"):
        r = _run_py(QUADS % ("P", 2, mi))
        assert r.returncode == 0 and "rc 1" in r.stdout and "min_inliers" in r.stdout, (mi, r.stdout, r.stderr)
    r = _run_py(QUADS.replace("5, 5, 9, 9", "0, 5, 9, 9") % ("P", 2, "10"))
    assert "rc 1" in r.stdout and "empty" in r.stdout, r.stdout


# ---- GPU -------------------------------------------------------------------------------------------------------------
def hlib():
    from grayskull_b200 import homography
    return homography.lib()


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()


def _s():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


class Case:
    """one find call: k1 (n, s1) KP, n1, k2 (n, s2) KP, n2, mt (n, ms) MATCH, mc; into poisoned H / inliers / records"""

    def __init__(self, k1, n1, k2, n2, mt, mc, hypotheses=64, seed=0, threshold=3.0):
        self.k1, self.n1, self.k2, self.n2, self.mt, self.mc = k1, n1, k2, n2, mt, mc
        self.hyp, self.seed, self.thr = hypotheses, seed, threshold
        self.n, self.ms = mt.shape

    def buffers(self, off=0, records=True):
        n = self.n
        self.r1 = Region(self.k1.nbytes, 4 * off, self.k1, seed=1)
        self.r2 = Region(self.k2.nbytes, 4 * off, self.k2, seed=2)
        self.rm = Region(self.mt.nbytes, 4 * off, self.mt, seed=3)
        self.c1 = Region(4 * n, 4 * off, np.asarray(self.n1, np.uint32), seed=4)
        self.c2 = Region(4 * n, 4 * off, np.asarray(self.n2, np.uint32), seed=5)
        self.cm = Region(4 * n, 4 * off, np.asarray(self.mc, np.uint32), seed=6)
        self.H = Region(72 * n, 8 * off, seed=7)
        self.inl = Region(4 * n, 4 * off, seed=8)
        self.rec = Region(12 * n * self.ms, 4 * off, seed=9) if records else None
        return self

    def call(self, s=None):
        return hlib().gs_b200_find_homography_batch(
            self.r1.ptr, self.c1.ptr, self.k1.shape[1], self.r2.ptr, self.c2.ptr, self.k2.shape[1], self.rm.ptr,
            self.cm.ptr, self.ms, self.n, self.hyp, self.seed, self.thr, self.H.ptr, self.inl.ptr,
            self.rec.ptr if self.rec else None, _s() if s is None else s)

    def check(self, what, frames=None):
        gH = self.H.read(what).view(np.uint64).reshape(self.n, 9)
        gi = self.inl.read(what).view(np.uint32)
        gr = self.rec.read(what).view(MATCH).reshape(self.n, self.ms) if self.rec else None
        rb = self.rec.before().view(MATCH).reshape(self.n, self.ms) if self.rec else None
        want = model_batch(self.k1, self.n1, self.k2, self.n2, self.mt, self.mc, self.hyp, self.seed, self.thr, frames)
        for f, (H, count, recs) in want.items():
            wH = np.array(H, np.float64).view(np.uint64)
            assert np.array_equal(gH[f], wH), "%s: frame %d: H %s, want %s" % (what, f, gH[f].view(np.float64), H)
            assert gi[f] == count, "%s: frame %d: %d inliers, want %d" % (what, f, gi[f], count)
            if gr is not None:
                q = len(recs)
                assert gr[f, :q].tobytes() == self.mt[f, recs].tobytes(), "%s: frame %d records" % (what, f)
                assert gr[f, q:].tobytes() == rb[f, q:].tobytes(), "%s: frame %d wrote past its count" % (what, f)
        return want


def synthetic(n, mstride, seed, outliers, m=None, extras=True):
    """per frame a random projective map and up to m correspondences (mstride if None), `outliers` of them off it, and
    some records that are not correspondences; random counts around the list lengths"""
    rng = np.random.default_rng(seed)
    m = mstride if m is None else m
    k1, k2 = np.zeros((n, m + 2), KP), np.zeros((n, m + 2), KP)
    mt = np.zeros((n, mstride), MATCH)
    for f in range(n):
        a = rng.uniform(0.7, 1.3)
        th = rng.uniform(-0.5, 0.5)
        Ht = [a * math.cos(th), -a * math.sin(th), rng.uniform(0, 300), a * math.sin(th), a * math.cos(th),
              rng.uniform(0, 300), rng.uniform(-2e-4, 2e-4), rng.uniform(-2e-4, 2e-4), 1.0]
        x, y = rng.integers(0, 640, m), rng.integers(0, 480, m)
        X, Y = np.zeros(m, np.int64), np.zeros(m, np.int64)
        for i in range(m):
            u, v = project(Ht, x[i], y[i])
            X[i], Y[i] = int(round(u)), int(round(v))
        bad = rng.random(m) < outliers
        X[bad] = rng.integers(0, 1200, bad.sum())
        Y[bad] = rng.integers(0, 1000, bad.sum())
        k1[f, :m]["x"], k1[f, :m]["y"], k2[f, :m]["x"], k2[f, :m]["y"] = x, y, np.maximum(X, 0), np.maximum(Y, 0)
        k1[f, m]["x"] = COORD                                   # a keypoint past the coordinate bound
        k2[f, m + 1]["y"] = COORD + 5
        perm = rng.permutation(m)
        mt[f]["idx1"] = np.resize(perm, mstride)
        mt[f]["idx2"] = mt[f]["idx1"]
        mt[f]["distance"] = rng.integers(0, 60, mstride)
        if extras and mstride > 8:
            at = rng.choice(mstride, max(1, mstride // 50), replace=False)
            mt[f]["idx1"][at[0::3]] = m                        # the out-of-bounds keypoint
            mt[f]["idx2"][at[1::3]] = m + 1
            mt[f]["idx1"][at[2::3]] = m + 2 + rng.integers(0, 5, len(at[2::3]))   # past the count
    n1 = np.full(n, m + 2, np.uint32)
    n2 = (m + 2 + rng.integers(-1, 3, n)).astype(np.uint32)
    mc = (mstride + rng.integers(-max(1, mstride // 10), 3, n)).clip(0).astype(np.uint32)
    return k1, n1, k2, n2, mt, mc


@pytest.mark.gpu
@pytest.mark.parametrize("mstride,hyp", [(4, 1024), (300, 1), (300, 1024), (300, 65536), (65536, 64)])
def test_synthetic_lists_match_the_model(lib, witness, mstride, hyp):
    outliers = (0.1, 0.5, 0.9)
    parts = [synthetic(1, mstride, 40 + i, o, m=None if mstride < 1000 else 3000) for i, o in enumerate(outliers)]
    k1, n1, k2, n2, mt, mc = (np.concatenate([p[i] for p in parts]) for i in range(6))
    if mstride == 4:
        mc[1] = 3                                               # m < 4
    c = Case(k1, n1, k2, n2, mt, mc, hypotheses=hyp, seed=hyp)
    frames = [0] if hyp == 65536 else None                      # the model's 65536 solves take a while

    def run():
        c.buffers()
        rc, seen = traced(lambda: c.call())
        assert rc == 0, hlib().gs_b200_homography_last_error()
        want = c.check("mstride %d, %d hypotheses" % (mstride, hyp), frames)
        if mstride == 300 and hyp > 1:
            assert all(v[1] >= 4 for v in want.values())
        return seen

    witnessed(witness, run, ["gsb::k_find"], "find")


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["offset", "no-records", "seeds"])
def test_layouts_match_the_model(lib, layout):
    k1, n1, k2, n2, mt, mc = synthetic(4, 120, 50, 0.4)
    for seed in ((0, 2 ** 64 - 1, 12345) if layout == "seeds" else (7,)):
        c = Case(k1, n1, k2, n2, mt, mc, hypotheses=300, seed=seed, threshold=2.0)
        c.buffers(off=3 if layout == "offset" else 0, records=layout != "no-records")
        assert c.call() == 0
        c.check("%s seed %d" % (layout, seed))


@pytest.mark.gpu
def test_hand_built_lists_on_the_device(lib):
    """the CPU cases' lists, one frame each, through the device"""
    cases = [planted([1, 0, 37, 0, 1, 12, 0, 0, 1], 60, 40, 1)[0], planted([2, 1, 100, 1, 3, 50, 0, 0, 1], 30, 30, 2)[0],
             [(10 * i, 20 * i, 10 * i + 5, 20 * i + 7) for i in range(12)],
             [(x, y, 500 - x, y) for x, y in ((0, 0), (100, 0), (0, 100), (100, 100), (50, 20), (20, 70))],
             [(5, 5, 6, 6)] * 10, [(0, 0, 10, 0), (100, 0, 110, 0), (0, 100, 10, 100)],
             [(0, 0, 13, 24), (500, 0, 513, 24), (0, 500, 13, 524), (500, 500, 513, 524), (250, 250, 263, 274)]]
    ms = max(len(x) for x in cases)
    n = len(cases)
    k1, k2, mt = np.zeros((n, ms), KP), np.zeros((n, ms), KP), np.zeros((n, ms), MATCH)
    for f, pairs in enumerate(cases):
        a, b, r = lists(pairs)
        k1[f, :len(a)], k2[f, :len(b)], mt[f, :len(r)] = a, b, r
    cnt = np.array([len(x) for x in cases], np.uint32)
    for thr in (3.0, 5.0, 0.5):
        c = Case(k1, cnt, k2, cnt, mt, cnt, hypotheses=200, threshold=thr).buffers()
        assert c.call() == 0
        c.check("hand-built threshold %g" % thr)


@pytest.mark.gpu
def test_batches_above_the_grid_limit(lib):
    n = 65536 + 3
    k1, n1, k2, n2, mt, mc = synthetic(64, 8, 60, 0.3, extras=False)
    rep = lambda a: np.ascontiguousarray(np.resize(a, (n,) + a.shape[1:]))   # noqa: E731
    k1, n1, k2, n2, mt, mc = (rep(a) for a in (k1, n1, k2, n2, mt, mc))
    mc[::7] = 3
    c = Case(k1, n1, k2, n2, mt, mc, hypotheses=16).buffers()
    assert c.call() == 0
    c.check("65539 frames", frames=list(range(70)) + list(range(n - 70, n)))


@pytest.mark.gpu
def test_quads_match_the_model(lib):
    import torch
    rng = np.random.default_rng(70)
    n = 4000
    H = rng.normal(0, 1, (n, 9)) * np.array([1, 0.3, 200, 0.3, 1, 200, 1e-3, 1e-3, 1])
    H[:, 8] = 1.0
    H[::5, 6:8] *= 10                                           # more frames with w <= 0 at a corner
    H[::11] = 0.0
    H[3, 2] = np.nan
    H[4, 0] = np.inf
    H[5] = [1.0, 0.0, 10.5, 0.0, 1.0, 11.5, 0.0, 0.0, 1.0]       # half-way corners
    inl = rng.integers(0, 30, n).astype(np.uint32)
    for tw, th, sw, sh, mi in ((200, 160, 512, 384, 10), (1, 1, 1, 1, 4), (640, 480, 300, 200, 25)):
        rH = Region(72 * n, 8, H, seed=11)
        ri = Region(4 * n, 4, inl, seed=12)
        rc, rf = Region(32 * n, 4, seed=13), Region(n, 1, seed=14)
        rcode, seen = traced(lambda: hlib().gs_b200_homography_quads_batch(rH.ptr, ri.ptr, n, mi, tw, th, sw, sh,
                                                                           rc.ptr, rf.ptr, _s()))
        assert rcode == 0
        gc = rc.read("quads").view(np.uint32).reshape(n, 4, 2)
        gf = rf.read("quads")
        for f in range(n):
            corners, found = model_quad([float(v) for v in H[f]], int(inl[f]), mi, tw, th, sw, sh)
            assert gf[f] == found and gc[f].tolist() == [list(p) for p in corners], (f, H[f], gc[f], corners)
        assert 0 < gf.sum() < n
    torch.cuda.synchronize()


# ---- GPU: the device's own ORB lists ---------------------------------------------------------------------------------
def device_lists(tpl, scenes, stride=2500, mm=300):
    """pyramid ORB of the template (once per frame) and of the scenes, then match_orb, all on the device -> numpy lists"""
    import torch
    from grayskull_b200 import api, pyramid
    n = len(scenes)
    tk, tc, _, _ = pyramid.orb_pyramid_batch(torch.from_numpy(np.stack([tpl] * n)).cuda(), stride, 20)
    sk, sc, _, _ = pyramid.orb_pyramid_batch(torch.from_numpy(np.stack(scenes)).cuda(), stride, 20)
    mt, mc = api.match_orb_batch(tk, tc, sk, sc, mm, 60.0)
    torch.cuda.synchronize()
    kp = lambda t: np.ascontiguousarray(t.cpu().numpy()).view(KP).reshape(n, -1)   # noqa: E731
    u = lambda t: t.cpu().numpy().view(np.uint32)                                    # noqa: E731
    return (kp(tk), u(tc), kp(sk), u(sc), np.ascontiguousarray(mt.cpu().numpy()).view(MATCH).reshape(n, mm), u(mc),
            (tk, tc, sk, sc, mt, mc))


@pytest.mark.gpu
def test_device_orb_lists_match_the_model_and_find_the_template(lib):
    import torch
    from grayskull_b200 import homography
    scenes, truths = [], []
    tpl = None
    for p in PARALLELOGRAMS:
        _, tpl, scene, truth = accuracy_scene(p)
        scenes.append(scene), truths.append(truth)
    scenes.append(L.natural_like(SCENE[0], SCENE[1], 77))      # the template is not there
    k1, n1, k2, n2, mt, mc, dev = device_lists(tpl, scenes)
    c = Case(k1, n1, k2, n2, mt, mc, hypotheses=1024, seed=0, threshold=3.0).buffers()
    assert c.call() == 0
    want = c.check("device ORB lists")
    # the Python binding gives the same, and the quads lie at the truth
    H, inl, rec = homography.find_homography_batch(*dev)
    corners, found = homography.homography_quads_batch(H, inl, tpl.shape[1], tpl.shape[0], SCENE[0], SCENE[1])
    torch.cuda.synchronize()
    for f in range(len(scenes)):
        assert np.array_equal(H[f].cpu().numpy().reshape(9).view(np.uint64), np.array(want[f][0]).view(np.uint64))
        q = len(want[f][2])
        assert int(inl[f]) == want[f][1] and rec[f, :q].cpu().numpy().tobytes() == mt[f, want[f][2]].tobytes()
        mq = model_quad(want[f][0], want[f][1], 10, tpl.shape[1], tpl.shape[0], SCENE[0], SCENE[1])
        assert corners[f].cpu().numpy().tolist() == [list(p) for p in mq[0]] and int(found[f]) == mq[1]
        if f < len(truths):
            assert mq[1] and np.abs(np.array(mq[0], np.float64) - truths[f]).max() <= ACCURACY_PX, (f, mq, truths[f])


# ---- GPU: streams ----------------------------------------------------------------------------------------------------
def _sleep(s, cycles):
    import torch
    with torch.cuda.stream(s):
        torch.cuda._sleep(int(cycles))


@pytest.mark.gpu
def test_ordered_behind_a_sleeping_stream_without_a_host_wait(lib):
    import torch
    k1, n1, k2, n2, mt, mc = synthetic(3, 200, 80, 0.5)
    c = Case(k1, n1, k2, n2, mt, mc, hypotheses=256).buffers()
    s, u = torch.cuda.Stream(), torch.cuda.Stream()
    real = _dev(mt)
    with torch.cuda.stream(s):
        c.rm.t[c.rm.off:c.rm.off + c.rm.nbytes].zero_()
    assert c.call(C.c_void_p(s.cuda_stream)) == 0           # warm, on zeroed records
    torch.cuda.synchronize()
    H0 = torch.from_numpy(c.H.host).cuda()
    _sleep(u, 400_000_000)
    _sleep(s, 200_000_000)
    with torch.cuda.stream(s):
        c.rm.t[c.rm.off:c.rm.off + c.rm.nbytes].copy_(real)
        c.H.t.copy_(H0)
    assert c.call(C.c_void_p(s.cuda_stream)) == 0
    s_done, u_done = s.query(), u.query()
    torch.cuda.synchronize()
    assert not s_done and not u_done, "the call waited for its stream or for the device"
    c.check("behind a sleep")


@pytest.mark.gpu
def test_two_streams_at_once(lib):
    import torch
    s0, s1 = torch.cuda.Stream(), torch.cuda.Stream()
    cases = [(Case(*synthetic(3, 150, seed, 0.3 + 0.1 * (seed % 4)), hypotheses=128, seed=seed).buffers(), st)
             for seed, st in ((81, s0), (82, s1), (83, s0), (84, s1))]
    _sleep(s1, 50_000_000)
    for c, st in cases:
        assert c.call(C.c_void_p(st.cuda_stream)) == 0
    torch.cuda.synchronize()
    for c, _ in cases:
        c.check("two streams")


@pytest.mark.gpu
def test_graph_capture_and_replay_on_new_inputs(lib):
    import torch
    k1, n1, k2, n2, mt, mc = synthetic(3, 250, 90, 0.5)
    c = Case(k1, n1, k2, n2, mt, mc, hypotheses=512).buffers()
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        assert c.call(C.c_void_p(s.cuda_stream)) == 0
    for seed in (91, 92):
        fk1, fn1, fk2, fn2, fmt, fmc = synthetic(3, 250, seed, 0.6)
        with torch.cuda.stream(s):
            for r, a in ((c.r1, fk1), (c.r2, fk2), (c.rm, fmt), (c.c1, fn1), (c.c2, fn2), (c.cm, fmc)):
                r.t[r.off:r.off + r.nbytes].copy_(_dev(a))
            c.H.t.copy_(torch.from_numpy(c.H.host).cuda())
            c.rec.t.copy_(torch.from_numpy(c.rec.host).cuda())   # poisoned again: slots past the count stay so
            g.replay()
        s.synchronize()
        c.k1, c.n1, c.k2, c.n2, c.mt, c.mc = fk1, fn1, fk2, fn2, fmt, fmc
        for r, a in ((c.r1, fk1), (c.r2, fk2), (c.rm, fmt), (c.c1, fn1), (c.c2, fn2), (c.cm, fmc)):
            r.host[r.off:r.off + r.nbytes] = np.frombuffer(np.ascontiguousarray(a).tobytes(), np.uint8)
        c.check("replay %d" % seed)


# ---- GPU: the chain and the CLI --------------------------------------------------------------------------------------
def _pgm(path, a):
    h, w = a.shape
    path.write_bytes(b"P5\n%d %d\n255\n" % (w, h) + a.tobytes())
    return str(path)


def _read_pgm(path):
    data = open(path, "rb").read()
    m = re.match(rb"P5\s+(\d+)\s+(\d+)\s+255\s", data)
    w, h = int(m.group(1)), int(m.group(2))
    return np.frombuffer(data[m.end():], np.uint8).reshape(h, w)


@pytest.mark.gpu
def test_gsb_magick_find_matches_the_library_chain(lib, tmp_path):
    """find:T:W:H prints the orb stage's lines and the find lines, and writes, byte for byte, the warp of the library
    chain orb -> match -> find -> quads -> perspective_correct; orb: prints the same orb lines"""
    import torch
    from grayskull_b200 import api, build, homography
    exe = os.path.join(os.path.dirname(build.LIB), "gsb_magick")
    scenes = []
    tpl = None
    for p in PARALLELOGRAMS:
        _, tpl, scene, _ = accuracy_scene(p)
        scenes.append(scene)
    scenes.append(L.natural_like(SCENE[0], SCENE[1], 77))
    d = tmp_path / "dir:with:colons"
    d.mkdir()
    tp = _pgm(d / "template.pgm", tpl)
    ins = [_pgm(tmp_path / ("in%d.pgm" % f), a) for f, a in enumerate(scenes)]
    dw, dh = 180, 150
    r = subprocess.run([exe, "find:%s:%d:%d" % (tp, dw, dh), str(tmp_path / "o_")] + ins, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    ro = subprocess.run([exe, "orb:" + tp, str(tmp_path / "p_")] + ins, capture_output=True, text=True, timeout=600)
    assert ro.returncode == 0, ro.stderr
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("frame ")]
    n = len(scenes)
    assert lines[:n] == [ln for ln in ro.stdout.splitlines() if ln.startswith("frame ")]
    # the library chain, on the orb verb's lists (which the orb stage reproduces) at the stage's strides
    k1, k2, mt = np.zeros((n, 2500), KP), np.zeros((n, 2500), KP), np.zeros((n, 300), MATCH)
    n1, n2, mc = (np.zeros(n, np.uint32) for _ in range(3))
    for f, s in enumerate(scenes):
        kt, ks, m = orb_lists(tpl, s)
        k1[f, :len(kt)], k2[f, :len(ks)], mt[f, :len(m)] = kt, ks, m
        n1[f], n2[f], mc[f] = len(kt), len(ks), len(m)
        assert lines[f] == "frame %d: Template: %d keypoints, Scene: %d keypoints, Matches: %d" % (f, len(kt), len(ks),
                                                                                                  len(m))
    t = lambda a, w: torch.from_numpy(np.ascontiguousarray(a).view(np.int32).reshape(n, -1, w)).cuda()   # noqa: E731
    c = lambda a: torch.from_numpy(a.view(np.int32)).cuda()                                               # noqa: E731
    H, inl, _ = homography.find_homography_batch(t(k1, 12), c(n1), t(k2, 12), c(n2), t(mt, 3), c(mc), 1024, 0, 3.0)
    corners, found = homography.homography_quads_batch(H, inl, tpl.shape[1], tpl.shape[0], SCENE[0], SCENE[1], 10)
    src = torch.from_numpy(np.stack(scenes)).cuda()
    warped = api.perspective_correct_batch(src, dw, dh, corners).cpu().numpy()
    inl, corners, found = inl.cpu().numpy(), corners.cpu().numpy(), found.cpu().numpy()
    assert found[:3].all() and not found[3]
    for f in range(n):
        out = tmp_path / ("o_%04d.pgm" % f)
        if found[f]:
            q = " ".join(str(int(v)) for v in corners[f].reshape(-1))
            assert lines[n + f] == "frame %d: found, %d inliers, quad %s" % (f, inl[f], q), lines
            assert np.array_equal(_read_pgm(out), warped[f]), f
        else:
            assert lines[n + f] == "frame %d: not found, %d inliers" % (f, inl[f]), lines
            assert not out.exists() and ("frame %d: template not found" % f) in r.stderr
    # and the chain's result is the model's
    for f, (Hm, cm, _) in model_batch(k1, n1, k2, n2, mt, mc, 1024, 0, 3.0).items():
        assert np.array_equal(H[f].cpu().numpy().reshape(9).view(np.uint64), np.array(Hm).view(np.uint64))
        assert inl[f] == cm
