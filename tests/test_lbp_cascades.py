"""gs_lbp_detect / gs_lbp_window on synthetic cascades built to expose what the frontalface cascade cannot.

frontalface has a square 24 x 24 window, 8 subset words per weak classifier, 20 stages of 3-10 weaks, features that
never leave their window and leaves of order 0.5-0.9.  The cascades here break each of those in turn:

  tall / wide      16 x 40 and 40 x 16 windows: any width / height transposition in the scale table, the tile plan,
                   the feature geometry or the emitted rects
  partial          weak_num_subsets in {0, 1, 3, 7, 8}; the words past nsub are all ones, so an ignored bound votes
  long1 / long2    stages of 0, 1, 2, 5, 9, 17, 32, 33, 64 and 65 weaks, as stage 0 and after stage 4: every lane
                   count P of k_lbp_scan3's flat (window, weak) mode and stages of 1-3 chunks of 32
  short1 / short2  1 and 2 stages: stage-group layouts with one and two groups
  order            leaves of +-2^24, +-1, +-0.75 and +-2^-10: fp32 stage sums that round differently in any other order
  overshoot        features that leave their window by 1-3 px to the right and bottom (the guarded kernels), on frames
                   where every corner a scanned window touches is still inside the table
  huge             a 12 x 64 window whose largest scale is taller than a TMA box (255 rows)

Every cascade has a feature at the window's origin and one that fills it to its bottom-right corner, and its weaks
share features and subset words.  Stage thresholds are calibrated on the test frames with a numpy model of the
reference: each is an actual stage sum of the windows still alive there (near the 40th percentile), so each stage
kills windows, some windows pass with sum == threshold exactly, and every frame keeps hits.

  * CPU: the model against the oracle (oracle/gs_oracle.c) and the compiled reference, every cascade, scale factors
    1.1 and 1.25, steps 1-4, max_rects that truncates mid-scale; the calibration and definedness properties; and the
    model's mutants (reversed or pairwise stage sums, nsub ignored, window transposed, `<=` for `<`, corners beyond
    the window read as 0), each of which must change the hits of the cascade built to catch it.
  * GPU: every cascade through every scan kernel that can take it, bit-exact against the oracle, each path witnessed
    under torch.profiler (tests/_gpu.py); k_lbp_window_one at ~500 positions per cascade; and the plan
    cache (keyed by the cascade's contents) across cascades that differ in one threshold or one subset bit, and across
    in-place edits of one cascade.
"""
import functools
import os

import numpy as np
import pytest

import _libs as L
from _gpu import O, Region, lib, stream, traced, witness, witnessed  # noqa: F401

F32 = np.float32
CAL = dict(sf=1.25, mn=1.0, step=2)        # the ladder the thresholds are calibrated on (max_scale per case)
BIG_MR = 1 << 18                          # above every hit count of the tests: no truncation


# ---- the model: gs_lbp_window / gs_lbp_detect (reference grayskull.h:790-835) in numpy ---------------------------
def ladder(win_w, win_h, iw, ih, sf, mn, mx):
    """the reference's scales: scale *= scale_factor in fp32, (int)(window * scale), stop when a window leaves the
    frame -> [(scale, win_w, win_h)]"""
    out, s = [], F32(mn)
    assert F32(sf) > 1
    while s <= F32(mx):
        ww, wh = int(F32(win_w) * s), int(F32(win_h) * s)
        if ww > iw or wh > ih:
            break
        out.append((s, ww, wh))
        s = F32(s * F32(sf))
    return out


def scaled_features(a, s):
    """(int)(feature * scale) with the reference's `< 1 -> 1` clamp of the cell size -> (nfeatures, 4) int64"""
    f = (a["features"].reshape(-1, 4).astype(F32) * F32(s)).astype(np.int64)
    f[:, 2:] = np.maximum(f[:, 2:], 1)
    return f


class Frame:
    """an 8-bit image and its cell sums.  box(fw, fh)[y, x] is the int64 sum of img[y:y+fh, x:x+fw], added up
    pixel row by pixel row (no integral table); the corner table is only for the `window_zero` mutant"""

    def __init__(self, img):
        self.img = np.ascontiguousarray(img)
        self.h, self.w = img.shape
        self._box = {}
        self._corner = None

    def box(self, fw, fh):
        if (fw, fh) not in self._box:
            a = self.img.astype(np.int64)
            r = sum(a[:, dx:self.w - fw + 1 + dx] for dx in range(fw))
            self._box[(fw, fh)] = sum(r[dy:self.h - fh + 1 + dy] for dy in range(fh))
        return self._box[(fw, fh)]

    def corners(self):
        """P[y + 1, x + 1] = sum of img[:y+1, :x+1]; row and column 0 are the x == -1 / y == -1 corners"""
        if self._corner is None:
            self._corner = np.zeros((self.h + 1, self.w + 1), np.int64)
            self._corner[1:, 1:] = self.img.astype(np.int64).cumsum(0).cumsum(1)
        return self._corner


def lbp_codes(frame, feat, xs, ys, zero_beyond=None):
    """gs_lbp_code (reference :769-783) of one scaled feature at the windows (xs, ys).  zero_beyond = (win_w, win_h):
    the mutant that reads every lattice corner right of or below the window as 0"""
    fx, fy, fw, fh = (int(v) for v in feat)
    if zero_beyond is None:
        B = frame.box(fw, fh)
        cell = [[B[ys + fy + j * fh, xs + fx + i * fw] for i in range(3)] for j in range(3)]
    else:
        P = frame.corners()

        def corner(i, j):
            rx, ry = fx - 1 + i * fw, fy - 1 + j * fh
            if rx >= zero_beyond[0] or ry >= zero_beyond[1]:
                return 0
            return P[ys + ry + 1, xs + rx + 1]
        cell = [[corner(i + 1, j + 1) + corner(i, j) - corner(i + 1, j) - corner(i, j + 1) for i in range(3)]
                for j in range(3)]
    m = cell[1][1]
    ring = (cell[0][0], cell[0][1], cell[0][2], cell[1][2], cell[2][2], cell[2][1], cell[2][0], cell[1][0])
    code = np.zeros(len(xs), np.int64)
    for b, v in zip(range(7, -1, -1), ring):
        code |= (np.asarray(v) >= m).astype(np.int64) << b
    return code


def stage_sum(frame, a, feats, k, xs, ys, mutant=None, win=None):
    """the fp32 sum of stage k's votes at the windows (xs, ys), added in weak order (reference :797-809)"""
    start, n = int(a["stage_weak_start"][k]), int(a["stage_nweaks"][k])
    sub = a["subsets"].view(np.uint32)
    codes, votes = {}, []
    for wi in range(start, start + n):
        fi = int(a["weak_feature_idx"][wi])
        if fi not in codes:
            codes[fi] = lbp_codes(frame, feats[fi], xs, ys, win if mutant == "window_zero" else None)
        code = codes[fi]
        idx, bit = code >> 5, code & 31
        off, nsub = int(a["weak_subset_offset"][wi]), int(a["weak_num_subsets"][wi])
        word = sub[np.minimum(off + idx, len(sub) - 1)] if len(sub) else np.zeros(len(xs), np.uint32)
        match = ((word.astype(np.int64) >> bit) & 1).astype(bool)
        if mutant != "nsub":
            match &= idx < nsub
        votes.append(np.where(match, a["weak_left_val"][wi], a["weak_right_val"][wi]).astype(F32))
    if mutant == "reverse":
        votes = votes[::-1]
    if mutant == "pairwise":
        while len(votes) > 1:
            votes = [votes[i] + votes[i + 1] if i + 1 < len(votes) else votes[i] for i in range(0, len(votes), 2)]
    total = np.zeros(len(xs), F32)
    for v in votes:
        total = total + v
    return total


def walk(frame, a, feats, win, xs, ys, mutant=None):
    """the cascade at every window (xs, ys) of one scale -> (stages passed per window, stage sums with NaN where the
    window was already dead)"""
    nst = len(a["stage_nweaks"])
    thr = a["stage_threshold"]
    alive = np.arange(len(xs))
    depth = np.zeros(len(xs), np.int64)
    sums = np.full((nst, len(xs)), np.nan, F32)
    for k in range(nst):
        if not len(alive):
            break
        s = stage_sum(frame, a, feats, k, xs[alive], ys[alive], mutant, win)
        sums[k, alive] = s
        alive = alive[s > thr[k]] if mutant == "le" else alive[~(s < thr[k])]
        depth[alive] += 1
    return depth, sums


def grid(iw, ih, ww, wh, step):
    """window origins of one scale in the reference's order (y, then x)"""
    nx, ny = (iw - ww) // step + 1, (ih - wh) // step + 1
    ys, xs = np.divmod(np.arange(nx * ny), nx)
    return xs * step, ys * step, nx, ny


def transposed(a):
    t = dict(a)
    t["window"] = a["window"][::-1].copy()
    t["features"] = np.ascontiguousarray(a["features"].reshape(-1, 4)[:, [1, 0, 3, 2]]).ravel()
    return t


def model_detect(frame, a, sf, mn, mx, step, mutant=None):
    """gs_lbp_detect without max_rects (its truncation is a prefix) -> (rects, per-scale walks)"""
    if mutant == "transpose":
        a = transposed(a)
    nst = len(a["stage_nweaks"])
    rects, per = [], []
    for s, ww, wh in ladder(int(a["window"][0]), int(a["window"][1]), frame.w, frame.h, sf, mn, mx):
        xs, ys, nx, ny = grid(frame.w, frame.h, ww, wh, step)
        depth, sums = walk(frame, a, scaled_features(a, s), (ww, wh), xs, ys, mutant)
        hit = depth == nst
        r = np.zeros(int(hit.sum()), L.RECT_DTYPE)
        r["x"], r["y"], r["w"], r["h"] = xs[hit], ys[hit], ww, wh
        rects.append(r)
        per.append(dict(scale=s, ww=ww, wh=wh, nx=nx, ny=ny, depth=depth, sums=sums))
    return (np.concatenate(rects) if rects else np.zeros(0, L.RECT_DTYPE)), per


def max_corner(a, iw, ih, sf, mn, mx, step):
    """the largest lattice corner (x, y) any window of the scan reads, over every scale, for the referenced features"""
    used = np.unique(a["weak_feature_idx"])
    bx = by = -1
    for s, ww, wh in ladder(int(a["window"][0]), int(a["window"][1]), iw, ih, sf, mn, mx):
        f = scaled_features(a, s)[used]
        if not len(f):
            continue
        bx = max(bx, (iw - ww) // step * step + int((f[:, 0] + 3 * f[:, 2]).max()) - 1)
        by = max(by, (ih - wh) // step * step + int((f[:, 1] + 3 * f[:, 3]).max()) - 1)
    return bx, by


# ---- the synthetic cascades --------------------------------------------------------------------------------------
def _words(rng, n):
    return rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32).view(np.int32)


def synth(win, stage_n, seed, nsub_set=(8,), leaves=(0.25, 0.5, 0.75, 1.0), over=(), nfeat=14):
    """a cascade with the given stage sizes.  Features 0 and 1 sit at the window's origin and fill it to its
    bottom-right corner; `over` adds features whose lattice leaves the window by (dx, dy) px.  Stage 0 references all
    of those; the other weaks pick features and subset blocks at random, so both are shared.  Thresholds are 0 until
    calibrate()."""
    rng = np.random.default_rng(seed)
    ww, wh = win
    cw, ch = max(1, ww // 6), max(1, wh // 6)
    feats = [(0, 0, cw + 1, ch + 1), (ww - 3 * cw, wh - 3 * ch, cw, ch)]
    for dx, dy in over:
        fw, fh = int(rng.integers(1, 4)), int(rng.integers(1, 4))
        feats.append((ww + dx - 3 * fw, wh + dy - 3 * fh, fw, fh))
    special = len(feats)
    while len(feats) < nfeat:
        fw, fh = int(rng.integers(1, max(2, ww // 4))), int(rng.integers(1, max(2, wh // 4)))
        feats.append((int(rng.integers(0, ww - 3 * fw + 1)), int(rng.integers(0, wh - 3 * fh + 1)), fw, fh))
    nw = int(sum(stage_n))
    assert stage_n[0] >= min(special, nw)
    wf = rng.integers(0, len(feats), nw)
    wf[:min(special, nw)] = np.arange(min(special, nw))
    nsub = rng.choice(np.array(nsub_set), nw)
    # subset blocks of 8 words, shared by weaks with the same nsub; the words past nsub are all ones
    offs, words = np.zeros(nw, np.int64), []
    for v in sorted(set(nsub.tolist())):
        who = np.flatnonzero(nsub == v)
        nblk = max(1, (len(who) + 1) // 2)
        first = len(words) // 8
        for _ in range(nblk):
            words += list(_words(rng, v)) + [-1] * (8 - v)
        offs[who] = 8 * (first + rng.integers(0, nblk, len(who)))
    lv = np.array(leaves, F32)
    left = (rng.choice(lv, nw) * rng.choice(np.array([-1, 1], F32), nw)).astype(F32)
    right = (rng.choice(lv, nw) * rng.choice(np.array([-1, 1], F32), nw)).astype(F32)
    sn = np.array(stage_n, np.uint16)
    return {"window": np.array(win, np.uint16), "features": np.array(feats, np.int8).ravel(),
            "weak_feature_idx": wf.astype(np.uint16), "weak_left_val": left, "weak_right_val": right,
            "weak_subset_offset": offs.astype(np.uint16), "weak_num_subsets": nsub.astype(np.uint16),
            "subsets": np.array(words, np.int32), "stage_weak_start": (np.cumsum(sn) - sn).astype(np.uint16),
            "stage_nweaks": sn, "stage_threshold": np.zeros(len(sn), F32)}


ORDER_LEAVES = (2.0 ** 24, 1.0, 0.75, 2.0 ** -10)
# name: (window, stage sizes, frame w x h, max_scale, synth options)
SPECS = {
    "tall": ((16, 40), [4, 5, 6, 6, 7, 8], (160, 120), 3.0, {}),
    "wide": ((40, 16), [4, 5, 6, 6, 7, 8], (160, 120), 3.0, {}),
    "partial": ((20, 20), [8, 7, 7, 6, 8], (160, 120), 4.0, dict(nsub_set=(0, 1, 3, 7, 8))),
    "long1": ((24, 20), [65, 2, 3, 2, 3, 64, 33, 17, 9, 0], (160, 120), 3.0, {}),
    "long2": ((20, 24), [33, 3, 2, 3, 2, 32, 65, 5, 2, 1], (160, 120), 3.0, {}),
    "short1": ((18, 18), [6], (160, 120), 4.0, {}),
    "short2": ((18, 18), [4, 5], (160, 120), 4.0, {}),
    "order": ((20, 20), [6, 6, 6, 6], (160, 120), 4.0, dict(leaves=ORDER_LEAVES)),
    "overshoot": ((20, 20), [7, 5, 5, 5], (167, 127), 2.0, dict(over=((1, 1), (2, 3), (3, 2), (3, 0), (0, 3)))),
    "huge": ((12, 64), [5, 5, 5, 5], (96, 320), 5.0, {}),
}
# stage indices of long1 / long2 placed after stage 4, where warps of k_lbp_scan3 are in the flat mode
FLAT_STAGES = {"long1": range(5, 10), "long2": range(5, 10)}
# overshoot's features leave the window by up to 3 px at every scale, so a scan of it is defined only where the last
# window of a row (and of a column) leaves that much room: (iw - win_w) % step >= the overshoot.  At step 4 that holds
# for one scale at a time, on frames sized for it: (scale_factor, scale, step, w, h); the scales are ladder values
OVER_SCANS = [(1.1, 0, 4, 167, 127), (1.1, 1, 4, 168, 125), (1.1, 2, 4, 167, 127), (1.25, 1, 4, 168, 128)]
MUTANTS = {"order": ("reverse", "pairwise"), "partial": ("nsub",), "tall": ("transpose",), "wide": ("transpose",),
           "overshoot": ("window_zero",)}


def synthetic_frames(w, h, seed=40):
    """a padded lena crop, natural_like and uniform noise"""
    lena = np.load(os.path.join(L.ROOT, "tests", "golden", "lena_golden.npz"))["lena"]
    a = np.pad(lena, ((0, max(0, h - 128)), (0, max(0, w - 128))), mode="edge")[:h, :w]
    b = L.natural_like(w, h, seed + w + h)
    c = np.random.default_rng(seed + w * h).integers(0, 256, (h, w), dtype=np.uint8)
    return np.ascontiguousarray(np.stack([a, b, c]))


@functools.lru_cache(maxsize=None)
def frames_at(w, h):
    imgs = synthetic_frames(w, h)
    return imgs, [Frame(f) for f in imgs]


def scan_windows(a, frame, sf, mn, mx, step):
    """(scale, win_w, win_h, xs, ys, nx, ny) of every scale of a scan"""
    for s, ww, wh in ladder(int(a["window"][0]), int(a["window"][1]), frame.w, frame.h, sf, mn, mx):
        xs, ys, nx, ny = grid(frame.w, frame.h, ww, wh, step)
        yield s, ww, wh, xs, ys, nx, ny


def calibrate(a, scans, q=0.4):
    """stage by stage: the threshold is the stage sum at quantile q of the windows alive there, over every frame of
    the calibration scans"""
    nst = len(a["stage_nweaks"])
    states = []
    for sf, mn, mx, step, w, h in scans:
        for fr in frames_at(w, h)[1]:
            for s, _, _, xs, ys, _, _ in scan_windows(a, fr, sf, mn, mx, step):
                states.append([fr, scaled_features(a, s), xs, ys])
    for k in range(nst):
        sums = [stage_sum(fr, a, f, k, xs, ys) for fr, f, xs, ys in states]
        allv = np.sort(np.concatenate(sums))
        t = allv[int(q * len(allv))] if len(allv) else F32(0)
        if len(allv) and t == allv[0] and allv[-1] > t:       # few distinct sums: the next one up kills some
            t = allv[allv > t][0]
        a["stage_threshold"][k] = t
        for st, s in zip(states, sums):
            keep = ~(s < a["stage_threshold"][k])
            st[2], st[3] = st[2][keep], st[3][keep]
    return a


class Case:
    """a calibrated synthetic cascade and the scans it is tested with: (scale_factor, min_scale, max_scale, step,
    frame w, frame h)"""

    def __init__(self, name):
        win, stage_n, (w, h), mx, opts = SPECS[name]
        self.name, self.w, self.h, self.mx = name, w, h, mx
        self.imgs, self.frames = frames_at(w, h)
        if name == "overshoot":
            self.cal_scans = []
            for sf, i, step, fw, fh in OVER_SCANS:
                s = float(ladder(win[0], win[1], fw, fh, sf, 1.0, mx)[i][0])
                self.cal_scans.append((sf, s, s, step, fw, fh))
            self.cpu_scans = self.cal_scans
        else:
            self.cal_scans = [(CAL["sf"], CAL["mn"], mx, CAL["step"], w, h)]
            self.cpu_scans = [(sf, 1.0, mx, step, w, h) for sf in (1.1, 1.25) for step in (1, 2, 3, 4)]
        self.arrays = calibrate(synth(win, stage_n, seed=sum(map(ord, name)), **opts), self.cal_scans)

    def cascade(self, arrays=None):
        from grayskull_b200._lib import HostCascade
        return HostCascade({k: v.copy() for k, v in (arrays or self.arrays).items()})


def integrals(O, imgs):
    return np.stack([L.o_integral(O, f) for f in imgs])


@functools.lru_cache(maxsize=None)
def case(name):
    return Case(name)


NAMES = list(SPECS)


# ---- CPU: calibration, definedness, model == oracle == reference, mutants ----------------------------------------
@pytest.mark.parametrize("name", NAMES)
def test_cascade_shape(name):
    cs = case(name)
    a = cs.arrays
    ww, wh = (int(v) for v in a["window"])
    f = a["features"].reshape(-1, 4).astype(np.int64)
    used = np.unique(a["weak_feature_idx"])
    assert ((f[used, 0] == 0) & (f[used, 1] == 0)).any()
    assert ((f[used, 0] + 3 * f[used, 2] == ww) & (f[used, 1] + 3 * f[used, 3] == wh)).any()
    assert len(used) < len(a["weak_feature_idx"]), "weaks share features"
    blocks = a["weak_subset_offset"][a["weak_num_subsets"] > 0]
    assert len(np.unique(blocks)) < len(blocks), "weaks share subset words"
    assert (a["weak_subset_offset"].astype(np.int64) + 8 <= len(a["subsets"])).all()
    if name == "tall" or name == "wide":
        assert (ww, wh) in ((16, 40), (40, 16))
    if name == "partial":
        assert set(a["weak_num_subsets"].tolist()) == {0, 1, 3, 7, 8}
        for off, n in zip(a["weak_subset_offset"], a["weak_num_subsets"]):
            assert (a["subsets"][off + n:off + 8] == -1).all()
    if name.startswith("long"):
        n = a["stage_nweaks"].tolist()
        assert n[0] > 32 and sorted(n[5:]) == sorted(set(n[5:]))
    if name == "long1":
        both = a["stage_nweaks"][5:].tolist() + case("long2").arrays["stage_nweaks"][5:].tolist()
        assert sorted(both) == [0, 1, 2, 5, 9, 17, 32, 33, 64, 65]
    if name == "overshoot":
        out = (f[used, 0] + 3 * f[used, 2] - ww, f[used, 1] + 3 * f[used, 3] - wh)
        assert out[0].max() == 3 and out[1].max() == 3 and (out[0] > 0).sum() >= 3 and (out[1] > 0).sum() >= 3
    if name == "huge":
        sc = ladder(ww, wh, cs.w, cs.h, 1.1, 1.0, cs.mx)
        assert max(s[2] for s in sc) > 255
        assert max(s[2] for s in ladder(ww, wh, cs.w, cs.h, CAL["sf"], CAL["mn"], cs.mx)) > 255


@pytest.mark.parametrize("name", NAMES)
def test_calibration(name):
    """on the calibration scans: every stage with weaks kills windows, some windows pass a stage with
    sum == threshold exactly, every frame keeps hits; the long stages after stage 4 are entered by some 32-window
    slots of a row with 1-8 survivors (k_lbp_scan3's flat-mode condition, lbp.cu k_lbp_scan3)"""
    cs = case(name)
    a = cs.arrays
    nst = len(a["stage_nweaks"])
    entered, passed, tie = np.zeros(nst, np.int64), np.zeros(nst, np.int64), np.zeros(nst, np.int64)
    flat = {k: 0 for k in FLAT_STAGES.get(name, ())}
    for sf, mn, mx, step, w, h in cs.cal_scans:
        for fr in frames_at(w, h)[1]:
            rects, per = model_detect(fr, a, sf, mn, mx, step)
            assert len(rects) > 0, "a frame without hits"
            for p in per:
                for k in range(nst):
                    entered[k] += (p["depth"] >= k).sum()
                    passed[k] += (p["depth"] > k).sum()
                    tie[k] += (p["sums"][k] == a["stage_threshold"][k]).sum()
                for k in flat:
                    alive = np.zeros((p["ny"], -(-p["nx"] // 32) * 32), bool)
                    alive[:, :p["nx"]] = p["depth"].reshape(p["ny"], p["nx"]) >= k
                    per_slot = alive.reshape(p["ny"], -1, 32).sum(-1)
                    flat[k] += ((per_slot >= 1) & (per_slot <= 8)).sum()
    for k in range(nst):
        if a["stage_nweaks"][k]:
            assert passed[k] < entered[k], "stage %d kills nothing" % k
        else:
            assert passed[k] == entered[k] and a["stage_threshold"][k] == 0
        assert tie[k] > 0, "no window with sum == threshold at stage %d" % k
    assert all(flat.values()), flat


@pytest.mark.parametrize("name", NAMES)
def test_scans_are_defined(name):
    """the largest corner any scanned window reads lies inside the table, on every scan the tests run; overshoot's
    features do leave their window at each of its scans"""
    cs = case(name)
    a = cs.arrays
    scans = set(cs.cpu_scans) | set(gpu_scans(cs))
    for sf, mn, mx, step, w, h in scans:
        bx, by = max_corner(a, w, h, sf, mn, mx, step)
        assert 0 <= bx < w and 0 <= by < h, (sf, mn, step, w, h, bx, by)
        if name == "overshoot":
            for s, ww, wh in ladder(20, 20, w, h, sf, mn, mx):
                f = scaled_features(a, s)[np.unique(a["weak_feature_idx"])]
                assert (f[:, 0] + 3 * f[:, 2]).max() > ww and (f[:, 1] + 3 * f[:, 3]).max() > wh, (sf, s)


def _detect_raw(lib, fn, cas, ii, mr, sf, mn, mx, step):
    r = np.zeros(max(mr, 1), L.RECT_DTYPE)
    n = getattr(lib, fn)(cas.ptr, L.ptr(ii), ii.shape[1], ii.shape[0], L.ptr(r), mr, sf, mn, mx, step)
    return r[:n]


def _mid_scale_cut(rects):
    """a max_rects that stops the scan inside a scale: the middle hit of the scale with the most hits (0: none)"""
    wh = [(int(r["w"]), int(r["h"])) for r in rects]
    if not wh:
        return 0
    best = max(set(wh), key=wh.count)
    first, cnt = wh.index(best), wh.count(best)
    return first + cnt // 2 if cnt >= 2 else 0


@pytest.mark.parametrize("name", NAMES)
def test_model_oracle_reference_detect(name, O):
    """gs_lbp_detect: the model, the oracle and (when built) the reference agree on every scan and frame, also with
    a max_rects that ends the scan inside a scale"""
    cs = case(name)
    cas = cs.cascade()
    libs = [(O, "gso_lbp_detect")] + ([(L.ref(), "gs_lbp_detect")] if L.have_ref() else [])
    cuts = 0
    for sf, mn, mx, step, w, h in cs.cpu_scans:
        imgs, frames = frames_at(w, h)
        ii = integrals(O, imgs)
        for i, fr in enumerate(frames):
            want, _ = model_detect(fr, cs.arrays, sf, mn, mx, step)
            assert len(want) < BIG_MR
            mr = _mid_scale_cut(want)
            cuts += mr > 0
            for lib, fn in libs:
                tag = (fn, sf, mn, step, i, len(want))
                assert _detect_raw(lib, fn, cas, ii[i], BIG_MR, sf, mn, mx, step).tobytes() == want.tobytes(), tag
                if mr:
                    assert _detect_raw(lib, fn, cas, ii[i], mr, sf, mn, mx, step).tobytes() == want[:mr].tobytes(), tag
    assert cuts > 0


def window_positions(cs, rng, n):
    """(x, y, scale) for single-window calls on cs's frames: ladder and off-ladder scales, random positions (some
    whose window does not fit the frame) and a quarter at hits of the calibration scan; only positions whose corners
    stay inside the table"""
    a = cs.arrays
    ww0, wh0 = (int(v) for v in a["window"])
    scales = [s for s, _, _ in ladder(ww0, wh0, cs.w, cs.h, 1.1, 1.0, cs.mx)] + [F32(1.37), F32(2.05)]
    used = np.unique(a["weak_feature_idx"])
    sf, mn, mx, step, w, h = cs.cal_scans[0]
    assert (w, h) == (cs.w, cs.h)
    hits, per = model_detect(cs.frames[1], a, sf, mn, mx, step)
    scale_of = {(p["ww"], p["wh"]): p["scale"] for p in per}
    out = [(int(r["x"]), int(r["y"]), scale_of[(int(r["w"]), int(r["h"]))])
           for r in hits[rng.permutation(len(hits))[:n // 4]]]
    while len(out) < n:
        s = scales[int(rng.integers(0, len(scales)))]
        ww, wh = int(F32(ww0) * s), int(F32(wh0) * s)
        if ww > cs.w or wh > cs.h:
            continue
        x, y = int(rng.integers(0, cs.w - ww + 3)), int(rng.integers(0, cs.h - wh + 3))
        f = scaled_features(a, s)[used]
        fits = x + ww <= cs.w and y + wh <= cs.h
        if fits and (x + (f[:, 0] + 3 * f[:, 2]).max() > cs.w or y + (f[:, 1] + 3 * f[:, 3]).max() > cs.h):
            continue
        out.append((x, y, s))
    return out


def model_windows(cs, frame, pos):
    """gs_lbp_window at each (x, y, scale) through the model"""
    a = cs.arrays
    nst = len(a["stage_nweaks"])
    out = np.zeros(len(pos), np.uint32)
    for s in sorted({p[2] for p in pos}):
        ww, wh = int(F32(a["window"][0]) * s), int(F32(a["window"][1]) * s)
        idx = [i for i, p in enumerate(pos) if p[2] == s and p[0] + ww <= frame.w and p[1] + wh <= frame.h]
        if idx:
            xs, ys = np.array([pos[i][0] for i in idx]), np.array([pos[i][1] for i in idx])
            out[idx] = walk(frame, a, scaled_features(a, s), (ww, wh), xs, ys)[0] == nst
    return out


@pytest.mark.parametrize("name", NAMES)
def test_model_oracle_reference_window(name, O):
    cs = case(name)
    cas = cs.cascade()
    libs = [(O, "gso_lbp_window")] + ([(L.ref(), "gs_lbp_window")] if L.have_ref() else [])
    ii = integrals(O, cs.imgs)
    pos = window_positions(cs, np.random.default_rng(7), 200)
    for i, fr in enumerate(cs.frames):
        want = model_windows(cs, fr, pos)
        assert i != 1 or 0 < want.sum() < len(want)          # a quarter of the positions are hits in frame 1
        for lib, fn in libs:
            got = [getattr(lib, fn)(cas.ptr, L.ptr(ii[i]), cs.w, cs.h, x, y, s) for x, y, s in pos]
            assert np.array_equal(got, want), (fn, i)


@pytest.mark.parametrize("name,mutant", [(n, m) for n in NAMES for m in MUTANTS.get(n, ()) + ("le",)])
def test_mutant_changes_hits(name, mutant):
    """each probed property decides hits on the test frames: the model with it broken gives another hit list"""
    cs = case(name)
    differ = 0
    for sf, mn, mx, step, w, h in cs.cal_scans:
        for fr in frames_at(w, h)[1]:
            want, _ = model_detect(fr, cs.arrays, sf, mn, mx, step)
            got, _ = model_detect(fr, cs.arrays, sf, mn, mx, step, mutant)
            differ += got.tobytes() != want.tobytes()
    assert differ, "the %s mutant gives the same hits: the %s cascade does not probe it" % (mutant, name)


# ---- GPU ---------------------------------------------------------------------------------------------------------
def gpu_detect(lib, cas, ii, mr, sf, mn, mx, step, off=0, env=None, generic=False):
    """gs_b200_lbp_detect_batch on the (n, h, w) tables at byte offset `off`, under torch.profiler -> (rects per
    frame, launched kernels)"""
    from grayskull_b200 import _lib
    n, h, w = ii.shape
    I = Region(ii.nbytes, off, ii, seed=3)
    RR, N = Region(16 * n * mr, 0, seed=4), Region(4 * n, 0, seed=5)
    env = env or {}
    os.environ.update(env)
    if generic:
        lib.gs_b200_force_generic(1)
    try:
        rc, seen = traced(lambda: lib.gs_b200_lbp_detect_batch(cas.ptr, I.ptr, w, h, n, RR.ptr, N.ptr, mr, sf, mn, mx,
                                                              step, stream()))
    finally:
        for k in env:
            os.environ.pop(k, None)
        if generic:
            lib.gs_b200_force_generic(0)
    _lib.check(rc, "lbp_detect_batch")
    counts = N.read("counts").view(np.uint32)
    rects = RR.read("rects").view(np.uint32).reshape(n, mr, 4)
    I.read("ii")
    return [np.ascontiguousarray(rects[i, :counts[i]]) for i in range(n)], seen


SCAN2, SCAN3 = "gsb::k_lbp_scan2", "gsb::k_lbp_scan3<%d>"
# path: (step, table byte offset, frame width added, environment, force_generic, kernel the path must launch)
PATHS = {
    "scan3_512": (2, 0, 0, {"GS_B200_LBP_BIG": "0"}, False, SCAN3 % 512),
    "scan3_1024": (2, 0, 0, {"GS_B200_LBP_BIG": "1"}, False, SCAN3 % 1024),
    "step1": (1, 0, 0, {}, False, SCAN2),
    "step3": (3, 0, 0, {}, False, SCAN2),
    "offset4": (2, 4, 0, {}, False, SCAN2),
    "ragged": (2, 0, 2, {}, False, SCAN2),                      # iw % 8 != 0
    "generic": (2, 0, 0, {}, True, SCAN2),
    "chunk1": (2, 0, 0, {"GS_B200_LBP_CHUNK_FRAMES": "1"}, False, SCAN3 % 512),
    "big_tables": (3, 0, 0, {}, False, "gsb::k_lbp_scan<false>"),   # + unreferenced features: tables over 160 KB
    "guarded": (4, 0, 0, {}, False, "gsb::k_lbp_scan<true>"),     # overshoot: features leave their window
    "whole_ladder_scan2": (2, 0, 0, {}, False, SCAN2),           # huge: one scale's tile cannot be a TMA box
}
GPU_CASES = ([(n, p) for n in NAMES if n not in ("overshoot", "huge") for p in list(PATHS)[:9]] +
             [("overshoot", "guarded"), ("huge", "whole_ladder_scan2"), ("huge", "step1"), ("huge", "big_tables")])


def gpu_scans(cs, path=None):
    """the (scale_factor, min_scale, max_scale, step, w, h) scans a GPU case runs"""
    paths = [path] if path else [p for n, p in GPU_CASES if n == cs.name]
    out = []
    for p in paths:
        step, _, dw, _, _, _ = PATHS[p]
        if cs.name == "overshoot":
            out += cs.cal_scans
        else:
            out.append((1.1, 1.0, cs.mx, step, cs.w + dw, cs.h))
    return out


def padded(a, nfeatures=5200):
    """the same cascade with unreferenced copies of feature 0 appended: k_lbp_scan2's tables pass 160 KB"""
    p = dict(a)
    f = a["features"].reshape(-1, 4)
    p["features"] = np.concatenate([f, np.tile(f[:1], (nfeatures - len(f), 1))]).ravel()
    return p


@pytest.mark.gpu
@pytest.mark.parametrize("name,path", GPU_CASES, ids=["%s-%s" % c for c in GPU_CASES])
def test_detect_path(lib, O, witness, name, path):
    """3 frames per batch through the path's kernel, counts and rects bit-exact against the oracle"""
    cs = case(name)
    _, off, _, env, generic, kernel = PATHS[path]
    a = padded(cs.arrays) if path == "big_tables" else cs.arrays
    cas = cs.cascade(a)
    scans = []
    for sf, mn, mx, step, w, h in gpu_scans(cs, path):
        assert PATHS[path][2] == 0 or w % 8
        ii = integrals(O, frames_at(w, h)[0])
        scans.append((sf, mn, mx, step, ii, [L.o_detect(O, cas, t, BIG_MR, sf, mn, mx, step) for t in ii]))
    assert sum(len(r) for *_, want in scans for r in want) > 0

    def run():
        seen = set()
        for sf, mn, mx, step, ii, want in scans:
            got, s = gpu_detect(lib, cas, ii, BIG_MR, sf, mn, mx, step, off, env, generic)
            for i in range(len(ii)):
                assert got[i].tobytes() == want[i].tobytes(), (sf, mn, step, i, len(got[i]), len(want[i]))
            seen |= s
        return seen
    witnessed(witness, run, [kernel], "%s-%s" % (name, path))


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_window_one(lib, O, witness, name):
    """single-window gs_lbp_window (k_lbp_window_one) against gso_lbp_window, 500 positions per cascade and frame"""
    cs = case(name)
    cas = cs.cascade()
    ii = integrals(O, cs.imgs)
    pos = window_positions(cs, np.random.default_rng(11), 500)
    hits = 0
    for i in range(len(ii)):
        t = np.ascontiguousarray(ii[i])
        for x, y, s in pos:
            want = O.gso_lbp_window(cas.ptr, L.ptr(t), cs.w, cs.h, x, y, s)
            assert lib.gs_lbp_window(cas.ptr, L.ptr(t), cs.w, cs.h, x, y, s) == want, (i, x, y, s)
            hits += want
    assert 0 < hits < len(ii) * len(pos)
    x, y, s = pos[0]                                   # a hit of the calibration scan
    t = np.ascontiguousarray(ii[1])
    want = O.gso_lbp_window(cas.ptr, L.ptr(t), cs.w, cs.h, x, y, s)
    assert want == 1

    def run():
        got, seen = traced(lambda: lib.gs_lbp_window(cas.ptr, L.ptr(t), cs.w, cs.h, x, y, s))
        assert got == want
        return seen
    witnessed(witness, run, ["gsb::k_lbp_window_one"], "%s window" % name)


def _flip_that_matters(O, cs, ii):
    """(word, bit): one subset bit of a stage-0 weak whose flip changes the hits of frame 0"""
    a = cs.arrays
    sf, mn, mx, step, _, _ = cs.cal_scans[0]
    base = L.o_detect(O, cs.cascade(), ii[0], BIG_MR, sf, mn, mx, step)
    for r in base[:20]:
        f = scaled_features(a, next(s for s, ww, wh in ladder(*a["window"], *ii.shape[1:][::-1], sf, mn, mx)
                                    if (ww, wh) == (r["w"], r["h"])))
        for wi in range(int(a["stage_nweaks"][0])):
            xy = np.array([int(r["x"])]), np.array([int(r["y"])])
            code = int(lbp_codes(cs.frames[0], f[a["weak_feature_idx"][wi]], *xy)[0])
            if code >> 5 >= a["weak_num_subsets"][wi]:
                continue
            word, bit = int(a["weak_subset_offset"][wi]) + (code >> 5), code & 31
            b = {k: v.copy() for k, v in a.items()}
            b["subsets"][word] ^= np.uint32(1 << bit).view(np.int32)
            if L.o_detect(O, cs.cascade(b), ii[0], BIG_MR, sf, mn, mx, step).tobytes() != base.tobytes():
                return word, bit
    raise AssertionError("no subset bit of stage 0 changes the hits")


@pytest.mark.gpu
@pytest.mark.parametrize("step", [2, 3])
def test_plan_cache_follows_the_cascade(lib, O, step):
    """cascades that differ in one threshold, then in one subset bit, alternate; then one cascade is edited in place
    (same struct, same pointer) between calls.  Every call's hits are those of the cascade as it is at that call."""
    cs = case("short2")
    ii = integrals(O, cs.imgs)
    a = cs.arrays
    b = {k: v.copy() for k, v in a.items()}
    b["stage_threshold"][-1] = np.nextafter(a["stage_threshold"][-1], F32(np.inf))   # kills the sum == thr windows
    word, bit = _flip_that_matters(O, cs, ii)
    c = {k: v.copy() for k, v in a.items()}
    c["subsets"][word] ^= np.uint32(1 << bit).view(np.int32)
    A, B, Cc = cs.cascade(a), cs.cascade(b), cs.cascade(c)
    args = (BIG_MR, CAL["sf"], CAL["mn"], cs.mx, step)

    def check(cas):
        got, _ = gpu_detect(lib, cas, ii, *args)
        want = [L.o_detect(O, cas, ii[i], *args) for i in range(len(ii))]
        for i in range(len(ii)):
            assert got[i].tobytes() == want[i].tobytes(), (i, len(got[i]), len(want[i]))
        return b"".join(w.tobytes() for w in want)

    ra, rb, rc = check(A), check(B), check(Cc)
    assert ra != rb and ra != rc
    for cas in (A, B, A, Cc, A, B, Cc):
        check(cas)
    X = cs.cascade(a)
    assert check(X) == ra
    X.arrays["stage_threshold"][-1] = b["stage_threshold"][-1]
    assert check(X) == rb
    X.arrays["stage_threshold"][-1] = a["stage_threshold"][-1]
    assert check(X) == ra
    X.arrays["subsets"][word] = c["subsets"][word]
    assert check(X) == rc
    X.arrays["subsets"][word] = a["subsets"][word]
    assert check(X) == ra
