"""gs_lbp_detect's scale ladder and scan parameters at their extremes: scale_factor, min_scale, max_scale, step and
max_rects.

The host builds the ladder once per plan (lbp.cu build_scales) and every scan kernel, the emit kernel,
gs_b200_lbp_window_count and the single-image gs_lbp_detect read that one table, so a wrong table is invisible to a
test that compares one kernel with another.  Here the ladder is checked against an fp32 model of the reference's loop
(grayskull.h:819-821) and the hits against the oracle, on:

  long        scale_factor 1.0001 and 1.00005 on 64 x 64 frames: 9,000 - 13,000 scales, with hits past the 4097th
  boundary    scales where (int)(window * s) or a feature's (int)(f * s) lands on an integer, the float just below,
              and scales where the fp32 product rounds up onto an integer that the exact product stays below (a
              double-precision ladder gives another window there); one ladder passes through such a scale
  small       min_scale 0.3, 0.5, 0.75: windows smaller than the cascade's, cells clamped to 1 px, features that
              leave their window (the guarded k_lbp_scan<true> for the real cascade)
  ends        max_scale < min_scale, == min_scale, +inf, NaN; scale_factor NaN; a first window larger than the frame
  step        1, 3, 7, iw - win_w and iw + 1, on widths with and without iw % 8 == 0
  max_rects   the hits of the first k scales of frame 0, one less, one more, and 1
  window      single gs_lbp_window calls at scales < 1 and at the boundary scales

each with the real cascade and a synthetic one (an 18 x 22 window with 1-px cells at its bottom-right corner).

  * CPU: the model's window count equals gs_b200_lbp_window_count; every case reaches the condition it is named for;
    the oracle equals the compiled reference (oracle/_ref) on every case, where the reference is defined (every
    lattice corner inside the table) and terminates.
  * GPU: gs_b200_lbp_detect_batch on 3 frames (lena crops and a natural frame) and the single-image gs_lbp_detect on
    each, bit-exact against the oracle, rects past the count untouched, each case's scan kernel witnessed under
    torch.profiler; a ladder longer than the library's limit is an error, not a shorter list.
"""
import functools
import os

import numpy as np
import pytest

import _libs as L
from _gpu import Region, lib, stream, traced, witness, witnessed  # noqa: F401

F32 = np.float32
O = L.oracle()
needs_ref = pytest.mark.skipif(not L.have_ref(), reason="oracle/_ref not built")
BIG_MR = 1 << 20                # above every hit count here: no truncation
OLD_CAP = 4097                  # the scales the device scanned before the ladder lost its cut-off
MAX_SCALES = 65536              # lbp.cu LBP_MAX_SCALES
INF, NAN = float("inf"), float("nan")


# ---- the model: the reference's ladder in fp32 (grayskull.h:819-821) ----------------------------------------------
def ladder(win_w, win_h, iw, ih, sf, mn, mx, limit=None):
    """the reference's scales: scale *= scale_factor in fp32, (int)(window * scale), stop when a window leaves the
    frame -> [(scale, win_w, win_h)].  A NaN scale_factor ends after one scale, as in the reference."""
    out, s = [], F32(mn)
    while s <= F32(mx):
        ww, wh = int(F32(win_w) * s), int(F32(win_h) * s)
        if ww > iw or wh > ih:
            break
        out.append((s, ww, wh))
        if limit is not None and len(out) > limit:
            break
        s = F32(s * F32(sf))
    return out


def scaled_features(a, s):
    """(int)(feature * scale) with the reference's `< 1 -> 1` clamp of the cell size -> (nfeatures, 4) int64"""
    f = (a["features"].reshape(-1, 4).astype(F32) * F32(s)).astype(np.int64)
    f[:, 2:] = np.maximum(f[:, 2:], 1)
    return f


def window_count(a, iw, ih, sf, mn, mx, step):
    return sum(((iw - ww) // step + 1) * ((ih - wh) // step + 1)
               for _, ww, wh in ladder(int(a["window"][0]), int(a["window"][1]), iw, ih, sf, mn, mx))


def max_corner(a, iw, ih, sf, mn, mx, step):
    """the largest lattice corner (x, y) any window of the scan reads, over every scale, for the referenced features"""
    used = np.unique(a["weak_feature_idx"])
    bx = by = -1
    for s, ww, wh in ladder(int(a["window"][0]), int(a["window"][1]), iw, ih, sf, mn, mx):
        f = scaled_features(a, s)[used]
        bx = max(bx, (iw - ww) // step * step + int((f[:, 0] + 3 * f[:, 2]).max()) - 1)
        by = max(by, (ih - wh) // step * step + int((f[:, 1] + 3 * f[:, 3]).max()) - 1)
    return bx, by


def leaves_window(a, s, ww, wh):
    f = scaled_features(a, s)
    return bool(((f[:, 0] + 3 * f[:, 2] > ww) | (f[:, 1] + 3 * f[:, 3] > wh)).any())


def rounds_up(v, s):
    """(int)(v * s) in fp32 lands on an integer that the exact product stays below"""
    return int(F32(v) * F32(s)) != int(np.floor(float(v) * float(s)))


# ---- cascades and frames ----------------------------------------------------------------------------------------
def synthetic():
    """an 18 x 22 window, 3 stages of 3 weaks with +-1 leaves (a window passes a stage with 2 matches of 3).  Feature 1
    is a 1 x 1 cell lattice at the bottom-right corner: below scale 1 its cells clamp to 1 px and it leaves the
    window.  Feature 0 fills the window."""
    rng = np.random.default_rng(2024)
    feats = [(0, 0, 6, 7), (15, 19, 1, 1), (5, 3, 3, 5), (9, 11, 2, 3), (2, 13, 5, 3), (11, 1, 2, 7), (7, 7, 1, 2)]
    wf = np.array([0, 1, 6, 2, 3, 1, 4, 5, 0], np.uint16)
    nw = len(wf)
    words = rng.integers(0, 1 << 32, 8 * nw, dtype=np.uint64).astype(np.uint32).view(np.int32)
    return {"window": np.array([18, 22], np.uint16), "features": np.array(feats, np.int8).ravel(),
            "weak_feature_idx": wf, "weak_left_val": np.ones(nw, F32), "weak_right_val": -np.ones(nw, F32),
            "weak_subset_offset": (8 * np.arange(nw)).astype(np.uint16), "weak_num_subsets": np.full(nw, 8, np.uint16),
            "subsets": words, "stage_weak_start": np.array([0, 3, 6], np.uint16),
            "stage_nweaks": np.array([3, 3, 3], np.uint16), "stage_threshold": np.ones(3, F32)}


def padded(a, nfeatures=5200):
    """the same cascade with unreferenced copies of feature 0 appended: k_lbp_scan2's tables pass 160 KB"""
    p = dict(a)
    f = a["features"].reshape(-1, 4)
    p["features"] = np.ascontiguousarray(np.concatenate([f, np.tile(f[:1], (nfeatures - len(f), 1))]).ravel())
    return p


@functools.lru_cache(maxsize=None)
def cascade(name):
    from grayskull_b200._lib import HostCascade, load_cascade
    if name == "synth":
        return HostCascade(synthetic())
    real = load_cascade()
    return real if name == "real" else HostCascade(padded(real.arrays))


@functools.lru_cache(maxsize=None)
def frames(w, h):
    """two lena crops around its face (lena's faces sit at scales 1.2 - 2.2 in a 64 px crop) and a natural frame"""
    lena = np.load(os.path.join(L.ROOT, "tests", "golden", "lena_golden.npz"))["lena"]
    big = np.pad(lena, ((0, 64), (0, 64)), mode="edge")
    return np.ascontiguousarray(np.stack([big[36:36 + h, 36:36 + w], L.natural_like(w, h, 77 + w + h),
                                          big[30:30 + h, 40:40 + w]]))


@functools.lru_cache(maxsize=None)
def integrals(w, h):
    return np.stack([L.o_integral(O, f) for f in frames(w, h)])


# ---- the cases ------------------------------------------------------------------------------------------------------
SCAN3, SCAN2 = "gsb::k_lbp_scan3<%d>", "gsb::k_lbp_scan2"
GUARDED, GENERIC = "gsb::k_lbp_scan<true>", "gsb::k_lbp_scan<false>"


def first_round_up(lo, hi, values):
    """the first float32 scale in [lo, hi) from a grid of k / v at which (int)(v * s) rounds up for one of `values`"""
    for v in values:
        for k in range(int(np.ceil(lo * v)), int(hi * v) + 1):
            for s in (F32(k / v), np.nextafter(F32(k / v), F32(0)), np.nextafter(F32(k / v), F32(INF))):
                if lo <= s < hi and rounds_up(v, s):
                    return F32(s)
    raise AssertionError("no round-up scale for %s in [%g, %g)" % (values, lo, hi))


def through(r, sf):
    """a min_scale whose fp32 ladder reaches exactly r at its second scale"""
    m = F32(F32(r) / F32(sf))
    for _ in range(64):
        p = F32(m * F32(sf))
        if p == r:
            return m
        m = np.nextafter(m, F32(INF) if p < r else F32(0))
    raise AssertionError("no min_scale with %r * %r == %r" % (m, sf, r))


def boundary_scales(name):
    """{label: scale}: a window on an integer (and the float below it), a feature on an integer (and below), the
    window and a feature rounding up onto an integer in fp32"""
    a = cascade(name).arrays
    ww = int(a["window"][0])
    fvals = sorted(set(int(v) for v in a["features"].reshape(-1, 4)[:, 2:].ravel()) - {0, 1, ww})
    s_win = F32((ww + 6) / ww)                                   # ww + 6 px exactly (30 for 24: s = 1.25)
    f = fvals[-1]
    s_feat = F32((f + 2) / f) if F32(F32(f) * F32((f + 2) / f)) == f + 2 else F32(2.0)
    return {"win_int": s_win, "win_below": np.nextafter(s_win, F32(0)), "feat_int": s_feat,
            "feat_below": np.nextafter(s_feat, F32(0)), "win_roundup": first_round_up(1.4, 2.5, [ww]),
            "feat_roundup": first_round_up(1.05, 2.5, fvals)}


def defined_frame(name, sf, mn, mx, step, w0, h0):
    """the first frame size from (w0, h0) up at which every corner the scan reads lies inside the table"""
    a = cascade(name).arrays
    w = next((w for w in range(w0, w0 + 64) if max_corner(a, w, h0 + 64, sf, mn, mx, step)[0] < w), None)
    h = next((h for h in range(h0, h0 + 64) if max_corner(a, w0 + 64, h, sf, mn, mx, step)[1] < h), None)
    assert w and h, "no defined frame for %s %s" % (name, (sf, mn, mx, step))
    return w, h


def build_cases():
    """id -> dict(name, w, h, sf, mn, mx, step, mr, env, kernel, kind)"""
    cases = {}

    def add(cid, name, w, h, sf, mn, mx, step, kernel, mr=BIG_MR, env=None, kind=None):
        cases[cid] = dict(name=name, w=w, h=h, sf=float(sf), mn=float(mn), mx=float(mx), step=step, mr=mr,
                          env=env or {}, kernel=kernel, kind=kind or cid.split("-")[0])

    for name in ("real", "synth"):
        # 1. long ladders
        add("long-%s-1.0001" % name, name, 64, 64, 1.0001, 1.0, 4.0, 2, SCAN3 % 512, env={"GS_B200_LBP_BIG": "0"})
        add("long-%s-1.00005" % name, name, 64, 64, 1.00005, 1.5, 4.0, 2, SCAN3 % 512, env={"GS_B200_LBP_BIG": "0"})
        add("long-%s-step3" % name, name, 64, 64, 1.0001, 1.2, 4.0, 3, SCAN2)
        # 2. scales on integer boundaries: single scales, then a ladder through a round-up scale
        for label, s in boundary_scales(name).items():
            add("boundary-%s-%s" % (name, label), name, 64, 64, 1.1, s, s, 1, SCAN2)
        r = boundary_scales(name)["win_roundup"]
        add("boundary-%s-ladder" % name, name, 64, 64, 1.1, through(r, 1.1), 4.0, 2, SCAN3 % 512)
        # 3. min_scale < 1: features leave their window; only frames on which every read corner is in the table
        for mn in (0.3, 0.5, 0.75):
            for sf, mx, step in ((1.25, mn, 3), (1.25, 1.2, 7)):
                w, h = defined_frame(name, sf, mn, mx, step, 61, 57)
                a = cascade(name).arrays
                unsafe = any(leaves_window(a, *sc) for sc in ladder(*a["window"], w, h, sf, mn, mx))
                add("small-%s-%g-to%g" % (name, mn, mx), name, w, h, sf, mn, mx, step, GUARDED if unsafe else SCAN2)
        # 4. ladder ends
        add("ends-%s-max_below_min" % name, name, 64, 64, 1.1, 1.5, np.nextafter(F32(1.5), F32(0)), 2, None)
        add("ends-%s-max_eq_min" % name, name, 64, 64, 1.1, 1.7, 1.7, 2, SCAN3 % 512)
        add("ends-%s-max_inf" % name, name, 64, 64, 1.1, 1.0, INF, 2, SCAN3 % 512)
        add("ends-%s-max_nan" % name, name, 64, 64, 1.1, 1.0, NAN, 2, None)
        add("ends-%s-sf_nan" % name, name, 64, 64, NAN, 1.3, 4.0, 2, SCAN3 % 512)
        add("ends-%s-window_over_frame" % name, name, 64, 64, 1.1, 3.0, 4.0, 2, None)
        # 5. step
        for w in (64, 61):
            ww = int(F32(cascade(name).arrays["window"][0]) * F32(1.0))
            for step in (1, 3, 7, w - ww, w + 1):
                add("step-%s-w%d-s%d" % (name, w, step), name, w, 60, 1.1, 1.0, 4.0, step, SCAN2)
    add("step-real-w64-s2-big", "real", 64, 64, 1.1, 1.0, 4.0, 2, SCAN3 % 1024, env={"GS_B200_LBP_BIG": "1"})
    add("step-real-w61-s2", "real", 61, 64, 1.1, 1.0, 4.0, 2, SCAN2)
    add("step-padded-w64-s3", "padded", 64, 64, 1.1, 1.0, 4.0, 3, GENERIC)
    # 6. max_rects: the hits of frame 0's first k scales, one less, one more, and 1
    for name in ("real", "synth"):
        sf, mn, mx, step = 1.1, 1.0, 4.0, 1
        cas = cascade(name)
        hits = L.o_detect(O, cas, integrals(64, 64)[0], BIG_MR, sf, mn, mx, step)
        wins = [(int(r["w"]), int(r["h"])) for r in hits]
        k = len(set(wins)) // 2
        scales = sorted(set(wins))
        exact = sum(1 for x in wins if x < scales[k]) if k else len(wins)
        for label, mr in (("exact", exact), ("less", exact - 1), ("more", exact + 1), ("one", 1)):
            add("maxrects-%s-%s" % (name, label), name, 64, 64, sf, mn, mx, step, SCAN2, mr=mr)
    return cases


CASES = build_cases()
DETECT = list(CASES)


def tables(c):
    return integrals(c["w"], c["h"])


def scales_of(c):
    a = cascade(c["name"]).arrays
    return ladder(int(a["window"][0]), int(a["window"][1]), c["w"], c["h"], c["sf"], c["mn"], c["mx"])


def oracle_detect(c, i):
    return L.o_detect(O, cascade(c["name"]), tables(c)[i], c["mr"], c["sf"], c["mn"], c["mx"], c["step"])


# ---- CPU: the model's count, the conditions, the oracle against the reference ---------------------------------------
@pytest.mark.parametrize("cid", DETECT)
def test_window_count(cid):
    """gs_b200_lbp_window_count is the fp32 model's count, the long ladders past 4097 scales included"""
    from grayskull_b200 import _lib
    c = CASES[cid]
    a = cascade(c["name"]).arrays
    want = window_count(a, c["w"], c["h"], c["sf"], c["mn"], c["mx"], c["step"])
    got = _lib.lib().gs_b200_lbp_window_count(cascade(c["name"]).ptr, c["w"], c["h"], c["sf"], c["mn"], c["mx"],
                                              c["step"])
    assert got == want, (got, want, len(scales_of(c)))


def test_window_count_past_the_limit():
    """a ladder longer than the plan's limit still has its full window count"""
    from grayskull_b200 import _lib
    cas = cascade("real")
    want = window_count(cas.arrays, 64, 64, 1.00001, 1.0, 4.0, 2)
    assert len(ladder(24, 24, 64, 64, 1.00001, 1.0, 4.0)) > MAX_SCALES
    assert _lib.lib().gs_b200_lbp_window_count(cas.ptr, 64, 64, 1.00001, 1.0, 4.0, 2) == want


def _hits_before_the_old_cap(c, i):
    """the hits of frame i in the first 4097 scales of the case's ladder"""
    sc = scales_of(c)
    cas = cascade(c["name"])
    n_upto = L.o_detect(O, cas, tables(c)[i], BIG_MR, c["sf"], c["mn"], float(sc[OLD_CAP - 1][0]), c["step"])
    return len(n_upto)


@pytest.mark.parametrize("cid", DETECT)
def test_case_reaches_its_condition(cid):
    c = CASES[cid]
    a = cascade(c["name"]).arrays
    ww0, wh0 = int(a["window"][0]), int(a["window"][1])
    sc = scales_of(c)
    kind = c["kind"]
    if kind == "long":
        assert 5000 <= len(sc) <= 15000, len(sc)
        # the first lena crop has hits past the 4097th scale
        hits = len(oracle_detect(c, 0))
        assert len(sc) > OLD_CAP and _hits_before_the_old_cap(c, 0) < hits < BIG_MR
    elif kind == "boundary":
        label = cid.split("-", 2)[2]
        s = F32(c["mn"])
        fv = set(int(v) for v in a["features"].reshape(-1, 4)[:, 2:].ravel())
        if label == "ladder":
            r = boundary_scales(c["name"])["win_roundup"]
            assert len(sc) > 2 and sc[1][0] == r and rounds_up(ww0, r)
        elif label == "win_int":
            assert float(F32(ww0) * s) == int(F32(ww0) * s) and sc[0][1] == ww0 + 6
        elif label == "win_below":
            assert sc[0][1] == ww0 + 5 and F32(np.nextafter(s, F32(INF))) == boundary_scales(c["name"])["win_int"]
        elif label in ("feat_int", "feat_below"):
            prods = [float(F32(v) * s) for v in fv - {0, 1}]
            hit = any(p == int(p) for p in prods)
            assert hit == (label == "feat_int")
        elif label == "win_roundup":
            assert rounds_up(ww0, s)
        elif label == "feat_roundup":
            assert any(rounds_up(v, s) for v in fv)
        if label != "ladder":
            assert len(sc) == 1
    elif kind == "small":
        assert F32(c["mn"]) < 1 and sc[0][1] < ww0 and sc[0][2] < wh0
        f = (a["features"].reshape(-1, 4)[:, 2:].astype(F32) * F32(c["mn"])).astype(int)
        assert (f < 1).any(), "no cell clamps to 1 px"
        assert c["name"] == "real" and c["mn"] == 0.75 or any(leaves_window(a, *t) for t in sc), "no feature leaves"
        bx, by = max_corner(a, c["w"], c["h"], c["sf"], c["mn"], c["mx"], c["step"])
        assert bx < c["w"] and by < c["h"]
    elif kind == "ends":
        label = cid.split("-", 2)[2]
        n = {"max_below_min": 0, "max_eq_min": 1, "max_nan": 0, "sf_nan": 1, "window_over_frame": 0}.get(label)
        if n is not None:
            assert len(sc) == n, (label, len(sc))
        if label == "max_inf":
            s_next = F32(sc[-1][0] * F32(c["sf"]))
            assert int(F32(ww0) * s_next) > c["w"] or int(F32(wh0) * s_next) > c["h"]
        if label == "window_over_frame":
            assert int(F32(ww0) * F32(c["mn"])) > c["w"] or int(F32(wh0) * F32(c["mn"])) > c["h"]
    elif kind == "step":
        assert c["step"] in (1, 2, 3, 7, c["w"] + 1) or c["step"] == c["w"] - sc[0][1]
        if c["step"] > c["w"]:
            assert all((c["w"] - ww) // c["step"] == 0 for _, ww, _ in sc)
    elif kind == "maxrects":
        total = len(L.o_detect(O, cascade(c["name"]), tables(c)[0], BIG_MR, c["sf"], c["mn"], c["mx"], c["step"]))
        assert 1 <= c["mr"] < total
    if c["kernel"] == GUARDED:
        assert any(leaves_window(a, s, ww, wh) for s, ww, wh in sc)
    if c["kernel"] is None:
        assert not sc


def test_hits_on_the_boundary_scales():
    """the window round-up scales and the ladder through one have hits (so a double-precision window shows)"""
    for name in ("real", "synth"):
        for label in ("win_roundup", "ladder"):
            c = CASES["boundary-%s-%s" % (name, label)]
            assert sum(len(oracle_detect(c, i)) for i in range(3)) > 0, (name, label)


def test_small_scales_have_hits():
    """the synthetic cascade hits at every scale below 1 (the real one finds no face in windows of 7 - 18 px)"""
    for k in CASES:
        if k.startswith("small-synth-"):
            c = CASES[k]
            wins = {int(r["w"]) for i in range(3) for r in oracle_detect(c, i)}
            assert wins == {ww for _, ww, _ in scales_of(c)}, (k, wins)


@needs_ref
@pytest.mark.parametrize("cid", DETECT)
def test_oracle_matches_reference(cid):
    R = L.ref()
    c = CASES[cid]
    cas = cascade(c["name"])
    for i, t in enumerate(tables(c)):
        r = np.zeros(max(c["mr"], 1), L.RECT_DTYPE)
        n = R.gs_lbp_detect(cas.ptr, L.ptr(t), c["w"], c["h"], L.ptr(r), c["mr"], c["sf"], c["mn"], c["mx"], c["step"])
        assert r[:n].tobytes() == oracle_detect(c, i).tobytes(), (i, n)


# ---- single windows -----------------------------------------------------------------------------------------------
def window_positions(name, w, h, n=160):
    """(x, y, scale) at scales < 1 and the boundary scales: random positions whose read corners lie in the table (some
    whose window does not fit), and the hits of the boundary single-scale cases"""
    a = cascade(name).arrays
    ww0, wh0 = int(a["window"][0]), int(a["window"][1])
    used = np.unique(a["weak_feature_idx"])
    scales = [F32(0.3), F32(0.5), F32(0.75), np.nextafter(F32(0.75), F32(0))] + list(boundary_scales(name).values())
    rng = np.random.default_rng(len(name) + w)
    out = []
    for label in boundary_scales(name):
        c = CASES["boundary-%s-%s" % (name, label)]
        for r in oracle_detect(c, 0)[:4]:
            out.append((int(r["x"]), int(r["y"]), F32(c["mn"])))
    while len(out) < n:
        s = scales[int(rng.integers(0, len(scales)))]
        ww, wh = int(F32(ww0) * s), int(F32(wh0) * s)
        x, y = int(rng.integers(0, w - ww + 3)), int(rng.integers(0, h - wh + 3))
        f = scaled_features(a, s)[used]
        fits = x + ww <= w and y + wh <= h
        if fits and (x + (f[:, 0] + 3 * f[:, 2]).max() > w or y + (f[:, 1] + 3 * f[:, 3]).max() > h):
            continue
        out.append((x, y, s))
    return out


@needs_ref
@pytest.mark.parametrize("name", ["real", "synth"])
def test_window_oracle_matches_reference(name):
    R = L.ref()
    cas = cascade(name)
    pos = window_positions(name, 64, 64)
    hits = 0
    for t in integrals(64, 64):
        for x, y, s in pos:
            want = O.gso_lbp_window(cas.ptr, L.ptr(t), 64, 64, x, y, s)
            assert R.gs_lbp_window(cas.ptr, L.ptr(t), 64, 64, x, y, s) == want, (x, y, s)
            hits += want
    assert 0 < hits < 3 * len(pos)


# ---- GPU ------------------------------------------------------------------------------------------------------------
def gpu_detect(lib, c):
    """gs_b200_lbp_detect_batch on the case's 3 tables under torch.profiler -> (counts, rects (n, mr, 4) u32, the rects
    buffer as it was before, launched kernels)"""
    from grayskull_b200 import _lib
    ii = tables(c)
    n, h, w = ii.shape
    mr = c["mr"]
    I = Region(ii.nbytes, 0, ii, seed=3)
    RR, N = Region(16 * n * mr, 0, seed=4), Region(4 * n, 0, seed=5)
    os.environ.update(c["env"])
    try:
        rc, seen = traced(lambda: lib.gs_b200_lbp_detect_batch(cascade(c["name"]).ptr, I.ptr, w, h, n, RR.ptr, N.ptr, mr,
                                                              c["sf"], c["mn"], c["mx"], c["step"], stream()))
    finally:
        for k in c["env"]:
            os.environ.pop(k, None)
    _lib.check(rc, "lbp_detect_batch")
    I.read("ii")
    before = RR.before().view(np.uint32).reshape(n, mr, 4)
    return N.read("counts").view(np.uint32), RR.read("rects").view(np.uint32).reshape(n, mr, 4), before, seen


@pytest.mark.gpu
@pytest.mark.parametrize("cid", DETECT)
def test_detect(lib, witness, cid):
    """3 frames through gs_b200_lbp_detect_batch and each through gs_lbp_detect: the oracle's rects, bit-exact; rects
    past the count keep their bytes"""
    c = CASES[cid]
    want = [oracle_detect(c, i) for i in range(3)]
    cas = cascade(c["name"])

    def run():
        counts, rects, before, seen = gpu_detect(lib, c)
        for i in range(3):
            assert counts[i] == len(want[i]), (i, int(counts[i]), len(want[i]))
            assert rects[i, :counts[i]].tobytes() == want[i].tobytes(), i
            assert np.array_equal(rects[i, counts[i]:], before[i, counts[i]:]), "rects past the count changed (%d)" % i
        return seen

    if c["kernel"] is None:
        run()
    else:
        witnessed(witness, run, [c["kernel"]], cid)
    for i, t in enumerate(tables(c)):
        r = np.zeros(max(c["mr"], 1), L.RECT_DTYPE)
        n = lib.gs_lbp_detect(cas.ptr, L.ptr(np.ascontiguousarray(t)), c["w"], c["h"], L.ptr(r), c["mr"], c["sf"],
                              c["mn"], c["mx"], c["step"])
        assert r[:n].tobytes() == want[i].tobytes(), ("single", i, n, len(want[i]))


@pytest.mark.gpu
def test_ladder_past_the_limit_is_an_error(lib):
    """65537 scales and more: the call fails and leaves counts and rects as they were"""
    cas = cascade("real")
    ii = integrals(64, 64)
    assert len(ladder(24, 24, 64, 64, 1.00001, 1.0, 4.0, limit=MAX_SCALES)) > MAX_SCALES
    I = Region(ii.nbytes, 0, ii, seed=3)
    RR, N = Region(16 * 3 * 64, 0, seed=4), Region(12, 0, seed=5)
    rc = lib.gs_b200_lbp_detect_batch(cas.ptr, I.ptr, 64, 64, 3, RR.ptr, N.ptr, 64, 1.00001, 1.0, 4.0, 2, stream())
    assert rc != 0
    assert b"lbp.cu" in lib.gs_b200_last_error()
    import torch
    torch.cuda.synchronize()
    assert np.array_equal(N.read("counts"), N.before()) and np.array_equal(RR.read("rects"), RR.before())


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["real", "synth"])
def test_window(lib, witness, name):
    """single gs_lbp_window calls (k_lbp_window_one) at scales < 1 and on the boundary scales"""
    cas = cascade(name)
    pos = window_positions(name, 64, 64)
    hits = 0
    for t in integrals(64, 64):
        t = np.ascontiguousarray(t)
        for x, y, s in pos:
            want = O.gso_lbp_window(cas.ptr, L.ptr(t), 64, 64, x, y, s)
            assert lib.gs_lbp_window(cas.ptr, L.ptr(t), 64, 64, x, y, s) == want, (x, y, s)
            hits += want
    assert hits > 0
    t = np.ascontiguousarray(integrals(64, 64)[0])
    x, y, s = pos[0]

    def run():
        got, seen = traced(lambda: lib.gs_lbp_window(cas.ptr, L.ptr(t), 64, 64, x, y, s))
        assert got == O.gso_lbp_window(cas.ptr, L.ptr(t), 64, 64, x, y, s) == 1
        return seen
    witnessed(witness, run, ["gsb::k_lbp_window_one"], "%s window" % name)
