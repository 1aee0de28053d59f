"""Every scalar parameter at its extremes, on each kernel that takes it.

test_dispatch_paths.py covers the geometry that picks a kernel; this suite covers the scalars several kernels take
shortcuts on, each only valid over part of the parameter's range:

  * adaptive c: k_box_tma / k_box_mid clamp c to [-256, 256] for their 16-bit lane compare; the reference's
    (int)(mean - (unsigned)c) wraps for c <= INT_MIN + 255, which launch_box routes to the literal kernels;
  * threshold / threshold_each: thresh & 0xFF and the per-frame (uint8_t)(thresh[f] + offset);
  * filter norm: k_filter3's umulhi magic divisor, taken only while a host test passes (filter.cu);
  * template width: k_match_template's u32 row sums, taken only below 66051 taps per row;
  * match_orb max_distance: the candidate threshold ceil(max_distance + 1) clamped to [0, 257];
  * radius: the fast division (r <= 63), k_box_mid / k_box_wide (r <= 120), k_box_generic beyond;
  * a 4400 x 4400 frame whose integral table wraps mod 2^32 before its faces, fed to the LBP detector;
  * the ORB candidate cap min(4 nkps, 5000) on a frame with more FAST survivors than that.

  * GPU: each case runs under torch.profiler (the launched kernels are printed as `launched ...` lines and the case's
    kernels must be among them) and every output is bit-exact against the oracle (tests/_libs.py).
  * CPU: the oracle is pinned against the compiled reference (oracle/_ref) at every new extreme value, on small
    inputs, wherever the reference terminates and is defined; the boundary values are derived from the host formulas
    the library uses.
"""
import os

import numpy as np
import pytest

import _libs as L
from _gpu import Region, frames, lib, stream, traced, witness, witnessed  # noqa: F401

INT_MIN, INT_MAX, UINT_MAX = -2 ** 31, 2 ** 31 - 1, 2 ** 32 - 1
O = L.oracle()
needs_ref = pytest.mark.skipif(not L.have_ref(), reason="oracle/_ref not built")


def _ok(rc):
    from grayskull_b200 import _lib
    _lib.check(rc, "extreme-parameter case")


def _cid(v):
    names = {INT_MIN: "INT_MIN", INT_MAX: "INT_MAX", UINT_MAX: "UINT_MAX"}
    for base, nm in ((INT_MIN, "INT_MIN"), (INT_MAX, "INT_MAX")):
        if v not in names and 0 < abs(v - base) <= 256:
            return "%s%+d" % (nm, v - base)
    return names.get(v, str(v))


# ---- a. adaptive c ---------------------------------------------------------------------------------------------------
LANE_C = 256                      # box_finish / k_box_mid clamp c to [-LANE_C, LANE_C] for the 16-bit lane compare
C_VALUES = (INT_MIN, INT_MIN + 1, INT_MIN + 100, INT_MIN + 255, INT_MIN + 256, -65536, -257, -256, -255, 0, 255, 256,
            257, INT_MAX)


def lane_c_ok(c):
    """launch_box's route: the lane compare is exact for c > INT_MIN + 255 (derived by test_lane_compare_boundary)"""
    return c > INT_MIN + LANE_C - 1


def _ref_expr(src, mean, c):
    """the reference's `int threshold = sum / count - c; src > threshold` (unsigned subtraction, then int)"""
    t = (mean.astype(np.int64) - c) % 2 ** 32
    t = np.where(t >= 2 ** 31, t - 2 ** 32, t)
    return np.where(src.astype(np.int64) > t, 255, 0)


def _lane_expr(src, mean, c):
    """k_box_tma / k_box_mid: E = src + (clamp(c) + 0x7FFF) - mean on a 16-bit lane, 255 where bit 15 is set"""
    cc = max(-LANE_C, min(LANE_C, c))
    e = src.astype(np.int64) + (cc + 0x7FFF) - mean.astype(np.int64)
    assert e.min() >= 0 and e.max() < 1 << 16          # no borrow out of or into the lane
    return np.where(e & 0x8000, 255, 0)


def test_lane_compare_boundary():
    """over every (src, mean) byte pair, the clamped lane compare equals the reference's expression exactly for
    c > INT_MIN + 255 (the c values below and the two sides of every clamp edge), and differs on 256 pairs or more
    for each c below: the range launch_box sends to k_box_wide / k_box_generic"""
    src, mean = np.meshgrid(np.arange(256), np.arange(256))
    edges = [INT_MIN + LANE_C - 1, INT_MIN + LANE_C, -LANE_C - 1, -LANE_C, LANE_C, LANE_C + 1]
    for c in sorted(set(C_VALUES) | set(edges)):
        diff = int((_ref_expr(src, mean, c) != _lane_expr(src, mean, c)).sum())
        assert (diff == 0) == lane_c_ok(c), (c, diff)
        if not lane_c_ok(c):
            assert diff >= 256, (c, diff)
    assert not lane_c_ok(INT_MIN + LANE_C - 1) and lane_c_ok(INT_MIN + LANE_C)


def _c_frames(w, h, seed):
    """random, natural_like, all 0 and all 255: both sides of mean >= c - INT_MIN occur"""
    rng = np.random.default_rng(seed)
    return np.stack([rng.integers(0, 256, (h, w), dtype=np.uint8), L.natural_like(w, h, seed),
                     np.zeros((h, w), np.uint8), np.full((h, w), 255, np.uint8)])


@needs_ref
def test_ref_adaptive_c_extremes():
    R = L.ref()
    rng = np.random.default_rng(21)
    imgs = [np.ascontiguousarray(a) for a in _c_frames(13, 9, 5)] + [rng.integers(0, 256, (h, w), dtype=np.uint8)
                                                                    for w, h in ((1, 1), (7, 3), (20, 17))]
    for a in imgs:
        h, w = a.shape
        for r in (0, 1, 2, 5, 9):
            for c in C_VALUES:
                d = np.empty_like(a); R.gs_adaptive_threshold(L.img(d), L.img(a), r, c)
                assert np.array_equal(d, L.o_adaptive(O, a, r, c)), (w, h, r, c)


def _adaptive_geoms():
    out = [("tma-r%d" % r, 272, 70, r, "gsb::k_box_tma<%d, true>" % r) for r in range(1, 8)]
    out += [("mid-tpf-r%d" % r, 272, 100, r, "gsb::k_box_mid<%d, true>" % (r & 3)) for r in (8, 9, 10, 11)]
    out += [("mid-r%d" % r, 1080, 70, r, "gsb::k_box_mid<%d, true>" % (r & 3)) for r in (5, 8)]
    out += [("wide-r15", 612, 70, 15, "gsb::k_box_wide<true>"), ("generic-r130", 100, 40, 130, "gsb::k_box_generic<true>"),
            ("single-host-r5", 272, 70, 5, "gsb::k_box_tma<5, true>")]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("c", C_VALUES, ids=_cid)
@pytest.mark.parametrize("name,w,h,r,kernel", [pytest.param(*g, id=g[0]) for g in _adaptive_geoms()])
def test_adaptive_c(lib, witness, name, w, h, r, kernel, c):
    if not lane_c_ok(c) and r <= 120:
        kernel = "gsb::k_box_wide<true>"
    fr = _c_frames(w, h, w + r)
    n = len(fr)

    def run():
        if name.startswith("single"):       # gs_adaptive_threshold on host images: staged through the workspace
            from grayskull_b200 import api
            got = np.empty_like(fr)
            seen = set()
            for i in range(n):
                d = np.empty_like(fr[i])
                _, s = traced(lambda: api.gs_adaptive_threshold(d, np.ascontiguousarray(fr[i]), r, c))
                got[i], seen = d, seen | s
        else:
            S, D = Region(fr.nbytes, 0, fr, 1), Region(fr.nbytes, 0, seed=2)
            rc, seen = traced(lambda: lib.gs_b200_adaptive_threshold_batch(D.ptr, S.ptr, w, h, n, r, c, stream()))
            _ok(rc)
            got = D.read("dst").reshape(n, h, w)
            assert np.array_equal(S.read("src"), fr.reshape(-1))
        bad = [i for i in range(n) if not np.array_equal(got[i], L.o_adaptive(O, fr[i], r, c))]
        assert not bad, "frames %s (random, natural, zeros, 255) differ from the oracle at c = %d" % (bad, c)
        return seen
    witnessed(witness, run, [kernel], "adaptive-%s-c%s" % (name, _cid(c)))


# ---- b. thresholds ---------------------------------------------------------------------------------------------------
THRESH = (0, 254, 255, 256, 511, UINT_MAX)
OFFSETS = (INT_MIN, -256, -1, 0, 1, 255, 256, INT_MAX - 254, INT_MAX)
EACH = np.array([0, 1, 254, 255], np.uint8)


@needs_ref
def test_ref_threshold_extremes():
    """gs_threshold takes a uint8_t: a C caller's unsigned threshold arrives as its low byte, which is what
    gs_b200_threshold_batch and the oracle take"""
    R = L.ref()
    a = np.random.default_rng(22).integers(0, 256, (9, 31), dtype=np.uint8)
    for t in THRESH + tuple(int(e) + o for e in EACH for o in OFFSETS):
        want = a.copy(); O.gso_threshold(L.ptr(want), 31, 9, t % 2 ** 32)
        d = a.copy(); R.gs_threshold(L.img(d), t & 0xFF)
        assert np.array_equal(d, want), t


def _thr_geoms():
    return [("vec", 272, 41, "gsb::k_threshold<true>"), ("scalar", 100, 37, "gsb::k_threshold<false>")]


@pytest.mark.gpu
@pytest.mark.parametrize("t", THRESH, ids=_cid)
@pytest.mark.parametrize("name,w,h,kernel", [pytest.param(*g, id=g[0]) for g in _thr_geoms()])
def test_threshold_extremes(lib, witness, name, w, h, kernel, t):
    fr = frames(w, h, 3, w + h)

    def run():
        S = Region(fr.nbytes, 0, fr, 1)
        rc, seen = traced(lambda: lib.gs_b200_threshold_batch(S.ptr, w, h, 3, t, stream()))
        _ok(rc)
        got = S.read("img").reshape(3, h, w)
        for i in range(3):
            want = fr[i].copy(); O.gso_threshold(L.ptr(want), w, h, t & 0xFF)
            assert np.array_equal(got[i], want), i
        return seen
    witnessed(witness, run, [kernel], "threshold-%s-t%s" % (name, _cid(t)))


@pytest.mark.gpu
@pytest.mark.parametrize("offset", OFFSETS, ids=_cid)
@pytest.mark.parametrize("name,w,h,kernel", [pytest.param(*g, id=g[0]) for g in _thr_geoms()])
def test_threshold_each_extremes(lib, witness, name, w, h, kernel, offset):
    n = len(EACH)
    fr = frames(w, h, n, w + h + 1)

    def run():
        S, T = Region(fr.nbytes, 0, fr, 1), Region(n, 3, EACH, seed=2)
        rc, seen = traced(lambda: lib.gs_b200_threshold_each_batch(S.ptr, w, h, n, T.ptr, offset, stream()))
        _ok(rc)
        T.read("thresholds")
        got = S.read("img").reshape(n, h, w)
        for i in range(n):
            want = fr[i].copy(); O.gso_threshold(L.ptr(want), w, h, (int(EACH[i]) + offset) % 256)  # (uint8_t)(t + off)
            assert np.array_equal(got[i], want), (i, int(EACH[i]))
        return seen
    witnessed(witness, run, [kernel], "threshold_each-%s-off%s" % (name, _cid(offset)))


# ---- c. filter -------------------------------------------------------------------------------------------------------
def filter3_route(k, norm):
    """filter.cu's host test for a 3x3 kernel on an aligned frame: 'true' (norm 1), 'false' (magic divisor) or None
    (k_filter_generic)"""
    pos = sum(255 * int(v) for v in k.view(np.int8).ravel() if v > 0)
    neg = sum(255 * -int(v) for v in k.view(np.int8).ravel() if v <= 0)
    if norm == 1:
        return "true"
    magic_ok = norm >= 2 and pos * norm < 2 ** 32 and (2 ** 32 - neg) // norm >= 256
    return "false" if magic_ok else None


def largest_magic_norm(k):
    """the largest norm filter3_route still sends to k_filter3<false>"""
    pos = sum(255 * int(v) for v in k.view(np.int8).ravel() if v > 0)
    neg = sum(255 * -int(v) for v in k.view(np.int8).ravel() if v <= 0)
    n = (2 ** 32 - neg) // 256
    if pos:
        n = min(n, (2 ** 32 - 1) // pos)
    assert filter3_route(k, n) == "false" and filter3_route(k, n + 1) is None
    return n


def _k(rows):
    return np.ascontiguousarray(np.array(rows, np.int8).view(np.uint8))


KERNELS3 = {"all-128": _k([[-128] * 3] * 3), "all127": _k([[127] * 3] * 3),
            "mixed": _k([[127, -128, 127], [-128, 127, -128], [127, -128, 127]])}


def _filter3_cases():
    out = []
    for name, k in KERNELS3.items():
        nmax = largest_magic_norm(k)
        for norm in sorted({nmax, nmax + 1, 1, 2, 2 ** 31, UINT_MAX}):
            out.append(("%s-norm%d" % (name, norm), name, norm))
    return out


def _shape_kernels():
    rng = np.random.default_rng(23)

    def rnd(kh, kw):
        v = rng.integers(-128, 128, (kh, kw)).astype(np.int8)
        v.flat[0], v.flat[-1] = -128, 127
        return np.ascontiguousarray(v.view(np.uint8))
    # (name, frame w, frame h, kernel or None, kw, kh)
    out = [("%dx%d" % (kw, kh), 272, 41, rnd(kh, kw), kw, kh) for kw, kh in ((1, 1), (1, 9), (9, 1), (2, 2), (4, 4))]
    out += [("wider-17x3", 16, 6, rnd(3, 17), 17, 3), ("taller-3x7", 16, 6, rnd(7, 3), 3, 7),
            ("both-20x9", 16, 6, rnd(9, 20), 20, 9), ("null", 272, 41, None, 0, 0),
            ("0x0", 272, 41, rnd(1, 1), 0, 0), ("3x0", 272, 41, rnd(1, 3), 3, 0)]
    return out


def _kptr(k):
    return None if k is None else k.ctypes.data


@needs_ref
def test_ref_filter_extremes():
    R = L.ref()
    rng = np.random.default_rng(24)
    imgs = [rng.integers(0, 256, (9, 13), dtype=np.uint8), np.full((5, 6), 255, np.uint8), np.zeros((4, 4), np.uint8),
            L.natural_like(16, 6, 3)]
    cases = [(KERNELS3[nm], 3, 3, norm) for _, nm, norm in _filter3_cases()]
    cases += [(k, kw, kh, norm) for _, _, _, k, kw, kh in _shape_kernels() for norm in (1, 7, UINT_MAX)]
    for a in imgs:
        a = np.ascontiguousarray(a)
        h, w = a.shape
        for k, kw, kh, norm in cases:
            want = np.zeros_like(a)
            O.gso_filter(L.ptr(want), L.ptr(a), w, h, _kptr(k), kw, kh, norm)
            d = np.zeros_like(a)
            R.gs_filter(L.img(d), L.img(a), L.Image(kw, kh, _kptr(k)), norm)
            assert np.array_equal(d, want), (w, h, kw, kh, norm)


def _run_filter(lib, fr, k, kw, kh, norm):
    n, h, w = fr.shape
    S, D = Region(fr.nbytes, 0, fr, 1), Region(fr.nbytes, 0, seed=2)
    rc, seen = traced(lambda: lib.gs_b200_filter_batch(D.ptr, S.ptr, w, h, n, _kptr(k), kw, kh, norm, stream()))
    _ok(rc)
    got = D.read("dst").reshape(n, h, w)
    assert np.array_equal(S.read("src"), fr.reshape(-1))
    for i in range(n):
        want = np.zeros_like(fr[i])
        O.gso_filter(L.ptr(want), L.ptr(fr[i]), w, h, _kptr(k), kw, kh, norm)
        assert np.array_equal(got[i], want), i
    return seen


@pytest.mark.gpu
@pytest.mark.parametrize("cid,kname,norm", [pytest.param(*c, id=c[0]) for c in _filter3_cases()])
def test_filter3_norm_extremes(lib, witness, cid, kname, norm):
    k = KERNELS3[kname]
    route = filter3_route(k, norm)
    kernel = "gsb::k_filter3<%s>" % route if route else "gsb::k_filter_generic"
    fr = frames(272, 41, 3, 7)
    witnessed(witness, lambda: _run_filter(lib, fr, k, 3, 3, norm), [kernel], "filter-" + cid)


@pytest.mark.gpu
@pytest.mark.parametrize("name,w,h,k,kw,kh", [pytest.param(*c, id=c[0]) for c in _shape_kernels()])
def test_filter_shapes(lib, witness, name, w, h, k, kw, kh):
    fr = frames(w, h, 3, w + kw + kh)

    def run():
        seen = set()
        for norm in (1, 7, UINT_MAX):
            seen |= _run_filter(lib, fr, k, kw, kh, norm)
        return seen
    witnessed(witness, run, ["gsb::k_filter_generic"], "filter-" + name)


# ---- d. template width -----------------------------------------------------------------------------------------------
ROW_TAPS = (2 ** 32 - 1) // (255 * 255)     # 66051: the most taps a u32 row sum of squared byte differences holds


def template_word_path(w, tw):
    """filter.cu: k_match_template (u32 row sums) for w % 4 == 0 on a word-aligned base and tw < 66051"""
    return w % 4 == 0 and tw < ROW_TAPS


TW = tuple(range(ROW_TAPS - 3, ROW_TAPS + 2))     # 66048 .. 66052


def _template_inputs(w, h, tw, th):
    rng = np.random.default_rng(tw + th)
    fr = np.stack([np.full((h, w), 255, np.uint8), rng.integers(0, 256, (h, w), dtype=np.uint8)])
    tmpls = [np.zeros((th, tw), np.uint8), rng.integers(0, 256, (th, tw), dtype=np.uint8)]
    return fr, tmpls


@needs_ref
def test_ref_template_width():
    assert ROW_TAPS * 255 * 255 < 2 ** 32 <= (ROW_TAPS + 1) * 255 * 255
    R = L.ref()
    for w in (ROW_TAPS + 1, ROW_TAPS + 2):
        for tw in TW:
            for th in (1, 2):
                fr, tmpls = _template_inputs(w, 2, tw, th)
                for a in fr:
                    for t in tmpls:
                        rw, rh = w - tw + 1, 2 - th + 1
                        want, d = np.zeros((rh, rw), np.uint8), np.zeros((rh, rw), np.uint8)
                        O.gso_match_template(L.ptr(a), w, 2, L.ptr(t), tw, th, L.ptr(want))
                        R.gs_match_template(L.img(a), L.img(t), L.img(d))
                        assert np.array_equal(d, want), (w, tw, th)


@pytest.mark.gpu
@pytest.mark.parametrize("th", (1, 2))
@pytest.mark.parametrize("tw", TW)
@pytest.mark.parametrize("w", (ROW_TAPS + 1, ROW_TAPS + 2))
def test_template_width(lib, witness, w, tw, th):
    h = 2
    fr, tmpls = _template_inputs(w, h, tw, th)
    rw, rh = w - tw + 1, h - th + 1
    kernels = ["gsb::k_pack_template", "gsb::k_match_template"] if template_word_path(w, tw) else \
        ["gsb::k_match_template_generic"]

    def run():
        seen = set()
        for tmpl in tmpls:
            S, T, D = Region(fr.nbytes, 0, fr, 1), Region(tmpl.nbytes, 0, tmpl, 3), Region(2 * rw * rh, 0, seed=2)
            rc, s = traced(lambda: lib.gs_b200_match_template_batch(D.ptr, S.ptr, w, h, 2, T.ptr, tw, th, stream()))
            _ok(rc)
            got = D.read("result").reshape(2, rh, rw)
            for i in range(2):
                want = np.zeros((rh, rw), np.uint8)
                O.gso_match_template(L.ptr(fr[i]), w, h, L.ptr(tmpl), tw, th, L.ptr(want))
                assert np.array_equal(got[i], want), (i, int(tmpl.max()))
            seen |= s
        return seen
    witnessed(witness, run, kernels, "match_template-w%d-tw%d-th%d" % (w, tw, th))


# ---- e. match_orb max_distance ---------------------------------------------------------------------------------------
# max_distance <= -2^24 is left out: there M = max_distance + 1 == max_distance in fp32, so a query with no candidate
# below M is emitted with distance (unsigned)M, a negative float converted to unsigned, which C leaves undefined
MAX_DIST = (float("nan"), float("-inf"), -1.0, -0.5, 0.0, 0.5, 59.5, 60.0, 60.5, 255.0, 255.5, 256.0, 257.0, 1e9,
            float("inf"))


def _flip(d, nbits, rng):
    d = d.copy()
    bits = rng.choice(256, nbits, replace=False)
    for b in bits:
        d[b // 32] ^= np.uint32(1 << int(b % 32))
    return d


def _match_sets():
    """(set1, set2) pairs: 120 x 90 with candidates at exactly 0, 1, 59, 60, 61, 255 and 256 bits from some queries;
    7 x 0; 40 x 1 (the one candidate the complement of query 0)"""
    rng = np.random.default_rng(25)
    a, b = L.desc_sets(rng, 120, 90)
    for i, nb in enumerate((0, 1, 59, 60, 61, 255, 256, 60, 59, 61)):
        b["descriptor"][10 + i] = _flip(a["descriptor"][i], nb, rng)
    c, _ = L.desc_sets(rng, 7, 0)
    e, f = L.desc_sets(rng, 40, 1)
    f["descriptor"][0] = ~e["descriptor"][0]
    e["descriptor"][1] = _flip(f["descriptor"][0], 60, rng)
    return [(a, b), (c, f[:0]), (e, f)]


@needs_ref
def test_ref_match_orb_extremes():
    R = L.ref()
    sets = _match_sets()
    for md in MAX_DIST:
        for k1, k2 in sets:
            for mm in (1, len(k1) - 1, UINT_MAX):
                want = L.o_match(O, k1, k2, mm, md)
                m = np.zeros(len(k1), L.MATCH_DTYPE)
                n = R.gs_match_orb(L.ptr(k1), len(k1), L.ptr(k2 if len(k2) else np.zeros(1, L.KP_DTYPE)), len(k2),
                                   L.ptr(m), mm, md)
                assert m[:n].tobytes() == want.tobytes(), (md, len(k1), len(k2), mm)
    assert len(L.o_match(O, *sets[0], UINT_MAX, 60.0)) > 10 and len(L.o_match(O, *sets[2], UINT_MAX, 256.0)) > 0


def _run_match(lib, sets, mm, md):
    n = len(sets)
    s1, s2 = max(len(a) for a, _ in sets), max(max(len(b) for _, b in sets), 1)
    k1, k2 = np.zeros((n, s1), L.KP_DTYPE), np.zeros((n, s2), L.KP_DTYPE)
    for i, (a, b) in enumerate(sets):
        k1[i, :len(a)], k2[i, :len(b)] = a, b
    c1 = np.array([len(a) for a, _ in sets], np.uint32)
    c2 = np.array([len(b) for _, b in sets], np.uint32)
    cap = min(mm, s1)                                    # records per pair the call can write
    K1, K2, C1, C2 = Region(k1.nbytes, 0, k1, 1), Region(k2.nbytes, 0, k2, 2), Region(4 * n, 0, c1, 3), Region(4 * n, 0, c2, 4)
    M, MC = Region(12 * n * cap, 0, seed=5), Region(4 * n, 0, seed=6)
    rc, seen = traced(lambda: lib.gs_b200_match_orb_batch(K1.ptr, C1.ptr, s1, K2.ptr, C2.ptr, s2, n, M.ptr, MC.ptr, mm, md,
                                                         stream()))
    _ok(rc)
    counts, m = MC.read("counts").view(np.uint32), M.read("matches").view(L.MATCH_DTYPE).reshape(n, cap)
    for i, (a, b) in enumerate(sets):
        want = L.o_match(O, a, b, mm, md)
        assert counts[i] == len(want) and m[i, :counts[i]].tobytes() == want.tobytes(), (i, int(counts[i]), len(want))
    return seen


@pytest.mark.gpu
@pytest.mark.parametrize("md", MAX_DIST, ids=lambda v: "md%s" % v)
def test_match_orb_max_distance(lib, witness, md):
    sets = _match_sets()

    def run():
        seen = _run_match(lib, sets, 1, md) | _run_match(lib, sets, len(sets[0][0]) - 1, md)
        for s in sets:     # matches hold npairs x max_matches records: UINT_MAX is one pair per call
            seen |= _run_match(lib, [s], UINT_MAX, md)
        return seen
    witnessed(witness, run, ["gsb::k_match_best", "gsb::k_match_compact"], "match_orb-md%s" % md)


# ---- f. radius -------------------------------------------------------------------------------------------------------
FAST_R, WIDE_R = 63, 120      # launch_box: the magic division only for r <= 63; k_box_mid / k_box_wide for r <= 120
TINY = ((3, 3), (8, 1), (1, 9))
MEDIUM = ((272, 70), (100, 37))


def radii(w, h):
    m = max(w, h)
    return sorted({FAST_R, FAST_R + 1, WIDE_R - 1, WIDE_R, WIDE_R + 1, m - 1, m, 4096, 65535, INT_MAX} - {0})


def box_route(w, r, adaptive, c=0):
    """launch_box's kernel for fresh (256-byte aligned) allocations"""
    a = "true" if adaptive else "false"
    ok = not adaptive or lane_c_ok(c)
    if ok and 1 <= r <= 7 and w % 16 == 0:
        return "gsb::k_box_tma<%d, %s>" % (r, a)
    if 1 <= r <= WIDE_R:
        return "gsb::k_box_mid<%d, %s>" % (r & 3, a) if ok and w % 8 == 0 else "gsb::k_box_wide<%s>" % a
    return "gsb::k_box_generic<%s>" % a


@needs_ref
def test_ref_radius_extremes():
    """the reference loops (2r+1)^2 times per pixel (and divides by zero from r = 2^31), so it is pinned up to r = 2000
    on images of 9 pixels or fewer; beyond that, every r >= max(w, h) - 1 covers the whole image, so the oracle must
    give what it gives at r = max(w, h)"""
    R = L.ref()
    rng = np.random.default_rng(26)
    for w, h in TINY + ((9, 1), (2, 4)):
        for a in (rng.integers(0, 256, (h, w), dtype=np.uint8), np.full((h, w), 255, np.uint8)):
            for r in [x for x in radii(w, h) if x <= 2000] + [2000]:
                d = np.empty_like(a); R.gs_blur(L.img(d), L.img(a), r)
                assert np.array_equal(d, L.o_blur(O, a, r)), ("blur", w, h, r)
                d = np.empty_like(a); R.gs_adaptive_threshold(L.img(d), L.img(a), r, -3)
                assert np.array_equal(d, L.o_adaptive(O, a, r, -3)), ("adaptive", w, h, r)
    for w, h in TINY + MEDIUM:
        a = L.natural_like(w, h, 4)
        full_b, full_a = L.o_blur(O, a, max(w, h)), L.o_adaptive(O, a, max(w, h), -3)
        for r in (max(w, h) - 1, 4096, 65535, INT_MAX):
            assert np.array_equal(L.o_blur(O, a, r), full_b) and np.array_equal(L.o_adaptive(O, a, r, -3), full_a), r


def _radius_cases():
    return [(w, h, r, op) for w, h in TINY + MEDIUM for r in radii(w, h) for op in ("blur", "adaptive")]


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,r,op", [pytest.param(*c, id="%s-%dx%d-r%d" % (c[3], c[0], c[1], c[2]))
                                      for c in _radius_cases()])
def test_radius_extremes(lib, witness, w, h, r, op):
    adaptive, c = op == "adaptive", -3
    fr = frames(w, h, 3, w + h)

    def run():
        S, D = Region(fr.nbytes, 0, fr, 1), Region(fr.nbytes, 0, seed=2)
        if adaptive:
            rc, seen = traced(lambda: lib.gs_b200_adaptive_threshold_batch(D.ptr, S.ptr, w, h, 3, r, c, stream()))
        else:
            rc, seen = traced(lambda: lib.gs_b200_blur_batch(D.ptr, S.ptr, w, h, 3, r, stream()))
        _ok(rc)
        got = D.read("dst").reshape(3, h, w)
        for i in range(3):
            want = L.o_adaptive(O, fr[i], r, c) if adaptive else L.o_blur(O, fr[i], r)
            assert np.array_equal(got[i], want), i
        return seen
    witnessed(witness, run, [box_route(w, r, adaptive, c)], "%s-%dx%d-r%d" % (op, w, h, r))


# ---- g. integral wrap, LBP on the wrapped table ----------------------------------------------------------------------
WRAP_W = 4400     # 255 * 4138^2 > 2^32: every corner the faces' windows read has wrapped


def wrap_frame(shift=0):
    """255 everywhere except four copies of lena (faces at scales 1.2 - 1.5) at the bottom right, at both parities"""
    lena = np.load(os.path.join(L.ROOT, "tests", "golden", "lena_golden.npz"))["lena"]
    f = np.full((WRAP_W, WRAP_W), 255, np.uint8)
    for i in range(2):
        for j in range(2):
            y0, x0 = WRAP_W - 130 * (i + 1) - i, WRAP_W - 130 * (j + 1) - j - shift
            f[y0:y0 + 128, x0:x0 + 128] = lena
    return f


def _assert_wrapped(f, rects):
    """every rect's lattice starts past the point where the table passed 2^32"""
    assert len(rects) > 0
    x0, y0 = int(rects["x"].min()), int(rects["y"].min())
    assert int(f[:y0, :x0].sum(dtype=np.uint64)) >= 2 ** 32, (x0, y0)


WRAP_LBP = (1.1, 1.0, 1.5, 2)     # scale_factor, min_scale, max_scale, step


@needs_ref
def test_ref_integral_wrap():
    R = L.ref()
    f = wrap_frame()
    ii = np.empty(f.shape, np.uint32); R.gs_integral(L.img(f), L.ptr(ii))
    assert np.array_equal(ii, L.o_integral(O, f))
    assert int(ii[-1, -1]) == int(f.sum(dtype=np.uint64)) % 2 ** 32 and int(f.sum(dtype=np.uint64)) >= 2 ** 32


@needs_ref
def test_ref_lbp_on_wrapped_table():
    """gs_lbp_detect reads the table in modular u32 arithmetic: on the table of lena plus 2^32 - 4096 (nearly every
    entry wraps), the oracle and the reference find the same rects, and the same as on the plain table away from the
    first row and column"""
    R = L.ref()
    lena = np.load(os.path.join(L.ROOT, "tests", "golden", "lena_golden.npz"))["lena"]
    ii = L.o_integral(O, np.ascontiguousarray(lena))
    wrapped = ((ii.astype(np.uint64) + 2 ** 32 - 4096) % 2 ** 32).astype(np.uint32)
    assert (wrapped < ii).mean() > 0.9
    cas = L.HostCascade()
    for t in (ii, wrapped):
        want = L.o_detect(O, cas, t, 1000, 1.1, 1.0, 4.0, 1)
        r = np.zeros(1000, L.RECT_DTYPE)
        n = R.gs_lbp_detect(cas.ptr, L.ptr(t), 128, 128, L.ptr(r), 1000, 1.1, 1.0, 4.0, 1)
        assert r[:n].tobytes() == want.tobytes() and n > 0


@pytest.mark.gpu
def test_integral_wrap_and_lbp(lib, witness):
    import torch
    frs = [wrap_frame(0), wrap_frame(1)]
    want = [torch.from_numpy(L.o_integral(O, f).view(np.int32)).cuda() for f in frs]
    px = WRAP_W * WRAP_W

    def integral(env, n, ii_off):
        src = torch.from_numpy(np.stack([frs[i % 2] for i in range(n)])).cuda()
        buf = torch.full((n * px + 8,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
        ptr = buf.data_ptr() + ii_off
        if env:
            os.environ["GS_B200_INTEGRAL"] = env
        try:
            rc, seen = traced(lambda: lib.gs_b200_integral_batch(ptr, src.data_ptr(), WRAP_W, WRAP_W, n, stream()))
        finally:
            os.environ.pop("GS_B200_INTEGRAL", None)
        _ok(rc)
        k = ii_off // 4
        assert bool((buf[:k] == 0x5A5A5A5A).all()) and bool((buf[k + n * px:] == 0x5A5A5A5A).all()), "bytes outside"
        tables = buf[k:k + n * px].view(n, WRAP_W, WRAP_W)
        for i in range(n):
            assert torch.equal(tables[i], want[i % 2]), (env, i)
        return seen, tables

    rows_cols = ["gsb::k_integral_rows<false>", "gsb::k_integral_cols"]
    for env, n, off, kernels in (("strips", 1, 0, ["gsb::k_integral_strips<128, 8>"]),
                                 ("bands", 32, 0, ["gsb::k_integral_bands<1024>"]), (None, 1, 4, rows_cols)):
        witnessed(witness, lambda: integral(env, n, off)[0], kernels,
                  "integral-%s-%dx%d-n%d-ii%d" % (env or "rows_cols", WRAP_W, WRAP_W, n, off))

    _, tables = integral("strips", 1, 0)
    cas = L.HostCascade()
    sf, mn, mx, step = WRAP_LBP
    mr = 1000
    ref_rects = L.o_detect(O, cas, want[0].cpu().numpy().view(np.uint32), mr, sf, mn, mx, step)
    _assert_wrapped(frs[0], ref_rects)

    def lbp():
        RR = torch.zeros(mr * 4, dtype=torch.int32, device="cuda")
        N = torch.zeros(1, dtype=torch.int32, device="cuda")
        rc, seen = traced(lambda: lib.gs_b200_lbp_detect_batch(cas.ptr, tables.data_ptr(), WRAP_W, WRAP_W, 1, RR.data_ptr(),
                                                               N.data_ptr(), mr, sf, mn, mx, step, stream()))
        _ok(rc)
        n = int(N.item())
        got = RR.cpu().numpy().view(np.uint32).reshape(mr, 4)[:n]
        assert got.tobytes() == ref_rects.tobytes(), (n, len(ref_rects))
        return seen
    witnessed(witness, lbp, ["gsb::k_lbp_emit"], "lbp-on-wrapped-table")


# ---- h. ORB nkps -----------------------------------------------------------------------------------------------------
ORB_MAXC = 5000    # the reference's static candidates[5000]
NKPS = (1, ORB_MAXC // 4 - 1, ORB_MAXC // 4, ORB_MAXC // 4 + 1)


def _orb_frame():
    return L.natural_like(1920, 1080, 5)


def _fast_survivors(a):
    return len(L.o_fast(O, a, np.zeros_like(a), 10 ** 6, 20))


@needs_ref
def test_ref_orb_nkps():
    a = _orb_frame()
    assert _fast_survivors(a) > ORB_MAXC
    assert [min(4 * k, ORB_MAXC) for k in NKPS] == [4, 4996, 5000, 5000]
    R = L.ref()
    for nk in NKPS:
        kr = np.zeros(nk, L.KP_DTYPE)
        n = R.gs_orb_extract(L.img(a), L.ptr(kr), nk, 20, L.ptr(np.zeros_like(a)))
        ko = L.o_orb(O, a, np.zeros_like(a), nk, 20)
        assert n == len(ko) and kr[:n].tobytes() == ko.tobytes(), nk
        assert n == (0 if nk == 1 else nk), (nk, n)    # nkps = 1: the 4 candidates all lie in the 15-px margin


@pytest.mark.gpu
@pytest.mark.parametrize("nk", NKPS)
def test_orb_nkps(lib, witness, nk):
    a = _orb_frame()
    h, w = a.shape

    def run():
        S, SM = Region(a.nbytes, 0, a, 1), Region(a.nbytes, 0, np.zeros_like(a), 4)
        K, N = Region(48 * nk, 0, seed=5), Region(4, 0, seed=6)
        rc, seen = traced(lambda: lib.gs_b200_orb_extract_batch(S.ptr, w, h, 1, SM.ptr, K.ptr, N.ptr, nk, 20, stream()))
        _ok(rc)
        cnt = int(N.read("counts").view(np.uint32)[0])
        got = K.read("kps").view(L.KP_DTYPE)[:cnt]
        sm = np.zeros_like(a)
        want = L.o_orb(O, a, sm, nk, 20)
        assert cnt == len(want) == (0 if nk == 1 else nk) and got.tobytes() == want.tobytes(), (cnt, len(want))
        assert np.array_equal(SM.read("scoremap").reshape(h, w), sm)
        return seen
    witnessed(witness, run, ["gsb::k_orb_select", "gsb::k_orb_brief<true>"], "orb-1920x1080-nkps%d" % nk)
