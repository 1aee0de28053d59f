"""Image content built to reach the data-dependent branches of FAST, ORB and blob labelling.

test_dispatch_paths.py picks kernels by geometry and test_param_extremes.py by scalar; here the pixels pick the branch.
Each family has a generator, and a numpy predicate that proves the generated frames reach the condition they are for
and tell it apart from its near miss:

  A  FAST      stamps: a centre p with an arc of 8, 9, 15 or 16 ring samples from each of the 16 start positions, on
               either side, at p +- t (not counted) or p +- (t + 1) (counted); 9-arcs that hold exactly two adjacent
               compass points; neutral samples nearer to p than the arc, so the score is the minimum over all 16
               samples; p in {0, 1, t-1, t, t+1, 254, 255} for t in {0, 1, 20, 254, 255} (t > p: the reference's
               unsigned wrap, every non-brighter sample counts as darker), and t = 256 / 2^32 - 200 on k_fast_score.
               Centres at every column residue mod 4, on k_fast_tiled2's tile seams (x0 - 1, x0, x0 + 127, x0 + 128:
               the scalar ring columns; y0 - 1, y0, y0 + 63, y0 + 64) and on the first / last scored row and column.
     NMS       equal-score plateaus (2 x 2 squares, 1 x 3 bars of one value) across tile seams, a higher neighbour across
               a seam, and non-zero stale bytes in the caller's score map on the ring cells FAST never writes.
     cap       nkps equal to a frame's survivor total, total - 1 and total + 1 in one batch; cuts at the first survivor
               of a row and mid-row; frames without survivors.
  B  ORB       more than 256 equal responses, interleaved with responses one above and below, and candidates at
               x, y = 14, 15, w - 16, w - 15 (the 15-px margin); nkps caps that land inside a 256-wide pass and a
               32-wide rank step; the FAST candidate cap min(4 nkps, 5000) cutting a row.
     angles    disc patches whose moments are set exactly (zero background, chosen values on the dx and dy axes):
               (0, 0), (0, -k), (+-k, 0); m10 = 1 (atan2f's x == 1 shortcut); |m01| = |m10|; |m01 / m10| within 32
               floats of atanf's reduction thresholds 7/16, 11/16, 19/16, 39/16 in all four quadrants; every pair with
               |m01|, |m10| <= 40.  Single image at r = 15 (int moments) and r = 16, 20 (fp32 moments); the same
               moments around FAST corner stamps through the batched ORB, where angle, sin / cos and all 256
               descriptor bits must match.
  C  blobs     the (nblobs + 1)-th seed at bit 0, bit 31 and mid-word, as its row's first seed, in row 0 and in the last
               row; seed totals nblobs - 1, nblobs, nblobs + 1 in one batch; after the overflow point, runs whose
               labelled contact is mid-run or their last pixel and runs that carry through whole words; nblobs = 1 and
               65534 on a checkerboard of isolated pixels.  Widths 1023, 1024, 1025, 2049 with runs across the
               1024-pixel chunk seam, all-ones and alternating rows; a spiral, a comb joined in its last row,
               4-connected staircases, interleaved spirals, nested U shapes; a 4096 x 4096 component whose x sum wraps
               mod 2^32, boxes touching all four borders; corners of diamonds, squares, lines and single pixels.

  * CPU: every predicate, the numpy FAST model against the oracle's score maps, and, where oracle/_ref is built, the
    oracle against the compiled reference on every generated frame.
  * GPU: batches that mix frames which reach a condition with frames which do not, bit-exact on every frame against the
    oracle, each through the kernels the dispatch rows name for it (tiled and fall-back), witnessed under torch.profiler.
"""
import functools

import numpy as np
import pytest

import _libs as L
from _gpu import Region, lib, stream, traced, witness, witnessed  # noqa: F401

O = L.oracle()
needs_ref = pytest.mark.skipif(not L.have_ref(), reason="oracle/_ref not built")
U32 = 2 ** 32


def _ok(rc):
    from grayskull_b200 import _lib
    _lib.check(rc, "content-edge case")


# ======================================================================================================================
# A. FAST
# ======================================================================================================================
RING = ((0, -3), (1, -3), (2, -2), (3, -1), (3, 0), (3, 1), (2, 2), (1, 3),
        (0, 3), (-1, 3), (-2, 2), (-3, 1), (-3, 0), (-3, -1), (-2, -2), (-1, -3))
COMPASS = (0, 4, 8, 12)
TS = (0, 1, 20, 254, 255)
BIG_TS = (256, U32 - 200)


def run9(m):
    """circular run of >= 9 set bits in a 16-bit mask (elementwise)"""
    m = np.asarray(m, np.int64)
    mm = m | (m << 16)
    r = mm & (mm >> 1)
    r &= r >> 2
    r &= r >> 4
    r &= mm >> 8
    return (r & 0xFFFF) != 0


def fast_model(img, t):
    """the reference's FAST-9 test (grayskull.h:491-510) in numpy over the interior pixels: (bright, dark, score),
    each (h - 6, w - 6); p + t and p - t in unsigned 32-bit arithmetic"""
    h, w = img.shape
    a = img.astype(np.int64)
    P = a[3:h - 3, 3:w - 3]
    hi, wrap = (P + t) % U32, t > P
    bright, dark = np.zeros_like(P), np.zeros_like(P)
    mind = np.full(P.shape, 255, np.int64)
    for i, (dx, dy) in enumerate(RING):
        V = a[3 + dy:h - 3 + dy, 3 + dx:w - 3 + dx]
        b = V > hi
        d = ~b & (wrap | (V < P - t))
        bright |= b.astype(np.int64) << i
        dark |= d.astype(np.int64) << i
        mind = np.minimum(mind, np.abs(V - P))
    return bright, dark, np.where(run9(bright) | run9(dark), mind, 0)


def score_map(img, t, fill=None):
    """the score map gs_fast leaves: the model's scores on the interior, `fill` (zeros) elsewhere"""
    h, w = img.shape
    sm = np.zeros((h, w), np.uint8) if fill is None else fill.copy()
    sm[3:h - 3, 3:w - 3] = fast_model(img, t)[2]
    return sm


def nms_model(sm, w, h):
    """survivors of the reference's 3x3 NMS (strict `>` suppresses) in raster order: [(x, y, score)]; sm may be any size
    (gs_get: 0 outside it)"""
    big = np.zeros((h + 2, w + 2), np.int64)
    sh, sw = min(sm.shape[0], h), min(sm.shape[1], w)
    big[1:sh + 1, 1:sw + 1] = sm[:sh, :sw]
    c = big[1:h + 1, 1:w + 1]
    keep = c > 0
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            if dx or dy:
                keep &= big[1 + dy:h + 1 + dy, 1 + dx:w + 1 + dx] <= c
    keep[:3], keep[h - 3:], keep[:, :3], keep[:, w - 3:] = False, False, False, False
    ys, xs = np.nonzero(keep)
    return [(int(x), int(y), int(c[y, x])) for y, x in zip(ys, xs)]


def arc_bits(start, length):
    return sum(1 << ((start + i) % 16) for i in range(length))


class Stamp:
    """a FAST centre p with `length` ring samples from `start` at p + side * (t + level) (level 1: counted, 0: exactly
    at the threshold, not counted) and the others neutral: at distance nd from p on the arc's side when t >= nd >= 1,
    on the other side and counted when t == 0; `near` makes one neutral sample the nearest (distance 1)"""

    def __init__(self, p, t, side, length, start, level, nd=None, near=False):
        self.p, self.t, self.side, self.length, self.start, self.level = p, t, side, length, start, level
        self.nd = nd if nd is not None else max(1, min(t, 7))
        self.near = near and length < 15
        arc = p + side * (t + level)
        if t == 0:
            neutral = [p - side] * 16
        else:
            v = p + self.nd if p + self.nd <= 255 else p - self.nd
            neutral = [v] * 16
            if self.near:
                neutral[(start + length + 2) % 16] = p + 1 if p + 1 <= 255 else p - 1
        bits = arc_bits(start, length)
        self.values = [arc if (bits >> i) & 1 else neutral[i] for i in range(16)]
        self.arc = bits

    def feasible(self):
        return 0 <= self.p <= 255 and all(0 <= v <= 255 for v in self.values) and (self.t > 0 or self.level == 1) and \
            (self.t == 0 or 1 <= self.nd <= self.t)

    def expect(self):
        """(bright mask, dark mask, corner?) the stamp is built to have, derived from the construction, not the model"""
        p, t, full = self.p, self.t, 0xFFFF
        wrap = t > p
        neutral_side = 0 if t else -self.side          # t == 0: the neutral samples are counted on the other side
        if self.side > 0:
            bright = self.arc if self.level else 0
            dark = full & ~bright if wrap else (full & ~self.arc if neutral_side < 0 else 0)
        else:
            dark = self.arc if self.level else 0
            bright = full & ~self.arc if neutral_side > 0 else 0
        corner = bool(run9(bright) or run9(dark))
        return bright, dark, corner

    def paint(self, img, x, y):
        img[y, x] = self.p
        for (dx, dy), v in zip(RING, self.values):
            img[y + dy, x + dx] = v

    def desc(self):
        return "p%d t%d %s%d@%d %s" % (self.p, self.t, "+" if self.side > 0 else "-", self.length, self.start,
                                       "counted" if self.level else "at-threshold")


def stamp_specs(t):
    """the stamps for one threshold: every (p, side, length, level) that fits in a byte, starts cycling through all 16
    positions; at t = 20 additionally the full 16-start x 4-length x 2-side x 2-level table around p = 100"""
    out = []
    ps = sorted({v for v in (0, 1, t - 1, t, t + 1, 254, 255) if 0 <= v <= 255})
    k = 0
    for p in ps:
        for side in (1, -1):
            for length in (8, 9, 15, 16):
                for level in (1, 0):
                    for near in (False, True):
                        s = Stamp(p, t, side, length, (5 * k + 3) % 16, level, near=near)
                        k += 1
                        if s.feasible():
                            out.append(s)
    if t == 20:
        for side in (1, -1):
            for length in (8, 9, 15, 16):
                for level in (1, 0):
                    for start in range(16):
                        out.append(Stamp(100, 20, side, length, start, level, nd=20 if start % 2 else 1,
                                         near=start % 4 == 1))
    return out


def slot_columns(w):
    """x0 - 1, x0, x0 + 127, x0 + 128 of every 128-column tile, the first and last scored columns, all residues mod 4"""
    cols = {3, w - 4}
    for x0 in range(128, w - 3, 128):
        cols |= {x0 - 1, x0}
    cols |= {40, 61, 82, 103, 161, 178, 195, 212}
    return sorted(c for c in cols if 3 <= c <= w - 4)


def slot_rows(h):
    """y0 - 1, y0, y0 + 63, y0 + 64 of every 64-row tile (y0 = 3 + 64k), the first and last scored rows"""
    rows = {3, h - 4}
    for y0 in range(67, h - 3, 64):
        rows |= {y0 - 1, y0}
    return sorted(r for r in rows if 3 <= r <= h - 4)


@functools.lru_cache(maxsize=None)
def slots(w, h, phase):
    """stamp centres, pairwise >= 9 apart in x or y: the seam rows x seam columns first (every other seam row and
    column first, alternating with `phase`, as neighbouring ones exclude each other), then a 9-px lattice"""
    taken = []
    cols, rows = slot_columns(w), slot_rows(h)
    cands = [(x, y) for y in rows[phase::2] + rows[1 - phase::2] for x in cols[phase::2] + cols[1 - phase::2]]
    cands += [(x, y) for y in slot_rows(h) for x in range(7, w - 4, 9)]
    cands += [(x, y) for y in range(7, h - 4, 9) for x in slot_columns(w)]
    cands += [(x, y) for y in range(12, h - 4, 9) for x in range(12, w - 4, 9)]
    occ = np.zeros((h + 20, w + 20), bool)
    for x, y in cands:
        if not occ[y + 10 - 8:y + 10 + 9, x + 10 - 8:x + 10 + 9].any():
            occ[y + 10, x + 10] = True
            taken.append((x, y))
    return taken


def stamp_frames(w, h, t, bg_seed):
    """the stamps of stamp_specs(t), corners and near misses in turn, over two or more frames whose slots favour
    alternate seam columns; backgrounds of 0 and of dimmed natural_like content -> (frames, [(frame, x, y, stamp)])"""
    specs = stamp_specs(t)
    yes, no = [s for s in specs if s.expect()[2]], [s for s in specs if not s.expect()[2]]
    specs = [s for pair in zip(yes, no) for s in pair] + yes[len(no):] + no[len(yes):]
    per = min(len(slots(w, h, 0)), len(slots(w, h, 1)), (len(specs) + 1) // 2)
    frames, placed = [], []
    for f0 in range(0, len(specs), per):
        img = np.zeros((h, w), np.uint8)
        if len(frames) % 2:
            img[:] = L.natural_like(w, h, bg_seed + f0) // 2
        for s, (x, y) in zip(specs[f0:f0 + per], slots(w, h, len(frames) % 2)):
            img[y - 3:y + 4, x - 3:x + 4] = s.p
            s.paint(img, x, y)
            placed.append((len(frames), x, y, s))
        frames.append(img)
    return frames, placed


def check_stamps(frames, placed, t):
    """every stamp has the bright / dark masks and corner verdict it was built for, and the model's score map equals
    the oracle's; returns the placed stamps that are corners"""
    models = [fast_model(f, t) for f in frames]
    corners = []
    for fi, x, y, s in placed:
        bright, dark, score = (m[y - 3, x - 3] for m in models[fi])
        eb, ed, ec = s.expect()
        assert (int(bright), int(dark)) == (eb, ed), (s.desc(), x, y, hex(int(bright)), hex(int(dark)), hex(eb), hex(ed))
        assert (score > 0) == ec or (ec and min(abs(v - s.p) for v in s.values) == 0), (s.desc(), int(score))
        if ec:
            assert score == min(abs(v - s.p) for v in s.values), (s.desc(), int(score))
            corners.append((fi, x, y, s))
    for f in frames:
        sm = np.zeros_like(f)
        O.gso_fast(L.ptr(f), f.shape[1], f.shape[0], L.ptr(sm), f.shape[1], f.shape[0], L.ptr(np.zeros(1, L.KP_DTYPE)), 1, t)
        assert np.array_equal(sm, score_map(f, t))
    return corners


FAST_W, FAST_H = 400, 210


def test_fast_stamp_predicates():
    """every family reaches its condition and its near miss"""
    for t in TS:
        frames, placed = stamp_frames(FAST_W, FAST_H, t, 10 + t)
        corners = check_stamps(frames, placed, t)
        specs = [s for _, _, _, s in placed]
        assert corners
        if t == 20:
            # the length-9 arcs are corners and the length-8 ones are not, from every start and on both sides
            for side in (1, -1):
                for start in range(16):
                    c = {(s.length, s.level) for _, _, _, s in corners if s.side == side and s.start == start and
                         s.p == 100}
                    assert c == {(9, 1), (15, 1), (16, 1)}, (side, start, c)
            # 9-arcs with exactly two adjacent compass points (starts not = 0 mod 4) are corners
            two = [s for _, _, _, s in corners if s.length == 9 and len([c for c in COMPASS if s.arc >> c & 1]) == 2]
            assert {s.start % 4 for s in two} == {1, 2, 3}
            assert all(abs(c - d) in (4, 12) for s in two for c in COMPASS for d in COMPASS
                       if s.arc >> c & 1 and s.arc >> d & 1 and c != d)
            # the score is the minimum over all 16 samples: stamps whose nearest sample is a neutral one
            assert any(s.near and s.level for _, _, _, s in corners)
        # the wrap case t > p is reached where it fits (t = 1, 20: p = 0 .. t - 1; t = 254, 255: p = 0, 1)
        if t:
            assert any(s.p < t for s in specs)
            assert any(s.p < t and s.level == 0 for _, _, _, s in corners) or t >= 254
        # centres on every column residue, every seam column and row, and the first / last scored row and column
        cx = {x for _, x, _, _ in corners}
        cy = {y for _, _, y, _ in corners}
        if t == 20:
            assert {x % 4 for x in cx} == {0, 1, 2, 3}
            assert set(slot_columns(FAST_W)) <= cx and set(slot_rows(FAST_H)) <= cy


def test_fast_big_threshold_predicates():
    """t = 256: every sample is non-brighter and t > p, so every interior pixel is a dark 16-arc; t = 2^32 - 200: p + t
    wraps to p - 200, so centres >= 200 see brighter samples"""
    frames, _ = stamp_frames(FAST_W, FAST_H, 20, 30)
    wrapped = 0
    for f in frames:
        b, d, s = fast_model(f, 256)
        assert not b.any() and (d == 0xFFFF).all()
        b, d, s = fast_model(f, U32 - 200)
        P = f[3:-3, 3:-3]
        assert not b[P < 200].any()
        wrapped += int((b[P >= 200] != 0).sum())
    assert wrapped > 0


# ---- NMS -------------------------------------------------------------------------------------------------------------
def nms_frame(w, h, stale_seed):
    """isolated bright pixels (scores = their value on a 0 background): 2x2 squares and 1x3 bars of one value across
    tile seams, a pixel with a higher neighbour across a seam, corners next to the never-written ring cells; and the
    caller's score map: stale bytes (above, equal to and below the corner next to them) on x = 2, w - 3, y = 2, h - 3
    -> (img, stale, plateaus, higher)"""
    img = np.zeros((h, w), np.uint8)
    plateaus, higher = [], []
    cols = [x0 - 1 for x0 in range(128, w - 24, 128)]
    rows = [y0 - 1 for y0 in range(67, h - 24, 64)]
    for i, c in enumerate(cols):
        for j, r in enumerate(rows):
            v = 60 + 10 * i + j
            sq = [(c, r), (c + 1, r), (c, r + 1), (c + 1, r + 1)]              # straddles both seams
            bar = [(c, r + 20), (c + 1, r + 20), (c + 2, r + 20)]            # across the column seam
            vbar = [(c + 20, r - 1), (c + 20, r), (c + 20, r + 1)]           # across the row seam
            for pl in (sq, bar, vbar):
                for x, y in pl:
                    img[y, x] = v
                plateaus.append(pl)
            img[r + 10, c], img[r + 10, c + 1] = v, v + 1                     # higher neighbour across the seam
            img[r - 12, c + 10], img[r - 11, c + 10] = v + 2, v + 1
            higher += [((c, r + 10), (c + 1, r + 10)), ((c + 10, r - 11), (c + 10, r - 12))]
    rng = np.random.default_rng(stale_seed)
    stale = np.zeros((h, w), np.uint8)
    edge = [(3, y) for y in range(12, h - 12, 17)] + [(w - 4, y) for y in range(15, h - 12, 17)]
    edge += [(x, 3) for x in range(20, w - 12, 23)] + [(x, h - 4) for x in range(25, w - 12, 23)]
    for k, (x, y) in enumerate(edge):
        v = 100 + k % 50
        img[y, x] = v
        nx, ny = (2 if x == 3 else w - 3 if x == w - 4 else x), (2 if y == 3 else h - 3 if y == h - 4 else y)
        stale[ny, nx] = (v + 1, v, v - 1, 0)[k % 4]
    stale[(rng.random((h, w)) < 0.3) & (stale == 0)] = 0
    return img, stale, plateaus, higher


def check_nms_frame(img, stale, plateaus, higher, t=20):
    h, w = img.shape
    sm = score_map(img, t, stale)
    kept = {(x, y) for x, y, _ in nms_model(sm, w, h)}
    for pl in plateaus:
        scores = {int(sm[y, x]) for x, y in pl}
        assert len(scores) == 1 and scores != {0}, pl
        assert all(p in kept for p in pl), pl                      # kept: equal neighbours do not suppress
        assert len({x >> 7 for x, _ in pl}) > 1 or len({(y - 3) >> 6 for _, y in pl}) > 1, pl
    for lo, hi in higher:
        assert sm[lo[1], lo[0]] < sm[hi[1], hi[0]] and lo not in kept and hi in kept
    # stale ring bytes suppress (above), keep (equal) and lose (below) against the corner beside them
    edge_kept = [(x, y) for x, y in kept if x in (3, w - 4) or y in (3, h - 4)]
    assert edge_kept and len(edge_kept) < sum(1 for x in range(w) for y in (3, h - 4) if sm[y, x]) + 2 * h
    k = np.zeros(1 << 14, L.KP_DTYPE)
    so = stale.copy()
    n = O.gso_fast(L.ptr(img), w, h, L.ptr(so), w, h, L.ptr(k), len(k), t)
    assert [(int(a["x"]), int(a["y"]), int(a["response"])) for a in k[:n]] == nms_model(sm, w, h)
    return sm


def test_fast_nms_predicates():
    img, stale, plateaus, higher = nms_frame(FAST_W, FAST_H, 3)
    check_nms_frame(img, stale, plateaus, higher)
    # the stale byte above a corner beside it suppresses it, the equal one does not
    sm = score_map(img, 20, stale)
    kept = {(x, y) for x, y, _ in nms_model(sm, FAST_W, FAST_H)}
    assert (3, 12) not in kept and (3, 29) in kept


# ---- cap -------------------------------------------------------------------------------------------------------------
CAP = 50


def cap_frame(w, h, per_row, total):
    """`total` isolated survivors, `per_row` per row (rows 9 apart, columns spread over every tile), values varying"""
    img = np.zeros((h, w), np.uint8)
    xs = np.linspace(5, w - 6, per_row).astype(int)
    k = 0
    for y in range(5, h - 5, 9):
        for x in xs:
            if k == total:
                return img
            img[y, x] = 40 + (7 * k) % 200
            k += 1
    assert k == total
    return img


def cap_frames(w, h):
    """survivor totals CAP + 1, CAP, CAP - 1, 0 (blank), and CAP + 5 in rows of 5 (the cut falls on the first
    survivor of a row) and CAP + 3 in rows of 4 (mid-row)"""
    return np.stack([cap_frame(w, h, 7, CAP + 1), cap_frame(w, h, 7, CAP), cap_frame(w, h, 7, CAP - 1),
                     np.zeros((h, w), np.uint8), cap_frame(w, h, 5, CAP + 5), cap_frame(w, h, 4, CAP + 3)])


def test_fast_cap_predicates():
    fr = cap_frames(FAST_W, FAST_H)
    tot = []
    for f in fr:
        sv = nms_model(score_map(f, 20), FAST_W, FAST_H)
        tot.append(len(sv))
        if len(sv) > CAP:
            last, nxt = sv[CAP - 1], sv[CAP]
            tot[-1] = (len(sv), last[1] == nxt[1])           # True: the cut falls mid-row
    assert tot == [(CAP + 1, True), CAP, CAP - 1, 0, (CAP + 5, False), (CAP + 3, True)], tot
    sv = nms_model(score_map(fr[4], 20), FAST_W, FAST_H)
    assert sv[CAP][1] != sv[CAP - 1][1] and sv[CAP][0] == min(x for x, y, _ in sv if y == sv[CAP][1])


@needs_ref
def test_ref_fast_content():
    R = L.ref()
    cases = [(f, t, np.zeros_like(f)) for t in TS for f in stamp_frames(FAST_W, FAST_H, t, 10 + t)[0]]
    cases += [(f, t, np.zeros_like(f)) for t in BIG_TS for f in stamp_frames(FAST_W, FAST_H, 20, 30)[0][:1]]
    img, stale, _, _ = nms_frame(FAST_W, FAST_H, 3)
    cases += [(img, 20, stale)] + [(f, 20, np.zeros_like(f)) for f in cap_frames(FAST_W, FAST_H)]
    for f, t, st in cases:
        for nk in (CAP, 1 << 14):
            a, b = st.copy(), st.copy()
            want = L.o_fast(O, f, a, nk, t)
            k = np.zeros(nk, L.KP_DTYPE)
            n = R.gs_fast(L.img(f), L.img(b), L.ptr(k), nk, t)
            assert k[:n].tobytes() == want.tobytes() and np.array_equal(a, b), (t, nk)


# ---- GPU -------------------------------------------------------------------------------------------------------------
def run_fast(lib, fr, stale, nk, t, src=0, score=0):
    """gs_b200_fast_batch on Region views; every frame's keypoints and score map bit-exact against the oracle"""
    n, h, w = fr.shape
    S, SM = Region(fr.nbytes, src, fr, 1), Region(fr.nbytes, score, stale, seed=4)
    K, N = Region(48 * n * nk, 0, seed=5), Region(4 * n, 0, seed=6)
    rc, seen = traced(lambda: lib.gs_b200_fast_batch(S.ptr, w, h, n, SM.ptr, K.ptr, N.ptr, nk, t, stream()))
    _ok(rc)
    counts = N.read("counts").view(np.uint32)
    kps = K.read("kps").view(np.uint32).reshape(n, nk, 12)
    sm = SM.read("scoremap").reshape(n, h, w)
    assert np.array_equal(S.read("src"), fr.reshape(-1))
    for i in range(n):
        so = stale[i].copy()
        want = L.o_fast(O, fr[i], so, nk, t)
        got = np.ascontiguousarray(kps[i, :counts[i]]).view(L.KP_DTYPE).reshape(-1)
        assert counts[i] == len(want) and got.tobytes() == want.tobytes(), (i, int(counts[i]), len(want))
        assert np.array_equal(sm[i], so), i
    return seen


TAIL = ("gsb::k_row_scan", "gsb::k_nms_emit_masks")
# (name, w, src offset, score offset, first kernels): the tiled kernel with TMA, and its fall-backs
FAST_GEOMS = [("tiled-tma", FAST_W, 0, 0, ("gsb::k_fast_tiled2<true>",)),
              ("tiled-src1", FAST_W, 1, 0, ("gsb::k_fast_tiled2<false>",)),
              ("tiled-w402", FAST_W + 2, 0, 0, ("gsb::k_fast_tiled2<false>",))]
BIG_GEOMS = [("score-vec", FAST_W, 0, 0, ("gsb::k_fast_score", "gsb::k_nms_mask<true>")),
             ("score-byte", FAST_W, 0, 1, ("gsb::k_fast_score", "gsb::k_nms_mask<false>"))]


def _stamp_batch(w, t):
    frames, _ = stamp_frames(w, FAST_H, t, 10 + t)
    rng = np.random.default_rng(t)
    frames = frames + [np.zeros((FAST_H, w), np.uint8), rng.integers(0, 256, (FAST_H, w), dtype=np.uint8)]
    return np.stack(frames)


@pytest.mark.gpu
@pytest.mark.parametrize("t", TS)
@pytest.mark.parametrize("name,w,src,score,kernels", [pytest.param(*g, id=g[0]) for g in FAST_GEOMS])
def test_fast_stamps(lib, witness, name, w, src, score, kernels, t):
    fr = _stamp_batch(w, t)
    stale = np.zeros_like(fr)
    for nk in (1 << 14, 37):
        witnessed(witness, lambda: run_fast(lib, fr, stale, nk, t, src, score), kernels + TAIL,
                  "fast-stamps-%s-t%d-nk%d" % (name, t, nk))


@pytest.mark.gpu
@pytest.mark.parametrize("t", BIG_TS)
@pytest.mark.parametrize("name,w,src,score,kernels", [pytest.param(*g, id=g[0]) for g in BIG_GEOMS])
def test_fast_stamps_big_threshold(lib, witness, name, w, src, score, kernels, t):
    fr = _stamp_batch(w, 20)
    stale = np.zeros_like(fr)
    witnessed(witness, lambda: run_fast(lib, fr, stale, 1 << 14, t, src, score), kernels + TAIL,
              "fast-stamps-%s-t%d" % (name, t))


@pytest.mark.gpu
@pytest.mark.parametrize("name,w,src,score,kernels", [pytest.param(*g, id=g[0]) for g in FAST_GEOMS + BIG_GEOMS[1:]])
def test_fast_nms_and_cap(lib, witness, name, w, src, score, kernels):
    t = 20 if "score" not in name else 256
    img, stale, _, _ = nms_frame(w, FAST_H, 3)
    caps = cap_frames(w, FAST_H)
    fr = np.stack([img, caps[0], img[::-1].copy()] + list(caps[1:]))
    st = np.stack([stale, np.zeros_like(stale), stale[::-1].copy()] + [np.zeros_like(stale)] * (len(caps) - 1))

    def run():
        return run_fast(lib, fr, st, CAP, t, src, score) | run_fast(lib, fr, st, 1 << 14, t, src, score)
    witnessed(witness, run, kernels + TAIL, "fast-nms-cap-%s" % name)


@pytest.mark.gpu
def test_fast_foreign_score_map(lib, witness):
    """the single-image gs_fast with a score map of another size: k_fast_score writes what fits, the NMS reads 0 beyond"""
    from grayskull_b200 import api
    frames, _ = stamp_frames(FAST_W, FAST_H, 20, 30)
    img, stale, _, _ = nms_frame(FAST_W, FAST_H, 3)

    def run():
        seen = set()
        for f in frames[:2] + [img]:
            for sh, sw in ((FAST_H - 50, FAST_W - 77), (FAST_H + 3, FAST_W + 5)):
                a = np.random.default_rng(sw).integers(0, 256, (sh, sw), dtype=np.uint8)
                b = a.copy()
                got = []
                _, s = traced(lambda: got.append(api.gs_fast(f, a, 3000, 20)))
                want = L.o_fast(O, f, b, 3000, 20)
                assert got[0].tobytes() == want.tobytes() and np.array_equal(a, b), (sh, sw)
                seen |= s
        return seen
    witnessed(witness, run, ["gsb::k_fast_score", "gsb::k_nms_mask<false>"] + list(TAIL), "fast-foreign-score-map")


# ======================================================================================================================
# B. ORB
# ======================================================================================================================
ORB_W, ORB_H = 640, 160
MARGIN = 15


def isolated(w, h, extra):
    """positions >= 4 apart in x or y: `extra` first, then a 4-px lattice from row 13 (one lattice row in the margin)"""
    occ = np.zeros((h + 8, w + 8), bool)
    out = []
    for x, y in list(extra) + [(x, y) for y in range(13, h - 3, 4) for x in range(3, w - 3, 4)]:
        if 3 <= x < w - 3 and 3 <= y < h - 3 and not occ[y + 4 - 3:y + 4 + 4, x + 4 - 3:x + 4 + 4].any():
            occ[y + 4, x + 4] = True
            out.append((x, y))
    return out


def select_frame(w, h, seed):
    """isolated bright pixels (each a dark 16-arc corner with response = its value): mostly 100, some 99 and 101, and
    candidates on the rows and columns 14, 15, w - 16, w - 15 on either side of the 15-px margin"""
    rng = np.random.default_rng(seed)
    edge = [(x, y) for x in (14, 15, w - 16, w - 15) for y in range(20 + 5 * (x % 2), h - 20, 10)]
    edge += [(x, y) for y in (14, 15, h - 16, h - 15) for x in range(22 + 6 * (y % 2), w - 20, 12)]
    img = np.zeros((h, w), np.uint8)
    for x, y in isolated(w, h, edge):
        img[y, x] = rng.choice([99, 100, 100, 100, 100, 101])
    return img


def orb_order(img, nkps, t=20):
    """the reference's candidate list (raster order, capped at min(4 nkps, 5000)), its stable sort and the selected
    positions -> (candidates, sorted, index in sorted of each selected keypoint)"""
    h, w = img.shape
    cand = nms_model(score_map(img, t), w, h)[:min(4 * nkps, 5000)]
    order = sorted(range(len(cand)), key=lambda i: -min(cand[i][2], 255))
    sel = [j for j, i in enumerate(order) if MARGIN <= cand[i][0] < w - MARGIN and MARGIN <= cand[i][1] < h - MARGIN]
    return cand, [cand[i] for i in order], sel[:nkps]


ORB_NKPS = (1250, 300, 77)


def test_orb_select_predicates():
    for seed in (1, 2):
        img = select_frame(ORB_W, ORB_H, seed)
        allc = nms_model(score_map(img, 20), ORB_W, ORB_H)
        resp = np.array([r for _, _, r in allc])
        assert len(allc) > 5000 and (resp == 100).sum() > 256 and {99, 101} <= set(resp)
        # candidates on both sides of the margin, on all four borders
        xs, ys = {x for x, _, _ in allc}, {y for _, y, _ in allc}
        assert {14, 15, ORB_W - 16, ORB_W - 15} <= xs and {14, 15, ORB_H - 16, ORB_H - 15} <= ys
        for nk in ORB_NKPS:
            cand, srt, sel = orb_order(img, nk)
            cap = min(4 * nk, 5000)
            assert len(cand) == cap and allc[cap][1] == allc[cap - 1][1], nk        # the cap cuts a row
            assert len(sel) == nk
            last = sel[-1]
            assert last % 32 not in (0, 31) and (nk < 256 or last >= 256), (nk, last)  # mid rank step, mid pass
            # some margin candidates are sorted before the cap and dropped
            assert any(not (MARGIN <= c[0] < ORB_W - MARGIN and MARGIN <= c[1] < ORB_H - MARGIN) for c in srt[:last])


# ---- orientation -----------------------------------------------------------------------------------------------------
THRESH = {"7/16": 0x3ee00000, "11/16": 0x3f300000, "19/16": 0x3f980000, "39/16": 0x401c0000}
MMAX = 30600                    # 255 * (1 + .. + 15): the largest moment the axis pixels of an r = 15 disc reach


def f32bits(v):
    return int(np.float32(v).view(np.uint32))


@functools.lru_cache(maxsize=None)
def threshold_pairs(k=8, bmax=MMAX):
    """{threshold: {ulp offset: (a, b)}}: the threshold's own quotient and the k nearest distinct floats below and above
    it that a quotient fl(a / b) of integers a, b <= bmax reaches, each with its pair of smallest b"""
    b = np.arange(1, bmax + 1, dtype=np.int64)
    out = {}
    for name, bits in THRESH.items():
        T = float(np.uint32(bits).view(np.float32))
        got = {}
        for da in range(-2 * k, 2 * k + 1):
            a = np.floor(T * b).astype(np.int64) + da
            ok = (a >= 1) & (a <= bmax)
            q = (a[ok].astype(np.float32) / b[ok].astype(np.float32)).view(np.uint32).astype(np.int64) - bits
            for off, aa, bb in zip(q.tolist(), a[ok].tolist(), b[ok].tolist()):
                if off not in got or bb < got[off][1]:
                    got[off] = (aa, bb)
        below, above = sorted(o for o in got if o < 0)[-k:], sorted(o for o in got if o > 0)[:k]
        out[name] = {o: got[o] for o in below + [0] + above}
    return out


def orientation_targets(grid=40, k=8):
    """(m01, m10) targets: the quadrant axes, the x == 1 shortcut, |m01| == |m10|, the quotients next to each atanf
    threshold (k on either side) in all four quadrants, and every pair with |m01|, |m10| <= grid"""
    ks = (1, 7, MMAX)
    out = [(0, 0)] + [(0, -v) for v in ks] + [(0, v) for v in ks] + [(s * v, 0) for v in ks for s in (1, -1)]
    out += [(y, 1) for y in (-MMAX, -5, -1, 0, 1, 2, 5, MMAX)]
    out += [(sy * v, sx * v) for v in (1, 3, 255, MMAX) for sy in (1, -1) for sx in (1, -1)]
    for name, pairs in threshold_pairs(k).items():
        for off, (a, b) in sorted(pairs.items()):
            out += [(sy * a, sx * b) for sy in (1, -1) for sx in (1, -1)]
    out += [(y, x) for y in range(-grid, grid + 1) for x in range(-grid, grid + 1)]
    return list(dict.fromkeys(out))


def axis_values(m, dmin, dmax):
    """{d: value} over d in +-[dmin, dmax], values 0..255, with sum(d * value) == m"""
    s, a = (1 if m >= 0 else -1), abs(m)
    v = {}
    for d in range(dmax, dmin - 1, -1):
        v[d] = min(255, a // d)
        a -= v[d] * d
    if a:                                   # a < dmin: (dmin + 1) * a - dmin * a
        v[dmin + 1] = v.get(dmin + 1, 0) + a
        v[-dmin] = a
    assert all(0 <= x <= 255 for x in v.values()) and sum(d * x for d, x in v.items()) == abs(m), (m, v)
    return {s * d: x for d, x in v.items() if x}


def moment_patch(img, cx, cy, m01, m10, dmin=1, dmax=15):
    """write the axis pixels that give the disc at (cx, cy) the moments (m01, m10) (zero elsewhere on the axes)"""
    for d, x in axis_values(m10, dmin, dmax).items():
        img[cy, cx + d] = x
    for d, x in axis_values(m01, dmin, dmax).items():
        img[cy + d, cx] = x


def disc_moments(img, cx, cy, r):
    ys, xs = np.mgrid[-r:r + 1, -r:r + 1]
    inside = xs * xs + ys * ys <= r * r
    p = img[cy - r:cy + r + 1, cx - r:cx + r + 1].astype(np.int64) * inside
    return int((ys * p).sum()), int((xs * p).sum())


def single_patch(m01, m10, r):
    n = 2 * r + 1
    img = np.zeros((n, n), np.uint8)
    moment_patch(img, r, r, m01, m10, 1, min(r, 15))
    return img


def _oracle_angle(img, r):
    return f32bits(O.gso_compute_orientation(L.ptr(img), img.shape[1], img.shape[0], r, r, r))


ORIENT_R = (15, 16, 20)


def test_orientation_predicates():
    tg = orientation_targets()
    assert len(tg) > 6561
    for m01, m10 in tg[:-6561:7] + tg[-6561::97] + [(0, 0), (1, 1), (0, -MMAX), (-MMAX, 1)]:
        for r in ORIENT_R:
            assert disc_moments(single_patch(m01, m10, r), r, r, r) == (m01, m10)
    # each threshold is reached exactly, and its nearest integer quotients on either side are the nearest there are:
    # no pair a, b <= 30600 gives a float between them and the threshold
    for name, pairs in threshold_pairs().items():
        offs = sorted(pairs)
        assert len(offs) == 17 and offs[8] == 0, (name, offs)
        a, b = pairs[0]
        assert f32bits(np.float32(a) / np.float32(b)) == THRESH[name]
        T = float(np.uint32(THRESH[name]).view(np.float32))
        bb = np.arange(1, MMAX + 1)
        for aa in (np.floor(T * bb), np.ceil(T * bb)):
            aa = np.where(aa <= MMAX, aa, 0)
            q = (aa.astype(np.float32) / bb.astype(np.float32)).view(np.uint32).astype(np.int64) - THRESH[name]
            assert not ((q != 0) & (q > offs[7]) & (q < offs[9])).any(), name
    # the special angles
    assert _oracle_angle(single_patch(0, -7, 15), 15) == f32bits(np.pi)
    assert _oracle_angle(single_patch(7, 0, 15), 15) == f32bits(np.pi / 2)
    assert _oracle_angle(single_patch(-7, 0, 15), 15) == f32bits(-np.pi / 2)
    assert _oracle_angle(single_patch(0, 0, 15), 15) == 0


@needs_ref
def test_ref_orientation_content():
    R = L.ref()
    for m01, m10 in orientation_targets():
        for r in ORIENT_R:
            a = single_patch(m01, m10, r)
            assert f32bits(R.gs_compute_orientation(L.img(a), r, r, r)) == _oracle_angle(a, r), (m01, m10, r)


@pytest.mark.gpu
@pytest.mark.parametrize("r", ORIENT_R)
def test_orientation_single(witness, r):
    from grayskull_b200 import api
    tg = orientation_targets()
    patches = [single_patch(m01, m10, r) for m01, m10 in tg]
    want = [_oracle_angle(p, r) for p in patches]

    def run():
        got = []
        _, seen = traced(lambda: [got.append(api.gs_compute_orientation(p, r, r, r)) for p in patches])
        bad = [(tg[i], hex(f32bits(g)), hex(want[i])) for i, g in enumerate(got) if f32bits(g) != want[i]]
        assert not bad, "%d of %d angles differ, first %s" % (len(bad), len(tg), bad[:5])
        return seen
    witnessed(witness, run, ["gsb::k_orient_one"], "orientation-r%d" % r)


# ---- ORB batch: the designed discs as keypoints ----------------------------------------------------------------------
DISC_STEP, DISC_W = 34, 8 * 34 + 16           # w % 16 == 0: the TMA path of k_fast_tiled2


def disc_targets():
    """the batch path's moment targets: axis pixels at 4 <= |d| <= 15 only (the FAST stamp holds |d| <= 3)"""
    tg = [m for m in orientation_targets(grid=6, k=2) if max(abs(m[0]), abs(m[1])) <= 28000]
    return tg


def disc_frames():
    """discs on a 34-px lattice: a FAST stamp (centre 0, all 16 ring samples 255: response 255, moments 0) plus the
    axis pixels of one target each -> (frames, [(frame, x, y, target)])"""
    tg = disc_targets()
    cells = [(20 + DISC_STEP * i, 20 + DISC_STEP * j) for j in range(8) for i in range(8)]
    frames, placed = [], []
    for f0 in range(0, len(tg), len(cells)):
        img = np.zeros((DISC_W, DISC_W), np.uint8)
        for (x, y), (m01, m10) in zip(cells, tg[f0:f0 + len(cells)]):
            for dx, dy in RING:
                img[y + dy, x + dx] = 255
            moment_patch(img, x, y, m01, m10, 4, 15)
            placed.append((len(frames), x, y, (m01, m10)))
        frames.append(img)
    return frames, placed


ORB_DISC_NKPS = 2000


def test_orb_disc_predicates():
    frames, placed = disc_frames()
    kps = [L.o_orb(O, f, np.zeros_like(f), ORB_DISC_NKPS, 20) for f in frames]
    for fi, x, y, m in placed:
        assert disc_moments(frames[fi], x, y, 15) == m, (x, y, m)
        k = [a for a in kps[fi] if (a["x"], a["y"]) == (x, y)]
        assert len(k) == 1 and k[0]["response"] == 255, (x, y, m)
        assert f32bits(k[0]["angle"]) == f32bits(O.gso_atan2f(float(m[0]), float(m[1])))
    angles = {f32bits(a["angle"]) for k in kps for a in k}
    assert {0, f32bits(np.pi), f32bits(np.pi / 2), f32bits(-np.pi / 2)} <= angles


@needs_ref
def test_ref_orb_content():
    R = L.ref()
    frames = [select_frame(ORB_W, ORB_H, s) for s in (1, 2)]
    cases = [(f, nk) for f in frames for nk in ORB_NKPS] + [(f, ORB_DISC_NKPS) for f in disc_frames()[0]]
    for f, nk in cases:
        kr = np.zeros(nk, L.KP_DTYPE)
        n = R.gs_orb_extract(L.img(f), L.ptr(kr), nk, 20, L.ptr(np.zeros_like(f)))
        assert kr[:n].tobytes() == L.o_orb(O, f, np.zeros_like(f), nk, 20).tobytes(), nk


def run_orb(lib, fr, nk, t=20, src=0):
    n, h, w = fr.shape
    S, SM = Region(fr.nbytes, src, fr, 1), Region(fr.nbytes, 0, np.zeros_like(fr), 4)
    K, N = Region(48 * n * nk, 0, seed=5), Region(4 * n, 0, seed=6)
    rc, seen = traced(lambda: lib.gs_b200_orb_extract_batch(S.ptr, w, h, n, SM.ptr, K.ptr, N.ptr, nk, t, stream()))
    _ok(rc)
    counts = N.read("counts").view(np.uint32)
    kps = K.read("kps").view(np.uint32).reshape(n, nk, 12)
    for i in range(n):
        want = L.o_orb(O, fr[i], np.zeros_like(fr[i]), nk, t)
        got = np.ascontiguousarray(kps[i, :counts[i]]).view(L.KP_DTYPE).reshape(-1)
        assert counts[i] == len(want) and got.tobytes() == want.tobytes(), (i, int(counts[i]), len(want))
    return seen


ORB_TAIL = ("gsb::k_orb_select", "gsb::k_orb_moments", "gsb::k_orb_trig")
ORB_GEOMS = [("tma", 0, ("gsb::k_fast_tiled2<true>", "gsb::k_orb_brief<true>")),
             ("src1", 1, ("gsb::k_fast_tiled2<false>", "gsb::k_orb_brief<false>"))]


@pytest.mark.gpu
@pytest.mark.parametrize("nk", ORB_NKPS)
@pytest.mark.parametrize("name,src,kernels", [pytest.param(*g, id=g[0]) for g in ORB_GEOMS])
def test_orb_select(lib, witness, name, src, kernels, nk):
    fr = np.stack([select_frame(ORB_W, ORB_H, 1), np.zeros((ORB_H, ORB_W), np.uint8), select_frame(ORB_W, ORB_H, 2),
                   L.natural_like(ORB_W, ORB_H, 5)])
    witnessed(witness, lambda: run_orb(lib, fr, nk, 20, src), kernels + ORB_TAIL, "orb-select-%s-nk%d" % (name, nk))


@pytest.mark.gpu
@pytest.mark.parametrize("name,src,kernels", [pytest.param(*g, id=g[0]) for g in ORB_GEOMS])
def test_orb_discs(lib, witness, name, src, kernels):
    frames, _ = disc_frames()
    fr = np.stack(frames + [np.zeros_like(frames[0])])
    witnessed(witness, lambda: run_orb(lib, fr, ORB_DISC_NKPS, 20, src), kernels + ORB_TAIL, "orb-discs-%s" % name)


# ======================================================================================================================
# C. blobs
# ======================================================================================================================
def o_blobs(a, nb):
    h, w = a.shape
    labels, blobs = np.zeros((h, w), np.uint16), np.zeros(nb, L.BLOB_DTYPE)
    m = O.gso_blobs(L.ptr(a), w, h, L.ptr(labels), L.ptr(blobs), nb)
    return labels, blobs[:m]


def seeds(img):
    """the reference's seed positions in raster order: foreground with neither the left nor the upper pixel foreground"""
    fg = img >= 128
    left = np.zeros_like(fg); left[:, 1:] = fg[:, :-1]
    up = np.zeros_like(fg); up[1:] = fg[:-1]
    ys, xs = np.nonzero(fg & ~left & ~up)
    return list(zip(xs.tolist(), ys.tolist()))


BW, BH = 256, 24


def overflow_frame(nb, fail, same_row=0, extra=3, w=BW, h=BH, structure=True):
    """a bar down column 0 (seed 1), isolated seeds in raster order so that seed nb + 1 falls on `fail` = (x, y) after
    `same_row` seeds of its own row, then (rows below the failing seed) a labelled arm [0, 150], a run on it
    [100, 150], a run [60, 180] whose labelled contact starts mid-run, a run [20, 100] whose only contact is its last
    pixel, and `extra` seeds after them; fail None: nb seeds in all"""
    img = np.zeros((h, w), np.uint8)
    img[:, 0] = 255
    xf, yf = fail if fail else (w, h - 1)
    before = nb - 1 - same_row
    spots = [(x, y) for y in range(yf) for x in range(2 + y % 2, w, 2) if (x, y) != (xf, yf - 1)]
    for x, y in spots[:before]:
        img[y, x] = 255
    assert len(spots) >= before
    for x in range(2 + yf % 2, xf - 1, 2)[:same_row]:
        img[yf, x] = 255
    if fail:
        img[yf, xf] = 255
        if structure and yf + 5 < h:
            r = yf + 1
            img[r, 0:151] = 255
            img[r + 1, 100:151] = 255
            img[r + 2, 60:181] = 255
            img[r + 3, 20:101] = 255
            img[r + 3, 0] = 255
        for x in range(w - 2 * extra, w, 2):
            img[h - 1, x] = 255 if (x, h - 1) != (xf, yf) and x > xf + 1 else img[h - 1, x]
    return img


OVF_NB = 120


def overflow_batch():
    """one batch at nblobs = OVF_NB: seed totals nb - 1, nb, nb + 1; failing seeds at bit 0, 31, mid-word, as the first
    seed of their row, in row 0 and in the last row -> [(frame, fail)]"""
    nb = OVF_NB
    return [(overflow_frame(nb - 1, None), None), (overflow_frame(nb, None), None),
            (overflow_frame(nb, (64, 2), 5, 0, structure=False), (64, 2)),      # bit 0 of word 2, total nb + 1
            (overflow_frame(nb, (95, 2), same_row=9), (95, 2)),                 # bit 31
            (overflow_frame(nb, (49, 2), same_row=3), (49, 2)),                 # mid-word
            (overflow_frame(nb, (33, 2), same_row=0), (33, 2)),                 # the row's first seed: need = 0
            (overflow_frame(nb, (250, 0), same_row=nb - 1), (250, 0)),          # row 0 (only the bar before it)
            (overflow_frame(nb, (31, BH - 1), same_row=2), (31, BH - 1))]       # the last row


def labelled_after_overflow(img, nb):
    """the reference's mask, straight from its rule: seeds beyond the nb-th get no label, and from the (nb+1)-th seed
    on a pixel is labelled only through a labelled left or upper neighbour"""
    h, w = img.shape
    fg = img >= 128
    m = np.zeros_like(fg)
    ns, over = 0, False
    for y in range(h):
        for x in range(w):
            left = x > 0 and m[y, x - 1]
            up = y > 0 and m[y - 1, x]
            if not over:
                m[y, x] = fg[y, x]
                if fg[y, x] and not left and not up:
                    if ns == nb:
                        over, m[y, x] = True, False
                    else:
                        ns += 1
            else:
                m[y, x] = fg[y, x] and (left or up)
    return m


def test_blob_overflow_predicates():
    nb = OVF_NB
    totals = []
    for img, fail in overflow_batch():
        s = seeds(img)
        totals.append(len(s))
        if fail is None:
            continue
        assert len(s) > nb and s[nb] == fail, (fail, s[nb - 1:nb + 2])
        xf, yf = fail
        need = sum(1 for x, y in s[:nb] if y == yf)
        assert (need == 0) == (fail == (33, 2)), need
        m = labelled_after_overflow(img, nb)
        labels, _ = o_blobs(img, nb)
        assert np.array_equal(labels > 0, m)
        if yf + 5 < BH and img[yf + 1, 0:151].all():
            r = yf + 1
            assert m[r, :151].all() and m[r + 1, 100:151].all()
            assert not m[r + 2, 60:100].any() and m[r + 2, 100:181].all()          # mid-run contact, carried on
            assert not m[r + 3, 20:100].any() and m[r + 3, 100]                   # contact on the last pixel only
            assert (m[r + 2, 128:160]).all()                                     # an all-ones word via the carry
    assert totals[0] == nb - 1 and totals[1] == nb and totals[2] == nb + 1
    assert {f[0] % 32 for _, f in overflow_batch() if f} >= {0, 31, 17}
    # nblobs = 1: every frame overflows at its second seed
    for img, _ in overflow_batch():
        assert np.array_equal(o_blobs(img, 1)[0] > 0, labelled_after_overflow(img, 1))


def checkerboard(w, h):
    return (((np.arange(h)[:, None] + np.arange(w)[None, :]) % 2) * 255).astype(np.uint8)


CHK_W, CHK_H = 512, 257


def test_blob_checkerboard_predicate():
    s = seeds(checkerboard(CHK_W, CHK_H))
    assert len(s) >= 65535
    labels, blobs = o_blobs(checkerboard(CHK_W, CHK_H), 65534)
    assert len(blobs) == 65534 and labels.max() == 65534 and (labels > 0).sum() == 65534


# ---- runs, unions, statistics ----------------------------------------------------------------------------------------
RUN_WIDTHS = (1023, 1024, 1025, 2049)


def runs_frame(w, h=12, seed=0):
    """rows: all ones; alternating bits; runs across the 1024- and 2048-pixel chunk seams and word seams; single
    pixels at x = 1023, 1024, 2048; a random row; vertical contacts between them"""
    rng = np.random.default_rng(seed + w)
    img = np.zeros((h, w), np.uint8)
    img[0] = 255
    img[2, ::2] = 255
    img[3, 1::2] = 255
    for a, b in ((1000, 1050), (1020, 1023), (1024, 1030), (2040, 2048), (31, 64), (990, 1023)):
        img[5, min(a, w - 1):min(b, w - 1) + 1] = 255
    for x in (1023, 1024, 2048):
        if x < w:
            img[7, x] = 255
    img[8] = (rng.random(w) < 0.6) * 255
    img[9, 500:] = 255
    img[10, : w // 2] = 255
    img[4, 1010:1040] = 255
    img[11, w - 1] = 255
    return img


def spiral(n, pitch=2):
    """a square spiral of 1-px lines `pitch` apart, drawn inwards from the top-left corner: each ring's top row, right
    column, bottom row and left column, up to the row where the next ring's top row starts"""
    img = np.zeros((n, n), np.uint8)
    o = 0
    while n - 1 - 2 * o > pitch:
        e = n - 1 - o
        img[o, o:e + 1] = img[o:e + 1, e] = img[e, o:e + 1] = 255
        img[o + pitch:e + 1, o] = 255
        img[o + pitch, o:o + pitch + 1] = 255
        o += pitch
    return img


def union_frame(w=256, h=256):
    """a spiral, two interleaved spirals, a comb joined only in its last row, staircases (1-px steps: separate blobs;
    2-px steps: one blob), nested U shapes"""
    img = np.zeros((h, w), np.uint8)
    img[2:63, 2:63] = spiral(61)
    s1, s2 = spiral(61, 4), spiral(57, 4)
    img[2:63, 70:131] = s1
    img[4:61, 72:129] |= s2
    img[70:130, 2:120:2] = 255
    img[130, 2:119] = 255
    for i in range(40):
        img[140 + i, 5 + i] = 255
        img[140 + i, 60 + i:62 + i] = 255
    for k in range(8):
        a, b = 150 + 4 * k, 250 - 4 * k
        img[140 + 4 * k:230 - 4 * k, a] = 255
        img[140 + 4 * k:230 - 4 * k, b] = 255
        img[229 - 4 * k, a:b + 1] = 255
    return img


def n_components(img):
    from scipy import ndimage
    return ndimage.label(img >= 128)[1]


def test_blob_union_predicates():
    img = union_frame()
    from scipy import ndimage
    lab = ndimage.label(img >= 128)[0]
    # the spiral is one component with many seeds, labelled by its raster-first seed (the smallest seed number)
    sp = lab[2:63, 2:63]
    assert len(set(sp[sp > 0].tolist())) == 1
    sp_seeds = [s for s in seeds(img) if 2 <= s[0] < 63 and 2 <= s[1] < 63]
    assert len(sp_seeds) > 10
    labels, blobs = o_blobs(img, 1000)
    assert labels[2, 2] == seeds(img).index((2, 2)) + 1 == labels[2:63, 2:63].max()
    # interleaved spirals stay two components, the comb is one with its teeth as seeds, 1-px staircases are not joined
    assert len(set(lab[2:63, 70:131][lab[2:63, 70:131] > 0].tolist())) == 2
    comb = lab[70:131, 2:120]
    assert len(set(comb[comb > 0].tolist())) == 1 and len([s for s in seeds(img) if s[1] == 70 and s[0] < 120]) == 59
    assert len(set(lab[140:180, 5:45][lab[140:180, 5:45] > 0].tolist())) == 40
    assert len(set(lab[140:180, 60:102][lab[140:180, 60:102] > 0].tolist())) == 1
    assert n_components(img) == len(blobs)


def test_blob_runs_predicates():
    for w in RUN_WIDTHS:
        img = runs_frame(w)
        assert img[0].all() and (img[2, ::2] == 255).all() and not img[2, 1::2].any()
        row = img[5] >= 128
        assert row[1022] and (w <= 1024 or row[1023] and row[1024])     # a run across the chunk seam
        labels, blobs = o_blobs(img, 65534)
        assert n_components(img) == len(blobs) > 500


STAT_N = 4096


def test_blob_stat_predicates():
    xs = np.arange(STAT_N, dtype=np.uint64)
    assert int(xs.sum()) * STAT_N >= U32                        # the x sum of the full frame wraps
    labels, blobs = o_blobs(np.full((STAT_N, STAT_N), 255, np.uint8), 4)
    assert len(blobs) == 1 and blobs[0]["cx"] == (int(xs.sum()) * STAT_N % U32) // STAT_N ** 2
    b = border_frame(300, 200)
    _, bl = o_blobs(b, 10)
    assert (bl[0]["bx"], bl[0]["by"], bl[0]["bw"], bl[0]["bh"]) == (0, 0, 300, 200)


def border_frame(w, h):
    img = np.zeros((h, w), np.uint8)
    img[0], img[-1], img[:, 0], img[:, -1] = 255, 255, 255, 255
    img[h // 2, w // 3:w // 2] = 255
    return img


# ---- corners ---------------------------------------------------------------------------------------------------------
def corner_frame(w=160, h=120):
    """diamonds, squares, horizontal / vertical lines, 4-connected diagonal and anti-diagonal lines, single pixels"""
    img = np.zeros((h, w), np.uint8)
    ys, xs = np.mgrid[0:h, 0:w]
    for cx, cy, r in ((20, 20, 8), (60, 20, 1), (100, 25, 12)):
        img[np.abs(xs - cx) + np.abs(ys - cy) <= r] = 255
    img[50:60, 5:15] = 255
    img[50:51, 30:50] = 255
    img[45:65, 60:61] = 255
    for i in range(15):
        img[70 + i, 80 + i:82 + i] = 255                  # 4-connected diagonal: x - y ties along it
        img[70 + i, 119 - i:121 - i] = 255                # anti-diagonal: x + y ties
        img[90 + i, 130 + i] = 255                        # 1-px steps: single pixels
    img[100, 10] = img[110, 150] = img[119, 159] = img[0, 0] = 255
    return img


def corner_ties(img, labels, b):
    """how many pixels of the blob reach each extreme (x + y min / x - y max / x + y max / x - y min)"""
    m = (labels == b["label"]) & (img >= 128)
    ys, xs = np.nonzero(m)
    s, d = xs + ys, xs - ys
    return [(s == s.min()).sum(), (d == d.max()).sum(), (s == s.max()).sum(), (d == d.min()).sum()]


def o_corners(img, labels, blob):
    c = np.zeros((4, 2), np.uint32)
    O.gso_blob_corners(L.ptr(img), img.shape[1], img.shape[0], L.ptr(labels), L.ptr(blob), L.ptr(c))
    return c


def test_blob_corner_predicates():
    img = corner_frame()
    labels, blobs = o_blobs(img, 100)
    ties = [corner_ties(img, labels, b) for b in blobs]
    assert sum(1 for t in ties if max(t) > 1) >= 5 and any(t == [1, 1, 1, 1] for t in ties)
    assert any(min(t) > 1 for t in ties)                                    # a diamond: every extreme ties


@needs_ref
def test_ref_blobs_content():
    R = L.ref()
    cases = [(img, OVF_NB) for img, _ in overflow_batch()] + [(img, 1) for img, _ in overflow_batch()[:3]]
    cases += [(checkerboard(CHK_W, CHK_H), 65534), (union_frame(), 1000), (border_frame(300, 200), 10),
              (corner_frame(), 100)] + [(runs_frame(w), 500) for w in RUN_WIDTHS]
    for img, nb in cases:
        lo, bo = o_blobs(img, nb)
        lr, br = np.zeros(img.shape, np.uint16), np.zeros(nb, L.BLOB_DTYPE)
        m = R.gs_blobs(L.img(img), L.ptr(lr), L.ptr(br), nb)
        assert np.array_equal(lr, lo) and L.blob_fields(br[:m]) == L.blob_fields(bo), (img.shape, nb)
        if img.shape == (120, 160):
            for j in range(len(bo)):
                c = np.zeros((4, 2), np.uint32)
                R.gs_blob_corners(L.img(img), L.ptr(lr), L.ptr(br[j:j + 1]), L.ptr(c))
                assert np.array_equal(c, o_corners(img, lo, bo[j:j + 1])), j


BLOB_KERNELS = ["gsb::k_blob_mask", "gsb::k_blob_seed", "gsb::k_row_scan", "gsb::k_blob_overflow", "gsb::k_blob_runs",
                "gsb::k_blob_union", "gsb::k_blob_label", "gsb::k_blob_compact"]


def run_blobs(lib, fr, nb, src=0):
    n, h, w = fr.shape
    S, LB = Region(fr.nbytes, src, fr, 1), Region(2 * n * w * h, 2, seed=2)
    B, N = Region(32 * n * nb, 0, seed=3), Region(4 * n, 0, seed=4)
    rc, seen = traced(lambda: lib.gs_b200_blobs_batch(S.ptr, w, h, n, LB.ptr, B.ptr, N.ptr, nb, stream()))
    _ok(rc)
    labels = LB.read("labels").view(np.uint16).reshape(n, h, w)
    blobs, counts = B.read("blobs").view(L.BLOB_DTYPE).reshape(n, nb), N.read("counts").view(np.uint32)
    for i in range(n):
        wl, wb = o_blobs(fr[i], nb)
        assert counts[i] == len(wb) and np.array_equal(labels[i], wl), (i, int(counts[i]), len(wb))
        assert L.blob_fields(blobs[i, :counts[i]]) == L.blob_fields(wb), i
    return seen


@pytest.mark.gpu
@pytest.mark.parametrize("src", (0, 1))
def test_blob_overflow(lib, witness, src):
    fr = np.stack([img for img, _ in overflow_batch()])

    def run():
        return run_blobs(lib, fr, OVF_NB, src) | run_blobs(lib, fr, 1, src) | run_blobs(lib, fr, OVF_NB - 1, src)
    witnessed(witness, run, BLOB_KERNELS, "blobs-overflow-src%d" % src)


@pytest.mark.gpu
def test_blob_checkerboard(lib, witness):
    c = checkerboard(CHK_W, CHK_H)
    fr = np.stack([c, 255 - c, np.zeros_like(c), overflow_frame(OVF_NB, (95, 2), 9, w=CHK_W, h=CHK_H)])
    witnessed(witness, lambda: run_blobs(lib, fr, 65534), BLOB_KERNELS, "blobs-checkerboard-65534")


@pytest.mark.gpu
@pytest.mark.parametrize("w", RUN_WIDTHS)
def test_blob_runs(lib, witness, w):
    fr = np.stack([runs_frame(w, seed=s) for s in range(3)] + [np.zeros((12, w), np.uint8)])
    witnessed(witness, lambda: run_blobs(lib, fr, 500) | run_blobs(lib, fr, 3), BLOB_KERNELS, "blobs-runs-w%d" % w)


@pytest.mark.gpu
def test_blob_unions(lib, witness):
    u = union_frame()
    fr = np.stack([u, u[::-1].copy(), u[:, ::-1].copy(), u.T.copy()])
    witnessed(witness, lambda: run_blobs(lib, fr, 1000) | run_blobs(lib, fr, 7), BLOB_KERNELS, "blobs-unions")


@pytest.mark.gpu
def test_blob_statistics(lib, witness):
    fr = np.stack([np.full((STAT_N, STAT_N), 255, np.uint8), border_frame(STAT_N, STAT_N)])
    witnessed(witness, lambda: run_blobs(lib, fr, 4), BLOB_KERNELS, "blobs-4096-wrap")


@pytest.mark.gpu
def test_blob_corners(lib, witness):
    img = corner_frame()
    h, w = img.shape
    labels, blobs = o_blobs(img, 100)

    def run():
        seen = set()
        S, LB = Region(img.nbytes, 1, img, 1), Region(labels.nbytes, 2, labels, seed=2)
        for j in range(len(blobs)):
            B, CO = Region(32, 0, blobs[j:j + 1], seed=3), Region(32, 0, seed=4)
            rc, s = traced(lambda: lib.gs_b200_blob_corners(S.ptr, w, h, LB.ptr, B.ptr, CO.ptr, stream()))
            _ok(rc)
            got = CO.read("corners").view(np.uint32).reshape(4, 2)
            assert np.array_equal(got, o_corners(img, labels, blobs[j:j + 1])), (j, corner_ties(img, labels, blobs[j]))
            seen |= s
        return seen
    witnessed(witness, run, ["gsb::k_blob_corners"], "blob-corners")
