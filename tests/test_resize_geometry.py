"""gs_resize's geometry: its fp32 coordinate map, the host's choice of kernel, and the source rectangle that
k_resize_tiled stages per dst tile.

k_resize_tiled loads, with one TMA box, the source rectangle that a 128 x 64 dst tile reads.  The host sizes the box
from the ratio with a fixed spare (resample.cu); a tile whose rectangle is larger stops the kernel with __trap(), and
a trap leaves the CUDA context unusable.  Each tile's rectangle comes from the reference's fp32 map
sx = ((x + 0.5f) * sw) / dw - 0.5f, whose rounding grows with the source size, so the staged kernel only takes sources
below RT_SRC_LIMIT in both dimensions, where the box is proven to cover every tile; larger ones take k_resize.

  * CPU: axis32 / resize32 restate resize_axis and the four-tap sum in numpy float32 (IEEE round to nearest, as the
    _rn intrinsics) and are checked against the C oracle, sizes past 2^24 included, where a tap the reference puts
    past the source is clamped to the last pixel.  resize_route restates the host's dispatch.  Every tile of every
    swept geometry that resize_route sends to k_resize_tiled must fit the box, and the exact-2:1 shortcut's size
    bound (2 * dw * dw < 2^24) must be exactly the range where the map is 2x + 0.5.
  * GPU: geometries at each change of route (the two sources that trapped before the size limit, each limit of
    k_resize_tiled, the 2:1 shortcut per axis, k_resize's pair loads, sizes of 1) and the clamped taps, every output
    byte against the oracle from a poisoned dst, with the kernel resize_route names witnessed.  The CPU bound check
    runs on each first, so a box too small fails here instead of trapping on the device.
The whole file, CPU and GPU tests, ran in 75 s on one H100 80GB (700 W power limit).
"""
import numpy as np
import pytest

import _calls as calls
import _libs as L
from _gpu import O, Region, frames, lib, stream, traced, witness, witnessed  # noqa: F401

F32 = np.float32
M32 = 0xFFFFFFFF
POISON = calls.POISON
CONST = L.tile_constants()
TILE = {"x": 128, "y": 8 * CONST["RS_ROWS"]}          # a k_resize_tiled CTA's dst tile
MAX_PITCH, MAX_ROWS = 1024, 256                          # a TMA box is at most 256 words by 256 rows
SRC_LIMIT = CONST.get("RT_SRC_LIMIT", 2 ** 32)          # csrc/ without the limit staged sources of every size


# ---- the fp32 model ---------------------------------------------------------------------------------------------------
def axis32(i, s, d, clamp=True):
    """resize_axis (resample.cuh, reference grayskull.h:174-180) for dst coordinates i of an axis from s to d pixels
    (d may be an array broadcast with i) -> (i0, i1, frac).  clamp=False leaves i0 as the reference computes it, which
    above 2^24 can lie past the source."""
    sx = (np.asarray(i).astype(F32) + F32(0.5)) * F32(s)
    sx = sx / np.asarray(d).astype(F32) - F32(0.5)
    sx = np.maximum(F32(0), np.minimum(sx, F32(s) - F32(1)))
    i0 = sx.astype(np.int64)                             # truncation: sx >= 0
    i1, frac = np.minimum(i0 + 1, s - 1), sx - i0.astype(F32)
    return np.minimum(i0, s - 1) if clamp else i0, i1, frac


def resize32(a, dw, dh):
    """gs_resize of one frame in float32: axis32 on both axes, then ((c * wx) * wy) summed left to right and truncated
    (reference grayskull.h:181-185)"""
    sh, sw = a.shape
    x0, x1, dx = axis32(np.arange(dw), sw, dw)
    y0, y1, dy = axis32(np.arange(dh), sh, dh)
    omx, omy, dy = F32(1) - dx, (F32(1) - dy)[:, None], dy[:, None]
    c = a.astype(F32)
    r0, r1 = c[y0], c[y1]
    p = r0[:, x0] * omx * omy
    p = p + r0[:, x1] * dx * omy
    p = p + r1[:, x0] * omx * dy
    p = p + r1[:, x1] * dx * dy
    return p.astype(np.uint8)


# ---- the host's dispatch ----------------------------------------------------------------------------------------------
def tiled_box(sw, sh, dw, dh):
    """k_resize_tiled's box as the host sizes it: (pitch in bytes, rows)"""
    cols = int(127.0 * (sw / dw)) + 22
    return (cols + 15) // 16 * 16, int((TILE["y"] - 1.0) * (sh / dh)) + 6


def resize_route(sw, sh, dw, dh, src_off=0, dst_off=0):
    """the kernel gs_b200_resize_batch launches (resample.cu), for a source and a dst at byte offsets src_off / dst_off
    of 256-byte aligned allocations"""
    if sw == (2 * dw) & M32 and sh == (2 * dh) & M32 and ((2 * dw) & M32) * dw < 2 ** 24 and \
            ((2 * dh) & M32) * dh < 2 ** 24:                # exact 2:1: gs_b200_downsample_batch
        return "gsb::k_downsample_vec" if sw % 16 == 0 and src_off % 16 == 0 and dst_off % 8 == 0 else \
            "gsb::k_downsample_generic"
    vec = "true" if dw % 4 == 0 and dst_off % 4 == 0 else "false"
    if sw < SRC_LIMIT and sh < SRC_LIMIT:
        pitch, rows = tiled_box(sw, sh, dw, dh)
        pairs_case = sw % 8 == 0 and src_off % 8 == 0 and sw == (2 * dw) & M32
        tma = sw % 16 == 0 and src_off % 16 == 0
        map_ok = sw * sh < 2 ** 40                          # the driver's bound on the tensor map's frame stride
        if pitch * rows <= CONST["RT_MAX_BYTES"] and pitch <= MAX_PITCH and rows <= MAX_ROWS and not pairs_case and \
                tma and map_ok:
            return "gsb::k_resize_tiled<%s>" % vec
    return "gsb::k_resize<%s>" % vec


def tiled(g):
    return resize_route(*g).startswith("gsb::k_resize_tiled")


# ---- the staged rectangle of each tile --------------------------------------------------------------------------------
def rect_need(s, d, t0, axis):
    """the box columns (axis "x": from the 16-byte aligned start) or rows the tiles starting at dst coordinate t0 read,
    as k_resize_tiled computes them from the tile's first and last pixel (the map is monotonic)"""
    a0 = axis32(t0, s, d)[0]
    a1 = axis32(np.minimum(t0 + TILE[axis] - 1, d - 1), s, d)[0]
    return a1 + 2 - (a0 & ~15 if axis == "x" else a0)


def axis_overflow(s, d, axis, box, chunk=1 << 21):
    """(first dst coordinate, need) of the last tile of the axis whose rectangle is larger than box, or None.  Tiles are
    checked in chunks from the last one, where sx and its rounding are largest."""
    n = -(-d // TILE[axis])
    for hi in range(n, 0, -chunk):
        t0 = np.arange(max(hi - chunk, 0), hi, dtype=np.int64) * TILE[axis]
        need = rect_need(s, d, t0, axis)
        bad = np.flatnonzero(need > box)
        if bad.size:
            return int(t0[bad[-1]]), int(need[bad[-1]])
    return None


def overflows(sw, sh, dw, dh):
    """the tiles of a geometry routed to k_resize_tiled whose rectangle does not fit the box: [(axis, tile, need, box)]"""
    if not tiled((sw, sh, dw, dh)):
        return []
    pitch, rows = tiled_box(sw, sh, dw, dh)
    out = []
    for axis, s, d, box in (("x", sw, dw, pitch), ("y", sh, dh, rows)):
        o = axis_overflow(s, d, axis, box)
        if o:
            out.append((axis,) + o + (box,))
    return out


# The swept axis runs against a fixed other axis that takes the staged kernel at every ratio it accepts: rows 1 -> 64
# (6 box rows) for the x sweeps, columns 16 -> 64 (a 64-byte pitch) for the y sweeps.
def sweep_geometry(axis, s, d):
    return (s, 1, d, 64) if axis == "x" else (16, s, 64, d)


# the two geometries that trapped before the size limit: 73 of the first one's 71,886 tiles need 498 bytes of its
# 496-byte pitch, 190 of the second one's 190,787 tiles 74 of its 73 rows
TRAPPED = {"x": (34_376_752, 1, 9_201_328, 1), "y": (16, 13_162_541, 16, 12_210_337)}


# ---- CPU: the model --------------------------------------------------------------------------------------------------
def _model_geometries():
    rng = np.random.default_rng(2024)
    size = lambda: int(rng.choice([1, 2, 3, int(rng.integers(1, 40)), int(rng.integers(40, 400))]))  # noqa: E731
    out = [(1, 1, 1, 1), (1, 1, 7, 5), (7, 5, 1, 1), (1, 37, 9, 1), (300, 1, 1, 200), (272, 60, 200, 50),
           (264, 60, 132, 50), (5794, 2, 2897, 1), (5792, 2, 2896, 1)]
    while len(out) < 300:
        out.append((size(), size(), size(), size()))
    return out


def test_resize32_matches_the_oracle():
    """resize32 against the C oracle's literal fp32 evaluation: down- and up-scaling, sources and targets of 1 pixel"""
    Oc = L.oracle()
    for k, (sw, sh, dw, dh) in enumerate(_model_geometries()):
        a = np.random.default_rng(k).integers(0, 256, (sh, sw), dtype=np.uint8)
        assert np.array_equal(resize32(a, dw, dh), L.o_resize(Oc, a, dw, dh)), (sw, sh, dw, dh)


@pytest.mark.parametrize("s,d", [(34_376_752, 9_201_328), (13_162_541, 12_210_337), (2 ** 22 - 1, 3_890_000),
                                 (5, 2 ** 24 + 5), (16_777_219, 16_000_000)])
def test_resize32_matches_the_oracle_on_long_rows(s, d):
    """the map where fp32 rounds: sizes and coordinates past 2^22 and 2^24, on one-row images (the two trapped
    geometries' axes and a clamped tap among them)"""
    a = np.random.default_rng(s).integers(0, 256, (1, s), dtype=np.uint8)
    assert np.array_equal(resize32(a, d, 1), L.o_resize(L.oracle(), a, d, 1))


# For about half the sizes above 2^24, (float)s - 1.0f rounds to s or past it, and the reference's first tap can lie
# past the source.  resize_axis, the oracle and axis32 take the last pixel there.
CLAMPED = {"x": (16_777_219, 2, 16_000_000, 3), "y": (2, 16_777_219, 3, 16_000_000)}


def test_taps_past_the_source_are_clamped_at_weight_one():
    """the geometries with a tap past the source, where it has weight 1 - frac = 1: the last pixel is the result"""
    for s, d in ((34_376_752, 9_201_328), (16_777_219, 16_000_000)):
        i0, _, frac = axis32(np.arange(d), s, d, clamp=False)
        past = i0 > s - 1
        assert past.any() and np.all(frac[past] == 0), (s, d)
        assert np.all(axis32(np.arange(d), s, d)[0][past] == s - 1)


# ---- CPU: the box covers every tile ----------------------------------------------------------------------------------
def test_source_size_limit_is_in_csrc():
    assert CONST.get("RT_SRC_LIMIT") == 2 ** 22, "resample.cu: k_resize_tiled needs its source-size limit"


def _small_sweep(axis):
    """every source size up to 1100 (for x the multiples of 16, the sizes TMA takes) at every target size up to 2200
    that takes k_resize_tiled -> [geometry whose rectangle overflows]"""
    bad = []
    for s in range(16 if axis == "x" else 1, 1101, 16 if axis == "x" else 1):
        staged = [(d, tiled_box(*g)[axis == "y"]) for d in range(1, 2201) for g in [sweep_geometry(axis, s, d)]
                  if tiled(g)]
        ds, boxes = np.array(staged, np.int64).T
        n = -(-ds // TILE[axis])
        first = np.repeat(np.cumsum(n) - n, n)
        t0 = (np.arange(n.sum()) - first) * TILE[axis]
        over = rect_need(s, np.repeat(ds, n), t0, axis) > np.repeat(boxes, n)
        bad += [sweep_geometry(axis, s, int(d)) for d in np.unique(np.repeat(ds, n)[over])]
    return bad


def _ratios(axis):
    """ratios from 1:2 up to the largest the staged kernel takes on the axis, on a grid of about 0.1"""
    top = (MAX_PITCH - 22) / 127 if axis == "x" else (MAX_ROWS - 6) / (TILE["y"] - 1)
    return np.linspace(0.5, top, int((top - 0.5) / 0.1) + 1)


def _power_sweep(axis):
    """source sizes at and around each power of two from 2^12 to 2^31 (x: multiples of 16) at each ratio"""
    step = 16 if axis == "x" else 1
    out = set()
    for k in range(12, 32):
        for s in (2 ** k - step, 2 ** k, 2 ** k + step):
            for r in _ratios(axis):
                d = min(int(round(s / r)), M32)
                out.add(sweep_geometry(axis, s, d))
    return sorted(out)


@pytest.mark.parametrize("axis", ["x", "y"])
def test_every_tile_fits_its_box(axis):
    """every tile of every swept geometry that takes k_resize_tiled reads inside the box the host sized: sources up to
    1100 at every target size up to 2200, sources around the powers of two at a grid of ratios, the two geometries that
    trapped"""
    bad = []
    for g in [TRAPPED[axis]] + _power_sweep(axis):
        bad += [(g, o) for o in overflows(*g)]
    bad += [(g, "small sizes") for g in _small_sweep(axis)]
    assert not bad, "%d geometries read past k_resize_tiled's box ((sw, sh, dw, dh), (axis, tile, need, box)): %s" % (
        len(bad), bad[:12])


def test_power_sweep_reaches_the_size_limit():
    """the largest source sizes the sweeps stage are right below the size limit, and the limit itself is not staged"""
    for axis, step in (("x", 16), ("y", 1)):
        staged = [g for g in _power_sweep(axis) if tiled(g)]
        assert max(g[0] if axis == "x" else g[1] for g in staged) == SRC_LIMIT - step
        assert not tiled(sweep_geometry(axis, SRC_LIMIT, SRC_LIMIT))
    assert [resize_route(*g) for g in TRAPPED.values()] == ["gsb::k_resize<true>"] * 2


# ---- CPU: the exact-2:1 shortcut -------------------------------------------------------------------------------------
def test_two_to_one_map_is_exact_exactly_where_the_shortcut_is_taken():
    """resize_axis maps x to 2x + 0.5 (taps 2x, 2x + 1 at weight 0.5, gs_downsample's sum) for every x of every
    dw <= 2896, and not for dw = 2897: the host's bound 2 * dw * dw < 2^24 is sufficient and tight"""
    exact = []
    for dw in range(1, 2898):
        x = np.arange(dw)
        i0, i1, fr = axis32(x, 2 * dw, dw)
        exact.append(bool(np.all(i0 == 2 * x) and np.all(i1 == 2 * x + 1) and np.all(fr == F32(0.5))))
    assert exact.index(False) == 2896, "the first dw whose map is not 2x + 0.5"
    for dw in (1, 2, 1000, 2896, 2897, 2900):
        for g in ((2 * dw, 40, dw, 20), (64, 2 * dw, 32, dw)):
            assert resize_route(*g).startswith("gsb::k_downsample") == (dw <= 2896), g


# ---- the GPU cases, chosen with resize_route -------------------------------------------------------------------------
def straddle(geometry, values):
    """the first of `values` whose geometry does not take k_resize_tiled, after one that does -> (inside, outside)"""
    for v0, v in zip(values, values[1:]):
        if not tiled(geometry(v)):
            assert tiled(geometry(v0))
            return geometry(v0), geometry(v)
    raise AssertionError("no value leaves k_resize_tiled")


# each limit of k_resize_tiled in turn, with the others well inside: (inside, outside)
LIMITS = {
    "pitch": straddle(lambda dw: (1600, 1, dw, 64), range(700, 0, -1)),         # 1024-byte pitch, then 1040
    "rows": straddle(lambda dh: (16, 1000, 64, dh), range(1000, 0, -1)),        # 256 rows, then 257
    "bytes": straddle(lambda dh: (512, 400, 133, dh), range(400, 0, -1)),       # a 512-byte pitch: 128 rows, then 129
    # the source-size limit, 2^22, at the ratio of the trapped row geometry
    "size_x": ((2 ** 22 - 16, 1, 3_890_000, 1), (2 ** 22, 1, 3_890_000, 1)),
    "size_y": ((16, 2 ** 22 - 1, 16, 3_890_000), (16, 2 ** 22, 16, 3_890_000)),
}


def limits_failed(g):
    """which of k_resize_tiled's limits a geometry fails"""
    pitch, rows = tiled_box(*g)
    fails = dict(pitch=pitch > MAX_PITCH, rows=rows > MAX_ROWS, bytes=pitch * rows > CONST["RT_MAX_BYTES"],
                 size_x=g[0] >= SRC_LIMIT, size_y=g[1] >= SRC_LIMIT)
    return [k for k, v in fails.items() if v]


def case(name, g, kernel=None, src_off=0, dst_off=0, n=3):
    return pytest.param(g, src_off, dst_off, n, kernel, id="%s-%s" % (name, "x".join(map(str, g))))


CASES = [case("trapped", g, "gsb::k_resize<true>", n=1) for g in TRAPPED.values()]
CASES += [case("clamped", CLAMPED["x"], "gsb::k_resize<true>", n=1),
          case("clamped", CLAMPED["y"], "gsb::k_resize<false>", n=1)]
for name, (inside, outside) in LIMITS.items():
    n = 1 if name.startswith("size") else 3
    CASES += [case(name + "-inside", inside, n=n), case(name + "-outside", outside, n=n)]
CASES += [
    # the exact-2:1 shortcut to gs_downsample in each axis, at its bound and past it (5800: sw % 8 == 0, pair loads)
    case("down-x2896", (5792, 40, 2896, 20), "gsb::k_downsample_vec"),
    case("down-y2896", (64, 5792, 32, 2896), "gsb::k_downsample_vec"),
    case("down-x2897", (5794, 40, 2897, 20), "gsb::k_resize<false>"),
    case("down-x2900", (5800, 40, 2900, 20), "gsb::k_resize<true>"),
    case("down-y2897", (64, 5794, 32, 2897), "gsb::k_resize<true>"),
    # exact 2:1 in x only: k_resize's 64-bit pair loads on an 8-byte aligned source, byte gathers 4 bytes off, and
    # dw % 4 = 1, 2, 3 (sw % 8 != 0: gathers) where the last thread of a row writes 1 to 3 bytes
    case("pairs", (528, 40, 264, 30), "gsb::k_resize<true>"),
    case("pairs-src4", (528, 40, 264, 30), "gsb::k_resize<true>", src_off=4),
    case("pairs-dw1", (530, 40, 265, 30), "gsb::k_resize<false>"),
    case("pairs-dw2", (532, 40, 266, 30), "gsb::k_resize<false>"),
    case("pairs-dw3", (534, 40, 267, 30), "gsb::k_resize<false>"),
    # sizes of 1 on k_resize, and where the staged kernel takes them: it needs sw % 16 == 0 and dw >= sw / 7.9, so
    # neither sw = 1 nor dw = 1
    case("sw1", (1, 40, 7, 30), "gsb::k_resize<false>"),
    case("dw1", (64, 40, 1, 30), "gsb::k_resize<false>"),
    case("sh1", (50, 1, 36, 6), "gsb::k_resize<true>"),
    case("dh1", (50, 40, 36, 1), "gsb::k_resize<true>"),
    case("src1", (1, 1, 9, 5), "gsb::k_resize<false>"),
    case("dst1", (64, 48, 1, 1), "gsb::k_resize<false>"),
    case("all1", (1, 1, 1, 1), "gsb::k_resize<false>"),
    case("tiled-sh1", (64, 1, 48, 5), "gsb::k_resize_tiled<true>"),
    case("tiled-dh1", (64, 3, 48, 1), "gsb::k_resize_tiled<true>"),
    case("tiled-sh1-dh1", (64, 1, 48, 1), "gsb::k_resize_tiled<true>"),
]


def test_limit_cases_straddle_one_limit_each():
    """inside: every limit holds, the named one with no room left for the step; outside: only the named limit fails"""
    edge = dict(pitch=lambda g: tiled_box(*g)[0] == MAX_PITCH, rows=lambda g: tiled_box(*g)[1] == MAX_ROWS,
                bytes=lambda g: np.prod(tiled_box(*g)) == CONST["RT_MAX_BYTES"],
                size_x=lambda g: g[0] == SRC_LIMIT - 16, size_y=lambda g: g[1] == SRC_LIMIT - 1)
    for name, (inside, outside) in LIMITS.items():
        assert limits_failed(inside) == [] and tiled(inside), (name, inside)
        assert edge[name](inside), (name, inside, tiled_box(*inside))
        assert limits_failed(outside) == [name] and not tiled(outside), (name, outside, tiled_box(*outside))


def test_cases_take_their_kernel():
    """every GPU case reaches the branch it is named for, and no staged geometry among them overflows its box"""
    for p in CASES:
        g, src_off, dst_off, n, kernel = p.values
        if kernel:
            assert resize_route(*g, src_off, dst_off) == kernel, p.id
        assert not overflows(*g), p.id


# ---- GPU -------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("g,src_off,dst_off,n,kernel", CASES)
def test_resize_geometry(lib, O, witness, g, src_off, dst_off, n, kernel):
    """every output byte against the oracle from a poisoned dst, the source and the bytes around both views unchanged,
    on the kernel resize_route names"""
    sw, sh, dw, dh = g
    assert not overflows(*g), "k_resize_tiled's box is too small: the kernel would trap"
    route = resize_route(*g, src_off, dst_off)
    assert kernel in (None, route)
    src = frames(sw, sh, n, sw + sh + dw + dh)
    want = np.stack([L.o_resize(O, a, dw, dh) for a in src]).ravel()
    S = Region(src.size, src_off, src, 1)

    def run():
        D = Region(want.size, dst_off, np.full(want.size, POISON, np.uint8), 2)
        rc, seen = traced(lambda: lib.gs_b200_resize_batch(D.ptr, dw, dh, S.ptr, sw, sh, n, stream()))
        assert rc == 0
        got = D.read("dst")
        assert np.array_equal(got, want), "dst byte %d of %d differs" % (int(np.argmax(got != want)), want.size)
        assert np.array_equal(S.read("src"), src.ravel())
        return seen

    witnessed(witness, run, [route], "resize %s" % (g,))
