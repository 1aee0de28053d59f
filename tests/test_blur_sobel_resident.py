"""k_blur_sobel_tma (box.cu) as a resident kernel: edge tiles made after other tiles of the same CTA.

The kernel runs min(tiles, resident) CTAs, resident = 3 CTAs per SM (its __launch_bounds__).  CTA b makes tile b first
and takes each next tile from a per-stream counter; it sets up its mbarrier, MMA bands and clipped-count table once,
and loads its next tile into the input buffer that phase A has just consumed.  A batch of fewer tiles than the
resident grid runs one tile per CTA, so every edge tile of the other blur→sobel test files is its CTA's first.  From a
CTA's second tile on, the blurred tile still holds the previous tile's values: in the bytes that an early-returning
strip (c0 >= w, or a step below the image) leaves alone, and in the rows of a step that stops at the image's last row.
Those bytes must feed only sobel outputs that are never written.

GS_B200_BLUR_SOBEL_CTAS=k caps the grid at k CTAs.  With k = 1 one CTA makes every tile in raster order; k = 2 and 3
interleave two or three CTAs through the counter.

GPU (each output bit-exact against the oracle chain gso_blur -> gso_sobel for r = 1..7, into dst pre-filled with random
bytes, so the untouched 1-px frame is checked too):
  * every GPU family of test_blur_sobel.py, test_blur_sobel_tiles.py and test_blur_sobel_band_seams.py, run through
    its own test body with each call made under caps 1, 2 and 3;
  * stale-content order with one CTA: [all 255, all 0], [all 0, all 255] and [0/255 stripes, random] batches, and one
    frame whose last column tile is dark after saturated tiles on its tile row, at right edges in every strip, bottom
    edges at every 8-row H tile and 16-row step, and last sobel rows at every phase-B band seam;
  * without the hook, one-tile frames in batches of resident - 1, resident, resident + 1, 2 resident +- 1 and
    5 resident + 7 tiles;
  * the counter's reset: many-, one- and many-tile calls back to back on one stream, and a graph under one CTA replayed
    twice.
Every case reads the launched grid of each k_blur_sobel_tma call from the profiler's trace and checks it: a cap that
is ignored fails there.
CPU: div_by / coords, the 64-bit reciprocal split of a tile index into (column tile, tile row, frame), against exact
integer division."""
import contextlib
import inspect
import os
import re

import numpy as np
import pytest

import _libs as L
import test_blur_sobel as TB
import test_blur_sobel_band_seams as TS
import test_blur_sobel_tiles as TT
from _gpu import G, O, dev, traced_grids, witness, lib  # noqa: F401

HOOK = "GS_B200_BLUR_SOBEL_CTAS"
KERNEL = "k_blur_sobel_tma"
RADII = range(1, 8)
_C = L.tile_constants()
TW, TH = _C["BS_STRIDE"], _C["BS_TH"]       # sobel columns and rows per tile
assert (TW, TH) == (TT.TW, TT.TH)


def ctas_per_sm():
    """the kernel's __launch_bounds__ minimum of CTAs per SM: the grid is that many per SM"""
    with open(os.path.join(L.ROOT, "grayskull_b200", "csrc", "box.cu")) as f:
        m = re.search(r"__launch_bounds__\(BS_THREADS,\s*(\d+)\)\s*k_blur_sobel_tma\(", f.read())
    return int(m.group(1))


def tiles_of(n, h, w):
    return -(-w // TW) * -(-h // TH) * n


@contextlib.contextmanager
def ctas(k):
    os.environ[HOOK] = str(k)
    try:
        yield
    finally:
        os.environ.pop(HOOK, None)


def grids_checked(witness, run, what):
    """run() makes a case's calls, checks every output and returns the grids its k_blur_sobel_tma launches should have,
    in order; they must be the traced ones.  The profiler sometimes loses kernel records, so on a mismatch the case runs
    again, up to 3 runs in all (as _gpu.witnessed does); a grid that is really wrong is wrong on every run."""
    for runs in range(1, 4):
        want, got = traced_grids(run, KERNEL)
        want = [(g, 1, 1) for g in want]
        if not witness or got == want:
            break
    if not witness:
        pytest.skip("parity holds; kineto recorded no kernel events for the probe launch, so the grid is not read")
    assert got == want, "%s: launched grids %s, expected %s (run %d)" % (what, got[:12], want[:12], runs)


# ---- GPU: the three edge-family files with the grid capped ---------------------------------------------------------
class Capped:
    """grayskull_b200.api for the families' test bodies: each blur_sobel_batch call runs once under each cap, each into
    its own copy of `out`, and returns the first cap's result for the body to check against the oracle.  It keeps the
    grid each launch must have and the calls whose caps disagreed."""

    def __init__(self, api, caps=(1, 2, 3)):
        self.api, self.caps, self.grids, self.differ = api, caps, [], []

    def blur_sobel_batch(self, src, radius, out=None):
        n, h, w = src.shape
        got = []
        for k in self.caps:
            with ctas(k):
                got.append(self.api.blur_sobel_batch(src, radius, out=None if out is None else out.clone()))
            self.grids.append(min(k, tiles_of(n, h, w)))
        for k, g in zip(self.caps[1:], got[1:]):
            if not bool((g == got[0]).all()):
                bad = sorted({int(i) for i in (g != got[0]).nonzero()[:, 0]})
                self.differ.append("%d x %d x %d, r %d: %d CTAs differ from %d in frames %s"
                                   % (n, h, w, radius, k, self.caps[0], bad))
        if out is not None:
            out.copy_(got[0])
            return out
        return got[0]


def _param_sets(fn):
    """the keyword sets of a test function's parametrize marks"""
    sets = [{}]
    for m in getattr(fn, "pytestmark", []):
        if m.name != "parametrize":
            continue
        names, values = m.args[0], m.args[1]
        names = [s.strip() for s in names.split(",")] if isinstance(names, str) else list(names)
        sets = [dict(s, **dict(zip(names, v if len(names) > 1 else (v,)))) for s in sets for v in values]
    return sets


def _families():
    out = []
    for mod in (TB, TT, TS):
        for name, fn in vars(mod).items():
            if not name.startswith("test_") or "O" not in inspect.signature(fn).parameters:
                continue
            assert any(m.name == "gpu" for m in fn.pytestmark), name
            for kw in _param_sets(fn):
                tag = ",".join("%s=%s" % kv for kv in kw.items())
                out.append(pytest.param(fn, kw, id="%s.%s%s" % (mod.__name__[len("test_"):], name[len("test_"):],
                                                                "-" + tag if tag else "")))
    return out


FAMILIES = _families()


@pytest.mark.gpu
@pytest.mark.parametrize("fn,kw", FAMILIES)
def test_edge_families_as_later_tiles(G, O, witness, fn, kw):
    def run():
        capped = Capped(G)
        fn(capped, O, **kw)
        assert not capped.differ, capped.differ
        return capped.grids
    grids_checked(witness, run, fn.__name__)


# ---- GPU: stale blurred bytes of the previous tile, one CTA ----------------------------------------------------------
EDGE_SHAPES = ([(TW + 16 * m + 16, 40) for m in range(16)] +                           # right edge at every strip end
               [(2 * TW, TH + 8 * j - 1 + d) for j in range(15) for d in (-1, 0, 1)] +  # bottom edge, H tiles / steps
               [(3 * TW, TH + s + d + 2) for s in TS.SEAMS for d in (-1, 0, 1)])        # last sobel row at band seams


def stale_batch(kind, w, h, seed):
    bright, dark = np.full((h, w), 255, np.uint8), np.zeros((h, w), np.uint8)
    if kind == "bright_dark":
        return [bright, dark]
    if kind == "dark_bright":
        return [dark, bright]
    if kind == "stripes_random":
        return [TB.stripes(w, h, 8)[3], np.random.default_rng(seed).integers(0, 256, (h, w))]
    # one frame: the last column tile dark, the tiles before it on every tile row saturated
    return [np.broadcast_to(np.where(np.arange(w) < TW * ((w - 1) // TW), 255, 0), (h, w))]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["bright_dark", "dark_bright", "stripes_random", "bright_row_dark_edge"])
def test_stale_content_before_edge_tiles(G, O, witness, kind):
    def run():
        grids = []
        with ctas(1):
            for w, h in EDGE_SHAPES:
                frames = np.stack(stale_batch(kind, w, h, w * h))
                TB.check(G, O, frames, w + h)
                grids += [1] * len(RADII)
        return grids
    grids_checked(witness, run, kind)


# ---- GPU: tile counts around the resident grid, no hook ------------------------------------------------------------
TW1, TH1 = 240, 70       # one clipped tile: strip 16 starts past the last column, steps 5 and 6 below the last row
assert tiles_of(1, TH1, TW1) == 1


def rotation_frames():
    """the distinct frames that batches of one-tile frames take in turn"""
    rng = np.random.default_rng(11)
    return np.stack([rng.integers(0, 256, (TH1, TW1)), L.natural_like(TW1, TH1, 3), np.full((TH1, TW1), 255),
                     TB.stripes(TW1, TH1, 3)[3], np.zeros((TH1, TW1)),
                     255 * (rng.random((TH1, TW1)) < 0.5)]).astype(np.uint8)


class Rotation:
    """n one-tile frames, frame i = distinct[(i + start) % len(distinct)]; the oracle runs once per distinct frame"""

    def __init__(self, O, n, start=0):
        import torch
        self.distinct = rotation_frames()
        self.idx = torch.tensor([(i + start) % len(self.distinct) for i in range(n)], device="cuda")
        self.src = dev(self.distinct)[self.idx].contiguous()
        self.O = O
        self.want = {}

    def expected(self, r):
        """the oracle's sobel rows and columns 1 .. -2 of every frame, on the device"""
        if r not in self.want:
            self.want[r] = dev(np.stack([L.o_sobel(self.O, L.o_blur(self.O, a, r))[1:-1, 1:-1]
                                         for a in self.distinct]))
        return self.want[r][self.idx]

    def fill(self, seed):
        """random bytes for dst"""
        import torch
        gen = torch.Generator(device="cuda").manual_seed(seed)
        return torch.randint(0, 256, self.src.shape, dtype=torch.uint8, device="cuda", generator=gen)

    def check(self, fill, got, r, what):
        bad = ~(got[:, 1:-1, 1:-1] == self.expected(r)).flatten(1).all(1)
        edge = got.clone()
        edge[:, 1:-1, 1:-1] = fill[:, 1:-1, 1:-1]
        bad |= ~(edge == fill).flatten(1).all(1)
        frames = bad.nonzero()[:, 0].tolist()
        assert not frames, "%s, r %d: %d frames differ from the oracle, first %s" % (what, r, len(frames), frames[:10])


@pytest.mark.gpu
@pytest.mark.parametrize("mul,add", [(1, -1), (1, 0), (1, 1), (2, -1), (2, 1), (5, 7)],
                         ids=["R-1", "R", "R+1", "2R-1", "2R+1", "5R+7"])
def test_tile_counts_around_the_resident_grid(G, O, witness, mul, add):
    import torch
    resident = ctas_per_sm() * torch.cuda.get_device_properties(0).multi_processor_count
    n = mul * resident + add
    batch = Rotation(O, n)

    def run():
        for r in RADII:
            fill = batch.fill(100 * n + r)
            got = G.blur_sobel_batch(batch.src, r, out=fill.clone())
            batch.check(fill, got, r, "%d frames" % n)
        return [min(n, resident)] * len(RADII)
    grids_checked(witness, run, "%d tiles, resident %d" % (n, resident))


# ---- GPU: the tile counter is reset for each call --------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cap", [None, 1])
def test_counter_reset_between_calls_on_one_stream(G, O, witness, cap):
    """many-, one- and many-tile calls queued back to back: a counter left at the previous call's count would skip the
    first tiles past the grid of the next call (the one-tile call follows a many-tile one, and precedes another)"""
    import torch
    resident = ctas_per_sm() * torch.cuda.get_device_properties(0).multi_processor_count
    n = 2 * resident + 1 if cap is None else 5
    calls = [(Rotation(O, n, 0), 1), (Rotation(O, 1, 1), 4), (Rotation(O, n, 2), 7)]
    for c, r in calls:
        c.expected(r)

    def run():
        fills = [c.fill(7 + r) for c, r in calls]
        outs = [f.clone() for f in fills]
        torch.cuda.synchronize()
        with contextlib.ExitStack() as stack:
            if cap is not None:
                stack.enter_context(ctas(cap))
            for (c, r), o in zip(calls, outs):                    # queued back to back, no synchronisation
                G.blur_sobel_batch(c.src, r, out=o)
        for (c, r), fill, got in zip(calls, fills, outs):
            c.check(fill, got, r, "call of %d tiles" % c.src.shape[0])
        grid = resident if cap is None else cap
        return [min(c.src.shape[0], grid) for c, _ in calls]
    grids_checked(witness, run, "cap %s" % cap)


@pytest.mark.gpu
def test_graph_replays_reset_the_counter(G, O, witness):
    """one CTA: a graph of the seven radii, captured with its counter memset, replayed twice on new frames"""
    import torch
    w, h, n = 528, 221, 2                                         # 3 x 3 tiles per frame, edges right and below
    s = torch.cuda.Stream()
    src = torch.zeros((n, h, w), dtype=torch.uint8, device="cuda")
    outs = [torch.zeros_like(src) for _ in RADII]
    with ctas(1):
        with torch.cuda.stream(s):
            for r in RADII:                                       # the stream's workspace, before the capture
                G.blur_sobel_batch(src, r, out=outs[r - 1])
        s.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for r in RADII:
                G.blur_sobel_batch(src, r, out=outs[r - 1])
    for seed in (1, 2):
        rng = np.random.default_rng(seed)
        frames = np.stack([rng.integers(0, 256, (h, w)), L.natural_like(w, h, seed)]).astype(np.uint8)
        fill = rng.integers(0, 256, frames.shape).astype(np.uint8)
        with torch.cuda.stream(s):
            src.copy_(dev(frames))
            for o in outs:
                o.copy_(dev(fill))
        s.synchronize()

        def replay():
            with torch.cuda.stream(s):
                g.replay()
            s.synchronize()
            for r in RADII:
                got = outs[r - 1].cpu().numpy()
                for i in range(n):
                    want = L.o_sobel(O, L.o_blur(O, frames[i], r), fill[i])
                    assert np.array_equal(got[i], want), ("replay", seed, r, i)
            return [1] * len(RADII)
        grids_checked(witness, replay, "replay %d" % seed)


# ---- CPU: the tile split of box.cu, restated -------------------------------------------------------------------------
M64 = (1 << 64) - 1


def div_by(d):
    """box.cu's host div_by(d) -> (m, shift): m = ceil(2^(32 + l) / d), l = ceil(log2 d)"""
    l = 0
    while (1 << l) < d:
        l += 1
    return ((1 << (32 + l)) + d - 1) // d, 32 + l


def div_by_x(x, m, shift):
    """the device's div_by(x, q): (unsigned)(x * m >> shift) in 64 bits, on uint64 arrays (x m < 2^64 checked first)"""
    x, m, shift = (np.asarray(v, np.uint64) for v in (x, m, shift))
    assert int(x.max()) * int(m.max()) <= M64
    return (x * m >> shift) & np.uint64(0xFFFFFFFF)


def coords(i, tiles_x, tiles_y):
    """the kernel's coords(i) -> (x, y, f), in 32-bit unsigned arithmetic"""
    u32 = np.uint64(0xFFFFFFFF)
    (mx, sx), (my, sy) = div_by(tiles_x), div_by(tiles_y)
    y = div_by_x(i, mx, sx)
    f = div_by_x(y, my, sy)
    x = (np.asarray(i, np.uint64) - y * np.uint64(tiles_x)) & u32
    y = (y - f * np.uint64(tiles_y)) & u32
    return x, y, f


X_MAX = (1 << 31) - 1                                 # tile indices are below 2^31 (the host refuses more)
TX_MAX = -(-((1 << 32) - 1) // TW)                    # the largest tiles_x and tiles_y of a frame below 2^32 pixels
TY_MAX = -(-((1 << 32) - 1) // TH)


def _check_divisors(ds, rng):
    """floor(x / d) at x = k d - 1 and k d for the smallest, largest and random k, and near 2^31"""
    ds = np.asarray(ds, np.int64)
    ms, shifts = zip(*(div_by(int(d)) for d in ds))
    ms, shifts = np.array(ms, np.uint64), np.array(shifts, np.uint64)
    assert int(ms.max()) <= 1 << 33 and int(shifts.max()) <= 63, "x m < 2^64 for every x < 2^31"
    kmax = X_MAX // ds
    ks = [np.minimum(j, kmax) for j in range(1, 9)] + [np.maximum(kmax - j, 1) for j in range(8)]
    ks += [rng.integers(1, kmax + 1) for _ in range(8)]
    xs = [k * ds + e for k in ks for e in (-1, 0)] + [np.full_like(ds, X_MAX - j) for j in range(4)] + [0 * ds]
    for x in xs:
        x = np.clip(x, 0, X_MAX)
        got = div_by_x(x.astype(np.uint64), ms, shifts).astype(np.int64)
        bad = np.nonzero(got != x // ds)[0]
        assert not len(bad), [(int(ds[b]), int(x[b]), int(got[b])) for b in bad[:5]]


def test_div_by_every_divisor_to_2_16():
    _check_divisors(np.arange(1, (1 << 16) + 1), np.random.default_rng(1))


def test_div_by_sampled_divisors_to_the_largest_tile_counts():
    """tiles_x < 2^24 + 1 (w < 2^32, TW columns per tile) and tiles_y up to (2^32 - 1) / TH"""
    rng = np.random.default_rng(2)
    top = max(TX_MAX, TY_MAX)
    near = {d + e for j in range(16, top.bit_length() + 1) for d in (1 << j,) for e in (-1, 0, 1)}
    ds = sorted({d for d in near if d <= top} | {TX_MAX, TX_MAX - 1, TY_MAX, TY_MAX - 1} |
                set(rng.integers((1 << 16) + 1, top + 1, 20000).tolist()))
    _check_divisors(ds, rng)


def _tile_indices(tx, ty, n, rng):
    total = tx * ty * n
    if total <= 1 << 16:
        return np.arange(total)
    per = tx * ty
    idx = [np.arange(512), total - 1 - np.arange(512), rng.integers(0, total, 512)]
    for f in sorted({0, 1, n // 2, n - 1}):                       # frame and tile-row seams of some frames
        for yy in sorted({0, 1, ty // 2, ty - 1}):
            base = f * per + yy * tx
            idx.append(base + np.array([-1, 0, 1, tx - 2, tx - 1, tx]))
    idx = np.concatenate(idx)
    return np.unique(idx[(idx >= 0) & (idx < total)])


@pytest.mark.parametrize("tx_pow", [0, 4, 8, 12, 16, 20, 24])
def test_tile_coords_around_powers_of_two(tx_pow):
    """coords(i) == (i % tiles_x, i / tiles_x % tiles_y, i / (tiles_x tiles_y)) for tiles_x near 2^tx_pow .. 2^(tx_pow
    + 3) and every tiles_y near a power of two that keeps the batch below 2^31 tiles; 1, 2, 3 frames and the most
    that fit.  Every index of small batches, the ends and the frame and row seams of large ones."""
    rng = np.random.default_rng(tx_pow)
    near = lambda j: ((1 << j) - 1, 1 << j, (1 << j) + 1)  # noqa: E731
    txs = sorted({t for j in range(tx_pow, tx_pow + 4) for t in near(j) if 1 <= t <= TX_MAX})
    tys = sorted({t for j in range(0, TY_MAX.bit_length()) for t in near(j) if 1 <= t <= TY_MAX})
    cases = 0
    for tx in txs:
        for ty in tys:
            most = X_MAX // (tx * ty)
            for n in sorted({v for v in (1, 2, 3, most) if 1 <= v <= most}):
                i = _tile_indices(tx, ty, n, rng)
                x, y, f = coords(i.astype(np.uint64), tx, ty)
                want = (i % tx, i // tx % ty, i // (tx * ty))
                for name, g, w in zip("xyf", (x, y, f), want):
                    bad = np.nonzero(g.astype(np.int64) != w)[0]
                    assert not len(bad), (tx, ty, n, name, [int(i[b]) for b in bad[:5]])
                cases += 1
    assert cases > 50
