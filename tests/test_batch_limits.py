"""Every batch entry point past the grid's 65535-frame limit and with a frame that starts past 4 GiB.

Grid y and z stop at 65535.  Kernels that take the frame from blockIdx.y / .z either loop over frames (f += gridDim.z)
or run behind gsb::for_frame_groups, which launches a larger batch as groups of at most 65535 frames with their own
bases.  ROWS is the coverage record: one row per batch entry point of the three public headers (plus rows that put a
looping generic kernel on its second pass), each with a frame geometry and the kernels the call must launch there.

  * CPU (census): every gs_b200_*_batch declared in include/ has a row.
  * GPU, frame counts: every row at n = 65535, 65536 and 2 * 65535 + 3.  Frame content (and every per-frame input)
    repeats with period 7; 65535 = 1 and 65536 = 2 (mod 7), so a frame read from the wrong group, or left unwritten,
    differs from expected[f % 7].  Outputs start as poison; list outputs must hold each frame's count, its records, and
    poison in the slots after the count; the bytes after each buffer's end stay poison.  Each case runs through
    witnessed(): at every n the row's kernels must launch, so a batch that falls back to another path fails.
  * GPU, past 4 GiB: the smallest batch whose last frame starts past 2^32 bytes in some input or output.  Every frame is
    zero except the first and the last; those two get a full oracle check, the rest the oracle's result for a zero
    frame.
  * GPU, a frame group past 4 GiB: 65536 frames of 272 x 256, so the second group's base passes 2^32 bytes in every
    image buffer; every frame checked as in the frame-count cases.
  * a frame past 65535 row tiles (the last section; its comment lists the launch sites and their old limits): TALL has
    one row per site, at a height just past the site's limit and at the last height it accepted; TALL_CONTROLS runs
    every other batch entry point on a frame of 524,300 rows; fp32 row coordinates past 2^24; the single-image calls on
    tall host arrays.  Its CPU half reads the tile constants from csrc/ to check each row crosses its site's limit,
    extends the census to tall rows, and checks that no GSB_ASSERT in csrc/ caps a grid count at 65535.

Device memory per case, measured on an H100 80GB: the larger of torch's peak allocation and the memory the case held
when its checks ended (its buffers plus what the library's workspace arenas grew by; the arenas are grow-only and stay
allocated for the process, the largest being blobs' 4.3 GB).
  frame counts (every row, every n)                          at most 3.5 GB
  past 4 GiB   adaptive_threshold, erode, dilate, erode_n,
               dilate_n, filter, match_template               9.2 GB
               fast 9.7, orb_extract 9.4, blobs 9.1, orb_pyramid 11.6, resize 6.6, downsample 5.9,
               perspective_correct 5.1, match_orb 5.0, histogram, otsu_threshold, threshold,
               threshold_each, find_best_match 4.9 GB
  group past 4 GiB  blur 9.7, blur_sobel 9.7, resize 7.5, find_best_match 5.1, fast 10.1, orb_extract 11.3,
                    orb_pyramid 13.9 GB
  a frame past 65535 row tiles  orb_pyramid 2.6 GB, blur / blur_sobel / filter (16 x 8.4M rows) 1.3 GB, others less;
                    the 58 cases take about 4.5 minutes on one H100 80GB (700 W power limit), mostly the CPU oracle
"""
import glob
import os
import re

import numpy as np
import pytest

import _calls as calls
import _libs as L
from _gpu import G, O, lib, stream, traced, witness, witnessed  # noqa: F401

POISON = calls.POISON
GUARD = 64
NS = (65535, 65536, 2 * 65535 + 3)
W, H = 48, 40


def row(sym, kernels, **g):
    g.setdefault("w", W)
    g.setdefault("h", H)
    return sym, tuple(kernels), g


TAIL = ("gsb::k_row_scan", "gsb::k_nms_emit_masks")
ORB = ("gsb::k_fast_tiled2<true>", "gsb::k_orb_brief<true>", "gsb::k_orb_select", "gsb::k_orb_moments", "gsb::k_orb_trig")
LBP3 = ("gsb::k_deinterleave2", "gsb::k_lbp_count", "gsb::k_row_scan", "gsb::k_lbp_emit")
BLOBS = ("gsb::k_blob_mask", "gsb::k_blob_seed", "gsb::k_row_scan", "gsb::k_blob_overflow", "gsb::k_blob_runs",
         "gsb::k_blob_union", "gsb::k_blob_label", "gsb::k_blob_compact")
ROWS = [
    row("blur", ["gsb::k_box_tma<5,false>"], r=5),
    row("adaptive_threshold", ["gsb::k_box_tma<5,true>"], r=5, c=3),
    row("sobel", ["gsb::k_stencil3_tma<0>"]),
    row("blur_sobel", ["gsb::k_blur_sobel_tma<5>"], r=5),
    row("erode", ["gsb::k_stencil3_tma<1>"]),
    row("dilate", ["gsb::k_stencil3_tma<2>"]),
    row("erode_n", ["gsb::k_morph_tma<1,2>"], iters=2),
    row("dilate_n", ["gsb::k_morph_tma<2,2>"], iters=2),
    row("resize", ["gsb::k_resize_tiled<true>"], dw=36, dh=30),
    row("downsample", ["gsb::k_downsample_vec"]),
    row("integral", ["gsb::k_integral_strips<128,8>"]),
    row("histogram", ["gsb::k_histogram<true>"]),
    row("otsu_threshold", ["gsb::k_histogram<true>", "gsb::k_otsu"]),
    row("threshold", ["gsb::k_threshold<true>"], t=100),
    row("threshold_each", ["gsb::k_threshold<true>"], offset=10),
    row("filter", ["gsb::k_filter3<true>"], k="sharpen"),
    row("match_template", ["gsb::k_pack_template", "gsb::k_match_template"], tw=9, th=7),
    row("find_best_match", ["gsb::k_best_match_partial", "gsb::k_best_match_final"]),
    row("blobs", BLOBS, nb=64),
    row("perspective_correct", ["gsb::k_perspective"], dw=30, dh=20),
    row("fast", ("gsb::k_fast_tiled2<true>",) + TAIL, nkps=32, t=20),
    row("orb_extract", ORB + TAIL, nkps=16, t=20),
    row("match_orb", ["gsb::k_match_best", "gsb::k_match_compact"], s1=40, s2=30, mm=24),
    row("lbp_detect", LBP3, w=64, h=64, mr=8),
    row("crop_resize", ["gsb::k_roi_gather<1>"], roi=(5, 4, 30, 25), dw=20, dh=16),
    row("rois_resize", ["gsb::k_roi_copy", "gsb::k_roi_gather<1>"], mr=3, dw=12, dh=10),
    row("orb_pyramid", ("gsb::k_downsample_vec", "gsb::k_pyr_quota", "gsb::k_pyr_merge") + ORB, w=128, h=64, levels=2,
        nkps=24, t=20),
    # the generic kernels that loop over frames in grid z / y, on their second pass
    row("blur", ["gsb::k_box_generic<false>"], r=0),
    row("sobel", ["gsb::k_stencil3_generic<0>"], w=50),
    row("downsample", ["gsb::k_downsample_generic"], w=50),
    row("resize", ["gsb::k_resize<false>"], w=50, dw=37, dh=30),
    row("integral", ["gsb::k_integral_rows<false>", "gsb::k_integral_cols"], w=50),
    row("filter", ["gsb::k_filter_generic"], w=50, k="k5"),
    row("match_template", ["gsb::k_match_template_generic"], w=50, tw=9, th=7),
]


def row_id(sym, g):
    return "-".join([sym] + ["%s%s" % (k, v) for k, v in g.items() if k not in ("roi",)])


def header_batch_symbols():
    out = set()
    for path in glob.glob(os.path.join(L.ROOT, "include", "grayskull_b200*.h")):
        with open(path) as f:
            out |= set(re.findall(r"\bgs_b200_(\w+)_batch\s*\(", f.read()))
    return out


# ---- CPU: the census ---------------------------------------------------------------------------------------------
def test_every_batch_entry_point_has_a_row():
    syms = header_batch_symbols()
    assert len(syms) >= 27, sorted(syms)
    have = {sym for sym, _, _ in ROWS}
    assert not sorted(syms - have), "batch entry points without a row: %s" % sorted(syms - have)
    assert not sorted(have - syms), "rows for entry points the headers do not declare: %s" % sorted(have - syms)
    ids = [row_id(s, g) for s, _, g in ROWS]
    assert len(ids) == len(set(ids))


# ---- per-row inputs: the distinct frames and their per-frame inputs ------------------------------------------------
def _frames7(w, h, seed):
    rng = np.random.default_rng(seed)
    out = [rng.integers(0, 256, (h, w), dtype=np.uint8), L.natural_like(w, h, seed), np.full((h, w), 255, np.uint8),
           np.zeros((h, w), np.uint8), L.natural_like(w, h, seed + 1), (rng.integers(0, 4, (h, w)) * 85).astype(np.uint8),
           L.natural_like(w, h, seed + 2)]
    return np.stack(out)


def _lbp_frames(w, h):
    at = [(44, 40), (0, 0), (48, 44), (52, 44), (20, 10), (40, 40), (64, 64)]
    return np.stack([np.ascontiguousarray(calls.lena()[y:y + h, x:x + w]) for x, y in at])


def row_inputs(O, sym, g, fr=None):
    """{buffer: its bytes for each distinct frame}: fr, else the period-7 frames, and the row's per-frame inputs"""
    w, h = g["w"], g["h"]
    if sym == "match_orb":
        rng = np.random.default_rng(16)
        sets = [L.desc_sets(rng, a, b) for a, b in g.get("sizes", [(40, 30), (7, 0), (0, 12), (33, 29), (1, 1), (40, 2),
                                                                    (25, 30)])]
        k1, k2 = np.zeros((len(sets), g["s1"]), L.KP_DTYPE), np.zeros((len(sets), g["s2"]), L.KP_DTYPE)
        for i, (a, b) in enumerate(sets):
            k1[i, :len(a)], k2[i, :len(b)] = a, b
        return {"kps1": k1, "n1": calls.counts([a for a, _ in sets]), "kps2": k2, "n2": calls.counts([b for _, b in sets])}
    if sym == "lbp_detect":
        return {"ii": np.stack([L.o_integral(O, a) for a in _lbp_frames(w, h)])}
    fr = _frames7(w, h, w * 7 + h) if fr is None else fr
    k = len(fr)
    if sym == "threshold_each":
        return {"src": fr, "thresh": np.array([100, 0, 250, 37, 255, 128, 1], np.uint8)[:k]}
    if sym == "match_template":
        return {"src": fr, "tmpl": np.ascontiguousarray(_frames7(w, h, w * 7 + h)[1, 10:10 + g["th"], 20:20 + g["tw"]])}
    if sym == "find_best_match":
        return {"res": (fr // 2).astype(np.uint8)}                    # a result map per frame, the 255 frame -> all ties
    if sym == "blobs" and g.get("binary", True):
        return {"src": np.stack([L.binary_like(w, h, 50 + i) if i % 3 else np.where(a >= 128, 255, 0).astype(np.uint8)
                                 for i, a in enumerate(fr)])}
    if sym == "perspective_correct":
        return {"src": fr, "corners": np.random.default_rng(5).integers(0, min(w, h), (k, 4, 2)).astype(np.uint32)}
    if sym in ("fast", "orb_extract"):
        return {"src": fr, "score": np.full_like(fr, POISON)}
    if sym == "rois_resize":
        dw, dh, mr = g["dw"], g["dh"], g["mr"]
        rng = np.random.default_rng(3)
        rects = np.zeros((k, mr), L.RECT_DTYPE)
        for i in range(k):
            for j in range(mr):
                rw, rh = (dw, dh) if j == 0 else (int(rng.integers(1, w)), int(rng.integers(1, h)))
                rects[i, j] = (int(rng.integers(0, w - rw + 1)), int(rng.integers(0, h - rh + 1)), rw, rh)
        return {"src": fr, "rects": rects, "rcounts": np.array([(3 + i) % (mr + 1) for i in range(k)], np.uint32)}
    if sym == "orb_pyramid":
        sizes = L.layout(w, h, g["levels"])[0]
        assert len(sizes) == 2
        return {"src": fr, "score": [np.full((k, a * b), POISON, np.uint8) for a, b in sizes]}
    return {"src": fr}


def _chunk(per):
    """frames per step of a copy or compare: about 256 MB"""
    return max(1, (256 << 20) // per)


class Batch:
    """a device buffer of n frames of `per` bytes (or level-major segments of such), plus GUARD poison bytes after it"""

    def __init__(self, segs, n, idx, src=False):
        import torch
        self.segs, self.n = segs, n
        size = sum(n * x.shape[1] for x in self.segs)
        self.t = torch.full((size + GUARD,), POISON, dtype=torch.uint8, device="cuda")
        if src:                                          # an input: frame f holds distinct frame idx[f]
            off = 0
            for x in self.segs:
                d, per = torch.from_numpy(x.copy()).cuda(), x.shape[1]
                dst, c = self.t[off:off + n * per].view(n, per), _chunk(per)
                for f0 in range(0, n, c):
                    dst[f0:f0 + c].copy_(d[idx[f0:f0 + c]])
                off += n * per
        self.ptr = self.t.data_ptr()

    def check(self, what, idx):
        """every frame f holds distinct frame idx[f]'s expected bytes; the guard is poison"""
        import torch
        off = 0
        for si, x in enumerate(self.segs):
            want = torch.from_numpy(x.copy()).cuda()
            per = x.shape[1]
            got = self.t[off:off + self.n * per].view(self.n, per)
            chunk = _chunk(per)
            for f0 in range(0, self.n, chunk):
                bad = (got[f0:f0 + chunk] != want[idx[f0:f0 + chunk]]).any(dim=1)
                if bool(bad.any()):
                    f = f0 + int(torch.nonzero(bad)[0])
                    raise AssertionError("%s (segment %d): frame %d of %d (distinct frame %d) differs" %
                                         (what, si, f, self.n, int(idx[f])))
            off += self.n * per
        assert bool((self.t[off:] == POISON).all()), "%s: bytes after the batch end changed" % what


def run_batch(lib, O, sym, g, n, idx, fr=None, ins=None):
    """one call over n frames, frame f being distinct frame idx[f] -> the kernels it launched.  The distinct frames and
    their inputs are `ins`, else row_inputs(fr).  Prints the device memory the case took: its buffers plus what the
    library's workspace arenas grew by (they stay allocated after it)."""
    import torch
    free0 = torch.cuda.mem_get_info()[0]
    torch.cuda.reset_peak_memory_stats()
    sp = calls.spec("gs_b200_%s_batch" % sym, g)
    ins = row_inputs(O, sym, g, fr) if ins is None else ins
    k = len(next(iter(ins.values())))                  # the first buffer is per frame and not segmented
    before = calls.filled(sp, k)
    want = sp.expect(ins, before)
    if sym == "lbp_detect":
        assert want["counts"].sum() > 0 and want["counts"].min() == 0
    shared = {b: torch.from_numpy(calls.flat(ins[b], 1)).cuda() for b in sp.shared}
    bufs = {b: Batch(calls.segments(x, k), n, idx, src=True) for b, x in ins.items() if b not in sp.shared}
    bufs.update({b: Batch(calls.segments(x, k), n, idx) for b, x in before.items()})
    P = dict({b: t.data_ptr() for b, t in shared.items()}, **{b: x.ptr for b, x in bufs.items()})
    rc, seen = traced(lambda: sp.call(P, n, stream()))
    assert rc == 0, lib.gs_b200_last_error().decode()
    for b, x in bufs.items():
        if b in want:
            x.segs = calls.segments(want[b], k)
        x.check(b, idx)
    took = free0 - torch.cuda.mem_get_info()[0]
    print("\n%s n=%d: device memory taken %.2f GB (torch peak %.2f GB)" %
          (sym, n, took / 1e9, torch.cuda.max_memory_allocated() / 1e9))
    del bufs
    torch.cuda.empty_cache()
    return seen


def _room(gb):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < gb * 2 ** 30:
        pytest.skip("needs %.0f GB of free device memory, %.1f GB free (the device is shared)" % (gb, free / 2 ** 30))


# ---- GPU: frame counts ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("sym,kernels,g", [pytest.param(s, k, g, id=row_id(s, g)) for s, k, g in ROWS])
def test_frame_count(lib, O, witness, sym, kernels, g, n):
    """device memory: at most 3.5 GB per case (the module docstring's table)"""
    import torch
    _room(4)
    idx = torch.arange(n, device="cuda") % 7
    witnessed(witness, lambda: run_batch(lib, O, sym, g, n, idx), kernels, "%s n=%d" % (row_id(sym, g), n))


# ---- GPU: a frame past 4 GiB ----------------------------------------------------------------------------------------
def _first_last(fr, n):
    import torch
    idx = torch.ones(n, dtype=torch.long, device="cuda")
    idx[0], idx[-1] = 0, 2
    return np.stack([fr[0], np.zeros_like(fr[0]), fr[1]]), idx


def _past_4gib(n_bytes_per_frame):
    """frames so that the last frame starts past 2^32 bytes"""
    return 2 ** 32 // n_bytes_per_frame + 2


# (sym, geometry, the buffer whose last frame starts past 4 GiB, bytes per frame of that buffer); the images are
# 2048 x 2048 (4 MiB a frame) except where a record array crosses first
BIG = [
    ("adaptive_threshold", dict(w=2048, h=2048, r=5, c=3), "src"),
    ("erode", dict(w=2048, h=2048), "src"),
    ("dilate", dict(w=2048, h=2048), "src"),
    ("erode_n", dict(w=2048, h=2048, iters=3), "src"),
    ("dilate_n", dict(w=2048, h=2048, iters=3), "src"),
    ("resize", dict(w=2048, h=2048, dw=1500, dh=1100), "src"),
    ("downsample", dict(w=2048, h=2048), "src"),
    ("histogram", dict(w=2048, h=2048), "src"),
    ("otsu_threshold", dict(w=2048, h=2048), "src"),
    ("threshold", dict(w=2048, h=2048, t=100), "img"),
    ("threshold_each", dict(w=2048, h=2048, offset=10), "img"),
    ("filter", dict(w=2048, h=2048, k="sharpen"), "src"),
    ("match_template", dict(w=2048, h=2048, tw=9, th=7), "img"),
    ("find_best_match", dict(w=2048, h=2048), "result"),
    ("perspective_correct", dict(w=2048, h=2048, dw=300, dh=200), "src"),
    ("fast", dict(w=2048, h=2048, nkps=500, t=20), "src"),
    ("orb_extract", dict(w=2048, h=2048, nkps=500, t=20), "src"),
    ("blobs", dict(w=48, h=40, nb=65534), "blobs"),
    ("match_orb", dict(w=0, h=0, s1=40, s2=30, mm=1 << 22), "matches"),
    ("orb_pyramid", dict(w=2048, h=2048, levels=2, nkps=500, t=20), "src"),
]


def _big_n(sym, g):
    if sym == "blobs":
        return _past_4gib(32 * g["nb"])
    if sym == "match_orb":
        return _past_4gib(12 * g["mm"])
    return _past_4gib(g["w"] * g["h"])


@pytest.mark.gpu
@pytest.mark.parametrize("sym,g,buf", [pytest.param(s, g, b, id=s) for s, g, b in BIG])
def test_last_frame_past_4gib(lib, O, sym, g, buf):
    """The first and last frames hold content, every other frame is zero.  Device memory per case: the module
    docstring's table."""
    import torch
    _room(20)
    n = _big_n(sym, g)
    if sym == "match_orb":
        g = dict(g, sizes=[(40, 30), (0, 0), (33, 29)])
        fr, idx = np.zeros(3), _first_last(np.zeros((2, 1, 1)), n)[1]
    else:
        base = _frames7(g["w"], g["h"], 11) if sym != "blobs" else np.stack([L.binary_like(g["w"], g["h"], 70 + i) for i in range(2)])
        fr, idx = _first_last(np.stack([base[1], base[4]]) if sym != "blobs" else base, n)
        if sym == "blobs":
            g = dict(g, binary=False)
    run_batch(lib, O, sym, g, n, idx, fr=None if sym == "match_orb" else fr)


# ---- GPU: a frame group that starts past 4 GiB ------------------------------------------------------------------------
# 65536 frames of 272 x 256 (69,632 bytes): the second group starts at frame 65535, byte 65535 * 69632 (4.56e9 > 2^32)
# of every image buffer, so a group base computed in 32 bits points into the first group.  The adaptive threshold
# shares the blur's dispatcher.  LBP and match_orb offset their groups in records (u32 tables, keypoints), whose
# element counts stay far below 2^32 within a device's memory.
GROUP_BIG = [
    row("blur", ["gsb::k_box_tma<5,false>"], w=272, h=256, r=5),
    row("blur_sobel", ["gsb::k_blur_sobel_tma<5>"], w=272, h=256, r=5),
    row("resize", ["gsb::k_resize_tiled<true>"], w=272, h=256, dw=200, dh=180),
    row("find_best_match", ["gsb::k_best_match_partial", "gsb::k_best_match_final"], w=272, h=256),
    row("fast", ("gsb::k_fast_tiled2<true>",) + TAIL, w=272, h=256, nkps=100, t=20),
    row("orb_extract", ORB + TAIL, w=272, h=256, nkps=100, t=20),
    row("orb_pyramid", ("gsb::k_downsample_vec", "gsb::k_pyr_quota", "gsb::k_pyr_merge") + ORB, w=272, h=256, levels=2,
        nkps=100, t=20),
]


@pytest.mark.gpu
@pytest.mark.parametrize("sym,kernels,g", [pytest.param(s, k, g, id=row_id(s, g)) for s, k, g in GROUP_BIG])
def test_group_past_4gib(lib, O, witness, sym, kernels, g):
    """every frame of both groups against the oracle, as in test_frame_count; device memory per case in the module
    docstring's table"""
    import torch
    _room(20)
    n = 65536
    assert (n - 1) * g["w"] * g["h"] >= 2 ** 32
    idx = torch.arange(n, device="cuda") % 7
    witnessed(witness, lambda: run_batch(lib, O, sym, g, n, idx), kernels, "%s n=%d" % (row_id(sym, g), n))


# ---- a frame past 65535 row tiles ------------------------------------------------------------------------------------
# Grid y stops at 65535 row tiles within one frame, too.  The TMA tile kernels (k_box_tma, k_blur_sobel_tma,
# k_fast_tiled2, k_resize_tiled, k_filter3) and k_resize run a taller frame through gsb::for_row_groups: launches of at
# most 65535 tile rows at a tile-row offset, each seeing the whole frame.  The generic kernels, k_match_template,
# k_downsample_vec and k_perspective loop over row tiles (y += gridDim.y ...).  Before that, every site below aborted
# on a GSB_ASSERT or failed its launch with cudaErrorInvalidConfiguration once a frame passed its limit:
#   perspective_correct (k_perspective, a row per CTA)             dh > 65,535            abort
#   sobel / erode / dilate, k_stencil3_generic (8-row tiles)        h > 524,280            launch error
#   blur / adaptive, k_box_generic (8-row tiles)                    h > 524,280            launch error
#   blur / adaptive, k_box_tma (BX_TH rows)                         h > 8,388,480          abort
#   blur_sobel, k_blur_sobel_tma (BS_TH rows)                       h > 8,257,410          abort
#   downsample, k_downsample_generic (8-row tiles)                  dh > 524,280           launch error
#   downsample, k_downsample_vec (a row per CTA)                    dh > 65,535            took the generic kernel
#   resize, k_resize_tiled / k_resize (8 * RS_ROWS rows)            dh > 4,194,240         abort
#   fast / orb_extract, k_fast_tiled2 (F2_TH rows from row 3)       h > 4,194,246          abort
#   fast, k_fast_score (8-row tiles from row 3)                     h > 524,286            launch error
#   filter, k_filter3 (8 * F3_ROWS rows) / k_filter_generic         h > 8,388,480 / 524,280  abort
#   match_template, both kernels (8-row tiles of result rows)      h - th + 1 > 524,280   abort
# TALL has one row per site, each at a height just past its old limit (with a partial last tile) and at the last height
# the old code accepted, n = 2, witnessed on the kernel a short frame of the same width takes.  TALL_CONTROLS runs every
# other batch entry point on a frame of 524,300 rows.  Frames are flat with seeded content in three bands: the top
# rows, rows straddling the first old group seam (65535 row tiles) and the last rows; every output byte is checked.
GRID = 65535
BAND = 24


# (sym, kernels, geometry without its tall key, tall key, rows of that key per old row tile, the first row of the
# first old row tile, extra rows of that key beyond its old limit (th - 1: the template's), the tall value)
def tall(sym, kernels, key, tile, first, past, extra=0, **g):
    g.setdefault("w", W)
    g.setdefault("h", H)
    return sym, tuple(kernels), g, key, tile, first, extra, past


TALL = [
    tall("perspective_correct", ["gsb::k_perspective"], "dh", lambda c: 1, 0, 65_537, dw=30, dh=None),
    tall("sobel", ["gsb::k_stencil3_generic<0>"], "h", lambda c: 8, 0, 524_300, w=24),
    tall("blur", ["gsb::k_box_generic<false>"], "h", lambda c: 8, 0, 524_300, r=0),
    tall("blur", ["gsb::k_box_tma<1,false>"], "h", lambda c: c["BX_TH"], 0, 8_388_600, w=16, r=1),
    tall("blur_sobel", ["gsb::k_blur_sobel_tma<1>"], "h", lambda c: c["BS_TH"], 0, 8_257_500, w=16, r=1),
    tall("downsample", ["gsb::k_downsample_generic"], "h", lambda c: 16, 0, 1_048_600, extra=1, w=50),
    tall("downsample", ["gsb::k_downsample_vec"], "h", lambda c: 2, 0, 1_048_600, extra=1, w=32),
    tall("resize", ["gsb::k_resize_tiled<true>"], "dh", lambda c: 8 * c["RS_ROWS"], 0, 4_194_300, dw=36, dh=None),
    tall("resize", ["gsb::k_resize<false>"], "dh", lambda c: 8 * c["RS_ROWS"], 0, 4_194_300, w=50, dw=37, dh=None),
    tall("fast", ("gsb::k_fast_tiled2<true>",) + TAIL, "h", lambda c: c["F2_TH"], 3, 4_194_300, w=16, nkps=4096,
         t=20),
    tall("fast", ("gsb::k_fast_score",) + TAIL, "h", lambda c: 8, 3, 524_300, w=16, nkps=4096, t=300),
    tall("filter", ["gsb::k_filter3<true>"], "h", lambda c: 8 * c["F3_ROWS"], 0, 8_388_600, w=16, k="sharpen"),
    tall("filter", ["gsb::k_filter_generic"], "h", lambda c: 8, 0, 524_300, w=50, k="k5"),
    tall("match_template", ["gsb::k_match_template", "gsb::k_pack_template"], "h", lambda c: 8, 0, 524_306,
         extra=6, tw=9, th=7),
    tall("match_template", ["gsb::k_match_template_generic"], "h", lambda c: 8, 0, 524_306, extra=6, w=50, tw=9,
         th=7),
    tall("orb_pyramid", ORB + ("gsb::k_downsample_vec", "gsb::k_pyr_quota", "gsb::k_pyr_merge"), "h",
         lambda c: c["F2_TH"], 3, 4_194_300, w=64, levels=2, nkps=4096, t=20),
]


def old_limit(c, tile, first, extra):
    """the largest value of a row's tall key that the old launch accepted: 65535 tiles from `first` (+ extra)"""
    return first + GRID * tile(c) + extra + (3 if first else 0)


def tall_geometry(row, c, which):
    sym, kernels, g, key, tile, first, extra, past = row
    v = past if which == "past" else old_limit(c, tile, first, extra)
    return dict(g, **{key: v})


def tall_id(row):
    sym, kernels, g, key, tile, first, extra, past = row
    return "-".join([sym, kernels[0].split("::")[-1]])


TALL_CONTROLS = [row(s, k, **dict(g, h=524_300)) for s, k, g in [
    ("adaptive_threshold", ["gsb::k_box_tma<5,true>"], dict(r=5, c=3)),
    ("sobel", ["gsb::k_stencil3_tma<0>"], {}),
    ("erode", ["gsb::k_stencil3_tma<1>"], {}),
    ("dilate", ["gsb::k_stencil3_tma<2>"], {}),
    ("erode_n", ["gsb::k_morph_tma<1,2>"], dict(iters=2)),
    ("dilate_n", ["gsb::k_morph_tma<2,2>"], dict(iters=2)),
    ("integral", ["gsb::k_integral_rows<true>", "gsb::k_integral_cols"], {}),
    ("histogram", ["gsb::k_histogram<true>"], {}),
    ("otsu_threshold", ["gsb::k_histogram<true>", "gsb::k_otsu"], {}),
    ("threshold", ["gsb::k_threshold<true>"], dict(t=100)),
    ("threshold_each", ["gsb::k_threshold<true>"], dict(offset=10)),
    ("find_best_match", ["gsb::k_best_match_partial", "gsb::k_best_match_final"], {}),
    ("blobs", BLOBS, dict(nb=4096)),
    ("orb_extract", ORB + TAIL, dict(nkps=4096, t=20)),
    ("lbp_detect", LBP3, dict(w=64, mr=256)),
    ("crop_resize", ["gsb::k_roi_gather<1>"], dict(roi=(5, 524_100, 30, 190), dw=20, dh=16)),
    ("rois_resize", ["gsb::k_roi_copy", "gsb::k_roi_gather<1>"], dict(mr=3, dw=12, dh=10)),
]]


# ---- CPU: the old limits and the census -------------------------------------------------------------------------------
def test_tall_rows_cross_their_old_limit():
    """each row's tall value passes its site's old limit, with a partial last tile, read from the tile constants in
    csrc/: a retuned tile height cannot move the limit past the test unnoticed"""
    c = L.tile_constants()
    assert {"BX_TH", "BS_TH", "F2_TH", "RS_ROWS", "F3_ROWS"} <= set(c), sorted(c)
    for row in TALL:
        sym, kernels, g, key, tile, first, extra, past = row
        lim = old_limit(c, tile, first, extra)
        assert past > lim, (tall_id(row), past, lim)
        rows = past - first - extra - (3 if first else 0)        # rows of the key that the row tiles cover
        assert rows > GRID * tile(c), tall_id(row)
        if tile(c) > 1:
            assert rows % tile(c), "%s: no partial last tile" % tall_id(row)


def test_every_batch_entry_point_has_a_tall_row():
    syms = header_batch_symbols() - {"match_orb"}             # match_orb has no image rows
    have = {r[0] for r in TALL} | {s for s, _, _ in TALL_CONTROLS}
    assert not sorted(syms - have), "batch entry points without a tall row: %s" % sorted(syms - have)
    assert not sorted(have - syms)
    assert all(g["h"] > GRID * 8 for _, _, g in TALL_CONTROLS)


def test_no_assert_caps_a_grid_at_65535():
    """a grid or tile count over 65535 is split into launches or loops, never refused: no GSB_ASSERT in csrc/ compares
    one with 65535"""
    bad = []
    for path in sorted(glob.glob(os.path.join(L.ROOT, "grayskull_b200", "csrc", "*.cu*"))):
        with open(path) as f:
            for i, line in enumerate(f, 1):
                if re.search(r"GSB_ASSERT\(.*\b(65535u?|0xFFFFu?|GRID_FRAMES)\b", line):
                    bad.append("%s:%d: %s" % (os.path.basename(path), i, line.strip()))
    assert not bad, "\n".join(bad)


# ---- tall frames: content in three bands ------------------------------------------------------------------------------
def banded(w, h, seams, seed, base=0, band=BAND, kind="random"):
    """a flat frame of `base` with seeded content in rows [0, band), around each seam row, and in the last band rows"""
    rng = np.random.default_rng(seed)
    a = np.full((h, w), base, np.uint8)
    for y0 in [0, h - band] + [s - band // 2 for s in seams]:
        y0 = min(max(y0, 0), h - band)
        if kind == "binary":
            a[y0:y0 + band] = (rng.random((band, w)) < 0.5) * 255
        elif kind == "natural":
            a[y0:y0 + band] = L.natural_like(w, band, int(rng.integers(1 << 30)))
        else:
            a[y0:y0 + band] = rng.integers(0, 256, (band, w), dtype=np.uint8)
    return a


def tall_inputs(O, sym, g, seams):
    """{buffer: its 2 distinct frames} for a tall case; src-tall calls get banded frames, dst-tall ones small random
    sources"""
    w, h = g["w"], g["h"]
    if sym == "lbp_detect":                                   # a face band (lena) at each place, then a flat frame
        face = np.ascontiguousarray(calls.lena()[40:104, 44:108])
        a = np.zeros((h, w), np.uint8)
        for y0 in [0, h - 64] + [s - 32 for s in seams]:
            y0 = min(max(y0, 0), h - 64)
            a[y0:y0 + 64] = face
        return {"ii": np.stack([L.o_integral(O, a), L.o_integral(O, np.zeros((h, w), np.uint8))])}
    kind = {"blobs": "binary", "orb_extract": "natural", "orb_pyramid": "natural"}.get(sym, "random")
    if sym in ("perspective_correct", "resize"):
        fr = np.random.default_rng(w + h).integers(0, 256, (2, h, w), dtype=np.uint8)
    else:
        fr = np.stack([banded(w, h, seams, 1, 0, kind=kind), banded(w, h, seams, 2, 200 if kind == "random" else 0,
                                                                    kind=kind)])
    if sym == "match_template":
        return {"src": fr, "tmpl": np.ascontiguousarray(fr[0, 3:3 + g["th"], 10:10 + g["tw"]])}
    if sym == "find_best_match":
        return {"res": fr // 2}
    if sym == "threshold_each":
        return {"src": fr, "thresh": np.array([100, 7], np.uint8)}
    if sym == "perspective_correct":
        return {"src": fr, "corners": np.random.default_rng(5).integers(0, min(w, h), (2, 4, 2)).astype(np.uint32)}
    if sym in ("fast", "orb_extract"):
        return {"src": fr, "score": np.full_like(fr, POISON)}
    if sym == "rois_resize":
        rng = np.random.default_rng(3)
        rects = np.zeros((2, g["mr"]), L.RECT_DTYPE)
        for i in range(2):
            rects[i] = [(int(rng.integers(0, w - 12)), int(rng.integers(0, h - 10)), 12, 10),   # a copy slot
                        (0, h - 700, w, 700), (3, 1000, 40, h - 1000)]
        return {"src": fr, "rects": rects, "rcounts": np.array([3, 2], np.uint32)}
    if sym == "orb_pyramid":
        sizes = L.layout(w, h, g["levels"])[0]
        return {"src": fr, "score": [np.full((2, a * b), POISON, np.uint8) for a, b in sizes]}
    return {"src": fr}


def run_tall(lib, O, witness, sym, kernels, g, seams, what):
    import torch
    ins = tall_inputs(O, sym, g, seams)
    if "nkps" in g and sym != "orb_pyramid":                  # nkps above each frame's count: the last band's keypoints
        sp = calls.spec("gs_b200_%s_batch" % sym, g)          # are in the list
        want = sp.expect(ins, calls.filled(sp, 2))
        assert int(want["counts"].max()) < g["nkps"] and int(want["counts"].min()) > 0, want["counts"]
    idx = torch.arange(2, device="cuda")
    witnessed(witness, lambda: run_batch(lib, O, sym, g, 2, idx, ins=ins), kernels, what)


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["past", "last_old"])
@pytest.mark.parametrize("row_", [pytest.param(r, id=tall_id(r)) for r in TALL])
def test_tall_frame(lib, O, witness, row_, which):
    """every output byte of a frame past (or at) its site's old row-tile limit against the oracle; device memory in the
    module docstring's table"""
    _room(4)
    sym, kernels, g0, key, tile, first, extra, past = row_
    c = L.tile_constants()
    g = tall_geometry(row_, c, which)
    seams = [first + GRID * tile(c)]
    run_tall(lib, O, witness, sym, kernels, g, seams, "%s %s=%d" % (tall_id(row_), key, g[key]))


@pytest.mark.gpu
@pytest.mark.parametrize("sym,kernels,g", [pytest.param(s, k, g, id=row_id(s, g)) for s, k, g in TALL_CONTROLS])
def test_tall_frame_control(lib, O, witness, sym, kernels, g):
    _room(4)
    run_tall(lib, O, witness, sym, kernels, g, [GRID * 8], "%s h=%d" % (row_id(sym, g), g["h"]))


# fp32 row coordinates past 2^24: (float)y itself rounds, as in the reference's (y + 0.5f) and y / (h - 1)
FP32_ROWS = [
    row("resize", ["gsb::k_resize<false>"], w=16, h=16, dw=1, dh=2 ** 24 + 5),
    row("perspective_correct", ["gsb::k_perspective"], w=48, h=40, dw=1, dh=2 ** 24 + 5),
]


@pytest.mark.gpu
@pytest.mark.parametrize("sym,kernels,g", [pytest.param(s, k, g, id=row_id(s, g)) for s, k, g in FP32_ROWS])
def test_tall_fp32_rows(lib, O, witness, sym, kernels, g):
    _room(4)
    run_tall(lib, O, witness, sym, kernels, g, [], "%s dh=%d" % (sym, g["dh"]))


# ---- the single-image drop-in calls on tall host arrays ---------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("call", ["perspective_correct", "sobel", "resize", "fast_foreign_map"])
def test_tall_single_image(G, O, call):
    """host numpy arrays through the reference-style gs_* calls, bit-exact with the oracle"""
    rng = np.random.default_rng(9)
    if call == "perspective_correct":
        src = rng.integers(0, 256, (40, 48), dtype=np.uint8)
        q = np.array([[3, 2], [44, 5], [40, 37], [1, 30]], np.uint32)
        got = G.gs_perspective_correct(np.full((65_536, 1), POISON, np.uint8), src, q)
        want = np.empty((65_536, 1), np.uint8)
        O.gso_perspective_correct(L.ptr(want), 1, 65_536, L.ptr(src), 48, 40, L.ptr(q))
    elif call == "sobel":
        src = banded(5, 600_000, [GRID * 8], 4)
        got = np.full_like(src, POISON)
        G.gs_sobel(got, src)
        want = L.o_sobel(O, src, POISON)
    elif call == "resize":
        src = rng.integers(0, 256, (16, 16), dtype=np.uint8)
        got = np.full((4_194_300, 3), POISON, np.uint8)
        G.gs_resize(got, src)
        want = L.o_resize(O, src, 3, 4_194_300)
    else:
        src = banded(16, 600_000, [3 + GRID * 8], 6)
        got_sm, want_sm = np.full((600_010, 20), POISON, np.uint8), np.full((600_010, 20), POISON, np.uint8)
        got = G.gs_fast(src, got_sm, 4096, 20)
        want = L.o_fast(O, src, want_sm, 4096, 20)
        assert 0 < len(want) < 4096
        assert np.array_equal(got_sm, want_sm), "score map"
    assert got.tobytes() == want.tobytes()
