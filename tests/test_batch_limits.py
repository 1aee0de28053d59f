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
"""
import glob
import os
import re

import numpy as np
import pytest

import _calls as calls
import _libs as L
from _gpu import O, lib, stream, traced, witness, witnessed  # noqa: F401

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


def run_batch(lib, O, sym, g, n, idx, fr=None):
    """one call over n frames, frame f being distinct frame idx[f] -> the kernels it launched.  Prints the device memory
    the case took: its buffers plus what the library's workspace arenas grew by (they stay allocated after it)."""
    import torch
    free0 = torch.cuda.mem_get_info()[0]
    torch.cuda.reset_peak_memory_stats()
    sp, ins = calls.spec("gs_b200_%s_batch" % sym, g), row_inputs(O, sym, g, fr)
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
