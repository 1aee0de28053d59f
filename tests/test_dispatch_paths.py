"""Every kernel the batched entry points can pick, each reached through the inputs that pick it.

The C entry points choose a kernel from the width's residue and from the alignment of the device pointers: the TMA
kernels need w % 16 == 0 and 16-byte bases, k_box_mid and k_filter3 w % 8 == 0 and 8-byte bases, the vector forms of
downsample / integral / histogram / threshold / match_template / ORB 4-, 8- or 16-byte bases, and so on.  A fresh
torch allocation is 256-byte aligned, so the branches in between are reached through views: a sub-batch frames[k:]
whose frame size is not a multiple of 16, or an out= view into a larger buffer.  ROWS is the coverage record: one
dispatch geometry per row (op, sizes, a byte offset for each base) and the kernels the dispatch code must launch.

  * GPU, per row: every frame of the batch is bit-exact against the oracle (tests/_libs.py), and the bytes of each
    allocation outside its view are untouched.  The call runs under torch.profiler, and the row's kernels must be
    among the launched ones (the path witness), so a dispatch change that moves a row to another kernel fails even
    when the other kernel computes the same bytes.
  * CPU (census): every kernel in the built library's SASS is named by a row or sits in ALLOWED with its reason, so
    a kernel added without a row fails without a GPU.
"""
import os
import re

import numpy as np
import pytest

import _libs as L
from _gpu import O, Region, frames, kernel_id, lib, stream, traced, witness, witnessed  # noqa: F401


def row(op, kernels, **p):
    p.setdefault("n", 3)
    return op, (kernels,) if isinstance(kernels, str) else tuple(kernels), p


def _box_rows():
    out = []
    for r in range(1, 8):                                        # TMA tiles: w % 16 == 0, 16-byte bases
        out.append(row("blur", "gsb::k_box_tma<%d, false>" % r, w=272, h=70, r=r))
        out.append(row("adaptive", "gsb::k_box_tma<%d, true>" % r, w=272, h=70, r=r, c=7 - 2 * r))
    for r in (8, 9, 10, 11):                                     # k_box_mid with the TMA L2 prefetch, every r & 3
        out.append(row("blur", "gsb::k_box_mid<%d, false>" % (r & 3), w=528, h=100, r=r, tpf=1))
        out.append(row("adaptive", "gsb::k_box_mid<%d, true>" % (r & 3), w=272, h=100, r=r, c=r - 9, tpf=1))
    for w in (24, 200, 360, 1080):                               # k_box_mid without it: w = 8 mod 16
        for r in (1, 3, 5, 7, 8, 11, 15, 31, 120):
            out.append(row("blur", "gsb::k_box_mid<%d, false>" % (r & 3), w=w, h=70, r=r, tpf=0))
    for r in (2, 5, 8, 11):
        out.append(row("adaptive", "gsb::k_box_mid<%d, true>" % (r & 3), w=1080, h=70, r=r, c=3 - r, tpf=0))
    out.append(row("adaptive", "gsb::k_box_mid<3, true>", w=24, h=70, r=31, c=-2, tpf=0))
    # w % 16 == 0, a base 8 but not 16-byte aligned: only dst misses TMA (the prefetch map is over src), or src does
    out += [row("blur", "gsb::k_box_mid<2, false>", w=256, h=70, r=2, src=8, dst=8, tpf=0),
            row("blur", "gsb::k_box_mid<1, false>", w=256, h=70, r=9, src=8, tpf=0),
            row("blur", "gsb::k_box_mid<1, false>", w=256, h=70, r=5, dst=8, tpf=1),
            row("adaptive", "gsb::k_box_mid<1, true>", w=256, h=70, r=13, c=4, src=8, tpf=0)]
    # ragged widths or 4-byte bases: k_box_wide (byte gathers / stores)
    out += [row("blur", "gsb::k_box_wide<false>", w=100, h=70, r=9),
            row("blur", "gsb::k_box_wide<false>", w=256, h=70, r=5, src=4),
            row("blur", "gsb::k_box_wide<false>", w=1080, h=70, r=31, dst=4),
            row("adaptive", "gsb::k_box_wide<true>", w=612, h=70, r=15, c=5),
            row("adaptive", "gsb::k_box_wide<true>", w=256, h=70, r=3, c=-1, src=4),
            # c <= INT_MIN + 255: the lane compare of k_box_tma / k_box_mid cannot express the wrap, so a TMA geometry
            # takes k_box_wide
            row("adaptive", "gsb::k_box_wide<true>", w=272, h=70, r=5, c=-2 ** 31)]
    # r = 0 and r > 120: one thread per pixel
    out += [row("blur", "gsb::k_box_generic<false>", w=200, h=40, r=121),
            row("blur", "gsb::k_box_generic<false>", w=272, h=40, r=0),
            row("adaptive", "gsb::k_box_generic<true>", w=100, h=40, r=130, c=2)]
    return out


def _blur_sobel_rows():
    out = [row("blur_sobel", "gsb::k_blur_sobel_tma<%d>" % r, w=272, h=70, r=r) for r in range(1, 8)]
    # the fall-back: blur into a scratch batch, then sobel into dst
    out += [row("blur_sobel", ("gsb::k_box_mid<1, false>", "gsb::k_stencil3_generic<0>"), w=1080, h=40, r=5),
            row("blur_sobel", ("gsb::k_box_mid<3, false>", "gsb::k_stencil3_generic<0>"), w=200, h=40, r=11),
            row("blur_sobel", ("gsb::k_box_mid<1, false>", "gsb::k_stencil3_tma<0>"), w=272, h=40, r=9),
            row("blur_sobel", ("gsb::k_box_mid<3, false>", "gsb::k_stencil3_tma<0>"), w=272, h=40, r=3, src=8),
            row("blur_sobel", ("gsb::k_box_tma<2, false>", "gsb::k_stencil3_generic<0>"), w=272, h=40, r=2, dst=1)]
    return out


def _stencil_rows():
    out = []
    for op, k in (("sobel", 0), ("erode", 1), ("dilate", 2)):
        out += [row(op, "gsb::k_stencil3_tma<%d>" % k, w=272, h=41),
                row(op, "gsb::k_stencil3_generic<%d>" % k, w=272, h=41, dst=1),
                row(op, "gsb::k_stencil3_generic<%d>" % k, w=100, h=37)]
    return out


def _resample_rows():
    return [row("downsample", "gsb::k_downsample_vec", w=272, h=41),
            row("downsample", "gsb::k_downsample_generic", w=272, h=41, dst=4),
            row("downsample", "gsb::k_downsample_generic", w=100, h=37),
            row("resize", "gsb::k_downsample_vec", w=272, h=40, dw=136, dh=20),           # exact 2:1
            row("resize", "gsb::k_resize_tiled<true>", w=272, h=60, dw=200, dh=50),
            row("resize", "gsb::k_resize_tiled<false>", w=272, h=60, dw=200, dh=50, dst=1),
            row("resize", "gsb::k_resize_tiled<false>", w=272, h=60, dw=201, dh=50),
            # k_resize: aligned8 (every source row 8-byte aligned) true, then false
            row("resize", "gsb::k_resize<true>", w=264, h=60, dw=200, dh=50),
            row("resize", "gsb::k_resize<true>", w=272, h=60, dw=200, dh=50, src=8),
            row("resize", "gsb::k_resize<true>", w=264, h=60, dw=132, dh=50),             # 2:1 in x only
            row("resize", "gsb::k_resize<false>", w=264, h=60, dw=201, dh=50),
            row("resize", "gsb::k_resize<true>", w=272, h=60, dw=200, dh=50, src=4),
            row("resize", "gsb::k_resize<false>", w=100, h=37, dw=37, dh=50)]


def _integral_rows():
    rows_cols = ("gsb::k_integral_rows<%s>", "gsb::k_integral_cols")
    return [row("integral", "gsb::k_integral_strips<64, 16>", w=1000, h=37, env="strips"),
            row("integral", "gsb::k_integral_strips<128, 8>", w=4104, h=9, env="strips"),
            row("integral", "gsb::k_integral_bands<512>", w=40, h=17, n=32, env="bands"),
            row("integral", "gsb::k_integral_bands<1024>", w=4104, h=5, n=32, env="bands"),
            row("integral", (rows_cols[0] % "true", rows_cols[1]), w=272, h=41, src=4),
            row("integral", (rows_cols[0] % "true", rows_cols[1]), w=100, h=37),
            row("integral", (rows_cols[0] % "false", rows_cols[1]), w=272, h=41, ii=4),
            row("integral", (rows_cols[0] % "false", rows_cols[1]), w=272, h=41, ii=8),
            row("integral", (rows_cols[0] % "false", rows_cols[1]), w=101, h=37, ii=12, src=1),
            row("integral", (rows_cols[0] % "false", rows_cols[1]), w=272, h=41, ii=8, env="strips")]


def _histogram_rows():
    return [row("histogram", "gsb::k_histogram<true>", w=272, h=41),
            row("histogram", "gsb::k_histogram<false>", w=272, h=41, src=1, hist=4),
            row("histogram", "gsb::k_histogram<false>", w=100, h=37),
            row("otsu", ("gsb::k_histogram<true>", "gsb::k_otsu"), w=272, h=41, n=5),
            row("otsu", ("gsb::k_histogram<false>", "gsb::k_otsu"), w=101, h=37, n=5, src=3),
            row("threshold", "gsb::k_threshold<true>", w=272, h=41, t=100),
            row("threshold", "gsb::k_threshold<false>", w=100, h=37, t=100),
            row("threshold_each", "gsb::k_threshold<true>", w=272, h=41, offset=10),
            row("threshold_each", "gsb::k_threshold<false>", w=272, h=41, offset=-20, src=4)]


def _filter_rows():
    return [row("filter", "gsb::k_filter3<true>", w=272, h=41, k="sharpen"),
            row("filter", "gsb::k_filter3<false>", w=200, h=41, k="gaussian"),
            row("filter", "gsb::k_filter_generic", w=272, h=41, k="sharpen", src=4),
            row("filter", "gsb::k_filter_generic", w=272, h=41, k="gaussian", dst=4),
            row("filter", "gsb::k_filter_generic", w=100, h=41, k="gaussian"),
            row("filter", "gsb::k_filter_generic", w=272, h=41, k="k5"),
            row("match_template", ("gsb::k_pack_template", "gsb::k_match_template"), w=256, h=60, tw=30, th=24),
            row("match_template", ("gsb::k_pack_template", "gsb::k_match_template"), w=256, h=60, tw=7, th=5, res=1),
            row("match_template", "gsb::k_match_template_generic", w=256, h=60, tw=30, th=24, src=1),
            row("match_template", "gsb::k_match_template_generic", w=101, h=37, tw=9, th=4),
            # result maps with odd rw * rh: frame bases fall mid-word; winners in a chunk's unaligned head and tail
            row("find_best_match", ("gsb::k_best_match_partial", "gsb::k_best_match_final"), w=101, h=37, n=5, res=1),
            row("find_best_match", ("gsb::k_best_match_partial", "gsb::k_best_match_final"), w=301, h=251, n=5, res=3)]


def _fast_orb_rows():
    tail = ("gsb::k_row_scan", "gsb::k_nms_emit_masks")
    orb = ("gsb::k_orb_select", "gsb::k_orb_moments", "gsb::k_orb_trig")
    return [row("fast", ("gsb::k_fast_tiled2<true>",) + tail, w=272, h=60, t=20),
            row("fast", ("gsb::k_fast_tiled2<false>",) + tail, w=272, h=60, t=20, score=4),
            row("fast", ("gsb::k_fast_tiled2<false>",) + tail, w=272, h=60, t=20, src=1),
            row("fast", ("gsb::k_fast_tiled2<false>",) + tail, w=101, h=37, t=10),
            # thresholds above 255 take the per-pixel score kernel and the separate NMS mask pass
            row("fast", ("gsb::k_fast_score", "gsb::k_nms_mask<true>") + tail, w=272, h=60, t=2 ** 32 - 200),
            row("fast", ("gsb::k_fast_score", "gsb::k_nms_mask<false>") + tail, w=272, h=60, t=300, score=1),
            row("orb", ("gsb::k_fast_tiled2<true>", "gsb::k_orb_brief<true>") + orb, w=272, h=60, t=20),
            row("orb", ("gsb::k_fast_tiled2<false>", "gsb::k_orb_brief<false>") + orb, w=272, h=60, t=20, src=1),
            row("orb", ("gsb::k_fast_tiled2<false>", "gsb::k_orb_brief<false>") + orb, w=202, h=60, t=20)]


def _lbp_rows():
    v3 = ("gsb::k_deinterleave2", "gsb::k_lbp_count", "gsb::k_row_scan", "gsb::k_lbp_emit")
    v2 = ("gsb::k_lbp_scan2", "gsb::k_lbp_count", "gsb::k_row_scan", "gsb::k_lbp_emit")
    v1 = ("gsb::k_row_scan", "gsb::k_lbp_emit")
    return [row("lbp", ("gsb::k_lbp_scan3<512>",) + v3, w=136, h=130, big="0"),
            row("lbp", ("gsb::k_lbp_scan3<1024>",) + v3, w=136, h=130, big="1"),
            row("lbp", v2, w=136, h=130, ii=4),
            row("lbp", v2, w=136, h=130, ii=8),
            row("lbp", v2, w=136, h=130, ii=12),
            row("lbp", v2, w=130, h=130),                              # iw % 8 != 0: no parity-plane tiles
            # cascade tables beyond k_lbp_scan2's 160 KB of shared memory; then a feature outside its window
            row("lbp", ("gsb::k_lbp_scan<false>",) + v1, w=136, h=130, ii=4, cascade="padded"),
            row("lbp", ("gsb::k_lbp_scan<true>",) + v1, w=136, h=130, cascade="unsafe")]


def _other_rows():
    blobs = ("gsb::k_blob_mask", "gsb::k_blob_seed", "gsb::k_row_scan", "gsb::k_blob_overflow", "gsb::k_blob_runs",
             "gsb::k_blob_union", "gsb::k_blob_label", "gsb::k_blob_compact")
    return [row("blobs", blobs, w=100, h=37, src=1),
            row("blob_corners", "gsb::k_blob_corners", w=100, h=37, n=1, src=1),
            row("perspective", "gsb::k_perspective", w=200, h=150, dw=90, dh=71, src=1, dst=3),
            row("perspective", "gsb::k_perspective", w=200, h=150, dw=90, dh=71, per_frame=1),
            row("match_orb", ("gsb::k_match_best", "gsb::k_match_compact"), n=3)]


ROWS = (_box_rows() + _blur_sobel_rows() + _stencil_rows() + _resample_rows() + _integral_rows() + _histogram_rows() +
        _filter_rows() + _fast_orb_rows() + _lbp_rows() + _other_rows())

# kernels without a row here, each with the reason
ALLOWED = {
    r"gsb::k_trig_selfcheck": "runs once per process on its own stream before the first ORB angle; "
                              "test_gpu_parity.py::test_trig_selfcheck_matches_this_libm checks its verdict",
    r"gsb::k_orient_one": "single-image gs_compute_orientation; test_gpu_parity.py golden and large-radius tests",
    r"gsb::k_brief_one": "single-image gs_brief_descriptor; test_gpu_parity.py golden test",
    r"gsb::k_lbp_window_one": "single-image gs_lbp_window; test_gpu_parity.py golden test",
    r"gsb::k_morph_(tma|rows|cols)<.*>": "erode_n / dilate_n: test_morph_iter.py runs both of its paths at pointer "
                                        "offsets and counts their launches",
}


def row_id(op, p):
    return "-".join([op] + ["%s%s" % (k, v) for k, v in p.items() if k != "n"] + ["n%d" % p["n"]])


# ---- CPU: the census -----------------------------------------------------------------------------------------------
def test_rows_are_unique_and_well_formed():
    ids = [row_id(op, p) for op, _, p in ROWS]
    assert len(ids) == len(set(ids)), sorted(i for i in ids if ids.count(i) > 1)
    for op, kernels, p in ROWS:
        assert kernels and all(k.startswith("gsb::k_") for k in kernels), (op, kernels)
        if "tpf" in p:   # k_box_mid prefetches through a TMA map over src: w % 16 == 0 and a 16-byte aligned base
            assert p["tpf"] == int(p["w"] % 16 == 0 and p.get("src", 0) % 16 == 0), p


def test_every_kernel_has_a_row():
    built = set(L.sass_functions())
    assert len(built) > 50, sorted(built)
    table = {kernel_id(k) for _, kernels, _ in ROWS for k in kernels}
    orphans = sorted(k for k in built if k not in table and not any(re.fullmatch(a, k) for a in ALLOWED))
    assert not orphans, "kernels with neither a dispatch row nor an ALLOWED entry: %s" % orphans
    assert not sorted(table - built), "rows naming kernels the library does not have: %s" % sorted(table - built)
    assert not [k for k in built if k.startswith("gsb::k_box_wide<") and k.count(",")], "k_box_wide has one parameter"


def test_kernel_id_normal_form():
    assert kernel_id("void gsb::k_box_mid<(int)1, (bool)0>(CUtensorMap_st, int)") == "gsb::k_box_mid<1,false>"
    assert kernel_id("void gsb::k_box_mid<1, false>(CUtensorMap_st, int, unsigned char*)") == "gsb::k_box_mid<1,false>"
    assert kernel_id("gsb::k_integral_strips<(int)128, (int)8>(unsigned int *)") == "gsb::k_integral_strips<128,8>"
    assert kernel_id("gsb::k_otsu(unsigned char*, unsigned int const*, unsigned int, unsigned int)") == "gsb::k_otsu"


def test_launch_policy_lives_in_one_place():
    """every kernel launch goes through gsb::launch (common.cuh), whose shared-memory opt-in and launch counter are in
    runtime.cu: so the counter gs_b200_launch_count reports counts each launch once, and no call site opts in by hand"""
    csrc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "grayskull_b200", "csrc")
    found = {"<<<": set(), "cudaFuncSetAttribute": set(), "g_launches": set()}
    for f in sorted(os.listdir(csrc)):
        with open(os.path.join(csrc, f)) as fh:
            text = fh.read()
        for needle, files in found.items():
            if needle in text:
                files.add(f)
    assert found == {"<<<": {"common.cuh"}, "cudaFuncSetAttribute": {"runtime.cu"}, "g_launches": {"runtime.cu"}}, found


# ---- GPU -----------------------------------------------------------------------------------------------------------
def _src(p, fr, seed=1):
    S = Region(fr.nbytes, p.get("src", 0), fr, seed)
    return S


def _src_kept(S, fr):
    assert np.array_equal(S.read("src"), fr.reshape(-1)), "the input changed"


def _ok(rc):
    from grayskull_b200 import _lib
    _lib.check(rc, "dispatch row")


def r_box(lib, O, p, adaptive):
    w, h, n, r = p["w"], p["h"], p["n"], p["r"]
    fr = frames(w, h, n, w + h + r)
    S, D = _src(p, fr), Region(fr.nbytes, p.get("dst", 0), seed=2)
    if adaptive:
        rc, seen = traced(lambda: lib.gs_b200_adaptive_threshold_batch(D.ptr, S.ptr, w, h, n, r, p["c"], stream()))
    else:
        rc, seen = traced(lambda: lib.gs_b200_blur_batch(D.ptr, S.ptr, w, h, n, r, stream()))
    _ok(rc)
    got = D.read("dst").reshape(n, h, w)
    _src_kept(S, fr)
    for i in range(n):
        want = L.o_adaptive(O, fr[i], r, p["c"]) if adaptive else L.o_blur(O, fr[i], r)
        assert np.array_equal(got[i], want), i
    return seen


def r_blur_sobel(lib, O, p):
    w, h, n, r = p["w"], p["h"], p["n"], p["r"]
    fr = frames(w, h, n, w + h + r)
    S, D = _src(p, fr), Region(fr.nbytes, p.get("dst", 0), seed=2)
    rc, seen = traced(lambda: lib.gs_b200_blur_sobel_batch(D.ptr, S.ptr, w, h, n, r, stream()))
    _ok(rc)
    got, fill = D.read("dst").reshape(n, h, w), D.before().reshape(n, h, w)
    _src_kept(S, fr)
    for i in range(n):
        want = fill[i].copy()                                   # the untouched 1-px frame keeps dst's bytes
        O.gso_sobel(L.ptr(want), L.ptr(L.o_blur(O, fr[i], r)), w, h)
        assert np.array_equal(got[i], want), i
    return seen


def r_stencil(lib, O, p, op):
    w, h, n = p["w"], p["h"], p["n"]
    fr = frames(w, h, n, w + h)
    S, D = _src(p, fr), Region(fr.nbytes, p.get("dst", 0), seed=2)
    fn = {"sobel": lib.gs_b200_sobel_batch, "erode": lib.gs_b200_erode_batch, "dilate": lib.gs_b200_dilate_batch}[op]
    rc, seen = traced(lambda: fn(D.ptr, S.ptr, w, h, n, stream()))
    _ok(rc)
    got, fill = D.read("dst").reshape(n, h, w), D.before().reshape(n, h, w)
    _src_kept(S, fr)
    for i in range(n):
        if op == "sobel":
            want = fill[i].copy()
            O.gso_sobel(L.ptr(want), L.ptr(fr[i]), w, h)
        else:
            want = L.o_morph(O, fr[i], op == "dilate")
        assert np.array_equal(got[i], want), i
    return seen


def r_resample(lib, O, p, op):
    w, h, n = p["w"], p["h"], p["n"]
    dw, dh = (w // 2, h // 2) if op == "downsample" else (p["dw"], p["dh"])
    fr = frames(w, h, n, w + h + dw)
    S, D = _src(p, fr), Region(n * dw * dh, p.get("dst", 0), seed=2)
    if op == "downsample":
        rc, seen = traced(lambda: lib.gs_b200_downsample_batch(D.ptr, S.ptr, w, h, n, stream()))
    else:
        rc, seen = traced(lambda: lib.gs_b200_resize_batch(D.ptr, dw, dh, S.ptr, w, h, n, stream()))
    _ok(rc)
    got = D.read("dst").reshape(n, dh, dw)
    _src_kept(S, fr)
    for i in range(n):
        want = L.o_down(O, fr[i]) if op == "downsample" else L.o_resize(O, fr[i], dw, dh)
        assert np.array_equal(got[i], want), i
    return seen


def r_integral(lib, O, p):
    w, h, n = p["w"], p["h"], p["n"]
    fr = frames(w, h, n, w + h + n)
    S, D = _src(p, fr), Region(4 * n * w * h, p.get("ii", 0), seed=2)
    if "env" in p:
        os.environ["GS_B200_INTEGRAL"] = p["env"]
    try:
        rc, seen = traced(lambda: lib.gs_b200_integral_batch(D.ptr, S.ptr, w, h, n, stream()))
    finally:
        os.environ.pop("GS_B200_INTEGRAL", None)
    _ok(rc)
    got = D.read("ii").view(np.uint32).reshape(n, h, w)
    _src_kept(S, fr)
    for i in range(n):
        assert np.array_equal(got[i], L.o_integral(O, fr[i])), i
    return seen


def r_histogram(lib, O, p, op):
    w, h, n = p["w"], p["h"], p["n"]
    fr = frames(w, h, n, w + h)
    fr[n - 1] = np.random.default_rng(3).integers(0, 256, (h, w), dtype=np.uint8) // 64 * 64   # four bins only
    S = _src(p, fr)
    if op == "histogram":
        D = Region(4 * 256 * n, p.get("hist", 0), seed=2)
        rc, seen = traced(lambda: lib.gs_b200_histogram_batch(D.ptr, S.ptr, w, h, n, stream()))
        _ok(rc)
        got = D.read("hist").view(np.uint32).reshape(n, 256)
        for i in range(n):
            assert np.array_equal(got[i], np.bincount(fr[i].ravel(), minlength=256)), i
    else:
        D = Region(n, 1, seed=2)
        rc, seen = traced(lambda: lib.gs_b200_otsu_threshold_batch(D.ptr, None, S.ptr, w, h, n, stream()))
        _ok(rc)
        got = D.read("thresholds")
        for i in range(n):
            assert got[i] == O.gso_otsu_threshold(L.ptr(fr[i]), w, h), i
    _src_kept(S, fr)
    return seen


def r_threshold(lib, O, p, each):
    w, h, n = p["w"], p["h"], p["n"]
    fr = frames(w, h, n, w + h)
    S = _src(p, fr)                                            # in place
    if each:
        thr = np.array([100, 0, 250, 37, 255][:n], np.uint8)
        T = Region(n, 3, thr, seed=2)
        rc, seen = traced(lambda: lib.gs_b200_threshold_each_batch(S.ptr, w, h, n, T.ptr, p["offset"], stream()))
        T.read("thresholds")
        ts = [(int(t) + p["offset"]) & 255 for t in thr]
    else:
        rc, seen = traced(lambda: lib.gs_b200_threshold_batch(S.ptr, w, h, n, p["t"], stream()))
        ts = [p["t"]] * n
    _ok(rc)
    got = S.read("img").reshape(n, h, w)
    for i in range(n):
        want = fr[i].copy()
        O.gso_threshold(L.ptr(want), w, h, ts[i])
        assert np.array_equal(got[i], want), i
    return seen


def r_filter(lib, O, p):
    w, h, n = p["w"], p["h"], p["n"]
    fr = frames(w, h, n, w + h)
    k, norm = L.filter_kernel(p["k"])
    S, D = _src(p, fr), Region(fr.nbytes, p.get("dst", 0), seed=2)
    ks = np.ascontiguousarray(k)
    rc, seen = traced(lambda: lib.gs_b200_filter_batch(D.ptr, S.ptr, w, h, n, ks.ctypes.data, ks.shape[1], ks.shape[0],
                                                      norm, stream()))
    _ok(rc)
    got = D.read("dst").reshape(n, h, w)
    _src_kept(S, fr)
    for i in range(n):
        want = np.zeros_like(fr[i])
        O.gso_filter(L.ptr(want), L.ptr(fr[i]), w, h, L.ptr(ks), ks.shape[1], ks.shape[0], norm)
        assert np.array_equal(got[i], want), i
    return seen


def r_match_template(lib, O, p):
    w, h, n, tw, th = p["w"], p["h"], p["n"], p["tw"], p["th"]
    fr = frames(w, h, n, w + h)
    tmpl = np.ascontiguousarray(fr[1, 10:10 + th, 20:20 + tw])
    rw, rh = w - tw + 1, h - th + 1
    S, T, D = _src(p, fr), Region(tmpl.nbytes, 0, tmpl, seed=3), Region(n * rw * rh, p.get("res", 0), seed=2)
    rc, seen = traced(lambda: lib.gs_b200_match_template_batch(D.ptr, S.ptr, w, h, n, T.ptr, tw, th, stream()))
    _ok(rc)
    got = D.read("result").reshape(n, rh, rw)
    _src_kept(S, fr)
    T.read("template")
    for i in range(n):
        want = np.zeros((rh, rw), np.uint8)
        O.gso_match_template(L.ptr(fr[i]), w, h, L.ptr(tmpl), tw, th, L.ptr(want))
        assert np.array_equal(got[i], want), i
    return seen


def r_find_best_match(lib, O, p):
    rw, rh, n = p["w"], p["h"], p["n"]
    px = rw * rh
    assert px % 2 == 1
    rng = np.random.default_rng(px)
    maps = (rng.integers(0, 200, (n, px)) * (rng.random((n, px)) < 0.5)).astype(np.uint8)
    maps[1, 0] = 255                                     # the first byte of a frame: the unaligned head of chunk 0
    maps[1, 5] = 255                                     # a tie after it: the first index wins
    maps[2, px - 1] = 255                                # the last byte: the unaligned tail of the last chunk
    maps[3] = 0                                          # nothing above 0: (0, 0)
    maps[4, px // 2] = 254                               # interior
    maps[4, px // 2 + 1] = 254
    M, B = Region(maps.nbytes, p.get("res", 0), maps, seed=3), Region(8 * n, 0, seed=2)
    rc, seen = traced(lambda: lib.gs_b200_find_best_match_batch(B.ptr, M.ptr, rw, rh, n, stream()))
    _ok(rc)
    got = B.read("best").view(np.uint32).reshape(n, 2)
    M.read("result")
    for i in range(n):
        b = O.gso_find_best_match(L.ptr(np.ascontiguousarray(maps[i])), rw, rh)
        assert tuple(got[i]) == (b % rw, b // rw), i
    assert tuple(got[1]) == (0, 0) and tuple(got[2]) == ((px - 1) % rw, (px - 1) // rw)
    return seen


def r_fast(lib, O, p, orb):
    w, h, n, t = p["w"], p["h"], p["n"], p["t"]
    nk = 400
    fr = frames(w, h, n, w + h)
    fr[2] = L.natural_like(w, h, 99)                     # corners in every frame
    rng = np.random.default_rng(w)
    stale = np.zeros_like(fr) if orb else (rng.integers(0, 256, fr.shape) * (rng.random(fr.shape) < 0.02)).astype(np.uint8)
    S, SM = _src(p, fr), Region(fr.nbytes, p.get("score", 0), stale, seed=4)
    K, N = Region(48 * n * nk, 0, seed=5), Region(4 * n, 0, seed=6)
    fn = lib.gs_b200_orb_extract_batch if orb else lib.gs_b200_fast_batch
    rc, seen = traced(lambda: fn(S.ptr, w, h, n, SM.ptr, K.ptr, N.ptr, nk, t, stream()))
    _ok(rc)
    counts = N.read("counts").view(np.uint32)
    kps = K.read("kps").view(np.uint32).reshape(n, nk, 12)
    sm = SM.read("scoremap").reshape(n, h, w)
    _src_kept(S, fr)
    for i in range(n):
        so = stale[i].copy()
        want = L.o_orb(O, fr[i], so, nk, t) if orb else L.o_fast(O, fr[i], so, nk, t)
        got = np.ascontiguousarray(kps[i, :counts[i]]).view(L.KP_DTYPE).reshape(-1)
        assert got.tobytes() == want.tobytes(), (i, len(got), len(want))
        if not orb:
            assert np.array_equal(sm[i], so), i
    assert counts.sum() > 0 or t > 255
    return seen


def _cascade(kind):
    from grayskull_b200._lib import HostCascade
    z = np.load(os.path.join(L.ROOT, "grayskull_b200", "data", "frontalface.npz"))
    a = {k: z[k] for k in z.files}
    if kind == "padded":        # 5000 features (copies of feature 0, never referenced): tables of ~170 KB
        a["features"] = np.concatenate([a["features"], np.tile(a["features"][:4], 5000 - len(a["features"]) // 4)])
    elif kind == "unsafe":      # one unreferenced feature whose 3x3 lattice leaves the window
        a["features"] = np.concatenate([a["features"], np.array([20, 0, 2, 1], np.int8)])
    return HostCascade(a)


def r_lbp(lib, O, p):
    w, h, n = p["w"], p["h"], p["n"]
    lena = np.load(os.path.join(L.ROOT, "tests", "golden", "lena_golden.npz"))["lena"]      # 128 x 128, faces found
    fr = np.stack([np.pad(np.roll(lena, 4 * i, axis=1), ((0, h - 128), (0, w - 128)), mode="edge") if i < 2 else
                   L.natural_like(w, h, 40 + i) for i in range(n)])
    ii = np.stack([L.o_integral(O, f) for f in fr])
    cas = _cascade(p.get("cascade", "frontalface"))
    I = Region(ii.nbytes, p.get("ii", 0), ii, seed=3)
    mr = 1000
    RR, N = Region(16 * n * mr, 0, seed=4), Region(4 * n, 0, seed=5)
    if "big" in p:
        os.environ["GS_B200_LBP_BIG"] = p["big"]
    try:
        rc, seen = traced(lambda: lib.gs_b200_lbp_detect_batch(cas.ptr, I.ptr, w, h, n, RR.ptr, N.ptr, mr, 1.1, 1.0, 4.0,
                                                              2, stream()))
    finally:
        os.environ.pop("GS_B200_LBP_BIG", None)
    _ok(rc)
    counts = N.read("counts").view(np.uint32)
    rects = RR.read("rects").view(np.uint32).reshape(n, mr, 4)
    I.read("ii")
    for i in range(n):
        want = L.o_detect(O, cas, ii[i], mr, 1.1, 1.0, 4.0, 2)
        assert np.ascontiguousarray(rects[i, :counts[i]]).tobytes() == want.tobytes(), (i, counts[i], len(want))
    assert counts.sum() > 0
    return seen


def _o_blobs(O, a, nb):
    h, w = a.shape
    labels, blobs = np.zeros((h, w), np.uint16), np.zeros(nb, L.BLOB_DTYPE)
    m = O.gso_blobs(L.ptr(a), w, h, L.ptr(labels), L.ptr(blobs), nb)
    return labels, blobs[:m]


def r_blobs(lib, O, p):
    w, h, n, nb = p["w"], p["h"], p["n"], 300
    fr = np.stack([L.binary_like(w, h, 50 + i) for i in range(n)])
    S, LB = _src(p, fr), Region(2 * n * w * h, 2, seed=2)
    B, N = Region(32 * n * nb, 0, seed=3), Region(4 * n, 0, seed=4)
    rc, seen = traced(lambda: lib.gs_b200_blobs_batch(S.ptr, w, h, n, LB.ptr, B.ptr, N.ptr, nb, stream()))
    _ok(rc)
    labels = LB.read("labels").view(np.uint16).reshape(n, h, w)
    blobs, counts = B.read("blobs").view(L.BLOB_DTYPE).reshape(n, nb), N.read("counts").view(np.uint32)
    _src_kept(S, fr)
    for i in range(n):
        wl, wb = _o_blobs(O, fr[i], nb)
        assert counts[i] == len(wb) and np.array_equal(labels[i], wl), i
        assert L.blob_fields(blobs[i, :counts[i]]) == L.blob_fields(wb), i
    return seen


def r_blob_corners(lib, O, p):
    w, h = p["w"], p["h"]
    a = L.binary_like(w, h, 7)
    labels, blobs = _o_blobs(O, a, 300)
    j = int(np.argmax(blobs["area"]))
    S, LB = _src(p, a), Region(labels.nbytes, 2, labels, seed=2)
    B, CO = Region(32, 0, blobs[j:j + 1], seed=3), Region(32, 0, seed=4)
    rc, seen = traced(lambda: lib.gs_b200_blob_corners(S.ptr, w, h, LB.ptr, B.ptr, CO.ptr, stream()))
    _ok(rc)
    got = CO.read("corners").view(np.uint32).reshape(4, 2)
    want = np.zeros((4, 2), np.uint32)
    O.gso_blob_corners(L.ptr(a), w, h, L.ptr(labels), L.ptr(blobs[j:j + 1]), L.ptr(want))
    assert np.array_equal(got, want)
    return seen


def r_perspective(lib, O, p):
    w, h, n, dw, dh = p["w"], p["h"], p["n"], p["dw"], p["dh"]
    fr = frames(w, h, n, w + h)
    quads = np.random.default_rng(5).integers(0, 140, (n, 4, 2)).astype(np.uint32)
    S, D = _src(p, fr), Region(n * dw * dh, p.get("dst", 0), seed=2)
    if p.get("per_frame"):
        Q = Region(quads.nbytes, 0, quads, seed=3)
        rc, seen = traced(lambda: lib.gs_b200_perspective_correct_batch(D.ptr, dw, dh, S.ptr, w, h, n, Q.ptr, 1, stream()))
    else:
        quads[:] = quads[0]
        q0 = np.ascontiguousarray(quads[0])
        rc, seen = traced(lambda: lib.gs_b200_perspective_correct_batch(D.ptr, dw, dh, S.ptr, w, h, n, q0.ctypes.data, 0,
                                                                       stream()))
    _ok(rc)
    got = D.read("dst").reshape(n, dh, dw)
    _src_kept(S, fr)
    for i in range(n):
        want = np.empty((dh, dw), np.uint8)
        O.gso_perspective_correct(L.ptr(want), dw, dh, L.ptr(fr[i]), w, h, L.ptr(np.ascontiguousarray(quads[i])))
        assert np.array_equal(got[i], want), i
    return seen


def r_match_orb(lib, O, p):
    n, s1, s2, mm = p["n"], 130, 90, 150
    rng = np.random.default_rng(16)
    sets = [L.desc_sets(rng, n1, n2) for n1, n2 in ((120, 90), (7, 0), (130, 61))][:n]
    k1, k2 = np.zeros((n, s1), L.KP_DTYPE), np.zeros((n, s2), L.KP_DTYPE)
    c1 = np.array([len(a) for a, _ in sets], np.uint32)
    c2 = np.array([len(b) for _, b in sets], np.uint32)
    for i, (a, b) in enumerate(sets):
        k1[i, :len(a)], k2[i, :len(b)] = a, b
    K1, K2, C1, C2 = Region(k1.nbytes, 0, k1, 1), Region(k2.nbytes, 0, k2, 2), Region(4 * n, 0, c1, 3), Region(4 * n, 0, c2, 4)
    M, MC = Region(12 * n * mm, 0, seed=5), Region(4 * n, 0, seed=6)
    rc, seen = traced(lambda: lib.gs_b200_match_orb_batch(K1.ptr, C1.ptr, s1, K2.ptr, C2.ptr, s2, n, M.ptr, MC.ptr, mm, 60.0,
                                                         stream()))
    _ok(rc)
    counts, m = MC.read("counts").view(np.uint32), M.read("matches").view(np.uint32).reshape(n, mm, 3)
    for i, (a, b) in enumerate(sets):
        want = L.o_match(O, a, b, mm, 60.0)
        assert counts[i] == len(want) and np.ascontiguousarray(m[i, :counts[i]]).tobytes() == want.tobytes(), i
    return seen


RUN = {
    "blur": lambda lib, O, p: r_box(lib, O, p, False),
    "adaptive": lambda lib, O, p: r_box(lib, O, p, True),
    "blur_sobel": r_blur_sobel,
    "sobel": lambda lib, O, p: r_stencil(lib, O, p, "sobel"),
    "erode": lambda lib, O, p: r_stencil(lib, O, p, "erode"),
    "dilate": lambda lib, O, p: r_stencil(lib, O, p, "dilate"),
    "downsample": lambda lib, O, p: r_resample(lib, O, p, "downsample"),
    "resize": lambda lib, O, p: r_resample(lib, O, p, "resize"),
    "integral": r_integral,
    "histogram": lambda lib, O, p: r_histogram(lib, O, p, "histogram"),
    "otsu": lambda lib, O, p: r_histogram(lib, O, p, "otsu"),
    "threshold": lambda lib, O, p: r_threshold(lib, O, p, False),
    "threshold_each": lambda lib, O, p: r_threshold(lib, O, p, True),
    "filter": r_filter,
    "match_template": r_match_template,
    "find_best_match": r_find_best_match,
    "fast": lambda lib, O, p: r_fast(lib, O, p, False),
    "orb": lambda lib, O, p: r_fast(lib, O, p, True),
    "lbp": r_lbp,
    "blobs": r_blobs,
    "blob_corners": r_blob_corners,
    "perspective": r_perspective,
    "match_orb": r_match_orb,
}


def test_every_row_has_a_runner():
    assert {op for op, _, _ in ROWS} <= set(RUN)


@pytest.mark.gpu
@pytest.mark.parametrize("op,kernels,p", [pytest.param(op, k, p, id=row_id(op, p)) for op, k, p in ROWS])
def test_dispatch_row(lib, O, witness, op, kernels, p):
    witnessed(witness, lambda: RUN[op](lib, O, p), kernels, row_id(op, p))
