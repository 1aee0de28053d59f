"""Every kernel the batched entry points can pick, each reached through the inputs that pick it.

The C entry points choose a kernel from the width's residue and from the alignment of the device pointers: the TMA
kernels need w % 16 == 0 and 16-byte bases, k_box_mid and k_filter3 w % 8 == 0 and 8-byte bases, the vector forms of
downsample / integral / histogram / threshold / match_template / ORB 4-, 8- or 16-byte bases, and so on.  A fresh
torch allocation is 256-byte aligned, so the branches in between are reached through views: a sub-batch frames[k:]
whose frame size is not a multiple of 16, or an out= view into a larger buffer.  ROWS is the coverage record: one
dispatch geometry per row (op, sizes, a byte offset for each base) and the kernels the dispatch code must launch.

  * GPU, per row: each buffer sits at the row's byte offset in a Region; every output is bit-exact against the
    call's expect() (tests/_calls.py), every input is unchanged, and the bytes of each allocation outside its view are
    untouched.  The call runs under torch.profiler, and the row's kernels must be
    among the launched ones (the path witness), so a dispatch change that moves a row to another kernel fails even
    when the other kernel computes the same bytes.
  * CPU (census): every kernel in the built library's SASS is named by a row or sits in ALLOWED with its reason, so
    a kernel added without a row fails without a GPU.
"""
import os

import numpy as np
import pytest

import _calls as calls
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


def _morph_n_rows():
    out = []
    for op, k in (("erode_n", 1), ("dilate_n", 2)):
        tma, s3 = "gsb::k_morph_tma<%d, %%d>" % k, "gsb::k_stencil3_tma<%d>" % k
        rows_cols = ("gsb::k_morph_rows<%d>" % k, "gsb::k_morph_cols<%d>" % k)
        # TMA geometry, 2 <= N <= 16: one launch of k_morph_tma<OP, N>
        out += [row(op, tma % it, w=272, h=70, iters=it) for it in range(2, 17)]
        # 17 <= N <= 48: launches of at most 16 composed through the workspace, a remainder of 1 on the 3x3 kernel
        out += [row(op, (tma % 16, s3), w=272, h=70, iters=17),
                row(op, (tma % 16, s3), w=272, h=70, iters=33),
                row(op, tma % 16, w=272, h=70, iters=48)]
        # the row and column passes: a ragged width, a base off 16 bytes, N' = max(min(N, w - 1), min(N, h - 1)) > 48
        out += [row(op, rows_cols, w=100, h=70, iters=3),
                row(op, rows_cols, w=272, h=70, iters=5, **({"src": 1} if k == 1 else {"dst": 1})),
                row(op, rows_cols, w=272, h=70, iters=1000)]
        # iters 1 is the 3x3 call; a saturating count clamps to N' = 271 (iters 0 is a device copy, no kernel)
        out += [row(op, s3, w=272, h=70, iters=1),
                row(op, rows_cols, w=272, h=70, iters=2 ** 32 - 1)]
    return out


def _roi_rows():
    copy, gather = "gsb::k_roi_copy", "gsb::k_roi_gather<%d>"
    # unscaled regions inside the frame take k_roi_copy in either mode, at any width, offset and alignment
    return [row("crop_resize", copy, w=272, h=70, roi=(3, 5, 160, 40), dw=160, dh=40, mode=0),
            row("crop_resize", copy, w=101, h=37, roi=(13, 7, 77, 29), dw=77, dh=29, mode=1, src=5, dst=3),
            # scaled regions: the mode's gather kernel
            row("crop_resize", gather % 0, w=272, h=70, roi=(7, 3, 50, 31), dw=64, dh=64, mode=0),
            row("crop_resize", gather % 1, w=101, h=37, roi=(2, 1, 97, 35), dw=40, dh=13, mode=1, src=7, dst=2),
            # device lists of unscaled and scaled regions: both kernels run over the list, each on its own slots
            row("rois_resize", (copy, gather % 0), w=272, h=70, dw=64, dh=48, mode=0),
            row("rois_resize", (copy, gather % 1), w=101, h=37, dw=33, dh=20, mode=1, src=3, dst=5)]


def _pyramid_rows():
    # the last level: FAST, the quota clamps around select, describe, then the merge of every level's list
    last = ("gsb::k_pyr_quota", "gsb::k_pyr_merge", "gsb::k_row_scan", "gsb::k_nms_emit_masks", "gsb::k_orb_select",
            "gsb::k_orb_moments", "gsb::k_orb_trig")
    tiled, plain = "gsb::k_fast_tiled2<true>", "gsb::k_fast_tiled2<false>"
    words, bytes_ = "gsb::k_orb_brief<true>", "gsb::k_orb_brief<false>"
    down_vec, down_generic = "gsb::k_downsample_vec", "gsb::k_downsample_generic"
    return [row("orb_pyramid", last + (tiled, words), w=272, h=70, levels=1),
            # level 1 is 136 wide (8 mod 16): FAST on plain loads there
            row("orb_pyramid", last + (tiled, plain, words, down_vec), w=272, h=70, levels=2),
            # level 2 is made from the 136-wide level 1 by the generic downsample
            row("orb_pyramid", last + (tiled, plain, words, down_vec, down_generic), w=272, h=140, levels=3),
            row("orb_pyramid", last + (plain, bytes_, words, down_generic), w=272, h=70, levels=2, src=1)]


ROWS = (_box_rows() + _blur_sobel_rows() + _stencil_rows() + _resample_rows() + _integral_rows() + _histogram_rows() +
        _filter_rows() + _fast_orb_rows() + _lbp_rows() + _other_rows() + _morph_n_rows() + _roi_rows() +
        _pyramid_rows())

# kernels without a row here, each with the reason
ALLOWED = {
    "gsb::k_trig_selfcheck": "runs once per process on its own stream before the first ORB angle; "
                             "test_gpu_parity.py::test_trig_selfcheck_matches_this_libm checks its verdict",
    "gsb::k_orient_one": "single-image gs_compute_orientation; test_gpu_parity.py golden and large-radius tests",
    "gsb::k_brief_one": "single-image gs_brief_descriptor; test_gpu_parity.py golden test",
    "gsb::k_lbp_window_one": "single-image gs_lbp_window; test_gpu_parity.py golden test",
}


def row_id(op, p):
    def text(v):
        return "_".join(map(str, v)) if isinstance(v, tuple) else v
    return "-".join([op] + ["%s%s" % (k, text(v)) for k, v in p.items() if k != "n"] + ["n%d" % p["n"]])


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
    orphans = sorted(built - table - set(ALLOWED))
    assert not orphans, "kernels with neither a dispatch row nor an ALLOWED entry: %s" % orphans
    assert not sorted(table - built), "rows naming kernels the library does not have: %s" % sorted(table - built)
    assert not sorted(set(ALLOWED) - built), "ALLOWED names kernels the library does not have"
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
# op -> its C symbol and what its rows leave implicit: the byte offsets of some buffers, list capacities, the null
# histogram of otsu and the host corners of perspective
OPS = {
    "blur": ("gs_b200_blur_batch", {}),
    "adaptive": ("gs_b200_adaptive_threshold_batch", {}),
    "blur_sobel": ("gs_b200_blur_sobel_batch", {}),
    "sobel": ("gs_b200_sobel_batch", {}),
    "erode": ("gs_b200_erode_batch", {}),
    "dilate": ("gs_b200_dilate_batch", {}),
    "downsample": ("gs_b200_downsample_batch", {}),
    "resize": ("gs_b200_resize_batch", {}),
    "integral": ("gs_b200_integral_batch", {}),
    "histogram": ("gs_b200_histogram_batch", {}),
    "otsu": ("gs_b200_otsu_threshold_batch", dict(with_hist=0, thresh=1)),
    "threshold": ("gs_b200_threshold_batch", {}),
    "threshold_each": ("gs_b200_threshold_each_batch", dict(thresh=3)),
    "filter": ("gs_b200_filter_batch", {}),
    "match_template": ("gs_b200_match_template_batch", {}),
    "find_best_match": ("gs_b200_find_best_match_batch", {}),
    "fast": ("gs_b200_fast_batch", dict(nkps=400)),
    "orb": ("gs_b200_orb_extract_batch", dict(nkps=400)),
    "lbp": ("gs_b200_lbp_detect_batch", dict(mr=1000)),
    "blobs": ("gs_b200_blobs_batch", dict(nb=300, labels=2)),
    "blob_corners": ("gs_b200_blob_corners", dict(labels=2)),
    "perspective": ("gs_b200_perspective_correct_batch", dict(per_frame=0)),
    "match_orb": ("gs_b200_match_orb_batch", dict(s1=130, s2=90, mm=150)),
    "erode_n": ("gs_b200_erode_n_batch", {}),
    "dilate_n": ("gs_b200_dilate_n_batch", {}),
    "crop_resize": ("gs_b200_crop_resize_batch", {}),
    "rois_resize": ("gs_b200_rois_resize_batch", dict(mr=5)),
    "orb_pyramid": ("gs_b200_orb_pyramid_batch", dict(nkps=400, t=20)),
}
# ops whose rows run on _calls.inputs' real inputs: region lists of unscaled and scaled slots, random score maps
DEFAULT_INPUTS = {"erode_n", "dilate_n", "crop_resize", "rois_resize", "orb_pyramid"}


def _cascade(kind):
    from grayskull_b200._lib import HostCascade
    z = np.load(os.path.join(L.ROOT, "grayskull_b200", "data", "frontalface.npz"))
    a = {k: z[k] for k in z.files}
    if kind == "padded":        # 5000 features (copies of feature 0, never referenced): tables of ~170 KB
        a["features"] = np.concatenate([a["features"], np.tile(a["features"][:4], 5000 - len(a["features"]) // 4)])
    elif kind == "unsafe":      # one unreferenced feature whose 3x3 lattice leaves the window
        a["features"] = np.concatenate([a["features"], np.array([20, 0, 2, 1], np.int8)])
    return HostCascade(a)


def row_inputs(O, op, g):
    """{buffer: its n frames} of a row"""
    w, h, n = g.get("w"), g.get("h"), g["n"]
    if op in DEFAULT_INPUTS:
        return calls.inputs(OPS[op][0], g, n, 1)
    if op == "find_best_match":
        # result maps with odd rw * rh: frame bases fall mid-word; winners in a chunk's unaligned head and tail
        px = w * h
        assert px % 2 == 1
        rng = np.random.default_rng(px)
        maps = (rng.integers(0, 200, (n, px)) * (rng.random((n, px)) < 0.5)).astype(np.uint8)
        maps[1, 0] = 255                                 # the first byte of a frame: the unaligned head of chunk 0
        maps[1, 5] = 255                                 # a tie after it: the first index wins
        maps[2, px - 1] = 255                            # the last byte: the unaligned tail of the last chunk
        maps[3] = 0                                      # nothing above 0: (0, 0)
        maps[4, px // 2] = 254                           # interior
        maps[4, px // 2 + 1] = 254
        return {"res": maps}
    if op == "lbp":
        fr = np.stack([np.pad(np.roll(calls.lena(), 4 * i, axis=1), ((0, h - 128), (0, w - 128)), mode="edge") if i < 2
                       else L.natural_like(w, h, 40 + i) for i in range(n)])
        return {"ii": np.stack([L.o_integral(O, f) for f in fr])}
    if op == "blobs":
        return {"src": np.stack([L.binary_like(w, h, 50 + i) for i in range(n)])}
    if op == "blob_corners":
        a = L.binary_like(w, h, 7)
        labels, blobs = calls.o_blobs(O, a, 300)
        j = int(np.argmax(blobs["area"]))
        return {"src": a[None], "labels": labels[None], "blob": blobs[j:j + 1]}
    if op == "match_orb":
        rng = np.random.default_rng(16)
        sets = [L.desc_sets(rng, n1, n2) for n1, n2 in ((120, 90), (7, 0), (130, 61))][:n]
        k1, k2 = np.zeros((n, g["s1"]), L.KP_DTYPE), np.zeros((n, g["s2"]), L.KP_DTYPE)
        for i, (a, b) in enumerate(sets):
            k1[i, :len(a)], k2[i, :len(b)] = a, b
        return {"kps1": k1, "n1": calls.counts([a for a, _ in sets]), "kps2": k2, "n2": calls.counts([b for _, b in sets])}
    seed = w + h + {"downsample": w // 2, "resize": g.get("dw", 0), "integral": n}.get(op, g.get("r", 0))
    fr = frames(w, h, n, seed)
    if op in ("histogram", "otsu"):
        fr[n - 1] = np.random.default_rng(3).integers(0, 256, (h, w), dtype=np.uint8) // 64 * 64   # four bins only
    if op in ("fast", "orb"):
        fr[2] = L.natural_like(w, h, 99)                 # corners in every frame
        rng = np.random.default_rng(w)
        stale = np.zeros_like(fr) if op == "orb" else \
            (rng.integers(0, 256, fr.shape) * (rng.random(fr.shape) < 0.02)).astype(np.uint8)
        return {"src": fr, "score": stale}
    if op == "threshold_each":
        return {"src": fr, "thresh": np.array([100, 0, 250, 37, 255][:n], np.uint8)}
    if op == "match_template":
        return {"src": fr, "tmpl": np.ascontiguousarray(fr[1, 10:10 + g["th"], 20:20 + g["tw"]])}
    if op == "perspective" and g["per_frame"]:
        return {"src": fr, "corners": np.random.default_rng(5).integers(0, 140, (n, 4, 2)).astype(np.uint32)}
    return {"src": fr}


def run_row(lib, O, op, p):
    """the row's call with each buffer in a Region at the row's byte offset for it: every output against the oracle,
    every input unchanged, the bytes around each view untouched -> the launched kernels"""
    from grayskull_b200 import _lib
    sym, implicit = OPS[op]
    g = dict(implicit, **p)
    if op == "lbp":
        g["cascade"] = _cascade(p.get("cascade", "frontalface"))
    sp, ins, n = calls.spec(sym, g), row_inputs(O, op, g), g["n"]
    bufs = [(b, calls.flat(x, 1 if b in sp.shared else n)) for b, x in ins.items()]
    bufs += [(b, n * sum(per if isinstance(per, list) else [per])) for b, per in sp.outs.items() if b not in ins]
    R = {b: Region(x, g.get(b, 0), seed=k) if isinstance(x, int) else Region(x.size, g.get(b, 0), x, k)
         for k, (b, x) in enumerate(bufs, 1)}
    before = {b: calls.unflat(R[b].before(), per, n) for b, per in sp.outs.items() if b not in ins}
    rc, seen = traced(lambda: sp.call({b: r.ptr for b, r in R.items()}, n, stream()))
    _lib.check(rc, "dispatch row")
    want = sp.expect(ins, before)
    for b, r in R.items():
        got, exp = r.read(b), calls.flat(want[b], n) if b in want else dict(bufs)[b]
        assert np.array_equal(got, exp), "%s: byte %d of %d differs" % (b, int(np.argmax(got != exp)), got.size)
    if op in ("fast", "orb", "orb_pyramid"):
        assert want["counts"].sum() > 0 or g["t"] > 255
    if op == "lbp":
        assert want["counts"].sum() > 0
    if op == "find_best_match":
        px = g["w"] * g["h"]
        assert tuple(want["best"][1]) == (0, 0) and tuple(want["best"][2]) == ((px - 1) % g["w"], (px - 1) // g["w"])
    return seen


def test_every_row_has_a_runner():
    assert {op for op, _, _ in ROWS} <= set(OPS)


@pytest.mark.gpu
@pytest.mark.parametrize("op,kernels,p", [pytest.param(op, k, p, id=row_id(op, p)) for op, k, p in ROWS])
def test_dispatch_row(lib, O, witness, op, kernels, p):
    witnessed(witness, lambda: run_row(lib, O, op, p), kernels, row_id(op, p))
