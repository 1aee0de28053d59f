"""ctypes binding of libgrayskull_homography.so (include/grayskull_homography.h) and its calls on torch CUDA tensors:
a RANSAC homography per frame from its ORB matches, and the template's outline in the scene.  The inputs are the
tensors pyramid.orb_pyramid_batch and api.match_orb_batch return; the corners go to api.perspective_correct_batch and
the inlier records to draw.draw_matches_batch as they are.  Every call runs on torch's current stream.  There is no
fallback: if the library is missing this raises."""
import ctypes as C
import os

from ._lib import HERE

LIB_PATH = os.path.join(HERE, "libgrayskull_homography.so")

_u, _p = C.c_uint, C.c_void_p

# name -> (restype, argtypes); the CPU test suite checks this table against include/grayskull_homography.h
SIGNATURES = {
    "gs_b200_find_homography_batch": (C.c_int, [_p, _p, _u, _p, _p, _u, _p, _p, _u, _u, _u, C.c_ulonglong, C.c_double,
                                                _p, _p, _p, _p]),
    "gs_b200_homography_quads_batch": (C.c_int, [_p, _p, _u, _u, _u, _u, _u, _u, _p, _p, _p]),
    "gs_b200_homography_last_error": (C.c_char_p, []),
}

_lib = None


def lib():
    """Load the companion C ABI."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError("libgrayskull_homography.so is not built: run `python -m grayskull_b200.build` "
                               "(or __graft_entry__.build())")
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)
            fn.restype, fn.argtypes = res, args
        _lib = handle
    return _lib


def check(rc, what=""):
    if rc:
        raise RuntimeError("grayskull_homography %s failed: %s" % (what, lib().gs_b200_homography_last_error().decode()))


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _list(t, n, words):
    """an (n, stride, words) int32 CUDA list -> its stride"""
    import torch
    assert t.is_cuda and t.dtype == torch.int32 and t.is_contiguous() and t.dim() == 3
    assert t.shape[0] == n and t.shape[2] == words
    return t.shape[1]


def _counts(t, n):
    import torch
    assert t.is_cuda and t.dtype == torch.int32 and t.is_contiguous() and t.numel() == n
    return C.c_void_p(t.data_ptr())


def find_homography_batch(kps1, counts1, kps2, counts2, matches, mcounts, hypotheses=1024, seed=0, threshold=3.0):
    """kps1 (n, stride1, 12) and kps2 (n, stride2, 12) int32 keypoint lists with their counts (n,) int32 -- frame f's
    template and scene keypoints --, matches (n, mstride, 3) and mcounts (n,) int32 as api.match_orb_batch returns
    them -> (H (n, 3, 3) float64, inliers (n,) int32, inlier_matches (n, mstride, 3) int32): frame f's homography from
    template to scene (all zero when none was found), its inlier count and its inlier records in record order (slots
    past the count are zero)."""
    import torch
    n = matches.shape[0]
    s1, s2, ms = _list(kps1, n, 12), _list(kps2, n, 12), _list(matches, n, 3)
    H = torch.empty((n, 3, 3), dtype=torch.float64, device=matches.device)
    inliers = torch.empty((n,), dtype=torch.int32, device=matches.device)
    inlier_matches = torch.zeros((n, ms, 3), dtype=torch.int32, device=matches.device)
    check(lib().gs_b200_find_homography_batch(C.c_void_p(kps1.data_ptr()), _counts(counts1, n), s1,
                                              C.c_void_p(kps2.data_ptr()), _counts(counts2, n), s2,
                                              C.c_void_p(matches.data_ptr()), _counts(mcounts, n), ms, n, hypotheses,
                                              seed, threshold, C.c_void_p(H.data_ptr()),
                                              C.c_void_p(inliers.data_ptr()), C.c_void_p(inlier_matches.data_ptr()),
                                              _stream()), "find_homography_batch")
    return H, inliers, inlier_matches


def homography_quads_batch(H, inliers, tw, th, sw, sh, min_inliers=10):
    """H (n, 3, 3) float64 and inliers (n,) int32 as find_homography_batch returns them, a tw x th template and sw x sh
    frames -> (corners (n, 4, 2) int32: top-left, top-right, bottom-right, bottom-left, as
    api.perspective_correct_batch takes them; found (n,) uint8)."""
    import torch
    assert H.is_cuda and H.dtype == torch.float64 and H.is_contiguous() and H.dim() == 3 and H.shape[1:] == (3, 3)
    n = H.shape[0]
    corners = torch.empty((n, 4, 2), dtype=torch.int32, device=H.device)
    found = torch.empty((n,), dtype=torch.uint8, device=H.device)
    check(lib().gs_b200_homography_quads_batch(C.c_void_p(H.data_ptr()), _counts(inliers, n), n, min_inliers, tw, th,
                                               sw, sh, C.c_void_p(corners.data_ptr()), C.c_void_p(found.data_ptr()),
                                               _stream()), "homography_quads_batch")
    return corners, found
