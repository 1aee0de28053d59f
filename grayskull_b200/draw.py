"""ctypes binding of libgrayskull_draw.so (include/grayskull_draw.h) and its calls on torch CUDA tensors: the reference
CLI's annotated pictures (its blobs, keypoints, faces and orb verbs) drawn onto frame batches on the device.  The list
inputs are the tensors api.blobs_batch, api.fast_batch, api.lbp_detect_batch and api.match_orb_batch return.  Every call
runs on torch's current stream.  There is no fallback: if the library is missing this raises."""
import ctypes as C
import os

from ._lib import HERE

LIB_PATH = os.path.join(HERE, "libgrayskull_draw.so")

_u, _p = C.c_uint, C.c_void_p

# name -> (restype, argtypes); the CPU test suite checks this table against include/grayskull_draw.h
SIGNATURES = {
    "gs_b200_draw_blobs_batch": (C.c_int, [_p, _p, _u, _u, _u, _p, _p, _u, _p]),
    "gs_b200_draw_keypoints_batch": (C.c_int, [_p, _p, _u, _u, _u, _p, _p, _u, _u, _p]),
    "gs_b200_draw_rects_batch": (C.c_int, [_p, _p, _u, _u, _u, _p, _p, _u, _p]),
    "gs_b200_draw_matches_batch": (C.c_int, [_p, _p, _u, _u, _u, _p, _u, _u, _p, _u, _p, _u, _p, _p, _u, _u, _p]),
    "gs_b200_draw_last_error": (C.c_char_p, []),
}

_lib = None


def lib():
    """Load the companion C ABI."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError("libgrayskull_draw.so is not built: run `python -m grayskull_b200.build` "
                               "(or __graft_entry__.build())")
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)
            fn.restype, fn.argtypes = res, args
        _lib = handle
    return _lib


def check(rc, what=""):
    if rc:
        raise RuntimeError("grayskull_draw %s failed: %s" % (what, lib().gs_b200_draw_last_error().decode()))


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _frames(src):
    import torch
    assert src.is_cuda and src.dtype == torch.uint8 and src.dim() == 3 and src.is_contiguous()
    return src.shape


def _list(t, n, words):
    """a (n, stride, words) int32 device list and its stride"""
    import torch
    assert t.is_cuda and t.dtype == torch.int32 and t.is_contiguous() and t.dim() == 3
    assert t.shape[0] == n and t.shape[2] == words
    return C.c_void_p(t.data_ptr()), t.shape[1]


def _counts(c, n):
    import torch
    assert c.is_cuda and c.dtype == torch.int32 and c.is_contiguous() and c.numel() == n
    return C.c_void_p(c.data_ptr())


def _same_size(fn, what, src, lst, counts, words, out, *extra):
    import torch
    n, h, w = _frames(src)
    lp, stride = _list(lst, n, words)
    out = torch.empty_like(src) if out is None else out
    assert out.shape == src.shape and out.dtype == torch.uint8 and out.is_contiguous()
    check(getattr(lib(), fn)(C.c_void_p(out.data_ptr()), C.c_void_p(src.data_ptr()), w, h, n, lp, _counts(counts, n),
                             stride, *extra, _stream()), what)
    return out


def draw_blobs_batch(src, blobs, counts, out=None):
    """the blobs verb's picture: src (n, h, w) uint8; blobs (n, stride, 8) int32 and counts (n,) int32 as
    api.blobs_batch returns them -> (n, h, w).  out may be src."""
    return _same_size("gs_b200_draw_blobs_batch", "draw_blobs_batch", src, blobs, counts, 8, out)


def draw_keypoints_batch(src, kps, counts, top, out=None):
    """the keypoints verb's picture: crosses at the `top` strongest keypoints (stable order) of kps (n, stride, 12)
    int32 and counts (n,) int32, as api.fast_batch returns them -> (n, h, w).  out may be src."""
    return _same_size("gs_b200_draw_keypoints_batch", "draw_keypoints_batch", src, kps, counts, 12, out, top)


def draw_rects_batch(src, rects, counts, out=None):
    """the faces verb's picture: each rect's outline, rects (n, stride, 4) int32 and counts (n,) int32 as
    api.lbp_detect_batch returns them -> (n, h, w).  out may be src."""
    return _same_size("gs_b200_draw_rects_batch", "draw_rects_batch", src, rects, counts, 4, out)


def draw_matches_batch(src, tmpl, kps1, kps2, matches, counts, top=15, out=None):
    """the orb verb's picture: src (n, h, w) and tmpl (th, tw) uint8; kps1 (n or 1, stride1, 12) int32 -- one list
    is shared by every frame --, kps2 (n, stride2, 12), matches (n, mstride, 3) and counts (n,) int32 as
    api.match_orb_batch takes and returns them -> (n, max(th, h), tw + w)."""
    import torch
    n, h, w = _frames(src)
    assert tmpl.is_cuda and tmpl.dtype == torch.uint8 and tmpl.dim() == 2 and tmpl.is_contiguous()
    th, tw = tmpl.shape
    assert kps1.is_cuda and kps1.dtype == torch.int32 and kps1.is_contiguous() and kps1.dim() == 3
    assert kps1.shape[0] in (1, n) and kps1.shape[2] == 12
    stride1 = 0 if kps1.shape[0] == 1 else kps1.shape[1]
    k2, stride2 = _list(kps2, n, 12)
    mp, mstride = _list(matches, n, 3)
    shape = (n, max(th, h), tw + w)
    out = torch.empty(shape, dtype=torch.uint8, device=src.device) if out is None else out
    assert tuple(out.shape) == shape and out.dtype == torch.uint8 and out.is_contiguous()
    check(lib().gs_b200_draw_matches_batch(C.c_void_p(out.data_ptr()), C.c_void_p(src.data_ptr()), w, h, n,
                                           C.c_void_p(tmpl.data_ptr()), tw, th, C.c_void_p(kps1.data_ptr()), stride1,
                                           k2, stride2, mp, _counts(counts, n), mstride, top, _stream()),
          "draw_matches_batch")
    return out
