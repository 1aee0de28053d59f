"""ctypes binding of libgrayskull_corners.so (include/grayskull_corners.h) and its calls on torch CUDA tensors: the
largest-blob pick of the reference's document scanner and wasm demo, and gs_blob_corners for every record of a frame
batch.  The blob inputs are the tensors api.blobs_batch returns.  Every call runs on torch's current stream.  There is
no fallback: if the library is missing this raises."""
import ctypes as C
import os

from ._lib import HERE

LIB_PATH = os.path.join(HERE, "libgrayskull_corners.so")

_u, _p = C.c_uint, C.c_void_p

# name -> (restype, argtypes); the CPU test suite checks this table against include/grayskull_corners.h
SIGNATURES = {
    "gs_b200_largest_blob_batch": (C.c_int, [_p, _p, _u, _u, _u, _p, _p, _p]),
    "gs_b200_blob_corners_batch": (C.c_int, [_p, _u, _u, _u, _p, _p, _p, _u, _p, _p]),
    "gs_b200_corners_last_error": (C.c_char_p, []),
}

_lib = None


def lib():
    """Load the companion C ABI."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError("libgrayskull_corners.so is not built: run `python -m grayskull_b200.build` "
                               "(or __graft_entry__.build())")
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)
            fn.restype, fn.argtypes = res, args
        _lib = handle
    return _lib


def check(rc, what=""):
    if rc:
        raise RuntimeError("grayskull_corners %s failed: %s" % (what, lib().gs_b200_corners_last_error().decode()))


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _counts(c, n):
    import torch
    if c is None:
        return None
    assert c.is_cuda and c.dtype == torch.int32 and c.is_contiguous() and c.numel() == n
    return C.c_void_p(c.data_ptr())


def _blobs(blobs):
    import torch
    assert blobs.is_cuda and blobs.dtype == torch.int32 and blobs.is_contiguous() and blobs.dim() == 3
    assert blobs.shape[2] == 8
    return blobs.shape[0], blobs.shape[1]


def largest_blob_batch(blobs, counts=None, min_area=0):
    """each frame's largest record (the first on ties) of blobs (n, stride, 8) int32 and counts (n,) int32 or None, as
    api.blobs_batch returns them -> (pick (n, 1, 8) int32, pcount (n,) int32): a list with stride 1 whose frame f holds
    one record when frame f has one of area >= min_area, none otherwise.  A frame without records picks gs_blobs'
    initial record {0, 0, {UINT_MAX, UINT_MAX, 0, 0}, {0, 0}}."""
    import torch
    n, stride = _blobs(blobs)
    pick = torch.empty((n, 1, 8), dtype=torch.int32, device=blobs.device)
    pcount = torch.empty((n,), dtype=torch.int32, device=blobs.device)
    check(lib().gs_b200_largest_blob_batch(C.c_void_p(blobs.data_ptr()), _counts(counts, n), stride, n, min_area,
                                           C.c_void_p(pick.data_ptr()), C.c_void_p(pcount.data_ptr()), _stream()),
          "largest_blob_batch")
    return pick, pcount


def blob_corners_batch(img, labels, blobs, counts=None):
    """gs_blob_corners for frame f's records k < min(counts[f], stride): img (n, h, w) uint8, labels (n, h, w) int16,
    blobs (n, stride, 8) int32, counts (n,) int32 or None (all `stride`) -> (n, stride, 4, 2) int32 points in tl, tr,
    br, bl order; zeros for the records past a frame's count"""
    import torch
    assert img.is_cuda and img.dtype == torch.uint8 and img.dim() == 3 and img.is_contiguous()
    n, h, w = img.shape
    assert labels.is_cuda and labels.dtype == torch.int16 and labels.shape == img.shape and labels.is_contiguous()
    bn, stride = _blobs(blobs)
    assert bn == n
    corners = torch.zeros((n, stride, 4, 2), dtype=torch.int32, device=img.device)
    check(lib().gs_b200_blob_corners_batch(C.c_void_p(img.data_ptr()), w, h, n, C.c_void_p(labels.data_ptr()),
                                           C.c_void_p(blobs.data_ptr()), _counts(counts, n), stride,
                                           C.c_void_p(corners.data_ptr()), _stream()), "blob_corners_batch")
    return corners
