"""ctypes binding of libgrayskull_contour.so (include/grayskull_contour.h) and its calls on torch CUDA tensors:
gs_trace_contour over frame batches on the device, and the wasm demo's contour start for blob records.  The blob inputs
are the tensors api.blobs_batch returns.  Every call runs on torch's current stream.  There is no fallback: if the
library is missing this raises."""
import ctypes as C
import os

import numpy as np

from ._lib import HERE

LIB_PATH = os.path.join(HERE, "libgrayskull_contour.so")

# struct gs_contour: box (x, y, w, h), start (x, y), length
CONTOUR_DTYPE = np.dtype([("bx", "<u4"), ("by", "<u4"), ("bw", "<u4"), ("bh", "<u4"), ("sx", "<u4"), ("sy", "<u4"),
                          ("length", "<u4")])
assert CONTOUR_DTYPE.itemsize == 28

# the end of each walk (GS_CONTOUR_RETURNED / _OPEN / _CYCLE)
RETURNED, OPEN, CYCLE = 0, 1, 2

_u, _p = C.c_uint, C.c_void_p

# name -> (restype, argtypes); the CPU test suite checks this table against include/grayskull_contour.h
SIGNATURES = {
    "gs_b200_trace_contours_batch": (C.c_int, [_p, _p, _u, _u, _u, _p, _p, _u, _p, _p, C.c_size_t, _p]),
    "gs_b200_trace_contours_work_bytes": (C.c_size_t, [_u, _u, _u]),
    "gs_b200_blob_contour_starts_batch": (C.c_int, [_p, _u, _u, _u, _p, _p, _u, _p, _p]),
    "gs_b200_contour_last_error": (C.c_char_p, []),
}

_lib = None


def lib():
    """Load the companion C ABI."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError("libgrayskull_contour.so is not built: run `python -m grayskull_b200.build` "
                               "(or __graft_entry__.build())")
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)
            fn.restype, fn.argtypes = res, args
        _lib = handle
    return _lib


def check(rc, what=""):
    if rc:
        raise RuntimeError("grayskull_contour %s failed: %s" % (what, lib().gs_b200_contour_last_error().decode()))


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _counts(c, n):
    import torch
    if c is None:
        return None
    assert c.is_cuda and c.dtype == torch.int32 and c.is_contiguous() and c.numel() == n
    return C.c_void_p(c.data_ptr())


def trace_contours_batch(img, starts, counts=None, visited=None):
    """gs_trace_contour for frame f's records k < min(counts[f], stride), in order k against frame f's visited.
    img (n, h, w) uint8; starts (n, stride, 2) int32 (x, y), or (n, stride, 7) int32 contour records whose start is
    used; counts (n,) int32 or None (all `stride`); visited (n, h, w) uint8, updated in place, or None (zeros).
    -> (contours (n, stride, 7) int32 as CONTOUR_DTYPE words, ends (n, stride) uint8, visited).  Records past a frame's
    count keep their start and zeros, and their ends stay 255."""
    import torch
    assert img.is_cuda and img.dtype == torch.uint8 and img.dim() == 3 and img.is_contiguous()
    n, h, w = img.shape
    assert starts.is_cuda and starts.dtype == torch.int32 and starts.dim() == 3 and starts.shape[0] == n
    assert starts.shape[2] in (2, 7)
    stride = starts.shape[1]
    contours = torch.zeros((n, stride, 7), dtype=torch.int32, device=img.device)
    contours[:, :, 4:6] = starts if starts.shape[2] == 2 else starts[:, :, 4:6]
    ends = torch.full((n, stride), 255, dtype=torch.uint8, device=img.device)
    if visited is None:
        visited = torch.zeros_like(img)
    assert visited.shape == img.shape and visited.dtype == torch.uint8 and visited.is_contiguous()
    nbytes = lib().gs_b200_trace_contours_work_bytes(w, h, n)
    work = torch.empty(nbytes, dtype=torch.uint8, device=img.device)
    check(lib().gs_b200_trace_contours_batch(C.c_void_p(img.data_ptr()), C.c_void_p(visited.data_ptr()), w, h, n,
                                             C.c_void_p(contours.data_ptr()), _counts(counts, n), stride,
                                             C.c_void_p(ends.data_ptr()), C.c_void_p(work.data_ptr()), nbytes,
                                             _stream()), "trace_contours_batch")
    return contours, ends, visited


def blob_contour_starts_batch(labels, blobs, counts):
    """the wasm demo's contour start for every blob record: labels (n, h, w) int16, blobs (n, stride, 8) int32 and
    counts (n,) int32 as api.blobs_batch returns them -> (n, stride, 7) int32 contour records, start set for the
    records each frame uses, zeros elsewhere"""
    import torch
    assert labels.is_cuda and labels.dtype == torch.int16 and labels.dim() == 3 and labels.is_contiguous()
    n, h, w = labels.shape
    assert blobs.is_cuda and blobs.dtype == torch.int32 and blobs.is_contiguous() and blobs.dim() == 3
    assert blobs.shape[0] == n and blobs.shape[2] == 8
    stride = blobs.shape[1]
    contours = torch.zeros((n, stride, 7), dtype=torch.int32, device=labels.device)
    check(lib().gs_b200_blob_contour_starts_batch(C.c_void_p(labels.data_ptr()), w, h, n, C.c_void_p(blobs.data_ptr()),
                                                  _counts(counts, n), stride, C.c_void_p(contours.data_ptr()),
                                                  _stream()), "blob_contour_starts_batch")
    return contours


def to_numpy(contours):
    """(n, stride, 7) int32 contour words -> (n, stride) CONTOUR_DTYPE on the host"""
    return contours.cpu().numpy().view(np.uint32).view(CONTOUR_DTYPE).reshape(contours.shape[:2])
