"""ctypes binding of libgrayskull_group.so (include/grayskull_group.h) and its call on torch CUDA tensors: each frame's
LBP detections grouped into neighbour-counted boxes.  The rect inputs are the tensors api.lbp_detect_batch returns, and
the outputs have the same layout, so draw.draw_rects_batch and roi take them as they are.  Every call runs on torch's
current stream.  There is no fallback: if the library is missing this raises."""
import ctypes as C
import os

from ._lib import HERE

LIB_PATH = os.path.join(HERE, "libgrayskull_group.so")

_u, _p = C.c_uint, C.c_void_p

# name -> (restype, argtypes); the CPU test suite checks this table against include/grayskull_group.h
SIGNATURES = {
    "gs_b200_group_rects_work_bytes": (C.c_size_t, [_u, _u]),
    "gs_b200_group_rects_batch": (C.c_int, [_p, _p, _u, _u, _u, C.c_double, _p, _p, _p, _u, _p, C.c_size_t, _p]),
    "gs_b200_group_last_error": (C.c_char_p, []),
}

_lib = None


def lib():
    """Load the companion C ABI."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError("libgrayskull_group.so is not built: run `python -m grayskull_b200.build` "
                               "(or __graft_entry__.build())")
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)
            fn.restype, fn.argtypes = res, args
        _lib = handle
    return _lib


def check(rc, what=""):
    if rc:
        raise RuntimeError("grayskull_group %s failed: %s" % (what, lib().gs_b200_group_last_error().decode()))


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def work_bytes(stride, n):
    """bytes of workspace that group_rects_batch needs to run n frames of `stride` records at once"""
    return int(lib().gs_b200_group_rects_work_bytes(stride, n))


def group_rects_batch(rects, counts=None, min_neighbors=3, eps=0.2, out_stride=None, work=None):
    """rects (n, stride, 4) int32 and counts (n,) int32 or None (all `stride`), as api.lbp_detect_batch returns them ->
    (groups (n, out_stride, 4) int32, weights (n, out_stride) int32, counts (n,) int32): the surviving groups of each
    frame in the order of their first record, and each one's number of records.  out_stride defaults to stride.  work
    (a uint8 CUDA tensor) defaults to one allocated for the whole batch; a smaller one runs the frames in chunks."""
    import torch
    assert rects.is_cuda and rects.dtype == torch.int32 and rects.is_contiguous() and rects.dim() == 3
    assert rects.shape[2] == 4
    n, stride = rects.shape[0], rects.shape[1]
    if counts is not None:
        assert counts.is_cuda and counts.dtype == torch.int32 and counts.is_contiguous() and counts.numel() == n
    out_stride = stride if out_stride is None else out_stride
    if work is None:
        work = torch.empty(work_bytes(stride, n), dtype=torch.uint8, device=rects.device)
    assert work.is_cuda and work.dtype == torch.uint8 and work.is_contiguous()
    groups = torch.zeros((n, out_stride, 4), dtype=torch.int32, device=rects.device)
    weights = torch.zeros((n, out_stride), dtype=torch.int32, device=rects.device)
    out_counts = torch.empty((n,), dtype=torch.int32, device=rects.device)
    check(lib().gs_b200_group_rects_batch(C.c_void_p(rects.data_ptr()),
                                          None if counts is None else C.c_void_p(counts.data_ptr()), stride, n,
                                          min_neighbors, eps, C.c_void_p(groups.data_ptr()),
                                          C.c_void_p(weights.data_ptr()), C.c_void_p(out_counts.data_ptr()),
                                          out_stride, C.c_void_p(work.data_ptr()), work.numel(), _stream()),
          "group_rects_batch")
    return groups, weights, out_counts
