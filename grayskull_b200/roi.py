"""Regions of interest cut out of frame batches and resized on the device (include/grayskull_b200_roi.h), on torch
CUDA tensors: bit-exact with the reference's gs_crop followed by gs_resize_nn (NEAREST) or gs_resize (BILINEAR)."""
import ctypes as C

from ._lib import Rect, check, lib

NEAREST, BILINEAR = 0, 1   # GS_B200_NEAREST, GS_B200_BILINEAR


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _frames(src):
    import torch
    assert src.is_cuda and src.dtype == torch.uint8 and src.dim() == 3 and src.is_contiguous()
    return src.shape


def crop_resize_batch(src, roi, dw, dh, mode=NEAREST, out=None):
    """src: (n, h, w) uint8; roi: (x, y, w, h), the same region of every frame -> (n, dh, dw)"""
    import torch
    n, sh, sw = _frames(src)
    out = torch.empty((n, dh, dw), dtype=torch.uint8, device=src.device) if out is None else out
    check(lib().gs_b200_crop_resize_batch(C.c_void_p(out.data_ptr()), dw, dh, C.c_void_p(src.data_ptr()), sw, sh, n,
                                          Rect(*roi), mode, _stream()), "crop_resize_batch")
    return out


def rois_resize_batch(src, rects, counts, dw, dh, mode=NEAREST, out=None):
    """src: (n, h, w) uint8; rects: (n, max_rects, 4) int32 device storage of gs_rect (x, y, w, h), as
    api.lbp_detect_batch returns them; counts: (n,) int32 on the device, or None for all max_rects
    -> (n, max_rects, dh, dw).  Slots at or past a frame's count are left as `out` holds them (uninitialised when
    out is None); a region gs_crop would reject gives a zero slot."""
    import torch
    n, sh, sw = _frames(src)
    assert rects.is_cuda and rects.dtype == torch.int32 and rects.is_contiguous() and rects.dim() == 3
    assert rects.shape[0] == n and rects.shape[2] == 4
    max_rects = rects.shape[1]
    if counts is not None:
        assert counts.is_cuda and counts.dtype == torch.int32 and counts.is_contiguous() and counts.numel() == n
    out = torch.empty((n, max_rects, dh, dw), dtype=torch.uint8, device=src.device) if out is None else out
    check(lib().gs_b200_rois_resize_batch(C.c_void_p(out.data_ptr()), dw, dh, C.c_void_p(src.data_ptr()), sw, sh, n,
                                          C.c_void_p(rects.data_ptr()),
                                          None if counts is None else C.c_void_p(counts.data_ptr()), max_rects, mode,
                                          _stream()), "rois_resize_batch")
    return out
