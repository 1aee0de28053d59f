"""ctypes binding of libgrayskull_color.so (include/grayskull_color.h) and its calls on torch CUDA tensors: the wasm
demo's RGB(A) -> gray and gray -> RGBA conversions over frame batches, bit-exact.  Every call runs on torch's current
stream.  There is no fallback: if the library is missing this raises."""
import ctypes as C
import os

from ._lib import HERE

LIB_PATH = os.path.join(HERE, "libgrayskull_color.so")

_u, _p = C.c_uint, C.c_void_p

# name -> (restype, argtypes); the CPU test suite checks this table against include/grayskull_color.h
SIGNATURES = {
    "gs_b200_rgb_to_gray_batch": (C.c_int, [_p, _p, _u, _u, _u, _u, _p]),
    "gs_b200_gray_to_rgba_batch": (C.c_int, [_p, _p, _u, _u, _u, _p]),
    "gs_b200_color_last_error": (C.c_char_p, []),
}

_lib = None


def lib():
    """Load the companion C ABI."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError("libgrayskull_color.so is not built: run `python -m grayskull_b200.build` "
                               "(or __graft_entry__.build())")
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)
            fn.restype, fn.argtypes = res, args
        _lib = handle
    return _lib


def check(rc, what=""):
    if rc:
        raise RuntimeError("grayskull_color %s failed: %s" % (what, lib().gs_b200_color_last_error().decode()))


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _out(out, shape, like):
    import torch
    if out is None:
        return torch.empty(shape, dtype=torch.uint8, device=like.device)
    assert out.is_cuda and out.dtype == torch.uint8 and out.is_contiguous() and tuple(out.shape) == shape
    return out


def rgb_to_gray_batch(src, out=None):
    """the demo's rgbaToGray: src (n, h, w, 3) RGB or (n, h, w, 4) RGBA uint8, contiguous, on the device ->
    (n, h, w) uint8 gray (written into `out` when given)"""
    import torch
    assert src.is_cuda and src.dtype == torch.uint8 and src.dim() == 4 and src.is_contiguous()
    n, h, w, c = src.shape
    assert c in (3, 4), "channels must be 3 (RGB) or 4 (RGBA)"
    out = _out(out, (n, h, w), src)
    check(lib().gs_b200_rgb_to_gray_batch(C.c_void_p(out.data_ptr()), C.c_void_p(src.data_ptr()), w, h, n, c,
                                          _stream()), "rgb_to_gray_batch")
    return out


def gray_to_rgba_batch(src, out=None):
    """the demo's grayToRgba: src (n, h, w) uint8 gray, contiguous, on the device -> (n, h, w, 4) uint8 RGBA,
    (g, g, g, 255) per pixel (written into `out` when given)"""
    import torch
    assert src.is_cuda and src.dtype == torch.uint8 and src.dim() == 3 and src.is_contiguous()
    n, h, w = src.shape
    out = _out(out, (n, h, w, 4), src)
    check(lib().gs_b200_gray_to_rgba_batch(C.c_void_p(out.data_ptr()), C.c_void_p(src.data_ptr()), w, h, n,
                                           _stream()), "gray_to_rgba_batch")
    return out
