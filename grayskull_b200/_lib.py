"""ctypes binding of libgrayskull_b200.so -- every symbol declared in include/grayskull.h,
include/grayskull_b200.h, include/grayskull_b200_roi.h and include/grayskull_b200_pyramid.h.  There is no fallback: if
the library is missing this raises."""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libgrayskull_b200.so")


class Image(C.Structure):  # struct gs_image, reference grayskull.h:14-17
    _fields_ = [("w", C.c_uint), ("h", C.c_uint), ("data", C.c_void_p)]


class Point(C.Structure):  # struct gs_point, reference grayskull.h:23-25
    _fields_ = [("x", C.c_uint), ("y", C.c_uint)]


class Keypoint(C.Structure):  # struct gs_keypoint, reference grayskull.h:42-47
    _fields_ = [("x", C.c_uint), ("y", C.c_uint), ("response", C.c_uint), ("angle", C.c_float),
                ("descriptor", C.c_uint32 * 8)]


class Rect(C.Structure):  # struct gs_rect, reference grayskull.h:19-21
    _fields_ = [("x", C.c_uint), ("y", C.c_uint), ("w", C.c_uint), ("h", C.c_uint)]


class Cascade(C.Structure):  # struct gs_lbp_cascade, reference grayskull.h:54-64
    _fields_ = [
        ("window_w", C.c_uint16), ("window_h", C.c_uint16),
        ("nfeatures", C.c_uint16), ("nweaks", C.c_uint16), ("nstages", C.c_uint16),
        ("features", C.c_void_p), ("weak_feature_idx", C.c_void_p),
        ("weak_left_val", C.c_void_p), ("weak_right_val", C.c_void_p),
        ("weak_subset_offset", C.c_void_p), ("weak_num_subsets", C.c_void_p),
        ("subsets", C.c_void_p), ("stage_weak_start", C.c_void_p), ("stage_nweaks", C.c_void_p),
        ("stage_threshold", C.c_void_p),
    ]


KP_DTYPE = np.dtype([("x", "<u4"), ("y", "<u4"), ("response", "<u4"), ("angle", "<f4"),
                     ("descriptor", "<u4", (8,))])
RECT_DTYPE = np.dtype([("x", "<u4"), ("y", "<u4"), ("w", "<u4"), ("h", "<u4")])
MATCH_DTYPE = np.dtype([("idx1", "<u4"), ("idx2", "<u4"), ("distance", "<u4")])
# struct gs_blob (reference grayskull.h:29-34): u16 label + 2 padding bytes, area, box, centroid
BLOB_DTYPE = np.dtype({"names": ["label", "area", "bx", "by", "bw", "bh", "cx", "cy"],
                       "formats": ["<u2", "<u4", "<u4", "<u4", "<u4", "<u4", "<u4", "<u4"],
                       "offsets": [0, 4, 8, 12, 16, 20, 24, 28], "itemsize": 32})

_u, _i, _f, _p, _sz = C.c_uint, C.c_int, C.c_float, C.c_void_p, C.c_size_t

# name -> (restype, argtypes); the CPU test suite checks this table against include/*.h
SIGNATURES = {
    # include/grayskull.h
    "gs_blur": (None, [Image, Image, _u]),
    "gs_sobel": (None, [Image, Image]),
    "gs_erode": (None, [Image, Image]),
    "gs_dilate": (None, [Image, Image]),
    "gs_adaptive_threshold": (None, [Image, Image, _u, _i]),
    "gs_resize": (None, [Image, Image]),
    "gs_downsample": (None, [Image, Image]),
    "gs_integral": (None, [Image, _p]),
    "gs_fast": (_u, [Image, Image, _p, _u, _u]),
    "gs_compute_orientation": (_f, [Image, _u, _u, _u]),
    "gs_brief_descriptor": (None, [Image, _p]),
    "gs_orb_extract": (_u, [Image, _p, _u, _u, _p]),
    "gs_match_orb": (_u, [_p, _u, _p, _u, _p, _u, _f]),
    "gs_filter": (None, [Image, Image, Image, _u]),
    "gs_match_template": (None, [Image, Image, Image]),
    "gs_find_best_match": (Point, [Image]),
    "gs_histogram": (None, [Image, _p]),
    "gs_otsu_threshold": (C.c_uint8, [Image]),
    "gs_threshold": (None, [Image, C.c_uint8]),
    "gs_blobs": (_u, [Image, _p, _p, _u]),
    "gs_blob_corners": (None, [Image, _p, _p, _p]),
    "gs_perspective_correct": (None, [Image, Image, _p]),
    "gs_lbp_window": (_u, [_p, _p, _u, _u, _i, _i, _f]),
    "gs_lbp_detect": (_u, [_p, _p, _u, _u, _p, _u, _f, _f, _f, _i]),
    # include/grayskull_b200.h
    "gs_b200_device_count": (_i, []),
    "gs_b200_set_device": (_i, [_i]),
    "gs_b200_last_error": (C.c_char_p, []),
    "gs_b200_version": (C.c_char_p, []),
    "gs_b200_uses_tma": (_i, [_u, _u, _p]),
    "gs_b200_force_generic": (None, [_i]),
    "gs_b200_launch_count": (C.c_ulonglong, []),
    "gs_b200_malloc": (_p, [_sz]),
    "gs_b200_free": (None, [_p]),
    "gs_b200_malloc_host": (_p, [_sz]),
    "gs_b200_free_host": (None, [_p]),
    "gs_b200_memcpy_h2d": (_i, [_p, _p, _sz, _p]),
    "gs_b200_memcpy_d2h": (_i, [_p, _p, _sz, _p]),
    "gs_b200_memset": (_i, [_p, _i, _sz, _p]),
    "gs_b200_stream_sync": (_i, [_p]),
    "gs_b200_alloc": (Image, [_u, _u]),
    "gs_b200_image_free": (None, [Image]),
    "gs_b200_blur_batch": (_i, [_p, _p, _u, _u, _u, _u, _p]),
    "gs_b200_adaptive_threshold_batch": (_i, [_p, _p, _u, _u, _u, _u, _i, _p]),
    "gs_b200_sobel_batch": (_i, [_p, _p, _u, _u, _u, _p]),
    "gs_b200_blur_sobel_batch": (_i, [_p, _p, _u, _u, _u, _u, _p]),
    "gs_b200_erode_batch": (_i, [_p, _p, _u, _u, _u, _p]),
    "gs_b200_dilate_batch": (_i, [_p, _p, _u, _u, _u, _p]),
    "gs_b200_erode_n_batch": (_i, [_p, _p, _u, _u, _u, _u, _p]),
    "gs_b200_dilate_n_batch": (_i, [_p, _p, _u, _u, _u, _u, _p]),
    "gs_b200_resize_batch": (_i, [_p, _u, _u, _p, _u, _u, _u, _p]),
    "gs_b200_downsample_batch": (_i, [_p, _p, _u, _u, _u, _p]),
    "gs_b200_integral_batch": (_i, [_p, _p, _u, _u, _u, _p]),
    "gs_b200_blobs_batch": (_i, [_p, _u, _u, _u, _p, _p, _p, _u, _p]),
    "gs_b200_blob_corners": (_i, [_p, _u, _u, _p, _p, _p, _p]),
    "gs_b200_perspective_correct_batch": (_i, [_p, _u, _u, _p, _u, _u, _u, _p, _i, _p]),
    "gs_b200_fast_batch": (_i, [_p, _u, _u, _u, _p, _p, _p, _u, _u, _p]),
    "gs_b200_orb_extract_batch": (_i, [_p, _u, _u, _u, _p, _p, _p, _u, _u, _p]),
    "gs_b200_set_trig_mode": (None, [_i]),
    "gs_b200_trig_selfcheck": (_i, []),
    "gs_b200_filter_batch": (_i, [_p, _p, _u, _u, _u, _p, _u, _u, _u, _p]),
    "gs_b200_match_template_batch": (_i, [_p, _p, _u, _u, _u, _p, _u, _u, _p]),
    "gs_b200_find_best_match_batch": (_i, [_p, _p, _u, _u, _u, _p]),
    "gs_b200_histogram_batch": (_i, [_p, _p, _u, _u, _u, _p]),
    "gs_b200_otsu_threshold_batch": (_i, [_p, _p, _p, _u, _u, _u, _p]),
    "gs_b200_threshold_batch": (_i, [_p, _u, _u, _u, _u, _p]),
    "gs_b200_threshold_each_batch": (_i, [_p, _u, _u, _u, _p, _i, _p]),
    "gs_b200_match_orb_batch": (_i, [_p, _p, _u, _p, _p, _u, _u, _p, _p, _u, _f, _p]),
    "gs_b200_lbp_detect_batch": (_i, [_p, _p, _u, _u, _u, _p, _p, _u, _f, _f, _f, _i, _p]),
    "gs_b200_lbp_window_count": (C.c_ulonglong, [_p, _u, _u, _f, _f, _f, _i]),
    # include/grayskull_b200_roi.h
    "gs_b200_crop_resize_batch": (_i, [_p, _u, _u, _p, _u, _u, _u, Rect, _i, _p]),
    "gs_b200_rois_resize_batch": (_i, [_p, _u, _u, _p, _u, _u, _u, _p, _p, _u, _i, _p]),
    # include/grayskull_b200_pyramid.h
    "gs_b200_orb_pyramid_levels": (_u, [_u, _u, _u]),
    "gs_b200_orb_pyramid_batch": (_i, [_p, _u, _u, _u, _u, _p, _p, _p, _p, _u, _u, _p]),
}

_lib = None


def lib():
    """Load the C ABI.  No CPU fallback: a missing library is an error."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError("libgrayskull_b200.so is not built: run `python -m grayskull_b200.build` "
                               "(or __graft_entry__.build())")
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)  # AttributeError if the symbol is missing
            fn.restype, fn.argtypes = res, args
        _lib = handle
    return _lib


def check(rc, what=""):
    if rc:
        raise RuntimeError("grayskull_b200 %s failed: %s" % (what, lib().gs_b200_last_error().decode()))


class HostCascade:
    """A struct gs_lbp_cascade on the host built from numpy tables (kept alive by this object)."""

    def __init__(self, arrays):
        a = self.arrays = {k: np.ascontiguousarray(v) for k, v in arrays.items()}
        self.struct = Cascade(int(a["window"][0]), int(a["window"][1]), len(a["features"]) // 4,
                              len(a["weak_feature_idx"]), len(a["stage_threshold"]),
                              a["features"].ctypes.data, a["weak_feature_idx"].ctypes.data,
                              a["weak_left_val"].ctypes.data, a["weak_right_val"].ctypes.data,
                              a["weak_subset_offset"].ctypes.data, a["weak_num_subsets"].ctypes.data,
                              a["subsets"].ctypes.data, a["stage_weak_start"].ctypes.data,
                              a["stage_nweaks"].ctypes.data, a["stage_threshold"].ctypes.data)

    @property
    def ptr(self):
        return C.addressof(self.struct)


def load_cascade(path=None):
    """The `frontalface` cascade fixture (data/frontalface.npz, exported from the reference's
    examples/nanomagick/frontalface.h by tools/gen_tables.py)."""
    path = path or os.path.join(HERE, "data", "frontalface.npz")
    z = np.load(path)
    return HostCascade({k: z[k] for k in z.files})
