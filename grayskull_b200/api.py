"""Host-side mirror of the reference interface.

Two layers, both thin wrappers over the C ABI (no arithmetic happens in Python):

* gs_<op>(...)  on numpy arrays: the reference's one-image, synchronous calls (grayskull.h);
                host pointers are staged by the C library.
* <op>_batch(...) on torch CUDA uint8 tensors of shape (n, h, w): device-resident, asynchronous
                on torch's current stream (include/grayskull_b200.h).
"""
import ctypes as C

import numpy as np

from ._lib import lib, check, Image, Point, KP_DTYPE, RECT_DTYPE, MATCH_DTYPE, BLOB_DTYPE


def _img(a):
    assert a.dtype == np.uint8 and a.ndim == 2 and a.flags.c_contiguous
    return Image(a.shape[1], a.shape[0], a.ctypes.data)


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


# ---------------------------------------------------------------- reference-style, numpy
def gs_blur(dst, src, radius):
    lib().gs_blur(_img(dst), _img(src), radius)


def gs_sobel(dst, src):
    lib().gs_sobel(_img(dst), _img(src))


def gs_erode(dst, src):
    lib().gs_erode(_img(dst), _img(src))


def gs_dilate(dst, src):
    lib().gs_dilate(_img(dst), _img(src))


def gs_adaptive_threshold(dst, src, radius, c):
    lib().gs_adaptive_threshold(_img(dst), _img(src), radius, c)


def gs_resize(dst, src):
    lib().gs_resize(_img(dst), _img(src))


def gs_downsample(dst, src):
    lib().gs_downsample(_img(dst), _img(src))


def gs_integral(src, ii):
    assert ii.dtype == np.uint32 and ii.shape == src.shape
    lib().gs_integral(_img(src), _vp(ii))


def gs_fast(img, scoremap, nkps, threshold):
    kps = np.zeros(nkps, KP_DTYPE)
    sm = _img(scoremap) if scoremap is not None else Image(0, 0, None)
    n = lib().gs_fast(_img(img), sm, _vp(kps), nkps, threshold)
    return kps[:n]


def gs_compute_orientation(img, x, y, r):
    return lib().gs_compute_orientation(_img(img), x, y, r)


def gs_brief_descriptor(img, kp):
    """kp: 1-element KP_DTYPE array (pt and angle in, descriptor out)"""
    lib().gs_brief_descriptor(_img(img), _vp(kp))


def gs_orb_extract(img, nkps, threshold, scoremap_buffer):
    kps = np.zeros(nkps, KP_DTYPE)
    n = lib().gs_orb_extract(_img(img), _vp(kps), nkps, threshold, _vp(scoremap_buffer))
    return kps[:n]


def gs_filter(dst, src, kernel, norm):
    """kernel: (kh, kw) int8 (or uint8 bit patterns) numpy array"""
    k = np.ascontiguousarray(kernel).view(np.uint8)
    lib().gs_filter(_img(dst), _img(src), _img(k), norm)
    return dst


def gs_match_template(img, tmpl):
    res = np.zeros((img.shape[0] - tmpl.shape[0] + 1, img.shape[1] - tmpl.shape[1] + 1), np.uint8)
    lib().gs_match_template(_img(img), _img(tmpl), _img(res))
    return res


def gs_find_best_match(result):
    p = lib().gs_find_best_match(_img(result))
    return p.x, p.y


def gs_histogram(img):
    hist = np.zeros(256, np.uint32)
    lib().gs_histogram(_img(img), _vp(hist))
    return hist


def gs_otsu_threshold(img):
    return int(lib().gs_otsu_threshold(_img(img)))


def gs_threshold(img, thresh):
    """in place, like the reference"""
    lib().gs_threshold(_img(img), thresh)
    return img


def gs_match_orb(kps1, kps2, max_matches, max_distance):
    """kps1, kps2: KP_DTYPE arrays -> MATCH_DTYPE array (reference gs_match_orb)"""
    m = np.zeros(max(max_matches, 1), MATCH_DTYPE)
    k2 = kps2 if len(kps2) else np.zeros(1, KP_DTYPE)
    n = lib().gs_match_orb(_vp(kps1), len(kps1), _vp(k2), len(kps2), _vp(m), max_matches, max_distance)
    return m[:n]


def gs_blobs(img, nblobs):
    """-> (labels (h, w) uint16, blobs BLOB_DTYPE[m])"""
    labels = np.zeros(img.shape, np.uint16)
    blobs = np.zeros(max(nblobs, 1), BLOB_DTYPE)
    m = lib().gs_blobs(_img(img), _vp(labels), _vp(blobs), nblobs)
    return labels, blobs[:m]


def gs_blob_corners(img, labels, blob):
    """blob: 1-element BLOB_DTYPE array -> (4, 2) uint32 corners tl, tr, br, bl"""
    c = np.zeros((4, 2), np.uint32)
    lib().gs_blob_corners(_img(img), _vp(labels), _vp(blob), _vp(c))
    return c


def gs_perspective_correct(dst, src, corners):
    c = np.ascontiguousarray(corners, np.uint32)
    lib().gs_perspective_correct(_img(dst), _img(src), _vp(c))
    return dst


def gs_lbp_window(cascade, ii, x, y, scale):
    return lib().gs_lbp_window(cascade.ptr, _vp(ii), ii.shape[1], ii.shape[0], x, y, scale)


def gs_lbp_detect(cascade, ii, max_rects, scale_factor, min_scale, max_scale, step):
    rects = np.zeros(max(max_rects, 1), RECT_DTYPE)
    n = lib().gs_lbp_detect(cascade.ptr, _vp(ii), ii.shape[1], ii.shape[0], _vp(rects), max_rects,
                            scale_factor, min_scale, max_scale, step)
    return rects[:n]


# ---------------------------------------------------------------- batched, torch CUDA tensors
def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _chk_frames(t):
    import torch
    assert t.is_cuda and t.dtype == torch.uint8 and t.dim() == 3 and t.is_contiguous()
    return t.shape[0], t.shape[1], t.shape[2]


def _p(t):
    return C.c_void_p(t.data_ptr())


def blur_batch(src, radius, out=None):
    import torch
    n, h, w = _chk_frames(src)
    out = torch.empty_like(src) if out is None else out
    check(lib().gs_b200_blur_batch(_p(out), _p(src), w, h, n, radius, _stream()), "blur_batch")
    return out


def adaptive_threshold_batch(src, radius, c, out=None):
    import torch
    n, h, w = _chk_frames(src)
    out = torch.empty_like(src) if out is None else out
    check(lib().gs_b200_adaptive_threshold_batch(_p(out), _p(src), w, h, n, radius, c, _stream()), "adaptive")
    return out


def sobel_batch(src, out=None):
    """`out` keeps its 1-px frame (reference semantics); a fresh output is zero-filled like gs_alloc."""
    import torch
    n, h, w = _chk_frames(src)
    out = torch.zeros_like(src) if out is None else out
    check(lib().gs_b200_sobel_batch(_p(out), _p(src), w, h, n, _stream()), "sobel_batch")
    return out


def blur_sobel_batch(src, radius, out=None):
    """gs_blur(radius) -> gs_sobel in one pass (no blurred intermediate in HBM); `out` keeps its 1-px frame,
    a fresh output is zero-filled like gs_alloc"""
    import torch
    n, h, w = _chk_frames(src)
    out = torch.zeros_like(src) if out is None else out
    check(lib().gs_b200_blur_sobel_batch(_p(out), _p(src), w, h, n, radius, _stream()), "blur_sobel_batch")
    return out


def erode_batch(src, out=None):
    import torch
    n, h, w = _chk_frames(src)
    out = torch.empty_like(src) if out is None else out
    check(lib().gs_b200_erode_batch(_p(out), _p(src), w, h, n, _stream()), "erode_batch")
    return out


def dilate_batch(src, out=None):
    import torch
    n, h, w = _chk_frames(src)
    out = torch.empty_like(src) if out is None else out
    check(lib().gs_b200_dilate_batch(_p(out), _p(src), w, h, n, _stream()), "dilate_batch")
    return out


def erode_n_batch(src, iters, out=None):
    """`iters` passes of the 3x3 erode in one call (bit-identical to `iters` chained erode_batch calls)"""
    import torch
    n, h, w = _chk_frames(src)
    if not 0 <= iters < 2 ** 32:
        raise ValueError("iters must be in [0, 2**32), got %r" % (iters,))
    out = torch.empty_like(src) if out is None else out
    check(lib().gs_b200_erode_n_batch(_p(out), _p(src), w, h, n, iters, _stream()), "erode_n_batch")
    return out


def dilate_n_batch(src, iters, out=None):
    """`iters` passes of the 3x3 dilate in one call (bit-identical to `iters` chained dilate_batch calls)"""
    import torch
    n, h, w = _chk_frames(src)
    if not 0 <= iters < 2 ** 32:
        raise ValueError("iters must be in [0, 2**32), got %r" % (iters,))
    out = torch.empty_like(src) if out is None else out
    check(lib().gs_b200_dilate_n_batch(_p(out), _p(src), w, h, n, iters, _stream()), "dilate_n_batch")
    return out


def resize_batch(src, dw, dh, out=None):
    import torch
    n, h, w = _chk_frames(src)
    out = torch.empty((n, dh, dw), dtype=torch.uint8, device=src.device) if out is None else out
    check(lib().gs_b200_resize_batch(_p(out), dw, dh, _p(src), w, h, n, _stream()), "resize_batch")
    return out


def downsample_batch(src, out=None):
    import torch
    n, h, w = _chk_frames(src)
    out = torch.empty((n, h // 2, w // 2), dtype=torch.uint8, device=src.device) if out is None else out
    check(lib().gs_b200_downsample_batch(_p(out), _p(src), w, h, n, _stream()), "downsample_batch")
    return out


def integral_batch(src, out=None):
    """returns int32-typed storage holding the uint32 tables (torch has no native uint32 math)"""
    import torch
    n, h, w = _chk_frames(src)
    out = torch.empty((n, h, w), dtype=torch.int32, device=src.device) if out is None else out
    check(lib().gs_b200_integral_batch(_p(out), _p(src), w, h, n, _stream()), "integral_batch")
    return out


def _kp_buffers(src, n, nkps):
    import torch
    kps = torch.empty((n, nkps, 12), dtype=torch.int32, device=src.device)   # 48-byte records
    counts = torch.empty((n,), dtype=torch.int32, device=src.device)
    return kps, counts


def fast_batch(src, nkps, threshold, scoremap=None):
    """-> (scoremap, kps[n, nkps, 12 words], counts[n])"""
    import torch
    n, h, w = _chk_frames(src)
    scoremap = torch.zeros_like(src) if scoremap is None else scoremap
    kps, counts = _kp_buffers(src, n, nkps)
    check(lib().gs_b200_fast_batch(_p(src), w, h, n, _p(scoremap), _p(kps), _p(counts), nkps, threshold,
                                   _stream()), "fast_batch")
    return scoremap, kps, counts


def orb_extract_batch(src, nkps, threshold, scoremap=None):
    import torch
    n, h, w = _chk_frames(src)
    scoremap = torch.zeros_like(src) if scoremap is None else scoremap
    kps, counts = _kp_buffers(src, n, nkps)
    check(lib().gs_b200_orb_extract_batch(_p(src), w, h, n, _p(scoremap), _p(kps), _p(counts), nkps,
                                          threshold, _stream()), "orb_extract_batch")
    return scoremap, kps, counts


def filter_batch(src, kernel, norm, out=None):
    """kernel: (kh, kw) int8 numpy array (host: the weights are call parameters)"""
    import torch
    n, h, w = _chk_frames(src)
    out = torch.empty_like(src) if out is None else out
    k = np.ascontiguousarray(kernel).view(np.int8)
    check(lib().gs_b200_filter_batch(_p(out), _p(src), w, h, n, _vp(k), k.shape[1], k.shape[0], norm, _stream()),
          "filter_batch")
    return out


def match_template_batch(img, tmpl, out=None):
    """img: (n, h, w) uint8, tmpl: (th, tw) uint8 device tensor -> (n, h-th+1, w-tw+1) uint8"""
    import torch
    n, h, w = _chk_frames(img)
    th, tw = tmpl.shape
    out = torch.empty((n, h - th + 1, w - tw + 1), dtype=torch.uint8, device=img.device) if out is None else out
    check(lib().gs_b200_match_template_batch(_p(out), _p(img), w, h, n, _p(tmpl), tw, th, _stream()), "match_template_batch")
    return out


def find_best_match_batch(result):
    """(n, rh, rw) uint8 -> (n, 2) int32 (x, y)"""
    import torch
    n, rh, rw = _chk_frames(result)
    best = torch.empty((n, 2), dtype=torch.int32, device=result.device)
    check(lib().gs_b200_find_best_match_batch(_p(best), _p(result), rw, rh, n, _stream()), "find_best_match_batch")
    return best


def histogram_batch(src, out=None):
    """(n, h, w) uint8 -> (n, 256) int32-typed storage of the unsigned counts"""
    import torch
    n, h, w = _chk_frames(src)
    out = torch.empty((n, 256), dtype=torch.int32, device=src.device) if out is None else out
    check(lib().gs_b200_histogram_batch(_p(out), _p(src), w, h, n, _stream()), "histogram_batch")
    return out


def otsu_threshold_batch(src, hist=None, out=None):
    """per-frame Otsu thresholds, (n,) uint8 on the device"""
    import torch
    n, h, w = _chk_frames(src)
    out = torch.empty((n,), dtype=torch.uint8, device=src.device) if out is None else out
    check(lib().gs_b200_otsu_threshold_batch(_p(out), _p(hist) if hist is not None else None, _p(src), w, h, n,
                                             _stream()), "otsu_threshold_batch")
    return out


def threshold_batch(img, thresh, offset=0):
    """in place; thresh is an int (all frames) or a (n,) uint8 device tensor (per frame, + offset)"""
    n, h, w = _chk_frames(img)
    if isinstance(thresh, int):
        check(lib().gs_b200_threshold_batch(_p(img), w, h, n, thresh, _stream()), "threshold_batch")
    else:
        check(lib().gs_b200_threshold_each_batch(_p(img), w, h, n, _p(thresh), offset, _stream()), "threshold_each_batch")
    return img


def match_orb_batch(kps1, counts1, kps2, counts2, max_matches, max_distance):
    """kps*: (npairs, stride, 12) int32 keypoint words as produced by orb_extract_batch, counts*: (npairs,)
    -> (matches[npairs, max_matches, 3], counts[npairs])"""
    import torch
    npairs, s1, s2 = kps1.shape[0], kps1.shape[1], kps2.shape[1]
    matches = torch.empty((npairs, max_matches, 3), dtype=torch.int32, device=kps1.device)
    counts = torch.empty((npairs,), dtype=torch.int32, device=kps1.device)
    check(lib().gs_b200_match_orb_batch(_p(kps1), _p(counts1), s1, _p(kps2), _p(counts2), s2, npairs, _p(matches),
                                        _p(counts), max_matches, max_distance, _stream()), "match_orb_batch")
    return matches, counts


def blobs_batch(src, nblobs):
    """(n, h, w) uint8 -> (labels (n, h, w) int16 storage of the uint16 labels, blobs (n, nblobs, 8) int32 words, counts (n,))"""
    import torch
    n, h, w = _chk_frames(src)
    labels = torch.empty((n, h, w), dtype=torch.int16, device=src.device)
    blobs = torch.zeros((n, nblobs, 8), dtype=torch.int32, device=src.device)
    counts = torch.empty((n,), dtype=torch.int32, device=src.device)
    check(lib().gs_b200_blobs_batch(_p(src), w, h, n, _p(labels), _p(blobs), _p(counts), nblobs, _stream()), "blobs_batch")
    return labels, blobs, counts


def perspective_correct_batch(src, dw, dh, corners, out=None):
    """corners: (4, 2) numpy (one quad for every frame, host) or an (n, 4, 2) int32 CUDA tensor (per frame)"""
    import torch
    n, h, w = _chk_frames(src)
    out = torch.empty((n, dh, dw), dtype=torch.uint8, device=src.device) if out is None else out
    if isinstance(corners, np.ndarray):
        c = np.ascontiguousarray(corners, np.uint32)
        check(lib().gs_b200_perspective_correct_batch(_p(out), dw, dh, _p(src), w, h, n, _vp(c), 0, _stream()), "perspective")
    else:
        assert corners.is_cuda and corners.dtype == torch.int32 and corners.is_contiguous() and corners.shape == (n, 4, 2)
        check(lib().gs_b200_perspective_correct_batch(_p(out), dw, dh, _p(src), w, h, n, _p(corners), 1, _stream()), "perspective")
    return out


def lbp_detect_batch(cascade, ii, max_rects, scale_factor, min_scale, max_scale, step):
    """ii: (n, h, w) int32 storage of uint32 tables -> (rects[n, max_rects, 4], counts[n])"""
    import torch
    assert ii.is_cuda and ii.dtype == torch.int32 and ii.dim() == 3 and ii.is_contiguous()
    n, h, w = ii.shape
    rects = torch.empty((n, max_rects, 4), dtype=torch.int32, device=ii.device)
    counts = torch.empty((n,), dtype=torch.int32, device=ii.device)
    check(lib().gs_b200_lbp_detect_batch(cascade.ptr, _p(ii), w, h, n, _p(rects), _p(counts), max_rects,
                                         scale_factor, min_scale, max_scale, step, _stream()), "lbp_detect")
    return rects, counts


def lbp_window_count(cascade, w, h, scale_factor, min_scale, max_scale, step):
    return int(lib().gs_b200_lbp_window_count(cascade.ptr, w, h, scale_factor, min_scale, max_scale, step))


def kps_to_numpy(kps, counts):
    """device keypoint words -> list of KP_DTYPE arrays (one per frame)"""
    k = kps.cpu().numpy().view(np.uint32)
    c = counts.cpu().numpy()
    return [np.ascontiguousarray(k[f, : c[f]]).view(KP_DTYPE).reshape(-1) for f in range(k.shape[0])]


def rects_to_numpy(rects, counts):
    r = rects.cpu().numpy().view(np.uint32)
    c = counts.cpu().numpy()
    return [np.ascontiguousarray(r[f, : c[f]]).view(RECT_DTYPE).reshape(-1) for f in range(r.shape[0])]
