"""ctypes loaders shared by the tests: the oracle restatement and numpy wrappers of its calls, the real reference build
(oracle/_ref, when present), synthetic-input generators and the built library's SASS.  TEST INFRASTRUCTURE only."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")


class Image(C.Structure):
    _fields_ = [("w", C.c_uint), ("h", C.c_uint), ("data", C.c_void_p)]


class Keypoint(C.Structure):
    _fields_ = [("x", C.c_uint), ("y", C.c_uint), ("response", C.c_uint), ("angle", C.c_float),
                ("descriptor", C.c_uint32 * 8)]


class Point(C.Structure):
    _fields_ = [("x", C.c_uint), ("y", C.c_uint)]


class Rect(C.Structure):
    _fields_ = [("x", C.c_uint), ("y", C.c_uint), ("w", C.c_uint), ("h", C.c_uint)]


class Cascade(C.Structure):
    _fields_ = [
        ("window_w", C.c_uint16), ("window_h", C.c_uint16),
        ("nfeatures", C.c_uint16), ("nweaks", C.c_uint16), ("nstages", C.c_uint16),
        ("features", C.c_void_p), ("weak_feature_idx", C.c_void_p),
        ("weak_left_val", C.c_void_p), ("weak_right_val", C.c_void_p),
        ("weak_subset_offset", C.c_void_p), ("weak_num_subsets", C.c_void_p),
        ("subsets", C.c_void_p), ("stage_weak_start", C.c_void_p), ("stage_nweaks", C.c_void_p),
        ("stage_threshold", C.c_void_p),
    ]


MATCH_DTYPE = np.dtype([("idx1", "<u4"), ("idx2", "<u4"), ("distance", "<u4")])
KP_DTYPE = np.dtype([("x", "<u4"), ("y", "<u4"), ("response", "<u4"), ("angle", "<f4"),
                     ("descriptor", "<u4", (8,))])
RECT_DTYPE = np.dtype([("x", "<u4"), ("y", "<u4"), ("w", "<u4"), ("h", "<u4")])
# struct gs_blob (reference grayskull.h:29-34): u16 label + 2 padding bytes, area, box, centroid = 32 bytes
BLOB_DTYPE = np.dtype({"names": ["label", "area", "bx", "by", "bw", "bh", "cx", "cy"],
                       "formats": ["<u2", "<u4", "<u4", "<u4", "<u4", "<u4", "<u4", "<u4"],
                       "offsets": [0, 4, 8, 12, 16, 20, 24, 28], "itemsize": 32})
assert KP_DTYPE.itemsize == 48 and RECT_DTYPE.itemsize == 16 and C.sizeof(Cascade) == 96


def ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def img(a):
    """numpy (h, w) uint8 array -> struct gs_image by value"""
    assert a.dtype == np.uint8 and a.flags.c_contiguous
    return Image(a.shape[1], a.shape[0], a.ctypes.data)


def build_oracle():
    subprocess.run(["make", "-s", "-C", ORACLE_DIR, "all"], check=True)


_cache = {}


def oracle():
    """our C restatement (oracle/libgs_oracle.so)"""
    if "o" not in _cache:
        path = os.path.join(ORACLE_DIR, "libgs_oracle.so")
        if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(
                os.path.join(ORACLE_DIR, "gs_oracle.c")):
            build_oracle()
        lib = C.CDLL(path)
        lib.gso_fast.restype = C.c_uint
        lib.gso_orb_extract.restype = C.c_uint
        lib.gso_lbp_window.restype = C.c_uint
        lib.gso_lbp_detect.restype = C.c_uint
        lib.gso_compute_orientation.restype = C.c_float
        lib.gso_sinf.restype = C.c_float
        lib.gso_sinf.argtypes = [C.c_float]
        lib.gso_atan2f.restype = C.c_float
        lib.gso_atan2f.argtypes = [C.c_float, C.c_float]
        lib.gso_match_orb.restype = C.c_uint
        lib.gso_lbp_depth_map.restype = None
        lib.gso_lbp_depth_map.argtypes = [C.c_void_p, C.c_void_p, C.c_uint, C.c_uint, C.c_float, C.c_int, C.c_void_p]
        lib.gso_filter.restype = None
        lib.gso_filter.argtypes = [C.c_void_p, C.c_void_p, C.c_uint, C.c_uint, C.c_void_p, C.c_uint, C.c_uint, C.c_uint]
        lib.gso_match_template.restype = None
        lib.gso_match_template.argtypes = [C.c_void_p, C.c_uint, C.c_uint, C.c_void_p, C.c_uint, C.c_uint, C.c_void_p]
        lib.gso_find_best_match.restype = C.c_uint
        lib.gso_find_best_match.argtypes = [C.c_void_p, C.c_uint, C.c_uint]
        lib.gso_histogram.restype = None
        lib.gso_histogram.argtypes = [C.c_void_p, C.c_uint, C.c_uint, C.c_void_p]
        lib.gso_otsu_from_hist.restype = C.c_uint
        lib.gso_otsu_from_hist.argtypes = [C.c_void_p, C.c_uint]
        lib.gso_otsu_threshold.restype = C.c_uint
        lib.gso_otsu_threshold.argtypes = [C.c_void_p, C.c_uint, C.c_uint]
        lib.gso_threshold.restype = None
        lib.gso_threshold.argtypes = [C.c_void_p, C.c_uint, C.c_uint, C.c_uint]
        lib.gso_match_orb.argtypes = [C.c_void_p, C.c_uint, C.c_void_p, C.c_uint, C.c_void_p, C.c_uint, C.c_float]
        lib.gso_blobs.restype = C.c_uint
        lib.gso_blobs.argtypes = [C.c_void_p, C.c_uint, C.c_uint, C.c_void_p, C.c_void_p, C.c_uint]
        lib.gso_blob_corners.restype = None
        lib.gso_blob_corners.argtypes = [C.c_void_p, C.c_uint, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.gso_perspective_correct.restype = None
        lib.gso_perspective_correct.argtypes = [C.c_void_p, C.c_uint, C.c_uint, C.c_void_p, C.c_uint, C.c_uint, C.c_void_p]
        lib.gso_compute_orientation.argtypes = [C.c_void_p, C.c_uint, C.c_uint, C.c_uint, C.c_uint, C.c_uint]
        lib.gso_lbp_window.argtypes = [C.c_void_p, C.c_void_p, C.c_uint, C.c_uint, C.c_int, C.c_int,
                                       C.c_float]
        lib.gso_lbp_detect.argtypes = [C.c_void_p, C.c_void_p, C.c_uint, C.c_uint, C.c_void_p,
                                       C.c_uint, C.c_float, C.c_float, C.c_float, C.c_int]
        _cache["o"] = lib
    return _cache["o"]


# ---- oracle calls on numpy arrays (O = oracle()) ---------------------------------------------------------------------
def o_blur(O, a, r):
    d = np.empty_like(a); O.gso_blur(ptr(d), ptr(a), a.shape[1], a.shape[0], r); return d
def o_adaptive(O, a, r, c):
    d = np.empty_like(a); O.gso_adaptive_threshold(ptr(d), ptr(a), a.shape[1], a.shape[0], r, c); return d
def o_morph(O, a, dil):
    d = np.empty_like(a); O.gso_morph(ptr(d), ptr(a), a.shape[1], a.shape[0], dil); return d
def o_sobel(O, a, fill=0):
    """gso_sobel into an array of `fill`: its 1-px frame keeps `fill` (an array: a copy of it)"""
    d = np.array(np.broadcast_to(fill, a.shape), np.uint8)
    O.gso_sobel(ptr(d), ptr(a), a.shape[1], a.shape[0]); return d
def o_resize(O, a, dw, dh):
    d = np.empty((dh, dw), np.uint8); O.gso_resize(ptr(d), dw, dh, ptr(a), a.shape[1], a.shape[0]); return d
def o_down(O, a):
    d = np.empty((a.shape[0] // 2, a.shape[1] // 2), np.uint8); O.gso_downsample(ptr(d), ptr(a), a.shape[1], a.shape[0]); return d
def o_integral(O, a):
    ii = np.empty(a.shape, np.uint32); O.gso_integral(ptr(a), a.shape[1], a.shape[0], ptr(ii)); return ii
def o_fast(O, a, sm, nkps, t):
    k = np.zeros(nkps, KP_DTYPE)
    n = O.gso_fast(ptr(a), a.shape[1], a.shape[0], ptr(sm), sm.shape[1], sm.shape[0], ptr(k), nkps, t)
    return k[:n]
def o_orb(O, a, sm, nkps, t):
    k = np.zeros(nkps, KP_DTYPE)
    n = O.gso_orb_extract(ptr(a), a.shape[1], a.shape[0], ptr(k), nkps, t, ptr(sm))
    return k[:n]
def o_detect(O, cas, ii, max_rects, sf, mn, mx, step):
    r = np.zeros(max(max_rects, 1), RECT_DTYPE)
    n = O.gso_lbp_detect(cas.ptr, ptr(ii), ii.shape[1], ii.shape[0], ptr(r), max_rects, sf, mn, mx, step)
    return r[:n]
def o_match(O, k1, k2, mm, md):
    m = np.zeros(max(1, min(mm, len(k1))), MATCH_DTYPE)          # at most one match per query
    n = O.gso_match_orb(ptr(k1), len(k1), ptr(k2 if len(k2) else np.zeros(1, KP_DTYPE)), len(k2), ptr(m), mm, md)
    return m[:n]


def have_ref():
    return os.path.exists(os.path.join(ORACLE_DIR, "_ref", "libgs_ref.so"))


def ref():
    """the UNMODIFIED reference header compiled as a shared object (oracle/_ref)"""
    if "r" not in _cache:
        lib = C.CDLL(os.path.join(ORACLE_DIR, "_ref", "libgs_ref.so"))
        for name in ("gs_blur", "gs_sobel", "gs_erode", "gs_dilate", "gs_resize", "gs_downsample"):
            getattr(lib, name).restype = None
        lib.gs_blur.argtypes = [Image, Image, C.c_uint]
        lib.gs_sobel.argtypes = [Image, Image]
        lib.gs_erode.argtypes = [Image, Image]
        lib.gs_dilate.argtypes = [Image, Image]
        lib.gs_resize.argtypes = [Image, Image]
        lib.gs_downsample.argtypes = [Image, Image]
        lib.gs_adaptive_threshold.argtypes = [Image, Image, C.c_uint, C.c_int]
        lib.gs_adaptive_threshold.restype = None
        lib.gs_integral.argtypes = [Image, C.c_void_p]
        lib.gs_integral.restype = None
        lib.gs_fast.argtypes = [Image, Image, C.c_void_p, C.c_uint, C.c_uint]
        lib.gs_fast.restype = C.c_uint
        lib.gs_compute_orientation.argtypes = [Image, C.c_uint, C.c_uint, C.c_uint]
        lib.gs_compute_orientation.restype = C.c_float
        lib.gs_brief_descriptor.argtypes = [Image, C.c_void_p]
        lib.gs_brief_descriptor.restype = None
        lib.gs_orb_extract.argtypes = [Image, C.c_void_p, C.c_uint, C.c_uint, C.c_void_p]
        lib.gs_orb_extract.restype = C.c_uint
        lib.gs_lbp_window.argtypes = [C.c_void_p, C.c_void_p, C.c_uint, C.c_uint, C.c_int, C.c_int,
                                      C.c_float]
        lib.gs_lbp_window.restype = C.c_uint
        lib.gs_lbp_detect.argtypes = [C.c_void_p, C.c_void_p, C.c_uint, C.c_uint, C.c_void_p,
                                      C.c_uint, C.c_float, C.c_float, C.c_float, C.c_int]
        lib.gs_lbp_detect.restype = C.c_uint
        lib.gs_match_orb.argtypes = [C.c_void_p, C.c_uint, C.c_void_p, C.c_uint, C.c_void_p, C.c_uint, C.c_float]
        lib.gs_match_orb.restype = C.c_uint
        lib.gs_filter.argtypes = [Image, Image, Image, C.c_uint]
        lib.gs_filter.restype = None
        lib.gs_match_template.argtypes = [Image, Image, Image]
        lib.gs_match_template.restype = None
        lib.gs_find_best_match.argtypes = [Image]
        lib.gs_find_best_match.restype = Point
        lib.gs_histogram.argtypes = [Image, C.c_void_p]
        lib.gs_histogram.restype = None
        lib.gs_otsu_threshold.argtypes = [Image]
        lib.gs_otsu_threshold.restype = C.c_uint8
        lib.gs_threshold.argtypes = [Image, C.c_uint8]
        lib.gs_threshold.restype = None
        lib.gs_blobs.argtypes = [Image, C.c_void_p, C.c_void_p, C.c_uint]
        lib.gs_blobs.restype = C.c_uint
        lib.gs_blob_corners.argtypes = [Image, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.gs_blob_corners.restype = None
        lib.gs_perspective_correct.argtypes = [Image, Image, C.c_void_p]
        lib.gs_perspective_correct.restype = None
        lib.ref_frontalface.restype = C.c_void_p
        lib.ref_sort_keypoints.argtypes = [C.c_void_p, C.c_uint]
        lib.ref_sort_keypoints.restype = None
        _cache["r"] = lib
    return _cache["r"]


class HostCascade:
    """frontalface tables from the committed fixture, as a struct gs_lbp_cascade on the host"""

    def __init__(self, path=None):
        path = path or os.path.join(ROOT, "grayskull_b200", "data", "frontalface.npz")
        z = np.load(path)
        self.arrays = {k: np.ascontiguousarray(z[k]) for k in z.files}
        a = self.arrays
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


def xorshift_frame(w, h, f=0):
    """SURVEY.md 8(d) synthetic input: 64-bit xorshift, seed 0x9E3779B97F4A7C15 + f, top byte"""
    n = w * h
    out = np.empty(n, np.uint8)
    s = np.uint64((0x9E3779B97F4A7C15 + f) & 0xFFFFFFFFFFFFFFFF)
    # vectorised in blocks: xorshift is sequential, so run it in a small python loop over a
    # jump-free chunk using numpy scalars only for small frames; large frames use the C-speed
    # generator below.
    if n > 1 << 16:
        return _xorshift_big(w, h, f)
    s = int(s)
    M = (1 << 64) - 1
    for i in range(n):
        s ^= (s << 13) & M
        s ^= s >> 7
        s ^= (s << 17) & M
        out[i] = s >> 56
    return out.reshape(h, w)


def _xorshift_big(w, h, f):
    # numpy's PCG is fine for big parity inputs; the exact xorshift stream only matters for the
    # documented small fixtures.  Seeded per frame for reproducibility.
    rng = np.random.default_rng(0x9E3779B9 + f)
    return rng.integers(0, 256, size=(h, w), dtype=np.uint8)


def natural_like(w, h, seed=0):
    """smooth-ish random image (sum of blobs + noise) so FAST/LBP see structure"""
    rng = np.random.default_rng(seed)
    small = rng.integers(0, 256, size=((h + 7) // 8 + 1, (w + 7) // 8 + 1)).astype(np.float32)
    up = np.kron(small, np.ones((8, 8), np.float32))[:h, :w]
    noise = rng.normal(0, 12, size=(h, w)).astype(np.float32)
    return np.clip(up * 0.7 + noise + 30, 0, 255).astype(np.uint8)


def blob_fields(b):
    """the defined fields of a gs_blob array (the 2 padding bytes after `label` are not part of the contract)"""
    return [tuple(int(b[k][i]) for k in BLOB_DTYPE.names) for i in range(len(b))]


def binary_like(w, h, seed, density=0.5, smooth=3):
    """0 / 255 image with blobs of assorted sizes (thresholded smooth noise) plus salt noise: many small
    components, a few large ones, touching the borders"""
    rng = np.random.default_rng(seed)
    a = rng.random((h + 2 * smooth, w + 2 * smooth)).astype(np.float32)
    k = 2 * smooth + 1
    c = np.cumsum(np.cumsum(np.pad(a, ((1, 0), (1, 0))), 0), 1)
    box = (c[k:, k:] - c[:-k, k:] - c[k:, :-k] + c[:-k, :-k]) / (k * k)
    img = (box[:h, :w] > np.quantile(box, 1 - density)).astype(np.uint8) * 255
    salt = rng.random((h, w))
    img[salt < 0.02] = 255
    img[salt > 0.98] = 0
    img[rng.random((h, w)) < 0.01] = 130          # values just above / below the >= 128 foreground test
    img[rng.random((h, w)) < 0.01] = 127
    return np.ascontiguousarray(img)


def desc_sets(rng, n1, n2, dup=0.3):
    """descriptor sets with near-duplicates and exact duplicates so ties and the ratio test trigger"""
    k1 = np.zeros(n1, KP_DTYPE); k2 = np.zeros(n2, KP_DTYPE)
    k2["descriptor"] = rng.integers(0, 2**32, (n2, 8), dtype=np.uint64).astype(np.uint32)
    k1["descriptor"] = rng.integers(0, 2**32, (n1, 8), dtype=np.uint64).astype(np.uint32)
    for i in range(n1):
        if n2 and rng.random() < dup:
            j = int(rng.integers(0, n2))
            d = k2["descriptor"][j].copy()
            for _ in range(int(rng.integers(0, 40))):
                d[int(rng.integers(0, 8))] ^= np.uint32(1 << int(rng.integers(0, 32)))
            k1["descriptor"][i] = d
    if n2 > 4:                                   # exact duplicates inside set 2: best == second
        k2["descriptor"][1] = k2["descriptor"][0]
    return k1, k2


FILTER_KERNELS = {   # (weights as int8 rows, norm): the reference's presets (grayskull.h:249-253) and stress cases
    "sharpen": ([[0, -1, 0], [-1, 5, -1], [0, -1, 0]], 1),
    "emboss": ([[-2, -1, 0], [-1, 1, 1], [0, 1, 2]], 1),
    "box": ([[1, 1, 1], [1, 1, 1], [1, 1, 1]], 9),
    "gaussian": ([[1, 2, 1], [2, 4, 2], [1, 2, 1]], 16),
    "emboss_norm3": ([[-2, -1, 0], [-1, 1, 1], [0, 1, 2]], 3),       # negative sums with norm > 1 -> 255
    "extreme": ([[127, -128, 127], [-128, 127, -128], [127, -128, 127]], 7),
    "huge_norm": ([[1, 1, 1], [1, 1, 1], [1, 1, 1]], 3000000000),     # norm above 2^31
    "big_norm_neg": ([[-1, 0, 0], [0, 0, 0], [0, 0, 0]], 20000000),   # (2^32 - s) / norm below 255
    "k5": ([[1, 4, 6, 4, 1], [4, 16, 24, 16, 4], [6, 24, 36, 24, 6], [4, 16, 24, 16, 4], [1, 4, 6, 4, 1]], 256),
    "k2x4": ([[1, -2, 3, -4], [5, 6, -7, 8]], 5),                     # even sizes: taps at -kw/2 .. kw-1-kw/2
    "k1x1": ([[3]], 2),
    "k7x3": ([[1, 0, -1, 2, -1, 0, 1], [2, 0, -2, 4, -2, 0, 2], [1, 0, -1, 2, -1, 0, 1]], 4),
}


def filter_kernel(name):
    rows, norm = FILTER_KERNELS[name]
    return np.ascontiguousarray(np.array(rows, np.int8).view(np.uint8)), norm


def check_next_golden(impl):
    """tests/golden/next_golden.npz (made by the REAL reference, tools/make_golden.py) against `impl`, an object
    with gs_histogram(a), gs_otsu_threshold(a), gs_threshold(a, t), gs_filter(dst, src, kernel_u8, norm),
    gs_match_template(img, tmpl), gs_find_best_match(res) -> (x, y), gs_orb(a, nkps, t), gs_match_orb(k1, k2, mm, md).
    Shared by the oracle test (CPU) and the CUDA test (GPU) so the checking logic itself is exercised on both."""
    z = np.load(os.path.join(ROOT, "tests", "golden", "next_golden.npz"))
    for tag in [str(t) for t in z["tags"]]:
        a = np.ascontiguousarray(z[tag + "img"])
        assert np.array_equal(impl.gs_histogram(a), z[tag + "hist"]), tag
        t = int(z[tag + "otsu"])
        assert impl.gs_otsu_threshold(a) == t, tag
        assert np.array_equal(impl.gs_threshold(a.copy(), t), z[tag + "threshold_otsu"]), tag
        for name in ("sharpen", "emboss", "box", "gaussian", "emboss_norm3", "k5", "k2x4"):
            k, norm = filter_kernel(name)
            assert np.array_equal(impl.gs_filter(np.zeros_like(a), a, k, norm), z[tag + "filter_" + name]), (tag, name)
        res = impl.gs_match_template(a, np.ascontiguousarray(z[tag + "tmpl"]))
        assert np.array_equal(res, z[tag + "tmatch"]), tag
        assert tuple(impl.gs_find_best_match(res)) == tuple(int(v) for v in z[tag + "tmatch_best"]), tag
        ka, kb = impl.gs_orb(a, 300, 20), impl.gs_orb(np.ascontiguousarray(z[tag + "shifted"]), 300, 20)
        assert ka.tobytes() == z[tag + "kps_a"].tobytes() and kb.tobytes() == z[tag + "kps_b"].tobytes(), tag
        m = impl.gs_match_orb(ka, kb, 300, 60.0)
        assert m.tobytes() == z[tag + "matches"].tobytes() and len(m) > 20, tag


def oracle_chain(cascade_ptr, frame, **params):
    """the C5 chain of grayskull_b200/pipeline.py (blur r=5 -> sobel -> orb_extract / integral + lbp_detect on
    the sobel map) on one frame through the oracle restatement"""
    import sys
    O, L = oracle(), sys.modules[__name__]
    p = dict(radius=5, nkps=1250, threshold=20, max_rects=4096, scale_factor=1.1, min_scale=1.0, max_scale=4.0, step=2)
    p.update(params)
    h, w = frame.shape
    b = np.empty_like(frame)
    O.gso_blur(L.ptr(b), L.ptr(frame), w, h, p["radius"])
    s = np.zeros_like(frame)
    O.gso_sobel(L.ptr(s), L.ptr(b), w, h)
    k = np.zeros(p["nkps"], L.KP_DTYPE)
    sm = np.zeros_like(frame)
    nk = O.gso_orb_extract(L.ptr(s), w, h, L.ptr(k), p["nkps"], p["threshold"], L.ptr(sm))
    t = np.empty(frame.shape, np.uint32)
    O.gso_integral(L.ptr(s), w, h, L.ptr(t))
    r = np.zeros(p["max_rects"], L.RECT_DTYPE)
    nr = O.gso_lbp_detect(cascade_ptr, L.ptr(t), w, h, L.ptr(r), p["max_rects"], p["scale_factor"], p["min_scale"],
                          p["max_scale"], p["step"])
    return {"sobel": s, "kps": k[:nk], "rects": r[:nr]}


def otsu_images(rng):
    """bimodal, flat, two-level, dark-heavy, noise and near-tie images: exercises wb == 0 skips, the wf == 0
    break and fp32 ties in varBetween"""
    out = []
    for (w, h) in ((3, 3), (64, 48), (257, 31), (640, 480), (1, 1), (5, 1)):
        out.append(rng.integers(0, 256, (h, w), dtype=np.uint8))
        a = np.where(rng.random((h, w)) < 0.3, rng.normal(60, 12, (h, w)), rng.normal(190, 20, (h, w)))
        out.append(np.clip(a, 0, 255).astype(np.uint8))
        out.append(np.full((h, w), int(rng.integers(0, 256)), np.uint8))
        b = np.full((h, w), 10, np.uint8); b.flat[:: max(1, (w * h) // 7)] = 250
        out.append(b)
        out.append((rng.integers(0, 2, (h, w)) * 255).astype(np.uint8))
        out.append(rng.integers(100, 104, (h, w), dtype=np.uint8))
    out.append(natural_like(1920, 1080, 3))
    return out


# ---- kernel names and the built library's SASS -----------------------------------------------------------------------
def kernel_id(name):
    """a demangled kernel name (kineto's 'void gsb::k_box_mid<1, false>(CUtensorMap_st, ...)' or cu++filt's
    'void gsb::k_box_mid<(int)1, (bool)0>(...)') -> 'gsb::k_box_mid<1,false>'"""
    s = name.strip()
    if s.startswith("void "):
        s = s[5:]
    depth = 0
    for i, ch in enumerate(s):
        depth += ch == "<"
        depth -= ch == ">"
        if ch == "(" and depth == 0:
            s = s[:i]
            break
    s = s.replace("(bool)0", "false").replace("(bool)1", "true")
    s = re.sub(r"\((?:unsigned )?int\)(-?\d+)", r"\1", s)
    s = re.sub(r"\b(\d+)u\b", r"\1", s)
    return s.replace(" ", "")


def cuda_tool(name):
    """a CUDA toolkit binary from PATH, else from /usr/local/cuda/bin; None when neither has it"""
    tool = shutil.which(name) or os.path.join("/usr/local/cuda/bin", name)
    return tool if os.path.exists(tool) else None


def demangle(names):
    """cu++filt over mangled names (returned as they are without the tool)"""
    tool = cuda_tool("cu++filt")
    if not names or tool is None:
        return list(names)
    out = subprocess.run([tool], input="\n".join(names) + "\n", capture_output=True, text=True, check=True).stdout
    return out.splitlines()


def sass_functions():
    """{kernel_id: SASS} of every function in the built library, from one `cuobjdump -sass` per process.  Each SASS
    starts with the 'code for sm_XX' line of the cubin that holds it.  Skips the calling test without cuobjdump."""
    if "sass" not in _cache:
        import pytest
        from grayskull_b200 import _lib
        tool = cuda_tool("cuobjdump")
        if tool is None:
            pytest.skip("cuobjdump not found")
        listing = subprocess.run([tool, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
        funcs = {}
        for cubin in re.split(r"^\s*(?=code for sm_\w+\s*$)", listing, flags=re.M)[1:]:
            arch, *parts = re.split(r"^\s*Function : (\S+)\s*$", cubin, flags=re.M)
            arch = arch.strip().splitlines()[0]
            for name, body in zip(demangle(parts[0::2]), parts[1::2]):
                funcs[kernel_id(name)] = arch + "\n" + body
        _cache["sass"] = funcs
    return _cache["sass"]
