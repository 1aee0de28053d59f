"""ORB features over an image pyramid for frame batches on the device (include/grayskull_b200_pyramid.h), on torch
CUDA tensors: bit-exact with the reference CLI's multi-scale ORB (extract_pyramid_orb_nm of its `orb` verb)."""
import ctypes as C

from ._lib import check, lib


def levels_for(w, h, levels):
    """the number of pyramid levels that run for a w x h frame when `levels` are asked for"""
    return lib().gs_b200_orb_pyramid_levels(w, h, levels)


def level_sizes(w, h, levels):
    """[(w_l, h_l)] of the levels that run"""
    out = []
    for _ in range(levels_for(w, h, levels)):
        out.append((w, h))
        w, h = w // 2, h // 2
    return out


def orb_pyramid_batch(src, nkps, threshold, levels=3, scoremap=None, pyr=None):
    """src: (n, h, w) uint8 on the device -> (kps, counts, scoremap, pyr) on the current stream.
    kps: (n, nkps, 12) int32 storage of struct gs_keypoint (api.kps_to_numpy reads it); counts: (n,) int32;
    scoremap: flat uint8, levels 0..L-1 of n maps each, level by level (pass one to choose the bytes that take part in
    each level's NMS; a new one is zeroed); pyr: flat uint8, levels 1..L-1 of n frames each (None when L <= 1)."""
    import torch
    assert src.is_cuda and src.dtype == torch.uint8 and src.dim() == 3 and src.is_contiguous()
    n, h, w = src.shape
    sizes = level_sizes(w, h, levels)
    maps = sum(a * b for a, b in sizes) * n
    below = sum(a * b for a, b in sizes[1:]) * n
    if scoremap is None:
        scoremap = torch.zeros(max(maps, 1), dtype=torch.uint8, device=src.device)
    assert scoremap.is_cuda and scoremap.dtype == torch.uint8 and scoremap.is_contiguous() and scoremap.numel() >= maps
    if pyr is None and below:
        pyr = torch.empty(below, dtype=torch.uint8, device=src.device)
    if below:
        assert pyr.is_cuda and pyr.dtype == torch.uint8 and pyr.is_contiguous() and pyr.numel() >= below
    kps = torch.empty((n, max(nkps, 1), 12), dtype=torch.int32, device=src.device)
    counts = torch.empty(n, dtype=torch.int32, device=src.device)
    check(lib().gs_b200_orb_pyramid_batch(C.c_void_p(src.data_ptr()), w, h, n, levels,
                                          C.c_void_p(pyr.data_ptr()) if below else None,
                                          C.c_void_p(scoremap.data_ptr()), C.c_void_p(kps.data_ptr()),
                                          C.c_void_p(counts.data_ptr()), nkps, threshold,
                                          C.c_void_p(torch.cuda.current_stream().cuda_stream)), "orb_pyramid_batch")
    return kps, counts, scoremap, pyr
