/*
 * grayskull_b200_roi.h -- regions of interest cut out of frame batches on the device, part of libgrayskull_b200.so
 * (link -lgrayskull_b200).
 *
 * Each output image is the reference's gs_crop (grayskull.h:154-157) of one region of a frame, followed by
 * gs_resize_nn (:164-169) or gs_resize (:171-187) of that crop to dw x dh -- bit for bit those calls made one after
 * the other, with the crop never written to memory.  A pure crop is dw == roi.w, dh == roi.h; a pure resize is the
 * whole frame as the region.  Conventions are grayskull_b200.h's: DEVICE pointers, n frames of sw x sh back to back,
 * work enqueued on `s` and not synchronised, 0 or a cudaError_t returned (gs_b200_last_error() gives the text, and
 * gs_b200_launch_count() counts these launches too).  All offsets are 64-bit, so batches over 4 GiB work.
 *
 * Reference arithmetic: source coordinates are 32-bit unsigned, as in the reference.  gs_crop's roi.x + x and
 * gs_resize_nn's x * crop.w may wrap; a coordinate outside the frame reads 0 (gs_get).  Bilinear mode keeps
 * gs_resize's fp32 evaluation order.
 */
#ifndef GRAYSKULL_B200_ROI_H
#define GRAYSKULL_B200_ROI_H

#include "grayskull_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#define GS_B200_NEAREST 0  /* gs_resize_nn */
#define GS_B200_BILINEAR 1 /* gs_resize   */

/* One region (host, by value) cut from each of n frames -> n images of dw x dh at dst + f*dw*dh.
 * Aborts with the reference's message when gs_crop's assert fails (its wrapping roi.x + roi.w <= sw,
 * roi.y + roi.h <= sh, a non-empty region) or, in bilinear mode, gs_resize's (dw, dh > 0).
 * An unknown mode returns cudaErrorInvalidValue. */
int gs_b200_crop_resize_batch(uint8_t *dst, unsigned dw, unsigned dh, const uint8_t *src, unsigned sw, unsigned sh,
                              unsigned n, struct gs_rect roi, int mode, gs_b200_stream s);

/* Per-frame region lists in DEVICE memory: rects = n x max_rects gs_rect (the layout gs_b200_lbp_detect_batch
 * writes), counts = n unsigned (NULL: all max_rects are used).  Slot (f, k) is at dst + (f*max_rects + k)*dw*dh.
 * Slot k of frame f with k >= min(counts[f], max_rects) is left untouched.  A region gs_crop's assert would reject
 * gives a zero-filled slot (the device cannot abort; detector and blob outputs never produce one).  Bilinear mode
 * aborts unless dw, dh > 0; an unknown mode returns cudaErrorInvalidValue. */
int gs_b200_rois_resize_batch(uint8_t *dst, unsigned dw, unsigned dh, const uint8_t *src, unsigned sw, unsigned sh,
                              unsigned n, const struct gs_rect *rects, const unsigned *counts, unsigned max_rects,
                              int mode, gs_b200_stream s);

#ifdef __cplusplus
}
#endif

#endif /* GRAYSKULL_B200_ROI_H */
