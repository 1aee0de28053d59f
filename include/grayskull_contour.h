/*
 * grayskull_contour.h -- gs_trace_contour over frame batches on the device, in the companion library
 * libgrayskull_contour.so (link -lgrayskull_contour; it does not need libgrayskull_b200.so).
 *
 * This header's name deliberately does not match grayskull_b200*.h: the main library's headers are the set whose
 * declarations libgrayskull_b200.so exports, and these calls live in their own library.
 *
 * Conventions are grayskull_b200.h's: DEVICE pointers, n frames of w x h back to back, work enqueued on `s` and not
 * synchronised, 0 or a cudaError_t returned (gs_b200_contour_last_error() gives the text), 64-bit offsets; batches above
 * 65535 frames and frames taller than 65535 row tiles run as any other.  A missing pointer or an empty frame aborts with
 * the reference's "Assertion failed: ..." message; n == 0 returns 0 and does nothing.  The calls allocate nothing and
 * synchronise nothing, so they can be captured into a CUDA graph.  In every list, frame f's records start at
 * f * stride and frame f uses its first min(counts[f], stride) of them; counts == NULL means all `stride`.
 *
 * The walk (reference grayskull.h:446-480): length = 0, box = {start.x, start.y, 1, 1}, p = start, dir = 7,
 * seenstart = 0; each step counts p if visited[p] == 0 (an out-of-frame p reads 0 and is not written) and sets
 * visited[p] = 255, then moves to the first of the 8 neighbours, searched from (dir + 1) % 8, that is inside the frame
 * and > 128, with the reference's unsigned/int arithmetic, and grows the box as the reference does (w = max(w, p.x -
 * box.x + 1) taken after box.x has moved, which is not the true width).  Each contour ends in one of three ways:
 */
#ifndef GRAYSKULL_CONTOUR_H
#define GRAYSKULL_CONTOUR_H

#include "grayskull_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

enum {
  GS_CONTOUR_RETURNED = 0, /* the walk reached start a second time: the reference's outputs, byte for byte */
  GS_CONTOUR_OPEN = 1,     /* p had no foreground neighbour: the reference's outputs, byte for byte */
  GS_CONTOUR_CYCLE = 2     /* the state (p, dir, seenstart) repeated, so the reference never returns: box, length and
                              visited as the reference's copies hold them from some step on, for ever */
};

/* Traces frame f's records k < min(counts[f], stride) at contours + f * stride, whose `start` the caller set, in
 * order k against frame f's `visited`: exactly what that many consecutive gs_trace_contour(img, visited, &c[k]) calls
 * do, except that a walk the reference never ends ends as GS_CONTOUR_CYCLE.  Writes each record's box and length and,
 * when ends != NULL, ends[f * stride + k]; records past the count and visited bytes no walk reaches are not written.
 * visited overlapping img returns cudaErrorInvalidValue (in the reference, aliasing changes the walk itself).
 * work: device scratch of work_bytes; gs_b200_trace_contours_work_bytes(w, h, n) holds all n frames at once, and a
 * smaller one runs the frames in chunks of as many as it holds.  Below one frame's share it returns
 * cudaErrorInvalidValue. */
int gs_b200_trace_contours_batch(const uint8_t *img, uint8_t *visited, unsigned w, unsigned h, unsigned n,
                                 struct gs_contour *contours, const unsigned *counts, unsigned stride, uint8_t *ends,
                                 void *work, size_t work_bytes, gs_b200_stream s);

/* the work_bytes at which gs_b200_trace_contours_batch handles n frames of w x h in one chunk (16 + 4 * w * h * n,
 * SIZE_MAX when that does not fit in a size_t) */
size_t gs_b200_trace_contours_work_bytes(unsigned w, unsigned h, unsigned n);

/* The start rule of the reference's wasm demo (examples/wasm/grayskull.c:303-318) for every blob record of
 * gs_b200_blobs_batch's output layout: start = the first pixel, in raster order over rows box.y .. box.y + box.h - 1
 * and columns box.x .. box.x + box.w - 1 (unsigned sums), whose label is blob.label; (box.x, box.y) when there is
 * none.  Pixels outside the frame are not read.  For gs_blobs records that pixel lies on row box.y.  Writes only
 * contours[f * stride + b].start, for b < min(counts[f], stride). */
int gs_b200_blob_contour_starts_batch(const gs_label *labels, unsigned w, unsigned h, unsigned n,
                                      const struct gs_blob *blobs, const unsigned *counts, unsigned stride,
                                      struct gs_contour *contours, gs_b200_stream s);

/* the text of the calling thread's last error of this library */
const char *gs_b200_contour_last_error(void);

#ifdef __cplusplus
}
#endif

#endif /* GRAYSKULL_CONTOUR_H */
