/*
 * grayskull_draw.h -- the reference CLI's annotated pictures drawn onto frame batches on the device, in the companion
 * library libgrayskull_draw.so (link -lgrayskull_draw; it does not need libgrayskull_b200.so).
 *
 * This header's name deliberately does not match grayskull_b200*.h: the main library's headers are the set whose
 * declarations libgrayskull_b200.so exports, and these calls live in their own library.
 *
 * Each call draws what one detector verb of the reference CLI (examples/nanomagick/nanomagick.c) writes, from the lists
 * the main library's batch calls write: gs_b200_blobs_batch, gs_b200_fast_batch, gs_b200_lbp_detect_batch and
 * gs_b200_match_orb_batch.  Values and sizes are the verbs': 255 and 128, crosses of radius 2, 15 matches in the CLI.
 *
 * Conventions are grayskull_b200.h's: DEVICE pointers, n frames of w x h back to back, work enqueued on `s` and not
 * synchronised, 0 or a cudaError_t returned (gs_b200_draw_last_error() gives the text), 64-bit offsets; batches above
 * 65535 frames and frames taller than 65535 row tiles run as any other.  A missing pointer or an empty frame aborts with
 * the reference's "Assertion failed: ..." message; n == 0 returns 0 and does nothing.  The calls allocate nothing and
 * synchronise nothing, so they can be captured into a CUDA graph.  For the three same-size calls dst may equal src; any
 * other overlap of dst with an input image returns cudaErrorInvalidValue.  In every list input, frame f uses its first
 * min(counts[f], stride) records.
 */
#ifndef GRAYSKULL_DRAW_H
#define GRAYSKULL_DRAW_H

#include "grayskull_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The blobs verb (nanomagick.c:161-169).  Each record covers the linear indices y*w + x for x1 <= x <= x2 and
 * y1 <= y <= y2, both ends inclusive, with x1 = max(0, (int)box.x - 2), x2 = min(w, box.x + box.w + 2) and y1, y2
 * alike: so a box with x2 == w also covers pixel (0, y + 1) of each of its rows, as the verb does.  Indices >= w*h are
 * not written (the verb writes them past its buffer).  dst[i] = src[i] > 128 ? 255 : covered(i) ? 128 : 0.  The cost
 * does not grow with the boxes' areas: nested boxes cost what disjoint ones do. */
int gs_b200_draw_blobs_batch(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n,
                             const struct gs_blob *blobs, const unsigned *counts, unsigned stride, gs_b200_stream s);

/* The keypoints verb (nanomagick.c:229-239): dst = src, then a cross of 255 at each of the first min(top, count)
 * keypoints of a stable sort by descending response -- (x, y + dy) and (x + dx, y) for dx, dy in [-2, 2], each pixel
 * only when it is inside the frame (gs_set, unsigned wrap-around included). */
int gs_b200_draw_keypoints_batch(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n,
                                 const struct gs_keypoint *kps, const unsigned *counts, unsigned stride,
                                 unsigned top, gs_b200_stream s);

/* The faces verb (nanomagick.c:369-375): dst = src, then each rect's four draw_line calls at 255, (x,y)-(x+w,y),
 * (x,y+h)-(x+w,y+h), (x,y)-(x,y+h) and (x+w,y)-(x+w,y+h).  The unsigned sums are taken as int (two's complement) and
 * every pixel between an edge's two ends, both included, is drawn where it lies inside the frame; so an edge costs at
 * most one frame row or column whatever the coordinates. */
int gs_b200_draw_rects_batch(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n,
                             const struct gs_rect *rects, const unsigned *counts, unsigned stride, gs_b200_stream s);

/* The orb verb's picture (nanomagick.c:313-343).  Output frame f is (tw + w) x max(th, h) at
 * dst + f * (tw + w) * max(th, h): zero, the template at (0, 0) and frame f at (tw, 0).  Frame f's first
 * c = min(mcounts[f], mstride) matches are ordered by the verb's exchange sort (for i, for j > i: if d[j] < d[i] swap,
 * which is not stable) and the first min(top, c) are drawn with the verb's draw_line, from kps1[idx1] to
 * kps2[idx2] + (tw, 0), at 255.  Frame f's lists start at kps1 + f * stride1 (stride1 == 0: one template list for every
 * frame), kps2 + f * stride2 and matches + f * mstride.  A match whose keypoint lies outside its own image, or whose
 * index is not below a non-zero stride, is skipped.  A frame without matches gets the side-by-side picture without
 * lines.  dst may not overlap src or tmpl.  mstride <= 16384, else cudaErrorInvalidValue. */
int gs_b200_draw_matches_batch(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n,
                               const uint8_t *tmpl, unsigned tw, unsigned th,
                               const struct gs_keypoint *kps1, unsigned stride1,
                               const struct gs_keypoint *kps2, unsigned stride2,
                               const struct gs_match *matches, const unsigned *mcounts, unsigned mstride,
                               unsigned top, gs_b200_stream s);

/* the text of the calling thread's last error of this library */
const char *gs_b200_draw_last_error(void);

#ifdef __cplusplus
}
#endif

#endif /* GRAYSKULL_DRAW_H */
