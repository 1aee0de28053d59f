/*
 * grayskull_group.h -- neighbour-counted grouping of each frame's raw LBP detections on the device, in the companion
 * library libgrayskull_group.so (link -lgrayskull_group; it does not need libgrayskull_b200.so).  It reads the rect
 * lists gs_b200_lbp_detect_batch writes and writes lists in the same layout, so the ROI, draw and host code take its
 * output unchanged: one box per face instead of every accepted window.
 *
 * This header's name deliberately does not match grayskull_b200*.h: the main library's headers are the set whose
 * declarations libgrayskull_b200.so exports, and these calls live in their own library.
 *
 * Conventions are grayskull_contour.h's: DEVICE pointers, work enqueued on `s` and not synchronised, 0 or a cudaError_t
 * returned (gs_b200_group_last_error() gives the text), 64-bit offsets; batches above 65535 frames run as any other.  A
 * missing pointer aborts with the reference's "Assertion failed: ..." message; n == 0 returns 0 and does nothing.  The
 * calls allocate nothing and synchronise nothing, so they can be captured into a CUDA graph.  Frame f's input records
 * start at rects + f * stride and it uses the first c = min(counts[f], stride) of them; counts == NULL means all
 * `stride`.
 */
#ifndef GRAYSKULL_GROUP_H
#define GRAYSKULL_GROUP_H

#include "grayskull_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Bytes of `work` that gs_b200_group_rects_batch needs to run n frames of `stride` records in one chunk. */
size_t gs_b200_group_rects_work_bytes(unsigned stride, unsigned n);

/* Groups each frame's records and keeps the groups with more than min_neighbors members, in the manner of
 * OpenCV's groupRectangles(rects, minNeighbors, eps).  The rule, with all integer arithmetic exact in 64 bits:
 *   1. records i and j are similar when |x_i - x_j|, |y_i - y_j|, |(x_i + w_i) - (x_j + w_j)| and
 *      |(y_i + h_i) - (y_j + h_j)| are each <= delta, delta = (eps * (double)(min(w_i, w_j) + min(h_i, h_j))) * 0.5
 *      in IEEE double, left to right, without FMA; each difference is compared as a double;
 *   2. groups are the transitive closure of similarity, numbered in order of their smallest record index;
 *   3. a group of m records with sums Sx, Sy, Sw, Sh has the rect rint((float)S * (1.0f / (float)m)) per field, in
 *      fp32, rounded half to even, clamped to [0, UINT_MAX], and the weight m;
 *   4. with K = min_neighbors, group i survives when m_i > K and no other group j with m_j > K contains it: x_i >=
 *      x_j - dx, y_i >= y_j - dy, x_i + w_i <= x_j + w_j + dx, y_i + h_i <= y_j + h_j + dy and (m_j > max(3, m_i) ||
 *      m_i < 3), where dx = rint((double)w_j * eps) and dy = rint((double)h_j * eps), half to even;
 *   5. the survivors, in group order, go to out + f * out_stride, the first min(survivors, out_stride) of them;
 *      out_counts[f] is that number and weights[f * out_stride + k] (weights may be NULL) the k-th one's m.  Slots
 *      past the count are not written.
 * K == 0 copies the first min(c, out_stride) records unchanged with weight 1.  stride == 0 or out_stride == 0 writes
 * out_counts[f] = 0 and nothing else.  `work` (any alignment) holds the per-frame state: with
 * gs_b200_group_rects_work_bytes(stride, n) bytes all frames run at once, with fewer the frames run in chunks of as
 * many as fit, one after another on `s`.  Fewer bytes than one frame needs, or an eps that is negative, NaN or
 * infinite, returns cudaErrorInvalidValue before anything is enqueued.  eps is a double so that 0.2 means the double
 * 0.2. */
int gs_b200_group_rects_batch(const struct gs_rect *rects, const unsigned *counts, unsigned stride, unsigned n,
                              unsigned min_neighbors, double eps, struct gs_rect *out, unsigned *weights,
                              unsigned *out_counts, unsigned out_stride, void *work, size_t work_bytes,
                              gs_b200_stream s);

/* the text of the calling thread's last error of this library */
const char *gs_b200_group_last_error(void);

#ifdef __cplusplus
}
#endif

#endif /* GRAYSKULL_GROUP_H */
