/*
 * grayskull_corners.h -- the largest-blob pick and gs_blob_corners over frame batches on the device, in the companion
 * library libgrayskull_corners.so (link -lgrayskull_corners; it does not need libgrayskull_b200.so).  With
 * gs_b200_blobs_batch and gs_b200_perspective_correct_batch(per_frame = 1) they keep the reference's document scanner
 * on the device from the first launch to the warped frames, and with the contour calls the wasm demo's largest-blob
 * contour.
 *
 * This header's name deliberately does not match grayskull_b200*.h: the main library's headers are the set whose
 * declarations libgrayskull_b200.so exports, and these calls live in their own library.
 *
 * Conventions are grayskull_contour.h's: DEVICE pointers, n frames of w x h back to back, work enqueued on `s` and not
 * synchronised, 0 or a cudaError_t returned (gs_b200_corners_last_error() gives the text), 64-bit offsets; batches
 * above 65535 frames and frames taller than 65535 row tiles run as any other.  A missing pointer or an empty frame
 * aborts with the reference's "Assertion failed: ..." message; n == 0 returns 0 and does nothing.  The calls allocate
 * nothing and synchronise nothing, so they can be captured into a CUDA graph.  In every list, frame f's records start
 * at f * stride and frame f uses its first min(counts[f], stride) of them; counts == NULL means all `stride`.
 */
#ifndef GRAYSKULL_CORNERS_H
#define GRAYSKULL_CORNERS_H

#include "grayskull_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The largest-blob rule of the reference's document scanner (nanomagick.c:196-199) and of the wasm demo
 * (grayskull.c:285-295): over frame f's c = min(counts[f], stride) records, largest = 0, then for i = 1 .. c-1
 * `if (blobs[i].area > blobs[largest].area) largest = i` (strict >, so the first record wins ties).
 *   pick[f]   = that record, all 32 bytes as they are; when c == 0, the record gs_blobs initialises every slot to
 *               (grayskull.h:337-338): {label 0, area 0, box {UINT_MAX, UINT_MAX, 0, 0}, centroid {0, 0}}, which is
 *               what the scan verb's blobs[0] holds for a frame without blobs
 *   pcount[f] = c > 0 && pick[f].area >= min_area   (min_area 0: the scan verb; 100: the demo, grayskull.c:295)
 * pcount may be NULL.  pick + pcount form a list with stride 1, in the layout the corners, contour-start, trace and
 * draw calls take.  stride == 0 makes every list empty. */
int gs_b200_largest_blob_batch(const struct gs_blob *blobs, const unsigned *counts, unsigned stride, unsigned n,
                               unsigned min_area, struct gs_blob *pick, unsigned *pcount, gs_b200_stream s);

/* gs_blob_corners (grayskull.h:404-421) for every record k < min(counts[f], stride) of frame f, against frame f's
 * img and labels: exactly what consecutive gs_blob_corners(img_f, labels_f, &blobs[f*stride + k], c) calls write,
 * in tl, tr, br, bl order at corners + 4 * (f * stride + k).  Records past the count are not written.  The same
 * contract as gs_b200_blob_corners: exact for pixels with x + y < 2^31, w * h < 2^32 - 1.  The call keeps 64-bit keys
 * in the output slots while it runs, so `corners` must be 8-byte aligned (every record boundary of a cudaMalloc'ed
 * list is); otherwise it returns cudaErrorInvalidValue.  stride == 0 writes nothing. */
int gs_b200_blob_corners_batch(const uint8_t *img, unsigned w, unsigned h, unsigned n, const gs_label *labels,
                               const struct gs_blob *blobs, const unsigned *counts, unsigned stride,
                               struct gs_point *corners, gs_b200_stream s);

/* the text of the calling thread's last error of this library */
const char *gs_b200_corners_last_error(void);

#ifdef __cplusplus
}
#endif

#endif /* GRAYSKULL_CORNERS_H */
