/*
 * grayskull_b200.h -- batched, device-resident C ABI of libgrayskull_b200.so.
 *
 * The reference API (include/grayskull.h, reference grayskull.h) is one-image-per-call and
 * synchronous.  A GPU is only kept busy by frame batches, so every hot-path op also has a
 * `_batch` entry point here: n frames stored back to back (frame f of a w x h image starts at
 * base + f*w*h, pitch = w, exactly n copies of the reference's dense row-major layout,
 * grayskull.h:144,147), all pointers DEVICE pointers, work enqueued on `stream`
 * (a cudaStream_t passed as void*; NULL = legacy default stream) and NOT synchronised.
 * The single-image gs_* functions are the n == 1 case plus staging and a stream sync.
 *
 * Plain C99: only pointers, sizes and PODs cross this boundary.  Every function returns 0 on
 * success or a non-zero cudaError_t value (gs_b200_last_error() gives the text).  Argument
 * contract violations (the reference's gs_assert conditions, cited per function) abort with
 * the reference's "Assertion failed: ..." message, like the reference does.
 */
#ifndef GRAYSKULL_B200_H
#define GRAYSKULL_B200_H

#include <stddef.h>
#include <stdint.h>

#include "grayskull.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef void *gs_b200_stream; /* cudaStream_t */

/* ---- runtime -------------------------------------------------------------------------- */
int gs_b200_device_count(void);
int gs_b200_set_device(int device); /* one process per GPU: call once with LOCAL_RANK */
const char *gs_b200_last_error(void);
const char *gs_b200_version(void);
/* 1 if the fast (TMA-tiled) kernels are used for this geometry, 0 if the generic kernels */
int gs_b200_uses_tma(unsigned w, unsigned h, const void *ptr);
/* testing hook: 1 = always take the generic (non-TMA) kernels; same as GS_B200_FORCE_GENERIC=1 */
void gs_b200_force_generic(int on);
/* number of kernel launches issued by this library since process start (bench bookkeeping) */
unsigned long long gs_b200_launch_count(void);

/* memory helpers so C99 callers need no CUDA headers */
void *gs_b200_malloc(size_t bytes);      /* device memory (cudaMalloc) */
void gs_b200_free(void *p);
void *gs_b200_malloc_host(size_t bytes); /* pinned host memory */
void gs_b200_free_host(void *p);
int gs_b200_memcpy_h2d(void *dst, const void *src, size_t bytes, gs_b200_stream s);
int gs_b200_memcpy_d2h(void *dst, const void *src, size_t bytes, gs_b200_stream s);
int gs_b200_memset(void *dst, int value, size_t bytes, gs_b200_stream s);
int gs_b200_stream_sync(gs_b200_stream s);
/* gs_alloc/gs_free look-alikes backed by managed memory (zero-filled like calloc): images
 * from these are device-resident for the gs_* calls and still readable by host code. */
struct gs_image gs_b200_alloc(unsigned w, unsigned h);
void gs_b200_image_free(struct gs_image img);

/* ---- stencils (2 B/pixel of compulsory HBM traffic each) ------------------------------- */
/* gs_blur, reference grayskull.h:268-283 */
int gs_b200_blur_batch(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n,
                       unsigned radius, gs_b200_stream s);
/* gs_adaptive_threshold, reference grayskull.h:230-247 */
int gs_b200_adaptive_threshold_batch(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h,
                                     unsigned n, unsigned radius, int c, gs_b200_stream s);
/* gs_sobel, reference grayskull.h:306-320 (dst border bytes are left untouched) */
int gs_b200_sobel_batch(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n,
                        gs_b200_stream s);
/* gs_blur(tmp, src, radius) followed by gs_sobel(dst, tmp) as ONE pass (reference grayskull.h:268-283 then
 * :306-320): bit-identical to the two calls, dst border bytes left untouched, the blurred intermediate never
 * written to memory -- 2 B/pixel of HBM traffic instead of 4 (BASELINE.json configs[1] is exactly this pair). */
int gs_b200_blur_sobel_batch(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n,
                             unsigned radius, gs_b200_stream s);
/* gs_erode / gs_dilate, reference grayskull.h:285-304 */
int gs_b200_erode_batch(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n,
                        gs_b200_stream s);
int gs_b200_dilate_batch(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n,
                         gs_b200_stream s);
/* `iters` passes of gs_erode / gs_dilate (reference grayskull.h:285-304) in one call, as the reference CLI's
 * `morph <op> <n>` verb (nanomagick.c:110-135) applies them: bit-identical to `iters` ping-ponged calls of
 * gs_b200_erode_batch / gs_b200_dilate_batch, i.e. the min (max) over the in-image pixels of the
 * (2*iters+1) x (2*iters+1) square.  Every dst byte is written; iters == 0 copies src to dst.  dst must not alias
 * src.  The arithmetic per pixel grows at most logarithmically with iters (DESIGN.md §3, §6 for times).  With iters
 * above 16, or geometry the TMA kernels cannot take, it uses library workspace of at most 256 MiB (or one frame, if
 * a frame is larger). */
int gs_b200_erode_n_batch(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n, unsigned iters,
                          gs_b200_stream s);
int gs_b200_dilate_n_batch(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n, unsigned iters,
                           gs_b200_stream s);

/* ---- resampling ------------------------------------------------------------------------- */
/* gs_resize, reference grayskull.h:171-187 */
int gs_b200_resize_batch(uint8_t *dst, unsigned dw, unsigned dh, const uint8_t *src, unsigned sw,
                         unsigned sh, unsigned n, gs_b200_stream s);
/* gs_downsample, reference grayskull.h:189-197 (dst is (sw/2) x (sh/2)) */
int gs_b200_downsample_batch(uint8_t *dst, const uint8_t *src, unsigned sw, unsigned sh,
                             unsigned n, gs_b200_stream s);

/* ---- integral image --------------------------------------------------------------------- */
/* gs_integral, reference grayskull.h:744-752; ii holds n tables of w*h uint32 */
int gs_b200_integral_batch(uint32_t *ii, const uint8_t *src, unsigned w, unsigned h, unsigned n,
                           gs_b200_stream s);

/* ---- histogram / Otsu / global threshold (SURVEY.md 8f N2) ------------------------------- */
/* gs_histogram, reference grayskull.h:199-203; hist holds n tables of 256 unsigned counts */
int gs_b200_histogram_batch(unsigned *hist, const uint8_t *src, unsigned w, unsigned h, unsigned n,
                            gs_b200_stream s);
/* gs_otsu_threshold, reference grayskull.h:205-224: thresh[f] for each frame.  hist (n x 256) receives the
 * histograms; NULL uses library workspace. */
int gs_b200_otsu_threshold_batch(uint8_t *thresh, unsigned *hist, const uint8_t *src, unsigned w,
                                 unsigned h, unsigned n, gs_b200_stream s);
/* gs_threshold, reference grayskull.h:226-229, in place, one threshold for every frame */
int gs_b200_threshold_batch(uint8_t *img, unsigned w, unsigned h, unsigned n, unsigned thresh,
                            gs_b200_stream s);
/* same with a device-resident per-frame threshold (uint8_t)(thresh[f] + offset), e.g. Otsu's output
 * (+10 in the reference's document scanner, nanomagick.c:191) without a host round trip */
int gs_b200_threshold_each_batch(uint8_t *img, unsigned w, unsigned h, unsigned n, const uint8_t *thresh,
                                 int offset, gs_b200_stream s);

/* ---- generic convolution / template matching (SURVEY.md 8f N3) --------------------------- */
/* gs_filter, reference grayskull.h:255-266.  kernel: kw*kh int8 weights in HOST memory (row major; they are
 * call parameters, not image data); NULL or a zero size behaves like the reference's invalid kernel image
 * (every sum is 0). */
int gs_b200_filter_batch(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n,
                         const int8_t *kernel, unsigned kw, unsigned kh, unsigned norm, gs_b200_stream s);
/* gs_match_template, reference grayskull.h:705-723: one device-resident tw x th template against n frames;
 * result holds n maps of (w-tw+1) x (h-th+1) bytes */
int gs_b200_match_template_batch(uint8_t *result, const uint8_t *img, unsigned w, unsigned h, unsigned n,
                                 const uint8_t *tmpl, unsigned tw, unsigned th, gs_b200_stream s);
/* gs_find_best_match, reference grayskull.h:725-738, per result map */
int gs_b200_find_best_match_batch(struct gs_point *best, const uint8_t *result, unsigned rw, unsigned rh,
                                  unsigned n, gs_b200_stream s);

/* ---- connected components / perspective warp (SURVEY.md 8f N4) ---------------------------------- */
/* gs_blobs, reference grayskull.h:333-405, over n frames.  labels: n*w*h gs_label; blobs: n x nblobs records, frame
 * f's first counts[f] entries valid (label order), the rest untouched; counts: n unsigned.  nblobs <= 65534. */
int gs_b200_blobs_batch(const uint8_t *img, unsigned w, unsigned h, unsigned n, gs_label *labels,
                        struct gs_blob *blobs, unsigned *counts, unsigned nblobs, gs_b200_stream s);
/* gs_blob_corners, reference grayskull.h:407-421: `blob` and `corners` (4 points: tl, tr, br, bl) in DEVICE memory */
int gs_b200_blob_corners(const uint8_t *img, unsigned w, unsigned h, const gs_label *labels,
                         const struct gs_blob *blob, struct gs_point *corners, gs_b200_stream s);
/* gs_perspective_correct, reference grayskull.h:423-444, n source frames -> n dst frames.  per_frame == 0: corners =
 * 4 points in HOST memory used for every frame; per_frame != 0: n x 4 points in DEVICE memory (e.g. written by
 * gs_b200_blob_corners) */
int gs_b200_perspective_correct_batch(uint8_t *dst, unsigned dw, unsigned dh, const uint8_t *src, unsigned sw,
                                      unsigned sh, unsigned n, const struct gs_point *corners, int per_frame,
                                      gs_b200_stream s);

/* ---- FAST / ORB ------------------------------------------------------------------------- */
/* gs_fast, reference grayskull.h:482-534.  scoremap: n maps of w*h bytes, only the interior
 * [3,w-4]x[3,h-4] is written and the untouched ring takes part in the NMS exactly as in the
 * reference.  kps: n x nkps records (frame f's start at kps + f*nkps); counts: n unsigned. */
int gs_b200_fast_batch(const uint8_t *src, unsigned w, unsigned h, unsigned n, uint8_t *scoremap,
                       struct gs_keypoint *kps, unsigned *counts, unsigned nkps,
                       unsigned threshold, gs_b200_stream s);
/* gs_orb_extract, reference grayskull.h:651-669 (FAST cap = min(4*nkps, 5000) as there).
 * Orientation/BRIEF trigonometry: see gs_b200_set_trig_mode. */
int gs_b200_orb_extract_batch(const uint8_t *src, unsigned w, unsigned h, unsigned n,
                              uint8_t *scoremap, struct gs_keypoint *kps, unsigned *counts,
                              unsigned nkps, unsigned threshold, gs_b200_stream s);
/* 0 (default): atan2f / sinf evaluated on the device with the same algorithm and constants as
 *              glibc 2.39's float routines (bit-identical angles and descriptors);
 * 1:           CUDA libdevice atan2f/sinf (angle within 1e-5 of the reference, descriptor bits
 *              may differ where a rotated offset sits on an integer boundary). */
void gs_b200_set_trig_mode(int mode);
/* Mode 0 restates ONE libm (glibc 2.39); the reference calls the host's.  The first ORB call compares the device
 * routines with this host's sinf/atan2f on 8192 samples and warns once on stderr if they differ.  This returns
 * the number of differing samples (0 = this host's libm agrees; runs the check if it has not run yet; -1 = the
 * check could not run). */
int gs_b200_trig_selfcheck(void);

/* gs_match_orb, reference grayskull.h:680-699, over npairs (set1, set2) pairs.  Pair p's sets start
 * at kps1 + p*stride1 / kps2 + p*stride2 and hold n1[p] / n2[p] keypoints (e.g. the output layout of
 * gs_b200_orb_extract_batch: stride = nkps, n = counts); matches: npairs x max_matches records. */
int gs_b200_match_orb_batch(const struct gs_keypoint *kps1, const unsigned *n1, unsigned stride1,
                            const struct gs_keypoint *kps2, const unsigned *n2, unsigned stride2,
                            unsigned npairs, struct gs_match *matches, unsigned *counts,
                            unsigned max_matches, float max_distance, gs_b200_stream s);

/* ---- LBP cascade ------------------------------------------------------------------------ */
/* gs_lbp_detect, reference grayskull.h:815-835, over n integral images (device, n*iw*ih
 * uint32).  `c` is a HOST struct (its tables are uploaded once and cached by content).
 * rects: n x max_rects records; counts: n unsigned (each min(hits, max_rects), rects in the
 * reference's (scale, y, x) order). */
int gs_b200_lbp_detect_batch(const struct gs_lbp_cascade *c, const uint32_t *ii, unsigned iw,
                             unsigned ih, unsigned n, struct gs_rect *rects, unsigned *counts,
                             unsigned max_rects, float scale_factor, float min_scale,
                             float max_scale, int step, gs_b200_stream s);
/* number of windows gs_lbp_detect visits for this geometry (the windows/s denominator) */
unsigned long long gs_b200_lbp_window_count(const struct gs_lbp_cascade *c, unsigned iw,
                                            unsigned ih, float scale_factor, float min_scale,
                                            float max_scale, int step);

#ifdef __cplusplus
}
#endif

#endif /* GRAYSKULL_B200_H */
