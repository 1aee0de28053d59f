/*
 * grayskull.h -- drop-in boundary header for the H100-native hot path.
 *
 * The reference library (zserge/grayskull) has no plugin registry: its boundary IS its
 * single header, every public function being declared GS_API (reference grayskull.h:7-9).
 * This header keeps that boundary -- the gs_* names, by-value `struct gs_image {w,h,data}`
 * arguments, and the error convention (gs_assert -> message + abort) -- and rebinds the
 * stencil / sliding-window hot path to libgrayskull_b200.so (hand-written sm_90a CUDA).
 *
 * Two ways to use it:
 *
 *  1. Overlay mode (what a maintainer of the reference would do): compile with
 *       -DGS_UPSTREAM_HEADER='"/path/to/upstream/grayskull.h"'
 *     The upstream header is included unchanged; its hot-path definitions are renamed
 *     gs_cpu_<op> (still callable, handy for A/B checks) and the gs_<op> names resolve to the
 *     extern "C" entry points below.  Everything else (crop, contour tracing, PGM I/O ...) stays
 *     the upstream CPU code, so test.c and examples/nanomagick/nanomagick.c build unmodified.
 *
 *  2. Stand-alone mode (no upstream tree available): this header provides the types, the
 *     inline helpers callers use directly (gs_valid/gs_get/gs_set/gs_for/gs_integral_sum,
 *     GS_MIN/GS_MAX, gs_assert, gs_alloc/gs_free) and the hot-path prototypes only.
 *
 * Each prototype cites the reference definition it replaces (file:line in the reference).
 * Host code stays C99; the shim is a plain C ABI (pointers, sizes, PODs).
 */
#ifndef GRAYSKULL_B200_DROPIN_H
#define GRAYSKULL_B200_DROPIN_H

#ifdef GS_UPSTREAM_HEADER
/* ---- overlay mode ------------------------------------------------------------------- */
#define gs_blur gs_cpu_blur
#define gs_sobel gs_cpu_sobel
#define gs_erode gs_cpu_erode
#define gs_dilate gs_cpu_dilate
#define gs_adaptive_threshold gs_cpu_adaptive_threshold
#define gs_resize gs_cpu_resize
#define gs_downsample gs_cpu_downsample
#define gs_integral gs_cpu_integral
#define gs_fast gs_cpu_fast
#define gs_compute_orientation gs_cpu_compute_orientation
#define gs_brief_descriptor gs_cpu_brief_descriptor
#define gs_orb_extract gs_cpu_orb_extract
#define gs_lbp_window gs_cpu_lbp_window
#define gs_lbp_detect gs_cpu_lbp_detect
#define gs_match_orb gs_cpu_match_orb
#define gs_histogram gs_cpu_histogram
#define gs_otsu_threshold gs_cpu_otsu_threshold
#define gs_threshold gs_cpu_threshold
#define gs_filter gs_cpu_filter
#define gs_match_template gs_cpu_match_template
#define gs_find_best_match gs_cpu_find_best_match
#define gs_blobs gs_cpu_blobs
#define gs_blob_corners gs_cpu_blob_corners
#define gs_perspective_correct gs_cpu_perspective_correct
#include GS_UPSTREAM_HEADER
#undef gs_blur
#undef gs_sobel
#undef gs_erode
#undef gs_dilate
#undef gs_adaptive_threshold
#undef gs_resize
#undef gs_downsample
#undef gs_integral
#undef gs_fast
#undef gs_compute_orientation
#undef gs_brief_descriptor
#undef gs_orb_extract
#undef gs_lbp_window
#undef gs_lbp_detect
#undef gs_match_orb
#undef gs_histogram
#undef gs_otsu_threshold
#undef gs_threshold
#undef gs_filter
#undef gs_match_template
#undef gs_find_best_match
#undef gs_blobs
#undef gs_blob_corners
#undef gs_perspective_correct

#else
/* ---- stand-alone mode --------------------------------------------------------------- */
#include <limits.h>
#include <stdint.h>

#ifndef GS_NO_STDLIB
#include <stdio.h>
#include <stdlib.h>
#endif

#define GS_MIN(a, b) ((a) < (b) ? (a) : (b))
#define GS_MAX(a, b) ((a) > (b) ? (a) : (b))

/* Layouts are ABI: they must match the reference byte for byte (grayskull.h:14-64). */
struct gs_image {
  unsigned w, h;
  uint8_t *data;
};
struct gs_rect {
  unsigned x, y, w, h;
};
struct gs_point {
  unsigned x, y;
};
typedef uint16_t gs_label;
struct gs_blob {
  gs_label label;
  unsigned area;
  struct gs_rect box;
  struct gs_point centroid;
};
struct gs_contour { /* traced on the device by include/grayskull_contour.h */
  struct gs_rect box;
  struct gs_point start;
  unsigned length;
};
struct gs_keypoint {
  struct gs_point pt;
  unsigned response;
  float angle;
  uint32_t descriptor[8];
};
struct gs_match {
  unsigned idx1, idx2;
  unsigned distance;
};
struct gs_lbp_cascade {
  uint16_t window_w, window_h;
  uint16_t nfeatures, nweaks, nstages;
  const int8_t *features;           /* nfeatures x {x, y, w, h} of one LBP cell */
  const uint16_t *weak_feature_idx; /* per weak classifier */
  const float *weak_left_val, *weak_right_val;
  const uint16_t *weak_subset_offset, *weak_num_subsets;
  const int32_t *subsets;           /* 256-bit LUT per weak (8 words) */
  const uint16_t *stage_weak_start, *stage_nweaks;
  const float *stage_threshold;
};

static inline int gs_valid(struct gs_image img) { return img.data && img.w > 0 && img.h > 0; }

#ifdef GS_NO_STDLIB
#define gs_assert(cond)
#else
#define gs_assert(cond)                               \
  if (!(cond)) {                                      \
    fprintf(stderr, "Assertion failed: %s\n", #cond); \
    abort();                                          \
  }
/* zero-filled, like the reference (callers rely on it for the sobel border and the FAST
 * score-map ring, e.g. nanomagick.c:139-140,228-229) */
static inline struct gs_image gs_alloc(unsigned w, unsigned h) {
  struct gs_image img = {0, 0, NULL};
  if (w == 0 || h == 0) return img;
  img.data = (uint8_t *)calloc((size_t)w * h, 1);
  if (img.data) img.w = w, img.h = h;
  return img;
}
static inline void gs_free(struct gs_image img) { free(img.data); }

/* Binary PGM (P5, maxval 255) I/O, "-" = stdin / stdout -- the reference's on-disk format
 * (grayskull.h:111-136).  Header tokens may be separated by any white space; '#' comments are skipped. */
static inline int gs__pgm_token(FILE *f, unsigned *out) {
  int c = fgetc(f);
  unsigned v = 0, digits = 0;
  while (c == ' ' || c == '\t' || c == '\n' || c == '\r' || c == '#') {
    if (c == '#')
      while (c != '\n' && c != EOF) c = fgetc(f);
    else
      c = fgetc(f);
  }
  while (c >= '0' && c <= '9') v = v * 10u + (unsigned)(c - '0'), digits++, c = fgetc(f);
  *out = v;
  return digits > 0 && digits < 10; /* the single white-space byte after the token has been consumed */
}
static inline struct gs_image gs_read_pgm(const char *path) {
  struct gs_image img = {0, 0, NULL};
  unsigned w = 0, h = 0, maxval = 0;
  FILE *f = (path[0] == '-' && !path[1]) ? stdin : fopen(path, "rb");
  if (!f) return img;
  if (fgetc(f) == 'P' && fgetc(f) == '5' && gs__pgm_token(f, &w) && gs__pgm_token(f, &h) &&
      gs__pgm_token(f, &maxval) && maxval == 255) {
    img = gs_alloc(w, h);
    if (img.data && fread(img.data, 1, (size_t)w * h, f) != (size_t)w * h) {
      gs_free(img);
      img.w = img.h = 0, img.data = NULL;
    }
  }
  if (f != stdin) fclose(f);
  return img;
}
static inline int gs_write_pgm(struct gs_image img, const char *path) {
  FILE *f;
  size_t n;
  if (!gs_valid(img)) return -1;
  f = (path[0] == '-' && !path[1]) ? stdout : fopen(path, "wb");
  if (!f) return -1;
  fprintf(f, "P5\n%u %u\n255\n", img.w, img.h);
  n = fwrite(img.data, 1, (size_t)img.w * img.h, f);
  if (f != stdout) fclose(f);
  else fflush(f);
  return n == (size_t)img.w * img.h ? 0 : -1;
}
#endif

#define gs_for(img, x, y)                \
  for (unsigned y = 0; y < (img).h; y++) \
    for (unsigned x = 0; x < (img).w; x++)

/* out-of-bounds read -> 0, out-of-bounds write -> dropped (reference grayskull.h:143-148) */
static inline uint8_t gs_get(struct gs_image img, unsigned x, unsigned y) {
  return (gs_valid(img) && x < img.w && y < img.h) ? img.data[y * img.w + x] : 0;
}
static inline void gs_set(struct gs_image img, unsigned x, unsigned y, uint8_t value) {
  if (gs_valid(img) && x < img.w && y < img.h) img.data[y * img.w + x] = value;
}

/* preset 3x3 kernels for gs_filter: int8 weights stored in a gs_image, with the norm to pass alongside
 * (reference grayskull.h:249-253) */
#define gs_sharpen ((struct gs_image){3, 3, (uint8_t[]){0, -1, 0, -1, 5, -1, 0, -1, 0}})        /* norm 1 */
#define gs_emboss ((struct gs_image){3, 3, (uint8_t[]){-2, -1, 0, -1, 1, 1, 0, 1, 2}})          /* norm 1 */
#define gs_blur_box ((struct gs_image){3, 3, (uint8_t[]){1, 1, 1, 1, 1, 1, 1, 1, 1}})           /* norm 9 */
#define gs_blur_gaussian ((struct gs_image){3, 3, (uint8_t[]){1, 2, 1, 2, 4, 2, 1, 2, 1}})      /* norm 16 */

/* popcount of the xor of two 256-bit descriptors (reference grayskull.h:671-678) */
static inline unsigned gs_hamming_distance(const uint32_t desc1[8], const uint32_t desc2[8]) {
  unsigned dist = 0;
  for (int i = 0; i < 8; i++) {
    uint32_t v = desc1[i] ^ desc2[i];
    for (; v; v &= v - 1) dist++;
  }
  return dist;
}

/* inclusive box sum over [x, x+w-1] x [y, y+h-1] of a gs_integral table (grayskull.h:754-763) */
static inline uint32_t gs_integral_sum(const unsigned *ii, unsigned iw, unsigned x, unsigned y,
                                       unsigned w, unsigned h) {
  unsigned xr = x + w - 1, yb = y + h - 1;
  unsigned above_left = (x && y) ? ii[(y - 1) * iw + (x - 1)] : 0;
  unsigned above = y ? ii[(y - 1) * iw + xr] : 0;
  unsigned left = x ? ii[yb * iw + (x - 1)] : 0;
  gs_assert(ii && iw > 0 && x + w <= iw);
  return ii[yb * iw + xr] + above_left - above - left;
}
#endif /* GS_UPSTREAM_HEADER */

/* ---- the hot path: extern "C" entry points of libgrayskull_b200.so -------------------- */
#ifdef __cplusplus
extern "C" {
#endif

/* Pointer kinds: every image / table pointer may be device, managed or plain host memory.
 * Device and managed pointers run in place; host pointers are staged through the library's
 * device workspace (correct, PCIe-bound).  All calls below are synchronous: on return the
 * results are visible through the pointers that were passed in.  dst/src aliasing is not
 * supported for the stencil ops (no reference caller does it either). */

/* box mean over the border-clipped (2r+1)^2 window, sum / count -- grayskull.h:268-283 */
void gs_blur(struct gs_image dst, struct gs_image src, unsigned radius);
/* 3x3 Sobel, (|gx|+|gy|)/2 clamped, interior only, dst border untouched -- grayskull.h:306-320 */
void gs_sobel(struct gs_image dst, struct gs_image src);
/* 3x3 min / max over in-bounds neighbours -- grayskull.h:285-304 */
void gs_erode(struct gs_image dst, struct gs_image src);
void gs_dilate(struct gs_image dst, struct gs_image src);
/* src > clipped-box-mean - c ? 255 : 0 -- grayskull.h:230-247 */
void gs_adaptive_threshold(struct gs_image dst, struct gs_image src, unsigned radius, int c);
/* pixel-centre bilinear resize, fp32 evaluation order preserved -- grayskull.h:171-187 */
void gs_resize(struct gs_image dst, struct gs_image src);
/* 2x2 mean, dst must be src/2 -- grayskull.h:189-197 */
void gs_downsample(struct gs_image dst, struct gs_image src);
/* inclusive u32 summed-area table, w*h entries -- grayskull.h:744-752 */
void gs_integral(struct gs_image src, unsigned *ii);
/* FAST-9 score map + 3x3 NMS, raster-ordered keypoints capped at nkps -- grayskull.h:482-534 */
unsigned gs_fast(struct gs_image img, struct gs_image scoremap, struct gs_keypoint *kps,
                 unsigned nkps, unsigned threshold);
/* intensity-centroid angle over the radius-r disc -- grayskull.h:608-621 */
float gs_compute_orientation(struct gs_image img, unsigned x, unsigned y, unsigned r);
/* rotated BRIEF-256 of one keypoint (kp->pt, kp->angle in; kp->descriptor out) -- :623-637 */
void gs_brief_descriptor(struct gs_image img, struct gs_keypoint *kp);
/* FAST -> stable sort by response -> 15 px margin filter -> angle + BRIEF -- grayskull.h:651-669 */
unsigned gs_orb_extract(struct gs_image img, struct gs_keypoint *kps, unsigned nkps,
                        unsigned threshold, uint8_t *scoremap_buffer);
/* one cascade window -- grayskull.h:790-813 */
unsigned gs_lbp_window(const struct gs_lbp_cascade *c, const unsigned *ii, unsigned iw,
                       unsigned ih, int x, int y, float scale);
/* multi-scale sliding window, (scale, y, x)-ordered rects capped at max_rects -- :815-835 */
unsigned gs_lbp_detect(const struct gs_lbp_cascade *c, const unsigned *ii, unsigned iw,
                       unsigned ih, struct gs_rect *rects, unsigned max_rects,
                       float scale_factor, float min_scale, float max_scale, int step);

/* brute-force Hamming matching of ORB descriptors with the 0.8 ratio test, matches in query order
 * capped at max_matches -- grayskull.h:680-699 (first "next" item after the hot path, SURVEY.md 8f) */
unsigned gs_match_orb(const struct gs_keypoint *kps1, unsigned n1, const struct gs_keypoint *kps2, unsigned n2,
                      struct gs_match *matches, unsigned max_matches, float max_distance);

/* 256-bin histogram of all w*h pixels -- grayskull.h:199-203 (SURVEY.md 8f N2) */
void gs_histogram(struct gs_image img, unsigned hist[256]);
/* Otsu's threshold from that histogram, the reference's fp32 evaluation order -- grayskull.h:205-224 */
uint8_t gs_otsu_threshold(struct gs_image img);
/* in place: pixel > thresh ? 255 : 0 -- grayskull.h:226-229 */
void gs_threshold(struct gs_image img, uint8_t thresh);

/* kw x kh int8 convolution with zero padding, (unsigned)sum / norm clamped to 0..255 -- grayskull.h:255-266
 * (SURVEY.md 8f N3) */
void gs_filter(struct gs_image dst, struct gs_image src, struct gs_image kernel, unsigned norm);
/* dense sum of squared differences, 255 - min(255, ssd*255 / (tw*th*255^2)) -- grayskull.h:705-723 */
void gs_match_template(struct gs_image img, struct gs_image tmpl, struct gs_image result);
/* first strict maximum in raster order -- grayskull.h:725-738 */
struct gs_point gs_find_best_match(struct gs_image result);

/* 4-connected components of the pixels >= 128 -- grayskull.h:333-405 (SURVEY.md 8f N4).  labels: w*h gs_label, 0 =
 * background; a component's label is the reference's: the rank (from 1) of its raster-first pixel among the
 * pixels that start a run with no foreground pixel above them.  blobs[0..return) hold the components in label
 * order (label, area, box {x, y, w, h}, centroid = coordinate sums / area in unsigned arithmetic); entries past
 * the returned count are unspecified (the reference leaves first-pass leftovers there).  Running out of labels
 * (more than nblobs run starts) behaves as in the reference: later pixels are labelled only through a labelled
 * left / upper neighbour.  nblobs <= 65534. */
unsigned gs_blobs(struct gs_image img, gs_label *labels, struct gs_blob *blobs, unsigned nblobs);
/* extreme points of one blob in x+y / x-y, first in raster order on ties -- grayskull.h:407-421 */
void gs_blob_corners(struct gs_image img, gs_label *labels, struct gs_blob *b, struct gs_point c[4]);
/* bilinear warp of the quad c[0..3] (tl, tr, br, bl) onto dst, fp32 order of the reference -- grayskull.h:423-444 */
void gs_perspective_correct(struct gs_image dst, struct gs_image src, struct gs_point c[4]);

#ifdef __cplusplus
}
#endif

#endif /* GRAYSKULL_B200_DROPIN_H */
