/*
 * gsb_magick -- batch image pipelines on the device-resident C ABI (SURVEY.md 8f N4: the caller side of
 * the hot path).  Plain C99 against include/grayskull.h (stand-alone mode) + include/grayskull_b200.h, linked against
 * libgrayskull_b200.so and, for the draw-* and faces stages, libgrayskull_draw.so (include/grayskull_draw.h), for
 * the contour stage libgrayskull_contour.so (include/grayskull_contour.h), for the contour and scan stages
 * libgrayskull_corners.so (include/grayskull_corners.h), for the faces-grouped stage libgrayskull_group.so
 * (include/grayskull_group.h), for the find stage libgrayskull_homography.so (include/grayskull_homography.h), and for
 * colour inputs libgrayskull_color.so (include/grayskull_color.h).
 *
 *   gsb_magick <pipeline> <out-prefix> in0.pgm|in0.ppm [in1 ...]
 *
 * All inputs (binary P5 PGM, or binary P6 PPM with maxval 255; all of one kind and one size) are read into ONE pinned
 * host batch, copied to the GPU once, taken through the pipeline without leaving the device (two ping-pong frame
 * batches), copied back once and written as <out-prefix>NNNN.pgm.  A P6 batch is first converted to gray on the device
 * by the wasm demo's rule (gs_b200_rgb_to_gray_batch, examples/wasm/grayskull.js:33-38); the outputs are gray P5.
 * "-" reads a P5 input from stdin.  Pipeline = comma-separated stages, arguments after ':'
 *   blur:R   sobel   erode[:N]   dilate[:N]   adaptive:R:C   threshold:T   threshold:otsu[+K]
 *   (erode:N / dilate:N are N passes of the 3x3 op in one call, gs_b200_erode_n_batch / gs_b200_dilate_n_batch)
 *   filter:sharpen|emboss|box|gaussian   downsample   resize:W:H
 *   crop:X:Y:W:H    (the reference's crop verb, nanomagick.c:69-77: gs_crop of one rectangle of every frame)
 *   keypoints:N:T   (prints the ORB keypoint count per frame; frames pass through unchanged)
 *   blobs:N         (prints the number of 4-connected components >= 128 per frame; frames pass through unchanged)
 *   draw-blobs:N    (the reference's blobs verb's picture, nanomagick.c:143-170: up to N blobs per frame, each box grown
 *                    by 2 px filled with 128, then 255 wherever the frame is > 128)
 *   draw-keypoints:N:T (the keypoints verb's picture, nanomagick.c:217-242: FAST at threshold T with cap 5000, then a
 *                    5-px cross of 255 at each of the N strongest keypoints)
 *   faces:N         (the faces verb's picture, nanomagick.c:347-376: LBP detection with the frontalface cascade, at most
 *                    100 rects, scales 1.0..4.0 by 1.2, N minimum neighbours, each rect's outline drawn at 255.  Runs at
 *                    any frame size; the verb refuses frames over 640x480)
 *   faces-grouped:S:K (faces as groups of windows rather than every window: LBP detection with the frontalface cascade,
 *                    at most 4096 rects, scales 1.0..4.0 by 1.2, scan step S; then gs_b200_group_rects_batch with
 *                    min_neighbors K and eps 0.2, and each group's outline drawn at 255; prints "frame F: R windows,
 *                    G faces")
 *   contour:N       (the reference's wasm demo's gs_detect_largest_blob_contour(src, N), examples/wasm/grayskull.c:
 *                    278-326, per frame: blobs of the frame with N records, the largest (the first on ties) when its
 *                    area is at least 100, its first label pixel in raster order as the start, then gs_trace_contour on
 *                    a zeroed visited map; prints "frame F: contour start X Y box X Y W H length L end
 *                    returned|open|cycle" or "frame F: no contour" and passes the frames through unchanged)
 *   scan:W:H        (the reference's document scanner, nanomagick.c:186-210, per frame on the device: blur 1 ->
 *                    Otsu + 10 threshold -> blobs -> corners of the largest blob -> perspective warp to W x H)
 *   orb:TEMPLATE.pgm (the reference's orb verb, nanomagick.c:292-311: pyramid ORB of the template and of every frame,
 *                    2500 keypoints, threshold 20, 3 levels, then gs_match_orb with at most 300 matches at distance
 *                    60; prints "frame F: Template: T keypoints, Scene: S keypoints, Matches: M" per frame and passes
 *                    the frames through unchanged.  The verb runs both extractions in one static 1 MiB buffer, so a
 *                    frame's score maps start with the bytes the template call left at their offsets; the stage
 *                    reproduces that.  When the template's or a frame's pyramid and score maps need more than 1 MiB
 *                    the verb overruns its buffer and its result is undefined; the stage then starts from zeroed maps.
 *                    The matches are not drawn.)
 *   draw-orb:TEMPLATE.pgm (all the orb stage does, printed line included, then the verb's picture, nanomagick.c:313-343:
 *                    (tw + w) x max(th, h), template and frame side by side, lines for the 15 best matches.  Like the
 *                    verb, a frame without matches gets no output file; gsb_magick says so on stderr)
 *   find:TEMPLATE.pgm:W:H (where the template lies in each frame: all the orb stage does, printed line included, then
 *                    gs_b200_find_homography_batch with 1024 hypotheses, seed 0 and a 3 px threshold, and
 *                    gs_b200_homography_quads_batch with at least 10 inliers -- choices of this tool, not reference
 *                    values --; prints "frame F: found, I inliers, quad x0 y0 x1 y1 x2 y2 x3 y3" or "frame F: not
 *                    found, I inliers", and warps each found quad to W x H with gs_b200_perspective_correct_batch, the
 *                    scan stage's bilinear quad warp.  A frame not found gets no output file.  W and H are the last two
 *                    fields, so the template path may hold ':')
 * e.g. the reference Makefile's lena chain:  blur:2,threshold:otsu,erode:2,dilate:2
 * Stage semantics are the reference's gs_* functions (same kernels as the drop-in gs_* entry points).
 */
#include <string.h>

#include "grayskull_b200_pyramid.h"
#include "grayskull_b200_roi.h"
#include "grayskull_color.h"
#include "grayskull_contour.h"
#include "grayskull_corners.h"
#include "grayskull_draw.h"
#include "grayskull_group.h"
#include "grayskull_homography.h"
#include "frontalface_cascade.h" /* generated by build.py from grayskull_b200/data/frontalface.npz */

#define DIE(...) (fprintf(stderr, "gsb_magick: " __VA_ARGS__), fprintf(stderr, "\n"), exit(1))
#define CK(call)                                                         \
  do {                                                                   \
    if ((call) != 0) DIE("%s failed: %s", #call, gs_b200_last_error());  \
  } while (0)
#define CKC(call)                                                                \
  do {                                                                           \
    if ((call) != 0) DIE("%s failed: %s", #call, gs_b200_contour_last_error());  \
  } while (0)
#define CKR(call)                                                                \
  do {                                                                           \
    if ((call) != 0) DIE("%s failed: %s", #call, gs_b200_corners_last_error());  \
  } while (0)
#define CKK(call)                                                              \
  do {                                                                         \
    if ((call) != 0) DIE("%s failed: %s", #call, gs_b200_color_last_error());  \
  } while (0)
#define CKG(call)                                                              \
  do {                                                                         \
    if ((call) != 0) DIE("%s failed: %s", #call, gs_b200_group_last_error());  \
  } while (0)
#define CKH(call)                                                                   \
  do {                                                                              \
    if ((call) != 0) DIE("%s failed: %s", #call, gs_b200_homography_last_error());  \
  } while (0)
#define CKD(call)                                                             \
  do {                                                                        \
    if ((call) != 0) DIE("%s failed: %s", #call, gs_b200_draw_last_error());  \
  } while (0)

/* frames that get no output file, and why: NO_MATCHES for the draw-orb stage's frames without matches, for which the
 * verb writes no picture; NOT_FOUND for the find stage's frames where the template was not found */
enum { NO_MATCHES = 1, NOT_FOUND = 2 };
static unsigned char *g_no_output;

static void no_output(unsigned f, unsigned n, unsigned char why) {
  if (!g_no_output) {
    g_no_output = (unsigned char *)calloc(n, 1);
    if (!g_no_output) DIE("allocation failed");
  }
  g_no_output[f] = why;
}

struct batch {
  uint8_t *dev;
  unsigned w, h, n;
};

static size_t frame_bytes(const struct batch *b) { return (size_t)b->w * b->h; }

static void ensure(struct batch *b, unsigned w, unsigned h, unsigned n, size_t *cap) {
  size_t need = (size_t)w * h * n;
  if (need > *cap) {
    if (b->dev) gs_b200_free(b->dev);
    b->dev = (uint8_t *)gs_b200_malloc(need);
    if (!b->dev) DIE("device allocation of %lu bytes failed", (unsigned long)need);
    *cap = need;
  }
  b->w = w, b->h = h, b->n = n;
}

/* bytes of pyramid levels 1..L-1 and of score maps 0..L-1 of one w x h image (nanomagick.c:255-270), and the offset
 * of level l's score map among the score maps */
static size_t pyr_bytes(unsigned w, unsigned h, unsigned L, size_t *maps, size_t off[4]) {
  size_t pyr = 0, sm = 0;
  unsigned l;
  for (l = 0; l < L; l++, w /= 2, h /= 2) {
    off[l] = sm;
    sm += (size_t)w * h;
    if (l) pyr += (size_t)w * h;
  }
  *maps = sm;
  return pyr;
}

/* what the orb stage leaves on the device for draw-orb and find: the template, its one keypoint list tk and its copy
 * per frame tks with the counts n1, frame f's keypoints, their counts scount and matches at stride ORB_NK / ORB_MM,
 * and the match counts (also on the host, hm) */
enum { ORB_NK = 2500, ORB_MM = 300 };
struct orb_out {
  struct gs_image tpl;
  uint8_t *tdev;
  struct gs_keypoint *tk, *tks, *sk;
  struct gs_match *matches;
  unsigned *n1, *scount, *mcount, *hm;
};

/* the orb stage (see the header comment): template as set 1 of every pair, frame f's keypoints as set 2 */
static void orb_run(const char *path, const struct batch *cur, struct orb_out *o) {
  enum { NK = ORB_NK, TH = 20, LV = 3, MM = ORB_MM };
  const size_t BUF = 1024 * 1024; /* nanomagick.c:299 */
  unsigned w = cur->w, h = cur->h, n = cur->n, f, l, tl, sl, ht, *tcount, *scount, *n1, *mcount, *hs, *hm, *h1;
  size_t tmaps, smaps, toff[4], soff[4], tpyr, spyr;
  struct gs_keypoint *tk, *tks, *sk, *htk;
  struct gs_match *matches;
  uint8_t *tdev, *tbuf, *spyrd, *ssm;
  int stale;
  struct gs_image tpl = gs_read_pgm(path);
  if (!gs_valid(tpl)) DIE("could not load template %s", path);
  tl = gs_b200_orb_pyramid_levels(tpl.w, tpl.h, LV);
  sl = gs_b200_orb_pyramid_levels(w, h, LV);
  tpyr = pyr_bytes(tpl.w, tpl.h, tl, &tmaps, toff);
  spyr = pyr_bytes(w, h, sl, &smaps, soff);
  stale = tpyr + tmaps <= BUF && spyr + smaps <= BUF;
  tdev = (uint8_t *)gs_b200_malloc((size_t)tpl.w * tpl.h);
  tbuf = (uint8_t *)gs_b200_malloc(tpyr + tmaps > BUF ? tpyr + tmaps : BUF);
  tk = (struct gs_keypoint *)gs_b200_malloc(sizeof(*tk) * NK);
  tks = (struct gs_keypoint *)gs_b200_malloc(sizeof(*tks) * NK * (size_t)n);
  tcount = (unsigned *)gs_b200_malloc(sizeof(unsigned));
  spyrd = spyr ? (uint8_t *)gs_b200_malloc(spyr * n) : NULL;
  ssm = (uint8_t *)gs_b200_malloc(smaps * n);
  sk = (struct gs_keypoint *)gs_b200_malloc(sizeof(*sk) * NK * (size_t)n);
  scount = (unsigned *)gs_b200_malloc(sizeof(unsigned) * n);
  n1 = (unsigned *)gs_b200_malloc(sizeof(unsigned) * n);
  matches = (struct gs_match *)gs_b200_malloc(sizeof(*matches) * MM * (size_t)n);
  mcount = (unsigned *)gs_b200_malloc(sizeof(unsigned) * n);
  htk = (struct gs_keypoint *)malloc(sizeof(*htk) * NK * (size_t)n);
  hs = (unsigned *)malloc(sizeof(unsigned) * n);
  hm = (unsigned *)malloc(sizeof(unsigned) * n);
  h1 = (unsigned *)malloc(sizeof(unsigned) * n);
  if (!tdev || !tbuf || !tk || !tks || !tcount || (spyr && !spyrd) || !ssm || !sk || !scount || !n1 || !matches ||
      !mcount || !htk || !hs || !hm || !h1)
    DIE("allocation failed");
  /* the template call, into the zeroed buffer laid out as nanomagick lays it out: pyramid, then score maps */
  CK(gs_b200_memcpy_h2d(tdev, tpl.data, (size_t)tpl.w * tpl.h, NULL));
  CK(gs_b200_memset(tbuf, 0, tpyr + tmaps > BUF ? tpyr + tmaps : BUF, NULL));
  CK(gs_b200_orb_pyramid_batch(tdev, tpl.w, tpl.h, 1, LV, tpyr ? tbuf : NULL, tbuf + tpyr, tk, tcount, NK, TH, NULL));
  if (stale) { /* frame f's level-l map starts as the buffer's bytes at the scene's offset of that map */
    uint8_t *hbuf = (uint8_t *)malloc(BUF), *hmaps = (uint8_t *)malloc(smaps * n);
    if (!hbuf || !hmaps) DIE("allocation failed");
    CK(gs_b200_memcpy_d2h(hbuf, tbuf, BUF, NULL));
    CK(gs_b200_stream_sync(NULL));
    for (l = 0; l < sl; l++) {
      size_t lb = (size_t)(w >> l) * (h >> l);
      for (f = 0; f < n; f++) memcpy(hmaps + soff[l] * n + lb * f, hbuf + spyr + soff[l], lb);
    }
    CK(gs_b200_memcpy_h2d(ssm, hmaps, smaps * n, NULL));
    CK(gs_b200_stream_sync(NULL));
    free(hbuf), free(hmaps);
  } else {
    CK(gs_b200_memset(ssm, 0, smaps * n, NULL));
  }
  CK(gs_b200_orb_pyramid_batch(cur->dev, w, h, n, LV, spyrd, ssm, sk, scount, NK, TH, NULL));
  /* the template's list as set 1 of each of the n pairs */
  CK(gs_b200_memcpy_d2h(htk, tk, sizeof(*tk) * NK, NULL));
  CK(gs_b200_memcpy_d2h(&ht, tcount, sizeof(unsigned), NULL));
  CK(gs_b200_stream_sync(NULL));
  for (f = 0; f < n; f++) {
    if (f) memcpy(htk + (size_t)NK * f, htk, sizeof(*htk) * NK);
    h1[f] = ht;
  }
  CK(gs_b200_memcpy_h2d(tks, htk, sizeof(*htk) * NK * (size_t)n, NULL));
  CK(gs_b200_memcpy_h2d(n1, h1, sizeof(unsigned) * n, NULL));
  CK(gs_b200_match_orb_batch(tks, n1, NK, sk, scount, NK, n, matches, mcount, MM, 60.0f, NULL));
  CK(gs_b200_memcpy_d2h(hs, scount, sizeof(unsigned) * n, NULL));
  CK(gs_b200_memcpy_d2h(hm, mcount, sizeof(unsigned) * n, NULL));
  CK(gs_b200_stream_sync(NULL));
  for (f = 0; f < n; f++) printf("frame %u: Template: %u keypoints, Scene: %u keypoints, Matches: %u\n", f, ht, hs[f], hm[f]);
  gs_b200_free(tbuf), gs_b200_free(tcount);
  if (spyrd) gs_b200_free(spyrd);
  gs_b200_free(ssm), free(htk), free(hs), free(h1);
  o->tpl = tpl, o->tdev = tdev, o->tk = tk, o->tks = tks, o->sk = sk, o->matches = matches, o->n1 = n1;
  o->scount = scount, o->mcount = mcount, o->hm = hm;
}

static void orb_free(struct orb_out *o) {
  gs_b200_free(o->tdev), gs_b200_free(o->tk), gs_b200_free(o->tks), gs_b200_free(o->sk), gs_b200_free(o->matches);
  gs_b200_free(o->n1), gs_b200_free(o->scount), gs_b200_free(o->mcount);
  free(o->hm);
  gs_free(o->tpl);
}

/* draw-orb: the orb stage, then the verb's side-by-side picture with its 15 best matches (nanomagick.c:313-343) in
 * *tmp; frames without matches are marked for no output */
static void draw_orb_stage(const char *path, const struct batch *cur, struct batch *tmp, size_t *cap_tmp) {
  struct orb_out o;
  unsigned f;
  orb_run(path, cur, &o);
  ensure(tmp, o.tpl.w + cur->w, o.tpl.h > cur->h ? o.tpl.h : cur->h, cur->n, cap_tmp);
  CKD(gs_b200_draw_matches_batch(tmp->dev, cur->dev, cur->w, cur->h, cur->n, o.tdev, o.tpl.w, o.tpl.h, o.tk, 0, o.sk,
                                 ORB_NK, o.matches, o.mcount, ORB_MM, 15, NULL));
  CK(gs_b200_stream_sync(NULL));
  for (f = 0; f < cur->n; f++)
    if (o.hm[f] == 0) no_output(f, cur->n, NO_MATCHES);
  orb_free(&o);
}

/* find:TEMPLATE.pgm:W:H (see the header comment): the orb stage, then homography -> quad -> warp to W x H in *tmp */
static void find_stage(const char *arg, const struct batch *cur, struct batch *tmp, size_t *cap_tmp) {
  enum { HYP = 1024, MIN_INLIERS = 10 };
  const char *c2 = strrchr(arg, ':'), *c1 = c2;
  char path[4096];
  unsigned f, n = cur->n, *inl, *hin;
  int dw, dh;
  double *H;
  struct gs_point *corners, *hc;
  uint8_t *found, *hf;
  struct orb_out o;
  while (c1 && c1 > arg && *--c1 != ':') {}
  if (!c2 || !c1 || *c1 != ':' || c1 == arg || (size_t)(c1 - arg) >= sizeof(path))
    DIE("bad find stage 'find:%s' (find:TEMPLATE.pgm:W:H)", arg);
  dw = atoi(c1 + 1), dh = atoi(c2 + 1);
  if (dw <= 0 || dh <= 0) DIE("bad size in 'find:%s'", arg);
  memcpy(path, arg, (size_t)(c1 - arg));
  path[c1 - arg] = 0;
  orb_run(path, cur, &o);
  H = (double *)gs_b200_malloc(sizeof(double) * 9 * n);
  inl = (unsigned *)gs_b200_malloc(sizeof(unsigned) * n);
  corners = (struct gs_point *)gs_b200_malloc(sizeof(*corners) * 4 * n);
  found = (uint8_t *)gs_b200_malloc(n);
  hin = (unsigned *)malloc(sizeof(unsigned) * n);
  hc = (struct gs_point *)malloc(sizeof(*hc) * 4 * n);
  hf = (uint8_t *)malloc(n);
  if (!H || !inl || !corners || !found || !hin || !hc || !hf) DIE("allocation failed");
  CKH(gs_b200_find_homography_batch(o.tks, o.n1, ORB_NK, o.sk, o.scount, ORB_NK, o.matches, o.mcount, ORB_MM, n, HYP,
                                    0, 3.0, H, inl, NULL, NULL));
  CKH(gs_b200_homography_quads_batch(H, inl, n, MIN_INLIERS, o.tpl.w, o.tpl.h, cur->w, cur->h, corners, found, NULL));
  ensure(tmp, (unsigned)dw, (unsigned)dh, n, cap_tmp);
  CK(gs_b200_perspective_correct_batch(tmp->dev, (unsigned)dw, (unsigned)dh, cur->dev, cur->w, cur->h, n, corners, 1,
                                       NULL));
  CK(gs_b200_memcpy_d2h(hin, inl, sizeof(unsigned) * n, NULL));
  CK(gs_b200_memcpy_d2h(hc, corners, sizeof(*hc) * 4 * n, NULL));
  CK(gs_b200_memcpy_d2h(hf, found, n, NULL));
  CK(gs_b200_stream_sync(NULL));
  for (f = 0; f < n; f++) {
    const struct gs_point *q = hc + 4 * (size_t)f;
    if (!hf[f]) {
      printf("frame %u: not found, %u inliers\n", f, hin[f]);
      no_output(f, n, NOT_FOUND);
      continue;
    }
    printf("frame %u: found, %u inliers, quad %u %u %u %u %u %u %u %u\n", f, hin[f], q[0].x, q[0].y, q[1].x, q[1].y,
           q[2].x, q[2].y, q[3].x, q[3].y);
  }
  gs_b200_free(H), gs_b200_free(inl), gs_b200_free(corners), gs_b200_free(found), free(hin), free(hc), free(hf);
  orb_free(&o);
}

/* one stage: reads *cur, leaves the result in *cur (swapping with *tmp when the op is out of place) */
static void stage(const char *spec, struct batch *cur, struct batch *tmp, size_t *cap_cur, size_t *cap_tmp) {
  char name[32] = {0}, a0[32] = {0}, a1[32] = {0};
  int nargs = sscanf(spec, "%31[^:]:%31[^:]:%31[^:]", name, a0, a1) - 1;
  unsigned w = cur->w, h = cur->h, n = cur->n;
  struct batch t;
  size_t tc;
  int swap = 1;
  if (!strcmp(name, "blur") && nargs == 1) {
    ensure(tmp, w, h, n, cap_tmp);
    CK(gs_b200_blur_batch(tmp->dev, cur->dev, w, h, n, (unsigned)atoi(a0), NULL));
  } else if (!strcmp(name, "sobel") && nargs == 0) {
    ensure(tmp, w, h, n, cap_tmp);
    CK(gs_b200_memset(tmp->dev, 0, frame_bytes(cur) * n, NULL)); /* gs_alloc'ed dst: zero frame */
    CK(gs_b200_sobel_batch(tmp->dev, cur->dev, w, h, n, NULL));
  } else if ((!strcmp(name, "erode") || !strcmp(name, "dilate")) && nargs <= 1) {
    int reps = nargs == 1 ? atoi(a0) : 1;
    if (reps <= 0) DIE("bad repeat count in '%s'", spec);
    ensure(tmp, w, h, n, cap_tmp);
    if (name[0] == 'e') CK(gs_b200_erode_n_batch(tmp->dev, cur->dev, w, h, n, (unsigned)reps, NULL));
    else CK(gs_b200_dilate_n_batch(tmp->dev, cur->dev, w, h, n, (unsigned)reps, NULL));
  } else if (!strcmp(name, "adaptive") && nargs == 2) {
    ensure(tmp, w, h, n, cap_tmp);
    CK(gs_b200_adaptive_threshold_batch(tmp->dev, cur->dev, w, h, n, (unsigned)atoi(a0), atoi(a1), NULL));
  } else if (!strcmp(name, "threshold") && nargs == 1) {
    swap = 0; /* in place, like gs_threshold */
    if (!strncmp(a0, "otsu", 4)) {
      uint8_t *th = (uint8_t *)gs_b200_malloc(n);
      if (!th) DIE("device allocation failed");
      CK(gs_b200_otsu_threshold_batch(th, NULL, cur->dev, w, h, n, NULL));
      CK(gs_b200_threshold_each_batch(cur->dev, w, h, n, th, a0[4] == '+' ? atoi(a0 + 5) : 0, NULL));
      CK(gs_b200_stream_sync(NULL));
      gs_b200_free(th);
    } else {
      CK(gs_b200_threshold_batch(cur->dev, w, h, n, (unsigned)atoi(a0) & 255u, NULL));
    }
  } else if (!strcmp(name, "filter") && nargs == 1) {
    static const int8_t sharpen[9] = {0, -1, 0, -1, 5, -1, 0, -1, 0}, emboss[9] = {-2, -1, 0, -1, 1, 1, 0, 1, 2};
    static const int8_t box[9] = {1, 1, 1, 1, 1, 1, 1, 1, 1}, gauss[9] = {1, 2, 1, 2, 4, 2, 1, 2, 1};
    const int8_t *k = !strcmp(a0, "sharpen") ? sharpen : !strcmp(a0, "emboss") ? emboss : !strcmp(a0, "box") ? box
                      : !strcmp(a0, "gaussian") ? gauss : NULL;
    if (!k) DIE("unknown filter '%s'", a0);
    ensure(tmp, w, h, n, cap_tmp);
    CK(gs_b200_filter_batch(tmp->dev, cur->dev, w, h, n, k, 3, 3, k == box ? 9u : k == gauss ? 16u : 1u, NULL));
  } else if (!strcmp(name, "downsample") && nargs == 0) {
    if (w < 2 || h < 2) DIE("downsample needs at least 2x2 frames");
    ensure(tmp, w / 2, h / 2, n, cap_tmp);
    CK(gs_b200_downsample_batch(tmp->dev, cur->dev, w, h, n, NULL));
  } else if (!strcmp(name, "resize") && nargs == 2) {
    int dw = atoi(a0), dh = atoi(a1);
    if (dw <= 0 || dh <= 0) DIE("bad size in '%s'", spec);
    ensure(tmp, (unsigned)dw, (unsigned)dh, n, cap_tmp);
    CK(gs_b200_resize_batch(tmp->dev, (unsigned)dw, (unsigned)dh, cur->dev, w, h, n, NULL));
  } else if (!strcmp(name, "crop")) {
    int x, y, cw, ch;
    char extra;
    struct gs_rect roi;
    if (sscanf(spec, "crop:%d:%d:%d:%d%c", &x, &y, &cw, &ch, &extra) != 4) DIE("bad rectangle in '%s' (crop:X:Y:W:H)", spec);
    if (x < 0 || y < 0 || cw <= 0 || ch <= 0 || (long)x + cw > (long)w || (long)y + ch > (long)h)
      DIE("invalid crop rectangle in '%s' for %ux%u frames", spec, w, h);
    roi.x = (unsigned)x, roi.y = (unsigned)y, roi.w = (unsigned)cw, roi.h = (unsigned)ch;
    ensure(tmp, roi.w, roi.h, n, cap_tmp);
    CK(gs_b200_crop_resize_batch(tmp->dev, roi.w, roi.h, cur->dev, w, h, n, roi, GS_B200_NEAREST, NULL));
  } else if (!strncmp(spec, "orb:", 4) && spec[4]) {
    struct orb_out o;
    swap = 0;
    orb_run(spec + 4, cur, &o);
    orb_free(&o);
  } else if (!strncmp(spec, "draw-orb:", 9) && spec[9]) {
    draw_orb_stage(spec + 9, cur, tmp, cap_tmp);
  } else if (!strncmp(spec, "find:", 5) && spec[5]) {
    find_stage(spec + 5, cur, tmp, cap_tmp);
  } else if (!strcmp(name, "draw-keypoints") && nargs == 2) {
    /* nanomagick.c:217-242: gs_fast into a zeroed score map with cap 5000, then the crosses of the N strongest */
    enum { CAP = 5000 };
    int nk = atoi(a0), th = atoi(a1);
    unsigned *counts;
    struct gs_keypoint *kps;
    uint8_t *sm;
    if (nk <= 0 || th < 0) DIE("bad keypoint count or threshold in '%s'", spec);
    kps = (struct gs_keypoint *)gs_b200_malloc(sizeof(*kps) * (size_t)CAP * n);
    counts = (unsigned *)gs_b200_malloc(sizeof(unsigned) * n);
    sm = (uint8_t *)gs_b200_malloc(frame_bytes(cur) * n);
    if (!kps || !counts || !sm) DIE("allocation failed");
    CK(gs_b200_memset(sm, 0, frame_bytes(cur) * n, NULL));
    CK(gs_b200_fast_batch(cur->dev, w, h, n, sm, kps, counts, CAP, (unsigned)th, NULL));
    ensure(tmp, w, h, n, cap_tmp);
    CKD(gs_b200_draw_keypoints_batch(tmp->dev, cur->dev, w, h, n, kps, counts, CAP, (unsigned)nk, NULL));
    CK(gs_b200_stream_sync(NULL));
    gs_b200_free(kps), gs_b200_free(counts), gs_b200_free(sm);
  } else if (!strcmp(name, "draw-blobs") && nargs == 1) {
    /* nanomagick.c:143-170: up to N blobs, then their grown boxes at 128 and the frame's > 128 pixels at 255 */
    int nb = atoi(a0);
    unsigned *counts;
    gs_label *labels;
    struct gs_blob *blobs;
    if (nb <= 0 || nb > 65534) DIE("bad blob count in '%s'", spec);
    labels = (gs_label *)gs_b200_malloc(sizeof(gs_label) * frame_bytes(cur) * n);
    blobs = (struct gs_blob *)gs_b200_malloc(sizeof(*blobs) * (size_t)nb * n);
    counts = (unsigned *)gs_b200_malloc(sizeof(unsigned) * n);
    if (!labels || !blobs || !counts) DIE("allocation failed");
    CK(gs_b200_blobs_batch(cur->dev, w, h, n, labels, blobs, counts, (unsigned)nb, NULL));
    ensure(tmp, w, h, n, cap_tmp);
    CKD(gs_b200_draw_blobs_batch(tmp->dev, cur->dev, w, h, n, blobs, counts, (unsigned)nb, NULL));
    CK(gs_b200_stream_sync(NULL));
    gs_b200_free(labels), gs_b200_free(blobs), gs_b200_free(counts);
  } else if (!strcmp(name, "faces") && nargs == 1) {
    /* nanomagick.c:347-376: integral, gs_lbp_detect(&frontalface, ..., 100 rects, 1.2, 1.0, 4.0, N), the outlines */
    enum { MR = 100 };
    int mn = atoi(a0);
    unsigned *counts;
    uint32_t *ii;
    struct gs_rect *rects;
    if (mn <= 0) DIE("minimum neighbors must be positive in '%s'", spec);
    ii = (uint32_t *)gs_b200_malloc(sizeof(uint32_t) * frame_bytes(cur) * n);
    rects = (struct gs_rect *)gs_b200_malloc(sizeof(*rects) * (size_t)MR * n);
    counts = (unsigned *)gs_b200_malloc(sizeof(unsigned) * n);
    if (!ii || !rects || !counts) DIE("allocation failed");
    CK(gs_b200_integral_batch(ii, cur->dev, w, h, n, NULL));
    CK(gs_b200_lbp_detect_batch(&frontalface, ii, w, h, n, rects, counts, MR, 1.2f, 1.0f, 4.0f, mn, NULL));
    ensure(tmp, w, h, n, cap_tmp);
    CKD(gs_b200_draw_rects_batch(tmp->dev, cur->dev, w, h, n, rects, counts, MR, NULL));
    CK(gs_b200_stream_sync(NULL));
    gs_b200_free(ii), gs_b200_free(rects), gs_b200_free(counts);
  } else if (!strcmp(name, "faces-grouped") && nargs == 2) {
    /* the faces stage's detection with a real scan step and room for every window, then the windows grouped on the
     * device (min_neighbors K, eps 0.2), as many frames per chunk as 256 MiB of grouping state holds */
    enum { MR = 4096 };
    int step = atoi(a0), k = atoi(a1);
    unsigned f, *counts, *gcounts, *hc, *hg;
    uint32_t *ii;
    struct gs_rect *rects, *groups;
    size_t wb = gs_b200_group_rects_work_bytes(MR, n), one = gs_b200_group_rects_work_bytes(MR, 1);
    void *work;
    if (step <= 0) DIE("scan step must be positive in '%s'", spec);
    if (k < 0) DIE("minimum neighbors must not be negative in '%s'", spec);
    if (wb > ((size_t)256 << 20)) wb = one > ((size_t)256 << 20) ? one : ((size_t)256 << 20);
    ii = (uint32_t *)gs_b200_malloc(sizeof(uint32_t) * frame_bytes(cur) * n);
    rects = (struct gs_rect *)gs_b200_malloc(sizeof(*rects) * (size_t)MR * n);
    groups = (struct gs_rect *)gs_b200_malloc(sizeof(*groups) * (size_t)MR * n);
    counts = (unsigned *)gs_b200_malloc(sizeof(unsigned) * n);
    gcounts = (unsigned *)gs_b200_malloc(sizeof(unsigned) * n);
    work = gs_b200_malloc(wb);
    hc = (unsigned *)malloc(sizeof(unsigned) * n);
    hg = (unsigned *)malloc(sizeof(unsigned) * n);
    if (!ii || !rects || !groups || !counts || !gcounts || !work || !hc || !hg) DIE("allocation failed");
    CK(gs_b200_integral_batch(ii, cur->dev, w, h, n, NULL));
    CK(gs_b200_lbp_detect_batch(&frontalface, ii, w, h, n, rects, counts, MR, 1.2f, 1.0f, 4.0f, step, NULL));
    CKG(gs_b200_group_rects_batch(rects, counts, MR, n, (unsigned)k, 0.2, groups, NULL, gcounts, MR, work, wb, NULL));
    ensure(tmp, w, h, n, cap_tmp);
    CKD(gs_b200_draw_rects_batch(tmp->dev, cur->dev, w, h, n, groups, gcounts, MR, NULL));
    CK(gs_b200_memcpy_d2h(hc, counts, sizeof(unsigned) * n, NULL));
    CK(gs_b200_memcpy_d2h(hg, gcounts, sizeof(unsigned) * n, NULL));
    CK(gs_b200_stream_sync(NULL));
    for (f = 0; f < n; f++) printf("frame %u: %u windows, %u faces\n", f, hc[f], hg[f]);
    gs_b200_free(ii), gs_b200_free(rects), gs_b200_free(groups), gs_b200_free(counts), gs_b200_free(gcounts);
    gs_b200_free(work), free(hc), free(hg);
  } else if (!strcmp(name, "keypoints") && nargs == 2) {
    unsigned nk = (unsigned)atoi(a0), f, *counts, *hc;
    struct gs_keypoint *kps;
    uint8_t *sm;
    swap = 0;
    if (nk == 0) DIE("bad keypoint count in '%s'", spec);
    kps = (struct gs_keypoint *)gs_b200_malloc(sizeof(*kps) * (size_t)nk * n);
    counts = (unsigned *)gs_b200_malloc(sizeof(unsigned) * n);
    sm = (uint8_t *)gs_b200_malloc(frame_bytes(cur) * n);
    hc = (unsigned *)malloc(sizeof(unsigned) * n);
    if (!kps || !counts || !sm || !hc) DIE("allocation failed");
    CK(gs_b200_memset(sm, 0, frame_bytes(cur) * n, NULL));
    CK(gs_b200_orb_extract_batch(cur->dev, w, h, n, sm, kps, counts, nk, (unsigned)atoi(a1), NULL));
    CK(gs_b200_memcpy_d2h(hc, counts, sizeof(unsigned) * n, NULL));
    CK(gs_b200_stream_sync(NULL));
    for (f = 0; f < n; f++) printf("frame %u: %u keypoints\n", f, hc[f]);
    gs_b200_free(kps), gs_b200_free(counts), gs_b200_free(sm), free(hc);
  } else if (!strcmp(name, "blobs") && nargs == 1) {
    unsigned nb = (unsigned)atoi(a0), f, *counts, *hc;
    gs_label *labels;
    struct gs_blob *blobs;
    swap = 0;
    if (nb == 0 || nb > 65534u) DIE("bad blob count in '%s'", spec);
    labels = (gs_label *)gs_b200_malloc(sizeof(gs_label) * frame_bytes(cur) * n);
    blobs = (struct gs_blob *)gs_b200_malloc(sizeof(*blobs) * (size_t)nb * n);
    counts = (unsigned *)gs_b200_malloc(sizeof(unsigned) * n);
    hc = (unsigned *)malloc(sizeof(unsigned) * n);
    if (!labels || !blobs || !counts || !hc) DIE("allocation failed");
    CK(gs_b200_blobs_batch(cur->dev, w, h, n, labels, blobs, counts, nb, NULL));
    CK(gs_b200_memcpy_d2h(hc, counts, sizeof(unsigned) * n, NULL));
    CK(gs_b200_stream_sync(NULL));
    for (f = 0; f < n; f++) printf("frame %u: %u blobs\n", f, hc[f]);
    gs_b200_free(labels), gs_b200_free(blobs), gs_b200_free(counts), free(hc);
  } else if (!strcmp(name, "contour") && nargs == 1) {
    /* grayskull.c:278-326: the largest of up to N blobs (strict >, so the first wins ties), none below area 100; its
     * start on the device; the trace on a zeroed visited map, as many frames per chunk as 256 MiB of owner maps hold.
     * Nothing comes back to the host before the contours. */
    static const char *end_name[] = {"returned", "open", "cycle"};
    unsigned nb = (unsigned)atoi(a0), f, *counts, *pcount, *hp;
    size_t wb = gs_b200_trace_contours_work_bytes(w, h, n), one = gs_b200_trace_contours_work_bytes(w, h, 1);
    gs_label *labels;
    struct gs_blob *blobs, *pick;
    struct gs_contour *contours, *hcont;
    uint8_t *visited, *ends, *hends;
    void *work;
    swap = 0;
    if (nb == 0 || nb > 65534u) DIE("bad blob count in '%s'", spec);
    if (wb > ((size_t)256 << 20)) wb = one > ((size_t)256 << 20) ? one : (size_t)256 << 20;
    labels = (gs_label *)gs_b200_malloc(sizeof(gs_label) * frame_bytes(cur) * n);
    blobs = (struct gs_blob *)gs_b200_malloc(sizeof(*blobs) * (size_t)nb * n);
    counts = (unsigned *)gs_b200_malloc(sizeof(unsigned) * n);
    pick = (struct gs_blob *)gs_b200_malloc(sizeof(*pick) * n);
    pcount = (unsigned *)gs_b200_malloc(sizeof(unsigned) * n);
    contours = (struct gs_contour *)gs_b200_malloc(sizeof(*contours) * n);
    visited = (uint8_t *)gs_b200_malloc(frame_bytes(cur) * n);
    ends = (uint8_t *)gs_b200_malloc(n);
    work = gs_b200_malloc(wb);
    hp = (unsigned *)malloc(sizeof(unsigned) * n);
    hcont = (struct gs_contour *)malloc(sizeof(*hcont) * n);
    hends = (uint8_t *)malloc(n);
    if (!labels || !blobs || !counts || !pick || !pcount || !contours || !visited || !ends || !work || !hp || !hcont ||
        !hends)
      DIE("allocation failed");
    CK(gs_b200_blobs_batch(cur->dev, w, h, n, labels, blobs, counts, nb, NULL));
    CKR(gs_b200_largest_blob_batch(blobs, counts, nb, n, 100, pick, pcount, NULL)); /* one record per frame, or none */
    CKC(gs_b200_blob_contour_starts_batch(labels, w, h, n, pick, pcount, 1, contours, NULL));
    CK(gs_b200_memset(visited, 0, frame_bytes(cur) * n, NULL));
    CKC(gs_b200_trace_contours_batch(cur->dev, visited, w, h, n, contours, pcount, 1, ends, work, wb, NULL));
    CK(gs_b200_memcpy_d2h(hcont, contours, sizeof(*hcont) * n, NULL));
    CK(gs_b200_memcpy_d2h(hends, ends, n, NULL));
    CK(gs_b200_memcpy_d2h(hp, pcount, sizeof(unsigned) * n, NULL));
    CK(gs_b200_stream_sync(NULL));
    for (f = 0; f < n; f++) {
      const struct gs_contour *c = &hcont[f];
      if (!hp[f]) {
        printf("frame %u: no contour\n", f);
        continue;
      }
      printf("frame %u: contour start %u %u box %u %u %u %u length %u end %s\n", f, c->start.x, c->start.y, c->box.x,
             c->box.y, c->box.w, c->box.h, c->length, end_name[hends[f]]);
    }
    gs_b200_free(labels), gs_b200_free(blobs), gs_b200_free(counts), gs_b200_free(pick), gs_b200_free(pcount);
    gs_b200_free(contours), gs_b200_free(visited), gs_b200_free(ends), gs_b200_free(work);
    free(hp), free(hcont), free(hends);
  } else if (!strcmp(name, "scan") && nargs == 2) {
    /* reference nanomagick.c:186-210: tmp = blur(img, 1); threshold(tmp, otsu(tmp) + 10); blobs(tmp, 1000); corners of
     * the largest blob (first one on ties); perspective_correct(out, img, corners).  All on the device: a frame without
     * blobs picks gs_blobs' initial record, whose corners are its centroid (0, 0), as in the reference. */
    enum { NB = 1000 };
    int dw = atoi(a0), dh = atoi(a1);
    unsigned *counts;
    uint8_t *bin, *th;
    gs_label *labels;
    struct gs_blob *blobs, *pick;
    struct gs_point *corners;
    if (dw <= 0 || dh <= 0) DIE("bad size in '%s'", spec);
    bin = (uint8_t *)gs_b200_malloc(frame_bytes(cur) * n);
    th = (uint8_t *)gs_b200_malloc(n);
    labels = (gs_label *)gs_b200_malloc(sizeof(gs_label) * frame_bytes(cur) * n);
    blobs = (struct gs_blob *)gs_b200_malloc(sizeof(*blobs) * (size_t)NB * n);
    pick = (struct gs_blob *)gs_b200_malloc(sizeof(*pick) * n);
    corners = (struct gs_point *)gs_b200_malloc(sizeof(*corners) * 4 * n);
    counts = (unsigned *)gs_b200_malloc(sizeof(unsigned) * n);
    if (!bin || !th || !labels || !blobs || !pick || !corners || !counts) DIE("allocation failed");
    CK(gs_b200_blur_batch(bin, cur->dev, w, h, n, 1, NULL));
    CK(gs_b200_otsu_threshold_batch(th, NULL, bin, w, h, n, NULL));
    CK(gs_b200_threshold_each_batch(bin, w, h, n, th, 10, NULL));
    CK(gs_b200_blobs_batch(bin, w, h, n, labels, blobs, counts, NB, NULL));
    CKR(gs_b200_largest_blob_batch(blobs, counts, NB, n, 0, pick, NULL, NULL));
    CKR(gs_b200_blob_corners_batch(bin, w, h, n, labels, pick, NULL, 1, corners, NULL));
    ensure(tmp, (unsigned)dw, (unsigned)dh, n, cap_tmp);
    CK(gs_b200_perspective_correct_batch(tmp->dev, (unsigned)dw, (unsigned)dh, cur->dev, w, h, n, corners, 1, NULL));
    CK(gs_b200_stream_sync(NULL));
    gs_b200_free(bin), gs_b200_free(th), gs_b200_free(labels), gs_b200_free(blobs), gs_b200_free(pick), gs_b200_free(corners);
    gs_b200_free(counts);
  } else {
    DIE("unknown stage or wrong argument count: '%s'", spec);
  }
  if (swap) t = *cur, *cur = *tmp, *tmp = t, tc = *cap_cur, *cap_cur = *cap_tmp, *cap_tmp = tc;
}

/* whether `path` is a file that starts with P6 ("-" is read as P5) */
static int is_p6(const char *path) {
  char magic[2] = {0, 0};
  FILE *f;
  if (path[0] == '-' && !path[1]) return 0;
  f = fopen(path, "rb");
  if (!f) return 0;
  if (fread(magic, 1, 2, f) != 2) magic[0] = 0;
  fclose(f);
  return magic[0] == 'P' && magic[1] == '6';
}

/* a binary P6 file's header, with the header grammar of gs_read_pgm: the file positioned at its first pixel */
static FILE *open_ppm(const char *path, unsigned *w, unsigned *h) {
  unsigned maxval = 0;
  FILE *f = fopen(path, "rb");
  if (!f || fgetc(f) != 'P' || fgetc(f) != '6' || !gs__pgm_token(f, w) || !gs__pgm_token(f, h) ||
      !gs__pgm_token(f, &maxval) || *w == 0 || *h == 0)
    DIE("could not load %s", path);
  if (maxval != 255) DIE("%s: P6 maxval %u, only 255 is supported", path, maxval);
  return f;
}

int main(int argc, char **argv) {
  struct batch cur = {NULL, 0, 0, 0}, tmp = {NULL, 0, 0, 0};
  size_t cap_cur = 0, cap_tmp = 0, out_bytes;
  unsigned n, f;
  uint8_t *host;
  char *pipeline, *tok;
  int p6;
  if (argc < 4) {
    fprintf(stderr, "usage: %s <stage[,stage...]> <out-prefix> in0.pgm|in0.ppm [in1 ...]\n"
                    "  inputs: binary P5, or binary P6 (maxval 255) converted to gray on the device; one kind and\n"
                    "  one size per batch; outputs are P5\n", argv[0]);
    return 1;
  }
  if (gs_b200_device_count() < 1) DIE("no CUDA device (this tool has no CPU path)");
  CK(gs_b200_set_device(0));
  n = (unsigned)(argc - 3);
  host = NULL;
  p6 = is_p6(argv[3]);
  for (f = 0; f < n && p6; f++) { /* P6: read straight into the pinned batch, 3 bytes a pixel */
    unsigned w, h;
    size_t got;
    FILE *in;
    if (!is_p6(argv[3 + f])) DIE("%s is not P6, the batch is P6", argv[3 + f]);
    in = open_ppm(argv[3 + f], &w, &h);
    if (f == 0) {
      ensure(&cur, w, h, n, &cap_cur);
      host = (uint8_t *)gs_b200_malloc_host(3 * frame_bytes(&cur) * n);
      if (!host) DIE("pinned host allocation failed");
    } else if (w != cur.w || h != cur.h) {
      DIE("%s is %ux%u, the batch is %ux%u", argv[3 + f], w, h, cur.w, cur.h);
    }
    got = fread(host + 3 * frame_bytes(&cur) * f, 1, 3 * frame_bytes(&cur), in);
    fclose(in);
    if (got != 3 * frame_bytes(&cur)) DIE("%s is truncated: %lu of %lu pixel bytes", argv[3 + f], (unsigned long)got,
                                          (unsigned long)(3 * frame_bytes(&cur)));
  }
  if (p6) { /* one copy of the colour batch, then the demo's gray on the device */
    uint8_t *rgb = (uint8_t *)gs_b200_malloc(3 * frame_bytes(&cur) * n);
    if (!rgb) DIE("device allocation failed");
    CK(gs_b200_memcpy_h2d(rgb, host, 3 * frame_bytes(&cur) * n, NULL));
    CKK(gs_b200_rgb_to_gray_batch(cur.dev, rgb, cur.w, cur.h, n, 3, NULL));
    CK(gs_b200_stream_sync(NULL));
    gs_b200_free(rgb);
  }
  for (f = 0; f < n && !p6; f++) { /* read straight into the pinned batch */
    if (is_p6(argv[3 + f])) DIE("%s is P6, the batch is P5", argv[3 + f]);
    struct gs_image img = gs_read_pgm(argv[3 + f]);
    if (!gs_valid(img)) DIE("could not load %s", argv[3 + f]);
    if (f == 0) {
      ensure(&cur, img.w, img.h, n, &cap_cur);
      host = (uint8_t *)gs_b200_malloc_host(frame_bytes(&cur) * n);
      if (!host) DIE("pinned host allocation failed");
    } else if (img.w != cur.w || img.h != cur.h) {
      DIE("%s is %ux%u, the batch is %ux%u", argv[3 + f], img.w, img.h, cur.w, cur.h);
    }
    memcpy(host + frame_bytes(&cur) * f, img.data, frame_bytes(&cur));
    gs_free(img);
  }
  if (!p6) CK(gs_b200_memcpy_h2d(cur.dev, host, frame_bytes(&cur) * n, NULL));
  pipeline = argv[1];
  for (tok = strtok(pipeline, ","); tok; tok = strtok(NULL, ",")) stage(tok, &cur, &tmp, &cap_cur, &cap_tmp);
  out_bytes = frame_bytes(&cur) * n;
  if (out_bytes > (size_t)0) {
    uint8_t *hout = (uint8_t *)gs_b200_malloc_host(out_bytes);
    if (!hout) DIE("pinned host allocation failed");
    CK(gs_b200_memcpy_d2h(hout, cur.dev, out_bytes, NULL));
    CK(gs_b200_stream_sync(NULL));
    for (f = 0; f < n; f++) {
      char path[4096];
      struct gs_image img;
      img.w = cur.w, img.h = cur.h, img.data = hout + frame_bytes(&cur) * f;
      snprintf(path, sizeof(path), "%s%04u.pgm", argv[2], f);
      if (g_no_output && g_no_output[f]) {
        fprintf(stderr, "gsb_magick: frame %u: %s, %s not written\n", f,
                g_no_output[f] == NO_MATCHES ? "no matches" : "template not found", path);
        continue;
      }
      if (gs_write_pgm(img, path) != 0) DIE("could not write %s", path);
    }
    gs_b200_free_host(hout);
  }
  gs_b200_free_host(host);
  free(g_no_output);
  gs_b200_free(cur.dev);
  if (tmp.dev) gs_b200_free(tmp.dev);
  return 0;
}
