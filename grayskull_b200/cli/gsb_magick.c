/*
 * gsb_magick -- batch image pipelines on the device-resident C ABI (SURVEY.md 8f N4: the caller side of
 * the hot path).  Plain C99 against include/grayskull.h (stand-alone mode) + include/grayskull_b200.h.
 *
 *   gsb_magick <pipeline> <out-prefix> in0.pgm [in1.pgm ...]
 *
 * All inputs (binary P5 PGM, same size) are read into ONE pinned host batch, copied to the GPU once,
 * taken through the pipeline without leaving the device (two ping-pong frame batches), copied back once
 * and written as <out-prefix>NNNN.pgm.  Pipeline = comma-separated stages, arguments after ':'
 *   blur:R   sobel   erode[:N]   dilate[:N]   adaptive:R:C   threshold:T   threshold:otsu[+K]
 *   (erode:N / dilate:N are N passes of the 3x3 op in one call, gs_b200_erode_n_batch / gs_b200_dilate_n_batch)
 *   filter:sharpen|emboss|box|gaussian   downsample   resize:W:H
 *   crop:X:Y:W:H    (the reference's crop verb, nanomagick.c:69-77: gs_crop of one rectangle of every frame)
 *   keypoints:N:T   (prints the ORB keypoint count per frame; frames pass through unchanged)
 *   blobs:N         (prints the number of 4-connected components >= 128 per frame; frames pass through unchanged)
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
 * e.g. the reference Makefile's lena chain:  blur:2,threshold:otsu,erode:2,dilate:2
 * Stage semantics are the reference's gs_* functions (same kernels as the drop-in gs_* entry points).
 */
#include <string.h>

#include "grayskull_b200_pyramid.h"
#include "grayskull_b200_roi.h"

#define DIE(...) (fprintf(stderr, "gsb_magick: " __VA_ARGS__), fprintf(stderr, "\n"), exit(1))
#define CK(call)                                                         \
  do {                                                                   \
    if ((call) != 0) DIE("%s failed: %s", #call, gs_b200_last_error());  \
  } while (0)

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

/* the orb stage (see the header comment): template as set 1 of every pair, frame f's keypoints as set 2 */
static void orb_stage(const char *path, const struct batch *cur) {
  enum { NK = 2500, TH = 20, LV = 3, MM = 300 };
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
  gs_b200_free(tdev), gs_b200_free(tbuf), gs_b200_free(tk), gs_b200_free(tks), gs_b200_free(tcount);
  if (spyrd) gs_b200_free(spyrd);
  gs_b200_free(ssm), gs_b200_free(sk), gs_b200_free(scount), gs_b200_free(n1), gs_b200_free(matches);
  gs_b200_free(mcount), free(htk), free(hs), free(hm), free(h1);
  gs_free(tpl);
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
    swap = 0;
    orb_stage(spec + 4, cur);
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
  } else if (!strcmp(name, "scan") && nargs == 2) {
    /* reference nanomagick.c:186-210: tmp = blur(img, 1); threshold(tmp, otsu(tmp) + 10); blobs(tmp, 1000); corners of
     * the largest blob (first one on ties); perspective_correct(out, img, corners) */
    enum { NB = 1000 };
    int dw = atoi(a0), dh = atoi(a1);
    unsigned f, i, *counts, *hc;
    uint8_t *bin, *th;
    gs_label *labels;
    struct gs_blob *blobs, *hb, *pick;
    struct gs_point *corners;
    if (dw <= 0 || dh <= 0) DIE("bad size in '%s'", spec);
    bin = (uint8_t *)gs_b200_malloc(frame_bytes(cur) * n);
    th = (uint8_t *)gs_b200_malloc(n);
    labels = (gs_label *)gs_b200_malloc(sizeof(gs_label) * frame_bytes(cur) * n);
    blobs = (struct gs_blob *)gs_b200_malloc(sizeof(*blobs) * (size_t)NB * n);
    pick = (struct gs_blob *)gs_b200_malloc(sizeof(*pick) * n);
    corners = (struct gs_point *)gs_b200_malloc(sizeof(*corners) * 4 * n);
    counts = (unsigned *)gs_b200_malloc(sizeof(unsigned) * n);
    hc = (unsigned *)malloc(sizeof(unsigned) * n);
    hb = (struct gs_blob *)malloc(sizeof(*hb) * (size_t)NB * n);
    if (!bin || !th || !labels || !blobs || !pick || !corners || !counts || !hc || !hb) DIE("allocation failed");
    CK(gs_b200_blur_batch(bin, cur->dev, w, h, n, 1, NULL));
    CK(gs_b200_otsu_threshold_batch(th, NULL, bin, w, h, n, NULL));
    CK(gs_b200_threshold_each_batch(bin, w, h, n, th, 10, NULL));
    CK(gs_b200_blobs_batch(bin, w, h, n, labels, blobs, counts, NB, NULL));
    CK(gs_b200_memcpy_d2h(hc, counts, sizeof(unsigned) * n, NULL));
    CK(gs_b200_memcpy_d2h(hb, blobs, sizeof(*hb) * (size_t)NB * n, NULL));
    CK(gs_b200_stream_sync(NULL));
    for (f = 0; f < n; f++) { /* the selection is a host-side scan of <= 1000 records, like the reference's */
      unsigned largest = 0;
      if (hc[f] == 0) memset(&hb[(size_t)f * NB], 0, sizeof(*hb)); /* no blob: corners fall back to the centroid (0, 0) */
      for (i = 1; i < hc[f]; i++)
        if (hb[(size_t)f * NB + i].area > hb[(size_t)f * NB + largest].area) largest = i;
      CK(gs_b200_memcpy_h2d(pick + f, &hb[(size_t)f * NB + largest], sizeof(*pick), NULL));
      CK(gs_b200_blob_corners(bin + frame_bytes(cur) * f, w, h, labels + frame_bytes(cur) * f, pick + f, corners + 4 * f, NULL));
    }
    ensure(tmp, (unsigned)dw, (unsigned)dh, n, cap_tmp);
    CK(gs_b200_perspective_correct_batch(tmp->dev, (unsigned)dw, (unsigned)dh, cur->dev, w, h, n, corners, 1, NULL));
    CK(gs_b200_stream_sync(NULL));
    gs_b200_free(bin), gs_b200_free(th), gs_b200_free(labels), gs_b200_free(blobs), gs_b200_free(pick), gs_b200_free(corners);
    gs_b200_free(counts), free(hc), free(hb);
  } else {
    DIE("unknown stage or wrong argument count: '%s'", spec);
  }
  if (swap) t = *cur, *cur = *tmp, *tmp = t, tc = *cap_cur, *cap_cur = *cap_tmp, *cap_tmp = tc;
}

int main(int argc, char **argv) {
  struct batch cur = {NULL, 0, 0, 0}, tmp = {NULL, 0, 0, 0};
  size_t cap_cur = 0, cap_tmp = 0, out_bytes;
  unsigned n, f;
  uint8_t *host;
  char *pipeline, *tok;
  if (argc < 4) {
    fprintf(stderr, "usage: %s <stage[,stage...]> <out-prefix> in0.pgm [in1.pgm ...]\n", argv[0]);
    return 1;
  }
  if (gs_b200_device_count() < 1) DIE("no CUDA device (this tool has no CPU path)");
  CK(gs_b200_set_device(0));
  n = (unsigned)(argc - 3);
  host = NULL;
  for (f = 0; f < n; f++) { /* read straight into the pinned batch */
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
  CK(gs_b200_memcpy_h2d(cur.dev, host, frame_bytes(&cur) * n, NULL));
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
      if (gs_write_pgm(img, path) != 0) DIE("could not write %s", path);
    }
    gs_b200_free_host(hout);
  }
  gs_b200_free_host(host);
  gs_b200_free(cur.dev);
  if (tmp.dev) gs_b200_free(tmp.dev);
  return 0;
}
