// api.cu -- the reference's single-image gs_* entry points (include/grayskull.h) on top of the
// batched kernels: n == 1, synchronous.  Re-entrant like the reference (SURVEY.md 8b "Threading"): every host
// thread works on its OWN stream per device -- and, because the library's scratch arenas are keyed by (device,
// stream, slot), on its own staging arenas -- so concurrent gs_* calls from several threads never share a
// buffer.  The per-thread streams are ordinary blocking streams: they keep the implicit ordering with work the
// caller queued on the legacy default stream (e.g. a gs_b200_*_batch call with stream NULL on the same images).  Device / managed pointers are
// used in place; plain host pointers are staged through the library's device workspace (copied
// in, processed, copied back), so unmodified callers such as the reference's test.c work.
// Precondition checks are the reference's gs_assert conditions (cited), CUDA failures abort with
// a message: there is no CPU fallback anywhere in this library.
#include <string.h>

#include "common.cuh"

namespace gsb {
// fast_orb.cu, lbp.cu
int fast_single(const uint8_t *src, unsigned w, unsigned h, uint8_t *score, unsigned sw, unsigned sh,
                struct gs_keypoint *kps, unsigned *count, unsigned nkps, unsigned threshold, cudaStream_t s);
int orient_single(const uint8_t *img, unsigned w, unsigned x, unsigned y, unsigned r, float *out, cudaStream_t s);
int brief_single(const uint8_t *img, unsigned w, unsigned h, struct gs_keypoint *kp, cudaStream_t s);
int lbp_window_single(const struct gs_lbp_cascade *c, const uint32_t *ii, unsigned iw, unsigned ih, int x, int y,
                      float scale, unsigned *out_dev, cudaStream_t s);
}  // namespace gsb

namespace {

void die(const char *what, int rc) {
  fprintf(stderr, "grayskull_b200: %s failed: %s\n", what, rc ? gs_b200_last_error() : "(no device?)");
  abort();
}
#define GS_DO(call)                \
  do {                             \
    int rc_ = (call);              \
    if (rc_) die(#call, rc_);      \
  } while (0)
#define GS_CUDA(call)                                           \
  do {                                                          \
    cudaError_t e_ = (call);                                    \
    if (e_ != cudaSuccess) die(#call, gsb::record_error(e_, __FILE__, __LINE__)); \
  } while (0)

bool on_device(const void *p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

// this thread's stream on the current device (created on first use, destroyed with the thread)
struct ThreadStreams {
  cudaStream_t s[64] = {};
  ~ThreadStreams() {
    for (int d = 0; d < 64; d++)
      if (s[d]) {
        int cur = 0;
        if (cudaGetDevice(&cur) != cudaSuccess) return;   // runtime already shut down
        if (cur != d) cudaSetDevice(d);
        cudaStreamDestroy(s[d]);
        if (cur != d) cudaSetDevice(cur);
      }
  }
};
thread_local ThreadStreams t_streams;
cudaStream_t S() {
  int dev = 0;
  GS_CUDA(cudaGetDevice(&dev));
  cudaStream_t &st = t_streams.s[dev & 63];
  if (!st) GS_CUDA(cudaStreamCreate(&st));
  return st;
}

inline int gs_ok(struct gs_image img) { return img.data && img.w > 0 && img.h > 0; }

// a buffer that lives on the device for the duration of one call
struct Buf {
  void *dev = nullptr;
  void *host = nullptr;  // non-null iff staged
  size_t bytes = 0;
};
Buf in_buf(const void *p, size_t bytes, int slot, bool copy_in = true) {
  Buf b;
  b.bytes = bytes;
  if (!p || bytes == 0) return b;
  if (on_device(p)) {
    b.dev = const_cast<void *>(p);
    return b;
  }
  b.dev = gsb::workspace(S(), slot, bytes);
  if (!b.dev) die("device workspace allocation", 1);
  b.host = const_cast<void *>(p);
  if (copy_in) GS_CUDA(cudaMemcpyAsync(b.dev, p, bytes, cudaMemcpyHostToDevice, S()));
  return b;
}
void out_buf(const Buf &b, size_t bytes = ~(size_t)0) {
  if (b.host) GS_CUDA(cudaMemcpyAsync(b.host, b.dev, bytes < b.bytes ? bytes : b.bytes, cudaMemcpyDeviceToHost, S()));
}
void finish() { GS_CUDA(cudaStreamSynchronize(S())); }

}  // namespace

extern "C" {

void gs_blur(struct gs_image dst, struct gs_image src, unsigned radius) {
  GSB_ASSERT(gs_ok(src) && gs_ok(dst) && dst.w == src.w && dst.h == src.h);  // reference :269
  const size_t n = (size_t)src.w * src.h;
  Buf s = in_buf(src.data, n, gsb::WS_STAGE_A), d = in_buf(dst.data, n, gsb::WS_STAGE_B, false);
  GS_DO(gs_b200_blur_batch((uint8_t *)d.dev, (const uint8_t *)s.dev, src.w, src.h, 1, radius, S()));
  out_buf(d);
  finish();
}

void gs_adaptive_threshold(struct gs_image dst, struct gs_image src, unsigned radius, int c) {
  GSB_ASSERT(gs_ok(dst) && gs_ok(src) && dst.w == src.w && dst.h == src.h);  // reference :232
  const size_t n = (size_t)src.w * src.h;
  Buf s = in_buf(src.data, n, gsb::WS_STAGE_A), d = in_buf(dst.data, n, gsb::WS_STAGE_B, false);
  GS_DO(gs_b200_adaptive_threshold_batch((uint8_t *)d.dev, (const uint8_t *)s.dev, src.w, src.h, 1, radius, c, S()));
  out_buf(d);
  finish();
}

void gs_sobel(struct gs_image dst, struct gs_image src) {
  GSB_ASSERT(gs_ok(dst) && gs_ok(src) && dst.w == src.w && dst.h == src.h);  // reference :307
  const size_t n = (size_t)src.w * src.h;
  if (src.w < 3 || src.h < 3) return;      // nothing is written (reference :308-309)
  // dst's 1-px frame must keep the caller's bytes (reference :308-309): a staged dst is not copied in at all,
  // only the interior (w-2) x (h-2) block travels back, as one strided copy
  Buf s = in_buf(src.data, n, gsb::WS_STAGE_A), d = in_buf(dst.data, n, gsb::WS_STAGE_B, false);
  GS_DO(gs_b200_sobel_batch((uint8_t *)d.dev, (const uint8_t *)s.dev, src.w, src.h, 1, S()));
  if (d.host)
    GS_CUDA(cudaMemcpy2DAsync((uint8_t *)d.host + src.w + 1, src.w, (const uint8_t *)d.dev + src.w + 1, src.w, src.w - 2,
                              src.h - 2, cudaMemcpyDeviceToHost, S()));
  finish();
}

static void morph(struct gs_image dst, struct gs_image src, int dilate) {
  GSB_ASSERT(gs_ok(dst) && gs_ok(src) && dst.w == src.w && dst.h == src.h);  // reference :287
  const size_t n = (size_t)src.w * src.h;
  Buf s = in_buf(src.data, n, gsb::WS_STAGE_A), d = in_buf(dst.data, n, gsb::WS_STAGE_B, false);
  if (dilate) GS_DO(gs_b200_dilate_batch((uint8_t *)d.dev, (const uint8_t *)s.dev, src.w, src.h, 1, S()));
  else GS_DO(gs_b200_erode_batch((uint8_t *)d.dev, (const uint8_t *)s.dev, src.w, src.h, 1, S()));
  out_buf(d);
  finish();
}
void gs_erode(struct gs_image dst, struct gs_image src) { morph(dst, src, 0); }
void gs_dilate(struct gs_image dst, struct gs_image src) { morph(dst, src, 1); }

void gs_resize(struct gs_image dst, struct gs_image src) {
  GSB_ASSERT(gs_ok(dst) && gs_ok(src));  // reference :172
  Buf s = in_buf(src.data, (size_t)src.w * src.h, gsb::WS_STAGE_A);
  Buf d = in_buf(dst.data, (size_t)dst.w * dst.h, gsb::WS_STAGE_B, false);
  GS_DO(gs_b200_resize_batch((uint8_t *)d.dev, dst.w, dst.h, (const uint8_t *)s.dev, src.w, src.h, 1, S()));
  out_buf(d);
  finish();
}

void gs_downsample(struct gs_image dst, struct gs_image src) {
  GSB_ASSERT(gs_ok(src) && gs_ok(dst) && dst.w == src.w / 2 && dst.h == src.h / 2);  // reference :190
  Buf s = in_buf(src.data, (size_t)src.w * src.h, gsb::WS_STAGE_A);
  Buf d = in_buf(dst.data, (size_t)dst.w * dst.h, gsb::WS_STAGE_B, false);
  GS_DO(gs_b200_downsample_batch((uint8_t *)d.dev, (const uint8_t *)s.dev, src.w, src.h, 1, S()));
  out_buf(d);
  finish();
}

void gs_integral(struct gs_image src, unsigned *ii) {
  GSB_ASSERT(gs_ok(src) && ii);  // reference :745
  const size_t n = (size_t)src.w * src.h;
  Buf s = in_buf(src.data, n, gsb::WS_STAGE_A), d = in_buf(ii, n * 4, gsb::WS_STAGE_B, false);
  GS_DO(gs_b200_integral_batch((uint32_t *)d.dev, (const uint8_t *)s.dev, src.w, src.h, 1, S()));
  out_buf(d);
  finish();
}

unsigned gs_fast(struct gs_image img, struct gs_image scoremap, struct gs_keypoint *kps, unsigned nkps,
                 unsigned threshold) {
  GSB_ASSERT(gs_ok(img) && kps && nkps > 0);  // reference :484
  Buf s = in_buf(img.data, (size_t)img.w * img.h, gsb::WS_STAGE_A);
  // an invalid score map drops every write and reads as 0 (gs_get/gs_set, reference :143-148)
  unsigned sw = gs_ok(scoremap) ? scoremap.w : 0, sh = gs_ok(scoremap) ? scoremap.h : 0;
  Buf m = in_buf(sw ? scoremap.data : nullptr, (size_t)sw * sh, gsb::WS_STAGE_B, true);
  Buf k = in_buf(kps, sizeof(struct gs_keypoint) * (size_t)nkps, gsb::WS_STAGE_C, false);
  unsigned *cnt = static_cast<unsigned *>(gsb::workspace(S(), gsb::WS_STAGE_D, 256));
  if (!cnt) die("device workspace allocation", 1);
  uint8_t *mp = sw ? (uint8_t *)m.dev : (uint8_t *)cnt;  // never dereferenced when sw == 0
  GS_DO(gsb::fast_single((const uint8_t *)s.dev, img.w, img.h, mp, sw, sh, (struct gs_keypoint *)k.dev, cnt, nkps,
                         threshold, S()));
  unsigned n = 0;
  GS_CUDA(cudaMemcpyAsync(&n, cnt, sizeof(n), cudaMemcpyDeviceToHost, S()));
  finish();
  out_buf(m);
  out_buf(k, sizeof(struct gs_keypoint) * (size_t)n);
  finish();
  return n;
}

float gs_compute_orientation(struct gs_image img, unsigned x, unsigned y, unsigned r) {
  GSB_ASSERT(gs_ok(img) && x >= r && y >= r && x < img.w - r && y < img.h - r);  // reference :609
  Buf s = in_buf(img.data, (size_t)img.w * img.h, gsb::WS_STAGE_A);
  float *out = static_cast<float *>(gsb::workspace(S(), gsb::WS_STAGE_D, 256));
  if (!out) die("device workspace allocation", 1);
  GS_DO(gsb::orient_single((const uint8_t *)s.dev, img.w, x, y, r, out, S()));
  float a = 0;
  GS_CUDA(cudaMemcpyAsync(&a, out, sizeof(a), cudaMemcpyDeviceToHost, S()));
  finish();
  return a;
}

void gs_brief_descriptor(struct gs_image img, struct gs_keypoint *kp) {
  GSB_ASSERT(gs_ok(img) && kp);  // reference :624
  Buf s = in_buf(img.data, (size_t)img.w * img.h, gsb::WS_STAGE_A);
  Buf k = in_buf(kp, sizeof(struct gs_keypoint), gsb::WS_STAGE_C, true);
  GS_DO(gsb::brief_single((const uint8_t *)s.dev, img.w, img.h, (struct gs_keypoint *)k.dev, S()));
  out_buf(k);
  finish();
}

unsigned gs_orb_extract(struct gs_image img, struct gs_keypoint *kps, unsigned nkps, unsigned threshold,
                        uint8_t *scoremap_buffer) {
  GSB_ASSERT(gs_ok(img) && kps && nkps > 0 && scoremap_buffer);  // reference :653
  const size_t n = (size_t)img.w * img.h;
  Buf s = in_buf(img.data, n, gsb::WS_STAGE_A), m = in_buf(scoremap_buffer, n, gsb::WS_STAGE_B, true);
  Buf k = in_buf(kps, sizeof(struct gs_keypoint) * (size_t)nkps, gsb::WS_STAGE_C, false);
  unsigned *cnt = static_cast<unsigned *>(gsb::workspace(S(), gsb::WS_STAGE_D, 256));
  if (!cnt) die("device workspace allocation", 1);
  GS_DO(gs_b200_orb_extract_batch((const uint8_t *)s.dev, img.w, img.h, 1, (uint8_t *)m.dev,
                                  (struct gs_keypoint *)k.dev, cnt, nkps, threshold, S()));
  unsigned c = 0;
  GS_CUDA(cudaMemcpyAsync(&c, cnt, sizeof(c), cudaMemcpyDeviceToHost, S()));
  finish();
  out_buf(m);
  out_buf(k, sizeof(struct gs_keypoint) * (size_t)c);
  finish();
  return c;
}

void gs_filter(struct gs_image dst, struct gs_image src, struct gs_image kernel, unsigned norm) {
  GSB_ASSERT(gs_ok(src) && gs_ok(dst) && dst.w == src.w && dst.h == src.h && norm > 0);  // reference :257
  const size_t n = (size_t)src.w * src.h;
  // the weights are call parameters: fetch them to the host if the kernel image lives on the device
  int8_t small[64], *kw_host = small;
  const size_t kn = gs_ok(kernel) ? (size_t)kernel.w * kernel.h : 0;
  if (kn > sizeof(small)) kw_host = static_cast<int8_t *>(malloc(kn));
  if (kn && !kw_host) die("host allocation", 1);
  if (kn) {
    if (on_device(kernel.data)) {
      GS_CUDA(cudaMemcpy(kw_host, kernel.data, kn, cudaMemcpyDeviceToHost));
    } else {
      memcpy(kw_host, kernel.data, kn);
    }
  }
  Buf s = in_buf(src.data, n, gsb::WS_STAGE_A), d = in_buf(dst.data, n, gsb::WS_STAGE_B, false);
  GS_DO(gs_b200_filter_batch((uint8_t *)d.dev, (const uint8_t *)s.dev, src.w, src.h, 1, kn ? kw_host : nullptr,
                             kn ? kernel.w : 0, kn ? kernel.h : 0, norm, S()));
  out_buf(d);
  finish();
  if (kw_host != small) free(kw_host);
}

void gs_match_template(struct gs_image img, struct gs_image tmpl, struct gs_image result) {
  GSB_ASSERT(gs_ok(img) && gs_ok(tmpl) && gs_ok(result));                                   // reference :706
  GSB_ASSERT(img.w >= tmpl.w && img.h >= tmpl.h);                                            // reference :707
  GSB_ASSERT(result.w == img.w - tmpl.w + 1 && result.h == img.h - tmpl.h + 1);              // reference :708
  Buf s = in_buf(img.data, (size_t)img.w * img.h, gsb::WS_STAGE_A);
  Buf t = in_buf(tmpl.data, (size_t)tmpl.w * tmpl.h, gsb::WS_STAGE_B);
  Buf r = in_buf(result.data, (size_t)result.w * result.h, gsb::WS_STAGE_C, false);
  GS_DO(gs_b200_match_template_batch((uint8_t *)r.dev, (const uint8_t *)s.dev, img.w, img.h, 1, (const uint8_t *)t.dev,
                                     tmpl.w, tmpl.h, S()));
  out_buf(r);
  finish();
}

struct gs_point gs_find_best_match(struct gs_image result) {
  GSB_ASSERT(gs_ok(result));  // reference :727
  Buf r = in_buf(result.data, (size_t)result.w * result.h, gsb::WS_STAGE_A);
  struct gs_point *p = static_cast<struct gs_point *>(gsb::workspace(S(), gsb::WS_STAGE_D, 256));
  if (!p) die("device workspace allocation", 1);
  GS_DO(gs_b200_find_best_match_batch(p, (const uint8_t *)r.dev, result.w, result.h, 1, S()));
  struct gs_point out = {0, 0};
  GS_CUDA(cudaMemcpyAsync(&out, p, sizeof(out), cudaMemcpyDeviceToHost, S()));
  finish();
  return out;
}

void gs_histogram(struct gs_image img, unsigned hist[256]) {
  GSB_ASSERT(gs_ok(img) && hist != NULL);  // reference :200
  Buf s = in_buf(img.data, (size_t)img.w * img.h, gsb::WS_STAGE_A);
  Buf d = in_buf(hist, sizeof(unsigned) * 256, gsb::WS_STAGE_B, false);
  GS_DO(gs_b200_histogram_batch((unsigned *)d.dev, (const uint8_t *)s.dev, img.w, img.h, 1, S()));
  out_buf(d);
  finish();
}

uint8_t gs_otsu_threshold(struct gs_image img) {
  GSB_ASSERT(gs_ok(img));  // reference :206
  Buf s = in_buf(img.data, (size_t)img.w * img.h, gsb::WS_STAGE_A);
  uint8_t *t = static_cast<uint8_t *>(gsb::workspace(S(), gsb::WS_STAGE_D, 256));
  if (!t) die("device workspace allocation", 1);
  GS_DO(gs_b200_otsu_threshold_batch(t, nullptr, (const uint8_t *)s.dev, img.w, img.h, 1, S()));
  uint8_t out = 0;
  GS_CUDA(cudaMemcpyAsync(&out, t, 1, cudaMemcpyDeviceToHost, S()));
  finish();
  return out;
}

void gs_threshold(struct gs_image img, uint8_t thresh) {
  GSB_ASSERT(gs_ok(img));  // reference :227
  Buf d = in_buf(img.data, (size_t)img.w * img.h, gsb::WS_STAGE_A);
  GS_DO(gs_b200_threshold_batch((uint8_t *)d.dev, img.w, img.h, 1, thresh, S()));
  out_buf(d);
  finish();
}

unsigned gs_match_orb(const struct gs_keypoint *kps1, unsigned n1, const struct gs_keypoint *kps2, unsigned n2,
                      struct gs_match *matches, unsigned max_matches, float max_distance) {
  GSB_ASSERT(kps1 && kps2 && matches);  // reference :683
  if (n1 == 0 || max_matches == 0) return 0;
  Buf a = in_buf(kps1, sizeof(struct gs_keypoint) * (size_t)n1, gsb::WS_STAGE_A);
  Buf b = in_buf(n2 ? kps2 : nullptr, sizeof(struct gs_keypoint) * (size_t)n2, gsb::WS_STAGE_B);
  Buf m = in_buf(matches, sizeof(struct gs_match) * (size_t)max_matches, gsb::WS_STAGE_C, false);
  unsigned *ctl = static_cast<unsigned *>(gsb::workspace(S(), gsb::WS_STAGE_D, 256));
  if (!ctl) die("device workspace allocation", 1);
  const unsigned hn[2] = {n1, n2};
  GS_CUDA(cudaMemcpyAsync(ctl, hn, sizeof(hn), cudaMemcpyHostToDevice, S()));
  const struct gs_keypoint *k2 = n2 ? (const struct gs_keypoint *)b.dev : (const struct gs_keypoint *)a.dev;
  GS_DO(gs_b200_match_orb_batch((const struct gs_keypoint *)a.dev, ctl, n1, k2, ctl + 1, n2 ? n2 : 1, 1,
                                (struct gs_match *)m.dev, ctl + 2, max_matches, max_distance, S()));
  unsigned c = 0;
  GS_CUDA(cudaMemcpyAsync(&c, ctl + 2, sizeof(c), cudaMemcpyDeviceToHost, S()));
  finish();
  out_buf(m, sizeof(struct gs_match) * (size_t)c);
  finish();
  return c;
}

unsigned gs_blobs(struct gs_image img, gs_label *labels, struct gs_blob *blobs, unsigned nblobs) {
  GSB_ASSERT(gs_ok(img) && labels != NULL && blobs != NULL && nblobs > 0);  // reference :335
  const size_t n = (size_t)img.w * img.h;
  Buf s = in_buf(img.data, n, gsb::WS_STAGE_A), l = in_buf(labels, n * sizeof(gs_label), gsb::WS_STAGE_B, false);
  Buf b = in_buf(blobs, sizeof(struct gs_blob) * (size_t)nblobs, gsb::WS_STAGE_C, false);
  unsigned *cnt = static_cast<unsigned *>(gsb::workspace(S(), gsb::WS_STAGE_D, 256));
  if (!cnt) die("device workspace allocation", 1);
  GS_DO(gs_b200_blobs_batch((const uint8_t *)s.dev, img.w, img.h, 1, (gs_label *)l.dev, (struct gs_blob *)b.dev, cnt, nblobs,
                            S()));
  unsigned m = 0;
  GS_CUDA(cudaMemcpyAsync(&m, cnt, sizeof(m), cudaMemcpyDeviceToHost, S()));
  finish();
  out_buf(l);
  out_buf(b, sizeof(struct gs_blob) * (size_t)m);
  finish();
  return m;
}

void gs_blob_corners(struct gs_image img, gs_label *labels, struct gs_blob *b, struct gs_point c[4]) {
  GSB_ASSERT(gs_ok(img) && b && labels);  // reference :409
  const size_t n = (size_t)img.w * img.h;
  Buf s = in_buf(img.data, n, gsb::WS_STAGE_A), l = in_buf(labels, n * sizeof(gs_label), gsb::WS_STAGE_B);
  Buf bb = in_buf(b, sizeof(struct gs_blob), gsb::WS_STAGE_C);
  unsigned *out = static_cast<unsigned *>(gsb::workspace(S(), gsb::WS_STAGE_D, 256));
  if (!out) die("device workspace allocation", 1);
  GS_DO(gs_b200_blob_corners((const uint8_t *)s.dev, img.w, img.h, (const gs_label *)l.dev, (const struct gs_blob *)bb.dev,
                             (struct gs_point *)out, S()));
  if (on_device(c)) {
    GS_CUDA(cudaMemcpyAsync(c, out, 4 * sizeof(struct gs_point), cudaMemcpyDeviceToDevice, S()));
  } else {
    GS_CUDA(cudaMemcpyAsync(c, out, 4 * sizeof(struct gs_point), cudaMemcpyDeviceToHost, S()));
  }
  finish();
}

void gs_perspective_correct(struct gs_image dst, struct gs_image src, struct gs_point c[4]) {
  GSB_ASSERT(gs_ok(dst) && gs_ok(src));  // reference :424
  struct gs_point hc[4];
  if (on_device(c)) {
    GS_CUDA(cudaMemcpy(hc, c, sizeof(hc), cudaMemcpyDeviceToHost));
  } else {
    memcpy(hc, c, sizeof(hc));
  }
  Buf s = in_buf(src.data, (size_t)src.w * src.h, gsb::WS_STAGE_A);
  Buf d = in_buf(dst.data, (size_t)dst.w * dst.h, gsb::WS_STAGE_B, false);
  GS_DO(gs_b200_perspective_correct_batch((uint8_t *)d.dev, dst.w, dst.h, (const uint8_t *)s.dev, src.w, src.h, 1, hc, 0, S()));
  out_buf(d);
  finish();
}

unsigned gs_lbp_window(const struct gs_lbp_cascade *c, const unsigned *ii, unsigned iw, unsigned ih, int x, int y,
                       float scale) {
  GSB_ASSERT(c && ii);
  const int win_w = (int)((float)c->window_w * scale), win_h = (int)((float)c->window_h * scale);
  if (x + win_w > (int)iw || y + win_h > (int)ih) return 0;  // reference :793
  Buf t = in_buf(ii, (size_t)iw * ih * 4, gsb::WS_STAGE_A);
  unsigned *out = static_cast<unsigned *>(gsb::workspace(S(), gsb::WS_STAGE_D, 256));
  if (!out) die("device workspace allocation", 1);
  GS_DO(gsb::lbp_window_single(c, (const uint32_t *)t.dev, iw, ih, x, y, scale, out, S()));
  unsigned r = 0;
  GS_CUDA(cudaMemcpyAsync(&r, out, sizeof(r), cudaMemcpyDeviceToHost, S()));
  finish();
  return r;
}

unsigned gs_lbp_detect(const struct gs_lbp_cascade *c, const unsigned *ii, unsigned iw, unsigned ih,
                       struct gs_rect *rects, unsigned max_rects, float scale_factor, float min_scale,
                       float max_scale, int step) {
  GSB_ASSERT(c && ii);
  if (max_rects == 0) return 0;
  Buf t = in_buf(ii, (size_t)iw * ih * 4, gsb::WS_STAGE_A);
  Buf r = in_buf(rects, sizeof(struct gs_rect) * (size_t)max_rects, gsb::WS_STAGE_C, false);
  unsigned *cnt = static_cast<unsigned *>(gsb::workspace(S(), gsb::WS_STAGE_D, 256));
  if (!cnt) die("device workspace allocation", 1);
  GS_DO(gs_b200_lbp_detect_batch(c, (const uint32_t *)t.dev, iw, ih, 1, (struct gs_rect *)r.dev, cnt, max_rects,
                                 scale_factor, min_scale, max_scale, step, S()));
  unsigned n = 0;
  GS_CUDA(cudaMemcpyAsync(&n, cnt, sizeof(n), cudaMemcpyDeviceToHost, S()));
  finish();
  out_buf(r, sizeof(struct gs_rect) * (size_t)n);
  finish();
  return n;
}

}  // extern "C"
