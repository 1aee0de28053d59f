/*
 * gs_oracle.c -- TEST INFRASTRUCTURE, not product code.
 *
 * A plain-C99 CPU restatement of the grayskull hot path, written from the reference's
 * semantics (each function cites the reference grayskull.h lines it follows) in the
 * data-parallel forms the CUDA kernels use: analytic clipped-window counts, separable box
 * sums, 16-bit ring masks for FAST, the 4x4 corner lattice for LBP codes, counting-sort
 * ranks for the stable keypoint sort, and double/float restatements of glibc 2.39's
 * sinf / atan2f.  Parity status: PINNED -- tests/test_oracle.py checks every function here
 * against (a) the literal vectors of the reference's own test.c, (b) the real reference
 * compiled from an upstream checkout (oracle/_ref/libgs_ref.so) on random inputs, and (c) the
 * committed fixtures in tests/golden/ that the real reference generated.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may load this file's
 * shared object; the product path (grayskull_b200/) never does.
 */
#include <limits.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "grayskull.h" /* ../include: stand-alone mode, types only */

#define GSO_API __attribute__((visibility("default")))

/* ------------------------------------------------------------------------------------------
 * clipped box statistics shared by blur and adaptive threshold (grayskull.h:233-243,270-280):
 * the sum is separable, the count is analytic: (#in-image columns) x (#in-image rows).
 * ---------------------------------------------------------------------------------------- */
static void box_sum_count(const uint8_t *src, unsigned w, unsigned h, unsigned r, uint32_t *sum,
                          uint32_t *count) {
  uint32_t *col = (uint32_t *)malloc((size_t)w * h * sizeof(uint32_t));
  for (unsigned x = 0; x < w; x++) { /* vertical pass */
    for (unsigned y = 0; y < h; y++) {
      long y0 = (long)y - (long)r, y1 = (long)y + (long)r;
      if (y0 < 0) y0 = 0;
      if (y1 > (long)h - 1) y1 = (long)h - 1;
      uint32_t s = 0;
      for (long yy = y0; yy <= y1; yy++) s += src[yy * w + x];
      col[(size_t)y * w + x] = s;
    }
  }
  for (unsigned y = 0; y < h; y++) { /* horizontal pass */
    long y0 = (long)y - (long)r, y1 = (long)y + (long)r;
    if (y0 < 0) y0 = 0;
    if (y1 > (long)h - 1) y1 = (long)h - 1;
    for (unsigned x = 0; x < w; x++) {
      long x0 = (long)x - (long)r, x1 = (long)x + (long)r;
      if (x0 < 0) x0 = 0;
      if (x1 > (long)w - 1) x1 = (long)w - 1;
      uint32_t s = 0;
      for (long xx = x0; xx <= x1; xx++) s += col[(size_t)y * w + xx];
      sum[(size_t)y * w + x] = s;
      count[(size_t)y * w + x] = (uint32_t)((x1 - x0 + 1) * (y1 - y0 + 1));
    }
  }
  free(col);
}

/* gs_blur, grayskull.h:268-283: dst = (u8)(sum / count), every pixel written */
GSO_API void gso_blur(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned r) {
  uint32_t *sum = (uint32_t *)malloc((size_t)w * h * 4), *cnt = (uint32_t *)malloc((size_t)w * h * 4);
  box_sum_count(src, w, h, r, sum, cnt);
  for (size_t i = 0; i < (size_t)w * h; i++) dst[i] = (uint8_t)(sum[i] / cnt[i]);
  free(sum);
  free(cnt);
}

/* gs_adaptive_threshold, grayskull.h:230-247: int threshold = mean - c; src > threshold ? 255:0 */
GSO_API void gso_adaptive_threshold(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h,
                                    unsigned r, int c) {
  uint32_t *sum = (uint32_t *)malloc((size_t)w * h * 4), *cnt = (uint32_t *)malloc((size_t)w * h * 4);
  box_sum_count(src, w, h, r, sum, cnt);
  for (size_t i = 0; i < (size_t)w * h; i++) {
    /* unsigned mean minus c wraps to the mathematically expected signed value */
    int threshold = (int)((sum[i] / cnt[i]) - (unsigned)c);
    dst[i] = ((int)src[i] > threshold) ? 255 : 0;
  }
  free(sum);
  free(cnt);
}

/* gs_erode / gs_dilate, grayskull.h:285-304: min/max over the in-bounds 3x3 neighbours */
GSO_API void gso_morph(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, int dilate) {
  for (unsigned y = 0; y < h; y++)
    for (unsigned x = 0; x < w; x++) {
      unsigned v = dilate ? 0u : 255u;
      for (int dy = -1; dy <= 1; dy++)
        for (int dx = -1; dx <= 1; dx++) {
          long yy = (long)y + dy, xx = (long)x + dx;
          if (yy < 0 || yy >= (long)h || xx < 0 || xx >= (long)w) continue;
          unsigned p = src[yy * w + xx];
          v = dilate ? (p > v ? p : v) : (p < v ? p : v);
        }
      dst[(size_t)y * w + x] = (uint8_t)v;
    }
}

/* gs_sobel, grayskull.h:306-320: interior only; the 1-px dst frame is never written.
 * Restated via |gx|+|gy| = max(|gx+gy|, |gx-gy|), which is how the kernel evaluates it. */
GSO_API void gso_sobel(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h) {
  if (w < 3 || h < 3) return;
  for (unsigned y = 1; y + 1 < h; y++)
    for (unsigned x = 1; x + 1 < w; x++) {
      const uint8_t *a = src + (size_t)(y - 1) * w + x, *b = a + w, *c = b + w;
      int A = (b[1] + c[0] + c[1]) - (a[-1] + a[0] + b[-1]); /* (gx + gy) / 2 */
      int B = (a[0] + a[1] + b[1]) - (b[-1] + c[-1] + c[0]); /* (gx - gy) / 2 */
      int m = abs(A) > abs(B) ? abs(A) : abs(B);
      dst[(size_t)y * w + x] = (uint8_t)(m > 255 ? 255 : m);
    }
}

/* gs_resize, grayskull.h:171-187.  fp32, evaluation order as written there, no contraction
 * (this file is built with -ffp-contract=off).  `volatile` pins each rounding step. */
GSO_API void gso_resize(uint8_t *dst, unsigned dw, unsigned dh, const uint8_t *src, unsigned sw,
                        unsigned sh) {
  for (unsigned y = 0; y < dh; y++)
    for (unsigned x = 0; x < dw; x++) {
      volatile float sx = ((float)x + 0.5f) * (float)sw;
      sx = sx / (float)dw;
      sx = sx - 0.5f;
      volatile float sy = ((float)y + 0.5f) * (float)sh;
      sy = sy / (float)dh;
      sy = sy - 0.5f;
      float mx = (float)sw - 1.0f, my = (float)sh - 1.0f;
      float fx = sx < mx ? sx : mx, fy = sy < my ? sy : my;
      fx = 0.0f > fx ? 0.0f : fx;
      fy = 0.0f > fy ? 0.0f : fy;
      unsigned x0 = (unsigned)fx, y0 = (unsigned)fy;
      unsigned x1 = x0 + 1 < sw - 1 ? x0 + 1 : sw - 1, y1 = y0 + 1 < sh - 1 ? y0 + 1 : sh - 1;
      float dx = fx - (float)x0, dy = fy - (float)y0;
      /* Above 2^24, (float)sw - 1.0f can round to sw or past it, and the reference then reads past the row (column).
       * Here that tap is the last pixel; dx (dy) is 0 there, so the result is the last pixel's value. */
      x0 = x0 < sw - 1 ? x0 : sw - 1;
      y0 = y0 < sh - 1 ? y0 : sh - 1;
      float c00 = src[(size_t)y0 * sw + x0], c01 = src[(size_t)y0 * sw + x1];
      float c10 = src[(size_t)y1 * sw + x0], c11 = src[(size_t)y1 * sw + x1];
      volatile float omx = 1 - dx, omy = 1 - dy;
      volatile float t0 = c00 * omx, t1 = c01 * dx, t2 = c10 * omx, t3 = c11 * dx;
      t0 = t0 * omy;
      t1 = t1 * omy;
      t2 = t2 * dy;
      t3 = t3 * dy;
      volatile float acc = t0 + t1;
      acc = acc + t2;
      acc = acc + t3;
      dst[(size_t)y * dw + x] = (uint8_t)acc;
    }
}

/* gs_downsample, grayskull.h:189-197: (a+b+c+d)/4, dst = floor(src/2) */
GSO_API void gso_downsample(uint8_t *dst, const uint8_t *src, unsigned sw, unsigned sh) {
  unsigned dw = sw / 2, dh = sh / 2;
  for (unsigned y = 0; y < dh; y++)
    for (unsigned x = 0; x < dw; x++) {
      const uint8_t *p = src + (size_t)(2 * y) * sw + 2 * x;
      dst[(size_t)y * dw + x] = (uint8_t)((p[0] + p[1] + p[sw] + p[sw + 1]) / 4);
    }
}

/* gs_integral, grayskull.h:744-752: inclusive SAT, modular u32.  Restated as column prefix
 * then row prefix (any association order is bit-identical in modular arithmetic). */
GSO_API void gso_integral(const uint8_t *src, unsigned w, unsigned h, uint32_t *ii) {
  for (unsigned x = 0; x < w; x++) {
    uint32_t s = 0;
    for (unsigned y = 0; y < h; y++) s += src[(size_t)y * w + x], ii[(size_t)y * w + x] = s;
  }
  for (unsigned y = 0; y < h; y++) {
    uint32_t s = 0;
    for (unsigned x = 0; x < w; x++) s += ii[(size_t)y * w + x], ii[(size_t)y * w + x] = s;
  }
}

/* ------------------------------------------------------------------------------------------
 * FAST-9, grayskull.h:482-534, mask form:
 *   brighter_i = v_i > p + t
 *   darker_i   = !brighter_i && (t > p ? 1 : v_i < p - t)     <- the unsigned wrap at :498
 *   corner     = a circular run of >= 9 set bits in either 16-bit mask
 *   score      = corner ? min_j |v_j - p| : 0, written for 3 <= x <= w-4, 3 <= y <= h-4 only
 * NMS (:517-532) reads the 8 neighbours out of the caller's map, including ring cells that
 * pass 1 never wrote; survivors are emitted in raster order while n < nkps.
 * ---------------------------------------------------------------------------------------- */
static const int fast_dx[16] = {0, 1, 2, 3, 3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1};
static const int fast_dy[16] = {-3, -3, -2, -1, 0, 1, 2, 3, 3, 3, 2, 1, 0, -1, -2, -3};

static int run9(unsigned m) { /* circular run >= 9 in a 16-bit mask */
  unsigned mm = m | (m << 16);
  unsigned r = mm & (mm >> 1);
  r &= r >> 2;
  r &= r >> 4;
  r &= mm >> 8;
  return (r & 0xFFFFu) != 0;
}

GSO_API unsigned gso_fast(const uint8_t *img, unsigned w, unsigned h, uint8_t *scoremap,
                          unsigned sw, unsigned sh, struct gs_keypoint *kps, unsigned nkps,
                          unsigned t) {
  unsigned n = 0;
  if (w < 7 || h < 7) return 0;
  for (unsigned y = 3; y + 3 < h; y++)
    for (unsigned x = 3; x + 3 < w; x++) {
      unsigned p = img[(size_t)y * w + x], hi = p + t, bright = 0, dark = 0, mind = 255;
      for (int i = 0; i < 16; i++) {
        unsigned v = img[(size_t)(y + fast_dy[i]) * w + (x + fast_dx[i])];
        int b = v > hi;
        int d = !b && (t > p ? 1 : v < p - t);
        bright |= (unsigned)b << i;
        dark |= (unsigned)d << i;
        unsigned ad = v > p ? v - p : p - v;
        if (ad < mind) mind = ad;
      }
      unsigned score = (run9(bright) || run9(dark)) ? mind : 0;
      if (scoremap && x < sw && y < sh) scoremap[(size_t)y * sw + x] = (uint8_t)score;
    }
  for (unsigned y = 3; y + 3 < h; y++)
    for (unsigned x = 3; x + 3 < w; x++) {
      /* gs_get semantics on the score map: out of range reads give 0 (grayskull.h:143-145) */
#define SM(xx, yy) ((scoremap && (xx) < sw && (yy) < sh) ? scoremap[(size_t)(yy) * sw + (xx)] : 0)
      unsigned s = SM(x, y);
      if (!s) continue;
      int is_max = 1;
      for (int yy = -1; yy <= 1 && is_max; yy++)
        for (int xx = -1; xx <= 1; xx++)
          if ((xx || yy) && SM(x + xx, y + yy) > s) {
            is_max = 0;
            break;
          }
#undef SM
      if (is_max && n < nkps) {
        memset(&kps[n], 0, sizeof(kps[n]));
        kps[n].pt.x = x, kps[n].pt.y = y, kps[n].response = s;
        n++;
      }
    }
  return n;
}

/* ------------------------------------------------------------------------------------------
 * glibc 2.39 float trigonometry, restated (the reference calls libm: grayskull.h:100-101).
 *   sinf   : sysdeps/ieee754/flt-32/s_sinf.c + sincosf.h (double evaluation, |x| < 120 path)
 *   atan2f : sysdeps/ieee754/flt-32/e_atan2f.c + s_atanf.c (float evaluation)
 * tools/validate_trig.c checks these exhaustively against the container's libm
 * (all floats |x| <= 8 for sinf, all floats for atanf, 2e8 moment pairs for atan2f: 0 diffs).
 * ---------------------------------------------------------------------------------------- */
static uint32_t f2u(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  return u;
}
static float u2f(uint32_t u) {
  float f;
  memcpy(&f, &u, 4);
  return f;
}

GSO_API float gso_sinf(float y) {
  static const double HPI_INV = 0x1.45F306DC9C883p+23, HPI = 0x1.921FB54442D18p0;
  static const double C0 = 0x1p0, C1 = -0x1.ffffffd0c621cp-2, C2 = 0x1.55553e1068f19p-5,
                      C3 = -0x1.6c087e89a359dp-10, C4 = 0x1.99343027bf8c3p-16;
  static const double S1 = -0x1.555545995a603p-3, S2 = 0x1.1107605230bc4p-7,
                      S3 = -0x1.994eb3774cf24p-13;
  double x = y, x2;
  int n = 0, negc = 0;
  uint32_t top = (f2u(y) >> 20) & 0x7ff;
  if (top < ((f2u(0x1.921FB6p-1f) >> 20) & 0x7ff)) {
    if (top < ((f2u(0x1p-12f) >> 20) & 0x7ff)) return y;
    x2 = x * x;
  } else if (top < ((f2u(120.0f) >> 20) & 0x7ff)) {
    double r = x * HPI_INV;
    n = ((int32_t)r + 0x800000) >> 24;
    double xr = fma(-(double)n, HPI, x);
    x2 = xr * xr;
    x = (n & 3) == 1 || (n & 3) == 2 ? -xr : xr;
    negc = (n & 2) != 0;
  } else {
    return sinf(y); /* outside the hot path's domain (|angle| <= pi + pi/2) */
  }
  if ((n & 1) == 0) {
    double x3 = x * x2, s1 = fma(x2, S3, S2), x7 = x3 * x2, s = fma(x3, S1, x);
    return (float)fma(x7, s1, s);
  } else {
    double sg = negc ? -1.0 : 1.0;
    double x4 = x2 * x2, c2 = fma(x2, sg * C4, sg * C3), c1 = fma(x2, sg * C1, sg * C0);
    double x6 = x4 * x2, c = fma(x4, sg * C2, c1);
    return (float)fma(x6, c2, c);
  }
}

static float gso_atanf(float x) {
  static const float atanhi[] = {4.6364760399e-01f, 7.8539812565e-01f, 9.8279368877e-01f,
                                 1.5707962513e+00f};
  static const float atanlo[] = {5.0121582440e-09f, 3.7748947079e-08f, 3.4473217170e-08f,
                                 7.5497894159e-08f};
  static const float aT[] = {3.3333334327e-01f,  -2.0000000298e-01f, 1.4285714924e-01f,
                             -1.1111110449e-01f, 9.0908870101e-02f,  -7.6918758452e-02f,
                             6.6610731184e-02f,  -5.8335702866e-02f, 4.9768779427e-02f,
                             -3.6531571299e-02f, 1.6285819933e-02f};
  float w, s1, s2, z;
  int32_t hx = (int32_t)f2u(x), ix = hx & 0x7fffffff, id;
  if (ix >= 0x4c000000) {
    if (ix > 0x7f800000) return x + x;
    return hx > 0 ? atanhi[3] + atanlo[3] : -atanhi[3] - atanlo[3];
  }
  if (ix < 0x3ee00000) {
    if (ix < 0x31000000) return x;
    id = -1;
  } else {
    x = fabsf(x);
    if (ix < 0x3f980000) {
      if (ix < 0x3f300000) id = 0, x = (2.0f * x - 1.0f) / (2.0f + x);
      else id = 1, x = (x - 1.0f) / (x + 1.0f);
    } else {
      if (ix < 0x401c0000) id = 2, x = (x - 1.5f) / (1.0f + 1.5f * x);
      else id = 3, x = -1.0f / x;
    }
  }
  z = x * x;
  w = z * z;
  s1 = z * (aT[0] + w * (aT[2] + w * (aT[4] + w * (aT[6] + w * (aT[8] + w * aT[10])))));
  s2 = w * (aT[1] + w * (aT[3] + w * (aT[5] + w * (aT[7] + w * aT[9]))));
  if (id < 0) return x - x * (s1 + s2);
  z = atanhi[id] - ((x * (s1 + s2) - atanlo[id]) - x);
  return hx < 0 ? -z : z;
}

GSO_API float gso_atan2f(float y, float x) {
  static const float pi_o_2 = 1.5707963705e+00f, pi = 3.1415927410e+00f,
                     pi_lo = -8.7422776573e-08f, tiny = 1.0e-30f;
  float z;
  int32_t hx = (int32_t)f2u(x), ix = hx & 0x7fffffff, hy = (int32_t)f2u(y), iy = hy & 0x7fffffff;
  if (ix > 0x7f800000 || iy > 0x7f800000) return x + y;
  if (hx == 0x3f800000) return gso_atanf(y);
  int m = ((hy >> 31) & 1) | ((hx >> 30) & 2);
  if (iy == 0) return m < 2 ? y : (m == 2 ? pi + tiny : -pi - tiny);
  if (ix == 0) return hy < 0 ? -pi_o_2 - tiny : pi_o_2 + tiny;
  int k = (iy - ix) >> 23;
  if (k > 60) z = pi_o_2 + 0.5f * pi_lo;
  else if (hx < 0 && k < -60) z = 0.0f;
  else z = gso_atanf(fabsf(y / x));
  switch (m) {
    case 0: return z;
    case 1: return u2f(f2u(z) ^ 0x80000000u);
    case 2: return pi - (z - pi_lo);
    default: return (z - pi_lo) - pi;
  }
}

/* gs_compute_orientation, grayskull.h:608-621: for r <= 15 the float accumulators there only ever hold
 * integers below 2^24 (r = 15: sum|dy| = 4528, x255 < 2^24), so int32 moments are identical; beyond
 * that the sums can round, and the fp32 accumulation is repeated in the reference's dy-outer / dx-inner order */
GSO_API float gso_compute_orientation(const uint8_t *img, unsigned w, unsigned h, unsigned x,
                                      unsigned y, unsigned r) {
  int m01 = 0, m10 = 0, ri = (int)r;
  (void)h;
  if (r > 15) {
    volatile float f01 = 0.0f, f10 = 0.0f;
    for (int dy = -ri; dy <= ri; dy++)
      for (int dx = -ri; dx <= ri; dx++)
        if (dx * dx + dy * dy <= (int)(r * r)) {
          int v = img[(size_t)((int)y + dy) * w + (size_t)((int)x + dx)];
          f01 = f01 + (float)(dy * v), f10 = f10 + (float)(dx * v);
        }
    return gso_atan2f(f01, f10);
  }
  for (int dy = -ri; dy <= ri; dy++)
    for (int dx = -ri; dx <= ri; dx++)
      if (dx * dx + dy * dy <= ri * ri) {
        int v = img[(size_t)((int)y + dy) * w + (size_t)((int)x + dx)];
        m01 += dy * v, m10 += dx * v;
      }
  return gso_atan2f((float)m01, (float)m10);
}

static const uint32_t brief_pairs[256] = {
#include "brief_pattern.inc"
};

/* gs_brief_descriptor, grayskull.h:623-637.  Note cos = sin(angle + 1.57079f) (6-digit pi/2),
 * products and sums in fp32 without contraction, (int) truncation, out-of-image samples = 0 */
GSO_API void gso_brief_descriptor(const uint8_t *img, unsigned w, unsigned h,
                                  struct gs_keypoint *kp) {
  int x = (int)kp->pt.x, y = (int)kp->pt.y;
  float sin_a = gso_sinf(kp->angle), cos_a = gso_sinf(kp->angle + 1.57079f);
  for (int i = 0; i < 8; i++) kp->descriptor[i] = 0;
  for (int i = 0; i < 256; i++) {
    uint32_t pk = brief_pairs[i];
    float p0 = (float)(int8_t)(pk & 0xFF), p1 = (float)(int8_t)((pk >> 8) & 0xFF);
    float p2 = (float)(int8_t)((pk >> 16) & 0xFF), p3 = (float)(int8_t)(pk >> 24);
    volatile float a, b;
    a = p0 * cos_a, b = p1 * sin_a;
    float dx1 = a - b;
    a = p0 * sin_a, b = p1 * cos_a;
    float dy1 = a + b;
    a = p2 * cos_a, b = p3 * sin_a;
    float dx2 = a - b;
    a = p2 * sin_a, b = p3 * cos_a;
    float dy2 = a + b;
    unsigned x1 = (unsigned)(x + (int)dx1), y1 = (unsigned)(y + (int)dy1);
    unsigned x2 = (unsigned)(x + (int)dx2), y2 = (unsigned)(y + (int)dy2);
    unsigned i1 = (x1 < w && y1 < h) ? img[(size_t)y1 * w + x1] : 0;
    unsigned i2 = (x2 < w && y2 < h) ? img[(size_t)y2 * w + x2] : 0;
    if (i1 > i2) kp->descriptor[i / 32] |= 1u << (i % 32);
  }
}

/* gs_sort_keypoints, grayskull.h:639-649: the bubble sort is a STABLE descending sort on
 * `response`; restated as a counting-sort rank (what the GPU does) */
GSO_API void gso_sort_keypoints(struct gs_keypoint *kps, unsigned n) {
  if (n < 2) return;
  struct gs_keypoint *tmp = (struct gs_keypoint *)malloc((size_t)n * sizeof(*tmp));
  unsigned hist[257];
  memset(hist, 0, sizeof(hist));
  for (unsigned i = 0; i < n; i++) hist[255 - (kps[i].response > 255 ? 255 : kps[i].response)]++;
  unsigned acc = 0;
  for (int b = 0; b < 256; b++) {
    unsigned c = hist[b];
    hist[b] = acc, acc += c;
  }
  for (unsigned i = 0; i < n; i++)
    tmp[hist[255 - (kps[i].response > 255 ? 255 : kps[i].response)]++] = kps[i];
  memcpy(kps, tmp, (size_t)n * sizeof(*tmp));
  free(tmp);
}

/* gs_orb_extract, grayskull.h:651-669 */
GSO_API unsigned gso_orb_extract(const uint8_t *img, unsigned w, unsigned h,
                                 struct gs_keypoint *kps, unsigned nkps, unsigned threshold,
                                 uint8_t *scoremap_buffer) {
  unsigned cap = nkps * 4 < 5000 ? nkps * 4 : 5000;
  struct gs_keypoint *cand = (struct gs_keypoint *)malloc(5000 * sizeof(*cand));
  unsigned nf = gso_fast(img, w, h, scoremap_buffer, w, h, cand, cap, threshold);
  gso_sort_keypoints(cand, nf);
  unsigned n = 0, radius = 15;
  for (unsigned i = 0; i < nf && n < nkps; i++) {
    unsigned x = cand[i].pt.x, y = cand[i].pt.y;
    if (x >= radius && y >= radius && x < w - radius && y < h - radius) {
      kps[n] = cand[i];
      kps[n].angle = gso_compute_orientation(img, w, h, x, y, radius);
      gso_brief_descriptor(img, w, h, &kps[n]);
      n++;
    }
  }
  free(cand);
  return n;
}

/* ------------------------------------------------------------------------------------------
 * gs_match_orb, grayskull.h:671-699 (SURVEY.md 8f, N1).  For query i the reference's sequential scan
 * keeps the two smallest Hamming distances of the multiset {d_j} U {M, M}, M = max_distance + 1
 * (fp32), best_idx = the first j attaining the smallest (0 if none is below M); a match is emitted
 * when best <= max_distance and best < 0.8f * second (fp32 product), in query order, until
 * max_matches.  Restated with an order-free two-minimum merge (what the GPU's lanes do).
 * ---------------------------------------------------------------------------------------- */
struct gso_match {
  unsigned idx1, idx2, distance;
};
static unsigned hamming256(const uint32_t *a, const uint32_t *b) {
  unsigned d = 0;
  for (int i = 0; i < 8; i++) d += (unsigned)__builtin_popcount(a[i] ^ b[i]);
  return d;
}
GSO_API unsigned gso_match_orb(const struct gs_keypoint *k1, unsigned n1, const struct gs_keypoint *k2, unsigned n2,
                               struct gso_match *matches, unsigned max_matches, float max_distance) {
  unsigned n = 0;
  const float M = max_distance + 1;
  for (unsigned i = 0; i < n1 && n < max_matches; i++) {
    /* four interleaved partial scans (as GPU lanes would), merged afterwards */
    float best[4], second[4];
    unsigned bidx[4];
    for (int l = 0; l < 4; l++) best[l] = M, second[l] = M, bidx[l] = 0xFFFFFFFFu;
    for (unsigned j = 0; j < n2; j++) {
      const int l = (int)(j & 3);
      const float d = (float)hamming256(k1[i].descriptor, k2[j].descriptor);
      if (d < best[l]) second[l] = best[l], best[l] = d, bidx[l] = j;
      else if (d < second[l]) second[l] = d;
    }
    float b = M, s = M;
    unsigned bi = 0xFFFFFFFFu;
    for (int l = 0; l < 4; l++) {
      /* merge (b, bi, s) with (best[l], bidx[l], second[l]) */
      float nb, ns, loser;
      unsigned ni;
      if (best[l] < b || (best[l] == b && bidx[l] < bi)) nb = best[l], ni = bidx[l], loser = b;
      else nb = b, ni = bi, loser = best[l];
      ns = loser < s ? loser : s;
      ns = second[l] < ns ? second[l] : ns;
      b = nb, bi = ni, s = ns;
    }
    if (bi == 0xFFFFFFFFu) bi = 0;
    if (b <= max_distance && b < 0.8f * s) {
      matches[n].idx1 = i, matches[n].idx2 = bi, matches[n].distance = (unsigned)b;
      n++;
    }
  }
  return n;
}

/* ------------------------------------------------------------------------------------------
 * LBP cascade, grayskull.h:769-835.  The 9 box sums of gs_lbp_code (36 loads) are taken from
 * a 4x4 lattice of integral-image corners (16 loads), corner(-1,.) = corner(.,-1) = 0.
 * ---------------------------------------------------------------------------------------- */
static uint32_t corner(const uint32_t *ii, unsigned iw, int x, int y) {
  return (x < 0 || y < 0) ? 0u : ii[(size_t)y * iw + (size_t)x];
}

static int lbp_code(const uint32_t *ii, unsigned iw, int x0, int y0, int fw, int fh) {
  uint32_t g[4][4], cell[3][3];
  for (int j = 0; j < 4; j++)
    for (int i = 0; i < 4; i++) g[j][i] = corner(ii, iw, x0 - 1 + i * fw, y0 - 1 + j * fh);
  for (int j = 0; j < 3; j++)
    for (int i = 0; i < 3; i++) cell[j][i] = g[j + 1][i + 1] + g[j][i] - g[j][i + 1] - g[j + 1][i];
  uint32_t c = cell[1][1];
  return ((cell[0][0] >= c) << 7) | ((cell[0][1] >= c) << 6) | ((cell[0][2] >= c) << 5) |
         ((cell[1][2] >= c) << 4) | ((cell[2][2] >= c) << 3) | ((cell[2][1] >= c) << 2) |
         ((cell[2][0] >= c) << 1) | ((cell[1][0] >= c) << 0);
}

/* gs_lbp_window, grayskull.h:790-813 */
GSO_API unsigned gso_lbp_window(const struct gs_lbp_cascade *c, const uint32_t *ii, unsigned iw,
                                unsigned ih, int x, int y, float scale) {
  int win_w = (int)((float)c->window_w * scale), win_h = (int)((float)c->window_h * scale);
  if (x + win_w > (int)iw || y + win_h > (int)ih) return 0;
  for (int si = 0; si < c->nstages; si++) {
    int start = c->stage_weak_start[si], n = c->stage_nweaks[si];
    float sum = 0.0f;
    for (int i = 0; i < n; i++) {
      int wi = start + i, fi = c->weak_feature_idx[wi];
      int fx = (int)((float)c->features[fi * 4 + 0] * scale);
      int fy = (int)((float)c->features[fi * 4 + 1] * scale);
      int fw = (int)((float)c->features[fi * 4 + 2] * scale);
      int fh = (int)((float)c->features[fi * 4 + 3] * scale);
      if (fw < 1) fw = 1;
      if (fh < 1) fh = 1;
      int code = lbp_code(ii, iw, x + fx, y + fy, fw, fh);
      int idx = code >> 5, bit = code & 31;
      int match = idx < (int)c->weak_num_subsets[wi] &&
                  ((uint32_t)c->subsets[c->weak_subset_offset[wi] + idx] >> bit & 1u);
      sum += match ? c->weak_left_val[wi] : c->weak_right_val[wi];
    }
    if (sum < c->stage_threshold[si]) return 0;
  }
  return 1;
}

/* Analysis helper (not part of the reference API): for every window position of ONE scale, the number of
 * cascade stages the window passes (nstages = a detection).  Same walk as gso_lbp_window; feeds the
 * divergence / load-balance model in tools/lbp_model.py.  out: ny x nx bytes, ny = (ih - win_h) / step + 1. */
GSO_API void gso_lbp_depth_map(const struct gs_lbp_cascade *c, const uint32_t *ii, unsigned iw, unsigned ih,
                               float scale, int step, uint8_t *out) {
  int win_w = (int)((float)c->window_w * scale), win_h = (int)((float)c->window_h * scale);
  if (win_w > (int)iw || win_h > (int)ih) return;
  size_t k = 0;
  for (int y = 0; y + win_h <= (int)ih; y += step)
    for (int x = 0; x + win_w <= (int)iw; x += step) {
      int si = 0;
      for (; si < c->nstages; si++) {
        int start = c->stage_weak_start[si], n = c->stage_nweaks[si];
        float sum = 0.0f;
        for (int i = 0; i < n; i++) {
          int wi = start + i, fi = c->weak_feature_idx[wi];
          int fx = (int)((float)c->features[fi * 4 + 0] * scale), fy = (int)((float)c->features[fi * 4 + 1] * scale);
          int fw = (int)((float)c->features[fi * 4 + 2] * scale), fh = (int)((float)c->features[fi * 4 + 3] * scale);
          if (fw < 1) fw = 1;
          if (fh < 1) fh = 1;
          int code = lbp_code(ii, iw, x + fx, y + fy, fw, fh);
          int idx = code >> 5, bit = code & 31;
          int match = idx < (int)c->weak_num_subsets[wi] &&
                      ((uint32_t)c->subsets[c->weak_subset_offset[wi] + idx] >> bit & 1u);
          sum += match ? c->weak_left_val[wi] : c->weak_right_val[wi];
        }
        if (sum < c->stage_threshold[si]) break;
      }
      out[k++] = (uint8_t)si;
    }
}

/* gs_lbp_detect, grayskull.h:815-835: scales by repeated fp32 multiply, (scale, y, x) order,
 * hard stop at max_rects */
GSO_API unsigned gso_lbp_detect(const struct gs_lbp_cascade *c, const uint32_t *ii, unsigned iw,
                                unsigned ih, struct gs_rect *rects, unsigned max_rects,
                                float scale_factor, float min_scale, float max_scale, int step) {
  unsigned n = 0;
  for (volatile float scale = min_scale; scale <= max_scale && n < max_rects;
       scale = scale * scale_factor) {
    float s = scale;
    int win_w = (int)((float)c->window_w * s), win_h = (int)((float)c->window_h * s);
    if (win_w > (int)iw || win_h > (int)ih) break;
    for (int y = 0; y + win_h <= (int)ih && n < max_rects; y += step)
      for (int x = 0; x + win_w <= (int)iw && n < max_rects; x += step)
        if (gso_lbp_window(c, ii, iw, ih, x, y, s)) {
          rects[n].x = (unsigned)x, rects[n].y = (unsigned)y;
          rects[n].w = (unsigned)win_w, rects[n].h = (unsigned)win_h;
          n++;
        }
  }
  return n;
}

/* ------------------------------------------------------------------------------------------
 * SURVEY.md 8(f) N2 -- gs_histogram / gs_otsu_threshold / gs_threshold, grayskull.h:199-228.
 * Histogram: four interleaved partial histograms merged at the end (integer counts, order free).
 * Otsu: the reference's fp32 loop, statement for statement -- every intermediate is a float
 * (FLT_EVAL_METHOD 0, no contraction): sum = sum_i (float)i * (float)hist[i] accumulated in bin
 * order; per t: wb += hist[t]; skip while wb == 0; wf = npix - wb (unsigned, npix = w*h wrapped
 * to 32 bits like the reference's unsigned product); stop at wf == 0; sumB += t*hist[t];
 * var = ((wb*wf)*(mB-mF))*(mB-mF); strict > keeps the first maximum.
 * ---------------------------------------------------------------------------------------- */
GSO_API void gso_histogram(const uint8_t *src, unsigned w, unsigned h, unsigned *hist) {
  unsigned part[4][256];
  memset(part, 0, sizeof(part));
  const unsigned n = w * h;
  unsigned i = 0;
  for (; i + 4 <= n; i += 4) part[0][src[i]]++, part[1][src[i + 1]]++, part[2][src[i + 2]]++, part[3][src[i + 3]]++;
  for (; i < n; i++) part[0][src[i]]++;
  for (unsigned b = 0; b < 256; b++) hist[b] = part[0][b] + part[1][b] + part[2][b] + part[3][b];
}

GSO_API unsigned gso_otsu_from_hist(const unsigned *hist, unsigned npix) {
  float sum = 0.0f, sum_b = 0.0f, var_max = -1.0f;
  unsigned wb = 0, best = 0;
  for (unsigned i = 0; i < 256; i++) {
    const float term = (float)i * (float)hist[i];
    sum = sum + term;
  }
  for (unsigned t = 0; t < 256; t++) {
    wb += hist[t];
    if (wb == 0) continue;
    const unsigned wf = npix - wb;
    if (wf == 0) break;
    const float term = (float)t * (float)hist[t];
    sum_b = sum_b + term;
    const float m_b = sum_b / (float)wb;
    const float rest = sum - sum_b;
    const float m_f = rest / (float)wf;
    const float diff = m_b - m_f;
    float var = (float)wb * (float)wf;
    var = var * diff;
    var = var * diff;
    if (var > var_max) var_max = var, best = t;
  }
  return best & 0xFFu;
}

GSO_API unsigned gso_otsu_threshold(const uint8_t *src, unsigned w, unsigned h) {
  unsigned hist[256];
  gso_histogram(src, w, h, hist);
  return gso_otsu_from_hist(hist, w * h);
}

GSO_API void gso_threshold(uint8_t *img, unsigned w, unsigned h, unsigned thresh) {
  const unsigned n = w * h;
  const uint8_t t = (uint8_t)thresh;
  for (unsigned i = 0; i < n; i++) img[i] = (uint8_t)(-(int)(img[i] > t)); /* 0xFF or 0x00 */
}

/* ------------------------------------------------------------------------------------------
 * SURVEY.md 8(f) N3 -- gs_filter (grayskull.h:255-266), gs_match_template / gs_find_best_match
 * (grayskull.h:705-738).
 * gs_filter: zero padding through gs_get, taps at (x + i - kw/2, y + j - kh/2), weights read as
 * int8.  `sum = sum / norm` divides an int by an unsigned: the int is converted to unsigned first,
 * the 32-bit quotient goes back into the int, then the clamp -- so a negative sum gives 0 for norm 1
 * and (for any sane norm) 255 otherwise.  Restated with signed coordinates and explicit casts.
 * gs_match_template: sum of squared differences in 64 bits, score = sum*255 / (tw*th*255^2),
 * result = 255 - min(score, 255).  Restated as sum(I^2) - 2 sum(I*T) + sum(T^2) (exact in integers).
 * ---------------------------------------------------------------------------------------- */
GSO_API void gso_filter(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, const uint8_t *kernel, unsigned kw,
                        unsigned kh, unsigned norm) {
  const long ox = (long)(kw / 2), oy = (long)(kh / 2);
  for (long y = 0; y < (long)h; y++)
    for (long x = 0; x < (long)w; x++) {
      int32_t sum = 0;
      for (long j = 0; j < (long)kh; j++) {
        const long sy = y + j - oy;
        if (sy < 0 || sy >= (long)h) continue;
        for (long i = 0; i < (long)kw; i++) {
          const long sx = x + i - ox;
          if (sx < 0 || sx >= (long)w) continue;
          sum += (int32_t)src[sy * w + sx] * (int32_t)(int8_t)kernel[j * kw + i];
        }
      }
      const uint32_t q = (uint32_t)sum / norm;
      const int32_t v = (int32_t)q;
      dst[y * w + x] = (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
    }
}

GSO_API void gso_match_template(const uint8_t *img, unsigned w, unsigned h, const uint8_t *tmpl, unsigned tw, unsigned th,
                                uint8_t *result) {
  const unsigned rw = w - tw + 1, rh = h - th + 1;
  uint64_t tt = 0;
  for (unsigned k = 0; k < tw * th; k++) tt += (uint64_t)tmpl[k] * tmpl[k];
  const uint64_t max_diff = (uint64_t)tw * th * 255u * 255u;
  for (unsigned ry = 0; ry < rh; ry++)
    for (unsigned rx = 0; rx < rw; rx++) {
      uint64_t ii = 0, it = 0;
      for (unsigned ty = 0; ty < th; ty++) {
        const uint8_t *p = img + (size_t)(ry + ty) * w + rx, *q = tmpl + (size_t)ty * tw;
        for (unsigned tx = 0; tx < tw; tx++) ii += (uint64_t)p[tx] * p[tx], it += (uint64_t)p[tx] * q[tx];
      }
      const uint64_t ssd = ii + tt - 2 * it;
      const uint64_t score = ssd * 255u / max_diff;
      result[(size_t)ry * rw + rx] = (uint8_t)(255u - (unsigned)(score < 255u ? score : 255u));
    }
}

/* first strict maximum in raster order (none above 0 -> (0, 0)); returns y * w + x */
GSO_API unsigned gso_find_best_match(const uint8_t *result, unsigned w, unsigned h) {
  unsigned best = 0, best_score = 0;
  for (unsigned k = 0; k < w * h; k++)
    if (result[k] > best_score) best_score = result[k], best = k;
  return best;
}

/* ------------------------------------------------------------------------------------------
 * SURVEY.md 8(f) N4 -- gs_blobs / gs_blob_corners / gs_perspective_correct, grayskull.h:325-444.
 *
 * gs_blobs.  The reference labels in one raster pass with a union-find over provisional labels and a
 * second pass that rewrites every label to its root.  Restated without provisional labels:
 *   - a pixel receives a NEW label exactly when it is foreground (>= 128) and neither its left nor
 *     its upper neighbour carries a label; while labels last every foreground pixel is labelled, so
 *     these "seeds" are the run starts with no foreground pixel above them, numbered in raster order;
 *   - unions always keep the smaller root, so a component's final label is the smallest seed number
 *     in it = the seed number of its raster-first pixel;
 *   - once `nblobs` seeds have been handed out (:349 "out of labels") no new label appears and a pixel
 *     is labelled only through a labelled left / upper neighbour (:345-347 read labels, not pixels):
 *     from the (nblobs+1)-th seed position on, mask(x,y) = fg(x,y) && (mask(x-1,y) || mask(x,y-1));
 *   - components, areas, boxes and coordinate sums are those of the 4-connected components of `mask`.
 * Components are found here by flood fill from each seed in raster order (the GPU uses a pixel
 * union-find); blobs[0..m) in label order, centroid = sums / area in unsigned arithmetic (:397-398).
 * ---------------------------------------------------------------------------------------- */
GSO_API unsigned gso_blobs(const uint8_t *img, unsigned w, unsigned h, gs_label *labels, struct gs_blob *blobs,
                           unsigned nblobs) {
  size_t npx = (size_t)w * h;
  uint8_t *mask = (uint8_t *)malloc(npx);
  uint32_t *stack = (uint32_t *)malloc(npx * sizeof(uint32_t));
  unsigned nseeds = 0, m = 0;
  int overflow = 0;
  for (size_t i = 0; i < npx; i++) labels[i] = 0;
  for (unsigned y = 0; y < h; y++)
    for (unsigned x = 0; x < w; x++) {
      size_t i = (size_t)y * w + x;
      int fg = img[i] >= 128;
      int left = x > 0 && mask[i - 1], top = y > 0 && mask[i - w];
      if (!overflow) {
        mask[i] = (uint8_t)fg;
        if (fg && !left && !top) {
          if (nseeds == nblobs) overflow = 1, mask[i] = 0;   /* the first seed that finds no label left */
          else nseeds++;
        }
      } else {
        mask[i] = (uint8_t)(fg && (left || top));
      }
    }
  /* flood fill in raster order: the first unlabelled mask pixel met is its component's raster-first pixel = a seed */
  unsigned seed_no = 0;
  for (unsigned y = 0; y < h; y++)
    for (unsigned x = 0; x < w; x++) {
      size_t i = (size_t)y * w + x;
      if (!mask[i]) continue;
      int left = x > 0 && mask[i - 1], top = y > 0 && mask[i - w];
      if (!left && !top) seed_no++;                 /* every seed consumes a number, component start or not */
      if (labels[i]) continue;
      /* a pixel reached here unlabelled is the raster-first pixel of a new component, hence a seed */
      unsigned area = 0, minx = x, maxx = x, miny = y, maxy = y, sx = 0, sy = 0, top_of_stack = 0;
      stack[top_of_stack++] = (uint32_t)i;
      labels[i] = (gs_label)seed_no;
      while (top_of_stack) {
        uint32_t p = stack[--top_of_stack];
        unsigned px = p % w, py = p / w;
        area++, sx += px, sy += py;
        if (px < minx) minx = px;
        if (px > maxx) maxx = px;
        if (py < miny) miny = py;
        if (py > maxy) maxy = py;
        if (px > 0 && mask[p - 1] && !labels[p - 1]) labels[p - 1] = (gs_label)seed_no, stack[top_of_stack++] = p - 1;
        if (px + 1 < w && mask[p + 1] && !labels[p + 1]) labels[p + 1] = (gs_label)seed_no, stack[top_of_stack++] = p + 1;
        if (py > 0 && mask[p - w] && !labels[p - w]) labels[p - w] = (gs_label)seed_no, stack[top_of_stack++] = p - w;
        if (py + 1 < h && mask[p + w] && !labels[p + w]) labels[p + w] = (gs_label)seed_no, stack[top_of_stack++] = p + w;
      }
      memset(&blobs[m], 0, sizeof(blobs[m]));
      blobs[m].label = (gs_label)seed_no, blobs[m].area = area;
      blobs[m].box.x = minx, blobs[m].box.y = miny, blobs[m].box.w = maxx - minx + 1, blobs[m].box.h = maxy - miny + 1;
      blobs[m].centroid.x = sx / area, blobs[m].centroid.y = sy / area;
      m++;
    }
  free(mask);
  free(stack);
  return m;
}

/* gs_blob_corners, grayskull.h:407-421: over the blob's box, pixels >= 128 carrying its label; the four extremes of
 * x+y (min -> tl, max -> br) and x-y (min -> bl, max -> tr), the FIRST pixel in raster order on ties (strict
 * comparisons); all four default to the centroid.  Restated as key minima: (value, raster index), in 64 bits from the
 * reference's starting values (INT_MAX for the minima, INT_MIN for the maxima): a pixel whose x + y (x - y) is INT_MAX
 * leaves tl (bl) at the centroid. */
GSO_API void gso_blob_corners(const uint8_t *img, unsigned w, unsigned h, const gs_label *labels, const struct gs_blob *b,
                              struct gs_point c[4]) {
  long long best[4] = {-1, -1, -1, -1};
  long long val[4] = {INT_MAX, -(long long)INT_MIN, -(long long)INT_MIN, INT_MAX};
  (void)h;
  for (unsigned y = b->box.y; y < b->box.y + b->box.h; y++)
    for (unsigned x = b->box.x; x < b->box.x + b->box.w; x++) {
      if (x >= w || y >= h || img[(size_t)y * w + x] < 128 || labels[(size_t)y * w + x] != b->label) continue;
      int sum = (int)x + (int)y, diff = (int)x - (int)y;
      long long idx = (long long)y * w + x;
      /* tl: min sum, tr: max diff, br: max sum, bl: min diff */
      long long cand[4] = {sum, -(long long)diff, -(long long)sum, diff};
      for (int k = 0; k < 4; k++)
        if (cand[k] < val[k]) best[k] = idx, val[k] = cand[k];
    }
  for (int k = 0; k < 4; k++) {
    if (best[k] < 0) c[k] = b->centroid;
    else c[k].x = (unsigned)(best[k] % w), c[k].y = (unsigned)(best[k] / w);
  }
}

/* gs_perspective_correct, grayskull.h:423-444.  fp32, the reference's evaluation order, no contraction: bilinear
 * interpolation of the quad edges (c[0]=tl, c[1]=tr, c[2]=br, c[3]=bl) gives the source point, clamped to the image,
 * then gs_resize-style bilinear sampling; dst.w == 1 / dst.h == 1 divide 0 by 0 like the reference (NaN clamps to the
 * last column / row through the ternaries of GS_MIN / GS_MAX). */
GSO_API void gso_perspective_correct(uint8_t *dst, unsigned dw, unsigned dh, const uint8_t *src, unsigned sw, unsigned sh,
                                     const struct gs_point c[4]) {
  volatile float w = (float)dw - 1.0f, h = (float)dh - 1.0f;
  float c0x = (float)c[0].x, c0y = (float)c[0].y, c1x = (float)c[1].x, c1y = (float)c[1].y;
  float c2x = (float)c[2].x, c2y = (float)c[2].y, c3x = (float)c[3].x, c3y = (float)c[3].y;
  float mx = (float)sw - 1.0f, my = (float)sh - 1.0f;
  for (unsigned y = 0; y < dh; y++)
    for (unsigned x = 0; x < dw; x++) {
      volatile float u = (float)x / w, v = (float)y / h;
      volatile float omu = 1 - u, omv = 1 - v;
      volatile float a, b2, top_x, top_y, bot_x, bot_y, src_x, src_y;
      a = c0x * omu, b2 = c1x * u, top_x = a + b2;
      a = c0y * omu, b2 = c1y * u, top_y = a + b2;
      a = c3x * omu, b2 = c2x * u, bot_x = a + b2;
      a = c3y * omu, b2 = c2y * u, bot_y = a + b2;
      a = top_x * omv, b2 = bot_x * v, src_x = a + b2;
      a = top_y * omv, b2 = bot_y * v, src_y = a + b2;
      float fx = src_x < mx ? src_x : mx, fy = src_y < my ? src_y : my;   /* GS_MIN(src_x, w-1): NaN -> w-1 */
      fx = 0.0f > fx ? 0.0f : fx;                                           /* GS_MAX(0, .) */
      fy = 0.0f > fy ? 0.0f : fy;
      unsigned x0 = (unsigned)fx, y0 = (unsigned)fy;
      unsigned x1 = x0 + 1 < sw - 1 ? x0 + 1 : sw - 1, y1 = y0 + 1 < sh - 1 ? y0 + 1 : sh - 1;
      volatile float dx = fx - (float)x0, dy = fy - (float)y0;
      /* gs_get's 0 outside the image: above 2^24, (float)sw - 1.0f can round past sw - 1, putting x0 at sw or
       * beyond (y0 likewise); x1 and y1 are clamped to the last pixel */
      int in_x = x0 < sw, in_y = y0 < sh;
      float c00 = in_x && in_y ? src[(size_t)y0 * sw + x0] : 0, c01 = in_y ? src[(size_t)y0 * sw + x1] : 0;
      float c10 = in_x ? src[(size_t)y1 * sw + x0] : 0, c11 = src[(size_t)y1 * sw + x1];
      volatile float omx = 1 - dx, omy = 1 - dy;
      volatile float t0 = c00 * omx, t1 = c01 * dx, t2 = c10 * omx, t3 = c11 * dx;
      t0 = t0 * omy;
      t1 = t1 * omy;
      t2 = t2 * dy;
      t3 = t3 * dy;
      volatile float acc = t0 + t1;
      acc = acc + t2;
      acc = acc + t3;
      dst[(size_t)y * dw + x] = (uint8_t)acc;
    }
}
