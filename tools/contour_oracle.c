/*
 * contour_oracle.c -- TEST AND MEASUREMENT INFRASTRUCTURE, not product code.
 *
 * A plain-C99 CPU restatement of gs_trace_contour (reference grayskull.h:446-480) with a defined end for walks the
 * reference never leaves, and the list-order semantics of a batch as consecutive calls on one visited map.  It is the
 * sequential model gs_b200_trace_contours_batch is checked against: the device walks every contour at once and applies
 * the list order afterwards, this walks them one after the other and marks visited as it goes.
 * tests/test_contour.py pins it against the reference's own test case, the compiled reference and a literal
 * step-capped walk; it and tools/bench_contour.py compile it on demand (tools/contour_oracle.py) into a temporary
 * directory.  The product path never loads it.
 */
#include <stddef.h>
#include <stdint.h>

#include "grayskull.h" /* ../include: stand-alone mode, types only */

#define GSO_API __attribute__((visibility("default")))

/* gs_trace_contour (grayskull.h:446-480) with a defined end for walks the reference never leaves.  Returns 0 when the
 * walk reaches start a second time, 1 when p has no foreground neighbour (both: the reference's outputs, byte for
 * byte), 2 when the state (p, dir, seenstart) repeats: the reference then runs for ever, and *c / visited are what its
 * copies hold from some step on.  Brent's test (one saved state, reset at steps 2^j - 1) finds the repeat; one more
 * lap after it applies the box update of every step of the cycle with the final box.x / box.y, since
 * w = max(w, p.x - box.x + 1) is taken with the box.x of its step.  The list-order semantics of a batch are consecutive
 * calls on one visited, as gso_trace_contours makes them. */
static unsigned trace_contour(const uint8_t *img, uint8_t *visited, unsigned w, unsigned h, struct gs_contour *c,
                              unsigned long long *steps) {
  static const int dx[] = {1, 1, 0, -1, -1, -1, 0, 1};
  static const int dy[] = {0, 1, 1, 1, 0, -1, -1, -1};
  struct gs_point p = c->start, saved = c->start;
  unsigned dir = 7, seenstart = 0, saved_ds = 7;
  unsigned long long power = 1, lam = 0, lap = 0;
  c->length = 0;
  c->box.x = c->start.x, c->box.y = c->start.y, c->box.w = 1, c->box.h = 1;
  for (;;) {
    int ndir = (dir + 1) % 8, found = 0, i;
    int in = p.x < w && p.y < h;
    if (!(in && visited[(size_t)p.y * w + p.x])) c->length++;
    if (in) visited[(size_t)p.y * w + p.x] = 255;
    for (i = 0; i < 8; i++) {
      int d = (ndir + i) % 8, nx = p.x + dx[d], ny = p.y + dy[d];
      if (nx >= 0 && nx < (int)w && ny >= 0 && ny < (int)h && img[(size_t)ny * w + nx] > 128) {
        p.x = (unsigned)nx, p.y = (unsigned)ny;
        dir = (d + 6) % 8;
        found = 1;
        break;
      }
    }
    if (!found) return 1;
    ++*steps;
    c->box.x = GS_MIN(c->box.x, p.x);
    c->box.y = GS_MIN(c->box.y, p.y);
    c->box.w = GS_MAX(c->box.w, p.x - c->box.x + 1);
    c->box.h = GS_MAX(c->box.h, p.y - c->box.y + 1);
    if (p.x == c->start.x && p.y == c->start.y) {
      if (seenstart) return 0;
      seenstart = 1;
    }
    if (lap) {
      if (--lap == 0) return 2;
      continue;
    }
    lam++;
    if (p.x == saved.x && p.y == saved.y && (dir | seenstart << 3) == saved_ds) {
      lap = lam;
      continue;
    }
    if (lam == power) saved = p, saved_ds = dir | seenstart << 3, power *= 2, lam = 0;
  }
}

GSO_API unsigned gso_trace_contour(const uint8_t *img, uint8_t *visited, unsigned w, unsigned h,
                                  struct gs_contour *c) {
  unsigned long long steps = 0;
  return trace_contour(img, visited, w, h, c, &steps);
}

/* count consecutive gso_trace_contour calls on one visited, the end kinds into ends (when not NULL); returns the
 * steps the walks took (moves to a neighbour, the closing lap of a cycle included) */
GSO_API unsigned long long gso_trace_contours(const uint8_t *img, uint8_t *visited, unsigned w, unsigned h,
                                              struct gs_contour *c, unsigned count, uint8_t *ends) {
  unsigned long long steps = 0;
  unsigned k;
  for (k = 0; k < count; k++) {
    unsigned e = trace_contour(img, visited, w, h, &c[k], &steps);
    if (ends) ends[k] = (uint8_t)e;
  }
  return steps;
}
