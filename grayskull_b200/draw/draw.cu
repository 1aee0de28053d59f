// draw.cu -- libgrayskull_draw.so: the reference CLI's annotated pictures drawn onto frame batches
// (include/grayskull_draw.h), bit-exact with the blobs, keypoints, faces and orb verbs of nanomagick.c.
//
//   k_draw_copy          dst = src for the keypoint and rect calls (skipped in place): 16-byte words when dst and src
//                        share their alignment, bytes otherwise
//   k_draw_blobs         one CTA per (frame, band of BH rows, TW columns).  Each box that meets the tile does one
//                        shared-memory atomicMax per row of its clipped right end (+1) at its left column; the wrap
//                        (x2 == w covers column 0 one row down) is one more such span.  A prefix max along each row
//                        then gives coverage: cost (tiles x boxes) + pixels, whatever the boxes' areas.
//   k_draw_keypoints     one CTA per frame: a radix select (4 passes of 8 bits) finds the response T of the top-th
//                        keypoint and how many of those tied at T are taken; an ordered scan takes the first of the
//                        ties, which is what a stable sort keeps.  Every cross is 255, so the draw order is free.
//   k_draw_rects         one warp per rect: each edge's span clipped to the frame analytically
//   k_draw_canvas        the orb picture's template | frame canvas, one CTA per output row
//   k_draw_match_lines   one CTA per frame: the matches' (distance, slot) in shared memory, the verb's exchange sort
//                        run by one thread for its first `top` outer passes only, then one thread per line
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <utility>

#include "../../include/grayskull_draw.h"

// the reference's gs_assert (grayskull.h:94-98): message + abort
#define GSD_ASSERT(cond)                                \
  do {                                                  \
    if (!(cond)) {                                      \
      fprintf(stderr, "Assertion failed: %s\n", #cond); \
      abort();                                          \
    }                                                   \
  } while (0)

namespace gsb {

static thread_local char t_last_error[512] = "no error";

static int record_error(cudaError_t e, const char *file, int line) {
  snprintf(t_last_error, sizeof(t_last_error), "%s (%s) at %s:%d", cudaGetErrorName(e), cudaGetErrorString(e), file,
           line);
  return static_cast<int>(e);
}

static int invalid(const char *what, const char *file, int line) {
  snprintf(t_last_error, sizeof(t_last_error), "cudaErrorInvalidValue (%s) at %s:%d", what, file, line);
  return static_cast<int>(cudaErrorInvalidValue);
}

// Every kernel launch of this library: opt in to more than 48 KiB of dynamic shared memory when asked, launch, check.
template <class... P, class... A>
static int launch(const char *file, int line, void (*k)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t s,
                  A &&...a) {
  if (smem > 48u * 1024u) {
    cudaError_t e = cudaFuncSetAttribute(reinterpret_cast<const void *>(k), cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(smem));
    if (e != cudaSuccess) return record_error(e, file, line);
  }
  k<<<grid, block, smem, s>>>(std::forward<A>(a)...);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : record_error(e, file, line);
}
#define GSD_LAUNCH(...)                                         \
  do {                                                          \
    int gsd_rc_ = gsb::launch(__FILE__, __LINE__, __VA_ARGS__); \
    if (gsd_rc_) return gsd_rc_;                                \
  } while (0)

constexpr unsigned GRID_MAX = 65535u;   // grid y / z limit, and the frame-loop grid of the per-frame kernels
constexpr unsigned TW = 1024, BH = 8;   // k_draw_blobs tile: 256 threads x 4 columns, 8 rows
constexpr unsigned MATCH_MAX_STRIDE = 16384;

__device__ __forceinline__ unsigned umin(unsigned a, unsigned b) { return a < b ? a : b; }

// ---- dst = src ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_draw_copy(uint8_t *__restrict__ dst, const uint8_t *__restrict__ src,
                                                   unsigned long long bytes) {
  const unsigned long long t = blockIdx.x * 256ull + threadIdx.x, step = gridDim.x * 256ull;
  if (((reinterpret_cast<uintptr_t>(dst) ^ reinterpret_cast<uintptr_t>(src)) & 15u) == 0) {
    // bytes up to dst's first 16-byte boundary, 16-byte words, then the last < 16 bytes
    const unsigned long long lead = (16u - (reinterpret_cast<uintptr_t>(dst) & 15u)) & 15u;
    const unsigned long long head = lead < bytes ? lead : bytes, words = (bytes - head) / 16, tail = head + words * 16;
    if (t < head) dst[t] = src[t];
    uint4 *d4 = reinterpret_cast<uint4 *>(dst + head);
    const uint4 *s4 = reinterpret_cast<const uint4 *>(src + head);
    for (unsigned long long i = t; i < words; i += step) d4[i] = s4[i];
    if (t < bytes - tail) dst[tail + t] = src[tail + t];
  } else {
    for (unsigned long long i = t; i < bytes; i += step) dst[i] = src[i];
  }
}

static int copy_frames(uint8_t *dst, const uint8_t *src, unsigned long long bytes, cudaStream_t s) {
  if (dst == src || bytes == 0) return 0;
  const unsigned long long words = bytes / 16 + 1;
  const unsigned blocks = static_cast<unsigned>(words / 256 + 1 < 132ull * 16 ? words / 256 + 1 : 132ull * 16);
  GSD_LAUNCH(k_draw_copy, dim3(blocks), dim3(256), 0, s, dst, src, bytes);
  return 0;
}

// ---- blobs ------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_draw_blobs(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n, const struct gs_blob *__restrict__ blobs,
             const unsigned *__restrict__ counts, unsigned stride) {
  __shared__ __align__(16) unsigned ends[BH][TW];   // per row: the largest (clipped right end + 1 - c0) starting here
  __shared__ unsigned wtot[8];
  const unsigned tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned bands = (h + BH - 1) / BH, c0 = blockIdx.x * TW;
  for (unsigned f = blockIdx.z; f < n; f += gridDim.z) {
    const unsigned cnt = umin(counts[f], stride);
    const struct gs_blob *fb = blobs + (size_t)f * stride;
    const size_t fbase = (size_t)f * w * h;
    for (unsigned band = blockIdx.y; band < bands; band += gridDim.y) {
      const unsigned r0 = band * BH, rl = umin(h - 1, r0 + BH - 1);   // rows r0..rl of the frame
      for (unsigned r = 0; r < BH; r++) reinterpret_cast<uint4 *>(ends[r])[tid] = make_uint4(0, 0, 0, 0);
      __syncthreads();
      const unsigned cl = umin(w - 1, c0 + TW - 1);                     // columns c0..cl
      for (unsigned b = tid; b < cnt; b += 256) {
        const struct gs_rect box = fb[b].box;
        // nanomagick.c:162-164, in its unsigned arithmetic ((int)box.x - 2 wrapping as gcc's does)
        const int ix1 = (int)(box.x - 2u), iy1 = (int)(box.y - 2u);
        const unsigned x1 = ix1 > 0 ? (unsigned)ix1 : 0u, y1 = iy1 > 0 ? (unsigned)iy1 : 0u;
        const unsigned x2 = umin(w, box.x + box.w + 2), y2 = umin(h, box.y + box.h + 2);
        if (x1 > x2 || y1 > y2) continue;
        // rows y1..y2 inside the frame, columns x1..min(x2, w - 1)
        const unsigned xe = umin(x2, w - 1), ye = umin(y2, h - 1);
        if (x1 <= xe) {
          const unsigned lo = x1 > c0 ? x1 : c0, hi = umin(xe, cl);
          const unsigned ya = y1 > r0 ? y1 : r0, yb = umin(ye, rl);
          if (lo <= hi)
            for (unsigned y = ya; y <= yb; y++) atomicMax(&ends[y - r0][lo - c0], hi - c0 + 1);
        }
        // x2 == w: index y*w + w is pixel (0, y + 1), so column 0 of rows y1 + 1 .. y2 + 1 inside the frame
        if (x2 == w && c0 == 0) {
          const unsigned long long ya = y1 + 1ull > r0 ? y1 + 1ull : r0, yb = y2 + 1ull < rl ? y2 + 1ull : rl;
          for (unsigned long long y = ya; y <= yb; y++) atomicMax(&ends[y - r0][0], 1u);
        }
      }
      __syncthreads();
      for (unsigned r = 0; r < BH && r0 + r < h; r++) {
        const uint4 v = reinterpret_cast<const uint4 *>(ends[r])[tid];
        const unsigned p0 = v.x, p1 = max(p0, v.y), p2 = max(p1, v.z), p3 = max(p2, v.w);
        unsigned inc = p3;   // inclusive max over this warp's threads up to tid
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const unsigned u = __shfl_up_sync(0xffffffffu, inc, o);
          if (lane >= (unsigned)o) inc = max(inc, u);
        }
        if (lane == 31) wtot[warp] = inc;
        __syncthreads();
        unsigned carry = __shfl_up_sync(0xffffffffu, inc, 1);
        if (lane == 0) carry = 0;
        for (unsigned k = 0; k < warp; k++) carry = max(carry, wtot[k]);
        const unsigned xr = tid * 4, x = c0 + xr;   // columns x..x+3, relative xr..xr+3
        const unsigned pm[4] = {max(carry, p0), max(carry, p1), max(carry, p2), max(carry, p3)};
        const size_t row = fbase + (size_t)(r0 + r) * w;
        if (x + 3 < w && ((reinterpret_cast<uintptr_t>(src + row + x) | reinterpret_cast<uintptr_t>(dst + row + x)) & 3u) == 0) {
          const uint32_t sv = *reinterpret_cast<const uint32_t *>(src + row + x);
          uint32_t out = 0;
#pragma unroll
          for (unsigned i = 0; i < 4; i++) {
            const unsigned sb = (sv >> (8 * i)) & 255u;
            out |= (sb > 128 ? 255u : pm[i] > xr + i ? 128u : 0u) << (8 * i);
          }
          *reinterpret_cast<uint32_t *>(dst + row + x) = out;
        } else {
#pragma unroll
          for (unsigned i = 0; i < 4; i++)
            if (x + i < w) {
              const unsigned sb = src[row + x + i];
              dst[row + x + i] = static_cast<uint8_t>(sb > 128 ? 255u : pm[i] > xr + i ? 128u : 0u);
            }
        }
        __syncthreads();   // wtot is rewritten by the next row
      }
      __syncthreads();     // ends is cleared for the next band
    }
  }
}

// ---- keypoints ----------------------------------------------------------------------------------------------------
__device__ __forceinline__ void set_px(uint8_t *frame, unsigned w, unsigned h, unsigned x, unsigned y) {
  if (x < w && y < h) frame[(size_t)y * w + x] = 255;   // gs_set
}

__global__ void __launch_bounds__(256)
k_draw_keypoints(uint8_t *dst, unsigned w, unsigned h, unsigned n, const struct gs_keypoint *__restrict__ kps,
                 const unsigned *__restrict__ counts, unsigned stride, unsigned top) {
  __shared__ unsigned hist[256];
  __shared__ unsigned s_digit, s_need, s_wcount[8], s_base;
  const unsigned tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (unsigned f = blockIdx.x; f < n; f += gridDim.x) {
    const unsigned c = umin(counts[f], stride), k = umin(top, c);
    if (k == 0) continue;
    const struct gs_keypoint *fk = kps + (size_t)f * stride;
    uint8_t *frame = dst + (size_t)f * w * h;
    // T: the k-th largest response; need: how many of the keypoints at T are taken
    unsigned T = 0, need = c, mask = 0;
    if (k < c) {
      need = k;
      for (int shift = 24; shift >= 0; shift -= 8) {
        hist[tid] = 0;
        __syncthreads();
        for (unsigned i = tid; i < c; i += 256) {
          const unsigned r = fk[i].response;
          if ((r & mask) == T) atomicAdd(&hist[(r >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (tid == 0) {
          unsigned above = 0, d = 255;
          for (;; d--) {
            if (above + hist[d] >= need || d == 0) break;
            above += hist[d];
          }
          s_digit = d, s_need = need - above;
        }
        __syncthreads();
        T |= s_digit << shift, mask |= 255u << shift, need = s_need;
        __syncthreads();
      }
    }
    // take every keypoint above T and the first `need` at T in list order
    unsigned base = 0;   // ties at T before this chunk
    for (unsigned i0 = 0; i0 < c; i0 += 256) {
      const unsigned i = i0 + tid;
      const bool in = i < c;
      const unsigned r = in ? fk[i].response : 0u;
      const bool tie = in && r == T;
      const unsigned bal = __ballot_sync(0xffffffffu, tie);
      if (lane == 0) s_wcount[warp] = __popc(bal);
      __syncthreads();
      unsigned before = base + __popc(bal & ((1u << lane) - 1u));
      for (unsigned q = 0; q < warp; q++) before += s_wcount[q];
      if (in && (r > T || (tie && before < need))) {
        const unsigned x = fk[i].pt.x, y = fk[i].pt.y;
        for (int d = -2; d <= 2; d++) set_px(frame, w, h, x, y + d);   // nanomagick.c:237-238
        for (int d = -2; d <= 2; d++) set_px(frame, w, h, x + d, y);
      }
      if (tid == 0) {
        unsigned t = 0;
        for (unsigned q = 0; q < 8; q++) t += s_wcount[q];
        s_base = base + t;
      }
      __syncthreads();
      base = s_base;
      __syncthreads();
    }
  }
}

// ---- rects ----------------------------------------------------------------------------------------------------------
// every pixel between a and b (ints, both included) along a row (horizontal) or column at `fixed`, inside the frame
__device__ __forceinline__ void span(uint8_t *frame, unsigned w, unsigned h, bool horizontal, int fixed, int a, int b,
                                     unsigned lane) {
  const long long lim = horizontal ? w : h, other = horizontal ? h : w;
  if (fixed < 0 || fixed >= other) return;
  const long long lo = max(min(a, b), 0), hi = min((long long)max(a, b), lim - 1);
  for (long long p = lo + lane; p <= hi; p += 32) {
    const size_t i = horizontal ? (size_t)fixed * w + (size_t)p : (size_t)p * w + (size_t)fixed;
    frame[i] = 255;
  }
}

__global__ void __launch_bounds__(256)
k_draw_rects(uint8_t *dst, unsigned w, unsigned h, unsigned n, const struct gs_rect *__restrict__ rects,
             const unsigned *__restrict__ counts, unsigned stride) {
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (unsigned f = blockIdx.y; f < n; f += gridDim.y) {
    const unsigned c = umin(counts[f], stride);
    uint8_t *frame = dst + (size_t)f * w * h;
    for (unsigned i = blockIdx.x * 8 + warp; i < c; i += gridDim.x * 8) {
      const struct gs_rect r = rects[(size_t)f * stride + i];
      const int x = (int)r.x, y = (int)r.y, xw = (int)(r.x + r.w), yh = (int)(r.y + r.h);   // nanomagick.c:371-374
      span(frame, w, h, true, y, x, xw, lane);
      span(frame, w, h, true, yh, x, xw, lane);
      span(frame, w, h, false, x, y, yh, lane);
      span(frame, w, h, false, xw, y, yh, lane);
    }
  }
}

// ---- matches --------------------------------------------------------------------------------------------------------
// output row `row` of the n canvases of cw x ch: template | frame, zero elsewhere (nanomagick.c:322-332)
__global__ void __launch_bounds__(256)
k_draw_canvas(uint8_t *__restrict__ dst, const uint8_t *__restrict__ src, unsigned w, unsigned h,
              const uint8_t *__restrict__ tmpl, unsigned tw, unsigned th, unsigned long long rows, unsigned ch) {
  const unsigned cw = tw + w;
  for (unsigned long long row = blockIdx.x; row < rows; row += gridDim.x) {
    const unsigned long long f = row / ch;
    const unsigned y = static_cast<unsigned>(row - f * ch);
    uint8_t *out = dst + row * cw;
    const uint8_t *srow = src + (f * h + y) * w;
    for (unsigned x = threadIdx.x; x < cw; x += 256) {
      uint8_t v = 0;
      if (x < tw) {
        if (y < th) v = tmpl[(size_t)y * tw + x];
      } else if (y < h) {
        v = srow[x - tw];
      }
      out[x] = v;
    }
  }
}

// draw_line of nanomagick.c:172-184
__device__ void draw_line(uint8_t *img, unsigned iw, unsigned ih, unsigned x1, unsigned y1, unsigned x2, unsigned y2) {
  const int dx = abs((int)x2 - (int)x1), dy = abs((int)y2 - (int)y1);
  const int sx = x1 < x2 ? 1 : -1, sy = y1 < y2 ? 1 : -1;
  int err = dx - dy, x = x1, y = y1;
  while (1) {
    if (x >= 0 && x < (int)iw && y >= 0 && y < (int)ih) img[(size_t)y * iw + x] = 255;
    if (x == (int)x2 && y == (int)y2) break;
    const int e2 = 2 * err;
    if (e2 > -dy) err -= dy, x += sx;
    if (e2 < dx) err += dx, y += sy;
  }
}

__global__ void __launch_bounds__(128)
k_draw_match_lines(uint8_t *dst, unsigned w, unsigned h, unsigned n, unsigned tw, unsigned th,
                   const struct gs_keypoint *__restrict__ kps1, unsigned stride1,
                   const struct gs_keypoint *__restrict__ kps2, unsigned stride2,
                   const struct gs_match *__restrict__ matches, const unsigned *__restrict__ mcounts, unsigned mstride,
                   unsigned top) {
  extern __shared__ uint2 m[];   // (distance, slot) of the frame's matches, in the verb's order
  const unsigned cw = tw + w, ch = th > h ? th : h;
  for (unsigned f = blockIdx.x; f < n; f += gridDim.x) {
    const unsigned c = umin(mcounts[f], mstride), k = umin(top, c);
    if (k == 0) continue;
    const struct gs_match *fm = matches + (size_t)f * mstride;
    for (unsigned i = threadIdx.x; i < c; i += blockDim.x) m[i] = make_uint2(fm[i].distance, i);
    __syncthreads();
    if (threadIdx.x == 0)   // nanomagick.c:315-321, its first k outer passes: positions 0..k-1 are final after them
      for (unsigned i = 0; i < k; i++) {
        uint2 mi = m[i];
        for (unsigned j = i + 1; j < c; j++) {
          const uint2 mj = m[j];
          if (mj.x < mi.x) m[j] = mi, mi = mj;
        }
        m[i] = mi;
      }
    __syncthreads();
    uint8_t *canvas = dst + (size_t)f * cw * ch;
    const struct gs_keypoint *k1 = kps1 + (size_t)f * stride1, *k2 = kps2 + (size_t)f * stride2;
    for (unsigned i = threadIdx.x; i < k; i += blockDim.x) {
      const struct gs_match mt = fm[m[i].y];
      if ((stride1 && mt.idx1 >= stride1) || (stride2 && mt.idx2 >= stride2)) continue;
      const unsigned x1 = k1[mt.idx1].pt.x, y1 = k1[mt.idx1].pt.y, x2 = k2[mt.idx2].pt.x, y2 = k2[mt.idx2].pt.y;
      if (x1 >= tw || y1 >= th || x2 >= w || y2 >= h) continue;   // outside its own image
      draw_line(canvas, cw, ch, x1, y1, x2 + tw, y2);
    }
    __syncthreads();   // m is reloaded for the next frame
  }
}

// ---- entry points ---------------------------------------------------------------------------------------------------
static bool overlap(const void *a, unsigned long long an, const void *b, unsigned long long bn) {
  const uintptr_t pa = reinterpret_cast<uintptr_t>(a), pb = reinterpret_cast<uintptr_t>(b);
  return an && bn && pa < pb + bn && pb < pa + an;
}

static void same_size_args(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, const void *list,
                           const unsigned *counts) {
  GSD_ASSERT(dst && src && list && counts);
  GSD_ASSERT(w > 0 && h > 0);
}

}  // namespace gsb

using namespace gsb;

extern "C" const char *gs_b200_draw_last_error(void) { return t_last_error; }

extern "C" int gs_b200_draw_blobs_batch(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n,
                                        const struct gs_blob *blobs, const unsigned *counts, unsigned stride,
                                        gs_b200_stream s) {
  if (n == 0) return 0;
  same_size_args(dst, src, w, h, blobs, counts);
  const unsigned long long bytes = (unsigned long long)w * h * n;
  if (dst != src && overlap(dst, bytes, src, bytes)) return invalid("dst overlaps src", __FILE__, __LINE__);
  const unsigned bands = (h + BH - 1) / BH;
  const dim3 grid((w + TW - 1) / TW, bands < GRID_MAX ? bands : GRID_MAX, n < GRID_MAX ? n : GRID_MAX);
  GSD_LAUNCH(k_draw_blobs, grid, dim3(256), 0, (cudaStream_t)s, dst, src, w, h, n, blobs, counts, stride);
  return 0;
}

extern "C" int gs_b200_draw_keypoints_batch(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n,
                                            const struct gs_keypoint *kps, const unsigned *counts, unsigned stride,
                                            unsigned top, gs_b200_stream s) {
  if (n == 0) return 0;
  same_size_args(dst, src, w, h, kps, counts);
  const unsigned long long bytes = (unsigned long long)w * h * n;
  if (dst != src && overlap(dst, bytes, src, bytes)) return invalid("dst overlaps src", __FILE__, __LINE__);
  if (int rc = copy_frames(dst, src, bytes, (cudaStream_t)s)) return rc;
  if (top == 0 || stride == 0) return 0;
  GSD_LAUNCH(k_draw_keypoints, dim3(n < GRID_MAX ? n : GRID_MAX), dim3(256), 0, (cudaStream_t)s, dst, w, h, n, kps,
             counts, stride, top);
  return 0;
}

extern "C" int gs_b200_draw_rects_batch(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n,
                                        const struct gs_rect *rects, const unsigned *counts, unsigned stride,
                                        gs_b200_stream s) {
  if (n == 0) return 0;
  same_size_args(dst, src, w, h, rects, counts);
  const unsigned long long bytes = (unsigned long long)w * h * n;
  if (dst != src && overlap(dst, bytes, src, bytes)) return invalid("dst overlaps src", __FILE__, __LINE__);
  if (int rc = copy_frames(dst, src, bytes, (cudaStream_t)s)) return rc;
  if (stride == 0) return 0;
  const unsigned rx = (stride + 7) / 8;
  GSD_LAUNCH(k_draw_rects, dim3(rx < 64 ? rx : 64, n < GRID_MAX ? n : GRID_MAX), dim3(256), 0, (cudaStream_t)s, dst, w,
             h, n, rects, counts, stride);
  return 0;
}

extern "C" int gs_b200_draw_matches_batch(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n,
                                          const uint8_t *tmpl, unsigned tw, unsigned th,
                                          const struct gs_keypoint *kps1, unsigned stride1,
                                          const struct gs_keypoint *kps2, unsigned stride2,
                                          const struct gs_match *matches, const unsigned *mcounts, unsigned mstride,
                                          unsigned top, gs_b200_stream s) {
  if (n == 0) return 0;
  GSD_ASSERT(dst && src && tmpl && kps1 && kps2 && matches && mcounts);
  GSD_ASSERT(w > 0 && h > 0 && tw > 0 && th > 0);
  if (mstride > MATCH_MAX_STRIDE) return invalid("mstride > 16384", __FILE__, __LINE__);
  const unsigned long long cw = (unsigned long long)tw + w, ch = th > h ? th : h;
  if (cw > 0xffffffffull) return invalid("tw + w does not fit in 32 bits", __FILE__, __LINE__);
  const unsigned long long out = cw * ch * n;
  if (overlap(dst, out, src, (unsigned long long)w * h * n) || overlap(dst, out, tmpl, (unsigned long long)tw * th))
    return invalid("dst overlaps src or tmpl", __FILE__, __LINE__);
  const unsigned long long rows = ch * n;
  GSD_LAUNCH(k_draw_canvas, dim3(static_cast<unsigned>(rows < 132ull * 64 ? rows : 132ull * 64)), dim3(256), 0,
             (cudaStream_t)s, dst, src, w, h, tmpl, tw, th, rows, static_cast<unsigned>(ch));
  if (top == 0 || mstride == 0) return 0;
  GSD_LAUNCH(k_draw_match_lines, dim3(n < GRID_MAX ? n : GRID_MAX), dim3(128), (size_t)mstride * sizeof(uint2),
             (cudaStream_t)s, dst, w, h, n, tw, th, kps1, stride1, kps2, stride2, matches, mcounts, mstride, top);
  return 0;
}
