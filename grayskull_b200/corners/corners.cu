// corners.cu -- libgrayskull_corners.so: the largest-blob pick and gs_blob_corners over frame batches
// (include/grayskull_corners.h), bit-exact with the reference's document scanner (nanomagick.c:186-210) and the wasm
// demo's largest-blob rule (grayskull.c:285-295).
//
// The pick is one warp per frame: an argmax over (area, lowest index).
//
// gs_blob_corners keeps, for each of tl / tr / br / bl, the first pixel in raster order with the extreme x + y or
// x - y.  Within one row every extreme is at the row's first or last qualifying pixel (the first has the least sum and
// the least difference, the last the greatest of both), so a row contributes at most two candidates, and across rows
// the winner is the lexicographic minimum of the key (value, raster index) -- k_blob_corners' rule.  A warp scans a
// row of up to 256 columns: each lane reads 8 columns, a row without a pixel >= 128 skips its labels, and two warp
// reductions give the row's first and last qualifying column.  Records are split by the size of their box clipped to
// the frame:
//   k_corners_small   one warp per record: a box of at most SMALL_H rows and SMALL_W columns is scanned by one warp,
//                     and its 4 points are written; a larger record's 4 slots are set to the empty key instead
//   k_corners_tiles   one CTA per (frame, TILE_W x TILE_H tile): the frame's records are staged in chunks, and each
//                     large record whose box meets the tile is scanned there, one row per warp; each warp's 4 keys go
//                     to the record's slots with a 64-bit atomicMin (skipped when the slot already holds a smaller key)
//   k_corners_final   one thread per large record: keys to points, the centroid where no pixel counted
// So a frame-sized record spreads over every tile of its frame, and many small records cost one warp each, with no
// workspace: the output slots hold the keys while the call runs.
#include <cuda_runtime.h>
#include <limits.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <utility>

#include "../../include/grayskull_corners.h"

// the reference's gs_assert (grayskull.h:94-98): message + abort
#define GSK_ASSERT(cond)                                \
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

// Every kernel launch of this library: launch, check.
template <class... P, class... A>
static int launch(const char *file, int line, void (*k)(P...), dim3 grid, dim3 block, cudaStream_t s, A &&...a) {
  k<<<grid, block, 0, s>>>(std::forward<A>(a)...);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : record_error(e, file, line);
}
#define GSK_LAUNCH(...)                                         \
  do {                                                          \
    int gsk_rc_ = gsb::launch(__FILE__, __LINE__, __VA_ARGS__); \
    if (gsk_rc_) return gsk_rc_;                                \
  } while (0)

constexpr unsigned GRID_MAX = 65535u;       // grid y limit: frames beyond it loop
constexpr unsigned CTA = 256, WARPS = CTA / 32;
constexpr unsigned TILE_W = 256, TILE_H = 64;
constexpr unsigned SMALL_W = 256, SMALL_H = 16;   // a clipped box within this is one warp's record
constexpr unsigned NONE = 0xffffffffu;
constexpr unsigned long long NOKEY = ~0ull;      // no pixel counted; w * h < 2^32 - 1 keeps every real key below it
constexpr unsigned FULL = 0xffffffffu;

__device__ __forceinline__ unsigned umin(unsigned a, unsigned b) { return a < b ? a : b; }
__device__ __forceinline__ unsigned umax(unsigned a, unsigned b) { return a > b ? a : b; }

// a record's label and its box clipped to the frame.  The reference's loop bounds box.x + box.w and box.y + box.h are
// 32-bit sums: a box whose end wraps past 2^32 visits nothing.
struct Rec {
  unsigned label, x, y, cw, ch;
};
__device__ __forceinline__ Rec load_rec(const struct gs_blob *b, unsigned w, unsigned h) {
  const unsigned *p = reinterpret_cast<const unsigned *>(b);
  const unsigned bx = p[2], by = p[3], xe = bx + p[4], ye = by + p[5];
  Rec r;
  r.label = p[0] & 0xffffu, r.x = bx, r.y = by;
  r.cw = xe < bx || bx >= w ? 0u : umin(xe, w) - bx;
  r.ch = ye < by || by >= h ? 0u : umin(ye, h) - by;
  return r;
}
__device__ __forceinline__ bool is_large(const Rec &r) { return r.cw > SMALL_W || r.ch > SMALL_H; }

// v: an int's two's-complement bits; flipping the sign bit orders every int as unsigned
__device__ __forceinline__ unsigned long long key(unsigned v, unsigned p) {
  return ((unsigned long long)(v ^ 0x80000000u) << 32) | p;
}

// One warp, one row of at most 256 columns starting at irow / lrow: the first and the last qualifying column (NONE
// when there is none).  Lane l reads columns l, l + 32, ..., l + 224, so the warp's loads of one step are contiguous.
__device__ __forceinline__ void scan_row(const uint8_t *__restrict__ irow, const uint16_t *__restrict__ lrow,
                                         unsigned cols, unsigned label, unsigned lane, unsigned &first,
                                         unsigned &last) {
  uint8_t v[8];
  bool any = false;
#pragma unroll
  for (unsigned j = 0; j < 8; j++) {
    const unsigned c = lane + 32 * j;
    v[j] = c < cols ? __ldg(irow + c) : 0;
    any |= v[j] >= 128;
  }
  unsigned lo = NONE, hi = 0;   // hi: last + 1
  if (__any_sync(FULL, any)) {
#pragma unroll
    for (unsigned j = 0; j < 8; j++) {
      const unsigned c = lane + 32 * j;
      if (v[j] >= 128 && __ldg(lrow + c) == label) lo = umin(lo, c), hi = c + 1;
    }
  }
  first = __reduce_min_sync(FULL, lo);
  last = __reduce_max_sync(FULL, hi) - 1;
}

// a row's candidates: tl (least x + y) and bl (least x - y) at its first pixel, tr (greatest x - y) and br (greatest
// x + y) at its last.  tl and bl start from INT_MAX in the reference, and only a smaller value replaces it.
// The reference's (int)x + (int)y and (int)x - (int)y, and their negations, as wrapping 32-bit arithmetic.
__device__ __forceinline__ void take(unsigned long long k[4], unsigned xl, unsigned xr, unsigned y, unsigned w) {
  const unsigned sl = xl + y, dl = xl - y, sr = xr + y, dr = xr - y;
  const unsigned pl = y * w + xl, pr = y * w + xr;   // w * h < 2^32 - 1
  unsigned long long c;
  if (sl != (unsigned)INT_MAX) c = key(sl, pl), k[0] = c < k[0] ? c : k[0];
  c = key(0u - dr, pr), k[1] = c < k[1] ? c : k[1];
  c = key(0u - sr, pr), k[2] = c < k[2] ? c : k[2];
  if (dl != (unsigned)INT_MAX) c = key(dl, pl), k[3] = c < k[3] ? c : k[3];
}

__device__ __forceinline__ unsigned long long pick4(const unsigned long long k[4], unsigned q) {
  return q == 0 ? k[0] : q == 1 ? k[1] : q == 2 ? k[2] : k[3];
}

// a key as the point it stands for, x in the low word; the centroid (cx, cy) for the empty key
__device__ __forceinline__ unsigned long long point_of(unsigned long long k, unsigned w, unsigned cx, unsigned cy) {
  if (k == NOKEY) return cx | (unsigned long long)cy << 32;
  const unsigned p = (unsigned)k;
  return (p % w) | (unsigned long long)(p / w) << 32;
}

__device__ __forceinline__ unsigned used(const unsigned *counts, unsigned long long f, unsigned stride) {
  return counts ? umin(counts[f], stride) : stride;
}

// ---- the pick -------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(CTA)
k_largest_blob(const struct gs_blob *__restrict__ blobs, const unsigned *__restrict__ counts, unsigned stride,
               unsigned n, unsigned min_area, struct gs_blob *__restrict__ pick, unsigned *__restrict__ pcount) {
  const unsigned lane = threadIdx.x & 31;
  for (unsigned long long f = (blockIdx.x * (unsigned long long)CTA + threadIdx.x) / 32; f < n;
       f += (unsigned long long)gridDim.x * WARPS) {
    const unsigned c = used(counts, f, stride);
    const unsigned *rec = reinterpret_cast<const unsigned *>(blobs + f * stride);
    // (area, ~index): the greatest is the largest area at the lowest index
    unsigned long long best = 0;
    for (unsigned i = lane; i < c; i += 32) {
      const unsigned long long k = (unsigned long long)rec[8ull * i + 1] << 32 | (~i);
      best = k > best ? k : best;
    }
#pragma unroll
    for (unsigned d = 16; d; d >>= 1) {
      const unsigned long long o = __shfl_xor_sync(FULL, best, d);
      best = o > best ? o : best;
    }
    unsigned *out = reinterpret_cast<unsigned *>(pick + f);
    if (lane < 8) {
      // gs_blobs' initial record (grayskull.h:338): label 0, area 0, box {UINT_MAX, UINT_MAX, 0, 0}, centroid {0, 0}
      const unsigned init = lane == 2 || lane == 3 ? NONE : 0u;
      out[lane] = c ? rec[8ull * (~(unsigned)best) + lane] : init;
    }
    if (pcount && lane == 0) pcount[f] = c > 0 && (unsigned)(best >> 32) >= min_area;
  }
}

// ---- corners ----------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(CTA)
k_corners_small(const uint8_t *__restrict__ img, unsigned w, unsigned h, unsigned n, const uint16_t *__restrict__ labels,
                const struct gs_blob *__restrict__ blobs, const unsigned *__restrict__ counts, unsigned stride,
                unsigned long long *__restrict__ slots) {
  const unsigned lane = threadIdx.x & 31;
  const unsigned long long total = (unsigned long long)n * stride, fpix = (unsigned long long)w * h;
  for (unsigned long long i = (blockIdx.x * (unsigned long long)CTA + threadIdx.x) / 32; i < total;
       i += (unsigned long long)gridDim.x * WARPS) {
    const unsigned long long f = i / stride;
    if (i - f * stride >= used(counts, f, stride)) continue;
    const Rec r = load_rec(blobs + i, w, h);
    unsigned long long *out = slots + 4 * i;
    if (is_large(r)) {
      if (lane < 4) out[lane] = NOKEY;   // k_corners_tiles gathers this record's keys here
      continue;
    }
    unsigned long long k[4] = {NOKEY, NOKEY, NOKEY, NOKEY};
    const uint8_t *fi = img + f * fpix;
    const uint16_t *fl = labels + f * fpix;
    for (unsigned y = r.y; y < r.y + r.ch; y++) {
      const size_t row = (size_t)y * w + r.x;
      unsigned first, last;
      scan_row(fi + row, fl + row, r.cw, r.label, lane, first, last);
      if (first != NONE) take(k, r.x + first, r.x + last, y, w);
    }
    if (lane < 4) {
      const unsigned *c = reinterpret_cast<const unsigned *>(blobs + i) + 6;
      out[lane] = point_of(pick4(k, lane), w, c[0], c[1]);
    }
  }
}

__global__ void __launch_bounds__(CTA)
k_corners_tiles(const uint8_t *__restrict__ img, unsigned w, unsigned h, unsigned n, const uint16_t *__restrict__ labels,
                const struct gs_blob *__restrict__ blobs, const unsigned *__restrict__ counts, unsigned stride,
                unsigned long long *__restrict__ slots, unsigned tiles_x) {
  __shared__ unsigned s_list[CTA];
  __shared__ unsigned s_n;
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned long long fpix = (unsigned long long)w * h;
  for (unsigned f = blockIdx.y; f < n; f += gridDim.y) {
    const unsigned cnt = used(counts, f, stride);
    const struct gs_blob *fb = blobs + (unsigned long long)f * stride;
    const uint8_t *fi = img + f * fpix;
    const uint16_t *fl = labels + f * fpix;
    {   // one tile per CTA: a loop over tiles here costs the kernel register spills
      const unsigned t = blockIdx.x;
      const unsigned tx0 = t % tiles_x * TILE_W, ty0 = t / tiles_x * TILE_H;
      const unsigned tx1 = tx0 + umin(TILE_W, w - tx0), ty1 = ty0 + umin(TILE_H, h - ty0);
      for (unsigned c0 = 0; c0 < cnt; c0 += CTA) {
        if (threadIdx.x == 0) s_n = 0;
        __syncthreads();
        const unsigned k = c0 + threadIdx.x;
        if (k < cnt) {
          const Rec r = load_rec(fb + k, w, h);
          if (is_large(r) && r.x < tx1 && r.x + r.cw > tx0 && r.y < ty1 && r.y + r.ch > ty0)
            s_list[atomicAdd(&s_n, 1u)] = k;
        }
        __syncthreads();
        const unsigned m = s_n;
        for (unsigned j = 0; j < m; j++) {
          const unsigned rk = s_list[j];
          const Rec r = load_rec(fb + rk, w, h);
          const unsigned x0 = umax(r.x, tx0), x1 = umin(r.x + r.cw, tx1);
          const unsigned y1 = umin(r.y + r.ch, ty1);
          unsigned long long kk[4] = {NOKEY, NOKEY, NOKEY, NOKEY};
          for (unsigned y = umax(r.y, ty0) + warp; y < y1; y += WARPS) {
            const size_t row = (size_t)y * w + x0;
            unsigned first, last;
            scan_row(fi + row, fl + row, x1 - x0, r.label, lane, first, last);
            if (first != NONE) take(kk, x0 + first, x0 + last, y, w);
          }
          if (lane < 4) {
            const unsigned long long mine = pick4(kk, lane);
            unsigned long long *slot = slots + 4 * ((unsigned long long)f * stride + rk) + lane;
            if (mine < *reinterpret_cast<volatile unsigned long long *>(slot)) atomicMin(slot, mine);
          }
        }
        __syncthreads();   // s_list and s_n are rewritten for the next chunk
      }
    }
  }
}

__global__ void __launch_bounds__(CTA)
k_corners_final(unsigned w, unsigned h, unsigned n, const struct gs_blob *__restrict__ blobs,
                const unsigned *__restrict__ counts, unsigned stride, unsigned long long *__restrict__ slots) {
  const unsigned long long total = (unsigned long long)n * stride;
  for (unsigned long long i = blockIdx.x * (unsigned long long)CTA + threadIdx.x; i < total;
       i += (unsigned long long)gridDim.x * CTA) {
    const unsigned long long f = i / stride;
    if (i - f * stride >= used(counts, f, stride) || !is_large(load_rec(blobs + i, w, h))) continue;
    const unsigned *c = reinterpret_cast<const unsigned *>(blobs + i) + 6;
    unsigned long long k[4];
#pragma unroll
    for (unsigned q = 0; q < 4; q++) k[q] = slots[4 * i + q];
#pragma unroll
    for (unsigned q = 0; q < 4; q++) slots[4 * i + q] = point_of(k[q], w, c[0], c[1]);
  }
}

static unsigned blocks_for(unsigned long long items, unsigned per_block, unsigned long long cap) {
  const unsigned long long b = (items + per_block - 1) / per_block;
  return static_cast<unsigned>(b < cap ? (b ? b : 1) : cap);
}

}  // namespace gsb

using namespace gsb;

extern "C" const char *gs_b200_corners_last_error(void) { return t_last_error; }

extern "C" int gs_b200_largest_blob_batch(const struct gs_blob *blobs, const unsigned *counts, unsigned stride,
                                          unsigned n, unsigned min_area, struct gs_blob *pick, unsigned *pcount,
                                          gs_b200_stream s) {
  if (n == 0) return 0;
  GSK_ASSERT(blobs && pick);
  GSK_LAUNCH(k_largest_blob, dim3(blocks_for(n, WARPS, 132ull * 64)), dim3(CTA), (cudaStream_t)s, blobs, counts,
             stride, n, min_area, pick, pcount);
  return 0;
}

extern "C" int gs_b200_blob_corners_batch(const uint8_t *img, unsigned w, unsigned h, unsigned n,
                                          const gs_label *labels, const struct gs_blob *blobs, const unsigned *counts,
                                          unsigned stride, struct gs_point *corners, gs_b200_stream s) {
  if (n == 0) return 0;
  GSK_ASSERT(img && labels && blobs && corners);
  GSK_ASSERT(w > 0 && h > 0);
  if (reinterpret_cast<uintptr_t>(corners) & 7u) return invalid("corners is not 8-byte aligned", __FILE__, __LINE__);
  if (stride == 0) return 0;
  const cudaStream_t st = (cudaStream_t)s;
  unsigned long long *slots = reinterpret_cast<unsigned long long *>(corners);
  const unsigned long long records = (unsigned long long)n * stride;
  // w * h < 2^32 keeps the tiles of a frame below 2^31, within the grid's x limit
  const unsigned tiles_x = (w - 1) / TILE_W + 1, tiles = tiles_x * ((h - 1) / TILE_H + 1);
  GSK_LAUNCH(k_corners_small, dim3(blocks_for(records, WARPS, 132ull * 32)), dim3(CTA), st, img, w, h, n, labels,
             blobs, counts, stride, slots);
  GSK_LAUNCH(k_corners_tiles, dim3(tiles, n < GRID_MAX ? n : GRID_MAX), dim3(CTA), st, img, w, h, n, labels, blobs,
             counts, stride, slots, tiles_x);
  GSK_LAUNCH(k_corners_final, dim3(blocks_for(records, CTA, 132ull * 32)), dim3(CTA), st, w, h, n, blobs, counts,
             stride, slots);
  return 0;
}
