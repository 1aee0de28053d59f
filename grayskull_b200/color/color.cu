// color.cu -- libgrayskull_color.so: the wasm demo's colour conversions over frame batches (include/grayskull_color.h),
// bit-exact with examples/wasm/grayskull.js:33-45.
//
// Frames are dense and back to back, so a batch is one stream of n * w * h pixels and neither the frame size nor the
// batch size picks a path; only the pointers' alignment does.  Pixel i of src is at src + C * i and of dst at dst + i
// (gray -> RGBA: src + i and dst + 4 * i), so 16-byte words line up on the colour side with aligned words on the gray
// side exactly when src - C * dst (gray -> RGBA: dst - 4 * src) is a multiple of 16.  That holds for any sub-batch
// view of two 16-byte aligned tensors, since there the two offsets are k * w * h * C and k * w * h.
//   k_rgb_gray_wide      RGB, 16 pixels per thread: three 16-byte loads, one 16-byte store
//   k_rgba_gray_wide     RGBA, 4 pixels per 16-byte word, one 4-byte store per word; each warp instruction covers one
//                        contiguous span
//   k_gray_rgba_wide     4 pixels per 4-byte load, one 16-byte store, laid out as k_rgba_gray_wide
//   k_rgb_gray_bytes<C>, k_gray_rgba_bytes   any other alignment: one pixel per thread, byte loads and stores
// The wide kernels take the pixels before dst's (gray -> RGBA: src's) first 16- or 4-byte boundary and the ragged end
// one per thread.
//
// Exactness.  The demo computes 0.299 * r + 0.587 * g + 0.114 * b in IEEE double, left to right, each operation
// rounded to nearest, and stores it into a Uint8Array, which truncates (ES ToUint8); the value lies in [0, 255], so
// that is floor.  gray_of() does the same five operations with __dmul_rn / __dadd_rn, which are never contracted into
// a DFMA (and -fmad=false forbids that anyway).  It avoids the I2F.F64 / F2I.F64 conversions: a byte b becomes the
// double with bit pattern 0x43300000:b, which is 2^52 + b exactly, minus 2^52 (exact); and floor(v) for v in [0, 256)
// is the low word of v + 2^52 rounded down, since the doubles in [2^52, 2^53) are the integers.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <utility>

#include "../../include/grayskull_color.h"

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

constexpr unsigned THREADS = 256;
constexpr unsigned CTAS_PER_SM = 8;   // 8 x 256 threads: a full SM, so the grid-stride loops keep every SM streaming

// ---- the demo's rule ------------------------------------------------------------------------------------------------
__device__ __forceinline__ double byte_to_double(unsigned b) {
  return __dadd_rn(__hiloint2double(0x43300000, static_cast<int>(b)), -0x1p52);
}

__device__ __forceinline__ unsigned gray_of(unsigned r, unsigned g, unsigned b) {
  const double v = __dadd_rn(__dadd_rn(__dmul_rn(0.299, byte_to_double(r)), __dmul_rn(0.587, byte_to_double(g))),
                             __dmul_rn(0.114, byte_to_double(b)));
  return static_cast<unsigned>(__double2loint(__dadd_rd(v, 0x1p52)));
}

// byte k (a compile-time constant after unrolling) of words w[0..], little-endian
template <unsigned N>
__device__ __forceinline__ unsigned byte_at(const unsigned (&w)[N], unsigned k) {
  return __byte_perm(w[k >> 2], 0u, 0x4440u | (k & 3u));
}

// ---- colour -> gray -------------------------------------------------------------------------------------------------
template <unsigned C>
__device__ __forceinline__ void rgb_gray_one(uint8_t *__restrict__ dst, const uint8_t *__restrict__ src,
                                             unsigned long long i) {
  const uint8_t *p = src + i * C;
  dst[i] = static_cast<uint8_t>(gray_of(p[0], p[1], p[2]));
}

// pixels [0, head) and [tail, pixels), fewer than 16 each, one per thread of the first warp
#define GSK_HEAD_AND_TAIL(one)                                                              \
  if (blockIdx.x == 0 && threadIdx.x < 32) {                                                \
    const unsigned long long i = threadIdx.x < 16 ? threadIdx.x : tail + threadIdx.x - 16; \
    if (threadIdx.x < 16 ? i < head : i < pixels) one;                                      \
  }

// RGB: groups of 16 pixels from `head` on, 48 bytes in and 16 out per thread
__global__ void __launch_bounds__(THREADS, CTAS_PER_SM)
k_rgb_gray_wide(uint8_t *__restrict__ dst, const uint8_t *__restrict__ src, unsigned long long pixels, unsigned head) {
  const unsigned long long groups = (pixels - head) / 16, tail = head + groups * 16;
  const uint4 *s4 = reinterpret_cast<const uint4 *>(src + (unsigned long long)head * 3);   // 16-byte aligned
  uint4 *d4 = reinterpret_cast<uint4 *>(dst + head);                                      // 16-byte aligned
  for (unsigned long long g = blockIdx.x * (unsigned long long)THREADS + threadIdx.x; g < groups;
       g += (unsigned long long)gridDim.x * THREADS) {
    unsigned w[12];
#pragma unroll
    for (unsigned k = 0; k < 3; k++) {
      const uint4 v = s4[g * 3 + k];
      w[4 * k] = v.x, w[4 * k + 1] = v.y, w[4 * k + 2] = v.z, w[4 * k + 3] = v.w;
    }
    unsigned o[4];
#pragma unroll
    for (unsigned q = 0; q < 4; q++) {
      unsigned y[4];
#pragma unroll
      for (unsigned j = 0; j < 4; j++) {
        const unsigned p = 4 * q + j;
        y[j] = gray_of(byte_at(w, 3 * p), byte_at(w, 3 * p + 1), byte_at(w, 3 * p + 2));
      }
      o[q] = __byte_perm(__byte_perm(y[0], y[1], 0x0040u), __byte_perm(y[2], y[3], 0x0040u), 0x5410u);
    }
    __stcs(d4 + g, make_uint4(o[0], o[1], o[2], o[3]));
  }
  GSK_HEAD_AND_TAIL(rgb_gray_one<3>(dst, src, i))
}

// RGBA: words of 4 pixels from `head` on, 16 bytes in and 4 out.  A CTA takes 4 * THREADS words at a time, thread t
// words t, t + THREADS, ... of them, so that every load and store instruction of a warp covers one contiguous span
// (512 bytes in, 128 out); all four loads are issued before the first word is converted.
__global__ void __launch_bounds__(THREADS, CTAS_PER_SM)
k_rgba_gray_wide(uint8_t *__restrict__ dst, const uint8_t *__restrict__ src, unsigned long long pixels,
                 unsigned head) {
  const unsigned long long words = (pixels - head) / 4, tail = head + words * 4;
  const uint4 *s4 = reinterpret_cast<const uint4 *>(src + (unsigned long long)head * 4);   // 16-byte aligned
  unsigned *d1 = reinterpret_cast<unsigned *>(dst + head);                                // 4-byte aligned
  for (unsigned long long base = blockIdx.x * 4ull * THREADS + threadIdx.x; base < words;
       base += gridDim.x * 4ull * THREADS) {
    uint4 v[4];
#pragma unroll
    for (unsigned k = 0; k < 4; k++)
      if (base + k * THREADS < words) v[k] = s4[base + k * THREADS];
#pragma unroll
    for (unsigned k = 0; k < 4; k++)
      if (base + k * THREADS < words) {
        const unsigned px[4] = {v[k].x, v[k].y, v[k].z, v[k].w};
        unsigned y[4];
#pragma unroll
        for (unsigned j = 0; j < 4; j++)
          y[j] = gray_of(byte_at(px, 4 * j), byte_at(px, 4 * j + 1), byte_at(px, 4 * j + 2));
        __stcs(d1 + base + k * THREADS,
               __byte_perm(__byte_perm(y[0], y[1], 0x0040u), __byte_perm(y[2], y[3], 0x0040u), 0x5410u));
      }
  }
  GSK_HEAD_AND_TAIL(rgb_gray_one<4>(dst, src, i))
}

template <unsigned C>
__global__ void __launch_bounds__(THREADS, CTAS_PER_SM)
k_rgb_gray_bytes(uint8_t *__restrict__ dst, const uint8_t *__restrict__ src, unsigned long long pixels) {
  for (unsigned long long i = blockIdx.x * (unsigned long long)THREADS + threadIdx.x; i < pixels;
       i += (unsigned long long)gridDim.x * THREADS)
    rgb_gray_one<C>(dst, src, i);
}

// ---- gray -> RGBA ---------------------------------------------------------------------------------------------------
// (g, g, g, 255) from byte j of word v
__device__ __forceinline__ unsigned rgba_of(unsigned v, unsigned j) {
  return __byte_perm(v, 0xffu, 0x4000u | j * 0x111u);
}

__device__ __forceinline__ void gray_rgba_one(uint8_t *__restrict__ dst, const uint8_t *__restrict__ src,
                                              unsigned long long i) {
  const uint8_t g = src[i];
  dst[4 * i] = dst[4 * i + 1] = dst[4 * i + 2] = g, dst[4 * i + 3] = 255;
}

// words of 4 pixels from `head` on, 4 bytes in and 16 out, laid over the CTA as in k_rgba_gray_wide
__global__ void __launch_bounds__(THREADS, CTAS_PER_SM)
k_gray_rgba_wide(uint8_t *__restrict__ dst, const uint8_t *__restrict__ src, unsigned long long pixels,
                 unsigned head) {
  const unsigned long long words = (pixels - head) / 4, tail = head + words * 4;
  const unsigned *s1 = reinterpret_cast<const unsigned *>(src + head);            // 4-byte aligned
  uint4 *d4 = reinterpret_cast<uint4 *>(dst + (unsigned long long)head * 4);    // 16-byte aligned
  for (unsigned long long base = blockIdx.x * 4ull * THREADS + threadIdx.x; base < words;
       base += gridDim.x * 4ull * THREADS) {
    unsigned v[4];
#pragma unroll
    for (unsigned k = 0; k < 4; k++)
      if (base + k * THREADS < words) v[k] = s1[base + k * THREADS];
#pragma unroll
    for (unsigned k = 0; k < 4; k++)
      if (base + k * THREADS < words)
        __stcs(d4 + base + k * THREADS, make_uint4(rgba_of(v[k], 0), rgba_of(v[k], 1), rgba_of(v[k], 2),
                                                   rgba_of(v[k], 3)));
  }
  GSK_HEAD_AND_TAIL(gray_rgba_one(dst, src, i))
}

__global__ void __launch_bounds__(THREADS, CTAS_PER_SM)
k_gray_rgba_bytes(uint8_t *__restrict__ dst, const uint8_t *__restrict__ src, unsigned long long pixels) {
  for (unsigned long long i = blockIdx.x * (unsigned long long)THREADS + threadIdx.x; i < pixels;
       i += (unsigned long long)gridDim.x * THREADS)
    gray_rgba_one(dst, src, i);
}

// ---- entry points ---------------------------------------------------------------------------------------------------
static bool overlap(const void *a, unsigned long long an, const void *b, unsigned long long bn) {
  const uintptr_t pa = reinterpret_cast<uintptr_t>(a), pb = reinterpret_cast<uintptr_t>(b);
  return an && bn && pa < pb + bn && pb < pa + an;
}

// enough CTAs for `items`, at most CTAS_PER_SM per SM of the current device
static int blocks_for(unsigned long long items, unsigned *blocks) {
  int dev = 0, sms = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (e != cudaSuccess) return record_error(e, __FILE__, __LINE__);
  const unsigned long long b = (items + THREADS - 1) / THREADS, cap = (unsigned long long)sms * CTAS_PER_SM;
  *blocks = static_cast<unsigned>(b < cap ? (b ? b : 1) : cap);
  return 0;
}

// the pixels before the first `align`-byte boundary of `p`, at most `pixels`
static unsigned head_of(const void *p, unsigned align, unsigned long long pixels) {
  const unsigned h = (align - (reinterpret_cast<uintptr_t>(p) & (align - 1))) & (align - 1);
  return pixels < h ? static_cast<unsigned>(pixels) : h;
}

}  // namespace gsb

using namespace gsb;

extern "C" const char *gs_b200_color_last_error(void) { return t_last_error; }

extern "C" int gs_b200_rgb_to_gray_batch(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n,
                                         unsigned channels, gs_b200_stream s) {
  if (n == 0) return 0;
  GSK_ASSERT(dst && src);
  GSK_ASSERT(w > 0 && h > 0);
  if (channels != 3 && channels != 4) return invalid("channels is neither 3 nor 4", __FILE__, __LINE__);
  const unsigned long long pixels = (unsigned long long)w * h * n;
  if (overlap(dst, pixels, src, pixels * channels)) return invalid("dst overlaps src", __FILE__, __LINE__);
  const cudaStream_t st = (cudaStream_t)s;
  unsigned blocks;
  if (((reinterpret_cast<uintptr_t>(src) - channels * reinterpret_cast<uintptr_t>(dst)) & 15u) == 0) {
    if (channels == 3) {
      const unsigned head = head_of(dst, 16, pixels);
      if (int rc = blocks_for((pixels - head) / 16, &blocks)) return rc;
      GSK_LAUNCH(k_rgb_gray_wide, dim3(blocks), dim3(THREADS), st, dst, src, pixels, head);
    } else {
      const unsigned head = head_of(dst, 4, pixels);
      if (int rc = blocks_for((pixels - head) / 16, &blocks)) return rc;
      GSK_LAUNCH(k_rgba_gray_wide, dim3(blocks), dim3(THREADS), st, dst, src, pixels, head);
    }
  } else {
    if (int rc = blocks_for(pixels, &blocks)) return rc;
    if (channels == 3) GSK_LAUNCH(k_rgb_gray_bytes<3>, dim3(blocks), dim3(THREADS), st, dst, src, pixels);
    else GSK_LAUNCH(k_rgb_gray_bytes<4>, dim3(blocks), dim3(THREADS), st, dst, src, pixels);
  }
  return 0;
}

extern "C" int gs_b200_gray_to_rgba_batch(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n,
                                          gs_b200_stream s) {
  if (n == 0) return 0;
  GSK_ASSERT(dst && src);
  GSK_ASSERT(w > 0 && h > 0);
  const unsigned long long pixels = (unsigned long long)w * h * n;
  if (overlap(dst, pixels * 4, src, pixels)) return invalid("dst overlaps src", __FILE__, __LINE__);
  const cudaStream_t st = (cudaStream_t)s;
  unsigned blocks;
  if (((reinterpret_cast<uintptr_t>(dst) - 4 * reinterpret_cast<uintptr_t>(src)) & 15u) == 0) {
    const unsigned head = head_of(src, 4, pixels);
    if (int rc = blocks_for((pixels - head) / 16, &blocks)) return rc;
    GSK_LAUNCH(k_gray_rgba_wide, dim3(blocks), dim3(THREADS), st, dst, src, pixels, head);
  } else {
    if (int rc = blocks_for(pixels, &blocks)) return rc;
    GSK_LAUNCH(k_gray_rgba_bytes, dim3(blocks), dim3(THREADS), st, dst, src, pixels);
  }
  return 0;
}
