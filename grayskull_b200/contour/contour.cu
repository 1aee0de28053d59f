// contour.cu -- libgrayskull_contour.so: gs_trace_contour over frame batches (include/grayskull_contour.h), bit-exact
// with the reference's walk (grayskull.h:446-480), plus the wasm demo's start rule for blob records.
//
// A walk's path depends only on img; only `length` and `visited` depend on the order of a frame's contours.  So every
// contour of every frame in a chunk walks at once, and the order is applied afterwards over the pixels:
//   k_contour_clear    the chunk's u32 owner maps (in `work`) to ~0
//   k_contour_walk     one thread per contour: the walk with Brent's repeat test, box and end written, length = 0
//                      (1 for an out-of-frame start, which the reference counts once per call); each walked pixel
//                      takes atomicMin(owner[p], k), so it ends up owned by the first contour in list order to walk it
//   k_contour_mark     one thread per pixel: where owner != ~0, one more length for the owner if visited was 0 (warp
//                      peers with the same owner add once), then visited = 255
// That is the sequential result: a pixel counts for the first contour that walks it, and only if it was 0 before the
// call; a repeated start gets length 0; bytes the caller set beforehand never count.
//   k_contour_starts   one CTA per (frame, blob record): rows of the box in raster order until one holds the label
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <utility>

#include "../../include/grayskull_contour.h"

// the reference's gs_assert (grayskull.h:94-98): message + abort
#define GSC_ASSERT(cond)                                \
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
#define GSC_LAUNCH(...)                                         \
  do {                                                          \
    int gsc_rc_ = gsb::launch(__FILE__, __LINE__, __VA_ARGS__); \
    if (gsc_rc_) return gsc_rc_;                                \
  } while (0)

constexpr unsigned GRID_MAX = 65535u;   // grid y limit, and the frame loop of k_contour_starts
constexpr unsigned WALK_THREADS = 64;   // small CTAs: the few long walks of a sparse list spread over more SMs
constexpr unsigned NONE = 0xffffffffu;  // owner of a pixel no walk reached

__device__ __forceinline__ unsigned umin(unsigned a, unsigned b) { return a < b ? a : b; }
__device__ __forceinline__ unsigned umax(unsigned a, unsigned b) { return a > b ? a : b; }
// the reference's dx[d] and dy[d] (grayskull.h:449-450) as unsigned, from 2-bit fields of dx + 1 and dy + 1
__device__ __forceinline__ unsigned dx_of(unsigned d) { return ((0x901au >> (2 * d)) & 3u) - 1u; }
__device__ __forceinline__ unsigned dy_of(unsigned d) { return ((0x01a9u >> (2 * d)) & 3u) - 1u; }

// ---- owner maps --------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_contour_clear(unsigned *owner, unsigned long long words) {
  const unsigned long long t = blockIdx.x * 256ull + threadIdx.x, step = gridDim.x * 256ull;
  uint4 *o4 = reinterpret_cast<uint4 *>(owner);   // 16-byte aligned by the entry point
  for (unsigned long long i = t; i < words / 4; i += step) o4[i] = make_uint4(NONE, NONE, NONE, NONE);
  if (t < words % 4) owner[words / 4 * 4 + t] = NONE;
}

// ---- the walk -------------------------------------------------------------------------------------------------------
// Why it ends.  The step from (p, dir, seenstart) to the next state is a function of that state, img and start alone:
// visited and length never feed back into it.  p is start or an in-frame pixel, dir one of 8, seenstart 0 or 1, so a
// walk has at most S = 16 * (w * h + 1) = 16wh + 16 states.  A walk that neither returns nor gets stuck therefore
// repeats a state, and from then on it goes round the same cycle of lam states for ever: both stop tests are functions
// of the state, so neither can fire later.  mu + lam <= S, where mu is the index of the first state on the cycle.
// Brent's test keeps one saved state, the one at step 2^j - 1, and compares every later state with it until step
// 2^(j+1) - 1.  With the first J such that 2^J >= max(mu + 1, lam), the saved state is on the cycle and the match
// comes at step 2^J - 1 + lam < 2 * S + S.  The match closes one whole lap from a state on the cycle, so every pixel
// of the cycle has been walked (visited and length are final) and box.x / box.y are the minima over everything the
// walk will ever see.  box.w = max(box.w, p.x - box.x + 1) is taken with the box.x of its step, so a pixel walked
// before box.x reached its minimum can still widen the box on the next lap: one more lap of lam <= S steps applies
// every step of the cycle with the final box.x and box.y, after which no step changes anything.  So a walk ends within
// 4 * S steps, and the loop is bounded by that.
__global__ void __launch_bounds__(WALK_THREADS)
k_contour_walk(const uint8_t *__restrict__ img, unsigned w, unsigned h, unsigned frames,
               struct gs_contour *__restrict__ contours, const unsigned *__restrict__ counts, unsigned stride,
               uint8_t *__restrict__ ends, unsigned *__restrict__ owner) {
  const unsigned long long total = (unsigned long long)frames * stride, fpix = (unsigned long long)w * h;
  const unsigned long long limit = 4ull * (16ull * fpix + 16ull);
  const int iw = (int)w, ih = (int)h;
  for (unsigned long long i = blockIdx.x * (unsigned long long)WALK_THREADS + threadIdx.x; i < total;
       i += (unsigned long long)gridDim.x * WALK_THREADS) {
    const unsigned long long f = i / stride;
    const unsigned k = static_cast<unsigned>(i - f * stride);
    if (k >= (counts ? umin(counts[f], stride) : stride)) continue;
    const uint8_t *fi = img + f * fpix;
    unsigned *fo = owner + f * fpix;
    const unsigned sx = contours[i].start.x, sy = contours[i].start.y;
    unsigned px = sx, py = sy, dir = 7, seen = 0;
    unsigned bx = sx, by = sy, bw = 1, bh = 1;
    unsigned vx = px, vy = py, vds = dir;                 // Brent's saved state: p and dir | seenstart << 3
    unsigned long long power = 1, lam = 0, lap = 0;       // lap: steps left of the closing lap, once matched
    uint8_t end = GS_CONTOUR_CYCLE;
    for (unsigned long long t = 0; t < limit; t++) {
      if (px < w && py < h) atomicMin(&fo[(size_t)py * w + px], k);
      // the 8 neighbours inside the frame and > 128, as a mask by direction; nx = p.x + dx in unsigned, then as int
      unsigned mask = 0;
#pragma unroll
      for (unsigned d = 0; d < 8; d++) {
        const int nx = (int)(px + dx_of(d)), ny = (int)(py + dy_of(d));
        if (nx >= 0 && nx < iw && ny >= 0 && ny < ih && __ldg(fi + (size_t)ny * w + nx) > 128) mask |= 1u << d;
      }
      if (!mask) {
        end = GS_CONTOUR_OPEN;
        break;
      }
      const unsigned nd = (dir + 1) & 7, rot = ((mask >> nd) | (mask << (8 - nd))) & 255u;
      const unsigned d = (nd + __ffs(rot) - 1) & 7;      // the first foreground neighbour from nd on
      px += dx_of(d), py += dy_of(d);
      dir = (d + 6) & 7;
      bx = umin(bx, px), by = umin(by, py);
      bw = umax(bw, px - bx + 1), bh = umax(bh, py - by + 1);
      if (px == sx && py == sy) {
        if (seen) {
          end = GS_CONTOUR_RETURNED;
          break;
        }
        seen = 1;
      }
      if (lap) {
        if (--lap == 0) break;
        continue;
      }
      lam++;
      if (px == vx && py == vy && (dir | seen << 3) == vds) {
        lap = lam;
        continue;
      }
      if (lam == power) vx = px, vy = py, vds = dir | seen << 3, power <<= 1, lam = 0;
    }
    contours[i].box = gs_rect{bx, by, bw, bh};
    contours[i].length = sx < w && sy < h ? 0u : 1u;
    if (ends) ends[i] = end;
  }
}

// ---- list order over the pixels ------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_contour_mark(uint8_t *__restrict__ visited, const unsigned *__restrict__ owner, unsigned long long pixels,
               unsigned long long fpix, struct gs_contour *__restrict__ contours, unsigned stride) {
  const unsigned lane = threadIdx.x & 31;
  for (unsigned long long base = blockIdx.x * 256ull; base < pixels; base += gridDim.x * 256ull) {
    const unsigned long long i = base + threadIdx.x;   // the warp runs the loop together: __match_any_sync below
    unsigned long long rec = ~0ull;                     // the record this pixel counts for, if it counts
    if (i < pixels) {
      const unsigned o = owner[i];
      if (o != NONE) {
        if (visited[i] == 0) rec = i / fpix * stride + o;
        visited[i] = 255;
      }
    }
    const unsigned peers = __match_any_sync(0xffffffffu, rec);
    if (rec != ~0ull && lane == (unsigned)__ffs(peers) - 1) atomicAdd(&contours[rec].length, (unsigned)__popc(peers));
  }
}

// ---- starts ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_contour_starts(const gs_label *__restrict__ labels, unsigned w, unsigned h, unsigned n,
                 const struct gs_blob *__restrict__ blobs, const unsigned *__restrict__ counts, unsigned stride,
                 struct gs_contour *__restrict__ contours) {
  __shared__ unsigned s_x;
  const unsigned long long fpix = (unsigned long long)w * h;
  for (unsigned f = blockIdx.y; f < n; f += gridDim.y) {
    const unsigned cnt = counts ? umin(counts[f], stride) : stride;
    const gs_label *fl = labels + f * fpix;
    for (unsigned b = blockIdx.x; b < cnt; b += gridDim.x) {
      const struct gs_blob blob = blobs[(size_t)f * stride + b];
      // the demo's loops run while y < box.y + box.h and x < box.x + box.w, in unsigned arithmetic; inside the frame
      const unsigned long long xe = umin(blob.box.x + blob.box.w, w), ye = umin(blob.box.y + blob.box.h, h);
      unsigned sx = blob.box.x, sy = blob.box.y;
      for (unsigned long long y = blob.box.y; y < ye; y++) {
        if (threadIdx.x == 0) s_x = NONE;
        __syncthreads();
        for (unsigned long long x = blob.box.x + (unsigned long long)threadIdx.x; x < xe; x += 256)
          if (fl[y * w + x] == blob.label) {
            atomicMin(&s_x, static_cast<unsigned>(x));
            break;
          }
        __syncthreads();
        const unsigned fx = s_x;
        __syncthreads();   // s_x is reset for the next row
        if (fx != NONE) {
          sx = fx, sy = static_cast<unsigned>(y);
          break;
        }
      }
      if (threadIdx.x == 0) contours[(size_t)f * stride + b].start = gs_point{sx, sy};
    }
  }
}

// ---- entry points ---------------------------------------------------------------------------------------------------
static bool overlap(const void *a, unsigned long long an, const void *b, unsigned long long bn) {
  const uintptr_t pa = reinterpret_cast<uintptr_t>(a), pb = reinterpret_cast<uintptr_t>(b);
  return an && bn && pa < pb + bn && pb < pa + an;
}

static unsigned blocks_for(unsigned long long items, unsigned per_block, unsigned long long cap) {
  const unsigned long long b = (items + per_block - 1) / per_block;
  return static_cast<unsigned>(b < cap ? (b ? b : 1) : cap);
}

}  // namespace gsb

using namespace gsb;

extern "C" const char *gs_b200_contour_last_error(void) { return t_last_error; }

extern "C" size_t gs_b200_trace_contours_work_bytes(unsigned w, unsigned h, unsigned n) {
  const unsigned __int128 b = (unsigned __int128)4u * w * h * n + 16u;
  return b > (unsigned __int128)SIZE_MAX ? SIZE_MAX : static_cast<size_t>(b);
}

extern "C" int gs_b200_trace_contours_batch(const uint8_t *img, uint8_t *visited, unsigned w, unsigned h, unsigned n,
                                            struct gs_contour *contours, const unsigned *counts, unsigned stride,
                                            uint8_t *ends, void *work, size_t work_bytes, gs_b200_stream s) {
  if (n == 0) return 0;
  GSC_ASSERT(img && visited && contours && work);
  GSC_ASSERT(w > 0 && h > 0);
  const unsigned long long fpix = (unsigned long long)w * h;
  if (overlap(img, fpix * n, visited, fpix * n)) return invalid("visited overlaps img", __FILE__, __LINE__);
  // the owner maps start at work's first 16-byte boundary
  const size_t pad = (16u - (reinterpret_cast<uintptr_t>(work) & 15u)) & 15u;
  if (work_bytes < pad || (work_bytes - pad) / 4 / fpix == 0)
    return invalid("work_bytes below one frame's owner map", __FILE__, __LINE__);
  if (stride == 0) return 0;
  unsigned *owner = reinterpret_cast<unsigned *>(static_cast<uint8_t *>(work) + pad);
  const unsigned long long fit = (work_bytes - pad) / 4 / fpix, chunk = fit < n ? fit : n;
  const cudaStream_t st = (cudaStream_t)s;
  for (unsigned long long f0 = 0; f0 < n; f0 += chunk) {
    const unsigned m = static_cast<unsigned>(n - f0 < chunk ? n - f0 : chunk);
    const unsigned long long pixels = fpix * m, walks = (unsigned long long)m * stride;
    GSC_LAUNCH(k_contour_clear, dim3(blocks_for(pixels / 4 + 1, 256, 132ull * 32)), dim3(256), st, owner, pixels);
    GSC_LAUNCH(k_contour_walk, dim3(blocks_for(walks, WALK_THREADS, 1ull << 30)), dim3(WALK_THREADS), st,
               img + f0 * fpix, w, h, m, contours + f0 * stride, counts ? counts + f0 : nullptr, stride,
               ends ? ends + f0 * stride : nullptr, owner);
    GSC_LAUNCH(k_contour_mark, dim3(blocks_for(pixels, 256, 132ull * 32)), dim3(256), st, visited + f0 * fpix, owner,
               pixels, fpix, contours + f0 * stride, stride);
  }
  return 0;
}

extern "C" int gs_b200_blob_contour_starts_batch(const gs_label *labels, unsigned w, unsigned h, unsigned n,
                                                 const struct gs_blob *blobs, const unsigned *counts, unsigned stride,
                                                 struct gs_contour *contours, gs_b200_stream s) {
  if (n == 0) return 0;
  GSC_ASSERT(labels && blobs && contours);
  GSC_ASSERT(w > 0 && h > 0);
  if (stride == 0) return 0;
  GSC_LAUNCH(k_contour_starts, dim3(stride < 4096u ? stride : 4096u, n < GRID_MAX ? n : GRID_MAX), dim3(256),
             (cudaStream_t)s, labels, w, h, n, blobs, counts, stride, contours);
  return 0;
}
