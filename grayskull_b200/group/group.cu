// group.cu -- libgrayskull_group.so: neighbour-counted grouping of each frame's LBP detections over frame batches
// (include/grayskull_group.h), the rule of OpenCV's groupRectangles as the header states it.
//
// A chunk of m frames runs as five kernels, each frame's state in `work`:
//   k_group_init    parent[i] = i and zeroed group sums for every used record
//   k_group_pairs   one CTA per (frame, tile i, tile j >= i) of TILE records: both tiles staged in shared memory, every
//                   similar pair united by hooking the larger root onto the smaller with atomicMin on parent[].  Every
//                   parent is at most its own index, so each group's final root is its smallest record index; the
//                   partition and its numbering do not depend on the order of the unions
//   k_group_roots   one CTA per frame: parent[] flattened to roots, an in-order scan of the root flags numbers the
//                   groups, then 64-bit integer atomicAdd of every record into its group's sums (order-free) and the
//                   fp32 average per group
//   k_group_filter  one CTA per (frame, GROUP_TILE groups): the containment test of each group with more than K
//                   members against every other such group
//   k_group_emit    one CTA per frame: an ordered compaction of the survivors into out, weights and out_counts
// K == 0, stride == 0 and out_stride == 0 are k_group_copy alone: the first min(c, out_stride) records, weight 1.
// The library is compiled with -fmad=false, and the rule's products are explicit __dmul_rn / __fmul_rn.
#include <cuda_runtime.h>
#include <math.h>
#include <limits.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <utility>

#include "../../include/grayskull_group.h"

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

constexpr unsigned GRID_MAX = 65535u;   // grid y limit: frames beyond it loop
constexpr unsigned CTA = 256;
constexpr unsigned SCAN_CTA = 1024;     // the per-frame scans
constexpr unsigned TILE = 128;          // records per pair tile: CTA threads = 2 * TILE
constexpr unsigned GROUP_TILE = CTA;    // groups per filter tile
constexpr unsigned FULL = 0xffffffffu;
constexpr long long FAR = 1ll << 40;    // beyond every difference of two 33-bit field sums
constexpr double FAR_D = 1099511627776.0;
// bytes of one frame's state per record: four u64 sums, the uint4 group rect, parent, group number, size, keep
constexpr unsigned long long PER_RECORD = 4 * 8 + 16 + 4 * 4;

__device__ __forceinline__ unsigned umin(unsigned a, unsigned b) { return a < b ? a : b; }

__device__ __forceinline__ unsigned used(const unsigned *counts, unsigned long long f, unsigned stride) {
  return counts ? umin(counts[f], stride) : stride;
}

// a record as (x, y, w, h); the lists need only gs_rect's 4-byte alignment
__device__ __forceinline__ uint4 load_rect(const struct gs_rect *r) { return make_uint4(r->x, r->y, r->w, r->h); }
__device__ __forceinline__ void store_rect(struct gs_rect *r, uint4 v) { r->x = v.x, r->y = v.y, r->w = v.z, r->h = v.w; }

__device__ __forceinline__ unsigned long long absdiff(unsigned long long a, unsigned long long b) {
  return a > b ? a - b : b - a;
}

// rule 1.  Every difference is an integer, so |d| <= delta is |d| <= floor(delta); a delta of 2^40 or more (eps large
// enough to overflow to inf included) admits every difference.
__device__ __forceinline__ bool similar(uint4 a, uint4 b, double eps) {
  const unsigned long long s = (unsigned long long)umin(a.z, b.z) + umin(a.w, b.w);
  const double delta = __dmul_rn(__dmul_rn(eps, __ull2double_rn(s)), 0.5);
  const unsigned long long d = delta >= FAR_D ? (unsigned long long)FAR : (unsigned long long)delta;
  return absdiff(a.x, b.x) <= d && absdiff(a.y, b.y) <= d &&
         absdiff((unsigned long long)a.x + a.z, (unsigned long long)b.x + b.z) <= d &&
         absdiff((unsigned long long)a.y + a.w, (unsigned long long)b.y + b.w) <= d;
}

// rint((double)v * eps), half to even, as an integer; 2^40 stands for anything larger
__device__ __forceinline__ long long slack(unsigned v, double eps) {
  const double r = rint(__dmul_rn(__uint2double_rn(v), eps));
  return r >= FAR_D ? FAR : (long long)r;
}

// rule 4: group j (rect bj, mj members) contains group i
__device__ __forceinline__ bool contains(uint4 bj, unsigned mj, uint4 bi, unsigned mi, double eps) {
  const long long dx = slack(bj.z, eps), dy = slack(bj.w, eps);
  return (long long)bi.x >= (long long)bj.x - dx && (long long)bi.y >= (long long)bj.y - dy &&
         (long long)bi.x + bi.z <= (long long)bj.x + bj.z + dx && (long long)bi.y + bi.w <= (long long)bj.y + bj.w + dy &&
         (mj > (mi > 3u ? mi : 3u) || mi < 3u);
}

// the root of x; parents only ever decrease, so a stale read is still an ancestor
__device__ __forceinline__ unsigned find(const unsigned *parent, unsigned x) {
  for (unsigned p = *(volatile const unsigned *)(parent + x); p != x; p = *(volatile const unsigned *)(parent + x))
    x = p;
  return x;
}

// hook the larger root onto the smaller; when another thread hooked it first, go on with the root it found
__device__ __forceinline__ void unite(unsigned *parent, unsigned a, unsigned b) {
  for (;;) {
    a = find(parent, a), b = find(parent, b);
    if (a == b) return;
    if (a > b) { const unsigned t = a; a = b; b = t; }
    const unsigned old = atomicMin(parent + b, a);
    if (old == b) return;
    b = old;
  }
}

// exclusive prefix of `flag` over the CTA in thread order, and the CTA's total; every thread calls it
__device__ __forceinline__ unsigned cta_scan(bool flag, unsigned *s_warp, unsigned &total) {
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned bal = __ballot_sync(FULL, flag);
  if (lane == 0) s_warp[warp] = __popc(bal);
  __syncthreads();
  unsigned before = 0, all = 0;
  for (unsigned w = 0; w < blockDim.x / 32; w++) {
    const unsigned v = s_warp[w];
    before += w < warp ? v : 0u, all += v;
  }
  __syncthreads();   // s_warp is rewritten by the next call
  total = all;
  return before + __popc(bal & ((1u << lane) - 1u));
}

// one chunk's state, each array m * stride long (ngroups m long); records and groups by their index in the frame
struct Work {
  unsigned long long *sx, *sy, *sw, *sh;
  uint4 *box;
  unsigned *parent, *gid, *cnt, *keep, *ngroups;
};

__global__ void __launch_bounds__(CTA)
k_group_init(const unsigned *__restrict__ counts, unsigned stride, unsigned m, Work w) {
  for (unsigned f = blockIdx.y; f < m; f += gridDim.y) {
    const unsigned c = used(counts, f, stride);
    const unsigned long long o = (unsigned long long)f * stride;
    for (unsigned long long i = blockIdx.x * (unsigned long long)CTA + threadIdx.x; i < c;
         i += (unsigned long long)gridDim.x * CTA) {
      w.parent[o + i] = (unsigned)i;
      w.sx[o + i] = w.sy[o + i] = w.sw[o + i] = w.sh[o + i] = 0;
      w.cnt[o + i] = 0;
    }
  }
}

__global__ void __launch_bounds__(2 * TILE)
k_group_pairs(const struct gs_rect *__restrict__ rects, const unsigned *__restrict__ counts, unsigned stride,
              unsigned m, double eps, Work w) {
  __shared__ uint4 s_a[TILE], s_b[TILE];
  const unsigned a = threadIdx.x % TILE, half = threadIdx.x / TILE;
  for (unsigned f = blockIdx.y; f < m; f += gridDim.y) {
    const unsigned c = used(counts, f, stride);
    const struct gs_rect *fr = rects + (unsigned long long)f * stride;
    unsigned *parent = w.parent + (unsigned long long)f * stride;
    const unsigned long long tiles = (c + (unsigned long long)TILE - 1) / TILE, pairs = tiles * (tiles + 1) / 2;
    for (unsigned long long p = blockIdx.x; p < pairs; p += gridDim.x) {
      // p = tj (tj + 1) / 2 + ti with ti <= tj
      unsigned long long tj = (unsigned long long)((sqrt(8.0 * (double)p + 1.0) - 1.0) / 2.0);
      while (tj * (tj + 1) / 2 > p) tj--;
      while ((tj + 1) * (tj + 2) / 2 <= p) tj++;
      const unsigned long long ti = p - tj * (tj + 1) / 2;
      const unsigned long long i0 = ti * TILE, j0 = tj * TILE;
      __syncthreads();   // the previous pair's tiles are read
      {
        const unsigned long long k = (half ? j0 : i0) + a;
        if (k < c) (half ? s_b : s_a)[a] = load_rect(fr + k);
      }
      __syncthreads();
      const unsigned long long ia = i0 + a;
      if (ia >= c) continue;
      const uint4 ra = s_a[a];
      // the two halves of the CTA take alternate records of tile j; on the diagonal tile only j > i
      for (unsigned b = half; b < TILE && j0 + b < c; b += 2) {
        const unsigned long long jb = j0 + b;
        if (jb > ia && similar(ra, s_b[b], eps)) unite(parent, (unsigned)ia, (unsigned)jb);
      }
    }
  }
}

__global__ void __launch_bounds__(SCAN_CTA)
k_group_roots(const struct gs_rect *__restrict__ rects, const unsigned *__restrict__ counts, unsigned stride,
              unsigned m, Work w) {
  __shared__ unsigned s_warp[SCAN_CTA / 32];
  for (unsigned f = blockIdx.x; f < m; f += gridDim.x) {
    const unsigned c = used(counts, f, stride);
    const unsigned long long o = (unsigned long long)f * stride;
    unsigned *parent = w.parent + o;
    // flatten, and number the roots in index order: a group's number is its smallest record's place among the roots
    unsigned groups = 0;
    for (unsigned i0 = 0; i0 < c; i0 += SCAN_CTA) {
      const unsigned i = i0 + threadIdx.x;
      bool root = false;
      if (i < c) {
        const unsigned r = find(parent, i);
        parent[i] = r;
        root = r == i;
      }
      unsigned total;
      const unsigned before = cta_scan(root, s_warp, total);
      if (root) w.gid[o + i] = groups + before;
      groups += total;
    }
    if (threadIdx.x == 0) w.ngroups[f] = groups;
    __syncthreads();   // every record's parent is its root, and every root has its number
    for (unsigned i = threadIdx.x; i < c; i += SCAN_CTA) {
      const unsigned long long g = o + w.gid[o + parent[i]];
      const uint4 r = load_rect(rects + o + i);
      atomicAdd(w.sx + g, (unsigned long long)r.x);
      atomicAdd(w.sy + g, (unsigned long long)r.y);
      atomicAdd(w.sw + g, (unsigned long long)r.z);
      atomicAdd(w.sh + g, (unsigned long long)r.w);
      atomicAdd(w.cnt + g, 1u);
    }
    __syncthreads();   // the sums are complete
    for (unsigned g = threadIdx.x; g < groups; g += SCAN_CTA) {
      // rule 3: rint((float)S * (1.0f / (float)m)), half to even, clamped to [0, UINT_MAX]
      const float s = __fdiv_rn(1.0f, __uint2float_rn(__ldcg(w.cnt + o + g)));
      const unsigned long long *sums[4] = {w.sx, w.sy, w.sw, w.sh};
      unsigned v[4];
#pragma unroll
      for (unsigned q = 0; q < 4; q++) {
        const float a = rintf(__fmul_rn(__ull2float_rn(__ldcg(sums[q] + o + g)), s));
        v[q] = a >= 4294967296.0f ? UINT_MAX : (unsigned)a;
      }
      w.box[o + g] = make_uint4(v[0], v[1], v[2], v[3]);
    }
    __syncthreads();   // s_warp and the next frame
  }
}

__global__ void __launch_bounds__(CTA)
k_group_filter(unsigned stride, unsigned m, unsigned k, double eps, Work w) {
  __shared__ uint4 s_box[GROUP_TILE];
  __shared__ unsigned s_cnt[GROUP_TILE];
  for (unsigned f = blockIdx.y; f < m; f += gridDim.y) {
    const unsigned groups = w.ngroups[f];
    const unsigned long long o = (unsigned long long)f * stride;
    for (unsigned long long t = blockIdx.x; t * GROUP_TILE < groups; t += gridDim.x) {
      const unsigned long long i = t * GROUP_TILE + threadIdx.x;
      uint4 bi = make_uint4(0, 0, 0, 0);
      unsigned mi = 0;
      if (i < groups) bi = w.box[o + i], mi = w.cnt[o + i];
      bool keep = i < groups && mi > k;
      for (unsigned j0 = 0; j0 < groups; j0 += GROUP_TILE) {
        __syncthreads();   // the previous chunk is read
        if (j0 + threadIdx.x < groups) {
          s_box[threadIdx.x] = w.box[o + j0 + threadIdx.x];
          s_cnt[threadIdx.x] = w.cnt[o + j0 + threadIdx.x];
        }
        __syncthreads();
        if (!keep) continue;
        const unsigned nj = umin(GROUP_TILE, groups - j0);
        for (unsigned jj = 0; jj < nj; jj++) {
          const unsigned mj = s_cnt[jj];
          if (mj > k && j0 + jj != i && contains(s_box[jj], mj, bi, mi, eps)) {
            keep = false;
            break;
          }
        }
      }
      if (i < groups) w.keep[o + i] = keep;
    }
  }
}

__global__ void __launch_bounds__(SCAN_CTA)
k_group_emit(unsigned stride, unsigned m, Work w, struct gs_rect *__restrict__ out, unsigned *__restrict__ weights,
             unsigned *__restrict__ out_counts, unsigned out_stride) {
  __shared__ unsigned s_warp[SCAN_CTA / 32];
  for (unsigned f = blockIdx.x; f < m; f += gridDim.x) {
    const unsigned groups = w.ngroups[f];
    const unsigned long long o = (unsigned long long)f * stride, oo = (unsigned long long)f * out_stride;
    unsigned kept = 0;
    for (unsigned g0 = 0; g0 < groups && kept < out_stride; g0 += SCAN_CTA) {
      const unsigned g = g0 + threadIdx.x;
      const bool keep = g < groups && w.keep[o + g];
      unsigned total;
      const unsigned at = kept + cta_scan(keep, s_warp, total);
      if (keep && at < out_stride) {
        store_rect(out + oo + at, w.box[o + g]);
        if (weights) weights[oo + at] = w.cnt[o + g];
      }
      kept += total;
    }
    if (threadIdx.x == 0) out_counts[f] = umin(kept, out_stride);
  }
}

__global__ void __launch_bounds__(CTA)
k_group_copy(const struct gs_rect *__restrict__ rects, const unsigned *__restrict__ counts, unsigned stride,
             unsigned n, struct gs_rect *__restrict__ out, unsigned *__restrict__ weights,
             unsigned *__restrict__ out_counts, unsigned out_stride) {
  for (unsigned f = blockIdx.y; f < n; f += gridDim.y) {
    const unsigned c = umin(used(counts, f, stride), out_stride);
    const unsigned long long o = (unsigned long long)f * stride, oo = (unsigned long long)f * out_stride;
    for (unsigned long long i = blockIdx.x * (unsigned long long)CTA + threadIdx.x; i < c;
         i += (unsigned long long)gridDim.x * CTA) {
      out[oo + i] = rects[o + i];
      if (weights) weights[oo + i] = 1;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) out_counts[f] = c;
  }
}

// grid x for a kernel whose grid y walks `frames`: up to `items` CTAs per frame, about 16384 CTAs in all
static unsigned grid_x(unsigned long long items, unsigned frames) {
  const unsigned long long y = frames < GRID_MAX ? frames : GRID_MAX, cap = 16384 / y ? 16384 / y : 1;
  return static_cast<unsigned>(items < cap ? (items ? items : 1) : cap);
}

static unsigned long long per_frame(unsigned stride) { return PER_RECORD * stride + 4; }

}  // namespace gsb

using namespace gsb;

extern "C" const char *gs_b200_group_last_error(void) { return t_last_error; }

extern "C" size_t gs_b200_group_rects_work_bytes(unsigned stride, unsigned n) {
  const unsigned __int128 b = (unsigned __int128)per_frame(stride) * n + 16u;
  return b > (unsigned __int128)SIZE_MAX ? SIZE_MAX : static_cast<size_t>(b);
}

extern "C" int gs_b200_group_rects_batch(const struct gs_rect *rects, const unsigned *counts, unsigned stride,
                                         unsigned n, unsigned min_neighbors, double eps, struct gs_rect *out,
                                         unsigned *weights, unsigned *out_counts, unsigned out_stride, void *work,
                                         size_t work_bytes, gs_b200_stream s) {
  if (n == 0) return 0;
  GSK_ASSERT(rects && out && out_counts && work);
  if (!(eps >= 0.0) || isinf(eps)) return invalid("eps is negative, NaN or infinite", __FILE__, __LINE__);
  // the state starts at work's first 16-byte boundary
  const size_t pad = (16u - (reinterpret_cast<uintptr_t>(work) & 15u)) & 15u;
  const unsigned long long one = per_frame(stride);
  if (work_bytes < pad || (work_bytes - pad) / one == 0)
    return invalid("work_bytes below one frame's state", __FILE__, __LINE__);
  const cudaStream_t st = (cudaStream_t)s;
  const unsigned ny = n < GRID_MAX ? n : GRID_MAX;
  if (min_neighbors == 0 || stride == 0 || out_stride == 0) {   // rule 6, and the empty lists
    const unsigned c = stride < out_stride ? stride : out_stride;
    GSK_LAUNCH(k_group_copy, dim3(grid_x((c + CTA - 1ull) / CTA, n), ny), dim3(CTA), st, rects, counts, stride, n, out,
               weights, out_counts, out_stride);
    return 0;
  }
  const unsigned long long fit = (work_bytes - pad) / one, chunk = fit < n ? fit : n;
  uint8_t *base = static_cast<uint8_t *>(work) + pad;
  const unsigned long long tiles = (stride + (unsigned long long)TILE - 1) / TILE;
  for (unsigned long long f0 = 0; f0 < n; f0 += chunk) {
    const unsigned m = static_cast<unsigned>(n - f0 < chunk ? n - f0 : chunk);
    const unsigned my = m < GRID_MAX ? m : GRID_MAX;
    const unsigned long long r = (unsigned long long)m * stride;
    Work w;
    w.sx = reinterpret_cast<unsigned long long *>(base);
    w.sy = w.sx + r, w.sw = w.sy + r, w.sh = w.sw + r;
    w.box = reinterpret_cast<uint4 *>(w.sh + r);
    w.parent = reinterpret_cast<unsigned *>(w.box + r);
    w.gid = w.parent + r, w.cnt = w.gid + r, w.keep = w.cnt + r, w.ngroups = w.keep + r;
    const struct gs_rect *fr = rects + f0 * stride;
    const unsigned *fc = counts ? counts + f0 : nullptr;
    GSK_LAUNCH(k_group_init, dim3(grid_x((stride + CTA - 1ull) / CTA, m), my), dim3(CTA), st, fc, stride, m, w);
    GSK_LAUNCH(k_group_pairs, dim3(grid_x(tiles * (tiles + 1) / 2, m), my), dim3(2 * TILE), st, fr, fc, stride, m, eps,
               w);
    GSK_LAUNCH(k_group_roots, dim3(my), dim3(SCAN_CTA), st, fr, fc, stride, m, w);
    GSK_LAUNCH(k_group_filter, dim3(grid_x((stride + GROUP_TILE - 1ull) / GROUP_TILE, m), my), dim3(CTA), st, stride,
               m, min_neighbors, eps, w);
    GSK_LAUNCH(k_group_emit, dim3(my), dim3(SCAN_CTA), st, stride, m, w, out + f0 * out_stride,
               weights ? weights + f0 * out_stride : nullptr, out_counts + f0, out_stride);
  }
  return 0;
}
