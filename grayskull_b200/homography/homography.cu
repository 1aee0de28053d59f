// homography.cu -- libgrayskull_homography.so: a RANSAC homography from each frame's ORB matches and the template's
// outline in the scene, over frame batches (include/grayskull_homography.h states the rule step for step).
//
// k_find runs one CTA of CTA threads per frame (frames past the grid loop):
//   1. a table of usable records before each of NBLK record blocks, so that a sample's i-th correspondence is found
//      by a binary search and a short scan; its total is m
//   2. the usable correspondences staged in shared memory, CHUNK or more at a time (all of them once when they fit)
//   3. per block of CTA hypotheses: each thread draws, checks and solves one; then each warp scores the block's
//      hypotheses against the staged correspondences with ballots and popc; a CTA max over (count, -k) keys keeps the
//      best so far and its H
//   4. the refit: centroid and exact __int128 sums over the best hypothesis's inliers (per-thread partials, then warp
//      and CTA reductions: integer sums do not depend on the order), one solve, one count
//   5. H, the count and the inlier records in record order (an ordered CTA compaction)
// k_quads runs one thread per frame.
// The library is compiled with -fmad=false, and every double operation of the rule is an explicit __d*_rn.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <utility>

#include "../../include/grayskull_homography.h"

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

constexpr unsigned CTA = 256;
constexpr unsigned WARPS = CTA / 32;
constexpr unsigned NBLK = 4 * CTA;         // record blocks of the usable-record table: four per thread
constexpr unsigned CHUNK = 1024;           // a staged chunk closes at the first CTA-record step that reaches CHUNK
constexpr unsigned SLOTS = CHUNK + CTA;
constexpr unsigned MAX_GRID = 1u << 20;
constexpr unsigned COORD = 1u << 20;
constexpr unsigned NSUMS = 22;
constexpr unsigned FULL = 0xffffffffu;
constexpr unsigned long long GOLDEN = 0x9E3779B97F4A7C15ull;

__device__ __forceinline__ unsigned umin(unsigned a, unsigned b) { return a < b ? a : b; }

// 2^e, exact, for |e| < 1000
__device__ __forceinline__ double pow2(int e) { return __longlong_as_double((long long)(1023 + e) << 52); }

// an __int128 to the nearest double, ties to even, as Python's float(int): the top 64 bits with the bits below them
// folded into a sticky bit 0 (far below the 53-bit rounding point), converted once, scaled exactly
__device__ double i128_to_double(__int128 v) {
  const bool neg = v < 0;
  const unsigned __int128 u = neg ? (unsigned __int128)0 - (unsigned __int128)v : (unsigned __int128)v;
  const unsigned long long hi = (unsigned long long)(u >> 64), lo = (unsigned long long)u;
  double d;
  if (hi == 0) {
    d = __ull2double_rn(lo);
  } else {
    const int sh = 64 - __clzll((long long)hi);   // 1..64: bits of u below its top 64
    const unsigned long long top = (unsigned long long)(u >> sh), dropped = sh == 64 ? lo : lo & ((1ull << sh) - 1);
    d = __dmul_rn(__ull2double_rn(top | (dropped ? 1ull : 0ull)), pow2(sh));
  }
  return neg ? -d : d;
}

// splitmix64's finaliser
__device__ __forceinline__ unsigned long long mix(unsigned long long z) {
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// one frame's inputs: its keypoint lists, its records, the used lengths
struct Frame {
  const struct gs_keypoint *k1, *k2;
  const struct gs_match *mt;
  unsigned c1, c2, c;
};

// rule 1: record i as a correspondence (x, y, X, Y), or false
__device__ __forceinline__ bool corr(const Frame &F, unsigned long long i, int4 &p) {
  const struct gs_match *r = F.mt + i;
  const unsigned i1 = r->idx1, i2 = r->idx2;
  if (i1 >= F.c1 || i2 >= F.c2) return false;
  const unsigned x = F.k1[i1].pt.x, y = F.k1[i1].pt.y, X = F.k2[i2].pt.x, Y = F.k2[i2].pt.y;
  if (x >= COORD || y >= COORD || X >= COORD || Y >= COORD) return false;
  p = make_int4((int)x, (int)y, (int)X, (int)Y);
  return true;
}

// rule 5's predicate
__device__ __forceinline__ bool inlier(const double *H, int4 p, double t2) {
  const double x = (double)p.x, y = (double)p.y, X = (double)p.z, Y = (double)p.w;
  const double u = __dadd_rn(__dadd_rn(__dmul_rn(H[0], x), __dmul_rn(H[1], y)), H[2]);
  const double v = __dadd_rn(__dadd_rn(__dmul_rn(H[3], x), __dmul_rn(H[4], y)), H[5]);
  const double w = __dadd_rn(__dadd_rn(__dmul_rn(H[6], x), __dmul_rn(H[7], y)), H[8]);
  const double du = __dsub_rn(u, __dmul_rn(X, w)), dv = __dsub_rn(v, __dmul_rn(Y, w));
  return w > 0.0 && __dadd_rn(__dmul_rn(du, du), __dmul_rn(dv, dv)) <= __dmul_rn(t2, __dmul_rn(w, w));
}

// the header's 22 integer sums of one centred correspondence (a, b) -> (A, B), added to s
__device__ __forceinline__ void add_terms(__int128 *s, long long a, long long b, long long A, long long B) {
  const long long aa = a * a, ab = a * b, bb = b * b, R = A * A + B * B;
  s[0] += a, s[1] += b, s[2] += A, s[3] += B, s[4] += aa, s[5] += ab, s[6] += bb;
  s[7] += a * A, s[8] += b * A, s[9] += a * B, s[10] += b * B;
  s[11] += aa * A, s[12] += ab * A, s[13] += bb * A, s[14] += aa * B, s[15] += ab * B, s[16] += bb * B;
  s[17] += a * R, s[18] += b * R;
  s[19] += (__int128)aa * R, s[20] += (__int128)ab * R, s[21] += (__int128)bb * R;
}

__device__ __forceinline__ int bit_length(unsigned long long v) { return 64 - __clzll((long long)v); }

// rule 4 from the sums: m correspondences centred on (cx, cy) -> (CX, CY), scaled by 2^-kt and 2^-ks.  H gets the
// result; false when the solve is invalid.
__device__ bool solve(const __int128 *s, long long m, long long cx, long long cy, long long CX, long long CY, int kt,
                      int ks, double *H) {
  const __int128 z = 0, mm = m;
  // the upper triangle of the integer normal matrix and its right-hand side, row by row
  const __int128 S[8][8] = {
      {s[4], s[5], s[0], z, z, z, -s[11], -s[12]},
      {z, s[6], s[1], z, z, z, -s[12], -s[13]},
      {z, z, mm, z, z, z, -s[7], -s[8]},
      {z, z, z, s[4], s[5], s[0], -s[14], -s[15]},
      {z, z, z, z, s[6], s[1], -s[15], -s[16]},
      {z, z, z, z, z, mm, -s[9], -s[10]},
      {z, z, z, z, z, z, s[19], s[20]},
      {z, z, z, z, z, z, z, s[21]}};
  const __int128 V[8] = {s[7], s[8], s[2], s[9], s[10], s[3], -s[17], -s[18]};
  const int E[8] = {kt, kt, 0, kt, kt, 0, kt + ks, kt + ks};
  double A[8][8], r[8];
#pragma unroll
  for (int p = 0; p < 8; p++) {
#pragma unroll
    for (int q = p; q < 8; q++) A[q][p] = __dmul_rn(i128_to_double(S[p][q]), pow2(-(E[p] + E[q])));
    r[p] = __dmul_rn(i128_to_double(V[p]), pow2(-(E[p] + ks)));
  }
  // Cholesky, in place in the lower triangle: column j, its pivot, then the rows below it
#pragma unroll
  for (int j = 0; j < 8; j++) {
    double d = A[j][j];
#pragma unroll
    for (int k = 0; k < j; k++) d = __dsub_rn(d, __dmul_rn(A[j][k], A[j][k]));
    if (!(d > 0.0 && d < INFINITY)) return false;
    A[j][j] = __dsqrt_rn(d);
#pragma unroll
    for (int i = j + 1; i < 8; i++) {
      double t = A[i][j];
#pragma unroll
      for (int k = 0; k < j; k++) t = __dsub_rn(t, __dmul_rn(A[i][k], A[j][k]));
      A[i][j] = __ddiv_rn(t, A[j][j]);
    }
  }
  // L y = r, then L^T h = y
#pragma unroll
  for (int i = 0; i < 8; i++) {
    double t = r[i];
#pragma unroll
    for (int k = 0; k < i; k++) t = __dsub_rn(t, __dmul_rn(A[i][k], r[k]));
    r[i] = __ddiv_rn(t, A[i][i]);
  }
#pragma unroll
  for (int i = 7; i >= 0; i--) {
    double t = r[i];
#pragma unroll
    for (int k = i + 1; k < 8; k++) t = __dsub_rn(t, __dmul_rn(A[k][i], r[k]));
    r[i] = __ddiv_rn(t, A[i][i]);
  }
  // un-normalise: G = Hn T, then H = S^-1 G, then H / H[8]
  const double st = pow2(-kt), up = pow2(ks), fx = (double)cx, fy = (double)cy;
  double G[9];
#pragma unroll
  for (int row = 0; row < 3; row++) {
    const double p = r[3 * row], q = r[3 * row + 1], c = row < 2 ? r[3 * row + 2] : 1.0;
    const double P = __dmul_rn(p, st), Q = __dmul_rn(q, st);
    G[3 * row] = P, G[3 * row + 1] = Q;
    G[3 * row + 2] = __dsub_rn(c, __dadd_rn(__dmul_rn(P, fx), __dmul_rn(Q, fy)));
  }
#pragma unroll
  for (int j = 0; j < 3; j++) {
    H[j] = __dadd_rn(__dmul_rn(G[j], up), __dmul_rn((double)CX, G[6 + j]));
    H[3 + j] = __dadd_rn(__dmul_rn(G[3 + j], up), __dmul_rn((double)CY, G[6 + j]));
    H[6 + j] = G[6 + j];
  }
  const double d = H[8];
  if (d == 0.0 || !(fabs(d) < INFINITY)) return false;
  bool ok = true;
#pragma unroll
  for (int i = 0; i < 9; i++) {
    H[i] = __ddiv_rn(H[i], d);
    ok = ok && fabs(H[i]) < INFINITY;
  }
  return ok;
}

// exclusive prefix of `v` over the CTA in thread order, and the CTA's total; every thread calls it
__device__ __forceinline__ unsigned cta_scan(unsigned v, unsigned *s_warp, unsigned &total) {
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned inc = v;
#pragma unroll
  for (unsigned o = 1; o < 32; o <<= 1) {
    const unsigned t = __shfl_up_sync(FULL, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  unsigned before = 0, all = 0;
  for (unsigned w = 0; w < WARPS; w++) {
    const unsigned x = s_warp[w];
    before += w < warp ? x : 0u, all += x;
  }
  __syncthreads();   // s_warp is rewritten by the next call
  total = all;
  return before + inc - v;
}

// the CTA's largest v; every thread calls it
__device__ __forceinline__ unsigned long long cta_max(unsigned long long v, unsigned long long *s_u64) {
#pragma unroll
  for (unsigned o = 16; o; o >>= 1) {
    const unsigned long long t = __shfl_xor_sync(FULL, v, o);
    v = t > v ? t : v;
  }
  if ((threadIdx.x & 31) == 0) s_u64[threadIdx.x >> 5] = v;
  __syncthreads();
  for (unsigned w = 0; w < WARPS; w++) v = s_u64[w] > v ? s_u64[w] : v;
  __syncthreads();
  return v;
}

// the CTA's sum of v; every thread calls it
__device__ __forceinline__ long long cta_sum(long long v, unsigned long long *s_u64) {
#pragma unroll
  for (unsigned o = 16; o; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
  if ((threadIdx.x & 31) == 0) s_u64[threadIdx.x >> 5] = (unsigned long long)v;
  __syncthreads();
  long long all = 0;
  for (unsigned w = 0; w < WARPS; w++) all += (long long)s_u64[w];
  __syncthreads();
  return all;
}

// the usable records from record r on, in record order, into s_c until CHUNK or more are staged or the records end;
// the count, and in `next` the record to go on from
__device__ unsigned stage(const Frame &F, unsigned long long r, unsigned long long &next, int4 *s_c, unsigned *s_warp) {
  unsigned filled = 0;
  for (; filled < CHUNK && r < F.c; r += CTA) {
    int4 p = make_int4(0, 0, 0, 0);
    const bool ok = r + threadIdx.x < F.c && corr(F, r + threadIdx.x, p);
    unsigned total;
    const unsigned at = filled + cta_scan(ok, s_warp, total);
    if (ok) s_c[at] = p;
    filled += total;
  }
  next = r;
  __syncthreads();
  return filled;
}

// the t-th usable correspondence (t < m): the last table block that starts at or before it, then a scan
__device__ int4 lookup(const Frame &F, const unsigned *s_pre, unsigned long long bs, unsigned t) {
  unsigned lo = 0, hi = NBLK - 1;
  while (lo < hi) {
    const unsigned mid = (lo + hi + 1) / 2;
    if (s_pre[mid] <= t) lo = mid;
    else hi = mid - 1;
  }
  unsigned left = t - s_pre[lo];
  int4 p = make_int4(0, 0, 0, 0);
  for (unsigned long long r = lo * bs;; r++)
    if (corr(F, r, p) && left-- == 0) return p;
}

__device__ __forceinline__ long long orient(int4 a, int4 b, int4 c, bool scene) {
  const long long ax = scene ? a.z : a.x, ay = scene ? a.w : a.y;
  return ((scene ? b.z : b.x) - ax) * ((scene ? c.w : c.y) - ay) - ((scene ? b.w : b.y) - ay) * ((scene ? c.z : c.x) - ax);
}

// rules 2-4 for hypothesis k of frame f: H, or false
__device__ bool hypothesis(const Frame &F, const unsigned *s_pre, unsigned long long bs, unsigned m,
                           unsigned long long seed, unsigned long long f, unsigned k, double *H) {
  unsigned idx[4];
#pragma unroll
  for (unsigned j = 0; j < 4; j++) {
    const unsigned J = m - 4 + j;
    const unsigned long long z = mix(seed + GOLDEN * ((f << 18) | ((unsigned long long)k << 2) | j));
    const unsigned t = (unsigned)(((z >> 32) * ((unsigned long long)J + 1)) >> 32);
    bool taken = false;
#pragma unroll
    for (unsigned q = 0; q < j; q++) taken = taken || idx[q] == t;
    idx[j] = taken ? J : t;
  }
#pragma unroll
  for (unsigned a = 0; a < 3; a++)
#pragma unroll
    for (unsigned b = 0; b < 3 - a; b++)
      if (idx[b] > idx[b + 1]) { const unsigned x = idx[b]; idx[b] = idx[b + 1]; idx[b + 1] = x; }
  int4 p[4];
#pragma unroll
  for (unsigned j = 0; j < 4; j++) p[j] = lookup(F, s_pre, bs, idx[j]);
  const unsigned tri[4][3] = {{0, 1, 2}, {0, 1, 3}, {0, 2, 3}, {1, 2, 3}};
#pragma unroll
  for (unsigned q = 0; q < 4; q++) {
    const long long ot = orient(p[tri[q][0]], p[tri[q][1]], p[tri[q][2]], false);
    const long long os = orient(p[tri[q][0]], p[tri[q][1]], p[tri[q][2]], true);
    if (ot == 0 || os == 0 || (ot > 0) != (os > 0)) return false;
  }
  long long sx = 0, sy = 0, sX = 0, sY = 0;
#pragma unroll
  for (unsigned j = 0; j < 4; j++) sx += p[j].x, sy += p[j].y, sX += p[j].z, sY += p[j].w;
  const long long cx = sx / 4, cy = sy / 4, CX = sX / 4, CY = sY / 4;
  unsigned long long mt = 0, ms = 0;
  __int128 s[NSUMS];
#pragma unroll
  for (unsigned q = 0; q < NSUMS; q++) s[q] = 0;
#pragma unroll
  for (unsigned j = 0; j < 4; j++) {
    const long long a = p[j].x - cx, b = p[j].y - cy, A = p[j].z - CX, B = p[j].w - CY;
    mt = max(mt, (unsigned long long)max(llabs(a), llabs(b)));
    ms = max(ms, (unsigned long long)max(llabs(A), llabs(B)));
    add_terms(s, a, b, A, B);
  }
  return solve(s, 4, cx, cy, CX, CY, bit_length(mt), bit_length(ms), H);
}

__global__ void __launch_bounds__(CTA, 1)
k_find(const struct gs_keypoint *__restrict__ kps1, const unsigned *__restrict__ n1, unsigned stride1,
       const struct gs_keypoint *__restrict__ kps2, const unsigned *__restrict__ n2, unsigned stride2,
       const struct gs_match *__restrict__ matches, const unsigned *__restrict__ mcounts, unsigned mstride, unsigned n,
       unsigned hyps, unsigned long long seed, double t2, double *__restrict__ Hout, unsigned *__restrict__ inliers,
       struct gs_match *__restrict__ inlier_matches) {
  __shared__ unsigned s_pre[NBLK];
  __shared__ int4 s_c[SLOTS];
  __shared__ double s_H[CTA][9];
  __shared__ double s_best[9];
  __shared__ unsigned s_cnt[CTA];
  __shared__ unsigned s_warp[WARPS];
  __shared__ unsigned long long s_u64[WARPS];
  __shared__ __int128 s_red[WARPS][NSUMS];
  const unsigned tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (unsigned long long f = blockIdx.x; f < n; f += gridDim.x) {
    Frame F;
    F.k1 = kps1 + f * stride1, F.k2 = kps2 + f * stride2, F.mt = matches + f * mstride;
    F.c1 = umin(n1[f], stride1), F.c2 = umin(n2[f], stride2), F.c = umin(mcounts[f], mstride);
    double *Hf = Hout + f * 9;
    // 1. usable records before each block of bs records
    const unsigned long long bs = F.c > NBLK ? (F.c + NBLK - 1ull) / NBLK : 1ull;
    unsigned own[4], mine = 0;
#pragma unroll
    for (unsigned q = 0; q < 4; q++) {
      own[q] = 0;
      const unsigned long long r0 = (4ull * tid + q) * bs;
      for (unsigned long long r = r0; r < r0 + bs && r < F.c; r++) {
        int4 p;
        own[q] += corr(F, r, p);
      }
      mine += own[q];
    }
    unsigned m;
    unsigned at = cta_scan(mine, s_warp, m);
#pragma unroll
    for (unsigned q = 0; q < 4; q++) s_pre[4 * tid + q] = at, at += own[q];
    if (m < 4) {
      if (tid < 9) Hf[tid] = 0.0;
      if (tid == 0) inliers[f] = 0;
      continue;   // s_pre is rewritten after the next frame's first barrier
    }
    // 2. the first chunk; when it holds every usable record it stays for all hypotheses
    unsigned long long next;
    unsigned nc = stage(F, 0, next, s_c, s_warp);
    const bool all_in = next >= F.c;
    // 3. the hypotheses, CTA at a time
    unsigned long long best = 0;   // (count << 32) | (2^32 - 1 - k) of the best valid hypothesis; 0: none yet
    for (unsigned k0 = 0; k0 < hyps; k0 += CTA) {
      const unsigned k = k0 + tid;
      const bool ok = k < hyps && hypothesis(F, s_pre, bs, m, seed, f, k, s_H[tid]);
      if (!ok) s_H[tid][8] = __longlong_as_double(0x7ff8000000000000ll);   // NaN: the scoring skips it
      s_cnt[tid] = 0;
      __syncthreads();
      const unsigned njobs = umin(CTA, hyps - k0);
      for (unsigned long long r = 0;;) {
        if (!all_in) nc = stage(F, r, r, s_c, s_warp);
        for (unsigned j = warp; j < njobs; j += WARPS) {
          double H[9];
#pragma unroll
          for (unsigned q = 0; q < 9; q++) H[q] = s_H[j][q];
          if (!(H[8] == H[8])) continue;   // invalid
          unsigned cnt = 0;
          for (unsigned i = lane; i - lane < nc; i += 32)
            cnt += __popc(__ballot_sync(FULL, i < nc && inlier(H, s_c[i], t2)));
          if (lane == 0) s_cnt[j] += cnt;
        }
        __syncthreads();   // s_cnt complete for this chunk, s_c free
        if (all_in || r >= F.c) break;
      }
      // an invalid hypothesis has key 0 and never wins
      const unsigned long long key = ok ? ((unsigned long long)s_cnt[tid] << 32) | (FULL - k) : 0ull;
      const unsigned long long top = cta_max(key, s_u64);
      if (top > best) {
        if (key == top)
          for (unsigned q = 0; q < 9; q++) s_best[q] = s_H[tid][q];
        best = top;
      }
      __syncthreads();   // s_best written; s_H free for the next block
    }
    if (best == 0) {   // no valid hypothesis
      if (tid < 9) Hf[tid] = 0.0;
      if (tid == 0) inliers[f] = 0;
      continue;
    }
    double Hb[9], Hr[9];
#pragma unroll
    for (unsigned q = 0; q < 9; q++) Hb[q] = s_best[q];
    const unsigned cb = (unsigned)(best >> 32);
    // 4. the refit on the best hypothesis's inliers: centroid, then the exact sums, then one solve and one count
    bool use_refit = false;
    unsigned count = cb;
    if (cb >= 4) {
      long long px = 0, py = 0, pX = 0, pY = 0;
      for (unsigned long long r = tid; r < F.c; r += CTA) {
        int4 p;
        if (corr(F, r, p) && inlier(Hb, p, t2)) px += p.x, py += p.y, pX += p.z, pY += p.w;
      }
      const long long cx = cta_sum(px, s_u64) / cb, cy = cta_sum(py, s_u64) / cb;
      const long long CX = cta_sum(pX, s_u64) / cb, CY = cta_sum(pY, s_u64) / cb;
      __int128 s[NSUMS];
#pragma unroll
      for (unsigned q = 0; q < NSUMS; q++) s[q] = 0;
      unsigned long long mt = 0, ms = 0;
      for (unsigned long long r = tid; r < F.c; r += CTA) {
        int4 p;
        if (!corr(F, r, p) || !inlier(Hb, p, t2)) continue;
        const long long a = p.x - cx, b = p.y - cy, A = p.z - CX, B = p.w - CY;
        mt = max(mt, (unsigned long long)max(llabs(a), llabs(b)));
        ms = max(ms, (unsigned long long)max(llabs(A), llabs(B)));
        add_terms(s, a, b, A, B);
      }
      mt = cta_max(mt, s_u64), ms = cta_max(ms, s_u64);
#pragma unroll
      for (unsigned q = 0; q < NSUMS; q++) {
        unsigned long long lo = (unsigned long long)s[q], hi = (unsigned long long)(s[q] >> 64);
#pragma unroll
        for (unsigned o = 16; o; o >>= 1) {
          const unsigned long long olo = __shfl_xor_sync(FULL, lo, o), ohi = __shfl_xor_sync(FULL, hi, o);
          const unsigned long long nlo = lo + olo;
          hi = hi + ohi + (nlo < lo ? 1ull : 0ull), lo = nlo;
        }
        if (lane == 0) s_red[warp][q] = (__int128)(((unsigned __int128)hi << 64) | lo);
      }
      __syncthreads();
      if (tid == 0) {
#pragma unroll
        for (unsigned q = 0; q < NSUMS; q++) {
          s[q] = 0;
          for (unsigned w = 0; w < WARPS; w++) s[q] += s_red[w][q];
        }
        const bool valid = solve(s, cb, cx, cy, CX, CY, bit_length(mt), bit_length(ms), Hr);
        for (unsigned q = 0; q < 9; q++) s_best[q] = valid ? Hr[q] : __longlong_as_double(0x7ff8000000000000ll);
      }
      __syncthreads();
#pragma unroll
      for (unsigned q = 0; q < 9; q++) Hr[q] = s_best[q];
      if (Hr[8] == Hr[8]) {
        unsigned cr = 0;
        for (unsigned long long r = tid; r < F.c; r += CTA) {
          int4 p;
          cr += corr(F, r, p) && inlier(Hr, p, t2);
        }
        cr = (unsigned)cta_sum(cr, s_u64);
        if (cr >= cb) use_refit = true, count = cr;
      }
    }
    const double *Hf_ = use_refit ? Hr : Hb;
    // 5. the outputs
    if (tid < 9) Hf[tid] = Hf_[tid];
    if (tid == 0) inliers[f] = count;
    if (inlier_matches) {
      struct gs_match *out = inlier_matches + f * mstride;
      unsigned done = 0;
      for (unsigned long long r = 0; r < F.c && done < count; r += CTA) {
        int4 p;
        const bool in = r + tid < F.c && corr(F, r + tid, p) && inlier(Hf_, p, t2);
        unsigned total;
        const unsigned pos = done + cta_scan(in, s_warp, total);
        if (in) out[pos] = F.mt[r + tid];
        done += total;
      }
    }
    __syncthreads();   // s_best and the tables are read; the next frame rewrites them
  }
}

// rule 7, one thread per frame
__global__ void __launch_bounds__(CTA)
k_quads(const double *__restrict__ H, const unsigned *__restrict__ inliers, unsigned n, unsigned min_inliers,
        unsigned tw, unsigned th, unsigned sw, unsigned sh, struct gs_point *__restrict__ corners,
        uint8_t *__restrict__ found) {
  for (unsigned long long f = blockIdx.x * (unsigned long long)CTA + threadIdx.x; f < n;
       f += (unsigned long long)gridDim.x * CTA) {
    double h[9];
    bool nonzero = false;
#pragma unroll
    for (unsigned q = 0; q < 9; q++) h[q] = H[f * 9 + q], nonzero = nonzero || h[q] != 0.0;
    bool ok = nonzero && inliers[f] >= min_inliers;
    const double xs[4] = {0.0, (double)(tw - 1), (double)(tw - 1), 0.0};
    const double ys[4] = {0.0, 0.0, (double)(th - 1), (double)(th - 1)};
    unsigned out[8];
#pragma unroll
    for (unsigned q = 0; q < 4; q++) {
      const double u = __dadd_rn(__dadd_rn(__dmul_rn(h[0], xs[q]), __dmul_rn(h[1], ys[q])), h[2]);
      const double v = __dadd_rn(__dadd_rn(__dmul_rn(h[3], xs[q]), __dmul_rn(h[4], ys[q])), h[5]);
      const double w = __dadd_rn(__dadd_rn(__dmul_rn(h[6], xs[q]), __dmul_rn(h[7], ys[q])), h[8]);
      const double px = rint(__ddiv_rn(u, w)), py = rint(__ddiv_rn(v, w));
      ok = ok && w > 0.0 && px == px && py == py;
      out[2 * q] = px > 0.0 ? (px < (double)(sw - 1) ? (unsigned)px : sw - 1) : 0u;
      out[2 * q + 1] = py > 0.0 ? (py < (double)(sh - 1) ? (unsigned)py : sh - 1) : 0u;
    }
#pragma unroll
    for (unsigned q = 0; q < 4; q++) {
      corners[f * 4 + q].x = ok ? out[2 * q] : 0u;
      corners[f * 4 + q].y = ok ? out[2 * q + 1] : 0u;
    }
    found[f] = ok;
  }
}

}  // namespace gsb

using namespace gsb;

extern "C" const char *gs_b200_homography_last_error(void) { return t_last_error; }

extern "C" int gs_b200_find_homography_batch(const struct gs_keypoint *kps1, const unsigned *n1, unsigned stride1,
                                             const struct gs_keypoint *kps2, const unsigned *n2, unsigned stride2,
                                             const struct gs_match *matches, const unsigned *mcounts, unsigned mstride,
                                             unsigned n, unsigned hypotheses, unsigned long long seed,
                                             double threshold, double *H, unsigned *inliers,
                                             struct gs_match *inlier_matches, gs_b200_stream s) {
  if (n == 0) return 0;
  GSK_ASSERT(kps1 && n1 && kps2 && n2 && matches && mcounts && H && inliers);
  if (!(threshold > 0.0) || isinf(threshold)) return invalid("threshold is not finite and > 0", __FILE__, __LINE__);
  if (hypotheses == 0 || hypotheses > 65536u) return invalid("hypotheses outside 1..65536", __FILE__, __LINE__);
  const double t2 = threshold * threshold;
  GSK_LAUNCH(k_find, dim3(n < MAX_GRID ? n : MAX_GRID), dim3(CTA), (cudaStream_t)s, kps1, n1, stride1, kps2, n2,
             stride2, matches, mcounts, mstride, n, hypotheses, seed, t2, H, inliers, inlier_matches);
  return 0;
}

extern "C" int gs_b200_homography_quads_batch(const double *H, const unsigned *inliers, unsigned n,
                                              unsigned min_inliers, unsigned tw, unsigned th, unsigned sw, unsigned sh,
                                              struct gs_point *corners, uint8_t *found, gs_b200_stream s) {
  if (n == 0) return 0;
  GSK_ASSERT(H && inliers && corners && found);
  if (min_inliers < 4) return invalid("min_inliers below 4", __FILE__, __LINE__);
  if (tw == 0 || th == 0 || sw == 0 || sh == 0) return invalid("an empty template or scene", __FILE__, __LINE__);
  const unsigned long long blocks = (n + CTA - 1ull) / CTA;
  GSK_LAUNCH(k_quads, dim3(blocks < MAX_GRID ? (unsigned)blocks : MAX_GRID), dim3(CTA), (cudaStream_t)s, H, inliers,
             n, min_inliers, tw, th, sw, sh, corners, found);
  return 0;
}
