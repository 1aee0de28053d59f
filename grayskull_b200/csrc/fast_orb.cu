// fast_orb.cu -- gs_fast, gs_compute_orientation, gs_brief_descriptor, gs_orb_extract
// (reference grayskull.h:482-669).
//
// gs_fast      pass 1  k_fast_tiled2 : FAST-9 score map, interior pixels only, and the 3x3 strict-greater
//                                     NMS bits of each row (smem tile, compass pre-test, candidate
//                                     compaction).  16-bit brighter / darker ring masks; "run of >= 9"
//                                     is the rotate-AND test; the unsigned-wrap quirk of reference :498
//                                     (p < t => every non-brighter sample counts as darker) is reproduced.
//                                     Foreign-sized score maps, force_generic and thresholds above 255
//                                     take the per-pixel k_fast_score and then k_nms_mask instead.
//              pass 2  k_row_scan -> k_nms_emit_masks : the NMS over the caller's score map (including
//                                     the ring cells pass 1 never writes, exactly like reference
//                                     :517-524) ends in a SCAN-based compaction, because the reference
//                                     emits keypoints in raster order and stops at nkps (:530).
// gs_orb_extract       k_orb_select : one CTA per frame: stable descending counting sort on the
//                                     8-bit response (== the reference's bubble sort, :639-649),
//                                     15-px margin filter and cap, all order-preserving.
//                      k_orb_describe: one warp per keypoint: the r=15 disc moments in int32
//                                     (exact, lanes = dx), atan2f, sinf, and BRIEF-256 where each
//                                     ballot yields one descriptor word.
// The reference calls libm atan2f / sinf (grayskull.h:100-101); trig mode 0 evaluates glibc
// 2.39's algorithms with IEEE-exact device arithmetic (see dev_sinf / dev_atan2f), so angles and
// descriptors are bit-identical to the reference on the same box.
#include <math.h>
#include <string.h>

#include <mutex>

#include "common.cuh"
#include "scan.cuh"

namespace gsb {

static int g_trig_mode = 0;

// read with one coalesced 128-byte load per 32 pairs (a __constant__ table indexed per lane would
// serialise into 32 constant-cache accesses)
__device__ const uint32_t c_brief[256] = {
#include "brief_pattern.inc"
};

// the same offsets as floats (x1, y1, x2, y2): k_orb_brief converts nothing on the conversion pipe (four I2F per lane and
// pattern word ran at 16 lanes/clk/SM next to the four float->int truncations).  Filled once per device by
// brief_table_init.
__device__ float4 c_brieff[256];
static const uint32_t h_brief[256] = {
#include "brief_pattern.inc"
};
// once per device, by upload(): the copy has landed before the first k_orb_brief is enqueued on any stream, so no
// stream can see a half-filled table.  The first ORB call on a device must not be captured into a graph.
static int brief_table_init(cudaStream_t user) {
  static std::mutex mu;
  static bool filled[64];
  int dev = 0;
  GSB_CHECK(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(mu);
  if (filled[dev & 63]) return 0;
  if (capturing(user)) return record_error(cudaErrorStreamCaptureUnsupported, __FILE__, __LINE__);
  float4 t[256];
  for (int i = 0; i < 256; i++) {
    const uint32_t pk = h_brief[i];
    t[i] = make_float4((float)(int)(int8_t)(pk & 0xFF), (float)(int)(int8_t)((pk >> 8) & 0xFF),
                       (float)(int)(int8_t)((pk >> 16) & 0xFF), (float)(int)(int8_t)(pk >> 24));
  }
  void *sym = nullptr;
  GSB_CHECK(cudaGetSymbolAddress(&sym, c_brieff));
  if (int rc = upload(sym, t, sizeof(t), __FILE__, __LINE__)) return rc;
  filled[dev & 63] = true;
  return 0;
}

// ---------------------------------------------------------------------------------------------
// glibc 2.39 sinf (sysdeps/ieee754/flt-32/s_sinf.c, sincosf.h; double evaluation) and atan2f /
// atanf (e_atan2f.c, s_atanf.c; float evaluation), restated with explicitly rounded ops.
// tools/validate_trig.c checks the same restatement against libm exhaustively on the CPU.
// Provenance: the polynomial coefficients, reduction constants and the order of operations follow the GNU C Library
// (glibc 2.39, LGPL-2.1-or-later; sinf/sincosf: Copyright (C) the FSF, contributed by Arm; atanf / atan2f: the
// fdlibm-derived float routines, Copyright (C) 1993 Sun Microsystems, "permission to use, copy, modify, and distribute
// this software is freely granted, provided that this notice is preserved").  They are third-party numerics restated
// because bit-exactness with the reference's libm calls leaves no freedom, not reference (grayskull) code.
// ---------------------------------------------------------------------------------------------
__device__ float dev_sinf(float y) {
  const double HPI_INV = 0x1.45F306DC9C883p+23, HPI = 0x1.921FB54442D18p0;
  const double C0 = 0x1p0, C1 = -0x1.ffffffd0c621cp-2, C2 = 0x1.55553e1068f19p-5,
               C3 = -0x1.6c087e89a359dp-10, C4 = 0x1.99343027bf8c3p-16;
  const double S1 = -0x1.555545995a603p-3, S2 = 0x1.1107605230bc4p-7, S3 = -0x1.994eb3774cf24p-13;
  double x = (double)y, x2;
  int n = 0;
  bool negc = false;
  const uint32_t top = (__float_as_uint(y) >> 20) & 0x7ffu;
  if (top < 0x3f4u) {             // |y| < pi/4
    if (top < 0x398u) return y;   // |y| < 2^-12
    x2 = __dmul_rn(x, x);
  } else if (top < 0x42fu) {      // |y| < 120
    const double r = __dmul_rn(x, HPI_INV);
    n = (__double2int_rz(r) + 0x800000) >> 24;
    const double xr = __fma_rn(-(double)n, HPI, x);
    x2 = __dmul_rn(xr, xr);
    x = ((n & 3) == 1 || (n & 3) == 2) ? -xr : xr;
    negc = (n & 2) != 0;
  } else {
    return sinf(y);  // outside the hot path's domain
  }
  if ((n & 1) == 0) {
    const double x3 = __dmul_rn(x, x2), s1 = __fma_rn(x2, S3, S2), x7 = __dmul_rn(x3, x2);
    const double s = __fma_rn(x3, S1, x);
    return __double2float_rn(__fma_rn(x7, s1, s));
  }
  const double sg = negc ? -1.0 : 1.0;
  const double x4 = __dmul_rn(x2, x2), c2 = __fma_rn(x2, sg * C4, sg * C3), c1 = __fma_rn(x2, sg * C1, sg * C0);
  const double x6 = __dmul_rn(x4, x2), c = __fma_rn(x4, sg * C2, c1);
  return __double2float_rn(__fma_rn(x6, c2, c));
}

__device__ float dev_atanf(float x) {
  const float atanhi[4] = {4.6364760399e-01f, 7.8539812565e-01f, 9.8279368877e-01f, 1.5707962513e+00f};
  const float atanlo[4] = {5.0121582440e-09f, 3.7748947079e-08f, 3.4473217170e-08f, 7.5497894159e-08f};
  const float aT[11] = {3.3333334327e-01f,  -2.0000000298e-01f, 1.4285714924e-01f, -1.1111110449e-01f,
                        9.0908870101e-02f,  -7.6918758452e-02f, 6.6610731184e-02f, -5.8335702866e-02f,
                        4.9768779427e-02f,  -3.6531571299e-02f, 1.6285819933e-02f};
  const int hx = (int)__float_as_uint(x), ix = hx & 0x7fffffff;
  int id;
  if (ix >= 0x4c000000) {
    if (ix > 0x7f800000) return __fadd_rn(x, x);
    return hx > 0 ? __fadd_rn(atanhi[3], atanlo[3]) : __fsub_rn(-atanhi[3], atanlo[3]);
  }
  if (ix < 0x3ee00000) {
    if (ix < 0x31000000) return x;
    id = -1;
  } else {
    x = fabsf(x);
    if (ix < 0x3f980000) {
      if (ix < 0x3f300000) id = 0, x = __fdiv_rn(__fsub_rn(__fmul_rn(2.0f, x), 1.0f), __fadd_rn(2.0f, x));
      else id = 1, x = __fdiv_rn(__fsub_rn(x, 1.0f), __fadd_rn(x, 1.0f));
    } else {
      if (ix < 0x401c0000) id = 2, x = __fdiv_rn(__fsub_rn(x, 1.5f), __fadd_rn(1.0f, __fmul_rn(1.5f, x)));
      else id = 3, x = __fdiv_rn(-1.0f, x);
    }
  }
  const float z = __fmul_rn(x, x), w = __fmul_rn(z, z);
#define MA(a, b, c) __fadd_rn((a), __fmul_rn((b), (c)))  /* a + b*c, two roundings */
  const float s1 = __fmul_rn(z, MA(aT[0], w, MA(aT[2], w, MA(aT[4], w, MA(aT[6], w, MA(aT[8], w, aT[10]))))));
  const float s2 = __fmul_rn(w, MA(aT[1], w, MA(aT[3], w, MA(aT[5], w, MA(aT[7], w, aT[9])))));
#undef MA
  const float t = __fmul_rn(x, __fadd_rn(s1, s2));
  if (id < 0) return __fsub_rn(x, t);
  const float r = __fsub_rn(atanhi[id], __fsub_rn(__fsub_rn(t, atanlo[id]), x));
  return hx < 0 ? -r : r;
}

__device__ float dev_atan2f(float y, float x) {
  const float pi_o_2 = 1.5707963705e+00f, pi = 3.1415927410e+00f, pi_lo = -8.7422776573e-08f, tiny = 1.0e-30f;
  const int hx = (int)__float_as_uint(x), ix = hx & 0x7fffffff;
  const int hy = (int)__float_as_uint(y), iy = hy & 0x7fffffff;
  if (ix > 0x7f800000 || iy > 0x7f800000) return __fadd_rn(x, y);
  if (hx == 0x3f800000) return dev_atanf(y);
  const int m = ((hy >> 31) & 1) | ((hx >> 30) & 2);
  if (iy == 0) return m < 2 ? y : (m == 2 ? __fadd_rn(pi, tiny) : __fsub_rn(-pi, tiny));
  if (ix == 0) return hy < 0 ? __fsub_rn(-pi_o_2, tiny) : __fadd_rn(pi_o_2, tiny);
  const int k = (iy - ix) >> 23;
  float z;
  if (k > 60) z = __fadd_rn(pi_o_2, __fmul_rn(0.5f, pi_lo));
  else if (hx < 0 && k < -60) z = 0.0f;
  else z = dev_atanf(fabsf(__fdiv_rn(y, x)));
  switch (m) {
    case 0: return z;
    case 1: return __uint_as_float(__float_as_uint(z) ^ 0x80000000u);
    case 2: return __fsub_rn(pi, __fsub_rn(z, pi_lo));
    default: return __fsub_rn(__fsub_rn(z, pi_lo), pi);
  }
}

// ---------------------------------------------------------------------------------------------
// FAST-9 score
// ---------------------------------------------------------------------------------------------
#define FAST_RING(F)                                                                         \
  F(0, 0, -3) F(1, 1, -3) F(2, 2, -2) F(3, 3, -1) F(4, 3, 0) F(5, 3, 1) F(6, 2, 2) F(7, 1, 3) \
  F(8, 0, 3) F(9, -1, 3) F(10, -2, 2) F(11, -3, 1) F(12, -3, 0) F(13, -3, -1) F(14, -2, -2) F(15, -1, -3)

__device__ __forceinline__ bool run9(unsigned m) {  // circular run of >= 9 set bits in 16
  const unsigned mm = m | (m << 16);
  unsigned r = mm & (mm >> 1);
  r &= r >> 2;
  r &= r >> 4;
  r &= mm >> 8;
  return (r & 0xFFFFu) != 0;
}

__global__ void __launch_bounds__(256)
k_fast_score(const uint8_t *__restrict__ src, unsigned w, unsigned h, unsigned n, uint8_t *__restrict__ score,
             unsigned sw, unsigned sh, unsigned t) {
  const unsigned x = 3 + blockIdx.x * 32 + threadIdx.x;
  const unsigned y = 3 + blockIdx.y * 8 + threadIdx.y;
  if (x + 3 >= w || y + 3 >= h) return;
  for (unsigned f = blockIdx.z; f < n; f += gridDim.z) {
    const uint8_t *c = src + (size_t)f * w * h + (size_t)y * w + x;
    const unsigned p = __ldg(c), hi = p + t;
    const bool wrap = t > p;          // reference :498: p - threshold wraps => always "darker"
    const unsigned lo = p - t;        // only meaningful when !wrap
    const int iw = (int)w;
    // compass pre-test: any 9-arc contains at least two of ring positions 0, 4, 8, 12
    unsigned v0 = __ldg(c - 3 * iw), v4 = __ldg(c + 3), v8 = __ldg(c + 3 * iw), v12 = __ldg(c - 3);
    unsigned nb = (v0 > hi) + (v4 > hi) + (v8 > hi) + (v12 > hi);
    unsigned nd = (!(v0 > hi) && (wrap || v0 < lo)) + (!(v4 > hi) && (wrap || v4 < lo)) +
                  (!(v8 > hi) && (wrap || v8 < lo)) + (!(v12 > hi) && (wrap || v12 < lo));
    unsigned s = 0;
    if (nb >= 2 || nd >= 2) {
      unsigned bright = 0, dark = 0, mind = 255;
#define FAST_TAP(i, dx, dy)                                        \
  {                                                                \
    const unsigned v = __ldg(c + (dy) * iw + (dx));                \
    const bool b = v > hi;                                         \
    const bool d = !b && (wrap || v < lo);                         \
    bright |= (unsigned)b << (i);                                  \
    dark |= (unsigned)d << (i);                                    \
    mind = min(mind, v > p ? v - p : p - v);                       \
  }
      FAST_RING(FAST_TAP)
#undef FAST_TAP
      if (run9(bright) || run9(dark)) s = mind;
    }
    if (x < sw && y < sh) score[(size_t)f * sw * sh + (size_t)y * sw + x] = (uint8_t)s;
  }
}

// score-map read with the reference's gs_get semantics (0 outside the map)
__device__ __forceinline__ unsigned sm_get(const uint8_t *sm, unsigned sw, unsigned sh, unsigned x, unsigned y) {
  return (x < sw && y < sh) ? sm[(size_t)y * sw + x] : 0u;
}
__device__ __forceinline__ bool nms_keep(const uint8_t *sm, unsigned sw, unsigned sh, unsigned x, unsigned y,
                                         unsigned &s) {
  s = sm_get(sm, sw, sh, x, y);
  if (s == 0) return false;
  return sm_get(sm, sw, sh, x - 1, y - 1) <= s && sm_get(sm, sw, sh, x, y - 1) <= s &&
         sm_get(sm, sw, sh, x + 1, y - 1) <= s && sm_get(sm, sw, sh, x - 1, y) <= s &&
         sm_get(sm, sw, sh, x + 1, y) <= s && sm_get(sm, sw, sh, x - 1, y + 1) <= s &&
         sm_get(sm, sw, sh, x, y + 1) <= s && sm_get(sm, sw, sh, x + 1, y + 1) <= s;
}

struct KpRec {  // struct gs_keypoint, 48 bytes
  uint32_t w[12];
};

// ---------------------------------------------------------------------------------------------
// Tiled FAST (used when the score map has the image's size and t <= 255): a CTA stages its source tile (+3 halo)
// in shared memory; every pixel runs a cheap compass pre-test on 16-bit lane pairs, 4 pixels per thread: with
// K = 0x7FFF - t per lane, bit 15 of (v + K - p) is "v > p + t" and bit 15 of (p + K - v) is "v < p - t"; bit 15
// of (0x7FFF + t - p) is the wrap case t > p (reference :498), where every non-brighter sample counts as darker.
// The few candidates are compacted into a dense list so that the full 16-sample test runs with full warps (with
// one thread per pixel, one candidate lane dragged its whole warp through it).  Arc test on sign bits:
// funnel-shifting the sign of (hi - v) / (v - lo) into the masks costs one IADD and one SHF per sample and mask.
constexpr int FT_W = 128, FT_SW = FT_W + 32;   // tile columns; 160-B pitch = one TMA box row
constexpr int FT_X = 16;                        // tile byte of the first pixel column

// 4 bytes -> 16-bit lane pairs (b0, b2) and (b1, b3)
__device__ __forceinline__ void pairs_eo(uint32_t v, uint32_t &e, uint32_t &o) {
  e = v & 0x00FF00FFu;
  o = prmt(v, 0, 0x4341);
}

// ---------------------------------------------------------------------------------------------
// k_fast_tiled2: FAST score AND the 3x3 non-maximum mask of a tile in one kernel (round 2).
// Round 1 ran k_nms_mask as a second, latency-bound pass over the score map (1.1 TB/s) that the score kernel
// had just held in shared memory.  Here a CTA scores a 66-row x 130-column region -- its 64 x 128 tile plus a
// 1-pixel ring, recomputed instead of exchanged -- and derives the tile's NMS bits straight from shared memory.
// Ring cells that FAST never writes (x = 2, x = w-3, y = 2, y = h-3: whatever the caller left in the map takes
// part in the NMS, reference :517-524) are fetched from the global score map; nobody writes those, so there is
// no race between tiles.  Outputs: the score tile (interior pixels only), the per-row survivor bit masks
// (pixel x -> bit x & 31 of word x >> 5) and per-row survivor counts (atomicAdd; zeroed by the launcher).
// The compass pre-test is the tighter "two ADJACENT compass points": nine consecutive ring positions always
// contain two consecutive multiples of four, so a corner needs (p0|p8) & (p4|p12) on the brighter or on the
// darker side -- fewer candidates for the 16-sample test than round 1's "any two of four".
// ---------------------------------------------------------------------------------------------
constexpr int F2_TH = 64;                          // tile rows (4x round 1's: the per-thread set-up is paid once per 64 rows)
constexpr int F2_ROWS = F2_TH + 2;                 // scored rows: y0-1 .. y0+64
constexpr int F2_SH = F2_ROWS + 6;                 // source rows: y0-4 .. y0+67
constexpr int F2_PITCH = 136;                      // score pitch: column lx (-1 .. 128) at byte lx + 4
constexpr int F2_THREADS = 288;                    // 9 warps; warp q scores rows q, q+9, .. (8 of them)
constexpr int F2_KROWS = 8;

template <bool TMA>
__global__ void __launch_bounds__(F2_THREADS)
k_fast_tiled2(const __grid_constant__ CUtensorMap tmap, const uint8_t *__restrict__ src, unsigned w, unsigned h,
              uint8_t *__restrict__ score, unsigned t, unsigned mw, unsigned *__restrict__ masks,
              unsigned *__restrict__ rowcount) {
  __shared__ __align__(128) uint8_t s_src[F2_SH * FT_SW];
  __shared__ __align__(8) uint64_t bar;
  __shared__ __align__(16) uint8_t s_score[F2_ROWS * F2_PITCH];
  __shared__ uint16_t s_list[F2_ROWS * 130];       // candidate = (row << 8) | (column + 4)
  __shared__ unsigned s_cnt;
  const unsigned f = blockIdx.z, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int x0 = blockIdx.x * FT_W, y0 = 3 + blockIdx.y * F2_TH;   // tile = columns [x0, x0+128), rows [y0, y0+64)
  const int iw = (int)w, ih = (int)h, ti = (int)min(t, 255u);
  const uint8_t *img = src + (size_t)f * w * h;
  if (tid == 0) s_cnt = 0;
  if (TMA) {
    if (tid == 0) {
      mbar_init(&bar, 1);
      mbar_fence_init();
    }
    __syncthreads();
    if (tid == 0) {
      mbar_expect_tx(&bar, F2_SH * FT_SW);
      tma_load_3d(s_src, &tmap, (x0 - FT_X) / 4, y0 - 4, (int)f, &bar);   // out-of-image reads as 0, never used
    }
  } else {
    for (int i = tid; i < F2_SH * FT_SW; i += F2_THREADS) {
      const int r = i / FT_SW, c = i % FT_SW;
      const int yy = min(max(y0 - 4 + r, 0), ih - 1), xx = min(max(x0 - FT_X + c, 0), iw - 1);
      s_src[i] = __ldg(img + (size_t)yy * w + xx);
    }
  }
  {
    uint4 *z = reinterpret_cast<uint4 *>(s_score);
    for (int i = tid; i < F2_ROWS * F2_PITCH / 16; i += F2_THREADS) z[i] = make_uint4(0, 0, 0, 0);
  }
  const int lx = 4 * lane;
  unsigned colmask = 0;                                     // interior columns: 3 <= x < w - 3
#pragma unroll
  for (int j = 0; j < 4; j++) colmask |= (unsigned)(x0 + lx + j >= 3 && x0 + lx + j + 3 < iw) << j;
  if (TMA) mbar_wait(&bar, 0);
  __syncthreads();

  // phase A: pre-test.  Row ly (0..65) <-> image row y0 - 1 + ly <-> s_src row ly + 3.
  {
    const uint32_t kb = (0x7FFFu - (uint32_t)ti) * 0x10001u, kw = (0x7FFFu + (uint32_t)ti) * 0x10001u;
    unsigned flags = 0;                                     // bit 4k + j: row warp + 9k, pixel j is a candidate
    const uint32_t *col0 = reinterpret_cast<const uint32_t *>(s_src) + (FT_X / 4) + lane;
#pragma unroll
    for (int k = 0; k < F2_KROWS; k++) {
      const int ly = (int)warp + 9 * k, y = y0 - 1 + ly;
      if (ly >= F2_ROWS || y < 3 || y + 3 >= ih || colmask == 0) continue;
      const uint32_t *rowc = col0 + (ly + 3) * (FT_SW / 4);
      const uint32_t wl = rowc[-1], wc = rowc[0], wr = rowc[1];
      const uint32_t up = rowc[-3 * (FT_SW / 4)], dn = rowc[3 * (FT_SW / 4)];
      const uint32_t v12 = __funnelshift_r(wl, wc, 8);      // bytes x-3 .. x
      const uint32_t v4 = __funnelshift_r(wc, wr, 24);      // bytes x+3 .. x+6
      uint32_t pe, po, ve[4], vo[4];
      pairs_eo(wc, pe, po);
      pairs_eo(up, ve[0], vo[0]);
      pairs_eo(v4, ve[1], vo[1]);
      pairs_eo(dn, ve[2], vo[2]);
      pairs_eo(v12, ve[3], vo[3]);
      unsigned cbits = 0;
#pragma unroll
      for (int hlf = 0; hlf < 2; hlf++) {
        const uint32_t P = hlf ? po : pe;
        const uint32_t q = kb - P, r = P + kb, wrap = kw - P;
        uint32_t b[4], d[4];
#pragma unroll
        for (int i = 0; i < 4; i++) {
          const uint32_t V = hlf ? vo[i] : ve[i];
          b[i] = V + q;                                     // bit 15 / 31: v > p + t
          d[i] = r - V;                                     // bit 15 / 31: v < p - t (when t <= p)
        }
        const uint32_t adj_b = (b[0] | b[2]) & (b[1] | b[3]);
        const uint32_t adj_d = (d[0] | d[2]) & (d[1] | d[3]);
        const uint32_t adj_nb = ~((b[0] & b[2]) | (b[1] & b[3]));     // wrap case (t > p): darker = not brighter
        const uint32_t cand = (adj_b | (wrap & adj_nb) | (~wrap & adj_d)) & 0x80008000u;
        cbits |= (cand >> (15 - hlf)) & (1u << hlf);        // bit 15 -> pixel hlf
        cbits |= cand >> (29 - hlf);                        // bit 31 -> pixel 2 + hlf
      }
      flags |= (cbits & colmask) << (4 * k);
    }
    // the two ring columns x0 - 1 and x0 + 128 (66 rows each): scalar form of the same pre-test
    bool hc = false;
    int hent = 0;
    if (tid < 2 * F2_ROWS) {
      const int hly = (int)tid >> 1, hlx = (tid & 1) ? FT_W : -1;
      const int x = x0 + hlx, y = y0 - 1 + hly;
      hent = (hly << 8) | (hlx + 4);
      if (x >= 3 && x + 3 < iw && y >= 3 && y + 3 < ih) {
        const uint8_t *c = s_src + (hly + 3) * FT_SW + (hlx + FT_X);
        const int p = c[0], hi = p + ti, lo = p - ti;
        const int v0 = c[-3 * FT_SW], v4 = c[3], v8 = c[3 * FT_SW], v12 = c[-3];
        const bool b0 = v0 > hi, b1 = v4 > hi, b2 = v8 > hi, b3 = v12 > hi;
        const bool wrp = ti > p;
        const bool d0 = wrp ? !b0 : v0 < lo, d1 = wrp ? !b1 : v4 < lo, d2 = wrp ? !b2 : v8 < lo, d3 = wrp ? !b3 : v12 < lo;
        hc = ((b0 || b2) && (b1 || b3)) || ((d0 || d2) && (d1 || d3));
      }
    }
    if (__any_sync(0xFFFFFFFFu, flags != 0 || hc)) {
      const unsigned c = __popc(flags) + (hc ? 1u : 0u);
      unsigned incl = c;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned u = __shfl_up_sync(0xFFFFFFFFu, incl, o);
        if (lane >= (unsigned)o) incl += u;
      }
      unsigned base = 0;
      if (lane == 31) base = atomicAdd(&s_cnt, incl);
      base = __shfl_sync(0xFFFFFFFFu, base, 31) + incl - c;
      if (hc) s_list[base++] = (uint16_t)hent;
      while (flags) {
        const int bit = __ffs(flags) - 1;
        flags &= flags - 1;
        s_list[base++] = (uint16_t)((((int)warp + 9 * (bit >> 2)) << 8) | (lx + (bit & 3) + 4));
      }
    }
  }
  __syncthreads();

  // phase B: the full 16-sample test on the dense candidate list
  {
    const unsigned ncand = s_cnt;
    for (unsigned k = tid; k < ncand; k += F2_THREADS) {
      const int e = s_list[k], ly = e >> 8, cx = e & 0xFF;                     // cx = lx + 4
      const uint8_t *c = s_src + (ly + 3) * FT_SW + (cx - 4 + FT_X);
      const int p = c[0], hi = p + ti, lo = p - ti;
      unsigned bright = 0, dark = 0;
      int mind = 255;
#define FAST_TAP3(i_, dx, dy)                                                       \
  {                                                                                 \
    const int v = c[(dy) * FT_SW + (dx)];                                           \
    bright = __funnelshift_l((unsigned)(hi - v), bright, 1);   /* bit = (v > hi) */  \
    dark = __funnelshift_l((unsigned)(v - lo), dark, 1);       /* bit = (v < lo) */  \
    mind = min(mind, abs(v - p));                                                   \
  }
      FAST_RING(FAST_TAP3)
#undef FAST_TAP3
      bright &= 0xFFFFu;
      dark = (ti > p) ? (~bright & 0xFFFFu) : (dark & 0xFFFFu);                // reference :498 wrap
      if (run9(bright) || run9(dark)) s_score[ly * F2_PITCH + cx] = (uint8_t)mind;
    }
    // Ring cells FAST never writes (x = 2, x = w-3, y = 2, y = h-3) keep the caller's bytes and take part in
    // the NMS: fetch the ones this region contains (border tiles only; other non-interior cells are never read)
    const bool border_tile = x0 < 4 || x0 + FT_W + 3 >= iw || y0 < 4 || y0 + F2_TH + 3 >= ih;
    if (border_tile) {
      const uint8_t *sm = score + (size_t)f * w * h;
      for (int i = tid; i < 2 * F2_ROWS + 2 * 130; i += F2_THREADS) {
        int x, y;
        if (i < 2 * F2_ROWS) x = (i & 1) ? iw - 3 : 2, y = y0 - 1 + (i >> 1);
        else x = x0 - 1 + ((i - 2 * F2_ROWS) >> 1), y = (i & 1) ? ih - 3 : 2;
        const int lxx = x - x0, lyy = y - (y0 - 1);
        if (lxx >= -1 && lxx <= FT_W && lyy >= 0 && lyy < F2_ROWS && x >= 0 && x < iw && y >= 0 && y < ih)
          s_score[lyy * F2_PITCH + lxx + 4] = __ldg(sm + (size_t)y * w + x);
      }
    }
  }
  __syncthreads();

  // phase C + D: write the tile's scores (interior pixels, a word per 4) and its NMS bits.  Warp wq = 0..7 owns tile
  // rows wq, wq + 8, ..; a lane owns 4 pixels; all-zero score words (almost all) skip the neighbour tests.
  if (warp < 8) {                                             // every lane stays in: warp collectives below
    const unsigned rows = h - 6;
    const bool full = colmask == 0xF && TMA;
    const unsigned word = (unsigned)(x0 + lx) >> 5;
    const bool mask_lane = (lane & 7) == 0 && word < mw;
    uint8_t *q = score + (size_t)f * w * h + (size_t)(y0 + (int)warp) * w + x0 + lx;
    unsigned *mrow = masks + ((size_t)f * rows + (unsigned)(y0 - 3 + (int)warp)) * mw + word;
    unsigned *rc = rowcount + (size_t)f * rows + (unsigned)(y0 - 3 + (int)warp);
    const uint8_t *srow = s_score + ((int)warp + 1) * F2_PITCH + 4 + lx;
    for (int k = 0; k < F2_TH / 8; k++) {
      const int y = y0 + (int)warp + 8 * k;
      if (y + 3 >= ih) break;                                 // warp-uniform
      const uint32_t v = *reinterpret_cast<const uint32_t *>(srow);
      if (full) {
        *reinterpret_cast<uint32_t *>(q) = v;
      } else if (colmask) {
#pragma unroll
        for (int j = 0; j < 4; j++)
          if ((colmask >> j) & 1u) q[j] = (uint8_t)(v >> (8 * j));
      }
      unsigned nib = 0;
      if (v != 0 && colmask) {
        const uint8_t *a = srow - F2_PITCH, *c = srow + F2_PITCH;
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const unsigned sc = (v >> (8 * j)) & 0xFFu;
          if (sc != 0 && ((colmask >> j) & 1u)) {
            const bool keep = a[j - 1] <= sc && a[j] <= sc && a[j + 1] <= sc && srow[j - 1] <= sc && srow[j + 1] <= sc &&
                              c[j - 1] <= sc && c[j] <= sc && c[j + 1] <= sc;
            nib |= (unsigned)keep << j;
          }
        }
      }
      unsigned m = 0;
      if (__any_sync(0xFFFFFFFFu, nib != 0)) {               // rare: a surviving corner in this 128-pixel row piece
        m = nib << (4 * (lane & 7));
        m |= __shfl_xor_sync(0xFFFFFFFFu, m, 1);
        m |= __shfl_xor_sync(0xFFFFFFFFu, m, 2);
        m |= __shfl_xor_sync(0xFFFFFFFFu, m, 4);
        if (mask_lane && m) atomicAdd(rc, __popc(m));
      }
      if (mask_lane) *mrow = m;
      q += (size_t)8 * w, mrow += (size_t)8 * mw, rc += 8, srow += 8 * F2_PITCH;
    }
  }
}

// NMS in one pass: per interior row a bit mask of survivors (pixel x -> bit x & 31 of word x >> 5)
// and their count.  A thread owns 4 pixels (one aligned word of the score row); all-zero words --
// the common case -- skip the neighbour rows entirely.
template <bool VEC>
__global__ void __launch_bounds__(256)
k_nms_mask(const uint8_t *__restrict__ score, unsigned sw, unsigned sh, unsigned w, unsigned h, unsigned mw,
           unsigned *__restrict__ masks, unsigned *__restrict__ rowcount) {
  const unsigned rows = h - 6, lane = threadIdx.x & 31;
  const unsigned row = blockIdx.x * 8 + (threadIdx.x >> 5), f = blockIdx.y;   // one warp per interior row
  if (row >= rows) return;
  const unsigned y = 3 + row;
  const uint8_t *sm = score + (size_t)f * sw * sh;
  unsigned *mrow = masks + ((size_t)f * rows + row) * mw;
  unsigned total = 0;
  for (unsigned xb = 0; xb < w; xb += 128) {         // 32 lanes x 4 pixels
    const unsigned x4 = xb + lane * 4;
    unsigned nib = 0;
    if (x4 < w) {
      bool any = true;
      if (VEC) any = __ldg(reinterpret_cast<const uint32_t *>(sm + (size_t)y * sw + x4)) != 0;
      if (any) {
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const unsigned x = x4 + j;
          unsigned s;
          if (x >= 3 && x + 3 < w && nms_keep(sm, sw, sh, x, y, s)) nib |= 1u << j;
        }
      }
    }
    // 8 lanes x 4 bits -> one 32-pixel mask word
    unsigned m = nib << (4 * (lane & 7));
    m |= __shfl_xor_sync(0xFFFFFFFFu, m, 1);
    m |= __shfl_xor_sync(0xFFFFFFFFu, m, 2);
    m |= __shfl_xor_sync(0xFFFFFFFFu, m, 4);
    const unsigned word = x4 >> 5;
    if ((lane & 7) == 0 && word < mw) mrow[word] = m;
    total += __popc(nib);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) total += __shfl_xor_sync(0xFFFFFFFFu, total, o);
  if (lane == 0) rowcount[(size_t)f * rows + row] = total;
}

// emit from the masks: one warp per interior row; rows past the cap or without survivors exit
__global__ void __launch_bounds__(256)
k_nms_emit_masks(const uint8_t *__restrict__ score, unsigned sw, unsigned sh, unsigned w, unsigned h, unsigned mw,
                 const unsigned *__restrict__ masks, const unsigned *__restrict__ rowoff, unsigned rows_total,
                 KpRec *__restrict__ kps, unsigned nkps) {
  const unsigned rows = h - 6;
  const unsigned long long gw = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const unsigned lane = threadIdx.x & 31;
  if (gw >= rows_total) return;
  const unsigned f = (unsigned)(gw / rows), row = (unsigned)(gw % rows), y = 3 + row;
  unsigned base = rowoff[gw];
  if (base >= nkps) return;
  if (row + 1 < rows && rowoff[gw + 1] == base) return;   // no survivor in this row (exclusive offsets: next == own)
  const unsigned *mrow = masks + gw * mw;
  const uint8_t *sm = score + (size_t)f * sw * sh;
  for (unsigned w0 = 0; w0 < mw && base < nkps; w0 += 32) {
    const unsigned m = (w0 + lane < mw) ? mrow[w0 + lane] : 0u;
    unsigned c = __popc(m), incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned u = __shfl_up_sync(0xFFFFFFFFu, incl, o);
      if (lane >= (unsigned)o) incl += u;
    }
    unsigned pos = base + incl - c;
    unsigned bits = m;
    while (bits && pos < nkps) {
      const unsigned b = __ffs(bits) - 1;
      bits &= bits - 1;
      const unsigned x = (w0 + lane) * 32 + b;
      uint4 *o = reinterpret_cast<uint4 *>(kps + (size_t)f * nkps + pos);
      o[0] = make_uint4(x, y, sm_get(sm, sw, sh, x, y), 0), o[1] = make_uint4(0, 0, 0, 0), o[2] = make_uint4(0, 0, 0, 0);
      pos++;
    }
    base += __shfl_sync(0xFFFFFFFFu, incl, 31);
  }
}

// ---------------------------------------------------------------------------------------------
// ORB: stable sort by response, margin filter, cap
// ---------------------------------------------------------------------------------------------
constexpr unsigned ORB_MAXC = 5000;  // the reference's static candidates[5000] (grayskull.h:655)

__global__ void __launch_bounds__(256)
k_orb_select(const KpRec *__restrict__ cand, const unsigned *__restrict__ cand_count, unsigned cap, unsigned w,
             unsigned h, KpRec *__restrict__ kps, unsigned *__restrict__ counts, unsigned nkps) {
  __shared__ uint8_t resp[ORB_MAXC];
  __shared__ uint16_t order[ORB_MAXC];
  __shared__ unsigned start[256];
  __shared__ unsigned wcnt[8];
  const unsigned f = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const KpRec *c = cand + (size_t)f * cap;
  const unsigned n = min(cand_count[f], cap);
  start[tid] = 0;
  __syncthreads();
  for (unsigned i = tid; i < n; i += 256) {
    const unsigned r = min(c[i].w[2], 255u);
    resp[i] = (uint8_t)r;
    atomicAdd(&start[r], 1u);
  }
  __syncthreads();
  if (tid == 0) {  // descending exclusive prefix: start[b] = #candidates with response > b
    unsigned acc = 0;
    for (int b = 255; b >= 0; b--) {
      const unsigned cnt = start[b];
      start[b] = acc, acc += cnt;
    }
  }
  __syncthreads();
  if (warp == 0) {  // stable rank inside equal-response groups, in candidate (raster) order
    for (unsigned b = 0; b < n; b += 32) {
      const unsigned i = b + lane;
      const unsigned key = i < n ? resp[i] : 0x10000u + lane;
      const unsigned m = __match_any_sync(0xFFFFFFFFu, key);
      if (i < n) order[start[key] + __popc(m & ((1u << lane) - 1u))] = (uint16_t)i;
      __syncwarp();
      if (i < n && lane == (unsigned)(__ffs(m) - 1)) start[key] += __popc(m);
      __syncwarp();
    }
  }
  __syncthreads();
  // first nkps sorted candidates at least 15 px away from every border (reference :659-667)
  unsigned running = 0;
  const unsigned radius = 15;
  for (unsigned b = 0; b < n && running < nkps; b += 256) {
    const unsigned pos = b + tid;
    unsigned x = 0, y = 0, r = 0;
    bool pass = false;
    if (pos < n) {
      const KpRec k = c[order[pos]];
      x = k.w[0], y = k.w[1], r = k.w[2];
      pass = x >= radius && y >= radius && x < w - radius && y < h - radius;
    }
    const unsigned bal = __ballot_sync(0xFFFFFFFFu, pass);
    if (lane == 0) wcnt[warp] = __popc(bal);
    __syncthreads();
    unsigned before = 0, total = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) {
      const unsigned cc = wcnt[i];
      before += (i < (int)warp) ? cc : 0;
      total += cc;
    }
    const unsigned j = running + before + __popc(bal & ((1u << lane) - 1u));
    if (pass && j < nkps) {
      uint4 *o = reinterpret_cast<uint4 *>(kps + (size_t)f * nkps + j);
      o[0] = make_uint4(x, y, r, 0), o[1] = make_uint4(0, 0, 0, 0), o[2] = make_uint4(0, 0, 0, 0);
    }
    running += total;
    __syncthreads();
  }
  if (tid == 0) counts[f] = min(running, nkps);
}

// r = 15 (the only radius gs_orb_extract uses, reference :658): row dy of the disc spans |dx| <= hw(dy),
// hw = floor(sqrt(225 - dy^2)), known at compile time; lane = dx + 15.
__device__ __forceinline__ constexpr int disc15_hw(int dy) {
  int a = dy < 0 ? -dy : dy, hw = 0;
  while ((hw + 1) * (hw + 1) + a * a <= 225) hw++;
  return hw;
}
__device__ __forceinline__ void disc_moments15(const uint8_t *img, unsigned w, int x, int y, unsigned lane, int &m01,
                                               int &m10) {
  const int dx = (int)lane - 15;
  const int adx = dx < 0 ? -dx : dx;
  const uint8_t *p = img + (size_t)(y - 15) * w + (x + dx);   // lane 31 is never dereferenced
  int a01 = 0, rowsum = 0, a10 = 0;
#pragma unroll
  for (int dy = -15; dy <= 15; dy++) {
    const int v = (adx <= disc15_hw(dy)) ? (int)__ldg(p) : 0;
    a01 += dy * v;
    rowsum += v;
    p += w;
  }
  a10 = dx * rowsum;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a01 += __shfl_xor_sync(0xFFFFFFFFu, a01, o);
    a10 += __shfl_xor_sync(0xFFFFFFFFu, a10, o);
  }
  m01 = a01, m10 = a10;
}

// intensity-centroid moments over the disc dx^2 + dy^2 <= r^2; lanes = dx (r <= 15 per pass)
__device__ __forceinline__ void disc_moments(const uint8_t *img, unsigned w, int x, int y, int r, unsigned lane,
                                             int &m01, int &m10) {
  int a01 = 0, a10 = 0;
  for (int dx0 = -r; dx0 <= r; dx0 += 32) {
    const int dx = dx0 + (int)lane;
    if (dx <= r)
      for (int dy = -r; dy <= r; dy++)
        if (dx * dx + dy * dy <= r * r) {
          const int v = __ldg(img + (size_t)(y + dy) * w + (x + dx));
          a01 += dy * v, a10 += dx * v;
        }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a01 += __shfl_xor_sync(0xFFFFFFFFu, a01, o);
    a10 += __shfl_xor_sync(0xFFFFFFFFu, a10, o);
  }
  m01 = a01, m10 = a10;
}

__device__ __forceinline__ float orient_from_moments(int m01, int m10, int trig_mode) {
  // the reference's float accumulators hold exact integers (< 2^24 for r = 15), so the int32
  // moments converted once are the same floats (reference :608-620)
  return trig_mode ? atan2f((float)m01, (float)m10) : dev_atan2f((float)m01, (float)m10);
}

// BRIEF-256 (reference :623-637); each ballot is one descriptor word
__device__ __forceinline__ void brief_words(const uint8_t *img, unsigned w, unsigned h, int x, int y, float angle,
                                            unsigned lane, int trig_mode, uint32_t (&desc)[8]) {
  const float a2 = __fadd_rn(angle, 1.57079f);
  const float sin_a = trig_mode ? sinf(angle) : dev_sinf(angle);
  const float cos_a = trig_mode ? sinf(a2) : dev_sinf(a2);
#pragma unroll
  for (int k = 0; k < 8; k++) {
    const uint32_t pk = __ldg(&c_brief[32 * k + lane]);
    const float p0 = (float)(int)(int8_t)(pk & 0xFF), p1 = (float)(int)(int8_t)((pk >> 8) & 0xFF);
    const float p2 = (float)(int)(int8_t)((pk >> 16) & 0xFF), p3 = (float)(int)(int8_t)(pk >> 24);
    const float dx1 = __fsub_rn(__fmul_rn(p0, cos_a), __fmul_rn(p1, sin_a));
    const float dy1 = __fadd_rn(__fmul_rn(p0, sin_a), __fmul_rn(p1, cos_a));
    const float dx2 = __fsub_rn(__fmul_rn(p2, cos_a), __fmul_rn(p3, sin_a));
    const float dy2 = __fadd_rn(__fmul_rn(p2, sin_a), __fmul_rn(p3, cos_a));
    const unsigned x1 = (unsigned)(x + __float2int_rz(dx1)), y1 = (unsigned)(y + __float2int_rz(dy1));
    const unsigned x2 = (unsigned)(x + __float2int_rz(dx2)), y2 = (unsigned)(y + __float2int_rz(dy2));
    const unsigned i1 = (x1 < w && y1 < h) ? __ldg(img + (size_t)y1 * w + x1) : 0u;
    const unsigned i2 = (x2 < w && y2 < h) ? __ldg(img + (size_t)y2 * w + x2) : 0u;
    desc[k] = __ballot_sync(0xFFFFFFFFu, i1 > i2);
  }
}

// gs_orb_extract's describe step in three kernels, so that the (expensive, double-precision) libm
// restatement runs once per keypoint on one thread instead of redundantly on all 32 lanes of a warp:
//   k_orb_moments : warp per keypoint -> int32 disc moments (stored in the record's descriptor words 0,1)
//   k_orb_trig    : thread per keypoint -> angle, sin, cos  (angle in place, sin/cos in descriptor words 2,3)
//   k_orb_brief   : warp per keypoint -> BRIEF-256, final record
__global__ void __launch_bounds__(256)
k_orb_moments(const uint8_t *__restrict__ src, unsigned w, unsigned h, KpRec *__restrict__ kps,
              const unsigned *__restrict__ counts, unsigned nkps, unsigned n) {
  const unsigned long long gw = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const unsigned lane = threadIdx.x & 31;
  if (gw >= (unsigned long long)n * nkps) return;
  const unsigned f = (unsigned)(gw / nkps), j = (unsigned)(gw % nkps);
  if (j >= counts[f]) return;
  KpRec *k = kps + (size_t)f * nkps + j;
  int m01, m10;
  disc_moments15(src + (size_t)f * w * h, w, (int)k->w[0], (int)k->w[1], lane, m01, m10);
  if (lane == 0) k->w[4] = (uint32_t)m01, k->w[5] = (uint32_t)m10;
}

__global__ void __launch_bounds__(256)
k_orb_trig(KpRec *__restrict__ kps, const unsigned *__restrict__ counts, unsigned nkps, unsigned n, int trig_mode) {
  const unsigned long long g = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (unsigned long long)n * nkps) return;
  const unsigned f = (unsigned)(g / nkps), j = (unsigned)(g % nkps);
  if (j >= counts[f]) return;
  KpRec *k = kps + (size_t)f * nkps + j;
  const float angle = orient_from_moments((int)k->w[4], (int)k->w[5], trig_mode);
  const float a2 = __fadd_rn(angle, 1.57079f);       // the reference's 6-digit pi/2 (:626)
  const float sin_a = trig_mode ? sinf(angle) : dev_sinf(angle);
  const float cos_a = trig_mode ? sinf(a2) : dev_sinf(a2);
  k->w[3] = __float_as_uint(angle);
  k->w[6] = __float_as_uint(sin_a), k->w[7] = __float_as_uint(cos_a);
}

// BRIEF-256 with given sin/cos (reference :628-636); each ballot is one descriptor word
__device__ __forceinline__ void brief_words_sc(const uint8_t *img, unsigned w, unsigned h, int x, int y, float sin_a,
                                               float cos_a, unsigned lane, uint32_t (&desc)[8]) {
#pragma unroll
  for (int k = 0; k < 8; k++) {
    const uint32_t pk = __ldg(&c_brief[32 * k + lane]);
    const float p0 = (float)(int)(int8_t)(pk & 0xFF), p1 = (float)(int)(int8_t)((pk >> 8) & 0xFF);
    const float p2 = (float)(int)(int8_t)((pk >> 16) & 0xFF), p3 = (float)(int)(int8_t)(pk >> 24);
    const float dx1 = __fsub_rn(__fmul_rn(p0, cos_a), __fmul_rn(p1, sin_a));
    const float dy1 = __fadd_rn(__fmul_rn(p0, sin_a), __fmul_rn(p1, cos_a));
    const float dx2 = __fsub_rn(__fmul_rn(p2, cos_a), __fmul_rn(p3, sin_a));
    const float dy2 = __fadd_rn(__fmul_rn(p2, sin_a), __fmul_rn(p3, cos_a));
    const unsigned x1 = (unsigned)(x + __float2int_rz(dx1)), y1 = (unsigned)(y + __float2int_rz(dy1));
    const unsigned x2 = (unsigned)(x + __float2int_rz(dx2)), y2 = (unsigned)(y + __float2int_rz(dy2));
    const unsigned i1 = (x1 < w && y1 < h) ? __ldg(img + (size_t)y1 * w + x1) : 0u;
    const unsigned i2 = (x2 < w && y2 < h) ? __ldg(img + (size_t)y2 * w + x2) : 0u;
    desc[k] = __ballot_sync(0xFFFFFFFFu, i1 > i2);
  }
}

// The 512 samples of a descriptor lie within +-22 px of the keypoint (pattern offsets <= 15 per axis,
// any rotation).  The warp stages that 45-row x 48-byte patch in shared memory with coalesced word
// loads (zeros outside the image = gs_get's out-of-bounds value) and gathers from there.
constexpr int BP_R = 22, BP_ROWS = 2 * BP_R + 1, BP_PITCH = 48;

template <bool STAGED>
__global__ void __launch_bounds__(256)
k_orb_brief(const uint8_t *__restrict__ src, unsigned w, unsigned h, KpRec *__restrict__ kps,
            const unsigned *__restrict__ counts, unsigned nkps, unsigned n) {
  __shared__ __align__(16) uint8_t s_patch[STAGED ? 8 : 1][BP_ROWS * BP_PITCH];
  const unsigned long long gw = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (gw >= (unsigned long long)n * nkps) return;
  const unsigned f = (unsigned)(gw / nkps), j = (unsigned)(gw % nkps);
  if (j >= counts[f]) return;
  KpRec *k = kps + (size_t)f * nkps + j;
  const uint8_t *img = src + (size_t)f * w * h;
  const int x = (int)k->w[0], y = (int)k->w[1];
  const float sin_a = __uint_as_float(k->w[6]), cos_a = __uint_as_float(k->w[7]);
  uint32_t desc[8];
  if (!STAGED) {
    brief_words_sc(img, w, h, x, y, sin_a, cos_a, lane, desc);
  } else {
    uint8_t *patch = s_patch[warp];
    const int xa = (x - BP_R) & ~3;                      // patch byte 0 <-> image column xa (w % 4 == 0)
    // all 17 word loads of a lane are issued before the first store (the rolled loop waited for each load in turn:
    // 53 % of the kernel's stall samples sat on its STS)
    constexpr int BP_WORDS = BP_ROWS * (BP_PITCH / 4), BP_ITERS = (BP_WORDS + 31) / 32;
    uint32_t pv[BP_ITERS];
#pragma unroll
    for (int k = 0; k < BP_ITERS; k++) {
      const int i = (int)lane + 32 * k;
      const int r = i / (BP_PITCH / 4), c = i % (BP_PITCH / 4);
      const int yy = y - BP_R + r, xx = xa + 4 * c;
      pv[k] = 0;
      if (i < BP_WORDS && yy >= 0 && yy < (int)h && xx >= 0 && xx < (int)w)
        pv[k] = __ldg(reinterpret_cast<const uint32_t *>(img + (size_t)yy * w + xx));
    }
#pragma unroll
    for (int k = 0; k < BP_ITERS; k++) {
      const int i = (int)lane + 32 * k;
      if (i < BP_WORDS) reinterpret_cast<uint32_t *>(patch)[i] = pv[k];
    }
    __syncwarp();
    const int ox = x - xa;                               // keypoint column inside the patch
#pragma unroll
    for (int kk = 0; kk < 8; kk++) {
      const float4 pf = __ldg(&c_brieff[32 * kk + lane]);
      const float p0 = pf.x, p1 = pf.y, p2 = pf.z, p3 = pf.w;
      const int dx1 = __float2int_rz(__fsub_rn(__fmul_rn(p0, cos_a), __fmul_rn(p1, sin_a)));
      const int dy1 = __float2int_rz(__fadd_rn(__fmul_rn(p0, sin_a), __fmul_rn(p1, cos_a)));
      const int dx2 = __float2int_rz(__fsub_rn(__fmul_rn(p2, cos_a), __fmul_rn(p3, sin_a)));
      const int dy2 = __float2int_rz(__fadd_rn(__fmul_rn(p2, sin_a), __fmul_rn(p3, cos_a)));
      // |d| <= 22 always (sqrt(2) * 15 = 21.2); the clamp only keeps a hypothetical outlier in bounds
      const int c1 = min(max(dx1, -BP_R), BP_R) + ox, r1 = min(max(dy1, -BP_R), BP_R) + BP_R;
      const int c2 = min(max(dx2, -BP_R), BP_R) + ox, r2 = min(max(dy2, -BP_R), BP_R) + BP_R;
      const unsigned i1 = patch[r1 * BP_PITCH + c1], i2 = patch[r2 * BP_PITCH + c2];
      desc[kk] = __ballot_sync(0xFFFFFFFFu, i1 > i2);
    }
  }
  __syncwarp();
  if (lane == 0) {
    uint4 *o = reinterpret_cast<uint4 *>(k);
    o[1] = make_uint4(desc[0], desc[1], desc[2], desc[3]);
    o[2] = make_uint4(desc[4], desc[5], desc[6], desc[7]);
  }
}

// single-call forms of gs_compute_orientation / gs_brief_descriptor (one warp)
__global__ void k_orient_one(const uint8_t *img, unsigned w, unsigned x, unsigned y, unsigned r, int trig_mode,
                             float *out) {
  if (r > 15) {
    // Beyond r = 15 the reference's float accumulators (:610-617) can exceed 2^24 and start rounding, so the
    // sums are rebuilt the way the reference does: one thread, fp32 adds in its dy-outer / dx-inner order.
    if (threadIdx.x == 0) {
      float m01 = 0.0f, m10 = 0.0f;
      const int ri = (int)r, r2 = (int)(r * r);
      for (int dy = -ri; dy <= ri; dy++)
        for (int dx = -ri; dx <= ri; dx++)
          if (dx * dx + dy * dy <= r2) {
            const int v = __ldg(img + (size_t)((int)y + dy) * w + ((int)x + dx));
            m01 = __fadd_rn(m01, (float)(dy * v));
            m10 = __fadd_rn(m10, (float)(dx * v));
          }
      *out = trig_mode ? atan2f(m01, m10) : dev_atan2f(m01, m10);
    }
    return;
  }
  int m01, m10;
  disc_moments(img, w, (int)x, (int)y, (int)r, threadIdx.x, m01, m10);
  // r <= 15: |moment| < 2^24, the reference's float sums are exact integers = these int32 sums
  const float a = orient_from_moments(m01, m10, trig_mode);
  if (threadIdx.x == 0) *out = a;
}
__global__ void k_brief_one(const uint8_t *img, unsigned w, unsigned h, KpRec *kp, int trig_mode) {
  uint32_t desc[8];
  brief_words(img, w, h, (int)kp->w[0], (int)kp->w[1], __uint_as_float(kp->w[3]), threadIdx.x, trig_mode, desc);
  if (threadIdx.x < 8) kp->w[4 + threadIdx.x] = desc[threadIdx.x];
}

// ---- first-use libm self-check (trig mode 0) --------------------------------------------------------------
// Trig mode 0 restates glibc 2.39's sinf / atan2f; the contract is "identical to the reference on the same box",
// and the reference calls whatever libm that box has.  On first use the device routines are compared with THIS
// host's libm on 8192 samples (the moment range atan2f sees, the angle range sinf sees); a host whose libm rounds
// differently gets a one-time warning on stderr and gs_b200_trig_selfcheck() reports the mismatch count.
constexpr int TRIG_CHECK_N = 4096;
__global__ void k_trig_selfcheck(float *out) {
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (unsigned)TRIG_CHECK_N) return;
  // same sample formulas as the host side below (integers -> exact floats)
  const int a = (int)((i * 2654435761u) >> 9) - (1 << 22), b = (int)((i * 40503u + 12345u) * 2246822519u >> 9) - (1 << 22);
  out[i] = dev_atan2f((float)a, (float)b);
  const float ang = __fmul_rn((float)((int)i - TRIG_CHECK_N / 2), 0.0023f);   // about [-4.7, 4.7]
  out[TRIG_CHECK_N + i] = dev_sinf(ang);
}
static int g_trig_mismatch = -1;      // -1: not run yet
static std::once_flag g_trig_once;
static void trig_selfcheck_run() {
  float *dev = nullptr;
  static float host[2 * TRIG_CHECK_N];
  cudaStream_t st = nullptr;
  if (cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) != cudaSuccess) return;
  if (cudaMalloc(&dev, sizeof(host)) == cudaSuccess) {
    (void)launch(__FILE__, __LINE__, k_trig_selfcheck, (TRIG_CHECK_N + 255) / 256, 256, 0, st, dev);
    if (cudaMemcpyAsync(host, dev, sizeof(host), cudaMemcpyDeviceToHost, st) == cudaSuccess &&
        cudaStreamSynchronize(st) == cudaSuccess) {
      int bad = 0;
      for (unsigned i = 0; i < (unsigned)TRIG_CHECK_N; i++) {
        const int a = (int)((i * 2654435761u) >> 9) - (1 << 22), b = (int)((i * 40503u + 12345u) * 2246822519u >> 9) - (1 << 22);
        volatile float fa = (float)a, fb = (float)b;
        const float ra = atan2f(fa, fb);
        volatile float ang = (float)((int)i - TRIG_CHECK_N / 2) * 0.0023f;
        const float rs = sinf(ang);
        bad += memcmp(&ra, &host[i], 4) != 0;
        bad += memcmp(&rs, &host[TRIG_CHECK_N + i], 4) != 0;
      }
      g_trig_mismatch = bad;
      if (bad)
        fprintf(stderr,
                "grayskull_b200: warning: this host's libm sinf/atan2f differ from the glibc-2.39 routines the "
                "device restates (%d of %d samples); ORB angles/descriptors follow glibc 2.39 "
                "(gs_b200_set_trig_mode(1) selects CUDA libdevice, angle within 1e-5)\n",
                bad, 2 * TRIG_CHECK_N);
    }
    cudaFree(dev);
  }
  cudaStreamDestroy(st);
}
static void trig_selfcheck_once(cudaStream_t user) {
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(user, &cs) != cudaSuccess || cs != cudaStreamCaptureStatusNone) {
    cudaGetLastError();
    return;   // never allocate / synchronise inside a graph capture; the check runs on a later call
  }
  std::call_once(g_trig_once, trig_selfcheck_run);
}

static int fast_impl(const uint8_t *src, unsigned w, unsigned h, unsigned n, uint8_t *score, unsigned sw,
                     unsigned sh, KpRec *kps, unsigned *counts, unsigned nkps, unsigned threshold,
                     cudaStream_t s) {
  if (n == 0) return 0;
  if (w < 7 || h < 7) {  // no interior pixel: nothing written, no keypoints
    GSB_CHECK(cudaMemsetAsync(counts, 0, sizeof(unsigned) * n, s));
    return 0;
  }
  const unsigned rows = h - 6, mw = (w + 31) / 32;
  unsigned *rowcount = static_cast<unsigned *>(workspace(s, WS_FAST_A, sizeof(unsigned) * (size_t)rows * n));
  unsigned *masks = static_cast<unsigned *>(workspace(s, WS_FAST_B, sizeof(unsigned) * (size_t)rows * n * mw));
  if (!rowcount || !masks) return gsb::workspace_error();
  GSB_ASSERT(n <= 65535u && rows <= 0x7FFFFFFFu);
  // thresholds above 255 (the reference computes p + t / p - t in unsigned arithmetic, :496-498, which wraps for
  // huge t) take the literal per-pixel kernel: the tiled kernel's 16-bit lane arithmetic assumes t <= 255
  if (sw == w && sh == h && !force_generic() && threshold <= 255u) {
    // score + NMS mask in one kernel (k_fast_tiled2); the per-row counts are accumulated with atomics
    dim3 grid((w + FT_W - 1) / FT_W, (h - 6 + F2_TH - 1) / F2_TH, n);
    GSB_ASSERT(grid.y <= 65535u);
    GSB_CHECK(cudaMemsetAsync(rowcount, 0, sizeof(unsigned) * (size_t)rows * n, s));
    CUtensorMap tmap;
    const bool tiled = tma_ok(src, w) && tma_ok(score, w) && make_tmap_u8frames(&tmap, src, w, h, n, FT_SW / 4, F2_SH);
    if (!tiled) memset(&tmap, 0, sizeof(tmap));
    GSB_LAUNCH(tiled ? k_fast_tiled2<true> : k_fast_tiled2<false>, grid, F2_THREADS, 0, s, tmap, src, w, h, score, threshold,
               mw, masks, rowcount);
  } else {
    // foreign-sized score map (single-image gs_fast only), force_generic or t > 255: gs_set semantics per pixel,
    // then the NMS mask as a second pass
    dim3 block(32, 8), grid((w - 6 + 31) / 32, (h - 6 + 7) / 8, n);
    GSB_LAUNCH(k_fast_score, grid, block, 0, s, src, w, h, n, score, sw, sh, threshold);
    const bool words = sw % 4 == 0 && reinterpret_cast<uintptr_t>(score) % 4 == 0 && sw >= w && sh >= h;   // word pre-test stays inside the map
    GSB_LAUNCH(words ? k_nms_mask<true> : k_nms_mask<false>, dim3((rows + 7) / 8, n), 256, 0, s, score, sw, sh, w, h, mw, masks,
               rowcount);
  }
  GSB_LAUNCH(k_row_scan, n, 1024, 0, s, rowcount, rows, counts, nkps);
  const unsigned long long rows_total = (unsigned long long)rows * n;
  GSB_ASSERT(rows_total < 0x7FFFFFFFull);
  GSB_LAUNCH(k_nms_emit_masks, (unsigned)((rows_total + 7) / 8), 256, 0, s, score, sw, sh, w, h, mw, masks, rowcount,
             (unsigned)rows_total, kps, nkps);
  return 0;
}

}  // namespace gsb

extern "C" {

void gs_b200_set_trig_mode(int mode) { gsb::g_trig_mode = mode ? 1 : 0; }
int gs_b200_trig_selfcheck(void) {
  std::call_once(gsb::g_trig_once, gsb::trig_selfcheck_run);
  return gsb::g_trig_mismatch;
}

int gs_b200_fast_batch(const uint8_t *src, unsigned w, unsigned h, unsigned n, uint8_t *scoremap,
                       struct gs_keypoint *kps, unsigned *counts, unsigned nkps, unsigned threshold,
                       gs_b200_stream s) {
  GSB_ASSERT(src && w > 0 && h > 0 && kps && nkps > 0);  // reference :484
  GSB_ASSERT(scoremap && counts);
  return gsb::fast_impl(src, w, h, n, scoremap, w, h, reinterpret_cast<gsb::KpRec *>(kps), counts, nkps,
                        threshold, static_cast<cudaStream_t>(s));
}

int gs_b200_orb_extract_batch(const uint8_t *src, unsigned w, unsigned h, unsigned n, uint8_t *scoremap,
                              struct gs_keypoint *kps, unsigned *counts, unsigned nkps, unsigned threshold,
                              gs_b200_stream s) {
  GSB_ASSERT(src && w > 0 && h > 0 && kps && nkps > 0 && scoremap);  // reference :653
  GSB_ASSERT(counts);
  if (n == 0) return 0;
  cudaStream_t st = static_cast<cudaStream_t>(s);
  const unsigned cap = nkps * 4ull < gsb::ORB_MAXC ? nkps * 4 : gsb::ORB_MAXC;  // reference :656
  gsb::KpRec *cand = static_cast<gsb::KpRec *>(gsb::workspace(st, gsb::WS_ORB_A, sizeof(gsb::KpRec) * (size_t)cap * n));
  unsigned *ccount = static_cast<unsigned *>(gsb::workspace(st, gsb::WS_ORB_B, sizeof(unsigned) * n));
  if (!cand || !ccount) return gsb::workspace_error();
  int rc = gsb::fast_impl(src, w, h, n, scoremap, w, h, cand, ccount, cap, threshold, st);
  if (rc) return rc;
  GSB_LAUNCH(gsb::k_orb_select, n, 256, 0, st, cand, ccount, cap, w, h, reinterpret_cast<gsb::KpRec *>(kps), counts, nkps);
  const unsigned long long warps = (unsigned long long)n * nkps;
  const unsigned long long blocks = (warps + 7) / 8;
  GSB_ASSERT(blocks < 0x7FFFFFFFull);
  gsb::KpRec *kr = reinterpret_cast<gsb::KpRec *>(kps);
  if (gsb::g_trig_mode == 0) gsb::trig_selfcheck_once(st);
  GSB_LAUNCH(gsb::k_orb_moments, (unsigned)blocks, 256, 0, st, src, w, h, kr, counts, nkps, n);
  GSB_LAUNCH(gsb::k_orb_trig, (unsigned)((warps + 255) / 256), 256, 0, st, kr, counts, nkps, n, gsb::g_trig_mode);
  if (int rcb = gsb::brief_table_init(st)) return rcb;
  const bool words = w % 4 == 0 && reinterpret_cast<uintptr_t>(src) % 4 == 0 && !gsb::force_generic();
  GSB_LAUNCH(words ? gsb::k_orb_brief<true> : gsb::k_orb_brief<false>, (unsigned)blocks, 256, 0, st, src, w, h, kr, counts, nkps,
             n);
  return 0;
}

// internal hooks used by api.cu for the single-image calls
int gsb_fast_single(const uint8_t *src, unsigned w, unsigned h, uint8_t *score, unsigned sw, unsigned sh,
                    struct gs_keypoint *kps, unsigned *count, unsigned nkps, unsigned threshold, cudaStream_t s) {
  return gsb::fast_impl(src, w, h, 1, score, sw, sh, reinterpret_cast<gsb::KpRec *>(kps), count, nkps, threshold, s);
}
int gsb_orient_single(const uint8_t *img, unsigned w, unsigned x, unsigned y, unsigned r, float *out, cudaStream_t s) {
  if (gsb::g_trig_mode == 0) gsb::trig_selfcheck_once(s);
  GSB_LAUNCH(gsb::k_orient_one, 1, 32, 0, s, img, w, x, y, r, gsb::g_trig_mode, out);
  return 0;
}
int gsb_brief_single(const uint8_t *img, unsigned w, unsigned h, struct gs_keypoint *kp, cudaStream_t s) {
  if (gsb::g_trig_mode == 0) gsb::trig_selfcheck_once(s);
  GSB_LAUNCH(gsb::k_brief_one, 1, 32, 0, s, img, w, h, reinterpret_cast<gsb::KpRec *>(kp), gsb::g_trig_mode);
  return 0;
}
}
