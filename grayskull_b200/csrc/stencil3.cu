// stencil3.cu -- gs_sobel, gs_erode, gs_dilate (reference grayskull.h:285-320).
//
// HBM-bound 3x3 stencils: 1 B/pixel in, 1 B/pixel out.  At the roofline an H100 moves ~6
// pixels per SM clock, i.e. the whole kernel may spend only a few issue slots per pixel, so the
// arithmetic is done on 16-bit lane pairs (two pixels per 32-bit register):
//   * a TMA box (cp.async.bulk.tensor, zero-filled outside the image) stages a
//     288 x 130 byte tile (256 x 128 outputs + a 16-byte halo left and right, 1 row above and
//     below) into shared memory.  The inner start offset of a TMA box must be a multiple of
//     16 bytes, hence the 16-byte column halo;
//   * each warp owns a 16-row band, each lane 8 adjacent columns, and walks down the band
//     keeping the previous rows' partial results in registers;
//   * bytes are split into pair words P_k = (pixel x+k, pixel x+k+2) with PRMT/LOP; as fp16
//     *bit patterns* a byte b is the denormal b * 2^-24, and every value this kernel forms is
//     an integer below 2048 in those units, so HADD2/HFMA2 arithmetic on them is exact and the
//     result's bit pattern is the integer again.  Non-negative quantities are therefore added
//     with integer ops (ALU pipe) and signed ones with half2 ops (FMA pipe, |x| is a free
//     operand modifier), which balances the two issue pipes;
//   * Sobel uses (|gx| + |gy|) / 2 == max(|A|, |B|) with A = (gx + gy)/2, B = (gx - gy)/2,
//     both 6-tap +-1 sums, so no shift/rounding step is needed;
//   * erode/dilate use the native 3-input 16x2 min/max (VIMNMX3.U16x2).
// Widths that are not a multiple of 16 (TMA stride rule) or misaligned bases take the generic
// kernels at the bottom: one thread per pixel, reference semantics spelled out directly.
#include "common.cuh"
#include "pairs.cuh"

namespace gsb {

enum { OP_SOBEL = 0, OP_ERODE = 1, OP_DILATE = 2 };

constexpr int S3_TW = 256;                   // output tile width (pixels)
constexpr int S3_BH = 16;                    // rows per warp band
constexpr int S3_WARPS = 8;
constexpr int S3_TH = S3_BH * S3_WARPS;      // 128 output rows per tile
constexpr int S3_PW = 72;                    // smem row pitch in words: image bytes [x0-16, x0+272)
constexpr int S3_ROWS = S3_TH + 2;           // + 1 halo row above and below
constexpr unsigned S3_TILE_BYTES = S3_PW * 4 * S3_ROWS;

struct MorphRow {
  uint32_t h[4];  // horizontal 3-min / 3-max for the four output pair words
};
template <int OP>
__device__ __forceinline__ uint32_t mm3(uint32_t a, uint32_t b, uint32_t c) {
  return OP == OP_ERODE ? __vimin3_u16x2(a, b, c) : __vimax3_u16x2(a, b, c);
}
template <int OP>
__device__ __forceinline__ MorphRow morph_row(const Pairs &p) {
  MorphRow r;
  r.h[0] = mm3<OP>(p.m1, p.p0, p.p1);
  r.h[1] = mm3<OP>(p.p0, p.p1, p.p2);
  r.h[2] = mm3<OP>(p.p3, p.p4, p.p5);
  r.h[3] = mm3<OP>(p.p4, p.p5, p.p6);
  return r;
}
template <int OP>
__device__ __forceinline__ uint2 morph_out(const MorphRow &a, const MorphRow &b, const MorphRow &c) {
  uint32_t m[4];
#pragma unroll
  for (int k = 0; k < 4; k++) m[k] = mm3<OP>(a.h[k], b.h[k], c.h[k]);
  uint2 o;
  o.x = prmt(m[0], m[1], 0x6240);
  o.y = prmt(m[2], m[3], 0x6240);
  return o;
}

template <int OP>
struct RowT {
  typedef MorphRow type;
};
template <>
struct RowT<OP_SOBEL> {
  typedef SobelRow type;
};

template <int OP>
__global__ void __launch_bounds__(S3_WARPS * 32)
k_stencil3_tma(const __grid_constant__ CUtensorMap tmap, uint8_t *__restrict__ dst, unsigned w,
               unsigned h, unsigned tiles_x, unsigned tiles_y) {
  __shared__ __align__(128) uint32_t tile[S3_ROWS * S3_PW];
  __shared__ __align__(8) uint64_t bar;

  unsigned bid = blockIdx.x;
  const unsigned tx = bid % tiles_x;
  bid /= tiles_x;
  const unsigned ty = bid % tiles_y;
  const unsigned frame = bid / tiles_y;
  const int x0 = tx * S3_TW, y0 = ty * S3_TH;

  if (threadIdx.x == 0) {
    mbar_init(&bar, 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(&bar, S3_TILE_BYTES);
    tma_load_3d(tile, &tmap, x0 / 4 - 4, y0 - 1, frame, &bar);
  }

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int x = x0 + lane * 8;           // first of this lane's 8 columns
  const int yb = y0 + warp * S3_BH;      // first output row of this warp's band
  uint8_t *out = dst + (size_t)frame * w * h + x;

  mbar_wait(&bar, 0);
  if (x >= (int)w || yb >= (int)h) return;

  // erode must ignore out-of-image taps (reference :293); TMA filled them with 0, so they are
  // replaced by 255.  Column masks are per lane, row masks per (uniform) row.
  uint32_t fix_l = 0, fix_r = 0;
  if (OP == OP_ERODE) {
    if (x == 0) fix_l = 0xFFFFFFFFu;
    if (x + 8 >= (int)w) fix_r = 0xFFFFFFFFu;
  }
  const uint32_t *base = tile + (warp * S3_BH) * S3_PW + 2 * lane + 2;  // word of byte x-8

  typedef typename RowT<OP>::type Row;
  auto load_row = [&](int r, int yimg) -> Row {
    const uint32_t *p = base + r * S3_PW;
    uint32_t wl = p[1];
    uint2 wm = *reinterpret_cast<const uint2 *>(p + 2);
    uint32_t wr = p[4];
    if (OP == OP_ERODE) {
      wl |= fix_l, wr |= fix_r;
      if (yimg < 0 || yimg >= (int)h) wl = wm.x = wm.y = wr = 0xFFFFFFFFu;
    }
    Pairs pr = split_pairs(wl, wm.x, wm.y, wr);
    if constexpr (OP == OP_SOBEL) return sobel_row(pr);
    else return morph_row<OP>(pr);
  };

  // Sobel writes only the interior (reference :308-309): rows 1..h-2, columns 1..w-2
  const int ylo = OP == OP_SOBEL ? 1 : 0, yhi = OP == OP_SOBEL ? (int)h - 2 : (int)h - 1;
  const bool edge_l = OP == OP_SOBEL && x == 0, edge_r = OP == OP_SOBEL && x + 8 == (int)w;

  Row ra = load_row(0, yb - 1), rb = load_row(1, yb);
  uint8_t *q = out + (size_t)yb * w;
  auto emit = [&](const Row &a, const Row &b, const Row &c) {
    uint2 o;
    if constexpr (OP == OP_SOBEL) o = sobel_out(a, b, c);
    else o = morph_out<OP>(a, b, c);
    if (edge_l) o.x = (o.x & 0xFFFFFF00u) | q[0];                    // keep dst(0, y)
    if (edge_r) o.y = (o.y & 0x00FFFFFFu) | ((uint32_t)q[7] << 24);  // keep dst(w-1, y)
    st_cs_u2(q, o);
  };
  if (yb >= ylo && yb + S3_BH - 1 <= yhi) {   // whole band inside the written range: no row tests
#pragma unroll
    for (int i = 0; i < S3_BH; i++) {
      Row rc = load_row(i + 2, yb + i + 1);
      emit(ra, rb, rc);
      q += w;
      ra = rb;
      rb = rc;
    }
  } else {
#pragma unroll 1
    for (int i = 0; i < S3_BH; i++) {
      const int y = yb + i;
      if (y > yhi) break;
      Row rc = load_row(i + 2, y + 1);
      if (y >= ylo) emit(ra, rb, rc);
      q += w;
      ra = rb;
      rb = rc;
    }
  }
}

// ---- generic kernels: any width / alignment, one thread per pixel ----------------------------
template <int OP>
__global__ void k_stencil3_generic(uint8_t *__restrict__ dst, const uint8_t *__restrict__ src,
                                   unsigned w, unsigned h, unsigned n) {
  const unsigned x = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= w || y >= h) return;
  for (unsigned f = blockIdx.z; f < n; f += gridDim.z) {
    const uint8_t *s = src + (size_t)f * w * h;
    uint8_t *d = dst + (size_t)f * w * h;
    if (OP == OP_SOBEL) {
      if (x == 0 || y == 0 || x + 1 >= w || y + 1 >= h) continue;
      const uint8_t *a = s + (size_t)(y - 1) * w + x, *b = a + w, *c = b + w;
      int gx = -a[-1] + a[1] - 2 * b[-1] + 2 * b[1] - c[-1] + c[1];
      int gy = -a[-1] - 2 * a[0] - a[1] + c[-1] + 2 * c[0] + c[1];
      int m = (abs(gx) + abs(gy)) / 2;
      d[(size_t)y * w + x] = (uint8_t)min(m, 255);
    } else {
      int v = OP == OP_ERODE ? 255 : 0;
      for (int dy = -1; dy <= 1; dy++)
        for (int dx = -1; dx <= 1; dx++) {
          int yy = (int)y + dy, xx = (int)x + dx;
          if (yy < 0 || yy >= (int)h || xx < 0 || xx >= (int)w) continue;
          int p = s[(size_t)yy * w + xx];
          v = OP == OP_ERODE ? min(v, p) : max(v, p);
        }
      d[(size_t)y * w + x] = (uint8_t)v;
    }
  }
}

template <int OP>
static int launch_stencil3(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n,
                           cudaStream_t s) {
  if (n == 0) return 0;
  if (OP == OP_SOBEL && (w < 3 || h < 3)) return 0;  // nothing is written (reference :308-309)
  CUtensorMap tmap;
  if (tma_ok(src, w) && tma_ok(dst, w) && make_tmap_u8frames(&tmap, src, w, h, n, S3_PW, S3_ROWS)) {
    const unsigned tiles_x = (w + S3_TW - 1) / S3_TW, tiles_y = (h + S3_TH - 1) / S3_TH;
    const unsigned long long blocks = (unsigned long long)tiles_x * tiles_y * n;
    GSB_ASSERT(blocks < 0x7FFFFFFFull);
    GSB_LAUNCH(k_stencil3_tma<OP>, (unsigned)blocks, S3_WARPS * 32, 0, s, tmap, dst, w, h, tiles_x, tiles_y);
  } else {
    dim3 block(32, 8), grid((w + 31) / 32, (h + 7) / 8, n < 65535u ? n : 65535u);
    GSB_LAUNCH(k_stencil3_generic<OP>, grid, block, 0, s, dst, src, w, h, n);
  }
  return 0;
}

}  // namespace gsb

extern "C" {
int gs_b200_sobel_batch(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n,
                        gs_b200_stream s) {
  GSB_ASSERT(dst && src && w > 0 && h > 0);  // gs_valid(dst) && gs_valid(src), reference :307
  return gsb::launch_stencil3<gsb::OP_SOBEL>(dst, src, w, h, n, static_cast<cudaStream_t>(s));
}
int gs_b200_erode_batch(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n,
                        gs_b200_stream s) {
  GSB_ASSERT(dst && src && w > 0 && h > 0);  // reference :287
  return gsb::launch_stencil3<gsb::OP_ERODE>(dst, src, w, h, n, static_cast<cudaStream_t>(s));
}
int gs_b200_dilate_batch(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n,
                         gs_b200_stream s) {
  GSB_ASSERT(dst && src && w > 0 && h > 0);  // reference :287
  return gsb::launch_stencil3<gsb::OP_DILATE>(dst, src, w, h, n, static_cast<cudaStream_t>(s));
}
}
