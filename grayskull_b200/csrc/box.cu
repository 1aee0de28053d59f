// box.cu -- gs_blur and gs_adaptive_threshold (reference grayskull.h:230-247, 268-283).
//
// Both need mean = floor(S / count), S = sum of the (2r+1)^2 window clipped to the image,
// count = number of in-image taps = (#in-image columns) * (#in-image rows).  2 B/pixel of
// compulsory HBM traffic regardless of the radius, so the kernel must stay under ~10 issue
// slots per pixel.  Fast path (radius 1..7, width % 16 == 0); no block-level barrier after the
// tile has landed, every warp is independent:
//   0. one TMA box loads a 256-column x (BH*warps + 2r)-row byte tile; outside the image reads
//      as 0, which is exactly the contribution of a clipped tap to the SUM.  Boxes start on
//      16-byte boundaries, tiles are laid out with a 240-pixel
//      stride: lanes 0 and 31 of a warp only contribute column sums, lanes 1..30 produce the
//      240 outputs, so no cross-warp exchange is ever needed;
//   1. vertical: a lane keeps the running column sums of its 8 columns as four u16x2 words
//      (adjacent-pixel pairs) and rolls them down its band with one IADD3 per word per row
//      (sum + entering row - leaving row on both 16-bit lanes at once: no lane can borrow
//      because every true lane value is in [0, 65535]);
//   2. horizontal: the neighbours' column sums come by warp shuffle; the (2r+1)-wide window
//      sums for two adjacent pixels are formed on 16-bit lane pairs from a rolling sum of pair
//      words (4 integer ops per 2 pixels, radius independent); max (2*7+1)^2*255 = 57375 < 65536;
//   3. exact division without integer divide: with m = ceil(2^24 / count),
//        fma_rd(float(S), m * 2^-24, 2^23) = 2^23 + floor(S * m / 2^24)
//      is computed exactly before its single round-down, and floor(S*m/2^24) == S / count for
//      all S <= 255 * count, count <= 225 (checked exhaustively in tests/test_host_logic.py);
//      the quotient is the low byte of the float's bit pattern.  float(S) comes straight from
//      either 16-bit half on the conversion pipe (I2F.U16): the kernel was ALU-pipe bound, so the
//      byte packing and the lane-total broadcast are multiply-adds (FMA pipe) for the same reason.  Tiles whose windows all lie
//      inside the image use compile-time constants for count = (2r+1)^2 on a branch-free path,
//      clipped pixels a 226-entry table.
// Other radii / widths take the generic kernel (one thread per pixel, any radius).
#include <limits.h>
#include <string.h>

#include <type_traits>

#include "common.cuh"
#include "pairs.cuh"

namespace gsb {

constexpr int BX_STRIDE = 240;             // output columns per tile (lanes 1..30 x 8 pixels)
constexpr int BX_PW = 64;                  // tile pitch in 32-bit words: image bytes [x0-16, x0+240)
constexpr int BX_RMAX = 7;
constexpr int BX_WARPS = 4;                // warps per CTA, one row band each
constexpr int BX_BH = 32;                  // rows per band
constexpr int BX_TH = BX_WARPS * BX_BH;    // 128 output rows per tile
constexpr int BX_THREADS = BX_WARPS * 32;
constexpr int BX_TILE_WORDS = BX_PW * (BX_TH + 2 * BX_RMAX);
constexpr int BX_SMEM = BX_TILE_WORDS * 4 + 226 * 8 + 16;

struct DivMagic {
  float inv, k;
};
__host__ __device__ inline DivMagic div_magic(unsigned count) {
  unsigned m = (16777216u + count - 1u) / count;          // ceil(2^24 / count) <= 2^24: exact float
  DivMagic d;
  d.inv = (float)m * 5.9604644775390625e-08f;             // m * 2^-24, exact
  d.k = 8388608.0f - 0.5f * (float)m;                     // 2^23 - m/2, exact (|.| < 2^23, ulp 0.5)
  return d;
}

// floor(s / count) for the low 16-bit lane s of t, as the low byte of the returned bit pattern: float(s) straight
// from the half on the conversion pipe (I2F.U16, exact), then fma_rd(S, m*2^-24, 2^23) = 2^23 + floor(S*m/2^24)
__device__ __forceinline__ uint32_t div_lo(uint32_t t, float inv) {
  float fl;
  asm("{ .reg .b16 lo, hi; mov.b32 {lo, hi}, %1; cvt.rn.f32.u16 %0, lo; }" : "=f"(fl) : "r"(t));
  return __float_as_uint(__fmaf_rd(fl, inv, 8388608.0f));
}
// the same for the high lane
__device__ __forceinline__ uint32_t div_hi(uint32_t t, float inv) {
  float fh;
  asm("{ .reg .b16 lo, hi; mov.b32 {lo, hi}, %1; cvt.rn.f32.u16 %0, hi; }" : "=f"(fh) : "r"(t));
  return __float_as_uint(__fmaf_rd(fh, inv, 8388608.0f));
}
// low bytes of four 2^23+q floats -> one word; the two 8-bit merges are multiply-adds (FMA pipe)
__device__ __forceinline__ uint32_t pack4(uint32_t q0, uint32_t q1, uint32_t q2, uint32_t q3) {
  uint32_t a, b;
  asm("mad.lo.u32 %0, %1, 256, %2;" : "=r"(a) : "r"(q1), "r"(q0));   // low 16 bits = q0 | q1 << 8
  asm("mad.lo.u32 %0, %1, 256, %2;" : "=r"(b) : "r"(q3), "r"(q2));
  return prmt(a, b, 0x5410);
}

// window sums for 4 output pixel pairs from 12 pair words V[m] = (s_2m, s_2m+1), s_i = column
// sum of image column x - 8 + i; output pair p = pixels (x+2p, x+2p+1).
template <int R>
__device__ __forceinline__ void window_sums(const uint32_t (&V)[12], uint32_t (&T)[4]) {
  constexpr bool ODD = (R & 1) != 0;
  constexpr int NP = ODD ? R : R + 1;
  constexpr int A0 = 8 - R;
  constexpr int M0 = ODD ? (A0 + 1) / 2 : A0 / 2;
  uint32_t ps = V[M0];
#pragma unroll
  for (int i = 1; i < NP; i++) ps += V[M0 + i];
#pragma unroll
  for (int p = 0; p < 4; p++) {
    const int m = M0 + p;
    // lane totals by IMAD (FMA pipe; the ALU pipe is the busy one): (ps * 0x10001) >> 16 = lane0 + lane1
    // (<= 57375, no carry out); * 0x10001 puts it in both lanes
    uint32_t x16, tot;
    asm("mad.lo.u32 %0, %1, 0x10001, 0;" : "=r"(x16) : "r"(ps));
    x16 >>= 16;
    if (ODD) {
      const uint32_t edge = prmt(V[m - 1], V[m + NP], 0x5432);
      asm("mad.lo.u32 %0, %1, 0x10001, %2;" : "=r"(tot) : "r"(x16), "r"(edge));
      T[p] = tot;
    } else {
      asm("mad.lo.u32 %0, %1, 0x10001, 0;" : "=r"(tot) : "r"(x16));
      T[p] = tot - prmt(V[m + R], V[m], 0x5432);
    }
    if (p < 3) ps = ps + V[m + NP] - V[m];
  }
}

// division of one row of 8 pixels from its 4 window-sum pair words: q[i] = bits of the float 2^23 + mean of pixel i
template <int R, bool INTERIOR>
__device__ __forceinline__ void box_quot(const uint32_t (&T)[4], const int (&cw)[8], int ch, const float2 *__restrict__ magic,
                                         uint32_t (&q)[8]) {
  constexpr int FULL = 2 * R + 1;
  constexpr float FINV = (float)((16777216u + FULL * FULL - 1u) / (FULL * FULL)) * 5.9604644775390625e-08f;
  if (INTERIOR) {
#pragma unroll
    for (int p = 0; p < 4; p++) {
      q[2 * p] = div_lo(T[p], FINV);
      q[2 * p + 1] = div_hi(T[p], FINV);
    }
  } else {
#pragma unroll
    for (int p = 0; p < 4; p++) {
      const float2 m0 = magic[cw[2 * p] * ch], m1 = magic[cw[2 * p + 1] * ch];
      q[2 * p] = div_lo(T[p], m0.x);
      q[2 * p + 1] = div_hi(T[p], m1.x);
    }
  }
}

// division + (threshold +) packing of one row of 8 pixels from its 4 window-sum pair words
template <int R, bool ADAPTIVE, bool INTERIOR>
__device__ __forceinline__ uint2 box_finish(const uint32_t (&T)[4], uint2 srcpx, const int (&cw)[8], int ch,
                                            const float2 *__restrict__ magic, int cparam) {
  uint32_t q[8];
  box_quot<R, INTERIOR>(T, cw, ch, magic, q);
  uint2 o;
  if (ADAPTIVE) {
    // dst = src > (int)mean - c ? 255 : 0   (reference :244-245), two pixels per 16-bit lane pair:
    // E = src + (c + 0x7FFF) - mean has bit 15 set exactly when src > mean - c, with c clamped to
    // [-256, 256]: exact for every c > INT_MIN + 255.  Below that, (int)(mean - (unsigned)c) wraps
    // negative for large means and the reference writes 255 there; launch_box routes that range to
    // k_box_wide / k_box_generic, which evaluate the expression literally.  A sign-replicating PRMT
    // turns the four bit-15s into 0x00 / 0xFF bytes.  q = 0x4B0000mm, so bytes 1 of q are zero.
    const int cc = max(-256, min(256, cparam));
    const uint32_t kc = (uint32_t)(cc + 0x7FFF) * 0x10001u;
    uint32_t e[4];
#pragma unroll
    for (int p = 0; p < 4; p++) {
      const uint32_t m = prmt(q[2 * p], q[2 * p + 1], 0x5410);                 // (mean_2p, mean_2p+1)
      const uint32_t sw = p < 2 ? srcpx.x : srcpx.y;
      const uint32_t sp = prmt(sw, 0, (p & 1) ? 0x4342 : 0x4140);              // (src_2p, src_2p+1)
      e[p] = sp + kc - m;
    }
    o.x = prmt_raw(e[0], e[1], 0xFDB9);
    o.y = prmt_raw(e[2], e[3], 0xFDB9);
  } else {
    o.x = pack4(q[0], q[1], q[2], q[3]);
    o.y = pack4(q[4], q[5], q[6], q[7]);
  }
  return o;
}

// bytes (b0..b7) of two words -> adjacent-pixel pair words (b0,b1) (b2,b3) (b4,b5) (b6,b7)
__device__ __forceinline__ void unpack_pairs(uint2 v, uint32_t (&p)[4]) {
  p[0] = prmt(v.x, 0, 0x4140), p[1] = prmt(v.x, 0, 0x4342);
  p[2] = prmt(v.y, 0, 0x4140), p[3] = prmt(v.y, 0, 0x4342);
}

template <int R, bool ADAPTIVE>
__global__ void __launch_bounds__(BX_THREADS)
k_box_tma(const __grid_constant__ CUtensorMap tmap, uint8_t *__restrict__ dst, unsigned w, unsigned h, int cparam) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  uint32_t *tile = reinterpret_cast<uint32_t *>(smem_raw);
  float2 *magic = reinterpret_cast<float2 *>(smem_raw + BX_TILE_WORDS * 4);
  uint64_t &bar = *reinterpret_cast<uint64_t *>(smem_raw + BX_TILE_WORDS * 4 + 226 * 8);
  constexpr int ROWS = BX_TH + 2 * R;
  constexpr int FULL = 2 * R + 1;

  const unsigned frame = blockIdx.z;
  const int xb = (int)blockIdx.x * BX_STRIDE - 16;   // image column of tile byte 0 (16-B aligned)
  const int y0 = (int)blockIdx.y * BX_TH;
  // every window of this tile's outputs lies inside the image: no clipping, no partial rows/cols
  const bool interior = xb + 8 - R >= 0 && xb + 8 + BX_STRIDE - 1 + R <= (int)w - 1 && y0 - R >= 0 &&
                        y0 + BX_TH - 1 + R <= (int)h - 1;
  if (threadIdx.x == 0) {
    mbar_init(&bar, 1);
    mbar_fence_init();
  }
  if (!interior) {                                            // clipped-count division table
    for (unsigned c = threadIdx.x + 1; c < 226; c += BX_THREADS) {
      const DivMagic d = div_magic(c);
      magic[c] = make_float2(d.inv, d.k);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(&bar, BX_PW * 4 * ROWS);
    tma_load_3d(tile, &tmap, xb / 4, y0 - R, frame, &bar);
  }

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int x = xb + 8 * lane;                 // first of this lane's 8 columns
  const int yb = y0 + warp * BX_BH;            // first output row of this warp's band
  const bool out_lane = lane >= 1 && lane <= 30 && x >= 0 && x < (int)w;
  const uint32_t *in = tile + (warp * BX_BH) * BX_PW + 2 * lane;   // tile row of image row yb - R
  uint8_t *outp = dst + (size_t)frame * w * h + (size_t)yb * w + x;
  int cw[8];
#pragma unroll
  for (int j = 0; j < 8; j++) cw[j] = out_lane ? min(x + j + R, (int)w - 1) - max(x + j - R, 0) + 1 : 1;

  mbar_wait(&bar, 0);
  if (yb >= (int)h) return;                    // warp-uniform

  uint32_t S[4] = {0, 0, 0, 0};                // column sums of the 2R rows above the next window row
  // interior tiles (fully unrolled walk): the unpacked pair words of the 2R+1 rows in the window stay in a register
  // ring, so the row that leaves is not loaded and unpacked a second time (one LDS.64 + four PRMT per row step)
  uint32_t ring[2 * R + 1][4];
#pragma unroll
  for (int i = 0; i < 2 * R; i++) {
    uint32_t e[4];
    unpack_pairs(*reinterpret_cast<const uint2 *>(in + i * BX_PW), e);
#pragma unroll
    for (int k = 0; k < 4; k++) {
      S[k] += e[k];
      ring[i][k] = e[k];
    }
  }
  uint32_t L[4] = {0, 0, 0, 0};                // the row that leaves the window at this step

  auto row_step = [&](int i, auto interior_tag) {
    constexpr bool INT = decltype(interior_tag)::value;
    uint32_t e[4];
    unpack_pairs(*reinterpret_cast<const uint2 *>(in + (i + 2 * R) * BX_PW), e);
#pragma unroll
    for (int k = 0; k < 4; k++) S[k] = S[k] + e[k] - L[k];   // one IADD3 per word
    if (INT) {
#pragma unroll
      for (int k = 0; k < 4; k++) {
        ring[(i + 2 * R) % (2 * R + 1)][k] = e[k];
        L[k] = ring[i % (2 * R + 1)][k];
      }
    } else {
      unpack_pairs(*reinterpret_cast<const uint2 *>(in + i * BX_PW), L);
    }
    // column sums of columns x-8 .. x+15 as pair words V[0..11]; V[4..7] are this lane's own
    uint32_t V[12], T[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
      V[4 + k] = S[k];
      V[k] = (R == 7 || k > 0) ? __shfl_up_sync(0xFFFFFFFFu, S[k], 1) : 0u;
      V[8 + k] = (R == 7 || k < 3) ? __shfl_down_sync(0xFFFFFFFFu, S[k], 1) : 0u;
    }
    window_sums<R>(V, T);
    uint2 srcpx = make_uint2(0, 0);
    if (ADAPTIVE) srcpx = *reinterpret_cast<const uint2 *>(in + (i + R) * BX_PW);
    int ch = FULL;
    if (!INT) {
      const int y = yb + i;
      ch = min(y + R, (int)h - 1) - max(y - R, 0) + 1;
    }
    const uint2 o = box_finish<R, ADAPTIVE, INT>(T, srcpx, cw, ch, magic, cparam);
    if (out_lane) st_cs_u2(outp, o);
    outp += w;
  };

  if (interior) {
#pragma unroll
    for (int i = 0; i < BX_BH; i++) row_step(i, std::true_type{});
  } else {
#pragma unroll 1
    for (int i = 0; i < BX_BH; i++) {
      if (yb + i >= (int)h) break;             // warp-uniform
      row_step(i, std::false_type{});
    }
  }
}



// ---- fused gs_blur(r) -> gs_sobel: the blurred frame never goes to HBM ------------------------
// gs_b200_blur_sobel_batch(dst, src, r) == gs_blur(tmp, src, r); gs_sobel(dst, tmp) bit for bit (dst's 1-px
// frame untouched, like gs_sobel), with 1 B/px read + 1 B/px written instead of 4 B/px.  A CTA makes 240 sobel
// columns x BS_TH rows in two phases with one barrier between them:
//   A. blur on the tensor cores.  One TMA box loads input bytes [xb, xb + 272) x rows [Y - 8, Y + BS_BROWS + 8),
//      Y = the tile's first blurred row; outside the image reads as 0, a clipped tap's contribution to the sum.  A
//      warp walks 16-column strips (blurred columns [c0, c0 + 16), c0 = xb + 8 + 16 s) down the tile:
//      1. horizontal sums, transposed: H^T = Bh * img with mma.m16n8k32.u8 (A = the constant 0/1 band, 16 output
//         columns x 32 input columns [c0 - 8, c0 + 24), enough for R <= 8; B = 8 image rows, one LDS.32 per register:
//         a thread's 4 bytes are consecutive bytes of one row).  H <= 15 * 255 = 3825;
//      2. H = 256 hi + lo with hi <= 14.  Two such 8-row tiles (a "pair", 16 H rows) hold in each thread exactly the
//         B fragment of a second MMA over 16 k slots per column (rows 2t, 2t+1 of each tile): four PRMT per column
//         give its lo and hi operand registers, and the slot order is baked into the constant A of that MMA;
//      3. vertical sums: S = Bv * H for 16 blurred rows from the 32 H rows of two pairs (A = the constant band over
//         the permuted slots), once for lo and once for hi.  A step advances 16 rows, so each pair is made once and
//         used by two steps.  The lo MMA accumulates onto C = 0x4B000000, so IMAD(D_hi, 256, D_lo) is the bit
//         pattern of the float 2^23 + S (S <= 57375; the MMA sums are exact integers);
//      4. exact division on the FMA pipe: fma_rd(2^23 + S, m 2^-24, 2^23 - m/2) = 2^23 + floor(S m / 2^24), the same
//         real value as k_box_tma's fma_rd(S, m 2^-24, 2^23) and rounded once (see div_magic); a strip with a clipped
//         window anywhere takes each pixel's (inv, k) from the 226-entry table;
//      5. two quotients of a row are adjacent columns of the MMA's D fragment: one IMAD packs their low bytes, one
//         STS.U16 stores them to the blurred tile.
//   B. sobel from the blurred tile, as k_stencil3_tma: each warp walks a 16-row band, each lane 8 columns, with the
//      previous two rows' partials in registers (pairs.cuh).  The lanes holding column 0 or w-1 keep dst's byte
//      there by writing the other seven bytes as three stores, so the kernel never reads dst.
// Blurred pixels outside the image (garbage counts, quotients possibly > 255) come in whole rows or in column pairs
// (2j, 2j+1) that the packing keeps together, and feed only sobel outputs that are never written.
constexpr int BS_STRIDE = 240;                 // sobel columns per tile (lanes 0..29 x 8 pixels)
constexpr int BS_PW = 68;                      // tile pitch in words: 68 = 4 mod 32, conflict-free MMA operand loads
constexpr int BS_STEPS = 8;                    // 16-row blur steps per tile
constexpr int BS_WARPS = 8;
constexpr int BS_THREADS = BS_WARPS * 32;
constexpr int BS_BROWS = 16 * BS_STEPS;        // blurred rows per tile
constexpr int BS_TH = BS_BROWS - 2;            // sobel rows per tile
constexpr int BS_IN_ROWS = BS_BROWS + 16;      // input rows: 8 above and below the blurred rows
constexpr int BS_STRIPS = 16;                  // 16-column blur strips: blurred columns [xb + 8, xb + 264)
constexpr int BS_IN_BYTES = BS_PW * 4 * BS_IN_ROWS;
constexpr int BS_BL_BYTES = BS_PW * 4 * BS_BROWS;
constexpr int BS_SMEM = BS_IN_BYTES + BS_BL_BYTES + 226 * 8 + 16;
static_assert(BS_IN_BYTES % 128 == 0, "the blurred tile follows the TMA destination");
static_assert(BS_TH % 16 == 14, "phase B: the last warp's band is 14 rows");

// div_magic of every count 1..225 as a compile-time table: a tile with clipped windows copies it to shared memory
// (the integer division of div_magic would put I2F / MUFU work in the kernel's prologue)
struct DivMagicTable {
  float2 e[226];
};
constexpr DivMagicTable make_div_magic_table() {
  DivMagicTable t{};
  for (unsigned c = 1; c < 226; c++) {
    const unsigned m = (16777216u + c - 1u) / c;
    t.e[c].x = (float)m * 5.9604644775390625e-08f;
    t.e[c].y = 8388608.0f - 0.5f * (float)m;
  }
  return t;
}
__constant__ DivMagicTable c_div_magic = make_div_magic_table();

// D (+)= A (16x32 u8, row) * B (32x8 u8, col), s32 accumulators
__device__ __forceinline__ void mma_u8(uint32_t (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1, uint32_t c) {
  asm("mma.sync.aligned.m16n8k32.row.col.s32.u8.u8.s32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%10, %10, %10, %10};"
      : "=r"(d[0]), "=r"(d[1]), "=r"(d[2]), "=r"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1), "r"(c));
}
__device__ __forceinline__ uint32_t imad256(uint32_t hi, uint32_t lo) {   // hi * 256 + lo on the FMA pipe
  uint32_t d;
  asm("mad.lo.u32 %0, %1, 256, %2;" : "=r"(d) : "r"(hi), "r"(lo));
  return d;
}

// the 8 output bytes of a lane whose first byte is image column 0 (left) or whose last is column w-1 (!left): the
// other seven bytes as three aligned stores, so that dst's border byte stays as it was without being read
__device__ __forceinline__ void st_cs_7of8(uint8_t *p, uint2 v, bool left) {
  if (left) {
    asm volatile("st.global.cs.u8 [%0], %1;" ::"l"(p + 1), "r"(v.x >> 8) : "memory");
    asm volatile("st.global.cs.u16 [%0], %1;" ::"l"(p + 2), "r"(v.x >> 16) : "memory");
    asm volatile("st.global.cs.u32 [%0], %1;" ::"l"(p + 4), "r"(v.y) : "memory");
  } else {
    asm volatile("st.global.cs.u32 [%0], %1;" ::"l"(p), "r"(v.x) : "memory");
    asm volatile("st.global.cs.u16 [%0], %1;" ::"l"(p + 4), "r"(v.y) : "memory");
    asm volatile("st.global.cs.u8 [%0], %1;" ::"l"(p + 6), "r"(v.y >> 16) : "memory");
  }
}

template <int R>
__global__ void __launch_bounds__(BS_THREADS, 3)
k_blur_sobel_tma(const __grid_constant__ CUtensorMap tmap, uint8_t *__restrict__ dst, unsigned w, unsigned h) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const uint32_t *in = reinterpret_cast<const uint32_t *>(smem_raw);          // input row i = image row Y - 8 + i
  unsigned char *bl = smem_raw + BS_IN_BYTES;                                 // blurred row i = image row Y + i
  float2 *magic = reinterpret_cast<float2 *>(smem_raw + BS_IN_BYTES + BS_BL_BYTES);
  uint64_t &bar = *reinterpret_cast<uint64_t *>(smem_raw + BS_IN_BYTES + BS_BL_BYTES + 226 * 8);
  constexpr int FULL = 2 * R + 1;
  constexpr unsigned FM = (16777216u + FULL * FULL - 1u) / (FULL * FULL);
  constexpr float FINV = (float)FM * 5.9604644775390625e-08f, FK = 8388608.0f - 0.5f * (float)FM;   // div_magic

  const unsigned frame = blockIdx.z;
  const int xb = (int)blockIdx.x * BS_STRIDE - 16;   // image column of tile byte 0 (16-B aligned)
  const int y0 = (int)blockIdx.y * BS_TH;            // first sobel row of the tile
  const int Y = y0 - 1;                              // first blurred row
  if (threadIdx.x == 0) {
    mbar_init(&bar, 1);
    mbar_fence_init();
    mbar_expect_tx(&bar, BS_IN_BYTES);
    tma_load_3d(smem_raw, &tmap, xb / 4, Y - 8, frame, &bar);
  }
  // the clipped-count division table, only in tiles with a clipped blurred pixel; built while the tile is in flight
  if (Y - R < 0 || Y + BS_BROWS - 1 + R > (int)h - 1 || xb + 8 - R < 0 || xb + 8 + 16 * BS_STRIPS - 1 + R > (int)w - 1) {
    for (unsigned c = threadIdx.x + 1; c < 226; c += BS_THREADS) magic[c] = c_div_magic.e[c];
  }
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;             // MMA fragment coordinates
  // the constant A operands: ah = horizontal band (row = output column c, k = input column c0 - 8 + k), av = vertical
  // band (row = blurred row y of the step, k = H row slot; slot 4t'+i of a pair holds tile i>>1, row 2t' + (i&1))
  uint32_t ah[4], av[4];
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const int row = g + 8 * (j & 1), kb = 16 * (j >> 1) + 4 * t;
    uint32_t a = 0, v = 0;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int k = kb + i;
      const int hrow = (k >> 4) * 16 + ((k >> 1) & 1) * 8 + 2 * ((k >> 2) & 3) + (k & 1);   // relative to y - 8
      a |= (uint32_t)(abs(k - 8 - row) <= R) << (8 * i);
      v |= (uint32_t)(abs(hrow - 8 - row) <= R) << (8 * i);
    }
    ah[j] = a, av[j] = v;
  }

  // built once per thread (the compiler would rebuild them per strip)
#pragma unroll
  for (int j = 0; j < 4; j++) asm("" : "+r"(ah[j]), "+r"(av[j]));
  // interior division constants, in registers (FFMA takes one immediate)
  float finv = FINV, fk = FK;
  asm("" : "+f"(finv), "+f"(fk));
  const bool rows_full = Y - R >= 0 && Y + BS_BROWS - 1 + R <= (int)h - 1;

  mbar_wait(&bar, 0);

  // ---- phase A: blurred tile
  for (int s = warp; s < BS_STRIPS; s += BS_WARPS) {
    const int c0 = xb + 8 + 16 * s;                  // image column of the strip's first blurred column
    if (c0 >= (int)w) break;                         // warp-uniform
    const uint32_t *ip = in + g * BS_PW + 4 * s + t;
    unsigned char *bp = bl + g * (BS_PW * 4) + 16 * s + 2 * t;
    const bool cols_full = c0 - R >= 0 && c0 + 15 + R <= (int)w - 1;
    // clipped column counts of the thread's four columns c0 + 8 hh + 2t + e
    int cw[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int c = c0 + 8 * (j >> 1) + 2 * t + (j & 1);
      cw[j] = max(min(c + R, (int)w - 1) - max(c - R, 0) + 1, 1);
    }
    // lo / hi operands of a pair of 8-row H tiles (input rows 16 p .. 16 p + 15), both column halves
    auto make_pair = [&](int p, uint32_t (&o)[4]) {
      uint32_t P[4], Q[4];
      const uint32_t *r0 = ip + 16 * p * BS_PW, *r1 = r0 + 8 * BS_PW;
      mma_u8(P, ah, r0[0], r0[4], 0u);
      mma_u8(Q, ah, r1[0], r1[4], 0u);
#pragma unroll
      for (int hh = 0; hh < 2; hh++) {
        const uint32_t x = prmt(P[2 * hh], P[2 * hh + 1], 0x5140), y = prmt(Q[2 * hh], Q[2 * hh + 1], 0x5140);
        o[2 * hh] = prmt(x, y, 0x5410);        // lo bytes
        o[2 * hh + 1] = prmt(x, y, 0x7632);    // hi bytes
      }
    };
    // pairs u and u+1 in registers pa / pb: pair u + 1 overwrites pair u - 1, so the MMA's B operand is (pa, pb) at
    // every step, and odd steps take the band with its two k halves swapped (slots 0..15 = pair u + 1)
    uint32_t pa[4], pb[4];
    make_pair(0, pa);
    auto walk = [&](auto full_tag) {
      constexpr bool FULLW = decltype(full_tag)::value;
#pragma unroll
      for (int u = 0; u < BS_STEPS; u++) {
        const int yu = Y + 16 * u;
        if (yu >= (int)h) break;                     // warp-uniform: blurred rows below the image are never used
        make_pair(u + 1, pb);
        int ch[2] = {FULL, FULL};
        if (!FULLW) {
#pragma unroll
          for (int e = 0; e < 2; e++) {
            const int y = yu + g + 8 * e;
            ch[e] = max(min(y + R, (int)h - 1) - max(y - R, 0) + 1, 1);
          }
        }
#pragma unroll
        for (int hh = 0; hh < 2; hh++) {
          uint32_t dl[4], dh[4];
          mma_u8(dl, av, pa[2 * hh], pb[2 * hh], 0x4B000000u);
          mma_u8(dh, av, pa[2 * hh + 1], pb[2 * hh + 1], 0u);
          uint32_t q[4];
#pragma unroll
          for (int j = 0; j < 4; j++) {             // D element j: row g + 8 (j >> 1), column 8 hh + 2t + (j & 1)
            float inv = finv, k = fk;
            if (!FULLW) {
              const float2 m = magic[cw[2 * hh + (j & 1)] * ch[j >> 1]];
              inv = m.x, k = m.y;
            }
            q[j] = __float_as_uint(__fmaf_rd(__uint_as_float(imad256(dh[j], dl[j])), inv, k));
          }
          unsigned char *o = bp + 16 * u * (BS_PW * 4) + 8 * hh;
          *reinterpret_cast<uint16_t *>(o) = (uint16_t)imad256(q[1], q[0]);
          *reinterpret_cast<uint16_t *>(o + 8 * (BS_PW * 4)) = (uint16_t)imad256(q[3], q[2]);
        }
#pragma unroll
        for (int j = 0; j < 4; j++) pa[j] = pb[j];
      }
    };
    // windows clipped anywhere in the strip: per-pixel counts from the table
    if (cols_full && rows_full) walk(std::true_type{});
    else walk(std::false_type{});
  }
  __syncthreads();

  // ---- phase B: sobel rows y0 + 16 warp .. + nb - 1 from blurred rows one above to one below
  const int r0 = 16 * warp, nb = min(16, BS_TH - r0);
  const int x = xb + 16 + 8 * lane;
  const int yb = y0 + r0;
  const bool live = lane < 30 && x < (int)w;
  const bool edge_l = x == 0, edge_r = x + 8 == (int)w;
  // a warp with a lane on column 0 or w-1 walks its own copy, so that the others keep the single 64-bit store
  const bool edge_warp = __any_sync(0xFFFFFFFFu, live && (edge_l || edge_r));
  if (!live || yb > (int)h - 2) return;
  const uint32_t *base = reinterpret_cast<const uint32_t *>(bl) + r0 * BS_PW + 2 * lane + 1;   // blurred bytes x-4 ..
  auto load_row = [&](int r) -> SobelRow {
    const uint32_t *p = base + r * BS_PW;
    const uint2 wm = *reinterpret_cast<const uint2 *>(p + 1);
    return sobel_row(split_pairs(p[0], wm.x, wm.y, p[3]));
  };
  uint8_t *outp = dst + (size_t)frame * w * h + (size_t)yb * w + x;
  SobelRow ra = load_row(0), rb = load_row(1);
  auto walk_full = [&](auto edge_tag) {
#pragma unroll
    for (int i = 0; i < 16; i++) {
      if (i >= BS_TH % 16 && i >= nb) break;
      const SobelRow rc = load_row(i + 2);
      const uint2 so = sobel_out(ra, rb, rc);
      if (!decltype(edge_tag)::value) {
        st_cs_u2(outp, so);
      } else {                                       // predicated, no lane branches
        if (!edge_l && !edge_r) st_cs_u2(outp, so);
        if (edge_l) st_cs_7of8(outp, so, true);
        if (edge_r) st_cs_7of8(outp, so, false);
      }
      outp += w;
      ra = rb;
      rb = rc;
    }
  };
  if (yb >= 1 && yb + nb - 1 <= (int)h - 2) {
    if (edge_warp) walk_full(std::true_type{});
    else walk_full(std::false_type{});
  } else {
#pragma unroll 1
    for (int i = 0; i < nb; i++) {
      const int y = yb + i;
      if (y > (int)h - 2) break;
      const SobelRow rc = load_row(i + 2);
      if (y >= 1) {
        const uint2 so = sobel_out(ra, rb, rc);
        if (edge_l) st_cs_7of8(outp, so, true);
        else if (edge_r) st_cs_7of8(outp, so, false);
        else st_cs_u2(outp, so);
      }
      outp += w;
      ra = rb;
      rb = rc;
    }
  }
}

// ---- wide radii (8 <= r <= 120): radius-independent work, u32 window sums -------------------
// The reference's own smoke runs use `blur 9` and `adaptive 15 5` (reference Makefile:17,20); the generic
// kernel below costs (2r+1)^2 taps per pixel there.  This one costs the same ~14 instructions per pixel for
// every radius.  Each WARP works alone (no CTA barrier) on a 256-column segment of a band of rows:
//   vertical   : a lane keeps the column sums of its 8 columns over rows [y-r, y+r] as four u16x2 pair words
//                ((2r+1) * 255 <= 65535 for r <= 128) and rolls them down the band, + entering row - leaving
//                row, one IADD3 per word; rows come straight from global memory as coalesced 64-bit loads,
//                prefetched one row ahead; out-of-image rows / columns read as 0 (a clipped tap's contribution);
//   horizontal : inclusive prefix of the 256 column sums in u32 (8 local adds, a 5-step warp scan, 8 adds),
//                written to a double-buffered 1 KB shared row; the window sum of column i is
//                P[i+r] - P[i-r-1]: two LDS and a subtract.  A segment carries R8 = roundup(r, 8) halo
//                columns on both sides, so 256 - 2*R8 outputs per warp-row;
//   division   : interior pixels (count = (2r+1)^2, r <= 63) use the exact fma_rd trick of the small-radius
//                kernel with m = ceil(2^k / count), k = 23 + floor(log2 count) (host-verified for every sum
//                that can occur, box_wide_magic_ok); clipped counts and r > 63 take
//                floor(fdiv_rn(S, count)), which is exact for count < 2^17 and quotients <= 255 (the distance of
//                S/count to the next integer is >= 1/count > half an ulp).
// launch_box sends every frame with w % 8 == 0 and 8-byte aligned bases to k_box_mid, so this kernel only ever sees
// ragged widths or unaligned bases: rows are gathered byte by byte and outputs stored byte by byte.
template <bool ADAPTIVE>
__global__ void __launch_bounds__(128)
k_box_wide(uint8_t *__restrict__ dst, const uint8_t *__restrict__ src, int w, int h, int r, int R8, int BH,
           int strips, int cparam, float minv, int fast_ok) {
  // prefix row of a warp, transposed: P(8 l + k) lives at [k][16 + l], so that for a fixed register index k the 32
  // lanes touch 32 consecutive words (the natural [8 l + k] layout is an 8-way bank conflict on every read)
  __shared__ uint32_t sp_all[4][8][64];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int strip = (int)blockIdx.x * 4 + warp;
  if (strip >= strips) return;                                  // warp-uniform; no CTA barriers below
  const int outw = 256 - 2 * R8;
  const int xs = strip * outw - R8;                             // image column of segment column 0 (multiple of 8)
  const int x0 = xs + 8 * lane;
  const int yb = (int)blockIdx.y * BH, ye = min(h, yb + BH);
  const uint8_t *frame = src + (size_t)blockIdx.z * w * h;
  uint8_t *out = dst + (size_t)blockIdx.z * w * h;
  const bool lane_in = x0 + 7 >= 0 && x0 < w;
  const bool out_lane = 8 * lane >= R8 && 8 * lane + 8 <= 256 - R8 && x0 < w && x0 + 7 >= 0;
  const int FULL = 2 * r + 1;
  // all 8 pixels of this lane have the full (2r+1)-column window inside the image
  const bool cols_full = x0 - r >= 0 && x0 + 7 + r <= w - 1;

  // row loads by pointer (advanced by w per row; the per-row 64-bit multiply of y * w showed up as 10 % of the
  // instructions in the first ncu capture)
  auto ldp = [&](const uint8_t *p, int y) -> uint2 {
    if (!lane_in || y < 0 || y >= h) return make_uint2(0u, 0u);
    uint32_t a = 0, b = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) {
      if (x0 + k >= 0 && x0 + k < w) a |= (uint32_t)__ldg(p + k) << (8 * k);
      if (x0 + 4 + k >= 0 && x0 + 4 + k < w) b |= (uint32_t)__ldg(p + 4 + k) << (8 * k);
    }
    return make_uint2(a, b);
  };
  auto ld = [&](int y) -> uint2 { return ldp(frame + (ptrdiff_t)y * w + x0, y); };

  uint32_t S[4] = {0, 0, 0, 0};
#pragma unroll 4
  for (int yy = yb - r; yy <= yb + r; yy++) {
    uint32_t e[4];
    unpack_pairs(ld(yy), e);
#pragma unroll
    for (int k = 0; k < 4; k++) S[k] += e[k];
  }
  uint2 en = ld(yb + r + 1), lv = ld(yb - r), cen = make_uint2(0u, 0u);
  if (ADAPTIVE) cen = ld(yb);
  const uint8_t *p_en = frame + (ptrdiff_t)(yb + r + 2) * w + x0, *p_lv = frame + (ptrdiff_t)(yb + 1 - r) * w + x0;
  const uint8_t *p_cen = frame + (ptrdiff_t)(yb + 1) * w + x0;
  uint8_t *qo = out + (size_t)yb * w + x0;
  // word offsets of P(i + r) and P(i - r - 1) in the transposed prefix row, for this lane's 8 pixels (row invariant)
  uint32_t (*sp)[64] = sp_all[warp];
  if (lane == 0) sp[7][15] = 0u;                                // P(-1) = 0
  __syncwarp();
  const uint32_t *pA[8], *pB[8];
#pragma unroll
  for (int k = 0; k < 8; k++) {
    const int ca = k + r, cb = k - r - 1 + 128;                // cb biased by 16 lanes: >= 0
    pA[k] = &sp[0][0] + (ca & 7) * 64 + 16 + lane + (ca >> 3);
    pB[k] = &sp[0][0] + (cb & 7) * 64 + lane + (cb >> 3);
  }

  for (int y = yb; y < ye; y++) {
    const uint2 en2 = ldp(p_en, y + r + 2), lv2 = ldp(p_lv, y + 1 - r);
    uint2 cen2 = make_uint2(0u, 0u);
    if (ADAPTIVE) cen2 = ldp(p_cen, y + 1);
    p_en += w, p_lv += w, p_cen += w;
    // ---- horizontal prefix of the column sums (u32)
    uint32_t p[8];
#pragma unroll
    for (int k = 0; k < 4; k++) p[2 * k] = S[k] & 0xFFFFu, p[2 * k + 1] = S[k] >> 16;
#pragma unroll
    for (int k = 1; k < 8; k++) p[k] += p[k - 1];
    uint32_t incl = p[7];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, o);
      if (lane >= o) incl += t;
    }
    const uint32_t excl = incl - p[7];
    __syncwarp();                                                 // the previous row's reads are done
#pragma unroll
    for (int k = 0; k < 8; k++) sp[k][16 + lane] = p[k] + excl;
    __syncwarp();
    if (out_lane) {
      uint32_t W[8];
#pragma unroll
      for (int k = 0; k < 8; k++) W[k] = *pA[k] - *pB[k];
      const int ch = min(y + r, h - 1) - max(y - r, 0) + 1;
      uint32_t q[8];
      if (fast_ok && cols_full && ch == FULL) {
#pragma unroll
        for (int k = 0; k < 8; k++) q[k] = __float_as_uint(__fmaf_rd((float)W[k], minv, 8388608.0f)) & 0xFFu;
      } else {
#pragma unroll
        for (int k = 0; k < 8; k++) {
          const int x = x0 + k;
          const int cw = min(x + r, w - 1) - max(x - r, 0) + 1;
          q[k] = __float2uint_rd(__fdiv_rn((float)W[k], (float)(cw * ch)));
        }
      }
      if (ADAPTIVE) {
#pragma unroll
        for (int k = 0; k < 8; k++) {
          const int sv = (int)(((k < 4 ? cen.x : cen.y) >> (8 * (k & 3))) & 0xFFu);
          q[k] = sv > (int)(q[k] - (unsigned)cparam) ? 255u : 0u;      // reference :244-245
        }
      }
      uint2 o;
      o.x = q[0] | (q[1] << 8) | (q[2] << 16) | (q[3] << 24);
      o.y = q[4] | (q[5] << 8) | (q[6] << 16) | (q[7] << 24);
#pragma unroll
      for (int k = 0; k < 8; k++)
        if (x0 + k >= 0 && x0 + k < w) qo[k] = (uint8_t)((k < 4 ? o.x : o.y) >> (8 * (k & 3)));
    }
    qo += w;
    // ---- roll the column sums down one row
    uint32_t e[4], l[4];
    unpack_pairs(en, e);
    unpack_pairs(lv, l);
#pragma unroll
    for (int k = 0; k < 4; k++) S[k] = S[k] + e[k] - l[k];
    en = en2, lv = lv2, cen = cen2;
  }
}

// ---- medium / wide radii, aligned frames: k_box_mid (round 2, second form) ---------------------
// k_box_wide pays ~37 lane-instructions per pixel: a 256-column prefix scan per row (shuffles + selects) and
// two scattered LDS per pixel.  This form keeps the same warp-autonomous 256-column segments and the same
// rolling u16x2 column sums, but turns the horizontal pass into a ROLLING sum too, by transposing through
// shared memory.  One warp per CTA (the warps never synchronise with each other; 16.3 KB each, 13 per SM)
// alternates between
//   V-phase : 32 rows; lanes = 8 columns each.  The column sums of a row (256 u16) go to the warp's private
//             C tile [32 rows][4 u16 pad + 256 u16], pitch 130 words.  Source rows come straight from global
//             memory through a register ring of four 4-row batches (loads 12 rows ahead of their use, also
//             across the H-phase); one lane asks the TMA unit to prefetch the next chunk's rows into L2
//             (UTMAPF.L2, no shared-memory destination): without it the DRAM latency of the entering rows is
//             not covered;
//   H-phase : lanes = ROWS.  Lane j walks row j from left to right: the window sums of four neighbouring outputs
//             are W + D_k, D_k = sum_{i<=k} C[c+i+r] - C[c+i-r-1] chained from zero, each term one IDP.2A (dp2a
//             reads either 16-bit half of a pair word through its byte multiplier: 0x0001 / 0x0100 add, 0x00FF /
//             0xFF00 subtract); the chains of different groups are independent, W advances once per group.  The C
//             values come as 64-bit groups of four (pitch = 2 mod 32 words: conflict-free with lanes on rows); r mod
//             4 fixes where the entering / leaving elements sit inside their groups, hence the template
//             parameter.  Quotients as in k_box_wide (clipped counts: MUFU.RCP quotient + integer remainder
//             check instead of the IEEE-division subroutine).  The 8 output bytes of a step overwrite the head of
//             the lane's own C row (already consumed: byte 16+8t <= 8*(gl0+2t+3)); a lane never reads or writes
//             another lane's row (racecheck-clean);
//   copy-out: lanes = columns again; rows leave as coalesced 64-bit stores (gs_adaptive_threshold compares
//             with the centre pixels here, on 16-bit lane pairs).
// 13.5 lane-instructions per pixel instead of ~37 for k_box_wide (ncu).
constexpr int BM_PITCH = 130;                       // words per C row
constexpr int BM_WARP_WORDS = 32 * BM_PITCH + 8;    // + the look-ahead groups of the last row
constexpr int BM_SMEM = BM_WARP_WORDS * 4;         // one warp per CTA: 16.3 KB, 13 CTAs per SM

__device__ const uint2 bm_zero8 = {0u, 0u};

// low bytes of four words -> one word, on the ALU pipe (the H-phase keeps the FMA pipe busy with IDP / FFMA)
__device__ __forceinline__ uint32_t pack4_alu(uint32_t q0, uint32_t q1, uint32_t q2, uint32_t q3) {
  return prmt(prmt(q0, q1, 0x0040), prmt(q2, q3, 0x0040), 0x5410);
}

template <bool SUB>
__device__ __forceinline__ uint32_t dp2a_half(uint32_t acc, uint32_t word, int half) {
  uint32_t d;
  if (!SUB) {
    if (half) asm("dp2a.lo.u32.u32 %0, %1, 0x0100, %2;" : "=r"(d) : "r"(word), "r"(acc));
    else asm("dp2a.lo.u32.u32 %0, %1, 0x0001, %2;" : "=r"(d) : "r"(word), "r"(acc));
  } else {
    if (half) asm("dp2a.lo.u32.s32 %0, %1, 0xFF00, %2;" : "=r"(d) : "r"(word), "r"(acc));
    else asm("dp2a.lo.u32.s32 %0, %1, 0x00FF, %2;" : "=r"(d) : "r"(word), "r"(acc));
  }
  return d;
}
// bytes (b0..b7) of two words -> pair words (b0,b2) (b1,b3) (b4,b6) (b5,b7): half of the unpacking is a plain AND
// (full-rate LOP3; PRMT issues at half rate).  The H-phase addresses single halves, so the
// order of the columns inside a group of four is free: element e of a group sits in word e & 1, half e >> 1.
__device__ __forceinline__ void unpack_pairs_alt(uint2 v, uint32_t (&p)[4]) {
  p[0] = v.x & 0x00FF00FFu, p[1] = prmt(v.x, 0, 0x4341);
  p[2] = v.y & 0x00FF00FFu, p[3] = prmt(v.y, 0, 0x4341);
}
// element idx (0..7) of the two groups of four u16 (a, b)
template <bool SUB>
__device__ __forceinline__ uint32_t dp2a_elem(uint32_t acc, uint2 a, uint2 b, int idx) {
  const uint2 g = idx < 4 ? a : b;
  return dp2a_half<SUB>(acc, (idx & 1) ? g.y : g.x, (idx >> 1) & 1);
}

template <int RM, bool ADAPTIVE>
__global__ void __launch_bounds__(32)
k_box_mid(const __grid_constant__ CUtensorMap tmap, int use_tpf, uint8_t *__restrict__ dst, const uint8_t *__restrict__ src,
          int w, int h, int r, int R8, int BH, int strips, int cparam, float minv, int fast_ok) {
  // one warp per CTA: a 4-warp CTA held its 66 KB until its slowest warp had finished (7 of 12 warp slots occupied on
  // average in the first ncu capture)
  extern __shared__ __align__(16) uint32_t bm_smem[];
  constexpr int LM = (3 - RM) & 3;
  const int lane = threadIdx.x;
  const int wid = (int)blockIdx.x;                              // warps are dealt over (band, strip)
  const int strip = wid % strips, band = wid / strips;
  uint32_t *cs = bm_smem;
  uint32_t *rw = cs + lane * BM_PITCH;                          // H-phase: this lane's row
  const int outw = 256 - 2 * R8;
  const int xs = strip * outw - R8;                             // image column of segment column 0 (multiple of 8)
  const int x0 = xs + 8 * lane;
  const int yb = band * BH, ye = min(h, yb + BH);
  const uint8_t *frame = src + (size_t)blockIdx.z * w * h;
  uint8_t *out = dst + (size_t)blockIdx.z * w * h;
  const bool lane_in = x0 >= 0 && x0 < w;                       // w % 8 == 0
  const bool out_lane = 8 * lane >= R8 && 8 * lane + 8 <= 256 - R8 && x0 < w;
  const int FULL = 2 * r + 1;

  rw[0] = 0u, rw[1] = 0u;                                       // C[-4..-1] = 0: what "leaves" before column 0 entered
  if (lane == 0) cs[32 * BM_PITCH] = 0u, cs[32 * BM_PITCH + 1] = 0u;

  // rows of this lane's 8 columns; lanes left / right of the image read a zero word with stride 0, rows above / below
  // the image are a warp-uniform test
  const unsigned wl = lane_in ? (unsigned)w : 0u;
  const uint8_t *col = lane_in ? frame + x0 : reinterpret_cast<const uint8_t *>(&bm_zero8);
  auto ld_row = [&](int y) -> uint2 {
    if ((unsigned)y >= (unsigned)h) return make_uint2(0u, 0u);
    return __ldg(reinterpret_cast<const uint2 *>(col + (size_t)(unsigned)y * wl));
  };
  auto ld_batch = [&](uint2 (&v)[4], int y, auto guard_tag) {   // rows y .. y+3
    if (!decltype(guard_tag)::value || (y >= 0 && y + 3 < h)) {
      const uint8_t *p = col + (size_t)(unsigned)y * wl;
#pragma unroll
      for (int k = 0; k < 4; k++) v[k] = __ldg(reinterpret_cast<const uint2 *>(p + (size_t)k * wl));
    } else {
#pragma unroll
      for (int k = 0; k < 4; k++) v[k] = ld_row(y + k);
    }
  };
  // one lane asks the TMA unit to pull a 288-byte x 32-row box of source rows into L2 (no shared-memory destination):
  // the entering rows a whole chunk before the register ring asks for them (the leaving rows were read 2r+1 rows
  // earlier and are L2 hits anyway).  One instruction per chunk; the per-row prefetch.global.L2 form cost 4.5
  // instructions per row for the same effect.
  auto pf_box = [&](int y) {
    if (use_tpf && lane == 0 && y < h) {
      const int xw = (max(xs, 0) >> 2) & ~3;
      asm volatile("cp.async.bulk.prefetch.tensor.3d.L2.global.tile [%0, {%1, %2, %3}];" ::"l"(&tmap), "r"(xw), "r"(y),
                   "r"((int)blockIdx.z)
                   : "memory");
    }
  };
  pf_box(yb - r), pf_box(yb - r + 32), pf_box(yb - r + 64);     // the band's first rows (window build-up and ring prologue) arrive together
  // the rows that enter / leave the window, in batches of four row steps; a ring of four batches keeps the loads
  // three batches (12 rows) ahead of their use, also across the H-phase
  uint2 en[4][4], lv[4][4];
#pragma unroll
  for (int i = 0; i < 3; i++) {
    ld_batch(en[i], yb + 4 * i + r + 1, std::true_type{});
    ld_batch(lv[i], yb + 4 * i - r, std::true_type{});
  }
  uint32_t S[4] = {0, 0, 0, 0};                                 // column sums over rows [y - r, y + r], y = yb
  for (int i0 = -r; i0 <= r; i0 += 16) {                        // 16 loads in flight (one at a time: 2r+1 latencies per band)
    uint2 v[16];
#pragma unroll
    for (int k = 0; k < 16; k++) v[k] = i0 + k <= r ? ld_row(yb + i0 + k) : make_uint2(0u, 0u);
#pragma unroll
    for (int k = 0; k < 16; k++) {
      uint32_t e[4];
      unpack_pairs_alt(v[k], e);
#pragma unroll
      for (int q = 0; q < 4; q++) S[q] += e[q];
    }
  }

  const int cc = max(-256, min(256, cparam));
  const uint32_t kc = (uint32_t)(cc + 0x7FFF) * 0x10001u;
  const int ge0 = (R8 + r + 4) >> 2, gl0 = (R8 - r + 3) >> 2;   // first entering / leaving group of a row
  const int iters = outw >> 3;

  for (int yc = yb; yc < ye; yc += 32) {
    // ---- V-phase: C rows of image rows yc .. yc+31
    __syncwarp();                                               // the previous chunk's copy-out is done
    pf_box(yc + r + 13 + 32 * use_tpf);                         // what the next chunk's ring loads will ask for
    auto v_phase = [&](auto guard_tag) {
      uint32_t *crow = cs + 2 + 4 * lane;
#pragma unroll 1
      for (int bb = 0; bb < 2; bb++) {
#pragma unroll
        for (int qb = 0; qb < 4; qb++) {
          const int yn = yc + 16 * bb + 4 * qb + 12;            // first row step of the batch three ahead
          ld_batch(en[(qb + 3) & 3], yn + r + 1, guard_tag);
          ld_batch(lv[(qb + 3) & 3], yn - r, guard_tag);
#pragma unroll
          for (int k = 0; k < 4; k++) {
            *reinterpret_cast<uint2 *>(crow) = make_uint2(S[0], S[1]);
            *reinterpret_cast<uint2 *>(crow + 2) = make_uint2(S[2], S[3]);
            crow += BM_PITCH;
            uint32_t e[4], l[4];
            unpack_pairs_alt(en[qb][k], e);
            unpack_pairs_alt(lv[qb][k], l);
#pragma unroll
            for (int q = 0; q < 4; q++) S[q] = S[q] + e[q] - l[q];
          }
        }
      }
    };
    // every row this chunk loads or prefetches (yc + 12 - r .. yc + 44 + r + 32) is inside the image
    if (yc + 12 - r >= 0 && yc + 76 + r < h) v_phase(std::false_type{});
    else v_phase(std::true_type{});
    __syncwarp();
    // ---- H-phase: lane = row
    const int y = yc + lane;
    if (y < ye) {
      const uint2 *grp = reinterpret_cast<const uint2 *>(rw);
      uint2 L0 = grp[gl0], E0 = grp[ge0];
      uint32_t W = 0;
#pragma unroll
      for (int k = LM; k < 4; k++) W = dp2a_elem<false>(W, L0, L0, k);
      for (int g = gl0 + 1; g < ge0; g++) {
        const uint2 t = grp[g];
        asm("dp2a.lo.u32.u32 %0, %1, 0x0101, %0;" : "+r"(W) : "r"(t.x));
        asm("dp2a.lo.u32.u32 %0, %1, 0x0101, %0;" : "+r"(W) : "r"(t.y));
      }
#pragma unroll
      for (int k = 0; k < RM; k++) W = dp2a_elem<false>(W, E0, E0, k);
      const int ch = min(y + r, h - 1) - max(y - r, 0) + 1;
      const bool row_fast = fast_ok && ch == FULL;
      const uint2 *pe = grp + ge0 + 1, *pl = grp + gl0 + 1;
      uint2 *po = reinterpret_cast<uint2 *>(rw + 2);
      const int xo = xs + R8;                                   // image column of this row's first output
      // eight outputs per step; FAST: unclipped windows, magic multiplier; else per-pixel counts.  The window sums of a
      // group of four are W + D_k with the D_k chained from zero: the chains of different groups are independent (the
      // single chain W(c) = W(c-1) + .. - .. left a warp waiting 4 cycles on every IDP), only one add per group is
      // serial.  The four groups a step consumes were loaded during the PREVIOUS step into the other of two register
      // sets (A, B); volatile ld / st keep that order (the output store aliases the row as far as the compiler can
      // tell, and with plain loads it sank them to the end of the step, right in front of their first use).
      const uint32_t pe_s = smem_u32(pe), pl_s = smem_u32(pl), po_s = smem_u32(po);
      auto lds2 = [](uint32_t addr) -> uint2 {
        uint2 v;
        asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(addr) : "memory");
        return v;
      };
      uint2 EA[2] = {lds2(pe_s), lds2(pe_s + 8)}, LA[2] = {lds2(pl_s), lds2(pl_s + 8)}, EB[2], LB[2];
      EB[1] = E0, LB[1] = L0;                                   // "the group before A[0]"
      const int u_in = (60 - ge0) >> 1;                         // t <= u_in: groups ge0 + 2t + 3, ge0 + 2t + 4 (step t+1's) are <= 64, the row's last
      // one step: consumes Ec / Lc (carry-in: the group before them, Ep / Lp), loads the next step's groups into Ex / Lx
      auto step8 = [&](int t, auto fast_tag, auto guard_tag, const uint2 (&Ec)[2], const uint2 (&Lc)[2], const uint2 Ep,
                       const uint2 Lp, uint2 (&Ex)[2], uint2 (&Lx)[2]) {
        constexpr bool FAST = decltype(fast_tag)::value;
        Lx[0] = lds2(pl_s + 16 * t + 16), Lx[1] = lds2(pl_s + 16 * t + 24);
        if (!decltype(guard_tag)::value || t <= u_in) {                                        // both entering groups of step t+1 lie inside this lane's row
          Ex[0] = lds2(pe_s + 16 * t + 16), Ex[1] = lds2(pe_s + 16 * t + 24);
        } else {                                                // at the end of the row: never read the neighbouring lane's row
          Ex[0] = ge0 + 2 * t + 3 <= 64 ? lds2(pe_s + 16 * t + 16) : make_uint2(0u, 0u);
          Ex[1] = make_uint2(0u, 0u);
        }
        uint32_t ow[2];
#pragma unroll
        for (int s = 0; s < 2; s++) {
          const uint2 Ea = s == 0 ? Ep : Ec[0], La = s == 0 ? Lp : Lc[0];
          uint32_t Wk[4], q[4], D = 0;
#pragma unroll
          for (int k = 0; k < 4; k++) {
            D = dp2a_elem<false>(D, Ea, Ec[s], RM + k);
            D = dp2a_elem<true>(D, La, Lc[s], LM + k);
            Wk[k] = W + D;
          }
          W = Wk[3];
          if (FAST) {
#pragma unroll
            for (int k = 0; k < 4; k++) q[k] = __float_as_uint(__fmaf_rd((float)Wk[k], minv, 8388608.0f));
          } else {
#pragma unroll
            for (int k = 0; k < 4; k++) {
              // floor(W / count), count = in-image columns x rows < 2^16, W <= 255 * count: the approximate quotient
              // (MUFU.RCP, |error| < 1e-3) truncates to the true floor or one off; the remainder decides
              const int x = xo + 8 * t + 4 * s + k;
              const int cnt = max(min(x + r, w - 1) - max(x - r, 0) + 1, 1) * ch;   // columns outside the image are never stored
              uint32_t q0 = (uint32_t)__fdividef((float)Wk[k], (float)cnt);
              const int rem = (int)Wk[k] - (int)q0 * cnt;
              q0 += rem >= cnt ? 1u : 0u;
              q0 -= rem < 0 ? 1u : 0u;
              q[k] = q0 & 0xFFu;
            }
          }
          ow[s] = pack4_alu(q[0], q[1], q[2], q[3]);
        }
        asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(po_s + 8 * t), "r"(ow[0]), "r"(ow[1]) : "memory");
      };
      // between loops the live set is A with the group before it in B[1]
      auto single = [&](int t, auto fast_tag) {
        step8(t, fast_tag, std::true_type{}, EA, LA, EB[1], LB[1], EB, LB);
        const uint2 e1 = EA[1], l1 = LA[1];
        EA[0] = EB[0], EA[1] = EB[1], LA[0] = LB[0], LA[1] = LB[1];
        EB[1] = e1, LB[1] = l1;
      };
      // steps that reach into the image: [0, t_img); of those, [t_lo, t_hi) are fast: xo + 8t - r >= 0 and
      // xo + 8t + 7 + r <= w - 1
      const int t_img = min(iters, (w - xo + 7) >> 3);
      int t_lo = 0, t_hi = 0;
      if (row_fast) {
        t_lo = min(t_img, max(0, (r - xo + 7) >> 3));
        t_hi = max(t_lo, min(t_img, (w - r - xo) >> 3));        // floor((w - 8 - r - xo) / 8) + 1, arithmetic shift
      }
      int t = 0;
#pragma unroll 1
      for (int seg = 0; seg < 2; seg++) {
        const int t_end = seg == 0 ? t_lo : t_img;
#pragma unroll 1
        for (; t < t_end; t++) single(t, std::false_type{});
        if (seg == 0) {
#pragma unroll 1
          for (; t + 1 < t_hi && t + 1 <= u_in; t += 2) {       // A -> B -> A: no register rotation; look-ahead inside the row
            step8(t, std::true_type{}, std::false_type{}, EA, LA, EB[1], LB[1], EB, LB);
            step8(t + 1, std::true_type{}, std::false_type{}, EB, LB, EA[1], LA[1], EA, LA);
          }
#pragma unroll 1
          for (; t < t_hi; t++) single(t, std::true_type{});    // the last one or two steps of the row: guarded look-ahead
        }
      }
    }
    __syncwarp();
    // ---- copy-out: lane = 8 columns
    const int nrows = min(32, ye - yc);
    if (out_lane) {
      const uint32_t *orow = cs + 2 + ((8 * lane - R8) >> 2);
      uint8_t *qo = out + (size_t)yc * w + x0;
      const uint8_t *qc = frame + (size_t)yc * w + x0;
      const unsigned wu = (unsigned)w;
      auto put_row = [&](int j) {
        uint2 o = *reinterpret_cast<const uint2 *>(orow + j * BM_PITCH);
        if (ADAPTIVE) {
          // dst = src > (int)mean - c ? 255 : 0 (reference :244-245), see box_finish
          const uint2 sp = __ldg(reinterpret_cast<const uint2 *>(qc + (size_t)j * wu));
          const uint32_t e0 = prmt(sp.x, 0, 0x4140) + kc - prmt(o.x, 0, 0x4140);
          const uint32_t e1 = prmt(sp.x, 0, 0x4342) + kc - prmt(o.x, 0, 0x4342);
          const uint32_t e2 = prmt(sp.y, 0, 0x4140) + kc - prmt(o.y, 0, 0x4140);
          const uint32_t e3 = prmt(sp.y, 0, 0x4342) + kc - prmt(o.y, 0, 0x4342);
          o.x = prmt_raw(e0, e1, 0xFDB9);
          o.y = prmt_raw(e2, e3, 0xFDB9);
        }
        st_cs_u2(qo + (size_t)j * wu, o);
      };
      if (nrows == 32) {
        if (ADAPTIVE) {
          // the centre rows (L2 hits: they entered the window r+1 rows ago), eight loads in flight
#pragma unroll
          for (int j0 = 0; j0 < 32; j0 += 8) {
            uint2 sp[8];
#pragma unroll
            for (int j = 0; j < 8; j++) sp[j] = __ldg(reinterpret_cast<const uint2 *>(qc + (size_t)(j0 + j) * wu));
#pragma unroll
            for (int j = 0; j < 8; j++) {
              uint2 o = *reinterpret_cast<const uint2 *>(orow + (j0 + j) * BM_PITCH);
              const uint32_t e0 = prmt(sp[j].x, 0, 0x4140) + kc - prmt(o.x, 0, 0x4140);
              const uint32_t e1 = prmt(sp[j].x, 0, 0x4342) + kc - prmt(o.x, 0, 0x4342);
              const uint32_t e2 = prmt(sp[j].y, 0, 0x4140) + kc - prmt(o.y, 0, 0x4140);
              const uint32_t e3 = prmt(sp[j].y, 0, 0x4342) + kc - prmt(o.y, 0, 0x4342);
              st_cs_u2(qo + (size_t)(j0 + j) * wu, make_uint2(prmt_raw(e0, e1, 0xFDB9), prmt_raw(e2, e3, 0xFDB9)));
            }
          }
        } else {
#pragma unroll
          for (int j = 0; j < 32; j++) put_row(j);
        }
      } else {
#pragma unroll 1
        for (int j = 0; j < nrows; j++) put_row(j);
      }
    }
  }
}

// k, m for the exact interior division of k_box_wide: floor(S * m / 2^k) == S / count for every S <= 255 * count
static bool box_wide_magic(unsigned count, float *minv) {
  int lg = 0;
  while ((2u << lg) <= count) lg++;
  const int k = 23 + lg;
  const unsigned long long m = ((1ull << k) + count - 1) / count;
  if (m >= (1ull << 24)) return false;
  // S*m/2^k = S/count + S*e/(count*2^k), e = m*count - 2^k: exact iff the excess stays below 1/count for S <= 255*count
  const unsigned long long e = m * count - (1ull << k);
  if (255ull * count * e >= (1ull << k)) return false;
  *minv = ldexpf((float)m, -k);
  return true;
}

// ---- generic: any radius, width, alignment; one thread per pixel ----------------------------
template <bool ADAPTIVE>
__global__ void k_box_generic(uint8_t *__restrict__ dst, const uint8_t *__restrict__ src, unsigned w,
                              unsigned h, unsigned n, unsigned r, int cparam) {
  const unsigned x = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= w || y >= h) return;
  const unsigned xa = x > r ? x - r : 0, xb = min(x + (unsigned long long)r, (unsigned long long)w - 1);
  const unsigned ya = y > r ? y - r : 0, yb = min(y + (unsigned long long)r, (unsigned long long)h - 1);
  const unsigned count = (xb - xa + 1) * (yb - ya + 1);
  for (unsigned f = blockIdx.z; f < n; f += gridDim.z) {
    const uint8_t *s = src + (size_t)f * w * h;
    unsigned sum = 0;
    for (unsigned yy = ya; yy <= yb; yy++)
      for (unsigned xx = xa; xx <= xb; xx++) sum += s[(size_t)yy * w + xx];
    const unsigned mean = sum / count;
    uint8_t v;
    if (ADAPTIVE) v = ((int)s[(size_t)y * w + x] > (int)(mean - (unsigned)cparam)) ? 255 : 0;
    else v = (uint8_t)mean;
    dst[(size_t)f * w * h + (size_t)y * w + x] = v;
  }
}

template <bool ADAPTIVE>
static int launch_box(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n, unsigned r,
                      int cparam, cudaStream_t s) {
  if (n == 0) return 0;
  // the clamped lane compare of k_box_tma / k_box_mid (box_finish) is exact only for c > INT_MIN + 255
  const bool lane_c_ok = !ADAPTIVE || cparam > INT_MIN + 255;
  CUtensorMap tmap;
  if (lane_c_ok && r >= 1 && r <= BX_RMAX && tma_ok(src, w) && tma_ok(dst, w) &&
      n <= 65535u && make_tmap_u8frames(&tmap, src, w, h, n, BX_PW, BX_TH + 2 * r)) {
    static decltype(&k_box_tma<1, ADAPTIVE>) const box_tma_fn[BX_RMAX] = {
        k_box_tma<1, ADAPTIVE>, k_box_tma<2, ADAPTIVE>, k_box_tma<3, ADAPTIVE>, k_box_tma<4, ADAPTIVE>,
        k_box_tma<5, ADAPTIVE>, k_box_tma<6, ADAPTIVE>, k_box_tma<7, ADAPTIVE>};
    // tile t covers output columns [240 t - 8, 240 t + 232)
    const unsigned tiles_x = (w + 8 + BX_STRIDE - 1) / BX_STRIDE, tiles_y = (h + BX_TH - 1) / BX_TH;
    GSB_ASSERT(tiles_y <= 65535u);   // grid y limit (z was checked above)
    GSB_LAUNCH(box_tma_fn[r - 1], dim3(tiles_x, tiles_y, n), BX_THREADS, BX_SMEM, s, tmap, dst, w, h, cparam);
    return 0;
  }
  if (r >= 1 && r <= 120 && !force_generic() && n <= 65535u && w < (1u << 30) && h < (1u << 30)) {
    // radius-independent path: warp-autonomous 256-column segments, u32 window sums (k_box_wide)
    const int R8 = (int)((r + 7) / 8 * 8), outw = 256 - 2 * R8;
    const int strips = (int)((w + outw - 1) / outw);
    // enough warps to fill every SM, bands no shorter than 4r rows (vertical halo re-reads <= 1/3)
    const long long want = (long long)sm_count() * 24;
    long long bands = (want + (long long)strips * n - 1) / ((long long)strips * n);
    const long long max_bands = ((long long)h + (4 * (long long)r > 32 ? 4 * (long long)r : 32) - 1) / (4 * (long long)r > 32 ? 4 * (long long)r : 32);
    if (bands > max_bands) bands = max_bands;
    if (bands < 1) bands = 1;
    int BH = (int)((h + bands - 1) / bands);
    const unsigned gy = (h + BH - 1) / BH;
    GSB_ASSERT(gy <= 65535u);
    float minv = 0.0f;
    const int fast_ok = (r <= 63 && box_wide_magic((2 * r + 1) * (2 * r + 1), &minv)) ? 1 : 0;
    const bool aligned = w % 8 == 0 && reinterpret_cast<uintptr_t>(src) % 8 == 0 && reinterpret_cast<uintptr_t>(dst) % 8 == 0;
    dim3 grid((strips + 3) / 4, gy, n);
    if (aligned && lane_c_ok) {
      // k_box_mid: chunks of 32 rows, so bands are multiples of 32 rows.  Short bands keep the grid many waves deep
      // (3 CTAs of 4 warps per SM); a band re-reads 2r + 1 + 12 rows of its upper neighbour (L2 hits) and spends ~7
      // instructions on each, against ~75 per regular row: the largest of 128 / 64 / 32 rows that still gives
      // four waves, but not below 4r rows.
      const long long four_waves = (long long)sm_count() * 13 * 4;
      BH = 32;
      for (int cand = 128; cand >= 32; cand >>= 1)
        if ((long long)strips * ((h + cand - 1) / cand) * n >= four_waves || cand == 32) { BH = cand; break; }
      while (BH < 4 * (int)r && BH < 256) BH <<= 1;
      const long long warps = (long long)strips * ((h + BH - 1) / BH);
      GSB_ASSERT(warps < (1ll << 31));
      grid = dim3((unsigned)warps, 1, n);
      CUtensorMap pmap;
      const int use_tpf = make_tmap_u8frames(&pmap, src, w, h, n, 72, 32) ? 1 : 0;   // needs w % 16 == 0 and a 16-byte aligned base
      if (!use_tpf) memset(&pmap, 0, sizeof(pmap));
      static decltype(&k_box_mid<0, ADAPTIVE>) const box_mid_fn[4] = {k_box_mid<0, ADAPTIVE>, k_box_mid<1, ADAPTIVE>,
                                                                      k_box_mid<2, ADAPTIVE>, k_box_mid<3, ADAPTIVE>};
      GSB_LAUNCH(box_mid_fn[r & 3], grid, 32, BM_SMEM, s, pmap, use_tpf, dst, src, (int)w, (int)h, (int)r, R8, BH, strips,
                 cparam, minv, fast_ok);
      return 0;
    }
    GSB_LAUNCH(k_box_wide<ADAPTIVE>, grid, 128, 0, s, dst, src, (int)w, (int)h, (int)r, R8, BH, strips, cparam, minv, fast_ok);
    return 0;
  }
  dim3 block(32, 8), grid((w + 31) / 32, (h + 7) / 8, n < 65535u ? n : 65535u);
  GSB_LAUNCH(k_box_generic<ADAPTIVE>, grid, block, 0, s, dst, src, w, h, n, r, cparam);
  return 0;
}

}  // namespace gsb

extern "C" {
int gs_b200_blur_sobel_batch(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n, unsigned radius,
                             gs_b200_stream st) {
  GSB_ASSERT(dst && src && w > 0 && h > 0);  // reference :269, :307
  cudaStream_t s = static_cast<cudaStream_t>(st);
  if (n == 0 || w < 3 || h < 3) return 0;    // gs_sobel writes nothing below 3x3 (reference :308-309)
  CUtensorMap tmap;
  if (radius >= 1 && radius <= gsb::BX_RMAX && gsb::tma_ok(src, w) && gsb::tma_ok(dst, w) && n <= 65535u &&
      gsb::make_tmap_u8frames(&tmap, src, w, h, n, gsb::BS_PW, gsb::BS_IN_ROWS)) {
    static decltype(&gsb::k_blur_sobel_tma<1>) const blur_sobel_fn[gsb::BX_RMAX] = {
        gsb::k_blur_sobel_tma<1>, gsb::k_blur_sobel_tma<2>, gsb::k_blur_sobel_tma<3>, gsb::k_blur_sobel_tma<4>,
        gsb::k_blur_sobel_tma<5>, gsb::k_blur_sobel_tma<6>, gsb::k_blur_sobel_tma<7>};
    const unsigned tiles_x = (w + gsb::BS_STRIDE - 1) / gsb::BS_STRIDE, tiles_y = (h + gsb::BS_TH - 1) / gsb::BS_TH;
    GSB_ASSERT(tiles_y <= 65535u);
    GSB_LAUNCH(blur_sobel_fn[radius - 1], dim3(tiles_x, tiles_y, n), gsb::BS_THREADS, gsb::BS_SMEM, s, tmap, dst, w, h);
    return 0;
  }
  // other radii / ragged widths: the two per-op kernels through a scratch frame batch (same result, 4 B/px)
  uint8_t *tmp = static_cast<uint8_t *>(gsb::workspace(s, gsb::WS_STAGE_FUSED, (size_t)w * h * n));
  if (!tmp) return gsb::workspace_error();
  int rc = gs_b200_blur_batch(tmp, src, w, h, n, radius, st);
  if (rc) return rc;
  return gs_b200_sobel_batch(dst, tmp, w, h, n, st);
}
int gs_b200_blur_batch(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n,
                       unsigned radius, gs_b200_stream s) {
  GSB_ASSERT(dst && src && w > 0 && h > 0);  // reference :269
  return gsb::launch_box<false>(dst, src, w, h, n, radius, 0, static_cast<cudaStream_t>(s));
}
int gs_b200_adaptive_threshold_batch(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h,
                                     unsigned n, unsigned radius, int c, gs_b200_stream s) {
  GSB_ASSERT(dst && src && w > 0 && h > 0);  // reference :232
  return gsb::launch_box<true>(dst, src, w, h, n, radius, c, static_cast<cudaStream_t>(s));
}
}
