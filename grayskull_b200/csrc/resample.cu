// resample.cu -- gs_resize and gs_downsample (reference grayskull.h:171-197).
#include "common.cuh"
#include "resample.cuh"

namespace gsb {

// ---- gs_downsample: (a+b+c+d)/4 over 2x2 blocks, 1.25 B per source pixel ----------------------
// Fast path: a thread reads two aligned 16-byte row segments (128-bit loads) and writes 8 output
// bytes.  Horizontal pair sums and the two rows are added on 16-bit lanes, >>2 under a mask.
__global__ void k_downsample_vec(uint8_t *__restrict__ dst, const uint8_t *__restrict__ src, unsigned sw,
                                 unsigned sh, unsigned dw, unsigned dh, unsigned n) {
  const unsigned gx = blockIdx.x * blockDim.x + threadIdx.x;  // 8 dst pixels each
  if (gx * 8 >= dw) return;
  for (unsigned y = blockIdx.y; y < dh; y += gridDim.y) {      // grid y: <= 65535 rows
    for (unsigned f = blockIdx.z; f < n; f += gridDim.z) {
      const uint4 *r0 = reinterpret_cast<const uint4 *>(src + (size_t)f * sw * sh + (size_t)(2 * y) * sw) + gx;
      const uint4 *r1 = reinterpret_cast<const uint4 *>(src + (size_t)f * sw * sh + (size_t)(2 * y + 1) * sw) + gx;
      const uint4 a = __ldg(r0), b = __ldg(r1);
      auto quad = [](uint32_t u, uint32_t v) -> uint32_t {  // lanes: (b0+b1+.., b2+b3+..) >> 2
        uint32_t s = (u & 0x00FF00FFu) + ((u >> 8) & 0x00FF00FFu) + (v & 0x00FF00FFu) + ((v >> 8) & 0x00FF00FFu);
        return (s >> 2) & 0x00FF00FFu;
      };
      uint2 o;
      o.x = prmt(quad(a.x, b.x), quad(a.y, b.y), 0x6420);
      o.y = prmt(quad(a.z, b.z), quad(a.w, b.w), 0x6420);
      st_cs_u2(dst + (size_t)f * dw * dh + (size_t)y * dw + gx * 8, o);
    }
  }
}

__global__ void k_downsample_generic(uint8_t *__restrict__ dst, const uint8_t *__restrict__ src,
                                     unsigned sw, unsigned sh, unsigned dw, unsigned dh, unsigned n) {
  const unsigned x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= dw) return;
  for (unsigned y = blockIdx.y * blockDim.y + threadIdx.y; y < dh; y += gridDim.y * blockDim.y) {   // grid y: <= 65535 row tiles
    for (unsigned f = blockIdx.z; f < n; f += gridDim.z) {
      const uint8_t *p = src + (size_t)f * sw * sh + (size_t)(2 * y) * sw + 2 * x;
      dst[(size_t)f * dw * dh + (size_t)y * dw + x] = (uint8_t)((p[0] + p[1] + p[sw] + p[sw + 1]) / 4);
    }
  }
}

// ---- gs_resize: pixel-centre bilinear, fp32 in the reference's exact evaluation order ---------
// (resize_axis and bilerp, in resample.cuh)
// A thread produces 4 adjacent dst pixels for RS_ROWS rows: the x-axis coefficients (two IEEE
// divisions per pixel in the reference's formula) are computed once per thread, the y-axis ones once
// per row, and the 4 results leave as one 32-bit store.
// PAIRS path: when a thread's eight taps are the eight consecutive source bytes x0[0] .. x0[0] + 7 (every
// 2:1 reduction in x, the pyramid / "half size" case) and that address is 8-byte aligned, a source row is
// ONE 64-bit load instead of eight byte gathers, and the u8 -> f32 conversions pick their byte straight out
// of the loaded words.  Threads that do not qualify (other ratios, clamped edges) take the gather path.
constexpr int RS_ROWS = 8;

// u8 -> f32 and f32 -> u8 without the conversion pipe (I2F / F2I run at 16 lanes/clk/SM and four conversions per
// dst pixel capped round 1's kernel at ~4 pixels/clk/SM): adding 2^23 to p in [0, 256) with round-toward-zero leaves
// trunc(p) in the low byte.
//
// [r2] The u8 -> f32 step needs no arithmetic.  The bit pattern of a byte b read as a float IS the
// subnormal b * 2^-149, and a power-of-two scaling commutes with round-to-nearest as long as nothing leaves the normal
// range: rn(b * 2^-149 * (wx * 2^126)) = rn(b * wx) * 2^-23 and rn(that * (wy * 2^23)) = rn(rn(b * wx) * wy), the
// reference's two products bit for bit (b * wx >= 2^-11 or 0; the weights are pre-scaled once per thread / per row;
// FMUL takes subnormal inputs at full rate, the library is built without -ftz).  Per tap: load + 2 FMUL.
constexpr float RS_WX_SCALE = 0x1p126f, RS_WY_SCALE = 0x1p23f;
__device__ __forceinline__ float byte_f(uint32_t w, int k) { return __uint_as_float(prmt(w, 0u, 0x4440u | (unsigned)k)); }
__device__ __forceinline__ float u8_f(unsigned b) { return __uint_as_float(b); }
__device__ __forceinline__ uint32_t f_trunc_bits(float p) { return __float_as_uint(__fadd_rz(p, 8388608.0f)); }  // low byte = (uint8_t)p

template <bool VEC>
__global__ void __launch_bounds__(256)
k_resize(uint8_t *__restrict__ dst, unsigned dw, unsigned dh, const uint8_t *__restrict__ src, unsigned sw,
         unsigned sh, unsigned n, bool src_aligned8, unsigned ty0 /* first row tile of the launch: for_row_groups */) {
  // the y-axis coefficients (an IEEE division each) of the CTA's 64 rows: once per CTA, not once per thread and row
  __shared__ unsigned s_y0[8 * RS_ROWS], s_y1[8 * RS_ROWS];
  __shared__ float s_dy[8 * RS_ROWS], s_omy[8 * RS_ROWS];   // pre-scaled y weights
  if (threadIdx.x < 8 * RS_ROWS) {
    const unsigned yy = (blockIdx.y + ty0) * 8 * RS_ROWS + threadIdx.x;
    unsigned a = 0, b = 0;
    float fr = 0.0f;
    if (yy < dh) resize_axis(yy, sh, dh, a, b, fr);
    s_y0[threadIdx.x] = a, s_y1[threadIdx.x] = b;
    s_dy[threadIdx.x] = __fmul_rn(fr, RS_WY_SCALE), s_omy[threadIdx.x] = __fmul_rn(__fsub_rn(1.0f, fr), RS_WY_SCALE);
  }
  __syncthreads();
  const unsigned x = (blockIdx.x * 32 + (threadIdx.x & 31)) * 4;
  const unsigned yb = ((blockIdx.y + ty0) * 8 + (threadIdx.x >> 5)) * RS_ROWS;
  if (x >= dw || yb >= dh) return;
  const unsigned yl = (threadIdx.x >> 5) * RS_ROWS;       // this warp's first row in the table
  unsigned x0[4], x1[4];
  float dx[4], omx[4];
#pragma unroll
  for (int j = 0; j < 4; j++) {
    resize_axis(min(x + j, dw - 1), sw, dw, x0[j], x1[j], dx[j]);
    omx[j] = __fmul_rn(__fsub_rn(1.0f, dx[j]), RS_WX_SCALE);
    dx[j] = __fmul_rn(dx[j], RS_WX_SCALE);
  }
  bool pairs = VEC && src_aligned8 && x0[0] % 8 == 0 && x + 3 < dw;
#pragma unroll
  for (int j = 0; j < 4; j++) pairs = pairs && x0[j] == x0[0] + 2 * j && x1[j] == x0[j] + 1;
  for (unsigned f = blockIdx.z; f < n; f += gridDim.z) {
    const uint8_t *s = src + (size_t)f * sw * sh;
    uint8_t *d = dst + (size_t)f * dw * dh;
    for (unsigned r = 0; r < (unsigned)RS_ROWS && yb + r < dh; r++) {
      const unsigned y = yb + r;
      const unsigned y0 = s_y0[yl + r], y1 = s_y1[yl + r];
      const float omy = s_omy[yl + r], dy = s_dy[yl + r];
      const uint8_t *r0 = s + (size_t)y0 * sw, *r1 = s + (size_t)y1 * sw;
      uint32_t out = 0;
      if (pairs) {
        const uint2 a = __ldg(reinterpret_cast<const uint2 *>(r0 + x0[0])), b = __ldg(reinterpret_cast<const uint2 *>(r1 + x0[0]));
        const float p0 = bilerp(byte_f(a.x, 0), byte_f(a.x, 1), byte_f(b.x, 0), byte_f(b.x, 1), omx[0], dx[0], omy, dy);
        const float p1 = bilerp(byte_f(a.x, 2), byte_f(a.x, 3), byte_f(b.x, 2), byte_f(b.x, 3), omx[1], dx[1], omy, dy);
        const float p2 = bilerp(byte_f(a.y, 0), byte_f(a.y, 1), byte_f(b.y, 0), byte_f(b.y, 1), omx[2], dx[2], omy, dy);
        const float p3 = bilerp(byte_f(a.y, 2), byte_f(a.y, 3), byte_f(b.y, 2), byte_f(b.y, 3), omx[3], dx[3], omy, dy);
        out = prmt(prmt(f_trunc_bits(p0), f_trunc_bits(p1), 0x0040), prmt(f_trunc_bits(p2), f_trunc_bits(p3), 0x0040), 0x5410);
      } else {
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const float c00 = u8_f(__ldg(r0 + x0[j])), c01 = u8_f(__ldg(r0 + x1[j]));
          const float c10 = u8_f(__ldg(r1 + x0[j])), c11 = u8_f(__ldg(r1 + x1[j]));
          out |= (f_trunc_bits(bilerp(c00, c01, c10, c11, omx[j], dx[j], omy, dy)) & 0xFFu) << (8 * j);
        }
      }
      uint8_t *q = d + (size_t)y * dw + x;
      if (VEC) {
        *reinterpret_cast<uint32_t *>(q) = out;
      } else {
        for (unsigned j = 0; j < 4 && x + j < dw; j++) q[j] = (uint8_t)(out >> (8 * j));
      }
    }
  }
}

// ---- [r2] k_resize_tiled: source rectangle staged in shared memory by TMA ---------------------------------------
// The gather kernel above is issue-bound at ~46 instructions per dst pixel (ncu): 12 of them
// are the 64-bit address arithmetic of sixteen byte gathers per thread and row.  Here ONE bulk tensor copy brings the
// source rectangle a 128 x 64 dst tile can touch into shared memory, then every tap is an LDS.U8 at a 32-bit offset:
// 4 address adds + 4 loads per pixel.  (Staging with ordinary loads was tried first: the index arithmetic per
// staged word cost more than the gathers it replaced.)  Same fp32 evaluation
// as k_resize.  Used when the rectangle fits (ratios up to about 2.8 : 1 per axis, all up-scalings) and TMA applies.
//
// The host sizes the rectangle from the ratio r = s / d with a fixed spare: 127 * rx + 22 columns, 63 * ry + 6 rows.
// That spare holds for source sizes below RT_SRC_LIMIT.  There every fp32 sx is within 7/8 of
// (x + 0.5) * s / (float)d - 0.5, whose (float)d is common to the whole tile: sx < 2^22, so the relative roundings of
// (float)x and x + 0.5 (1.5 * 2^-24 together) and of the product (2^-24) move it by at most 3/8 and 1/4, and the
// division and the subtraction by half an ulp, 1/8, each.  So a tile's last tap starts less than 127 * rx + 2.75
// columns (63 * ry + 2.75 rows) after its first, and the rectangle, a1 + 2 - (a0 & ~15) < 127 * rx + 19.75 columns
// and a1 + 2 - a0 < 63 * ry + 4.75 rows, fits the box.  Past 2^22 the error grows with s until the spare runs out:
// a 13,162,541-row source resized to 12,210,337 rows needs 74 rows where the box has 73.  Larger sources take
// k_resize, which stages nothing.  tests/test_resize_geometry.py checks every tile on sweeps of sizes.
constexpr int RT_MAX_BYTES = 64 * 1024;
constexpr int RT_SRC_LIMIT = 1 << 22;

template <bool VEC>
__global__ void __launch_bounds__(256)
k_resize_tiled(const __grid_constant__ CUtensorMap tmap, uint8_t *__restrict__ dst, unsigned dw, unsigned dh, unsigned sw,
               unsigned sh, unsigned n, unsigned pitch /* bytes, multiple of 16 = the TMA box width */, unsigned max_rows,
               unsigned ty0 /* first row tile of the launch: for_row_groups */) {
  extern __shared__ __align__(128) uint8_t s_tile[];
  __shared__ __align__(8) uint64_t bar;
  __shared__ unsigned s_roff[8 * RS_ROWS];           // byte offset of source row y0 in the staged rectangle
  __shared__ float s_dy[8 * RS_ROWS], s_omy[8 * RS_ROWS];   // pre-scaled y weights
  __shared__ unsigned s_reg[2];                      // cxa (first staged column, 16-aligned), cya (first staged row)
  const unsigned tid = threadIdx.x;
  const unsigned tx0 = blockIdx.x * 128, y0 = (blockIdx.y + ty0) * 8 * RS_ROWS;
  if (tid == 0) {   // the mapping is monotonic: the tile's first / last pixel bound the rectangle
    unsigned a0, b0, a1, b1;
    float f;
    resize_axis(tx0, sw, dw, a0, b0, f);
    resize_axis(min(tx0 + 127u, dw - 1), sw, dw, a1, b1, f);
    const unsigned cxa = a0 & ~15u;                  // the inner TMA coordinate must be a multiple of 16 bytes
    const unsigned cols = a1 + 2 - cxa;              // taps x0 and x0 + 1
    resize_axis(y0, sh, dh, a0, b0, f);
    resize_axis(min(y0 + 8u * RS_ROWS - 1, dh - 1), sh, dh, a1, b1, f);
    s_reg[0] = cxa, s_reg[1] = a0;
    // the host's box covers every tile of a source below RT_SRC_LIMIT in both dimensions (proof above); never silently wrong
    if (cols > pitch || a1 + 2 - a0 > max_rows) __trap();
    mbar_init(&bar, 1);
    mbar_fence_init();
  }
  __syncthreads();
  const unsigned cxa = s_reg[0], cya = s_reg[1];
  if (tid < 8 * RS_ROWS) {
    const unsigned yy = y0 + tid;
    unsigned a = cya, b = 0;
    float fr = 0.0f;
    if (yy < dh) resize_axis(yy, sh, dh, a, b, fr);
    s_roff[tid] = (a - cya) * pitch;
    s_dy[tid] = __fmul_rn(fr, RS_WY_SCALE), s_omy[tid] = __fmul_rn(__fsub_rn(1.0f, fr), RS_WY_SCALE);
  }
  const unsigned x = tx0 + (tid & 31) * 4;
  const unsigned yl = (tid >> 5) * RS_ROWS, yb = y0 + yl;
  // The second tap of each axis is read at x0 + 1 / y0 + 1 WITHOUT the reference's clamp: x0 == sw - 1 only when the
  // clamped coordinate is exactly sw - 1, i.e. dx == 0, and then whatever (finite) byte sits at x0 + 1 is multiplied
  // by zero; same for y.  (TMA zero-fills outside the image and the rectangle has the spare column / row.)
  unsigned ox0[4];
  float dx[4], omx[4];
#pragma unroll
  for (int j = 0; j < 4; j++) {
    unsigned a, b;
    resize_axis(min(x + j, dw - 1), sw, dw, a, b, dx[j]);
    omx[j] = __fmul_rn(__fsub_rn(1.0f, dx[j]), RS_WX_SCALE);
    dx[j] = __fmul_rn(dx[j], RS_WX_SCALE);
    ox0[j] = a - cxa;
  }
  unsigned phase = 0;
  for (unsigned f = blockIdx.z; f < n; f += gridDim.z) {
    uint8_t *d = dst + (size_t)f * dw * dh;
    __syncthreads();                                 // the tables are written / the previous frame's taps are done
    // stage the source rectangle with ONE bulk tensor copy: no instructions per staged byte
    if (tid == 0) {
      mbar_expect_tx(&bar, pitch * max_rows);
      tma_load_3d(s_tile, &tmap, (int)(cxa / 4), (int)cya, (int)f, &bar);
    }
    mbar_wait(&bar, phase);
    phase ^= 1u;
    if (x < dw && yb < dh) {
      for (unsigned r = 0; r < (unsigned)RS_ROWS && yb + r < dh; r++) {
        const float omy = s_omy[yl + r], dy = s_dy[yl + r];
        const uint8_t *t0 = s_tile + s_roff[yl + r];
        float p[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const uint8_t *a = t0 + ox0[j], *b = a + pitch;
          p[j] = bilerp(u8_f(a[0]), u8_f(a[1]), u8_f(b[0]), u8_f(b[1]), omx[j], dx[j], omy, dy);
        }
        const uint32_t out = prmt(prmt(f_trunc_bits(p[0]), f_trunc_bits(p[1]), 0x0040), prmt(f_trunc_bits(p[2]), f_trunc_bits(p[3]), 0x0040), 0x5410);
        uint8_t *q = d + (size_t)(yb + r) * dw + x;
        if (VEC) {
          *reinterpret_cast<uint32_t *>(q) = out;
        } else {
          for (unsigned j = 0; j < 4 && x + j < dw; j++) q[j] = (uint8_t)(out >> (8 * j));
        }
      }
    }
  }
}

}  // namespace gsb

extern "C" {
int gs_b200_downsample_batch(uint8_t *dst, const uint8_t *src, unsigned sw, unsigned sh, unsigned n,
                             gs_b200_stream s) {
  GSB_ASSERT(dst && src && sw > 0 && sh > 0);  // reference :190
  const unsigned dw = sw / 2, dh = sh / 2;
  if (n == 0 || dw == 0 || dh == 0) return 0;
  cudaStream_t st = static_cast<cudaStream_t>(s);
  const unsigned zn = n < 65535u ? n : 65535u, gy = dh < gsb::GRID_FRAMES ? dh : gsb::GRID_FRAMES;
  if (gsb::tma_ok(src, sw) && reinterpret_cast<uintptr_t>(dst) % 8 == 0) {
    dim3 block(128), grid((dw / 8 + 127) / 128, gy, zn);
    GSB_LAUNCH(gsb::k_downsample_vec, grid, block, 0, st, dst, src, sw, sh, dw, dh, n);
  } else {
    dim3 block(32, 8), grid((dw + 31) / 32, min((dh + 7) / 8, gsb::GRID_FRAMES), zn);
    GSB_LAUNCH(gsb::k_downsample_generic, grid, block, 0, st, dst, src, sw, sh, dw, dh, n);
  }
  return 0;
}

int gs_b200_resize_batch(uint8_t *dst, unsigned dw, unsigned dh, const uint8_t *src, unsigned sw,
                         unsigned sh, unsigned n, gs_b200_stream s) {
  GSB_ASSERT(dst && src && dw > 0 && dh > 0 && sw > 0 && sh > 0);  // reference :172
  if (n == 0) return 0;
  // Exact 2:1 in both axes: sx = ((x + 0.5) * 2dw) / dw - 0.5 = 2x + 0.5 with every fp32 step exact while
  // (2x + 1) * dw < 2^24, so all four weights are 0.25, the products and their sum are exact, and the truncated
  // result is (a + b + c + d) / 4 -- gs_downsample's arithmetic (reference :189-197), bit for bit.  Checked against
  // the oracle's literal fp32 evaluation in tests/test_gpu_parity.py::test_stencils_vs_oracle (w/2, h/2 targets); the
  // bound is tight: dw = 2897 is the first size whose fp32 map is not 2x + 0.5 (tests/test_resize_geometry.py).
  if (sw == 2 * dw && sh == 2 * dh && (unsigned long long)(2 * dw) * dw < (1ull << 24) &&
      (unsigned long long)(2 * dh) * dh < (1ull << 24) && !gsb::force_generic())
    return gs_b200_downsample_batch(dst, src, sw, sh, n, s);
  const unsigned tiles_y = (dh + 8 * gsb::RS_ROWS - 1) / (8 * gsb::RS_ROWS);
  dim3 grid((dw + 127) / 128, 1, n < gsb::GRID_FRAMES ? n : gsb::GRID_FRAMES);
  const bool aligned8 = sw % 8 == 0 && reinterpret_cast<uintptr_t>(src) % 8 == 0;   // every source row 8-byte aligned
  const bool vec_dst = dw % 4 == 0 && reinterpret_cast<uintptr_t>(dst) % 4 == 0;
  if (sw < (unsigned)gsb::RT_SRC_LIMIT && sh < (unsigned)gsb::RT_SRC_LIMIT) {
    // staged-tile kernel: bound the source rectangle of a 128 x 64 dst tile (+3 columns of alignment slack, +2 rows / columns
    // of neighbours) and use it when it fits the shared-memory budget.  Below the size limit the ratios are below 2^22,
    // so the conversions to unsigned below stay in range.
    const double rx = (double)sw / dw, ry = (double)sh / dh;
    const unsigned cols = (unsigned)(127.0 * rx) + 22, rows = (unsigned)((8.0 * gsb::RS_ROWS - 1) * ry) + 6;   // spare: fp32 vs double, 16-byte alignment
    const unsigned pitch = (cols + 15) / 16 * 16;
    const size_t bytes = (size_t)pitch * rows;
    const bool pairs_case = aligned8 && sw == 2 * dw;     // exact 2:1 in x: the 64-bit pair loads of k_resize are already good
    // one tensor map per frame group (grid z).  The first group's is made up front: a map the driver refuses takes
    // k_resize below, before anything is queued.  The later groups differ only in base (16-byte aligned, as the first)
    // and in a frame count no larger.
    CUtensorMap tm;
    const auto group_map = [&](unsigned f0, unsigned c) {
      return gsb::make_tmap_u8frames(&tm, src + (size_t)f0 * sw * sh, sw, sh, c, pitch / 4, rows);
    };
    if (bytes <= (size_t)gsb::RT_MAX_BYTES && pitch <= 1024 && rows <= 256 && !pairs_case && gsb::tma_ok(src, sw) &&
        group_map(0, n < gsb::GRID_FRAMES ? n : gsb::GRID_FRAMES)) {
      return gsb::for_frame_groups(n, [&](unsigned f0, unsigned c) {
        if (f0 && !group_map(f0, c)) return gsb::record_error(cudaErrorInvalidValue, __FILE__, __LINE__);
        grid.z = c;
        return gsb::for_row_groups(tiles_y, [&](unsigned t0, unsigned cy) {
          grid.y = cy;
          return gsb::launch(__FILE__, __LINE__, vec_dst ? gsb::k_resize_tiled<true> : gsb::k_resize_tiled<false>, grid, 256,
                             bytes, static_cast<cudaStream_t>(s), tm, dst + (size_t)f0 * dw * dh, dw, dh, sw, sh, c, pitch, rows,
                             t0);
        });
      });
    }
  }
  return gsb::for_row_groups(tiles_y, [&](unsigned t0, unsigned cy) {
    grid.y = cy;
    return gsb::launch(__FILE__, __LINE__, vec_dst ? gsb::k_resize<true> : gsb::k_resize<false>, grid, 256, 0,
                       static_cast<cudaStream_t>(s), dst, dw, dh, src, sw, sh, n, aligned8, t0);
  });
}
}
