// filter.cu -- gs_filter (reference grayskull.h:255-266) and gs_match_template / gs_find_best_match
// (grayskull.h:705-738); SURVEY.md 8f "next" item N3.
//
// gs_filter, 3x3 fast path (k_filter3): a thread owns 8 adjacent pixels and walks a 16-row band.  Per source
// row it loads its 8 bytes plus the word on either side and forms, for every pixel, the 32-bit window
// (x-1, x, x+1, x+2) with funnel shifts (2 of every 4 windows are free: one is the word itself).  Each kernel
// row is one packed int8x4 word (k0, k1, k2, 0), so an output pixel is three chained IDP.4A (u8 x s8 -> s32)
// over the windows of rows y-1, y, y+1; windows are built once per source row and reused by three output rows.
// `sum / norm` in the reference divides an int by an unsigned (the int is converted first, the quotient goes
// back into the int before the clamp).  For norm >= 2 this is min(255, umulhi((unsigned)sum, M)),
// M = floor(2^32 / norm) + 1: exact for the non-negative sums the weights can produce (host-checked:
// max_sum * norm < 2^32) and >= 255 -- as in the reference -- for negative ones (host-checked).  norm == 1
// is a plain clamp.  Anything else (other kernel sizes, ragged widths, exotic norms) takes k_filter_generic,
// which evaluates the reference's expression literally.
//
// gs_match_template (k_match_template): a thread owns 4 adjacent result columns of one row.  Per template
// word (4 taps) it loads one new image word, builds the 4 byte-shifted windows with funnel shifts, takes
// |I - T| on four bytes at once (VABSDIFF4.U8) and squares-and-accumulates it with one IDP.4A (u8 x u8):
// 11 instructions per 16 squared differences.  Row sums are u32 (exact below 66051 taps per row), totals u64.
#include "common.cuh"

namespace gsb {

__device__ __forceinline__ int dp4a_us(uint32_t a, uint32_t b, int c) {
  int d;
  asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  return d;
}
__device__ __forceinline__ uint32_t dp4a_uu(uint32_t a, uint32_t b, uint32_t c) {
  uint32_t d;
  asm("dp4a.u32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  return d;
}

constexpr int F3_ROWS = 16;

template <bool NORM1>
__global__ void __launch_bounds__(256)
k_filter3(uint8_t *__restrict__ dst, const uint8_t *__restrict__ src, unsigned w, unsigned h, unsigned n,
          uint32_t k0, uint32_t k1, uint32_t k2, uint32_t magic) {
  const unsigned x = (blockIdx.x * 32 + (threadIdx.x & 31)) * 8;
  const unsigned yb = (blockIdx.y * 8 + (threadIdx.x >> 5)) * F3_ROWS;
  if (x >= w || yb >= h) return;
  for (unsigned f = blockIdx.z; f < n; f += gridDim.z) {
    const uint8_t *s = src + (size_t)f * w * h;
    uint8_t *d = dst + (size_t)f * w * h;
    auto windows = [&](unsigned y, uint32_t (&win)[8]) {   // y may be "-1" (wraps) or >= h: zero row
      uint2 c = make_uint2(0, 0);
      uint32_t l = 0, r = 0;
      if (y < h) {
        const uint8_t *row = s + (size_t)y * w + x;
        c = __ldg(reinterpret_cast<const uint2 *>(row));
        if (x) l = __ldg(reinterpret_cast<const uint32_t *>(row) - 1);
        if (x + 8 < w) r = __ldg(reinterpret_cast<const uint32_t *>(row) + 2);
      }
      win[0] = __funnelshift_r(l, c.x, 24), win[1] = c.x;
      win[2] = __funnelshift_r(c.x, c.y, 8), win[3] = __funnelshift_r(c.x, c.y, 16);
      win[4] = __funnelshift_r(c.x, c.y, 24), win[5] = c.y;
      win[6] = __funnelshift_r(c.y, r, 8), win[7] = __funnelshift_r(c.y, r, 16);
    };
    uint32_t a[8], b[8], c[8];
    windows(yb - 1, a);
    windows(yb, b);
#pragma unroll 2
    for (unsigned rr = 0; rr < (unsigned)F3_ROWS; rr++) {
      const unsigned y = yb + rr;
      if (y >= h) break;
      windows(y + 1, c);
      uint32_t q[8];
#pragma unroll
      for (int j = 0; j < 8; j++) {
        const int sum = dp4a_us(c[j], k2, dp4a_us(b[j], k1, dp4a_us(a[j], k0, 0)));
        if (NORM1) q[j] = (uint32_t)min(max(sum, 0), 255);
        else q[j] = min(__umulhi((uint32_t)sum, magic), 255u);
      }
      uint2 o;
      o.x = q[0] | (q[1] << 8) | (q[2] << 16) | (q[3] << 24);
      o.y = q[4] | (q[5] << 8) | (q[6] << 16) | (q[7] << 24);
      st_cs_u2(d + (size_t)y * w + x, o);
#pragma unroll
      for (int j = 0; j < 8; j++) a[j] = b[j], b[j] = c[j];
    }
  }
}

// literal evaluation of grayskull.h:258-264 for any kernel size / norm (weights: kw*kh int8 on the device)
__global__ void __launch_bounds__(256)
k_filter_generic(uint8_t *__restrict__ dst, const uint8_t *__restrict__ src, unsigned w, unsigned h, unsigned n,
                 const int8_t *__restrict__ kern, unsigned kw, unsigned kh, unsigned norm) {
  const unsigned x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= w || y >= h) return;
  for (unsigned f = blockIdx.z; f < n; f += gridDim.z) {
    const uint8_t *s = src + (size_t)f * w * h;
    int sum = 0;
    for (unsigned j = 0; j < kh; j++) {
      const unsigned sy = y + j - kh / 2;            // unsigned wrap == out of bounds, like gs_get
      if (sy >= h) continue;
      for (unsigned i = 0; i < kw; i++) {
        const unsigned sx = x + i - kw / 2;
        if (sx < w) sum += (int)__ldg(s + (size_t)sy * w + sx) * (int)__ldg(kern + j * kw + i);
      }
    }
    const int v = (int)((unsigned)sum / norm);
    dst[(size_t)f * w * h + (size_t)y * w + x] = (uint8_t)min(255, max(0, v));
  }
}

// ---- template matching ---------------------------------------------------------------------
// tpack: th rows of twords = ceil(tw/4) little-endian words, zero padded
__global__ void k_pack_template(uint32_t *__restrict__ tpack, const uint8_t *__restrict__ tmpl, unsigned tw, unsigned th,
                                unsigned twords) {
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= twords * th) return;
  const unsigned ty = i / twords, k = i % twords;
  uint32_t v = 0;
  for (unsigned b = 0; b < 4; b++)
    if (4 * k + b < tw) v |= (uint32_t)tmpl[(size_t)ty * tw + 4 * k + b] << (8 * b);
  tpack[i] = v;
}

__device__ __forceinline__ uint8_t template_score(unsigned long long ssd, unsigned long long max_diff) {
  const unsigned long long score = ssd * 255ull / max_diff;                     // reference :720-721
  return (uint8_t)(255u - (unsigned)(score < 255ull ? score : 255ull));
}

// fast path: w % 4 == 0, frames word aligned
__global__ void __launch_bounds__(256)
k_match_template(uint8_t *__restrict__ result, const uint8_t *__restrict__ img, unsigned w, unsigned h, unsigned n,
                 const uint32_t *__restrict__ tpack, unsigned tw, unsigned th, unsigned twords) {
  const unsigned rw = w - tw + 1, rh = h - th + 1, wwords = w / 4;
  const unsigned cx = blockIdx.x * 32 + (threadIdx.x & 31);       // word column: results 4*cx .. 4*cx+3
  const unsigned ry = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (4 * cx >= rw || ry >= rh) return;
  const uint32_t tail_mask = (tw & 3) ? (0xFFFFFFFFu >> (8 * (4 - (tw & 3)))) : 0xFFFFFFFFu;
  const unsigned long long max_diff = (unsigned long long)tw * th * 255ull * 255ull;
  for (unsigned f = blockIdx.z; f < n; f += gridDim.z) {
    const uint32_t *base = reinterpret_cast<const uint32_t *>(img + (size_t)f * w * h);
    unsigned long long tot0 = 0, tot1 = 0, tot2 = 0, tot3 = 0;
    for (unsigned ty = 0; ty < th; ty++) {
      const uint32_t *row = base + (size_t)(ry + ty) * wwords;
      const uint32_t *trow = tpack + (size_t)ty * twords;
      uint32_t s0 = 0, s1 = 0, s2 = 0, s3 = 0;
      uint32_t A = __ldg(row + cx);
      for (unsigned k = 0; k < twords; k++) {
        const uint32_t B = cx + k + 1 < wwords ? __ldg(row + cx + k + 1) : 0u;
        const uint32_t T = __ldg(trow + k);
        uint32_t d0 = __vabsdiffu4(A, T), d1 = __vabsdiffu4(__funnelshift_r(A, B, 8), T);
        uint32_t d2 = __vabsdiffu4(__funnelshift_r(A, B, 16), T), d3 = __vabsdiffu4(__funnelshift_r(A, B, 24), T);
        if (k + 1 == twords) d0 &= tail_mask, d1 &= tail_mask, d2 &= tail_mask, d3 &= tail_mask;
        s0 = dp4a_uu(d0, d0, s0), s1 = dp4a_uu(d1, d1, s1), s2 = dp4a_uu(d2, d2, s2), s3 = dp4a_uu(d3, d3, s3);
        A = B;
      }
      tot0 += s0, tot1 += s1, tot2 += s2, tot3 += s3;
    }
    uint8_t *o = result + (size_t)f * rw * rh + (size_t)ry * rw + 4 * cx;
    o[0] = template_score(tot0, max_diff);
    if (4 * cx + 1 < rw) o[1] = template_score(tot1, max_diff);
    if (4 * cx + 2 < rw) o[2] = template_score(tot2, max_diff);
    if (4 * cx + 3 < rw) o[3] = template_score(tot3, max_diff);
  }
}

__global__ void __launch_bounds__(256)
k_match_template_generic(uint8_t *__restrict__ result, const uint8_t *__restrict__ img, unsigned w, unsigned h, unsigned n,
                         const uint8_t *__restrict__ tmpl, unsigned tw, unsigned th) {
  const unsigned rw = w - tw + 1, rh = h - th + 1;
  const unsigned rx = blockIdx.x * 32 + (threadIdx.x & 31), ry = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (rx >= rw || ry >= rh) return;
  const unsigned long long max_diff = (unsigned long long)tw * th * 255ull * 255ull;
  for (unsigned f = blockIdx.z; f < n; f += gridDim.z) {
    const uint8_t *s = img + (size_t)f * w * h;
    unsigned long long tot = 0;
    for (unsigned ty = 0; ty < th; ty++) {
      const uint8_t *p = s + (size_t)(ry + ty) * w + rx, *q = tmpl + (size_t)ty * tw;
      for (unsigned tx = 0; tx < tw; tx++) {
        const int diff = (int)__ldg(p + tx) - (int)__ldg(q + tx);
        tot += (unsigned long long)(diff * diff);
      }
    }
    result[(size_t)f * rw * rh + (size_t)ry * rw + rx] = template_score(tot, max_diff);
  }
}

// gs_find_best_match: first strict maximum in raster order == max over keys (score << 32 | ~index); a
// zero map gives (0, 0) like the reference's initial value.  Chunks of a map reduce to one 64-bit
// atomicMax each; a second tiny kernel turns the winning key into a point.
constexpr unsigned BM_CHUNK = 256 * 16 * 16;   // bytes of one result map per CTA

__global__ void __launch_bounds__(256)
k_best_match_partial(unsigned long long *__restrict__ keys, const uint8_t *__restrict__ result, size_t px) {
  __shared__ unsigned long long s_key[8];
  const unsigned f = blockIdx.y, tid = threadIdx.x;
  const uint8_t *r = result + (size_t)f * px;
  const size_t begin = (size_t)blockIdx.x * BM_CHUNK, end = begin + BM_CHUNK < px ? begin + BM_CHUNK : px;
  unsigned long long key = 0;
  const size_t abegin = (begin + ((16 - (reinterpret_cast<uintptr_t>(r) + begin)) & 15));   // first 16-B aligned byte
  auto take = [&](unsigned v, size_t i) {
    const unsigned long long k = ((unsigned long long)v << 32) | (0xFFFFFFFFu - (unsigned)i);
    key = k > key ? k : key;
  };
  for (size_t i = begin + tid; i < (abegin < end ? abegin : end); i += 256) take(__ldg(r + i), i);
  if (abegin < end) {
    const size_t nvec = (end - abegin) / 16;
    for (size_t v = tid; v < nvec; v += 256) {
      const uint4 q = __ldg(reinterpret_cast<const uint4 *>(r + abegin) + v);
      const uint32_t ws[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
      for (int k = 0; k < 4; k++) {
        if (ws[k] == 0) continue;                       // score 0 never beats the initial best
#pragma unroll
        for (int b = 0; b < 4; b++) take((ws[k] >> (8 * b)) & 0xFFu, abegin + v * 16 + 4 * k + b);
      }
    }
    for (size_t i = abegin + nvec * 16 + tid; i < end; i += 256) take(__ldg(r + i), i);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long other = __shfl_xor_sync(0xFFFFFFFFu, key, o);
    key = other > key ? other : key;
  }
  if ((tid & 31) == 0) s_key[tid >> 5] = key;
  __syncthreads();
  if (tid == 0) {
    for (int k = 1; k < 8; k++) key = s_key[k] > key ? s_key[k] : key;
    if (key >> 32) atomicMax(keys + f, key);
  }
}

__global__ void k_best_match_final(unsigned *__restrict__ best_xy, const unsigned long long *__restrict__ keys, unsigned rw,
                                   unsigned n) {
  const unsigned f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n) return;
  const unsigned long long key = keys[f];
  const unsigned idx = (key >> 32) ? 0xFFFFFFFFu - (unsigned)(key & 0xFFFFFFFFu) : 0u;
  best_xy[2 * f] = idx % rw;
  best_xy[2 * f + 1] = idx / rw;
}

}  // namespace gsb

extern "C" {

int gs_b200_filter_batch(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n, const int8_t *kernel,
                         unsigned kw, unsigned kh, unsigned norm, gs_b200_stream s) {
  GSB_ASSERT(dst && src && w > 0 && h > 0 && norm > 0);   // reference :257
  if (n == 0) return 0;
  cudaStream_t st = static_cast<cudaStream_t>(s);
  const unsigned zn = n < 65535u ? n : 65535u;
  const bool has_kernel = kernel && kw > 0 && kh > 0;     // an invalid kernel image iterates over nothing: sum = 0
  if (has_kernel && kw == 3 && kh == 3 && w % 8 == 0 && reinterpret_cast<uintptr_t>(src) % 8 == 0 &&
      reinterpret_cast<uintptr_t>(dst) % 8 == 0) {
    unsigned long long pos = 0, neg = 0;
    uint32_t kr[3];
    for (int j = 0; j < 3; j++) {
      kr[j] = 0;
      for (int i = 0; i < 3; i++) {
        const int v = kernel[j * 3 + i];
        kr[j] |= (uint32_t)(uint8_t)v << (8 * i);
        if (v > 0) pos += 255ull * v;
        else neg += 255ull * (unsigned)(-v);
      }
    }
    const bool magic_ok = norm >= 2 && pos * norm < (1ull << 32) && ((1ull << 32) - neg) / norm >= 256;
    if (norm == 1 || magic_ok) {
      dim3 grid((w / 8 + 31) / 32, (h + 8 * gsb::F3_ROWS - 1) / (8 * gsb::F3_ROWS), zn);
      GSB_ASSERT(grid.y <= 65535u);
      const uint32_t magic = norm == 1 ? 0 : (uint32_t)((1ull << 32) / norm + 1);
      GSB_LAUNCH(norm == 1 ? gsb::k_filter3<true> : gsb::k_filter3<false>, grid, 256, 0, st, dst, src, w, h, n, kr[0], kr[1],
                 kr[2], magic);
      return 0;
    }
  }
  const size_t kbytes = has_kernel ? (size_t)kw * kh : 0;
  // The weights go to the device by a copy from the caller's (pageable) host memory.  A graph would capture the host
  // pointer, not the values, so this path refuses capture; the 3x3 path above passes its weights by value.
  if (kbytes && gsb::capturing(st)) {
    gsb::record_error(cudaErrorStreamCaptureUnsupported, __FILE__, __LINE__);
    return (int)cudaErrorStreamCaptureUnsupported;
  }
  int8_t *dk = static_cast<int8_t *>(gsb::workspace(st, gsb::WS_HIST, kbytes + 16));
  if (!dk) return gsb::workspace_error();
  if (kbytes) GSB_CHECK(cudaMemcpyAsync(dk, kernel, kbytes, cudaMemcpyHostToDevice, st));
  dim3 grid((w + 31) / 32, (h + 7) / 8, zn);
  GSB_ASSERT(grid.y <= 65535u);
  GSB_LAUNCH(gsb::k_filter_generic, grid, 256, 0, st, dst, src, w, h, n, dk, has_kernel ? kw : 0, has_kernel ? kh : 0, norm);
  return 0;
}

int gs_b200_match_template_batch(uint8_t *result, const uint8_t *img, unsigned w, unsigned h, unsigned n,
                                 const uint8_t *tmpl, unsigned tw, unsigned th, gs_b200_stream s) {
  GSB_ASSERT(result && img && tmpl && w > 0 && h > 0 && tw > 0 && th > 0);   // reference :706
  GSB_ASSERT(w >= tw && h >= th);                                            // reference :707
  if (n == 0) return 0;
  cudaStream_t st = static_cast<cudaStream_t>(s);
  const unsigned rw = w - tw + 1, rh = h - th + 1;
  const unsigned zn = n < 65535u ? n : 65535u;
  if (w % 4 == 0 && reinterpret_cast<uintptr_t>(img) % 4 == 0 && tw < 66051u) {
    const unsigned twords = (tw + 3) / 4;
    uint32_t *tpack = static_cast<uint32_t *>(gsb::workspace(st, gsb::WS_HIST, sizeof(uint32_t) * (size_t)twords * th));
    if (!tpack) return gsb::workspace_error();
    GSB_LAUNCH(gsb::k_pack_template, (twords * th + 255) / 256, 256, 0, st, tpack, tmpl, tw, th, twords);
    dim3 grid(((rw + 3) / 4 + 31) / 32, (rh + 7) / 8, zn);
    GSB_ASSERT(grid.y <= 65535u);
    GSB_LAUNCH(gsb::k_match_template, grid, 256, 0, st, result, img, w, h, n, tpack, tw, th, twords);
  } else {
    dim3 grid((rw + 31) / 32, (rh + 7) / 8, zn);
    GSB_ASSERT(grid.y <= 65535u);
    GSB_LAUNCH(gsb::k_match_template_generic, grid, 256, 0, st, result, img, w, h, n, tmpl, tw, th);
  }
  return 0;
}

int gs_b200_find_best_match_batch(struct gs_point *best, const uint8_t *result, unsigned rw, unsigned rh, unsigned n,
                                  gs_b200_stream s) {
  GSB_ASSERT(best && result && rw > 0 && rh > 0);   // reference :727
  GSB_ASSERT((unsigned long long)rw * rh < 0xFFFFFFFFull);
  if (n == 0) return 0;
  cudaStream_t st = static_cast<cudaStream_t>(s);
  GSB_ASSERT(n <= 65535u);
  const size_t px = (size_t)rw * rh;
  unsigned long long *keys = static_cast<unsigned long long *>(gsb::workspace(st, gsb::WS_HIST, sizeof(unsigned long long) * n));
  if (!keys) return gsb::workspace_error();
  GSB_CHECK(cudaMemsetAsync(keys, 0, sizeof(unsigned long long) * n, st));
  dim3 grid((unsigned)((px + gsb::BM_CHUNK - 1) / gsb::BM_CHUNK), n);
  GSB_LAUNCH(gsb::k_best_match_partial, grid, 256, 0, st, keys, result, px);
  GSB_LAUNCH(gsb::k_best_match_final, (n + 127) / 128, 128, 0, st, reinterpret_cast<unsigned *>(best), keys, rw, n);
  return 0;
}
}
