// integral.cu -- gs_integral (reference grayskull.h:744-752): inclusive u32 summed-area table,
// ii[y][x] = sum of src over [0..x] x [0..y], modular 32-bit arithmetic (any association order
// is bit-identical).  Compulsory traffic: 1 B read + 4 B written per pixel.
//
// Batched path (n >= 32, w % 8 == 0, w <= 8192): k_integral_bands, single pass, 5 B/pixel + one
// re-read of a table row per band (from L2).  A CTA owns a band of 16 rows of one frame, a thread
// 8 columns.  SAT(x, y) = top(x) + sum_{i<=x} V(i, y), with V the vertical prefix inside the band
// (thread-local) and top = the table row just above the band.  All band-local work (pixel loads,
// V, the block-wide horizontal scans of the 16 row totals) happens BEFORE the CTA looks at the band
// above; then it waits for that band's flag, reads `top`, writes its own LAST row first and raises
// its flag, so the chain down a frame costs one row round trip per band while the other frames'
// bands (tickets are handed out band-major across frames) keep the SMs and HBM busy.
// Fallback (small batches, ragged widths): two passes, 13 B/pixel.
//   k_integral_rows : a warp per row; each lane takes 4 (vectorised) or 1 pixels per step,
//                     lane-local prefix + warp shuffle scan + running carry; writes row prefixes.
//   k_integral_cols : a thread per column; running sum down the rows, in place (coalesced over x).
#include "common.cuh"

namespace gsb {

template <bool VEC>
__global__ void k_integral_rows(uint32_t *__restrict__ ii, const uint8_t *__restrict__ src, unsigned w,
                                unsigned h, unsigned n) {
  const unsigned lane = threadIdx.x & 31;
  const unsigned long long row = (unsigned long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= (unsigned long long)h * n) return;
  const uint8_t *s = src + row * w;
  uint32_t *d = ii + row * w;
  uint32_t carry = 0;
  if (VEC) {
    for (unsigned x = lane * 4; x < ((w + 127) / 128) * 128; x += 128) {
      uint32_t v = x < w ? __ldg(reinterpret_cast<const uint32_t *>(s + x)) : 0u;
      uint32_t p0 = v & 0xFF, p1 = p0 + ((v >> 8) & 0xFF), p2 = p1 + ((v >> 16) & 0xFF), p3 = p2 + (v >> 24);
      uint32_t incl = p3;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, o);
        if (lane >= (unsigned)o) incl += t;
      }
      const uint32_t base = carry + incl - p3;
      if (x < w) *reinterpret_cast<uint4 *>(d + x) = make_uint4(base + p0, base + p1, base + p2, base + p3);
      carry += __shfl_sync(0xFFFFFFFFu, incl, 31);
    }
  } else {
    for (unsigned x = lane; x < ((w + 31) / 32) * 32; x += 32) {
      uint32_t p = x < w ? s[x] : 0u;
      uint32_t incl = p;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, o);
        if (lane >= (unsigned)o) incl += t;
      }
      if (x < w) d[x] = carry + incl;
      carry += __shfl_sync(0xFFFFFFFFu, incl, 31);
    }
  }
}

__global__ void k_integral_cols(uint32_t *__restrict__ ii, unsigned w, unsigned h, unsigned n) {
  const unsigned x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= w) return;
  for (unsigned f = blockIdx.y; f < n; f += gridDim.y) {
    uint32_t *p = ii + (size_t)f * w * h + x;
    uint32_t acc = 0;
    unsigned y = 0;
    for (; y + 4 <= h; y += 4) {
      uint32_t a = p[(size_t)y * w], b = p[(size_t)(y + 1) * w], c = p[(size_t)(y + 2) * w],
               d = p[(size_t)(y + 3) * w];
      a += acc, b += a, c += b, d += c;
      p[(size_t)y * w] = a, p[(size_t)(y + 1) * w] = b, p[(size_t)(y + 2) * w] = c, p[(size_t)(y + 3) * w] = d;
      acc = d;
    }
    for (; y < h; y++) acc += p[(size_t)y * w], p[(size_t)y * w] = acc;
  }
}

constexpr int IB_BH = 16;   // rows per band

// ctrl[0] = ticket counter, ctrl[1 + f * nbands + b] = 1 once band b of frame f has published its last row
template <int MAXT>   // block-size bound; per-row thread offsets live in shared memory to stay <= 64 registers
__global__ void __launch_bounds__(MAXT, 1024 / MAXT)
k_integral_bands(uint32_t *__restrict__ ii, const uint8_t *__restrict__ src, unsigned w, unsigned h, unsigned n,
                 unsigned nbands, unsigned *__restrict__ ctrl) {
  __shared__ uint32_t wtot[IB_BH][32];   // per-row warp totals
  __shared__ unsigned s_ticket;
  extern __shared__ uint32_t s_off[];    // [IB_BH][blockDim.x]: exclusive horizontal offset of each thread, per row
  const unsigned tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  if (tid == 0) s_ticket = atomicAdd(&ctrl[0], 1u);
  __syncthreads();
  const unsigned ticket = s_ticket;
  const unsigned band = ticket / n, frame = ticket % n;   // band-major: band b of every frame before band b+1
  const unsigned y0 = band * IB_BH;
  const unsigned rows = min((unsigned)IB_BH, h - y0);
  const unsigned x = tid * 8;
  const bool live = x < w;
  const uint8_t *sp = src + (size_t)frame * w * h + (size_t)y0 * w + x;
  uint32_t *dp = ii + (size_t)frame * w * h + (size_t)y0 * w + x;

  // ---- band-local work ----------------------------------------------------------------------
  // rows beyond the image read as zeros, so acc ends up holding V(., rows-1)
#define IB_LOAD_ROW(r) ((live && (unsigned)(r) < rows) ? __ldg(reinterpret_cast<const uint2 *>(sp + (size_t)(r) * w)) : make_uint2(0, 0))
  uint32_t acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};   // V(c, r): vertical prefix of this thread's 8 columns
#pragma unroll
  for (int r = 0; r < IB_BH; r++) {
    const uint2 p = IB_LOAD_ROW(r);
#pragma unroll
    for (int c = 0; c < 4; c++) {
      acc[c] += (p.x >> (8 * c)) & 0xFF;
      acc[4 + c] += (p.y >> (8 * c)) & 0xFF;
    }
    uint32_t t = acc[0] + acc[1] + acc[2] + acc[3] + acc[4] + acc[5] + acc[6] + acc[7];
    uint32_t incl = t;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t u = __shfl_up_sync(0xFFFFFFFFu, incl, o);
      if (lane >= (unsigned)o) incl += u;
    }
    if (lane == 31) wtot[r][warp] = incl;
    s_off[r * blockDim.x + tid] = incl - t;
  }
  __syncthreads();
  for (unsigned r = warp; r < (unsigned)IB_BH; r += nwarps) {   // row r's warp totals -> exclusive warp offsets
    const uint32_t t = lane < nwarps ? wtot[r][lane] : 0u;
    uint32_t incl = t;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t u = __shfl_up_sync(0xFFFFFFFFu, incl, o);
      if (lane >= (unsigned)o) incl += u;
    }
    wtot[r][lane] = incl - t;
  }
  __syncthreads();

  // ---- the row above the band -----------------------------------------------------------------
  uint32_t top[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (band > 0) {
    if (tid == 0) {
      volatile unsigned *flag = ctrl + 1 + (size_t)frame * nbands + (band - 1);
      while (*flag == 0) __nanosleep(40);
      __threadfence();
    }
    __syncthreads();
    if (live) {
      const uint4 a = __ldcg(reinterpret_cast<const uint4 *>(dp - w)), b = __ldcg(reinterpret_cast<const uint4 *>(dp - w) + 1);
      top[0] = a.x, top[1] = a.y, top[2] = a.z, top[3] = a.w, top[4] = b.x, top[5] = b.y, top[6] = b.z, top[7] = b.w;
    }
  }
  auto emit_row = [&](int r, const uint32_t (&v)[8]) {   // v = V(c, r) for the 8 columns
    uint32_t o[8];
    uint32_t run = s_off[r * blockDim.x + tid] + wtot[r][warp];
#pragma unroll
    for (int c = 0; c < 8; c++) run += v[c], o[c] = run + top[c];
    uint4 *q = reinterpret_cast<uint4 *>(dp + (size_t)r * w);
    q[0] = make_uint4(o[0], o[1], o[2], o[3]);
    q[1] = make_uint4(o[4], o[5], o[6], o[7]);
  };
  // last row first (acc holds V(., rows-1))
  if (live) {
    const int last = (int)rows - 1;
    uint32_t o[8];
    uint32_t run = s_off[last * blockDim.x + tid] + wtot[last][warp];
#pragma unroll
    for (int c = 0; c < 8; c++) run += acc[c], o[c] = run + top[c];
    uint4 *q = reinterpret_cast<uint4 *>(dp + (size_t)last * w);
    q[0] = make_uint4(o[0], o[1], o[2], o[3]);
    q[1] = make_uint4(o[4], o[5], o[6], o[7]);
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    volatile unsigned *flag = ctrl + 1 + (size_t)frame * nbands + band;
    *flag = 1u;
  }
  // remaining rows
  if (live) {
    uint32_t v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
    for (int r = 0; r < IB_BH - 1; r++) {
      const uint2 p = IB_LOAD_ROW(r);     // second read of the band's pixels: L1/L2 hits
#pragma unroll
      for (int c = 0; c < 4; c++) {
        v[c] += (p.x >> (8 * c)) & 0xFF;
        v[4 + c] += (p.y >> (8 * c)) & 0xFF;
      }
      if ((unsigned)r + 1 < rows) emit_row(r, v);
    }
  }
#undef IB_LOAD_ROW
}

// ---- round 2: k_integral_strips -- no inter-CTA chain on table rows, no band-local second pass ------------------
// k_integral_bands (kept below the batch threshold) chains the bands of a frame through a 16 KB table row and a flag
// and computes band-local vertical prefixes first (13.5 lane-instr/px, with stalls on the
// spin).  Here a CTA owns a 1024-column STRIP of one frame and walks down ALL its rows, RB at
// a time, with the previous output row in registers:
//     SAT(x, y) = SAT(x, y-1) + left(y) + sum_{i <= x} src(i, y)
// per row a thread needs (a) the sum of its 8 pixels -- two IDP.4A against 0x01010101 --, (b) an exclusive scan of
// those sums over the strip (warp shuffle scan + the warps' totals through shared memory), (c) `left(y)`, the row
// sums of the strips to its left: every strip publishes its RB row sums as soon as its scan is done (64-bit words
// carrying a band tag: no flag / fence pair) and a strip adds up the words of its left neighbours -- they run in
// lockstep, nobody waits for a predecessor's OUTPUT --, and (d) its 8 inclusive in-thread prefixes, ONE IDP.4A each
// (byte masks 0x01, 0x0101, ...) accumulated straight onto previous row + offset.  ~4.5 instructions per pixel
// instead of 13.5, ~50-100 registers.  The next RB rows are requested before the current ones are scanned.  Tickets
// are handed out strip-major, so a strip's left neighbours always hold earlier tickets (resident or done).
constexpr int IS_MINB = 4;                   // CTAs of 128 threads per SM the register allocation must allow

template <int IS_TPB, int RB>
__global__ void __launch_bounds__(IS_TPB, IS_MINB * 128 / IS_TPB)
k_integral_strips(uint32_t *__restrict__ ii, const uint8_t *__restrict__ src, unsigned w, unsigned h, unsigned n,
                  unsigned strips, unsigned nbands, unsigned *__restrict__ ticket_ctr,
                  unsigned long long *__restrict__ slots /* [n][strips][nbands][RB] : tag << 32 | row sum of the strip */) {
  __shared__ uint32_t wtot[RB][IS_TPB / 32];
  __shared__ uint32_t lsum[RB];
  __shared__ unsigned s_ticket;
  constexpr int IS_SW = IS_TPB * 8;
  constexpr uint32_t ONES = 0x01010101u;
  const unsigned tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s_ticket = atomicAdd(ticket_ctr, 1u);
  __syncthreads();
  const unsigned frame = s_ticket / strips, strip = s_ticket % strips;
  const unsigned x = strip * IS_SW + tid * 8;
  const bool live = x < w;
  const uint8_t *sp = src + (size_t)frame * w * h + x;
  uint32_t *dp = ii + (size_t)frame * w * h + x;
  unsigned long long *myslots = slots + ((size_t)frame * strips + strip) * nbands * RB;
  uint32_t prev[8] = {0, 0, 0, 0, 0, 0, 0, 0};            // the output row above

  uint2 pxn[RB];
#pragma unroll
  for (int r = 0; r < RB; r++) {
    pxn[r] = (live && (unsigned)r < h) ? __ldg(reinterpret_cast<const uint2 *>(sp)) : make_uint2(0u, 0u);
    sp += w;
  }
  for (unsigned band = 0; band < nbands; band++) {
    const unsigned y0 = band * RB, rows = min((unsigned)RB, h - y0);
    uint2 px[RB];
#pragma unroll
    for (int r = 0; r < RB; r++) px[r] = pxn[r];
#pragma unroll
    for (int r = 0; r < RB; r++) {                          // prefetch the next band (sp already points at it)
      pxn[r] = (live && y0 + RB + r < h) ? __ldg(reinterpret_cast<const uint2 *>(sp)) : make_uint2(0u, 0u);
      sp += w;
    }
    uint32_t off[RB];                                       // exclusive offset of this thread inside its warp, per row
#pragma unroll
    for (int r = 0; r < RB; r++) {
      const uint32_t t = __dp4a(px[r].y, ONES, __dp4a(px[r].x, ONES, 0u));
      uint32_t incl = t;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t u = __shfl_up_sync(0xFFFFFFFFu, incl, o);
        if (lane >= (unsigned)o) incl += u;
      }
      if (lane == 31) wtot[r][warp] = incl;
      off[r] = incl - t;
    }
    __syncthreads();
    if (tid < RB) {
      uint32_t tot = 0;
#pragma unroll
      for (int q = 0; q < IS_TPB / 32; q++) tot += wtot[tid][q];
      if (strip + 1 < strips)
        *reinterpret_cast<volatile unsigned long long *>(myslots + (size_t)band * RB + tid) = ((unsigned long long)(band + 1) << 32) | tot;
      lsum[tid] = 0;
    }
    __syncthreads();
    for (unsigned i = tid; i < RB * strip; i += IS_TPB) {   // (j, r): row sum r of strip j < strip
      const unsigned j = i / RB, r = i % RB;
      volatile unsigned long long *sl = slots + (((size_t)frame * strips + j) * nbands + band) * RB + r;
      unsigned long long v = *sl;
      while ((unsigned)(v >> 32) != band + 1) {
        __nanosleep(20);
        v = *sl;
      }
      atomicAdd(&lsum[r], (uint32_t)v);
    }
    __syncthreads();
    if (live) {
      uint32_t *q = dp + (size_t)y0 * w;
#pragma unroll
      for (int r = 0; r < RB; r++) {
        if ((unsigned)r < rows) {
          uint32_t base = off[r] + lsum[r];
#pragma unroll
          for (int k = 0; k < IS_TPB / 32; k++) base += (k < (int)warp) ? wtot[r][k] : 0u;
          const uint32_t base2 = __dp4a(px[r].x, ONES, base);
          prev[0] = __dp4a(px[r].x, 0x00000001u, prev[0] + base);
          prev[1] = __dp4a(px[r].x, 0x00000101u, prev[1] + base);
          prev[2] = __dp4a(px[r].x, 0x00010101u, prev[2] + base);
          prev[3] = prev[3] + base2;
          prev[4] = __dp4a(px[r].y, 0x00000001u, prev[4] + base2);
          prev[5] = __dp4a(px[r].y, 0x00000101u, prev[5] + base2);
          prev[6] = __dp4a(px[r].y, 0x00010101u, prev[6] + base2);
          prev[7] = __dp4a(px[r].y, ONES, prev[7] + base2);
          uint4 *q4 = reinterpret_cast<uint4 *>(q);
          q4[0] = make_uint4(prev[0], prev[1], prev[2], prev[3]);
          q4[1] = make_uint4(prev[4], prev[5], prev[6], prev[7]);
          q += w;
        }
      }
    }
    __syncthreads();                                        // wtot / lsum are reused by the next band
  }
}

}  // namespace gsb

extern "C" int gs_b200_integral_batch(uint32_t *ii, const uint8_t *src, unsigned w, unsigned h, unsigned n,
                                      gs_b200_stream s) {
  GSB_ASSERT(src && ii && w > 0 && h > 0);  // reference :745
  if (n == 0) return 0;
  cudaStream_t st = static_cast<cudaStream_t>(s);
  const bool aligned = reinterpret_cast<uintptr_t>(src) % 8 == 0 && reinterpret_cast<uintptr_t>(ii) % 16 == 0;
  {
    // 1024-column strips of 8 rows per step (128 threads) when that already fills the machine, else 512-column strips
    // of 16 rows per step (64 threads: twice the CTAs, twice the loads in flight per thread)
    const unsigned long long sms = (unsigned long long)gsb::sm_count();
    const bool narrow = (unsigned long long)n * ((w + 1023) / 1024) < 4 * sms && w <= 4096;
    const unsigned sw_cols = narrow ? 512u : 1024u, rb = narrow ? 16u : 8u;
    const unsigned strips = (w + sw_cols - 1) / sw_cols, nbands = (h + rb - 1) / rb;
    const unsigned long long ctas = (unsigned long long)n * strips;
    const char *env = getenv("GS_B200_INTEGRAL");      // test hook: "bands" or "strips"
    const bool want = env ? env[0] == 's' : ctas >= sms;
    if (want && !(env && env[0] == 'b') && w % 8 == 0 && strips <= 16 && aligned && !gsb::force_generic() && ctas < 0x7FFFFFFFull) {
      const size_t slot_bytes = sizeof(unsigned long long) * (size_t)ctas * nbands * rb;
      unsigned char *ws = static_cast<unsigned char *>(gsb::workspace(st, gsb::WS_INTEGRAL, 256 + slot_bytes));
      if (!ws) return gsb::workspace_error();
      GSB_CHECK(cudaMemsetAsync(ws, 0, 256 + (strips > 1 ? slot_bytes : 0), st));
      GSB_LAUNCH(narrow ? gsb::k_integral_strips<64, 16> : gsb::k_integral_strips<128, 8>, (unsigned)ctas, narrow ? 64 : 128, 0,
                 st, ii, src, w, h, n, strips, nbands, reinterpret_cast<unsigned *>(ws),
                 reinterpret_cast<unsigned long long *>(ws + 256));
      return 0;
    }
  }
  if (n >= 32 && w % 8 == 0 && w <= 8192 && aligned && !gsb::force_generic() &&
      (unsigned long long)n * ((h + gsb::IB_BH - 1) / gsb::IB_BH) < 0x7FFFFFFFull) {
    const unsigned nbands = (h + gsb::IB_BH - 1) / gsb::IB_BH;
    const size_t ctrl_bytes = sizeof(unsigned) * (1 + (size_t)n * nbands);
    unsigned *ctrl = static_cast<unsigned *>(gsb::workspace(st, gsb::WS_INTEGRAL, ctrl_bytes));
    if (!ctrl) return gsb::workspace_error();
    GSB_CHECK(cudaMemsetAsync(ctrl, 0, ctrl_bytes, st));
    const unsigned threads = ((w / 8 + 31) / 32) * 32;
    const size_t smem = sizeof(uint32_t) * gsb::IB_BH * threads;   // <= 64 KB
    GSB_LAUNCH(threads <= 512 ? gsb::k_integral_bands<512> : gsb::k_integral_bands<1024>, n * nbands, threads, smem, st, ii,
               src, w, h, n, nbands, ctrl);
    return 0;
  }
  const unsigned long long rows = (unsigned long long)h * n;
  const unsigned blocks = (unsigned)((rows + 7) / 8);
  const bool vec = (w % 4 == 0) && reinterpret_cast<uintptr_t>(src) % 4 == 0 &&
                   reinterpret_cast<uintptr_t>(ii) % 16 == 0;
  GSB_LAUNCH(vec ? gsb::k_integral_rows<true> : gsb::k_integral_rows<false>, blocks, 256, 0, st, ii, src, w, h, n);
  dim3 grid((w + 127) / 128, n < 65535u ? n : 65535u);
  GSB_LAUNCH(gsb::k_integral_cols, grid, 128, 0, st, ii, w, h, n);
  return 0;
}
