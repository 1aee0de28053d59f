// morph.cu -- gs_b200_erode_n_batch / gs_b200_dilate_n_batch: `iters` passes of the 3x3 gs_erode / gs_dilate
// (reference grayskull.h:285-304) in one call, the repeated morphology of the reference CLI's `morph <op> <n>`
// (nanomagick.c:110-135).
//
// The reference's 3x3 op takes the min (max) over the IN-IMAGE pixels of the neighbourhood.  `iters` passes of it
// give, at (x, y), the min (max) over the in-image pixels of the (2N+1) x (2N+1) square centred there, N = iters
// (each pass reaches one pixel further in L-inf, and any in-image pixel within N can be reached by stepping
// componentwise towards it without leaving the image).  So the result is separable -- a clipped row window, then a
// clipped column window -- only Nx = min(N, w-1) and Ny = min(N, h-1) matter, and padding with the identity (255 for
// erode, 0 for dilate) gives the clipped window exactly.
//
//   * iters == 0 copies src to dst; iters == 1 is gs_b200_erode_batch / gs_b200_dilate_batch itself.
//   * path A, 2 <= N <= 16 on TMA-able geometry (w % 16 == 0, 16-byte aligned bases): k_morph_tma<OP, N>, one
//     launch, 2 B/px.  A TMA box of 72 words x (128 + 2N) rows (the same 16-byte column halo as k_stencil3_tma,
//     which is what bounds N) lands in shared memory.  Windows of 2N+1 are built by a ternary ladder: windows of 3,
//     9, 27 by VIMNMX3.U16x2 on 16-bit pair words, then one more 3-input min of three overlapping windows of the
//     largest power of 3 <= 2N+1.  Each warp forms the horizontal windows of whole tile rows in registers and writes
//     them back over the row; then each of 64 threads walks one 4-byte column word down the tile, ladder level by
//     ladder level in place, and stores the last level with streaming stores.
//   Path A takes N clamped to max(min(N, w-1), min(N, h-1)), the largest reach that still changes the result.
//   * 17 <= N <= 48 on TMA geometry: N passes then M passes are N+M passes, so path A launches of at most 16 are
//     composed through the workspace (ceil(N/16) launches, a remainder of 1 being the 3x3 kernel).
//   * path B, everything else (any width, alignment, N): a row pass into workspace, then a column pass into dst,
//     each van Herk / Gil-Werman: the padded line is cut into blocks of L = 2R+1, and the window starting in block
//     k is min(suffix of block k, prefix of block k+1), so the work per pixel does not depend on N.  Row pass: a
//     warp per 32 rows, 32 x 32-byte tiles moved through shared memory with coalesced byte accesses, a right-to-left
//     sweep for the suffixes and a left-to-right one for the prefixes.  Column pass: one thread per (column, block),
//     adjacent threads on adjacent columns.  Plain byte loads, 4 B/px of algorithmic traffic.  The workspace (path B
//     and the composed passes) holds at most 256 MiB of frames (or one frame, if a frame is larger): the passes run
//     over chunks of frames of that size.
#include <utility>

#include "common.cuh"

namespace gsb {

enum { MOP_ERODE = 1, MOP_DILATE = 2 };  // the same values as stencil3.cu's OP_ERODE / OP_DILATE

constexpr int MT_TW = 256;   // output tile width (pixels)
constexpr int MT_TH = 128;   // output tile height (rows)
constexpr int MT_PW = 72;    // smem row pitch in words: image bytes [x0-16, x0+272)
constexpr int MT_THREADS = 256;
constexpr int MT_MAX_N = 16;  // the 16-byte column halo of the TMA box
constexpr unsigned MT_COMPOSE_MAX = 3 * MT_MAX_N;
constexpr size_t MORPH_WS_BYTES = size_t(256) << 20;

template <int OP>
__device__ __forceinline__ uint32_t mm3(uint32_t a, uint32_t b, uint32_t c) {
  return OP == MOP_ERODE ? __vimin3_u16x2(a, b, c) : __vimax3_u16x2(a, b, c);
}
// the same on four packed bytes: split into pair words (bytes 0,2) and (1,3), repack
template <int OP>
__device__ __forceinline__ uint32_t mm3_bytes(uint32_t a, uint32_t b, uint32_t c) {
  const uint32_t lo = mm3<OP>(a & 0x00FF00FFu, b & 0x00FF00FFu, c & 0x00FF00FFu);
  const uint32_t hi = mm3<OP>(prmt(a, 0, 0x4341), prmt(b, 0, 0x4341), prmt(c, 0, 0x4341));
  return prmt(lo, hi, 0x6240);
}
__device__ __forceinline__ void st_cs_u1(void *p, uint32_t v) {
  asm volatile("st.global.cs.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

__host__ __device__ constexpr int pow3_le(int l) { return l >= 27 ? 27 : l >= 9 ? 9 : l >= 3 ? 3 : 1; }

// horizontal window of 2N+1 for a lane's 8 columns x..x+7.  wd = image bytes [x-16, x+24).  P[i] is the pair word
// (byte i, byte i+2), i.e. pixels (x+i-16, x+i-14); the ladder turns P[i] into the window of `m` pixels starting
// there, in place (ascending i only reads entries not yet overwritten).
template <int OP, int N>
__device__ __forceinline__ uint2 hwindow(const uint32_t (&wd)[10]) {
  constexpr int NP = 38, L = 2 * N + 1, M = pow3_le(L), E = (L - M) / 2;
  uint32_t P[NP];
#pragma unroll
  for (int g = 0; g < 10; g++) {
    const uint32_t s = __funnelshift_r(wd[g], g + 1 < 10 ? wd[g + 1] : 0u, 16);  // bytes 4g+2 .. 4g+5
    P[4 * g] = wd[g] & 0x00FF00FFu;
    P[4 * g + 1] = prmt(wd[g], 0, 0x4341);
    if (4 * g + 2 < NP) P[4 * g + 2] = s & 0x00FF00FFu;
    if (4 * g + 3 < NP) P[4 * g + 3] = prmt(s, 0, 0x4341);
  }
#pragma unroll
  for (int i = 0; i + 2 < NP; i++) P[i] = mm3<OP>(P[i], P[i + 1], P[i + 2]);
  if constexpr (M >= 9) {
#pragma unroll
    for (int i = 0; i + 6 < NP; i++) P[i] = mm3<OP>(P[i], P[i + 3], P[i + 6]);
  }
  if constexpr (M >= 27) {
#pragma unroll
    for (int i = 0; i + 18 < NP; i++) P[i] = mm3<OP>(P[i], P[i + 9], P[i + 18]);
  }
  // output pair words k = 0, 1, 4, 5 (pixels (x+k, x+k+2)) are the windows starting at pixel x+k-N: i = k-N+16
  uint32_t m[4];
  const int ks[4] = {0, 1, 4, 5};
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const int i = ks[j] - N + 16;
    m[j] = mm3<OP>(P[i], P[i + E], P[i + L - M]);
  }
  return make_uint2(prmt(m[0], m[1], 0x6240), prmt(m[2], m[3], 0x6240));
}

// one ladder level down a column word: col[r] = op(col[r], col[r+m], col[r+2m]) for r < rows
template <int OP, int m>
__device__ __forceinline__ void vlevel(uint32_t *col, int rows) {
#pragma unroll 4
  for (int r = 0; r < rows; r++)
    col[r * MT_PW] = mm3_bytes<OP>(col[r * MT_PW], col[(r + m) * MT_PW], col[(r + 2 * m) * MT_PW]);
}

template <int OP, int N>
__global__ void __launch_bounds__(MT_THREADS)
k_morph_tma(const __grid_constant__ CUtensorMap tmap, uint8_t *__restrict__ dst, unsigned w, unsigned h,
            unsigned tiles_x, unsigned tiles_y) {
  constexpr int R = MT_TH + 2 * N, L = 2 * N + 1, M = pow3_le(L), E = (L - M) / 2;
  __shared__ __align__(128) uint32_t tile[R * MT_PW];
  __shared__ __align__(8) uint64_t bar;

  unsigned bid = blockIdx.x;
  const unsigned tx = bid % tiles_x;
  bid /= tiles_x;
  const unsigned ty = bid % tiles_y;
  const unsigned frame = bid / tiles_y;
  const int x0 = tx * MT_TW, y0 = ty * MT_TH;

  if (threadIdx.x == 0) {
    mbar_init(&bar, 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(&bar, R * MT_PW * 4);
    tma_load_3d(tile, &tmap, x0 / 4 - 4, y0 - N, frame, &bar);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int hv = min(MT_TH, (int)h - y0);  // output rows of this tile
  const int rows = hv + 2 * N;             // tile rows they read
  mbar_wait(&bar, 0);

  // ---- horizontal: warp per tile row, lane per 8 columns, result written back over the row's bytes [x, x+8)
  const int x = x0 + lane * 8;
  uint32_t fix = 0;  // erode: bit g set when word g (image bytes x-16+4g ..) lies outside the image (TMA gave 0)
  if (OP == MOP_ERODE) {
#pragma unroll
    for (int g = 0; g < 10; g++) {
      const int xw = x - 16 + 4 * g;
      if (xw < 0 || xw >= (int)w) fix |= 1u << g;
    }
  }
  for (int r = warp; r < rows; r += MT_THREADS / 32) {
    uint32_t *row = tile + r * MT_PW + 2 * lane;
    uint32_t wd[10];
#pragma unroll
    for (int g = 0; g < 5; g++) {
      const uint2 v = *reinterpret_cast<const uint2 *>(row + 2 * g);
      wd[2 * g] = v.x, wd[2 * g + 1] = v.y;
    }
    if (OP == MOP_ERODE) {
      const int yimg = y0 - N + r;
      const uint32_t rowfix = (yimg < 0 || yimg >= (int)h) ? 0x3FFu : fix;
#pragma unroll
      for (int g = 0; g < 10; g++)
        if (rowfix >> g & 1u) wd[g] = 0xFFFFFFFFu;
    }
    const uint2 o = hwindow<OP, N>(wd);
    __syncwarp();
    *reinterpret_cast<uint2 *>(row + 4) = o;
  }
  __syncthreads();

  // ---- vertical: thread per 4-column word, the ladder in place down the tile, the last level stored
  const int c = threadIdx.x;
  if (c >= MT_TW / 4 || x0 + 4 * c >= (int)w) return;
  uint32_t *col = tile + 4 + c;
  if constexpr (M >= 3) vlevel<OP, 1>(col, hv + L - 3);
  if constexpr (M >= 9) vlevel<OP, 3>(col, hv + L - 9);
  if constexpr (M >= 27) vlevel<OP, 9>(col, hv + L - 27);
  uint8_t *q = dst + ((size_t)frame * h + y0) * w + x0 + 4 * c;
#pragma unroll 4
  for (int o = 0; o < hv; o++) {
    st_cs_u1(q, mm3_bytes<OP>(col[o * MT_PW], col[(o + E) * MT_PW], col[(o + L - M) * MT_PW]));
    q += w;
  }
}

// ---- path B: van Herk / Gil-Werman --------------------------------------------------------------------------------
// Along a line of `len` elements, padded position p holds element p - R (the identity outside [0, len)), and the output
// at element u is the window of L = 2R+1 padded positions starting at u: min(h[u], g[u+2R]) with h the suffix minimum
// and g the prefix minimum inside the blocks [kL, kL+L).
template <int OP>
__device__ __forceinline__ unsigned mop(unsigned a, unsigned b) {
  return OP == MOP_ERODE ? min(a, b) : max(a, b);
}

// Row pass: one warp per 32 rows, lane i walking row i.  32 x 32-byte tiles are read and written a row at a time (32
// consecutive bytes per warp access) through shared memory; the walk is along the tile's rows there.  A right-to-left
// sweep writes h into dst, then a left-to-right sweep carries g and replaces h[u] by min(h[u], g[u+2R]).
constexpr int RP_WARPS = 4;
template <int OP>
__global__ void __launch_bounds__(RP_WARPS * 32)
k_morph_rows(uint8_t *__restrict__ dst, const uint8_t *__restrict__ src, unsigned len, unsigned R,
             unsigned long long nrows) {
  typedef long long i64;
  __shared__ uint32_t tiles[RP_WARPS][2][32][33];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned long long row0 = ((unsigned long long)blockIdx.x * RP_WARPS + warp) * 32;
  if (row0 >= nrows) return;
  const int nr = (int)min(32ull, nrows - row0);
  const uint8_t *s = src + row0 * len;
  uint8_t *d = dst + row0 * len;
  uint32_t(*A)[33] = tiles[warp][0];
  uint32_t(*B)[33] = tiles[warp][1];
  const unsigned ident = OP == MOP_ERODE ? 255u : 0u;
  const i64 L = 2ll * R + 1, n = len;
  auto load_v = [&](i64 q) {  // A[r][j] = padded position q + j of row r
    const i64 e = q + lane - R;
    const bool in = e >= 0 && e < n;
    for (int r = 0; r < nr; r++) A[r][lane] = in ? s[(size_t)r * len + e] : ident;
    __syncwarp();
  };
  // right to left: suffix minima h[p] for p < len (positions >= len + R are the identity)
  const i64 top = (n + R + 31) / 32 * 32;
  i64 k = (top - 1) % L;  // block offset of the position being consumed
  unsigned c = ident;
  for (i64 q = top - 32; q >= 0; q -= 32) {
    load_v(q);
#pragma unroll 8
    for (int j = 31; j >= 0; j--) {
      if (k == L - 1) c = ident;
      c = mop<OP>(c, A[lane][j]);
      A[lane][j] = c;
      k = k ? k - 1 : L - 1;
    }
    __syncwarp();
    const i64 u = q + lane;
    if (u < n)
      for (int r = 0; r < nr; r++) d[(size_t)r * len + u] = (uint8_t)A[r][lane];
    __syncwarp();
  }
  // left to right: g over positions t, output u = t - 2R
  k = 0, c = ident;
  for (i64 q = 0; q < n + 2 * R; q += 32) {
    load_v(q);
    const i64 u = q - 2 * R + lane;
    const bool uin = u >= 0 && u < n;
    for (int r = 0; r < nr; r++) B[r][lane] = uin ? d[(size_t)r * len + u] : ident;
    __syncwarp();
#pragma unroll 8
    for (int j = 0; j < 32; j++) {
      if (k == 0) c = ident;
      c = mop<OP>(c, A[lane][j]);
      B[lane][j] = mop<OP>(B[lane][j], c);
      k = k + 1 == L ? 0 : k + 1;
    }
    __syncwarp();
    if (uin)
      for (int r = 0; r < nr; r++) d[(size_t)r * len + u] = (uint8_t)B[r][lane];
    __syncwarp();
  }
}

// Column pass: one thread per (column, block of L): adjacent threads take adjacent columns, so every access of a
// warp is 32 consecutive bytes of one row.  The thread walks block k backwards, parking the suffix minima in its own
// output bytes, then walks block k+1 forwards.
template <int OP>
__global__ void k_morph_cols(uint8_t *__restrict__ dst, const uint8_t *__restrict__ src, unsigned w, unsigned h,
                             unsigned R, unsigned long long ncols) {
  typedef unsigned long long u64;
  const u64 L = 2ull * R + 1, nb = (h - 1) / L + 1, total = nb * ncols;
  const unsigned ident = OP == MOP_ERODE ? 255u : 0u;
  const size_t es = w;
  for (u64 t = blockIdx.x * (u64)blockDim.x + threadIdx.x; t < total; t += (u64)gridDim.x * blockDim.x) {
    const u64 col = t % ncols, b0 = (t / ncols) * L;  // this thread's block starts at padded position b0
    const size_t base = (size_t)(col / w) * w * h + col % w;
    const uint8_t *s = src + base;
    uint8_t *d = dst + base;
    const u64 ob = min(b0 + L, (u64)h);  // outputs b0 .. ob-1 belong to this thread
    unsigned hc = ident;
#pragma unroll 4
    for (u64 p = min(b0 + L, (u64)h + R); p > b0;) {
      --p;
      if (p >= R) hc = mop<OP>(hc, s[(p - R) * es]);
      if (p < ob) d[p * es] = (uint8_t)hc;
    }
    // output b0+j = op(suffix of block k from b0+j, prefix of block k+1 up to b0+L+j-1)
    unsigned g = ident;
#pragma unroll 4
    for (u64 u = b0 + 1; u < ob; u++) {
      const u64 q = u + L - 1 - R;  // image element entering the prefix
      if (q < h) g = mop<OP>(g, s[q * es]);
      d[u * es] = (uint8_t)mop<OP>(d[u * es], g);
    }
  }
}

typedef void (*MorphTmaFn)(CUtensorMap, uint8_t *, unsigned, unsigned, unsigned, unsigned);
template <int OP, int... Ns>
static MorphTmaFn morph_tma_fn(unsigned n, std::integer_sequence<int, Ns...>) {
  static const MorphTmaFn table[] = {k_morph_tma<OP, Ns + 2>...};
  return table[n - 2];
}

// one launch of k_morph_tma<OP, k>; -1 if no tensor map could be made (the caller takes another path)
template <int OP>
static int morph_tma_step(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n, unsigned k,
                          cudaStream_t s) {
  CUtensorMap tmap;
  if (!make_tmap_u8frames(&tmap, src, w, h, n, MT_PW, MT_TH + 2 * k)) return -1;
  const unsigned tiles_x = (w + MT_TW - 1) / MT_TW, tiles_y = (h + MT_TH - 1) / MT_TH;
  const unsigned long long blocks = (unsigned long long)tiles_x * tiles_y * n;
  GSB_ASSERT(blocks < 0x7FFFFFFFull);
  GSB_LAUNCH(morph_tma_fn<OP>(k, std::make_integer_sequence<int, MT_MAX_N - 1>()), (unsigned)blocks, MT_THREADS, 0, s, tmap,
             dst, w, h, tiles_x, tiles_y);
  return 0;
}

template <int OP>
static int launch_morph_n(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n, unsigned iters,
                          cudaStream_t s) {
  if (n == 0) return 0;
  const size_t fb = (size_t)w * h;
  if (iters == 0) {
    GSB_CHECK(cudaMemcpyAsync(dst, src, fb * n, cudaMemcpyDeviceToDevice, s));
    return 0;
  }
  if (iters == 1)
    return OP == MOP_ERODE ? gs_b200_erode_batch(dst, src, w, h, n, s) : gs_b200_dilate_batch(dst, src, w, h, n, s);
  // only Nx = min(N, w-1) and Ny = min(N, h-1) matter; clamp before any index arithmetic, so a huge iters neither
  // overflows nor runs longer
  const unsigned nx = iters < w - 1 ? iters : w - 1, ny = iters < h - 1 ? iters : h - 1, ne = nx > ny ? nx : ny;
  if (ne <= 1)  // the 3x3 op already covers the frame
    return OP == MOP_ERODE ? gs_b200_erode_batch(dst, src, w, h, n, s) : gs_b200_dilate_batch(dst, src, w, h, n, s);
  CUtensorMap probe;  // TMA geometry, and a tensor map the driver accepts for it
  const bool tma = tma_ok(src, w) && tma_ok(dst, w) &&
                   make_tmap_u8frames(&probe, src, w, h, n, MT_PW, MT_TH + 2 * MT_MAX_N);
  if (ne <= MT_MAX_N && tma) return morph_tma_step<OP>(dst, src, w, h, n, ne, s);
  size_t chunk = MORPH_WS_BYTES / fb;
  if (chunk < 1) chunk = 1;
  if (chunk > n) chunk = n;
  // TMA geometry and N up to 3 x 16: passes of the TMA kernel composed through the workspace (N passes then M passes
  // are N+M passes), ceil(N/16) launches of 2 B/px, which beats the row / column passes up to N = 48 (DESIGN.md §6)
  if (ne <= MT_COMPOSE_MAX && tma) {
    uint8_t *ws = static_cast<uint8_t *>(workspace(s, WS_MORPH, chunk * fb));
    if (!ws) return gsb::workspace_error();
    const unsigned steps = (ne + MT_MAX_N - 1) / MT_MAX_N;
    for (size_t f0 = 0; f0 < n; f0 += chunk) {
      const unsigned c = (unsigned)(n - f0 < chunk ? n - f0 : chunk);
      const uint8_t *in = src + f0 * fb;
      unsigned left = ne;
      for (unsigned i = 1; i <= steps; i++) {  // the last step lands in dst, the one before in ws, ...
        uint8_t *out = (steps - i) % 2 ? ws : dst + f0 * fb;
        const unsigned k = left < MT_MAX_N ? left : MT_MAX_N;
        int rc;
        if (k == 1)
          rc = OP == MOP_ERODE ? gs_b200_erode_batch(out, in, w, h, c, s) : gs_b200_dilate_batch(out, in, w, h, c, s);
        else
          rc = morph_tma_step<OP>(out, in, w, h, c, k, s);
        if (rc) return rc > 0 ? rc : static_cast<int>(cudaErrorInvalidValue);  // the probe map was accepted
        left -= k, in = out;
      }
    }
    return 0;
  }
  // path B: row pass into the workspace, column pass into dst
  uint8_t *ws = static_cast<uint8_t *>(workspace(s, WS_MORPH, chunk * fb));
  if (!ws) return gsb::workspace_error();
  for (size_t f0 = 0; f0 < n; f0 += chunk) {
    const size_t c = n - f0 < chunk ? n - f0 : chunk;
    const unsigned long long rows = (unsigned long long)c * h, cols = (unsigned long long)c * w;
    const unsigned long long rblocks = (rows + RP_WARPS * 32 - 1) / (RP_WARPS * 32);
    GSB_ASSERT(rblocks < 0x7FFFFFFFull);
    GSB_LAUNCH(k_morph_rows<OP>, (unsigned)rblocks, RP_WARPS * 32, 0, s, ws, src + f0 * fb, w, nx, rows);
    const unsigned long long ctotal = ((h - 1) / (2ull * ny + 1) + 1) * cols;
    const unsigned cblocks = (unsigned)min((ctotal + 255) / 256, (unsigned long long)sm_count() * 64);
    GSB_LAUNCH(k_morph_cols<OP>, cblocks, 256, 0, s, dst + f0 * fb, ws, w, h, ny, cols);
  }
  return 0;
}

}  // namespace gsb

extern "C" {
int gs_b200_erode_n_batch(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n, unsigned iters,
                          gs_b200_stream s) {
  GSB_ASSERT(dst && src && w > 0 && h > 0);  // reference :287
  return gsb::launch_morph_n<gsb::MOP_ERODE>(dst, src, w, h, n, iters, static_cast<cudaStream_t>(s));
}
int gs_b200_dilate_n_batch(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n, unsigned iters,
                           gs_b200_stream s) {
  GSB_ASSERT(dst && src && w > 0 && h > 0);  // reference :287
  return gsb::launch_morph_n<gsb::MOP_DILATE>(dst, src, w, h, n, iters, static_cast<cudaStream_t>(s));
}
}
