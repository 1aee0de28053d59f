// blobs.cu -- gs_blobs, gs_blob_corners, gs_perspective_correct (reference grayskull.h:325-444; SURVEY.md 8f N4).
//
// gs_blobs is a raster-order union-find over provisional labels in the reference; what it RETURNS has an
// order-free description (oracle/gs_oracle.c states and tests it against the reference):
//   * a pixel opens a new label exactly when it is foreground (>= 128) and neither its left nor its upper
//     neighbour is labelled -- while labels last: a run start with background above it ("seed"); seeds are
//     numbered in raster order from 1;
//   * unions keep the smaller root, so a component's label is the number of its raster-first pixel's seed;
//   * if more than nblobs seeds exist, nothing after the (nblobs+1)-th seed position gets a NEW label and a
//     pixel is labelled only through a labelled left / upper neighbour.
// GPU form, all per frame and batched over frames:
//   k_blob_mask     foreground bit masks (1 bit / pixel, 32 pixels per word)
//   k_blob_seed     seed bits = m & ~(m << 1) & ~m_above, their per-word exclusive counts, per-row totals
//   k_row_scan      raster-order numbering of the seeds (scan.cuh)
//   k_blob_overflow only when seeds > nblobs: one thread re-derives the rows after the overflow point with the
//                   adder trick  M = F & (~(F + G) | G),  G = F & M_above  (a carry ripples from each labelled
//                   contact to the end of its run), word by word with carry
//   k_blob_runs     parent[p] = first pixel of p's horizontal run (warp per row, run starts carried across words
//                   by a warp scan): horizontal connectivity is resolved at initialisation
//   k_blob_union    one atomicMin union per vertical contact SEGMENT (not per pixel)
//   k_blob_label    root -> seed number -> gs_label per pixel; area / box / coordinate sums accumulated with one
//                   atomic group per (32-pixel word, label)
//   k_blob_compact  blobs[0..m) in label order, centroid = sums / area in unsigned arithmetic (:397-398)
// Entries of `blobs` past the returned count are left untouched (the reference leaves first-pass leftovers there).
#include "common.cuh"
#include "scan.cuh"

namespace gsb {

struct BlobRec {  // struct gs_blob: u16 label (+2 pad), area, box {x, y, w, h}, centroid {x, y} = 32 bytes
  uint32_t w[8];
};

// bit x & 31 of word x >> 5 = (pixel >= 128); one warp per row, 128 pixels per iteration
__global__ void __launch_bounds__(256)
k_blob_mask(const uint8_t *__restrict__ img, unsigned w, unsigned h, unsigned mw, unsigned *__restrict__ mask,
            unsigned long long rows_total) {
  const unsigned long long gw = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (gw >= rows_total) return;
  const unsigned lane = threadIdx.x & 31;
  const uint8_t *row = img + gw * w;
  unsigned *mrow = mask + gw * mw;
  const bool vec = (w % 4u) == 0 && (reinterpret_cast<uintptr_t>(img) % 4u) == 0;
  for (unsigned xb = 0; xb < w; xb += 128) {
    const unsigned x4 = xb + 4 * lane;
    unsigned nib = 0;
    if (x4 < w) {
      if (vec) {
        const uint32_t v = __ldg(reinterpret_cast<const uint32_t *>(row + x4));
        nib = ((v >> 7) & 1u) | ((v >> 14) & 2u) | ((v >> 21) & 4u) | ((v >> 28) & 8u);
      } else {
#pragma unroll
        for (int j = 0; j < 4; j++)
          if (x4 + j < w && __ldg(row + x4 + j) >= 128) nib |= 1u << j;
      }
    }
    unsigned m = nib << (4 * (lane & 7));
    m |= __shfl_xor_sync(0xFFFFFFFFu, m, 1);
    m |= __shfl_xor_sync(0xFFFFFFFFu, m, 2);
    m |= __shfl_xor_sync(0xFFFFFFFFu, m, 4);
    const unsigned word = x4 >> 5;
    if ((lane & 7) == 0 && word < mw) mrow[word] = m;
  }
}

// seeds of one row: S = M & ~(M << 1 | carry) & ~M_above; sprefix[k] = seeds in words < k of the row; rowseed = total
__global__ void __launch_bounds__(256)
k_blob_seed(const unsigned *__restrict__ mask, unsigned h, unsigned mw, unsigned *__restrict__ seed,
            unsigned *__restrict__ sprefix, unsigned *__restrict__ rowseed, unsigned long long rows_total) {
  const unsigned long long gw = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (gw >= rows_total) return;
  const unsigned lane = threadIdx.x & 31;
  const unsigned y = (unsigned)(gw % h);
  const unsigned *m = mask + gw * mw;
  unsigned running = 0;
  for (unsigned k0 = 0; k0 < mw; k0 += 32) {
    const unsigned k = k0 + lane;
    unsigned s = 0;
    if (k < mw) {
      const unsigned cur = m[k], prev = k ? m[k - 1] : 0u, above = y ? (m - mw)[k] : 0u;   // (m - mw): k - mw would wrap
      s = cur & ~((cur << 1) | (prev >> 31)) & ~above;
      seed[gw * mw + k] = s;
    }
    const unsigned c = __popc(s);
    unsigned incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned u = __shfl_up_sync(0xFFFFFFFFu, incl, o);
      if (lane >= (unsigned)o) incl += u;
    }
    if (k < mw) sprefix[gw * mw + k] = running + incl - c;
    running += __shfl_sync(0xFFFFFFFFu, incl, 31);
  }
  if (lane == 0) rowseed[gw] = running;
}

// More seeds than labels: from the (nblobs+1)-th seed on, a pixel is labelled only through a labelled left / upper
// neighbour (reference :345-350).  One thread per frame (rare path): rows are sequential, words carry.
__global__ void k_blob_overflow(unsigned *__restrict__ mask, const unsigned *__restrict__ seed, const unsigned *__restrict__ sprefix,
                                const unsigned *__restrict__ rowoff, const unsigned *__restrict__ totals, unsigned h,
                                unsigned mw, unsigned nblobs, unsigned n) {
  const unsigned f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n || totals[f] <= nblobs) return;
  const unsigned *ro = rowoff + (size_t)f * h;
  unsigned lo = 0, hi = h - 1;                       // last row whose exclusive offset is <= nblobs: holds seed nblobs+1
  while (lo < hi) {
    const unsigned mid = (lo + hi + 1) / 2;
    if (ro[mid] <= nblobs) lo = mid;
    else hi = mid - 1;
  }
  const unsigned ys = lo;
  unsigned need = nblobs - ro[ys];                    // seeds of row ys that still get a label
  unsigned ks = 0, bs = 0;
  {
    const unsigned *sr = seed + ((size_t)f * h + ys) * mw, *sp = sprefix + ((size_t)f * h + ys) * mw;
    for (unsigned k = 0; k < mw; k++) {
      const unsigned c = __popc(sr[k]);
      if (sp[k] + c > need) {                         // the failing seed is in this word
        unsigned s = sr[k];
        for (unsigned i = sp[k]; i < need; i++) s &= s - 1;
        ks = k, bs = __ffs(s) - 1;
        break;
      }
    }
  }
  unsigned *M = mask + (size_t)f * h * mw;
  for (unsigned y = ys; y < h; y++) {
    unsigned *row = M + (size_t)y * mw;
    const unsigned *above = y ? row - mw : nullptr;
    unsigned carry = 0;
    for (unsigned k = (y == ys ? ks : 0); k < mw; k++) {
      unsigned F = row[k], keep = 0;
      if (y == ys && k == ks) {                       // pixels before the failing seed keep their labels; no run crosses it
        const unsigned low = bs ? (0xFFFFFFFFu >> (32 - bs)) : 0u;
        keep = F & low;
        F &= ~low;
      }
      const unsigned G = F & (above ? above[k] : 0u);
      const unsigned long long sum = (unsigned long long)F + G + carry;
      const unsigned gin = carry & F & 1u;            // a run continuing from the previous word, already labelled
      row[k] = (F & (~(unsigned)sum | G | gin)) | keep;
      carry = (unsigned)(sum >> 32);
    }
  }
}

// parent[p] = index (y*w + x, per frame) of the first pixel of p's horizontal run in M; 0xFFFFFFFF outside M
__global__ void __launch_bounds__(256)
k_blob_runs(const unsigned *__restrict__ mask, unsigned w, unsigned h, unsigned mw, unsigned *__restrict__ parent,
            unsigned long long rows_total) {
  const unsigned long long gw = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (gw >= rows_total) return;
  const unsigned lane = threadIdx.x & 31;
  const unsigned y = (unsigned)(gw % h);
  const unsigned *m = mask + gw * mw;
  unsigned *prow = parent + gw * w;
  const unsigned base = y * w;
  unsigned open_in = 0xFFFFFFFFu;                      // run open at the end of the previous chunk (its start), or none
  for (unsigned k0 = 0; k0 < mw; k0 += 32) {
    const unsigned k = k0 + lane;
    const unsigned cur = k < mw ? m[k] : 0u, prev = (k && k < mw) ? m[k - 1] : 0u;
    const unsigned starts = cur & ~((cur << 1) | (prev >> 31));
    // open(k): start of the run that contains bit 31 of word k.  f_k(x) = has ? val : x  (pass-through when the word is
    // all ones without a start); composed by a warp scan
    bool has = true;
    unsigned val = 0xFFFFFFFFu;
    if (cur >> 31) {
      if (starts) val = base + 32 * k + (31 - __clz(starts));
      else has = false;                                // continuation of whatever was open before
    }
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned pv = __shfl_up_sync(0xFFFFFFFFu, val, o);
      const bool ph = __shfl_up_sync(0xFFFFFFFFu, has, o);
      if (lane >= (unsigned)o && !has) val = pv, has = ph;
    }
    const unsigned open_k = has ? val : open_in;       // open run at the end of word k
    unsigned open_prev = __shfl_up_sync(0xFFFFFFFFu, open_k, 1);
    if (lane == 0) open_prev = open_in;
    // the 32 lanes now act as the 32 pixels of word k0 + i, i = 0..31: coalesced parent stores
    for (unsigned i = 0; i < 32 && k0 + i < mw; i++) {
      const unsigned wv = __shfl_sync(0xFFFFFFFFu, cur, i), st = __shfl_sync(0xFFFFFFFFu, starts, i);
      const unsigned op = __shfl_sync(0xFFFFFFFFu, open_prev, i);
      const unsigned x = 32 * (k0 + i) + lane;
      if (x < w) {
        unsigned pv = 0xFFFFFFFFu;
        if ((wv >> lane) & 1u) {
          const unsigned below = st & (0xFFFFFFFFu >> (31 - lane));
          pv = below ? base + 32 * (k0 + i) + (31 - __clz(below)) : op;
        }
        prow[x] = pv;
      }
    }
    open_in = __shfl_sync(0xFFFFFFFFu, open_k, 31);
  }
}

__device__ __forceinline__ unsigned uf_find(unsigned *parent, unsigned p) {
  unsigned q = parent[p];
  while (q != p) {
    const unsigned g = parent[q];
    if (g != q) parent[p] = g;                         // path halving (benign race: only ever moves towards the root)
    p = q, q = g;
  }
  return p;
}
__device__ __forceinline__ void uf_union(unsigned *parent, unsigned a, unsigned b) {
  while (true) {
    a = uf_find(parent, a), b = uf_find(parent, b);
    if (a == b) return;
    if (a < b) {
      const unsigned t = a;
      a = b, b = t;
    }
    const unsigned old = atomicMin(&parent[a], b);     // the larger root points to the smaller one
    if (old == a) return;
    a = old;
  }
}

// one union per vertical contact segment: the first pixel of every run of (M & M_above)
__global__ void __launch_bounds__(256)
k_blob_union(const unsigned *__restrict__ mask, unsigned w, unsigned h, unsigned mw, unsigned *__restrict__ parent,
             unsigned long long words_total) {
  const unsigned long long g = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= words_total) return;
  const unsigned k = (unsigned)(g % mw);
  const unsigned long long row = g / mw;
  const unsigned y = (unsigned)(row % h);
  if (y == 0) return;
  const unsigned c = mask[g] & mask[g - mw];
  if (!c) return;
  const unsigned cp = k ? (mask[g - 1] & mask[g - 1 - mw]) : 0u;
  unsigned u = c & ~((c << 1) | (cp >> 31));
  unsigned *par = parent + (row - y) * w;              // this frame's table (row - y = f * h)
  while (u) {
    const unsigned b = __ffs(u) - 1;
    u &= u - 1;
    const unsigned p = y * w + 32 * k + b;
    uf_union(par, p, p - w);
  }
}

struct BlobStats {   // per frame: 7 arrays of nblobs
  unsigned *area, *minx, *miny, *maxx, *maxy, *sx, *sy;
};

// gs_label per pixel + per-component statistics; a warp = one 32-pixel word
__global__ void __launch_bounds__(256)
k_blob_label(const unsigned *__restrict__ mask, const unsigned *__restrict__ seed, const unsigned *__restrict__ sprefix,
             const unsigned *__restrict__ rowoff, unsigned w, unsigned h, unsigned mw, unsigned *__restrict__ parent,
             uint16_t *__restrict__ labels, BlobStats st, unsigned nblobs, unsigned long long words_total) {
  const unsigned long long g = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (g >= words_total) return;
  const unsigned lane = threadIdx.x & 31;
  const unsigned k = (unsigned)(g % mw);
  const unsigned long long row = g / mw;
  const unsigned y = (unsigned)(row % h);
  const unsigned long long f = row / h;
  const unsigned x = 32 * k + lane;
  const unsigned mv = mask[g];
  unsigned label = 0;
  if (x < w && ((mv >> lane) & 1u)) {
    unsigned *par = parent + f * (unsigned long long)w * h;
    const unsigned r = uf_find(par, y * w + x);
    const unsigned ry = r / w, rx = r % w;             // the component's raster-first pixel: a seed
    const unsigned long long rw = (f * h + ry) * mw + (rx >> 5);
    label = rowoff[f * h + ry] + sprefix[rw] + __popc(seed[rw] & ((1u << (rx & 31)) - 1u)) + 1u;
  }
  if (x < w) labels[row * w + x] = (uint16_t)label;
  const unsigned grp = __match_any_sync(0xFFFFFFFFu, label);
  if (label != 0 && lane == (unsigned)(__ffs(grp) - 1) && label <= nblobs) {
    const unsigned cnt = __popc(grp);
    // sum of the set bit positions of grp
    const unsigned pos = __popc(grp & 0xAAAAAAAAu) + 2 * __popc(grp & 0xCCCCCCCCu) + 4 * __popc(grp & 0xF0F0F0F0u) +
                         8 * __popc(grp & 0xFF00FF00u) + 16 * __popc(grp & 0xFFFF0000u);
    const size_t i = (size_t)f * nblobs + (label - 1);
    atomicAdd(&st.area[i], cnt);
    atomicAdd(&st.sx[i], 32 * k * cnt + pos);
    atomicAdd(&st.sy[i], y * cnt);
    atomicMin(&st.minx[i], 32 * k + (unsigned)(__ffs(grp) - 1));
    atomicMax(&st.maxx[i], 32 * k + (31u - (unsigned)__clz(grp)));
    atomicMin(&st.miny[i], y);
    atomicMax(&st.maxy[i], y);
  }
}

// blobs[0..m) in label order; counts[f] = m
__global__ void __launch_bounds__(256)
k_blob_compact(BlobStats st, const unsigned *__restrict__ totals, unsigned nblobs, BlobRec *__restrict__ blobs,
               unsigned *__restrict__ counts) {
  __shared__ unsigned wcnt[8];
  __shared__ unsigned running;
  const unsigned f = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned nl = min(totals[f], nblobs);
  if (tid == 0) running = 0;
  __syncthreads();
  for (unsigned b0 = 0; b0 < nl; b0 += 256) {
    const unsigned i = b0 + tid;
    const size_t si = (size_t)f * nblobs + i;
    const unsigned area = i < nl ? st.area[si] : 0u;
    const unsigned bal = __ballot_sync(0xFFFFFFFFu, area != 0);
    if (lane == 0) wcnt[warp] = __popc(bal);
    __syncthreads();
    unsigned before = 0, total = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) {
      const unsigned c = wcnt[j];
      before += j < (int)warp ? c : 0u;
      total += c;
    }
    if (area) {
      const unsigned pos = running + before + __popc(bal & ((1u << lane) - 1u));
      BlobRec r;
      r.w[0] = i + 1;                                  // gs_label in the low 16 bits, padding zero
      r.w[1] = area;
      r.w[2] = st.minx[si], r.w[3] = st.miny[si];
      r.w[4] = st.maxx[si] - st.minx[si] + 1, r.w[5] = st.maxy[si] - st.miny[si] + 1;
      r.w[6] = st.sx[si] / area, r.w[7] = st.sy[si] / area;
      uint4 *o = reinterpret_cast<uint4 *>(blobs + (size_t)f * nblobs + pos);
      o[0] = make_uint4(r.w[0], r.w[1], r.w[2], r.w[3]);
      o[1] = make_uint4(r.w[4], r.w[5], r.w[6], r.w[7]);
    }
    __syncthreads();
    if (tid == 0) running += total;
    __syncthreads();
  }
  if (tid == 0) counts[f] = running;
}

// gs_blob_corners (reference :407-421): one CTA scans the blob's box; lexicographic (value, raster index) minima
__global__ void __launch_bounds__(256)
k_blob_corners(const uint8_t *__restrict__ img, unsigned w, unsigned h, const uint16_t *__restrict__ labels,
               const BlobRec *__restrict__ blob, unsigned *__restrict__ out /* 4 points */) {
  __shared__ unsigned long long best[4];
  const BlobRec b = *blob;
  const unsigned label = b.w[0] & 0xFFFFu, bx = b.w[2], by = b.w[3], bw = b.w[4], bh = b.w[5];
  if (threadIdx.x < 4) best[threadIdx.x] = ~0ull;
  __syncthreads();
  unsigned long long mine[4] = {~0ull, ~0ull, ~0ull, ~0ull};
  const unsigned long long cells = (unsigned long long)bw * bh;
  for (unsigned long long i = threadIdx.x; i < cells; i += blockDim.x) {
    const unsigned x = bx + (unsigned)(i % bw), y = by + (unsigned)(i / bw);
    if (x >= w || y >= h) continue;
    const size_t p = (size_t)y * w + x;
    if (img[p] < 128 || labels[p] != label) continue;
    const int sum = (int)x + (int)y, diff = (int)x - (int)y;
    const int v[4] = {sum, -diff, -sum, diff};          // tl: min sum, tr: max diff, br: max sum, bl: min diff
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const unsigned long long key = ((unsigned long long)(unsigned)(v[q] + 0x40000000) << 32) | (unsigned)p;
      mine[q] = key < mine[q] ? key : mine[q];
    }
  }
#pragma unroll
  for (int q = 0; q < 4; q++)
    if (mine[q] != ~0ull) atomicMin(&best[q], mine[q]);
  __syncthreads();
  if (threadIdx.x < 4) {
    const unsigned long long k = best[threadIdx.x];
    if (k == ~0ull) out[2 * threadIdx.x] = b.w[6], out[2 * threadIdx.x + 1] = b.w[7];   // the centroid
    else {
      const unsigned p = (unsigned)k;
      out[2 * threadIdx.x] = p % w, out[2 * threadIdx.x + 1] = p / w;
    }
  }
}

struct Quad {
  float x[4], y[4];
};
// gs_perspective_correct (reference :423-444): every fp32 operation in the reference's order, no contraction
__global__ void __launch_bounds__(256)
k_perspective(uint8_t *__restrict__ dst, unsigned dw, unsigned dh, const uint8_t *__restrict__ src, unsigned sw, unsigned sh,
              unsigned n, const unsigned *__restrict__ corners /* n x 8 (device) or null */, Quad q0) {
  const unsigned x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= dw) return;
  const float wm = __fsub_rn((float)dw, 1.0f), hm = __fsub_rn((float)dh, 1.0f);
  const float mx = __fsub_rn((float)sw, 1.0f), my = __fsub_rn((float)sh, 1.0f);
  const float u = __fdiv_rn((float)x, wm), v = __fdiv_rn((float)y, hm);
  const float omu = __fsub_rn(1.0f, u), omv = __fsub_rn(1.0f, v);
  for (unsigned f = blockIdx.z; f < n; f += gridDim.z) {
    Quad q = q0;
    if (corners) {
#pragma unroll
      for (int i = 0; i < 4; i++) q.x[i] = (float)corners[f * 8 + 2 * i], q.y[i] = (float)corners[f * 8 + 2 * i + 1];
    }
    const float top_x = __fadd_rn(__fmul_rn(q.x[0], omu), __fmul_rn(q.x[1], u));
    const float top_y = __fadd_rn(__fmul_rn(q.y[0], omu), __fmul_rn(q.y[1], u));
    const float bot_x = __fadd_rn(__fmul_rn(q.x[3], omu), __fmul_rn(q.x[2], u));
    const float bot_y = __fadd_rn(__fmul_rn(q.y[3], omu), __fmul_rn(q.y[2], u));
    float sx = __fadd_rn(__fmul_rn(top_x, omv), __fmul_rn(bot_x, v));
    float sy = __fadd_rn(__fmul_rn(top_y, omv), __fmul_rn(bot_y, v));
    sx = sx < mx ? sx : mx;                             // GS_MIN(src_x, w - 1): a NaN falls to w - 1
    sy = sy < my ? sy : my;
    sx = 0.0f > sx ? 0.0f : sx;                         // GS_MAX(0, .)
    sy = 0.0f > sy ? 0.0f : sy;
    const unsigned x0 = (unsigned)sx, y0 = (unsigned)sy;
    const unsigned x1 = min(x0 + 1, sw - 1), y1 = min(y0 + 1, sh - 1);
    const float dx = __fsub_rn(sx, (float)x0), dy = __fsub_rn(sy, (float)y0);
    const uint8_t *s = src + (size_t)f * sw * sh;
    const float c00 = (float)s[(size_t)y0 * sw + x0], c01 = (float)s[(size_t)y0 * sw + x1];
    const float c10 = (float)s[(size_t)y1 * sw + x0], c11 = (float)s[(size_t)y1 * sw + x1];
    const float omx = __fsub_rn(1.0f, dx), omy = __fsub_rn(1.0f, dy);
    float acc = __fmul_rn(__fmul_rn(c00, omx), omy);
    acc = __fadd_rn(acc, __fmul_rn(__fmul_rn(c01, dx), omy));
    acc = __fadd_rn(acc, __fmul_rn(__fmul_rn(c10, omx), dy));
    acc = __fadd_rn(acc, __fmul_rn(__fmul_rn(c11, dx), dy));
    dst[(size_t)f * dw * dh + (size_t)y * dw + x] = (uint8_t)(unsigned)acc;
  }
}

}  // namespace gsb

extern "C" {

int gs_b200_blobs_batch(const uint8_t *img, unsigned w, unsigned h, unsigned n, uint16_t *labels, struct gs_blob *blobs,
                        unsigned *counts, unsigned nblobs, gs_b200_stream s) {
  GSB_ASSERT(img && w > 0 && h > 0 && labels && blobs && counts && nblobs > 0);   // reference :335
  GSB_ASSERT(nblobs <= 65534u && (unsigned long long)w * h < 0xFFFFFFFFull);       // gs_label is 16 bits wide
  if (n == 0) return 0;
  cudaStream_t st = static_cast<cudaStream_t>(s);
  const unsigned mw = (w + 31) / 32;
  const unsigned long long rows_total = (unsigned long long)h * n, words_total = rows_total * mw;
  GSB_ASSERT(words_total * 32 < (1ull << 40));
  // workspace: mask | seed | sprefix (words_total each) | rowoff (rows_total) | totals (n) | stats (7 * nblobs * n)
  const size_t words_b = sizeof(unsigned) * words_total;
  const size_t ws_a = 3 * words_b + sizeof(unsigned) * (rows_total + n) + 7 * sizeof(unsigned) * (size_t)nblobs * n;
  unsigned *wa = static_cast<unsigned *>(gsb::workspace(st, gsb::WS_BLOB_A, ws_a));
  unsigned *parent = static_cast<unsigned *>(gsb::workspace(st, gsb::WS_BLOB_B, sizeof(unsigned) * (size_t)w * h * n));
  if (!wa || !parent) return gsb::workspace_error();
  unsigned *mask = wa, *seed = wa + words_total, *sprefix = seed + words_total, *rowoff = sprefix + words_total;
  unsigned *totals = rowoff + rows_total, *stats = totals + n;
  const size_t sn = (size_t)nblobs * n;
  gsb::BlobStats bs = {stats, stats + sn, stats + 2 * sn, stats + 3 * sn, stats + 4 * sn, stats + 5 * sn, stats + 6 * sn};
  GSB_CHECK(cudaMemsetAsync(bs.area, 0, sizeof(unsigned) * sn, st));
  GSB_CHECK(cudaMemsetAsync(bs.minx, 0xFF, 2 * sizeof(unsigned) * sn, st));          // minx, miny
  GSB_CHECK(cudaMemsetAsync(bs.maxx, 0, 4 * sizeof(unsigned) * sn, st));             // maxx, maxy, sx, sy
  const unsigned row_blocks = (unsigned)((rows_total + 7) / 8);
  GSB_LAUNCH(gsb::k_blob_mask, row_blocks, 256, 0, st, img, w, h, mw, mask, rows_total);
  GSB_LAUNCH(gsb::k_blob_seed, row_blocks, 256, 0, st, mask, h, mw, seed, sprefix, rowoff, rows_total);
  GSB_LAUNCH(gsb::k_row_scan, n, 1024, 0, st, rowoff, h, totals, 0xFFFFFFFFu);
  GSB_LAUNCH(gsb::k_blob_overflow, (n + 63) / 64, 64, 0, st, mask, seed, sprefix, rowoff, totals, h, mw, nblobs, n);
  GSB_LAUNCH(gsb::k_blob_runs, row_blocks, 256, 0, st, mask, w, h, mw, parent, rows_total);
  GSB_LAUNCH(gsb::k_blob_union, (unsigned)((words_total + 255) / 256), 256, 0, st, mask, w, h, mw, parent, words_total);
  GSB_LAUNCH(gsb::k_blob_label, (unsigned)((words_total + 7) / 8), 256, 0, st, mask, seed, sprefix, rowoff, w, h, mw, parent,
             labels, bs, nblobs, words_total);
  GSB_LAUNCH(gsb::k_blob_compact, n, 256, 0, st, bs, totals, nblobs, reinterpret_cast<gsb::BlobRec *>(blobs), counts);
  return 0;
}

int gs_b200_blob_corners(const uint8_t *img, unsigned w, unsigned h, const uint16_t *labels, const struct gs_blob *blob,
                         struct gs_point *corners, gs_b200_stream s) {
  GSB_ASSERT(img && w > 0 && h > 0 && blob && labels && corners);   // reference :409
  GSB_LAUNCH(gsb::k_blob_corners, 1, 256, 0, static_cast<cudaStream_t>(s), img, w, h, labels,
             reinterpret_cast<const gsb::BlobRec *>(blob), reinterpret_cast<unsigned *>(corners));
  return 0;
}

int gs_b200_perspective_correct_batch(uint8_t *dst, unsigned dw, unsigned dh, const uint8_t *src, unsigned sw, unsigned sh,
                                      unsigned n, const struct gs_point *corners, int per_frame, gs_b200_stream s) {
  GSB_ASSERT(dst && dw > 0 && dh > 0 && src && sw > 0 && sh > 0 && corners);   // reference :424
  if (n == 0) return 0;
  GSB_ASSERT(dh <= 65535u);
  gsb::Quad q = {};
  const unsigned *dev = nullptr;
  if (per_frame) dev = reinterpret_cast<const unsigned *>(corners);             // n x 4 points in DEVICE memory
  else
    for (int i = 0; i < 4; i++) q.x[i] = (float)corners[i].x, q.y[i] = (float)corners[i].y;   // 4 points in HOST memory
  dim3 grid((dw + 255) / 256, dh, n < 64u ? n : 64u);
  GSB_LAUNCH(gsb::k_perspective, grid, 256, 0, static_cast<cudaStream_t>(s), dst, dw, dh, src, sw, sh, n, dev, q);
  return 0;
}

}  // extern "C"
