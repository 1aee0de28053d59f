// histogram.cu -- gs_histogram / gs_otsu_threshold / gs_threshold (reference grayskull.h:199-228;
// SURVEY.md 8f "next" item N2: the step between sobel and morphology in the reference's pipelines).
//
// gs_histogram is 1 B/pixel of HBM traffic, i.e. ~12 pixels per SM-clock at the H100's 3.35 TB/s, but every
// pixel needs one shared-memory atomic, and those issue at 16 lanes/clk/SM when conflict-free -- the bound
// this kernel is built around:
//   * counters are laid out [bin][lane] (u32), so lane L only ever touches bank L: no bank conflict and no
//     same-address serialisation for ANY image content (a constant frame is as fast as noise);
//   * two warps share one 32 KB array (atomics keep that correct), 7 arrays = 224 KB = one 14-warp CTA per SM;
//   * per pixel: one byte extract, one multiply-add for the address, one RED.shared -- 3 instructions;
//   * CTAs own contiguous runs of (frame, chunk) units and fold their arrays into the global table only when
//     the frame changes (256 warp reductions + global atomics, ~1 % of a 256 Kpx chunk).
// gs_otsu_threshold: one warp per frame stages the 256 counts and evaluates the reference's fp32 loop with
// explicitly rounded operations in the reference's order (bit-exact thresholds).
// gs_threshold: in place, 16 px per thread, per-byte unsigned compare.
#include "common.cuh"

namespace gsb {

constexpr int HG_WARPS = 14, HG_THREADS = HG_WARPS * 32, HG_ARRAYS = HG_WARPS / 2;
constexpr int HG_ARRAY_WORDS = 256 * 32;
constexpr int HG_SMEM = HG_ARRAYS * HG_ARRAY_WORDS * 4;   // 229376 B

__device__ __forceinline__ void red_shared_inc(uint32_t saddr) {
  asm volatile("red.shared.add.u32 [%0], 1;" ::"r"(saddr) : "memory");
}
__device__ __forceinline__ void count_word(uint32_t w, uint32_t lanebase) {
  // PRMT byte extract + one multiply-add (left to itself nvcc emits shift, mask and add: 3 instead of 2)
  red_shared_inc(lanebase + prmt(w, 0, 0x4440) * 128u);
  red_shared_inc(lanebase + prmt(w, 0, 0x4441) * 128u);
  red_shared_inc(lanebase + prmt(w, 0, 0x4442) * 128u);
  red_shared_inc(lanebase + prmt(w, 0, 0x4443) * 128u);
}

template <bool VEC>
__global__ void __launch_bounds__(HG_THREADS, 1)
k_histogram(unsigned *__restrict__ hist, const uint8_t *__restrict__ src, size_t frame_px, unsigned units,
            unsigned chunks_per_frame, size_t chunk_px) {
  extern __shared__ __align__(16) uint32_t s_h[];
  const unsigned tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (unsigned i = tid; i < HG_ARRAYS * HG_ARRAY_WORDS / 4; i += HG_THREADS)
    reinterpret_cast<uint4 *>(s_h)[i] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  const uint32_t lanebase = (uint32_t)__cvta_generic_to_shared(s_h + (warp >> 1) * HG_ARRAY_WORDS + lane);
  // contiguous run of units for this CTA
  const unsigned u0 = (unsigned)(((unsigned long long)units * blockIdx.x) / gridDim.x);
  const unsigned u1 = (unsigned)(((unsigned long long)units * (blockIdx.x + 1)) / gridDim.x);
  unsigned cur = 0xFFFFFFFFu;
  for (unsigned u = u0; u <= u1; u++) {
    const unsigned f = u < u1 ? u / chunks_per_frame : 0xFFFFFFFFu;
    if (f != cur) {
      if (cur != 0xFFFFFFFFu) {                       // fold this CTA's counts of frame `cur` into the table
        __syncthreads();
        for (unsigned bin = warp; bin < 256; bin += HG_WARPS) {
          unsigned v = 0;
#pragma unroll
          for (int a = 0; a < HG_ARRAYS; a++) {
            uint32_t *p = s_h + a * HG_ARRAY_WORDS + bin * 32 + lane;
            v += *p;
            *p = 0;
          }
          v = __reduce_add_sync(0xFFFFFFFFu, v);
          if (lane == 0 && v) atomicAdd(hist + (size_t)cur * 256 + bin, v);
        }
        __syncthreads();
      }
      cur = f;
    }
    if (u == u1) break;
    const unsigned c = u % chunks_per_frame;
    const size_t begin = (size_t)c * chunk_px;
    const size_t end = begin + chunk_px < frame_px ? begin + chunk_px : frame_px;
    const uint8_t *p = src + (size_t)f * frame_px;
    if (VEC) {
      const uint4 *q = reinterpret_cast<const uint4 *>(p);
      const size_t e = end / 16;
      size_t i = begin / 16 + tid;
      for (; i + 3 * HG_THREADS < e; i += 4 * HG_THREADS) {
        const uint4 a = __ldg(q + i), b = __ldg(q + i + HG_THREADS), cc = __ldg(q + i + 2 * HG_THREADS),
                    d = __ldg(q + i + 3 * HG_THREADS);
        count_word(a.x, lanebase), count_word(a.y, lanebase), count_word(a.z, lanebase), count_word(a.w, lanebase);
        count_word(b.x, lanebase), count_word(b.y, lanebase), count_word(b.z, lanebase), count_word(b.w, lanebase);
        count_word(cc.x, lanebase), count_word(cc.y, lanebase), count_word(cc.z, lanebase), count_word(cc.w, lanebase);
        count_word(d.x, lanebase), count_word(d.y, lanebase), count_word(d.z, lanebase), count_word(d.w, lanebase);
      }
      for (; i < e; i += HG_THREADS) {
        const uint4 a = __ldg(q + i);
        count_word(a.x, lanebase), count_word(a.y, lanebase), count_word(a.z, lanebase), count_word(a.w, lanebase);
      }
    } else {
      for (size_t i = begin + tid; i < end; i += HG_THREADS) red_shared_inc(lanebase + (uint32_t)__ldg(p + i) * 128u);
    }
  }
}

// One warp per frame, the reference's fp32 loop (grayskull.h:205-224) split where its dependences allow:
//   serial  : sum, and the running wb[t] / sumB[t] (fp32 accumulations in bin order -- order is the result),
//             ~2 dependent adds per bin;
//   parallel: mB, mF, varBetween for 8 thresholds per lane (the two IEEE divisions are the expensive part);
//   argmax  : `var > varMax` from varMax = -1 keeps the FIRST maximum over the valid thresholds (wb > 0 and
//             wf > 0: the reference `continue`s while wb == 0 and `break`s at the first wf == 0, after which
//             wf stays 0), so a (var, t) max-reduction with ties to the smaller t gives the same threshold.
__global__ void __launch_bounds__(128)
k_otsu(uint8_t *__restrict__ thresh, const unsigned *__restrict__ hist, unsigned npix, unsigned n) {
  __shared__ unsigned s_hist[4][256];
  __shared__ unsigned s_wb[4][256];
  __shared__ float s_sumb[4][256];
  const unsigned warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned f = blockIdx.x * 4 + warp;
  if (f >= n) return;
  unsigned *h = s_hist[warp];
  for (unsigned i = lane; i < 256; i += 32) h[i] = hist[(size_t)f * 256 + i];
  __syncwarp();
  float sum = 0.0f;
  if (lane == 0) {
    float sum_b = 0.0f;
    unsigned wb = 0;
#pragma unroll 8
    for (unsigned t = 0; t < 256; t++) {
      const unsigned c = h[t];
      const float term = __fmul_rn((float)t, __uint2float_rn(c));
      sum = __fadd_rn(sum, term);
      wb += c;
      // the reference adds the term only once wb != 0 (and before the wf test); while wb == 0 the term is +0
      sum_b = __fadd_rn(sum_b, term);
      s_wb[warp][t] = wb;
      s_sumb[warp][t] = sum_b;
    }
  }
  sum = __shfl_sync(0xFFFFFFFFu, sum, 0);
  __syncwarp();
  float best_v = -1.0f;
  unsigned best_t = 0;
#pragma unroll
  for (unsigned k = 0; k < 8; k++) {
    const unsigned t = k * 32 + lane;
    const unsigned wb = s_wb[warp][t], wf = npix - wb;
    const float sum_b = s_sumb[warp][t];
    const float fwb = __uint2float_rn(wb), fwf = __uint2float_rn(wf);
    const float m_b = __fdiv_rn(sum_b, fwb);
    const float m_f = __fdiv_rn(__fsub_rn(sum, sum_b), fwf);
    const float diff = __fsub_rn(m_b, m_f);
    const float var = __fmul_rn(__fmul_rn(__fmul_rn(fwb, fwf), diff), diff);
    if (wb != 0 && wf != 0 && var > best_v) best_v = var, best_t = t;   // t ascends per lane: first max kept
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xFFFFFFFFu, best_v, o);
    const unsigned ot = __shfl_xor_sync(0xFFFFFFFFu, best_t, o);
    if (ov > best_v || (ov == best_v && ot < best_t)) best_v = ov, best_t = ot;
  }
  if (lane == 0) thresh[f] = (uint8_t)best_t;
}

// img > t ? 255 : 0 per byte.  `t` is either the scalar or (thresh[f] + offset) & 255.
template <bool VEC>
__global__ void __launch_bounds__(256)
k_threshold(uint8_t *__restrict__ img, size_t frame_px, const uint8_t *__restrict__ thresh, unsigned scalar,
            int offset) {
  const unsigned f = blockIdx.y;
  // unsigned add: (int)thresh[f] + offset would overflow for offset > INT_MAX - 255; the low byte is the same
  const unsigned t = thresh ? ((unsigned)thresh[f] + (unsigned)offset) & 0xFFu : scalar & 0xFFu;
  uint8_t *p = img + (size_t)f * frame_px;
  if (VEC) {
    const uint32_t t4 = t * 0x01010101u;
    const size_t e = frame_px / 16;
    for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < e; i += (size_t)gridDim.x * 256) {
      uint4 v = *(reinterpret_cast<const uint4 *>(p) + i);
      v.x = __vcmpgtu4(v.x, t4), v.y = __vcmpgtu4(v.y, t4), v.z = __vcmpgtu4(v.z, t4), v.w = __vcmpgtu4(v.w, t4);
      *(reinterpret_cast<uint4 *>(p) + i) = v;
    }
  } else {
    for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < frame_px; i += (size_t)gridDim.x * 256)
      p[i] = p[i] > t ? 255 : 0;
  }
}

static int threshold_launch(uint8_t *img, unsigned w, unsigned h, unsigned n, const uint8_t *thresh, unsigned scalar,
                            int offset, cudaStream_t st) {
  const size_t px = (size_t)w * h;
  const bool vec = px % 16 == 0 && reinterpret_cast<uintptr_t>(img) % 16 == 0;
  for (unsigned f0 = 0; f0 < n; f0 += 65535u) {      // grid.y limit
    const unsigned nf = n - f0 < 65535u ? n - f0 : 65535u;
    const size_t items = vec ? px / 16 : px;
    unsigned gx = (unsigned)((items + 256 * 4 - 1) / (256 * 4));
    gx = gx < 1 ? 1 : (gx > 4096 ? 4096 : gx);
    dim3 grid(gx, nf);
    uint8_t *p = img + (size_t)f0 * px;
    const uint8_t *tp = thresh ? thresh + f0 : nullptr;
    GSB_LAUNCH(vec ? k_threshold<true> : k_threshold<false>, grid, 256, 0, st, p, px, tp, scalar, offset);
  }
  return 0;
}

}  // namespace gsb

extern "C" {

int gs_b200_histogram_batch(unsigned *hist, const uint8_t *src, unsigned w, unsigned h, unsigned n, gs_b200_stream s) {
  GSB_ASSERT(src && hist && w > 0 && h > 0);   // reference :200
  if (n == 0) return 0;
  cudaStream_t st = static_cast<cudaStream_t>(s);
  GSB_CHECK(cudaMemsetAsync(hist, 0, sizeof(unsigned) * 256 * (size_t)n, st));
  const size_t px = (size_t)w * h;
  // chunks of ~256 Kpx, a multiple of one unrolled CTA sweep (4 x 448 x 16 B)
  const size_t sweep = (size_t)4 * gsb::HG_THREADS * 16;
  size_t chunk = ((size_t)262144 + sweep - 1) / sweep * sweep;
  unsigned cpf = (unsigned)((px + chunk - 1) / chunk);
  GSB_ASSERT((unsigned long long)cpf * n < 0xFFFFFFFFull);
  const unsigned units = cpf * n;
  const unsigned sms = (unsigned)gsb::sm_count();
  const unsigned grid = units < sms ? units : sms;
  const bool vec = px % 16 == 0 && reinterpret_cast<uintptr_t>(src) % 16 == 0;
  GSB_LAUNCH(vec ? gsb::k_histogram<true> : gsb::k_histogram<false>, grid, gsb::HG_THREADS, gsb::HG_SMEM, st, hist, src, px,
             units, cpf, chunk);
  return 0;
}

int gs_b200_otsu_threshold_batch(uint8_t *thresh, unsigned *hist, const uint8_t *src, unsigned w, unsigned h,
                                 unsigned n, gs_b200_stream s) {
  GSB_ASSERT(src && thresh && w > 0 && h > 0);   // reference :207
  if (n == 0) return 0;
  cudaStream_t st = static_cast<cudaStream_t>(s);
  if (!hist) {
    hist = static_cast<unsigned *>(gsb::workspace(st, gsb::WS_HIST, sizeof(unsigned) * 256 * (size_t)n));
    if (!hist) return gsb::workspace_error();
  }
  int rc = gs_b200_histogram_batch(hist, src, w, h, n, s);
  if (rc) return rc;
  GSB_LAUNCH(gsb::k_otsu, (n + 3) / 4, 128, 0, st, thresh, hist, w * h, n);
  return 0;
}

int gs_b200_threshold_batch(uint8_t *img, unsigned w, unsigned h, unsigned n, unsigned thresh, gs_b200_stream s) {
  GSB_ASSERT(img && w > 0 && h > 0);   // reference :227
  if (n == 0) return 0;
  return gsb::threshold_launch(img, w, h, n, nullptr, thresh, 0, static_cast<cudaStream_t>(s));
}

int gs_b200_threshold_each_batch(uint8_t *img, unsigned w, unsigned h, unsigned n, const uint8_t *thresh, int offset,
                                 gs_b200_stream s) {
  GSB_ASSERT(img && thresh && w > 0 && h > 0);
  if (n == 0) return 0;
  return gsb::threshold_launch(img, w, h, n, thresh, 0, offset, static_cast<cudaStream_t>(s));
}
}
