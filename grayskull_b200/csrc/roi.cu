// roi.cu -- crop-and-resize of regions of interest over frame batches (include/grayskull_b200_roi.h), bit-exact with
// the reference's gs_crop followed by gs_resize_nn or gs_resize.
//
// Two kernels per call geometry:
//   k_roi_copy         unscaled regions (dw == roi.w, dh == roi.h) that lie inside the frame without wrapping and whose
//                      sides keep both modes the identity (ROI_IDENTITY_*): 16-byte aligned dst chunks, each assembled
//                      from the two aligned 16-byte source blocks it overlaps by funnel shifts, so any source offset
//                      and any base alignment take the vector path.
//   k_roi_gather<M>    everything else: per-CTA column and row tables (nearest: the source index; bilinear: the
//                      indices and fractions of gs_resize), then byte gathers of 4 adjacent pixels per thread.
// The choice is a function of the slot's region and the call's dw, dh, sw, sh and mode (roi_copy): made on the host
// for gs_b200_crop_resize_batch, per slot on the device for gs_b200_rois_resize_batch, where both kernels run over
// the list and each takes the slots that are its own.
#include "../../include/grayskull_b200_roi.h"
#include "common.cuh"
#include "resample.cuh"

namespace gsb {

// Largest side at which the mode maps x to x when dw == roi.w: nearest computes x * w / w in 32 bits, exact while
// (w - 1) * w < 2^32; bilinear's ((x + 0.5f) * w) / w - 0.5f is x for every x < w up to w = 2896 and first misses
// at w = 2897, x = 2896 (2895.99976; checked exhaustively).  Larger unscaled regions take the gather kernel.
constexpr unsigned ROI_IDENTITY_NEAREST = 65536u, ROI_IDENTITY_BILINEAR = 2896u;

// gs_crop's assert on the region (reference grayskull.h:155-156), in its 32-bit wrapping arithmetic
__host__ __device__ __forceinline__ bool roi_valid(const gs_rect &r, unsigned sw, unsigned sh) {
  return r.w && r.h && r.x + r.w <= sw && r.y + r.h <= sh;
}

// whether the slot is a plain copy of the region (k_roi_copy) rather than a gather (k_roi_gather)
__host__ __device__ __forceinline__ bool roi_copy(const gs_rect &r, unsigned sw, unsigned sh, unsigned dw, unsigned dh,
                                                  int mode) {
  const unsigned lim = mode == GS_B200_NEAREST ? ROI_IDENTITY_NEAREST : ROI_IDENTITY_BILINEAR;
  return roi_valid(r, sw, sh) && r.w == dw && r.h == dh && dw <= lim && dh <= lim &&
         (unsigned long long)r.x + r.w <= sw && (unsigned long long)r.y + r.h <= sh;
}

// Where slot s = f * max_rects + k takes its region: rects[s] of a device list, or `roi` for every frame when rects is
// null.  counts (nullable) bounds each frame's list.
struct Slots {
  const gs_rect *rects;
  gs_rect roi;
  const unsigned *counts;
  unsigned max_rects;
  unsigned long long nslots;
};

// the slot's region, or false when the slot is past its frame's count (then nothing of it is read or written)
__device__ __forceinline__ bool slot_region(const Slots &q, unsigned long long s, gs_rect &r) {
  if (q.counts && s % q.max_rects >= q.counts[s / q.max_rects]) return false;
  r = q.rects ? q.rects[s] : q.roi;
  return true;
}

// ---- k_roi_copy ------------------------------------------------------------------------------------------------------
// Thread (chunk, row): the 16-byte aligned dst chunk `chunk` of the row's span [d, d + dw).  Its source bytes start at
// S = row source + (A - d) and overlap at most two aligned 16-byte blocks; a block is loaded only when it holds a byte
// the chunk needs (so no load leaves the 16-byte granule of a byte the region covers).  Interior chunks leave as one
// 16-byte streaming store, the row's head and tail chunks byte by byte.
constexpr int CP_ROWS = 32;   // rows per CTA: 8 warps x 4

__device__ __forceinline__ uint4 ld_nc_v4(const void *p) {
  uint4 v;
  asm volatile("ld.global.nc.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}
__device__ __forceinline__ void st_cs_v4(void *p, uint4 v) {
  asm volatile("st.global.cs.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}

__global__ void __launch_bounds__(256)
k_roi_copy(uint8_t *__restrict__ dst, unsigned dw, unsigned dh, const uint8_t *__restrict__ src, unsigned sw,
           unsigned sh, Slots q, int mode) {
  const unsigned chunk = blockIdx.x * 32 + threadIdx.x;
  for (unsigned long long s = blockIdx.z; s < q.nslots; s += gridDim.z) {
    gs_rect r;
    if (!slot_region(q, s, r) || !roi_copy(r, sw, sh, dw, dh, mode)) continue;
    const uint8_t *fs = src + (size_t)(s / q.max_rects) * sw * sh + (size_t)r.y * sw + r.x;
    uint8_t *ds = dst + (size_t)s * dw * dh;
    for (unsigned yb = blockIdx.y * CP_ROWS; yb < dh; yb += gridDim.y * CP_ROWS) {
#pragma unroll
      for (int i = 0; i < CP_ROWS / 8; i++) {
        const unsigned y = yb + threadIdx.y + 8 * i;
        if (y >= dh) break;
        const uintptr_t d = reinterpret_cast<uintptr_t>(ds + (size_t)y * dw);
        const uintptr_t A = (d & ~(uintptr_t)15) + 16 * (uintptr_t)chunk;
        if (A >= d + dw) continue;
        const unsigned lo = A < d ? (unsigned)(d - A) : 0u;
        const unsigned hi = A + 16 <= d + dw ? 16u : (unsigned)(d + dw - A);
        const uintptr_t S = reinterpret_cast<uintptr_t>(fs + (size_t)y * sw) + (A - d);   // wraps back for the head
        const uintptr_t B = S & ~(uintptr_t)15;
        uint4 v0 = make_uint4(0, 0, 0, 0), v1 = make_uint4(0, 0, 0, 0);
        if (S + lo < B + 16) v0 = ld_nc_v4(reinterpret_cast<const void *>(B));
        if (S + hi > B + 16) v1 = ld_nc_v4(reinterpret_cast<const void *>(B + 16));
        const unsigned o = (unsigned)(S & 15), q4 = o >> 2, sh8 = (o & 3) * 8;
        const uint32_t w[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
        uint32_t v[5];
#pragma unroll
        for (int j = 0; j < 5; j++)
          v[j] = q4 == 0 ? w[j] : q4 == 1 ? w[j + 1] : q4 == 2 ? w[j + 2] : w[j + 3];
        uint32_t out[4];
#pragma unroll
        for (int j = 0; j < 4; j++) out[j] = __funnelshift_r(v[j], v[j + 1], sh8);
        uint8_t *a = reinterpret_cast<uint8_t *>(A);
        if (lo == 0 && hi == 16) {
          st_cs_v4(a, make_uint4(out[0], out[1], out[2], out[3]));
        } else {
#pragma unroll
          for (int j = 0; j < 16; j++)
            if (j >= (int)lo && j < (int)hi) a[j] = (uint8_t)(out[j >> 2] >> (8 * (j & 3)));
        }
      }
    }
  }
}

// ---- k_roi_gather ----------------------------------------------------------------------------------------------------
// A CTA makes a tw x GT_ROWS tile of one slot (tw = 64 or 128 dst columns).  The tile's column and row tables are built
// once per tile: absolute source column / row of each tap (ROI_OUT when gs_get would read outside the frame or the
// region is invalid, so an invalid region gives zeros) and, in bilinear mode, gs_resize's fractions.  Then each thread
// makes 4 adjacent pixels of a row and stores them as one 32-bit word when the address allows.
constexpr int GT_ROWS = 64;
constexpr unsigned ROI_OUT = 0xFFFFFFFFu;   // never a column or row of a frame: those are < sw, sh <= 2^32 - 1

template <int MODE>
__global__ void __launch_bounds__(256)
k_roi_gather(uint8_t *__restrict__ dst, unsigned dw, unsigned dh, const uint8_t *__restrict__ src, unsigned sw,
             unsigned sh, Slots q, unsigned tw) {
  __shared__ unsigned s_x0[128], s_x1[128], s_y0[GT_ROWS], s_y1[GT_ROWS];
  __shared__ float s_fx[128], s_fy[GT_ROWS];
  const unsigned tid = threadIdx.x, groups = tw / 4, tx0 = blockIdx.x * tw;
  const unsigned x = tx0 + (tid % groups) * 4;
  for (unsigned long long s = blockIdx.z; s < q.nslots; s += gridDim.z) {
    gs_rect r;
    if (!slot_region(q, s, r) || roi_copy(r, sw, sh, dw, dh, MODE)) continue;
    const bool ok = roi_valid(r, sw, sh);
    const uint8_t *fs = src + (size_t)(s / q.max_rects) * sw * sh;
    uint8_t *ds = dst + (size_t)s * dw * dh;
    for (unsigned ty0 = blockIdx.y * GT_ROWS; ty0 < dh; ty0 += gridDim.y * GT_ROWS) {
      __syncthreads();   // the previous tile's tables are consumed
      // threads 0..127 build the column table, 128..191 the row table (same formulas per axis)
      const bool col = tid < 128;
      const unsigned i = col ? tx0 + tid : ty0 + (tid - 128);
      if (col || tid < 128 + GT_ROWS) {
        const unsigned ddim = col ? dw : dh, rdim = col ? r.w : r.h, org = col ? r.x : r.y, fdim = col ? sw : sh;
        unsigned a = ROI_OUT, b = ROI_OUT;
        float fr = 0.0f;
        if (ok && i < ddim) {
          unsigned i0, i1;
          if (MODE == GS_B200_NEAREST) {
            i0 = i1 = i * rdim / ddim;   // gs_resize_nn, 32-bit (may wrap)
          } else {
            resize_axis(i, rdim, ddim, i0, i1, fr);
          }
          a = org + i0, b = org + i1;   // gs_crop's roi.x + x, 32-bit (may wrap)
          a = a < fdim ? a : ROI_OUT, b = b < fdim ? b : ROI_OUT;
        }
        if (col) {
          if (tid < tw) s_x0[tid] = a, s_x1[tid] = b, s_fx[tid] = fr;
        } else {
          s_y0[tid - 128] = a, s_y1[tid - 128] = b, s_fy[tid - 128] = fr;
        }
      }
      __syncthreads();
      if (x >= dw) continue;
      const unsigned c = x - tx0;
      for (unsigned row = tid / groups; row < (unsigned)GT_ROWS && ty0 + row < dh; row += 256 / groups) {
        const unsigned y0 = s_y0[row], y1 = s_y1[row];
        const uint8_t *r0 = fs + (size_t)y0 * sw, *r1 = fs + (size_t)y1 * sw;
        uint32_t out = 0;
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const unsigned x0 = s_x0[c + j];
          uint32_t p;
          if (MODE == GS_B200_NEAREST) {
            p = x0 != ROI_OUT && y0 != ROI_OUT ? __ldg(r0 + x0) : 0u;
          } else {
            const unsigned x1 = s_x1[c + j];
            const float dx = s_fx[c + j], dy = s_fy[row];
            const float c00 = x0 != ROI_OUT && y0 != ROI_OUT ? (float)__ldg(r0 + x0) : 0.0f;
            const float c01 = x1 != ROI_OUT && y0 != ROI_OUT ? (float)__ldg(r0 + x1) : 0.0f;
            const float c10 = x0 != ROI_OUT && y1 != ROI_OUT ? (float)__ldg(r1 + x0) : 0.0f;
            const float c11 = x1 != ROI_OUT && y1 != ROI_OUT ? (float)__ldg(r1 + x1) : 0.0f;
            p = __float2uint_rz(bilerp(c00, c01, c10, c11, __fsub_rn(1.0f, dx), dx, __fsub_rn(1.0f, dy), dy)) & 0xFFu;
          }
          out |= p << (8 * j);
        }
        uint8_t *o = ds + (size_t)(ty0 + row) * dw + x;
        if (x + 3 < dw && reinterpret_cast<uintptr_t>(o) % 4 == 0) {
          *reinterpret_cast<uint32_t *>(o) = out;
        } else {
          for (unsigned j = 0; j < 4 && x + j < dw; j++) o[j] = (uint8_t)(out >> (8 * j));
        }
      }
    }
  }
}

static unsigned cap16(unsigned long long v) { return v < 65535ull ? (unsigned)v : 65535u; }

static int launch_copy(uint8_t *dst, unsigned dw, unsigned dh, const uint8_t *src, unsigned sw, unsigned sh,
                       const Slots &q, int mode, cudaStream_t st) {
  const dim3 grid((dw / 16 + 2 + 31) / 32, cap16((dh + CP_ROWS - 1) / CP_ROWS), cap16(q.nslots));
  GSB_LAUNCH(k_roi_copy, grid, dim3(32, 8), 0, st, dst, dw, dh, src, sw, sh, q, mode);
  return 0;
}

static int launch_gather(uint8_t *dst, unsigned dw, unsigned dh, const uint8_t *src, unsigned sw, unsigned sh,
                         const Slots &q, int mode, cudaStream_t st) {
  const unsigned tw = dw <= 64 ? 64u : 128u;
  const dim3 grid((dw + tw - 1) / tw, cap16((dh + GT_ROWS - 1) / GT_ROWS), cap16(q.nslots));
  if (mode == GS_B200_NEAREST)
    GSB_LAUNCH(k_roi_gather<GS_B200_NEAREST>, grid, 256, 0, st, dst, dw, dh, src, sw, sh, q, tw);
  else
    GSB_LAUNCH(k_roi_gather<GS_B200_BILINEAR>, grid, 256, 0, st, dst, dw, dh, src, sw, sh, q, tw);
  return 0;
}

// the reference's asserts, on the images the two calls would see: gs_crop(crop, frame, roi), gs_resize(out, crop)
static void crop_assert(struct gs_image dst, struct gs_image src, struct gs_rect roi) {
  GSB_ASSERT(gs_valid(dst) && gs_valid(src) && roi.x + roi.w <= src.w && roi.y + roi.h <= src.h && dst.w == roi.w &&
             dst.h == roi.h);
}
static void resize_assert(struct gs_image dst, struct gs_image src) { GSB_ASSERT(gs_valid(dst) && gs_valid(src)); }

static bool known_mode(int mode) { return mode == GS_B200_NEAREST || mode == GS_B200_BILINEAR; }

}  // namespace gsb

extern "C" {

int gs_b200_crop_resize_batch(uint8_t *dst, unsigned dw, unsigned dh, const uint8_t *src, unsigned sw, unsigned sh,
                              unsigned n, struct gs_rect roi, int mode, gs_b200_stream s) {
  if (!gsb::known_mode(mode)) return gsb::record_error(cudaErrorInvalidValue, __FILE__, __LINE__);
  const struct gs_image crop = {roi.w, roi.h, dst};   // the intermediate is never stored: dst stands for its data
  gsb::crop_assert(crop, gs_image{sw, sh, const_cast<uint8_t *>(src)}, roi);
  if (mode == GS_B200_BILINEAR) gsb::resize_assert(gs_image{dw, dh, dst}, crop);
  if (n == 0 || dw == 0 || dh == 0) return 0;   // gs_resize_nn of an empty dst writes nothing
  const gsb::Slots q = {nullptr, roi, nullptr, 1u, n};
  cudaStream_t st = static_cast<cudaStream_t>(s);
  return gsb::roi_copy(roi, sw, sh, dw, dh, mode) ? gsb::launch_copy(dst, dw, dh, src, sw, sh, q, mode, st)
                                                  : gsb::launch_gather(dst, dw, dh, src, sw, sh, q, mode, st);
}

int gs_b200_rois_resize_batch(uint8_t *dst, unsigned dw, unsigned dh, const uint8_t *src, unsigned sw, unsigned sh,
                              unsigned n, const struct gs_rect *rects, const unsigned *counts, unsigned max_rects,
                              int mode, gs_b200_stream s) {
  if (!gsb::known_mode(mode)) return gsb::record_error(cudaErrorInvalidValue, __FILE__, __LINE__);
  if (mode == GS_B200_BILINEAR) GSB_ASSERT(dw > 0 && dh > 0);   // gs_resize's gs_valid(dst)
  if (n == 0 || max_rects == 0 || dw == 0 || dh == 0) return 0;
  GSB_ASSERT(dst && src && rects && sw > 0 && sh > 0);
  const gsb::Slots q = {rects, gs_rect{0, 0, 0, 0}, counts, max_rects, (unsigned long long)n * max_rects};
  cudaStream_t st = static_cast<cudaStream_t>(s);
  // a slot is a copy only when dw x dh is its region's size; past the identity limit no slot can be
  const unsigned lim = mode == GS_B200_NEAREST ? gsb::ROI_IDENTITY_NEAREST : gsb::ROI_IDENTITY_BILINEAR;
  if (dw <= lim && dh <= lim)
    if (int rc = gsb::launch_copy(dst, dw, dh, src, sw, sh, q, mode, st)) return rc;
  return gsb::launch_gather(dst, dw, dh, src, sw, sh, q, mode, st);
}

}  // extern "C"
