// resample.cuh -- gs_resize's per-axis coordinate mapping and its four-tap sum (reference grayskull.h:174-184), shared
// by resample.cu and the region kernels of roi.cu.
#pragma once
#include <cuda_runtime.h>

namespace gsb {

#ifdef __CUDACC__
// Every rounding step of grayskull.h:174-184 is reproduced with the _rn intrinsics (never
// contracted into FMAs): sx = ((x + 0.5f) * sw) / dw - 0.5f, clamp, truncate, and the sum of
// four products ((c * wx) * wy) added left to right.
// One departure: for about half the sizes above 2^24, (float)sdim - 1.0f rounds to sdim or past it (by up to 128 near
// 2^32), and the reference's first tap then lies past the row or column.  Here that tap is the last pixel.  frac is 0
// there already (every float of that size is an integer), so the result is the last pixel's value.
__device__ __forceinline__ void resize_axis(unsigned i, unsigned sdim, unsigned ddim, unsigned &i0,
                                            unsigned &i1, float &frac) {
  float s = __fsub_rn(__fdiv_rn(__fmul_rn(__fadd_rn((float)i, 0.5f), (float)sdim), (float)ddim), 0.5f);
  const float hi = __fsub_rn((float)sdim, 1.0f);
  s = s < hi ? s : hi;
  s = 0.0f > s ? 0.0f : s;
  i0 = __float2uint_rz(s);
  i1 = i0 + 1 < sdim - 1 ? i0 + 1 : sdim - 1;
  frac = __fsub_rn(s, (float)i0);
  i0 = i0 < sdim - 1 ? i0 : sdim - 1;
}

__device__ __forceinline__ float bilerp(float c00, float c01, float c10, float c11, float omx, float dx, float omy,
                                        float dy) {
  float p = __fmul_rn(__fmul_rn(c00, omx), omy);                  // reference :181-184, left to right
  p = __fadd_rn(p, __fmul_rn(__fmul_rn(c01, dx), omy));
  p = __fadd_rn(p, __fmul_rn(__fmul_rn(c10, omx), dy));
  p = __fadd_rn(p, __fmul_rn(__fmul_rn(c11, dx), dy));
  return p;
}
#endif  // __CUDACC__

}  // namespace gsb
