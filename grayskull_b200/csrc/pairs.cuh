// pairs.cuh -- 16-bit lane-pair helpers of the 3x3 stencils (gs_sobel), shared by stencil3.cu and the fused
// blur -> sobel kernel in box.cu.  See stencil3.cu's header comment for the number representation.
#pragma once
#include "common.cuh"

namespace gsb {

struct Pairs {  // pair words P_k = (x+k, x+k+2) for k = -1 .. 6, 16-bit lanes
  uint32_t m1, p0, p1, p2, p3, p4, p5, p6;
};

// wl,w0,w1,wr = image bytes [x-4,x), [x,x+4), [x+4,x+8), [x+8,x+12).  Eight ALU operations: the four aligned pairs are
// masked or permuted against zero, and each misaligned pair is one PRMT against an aligned pair that holds its second
// byte in byte 0 and a zero in byte 1 (or, for P_6, its first byte in byte 2 and a zero in byte 1)
__device__ __forceinline__ Pairs split_pairs(uint32_t wl, uint32_t w0, uint32_t w1, uint32_t wr) {
  Pairs p;
  p.p0 = w0 & 0x00FF00FFu;            // (x,   x+2)
  p.p1 = prmt(w0, 0, 0x4341);         // (x+1, x+3)
  p.p4 = w1 & 0x00FF00FFu;            // (x+4, x+6)
  p.p5 = prmt(w1, 0, 0x4341);         // (x+5, x+7)
  p.m1 = prmt(wl, p.p1, 0x5453);      // (x-1, x+1): byte 3 of wl, byte 0 of P_1
  p.p2 = prmt(w0, p.p4, 0x5452);      // (x+2, x+4): byte 2 of w0, byte 0 of P_4
  p.p3 = prmt(w0, p.p5, 0x5453);      // (x+3, x+5): byte 3 of w0, byte 0 of P_5
  p.p6 = prmt(p.p4, wr, 0x1412);      // (x+6, x+8): byte 2 of P_4, byte 0 of wr
  return p;
}

__device__ __forceinline__ __half2 as_h2(uint32_t v) { return *reinterpret_cast<__half2 *>(&v); }
__device__ __forceinline__ uint32_t as_u32(__half2 v) { return *reinterpret_cast<uint32_t *>(&v); }

struct SobelRow {   // per-row horizontal partials for the four output pair words k = 0,1,4,5
  uint32_t ua[4];   // u_{k-1} = P_{k-1} + P_k      (left pair sums)
  uint32_t ub[4];   // u_k     = P_k + P_{k+1}      (right pair sums)
  __half2 d[4];     // d_k     = P_{k+1} - P_{k-1}  (signed)
};

__device__ __forceinline__ SobelRow sobel_row(const Pairs &p) {
  SobelRow r;
  uint32_t um1 = p.m1 + p.p0, u0 = p.p0 + p.p1, u1 = p.p1 + p.p2;
  uint32_t u3 = p.p3 + p.p4, u4 = p.p4 + p.p5, u5 = p.p5 + p.p6;
  r.ua[0] = um1, r.ub[0] = u0;  // k = 0: pixels (x, x+2)
  r.ua[1] = u0, r.ub[1] = u1;   // k = 1: pixels (x+1, x+3)
  r.ua[2] = u3, r.ub[2] = u4;   // k = 4: pixels (x+4, x+6)
  r.ua[3] = u4, r.ub[3] = u5;   // k = 5: pixels (x+5, x+7)
  r.d[0] = __hsub2(as_h2(p.p1), as_h2(p.m1));
  r.d[1] = __hsub2(as_h2(p.p2), as_h2(p.p0));
  r.d[2] = __hsub2(as_h2(p.p5), as_h2(p.p3));
  r.d[3] = __hsub2(as_h2(p.p6), as_h2(p.p4));
  return r;
}

// out row y from rows y-1 (a), y (b: only d used), y+1 (c).  Returns 8 output bytes.
__device__ __forceinline__ uint2 sobel_out(const SobelRow &a, const SobelRow &b, const SobelRow &c) {
  uint32_t m[4];
  const __half2 cap = as_h2(0x00FF00FFu);  // 255 in the same units
#pragma unroll
  for (int k = 0; k < 4; k++) {
    // A = u_k(y+1) - u_{k-1}(y-1) + d_k(y);  B = u_k(y-1) - u_{k-1}(y+1) + d_k(y)
    __half2 A = __hadd2(__hsub2(as_h2(c.ub[k]), as_h2(a.ua[k])), b.d[k]);
    __half2 B = __hadd2(__hsub2(as_h2(a.ub[k]), as_h2(c.ua[k])), b.d[k]);
    __half2 mx = __hmax2(__habs2(A), __habs2(B));
    m[k] = as_u32(__hmin2(mx, cap));
  }
  uint2 o;
  o.x = prmt(m[0], m[1], 0x6240);
  o.y = prmt(m[2], m[3], 0x6240);
  return o;
}

}  // namespace gsb
