// common.cuh -- shared plumbing of libgrayskull_b200.so: error recording, the kernel launch helper,
// per-stream device workspace, TMA tensor maps and the mbarrier / bulk-tensor-copy PTX wrappers.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <utility>

#include "../../include/grayskull_b200.h"

namespace gsb {

// ---- host side ------------------------------------------------------------------------------
int record_error(cudaError_t e, const char *file, int line);
bool force_generic();  // GS_B200_FORCE_GENERIC=1: never take the TMA-tiled kernels (tests)
int sm_count();        // SMs of the current device (grid sizing)

#define GSB_CHECK(expr)                                                        \
  do {                                                                         \
    cudaError_t gsb_e_ = (expr);                                               \
    if (gsb_e_ != cudaSuccess) return gsb::record_error(gsb_e_, __FILE__, __LINE__); \
  } while (0)

// the two out-of-line halves of launch(): raise kernel k's dynamic shared-memory limit on the current device to at
// least `smem` bytes (once per size it grows to), and count one launch and check it
int opt_in_smem(const void *k, size_t smem, const char *file, int line);
int launched(const char *file, int line);

#ifdef __CUDACC__
// Every kernel launch of the library: opt-in, launch, count, check.  The arguments convert to the kernel's own
// parameter types exactly as in a direct <<<>>> call.  Returns 0 or the CUDA error (recorded at file:line).
template <class... P, class... A>
int launch(const char *file, int line, void (*k)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t s,
           A &&...a) {
  if (smem)
    if (int rc = opt_in_smem(reinterpret_cast<const void *>(k), smem, file, line)) return rc;
  k<<<grid, block, smem, s>>>(std::forward<A>(a)...);
  return launched(file, line);
}
#define GSB_LAUNCH(...)                                         \
  do {                                                          \
    int gsb_rc_ = gsb::launch(__FILE__, __LINE__, __VA_ARGS__); \
    if (gsb_rc_) return gsb_rc_;                                \
  } while (0)
#endif  // __CUDACC__

// Grid y and z stop at 65535.  A call whose kernels take the frame from blockIdx.y or .z without a loop over frames
// runs a larger batch as consecutive groups of at most GRID_FRAMES frames: for_frame_groups calls fn(f0, count) for
// each group in order, and fn launches that group's kernels with every per-frame base advanced by f0 frames.  The
// groups queue on the caller's stream one after the other, so per-call workspace sized for a group is reused by the
// next one in stream order.  Returns the first non-zero result of fn (the later groups do not run), else 0.
constexpr unsigned GRID_FRAMES = 65535u;
template <class F>
int for_frame_groups(unsigned n, F &&fn) {
  for (unsigned long long f0 = 0; f0 < n; f0 += GRID_FRAMES) {
    const unsigned long long left = n - f0;
    if (int rc = fn(static_cast<unsigned>(f0), static_cast<unsigned>(left < GRID_FRAMES ? left : GRID_FRAMES))) return rc;
  }
  return 0;
}

// Row tiles meet the same limit within one frame.  A kernel that takes its row tile from blockIdx.y without a loop over
// row tiles takes a tile-row offset t0 and works on row tile blockIdx.y + t0; for_row_groups calls fn(t0, count) for
// each group of at most GRID_FRAMES tile rows, and fn launches count tile rows at offset t0.  Every launch still sees
// the whole frame (its h, its tensor map), so halos and edge clipping are those of one launch.  A frame of at most
// GRID_FRAMES row tiles is one launch at t0 = 0.
template <class F>
int for_row_groups(unsigned tiles_y, F &&fn) {
  return for_frame_groups(tiles_y, static_cast<F &&>(fn));
}

// the reference's gs_assert (grayskull.h:94-98): message + abort
#define GSB_ASSERT(cond)                                \
  do {                                                  \
    if (!(cond)) {                                      \
      fprintf(stderr, "Assertion failed: %s\n", #cond); \
      abort();                                          \
    }                                                   \
  } while (0)

// Grow-only device scratch, one arena per (device, stream, slot); cudaStreamPerThread has one per (host thread, device,
// slot), freed at thread exit.  Not freed until process exit otherwise: the hot path must not cudaMalloc per call.
// Returns nullptr when it cannot allocate, or when it would have to grow while `s` is capturing a graph;
// workspace_error() is then the calling thread's error code (its text is in gs_b200_last_error()).
void *workspace(cudaStream_t s, int slot, size_t bytes);
int workspace_error();
// whether `s` is capturing a CUDA graph (true also when the query itself is not legal in the current capture)
bool capturing(cudaStream_t s);
// Blocking host -> device copy that no caller's stream can overtake: a copy on a private non-blocking stream, then a
// sync of that stream.  (A pageable cudaMemcpy on the legacy stream may return before its DMA lands, and kernels on
// non-blocking streams are not ordered after it.)  For rare uploads only: LBP plan misses, once-per-device tables.
int upload(void *dst, const void *src, size_t bytes, const char *file, int line);

enum { WS_INTEGRAL = 0, WS_FAST_A, WS_FAST_B, WS_ORB_A, WS_ORB_B, WS_LBP_A, WS_LBP_B, WS_LBP_C,
       WS_STAGE_A, WS_STAGE_B, WS_STAGE_C, WS_STAGE_D, WS_HIST, WS_STAGE_FUSED, WS_BLOB_A, WS_BLOB_B, WS_BLOB_C, WS_MORPH,
       // csrc/pyramid.cu: per-level keypoint lists, the last level's FAST candidates, per-level counts.  Distinct from
       // WS_FAST_* / WS_ORB_*, which the calls it makes in between use.
       WS_PYR_LISTS, WS_PYR_CAND, WS_PYR_COUNTS,
       // csrc/box.cu: the tile counter of k_blur_sobel_tma
       WS_BLUR_SOBEL_TILES, WS_SLOTS };

// 3-D tensor map over n dense u8 frames of w x h, viewed as 32-bit words {w/4, h, n}
// (TMA boxes are limited to 256 elements per dimension: u32 elements give 1 KiB wide boxes).
// Requires w % 16 == 0 and a 16-byte aligned base.  Out-of-range box elements read as 0.
bool make_tmap_u8frames(CUtensorMap *m, const void *base, unsigned w, unsigned h, unsigned n,
                        unsigned box_words, unsigned box_rows);
// same for n dense u32 tables of w x h (integral images): dims {w, h, n}
bool make_tmap_u32frames(CUtensorMap *m, const void *base, unsigned w, unsigned h, unsigned n,
                         unsigned box_w, unsigned box_h);
inline bool tma_ok(const void *p, unsigned w) {
  return !force_generic() && (w % 16u) == 0 && (reinterpret_cast<uintptr_t>(p) % 16u) == 0;
}

// ---- device side ----------------------------------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
// make the barrier init visible to the async (TMA) proxy before the first bulk copy targets it
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// order the generic-proxy shared-memory accesses before it (the whole CTA's, after a barrier) before later async-proxy
// ones: a TMA load may then refill a buffer that the CTA has just read
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, unsigned parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// 3-D tiled bulk tensor load global -> shared, completion signalled on `bar` (SASS: UTMALDG)
__device__ __forceinline__ void tma_load_3d(void *smem_dst, const CUtensorMap *map, int c0, int c1,
                                            int c2, uint64_t *bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar))
      : "memory");
}

__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
  return __byte_perm(a, b, sel);
}
// raw prmt.b32: selector nibble bit 3 replicates the SIGN of the selected byte over the result byte
// (__byte_perm masks the selector with 0x7777, so that mode needs inline PTX)
__device__ __forceinline__ uint32_t prmt_raw(uint32_t a, uint32_t b, uint32_t sel) {
  uint32_t d;
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(sel));
  return d;
}
// streaming 64-bit store (outputs are written once and not re-read by the same kernel)
__device__ __forceinline__ void st_cs_u2(void *p, uint2 v) {
  asm volatile("st.global.cs.v2.u32 [%0], {%1, %2};" ::"l"(p), "r"(v.x), "r"(v.y) : "memory");
}
#endif  // __CUDACC__

}  // namespace gsb
