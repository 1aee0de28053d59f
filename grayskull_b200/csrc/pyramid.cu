// pyramid.cu -- ORB features over an image pyramid for frame batches (include/grayskull_b200_pyramid.h), bit-exact with
// the reference CLI's multi-scale ORB (nanomagick.c:245-290).
//
// The call is the library's tested batch steps in sequence, with two small kernels of its own:
//   levels 1..L-1      gs_b200_downsample_batch into pyr, each level from the one before
//   levels 0..L-2      gs_b200_orb_extract_batch, one call per level: their quota nkps / L is the same for every frame
//   level L-1          its quota q_f = nkps - (frame f's earlier counts) differs per frame, so it runs as
//                        gs_b200_fast_batch with the largest cap min(4 * nkps, 5000) -> k_pyr_quota clamps each frame's
//                        candidate count to min(4 * q_f, 5000) -> orb_select (output cap nkps) -> k_pyr_quota
//                        clamps the count to q_f -> orb_describe.
//                      FAST emits survivors in raster order and stops at its cap, so its first c survivors are those of
//                      a run capped at c; select keeps the response-sorted, margin-filtered candidates in order, so its
//                      first q are those of a select capped at q.  Each clamp therefore gives gs_orb_extract's list for
//                      that frame's quota.
//   k_pyr_merge        per frame, the level blocks back to back at their per-frame offsets, coordinates times 1 << l
//                      (after describe ran on level l), and the total count.
// The per-level lists, the candidates and the counts live in the workspace arenas (gsb::workspace), so they are per
// stream, per thread for cudaStreamPerThread, and refuse to grow under graph capture.
#include "../../include/grayskull_b200_pyramid.h"
#include "common.cuh"

namespace gsb {

// the two steps of gs_b200_orb_extract_batch after FAST (fast_orb.cu)
int orb_select(const struct gs_keypoint *cand, const unsigned *cand_count, unsigned cap, unsigned w, unsigned h,
               struct gs_keypoint *kps, unsigned *counts, unsigned nkps, unsigned n, cudaStream_t st);
int orb_describe(const uint8_t *src, unsigned w, unsigned h, struct gs_keypoint *kps, const unsigned *counts,
                 unsigned nkps, unsigned n, cudaStream_t st);

constexpr unsigned PYR_MAX_LEVELS = 4;     // nanomagick.c:247
constexpr unsigned PYR_MIN_SIDE = 32;      // nanomagick.c:257: no level narrower or shorter than this
constexpr unsigned PYR_MAXC = 5000;        // gs_orb_extract's candidates[5000] (grayskull.h:655-656)

// count[f] = min(count[f], min(mult * q_f, cap)) with q_f = nkps - sum of frame f's counts on the `early` levels before
// the last (lcounts[l * n + f]); mult 4, cap 5000 clamps the FAST candidates, mult 1, cap ~0 the selected keypoints
__global__ void __launch_bounds__(256)
k_pyr_quota(unsigned *__restrict__ count, const unsigned *__restrict__ lcounts, unsigned early, unsigned n,
            unsigned nkps, unsigned mult, unsigned cap) {
  const unsigned f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n) return;
  unsigned used = 0;
  for (unsigned l = 0; l < early; l++) used += lcounts[(size_t)l * n + f];
  const unsigned long long lim = min((unsigned long long)(nkps - used) * mult, (unsigned long long)cap);
  count[f] = (unsigned)min((unsigned long long)count[f], lim);
}

// the per-level lists of one call: level l's records of frame f start at list[l] + f * stride[l]; count[l] is null for
// a skipped level
struct PyrLists {
  const uint4 *list[PYR_MAX_LEVELS];
  const unsigned *count[PYR_MAX_LEVELS];
  unsigned stride[PYR_MAX_LEVELS];
};

// thread (j, f): output slot j of frame f, taken from the level block that holds it; slots past the total are not
// written
__global__ void __launch_bounds__(256)
k_pyr_merge(PyrLists p, unsigned levels, uint4 *__restrict__ kps, unsigned *__restrict__ counts, unsigned nkps) {
  const unsigned f = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned c[PYR_MAX_LEVELS], total = 0;
#pragma unroll
  for (unsigned l = 0; l < PYR_MAX_LEVELS; l++) {
    c[l] = l < levels && p.count[l] ? p.count[l][f] : 0u;
    total += c[l];
  }
  if (j == 0) counts[f] = total;
  if (j >= total) return;
  unsigned k = j, l = 0;
#pragma unroll
  for (unsigned i = 0; i + 1 < PYR_MAX_LEVELS; i++)
    if (l == i && k >= c[i]) k -= c[i], l = i + 1;
  const uint4 *list = p.list[0];
  unsigned stride = p.stride[0];
#pragma unroll
  for (unsigned i = 1; i < PYR_MAX_LEVELS; i++)   // constant indices: the parameter block is not copied to the stack
    if (l == i) list = p.list[i], stride = p.stride[i];
  const uint4 *r = list + ((size_t)f * stride + k) * 3;
  uint4 a = r[0];
  a.x *= 1u << l, a.y *= 1u << l;   // nanomagick.c:282-285, in unsigned arithmetic
  uint4 *o = kps + ((size_t)f * nkps + j) * 3;
  o[0] = a, o[1] = r[1], o[2] = r[2];
}

#define PYR_DO(call)             \
  do {                           \
    int pyr_rc_ = (call);        \
    if (pyr_rc_) return pyr_rc_; \
  } while (0)

static unsigned pyr_levels(unsigned w, unsigned h, unsigned levels) {
  const unsigned want = levels < PYR_MAX_LEVELS ? levels : PYR_MAX_LEVELS;
  for (unsigned l = 1; l < want; l++) {
    w /= 2, h /= 2;
    if (w < PYR_MIN_SIDE || h < PYR_MIN_SIDE) return l;
  }
  return want;
}

}  // namespace gsb

extern "C" {

unsigned gs_b200_orb_pyramid_levels(unsigned w, unsigned h, unsigned levels) { return gsb::pyr_levels(w, h, levels); }

int gs_b200_orb_pyramid_batch(const uint8_t *src, unsigned w, unsigned h, unsigned n, unsigned levels, uint8_t *pyr,
                              uint8_t *scoremap, struct gs_keypoint *kps, unsigned *counts, unsigned nkps,
                              unsigned threshold, gs_b200_stream s) {
  if (n == 0) return 0;
  GSB_ASSERT(counts);
  cudaStream_t st = static_cast<cudaStream_t>(s);
  if (nkps == 0 || levels == 0) {   // every level's quota is 0: nothing runs, the reference returns 0
    GSB_CHECK(cudaMemsetAsync(counts, 0, sizeof(unsigned) * n, st));
    return 0;
  }
  GSB_ASSERT(src && w > 0 && h > 0 && kps && scoremap);   // gs_orb_extract's assert (reference :653)
  const unsigned L = gsb::pyr_levels(w, h, levels);
  if (L > 1) GSB_ASSERT(pyr);
  unsigned lw[gsb::PYR_MAX_LEVELS], lh[gsb::PYR_MAX_LEVELS];
  const uint8_t *img[gsb::PYR_MAX_LEVELS];
  uint8_t *score[gsb::PYR_MAX_LEVELS];
  lw[0] = w, lh[0] = h, img[0] = src, score[0] = scoremap;
  for (unsigned l = 1; l < L; l++) {
    lw[l] = lw[l - 1] / 2, lh[l] = lh[l - 1] / 2;
    const size_t below = (size_t)lw[l - 1] * lh[l - 1] * n;
    img[l] = l == 1 ? pyr : img[l - 1] + below;
    score[l] = score[l - 1] + below;
  }
  const unsigned q0 = nkps / L, early = q0 ? L - 1 : 0;   // levels before the last run only with a quota
  const unsigned cap = nkps * 4ull < gsb::PYR_MAXC ? nkps * 4 : gsb::PYR_MAXC;
  // k_pyr_merge puts the frame in grid y: the call runs per frame group, each group on its frames of every level
  // (level l of frame f is at img[l] + f * lw[l] * lh[l]) with its own workspace lists
  return gsb::for_frame_groups(n, [&](unsigned f0, unsigned m) {
    const uint8_t *gimg[gsb::PYR_MAX_LEVELS];
    uint8_t *gscore[gsb::PYR_MAX_LEVELS];
    for (unsigned l = 0; l < L; l++) {
      const size_t o = (size_t)f0 * lw[l] * lh[l];
      gimg[l] = img[l] + o, gscore[l] = score[l] + o;
    }
    const size_t early_recs = (size_t)m * q0 * (L - 1), last_recs = (size_t)m * nkps;
    struct gs_keypoint *lists = static_cast<struct gs_keypoint *>(
        gsb::workspace(st, gsb::WS_PYR_LISTS, sizeof(struct gs_keypoint) * (early_recs + last_recs)));
    struct gs_keypoint *cand =
        static_cast<struct gs_keypoint *>(gsb::workspace(st, gsb::WS_PYR_CAND, sizeof(struct gs_keypoint) * (size_t)m * cap));
    unsigned *lcounts = static_cast<unsigned *>(gsb::workspace(st, gsb::WS_PYR_COUNTS, sizeof(unsigned) * (size_t)m * (L + 1)));
    if (!lists || !cand || !lcounts) return gsb::workspace_error();
    unsigned *ccount = lcounts + (size_t)m * L;

    for (unsigned l = 1; l < L; l++)
      PYR_DO(gs_b200_downsample_batch(const_cast<uint8_t *>(gimg[l]), gimg[l - 1], lw[l - 1], lh[l - 1], m, s));

    gsb::PyrLists p = {};
    for (unsigned l = 0; l < early; l++) {
      struct gs_keypoint *list = lists + (size_t)m * q0 * l;
      PYR_DO(gs_b200_orb_extract_batch(gimg[l], lw[l], lh[l], m, gscore[l], list, lcounts + (size_t)m * l, q0, threshold, s));
      p.list[l] = reinterpret_cast<const uint4 *>(list), p.count[l] = lcounts + (size_t)m * l, p.stride[l] = q0;
    }

    const unsigned t = L - 1;
    struct gs_keypoint *last = lists + early_recs;
    unsigned *lcount = lcounts + (size_t)m * t;
    const dim3 fgrid((m + 255) / 256);
    PYR_DO(gs_b200_fast_batch(gimg[t], lw[t], lh[t], m, gscore[t], cand, ccount, cap, threshold, s));
    GSB_LAUNCH(gsb::k_pyr_quota, fgrid, 256, 0, st, ccount, lcounts, early, m, nkps, 4u, gsb::PYR_MAXC);
    PYR_DO(gsb::orb_select(cand, ccount, cap, lw[t], lh[t], last, lcount, nkps, m, st));
    GSB_LAUNCH(gsb::k_pyr_quota, fgrid, 256, 0, st, lcount, lcounts, early, m, nkps, 1u, 0xFFFFFFFFu);
    PYR_DO(gsb::orb_describe(gimg[t], lw[t], lh[t], last, lcount, nkps, m, st));
    p.list[t] = reinterpret_cast<const uint4 *>(last), p.count[t] = lcount, p.stride[t] = nkps;

    GSB_LAUNCH(gsb::k_pyr_merge, dim3((nkps + 255) / 256, m), 256, 0, st, p, L,
               reinterpret_cast<uint4 *>(kps) + (size_t)f0 * nkps * 3, counts + f0, nkps);
    return 0;
  });
}

}  // extern "C"
