// lbp.cu -- gs_lbp_window / gs_lbp_detect (reference grayskull.h:769-835).
//
// A boosted cascade of 3x3 multi-block LBP features evaluated on an integral image, scanned over
// a fp32 scale ladder.  Not HBM-bound (about 1.1 B of compulsory traffic per window, but >= 6
// weak classifiers x 16 integral-image gathers): throughput is decided by gather rate and
// divergence.  Round-1 structure:
//   host    : the scale ladder (repeated fp32 multiply, reference :819), per-scale window size and
//             the per-scale truncated feature geometry (int)(int8 * scale) (:799-804) are computed
//             on the host with the reference's exact fp32 operations and cached on the device,
//             together with the cascade tables (keyed by content hash);
//   k_lbp_scan2  : a CTA owns 4096 consecutive windows of ONE scale (128 "slots" of 32 x-adjacent
//             windows).  The cascade tables and that scale's feature geometry (precomputed 32-bit
//             row / column offsets of the 4x4 corner lattice: 16 loads per weak instead of the
//             reference's 36, one IADD per address) live in shared memory.  Windows run the cascade
//             in stage groups; after each group the survivors are RE-PACKED into a dense list in
//             shared memory (warp ballot + one atomic per warp), so later stages run with full
//             warps instead of a few live lanes (v1 measured 7.8 of 32 lanes active).  Stage sums
//             are accumulated with sequential fp32 adds exactly as :808.  Hits are recorded as one
//             bit per window, which keeps the reference's order for free.  It takes the scans
//             k_lbp_scan3 cannot: step != 2, iw % 8 != 0, a table base that is not 16-byte aligned,
//             force_generic, or a scale whose tile does not fit;
//   k_lbp_scan3  : step-2 scans of 8-px-aligned, 16-byte-aligned tables whose features stay inside
//             their window: the same cascade walk on a 2-D window tile whose integral-image boxes (even- and
//             odd-column planes made by k_deinterleave2, so that step-2 windows gather from adjacent words)
//             are staged into shared memory by two TMA bulk-tensor copies (zero fill = the x == 0 / y == 0
//             corner rule); each warp re-packs its own survivors (no CTA barriers) and finishes its last few
//             in a flat (window, weak) mode;
//   k_lbp_scan   : round-1 kernel (lane per window, ballot early exit), kept for cascades whose
//             tables do not fit shared memory or whose features leave their window;
//   k_lbp_count / k_row_scan : hits per 256-window block and their per-frame exclusive scan;
//   k_lbp_emit   : rects written in the reference's (scale, y, x) order, truncated at max_rects
//             (the reference stops scanning there, :819-823).
#include <list>
#include <memory>
#include <mutex>
#include <string.h>
#include <vector>

#include "common.cuh"
#include "scan.cuh"

namespace gsb {

struct ScaleInfo {
  int win_w, win_h, nx, ny;
  unsigned chunks;             // 32-window slots per scan row
  unsigned feat_off;           // first entry of this scale's geometry in feat / geo / tgeo (shared by equal scales)
  unsigned long long slot0;    // first slot of this scale (a multiple of LBP_SLOTS_PER_CTA)
};
// Longest ladder gs_b200_lbp_detect_batch scans; a longer one is an error (cudaErrorInvalidValue), never a shorter
// list.  65536 scales hold any scale_factor >= 1.0001 over a 700x range of scales; scale_factor = 1 + 2^-23 needs
// millions.  A scale costs 32 B of tables, 512 B of hit masks per frame and one CTA of the scan.
constexpr int LBP_MAX_SCALES = 65536;
struct FeatGeo {               // corner lattice of one feature at one scale, as element offsets
  int row[4];                  // (fy - 1 + j*fh) * iw
  int col[4];                  // fx - 1 + i*fw
};
constexpr int LBP_SLOTS_PER_CTA = 128;                      // 32 windows each
constexpr int LBP_WIN_PER_CTA = LBP_SLOTS_PER_CTA * 32;
constexpr int LBP_THREADS = 256;
constexpr int LBP_MAX_GROUPS = 8;
struct Weak {
  float left, right;
  uint16_t fidx, sub_off, nsub, pad;
};
struct Stage {
  float thr;
  uint16_t start, n;
};

struct TileGeo {               // the same lattice inside the shared-memory tile (two parity planes): BYTE offsets
  int row[4];                  // (fy + j*fh) * plane_pitch_bytes
  int col[4];                  // parity(fx + i*fw + 7) * plane_bytes + ((fx + i*fw + 7) / 2) * 4
};
struct TilePlan {              // host side, per scale: window tile of k_lbp_scan3
  int twx, twy;                // windows per tile (twx a multiple of 32)
  int bw, ph;                  // box staged by TMA from EACH column-parity plane: bw x ph u32
  int tiles_x, tiles_y;
  int threads;                 // LBP3_THREADS or LBP3_BIG_THREADS
  size_t smem;
};
struct DevCascade {            // pointers into one device blob
  const ScaleInfo *scales;
  const short4 *feat;          // [nscales][nfeatures] = (fx, fy, fw, fh) after scaling/clamping
  const Weak *weaks;
  const int *subsets;
  const Stage *stages;
  const FeatGeo *geo;          // [nscales][nfeatures]
  const TileGeo *tgeo;         // [nscales][nfeatures], only when every scale has a TilePlan
  int group_end[LBP_MAX_GROUPS];   // stage groups: survivors are re-packed after each group
  int ngroups, nweaks, nsubsets;
  int nscales, nfeatures, nstages;
  unsigned long long total_slots, total_windows;
  int step;
  bool safe_geometry;          // every feature stays inside its window at every scale
};

// the scale that owns `slot`: the last one with slot0 <= slot (slot0 grows strictly, every scale has slots)
__device__ __forceinline__ int scale_of(const DevCascade &dc, unsigned long long slot) {
  int lo = 0, hi = dc.nscales - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (dc.scales[mid].slot0 <= slot) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

template <bool GUARD>
__device__ __forceinline__ uint32_t corner(const uint32_t *__restrict__ ii, unsigned iw, unsigned ih, int x, int y) {
  if (x < 0 || y < 0) return 0u;   // gs_integral_sum's x == 0 / y == 0 guards (reference :758-760)
  if (GUARD && ((unsigned)x >= iw || (unsigned)y >= ih)) return 0u;
  return __ldg(ii + (size_t)y * iw + (unsigned)x);
}

// gs_lbp_code (reference :769-783) from the 4x4 corner lattice
template <bool GUARD>
__device__ __forceinline__ int lbp_code(const uint32_t *__restrict__ ii, unsigned iw, unsigned ih, int x0, int y0,
                                        int fw, int fh) {
  uint32_t g[4][4];
#pragma unroll
  for (int j = 0; j < 4; j++)
#pragma unroll
    for (int i = 0; i < 4; i++) g[j][i] = corner<GUARD>(ii, iw, ih, x0 - 1 + i * fw, y0 - 1 + j * fh);
  uint32_t c[3][3];
#pragma unroll
  for (int j = 0; j < 3; j++)
#pragma unroll
    for (int i = 0; i < 3; i++) c[j][i] = g[j + 1][i + 1] + g[j][i] - g[j][i + 1] - g[j + 1][i];
  const uint32_t m = c[1][1];
  return ((c[0][0] >= m) << 7) | ((c[0][1] >= m) << 6) | ((c[0][2] >= m) << 5) | ((c[1][2] >= m) << 4) |
         ((c[2][2] >= m) << 3) | ((c[2][1] >= m) << 2) | ((c[2][0] >= m) << 1) | ((c[1][0] >= m) << 0);
}

// the cascade for one window per lane (reference gs_lbp_window :794-812); warp-collective
template <bool GUARD>
__device__ __forceinline__ bool cascade_eval(const uint32_t *__restrict__ ii, unsigned iw, unsigned ih, int x, int y,
                                             const short4 *__restrict__ feat, const Weak *__restrict__ weaks,
                                             const int *__restrict__ subsets, const Stage *__restrict__ stages,
                                             int nstages, bool alive) {
  for (int si = 0; si < nstages; si++) {
    if (!__any_sync(0xFFFFFFFFu, alive)) break;
    const Stage st = stages[si];
    if (alive) {
      float sum = 0.0f;
      for (int i = 0; i < st.n; i++) {
        const Weak wk = weaks[st.start + i];
        const short4 f = feat[wk.fidx];
        const int code = lbp_code<GUARD>(ii, iw, ih, x + f.x, y + f.y, f.z, f.w);
        const int idx = code >> 5;
        const bool match = idx < (int)wk.nsub && ((((unsigned)__ldg(subsets + wk.sub_off + idx)) >> (code & 31)) & 1u);
        sum = __fadd_rn(sum, match ? wk.left : wk.right);
      }
      if (sum < st.thr) alive = false;
    }
  }
  return alive;
}

template <bool GUARD>
__global__ void __launch_bounds__(256)
k_lbp_scan(const uint32_t *__restrict__ ii_all, unsigned iw, unsigned ih, DevCascade dc, unsigned *__restrict__ masks,
           unsigned *__restrict__ blockcount) {
  __shared__ unsigned wcnt[8];
  const unsigned f = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned long long slot = (unsigned long long)blockIdx.x * 8 + warp;
  const uint32_t *ii = ii_all + (size_t)f * iw * ih;
  unsigned mask = 0;
  if (slot < dc.total_slots) {
    const ScaleInfo sc = dc.scales[scale_of(dc, slot)];
    const unsigned long long rel = slot - sc.slot0;
    const unsigned yi = (unsigned)(rel / sc.chunks), xi = (unsigned)(rel % sc.chunks) * 32 + lane;
    const bool valid = xi < (unsigned)sc.nx && yi < (unsigned)sc.ny;   // padding slots are empty
    const bool hit = cascade_eval<GUARD>(ii, iw, ih, (int)xi * dc.step, (int)yi * dc.step, dc.feat + sc.feat_off,
                                         dc.weaks, dc.subsets, dc.stages, dc.nstages, valid);
    mask = __ballot_sync(0xFFFFFFFFu, hit);
    if (lane == 0) masks[(size_t)f * dc.total_slots + slot] = mask;
  }
  if (lane == 0) wcnt[warp] = __popc(mask);
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned t = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) t += wcnt[i];
    blockcount[(size_t)f * gridDim.x + blockIdx.x] = t;
  }
}

// the 8-bit LBP code from the eight neighbour cells (clockwise from top-left, reference :776-782) and the centre
__device__ __forceinline__ int lbp_code_of(uint32_t n7, uint32_t n6, uint32_t n5, uint32_t n4, uint32_t n3, uint32_t n2,
                                           uint32_t n1, uint32_t n0, uint32_t m) {
  return ((n7 >= m) << 7) | ((n6 >= m) << 6) | ((n5 >= m) << 5) | ((n4 >= m) << 4) | ((n3 >= m) << 3) | ((n2 >= m) << 2) |
         ((n1 >= m) << 1) | ((n0 >= m) << 0);
}

// one weak classifier for one window (reference gs_lbp_code + gs_lbp_match, :769-788)
template <bool EDGE>
__device__ __forceinline__ bool weak_match(const uint32_t *__restrict__ ii, int base, bool x0, bool y0, const FeatGeo &g,
                                           const Weak &wk, const int *__restrict__ subsets) {
  uint32_t v[4][4];
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const int rb = base + g.row[j];
#pragma unroll
    for (int i = 0; i < 4; i++) {
      int idx = rb + g.col[i];
      if (EDGE) {   // corner(-1, .) = corner(., -1) = 0: gs_integral_sum's x == 0 / y == 0 guards (:758-760)
        const bool off = (i == 0 && x0 && g.col[0] < 0) || (j == 0 && y0 && g.row[0] < 0);
        idx = off ? 0 : idx;
        const uint32_t t = __ldg(ii + (unsigned)idx);
        v[j][i] = off ? 0u : t;
      } else {
        v[j][i] = __ldg(ii + (unsigned)idx);
      }
    }
  }
  uint32_t c[3][3];
#pragma unroll
  for (int j = 0; j < 3; j++)
#pragma unroll
    for (int i = 0; i < 3; i++) c[j][i] = v[j + 1][i + 1] + v[j][i] - v[j][i + 1] - v[j + 1][i];
  const uint32_t m = c[1][1];
  const int code = lbp_code_of(c[0][0], c[0][1], c[0][2], c[1][2], c[2][2], c[2][1], c[2][0], c[1][0], m);
  const int idx = code >> 5;
  return idx < (int)wk.nsub && (((unsigned)subsets[wk.sub_off + idx] >> (code & 31)) & 1u);
}

__global__ void __launch_bounds__(LBP_THREADS)
k_lbp_scan2(const uint32_t *__restrict__ ii_all, unsigned iw, unsigned ih, DevCascade dc, unsigned *__restrict__ masks) {
  extern __shared__ __align__(16) unsigned char lsm[];
  FeatGeo *s_geo = reinterpret_cast<FeatGeo *>(lsm);
  Weak *s_weak = reinterpret_cast<Weak *>(s_geo + dc.nfeatures);
  Stage *s_stage = reinterpret_cast<Stage *>(s_weak + dc.nweaks);
  int *s_sub = reinterpret_cast<int *>(s_stage + dc.nstages);
  uint16_t *list_a = reinterpret_cast<uint16_t *>(s_sub + dc.nsubsets);
  uint16_t *list_b = list_a + LBP_WIN_PER_CTA;
  __shared__ unsigned hit[LBP_SLOTS_PER_CTA];
  __shared__ int slot_y[LBP_SLOTS_PER_CTA], slot_x[LBP_SLOTS_PER_CTA];   // window origin of lane 0, -1 = empty slot
  __shared__ int s_scale;
  __shared__ unsigned cnt[2];

  const unsigned f = blockIdx.y, tid = threadIdx.x, lane = tid & 31;
  const unsigned long long slot_first = (unsigned long long)blockIdx.x * LBP_SLOTS_PER_CTA;
  const uint32_t *ii = ii_all + (size_t)f * iw * ih;
  if (tid == 0) {
    s_scale = scale_of(dc, slot_first);
    cnt[0] = cnt[1] = 0;
  }
  __syncthreads();
  const ScaleInfo sc = dc.scales[s_scale];
  {  // tables -> shared memory (word copies)
    const uint32_t *g0 = reinterpret_cast<const uint32_t *>(dc.geo + sc.feat_off);
    uint32_t *d0 = reinterpret_cast<uint32_t *>(s_geo);
    for (int i = tid; i < dc.nfeatures * 8; i += LBP_THREADS) d0[i] = g0[i];
    const uint32_t *g1 = reinterpret_cast<const uint32_t *>(dc.weaks);
    uint32_t *d1 = reinterpret_cast<uint32_t *>(s_weak);
    for (int i = tid; i < dc.nweaks * 4; i += LBP_THREADS) d1[i] = g1[i];
    const uint32_t *g2 = reinterpret_cast<const uint32_t *>(dc.stages);
    uint32_t *d2 = reinterpret_cast<uint32_t *>(s_stage);
    for (int i = tid; i < dc.nstages * 2; i += LBP_THREADS) d2[i] = g2[i];
    for (int i = tid; i < dc.nsubsets; i += LBP_THREADS) s_sub[i] = dc.subsets[i];
  }
  for (unsigned sl = tid; sl < LBP_SLOTS_PER_CTA; sl += LBP_THREADS) {
    const unsigned long long rel = slot_first + sl - sc.slot0;
    const bool live = rel < (unsigned long long)sc.chunks * sc.ny;
    slot_y[sl] = live ? (int)(rel / sc.chunks) * dc.step : -1;
    slot_x[sl] = live ? (int)(rel % sc.chunks) * 32 : 0;
    hit[sl] = 0;
  }
  __syncthreads();

  // run stages [s0, s1) for window `id` (slot-local id: slot = id >> 5, lane-in-slot = id & 31)
  auto run = [&](unsigned id, int s0, int s1) -> bool {
    const int sl = id >> 5, xi = slot_x[sl] + (int)(id & 31);
    const int y = slot_y[sl], x = xi * dc.step;
    const int base = y * (int)iw + x;
    const bool x0 = x == 0, y0 = y == 0;
    for (int si = s0; si < s1; si++) {
      const Stage st = s_stage[si];
      float sum = 0.0f;
      if (x0 || y0) {
        for (int i = 0; i < st.n; i++) {
          const Weak wk = s_weak[st.start + i];
          sum = __fadd_rn(sum, weak_match<true>(ii, base, x0, y0, s_geo[wk.fidx], wk, s_sub) ? wk.left : wk.right);
        }
      } else {
        for (int i = 0; i < st.n; i++) {
          const Weak wk = s_weak[st.start + i];
          sum = __fadd_rn(sum, weak_match<false>(ii, base, false, false, s_geo[wk.fidx], wk, s_sub) ? wk.left : wk.right);
        }
      }
      if (sum < st.thr) return false;
    }
    return true;
  };
  // survivors -> next list (one shared-memory atomic per warp) or, after the last group, -> hit bits
  auto keep = [&](bool alive, unsigned id, uint16_t *next, unsigned *next_cnt, bool last) {
    if (last) {
      if (alive) atomicOr(&hit[id >> 5], 1u << (id & 31));
      return;
    }
    const unsigned bal = __ballot_sync(0xFFFFFFFFu, alive);
    unsigned pos = 0;
    if (lane == 0 && bal) pos = atomicAdd(next_cnt, __popc(bal));
    pos = __shfl_sync(0xFFFFFFFFu, pos, 0);
    if (alive) next[pos + __popc(bal & ((1u << lane) - 1u))] = (uint16_t)id;
  };

  // group 0: every window of the chunk
  {
    const bool last = dc.ngroups == 1;
    for (unsigned id = tid; id < LBP_WIN_PER_CTA; id += LBP_THREADS) {
      const int sl = id >> 5;
      const bool valid = slot_y[sl] >= 0 && slot_x[sl] + (int)(id & 31) < sc.nx;
      const bool alive = valid && run(id, 0, dc.group_end[0]);
      keep(alive, id, list_a, &cnt[0], last);
    }
  }
  __syncthreads();
  uint16_t *cur = list_a, *nxt = list_b;
  for (int g = 1; g < dc.ngroups; g++) {
    const unsigned n = cnt[(g - 1) & 1];
    const bool last = g == dc.ngroups - 1;
    if (tid == 0) cnt[g & 1] = 0;
    __syncthreads();
    for (unsigned i0 = 0; i0 < n; i0 += LBP_THREADS) {     // uniform trip count (ballots inside)
      const unsigned i = i0 + tid;
      const unsigned id = i < n ? cur[i] : 0;
      const bool alive = i < n && run(id, dc.group_end[g - 1], dc.group_end[g]);
      keep(alive, id, nxt, &cnt[g & 1], last);
    }
    __syncthreads();
    uint16_t *t = cur;
    cur = nxt, nxt = t;
  }
  __syncthreads();
  for (unsigned sl = tid; sl < LBP_SLOTS_PER_CTA; sl += LBP_THREADS) masks[(size_t)f * dc.total_slots + slot_first + sl] = hit[sl];
}


// ---- k_lbp_scan3: window tiles on TMA-staged integral-image boxes --------------------------------
// step == 2 only.  With windows every 2 px, a warp's 32 lanes gather from every other 32-bit word: two
// wavefronts per load on the L1 / shared-memory data path, which is what bounds the cascade (ncu:
// l1tex__data_pipe_lsu_wavefronts 80 % of peak, 2.2x the ideal wavefront count).  k_deinterleave2 therefore first splits each table into its even-column and
// odd-column planes (one 8 B/entry streaming pass, ~1 % of the scan) so that adjacent windows read ADJACENT
// words of one plane -- which plane is a per-(feature, corner) constant, because window x positions are even.
// A CTA owns a 2-D tile of twx x twy window positions of one scale.  The box those windows can touch --
// per plane (twx + (win_w + 7) / 2) x ((twy-1)*step + win_h + 1) words, starting one row above / eight
// columns left of the first window so that the inner TMA coordinate is 16-byte aligned -- is fetched by two
// cp.async.bulk.tensor.3d copies (one per plane) into shared memory while the threads copy the cascade tables.
// TMA's zero fill supplies gs_integral_sum's "x == 0 / y == 0 -> 0" corners (reference :758-760) for free,
// so there is no edge variant.  Every lattice corner is then an LDS at base + row[j] + col[i] (byte offsets
// precomputed per scale): 20 integer adds + 16 LDS per weak classifier, against 16 LDG + ~50 address
// instructions for the global-memory gather.  Stage groups / survivor re-packing as in k_lbp_scan2, but per
// WARP (no CTA barrier between the tile load and the mask stores); hit bits land in the same per-slot mask
// words (a tile spans whole 32-window slots, so plain stores).  History on 32 UHD frames (ms): scan2 79.0;
// dense tile 81.7; parity planes 78.9; + CTA-wide flat tail 77.0; warp-autonomous lists + flat tail 63.7.
// [n][h][w] u32 -> [n][2][h][w/2]: plane q of frame f holds the columns x with x % 2 == q.  w % 8 == 0.
__global__ void __launch_bounds__(256)
k_deinterleave2(uint32_t *__restrict__ planes, const uint32_t *__restrict__ ii, unsigned w, unsigned h, unsigned n) {
  const size_t groups = (size_t)w / 8 * h;              // 8 input words -> 4 + 4 output words
  const size_t g = (size_t)blockIdx.x * 256 + threadIdx.x;
  if (g >= groups) return;
  const unsigned y = (unsigned)(g / (w / 8)), xg = (unsigned)(g % (w / 8));
  for (unsigned f = blockIdx.y; f < n; f += gridDim.y) {
    const uint4 *src = reinterpret_cast<const uint4 *>(ii + (size_t)f * w * h + (size_t)y * w + xg * 8);
    const uint4 a = __ldg(src), b = __ldg(src + 1);
    uint32_t *dst = planes + (size_t)f * w * h + (size_t)y * (w / 2) + xg * 4;
    *reinterpret_cast<uint4 *>(dst) = make_uint4(a.x, a.z, b.x, b.z);
    *reinterpret_cast<uint4 *>(dst + (size_t)(w / 2) * h) = make_uint4(a.y, a.w, b.y, b.w);
  }
}

constexpr int LBP3_THREADS = 512;                // small-window scales: two CTAs per SM
constexpr int LBP3_BIG_THREADS = 1024;           // large-window scales: one CTA per SM with a tile up to 224 KB
constexpr int LBP3_HIT_WORDS = 128;              // mask words of a tile: at most 4096 windows
constexpr int LBP3_FLAT = 8;                     // flat_n: a warp with this many survivors or fewer switches to the (window, weak) flat mode

template <int LBP3_THREADS>
__global__ void __launch_bounds__(LBP3_THREADS)
k_lbp_scan3(const __grid_constant__ CUtensorMap tmap, DevCascade dc, int si, int twx, int twy, int bw, int ph,
            int tiles_x, int flat_n, int grab, unsigned *__restrict__ masks) {
  extern __shared__ __align__(128) unsigned char lsm[];
  // two column-parity planes of bw x ph words each (see k_deinterleave2), 128-byte aligned
  const uint32_t plane_bytes = ((uint32_t)bw * ph * 4u + 127u) & ~127u;
  const uint32_t tile_bytes = 2u * plane_bytes;
  unsigned char *tile = lsm;
  // everything lives in the dynamic segment (no static __shared__: the TMA destination must stay the
  // 128-byte aligned start of it): tile | barrier, counters, 64 hit words | tables | survivor lists
  unsigned char *ctl = lsm + ((tile_bytes + 127u) & ~127u);
  uint64_t &bar = *reinterpret_cast<uint64_t *>(ctl);
  unsigned &next_slot = *reinterpret_cast<unsigned *>(ctl + 8);   // dynamic slot hand-out (grab > 0)
  unsigned *hit = reinterpret_cast<unsigned *>(ctl + 16);   // twy * (twx / 32) <= LBP3_HIT_WORDS mask words
  TileGeo *s_geo = reinterpret_cast<TileGeo *>(ctl + 640);
  Weak *s_weak = reinterpret_cast<Weak *>(s_geo + dc.nfeatures);
  Stage *s_stage = reinterpret_cast<Stage *>(s_weak + dc.nweaks);
  int *s_sub = reinterpret_cast<int *>(s_stage + dc.nstages);
  const int nwin = twx * twy;
  uint16_t *list_a = reinterpret_cast<uint16_t *>(s_sub + dc.nsubsets);

  const unsigned f = blockIdx.y, tid = threadIdx.x, lane = tid & 31;
  const ScaleInfo sc = dc.scales[si];
  const int tx = (int)(blockIdx.x % (unsigned)tiles_x), ty = (int)(blockIdx.x / (unsigned)tiles_x);
  const int wx0 = tx * twx, wy0 = ty * twy;                 // first window of the tile (window indices)
  if (tid == 0) {
    mbar_init(&bar, 1);
    mbar_fence_init();
    mbar_expect_tx(&bar, 2u * (uint32_t)bw * ph * 4u);
    // plane column of the first window's (x - 8): wx0 * step / 2 - 4 = wx0 - 4 (16-byte aligned: twx % 4 == 0)
    tma_load_3d(tile, &tmap, wx0 - 4, wy0 * dc.step - 1, 2 * (int)f, &bar);
    tma_load_3d(tile + plane_bytes, &tmap, wx0 - 4, wy0 * dc.step - 1, 2 * (int)f + 1, &bar);
  }
  {  // tables -> shared memory while the boxes are in flight
    const uint32_t *g0 = reinterpret_cast<const uint32_t *>(dc.tgeo + sc.feat_off);
    uint32_t *d0 = reinterpret_cast<uint32_t *>(s_geo);
    for (int i = tid; i < dc.nfeatures * 8; i += LBP3_THREADS) d0[i] = g0[i];
    const uint32_t *g1 = reinterpret_cast<const uint32_t *>(dc.weaks);
    uint32_t *d1 = reinterpret_cast<uint32_t *>(s_weak);
    for (int i = tid; i < dc.nweaks * 4; i += LBP3_THREADS) d1[i] = g1[i];
    const uint32_t *g2 = reinterpret_cast<const uint32_t *>(dc.stages);
    uint32_t *d2 = reinterpret_cast<uint32_t *>(s_stage);
    for (int i = tid; i < dc.nstages * 2; i += LBP3_THREADS) d2[i] = g2[i];
    for (int i = tid; i < dc.nsubsets; i += LBP3_THREADS) s_sub[i] = dc.subsets[i];
  }
  if (tid < LBP3_HIT_WORDS) hit[tid] = 0;
  if (tid == 0) next_slot = 0;
  __syncthreads();
  mbar_wait(&bar, 0);

  // adjacent windows (2 px apart) are adjacent WORDS of a parity plane: a warp's 32 lanes hit 32 banks
  const int pitch = bw * 4, xstep = 4, ystep = dc.step * pitch;
  const int shift = twx == 64 ? 6 : 5;                      // twx is 32 or 64
  // one weak classifier of window `id`: its vote (reference gs_lbp_code + gs_lbp_match, :769-788)
  auto vote = [&](unsigned id, const Weak &wk) -> float {
    const int lx = (int)(id & (unsigned)(twx - 1)), ly = (int)(id >> shift);
    const unsigned char *base = tile + ly * ystep + lx * xstep;
    const TileGeo &g = s_geo[wk.fidx];
    uint32_t v[4][4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const unsigned char *rb = base + g.row[j];
#pragma unroll
      for (int k = 0; k < 4; k++) v[j][k] = *reinterpret_cast<const uint32_t *>(rb + g.col[k]);
    }
    // cell = D + A - B - C as a difference of horizontal differences: 12 + 9 subtractions instead of 27 add/subs
    uint32_t c[3][3], hd[4][3];
#pragma unroll
    for (int j = 0; j < 4; j++)
#pragma unroll
      for (int k = 0; k < 3; k++) hd[j][k] = v[j][k + 1] - v[j][k];
#pragma unroll
    for (int j = 0; j < 3; j++)
#pragma unroll
      for (int k = 0; k < 3; k++) c[j][k] = hd[j + 1][k] - hd[j][k];
    const uint32_t m = c[1][1];
    const int code = lbp_code_of(c[0][0], c[0][1], c[0][2], c[1][2], c[2][2], c[2][1], c[2][0], c[1][0], m);
    const int idx = code >> 5;
    const bool match = idx < (int)wk.nsub && (((unsigned)s_sub[wk.sub_off + idx] >> (code & 31)) & 1u);
    return match ? wk.left : wk.right;
  };
  auto run = [&](unsigned id, int s0, int s1) -> bool {
    for (int sgi = s0; sgi < s1; sgi++) {
      const Stage st = s_stage[sgi];
      float sum = 0.0f;
      for (int i = 0; i < st.n; i++) sum = __fadd_rn(sum, vote(id, s_weak[st.start + i]));   // sequential adds, :808
      if (sum < st.thr) return false;
    }
    return true;
  };
  // From here on every warp works alone on 32-window slots: its survivors are re-packed into a warp-private list with
  // ballots -- no shared counters inside the cascade, no CTA barrier until the masks are written -- so a warp that is
  // stuck in a deep stage never holds the other fifteen up.  Which slots a warp takes: grab == 0: slot = warp,
  // warp + nwarps, ... (static; a warp whose slots hold the faces of the tile finishes long after the others, and the CTA
  // keeps its tile and warp slots until then: 24 of 32 warp slots occupied on average, ncu); grab > 0: `grab`
  // consecutive slots at a time from a shared counter, taken through all stage groups before the next hand-out.
  // The launcher always passes grab = 0.  The hand-out still stays in the kernel: without it, nvcc 12.9 compiles
  // the static walk to code that ran c4 1.2 % slower (570.1 vs 563.3 ms per step, median of three alternated runs,
  // H100 80GB HBM3 at 400 W), also with the grab parameter kept and take fixed at 0.
  constexpr int NWARPS = LBP3_THREADS / 32;
  const unsigned warp = tid >> 5, lt = (1u << lane) - 1u;
  const int nslots = nwin >> 5;
  const int cap = ((nslots + NWARPS - 1) / NWARPS) * 32;
  const int take = min(grab, cap / 32);
  const int sx_n = twx >> 5;
  // slots sb, sb + stride, ... < se through the whole cascade, then their mask words to global memory
  auto process = [&](int sb, int se, int stride) {
  uint16_t *cur = list_a + warp * cap, *nxt = list_a + (NWARPS + warp) * cap;
  unsigned n = 0;
  {
    const bool last = dc.ngroups == 1;
    for (int slot = sb; slot < se; slot += stride) {
      const unsigned id = (unsigned)slot * 32u + lane;
      const int lx = (int)(id & (unsigned)(twx - 1)), ly = (int)(id >> shift);
      const bool valid = wx0 + lx < sc.nx && wy0 + ly < sc.ny;
      const bool alive = valid && run(id, 0, dc.group_end[0]);
      const unsigned bal = __ballot_sync(0xFFFFFFFFu, alive);
      if (last) {
        if (lane == 0 && bal) hit[slot] = bal;               // bit = lane = lx % 32
      } else {
        if (alive) cur[n + __popc(bal & lt)] = (uint16_t)id;
        n += __popc(bal);
      }
    }
  }
  __syncwarp();
  for (int g = 1; g < dc.ngroups && n; g++) {
    if (n <= (unsigned)flat_n) {
      // Few survivors: spread the (window, weak) pairs of ONE stage over the lanes -- a window owns
      // P = 2^k >= stage.n adjacent lanes -- and rebuild the stage sum in the reference's order with
      // shuffles; re-pack after every stage.
      for (int sgi = dc.group_end[g - 1]; sgi < dc.nstages && n; sgi++) {
        const Stage st = s_stage[sgi];
        const bool last = sgi == dc.nstages - 1;
        int P = 1;
        while (P < (int)st.n && P < 32) P <<= 1;
        const unsigned wpw = 32u / (unsigned)P;
        const unsigned seg = lane & ~(unsigned)(P - 1), li = lane & (unsigned)(P - 1);
        unsigned m = 0;
        for (unsigned b0 = 0; b0 < n; b0 += wpw) {
          const unsigned w = b0 + lane / (unsigned)P;
          const unsigned id = w < n ? cur[w] : 0;
          float sum = 0.0f;
          for (int c0 = 0; c0 < (int)st.n; c0 += P) {                       // stages longer than 32: chunks
            const int wi = c0 + (int)li;
            const float val = (w < n && wi < (int)st.n) ? vote(id, s_weak[st.start + wi]) : 0.0f;
            const int mm = min(P, (int)st.n - c0);
            for (int i = 0; i < mm; i++) sum = __fadd_rn(sum, __shfl_sync(0xFFFFFFFFu, val, (int)seg + i));
          }
          const bool alive = w < n && li == 0 && !(sum < st.thr);
          const unsigned bal = __ballot_sync(0xFFFFFFFFu, alive);
          if (last) {
            if (alive) atomicOr(&hit[id >> 5], 1u << (id & 31));
          } else {
            if (alive) nxt[m + __popc(bal & lt)] = (uint16_t)id;
            m += __popc(bal);
          }
        }
        __syncwarp();
        n = last ? 0 : m;
        uint16_t *t = cur;
        cur = nxt, nxt = t;
      }
      break;
    }
    const bool last = g == dc.ngroups - 1;
    unsigned m = 0;
    for (unsigned i0 = 0; i0 < n; i0 += 32) {
      const unsigned i = i0 + lane;
      const unsigned id = i < n ? cur[i] : 0;
      const bool alive = i < n && run(id, dc.group_end[g - 1], dc.group_end[g]);
      const unsigned bal = __ballot_sync(0xFFFFFFFFu, alive);
      if (last) {
        if (alive) atomicOr(&hit[id >> 5], 1u << (id & 31));
      } else {
        if (alive) nxt[m + __popc(bal & lt)] = (uint16_t)id;
        m += __popc(bal);
      }
    }
    __syncwarp();
    n = last ? 0 : m;
    uint16_t *t = cur;
    cur = nxt, nxt = t;
  }
  // the slots were touched by nobody else: store their mask words -- no CTA barrier
  __syncwarp();
  for (int slot = sb + (int)lane * stride; slot < se; slot += 32 * stride) {
    const int ly = slot / sx_n, sx = slot % sx_n;
    const unsigned chunk = (unsigned)(wx0 >> 5) + (unsigned)sx;
    if (wy0 + ly < sc.ny && chunk < sc.chunks)
      masks[(size_t)f * dc.total_slots + sc.slot0 + (unsigned long long)(wy0 + ly) * sc.chunks + chunk] = hit[slot];
  }
  __syncwarp();
  };
  if (take <= 0) {
    process((int)warp, nslots, NWARPS);
  } else {
    for (;;) {
      int s0 = 0;
      if (lane == 0) s0 = (int)atomicAdd(&next_slot, (unsigned)take);
      s0 = __shfl_sync(0xFFFFFFFFu, s0, 0);
      if (s0 >= nslots) break;
      process(s0, min(s0 + take, nslots), 1);
    }
  }
}

// hits per 8-slot block, for the ordered-compaction scan
__global__ void __launch_bounds__(256)
k_lbp_count(const unsigned *__restrict__ masks, unsigned long long total_slots, unsigned *__restrict__ blockcount) {
  const unsigned long long nb = total_slots / 8;
  const unsigned long long b = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nb) return;
  const unsigned f = blockIdx.y;
  const uint4 *m = reinterpret_cast<const uint4 *>(masks + (size_t)f * total_slots + b * 8);
  const uint4 a = m[0], c = m[1];
  blockcount[(size_t)f * nb + b] = __popc(a.x) + __popc(a.y) + __popc(a.z) + __popc(a.w) + __popc(c.x) + __popc(c.y) +
                                   __popc(c.z) + __popc(c.w);
}

// one warp per 8-slot block (256 windows): blocks without hits -- almost all of them -- leave after
// two loads of the scanned counts
__global__ void __launch_bounds__(256)
k_lbp_emit(DevCascade dc, const unsigned *__restrict__ masks, const unsigned *__restrict__ blockoff,
           const unsigned *__restrict__ counts, struct gs_rect *__restrict__ rects, unsigned max_rects) {
  const unsigned f = blockIdx.y, lane = threadIdx.x & 31;
  const unsigned long long nb = dc.total_slots / 8;
  const unsigned long long b = (unsigned long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (b >= nb) return;
  const unsigned off = blockoff[(size_t)f * nb + b];
  if (off >= max_rects) return;
  // exclusive offsets: this block is empty iff the next offset (or the frame total) equals its own
  const unsigned next = b + 1 < nb ? blockoff[(size_t)f * nb + b + 1] : 0xFFFFFFFFu;
  if (next == off) return;
  (void)counts;
  const unsigned long long slot0 = b * 8;
  unsigned pos = off;
  for (int i = 0; i < 8; i++) {
    const unsigned m = masks[(size_t)f * dc.total_slots + slot0 + i];
    if (m == 0) continue;                                      // warp-uniform
    if ((m >> lane) & 1u) {
      const unsigned p = pos + __popc(m & ((1u << lane) - 1u));
      if (p < max_rects) {
        const unsigned long long slot = slot0 + i;
        const ScaleInfo sc = dc.scales[scale_of(dc, slot)];
        const unsigned long long rel = slot - sc.slot0;
        const unsigned yi = (unsigned)(rel / sc.chunks), xi = (unsigned)(rel % sc.chunks) * 32 + lane;
        *reinterpret_cast<uint4 *>(rects + (size_t)f * max_rects + p) =
            make_uint4(xi * dc.step, yi * dc.step, (unsigned)sc.win_w, (unsigned)sc.win_h);
      }
    }
    pos += __popc(m);
  }
}

// gs_lbp_window for a single window: all 32 lanes evaluate the same window
__global__ void k_lbp_window_one(const uint32_t *ii, unsigned iw, unsigned ih, int x, int y, const short4 *feat,
                                 const Weak *weaks, const int *subsets, const Stage *stages, int nstages,
                                 unsigned *out) {
  const bool hit = cascade_eval<true>(ii, iw, ih, x, y, feat, weaks, subsets, stages, nstages, true);
  if (threadIdx.x == 0) *out = hit ? 1u : 0u;
}

// ---- host: plan + device cache ---------------------------------------------------------------
struct PlanKey {
  unsigned long long hash;
  unsigned iw, ih;
  float sf, mn, mx;
  int step, device;
  int big_mode;                // GS_B200_LBP_BIG (a test flips it inside one process): -1 auto, 0 never, 1 always
  bool operator==(const PlanKey &o) const {
    return hash == o.hash && iw == o.iw && ih == o.ih && sf == o.sf && mn == o.mn && mx == o.mx && step == o.step &&
           device == o.device && big_mode == o.big_mode;
  }
};
struct PlanEntry {
  PlanKey key;
  void *blob = nullptr;
  DevCascade dc;
  std::vector<ScaleInfo> scales;
  std::vector<TilePlan> tiles;   // empty: k_lbp_scan3 not applicable
  PlanEntry() = default;
  PlanEntry(const PlanEntry &) = delete;
  PlanEntry &operator=(const PlanEntry &) = delete;
  // The device blob goes when the LAST holder lets go (the cache or a caller that is still enqueueing kernels on
  // it); cudaFree waits for work already enqueued on the device, so kernels in flight keep valid tables.
  ~PlanEntry() {
    if (!blob) return;
    int cur = 0;
    cudaGetDevice(&cur);
    if (cur != key.device) cudaSetDevice(key.device);
    cudaFree(blob);
    if (cur != key.device) cudaSetDevice(cur);
  }
};
typedef std::shared_ptr<PlanEntry> PlanRef;
static std::mutex g_plan_mutex;
static std::list<PlanRef> g_plans;   // callers hold a PlanRef: eviction / another thread's insert never invalidates it

static unsigned long long fnv(unsigned long long h, const void *p, size_t n) {
  const unsigned char *b = static_cast<const unsigned char *>(p);
  for (size_t i = 0; i < n; i++) h = (h ^ b[i]) * 1099511628211ull;
  return h;
}

static unsigned subsets_len(const struct gs_lbp_cascade *c) {
  unsigned n = 0;
  for (unsigned i = 0; i < c->nweaks; i++) {
    unsigned e = (unsigned)c->weak_subset_offset[i] + c->weak_num_subsets[i];
    if (e > n) n = e;
  }
  return n;
}

static unsigned long long cascade_hash(const struct gs_lbp_cascade *c) {
  unsigned long long h = 1469598103934665603ull;
  h = fnv(h, &c->window_w, 2), h = fnv(h, &c->window_h, 2);
  h = fnv(h, &c->nfeatures, 2), h = fnv(h, &c->nweaks, 2), h = fnv(h, &c->nstages, 2);
  h = fnv(h, c->features, (size_t)c->nfeatures * 4);
  h = fnv(h, c->weak_feature_idx, (size_t)c->nweaks * 2);
  h = fnv(h, c->weak_left_val, (size_t)c->nweaks * 4), h = fnv(h, c->weak_right_val, (size_t)c->nweaks * 4);
  h = fnv(h, c->weak_subset_offset, (size_t)c->nweaks * 2), h = fnv(h, c->weak_num_subsets, (size_t)c->nweaks * 2);
  h = fnv(h, c->subsets, (size_t)subsets_len(c) * 4);
  h = fnv(h, c->stage_weak_start, (size_t)c->nstages * 2), h = fnv(h, c->stage_nweaks, (size_t)c->nstages * 2);
  h = fnv(h, c->stage_threshold, (size_t)c->nstages * 4);
  return h;
}

// The reference's scale ladder (:819-821): fn(scale, win_w, win_h) for each scale it scans, until fn returns false.
// A ladder that does not grow (scale_factor <= 1) ends after its first scale here; the reference repeats that scale
// until max_rects fills, and never returns when it has no hit.  A NaN scale_factor ends after the first scale in both.
template <class F>
static void walk_ladder(const struct gs_lbp_cascade *c, unsigned iw, unsigned ih, float scale_factor, float min_scale,
                        float max_scale, F fn) {
  for (volatile float scale = min_scale; scale <= max_scale; scale = scale * scale_factor) {
    const float s = scale;
    const int win_w = (int)((float)c->window_w * s), win_h = (int)((float)c->window_h * s);
    if (win_w > (int)iw || win_h > (int)ih) break;
    if (!fn(s, win_w, win_h) || !(scale_factor > 1.0f)) break;
  }
}

// one entry per scale of the ladder; false (and the first LBP_MAX_SCALES entries) when it has more scales than that
static bool build_scales(const struct gs_lbp_cascade *c, unsigned iw, unsigned ih, float scale_factor, float min_scale,
                         float max_scale, int step, std::vector<float> &scale_vals, std::vector<ScaleInfo> &out) {
  unsigned long long slot = 0;
  bool fits = true;
  walk_ladder(c, iw, ih, scale_factor, min_scale, max_scale, [&](float s, int win_w, int win_h) {
    if (out.size() == (size_t)LBP_MAX_SCALES) return fits = false;
    ScaleInfo si;
    si.win_w = win_w, si.win_h = win_h;
    si.nx = ((int)iw - win_w) / step + 1, si.ny = ((int)ih - win_h) / step + 1;
    si.chunks = (unsigned)(si.nx + 31) / 32;
    si.feat_off = 0;   // set with the feature tables (get_plan)
    si.slot0 = slot;
    slot += (unsigned long long)si.chunks * si.ny;
    slot = (slot + LBP_SLOTS_PER_CTA - 1) / LBP_SLOTS_PER_CTA * LBP_SLOTS_PER_CTA;   // CTAs never straddle scales
    out.push_back(si);
    scale_vals.push_back(s);
    return true;
  });
  return fits;
}

// the cached plan of this cascade and geometry; on a miss it is built and uploaded (blocking) unless !may_build.
// nullptr with the recorded error in *err when there is none
static PlanRef get_plan(const struct gs_lbp_cascade *c, unsigned iw, unsigned ih, float sf, float mn, float mx,
                        int step, bool may_build, int *err) {
  int dev = 0;
  cudaGetDevice(&dev);
  // test hook: 1 = every scale on the 1024-thread tile form, 0 = none, unset = by tile height (tests reach both
  // forms on frames where the automatic choice takes only one)
  const char *be = getenv("GS_B200_LBP_BIG");
  PlanKey key = {cascade_hash(c), iw, ih, sf, mn, mx, step, dev, be ? atoi(be) : -1};
  std::lock_guard<std::mutex> lock(g_plan_mutex);
  for (auto &r : g_plans)
    if (r->key == key) return r;
  if (!may_build) {
    *err = record_error(cudaErrorStreamCaptureUnsupported, __FILE__, __LINE__);
    return nullptr;
  }

  PlanRef ref = std::make_shared<PlanEntry>();
  PlanEntry &e = *ref;
  e.key = key;
  std::vector<float> svals;
  if (!build_scales(c, iw, ih, sf, mn, mx, step, svals, e.scales)) {
    *err = record_error(cudaErrorInvalidValue, __FILE__, __LINE__);   // a ladder of more than LBP_MAX_SCALES scales
    return nullptr;
  }
  const int ns = (int)e.scales.size(), nf = c->nfeatures, nw = c->nweaks, nst = c->nstages;
  const unsigned nsub = subsets_len(c);
  // Neighbouring scales of a long ladder mostly truncate to the same window and features: such a scale scans with
  // the previous scale's tables (its hits are the same windows again).
  std::vector<short4> feat;
  bool safe = true;
  for (int s = 0; s < ns; s++) {
    const size_t at = feat.size();
    for (int i = 0; i < nf; i++) {
      const float sc = svals[s];
      int fx = (int)((float)c->features[i * 4 + 0] * sc), fy = (int)((float)c->features[i * 4 + 1] * sc);
      int fw = (int)((float)c->features[i * 4 + 2] * sc), fh = (int)((float)c->features[i * 4 + 3] * sc);
      if (fw < 1) fw = 1;
      if (fh < 1) fh = 1;
      feat.push_back(make_short4((short)fx, (short)fy, (short)fw, (short)fh));
      if (fx < 0 || fy < 0 || fx + 3 * fw > e.scales[s].win_w || fy + 3 * fh > e.scales[s].win_h) safe = false;
    }
    const bool same = s > 0 && e.scales[s].win_w == e.scales[s - 1].win_w && e.scales[s].win_h == e.scales[s - 1].win_h &&
                      memcmp(feat.data() + at, feat.data() + e.scales[s - 1].feat_off, sizeof(short4) * nf) == 0;
    if (same) feat.resize(at);
    e.scales[s].feat_off = same ? e.scales[s - 1].feat_off : (unsigned)at;
  }
  std::vector<FeatGeo> geo(feat.size());
  for (size_t i = 0; i < feat.size(); i++) {
    const short4 ft = feat[i];
    for (int k = 0; k < 4; k++) {
      geo[i].row[k] = (ft.y - 1 + k * ft.w) * (int)iw;
      geo[i].col[k] = ft.x - 1 + k * ft.z;
    }
  }
  // window tiles for k_lbp_scan3: per scale the widest tile whose box fits a TMA box (256 elements per
  // dimension) and the tallest one whose box fits the shared-memory budget
  const size_t table_bytes_t = sizeof(TileGeo) * nf + sizeof(Weak) * nw + sizeof(Stage) * nst + 4 * (size_t)nsub;
  // per-CTA shared-memory budget (tile planes + tables + survivor lists): 113 KB lets two 512-thread CTAs share an
  // SM at every scale (round 1 bounded the planes alone by 100 KB, and scale 10 of the UHD ladder came out at
  // 119.9 KB: one CTA per SM, 705 us instead of ~500)
  const size_t tile_budget = (size_t)113 * 1024;
  const int big_auto_rows = 32;                                      // scales whose 2-per-SM tile has fewer window rows go big
  std::vector<TileGeo> tgeo;
  bool tiles_ok = safe && ns > 0 && iw % 8 == 0 && step == 2;
  for (int s2 = 0; s2 < ns && tiles_ok; s2++) {
    const ScaleInfo &si = e.scales[s2];
    TilePlan tp;
    tp.twx = 0;
    for (int cand = 64; cand >= 32; cand /= 2)
      if (cand + (si.win_w + 7) / 2 + 4 <= 256) {
        tp.twx = cand;
        break;
      }
    if (!tp.twx) {
      tiles_ok = false;
      break;
    }
    tp.bw = (tp.twx - 1 + (si.win_w + 7) / 2 + 1 + 3) & ~3;   // plane columns: lx + (fx + i*fw + 7) / 2
    // Tallest tile under a per-CTA shared-memory budget.  A window row costs 2 table rows, the first one win_h + 1:
    // for the large scales a 113 KB CTA (two per SM) holds only 8-16 window rows -- 1 or 2 slots per warp, and a
    // (win_h + 1)-row halo re-read per 16 rows -- so those scales run one 1024-thread CTA per SM on a tile of up to
    // 224 KB instead (round 1: scales 10..14 of the UHD ladder took 30-60 % longer than the small ones).
    auto fit = [&](int nthreads, size_t budget, int max_windows, TilePlan &o) {
      o = tp;
      o.twy = 0, o.threads = nthreads;
      for (int cand = max_windows / tp.twx; cand >= 1; cand--) {
        if (cand > 32 && cand % 8) continue;                       // keep the candidate list short
        const int ph = (cand - 1) * step + si.win_h + 1;
        const size_t plane = ((size_t)tp.bw * ph * 4 + 127) & ~(size_t)127;
        const size_t nwarps = nthreads / 32, slots = (size_t)tp.twx * cand / 32;
        const size_t total = 2 * plane + 640 + table_bytes_t + 4 * nwarps * ((slots + nwarps - 1) / nwarps) * 32 + 64;
        if (ph <= 256 && (total <= budget || cand == 1) && total <= (size_t)226 * 1024) {
          o.twy = cand, o.ph = ph, o.smem = total;
          break;
        }
      }
    };
    TilePlan small, big;
    fit(LBP3_THREADS, tile_budget, 2048, small);
    fit(LBP3_BIG_THREADS, (size_t)224 * 1024, 32 * LBP3_HIT_WORDS, big);
    const bool use_big = big.twy > 0 && (key.big_mode == 1 || (key.big_mode < 0 && small.twy < big_auto_rows));
    tp = use_big ? big : small;
    if (!tp.twy) {
      tiles_ok = false;
      break;
    }
    tp.tiles_x = (si.nx + tp.twx - 1) / tp.twx, tp.tiles_y = (si.ny + tp.twy - 1) / tp.twy;
    if ((unsigned long long)tp.tiles_x * tp.tiles_y > 0x7FFFFFFFull) tiles_ok = false;
    e.tiles.push_back(tp);
    if (s2 > 0 && si.feat_off == e.scales[s2 - 1].feat_off) continue;   // the same window: the same tile plan and tgeo
    for (int i = 0; i < nf; i++) {
      const short4 ft = feat[si.feat_off + i];
      TileGeo g;
      const int plane = (int)((((size_t)tp.bw * tp.ph * 4 + 127) & ~(size_t)127));
      for (int k = 0; k < 4; k++) {
        const int d = ft.x + k * ft.z + 7;          // dense column relative to the box origin (x - 8)
        g.row[k] = (ft.y + k * ft.w) * tp.bw * 4;
        g.col[k] = (d & 1) * plane + (d >> 1) * 4;
      }
      tgeo.push_back(g);
    }
  }
  if (!tiles_ok) e.tiles.clear(), tgeo.clear();
  std::vector<Weak> weaks(nw);
  for (int i = 0; i < nw; i++) {
    weaks[i].left = c->weak_left_val[i], weaks[i].right = c->weak_right_val[i];
    weaks[i].fidx = c->weak_feature_idx[i], weaks[i].sub_off = c->weak_subset_offset[i];
    weaks[i].nsub = c->weak_num_subsets[i], weaks[i].pad = 0;
  }
  std::vector<Stage> stages(nst);
  for (int i = 0; i < nst; i++) {
    stages[i].thr = c->stage_threshold[i];
    stages[i].start = c->stage_weak_start[i], stages[i].n = c->stage_nweaks[i];
  }
  auto align16 = [](size_t v) { return (v + 15) & ~(size_t)15; };
  const size_t o_sc = 0, o_ft = align16(o_sc + sizeof(ScaleInfo) * (ns ? ns : 1));
  const size_t o_wk = align16(o_ft + sizeof(short4) * feat.size()), o_sb = align16(o_wk + sizeof(Weak) * nw);
  const size_t o_st = align16(o_sb + 4 * (size_t)nsub), o_ge = align16(o_st + sizeof(Stage) * nst);
  const size_t o_tg = align16(o_ge + sizeof(FeatGeo) * geo.size());
  const size_t total = align16(o_tg + sizeof(TileGeo) * tgeo.size());
  std::vector<unsigned char> host(total, 0);
  if (!tgeo.empty()) memcpy(&host[o_tg], tgeo.data(), sizeof(TileGeo) * tgeo.size());
  if (ns) memcpy(&host[o_sc], e.scales.data(), sizeof(ScaleInfo) * ns);
  if (!feat.empty()) memcpy(&host[o_ft], feat.data(), sizeof(short4) * feat.size());
  memcpy(&host[o_wk], weaks.data(), sizeof(Weak) * nw);
  memcpy(&host[o_sb], c->subsets, 4 * (size_t)nsub);
  memcpy(&host[o_st], stages.data(), sizeof(Stage) * nst);
  if (!geo.empty()) memcpy(&host[o_ge], geo.data(), sizeof(FeatGeo) * geo.size());
  if (cudaMalloc(&e.blob, total) != cudaSuccess) {
    *err = record_error(cudaErrorMemoryAllocation, __FILE__, __LINE__);
    return nullptr;
  }
  if ((*err = upload(e.blob, host.data(), total, __FILE__, __LINE__))) return nullptr;
  unsigned char *b = static_cast<unsigned char *>(e.blob);
  e.dc.scales = reinterpret_cast<const ScaleInfo *>(b + o_sc);
  e.dc.feat = reinterpret_cast<const short4 *>(b + o_ft);
  e.dc.weaks = reinterpret_cast<const Weak *>(b + o_wk);
  e.dc.subsets = reinterpret_cast<const int *>(b + o_sb);
  e.dc.stages = reinterpret_cast<const Stage *>(b + o_st);
  e.dc.geo = reinterpret_cast<const FeatGeo *>(b + o_ge);
  e.dc.tgeo = reinterpret_cast<const TileGeo *>(b + o_tg);
  e.dc.nweaks = nw, e.dc.nsubsets = (int)nsub;
  {  // stage groups: re-pack after each of the first stages (most windows die there), then coarser
    const int cuts[7] = {1, 2, 3, 4, 6, 9, 13};
    int ng = 0;
    for (int k = 0; k < 7 && ng < LBP_MAX_GROUPS - 1; k++)
      if (cuts[k] < nst) e.dc.group_end[ng++] = cuts[k];
    e.dc.group_end[ng++] = nst;
    e.dc.ngroups = ng;
    for (int k = ng; k < LBP_MAX_GROUPS; k++) e.dc.group_end[k] = nst;
  }
  e.dc.nscales = ns, e.dc.nfeatures = nf, e.dc.nstages = nst, e.dc.step = step;
  e.dc.safe_geometry = safe;
  e.dc.total_slots = 0, e.dc.total_windows = 0;
  for (auto &s : e.scales) {
    const unsigned long long end = s.slot0 + (unsigned long long)s.chunks * s.ny;
    e.dc.total_slots = (end + LBP_SLOTS_PER_CTA - 1) / LBP_SLOTS_PER_CTA * LBP_SLOTS_PER_CTA;
    e.dc.total_windows += (unsigned long long)s.nx * s.ny;
  }
  if (g_plans.size() >= 16) g_plans.pop_front();   // tiny cache: drop the oldest (freed once nobody uses it)
  g_plans.push_back(ref);
  return ref;
}

}  // namespace gsb

extern "C" {

unsigned long long gs_b200_lbp_window_count(const struct gs_lbp_cascade *c, unsigned iw, unsigned ih,
                                            float scale_factor, float min_scale, float max_scale, int step) {
  GSB_ASSERT(c && step > 0);
  unsigned long long n = 0;
  gsb::walk_ladder(c, iw, ih, scale_factor, min_scale, max_scale, [&](float, int win_w, int win_h) {
    n += (unsigned long long)(((int)iw - win_w) / step + 1) * (((int)ih - win_h) / step + 1);
    return true;
  });
  return n;
}

int gs_b200_lbp_detect_batch(const struct gs_lbp_cascade *c, const uint32_t *ii, unsigned iw, unsigned ih,
                             unsigned n, struct gs_rect *rects, unsigned *counts, unsigned max_rects,
                             float scale_factor, float min_scale, float max_scale, int step, gs_b200_stream s) {
  GSB_ASSERT(c && ii && iw > 0 && ih > 0 && counts && step > 0);  // step <= 0 never terminates in the reference
  GSB_ASSERT(rects || max_rects == 0);
  if (n == 0) return 0;
  if (n > gsb::GRID_FRAMES)   // the scan, count and emit kernels put the frame in grid y
    return gsb::for_frame_groups(n, [&](unsigned f0, unsigned m) {
      return gs_b200_lbp_detect_batch(c, ii + (size_t)f0 * iw * ih, iw, ih, m, rects ? rects + (size_t)f0 * max_rects : rects,
                                      counts + f0, max_rects, scale_factor, min_scale, max_scale, step, s);
    });
  cudaStream_t st = static_cast<cudaStream_t>(s);
  // a plan miss allocates and uploads synchronously, which a graph capture cannot hold
  const bool cap = gsb::capturing(st);
  int err = 0;
  gsb::PlanRef p = gsb::get_plan(c, iw, ih, scale_factor, min_scale, max_scale, step, !cap, &err);
  if (!p) return err;
  const gsb::DevCascade &dc = p->dc;
  if (dc.total_slots == 0 || max_rects == 0) {
    GSB_CHECK(cudaMemsetAsync(counts, 0, sizeof(unsigned) * n, st));
    return 0;
  }
  const unsigned long long nblocks = (dc.total_slots + 7) / 8;
  GSB_ASSERT(nblocks < 0x7FFFFFFFull);
  unsigned *masks = static_cast<unsigned *>(gsb::workspace(st, gsb::WS_LBP_A, 4 * (size_t)dc.total_slots * n));
  unsigned *bcount = static_cast<unsigned *>(gsb::workspace(st, gsb::WS_LBP_B, 4 * (size_t)nblocks * n));
  if (!masks || !bcount) return gsb::workspace_error();
  dim3 grid((unsigned)nblocks, n);
  const size_t table_bytes = sizeof(gsb::FeatGeo) * dc.nfeatures + sizeof(gsb::Weak) * dc.nweaks +
                             sizeof(gsb::Stage) * dc.nstages + 4 * (size_t)dc.nsubsets;
  const size_t smem2 = table_bytes + 2 * sizeof(uint16_t) * gsb::LBP_WIN_PER_CTA;
  // k_lbp_scan3 (TMA-staged parity-plane tiles, warp-autonomous survivor lists) when the scan is the usual
  // step-2 one on 8-px-aligned tables; bit-exact with k_lbp_scan2, half its instructions.
  const bool v3 = !p->tiles.empty() && reinterpret_cast<uintptr_t>(ii) % 16 == 0 && !gsb::force_generic();
  const bool v2 = !v3 && dc.safe_geometry && smem2 <= 160 * 1024 && (unsigned long long)iw * ih < 0x7FFFFFFFull;
  if (v3) {
    GSB_CHECK(cudaMemsetAsync(masks, 0, 4 * (size_t)dc.total_slots * n, st));   // padding slots between scales
    // frames go through in chunks so that the de-interleaved copy stays small (<= 1 GiB of workspace)
    const size_t frame_bytes = (size_t)iw * ih * 4;
    unsigned chunk = (unsigned)(((size_t)1 << 30) / frame_bytes);
    if (const char *ce = getenv("GS_B200_LBP_CHUNK_FRAMES")) chunk = (unsigned)atoi(ce);   // test hook
    chunk = chunk < 1 ? 1 : (chunk > n ? n : chunk);
    uint32_t *planes = static_cast<uint32_t *>(gsb::workspace(st, gsb::WS_LBP_C, frame_bytes * chunk));
    if (!planes) return gsb::workspace_error();
    for (unsigned f0 = 0; f0 < n; f0 += chunk) {
      const unsigned nf = n - f0 < chunk ? n - f0 : chunk;
      const uint32_t *src = ii + (size_t)f0 * iw * ih;
      const size_t groups = (size_t)iw / 8 * ih;
      GSB_LAUNCH(gsb::k_deinterleave2, dim3((unsigned)((groups + 255) / 256), nf < 64u ? nf : 64u), 256, 0, st, planes, src,
                 iw, ih, nf);
      for (int si = 0; si < dc.nscales; si++) {
        const gsb::TilePlan &tp = p->tiles[si];
        CUtensorMap tm;
        if (!gsb::make_tmap_u32frames(&tm, planes, iw / 2, ih, 2 * nf, (unsigned)tp.bw, (unsigned)tp.ph))
          return gsb::record_error(cudaErrorInvalidValue, __FILE__, __LINE__);
        const bool big = tp.threads == gsb::LBP3_BIG_THREADS;
        GSB_LAUNCH(big ? gsb::k_lbp_scan3<gsb::LBP3_BIG_THREADS> : gsb::k_lbp_scan3<gsb::LBP3_THREADS>,
                   dim3((unsigned)(tp.tiles_x * tp.tiles_y), nf), big ? gsb::LBP3_BIG_THREADS : gsb::LBP3_THREADS, tp.smem, st,
                   tm, dc, si, tp.twx, tp.twy, tp.bw, tp.ph, tp.tiles_x, gsb::LBP3_FLAT, 0, masks + (size_t)f0 * dc.total_slots);
      }
    }
  } else if (v2) {
    dim3 grid2((unsigned)(dc.total_slots / gsb::LBP_SLOTS_PER_CTA), n);
    GSB_LAUNCH(gsb::k_lbp_scan2, grid2, gsb::LBP_THREADS, smem2, st, ii, iw, ih, dc, masks);
  } else {
    GSB_LAUNCH(dc.safe_geometry ? gsb::k_lbp_scan<false> : gsb::k_lbp_scan<true>, grid, 256, 0, st, ii, iw, ih, dc, masks, bcount);
  }
  if (v3 || v2)   // k_lbp_scan counts its blocks' survivors itself
    GSB_LAUNCH(gsb::k_lbp_count, dim3((unsigned)((nblocks + 255) / 256), n), 256, 0, st, masks, dc.total_slots, bcount);
  GSB_LAUNCH(gsb::k_row_scan, n, 1024, 0, st, bcount, (unsigned)nblocks, counts, max_rects);
  GSB_LAUNCH(gsb::k_lbp_emit, dim3((unsigned)((nblocks + 7) / 8), n), 256, 0, st, dc, masks, bcount, counts, rects, max_rects);
  return 0;
}

}  // extern "C"

namespace gsb {

// single-window call of api.cu (gs_lbp_window): scale-specific geometry is built on the fly
int lbp_window_single(const struct gs_lbp_cascade *c, const uint32_t *ii, unsigned iw, unsigned ih, int x, int y,
                      float scale, unsigned *out_dev, cudaStream_t s) {
  const int nf = c->nfeatures, nw = c->nweaks, nst = c->nstages;
  const unsigned nsub = gsb::subsets_len(c);
  std::vector<short4> feat(nf);
  for (int i = 0; i < nf; i++) {
    int fx = (int)((float)c->features[i * 4 + 0] * scale), fy = (int)((float)c->features[i * 4 + 1] * scale);
    int fw = (int)((float)c->features[i * 4 + 2] * scale), fh = (int)((float)c->features[i * 4 + 3] * scale);
    feat[i] = make_short4((short)fx, (short)fy, (short)(fw < 1 ? 1 : fw), (short)(fh < 1 ? 1 : fh));
  }
  std::vector<gsb::Weak> weaks(nw);
  for (int i = 0; i < nw; i++) {
    weaks[i].left = c->weak_left_val[i], weaks[i].right = c->weak_right_val[i];
    weaks[i].fidx = c->weak_feature_idx[i], weaks[i].sub_off = c->weak_subset_offset[i];
    weaks[i].nsub = c->weak_num_subsets[i], weaks[i].pad = 0;
  }
  std::vector<gsb::Stage> stages(nst);
  for (int i = 0; i < nst; i++) {
    stages[i].thr = c->stage_threshold[i];
    stages[i].start = c->stage_weak_start[i], stages[i].n = c->stage_nweaks[i];
  }
  const size_t o_ft = 0, o_wk = (sizeof(short4) * nf + 15) & ~(size_t)15;
  const size_t o_sb = (o_wk + sizeof(gsb::Weak) * nw + 15) & ~(size_t)15;
  const size_t o_st = (o_sb + 4 * (size_t)nsub + 15) & ~(size_t)15, total = o_st + sizeof(gsb::Stage) * nst;
  unsigned char *blob = static_cast<unsigned char *>(gsb::workspace(s, gsb::WS_LBP_C, total));
  if (!blob) return gsb::workspace_error();
  GSB_CHECK(cudaMemcpyAsync(blob + o_ft, feat.data(), sizeof(short4) * nf, cudaMemcpyHostToDevice, s));
  GSB_CHECK(cudaMemcpyAsync(blob + o_wk, weaks.data(), sizeof(gsb::Weak) * nw, cudaMemcpyHostToDevice, s));
  GSB_CHECK(cudaMemcpyAsync(blob + o_sb, c->subsets, 4 * (size_t)nsub, cudaMemcpyHostToDevice, s));
  GSB_CHECK(cudaMemcpyAsync(blob + o_st, stages.data(), sizeof(gsb::Stage) * nst, cudaMemcpyHostToDevice, s));
  GSB_CHECK(cudaStreamSynchronize(s));  // the host vectors above go out of scope
  GSB_LAUNCH(gsb::k_lbp_window_one, 1, 32, 0, s, ii, iw, ih, x, y, reinterpret_cast<const short4 *>(blob + o_ft),
             reinterpret_cast<const gsb::Weak *>(blob + o_wk), reinterpret_cast<const int *>(blob + o_sb),
             reinterpret_cast<const gsb::Stage *>(blob + o_st), nst, out_dev);
  return 0;
}
}  // namespace gsb
