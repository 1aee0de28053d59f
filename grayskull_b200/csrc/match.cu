// match.cu -- gs_match_orb (reference grayskull.h:671-699; SURVEY.md 8f "next" item N1).
//
// Brute-force Hamming nearest neighbour with the 0.8 ratio test.  For query i the reference's scan
// keeps the two smallest distances of {d_j} U {M, M}, M = max_distance + 1 (fp32), and the first j
// attaining the smallest; it emits {i, j, (unsigned)best} when best <= max_distance and
// best < 0.8f * second (fp32 product), in query order, until max_matches.
//   k_match_best    : a CTA owns 16 consecutive queries of one (set1, set2) pair, two per warp.  The
//                     candidate descriptors are staged through shared memory in chunks of 256 (so each
//                     is fetched once per 16 queries), every lane scans a strided subset keeping its own
//                     two smallest (distance, index) keys and the warp merges them with an order-free
//                     two-minimum merge (ties -> lower index), which equals the sequential scan's result.
//   k_match_compact : one CTA per pair: accepted queries are compacted in query order up to the cap.
#include "common.cuh"

namespace gsb {

struct KpRec48 {
  uint32_t w[12];
};
struct MatchRec {
  unsigned idx1, idx2, distance;
};
constexpr int MT_CHUNK = 256;   // candidate descriptors per shared-memory chunk

// popcount of 8 words.  POPC issues at 16 lanes/clk/SM against 64 for LOP3, so 8 POPCs per comparison
// bound the plain form.  A carry-save adder tree (LOP3 pairs: 0x96 sum, 0xE8 majority) compresses the
// words first.  Two levels (5 POPC + 6 LOP3) balance the two pipes: one level (6 POPC + 4 LOP3) leaves
// POPC the bound, three (4 POPC + 14 LOP3) make the ALU pipe the bound again.
__device__ __forceinline__ void csa(uint32_t a, uint32_t b, uint32_t c, uint32_t &sum, uint32_t &carry) {
  // explicit LOP3s (0x96 = a^b^c, 0xE8 = majority): left to itself nvcc folds the caller's q^d xors into
  // 4-input expressions and spends ~50 % more LOP3s
  asm("lop3.b32 %0, %1, %2, %3, 0x96;" : "=r"(sum) : "r"(a), "r"(b), "r"(c));
  asm("lop3.b32 %0, %1, %2, %3, 0xE8;" : "=r"(carry) : "r"(a), "r"(b), "r"(c));
}
__device__ __forceinline__ unsigned popc8(const uint32_t (&x)[8]) {
  uint32_t s1, c1, s2, c2, s3, c3;
  csa(x[0], x[1], x[2], s1, c1);
  csa(x[3], x[4], x[5], s2, c2);
  csa(s1, s2, x[6], s3, c3);
  return __popc(s3) + __popc(x[7]) + 2 * (__popc(c1) + __popc(c2) + __popc(c3));
}

// Scan state in the integer domain: key = distance << 22 | candidate index, so that min() over keys also
// breaks distance ties towards the lower index, and the two smallest keys carry the two smallest
// distances.  M is represented by thr << 22 with thr = ceil(M) clamped to [0, 257]: for an integer d,
// d < M <=> d < thr, so a key replaces the M stand-in exactly when the reference's fp32 compare does,
// and a state still >= thr << 22 at the end means "M".
constexpr int MT_IDX_BITS = 22;
constexpr int MT_QPW = 2;            // queries per warp: each staged candidate is read once for QPW queries
constexpr int MT_QPC = 8 * MT_QPW;   // queries per CTA

__global__ void __launch_bounds__(256)
k_match_best(const KpRec48 *__restrict__ k1, const unsigned *__restrict__ n1, unsigned stride1,
             const KpRec48 *__restrict__ k2, const unsigned *__restrict__ n2, unsigned stride2, float max_distance,
             uint2 *__restrict__ cand) {
  __shared__ __align__(16) uint32_t s_desc[MT_CHUNK][8];
  const unsigned pair = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned i0 = blockIdx.x * MT_QPC + warp * MT_QPW;
  const unsigned cn1 = min(n1[pair], stride1), cn2 = min(n2[pair], stride2);
  if (blockIdx.x * MT_QPC >= cn1) return;                // whole CTA
  const bool active = i0 < cn1;
  uint32_t q[MT_QPW][8];
#pragma unroll
  for (int t = 0; t < MT_QPW; t++) {
    const unsigned i = min(i0 + t, cn1 - 1);
    const uint4 *p = reinterpret_cast<const uint4 *>(k1 + (size_t)pair * stride1 + i);
    const uint4 a = __ldg(p + 1), b = __ldg(p + 2);
    q[t][0] = a.x, q[t][1] = a.y, q[t][2] = a.z, q[t][3] = a.w, q[t][4] = b.x, q[t][5] = b.y, q[t][6] = b.z, q[t][7] = b.w;
  }
  const float M = __fadd_rn(max_distance, 1.0f);
  const unsigned thr = (unsigned)fminf(fmaxf(ceilf(M), 0.0f), 257.0f);
  const unsigned sentinel = thr << MT_IDX_BITS;
  unsigned best[MT_QPW], second[MT_QPW];
#pragma unroll
  for (int t = 0; t < MT_QPW; t++) best[t] = second[t] = sentinel;
  const KpRec48 *set2 = k2 + (size_t)pair * stride2;
  for (unsigned c0 = 0; c0 < cn2; c0 += MT_CHUNK) {
    const unsigned cn = min((unsigned)MT_CHUNK, cn2 - c0);
    __syncthreads();
    for (unsigned t = threadIdx.x; t < cn * 2; t += 256) {          // two 16-byte halves per descriptor
      const uint4 v = __ldg(reinterpret_cast<const uint4 *>(set2 + c0 + (t >> 1)) + 1 + (t & 1));
      *reinterpret_cast<uint4 *>(&s_desc[t >> 1][4 * (t & 1)]) = v;
    }
    __syncthreads();
    if (active) {
#pragma unroll 2
      for (unsigned j = lane; j < cn; j += 32) {
        const uint4 a = *reinterpret_cast<const uint4 *>(&s_desc[j][0]), b = *reinterpret_cast<const uint4 *>(&s_desc[j][4]);
#pragma unroll
        for (int t = 0; t < MT_QPW; t++) {
          const uint32_t x[8] = {q[t][0] ^ a.x, q[t][1] ^ a.y, q[t][2] ^ a.z, q[t][3] ^ a.w,
                                 q[t][4] ^ b.x, q[t][5] ^ b.y, q[t][6] ^ b.z, q[t][7] ^ b.w};
          const unsigned key = (popc8(x) << MT_IDX_BITS) + (c0 + j);  // reference :690-693, in key form
          second[t] = min(second[t], max(key, best[t]));
          best[t] = min(best[t], key);
        }
      }
    }
  }
  if (!active) return;
#pragma unroll
  for (int t = 0; t < MT_QPW; t++) {
    unsigned b = best[t], s = second[t];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned ob = __shfl_xor_sync(0xFFFFFFFFu, b, o), os = __shfl_xor_sync(0xFFFFFFFFu, s, o);
      s = min(min(s, os), max(b, ob));
      b = min(b, ob);
    }
    if (lane == 0 && i0 + t < cn1) {
      const float fb = b >= sentinel ? M : (float)(b >> MT_IDX_BITS);
      const float fs = s >= sentinel ? M : (float)(s >> MT_IDX_BITS);
      const bool accept = fb <= max_distance && fb < __fmul_rn(0.8f, fs);   // reference :695
      const unsigned idx = b >= sentinel ? 0u : (b & ((1u << MT_IDX_BITS) - 1u));
      cand[(size_t)pair * stride1 + i0 + t] = make_uint2(idx | (accept ? 0x80000000u : 0u), (unsigned)fb);
    }
  }
}

__global__ void __launch_bounds__(256)
k_match_compact(const uint2 *__restrict__ cand, const unsigned *__restrict__ n1, unsigned stride1,
                MatchRec *__restrict__ matches, unsigned *__restrict__ counts, unsigned max_matches) {
  __shared__ unsigned wcnt[8];
  const unsigned pair = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned cn1 = min(n1[pair], stride1);
  unsigned running = 0;
  for (unsigned b = 0; b < cn1 && running < max_matches; b += 256) {
    const unsigned i = b + tid;
    uint2 c = make_uint2(0, 0);
    if (i < cn1) c = cand[(size_t)pair * stride1 + i];
    const bool acc = (c.x >> 31) != 0;
    const unsigned bal = __ballot_sync(0xFFFFFFFFu, acc);
    if (lane == 0) wcnt[warp] = __popc(bal);
    __syncthreads();
    unsigned before = 0, total = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) {
      const unsigned cc = wcnt[k];
      before += (k < (int)warp) ? cc : 0;
      total += cc;
    }
    const unsigned pos = running + before + __popc(bal & ((1u << lane) - 1u));
    if (acc && pos < max_matches) {
      MatchRec m;
      m.idx1 = i, m.idx2 = c.x & 0x7FFFFFFFu, m.distance = c.y;
      matches[(size_t)pair * max_matches + pos] = m;
    }
    running += total;
    __syncthreads();
  }
  if (tid == 0) counts[pair] = min(running, max_matches);
}

}  // namespace gsb

extern "C" int gs_b200_match_orb_batch(const struct gs_keypoint *kps1, const unsigned *n1, unsigned stride1,
                                       const struct gs_keypoint *kps2, const unsigned *n2, unsigned stride2,
                                       unsigned npairs, struct gs_match *matches, unsigned *counts,
                                       unsigned max_matches, float max_distance, gs_b200_stream s) {
  GSB_ASSERT(kps1 && kps2 && matches);   // reference :683
  GSB_ASSERT(n1 && n2 && counts);
  if (npairs == 0) return 0;
  cudaStream_t st = static_cast<cudaStream_t>(s);
  if (stride1 == 0 || max_matches == 0) {
    GSB_CHECK(cudaMemsetAsync(counts, 0, sizeof(unsigned) * npairs, st));
    return 0;
  }
  GSB_ASSERT(npairs <= 65535u && stride1 < 0x7FFFFFFFu && stride2 < (1u << gsb::MT_IDX_BITS));
  uint2 *cand = static_cast<uint2 *>(gsb::workspace(st, gsb::WS_ORB_A, sizeof(uint2) * (size_t)stride1 * npairs));
  if (!cand) return gsb::workspace_error();
  GSB_LAUNCH(gsb::k_match_best, dim3((stride1 + gsb::MT_QPC - 1) / gsb::MT_QPC, npairs), 256, 0, st,
             reinterpret_cast<const gsb::KpRec48 *>(kps1), n1, stride1, reinterpret_cast<const gsb::KpRec48 *>(kps2), n2, stride2,
             max_distance, cand);
  GSB_LAUNCH(gsb::k_match_compact, npairs, 256, 0, st, cand, n1, stride1, reinterpret_cast<gsb::MatchRec *>(matches), counts,
             max_matches);
  return 0;
}
