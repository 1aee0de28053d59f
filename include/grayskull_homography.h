/*
 * grayskull_homography.h -- where an ORB template lies in each frame of a batch, on the device, in the companion
 * library libgrayskull_homography.so (link -lgrayskull_homography; it does not need libgrayskull_b200.so).  It reads
 * the keypoint and match lists gs_b200_orb_pyramid_batch / gs_b200_match_orb_batch write, fits a RANSAC homography per
 * frame, and gives the template's outline in the scene in the corner layout gs_b200_perspective_correct_batch(...,
 * per_frame = 1) reads; the inlier records keep the match layout, so gs_b200_draw_matches_batch draws them unchanged.
 *
 * This header's name deliberately does not match grayskull_b200*.h: the main library's headers are the set whose
 * declarations libgrayskull_b200.so exports, and these calls live in their own library.
 *
 * Conventions are grayskull_group.h's: DEVICE pointers, work enqueued on `s` and not synchronised, 0 or a cudaError_t
 * returned (gs_b200_homography_last_error() gives the text), 64-bit offsets; batches above 65535 frames run as any
 * other.  A missing pointer aborts with the reference's "Assertion failed: ..." message; n == 0 returns 0 and does
 * nothing.  The calls allocate nothing and synchronise nothing, so they can be captured into a CUDA graph.
 */
#ifndef GRAYSKULL_HOMOGRAPHY_H
#define GRAYSKULL_HOMOGRAPHY_H

#include "grayskull_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* A homography per frame from its matches, by RANSAC with a refit.  Frame f's template keypoints start at
 * kps1 + f * stride1 (c1 = min(n1[f], stride1) of them used), its scene keypoints at kps2 + f * stride2 (c2 =
 * min(n2[f], stride2)), its records at matches + f * mstride (c = min(mcounts[f], mstride)).  Every double operation
 * below is one IEEE double operation, rounded to nearest even, in the order written, without FMA:
 *   1. record i < c is usable when idx1 < c1, idx2 < c2 and all four coordinates are < 2^20; the usable records in
 *      record order are the m correspondences (x, y) -> (X, Y) (template point, scene point).  m < 4: H = 0 (all
 *      nine), inliers[f] = 0, nothing else;
 *   2. hypothesis k (0 <= k < hypotheses) draws 4 distinct indices by Floyd's algorithm: for j = 0..3, J = m - 4 + j,
 *      z = splitmix64's finaliser of (seed + 0x9E3779B97F4A7C15 * ((f << 18) | (k << 2) | j)) mod 2^64, t = ((z >> 32)
 *      * (J + 1)) >> 32; it takes t, or J when t is taken.  The four are sorted ascending;
 *   3. the sample is rejected when, for any of its triples (0,1,2), (0,1,3), (0,2,3), (1,2,3), the 64-bit integer
 *      orientation (q - p) x (r - p) of the template points or of the scene points is 0, or the two differ in sign;
 *   4. the solve of a set of m' correspondences: centres cx = floor(sum x / m'), likewise cy, CX, CY; centred a = x -
 *      cx, b = y - cy, A = X - CX, B = Y - CY; kt = bit length of max |a|, |b| and ks of max |A|, |B| (0 for 0).  With
 *      R = A^2 + B^2 the exact integer sums
 *        S = [[Saa, Sab, Sa, 0, 0, 0, -SaaA, -SabA], [., Sbb, Sb, 0, 0, 0, -SabA, -SbbA], [., ., m', 0, 0, 0, -SaA,
 *             -SbA], [., ., ., Saa, Sab, Sa, -SaaB, -SabB], [., ., ., ., Sbb, Sb, -SabB, -SbbB], [., ., ., ., ., m',
 *             -SaB, -SbB], [., ., ., ., ., ., SaaR, SabR], [., ., ., ., ., ., ., SbbR]]  (upper triangle)
 *        V = [SaA, SbA, SA, SaB, SbB, SB, -SaR, -SbR]
 *      (the normal equations of the inhomogeneous DLT, h33 = 1, in integer centred coordinates) are each rounded once
 *      to the nearest double, ties to even, and scaled exactly: N[p][q] = S[p][q] * 2^-(E[p] + E[q]), r[p] = V[p] *
 *      2^-(E[p] + ks), E = (kt, kt, 0, kt, kt, 0, kt + ks, kt + ks).  Cholesky of N in place, columns j = 0..7: d =
 *      N[j][j] - L[j][0]^2 - ... - L[j][j-1]^2 (left to right), invalid unless 0 < d < inf, L[j][j] = sqrt(d); then
 *      for i = j+1..7, L[i][j] = (N[i][j] - L[i][0] L[j][0] - ... - L[i][j-1] L[j][j-1]) / L[j][j].  Then y[i] = (r[i]
 *      - L[i][0] y[0] - ... - L[i][i-1] y[i-1]) / L[i][i] for i = 0..7, and h[i] = (y[i] - L[i+1][i] h[i+1] - ... -
 *      L[7][i] h[7]) / L[i][i] for i = 7..0.  With (p, q, c) = (h0, h1, h2), (h3, h4, h5), (h6, h7, 1.0) for rows 0, 1,
 *      2: P = p * 2^-kt, Q = q * 2^-kt, G = (P, Q, c - ((P * cx) + (Q * cy))); H row 0 = G0[j] * 2^ks + CX * G2[j], row
 *      1 = G1[j] * 2^ks + CY * G2[j], row 2 = G2[j]; invalid when H[8] is 0 or not finite; every entry is divided by
 *      H[8] (so H[8] = 1); invalid when any entry is not finite;
 *   5. correspondence (x, y) -> (X, Y) is an inlier of H when w > 0 and (du * du) + (dv * dv) <= t2 * (w * w), with u =
 *      ((H0 * x) + (H1 * y)) + H2, v = ((H3 * x) + (H4 * y)) + H5, w = ((H6 * x) + (H7 * y)) + H8, du = u - (X * w), dv =
 *      v - (Y * w), t2 = threshold * threshold.  A rejected sample or an invalid solve is an invalid hypothesis; the
 *      best hypothesis is the valid one with the most inliers, the lowest k on ties;
 *   6. with c_b inliers of the best hypothesis: when c_b >= 4, the solve of rule 4 over them; the refit is kept when it
 *      is valid and has at least c_b inliers, otherwise the best hypothesis is.  H[f * 9 ..] gets it, row-major,
 *      inliers[f] its inlier count, and inlier_matches + f * mstride (may be NULL) the records of its inliers in
 *      record order.  No valid hypothesis: H = 0, inliers[f] = 0.  Slots past the count are not written.
 * hypotheses outside 1..65536, or a threshold that is not finite and > 0, returns cudaErrorInvalidValue before anything
 * is enqueued. */
int gs_b200_find_homography_batch(const struct gs_keypoint *kps1, const unsigned *n1, unsigned stride1,
                                  const struct gs_keypoint *kps2, const unsigned *n2, unsigned stride2,
                                  const struct gs_match *matches, const unsigned *mcounts, unsigned mstride,
                                  unsigned n, unsigned hypotheses, unsigned long long seed, double threshold,
                                  double *H, unsigned *inliers, struct gs_match *inlier_matches, gs_b200_stream s);

/* The template's outline in each frame (rule 7): frame f is found when H[f * 9 ..] is not all zero, inliers[f] >=
 * min_inliers and the four template corners (0, 0), (tw-1, 0), (tw-1, th-1), (0, th-1) all project with w > 0 and
 * u / w, v / w not NaN (u, v, w as in rule 5).  Corner q is then (rint(u / w), rint(v / w)), half to even, clamped to
 * [0, sw-1] x [0, sh-1], at corners[f * 4 + q] (top-left, top-right, bottom-right, bottom-left), and found[f] = 1; a
 * frame not found gets four (0, 0) corners and found[f] = 0.  min_inliers < 4, or tw, th, sw or sh 0, returns
 * cudaErrorInvalidValue before anything is enqueued. */
int gs_b200_homography_quads_batch(const double *H, const unsigned *inliers, unsigned n, unsigned min_inliers,
                                   unsigned tw, unsigned th, unsigned sw, unsigned sh, struct gs_point *corners,
                                   uint8_t *found, gs_b200_stream s);

/* the text of the calling thread's last error of this library */
const char *gs_b200_homography_last_error(void);

#ifdef __cplusplus
}
#endif

#endif /* GRAYSKULL_HOMOGRAPHY_H */
