/*
 * grayskull_b200_pyramid.h -- ORB features over an image pyramid for frame batches on the device, part of
 * libgrayskull_b200.so (link -lgrayskull_b200).
 *
 * Each frame gets exactly what the reference CLI's multi-scale ORB (examples/nanomagick/nanomagick.c:245-290, the
 * `orb` verb's extract_pyramid_orb_nm) gives it: up to 4 levels made by gs_downsample, gs_orb_extract on each level
 * with a quota of nkps / L keypoints (the last level: nkps minus what the earlier levels of that frame returned), and
 * each level's coordinates multiplied by 1 << level.  Conventions are grayskull_b200.h's: DEVICE pointers, n frames of
 * w x h back to back, work enqueued on `s` and not synchronised, 0 or a cudaError_t returned (gs_b200_last_error()
 * gives the text, gs_b200_launch_count() counts these launches too), 64-bit offsets.  Trigonometry follows
 * gs_b200_set_trig_mode.  As for gs_b200_orb_extract_batch, the first call on a device uploads the BRIEF table and must
 * not be captured into a CUDA graph; a call that would grow its workspace under capture returns
 * cudaErrorStreamCaptureUnsupported.
 *
 * Workspace (per stream, grow-only): keypoint lists of n * (nkps + (L-1) * (nkps / L)) records, the last level's
 * FAST candidates of n * min(4 * nkps, 5000) records (48 bytes each), n * (L + 1) counts, plus what
 * gs_b200_orb_extract_batch takes for levels 0..L-2.  For 1024 frames, nkps 2500, 3 levels: about 0.2 GB of lists and
 * 0.25 GB of candidates.
 */
#ifndef GRAYSKULL_B200_PYRAMID_H
#define GRAYSKULL_B200_PYRAMID_H

#include "grayskull_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Levels that run for a w x h image when `levels` are asked for: min(levels, 4), stopping before a level with
 * w/2 < 32 or h/2 < 32 (halving the previous level's sizes); level 0 always runs when levels >= 1, none when 0. */
unsigned gs_b200_orb_pyramid_levels(unsigned w, unsigned h, unsigned levels);

/* For every frame f: bit for bit extract_pyramid_orb_nm(frame f, kps + f*nkps, nkps, threshold, buffer, levels).
 * L = gs_b200_orb_pyramid_levels(w, h, levels); level l is w_l x h_l, the sizes floor-halved l times.
 *   pyr       receives levels 1..L-1, level by level; level l holds n frames of w_l*h_l bytes back to back (a batch
 *             of the main library).  May be NULL when L <= 1.
 *   scoremap  levels 0..L-1 in the same level-major layout.  As in gs_b200_orb_extract_batch the caller's bytes take
 *             part in each level's NMS, the ring FAST never writes included.  For n == 1, pyr immediately followed by
 *             scoremap is the reference CLI's buffer layout.
 *   kps       n lists of stride nkps, each the level blocks in order; counts[f] is frame f's total and slots past it
 *             are not written.
 * Level l < L-1 gets nkps / L keypoints and is skipped (no FAST, its score map untouched) when that is 0; the last level
 * gets nkps minus the frame's earlier levels, with gs_orb_extract's FAST cap min(4 * quota, 5000) for that quota.
 * nkps == 0 or levels == 0 writes zero counts and nothing else.  Aborts with the reference's assert message style on a
 * missing pointer or an empty frame. */
int gs_b200_orb_pyramid_batch(const uint8_t *src, unsigned w, unsigned h, unsigned n, unsigned levels, uint8_t *pyr,
                              uint8_t *scoremap, struct gs_keypoint *kps, unsigned *counts, unsigned nkps,
                              unsigned threshold, gs_b200_stream s);

#ifdef __cplusplus
}
#endif

#endif /* GRAYSKULL_B200_PYRAMID_H */
