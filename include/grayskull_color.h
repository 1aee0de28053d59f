/*
 * grayskull_color.h -- the wasm demo's colour conversions over frame batches on the device, in the companion library
 * libgrayskull_color.so (link -lgrayskull_color; it does not need libgrayskull_b200.so).
 *
 * Every other call of this project takes 8-bit gray frames.  The reference defines one colour conversion, in its wasm
 * demo (examples/wasm/grayskull.js:33-45): each webcam frame goes to gray before the pipeline and back to RGBA for
 * display.  These calls are that rule, bit-exact, for frame batches already on the device.
 *
 * This header's name deliberately does not match grayskull_b200*.h: the main library's headers are the set whose
 * declarations libgrayskull_b200.so exports, and these calls live in their own library.
 *
 * Conventions are grayskull_b200.h's: DEVICE pointers, n dense frames of w x h pixels back to back (no row pitch),
 * work enqueued on `s` and not synchronised, 0 or a cudaError_t returned (gs_b200_color_last_error() gives the text),
 * 64-bit offsets; batches above 65535 frames and frames taller than 65535 row tiles run as any other.  A missing
 * pointer or an empty frame aborts with the reference's "Assertion failed: ..." message; n == 0 returns 0 and does
 * nothing.  The calls allocate nothing and synchronise nothing, so they can be captured into a CUDA graph.
 *
 * The rule's quirks, which these calls keep: gray is not floor((299 r + 587 g + 114 b) / 1000) but one below it for
 * 3464 of the 2^24 triples, all with 299 r + 587 g + 114 b a multiple of 1000; among them are 65 pure grays (v, v, v),
 * such as (1,1,1) -> 0 and (8,8,8) -> 7, so gray -> RGBA -> gray changes those 65 levels.
 */
#ifndef GRAYSKULL_COLOR_H
#define GRAYSKULL_COLOR_H

#include "grayskull_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* examples/wasm/grayskull.js:33-38 over n frames of `channels`-byte pixels (3: R,G,B; 4: R,G,B,A with A ignored):
 * dst[i] = (uint8_t) floor(((0.299 * R) + (0.587 * G)) + (0.114 * B)), IEEE double, each operation rounded
 * to nearest, nothing fused.  channels other than 3 or 4, or dst overlapping src: cudaErrorInvalidValue. */
int gs_b200_rgb_to_gray_batch(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n,
                              unsigned channels, gs_b200_stream s);

/* examples/wasm/grayskull.js:40-45: dst pixel i = (g, g, g, 255), g = src[i]; overlap: cudaErrorInvalidValue */
int gs_b200_gray_to_rgba_batch(uint8_t *dst, const uint8_t *src, unsigned w, unsigned h, unsigned n,
                               gs_b200_stream s);

/* the text of the calling thread's last error of this library */
const char *gs_b200_color_last_error(void);

#ifdef __cplusplus
}
#endif

#endif /* GRAYSKULL_COLOR_H */
