/*
 * msda_flatten.h -- C ABI of the encoder's input preparation (DESIGN.md section 3.16; deformable_transformer_dino.py:181-201),
 * exported by libmsda_b200.so next to the functions of msda_b200.h and following its conventions: device pointers on the
 * current device; return 0, a positive cudaError_t, or a negative MSDA_E_* of msda_b200.h (msda_strerror renders it); a
 * caller-provided workspace whose size the matching *_workspace function gives; the stream last.  The level tables
 * (pointer arrays, H, W) are HOST arrays of L entries, copied into the kernels' arguments: nothing is allocated, nothing
 * synchronises with the host, so every call can be captured into a CUDA graph.  No float atomics: every result has the
 * same bits on every run.
 *
 * Sizes: L levels (1 .. 8), N images (1 .. 65535), C channels (C % 4 == 0, 4 <= C <= 1024), H[l], W[l] >= 1,
 * S = sum of H[l] * W[l].  Offsets are 64-bit.
 *
 * msda_flatten_levels_forward_f32: per level src[l], pos[l] [N, C, H_l, W_l] fp32 (NCHW), mask[l] [N, H_l, W_l] uint8;
 *   level_embed [L, C].  src_flat [N, S, C] = the levels' positions in order, each a row of C channels;
 *   pos_flat [N, S, C] = the same of pos + level_embed[l]; mask_flat [N, S] uint8.  One launch.
 * msda_flatten_levels_workspace: the workspace bytes of the backward with grad_level_embed (0 bytes are needed without).
 * msda_flatten_levels_backward_f32: the transpose back.  grad_src[l] [N, C, H_l, W_l] from grad_src_flat [N, S, C];
 *   grad_pos[l] from grad_pos_flat; grad_level_embed [L, C] = the sum over images and level-l positions of grad_pos_flat,
 *   as partial sums over fixed 32-position tiles in the workspace, then summed in a fixed order.  The grad_src array,
 *   the grad_pos array and grad_level_embed may each be NULL (that output is not written); grad_src_flat is read when
 *   grad_src is given, grad_pos_flat when grad_pos or grad_level_embed is.  At most two launches.
 *
 * Limits: sizes out of range, a NULL required pointer (array or entry), a misaligned (16-byte) [N, S, C] operand or
 * level_embed, or too small a workspace give MSDA_E_BADARG.
 */
#ifndef MSDA_FLATTEN_H_
#define MSDA_FLATTEN_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

int msda_flatten_levels_forward_f32(const float *const *src, const float *const *pos, const uint8_t *const *mask,
                                    const int *H, const int *W, int L, int N, int C, const float *level_embed,
                                    float *src_flat, float *pos_flat, uint8_t *mask_flat, void *stream);
int msda_flatten_levels_workspace(const int *H, const int *W, int L, int N, int C, int64_t *bytes);
int msda_flatten_levels_backward_f32(const float *grad_src_flat, const float *grad_pos_flat, const int *H, const int *W,
                                     int L, int N, int C, float *const *grad_src, float *const *grad_pos,
                                     float *grad_level_embed, void *workspace, int64_t workspace_bytes, void *stream);

#ifdef __cplusplus
}
#endif

#endif  /* MSDA_FLATTEN_H_ */
