/*
 * msda_twostage.h -- C ABI of the two-stage query selection (DESIGN.md section 3.15, row f-3;
 * deformable_transformer_dino.py:153-161,216-224), exported by libmsda_b200.so next to the functions of msda_b200.h and
 * following its conventions: device pointers on the current device, dense row-major, 16-byte aligned where a row is
 * read as float4; return 0, a positive cudaError_t, or a negative MSDA_E_* of msda_b200.h (msda_strerror renders it);
 * a caller-provided workspace whose size the matching *_workspace function gives; the stream last.  Nothing is allocated
 * and nothing synchronises with the host, so every call can be captured into a CUDA graph.  No float atomics: every
 * result has the same bits on every run.
 *
 * Sizes: N images (1 .. 65535), S rows per image (S >= 1), C the model width (must be 256), k proposals (1 <= k <= S).
 *
 * msda_twostage_head_forward_f32: y [N, S, C] = enc_output(memory); keep [N, S] uint8 (0: padded or invalid proposal);
 *   b_e [C] enc_output.bias; gamma, beta [C] enc_output_norm; u [N, C], c [N] the class head as an affine map per image.
 *   Per row: v = keep ? y : b_e (Linear of a zeroed row); om = LayerNorm(v; eps, gamma, beta) [N, S, C];
 *   mean, rstd [N, S]; logit [N, S] = om . u[n] + c[n], clamped to [-5e4, 5e4] when clamp != 0 (NaN stays NaN).
 * msda_twostage_head_backward_f32: grad_om [N, S, C], grad_logit [N, S] and the forward's inputs and mean / rstd.
 *   g = grad_om + grad_logit' * u[n], grad_logit' = 0 where clamp != 0 and the unclamped logit is outside [-5e4, 5e4];
 *   grad_y [N, S, C] = the LayerNorm backward of g on kept rows, 0 on dropped rows; grad_b_e [C] = its sum over the
 *   dropped rows; grad_gamma, grad_beta [C]; grad_u [N, C] = sum over image n of grad_logit' * om; grad_c [N] = sum of
 *   grad_logit'.  Partial sums over fixed 64-row tiles, then summed in a fixed order.
 * msda_twostage_select_forward_f32: logit [N, S], box [N, S, 4] = bbox_embed(om), proposals [N, S, 4] (+inf on dropped
 *   rows).  coord_unact [N, S, 4] = box + proposals; topk_index [N, k] int64 = the rows of the k largest logits of each
 *   image, by descending logit, ties by ascending row (torch.sort(descending=True, stable=True)), every NaN first;
 *   reference_points [N, k, 4] = sigmoid(coord_unact[topk_index]).
 * msda_twostage_select_backward_f32: grad_coord [N, S, 4] holds the incoming gradient of coord_unact on entry; on return
 *   grad_coord[n, topk_index[n, j]] += grad_ref[n, j] * (1 - reference_points[n, j]) * reference_points[n, j].
 *
 * Limits: C != 256, k < 1, k > S, N or S out of range, a NULL pointer, a misaligned float4 operand or too small a
 * workspace give MSDA_E_BADARG.
 */
#ifndef MSDA_TWOSTAGE_H_
#define MSDA_TWOSTAGE_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

int msda_twostage_head_forward_f32(const float *y, const uint8_t *keep, const float *b_e, const float *gamma,
                                   const float *beta, const float *u, const float *c, int N, int S, int C, float eps,
                                   int clamp, float *om, float *logit, float *mean, float *rstd, void *stream);
int msda_twostage_head_workspace(int N, int S, int C, int64_t *bytes);
int msda_twostage_head_backward_f32(const float *grad_om, const float *grad_logit, const float *y, const uint8_t *keep,
                                    const float *b_e, const float *gamma, const float *beta, const float *u,
                                    const float *c, const float *mean, const float *rstd, int N, int S, int C, int clamp,
                                    float *grad_y, float *grad_b_e, float *grad_gamma, float *grad_beta, float *grad_u,
                                    float *grad_c, void *workspace, int64_t workspace_bytes, void *stream);
int msda_twostage_select_workspace(int N, int S, int k, int64_t *bytes);
int msda_twostage_select_forward_f32(const float *logit, const float *box, const float *proposals, int N, int S, int k,
                                     float *coord_unact, float *reference_points, int64_t *topk_index, void *workspace,
                                     int64_t workspace_bytes, void *stream);
int msda_twostage_select_backward_f32(const float *grad_ref, const float *reference_points, const int64_t *topk_index,
                                      int N, int S, int k, float *grad_coord, void *stream);

#ifdef __cplusplus
}
#endif

#endif  /* MSDA_TWOSTAGE_H_ */
