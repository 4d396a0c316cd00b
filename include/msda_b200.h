/*
 * msda_b200.h -- C ABI of the sm_90a (H100) multi-scale deformable attention library (libmsda_b200.so; the name is
 * historical).
 *
 * This is the drop-in boundary for the reference's native module `MultiScaleDeformableAttention`
 * (projects/UNINEXT/uninext/models/deformable_detr/ops/src/vision.cpp:13-16), whose two functions
 *     ms_deform_attn_forward  (ops/src/ms_deform_attn.h:19-39  -> ops/src/cuda/ms_deform_attn_cuda.cu:20-80)
 *     ms_deform_attn_backward (ops/src/ms_deform_attn.h:41-62  -> ops/src/cuda/ms_deform_attn_cuda.cu:83-153)
 * take ATen tensors. Here the same work is exposed with plain pointers and sizes; no torch / ATen type crosses
 * this interface. The reference-side binding (a 40-line pybind or ctypes shim) is shown in INTEGRATION.md and
 * shipped as uninext_b200/dropin/MultiScaleDeformableAttention.py.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer on the current CUDA device, dense row-major.  16-byte aligned tensors (what
 *     any allocator returns) take the tiled / slab sm_90a kernels; a merely element-aligned pointer (a contiguous view
 *     with a storage offset, which the reference accepts too) is served by the generic kernels:
 *       value              [N, S, M, D]          (reference: ms_deform_attn_cuda.cu:40-43)
 *       spatial_shapes     [L, 2] int64 (H_l,W_l)  -- read on the device, no host sync (cu:67)
 *       level_start_index  [L]    int64            (cu:68)
 *       sampling_loc       [N, Lq, M, L, P, 2]   last dim (x, y) in [0,1] of the level map (cu:69)
 *       attn_weight        [N, Lq, M, L, P]      (cu:70)
 *       out / grad_out     [N, Lq, M*D]          (cu:54,77)
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream). Calls are asynchronous with
 *     respect to the host, stateless and re-entrant (reference: at::cuda::getCurrentCUDAStream(), cu:65,135).
 *   - return value: 0 on success; a positive cudaError_t if a CUDA call or kernel launch failed (the reference
 *     only printf()s these, ms_deform_im2col_cuda.cuh:948-952,1321-1325 -- here they are returned);
 *     a negative MSDA_E_* for argument errors. msda_strerror() renders either.
 *   - there is no im2col_step: the reference chunks the batch only to bound its int32 indexing and temporary
 *     sizes (cu:50-52,61-75); these kernels use 64-bit offsets and take the whole batch in one launch. The
 *     Python shim still validates `batch % min(batch, im2col_step) == 0` like the reference (cu:52).
 *   - the *_bf16 entry points are new (the reference dispatches float/double only, cu:64,134): value, out and
 *     grad_out are bfloat16 bit patterns (uint16_t), sampling_loc / attn_weight and their gradients stay fp32,
 *     accumulation is fp32.
 *   - backward: grad_value is zero-filled by the callee (the reference's at::zeros_like, cu:121); grad_sampling_loc
 *     and grad_attn_weight are fully overwritten.  msda_backward_* accumulate grad_value with atomics, like the
 *     reference: its summation order, hence its last bits, vary from run to run.  msda_backward_det_* compute the same
 *     gradients with a fixed summation order (the contract below), at the price of a caller-provided workspace.
 */
#ifndef MSDA_B200_H_
#define MSDA_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MSDA_ABI_VERSION 8   /* 4: MSDA_KNOB_REGION_BWD; 5: msda_backward_det_*; 6: msda_vlfuse_*; 7: msda_vlfuse_*_tf32;
                                8: msda_vlfuse_*_bf16 */

#define MSDA_E_BADARG   (-1)   /* null pointer, non-positive dimension, unknown knob                  */
#define MSDA_E_TOOLARGE (-2)   /* a dimension product exceeds what the kernels index (see msda_b200.h) */
#define MSDA_E_NODEVICE (-3)   /* no usable CUDA device is current                                     */

int msda_abi_version(void);
const char *msda_strerror(int code);

/* Which kernel family a (dtype, D, L, P) problem is routed to: 1 = tiled sm_90a fast path, 0 = generic.
 * dtype_bytes: 2 (bf16), 4 (fp32), 8 (fp64). Used by the tests to prove the fast path is the one exercised. */
int msda_uses_fast_path(int dtype_bytes, int D, int L, int P);

/* Number of kernel launches (memsets excluded) this process has issued through this library. */
uint64_t msda_launch_count(void);

/* Kernel-selection knobs (process-wide; initial values come from the environment variables of the same name with an
 * MSDA_ prefix, e.g. MSDA_SLAB=0).  They never change results, only which kernel computes them; the tests use
 * them to run every kernel family on small shapes, the tools to sweep them.  Returns the previous value, or
 * MSDA_E_BADARG for an unknown knob.  value == MSDA_KNOB_QUERY reads without writing.
 *   MSDA_KNOB_SLAB          1 = slab-ordered kernels (msda_slab.cuh) whenever D == 32 and L*P <= 16; 2 = tiled forward +
 *                           backward with the coarse levels accumulated by dedicated consumer warps in a shared-memory
 *                           window (msda_tmem.cuh); -1 (auto) and
 *                           0 = tiled kernels
 *   MSDA_KNOB_BWD_WIN_ROWS  shared-memory window of the slab backward in rows of 128 B (-1 = all that fits)
 *   MSDA_KNOB_BWD_LIST_CAP  entries per row-class list of the slab backward (even, >= 8)
 *   MSDA_KNOB_FWD_SLAB_CTAS resident CTAs per SM of the slab forward (1 or 2)
 *   MSDA_KNOB_F32_VEC8_FWD / _BWD   lane shape of the fp32 tiled kernels: 1 = 4 lanes x 32 B per row, 0 = 8 lanes x 16 B
 *   MSDA_KNOB_BF16_FINE_ROWS        msda_backward_bf16 with a bf16 result: levels of at least this many rows accumulate
 *                                   grad_value directly in bf16 (packed 8-byte reds); the others in fp32.  0 = all fp32.
 *                                   (changes results within the 1e-2 bf16 tolerance, see DESIGN.md.)
 *   MSDA_KNOB_BF16_PACKED_FWD       bf16 forward (D = 32 / 64, large launches): blend the 4 corners of a tap in packed bf16 and
 *                                   accumulate taps in fp32 (~3 extra bf16 roundings per tap; also changes results slightly).
 *   MSDA_KNOB_ZERO_FILL             how msda_backward_* zero-fills grad_value (results identical): 0 = cudaMemsetAsync,
 *                                   1 = msda_zero_fill kernel (16-byte stores, one wave), 2 = the same kernel launched as the
 *                                   programmatic-dependent-launch primary of the tiled backward kernel, whose prologue then
 *                                   overlaps the fill (not while the stream is being captured into a CUDA graph).  Default 2.
 *   MSDA_KNOB_REGION_BWD            fp32 backward of encoder self-attention (D = 32, L*P <= 16, Lq == S, large launches):
 *                                   -1 (auto, default) = msda_bwd_region, which sums grad_value per spatial region in shared
 *                                   memory before it reaches L2 (msda_region.cuh); 0 = msda_bwd_tiled. */
#define MSDA_KNOB_SLAB          0
#define MSDA_KNOB_BWD_WIN_ROWS  1
#define MSDA_KNOB_BWD_LIST_CAP  2
#define MSDA_KNOB_FWD_SLAB_CTAS 3
#define MSDA_KNOB_F32_VEC8_FWD  4   /* fp32 tiled forward: 8 channels per lane (2 x 16 B), D in {32, 64}; 0 / 1      */
#define MSDA_KNOB_F32_VEC8_BWD  5   /* fp32 tiled backward: same lane shape; 0 / 1                                     */
#define MSDA_KNOB_BF16_FINE_ROWS 6  /* bf16 backward: levels with H*W >= this accumulate grad_value in bf16; 0 = off */
#define MSDA_KNOB_BF16_PACKED_FWD 7 /* bf16 forward: corners of a tap blended in packed bf16 (HFMA2); 0 / 1            */
#define MSDA_KNOB_ZERO_FILL     8   /* grad_value zero-fill of the backward: 0 cudaMemsetAsync, 1 own kernel, 2 own kernel
                                       as the PDL primary of the tiled backward kernel (prologue overlaps the fill)   */
#define MSDA_KNOB_REGION_BWD    9   /* fp32 encoder backward: -1 auto = region kernel, 0 = tiled kernel                */
#define MSDA_KNOB_COUNT         10
#define MSDA_KNOB_QUERY         (-1000000)
int msda_set_knob(int knob, int value);

/* ---- forward: replaces ms_deform_attn_cuda_forward (ms_deform_attn_cuda.cu:20-80) ---- */
int msda_forward_f32(const float *value, const int64_t *spatial_shapes, const int64_t *level_start_index,
                     const float *sampling_loc, const float *attn_weight,
                     int N, int S, int M, int D, int L, int Lq, int P,
                     float *out, void *stream);
int msda_forward_f64(const double *value, const int64_t *spatial_shapes, const int64_t *level_start_index,
                     const double *sampling_loc, const double *attn_weight,
                     int N, int S, int M, int D, int L, int Lq, int P,
                     double *out, void *stream);
int msda_forward_bf16(const uint16_t *value, const int64_t *spatial_shapes, const int64_t *level_start_index,
                      const float *sampling_loc, const float *attn_weight,
                      int N, int S, int M, int D, int L, int Lq, int P,
                      uint16_t *out, void *stream);

/* ---- backward: replaces ms_deform_attn_cuda_backward (ms_deform_attn_cuda.cu:83-153) ---- */
int msda_backward_f32(const float *grad_out, const float *value,
                      const int64_t *spatial_shapes, const int64_t *level_start_index,
                      const float *sampling_loc, const float *attn_weight,
                      int N, int S, int M, int D, int L, int Lq, int P,
                      float *grad_value, float *grad_sampling_loc, float *grad_attn_weight, void *stream);
int msda_backward_f64(const double *grad_out, const double *value,
                      const int64_t *spatial_shapes, const int64_t *level_start_index,
                      const double *sampling_loc, const double *attn_weight,
                      int N, int S, int M, int D, int L, int Lq, int P,
                      double *grad_value, double *grad_sampling_loc, double *grad_attn_weight, void *stream);
/* bf16 backward accumulates grad_value in fp32: `grad_value_f32` [N,S,M,D] fp32 is the accumulator (zero-filled by
 * the callee) and `grad_value` receives its bf16 rounding. Pass grad_value == NULL to keep only the fp32 result.
 * With MSDA_KNOB_BF16_FINE_ROWS > 0 and grad_value != NULL the big ("fine") levels are accumulated directly in
 * `grad_value` and only the rows of the coarse levels of `grad_value_f32` are used (as scratch). */
int msda_backward_bf16(const uint16_t *grad_out, const uint16_t *value,
                       const int64_t *spatial_shapes, const int64_t *level_start_index,
                       const float *sampling_loc, const float *attn_weight,
                       int N, int S, int M, int D, int L, int Lq, int P,
                       float *grad_value_f32, uint16_t *grad_value,
                       float *grad_sampling_loc, float *grad_attn_weight, void *stream);

/* ---- deterministic backward (DESIGN.md section 3.10) ----------------------------------------------------------------
 * Same arguments as msda_backward_* plus a device workspace of `workspace_bytes` bytes (before `stream`).
 * The contract: grad_value is bit-for-bit what the CPU oracle (oracle/) computes, whatever the launch
 * geometry, SM count, stream, CUDA graph or chunking:
 *   - entries: every tap (b, q, m, l, p) passing the window test (h_im > -1 && w_im > -1 && h_im < H && w_im < W)
 *     contributes, for every corner k inside the map (weight zero included), to row (b, m, r_k);
 *   - order: within one (b, m, row), contributions are added in ascending e = ((q*M + m)*L*P + l*P + p)*4 + k;
 *   - rounding: h_im = fl(fl(y*H) - 0.5), lh = h_im - floor(h_im), hh = fl(1 - lh) (w likewise),
 *     cw = {hh*hw, hh*lw, lh*hw, lh*lw}; contribution fl(cw_k * fl(g_c * a)); acc = fl(acc + contribution) from +0;
 *     fp64 in double, fp32 and bf16 in float;
 *   - bf16: grad_out is widened exactly to fp32; the fp32 accumulator `grad_value_f32` follows the rules above and
 *     `grad_value` (may be NULL) receives its bf16 rounding once.
 * grad_sampling_loc and grad_attn_weight come from the kernel msda_backward_* would pick at default knob settings, with
 * its grad_value atomics compiled out: they are bit-identical to msda_backward_*'s.  The knobs are ignored.
 * grad_value is zero-filled by the callee.  The work runs in chunks of whole queries of one batch element, the largest
 * that fit the workspace; nothing is allocated, so the call can be captured into a CUDA graph.  Returns MSDA_E_BADARG
 * if one query does not fit, MSDA_E_TOOLARGE if M*S + 1 > 2^32 or one query's M*L*P*4 entries exceed 2^32 - 1.
 * msda_backward_det_workspace: bytes needed for chunks of `chunk_queries` queries (>= 1; clipped to Lq); dtype_bytes
 *   2, 4 or 8.  It asks CUB for the sort's temporary storage, which needs a current CUDA device. */
int msda_backward_det_workspace(int dtype_bytes, int N, int S, int M, int D, int L, int Lq, int P, int chunk_queries,
                                int64_t *bytes);
int msda_backward_det_f32(const float *grad_out, const float *value,
                          const int64_t *spatial_shapes, const int64_t *level_start_index,
                          const float *sampling_loc, const float *attn_weight,
                          int N, int S, int M, int D, int L, int Lq, int P,
                          float *grad_value, float *grad_sampling_loc, float *grad_attn_weight,
                          void *workspace, int64_t workspace_bytes, void *stream);
int msda_backward_det_f64(const double *grad_out, const double *value,
                          const int64_t *spatial_shapes, const int64_t *level_start_index,
                          const double *sampling_loc, const double *attn_weight,
                          int N, int S, int M, int D, int L, int Lq, int P,
                          double *grad_value, double *grad_sampling_loc, double *grad_attn_weight,
                          void *workspace, int64_t workspace_bytes, void *stream);
int msda_backward_det_bf16(const uint16_t *grad_out, const uint16_t *value,
                           const int64_t *spatial_shapes, const int64_t *level_start_index,
                           const float *sampling_loc, const float *attn_weight,
                           int N, int S, int M, int D, int L, int Lq, int P,
                           float *grad_value_f32, uint16_t *grad_value,
                           float *grad_sampling_loc, float *grad_attn_weight,
                           void *workspace, int64_t workspace_bytes, void *stream);

/* ---- callers of the op (SURVEY.md section 8 rows f-1 / f-2): one-pass fp32 kernels around the cuBLAS GEMMs --------
 * msda_prologue_forward_f32: raw projection -> attention softmax + sampling locations in the op's layouts.
 *   Replaces the five elementwise passes of ops/modules/ms_deform_attn.py:99-112.
 *   proj [R, M*L*P*3]: columns [0, M*L*P*2) = sampling offsets ordered (m,l,p,xy) (ms_deform_attn.py:99),
 *                      columns [M*L*P*2, M*L*P*3) = attention logits ordered (m, l*p) (ms_deform_attn.py:100);
 *   ref  [R, L, refdim] reference points (refdim 2) or boxes (refdim 4) (ms_deform_attn.py:103-109); R = N*Lq;
 *   loc  [R, M, L, P, 2], attn [R, M, L, P] outputs.  L*P <= 32.
 * msda_prologue_backward_f32: gradient of the raw projection from grad_loc / grad_attn (reference points are
 *   treated as constants).
 * msda_colsum_f32: out[c] = sum_r x[r,c] (bias gradients); cols % 4 == 0; `out` is zero-filled by the callee.
 * msda_add_layernorm_forward_f32 / msda_layernorm_backward_f32: y = LayerNorm(a + b) over the last dimension
 *   (deformable_transformer.py:354-356,359); cols in {128, 256, 384, 512}; b and z may be NULL (z = a + b is needed by
 *   the backward when b != NULL); dgamma / dbeta are zero-filled by the callee. */
int msda_prologue_forward_f32(const float *proj, const float *ref, const int64_t *spatial_shapes,
                              int64_t R, int M, int L, int P, int refdim, float *loc, float *attn, void *stream);
int msda_prologue_backward_f32(const float *grad_loc, const float *grad_attn, const float *attn, const float *ref,
                               const int64_t *spatial_shapes, int64_t R, int M, int L, int P, int refdim,
                               float *grad_proj, void *stream);
int msda_colsum_f32(const float *x, int64_t rows, int cols, float *out, void *stream);
/* ReLU backward fused with the bias gradient of the Linear before it (FFN linear1): g2 = g where y > 0 else 0;
 * colsum[c] = sum_r g2[r, c] (zero-filled by the callee).  cols % 4 == 0. */
int msda_relu_backward_colsum_f32(const float *g, const float *y, int64_t rows, int cols, float *g2, float *colsum, void *stream);
int msda_add_layernorm_forward_f32(const float *a, const float *b, const float *gamma, const float *beta,
                                   int64_t rows, int cols, float eps, float *z, float *y, float *mean, float *rstd,
                                   void *stream);
int msda_layernorm_backward_f32(const float *dy, const float *z, const float *gamma, const float *mean,
                                const float *rstd, int64_t rows, int cols, float *dz, float *dgamma, float *dbeta,
                                void *stream);

/* ---- geometry feeding the op (SURVEY.md section 8 f-3; deformable_transformer_dino.py:132-171,289-301,612-646): one launch each
 *   msda_valid_counts:            mask [N, S] bytes (non-zero = padded) -> counts [N, L, 2] int32 = (valid_W, valid_H)  (get_valid_ratio)
 *   msda_encoder_ref_points_f32:  valid_ratios [N, L, 2] -> reference points [N, S, L, 2]                          (get_reference_points)
 *   msda_encoder_proposals_f32:   mask + counts -> proposals [N, S, 4] in logit space (+inf = dropped), keep [N, S] bytes
 *                                 (the geometry half of gen_encoder_output_proposals)
 *   msda_sine_pos_embed_forward/backward_f32: pos [R, n] -> [R, n * F]                                              (get_sine_pos_embed) */
int msda_valid_counts(const uint8_t *mask, const int64_t *spatial_shapes, const int64_t *level_start_index, int N, int S, int L,
                      int32_t *counts, void *stream);
int msda_encoder_ref_points_f32(const float *valid_ratios, const int64_t *spatial_shapes, const int64_t *level_start_index, int N,
                                int S, int L, float *ref, void *stream);
int msda_encoder_proposals_f32(const uint8_t *mask, const int32_t *counts, const int64_t *spatial_shapes,
                               const int64_t *level_start_index, int N, int S, int L, float base_scale, float *proposals,
                               uint8_t *keep, void *stream);
int msda_sine_pos_embed_forward_f32(const float *pos, int64_t R, int n, int F, float temperature, int exchange_xy, float *out,
                                    void *stream);
int msda_sine_pos_embed_backward_f32(const float *pos, const float *grad_out, int64_t R, int n, int F, float temperature,
                                     int exchange_xy, float *grad_pos, void *stream);

/* ---- CondInst dynamic mask head (SURVEY.md section 8 f-4; uninext/models/ddetrs.py:488-598, 895-958) ----------------
 * msda_condinst_forward_f32: logits[i, y, x] = MLP_i(rel_x, rel_y, feats[b(i), :, y, x]) for every selected instance i --
 *   the reference's three grouped 1x1 convolutions (groups = #instances, `mask_heads_forward`) over a materialised
 *   [1, I*10, H, W] input, fused into one pass that materialises nothing.
 *     feats [N, 8, H, W]; params [I, 169] laid out as parse_dynamic_params expects (w1[8][10] | w2[8][8] | w3[8] | b1 | b2 | b3);
 *     refs [I, 2] reference points in input-image pixels; inst_start [N + 1] int32 (device): instances of image b are
 *     [inst_start[b], inst_start[b+1]); max_inst = largest per-image count (host value, sizes the grid);
 *     stride = mask_feat_stride; rel_coord = 1 prepends (ref - pixel location) as two input channels, 0 feeds zeros;
 *     logits [I, H, W].
 * msda_condinst_backward_f32: grad_feats [N, 8, H, W], grad_params [I, 169] and grad_refs [I, 2] (all zero-filled by the
 *   callee, then accumulated with fp32 reductions: summation order, hence the last bits, vary from run to run).
 * msda_aligned_bilinear_forward/backward_f32: `aligned_bilinear` (ddetrs.py:921-942) on [planes, h, w] -> [planes, f*h, f*w]. */
int msda_condinst_forward_f32(const float *feats, const float *params, const float *refs, const int32_t *inst_start,
                              int N, int H, int W, int I, int max_inst, int stride, int rel_coord, float *logits,
                              void *stream);
int msda_condinst_backward_f32(const float *grad_logits, const float *feats, const float *params, const float *refs,
                               const int32_t *inst_start, int N, int H, int W, int I, int max_inst, int stride,
                               int rel_coord, float *grad_feats, float *grad_params, float *grad_refs, void *stream);
int msda_aligned_bilinear_forward_f32(const float *in, int64_t planes, int h, int w, int factor, float *out, void *stream);
int msda_aligned_bilinear_backward_f32(const float *grad_out, int64_t planes, int h, int w, int factor, float *grad_in,
                                       void *stream);

/* ---- TF32 GEMM for the Linears that bracket the op:  C[M,N] = A[M,K] . W[N,K]^T + bias[N]  (fp32 storage, sm_90 wgmma TF32
 * MMA with fp32 accumulation; TMA-fed).  K % 32 == 0, N % 32 == 0 (N % 64 == 0 above 256), N <= 512.
 * Replaces torch.nn.functional.linear for value_proj / output_proj / the concatenated sampling projection
 * (ops/modules/ms_deform_attn.py:95,99-100,115) when TF32 GEMMs are allowed. bias may be NULL. */
int msda_linear_tf32(const float *A, const float *W, const float *bias, int64_t M, int N, int K, float *C, void *stream);
/* The same GEMM with a fused tail, for N <= 256 (N % 64 == 0; msda_linear_tf32_ws_ok tells):
 *   C = A . W^T + bias;  rows with row_mask[m] != 0 are written as zeros (the `masked_fill(input_padding_mask)` that follows
 *   value_proj, ops/modules/ms_deform_attn.py:96-97);  relu != 0 applies max(., 0) (FFN linear1).  bias / row_mask may be NULL.
 *   A, W, C (and bias) must be 16-byte aligned. */
int msda_linear_tf32_ex(const float *A, const float *W, const float *bias, const uint8_t *row_mask, int64_t M, int N, int K,
                        int relu, float *C, void *stream);
int msda_linear_tf32_ws_ok(int N, int K);

/* ---- fused image-text attention of the early-fusion block (DESIGN.md section 3.11; fuse_helper.py:54-139) ----------
 * Per (b, h): x = clamp(Q K^T) (clamp_min / clamp_max: the clamps at -50000 / 50000), P_v = softmax over T of
 * (x + text_bias[b]), P_l = softmax over S of (x^T - max over S of x^T), O_v = dropout(P_v) Vl, O_l = dropout(P_l) Vv.
 *   q, v_v, out_v      [B, S, H, head_dim]   (q already multiplied by head_dim^-0.5)
 *   k, v_l, out_l      [B, T, H, head_dim]
 *   text_bias          [B, T] fp32 additive mask, as the reference adds it (-9e15 at padding), or NULL
 *   stats              [B*H*(S + T)*2] fp32: per-row and per-column softmax statistics saved for the backward
 *   seed               device int64 scalar keying the dropout masks (counter-based Philox); read only when
 *                      dropout_p > 0.  The same seed gives the same masks in the forward, the backward and
 *                      msda_vlfuse_dropout_mask_f32.
 * Limits: head_dim 128 or 256, 1 <= T <= 256, 0 <= dropout_p < 1; every tensor pointer 16-byte aligned and contiguous.
 * No S x T tensor is stored and no float atomics are used: every output is bit-identical from run to run.  Nothing is
 * allocated and nothing synchronises with the host; the calls can be captured into a CUDA graph.
 * msda_vlfuse_workspace: bytes of `workspace` both calls need for these sizes.
 * msda_vlfuse_backward_f32 writes all four gradients (overwritten, not accumulated).
 * msda_vlfuse_dropout_mask_f32: the keep decisions as 1.0 / 0.0, mask_v [B*H, S, T] (vision), mask_l [B*H, T, S] (text).
 * msda_vlfuse_forward_tf32 / _backward_tf32: the same calls with every S x T x d product on TF32 tensor cores (each
 * operand rounded once to TF32, round to nearest; fp32 accumulation; everything between the products fp32 as above).
 * Same workspace, stats layout, dropout masks, determinism and launch count.  A backward must use the mode of the
 * forward that wrote `stats`.
 * msda_vlfuse_forward_bf16 / _backward_bf16: the same calls on bf16 tensors (uint16_t bit patterns) with every S x T x d
 * product on bf16 tensor cores: P_v, P_l and dS rounded once to bf16 (round to nearest even), fp32 accumulation, every
 * output rounded once to bf16.  text_bias and stats stay fp32.  Same workspace, alignment rule, dropout masks
 * (msda_vlfuse_dropout_mask_f32), determinism and launch count. */
int msda_vlfuse_workspace(int B, int H, int S, int T, int head_dim, int64_t *bytes);
int msda_vlfuse_forward_f32(const float *q, const float *k, const float *v_v, const float *v_l, const float *text_bias,
                            int B, int H, int S, int T, int head_dim, int clamp_min, int clamp_max, float dropout_p,
                            const int64_t *seed, float *out_v, float *out_l, float *stats, void *workspace,
                            int64_t workspace_bytes, void *stream);
int msda_vlfuse_backward_f32(const float *grad_out_v, const float *grad_out_l, const float *q, const float *k,
                             const float *v_v, const float *v_l, const float *text_bias, const float *out_v,
                             const float *out_l, const float *stats, int B, int H, int S, int T, int head_dim,
                             int clamp_min, int clamp_max, float dropout_p, const int64_t *seed, float *grad_q,
                             float *grad_k, float *grad_v_v, float *grad_v_l, void *workspace, int64_t workspace_bytes,
                             void *stream);
int msda_vlfuse_dropout_mask_f32(const int64_t *seed, int B, int H, int S, int T, float dropout_p, float *mask_v,
                                 float *mask_l, void *stream);
int msda_vlfuse_forward_tf32(const float *q, const float *k, const float *v_v, const float *v_l, const float *text_bias,
                             int B, int H, int S, int T, int head_dim, int clamp_min, int clamp_max, float dropout_p,
                             const int64_t *seed, float *out_v, float *out_l, float *stats, void *workspace,
                             int64_t workspace_bytes, void *stream);
int msda_vlfuse_backward_tf32(const float *grad_out_v, const float *grad_out_l, const float *q, const float *k,
                              const float *v_v, const float *v_l, const float *text_bias, const float *out_v,
                              const float *out_l, const float *stats, int B, int H, int S, int T, int head_dim,
                              int clamp_min, int clamp_max, float dropout_p, const int64_t *seed, float *grad_q,
                              float *grad_k, float *grad_v_v, float *grad_v_l, void *workspace, int64_t workspace_bytes,
                              void *stream);
int msda_vlfuse_forward_bf16(const uint16_t *q, const uint16_t *k, const uint16_t *v_v, const uint16_t *v_l,
                             const float *text_bias, int B, int H, int S, int T, int head_dim, int clamp_min, int clamp_max,
                             float dropout_p, const int64_t *seed, uint16_t *out_v, uint16_t *out_l, float *stats,
                             void *workspace, int64_t workspace_bytes, void *stream);
int msda_vlfuse_backward_bf16(const uint16_t *grad_out_v, const uint16_t *grad_out_l, const uint16_t *q,
                              const uint16_t *k, const uint16_t *v_v, const uint16_t *v_l, const float *text_bias,
                              const uint16_t *out_v, const uint16_t *out_l, const float *stats, int B, int H, int S,
                              int T, int head_dim, int clamp_min, int clamp_max, float dropout_p, const int64_t *seed,
                              uint16_t *grad_q, uint16_t *grad_k, uint16_t *grad_v_v, uint16_t *grad_v_l,
                              void *workspace, int64_t workspace_bytes, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* MSDA_B200_H_ */
