/*
 * msda_trackpost.h -- C ABI of the video trackers' per-frame detection selection (DESIGN.md section 3.17;
 * uninext_vid.py:1224-1250 inference_mot, :1380-1415 inference_vis), exported by libmsda_b200.so next to the functions of
 * msda_b200.h and following its conventions: device pointers on the current device; return 0, a positive cudaError_t,
 * or a negative MSDA_E_* of msda_b200.h (msda_strerror renders it); a caller-provided workspace whose size the matching
 * *_workspace function gives; the stream last.  Nothing is allocated, nothing synchronises with the host, so a call can
 * be captured into a CUDA graph.  No float atomics: every result has the same bits on every run.
 *
 * Sizes: B frames (0 .. 65535), Q queries (1 .. 1024), T tokens (1 .. 256), C classes (1 .. 4096), as msda_detpost_f32.
 *
 * msda_trackpost_f32: box_cls [B, Q, T] token logits, box_pred [B, Q, 4] normalised cxcywh, iou_pred [B, Q] or NULL,
 *   the positive map as CSR (class_start [C + 1], tokens [nnz] int32, each token in [0, T)), as msda_detpost_f32.  Per
 *   frame b:
 *     prob[q, c] = sigmoid(mean of class c's tokens) [; sqrt(prob * sigmoid(iou_pred[q]))]; max_score[q], label[q] = the
 *       max and argmax over c (the lowest class on ties);
 *     the candidates are the queries with max_score > score_thres, in ascending query order;
 *     none: the result is the query of the largest max_score (the lowest query on ties), without NMS;
 *     else: torchvision's batched_nms on the candidates (box_cxcywh_to_xyxy of the normalised boxes, offset
 *       label * (m + 1) with m the candidates' largest coordinate, stable descending score order, IoU > nms_iou dropped).
 *   Outputs in keep order, [B, Q] capacity each: scores (max_score), labels (int32, 0-based), query_index (int32),
 *   boxes [B, Q, 4] (16-byte aligned), count [B] >= 1.  Entries past count[b]: score 0, label -1, query_index -1, box 0.
 *   box_format MSDA_TRACKPOST_CXCYWH: the normalised cxcywh boxes unchanged (inference_vis); MSDA_TRACKPOST_XYXY_PIXELS:
 *   the cxcywh box scaled by (W, H, W, H) of ori_sizes[b] = (H, W) (int32 [B, 2]), then box_cxcywh_to_xyxy
 *   (inference_mot's det_bboxes[:, :4]).  ori_sizes is read only for MSDA_TRACKPOST_XYXY_PIXELS and may otherwise be NULL.
 *   Every multiply and add is rounded once (no FMA contraction).  Two launches, whatever B, Q, C and the candidates.
 * msda_trackpost_workspace: the workspace bytes for these sizes (prob and the per-query max / argmax).
 *
 * Limits: sizes out of range, a NULL required pointer, an unknown box_format, misaligned (16-byte) boxes or workspace, or
 * too small a workspace give MSDA_E_BADARG.
 */
#ifndef MSDA_TRACKPOST_H_
#define MSDA_TRACKPOST_H_

#include <stdint.h>

#define MSDA_TRACKPOST_CXCYWH 0
#define MSDA_TRACKPOST_XYXY_PIXELS 1

#ifdef __cplusplus
extern "C" {
#endif

int msda_trackpost_workspace(int B, int Q, int T, int C, int64_t *bytes);
int msda_trackpost_f32(const float *box_cls, const float *box_pred, const float *iou_pred, const int *class_start,
                       const int *tokens, const int *ori_sizes, int B, int Q, int T, int C, float score_thres,
                       float nms_iou, int box_format, float *scores, int *labels, int *query_index, float *boxes,
                       int *count, void *workspace, int64_t workspace_bytes, void *stream);

#ifdef __cplusplus
}
#endif

#endif  /* MSDA_TRACKPOST_H_ */
