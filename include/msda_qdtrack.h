/*
 * msda_qdtrack.h -- C ABI of the QuasiDense tracker's association step (DESIGN.md section 3.19; models/tracker.py:304-503,
 * QuasiDenseEmbedTracker.match with match_metric "bisoftmax" and with_cats), exported by libmsda_b200.so next to the
 * functions of msda_b200.h and following its conventions: device pointers on the current device; return 0, a positive
 * cudaError_t, or a negative MSDA_E_* of msda_b200.h (msda_strerror renders it); a caller-provided workspace whose size
 * msda_qdtrack_workspace gives; the stream last.  Nothing is allocated and nothing synchronises with the host.  No float
 * atomics.
 *
 * msda_qdtrack_match_f32: one frame.  Row r < n = min(*count, n_cap) (count is read on the device) is boxes[r] ([n_cap, 4]
 *   xyxy fp32), scores[r] ([n_cap] fp32), labels[r] ([n_cap] int32) and embeds[rows[r]] ([n_src, dim] fp32).  Per frame:
 *     the rows sorted by score, descending, ties in row order (order[p] = the row at sorted position p);
 *     IoU = mmcv's bbox_overlaps with each operation rounded once: overlap / max(area_a + area_b - overlap, 1e-6f);
 *     duplicate removal: sorted row j is removed when IoU(i, j) > thr_j for any sorted row i < j, removed or not, with
 *       thr_j = nms_backdrop_iou_thr if score_j < obj_score_thr, else nms_class_iou_thr;
 *     the memo: the live tracklets in ascending id order, then with MSDA_QD_BACKDROPS last frame's backdrops in their
 *       row order; matching runs when a tracklet is live.  Score = (softmax over the memo + softmax over the kept rows)
 *       / 2 of the fp32 products of the embeddings, times (row label == column label).  Rows in order take the best
 *       column not yet taken (ties to the lowest): conf > match_score_thr on a tracklet gives the row its id when
 *       score > obj_score_thr (the tracklet is taken), else -2 when conf > nms_conf_thr; a backdrop leaves the row at -1;
 *     rows still at -1 with score > init_score_thr get new ids in row order;
 *     backdrops: rows at -1 with no IoU > nms_backdrop_iou_thr against an earlier kept row; with MSDA_QD_BACKDROPS they
 *       replace last frame's;
 *     memory: a matched tracklet's embedding becomes fp32(1 - memo_momentum) * embed + fp32(memo_momentum) * e, its
 *       label the row's, last_frame = frame_id; a new one starts from e; then the tracklets with frame_id - last_frame
 *       >= memo_tracklet_frames are dropped.
 *   Outputs: order [n_cap] int32 (-1 past n); ids [n_cap] int32 per sorted row (>= 0 a tracklet id, -1 left, -2
 *   suppressed by the nms_conf_thr rule, -3 removed as a duplicate or past n); tracked [n_cap] int32, the rows r with an
 *   id >= 0 in sorted order (-1 after them); tracked_count [1].
 *   State, owned by the caller and zero-filled for an empty tracker: state int32 [MSDA_QD_STATE_INTS(max_tracklets)],
 *   embed [max_tracklets, dim] and backdrop_embed [MSDA_QD_MAX_BACKDROPS, dim] fp32.  state[MSDA_QD_STATE_FLAGS] is a
 *   sticky error word: MSDA_QD_OVERFLOW when a frame would leave more than max_tracklets live tracklets, MSDA_QD_BAD_ROW
 *   when a row index is outside [0, n_src).  The flagged frame changes no state, and later calls change none; the
 *   caller reads the word with the outputs.
 *   Eight launches, whatever n, the live tracklets and the branch taken.
 * msda_qdtrack_workspace: the workspace bytes for these sizes.
 *
 * Limits: 1 <= n_cap <= 1024, 1 <= max_tracklets <= 1024, dim >= 1, memo_tracklet_frames >= 1, n_src >= 1; a NULL
 * required pointer, a misaligned (16-byte) workspace, too small a workspace or unknown flags give MSDA_E_BADARG.
 */
#ifndef MSDA_QDTRACK_H_
#define MSDA_QDTRACK_H_

#include <stdint.h>

#define MSDA_QD_BACKDROPS 1
#define MSDA_QD_MAX_BACKDROPS 1024
#define MSDA_QD_STATE_INTS(max_tracklets) (4 + 4 * (max_tracklets) + 1024)
#define MSDA_QD_STATE_LIVE 0
#define MSDA_QD_STATE_NEXT_ID 1
#define MSDA_QD_STATE_FLAGS 2
#define MSDA_QD_STATE_BACKDROPS 3
#define MSDA_QD_OVERFLOW 1
#define MSDA_QD_BAD_ROW 2

#ifdef __cplusplus
extern "C" {
#endif

int msda_qdtrack_workspace(int n_cap, int max_tracklets, int dim, int64_t *bytes);
int msda_qdtrack_match_f32(const float *boxes, const float *scores, const int *labels, const float *embeds,
                           const int *rows, const int *count, int n_src, int n_cap, int dim, float init_score_thr,
                           float obj_score_thr, float match_score_thr, float nms_conf_thr, float nms_backdrop_iou_thr,
                           float nms_class_iou_thr, double memo_momentum, int memo_tracklet_frames, int flags,
                           int frame_id, int max_tracklets, int *state, float *embed, float *backdrop_embed, int *order,
                           int *ids, int *tracked, int *tracked_count, void *workspace, int64_t workspace_bytes,
                           void *stream);

#ifdef __cplusplus
}
#endif

#endif  /* MSDA_QDTRACK_H_ */
