/*
 * msda_tracker.h -- C ABI of the IDOL tracker's association step (DESIGN.md section 3.18; models/tracker.py:207-298,
 * IDOL_Tracker.match with match_metric "bisoftmax"), exported by libmsda_b200.so next to the functions of msda_b200.h
 * and following its conventions: device pointers on the current device; return 0, a positive cudaError_t, or a negative
 * MSDA_E_* of msda_b200.h (msda_strerror renders it); a caller-provided workspace whose size msda_idol_workspace gives;
 * the stream last.  Nothing is allocated and nothing synchronises with the host.  No float atomics.
 *
 * msda_idol_match_f32: one frame.  Row r < n = min(*count, n_cap) (count is read on the device) is masks[rows[r]]
 *   ([n_src, h, w] fp32 stride-4 logits), embeds[rows[r]] ([n_src, dim] fp32) and scores[r] ([n_cap] fp32), in the
 *   caller's order.  Per frame:
 *     mask = 1 / (1 + expf(-x)) > 0.5 (torch's CUDA sigmoid); IoU = (float(inter) + 1e-6f) / (float(union) + 1e-6f);
 *     mask NMS: row 0 kept, row j dropped when IoU(i, j) > nms_thr_pre for a kept i < j;
 *     no live tracklet: a kept row with score > init_score_thr gets a new id;
 *     else bi-softmax matching against the live tracklets in ascending id order (memo embedding: the EMA embedding, or
 *       with MSDA_IDOL_LONG_MATCH the score-weighted mean of the last memory_len embeddings, the scores plus row len - 1
 *       of temporal_weights [memory_len, memory_len] with MSDA_IDOL_TEMPORAL_WEIGHT; MSDA_IDOL_FRAME_WEIGHT: the
 *       exist-frame weighting), rows in order, a tracklet taken by one row only, ties to the lowest column; then the
 *       unmatched rows with score > addnew_score_thr get new ids in row order;
 *     a row left without id becomes a backdrop (-1) when its IoU with every earlier kept row is < nms_thr_post, else -2;
 *     memory: a matched tracklet's embedding becomes fp32(1 - memo_momentum) * embed + fp32(memo_momentum) * e, e and the
 *       score enter its rings of memory_len, last_frame = frame_id, exist_frame += 1; a new one starts from e; then the
 *       tracklets with frame_id - last_frame >= memo_tracklet_frames are dropped.
 *   Outputs: ids [n_cap] int32 per row (>= 0 a tracklet id, -1 a backdrop, -2 neither, -3 removed by the NMS or past
 *   n); tracked [n_cap] int32, the rows with an id >= 0 in row order (-1 after them); tracked_count [1].
 *   State, owned by the caller and zero-filled for an empty tracker: state int32 [MSDA_IDOL_STATE_INTS(max_tracklets)],
 *   embed [max_tracklets, dim], ring_embed [max_tracklets, memory_len, dim], ring_score [max_tracklets, memory_len]
 *   fp32.  state[MSDA_IDOL_STATE_FLAGS] is a sticky error word: MSDA_IDOL_OVERFLOW when a frame would leave more than
 *   max_tracklets live tracklets, MSDA_IDOL_BAD_ROW when a row index is outside [0, n_src).  The flagged frame changes
 *   no state, and later calls change none; the caller reads the word with the outputs.
 *   Eight launches, whatever n, the live tracklets and the branch taken.
 * msda_idol_workspace: the workspace bytes for these sizes.
 *
 * Limits: 1 <= n_cap <= 1024, 1 <= max_tracklets <= 1024, dim >= 1, h, w >= 1 with h * w < 2^24, 1 <= memory_len <= 64,
 * memo_tracklet_frames >= 1, n_src >= 1; a NULL required pointer, a misaligned (16-byte) workspace, too small a workspace
 * or unknown flags give MSDA_E_BADARG.
 */
#ifndef MSDA_TRACKER_H_
#define MSDA_TRACKER_H_

#include <stdint.h>

#define MSDA_IDOL_LONG_MATCH 1
#define MSDA_IDOL_FRAME_WEIGHT 2
#define MSDA_IDOL_TEMPORAL_WEIGHT 4
#define MSDA_IDOL_STATE_INTS(max_tracklets) (4 + 5 * (max_tracklets))
#define MSDA_IDOL_STATE_LIVE 0
#define MSDA_IDOL_STATE_NEXT_ID 1
#define MSDA_IDOL_STATE_FLAGS 2
#define MSDA_IDOL_OVERFLOW 1
#define MSDA_IDOL_BAD_ROW 2

#ifdef __cplusplus
extern "C" {
#endif

int msda_idol_workspace(int n_cap, int max_tracklets, int dim, int h, int w, int64_t *bytes);
int msda_idol_match_f32(const float *masks, const float *embeds, const float *scores, const int *rows, const int *count,
                        int n_src, int n_cap, int h, int w, int dim, float nms_thr_pre, float nms_thr_post,
                        float init_score_thr, float addnew_score_thr, float match_score_thr, double memo_momentum,
                        int memo_tracklet_frames, int memory_len, int flags, const float *temporal_weights, int frame_id,
                        int max_tracklets, int *state, float *embed, float *ring_embed, float *ring_score, int *ids,
                        int *tracked, int *tracked_count, void *workspace, int64_t workspace_bytes, void *stream);

#ifdef __cplusplus
}
#endif

#endif  /* MSDA_TRACKER_H_ */
