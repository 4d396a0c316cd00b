// msda_cabi_tracker.cu -- C ABI of the video trackers' association steps: IDOL (msda_tracker.cuh, include/msda_tracker.h)
// and QuasiDense (msda_qdtrack.cuh, include/msda_qdtrack.h), in one translation unit because they share kernels.
#include "../../include/msda_b200.h"
#include "../../include/msda_qdtrack.h"
#include "../../include/msda_tracker.h"
#include "msda_host.cuh"
#include "msda_qdtrack.cuh"

using namespace msda_host;

namespace {

static_assert(MSDA_IDOL_STATE_INTS(0) == msda::kIdolHeader, "state header");
static_assert(MSDA_QD_STATE_INTS(0) == msda::kQdHeader + msda::kQdMaxBackdrops, "state header");
static_assert(MSDA_QD_MAX_BACKDROPS == msda::kQdMaxBackdrops, "backdrop store");

int idol_check(int n_cap, int T, int dim, int h, int w) {
    if (n_cap < 1 || n_cap > msda::kIdolMaxRows || T < 1 || T > msda::kIdolMaxTracklets || dim < 1 || h < 1 || w < 1 ||
        (long long)h * w >= (1ll << 24))
        return MSDA_E_BADARG;
    return 0;
}

struct IdolLayout {
    size_t bits, popc, pre, post, ints, memo, feats, rstat, cstat, total;
    int words4;
};

IdolLayout idol_layout(int n_cap, int T, int dim, int h, int w) {
    IdolLayout l{};
    const long long words = ((long long)h * w + 31) / 32;
    l.words4 = (int)((words + 3) / 4 * 4);
    const size_t mask_bytes = (size_t)n_cap * ((n_cap + 63) / 64) * sizeof(unsigned long long);
    l.bits = 0;
    l.popc = align256(l.bits + (size_t)n_cap * l.words4 * sizeof(unsigned));
    l.pre = align256(l.popc + (size_t)n_cap * sizeof(int));
    l.post = align256(l.pre + mask_bytes);
    l.ints = align256(l.post + mask_bytes);                              // kept_count, kept [n_cap], row_slot [n_cap]
    l.memo = align256(l.ints + (1 + 2 * (size_t)n_cap) * sizeof(int));
    l.feats = align256(l.memo + (size_t)T * dim * sizeof(float));
    l.rstat = align256(l.feats + (size_t)n_cap * T * sizeof(float));
    l.cstat = align256(l.rstat + 2 * (size_t)n_cap * sizeof(float));
    l.total = align256(l.cstat + 2 * (size_t)T * sizeof(float));
    return l;
}

int qd_check(int n_cap, int T, int dim) {
    if (n_cap < 1 || n_cap > msda::kQdMaxRows || T < 1 || T > msda::kQdMaxTracklets || dim < 1) return MSDA_E_BADARG;
    return 0;
}

struct QdLayout {
    size_t dup, back, ints, memo, feats, rstat, cstat, total;
    int cols;                                                            // the memo's column capacity, F's row stride
};

QdLayout qd_layout(int n_cap, int T, int dim) {
    QdLayout l{};
    l.cols = T + msda::kQdMaxBackdrops;
    const size_t mask_bytes = (size_t)n_cap * ((n_cap + 63) / 64) * sizeof(unsigned long long);
    l.dup = 0;
    l.back = align256(l.dup + mask_bytes);
    l.ints = align256(l.back + mask_bytes);        // kept_count, ncols, kept_pos [n_cap], kept_r [n_cap], row_slot [n_cap],
    l.memo = align256(l.ints + (2 + 3 * (size_t)n_cap + l.cols) * sizeof(int));      // mlabel [cols]
    l.feats = align256(l.memo + (size_t)l.cols * dim * sizeof(float));
    l.rstat = align256(l.feats + (size_t)n_cap * l.cols * sizeof(float));
    l.cstat = align256(l.rstat + 2 * (size_t)n_cap * sizeof(float));
    l.total = align256(l.cstat + 2 * (size_t)l.cols * sizeof(float));
    return l;
}

}  // namespace

extern "C" {

int msda_idol_workspace(int n_cap, int max_tracklets, int dim, int h, int w, int64_t *bytes) {
    if (!bytes) return MSDA_E_BADARG;
    if (const int c = idol_check(n_cap, max_tracklets, dim, h, w)) return c;
    *bytes = (int64_t)idol_layout(n_cap, max_tracklets, dim, h, w).total;
    return 0;
}

int msda_idol_match_f32(const float *masks, const float *embeds, const float *scores, const int *rows, const int *count,
                        int n_src, int n_cap, int h, int w, int dim, float nms_thr_pre, float nms_thr_post,
                        float init_score_thr, float addnew_score_thr, float match_score_thr, double memo_momentum,
                        int memo_tracklet_frames, int memory_len, int flags, const float *temporal_weights, int frame_id,
                        int max_tracklets, int *state, float *embed, float *ring_embed, float *ring_score, int *ids,
                        int *tracked, int *tracked_count, void *workspace, int64_t workspace_bytes, void *stream) {
    constexpr int kAll = MSDA_IDOL_LONG_MATCH | MSDA_IDOL_FRAME_WEIGHT | MSDA_IDOL_TEMPORAL_WEIGHT;
    const bool long_match = flags & MSDA_IDOL_LONG_MATCH;
    const bool temporal = long_match && (flags & MSDA_IDOL_TEMPORAL_WEIGHT);
    if (!masks || !embeds || !scores || !rows || !count || !state || !embed || !ring_embed || !ring_score || !ids ||
        !tracked || !tracked_count || !workspace || !aligned16(workspace) || (temporal && !temporal_weights) ||
        (flags & ~kAll))
        return MSDA_E_BADARG;
    if (const int c = idol_check(n_cap, max_tracklets, dim, h, w)) return c;
    if (n_src < 1 || memory_len < 1 || memory_len > msda::kIdolMaxMemory || memo_tracklet_frames < 1)
        return MSDA_E_BADARG;
    const int T = max_tracklets;
    const IdolLayout l = idol_layout(n_cap, T, dim, h, w);
    if (workspace_bytes < (int64_t)l.total) return MSDA_E_BADARG;
    char *ws = static_cast<char *>(workspace);
    unsigned *bits = reinterpret_cast<unsigned *>(ws + l.bits);
    int *popc = reinterpret_cast<int *>(ws + l.popc);
    int *kept_count = reinterpret_cast<int *>(ws + l.ints), *kept = kept_count + 1, *row_slot = kept + n_cap;
    float *M = reinterpret_cast<float *>(ws + l.memo), *F = reinterpret_cast<float *>(ws + l.feats);
    float *rstat = reinterpret_cast<float *>(ws + l.rstat), *cstat = reinterpret_cast<float *>(ws + l.cstat);
    const msda::IdolParams p{nms_thr_post, init_score_thr, addnew_score_thr, match_score_thr,
                             (float)(1.0 - memo_momentum), (float)memo_momentum, (flags & MSDA_IDOL_FRAME_WEIGHT) ? 1 : 0,
                             memo_tracklet_frames, frame_id, long_match ? 1 : 0, memory_len};
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const unsigned row_tiles = (unsigned)((n_cap + msda::kIdolTile - 1) / msda::kIdolTile);
    const unsigned halves = (unsigned)(2 * ((n_cap + 63) / 64));
    const unsigned col_tiles = (unsigned)((T + msda::kIdolTile - 1) / msda::kIdolTile);
    cudaError_t e;
    if ((e = launch(msda::idol_pack, dim3((unsigned)n_cap), msda::kIdolThreads, 0, st, masks, rows, count, n_cap, n_src,
                    (long long)h * w, l.words4, bits, popc, state)) ||
        (e = launch(msda::idol_iou, dim3(halves, row_tiles), msda::kIdolThreads, 0, st, (const unsigned *)bits,
                    (const int *)popc, count, n_cap, l.words4, nms_thr_pre, nms_thr_post,
                    reinterpret_cast<unsigned *>(ws + l.pre), reinterpret_cast<unsigned *>(ws + l.post))) ||
        (e = launch(msda::idol_nms, dim3(1), 32, 0, st, reinterpret_cast<const unsigned long long *>(ws + l.pre), count,
                    n_cap, kept, kept_count)) ||
        (e = launch(msda::idol_memo, dim3((unsigned)T), msda::kIdolThreads, 0, st, (const int *)state,
                    (const float *)embed, (const float *)ring_embed, (const float *)ring_score,
                    temporal ? temporal_weights : nullptr, T, memory_len, dim, p.long_match, M)) ||
        (e = launch(msda::idol_feats, dim3(col_tiles, row_tiles), msda::kIdolThreads, 0, st, embeds, rows,
                    (const int *)kept, (const int *)kept_count, (const int *)state, (const int *)state + 2,
                    (const float *)M, T, dim, F)) ||
        (e = launch(msda::idol_softmax_stats, dim3((unsigned)(n_cap + T)), msda::kIdolThreads, 0, st, (const float *)F,
                    (const int *)kept_count, (const int *)state, (const int *)state + 2, n_cap, T, rstat, cstat)) ||
        (e = launch(msda::idol_assign, dim3(1), msda::kIdolAssignThreads, 0, st, (const float *)F, (const float *)rstat,
                    (const float *)cstat, (const int *)kept, (const int *)kept_count, count, scores,
                    reinterpret_cast<const unsigned long long *>(ws + l.post), n_cap, T, p, state, ids, tracked,
                    tracked_count, row_slot)))
        return (int)e;
    return (int)launch(msda::idol_update, dim3((unsigned)n_cap), msda::kIdolThreads, 0, st, embeds, rows, scores,
                       (const int *)kept, (const int *)kept_count, (const int *)row_slot, T, dim, p, state, embed,
                       ring_embed, ring_score);
}

int msda_qdtrack_workspace(int n_cap, int max_tracklets, int dim, int64_t *bytes) {
    if (!bytes) return MSDA_E_BADARG;
    if (const int c = qd_check(n_cap, max_tracklets, dim)) return c;
    *bytes = (int64_t)qd_layout(n_cap, max_tracklets, dim).total;
    return 0;
}

int msda_qdtrack_match_f32(const float *boxes, const float *scores, const int *labels, const float *embeds,
                           const int *rows, const int *count, int n_src, int n_cap, int dim, float init_score_thr,
                           float obj_score_thr, float match_score_thr, float nms_conf_thr, float nms_backdrop_iou_thr,
                           float nms_class_iou_thr, double memo_momentum, int memo_tracklet_frames, int flags,
                           int frame_id, int max_tracklets, int *state, float *embed, float *backdrop_embed, int *order,
                           int *ids, int *tracked, int *tracked_count, void *workspace, int64_t workspace_bytes,
                           void *stream) {
    if (!boxes || !scores || !labels || !embeds || !rows || !count || !state || !embed || !backdrop_embed || !order ||
        !ids || !tracked || !tracked_count || !workspace || !aligned16(workspace) || (flags & ~MSDA_QD_BACKDROPS))
        return MSDA_E_BADARG;
    if (const int c = qd_check(n_cap, max_tracklets, dim)) return c;
    if (n_src < 1 || memo_tracklet_frames < 1) return MSDA_E_BADARG;
    const int T = max_tracklets;
    const QdLayout l = qd_layout(n_cap, T, dim);
    if (workspace_bytes < (int64_t)l.total) return MSDA_E_BADARG;
    char *ws = static_cast<char *>(workspace);
    const auto *dup = reinterpret_cast<const unsigned long long *>(ws + l.dup);
    const auto *back = reinterpret_cast<const unsigned long long *>(ws + l.back);
    int *kept_count = reinterpret_cast<int *>(ws + l.ints), *ncols = kept_count + 1, *kept_pos = ncols + 1;
    int *kept_r = kept_pos + n_cap, *row_slot = kept_r + n_cap, *mlabel = row_slot + n_cap;
    float *M = reinterpret_cast<float *>(ws + l.memo), *F = reinterpret_cast<float *>(ws + l.feats);
    float *rstat = reinterpret_cast<float *>(ws + l.rstat), *cstat = reinterpret_cast<float *>(ws + l.cstat);
    const msda::QdParams p{init_score_thr,       obj_score_thr,      match_score_thr,
                           nms_conf_thr,         nms_backdrop_iou_thr, nms_class_iou_thr,
                           (float)(1.0 - memo_momentum), (float)memo_momentum, memo_tracklet_frames,
                           (flags & MSDA_QD_BACKDROPS) ? 1 : 0, frame_id};
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const unsigned row_tiles = (unsigned)((n_cap + msda::kIdolTile - 1) / msda::kIdolTile);
    const unsigned halves = (unsigned)(2 * ((n_cap + 63) / 64));
    const unsigned col_tiles = (unsigned)((l.cols + msda::kIdolTile - 1) / msda::kIdolTile);
    const int *err = state + 2;
    cudaError_t e;
    if ((e = launch(msda::qd_sort, dim3(1), msda::kQdThreads, 0, st, scores, rows, count, n_cap, n_src, order, state)) ||
        (e = launch(msda::qd_iou, dim3(halves, row_tiles), msda::kIdolThreads, 0, st, boxes, scores, (const int *)order,
                    count, n_cap, p, reinterpret_cast<unsigned *>(ws + l.dup),
                    reinterpret_cast<unsigned *>(ws + l.back))) ||
        (e = launch(msda::qd_dedup, dim3(1), msda::kQdThreads, 0, st, dup, (const int *)order, count, n_cap, kept_pos,
                    kept_r, kept_count)) ||
        (e = launch(msda::qd_memo, dim3(msda::kQdMemoCtas), msda::kIdolThreads, 0, st, (const int *)state,
                    (const float *)embed, (const float *)backdrop_embed, T, dim, M, mlabel, ncols)) ||
        (e = launch(msda::idol_feats, dim3(col_tiles, row_tiles), msda::kIdolThreads, 0, st, embeds, rows,
                    (const int *)kept_r, (const int *)kept_count, (const int *)ncols, err, (const float *)M, l.cols,
                    dim, F)) ||
        (e = launch(msda::idol_softmax_stats, dim3((unsigned)(n_cap + l.cols)), msda::kIdolThreads, 0, st,
                    (const float *)F, (const int *)kept_count, (const int *)ncols, err, n_cap, l.cols, rstat, cstat)) ||
        (e = launch(msda::qd_assign, dim3(1), msda::kQdThreads, 0, st, (const float *)F, (const float *)rstat,
                    (const float *)cstat, (const int *)kept_pos, (const int *)kept_r, (const int *)kept_count, count,
                    scores, labels, (const int *)mlabel, back, n_cap, l.cols, T, p, state, ids, tracked,
                    tracked_count, row_slot)))
        return (int)e;
    return (int)launch(msda::qd_update, dim3((unsigned)n_cap), msda::kIdolThreads, 0, st, embeds, rows,
                       (const int *)kept_r, (const int *)kept_count, (const int *)row_slot, dim, p, embed,
                       backdrop_embed);
}

}  // extern "C"
