// msda_qdtrack.cuh -- the association step of the QuasiDense tracker (DESIGN.md section 3.19; the reference's
// QuasiDenseEmbedTracker.match, update_memo and memo, models/tracker.py:304-503) on the device: the rows sorted by score,
// the pairwise box IoU as two bitmasks, the duplicate removal, the memo columns (tracklets, then last frame's backdrops),
// the bi-softmax scores with the category mask, the greedy assignment, the new ids, the backdrops and the track memory.
// Eight launches per call, whatever the sizes and the branch taken; every row and tracklet count is read on the device.
// Integer atomics only.  The embedding product, the softmax statistics, the block reductions, the rank and the momentum
// update are msda_tracker.cuh's, shared with the IDOL tracker.
//
// State (caller-owned, zero = an empty tracker), int32 [kQdHeader + 4 * T + kQdMaxBackdrops]: live, next_id, error
// flags, backdrops; then order[T] (the live slots in ascending id order: the memo's first columns), and per slot id[T],
// last_frame[T], label[T]; then the backdrops' labels.  Per slot the embedding [T, D]; the backdrops' embeddings
// [kQdMaxBackdrops, D] in their row order.
#pragma once

#include "msda_tracker.cuh"

namespace msda {

constexpr int kQdMaxRows = 1024, kQdMaxTracklets = 1024, kQdMaxBackdrops = kQdMaxRows;
constexpr int kQdHeader = 4;
constexpr int kQdOverflow = 1, kQdBadRow = 2;                // state[2] bits; sticky
constexpr int kQdThreads = 1024, kQdMemoCtas = 128;
constexpr int kQdBack = 1 << 29;                             // row_slot: a backdrop's store index carries this bit

struct QdParams {
    float init_thr, obj_thr, match_thr, conf_thr, back_iou, class_iou, keep_w, new_w;   // keep_w = fp32(1 - momentum)
    int memo_frames, keep_backdrops, frame_id;
};

// mmcv's bbox_overlaps (mode "iou") as torch evaluates it on fp32 tensors, each operation rounded once: areas
// (x2 - x1) * (y2 - y1), wh = max(min(rb) - max(lt), 0), union = max(area_a + area_b - overlap, 1e-6f), overlap /
// union.  Unlike dp_iou_above (msda_nms.cuh) the union is clamped, which changes the result on degenerate and inverted
// boxes.
__device__ __forceinline__ float qd_box_iou(float4 a, float4 b) {
    const float aa = __fmul_rn(__fsub_rn(a.z, a.x), __fsub_rn(a.w, a.y));
    const float ab = __fmul_rn(__fsub_rn(b.z, b.x), __fsub_rn(b.w, b.y));
    const float w = fmaxf(__fsub_rn(fminf(a.z, b.z), fmaxf(a.x, b.x)), 0.f);
    const float h = fmaxf(__fsub_rn(fminf(a.w, b.w), fmaxf(a.y, b.y)), 0.f);
    const float overlap = __fmul_rn(w, h);
    const float uni = fmaxf(__fsub_rn(__fadd_rn(aa, ab), overlap), 1e-6f);
    return __fdiv_rn(overlap, uni);
}

// A score as an unsigned key that orders as the float does (-0 as +0, NaN above +inf, as torch's sort places it).
__device__ __forceinline__ unsigned qd_score_key(float s) {
    if (s != s) return 0xffffffffu;
    const unsigned u = __float_as_uint(s == 0.f ? 0.f : s);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float4 qd_box(const float *boxes, int r) {
    const float *b = boxes + (size_t)r * 4;
    return make_float4(b[0], b[1], b[2], b[3]);
}

// One CTA of 1024 threads: order[p] = the input row at sorted position p < n = count (score descending, a stable
// counting rank), -1 past n; flags a row index outside [0, n_src).
__global__ void __launch_bounds__(kQdThreads) qd_sort(const float *__restrict__ scores, const int *__restrict__ rows,
                                                      const int *__restrict__ count, int n_cap, int n_src,
                                                      int *__restrict__ order, int *__restrict__ state)
{
    __shared__ unsigned s_key[kQdMaxRows];
    const int n = min(*count, n_cap), t = threadIdx.x;
    unsigned key = 0u;
    if (t < n) {
        key = qd_score_key(scores[t]);
        s_key[t] = key;
        const int row = rows[t];
        if (row < 0 || row >= n_src) atomicOr(&state[2], kQdBadRow);
    }
    __syncthreads();
    if (t < n) {
        int rank = 0;
        for (int j = 0; j < n; ++j) {
            const unsigned kj = s_key[j];
            rank += kj > key || (kj == key && j < t);
        }
        order[rank] = t;
    }
    for (int p = n + t; p < n_cap; p += kQdThreads) order[p] = -1;
}

// Tile (blockIdx.y, blockIdx.x) of 32 sorted rows i by 32 sorted rows j: the u32 halves of dup[i] / back[i] (n x
// ceil(n/64) u64 words, n = count) for j0 .. j0 + 31.  Bit j - 64 w is set when j > i and IoU(i, j) > thr_j (dup;
// thr_j = back_iou when score_j < obj_thr, else class_iou), > back_iou (back).  Warp a of 8 takes rows a, a + 8, ...
// of the tile, lane l column j0 + l.
__global__ void __launch_bounds__(kIdolThreads) qd_iou(const float *__restrict__ boxes, const float *__restrict__ scores,
                                                       const int *__restrict__ order, const int *__restrict__ count,
                                                       int n_cap, QdParams p, unsigned *__restrict__ dup,
                                                       unsigned *__restrict__ back)
{
    const int n = min(*count, n_cap), halves = 2 * ((n + 63) / 64);
    const int i0 = blockIdx.y * kIdolTile, j0 = blockIdx.x * kIdolTile, t = threadIdx.x;
    if (i0 >= n || (int)blockIdx.x >= halves) return;
    __shared__ float4 si[kIdolTile], sj[kIdolTile];
    __shared__ float sthr[kIdolTile];
    if (t < kIdolTile && i0 + t < n) si[t] = qd_box(boxes, order[i0 + t]);
    if (t >= kIdolTile && t < 2 * kIdolTile && j0 + t - kIdolTile < n) {
        const int r = order[j0 + t - kIdolTile];
        sj[t - kIdolTile] = qd_box(boxes, r);
        sthr[t - kIdolTile] = scores[r] < p.obj_thr ? p.back_iou : p.class_iou;
    }
    __syncthreads();
    const int lane = t & 31, j = j0 + lane;
    for (int a = t >> 5; a < kIdolTile && i0 + a < n; a += kIdolThreads / 32) {
        const int i = i0 + a;
        const bool pair = j < n && j > i;
        const float iou = pair ? qd_box_iou(si[a], sj[lane]) : 0.f;
        const unsigned d = __ballot_sync(kFullMask, pair && iou > sthr[lane]);
        const unsigned b = __ballot_sync(kFullMask, pair && iou > p.back_iou);
        if (lane == 0) {
            dup[(size_t)i * halves + blockIdx.x] = d;
            back[(size_t)i * halves + blockIdx.x] = b;
        }
    }
}

// The block's OR of rows[e * W + w] over e in [0, k) (e -> pos[e] when pos is given) into hit[w], W <= 16 words
// (every thread; hit zeroed by the caller before a barrier).
__device__ __forceinline__ void qd_or_rows(const unsigned long long *__restrict__ rows, const int *pos, int k, int W,
                                           unsigned long long *hit) {
    const int t = threadIdx.x;
    if (W > 0 && t < ((int)blockDim.x / W) * W) {
        const int w = t % W, G = blockDim.x / W;
        unsigned long long acc = 0ull;
        for (int e = t / W; e < k; e += G) acc |= rows[(size_t)(pos ? pos[e] : e) * W + w];
        if (acc) atomicOr(&hit[w], acc);
    }
    __syncthreads();
}

// One CTA of 1024 threads: the duplicate removal.  Sorted row j is dropped when a dup bit (i, j) is set for any i < j,
// dropped or not: an OR over every row's mask.  kept_pos[0 .. k) the kept sorted positions in order, kept_r the
// input rows there, *kept_count = k.
__global__ void __launch_bounds__(kQdThreads) qd_dedup(const unsigned long long *__restrict__ dup,
                                                       const int *__restrict__ order, const int *__restrict__ count,
                                                       int n_cap, int *__restrict__ kept_pos, int *__restrict__ kept_r,
                                                       int *__restrict__ kept_count)
{
    __shared__ unsigned long long s_hit[kQdMaxRows / 64];
    __shared__ int warp_tot[32];
    const int n = min(*count, n_cap), W = (n + 63) / 64, t = threadIdx.x;
    if (t < kQdMaxRows / 64) s_hit[t] = 0ull;
    __syncthreads();
    qd_or_rows(dup, nullptr, n, W, s_hit);
    const bool keep = t < n && !((s_hit[t >> 6] >> (t & 63)) & 1ull);
    int k;
    const int rank = idol_rank(keep, warp_tot, k);
    if (keep) {
        kept_pos[rank] = t;
        kept_r[rank] = order[t];
    }
    if (t == 0) *kept_count = k;
}

// kQdMemoCtas CTAs: the memo's columns c < cols = live + backdrops, M[c] and mlabel[c]: the live slots' embeddings and
// labels in ascending id order, then the backdrops' in their row order; *ncols = cols.
__global__ void __launch_bounds__(kIdolThreads) qd_memo(const int *__restrict__ state, const float *__restrict__ embed,
                                                        const float *__restrict__ back_embed, int T, int D,
                                                        float *__restrict__ M, int *__restrict__ mlabel,
                                                        int *__restrict__ ncols)
{
    const int live = state[0], cols = live + state[3];
    const int *order = state + kQdHeader, *label = order + 3 * T, *back_label = order + 4 * T;
    if (blockIdx.x == 0 && threadIdx.x == 0) *ncols = cols;
    for (int c = blockIdx.x; c < cols; c += gridDim.x) {
        const bool trk = c < live;
        const int slot = trk ? order[c] : c - live;
        const float *src = (trk ? embed : back_embed) + (size_t)slot * D;
        for (int d = threadIdx.x; d < D; d += kIdolThreads) M[(size_t)c * D + d] = src[d];
        if (threadIdx.x == 0) mlabel[c] = trk ? label[slot] : back_label[slot];
    }
}

// The bi-softmax score of kept row i and column c from its feature and the two softmaxes' (max, sum), masked by the
// category: (exp(f - rmax) / rsum + exp(f - cmax) / csum) / 2, times (row label == column label).
__device__ __forceinline__ float qd_score(float f, float rmax, float rsum, float cmax, float csum, bool same) {
    const float d2t = __fdiv_rn(expf(f - rmax), rsum), t2d = __fdiv_rn(expf(f - cmax), csum);
    return same ? __fmul_rn(__fadd_rn(d2t, t2d), 0.5f) : 0.f;
}

// One CTA of 1024 threads (thread t: kept row t and memo columns t and t + 1024): the greedy assignment, the new ids,
// the backdrops, the outputs, and the bookkeeping (expiry, slots for the new tracklets, the memo order, the backdrops'
// labels).  Leaves the state as it was when it is flagged, or would be after this frame (kQdOverflow, set here: more
// live tracklets than slots).
__global__ void __launch_bounds__(kQdThreads, 1) qd_assign(
    const float *__restrict__ F, const float *__restrict__ rstat, const float *__restrict__ cstat,
    const int *__restrict__ kept_pos, const int *__restrict__ kept_r, const int *__restrict__ kept_count,
    const int *__restrict__ count, const float *__restrict__ scores, const int *__restrict__ labels,
    const int *__restrict__ mlabel, const unsigned long long *__restrict__ back, int n_cap, int S, int T, QdParams p,
    int *__restrict__ state, int *__restrict__ ids, int *__restrict__ tracked, int *__restrict__ tracked_count,
    int *__restrict__ row_slot)
{
    __shared__ int s_id[kQdMaxRows], s_mcol[kQdMaxRows], s_label[kQdMaxRows], s_colid[kQdMaxTracklets];
    __shared__ int s_taken[kQdMaxTracklets], s_used[kQdMaxTracklets], s_newslot[kQdMaxTracklets];
    __shared__ int s_order[kQdMaxTracklets], warp_tot[32];
    __shared__ float s_score[kQdMaxRows];
    __shared__ unsigned long long s_hit[kQdMaxRows / 64], red[32];
    const int t = threadIdx.x;
    const int n = min(*count, n_cap), k = *kept_count, live = state[0], next = state[1], bad = state[2];
    const int cols = live + state[3];
    int *order = state + kQdHeader, *sid = order + T, *last = sid + T, *lab = last + T, *back_label = lab + T;
    const int my_slot = t < live ? order[t] : -1;
    for (int r = t; r < n_cap; r += kQdThreads) {
        ids[r] = -3;
        tracked[r] = -1;
    }
    if (t < live) {
        s_colid[t] = sid[my_slot];
        s_taken[t] = 0;
    }
    if (t < k) {
        const int r = kept_r[t];
        s_id[t] = -1;
        s_mcol[t] = -1;
        s_score[t] = scores[r];
        s_label[t] = labels[r];
    }
    if (t < kQdMaxRows / 64) s_hit[t] = 0ull;
    __syncthreads();

    if (live > 0 && !bad) {                                  // the backdrops alone do not make the memo
        const int c1 = t + kQdThreads;
        const bool v0 = t < cols, v1 = c1 < cols;
        const float cm0 = v0 ? cstat[2 * t] : 0.f, cs0 = v0 ? cstat[2 * t + 1] : 1.f;
        const float cm1 = v1 ? cstat[2 * c1] : 0.f, cs1 = v1 ? cstat[2 * c1 + 1] : 1.f;
        const int l0 = v0 ? mlabel[t] : 0, l1 = v1 ? mlabel[c1] : 0;
        for (int i = 0; i < k; ++i) {
            const float rmax = rstat[2 * i], rsum = rstat[2 * i + 1];
            const int li = s_label[i];
            // a taken tracklet scores 0 for every later row; non-negative floats order as their bits, ties go to the
            // lowest column
            unsigned long long key = 0ull;
            if (v0) {
                const float s = (t < live && s_taken[t]) ? 0.f
                                                         : qd_score(F[(size_t)i * S + t], rmax, rsum, cm0, cs0, l0 == li);
                key = ((unsigned long long)__float_as_uint(s) << 32) | (0xffffffffu - (unsigned)t);
            }
            if (v1) {                                        // a backdrop column: never taken
                const float s = qd_score(F[(size_t)i * S + c1], rmax, rsum, cm1, cs1, l1 == li);
                const unsigned long long k1 = ((unsigned long long)__float_as_uint(s) << 32) | (0xffffffffu - (unsigned)c1);
                key = k1 > key ? k1 : key;
            }
            const unsigned long long best = idol_block_max_u64(key, red);
            const float conf = __uint_as_float((unsigned)(best >> 32));
            const int c = (int)(0xffffffffu - (unsigned)best);
            if (t == 0 && conf > p.match_thr && c < live) {
                if (s_score[i] > p.obj_thr) {
                    s_id[i] = s_colid[c];
                    s_mcol[i] = c;
                    s_taken[c] = 1;
                } else if (conf > p.conf_thr) {
                    s_id[i] = -2;
                }
            }
            __syncthreads();
        }
    }

    // new ids in row order
    int m;
    const bool is_new = t < k && s_id[t] == -1 && s_score[t] > p.init_thr;
    const int new_rank = idol_rank(is_new, warp_tot, m);
    if (is_new) s_id[t] = next + new_rank;
    __syncthreads();

    // backdrops: a row still at -1 with IoU <= back_iou against every earlier kept row
    qd_or_rows(back, kept_pos, k, (n + 63) / 64, s_hit);
    int nb;
    const int pos = t < k ? kept_pos[t] : 0;
    const bool is_back = t < k && s_id[t] == -1 && !((s_hit[pos >> 6] >> (pos & 63)) & 1ull);
    const int back_rank = idol_rank(is_back, warp_tot, nb);
    if (t < k) ids[pos] = s_id[t];
    int nt;
    const bool is_tracked = t < k && s_id[t] > -1;
    const int tr = idol_rank(is_tracked, warp_tot, nt);
    if (is_tracked) tracked[tr] = kept_r[t];
    if (t == 0) *tracked_count = nt;

    // the memory's bookkeeping
    const bool matched = t < live && s_taken[t];
    const bool survive = t < live && (matched || p.frame_id - last[my_slot] < p.memo_frames);
    int ns;
    const int sr = idol_rank(survive, warp_tot, ns);
    if (bad || ns + m > T) {
        if (t < n_cap) row_slot[t] = -1;
        if (t == 0 && !bad) atomicOr(&state[2], kQdOverflow);
        return;
    }
    if (t < T) s_used[t] = 0;
    __syncthreads();
    if (survive) s_used[my_slot] = 1;
    __syncthreads();
    int nf;
    const bool is_free = t < T && !s_used[t];
    const int fr = idol_rank(is_free, warp_tot, nf);
    if (is_free && fr < m) s_newslot[fr] = t;
    if (survive) s_order[sr] = my_slot;
    __syncthreads();
    const bool stored = is_back && p.keep_backdrops;
    const int mslot = t < k && s_mcol[t] >= 0 ? order[s_mcol[t]] : -1;
    if (is_new) s_order[ns + new_rank] = s_newslot[new_rank];
    if (t < n_cap)
        row_slot[t] = t >= k ? -1 : is_new ? (s_newslot[new_rank] | kIdolNew) : mslot >= 0 ? mslot
                    : stored ? (back_rank | kQdBack) : -1;
    __syncthreads();                                               // every read of order[] is done
    if (mslot >= 0) {
        last[mslot] = p.frame_id;
        lab[mslot] = s_label[t];
    }
    if (is_new) {
        const int slot = s_newslot[new_rank];
        sid[slot] = s_id[t];
        last[slot] = p.frame_id;
        lab[slot] = s_label[t];
    }
    if (stored) back_label[back_rank] = s_label[t];
    if (t < ns + m) order[t] = s_order[t];
    if (t == 0) {
        state[0] = ns + m;
        state[1] = next + m;
        state[3] = p.keep_backdrops ? nb : 0;
    }
}

// One CTA per kept row i with a tracklet or a stored backdrop: a new tracklet takes e as its embedding, a matched one's
// becomes keep_w * embed + new_w * e, a backdrop's e goes to its place in the store (read by qd_memo, two launches
// before).
__global__ void __launch_bounds__(kIdolThreads) qd_update(const float *__restrict__ embeds, const int *__restrict__ rows,
                                                          const int *__restrict__ kept_r,
                                                          const int *__restrict__ kept_count,
                                                          const int *__restrict__ row_slot, int D, QdParams p,
                                                          float *__restrict__ embed, float *__restrict__ back_embed)
{
    const int i = blockIdx.x;
    if (i >= *kept_count) return;
    const int rs = row_slot[i];
    if (rs < 0) return;
    const float *e = embeds + (size_t)rows[kept_r[i]] * D;
    if (rs & kQdBack) {
        float *dst = back_embed + (size_t)(rs & ~kQdBack) * D;
        for (int d = threadIdx.x; d < D; d += kIdolThreads) dst[d] = e[d];
        return;
    }
    const bool fresh = rs & kIdolNew;
    float *em = embed + (size_t)(rs & ~kIdolNew) * D;
    for (int d = threadIdx.x; d < D; d += kIdolThreads) em[d] = fresh ? e[d] : tracker_ema(p.keep_w, em[d], p.new_w, e[d]);
}

}  // namespace msda
