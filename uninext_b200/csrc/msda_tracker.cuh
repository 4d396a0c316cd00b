// msda_tracker.cuh -- the association step of the IDOL tracker (DESIGN.md section 3.18; the reference's IDOL_Tracker.match,
// models/tracker.py:207-298) on the device: the binarised masks packed into bits, the pairwise mask IoU as two
// bitmasks, the mask NMS (msda_nms.cuh's sweep), the memo embeddings, the bi-softmax scores, the greedy assignment, the
// new ids, the backdrops and the track memory.  Eight launches per call, whatever the sizes and the branch taken; every
// row and tracklet count is read on the device.  Integer atomics only.
//
// State (caller-owned, zero = an empty tracker), int32 [kIdolHeader + 5 * T]: live, next_id, error flags, 0; then
// order[T] (the live slots in ascending id order: the memo's columns), and per slot id[T], last_frame[T],
// exist_frame[T], ring_len[T].  Per slot the EMA embedding [T, D], the ring of the last L embeddings [T, L, D] and of
// their scores [T, L], oldest first.
#pragma once

#include "msda_nms.cuh"

namespace msda {

constexpr int kIdolMaxRows = 1024, kIdolMaxTracklets = 1024, kIdolMaxMemory = 64;
constexpr int kIdolHeader = 4;
constexpr int kIdolOverflow = 1, kIdolBadRow = 2;            // state[2] bits; sticky
constexpr int kIdolTile = 32, kIdolThreads = 256, kIdolAssignThreads = 1024;
constexpr int kIdolNew = 1 << 30;                            // row_slot: a new tracklet's slot carries this bit

struct IdolParams {
    float thr_post, init_thr, addnew_thr, match_thr, keep_w, new_w;   // keep_w = fp32(1 - momentum), new_w = fp32(momentum)
    int frame_weight, memo_frames, frame_id, long_match, L;
};

// The momentum update of a tracklet's embedding, (1 - m) * old + m * x as torch evaluates it on fp32 tensors: the two
// weights rounded to fp32, each product and the sum rounded once.  Shared by both trackers.
__device__ __forceinline__ float tracker_ema(float keep_w, float old, float new_w, float x) {
    return __fadd_rn(__fmul_rn(keep_w, old), __fmul_rn(new_w, x));
}

// torch's CUDA sigmoid (1 / (1 + exp(-x)) in fp32, IEEE division) compared with 0.5, as the reference binarises.
__device__ __forceinline__ bool idol_on(float x) { return 1.0f / (1.0f + expf(-x)) > 0.5f; }

// One CTA per row r < count: the row's mask (masks + rows[r] * hw) as 32-pixel words, and its popcount.
__global__ void __launch_bounds__(kIdolThreads) idol_pack(const float *__restrict__ masks, const int *__restrict__ rows,
                                                          const int *__restrict__ count, int n_cap, int n_src,
                                                          long long hw, int words4, unsigned *__restrict__ bits,
                                                          int *__restrict__ popc, int *__restrict__ state)
{
    const int r = blockIdx.x;
    if (r >= min(*count, n_cap)) return;
    const int row = rows[r];
    if (row < 0 || row >= n_src) {
        if (threadIdx.x == 0) atomicOr(&state[2], kIdolBadRow);
        return;
    }
    __shared__ int total;
    if (threadIdx.x == 0) total = 0;
    __syncthreads();
    const float *src = masks + (long long)row * hw;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int mine = 0;
    for (int wd = warp; wd < words4; wd += kIdolThreads / 32) {
        const long long p = (long long)wd * 32 + lane;
        const unsigned b = __ballot_sync(kFullMask, p < hw && idol_on(src[p]));
        if (lane == 0) {
            bits[(size_t)r * words4 + wd] = b;
            mine += __popc(b);
        }
    }
    if (lane == 0) atomicAdd(&total, mine);
    __syncthreads();
    if (threadIdx.x == 0) popc[r] = total;
}

// Tile (blockIdx.y, blockIdx.x) of 32 rows i by 32 columns j: the u32 halves of pre[i] / post[i] (n x ceil(n/64) u64
// words, n = count) for columns j0 .. j0 + 31.  Bit j - 64 w is set when j > i and IoU(i, j) > thr_pre (pre), >= thr_post
// (post); IoU = (float(inter) + 1e-6f) / (float(union) + 1e-6f), the counts exact below 2^24.
__global__ void __launch_bounds__(kIdolThreads) idol_iou(const unsigned *__restrict__ bits, const int *__restrict__ popc,
                                                         const int *__restrict__ count, int n_cap, int words4,
                                                         float thr_pre, float thr_post, unsigned *__restrict__ pre,
                                                         unsigned *__restrict__ post)
{
    const int n = min(*count, n_cap), halves = 2 * ((n + 63) / 64);
    const int i0 = blockIdx.y * kIdolTile, j0 = blockIdx.x * kIdolTile, t = threadIdx.x;
    if (i0 >= n || blockIdx.x >= halves) return;
    __shared__ unsigned sp[kIdolTile], sq[kIdolTile];
    if (j0 + kIdolTile - 1 <= i0 || j0 >= n) {                       // no pair j > i, j < n here: zero halves
        if (t < kIdolTile && i0 + t < n) {
            pre[(size_t)(i0 + t) * halves + blockIdx.x] = 0u;
            post[(size_t)(i0 + t) * halves + blockIdx.x] = 0u;
        }
        return;
    }
    __shared__ unsigned sa[kIdolTile][kIdolTile + 1], sb[kIdolTile][kIdolTile + 1];
    const int ty = t / 16, tx = t % 16;
    int acc[2][2] = {{0, 0}, {0, 0}};
    const int lr = t / 8, lq = t % 8;                                // staging: row lr, uint4 lq of the 32-word chunk
    for (int k0 = 0; k0 < words4; k0 += kIdolTile) {
        const int kw = k0 + lq * 4;
        uint4 va = make_uint4(0, 0, 0, 0), vb = make_uint4(0, 0, 0, 0);
        if (kw < words4) {
            if (i0 + lr < n) va = *reinterpret_cast<const uint4 *>(bits + (size_t)(i0 + lr) * words4 + kw);
            if (j0 + lr < n) vb = *reinterpret_cast<const uint4 *>(bits + (size_t)(j0 + lr) * words4 + kw);
        }
        sa[lr][lq * 4] = va.x; sa[lr][lq * 4 + 1] = va.y; sa[lr][lq * 4 + 2] = va.z; sa[lr][lq * 4 + 3] = va.w;
        sb[lr][lq * 4] = vb.x; sb[lr][lq * 4 + 1] = vb.y; sb[lr][lq * 4 + 2] = vb.z; sb[lr][lq * 4 + 3] = vb.w;
        __syncthreads();
#pragma unroll 8
        for (int k = 0; k < kIdolTile; ++k) {
            const unsigned a0 = sa[ty][k], a1 = sa[ty + 16][k], b0 = sb[tx][k], b1 = sb[tx + 16][k];
            acc[0][0] += __popc(a0 & b0);
            acc[0][1] += __popc(a0 & b1);
            acc[1][0] += __popc(a1 & b0);
            acc[1][1] += __popc(a1 & b1);
        }
        __syncthreads();
    }
    if (t < kIdolTile) sp[t] = sq[t] = 0u;
    __syncthreads();
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int b = 0; b < 2; ++b) {
            const int i = i0 + ty + 16 * a, j = j0 + tx + 16 * b;
            if (i < n && j < n && j > i) {
                const int inter = acc[a][b], uni = popc[i] + popc[j] - inter;
                const float iou = __fdiv_rn(__fadd_rn((float)inter, 1e-6f), __fadd_rn((float)uni, 1e-6f));
                const unsigned bit = 1u << (tx + 16 * b);
                if (iou > thr_pre) atomicOr(&sp[ty + 16 * a], bit);
                if (iou >= thr_post) atomicOr(&sq[ty + 16 * a], bit);
            }
        }
    __syncthreads();
    if (t < kIdolTile && i0 + t < n) {
        pre[(size_t)(i0 + t) * halves + blockIdx.x] = sp[t];
        post[(size_t)(i0 + t) * halves + blockIdx.x] = sq[t];
    }
}

// One warp: the mask NMS over the n = count rows in order; kept[0 .. k) the kept rows, *kept_count = k.
__global__ void __launch_bounds__(32) idol_nms(const unsigned long long *__restrict__ pre, const int *__restrict__ count,
                                               int n_cap, int *__restrict__ kept, int *__restrict__ kept_count)
{
    __shared__ int order[kIdolMaxRows];
    const int n = min(*count, n_cap);
    for (int i = threadIdx.x; i < n; i += 32) order[i] = i;
    __syncwarp();
    const int k = n > 0 ? nms_sweep(pre, n, order) : 0;
    __syncwarp();
    for (int i = threadIdx.x; i < k; i += 32) kept[i] = order[i];
    if (threadIdx.x == 0) *kept_count = k;
}

// One CTA per memo column c < live: M[c] = the slot's EMA embedding, or with long_match the weighted mean of its ring,
// sum_l w_l e_l / sum_l w_l oldest first, w_l = score_l (+ tw[len - 1][l] with the temporal weight).
__global__ void __launch_bounds__(kIdolThreads) idol_memo(const int *__restrict__ state, const float *__restrict__ embed,
                                                          const float *__restrict__ ring_e, const float *__restrict__ ring_s,
                                                          const float *__restrict__ tw, int T, int L, int D,
                                                          int long_match, float *__restrict__ M)
{
    const int c = blockIdx.x;
    if (c >= state[0]) return;
    const int slot = state[kIdolHeader + c];
    if (!long_match) {
        for (int d = threadIdx.x; d < D; d += kIdolThreads) M[(size_t)c * D + d] = embed[(size_t)slot * D + d];
        return;
    }
    __shared__ float w[kIdolMaxMemory], wsum;
    const int len = state[kIdolHeader + 4 * T + slot];
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int l = 0; l < len; ++l) {
            float wl = ring_s[(size_t)slot * L + l];
            if (tw) wl = __fadd_rn(wl, tw[(len - 1) * L + l]);
            w[l] = wl;
            s = __fadd_rn(s, wl);
        }
        wsum = s;
    }
    __syncthreads();
    const float *e = ring_e + (size_t)slot * L * D;
    for (int d = threadIdx.x; d < D; d += kIdolThreads) {
        float acc = 0.f;
        for (int l = 0; l < len; ++l) acc = __fadd_rn(acc, __fmul_rn(e[(size_t)l * D + d], w[l]));
        M[(size_t)c * D + d] = __fdiv_rn(acc, wsum);
    }
}

// feats[i, c] = E[rows[kept[i]]] . M[c] for i < k, c < live = *cols, fp32, in 32 x 32 tiles (row stride T).  Nothing
// when the error word *err is set.  Shared by both trackers (msda_qdtrack.cuh).
__global__ void __launch_bounds__(kIdolThreads) idol_feats(const float *__restrict__ embeds, const int *__restrict__ rows,
                                                           const int *__restrict__ kept, const int *__restrict__ kept_count,
                                                           const int *__restrict__ cols, const int *__restrict__ err,
                                                           const float *__restrict__ M, int T, int D,
                                                           float *__restrict__ F)
{
    const int k = *kept_count, live = *cols;
    const int i0 = blockIdx.y * kIdolTile, c0 = blockIdx.x * kIdolTile, t = threadIdx.x;
    if (i0 >= k || c0 >= live || *err) return;
    __shared__ float sa[kIdolTile][kIdolTile + 1], sb[kIdolTile][kIdolTile + 1];
    __shared__ const float *arow[kIdolTile];
    if (t < kIdolTile) arow[t] = i0 + t < k ? embeds + (size_t)rows[kept[i0 + t]] * D : nullptr;
    __syncthreads();
    const int ty = t / 16, tx = t % 16;
    float acc[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
    for (int d0 = 0; d0 < D; d0 += kIdolTile) {
        for (int e = t; e < kIdolTile * kIdolTile; e += kIdolThreads) {
            const int r = e / kIdolTile, dd = e % kIdolTile, d = d0 + dd;
            sa[r][dd] = arow[r] && d < D ? arow[r][d] : 0.f;
            sb[r][dd] = c0 + r < live && d < D ? M[(size_t)(c0 + r) * D + d] : 0.f;
        }
        __syncthreads();
#pragma unroll 8
        for (int dd = 0; dd < kIdolTile; ++dd) {
            const float a0 = sa[ty][dd], a1 = sa[ty + 16][dd], b0 = sb[tx][dd], b1 = sb[tx + 16][dd];
            acc[0][0] = fmaf(a0, b0, acc[0][0]);
            acc[0][1] = fmaf(a0, b1, acc[0][1]);
            acc[1][0] = fmaf(a1, b0, acc[1][0]);
            acc[1][1] = fmaf(a1, b1, acc[1][1]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int b = 0; b < 2; ++b) {
            const int i = i0 + ty + 16 * a, c = c0 + tx + 16 * b;
            if (i < k && c < live) F[(size_t)i * T + c] = acc[a][b];
        }
}

__device__ __forceinline__ float idol_block_max(float v, float *red) {
    for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(kFullMask, v, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    v = red[0];
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) v = fmaxf(v, red[w]);
    __syncthreads();
    return v;
}

__device__ __forceinline__ float idol_block_sum(float v, float *red) {
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(kFullMask, v, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    v = red[0];
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) v += red[w];
    __syncthreads();
    return v;
}

// CTAs 0 .. n_cap - 1: row i's max and sum of exp(f - max) over the live = *cols columns (softmax over the memo); CTAs
// n_cap + c: column c's over the kept rows (softmax over the detections).  stat[2 x] = (max, sum).  Nothing when the
// error word *err is set.  Shared by both trackers.
__global__ void __launch_bounds__(kIdolThreads) idol_softmax_stats(const float *__restrict__ F,
                                                                   const int *__restrict__ kept_count,
                                                                   const int *__restrict__ cols,
                                                                   const int *__restrict__ err, int n_cap, int T,
                                                                   float *__restrict__ rstat, float *__restrict__ cstat)
{
    __shared__ float red[kIdolThreads / 32];
    const int k = *kept_count, live = *cols, b = blockIdx.x;
    if (*err) return;
    const bool row = b < n_cap;
    const int x = row ? b : b - n_cap, len = row ? live : k;
    if (x >= (row ? k : live) || len == 0) return;
    const float *base = row ? F + (size_t)x * T : F + x;
    const size_t stride = row ? 1 : (size_t)T;
    float m = -INFINITY;
    for (int e = threadIdx.x; e < len; e += kIdolThreads) m = fmaxf(m, base[e * stride]);
    m = idol_block_max(m, red);
    float s = 0.f;
    for (int e = threadIdx.x; e < len; e += kIdolThreads) s += expf(base[e * stride] - m);
    s = idol_block_sum(s, red);
    if (threadIdx.x == 0) {
        float *out = row ? rstat + 2 * x : cstat + 2 * x;
        out[0] = m;
        out[1] = s;
    }
}

// rank of `flag` among the block's set flags in thread order, and their total (every thread).  warp_tot: 32 ints.
__device__ __forceinline__ int idol_rank(bool flag, int *warp_tot, int &total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned b = __ballot_sync(kFullMask, flag);
    if (lane == 0) warp_tot[warp] = __popc(b);
    __syncthreads();
    int before = 0;
    total = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) {
        if (w < warp) before += warp_tot[w];
        total += warp_tot[w];
    }
    __syncthreads();
    return before + __popc(b & ((1u << lane) - 1u));
}

// The block's largest key (every thread).
__device__ __forceinline__ unsigned long long idol_block_max_u64(unsigned long long v, unsigned long long *red) {
    for (int o = 16; o; o >>= 1) {
        const unsigned long long u = __shfl_xor_sync(kFullMask, v, o);
        v = u > v ? u : v;
    }
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    v = red[0];
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) v = red[w] > v ? red[w] : v;
    __syncthreads();
    return v;
}

// One CTA of 1024 threads (thread t: kept row t and memo column t): the greedy assignment, the new ids, the backdrops,
// the outputs, and the tracklets' bookkeeping (expiry, slots for the new ones, the memo order).  Leaves the state as it
// was when it is flagged, or would be after this frame (kIdolOverflow, set here: more live tracklets than slots).
__global__ void __launch_bounds__(kIdolAssignThreads) idol_assign(
    const float *__restrict__ F, const float *__restrict__ rstat, const float *__restrict__ cstat,
    const int *__restrict__ kept, const int *__restrict__ kept_count, const int *__restrict__ count,
    const float *__restrict__ scores, const unsigned long long *__restrict__ post, int n_cap, int T, IdolParams p,
    int *__restrict__ state, int *__restrict__ ids, int *__restrict__ tracked, int *__restrict__ tracked_count,
    int *__restrict__ row_slot)
{
    __shared__ int s_id[kIdolMaxRows], s_mcol[kIdolMaxRows], s_colid[kIdolMaxTracklets], s_ef[kIdolMaxTracklets];
    __shared__ int s_taken[kIdolMaxTracklets], s_used[kIdolMaxTracklets], s_newslot[kIdolMaxTracklets];
    __shared__ int s_order[kIdolMaxTracklets], warp_tot[32];
    __shared__ unsigned long long s_hit[kIdolMaxRows / 64], red[32];
    __shared__ float fred[32];
    const int t = threadIdx.x;
    const int n = min(*count, n_cap), k = *kept_count, live = state[0], next = state[1], bad = state[2];
    int *order = state + kIdolHeader, *sid = order + T, *last = sid + T, *exist = last + T;
    const int my_slot = t < live ? order[t] : -1;
    for (int r = t; r < n_cap; r += kIdolAssignThreads) {
        ids[r] = -3;
        tracked[r] = -1;
    }
    if (t < live) {
        s_colid[t] = sid[my_slot];
        s_ef[t] = exist[my_slot];
        s_taken[t] = 0;
    }
    if (t < k) { s_id[t] = -2; s_mcol[t] = -1; }
    if (t < kIdolMaxRows / 64) s_hit[t] = 0ull;
    __syncthreads();

    if (live > 0 && !bad) {
        float cmax = 0.f, csum = 1.f;
        if (t < live) { cmax = cstat[2 * t]; csum = cstat[2 * t + 1]; }
        const float ef = t < live ? (float)s_ef[t] : 0.f;
        for (int i = 0; i < k; ++i) {
            float s = 0.f;
            if (t < live && !s_taken[t]) {
                const float f = F[(size_t)i * T + t];
                const float d2t = __fdiv_rn(expf(f - rstat[2 * i]), rstat[2 * i + 1]);
                const float t2d = __fdiv_rn(expf(f - cmax), csum);
                s = __fmul_rn(__fadd_rn(d2t, t2d), 0.5f);
            }
            const bool in_p = t < live && s > 0.5f;
            const int np = __syncthreads_count(in_p);
            float w = s;
            if (p.frame_weight && np > 1) {
                const float sum_ef = idol_block_sum(in_p ? ef : 0.f, fred);       // integers below 2^24: exact
                w = in_p ? __fmul_rn(s, ef) : __fmul_rn(s, __fdiv_rn(sum_ef, (float)np));
            }
            // non-negative floats order as their bits; ties go to the lowest column
            const unsigned long long key =
                t < live ? ((unsigned long long)__float_as_uint(w) << 32) | (0xffffffffu - (unsigned)t) : 0ull;
            const unsigned long long best = idol_block_max_u64(key, red);
            const float conf = __uint_as_float((unsigned)(best >> 32));
            const int j = (int)(0xffffffffu - (unsigned)best);
            if (t == 0 && conf > p.match_thr) {
                s_id[i] = s_colid[j];
                s_mcol[i] = j;
                s_taken[j] = 1;
            }
            __syncthreads();
        }
    }

    // new ids in row order
    int m;
    const float thr = live > 0 ? p.addnew_thr : p.init_thr;
    const bool is_new = t < k && s_id[t] == -2 && scores[kept[t]] > thr;
    const int new_rank = idol_rank(is_new, warp_tot, m);
    if (is_new) s_id[t] = next + new_rank;

    // backdrops: a row still at -2 with IoU < thr_post against every earlier kept row
    const int W = (n + 63) / 64;
    if (W > 0 && t < (kIdolAssignThreads / W) * W) {
        const int w = t % W, G = kIdolAssignThreads / W;
        unsigned long long acc = 0ull;
        for (int e = t / W; e < k; e += G) acc |= post[(size_t)kept[e] * W + w];
        if (acc) atomicOr(&s_hit[w], acc);
    }
    __syncthreads();
    if (t < k && s_id[t] == -2) {
        const int r = kept[t];
        if (!((s_hit[r >> 6] >> (r & 63)) & 1ull)) s_id[t] = -1;
    }
    __syncthreads();
    if (t < k) ids[kept[t]] = s_id[t];
    int nt;
    const bool is_tracked = t < k && s_id[t] > -1;
    const int tr = idol_rank(is_tracked, warp_tot, nt);
    if (is_tracked) tracked[tr] = kept[t];
    if (t == 0) *tracked_count = nt;

    // the memory's bookkeeping
    const bool matched = t < live && s_taken[t];
    const bool survive = t < live && (matched || p.frame_id - last[my_slot] < p.memo_frames);
    int ns;
    const int sr = idol_rank(survive, warp_tot, ns);
    if (bad || ns + m > T) {
        if (t < n_cap) row_slot[t] = -1;
        if (t == 0 && !bad) atomicOr(&state[2], kIdolOverflow);
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
    if (is_new) s_order[ns + new_rank] = s_newslot[new_rank];
    if (t < n_cap)
        row_slot[t] = t >= k ? -1 : is_new ? (s_newslot[new_rank] | kIdolNew) : s_mcol[t] >= 0 ? order[s_mcol[t]] : -1;
    __syncthreads();                                               // every read of order[] is done
    if (matched) {
        last[my_slot] = p.frame_id;
        exist[my_slot] += 1;
    }
    if (is_new) {
        const int slot = s_newslot[new_rank];
        sid[slot] = s_id[t];
        last[slot] = p.frame_id;
        exist[slot] = 1;
    }
    if (t < ns + m) order[t] = s_order[t];
    if (t == 0) {
        state[0] = ns + m;
        state[1] = next + m;
    }
}

// One CTA per kept row i with a tracklet: a new one takes e as its embedding and ring; a matched one's embedding becomes
// keep_w * embed + new_w * e, and e and the score are pushed into its rings (the oldest dropped at L).
__global__ void __launch_bounds__(kIdolThreads) idol_update(const float *__restrict__ embeds, const int *__restrict__ rows,
                                                            const float *__restrict__ scores, const int *__restrict__ kept,
                                                            const int *__restrict__ kept_count,
                                                            const int *__restrict__ row_slot, int T, int D, IdolParams p,
                                                            int *__restrict__ state, float *__restrict__ embed,
                                                            float *__restrict__ ring_e, float *__restrict__ ring_s)
{
    const int i = blockIdx.x;
    if (i >= *kept_count) return;
    const int rs = row_slot[i];
    if (rs < 0) return;
    const bool fresh = rs & kIdolNew;
    const int slot = rs & ~kIdolNew, r = kept[i], L = p.L;
    int *len_p = state + kIdolHeader + 4 * T + slot;
    const int len = fresh ? 0 : *len_p;
    const float *e = embeds + (size_t)rows[r] * D;
    float *em = embed + (size_t)slot * D, *re = ring_e + (size_t)slot * L * D, *rsc = ring_s + (size_t)slot * L;
    for (int d = threadIdx.x; d < D; d += kIdolThreads) {
        const float x = e[d];
        em[d] = fresh ? x : tracker_ema(p.keep_w, em[d], p.new_w, x);
        if (len < L) {
            re[(size_t)len * D + d] = x;
        } else {
            for (int l = 1; l < L; ++l) re[(size_t)(l - 1) * D + d] = re[(size_t)l * D + d];
            re[(size_t)(L - 1) * D + d] = x;
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        if (len < L) {
            rsc[len] = scores[r];
        } else {
            for (int l = 1; l < L; ++l) rsc[l - 1] = rsc[l];
            rsc[L - 1] = scores[r];
        }
        *len_p = len < L ? len + 1 : L;
    }
}

}  // namespace msda
