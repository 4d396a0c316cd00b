// msda_detpost.cuh -- detection post-processing for UNINEXT inference (DESIGN.md section 3.13, row f-6): grounding
// logits [B, Q, T] -> class scores -> class-aware NMS -> top-k boxes, scores, labels and query indices, on the device.
//
// The reference runs, per image in a Python loop (uninext_img.py:393-472, uninext_vid.py:1092-1197):
//     convert_grounding_to_od_logits (a Python loop over the classes, one host-to-device copy each)
//     prob = sigmoid(logits) [; prob = sqrt(prob * sigmoid(iou))]
//     [OTA: score, class = prob.max(1); batched_nms(cxcywh_to_xyxy(boxes), score, class, 0.7); prob = prob[keep]]
//     topk(prob.flatten(), min(max_num_inst, K*C)); boxes cxcywh -> xyxy, scaled by (w, h)
// Here that is two launches for the whole batch, whatever B, Q and C:
//   detpost_scores   one warp per query: the [T] row in shared memory, a lane per class (CSR positive map), the fp32
//                    mean and sigmoid exactly as torch forms them, prob [B, Q, C] and the per-query max / argmax to the
//                    workspace;
//   detpost_select   one CTA per image: [NMS: stable rank sort of the Q maxima, the Q x ceil(Q/64) IoU bitmask in shared
//                    memory, the greedy sweep in one warp,] then a radix select of the top `count` of the K*C candidates
//                    on a unique 64-bit key (value, flat index), a bitonic sort of those, and the outputs.
// The video trackers' per-frame selection (uninext_vid.py:1224-1250 MOT, :1380-1415 VIS; DESIGN.md section 3.17) is two
// launches as well: detpost_scores, then
//   trackpost_select one CTA per frame: the candidates max_score > score_thres compacted in query order, [none: the
//                    query of the largest max_score; else: the stable rank sort of the candidates, the bitmask and the
//                    sweep (msda_nms.cuh) on the compacted set,] then the kept queries in keep order.
// Every multiply and add is written with __fmul_rn / __fadd_rn / __fsub_rn so that nvcc does not contract it into an
// FMA: the contract is this uncontracted arithmetic (DESIGN.md section 3.13).
#pragma once

#include "msda_common.cuh"
#include "msda_nms.cuh"
#include "msda_topk.cuh"

namespace msda {

constexpr int kDpScoreWarps = 8;                // queries per block of detpost_scores
constexpr int kDpThreads = 1024;                // threads of detpost_select (one CTA per image)
constexpr int kDpMaxQ = 1024, kDpMaxT = 256, kDpMaxC = 4096;
constexpr int kDpSmemSort = 2048;               // selected candidates sorted in shared memory; more sort in the workspace

// torch's fp32 sigmoid (UnarySpecialOpsKernel.cu): 1 / (1 + exp(-x)), IEEE division, accurate expf.
__device__ __forceinline__ float dp_sigmoid(float x) { return 1.f / (1.f + expf(-x)); }

// block: kDpScoreWarps warps, warp w -> query blockIdx.x * kDpScoreWarps + w; grid.y = image.
__global__ void __launch_bounds__(kDpScoreWarps * 32)
detpost_scores(const float *__restrict__ box_cls, const float *__restrict__ iou_pred, const int *__restrict__ class_start,
               const int *__restrict__ tokens, int Q, int T, int C, float *__restrict__ prob, float *__restrict__ qmax,
               int *__restrict__ qarg)
{
    __shared__ float row[kDpScoreWarps][kDpMaxT];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q = blockIdx.x * kDpScoreWarps + warp;
    if (q >= Q) return;                         // whole warps leave; only __syncwarp below
    const size_t bq = (size_t)blockIdx.y * Q + q;
    const float *src = box_cls + bq * T;
    for (int t = lane; t < T; t += 32) row[warp][t] = __ldg(src + t);
    __syncwarp();
    const float s_iou = iou_pred ? dp_sigmoid(__ldg(iou_pred + bq)) : 0.f;
    float *out = prob + bq * C;
    float best = -1.f;                          // every probability is >= 0
    int barg = C;
    for (int c = lane; c < C; c += 32) {
        const int j0 = __ldg(class_start + c), j1 = __ldg(class_start + c + 1);
        float sum = 0.f;                        // torch's mean: fp32 sum, then times (float)1/n (MeanOps::project)
        for (int j = j0; j < j1; ++j) {
            const int t = __ldg(tokens + j);
            sum = __fadd_rn(sum, (unsigned)t < (unsigned)T ? row[warp][t] : __int_as_float(0x7fffffff));
        }
        const float x = __fmul_rn(sum, 1.f / (float)(j1 - j0));
        float p = dp_sigmoid(x);
        if (iou_pred) p = sqrtf(__fmul_rn(p, s_iou));
        out[c] = p;
        if (p > best) { best = p; barg = c; }   // a lane's classes ascend: the first maximum stays
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {    // torch.max(dim): the lowest index among equal maxima
        const float ob = __shfl_xor_sync(0xffffffffu, best, off);
        const int oa = __shfl_xor_sync(0xffffffffu, barg, off);
        if (ob > best || (ob == best && oa < barg)) { best = ob; barg = oa; }
    }
    if (lane == 0) { qmax[bq] = best; qarg[bq] = barg; }
}

// box_cxcywh_to_xyxy: (x_c - 0.5 * w, y_c - 0.5 * h, x_c + 0.5 * w, y_c + 0.5 * h), each operation rounded once.
__device__ __forceinline__ float4 dp_xyxy(float cx, float cy, float w, float h) {
    const float hw = __fmul_rn(0.5f, w), hh = __fmul_rn(0.5f, h);
    return make_float4(__fsub_rn(cx, hw), __fsub_rn(cy, hh), __fadd_rn(cx, hw), __fadd_rn(cy, hh));
}
__device__ __forceinline__ float4 dp_xyxy(const float *b) { return dp_xyxy(__ldg(b), __ldg(b + 1), __ldg(b + 2), __ldg(b + 3)); }

__device__ __forceinline__ float dp_block_max(float v, float *red) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, off));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    v = red[0];
    for (int w = 1; w < kDpThreads / 32; ++w) v = fmaxf(v, red[w]);
    __syncthreads();
    return v;
}

// One CTA per image (grid = B).  Dynamic shared memory (NMS only): float4 boxes[Q] in score order, then the bitmask
// u64 mask[Q][ceil(Q/64)] (bit j of row i: IoU(i, j) > nms_iou, j > i).  sort_ws: [B, sort_cap] u64 when the selected
// count exceeds kDpSmemSort (sort_cap = 0 otherwise).
template <bool NMS>
__global__ void __launch_bounds__(kDpThreads, 1)
detpost_select(const float *__restrict__ box_pred, const int *__restrict__ image_sizes, const float *__restrict__ prob,
               const float *__restrict__ qmax, const int *__restrict__ qarg, int Q, int C, float nms_iou, int max_inst,
               long long sort_cap, unsigned long long *__restrict__ sort_ws, float *__restrict__ scores,
               int *__restrict__ labels, int *__restrict__ query_index, float *__restrict__ boxes, int *__restrict__ count)
{
    extern __shared__ float4 dp_dyn[];
    __shared__ int s_keep[kDpMaxQ];             // NMS: kept queries in score order
    __shared__ float s_red[kDpThreads / 32];
    __shared__ unsigned s_hist[256];
    __shared__ unsigned long long s_sort[kDpSmemSort];
    __shared__ int s_K, s_digit;
    __shared__ unsigned s_rem, s_bucket, s_n;
    const int b = blockIdx.x, tid = threadIdx.x;
    const float *bp = box_pred + (size_t)b * Q * 4;
    const float *pr = prob + (size_t)b * Q * C;
    int K = Q;
    if constexpr (NMS) {
        float4 *sbox = dp_dyn;
        unsigned long long *mask = reinterpret_cast<unsigned long long *>(sbox + Q);
        const float *qm = qmax + (size_t)b * Q;
        // batched_nms's coordinate trick: m = boxes.max(), offset = class * (m + 1) added to each coordinate
        float m = -INFINITY;
        for (int i = tid; i < Q; i += kDpThreads) {
            const float4 x = dp_xyxy(bp + 4 * i);
            m = fmaxf(m, fmaxf(fmaxf(x.x, x.y), fmaxf(x.z, x.w)));
        }
        m = dp_block_max(m, s_red);
        const float m1 = __fadd_rn(m, 1.f);
        // stable descending sort by rank counting: rank = #{j : s_j > s_i, or s_j == s_i and j < i}
        for (int i = tid; i < Q; i += kDpThreads) {
            const float si = qm[i];
            int rank = 0;
            for (int j = 0; j < Q; ++j) {
                const float sj = qm[j];
                rank += (sj > si || (sj == si && j < i)) ? 1 : 0;
            }
            const float4 x = dp_xyxy(bp + 4 * i);
            const float off = __fmul_rn((float)qarg[(size_t)b * Q + i], m1);
            sbox[rank] = make_float4(__fadd_rn(x.x, off), __fadd_rn(x.y, off), __fadd_rn(x.z, off), __fadd_rn(x.w, off));
            s_keep[rank] = i;                   // s_keep holds the sorted order until the sweep compacts it
        }
        __syncthreads();
        nms_bitmask<kDpThreads>(sbox, Q, nms_iou, mask);
        __syncthreads();
        if (tid < 32) {
            const int k = nms_sweep(mask, Q, s_keep);
            if (tid == 0) s_K = k;
        }
        __syncthreads();
        K = s_K;
    }
    // top-k over the K*C candidates (kept rank r, class c), flat index r * C + c
    const unsigned N = (unsigned)K * (unsigned)C;
    const unsigned cnt = min((unsigned)max_inst, N);
    auto key_of = [&](unsigned f) {
        const unsigned r = f / (unsigned)C, c = f - r * (unsigned)C;
        const int qi = NMS ? s_keep[r] : (int)r;
        return dp_key(pr[(size_t)qi * C + c], f);
    };
    // the cnt-th smallest key; the candidate keys are unique (flat index in the low word), so exactly cnt are <= thr
    const unsigned long long thr = block_radix_threshold<kDpThreads>(N, cnt, key_of, s_hist, &s_digit, &s_rem, &s_bucket);
    // collect the cnt keys <= thr (in any order), pad to a power of two, bitonic sort ascending
    unsigned P = 1;
    while (P < cnt) P <<= 1;
    unsigned long long *buf = P <= (unsigned)kDpSmemSort ? s_sort : sort_ws + (size_t)b * sort_cap;
    if (tid == 0) s_n = 0;
    __syncthreads();
    for (unsigned f = tid; f < N; f += kDpThreads) {
        const unsigned long long k = key_of(f);
        if (k <= thr) buf[atomicAdd(&s_n, 1u)] = k;
    }
    for (unsigned i = cnt + tid; i < P; i += kDpThreads) buf[i] = ~0ull;
    __syncthreads();
    block_bitonic_sort<kDpThreads>(buf, P);
    // outputs: boxes xyxy then Boxes.scale (x * w, y * h); entries past cnt get the fill values
    const float sh = (float)image_sizes[2 * b], sw = (float)image_sizes[2 * b + 1];
    const size_t o = (size_t)b * max_inst;
    for (int j = tid; j < max_inst; j += kDpThreads) {
        if ((unsigned)j < cnt) {
            const unsigned f = (unsigned)(buf[j] & 0xffffffffull);
            const unsigned r = f / (unsigned)C, c = f - r * (unsigned)C;
            const int qi = NMS ? s_keep[r] : (int)r;
            scores[o + j] = pr[(size_t)qi * C + c];
            labels[o + j] = (int)c;
            query_index[o + j] = qi;
            const float4 x = dp_xyxy(bp + 4 * qi);
            reinterpret_cast<float4 *>(boxes)[o + j] =
                make_float4(__fmul_rn(x.x, sw), __fmul_rn(x.y, sh), __fmul_rn(x.z, sw), __fmul_rn(x.w, sh));
        } else {
            scores[o + j] = 0.f;
            labels[o + j] = -1;
            query_index[o + j] = -1;
            reinterpret_cast<float4 *>(boxes)[o + j] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
    if (tid == 0) count[b] = (int)cnt;
}

// One CTA per frame (grid = B), thread i <-> query i (Q <= kDpThreads).  Dynamic shared memory as detpost_select<true>'s
// for Q queries, of which the n candidates use float4 boxes[n] in score order and the bitmask u64 mask[n][ceil(n/64)].
// pixels: boxes are box_cxcywh_to_xyxy of the cxcywh box scaled by (W, H, W, H) of ori_sizes[b] = (H, W); else the
// normalised cxcywh box as it is.
__global__ void __launch_bounds__(kDpThreads, 1)
trackpost_select(const float *__restrict__ box_pred, const int *__restrict__ ori_sizes, const float *__restrict__ qmax,
                 const int *__restrict__ qarg, int Q, float score_thres, float nms_iou, int pixels,
                 float *__restrict__ scores, int *__restrict__ labels, int *__restrict__ query_index,
                 float *__restrict__ boxes, int *__restrict__ count)
{
    extern __shared__ float4 dp_dyn[];
    __shared__ int s_cand[kDpMaxQ];             // the candidates' queries, ascending (torch.nonzero's order)
    __shared__ float s_cscore[kDpMaxQ];         // and their max_score
    __shared__ int s_order[kDpMaxQ];            // the candidates in score order, then the kept ones
    __shared__ int s_wsum[kDpThreads / 32];
    __shared__ float s_red[kDpThreads / 32];
    __shared__ int s_n, s_K;
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
    const float *bp = box_pred + (size_t)b * Q * 4;
    const float *qm = qmax + (size_t)b * Q;
    const int *qa = qarg + (size_t)b * Q;
    const float mine = tid < Q ? qm[tid] : -INFINITY;
    // block-wide compaction of the candidates in query order: ballot per warp, warp offsets from the warps' counts
    const bool cand = tid < Q && mine > score_thres;
    const unsigned ballot = __ballot_sync(0xffffffffu, cand);
    if (lane == 0) s_wsum[tid >> 5] = __popc(ballot);
    if (tid == 0) s_K = Q;
    __syncthreads();
    int base = 0;
    for (int w = 0; w < (tid >> 5); ++w) base += s_wsum[w];
    if (cand) {
        const int at = base + __popc(ballot & ((1u << lane) - 1u));
        s_cand[at] = tid;
        s_cscore[at] = mine;
    }
    if (tid == kDpThreads - 1) s_n = base + s_wsum[tid >> 5];
    __syncthreads();
    const int n = s_n;
    if (n == 0) {
        // no candidate: the query of the largest max_score, the lowest one on exact ties (qmax is never NaN)
        const float m = dp_block_max(mine, s_red);
        if (tid < Q && mine == m) atomicMin(&s_K, tid);
        __syncthreads();
        if (tid == 0) { s_order[0] = s_K; s_K = 1; }
    } else {
        float4 *sbox = dp_dyn;
        unsigned long long *mask = reinterpret_cast<unsigned long long *>(sbox + Q);
        // batched_nms's coordinate trick on the candidates: m = boxes.max(), offset = class * (m + 1)
        float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
        float m = -INFINITY;
        if (tid < n) {
            x = dp_xyxy(bp + 4 * s_cand[tid]);
            m = fmaxf(fmaxf(x.x, x.y), fmaxf(x.z, x.w));
        }
        m = dp_block_max(m, s_red);
        const float m1 = __fadd_rn(m, 1.f);
        // stable descending sort by rank counting over the candidates in query order
        if (tid < n) {
            const float si = s_cscore[tid];
            int rank = 0;
            for (int j = 0; j < n; ++j) {
                const float sj = s_cscore[j];
                rank += (sj > si || (sj == si && j < tid)) ? 1 : 0;
            }
            const int qi = s_cand[tid];
            const float off = __fmul_rn((float)qa[qi], m1);
            sbox[rank] = make_float4(__fadd_rn(x.x, off), __fadd_rn(x.y, off), __fadd_rn(x.z, off), __fadd_rn(x.w, off));
            s_order[rank] = qi;
        }
        __syncthreads();
        nms_bitmask<kDpThreads>(sbox, n, nms_iou, mask);
        __syncthreads();
        if (tid < 32) {
            const int k = nms_sweep(mask, n, s_order);
            if (tid == 0) s_K = k;
        }
    }
    __syncthreads();
    const int K = s_K;
    // outputs in keep order; entries past K get detpost's fill values
    const size_t o = (size_t)b * Q + tid;
    if (tid < K) {
        const int qi = s_order[tid];
        scores[o] = qm[qi];
        labels[o] = qa[qi];
        query_index[o] = qi;
        const float *src = bp + 4 * qi;
        float4 box;
        if (pixels) {                           // output_boxes[:, 0::2] *= W; output_boxes[:, 1::2] *= H; then to xyxy
            const float sh = (float)ori_sizes[2 * b], sw = (float)ori_sizes[2 * b + 1];
            box = dp_xyxy(__fmul_rn(__ldg(src), sw), __fmul_rn(__ldg(src + 1), sh), __fmul_rn(__ldg(src + 2), sw),
                          __fmul_rn(__ldg(src + 3), sh));
        } else {
            box = make_float4(__ldg(src), __ldg(src + 1), __ldg(src + 2), __ldg(src + 3));
        }
        reinterpret_cast<float4 *>(boxes)[o] = box;
    } else if (tid < Q) {
        scores[o] = 0.f;
        labels[o] = -1;
        query_index[o] = -1;
        reinterpret_cast<float4 *>(boxes)[o] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (tid == 0) count[b] = K;
}

}  // namespace msda
