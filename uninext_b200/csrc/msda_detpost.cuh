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
// Every multiply and add is written with __fmul_rn / __fadd_rn / __fsub_rn so that nvcc does not contract it into an
// FMA: the contract is this uncontracted arithmetic (DESIGN.md section 3.13).
#pragma once

#include "msda_common.cuh"
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
__device__ __forceinline__ float4 dp_xyxy(const float *b) {
    const float cx = __ldg(b), cy = __ldg(b + 1), hw = __fmul_rn(0.5f, __ldg(b + 2)), hh = __fmul_rn(0.5f, __ldg(b + 3));
    return make_float4(__fsub_rn(cx, hw), __fsub_rn(cy, hh), __fadd_rn(cx, hw), __fadd_rn(cy, hh));
}

// The expression of torchvision's devIoU (ops/cuda/nms_kernel.cu) with every operation rounded once.  torchvision's
// build may contract parts of it into FMAs, so the two can differ in the last bit of the IoU.
__device__ __forceinline__ bool dp_iou_above(float4 a, float4 b, float thr) {
    const float left = fmaxf(a.x, b.x), right = fminf(a.z, b.z);
    const float top = fmaxf(a.y, b.y), bottom = fminf(a.w, b.w);
    const float width = fmaxf(__fsub_rn(right, left), 0.f), height = fmaxf(__fsub_rn(bottom, top), 0.f);
    const float inter = __fmul_rn(width, height);
    const float sa = __fmul_rn(__fsub_rn(a.z, a.x), __fsub_rn(a.w, a.y));
    const float sb = __fmul_rn(__fsub_rn(b.z, b.x), __fsub_rn(b.w, b.y));
    return __fdiv_rn(inter, __fsub_rn(__fadd_rn(sa, sb), inter)) > thr;
}

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
        const int W = (Q + 63) / 64;
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
        for (int it = tid; it < Q * W; it += kDpThreads) {
            const int i = it / W, w = it - i * W;
            unsigned long long bits = 0;
            const int j0 = max(w * 64, i + 1), j1 = min(w * 64 + 64, Q);
            if (j0 < j1) {
                const float4 a = sbox[i];
                for (int j = j0; j < j1; ++j)
                    if (dp_iou_above(a, sbox[j], nms_iou)) bits |= 1ull << (j - w * 64);
            }
            mask[it] = bits;
        }
        __syncthreads();
        if (tid < 32) {                         // greedy sweep: lane l holds removed-word l (W <= 16)
            unsigned long long removed = 0;
            int k = 0;
            for (int i = 0; i < Q; ++i) {
                const unsigned long long word = __shfl_sync(0xffffffffu, removed, i >> 6);
                if (!((word >> (i & 63)) & 1ull)) {
                    const int qi = s_keep[i];   // read before any lane overwrites slot k <= i
                    __syncwarp();
                    if (tid == 0) s_keep[k] = qi;
                    ++k;
                    if (tid < W) removed |= mask[(size_t)i * W + tid];
                }
                __syncwarp();
            }
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

}  // namespace msda
