// msda_nms.cuh -- the greedy NMS of torchvision's CUDA kernel (ops/cuda/nms_kernel.cu) on boxes already in score order
// in shared memory, shared by the detection post-processor (detpost_select<true>) and the video trackers' detection
// selection (trackpost_select), both in msda_detpost.cuh: the n x ceil(n/64) IoU bitmask, then the sweep in one warp.
// Every multiply and add is written with __fmul_rn / __fadd_rn / __fsub_rn so that nvcc does not contract it into an FMA
// (DESIGN.md section 3.13).
#pragma once

#include "msda_common.cuh"

namespace msda {

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

// mask[i * W + w], W = ceil(n / 64): bit j - 64 w is set when IoU(sbox[i], sbox[j]) > thr and j > i.  Every thread of the
// block calls it; the caller puts a barrier between it and nms_sweep.
template <int Threads>
__device__ __forceinline__ void nms_bitmask(const float4 *sbox, int n, float thr, unsigned long long *mask)
{
    const int W = (n + 63) / 64;
    for (int it = threadIdx.x; it < n * W; it += Threads) {
        const int i = it / W, w = it - i * W;
        unsigned long long bits = 0;
        const int j0 = max(w * 64, i + 1), j1 = min(w * 64 + 64, n);
        if (j0 < j1) {
            const float4 a = sbox[i];
            for (int j = j0; j < j1; ++j)
                if (dp_iou_above(a, sbox[j], thr)) bits |= 1ull << (j - w * 64);
        }
        mask[it] = bits;
    }
}

// The greedy sweep, by the 32 lanes of one warp (n <= 1024: lane l holds removed-word l).  order[0 .. n) holds the
// candidates in score order; on return order[0 .. k) holds the kept ones in score order, and every lane gets k.
__device__ __forceinline__ int nms_sweep(const unsigned long long *mask, int n, int *order)
{
    const int lane = threadIdx.x & 31, W = (n + 63) / 64;
    unsigned long long removed = 0;
    int k = 0;
    for (int i = 0; i < n; ++i) {
        const unsigned long long word = __shfl_sync(0xffffffffu, removed, i >> 6);
        if (!((word >> (i & 63)) & 1ull)) {
            const int qi = order[i];            // read before any lane overwrites slot k <= i
            __syncwarp();
            if (lane == 0) order[k] = qi;
            ++k;
            if (lane < W) removed |= mask[(size_t)i * W + lane];
        }
        __syncwarp();
    }
    return k;
}

}  // namespace msda
