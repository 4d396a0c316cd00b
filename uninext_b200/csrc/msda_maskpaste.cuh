// msda_maskpaste.cuh -- mask pasting for UNINEXT inference (DESIGN.md section 3.12, row f-5): stride-s mask logits
// [I, Hs, Ws] -> full-resolution masks [I, H_out, W_out] in one pass.
//
// The reference runs, per image or per track (uninext_img.py:474-479 + ddetrs.py:1060-1064, uninext_vid.py:620-622,
// 1187-1192, 1264-1266, 1335-1337, 1428-1431):
//     F.interpolate(logits, size=(s*Hs, s*Ws), mode="bilinear", align_corners=False).sigmoid() [> thr]
//       [:, :, :h, :w]  ->  F.interpolate(., size=(H_out, W_out), mode="nearest")
// and writes every intermediate at the padded input resolution.  Nearest selection and the threshold commute, so output
// pixel (Y, X) of instance i is
//     y' = min((int)floorf(Y * (float)h / H_out), h - 1)                                     (x' likewise)
//     bilinear of the logits at padded pixel (y', x') with upsample_bilinear2d's align_corners=False source indices
//     p = 1 / (1 + exp(-v)) in fp32;  out = p, or (p > thr) as a 0/1 byte.
// Here that is a pure gather: a thread owns 8 consecutive output columns of one row, resolves their source taps once
// (registers) and loops over a chunk of instances, one 8-byte store (binary) or two 16-byte stores (probabilities) per
// instance.  Nothing else is written; the logits (27 MB for 100 x 200 x 336) stay in L2.  16 columns per thread took
// 1.3-1.6x as long on an H100 (DESIGN.md section 3.12): 170-190 registers, one block per SM.
#pragma once

#include "msda_common.cuh"

namespace msda {

constexpr int kMpCols = 8;                      // output columns per thread
constexpr int kMpGroups = 16;                   // column groups per block: 128 columns; a warp = 16 groups x 2 rows
constexpr int kMpRows = 16;                     // output rows per block, one per thread row
constexpr int kMpThreads = kMpGroups * kMpRows;
constexpr int kMpInst = 8;                      // instances per thread and grid-z step

// Output coordinate o -> nearest pixel of the crop (upsample_nearest2d: floorf(o * scale), clamped) -> source taps of
// that padded pixel (upsample_bilinear2d, align_corners=False: src = max(scale * (c + 0.5) - 0.5, 0)).
__device__ __forceinline__ void mp_source(int o, float near_scale, int crop, float lin_scale, int n, int &i0, int &i1,
                                          float &l1) {
    const int c = min((int)floorf((float)o * near_scale), crop - 1);
    float src = lin_scale * ((float)c + 0.5f) - 0.5f;
    src = src < 0.f ? 0.f : src;
    i0 = (int)src;
    i1 = i0 + (i0 < n - 1 ? 1 : 0);
    l1 = src - (float)i0;
}

// The probability at one output pixel: upsample_bilinear2d's expression and order over the taps t0[0], t0[dx], t1[0],
// t1[dx] (t0, t1 = the source rows at the pixel's first tap column, hy0 = 1 - ly), then torch's fp32 sigmoid.  mask_paste
// and the RLE pass (msda_maskrle.cuh) both evaluate pixels through this, so their bits cannot differ.
__device__ __forceinline__ float mp_prob(const float *t0, const float *t1, int dx, float lx, float hy0, float ly) {
    const float w0 = 1.f - lx;
    const float v = hy0 * (w0 * __ldg(t0) + lx * __ldg(t0 + dx)) + ly * (w0 * __ldg(t1) + lx * __ldg(t1 + dx));
    return 1.f / (1.f + expf(-v));
}

// block: (kMpGroups, kMpRows); grid: (column tiles, row tiles, instance chunks of kMpInst; grid-z strides over I).
// out: uint8 [I, out_h, out_w] (BINARY) or fp32.  VEC: out is 16-byte aligned and out_w is a multiple of the store
// vector (8 bytes / 4 floats), so a vector is either wholly inside a row or wholly past its end.
template <bool BINARY, bool VEC>
__global__ void __launch_bounds__(kMpThreads)
mask_paste(const float *__restrict__ logits, long long I, int Hs, int Ws, int crop_h, int crop_w, int out_h, int out_w,
           float near_y, float near_x, float lin_y, float lin_x, float threshold, void *__restrict__ out)
{
    const int X0 = (blockIdx.x * kMpGroups + threadIdx.x) * kMpCols;
    const int Y = blockIdx.y * kMpRows + threadIdx.y;
    if (X0 >= out_w || Y >= out_h) return;
    int y0, y1;
    float ly;
    mp_source(Y, near_y, crop_h, lin_y, Hs, y0, y1, ly);
    const float hy0 = 1.f - ly;
    int x0[kMpCols], dx[kMpCols];               // taps x0 and x0 + dx (dx = 0 at the last column)
    float lx[kMpCols];
#pragma unroll
    for (int k = 0; k < kMpCols; ++k) {
        int x1;
        mp_source(min(X0 + k, out_w - 1), near_x, crop_w, lin_x, Ws, x0[k], x1, lx[k]);
        dx[k] = x1 - x0[k];
    }
    const size_t plane = (size_t)Hs * Ws, out_plane = (size_t)out_h * out_w, out_row = (size_t)Y * out_w + X0;
    for (long long ib = (long long)blockIdx.z * kMpInst; ib < I; ib += (long long)gridDim.z * kMpInst) {
        const int n = (int)min((long long)kMpInst, I - ib);
#pragma unroll 1
        for (int j = 0; j < n; ++j) {
            const long long i = ib + j;
            const float *base = logits + i * plane;
            // Opaque to the optimiser: otherwise it strength-reduces the 64 tap addresses into 64-bit pointers carried
            // across instances (128 registers, spills).  Here each tap is one IMAD.WIDE off the instance's base.
            asm volatile("" : "+l"(base));
            const float *r0 = base + (size_t)y0 * Ws, *r1 = base + (size_t)y1 * Ws;
            float p[kMpCols];
#pragma unroll
            for (int k = 0; k < kMpCols; ++k) p[k] = mp_prob(r0 + x0[k], r1 + x0[k], dx[k], lx[k], hy0, ly);
            const size_t o = (size_t)i * out_plane + out_row;
            if constexpr (BINARY) {
                uint8_t *dst = static_cast<uint8_t *>(out) + o;
                if constexpr (VEC) {
                    unsigned w[2] = {0u, 0u};
#pragma unroll
                    for (int k = 0; k < kMpCols; ++k) w[k / 4] |= (p[k] > threshold ? 1u : 0u) << (8 * (k % 4));
                    *reinterpret_cast<uint2 *>(dst) = make_uint2(w[0], w[1]);
                } else {
#pragma unroll
                    for (int k = 0; k < kMpCols; ++k)
                        if (X0 + k < out_w) dst[k] = p[k] > threshold ? 1 : 0;
                }
            } else {
                float *dst = static_cast<float *>(out) + o;
                if constexpr (VEC) {
#pragma unroll
                    for (int q = 0; q < kMpCols / 4; ++q)
                        if (X0 + 4 * q < out_w)
                            *reinterpret_cast<float4 *>(dst + 4 * q) = make_float4(p[4 * q], p[4 * q + 1], p[4 * q + 2], p[4 * q + 3]);
                } else {
#pragma unroll
                    for (int k = 0; k < kMpCols; ++k)
                        if (X0 + k < out_w) dst[k] = p[k];
                }
            }
        }
    }
}

}  // namespace msda
