// msda_flatten.cuh -- the encoder's input preparation of the DINO-style transformer (DESIGN.md section 3.16;
// deformable_transformer_dino.py:181-201): the L pyramid levels, NCHW as input_proj emits them, flattened to the
// [N, S, C] rows the encoder reads, for all levels and all three outputs in one launch.
//   flatten_levels_fwd      one CTA per (32 positions x 32 channels tile, image): src_l and pos_l are read along the
//                           positions (scalar loads: a level's channel rows are 16-byte aligned only when H_l * W_l is a
//                           multiple of 4), transposed through shared memory and written as float4 along the channels;
//                           pos_flat = pos + level_embed[l] (one fp32 add, as the reference); the CTAs of channel tile 0
//                           copy the mask;
//   flatten_levels_bwd      the transpose back, per tile: grad_src_l, grad_pos_l, and the tile's column sums of
//                           grad_pos_flat (the partials of grad_level_embed) written to the workspace;
//   flatten_levels_reduce   grad_level_embed[l, c] = the partials of level l summed in a fixed order: no float atomics,
//                           the same bits on every run.
#pragma once

#include "msda_common.cuh"

namespace msda {

constexpr int kFlTile = 32;                      // positions and channels per tile
constexpr int kFlThreads = 256;

// The pyramid, copied into the kernels' arguments by value: the call reads no host or device level table.
struct FlattenTable {
    int L, C, ctiles;                            // ctiles = ceil(C / kFlTile)
    long long S;                                 // positions per image
    long long hw[kMaxLevels], start[kMaxLevels]; // H_l * W_l and the first flattened position of level l
    int tile0[kMaxLevels + 1];                   // first tile of level l within one image
    int ptile0[kMaxLevels + 1];                  // first 32-position tile of level l (rows of the backward's partials)
};

struct FlattenFwdArgs {
    FlattenTable t;
    const float *src[kMaxLevels], *pos[kMaxLevels];
    const unsigned char *mask[kMaxLevels];
    const float *level_embed;
    float *src_flat, *pos_flat;
    unsigned char *mask_flat;
};

struct FlattenBwdArgs {
    FlattenTable t;
    const float *grad_src_flat, *grad_pos_flat;  // NULL when nothing reads them
    float *grad_src[kMaxLevels], *grad_pos[kMaxLevels];   // entries NULL when not wanted
    float *part;                                 // [N, ptile0[L], C] partials, NULL without grad_level_embed
};

// blockIdx.x -> (level, first position, first channel) of the tile.
__device__ __forceinline__ int fl_tile(const FlattenTable &t, long long &p0, int &c0) {
    int tile = blockIdx.x, l = 0;
    while (l + 1 < t.L && tile >= t.tile0[l + 1]) ++l;
    tile -= t.tile0[l];
    const int pt = tile / t.ctiles;
    p0 = (long long)pt * kFlTile;
    c0 = (tile - pt * t.ctiles) * kFlTile;
    return l;
}

__global__ void __launch_bounds__(kFlThreads)
flatten_levels_fwd(const FlattenFwdArgs a)
{
    __shared__ float ts[kFlTile][kFlTile + 1], tp[kFlTile][kFlTile + 1];     // [channel][position]
    const FlattenTable &t = a.t;
    long long p0;
    int c0;
    const int l = fl_tile(t, p0, c0), n = blockIdx.y, tid = threadIdx.x, C = t.C;
    const long long hw = t.hw[l];
    // NCHW side: a warp reads 32 consecutive positions of one channel
    const int px = tid & 31, cy = tid >> 5;
    const long long img = (long long)n * C * hw;
#pragma unroll
    for (int i = 0; i < kFlTile / 8; ++i) {
        const int c = cy + 8 * i;
        float vs = 0.f, vp = 0.f;
        if (c0 + c < C && p0 + px < hw) {
            const long long o = img + (long long)(c0 + c) * hw + p0 + px;
            vs = __ldg(a.src[l] + o);
            vp = __ldg(a.pos[l] + o);
        }
        ts[c][px] = vs;
        tp[c][px] = vp;
    }
    if (c0 == 0 && tid < kFlTile && p0 + tid < hw)
        a.mask_flat[(long long)n * t.S + t.start[l] + p0 + tid] = a.mask[l][(long long)n * hw + p0 + tid];
    __syncthreads();
    // [N, S, C] side: a thread writes 4 channels of one position
    const int pr = tid >> 3, c4 = (tid & 7) * 4;
    if (p0 + pr < hw && c0 + c4 < C) {
        const float4 e = __ldg(reinterpret_cast<const float4 *>(a.level_embed + (long long)l * C + c0 + c4));
        const long long o = ((long long)n * t.S + t.start[l] + p0 + pr) * C + c0 + c4;
        *reinterpret_cast<float4 *>(a.src_flat + o) = make_float4(ts[c4][pr], ts[c4 + 1][pr], ts[c4 + 2][pr], ts[c4 + 3][pr]);
        *reinterpret_cast<float4 *>(a.pos_flat + o) =
            make_float4(tp[c4][pr] + e.x, tp[c4 + 1][pr] + e.y, tp[c4 + 2][pr] + e.z, tp[c4 + 3][pr] + e.w);
    }
}

__global__ void __launch_bounds__(kFlThreads)
flatten_levels_bwd(const FlattenBwdArgs a)
{
    __shared__ float ts[kFlTile][kFlTile + 1], tp[kFlTile][kFlTile + 1];     // [channel][position], 0 outside
    const FlattenTable &t = a.t;
    long long p0;
    int c0;
    const int l = fl_tile(t, p0, c0), n = blockIdx.y, tid = threadIdx.x, C = t.C;
    const long long hw = t.hw[l];
    const bool want_src = a.grad_src[l] != nullptr, read_pos = a.grad_pos_flat != nullptr;
    const int pr = tid >> 3, c4 = (tid & 7) * 4;
    float4 gs = make_float4(0.f, 0.f, 0.f, 0.f), gp = gs;
    if (p0 + pr < hw && c0 + c4 < C) {
        const long long o = ((long long)n * t.S + t.start[l] + p0 + pr) * C + c0 + c4;
        if (want_src) gs = __ldg(reinterpret_cast<const float4 *>(a.grad_src_flat + o));
        if (read_pos) gp = __ldg(reinterpret_cast<const float4 *>(a.grad_pos_flat + o));
    }
    ts[c4][pr] = gs.x; ts[c4 + 1][pr] = gs.y; ts[c4 + 2][pr] = gs.z; ts[c4 + 3][pr] = gs.w;
    tp[c4][pr] = gp.x; tp[c4 + 1][pr] = gp.y; tp[c4 + 2][pr] = gp.z; tp[c4 + 3][pr] = gp.w;
    __syncthreads();
    const int px = tid & 31, cy = tid >> 5;
    const long long img = (long long)n * C * hw;
#pragma unroll
    for (int i = 0; i < kFlTile / 8; ++i) {
        const int c = cy + 8 * i;
        if (c0 + c < C && p0 + px < hw) {
            const long long o = img + (long long)(c0 + c) * hw + p0 + px;
            if (want_src) a.grad_src[l][o] = ts[c][px];
            if (a.grad_pos[l]) a.grad_pos[l][o] = tp[c][px];
        }
    }
    if (a.part && tid < kFlTile && c0 + tid < C) {           // this tile's sum over its 32 positions, in order
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < kFlTile; ++k) s += tp[tid][k];
        a.part[((long long)n * t.ptile0[t.L] + t.ptile0[l] + p0 / kFlTile) * C + c0 + tid] = s;
    }
}

// grid (L, ctiles), block (32, 32): lane x owns one channel; row y sums the partials y, y + 32, ... of level l (image
// by image, tile by tile), then row 0 adds the 32 row sums in order.
__global__ void __launch_bounds__(1024)
flatten_levels_reduce(const float *__restrict__ part, const FlattenTable t, int N, float *__restrict__ grad_level_embed)
{
    __shared__ float red[32][33];
    const int l = blockIdx.x, c = blockIdx.y * 32 + threadIdx.x, x = threadIdx.x, y = threadIdx.y, C = t.C;
    int first = 0, per = 0, total = 0;
#pragma unroll
    for (int k = 0; k < kMaxLevels; ++k) {       // constant indices: the table stays in the parameter space
        if (k == l) { first = t.ptile0[k]; per = t.ptile0[k + 1] - first; }
        if (k + 1 == t.L) total = t.ptile0[k + 1];
    }
    const int rows = N * per;
    float s = 0.f;
    if (c < C)
        for (int r = y; r < rows; r += 32) {
            const int n = r / per;
            s += part[((long long)n * total + first + (r - n * per)) * C + c];
        }
    red[y][x] = s;
    __syncthreads();
    if (y == 0 && c < C) {
        float v = 0.f;
#pragma unroll
        for (int k = 0; k < 32; ++k) v += red[k][x];
        grad_level_embed[(long long)l * C + c] = v;
    }
}

}  // namespace msda
