// msda_slab.cuh -- slab-ordered kernels for large launches (encoder-shaped calls), D = 32, L*P <= 16.
//
// A "slab" is one (batch element, head): the S x 128-byte (fp32) / 64-byte (bf16) strip of value / grad_value that all
// taps of the pairs (b, *, m) read / update.  These kernels walk the pairs SLAB-MAJOR -- a CTA owns a contiguous range
// of 64-pair tiles of the (b, m, q) space, i.e. consecutive queries of ONE head -- instead of the memory order
// (q, m) of msda_tiled.cuh.  That buys two things:
//
//   forward  -- the rows gathered by one SM come from one slab whose coarse levels (169 KB at cfg2) stay L1-resident,
//               and the gather uses 32-byte lanes (two 16-byte loads: 4 lanes per 128-byte row).
//   backward -- grad_value traffic is limited by each SM's path into the crossbar (~25 B/clk/SM of red payload, not by
//               the L2 atomic units).  The coarse levels of the CTA's current slab are therefore accumulated in a
//               shared-memory WINDOW and leave the SM once, when the CTA moves to another slab.  The SM has no fp32
//               shared-memory atomic (atomicAdd(float) = CAS loop, 12 cycles per row against 2.1 for a plain
//               LDS.128 / FFMA / STS.128), so the window is updated WITHOUT atomics under exclusive ownership:
//               phase P (produce): every group resolves its pair's taps; corners that fall into a window level are
//                                  appended to one of 64 row-class lists (class = window row mod 64) instead of going
//                                  to L2; everything else is the msda_tiled backward (gathers, dot products,
//                                  red.global for the fine levels, grad_loc / grad_attn).
//               phase C (consume): group g of warp w owns classes w + 16 g exclusively and applies its list to the
//                                  window with plain read-modify-writes -- no two groups ever touch the same row.
//               A full list falls back to the red.global path, so capacity never affects the result.
// Results are the same sums as the reference backward (cuh:87-159) in a different order.
#pragma once

#include "msda_tiled.cuh"

namespace msda {

constexpr int kSlabThreads = 512;
constexpr int kSlabWarps = kSlabThreads / 32;
constexpr int kSlabTile = kSlabWarps * 4;          // pairs per tile: 4 groups of 8 lanes per warp, one pair each
constexpr int kSlabClasses = 64;                   // row classes of the backward window (4 per warp: one per group)

struct SlabMap {
    int H[kMaxLevels], W[kMaxLevels], start[kMaxLevels];
    int wbase[kMaxLevels];        // first window row of level l, or -1 when the level is not privatised
    int wrows;                    // window rows in use
    unsigned tiles_per_slab, ntiles;
};

// Level table + tile counts; the backward also chooses which levels live in the shared-memory window: levels are taken
// smallest first while they fit `win_cap_rows` (cfg2: 13x21 + 25x42 = 1323 rows).  Derived on the device from the
// device-resident level table, like every other map in this library (no host read of spatial_shapes).
__device__ __forceinline__ void build_slab_map(SlabMap &sm, const int64_t *shapes, const int64_t *lsi, int L, int N, int M,
                                               int Lq, int win_cap_rows, int tile_pairs = kSlabTile) {
    if (threadIdx.x == 0) {
        int rows[kMaxLevels];
        for (int l = 0; l < L; ++l) {
            sm.H[l] = (int)shapes[2 * l]; sm.W[l] = (int)shapes[2 * l + 1]; sm.start[l] = (int)lsi[l];
            rows[l] = sm.H[l] * sm.W[l];
            sm.wbase[l] = -1;
        }
        int used = 0;
        for (int round = 0; round < L; ++round) {               // selection by increasing size (L <= 8)
            int best = -1;
            for (int l = 0; l < L; ++l)
                if (sm.wbase[l] < 0 && rows[l] > 0 && (best < 0 || rows[l] < rows[best])) best = l;
            if (best < 0 || used + rows[best] > win_cap_rows) break;
            sm.wbase[best] = used;
            used += rows[best];
        }
        sm.wrows = used;
        sm.tiles_per_slab = (unsigned)((Lq + tile_pairs - 1) / tile_pairs);
        sm.ntiles = (unsigned)N * (unsigned)M * sm.tiles_per_slab;
    }
    __syncthreads();
}

// CTAs that are co-resident on one SM should work on neighbouring tile ranges (shared L1 working set): with a grid of
// k * #SM CTAs, CTA c and c + #SM get adjacent ranges.
__device__ __forceinline__ void cta_tile_range(unsigned ntiles, unsigned sms, unsigned &first, unsigned &last) {
    const unsigned per_sm = (gridDim.x + sms - 1) / sms;
    const unsigned r = (blockIdx.x % sms) * per_sm + blockIdx.x / sms;
    const unsigned nr = sms * per_sm;
    first = (unsigned)(((unsigned long long)ntiles * r) / nr);
    last = (unsigned)(((unsigned long long)ntiles * (r + 1)) / nr);
}

// 8 consecutive channels of one row, widened to fp32: 32 bytes (fp32) / 16 bytes (bf16) per lane.
template <typename T> struct Row8;
template <> struct Row8<float> {
    __device__ static __forceinline__ void load(const unsigned char *p, float (&v)[8]) {
        RowVec<float, 8>::load(reinterpret_cast<const float *>(p), v);
    }
    __device__ static __forceinline__ void store(float *p, const float (&v)[8]) {
        reinterpret_cast<float4 *>(p)[0] = make_float4(v[0], v[1], v[2], v[3]);
        reinterpret_cast<float4 *>(p)[1] = make_float4(v[4], v[5], v[6], v[7]);
    }
};
template <> struct Row8<__nv_bfloat16> {
    __device__ static __forceinline__ void load(const unsigned char *p, float (&v)[8]) {
        RowVec<__nv_bfloat16, 8>::load(reinterpret_cast<const __nv_bfloat16 *>(p), v);
    }
    __device__ static __forceinline__ void store(__nv_bfloat16 *p, const float (&v)[8]) {
        RowVec<__nv_bfloat16, 8>::store(p, v);
    }
};

// ------------------------------------------------------------------------------------------------------------
// forward, slab-major (reference cuh:237-299).  8 lanes per pair; the two half-groups take the upper / lower corner
// pair of every tap with 8 channels per lane, and are combined with one xor-shuffle per channel at the end.
// ------------------------------------------------------------------------------------------------------------
template <typename T, int LP_MAX, int MIN_CTAS>
__global__ void __launch_bounds__(kSlabThreads, MIN_CTAS)
msda_fwd_slab(const T *__restrict__ value, const int64_t *__restrict__ shapes, const int64_t *__restrict__ lsi,
              const float *__restrict__ loc, const float *__restrict__ attn, int N, int S, int M, int L, int Lq, int P,
              int sms, T *__restrict__ out)
{
    constexpr int D = 32, LPR = 8, NSL = LP_MAX / LPR;
    static_assert(LP_MAX % LPR == 0, "tap capacity must be whole record rounds");
    __shared__ SlabMap sm;
    __shared__ __align__(16) unsigned char slab_mem[kSlabWarps * TapSlab<LPR>::kBytes];
    build_slab_map(sm, shapes, lsi, L, N, M, Lq, 0);

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sub = lane % LPR, grp = lane / LPR;
    const int half = sub >> 2, hs = sub & 3;
    const int LP = L * P;
    const unsigned row_bytes = (unsigned)(M * D) * (unsigned)sizeof(T);
    TapSlab<LPR> slab(slab_mem + warp * TapSlab<LPR>::kBytes, grp);

    unsigned first, last;
    cta_tile_range(sm.ntiles, (unsigned)sms, first, last);
#pragma unroll 1
    for (unsigned tile = first; tile < last; ++tile) {
        const unsigned sl = tile / sm.tiles_per_slab, qt = tile - sl * sm.tiles_per_slab;
        const int b = (int)(sl / (unsigned)M), m = (int)(sl - (unsigned)b * (unsigned)M);
        const int q = (int)qt * kSlabTile + warp * 4 + grp;
        const bool active = q < Lq;
        const size_t pair = ((size_t)b * Lq + (active ? q : Lq - 1)) * M + m;

        // ---- stage 1: this lane resolves its taps (dead taps: zero weight, row 0) ----
        float4 tw[NSL];
        int2 tr[NSL];
#pragma unroll
        for (int k = 0; k < NSL; ++k) {
            const int s = sub + k * LPR;
            tw[k] = make_float4(0.f, 0.f, 0.f, 0.f);
            tr[k] = make_int2(0, 0);
            if (s < LP && active) {
                const size_t t = pair * LP + s;
                const float2 xy = __ldg(reinterpret_cast<const float2 *>(loc) + t);
                const float a = __ldg(attn + t);
                const int l = s / P;
                const TapGeom g = tap_geometry(xy.x, xy.y, sm.H[l], sm.W[l], sm.start[l]);
                tw[k] = masked_weights(g, a);
                tr[k] = make_int2(g.r0, g.r1 | (g.dw << 31));
            }
        }

        // ---- stage 2: half 0 gathers corners 00 / 01, half 1 corners 10 / 11, 8 channels per lane ----
        const unsigned char *base = reinterpret_cast<const unsigned char *>(value + ((size_t)b * S * M + m) * D + hs * 8);
        float acc[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] = 0.f;
#pragma unroll
        for (int k = 0; k < NSL; ++k) {
            __syncwarp();
            slab.put(sub, tw[k], tr[k]);
            __syncwarp();
#pragma unroll
            for (int j = 0; j < LPR; ++j) {
                const float4 w = slab.weights(j);
                const int2 rr = slab.rows(j);
                const unsigned dwo = (rr.y < 0) ? row_bytes : 0u;
                const unsigned row = half ? (unsigned)(rr.y & 0x7fffffff) : (unsigned)rr.x;
                const float wa = half ? w.z : w.x, wb = half ? w.w : w.y;
                const unsigned char *p = base + (unsigned long long)row * row_bytes;
                float va[8], vb[8];
                Row8<T>::load(p, va);
                Row8<T>::load(p + dwo, vb);
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    acc[e] = fmaf(wa, va[e], acc[e]);
                    acc[e] = fmaf(wb, vb[e], acc[e]);
                }
            }
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] += __shfl_xor_sync(kFullMask, acc[e], 4);
        if (active && half == 0) Row8<T>::store(out + pair * D + hs * 8, acc);
    }
}

// ------------------------------------------------------------------------------------------------------------
// backward, slab-major, coarse levels of grad_value privatised in a shared-memory window (see the file comment).
// Dynamic shared memory:  window  [win_cap_rows][32] float | lists [64][list_cap] uint2 | g stash [64][32] float |
//                         tap slabs [16 warps] | cursors [64] int
// ------------------------------------------------------------------------------------------------------------
struct BwdSlabSmem {
    float *window; uint2 *lists; float *gstash; unsigned char *slabs; int *cursor;
};

__host__ __device__ inline size_t bwd_slab_smem_bytes(int win_cap_rows, int list_cap) {
    return (size_t)win_cap_rows * 128 + (size_t)kSlabClasses * list_cap * 8 + (size_t)kSlabTile * 128 +
           (size_t)kSlabWarps * TapSlab<8>::kBytes + (size_t)kSlabClasses * 4;
}

template <typename T, int LP_MAX>
__global__ void __launch_bounds__(kSlabThreads, 1)
msda_bwd_slab(const T *__restrict__ grad_out, const T *__restrict__ value, const int64_t *__restrict__ shapes,
              const int64_t *__restrict__ lsi, const float *__restrict__ loc, const float *__restrict__ attn,
              int N, int S, int M, int L, int Lq, int P, int sms, int win_cap_rows, int list_cap,
              float *__restrict__ grad_value, float *__restrict__ grad_loc, float *__restrict__ grad_attn)
{
    constexpr int D = 32, VEC = 4, LPR = 8, NSL = LP_MAX / LPR;
    static_assert(LP_MAX % LPR == 0, "tap capacity must be whole record rounds");
    extern __shared__ __align__(16) unsigned char dyn[];
    __shared__ SlabMap sm;
    BwdSlabSmem s;
    s.window = reinterpret_cast<float *>(dyn);
    s.lists = reinterpret_cast<uint2 *>(dyn + (size_t)win_cap_rows * 128);
    s.gstash = reinterpret_cast<float *>(reinterpret_cast<unsigned char *>(s.lists) + (size_t)kSlabClasses * list_cap * 8);
    s.slabs = reinterpret_cast<unsigned char *>(s.gstash) + (size_t)kSlabTile * 128;
    s.cursor = reinterpret_cast<int *>(s.slabs + (size_t)kSlabWarps * TapSlab<LPR>::kBytes);
    build_slab_map(sm, shapes, lsi, L, N, M, Lq, win_cap_rows);

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sub = lane % LPR, grp = lane / LPR;
    const int slot = warp * 4 + grp;                      // this group's pair slot inside the tile
    const int LP = L * P;
    const unsigned row_elems = (unsigned)(M * D);
    TapSlab<LPR> slab(s.slabs + warp * TapSlab<LPR>::kBytes, grp);
    const int wrows = sm.wrows;

    if (threadIdx.x < kSlabClasses) s.cursor[threadIdx.x] = 0;
    for (int i = threadIdx.x; i < wrows * 8; i += kSlabThreads)
        reinterpret_cast<float4 *>(s.window)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    __syncthreads();

    // window -> grad_value of slab `sl` (vector reds: other CTAs work on the same slab), then re-zero
    auto flush = [&](unsigned sl) {
        const int b = (int)(sl / (unsigned)M), m = (int)(sl - (unsigned)b * (unsigned)M);
        float *gslab = grad_value + ((size_t)b * S * M + m) * D;
        for (int i = threadIdx.x; i < wrows * 8; i += kSlabThreads) {
            const int wr = i >> 3, c4 = i & 7;
            float4 v = reinterpret_cast<float4 *>(s.window)[i];
            if (v.x != 0.f || v.y != 0.f || v.z != 0.f || v.w != 0.f) {
                int row = 0;
#pragma unroll 1
                for (int l = 0; l < L; ++l) {
                    const int wb = sm.wbase[l];
                    if (wb >= 0 && wr >= wb && wr < wb + sm.H[l] * sm.W[l]) row = sm.start[l] + (wr - wb);
                }
                red_add_v4(gslab + (size_t)row * row_elems + c4 * 4, v.x, v.y, v.z, v.w);
                reinterpret_cast<float4 *>(s.window)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            }
        }
    };

    unsigned first, last;
    cta_tile_range(sm.ntiles, (unsigned)sms, first, last);
    unsigned cur_slab = first < last ? first / sm.tiles_per_slab : 0u;
#pragma unroll 1
    for (unsigned tile = first; tile < last; ++tile) {
        const unsigned sl = tile / sm.tiles_per_slab, qt = tile - sl * sm.tiles_per_slab;
        if (sl != cur_slab) {                      // CTA-uniform: the window belongs to one slab at a time
            flush(cur_slab);
            cur_slab = sl;
            __syncthreads();
        }
        const int b = (int)(sl / (unsigned)M), m = (int)(sl - (unsigned)b * (unsigned)M);
        const int q = (int)qt * kSlabTile + slot;
        const bool active = q < Lq;
        const size_t pair = ((size_t)b * Lq + (active ? q : Lq - 1)) * M + m;

        // =============================== phase P ===============================
        float g[VEC];
        RowVec<T, VEC>::load(grad_out + pair * D + (size_t)sub * VEC, g);
        if (!active) { g[0] = g[1] = g[2] = g[3] = 0.f; }
        *reinterpret_cast<float4 *>(s.gstash + slot * 32 + sub * 4) = make_float4(g[0], g[1], g[2], g[3]);

        float4 tw[NSL];
        int2 tr[NSL];
        float tlh[NSL], tlw[NSL], ta[NSL];
        unsigned tmeta[NSL];                 // corner mask | level << 4
#pragma unroll
        for (int k = 0; k < NSL; ++k) {
            const int sidx = sub + k * LPR;
            tw[k] = make_float4(0.f, 0.f, 0.f, 0.f);
            tr[k] = make_int2(0, 0);
            tlh[k] = tlw[k] = ta[k] = 0.f; tmeta[k] = 0;
            if (sidx < LP && active) {
                const size_t t = pair * LP + sidx;
                const float2 xy = __ldg(reinterpret_cast<const float2 *>(loc) + t);
                const float a = __ldg(attn + t);
                const int l = sidx / P;
                const TapGeom gm = tap_geometry(xy.x, xy.y, sm.H[l], sm.W[l], sm.start[l]);
                float4 w4 = masked_weights(gm, a);
                tr[k] = make_int2(gm.r0, gm.r1 | (gm.dw << 31));
                tlh[k] = gm.lh; tlw[k] = gm.lw; ta[k] = a; tmeta[k] = gm.mask | ((unsigned)l << 4);
                const int wb = sm.wbase[l];
                if (wb >= 0) {
                    // window level: append the non-zero corners to their row-class lists; a corner that got a list
                    // slot has its weight cleared in the record, which is what skips the red.global in stage 2
                    const int w0 = wb + (gm.r0 - sm.start[l]), w1 = wb + (gm.r1 - sm.start[l]);
                    float wc[4] = {w4.x, w4.y, w4.z, w4.w};
                    const int wr[4] = {w0, w0 + gm.dw, w1, w1 + gm.dw};
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        if (wc[c] != 0.f) {
                            const int cls = wr[c] & (kSlabClasses - 1);
                            const int pos = atomicAdd(s.cursor + cls, 1);
                            if (pos < list_cap) {
                                s.lists[cls * list_cap + pos] = make_uint2(((unsigned)wr[c] << 8) | (unsigned)slot,
                                                                           __float_as_uint(wc[c]));
                                wc[c] = 0.f;
                            }
                        }
                    }
                    w4 = make_float4(wc[0], wc[1], wc[2], wc[3]);
                }
                tw[k] = w4;
            }
        }

        const size_t slab_off = ((size_t)b * S * M + m) * D + (size_t)sub * VEC;
        const T *base = value + slab_off;
        float *gbase = grad_value + slab_off;
#pragma unroll
        for (int k = 0; k < NSL; ++k) {
            __syncwarp();
            slab.put(sub, tw[k], tr[k]);
            __syncwarp();
            float part[LPR][4];
#pragma unroll
            for (int j = 0; j < LPR; ++j) {
                const float4 w4 = slab.weights(j);
                const int2 rr = slab.rows(j);
                const float w[4] = {w4.x, w4.y, w4.z, w4.w};
                const unsigned dwo = (rr.y < 0) ? row_elems : 0u;
                unsigned long long off[4];
                off[0] = (unsigned long long)(unsigned)rr.x * row_elems;
                off[1] = off[0] + dwo;
                off[2] = (unsigned long long)(unsigned)(rr.y & 0x7fffffff) * row_elems;
                off[3] = off[2] + dwo;
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    float v[VEC];
                    RowVec<T, VEC>::load(base + off[c], v);
                    float dsum = 0.f;
#pragma unroll
                    for (int e = 0; e < VEC; ++e) dsum = fmaf(g[e], v[e], dsum);
                    part[j][c] = dsum;
                    if (w[c] != 0.f)
                        red_add_v4(gbase + off[c], w[c] * g[0], w[c] * g[1], w[c] * g[2], w[c] * g[3]);
                }
            }
            float dot[4];
            group_reduce_scatter<LPR>(part, sub, dot);

            const int sidx = sub + k * LPR;
            if (sidx < LP && active) {
                const unsigned mk = tmeta[k];
                const int l = (int)(mk >> 4);
                const float d0 = (mk & 1u) ? dot[0] : 0.f, d1 = (mk & 2u) ? dot[1] : 0.f;
                const float d2 = (mk & 4u) ? dot[2] : 0.f, d3 = (mk & 8u) ? dot[3] : 0.f;
                const float lh = tlh[k], lw = tlw[k], hh = 1.f - lh, hw = 1.f - lw;
                const float val = hh * hw * d0 + hh * lw * d1 + lh * hw * d2 + lh * lw * d3;   // cuh:155-156
                const float gw = hh * (d1 - d0) + lh * (d3 - d2);                               // cuh:124,133,142,151
                const float gh = hw * (d2 - d0) + lw * (d3 - d1);                               // cuh:123,132,141,150
                const size_t t = pair * LP + sidx;
                grad_attn[t] = val;
                const float a = ta[k];
                reinterpret_cast<float2 *>(grad_loc)[t] =
                    make_float2((float)sm.W[l] * a * gw, (float)sm.H[l] * a * gh);              // cuh:157-158
            }
        }
        __syncthreads();                       // lists and g stash of this tile are complete

        // =============================== phase C ===============================
        if (wrows > 0) {
            const int cls = warp + kSlabWarps * grp;                   // classes owned by this group: disjoint rows
            const int n = min(s.cursor[cls], list_cap);
            const uint2 *lst = s.lists + cls * list_cap;
#pragma unroll 2
            for (int i = 0; i < n; ++i) {
                const uint2 e = lst[i];
                const float w = __uint_as_float(e.y);
                const float4 gv = *reinterpret_cast<const float4 *>(s.gstash + (e.x & 255u) * 32 + sub * 4);
                float4 *ap = reinterpret_cast<float4 *>(s.window + (size_t)(e.x >> 8) * 32 + sub * 4);
                float4 av = *ap;
                av.x = fmaf(w, gv.x, av.x); av.y = fmaf(w, gv.y, av.y);
                av.z = fmaf(w, gv.z, av.z); av.w = fmaf(w, gv.w, av.w);
                *ap = av;
            }
            __syncwarp();
            if (sub == 0) s.cursor[cls] = 0;
        }
        __syncthreads();                       // window updated, lists free for the next tile
    }
    if (first < last) flush(cur_slab);
}

}  // namespace msda
