// msda_tmem.cuh -- backward with the coarse levels of grad_value accumulated in a shared-memory window owned by four
// consumer warps (D = 32, L*P <= 16).  MSDA_KNOB_SLAB = 2.
//
// Why: the backward is bound by each SM's path into the crossbar (red.global payload).  Combining the
// coarse levels' contributions inside the SM halves that traffic.  msda_slab.cuh does it with every warp taking turns
// as producer and consumer; here the roles are split over dedicated warps so that the gathers never wait for the window.
//
// Layout: a window row (32 channels, fp32) is 128 bytes of dynamic shared memory; row r belongs to consumer q = r % 4.
// The number of rows is what the device's opt-in shared memory leaves after the lists (227 KB on sm_90: 1323 rows, the
// levels 13x21 and 25x42 of cfg2, fit next to the default lists).
//
// Roles (512 threads, one CTA per SM):
//   warps 0..11  producers -- the msda_bwd_tiled work for 4 pairs each (tap geometry, row gathers, dot products, grad_loc /
//                grad_attn, red.global for the non-window levels).  Non-zero corners that fall into a window level are
//                appended to the warp's PRIVATE list for the row's consumer (positions from ballots: no atomics) and
//                their weight is cleared in the tap record, which skips the red.global.
//   warps 12..15 consumers -- warp 12 + q owns the rows r % 4 == q exclusively: it drains the 12 producer lists of its
//                rows with plain shared-memory read-modify-writes (lane = channel).  Exclusive ownership = no atomics.
//   Lists and the stashed grad_out rows are double-buffered per tile: producers fill buffer t while consumers drain t-1;
//   one __syncthreads per tile.  When the CTA's tile range moves to another (batch, head) slab, and at the end, the
//   consumers add their rows to grad_value (red.global.add.f32, one 128-byte row per instruction) and zero them.
// A full list falls back to red.global, so capacity never affects the result.
#pragma once

#include "msda_slab.cuh"

namespace msda {

constexpr int kTmThreads = 512;
constexpr int kTmProd = 12;                    // producer warps
constexpr int kTmCons = 4;                     // consumer warps
constexpr int kTmTile = kTmProd * 4;           // pairs per tile

__host__ __device__ inline size_t bwd_tmem_smem_bytes(int list_cap, int win_rows) {
    return 2 * ((size_t)kTmProd * kTmCons * list_cap * 8        // entry lists
                + (size_t)kTmProd * kTmCons * 4                 // entry counts
                + (size_t)kTmTile * 128)                        // grad_out rows of the tile
           + (size_t)kTmProd * TapSlab<8>::kBytes                // tap slabs
           + (size_t)win_rows * 128;                             // window
}

template <typename T, int LP_MAX>
__global__ void __launch_bounds__(kTmThreads, 1)
msda_bwd_tmem(const T *__restrict__ grad_out, const T *__restrict__ value, const int64_t *__restrict__ shapes,
              const int64_t *__restrict__ lsi, const float *__restrict__ loc, const float *__restrict__ attn,
              int N, int S, int M, int L, int Lq, int P, int sms, int list_cap, int win_rows,
              float *__restrict__ grad_value, float *__restrict__ grad_loc, float *__restrict__ grad_attn)
{
    constexpr int D = 32, VEC = 4, LPR = 8, NSL = LP_MAX / LPR;
    static_assert(LP_MAX % LPR == 0, "tap capacity must be whole record rounds");
    extern __shared__ __align__(16) unsigned char dyn[];
    __shared__ SlabMap sm;

    // dynamic shared memory: [2] lists | [2] counts | [2] g stash | tap slabs | window
    const size_t list_bytes = (size_t)kTmProd * kTmCons * list_cap * 8;
    uint2 *lists = reinterpret_cast<uint2 *>(dyn);                                        // [buf][warp][quad][cap]
    int *counts = reinterpret_cast<int *>(dyn + 2 * list_bytes);                          // [buf][warp][quad]
    float *gstash = reinterpret_cast<float *>(dyn + 2 * list_bytes + 2 * kTmProd * kTmCons * 4);      // [buf][slot][32]
    unsigned char *slabs = reinterpret_cast<unsigned char *>(gstash) + 2 * (size_t)kTmTile * 128;
    float *win = reinterpret_cast<float *>(slabs + (size_t)kTmProd * TapSlab<8>::kBytes);     // [row][32]

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    build_slab_map(sm, shapes, lsi, L, N, M, Lq, win_rows & ~(kTmCons - 1), kTmTile);
    const int wrows = sm.wrows;
    const int LP = L * P;
    const unsigned row_elems = (unsigned)(M * D);

    unsigned first, last;
    cta_tile_range(sm.ntiles, (unsigned)sms, first, last);
    const unsigned ntile = last > first ? last - first : 0u;

    if (warp >= kTmProd) {
        // ======================================= consumers =======================================
        const int q = warp - kTmProd;                                        // this warp owns the rows r % 4 == q
        float *wq = win + q * 32 + lane;                                     // row r = 4 c + q  ->  wq[c * 128]
        const int ncols = wrows > q ? (wrows - q + 3) / 4 : 0;
        for (int c = 0; c < ncols; ++c) wq[c * 128] = 0.f;

        auto flush = [&](unsigned sl) {                                       // rows -> grad_value of slab `sl`, then zero
            const int b = (int)(sl / (unsigned)M), m = (int)(sl - (unsigned)b * (unsigned)M);
            float *gslab = grad_value + ((size_t)b * S * M + m) * D + lane;
            for (int c = 0; c < ncols; ++c) {
                const int wr = c * 4 + q;
                int row = 0;
                for (int l = 0; l < L; ++l) {
                    const int wb = sm.wbase[l];
                    if (wb >= 0 && wr >= wb && wr < wb + sm.H[l] * sm.W[l]) row = sm.start[l] + (wr - wb);
                }
                const float f = wq[c * 128];
                if (f != 0.f) atomicAdd(gslab + (size_t)row * row_elems, f);          // RED.E.ADD.F32: 128 B per warp
                wq[c * 128] = 0.f;
            }
        };

        for (unsigned it = 0; it <= ntile; ++it) {
            if (it > 0 && wrows > 0) {
                const unsigned tile = first + it - 1;
                const int buf = (int)((it - 1) & 1u);
                const float *gs = gstash + (size_t)buf * kTmTile * 32 + lane;
                for (int w = 0; w < kTmProd; ++w) {
                    const int n = min(counts[(buf * kTmProd + w) * kTmCons + q], list_cap);
                    const uint2 *lst = lists + ((size_t)(buf * kTmProd + w) * kTmCons + q) * list_cap;
                    for (int i = 0; i < n; ++i) {
                        const uint2 e = lst[i];
                        float *dst = wq + (size_t)(e.x >> 8) * 128;
                        *dst = fmaf(__uint_as_float(e.y), gs[(e.x & 255u) * 32], *dst);
                    }
                }
                const unsigned sl = tile / sm.tiles_per_slab;
                if (it == ntile || (tile + 1) / sm.tiles_per_slab != sl) flush(sl);
            }
            __syncthreads();
        }
    } else {
        // ======================================= producers =======================================
        const int sub = lane % LPR, grp = lane / LPR;
        const int slot = warp * 4 + grp;
        TapSlab<LPR> slab(slabs + warp * TapSlab<LPR>::kBytes, grp);
        const unsigned lt_mask = (1u << lane) - 1u;

        for (unsigned it = 0; it <= ntile; ++it) {
            if (it < ntile) {
                const unsigned tile = first + it;
                const int buf = (int)(it & 1u);
                const unsigned sl = tile / sm.tiles_per_slab, qt = tile - sl * sm.tiles_per_slab;
                const int b = (int)(sl / (unsigned)M), m = (int)(sl - (unsigned)b * (unsigned)M);
                const int qi = (int)qt * kTmTile + slot;
                const bool active = qi < Lq;
                const size_t pair = ((size_t)b * Lq + (active ? qi : Lq - 1)) * M + m;
                uint2 *mylist = lists + (size_t)(buf * kTmProd + warp) * kTmCons * list_cap;
                int cnt[kTmCons] = {0, 0, 0, 0};                              // warp-uniform list lengths

                float g[VEC];
                RowVec<T, VEC>::load(grad_out + pair * D + (size_t)sub * VEC, g);
                if (!active) { g[0] = g[1] = g[2] = g[3] = 0.f; }
                *reinterpret_cast<float4 *>(gstash + ((size_t)buf * kTmTile + slot) * 32 + sub * 4) = make_float4(g[0], g[1], g[2], g[3]);

                float4 tw[NSL];
                int2 tr[NSL];
                float tlh[NSL], tlw[NSL], ta[NSL];
                unsigned tmeta[NSL];
#pragma unroll
                for (int k = 0; k < NSL; ++k) {
                    const int sidx = sub + k * LPR;
                    float wc[4] = {0.f, 0.f, 0.f, 0.f};
                    int wr[4] = {-1, -1, -1, -1};                             // window row of each corner, -1 = not a window level
                    tr[k] = make_int2(0, 0);
                    tlh[k] = tlw[k] = ta[k] = 0.f; tmeta[k] = 0;
                    if (sidx < LP && active) {
                        const size_t t = pair * LP + sidx;
                        const float2 xy = __ldg(reinterpret_cast<const float2 *>(loc) + t);
                        const float a = __ldg(attn + t);
                        const int l = sidx / P;
                        const TapGeom gm = tap_geometry(xy.x, xy.y, sm.H[l], sm.W[l], sm.start[l]);
                        const float4 w4 = masked_weights(gm, a);
                        wc[0] = w4.x; wc[1] = w4.y; wc[2] = w4.z; wc[3] = w4.w;
                        tr[k] = make_int2(gm.r0, gm.r1 | (gm.dw << 31));
                        tlh[k] = gm.lh; tlw[k] = gm.lw; ta[k] = a; tmeta[k] = gm.mask | ((unsigned)l << 4);
                        const int wb = sm.wbase[l];
                        if (wb >= 0) {
                            const int w0 = wb + (gm.r0 - sm.start[l]), w1 = wb + (gm.r1 - sm.start[l]);
                            wr[0] = w0; wr[1] = w0 + gm.dw; wr[2] = w1; wr[3] = w1 + gm.dw;
                        }
                    }
                    // converged again: warp-aggregated append of the non-zero window corners (no atomics; order = lane order)
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        const bool want = wr[c] >= 0 && wc[c] != 0.f;
#pragma unroll
                        for (int qd = 0; qd < kTmCons; ++qd) {
                            const unsigned mk = __ballot_sync(kFullMask, want && (wr[c] & 3) == qd);
                            if (want && (wr[c] & 3) == qd) {
                                const int pos = cnt[qd] + __popc(mk & lt_mask);
                                if (pos < list_cap) {
                                    mylist[qd * list_cap + pos] = make_uint2(((unsigned)(wr[c] >> 2) << 8) | (unsigned)slot,
                                                                             __float_as_uint(wc[c]));
                                    wc[c] = 0.f;                              // in the list: no red.global for this corner
                                }
                            }
                            cnt[qd] += __popc(mk);
                        }
                    }
                    tw[k] = make_float4(wc[0], wc[1], wc[2], wc[3]);
                }
                if (lane < kTmCons)
                    counts[(buf * kTmProd + warp) * kTmCons + lane] = lane == 0 ? cnt[0] : lane == 1 ? cnt[1] : lane == 2 ? cnt[2] : cnt[3];

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
            }
            __syncthreads();
        }
    }

}

}  // namespace msda
