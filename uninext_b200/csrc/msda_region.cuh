// msda_region.cuh -- fp32 encoder backward (D = 32, L*P <= 16, Lq == S) that sums grad_value contributions per spatial
// region on chip and sends each touched row to L2 once.
//
// msda_bwd_tiled issues one 16-byte red.global per lane and live corner: a 128-byte row-add per corner, ~20 M of them per
// cfg2 encoder call, 8x the compulsory grad_value bytes.  In encoder self-attention the queries ARE the pixels of the
// pyramid and every query samples within a few pixels of its own position on every level.  So a CTA that takes all
// queries of one (batch, head) whose pixel centre lies in one R x R region of the finest level touches only a small
// rectangle ("window") of each level, and it can add those contributions up on chip first.
//
// grad_value's sums need each tap's geometry and the pair's grad_out, never `value`, and nothing of grad_loc /
// grad_attn.  So the backward is two kernels, each with its own register and shared-memory budget:
//   msda_bwd_region (tap pass, 2 CTAs/SM): msda_bwd_tiled's NORED body (linear chunks of pairs, taps TMA-staged one
//             iteration ahead when L*P % 4 == 0): the gathers, grad_loc and grad_attn, from the same device code and in
//             the same FMA order as msda_bwd_tiled.
//   msda_region_grad_value_pass (__launch_bounds__ for 3 CTAs/SM), per tile = (b, m, region).  A query at pixel (x, y) of level l belongs to
//             region floor((x + 0.5) * Wref / W_l / R) in x (likewise in y; Wref / Href = the largest level), so a
//             region holds one contiguous x-range and y-range per level, in closed form.  The window on level l is the
//             region scaled to level l plus kRegionHalo pixels.
//     phase A: one 8-lane group per pair; the lane that resolves a tap files its non-zero in-window corners as entries
//              {window row, coefficient} at the fixed positions (slot, tap, corner) and counts each for its window row with
//              a non-returning shared atomic.  The pair's grad_out row is stashed in shared memory.  A corner outside the
//              window, or of a query past the stash, reds directly as in msda_bwd_tiled (its weight and rows go through
//              the group's tap slab), so the capacities never change a result.  No value row is read.
//     phase B: scan of the row counts, then scatter of the entry indices by window row (integer shared atomics only:
//              fp32 shared atomics are CAS loops) into one u16 array.
//     phase C: one group per touched row sums coefficient x stashed grad_out in registers and issues one red per lane.
// The two kernels share no data (the tap pass writes grad_loc / grad_attn, the grad_value pass grad_value), and they are
// limited by different things: the tap pass by its gathers, the grad_value pass by latency.  So they run side by side on
// every SM, 2 grad_value CTAs beside 1 tap CTA (the host sizes both grids for that), chained by PDL:
//   zero-fill (primary) -> grad_value kernel -> tap kernel.
// The grad_value kernel lets its dependent launch at once, so the tap CTAs fill the room its CTAs leave, and waits for the
// fill before its first red (and, if it had none, before it exits).  The tap kernel waits for the grad_value kernel as its
// last statement: its completion then implies the grad_value kernel's and, through it, the fill's.
// A level table that does not tile [0, S) (the patch-order condition) runs the grad_value pass in linear chunks of pairs
// with no window: every corner reds directly.
#pragma once

#include "msda_tiled.cuh"

namespace msda {

constexpr int kRegionEdge = 8;            // region edge, in pixels of the finest level
constexpr int kRegionHalo = 2;            // window margin around the scaled region, in pixels of each level (swept 1-6)
constexpr int kRegionSlots = 96;          // queries per tile whose grad_out row is stashed (the rest red directly)
constexpr int kRegionWinRows = 1024;      // window rows per tile (levels past this budget red directly)
// Not used by the kernel, which stages no value rows: only the tests' restatement of the window layout
// (tests/region_layout.py) reads it.
constexpr int kRegionStageRows = 384;
constexpr int kRegionEntries = kRegionSlots * 16 * 4;   // one entry position per (slot, tap, corner); L*P <= 16
// __launch_bounds__ minimum CTAs per SM.  They fix each kernel's register budget; the grids are sized on the host
// (2 grad_value CTAs + 1 tap CTA per SM on an H100).
constexpr int kRegionTapCtas = 2;         // tap kernel: it needs 128 registers per thread
constexpr int kRegionGvCtas = 3;          // grad_value kernel: latency-bound, 46 registers
constexpr int kRegionIterSlots = kTiledWarps * 4;       // pairs per CTA iteration (D = 32: 4 groups of 8 lanes per warp)

// The tap kernel's TMA stage buffers (kTiledWarps per-warp double buffers of one iteration's (x, y, a)).
using RegionTapStage = TapStage<4, 16, true>;

// Dynamic shared memory of the tap kernel: its stage buffers.
constexpr size_t region_tap_smem_bytes() { return (size_t)kTiledWarps * RegionTapStage::kBytes; }

// Dynamic shared memory of the grad_value kernel: entry coefficients (f32) + grad_out stash + row counts + entry rows
// (u16) + the entry indices sorted by window row (u16).
constexpr size_t region_gv_smem_bytes() {
    static_assert(kRegionEntries <= 0x10000, "entry indices are u16");
    return (size_t)kRegionEntries * (4 + 2 + 2) + (size_t)kRegionSlots * 128 + (size_t)kRegionWinRows * 4;
}

#ifdef MSDA_REGION_PHASE_CLOCKS
// Timing hook for tools/region_phases.py; the library build never defines it.  Thread 0 of each grad_value CTA adds the
// clock64() span since the previous stamp into g_region_clocks[blockIdx.x * kRegionSpans + span], after a CTA barrier:
// span 0 = tile geometry + count reset, 1 = phase A, 2 = phase B, 3 = phase C.  g_region_knockout bit 0 drops phase A's
// direct reds, bit 1 phase C's (the sums are still formed); results are then wrong by construction and serve only for
// timing.
constexpr int kRegionSpans = 4;
__device__ unsigned long long *g_region_clocks;
__device__ int g_region_knockout;
#define MSDA_REGION_CLOCK_INIT long long region_clk = clock64()
#define MSDA_REGION_CLOCK(span)                                                                  \
    if (threadIdx.x == 0) {                                                                      \
        const long long now = clock64();                                                         \
        g_region_clocks[blockIdx.x * kRegionSpans + (span)] += (unsigned long long)(now - region_clk); \
        region_clk = now;                                                                        \
    }
#define MSDA_REGION_KEEP_RED(bit) (!(g_region_knockout & (bit)))
#else
#define MSDA_REGION_CLOCK_INIT
#define MSDA_REGION_CLOCK(span)
#define MSDA_REGION_KEEP_RED(bit) true
#endif

#ifdef MSDA_REGION_COSCHED
// Placement hook for tools/region_cosched.py; the library build never defines it.  Thread 0 of each CTA of kernel k
// (0 = grad_value, 1 = tap) writes {%smid, %globaltimer at its start, %globaltimer when its work is done} into
// g_region_cosched[k][3 * blockIdx.x ...], the end after a CTA barrier (and, in the tap kernel, before its PDL wait).
__device__ unsigned long long *g_region_cosched[2];
__device__ __forceinline__ unsigned long long region_globaltimer() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
#define MSDA_REGION_COSCHED_START(k)                                                               \
    if (threadIdx.x == 0) {                                                                        \
        unsigned smid;                                                                             \
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));                                         \
        g_region_cosched[k][3 * blockIdx.x] = smid;                                                \
        g_region_cosched[k][3 * blockIdx.x + 1] = region_globaltimer();                            \
    }
#define MSDA_REGION_COSCHED_END(k)                                                                 \
    __syncthreads();                                                                               \
    if (threadIdx.x == 0) g_region_cosched[k][3 * blockIdx.x + 2] = region_globaltimer();
#else
#define MSDA_REGION_COSCHED_START(k)
#define MSDA_REGION_COSCHED_END(k)
#endif

struct RegionMap {
    int H[kMaxLevels], W[kMaxLevels], start[kMaxLevels];
    int Href, Wref, nry, nrx;
    int region;                 // 1: region tiles; 0: linear chunks of kRegionIterSlots pairs, no window
    unsigned ntiles;
};

struct RegionTile {
    int b, m, nq, nwin;
    unsigned base_pair;         // linear chunks
    int qy0[kMaxLevels], qx0[kMaxLevels], qny[kMaxLevels], qnx[kMaxLevels], qpre[kMaxLevels + 1];
    int wy0[kMaxLevels], wx0[kMaxLevels], wh[kMaxLevels], ww[kMaxLevels], wbase[kMaxLevels + 1];
};

// First pixel of a level of n pixels (reference extent `ref`) whose region index is >= r.
__device__ __forceinline__ int region_first(int r, int n, int ref, int R) {
    const long long num = 2ll * r * n * R - ref;
    return num <= 0 ? 0 : (int)min((long long)n, (num + 2ll * ref - 1) / (2ll * ref));
}

// The grad_value pass, a persistent PDL secondary of the zero-fill and the PDL primary of the tap kernel
// (msda_bwd_region).  It waits for the fill before its first red; its first tile's geometry and entries overlap the fill.
template <int R, int HALO>
__global__ void __launch_bounds__(kTiledThreads, kRegionGvCtas)
msda_region_grad_value_pass(const float *__restrict__ grad_out, const int64_t *__restrict__ shapes,
                            const int64_t *__restrict__ lsi, const float *__restrict__ loc,
                            const float *__restrict__ attn, int N, int S, int M, int L, int Lq, int P, unsigned npairs,
                            float *__restrict__ grad_value)
{
    constexpr int D = 32, VEC = 4, LPR = D / VEC, GPW = 32 / LPR, LP_MAX = 16, NSL = LP_MAX / LPR;
    static_assert(GPW * kTiledWarps == kRegionIterSlots && kRegionSlots <= 256 && kRegionWinRows < 0xffff &&
                  kRegionSlots % kRegionIterSlots == 0, "entry layout");
    constexpr unsigned short kNoRow = 0xffff;

    __shared__ RegionMap rm;
    __shared__ RegionTile tl;
    __shared__ int wsum[kTiledWarps];
    __shared__ __align__(16) unsigned char slab_mem[kTiledWarps * TapSlab<LPR>::kBytes];
    extern __shared__ __align__(128) unsigned char region_dyn[];
    float *e_coef = reinterpret_cast<float *>(region_dyn);                            // [slot][tap][corner]
    float4 *gstash = reinterpret_cast<float4 *>(e_coef + kRegionEntries);             // [slot][lane] grad_out slices
    int *cnt = reinterpret_cast<int *>(gstash + kRegionSlots * LPR);                  // [window row]
    unsigned short *e_row = reinterpret_cast<unsigned short *>(cnt + kRegionWinRows); // [slot][tap][corner], kNoRow = none
    unsigned short *s_idx = e_row + kRegionEntries;     // phases B, C: entry indices sorted by window row

    pdl_launch_dependents();     // the tap kernel's CTAs may take the room this kernel leaves on each SM
    MSDA_REGION_COSCHED_START(0);
    MSDA_REGION_CLOCK_INIT;
    if (threadIdx.x == 0) {            // the map comes from the device-resident level table: no host read, capture-safe
        int run = 0, href = 0, wref = 0;
        bool tiled = (Lq == S);
        for (int l = 0; l < L; ++l) {
            const int h = (int)shapes[2 * l], w = (int)shapes[2 * l + 1], st = (int)lsi[l];
            rm.H[l] = h; rm.W[l] = w; rm.start[l] = st;
            tiled = tiled && (st == run) && h > 0 && w > 0;
            run += h * w;
            href = max(href, h); wref = max(wref, w);
        }
        tiled = tiled && (run == S);
        rm.region = tiled ? 1 : 0;
        rm.Href = href; rm.Wref = wref;
        rm.nry = (href + R - 1) / R; rm.nrx = (wref + R - 1) / R;
        rm.ntiles = tiled ? (unsigned)N * (unsigned)M * (unsigned)(rm.nry * rm.nrx)
                          : (npairs + kRegionIterSlots - 1) / kRegionIterSlots;
    }
    __syncthreads();

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sub = lane % LPR, grp = lane / LPR;
    const int LP = L * P;
    const unsigned row_elems = (unsigned)(M * D);
    TapSlab<LPR> slab(slab_mem + warp * TapSlab<LPR>::kBytes, grp);
    bool primary_done = false;         // CTA-uniform: pdl_wait_primary() has returned
    for (unsigned tile = blockIdx.x; tile < rm.ntiles; tile += gridDim.x) {
        // ---- tile geometry: thread l resolves level l, thread 0 then lays the levels out ----
        if (rm.region) {
            const int m = (int)(tile % (unsigned)M);         // heads fastest: concurrent tiles share loc / attn pages
            const unsigned r = tile / (unsigned)M, per_b = (unsigned)(rm.nry * rm.nrx);
            const int reg = (int)(r % per_b), ry = reg / rm.nrx, rx = reg % rm.nrx;
            const int l = threadIdx.x;
            if (l < L) {
                const int H = rm.H[l], W = rm.W[l];
                const int y0 = region_first(ry, H, rm.Href, R), y1 = region_first(ry + 1, H, rm.Href, R);
                const int x0 = region_first(rx, W, rm.Wref, R), x1 = region_first(rx + 1, W, rm.Wref, R);
                tl.qy0[l] = y0; tl.qny[l] = y1 - y0; tl.qx0[l] = x0; tl.qnx[l] = x1 - x0;
                const int wy0 = max(0, (int)((long long)ry * R * H / rm.Href) - HALO);
                const int wy1 = min(H, (int)(((long long)(ry + 1) * R * H + rm.Href - 1) / rm.Href) + HALO);
                const int wx0 = max(0, (int)((long long)rx * R * W / rm.Wref) - HALO);
                const int wx1 = min(W, (int)(((long long)(rx + 1) * R * W + rm.Wref - 1) / rm.Wref) + HALO);
                tl.wy0[l] = wy0; tl.wh[l] = wy1 - wy0; tl.wx0[l] = wx0; tl.ww[l] = wx1 - wx0;
            }
            if (threadIdx.x == 0) { tl.m = m; tl.b = (int)(r / per_b); }
            __syncthreads();
            if (threadIdx.x == 0) {
                int nq = 0, nw = 0;
                for (int k = 0; k < L; ++k) {
                    tl.qpre[k] = nq; nq += tl.qny[k] * tl.qnx[k];
                    const int rows = tl.wh[k] * tl.ww[k];
                    if (nw + rows > kRegionWinRows) { tl.wh[k] = tl.ww[k] = 0; }     // over budget: this level reds directly
                    tl.wbase[k] = nw; nw += tl.wh[k] * tl.ww[k];
                }
                tl.qpre[L] = nq; tl.wbase[L] = nw;
                tl.nq = nq; tl.nwin = nw;
            }
        } else if (threadIdx.x == 0) {
            tl.base_pair = tile * kRegionIterSlots;
            tl.nq = (int)min((unsigned)kRegionIterSlots, npairs - tl.base_pair);
            tl.nwin = 0;
        }
        __syncthreads();
        for (int i = threadIdx.x; i < tl.nwin; i += kTiledThreads) cnt[i] = 0;
        __syncthreads();
        MSDA_REGION_CLOCK(0);

        // ---- phase A: in-window corners become entries, the others red ----
#pragma unroll 1
        for (int it = 0; it * kRegionIterSlots < tl.nq; ++it) {
            const int slot = it * kRegionIterSlots + warp * GPW + grp;
            const bool active = slot < tl.nq;
            unsigned pair = 0; int b = 0, m = 0;
            if (active) {
                if (rm.region) {
                    int l = 0;
                    while (l + 1 < L && slot >= tl.qpre[l + 1]) ++l;
                    const int k = slot - tl.qpre[l], y = tl.qy0[l] + k / tl.qnx[l], x = tl.qx0[l] + k % tl.qnx[l];
                    b = tl.b; m = tl.m;
                    pair = ((unsigned)b * (unsigned)Lq + (unsigned)(rm.start[l] + y * rm.W[l] + x)) * (unsigned)M + (unsigned)m;
                } else {
                    pair = tl.base_pair + (unsigned)slot;
                    m = (int)(pair % (unsigned)M);
                    b = (int)((pair / (unsigned)M) / (unsigned)Lq);
                }
            }
            const bool stash = rm.region && active && slot < kRegionSlots;        // group-uniform

            float g[VEC] = {0.f, 0.f, 0.f, 0.f};
            if (active) RowVec<float, VEC>::load(grad_out + (size_t)pair * D + (size_t)sub * VEC, g);
            if (stash) gstash[slot * LPR + sub] = make_float4(g[0], g[1], g[2], g[3]);

            // ---- this lane resolves taps sub, sub + LPR and files their in-window corners; the rest go to the slab ----
            float4 tw[NSL];              // weights of the corners that red directly (the others 0)
            int2 tr[NSL];
#pragma unroll
            for (int k = 0; k < NSL; ++k) {
                const int s = sub + k * LPR;
                tw[k] = make_float4(0.f, 0.f, 0.f, 0.f);
                tr[k] = make_int2(0, 0);
                unsigned filed = 0;
                ushort4 rows4 = make_ushort4(kNoRow, kNoRow, kNoRow, kNoRow);
                float4 w4 = make_float4(0.f, 0.f, 0.f, 0.f);
                if (s < LP && active) {
                    const size_t t = (size_t)pair * LP + s;
                    const float2 xy = __ldg(reinterpret_cast<const float2 *>(loc) + t);
                    const float a = __ldg(attn + t);
                    const int l = s / P;
                    const TapGeom gm = tap_geometry(xy.x, xy.y, rm.H[l], rm.W[l], rm.start[l]);
                    w4 = masked_weights(gm, a);
                    tr[k] = make_int2(gm.r0, gm.r1 | (gm.dw << 31));
                    const unsigned nz = (unsigned)(w4.x != 0.f) | ((unsigned)(w4.y != 0.f) << 1) |
                                        ((unsigned)(w4.z != 0.f) << 2) | ((unsigned)(w4.w != 0.f) << 3);
                    if (stash) {
                        const int W = rm.W[l], o0 = gm.r0 - rm.start[l], o1 = gm.r1 - rm.start[l];
                        const int y0 = o0 / W, x0 = o0 - y0 * W, y1 = o1 / W;
                        const int wwl = tl.ww[l], whl = tl.wh[l];
                        const int ry0 = y0 - tl.wy0[l], ry1 = y1 - tl.wy0[l], rx0 = x0 - tl.wx0[l], rx1 = rx0 + gm.dw;
                        const unsigned iy0 = (unsigned)ry0 < (unsigned)whl, iy1 = (unsigned)ry1 < (unsigned)whl;
                        const unsigned ix0 = (unsigned)rx0 < (unsigned)wwl, ix1 = (unsigned)rx1 < (unsigned)wwl;
                        const unsigned inwin = (iy0 & ix0) | ((iy0 & ix1) << 1) | ((iy1 & ix0) << 2) | ((iy1 & ix1) << 3);
                        filed = inwin & nz;
                        const int w00 = tl.wbase[l] + ry0 * wwl + rx0, dhw = (y1 - y0) * wwl;
                        const int wr[4] = {w00, w00 + gm.dw, w00 + dhw, w00 + dhw + gm.dw};
#pragma unroll
                        for (int c = 0; c < 4; ++c)
                            if ((filed >> c) & 1u) atomicAdd(&cnt[wr[c]], 1);      // phase B's row count; result unused
                        rows4 = make_ushort4((filed & 1u) ? (unsigned short)wr[0] : kNoRow,
                                             (filed & 2u) ? (unsigned short)wr[1] : kNoRow,
                                             (filed & 4u) ? (unsigned short)wr[2] : kNoRow,
                                             (filed & 8u) ? (unsigned short)wr[3] : kNoRow);
                    }
                    tw[k] = make_float4((filed & 1u) ? 0.f : w4.x, (filed & 2u) ? 0.f : w4.y,
                                        (filed & 4u) ? 0.f : w4.z, (filed & 8u) ? 0.f : w4.w);
                }
                if (stash) {
                    const int e = (slot * LP_MAX + s) << 2;
                    *reinterpret_cast<ushort4 *>(e_row + e) = rows4;
                    *reinterpret_cast<float4 *>(e_coef + e) = w4;
                }
            }

            // ---- direct reds: the group walks the taps of its pair that have a corner to red ----
            if (!primary_done) {       // grad_value's zero-fill is complete and visible
                pdl_wait_primary();
                primary_done = true;
            }
            const size_t slab_off = ((size_t)b * S * M + m) * D + (size_t)sub * VEC;
            float *gbase = grad_value + slab_off;
#pragma unroll
            for (int k = 0; k < NSL; ++k) {
                __syncwarp();
                slab.put(sub, tw[k], tr[k]);
                __syncwarp();
                const bool any = tw[k].x != 0.f || tw[k].y != 0.f || tw[k].z != 0.f || tw[k].w != 0.f;
                unsigned todo = (__ballot_sync(kFullMask, any) >> (grp * LPR)) & ((1u << LPR) - 1u);
                while (todo) {
                    const int j = __ffs(todo) - 1;
                    todo &= todo - 1u;
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
                    for (int c = 0; c < 4; ++c)
                        if (w[c] != 0.f && MSDA_REGION_KEEP_RED(1))
                            red_add_v4(gbase + off[c], w[c] * g[0], w[c] * g[1], w[c] * g[2], w[c] * g[3]);
                }
            }
        }

        const int nwin = tl.nwin;
        if (nwin > 0) {
            __syncthreads();
            MSDA_REGION_CLOCK(1);
            const int n = min(tl.nq, kRegionSlots) * LP_MAX * 4;
            // ---- phase B: counting sort of the entries by window row (phase A counted them) ----
            {   // exclusive scan of cnt[0, nwin): 4 rows per thread
                const int i0 = threadIdx.x * 4;
                int c[4], sum = 0;
#pragma unroll
                for (int q = 0; q < 4; ++q) { c[q] = (i0 + q < nwin) ? cnt[i0 + q] : 0; sum += c[q]; }
                int incl = sum;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    const int t = __shfl_up_sync(kFullMask, incl, d);
                    if (lane >= d) incl += t;
                }
                if (lane == 31) wsum[warp] = incl;
                __syncthreads();
                int run = incl - sum;
                for (int w = 0; w < warp; ++w) run += wsum[w];
#pragma unroll
                for (int q = 0; q < 4; ++q)
                    if (i0 + q < nwin) { cnt[i0 + q] = run; run += c[q]; }
            }
            static_assert(kRegionWinRows <= 4 * kTiledThreads, "scan covers 4 rows per thread");
            __syncthreads();
            for (int e = threadIdx.x; e < n; e += kTiledThreads) {
                const unsigned short r = e_row[e];
                if (r != kNoRow) s_idx[atomicAdd(&cnt[r], 1)] = (unsigned short)e;
            }
            __syncthreads();          // bucket r is now [r ? cnt[r - 1] : 0, cnt[r]) of s_idx
            MSDA_REGION_CLOCK(2);

            // ---- phase C: one group per touched row, one red per lane ----
            const int b = tl.b, m = tl.m;
            for (int r = warp * GPW + grp; r < nwin; r += kRegionIterSlots) {
                const int beg = r ? cnt[r - 1] : 0, end = cnt[r];
                if (beg == end) continue;
                float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
                for (int i = beg; i < end; ++i) {
                    const int e = s_idx[i];
                    const float cf = e_coef[e];
                    const float4 gs = gstash[(e / (LP_MAX * 4)) * LPR + sub];
                    acc.x = fmaf(cf, gs.x, acc.x); acc.y = fmaf(cf, gs.y, acc.y);
                    acc.z = fmaf(cf, gs.z, acc.z); acc.w = fmaf(cf, gs.w, acc.w);
                }
                int l = 0;
                while (l + 1 < L && r >= tl.wbase[l + 1]) ++l;
                const int k = r - tl.wbase[l], y = tl.wy0[l] + k / tl.ww[l], x = tl.wx0[l] + k % tl.ww[l];
                const int row = rm.start[l] + y * rm.W[l] + x;
                if (MSDA_REGION_KEEP_RED(2))
                    red_add_v4(grad_value + (((size_t)b * S + row) * M + m) * D + (size_t)sub * VEC, acc.x, acc.y, acc.z, acc.w);
            }
        }
        __syncthreads();              // the next tile rewrites tl, the entry list, the stash and the counts
        MSDA_REGION_CLOCK(nwin > 0 ? 3 : 1);
    }
    // The tap kernel takes this kernel's completion to imply the fill's, so a CTA that issued no red waits here.
    if (!primary_done) pdl_wait_primary();
    MSDA_REGION_COSCHED_END(0);
}

// The tap pass: grad_loc / grad_attn.  tma: it stages (x, y, a) with TMA (use_tma_staging on the host: L*P % 4 == 0).
template <int R, int HALO>
__global__ void __launch_bounds__(kTiledThreads, kRegionTapCtas)
msda_bwd_region(const float *__restrict__ grad_out, const float *__restrict__ value,
                const int64_t *__restrict__ shapes, const int64_t *__restrict__ lsi,
                const float *__restrict__ loc, const float *__restrict__ attn,
                int N, int S, int M, int L, int Lq, int P, unsigned npairs, int tma,
                float *__restrict__ grad_loc, float *__restrict__ grad_attn)
{
    __shared__ WorkMap wm;
    __shared__ __align__(16) unsigned char slab_mem[kTiledWarps * TapSlab<8>::kBytes];
    __shared__ __align__(8) unsigned long long stage_bar[kTiledWarps * 2];
    extern __shared__ __align__(128) unsigned char stage_mem[];        // region_tap_smem_bytes()

    MSDA_REGION_COSCHED_START(1);
    if (tma)
        bwd_tiled_body<float, 4, 32, 16, true, false, false, true, false>(
            wm, slab_mem, stage_mem, stage_bar, grad_out, value, shapes, lsi, loc, attn, N, S, M, L, Lq, P, npairs, 0,
            nullptr, grad_loc, grad_attn, nullptr, 0);
    else
        bwd_tiled_body<float, 4, 32, 16, false, false, false, true, false>(
            wm, slab_mem, stage_mem, stage_bar, grad_out, value, shapes, lsi, loc, attn, N, S, M, L, Lq, P, npairs, 0,
            nullptr, grad_loc, grad_attn, nullptr, 0);
    MSDA_REGION_COSCHED_END(1);
    // Nothing here touches grad_value, but the next operation on the stream relies on this kernel's completion implying
    // the grad_value kernel's (and the fill's): wait for the PDL primary last.
    pdl_wait_primary();
}

// Launch sizes of the region backward's two kernels.  Side by side (the PDL chain): the most grad_value CTAs per SM, g (at
// most its own occupancy), that leave room for one tap CTA in the SM's registers (allocated per warp in units of 256),
// shared memory (static + dynamic + the per-CTA reservation) and threads; on an H100 that is 2 + 1, 2 x 12 288 + 32 768
// registers.  The block scheduler places a kernel's CTAs wherever they fit, so if g + 1 grad_value CTAs fit an SM it puts
// g + 1 on some SMs and none on others, and two tap CTAs then run alone there.  The grad_value kernel's dynamic shared
// memory is therefore padded until g + 1 no longer fit, and it asks for the largest shared-memory carveout, so that the
// SM keeps room for the tap CTA.  Alone (no chain, or where no grad_value CTA fits beside a tap CTA) each kernel gets its
// own occupancy.  Host code, shared by the library and tools/region_cosched.cu; the caller has opted the grad_value
// kernel in to gv_smem bytes of dynamic shared memory.
struct RegionGrids {
    int gv, tap;                // side by side: grids
    size_t gv_smem;             // side by side: the grad_value kernel's (padded) dynamic shared memory
    int gv_solo, tap_solo;      // one after the other: grids
};

template <class GV, class TAP>
RegionGrids region_grids(GV gvk, size_t gv_smem, TAP tap, size_t tap_smem, int sms) {
    const auto occupancy = [](auto kern, size_t smem) {
        int per_sm = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kTiledThreads, smem) != cudaSuccess || per_sm < 1)
            per_sm = 1;
        return per_sm;
    };
    const int gv_occ = occupancy(gvk, gv_smem), tap_occ = occupancy(tap, tap_smem);
    const RegionGrids solo = {gv_occ * sms, tap_occ * sms, gv_smem, gv_occ * sms, tap_occ * sms};
    int dev = 0, regs_sm = 0, smem_sm = 0, smem_optin = 0, reserved = 0, threads_sm = 0;
    cudaFuncAttributes ga{}, ta{};
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&regs_sm, cudaDevAttrMaxRegistersPerMultiprocessor, dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&smem_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&reserved, cudaDevAttrReservedSharedMemoryPerBlock, dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&threads_sm, cudaDevAttrMaxThreadsPerMultiProcessor, dev) != cudaSuccess ||
        cudaFuncGetAttributes(&ga, gvk) != cudaSuccess || cudaFuncGetAttributes(&ta, tap) != cudaSuccess)
        return solo;
    constexpr int warps = kTiledThreads / 32;
    const auto regs = [](int per_thread) { return warps * ((per_thread * 32 + 255) / 256 * 256); };
    const auto smem = [&](const cudaFuncAttributes &a, size_t dyn) { return (long long)a.sharedSizeBytes + (long long)dyn + reserved; };
    for (int g = gv_occ; g >= 1; --g) {
        size_t dyn = gv_smem;
        if (g < gv_occ) {           // pad in 1 KB steps until g + 1 CTAs exceed the SM
            const long long over = (long long)smem_sm / (g + 1) + 1 - smem(ga, 0);
            dyn = (size_t)((over + 1023) / 1024 * 1024);
        }
        if ((long long)g * regs(ga.numRegs) + regs(ta.numRegs) <= regs_sm && (long long)dyn <= smem_optin &&
            g * smem(ga, dyn) + smem(ta, tap_smem) <= smem_sm && (g + 1) * kTiledThreads <= threads_sm) {
            if (dyn != gv_smem &&
                (cudaFuncSetAttribute(gvk, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn) != cudaSuccess ||
                 cudaFuncSetAttribute(gvk, cudaFuncAttributePreferredSharedMemoryCarveout,
                                      (int)cudaSharedmemCarveoutMaxShared) != cudaSuccess ||
                 occupancy(gvk, dyn) != g))
                return solo;
            return {g * sms, sms, dyn, solo.gv_solo, solo.tap_solo};
        }
    }
    return solo;
}

}  // namespace msda
