// msda_det.cuh -- deterministic grad_value of the backward (msda_backward_det_*; contract in include/msda_b200.h and
// DESIGN.md section 3.10).
//
// grad_value is summed without atomics, in the order of the repository's CPU oracle (oracle/): within one
// (b, m, row), contributions are added in ascending entry id  e = ((q*M + m)*L*P + l*P + p)*4 + k, each one rounded as
// fl(cw_k * fl(g_c * a)) and added with one rounding.  The pipeline works on chunks of whole queries of one batch
// element, in ascending (b, q) order, so a chunk's entries land after every earlier chunk's entries:
//   1. msda_det_keys        one (key, e) pair per (tap, corner) of the chunk; key = m*S + row, or the sentinel M*S for a
//                           corner outside the map or a tap outside the window;
//   2. cub radix sort       stable, by key: each row's entries stay in ascending e;
//   3. msda_det_bounds      first sorted position of every key;
//   4. msda_det_accumulate  one lane group per (m, row) segment, rows handed out dynamically; the group loads the row,
//                           walks its entries in order and stores the row once.
// Every product and sum uses explicit round-to-nearest intrinsics, so nvcc cannot contract anything into an FMA.
#pragma once

#include <cub/device/device_radix_sort.cuh>

#include "msda_generic.cuh"

namespace msda {

constexpr int kDetThreads = 256;

__device__ __forceinline__ float rn_mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double rn_mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float rn_add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double rn_add(double a, double b) { return __dadd_rn(a, b); }

// The tap's window test and bilinear fractions in the oracle's rounding: h_im = fl(fl(y*H) - 0.5), lh = h_im - floor(h_im).
template <typename C>
__device__ __forceinline__ bool det_tap(C x, C y, int H, int W, int &h0, int &w0, C &lh, C &lw) {
    const C h_im = rn_add(rn_mul(y, (C)H), (C)-0.5);
    const C w_im = rn_add(rn_mul(x, (C)W), (C)-0.5);
    if (!(h_im > (C)-1 && w_im > (C)-1 && h_im < (C)H && w_im < (C)W)) return false;
    const C hf = floor(h_im), wf = floor(w_im);
    h0 = (int)hf;
    w0 = (int)wf;
    lh = rn_add(h_im, -hf);
    lw = rn_add(w_im, -wf);
    return true;
}

// Corner k = (dh, dw) = (k >> 1, k & 1): row within the level map, or -1 outside it.
__device__ __forceinline__ int det_corner_row(int h0, int w0, int k, int H, int W) {
    const int h = h0 + (k >> 1), w = w0 + (k & 1);
    return (h >= 0 && h < H && w >= 0 && w < W) ? h * W + w : -1;
}

// cw_k = {hh*hw, hh*lw, lh*hw, lh*lw}[k] with hh = fl(1 - lh), hw = fl(1 - lw).
template <typename C>
__device__ __forceinline__ C det_corner_weight(C lh, C lw, int k) {
    const C fh = (k >> 1) ? lh : rn_add((C)1, -lh);
    const C fw = (k & 1) ? lw : rn_add((C)1, -lw);
    return rn_mul(fh, fw);
}

// An entry of the chunk decoded for the accumulate step: its corner weight, attention weight and grad_out row
// (pair index relative to the chunk's first pair).
template <typename C, typename TL>
__device__ __forceinline__ void det_decode(unsigned e, const TL *__restrict__ loc, const TL *__restrict__ attn,
                                           const int64_t *__restrict__ shapes, int L, int P, long long tap0, C &w,
                                           C &a, unsigned &pair) {
    const unsigned k = e & 3u, t = e >> 2, LP = (unsigned)(L * P);
    const unsigned lp = t % LP;
    const int l = (int)(lp / (unsigned)P);
    const long long tap = tap0 + t;
    const int H = (int)shapes[2 * l], W = (int)shapes[2 * l + 1];
    int h0 = 0, w0 = 0;
    C lh = 0, lw = 0;
    det_tap<C>((C)loc[2 * tap], (C)loc[2 * tap + 1], H, W, h0, w0, lh, lw);    // passes: the key step filed the entry
    w = det_corner_weight<C>(lh, lw, (int)k);
    a = (C)attn[tap];
    pair = t / LP;
}

// 1. keys: entry e of the chunk (taps tap0 + e / 4) at position e.
template <typename TL>
__global__ void __launch_bounds__(kDetThreads)
msda_det_keys(const TL *__restrict__ loc, const int64_t *__restrict__ shapes, const int64_t *__restrict__ lsi, int S,
              int M, int L, int P, long long tap0, unsigned n, unsigned *__restrict__ keys, unsigned *__restrict__ vals)
{
    const unsigned LP = (unsigned)(L * P), sentinel = (unsigned)M * (unsigned)S;
    for (unsigned e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) {
        const unsigned k = e & 3u, t = e >> 2;
        const unsigned m = (t / LP) % (unsigned)M;
        const int l = (int)((t % LP) / (unsigned)P);
        const long long tap = tap0 + t;
        const int H = (int)shapes[2 * l], W = (int)shapes[2 * l + 1];
        int h0, w0;
        TL lh, lw;
        unsigned key = sentinel;
        if (det_tap<TL>(loc[2 * tap], loc[2 * tap + 1], H, W, h0, w0, lh, lw)) {
            const int r = det_corner_row(h0, w0, (int)k, H, W);
            if (r >= 0) key = m * (unsigned)S + (unsigned)(lsi[l] + r);
        }
        keys[e] = key;
        vals[e] = e;
    }
}

// 3. start[k] = first position of key k in the sorted keys (lower bound), for k in [0, nkeys]; segment k is
// [start[k], start[k + 1]).
__global__ void __launch_bounds__(kDetThreads)
msda_det_bounds(const unsigned *__restrict__ keys, unsigned n, unsigned nkeys, unsigned *__restrict__ start)
{
    for (unsigned k = blockIdx.x * blockDim.x + threadIdx.x; k <= nkeys; k += gridDim.x * blockDim.x) {
        unsigned lo = 0, hi = n;
        while (lo < hi) {
            const unsigned mid = lo + (hi - lo) / 2;
            if (keys[mid] < k) lo = mid + 1; else hi = mid;
        }
        start[k] = lo;
    }
}

// 4a. ordered accumulate, D = 32, fp32 accumulator (fp32 or bf16 grad_out): 8 lanes x 4 channels per row.  Each round
// decodes 8 entries (one per lane), issues their 8 grad_out loads, decodes the next 8, then retires the adds in order.
template <typename T>
__global__ void __launch_bounds__(kDetThreads)
msda_det_accumulate_v4(const T *__restrict__ grad_out, const float *__restrict__ loc, const float *__restrict__ attn,
                       const int64_t *__restrict__ shapes, int S, int M, int L, int P, long long tap0, int b,
                       const unsigned *__restrict__ start, const unsigned *__restrict__ vals,
                       unsigned *__restrict__ next_row, float *__restrict__ grad_value)
{
    constexpr int D = 32, G = 8;
    const int lane = threadIdx.x & 31, sub = lane & (G - 1), lead = lane & ~(G - 1);
    const unsigned gmask = 0xffu << lead;
    const unsigned nrows = (unsigned)M * (unsigned)S;
    const T *go = grad_out + (size_t)sub * 4;
    for (;;) {
        unsigned key = 0;
        if (sub == 0) key = atomicAdd(next_row, 1u);
        key = __shfl_sync(gmask, key, lead);
        if (key >= nrows) break;
        const unsigned s0 = start[key], s1 = start[key + 1];
        if (s0 == s1) continue;
        const unsigned m = key / (unsigned)S, row = key % (unsigned)S;
        float *gv = grad_value + (((size_t)b * S + row) * M + m) * D + (size_t)sub * 4;
        float acc[4];
        RowVec<float, 4>::load(gv, acc);
        float w = 0.f, a = 0.f;
        unsigned pair = 0;
        if (s0 + sub < s1) det_decode<float, float>(vals[s0 + sub], loc, attn, shapes, L, P, tap0, w, a, pair);
        for (unsigned base = s0; base < s1; base += G) {
            const unsigned cnt = min((unsigned)G, s1 - base);
            float g[G][4], wj[G], aj[G];
#pragma unroll
            for (int j = 0; j < G; ++j) {
                wj[j] = __shfl_sync(gmask, w, lead + j);
                aj[j] = __shfl_sync(gmask, a, lead + j);
                const unsigned pj = __shfl_sync(gmask, pair, lead + j);
                if ((unsigned)j < cnt) RowVec<T, 4>::load(go + (size_t)pj * D, g[j]);
            }
            const unsigned nxt = base + G + sub;
            if (nxt < s1) det_decode<float, float>(vals[nxt], loc, attn, shapes, L, P, tap0, w, a, pair);
#pragma unroll
            for (int j = 0; j < G; ++j) {
                if ((unsigned)j < cnt) {
#pragma unroll
                    for (int c = 0; c < 4; ++c) acc[c] = __fadd_rn(acc[c], __fmul_rn(wj[j], __fmul_rn(g[j][c], aj[j])));
                }
            }
        }
        RowVec<float, 4>::store(gv, acc);
    }
}

// 4b. ordered accumulate, any D and storage type (compute type C = double for fp64, float otherwise): one warp per row,
// one channel per lane, 32-channel passes over the segment.
template <typename T, typename TL>
__global__ void __launch_bounds__(kDetThreads)
msda_det_accumulate(const T *__restrict__ grad_out, const TL *__restrict__ loc, const TL *__restrict__ attn,
                    const int64_t *__restrict__ shapes, int S, int M, int D, int L, int P, long long tap0, int b,
                    const unsigned *__restrict__ start, const unsigned *__restrict__ vals,
                    unsigned *__restrict__ next_row, typename Num<T>::C *__restrict__ grad_value)
{
    using C = typename Num<T>::C;
    constexpr int U = 8;
    const int lane = threadIdx.x & 31;
    const unsigned nrows = (unsigned)M * (unsigned)S;
    for (;;) {
        unsigned key = 0;
        if (lane == 0) key = atomicAdd(next_row, 1u);
        key = __shfl_sync(kFullMask, key, 0);
        if (key >= nrows) break;
        const unsigned s0 = start[key], s1 = start[key + 1];
        if (s0 == s1) continue;
        const unsigned m = key / (unsigned)S, row = key % (unsigned)S;
        C *gv = grad_value + (((size_t)b * S + row) * M + m) * D;
        for (int c0 = 0; c0 < D; c0 += 32) {
            const int c = c0 + lane;
            const bool live = c < D;
            C acc = live ? gv[c] : (C)0;
            for (unsigned base = s0; base < s1; base += 32) {
                C w = 0, a = 0;
                unsigned pair = 0;
                if (base + lane < s1) det_decode<C, TL>(vals[base + lane], loc, attn, shapes, L, P, tap0, w, a, pair);
                const int cnt = (int)min(32u, s1 - base);
                for (int j0 = 0; j0 < cnt; j0 += U) {
                    C gj[U], wj[U], aj[U];
#pragma unroll
                    for (int u = 0; u < U; ++u) {
                        wj[u] = __shfl_sync(kFullMask, w, (j0 + u) & 31);
                        aj[u] = __shfl_sync(kFullMask, a, (j0 + u) & 31);
                        const unsigned pj = __shfl_sync(kFullMask, pair, (j0 + u) & 31);
                        gj[u] = (live && j0 + u < cnt) ? (C)Num<T>::ld(grad_out + (size_t)pj * D + c) : (C)0;
                    }
#pragma unroll
                    for (int u = 0; u < U; ++u)
                        if (j0 + u < cnt) acc = rn_add(acc, rn_mul(wj[u], rn_mul(gj[u], aj[u])));
                }
            }
            if (live) gv[c] = acc;
        }
    }
}

// 2. the sort, shared by the workspace query (d_temp == nullptr) and the run.
inline cudaError_t det_sort(void *d_temp, size_t &temp_bytes, const unsigned *keys_in, unsigned *keys_out,
                            const unsigned *vals_in, unsigned *vals_out, unsigned n, int end_bit, cudaStream_t st) {
    return cub::DeviceRadixSort::SortPairs(d_temp, temp_bytes, keys_in, keys_out, vals_in, vals_out, n, 0, end_bit, st);
}

}  // namespace msda
