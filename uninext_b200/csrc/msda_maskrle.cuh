// msda_maskrle.cuh -- COCO run-length encoding of instance masks for UNINEXT inference (DESIGN.md section 3.14, row f-7):
// stride-s mask logits [I, Hs, Ws] (or binary masks [I, H, W] already on the device) -> the `counts` strings of
// pycocotools' mask.encode, without storing full-resolution masks.
//
// The reference pastes each mask, copies it to the host and calls mask.encode per instance (uninext_vid.py:1425-1432,
// :1263-1271 + :1686-1700, detectron2/evaluation/coco_evaluation.py:478-490).  The COCO API scans the mask column-major
// (k = X * H + Y), emits the run lengths starting with a run of zeros (rleEncode), then writes each count as 5-bit groups
// (rleToString: x = counts[j] - counts[j - 2] for j > 2; 0x20 marks a continued group; +48).  Here:
//   pass 1  rle_bits_logits / rle_bits_u8: one thread per column (per 4 columns for masks) walks the column top to
//           bottom, writes 1 bit per pixel into a bitmap [I][ceil(H/32)][W] (lanes of a warp own consecutive columns,
//           so every bitmap word and every mask row is read or written coalesced) and the column's boundary count;
//           the logits are evaluated by mp_source / mp_prob, the code mask_paste runs, so the bits are paste_masks'.
//   scan    cub::DeviceScan, in place over the [I * W + 1] column counts: each column's first boundary, each instance's
//           first boundary (entry i * W) and the total (entry I * W), which the caller reads to size the next buffers.
//   pass 2  rle_boundaries: from the bitmap alone, each column's boundary positions k in ascending order.
//   pass 3  rle_tile_bytes / rle_scan_tiles / rle_write: counts are differences of positions; the characters of each
//           count are measured, scanned per tile of kRleTile counts and then across tiles, and written.
// Offsets of pixels, words, boundaries, counts and characters are 64-bit; positions within one instance are < 2^32.
#pragma once

#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>
#include <cub/device/device_scan.cuh>

#include "msda_maskpaste.cuh"

namespace msda {

constexpr int kRleThreads = 128;                 // passes 1 and 2
constexpr int kRleU8Cols = 4;                    // mask columns per thread in pass 1: a warp reads 128 bytes of a row
constexpr int kRleTileThreads = 256;             // pass 3
constexpr int kRleTileItems = 8;                 // consecutive counts per thread in pass 3
constexpr int kRleTile = kRleTileThreads * kRleTileItems;
constexpr int kRleScanThreads = 256;             // the one-block scan over pass 3's tile sums

// The boundaries inside one bitmap word with `nbits` valid bits, given the bit before its first one.
__device__ __forceinline__ unsigned rle_edges(unsigned word, int nbits, unsigned carry) {
    const unsigned valid = nbits >= 32 ? ~0u : (1u << nbits) - 1u;
    return (word ^ ((word << 1) | carry)) & valid;
}

// Pass 1 on logits.  grid: (column tiles of kRleThreads, instances; grid-y strides over I).  The bit before the column's
// first pixel is the previous column's last pixel, evaluated here once more (one pixel per column).
__global__ void __launch_bounds__(kRleThreads)
rle_bits_logits(const float *__restrict__ logits, long long I, int Hs, int Ws, int crop_h, int crop_w, int out_h,
                int out_w, float near_y, float near_x, float lin_y, float lin_x, float threshold,
                unsigned *__restrict__ bitmap, long long *__restrict__ col_count)
{
    if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) col_count[I * out_w] = 0;   // becomes the total
    const int X = blockIdx.x * kRleThreads + threadIdx.x;
    if (X >= out_w) return;
    int x0, x1, p0 = 0, p1 = 0, l0, l1;
    float lx, lp = 0.f, ll;
    mp_source(X, near_x, crop_w, lin_x, Ws, x0, x1, lx);
    if (X > 0) mp_source(X - 1, near_x, crop_w, lin_x, Ws, p0, p1, lp);
    mp_source(out_h - 1, near_y, crop_h, lin_y, Hs, l0, l1, ll);
    float hl = 1.f - ll;
    asm("" : "+f"(hl));                          // see hy0 below
    const int nw = (out_h + 31) >> 5;
    const size_t plane = (size_t)Hs * Ws, wplane = (size_t)nw * out_w;
    for (long long i = blockIdx.y; i < I; i += gridDim.y) {
        const float *base = logits + i * plane;
        unsigned carry = 0;
        if (X > 0)
            carry = mp_prob(base + (size_t)l0 * Ws + p0, base + (size_t)l1 * Ws + p0, p1 - p0, lp, hl, ll) > threshold;
        unsigned *dst = bitmap + i * wplane + X;
        long long edges = 0;
        for (int w = 0; w < nw; ++w) {
            const int nbits = min(32, out_h - 32 * w);
            unsigned word = 0;
#pragma unroll 4
            for (int b = 0; b < nbits; ++b) {
                int y0, y1;
                float ly;
                mp_source(32 * w + b, near_y, crop_h, lin_y, Hs, y0, y1, ly);
                // Opaque, as mask_paste's loop-invariant hy0 is: otherwise nvcc fuses ly * bot instead of hy0 * top into
                // the last FMA of mp_prob, and a pixel within an ulp of the threshold can come out differently.
                float hy0 = 1.f - ly;
                asm("" : "+f"(hy0));
                const float p = mp_prob(base + (size_t)y0 * Ws + x0, base + (size_t)y1 * Ws + x0, x1 - x0, lx, hy0, ly);
                word |= (p > threshold ? 1u : 0u) << b;
            }
            dst[(size_t)w * out_w] = word;
            edges += __popc(rle_edges(word, nbits, carry));
            carry = (word >> (nbits - 1)) & 1u;
        }
        col_count[i * out_w + X] = edges;
    }
}

// Pass 1 on masks [I, H, W] (uint8 / bool, row-major).  A thread owns kRleU8Cols consecutive columns; VEC: the rows
// are 4-byte aligned (masks and W), so each row step is one 4-byte load and a warp reads 128 contiguous bytes.  Each
// column's boundary with the previous column is added at the end, from the first and last bits kept on the way.
template <bool VEC>
__global__ void __launch_bounds__(kRleThreads)
rle_bits_u8(const uint8_t *__restrict__ masks, long long I, int out_h, int out_w, unsigned *__restrict__ bitmap,
            long long *__restrict__ col_count)
{
    if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) col_count[I * out_w] = 0;
    const int X0 = (blockIdx.x * kRleThreads + threadIdx.x) * kRleU8Cols;
    if (X0 >= out_w) return;
    const int ncols = min(kRleU8Cols, out_w - X0);
    const int nw = (out_h + 31) >> 5;
    const size_t plane = (size_t)out_h * out_w, wplane = (size_t)nw * out_w;
    for (long long i = blockIdx.y; i < I; i += gridDim.y) {
        const uint8_t *base = masks + i * plane + X0;
        unsigned *dst = bitmap + i * wplane + X0;
        unsigned first = 0, last[kRleU8Cols] = {0u, 0u, 0u, 0u};
        int edges[kRleU8Cols] = {0, 0, 0, 0};
        for (int w = 0; w < nw; ++w) {
            const int nbits = min(32, out_h - 32 * w);
            unsigned word[kRleU8Cols] = {0u, 0u, 0u, 0u};
#pragma unroll 4
            for (int b = 0; b < nbits; ++b) {
                const uint8_t *row = base + (size_t)(32 * w + b) * out_w;
                unsigned v;
                if constexpr (VEC) {
                    v = __ldg(reinterpret_cast<const unsigned *>(row));
                } else {
                    v = 0;
#pragma unroll
                    for (int c = 0; c < kRleU8Cols; ++c)
                        if (c < ncols) v |= (unsigned)__ldg(row + c) << (8 * c);
                }
#pragma unroll
                for (int c = 0; c < kRleU8Cols; ++c) word[c] |= (((v >> (8 * c)) & 0xffu) ? 1u : 0u) << b;
            }
#pragma unroll
            for (int c = 0; c < kRleU8Cols; ++c) {
                if (c < ncols) dst[(size_t)w * out_w + c] = word[c];
                // inside the column only: at w = 0 the carry is the first bit itself, the column start comes below
                edges[c] += __popc(rle_edges(word[c], nbits, w == 0 ? word[c] & 1u : last[c]));
                last[c] = (word[c] >> (nbits - 1)) & 1u;
                if (w == 0) first |= (word[c] & 1u) << c;
            }
        }
        unsigned prev = X0 > 0 && base[(size_t)(out_h - 1) * out_w - 1] ? 1u : 0u;   // last pixel of column X0 - 1
#pragma unroll
        for (int c = 0; c < kRleU8Cols; ++c) {
            if (c < ncols) col_count[i * out_w + X0 + c] = edges[c] + (int)(((first >> c) & 1u) != prev);
            prev = last[c];
        }
    }
}

// Pass 2.  Thread = column X of instance i: the column's boundaries, k = X * out_h + Y ascending, from col_off[i, X].
__global__ void __launch_bounds__(kRleThreads)
rle_boundaries(const unsigned *__restrict__ bitmap, const long long *__restrict__ col_off, long long I, int out_h,
               int out_w, unsigned *__restrict__ pos)
{
    const int X = blockIdx.x * kRleThreads + threadIdx.x;
    if (X >= out_w) return;
    const int nw = (out_h + 31) >> 5, last_bits = out_h - 32 * (nw - 1);
    const size_t wplane = (size_t)nw * out_w;
    const unsigned k0 = (unsigned)X * (unsigned)out_h;
    for (long long i = blockIdx.y; i < I; i += gridDim.y) {
        const unsigned *src = bitmap + i * wplane + X;
        unsigned carry = X > 0 ? (src[(size_t)(nw - 1) * out_w - 1] >> (last_bits - 1)) & 1u : 0u;
        long long o = col_off[i * out_w + X];
        for (int w = 0; w < nw; ++w) {
            const int nbits = min(32, out_h - 32 * w);
            const unsigned word = src[(size_t)w * out_w];
            for (unsigned e = rle_edges(word, nbits, carry); e; e &= e - 1)
                pos[o++] = k0 + 32u * (unsigned)w + (unsigned)(__ffs(e) - 1);
            carry = (word >> (nbits - 1)) & 1u;
        }
    }
}

// Pass 3.  Counts are numbered globally: instance i owns g in [s_i, s_{i+1}), s_i = col_off[i * W] + i (its boundaries
// plus one).  Count j of instance i is pos(j) - pos(j - 1) with pos(-1) = 0 and pos(n_i) = H * W.
struct RleCounts {
    const long long *col_off;                    // [I * W + 1], scanned
    const unsigned *pos;
    long long I, N, hw;                          // N = total boundaries + I
    int W;

    __device__ __forceinline__ long long start(long long i) const { return col_off[i * W] + i; }

    // the instance owning count g: the largest i with start(i) <= g
    __device__ __forceinline__ long long owner(long long g) const {
        long long lo = 0, hi = I - 1;
        while (lo < hi) {
            const long long mid = (lo + hi + 1) >> 1;
            if (start(mid) <= g) lo = mid; else hi = mid - 1;
        }
        return lo;
    }

    // the value rleToString writes for count j of instance i
    __device__ __forceinline__ long long value(long long i, long long j) const {
        const long long b = col_off[i * W], n = col_off[(i + 1) * W] - b;
        auto at = [&](long long t) -> long long { return t < 0 ? 0 : t == n ? hw : (long long)pos[b + t]; };
        long long x = at(j) - at(j - 1);
        if (j > 2) x -= at(j - 2) - at(j - 3);
        return x;
    }
};

__device__ __forceinline__ int rle_chars(long long x) {
    int n = 0;
    bool more = true;
    while (more) {
        const int c = (int)(x & 0x1f);
        x >>= 5;
        more = (c & 0x10) ? x != -1 : x != 0;
        ++n;
    }
    return n;
}

// The kRleTileItems counts of this thread (those below N): their values, instances and positions within the instance.
struct RleItems {
    long long x[kRleTileItems];
    long long g0;
    int n;

    __device__ __forceinline__ void load(const RleCounts &rc, long long g) {
        g0 = g;
        n = (int)max(0ll, min((long long)kRleTileItems, rc.N - g));
        if (n == 0) return;
        long long i = rc.owner(g), next = i + 1 < rc.I ? rc.start(i + 1) : rc.N;
#pragma unroll
        for (int t = 0; t < kRleTileItems; ++t) {
            if (t < n) {
                while (g + t >= next) { ++i; next = i + 1 < rc.I ? rc.start(i + 1) : rc.N; }
                x[t] = rc.value(i, g + t - rc.start(i));
            }
        }
    }
};

// tile_sum[tile] = the characters of the tile's counts.
__global__ void __launch_bounds__(kRleTileThreads)
rle_tile_bytes(RleCounts rc, long long *__restrict__ tile_sum)
{
    using Reduce = cub::BlockReduce<long long, kRleTileThreads>;
    __shared__ typename Reduce::TempStorage tmp;
    RleItems it;
    it.load(rc, (long long)blockIdx.x * kRleTile + (long long)threadIdx.x * kRleTileItems);
    long long s = 0;
#pragma unroll
    for (int t = 0; t < kRleTileItems; ++t)
        if (t < it.n) s += rle_chars(it.x[t]);
    s = Reduce(tmp).Sum(s);
    if (threadIdx.x == 0) tile_sum[blockIdx.x] = s;
}

// One block: tile_sum becomes its exclusive prefix, in place.
__global__ void __launch_bounds__(kRleScanThreads)
rle_scan_tiles(long long *__restrict__ tile_sum, long long ntiles)
{
    using Scan = cub::BlockScan<long long, kRleScanThreads>;
    __shared__ typename Scan::TempStorage tmp;
    __shared__ long long carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (long long t0 = 0; t0 < ntiles; t0 += kRleScanThreads) {
        const long long t = t0 + threadIdx.x;
        const long long v = t < ntiles ? tile_sum[t] : 0;
        long long ex, total;
        Scan(tmp).ExclusiveSum(v, ex, total);
        if (t < ntiles) tile_sum[t] = carry + ex;
        __syncthreads();                         // every thread has read carry and tmp
        if (threadIdx.x == 0) carry += total;
        __syncthreads();
    }
}

// Writes the characters; byte_offsets[i] = where instance i's string starts, byte_offsets[I] = the total.
__global__ void __launch_bounds__(kRleTileThreads)
rle_write(RleCounts rc, const long long *__restrict__ tile_off, long long *__restrict__ byte_offsets,
          char *__restrict__ chars)
{
    using Scan = cub::BlockScan<long long, kRleTileThreads>;
    __shared__ typename Scan::TempStorage tmp;
    RleItems it;
    it.load(rc, (long long)blockIdx.x * kRleTile + (long long)threadIdx.x * kRleTileItems);
    long long s = 0;
#pragma unroll
    for (int t = 0; t < kRleTileItems; ++t)
        if (t < it.n) s += rle_chars(it.x[t]);
    long long o;
    Scan(tmp).ExclusiveSum(s, o);
    if (it.n == 0) return;
    o += tile_off[blockIdx.x];
    long long i = rc.owner(it.g0);
#pragma unroll
    for (int t = 0; t < kRleTileItems; ++t) {
        if (t >= it.n) break;
        const long long g = it.g0 + t;
        while (i + 1 < rc.I && rc.start(i + 1) <= g) ++i;
        if (g == rc.start(i)) byte_offsets[i] = o;
        long long x = it.x[t];
        bool more = true;
        while (more) {
            int c = (int)(x & 0x1f);
            x >>= 5;
            more = (c & 0x10) ? x != -1 : x != 0;
            if (more) c |= 0x20;
            chars[o++] = (char)(c + 48);
        }
        if (g == rc.N - 1) byte_offsets[rc.I] = o;
    }
}

}  // namespace msda
