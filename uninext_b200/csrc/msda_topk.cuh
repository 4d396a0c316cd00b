// msda_topk.cuh -- block-wide top-k on unique 64-bit keys, shared by the detection post-processor (msda_detpost.cuh) and
// the two-stage query selection (msda_twostage.cuh): a radix select of the cnt-th smallest key, then a bitonic sort of
// the keys at or below it.  A key holds the descending value in its high word and the ascending index in its low word,
// so "the cnt smallest keys, ascending" is the top-k by value with ties broken by ascending index.
#pragma once

#include "msda_common.cuh"

namespace msda {

// The sort key of (value, index): descending value in the high word, ascending index in the low word.
__device__ __forceinline__ unsigned long long dp_key(float v, unsigned flat) {
    unsigned u = __float_as_uint(v);
    u ^= (u >> 31) ? 0xffffffffu : 0x80000000u;             // ascending unsigned order = ascending float order
    return ((unsigned long long)(~u) << 32) | flat;
}

// The cnt-th smallest of the n keys key_of(0 .. n-1), 1 <= cnt <= n, by a radix select 8 bits at a time from the top
// that stops once the chosen bucket is taken whole.  With unique keys exactly cnt keys are <= the result.  Every thread of
// the block calls it (it holds barriers); s_hist is [256] shared, s_digit / s_rem / s_bucket shared scalars.
template <int Threads, class KeyOf>
__device__ __forceinline__ unsigned long long block_radix_threshold(unsigned n, unsigned cnt, KeyOf key_of, unsigned *s_hist,
                                                                    int *s_digit, unsigned *s_rem, unsigned *s_bucket)
{
    const int tid = threadIdx.x;
    unsigned long long prefix = 0, pmask = 0, thr = ~0ull;
    unsigned remaining = cnt;
    for (int shift = 56; shift >= 0; shift -= 8) {
        for (int d = tid; d < 256; d += Threads) s_hist[d] = 0;
        __syncthreads();
        for (unsigned f = tid; f < n; f += Threads) {
            const unsigned long long k = key_of(f);
            if ((k & pmask) == prefix) atomicAdd(&s_hist[(k >> shift) & 255], 1u);
        }
        __syncthreads();
        if (tid == 0) {
            unsigned cum = 0;
            for (int d = 0; d < 256; ++d) {
                const unsigned h = s_hist[d];
                if (cum + h >= remaining) { *s_digit = d; *s_rem = remaining - cum; *s_bucket = h; break; }
                cum += h;
            }
        }
        __syncthreads();
        prefix |= (unsigned long long)*s_digit << shift;
        pmask |= 0xffull << shift;
        remaining = *s_rem;
        const bool whole = *s_bucket == remaining;
        __syncthreads();                        // s_digit / s_rem / s_bucket are rewritten by the next pass
        if (whole) { thr = prefix | ~pmask; break; }
    }
    return thr;
}

// Ascending bitonic sort of buf[0 .. P), P a power of two, by the whole block.  Ends with a barrier.
template <int Threads>
__device__ __forceinline__ void block_bitonic_sort(unsigned long long *buf, unsigned P)
{
    for (unsigned k = 2; k <= P; k <<= 1) {
        for (unsigned j = k >> 1; j > 0; j >>= 1) {
            for (unsigned i = threadIdx.x; i < P; i += Threads) {
                const unsigned ixj = i ^ j;
                if (ixj > i) {
                    const unsigned long long x = buf[i], y = buf[ixj];
                    if ((x > y) == ((i & k) == 0)) { buf[i] = y; buf[ixj] = x; }
                }
            }
            __syncthreads();
        }
    }
}

}  // namespace msda
