// msda_vlfuse.cuh -- fused bidirectional image-text attention of UNINEXT's early-fusion block (BiMultiHeadAttention,
// fuse_helper.py:54-139), forward and backward, fp32, sm_90a.  DESIGN.md section 3.11.
//
// Per (b, h), with Q [S, d] (already scaled), K [T, d], Vv [S, d], Vl [T, d]:
//   x    = clamp(Q K^T)                                  (each clamp optional)
//   P_v  = softmax_t(x + bias[b])                        (bias: the reference's additive text mask, -9e15 at padding)
//   P_l  = softmax_s(x^T - max_s x^T)                    (the second pair of clamps cannot change a value or a gradient)
//   O_v  = drop(P_v) Vl,  O_l = drop(P_l) Vv
// No S x T tensor is stored.  The logits are recomputed tile by tile: a row-side kernel works on 64 image tokens against
// all T <= 256 text tokens (every vision softmax is local to it), a column-side kernel on 32 text tokens against a
// range of image tokens.  Column-side results (O_l, dK, dVl) are per-range partial slots reduced in a fixed order, so
// there are no float atomics and every output is bit-identical from run to run.
//
// Products are plain fp32 FMAs on a register-tiled SIMT GEMM (8x8 or 4x8 outputs per thread): the tolerances are fp32
// ones.  Tensors are [B, L, H, d] (the Linear outputs viewed per head), rows of H*d floats.
#pragma once

#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace vlf {

constexpr int kThreads = 256;      // 8 warps; warp ty owns rows ty*RM .. ty*RM+RM-1 of a tile, lane tx columns tx + 32 j
constexpr int kKC = 32;            // inner-dimension chunk staged in shared memory
constexpr int kMaxT = 256;         // text tokens (columns of the row-side tile)
constexpr int kChunkS = 256;       // image tokens per step of the column-side kernels
constexpr int kLdb = kMaxT + 4;    // row stride of the staged B operand
constexpr int kRowTile = 64;       // image tokens per row-side CTA
constexpr int kColTile = 32;       // text tokens per column-side CTA
constexpr float kClampAbs = 50000.f;

// E: the element type of the tensors in [B, L, H, d] layout (float, or __nv_bfloat16 in bf16 mode); the text bias, the
// statistics, the partial slots and the deltas are fp32 in every mode.
template <class E>
struct ParamsT {
    const E *q, *k, *vv, *vl;              // [B,S,H,d], [B,T,H,d], [B,S,H,d], [B,T,H,d]
    const float *bias;                     // [B,T] additive text mask, or null
    const E *dov, *dol, *ov, *ol;          // backward: grad_out / out, shapes of O_v [B,S,H,d] and O_l [B,T,H,d]
    E *out_v, *out_l;
    E *dq, *dk, *dvv, *dvl;
    float *rowstat;                        // [BH, S, 2]: (max, sum of exp) of the vision softmax of each image token
    float *colstat;                        // [BH, T, 2]: (max, sum of exp) over S of the clamped logits of each text token
    float *colpart;                        // [BH, row tiles, T, 2]: per-tile column partials of the forward
    float *part0, *part1;                  // [nsplit, BH, T, d]: column-side partial slots
    float *delta_v, *delta_l;              // [BH, S], [BH, T]: rowsum(dO o O)
    const int64_t *seed;                   // device scalar; read only when p > 0
    int B, H, S, T;
    int clamp_min, clamp_max;
    float p, keep_scale;                   // dropout probability and 1 / (1 - p)
    int split_rows;                        // image tokens per column-side CTA (a multiple of kChunkS)
};
using Params = ParamsT<float>;

__device__ __forceinline__ float to_f32(float x) { return x; }
__device__ __forceinline__ float to_f32(__nv_bfloat16 x) { return __bfloat162float(x); }
__device__ __forceinline__ void store_as(float *dst, float v) { *dst = v; }
__device__ __forceinline__ void store_as(__nv_bfloat16 *dst, float v) { *dst = __float2bfloat16_rn(v); }

// ---- dropout: counter-based Philox4x32-10 keyed by (seed, direction, b*H + h, s, t) -------------------------------------
__device__ __forceinline__ uint32_t philox_first(uint64_t seed, uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3) {
    uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        c0 = hi1 ^ c1 ^ k0;
        c1 = lo1;
        c2 = hi0 ^ c3 ^ k1;
        c3 = lo0;
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
    }
    return c0;
}

// The one keep decision every kernel (and vlf_dropout_mask) uses.  dir 0 = vision P_v[s, t], 1 = text P_l[t, s].
__device__ __forceinline__ bool vlf_keep(uint64_t seed, uint32_t dir, uint32_t bh, uint32_t s, uint32_t t, float p) {
    return (float)(philox_first(seed, s, t, bh, dir) >> 8) * 5.9604644775390625e-8f >= p;
}

template <class P>
__device__ __forceinline__ float clamp_logit(float x, const P &p) {
    if (p.clamp_min) x = fmaxf(x, -kClampAbs);
    if (p.clamp_max) x = fminf(x, kClampAbs);
    return x;
}
// torch.clamp passes the gradient where min <= x <= max (inclusive).
template <class P>
__device__ __forceinline__ bool clamp_passes(float x, const P &p) {
    return (!p.clamp_min || x >= -kClampAbs) && (!p.clamp_max || x <= kClampAbs);
}

__device__ __forceinline__ float4 ld4(const float *p) { return __ldg(reinterpret_cast<const float4 *>(p)); }

// acc[i][j] += sum_k A[r][k] * B[n][k] for r = ty*RM + i, n = tx + 32 j (j < nj).  A and B are row-major in global memory
// with row stride ld; `arows` / `brows` rows are valid (the others read as zero); the inner dimension KD is a multiple of 32.
template <int RM>
__device__ __forceinline__ void mm_nt(float (&acc)[RM][8], const float *A, int arows, const float *B, int brows, long ld,
                                      int KD, int nj, float *As, float *Bs) {
    constexpr int BM = 8 * RM, LDA = BM + 4;
    const int tid = threadIdx.x, tx = tid & 31, ty = tid >> 5;
    for (int kc = 0; kc < KD; kc += kKC) {
        __syncthreads();
        for (int idx = tid; idx < BM * 8; idx += kThreads) {
            const int r = idx >> 3, k4 = (idx & 7) * 4;
            const float4 v = r < arows ? ld4(A + r * ld + kc + k4) : make_float4(0.f, 0.f, 0.f, 0.f);
            As[(k4 + 0) * LDA + r] = v.x; As[(k4 + 1) * LDA + r] = v.y;
            As[(k4 + 2) * LDA + r] = v.z; As[(k4 + 3) * LDA + r] = v.w;
        }
        for (int idx = tid; idx < nj * 32 * 8; idx += kThreads) {
            const int n = idx >> 3, k4 = (idx & 7) * 4;
            const float4 v = n < brows ? ld4(B + n * ld + kc + k4) : make_float4(0.f, 0.f, 0.f, 0.f);
            Bs[(k4 + 0) * kLdb + n] = v.x; Bs[(k4 + 1) * kLdb + n] = v.y;
            Bs[(k4 + 2) * kLdb + n] = v.z; Bs[(k4 + 3) * kLdb + n] = v.w;
        }
        __syncthreads();
#pragma unroll 4
        for (int k = 0; k < kKC; ++k) {
            float a[RM];
#pragma unroll
            for (int i = 0; i < RM; i += 4) {
                const float4 v = *reinterpret_cast<const float4 *>(As + k * LDA + ty * RM + i);
                a[i] = v.x; a[i + 1] = v.y; a[i + 2] = v.z; a[i + 3] = v.w;
            }
#pragma unroll
            for (int j = 0; j < 8; ++j)
                if (j < nj) {
                    const float b = Bs[k * kLdb + tx + 32 * j];
#pragma unroll
                    for (int i = 0; i < RM; ++i) acc[i][j] = fmaf(a[i], b, acc[i][j]);
                }
        }
    }
}

// acc[i][j] += sum_k P[k][r] * V[k][n] for r = ty*RM + i, n = tx + 32 j (j < NJ).  P is in shared memory, k-major with row
// stride 8*RM + 4, and holds zeros past the valid k; V is row-major in global memory (row stride ld, `vrows` valid rows).
template <int RM, int NJ>
__device__ __forceinline__ void mm_nn(float (&acc)[RM][8], const float *P, const float *V, int vrows, long ld, int KN,
                                      float *Bs) {
    constexpr int LDA = 8 * RM + 4;
    const int tid = threadIdx.x, tx = tid & 31, ty = tid >> 5;
    for (int kc = 0; kc < KN; kc += kKC) {
        __syncthreads();
        for (int idx = tid; idx < kKC * NJ * 8; idx += kThreads) {
            const int k = idx / (NJ * 8), n4 = (idx % (NJ * 8)) * 4;
            const float4 v = kc + k < vrows ? ld4(V + (kc + k) * ld + n4) : make_float4(0.f, 0.f, 0.f, 0.f);
            *reinterpret_cast<float4 *>(Bs + k * kLdb + n4) = v;
        }
        __syncthreads();
#pragma unroll 4
        for (int k = 0; k < kKC; ++k) {
            float a[RM];
#pragma unroll
            for (int i = 0; i < RM; i += 4) {
                const float4 v = *reinterpret_cast<const float4 *>(P + (kc + k) * LDA + ty * RM + i);
                a[i] = v.x; a[i + 1] = v.y; a[i + 2] = v.z; a[i + 3] = v.w;
            }
#pragma unroll
            for (int j = 0; j < NJ; ++j) {
                const float b = Bs[k * kLdb + tx + 32 * j];
#pragma unroll
                for (int i = 0; i < RM; ++i) acc[i][j] = fmaf(a[i], b, acc[i][j]);
            }
        }
    }
}

template <int RM>
__device__ __forceinline__ void zero(float (&acc)[RM][8]) {
#pragma unroll
    for (int i = 0; i < RM; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
}

// A thread's RM consecutive rows of column c of a k-major tile buffer (row stride 8*RM + 4), as float4s.
template <int RM>
__device__ __forceinline__ void put_col(float *buf, int c, const float (&v)[RM]) {
    float *dst = buf + c * (8 * RM + 4) + (threadIdx.x >> 5) * RM;
#pragma unroll
    for (int i = 0; i < RM; i += 4) *reinterpret_cast<float4 *>(dst + i) = make_float4(v[i], v[i + 1], v[i + 2], v[i + 3]);
}
template <int RM>
__device__ __forceinline__ void get_col(const float *buf, int c, float (&v)[RM]) {
    const float *src = buf + c * (8 * RM + 4) + (threadIdx.x >> 5) * RM;
#pragma unroll
    for (int i = 0; i < RM; i += 4) {
        const float4 f = *reinterpret_cast<const float4 *>(src + i);
        v[i] = f.x; v[i + 1] = f.y; v[i + 2] = f.z; v[i + 3] = f.w;
    }
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

template <int RM>
constexpr int smem_floats(int bufs) { return kKC * (8 * RM + 4) + kKC * kLdb + bufs * kMaxT * (8 * RM + 4); }

constexpr int kFwdRowsSmem = (smem_floats<8>(1) + 8 * kMaxT + kMaxT) * 4;
constexpr int kFwdColsSmem = smem_floats<4>(1) * 4;
constexpr int kBwdRowsSmem = smem_floats<8>(2) * 4;
constexpr int kBwdColsSmem = smem_floats<4>(3) * 4;

// ---- forward, row side: one CTA per (64 image tokens, b*H + h) ----------------------------------------------------------
// x = clamp(Q K^T) for the tile; the vision softmax (its statistics are saved), dropout, O_v = P_v Vl; and the tile's
// per-column (max, sum of exp) of x, which vlf_colstats combines.
template <int D>
__global__ void __launch_bounds__(kThreads, 1) vlf_fwd_rows(Params p) {
    extern __shared__ float4 smem4[];
    float *As = reinterpret_cast<float *>(smem4), *Bs = As + kKC * 68, *Pb = Bs + kKC * kLdb;
    float *red = Pb + kMaxT * 68, *colm = red + 8 * kMaxT;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int bh = blockIdx.y, b = bh / p.H, h = bh % p.H, s0 = blockIdx.x * kRowTile;
    const int T = p.T, nj = (T + 31) >> 5, rows = min(kRowTile, p.S - s0);
    const long ld = (long)p.H * D;
    const float *Q = p.q + ((long)b * p.S + s0) * ld + h * D;
    const float *Kp = p.k + (long)b * T * ld + h * D;
    const uint64_t seed = p.p > 0.f ? (uint64_t)*p.seed : 0;

    float acc[8][8];
    zero(acc);
    mm_nt<8>(acc, Q, rows, Kp, T, ld, D, nj, As, Bs);

    float cmax[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) cmax[j] = -INFINITY;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int r = ty * 8 + i;
        float m = -INFINITY;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int t = tx + 32 * j;
            const float x = clamp_logit(acc[i][j], p);
            acc[i][j] = x;
            if (j < nj && t < T) {
                if (r < rows) cmax[j] = fmaxf(cmax[j], x);
                m = fmaxf(m, p.bias ? x + p.bias[b * T + t] : x);
            }
        }
        m = warp_max(m);
        float sum = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int t = tx + 32 * j;
            if (j < nj && t < T) sum += expf((p.bias ? acc[i][j] + p.bias[b * T + t] : acc[i][j]) - m);
        }
        sum = warp_sum(sum);
        if (tx == 0 && r < rows) {
            p.rowstat[((long)bh * p.S + s0 + r) * 2] = m;
            p.rowstat[((long)bh * p.S + s0 + r) * 2 + 1] = sum;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int t = tx + 32 * j;
            float pv = 0.f;
            if (j < nj && t < T && r < rows) {
                pv = expf((p.bias ? acc[i][j] + p.bias[b * T + t] : acc[i][j]) - m) / sum;
                if (p.p > 0.f) pv = vlf_keep(seed, 0, bh, s0 + r, t, p.p) ? pv * p.keep_scale : 0.f;
            }
            Pb[t * 68 + r] = pv;   // read back only by the O_v product, after its barrier
        }
    }
    // column partials of x over the tile's valid rows: max, then sum of exp(x - max), each combined over warps in order
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 8; ++j)
        if (j < nj) red[ty * kMaxT + tx + 32 * j] = cmax[j];
    __syncthreads();
    if (threadIdx.x < T) {
        float m = red[threadIdx.x];
        for (int w = 1; w < 8; ++w) m = fmaxf(m, red[w * kMaxT + threadIdx.x]);
        colm[threadIdx.x] = m;
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 8; ++j)
        if (j < nj) {
            const int t = tx + 32 * j;
            float l = 0.f;
            if (t < T) {
                const float m = colm[t];
#pragma unroll
                for (int i = 0; i < 8; ++i)
                    if (ty * 8 + i < rows) l += expf(acc[i][j] - m);
            }
            red[ty * kMaxT + t] = l;
        }
    __syncthreads();
    if (threadIdx.x < T) {
        float l = 0.f;
        for (int w = 0; w < 8; ++w) l += red[w * kMaxT + threadIdx.x];
        float *dst = p.colpart + (((long)bh * gridDim.x + blockIdx.x) * T + threadIdx.x) * 2;
        dst[0] = colm[threadIdx.x];
        dst[1] = l;
    }

    zero(acc);
    mm_nn<8, D / 32>(acc, Pb, p.vl + (long)b * T * ld + h * D, T, ld, nj * 32, Bs);
    float *O = p.out_v + ((long)b * p.S + s0) * ld + h * D;
#pragma unroll
    for (int i = 0; i < 8; ++i)
        if (ty * 8 + i < rows)
#pragma unroll
            for (int j = 0; j < D / 32; ++j) O[(ty * 8 + i) * ld + tx + 32 * j] = acc[i][j];
}

// Column statistics over all S: max, and sum of exp(x - max) rescaled from the tile partials in tile order.
template <class E>
__global__ void vlf_colstats(ParamsT<E> p, int tiles) {
    const int bh = blockIdx.x, t = threadIdx.x;
    if (t >= p.T) return;
    const float *src = p.colpart + ((long)bh * tiles * p.T + t) * 2;
    const long step = (long)p.T * 2;
    float m = -INFINITY;
    for (int i = 0; i < tiles; ++i) m = fmaxf(m, src[i * step]);
    float l = 0.f;
    for (int i = 0; i < tiles; ++i) l += src[i * step + 1] * expf(src[i * step] - m);
    p.colstat[((long)bh * p.T + t) * 2] = m;
    p.colstat[((long)bh * p.T + t) * 2 + 1] = l;
}

// ---- forward, column side: one CTA per (32 text tokens, range of image tokens, b*H + h) ---------------------------------
// P_l for the tile from the column statistics, dropout, and the range's share of O_l = P_l Vv into its partial slot.
template <int D>
__global__ void __launch_bounds__(kThreads, 1) vlf_fwd_cols(Params p) {
    extern __shared__ float4 smem4[];
    float *As = reinterpret_cast<float *>(smem4), *Bs = As + kKC * 36, *Pb = Bs + kKC * kLdb;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int bh = blockIdx.z, b = bh / p.H, h = bh % p.H, t0 = blockIdx.x * kColTile;
    const int T = p.T, trows = min(kColTile, T - t0);
    const int sbeg = blockIdx.y * p.split_rows, send = min(p.S, sbeg + p.split_rows);
    const long ld = (long)p.H * D;
    const float *Kt = p.k + ((long)b * T + t0) * ld + h * D;
    const float *Q = p.q + (long)b * p.S * ld + h * D, *Vv = p.vv + (long)b * p.S * ld + h * D;
    const uint64_t seed = p.p > 0.f ? (uint64_t)*p.seed : 0;
    float cm[4], cs[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int t = t0 + ty * 4 + i;
        cm[i] = t < T ? p.colstat[((long)bh * T + t) * 2] : 0.f;
        cs[i] = t < T ? p.colstat[((long)bh * T + t) * 2 + 1] : 1.f;
    }
    float o[4][8];
    zero(o);
    for (int sc = sbeg; sc < send; sc += kChunkS) {
        const int ncols = min(kChunkS, send - sc), njs = (ncols + 31) >> 5;
        float x[4][8];
        zero(x);
        mm_nt<4>(x, Kt, trows, Q + sc * ld, ncols, ld, D, njs, As, Bs);
#pragma unroll
        for (int j = 0; j < 8; ++j)
            if (j < njs) {
                const int c = tx + 32 * j;
                float pl[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int t = t0 + ty * 4 + i;
                    pl[i] = 0.f;
                    if (t < T && c < ncols) {
                        pl[i] = expf(clamp_logit(x[i][j], p) - cm[i]) / cs[i];
                        if (p.p > 0.f) pl[i] = vlf_keep(seed, 1, bh, sc + c, t, p.p) ? pl[i] * p.keep_scale : 0.f;
                    }
                }
                put_col<4>(Pb, c, pl);
            }
        mm_nn<4, D / 32>(o, Pb, Vv + sc * ld, ncols, ld, njs * 32, Bs);
    }
    float *dst = p.part0 + (((long)blockIdx.y * gridDim.z + bh) * T + t0) * D;
#pragma unroll
    for (int i = 0; i < 4; ++i)
        if (ty * 4 + i < trows)
#pragma unroll
            for (int j = 0; j < D / 32; ++j) dst[(ty * 4 + i) * D + tx + 32 * j] = o[i][j];
}

// out[b, t, h, :] = sum over ranges, in range order, of part[range, b*H + h, t, :], rounded once to OutT.  One CTA per
// (t, b*H + h), D threads.
template <class OutT>
__global__ void vlf_reduce(const float *part, int nsplit, int BH, int H, int T, int D, OutT *out) {
    const int t = blockIdx.x, bh = blockIdx.y, n = threadIdx.x;
    const long step = (long)BH * T * D;
    const float *src = part + ((long)bh * T + t) * D + n;
    float acc = 0.f;
    for (int i = 0; i < nsplit; ++i) acc += src[i * step];
    store_as(out + (((long)(bh / H) * T + t) * H + bh % H) * D + n, acc);
}

// ---- backward ---------------------------------------------------------------------------------------------------------
// delta_v[bh, s] = dO_v . O_v and delta_l[bh, t] = dO_l . O_l in fp32; one warp per row, lanes combined in a fixed
// butterfly.
template <class E>
__global__ void vlf_bwd_delta(ParamsT<E> p, int D) {
    const long rows_v = (long)p.B * p.H * p.S, rows = rows_v + (long)p.B * p.H * p.T;
    const long g = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (g >= rows) return;
    const bool vis = g < rows_v;
    const long gi = vis ? g : g - rows_v;
    const int L = vis ? p.S : p.T;
    const int bh = (int)(gi / L), i = (int)(gi % L), b = bh / p.H, h = bh % p.H;
    const long off = (((long)b * L + i) * p.H + h) * D;
    const E *go = (vis ? p.dov : p.dol) + off, *o = (vis ? p.ov : p.ol) + off;
    float acc = 0.f;
    for (int n = lane; n < D; n += 32) acc = fmaf(to_f32(go[n]), to_f32(o[n]), acc);
    acc = warp_sum(acc);
    if (lane == 0) (vis ? p.delta_v : p.delta_l)[gi] = acc;
}

// Row side: one CTA per (64 image tokens, b*H + h).  Recomputes x, P_v, P_l and both dropout masks, forms the tile's
// dS = [clamp passes] (P_v o (dP_v - delta_v) + P_l^T o (dP_l^T - delta_l)), then dQ = dS K and dVv = drop(P_l)^T dO_l.
template <int D>
__global__ void __launch_bounds__(kThreads, 1) vlf_bwd_rows(Params p) {
    extern __shared__ float4 smem4[];
    float *As = reinterpret_cast<float *>(smem4), *Bs = As + kKC * 68, *B1 = Bs + kKC * kLdb, *B2 = B1 + kMaxT * 68;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int bh = blockIdx.y, b = bh / p.H, h = bh % p.H, s0 = blockIdx.x * kRowTile;
    const int T = p.T, nj = (T + 31) >> 5, rows = min(kRowTile, p.S - s0);
    const long ld = (long)p.H * D, so = ((long)b * p.S + s0) * ld + h * D, to = (long)b * T * ld + h * D;
    const uint64_t seed = p.p > 0.f ? (uint64_t)*p.seed : 0;
    const bool drop = p.p > 0.f;

    float rm[8], rs[8], dv[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int r = ty * 8 + i;
        const long s = (long)bh * p.S + s0 + (r < rows ? r : 0);
        rm[i] = p.rowstat[s * 2];
        rs[i] = p.rowstat[s * 2 + 1];
        dv[i] = p.delta_v[s];
    }
    float cm[8], cs[8], dl[8], bias[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int t = min(tx + 32 * j, T - 1);
        cm[j] = p.colstat[((long)bh * T + t) * 2];
        cs[j] = p.colstat[((long)bh * T + t) * 2 + 1];
        dl[j] = p.delta_l[(long)bh * T + t];
        bias[j] = p.bias ? p.bias[b * T + t] : 0.f;
    }

    float acc[8][8];
    uint64_t pass = 0;   // bit i*8+j: the clamps pass the gradient of element (i, j)
    zero(acc);
    mm_nt<8>(acc, p.q + so, rows, p.k + to, T, ld, D, nj, As, Bs);
#pragma unroll
    for (int j = 0; j < 8; ++j)
        if (j < nj) {
            const int t = tx + 32 * j;
            float pv[8], pl[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const bool ok = t < T && ty * 8 + i < rows;
                const float x = clamp_logit(acc[i][j], p);
                if (clamp_passes(acc[i][j], p)) pass |= 1ull << (i * 8 + j);
                pv[i] = ok ? expf((p.bias ? x + bias[j] : x) - rm[i]) / rs[i] : 0.f;
                pl[i] = ok ? expf(x - cm[j]) / cs[j] : 0.f;
            }
            put_col<8>(B1, t, pv);
            put_col<8>(B2, t, pl);
        }

    zero(acc);
    mm_nt<8>(acc, p.dov + so, rows, p.vl + to, T, ld, D, nj, As, Bs);            // dO_v Vl^T
#pragma unroll
    for (int j = 0; j < 8; ++j)
        if (j < nj) {
            const int t = tx + 32 * j;
            float pv[8];
            get_col<8>(B1, t, pv);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                float g = acc[i][j];
                if (drop) g = vlf_keep(seed, 0, bh, s0 + ty * 8 + i, t, p.p) ? g * p.keep_scale : 0.f;
                pv[i] = pv[i] * (g - dv[i]);
            }
            put_col<8>(B1, t, pv);
        }

    zero(acc);
    mm_nt<8>(acc, p.vv + so, rows, p.dol + to, T, ld, D, nj, As, Bs);            // (dO_l Vv^T)^T
#pragma unroll
    for (int j = 0; j < 8; ++j)
        if (j < nj) {
            const int t = tx + 32 * j;
            float dxv[8], pl[8];
            get_col<8>(B1, t, dxv);
            get_col<8>(B2, t, pl);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                float g = acc[i][j];
                bool keep = true;
                if (drop) keep = vlf_keep(seed, 1, bh, s0 + ty * 8 + i, t, p.p);
                g = keep ? g * (drop ? p.keep_scale : 1.f) : 0.f;
                const float ds = dxv[i] + pl[i] * (g - dl[j]);
                dxv[i] = (pass >> (i * 8 + j)) & 1 ? ds : 0.f;
                pl[i] = keep ? pl[i] * (drop ? p.keep_scale : 1.f) : 0.f;
            }
            put_col<8>(B1, t, dxv);
            put_col<8>(B2, t, pl);
        }

    zero(acc);
    mm_nn<8, D / 32>(acc, B1, p.k + to, T, ld, nj * 32, Bs);
#pragma unroll
    for (int i = 0; i < 8; ++i)
        if (ty * 8 + i < rows)
#pragma unroll
            for (int j = 0; j < D / 32; ++j) p.dq[so + (ty * 8 + i) * ld + tx + 32 * j] = acc[i][j];
    zero(acc);
    mm_nn<8, D / 32>(acc, B2, p.dol + to, T, ld, nj * 32, Bs);
#pragma unroll
    for (int i = 0; i < 8; ++i)
        if (ty * 8 + i < rows)
#pragma unroll
            for (int j = 0; j < D / 32; ++j) p.dvv[so + (ty * 8 + i) * ld + tx + 32 * j] = acc[i][j];
}

// Column side: one CTA per (32 text tokens, range of image tokens, b*H + h).  Recomputes the same dS (as its transpose)
// and accumulates the range's dK = dS^T Q and dVl = drop(P_v)^T dO_v into partial slots part0 / part1.
template <int D>
__global__ void __launch_bounds__(kThreads, 1) vlf_bwd_cols(Params p) {
    extern __shared__ float4 smem4[];
    float *As = reinterpret_cast<float *>(smem4), *Bs = As + kKC * 36, *B1 = Bs + kKC * kLdb;
    float *B2 = B1 + kMaxT * 36, *B3 = B2 + kMaxT * 36;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int bh = blockIdx.z, b = bh / p.H, h = bh % p.H, t0 = blockIdx.x * kColTile;
    const int T = p.T, trows = min(kColTile, T - t0);
    const int sbeg = blockIdx.y * p.split_rows, send = min(p.S, sbeg + p.split_rows);
    const long ld = (long)p.H * D, to = ((long)b * T + t0) * ld + h * D, so = (long)b * p.S * ld + h * D;
    const uint64_t seed = p.p > 0.f ? (uint64_t)*p.seed : 0;
    const bool drop = p.p > 0.f;
    float cm[4], cs[4], dl[4], bias[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int t = min(t0 + ty * 4 + i, T - 1);
        cm[i] = p.colstat[((long)bh * T + t) * 2];
        cs[i] = p.colstat[((long)bh * T + t) * 2 + 1];
        dl[i] = p.delta_l[(long)bh * T + t];
        bias[i] = p.bias ? p.bias[b * T + t] : 0.f;
    }
    float dk[4][8], dvl[4][8], acc[4][8];
    zero(dk);
    zero(dvl);
    for (int sc = sbeg; sc < send; sc += kChunkS) {
        const int ncols = min(kChunkS, send - sc), njs = (ncols + 31) >> 5;
        uint32_t pass = 0;
        zero(acc);
        mm_nt<4>(acc, p.k + to, trows, p.q + so + sc * ld, ncols, ld, D, njs, As, Bs);
#pragma unroll
        for (int j = 0; j < 8; ++j)
            if (j < njs) {
                const int c = tx + 32 * j;
                const long srow = (long)bh * p.S + sc + min(c, ncols - 1);
                const float rm = p.rowstat[srow * 2], rs = p.rowstat[srow * 2 + 1];
                float pv[4], pl[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const bool ok = ty * 4 + i < trows && c < ncols;
                    const float x = clamp_logit(acc[i][j], p);
                    if (clamp_passes(acc[i][j], p)) pass |= 1u << (i * 8 + j);
                    pv[i] = ok ? expf((p.bias ? x + bias[i] : x) - rm) / rs : 0.f;
                    pl[i] = ok ? expf(x - cm[i]) / cs[i] : 0.f;
                }
                put_col<4>(B1, c, pv);
                put_col<4>(B2, c, pl);
            }

        zero(acc);
        mm_nt<4>(acc, p.vl + to, trows, p.dov + so + sc * ld, ncols, ld, D, njs, As, Bs);     // (dO_v Vl^T)^T
#pragma unroll
        for (int j = 0; j < 8; ++j)
            if (j < njs) {
                const int c = tx + 32 * j;
                const float dv = p.delta_v[(long)bh * p.S + sc + min(c, ncols - 1)];
                float pv[4], dxv[4];
                get_col<4>(B1, c, pv);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    bool keep = true;
                    if (drop) keep = vlf_keep(seed, 0, bh, sc + c, t0 + ty * 4 + i, p.p);
                    const float g = keep ? acc[i][j] * (drop ? p.keep_scale : 1.f) : 0.f;
                    dxv[i] = pv[i] * (g - dv);
                    pv[i] = keep ? pv[i] * (drop ? p.keep_scale : 1.f) : 0.f;
                }
                put_col<4>(B1, c, pv);
                put_col<4>(B3, c, dxv);
            }
        mm_nn<4, D / 32>(dvl, B1, p.dov + so + sc * ld, ncols, ld, njs * 32, Bs);

        zero(acc);
        mm_nt<4>(acc, p.dol + to, trows, p.vv + so + sc * ld, ncols, ld, D, njs, As, Bs);     // dO_l Vv^T
#pragma unroll
        for (int j = 0; j < 8; ++j)
            if (j < njs) {
                const int c = tx + 32 * j;
                float pl[4], dxv[4];
                get_col<4>(B2, c, pl);
                get_col<4>(B3, c, dxv);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    float g = acc[i][j];
                    if (drop) g = vlf_keep(seed, 1, bh, sc + c, t0 + ty * 4 + i, p.p) ? g * p.keep_scale : 0.f;
                    const float ds = dxv[i] + pl[i] * (g - dl[i]);
                    pl[i] = (pass >> (i * 8 + j)) & 1 ? ds : 0.f;
                }
                put_col<4>(B2, c, pl);
            }
        mm_nn<4, D / 32>(dk, B2, p.q + so + sc * ld, ncols, ld, njs * 32, Bs);
    }
    const long slot = (((long)blockIdx.y * gridDim.z + bh) * T + t0) * D;
#pragma unroll
    for (int i = 0; i < 4; ++i)
        if (ty * 4 + i < trows)
#pragma unroll
            for (int j = 0; j < D / 32; ++j) {
                p.part0[slot + (ty * 4 + i) * D + tx + 32 * j] = dk[i][j];
                p.part1[slot + (ty * 4 + i) * D + tx + 32 * j] = dvl[i][j];
            }
}

// The keep-masks every kernel above applies, as 1.0 / 0.0: mask_v [BH, S, T] (vision), mask_l [BH, T, S] (text).
__global__ void vlf_dropout_mask(const int64_t *seed_ptr, int BH, int S, int T, float p, float *mask_v, float *mask_l) {
    const long n = (long)BH * S * T;
    const uint64_t seed = (uint64_t)*seed_ptr;
    for (long e = (long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long)gridDim.x * blockDim.x) {
        const int t = (int)(e % T), s = (int)((e / T) % S), bh = (int)(e / ((long)S * T));
        mask_v[e] = vlf_keep(seed, 0, bh, s, t, p) ? 1.f : 0.f;
        mask_l[((long)bh * T + t) * S + s] = vlf_keep(seed, 1, bh, s, t, p) ? 1.f : 0.f;
    }
}

}  // namespace vlf
