// msda_vlfuse_tc.cuh -- TF32 tensor-core versions of the four product kernels of msda_vlfuse.cuh (the fused image-text
// attention of UNINEXT's early-fusion block), sm_90a.  DESIGN.md section 3.11, "TF32 mode".
//
// vlf_tc_fwd_rows / _fwd_cols / _bwd_rows / _bwd_cols compute what vlf_fwd_rows / _fwd_cols / _bwd_rows / _bwd_cols
// compute, with every S x T x d product on warp-level mma.sync.m16n8k8 TF32 tensor cores.  Params, the workspace layout,
// the range split, the tile geometry (64 image tokens per row-side CTA, 32 text tokens per column-side CTA, 256-token
// chunks), vlf_keep, the clamps and the other kernels (vlf_colstats, vlf_reduce, vlf_bwd_delta) are shared with the fp32
// path.
//
// Numeric contract of TF32 mode:
//   * every operand of every product (Q, K, Vv, Vl, dO_v, dO_l, P_v, P_l, dS) is rounded once to TF32 with
//     cvt.rna.tf32.f32 (round to nearest) where it is staged in shared memory; accumulation is fp32;
//   * everything between the products is fp32 with the formulas of the fp32 kernels (the clamps, the additive text mask,
//     max / exp / sum, the saved row and column statistics, dropout and keep_scale, delta, dS);
//   * every kernel forms the logits with the image-token operand (Q) as the A operand and K as B, in the same k order,
//     so the row side and the column side, forward and backward, see the same x bits (likewise dP_v and dP_l);
//   * no float atomics and a fixed reduction order: outputs are bit-identical from run to run.  Nothing is allocated and
//     nothing synchronises with the host.
//
// Fragment layout (m16n8k8, g = lane / 4, q = lane % 4): A holds (g, q), (g+8, q), (g, q+4), (g+8, q+4); B holds
// (k = q, n = g), (q+4, g); C element e holds (g + 8 (e / 2), 2 q + e % 2).  A warp owns MT x NT such tiles.  Row
// reductions are per-thread, then over the quad (shuffles), then over the warps sharing the row in shared memory, in
// warp order; column reductions the same over g.
#pragma once

#include "msda_vlfuse.cuh"

namespace vlf {

constexpr int kLds = kKC + 4;          // [row][k] staging stride: A(m, k) / B(n, k) fragment reads are conflict-free
constexpr int kLdp = kMaxT + 4;        // row side [s][t] tiles, read as A(m = s, k = t)
constexpr int kLdq = kColTile + 8;     // column side [s][t] tiles, read as A(m = t, k = s)
static_assert(kThreads == kMaxT && kThreads == kChunkS, "statistics are staged one token per thread");

constexpr int kTcFwdRowsSmem = (kRowTile * kLds + kMaxT * kLds + kRowTile * kLdp + 8 * kRowTile + 4 * kMaxT + kMaxT) * 4;
constexpr int kTcFwdColsSmem = (kChunkS * kLds + kColTile * kLds + kChunkS * kLdq + 2 * kColTile) * 4;
constexpr int kTcBwdRowsSmem = (kRowTile * kLds + kMaxT * kLds + 2 * kRowTile * kLdp + 4 * kMaxT) * 4;
constexpr int kTcBwdColsSmem = (kChunkS * kLds + kColTile * kLds + 3 * kChunkS * kLdq + 4 * kColTile + 3 * kChunkS) * 4;

// ---- per-element maths shared by the four kernels ---------------------------------------------------------------------
template <class P>
__device__ __forceinline__ float vis_logit(float x, float bias, const P &p) { return p.bias ? x + bias : x; }
__device__ __forceinline__ float vis_prob(float xb, float m, float sum) { return expf(xb - m) / sum; }
__device__ __forceinline__ float txt_prob(float x, float cm, float cs) { return expf(x - cm) / cs; }
template <class P>
__device__ __forceinline__ float keep_scale(bool keep, float v, const P &p) {
    return keep ? v * (p.p > 0.f ? p.keep_scale : 1.f) : 0.f;
}

__device__ __forceinline__ float to_tf32(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}
__device__ __forceinline__ float2 tf32x2(float a, float b) { return make_float2(to_tf32(a), to_tf32(b)); }

__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
        "{%0, %1, %2, %3};\n"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

template <int MT, int NT>
__device__ __forceinline__ void zero(float (&acc)[MT][NT][4]) {
#pragma unroll
    for (int i = 0; i < MT; ++i)
#pragma unroll
        for (int j = 0; j < NT; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.f;
}

// One k8 step of a warp's MT x NT tiles.  A(m, k) = A[m * lda + k] (AT: A[k * lda + m]); B(k, n) = B[n * ldb + k]
// (BT: B[k * ldb + n]); A and B point at the warp's first row / column at the step's k, and hold TF32 values.  n-tiles
// at or past nlim are skipped.  lda / ldb = 4 (mod 32) for the plain reads and 8 (mod 32) for the transposed ones.
template <int MT, int NT, bool AT, bool BT>
__device__ __forceinline__ void mma_k8(float (&acc)[MT][NT][4], const float *A, int lda, const float *B, int ldb,
                                       int nlim) {
    const int g = (threadIdx.x & 31) >> 2, q = threadIdx.x & 3;
    uint32_t a[MT][4];
#pragma unroll
    for (int mi = 0; mi < MT; ++mi) {
        const int m = mi * 16 + g;
        a[mi][0] = __float_as_uint(AT ? A[q * lda + m] : A[m * lda + q]);
        a[mi][1] = __float_as_uint(AT ? A[q * lda + m + 8] : A[(m + 8) * lda + q]);
        a[mi][2] = __float_as_uint(AT ? A[(q + 4) * lda + m] : A[m * lda + q + 4]);
        a[mi][3] = __float_as_uint(AT ? A[(q + 4) * lda + m + 8] : A[(m + 8) * lda + q + 4]);
    }
#pragma unroll
    for (int ni = 0; ni < NT; ++ni)
        if (ni * 8 < nlim) {
            const int n = ni * 8 + g;
            const uint32_t b0 = __float_as_uint(BT ? B[q * ldb + n] : B[n * ldb + q]);
            const uint32_t b1 = __float_as_uint(BT ? B[(q + 4) * ldb + n] : B[n * ldb + q + 4]);
#pragma unroll
            for (int mi = 0; mi < MT; ++mi) mma_tf32(acc[mi][ni], a[mi], b0, b1);
        }
}

// A KC-wide chunk of ROWS rows of a row-major global operand (row stride ld; rows at or past `valid` read as zero),
// held in registers between its load and its store to dst[r * kLds + k], rounded to TF32.
template <int ROWS, int KC>
struct RowChunk {
    static constexpr int E = ROWS * (KC / 4), N = (E + kThreads - 1) / kThreads;   // float4s, per thread
    float4 v[N];
    __device__ __forceinline__ void load(const float *src, int valid, long ld, int kc) {
#pragma unroll
        for (int i = 0; i < N; ++i) {
            const int idx = threadIdx.x + i * kThreads, r = idx / (KC / 4), k4 = (idx % (KC / 4)) * 4;
            if (E % kThreads && idx >= E) break;
            v[i] = r < valid ? ld4(src + r * ld + kc + k4) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
    __device__ __forceinline__ void store(float *dst) const {
#pragma unroll
        for (int i = 0; i < N; ++i) {
            const int idx = threadIdx.x + i * kThreads, r = idx / (KC / 4), k4 = (idx % (KC / 4)) * 4;
            if (E % kThreads && idx >= E) break;
            *reinterpret_cast<float4 *>(dst + r * kLds + k4) =
                make_float4(to_tf32(v[i].x), to_tf32(v[i].y), to_tf32(v[i].z), to_tf32(v[i].w));
        }
    }
};

// KC rows (k = kc .. kc + KC - 1) of a row-major global operand [k][D] (row stride ld; rows at or past `valid` read as
// zero), stored to dst[k * (D + 8) + n], rounded to TF32.
template <int D, int KC>
struct KChunk {
    static constexpr int N = KC * D / 4 / kThreads;
    float4 v[N];
    __device__ __forceinline__ void load(const float *src, int valid, long ld, int kc) {
#pragma unroll
        for (int i = 0; i < N; ++i) {
            const int idx = threadIdx.x + i * kThreads, k = idx / (D / 4), n4 = (idx % (D / 4)) * 4;
            v[i] = kc + k < valid ? ld4(src + (kc + k) * ld + n4) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
    __device__ __forceinline__ void store(float *dst) const {
#pragma unroll
        for (int i = 0; i < N; ++i) {
            const int idx = threadIdx.x + i * kThreads, k = idx / (D / 4), n4 = (idx % (D / 4)) * 4;
            *reinterpret_cast<float4 *>(dst + k * (D + 8) + n4) =
                make_float4(to_tf32(v[i].x), to_tf32(v[i].y), to_tf32(v[i].z), to_tf32(v[i].w));
        }
    }
};

// acc += A B^T over the inner dimension KD (a multiple of kKC).  A: MROWS rows, B: NROWS rows, both row-major in global
// memory with row stride ld.  KC-wide chunks are staged in As / Bs, the next one loaded into registers while this one
// runs; the k order (steps of 8 from 0) does not depend on KC.  Warp w owns rows (w / WN) 16 MT .. and columns
// (w % WN) 8 NT ..; n-tiles at or past nlim are skipped.
template <int MROWS, int NROWS, int WN, int KC = kKC, int MT, int NT>
__device__ __forceinline__ void tc_nt(float (&acc)[MT][NT][4], const float *A, int avalid, const float *B, int bvalid,
                                      long ld, int KD, int nlim, float *As, float *Bs) {
    const int w = threadIdx.x >> 5, m0 = (w / WN) * 16 * MT, n0 = (w % WN) * 8 * NT;
    RowChunk<MROWS, KC> ra;
    RowChunk<NROWS, KC> rb;
    ra.load(A, avalid, ld, 0);
    rb.load(B, bvalid, ld, 0);
#pragma unroll 1
    for (int kc = 0; kc < KD; kc += KC) {
        __syncthreads();
        ra.store(As);
        rb.store(Bs);
        __syncthreads();
        if (kc + KC < KD) {
            ra.load(A, avalid, ld, kc + KC);
            rb.load(B, bvalid, ld, kc + KC);
        }
#pragma unroll
        for (int k = 0; k < KC; k += 8)
            mma_k8<MT, NT, false, false>(acc, As + m0 * kLds + k, kLds, Bs + n0 * kLds + k, kLds, nlim - n0);
    }
}

// acc += P V over the inner dimension KN (a multiple of kKC).  P: TF32 values in shared memory, P(m, k) = P[m * ldp + k]
// (AT: P[k * ldp + m]), zero past the valid k.  V: rows [k][D] in global memory (row stride ld, rows at or past vvalid
// read as zero), staged KC rows at a time in Vs.  Warp w owns rows (w / WN) 16 MT .. and columns (w % WN) 8 NT ...
template <int D, int WN, bool AT, int KC = kKC, int MT, int NT>
__device__ __forceinline__ void tc_nn(float (&acc)[MT][NT][4], const float *P, int ldp, const float *V, int vvalid,
                                      long ld, int KN, float *Vs) {
    const int w = threadIdx.x >> 5, m0 = (w / WN) * 16 * MT, n0 = (w % WN) * 8 * NT;
    KChunk<D, KC> rv;
    rv.load(V, vvalid, ld, 0);
#pragma unroll 1
    for (int kc = 0; kc < KN; kc += KC) {
        __syncthreads();
        rv.store(Vs);
        __syncthreads();
        if (kc + KC < KN) rv.load(V, vvalid, ld, kc + KC);
#pragma unroll
        for (int k = 0; k < KC; k += 8)
            mma_k8<MT, NT, AT, true>(acc, AT ? P + (kc + k) * ldp + m0 : P + m0 * ldp + kc + k, ldp,
                                     Vs + k * (D + 8) + n0, D + 8, NT * 8);
    }
}

__device__ __forceinline__ float quad_max(float v) {
    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
    return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v + __shfl_xor_sync(0xffffffffu, v, 2);
}
__device__ __forceinline__ float g_max(float v) {   // over g = lane / 4
    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 4));
    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 8));
    return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 16));
}
__device__ __forceinline__ float g_sum(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 4);
    v += __shfl_xor_sync(0xffffffffu, v, 8);
    return v + __shfl_xor_sync(0xffffffffu, v, 16);
}

// Output fragments [2][NT][4] of a warp whose rows start at row r0 (= 16-row tile base + g) and columns at c0 (+ 2 q),
// written as float2s to dst[r * ldd + c] for rows < rows.
template <int NT>
__device__ __forceinline__ void store_frag(const float (&o)[2][NT][4], float *dst, long ldd, int r0, int c0, int rows) {
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            const int r = r0 + 16 * mi + 8 * hh;
            if (r < rows)
#pragma unroll
                for (int ni = 0; ni < NT; ++ni)
                    *reinterpret_cast<float2 *>(dst + r * ldd + c0 + 8 * ni) =
                        make_float2(o[mi][ni][2 * hh], o[mi][ni][2 * hh + 1]);
        }
}

// ---- forward, row side: one CTA per (64 image tokens, b*H + h); warps 2 (rows) x 4 (columns) ------------------------
template <int D>
__global__ void __launch_bounds__(kThreads, 1) vlf_tc_fwd_rows(Params p) {
    extern __shared__ float4 smem4[];
    float *As = reinterpret_cast<float *>(smem4), *Bs = As + kRowTile * kLds, *Pb = Bs + kMaxT * kLds;
    float *rred = Pb + kRowTile * kLdp, *cred = rred + 8 * kRowTile, *tb = cred + 4 * kMaxT;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, g = lane >> 2, q = lane & 3, wm = w >> 2, wn = w & 3;
    const int bh = blockIdx.y, b = bh / p.H, h = bh % p.H, s0 = blockIdx.x * kRowTile;
    const int T = p.T, rows = min(kRowTile, p.S - s0);
    const long ld = (long)p.H * D;
    const float *Q = p.q + ((long)b * p.S + s0) * ld + h * D;
    const float *Kp = p.k + (long)b * T * ld + h * D;
    const uint64_t seed = p.p > 0.f ? (uint64_t)*p.seed : 0;
    tb[threadIdx.x] = p.bias && (int)threadIdx.x < T ? p.bias[b * T + threadIdx.x] : 0.f;

    float acc[2][8][4];
    zero(acc);
    tc_nt<kRowTile, kMaxT, 4>(acc, Q, rows, Kp, T, ld, D, T, As, Bs);
    // acc[mi][ni][2 hh + j] is x[r0 + 16 mi + 8 hh][c0 + 8 ni + j]
    const int r0 = wm * 32 + g, c0 = wn * 64 + 2 * q;

    float rm[2][2], rs[2][2];
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            float m = -INFINITY;
#pragma unroll
            for (int ni = 0; ni < 8; ++ni)
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const int c = c0 + 8 * ni + j;
                    const float x = clamp_logit(acc[mi][ni][2 * hh + j], p);
                    acc[mi][ni][2 * hh + j] = x;
                    if (c < T) m = fmaxf(m, vis_logit(x, tb[c], p));
                }
            m = quad_max(m);
            if (q == 0) rred[wn * kRowTile + r0 + 16 * mi + 8 * hh] = m;
        }
    __syncthreads();
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            const int r = r0 + 16 * mi + 8 * hh;
            float m = rred[r];
            for (int k = 1; k < 4; ++k) m = fmaxf(m, rred[k * kRowTile + r]);
            float sum = 0.f;
#pragma unroll
            for (int ni = 0; ni < 8; ++ni)
#pragma unroll
                for (int j = 0; j < 2; ++j)
                    if (c0 + 8 * ni + j < T) sum += expf(vis_logit(acc[mi][ni][2 * hh + j], tb[c0 + 8 * ni + j], p) - m);
            sum = quad_sum(sum);
            if (q == 0) rred[(4 + wn) * kRowTile + r] = sum;
            rm[mi][hh] = m;
        }
    __syncthreads();
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            const int r = r0 + 16 * mi + 8 * hh;
            float sum = rred[4 * kRowTile + r];
            for (int k = 5; k < 8; ++k) sum += rred[k * kRowTile + r];
            rs[mi][hh] = sum;
            if (wn == 0 && q == 0 && r < rows) {
                p.rowstat[((long)bh * p.S + s0 + r) * 2] = rm[mi][hh];
                p.rowstat[((long)bh * p.S + s0 + r) * 2 + 1] = sum;
            }
#pragma unroll
            for (int ni = 0; ni < 8; ++ni) {
                float pv[2];
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const int c = c0 + 8 * ni + j;
                    pv[j] = 0.f;
                    if (c < T && r < rows) {
                        pv[j] = vis_prob(vis_logit(acc[mi][ni][2 * hh + j], tb[c], p), rm[mi][hh], sum);
                        if (p.p > 0.f) pv[j] = keep_scale(vlf_keep(seed, 0, bh, s0 + r, c, p.p), pv[j], p);
                    }
                }
                *reinterpret_cast<float2 *>(Pb + r * kLdp + c0 + 8 * ni) = tf32x2(pv[0], pv[1]);
            }
        }

    // column partials of x over the tile's valid rows: max, then sum of exp(x - max); over g, then the two warp rows
#pragma unroll
    for (int ni = 0; ni < 8; ++ni)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            float m = -INFINITY;
#pragma unroll
            for (int mi = 0; mi < 2; ++mi)
#pragma unroll
                for (int hh = 0; hh < 2; ++hh)
                    if (r0 + 16 * mi + 8 * hh < rows) m = fmaxf(m, acc[mi][ni][2 * hh + j]);
            m = g_max(m);
            if (g == 0) cred[wm * kMaxT + c0 + 8 * ni + j] = m;
        }
    __syncthreads();
#pragma unroll
    for (int ni = 0; ni < 8; ++ni)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int c = c0 + 8 * ni + j;
            const float m = fmaxf(cred[c], cred[kMaxT + c]);
            float l = 0.f;
#pragma unroll
            for (int mi = 0; mi < 2; ++mi)
#pragma unroll
                for (int hh = 0; hh < 2; ++hh)
                    if (r0 + 16 * mi + 8 * hh < rows) l += expf(acc[mi][ni][2 * hh + j] - m);
            l = g_sum(l);
            if (g == 0) cred[(2 + wm) * kMaxT + c] = l;
        }
    __syncthreads();
    if (threadIdx.x < T) {
        const int c = threadIdx.x;
        float *dst = p.colpart + (((long)bh * gridDim.x + blockIdx.x) * T + c) * 2;
        dst[0] = fmaxf(cred[c], cred[kMaxT + c]);
        dst[1] = cred[2 * kMaxT + c] + cred[3 * kMaxT + c];
    }

    float o[2][D / 32][4];
    zero(o);
    tc_nn<D, 4, false>(o, Pb, kLdp, p.vl + (long)b * T * ld + h * D, T, ld, (T + kKC - 1) / kKC * kKC, Bs);
    store_frag(o, p.out_v + ((long)b * p.S + s0) * ld + h * D, ld, r0, wn * (D / 4) + 2 * q, rows);
}

// ---- forward, column side: one CTA per (32 text tokens, range of image tokens, b*H + h) ----------------------------
// Per 256-token chunk: x with the 8 warps on 32 image tokens each, P_l into Pb ([s][t]), then O_l += P_l Vv with the
// warps on D / 8 columns each.
template <int D>
__global__ void __launch_bounds__(kThreads, 1) vlf_tc_fwd_cols(Params p) {
    extern __shared__ float4 smem4[];
    float *As = reinterpret_cast<float *>(smem4), *Bs = As + kChunkS * kLds, *Pb = Bs + kColTile * kLds;
    float *tcm = Pb + kChunkS * kLdq, *tcs = tcm + kColTile;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, g = lane >> 2, q = lane & 3;
    const int bh = blockIdx.z, b = bh / p.H, h = bh % p.H, t0 = blockIdx.x * kColTile;
    const int T = p.T, trows = min(kColTile, T - t0);
    const int sbeg = blockIdx.y * p.split_rows, send = min(p.S, sbeg + p.split_rows);
    const long ld = (long)p.H * D;
    const float *Kt = p.k + ((long)b * T + t0) * ld + h * D;
    const float *Q = p.q + (long)b * p.S * ld + h * D, *Vv = p.vv + (long)b * p.S * ld + h * D;
    const uint64_t seed = p.p > 0.f ? (uint64_t)*p.seed : 0;
    if (threadIdx.x < kColTile) {
        const int t = t0 + threadIdx.x;
        tcm[threadIdx.x] = t < T ? p.colstat[((long)bh * T + t) * 2] : 0.f;
        tcs[threadIdx.x] = t < T ? p.colstat[((long)bh * T + t) * 2 + 1] : 1.f;
    }
    float o[2][D / 64][4];
    zero(o);
    for (int sc = sbeg; sc < send; sc += kChunkS) {
        const int ncols = min(kChunkS, send - sc);
        float x[2][4][4];
        zero(x);
        tc_nt<kChunkS, kColTile, 1>(x, Q + sc * ld, ncols, Kt, trows, ld, D, trows, As, Bs);
        // x[mi][ni][2 hh + j] is x[s = w 32 + 16 mi + 8 hh + g][t = 8 ni + 2 q + j]
#pragma unroll
        for (int mi = 0; mi < 2; ++mi)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                const int s = w * 32 + 16 * mi + 8 * hh + g;
#pragma unroll
                for (int ni = 0; ni < 4; ++ni) {
                    float pl[2];
#pragma unroll
                    for (int j = 0; j < 2; ++j) {
                        const int t = 8 * ni + 2 * q + j;
                        pl[j] = 0.f;
                        if (t < trows && s < ncols) {
                            pl[j] = txt_prob(clamp_logit(x[mi][ni][2 * hh + j], p), tcm[t], tcs[t]);
                            if (p.p > 0.f) pl[j] = keep_scale(vlf_keep(seed, 1, bh, sc + s, t0 + t, p.p), pl[j], p);
                        }
                    }
                    *reinterpret_cast<float2 *>(Pb + s * kLdq + 8 * ni + 2 * q) = tf32x2(pl[0], pl[1]);
                }
            }
        tc_nn<D, 8, true>(o, Pb, kLdq, Vv + sc * ld, ncols, ld, (ncols + kKC - 1) / kKC * kKC, As);
    }
    store_frag(o, p.part0 + (((long)blockIdx.y * gridDim.z + bh) * T + t0) * D, D, g, w * (D / 8) + 2 * q, trows);
}

// ---- backward, row side: one CTA per (64 image tokens, b*H + h); warps 2 x 4 ----------------------------------------
// Recomputes x, P_v, P_l and both masks, forms dS, then dQ = dS K and dVv = drop(P_l)^T dO_l (B1 = P_v, then dS;
// B2 = P_l, then drop(P_l)^T, both [s][t]).
template <int D>
__global__ void __launch_bounds__(kThreads, 1) vlf_tc_bwd_rows(Params p) {
    extern __shared__ float4 smem4[];
    float *As = reinterpret_cast<float *>(smem4), *Bs = As + kRowTile * kLds, *B1 = Bs + kMaxT * kLds;
    float *B2 = B1 + kRowTile * kLdp, *tcm = B2 + kRowTile * kLdp, *tcs = tcm + kMaxT, *tdl = tcs + kMaxT;
    float *tb = tdl + kMaxT;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, g = lane >> 2, q = lane & 3, wm = w >> 2, wn = w & 3;
    const int bh = blockIdx.y, b = bh / p.H, h = bh % p.H, s0 = blockIdx.x * kRowTile;
    const int T = p.T, rows = min(kRowTile, p.S - s0), KN = (T + kKC - 1) / kKC * kKC;
    const long ld = (long)p.H * D, so = ((long)b * p.S + s0) * ld + h * D, to = (long)b * T * ld + h * D;
    const uint64_t seed = p.p > 0.f ? (uint64_t)*p.seed : 0;
    const bool drop = p.p > 0.f;
    {
        const int t = threadIdx.x;
        const bool ok = t < T;
        tcm[t] = ok ? p.colstat[((long)bh * T + t) * 2] : 0.f;
        tcs[t] = ok ? p.colstat[((long)bh * T + t) * 2 + 1] : 1.f;
        tdl[t] = ok ? p.delta_l[(long)bh * T + t] : 0.f;
        tb[t] = ok && p.bias ? p.bias[b * T + t] : 0.f;
    }
    const int r0 = wm * 32 + g, c0 = wn * 64 + 2 * q;
    float rm[2][2], rs[2][2], dv[2][2];
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            const int r = r0 + 16 * mi + 8 * hh;
            const long s = (long)bh * p.S + s0 + (r < rows ? r : 0);
            rm[mi][hh] = p.rowstat[s * 2];
            rs[mi][hh] = p.rowstat[s * 2 + 1];
            dv[mi][hh] = p.delta_v[s];
        }

    float acc[2][8][4];
    uint64_t pass = 0;   // bit 32 mi + 4 ni + e: the clamps pass the gradient of acc[mi][ni][e]
    zero(acc);
    tc_nt<kRowTile, kMaxT, 4>(acc, p.q + so, rows, p.k + to, T, ld, D, T, As, Bs);
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
#pragma unroll
            for (int ni = 0; ni < 8; ++ni) {
                const int r = r0 + 16 * mi + 8 * hh, c = c0 + 8 * ni;
                float pv[2], pl[2];
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const float a = acc[mi][ni][2 * hh + j], x = clamp_logit(a, p);
                    const bool ok = c + j < T && r < rows;
                    if (clamp_passes(a, p)) pass |= 1ull << (32 * mi + 4 * ni + 2 * hh + j);
                    pv[j] = ok ? vis_prob(vis_logit(x, tb[c + j], p), rm[mi][hh], rs[mi][hh]) : 0.f;
                    pl[j] = ok ? txt_prob(x, tcm[c + j], tcs[c + j]) : 0.f;
                }
                *reinterpret_cast<float2 *>(B1 + r * kLdp + c) = make_float2(pv[0], pv[1]);
                *reinterpret_cast<float2 *>(B2 + r * kLdp + c) = make_float2(pl[0], pl[1]);
            }

    zero(acc);
    tc_nt<kRowTile, kMaxT, 4>(acc, p.dov + so, rows, p.vl + to, T, ld, D, T, As, Bs);            // dO_v Vl^T
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
#pragma unroll
            for (int ni = 0; ni < 8; ++ni) {
                const int r = r0 + 16 * mi + 8 * hh, c = c0 + 8 * ni;
                float2 *cell = reinterpret_cast<float2 *>(B1 + r * kLdp + c);
                float pv[2] = {cell->x, cell->y};
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    float gr = acc[mi][ni][2 * hh + j];
                    if (drop) gr = keep_scale(vlf_keep(seed, 0, bh, s0 + r, c + j, p.p), gr, p);
                    pv[j] = pv[j] * (gr - dv[mi][hh]);
                }
                *cell = make_float2(pv[0], pv[1]);
            }

    zero(acc);
    tc_nt<kRowTile, kMaxT, 4>(acc, p.vv + so, rows, p.dol + to, T, ld, D, T, As, Bs);            // (dO_l Vv^T)^T
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
#pragma unroll
            for (int ni = 0; ni < 8; ++ni) {
                const int r = r0 + 16 * mi + 8 * hh, c = c0 + 8 * ni;
                float2 *c1 = reinterpret_cast<float2 *>(B1 + r * kLdp + c), *c2 = reinterpret_cast<float2 *>(B2 + r * kLdp + c);
                float dxv[2] = {c1->x, c1->y}, pl[2] = {c2->x, c2->y};
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const bool keep = drop ? vlf_keep(seed, 1, bh, s0 + r, c + j, p.p) : true;
                    const float gr = keep_scale(keep, acc[mi][ni][2 * hh + j], p);
                    const float ds = dxv[j] + pl[j] * (gr - tdl[c + j]);
                    dxv[j] = (pass >> (32 * mi + 4 * ni + 2 * hh + j)) & 1 ? ds : 0.f;
                    pl[j] = keep_scale(keep, pl[j], p);
                }
                *c1 = tf32x2(dxv[0], dxv[1]);
                *c2 = tf32x2(pl[0], pl[1]);
            }

    float o[2][D / 32][4];
    zero(o);
    tc_nn<D, 4, false>(o, B1, kLdp, p.k + to, T, ld, KN, Bs);
    store_frag(o, p.dq + so, ld, r0, wn * (D / 4) + 2 * q, rows);
    zero(o);
    tc_nn<D, 4, false>(o, B2, kLdp, p.dol + to, T, ld, KN, Bs);
    store_frag(o, p.dvv + so, ld, r0, wn * (D / 4) + 2 * q, rows);
}

// ---- backward, column side: one CTA per (32 text tokens, range of image tokens, b*H + h) ----------------------------
// Per chunk: the same dS (as [s][t] tiles: B1 = P_v, then drop(P_v); B2 = P_l where the clamps pass (else 0), then dS;
// B3 = where the clamps pass (1 / 0), then the vision part of dS), and the range's dK += dS^T Q, dVl += drop(P_v)^T dO_v
// into partial slots part0 / part1.  The clamp mask travels in B3 rather than in a register: this kernel is at the
// register limit.
template <int D>
__global__ void __launch_bounds__(kThreads, 1) vlf_tc_bwd_cols(Params p) {
    extern __shared__ float4 smem4[];
    float *As = reinterpret_cast<float *>(smem4), *Bs = As + kChunkS * kLds, *B1 = Bs + kColTile * kLds;
    float *B2 = B1 + kChunkS * kLdq, *B3 = B2 + kChunkS * kLdq, *tcm = B3 + kChunkS * kLdq, *tcs = tcm + kColTile;
    float *tdl = tcs + kColTile, *tb = tdl + kColTile, *srm = tb + kColTile, *srs = srm + kChunkS, *sdv = srs + kChunkS;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, g = lane >> 2, q = lane & 3;
    const int bh = blockIdx.z, b = bh / p.H, h = bh % p.H, t0 = blockIdx.x * kColTile;
    const int T = p.T, trows = min(kColTile, T - t0);
    const int sbeg = blockIdx.y * p.split_rows, send = min(p.S, sbeg + p.split_rows);
    const long ld = (long)p.H * D, to = ((long)b * T + t0) * ld + h * D, so = (long)b * p.S * ld + h * D;
    const uint64_t seed = p.p > 0.f ? (uint64_t)*p.seed : 0;
    const bool drop = p.p > 0.f;
    if (threadIdx.x < kColTile) {
        const int t = t0 + threadIdx.x;
        const bool ok = t < T;
        tcm[threadIdx.x] = ok ? p.colstat[((long)bh * T + t) * 2] : 0.f;
        tcs[threadIdx.x] = ok ? p.colstat[((long)bh * T + t) * 2 + 1] : 1.f;
        tdl[threadIdx.x] = ok ? p.delta_l[(long)bh * T + t] : 0.f;
        tb[threadIdx.x] = ok && p.bias ? p.bias[b * T + t] : 0.f;
    }
    float dk[2][D / 64][4], dvl[2][D / 64][4], acc[2][4][4];
    zero(dk);
    zero(dvl);
    for (int sc = sbeg; sc < send; sc += kChunkS) {
        const int ncols = min(kChunkS, send - sc), KN = (ncols + kKC - 1) / kKC * kKC;
        {   // the chunk's row statistics and delta_v, one image token per thread (kThreads == kChunkS)
            const long srow = (long)bh * p.S + sc + min((int)threadIdx.x, ncols - 1);
            srm[threadIdx.x] = p.rowstat[srow * 2];
            srs[threadIdx.x] = p.rowstat[srow * 2 + 1];
            sdv[threadIdx.x] = p.delta_v[srow];
        }
        zero(acc);
        tc_nt<kChunkS, kColTile, 1>(acc, p.q + so + sc * ld, ncols, p.k + to, trows, ld, D, trows, As, Bs);
        // acc[mi][ni][2 hh + j] is at s = w 32 + 16 mi + 8 hh + g, t = 8 ni + 2 q + j
#pragma unroll
        for (int mi = 0; mi < 2; ++mi)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh)
#pragma unroll
                for (int ni = 0; ni < 4; ++ni) {
                    const int s = w * 32 + 16 * mi + 8 * hh + g, t = 8 * ni + 2 * q;
                    float pv[2], pl[2], ps[2];
#pragma unroll
                    for (int j = 0; j < 2; ++j) {
                        const float a = acc[mi][ni][2 * hh + j], x = clamp_logit(a, p);
                        const bool ok = t + j < trows && s < ncols;
                        ps[j] = clamp_passes(a, p) ? 1.f : 0.f;
                        pv[j] = ok ? vis_prob(vis_logit(x, tb[t + j], p), srm[s], srs[s]) : 0.f;
                        pl[j] = ok && ps[j] != 0.f ? txt_prob(x, tcm[t + j], tcs[t + j]) : 0.f;
                    }
                    *reinterpret_cast<float2 *>(B1 + s * kLdq + t) = make_float2(pv[0], pv[1]);
                    *reinterpret_cast<float2 *>(B2 + s * kLdq + t) = make_float2(pl[0], pl[1]);
                    *reinterpret_cast<float2 *>(B3 + s * kLdq + t) = make_float2(ps[0], ps[1]);
                }

        zero(acc);
        tc_nt<kChunkS, kColTile, 1>(acc, p.dov + so + sc * ld, ncols, p.vl + to, trows, ld, D, trows, As, Bs);  // dO_v Vl^T
#pragma unroll
        for (int mi = 0; mi < 2; ++mi)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh)
#pragma unroll
                for (int ni = 0; ni < 4; ++ni) {
                    const int s = w * 32 + 16 * mi + 8 * hh + g, t = 8 * ni + 2 * q;
                    float2 *c1 = reinterpret_cast<float2 *>(B1 + s * kLdq + t), *c3 = reinterpret_cast<float2 *>(B3 + s * kLdq + t);
                    float pv[2] = {c1->x, c1->y}, dxv[2] = {c3->x, c3->y};
#pragma unroll
                    for (int j = 0; j < 2; ++j) {
                        const bool keep = drop ? vlf_keep(seed, 0, bh, sc + s, t0 + t + j, p.p) : true;
                        const float gr = keep_scale(keep, acc[mi][ni][2 * hh + j], p);
                        dxv[j] = dxv[j] != 0.f ? pv[j] * (gr - sdv[s]) : 0.f;
                        pv[j] = keep_scale(keep, pv[j], p);
                    }
                    *c1 = tf32x2(pv[0], pv[1]);
                    *c3 = make_float2(dxv[0], dxv[1]);
                }
        tc_nn<D, 8, true, kKC / 2>(dvl, B1, kLdq, p.dov + so + sc * ld, ncols, ld, KN, As);

        zero(acc);
        tc_nt<kChunkS, kColTile, 1>(acc, p.vv + so + sc * ld, ncols, p.dol + to, trows, ld, D, trows, As, Bs);  // (dO_l Vv^T)^T
#pragma unroll
        for (int mi = 0; mi < 2; ++mi)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh)
#pragma unroll
                for (int ni = 0; ni < 4; ++ni) {
                    const int s = w * 32 + 16 * mi + 8 * hh + g, t = 8 * ni + 2 * q;
                    float2 *c2 = reinterpret_cast<float2 *>(B2 + s * kLdq + t);
                    const float2 c3 = *reinterpret_cast<const float2 *>(B3 + s * kLdq + t);
                    float pl[2] = {c2->x, c2->y}, dxv[2] = {c3.x, c3.y};
#pragma unroll
                    for (int j = 0; j < 2; ++j) {
                        float gr = acc[mi][ni][2 * hh + j];
                        if (drop) gr = keep_scale(vlf_keep(seed, 1, bh, sc + s, t0 + t + j, p.p), gr, p);
                        const float ds = dxv[j] + pl[j] * (gr - tdl[t + j]);
                        pl[j] = ds;
                    }
                    *c2 = tf32x2(pl[0], pl[1]);
                }
        tc_nn<D, 8, true, kKC / 2>(dk, B2, kLdq, p.q + so + sc * ld, ncols, ld, KN, As);
    }
    const long slot = (((long)blockIdx.y * gridDim.z + bh) * T + t0) * D;
    store_frag(dk, p.part0 + slot, D, g, w * (D / 8) + 2 * q, trows);
    store_frag(dvl, p.part1 + slot, D, g, w * (D / 8) + 2 * q, trows);
}

}  // namespace vlf
