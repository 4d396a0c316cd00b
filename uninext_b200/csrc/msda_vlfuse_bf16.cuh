// msda_vlfuse_bf16.cuh -- bf16 tensor-core versions of the four product kernels of msda_vlfuse.cuh (the fused image-text
// attention of UNINEXT's early-fusion block), sm_90a.  DESIGN.md section 3.11, "bf16 mode".
//
// vlf_bf16_fwd_rows / _fwd_cols / _bwd_rows / _bwd_cols compute what vlf_tc_fwd_rows / _fwd_cols / _bwd_rows / _bwd_cols
// compute, on bf16 tensors, with every S x T x d product on warp-level mma.sync.m16n8k16 bf16 tensor cores.  The tile
// geometry, the warp layout, the fragment-order reductions and the per-element maths are those of msda_vlfuse_tc.cuh
// (the m16n8k16 accumulator fragment is laid out as the m16n8k8 one); Params (as ParamsT<__nv_bfloat16>), the workspace,
// the range split, vlf_keep, the clamps and the other kernels (vlf_colstats, vlf_reduce, vlf_bwd_delta) are shared.
//
// Numeric contract of bf16 mode:
//   * Q, K, Vv, Vl, dO_v and dO_l are bf16 in global memory and staged as they are; P_v, P_l and dS are formed in fp32
//     and rounded once to bf16 (cvt.rn.bf16x2.f32, round to nearest even) where they are staged; accumulation is fp32;
//   * everything between the products is fp32 with the formulas of the fp32 kernels, and the saved statistics, the
//     partial slots, the text bias and delta = rowsum(dO o O) are fp32;
//   * O_v, dQ and dVv are rounded once to bf16 where they are stored; O_l, dK and dVl once by vlf_reduce, after the
//     range-ordered fp32 sum;
//   * every kernel forms the logits with Q as the A operand and K as B in the same k order (steps of 16 from 0), so the
//     row side and the column side, forward and backward, see the same x bits (likewise dP_v and dP_l);
//   * no float atomics and a fixed reduction order: outputs are bit-identical from run to run.  Nothing is allocated and
//     nothing synchronises with the host.
//
// Operands reach the tensor cores through ldmatrix (ldmatrix.trans where the staged layout is the transpose of the
// fragment's: P^T on the column side, and every V / dO / K / Q chunk of a P V product, staged [k][n]).  Every staged row
// stride is an odd multiple of 16 bytes, so the eight row addresses of each 8x8 matrix fall in distinct bank groups.
#pragma once

#include <cuda_bf16.h>

#include "msda_vlfuse_tc.cuh"

namespace vlf {

using bf16 = __nv_bfloat16;
using ParamsH = ParamsT<bf16>;

constexpr int kLdsH = kKC + 8;         // [row][k] staging stride (80 bytes)
constexpr int kLdpH = kMaxT + 8;       // row side [s][t] product operands (528 bytes)
constexpr int kLdqH = kColTile + 8;    // column side [s][t] product operands (80 bytes)
static_assert(kKC % 16 == 0, "k chunks are whole m16n8k16 steps");

// Shared memory: fp32 statistics and fp32 S x T buffers first, then the bf16 staging and product-operand buffers.
constexpr int kH_FwdRowsSmem = (8 * kRowTile + 4 * kMaxT + kMaxT) * 4 + (kRowTile * kLdsH + kMaxT * kLdsH + kRowTile * kLdpH) * 2;
constexpr int kH_FwdColsSmem = 2 * kColTile * 4 + (kChunkS * kLdsH + kColTile * kLdsH + kChunkS * kLdqH) * 2;
constexpr int kH_BwdRowsSmem = (2 * kRowTile * kLdp + 4 * kMaxT) * 4 + (kRowTile * kLdsH + kMaxT * kLdsH + 2 * kRowTile * kLdpH) * 2;
constexpr int kH_BwdColsSmem =
    (3 * kChunkS * kLdq + 4 * kColTile + 3 * kChunkS) * 4 + (kChunkS * kLdsH + kColTile * kLdsH + 2 * kChunkS * kLdqH) * 2;
static_assert(kH_BwdRowsSmem <= 227 * 1024, "bwd_rows exceeds the sm_90 shared-memory limit per block");

__device__ __forceinline__ uint32_t bf16x2(float lo, float hi) {   // lo at the lower address
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}

__device__ __forceinline__ uint4 ld16(const bf16 *p) { return __ldg(reinterpret_cast<const uint4 *>(p)); }

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], const bf16 *p, bool trans) {
    const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
    if (trans)
        asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];\n"
                     : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a) : "memory");
    else
        asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];\n"
                     : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a) : "memory");
}
__device__ __forceinline__ void ldsm_x2(uint32_t &r0, uint32_t &r1, const bf16 *p, bool trans) {
    const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
    if (trans)
        asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0, %1}, [%2];\n" : "=r"(r0), "=r"(r1) : "r"(a) : "memory");
    else
        asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0, %1}, [%2];\n" : "=r"(r0), "=r"(r1) : "r"(a) : "memory");
}

__device__ __forceinline__ void mma_bf16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
        "{%0, %1, %2, %3};\n"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// One k16 step of a warp's MT x NT tiles.  A(m, k) = A[m * lda + k] (AT: A[k * lda + m]); B(k, n) = B[n * ldb + k]
// (BT: B[k * ldb + n]); A and B point at the warp's first row / column at the step's k.  n-tiles at or past nlim are
// skipped.  Lane l addresses row l % 8 of 8x8 matrix l / 8: for A the matrices are (m 0-7, k 0-7), (m 8-15, k 0-7),
// (m 0-7, k 8-15), (m 8-15, k 8-15); for B (k 0-7), (k 8-15).
template <int MT, int NT, bool AT, bool BT>
__device__ __forceinline__ void mma_k16(float (&acc)[MT][NT][4], const bf16 *A, int lda, const bf16 *B, int ldb,
                                        int nlim) {
    const int l = threadIdx.x & 31;
    uint32_t a[MT][4];
#pragma unroll
    for (int mi = 0; mi < MT; ++mi)
        ldsm_x4(a[mi], AT ? A + ((l & 7) + (l >> 4) * 8) * lda + mi * 16 + ((l >> 3) & 1) * 8
                          : A + (mi * 16 + (l & 15)) * lda + (l >> 4) * 8, AT);
#pragma unroll
    for (int ni = 0; ni < NT; ++ni)
        if (ni * 8 < nlim) {
            uint32_t b0, b1;
            ldsm_x2(b0, b1, BT ? B + (l & 15) * ldb + ni * 8 : B + (ni * 8 + (l & 7)) * ldb + ((l >> 3) & 1) * 8, BT);
#pragma unroll
            for (int mi = 0; mi < MT; ++mi) mma_bf16(acc[mi][ni], a[mi], b0, b1);
        }
}

// A KC-wide chunk of ROWS rows of a row-major bf16 global operand (row stride ld; rows at or past `valid` read as zero),
// held in registers between its load and its store to dst[r * kLdsH + k].
template <int ROWS, int KC>
struct RowChunkH {
    static constexpr int E = ROWS * (KC / 8), N = (E + kThreads - 1) / kThreads;   // 16-byte vectors, per thread
    uint4 v[N];
    __device__ __forceinline__ void load(const bf16 *src, int valid, long ld, int kc) {
#pragma unroll
        for (int i = 0; i < N; ++i) {
            const int idx = threadIdx.x + i * kThreads, r = idx / (KC / 8), k8 = (idx % (KC / 8)) * 8;
            if (E % kThreads && idx >= E) break;
            v[i] = r < valid ? ld16(src + r * ld + kc + k8) : make_uint4(0u, 0u, 0u, 0u);
        }
    }
    __device__ __forceinline__ void store(bf16 *dst) const {
#pragma unroll
        for (int i = 0; i < N; ++i) {
            const int idx = threadIdx.x + i * kThreads, r = idx / (KC / 8), k8 = (idx % (KC / 8)) * 8;
            if (E % kThreads && idx >= E) break;
            *reinterpret_cast<uint4 *>(dst + r * kLdsH + k8) = v[i];
        }
    }
};

// KC rows (k = kc .. kc + KC - 1) of a row-major bf16 global operand [k][D] (row stride ld; rows at or past `valid`
// read as zero), stored to dst[k * (D + 8) + n].
template <int D, int KC>
struct KChunkH {
    static constexpr int N = KC * D / 8 / kThreads;
    uint4 v[N];
    __device__ __forceinline__ void load(const bf16 *src, int valid, long ld, int kc) {
#pragma unroll
        for (int i = 0; i < N; ++i) {
            const int idx = threadIdx.x + i * kThreads, k = idx / (D / 8), n8 = (idx % (D / 8)) * 8;
            v[i] = kc + k < valid ? ld16(src + (kc + k) * ld + n8) : make_uint4(0u, 0u, 0u, 0u);
        }
    }
    __device__ __forceinline__ void store(bf16 *dst) const {
#pragma unroll
        for (int i = 0; i < N; ++i) {
            const int idx = threadIdx.x + i * kThreads, k = idx / (D / 8), n8 = (idx % (D / 8)) * 8;
            *reinterpret_cast<uint4 *>(dst + k * (D + 8) + n8) = v[i];
        }
    }
};

// acc += A B^T over the inner dimension KD (a multiple of kKC), as tc_nt in msda_vlfuse_tc.cuh: KC-wide chunks staged in
// As / Bs, the next one loaded into registers while this one runs, k in steps of 16 from 0.
template <int MROWS, int NROWS, int WN, int KC = kKC, int MT, int NT>
__device__ __forceinline__ void bf_nt(float (&acc)[MT][NT][4], const bf16 *A, int avalid, const bf16 *B, int bvalid,
                                      long ld, int KD, int nlim, bf16 *As, bf16 *Bs) {
    const int w = threadIdx.x >> 5, m0 = (w / WN) * 16 * MT, n0 = (w % WN) * 8 * NT;
    RowChunkH<MROWS, KC> ra;
    RowChunkH<NROWS, KC> rb;
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
        for (int k = 0; k < KC; k += 16)
            mma_k16<MT, NT, false, false>(acc, As + m0 * kLdsH + k, kLdsH, Bs + n0 * kLdsH + k, kLdsH, nlim - n0);
    }
}

// acc += P V over the inner dimension KN (a multiple of kKC), as tc_nn: P bf16 in shared memory, P(m, k) = P[m * ldp + k]
// (AT: P[k * ldp + m]), zero past the valid k; V rows [k][D] in global memory staged KC rows at a time in Vs.
template <int D, int WN, bool AT, int KC = kKC, int MT, int NT>
__device__ __forceinline__ void bf_nn(float (&acc)[MT][NT][4], const bf16 *P, int ldp, const bf16 *V, int vvalid,
                                      long ld, int KN, bf16 *Vs) {
    const int w = threadIdx.x >> 5, m0 = (w / WN) * 16 * MT, n0 = (w % WN) * 8 * NT;
    KChunkH<D, KC> rv;
    rv.load(V, vvalid, ld, 0);
#pragma unroll 1
    for (int kc = 0; kc < KN; kc += KC) {
        __syncthreads();
        rv.store(Vs);
        __syncthreads();
        if (kc + KC < KN) rv.load(V, vvalid, ld, kc + KC);
#pragma unroll
        for (int k = 0; k < KC; k += 16)
            mma_k16<MT, NT, AT, true>(acc, AT ? P + (kc + k) * ldp + m0 : P + m0 * ldp + kc + k, ldp,
                                      Vs + k * (D + 8) + n0, D + 8, NT * 8);
    }
}

// Output fragments [2][NT][4] (rows from r0, columns from c0, as store_frag), rounded once to bf16.
template <int NT>
__device__ __forceinline__ void store_frag_h(const float (&o)[2][NT][4], bf16 *dst, long ldd, int r0, int c0, int rows) {
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            const int r = r0 + 16 * mi + 8 * hh;
            if (r < rows)
#pragma unroll
                for (int ni = 0; ni < NT; ++ni)
                    *reinterpret_cast<uint32_t *>(dst + r * ldd + c0 + 8 * ni) =
                        bf16x2(o[mi][ni][2 * hh], o[mi][ni][2 * hh + 1]);
        }
}

// ---- forward, row side: one CTA per (64 image tokens, b*H + h); warps 2 (rows) x 4 (columns) ------------------------
template <int D>
__global__ void __launch_bounds__(kThreads, 1) vlf_bf16_fwd_rows(ParamsH p) {
    extern __shared__ float4 smem4[];
    float *rred = reinterpret_cast<float *>(smem4), *cred = rred + 8 * kRowTile, *tb = cred + 4 * kMaxT;
    bf16 *As = reinterpret_cast<bf16 *>(tb + kMaxT), *Bs = As + kRowTile * kLdsH, *Pb = Bs + kMaxT * kLdsH;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, g = lane >> 2, q = lane & 3, wm = w >> 2, wn = w & 3;
    const int bh = blockIdx.y, b = bh / p.H, h = bh % p.H, s0 = blockIdx.x * kRowTile;
    const int T = p.T, rows = min(kRowTile, p.S - s0);
    const long ld = (long)p.H * D;
    const bf16 *Q = p.q + ((long)b * p.S + s0) * ld + h * D;
    const bf16 *Kp = p.k + (long)b * T * ld + h * D;
    const uint64_t seed = p.p > 0.f ? (uint64_t)*p.seed : 0;
    tb[threadIdx.x] = p.bias && (int)threadIdx.x < T ? p.bias[b * T + threadIdx.x] : 0.f;

    float acc[2][8][4];
    zero(acc);
    bf_nt<kRowTile, kMaxT, 4>(acc, Q, rows, Kp, T, ld, D, T, As, Bs);
    // acc[mi][ni][2 hh + j] is x[r0 + 16 mi + 8 hh][c0 + 8 ni + j]
    const int r0 = wm * 32 + g, c0 = wn * 64 + 2 * q;

    float rm[2][2];
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
                *reinterpret_cast<uint32_t *>(Pb + r * kLdpH + c0 + 8 * ni) = bf16x2(pv[0], pv[1]);
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
    bf_nn<D, 4, false>(o, Pb, kLdpH, p.vl + (long)b * T * ld + h * D, T, ld, (T + kKC - 1) / kKC * kKC, Bs);
    store_frag_h(o, p.out_v + ((long)b * p.S + s0) * ld + h * D, ld, r0, wn * (D / 4) + 2 * q, rows);
}

// ---- forward, column side: one CTA per (32 text tokens, range of image tokens, b*H + h) ----------------------------
// Per 256-token chunk: x with the 8 warps on 32 image tokens each, P_l into Pb ([s][t]), then O_l += P_l Vv with the
// warps on D / 8 columns each; the range's O_l goes to its fp32 partial slot.
template <int D>
__global__ void __launch_bounds__(kThreads, 1) vlf_bf16_fwd_cols(ParamsH p) {
    extern __shared__ float4 smem4[];
    float *tcm = reinterpret_cast<float *>(smem4), *tcs = tcm + kColTile;
    bf16 *As = reinterpret_cast<bf16 *>(tcs + kColTile), *Bs = As + kChunkS * kLdsH, *Pb = Bs + kColTile * kLdsH;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, g = lane >> 2, q = lane & 3;
    const int bh = blockIdx.z, b = bh / p.H, h = bh % p.H, t0 = blockIdx.x * kColTile;
    const int T = p.T, trows = min(kColTile, T - t0);
    const int sbeg = blockIdx.y * p.split_rows, send = min(p.S, sbeg + p.split_rows);
    const long ld = (long)p.H * D;
    const bf16 *Kt = p.k + ((long)b * T + t0) * ld + h * D;
    const bf16 *Q = p.q + (long)b * p.S * ld + h * D, *Vv = p.vv + (long)b * p.S * ld + h * D;
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
        bf_nt<kChunkS, kColTile, 1>(x, Q + sc * ld, ncols, Kt, trows, ld, D, trows, As, Bs);
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
                    *reinterpret_cast<uint32_t *>(Pb + s * kLdqH + 8 * ni + 2 * q) = bf16x2(pl[0], pl[1]);
                }
            }
        bf_nn<D, 8, true>(o, Pb, kLdqH, Vv + sc * ld, ncols, ld, (ncols + kKC - 1) / kKC * kKC, As);
    }
    store_frag(o, p.part0 + (((long)blockIdx.y * gridDim.z + bh) * T + t0) * D, D, g, w * (D / 8) + 2 * q, trows);
}

// ---- backward, row side: one CTA per (64 image tokens, b*H + h); warps 2 x 4 ----------------------------------------
// Recomputes x, P_v, P_l and both masks, forms dS in fp32 (B1 = P_v, then the vision part of dS; B2 = P_l), then
// dQ = dS K and dVv = drop(P_l)^T dO_l from their bf16 roundings H1 = dS, H2 = drop(P_l) ([s][t]).
template <int D>
__global__ void __launch_bounds__(kThreads, 1) vlf_bf16_bwd_rows(ParamsH p) {
    extern __shared__ float4 smem4[];
    float *B1 = reinterpret_cast<float *>(smem4), *B2 = B1 + kRowTile * kLdp, *tcm = B2 + kRowTile * kLdp;
    float *tcs = tcm + kMaxT, *tdl = tcs + kMaxT, *tb = tdl + kMaxT;
    bf16 *As = reinterpret_cast<bf16 *>(tb + kMaxT), *Bs = As + kRowTile * kLdsH, *H1 = Bs + kMaxT * kLdsH;
    bf16 *H2 = H1 + kRowTile * kLdpH;
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
    bf_nt<kRowTile, kMaxT, 4>(acc, p.q + so, rows, p.k + to, T, ld, D, T, As, Bs);
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
    bf_nt<kRowTile, kMaxT, 4>(acc, p.dov + so, rows, p.vl + to, T, ld, D, T, As, Bs);            // dO_v Vl^T
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
    bf_nt<kRowTile, kMaxT, 4>(acc, p.vv + so, rows, p.dol + to, T, ld, D, T, As, Bs);            // (dO_l Vv^T)^T
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
#pragma unroll
            for (int ni = 0; ni < 8; ++ni) {
                const int r = r0 + 16 * mi + 8 * hh, c = c0 + 8 * ni;
                const float2 c1 = *reinterpret_cast<const float2 *>(B1 + r * kLdp + c);
                const float2 c2 = *reinterpret_cast<const float2 *>(B2 + r * kLdp + c);
                float dxv[2] = {c1.x, c1.y}, pl[2] = {c2.x, c2.y};
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const bool keep = drop ? vlf_keep(seed, 1, bh, s0 + r, c + j, p.p) : true;
                    const float gr = keep_scale(keep, acc[mi][ni][2 * hh + j], p);
                    const float ds = dxv[j] + pl[j] * (gr - tdl[c + j]);
                    dxv[j] = (pass >> (32 * mi + 4 * ni + 2 * hh + j)) & 1 ? ds : 0.f;
                    pl[j] = keep_scale(keep, pl[j], p);
                }
                *reinterpret_cast<uint32_t *>(H1 + r * kLdpH + c) = bf16x2(dxv[0], dxv[1]);
                *reinterpret_cast<uint32_t *>(H2 + r * kLdpH + c) = bf16x2(pl[0], pl[1]);
            }

    float o[2][D / 32][4];
    zero(o);
    bf_nn<D, 4, false>(o, H1, kLdpH, p.k + to, T, ld, KN, Bs);
    store_frag_h(o, p.dq + so, ld, r0, wn * (D / 4) + 2 * q, rows);
    zero(o);
    bf_nn<D, 4, false>(o, H2, kLdpH, p.dol + to, T, ld, KN, Bs);
    store_frag_h(o, p.dvv + so, ld, r0, wn * (D / 4) + 2 * q, rows);
}

// ---- backward, column side: one CTA per (32 text tokens, range of image tokens, b*H + h) ----------------------------
// Per chunk, as vlf_tc_bwd_cols: fp32 [s][t] tiles B1 = P_v, B2 = P_l where the clamps pass (else 0), B3 = where the
// clamps pass (1 / 0), then the vision part of dS; the product operands H1 = drop(P_v) and H2 = dS in bf16; the range's
// dK += dS^T Q and dVl += drop(P_v)^T dO_v into the fp32 partial slots part0 / part1.
template <int D>
__global__ void __launch_bounds__(kThreads, 1) vlf_bf16_bwd_cols(ParamsH p) {
    extern __shared__ float4 smem4[];
    float *B1 = reinterpret_cast<float *>(smem4), *B2 = B1 + kChunkS * kLdq, *B3 = B2 + kChunkS * kLdq;
    float *tcm = B3 + kChunkS * kLdq, *tcs = tcm + kColTile, *tdl = tcs + kColTile, *tb = tdl + kColTile;
    float *srm = tb + kColTile, *srs = srm + kChunkS, *sdv = srs + kChunkS;
    bf16 *As = reinterpret_cast<bf16 *>(sdv + kChunkS), *Bs = As + kChunkS * kLdsH, *H1 = Bs + kColTile * kLdsH;
    bf16 *H2 = H1 + kChunkS * kLdqH;
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
        bf_nt<kChunkS, kColTile, 1>(acc, p.q + so + sc * ld, ncols, p.k + to, trows, ld, D, trows, As, Bs);
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
        bf_nt<kChunkS, kColTile, 1>(acc, p.dov + so + sc * ld, ncols, p.vl + to, trows, ld, D, trows, As, Bs);  // dO_v Vl^T
#pragma unroll
        for (int mi = 0; mi < 2; ++mi)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh)
#pragma unroll
                for (int ni = 0; ni < 4; ++ni) {
                    const int s = w * 32 + 16 * mi + 8 * hh + g, t = 8 * ni + 2 * q;
                    const float2 c1 = *reinterpret_cast<const float2 *>(B1 + s * kLdq + t);
                    float2 *c3 = reinterpret_cast<float2 *>(B3 + s * kLdq + t);
                    float pv[2] = {c1.x, c1.y}, dxv[2] = {c3->x, c3->y};
#pragma unroll
                    for (int j = 0; j < 2; ++j) {
                        const bool keep = drop ? vlf_keep(seed, 0, bh, sc + s, t0 + t + j, p.p) : true;
                        const float gr = keep_scale(keep, acc[mi][ni][2 * hh + j], p);
                        dxv[j] = dxv[j] != 0.f ? pv[j] * (gr - sdv[s]) : 0.f;
                        pv[j] = keep_scale(keep, pv[j], p);
                    }
                    *reinterpret_cast<uint32_t *>(H1 + s * kLdqH + t) = bf16x2(pv[0], pv[1]);
                    *c3 = make_float2(dxv[0], dxv[1]);
                }
        bf_nn<D, 8, true>(dvl, H1, kLdqH, p.dov + so + sc * ld, ncols, ld, KN, As);

        zero(acc);
        bf_nt<kChunkS, kColTile, 1>(acc, p.vv + so + sc * ld, ncols, p.dol + to, trows, ld, D, trows, As, Bs);  // (dO_l Vv^T)^T
#pragma unroll
        for (int mi = 0; mi < 2; ++mi)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh)
#pragma unroll
                for (int ni = 0; ni < 4; ++ni) {
                    const int s = w * 32 + 16 * mi + 8 * hh + g, t = 8 * ni + 2 * q;
                    const float2 c2 = *reinterpret_cast<const float2 *>(B2 + s * kLdq + t);
                    const float2 c3 = *reinterpret_cast<const float2 *>(B3 + s * kLdq + t);
                    float pl[2] = {c2.x, c2.y}, dxv[2] = {c3.x, c3.y};
#pragma unroll
                    for (int j = 0; j < 2; ++j) {
                        float gr = acc[mi][ni][2 * hh + j];
                        if (drop) gr = keep_scale(vlf_keep(seed, 1, bh, sc + s, t0 + t + j, p.p), gr, p);
                        pl[j] = dxv[j] + pl[j] * (gr - tdl[t + j]);
                    }
                    *reinterpret_cast<uint32_t *>(H2 + s * kLdqH + t) = bf16x2(pl[0], pl[1]);
                }
        bf_nn<D, 8, true>(dk, H2, kLdqH, p.q + so + sc * ld, ncols, ld, KN, As);
    }
    const long slot = (((long)blockIdx.y * gridDim.z + bh) * T + t0) * D;
    store_frag(dk, p.part0 + slot, D, g, w * (D / 8) + 2 * q, trows);
    store_frag(dvl, p.part1 + slot, D, g, w * (D / 8) + 2 * q, trows);
}

}  // namespace vlf
