// msda_vlfuse_tc.cuh -- tensor-core versions of the four product kernels of msda_vlfuse.cuh (the fused image-text
// attention of UNINEXT's early-fusion block), in TF32 and in bf16 mode, sm_90a.  DESIGN.md section 3.11, "TF32 mode" and
// "bf16 mode".
//
// vlf_tc_fwd_rows / _fwd_cols / _bwd_rows / _bwd_cols (TF32 mode, fp32 tensors) and vlf_bf16_fwd_rows / ... (bf16 mode,
// bf16 tensors) compute what vlf_fwd_rows / _fwd_cols / _bwd_rows / _bwd_cols compute, with every S x T x d product on
// warp-level tensor cores: mma.sync.m16n8k8 TF32 or mma.sync.m16n8k16 bf16.  Each kernel body is written once, as a
// template on the mode (Tf32, Bf16), which holds everything the modes do differently.  Params (ParamsT<element type>),
// the workspace layout, the range split, the tile geometry (64 image tokens per row-side CTA, 32 text tokens per
// column-side CTA, 256-token chunks), vlf_keep, the clamps and the other kernels (vlf_colstats, vlf_reduce,
// vlf_bwd_delta) are shared with the fp32 path.
//
// Numeric contract of both modes:
//   * everything between the products is fp32 with the formulas of the fp32 kernels (the clamps, the additive text mask,
//     max / exp / sum, the saved row and column statistics, dropout and keep_scale, delta, dS); the statistics, the
//     partial slots, the text bias and delta = rowsum(dO o O) are fp32; accumulation is fp32;
//   * every kernel forms the logits with the image-token operand (Q) as the A operand and K as B, in the same k order,
//     so the row side and the column side, forward and backward, see the same x bits (likewise dP_v and dP_l);
//   * no float atomics and a fixed reduction order: outputs are bit-identical from run to run.  Nothing is allocated and
//     nothing synchronises with the host.
// TF32 mode: every operand of every product (Q, K, Vv, Vl, dO_v, dO_l, P_v, P_l, dS) is rounded once to TF32 with
// cvt.rna.tf32.f32 (round to nearest) where it is staged in shared memory.
// bf16 mode: Q, K, Vv, Vl, dO_v and dO_l are bf16 in global memory and staged as they are; P_v, P_l and dS are formed in
// fp32 and rounded once to bf16 (cvt.rn.bf16x2.f32, round to nearest even) where they are staged; O_v, dQ and dVv are
// rounded once to bf16 where they are stored, O_l, dK and dVl once by vlf_reduce, after the range-ordered fp32 sum.
//
// Fragment layout (m16n8k8, g = lane / 4, q = lane % 4): A holds (g, q), (g+8, q), (g, q+4), (g+8, q+4); B holds
// (k = q, n = g), (q+4, g); C element e holds (g + 8 (e / 2), 2 q + e % 2), as in m16n8k16.  A warp owns MT x NT such
// tiles.  Row reductions are per-thread, then over the quad (shuffles), then over the warps sharing the row in shared
// memory, in warp order; column reductions the same over g.
//
// bf16 operands reach the tensor cores through ldmatrix (ldmatrix.trans where the staged layout is the transpose of the
// fragment's: P^T on the column side, and every V / dO / K / Q chunk of a P V product, staged [k][n]).  Every bf16 staged
// row stride is an odd multiple of 16 bytes, so the eight row addresses of each 8x8 matrix fall in distinct bank groups.
#pragma once

#include <cuda_bf16.h>

#include "msda_vlfuse.cuh"

namespace vlf {

using bf16 = __nv_bfloat16;
using ParamsH = ParamsT<bf16>;

constexpr int kLdpF = kMaxT + 4;       // row side fp32 [s][t] tiles (TF32: read as A(m = s, k = t))
constexpr int kLdqF = kColTile + 8;    // column side fp32 [s][t] tiles (TF32: read as A(m = t, k = s))
static_assert(kThreads == kMaxT && kThreads == kChunkS, "statistics are staged one token per thread");
static_assert(kKC % 16 == 0, "k chunks are whole m16n8k16 steps");

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

__device__ __forceinline__ uint32_t bf16x2(float lo, float hi) {   // lo at the lower address
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}

// Two adjacent fp32 values stored as they are, or rounded once to bf16.
__device__ __forceinline__ void store2(float *dst, float lo, float hi) {
    *reinterpret_cast<float2 *>(dst) = make_float2(lo, hi);
}
__device__ __forceinline__ void store2(bf16 *dst, float lo, float hi) {
    *reinterpret_cast<uint32_t *>(dst) = bf16x2(lo, hi);
}

// ---- TF32: mma.sync.m16n8k8 with scalar fragment loads ----------------------------------------------------------------
__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
        "{%0, %1, %2, %3};\n"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
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

// ---- bf16: mma.sync.m16n8k16 with ldmatrix fragment loads -------------------------------------------------------------
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

// One k16 step of a warp's MT x NT tiles, addressed as mma_k8's.  Lane l addresses row l % 8 of 8x8 matrix l / 8: for A
// the matrices are (m 0-7, k 0-7), (m 8-15, k 0-7), (m 0-7, k 8-15), (m 8-15, k 8-15); for B (k 0-7), (k 8-15).
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

// ---- the modes: everything in which TF32 and bf16 mode differ --------------------------------------------------------
// E: element type of the [B, L, H, d] tensors, V: 16 bytes of E, S: staged operand type.  kStep / mma: one k step of a
// warp's tiles.  stage: a 16-byte vector of a global operand as it is staged; pack: two fp32 product operands (P, dS),
// adjacent in a row, rounded to S at dst.  kLds: [row][k] staging stride; kLdp / kLdq: row side / column side [s][t]
// product operands.  kAlias: the backward kernels round their product operands in place, over the fp32 [s][t] tiles
// they are formed in, instead of writing them to buffers of their own.  kPvChunk: k chunk of bwd_cols's P V products.
struct Tf32 {
    using E = float;
    using V = float4;
    using S = float;
    static constexpr int kStep = 8;
    static constexpr int kLds = kKC + 4;      // fragment reads are conflict-free
    static constexpr int kLdp = kLdpF, kLdq = kLdqF;
    static constexpr bool kAlias = true;      // two more 64 x 260 fp32 tiles would take bwd_rows past 227 KB
    static constexpr int kPvChunk = kKC / 2;  // bwd_cols is at 248 registers for d = 256
    static constexpr bool kStagedFirst = true;
    template <int MT, int NT, bool AT, bool BT>
    static __device__ __forceinline__ void mma(float (&acc)[MT][NT][4], const S *A, int lda, const S *B, int ldb,
                                               int nlim) {
        mma_k8<MT, NT, AT, BT>(acc, A, lda, B, ldb, nlim);
    }
    static __device__ __forceinline__ V stage(V v) {
        return make_float4(to_tf32(v.x), to_tf32(v.y), to_tf32(v.z), to_tf32(v.w));
    }
    static __device__ __forceinline__ void pack(S *dst, float lo, float hi) {
        *reinterpret_cast<float2 *>(dst) = make_float2(to_tf32(lo), to_tf32(hi));
    }
};

struct Bf16 {
    using E = bf16;
    using V = uint4;
    using S = bf16;
    static constexpr int kStep = 16;
    static constexpr int kLds = kKC + 8;          // 80 bytes
    static constexpr int kLdp = kMaxT + 8;        // 528 bytes
    static constexpr int kLdq = kColTile + 8;     // 80 bytes
    static constexpr bool kAlias = false;
    static constexpr int kPvChunk = kKC;
    static constexpr bool kStagedFirst = false;
    template <int MT, int NT, bool AT, bool BT>
    static __device__ __forceinline__ void mma(float (&acc)[MT][NT][4], const S *A, int lda, const S *B, int ldb,
                                               int nlim) {
        mma_k16<MT, NT, AT, BT>(acc, A, lda, B, ldb, nlim);
    }
    static __device__ __forceinline__ V stage(V v) { return v; }
    static __device__ __forceinline__ void pack(S *dst, float lo, float hi) { store2(dst, lo, hi); }
};

// A CTA's shared memory: NF fp32 words and NS elements of the staged type (staging and product operands), each group
// contiguous, the staged group first when M::kStagedFirst.  f / s: the base of each group.
template <class M, int NF, int NS>
struct Smem {
    using S = typename M::S;
    static constexpr int kBytes = NF * 4 + NS * (int)sizeof(S);
    static_assert(kBytes <= 227 * 1024, "exceeds the sm_90 shared-memory limit per block");
    float *f;
    S *s;
    __device__ __forceinline__ explicit Smem(float4 *base) {
        char *b = reinterpret_cast<char *>(base);
        f = reinterpret_cast<float *>(b + (M::kStagedFirst ? NS * sizeof(S) : 0));
        s = reinterpret_cast<S *>(b + (M::kStagedFirst ? 0 : NF * 4));
    }
};
template <class M>
using FwdRowsSmem = Smem<M, 8 * kRowTile + 5 * kMaxT, (kRowTile + kMaxT) * M::kLds + kRowTile * M::kLdp>;
template <class M>
using FwdColsSmem = Smem<M, 2 * kColTile, (kChunkS + kColTile) * M::kLds + kChunkS * M::kLdq>;
template <class M>
using BwdRowsSmem = Smem<M, 2 * kRowTile * kLdpF + 4 * kMaxT,
                         (kRowTile + kMaxT) * M::kLds + (M::kAlias ? 0 : 2 * kRowTile * M::kLdp)>;
template <class M>
using BwdColsSmem = Smem<M, 3 * kChunkS * kLdqF + 4 * kColTile + 3 * kChunkS,
                         (kChunkS + kColTile) * M::kLds + (M::kAlias ? 0 : 2 * kChunkS * M::kLdq)>;

// ---- staging and the two product shapes -------------------------------------------------------------------------------
// A KC-wide chunk of ROWS rows of a row-major global operand (row stride ld; rows at or past `valid` read as zero),
// held in registers between its load and its store to dst[r * M::kLds + k], staged by M::stage.
template <class M, int ROWS, int KC>
struct RowChunk {
    using E = typename M::E;
    using V = typename M::V;
    static constexpr int W = 16 / sizeof(E), NV = ROWS * (KC / W), N = (NV + kThreads - 1) / kThreads;   // vectors
    V v[N];
    __device__ __forceinline__ void load(const E *src, int valid, long ld, int kc) {
#pragma unroll
        for (int i = 0; i < N; ++i) {
            const int idx = threadIdx.x + i * kThreads, r = idx / (KC / W), k = (idx % (KC / W)) * W;
            if (NV % kThreads && idx >= NV) break;
            v[i] = r < valid ? __ldg(reinterpret_cast<const V *>(src + r * ld + kc + k)) : V{};
        }
    }
    __device__ __forceinline__ void store(typename M::S *dst) const {
#pragma unroll
        for (int i = 0; i < N; ++i) {
            const int idx = threadIdx.x + i * kThreads, r = idx / (KC / W), k = (idx % (KC / W)) * W;
            if (NV % kThreads && idx >= NV) break;
            *reinterpret_cast<V *>(dst + r * M::kLds + k) = M::stage(v[i]);
        }
    }
};

// KC rows (k = kc .. kc + KC - 1) of a row-major global operand [k][D] (row stride ld; rows at or past `valid` read as
// zero), stored to dst[k * (D + 8) + n], staged by M::stage.
template <class M, int D, int KC>
struct KChunk {
    using E = typename M::E;
    using V = typename M::V;
    static constexpr int W = 16 / sizeof(E), N = KC * D / W / kThreads;
    V v[N];
    __device__ __forceinline__ void load(const E *src, int valid, long ld, int kc) {
#pragma unroll
        for (int i = 0; i < N; ++i) {
            const int idx = threadIdx.x + i * kThreads, k = idx / (D / W), n = (idx % (D / W)) * W;
            v[i] = kc + k < valid ? __ldg(reinterpret_cast<const V *>(src + (kc + k) * ld + n)) : V{};
        }
    }
    __device__ __forceinline__ void store(typename M::S *dst) const {
#pragma unroll
        for (int i = 0; i < N; ++i) {
            const int idx = threadIdx.x + i * kThreads, k = idx / (D / W), n = (idx % (D / W)) * W;
            *reinterpret_cast<V *>(dst + k * (D + 8) + n) = M::stage(v[i]);
        }
    }
};

template <int MT, int NT>
__device__ __forceinline__ void zero(float (&acc)[MT][NT][4]) {
#pragma unroll
    for (int i = 0; i < MT; ++i)
#pragma unroll
        for (int j = 0; j < NT; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.f;
}

// acc += A B^T over the inner dimension KD (a multiple of kKC).  A: MROWS rows, B: NROWS rows, both row-major in global
// memory with row stride ld.  kKC-wide chunks are staged in As / Bs, the next one loaded into registers while this one
// runs; k runs in steps of M::kStep from 0.  Warp w owns rows (w / WN) 16 MT .. and columns (w % WN) 8 NT ..; n-tiles
// at or past nlim are skipped.
template <class M, int MROWS, int NROWS, int WN, int MT, int NT>
__device__ __forceinline__ void mma_nt(float (&acc)[MT][NT][4], const typename M::E *A, int avalid,
                                       const typename M::E *B, int bvalid, long ld, int KD, int nlim, typename M::S *As,
                                       typename M::S *Bs) {
    const int w = threadIdx.x >> 5, m0 = (w / WN) * 16 * MT, n0 = (w % WN) * 8 * NT;
    RowChunk<M, MROWS, kKC> ra;
    RowChunk<M, NROWS, kKC> rb;
    ra.load(A, avalid, ld, 0);
    rb.load(B, bvalid, ld, 0);
#pragma unroll 1
    for (int kc = 0; kc < KD; kc += kKC) {
        __syncthreads();
        ra.store(As);
        rb.store(Bs);
        __syncthreads();
        if (kc + kKC < KD) {
            ra.load(A, avalid, ld, kc + kKC);
            rb.load(B, bvalid, ld, kc + kKC);
        }
#pragma unroll
        for (int k = 0; k < kKC; k += M::kStep)
            M::template mma<MT, NT, false, false>(acc, As + m0 * M::kLds + k, M::kLds, Bs + n0 * M::kLds + k, M::kLds,
                                                  nlim - n0);
    }
}

// acc += P V over the inner dimension KN (a multiple of kKC).  P: product operands in shared memory, P(m, k) =
// P[m * ldp + k] (AT: P[k * ldp + m]), zero past the valid k.  V: rows [k][D] in global memory (row stride ld, rows at
// or past vvalid read as zero), staged KC rows at a time in Vs.  Warp w owns rows (w / WN) 16 MT .. and columns
// (w % WN) 8 NT ...
template <class M, int D, int WN, bool AT, int KC = kKC, int MT, int NT>
__device__ __forceinline__ void mma_nn(float (&acc)[MT][NT][4], const typename M::S *P, int ldp, const typename M::E *V,
                                       int vvalid, long ld, int KN, typename M::S *Vs) {
    const int w = threadIdx.x >> 5, m0 = (w / WN) * 16 * MT, n0 = (w % WN) * 8 * NT;
    KChunk<M, D, KC> rv;
    rv.load(V, vvalid, ld, 0);
#pragma unroll 1
    for (int kc = 0; kc < KN; kc += KC) {
        __syncthreads();
        rv.store(Vs);
        __syncthreads();
        if (kc + KC < KN) rv.load(V, vvalid, ld, kc + KC);
#pragma unroll
        for (int k = 0; k < KC; k += M::kStep)
            M::template mma<MT, NT, AT, true>(acc, AT ? P + (kc + k) * ldp + m0 : P + m0 * ldp + kc + k, ldp,
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
// written to dst[r * ldd + c] for rows < rows: as float2s, or rounded once to bf16.
template <int NT, class T>
__device__ __forceinline__ void store_frag(const float (&o)[2][NT][4], T *dst, long ldd, int r0, int c0, int rows) {
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            const int r = r0 + 16 * mi + 8 * hh;
            if (r < rows)
#pragma unroll
                for (int ni = 0; ni < NT; ++ni)
                    store2(dst + r * ldd + c0 + 8 * ni, o[mi][ni][2 * hh], o[mi][ni][2 * hh + 1]);
        }
}

// ---- forward, row side: one CTA per (64 image tokens, b*H + h); warps 2 (rows) x 4 (columns) ------------------------
template <class M, int D>
__device__ __forceinline__ void fwd_rows(ParamsT<typename M::E> p) {
    using E = typename M::E;
    using S = typename M::S;
    extern __shared__ float4 smem4[];
    const FwdRowsSmem<M> sm(smem4);
    float *rred = sm.f, *cred = rred + 8 * kRowTile, *tb = cred + 4 * kMaxT;
    S *As = sm.s, *Bs = As + kRowTile * M::kLds, *Pb = Bs + kMaxT * M::kLds;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, g = lane >> 2, q = lane & 3, wm = w >> 2, wn = w & 3;
    const int bh = blockIdx.y, b = bh / p.H, h = bh % p.H, s0 = blockIdx.x * kRowTile;
    const int T = p.T, rows = min(kRowTile, p.S - s0);
    const long ld = (long)p.H * D;
    const E *Q = p.q + ((long)b * p.S + s0) * ld + h * D;
    const E *Kp = p.k + (long)b * T * ld + h * D;
    const uint64_t seed = p.p > 0.f ? (uint64_t)*p.seed : 0;
    tb[threadIdx.x] = p.bias && (int)threadIdx.x < T ? p.bias[b * T + threadIdx.x] : 0.f;

    float acc[2][8][4];
    zero(acc);
    mma_nt<M, kRowTile, kMaxT, 4>(acc, Q, rows, Kp, T, ld, D, T, As, Bs);
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
                M::pack(Pb + r * M::kLdp + c0 + 8 * ni, pv[0], pv[1]);
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
    mma_nn<M, D, 4, false>(o, Pb, M::kLdp, p.vl + (long)b * T * ld + h * D, T, ld, (T + kKC - 1) / kKC * kKC, Bs);
    store_frag(o, p.out_v + ((long)b * p.S + s0) * ld + h * D, ld, r0, wn * (D / 4) + 2 * q, rows);
}

// ---- forward, column side: one CTA per (32 text tokens, range of image tokens, b*H + h) ----------------------------
// Per 256-token chunk: x with the 8 warps on 32 image tokens each, P_l into Pb ([s][t]), then O_l += P_l Vv with the
// warps on D / 8 columns each; the range's O_l goes to its fp32 partial slot.
template <class M, int D>
__device__ __forceinline__ void fwd_cols(ParamsT<typename M::E> p) {
    using E = typename M::E;
    using S = typename M::S;
    extern __shared__ float4 smem4[];
    const FwdColsSmem<M> sm(smem4);
    float *tcm = sm.f, *tcs = tcm + kColTile;
    S *As = sm.s, *Bs = As + kChunkS * M::kLds, *Pb = Bs + kColTile * M::kLds;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, g = lane >> 2, q = lane & 3;
    const int bh = blockIdx.z, b = bh / p.H, h = bh % p.H, t0 = blockIdx.x * kColTile;
    const int T = p.T, trows = min(kColTile, T - t0);
    const int sbeg = blockIdx.y * p.split_rows, send = min(p.S, sbeg + p.split_rows);
    const long ld = (long)p.H * D;
    const E *Kt = p.k + ((long)b * T + t0) * ld + h * D;
    const E *Q = p.q + (long)b * p.S * ld + h * D, *Vv = p.vv + (long)b * p.S * ld + h * D;
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
        mma_nt<M, kChunkS, kColTile, 1>(x, Q + sc * ld, ncols, Kt, trows, ld, D, trows, As, Bs);
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
                    M::pack(Pb + s * M::kLdq + 8 * ni + 2 * q, pl[0], pl[1]);
                }
            }
        mma_nn<M, D, 8, true>(o, Pb, M::kLdq, Vv + sc * ld, ncols, ld, (ncols + kKC - 1) / kKC * kKC, As);
    }
    store_frag(o, p.part0 + (((long)blockIdx.y * gridDim.z + bh) * T + t0) * D, D, g, w * (D / 8) + 2 * q, trows);
}

// ---- backward, row side: one CTA per (64 image tokens, b*H + h); warps 2 x 4 ----------------------------------------
// Recomputes x, P_v, P_l and both masks, forms dS in fp32 (B1 = P_v, then the vision part of dS; B2 = P_l, both
// [s][t]), then dQ = dS K and dVv = drop(P_l)^T dO_l from their roundings H1 = dS, H2 = drop(P_l).  With M::kAlias, H1
// and H2 are B1 and B2: each thread reads its cells before it overwrites them.
template <class M, int D>
__device__ __forceinline__ void bwd_rows(ParamsT<typename M::E> p) {
    using S = typename M::S;
    extern __shared__ float4 smem4[];
    const BwdRowsSmem<M> sm(smem4);
    float *B1 = sm.f, *B2 = B1 + kRowTile * kLdpF, *tcm = B2 + kRowTile * kLdpF;
    float *tcs = tcm + kMaxT, *tdl = tcs + kMaxT, *tb = tdl + kMaxT;
    S *As = sm.s, *Bs = As + kRowTile * M::kLds, *H1, *H2;
    if constexpr (M::kAlias) {
        H1 = B1;
        H2 = B2;
    } else {
        H1 = Bs + kMaxT * M::kLds;
        H2 = H1 + kRowTile * M::kLdp;
    }
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
    mma_nt<M, kRowTile, kMaxT, 4>(acc, p.q + so, rows, p.k + to, T, ld, D, T, As, Bs);
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
                *reinterpret_cast<float2 *>(B1 + r * kLdpF + c) = make_float2(pv[0], pv[1]);
                *reinterpret_cast<float2 *>(B2 + r * kLdpF + c) = make_float2(pl[0], pl[1]);
            }

    zero(acc);
    mma_nt<M, kRowTile, kMaxT, 4>(acc, p.dov + so, rows, p.vl + to, T, ld, D, T, As, Bs);            // dO_v Vl^T
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
#pragma unroll
            for (int ni = 0; ni < 8; ++ni) {
                const int r = r0 + 16 * mi + 8 * hh, c = c0 + 8 * ni;
                float2 *cell = reinterpret_cast<float2 *>(B1 + r * kLdpF + c);
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
    mma_nt<M, kRowTile, kMaxT, 4>(acc, p.vv + so, rows, p.dol + to, T, ld, D, T, As, Bs);            // (dO_l Vv^T)^T
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
#pragma unroll
            for (int ni = 0; ni < 8; ++ni) {
                const int r = r0 + 16 * mi + 8 * hh, c = c0 + 8 * ni;
                float2 *c1 = reinterpret_cast<float2 *>(B1 + r * kLdpF + c);
                float2 *c2 = reinterpret_cast<float2 *>(B2 + r * kLdpF + c);
                float dxv[2] = {c1->x, c1->y}, pl[2] = {c2->x, c2->y};
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const bool keep = drop ? vlf_keep(seed, 1, bh, s0 + r, c + j, p.p) : true;
                    const float gr = keep_scale(keep, acc[mi][ni][2 * hh + j], p);
                    const float ds = dxv[j] + pl[j] * (gr - tdl[c + j]);
                    dxv[j] = (pass >> (32 * mi + 4 * ni + 2 * hh + j)) & 1 ? ds : 0.f;
                    pl[j] = keep_scale(keep, pl[j], p);
                }
                M::pack(H1 + r * M::kLdp + c, dxv[0], dxv[1]);
                M::pack(H2 + r * M::kLdp + c, pl[0], pl[1]);
            }

    float o[2][D / 32][4];
    zero(o);
    mma_nn<M, D, 4, false>(o, H1, M::kLdp, p.k + to, T, ld, KN, Bs);
    store_frag(o, p.dq + so, ld, r0, wn * (D / 4) + 2 * q, rows);
    zero(o);
    mma_nn<M, D, 4, false>(o, H2, M::kLdp, p.dol + to, T, ld, KN, Bs);
    store_frag(o, p.dvv + so, ld, r0, wn * (D / 4) + 2 * q, rows);
}

// ---- backward, column side: one CTA per (32 text tokens, range of image tokens, b*H + h) ----------------------------
// Per chunk: the same dS, as fp32 [s][t] tiles B1 = P_v, B2 = P_l where the clamps pass (else 0), B3 = where the clamps
// pass (1 / 0), then the vision part of dS; the product operands H1 = drop(P_v) and H2 = dS (B1 and B2 with M::kAlias);
// the range's dK += dS^T Q and dVl += drop(P_v)^T dO_v into the fp32 partial slots part0 / part1.  The clamp mask
// travels in B3 rather than in a register: TF32 mode is at the register limit here.
template <class M, int D>
__device__ __forceinline__ void bwd_cols(ParamsT<typename M::E> p) {
    using S = typename M::S;
    extern __shared__ float4 smem4[];
    const BwdColsSmem<M> sm(smem4);
    float *B1 = sm.f, *B2 = B1 + kChunkS * kLdqF, *B3 = B2 + kChunkS * kLdqF;
    float *tcm = B3 + kChunkS * kLdqF, *tcs = tcm + kColTile, *tdl = tcs + kColTile, *tb = tdl + kColTile;
    float *srm = tb + kColTile, *srs = srm + kChunkS, *sdv = srs + kChunkS;
    S *As = sm.s, *Bs = As + kChunkS * M::kLds, *H1, *H2;
    if constexpr (M::kAlias) {
        H1 = B1;
        H2 = B2;
    } else {
        H1 = Bs + kColTile * M::kLds;
        H2 = H1 + kChunkS * M::kLdq;
    }
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
        mma_nt<M, kChunkS, kColTile, 1>(acc, p.q + so + sc * ld, ncols, p.k + to, trows, ld, D, trows, As, Bs);
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
                    *reinterpret_cast<float2 *>(B1 + s * kLdqF + t) = make_float2(pv[0], pv[1]);
                    *reinterpret_cast<float2 *>(B2 + s * kLdqF + t) = make_float2(pl[0], pl[1]);
                    *reinterpret_cast<float2 *>(B3 + s * kLdqF + t) = make_float2(ps[0], ps[1]);
                }

        zero(acc);
        // dO_v Vl^T
        mma_nt<M, kChunkS, kColTile, 1>(acc, p.dov + so + sc * ld, ncols, p.vl + to, trows, ld, D, trows, As, Bs);
#pragma unroll
        for (int mi = 0; mi < 2; ++mi)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh)
#pragma unroll
                for (int ni = 0; ni < 4; ++ni) {
                    const int s = w * 32 + 16 * mi + 8 * hh + g, t = 8 * ni + 2 * q;
                    float2 *c1 = reinterpret_cast<float2 *>(B1 + s * kLdqF + t);
                    float2 *c3 = reinterpret_cast<float2 *>(B3 + s * kLdqF + t);
                    float pv[2] = {c1->x, c1->y}, dxv[2] = {c3->x, c3->y};
#pragma unroll
                    for (int j = 0; j < 2; ++j) {
                        const bool keep = drop ? vlf_keep(seed, 0, bh, sc + s, t0 + t + j, p.p) : true;
                        const float gr = keep_scale(keep, acc[mi][ni][2 * hh + j], p);
                        dxv[j] = dxv[j] != 0.f ? pv[j] * (gr - sdv[s]) : 0.f;
                        pv[j] = keep_scale(keep, pv[j], p);
                    }
                    M::pack(H1 + s * M::kLdq + t, pv[0], pv[1]);
                    *c3 = make_float2(dxv[0], dxv[1]);
                }
        mma_nn<M, D, 8, true, M::kPvChunk>(dvl, H1, M::kLdq, p.dov + so + sc * ld, ncols, ld, KN, As);

        zero(acc);
        // (dO_l Vv^T)^T
        mma_nt<M, kChunkS, kColTile, 1>(acc, p.vv + so + sc * ld, ncols, p.dol + to, trows, ld, D, trows, As, Bs);
#pragma unroll
        for (int mi = 0; mi < 2; ++mi)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh)
#pragma unroll
                for (int ni = 0; ni < 4; ++ni) {
                    const int s = w * 32 + 16 * mi + 8 * hh + g, t = 8 * ni + 2 * q;
                    float2 *c2 = reinterpret_cast<float2 *>(B2 + s * kLdqF + t);
                    const float2 c3 = *reinterpret_cast<const float2 *>(B3 + s * kLdqF + t);
                    float pl[2] = {c2->x, c2->y}, dxv[2] = {c3.x, c3.y};
#pragma unroll
                    for (int j = 0; j < 2; ++j) {
                        float gr = acc[mi][ni][2 * hh + j];
                        if (drop) gr = keep_scale(vlf_keep(seed, 1, bh, sc + s, t0 + t + j, p.p), gr, p);
                        pl[j] = dxv[j] + pl[j] * (gr - tdl[t + j]);
                    }
                    M::pack(H2 + s * M::kLdq + t, pl[0], pl[1]);
                }
        mma_nn<M, D, 8, true, M::kPvChunk>(dk, H2, M::kLdq, p.q + so + sc * ld, ncols, ld, KN, As);
    }
    const long slot = (((long)blockIdx.y * gridDim.z + bh) * T + t0) * D;
    store_frag(dk, p.part0 + slot, D, g, w * (D / 8) + 2 * q, trows);
    store_frag(dvl, p.part1 + slot, D, g, w * (D / 8) + 2 * q, trows);
}

// ---- entry points: one name per mode, so that profiles and the compiler's report tell the modes apart ---------------
template <int D> __global__ void __launch_bounds__(kThreads, 1) vlf_tc_fwd_rows(Params p) { fwd_rows<Tf32, D>(p); }
template <int D> __global__ void __launch_bounds__(kThreads, 1) vlf_tc_fwd_cols(Params p) { fwd_cols<Tf32, D>(p); }
template <int D> __global__ void __launch_bounds__(kThreads, 1) vlf_tc_bwd_rows(Params p) { bwd_rows<Tf32, D>(p); }
template <int D> __global__ void __launch_bounds__(kThreads, 1) vlf_tc_bwd_cols(Params p) { bwd_cols<Tf32, D>(p); }
template <int D> __global__ void __launch_bounds__(kThreads, 1) vlf_bf16_fwd_rows(ParamsH p) { fwd_rows<Bf16, D>(p); }
template <int D> __global__ void __launch_bounds__(kThreads, 1) vlf_bf16_fwd_cols(ParamsH p) { fwd_cols<Bf16, D>(p); }
template <int D> __global__ void __launch_bounds__(kThreads, 1) vlf_bf16_bwd_rows(ParamsH p) { bwd_rows<Bf16, D>(p); }
template <int D> __global__ void __launch_bounds__(kThreads, 1) vlf_bf16_bwd_cols(ParamsH p) { bwd_cols<Bf16, D>(p); }

}  // namespace vlf
