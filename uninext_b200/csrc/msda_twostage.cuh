// msda_twostage.cuh -- two-stage query selection of the DINO-style transformer (DESIGN.md section 3.15, row f-3):
// encoder memory -> enc_outputs_class, enc_outputs_coord_unact and the decoder's initial boxes
// (deformable_transformer_dino.py:153-161,216-224).  Y = enc_output(memory) is the caller's GEMM; around it:
//   twostage_head_fwd       one warp per row: Y (b_e where the row is dropped), LayerNorm -> om, mean, rstd, and the
//                           class logit om . u[n] + c[n] (clamped to +-5e4 for VL_Align's clamp);
//   twostage_head_bwd       one warp per row, kTsRows rows per CTA: g_om += g_logit * u[n], the LayerNorm backward -> g_Y
//                           (zero on dropped rows), and per-CTA partial sums of g_b_e (dropped rows), g_gamma, g_beta,
//                           g_u[n], g_c[n] written to the workspace;
//   twostage_head_reduce    the partials summed in a fixed order: no float atomics, the same bits on every run and GPU;
//   twostage_select_fwd     one CTA per image: the radix select of the k largest logits (ties: ascending row), their
//                           bitonic sort, gather + sigmoid -> reference_points; the other CTAs write coord = box + proposals;
//   twostage_select_bwd     one thread per selected coordinate: g_coord[idx] += g_ref * s * (1 - s).
#pragma once

#include "msda_layernorm.cuh"
#include "msda_topk.cuh"

namespace msda {

constexpr int kTsC = 256;                       // d_model: the kernels hold a row as 2 float4 per lane
constexpr int kTsV = kTsC / 128;
constexpr int kTsRows = 64;                     // rows per CTA of the head backward: fixed, independent of the GPU
constexpr int kTsPart = 4 * kTsC + 4;           // floats per partial: g_gamma, g_beta, g_b_e, g_u, g_c (+ 3 pad)
constexpr int kTsThreads = 1024;                // threads of twostage_select_fwd
constexpr int kTsSmemSort = 2048;               // selected keys sorted in shared memory; more sort in the workspace
constexpr float kTsClamp = 50000.f;             // VL_Align's clamp_dot_product

// The row the LayerNorm sees: Y, or b_e (= Linear of a zeroed row) where the row is dropped.
__device__ __forceinline__ void ts_load_row(const float *y, const unsigned char *keep, const float *b_e, long long row,
                                            int lane, float4 (&v)[kTsV]) {
    const float4 *src = keep[row] ? reinterpret_cast<const float4 *>(y) + row * (kTsC / 4) : reinterpret_cast<const float4 *>(b_e);
#pragma unroll
    for (int i = 0; i < kTsV; ++i) v[i] = __ldg(src + i * 32 + lane);
}

// torch.clamp(x, -5e4, 5e4): NaN stays NaN.
__device__ __forceinline__ float ts_clamp(float x) { return x > kTsClamp ? kTsClamp : (x < -kTsClamp ? -kTsClamp : x); }

// rows = N * S; warp -> row.  logit[row] = om[row] . u[n] + c[n].
__global__ void __launch_bounds__(256)
twostage_head_fwd(const float *__restrict__ y, const unsigned char *__restrict__ keep, const float *__restrict__ b_e,
                  const float *__restrict__ gamma, const float *__restrict__ beta, const float *__restrict__ u,
                  const float *__restrict__ c, long long rows, int S, float eps, int clamp, float *__restrict__ om,
                  float *__restrict__ logit, float *__restrict__ mean, float *__restrict__ rstd)
{
    const int lane = threadIdx.x & 31;
    const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (row >= rows) return;
    const int n = (int)(row / S);
    float4 v[kTsV];
    ts_load_row(y, keep, b_e, row, lane, v);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < kTsV; ++i) s += v[i].x + v[i].y + v[i].z + v[i].w;
    float mu, rs;
    ln_row_stats<kTsV>(v, s, eps, mu, rs);
    float dot = 0.f;
#pragma unroll
    for (int i = 0; i < kTsV; ++i) {
        const float4 g = __ldg(reinterpret_cast<const float4 *>(gamma) + i * 32 + lane);
        const float4 bt = __ldg(reinterpret_cast<const float4 *>(beta) + i * 32 + lane);
        const float4 uu = __ldg(reinterpret_cast<const float4 *>(u) + n * (kTsC / 4) + i * 32 + lane);
        const float4 o = ln_affine(v[i], mu, rs, g, bt);
        reinterpret_cast<float4 *>(om)[row * (kTsC / 4) + i * 32 + lane] = o;
        dot += o.x * uu.x + o.y * uu.y + o.z * uu.z + o.w * uu.w;
    }
    dot = group_sum<32>(dot) + __ldg(c + n);
    if (lane == 0) {
        logit[row] = clamp ? ts_clamp(dot) : dot;
        mean[row] = mu;
        rstd[row] = rs;
    }
}

__device__ __forceinline__ void ts_acc(float4 &a, float4 b) { a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w; }

// grid (tiles, N): CTA (t, n) takes rows t * kTsRows .. of image n, warp w rows w, w + 8, ... of those.  Partial p =
// n * tiles + t at part + p * kTsPart: [g_gamma | g_beta | g_b_e | g_u | g_c].
__global__ void __launch_bounds__(256)
twostage_head_bwd(const float *__restrict__ g_om, const float *__restrict__ g_logit, const float *__restrict__ y,
                  const unsigned char *__restrict__ keep, const float *__restrict__ b_e, const float *__restrict__ gamma,
                  const float *__restrict__ beta, const float *__restrict__ u, const float *__restrict__ c,
                  const float *__restrict__ mean, const float *__restrict__ rstd, int S, int clamp,
                  float *__restrict__ g_y, float *__restrict__ part)
{
    __shared__ float4 sp[4][8][kTsC / 4];
    __shared__ float sc[8];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int n = blockIdx.y;
    const long long base = (long long)n * S;
    const int r0 = blockIdx.x * kTsRows, r1 = min(S, r0 + kTsRows);
    float4 g[kTsV], bt[kTsV], uu[kTsV], ag[kTsV], ab[kTsV], ae[kTsV], au[kTsV];
    const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int i = 0; i < kTsV; ++i) {
        g[i] = __ldg(reinterpret_cast<const float4 *>(gamma) + i * 32 + lane);
        bt[i] = __ldg(reinterpret_cast<const float4 *>(beta) + i * 32 + lane);
        uu[i] = __ldg(reinterpret_cast<const float4 *>(u) + n * (kTsC / 4) + i * 32 + lane);
        ag[i] = ab[i] = ae[i] = au[i] = z4;
    }
    const float cn = __ldg(c + n);
    float ac = 0.f;
    for (int r = r0 + warp; r < r1; r += 8) {
        const long long row = base + r;
        const float mu = __ldg(mean + row), rs = __ldg(rstd + row);
        float4 v[kTsV], xh[kTsV], o[kTsV], d[kTsV], dz[kTsV];
        ts_load_row(y, keep, b_e, row, lane, v);
        float dot = 0.f;
#pragma unroll
        for (int i = 0; i < kTsV; ++i) {
            xh[i] = make_float4((v[i].x - mu) * rs, (v[i].y - mu) * rs, (v[i].z - mu) * rs, (v[i].w - mu) * rs);
            o[i] = ln_affine(v[i], mu, rs, g[i], bt[i]);                         // om, exactly as the forward wrote it
            dot += o[i].x * uu[i].x + o[i].y * uu[i].y + o[i].z * uu[i].z + o[i].w * uu[i].w;
        }
        dot = group_sum<32>(dot) + cn;                                           // the logit before the clamp
        float gl = __ldg(g_logit + row);
        if (clamp && !(dot >= -kTsClamp && dot <= kTsClamp)) gl = 0.f;           // torch.clamp's backward
        ac += gl;
#pragma unroll
        for (int i = 0; i < kTsV; ++i) {
            const float4 gm = __ldg(reinterpret_cast<const float4 *>(g_om) + row * (kTsC / 4) + i * 32 + lane);
            d[i] = make_float4(gm.x + gl * uu[i].x, gm.y + gl * uu[i].y, gm.z + gl * uu[i].z, gm.w + gl * uu[i].w);
            ts_acc(ab[i], d[i]);
            ts_acc(ag[i], make_float4(d[i].x * xh[i].x, d[i].y * xh[i].y, d[i].z * xh[i].z, d[i].w * xh[i].w));
            ts_acc(au[i], make_float4(gl * o[i].x, gl * o[i].y, gl * o[i].z, gl * o[i].w));
        }
        ln_row_bwd<kTsV>(d, xh, g, rs, dz);
        const bool kept = keep[row] != 0;
#pragma unroll
        for (int i = 0; i < kTsV; ++i) {
            reinterpret_cast<float4 *>(g_y)[row * (kTsC / 4) + i * 32 + lane] = kept ? dz[i] : z4;
            if (!kept) ts_acc(ae[i], dz[i]);
        }
    }
#pragma unroll
    for (int i = 0; i < kTsV; ++i) {
        sp[0][warp][i * 32 + lane] = ag[i];
        sp[1][warp][i * 32 + lane] = ab[i];
        sp[2][warp][i * 32 + lane] = ae[i];
        sp[3][warp][i * 32 + lane] = au[i];
    }
    if (lane == 0) sc[warp] = ac;
    __syncthreads();
    float *out = part + ((long long)n * gridDim.x + blockIdx.x) * kTsPart;
    {                                           // 256 threads: thread t sums float4 column t % 64 of quantity t / 64
        const int q = threadIdx.x >> 6, col = threadIdx.x & 63;
        float4 s = sp[q][0][col];
#pragma unroll
        for (int w = 1; w < 8; ++w) ts_acc(s, sp[q][w][col]);
        reinterpret_cast<float4 *>(out)[q * (kTsC / 4) + col] = s;
    }
    if (threadIdx.x == 0) {
        float s = sc[0];
#pragma unroll
        for (int w = 1; w < 8; ++w) s += sc[w];
        reinterpret_cast<float4 *>(out)[kTsC] = make_float4(s, 0.f, 0.f, 0.f);
    }
}

// block (32, 32): x = column lane, y = partial lane.  Blocks 0 .. 23 sum columns 0 .. 767 (g_gamma, g_beta, g_b_e) over
// all N * tiles partials; block 24 + n * 9 + j sums columns 768 + 32 j .. (g_u[n], then g_c[n] at 1024) over image n's
// partials.  Each (column, partial lane) sums partials y, y + 32, ... in order, then the 32 lanes in order.
__global__ void __launch_bounds__(1024)
twostage_head_reduce(const float *__restrict__ part, int N, int tiles, float *__restrict__ g_gamma, float *__restrict__ g_beta,
                     float *__restrict__ g_be, float *__restrict__ g_u, float *__restrict__ g_c)
{
    __shared__ float s[32][33];
    const int lx = threadIdx.x, ly = threadIdx.y;
    int col, p0, p1, n = 0;
    if (blockIdx.x < 24) {
        col = blockIdx.x * 32 + lx; p0 = 0; p1 = N * tiles;
    } else {
        const int j = blockIdx.x - 24;
        n = j / 9;
        col = 3 * kTsC + (j - n * 9) * 32 + lx; p0 = n * tiles; p1 = p0 + tiles;
    }
    const bool live = col <= 4 * kTsC;
    float acc = 0.f;
    if (live)
        for (int p = p0 + ly; p < p1; p += 32) acc += __ldg(part + (long long)p * kTsPart + col);
    s[ly][lx] = acc;
    __syncthreads();
    if (ly != 0 || !live) return;
    for (int k = 1; k < 32; ++k) acc += s[k][lx];
    if (col < kTsC) g_gamma[col] = acc;
    else if (col < 2 * kTsC) g_beta[col - kTsC] = acc;
    else if (col < 3 * kTsC) g_be[col - 2 * kTsC] = acc;
    else if (col < 4 * kTsC) g_u[n * kTsC + col - 3 * kTsC] = acc;
    else g_c[n] = acc;
}

// torch's fp32 sigmoid: 1 / (1 + exp(-x)), IEEE division, accurate expf.
__device__ __forceinline__ float ts_sigmoid(float x) { return 1.f / (1.f + expf(-x)); }

// The order key of a logit: torch.sort(descending=True, stable=True) order.  Every NaN ranks first (as torch's sorts
// and topk rank NaN above +inf) and -0 ties with +0.
__device__ __forceinline__ unsigned long long ts_key(float v, unsigned row) {
    if (v != v) v = __int_as_float(0x7fffffff);
    if (v == 0.f) v = 0.f;
    return dp_key(v, row);
}

// grid = N + add_ctas.  CTA n < N selects image n's top k; the others write coord = box + proposals for all rows.
// sort_ws: [N, sort_cap] u64 when the padded count exceeds kTsSmemSort (sort_cap = 0 otherwise).
__global__ void __launch_bounds__(kTsThreads, 1)
twostage_select_fwd(const float *__restrict__ logit, const float *__restrict__ box, const float *__restrict__ prop, int N,
                    int S, int k, long long sort_cap, unsigned long long *__restrict__ sort_ws, float *__restrict__ coord,
                    float *__restrict__ ref, long long *__restrict__ topk_index)
{
    __shared__ unsigned s_hist[256];
    __shared__ unsigned long long s_sort[kTsSmemSort];
    __shared__ int s_digit;
    __shared__ unsigned s_rem, s_bucket, s_n;
    const int tid = threadIdx.x;
    const float4 *bx = reinterpret_cast<const float4 *>(box), *pp = reinterpret_cast<const float4 *>(prop);
    if ((int)blockIdx.x >= N) {
        const long long total = (long long)N * S, stride = (long long)(gridDim.x - N) * kTsThreads;
        for (long long i = (long long)(blockIdx.x - N) * kTsThreads + tid; i < total; i += stride) {
            const float4 a = __ldg(bx + i), b = __ldg(pp + i);
            reinterpret_cast<float4 *>(coord)[i] = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
        }
        return;
    }
    const int n = blockIdx.x;
    const float *lg = logit + (long long)n * S;
    auto key_of = [&](unsigned s) { return ts_key(__ldg(lg + s), s); };
    const unsigned long long thr = block_radix_threshold<kTsThreads>((unsigned)S, (unsigned)k, key_of, s_hist, &s_digit,
                                                                     &s_rem, &s_bucket);
    unsigned P = 1;
    while (P < (unsigned)k) P <<= 1;
    unsigned long long *buf = P <= (unsigned)kTsSmemSort ? s_sort : sort_ws + (long long)n * sort_cap;
    if (tid == 0) s_n = 0;
    __syncthreads();
    for (unsigned s = tid; s < (unsigned)S; s += kTsThreads) {
        const unsigned long long key = key_of(s);
        if (key <= thr) buf[atomicAdd(&s_n, 1u)] = key;
    }
    for (unsigned i = k + tid; i < P; i += kTsThreads) buf[i] = ~0ull;
    __syncthreads();
    block_bitonic_sort<kTsThreads>(buf, P);
    for (int j = tid; j < k; j += kTsThreads) {
        const unsigned s = (unsigned)(buf[j] & 0xffffffffull);
        const long long r = (long long)n * S + s;
        const float4 a = __ldg(bx + r), b = __ldg(pp + r);
        reinterpret_cast<float4 *>(ref)[(long long)n * k + j] =
            make_float4(ts_sigmoid(a.x + b.x), ts_sigmoid(a.y + b.y), ts_sigmoid(a.z + b.z), ts_sigmoid(a.w + b.w));
        topk_index[(long long)n * k + j] = s;
    }
}

// One thread per (image, rank, coordinate): g_coord[n, idx, c] += g_ref * (1 - s) * s.  The k indices of an image are
// distinct, so no two threads write one element.
__global__ void __launch_bounds__(256)
twostage_select_bwd(const float *__restrict__ g_ref, const float *__restrict__ ref, const long long *__restrict__ topk_index,
                    int S, int k, long long total, float *__restrict__ g_coord)
{
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= total) return;
    const long long nk = t >> 2;
    const int cc = (int)(t & 3);
    const long long n = nk / k;
    const float s = __ldg(ref + t);
    g_coord[(n * S + __ldg(topk_index + nk)) * 4 + cc] += __ldg(g_ref + t) * (1.f - s) * s;
}

}  // namespace msda
