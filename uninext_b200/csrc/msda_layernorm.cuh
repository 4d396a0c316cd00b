// msda_layernorm.cuh -- LayerNorm over one row of C = 128*V channels held by a warp, V float4 per lane (lane's slice i:
// channels 4 * (i * 32 + lane) .. +3).  The row code of add + LayerNorm (msda_module.cuh) and of the two-stage head
// (msda_twostage.cuh).  Device functions only.
#pragma once

#include "msda_common.cuh"

namespace msda {

// Sum over each group of G lanes (G a power of two <= 32), the result in every lane of the group.
template <int G>
__device__ __forceinline__ float group_sum(float v) {
#pragma unroll
    for (int d = G / 2; d >= 1; d >>= 1) v += __shfl_xor_sync(kFullMask, v, d, G);
    return v;
}

// mean and 1 / sqrt(var + eps) of the row; s is the lane's sum of its v[i].x + v[i].y + v[i].z + v[i].w, in i order.
template <int V>
__device__ __forceinline__ void ln_row_stats(const float4 (&v)[V], float s, float eps, float &mu, float &rs) {
    constexpr int C = 128 * V;
    mu = group_sum<32>(s) * (1.f / C);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < V; ++i) {
        const float dx = v[i].x - mu, dy = v[i].y - mu, dz = v[i].z - mu, dw = v[i].w - mu;
        q += dx * dx + dy * dy + dz * dz + dw * dw;
    }
    rs = rsqrtf(group_sum<32>(q) * (1.f / C) + eps);
}

// (v - mean) * rstd * gamma + beta for one float4 slice.
__device__ __forceinline__ float4 ln_affine(float4 v, float mu, float rs, float4 g, float4 bt) {
    return make_float4((v.x - mu) * rs * g.x + bt.x, (v.y - mu) * rs * g.y + bt.y, (v.z - mu) * rs * g.z + bt.z,
                       (v.w - mu) * rs * g.w + bt.w);
}

// dz = rstd * (dy*gamma - mean(dy*gamma) - xhat * mean(dy*gamma*xhat)) of the row; d holds dy on entry, dy*gamma on return.
template <int V>
__device__ __forceinline__ void ln_row_bwd(float4 (&d)[V], const float4 (&xh)[V], const float4 (&g)[V], float rs,
                                           float4 (&dz)[V]) {
    constexpr int C = 128 * V;
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < V; ++i) {
        d[i].x *= g[i].x; d[i].y *= g[i].y; d[i].z *= g[i].z; d[i].w *= g[i].w;
        s1 += d[i].x + d[i].y + d[i].z + d[i].w;
        s2 += d[i].x * xh[i].x + d[i].y * xh[i].y + d[i].z * xh[i].z + d[i].w * xh[i].w;
    }
    s1 = group_sum<32>(s1) * (1.f / C);
    s2 = group_sum<32>(s2) * (1.f / C);
#pragma unroll
    for (int i = 0; i < V; ++i)
        dz[i] = make_float4(rs * (d[i].x - s1 - xh[i].x * s2), rs * (d[i].y - s1 - xh[i].y * s2),
                            rs * (d[i].z - s1 - xh[i].z * s2), rs * (d[i].w - s1 - xh[i].w * s2));
}

}  // namespace msda
