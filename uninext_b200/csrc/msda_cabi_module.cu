// msda_cabi_module.cu -- C ABI of the kernels around the op (msda_module.cuh): the sampling prologue, the bias-gradient
// column sums, add + LayerNorm, and the geometry feeding the op (valid counts, encoder reference points and proposals,
// sine position embeddings).
#include "../../include/msda_b200.h"
#include "msda_host.cuh"
#include "msda_module.cuh"

using namespace msda_host;

namespace {
int group_width(int LP) { return LP <= 4 ? 4 : LP <= 8 ? 8 : LP <= 16 ? 16 : 32; }

// Column sums: at least 16 rows per CTA, at most ctas_per_sm CTAs per SM.
int colsum_rows_per_cta(long long rows, int ctas_per_sm) {
    const long long ctas = (long long)num_sms() * ctas_per_sm;
    const int r = (int)((rows + ctas - 1) / ctas);
    return r < 16 ? 16 : r;
}
}  // namespace

extern "C" {

int msda_prologue_forward_f32(const float *proj, const float *ref, const int64_t *spatial_shapes, int64_t R, int M, int L,
                              int P, int refdim, float *loc, float *attn, void *stream) {
    if (!proj || !ref || !spatial_shapes || !loc || !attn || R <= 0 || M <= 0 || L <= 0 || P <= 0 || L * P > 32 ||
        (refdim != 2 && refdim != 4) || (long long)R * M * 32 >= (1ll << 40) || !aligned8(loc))      // float2 stores
        return MSDA_E_BADARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long np = (long long)R * M;
    const auto go = [&](auto kernel, int G) {
        return (int)launch(kernel, (unsigned)((np * G + 255) / 256), 256, 0, st, proj, ref, spatial_shapes, np, M, L, P,
                           refdim, loc, attn);
    };
    switch (group_width(L * P)) {
        case 4: return go(msda::msda_prologue_fwd<4>, 4);
        case 8: return go(msda::msda_prologue_fwd<8>, 8);
        case 16: return go(msda::msda_prologue_fwd<16>, 16);
        default: return go(msda::msda_prologue_fwd<32>, 32);
    }
}

int msda_prologue_backward_f32(const float *grad_loc, const float *grad_attn, const float *attn, const float *ref,
                               const int64_t *spatial_shapes, int64_t R, int M, int L, int P, int refdim,
                               float *grad_proj, void *stream) {
    if (!grad_loc || !grad_attn || !attn || !ref || !spatial_shapes || !grad_proj || R <= 0 || M <= 0 || L <= 0 || P <= 0 ||
        L * P > 32 || (refdim != 2 && refdim != 4) || !aligned8(grad_loc))                             // float2 loads
        return MSDA_E_BADARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long np = (long long)R * M;
    const auto go = [&](auto kernel, int G) {
        return (int)launch(kernel, (unsigned)((np * G + 255) / 256), 256, 0, st, grad_loc, grad_attn, attn, ref,
                           spatial_shapes, np, M, L, P, refdim, grad_proj);
    };
    switch (group_width(L * P)) {
        case 4: return go(msda::msda_prologue_bwd<4>, 4);
        case 8: return go(msda::msda_prologue_bwd<8>, 8);
        case 16: return go(msda::msda_prologue_bwd<16>, 16);
        default: return go(msda::msda_prologue_bwd<32>, 32);
    }
}

int msda_colsum_f32(const float *x, int64_t rows, int cols, float *out, void *stream) {
    if (!x || !out || rows <= 0 || cols <= 0 || cols % 4 != 0 || !aligned16(x) || !aligned16(out)) return MSDA_E_BADARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaError_t err = cudaMemsetAsync(out, 0, sizeof(float) * (size_t)cols, st);
    if (err != cudaSuccess) return (int)err;
    const int rows_per_cta = colsum_rows_per_cta(rows, 4);
    return (int)launch(msda::msda_colsum, (unsigned)((rows + rows_per_cta - 1) / rows_per_cta), 256, 0, st, x, rows, cols,
                       rows_per_cta, out);
}

int msda_relu_backward_colsum_f32(const float *g, const float *y, int64_t rows, int cols, float *g2, float *colsum, void *stream) {
    if (!g || !y || !g2 || !colsum || rows <= 0 || cols <= 0 || cols % 4 != 0 || !aligned16(g) || !aligned16(y) || !aligned16(g2) ||
        !aligned16(colsum))
        return MSDA_E_BADARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaError_t err = cudaMemsetAsync(colsum, 0, sizeof(float) * (size_t)cols, st);
    if (err != cudaSuccess) return (int)err;
    const int rows_per_cta = colsum_rows_per_cta(rows, 8);
    return (int)launch(msda::msda_relu_bwd_colsum, (unsigned)((rows + rows_per_cta - 1) / rows_per_cta), 256, 0, st, g, y,
                       rows, cols, rows_per_cta, g2, colsum);
}

int msda_add_layernorm_forward_f32(const float *a, const float *b, const float *gamma, const float *beta, int64_t rows,
                                   int cols, float eps, float *z, float *y, float *mean, float *rstd, void *stream) {
    if (!a || !gamma || !beta || !y || !mean || !rstd || rows <= 0 || (b != nullptr && z == nullptr)) return MSDA_E_BADARG;
    if (cols != 128 && cols != 256 && cols != 384 && cols != 512) return MSDA_E_BADARG;
    if (!aligned16(a) || !aligned16(gamma) || !aligned16(beta) || !aligned16(y) || (b && !aligned16(b)) || (z && !aligned16(z)))
        return MSDA_E_BADARG;                                                                        // float4 accesses
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const unsigned grid = (unsigned)((rows + 7) / 8);
    const auto go = [&](auto kernel) {
        return (int)launch(kernel, grid, 256, 0, st, a, b, gamma, beta, rows, eps, z, y, mean, rstd);
    };
    switch (cols / 128) {
        case 1: return go(msda::msda_add_layernorm_fwd<1>);
        case 2: return go(msda::msda_add_layernorm_fwd<2>);
        case 3: return go(msda::msda_add_layernorm_fwd<3>);
        default: return go(msda::msda_add_layernorm_fwd<4>);
    }
}

int msda_layernorm_backward_f32(const float *dy, const float *z, const float *gamma, const float *mean, const float *rstd,
                                int64_t rows, int cols, float *dz, float *dgamma, float *dbeta, void *stream) {
    if (!dy || !z || !gamma || !mean || !rstd || !dz || !dgamma || !dbeta || rows <= 0) return MSDA_E_BADARG;
    if (cols != 128 && cols != 256 && cols != 384 && cols != 512) return MSDA_E_BADARG;
    if (!aligned16(dy) || !aligned16(z) || !aligned16(gamma) || !aligned16(dz) || !aligned16(dgamma) || !aligned16(dbeta))
        return MSDA_E_BADARG;                                                                        // float4 accesses, 16-byte reds
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaError_t err = cudaMemsetAsync(dgamma, 0, sizeof(float) * (size_t)cols, st);
    if (err == cudaSuccess) err = cudaMemsetAsync(dbeta, 0, sizeof(float) * (size_t)cols, st);
    if (err != cudaSuccess) return (int)err;
    const long long ctas = (long long)num_sms() * 4;
    int rows_per_cta = (int)((rows + ctas - 1) / ctas);
    rows_per_cta = ((rows_per_cta + 7) / 8) * 8;
    const unsigned grid = (unsigned)((rows + rows_per_cta - 1) / rows_per_cta);
    const auto go = [&](auto kernel) {
        return (int)launch(kernel, grid, 256, 0, st, dy, z, gamma, mean, rstd, rows, rows_per_cta, dz, dgamma, dbeta);
    };
    switch (cols / 128) {
        case 1: return go(msda::msda_layernorm_bwd<1>);
        case 2: return go(msda::msda_layernorm_bwd<2>);
        case 3: return go(msda::msda_layernorm_bwd<3>);
        default: return go(msda::msda_layernorm_bwd<4>);
    }
}

int msda_valid_counts(const uint8_t *mask, const int64_t *spatial_shapes, const int64_t *level_start_index, int N, int S, int L,
                      int32_t *counts, void *stream) {
    if (!mask || !spatial_shapes || !level_start_index || !counts || N <= 0 || S <= 0 || L <= 0) return MSDA_E_BADARG;
    const int warps = N * L;
    return (int)launch(msda::msda_valid_counts, (warps * 32 + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream), mask,
                       spatial_shapes, level_start_index, N, S, L, counts);
}

int msda_encoder_ref_points_f32(const float *valid_ratios, const int64_t *spatial_shapes, const int64_t *level_start_index, int N,
                                int S, int L, float *ref, void *stream) {
    if (!valid_ratios || !spatial_shapes || !level_start_index || !ref || N <= 0 || S <= 0 || L <= 0 || !aligned16(ref)) return MSDA_E_BADARG;
    const long long total = (long long)N * S;
    return (int)launch(msda::msda_encoder_ref_points, (unsigned)((total + 255) / 256), 256, 0,
                       static_cast<cudaStream_t>(stream), valid_ratios, spatial_shapes, level_start_index, N, S, L, ref);
}

int msda_encoder_proposals_f32(const uint8_t *mask, const int32_t *counts, const int64_t *spatial_shapes,
                               const int64_t *level_start_index, int N, int S, int L, float base_scale, float *proposals,
                               uint8_t *keep, void *stream) {
    if (!mask || !counts || !spatial_shapes || !level_start_index || !proposals || !keep || N <= 0 || S <= 0 || L <= 0 || L > 30 ||
        !aligned16(proposals))
        return MSDA_E_BADARG;
    const long long total = (long long)N * S;
    return (int)launch(msda::msda_encoder_proposals, (unsigned)((total + 255) / 256), 256, 0,
                       static_cast<cudaStream_t>(stream), mask, counts, spatial_shapes, level_start_index, N, S, L,
                       base_scale, proposals, keep);
}

int msda_sine_pos_embed_forward_f32(const float *pos, int64_t R, int n, int F, float temperature, int exchange_xy, float *out,
                                    void *stream) {
    if (!pos || !out || R <= 0 || n <= 0 || F <= 0) return MSDA_E_BADARG;
    const long long warps = (long long)R * n;
    return (int)launch(msda::msda_sine_pos_embed<false>, (unsigned)((warps * 32 + 255) / 256), 256, 0,
                       static_cast<cudaStream_t>(stream), pos, nullptr, R, n, F, temperature, exchange_xy, out);
}

int msda_sine_pos_embed_backward_f32(const float *pos, const float *grad_out, int64_t R, int n, int F, float temperature,
                                     int exchange_xy, float *grad_pos, void *stream) {
    if (!pos || !grad_out || !grad_pos || R <= 0 || n <= 0 || F <= 0) return MSDA_E_BADARG;
    const long long warps = (long long)R * n;
    return (int)launch(msda::msda_sine_pos_embed<true>, (unsigned)((warps * 32 + 255) / 256), 256, 0,
                       static_cast<cudaStream_t>(stream), pos, grad_out, R, n, F, temperature, exchange_xy, grad_pos);
}

}  // extern "C"
