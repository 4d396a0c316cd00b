// msda_cabi_twostage.cu -- C ABI of the two-stage query selection (msda_twostage.cuh, include/msda_twostage.h).
#include "../../include/msda_b200.h"
#include "../../include/msda_twostage.h"
#include "msda_host.cuh"
#include "msda_twostage.cuh"

using namespace msda_host;

namespace {

int sizes_check(int N, int S, int C) {
    return (N < 1 || N > 65535 || S < 1 || C != msda::kTsC) ? MSDA_E_BADARG : 0;
}

int head_tiles(int S) { return (S + msda::kTsRows - 1) / msda::kTsRows; }

size_t head_workspace(int N, int S) { return align256((size_t)N * head_tiles(S) * msda::kTsPart * sizeof(float)); }

// [N, sort_cap] u64 sort slots when the padded count exceeds the on-chip buffer (sort_cap = 0 otherwise).
long long select_sort_cap(int k) {
    long long p = 1;
    while (p < k) p <<= 1;
    return p > msda::kTsSmemSort ? p : 0;
}

}  // namespace

extern "C" {

int msda_twostage_head_forward_f32(const float *y, const uint8_t *keep, const float *b_e, const float *gamma,
                                   const float *beta, const float *u, const float *c, int N, int S, int C, float eps,
                                   int clamp, float *om, float *logit, float *mean, float *rstd, void *stream) {
    if (!keep || !c || !logit || !mean || !rstd || !all_aligned16({y, b_e, gamma, beta, u, om})) return MSDA_E_BADARG;
    if (const int e = sizes_check(N, S, C)) return e;
    const long long rows = (long long)N * S;
    return (int)launch(msda::twostage_head_fwd, (unsigned)((rows + 7) / 8), 256, 0, static_cast<cudaStream_t>(stream), y,
                       keep, b_e, gamma, beta, u, c, rows, S, eps, clamp, om, logit, mean, rstd);
}

int msda_twostage_head_workspace(int N, int S, int C, int64_t *bytes) {
    if (!bytes) return MSDA_E_BADARG;
    if (const int e = sizes_check(N, S, C)) return e;
    *bytes = (int64_t)head_workspace(N, S);
    return 0;
}

int msda_twostage_head_backward_f32(const float *grad_om, const float *grad_logit, const float *y, const uint8_t *keep,
                                    const float *b_e, const float *gamma, const float *beta, const float *u,
                                    const float *c, const float *mean, const float *rstd, int N, int S, int C, int clamp,
                                    float *grad_y, float *grad_b_e, float *grad_gamma, float *grad_beta, float *grad_u,
                                    float *grad_c, void *workspace, int64_t workspace_bytes, void *stream) {
    if (!grad_logit || !keep || !c || !mean || !rstd || !grad_b_e || !grad_gamma || !grad_beta || !grad_u || !grad_c ||
        !all_aligned16({grad_om, y, b_e, gamma, beta, u, grad_y, workspace}))
        return MSDA_E_BADARG;
    if (const int e = sizes_check(N, S, C)) return e;
    if (workspace_bytes < (int64_t)head_workspace(N, S)) return MSDA_E_BADARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    float *part = static_cast<float *>(workspace);
    const int tiles = head_tiles(S);
    const cudaError_t e = launch(msda::twostage_head_bwd, dim3((unsigned)tiles, (unsigned)N), 256, 0, st, grad_om,
                                 grad_logit, y, keep, b_e, gamma, beta, u, c, mean, rstd, S, clamp, grad_y, part);
    if (e != cudaSuccess) return (int)e;
    return (int)launch(msda::twostage_head_reduce, (unsigned)(24 + 9 * N), dim3(32, 32), 0, st, part, N, tiles,
                       grad_gamma, grad_beta, grad_b_e, grad_u, grad_c);
}

int msda_twostage_select_workspace(int N, int S, int k, int64_t *bytes) {
    if (!bytes) return MSDA_E_BADARG;
    if (const int e = sizes_check(N, S, msda::kTsC)) return e;
    if (k < 1 || k > S) return MSDA_E_BADARG;
    *bytes = (int64_t)align256((size_t)N * select_sort_cap(k) * sizeof(unsigned long long));
    return 0;
}

int msda_twostage_select_forward_f32(const float *logit, const float *box, const float *proposals, int N, int S, int k,
                                     float *coord_unact, float *reference_points, int64_t *topk_index, void *workspace,
                                     int64_t workspace_bytes, void *stream) {
    if (!logit || !topk_index || !all_aligned16({box, proposals, coord_unact, reference_points})) return MSDA_E_BADARG;
    if (const int e = sizes_check(N, S, msda::kTsC)) return e;
    if (k < 1 || k > S) return MSDA_E_BADARG;
    const long long cap = select_sort_cap(k);
    if (cap > 0 && (!workspace || !aligned16(workspace) ||
                    workspace_bytes < (int64_t)((size_t)N * cap * sizeof(unsigned long long))))
        return MSDA_E_BADARG;
    // Beside the N selecting CTAs, enough CTAs to write coord_unact (N * S float4) at 4 per thread, at most 4 per SM.
    const int add = capped_grid((long long)N * S, 4ll * msda::kTsThreads, 4);
    return (int)launch(msda::twostage_select_fwd, (unsigned)(N + add), msda::kTsThreads, 0,
                       static_cast<cudaStream_t>(stream), logit, box, proposals, N, S, k, cap,
                       static_cast<unsigned long long *>(workspace), coord_unact, reference_points,
                       reinterpret_cast<long long *>(topk_index));
}

int msda_twostage_select_backward_f32(const float *grad_ref, const float *reference_points, const int64_t *topk_index,
                                      int N, int S, int k, float *grad_coord, void *stream) {
    if (!grad_ref || !reference_points || !topk_index || !grad_coord) return MSDA_E_BADARG;
    if (const int e = sizes_check(N, S, msda::kTsC)) return e;
    if (k < 1 || k > S) return MSDA_E_BADARG;
    const long long total = (long long)N * k * 4;
    return (int)launch(msda::twostage_select_bwd, (unsigned)((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream),
                       grad_ref, reference_points, reinterpret_cast<const long long *>(topk_index), S, k, total, grad_coord);
}

}  // extern "C"
