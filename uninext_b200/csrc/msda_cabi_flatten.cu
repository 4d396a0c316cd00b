// msda_cabi_flatten.cu -- C ABI of the encoder's input preparation (msda_flatten.cuh, include/msda_flatten.h).
#include <climits>

#include "../../include/msda_b200.h"
#include "../../include/msda_flatten.h"
#include "msda_flatten.cuh"
#include "msda_host.cuh"

using namespace msda_host;

namespace {

// The level table from the host arrays, or MSDA_E_BADARG for sizes out of range.
int make_table(const int *H, const int *W, int L, int N, int C, msda::FlattenTable &t) {
    if (!H || !W || L < 1 || L > msda::kMaxLevels || N < 1 || N > 65535 || C < 4 || C > 1024 || C % 4) return MSDA_E_BADARG;
    t = msda::FlattenTable{};
    t.L = L;
    t.C = C;
    t.ctiles = (C + msda::kFlTile - 1) / msda::kFlTile;
    long long s = 0, tiles = 0, ptiles = 0;
    for (int l = 0; l < L; ++l) {
        if (H[l] < 1 || W[l] < 1) return MSDA_E_BADARG;
        const long long hw = (long long)H[l] * W[l], pt = (hw + msda::kFlTile - 1) / msda::kFlTile;
        t.hw[l] = hw;
        t.start[l] = s;
        t.tile0[l] = (int)tiles;
        t.ptile0[l] = (int)ptiles;
        s += hw;
        ptiles += pt;
        tiles += pt * t.ctiles;
        if (tiles > INT_MAX) return MSDA_E_BADARG;             // tiles of one image are the grid's x extent
    }
    t.S = s;
    t.tile0[L] = (int)tiles;
    t.ptile0[L] = (int)ptiles;
    return 0;
}

size_t workspace_bytes(const msda::FlattenTable &t, int N) {
    return align256((size_t)N * t.ptile0[t.L] * t.C * sizeof(float));
}

template <class P>
bool all_set(const P *const *ptrs, int L) {
    if (!ptrs) return false;
    for (int l = 0; l < L; ++l)
        if (!ptrs[l]) return false;
    return true;
}

}  // namespace

extern "C" {

int msda_flatten_levels_forward_f32(const float *const *src, const float *const *pos, const uint8_t *const *mask,
                                    const int *H, const int *W, int L, int N, int C, const float *level_embed,
                                    float *src_flat, float *pos_flat, uint8_t *mask_flat, void *stream) {
    msda::FlattenFwdArgs a{};
    if (const int e = make_table(H, W, L, N, C, a.t)) return e;
    if (!all_set(src, L) || !all_set(pos, L) || !all_set(mask, L) || !mask_flat ||
        !all_aligned16({level_embed, src_flat, pos_flat}))
        return MSDA_E_BADARG;
    for (int l = 0; l < L; ++l) {
        a.src[l] = src[l];
        a.pos[l] = pos[l];
        a.mask[l] = mask[l];
    }
    a.level_embed = level_embed;
    a.src_flat = src_flat;
    a.pos_flat = pos_flat;
    a.mask_flat = mask_flat;
    return (int)launch(msda::flatten_levels_fwd, dim3((unsigned)a.t.tile0[L], (unsigned)N), msda::kFlThreads, 0,
                       static_cast<cudaStream_t>(stream), a);
}

int msda_flatten_levels_workspace(const int *H, const int *W, int L, int N, int C, int64_t *bytes) {
    msda::FlattenTable t;
    if (!bytes) return MSDA_E_BADARG;
    if (const int e = make_table(H, W, L, N, C, t)) return e;
    *bytes = (int64_t)workspace_bytes(t, N);
    return 0;
}

int msda_flatten_levels_backward_f32(const float *grad_src_flat, const float *grad_pos_flat, const int *H, const int *W,
                                     int L, int N, int C, float *const *grad_src, float *const *grad_pos,
                                     float *grad_level_embed, void *workspace, int64_t workspace_bytes_, void *stream) {
    msda::FlattenBwdArgs a{};
    if (const int e = make_table(H, W, L, N, C, a.t)) return e;
    if ((grad_src && (!all_set(grad_src, L) || !all_aligned16({grad_src_flat}))) ||
        (grad_pos && !all_set(grad_pos, L)) ||
        ((grad_pos || grad_level_embed) && !all_aligned16({grad_pos_flat})))
        return MSDA_E_BADARG;
    if (grad_level_embed && (!workspace || workspace_bytes_ < (int64_t)workspace_bytes(a.t, N))) return MSDA_E_BADARG;
    if (!grad_src && !grad_pos && !grad_level_embed) return 0;
    for (int l = 0; l < L; ++l) {
        a.grad_src[l] = grad_src ? grad_src[l] : nullptr;
        a.grad_pos[l] = grad_pos ? grad_pos[l] : nullptr;
    }
    a.grad_src_flat = grad_src ? grad_src_flat : nullptr;
    a.grad_pos_flat = (grad_pos || grad_level_embed) ? grad_pos_flat : nullptr;
    a.part = grad_level_embed ? static_cast<float *>(workspace) : nullptr;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const cudaError_t e = launch(msda::flatten_levels_bwd, dim3((unsigned)a.t.tile0[L], (unsigned)N), msda::kFlThreads, 0,
                                 st, a);
    if (e != cudaSuccess || !grad_level_embed) return (int)e;
    return (int)launch(msda::flatten_levels_reduce, dim3((unsigned)L, (unsigned)a.t.ctiles), dim3(32, 32), 0, st, a.part,
                       a.t, N, grad_level_embed);
}

}  // extern "C"
