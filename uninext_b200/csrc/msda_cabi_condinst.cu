// msda_cabi_condinst.cu -- C ABI of the CondInst dynamic mask head and aligned_bilinear (msda_condinst.cuh).
#include "../../include/msda_b200.h"
#include "msda_condinst.cuh"
#include "msda_host.cuh"

using namespace msda_host;

extern "C" {

int msda_condinst_forward_f32(const float *feats, const float *params, const float *refs, const int32_t *inst_start, int N,
                              int H, int W, int I, int max_inst, int stride, int rel_coord, float *logits, void *stream) {
    if (!feats || !params || !refs || !inst_start || !logits || N <= 0 || H <= 0 || W <= 0 || I < 0 || stride <= 0 ||
        max_inst < 0 || (long long)H * W >= (1ll << 30))
        return MSDA_E_BADARG;
    if (I == 0 || max_inst == 0) return 0;
    const int HW = H * W, tile = msda::kCiFwdThreads * msda::kCiFwdPpt;
    const dim3 grid((unsigned)((HW + tile - 1) / tile), (unsigned)((max_inst + msda::kCiChunk - 1) / msda::kCiChunk), (unsigned)N);
    // 16-byte accesses need every row of feats / logits 16-byte aligned: HW % 4 == 0 and aligned base pointers (a view with a
    // storage offset is not); anything else takes the scalar path
    const int vec = HW % 4 == 0 && aligned16(feats) && aligned16(logits);
    return (int)launch(msda::condinst_fwd, grid, msda::kCiFwdThreads, 0, static_cast<cudaStream_t>(stream), feats, params,
                       refs, inst_start, HW, W, stride, rel_coord, vec, logits);
}

int msda_condinst_backward_f32(const float *grad_logits, const float *feats, const float *params, const float *refs,
                               const int32_t *inst_start, int N, int H, int W, int I, int max_inst, int stride, int rel_coord,
                               float *grad_feats, float *grad_params, float *grad_refs, void *stream) {
    if (!grad_logits || !feats || !params || !refs || !inst_start || !grad_feats || !grad_params || !grad_refs || N <= 0 ||
        H <= 0 || W <= 0 || I < 0 || max_inst < 0 || stride <= 0 || (long long)H * W >= (1ll << 30))
        return MSDA_E_BADARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int HW = H * W, tile = msda::kCiThreads * msda::kCiBwdPpt;
    cudaError_t e = cudaMemsetAsync(grad_feats, 0, sizeof(float) * (size_t)N * msda::kCiFeat * HW, st);
    if (e == cudaSuccess && I > 0) e = cudaMemsetAsync(grad_params, 0, sizeof(float) * (size_t)I * msda::kCiParams, st);
    if (e == cudaSuccess && I > 0) e = cudaMemsetAsync(grad_refs, 0, sizeof(float) * (size_t)I * 2, st);
    if (e != cudaSuccess) return (int)e;
    if (I == 0 || max_inst == 0) return 0;
    const dim3 grid((unsigned)((HW + tile - 1) / tile), (unsigned)((max_inst + msda::kCiChunk - 1) / msda::kCiChunk), (unsigned)N);
    return (int)launch(msda::condinst_bwd, grid, msda::kCiThreads, 0, st, grad_logits, feats, params, refs, inst_start, HW, W,
                       stride, rel_coord, grad_feats, grad_params, grad_refs);
}

int msda_aligned_bilinear_forward_f32(const float *in, int64_t planes, int h, int w, int factor, float *out, void *stream) {
    if (!in || !out || planes < 0 || planes >= (1ll << 31) || h <= 0 || w <= 0 || factor < 1 ||
        (long long)h * factor * w * factor >= (1ll << 31))
        return MSDA_E_BADARG;
    if (planes == 0) return 0;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const dim3 grid((unsigned)planes, (unsigned)((h * factor + msda::kAbRows - 1) / msda::kAbRows));
    const bool vec = (w * factor) % 4 == 0 && aligned16(out);
    if (factor == 2 && vec) return (int)launch(msda::aligned_bilinear2_fwd, grid, 256, 0, st, in, h, w, out);
    if (vec) return (int)launch(msda::aligned_bilinear_fwd<0, 4>, grid, 256, 0, st, in, h, w, factor, out);
    return (int)launch(msda::aligned_bilinear_fwd<0, 1>, grid, 256, 0, st, in, h, w, factor, out);
}

int msda_aligned_bilinear_backward_f32(const float *grad_out, int64_t planes, int h, int w, int factor, float *grad_in,
                                       void *stream) {
    if (!grad_out || !grad_in || planes < 0 || planes >= (1ll << 31) || h <= 0 || w <= 0 || factor < 1 ||
        (long long)h * factor * w * factor >= (1ll << 31))
        return MSDA_E_BADARG;
    if (planes == 0) return 0;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const dim3 grid((unsigned)planes, (unsigned)((h + msda::kAbRows - 1) / msda::kAbRows));
    const bool vec = w % 2 == 0 && aligned16(grad_out) && aligned8(grad_in);
    if (factor == 2 && vec) return (int)launch(msda::aligned_bilinear2_bwd, grid, 256, 0, st, grad_out, h, w, grad_in);
    return (int)launch(msda::aligned_bilinear_bwd<0>, grid, 256, 0, st, grad_out, h, w, factor, grad_in);
}

}  // extern "C"
