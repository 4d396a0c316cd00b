// TEST / BENCH INFRASTRUCTURE ONLY -- exposes the REFERENCE's own CUDA kernels (compiled unmodified from where they
// lie under /root/reference, see oracle/build_refcuda.sh) through a C ABI, so that on the GPU box
//   * parity tests can compare the sm_90a kernels against the reference op itself on identical tensors, and
//   * bench tools can time the reference kernels (K1 forward, K2 backward) on the same GPU.
// Only the two templated launchers of ms_deform_im2col_cuda.cuh are used (cuh:923-954, cuh:956-1327); the ATen host
// wrapper ms_deform_attn_cuda.cu is not (it needs torch 1.x's Tensor::type()).  No reference source is copied here.
#include <cstdint>
#include "cuda/ms_deform_im2col_cuda.cuh"

extern "C" int refcuda_forward_f32(const float *value, const int64_t *shapes, const int64_t *lsi, const float *loc,
                                   const float *attn, int N, int S, int M, int D, int L, int Lq, int P, float *out,
                                   void *stream) {
    ms_deformable_im2col_cuda<float>(static_cast<cudaStream_t>(stream), value, shapes, lsi, loc, attn, N, S, M, D, L, Lq, P, out);
    return (int)cudaGetLastError();
}

extern "C" int refcuda_forward_f64(const double *value, const int64_t *shapes, const int64_t *lsi, const double *loc,
                                   const double *attn, int N, int S, int M, int D, int L, int Lq, int P, double *out,
                                   void *stream) {
    ms_deformable_im2col_cuda<double>(static_cast<cudaStream_t>(stream), value, shapes, lsi, loc, attn, N, S, M, D, L, Lq, P, out);
    return (int)cudaGetLastError();
}

// grad_value / grad_loc / grad_attn must be zero-filled by the caller (the reference wrapper uses at::zeros_like,
// ms_deform_attn_cuda.cu:121-123).
extern "C" int refcuda_backward_f32(const float *grad_out, const float *value, const int64_t *shapes, const int64_t *lsi,
                                    const float *loc, const float *attn, int N, int S, int M, int D, int L, int Lq,
                                    int P, float *grad_value, float *grad_loc, float *grad_attn, void *stream) {
    ms_deformable_col2im_cuda<float>(static_cast<cudaStream_t>(stream), grad_out, value, shapes, lsi, loc, attn, N, S, M,
                                     D, L, Lq, P, grad_value, grad_loc, grad_attn);
    return (int)cudaGetLastError();
}

extern "C" int refcuda_backward_f64(const double *grad_out, const double *value, const int64_t *shapes,
                                    const int64_t *lsi, const double *loc, const double *attn, int N, int S, int M,
                                    int D, int L, int Lq, int P, double *grad_value, double *grad_loc,
                                    double *grad_attn, void *stream) {
    ms_deformable_col2im_cuda<double>(static_cast<cudaStream_t>(stream), grad_out, value, shapes, lsi, loc, attn, N, S,
                                      M, D, L, Lq, P, grad_value, grad_loc, grad_attn);
    return (int)cudaGetLastError();
}
