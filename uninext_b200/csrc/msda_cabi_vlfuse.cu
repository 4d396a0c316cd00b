// msda_cabi_vlfuse.cu -- C ABI of the fused image-text attention of the early-fusion block: the F32 kernels
// (msda_vlfuse.cuh), the TF32 and bf16 tensor-core kernels (msda_vlfuse_tc.cuh), the workspace size and the dropout mask.
#include "../../include/msda_b200.h"
#include "msda_host.cuh"
#include "msda_vlfuse_tc.cuh"

using namespace msda_host;

namespace {

struct VlfLayout {
    size_t part0, part1, colpart, delta_v, delta_l, total;
    int row_tiles, col_tiles, nsplit, split_rows;
};

// Workspace carve-up.  The image-token ranges of the column-side kernels depend on the shape only (about 1024 CTAs), so
// the summation order, hence every bit of the result, does not depend on the device.
VlfLayout vlf_layout(int B, int H, int S, int T, int D) {
    VlfLayout l{};
    const long long BH = (long long)B * H;
    l.row_tiles = (S + vlf::kRowTile - 1) / vlf::kRowTile;
    l.col_tiles = (T + vlf::kColTile - 1) / vlf::kColTile;
    const long long per = BH * l.col_tiles, want = (1024 + per - 1) / per;
    long long rows = (S + want - 1) / want;
    rows = (rows + vlf::kChunkS - 1) / vlf::kChunkS * vlf::kChunkS;
    l.split_rows = (int)rows;
    l.nsplit = (int)((S + rows - 1) / rows);
    const size_t part = align256(sizeof(float) * (size_t)l.nsplit * BH * T * D);
    l.part0 = 0;
    l.part1 = l.colpart = part;                                             // forward: part0 + colpart
    const size_t fwd = part + align256(sizeof(float) * (size_t)BH * l.row_tiles * T * 2);
    l.delta_v = 2 * part;                                                   // backward: part0 + part1 + deltas
    l.delta_l = l.delta_v + align256(sizeof(float) * (size_t)BH * S);
    const size_t bwd = l.delta_l + align256(sizeof(float) * (size_t)BH * T);
    l.total = fwd > bwd ? fwd : bwd;
    return l;
}

int vlf_check(int B, int H, int S, int T, int D, float p) {
    if (B <= 0 || H <= 0 || S <= 0 || T <= 0 || T > vlf::kMaxT || (D != 128 && D != 256) || !(p >= 0.f && p < 1.f))
        return MSDA_E_BADARG;
    if ((long long)B * S * H * D >= (1ll << 40) || (long long)B * H >= 65536 || S >= (1 << 30)) return MSDA_E_TOOLARGE;
    return 0;
}

// The launch sequence every mode shares: the mode's row-side and column-side product kernels around vlf_colstats,
// vlf_reduce and vlf_bwd_delta.
template <int D, auto rows, auto cols, class T>
cudaError_t vlf_forward_launch(const vlf::ParamsT<T> &p, const VlfLayout &l, int rows_smem, int cols_smem, cudaStream_t st) {
    cudaError_t e;
    if ((e = opt_in_smem<rows>(rows_smem)) || (e = opt_in_smem<cols>(cols_smem))) return e;
    const unsigned BH = (unsigned)(p.B * p.H);
    rows<<<dim3(l.row_tiles, BH), vlf::kThreads, rows_smem, st>>>(p);
    vlf::vlf_colstats<<<BH, vlf::kMaxT, 0, st>>>(p, l.row_tiles);
    cols<<<dim3(l.col_tiles, l.nsplit, BH), vlf::kThreads, cols_smem, st>>>(p);
    vlf::vlf_reduce<<<dim3(p.T, BH), D, 0, st>>>(p.part0, l.nsplit, (int)BH, p.H, p.T, D, p.out_l);
    g_launches.fetch_add(4, std::memory_order_relaxed);
    return cudaGetLastError();
}

template <int D, auto rows_k, auto cols_k, class T>
cudaError_t vlf_backward_launch(const vlf::ParamsT<T> &p, const VlfLayout &l, int rows_smem, int cols_smem, cudaStream_t st) {
    cudaError_t e;
    if ((e = opt_in_smem<rows_k>(rows_smem)) || (e = opt_in_smem<cols_k>(cols_smem))) return e;
    const unsigned BH = (unsigned)(p.B * p.H);
    const long long rows = (long long)BH * (p.S + p.T);
    vlf::vlf_bwd_delta<<<(unsigned)((rows * 32 + 255) / 256), 256, 0, st>>>(p, D);
    rows_k<<<dim3(l.row_tiles, BH), vlf::kThreads, rows_smem, st>>>(p);
    cols_k<<<dim3(l.col_tiles, l.nsplit, BH), vlf::kThreads, cols_smem, st>>>(p);
    vlf::vlf_reduce<<<dim3(p.T, BH), D, 0, st>>>(p.part0, l.nsplit, (int)BH, p.H, p.T, D, p.dk);
    vlf::vlf_reduce<<<dim3(p.T, BH), D, 0, st>>>(p.part1, l.nsplit, (int)BH, p.H, p.T, D, p.dvl);
    g_launches.fetch_add(5, std::memory_order_relaxed);
    return cudaGetLastError();
}

// The product kernels of each mode: F32 (msda_vlfuse.cuh), TF32 and BF16 (msda_vlfuse_tc.cuh).
enum VlfMode { kVlfF32, kVlfTF32, kVlfBF16 };

template <int D>
cudaError_t vlf_forward_mode(const vlf::Params &p, const VlfLayout &l, VlfMode mode, cudaStream_t st) {
    if (mode == kVlfTF32)
        return vlf_forward_launch<D, vlf::vlf_tc_fwd_rows<D>, vlf::vlf_tc_fwd_cols<D>>(
            p, l, vlf::FwdRowsSmem<vlf::Tf32>::kBytes, vlf::FwdColsSmem<vlf::Tf32>::kBytes, st);
    return vlf_forward_launch<D, vlf::vlf_fwd_rows<D>, vlf::vlf_fwd_cols<D>>(p, l, vlf::kFwdRowsSmem, vlf::kFwdColsSmem, st);
}
template <int D>
cudaError_t vlf_forward_mode(const vlf::ParamsH &p, const VlfLayout &l, VlfMode, cudaStream_t st) {
    return vlf_forward_launch<D, vlf::vlf_bf16_fwd_rows<D>, vlf::vlf_bf16_fwd_cols<D>>(
        p, l, vlf::FwdRowsSmem<vlf::Bf16>::kBytes, vlf::FwdColsSmem<vlf::Bf16>::kBytes, st);
}
template <int D>
cudaError_t vlf_backward_mode(const vlf::Params &p, const VlfLayout &l, VlfMode mode, cudaStream_t st) {
    if (mode == kVlfTF32)
        return vlf_backward_launch<D, vlf::vlf_tc_bwd_rows<D>, vlf::vlf_tc_bwd_cols<D>>(
            p, l, vlf::BwdRowsSmem<vlf::Tf32>::kBytes, vlf::BwdColsSmem<vlf::Tf32>::kBytes, st);
    return vlf_backward_launch<D, vlf::vlf_bwd_rows<D>, vlf::vlf_bwd_cols<D>>(p, l, vlf::kBwdRowsSmem, vlf::kBwdColsSmem, st);
}
template <int D>
cudaError_t vlf_backward_mode(const vlf::ParamsH &p, const VlfLayout &l, VlfMode, cudaStream_t st) {
    return vlf_backward_launch<D, vlf::vlf_bf16_bwd_rows<D>, vlf::vlf_bf16_bwd_cols<D>>(
        p, l, vlf::BwdRowsSmem<vlf::Bf16>::kBytes, vlf::BwdColsSmem<vlf::Bf16>::kBytes, st);
}

// The tensors' element type behind an ABI pointer type: float, or bf16 passed as uint16_t.
template <class A> struct VlfElem { using type = float; };
template <> struct VlfElem<uint16_t> { using type = __nv_bfloat16; };

template <class A>
int vlf_forward(VlfMode mode, const A *q, const A *k, const A *v_v, const A *v_l, const float *text_bias, int B, int H,
                int S, int T, int head_dim, int clamp_min, int clamp_max, float dropout_p, const int64_t *seed, A *out_v,
                A *out_l, float *stats, void *workspace, int64_t workspace_bytes, void *stream) {
    using E = typename VlfElem<A>::type;
    if (const int c = vlf_check(B, H, S, T, head_dim, dropout_p)) return c;
    if (!all_aligned16({q, k, v_v, v_l, out_v, out_l, stats, workspace}) || (dropout_p > 0.f && !seed)) return MSDA_E_BADARG;
    const VlfLayout l = vlf_layout(B, H, S, T, head_dim);
    if (workspace_bytes < (int64_t)l.total) return MSDA_E_BADARG;
    char *ws = static_cast<char *>(workspace);
    vlf::ParamsT<E> p{};
    p.q = reinterpret_cast<const E *>(q); p.k = reinterpret_cast<const E *>(k);
    p.vv = reinterpret_cast<const E *>(v_v); p.vl = reinterpret_cast<const E *>(v_l); p.bias = text_bias;
    p.out_v = reinterpret_cast<E *>(out_v); p.out_l = reinterpret_cast<E *>(out_l);
    p.rowstat = stats;
    p.colstat = stats + (size_t)B * H * S * 2;
    p.colpart = reinterpret_cast<float *>(ws + l.colpart);
    p.part0 = reinterpret_cast<float *>(ws + l.part0);
    p.seed = seed;
    p.B = B; p.H = H; p.S = S; p.T = T;
    p.clamp_min = clamp_min != 0; p.clamp_max = clamp_max != 0;
    p.p = dropout_p; p.keep_scale = 1.f / (1.f - dropout_p);
    p.split_rows = l.split_rows;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return (int)(head_dim == 128 ? vlf_forward_mode<128>(p, l, mode, st) : vlf_forward_mode<256>(p, l, mode, st));
}

template <class A>
int vlf_backward(VlfMode mode, const A *grad_out_v, const A *grad_out_l, const A *q, const A *k, const A *v_v,
                 const A *v_l, const float *text_bias, const A *out_v, const A *out_l, const float *stats, int B, int H,
                 int S, int T, int head_dim, int clamp_min, int clamp_max, float dropout_p, const int64_t *seed, A *grad_q,
                 A *grad_k, A *grad_v_v, A *grad_v_l, void *workspace, int64_t workspace_bytes, void *stream) {
    using E = typename VlfElem<A>::type;
    if (const int c = vlf_check(B, H, S, T, head_dim, dropout_p)) return c;
    if (!all_aligned16({grad_out_v, grad_out_l, q, k, v_v, v_l, out_v, out_l, stats, grad_q, grad_k, grad_v_v, grad_v_l,
                        workspace}) || (dropout_p > 0.f && !seed))
        return MSDA_E_BADARG;
    const VlfLayout l = vlf_layout(B, H, S, T, head_dim);
    if (workspace_bytes < (int64_t)l.total) return MSDA_E_BADARG;
    char *ws = static_cast<char *>(workspace);
    vlf::ParamsT<E> p{};
    p.q = reinterpret_cast<const E *>(q); p.k = reinterpret_cast<const E *>(k);
    p.vv = reinterpret_cast<const E *>(v_v); p.vl = reinterpret_cast<const E *>(v_l); p.bias = text_bias;
    p.dov = reinterpret_cast<const E *>(grad_out_v); p.dol = reinterpret_cast<const E *>(grad_out_l);
    p.ov = reinterpret_cast<const E *>(out_v); p.ol = reinterpret_cast<const E *>(out_l);
    p.dq = reinterpret_cast<E *>(grad_q); p.dk = reinterpret_cast<E *>(grad_k);
    p.dvv = reinterpret_cast<E *>(grad_v_v); p.dvl = reinterpret_cast<E *>(grad_v_l);
    p.rowstat = const_cast<float *>(stats);
    p.colstat = const_cast<float *>(stats) + (size_t)B * H * S * 2;
    p.part0 = reinterpret_cast<float *>(ws + l.part0);
    p.part1 = reinterpret_cast<float *>(ws + l.part1);
    p.delta_v = reinterpret_cast<float *>(ws + l.delta_v);
    p.delta_l = reinterpret_cast<float *>(ws + l.delta_l);
    p.seed = seed;
    p.B = B; p.H = H; p.S = S; p.T = T;
    p.clamp_min = clamp_min != 0; p.clamp_max = clamp_max != 0;
    p.p = dropout_p; p.keep_scale = 1.f / (1.f - dropout_p);
    p.split_rows = l.split_rows;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return (int)(head_dim == 128 ? vlf_backward_mode<128>(p, l, mode, st) : vlf_backward_mode<256>(p, l, mode, st));
}

}  // namespace

extern "C" {

int msda_vlfuse_workspace(int B, int H, int S, int T, int head_dim, int64_t *bytes) {
    if (!bytes) return MSDA_E_BADARG;
    if (const int c = vlf_check(B, H, S, T, head_dim, 0.f)) return c;
    *bytes = (int64_t)vlf_layout(B, H, S, T, head_dim).total;
    return 0;
}

// The public entries: one signature per direction and element type, the mode as a flag.
#define VLF_FORWARD_ARGS(A)                                                                                              \
    const A *q, const A *k, const A *v_v, const A *v_l, const float *text_bias, int B, int H, int S, int T,            \
        int head_dim, int clamp_min, int clamp_max, float dropout_p, const int64_t *seed, A *out_v, A *out_l,           \
        float *stats, void *workspace, int64_t workspace_bytes, void *stream
#define VLF_FORWARD_PASS q, k, v_v, v_l, text_bias, B, H, S, T, head_dim, clamp_min, clamp_max, dropout_p, seed, out_v, \
                         out_l, stats, workspace, workspace_bytes, stream
#define VLF_BACKWARD_ARGS(A)                                                                                             \
    const A *grad_out_v, const A *grad_out_l, const A *q, const A *k, const A *v_v, const A *v_l,                      \
        const float *text_bias, const A *out_v, const A *out_l, const float *stats, int B, int H, int S, int T,          \
        int head_dim, int clamp_min, int clamp_max, float dropout_p, const int64_t *seed, A *grad_q, A *grad_k,         \
        A *grad_v_v, A *grad_v_l, void *workspace, int64_t workspace_bytes, void *stream
#define VLF_BACKWARD_PASS grad_out_v, grad_out_l, q, k, v_v, v_l, text_bias, out_v, out_l, stats, B, H, S, T, head_dim, \
                          clamp_min, clamp_max, dropout_p, seed, grad_q, grad_k, grad_v_v, grad_v_l, workspace,         \
                          workspace_bytes, stream

int msda_vlfuse_forward_f32(VLF_FORWARD_ARGS(float)) { return vlf_forward(kVlfF32, VLF_FORWARD_PASS); }
int msda_vlfuse_forward_tf32(VLF_FORWARD_ARGS(float)) { return vlf_forward(kVlfTF32, VLF_FORWARD_PASS); }
int msda_vlfuse_forward_bf16(VLF_FORWARD_ARGS(uint16_t)) { return vlf_forward(kVlfBF16, VLF_FORWARD_PASS); }
int msda_vlfuse_backward_f32(VLF_BACKWARD_ARGS(float)) { return vlf_backward(kVlfF32, VLF_BACKWARD_PASS); }
int msda_vlfuse_backward_tf32(VLF_BACKWARD_ARGS(float)) { return vlf_backward(kVlfTF32, VLF_BACKWARD_PASS); }
int msda_vlfuse_backward_bf16(VLF_BACKWARD_ARGS(uint16_t)) { return vlf_backward(kVlfBF16, VLF_BACKWARD_PASS); }

int msda_vlfuse_dropout_mask_f32(const int64_t *seed, int B, int H, int S, int T, float dropout_p, float *mask_v,
                                 float *mask_l, void *stream) {
    if (!seed || !mask_v || !mask_l || B <= 0 || H <= 0 || S <= 0 || T <= 0 || !(dropout_p >= 0.f && dropout_p < 1.f))
        return MSDA_E_BADARG;
    const long long n = (long long)B * H * S * T;
    const unsigned grid = (unsigned)((n + 255) / 256 < 65535 ? (n + 255) / 256 : 65535);
    return (int)launch(vlf::vlf_dropout_mask, grid, 256, 0, static_cast<cudaStream_t>(stream), seed, B * H, S, T, dropout_p,
                       mask_v, mask_l);
}

}  // extern "C"
