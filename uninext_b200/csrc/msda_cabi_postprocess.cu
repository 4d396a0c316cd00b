// msda_cabi_postprocess.cu -- C ABI of the inference post-processing: mask pasting (msda_maskpaste.cuh), COCO run-length
// encoding of masks (msda_maskrle.cuh), detection post-processing and the video trackers' detection selection
// (msda_detpost.cuh; the latter's entry points are declared in include/msda_trackpost.h).
#include "../../include/msda_b200.h"
#include "../../include/msda_trackpost.h"
#include "msda_detpost.cuh"
#include "msda_host.cuh"
#include "msda_maskpaste.cuh"
#include "msda_maskrle.cuh"

using namespace msda_host;

namespace {

// ---- mask pasting (f-5) -------------------------------------------------------------------------------------------------
// msda_mask_paste_f32's limits.  msda_mask_rle_count_f32 checks the same ones: its bits are the pixels the paste writes.
int paste_check(int64_t I, int Hs, int Ws, int stride, int crop_h, int crop_w, int out_h, int out_w) {
    if (I < 0 || Hs <= 0 || Ws <= 0 || stride <= 0 || crop_h <= 0 || crop_w <= 0 || out_h <= 0 || out_w <= 0 ||
        (long long)stride * Hs >= (1ll << 31) || (long long)stride * Ws >= (1ll << 31) || crop_h > stride * Hs ||
        crop_w > stride * Ws)
        return MSDA_E_BADARG;
    if (out_h > 65535 * msda::kMpRows || out_w >= (1 << 30)) return MSDA_E_TOOLARGE;
    return 0;
}

// The scales exactly as torch forms them for an explicit output size: (float)input_size / output_size.
struct PasteScales { float near_y, near_x, lin_y, lin_x; };

PasteScales paste_scales(int Hs, int Ws, int stride, int crop_h, int crop_w, int out_h, int out_w) {
    return {(float)crop_h / (float)out_h, (float)crop_w / (float)out_w, (float)Hs / (float)(stride * Hs),
            (float)Ws / (float)(stride * Ws)};
}

// ---- detection post-processing (f-6) ----------------------------------------------------------------------------------
struct DetpostLayout {
    size_t prob, qmax, qarg, sort, total;
    long long sort_cap;                         // u64 sort slots per image in the workspace (0: the CTA sorts on chip)
};

int detpost_check(int B, int Q, int T, int C, int max_num_inst) {
    if (B < 0 || B > 65535 || Q < 1 || Q > msda::kDpMaxQ || T < 1 || T > msda::kDpMaxT || C < 1 || C > msda::kDpMaxC ||
        max_num_inst < 1 || (long long)max_num_inst > (long long)Q * C)
        return MSDA_E_BADARG;
    return 0;
}

DetpostLayout detpost_layout(int B, int Q, int C, int max_num_inst) {
    DetpostLayout l{};
    long long p = 1;
    while (p < max_num_inst) p <<= 1;
    l.sort_cap = p > msda::kDpSmemSort ? p : 0;
    l.prob = 0;
    l.qmax = align256(l.prob + (size_t)B * Q * C * sizeof(float));
    l.qarg = align256(l.qmax + (size_t)B * Q * sizeof(float));
    l.sort = align256(l.qarg + (size_t)B * Q * sizeof(int));
    l.total = align256(l.sort + (size_t)B * l.sort_cap * sizeof(unsigned long long));
    return l;
}

// ---- COCO run-length encoding of masks (f-7) ----------------------------------------------------------------------------
struct RleLayout {
    size_t col_off, bitmap, scan, scan_bytes, tiles, total;
};

int rle_check(long long I, int out_h, int out_w) {
    if (I < 0 || out_h < 1 || out_w < 1) return MSDA_E_BADARG;
    // The COCO API's counts are 32-bit unsigned: a mask of more than 2^32 - 1 pixels has no RLE.
    if (I >= (1ll << 31) || (unsigned long long)out_h * (unsigned)out_w > 0xffffffffull || out_w >= (1 << 30))
        return MSDA_E_TOOLARGE;
    return 0;
}

// [I * W + 1] column offsets (first, so the caller finds the total at entry I * W), the bitmap, cub's scan storage and
// pass 3's tile sums for the most counts an instance can have (every pixel a boundary, plus one).
int rle_layout(long long I, int out_h, int out_w, RleLayout &l) {
    const long long cols = I * out_w + 1, nw = (out_h + 31) / 32;
    const long long max_tiles = (I * ((long long)out_h * out_w + 1) + msda::kRleTile - 1) / msda::kRleTile;
    l.scan_bytes = 0;
    const cudaError_t e = cub::DeviceScan::ExclusiveSum(nullptr, l.scan_bytes, (long long *)nullptr, cols);
    if (e != cudaSuccess) return (int)e;
    l.col_off = 0;
    l.bitmap = align256(l.col_off + (size_t)cols * sizeof(long long));
    l.scan = align256(l.bitmap + (size_t)I * nw * out_w * sizeof(unsigned));
    l.tiles = align256(l.scan + l.scan_bytes);
    l.total = align256(l.tiles + (size_t)max_tiles * sizeof(long long));
    return 0;
}

dim3 rle_grid(long long I, int out_w, int cols_per_thread) {
    const long long per_block = (long long)msda::kRleThreads * cols_per_thread;
    return dim3((unsigned)((out_w + per_block - 1) / per_block), (unsigned)(I < 65535 ? I : 65535));
}

// The scan after pass 1 (cub: an init kernel and the scan kernel); counts pass 1 and the scan's two launches.
int rle_scan(long long I, int out_w, const RleLayout &l, char *ws, cudaStream_t st) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return (int)e;
    size_t scan_bytes = l.scan_bytes;
    e = cub::DeviceScan::ExclusiveSum(ws + l.scan, scan_bytes, reinterpret_cast<long long *>(ws + l.col_off),
                                      I * out_w + 1, st);
    g_launches.fetch_add(3, std::memory_order_relaxed);
    return e != cudaSuccess ? (int)e : (int)cudaGetLastError();
}

}  // namespace

extern "C" {

int msda_mask_paste_f32(const float *logits, int64_t I, int Hs, int Ws, int stride, int crop_h, int crop_w, int out_h,
                        int out_w, float threshold, int binary, void *out, void *stream) {
    if (!logits || !out) return MSDA_E_BADARG;
    if (const int c = paste_check(I, Hs, Ws, stride, crop_h, crop_w, out_h, out_w)) return c;
    if (I == 0) return 0;
    constexpr int cols = msda::kMpGroups * msda::kMpCols, rows = msda::kMpRows;
    const PasteScales s = paste_scales(Hs, Ws, stride, crop_h, crop_w, out_h, out_w);
    const long long chunks = (I + msda::kMpInst - 1) / msda::kMpInst;
    const dim3 grid((unsigned)((out_w + cols - 1) / cols), (unsigned)((out_h + rows - 1) / rows),
                    (unsigned)(chunks < 65535 ? chunks : 65535));
    const dim3 block(msda::kMpGroups, rows);
    const bool vec = aligned16(out) && out_w % (binary ? msda::kMpCols : 4) == 0;
    const auto go = [&](auto kernel) {
        return (int)launch(kernel, grid, block, 0, static_cast<cudaStream_t>(stream), logits, I, Hs, Ws, crop_h, crop_w,
                           out_h, out_w, s.near_y, s.near_x, s.lin_y, s.lin_x, threshold, out);
    };
    if (binary) return vec ? go(msda::mask_paste<true, true>) : go(msda::mask_paste<true, false>);
    return vec ? go(msda::mask_paste<false, true>) : go(msda::mask_paste<false, false>);
}

int msda_detpost_workspace(int B, int Q, int T, int C, int max_num_inst, int64_t *bytes) {
    if (!bytes) return MSDA_E_BADARG;
    if (const int c = detpost_check(B, Q, T, C, max_num_inst)) return c;
    *bytes = (int64_t)detpost_layout(B, Q, C, max_num_inst).total;
    return 0;
}

int msda_detpost_f32(const float *box_cls, const float *box_pred, const float *iou_pred, const int *class_start,
                     const int *tokens, const int *image_sizes, int B, int Q, int T, int C, int nms, float nms_iou,
                     int max_num_inst, float *scores, int *labels, int *query_index, float *boxes, int *count,
                     void *workspace, int64_t workspace_bytes, void *stream) {
    if (!box_cls || !box_pred || !class_start || !tokens || !image_sizes || !scores || !labels || !query_index ||
        !boxes || !count || !workspace || !aligned16(boxes) || !aligned16(workspace))
        return MSDA_E_BADARG;
    if (const int c = detpost_check(B, Q, T, C, max_num_inst)) return c;
    const DetpostLayout l = detpost_layout(B, Q, C, max_num_inst);
    if (workspace_bytes < (int64_t)l.total) return MSDA_E_BADARG;
    if (B == 0) return 0;
    char *ws = static_cast<char *>(workspace);
    float *prob = reinterpret_cast<float *>(ws + l.prob), *qmax = reinterpret_cast<float *>(ws + l.qmax);
    int *qarg = reinterpret_cast<int *>(ws + l.qarg);
    unsigned long long *sort_ws = reinterpret_cast<unsigned long long *>(ws + l.sort);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const dim3 sgrid((unsigned)((Q + msda::kDpScoreWarps - 1) / msda::kDpScoreWarps), (unsigned)B);
    msda::detpost_scores<<<sgrid, msda::kDpScoreWarps * 32, 0, st>>>(box_cls, iou_pred, class_start, tokens, Q, T, C,
                                                                     prob, qmax, qarg);
    if (nms) {
        // The opt-in is set once per device, to the Q = kDpMaxQ size, so no call can lower it under another's launch.
        constexpr int kDynMax = msda::kDpMaxQ * (int)sizeof(float4) +
                                msda::kDpMaxQ * ((msda::kDpMaxQ + 63) / 64) * (int)sizeof(unsigned long long);
        if (const cudaError_t e = opt_in_smem<msda::detpost_select<true>>(kDynMax)) return (int)e;
        const size_t dyn = (size_t)Q * sizeof(float4) + (size_t)Q * ((Q + 63) / 64) * sizeof(unsigned long long);
        msda::detpost_select<true><<<B, msda::kDpThreads, dyn, st>>>(box_pred, image_sizes, prob, qmax, qarg, Q, C,
                                                                     nms_iou, max_num_inst, l.sort_cap, sort_ws, scores,
                                                                     labels, query_index, boxes, count);
    } else {
        msda::detpost_select<false><<<B, msda::kDpThreads, 0, st>>>(box_pred, image_sizes, prob, qmax, qarg, Q, C,
                                                                    nms_iou, max_num_inst, l.sort_cap, sort_ws, scores,
                                                                    labels, query_index, boxes, count);
    }
    g_launches.fetch_add(2, std::memory_order_relaxed);
    return (int)cudaGetLastError();
}

int msda_trackpost_workspace(int B, int Q, int T, int C, int64_t *bytes) {
    if (!bytes) return MSDA_E_BADARG;
    if (const int c = detpost_check(B, Q, T, C, 1)) return c;
    *bytes = (int64_t)detpost_layout(B, Q, C, 1).total;        // prob, qmax, qarg; one result needs no sort buffer
    return 0;
}

int msda_trackpost_f32(const float *box_cls, const float *box_pred, const float *iou_pred, const int *class_start,
                       const int *tokens, const int *ori_sizes, int B, int Q, int T, int C, float score_thres,
                       float nms_iou, int box_format, float *scores, int *labels, int *query_index, float *boxes,
                       int *count, void *workspace, int64_t workspace_bytes, void *stream) {
    if (box_format != MSDA_TRACKPOST_CXCYWH && box_format != MSDA_TRACKPOST_XYXY_PIXELS) return MSDA_E_BADARG;
    const bool pixels = box_format == MSDA_TRACKPOST_XYXY_PIXELS;
    if (!box_cls || !box_pred || !class_start || !tokens || (pixels && !ori_sizes) || !scores || !labels ||
        !query_index || !boxes || !count || !workspace || !aligned16(boxes) || !aligned16(workspace))
        return MSDA_E_BADARG;
    if (const int c = detpost_check(B, Q, T, C, 1)) return c;
    const DetpostLayout l = detpost_layout(B, Q, C, 1);
    if (workspace_bytes < (int64_t)l.total) return MSDA_E_BADARG;
    if (B == 0) return 0;
    char *ws = static_cast<char *>(workspace);
    float *prob = reinterpret_cast<float *>(ws + l.prob), *qmax = reinterpret_cast<float *>(ws + l.qmax);
    int *qarg = reinterpret_cast<int *>(ws + l.qarg);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const dim3 sgrid((unsigned)((Q + msda::kDpScoreWarps - 1) / msda::kDpScoreWarps), (unsigned)B);
    if (const cudaError_t e = launch(msda::detpost_scores, sgrid, msda::kDpScoreWarps * 32, 0, st, box_cls, iou_pred,
                                     class_start, tokens, Q, T, C, prob, qmax, qarg))
        return (int)e;
    // The opt-in is set once per device, to the Q = kDpMaxQ size, as for detpost_select<true>.
    constexpr int kDynMax = msda::kDpMaxQ * (int)sizeof(float4) +
                            msda::kDpMaxQ * ((msda::kDpMaxQ + 63) / 64) * (int)sizeof(unsigned long long);
    if (const cudaError_t e = opt_in_smem<msda::trackpost_select>(kDynMax)) return (int)e;
    const size_t dyn = (size_t)Q * sizeof(float4) + (size_t)Q * ((Q + 63) / 64) * sizeof(unsigned long long);
    return (int)launch(msda::trackpost_select, dim3((unsigned)B), msda::kDpThreads, dyn, st, box_pred,
                       pixels ? ori_sizes : nullptr, qmax, qarg, Q, score_thres, nms_iou, (int)pixels, scores, labels,
                       query_index, boxes, count);
}

int msda_mask_rle_workspace(int64_t I, int out_h, int out_w, int64_t *bytes) {
    if (!bytes) return MSDA_E_BADARG;
    if (const int c = rle_check(I, out_h, out_w)) return c;
    if (I == 0) { *bytes = 0; return 0; }
    RleLayout l;
    if (const int e = rle_layout(I, out_h, out_w, l)) return e;
    *bytes = (int64_t)l.total;
    return 0;
}

int msda_mask_rle_count_f32(const float *logits, int64_t I, int Hs, int Ws, int stride, int crop_h, int crop_w,
                            int out_h, int out_w, float threshold, void *workspace, int64_t workspace_bytes,
                            void *stream) {
    if (!logits || !workspace || !aligned16(workspace)) return MSDA_E_BADARG;
    if (const int c = paste_check(I, Hs, Ws, stride, crop_h, crop_w, out_h, out_w)) return c;
    if (const int c = rle_check(I, out_h, out_w)) return c;
    if (I == 0) return 0;
    RleLayout l;
    if (const int e = rle_layout(I, out_h, out_w, l)) return e;
    if (workspace_bytes < (int64_t)l.total) return MSDA_E_BADARG;
    char *ws = static_cast<char *>(workspace);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const PasteScales s = paste_scales(Hs, Ws, stride, crop_h, crop_w, out_h, out_w);
    msda::rle_bits_logits<<<rle_grid(I, out_w, 1), msda::kRleThreads, 0, st>>>(
        logits, I, Hs, Ws, crop_h, crop_w, out_h, out_w, s.near_y, s.near_x, s.lin_y, s.lin_x, threshold,
        reinterpret_cast<unsigned *>(ws + l.bitmap), reinterpret_cast<long long *>(ws + l.col_off));
    return rle_scan(I, out_w, l, ws, st);
}

int msda_mask_rle_count_u8(const uint8_t *masks, int64_t I, int out_h, int out_w, void *workspace,
                           int64_t workspace_bytes, void *stream) {
    if (!masks || !workspace || !aligned16(workspace)) return MSDA_E_BADARG;
    if (const int c = rle_check(I, out_h, out_w)) return c;
    if (I == 0) return 0;
    RleLayout l;
    if (const int e = rle_layout(I, out_h, out_w, l)) return e;
    if (workspace_bytes < (int64_t)l.total) return MSDA_E_BADARG;
    char *ws = static_cast<char *>(workspace);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    unsigned *bitmap = reinterpret_cast<unsigned *>(ws + l.bitmap);
    long long *col_count = reinterpret_cast<long long *>(ws + l.col_off);
    const dim3 grid = rle_grid(I, out_w, msda::kRleU8Cols);
    if ((reinterpret_cast<uintptr_t>(masks) & 3u) == 0 && out_w % 4 == 0)
        msda::rle_bits_u8<true><<<grid, msda::kRleThreads, 0, st>>>(masks, I, out_h, out_w, bitmap, col_count);
    else
        msda::rle_bits_u8<false><<<grid, msda::kRleThreads, 0, st>>>(masks, I, out_h, out_w, bitmap, col_count);
    return rle_scan(I, out_w, l, ws, st);
}

int msda_mask_rle_encode(int64_t I, int out_h, int out_w, int64_t boundaries, void *workspace, int64_t workspace_bytes,
                         uint32_t *positions, int64_t *byte_offsets, char *chars, void *stream) {
    if (!workspace || !aligned16(workspace) || !byte_offsets || !chars || (boundaries > 0 && !positions) ||
        (reinterpret_cast<uintptr_t>(positions) & 3u) || !aligned8(byte_offsets))
        return MSDA_E_BADARG;
    if (const int c = rle_check(I, out_h, out_w)) return c;
    if (boundaries < 0 || (I > 0 && boundaries > I * ((long long)out_h * out_w))) return MSDA_E_BADARG;
    if (I == 0) return 0;
    RleLayout l;
    if (const int e = rle_layout(I, out_h, out_w, l)) return e;
    if (workspace_bytes < (int64_t)l.total) return MSDA_E_BADARG;
    char *ws = static_cast<char *>(workspace);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long *col_off = reinterpret_cast<const long long *>(ws + l.col_off);
    long long *tiles = reinterpret_cast<long long *>(ws + l.tiles);
    msda::rle_boundaries<<<rle_grid(I, out_w, 1), msda::kRleThreads, 0, st>>>(
        reinterpret_cast<const unsigned *>(ws + l.bitmap), col_off, I, out_h, out_w, positions);
    const msda::RleCounts rc{col_off, positions, I, boundaries + I, (long long)out_h * out_w, out_w};
    const long long ntiles = (rc.N + msda::kRleTile - 1) / msda::kRleTile;
    msda::rle_tile_bytes<<<(unsigned)ntiles, msda::kRleTileThreads, 0, st>>>(rc, tiles);
    msda::rle_scan_tiles<<<1, msda::kRleScanThreads, 0, st>>>(tiles, ntiles);
    msda::rle_write<<<(unsigned)ntiles, msda::kRleTileThreads, 0, st>>>(rc, tiles, reinterpret_cast<long long *>(byte_offsets), chars);
    g_launches.fetch_add(4, std::memory_order_relaxed);
    return (int)cudaGetLastError();
}

}  // extern "C"
