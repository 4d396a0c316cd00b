// Driver for tools/region_cosched.py: the region backward's chain as the library launches it -- msda_zero_fill, then
// msda_region_grad_value_pass<8, 2> as its PDL secondary, then msda_bwd_region<8, 2> (tap pass) as the grad_value
// kernel's PDL secondary, grids and the grad_value kernel's padded shared memory from msda::region_grids -- with the kernels built with the placement hook
// (MSDA_REGION_COSCHED, msda_region.cuh).  Plain C entry points for ctypes; the caller owns the record buffers
// ([grid x 3] u64 per kernel: %smid, start and end %globaltimer of each CTA).
#define MSDA_REGION_COSCHED
#include "msda_generic.cuh"
#include "msda_region.cuh"

namespace {

constexpr auto kTap = msda::msda_bwd_region<msda::kRegionEdge, msda::kRegionHalo>;
constexpr auto kGv = msda::msda_region_grad_value_pass<msda::kRegionEdge, msda::kRegionHalo>;

int sm_count() {
    int dev = 0, sms = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
        return -1;
    return sms;
}

template <class K, class... Args>
cudaError_t launch_pdl(K kern, int grid, size_t smem, cudaStream_t st, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3(msda::kTiledThreads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kern, args...);
}

msda::RegionGrids grids() {
    return msda::region_grids(kGv, msda::region_gv_smem_bytes(), kTap, msda::region_tap_smem_bytes(), sm_count());
}

}  // namespace

// grids[0] = grad_value CTAs, grids[1] = tap CTAs, grids[2] = SMs, grids[3] = the grad_value kernel's dynamic shared
// memory.  Returns 0, or -1 on error.
extern "C" int region_cosched_grids(int *out) {
    if (cudaFuncSetAttribute(kGv, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)msda::region_gv_smem_bytes()) !=
        cudaSuccess)
        return -1;
    const msda::RegionGrids g = grids();
    out[0] = g.gv; out[1] = g.tap; out[2] = sm_count(); out[3] = (int)g.gv_smem;
    return out[2] > 0 ? 0 : -1;
}

// One region backward on `stream`: fill -> grad_value kernel -> tap kernel, recording into gv_rec / tap_rec.  Returns 0,
// or -1 on error.
extern "C" int region_cosched_run(void *stream, unsigned long long *gv_rec, unsigned long long *tap_rec, const float *go,
                                  const float *value, const int64_t *shapes, const int64_t *lsi, const float *loc,
                                  const float *attn, int N, int S, int M, int L, int Lq, int P, float *gv, float *gl,
                                  float *ga) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    unsigned long long *rec[2] = {gv_rec, tap_rec};
    if (cudaMemcpyToSymbolAsync(msda::g_region_cosched, rec, sizeof(rec), 0, cudaMemcpyHostToDevice, st) != cudaSuccess)
        return -1;
    const msda::RegionGrids g = grids();
    const int sms = sm_count();
    const unsigned long long n16 = (unsigned long long)N * S * M * 32 * sizeof(float) / 16;
    const unsigned long long fill_blocks = (n16 + 255) / 256, cap = (unsigned long long)sms * 8;
    msda::msda_zero_fill<<<(unsigned)(fill_blocks < cap ? fill_blocks : cap), 256, 0, st>>>(reinterpret_cast<uint4 *>(gv), n16);
    if (cudaGetLastError() != cudaSuccess) return -1;
    const unsigned npairs = (unsigned)((long long)N * Lq * M);
    if (launch_pdl(kGv, g.gv, g.gv_smem, st, go, shapes, lsi, loc, attn, N, S, M, L, Lq, P, npairs, gv) !=
        cudaSuccess)
        return -1;
    const int tma = (L * P) % 4 == 0 ? 1 : 0;
    if (launch_pdl(kTap, g.tap, msda::region_tap_smem_bytes(), st, go, value, shapes, lsi, loc, attn, N, S, M, L, Lq, P,
                   npairs, tma, gl, ga) != cudaSuccess)
        return -1;
    return 0;
}
