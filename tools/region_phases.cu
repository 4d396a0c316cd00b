// Driver for tools/region_phases.py: the region backward's two kernels, msda_bwd_region<8, HALO> (tap pass) and
// msda_region_grad_value_pass<8, HALO> built with the phase-clock hook (MSDA_REGION_PHASE_CLOCKS, msda_region.cuh), for
// HALO in 1..6, launched as the library launches them (occupancy x SMs CTAs each, TMA-staged taps when L*P % 4 == 0) but
// without the PDL pairing, so that CUDA events can time each kernel on its own.  Plain C entry points for ctypes; the
// caller zero-fills grad_value and owns the clock buffer ([grid x kRegionSpans] u64).
#define MSDA_REGION_PHASE_CLOCKS
#include "msda_region.cuh"

namespace {

int sm_count() {
    int dev = 0, sms = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
        return -1;
    return sms;
}

// Dynamic shared memory of the grad_value kernel: region_gv_smem_bytes(), padded in 1 KB steps until at most `ctas`
// CTAs fit on an SM when ctas > 0 (the same code at a lower occupancy, for comparisons).  Sets the opt-in and *per_sm.
template <class K>
int gv_smem(K kern, int ctas, int *per_sm) {
    size_t smem = msda::region_gv_smem_bytes();
    int max_optin = 0, dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&max_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess)
        return -1;
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, max_optin - 8192) != cudaSuccess) return -1;
    for (;;) {
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(per_sm, kern, msda::kTiledThreads, smem) != cudaSuccess) return -1;
        if (ctas <= 0 || *per_sm <= ctas || smem + 1024 > (size_t)max_optin - 8192) break;
        smem += 1024;
    }
    return (int)smem;
}

template <int HALO>
int launch(int which, int ctas, int setup, unsigned long long *clocks, int knockout, const float *go, const float *value,
           const int64_t *shapes, const int64_t *lsi, const float *loc, const float *attn, int N, int S, int M, int L,
           int Lq, int P, float *gv, float *gl, float *ga) {
    auto tap = msda::msda_bwd_region<msda::kRegionEdge, HALO>;
    auto gvk = msda::msda_region_grad_value_pass<msda::kRegionEdge, HALO>;
    const int sms = sm_count();
    int per_sm = 0;
    const int smem = gv_smem(gvk, ctas, &per_sm);
    if (sms < 0 || smem < 0) return -1;
    const int grid = (per_sm < 1 ? 1 : per_sm) * sms;
    if (setup) {          // symbols are set outside the timed launches (cudaMemcpyToSymbol synchronises)
        if (cudaMemcpyToSymbol(msda::g_region_clocks, &clocks, sizeof(clocks)) != cudaSuccess ||
            cudaMemcpyToSymbol(msda::g_region_knockout, &knockout, sizeof(knockout)) != cudaSuccess)
            return -1;
        return grid;
    }
    const unsigned npairs = (unsigned)((long long)N * Lq * M);
    if (which == 0) {
        int tap_per_sm = 0;
        constexpr size_t tap_smem = msda::region_tap_smem_bytes();
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&tap_per_sm, tap, msda::kTiledThreads, tap_smem) != cudaSuccess)
            return -1;
        const int tap_grid = (tap_per_sm < 1 ? 1 : tap_per_sm) * sms;
        const int tma = (L * P) % 4 == 0 ? 1 : 0;
        tap<<<tap_grid, msda::kTiledThreads, tap_smem>>>(go, value, shapes, lsi, loc, attn, N, S, M, L, Lq, P, npairs, tma,
                                                          gl, ga);
        return cudaGetLastError() == cudaSuccess ? tap_grid : -1;
    }
    gvk<<<grid, msda::kTiledThreads, smem>>>(go, shapes, lsi, loc, attn, N, S, M, L, Lq, P, npairs, gv);
    return cudaGetLastError() == cudaSuccess ? grid : -1;
}

}  // namespace

// which = 0: the tap kernel, 1: the grad_value kernel.  ctas > 0 caps the grad_value kernel's CTAs per SM (padded
// dynamic shared memory); 0 launches it as the library does.
// setup != 0: point the hook at `clocks` ([grid x kRegionSpans] u64) and set the knockout bits; returns the grad_value
// kernel's grid size (-1 on error).
// setup == 0: one launch on the legacy default stream; returns the grid size (-1 on error).
extern "C" int region_phases_run(int halo, int which, int ctas, int setup, unsigned long long *clocks, int knockout,
                                 const float *go, const float *value, const int64_t *shapes, const int64_t *lsi,
                                 const float *loc, const float *attn, int N, int S, int M, int L, int Lq, int P,
                                 float *gv, float *gl, float *ga) {
#define MSDA_REGION_HALO_CASE(h)                                                                                       \
    case h:                                                                                                            \
        return launch<h>(which, ctas, setup, clocks, knockout, go, value, shapes, lsi, loc, attn, N, S, M, L, Lq, P, gv, \
                         gl, ga);
    switch (halo) {
        MSDA_REGION_HALO_CASE(1)
        MSDA_REGION_HALO_CASE(2)
        MSDA_REGION_HALO_CASE(3)
        MSDA_REGION_HALO_CASE(4)
        MSDA_REGION_HALO_CASE(5)
        MSDA_REGION_HALO_CASE(6)
    }
#undef MSDA_REGION_HALO_CASE
    return -1;
}

extern "C" int region_phases_spans() { return msda::kRegionSpans; }
