// Driver for tools/region_phases.py: msda_bwd_region<8, HALO> built with the phase-clock hook (MSDA_REGION_PHASE_CLOCKS,
// msda_region.cuh) for HALO in 1..6, launched as the library launches it (region_smem_bytes() of dynamic shared memory,
// occupancy x SMs CTAs, TMA-staged taps when L*P % 4 == 0).  Plain C entry points for ctypes; the caller zero-fills
// grad_value and owns the clock buffer ([grid x kRegionSpans] u64).
#define MSDA_REGION_PHASE_CLOCKS
#include "msda_region.cuh"

namespace {

template <int HALO>
int launch(int setup, unsigned long long *clocks, int knockout, const float *go, const float *value, const int64_t *shapes,
           const int64_t *lsi, const float *loc, const float *attn, int N, int S, int M, int L, int Lq, int P, float *gv,
           float *gl, float *ga) {
    auto kern = msda::msda_bwd_region<msda::kRegionEdge, HALO>;
    constexpr size_t smem = msda::region_smem_bytes();
    int dev = 0, sms = 0, per_sm = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
        return -1;
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return -1;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, msda::kTiledThreads, smem) != cudaSuccess) return -1;
    const int grid = (per_sm < 1 ? 1 : per_sm) * sms;
    if (setup) {          // symbols are set outside the timed launches (cudaMemcpyToSymbol synchronises)
        if (cudaMemcpyToSymbol(msda::g_region_clocks, &clocks, sizeof(clocks)) != cudaSuccess ||
            cudaMemcpyToSymbol(msda::g_region_knockout, &knockout, sizeof(knockout)) != cudaSuccess)
            return -1;
        return grid;
    }
    const unsigned npairs = (unsigned)((long long)N * Lq * M);
    const int tma = (L * P) % 4 == 0 ? 1 : 0;
    kern<<<grid, msda::kTiledThreads, smem>>>(go, value, shapes, lsi, loc, attn, N, S, M, L, Lq, P, npairs, tma, gv, gl, ga);
    return cudaGetLastError() == cudaSuccess ? grid : -1;
}

}  // namespace

// setup != 0: point the hook at `clocks` ([grid x kRegionSpans] u64) and set the knockout bits; returns the grid size (-1 on error).
// setup == 0: one launch on the legacy default stream; returns the grid size (-1 on error).
extern "C" int region_phases_run(int halo, int setup, unsigned long long *clocks, int knockout, const float *go,
                                 const float *value, const int64_t *shapes, const int64_t *lsi, const float *loc,
                                 const float *attn, int N, int S, int M, int L, int Lq, int P, float *gv, float *gl,
                                 float *ga) {
    switch (halo) {
        case 1: return launch<1>(setup, clocks, knockout, go, value, shapes, lsi, loc, attn, N, S, M, L, Lq, P, gv, gl, ga);
        case 2: return launch<2>(setup, clocks, knockout, go, value, shapes, lsi, loc, attn, N, S, M, L, Lq, P, gv, gl, ga);
        case 3: return launch<3>(setup, clocks, knockout, go, value, shapes, lsi, loc, attn, N, S, M, L, Lq, P, gv, gl, ga);
        case 4: return launch<4>(setup, clocks, knockout, go, value, shapes, lsi, loc, attn, N, S, M, L, Lq, P, gv, gl, ga);
        case 5: return launch<5>(setup, clocks, knockout, go, value, shapes, lsi, loc, attn, N, S, M, L, Lq, P, gv, gl, ga);
        case 6: return launch<6>(setup, clocks, knockout, go, value, shapes, lsi, loc, attn, N, S, M, L, Lq, P, gv, gl, ga);
    }
    return -1;
}

extern "C" int region_phases_spans() { return msda::kRegionSpans; }
