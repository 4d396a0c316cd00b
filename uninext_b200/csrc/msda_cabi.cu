// msda_cabi.cu -- the op's part of the C ABI declared in include/msda_b200.h: knobs, argument checks, kernel routing and
// launches of the forward, the backward and the deterministic backward.  The other entry points are in
// msda_cabi_{module,condinst,postprocess,vlfuse}.cu, one translation unit per kernel family.
// Replaces the reference host wrappers ms_deform_attn_cuda_forward/backward (ops/src/cuda/ms_deform_attn_cuda.cu)
// and launchers ms_deformable_im2col_cuda / ms_deformable_col2im_cuda (ms_deform_im2col_cuda.cuh:923-954,956-1327).
#include <type_traits>

#include "../../include/msda_b200.h"
#include "msda_det.cuh"
#include "msda_generic.cuh"
#include "msda_host.cuh"
#include "msda_region.cuh"
#include "msda_slab.cuh"
#include "msda_tmem.cuh"
#include "msda_tiled.cuh"

std::atomic<uint64_t> msda_host::g_launches{0};

namespace {

using namespace msda_host;

struct Dims { int N, S, M, D, L, Lq, P; };

int check_dims(const Dims &d) {
    if (d.N <= 0 || d.S <= 0 || d.M <= 0 || d.D <= 0 || d.L <= 0 || d.Lq <= 0 || d.P <= 0) return MSDA_E_BADARG;
    // rows are indexed with int32 inside a batch element; tap counts with int64 everywhere.
    if ((long long)d.S >= (1ll << 30)) return MSDA_E_TOOLARGE;
    if ((long long)d.N * d.Lq * d.M >= (1ll << 40)) return MSDA_E_TOOLARGE;
    return 0;
}

// Kernel-selection knobs (msda_set_knob): environment defaults, overridable at run time.  g_knob_epoch invalidates the
// per-device launch configurations derived from them.
struct Knobs {
    std::atomic<int> v[MSDA_KNOB_COUNT];
    std::atomic<int> epoch{1};
    Knobs() {
        v[MSDA_KNOB_SLAB].store(env_int("MSDA_SLAB", -1));
        v[MSDA_KNOB_BWD_WIN_ROWS].store(env_int("MSDA_BWD_WIN_ROWS", -1));
        v[MSDA_KNOB_BWD_LIST_CAP].store(env_int("MSDA_BWD_LIST_CAP", 48));
        v[MSDA_KNOB_FWD_SLAB_CTAS].store(env_int("MSDA_FWD_SLAB_CTAS", 2));
        v[MSDA_KNOB_F32_VEC8_FWD].store(env_int("MSDA_F32_VEC8_FWD", 0));
        v[MSDA_KNOB_F32_VEC8_BWD].store(env_int("MSDA_F32_VEC8_BWD", 0));
        v[MSDA_KNOB_BF16_FINE_ROWS].store(env_int("MSDA_BF16_FINE_ROWS", 0));
        v[MSDA_KNOB_BF16_PACKED_FWD].store(env_int("MSDA_BF16_PACKED_FWD", 0));
        v[MSDA_KNOB_ZERO_FILL].store(env_int("MSDA_ZERO_FILL", 2));
        v[MSDA_KNOB_REGION_BWD].store(env_int("MSDA_REGION_BWD", -1));
    }
};
Knobs &knobs() { static Knobs k; return k; }
int knob(int i) { return knobs().v[i].load(std::memory_order_relaxed); }

// Zero-fill of grad_value before the backward kernels (MSDA_KNOB_ZERO_FILL).  *pdl is set when the fill went out as a
// kernel that the NEXT launch on `st` may take as its programmatic-dependent-launch primary.  The fill kernel stands in
// for a memset and is not counted by msda_launch_count().
cudaError_t zero_fill(void *p, size_t bytes, cudaStream_t st, bool *pdl = nullptr) {
    if (pdl) *pdl = false;
    const int mode = knob(MSDA_KNOB_ZERO_FILL);
    if (mode <= 0 || bytes < (1u << 16) || !aligned16(p) || (bytes & 15u)) return cudaMemsetAsync(p, 0, bytes, st);
    const unsigned long long n16 = bytes >> 4;
    // 8 x 256 threads = every thread slot of an SM
    msda::msda_zero_fill<<<capped_grid((long long)n16, 256, 8), 256, 0, st>>>(static_cast<uint4 *>(p), n16);
    const cudaError_t err = cudaGetLastError();
    if (pdl && mode >= 2 && err == cudaSuccess) {
        cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
        *pdl = cudaStreamIsCapturing(st, &cap) == cudaSuccess && cap == cudaStreamCaptureStatusNone;
    }
    return err;
}

// ---- routing ------------------------------------------------------------------------------------------------
// Fast path: D in {16,32,64} (fp32) / {32,64} (bf16), L <= kMaxLevels, L*P <= 32.  LP_MAX is the compile-time tap
// capacity (taps beyond L*P are dead: zero weight, row 0).
bool fast_ok(int dtype_bytes, int D, int L, int P) {
    if (L > msda::kMaxLevels || L * P > 32) return false;
    if (dtype_bytes == 4) return D == 16 || D == 32 || D == 64;
    if (dtype_bytes == 2) return D == 32 || D == 64;
    return false;
}

bool use_fast(int dtype_bytes, const Dims &d) {      // the tiled kernels index (b,q,m) pairs with 31 bits
    return fast_ok(dtype_bytes, d.D, d.L, d.P) && (long long)d.N * d.Lq * d.M < (1ll << 31);
}

unsigned num_pairs(const Dims &d) { return (unsigned)((long long)d.N * d.Lq * d.M); }

// The tiled instantiations, one per (D, LP_MAX): D in {16 (fp32 only), 32, 64}, LP_MAX in {16, 32}.  f(D, LP_MAX)
// receives them as std::integral_constant.
template <typename T, class F>
cudaError_t route_tiled(const Dims &d, F f) {
    using L16 = std::integral_constant<int, 16>;
    using L32 = std::integral_constant<int, 32>;
    const bool lp16 = d.L * d.P <= 16;
    switch (d.D) {
        case 16:
            if constexpr (sizeof(T) == 4) return lp16 ? f(L16{}, L16{}) : f(L16{}, L32{});
            break;
        case 32: return lp16 ? f(L32{}, L16{}) : f(L32{}, L32{});
        case 64: return lp16 ? f(std::integral_constant<int, 64>{}, L16{}) : f(std::integral_constant<int, 64>{}, L32{});
    }
    return cudaErrorInvalidValue;
}

// Persistent launch: one CTA per resident slot (SM count x occupancy); tiles are walked with a grid stride inside the
// kernel, which derives the tile map from the device-resident level table (no host read of spatial_shapes).
template <typename K>
int resident_ctas(K kernel) {
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, msda::kTiledThreads, 0) != cudaSuccess || per_sm < 1)
        per_sm = 1;
    return per_sm * num_sms();
}

// Slot order.  The 8x8-pixel patch order raises the forward's L1 hit rate and cuts L2 traffic, but the kernels are bound
// by the LSU's global-load issue rate, not by L1 misses, while partially filled border patches leave slots idle.  Linear
// order is therefore the default; MSDA_PATCHES=1 re-enables the patch order for experiments.
int allow_patches() {
    static const int v = env_flag("MSDA_PATCHES") == 1;
    return v;
}

// TMA staging of (x, y, a): linear slot order only, and every pair's tap run must start 16-byte aligned (L*P % 4 == 0).
// MSDA_NO_TMA=1 switches it off (A/B measurements).
bool use_tma_staging(const Dims &d) {
    static const bool off = env_flag("MSDA_NO_TMA") == 1;
    return !off && !allow_patches() && ((d.L * d.P) % 4 == 0);
}

// Small launches (decoder-style calls: a few thousand pairs) cannot hide the row-load latency with other warps; there the
// taps of each pair are split over the groups of a warp (template SPLIT).  MSDA_SPLIT=0/1 forces the choice (A/B).
bool use_split(unsigned npairs) {
    static const int force = env_flag("MSDA_SPLIT");
    if (force >= 0) return force == 1;
    // splitting is meant for decoder-sized launches (cfg2: 4 800 pairs), whose few pairs cannot hide the row-load latency
    // with other warps: launches with fewer than ~56 pairs per SM are split
    return npairs <= (unsigned)num_sms() * 56u;
}

constexpr int kFwdMinCtas = 4, kBwdMinCtas = 2;     // r01d sweep: fwd flat for 3..5, bwd best at 2 (128 regs, no spills)


template <typename T> struct FwdVec { static constexpr int v = 16 / sizeof(T); };      // 16-byte row slices
template <typename T> struct BwdVec { static constexpr int v = 4; };                  // 4 channels per lane (see RowVec)

// Launch of a kernel of kTiledThreads threads.  pdl: the kernel just issued on `st` is the programmatic-dependent-launch
// primary (the grad_value zero-fill, as zero_fill reported it, or the region backward's grad_value kernel): the kernel's
// prologue overlaps the primary, and the kernel must wait for it (pdl_wait_primary) before touching grad_value, or, the
// region tap kernel, before it exits.  Only the backward kernels that do so take `pdl`.
template <typename K, typename... Args>
cudaError_t launch_after_fill(K kern, int grid, size_t smem, cudaStream_t st, bool pdl, Args... args) {
    if (pdl) {
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
        const cudaError_t e = cudaLaunchKernelEx(&cfg, kern, args...);
        return e != cudaSuccess ? e : cudaGetLastError();
    }
    kern<<<grid, msda::kTiledThreads, smem, st>>>(args...);
    return cudaGetLastError();
}

// Persistent launch of a tiled kernel: one CTA per resident slot (cached per kernel and device), but no more CTAs than
// the linear order has tiles (the patch order has fewer, larger ones).
template <typename K, typename... Args>
cudaError_t launch_tiled(K kern, PerDevice<int> &slots, unsigned npairs, unsigned iter_pairs, bool pdl, cudaStream_t st,
                         Args... args) {
    const unsigned n = (unsigned)slots.get([&](int) { return resident_ctas(kern); });
    const unsigned tiles_ub = (npairs + iter_pairs - 1) / iter_pairs;
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return launch_after_fill(kern, (int)(tiles_ub < n ? tiles_ub : n), 0, st, pdl, args...);
}

template <typename T, int D, int LP_MAX, int VEC = FwdVec<T>::v>
cudaError_t launch_fwd(const T *value, const int64_t *shapes, const int64_t *lsi, const float *loc, const float *attn,
                       const Dims &d, T *out, cudaStream_t st) {
    using Shape = msda::TiledShape<VEC, D, LP_MAX, false>;
    constexpr bool kCanStage = (LP_MAX <= 16);          // per-warp double buffer must fit static shared memory
    constexpr bool kCanSplit = Shape::kCanSplit;
    constexpr bool kCanPack = sizeof(T) == 2 && VEC == 8;
    const unsigned npairs = num_pairs(d);
    const bool split = kCanSplit && use_split(npairs);
    const bool tma = !split && kCanStage && use_tma_staging(d);
    // bf16: packed-bf16 corner blend for the large (non-split) launches
    const bool packed = kCanPack && !split && knob(MSDA_KNOB_BF16_PACKED_FWD) == 1;
    static decltype(&msda::msda_fwd_tiled<T, VEC, D, LP_MAX, kFwdMinCtas, false, false>) const kern[] = {   // split, tma, ldg,
        msda::msda_fwd_tiled<T, VEC, D, LP_MAX, kFwdMinCtas, false, kCanSplit>,                          // packed tma / ldg
        msda::msda_fwd_tiled<T, VEC, D, LP_MAX, kFwdMinCtas, kCanStage, false>,
        msda::msda_fwd_tiled<T, VEC, D, LP_MAX, kFwdMinCtas, false, false>,
        msda::msda_fwd_tiled<T, VEC, D, LP_MAX, kFwdMinCtas, kCanStage, false, kCanPack>,
        msda::msda_fwd_tiled<T, VEC, D, LP_MAX, kFwdMinCtas, false, false, kCanPack>};
    static PerDevice<int> slots[5];
    const int k = split ? 0 : (packed ? 3 : 1) + (tma ? 0 : 1);
    return launch_tiled(kern[k], slots[k], npairs, split ? msda::TiledShape<VEC, D, LP_MAX, kCanSplit>::kIterPairs
                                                         : Shape::kIterPairs,
                        false, st, value, shapes, lsi, loc, attn, d.N, d.S, d.M, d.L, d.Lq, d.P, npairs, allow_patches(), out);
}

template <typename T, int D, int LP_MAX, int VEC = BwdVec<T>::v, bool NORED = false>
cudaError_t launch_bwd(const T *grad_out, const T *value, const int64_t *shapes, const int64_t *lsi, const float *loc,
                       const float *attn, const Dims &d, float *gv, float *gl, float *ga, bool pdl, cudaStream_t st) {
    using Shape = msda::TiledShape<VEC, D, LP_MAX, false>;
    constexpr bool kCanStage = (LP_MAX <= 16);
    constexpr bool kCanSplit = Shape::kCanSplit;
    const unsigned npairs = num_pairs(d);
    const bool split = kCanSplit && use_split(npairs);
    const bool tma = !split && kCanStage && use_tma_staging(d);
    static decltype(&msda::msda_bwd_tiled<T, VEC, D, LP_MAX, kBwdMinCtas, false, false, false, NORED>) const kern[] = {
        msda::msda_bwd_tiled<T, VEC, D, LP_MAX, kBwdMinCtas, false, kCanSplit, false, NORED>,          // split, tma, ldg
        msda::msda_bwd_tiled<T, VEC, D, LP_MAX, kBwdMinCtas, kCanStage, false, false, NORED>,
        msda::msda_bwd_tiled<T, VEC, D, LP_MAX, kBwdMinCtas, false, false, false, NORED>};
    static PerDevice<int> slots[3];
    const int k = split ? 0 : tma ? 1 : 2;
    return launch_tiled(kern[k], slots[k], npairs, split ? msda::TiledShape<VEC, D, LP_MAX, kCanSplit>::kIterPairs
                                                         : Shape::kIterPairs,
                        pdl, st, grad_out, value, shapes, lsi, loc, attn, d.N, d.S, d.M, d.L, d.Lq, d.P, npairs,
                        allow_patches(), gv, gl, ga, (__nv_bfloat16 *)nullptr, 0);
}

// ---- slab-ordered kernels (msda_slab.cuh): D = 32 and L*P <= 16 (every UNINEXT call) ------------------------------
// OPT-IN (MSDA_KNOB_SLAB = 1).  They halve L2 sectors, but the shared-memory traffic of the window (4 wavefronts per
// privatised row-add) lands on the same LSU data pipe that the gathers already keep busy, and they were slower than the
// tiled kernels where they were first measured.  MSDA_KNOB_SLAB = -1 (auto) therefore selects the tiled kernels.

bool use_slab(const Dims &d, const void *value, const void *out) {
    if (d.D != 32 || d.L * d.P > 16 || d.L > msda::kMaxLevels) return false;
    if ((reinterpret_cast<uintptr_t>(value) & 31u) || !aligned16(out)) return false;   // 32-byte row slices
    return knob(MSDA_KNOB_SLAB) == 1;
}

template <typename T>
cudaError_t launch_fwd_slab(const T *value, const int64_t *shapes, const int64_t *lsi, const float *loc, const float *attn,
                            const Dims &d, T *out, cudaStream_t st) {
    const int sms = num_sms();
    if (knob(MSDA_KNOB_FWD_SLAB_CTAS) == 1)
        return launch(msda::msda_fwd_slab<T, 16, 1>, sms, msda::kSlabThreads, 0, st, value, shapes, lsi, loc, attn, d.N,
                      d.S, d.M, d.L, d.Lq, d.P, sms, out);
    return launch(msda::msda_fwd_slab<T, 16, 2>, sms * 2, msda::kSlabThreads, 0, st, value, shapes, lsi, loc, attn, d.N,
                  d.S, d.M, d.L, d.Lq, d.P, sms, out);
}

// Shared-memory window of the slab and consumer-warp backward kernels, in rows of 128 B: the device's opt-in maximum
// minus the kernel's static part and the lists / g stash / tap slabs of `cap` entries per list
// (smem(rows, cap) - smem(0, cap)), clamped by the route's fit(rows).  Derived per device and again whenever a knob
// changes: the knob epoch it was derived at travels in the cached value (epoch << 32 | rows << 16 | cap).
struct Window { int rows, cap; };

template <auto Kernel, class Smem, class Fit>
cudaError_t bwd_window(int cap_max, Smem smem, Fit fit, Window &w) {
    static PerDevice<uint64_t> cache;
    const uint64_t epoch = (uint32_t)knobs().epoch.load(std::memory_order_acquire);
    cudaError_t e = cudaSuccess;
    const uint64_t v = cache.get([&](int dev) -> uint64_t {
        int cap = knob(MSDA_KNOB_BWD_LIST_CAP) & ~1;
        if (cap < 8) cap = 8;
        if (cap > cap_max) cap = cap_max;
        int max_optin = 0;
        cudaDeviceGetAttribute(&max_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
        cudaFuncAttributes fa{};
        cudaFuncGetAttributes(&fa, Kernel);
        const long long fixed = (long long)smem(0, cap) + (long long)fa.sharedSizeBytes + 64;
        int rows = fit((int)((max_optin - fixed) / 128));
        if (rows < 0) rows = 0;
        if ((e = opt_in_smem<Kernel>((int)smem(rows, cap))) != cudaSuccess) return 0;
        return epoch << 32 | (uint64_t)rows << 16 | (uint64_t)cap;     // a cap that fits is < 2^16 entries
    }, [&](uint64_t c) { return c >> 32 == epoch; });
    w = Window{(int)(v >> 16 & 0xffff), (int)(v & 0xffff)};
    return e;
}

template <typename T>
cudaError_t launch_bwd_slab(const T *grad_out, const T *value, const int64_t *shapes, const int64_t *lsi, const float *loc,
                            const float *attn, const Dims &d, float *gv, float *gl, float *ga, cudaStream_t st) {
    // MSDA_BWD_WIN_ROWS / MSDA_BWD_LIST_CAP override (sweeps).
    constexpr auto kern = msda::msda_bwd_slab<T, 16>;
    const auto smem = [](int rows, int cap) { return msda::bwd_slab_smem_bytes(rows, cap); };
    Window w;
    const cudaError_t e = bwd_window<kern>(1 << 30, smem, [](int rows) {
        const int want = knob(MSDA_KNOB_BWD_WIN_ROWS);
        return want >= 0 && want < rows ? want : rows;
    }, w);
    if (e != cudaSuccess) return e;
    const int sms = num_sms();
    return launch(kern, sms, msda::kSlabThreads, smem(w.rows, w.cap), st, grad_out, value, shapes, lsi, loc, attn, d.N,
                  d.S, d.M, d.L, d.Lq, d.P, sms, w.rows, w.cap, gv, gl, ga);
}

// bf16 backward with the fine levels accumulated in the bf16 result (msda_bwd_tiled MIXED): D = 32, L*P <= 16, large launches.
cudaError_t launch_bwd_mixed(const __nv_bfloat16 *go, const __nv_bfloat16 *value, const int64_t *shapes, const int64_t *lsi,
                             const float *loc, const float *attn, const Dims &d, float *scratch, __nv_bfloat16 *gv16,
                             float *gl, float *ga, int fine_min_rows, cudaStream_t st) {
    using T = __nv_bfloat16;
    constexpr int VEC = 4, DD = 32, LP_MAX = 16;
    const unsigned npairs = num_pairs(d);
    static decltype(&msda::msda_bwd_tiled<T, VEC, DD, LP_MAX, kBwdMinCtas, false, false, true>) const kern[] = {
        msda::msda_bwd_tiled<T, VEC, DD, LP_MAX, kBwdMinCtas, true, false, true>,                     // tma, ldg
        msda::msda_bwd_tiled<T, VEC, DD, LP_MAX, kBwdMinCtas, false, false, true>};
    static PerDevice<int> slots[2];
    const int k = use_tma_staging(d) ? 0 : 1;
    return launch_tiled(kern[k], slots[k], npairs, msda::TiledShape<VEC, DD, LP_MAX, false>::kIterPairs, false, st, go,
                        value, shapes, lsi, loc, attn, d.N, d.S, d.M, d.L, d.Lq, d.P, npairs, allow_patches(), scratch,
                        gl, ga, gv16, fine_min_rows);
}

// Backward with the coarse levels accumulated by dedicated consumer warps (msda_tmem.cuh): MSDA_KNOB_SLAB = 2.  Its window
// is rounded down to whole rows per consumer warp, and its lists hold at most 128 entries.
template <typename T>
cudaError_t launch_bwd_tmem(const T *grad_out, const T *value, const int64_t *shapes, const int64_t *lsi, const float *loc,
                            const float *attn, const Dims &d, float *gv, float *gl, float *ga, cudaStream_t st) {
    constexpr auto kern = msda::msda_bwd_tmem<T, 16>;
    const auto smem = [](int rows, int cap) { return msda::bwd_tmem_smem_bytes(cap, rows); };
    Window w;
    const cudaError_t e = bwd_window<kern>(128, smem, [](int rows) { return rows & ~(msda::kTmCons - 1); }, w);
    if (e != cudaSuccess) return e;
    const int sms = num_sms();
    return launch(kern, sms, msda::kTmThreads, smem(w.rows, w.cap), st, grad_out, value, shapes, lsi, loc, attn, d.N, d.S,
                  d.M, d.L, d.Lq, d.P, sms, w.cap, w.rows, gv, gl, ga);
}

// ---- region backward (msda_region.cuh): fp32 encoder self-attention, D = 32, L*P <= 16, Lq == S, large launches --------
// Auto-selected (MSDA_KNOB_REGION_BWD = -1); 0 keeps msda_bwd_tiled.
bool use_region(const Dims &d) {
    return knob(MSDA_KNOB_REGION_BWD) != 0 && d.D == 32 && d.L * d.P <= 16 && d.L <= msda::kMaxLevels && d.Lq == d.S &&
           !use_split(num_pairs(d));
}

// Two launches: the grad_value kernel, a PDL secondary of the zero-fill when `pdl`, then the tap kernel (grad_loc /
// grad_attn), a PDL secondary of the grad_value kernel whenever the stream is not capturing, so that its CTAs run beside
// the grad_value CTAs (msda_region.cuh: the chain is transitive).  Under capture the tap kernel follows in plain stream
// order.
cudaError_t launch_bwd_region(const float *go, const float *value, const int64_t *shapes, const int64_t *lsi,
                              const float *loc, const float *attn, const Dims &d, float *gv, float *gl, float *ga,
                              bool pdl, cudaStream_t st) {
    constexpr auto tap = msda::msda_bwd_region<msda::kRegionEdge, msda::kRegionHalo>;
    constexpr auto gvk = msda::msda_region_grad_value_pass<msda::kRegionEdge, msda::kRegionHalo>;
    constexpr size_t tap_smem = msda::region_tap_smem_bytes(), gv_smem = msda::region_gv_smem_bytes();
    static PerDevice<int> ready;
    static msda::RegionGrids grids[kMaxDevices];
    cudaError_t e = cudaSuccess;
    const int dev = current_device();
    ready.get([&](int dv) {
        if ((e = cudaFuncSetAttribute(gvk, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gv_smem)) != cudaSuccess)
            return 0;
        grids[dv] = msda::region_grids(gvk, gv_smem, tap, tap_smem, num_sms());
        return 1;
    });
    if (e != cudaSuccess) return e;
    const msda::RegionGrids &rg = grids[dev];
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    const bool chain = cudaStreamIsCapturing(st, &cap) == cudaSuccess && cap == cudaStreamCaptureStatusNone;
    const unsigned npairs = num_pairs(d);
    const int tma = use_tma_staging(d) ? 1 : 0;            // the tap pass: TMA-staged or __ldg taps, as msda_bwd_tiled
    g_launches.fetch_add(2, std::memory_order_relaxed);
    // Under capture the two kernels run one after the other, each at its own occupancy and unpadded.
    e = launch_after_fill(gvk, chain ? rg.gv : rg.gv_solo, chain ? rg.gv_smem : gv_smem, st, pdl, go, shapes, lsi, loc,
                          attn, d.N, d.S, d.M, d.L, d.Lq, d.P, npairs, gv);
    if (e != cudaSuccess) return e;
    return launch_after_fill(tap, chain ? rg.tap : rg.tap_solo, tap_smem, st, chain, go, value, shapes, lsi, loc, attn, d.N,
                             d.S, d.M, d.L, d.Lq, d.P, npairs, tma, gl, ga);
}

template <typename T>
cudaError_t fwd_fast(const T *value, const int64_t *shapes, const int64_t *lsi, const float *loc, const float *attn,
                     const Dims &d, T *out, cudaStream_t st) {
    if (use_slab(d, value, out)) return launch_fwd_slab<T>(value, shapes, lsi, loc, attn, d, out, st);
    if constexpr (sizeof(T) == 4) {           // fp32, 32-byte lanes: needs 32-byte aligned rows
        if (knob(MSDA_KNOB_F32_VEC8_FWD) == 1 && d.L * d.P <= 16 && (d.D == 32 || d.D == 64) &&
            !(reinterpret_cast<uintptr_t>(value) & 31u))
            return d.D == 32 ? launch_fwd<T, 32, 16, 8>(value, shapes, lsi, loc, attn, d, out, st)
                             : launch_fwd<T, 64, 16, 8>(value, shapes, lsi, loc, attn, d, out, st);
    }
    return route_tiled<T>(d, [&](auto D, auto LP) {
        return launch_fwd<T, decltype(D)::value, decltype(LP)::value>(value, shapes, lsi, loc, attn, d, out, st);
    });
}

// pdl: the zero-fill just issued is a PDL primary (zero_fill); only the routes whose kernels wait for it use it.
template <typename T>
cudaError_t bwd_fast(const T *go, const T *value, const int64_t *shapes, const int64_t *lsi, const float *loc,
                     const float *attn, const Dims &d, float *gv, float *gl, float *ga, bool pdl, cudaStream_t st) {
    const int LP = d.L * d.P;
    if (knob(MSDA_KNOB_SLAB) == 2 && d.D == 32 && LP <= 16 && d.L <= msda::kMaxLevels)
        return launch_bwd_tmem<T>(go, value, shapes, lsi, loc, attn, d, gv, gl, ga, st);
    if (use_slab(d, value, gv)) return launch_bwd_slab<T>(go, value, shapes, lsi, loc, attn, d, gv, gl, ga, st);
    if constexpr (sizeof(T) == 4) {
        if (knob(MSDA_KNOB_F32_VEC8_BWD) == 1 && LP <= 16 && d.D == 32 &&
            !((reinterpret_cast<uintptr_t>(value) | reinterpret_cast<uintptr_t>(go)) & 31u))
            return launch_bwd<T, 32, 16, 8>(go, value, shapes, lsi, loc, attn, d, gv, gl, ga, pdl, st);
        if (use_region(d)) return launch_bwd_region(go, value, shapes, lsi, loc, attn, d, gv, gl, ga, pdl, st);
    }
    return route_tiled<T>(d, [&](auto D, auto LPM) {
        return launch_bwd<T, decltype(D)::value, decltype(LPM)::value>(go, value, shapes, lsi, loc, attn, d, gv, gl, ga,
                                                                       pdl, st);
    });
}

template <typename T, typename TL>
cudaError_t fwd_generic(const T *value, const int64_t *shapes, const int64_t *lsi, const TL *loc, const TL *attn,
                        const Dims &d, T *out, cudaStream_t st) {
    const long long total = (long long)d.N * d.Lq * d.M * d.D;
    return launch(msda::msda_fwd_generic<T, TL>, capped_grid(total, 256, 32), 256, 0, st, value, shapes, lsi, loc, attn,
                  d.S, d.M, d.D, d.L, d.Lq, d.P, total, out);
}

template <typename T, typename TL, typename GA, bool NORED = false>
cudaError_t bwd_generic(const T *go, const T *value, const int64_t *shapes, const int64_t *lsi, const TL *loc,
                        const TL *attn, const Dims &d, GA *gv, TL *gl, TL *ga, cudaStream_t st) {
    const long long npairs = (long long)d.N * d.Lq * d.M;
    int threads = ((d.D + 31) / 32) * 32;
    if (threads > 256) threads = 256;
    return launch(msda::msda_bwd_generic<T, TL, GA, NORED>, capped_grid(npairs, 1, 64), threads, 0, st, go, value, shapes,
                  lsi, loc, attn, d.S, d.M, d.D, d.L, d.Lq, d.P, npairs, gv, gl, ga);
}

// The bf16 result of the bf16 backward: one rounding of its fp32 accumulator.
cudaError_t round_to_bf16(const float *gv32, uint16_t *gv, size_t nval, cudaStream_t st) {
    return launch(msda::msda_f32_to_bf16, capped_grid((long long)nval, 256, 16), 256, 0, st, gv32,
                  reinterpret_cast<__nv_bfloat16 *>(gv), (long long)nval);
}

// The tensors' element type behind an ABI pointer type: bf16 is passed as uint16_t.
template <class A> struct Elem { using type = A; };
template <> struct Elem<uint16_t> { using type = __nv_bfloat16; };

// Null pointers are argument errors.  Alignment is a ROUTING property: the tiled / slab kernels need 16-byte aligned
// tensors (vector loads, vector reds); anything else -- e.g. a contiguous view with a storage offset, which the
// reference accepts -- runs on the generic scalar kernels (natural alignment only).
#define MSDA_CHECK_PTRS(ALIGNED, ...)                                    \
    bool ALIGNED = true;                                                 \
    do {                                                                 \
        const void *ptrs_[] = {__VA_ARGS__};                             \
        for (const void *p_ : ptrs_) {                                   \
            if (p_ == nullptr) return MSDA_E_BADARG;                     \
            ALIGNED = ALIGNED && aligned16(p_);                          \
        }                                                                \
    } while (0)

// The forward of every dtype.  fp64 never takes the tiled kernels.
template <class A, class TL>
int forward(const A *value, const int64_t *shapes, const int64_t *lsi, const TL *loc, const TL *attn, const Dims &d, A *out,
            void *stream) {
    using T = typename Elem<A>::type;
    if (int e = check_dims(d)) return e;
    MSDA_CHECK_PTRS(al, value, loc, attn, out);
    if (!shapes || !lsi) return MSDA_E_BADARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const T *v = reinterpret_cast<const T *>(value);
    T *o = reinterpret_cast<T *>(out);
    if constexpr (sizeof(T) != 8)
        if (al && use_fast(sizeof(T), d)) return (int)fwd_fast<T>(v, shapes, lsi, loc, attn, d, o, st);
    return (int)fwd_generic<T, TL>(v, shapes, lsi, loc, attn, d, o, st);
}

// bf16 backward, mixed accumulation: bf16 result zero-filled (fine levels add into it), fp32 scratch zero-filled for the
// coarse levels only, one rounding pass over the coarse rows at the end -- no full-size fp32 round trip.
int backward_mixed(const __nv_bfloat16 *go, const __nv_bfloat16 *v, const int64_t *shapes, const int64_t *lsi,
                   const float *loc, const float *attn, const Dims &d, float *gv32, uint16_t *gv, float *gl, float *ga,
                   int fine_rows, cudaStream_t st) {
    __nv_bfloat16 *gv16 = reinterpret_cast<__nv_bfloat16 *>(gv);
    cudaError_t e = zero_fill(gv, sizeof(uint16_t) * (size_t)d.N * d.S * d.M * d.D, st);
    if (e != cudaSuccess) return (int)e;
    const dim3 hgrid((unsigned)(num_sms() * 2 / d.N + 1), (unsigned)d.N);
    if ((e = launch(msda::msda_coarse_rows<false>, hgrid, 256, 0, st, gv32, gv16, shapes, lsi, d.L, d.S, d.M * d.D,
                    fine_rows)) != cudaSuccess)
        return (int)e;
    e = launch_bwd_mixed(go, v, shapes, lsi, loc, attn, d, gv32, gv16, gl, ga, fine_rows, st);
    if (e != cudaSuccess) return (int)e;
    return (int)launch(msda::msda_coarse_rows<true>, hgrid, 256, 0, st, gv32, gv16, shapes, lsi, d.L, d.S, d.M * d.D,
                       fine_rows);
}

// The backward of every dtype.  gv accumulates grad_value in the compute type; bf16 also rounds it into gv16 when given.
template <class A, class TL, class C>
int backward(const A *grad_out, const A *value, const int64_t *shapes, const int64_t *lsi, const TL *loc, const TL *attn,
             const Dims &d, C *gv, uint16_t *gv16, TL *gl, TL *ga, void *stream) {
    using T = typename Elem<A>::type;
    if (int e = check_dims(d)) return e;
    MSDA_CHECK_PTRS(al, grad_out, value, loc, attn, gv, gl, ga);
    if (!shapes || !lsi) return MSDA_E_BADARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t nval = (size_t)d.N * d.S * d.M * d.D;
    const T *go = reinterpret_cast<const T *>(grad_out), *v = reinterpret_cast<const T *>(value);
    const bool fast = al && use_fast(sizeof(T), d);
    if constexpr (sizeof(T) == 2) {
        const int fine_rows = knob(MSDA_KNOB_BF16_FINE_ROWS);
        if (fine_rows > 0 && gv16 != nullptr && fast && d.D == 32 && d.L * d.P <= 16 && !use_split(num_pairs(d)) &&
            aligned16(gv16))
            return backward_mixed(go, v, shapes, lsi, loc, attn, d, gv, gv16, gl, ga, fine_rows, st);
    }
    bool pdl = false;
    cudaError_t err = zero_fill(gv, sizeof(C) * nval, st, sizeof(T) != 8 ? &pdl : nullptr);
    if (err != cudaSuccess) return (int)err;
    if constexpr (sizeof(T) != 8) {
        if (fast) err = bwd_fast<T>(go, v, shapes, lsi, loc, attn, d, gv, gl, ga, pdl, st);
    }
    if (!fast) err = bwd_generic<T, TL, C>(go, v, shapes, lsi, loc, attn, d, gv, gl, ga, st);
    if constexpr (sizeof(T) == 2) {
        if (err == cudaSuccess && gv16 != nullptr) err = round_to_bf16(gv, gv16, nval, st);
    }
    return (int)err;
}


// ---- deterministic backward (msda_det.cuh) ------------------------------------------------------------------------
// Workspace of one chunk of nq queries (n = nq*M*L*P*4 entries): sort keys and values in and out (4 x n x 4 bytes), the
// segment starts (M*S + 1 words), the row counter of the accumulate step and CUB's temporary storage, each 256-byte aligned.
struct DetLayout { size_t keys_in, keys_out, vals_in, vals_out, start, counter, temp, temp_bytes, total; unsigned n; };

int det_end_bit(const Dims &d) {                   // bits of the largest key, the sentinel M*S
    const unsigned long long top = (unsigned long long)d.M * d.S;
    int bits = 0;
    while (bits < 32 && (top >> bits) != 0) ++bits;
    return bits;
}

int det_layout(const Dims &d, long long nq, DetLayout &lay) {
    const unsigned long long n = (unsigned long long)nq * d.M * d.L * d.P * 4;
    if (n > 0xffffffffull) return MSDA_E_TOOLARGE;
    lay.n = (unsigned)n;
    size_t off = 0;
    auto take = [&](size_t bytes) { const size_t at = off; off += align256(bytes); return at; };
    lay.keys_in = take(4 * n);
    lay.keys_out = take(4 * n);
    lay.vals_in = take(4 * n);
    lay.vals_out = take(4 * n);
    lay.start = take(4 * ((size_t)d.M * d.S + 1));
    lay.counter = take(4);
    lay.temp_bytes = 0;
    const cudaError_t e = msda::det_sort(nullptr, lay.temp_bytes, nullptr, nullptr, nullptr, nullptr, lay.n, det_end_bit(d), 0);
    if (e != cudaSuccess) return (int)e;
    lay.temp = take(lay.temp_bytes);
    lay.total = off;
    return 0;
}

int det_check(const Dims &d) {
    if (int e = check_dims(d)) return e;
    if ((unsigned long long)d.M * d.S + 1 > (1ull << 32)) return MSDA_E_TOOLARGE;     // keys and the sentinel are 32-bit
    return 0;
}

// grad_loc / grad_attn: the kernel the default route picks (the region kernel's are bit-identical to msda_bwd_tiled's),
// with its grad_value reds compiled out.
template <typename T, typename TL, typename GA>
cudaError_t det_loc_attn(const T *go, const T *value, const int64_t *shapes, const int64_t *lsi, const TL *loc,
                         const TL *attn, const Dims &d, bool fast, GA *gv, TL *gl, TL *ga, cudaStream_t st) {
    if constexpr (sizeof(T) != 8) {
        if (fast)
            return route_tiled<T>(d, [&](auto D, auto LP) {
                return launch_bwd<T, decltype(D)::value, decltype(LP)::value, 4, true>(go, value, shapes, lsi, loc, attn, d,
                                                                                       gv, gl, ga, false, st);
            });
    }
    return bwd_generic<T, TL, GA, true>(go, value, shapes, lsi, loc, attn, d, gv, gl, ga, st);
}

// The whole deterministic backward into the zero-filled accumulator gv (compute type of T).  `fast`: the default route
// would take the tiled kernels (16-byte aligned tensors, fast-path shape).
template <typename T, typename TL>
int det_backward(const T *go, const T *value, const int64_t *shapes, const int64_t *lsi, const TL *loc, const TL *attn,
                 const Dims &d, bool fast, typename msda::Num<T>::C *gv, TL *gl, TL *ga, void *ws, int64_t ws_bytes,
                 cudaStream_t st) {
    using C = typename msda::Num<T>::C;
    if (ws == nullptr || ws_bytes <= 0) return MSDA_E_BADARG;
    DetLayout lay{};
    if (int e = det_layout(d, 1, lay)) return e;
    if ((long long)lay.total > ws_bytes) return MSDA_E_BADARG;           // one query does not fit
    long long lo = 1, hi = d.Lq;                                         // largest chunk that fits
    while (lo < hi) {
        const long long mid = hi - (hi - lo) / 2;
        DetLayout t{};
        const int e = det_layout(d, mid, t);
        if (e == 0 && (long long)t.total <= ws_bytes) lo = mid; else if (e != 0 && e != MSDA_E_TOOLARGE) return e; else hi = mid - 1;
    }
    const long long chunk = lo;
    cudaError_t err = cudaMemsetAsync(gv, 0, sizeof(C) * (size_t)d.N * d.S * d.M * d.D, st);
    if (err != cudaSuccess) return (int)err;
    err = det_loc_attn<T, TL, C>(go, value, shapes, lsi, loc, attn, d, fast, gv, gl, ga, st);
    if (err != cudaSuccess) return (int)err;

    unsigned char *w = static_cast<unsigned char *>(ws);
    const int end_bit = det_end_bit(d);
    const unsigned nkeys = (unsigned)d.M * (unsigned)d.S;
    const bool v4 = sizeof(T) != 8 && d.D == 32 && fast;
    const int sms = num_sms();
    const int LP = d.L * d.P;
    for (int b = 0; b < d.N; ++b) {
        for (long long q0 = 0; q0 < d.Lq; q0 += chunk) {
            const long long nq = q0 + chunk <= d.Lq ? chunk : d.Lq - q0;
            if (int e = det_layout(d, nq, lay)) return e;
            unsigned *keys_in = reinterpret_cast<unsigned *>(w + lay.keys_in), *keys_out = reinterpret_cast<unsigned *>(w + lay.keys_out);
            unsigned *vals_in = reinterpret_cast<unsigned *>(w + lay.vals_in), *vals_out = reinterpret_cast<unsigned *>(w + lay.vals_out);
            unsigned *start = reinterpret_cast<unsigned *>(w + lay.start), *counter = reinterpret_cast<unsigned *>(w + lay.counter);
            const long long tap0 = ((long long)b * d.Lq + q0) * d.M * LP;
            const T *go_chunk = go + ((size_t)b * d.Lq + q0) * d.M * d.D;
            msda::msda_det_keys<TL><<<capped_grid(lay.n, msda::kDetThreads, 16), msda::kDetThreads, 0, st>>>(
                loc, shapes, lsi, d.S, d.M, d.L, d.P, tap0, lay.n, keys_in, vals_in);
            if ((err = cudaGetLastError()) != cudaSuccess) return (int)err;
            size_t temp_bytes = lay.temp_bytes;
            err = msda::det_sort(w + lay.temp, temp_bytes, keys_in, keys_out, vals_in, vals_out, lay.n, end_bit, st);
            if (err != cudaSuccess) return (int)err;
            msda::msda_det_bounds<<<capped_grid((long long)nkeys + 1, msda::kDetThreads, 16), msda::kDetThreads, 0, st>>>(
                keys_out, lay.n, nkeys, start);
            if ((err = cudaGetLastError()) != cudaSuccess) return (int)err;
            if ((err = cudaMemsetAsync(counter, 0, 4, st)) != cudaSuccess) return (int)err;
            if constexpr (sizeof(T) != 8) {
                if (v4) {
                    msda::msda_det_accumulate_v4<T><<<sms * 8, msda::kDetThreads, 0, st>>>(
                        go_chunk, loc, attn, shapes, d.S, d.M, d.L, d.P, tap0, b, start, vals_out, counter, gv);
                }
            }
            if (!v4)
                msda::msda_det_accumulate<T, TL><<<sms * 8, msda::kDetThreads, 0, st>>>(
                    go_chunk, loc, attn, shapes, d.S, d.M, d.D, d.L, d.P, tap0, b, start, vals_out, counter, gv);
            if ((err = cudaGetLastError()) != cudaSuccess) return (int)err;
            g_launches.fetch_add(4, std::memory_order_relaxed);       // keys, sort (counted once), bounds, accumulate
        }
    }
    return 0;
}

// The deterministic backward of every dtype: argument checks, then det_backward; bf16 also rounds into gv16 when given.
template <class A, class TL, class C>
int det_entry(const A *grad_out, const A *value, const int64_t *shapes, const int64_t *lsi, const TL *loc, const TL *attn,
              const Dims &d, C *gv, uint16_t *gv16, TL *gl, TL *ga, void *ws, int64_t ws_bytes, void *stream) {
    using T = typename Elem<A>::type;
    if (int e = det_check(d)) return e;
    MSDA_CHECK_PTRS(al, grad_out, value, loc, attn, gv, gl, ga);
    if (!shapes || !lsi) return MSDA_E_BADARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int e = det_backward<T, TL>(reinterpret_cast<const T *>(grad_out), reinterpret_cast<const T *>(value), shapes,
                                      lsi, loc, attn, d, al && use_fast(sizeof(T), d), gv, gl, ga, ws, ws_bytes, st);
    if constexpr (sizeof(T) == 2) {
        if (e == 0 && gv16 != nullptr) return (int)round_to_bf16(gv, gv16, (size_t)d.N * d.S * d.M * d.D, st);
    }
    return e;
}

}  // namespace

extern "C" {

int msda_abi_version(void) { return MSDA_ABI_VERSION; }

const char *msda_strerror(int code) {
    if (code == 0) return "success";
    if (code == MSDA_E_BADARG) return "msda: bad argument (null pointer, non-positive dimension or unknown knob)";
    if (code == MSDA_E_TOOLARGE) return "msda: problem too large for the kernel index types";
    if (code == MSDA_E_NODEVICE) return "msda: no CUDA device";
    if (code > 0) return cudaGetErrorString(static_cast<cudaError_t>(code));
    return "msda: unknown error";
}

int msda_uses_fast_path(int dtype_bytes, int D, int L, int P) { return fast_ok(dtype_bytes, D, L, P) ? 1 : 0; }

uint64_t msda_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

int msda_set_knob(int k, int value) {
    if (k < 0 || k >= MSDA_KNOB_COUNT) return MSDA_E_BADARG;
    Knobs &kn = knobs();
    if (value == MSDA_KNOB_QUERY) return kn.v[k].load(std::memory_order_relaxed);
    const int old = kn.v[k].exchange(value, std::memory_order_relaxed);
    kn.epoch.fetch_add(1, std::memory_order_release);
    return old;
}

int msda_forward_f32(const float *value, const int64_t *spatial_shapes, const int64_t *level_start_index,
                     const float *sampling_loc, const float *attn_weight, int N, int S, int M, int D, int L, int Lq,
                     int P, float *out, void *stream) {
    return forward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, {N, S, M, D, L, Lq, P}, out, stream);
}

int msda_forward_f64(const double *value, const int64_t *spatial_shapes, const int64_t *level_start_index,
                     const double *sampling_loc, const double *attn_weight, int N, int S, int M, int D, int L, int Lq,
                     int P, double *out, void *stream) {
    return forward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, {N, S, M, D, L, Lq, P}, out, stream);
}

int msda_forward_bf16(const uint16_t *value, const int64_t *spatial_shapes, const int64_t *level_start_index,
                      const float *sampling_loc, const float *attn_weight, int N, int S, int M, int D, int L, int Lq,
                      int P, uint16_t *out, void *stream) {
    return forward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, {N, S, M, D, L, Lq, P}, out, stream);
}

int msda_backward_f32(const float *grad_out, const float *value, const int64_t *spatial_shapes,
                      const int64_t *level_start_index, const float *sampling_loc, const float *attn_weight, int N,
                      int S, int M, int D, int L, int Lq, int P, float *grad_value, float *grad_sampling_loc,
                      float *grad_attn_weight, void *stream) {
    return backward(grad_out, value, spatial_shapes, level_start_index, sampling_loc, attn_weight, {N, S, M, D, L, Lq, P},
                    grad_value, nullptr, grad_sampling_loc, grad_attn_weight, stream);
}

int msda_backward_f64(const double *grad_out, const double *value, const int64_t *spatial_shapes,
                      const int64_t *level_start_index, const double *sampling_loc, const double *attn_weight, int N,
                      int S, int M, int D, int L, int Lq, int P, double *grad_value, double *grad_sampling_loc,
                      double *grad_attn_weight, void *stream) {
    return backward(grad_out, value, spatial_shapes, level_start_index, sampling_loc, attn_weight, {N, S, M, D, L, Lq, P},
                    grad_value, nullptr, grad_sampling_loc, grad_attn_weight, stream);
}

int msda_backward_bf16(const uint16_t *grad_out, const uint16_t *value, const int64_t *spatial_shapes,
                       const int64_t *level_start_index, const float *sampling_loc, const float *attn_weight, int N,
                       int S, int M, int D, int L, int Lq, int P, float *grad_value_f32, uint16_t *grad_value,
                       float *grad_sampling_loc, float *grad_attn_weight, void *stream) {
    return backward(grad_out, value, spatial_shapes, level_start_index, sampling_loc, attn_weight, {N, S, M, D, L, Lq, P},
                    grad_value_f32, grad_value, grad_sampling_loc, grad_attn_weight, stream);
}

int msda_backward_det_workspace(int dtype_bytes, int N, int S, int M, int D, int L, int Lq, int P, int chunk_queries,
                                int64_t *bytes) {
    const Dims d{N, S, M, D, L, Lq, P};
    if (dtype_bytes != 2 && dtype_bytes != 4 && dtype_bytes != 8) return MSDA_E_BADARG;
    if (!bytes || chunk_queries <= 0) return MSDA_E_BADARG;
    if (int e = det_check(d)) return e;
    DetLayout lay{};
    if (int e = det_layout(d, chunk_queries < Lq ? chunk_queries : Lq, lay)) return e;
    *bytes = (int64_t)lay.total;
    return 0;
}

int msda_backward_det_f32(const float *grad_out, const float *value, const int64_t *spatial_shapes,
                          const int64_t *level_start_index, const float *sampling_loc, const float *attn_weight, int N,
                          int S, int M, int D, int L, int Lq, int P, float *grad_value, float *grad_sampling_loc,
                          float *grad_attn_weight, void *workspace, int64_t workspace_bytes, void *stream) {
    return det_entry(grad_out, value, spatial_shapes, level_start_index, sampling_loc, attn_weight, {N, S, M, D, L, Lq, P},
                     grad_value, nullptr, grad_sampling_loc, grad_attn_weight, workspace, workspace_bytes, stream);
}

int msda_backward_det_f64(const double *grad_out, const double *value, const int64_t *spatial_shapes,
                          const int64_t *level_start_index, const double *sampling_loc, const double *attn_weight, int N,
                          int S, int M, int D, int L, int Lq, int P, double *grad_value, double *grad_sampling_loc,
                          double *grad_attn_weight, void *workspace, int64_t workspace_bytes, void *stream) {
    return det_entry(grad_out, value, spatial_shapes, level_start_index, sampling_loc, attn_weight, {N, S, M, D, L, Lq, P},
                     grad_value, nullptr, grad_sampling_loc, grad_attn_weight, workspace, workspace_bytes, stream);
}

int msda_backward_det_bf16(const uint16_t *grad_out, const uint16_t *value, const int64_t *spatial_shapes,
                           const int64_t *level_start_index, const float *sampling_loc, const float *attn_weight, int N,
                           int S, int M, int D, int L, int Lq, int P, float *grad_value_f32, uint16_t *grad_value,
                           float *grad_sampling_loc, float *grad_attn_weight, void *workspace, int64_t workspace_bytes,
                           void *stream) {
    return det_entry(grad_out, value, spatial_shapes, level_start_index, sampling_loc, attn_weight, {N, S, M, D, L, Lq, P},
                     grad_value_f32, grad_value, grad_sampling_loc, grad_attn_weight, workspace, workspace_bytes, stream);
}

}  // extern "C"
