// msda_cabi.cu -- the C ABI declared in include/msda_b200.h: argument checks, kernel routing, launches.
// Replaces the reference host wrappers ms_deform_attn_cuda_forward/backward (ops/src/cuda/ms_deform_attn_cuda.cu)
// and launchers ms_deformable_im2col_cuda / ms_deformable_col2im_cuda (ms_deform_im2col_cuda.cuh:923-954,956-1327).
#include <atomic>
#include <cstdio>
#include <cstdlib>

#include "../../include/msda_b200.h"
#include "msda_condinst.cuh"
#include "msda_det.cuh"
#include "msda_detpost.cuh"
#include "msda_generic.cuh"
#include "msda_maskpaste.cuh"
#include "msda_maskrle.cuh"
#include "msda_module.cuh"
#include "msda_region.cuh"
#include "msda_slab.cuh"
#include "msda_tmem.cuh"
#include "msda_tiled.cuh"
#include "msda_vlfuse.cuh"
#include "msda_vlfuse_tc.cuh"

namespace {

std::atomic<uint64_t> g_launches{0};

struct Dims { int N, S, M, D, L, Lq, P; };

inline bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
inline bool aligned8(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 7u) == 0; }

int check_dims(const Dims &d) {
    if (d.N <= 0 || d.S <= 0 || d.M <= 0 || d.D <= 0 || d.L <= 0 || d.Lq <= 0 || d.P <= 0) return MSDA_E_BADARG;
    // rows are indexed with int32 inside a batch element; tap counts with int64 everywhere.
    if ((long long)d.S >= (1ll << 30)) return MSDA_E_TOOLARGE;
    if ((long long)d.N * d.Lq * d.M >= (1ll << 40)) return MSDA_E_TOOLARGE;
    return 0;
}

// Per-device caches (a process may drive several GPUs: SM counts, occupancy and function attributes are per device).
constexpr int kMaxDevices = 64;

int current_device() {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) dev = 0;
    return dev;
}

int num_sms() {
    static std::atomic<int> sms[kMaxDevices];
    const int dev = current_device();
    int v = sms[dev].load(std::memory_order_relaxed);
    if (v == 0) {
        if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;
        sms[dev].store(v, std::memory_order_relaxed);
    }
    return v;
}

int env_int(const char *name, int dflt) {
    const char *e = getenv(name);
    return (e && e[0]) ? atoi(e) : dflt;
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

// Set by msda_backward_* when the zero-fill just issued on the stream may be the PDL primary of the next launch; consumed
// (and cleared) by launch_after_fill, cleared by msda_backward_* on every other route.  Only kernels that wait for the
// primary (pdl_wait_primary) before touching grad_value may be launched through launch_after_fill.
thread_local bool t_pdl_next = false;

// Zero-fill of grad_value before the backward kernels (MSDA_KNOB_ZERO_FILL).  *pdl is set when the fill went out as a
// kernel that the NEXT launch on `st` may take as its programmatic-dependent-launch primary.  The fill kernel stands in
// for a memset and is not counted by msda_launch_count().
cudaError_t zero_fill(void *p, size_t bytes, cudaStream_t st, bool *pdl = nullptr) {
    if (pdl) *pdl = false;
    const int mode = knob(MSDA_KNOB_ZERO_FILL);
    if (mode <= 0 || bytes < (1u << 16) || !aligned16(p) || (bytes & 15u)) return cudaMemsetAsync(p, 0, bytes, st);
    const unsigned long long n16 = bytes >> 4;
    unsigned long long blocks = (n16 + 255) / 256;
    const unsigned long long wave = (unsigned long long)num_sms() * 8;       // 8 x 256 threads = every thread slot of an SM
    if (blocks > wave) blocks = wave;
    msda::msda_zero_fill<<<(unsigned)blocks, 256, 0, st>>>(static_cast<uint4 *>(p), n16);
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

// Persistent launch: one CTA per resident slot (SM count x occupancy); tiles are walked with a grid stride inside the
// kernel, which derives the tile map from the device-resident level table (no host read of spatial_shapes).
template <typename K>
int resident_ctas(K kernel) {
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, msda::kTiledThreads, 0) != cudaSuccess || per_sm < 1)
        per_sm = 1;
    return per_sm * num_sms();
}

// resident_ctas() cached per (kernel instantiation, device)
template <typename K>
int resident_ctas_cached(K kernel, std::atomic<int> (&cache)[kMaxDevices]) {
    const int dev = current_device();
    int v = cache[dev].load(std::memory_order_relaxed);
    if (v == 0) { v = resident_ctas(kernel); cache[dev].store(v, std::memory_order_relaxed); }
    return v;
}

// Slot order.  The 8x8-pixel patch order raises the forward's L1 hit rate and cuts L2 traffic, but the kernels are bound
// by the LSU's global-load issue rate, not by L1 misses, while partially filled border patches leave slots idle.  Linear
// order is therefore the default; MSDA_PATCHES=1 re-enables the patch order for experiments.
int allow_patches() {
    static int v = -1;
    if (v < 0) { const char *e = getenv("MSDA_PATCHES"); v = (e && e[0] == '1') ? 1 : 0; }
    return v;
}

// TMA staging of (x, y, a): linear slot order only, and every pair's tap run must start 16-byte aligned (L*P % 4 == 0).
// MSDA_NO_TMA=1 switches it off (A/B measurements).
bool use_tma_staging(const Dims &d) {
    static int off = -1;
    if (off < 0) { const char *e = getenv("MSDA_NO_TMA"); off = (e && e[0] == '1') ? 1 : 0; }
    return !off && !allow_patches() && ((d.L * d.P) % 4 == 0);
}

// Small launches (decoder-style calls: a few thousand pairs) cannot hide the row-load latency with other warps; there the
// taps of each pair are split over the groups of a warp (template SPLIT).  MSDA_SPLIT=0/1 forces the choice (A/B).
bool use_split(unsigned npairs) {
    static int force = -2;
    if (force == -2) { const char *e = getenv("MSDA_SPLIT"); force = (e && (e[0] == '0' || e[0] == '1')) ? e[0] - '0' : -1; }
    if (force >= 0) return force == 1;
    // splitting is meant for decoder-sized launches (cfg2: 4 800 pairs), whose few pairs cannot hide the row-load latency
    // with other warps: launches with fewer than ~56 pairs per SM are split
    return npairs <= (unsigned)num_sms() * 56u;
}

constexpr int kFwdMinCtas = 4, kBwdMinCtas = 2;     // r01d sweep: fwd flat for 3..5, bwd best at 2 (128 regs, no spills)


template <typename T> struct FwdVec { static constexpr int v = 16 / sizeof(T); };      // 16-byte row slices
template <typename T> struct BwdVec { static constexpr int v = 4; };                  // 4 channels per lane (see RowVec)

// Launch of a backward kernel right after the grad_value zero-fill.  When msda_backward_* left t_pdl_next set, the fill
// kernel just issued on `st` is the programmatic-dependent-launch primary: the backward kernel's prologue overlaps it and
// the kernel waits for it (pdl_wait_primary) before its first red.
template <typename K, typename... Args>
cudaError_t launch_after_fill(K kern, int grid, size_t smem, cudaStream_t st, Args... args) {
    const bool pdl = t_pdl_next;
    t_pdl_next = false;
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

// Persistent launch of a tiled kernel: one CTA per resident slot, but no more CTAs than the linear order has tiles (the
// patch order has fewer, larger ones).  after_fill: the launch follows the grad_value zero-fill and honours the PDL
// pairing with it (launch_after_fill); every other launch is a plain one and leaves t_pdl_next alone.
template <typename K, typename... Args>
cudaError_t launch_tiled(K kern, std::atomic<int> (&cache)[kMaxDevices], unsigned npairs, unsigned iter_pairs,
                         bool after_fill, cudaStream_t st, Args... args) {
    const unsigned slots = (unsigned)resident_ctas_cached(kern, cache);
    const unsigned tiles_ub = (npairs + iter_pairs - 1) / iter_pairs;
    const int grid = (int)(tiles_ub < slots ? tiles_ub : slots);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    if (after_fill) return launch_after_fill(kern, grid, 0, st, args...);
    kern<<<grid, msda::kTiledThreads, 0, st>>>(args...);
    return cudaGetLastError();
}

template <typename T, int D, int LP_MAX, int VEC = FwdVec<T>::v>
cudaError_t launch_fwd(const T *value, const int64_t *shapes, const int64_t *lsi, const float *loc, const float *attn,
                       const Dims &d, T *out, cudaStream_t st) {
    using Shape = msda::TiledShape<VEC, D, LP_MAX, false>;
    constexpr bool kCanStage = (LP_MAX <= 16);          // per-warp double buffer must fit static shared memory
    constexpr bool kCanSplit = Shape::kCanSplit;
    constexpr bool kCanPack = sizeof(T) == 2 && VEC == 8;
    const unsigned npairs = (unsigned)((long long)d.N * d.Lq * d.M);
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
    static std::atomic<int> cache[5][kMaxDevices];
    const int k = split ? 0 : (packed ? 3 : 1) + (tma ? 0 : 1);
    return launch_tiled(kern[k], cache[k], npairs, split ? msda::TiledShape<VEC, D, LP_MAX, kCanSplit>::kIterPairs
                                                         : Shape::kIterPairs,
                        false, st, value, shapes, lsi, loc, attn, d.N, d.S, d.M, d.L, d.Lq, d.P, npairs, allow_patches(), out);
}

template <typename T, int D, int LP_MAX, int VEC = BwdVec<T>::v, bool NORED = false>
cudaError_t launch_bwd(const T *grad_out, const T *value, const int64_t *shapes, const int64_t *lsi, const float *loc,
                       const float *attn, const Dims &d, float *gv, float *gl, float *ga, cudaStream_t st) {
    using Shape = msda::TiledShape<VEC, D, LP_MAX, false>;
    constexpr bool kCanStage = (LP_MAX <= 16);
    constexpr bool kCanSplit = Shape::kCanSplit;
    const unsigned npairs = (unsigned)((long long)d.N * d.Lq * d.M);
    const bool split = kCanSplit && use_split(npairs);
    const bool tma = !split && kCanStage && use_tma_staging(d);
    static decltype(&msda::msda_bwd_tiled<T, VEC, D, LP_MAX, kBwdMinCtas, false, false, false, NORED>) const kern[] = {
        msda::msda_bwd_tiled<T, VEC, D, LP_MAX, kBwdMinCtas, false, kCanSplit, false, NORED>,          // split, tma, ldg
        msda::msda_bwd_tiled<T, VEC, D, LP_MAX, kBwdMinCtas, kCanStage, false, false, NORED>,
        msda::msda_bwd_tiled<T, VEC, D, LP_MAX, kBwdMinCtas, false, false, false, NORED>};
    static std::atomic<int> cache[3][kMaxDevices];
    const int k = split ? 0 : tma ? 1 : 2;
    return launch_tiled(kern[k], cache[k], npairs, split ? msda::TiledShape<VEC, D, LP_MAX, kCanSplit>::kIterPairs
                                                         : Shape::kIterPairs,
                        true, st, grad_out, value, shapes, lsi, loc, attn, d.N, d.S, d.M, d.L, d.Lq, d.P, npairs,
                        allow_patches(), gv, gl, ga, (__nv_bfloat16 *)nullptr, 0);
}

// ---- slab-ordered kernels (msda_slab.cuh): D = 32 and L*P <= 16 (every UNINEXT call) ------------------------------
// OPT-IN (MSDA_KNOB_SLAB = 1).  They halve L2 sectors, but the shared-memory traffic of the window (4 wavefronts per
// privatised row-add) lands on the same LSU data pipe that the gathers already keep busy, and they were slower than the
// tiled kernels where they were first measured.  MSDA_KNOB_SLAB = -1 (auto) therefore selects the tiled kernels.

bool use_slab(const Dims &d, unsigned npairs, const void *value, const void *out) {
    if (d.D != 32 || d.L * d.P > 16 || d.L > msda::kMaxLevels) return false;
    if ((reinterpret_cast<uintptr_t>(value) & 31u) || (reinterpret_cast<uintptr_t>(out) & 15u)) return false;   // 32-byte row slices
    (void)npairs;
    return knob(MSDA_KNOB_SLAB) == 1;
}

template <typename T>
cudaError_t launch_fwd_slab(const T *value, const int64_t *shapes, const int64_t *lsi, const float *loc, const float *attn,
                            const Dims &d, T *out, cudaStream_t st) {
    const int ctas_per_sm = knob(MSDA_KNOB_FWD_SLAB_CTAS) == 1 ? 1 : 2;
    const int sms = num_sms();
    if (ctas_per_sm == 2)
        msda::msda_fwd_slab<T, 16, 2><<<sms * 2, msda::kSlabThreads, 0, st>>>(value, shapes, lsi, loc, attn, d.N, d.S, d.M, d.L,
                                                                              d.Lq, d.P, sms, out);
    else
        msda::msda_fwd_slab<T, 16, 1><<<sms, msda::kSlabThreads, 0, st>>>(value, shapes, lsi, loc, attn, d.N, d.S, d.M, d.L,
                                                                          d.Lq, d.P, sms, out);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return cudaGetLastError();
}

template <typename T>
cudaError_t launch_bwd_slab(const T *grad_out, const T *value, const int64_t *shapes, const int64_t *lsi, const float *loc,
                            const float *attn, const Dims &d, float *gv, float *gl, float *ga, cudaStream_t st) {
    // shared-memory budget: the opt-in maximum of the device minus the kernel's static part; the window gets what the
    // lists / g stash / tap slabs leave.  MSDA_BWD_WIN_ROWS / MSDA_BWD_LIST_CAP override (sweeps).
    static std::atomic<int> win_rows[kMaxDevices], cap_c[kMaxDevices], epoch_c[kMaxDevices];
    const int dev = current_device();
    const int epoch = knobs().epoch.load(std::memory_order_acquire);
    int rows = win_rows[dev].load(std::memory_order_relaxed), cap = cap_c[dev].load(std::memory_order_relaxed);
    auto kern = msda::msda_bwd_slab<T, 16>;
    if (rows == 0 || epoch_c[dev].load(std::memory_order_relaxed) != epoch) {
        int max_optin = 0;
        cudaDeviceGetAttribute(&max_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
        cudaFuncAttributes fa{};
        cudaFuncGetAttributes(&fa, kern);
        cap = knob(MSDA_KNOB_BWD_LIST_CAP) & ~1;
        if (cap < 8) cap = 8;
        const long long fixed = (long long)msda::bwd_slab_smem_bytes(0, cap) + (long long)fa.sharedSizeBytes + 64;
        rows = (int)((max_optin - fixed) / 128);
        const int want = knob(MSDA_KNOB_BWD_WIN_ROWS);
        if (want >= 0 && want < rows) rows = want;
        if (rows < 0) rows = 0;
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)msda::bwd_slab_smem_bytes(rows, cap));
        if (e != cudaSuccess) return e;
        cap_c[dev].store(cap, std::memory_order_relaxed);
        win_rows[dev].store(rows == 0 ? -1 : rows, std::memory_order_relaxed);
        epoch_c[dev].store(epoch, std::memory_order_relaxed);
    }
    if (rows < 0) rows = 0;
    const int sms = num_sms();
    kern<<<sms, msda::kSlabThreads, msda::bwd_slab_smem_bytes(rows, cap), st>>>(grad_out, value, shapes, lsi, loc, attn, d.N,
                                                                               d.S, d.M, d.L, d.Lq, d.P, sms, rows, cap, gv,
                                                                               gl, ga);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return cudaGetLastError();
}

// bf16 backward with the fine levels accumulated in the bf16 result (msda_bwd_tiled MIXED): D = 32, L*P <= 16, large launches.
cudaError_t launch_bwd_mixed(const __nv_bfloat16 *go, const __nv_bfloat16 *value, const int64_t *shapes, const int64_t *lsi,
                             const float *loc, const float *attn, const Dims &d, float *scratch, __nv_bfloat16 *gv16,
                             float *gl, float *ga, int fine_min_rows, cudaStream_t st) {
    using T = __nv_bfloat16;
    constexpr int VEC = 4, DD = 32, LP_MAX = 16;
    const unsigned npairs = (unsigned)((long long)d.N * d.Lq * d.M);
    static decltype(&msda::msda_bwd_tiled<T, VEC, DD, LP_MAX, kBwdMinCtas, false, false, true>) const kern[] = {
        msda::msda_bwd_tiled<T, VEC, DD, LP_MAX, kBwdMinCtas, true, false, true>,                     // tma, ldg
        msda::msda_bwd_tiled<T, VEC, DD, LP_MAX, kBwdMinCtas, false, false, true>};
    static std::atomic<int> cache[2][kMaxDevices];
    const int k = use_tma_staging(d) ? 0 : 1;
    return launch_tiled(kern[k], cache[k], npairs, msda::TiledShape<VEC, DD, LP_MAX, false>::kIterPairs, false, st, go,
                        value, shapes, lsi, loc, attn, d.N, d.S, d.M, d.L, d.Lq, d.P, npairs, allow_patches(), scratch,
                        gl, ga, gv16, fine_min_rows);
}

// Backward with the coarse levels accumulated by dedicated consumer warps (msda_tmem.cuh): MSDA_KNOB_SLAB = 2.  The window
// gets the device's opt-in shared memory minus the lists / g stash / tap slabs.
template <typename T>
cudaError_t launch_bwd_tmem(const T *grad_out, const T *value, const int64_t *shapes, const int64_t *lsi, const float *loc,
                            const float *attn, const Dims &d, float *gv, float *gl, float *ga, cudaStream_t st) {
    static std::atomic<int> win_rows[kMaxDevices], cap_c[kMaxDevices], epoch_c[kMaxDevices];
    const int dev = current_device();
    const int epoch = knobs().epoch.load(std::memory_order_acquire);
    auto kern = msda::msda_bwd_tmem<T, 16>;
    int cap = cap_c[dev].load(std::memory_order_relaxed), rows = win_rows[dev].load(std::memory_order_relaxed);
    if (rows == 0 || epoch_c[dev].load(std::memory_order_relaxed) != epoch) {
        cap = knob(MSDA_KNOB_BWD_LIST_CAP) & ~1;
        if (cap < 8) cap = 8;
        if (cap > 128) cap = 128;
        int max_optin = 0;
        cudaDeviceGetAttribute(&max_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
        cudaFuncAttributes fa{};
        cudaFuncGetAttributes(&fa, kern);
        const long long fixed = (long long)msda::bwd_tmem_smem_bytes(cap, 0) + (long long)fa.sharedSizeBytes + 64;
        rows = (int)((max_optin - fixed) / 128) & ~(msda::kTmCons - 1);
        if (rows < 0) rows = 0;
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)msda::bwd_tmem_smem_bytes(cap, rows));
        if (e != cudaSuccess) return e;
        cap_c[dev].store(cap, std::memory_order_relaxed);
        win_rows[dev].store(rows == 0 ? -1 : rows, std::memory_order_relaxed);
        epoch_c[dev].store(epoch, std::memory_order_relaxed);
    }
    if (rows < 0) rows = 0;
    const int sms = num_sms();
    kern<<<sms, msda::kTmThreads, msda::bwd_tmem_smem_bytes(cap, rows), st>>>(grad_out, value, shapes, lsi, loc, attn, d.N, d.S,
                                                                              d.M, d.L, d.Lq, d.P, sms, cap, rows, gv, gl, ga);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return cudaGetLastError();
}

// ---- region backward (msda_region.cuh): fp32 encoder self-attention, D = 32, L*P <= 16, Lq == S, large launches --------
// Auto-selected (MSDA_KNOB_REGION_BWD = -1); 0 keeps msda_bwd_tiled.
bool use_region(const Dims &d) {
    return knob(MSDA_KNOB_REGION_BWD) != 0 && d.D == 32 && d.L * d.P <= 16 && d.L <= msda::kMaxLevels && d.Lq == d.S &&
           !use_split((unsigned)((long long)d.N * d.Lq * d.M));
}

cudaError_t launch_bwd_region(const float *go, const float *value, const int64_t *shapes, const int64_t *lsi,
                              const float *loc, const float *attn, const Dims &d, float *gv, float *gl, float *ga,
                              cudaStream_t st) {
    auto kern = msda::msda_bwd_region<msda::kRegionEdge, msda::kRegionHalo>;
    constexpr size_t smem = msda::region_smem_bytes();
    static std::atomic<int> slots_c[kMaxDevices];
    const int dev = current_device();
    int slots = slots_c[dev].load(std::memory_order_relaxed);
    if (slots == 0) {
        const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        int per_sm = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, msda::kTiledThreads, smem) != cudaSuccess || per_sm < 1)
            per_sm = 1;
        slots = per_sm * num_sms();
        slots_c[dev].store(slots, std::memory_order_relaxed);
    }
    const unsigned npairs = (unsigned)((long long)d.N * d.Lq * d.M);
    const int tma = use_tma_staging(d) ? 1 : 0;            // the tap pass: TMA-staged or __ldg taps, as msda_bwd_tiled
    const cudaError_t e = launch_after_fill(kern, slots, smem, st, go, value, shapes, lsi, loc, attn, d.N, d.S, d.M, d.L, d.Lq,
                                            d.P, npairs, tma, gv, gl, ga);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return e;
}

#define MSDA_ROUTE_LP(T, DD, CALL, ...)                              \
    (LP <= 16 ? CALL<T, DD, 16, ##__VA_ARGS__> : CALL<T, DD, 32, ##__VA_ARGS__>)

template <typename T>
cudaError_t fwd_fast(const T *value, const int64_t *shapes, const int64_t *lsi, const float *loc, const float *attn,
                     const Dims &d, T *out, cudaStream_t st) {
    const int LP = d.L * d.P;
    if (use_slab(d, (unsigned)((long long)d.N * d.Lq * d.M), value, out))
        return launch_fwd_slab<T>(value, shapes, lsi, loc, attn, d, out, st);
    if constexpr (sizeof(T) == 4) {           // fp32, 32-byte lanes: needs 32-byte aligned rows
        if (knob(MSDA_KNOB_F32_VEC8_FWD) == 1 && LP <= 16 && (d.D == 32 || d.D == 64) &&
            !(reinterpret_cast<uintptr_t>(value) & 31u))
            return d.D == 32 ? launch_fwd<T, 32, 16, 8>(value, shapes, lsi, loc, attn, d, out, st)
                             : launch_fwd<T, 64, 16, 8>(value, shapes, lsi, loc, attn, d, out, st);
    }
    switch (d.D) {
        case 16: if constexpr (sizeof(T) == 4) return MSDA_ROUTE_LP(T, 16, launch_fwd)(value, shapes, lsi, loc, attn, d, out, st); break;
        case 32: return MSDA_ROUTE_LP(T, 32, launch_fwd)(value, shapes, lsi, loc, attn, d, out, st);
        case 64: return MSDA_ROUTE_LP(T, 64, launch_fwd)(value, shapes, lsi, loc, attn, d, out, st);
    }
    return cudaErrorInvalidValue;
}

template <typename T>
cudaError_t bwd_fast(const T *go, const T *value, const int64_t *shapes, const int64_t *lsi, const float *loc,
                     const float *attn, const Dims &d, float *gv, float *gl, float *ga, cudaStream_t st) {
    const int LP = d.L * d.P;
    if (knob(MSDA_KNOB_SLAB) == 2 && d.D == 32 && LP <= 16 && d.L <= msda::kMaxLevels)
        return launch_bwd_tmem<T>(go, value, shapes, lsi, loc, attn, d, gv, gl, ga, st);
    if (use_slab(d, (unsigned)((long long)d.N * d.Lq * d.M), value, gv))
        return launch_bwd_slab<T>(go, value, shapes, lsi, loc, attn, d, gv, gl, ga, st);
    if constexpr (sizeof(T) == 4) {
        if (knob(MSDA_KNOB_F32_VEC8_BWD) == 1 && LP <= 16 && d.D == 32 &&
            !((reinterpret_cast<uintptr_t>(value) | reinterpret_cast<uintptr_t>(go)) & 31u))
            return launch_bwd<T, 32, 16, 8>(go, value, shapes, lsi, loc, attn, d, gv, gl, ga, st);
        if (use_region(d)) return launch_bwd_region(go, value, shapes, lsi, loc, attn, d, gv, gl, ga, st);
    }
    switch (d.D) {
        case 16: if constexpr (sizeof(T) == 4) return MSDA_ROUTE_LP(T, 16, launch_bwd)(go, value, shapes, lsi, loc, attn, d, gv, gl, ga, st); break;
        case 32: return MSDA_ROUTE_LP(T, 32, launch_bwd)(go, value, shapes, lsi, loc, attn, d, gv, gl, ga, st);
        case 64: return MSDA_ROUTE_LP(T, 64, launch_bwd)(go, value, shapes, lsi, loc, attn, d, gv, gl, ga, st);
    }
    return cudaErrorInvalidValue;
}

template <typename T, typename TL>
cudaError_t fwd_generic(const T *value, const int64_t *shapes, const int64_t *lsi, const TL *loc, const TL *attn,
                        const Dims &d, T *out, cudaStream_t st) {
    const long long total = (long long)d.N * d.Lq * d.M * d.D;
    long long blocks = (total + 255) / 256;
    const long long cap = (long long)num_sms() * 32;
    if (blocks > cap) blocks = cap;
    msda::msda_fwd_generic<T, TL><<<(int)blocks, 256, 0, st>>>(value, shapes, lsi, loc, attn, d.S, d.M, d.D, d.L, d.Lq,
                                                               d.P, total, out);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return cudaGetLastError();
}

template <typename T, typename TL, typename GA, bool NORED = false>
cudaError_t bwd_generic(const T *go, const T *value, const int64_t *shapes, const int64_t *lsi, const TL *loc,
                        const TL *attn, const Dims &d, GA *gv, TL *gl, TL *ga, cudaStream_t st) {
    const long long npairs = (long long)d.N * d.Lq * d.M;
    int threads = ((d.D + 31) / 32) * 32;
    if (threads > 256) threads = 256;
    long long blocks = npairs;
    const long long cap = (long long)num_sms() * 64;
    if (blocks > cap) blocks = cap;
    msda::msda_bwd_generic<T, TL, GA, NORED><<<(int)blocks, threads, 0, st>>>(go, value, shapes, lsi, loc, attn, d.S, d.M,
                                                                              d.D, d.L, d.Lq, d.P, npairs, gv, gl, ga);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return cudaGetLastError();
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
    auto take = [&](size_t bytes) { const size_t at = off; off += (bytes + 255) & ~(size_t)255; return at; };
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
        if (fast) {
            const int LP = d.L * d.P;
            switch (d.D) {
                case 16: if constexpr (sizeof(T) == 4) return MSDA_ROUTE_LP(T, 16, launch_bwd, 4, true)(go, value, shapes, lsi, loc, attn, d, gv, gl, ga, st); break;
                case 32: return MSDA_ROUTE_LP(T, 32, launch_bwd, 4, true)(go, value, shapes, lsi, loc, attn, d, gv, gl, ga, st);
                case 64: return MSDA_ROUTE_LP(T, 64, launch_bwd, 4, true)(go, value, shapes, lsi, loc, attn, d, gv, gl, ga, st);
            }
            return cudaErrorInvalidValue;
        }
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
            long long blocks = ((long long)lay.n + msda::kDetThreads - 1) / msda::kDetThreads;
            if (blocks > (long long)sms * 16) blocks = (long long)sms * 16;
            msda::msda_det_keys<TL><<<(int)blocks, msda::kDetThreads, 0, st>>>(loc, shapes, lsi, d.S, d.M, d.L, d.P, tap0,
                                                                               lay.n, keys_in, vals_in);
            if ((err = cudaGetLastError()) != cudaSuccess) return (int)err;
            size_t temp_bytes = lay.temp_bytes;
            err = msda::det_sort(w + lay.temp, temp_bytes, keys_in, keys_out, vals_in, vals_out, lay.n, end_bit, st);
            if (err != cudaSuccess) return (int)err;
            long long kblocks = ((long long)nkeys + 1 + msda::kDetThreads - 1) / msda::kDetThreads;
            if (kblocks > (long long)sms * 16) kblocks = (long long)sms * 16;
            msda::msda_det_bounds<<<(int)kblocks, msda::kDetThreads, 0, st>>>(keys_out, lay.n, nkeys, start);
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

int msda_forward_f32(const float *value, const int64_t *spatial_shapes, const int64_t *level_start_index,
                     const float *sampling_loc, const float *attn_weight, int N, int S, int M, int D, int L, int Lq,
                     int P, float *out, void *stream) {
    const Dims d{N, S, M, D, L, Lq, P};
    if (int e = check_dims(d)) return e;
    MSDA_CHECK_PTRS(al, value, sampling_loc, attn_weight, out);
    if (!spatial_shapes || !level_start_index) return MSDA_E_BADARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (al && use_fast(4, d)) return (int)fwd_fast<float>(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, d, out, st);
    return (int)fwd_generic<float, float>(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, d, out, st);
}

int msda_forward_f64(const double *value, const int64_t *spatial_shapes, const int64_t *level_start_index,
                     const double *sampling_loc, const double *attn_weight, int N, int S, int M, int D, int L, int Lq,
                     int P, double *out, void *stream) {
    const Dims d{N, S, M, D, L, Lq, P};
    if (int e = check_dims(d)) return e;
    if (!value || !spatial_shapes || !level_start_index || !sampling_loc || !attn_weight || !out) return MSDA_E_BADARG;
    return (int)fwd_generic<double, double>(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, d, out,
                                            static_cast<cudaStream_t>(stream));
}

int msda_forward_bf16(const uint16_t *value, const int64_t *spatial_shapes, const int64_t *level_start_index,
                      const float *sampling_loc, const float *attn_weight, int N, int S, int M, int D, int L, int Lq,
                      int P, uint16_t *out, void *stream) {
    const Dims d{N, S, M, D, L, Lq, P};
    if (int e = check_dims(d)) return e;
    MSDA_CHECK_PTRS(al, value, sampling_loc, attn_weight, out);
    if (!spatial_shapes || !level_start_index) return MSDA_E_BADARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const __nv_bfloat16 *v = reinterpret_cast<const __nv_bfloat16 *>(value);
    __nv_bfloat16 *o = reinterpret_cast<__nv_bfloat16 *>(out);
    if (al && use_fast(2, d)) return (int)fwd_fast<__nv_bfloat16>(v, spatial_shapes, level_start_index, sampling_loc, attn_weight, d, o, st);
    return (int)fwd_generic<__nv_bfloat16, float>(v, spatial_shapes, level_start_index, sampling_loc, attn_weight, d, o, st);
}

int msda_backward_f32(const float *grad_out, const float *value, const int64_t *spatial_shapes,
                      const int64_t *level_start_index, const float *sampling_loc, const float *attn_weight, int N,
                      int S, int M, int D, int L, int Lq, int P, float *grad_value, float *grad_sampling_loc,
                      float *grad_attn_weight, void *stream) {
    const Dims d{N, S, M, D, L, Lq, P};
    if (int e = check_dims(d)) return e;
    MSDA_CHECK_PTRS(al, grad_out, value, sampling_loc, attn_weight, grad_value, grad_sampling_loc, grad_attn_weight);
    if (!spatial_shapes || !level_start_index) return MSDA_E_BADARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    bool pdl = false;
    cudaError_t err = zero_fill(grad_value, sizeof(float) * (size_t)N * S * M * D, st, &pdl);
    if (err != cudaSuccess) return (int)err;
    if (al && use_fast(4, d)) {
        t_pdl_next = pdl;
        err = bwd_fast<float>(grad_out, value, spatial_shapes, level_start_index, sampling_loc, attn_weight, d,
                              grad_value, grad_sampling_loc, grad_attn_weight, st);
        t_pdl_next = false;
        return (int)err;
    }
    return (int)bwd_generic<float, float, float>(grad_out, value, spatial_shapes, level_start_index, sampling_loc,
                                                 attn_weight, d, grad_value, grad_sampling_loc, grad_attn_weight, st);
}

int msda_backward_f64(const double *grad_out, const double *value, const int64_t *spatial_shapes,
                      const int64_t *level_start_index, const double *sampling_loc, const double *attn_weight, int N,
                      int S, int M, int D, int L, int Lq, int P, double *grad_value, double *grad_sampling_loc,
                      double *grad_attn_weight, void *stream) {
    const Dims d{N, S, M, D, L, Lq, P};
    if (int e = check_dims(d)) return e;
    if (!grad_out || !value || !spatial_shapes || !level_start_index || !sampling_loc || !attn_weight || !grad_value ||
        !grad_sampling_loc || !grad_attn_weight)
        return MSDA_E_BADARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaError_t err = zero_fill(grad_value, sizeof(double) * (size_t)N * S * M * D, st);
    if (err != cudaSuccess) return (int)err;
    return (int)bwd_generic<double, double, double>(grad_out, value, spatial_shapes, level_start_index, sampling_loc,
                                                    attn_weight, d, grad_value, grad_sampling_loc, grad_attn_weight, st);
}

int msda_backward_bf16(const uint16_t *grad_out, const uint16_t *value, const int64_t *spatial_shapes,
                       const int64_t *level_start_index, const float *sampling_loc, const float *attn_weight, int N,
                       int S, int M, int D, int L, int Lq, int P, float *grad_value_f32, uint16_t *grad_value,
                       float *grad_sampling_loc, float *grad_attn_weight, void *stream) {
    const Dims d{N, S, M, D, L, Lq, P};
    if (int e = check_dims(d)) return e;
    MSDA_CHECK_PTRS(al, grad_out, value, sampling_loc, attn_weight, grad_value_f32, grad_sampling_loc, grad_attn_weight);
    if (!spatial_shapes || !level_start_index) return MSDA_E_BADARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t nval = (size_t)N * S * M * D;
    const __nv_bfloat16 *go = reinterpret_cast<const __nv_bfloat16 *>(grad_out);
    const __nv_bfloat16 *v = reinterpret_cast<const __nv_bfloat16 *>(value);
    const int fine_rows = knob(MSDA_KNOB_BF16_FINE_ROWS);
    if (fine_rows > 0 && grad_value != nullptr && al && use_fast(2, d) && D == 32 && L * P <= 16 &&
        !use_split((unsigned)((long long)N * Lq * M)) && !(reinterpret_cast<uintptr_t>(grad_value) & 15u)) {
        // mixed accumulation: bf16 result zero-filled (fine levels add into it), fp32 scratch zero-filled for the coarse
        // levels only, one rounding pass over the coarse rows at the end -- no full-size fp32 round trip
        __nv_bfloat16 *gv16 = reinterpret_cast<__nv_bfloat16 *>(grad_value);
        cudaError_t e = zero_fill(grad_value, sizeof(uint16_t) * nval, st);
        if (e != cudaSuccess) return (int)e;
        const dim3 hgrid((unsigned)(num_sms() * 2 / (N < 1 ? 1 : N) + 1), (unsigned)N);
        msda::msda_coarse_rows<false><<<hgrid, 256, 0, st>>>(grad_value_f32, gv16, spatial_shapes, level_start_index, L, S,
                                                             M * D, fine_rows);
        g_launches.fetch_add(1, std::memory_order_relaxed);
        e = launch_bwd_mixed(go, v, spatial_shapes, level_start_index, sampling_loc, attn_weight, d, grad_value_f32, gv16,
                             grad_sampling_loc, grad_attn_weight, fine_rows, st);
        if (e != cudaSuccess) return (int)e;
        msda::msda_coarse_rows<true><<<hgrid, 256, 0, st>>>(grad_value_f32, gv16, spatial_shapes, level_start_index, L, S,
                                                            M * D, fine_rows);
        g_launches.fetch_add(1, std::memory_order_relaxed);
        return (int)cudaGetLastError();
    }
    bool pdl = false;
    cudaError_t err = zero_fill(grad_value_f32, sizeof(float) * nval, st, &pdl);
    if (err != cudaSuccess) return (int)err;
    if (al && use_fast(2, d)) {
        t_pdl_next = pdl;
        err = bwd_fast<__nv_bfloat16>(go, v, spatial_shapes, level_start_index, sampling_loc, attn_weight, d,
                                      grad_value_f32, grad_sampling_loc, grad_attn_weight, st);
        t_pdl_next = false;
    } else
        err = bwd_generic<__nv_bfloat16, float, float>(go, v, spatial_shapes, level_start_index, sampling_loc,
                                                       attn_weight, d, grad_value_f32, grad_sampling_loc,
                                                       grad_attn_weight, st);
    if (err != cudaSuccess) return (int)err;
    if (grad_value != nullptr) {
        long long blocks = (long long)((nval + 255) / 256);
        const long long cap = (long long)num_sms() * 16;
        if (blocks > cap) blocks = cap;
        msda::msda_f32_to_bf16<<<(int)blocks, 256, 0, st>>>(grad_value_f32, reinterpret_cast<__nv_bfloat16 *>(grad_value),
                                                            (long long)nval);
        g_launches.fetch_add(1, std::memory_order_relaxed);
        err = cudaGetLastError();
    }
    return (int)err;
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
    const Dims d{N, S, M, D, L, Lq, P};
    if (int e = det_check(d)) return e;
    MSDA_CHECK_PTRS(al, grad_out, value, sampling_loc, attn_weight, grad_value, grad_sampling_loc, grad_attn_weight);
    if (!spatial_shapes || !level_start_index) return MSDA_E_BADARG;
    return det_backward<float, float>(grad_out, value, spatial_shapes, level_start_index, sampling_loc, attn_weight, d,
                                      al && use_fast(4, d), grad_value, grad_sampling_loc, grad_attn_weight, workspace,
                                      workspace_bytes, static_cast<cudaStream_t>(stream));
}

int msda_backward_det_f64(const double *grad_out, const double *value, const int64_t *spatial_shapes,
                          const int64_t *level_start_index, const double *sampling_loc, const double *attn_weight, int N,
                          int S, int M, int D, int L, int Lq, int P, double *grad_value, double *grad_sampling_loc,
                          double *grad_attn_weight, void *workspace, int64_t workspace_bytes, void *stream) {
    const Dims d{N, S, M, D, L, Lq, P};
    if (int e = det_check(d)) return e;
    if (!grad_out || !value || !spatial_shapes || !level_start_index || !sampling_loc || !attn_weight || !grad_value ||
        !grad_sampling_loc || !grad_attn_weight)
        return MSDA_E_BADARG;
    return det_backward<double, double>(grad_out, value, spatial_shapes, level_start_index, sampling_loc, attn_weight, d,
                                        false, grad_value, grad_sampling_loc, grad_attn_weight, workspace, workspace_bytes,
                                        static_cast<cudaStream_t>(stream));
}

int msda_backward_det_bf16(const uint16_t *grad_out, const uint16_t *value, const int64_t *spatial_shapes,
                           const int64_t *level_start_index, const float *sampling_loc, const float *attn_weight, int N,
                           int S, int M, int D, int L, int Lq, int P, float *grad_value_f32, uint16_t *grad_value,
                           float *grad_sampling_loc, float *grad_attn_weight, void *workspace, int64_t workspace_bytes,
                           void *stream) {
    const Dims d{N, S, M, D, L, Lq, P};
    if (int e = det_check(d)) return e;
    MSDA_CHECK_PTRS(al, grad_out, value, sampling_loc, attn_weight, grad_value_f32, grad_sampling_loc, grad_attn_weight);
    if (!spatial_shapes || !level_start_index) return MSDA_E_BADARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int e = det_backward<__nv_bfloat16, float>(
        reinterpret_cast<const __nv_bfloat16 *>(grad_out), reinterpret_cast<const __nv_bfloat16 *>(value), spatial_shapes,
        level_start_index, sampling_loc, attn_weight, d, al && use_fast(2, d), grad_value_f32, grad_sampling_loc,
        grad_attn_weight, workspace, workspace_bytes, st);
    if (e != 0 || grad_value == nullptr) return e;
    const size_t nval = (size_t)N * S * M * D;
    long long blocks = (long long)((nval + 255) / 256);
    const long long cap = (long long)num_sms() * 16;
    if (blocks > cap) blocks = cap;
    msda::msda_f32_to_bf16<<<(int)blocks, 256, 0, st>>>(grad_value_f32, reinterpret_cast<__nv_bfloat16 *>(grad_value),
                                                        (long long)nval);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return (int)cudaGetLastError();
}


}  // extern "C"

// ---- callers of the op --------------------------------------------------------------------------------------------
namespace {
template <int G>
cudaError_t prologue_fwd_launch(const float *proj, const float *ref, const int64_t *shapes, long long npairs, int M, int L,
                                int P, int refdim, float *loc, float *attn, cudaStream_t st) {
    const long long threads = npairs * G;
    msda::msda_prologue_fwd<G><<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(proj, ref, shapes, npairs, M, L, P, refdim, loc, attn);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return cudaGetLastError();
}
template <int G>
cudaError_t prologue_bwd_launch(const float *gl, const float *ga, const float *attn, const float *ref, const int64_t *shapes,
                                long long npairs, int M, int L, int P, int refdim, float *gp, cudaStream_t st) {
    const long long threads = npairs * G;
    msda::msda_prologue_bwd<G><<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(gl, ga, attn, ref, shapes, npairs, M, L, P, refdim, gp);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return cudaGetLastError();
}
int group_width(int LP) { return LP <= 4 ? 4 : LP <= 8 ? 8 : LP <= 16 ? 16 : 32; }
}  // namespace

extern "C" {

int msda_prologue_forward_f32(const float *proj, const float *ref, const int64_t *spatial_shapes, int64_t R, int M, int L,
                              int P, int refdim, float *loc, float *attn, void *stream) {
    if (!proj || !ref || !spatial_shapes || !loc || !attn || R <= 0 || M <= 0 || L <= 0 || P <= 0 || L * P > 32 ||
        (refdim != 2 && refdim != 4) || (long long)R * M * 32 >= (1ll << 40) || !aligned8(loc))      // float2 stores
        return MSDA_E_BADARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long np = (long long)R * M;
    switch (group_width(L * P)) {
        case 4: return (int)prologue_fwd_launch<4>(proj, ref, spatial_shapes, np, M, L, P, refdim, loc, attn, st);
        case 8: return (int)prologue_fwd_launch<8>(proj, ref, spatial_shapes, np, M, L, P, refdim, loc, attn, st);
        case 16: return (int)prologue_fwd_launch<16>(proj, ref, spatial_shapes, np, M, L, P, refdim, loc, attn, st);
        default: return (int)prologue_fwd_launch<32>(proj, ref, spatial_shapes, np, M, L, P, refdim, loc, attn, st);
    }
}

int msda_prologue_backward_f32(const float *grad_loc, const float *grad_attn, const float *attn, const float *ref,
                               const int64_t *spatial_shapes, int64_t R, int M, int L, int P, int refdim,
                               float *grad_proj, void *stream) {
    if (!grad_loc || !grad_attn || !attn || !ref || !spatial_shapes || !grad_proj || R <= 0 || M <= 0 || L <= 0 || P <= 0 ||
        L * P > 32 || (refdim != 2 && refdim != 4) || !aligned8(grad_loc))                             // float2 loads
        return MSDA_E_BADARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long np = (long long)R * M;
    switch (group_width(L * P)) {
        case 4: return (int)prologue_bwd_launch<4>(grad_loc, grad_attn, attn, ref, spatial_shapes, np, M, L, P, refdim, grad_proj, st);
        case 8: return (int)prologue_bwd_launch<8>(grad_loc, grad_attn, attn, ref, spatial_shapes, np, M, L, P, refdim, grad_proj, st);
        case 16: return (int)prologue_bwd_launch<16>(grad_loc, grad_attn, attn, ref, spatial_shapes, np, M, L, P, refdim, grad_proj, st);
        default: return (int)prologue_bwd_launch<32>(grad_loc, grad_attn, attn, ref, spatial_shapes, np, M, L, P, refdim, grad_proj, st);
    }
}

int msda_colsum_f32(const float *x, int64_t rows, int cols, float *out, void *stream) {
    if (!x || !out || rows <= 0 || cols <= 0 || cols % 4 != 0 || !aligned16(x) || !aligned16(out)) return MSDA_E_BADARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaError_t err = cudaMemsetAsync(out, 0, sizeof(float) * (size_t)cols, st);
    if (err != cudaSuccess) return (int)err;
    long long ctas = (long long)num_sms() * 4;
    int rows_per_cta = (int)((rows + ctas - 1) / ctas);
    if (rows_per_cta < 16) rows_per_cta = 16;
    const unsigned grid = (unsigned)((rows + rows_per_cta - 1) / rows_per_cta);
    msda::msda_colsum<<<grid, 256, 0, st>>>(x, rows, cols, rows_per_cta, out);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return (int)cudaGetLastError();
}

int msda_relu_backward_colsum_f32(const float *g, const float *y, int64_t rows, int cols, float *g2, float *colsum, void *stream) {
    if (!g || !y || !g2 || !colsum || rows <= 0 || cols <= 0 || cols % 4 != 0 || !aligned16(g) || !aligned16(y) || !aligned16(g2) ||
        !aligned16(colsum))
        return MSDA_E_BADARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaError_t err = cudaMemsetAsync(colsum, 0, sizeof(float) * (size_t)cols, st);
    if (err != cudaSuccess) return (int)err;
    long long ctas = (long long)num_sms() * 8;
    int rows_per_cta = (int)((rows + ctas - 1) / ctas);
    if (rows_per_cta < 16) rows_per_cta = 16;
    const unsigned grid = (unsigned)((rows + rows_per_cta - 1) / rows_per_cta);
    msda::msda_relu_bwd_colsum<<<grid, 256, 0, st>>>(g, y, rows, cols, rows_per_cta, g2, colsum);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return (int)cudaGetLastError();
}

int msda_add_layernorm_forward_f32(const float *a, const float *b, const float *gamma, const float *beta, int64_t rows,
                                   int cols, float eps, float *z, float *y, float *mean, float *rstd, void *stream) {
    if (!a || !gamma || !beta || !y || !mean || !rstd || rows <= 0 || (b != nullptr && z == nullptr)) return MSDA_E_BADARG;
    if (cols != 128 && cols != 256 && cols != 384 && cols != 512) return MSDA_E_BADARG;
    if (!aligned16(a) || !aligned16(gamma) || !aligned16(beta) || !aligned16(y) || (b && !aligned16(b)) || (z && !aligned16(z)))
        return MSDA_E_BADARG;                                                                        // float4 accesses
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const unsigned grid = (unsigned)((rows + 7) / 8);
    switch (cols / 128) {
        case 1: msda::msda_add_layernorm_fwd<1><<<grid, 256, 0, st>>>(a, b, gamma, beta, rows, eps, z, y, mean, rstd); break;
        case 2: msda::msda_add_layernorm_fwd<2><<<grid, 256, 0, st>>>(a, b, gamma, beta, rows, eps, z, y, mean, rstd); break;
        case 3: msda::msda_add_layernorm_fwd<3><<<grid, 256, 0, st>>>(a, b, gamma, beta, rows, eps, z, y, mean, rstd); break;
        default: msda::msda_add_layernorm_fwd<4><<<grid, 256, 0, st>>>(a, b, gamma, beta, rows, eps, z, y, mean, rstd); break;
    }
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return (int)cudaGetLastError();
}

int msda_layernorm_backward_f32(const float *dy, const float *z, const float *gamma, const float *mean, const float *rstd,
                                int64_t rows, int cols, float *dz, float *dgamma, float *dbeta, void *stream) {
    if (!dy || !z || !gamma || !mean || !rstd || !dz || !dgamma || !dbeta || rows <= 0) return MSDA_E_BADARG;
    if (cols != 128 && cols != 256 && cols != 384 && cols != 512) return MSDA_E_BADARG;
    if (!aligned16(dy) || !aligned16(z) || !aligned16(gamma) || !aligned16(dz) || !aligned16(dgamma) || !aligned16(dbeta))
        return MSDA_E_BADARG;                                                                        // float4 accesses, 16-byte reds
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaError_t err = cudaMemsetAsync(dgamma, 0, sizeof(float) * (size_t)cols, st);
    if (err == cudaSuccess) err = cudaMemsetAsync(dbeta, 0, sizeof(float) * (size_t)cols, st);
    if (err != cudaSuccess) return (int)err;
    long long ctas = (long long)num_sms() * 4;
    int rows_per_cta = (int)((rows + ctas - 1) / ctas);
    rows_per_cta = ((rows_per_cta + 7) / 8) * 8;
    const unsigned grid = (unsigned)((rows + rows_per_cta - 1) / rows_per_cta);
    switch (cols / 128) {
        case 1: msda::msda_layernorm_bwd<1><<<grid, 256, 0, st>>>(dy, z, gamma, mean, rstd, rows, rows_per_cta, dz, dgamma, dbeta); break;
        case 2: msda::msda_layernorm_bwd<2><<<grid, 256, 0, st>>>(dy, z, gamma, mean, rstd, rows, rows_per_cta, dz, dgamma, dbeta); break;
        case 3: msda::msda_layernorm_bwd<3><<<grid, 256, 0, st>>>(dy, z, gamma, mean, rstd, rows, rows_per_cta, dz, dgamma, dbeta); break;
        default: msda::msda_layernorm_bwd<4><<<grid, 256, 0, st>>>(dy, z, gamma, mean, rstd, rows, rows_per_cta, dz, dgamma, dbeta); break;
    }
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return (int)cudaGetLastError();
}

}  // extern "C"

// ---- CondInst dynamic mask head -------------------------------------------------------------------------------------
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
    msda::condinst_fwd<<<grid, msda::kCiFwdThreads, 0, static_cast<cudaStream_t>(stream)>>>(feats, params, refs, inst_start, HW,
                                                                                          W, stride, rel_coord, vec, logits);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return (int)cudaGetLastError();
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
    msda::condinst_bwd<<<grid, msda::kCiThreads, 0, st>>>(grad_logits, feats, params, refs, inst_start, HW, W, stride, rel_coord,
                                                          grad_feats, grad_params, grad_refs);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return (int)cudaGetLastError();
}

int msda_aligned_bilinear_forward_f32(const float *in, int64_t planes, int h, int w, int factor, float *out, void *stream) {
    if (!in || !out || planes < 0 || planes >= (1ll << 31) || h <= 0 || w <= 0 || factor < 1 ||
        (long long)h * factor * w * factor >= (1ll << 31))
        return MSDA_E_BADARG;
    if (planes == 0) return 0;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const dim3 grid((unsigned)planes, (unsigned)((h * factor + msda::kAbRows - 1) / msda::kAbRows));
    const bool vec = (w * factor) % 4 == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0;
    if (factor == 2 && vec) msda::aligned_bilinear2_fwd<<<grid, 256, 0, st>>>(in, h, w, out);
    else if (vec) msda::aligned_bilinear_fwd<0, 4><<<grid, 256, 0, st>>>(in, h, w, factor, out);
    else msda::aligned_bilinear_fwd<0, 1><<<grid, 256, 0, st>>>(in, h, w, factor, out);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return (int)cudaGetLastError();
}

int msda_aligned_bilinear_backward_f32(const float *grad_out, int64_t planes, int h, int w, int factor, float *grad_in,
                                       void *stream) {
    if (!grad_out || !grad_in || planes < 0 || planes >= (1ll << 31) || h <= 0 || w <= 0 || factor < 1 ||
        (long long)h * factor * w * factor >= (1ll << 31))
        return MSDA_E_BADARG;
    if (planes == 0) return 0;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const dim3 grid((unsigned)planes, (unsigned)((h + msda::kAbRows - 1) / msda::kAbRows));
    const bool vec = w % 2 == 0 && (reinterpret_cast<uintptr_t>(grad_out) & 15) == 0 && (reinterpret_cast<uintptr_t>(grad_in) & 7) == 0;
    if (factor == 2 && vec) msda::aligned_bilinear2_bwd<<<grid, 256, 0, st>>>(grad_out, h, w, grad_in);
    else msda::aligned_bilinear_bwd<0><<<grid, 256, 0, st>>>(grad_out, h, w, factor, grad_in);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return (int)cudaGetLastError();
}

int msda_mask_paste_f32(const float *logits, int64_t I, int Hs, int Ws, int stride, int crop_h, int crop_w, int out_h,
                        int out_w, float threshold, int binary, void *out, void *stream) {
    if (!logits || !out || I < 0 || Hs <= 0 || Ws <= 0 || stride <= 0 || crop_h <= 0 || crop_w <= 0 || out_h <= 0 ||
        out_w <= 0 || (long long)stride * Hs >= (1ll << 31) || (long long)stride * Ws >= (1ll << 31) ||
        crop_h > stride * Hs || crop_w > stride * Ws)
        return MSDA_E_BADARG;
    constexpr int cols = msda::kMpGroups * msda::kMpCols, rows = msda::kMpRows;
    if (out_h > 65535 * rows || out_w >= (1 << 30)) return MSDA_E_TOOLARGE;
    if (I == 0) return 0;
    // The scales exactly as torch forms them for an explicit output size: (float)input_size / output_size.
    const float near_y = (float)crop_h / (float)out_h, near_x = (float)crop_w / (float)out_w;
    const float lin_y = (float)Hs / (float)(stride * Hs), lin_x = (float)Ws / (float)(stride * Ws);
    const long long chunks = (I + msda::kMpInst - 1) / msda::kMpInst;
    const dim3 grid((unsigned)((out_w + cols - 1) / cols), (unsigned)((out_h + rows - 1) / rows),
                    (unsigned)(chunks < 65535 ? chunks : 65535));
    const dim3 block(msda::kMpGroups, rows);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool vec = aligned16(out) && out_w % (binary ? msda::kMpCols : 4) == 0;
#define MP_LAUNCH(B, V)                                                                                                  \
    msda::mask_paste<B, V><<<grid, block, 0, st>>>(logits, I, Hs, Ws, crop_h, crop_w, out_h, out_w, near_y, near_x,   \
                                                   lin_y, lin_x, threshold, out)
    if (binary) { if (vec) MP_LAUNCH(true, true); else MP_LAUNCH(true, false); }
    else { if (vec) MP_LAUNCH(false, true); else MP_LAUNCH(false, false); }
#undef MP_LAUNCH
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return (int)cudaGetLastError();
}

}  // extern "C"

// ---- detection post-processing (f-6) ----------------------------------------------------------------------------------
namespace {

struct DetpostLayout {
    size_t prob, qmax, qarg, sort, total;
    long long sort_cap;                         // u64 sort slots per image in the workspace (0: the CTA sorts on chip)
};

inline size_t dp_align(size_t x) { return (x + 255) & ~(size_t)255; }

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
    l.qmax = dp_align(l.prob + (size_t)B * Q * C * sizeof(float));
    l.qarg = dp_align(l.qmax + (size_t)B * Q * sizeof(float));
    l.sort = dp_align(l.qarg + (size_t)B * Q * sizeof(int));
    l.total = dp_align(l.sort + (size_t)B * l.sort_cap * sizeof(unsigned long long));
    return l;
}

}  // namespace

extern "C" {

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
        static std::atomic<bool> opted_in[kMaxDevices];
        const int dev = current_device();
        if (!opted_in[dev].load(std::memory_order_acquire)) {
            const cudaError_t e = cudaFuncSetAttribute(msda::detpost_select<true>,
                                                       cudaFuncAttributeMaxDynamicSharedMemorySize, kDynMax);
            if (e != cudaSuccess) return (int)e;
            opted_in[dev].store(true, std::memory_order_release);
        }
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

}  // extern "C"

// ---- COCO run-length encoding of masks (f-7) ----------------------------------------------------------------------------
namespace {

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
    l.bitmap = dp_align(l.col_off + (size_t)cols * sizeof(long long));
    l.scan = dp_align(l.bitmap + (size_t)I * nw * out_w * sizeof(unsigned));
    l.tiles = dp_align(l.scan + l.scan_bytes);
    l.total = dp_align(l.tiles + (size_t)max_tiles * sizeof(long long));
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
    if (!logits || !workspace || !aligned16(workspace) || I < 0 || Hs <= 0 || Ws <= 0 || stride <= 0 || crop_h <= 0 ||
        crop_w <= 0 || out_h <= 0 || out_w <= 0 || (long long)stride * Hs >= (1ll << 31) ||
        (long long)stride * Ws >= (1ll << 31) || crop_h > stride * Hs || crop_w > stride * Ws)
        return MSDA_E_BADARG;
    if (out_h > 65535 * msda::kMpRows) return MSDA_E_TOOLARGE;           // msda_mask_paste_f32's limits
    if (const int c = rle_check(I, out_h, out_w)) return c;
    if (I == 0) return 0;
    RleLayout l;
    if (const int e = rle_layout(I, out_h, out_w, l)) return e;
    if (workspace_bytes < (int64_t)l.total) return MSDA_E_BADARG;
    char *ws = static_cast<char *>(workspace);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // The scales exactly as msda_mask_paste_f32 forms them.
    const float near_y = (float)crop_h / (float)out_h, near_x = (float)crop_w / (float)out_w;
    const float lin_y = (float)Hs / (float)(stride * Hs), lin_x = (float)Ws / (float)(stride * Ws);
    msda::rle_bits_logits<<<rle_grid(I, out_w, 1), msda::kRleThreads, 0, st>>>(
        logits, I, Hs, Ws, crop_h, crop_w, out_h, out_w, near_y, near_x, lin_y, lin_x, threshold,
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
        (reinterpret_cast<uintptr_t>(positions) & 3u) || (reinterpret_cast<uintptr_t>(byte_offsets) & 7u))
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

// ---- geometry feeding the op (f-3) --------------------------------------------------------------------------------------
extern "C" {

int msda_valid_counts(const uint8_t *mask, const int64_t *spatial_shapes, const int64_t *level_start_index, int N, int S, int L,
                      int32_t *counts, void *stream) {
    if (!mask || !spatial_shapes || !level_start_index || !counts || N <= 0 || S <= 0 || L <= 0) return MSDA_E_BADARG;
    const int warps = N * L;
    msda::msda_valid_counts<<<(warps * 32 + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(mask, spatial_shapes,
                                                                                                      level_start_index, N, S, L, counts);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return (int)cudaGetLastError();
}

int msda_encoder_ref_points_f32(const float *valid_ratios, const int64_t *spatial_shapes, const int64_t *level_start_index, int N,
                                int S, int L, float *ref, void *stream) {
    if (!valid_ratios || !spatial_shapes || !level_start_index || !ref || N <= 0 || S <= 0 || L <= 0 || !aligned16(ref)) return MSDA_E_BADARG;
    const long long total = (long long)N * S;
    msda::msda_encoder_ref_points<<<(unsigned)((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        valid_ratios, spatial_shapes, level_start_index, N, S, L, ref);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return (int)cudaGetLastError();
}

int msda_encoder_proposals_f32(const uint8_t *mask, const int32_t *counts, const int64_t *spatial_shapes,
                               const int64_t *level_start_index, int N, int S, int L, float base_scale, float *proposals,
                               uint8_t *keep, void *stream) {
    if (!mask || !counts || !spatial_shapes || !level_start_index || !proposals || !keep || N <= 0 || S <= 0 || L <= 0 || L > 30 ||
        !aligned16(proposals))
        return MSDA_E_BADARG;
    const long long total = (long long)N * S;
    msda::msda_encoder_proposals<<<(unsigned)((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        mask, counts, spatial_shapes, level_start_index, N, S, L, base_scale, proposals, keep);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return (int)cudaGetLastError();
}

int msda_sine_pos_embed_forward_f32(const float *pos, int64_t R, int n, int F, float temperature, int exchange_xy, float *out,
                                    void *stream) {
    if (!pos || !out || R <= 0 || n <= 0 || F <= 0) return MSDA_E_BADARG;
    const long long warps = (long long)R * n;
    msda::msda_sine_pos_embed<false><<<(unsigned)((warps * 32 + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        pos, nullptr, R, n, F, temperature, exchange_xy, out);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return (int)cudaGetLastError();
}

int msda_sine_pos_embed_backward_f32(const float *pos, const float *grad_out, int64_t R, int n, int F, float temperature,
                                     int exchange_xy, float *grad_pos, void *stream) {
    if (!pos || !grad_out || !grad_pos || R <= 0 || n <= 0 || F <= 0) return MSDA_E_BADARG;
    const long long warps = (long long)R * n;
    msda::msda_sine_pos_embed<true><<<(unsigned)((warps * 32 + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        pos, grad_out, R, n, F, temperature, exchange_xy, grad_pos);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return (int)cudaGetLastError();
}

}  // extern "C"

// ---- fused image-text attention of the early-fusion block (msda_vlfuse.cuh) -----------------------------------------
namespace {

struct VlfLayout {
    size_t part0, part1, colpart, delta_v, delta_l, total;
    int row_tiles, col_tiles, nsplit, split_rows;
};

inline size_t align256(size_t x) { return (x + 255) & ~size_t(255); }

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
template <int D, class T>
cudaError_t vlf_forward_launch(const vlf::ParamsT<T> &p, const VlfLayout &l, void (*rows)(vlf::ParamsT<T>), int rows_smem,
                               void (*cols)(vlf::ParamsT<T>), int cols_smem, cudaStream_t st) {
    cudaError_t e;
    if ((e = cudaFuncSetAttribute(rows, cudaFuncAttributeMaxDynamicSharedMemorySize, rows_smem)) ||
        (e = cudaFuncSetAttribute(cols, cudaFuncAttributeMaxDynamicSharedMemorySize, cols_smem)))
        return e;
    const unsigned BH = (unsigned)(p.B * p.H);
    rows<<<dim3(l.row_tiles, BH), vlf::kThreads, rows_smem, st>>>(p);
    vlf::vlf_colstats<<<BH, vlf::kMaxT, 0, st>>>(p, l.row_tiles);
    cols<<<dim3(l.col_tiles, l.nsplit, BH), vlf::kThreads, cols_smem, st>>>(p);
    vlf::vlf_reduce<<<dim3(p.T, BH), D, 0, st>>>(p.part0, l.nsplit, (int)BH, p.H, p.T, D, p.out_l);
    g_launches.fetch_add(4, std::memory_order_relaxed);
    return cudaGetLastError();
}

template <int D, class T>
cudaError_t vlf_backward_launch(const vlf::ParamsT<T> &p, const VlfLayout &l, void (*rows_k)(vlf::ParamsT<T>),
                                int rows_smem, void (*cols_k)(vlf::ParamsT<T>), int cols_smem, cudaStream_t st) {
    cudaError_t e;
    if ((e = cudaFuncSetAttribute(rows_k, cudaFuncAttributeMaxDynamicSharedMemorySize, rows_smem)) ||
        (e = cudaFuncSetAttribute(cols_k, cudaFuncAttributeMaxDynamicSharedMemorySize, cols_smem)))
        return e;
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
        return vlf_forward_launch<D>(p, l, vlf::vlf_tc_fwd_rows<D>, vlf::FwdRowsSmem<vlf::Tf32>::kBytes,
                                     vlf::vlf_tc_fwd_cols<D>, vlf::FwdColsSmem<vlf::Tf32>::kBytes, st);
    return vlf_forward_launch<D>(p, l, vlf::vlf_fwd_rows<D>, vlf::kFwdRowsSmem, vlf::vlf_fwd_cols<D>, vlf::kFwdColsSmem, st);
}
template <int D>
cudaError_t vlf_forward_mode(const vlf::ParamsH &p, const VlfLayout &l, VlfMode, cudaStream_t st) {
    return vlf_forward_launch<D>(p, l, vlf::vlf_bf16_fwd_rows<D>, vlf::FwdRowsSmem<vlf::Bf16>::kBytes,
                                 vlf::vlf_bf16_fwd_cols<D>, vlf::FwdColsSmem<vlf::Bf16>::kBytes, st);
}
template <int D>
cudaError_t vlf_backward_mode(const vlf::Params &p, const VlfLayout &l, VlfMode mode, cudaStream_t st) {
    if (mode == kVlfTF32)
        return vlf_backward_launch<D>(p, l, vlf::vlf_tc_bwd_rows<D>, vlf::BwdRowsSmem<vlf::Tf32>::kBytes,
                                      vlf::vlf_tc_bwd_cols<D>, vlf::BwdColsSmem<vlf::Tf32>::kBytes, st);
    return vlf_backward_launch<D>(p, l, vlf::vlf_bwd_rows<D>, vlf::kBwdRowsSmem, vlf::vlf_bwd_cols<D>, vlf::kBwdColsSmem,
                                  st);
}
template <int D>
cudaError_t vlf_backward_mode(const vlf::ParamsH &p, const VlfLayout &l, VlfMode, cudaStream_t st) {
    return vlf_backward_launch<D>(p, l, vlf::vlf_bf16_bwd_rows<D>, vlf::BwdRowsSmem<vlf::Bf16>::kBytes,
                                  vlf::vlf_bf16_bwd_cols<D>, vlf::BwdColsSmem<vlf::Bf16>::kBytes, st);
}

// The tensors' element type behind an ABI pointer type: float, or bf16 passed as uint16_t.
template <class A> struct VlfElem { using type = float; };
template <> struct VlfElem<uint16_t> { using type = __nv_bfloat16; };

bool all_aligned16(std::initializer_list<const void *> ptrs) {
    for (const void *q : ptrs)
        if (!q || !aligned16(q)) return false;
    return true;
}

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
    vlf::vlf_dropout_mask<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(seed, B * H, S, T, dropout_p, mask_v, mask_l);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return (int)cudaGetLastError();
}

}  // extern "C"
