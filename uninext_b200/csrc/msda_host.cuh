// msda_host.cuh -- host-side plumbing shared by the C-ABI translation units (msda_cabi*.cu) and the GEMM: the launch
// counter, per-device caches, environment flags and launch helpers.  Host code only: no kernels.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <cstdlib>
#include <initializer_list>
#include <utility>

namespace msda_host {

// Kernel launches counted by msda_launch_count() (defined in msda_cabi.cu).  The GEMM does not count.
extern std::atomic<uint64_t> g_launches;

inline bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
inline bool aligned8(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 7u) == 0; }
inline bool all_aligned16(std::initializer_list<const void *> ptrs) {       // and non-null
    for (const void *q : ptrs)
        if (!q || !aligned16(q)) return false;
    return true;
}

inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

inline int env_int(const char *name, int dflt) {
    const char *e = getenv(name);
    return (e && e[0]) ? atoi(e) : dflt;
}

// A 0 / 1 switch from the environment: its value when the variable starts with '0' or '1', else -1.  Callers keep the
// result in a function-local static: these switches are read once per process.
inline int env_flag(const char *name) {
    const char *e = getenv(name);
    return (e && (e[0] == '0' || e[0] == '1')) ? e[0] - '0' : -1;
}

// Per-device caches (a process may drive several GPUs: SM counts, occupancy and function attributes are per device).
constexpr int kMaxDevices = 64;

inline int current_device() {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) dev = 0;
    return dev;
}

// A value derived once per device: get(init) returns the cached value, or calls init(dev) and caches what it returns
// while the slot holds T{} ("not derived yet") or fails `fresh`.  An init that fails returns T{}, so the next call
// retries.
template <class T>
struct PerDevice {
    std::atomic<T> slot[kMaxDevices];
    template <class F, class Fresh>
    T get(F init, Fresh fresh) {
        const int dev = current_device();
        T v = slot[dev].load(std::memory_order_relaxed);
        if (v == T{} || !fresh(v)) {
            v = init(dev);
            slot[dev].store(v, std::memory_order_relaxed);
        }
        return v;
    }
    template <class F>
    T get(F init) { return get(init, [](T) { return true; }); }
};

inline int num_sms() {
    static PerDevice<int> sms;
    return sms.get([](int dev) {
        int v = 0;
        if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;
        return v;
    });
}

// Dynamic shared memory above 48 KB needs a per-(kernel, device) opt-in.  It is set when `bytes` differs from what was
// last set for this kernel on this device, so a kernel launched at one fixed size sets it once per device.
// The kernel is a template argument so that each kernel has a cache of its own (kernels share function types).
template <auto Kernel>
cudaError_t opt_in_smem(int bytes) {
    static PerDevice<int> set;
    cudaError_t e = cudaSuccess;
    set.get([&](int) { e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
                       return e == cudaSuccess ? bytes : 0; },
            [&](int v) { return v == bytes; });
    return e;
}

// ceil(n / per_block) blocks, at most k per SM: grid-stride kernels.
inline int capped_grid(long long n, long long per_block, int k) {
    const long long blocks = (n + per_block - 1) / per_block, cap = (long long)num_sms() * k;
    return (int)(blocks < cap ? blocks : cap);
}

// One counted launch: msda_launch_count() goes up by one whether or not the launch succeeds.
template <class... P, class... A>
cudaError_t launch(void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, A &&...args) {
    kernel<<<grid, block, smem, st>>>(std::forward<A>(args)...);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return cudaGetLastError();
}

}  // namespace msda_host
