// Micro-benchmark: TMA bulk reduction (cp.reduce.async.bulk ... add.f32) of 128-byte rows from shared memory into random
// rows of an L2-resident fp32 table, vs the LSU path (red.global.add.v4.f32) measured by ubench_gather.cu.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/ubench_bulkred tools/ubench_bulkred.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }

// ROWS_PER_OP: how many 128-byte rows one bulk op covers (1 = the op's natural granularity; >1 only to see how the
// engine scales with op size -- contiguous rows, not usable by the op).
template <int ROWS_PER_OP, int DEPTH>
__global__ void __launch_bounds__(256) bulkred(float *table, unsigned rows, int iters, unsigned seed) {
    extern __shared__ __align__(128) unsigned char smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // per warp: DEPTH stages x 16 rows x 128 B
    float *stage = reinterpret_cast<float *>(smem) + (size_t)warp * DEPTH * 16 * 32;
    for (int i = lane; i < DEPTH * 16 * 32; i += 32) stage[i] = 1.0f;
    __syncwarp();
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    unsigned s = seed + (blockIdx.x * blockDim.x + threadIdx.x) * 2654435761u;
    for (int it = 0; it < iters; ++it) {
        const int st = it % DEPTH;
        // recycle: wait until the bulk ops issued DEPTH-1 iterations ago have finished READING shared memory
        asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(DEPTH - 1) : "memory");
        // (a real kernel would now overwrite stage `st` with 16 new payload rows: 16 x STS.128 per warp)
        float4 *dst = reinterpret_cast<float4 *>(stage + (size_t)st * 16 * 32);
        dst[lane] = make_float4(1.f, 2.f, 3.f, 4.f);
        dst[lane + 32] = make_float4(1.f, 2.f, 3.f, 4.f);
        dst[lane + 64] = make_float4(1.f, 2.f, 3.f, 4.f);
        dst[lane + 96] = make_float4(1.f, 2.f, 3.f, 4.f);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncwarp();
        s = s * 1664525u + 1013904223u;
        if (lane < 16 / ROWS_PER_OP) {
            const unsigned r = (unsigned)(((unsigned long long)(s >> 4) * (rows - ROWS_PER_OP)) >> 28);
            float *g = table + (size_t)r * 32;
            const float *src = stage + ((size_t)st * 16 + lane * ROWS_PER_OP) * 32;
            asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f32 [%0], [%1], %2;"
                         ::"l"(g), "r"(smem_u32(src)), "n"(128 * ROWS_PER_OP) : "memory");
        }
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

template <int ROWS_PER_OP, int DEPTH>
void run(float *tab, size_t table_bytes, int ctas_per_sm) {
    const unsigned rows = (unsigned)(table_bytes / 128);
    int sms; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    const int iters = 2000;
    const size_t smem = 8 * DEPTH * 16 * 128;
    cudaFuncSetAttribute(bulkred<ROWS_PER_OP, DEPTH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    bulkred<ROWS_PER_OP, DEPTH><<<sms * ctas_per_sm, 256, smem>>>(tab, rows, 10, 1u);
    cudaError_t err = cudaDeviceSynchronize();
    if (err != cudaSuccess) { printf("launch failed: %s\n", cudaGetErrorString(err)); return; }
    cudaEventRecord(e0);
    bulkred<ROWS_PER_OP, DEPTH><<<sms * ctas_per_sm, 256, smem>>>(tab, rows, iters, 7u);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    const double rows_per_sm = (double)ctas_per_sm * 8 * iters * 16;
    const double cycles = ms * 1e-3 * 1.965e9;
    printf("bulk reduce %4d B/op depth %d ctas/sm %d : %6.2f cyc per 128-B row per SM   %6.2f TB/s payload   (LSU red.v4 path: 5.8 cyc/row, 6.4 TB/s)\n",
           128 * ROWS_PER_OP, DEPTH, ctas_per_sm, cycles / rows_per_sm, rows_per_sm * sms * 128.0 / (ms * 1e-3) / 1e12);
}

int main() {
    float *tab; cudaMalloc(&tab, 64u << 20); cudaMemset(tab, 0, 64u << 20);
    run<1, 2>(tab, 46u << 20, 2);
    run<1, 4>(tab, 46u << 20, 2);
    run<1, 4>(tab, 46u << 20, 4);
    run<2, 4>(tab, 46u << 20, 2);
    run<4, 4>(tab, 46u << 20, 2);
    run<16, 4>(tab, 46u << 20, 2);
    return 0;
}
