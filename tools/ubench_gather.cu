// Micro-benchmark: what does one SM sustain for "4 rows x 128 B per LDG.128" gathers (the op's access shape)?
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/ubench_gather tools/ubench_gather.cu
// Prints cycles per LDG.128 warp-instruction per SM for several table sizes (L1-resident ... L2-resident), for
// 8-lane x 16 B (fp32 rows) and 4-lane x 16 B (bf16 rows) and 32-lane x 4 B (reference-style scalar) shapes.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

template <int LANES_PER_ROW, int UNROLL>
__global__ void __launch_bounds__(256) gather(const float4 *__restrict__ table, unsigned rows, unsigned row_f4,
                                              int iters, float *out, unsigned seed) {
    const int lane = threadIdx.x & 31;
    const int sub = lane % LANES_PER_ROW, grp = lane / LANES_PER_ROW;
    unsigned s = seed + (blockIdx.x * blockDim.x + threadIdx.x) / LANES_PER_ROW * 2654435761u + grp * 40503u;
    float acc = 0.f;
    for (int it = 0; it < iters; ++it) {
        float4 v[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            s = s * 1664525u + 1013904223u;
            const unsigned r = (unsigned)(((unsigned long long)(s >> 4) * rows) >> 28);
            v[u] = __ldg(table + (size_t)r * row_f4 + sub);
        }
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) acc += v[u].x + v[u].y + v[u].z + v[u].w;
    }
    if (acc == 123.456f) out[0] = acc;
}

// scatter: red.global.add.v4.f32 of 4 rows x 128 B per warp instruction (the backward's grad_value traffic),
// optionally interleaved 1:1 with LDG.128 gathers (the backward does both per tap).
template <int UNROLL, bool WITH_LOADS>
__global__ void __launch_bounds__(256) scatter(float *table, const float4 *__restrict__ rd, unsigned rows, int iters,
                                               float *out, unsigned seed) {
    const int lane = threadIdx.x & 31;
    const int sub = lane % 8, grp = lane / 8;
    unsigned s = seed + (blockIdx.x * blockDim.x + threadIdx.x) / 8 * 2654435761u + grp * 40503u;
    float acc = 0.f;
    for (int it = 0; it < iters; ++it) {
        float4 v[UNROLL];
        unsigned r[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            s = s * 1664525u + 1013904223u;
            r[u] = (unsigned)(((unsigned long long)(s >> 4) * rows) >> 28);
            if (WITH_LOADS) v[u] = __ldg(rd + (size_t)r[u] * 8 + sub);
        }
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            float x = WITH_LOADS ? v[u].x : 1.f;
            acc += x;
            float *a = table + ((size_t)r[u] * 8 + sub) * 4;
            asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(a), "f"(x), "f"(1.f), "f"(2.f), "f"(3.f) : "memory");
        }
    }
    if (acc == 123.456f) out[0] = acc;
}

template <int UNROLL, bool WITH_LOADS>
void run_scatter(const char *name, float *tab, const float4 *rd, size_t table_bytes, int ctas_per_sm) {
    const unsigned rows = (unsigned)(table_bytes / 128);
    int sms; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    float *out; cudaMalloc(&out, 4);
    const int iters = 1000 / UNROLL * 4;
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    scatter<UNROLL, WITH_LOADS><<<sms * ctas_per_sm, 256>>>(tab, rd, rows, 10, out, 1u);
    cudaDeviceSynchronize();
    cudaEventRecord(e0);
    scatter<UNROLL, WITH_LOADS><<<sms * ctas_per_sm, 256>>>(tab, rd, rows, iters, out, 7u);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    const double n_per_sm = (double)ctas_per_sm * 8 * iters * UNROLL;
    const double cycles = ms * 1e-3 * 1.965e9;
    printf("%-34s table %8.1f MB  ctas/sm %d : %6.2f cyc per RED.128%s per SM   %6.2f TB/s red payload\n", name,
           table_bytes / 1e6, ctas_per_sm, cycles / n_per_sm, WITH_LOADS ? " (+1 LDG.128)" : "",
           n_per_sm * sms * 512.0 / (ms * 1e-3) / 1e12);
    cudaFree(out);
}

template <int LPR, int UNROLL>
void run(const char *name, const float4 *tab, size_t table_bytes, int ctas_per_sm) {
    const unsigned row_f4 = LPR;                       // row = LPR float4 = LPR*16 bytes
    const unsigned rows = (unsigned)(table_bytes / (LPR * 16));
    int sms; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    int clk; cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0);
    float *out; cudaMalloc(&out, 4);
    const int iters = 2000 / UNROLL * 4;
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    gather<LPR, UNROLL><<<sms * ctas_per_sm, 256>>>(tab, rows, row_f4, 10, out, 1u);
    cudaDeviceSynchronize();
    cudaEventRecord(e0);
    gather<LPR, UNROLL><<<sms * ctas_per_sm, 256>>>(tab, rows, row_f4, iters, out, 7u);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    const double ldg_per_sm = (double)ctas_per_sm * 8 * iters * UNROLL;
    const double cycles = ms * 1e-3 * 1.965e9;          // at max SM clock
    const double bytes = ldg_per_sm * sms * 512.0;
    printf("%-28s table %8.1f MB  ctas/sm %d unroll %2d : %6.2f cyc/LDG.128/SM  %7.1f B/clk/SM  %6.2f TB/s\n", name,
           table_bytes / 1e6, ctas_per_sm, UNROLL, cycles / ldg_per_sm, 512.0 * ldg_per_sm / cycles, bytes / (ms * 1e-3) / 1e12);
    cudaFree(out);
}

int main() {
    float4 *tab; size_t maxb = 256u << 20;
    cudaMalloc(&tab, maxb); cudaMemset(tab, 0, maxb);
    const size_t sizes[] = {32u << 10, 128u << 10, 8u << 20, 46u << 20, 256u << 20};
    for (size_t sz : sizes) {
        run<8, 8>("8 lanes/row (fp32 D=32)", tab, sz, 4);
        run<8, 16>("8 lanes/row (fp32 D=32)", tab, sz, 2);
        run<4, 8>("4 lanes/row (bf16 D=32)", tab, sz, 4);
        run<32, 8>("32 lanes/row (512 B rows)", tab, sz, 4);
        run<1, 8>("1 lane/row (16 B rows)", tab, sz, 4);
    }
    float *acc; cudaMalloc(&acc, 64u << 20); cudaMemset(acc, 0, 64u << 20);
    for (int c : {2, 4}) {
        run_scatter<8, false>("red.v4.f32 scatter only", acc, tab, 46u << 20, c);
        run_scatter<8, true>("red.v4.f32 scatter + gather", acc, tab, 46u << 20, c);
    }
    return 0;
}
