// msda_gemm_sm90.cu -- hand-written Hopper GEMM for the Linears that bracket the op:
//     C[M, N] = A[M, K] . W[N, K]^T + bias[N]        (fp32 in/out, TF32 wgmma, fp32 accumulation in registers)
// with an optional fused tail: rows with row_mask[m] != 0 written as zeros (value_proj's padding mask,
// ops/modules/ms_deform_attn.py:96-97) and ReLU (FFN linear1).
//
// Shape regime: M = N_batch * S tokens (tens of thousands), K = d_model (256), N in {256, 384}.  Memory-bound: A is read
// once, C written once, the W tile (<= 256 KB) is re-read by every CTA from L2.
//
// Structure (persistent; one CTA = 128-row x BN-column tiles of C walked with a grid stride):
//   warp 8     : TMA producer -- one lane issues cp.async.bulk.tensor 2D loads of A[128 x 32] and W[BN x 32] (128-byte
//                rows, SWIZZLE_128B) into a ring of shared-memory stages, completion on mbarriers (full / empty).  The ring
//                runs across tiles, so the next tile's loads stream while the consumers run the epilogue.
//   warps 0-7  : two consumer warpgroups, 64 rows each: wgmma.mma_async m64nBNk8 (TF32, both operands K-major from
//                shared memory), 4 per 32-wide k-block, accumulators in registers; then bias / mask / ReLU and 8-byte
//                stores straight from the accumulator fragments (each quad of lanes writes one 32-byte sector of a row).
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <mutex>

#include "../../include/msda_b200.h"

extern std::atomic<uint64_t> g_msda_gemm_launches;
std::atomic<uint64_t> g_msda_gemm_launches{0};

namespace gemm {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 32;                 // fp32 elements = 128 bytes = one swizzle row
constexpr int MMA_K = 8;                    // tf32: 32 bytes per instruction
constexpr int kConsumers = 8;               // warps 0-7: two warpgroups
constexpr int kThreads = 32 * kConsumers + 32;
constexpr int kMaxStages = 8;
constexpr int kSmemMax = 232448;            // sm_90 opt-in shared memory per block (227 KB)

__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, unsigned parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "W_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra D_%=;\n\t"
        "bra W_%=;\n\t"
        "D_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void *dst, const CUtensorMap *map, int c0, int c1, uint64_t *bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(smem_u32(dst)), "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar)) : "memory");
}

// K-major, SWIZZLE_128B shared-memory matrix descriptor of sm_90 wgmma: start address >> 4 in bits [0,14), leading byte
// offset [16,30) (unused for swizzled K-major: 1), stride byte offset [32,46) = 1024 B between 8-row groups, layout type
// SWIZZLE_128B = 1 at [62,64).  The operand tiles start 1024-byte aligned; the k-th 8-wide slice of a 128-byte row is
// addressed by adding k * 32 bytes to the start address (the swizzle is applied to the absolute address bits).
__device__ __forceinline__ uint64_t wgmma_desc(const void *smem) {
    const uint64_t addr = smem_u32(smem) >> 4;
    return (addr & 0x3fffull) | (1ull << 16) | ((1024ull >> 4) << 32) | (1ull << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// m64nBNk8 TF32 wgmma: d (BN / 2 fp32 per thread) += A[64 x 8] . B[BN x 8]^T; accumulate = 0 overwrites d.
__device__ __forceinline__ void wgmma_tf32_n32(float (&d)[16], uint64_t adesc, uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
        "%16, %17, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_tf32_n64(float (&d)[32], uint64_t adesc, uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "%32, %33, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_tf32_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_tf32_n256(float (&d)[128], uint64_t adesc, uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
        "%128, %129, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

template <int BN> struct Wgmma;
template <> struct Wgmma<32> { template <class D> __device__ static void mma(D &d, uint64_t a, uint64_t b, int acc) { wgmma_tf32_n32(d, a, b, acc); } };
template <> struct Wgmma<64> { template <class D> __device__ static void mma(D &d, uint64_t a, uint64_t b, int acc) { wgmma_tf32_n64(d, a, b, acc); } };
template <> struct Wgmma<128> { template <class D> __device__ static void mma(D &d, uint64_t a, uint64_t b, int acc) { wgmma_tf32_n128(d, a, b, acc); } };
template <> struct Wgmma<256> { template <class D> __device__ static void mma(D &d, uint64_t a, uint64_t b, int acc) { wgmma_tf32_n256(d, a, b, acc); } };

struct Params {
    long long M;
    int N, K, stages, relu;
    const float *bias;
    const unsigned char *row_mask;      // [M] bytes, non-zero = zero the whole output row; may be null
    float *C;
};

template <int BN>
__global__ void __launch_bounds__(kThreads, 1)
linear_tf32_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_w, const Params p)
{
    extern __shared__ unsigned char smem_raw[];
    // SWIZZLE_128B atoms (8 rows x 128 B) must start 1024-byte aligned
    unsigned char *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    __shared__ __align__(8) uint64_t full_bar[kMaxStages], empty_bar[kMaxStages];

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int KB = p.K / BLOCK_K;
    constexpr unsigned a_bytes = BLOCK_M * BLOCK_K * 4, w_bytes = BN * BLOCK_K * 4, stage_bytes = a_bytes + w_bytes;
    const long long mtiles = (p.M + BLOCK_M - 1) / BLOCK_M;
    const int ntiles_n = p.N / BN;
    const long long ntiles = mtiles * ntiles_n;

    if (threadIdx.x == 0) {
        for (int s = 0; s < p.stages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kConsumers); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == kConsumers) {
        // ===== TMA producer =====
        if (lane == 0) {
            asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
            asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w) : "memory");
            unsigned s = 0, ph = 0;                                      // ring position across tiles (no div / mod)
            for (long long t = blockIdx.x; t < ntiles; t += gridDim.x) {
                const int row0 = (int)((t / ntiles_n) * BLOCK_M);       // may reach beyond M: TMA zero-fills
                const int col0 = (int)(t % ntiles_n) * BN;
                for (int kb = 0; kb < KB; ++kb) {
                    mbar_wait(&empty_bar[s], ph ^ 1);                    // every consumer warp has drained this stage
                    unsigned char *sa = smem + (size_t)s * stage_bytes;
                    mbar_expect_tx(&full_bar[s], stage_bytes);
                    tma_load_2d(sa, &map_a, kb * BLOCK_K, row0, &full_bar[s]);
                    tma_load_2d(sa + a_bytes, &map_w, kb * BLOCK_K, col0, &full_bar[s]);
                    if (++s == (unsigned)p.stages) { s = 0; ph ^= 1u; }
                }
            }
        }
        return;
    }

    // ===== consumers: warpgroup wg owns rows [64 wg, 64 wg + 64) of every tile =====
    const int wg = warp >> 2;
    const uint64_t a_desc0 = wgmma_desc(smem + wg * (64 * BLOCK_K * 4)), w_desc0 = wgmma_desc(smem + a_bytes);
    constexpr uint32_t st_step = stage_bytes >> 4, k_step = (MMA_K * 4) >> 4;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    unsigned s = 0, ph = 0;
    for (long long t = blockIdx.x; t < ntiles; t += gridDim.x) {
        for (int kb = 0; kb < KB; ++kb) {
            mbar_wait(&full_bar[s], ph);
            wgmma_fence();
            const uint64_t ad = a_desc0 + (uint64_t)(s * st_step), wd = w_desc0 + (uint64_t)(s * st_step);
#pragma unroll
            for (int k = 0; k < BLOCK_K / MMA_K; ++k)
                Wgmma<BN>::mma(acc, ad + (uint64_t)(k * k_step), wd + (uint64_t)(k * k_step), (kb | k) != 0);
            wgmma_commit();
            wgmma_wait0();
            if (lane == 0) mbar_arrive(&empty_bar[s]);                   // this warp's share of the stage has been read
            if (++s == (unsigned)p.stages) { s = 0; ph ^= 1u; }
        }
        // epilogue from the accumulator fragments: d[4j + {0,1}] = (row, 8j + 2 (lane % 4) + {0,1}), d[4j + {2,3}] = row + 8
        const long long r0 = (t / ntiles_n) * BLOCK_M + wg * 64 + (warp & 3) * 16 + (lane >> 2), r1 = r0 + 8;
        const int c0 = (int)(t % ntiles_n) * BN + 2 * (lane & 3);
        const bool live0 = r0 < p.M, live1 = r1 < p.M;
        const bool dead0 = live0 && p.row_mask != nullptr && p.row_mask[r0] != 0;
        const bool dead1 = live1 && p.row_mask != nullptr && p.row_mask[r1] != 0;
        float *c_r0 = p.C + (live0 ? r0 : 0) * (long long)p.N + c0, *c_r1 = p.C + (live1 ? r1 : 0) * (long long)p.N + c0;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            const float2 b = p.bias != nullptr ? __ldg(reinterpret_cast<const float2 *>(p.bias + c0 + 8 * j)) : make_float2(0.f, 0.f);
            float o[4] = {acc[4 * j] + b.x, acc[4 * j + 1] + b.y, acc[4 * j + 2] + b.x, acc[4 * j + 3] + b.y};
            if (p.relu) {
#pragma unroll
                for (int e = 0; e < 4; ++e) o[e] = fmaxf(o[e], 0.f);
            }
            if (dead0) o[0] = o[1] = 0.f;
            if (dead1) o[2] = o[3] = 0.f;
            if (live0) *reinterpret_cast<float2 *>(c_r0 + 8 * j) = make_float2(o[0], o[1]);
            if (live1) *reinterpret_cast<float2 *>(c_r1 + 8 * j) = make_float2(o[2], o[3]);
        }
    }
}

// ---- host side -------------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    });
    return fn;
}

bool make_map(CUtensorMap *map, const float *base, long long rows, int K, int box_rows) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) return false;
    const cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)K * 4};
    const cuuint32_t box[2] = {(cuuint32_t)BLOCK_K, (cuuint32_t)box_rows};
    const cuuint32_t estr[2] = {1, 1};
    return fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float *>(base), dims, strides, box, estr,
              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// Fused-tail eligibility (msda_linear_tf32_ex): whole 64-column tiles up to N = 256.
bool ws_ok(int N, int K) { return N % 64 == 0 && N >= 64 && N <= 256 && K % BLOCK_K == 0 && K > 0; }

template <int BN>
int launch(const float *A, const float *W, const float *bias, const unsigned char *row_mask, long long M, int N, int K,
           int relu, float *C, cudaStream_t stream) {
    CUtensorMap map_a, map_w;
    if (!make_map(&map_a, A, M, K, BLOCK_M) || !make_map(&map_w, W, N, K, BN)) return MSDA_E_NODEVICE;
    constexpr size_t stage_bytes = (size_t)(BLOCK_M + BN) * BLOCK_K * 4;
    constexpr size_t dyn_max = kSmemMax - 1024;                 // static barriers + alignment slack
    int stages = (int)((dyn_max - 1024) / stage_bytes);
    if (stages > kMaxStages) stages = kMaxStages;
    Params p;
    p.M = M; p.N = N; p.K = K; p.stages = stages; p.relu = relu; p.bias = bias; p.row_mask = row_mask; p.C = C;
    const size_t smem = (size_t)stages * stage_bytes + 1024;
    // function attributes and SM counts are per DEVICE: cache them per ordinal (a process may drive several GPUs)
    constexpr int kMaxDev = 64;
    static std::atomic<int> sms_of[kMaxDev];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDev) dev = 0;
    int sms = sms_of[dev].load(std::memory_order_relaxed);
    if (sms == 0) {
        const cudaError_t e = cudaFuncSetAttribute(linear_tf32_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn_max);
        if (e != cudaSuccess) return (int)e;
        if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
        sms_of[dev].store(sms, std::memory_order_relaxed);
    }
    const long long tiles = (M + BLOCK_M - 1) / BLOCK_M * (N / BN);
    const unsigned grid = (unsigned)(tiles < sms ? tiles : sms);
    linear_tf32_kernel<BN><<<grid, kThreads, smem, stream>>>(map_a, map_w, p);
    g_msda_gemm_launches.fetch_add(1, std::memory_order_relaxed);
    return (int)cudaGetLastError();
}

// widest column tile (<= 256, the largest wgmma N) that divides N
int dispatch(const float *A, const float *W, const float *bias, const unsigned char *row_mask, long long M, int N, int K,
             int relu, float *C, cudaStream_t st) {
    if (N % 256 == 0) return launch<256>(A, W, bias, row_mask, M, N, K, relu, C, st);
    if (N % 128 == 0) return launch<128>(A, W, bias, row_mask, M, N, K, relu, C, st);
    if (N % 64 == 0) return launch<64>(A, W, bias, row_mask, M, N, K, relu, C, st);
    return launch<32>(A, W, bias, row_mask, M, N, K, relu, C, st);
}

bool aligned_operands(const float *A, const float *W, const float *bias, const float *C) {
    return !((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(W) | reinterpret_cast<uintptr_t>(C) |
              reinterpret_cast<uintptr_t>(bias)) & 15u);
}

}  // namespace gemm

extern "C" int msda_linear_tf32_ex(const float *A, const float *W, const float *bias, const uint8_t *row_mask, int64_t M, int N,
                                   int K, int relu, float *C, void *stream) {
    using namespace gemm;
    if (!A || !W || !C || M <= 0 || N <= 0 || K <= 0 || !aligned_operands(A, W, bias, C)) return MSDA_E_BADARG;
    if (!ws_ok(N, K)) return MSDA_E_BADARG;
    return dispatch(A, W, bias, row_mask, M, N, K, relu ? 1 : 0, C, static_cast<cudaStream_t>(stream));
}

extern "C" int msda_linear_tf32_ws_ok(int N, int K) { return gemm::ws_ok(N, K) ? 1 : 0; }

extern "C" int msda_linear_tf32(const float *A, const float *W, const float *bias, int64_t M, int N, int K, float *C,
                                void *stream) {
    using namespace gemm;
    if (!A || !W || !C || M <= 0 || N <= 0 || K <= 0 || K % BLOCK_K || N % 32 || N > 512) return MSDA_E_BADARG;
    if (N > 256 && (N % 64)) return MSDA_E_BADARG;
    if (!aligned_operands(A, W, bias, C)) return MSDA_E_BADARG;
    return dispatch(A, W, bias, nullptr, M, N, K, 0, C, static_cast<cudaStream_t>(stream));
}
