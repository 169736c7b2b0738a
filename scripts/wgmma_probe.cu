// The tensor-pipe rate of m64nNk16 wgmma (A from registers, B from a 128-byte-swizzled shared tile) for N = 32, 64, 128
// on the skeleton of the fused solve's field product (solve_tc.cu: wg::field) at config 3's grid: 1,024 CTAs of one
// warpgroup, 1,020 stages, per stage the six split products over all 256 columns onto two alternating accumulators.
// No contraction and no Runge-Kutta work: each stage only folds its accumulators into one running sum, and the next
// stage's A fragments depend on that sum, so the stages of a warpgroup are serial as in the solve.  The residency (CTAs
// per SM) is capped with the dynamic shared-memory size; the registers allow 3 per SM only at N = 32 (at the 168-register
// cap of __launch_bounds__(128, 3) ptxas serializes the N >= 64 probe's wgmmas), and the runtime's occupancy is reported
// beside every time.  Built as its own small library by torchcde_b200/csrc/Makefile; scripts/wgmma_probe.py loads it.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace {

constexpr int kCols = 256;
constexpr int kTile = kCols * 128;               // prepare_b<1>'s tile: [256 rows][hi 32 | lo 32 halves]

__device__ __forceinline__ uint64_t desc_sw128(uint32_t addr) {
    return (uint64_t)((addr & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}

template <int N> __device__ __forceinline__ void mma(float* d, const uint32_t* a, uint64_t b);
template <> __device__ __forceinline__ void mma<32>(float* d, const uint32_t* a, uint64_t b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b));
}
template <> __device__ __forceinline__ void mma<64>(float* d, const uint32_t* a, uint64_t b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
        "%24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b));
}
template <> __device__ __forceinline__ void mma<128>(float* d, const uint32_t* a, uint64_t b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
        "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, "
        "%46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "{%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
          "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
          "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
          "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
          "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b));
}

__device__ __forceinline__ void mma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void mma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int W> __device__ __forceinline__ void mma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(W) : "memory"); }

template <int N>
__global__ void __launch_bounds__(128, 2) probe_kernel(float* out, int stages) {
    constexpr int kAcc = N / 2, kChunks = kCols / N;
    extern __shared__ unsigned char smem_unaligned[];
    const uint32_t base = (uint32_t)__cvta_generic_to_shared(smem_unaligned);
    unsigned char* smem = smem_unaligned + ((1024u - (base & 1023u)) & 1023u);
    const int tid = threadIdx.x;
    __half* bt = reinterpret_cast<__half*>(smem);
    for (int e = tid; e < kTile / 2; e += 128) bt[e] = __float2half_rn((float)((e * 37 + blockIdx.x) & 255) * (1.f / 256.f));
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    const uint32_t b_tile = (uint32_t)__cvta_generic_to_shared(smem);

    float acc[2][kAcc];
    float sum = 0.f;
    for (int st = 0; st < stages; ++st) {
        // A fragments built afresh every stage from the previous stage's result, as the solve builds them from its state
        const uint32_t flip = __float_as_uint(sum) & 1u;
        uint32_t ahi[2][4], alo[2][4];
#pragma unroll
        for (int k = 0; k < 2; ++k)
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                ahi[k][t] = (0x3c003c00u ^ (uint32_t)(tid + 8 * k + t)) ^ flip;
                alo[k][t] = (0x14001400u ^ (uint32_t)(tid * 3 + k + t)) ^ flip;
            }
        auto issue = [&](int chunk, float* d) {
#pragma unroll
            for (int i = 0; i < kAcc; ++i) d[i] = 0.f;
            mma_fence();
            const uint32_t rows = b_tile + chunk * N * 128;
            mma<N>(d, alo[0], desc_sw128(rows + 0));
            mma<N>(d, alo[1], desc_sw128(rows + 32));
            mma<N>(d, ahi[0], desc_sw128(rows + 64));
            mma<N>(d, ahi[1], desc_sw128(rows + 96));
            mma<N>(d, ahi[0], desc_sw128(rows + 0));
            mma<N>(d, ahi[1], desc_sw128(rows + 32));
            mma_commit();
        };
        issue(0, acc[0]);
#pragma unroll
        for (int c = 0; c < kChunks; ++c) {
            float* d = acc[c & 1];
            if (c + 1 < kChunks) {
                issue(c + 1, acc[(c + 1) & 1]);
                mma_wait<1>();
            } else {
                mma_wait<0>();
            }
#pragma unroll
            for (int i = 0; i < kAcc; ++i) asm volatile("" : "+f"(d[i])::"memory");
#pragma unroll
            for (int i = 0; i < kAcc; ++i) sum += d[i];
        }
    }
    out[blockIdx.x * 128 + tid] = sum;
}

template <int N>
int run(int ctas_per_sm, int n_ctas, int stages, int reps, float* ms, int* resident) {
    // a dynamic shared-memory size that admits ctas_per_sm CTAs and not one more (228 KB per SM, 1 KB per CTA reserved)
    const int smem = ctas_per_sm == 2 ? 100 * 1024 : ctas_per_sm == 3 ? 64 * 1024 : 0;
    if (smem == 0) return 1;
    if (cudaFuncSetAttribute(probe_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) return 2;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(resident, probe_kernel<N>, 128, smem) != cudaSuccess) return 3;
    float* out = nullptr;
    if (cudaMalloc(&out, (size_t)n_ctas * 128 * sizeof(float)) != cudaSuccess) return 4;
    cudaEvent_t a, b;
    cudaEventCreate(&a);
    cudaEventCreate(&b);
    probe_kernel<N><<<n_ctas, 128, smem>>>(out, stages);                  // warm-up
    for (int r = 0; r < reps; ++r) {
        cudaEventRecord(a);
        probe_kernel<N><<<n_ctas, 128, smem>>>(out, stages);
        cudaEventRecord(b);
        cudaEventSynchronize(b);
        cudaEventElapsedTime(ms + r, a, b);
    }
    const cudaError_t err = cudaDeviceSynchronize();
    cudaEventDestroy(a);
    cudaEventDestroy(b);
    cudaFree(out);
    return err == cudaSuccess ? 0 : 5;
}

}  // namespace

// Times `reps` launches of the probe with chunk width n (32, 64 or 128) at ctas_per_sm (2 or 3) into ms[reps]; resident
// receives the occupancy the runtime reports for that configuration.  Returns 0 on success.
extern "C" __attribute__((visibility("default"))) int wgmma_probe(int n, int ctas_per_sm, int n_ctas, int stages, int reps, float* ms, int* resident) {
    switch (n) {
        case 32: return run<32>(ctas_per_sm, n_ctas, stages, reps, ms, resident);
        case 64: return run<64>(ctas_per_sm, n_ctas, stages, reps, ms, resident);
        case 128: return run<128>(ctas_per_sm, n_ctas, stages, reps, ms, resident);
        default: return 1;
    }
}
