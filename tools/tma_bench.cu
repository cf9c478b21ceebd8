// tma_bench.cu -- microbenchmark: how fast can a persistent CTA-per-SM kernel stream a [B, C, g] fp32 tensor
// through shared memory with TMA tensor copies, as a function of box shape / stages / boxes per tile.
// Consumers only wait + release (no compute), so this is the copy-engine ceiling for the scan kernel.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/tma_bench tools/tma_bench.cu
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* b, uint32_t c) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(c)); }
__device__ __forceinline__ void mbar_expect(uint64_t* b, uint32_t tx) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(tx) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(b)) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t* b, uint32_t parity) {
    uint32_t done;
    do {
        asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n" : "=r"(done) : "r"(smem_u32(b)), "r"(parity) : "memory");
    } while (!done);
}
__device__ __forceinline__ void tma3d(void* dst, const CUtensorMap* m, int c0, int c1, int c2, uint64_t* bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(smem_u32(dst)), "l"(m), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar)) : "memory");
}

// tile = [C rows x cols] ; loaded as `nbox` boxes of [C/nbox rows x cols]
__global__ void __launch_bounds__(160, 1) stream_kernel(const __grid_constant__ CUtensorMap map, int tiles_per_image, int total_tiles,
                                                        int C, int cols, int nbox, int stages, int touch, float* sink) {
    extern __shared__ __align__(1024) unsigned char smem[];
    const int stage_bytes = C * cols * 4;
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)stages * stage_bytes);
    uint64_t* empty = full + 8;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 4); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (warp == 4) {
        if (lane == 0) {
            int it = 0;
            for (int T = blockIdx.x; T < total_tiles; T += gridDim.x, ++it) {
                const int s = it % stages; const uint32_t ph = (it / stages) & 1;
                mbar_wait(&empty[s], ph ^ 1);
                const int b = T / tiles_per_image, t = T % tiles_per_image;
                mbar_expect(&full[s], stage_bytes);
                const int rows = C / nbox;
                for (int k = 0; k < nbox; ++k)
                    tma3d(smem + (size_t)s * stage_bytes + (size_t)k * rows * cols * 4, &map, t * cols, k * rows, b, &full[s]);
            }
        }
        return;
    }
    float acc = 0.f;
    int it = 0;
    for (int T = blockIdx.x; T < total_tiles; T += gridDim.x, ++it) {
        const int s = it % stages; const uint32_t ph = (it / stages) & 1;
        mbar_wait(&full[s], ph);
        if (touch) {
            const float4* p = reinterpret_cast<const float4*>(smem + (size_t)s * stage_bytes);
            const int n4 = stage_bytes / 16;
            for (int i = threadIdx.x; i < n4; i += 128) { float4 v = p[i]; acc += v.x + v.y + v.z + v.w; }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);
    }
    if (acc == 123.456f) sink[0] = acc;
}

typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                             const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int main() {
    const int B = 32, C = 84, g = 8192;  // 88 MB
    const size_t n = (size_t)B * C * g;
    float* d; cudaMalloc(&d, n * 4 * 4);  // 4 copies to rotate (> L2)
    cudaMemset(d, 0, n * 4 * 4);
    float* sink; cudaMalloc(&sink, 4);
    void* fp; cudaDriverEntryPointQueryResult q;
    cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &q);
    EncodeFn enc = (EncodeFn)fp;
    int sms; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    cudaFuncSetAttribute(stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
    struct Cfg { int cols, nbox, stages, touch, promo; };
    Cfg cfgs[] = {{128, 1, 4, 0, 2}, {128, 1, 4, 1, 2}, {128, 1, 2, 0, 2}, {128, 2, 4, 0, 2}, {128, 4, 4, 0, 2}, {128, 12, 4, 0, 2},
                  {128, 84, 4, 0, 2}, {64, 1, 8, 0, 2}, {32, 1, 8, 0, 2}, {256, 1, 2, 0, 2}, {128, 1, 4, 0, 0}, {128, 1, 4, 0, 1}, {128, 1, 4, 0, 3},
                  {32, 1, 16, 0, 2}, {64, 2, 8, 1, 2}};
    for (auto c : cfgs) {
        const int stage_bytes = C * c.cols * 4;
        int stages = c.stages;
        while ((size_t)stages * stage_bytes + 256 > 220 * 1024) --stages;
        if (stages > 8) stages = 8;
        CUtensorMap maps[4];
        for (int r = 0; r < 4; ++r) {
            cuuint64_t gd[3] = {(cuuint64_t)g, (cuuint64_t)C, (cuuint64_t)B};
            cuuint64_t gs[2] = {(cuuint64_t)g * 4, (cuuint64_t)C * g * 4};
            cuuint32_t box[3] = {(cuuint32_t)c.cols, (cuuint32_t)(C / c.nbox), 1};
            cuuint32_t es[3] = {1, 1, 1};
            CUresult rc = enc(&maps[r], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, d + r * n, gd, gs, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                              CU_TENSOR_MAP_SWIZZLE_NONE, (CUtensorMapL2promotion)c.promo, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (rc != CUDA_SUCCESS) { printf("encode failed %d\n", (int)rc); return 1; }
        }
        const int tpi = g / c.cols, total = B * tpi;
        const size_t smem = (size_t)stages * stage_bytes + 256;
        cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
        for (int i = 0; i < 4; ++i) stream_kernel<<<sms, 160, smem>>>(maps[i % 4], tpi, total, C, c.cols, c.nbox, stages, c.touch, sink);
        cudaDeviceSynchronize();
        const int K = 40;
        cudaEventRecord(e0);
        for (int i = 0; i < K; ++i) stream_kernel<<<sms, 160, smem>>>(maps[i % 4], tpi, total, C, c.cols, c.nbox, stages, c.touch, sink);
        cudaEventRecord(e1);
        cudaDeviceSynchronize();
        float ms; cudaEventElapsedTime(&ms, e0, e1);
        cudaError_t err = cudaGetLastError();
        printf("cols=%3d nbox=%2d stages=%d touch=%d promo=%d : %7.2f us  %7.1f GB/s  (%s)\n", c.cols, c.nbox, stages, c.touch, c.promo,
               ms / K * 1e3, n * 4.0 / (ms / K * 1e-3) / 1e9, cudaGetErrorString(err));
    }
    return 0;
}
