// lb_ceiling.cu -- what the card can do for the letterbox's byte stream at the benchmark shape (b32, 640x640x3 u8 -> 3x640x640
// fp32 planar), measured without the letterbox's arithmetic:
//   a  contiguous u8 -> fp32 expand with the letterbox's byte counts (39.3 MB read, 157.3 MB written): the letterbox's floor
//   b  a 90.3 MB read (the YOLOv8n b32 head tensors): the scan's floor
//   c  a || b as two chains of one CUDA graph, b on a high-priority stream, 4 steps per graph (as bench.py runs the step)
//   d  store patterns for the same planar output: 256-B pieces 4 rows apart (64 x 32 tiles), 512-B runs per warp (128 x 16
//      tiles), full-width row bands (every plane of a CTA one contiguous run), and row bands staged in shared memory and
//      written with TMA bulk stores
// Every kernel rotates over 4 buffer sets (> the 50 MB L2).  CUDA events around 200 launches.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/lb_ceiling tools/lb_ceiling.cu && tools/lb_ceiling
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

constexpr int B = 32, W = 640, H = 640;
constexpr size_t SRC_BYTES = (size_t)B * W * H * 3;   // 39 321 600
constexpr size_t OUT_FLOATS = SRC_BYTES;              // 3 planes x W x H per image
constexpr size_t HEAD_BYTES = (size_t)B * 84 * 8400 * 4;  // 90 316 800
constexpr int NSET = 4, LAUNCHES = 200;

#define CK(x)                                                                                 \
    do {                                                                                      \
        cudaError_t e_ = (x);                                                                 \
        if (e_ != cudaSuccess) {                                                              \
            fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); \
            exit(1);                                                                          \
        }                                                                                     \
    } while (0)

__device__ __forceinline__ float4 expand(uint32_t v) {
    return make_float4((float)(v & 255u), (float)((v >> 8) & 255u), (float)((v >> 16) & 255u), (float)(v >> 24));
}

// a: thread i of a 256-thread CTA converts words i, i+256, i+512, i+768 of the CTA's 4 KB: every warp store is 512 contiguous bytes
__global__ void __launch_bounds__(256) expand_contig(const uint32_t* __restrict__ src, float4* __restrict__ dst, size_t n) {
    const size_t base = (size_t)blockIdx.x * 1024 + threadIdx.x;
    uint32_t v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = base + j * 256 < n ? __ldg(src + base + j * 256) : 0u;
#pragma unroll
    for (int j = 0; j < 4; ++j)
        if (base + j * 256 < n) dst[base + j * 256] = expand(v[j]);
}

// b: read-only stream
__global__ void __launch_bounds__(256) read_only(const float4* __restrict__ src, size_t n, float* sink) {
    const size_t base = (size_t)blockIdx.x * 1024 + threadIdx.x;
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j)
        if (base + j * 256 < n) {
            const float4 v = __ldg(src + base + j * 256);
            acc += v.x + v.y + v.z + v.w;
        }
    if (acc == 123.456f) sink[0] = acc;
}

// d: planar output.  A thread owns 4 adjacent pixels of one image row: reads 3 words (12 source bytes = 4 BGR pixels) and
// writes one 16-byte store per plane.  `px` = first pixel of the 4, `row` = image row, `b` = image.
__device__ __forceinline__ void px4(const uint8_t* __restrict__ src, float* __restrict__ dst, int b, int row, int px) {
    const uint32_t* s = reinterpret_cast<const uint32_t*>(src + ((size_t)b * H + row) * W * 3 + (size_t)px * 3);
    const uint32_t w0 = __ldg(s), w1 = __ldg(s + 1), w2 = __ldg(s + 2);
    const float4 f0 = expand(w0), f1 = expand(w1), f2 = expand(w2);
    float* o = dst + (size_t)b * 3 * W * H + (size_t)row * W + px;
    *reinterpret_cast<float4*>(o) = make_float4(f0.x, f0.w, f1.z, f2.y);
    *reinterpret_cast<float4*>(o + (size_t)W * H) = make_float4(f0.y, f1.x, f1.w, f2.z);
    *reinterpret_cast<float4*>(o + (size_t)2 * W * H) = make_float4(f0.z, f1.y, f2.x, f2.w);
}

// d1: today's letterbox pattern -- 64 x 32 tile per 128-thread CTA, half-warps 4 rows apart: each warp store = 2 x 256 B
__global__ void __launch_bounds__(128) store_tile256(const uint8_t* __restrict__ src, float* __restrict__ dst) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int px = blockIdx.x * 64 + 4 * (lane & 15), r0 = blockIdx.y * 32 + warp * 8 + (lane >> 4) * 4;
#pragma unroll
    for (int r = 0; r < 4; ++r) px4(src, dst, blockIdx.z, r0 + r, px);
}
// d2: 128 x 16 tile per 128-thread CTA: each warp store = one 512-B run
__global__ void __launch_bounds__(128) store_run512(const uint8_t* __restrict__ src, float* __restrict__ dst) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int px = blockIdx.x * 128 + 4 * lane, r0 = blockIdx.y * 16 + warp * 4;
#pragma unroll
    for (int r = 0; r < 4; ++r) px4(src, dst, blockIdx.z, r0 + r, px);
}
// d3: full-width band of R rows per 160-thread CTA: each plane of the CTA is one contiguous R x 2560-B run
template <int R>
__global__ void __launch_bounds__(160) store_band(const uint8_t* __restrict__ src, float* __restrict__ dst) {
    const int px = 4 * threadIdx.x, r0 = blockIdx.x * R;
#pragma unroll
    for (int r = 0; r < R; ++r) px4(src, dst, blockIdx.y, r0 + r, px);
}
// d4: full-width band of 4 rows staged in shared memory, each plane written by one TMA bulk store (cp.async.bulk)
__global__ void __launch_bounds__(160) store_band_tma(const uint8_t* __restrict__ src, float* __restrict__ dst) {
    constexpr int R = 4;
    __shared__ __align__(128) float st[3][R * W];
    const int px = 4 * threadIdx.x, r0 = blockIdx.x * R, b = blockIdx.y;
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const uint32_t* s = reinterpret_cast<const uint32_t*>(src + ((size_t)b * H + r0 + r) * W * 3 + (size_t)px * 3);
        const float4 f0 = expand(__ldg(s)), f1 = expand(__ldg(s + 1)), f2 = expand(__ldg(s + 2));
        *reinterpret_cast<float4*>(&st[0][r * W + px]) = make_float4(f0.x, f0.w, f1.z, f2.y);
        *reinterpret_cast<float4*>(&st[1][r * W + px]) = make_float4(f0.y, f1.x, f1.w, f2.z);
        *reinterpret_cast<float4*>(&st[2][r * W + px]) = make_float4(f0.z, f1.y, f2.x, f2.w);
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    if (threadIdx.x < 3) {
        float* o = dst + ((size_t)b * 3 + threadIdx.x) * W * H + (size_t)r0 * W;
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(o),
                     "r"((uint32_t)__cvta_generic_to_shared(&st[threadIdx.x][0])), "r"((uint32_t)(R * W * 4))
                     : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // shared memory must outlive the read
    }
}

struct Bufs {
    uint8_t* src[NSET];
    float* out[NSET];
    float* head[NSET];
    float* sink;
};

template <typename F>
static float time_launches(F launch, cudaStream_t st) {
    for (int i = 0; i < 8; ++i) launch(i % NSET, st);
    CK(cudaStreamSynchronize(st));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    CK(cudaEventRecord(e0, st));
    for (int i = 0; i < LAUNCHES; ++i) launch(i % NSET, st);
    CK(cudaEventRecord(e1, st));
    CK(cudaEventSynchronize(e1));
    CK(cudaGetLastError());
    float ms;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    CK(cudaEventDestroy(e0));
    CK(cudaEventDestroy(e1));
    return ms * 1e3f / LAUNCHES;
}

static void report(const char* name, float us, double bytes) {
    printf("{\"probe\": \"%s\", \"us\": %.2f, \"GB_per_s\": %.0f, \"MB\": %.1f}\n", name, us, bytes / (us * 1e-6) / 1e9, bytes / 1e6);
    fflush(stdout);
}

int main() {
    cudaDeviceProp p;
    CK(cudaGetDeviceProperties(&p, 0));
    printf("# %s, %d SMs, L2 %d MB\n", p.name, p.multiProcessorCount, p.l2CacheSize >> 20);
    Bufs bf;
    for (int s = 0; s < NSET; ++s) {
        CK(cudaMalloc(&bf.src[s], SRC_BYTES));
        CK(cudaMalloc(&bf.out[s], OUT_FLOATS * 4));
        CK(cudaMalloc(&bf.head[s], HEAD_BYTES));
        CK(cudaMemset(bf.src[s], 0x5a + s, SRC_BYTES));
        CK(cudaMemset(bf.head[s], 0, HEAD_BYTES));
    }
    CK(cudaMalloc(&bf.sink, 4));
    cudaStream_t lo, hi;
    int prio_lo, prio_hi;
    CK(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
    CK(cudaStreamCreateWithPriority(&lo, cudaStreamNonBlocking, prio_lo));
    CK(cudaStreamCreateWithPriority(&hi, cudaStreamNonBlocking, prio_hi));

    const size_t nsrc = SRC_BYTES / 4, nhead = HEAD_BYTES / 16;
    auto a = [&](int s, cudaStream_t st) {
        expand_contig<<<(unsigned)((nsrc + 1023) / 1024), 256, 0, st>>>(reinterpret_cast<const uint32_t*>(bf.src[s]),
                                                                        reinterpret_cast<float4*>(bf.out[s]), nsrc);
    };
    auto b = [&](int s, cudaStream_t st) {
        read_only<<<(unsigned)((nhead + 1023) / 1024), 256, 0, st>>>(reinterpret_cast<const float4*>(bf.head[s]), nhead, bf.sink);
    };
    const double lb_bytes = SRC_BYTES + OUT_FLOATS * 4.0;
    report("a_expand_contiguous", time_launches(a, lo), lb_bytes);
    report("b_read_only", time_launches(b, lo), (double)HEAD_BYTES);

    // c: one graph = 4 steps, chain 1 = a(set 0..3) on the low-priority stream, chain 2 = b(set 0..3) on the high-priority one
    cudaGraph_t g;
    cudaGraphExec_t ge;
    cudaEvent_t fork, join;
    CK(cudaEventCreateWithFlags(&fork, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&join, cudaEventDisableTiming));
    CK(cudaStreamBeginCapture(lo, cudaStreamCaptureModeThreadLocal));
    CK(cudaEventRecord(fork, lo));
    CK(cudaStreamWaitEvent(hi, fork, 0));
    for (int s = 0; s < NSET; ++s) {
        b(s, hi);
        a(s, lo);
    }
    CK(cudaEventRecord(join, hi));
    CK(cudaStreamWaitEvent(lo, join, 0));
    CK(cudaStreamEndCapture(lo, &g));
    CK(cudaGraphInstantiate(&ge, g, 0));
    const float us_c = time_launches([&](int, cudaStream_t st) { CK(cudaGraphLaunch(ge, st)); }, lo) / NSET;
    report("c_a_parallel_b_graph_per_step", us_c, lb_bytes + HEAD_BYTES);

    auto d = [&](const char* name, auto launch) { report(name, time_launches(launch, lo), lb_bytes); };
    d("d1_tile64x32_256B_pieces", [&](int s, cudaStream_t st) { store_tile256<<<dim3(W / 64, H / 32, B), 128, 0, st>>>(bf.src[s], bf.out[s]); });
    d("d2_tile128x16_512B_runs", [&](int s, cudaStream_t st) { store_run512<<<dim3(W / 128, H / 16, B), 128, 0, st>>>(bf.src[s], bf.out[s]); });
    d("d3_band4_full_rows", [&](int s, cudaStream_t st) { store_band<4><<<dim3(H / 4, B), 160, 0, st>>>(bf.src[s], bf.out[s]); });
    d("d3_band8_full_rows", [&](int s, cudaStream_t st) { store_band<8><<<dim3(H / 8, B), 160, 0, st>>>(bf.src[s], bf.out[s]); });
    d("d4_band4_tma_bulk_store", [&](int s, cudaStream_t st) { store_band_tma<<<dim3(H / 4, B), 160, 0, st>>>(bf.src[s], bf.out[s]); });
    // a again last: drift of the card over the run
    report("a_expand_contiguous_again", time_launches(a, lo), lb_bytes);
    return 0;
}
