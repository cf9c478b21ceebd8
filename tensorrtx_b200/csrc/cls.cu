// cls.cu -- YOLO classification post-process for sm_90a: softmax and top-k of the cls drivers, on the device.
// Replaces, per image, the host loop of yolov8/yolov8_cls.cpp:274-282 (the same in yolo11_cls.cpp and yolov5_cls.cpp:264-272)
// after the D2H copy of every logit:
//     auto res = softmax(p, kOutputSize);       // :48-61   t_i = expf(x_i); sum += t_i in ascending i; res_i = t_i / sum
//     auto topk_idx = topk(res, 3);             // :63-78   std::sort of all indices by res, descending, first min(k, n)
// and yolo26/yolo26_cls.cpp:218-225, which ranks the raw output (the engine's last layer is a sigmoid) with the same topk.
//
// One CTA of kSelThreads per image: expf in parallel, the sum sequentially in one thread (the reference's loop order: the
// ~1 000 dependent adds take a few microseconds), the divisions in parallel, then the exact radix select of the k largest and a
// bitonic sort of only those (select_sort.cuh), ordered like every other descending sort of the library: by float_key, so
// -0.0 == +0.0, ties keep ascending index, +NaN ranks above +inf and -NaN below -inf.  std::sort with `a > b` is not stable,
// and with a NaN (an overflowing expf makes a probability inf / inf, an all-underflow row makes every one 0 / 0) its order is
// undefined: DESIGN section 2.
#include "select_sort.cuh"

namespace trtx {

constexpr int kClsMaxClasses = 8192;  // res in shared memory with the sort keys: at most 96 KB per CTA

struct ClsPostArgs {
    const float* logits;
    int32_t* index;
    float* value;
    float* probs;  // nullable
    int n, k, kk;  // classes, output row stride, entries written = min(k, n)
    int sort_n;    // power of two >= kk
    int softmax;
};

__global__ void __launch_bounds__(kSelThreads) cls_postprocess_kernel(const __grid_constant__ ClsPostArgs a) {
    extern __shared__ __align__(16) unsigned long long keys[];  // [a.sort_n], then res [a.n]
    float* res = reinterpret_cast<float*>(keys + a.sort_n);
    __shared__ SelectScratch sc;
    __shared__ float s_sum;
    __shared__ int s_count;
    const int tid = threadIdx.x, n = a.n, b = blockIdx.x;
    const float* x = a.logits + (size_t)b * n;
    for (int i = tid; i < n; i += kSelThreads) res[i] = a.softmax ? expf(x[i]) : x[i];
    if (a.softmax) {
        __syncthreads();
        if (tid == 0) {  // float sum in ascending i, as softmax's loop adds
            float sum = 0.0f;
            for (int i = 0; i < n; ++i) sum = __fadd_rn(sum, res[i]);
            s_sum = sum;
        }
        __syncthreads();
        const float sum = s_sum;
        for (int i = tid; i < n; i += kSelThreads) res[i] = __fdiv_rn(res[i], sum);
    }
    if (tid == 0) s_count = 0;
    __syncthreads();
    if (a.probs)
        for (int i = tid; i < n; i += kSelThreads) a.probs[(size_t)b * n + i] = res[i];
    const int kk = a.kk;
    uint32_t key_cut = 0, id_cut = 0xffffffffu;  // kk == n: every element is selected
    if (kk < n) block_select_topk([&](int i) { return float_key(res[i]); }, n, kk, sc, &key_cut, &id_cut);
    // the selected elements, in any order (the sort orders them), then sentinels that sort last
    for (int i = tid; i < n; i += kSelThreads) {
        const uint32_t key = float_key(res[i]);
        if (key > key_cut || (key == key_cut && (uint32_t)i <= id_cut)) keys[atomicAdd(&s_count, 1)] = desc_key(res[i], (uint32_t)i);
    }
    for (int i = kk + tid; i < a.sort_n; i += kSelThreads) keys[i] = ~0ull;
    __syncthreads();
    block_bitonic_sort_u64(keys, a.sort_n);
    for (int j = tid; j < kk; j += kSelThreads) {
        const int idx = (int)(uint32_t)keys[j];
        a.index[(size_t)b * a.k + j] = idx;
        a.value[(size_t)b * a.k + j] = res[idx];
    }
}

}  // namespace trtx

using namespace trtx;

extern "C" {

TRTX_API int trtx_cls_postprocess_enqueue(int softmax, int batch, int num_classes, const float* logits_dev, int k,
                                          int32_t* index_dev, float* value_dev, float* probs_dev, trtx_stream_t stream) {
    if (!logits_dev || !index_dev || !value_dev || batch <= 0 || num_classes <= 0 || k <= 0) return TRTX_ERR_INVALID;
    if (softmax != 0 && softmax != 1) return TRTX_ERR_INVALID;
    if (num_classes > kClsMaxClasses) return TRTX_ERR_UNSUPPORTED;
    ClsPostArgs a;
    a.logits = logits_dev;
    a.index = index_dev;
    a.value = value_dev;
    a.probs = probs_dev;
    a.n = num_classes;
    a.k = k;
    a.kk = k < num_classes ? k : num_classes;
    a.sort_n = 1;
    while (a.sort_n < a.kk) a.sort_n <<= 1;
    a.softmax = softmax;
    const size_t smem = (size_t)a.sort_n * sizeof(unsigned long long) + (size_t)num_classes * sizeof(float);
    if (const int rc = opt_in_smem(cls_postprocess_kernel, smem)) return rc;
    cls_postprocess_kernel<<<(unsigned)batch, kSelThreads, smem, static_cast<cudaStream_t>(stream)>>>(a);
    return check_launch();
}

}  // extern "C"
