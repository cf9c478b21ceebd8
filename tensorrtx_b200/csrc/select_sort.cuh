// select_sort.cuh -- block-level radix top-k select + bitonic sort, for one 1024-thread CTA.
//
// The reference sorts EVERYTHING with cub::DeviceRadixSort::SortPairsDescending (a stable descending
// sort of fp32 keys with an iota payload: ties keep ascending index; -0.0 and +0.0 are equal keys) and then uses the
// first k entries (rcnn/RpnDecode.cu:82, PredictorDecode.cu:75, RpnNms.cu:100, BatchedNms.cu:134).  The same ordered
// prefix is obtained here by (1) an exact radix SELECT of the k largest (key, lower index first) --
// 4 histogram passes over the keys (2 over the 16-bit keys of half scores) plus 4 over the indices of the elements tied
// at the cut -- and (2) a bitonic SORT of only those k elements in shared memory, keyed by (~key << 32 | index).
#pragma once
#include "common.cuh"

namespace trtx {

constexpr int kSelThreads = 1024;

struct SelectScratch {
    int hist[256];
    int need;
    int bucket;
};

__device__ __forceinline__ void pick_bucket_dev(const int* hist, bool descending, int* need_io, int* bucket_out) {
    int need = *need_io, c = 0, d;
    if (descending) {
        for (d = 255; d > 0; --d) {
            if (c + hist[d] >= need) break;
            c += hist[d];
        }
    } else {
        for (d = 0; d < 255; ++d) {
            if (c + hist[d] >= need) break;
            c += hist[d];
        }
    }
    *need_io = need - c;
    *bucket_out = d;
}

// Exact cut for "the k largest of key(i), i in [0,n), ties -> smaller i":
// element i is selected  <=>  key(i) > key_cut || (key(i) == key_cut && i <= id_cut).   Requires n > k > 0.
// kKeyBits: the width of the keys (32 or 16), one 8-bit histogram pass per byte.
template <int kKeyBits = 32, typename KeyFn>
__device__ void block_select_topk(KeyFn key, int n, int k, SelectScratch& sc, uint32_t* key_cut_out, uint32_t* id_cut_out) {
    static_assert(kKeyBits == 32 || kKeyBits == 16, "keys of 4 or 2 bytes");
    const int tid = threadIdx.x;
    uint32_t prefix = 0, mask = 0;
    __syncthreads();
    if (tid == 0) sc.need = k;
    for (int pass = 0; pass < kKeyBits / 8; ++pass) {
        const int shift = kKeyBits - 8 - 8 * pass;
        if (tid < 256) sc.hist[tid] = 0;
        __syncthreads();
        for (int i = tid; i < n; i += kSelThreads) {
            const uint32_t kk = key(i);
            if ((kk & mask) == prefix) atomicAdd(&sc.hist[(kk >> shift) & 255], 1);
        }
        __syncthreads();
        if (tid == 0) {
            int need = sc.need, d;
            pick_bucket_dev(sc.hist, true, &need, &d);
            sc.need = need;
            sc.bucket = d;
        }
        __syncthreads();
        prefix |= (uint32_t)sc.bucket << shift;
        mask |= 255u << shift;
    }
    const uint32_t key_cut = prefix;
    uint32_t ip = 0, im = 0;  // sc.need now = how many elements with key == key_cut are taken
    for (int pass = 0; pass < 4; ++pass) {
        const int shift = 24 - 8 * pass;
        if (tid < 256) sc.hist[tid] = 0;
        __syncthreads();
        for (int i = tid; i < n; i += kSelThreads) {
            if (key(i) == key_cut && (((uint32_t)i) & im) == ip) atomicAdd(&sc.hist[((uint32_t)i >> shift) & 255], 1);
        }
        __syncthreads();
        if (tid == 0) {
            int need = sc.need, d;
            pick_bucket_dev(sc.hist, false, &need, &d);
            sc.need = need;
            sc.bucket = d;
        }
        __syncthreads();
        ip |= (uint32_t)sc.bucket << shift;
        im |= 255u << shift;
    }
    *key_cut_out = key_cut;
    *id_cut_out = ip;
    __syncthreads();
}

// ascending bitonic sort of S (power of two) 64-bit keys in shared memory
__device__ __forceinline__ void block_bitonic_sort_u64(unsigned long long* keys, int S) {
    const int tid = threadIdx.x;
    for (int k = 2; k <= S; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = tid; i < S; i += blockDim.x) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const unsigned long long a = keys[i], b = keys[ixj];
                    if ((a > b) == ((i & k) == 0)) {
                        keys[i] = b;
                        keys[ixj] = a;
                    }
                }
            }
            __syncthreads();
        }
    }
}

// key for "descending score, ascending index" under an ASCENDING 64-bit sort
__device__ __forceinline__ unsigned long long desc_key(float score, uint32_t idx) {
    return ((unsigned long long)(~float_key(score)) << 32) | idx;
}

// 16-bit key of a half that orders and ties exactly as float_key(__half2float(h)): widening is exact and monotonic, so every
// pattern that is not a NaN takes float_key's transform on its own 16 bits (-0 -> +0, then the sign flip).  A NaN takes the
// key of the half whose sign, exponent and top 10 mantissa bits are those of the float the device widens it to, so NaNs
// rank among themselves and against +-inf as their widened floats do, whether the conversion keeps the payload or returns
// one canonical NaN (a widened NaN's low 13 mantissa bits are then all zero or all one, the same for every NaN).
__device__ __forceinline__ uint32_t half_key(__half h) {
    uint32_t b = __half_as_ushort(h);
    if ((b & 0x7fffu) > 0x7c00u) {
        const uint32_t w = __float_as_uint(__half2float(h));
        b = ((w >> 16) & 0x8000u) | 0x7c00u | ((w >> 13) & 0x3ffu);
    }
    b = b == 0x8000u ? 0u : b;
    return (b & 0x8000u) ? (~b & 0xffffu) : (b | 0x8000u);
}

// The select key of an input element type: the 32-bit float_key, or the 16-bit half_key (two histogram passes, not four).
template <typename T>
struct SelectKey;
template <>
struct SelectKey<float> {
    static constexpr int kBits = 32;
    static __device__ __forceinline__ uint32_t of(float s) { return float_key(s); }
};
template <>
struct SelectKey<__half> {
    static constexpr int kBits = 16;
    static __device__ __forceinline__ uint32_t of(__half s) { return half_key(s); }
};

__device__ __forceinline__ float widen(float v) { return v; }
__device__ __forceinline__ float widen(__half v) { return __half2float(v); }

}  // namespace trtx
