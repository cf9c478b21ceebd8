// select_sort.cuh -- block-level radix top-k select + bitonic sort, for one 1024-thread CTA.
//
// The reference sorts EVERYTHING with cub::DeviceRadixSort::SortPairsDescending (a stable descending
// sort of fp32 keys with an iota payload: ties keep ascending index; -0.0 and +0.0 are equal keys) and then uses the
// first k entries (rcnn/RpnDecode.cu:82, PredictorDecode.cu:75, RpnNms.cu:100, BatchedNms.cu:134).  The same ordered
// prefix is obtained here by (1) an exact radix SELECT of the k largest (key, lower index first) --
// 4 histogram passes over the keys plus 4 over the indices of the elements tied at the cut -- and
// (2) a bitonic SORT of only those k elements in shared memory, keyed by (~key << 32 | index).
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
template <typename KeyFn>
__device__ void block_select_topk(KeyFn key, int n, int k, SelectScratch& sc, uint32_t* key_cut_out, uint32_t* id_cut_out) {
    const int tid = threadIdx.x;
    uint32_t prefix = 0, mask = 0;
    __syncthreads();
    if (tid == 0) sc.need = k;
    for (int pass = 0; pass < 4; ++pass) {
        const int shift = 24 - 8 * pass;
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

}  // namespace trtx
