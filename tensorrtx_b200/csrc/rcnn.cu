// rcnn.cu -- Faster R-CNN plugins for sm_90a: RpnDecode, RpnNms, PredictorDecode, BatchedNms.
// Replaces rcnn/RpnDecode.cu, RpnNms.cu, PredictorDecode.cu, BatchedNms.cu, which per IMAGE (host loop)
// run 1-2 cub::DeviceRadixSort passes + thrust transforms/gathers + an NMS kernel that iterates
// `for m in 0..N` with a __syncthreads() per m (and, launched over ceil(N/1024) blocks, races across
// blocks -- SURVEY section 5), after uploading an iota index vector from a std::vector every enqueue.
//
// Here every plugin is ONE launch for the whole batch (one 1024-thread CTA per image), no host-side
// index upload, no thrust/cub temporaries:
//   * "sort all, keep the first k" -> exact radix select of the top k + shared-memory bitonic sort of k
//     (select_sort.cuh) -- same ordered prefix as the stable descending radix sort of the reference;
//   * greedy NMS -> chunks of 32 sorted boxes against the kept list (IoU tile in shared memory, warp
//     ballot bitmaps, serial resolve by one warp): 2 barriers per 32 boxes instead of 1 per box, with
//     early exit once post_nms_topk boxes are kept;
//   * soft-NMS (linear / gaussian) keeps the reference's sequential score semantics exactly: chunk
//     members are resolved in order by one warp, then their decay is applied to all later boxes.
// These kernels are latency/occupancy-bound (<= 1 MB per image): report microseconds, not a roofline.
// The INTENDED (race-free) semantics of the reference kernels are implemented.
#include <float.h>

#include "select_sort.cuh"

namespace trtx {

// rcnn/RpnNms.cu:38-50 == BatchedNms.cu:43-55 (device code there; contraction-free here)
__device__ __forceinline__ float iou_plain(const float4 i, const float4 m) {
    float x1 = fmaxf(i.x, m.x), y1 = fmaxf(i.y, m.y);
    float x2 = fminf(i.z, m.z), y2 = fminf(i.w, m.w);
    float w = fmaxf(0.0f, __fsub_rn(x2, x1)), h = fmaxf(0.0f, __fsub_rn(y2, y1));
    float iarea = __fmul_rn(__fsub_rn(i.z, i.x), __fsub_rn(i.w, i.y));
    float marea = __fmul_rn(__fsub_rn(m.z, m.x), __fsub_rn(m.w, m.y));
    float inter = __fmul_rn(w, h);
    return __fdiv_rn(inter, __fsub_rn(__fadd_rn(iarea, marea), inter));
}

constexpr int kMaxAnchors = 64;

struct RpnDecodeArgs {
    const float* scores;
    const float* deltas;
    float* out_scores;
    float* out_boxes;
    int height, width, image_height, image_width;
    float stride;
    int num_anchors, top_n, sort_cap;
    float anchors[kMaxAnchors * 4];
};

// ---------------------------------------------------------------------------------------------
// RpnDecode (rcnn/RpnDecode.cu:27-143)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kSelThreads, 1) rpn_decode_kernel(const __grid_constant__ RpnDecodeArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    unsigned long long* keys = reinterpret_cast<unsigned long long*>(smem_raw);
    __shared__ SelectScratch sc;
    __shared__ int s_cnt;
    const int b = blockIdx.x, tid = threadIdx.x;
    const int hw = a.height * a.width;
    const int n = a.num_anchors * hw;
    const float* in_scores = a.scores + (size_t)b * n;
    const float* in_boxes = a.deltas + (size_t)b * n * 4;
    float* out_scores = a.out_scores + (size_t)b * a.top_n;
    float4* out_boxes = reinterpret_cast<float4*>(a.out_boxes) + (size_t)b * a.top_n;

    int num_det = n;
    const bool sorted = n > a.top_n;  // RpnDecode.cu:79-86
    if (sorted) {
        uint32_t kc, ic;
        block_select_topk([&](int i) { return float_key(in_scores[i]); }, n, a.top_n, sc, &kc, &ic);
        if (tid == 0) s_cnt = 0;
        for (int i = tid; i < a.sort_cap; i += kSelThreads) keys[i] = ~0ull;
        __syncthreads();
        for (int i = tid; i < n; i += kSelThreads) {
            const float s = in_scores[i];
            const uint32_t k = float_key(s);
            if (k > kc || (k == kc && (uint32_t)i <= ic)) keys[atomicAdd(&s_cnt, 1)] = desc_key(s, (uint32_t)i);
        }
        __syncthreads();
        block_bitonic_sort_u64(keys, a.sort_cap);
        num_det = a.top_n;
    }
    for (int r = tid; r < num_det; r += kSelThreads) {
        const int i = sorted ? (int)(keys[r] & 0xffffffffull) : r;
        const int x = i % a.width;
        const int y = (i / a.width) % a.height;
        const int an = (i / a.height / a.width) % a.num_anchors;
        float4 box = make_float4(in_boxes[((size_t)(an * 4 + 0) * a.height + y) * a.width + x],
                                 in_boxes[((size_t)(an * 4 + 1) * a.height + y) * a.width + x],
                                 in_boxes[((size_t)(an * 4 + 2) * a.height + y) * a.width + x],
                                 in_boxes[((size_t)(an * 4 + 3) * a.height + y) * a.width + x]);
        if (a.num_anchors > 0) {  // has_anchors, :107-131
            const float fx = __fmul_rn((float)x, a.stride);
            const float fy = __fmul_rn((float)y, a.stride);
            const float* d = a.anchors + 4 * an;
            const float x1 = __fadd_rn(fx, d[0]), y1 = __fadd_rn(fy, d[1]);
            const float x2 = __fadd_rn(fx, d[2]), y2 = __fadd_rn(fy, d[3]);
            const float w = __fsub_rn(x2, x1), h = __fsub_rn(y2, y1);
            const float pcx = __fadd_rn(__fadd_rn(__fmul_rn(box.x, w), x1), __fmul_rn(0.5f, w));
            const float pcy = __fadd_rn(__fadd_rn(__fmul_rn(box.y, h), y1), __fmul_rn(0.5f, h));
            const float pw = __fmul_rn(expf(box.z), w);
            const float ph = __fmul_rn(expf(box.w), h);
            box = make_float4(fmaxf(0.0f, __fsub_rn(pcx, __fmul_rn(0.5f, pw))), fmaxf(0.0f, __fsub_rn(pcy, __fmul_rn(0.5f, ph))),
                              fminf(__fadd_rn(pcx, __fmul_rn(0.5f, pw)), (float)a.image_width),
                              fminf(__fadd_rn(pcy, __fmul_rn(0.5f, ph)), (float)a.image_height));
        }
        out_boxes[r] = box;
        // filter empty boxes, :129-132
        out_scores[r] = (box.z - box.x <= 0.0f || box.w - box.y <= 0.0f) ? -FLT_MAX : in_scores[i];
    }
    for (int r = num_det + tid; r < a.top_n; r += kSelThreads) out_scores[r] = -FLT_MAX;  // :136-139
}

// ---------------------------------------------------------------------------------------------
// PredictorDecode (rcnn/PredictorDecode.cu:24-110)
// ---------------------------------------------------------------------------------------------
struct PredictorArgs {
    const float* scores;
    const float* deltas;
    const float* proposals;
    float* out_scores;
    float* out_boxes;
    float* out_classes;
    int num_boxes, num_classes, image_height, image_width, sort_cap;
    float w[4];
};

__global__ void __launch_bounds__(kSelThreads, 1) predictor_decode_kernel(const __grid_constant__ PredictorArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    unsigned long long* keys = reinterpret_cast<unsigned long long*>(smem_raw);
    __shared__ SelectScratch sc;
    __shared__ int s_cnt;
    const int b = blockIdx.x, tid = threadIdx.x;
    const int n = a.num_boxes * a.num_classes;
    const float* in_scores = a.scores + (size_t)b * n;
    const float4* in_boxes = reinterpret_cast<const float4*>(a.deltas) + (size_t)b * n;
    const float4* in_prop = reinterpret_cast<const float4*>(a.proposals) + (size_t)b * a.num_boxes;
    const int k = a.num_boxes;  // the reference sorts all n scores and keeps the first num_boxes (:75-79)

    for (int i = tid; i < a.sort_cap; i += kSelThreads) keys[i] = ~0ull;
    if (tid == 0) s_cnt = 0;
    __syncthreads();
    if (n > k) {
        uint32_t kc, ic;
        block_select_topk([&](int i) { return float_key(in_scores[i]); }, n, k, sc, &kc, &ic);
        for (int i = tid; i < n; i += kSelThreads) {
            const float s = in_scores[i];
            const uint32_t kk = float_key(s);
            if (kk > kc || (kk == kc && (uint32_t)i <= ic)) keys[atomicAdd(&s_cnt, 1)] = desc_key(s, (uint32_t)i);
        }
    } else {
        for (int i = tid; i < n; i += kSelThreads) keys[i] = desc_key(in_scores[i], (uint32_t)i);
    }
    __syncthreads();
    block_bitonic_sort_u64(keys, a.sort_cap);
    for (int r = tid; r < k && r < n; r += kSelThreads) {
        const int i = (int)(keys[r] & 0xffffffffull);
        const int cls = i % a.num_classes;
        const int nb = i / a.num_classes;
        const float4 d = in_boxes[i];
        const float4 p = in_prop[nb];
        const float w = __fsub_rn(p.z, p.x), h = __fsub_rn(p.w, p.y);
        const float pcx = __fadd_rn(__fadd_rn(__fmul_rn(__fdiv_rn(d.x, a.w[0]), w), p.x), __fmul_rn(0.5f, w));
        const float pcy = __fadd_rn(__fadd_rn(__fmul_rn(__fdiv_rn(d.y, a.w[1]), h), p.y), __fmul_rn(0.5f, h));
        const float pw = __fmul_rn(expf(__fdiv_rn(d.z, a.w[2])), w);
        const float ph = __fmul_rn(expf(__fdiv_rn(d.w, a.w[3])), h);
        const float4 box = make_float4(fmaxf(0.0f, __fsub_rn(pcx, __fmul_rn(0.5f, pw))), fmaxf(0.0f, __fsub_rn(pcy, __fmul_rn(0.5f, ph))),
                                       fminf(__fadd_rn(pcx, __fmul_rn(0.5f, pw)), (float)a.image_width),
                                       fminf(__fadd_rn(pcy, __fmul_rn(0.5f, ph)), (float)a.image_width));  // sic: :99 uses image_width
        reinterpret_cast<float4*>(a.out_boxes)[(size_t)b * a.num_boxes + r] = box;
        a.out_scores[(size_t)b * a.num_boxes + r] = (box.z - box.x <= 0.0f || box.w - box.y <= 0.0f) ? 0.0f : in_scores[i];
        a.out_classes[(size_t)b * a.num_boxes + r] = (float)cls;
    }
}

// ---------------------------------------------------------------------------------------------
// RpnNms (rcnn/RpnNms.cu:27-121)
// ---------------------------------------------------------------------------------------------
struct RpnNmsArgs {
    const float* scores;
    const float* boxes;
    float* out_boxes;
    int pre, post, sort_cap;
    int key_area;  // bytes: max(sort keys, kept boxes + state), 16-byte aligned
    float thresh;
};

__global__ void __launch_bounds__(kSelThreads, 1) rpn_nms_kernel(const __grid_constant__ RpnNmsArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    // [ keys (sort_cap u64)  |  boxes (pre float4) ];  after the gather the key area is reused for
    // [ kept boxes (post float4) | state (pre bytes) ]
    unsigned long long* keys = reinterpret_cast<unsigned long long*>(smem_raw);
    float4* s_box = reinterpret_cast<float4*>(smem_raw + a.key_area);
    float4* s_kbox = reinterpret_cast<float4*>(smem_raw);
    unsigned char* s_state = reinterpret_cast<unsigned char*>(s_kbox + a.post);  // 0 alive-candidate, 1 kept, 2 dead
    __shared__ unsigned s_rem, s_sup[32];
    __shared__ int s_nkept;

    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n = a.pre;
    const float* sc = a.scores + (size_t)b * n;
    const float4* bx = reinterpret_cast<const float4*>(a.boxes) + (size_t)b * n;
    float4* ob = reinterpret_cast<float4*>(a.out_boxes) + (size_t)b * a.post;

    for (int i = tid; i < a.sort_cap; i += kSelThreads) keys[i] = i < n ? desc_key(sc[i], (uint32_t)i) : ~0ull;
    __syncthreads();
    block_bitonic_sort_u64(keys, a.sort_cap);
    // gather boxes in sorted order; remember which entries are born dead (score == -FLT_MAX, :34)
    uint32_t my_idx[8];
    float my_sc[8];
    int cnt = 0;
    for (int r = tid; r < n; r += kSelThreads) {
        my_idx[cnt] = (uint32_t)(keys[r] & 0xffffffffull);
        my_sc[cnt] = sc[my_idx[cnt]];
        s_box[r] = bx[my_idx[cnt]];
        ++cnt;
    }
    __syncthreads();  // keys are dead: the area becomes kept boxes + state
    cnt = 0;
    for (int r = tid; r < n; r += kSelThreads) s_state[r] = (my_sc[cnt++] > -FLT_MAX) ? 0 : 2;
    if (tid == 0) {
        s_nkept = 0;
        s_rem = 0;
    }
    __syncthreads();

    int n_kept = 0;
    for (int c0 = 0; c0 < n && n_kept < a.post; c0 += 32) {
        const int nchunk = min(32, n - c0);
        // members already dead never become suppressors and need no test
        const int P = 32 * n_kept;
        for (int p = tid; p < P; p += kSelThreads) {
            const int i = p & 31, k = p >> 5;
            if (i < nchunk && s_state[c0 + i] == 0) {
                if (iou_plain(s_box[c0 + i], s_kbox[k]) > a.thresh) atomicOr(&s_rem, 1u << i);
            }
        }
        {
            const int i = warp, j = lane;
            bool hit = false;
            if (i < nchunk && j < i && s_state[c0 + i] == 0 && s_state[c0 + j] == 0)
                hit = iou_plain(s_box[c0 + i], s_box[c0 + j]) > a.thresh;
            const unsigned m = __ballot_sync(0xffffffffu, hit);
            if (lane == 0) s_sup[i] = m;
        }
        __syncthreads();
        if (warp == 0) {
            const unsigned my = s_sup[lane];
            const bool cand = lane < nchunk && s_state[c0 + lane] == 0;
            unsigned alive = __ballot_sync(0xffffffffu, cand) & ~s_rem;
#pragma unroll
            for (int j = 0; j < 32; ++j) {
                const unsigned kill = __ballot_sync(0xffffffffu, (my >> j) & 1u);
                if ((alive >> j) & 1u) alive &= ~kill;
            }
            if (cand) {
                if ((alive >> lane) & 1u) {
                    const int pos = n_kept + __popc(alive & ((1u << lane) - 1u));
                    if (pos < a.post) {
                        s_kbox[pos] = s_box[c0 + lane];
                        s_state[c0 + lane] = 1;
                    }
                } else {
                    s_state[c0 + lane] = 2;
                }
            }
            if (lane == 0) {
                s_nkept = min(a.post, n_kept + __popc(alive));
                s_rem = 0;
            }
        }
        __syncthreads();
        n_kept = s_nkept;
    }
    // re-sort + gather (:111-117): kept boxes first (score order), then everything else in sorted position
    // order (their keys are all -FLT_MAX; the radix sort is stable), truncated to post_nms_topk.
    const int n_out = min(a.post, n);
    for (int r = tid; r < n_kept; r += kSelThreads) ob[r] = s_kbox[r];
    if (n_kept < n_out) {
        // rank of each non-kept entry among non-kept entries = position - #kept before it
        // (sequential prefix by warp 0 over <= pre entries; only reached when fewer than `post` survive)
        if (warp == 0) {
            int carry = 0;
            for (int base = 0; base < n; base += 32) {
                const int r = base + lane;
                const bool nk = r < n && s_state[r] != 1;
                const unsigned m = __ballot_sync(0xffffffffu, nk);
                if (nk) {
                    const int pos = n_kept + carry + __popc(m & ((1u << lane) - 1u));
                    if (pos < n_out) ob[pos] = s_box[r];
                }
                carry += __popc(m);
                if (n_kept + carry >= n_out) break;
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// BatchedNms (rcnn/BatchedNms.cu:28-162): class-aware hard / soft-linear / soft-gaussian
// ---------------------------------------------------------------------------------------------
struct BatchedNmsArgs {
    const float* scores;
    const float* boxes;
    const float* classes;
    float* out_scores;
    float* out_boxes;
    float* out_classes;
    int method, count, dets, sort_cap;
    float thresh;
};

__device__ __forceinline__ float soft_update(int method, float overlap, float s) {
    // BatchedNms.cu:60-88 (sigma = 0.5)
    if (method == 1) return __fmul_rn(__fsub_rn(1.0f, overlap), s);
    if (method == 2) return __fmul_rn(expf(__fdiv_rn(-__fmul_rn(overlap, overlap), 0.5f)), s);
    return 0.0f;
}

__global__ void __launch_bounds__(kSelThreads, 1) batched_nms_kernel(const __grid_constant__ BatchedNmsArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    unsigned long long* keys = reinterpret_cast<unsigned long long*>(smem_raw);  // sort_cap
    float4* s_box = reinterpret_cast<float4*>(keys + a.sort_cap);               // count
    float* s_sc = reinterpret_cast<float*>(s_box + a.count);                    // count (current scores)
    int* s_cls = reinterpret_cast<int*>(s_sc + a.count);                        // count
    uint32_t* s_src = reinterpret_cast<uint32_t*>(s_cls + a.count);             // count (original index)
    __shared__ unsigned s_alive;

    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n = a.count;
    const float* sc = a.scores + (size_t)b * n;
    const float4* bx = reinterpret_cast<const float4*>(a.boxes) + (size_t)b * n;
    const float* cl = a.classes + (size_t)b * n;

    for (int i = tid; i < a.sort_cap; i += kSelThreads) keys[i] = i < n ? desc_key(sc[i], (uint32_t)i) : ~0ull;
    __syncthreads();
    block_bitonic_sort_u64(keys, a.sort_cap);
    for (int r = tid; r < n; r += kSelThreads) {
        const uint32_t i = (uint32_t)(keys[r] & 0xffffffffull);
        s_src[r] = i;
        s_box[r] = bx[i];
        s_sc[r] = sc[i];
        s_cls[r] = (int)cl[i];  // `int icls = classes[idx]` (:38-39)
    }
    __syncthreads();

    for (int c0 = 0; c0 < n; c0 += 32) {
        const int nchunk = min(32, n - c0);
        // (a) resolve the chunk in order (one warp): member j is a suppressor iff its CURRENT score > 0 (:35)
        if (warp == 0) {
            const bool in = lane < nchunk;
            float4 mybox = in ? s_box[c0 + lane] : make_float4(0, 0, 0, 0);
            int mycls = in ? s_cls[c0 + lane] : -1;
            float mys = in ? s_sc[c0 + lane] : 0.0f;
            unsigned alive = 0;
            for (int j = 0; j < nchunk; ++j) {
                const float sj = __shfl_sync(0xffffffffu, mys, j);
                const bool aj = sj > 0.0f;
                if (aj) alive |= 1u << j;
                const int cj = __shfl_sync(0xffffffffu, mycls, j);
                float4 bj;
                bj.x = __shfl_sync(0xffffffffu, mybox.x, j);
                bj.y = __shfl_sync(0xffffffffu, mybox.y, j);
                bj.z = __shfl_sync(0xffffffffu, mybox.z, j);
                bj.w = __shfl_sync(0xffffffffu, mybox.w, j);
                if (aj && in && lane > j && cj == mycls) {
                    const float ov = iou_plain(mybox, bj);
                    if (ov > a.thresh) mys = soft_update(a.method, ov, mys);
                }
            }
            if (in) s_sc[c0 + lane] = mys;
            if (lane == 0) s_alive = alive;
        }
        __syncthreads();
        // (b) apply the chunk's suppressors, in order, to every later box
        const unsigned alive = s_alive;
        if (alive) {
            for (int i = c0 + 32 + tid; i < n; i += kSelThreads) {
                const float4 ib = s_box[i];
                const int ic = s_cls[i];
                float s = s_sc[i];
                for (int j = 0; j < nchunk; ++j) {
                    if (((alive >> j) & 1u) && s_cls[c0 + j] == ic) {
                        const float ov = iou_plain(ib, s_box[c0 + j]);
                        if (ov > a.thresh) s = soft_update(a.method, ov, s);
                    }
                }
                s_sc[i] = s;
            }
        }
        __syncthreads();
    }
    // re-sort by the updated scores (stable: ties keep first-sort position), take the first `dets` (:146-158)
    for (int r = tid; r < a.sort_cap; r += kSelThreads) keys[r] = r < n ? desc_key(s_sc[r], (uint32_t)r) : ~0ull;
    __syncthreads();
    block_bitonic_sort_u64(keys, a.sort_cap);
    const int n_out = min(a.dets, n);
    for (int r = tid; r < a.dets; r += kSelThreads) {
        float* os = a.out_scores + (size_t)b * a.dets + r;
        if (r < n_out) {
            const uint32_t pos = (uint32_t)(keys[r] & 0xffffffffull);
            *os = s_sc[pos];
            reinterpret_cast<float4*>(a.out_boxes)[(size_t)b * a.dets + r] = s_box[pos];
            a.out_classes[(size_t)b * a.dets + r] = cl[s_src[pos]];
        } else {
            *os = 0.0f;  // :152-154 (boxes / classes beyond num_detections are left untouched by the reference)
        }
    }
}

static int pow2_at_least(int v) {
    int s = 32;
    while (s < v) s <<= 1;
    return s;
}
constexpr int kMaxSortCap = 8192;

}  // namespace trtx

using namespace trtx;

extern "C" {

// Workspace: none of these kernels needs global scratch (everything lives in shared memory); the
// "null workspace -> size" idiom is kept and reports a nominal 256 bytes so that TensorRT's
// allocation path is exercised exactly as with the reference plugins.
static const int64_t kNominalWorkspace = 256;

TRTX_API int64_t trtx_rpn_decode(int batch, const float* scores_dev, const float* deltas_dev, float* out_scores_dev,
                                 float* out_boxes_dev, int height, int width, int image_height, int image_width,
                                 float stride, const float* anchors_host, int num_anchors, int top_n,
                                 void* workspace_dev, size_t workspace_bytes, trtx_stream_t stream) {
    if (!workspace_dev || !workspace_bytes) return kNominalWorkspace;
    if (batch <= 0 || !scores_dev || !deltas_dev || !out_scores_dev || !out_boxes_dev) return -TRTX_ERR_INVALID;
    if (height <= 0 || width <= 0 || top_n <= 0 || num_anchors < 0 || (num_anchors > 0 && !anchors_host))
        return -TRTX_ERR_INVALID;
    if (num_anchors > kMaxAnchors || top_n > kMaxSortCap) return -TRTX_ERR_UNSUPPORTED;
    if (num_anchors == 0) return -TRTX_ERR_UNSUPPORTED;  // scores_size would be 0 in the reference too
    RpnDecodeArgs a{};
    a.scores = scores_dev;
    a.deltas = deltas_dev;
    a.out_scores = out_scores_dev;
    a.out_boxes = out_boxes_dev;
    a.height = height;
    a.width = width;
    a.image_height = image_height;
    a.image_width = image_width;
    a.stride = stride;
    a.num_anchors = num_anchors;
    a.top_n = top_n;
    a.sort_cap = pow2_at_least(top_n);
    for (int i = 0; i < num_anchors * 4; ++i) a.anchors[i] = anchors_host[i];
    const size_t smem = sizeof(unsigned long long) * a.sort_cap;
    cudaFuncSetAttribute(rpn_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(unsigned long long) * kMaxSortCap));
    rpn_decode_kernel<<<batch, kSelThreads, smem, static_cast<cudaStream_t>(stream)>>>(a);
    return -(int64_t)check_launch();
}

TRTX_API int64_t trtx_rpn_nms(int batch, const float* scores_dev, const float* boxes_dev, float* out_boxes_dev,
                              int pre_nms_topk, int post_nms_topk, float nms_thresh, void* workspace_dev,
                              size_t workspace_bytes, trtx_stream_t stream) {
    if (!workspace_dev || !workspace_bytes) return kNominalWorkspace;
    if (batch <= 0 || !scores_dev || !boxes_dev || !out_boxes_dev || pre_nms_topk <= 0 || post_nms_topk <= 0)
        return -TRTX_ERR_INVALID;
    if (pre_nms_topk > kMaxSortCap) return -TRTX_ERR_UNSUPPORTED;
    RpnNmsArgs a{};
    a.scores = scores_dev;
    a.boxes = boxes_dev;
    a.out_boxes = out_boxes_dev;
    a.pre = pre_nms_topk;
    a.post = post_nms_topk;
    a.sort_cap = pow2_at_least(pre_nms_topk);
    a.thresh = nms_thresh;
    const size_t key_bytes = sizeof(unsigned long long) * a.sort_cap;
    const size_t reuse = align_up(sizeof(float4) * (size_t)a.post + (size_t)a.pre, 16);
    a.key_area = (int)(key_bytes > reuse ? key_bytes : reuse);
    const size_t smem2 = (size_t)a.key_area + sizeof(float4) * (size_t)a.pre;
    if (smem2 > 220 * 1024) return -TRTX_ERR_UNSUPPORTED;
    cudaFuncSetAttribute(rpn_nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
    rpn_nms_kernel<<<batch, kSelThreads, smem2, static_cast<cudaStream_t>(stream)>>>(a);
    return -(int64_t)check_launch();
}

TRTX_API int64_t trtx_predictor_decode(int batch, const float* scores_dev, const float* deltas_dev,
                                       const float* proposals_dev, float* out_scores_dev, float* out_boxes_dev,
                                       float* out_classes_dev, int num_boxes, int num_classes, int image_height,
                                       int image_width, const float* bbox_reg_weights_host, void* workspace_dev,
                                       size_t workspace_bytes, trtx_stream_t stream) {
    if (!workspace_dev || !workspace_bytes) return kNominalWorkspace;
    if (batch <= 0 || !scores_dev || !deltas_dev || !proposals_dev || !out_scores_dev || !out_boxes_dev ||
        !out_classes_dev || num_boxes <= 0 || num_classes <= 0 || !bbox_reg_weights_host)
        return -TRTX_ERR_INVALID;
    if (num_boxes > kMaxSortCap) return -TRTX_ERR_UNSUPPORTED;
    PredictorArgs a{};
    a.scores = scores_dev;
    a.deltas = deltas_dev;
    a.proposals = proposals_dev;
    a.out_scores = out_scores_dev;
    a.out_boxes = out_boxes_dev;
    a.out_classes = out_classes_dev;
    a.num_boxes = num_boxes;
    a.num_classes = num_classes;
    a.image_height = image_height;
    a.image_width = image_width;
    a.sort_cap = pow2_at_least(num_boxes);
    for (int i = 0; i < 4; ++i) a.w[i] = bbox_reg_weights_host[i];
    const size_t smem = sizeof(unsigned long long) * a.sort_cap;
    cudaFuncSetAttribute(predictor_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(unsigned long long) * kMaxSortCap));
    predictor_decode_kernel<<<batch, kSelThreads, smem, static_cast<cudaStream_t>(stream)>>>(a);
    return -(int64_t)check_launch();
}

TRTX_API int64_t trtx_batched_nms(int nms_method, int batch, const float* scores_dev, const float* boxes_dev,
                                  const float* classes_dev, float* out_scores_dev, float* out_boxes_dev,
                                  float* out_classes_dev, int count, int detections_per_im, float nms_thresh,
                                  void* workspace_dev, size_t workspace_bytes, trtx_stream_t stream) {
    if (!workspace_dev || !workspace_bytes) return kNominalWorkspace;
    if (batch <= 0 || !scores_dev || !boxes_dev || !classes_dev || !out_scores_dev || !out_boxes_dev ||
        !out_classes_dev || count <= 0 || detections_per_im <= 0 || nms_method < 0)
        return -TRTX_ERR_INVALID;
    if (count > 4096) return -TRTX_ERR_UNSUPPORTED;
    BatchedNmsArgs a{};
    a.scores = scores_dev;
    a.boxes = boxes_dev;
    a.classes = classes_dev;
    a.out_scores = out_scores_dev;
    a.out_boxes = out_boxes_dev;
    a.out_classes = out_classes_dev;
    a.method = nms_method;
    a.count = count;
    a.dets = detections_per_im;
    a.sort_cap = pow2_at_least(count);
    a.thresh = nms_thresh;
    const size_t smem = sizeof(unsigned long long) * a.sort_cap + (size_t)count * (16 + 4 + 4 + 4);
    cudaFuncSetAttribute(batched_nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    batched_nms_kernel<<<batch, kSelThreads, smem, static_cast<cudaStream_t>(stream)>>>(a);
    return -(int64_t)check_launch();
}

}  // extern "C"
