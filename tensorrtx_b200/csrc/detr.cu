// detr.cu -- DETR post-process for sm_90a: the driver's per-query loop on the device.
// Replaces, per batch, the D2H copy of the engine's softmax scores [B, Q, C] and boxes [B, Q, 4] (detr/detr.cpp:643-648) and
// the host loop of detr/detr.cpp:777-806:
//     label = -1, score = -1;  for j: if (score < s[j]) label = j, score = s[j];      the first maximum; a NaN is never taken
//     if (score > SCORE_THRESH && label % NUM_CLASS != NUM_CLASS - 1)                 drop the no-object class
//         cv::Rect r(x1, y1, x2 - x1, y2 - y1)                                        detr_get_rect (common.cuh)
// into rows (x, y, w, h, score, class) per kept query, in query order.
//
// One CTA of kDetrThreads per frame, the queries in passes of kDetrThreads:
//   1. argmax: warp w takes queries w, w + kDetrWarps, ... of the pass; each lane scans classes lane, lane + 32, ... with the
//      reference's `score < s[j]`, then a shuffle reduction keeps the larger score and, on equal scores, the smaller class,
//      which is the first maximum of the whole row;
//   2. keep flags, a ballot per warp and a scan of the warps' counts give each kept query its output slot (query order, no
//      atomics); its owning thread computes the rectangle into shared memory;
//   3. the CTA writes the pass's kept rows as one contiguous run of floats (coalesced).
// Rows past the kept count are zeroed, and float 0 gets the count.
#include "common.cuh"

namespace trtx {

constexpr int kDetrThreads = 1024;  // queries per pass: 32 warps, so that DETR's 100 queries take 3 to 4 argmaxes per warp
constexpr int kDetrWarps = kDetrThreads / kWarp;
constexpr int kDetrRow = 6;         // x, y, w, h, score, class
constexpr int kDetrMaxDim = 1 << 24;  // Q and C: the count and the class are stored as floats, exact up to 2^24

struct DetrPostArgs {
    FrameSizes sizes;
    int num_queries, num_classes;
    float score_thresh;
    const float* scores;  // [B, Q, C]
    const float* boxes;   // [B, Q, 4]
    float* rows;          // [B, 1 + Q * 6]
};

__global__ void __launch_bounds__(kDetrThreads) detr_postprocess_kernel(const __grid_constant__ DetrPostArgs a) {
    __shared__ float s_score[kDetrThreads];   // argmax of each query of the pass
    __shared__ int s_label[kDetrThreads];
    __shared__ int s_src[kDetrThreads];       // query of the pass of each kept slot
    __shared__ int s_rect[kDetrThreads][4];   // its rectangle
    __shared__ int s_warp[kDetrWarps];        // kept queries per warp of the pass
    const int tid = threadIdx.x, lane = tid & (kWarp - 1), warp = tid / kWarp, b = a.sizes.base + blockIdx.x;
    const int Q = a.num_queries, C = a.num_classes, img_w = a.sizes.w[blockIdx.x], img_h = a.sizes.h[blockIdx.x];
    const float* scores = a.scores + (size_t)b * Q * C;
    const float* boxes = a.boxes + (size_t)b * Q * 4;
    float* out = a.rows + (size_t)b * (1 + (size_t)Q * kDetrRow);
    int kept = 0;  // rows written by the earlier passes
    for (int q0 = 0; q0 < Q; q0 += kDetrThreads) {
        const int n = min(kDetrThreads, Q - q0);
        for (int k = warp; k < n; k += kDetrWarps) {
            const float* s = scores + (size_t)(q0 + k) * C;
            float best = -1.f;
            int label = -1;
#pragma unroll 4
            for (int j = lane; j < C; j += kWarp) {
                const float v = __ldg(s + j);
                if (best < v) best = v, label = j;
            }
            // no candidate is NaN and a taken one is > -1, so the start (-1, -1) ties only itself
#pragma unroll
            for (int o = kWarp / 2; o > 0; o >>= 1) {
                const float ob = __shfl_xor_sync(0xffffffffu, best, o);
                const int ol = __shfl_xor_sync(0xffffffffu, label, o);
                if (best < ob || (best == ob && ol < label)) best = ob, label = ol;
            }
            if (lane == 0) s_score[k] = best, s_label[k] = label;
        }
        __syncthreads();
        const bool keep = tid < n && s_score[tid] > a.score_thresh && s_label[tid] != C - 1;
        const unsigned m = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) s_warp[warp] = __popc(m);
        __syncthreads();
        int before = 0, total = 0;
#pragma unroll 8
        for (int w = 0; w < kDetrWarps; ++w) {
            const int c = s_warp[w];
            before += w < warp ? c : 0;
            total += c;
        }
        if (keep) {
            const int slot = before + __popc(m & ((1u << lane) - 1u));
            detr_get_rect(img_w, img_h, boxes + (size_t)(q0 + tid) * 4, s_rect[slot]);
            s_src[slot] = tid;
        }
        __syncthreads();
        float* o = out + 1 + (size_t)kept * kDetrRow;
        for (int f = tid; f < total * kDetrRow; f += kDetrThreads) {
            const int r = f / kDetrRow, e = f - r * kDetrRow;
            o[f] = e < 4 ? (float)s_rect[r][e] : (e == 4 ? s_score[s_src[r]] : (float)s_label[s_src[r]]);
        }
        kept += total;
        __syncthreads();  // the next pass reuses the shared arrays
    }
    const size_t end = 1 + (size_t)Q * kDetrRow;
    for (size_t f = 1 + (size_t)kept * kDetrRow + tid; f < end; f += kDetrThreads) out[f] = 0.0f;
    if (tid == 0) out[0] = (float)kept;
}

}  // namespace trtx

using namespace trtx;

extern "C" {

// the rectangle of detr/detr.cpp:795-803 on the host (detr_get_rect in common.cuh, shared with detr_postprocess_kernel)
TRTX_API int trtx_detr_get_rect(int img_w, int img_h, const float box[4], int rect[4]) {
    if (!box || !rect || img_w <= 0 || img_h <= 0) return TRTX_ERR_INVALID;
    detr_get_rect(img_w, img_h, box, rect);
    return TRTX_OK;
}

TRTX_API int trtx_detr_postprocess_enqueue(const trtx_detr_post_params* p, const int32_t* frame_wh_host, int batch,
                                           const float* scores_dev, const float* boxes_dev, float* rows_dev,
                                           trtx_stream_t stream) {
    if (!p || !frame_wh_host || batch <= 0 || !scores_dev || !boxes_dev || !rows_dev) return TRTX_ERR_INVALID;
    // a threshold below -1 would keep the queries whose argmax the reference leaves at label -1, score -1
    if (p->num_queries <= 0 || p->num_classes < 2 || !(p->score_thresh >= -1.f)) return TRTX_ERR_INVALID;
    if (!frames_valid(frame_wh_host, batch)) return TRTX_ERR_INVALID;
    if (p->num_queries > kDetrMaxDim || p->num_classes > kDetrMaxDim) return TRTX_ERR_UNSUPPORTED;
    DetrPostArgs a;
    a.scores = scores_dev;
    a.boxes = boxes_dev;
    a.rows = rows_dev;
    a.num_queries = p->num_queries;
    a.num_classes = p->num_classes;
    a.score_thresh = p->score_thresh;
    return launch_frames(detr_postprocess_kernel, a, a.sizes, batch, kDetrThreads, 0, static_cast<cudaStream_t>(stream),
                         frame_wh(frame_wh_host));
}

}  // extern "C"
