// pyrunner.cu -- the Python runners' post_process for sm_90a.
// Replaces post_process + non_max_suppression + bbox_iou + xywh2xyxy of the detection runners (yolov8/yolov8_det_trt.py:255-381,
// yolov5/yolov5_det_trt.py:250-276; the same bodies in the yolov3, yolov7, yolov9, yolov10, yolo11, yolov12-tubro and yolov13
// runners), which run in numpy on one core per frame.  Their pre-process is trtx_linear_preprocess_enqueue(TRTX_LINEAR_PY).
//
// One 1024-thread CTA per frame, one launch per 64 frames (the frames' geometry rides in the launch parameters):
//   1. the first n rows are read once; conf (times the yolov3 column) >= conf_thresh picks the candidates, which a block
//      rank compacts in row order as desc_key(conf, row) -- no atomics;
//   2. block_bitonic_sort_u64 orders them by descending conf, equal confs by ascending row;
//   3. each sorted candidate's box is mapped to the frame and clipped, in float32 as numpy does, into shared memory with
//      its label (NaN where a corner is NaN: such a pair's IoU is NaN and never suppresses, so the label test stands for it);
//   4. the greedy sweep in chunks of 64 sorted rows: the whole CTA builds the chunk's suppression bitmask against every
//      later row (bbox_iou > nms_thresh and equal labels), then warp 0 resolves the chunk in order, lane w holding word w
//      of the removed set.  A kept row is consumed whether or not it suppresses itself -- the runner's `while` never ends
//      where it does not;
//   5. the kept rows are written as (x1, y1, x2, y2, conf, row[5]), coalesced, and the rest of the row buffer is zeroed.
#include <string.h>

#include "select_sort.cuh"

namespace trtx {

constexpr int kPyThreads = kSelThreads;        // 1024
constexpr int kPyMaxRows = TRTX_NMS_MAX_ROWS;  // 2048
constexpr int kPyWords = kPyMaxRows / 64;      // 32: the removed set fits one warp, a 64-bit word per lane
constexpr int kPyChunk = 64;                   // sorted rows per sweep step: one mask word
constexpr int kPyMaxFrames = 64;               // frames per launch (launch-parameter arrays)
constexpr int kPyRow = 6;

// xywh2xyxy's geometry of one frame, computed on the host in double as Python does and rounded to float as numpy casts a
// Python float against a float32 array: r_w = net_w / w, r_h = net_h / h; if r_h > r_w the pad is (net_h - r_w * h) / 2
// on y and r = r_w, else (net_w - r_h * w) / 2 on x and r = r_h.  xmax, ymax: np.clip's bounds w - 1, h - 1.
struct PyFrame {
    float pad, r, xmax, ymax;
    int on_y;
};

struct PyArgs {
    PyFrame fr[kPyMaxFrames];
    const float* dets;  // [B, 1 + max_rows * row_floats]
    float* rows;        // [B, 1 + max_rows * 6]
    int base, max_rows, row_floats, label_col, conf_col, cxcywh;
    float conf_thresh, nms_thresh;
};

__device__ __forceinline__ float py_conf(const PyArgs& a, const float* d) {
    return a.conf_col >= 0 ? __fmul_rn(d[4], d[a.conf_col]) : d[4];  // `pred[:, 4] *= pred[:, 6]`
}

// np.clip(v, 0, hi) on float32: min(max(v, 0), hi) with numpy's comparisons, so a NaN passes through and -0.0 stays
__device__ __forceinline__ float py_clip(float v, float hi) {
    v = v < 0.f ? 0.f : v;
    return v > hi ? hi : v;
}

// xywh2xyxy then the clip of non_max_suppression, statement by statement (each numpy op rounds on its own)
__device__ __forceinline__ float4 py_map(const PyArgs& a, const PyFrame& f, const float* d) {
    float b[4] = {d[0], d[1], d[2], d[3]};
    if (a.cxcywh) {  // yolov5_det_trt.py:261-274: x - w / 2, x + w / 2, then the pad
        const float hw = __fdiv_rn(d[2], 2.f), hh = __fdiv_rn(d[3], 2.f);
        b[0] = __fsub_rn(d[0], hw);
        b[2] = __fadd_rn(d[0], hw);
        b[1] = __fsub_rn(d[1], hh);
        b[3] = __fadd_rn(d[1], hh);
    }
    const int o = f.on_y ? 1 : 0;
    b[o] = __fsub_rn(b[o], f.pad);
    b[o + 2] = __fsub_rn(b[o + 2], f.pad);
#pragma unroll
    for (int e = 0; e < 4; ++e) b[e] = __fdiv_rn(b[e], f.r);
    return make_float4(py_clip(b[0], f.xmax), py_clip(b[1], f.ymax), py_clip(b[2], f.xmax), py_clip(b[3], f.ymax));
}

// bbox_iou of two clipped boxes without a NaN corner (so max / min need no NaN rule, and no zero's sign reaches the result)
__device__ __forceinline__ float py_iou(const float4 p, const float4 q) {
    const float iw = fmaxf(__fadd_rn(__fsub_rn(fminf(p.z, q.z), fmaxf(p.x, q.x)), 1.f), 0.f);
    const float ih = fmaxf(__fadd_rn(__fsub_rn(fminf(p.w, q.w), fmaxf(p.y, q.y)), 1.f), 0.f);
    const float inter = __fmul_rn(iw, ih);
    const float ap = __fmul_rn(__fadd_rn(__fsub_rn(p.z, p.x), 1.f), __fadd_rn(__fsub_rn(p.w, p.y), 1.f));
    const float aq = __fmul_rn(__fadd_rn(__fsub_rn(q.z, q.x), 1.f), __fadd_rn(__fsub_rn(q.w, q.y), 1.f));
    return __fdiv_rn(inter, __fadd_rn(__fsub_rn(__fadd_rn(ap, aq), inter), 1e-16f));
}

__global__ void __launch_bounds__(kPyThreads) pyrunner_kernel(const __grid_constant__ PyArgs a) {
    extern __shared__ __align__(16) unsigned char smem[];
    __shared__ unsigned long long s_mask[kPyChunk * kPyWords];  // row r of the chunk: word w = the later rows it removes
    __shared__ unsigned long long s_removed[kPyWords];
    __shared__ int s_warp[kPyThreads / kWarp];
    __shared__ int s_kept_n;
    const int tid = threadIdx.x, lane = tid & (kWarp - 1), R = a.row_floats, M = a.max_rows;
    const PyFrame& fr = a.fr[blockIdx.x];
    const size_t b = (size_t)(a.base + blockIdx.x);
    const float* src = a.dets + b * (1 + (size_t)M * R);
    float* out = a.rows + b * (1 + (size_t)M * kPyRow);
    float4* s_box = reinterpret_cast<float4*>(smem);                              // [M], by sorted position
    unsigned long long* s_key = reinterpret_cast<unsigned long long*>(s_box + M);  // [pow2 >= M]
    int S = 1;
    while (S < M) S <<= 1;
    float* s_lab = reinterpret_cast<float*>(s_key + S);  // [M]
    int* s_kept = reinterpret_cast<int*>(s_lab + M);     // [M]: sorted positions of the kept rows

    // `num = int(output[0])`, `[:num]`: truncated, at most M; below 1 (or NaN) no rows
    const float cnt = src[0];
    const int n = cnt >= 1.f ? (cnt < (float)M ? (int)cnt : M) : 0;
    int m = 0;
    for (int i0 = 0; i0 < n; i0 += kPyThreads) {  // uniform
        const int i = i0 + tid;
        float c = 0.f;
        bool cand = false;
        if (i < n) {
            c = py_conf(a, src + 1 + (size_t)i * R);
            cand = c >= a.conf_thresh;
        }
        int total;
        const int rank = block_rank<kPyThreads>(cand, s_warp, &total);
        if (cand) s_key[m + rank] = desc_key(c, (uint32_t)i);
        m += total;
    }
    int Sm = 1;
    while (Sm < m) Sm <<= 1;
    for (int i = m + tid; i < Sm; i += kPyThreads) s_key[i] = ~0ull;
    if (tid < kPyWords) s_removed[tid] = 0ull;
    __syncthreads();
    block_bitonic_sort_u64(s_key, Sm);
    for (int p = tid; p < m; p += kPyThreads) {
        const float* d = src + 1 + (size_t)(uint32_t)s_key[p] * R;
        const float4 bx = py_map(a, fr, d);
        const bool nan = isnan(bx.x) || isnan(bx.y) || isnan(bx.z) || isnan(bx.w);
        s_box[p] = bx;
        s_lab[p] = nan ? __int_as_float(0x7fc00000) : d[a.label_col];
    }
    __syncthreads();

    const int W = (m + kPyChunk - 1) / kPyChunk;
    const float thr = a.nms_thresh;
    int kept = 0;  // warp 0's count
    for (int c = 0; c < W; ++c) {  // uniform
        const int span = W - c, i0 = kPyChunk * c;
        const unsigned long long gone = s_removed[c];
        for (int t = tid; t < kPyChunk * span; t += kPyThreads) {
            const int r = t / span, w = c + (t - r * span), i = i0 + r;
            if (i >= m || ((gone >> r) & 1ull)) continue;  // a removed row's mask is never read
            const float4 bi = s_box[i];
            const float li = s_lab[i];
            unsigned long long bits = 0ull;
            const int j1 = min(m, kPyChunk * w + kPyChunk);
            for (int j = max(i + 1, kPyChunk * w); j < j1; ++j)
                if (li == s_lab[j] && py_iou(bi, s_box[j]) > thr) bits |= 1ull << (j & 63);
            s_mask[r * kPyWords + w] = bits;
        }
        __syncthreads();
        if (tid < kWarp) {
            unsigned long long removed = s_removed[lane];
            const int rows = min(kPyChunk, m - i0);
            for (int r = 0; r < rows; ++r) {
                const unsigned long long word = __shfl_sync(0xffffffffu, removed, c);
                if ((word >> r) & 1ull) continue;  // uniform across the warp
                if (lane == 0) s_kept[kept] = i0 + r;
                ++kept;
                if (lane >= c && lane < W) removed |= s_mask[r * kPyWords + lane];
            }
            s_removed[lane] = removed;
        }
        __syncthreads();
    }
    if (tid == 0) s_kept_n = kept;
    __syncthreads();
    const int K = s_kept_n;
    for (int f = tid; f < K * kPyRow; f += kPyThreads) {
        const int k = f / kPyRow, e = f - k * kPyRow, p = s_kept[k];
        float v;
        if (e < 4) {
            v = reinterpret_cast<const float*>(s_box + p)[e];
        } else {
            const float* d = src + 1 + (size_t)(uint32_t)s_key[p] * R;
            v = e == 4 ? py_conf(a, d) : d[5];
        }
        out[1 + f] = v;
    }
    const size_t end = 1 + (size_t)M * kPyRow;
    for (size_t f = 1 + (size_t)K * kPyRow + tid; f < end; f += kPyThreads) out[f] = 0.f;
    if (tid == 0) out[0] = (float)K;
}

inline size_t py_smem(int max_rows) {
    size_t s = 1;
    while (s < (size_t)max_rows) s <<= 1;
    return (size_t)max_rows * (sizeof(float4) + sizeof(float) + sizeof(int)) + s * sizeof(unsigned long long);
}

}  // namespace trtx

using namespace trtx;

extern "C" {

TRTX_API int trtx_pyrunner_postprocess_enqueue(const trtx_pyrunner_params* p, const int32_t* frame_wh_host, int batch,
                                               const float* dets_dev, int max_rows, float* rows_dev, trtx_stream_t stream) {
    if (!p || !frame_wh_host || !dets_dev || !rows_dev || batch <= 0 || max_rows <= 0) return TRTX_ERR_INVALID;
    if (p->box_format != TRTX_BOX_LTRB && p->box_format != TRTX_BOX_CXCYWH) return TRTX_ERR_INVALID;
    if (p->net_w <= 0 || p->net_h <= 0 || p->label_col < 5 || p->label_col >= p->row_floats) return TRTX_ERR_INVALID;
    if (p->conf_col != -1 && (p->conf_col < 5 || p->conf_col >= p->row_floats || p->conf_col == p->label_col))
        return TRTX_ERR_INVALID;
    if (p->conf_thresh != p->conf_thresh || p->nms_thresh != p->nms_thresh) return TRTX_ERR_INVALID;
    if (reinterpret_cast<uintptr_t>(dets_dev) % sizeof(float) || reinterpret_cast<uintptr_t>(rows_dev) % sizeof(float))
        return TRTX_ERR_INVALID;
    if (max_rows > kPyMaxRows) return TRTX_ERR_UNSUPPORTED;
    for (int i = 0; i < batch; ++i)
        if (frame_wh_host[2 * i] <= 0 || frame_wh_host[2 * i + 1] <= 0) return TRTX_ERR_INVALID;
    const size_t smem = py_smem(max_rows);
    if (cudaFuncSetAttribute(pyrunner_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
        g_last_cuda_error = (int)cudaGetLastError();
        return TRTX_ERR_CUDA;
    }
    PyArgs a;
    memset(&a, 0, sizeof(a));
    a.dets = dets_dev;
    a.rows = rows_dev;
    a.max_rows = max_rows;
    a.row_floats = p->row_floats;
    a.label_col = p->label_col;
    a.conf_col = p->conf_col;
    a.cxcywh = p->box_format == TRTX_BOX_CXCYWH;
    a.conf_thresh = p->conf_thresh;
    a.nms_thresh = p->nms_thresh;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    for (int i0 = 0; i0 < batch; i0 += kPyMaxFrames) {
        const int n = min(batch - i0, kPyMaxFrames);
        a.base = i0;
        for (int j = 0; j < n; ++j) {
            const int w = frame_wh_host[2 * (i0 + j)], h = frame_wh_host[2 * (i0 + j) + 1];
            const double r_w = (double)p->net_w / w, r_h = (double)p->net_h / h;
            PyFrame& f = a.fr[j];
            f.on_y = r_h > r_w;
            f.pad = f.on_y ? (float)((p->net_h - r_w * h) / 2) : (float)((p->net_w - r_h * w) / 2);
            f.r = f.on_y ? (float)r_w : (float)r_h;
            f.xmax = (float)(w - 1);
            f.ymax = (float)(h - 1);
        }
        pyrunner_kernel<<<n, kPyThreads, smem, st>>>(a);
        const int rc = check_launch();
        if (rc) return rc;
    }
    return TRTX_OK;
}

}  // extern "C"
