// refinedet.cu -- RefineDet post-process for sm_90a.
// Replaces the libtorch post-process of refinedet/refinedet.cpp (doInference, :730-791: PriorBox, the two-step decode, the
// ARM objectness filter and the per-class nms(), all in float64) and the driver's rectangles (:957-993, RoiCorrect :22-35).
// The pre-process (base_transform) is the whole-frame stretch of preprocess.cu.
//
// Two launches, no atomics on global memory, no host synchronisation:
//   1. refinedet_nms_kernel, one CTA per (frame, class c >= 1): the candidates (score > conf_thresh after the ARM filter)
//      are counted; above top_k, block_select_topk cuts them to the top_k best.  The kept ones are compacted into shared
//      memory as desc_key(score, prior), sorted by block_bitonic_sort_u64 and decoded (priors computed in the kernel, the
//      ARM step, the ODM step and the corners, all float64 without contraction).  A suppression bitmask over the sorted
//      boxes (j suppressed by i < j), then one warp resolves it in order; the kept priors and their count go to the
//      workspace.
//   2. refinedet_rows_kernel, one CTA of 512 threads per frame (one launch per 64 frames): the classes are concatenated in
//      class order, the first max_det rows are decoded again (the same code, so the same bits) and written; with frame
//      sizes, the driver's score filter, rectangles and RoiCorrect give the frame rows.
// Order within a class: descending score, ties to the lower prior index (torch::sort on CUDA leaves ties open).
#include "common.cuh"
#include "select_sort.cuh"

namespace trtx {

constexpr int kRdThreads = kSelThreads;  // 1024: block_select_topk's block
constexpr int kRdRowsThreads = 512;      // the rows kernel: two exp chains per row need more than 64 registers
constexpr int kRdMaxTopK = 1024;
constexpr int kRdMaxPriors = 1 << 16;    // prior indices are stored as uint16
constexpr int kRdMaxClasses = 1024;
constexpr int kRdMaxDet = 1 << 24;       // counts are stored as floats
constexpr int kRdMaxSide = 1 << 24;      // frame sides: rectangles are stored as floats
constexpr int kRdMaxFrames = 64;         // frames per rows launch (launch-parameter arrays)
constexpr int kRdRow = 6;

struct RdArgs {
    const float* arm_loc;   // [B, P, 4]
    const float* arm_conf;  // [B, P, 2]
    const float* odm_loc;   // [B, P, 4]
    const float* odm_conf;  // [B, P, C]
    int32_t* count;         // workspace [B, C - 1]
    uint16_t* keep;         // workspace [B, C - 1, top_k]
    float* dets;            // [B, 1 + max_det * 6]
    float* rows;            // [B, 1 + max_det * 6] or null
    int net, P, C, top_k, max_det, base;
    float obj_thresh, conf_thresh, nms_thresh, score_thresh;
    int wh[2 * kRdMaxFrames];
};

// Priors of a square net S: levels k = 0..3 with step 8 << k, min_size 32 << k and f = S / step cells a side; prior index
// = level offset + (i * f + j) * 3 + a.  Every statement of PriorBox (:553-597) in float and double as there; sqrt(ar) is the
// float overload, sqrtf(2.f), widened (the double one gives the same table at S = 320, not at every S: trtx_hot.h).  Then
// clamp(0, 1).
__device__ __forceinline__ void rd_prior(int p, int net, double pr[4]) {
    int k = 0, f = net >> 3;
    while (k < 3 && p >= 3 * f * f) {
        p -= 3 * f * f;
        ++k;
        f >>= 1;
    }
    const int cell = p / 3, a = p - 3 * cell, i = cell / f, j = cell - i * f;
    const float fk = __double2float_rn(__ddiv_rn((double)net, (double)(8 << k)));
    const float cx = __double2float_rn(__ddiv_rn(__dadd_rn((double)j, 0.5), (double)fk));
    const float cy = __double2float_rn(__ddiv_rn(__dadd_rn((double)i, 0.5), (double)fk));
    const float sk = __double2float_rn(__ddiv_rn((double)(32 << k), (double)net));
    const double sq = (double)1.41421353816986083984375f;  // sqrtf(2.f)
    const float big = __double2float_rn(__dmul_rn((double)sk, sq)), small = __double2float_rn(__ddiv_rn((double)sk, sq));
    const float w = a == 0 ? sk : (a == 1 ? big : small), h = a == 0 ? sk : (a == 1 ? small : big);
    pr[0] = (double)fminf(fmaxf(cx, 0.f), 1.f);
    pr[1] = (double)fminf(fmaxf(cy, 0.f), 1.f);
    pr[2] = (double)fminf(fmaxf(w, 0.f), 1.f);
    pr[3] = (double)fminf(fmaxf(h, 0.f), 1.f);
}

// decode (:600-619) twice, in double, each libtorch op rounded on its own: d = (p01 + (l01 * v0) * p23, p23 * exp(l23 * v1))
// over the prior with arm_loc, then over d with odm_loc, then x1 = cx - w / 2, x2 = x1 + w.  exp is CUDA's double exp, the one
// ATen's CUDA kernel calls.
__device__ __forceinline__ void rd_decode(const RdArgs& a, int b, int p, double box[4]) {
    double pr[4];
    rd_prior(p, a.net, pr);
    const float* al = a.arm_loc + ((size_t)b * a.P + p) * 4;
    const float* ol = a.odm_loc + ((size_t)b * a.P + p) * 4;
    const double v0 = (double)0.1f, v1 = (double)0.2f;
#pragma unroll
    for (int e = 0; e < 2; ++e) {
        const double d0 = __dadd_rn(pr[e], __dmul_rn(__dmul_rn((double)__ldg(al + e), v0), pr[2 + e]));
        const double d1 = __dmul_rn(pr[2 + e], exp(__dmul_rn((double)__ldg(al + 2 + e), v1)));
        const double c = __dadd_rn(d0, __dmul_rn(__dmul_rn((double)__ldg(ol + e), v0), d1));
        const double s = __dmul_rn(d1, exp(__dmul_rn((double)__ldg(ol + 2 + e), v1)));
        box[e] = __dsub_rn(c, __ddiv_rn(s, 2.0));
        box[2 + e] = __dadd_rn(box[e], s);
    }
}

// The score of class c at prior p after the ARM filter (:738-746): kept where arm_conf[p, 1] > obj_thresh, else times 0.0
// (so an inf or NaN score becomes NaN).  The float product is the double one rounded, exactly.
__device__ __forceinline__ float rd_score(const RdArgs& a, int b, int p, int c) {
    const float s = __ldg(a.odm_conf + ((size_t)b * a.P + p) * a.C + c);
    return __ldg(a.arm_conf + ((size_t)b * a.P + p) * 2 + 1) > a.obj_thresh ? s : __fmul_rn(s, 0.f);
}

// Tensor::clamp(lo, hi) on CUDA: a NaN bound fills the result with NaN, a NaN value stays, else min(max(v, lo), hi)
__device__ __forceinline__ double rd_clamp(double v, double lo, double hi) {
    if (isnan(lo) || isnan(hi)) return __longlong_as_double(0x7ff8000000000000ll);
    return isnan(v) ? v : fmin(fmax(v, lo), hi);
}

struct RdNmsScratch {
    SelectScratch sel;
    int n;
};

__global__ void __launch_bounds__(kRdThreads) refinedet_nms_kernel(const __grid_constant__ RdArgs a) {
    extern __shared__ __align__(16) unsigned char smem[];
    __shared__ RdNmsScratch sc;
    const int tid = threadIdx.x, lane = tid & (kWarp - 1), ncls = a.C - 1;
    const int b = blockIdx.x / ncls, c = 1 + blockIdx.x % ncls, K = a.top_k, W = (K + 63) / 64;
    unsigned long long* s_key = reinterpret_cast<unsigned long long*>(smem);  // kRdMaxTopK
    double* s_box = reinterpret_cast<double*>(s_key + kRdMaxTopK);          // x1, y1, x2, y2, area: 5 runs of K
    unsigned long long* s_mask = reinterpret_cast<unsigned long long*>(s_box + 5 * K);  // K x W
    auto key = [&](int p) -> uint32_t {
        const float s = rd_score(a, b, p, c);
        return s > a.conf_thresh ? float_key(s) : 0u;  // a candidate is never NaN, so its key is above 0
    };
    if (tid == 0) sc.n = 0;
    __syncthreads();
    int cnt = 0;
    for (int p = tid; p < a.P; p += kRdThreads) cnt += key(p) != 0u;
    if (cnt) atomicAdd(&sc.n, cnt);
    __syncthreads();
    const int total = sc.n;
    __syncthreads();
    uint32_t key_cut = 1u, id_cut = 0xffffffffu;  // everything with a key above 0
    if (total > K) block_select_topk(key, a.P, K, sc.sel, &key_cut, &id_cut);
    if (tid == 0) sc.n = 0;
    __syncthreads();
    for (int p = tid; p < a.P; p += kRdThreads) {
        const uint32_t kk = key(p);
        if (kk != 0u && (kk > key_cut || (kk == key_cut && (uint32_t)p <= id_cut)))
            s_key[atomicAdd(&sc.n, 1)] = ((unsigned long long)(~kk) << 32) | (uint32_t)p;
    }
    __syncthreads();
    const int m = sc.n;
    int S = 1;
    while (S < m) S <<= 1;
    for (int i = m + tid; i < S; i += kRdThreads) s_key[i] = ~0ull;
    __syncthreads();
    block_bitonic_sort_u64(s_key, S);
    if (tid < m) {
        double box[4];
        rd_decode(a, b, (int)(s_key[tid] & 0xffffffffu), box);
#pragma unroll
        for (int e = 0; e < 4; ++e) s_box[e * K + tid] = box[e];
        s_box[4 * K + tid] = __dmul_rn(__dsub_rn(box[2], box[0]), __dsub_rn(box[3], box[1]));
    }
    __syncthreads();
    // bit j of row i: the kept box i suppresses j > i (nms :669-692).  i's bounds are its coordinates rounded to float
    // (`x1[i].item().toFloat()`), its area is not; IoU = inter * 1.0 / ((area_j - inter) + area_i), kept iff < nms_thresh,
    // so a NaN IoU suppresses.
    const int Wm = (m + 63) / 64;
    const double nms = (double)a.nms_thresh, imax = 2147483647.0, imin = -2147483648.0;
    for (int t = tid; t < m * Wm; t += kRdThreads) {
        const int i = t / Wm, w = t - i * Wm;
        if (w < (i >> 6)) continue;
        const double bx1 = (double)__double2float_rn(s_box[i]), by1 = (double)__double2float_rn(s_box[K + i]);
        const double bx2 = (double)__double2float_rn(s_box[2 * K + i]), by2 = (double)__double2float_rn(s_box[3 * K + i]);
        const double ai = s_box[4 * K + i];
        unsigned long long bits = 0ull;
        const int j1 = min(m, 64 * w + 64);
        for (int j = max(i + 1, 64 * w); j < j1; ++j) {
            const double xx1 = rd_clamp(s_box[j], bx1, imax), yy1 = rd_clamp(s_box[K + j], by1, imax);
            const double xx2 = rd_clamp(s_box[2 * K + j], imin, bx2), yy2 = rd_clamp(s_box[3 * K + j], imin, by2);
            const double iw = rd_clamp(__dsub_rn(xx2, xx1), 0.0, imax), ih = rd_clamp(__dsub_rn(yy2, yy1), 0.0, imax);
            const double inter = __dmul_rn(iw, ih);
            const double iou = __ddiv_rn(__dmul_rn(inter, 1.0), __dadd_rn(__dsub_rn(s_box[4 * K + j], inter), ai));
            if (!(iou < nms)) bits |= 1ull << (j & 63);
        }
        s_mask[i * W + w] = bits;
    }
    __syncthreads();
    if (tid >= kWarp) return;
    // the greedy sweep in score order: lane w holds word w of the removed set
    uint16_t* keep = a.keep + ((size_t)b * ncls + (c - 1)) * K;
    unsigned long long removed = 0ull;
    int nk = 0;
    for (int i = 0; i < m; ++i) {
        const unsigned long long word = __shfl_sync(0xffffffffu, removed, i >> 6);
        if ((word >> (i & 63)) & 1ull) continue;  // uniform across the warp
        if (lane < Wm && lane >= (i >> 6)) removed |= s_mask[i * W + lane];
        if (lane == 0) keep[nk] = (uint16_t)(s_key[i] & 0xffffffffu);
        ++nk;
    }
    if (lane == 0) a.count[(size_t)b * ncls + (c - 1)] = nk;
}

// The driver's rectangle (:974-980): r.x = x1 * cols (float times int, then the int conversion), r.width = x2 * cols - r.x
// in float, likewise y and height, then RoiCorrect (:22-35) statement by statement.  Conversions as x86-64 performs them
// (trunc_to_int_x86), and `r.x + r.width` wraps as there.
__device__ __forceinline__ void rd_rect(const float box[4], int cols, int rows, int r[4]) {
    const float fc = (float)cols, fr = (float)rows;
    int x = trunc_to_int_x86(__fmul_rn(box[0], fc)), y = trunc_to_int_x86(__fmul_rn(box[1], fr));
    int w = trunc_to_int_x86(__fsub_rn(__fmul_rn(box[2], fc), (float)x));
    int h = trunc_to_int_x86(__fsub_rn(__fmul_rn(box[3], fr), (float)y));
    if (x < 0) x = 0;
    if (y < 0) y = 0;
    if (x >= cols - 1) x = 0;
    if (y >= rows - 1) y = 0;
    if (w <= 0) w = 1;
    if (h <= 0) h = 1;
    if ((int)((uint32_t)x + (uint32_t)w) > cols - 1) w = cols - 1 - x;
    if ((int)((uint32_t)y + (uint32_t)h) > rows - 1) h = rows - 1 - y;
    r[0] = x;
    r[1] = y;
    r[2] = w;
    r[3] = h;
}

__global__ void __launch_bounds__(kRdRowsThreads) refinedet_rows_kernel(const __grid_constant__ RdArgs a) {
    __shared__ int s_off[kRdMaxClasses];  // s_off[k]: rows of classes 1..k
    __shared__ int s_warp[kRdRowsThreads / kWarp];
    const int tid = threadIdx.x, b = a.base + blockIdx.x, ncls = a.C - 1, K = a.top_k;
    const int32_t* cnt = a.count + (size_t)b * ncls;
    if (tid == 0) {
        int o = 0;
        s_off[0] = 0;
        for (int k = 0; k < ncls; ++k) s_off[k + 1] = o += cnt[k];
    }
    __syncthreads();
    const int n = min(s_off[ncls], a.max_det), len = 1 + a.max_det * kRdRow;
    float* dets = a.dets + (size_t)b * len;
    float* rows = a.rows ? a.rows + (size_t)b * len : nullptr;
    const int cols = a.wh[2 * blockIdx.x], frows = a.wh[2 * blockIdx.x + 1];
    int kept = 0;
    for (int r0 = 0; r0 < n; r0 += kRdRowsThreads) {  // uniform
        const int r = r0 + tid;
        float box[4] = {0.f, 0.f, 0.f, 0.f}, score = 0.f, label = 0.f;
        if (r < n) {
            int lo = 0, hi = ncls - 1;  // the class k with s_off[k] <= r < s_off[k + 1]
            while (lo < hi) {
                const int mid = (lo + hi + 1) >> 1;
                if (s_off[mid] <= r) lo = mid;
                else hi = mid - 1;
            }
            const int p = a.keep[((size_t)b * ncls + lo) * K + (r - s_off[lo])];
            double d[4];
            rd_decode(a, b, p, d);
#pragma unroll
            for (int e = 0; e < 4; ++e) box[e] = __double2float_rn(d[e]);
            score = rd_score(a, b, p, lo + 1);
            label = (float)(lo + 1);
            float* o = dets + 1 + (size_t)r * kRdRow;
#pragma unroll
            for (int e = 0; e < 4; ++e) o[e] = box[e];
            o[4] = score;
            o[5] = label;
        }
        if (!rows) continue;  // uniform
        const bool keep = r < n && !(score < a.score_thresh);  // the driver's `if (score < TH) continue`
        int t;
        const int rank = block_rank<kRdRowsThreads>(keep, s_warp, &t);
        if (keep) {
            int rc[4];
            rd_rect(box, cols, frows, rc);
            float* o = rows + 1 + (size_t)(kept + rank) * kRdRow;
#pragma unroll
            for (int e = 0; e < 4; ++e) o[e] = (float)rc[e];
            o[4] = score;
            o[5] = label;
        }
        kept += t;
    }
    for (int f = 1 + n * kRdRow + tid; f < len; f += kRdRowsThreads) dets[f] = 0.f;
    if (tid == 0) dets[0] = (float)n;
    if (!rows) return;
    for (int f = 1 + kept * kRdRow + tid; f < len; f += kRdRowsThreads) rows[f] = 0.f;
    if (tid == 0) rows[0] = (float)kept;
}

// P = 3 * sum over the four levels of (S / step)^2
inline int64_t rd_num_priors(int net) {
    int64_t n = 0;
    for (int k = 0; k < 4; ++k) n += 3 * (int64_t)(net >> (3 + k)) * (net >> (3 + k));
    return n;
}

inline size_t rd_nms_smem(int top_k) {
    return (size_t)kRdMaxTopK * 8 + (size_t)5 * top_k * 8 + (size_t)top_k * ((top_k + 63) / 64) * 8;
}

}  // namespace trtx

using namespace trtx;

extern "C" {

// Everything in the parameters that can reject a post-process call, before the first launch; TRTX_OK or the error code.
static int refinedet_check(const trtx_refinedet_params* p, int batch) {
    if (!p || batch <= 0) return TRTX_ERR_INVALID;
    if (p->net <= 0 || p->num_classes < 2 || p->top_k <= 0 || p->max_det <= 0) return TRTX_ERR_INVALID;
    if (p->obj_thresh != p->obj_thresh || p->conf_thresh != p->conf_thresh || p->nms_thresh != p->nms_thresh ||
        p->score_thresh != p->score_thresh)
        return TRTX_ERR_INVALID;
    if (p->net % 64 != 0 || rd_num_priors(p->net) > kRdMaxPriors || p->top_k > kRdMaxTopK ||
        p->num_classes > kRdMaxClasses || p->max_det > kRdMaxDet)
        return TRTX_ERR_UNSUPPORTED;
    return TRTX_OK;
}

TRTX_API size_t trtx_refinedet_workspace_size(const trtx_refinedet_params* p, int batch) {
    if (refinedet_check(p, batch) != TRTX_OK) return 0;
    const size_t lists = (size_t)batch * (p->num_classes - 1);
    return align_up(lists * sizeof(int32_t)) + align_up(lists * p->top_k * sizeof(uint16_t));
}

TRTX_API int trtx_refinedet_postprocess_enqueue(const trtx_refinedet_params* p, int batch, const float* arm_loc_dev,
                                                const float* arm_conf_dev, const float* odm_loc_dev, const float* odm_conf_dev,
                                                void* workspace_dev, size_t workspace_bytes, float* dets_dev,
                                                const int32_t* frame_wh_host, float* rows_dev, trtx_stream_t stream) {
    const int rc0 = refinedet_check(p, batch);
    if (rc0 != TRTX_OK) return rc0;
    if (!arm_loc_dev || !arm_conf_dev || !odm_loc_dev || !odm_conf_dev || !workspace_dev || !dets_dev) return TRTX_ERR_INVALID;
    if (!frame_wh_host != !rows_dev) return TRTX_ERR_INVALID;  // the frame rows need both
    if (frame_wh_host) {
        for (int i = 0; i < batch; ++i) {
            const int w = frame_wh_host[2 * i], h = frame_wh_host[2 * i + 1];
            if (w <= 0 || h <= 0) return TRTX_ERR_INVALID;
            if (w > kRdMaxSide || h > kRdMaxSide) return TRTX_ERR_UNSUPPORTED;
        }
    }
    if (workspace_bytes < trtx_refinedet_workspace_size(p, batch)) return TRTX_ERR_WORKSPACE;
    if (reinterpret_cast<uintptr_t>(workspace_dev) % kAlign) return TRTX_ERR_INVALID;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t smem = rd_nms_smem(p->top_k);
    if (cudaFuncSetAttribute(refinedet_nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
        g_last_cuda_error = (int)cudaGetLastError();
        return TRTX_ERR_CUDA;
    }
    RdArgs a;
    a.arm_loc = arm_loc_dev;
    a.arm_conf = arm_conf_dev;
    a.odm_loc = odm_loc_dev;
    a.odm_conf = odm_conf_dev;
    const size_t lists = (size_t)batch * (p->num_classes - 1);
    a.count = static_cast<int32_t*>(workspace_dev);
    a.keep = reinterpret_cast<uint16_t*>(static_cast<char*>(workspace_dev) + align_up(lists * sizeof(int32_t)));
    a.dets = dets_dev;
    a.rows = rows_dev;
    a.net = p->net;
    a.P = (int)rd_num_priors(p->net);
    a.C = p->num_classes;
    a.top_k = p->top_k;
    a.max_det = p->max_det;
    a.obj_thresh = p->obj_thresh;
    a.conf_thresh = p->conf_thresh;
    a.nms_thresh = p->nms_thresh;
    a.score_thresh = p->score_thresh;
    a.base = 0;
    for (int j = 0; j < 2 * kRdMaxFrames; ++j) a.wh[j] = 0;
    refinedet_nms_kernel<<<(unsigned)lists, kRdThreads, smem, st>>>(a);
    int rc = check_launch();
    if (rc) return rc;
    for (int i0 = 0; i0 < batch; i0 += kRdMaxFrames) {
        const int n = min(batch - i0, kRdMaxFrames);
        a.base = i0;
        for (int j = 0; frame_wh_host && j < n; ++j) {
            a.wh[2 * j] = frame_wh_host[2 * (i0 + j)];
            a.wh[2 * j + 1] = frame_wh_host[2 * (i0 + j) + 1];
        }
        refinedet_rows_kernel<<<n, kRdRowsThreads, 0, st>>>(a);
        rc = check_launch();
        if (rc) return rc;
    }
    return TRTX_OK;
}

}  // extern "C"
