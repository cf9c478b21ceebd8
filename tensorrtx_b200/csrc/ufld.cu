// ufld.cu -- UFLD (Ultra-Fast Lane Detection, row anchors) post-process for sm_90a: the driver's host stages after inference
// on the device.  Replaces, per batch, the D2H copy of `prob` [C, H, W] and the host loops of ufld/lane_det.cpp:358-410:
//     the row flip                          prob_reverse[k][H - 1 - j][l] = prob[k][j][l]
//     argmax (:251-270)                     int max = -10000000, max_ind = -1; for c: if (v > max) max = v (truncated), max_ind = c
//     softmax_mul (:224-249)                e_c = exp(v_c), sum += e_c, then expect += (e_c / sum) * (c + 1), over c < C - 1
//     "no lane"                             expect = 0 where max_ind == C - 1 (the driver's literal 100)
//     the lanes                             lane l is kept when more than 2 of its H cells have expect != 0
//     the points                            per kept cell with expect > 0: x = int(expect * col_sample_w * w / net_w) - 1,
//                                           y = h * anchor[j] / net_h - 1 (int)
// into rows (x, y, lane) in the driver's draw order: engine rows j = H - 1 .. 0, the kept lanes ascending in each.
//
// One CTA of kUfldThreads per frame:
//   1. every thread computes e = (float)exp((double)v) for a strided share of the (C - 1) * H * W logits into shared memory;
//   2. thread t < H * W owns cell t (row t / W, lane t % W): the argmax over the C logits, then the float sum of its e in
//      c order, then the expectation in c order -- each statement of the reference rounded as it is there (_rn intrinsics);
//   3. W threads count each lane's non-zero cells;
//   4. thread t takes draw position t (flipped row t / W, lane t % W); a ballot per warp and a scan of the warps' counts give
//      each point its row (no atomics).  Rows past the count are zeroed, and float 0 gets the count.
#include "common.cuh"

namespace trtx {

constexpr int kUfldThreads = 1024;        // H * W <= kUfldThreads: one thread per cell, one per draw position
constexpr int kUfldWarps = kUfldThreads / kWarp;
constexpr int kUfldMaxTable = 52 * 1024;  // (C - 1) * H * W exponentials in dynamic shared memory (208 KiB)
constexpr int kUfldMaxSide = 1 << 24;     // frame sides: the rows are exact floats
constexpr int kUfldRow = 3;               // x, y, lane

struct UfldPostArgs {
    FrameSizes sizes;          // of the picture the points are for
    int C, H, W, net_w, net_h, col_sample_w;
    int anchor[kUfldThreads];  // H row anchors
    const float* prob;         // [B, C, H, W]
    float* rows;               // [B, 1 + H * W * 3]
};

// exp of a float as the double exp, rounded once to float: the correctly rounded expf except within about 2^-29 of a
// rounding boundary (DESIGN §4.8)
__device__ __forceinline__ float ufld_exp(float v) { return __double2float_rn(exp((double)v)); }

__global__ void __launch_bounds__(kUfldThreads) ufld_postprocess_kernel(const __grid_constant__ UfldPostArgs a) {
    extern __shared__ float s_e[];               // [C - 1][H * W]
    __shared__ float s_expect[kUfldThreads];     // per cell
    __shared__ unsigned char s_lane[kUfldThreads];  // lane kept
    __shared__ int s_warp[kUfldWarps];           // points per warp
    const int tid = threadIdx.x, lane = tid & (kWarp - 1), warp = tid / kWarp, b = a.sizes.base + blockIdx.x;
    const int C = a.C, H = a.H, W = a.W, HW = H * W;
    const float* prob = a.prob + (size_t)b * C * HW;
    float* out = a.rows + (size_t)b * (1 + (size_t)HW * kUfldRow);

    for (int i = tid; i < (C - 1) * HW; i += kUfldThreads) s_e[i] = ufld_exp(__ldg(prob + i));
    __syncthreads();

    if (tid < HW) {
        int max = -10000000, max_ind = -1;
        for (int c = 0; c < C; ++c) {
            const float v = __ldg(prob + (size_t)c * HW + tid);
            if (v > (float)max) {  // the int converts to float; a NaN is never taken
                max = trunc_to_int_x86(v);
                max_ind = c;
            }
        }
        float sum = 0.0f, expect = 0.0f;
        for (int c = 0; c < C - 1; ++c) sum = __fadd_rn(sum, s_e[c * HW + tid]);
        for (int c = 0; c < C - 1; ++c) expect = __fadd_rn(expect, __fmul_rn(__fdiv_rn(s_e[c * HW + tid], sum), (float)(c + 1)));
        s_expect[tid] = max_ind == C - 1 ? 0.0f : expect;
    }
    __syncthreads();
    if (tid < W) {
        int n = 0;
        for (int j = 0; j < H; ++j) n += s_expect[j * W + tid] != 0.0f;  // a NaN counts
        s_lane[tid] = n > 2;
    }
    __syncthreads();

    const int l = tid % W, j = H - 1 - tid / W;  // draw position tid: the flipped row tid / W
    const float e = tid < HW ? s_expect[j * W + l] : 0.0f;
    const bool emit = tid < HW && s_lane[l] && e > 0.0f;
    const unsigned m = __ballot_sync(0xffffffffu, emit);
    if (lane == 0) s_warp[warp] = __popc(m);
    __syncthreads();
    int before = 0, total = 0;
#pragma unroll 8
    for (int w = 0; w < kUfldWarps; ++w) {
        const int c = s_warp[w];
        before += w < warp ? c : 0;
        total += c;
    }
    if (emit) {
        const int ow = a.sizes.w[blockIdx.x], oh = a.sizes.h[blockIdx.x];
        const float fx = __fdiv_rn(__fmul_rn(__fmul_rn(e, (float)a.col_sample_w), (float)ow), (float)a.net_w);
        const int x = (int)((uint32_t)trunc_to_int_x86(fx) - 1u);  // wraps as on x86-64
        const int y = oh * a.anchor[j] / a.net_h - 1;               // in range: checked on the host
        float* o = out + 1 + (size_t)(before + __popc(m & ((1u << lane) - 1u))) * kUfldRow;
        o[0] = (float)x;
        o[1] = (float)y;
        o[2] = (float)l;
    }
    for (int f = 1 + total * kUfldRow + tid; f < 1 + HW * kUfldRow; f += kUfldThreads) out[f] = 0.0f;
    if (tid == 0) out[0] = (float)total;
}

}  // namespace trtx

using namespace trtx;

extern "C" {

TRTX_API int trtx_ufld_postprocess_enqueue(const trtx_ufld_post_params* p, const int32_t* row_anchor_host,
                                           const int32_t* frame_wh_host, int batch, const float* prob_dev, float* rows_dev,
                                           trtx_stream_t stream) {
    if (!p || !row_anchor_host || !frame_wh_host || batch <= 0 || !prob_dev || !rows_dev) return TRTX_ERR_INVALID;
    const int C = p->num_cells, H = p->num_rows, W = p->num_lanes;
    if (C < 2 || H <= 0 || W <= 0 || p->net_w <= 0 || p->net_h <= 0 || p->col_sample_w <= 0) return TRTX_ERR_INVALID;
    if (!frames_valid(frame_wh_host, batch)) return TRTX_ERR_INVALID;
    if ((int64_t)H * W > kUfldThreads || (int64_t)(C - 1) * H * W > kUfldMaxTable) return TRTX_ERR_UNSUPPORTED;
    // every frame and anchor is checked before the first launch, so that a rejected call writes nothing: h * anchor must not
    // overflow int32 (the driver's int product), and the point's y must be an exact float
    for (int i = 0; i < batch; ++i) {
        int w, h;
        frame_wh(frame_wh_host)(i, w, h);
        if (w > kUfldMaxSide || h > kUfldMaxSide) return TRTX_ERR_UNSUPPORTED;
        for (int j = 0; j < H; ++j) {
            const int64_t prod = (int64_t)h * row_anchor_host[j];
            if (prod < INT32_MIN || prod > INT32_MAX) return TRTX_ERR_UNSUPPORTED;
            const int64_t y = prod / p->net_h - 1;
            if (y < -kUfldMaxSide || y > kUfldMaxSide) return TRTX_ERR_UNSUPPORTED;
        }
    }
    const size_t smem = (size_t)(C - 1) * H * W * sizeof(float);
    if (const int rc = opt_in_smem(ufld_postprocess_kernel, smem)) return rc;
    UfldPostArgs a;
    a.prob = prob_dev;
    a.rows = rows_dev;
    a.C = C, a.H = H, a.W = W;
    a.net_w = p->net_w, a.net_h = p->net_h, a.col_sample_w = p->col_sample_w;
    for (int j = 0; j < H; ++j) a.anchor[j] = row_anchor_host[j];
    return launch_frames(ufld_postprocess_kernel, a, a.sizes, batch, kUfldThreads, smem, static_cast<cudaStream_t>(stream),
                         frame_wh(frame_wh_host));
}

}  // extern "C"
