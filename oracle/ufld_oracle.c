/*
 * ufld_oracle.c -- CPU ORACLE of the UFLD lane-detection pre- and post-process.  TEST INFRASTRUCTURE ONLY, like trtx_oracle.c:
 * plain C, single thread, built with -ffp-contract=off, independent of the library's code.
 *   prepareImage      ufld/lane_det.cpp:194-221
 *   argmax            :251-270, restated with the reference's signature (the reference's own build is compared with it)
 *   softmax_mul       :224-249, likewise
 *   the driver loop   :358-410 (the row flip, argmax, softmax_mul, the "no lane" zeroing, the lane choice and the points),
 *                     restated statement by statement for one frame: it sits inside the driver's main(), next to the engine
 *                     calls, so there is no reference build of it.
 * Pinned to cv2 and to the reference's compiled functions by tests/test_ufld_cpu.py.
 */
/* cls_oracle.c's 8-bit INTER_LINEAR resize (resize_linear_u8), a static function: this oracle includes that file, so the
 * library also exports the classification oracle's entry points. */
#include "cls_oracle.c"

#include <limits.h>

/* ------------------------------------------------------------------------------------------
 * prepareImage for one image: cvtColor BGR2RGB; cv::resize(img, resized, Size(net_w, net_h)) of the whole frame, 8-bit
 * INTER_LINEAR; convertTo(CV_32FC3, 1. / 255.) (a float product by (float)(1. / 255.)); cv::split; per plane c the MatExpr
 * `(ch - mean[c]) / std[c]`, which OpenCV 4.x evaluates as one convertTo(-1, 1 / std, -mean / std) (alpha and beta in double
 * from the float literals, cast to float, fused: fmaf).  out: [3, net_h, net_w] fp32 in R, G, B order.
 * ------------------------------------------------------------------------------------------ */
static const float kMean[3] = {0.485, 0.456, 0.406}, kStd[3] = {0.229, 0.224, 0.225};  /* the driver's `static float` */

ORACLE_API float oracle_ufld_input_value(int c, int u) {
    const float s = (float)u * (float)(1. / 255.);
    const double alpha = 1.0 / (double)kStd[c], beta = -(double)kMean[c] / (double)kStd[c];
    return fmaf(s, (float)alpha, (float)beta);
}

ORACLE_API void oracle_ufld_preprocess(const uint8_t* img, int img_w, int img_h, size_t pitch, int net_w, int net_h,
                                       float* out) {
    uint8_t* re = (uint8_t*)malloc((size_t)net_w * net_h * 3);
    resize_linear_u8(img, img_w, img_h, pitch, net_w, net_h, re);  /* per channel: the same bytes after or before cvtColor */
    const size_t plane = (size_t)net_w * net_h;
    for (int c = 0; c < 3; ++c)
        for (size_t i = 0; i < plane; ++i) out[(size_t)c * plane + i] = oracle_ufld_input_value(c, re[3 * i + (2 - c)]);
    free(re);
}

/* float -> int as the compiled x86-64 reference converts (cvttss2si): truncation, INT_MIN for NaN, inf and out of range */
static int trunc_x86(float v) { return v >= -2147483648.0f && v < 2147483648.0f ? (int)v : INT_MIN; }

/* The driver's exp(float): glibc's double exp, rounded once to float (DESIGN §4.8) */
static float ufld_exp(float v) { return (float)exp((double)v); }

/* argmax over the chan axis of x [chan, rows, cols] -> y [rows, cols] (the index as a float) */
ORACLE_API void oracle_ufld_argmax(const float* x, float* y, int rows, int cols, int chan) {
    for (int i = 0, wh = rows * cols; i < rows; i++) {
        for (int j = 0; j < cols; j++) {
            int max = -10000000;
            int max_ind = -1;
            for (int k = 0; k < chan; k++) {
                if (x[k * wh + i * cols + j] > max) {
                    max = trunc_x86(x[k * wh + i * cols + j]);
                    max_ind = k;
                }
            }
            y[i * cols + j] = max_ind;
        }
    }
}

/* softmax over the first chan - 1 entries of the chan axis and its expectation -> y [rows, cols]; x is overwritten as in
 * the reference */
ORACLE_API void oracle_ufld_softmax_mul(float* x, float* y, int rows, int cols, int chan) {
    for (int i = 0, wh = rows * cols; i < rows; i++) {
        for (int j = 0; j < cols; j++) {
            float sum = 0.0;
            float expect = 0.0;
            for (int k = 0; k < chan - 1; k++) {
                x[k * wh + i * cols + j] = ufld_exp(x[k * wh + i * cols + j]);
                sum += x[k * wh + i * cols + j];
            }
            for (int k = 0; k < chan - 1; k++) x[k * wh + i * cols + j] /= sum;
            for (int k = 0; k < chan - 1; k++) {
                x[k * wh + i * cols + j] = x[k * wh + i * cols + j] * (k + 1);
                expect += x[k * wh + i * cols + j];
            }
            y[i * cols + j] = expect;
        }
    }
}

/* The driver loop of lane_det.cpp:358-410 over one frame: prob [C, H, W] -> rows [1 + H * W * 3]: the point count, then
 * (x, y, lane) per point in the order the driver draws them, zeros past the count.  vis_w x vis_h is the picture the points
 * are for (the driver's 1280 x 720).  The - 1 after the x conversion wraps as on x86-64. */
ORACLE_API int oracle_ufld_postprocess(const float* prob, int C, int H, int W, const int* row_anchor, int net_w, int net_h,
                                       int col_sample_w, int vis_w, int vis_h, float* rows) {
    const size_t wh = (size_t)W * H, size = (size_t)C * wh;
    float* max_ind = (float*)malloc(sizeof(float) * wh);
    float* prob_reverse = (float*)calloc(size, sizeof(float));
    float* expect = (float*)malloc(sizeof(float) * wh);
    int* i_ind = (int*)malloc(sizeof(int) * (size_t)W);
    int n_ind = 0, n = 0;
    memset(rows, 0, sizeof(float) * (1 + wh * 3));
    for (int k = 0; k < C; k++)
        for (int j = 0; j < H; j++)
            for (int l = 0; l < W; l++) prob_reverse[k * wh + (H - 1 - j) * W + l] = prob[k * wh + j * W + l];
    oracle_ufld_argmax(prob_reverse, max_ind, H, W, C);
    oracle_ufld_softmax_mul(prob_reverse, expect, H, W, C);
    for (int k = 0; k < H; k++)
        for (int j = 0; j < W; j++)
            if (max_ind[k * W + j] == C - 1) expect[k * W + j] = 0;
    for (int k = 0; k < W; k++) {
        int ii = 0;
        for (int g = 0; g < H; g++)
            if (expect[g * W + k] != 0) ii++;
        if (ii > 2) i_ind[n_ind++] = k;
    }
    for (int k = 0; k < H; k++) {
        for (int ll = 0; ll < n_ind; ll++) {
            if (expect[W * k + i_ind[ll]] > 0) {
                const int x = (int)((unsigned)trunc_x86(expect[W * k + i_ind[ll]] * col_sample_w * vis_w / net_w) - 1u);
                const int y = (int)(vis_h * row_anchor[H - 1 - k] / net_h) - 1;
                float* o = rows + 1 + (size_t)n * 3;
                o[0] = (float)x;
                o[1] = (float)y;
                o[2] = (float)i_ind[ll];
                ++n;
            }
        }
    }
    rows[0] = (float)n;
    free(max_ind);
    free(prob_reverse);
    free(expect);
    free(i_ind);
    return n;
}

/* How many floats x with 0 <= x <= hi (sign 0) or -lo >= -x >= 0 (sign 1), every `stride`-th bit pattern from zero up, have
 * expf(x) != (float)exp((double)x) in this C library */
static long exp_disagreements_half(uint32_t sign, float limit, unsigned stride) {
    long bad = 0;
    for (uint64_t b = 0; b < 0x7f800000u; b += stride) {
        const uint32_t bits = sign | (uint32_t)b;
        float x;
        memcpy(&x, &bits, sizeof x);
        if (fabsf(x) > limit) break;
        if (expf(x) != ufld_exp(x)) ++bad;
    }
    return bad;
}

ORACLE_API long oracle_ufld_exp_disagreements(float lo, float hi, unsigned stride) {
    return exp_disagreements_half(0u, hi, stride) + exp_disagreements_half(0x80000000u, -lo, stride);
}
