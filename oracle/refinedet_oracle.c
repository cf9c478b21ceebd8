/*
 * refinedet_oracle.c -- CPU ORACLE of the RefineDet pre- and post-process.  TEST INFRASTRUCTURE ONLY, like trtx_oracle.c:
 * plain C, single thread, built with -ffp-contract=off, independent of the library's code.
 *   base_transform    refinedet/refinedet.cpp:822-839
 *   PriorBox          :553-597
 *   decode            :600-619, both steps
 *   the ARM filter    :738-746
 *   nms               :632-695, per class, with the library's tie rule (a lower prior index ranks higher)
 *   the rows          :756-815 (class order, keep order, each value rounded to float)
 *   the rectangles    :957-993 with RoiCorrect (:22-35)
 * The post-process runs in libtorch on the device in the reference; this restatement uses glibc's exp, so its boxes may
 * differ from the device's in the last bits.  Pinned by tests/test_refinedet_cpu.py to a line-by-line transcription of the
 * reference in torch.
 */
/* cls_oracle.c's 8-bit INTER_LINEAR resize (resize_linear_u8), a static function: this oracle includes that file, so the
 * library also exports the classification oracle's entry points. */
#include "cls_oracle.c"

#include <limits.h>

/* ------------------------------------------------------------------------------------------
 * base_transform for one image: cv::resize(m_src, image, Size(net, net)) of the whole frame, 8-bit INTER_LINEAR; then plane
 * 0 = R - 123, plane 1 = G - 117, plane 2 = B - 104, each (float)(u * 1.0 - mean).  out: [3, net, net] fp32.
 * ------------------------------------------------------------------------------------------ */
static const double kMeanRgb[3] = {123.0, 117.0, 104.0};

ORACLE_API float oracle_refinedet_input_value(int c, int u) { return (float)(u * 1.0 - kMeanRgb[c]); }

ORACLE_API void oracle_refinedet_preprocess(const uint8_t* img, int img_w, int img_h, size_t pitch, int net, float* out) {
    uint8_t* re = (uint8_t*)malloc((size_t)net * net * 3);
    resize_linear_u8(img, img_w, img_h, pitch, net, net, re);
    const size_t plane = (size_t)net * net;
    for (int c = 0; c < 3; ++c)
        for (size_t i = 0; i < plane; ++i) out[(size_t)c * plane + i] = oracle_refinedet_input_value(c, re[3 * i + (2 - c)]);
    free(re);
}

/* ------------------------------------------------------------------------------------------
 * PriorBox for a square net: the four levels f = net / step, steps 8, 16, 32, 64, min sizes 32, 64, 128, 256, three anchors a
 * cell; sqrt(ar) is sqrtf(2.f) (double_sqrt != 0: sqrt(2.0)); clamp(0, 1); widened.  out: [P, 4] doubles; returns P.
 * ------------------------------------------------------------------------------------------ */
ORACLE_API int oracle_refinedet_priors(int net, int double_sqrt, double* out) {
    static const int steps[4] = {8, 16, 32, 64}, min_sizes[4] = {32, 64, 128, 256};
    int n = 0;
    for (int k = 0; k < 4; k++) {
        const int f = net / steps[k];
        for (int i = 0; i < f; i++) {
            for (int j = 0; j < f; j++) {
                float f_k = net * 1.0 / steps[k];
                float cx = (j + 0.5) / f_k;
                float cy = (i + 0.5) / f_k;
                float s_k = min_sizes[k] * 1.0 / net;
                float ar = 2;
                const double sq = double_sqrt ? sqrt((double)ar) : (double)sqrtf(ar);
                const float v[12] = {cx, cy, s_k, s_k, cx, cy, s_k * 1.0 * sq, s_k * 1.0 / sq, cx, cy, s_k * 1.0 / sq,
                                     s_k * 1.0 * sq};
                for (int e = 0; e < 12; e++) {
                    const float c = v[e] < 0.f ? 0.f : (v[e] > 1.f ? 1.f : v[e]);
                    out[(size_t)n * 4 + e] = (double)c;
                }
                n += 3;
            }
        }
    }
    return n;
}

/* decode (:600-619): d = (p01 + (l01 * v0) * p23, p23 * exp(l23 * v1)); corners: c3 = d01 - d23 / 2, c4 = c3 + d23 */
static void decode(const double* prior, const float* loc, int corners, double* out) {
    const double v0 = (double)0.1f, v1 = (double)0.2f;
    double d[4];
    for (int e = 0; e < 2; e++) {
        d[e] = prior[e] + ((double)loc[e] * v0) * prior[2 + e];
        d[2 + e] = prior[2 + e] * exp((double)loc[2 + e] * v1);
    }
    for (int e = 0; e < 2; e++) {
        if (corners) {
            out[e] = d[e] - d[2 + e] / 2;
            out[2 + e] = out[e] + d[2 + e];
        } else {
            out[e] = d[e];
            out[2 + e] = d[2 + e];
        }
    }
}

/* Tensor::clamp(lo, hi): a NaN bound gives NaN, a NaN value stays, else min(max(v, lo), hi) */
static double tclamp(double v, double lo, double hi) {
    if (isnan(lo) || isnan(hi)) return NAN;
    if (isnan(v)) return v;
    v = v < lo ? lo : v;
    return v > hi ? hi : v;
}

typedef struct {
    double score;
    int idx;  /* prior */
} Cand;

static int cand_cmp(const void* pa, const void* pb) {  /* descending score, ascending prior */
    const Cand *a = (const Cand*)pa, *b = (const Cand*)pb;
    if (a->score != b->score) return a->score > b->score ? -1 : 1;
    return (a->idx > b->idx) - (a->idx < b->idx);
}

/* ------------------------------------------------------------------------------------------
 * doInference's post-process (:730-815) for one frame: arm_loc [P, 4], arm_conf [P, 2], odm_loc [P, 4], odm_conf [P, C]
 * -> dets [1 + max_det * 6]: n = min(total, max_det), then (x1, y1, x2, y2, score, label) as floats, zeros past n.
 * Returns total (the rows before the max_det cut), or -1 for a net without priors.
 * ------------------------------------------------------------------------------------------ */
ORACLE_API int oracle_refinedet_postprocess(const float* arm_loc, const float* arm_conf, const float* odm_loc,
                                            const float* odm_conf, int net, int C, float obj_thresh, float conf_thresh,
                                            float nms_thresh, int top_k, int max_det, float* dets) {
    int P = 0;
    for (int k = 0; k < 4; k++) P += 3 * (net / (8 << k)) * (net / (8 << k));
    double* prior = (double*)malloc(sizeof(double) * 4 * (size_t)P);
    if (oracle_refinedet_priors(net, 0, prior) != P) {
        free(prior);
        return -1;
    }
    double* box = (double*)malloc(sizeof(double) * 4 * (size_t)P);
    double* area = (double*)malloc(sizeof(double) * (size_t)P);
    for (int p = 0; p < P; p++) {
        double d[4];
        decode(prior + 4 * (size_t)p, arm_loc + 4 * (size_t)p, 0, d);
        decode(d, odm_loc + 4 * (size_t)p, 1, box + 4 * (size_t)p);
        const double* b = box + 4 * (size_t)p;
        area[p] = (b[2] - b[0]) * (b[3] - b[1]);
    }
    Cand* cand = (Cand*)malloc(sizeof(Cand) * (size_t)P);
    char* removed = (char*)malloc((size_t)P);
    const size_t len = 1 + (size_t)max_det * 6;
    memset(dets, 0, sizeof(float) * len);
    int total = 0;
    for (int c = 1; c < C; c++) {
        int m = 0;
        for (int p = 0; p < P; p++) {
            const double s = (double)odm_conf[(size_t)p * C + c] * ((double)arm_conf[2 * (size_t)p + 1] > (double)obj_thresh ? 1.0 : 0.0);
            if (s > (double)conf_thresh) cand[m].score = s, cand[m].idx = p, m++;
        }
        qsort(cand, (size_t)m, sizeof(Cand), cand_cmp);
        if (m > top_k) m = top_k;
        for (int i = 0; i < m; i++) removed[i] = 0;
        for (int i = 0; i < m; i++) {
            if (removed[i]) continue;
            const double* bi = box + 4 * (size_t)cand[i].idx;
            if (total < max_det) {
                float* o = dets + 1 + (size_t)total * 6;
                for (int e = 0; e < 4; e++) o[e] = (float)bi[e];
                o[4] = (float)cand[i].score;
                o[5] = (float)c;
            }
            total++;
            const double lx = (float)bi[0], ly = (float)bi[1], hx = (float)bi[2], hy = (float)bi[3];
            for (int j = i + 1; j < m; j++) {
                if (removed[j]) continue;
                const double* bj = box + 4 * (size_t)cand[j].idx;
                const double xx1 = tclamp(bj[0], lx, INT_MAX * 1.0), yy1 = tclamp(bj[1], ly, INT_MAX * 1.0);
                const double xx2 = tclamp(bj[2], INT_MIN * 1.0, hx), yy2 = tclamp(bj[3], INT_MIN * 1.0, hy);
                const double w = tclamp(xx2 - xx1, 0, INT_MAX), h = tclamp(yy2 - yy1, 0, INT_MAX);
                const double inter = w * h;
                const double uni = (area[cand[j].idx] - inter) + area[cand[i].idx];
                const double iou = inter * 1.0 / uni;
                if (!(iou < (double)nms_thresh)) removed[j] = 1;
            }
        }
    }
    dets[0] = (float)(total < max_det ? total : max_det);
    free(prior);
    free(box);
    free(area);
    free(cand);
    free(removed);
    return total;
}

/* float -> int as the compiled x86-64 reference converts (cvttss2si): truncation, INT_MIN for NaN, inf and out of range */
static int trunc_x86(float v) { return v >= -2147483648.0f && v < 2147483648.0f ? (int)v : INT_MIN; }

/* RoiCorrect (:22-35); the sums wrap as on x86-64 */
static void roi_correct(int cols, int rows, int* r) {
    if (r[0] < 0) r[0] = 0;
    if (r[1] < 0) r[1] = 0;
    if (r[0] >= cols - 1) r[0] = 0;
    if (r[1] >= rows - 1) r[1] = 0;
    if (r[2] <= 0) r[2] = 1;
    if (r[3] <= 0) r[3] = 1;
    if ((int)((unsigned)r[0] + (unsigned)r[2]) > cols - 1) r[2] = cols - 1 - r[0];
    if ((int)((unsigned)r[1] + (unsigned)r[3]) > rows - 1) r[3] = rows - 1 - r[1];
}

/* The driver loop (:957-993) over dets [1 + max_det * 6] of a cols x rows frame -> out [1 + max_det * 6]: the count, then
 * (x, y, w, h, score, label) as floats for the rows with !(score < score_thresh), zeros past the count.  Returns the count. */
ORACLE_API int oracle_refinedet_rows(const float* dets, int max_det, int cols, int rows, float score_thresh, float* out) {
    const int n = (int)dets[0];
    int kept = 0;
    memset(out, 0, sizeof(float) * (1 + (size_t)max_det * 6));
    for (int i = 0; i < n; i++) {
        const float* d = dets + 1 + (size_t)i * 6;
        const float score = d[4];
        if (score < score_thresh) continue;
        int r[4];
        r[0] = trunc_x86(d[0] * (float)cols);
        r[1] = trunc_x86(d[1] * (float)rows);
        r[2] = trunc_x86(d[2] * (float)cols - (float)r[0]);
        r[3] = trunc_x86(d[3] * (float)rows - (float)r[1]);
        roi_correct(cols, rows, r);
        float* o = out + 1 + (size_t)kept * 6;
        for (int e = 0; e < 4; e++) o[e] = (float)r[e];
        o[4] = score;
        o[5] = d[5];
        kept++;
    }
    out[0] = (float)kept;
    return kept;
}
