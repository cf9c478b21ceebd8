/*
 * detr_oracle.c -- CPU ORACLE of the DETR pre- and post-process.  TEST INFRASTRUCTURE ONLY, like trtx_oracle.c: plain C,
 * single thread, built with -ffp-contract=off, independent of the library's code.
 *   preprocessImg   detr/common.hpp:81-89 + the driver's plane loop (detr/detr.cpp:754-767)
 *   the post loop   detr/detr.cpp:777-806 (argmax, threshold, no-object class, cv::Rect), restated line by line for one frame
 * The post loop sits inside the driver's main(), next to the engine calls, so there is no reference build of it to compare
 * against: oracle_detr_postprocess below keeps the reference's statements and their order.  Pinned to cv2 by
 * tests/test_detr_cpu.py.
 */
/* cls_oracle.c's 8-bit INTER_LINEAR resize (resize_linear_u8), a static function: this oracle includes that file, so the
 * library also exports the classification oracle's entry points. */
#include "cls_oracle.c"

#include <limits.h>

/* ------------------------------------------------------------------------------------------
 * preprocessImg for one image: cvtColor BGR2RGB; cv::resize(img, img, Size(net_w, net_h)) of the whole frame, 8-bit
 * INTER_LINEAR; convertTo(CV_32FC3); img /= 255 (convertTo(-1, 1. / 255): a float product by (float)(1. / 255));
 * img -= Scalar(0.485, 0.456, 0.406) in float; img /= Scalar(0.229, 0.224, 0.225) in double; the driver's planes 0, 1, 2 are
 * R, G, B.  img: img_h rows of `pitch` bytes, u8 BGR; out: [3, net_h, net_w] fp32.
 * ------------------------------------------------------------------------------------------ */
ORACLE_API float oracle_detr_input_value(int c, int u) {
    static const double mean[3] = {0.485, 0.456, 0.406}, sd[3] = {0.229, 0.224, 0.225};  /* R, G, B */
    const float t = (float)u * (float)(1. / 255);
    const float s = t - (float)mean[c];
    return (float)((double)s / sd[c]);
}

ORACLE_API void oracle_detr_preprocess(const uint8_t* img, int img_w, int img_h, size_t pitch, int net_w, int net_h,
                                       float* out) {
    uint8_t* re = (uint8_t*)malloc((size_t)net_w * net_h * 3);
    resize_linear_u8(img, img_w, img_h, pitch, net_w, net_h, re);  /* per channel: the same bytes after or before cvtColor */
    const size_t plane = (size_t)net_w * net_h;
    for (int c = 0; c < 3; ++c)
        for (size_t i = 0; i < plane; ++i) out[(size_t)c * plane + i] = oracle_detr_input_value(c, re[3 * i + (2 - c)]);
    free(re);
}

/* float -> int as the compiled x86-64 reference converts (cvttss2si): truncation, INT_MIN for NaN, inf and out of range */
static int trunc_x86(float v) { return v >= -2147483648.0f && v < 2147483648.0f ? (int)v : INT_MIN; }

/* detr.cpp:795-803 for one box: the corners are double expressions stored to float; cv::Rect(x1, y1, x2 - x1, y2 - y1)
 * converts four floats to int. */
ORACLE_API void oracle_detr_get_rect(int img_cols, int img_rows, const float* box, int* rect) {
    float cx = box[0];
    float cy = box[1];
    float w = box[2];
    float h = box[3];
    float x1 = (cx - w / 2.0) * img_cols;
    float y1 = (cy - h / 2.0) * img_rows;
    float x2 = (cx + w / 2.0) * img_cols;
    float y2 = (cy + h / 2.0) * img_rows;
    rect[0] = trunc_x86(x1);
    rect[1] = trunc_x86(y1);
    rect[2] = trunc_x86(x2 - x1);
    rect[3] = trunc_x86(y2 - y1);
}

/* detr.cpp:777-806 over one frame's queries: scores [Q, C], boxes [Q, 4] -> rows [1 + Q * 6]: the kept count, then
 * (x, y, w, h, score, class) per kept query in query order, zeros past the count.  The loop runs over this frame's queries
 * (the reference's runs over every query of the batch; the same at its BATCH_SIZE 1). */
ORACLE_API int oracle_detr_postprocess(const float* scores_h, const float* boxes_h, int num_queries, int num_class,
                                       float score_thresh, int img_cols, int img_rows, float* rows) {
    int kept = 0;
    memset(rows, 0, sizeof(float) * (1 + (size_t)num_queries * 6));
    for (size_t i = 0; i < (size_t)num_queries * num_class; i += num_class) {
        long label = -1;
        float score = -1;
        for (size_t j = i; j < i + num_class; j++) {
            if (score < scores_h[j]) {
                label = (long)j;
                score = scores_h[j];
            }
        }
        if (score > score_thresh && (label % num_class != num_class - 1)) {
            long ind = label / num_class;
            label = label % num_class;
            int r[4];
            oracle_detr_get_rect(img_cols, img_rows, boxes_h + ind * 4, r);
            float* o = rows + 1 + (size_t)kept * 6;
            for (int k = 0; k < 4; ++k) o[k] = (float)r[k];
            o[4] = score;
            o[5] = (float)label;
            ++kept;
        }
    }
    rows[0] = (float)kept;
    return kept;
}
