/* anchor_free_oracle.c -- TEST INFRASTRUCTURE.  The CPU oracle of the two host post-processes of yolov9 and yolov10 that the
 * library runs on the device (oracle/Makefile links it to libtrtx_oracle.so, whose oracle_nms and oracle_get_rect it
 * reuses):
 *   oracle_v9_nms   yolov9's nms() (yolov9/src/postprocess.cpp:48-83): rows i < output[0] and i < max_rows, each l, t, r, b
 *                   box converted to c_x = (b0 + b2) / 2, c_y = (b1 + b3) / 2, w = b2 - b0, h = b3 - b1 in float, then
 *                   yolov5's centre-size greedy NMS (oracle_nms variant 1) on the converted rows, which it pushes.  A NaN
 *                   confidence is dropped (the library's rule; the reference sorts it with a comparator that is no order).
 *   oracle_topk     yolov10's get_topk (:35-44) + get_rect (:3-33): rows i < min(output[0], max_rows) with
 *                   !(conf <= conf_thresh), a NaN confidence included, in input order, as (x, y, w, h, conf, class). */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORACLE_API __attribute__((visibility("default")))

int oracle_nms(int variant, const float* plugin_out, int max_rows, int det_floats, double conf_thresh, float nms_thresh,
               float* res, int32_t* res_src);
void oracle_get_rect(int variant, int net_w, int net_h, int img_w, int img_h, const float* bbox, int* rect);

static int first_rows(const float* output, int max_rows) {
    int n = (int)output[0]; /* `i < output[0]` */
    if (n > max_rows) n = max_rows;
    return n < 0 ? 0 : n;
}

ORACLE_API int oracle_v9_nms(const float* output, int max_rows, int det_floats, float conf_thresh, float nms_thresh, float* res,
                             int32_t* res_src) {
    const int n = first_rows(output, max_rows);
    float* conv = (float*)malloc(sizeof(float) * (1 + (size_t)(n > 0 ? n : 1) * det_floats));
    conv[0] = (float)n;
    for (int i = 0; i < n; ++i) {
        const float* d = output + 1 + (size_t)i * det_floats;
        float* c = conv + 1 + (size_t)i * det_floats;
        memcpy(c, d, sizeof(float) * det_floats);
        c[0] = (d[0] + d[2]) / 2;
        c[1] = (d[1] + d[3]) / 2;
        c[2] = d[2] - d[0];
        c[3] = d[3] - d[1];
        if (isnan(c[4])) c[4] = -INFINITY; /* dropped by `conf <= conf_thresh` below */
    }
    const int k = oracle_nms(1, conv, n, det_floats, (double)conf_thresh, nms_thresh, res, res_src);
    free(conv);
    return k;
}

ORACLE_API int oracle_topk(const float* output, int max_rows, int row_floats, float conf_thresh, int variant, int net_w, int net_h,
                           int img_w, int img_h, float* rows) {
    const int n = first_rows(output, max_rows);
    int k = 0;
    for (int i = 0; i < n; ++i) {
        const float* d = output + 1 + (size_t)i * row_floats;
        if (d[4] <= conf_thresh) continue;
        int r[4];
        oracle_get_rect(variant, net_w, net_h, img_w, img_h, d, r);
        float* o = rows + (size_t)k * 6;
        for (int e = 0; e < 4; ++e) o[e] = (float)r[e];
        o[4] = d[4];
        o[5] = d[5];
        ++k;
    }
    return k;
}
