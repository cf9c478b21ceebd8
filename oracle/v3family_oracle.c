/* v3family_oracle.c -- TEST INFRASTRUCTURE.  Plain-C restatement of the yolov3 family's CalDetection, one driver's box
 * arithmetic at a time, built by oracle/Makefile into oracle/libv3family_oracle.so (-ffp-contract=off).
 * box_mode takes the library's variant values (include/trtx_hot.h section 1):
 *   2 (spp)  x = (col + Logist(x0)) * stride                                  yolov3-spp/yololayer.cu:183-186
 *   4 (net)  x = (col + Logist(x0)) * INPUT_W / yoloWidth, in float            yolov3/yololayer.cu:173-176, yolov3-tiny :172-175
 *   5 (v4)   the same box with the double Logist `1./(1. + exp(-data))`       yolov4/yololayer.cu:154, :191-194
 *   6 (csp)  x = ((col + 2 * Logist(x0)) - 0.5) * INPUT_W / yoloWidth: `- 0.5` is a double literal, so the subtraction,
 *            multiply and divide run in double; w = powf(2 * Logist(x2), 2) * anchor; double Logist
 *                                                                             scaled-yolov4/yololayer.cu:154, :191-194
 * Modes 5 and 6 take the double Logist for the gates and both confidences too; modes 2 and 4 the float one.  Mode 2 is
 * oracle_yolov3_decode of trtx_oracle.c.
 * inputs[l] : [B, 3*(5+classes), gh*gw] fp32, levels in the caller's order; anchors[l*6 + 2k (+1)]; strides[l] (mode 2).
 * out rows  : x, y, w, h, det_confidence, class_id, class_confidence.  The count runs past max_out as the reference's
 *             atomicAdd does; rows stop there (`if (count >= MAX_OUTPUT_BBOX_COUNT) return;`).  Flat anchor id =
 *             level_off + cell*3 + k.
 * Class loop first (all classes, sigmoid, strict `>` from 0), THEN both gates. */
#include <math.h>
#include <stdint.h>
#include <string.h>

#define ORACLE_API __attribute__((visibility("default")))

static float logist_f32(float x) { return 1.0f / (1.0f + expf(-x)); }
static float logist_f64(float x) { return (float)(1. / (1. + (double)expf(-x))); }

ORACLE_API void oracle_v3family_decode(const float* const* inputs, int batch, int num_levels, const int* grid_h,
                                       const int* grid_w, const int* strides, const float* anchors, int classes, int max_out,
                                       float ignore_thresh, int box_mode, int net_w, int net_h, float* out,
                                       int32_t* anchor_idx) {
    float (*sig)(float) = (box_mode == 5 || box_mode == 6) ? logist_f64 : logist_f32;
    const int det_floats = 7;
    const int out_elem = 1 + max_out * det_floats;
    const int info_len_i = 5 + classes;
    memset(out, 0, sizeof(float) * (size_t)batch * out_elem);
    int level_off = 0;
    for (int l = 0; l < num_levels; ++l) {
        const int yw = grid_w[l], yh = grid_h[l];
        const int total_grid = yw * yh;
        const float* anc = anchors + l * 6;
        for (int t = 0; t < batch * total_grid; ++t) {
            const int bn = t / total_grid;
            const int idx = t - total_grid * bn;
            const float* cur = inputs[l] + (size_t)bn * ((size_t)info_len_i * total_grid * 3);
            float* o = out + (size_t)bn * out_elem;
            for (int k = 0; k < 3; ++k) {
                const float* ck = cur + (size_t)k * info_len_i * total_grid;
                int class_id = 0;
                float max_cls_prob = 0.0f;
                for (int i = 5; i < info_len_i; ++i) {
                    float p = sig(ck[idx + (size_t)i * total_grid]);
                    if (p > max_cls_prob) {
                        max_cls_prob = p;
                        class_id = i - 5;
                    }
                }
                float box_prob = sig(ck[idx + 4 * (size_t)total_grid]);
                if (max_cls_prob < ignore_thresh || box_prob < ignore_thresh) continue;
                int count = (int)o[0];
                o[0] += 1.0f;
                if (count >= max_out) break; /* `return`: this cell's later anchors are not written either */
                float* det = o + 1 + (size_t)count * det_floats;
                if (anchor_idx) anchor_idx[(size_t)bn * max_out + count] = level_off + idx * 3 + k;
                const int row = idx / yw, col = idx % yw;
                const float x0 = ck[idx], x1 = ck[idx + (size_t)total_grid];
                const float x2 = ck[idx + 2 * (size_t)total_grid], x3 = ck[idx + 3 * (size_t)total_grid];
                if (box_mode == 6) {
                    det[0] = (float)(((double)((float)col + 2.0f * sig(x0)) - 0.5) * net_w / yw);
                    det[1] = (float)(((double)((float)row + 2.0f * sig(x1)) - 0.5) * net_h / yh);
                    det[2] = powf(2.0f * sig(x2), 2.0f) * anc[2 * k];
                    det[3] = powf(2.0f * sig(x3), 2.0f) * anc[2 * k + 1];
                } else {
                    if (box_mode == 2) {
                        det[0] = (col + sig(x0)) * strides[l];
                        det[1] = (row + sig(x1)) * strides[l];
                    } else {
                        det[0] = ((float)col + sig(x0)) * (float)net_w / (float)yw;
                        det[1] = ((float)row + sig(x1)) * (float)net_h / (float)yh;
                    }
                    det[2] = expf(x2) * anc[2 * k];
                    det[3] = expf(x3) * anc[2 * k + 1];
                }
                det[4] = box_prob;
                det[5] = (float)class_id;
                det[6] = max_cls_prob;
            }
        }
        level_off += total_grid * 3;
    }
}
