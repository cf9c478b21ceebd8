/*
 * rcnn_post_oracle.c -- CPU ORACLE of the Mask R-CNN post-process (rcnn/rcnn.cpp:516-550) and of preprocessImg's pads
 * (rcnn/common.hpp:79-102).  TEST INFRASTRUCTURE ONLY, like trtx_oracle.c: plain C, single thread, built with
 * -ffp-contract=off so that the arithmetic is the IEEE fp32 sequence of the reference source.  The mask resize is
 * oracle_resize_bilinear of libtrtx_oracle.so (OpenCV's float bilinear kernel, pinned to cv2 in tests/test_oracle_cpu.py).
 * Pinned here by tests/test_rcnn_post_cpu.py: the pads against the reference's compiled preprocessImg, the canvases against
 * cv2, the rows and rectangles against a numpy float32 restatement.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORACLE_API __attribute__((visibility("default")))

void oracle_resize_bilinear(const float* src, int sh, int sw, float* dst, int dh, int dw); /* libtrtx_oracle.so */

/* ------------------------------------------------------------------------------------------
 * Mask R-CNN post-process.
 * oracle_rcnn_letterbox_pads: the four pads preprocessImg writes (rcnn/common.hpp:79-102): `input_w / (img.cols*1.0)` is a
 * double division stored to float, `r_w * img.rows` a float product truncated to int, `(input_h - h) / 2.f` float, and the
 * pads are round() of that float -/+ the double 0.1.  pads = {left, right, top, bottom}.
 * ------------------------------------------------------------------------------------------ */
ORACLE_API void oracle_rcnn_letterbox_pads(int img_w, int img_h, int net_w, int net_h, int* pads) {
    int w, h;
    float x, y;
    float r_w = (float)(net_w / (img_w * 1.0));
    float r_h = (float)(net_h / (img_h * 1.0));
    if (r_h > r_w) {
        w = net_w;
        h = (int)(r_w * (float)img_h);
        x = 0.0f;
        y = (float)(net_h - h) / 2.f;
    } else {
        w = (int)(r_h * (float)img_w);
        h = net_h;
        x = (float)(net_w - w) / 2.f;
        y = 0.0f;
    }
    (void)w;
    (void)h;
    pads[0] = (int)round(x - 0.1);
    pads[1] = (int)round(x + 0.1);
    pads[2] = (int)round(y - 0.1);
    pads[3] = (int)round(y + 0.1);
}

/* The paste rectangle of rcnn/rcnn.cpp:543-546 for a box (x1, y1, x2, y2) in original-image pixels: cv::Rect(Point(floor(x1) - 1
 * clamped at 0, ...), Point(ceil(x2) + 1 clamped at w_ori, ...)), which cv::Rect normalises to the min corner and |delta| sizes.
 * Returns 0 where the reference throws: cv::resize to an empty size (:547), or Mat::operator()(Rect) with a rectangle that
 * leaves the image (:550; a corner past the image, or one whose int conversion overflows).  Non-finite coordinates count as a
 * throw too: the reference converts them to int, which is undefined.  rect = {x, y, w, h}. */
static int rcnn_rect_axis(float c0, float c1, int size, int* o, int* len) {
    double lo = floor(c0) - 1 < 0 ? 0 : floor(c0) - 1;
    double hi = ceil(c1) + 1 > size ? size : ceil(c1) + 1;
    if (lo > size || hi < 0) return 0;
    int a = (int)lo, b = (int)hi;
    *o = a < b ? a : b;
    *len = a < b ? b - a : a - b;
    return *len > 0;
}
ORACLE_API int oracle_rcnn_mask_rect(const float* box, int img_w, int img_h, int* rect) {
    for (int j = 0; j < 4; ++j)
        if (!isfinite(box[j])) return 0;
    return rcnn_rect_axis(box[0], box[2], img_w, &rect[0], &rect[2]) && rcnn_rect_axis(box[1], box[3], img_h, &rect[1], &rect[3]);
}

/* rcnn/rcnn.cpp:516-550 for one image, with the image's own size (the reference uses the last image's, a defect).
 * scores [D], boxes [D,4], classes [D] (BatchedNms outputs), masks [D,S,S] (MaskRcnnInference output) or NULL.
 * rows [1 + D*7]: count, then (x1, y1, x2, y2, score, class, slot) for every slot i with score > score_thresh, ascending i;
 * rows past the count are zeroed.  canvases [max_masks, img_h, img_w] u8: canvas k of the k-th kept row (k < max_masks) is
 * zeroed and gets 255 where the resized mask is > 0.5 inside the paste rectangle; it stays zero where the reference throws.
 * Canvases at or past min(count, max_masks) are not touched.  Returns the count. */
ORACLE_API int oracle_rcnn_postprocess(const float* scores, const float* boxes, const float* classes, const float* masks, int D,
                                       int S, int net_w, int net_h, int img_w, int img_h, float score_thresh, int max_masks,
                                       float* rows, uint8_t* canvases) {
    int pads[4];
    oracle_rcnn_letterbox_pads(img_w, img_h, net_w, net_h, pads);
    float h_ratio = (float)img_h / (float)(net_h - (pads[2] + pads[3])); /* :516-517 */
    float w_ratio = (float)img_w / (float)(net_w - (pads[0] + pads[1]));
    memset(rows, 0, (1 + (size_t)D * 7) * sizeof(float));
    int n = 0;
    for (int i = 0; i < D; ++i) {
        if (!(scores[i] > score_thresh)) continue; /* :522 */
        float x1 = (boxes[i * 4 + 0] - (float)pads[0]) * w_ratio; /* :523-526 */
        float y1 = (boxes[i * 4 + 1] - (float)pads[2]) * h_ratio;
        float x2 = (boxes[i * 4 + 2] - (float)pads[0]) * w_ratio;
        float y2 = (boxes[i * 4 + 3] - (float)pads[2]) * h_ratio;
        float* r = rows + 1 + (size_t)n * 7;
        r[0] = x1;
        r[1] = y1;
        r[2] = x2;
        r[3] = y2;
        r[4] = scores[i];
        r[5] = classes[i];
        r[6] = (float)i;
        if (masks && canvases && n < max_masks) {
            uint8_t* cur = canvases + (size_t)n * img_h * img_w; /* :548 curMask = zeros(w_ori x h_ori) */
            memset(cur, 0, (size_t)img_h * img_w);
            int rect[4];
            if (oracle_rcnn_mask_rect(r, img_w, img_h, rect)) { /* :543-546 */
                float* part = (float*)malloc((size_t)rect[2] * rect[3] * sizeof(float));
                oracle_resize_bilinear(masks + (size_t)i * S * S, S, S, part, rect[3], rect[2]); /* :547 */
                for (int yy = 0; yy < rect[3]; ++yy)
                    for (int xx = 0; xx < rect[2]; ++xx) {
                        float v = part[(size_t)yy * rect[2] + xx] > 0.5f ? 255.0f : 0.0f; /* :549 threshold */
                        uint8_t* px = cur + (size_t)(rect[1] + yy) * img_w + rect[0] + xx;   /* :550 curMask(r) += */
                        float s = (float)*px + v;
                        *px = (uint8_t)(s > 255.0f ? 255.0f : s);
                    }
                free(part);
            }
        }
        ++n;
    }
    rows[0] = (float)n;
    return n;
}
