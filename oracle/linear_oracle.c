/*
 * linear_oracle.c -- CPU ORACLE of the bilinear letterbox pre-process of yolov3, yolov4, scaled-yolov4, yolov3-spp and
 * RetinaFace, and of the truncating get_rect of yolov3, yolov4, scaled-yolov4, yolov3-tiny and yolov3-spp.  TEST
 * INFRASTRUCTURE ONLY, like trtx_oracle.c: plain C, single thread, built with -ffp-contract=off, independent of the library's
 * code.
 *   preprocess_img   yolov3/utils.h:41-61 (yolov4/yolov4.cpp:33-53, scaled-yolov4/common.hpp:14-34, retinaface/common.hpp:21-41:
 *                    the same statements) + the plane loops (yolov3.cpp:477-481, yolov4.cpp:637-641, yolov4_csp.cpp:466-468,
 *                    retina_r50.cpp:342-352)
 *   letterbox        yolov3-spp/yolov3-spp.cpp:43-56 + cv::dnn::blobFromImage(pr, 1 / 255.0, size, 0, swapRB, crop = false)
 *   get_rect         yolov3/yolov3.cpp:30-52 (yolov4.cpp:55-77, scaled-yolov4/common.hpp:36-58, yolov3-tiny.cpp:62-84) and
 *                    yolov3-spp.cpp:58-75
 * Pinned to cv2 (IPP on and off) and to the drivers' own compiled get_rect and letterbox by tests/test_linear_pre_cpu.py.
 */
/* cls_oracle.c's 8-bit INTER_LINEAR resize (resize_linear_u8), a static function: this oracle includes that file, so the
 * library also exports the classification oracle's entry points. */
#include "cls_oracle.c"

#include <limits.h>

enum { V3 = 0, RETINA = 1, SPP = 2 }; /* TRTX_LINEAR_* */

/* The plane loops' value of byte u in plane c: yolov3 family `u / 255.0` (planes R, G, B); RetinaFace `u - 104.0`, `- 117.0`,
 * `- 123.0` (planes B, G, R); blobFromImage: convertTo(CV_32F), subtract Scalar(0), multiply by the float Scalar 1 / 255.0. */
ORACLE_API float oracle_linear_input_value(int variant, int c, int u) {
    static const double mean[3] = {104.0, 117.0, 123.0};
    if (variant == V3) return (float)(u / 255.0);
    if (variant == RETINA) return (float)(u - mean[c]);
    return ((float)u - 0.f) * (float)(1 / 255.0);
}

/* yolov3-spp's letterbox: out = {canvas_w, canvas_h, x, y, w, h} */
ORACLE_API void oracle_yolov3spp_letterbox(int img_w, int img_h, int max_size, int* out) {
    const double a = max_size / (img_w * 1.0), b = max_size / (img_h * 1.0);
    float r = (float)(a < b ? a : b);
    r = r < 1.0f ? r : 1.0f;
    int unpad_w = (int)(r * (float)img_w);
    int unpad_h = (int)(r * (float)img_h);
    int dw = (max_size - unpad_w) % 32;
    int dh = (max_size - unpad_h) % 32;
    out[0] = unpad_w + dw;
    out[1] = unpad_h + dh;
    out[2] = dw / 2;
    out[3] = dh / 2;
    out[4] = unpad_w;
    out[5] = unpad_h;
}

/* ------------------------------------------------------------------------------------------
 * One frame: img = img_h rows of `pitch` bytes, u8 BGR -> out [3, net_h, net_w] fp32 planes; rect = {x, y, w, h} of the pasted
 * resize.  V3 / RETINA: preprocess_img (r_w = input_w / (cols * 1.0) stored to float, the products truncated to int) on a
 * net_w x net_h 128 canvas; SPP: the letterbox for max_size, whose canvas must be net_w x net_h.  Returns 0, or -1 where the
 * reference throws (an empty resize, a paste outside the canvas) or the SPP canvas is another size; then `out` is not written.
 * ------------------------------------------------------------------------------------------ */
ORACLE_API int oracle_linear_preprocess(int variant, const uint8_t* img, int img_w, int img_h, size_t pitch, int net_w, int net_h,
                                        int max_size, float* out, int* rect) {
    int w, h, x, y;
    if (variant == SPP) {
        int g[6];
        oracle_yolov3spp_letterbox(img_w, img_h, max_size, g);
        if (g[0] != net_w || g[1] != net_h) return -1;
        x = g[2], y = g[3], w = g[4], h = g[5];
    } else {
        float r_w = (float)(net_w / (img_w * 1.0));
        float r_h = (float)(net_h / (img_h * 1.0));
        if (r_h > r_w) {
            w = net_w;
            h = (int)(r_w * (float)img_h);
            x = 0;
            y = (net_h - h) / 2;
        } else {
            w = (int)(r_h * (float)img_w);
            h = net_h;
            x = (net_w - w) / 2;
            y = 0;
        }
    }
    if (w <= 0 || h <= 0) return -1;
    if (x < 0 || y < 0 || x + w > net_w || y + h > net_h) return -1;
    if (rect) rect[0] = x, rect[1] = y, rect[2] = w, rect[3] = h;
    uint8_t* re = (uint8_t*)malloc((size_t)w * h * 3);
    resize_linear_u8(img, img_w, img_h, pitch, w, h, re);
    const size_t plane = (size_t)net_w * net_h;
    for (int py = 0; py < net_h; ++py)
        for (int px = 0; px < net_w; ++px) {
            const int in = px >= x && px < x + w && py >= y && py < y + h;
            const uint8_t* u = in ? re + ((size_t)(py - y) * w + (px - x)) * 3 : NULL;
            for (int c = 0; c < 3; ++c) {
                const int ch = variant == RETINA ? c : 2 - c;
                out[(size_t)c * plane + (size_t)py * net_w + px] = oracle_linear_input_value(variant, c, in ? u[ch] : 128);
            }
        }
    free(re);
    return 0;
}

/* float -> int where C++ defines it (truncation); 0 for NaN, inf and out of range */
static int trunc_ok(float v, int* out) {
    if (!(v >= -2147483648.0f && v < 2147483648.0f)) return 0;
    *out = (int)v;
    return 1;
}

/* ------------------------------------------------------------------------------------------
 * get_rect: variant V3 = yolov3.cpp:30-52 with INPUT_W x INPUT_H = net_w x net_h; SPP = yolov3-spp.cpp:58-75 with
 * MAX_INPUT_SIZE = net_w.  rect = {l, t, r - l, b - t}.  Returns 1, or 0 with rect {0, 0, 0, 0} where the reference is
 * undefined (a conversion of NaN, inf or a float outside the int range, or an r - l that overflows).
 * ------------------------------------------------------------------------------------------ */
ORACLE_API int oracle_linear_get_rect(int variant, int net_w, int net_h, int img_w, int img_h, const float* bbox, int* rect) {
    int l, r, t, b, ok = 1;
    float c[4], ratio;
    rect[0] = rect[1] = rect[2] = rect[3] = 0;
    if (variant == SPP) {
        const double da = net_w / (img_w * 1.0), db = net_w / (img_h * 1.0);
        float ra = (float)(da < db ? da : db);
        ra = ra < 1.0f ? ra : 1.0f;
        int unpad_w = (int)(ra * (float)img_w);
        int unpad_h = (int)(ra * (float)img_h);
        int dw = (net_w - unpad_w) % 32;
        int dh = (net_w - unpad_h) % 32;
        c[0] = bbox[0] - bbox[2] / 2.f - (float)(dw / 2);
        c[1] = bbox[0] + bbox[2] / 2.f - (float)(dw / 2);
        c[2] = bbox[1] - bbox[3] / 2.f - (float)(dh / 2);
        c[3] = bbox[1] + bbox[3] / 2.f - (float)(dh / 2);
        ratio = ra;
    } else {
        float r_w = (float)(net_w / (img_w * 1.0));
        float r_h = (float)(net_h / (img_h * 1.0));
        if (r_h > r_w) {
            c[0] = bbox[0] - bbox[2] / 2.f;
            c[1] = bbox[0] + bbox[2] / 2.f;
            c[2] = bbox[1] - bbox[3] / 2.f - ((float)net_h - r_w * (float)img_h) / 2;
            c[3] = bbox[1] + bbox[3] / 2.f - ((float)net_h - r_w * (float)img_h) / 2;
            ratio = r_w;
        } else {
            c[0] = bbox[0] - bbox[2] / 2.f - ((float)net_w - r_h * (float)img_w) / 2;
            c[1] = bbox[0] + bbox[2] / 2.f - ((float)net_w - r_h * (float)img_w) / 2;
            c[2] = bbox[1] - bbox[3] / 2.f;
            c[3] = bbox[1] + bbox[3] / 2.f;
            ratio = r_h;
        }
    }
    ok = trunc_ok(c[0], &l) && trunc_ok(c[1], &r) && trunc_ok(c[2], &t) && trunc_ok(c[3], &b);
    ok = ok && trunc_ok((float)l / ratio, &l) && trunc_ok((float)r / ratio, &r) && trunc_ok((float)t / ratio, &t) &&
         trunc_ok((float)b / ratio, &b);
    if (!ok) return 0;
    const long long w = (long long)r - l, h = (long long)b - t;
    if (w < INT_MIN || w > INT_MAX || h < INT_MIN || h > INT_MAX) return 0;
    rect[0] = l;
    rect[1] = t;
    rect[2] = (int)w;
    rect[3] = (int)h;
    return 1;
}
