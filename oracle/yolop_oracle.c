/*
 * yolop_oracle.c -- CPU ORACLE of the YOLOP pre- and post-process.  TEST INFRASTRUCTURE ONLY, like trtx_oracle.c: plain C,
 * single thread, built with -ffp-contract=off, independent of the library's code.
 *   preprocess_img   yolop/utils.h:11-36 + the driver's plane loop (yolop/yolop.cpp:110-127)
 *   get_rect         yolop/common.hpp:13-37
 *   labels           yolop/yolop.cpp:148-169: cv::resize(INTER_NEAREST) of the two maps, then lane / drivable area / none
 * The NMS is oracle_nms's yolov5 variant (trtx_oracle.c).  Pinned to cv2 and to the reference's compiled nms() and
 * get_rect by tests/test_yolop_cpu.py.
 */
/* cls_oracle.c's 8-bit INTER_LINEAR resize (resize_linear_u8), a static function: this oracle includes that file, so the
 * library also exports the classification oracle's entry points. */
#include "cls_oracle.c"

#include <limits.h>

/* ------------------------------------------------------------------------------------------
 * preprocess_img for one image: r_w = input_w / (cols * 1.0) stored to float, ..., the products truncated to int; the resized
 * image pasted at (x, y) on a 114-grey canvas; convertTo(CV_32FC3, 1.f / 255.f), cv::subtract of Scalar(0.485, 0.456, 0.406)
 * in float, cv::divide by Scalar(0.229, 0.224, 0.225) in double; planes in the driver's order, B, G, R.
 * img: img_h rows of `pitch` bytes, u8 BGR; out: [3, net_h, net_w] fp32; rect = {x, y, w, h} of the pasted image.
 * Returns 0, or -1 where the reference throws (an empty size, a paste outside the canvas); then `out` is not written.
 * ------------------------------------------------------------------------------------------ */
ORACLE_API float oracle_yolop_input_value(int c, int u) {
    static const double mean[3] = {0.485, 0.456, 0.406}, sd[3] = {0.229, 0.224, 0.225};
    const float t = (float)u * (1.f / 255.f);
    const float s = t - (float)mean[c];
    return (float)((double)s / sd[c]);
}

ORACLE_API int oracle_yolop_preprocess(const uint8_t* img, int img_w, int img_h, size_t pitch, int net_w, int net_h, float* out,
                                       int* rect) {
    int w, h, x, y;
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
            for (int c = 0; c < 3; ++c)
                out[(size_t)c * plane + (size_t)py * net_w + px] = oracle_yolop_input_value(c, in ? u[c] : 114);
        }
    free(re);
    return 0;
}

/* float -> int as the compiled x86-64 reference converts (cvttss2si): truncation, INT_MIN for NaN, inf and out of range */
static int trunc_x86(float v) { return v >= -2147483648.0f && v < 2147483648.0f ? (int)v : INT_MIN; }

/* get_rect, yolop/common.hpp:13-37, with INPUT_W x INPUT_H = net_w x net_h: every statement stores to int; no clamp;
 * rect = {l, t, r - l, b - t}, the differences wrapping modulo 2^32. */
ORACLE_API void oracle_yolop_get_rect(int net_w, int net_h, int img_w, int img_h, const float* bbox, int* rect) {
    int l, r, t, b;
    float r_w = (float)(net_w / (img_w * 1.0));
    float r_h = (float)(net_h / (img_h * 1.0));
    if (r_h > r_w) {
        l = trunc_x86(bbox[0] - bbox[2] / 2.f);
        r = trunc_x86(bbox[0] + bbox[2] / 2.f);
        t = trunc_x86(bbox[1] - bbox[3] / 2.f - ((float)net_h - r_w * (float)img_h) / 2);
        b = trunc_x86(bbox[1] + bbox[3] / 2.f - ((float)net_h - r_w * (float)img_h) / 2);
        l = trunc_x86((float)l / r_w);
        r = trunc_x86((float)r / r_w);
        t = trunc_x86((float)t / r_w);
        b = trunc_x86((float)b / r_w);
    } else {
        l = trunc_x86(bbox[0] - bbox[2] / 2.f - ((float)net_w - r_h * (float)img_w) / 2);
        r = trunc_x86(bbox[0] + bbox[2] / 2.f - ((float)net_w - r_h * (float)img_w) / 2);
        t = trunc_x86(bbox[1] - bbox[3] / 2.f);
        b = trunc_x86(bbox[1] + bbox[3] / 2.f);
        l = trunc_x86((float)l / r_h);
        r = trunc_x86((float)r / r_h);
        t = trunc_x86((float)t / r_h);
        b = trunc_x86((float)b / r_h);
    }
    rect[0] = l;
    rect[1] = t;
    rect[2] = (int)((unsigned)r - (unsigned)l);
    rect[3] = (int)((unsigned)b - (unsigned)t);
}

/* OpenCV 4.x's INTER_NEAREST source index of every destination index along an axis of dn destination and sn source samples:
 * min(floor(d * (1. / ((double)dn / sn))), sn - 1) (imgproc/src/resize.cpp, resizeNN). */
ORACLE_API void oracle_yolop_nearest(int dn, int sn, int* idx) {
    const double ifx = 1. / ((double)dn / sn);
    for (int d = 0; d < dn; ++d) {
        const int s = (int)floor(d * ifx);
        idx[d] = s < sn - 1 ? s : sn - 1;
    }
}

/* The driver's label loop for one frame: seg, lane = [map_h, map_w] int32 maps; canvas = img_h rows of `pitch` bytes, of which
 * the first img_w are written: 2 where the nearest lane value is nonzero, else 1 where the nearest seg value is, else 0. */
ORACLE_API void oracle_yolop_labels(const int32_t* seg, const int32_t* lane, int map_w, int map_h, int img_w, int img_h,
                                    uint8_t* canvas, size_t pitch) {
    int* sx = (int*)malloc(sizeof(int) * (size_t)img_w);
    int* sy = (int*)malloc(sizeof(int) * (size_t)img_h);
    oracle_yolop_nearest(img_w, map_w, sx);
    oracle_yolop_nearest(img_h, map_h, sy);
    for (int y = 0; y < img_h; ++y)
        for (int x = 0; x < img_w; ++x) {
            const size_t o = (size_t)sy[y] * map_w + sx[x];
            canvas[(size_t)y * pitch + x] = lane[o] ? 2 : (seg[o] ? 1 : 0);
        }
    free(sx);
    free(sy);
}
