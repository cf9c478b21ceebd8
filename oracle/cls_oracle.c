/*
 * cls_oracle.c -- CPU ORACLE of the YOLO classification pre- and post-process.  TEST INFRASTRUCTURE ONLY, like trtx_oracle.c:
 * plain C, single thread, built with -ffp-contract=off, independent of the library's code.
 *   batch_preprocess   yolov8/yolov8_cls.cpp:19-46 (yolo11_cls.cpp and yolo26/yolo26_cls.cpp: the same code) and
 *                      yolov5/yolov5_cls.cpp:19-36 (preprocess_img, yolov5/src/calibrator.cpp:11-31, then the mean / std loop)
 *   softmax            yolov8_cls.cpp:48-61, yolov5_cls.cpp:38-51
 *   topk               yolov8_cls.cpp:63-78, yolov5_cls.cpp:53-68, yolo26_cls.cpp:120-135, in the library's order (below)
 * Pinned to cv2 (IPP on and off) and to the drivers' own compiled functions by tests/test_cls_cpu.py.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORACLE_API __attribute__((visibility("default")))

/* OpenCV 4.x's cv::resize(INTER_LINEAR) of an 8-bit 3-channel image (imgproc/src/resize.cpp), restated: scale =
 * 1. / ((double)dsize / ssize); per destination index fx = (float)((d + 0.5) * scale - 0.5), sx = floor(fx), fx -= sx; x taps
 * outside [0, ssize - 1) move to the border with a zero fraction, y taps keep theirs and clip the rows they read; weights
 * saturate_cast<short>((1 - fx) * 2048) and (fx * 2048) (round half to even); horizontal pass in int, vertical pass
 * ((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2 saturated to 0..255.  dst: dh rows of 3 * dw bytes. */
static void linear_axis(int dn, int sn, int clamp, int* ofs, short* c) {
    double scale = 1. / ((double)dn / sn);
    for (int d = 0; d < dn; ++d) {
        float f = (float)((d + 0.5) * scale - 0.5);
        int s = (int)floorf(f);
        f -= (float)s;
        if (clamp && s < 0) {
            s = 0;
            f = 0.f;
        }
        if (clamp && s >= sn - 1) {
            s = sn - 1;
            f = 0.f;
        }
        ofs[d] = s;
        c[2 * d] = (short)lrintf((1.f - f) * 2048.f);
        c[2 * d + 1] = (short)lrintf(f * 2048.f);
    }
}

static void resize_linear_u8(const uint8_t* src, int sw, int sh, size_t pitch, int dw, int dh, uint8_t* dst) {
    int* xofs = (int*)malloc(sizeof(int) * (size_t)dw);
    int* yofs = (int*)malloc(sizeof(int) * (size_t)dh);
    short* alpha = (short*)malloc(sizeof(short) * 2 * (size_t)dw);
    short* beta = (short*)malloc(sizeof(short) * 2 * (size_t)dh);
    int* S0 = (int*)malloc(sizeof(int) * 3 * (size_t)dw);
    int* S1 = (int*)malloc(sizeof(int) * 3 * (size_t)dw);
    linear_axis(dw, sw, 1, xofs, alpha);
    linear_axis(dh, sh, 0, yofs, beta);
    for (int dy = 0; dy < dh; ++dy) {
        int sy0 = yofs[dy] < 0 ? 0 : (yofs[dy] > sh - 1 ? sh - 1 : yofs[dy]);
        int sy1 = yofs[dy] + 1 < 0 ? 0 : (yofs[dy] + 1 > sh - 1 ? sh - 1 : yofs[dy] + 1);
        const uint8_t* r0 = src + (size_t)sy0 * pitch;
        const uint8_t* r1 = src + (size_t)sy1 * pitch;
        for (int dx = 0; dx < dw; ++dx) {
            int sx0 = xofs[dx], sx1 = xofs[dx] + 1 < sw ? xofs[dx] + 1 : sw - 1;
            for (int c = 0; c < 3; ++c) {
                S0[3 * dx + c] = r0[3 * sx0 + c] * alpha[2 * dx] + r0[3 * sx1 + c] * alpha[2 * dx + 1];
                S1[3 * dx + c] = r1[3 * sx0 + c] * alpha[2 * dx] + r1[3 * sx1 + c] * alpha[2 * dx + 1];
            }
        }
        int b0 = beta[2 * dy], b1 = beta[2 * dy + 1];
        for (int i = 0; i < 3 * dw; ++i) {
            int v = (((b0 * (S0[i] >> 4)) >> 16) + ((b1 * (S1[i] >> 4)) >> 16) + 2) >> 2;
            dst[(size_t)dy * 3 * dw + i] = (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
        }
    }
    free(xofs), free(yofs), free(alpha), free(beta), free(S0), free(S1);
}

/* ------------------------------------------------------------------------------------------
 * batch_preprocess for one image.  variant 0 (yolov8 / yolo11 / yolo26): m = std::min(h, w); cv::Mat img = imgs[b](cv::Rect(
 * (w - m) / 2, (h - m) / 2, m, m)); cv::resize to (net_w, net_h); cvtColor BGR2RGB; convertTo(CV_32F, 1 / 255.0), which is
 * (float)u * (float)(1 / 255.0); split into planes R, G, B.  variant 1 (yolov5): preprocess_img (r_w = input_w / (cols * 1.0)
 * stored to float, ..., products truncated to int, the resized image pasted at (x, y) on a 128-grey canvas), then per pixel
 * ((float)u / 255.0 - mean) / std in double, stored to float, planes R, G, B.
 * img: img_h rows of `pitch` bytes, u8 BGR; out: [3, net_h, net_w] fp32.  rect = {x, y, w, h}: the crop (variant 0) or the
 * pasted rectangle (variant 1).  Returns 0, or -1 where the reference throws (cv::resize to an empty size, or a paste outside
 * the canvas); then `out` is not written.
 * ------------------------------------------------------------------------------------------ */
ORACLE_API int oracle_cls_preprocess(int variant, const uint8_t* img, int img_w, int img_h, size_t pitch, int net_w, int net_h,
                                     float* out, int* rect) {
    const size_t plane = (size_t)net_w * net_h;
    if (variant == 0) {
        int m = img_h < img_w ? img_h : img_w;
        int top = (img_h - m) / 2, left = (img_w - m) / 2;
        if (rect) rect[0] = left, rect[1] = top, rect[2] = m, rect[3] = m;
        uint8_t* re = (uint8_t*)malloc(plane * 3);
        resize_linear_u8(img + (size_t)top * pitch + 3 * (size_t)left, m, m, pitch, net_w, net_h, re);
        const float s = (float)(1 / 255.0);
        for (size_t p = 0; p < plane; ++p)
            for (int c = 0; c < 3; ++c) out[(size_t)c * plane + p] = (float)re[3 * p + (2 - c)] * s;
        free(re);
        return 0;
    }
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
    if (w <= 0 || h <= 0) return -1;                                             /* cv::resize throws on an empty size */
    if (x < 0 || y < 0 || x + w > net_w || y + h > net_h) return -1;             /* out(cv::Rect) throws */
    if (rect) rect[0] = x, rect[1] = y, rect[2] = w, rect[3] = h;
    uint8_t* re = (uint8_t*)malloc((size_t)w * h * 3);
    resize_linear_u8(img, img_w, img_h, pitch, w, h, re);
    static const double mean[3] = {0.485, 0.456, 0.406}, sd[3] = {0.229, 0.224, 0.225};
    for (int py = 0; py < net_h; ++py)
        for (int px = 0; px < net_w; ++px) {
            const int in = px >= x && px < x + w && py >= y && py < y + h;
            const uint8_t* u = in ? re + ((size_t)(py - y) * w + (px - x)) * 3 : NULL;
            for (int c = 0; c < 3; ++c) {
                const uint8_t v = in ? u[2 - c] : 128;
                out[(size_t)c * plane + (size_t)py * net_w + px] = (float)(((double)(float)v / 255.0 - mean[c]) / sd[c]);
            }
        }
    free(re);
    return 0;
}

/* softmax, yolov8_cls.cpp:48-61: t = expf(x_i), sum += t in float in ascending i, res_i = t_i / sum (glibc's expf here) */
ORACLE_API void oracle_cls_softmax(const float* x, int n, float* res) {
    float sum = 0.0f;
    for (int i = 0; i < n; ++i) {
        res[i] = expf(x[i]);
        sum += res[i];
    }
    for (int i = 0; i < n; ++i) res[i] /= sum;
}

/* topk in the library's order: descending by the order-preserving key of the float bits with -0.0 mapped to +0.0 (so +NaN
 * ranks above +inf and -NaN below -inf), ties in ascending index; the first min(k, n) indices. */
static uint32_t desc_key(float f) {
    uint32_t b;
    memcpy(&b, &f, 4);
    b = b == 0x80000000u ? 0u : b;
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
static const float* g_vals;
static int cmp_desc(const void* pa, const void* pb) {
    const int a = *(const int*)pa, b = *(const int*)pb;
    const uint32_t ka = desc_key(g_vals[a]), kb = desc_key(g_vals[b]);
    if (ka != kb) return ka > kb ? -1 : 1;
    return a < b ? -1 : (a > b);
}
ORACLE_API int oracle_cls_topk(const float* res, int n, int k, int* idx) {
    int* all = (int*)malloc(sizeof(int) * (size_t)n);
    for (int i = 0; i < n; ++i) all[i] = i;
    g_vals = res;
    qsort(all, (size_t)n, sizeof(int), cmp_desc);
    const int kk = k < n ? k : n;
    memcpy(idx, all, sizeof(int) * (size_t)kk);
    free(all);
    return kk;
}
