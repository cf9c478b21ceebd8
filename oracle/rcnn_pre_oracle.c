/*
 * rcnn_pre_oracle.c -- CPU ORACLE of the Mask R-CNN pre-process: preprocessImg (rcnn/common.hpp:79-110) + the float widening
 * of rcnn/rcnn.cpp:504-505.  TEST INFRASTRUCTURE ONLY, like trtx_oracle.c: plain C, single thread, built with
 * -ffp-contract=off, independent of the library's code.  Pinned to cv2 (IPP on and off) by tests/test_rcnn_pre_cpu.py.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#define ORACLE_API __attribute__((visibility("default")))

/* ------------------------------------------------------------------------------------------
 * Mask R-CNN pre-process: preprocessImg (rcnn/common.hpp:79-110) + the float widening of rcnn/rcnn.cpp:504-505, line by line.
 * The resize is OpenCV 4.x's cv::resize(INTER_LINEAR) of an 8-bit 3-channel image (imgproc/src/resize.cpp), restated here on
 * its own: scale = 1. / ((double)dsize / ssize); per destination index fx = (float)((d + 0.5) * scale - 0.5), sx = floor(fx),
 * fx -= sx; x taps outside [0, ssize - 1) move to the border with a zero fraction, y taps keep theirs and clip the rows they
 * read; weights saturate_cast<short>((1 - fx) * 2048) and (fx * 2048) (round half to even); horizontal pass in int, vertical
 * pass ((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2 saturated to 0..255 (VResizeLinearVec_32s8u).
 * img: img_h rows of `pitch` bytes, u8 BGR; out: [net_h, net_w, 3] fp32.  Returns 0, or -1 where the reference throws
 * (cv::resize to an empty size); then `out` is not written.  rect (may be NULL) = {x, y, w, h} of the pasted image.
 * ------------------------------------------------------------------------------------------ */
static void cv_linear_axis(int dn, int sn, int clamp, int* ofs, short* c) {
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

ORACLE_API int oracle_rcnn_preprocess(const uint8_t* img, int img_w, int img_h, size_t pitch, int net_w, int net_h, float* out,
                                      int* rect) {
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
    int X_LEFT_PAD = (int)round(x - 0.1);
    int Y_TOP_PAD = (int)round(y - 0.1);
    if (w <= 0 || h <= 0) return -1; /* cv::resize(img, re, re.size()) throws on an empty size */
    if (X_LEFT_PAD < 0 || Y_TOP_PAD < 0 || X_LEFT_PAD + w > net_w || Y_TOP_PAD + h > net_h) return -1; /* out(cv::Rect) throws */
    if (rect) rect[0] = X_LEFT_PAD, rect[1] = Y_TOP_PAD, rect[2] = w, rect[3] = h;
    int* xofs = (int*)malloc(sizeof(int) * (size_t)w);
    int* yofs = (int*)malloc(sizeof(int) * (size_t)h);
    short* alpha = (short*)malloc(sizeof(short) * 2 * (size_t)w);
    short* beta = (short*)malloc(sizeof(short) * 2 * (size_t)h);
    int* S0 = (int*)malloc(sizeof(int) * 3 * (size_t)w);
    int* S1 = (int*)malloc(sizeof(int) * 3 * (size_t)w);
    uint8_t* re = (uint8_t*)malloc(3 * (size_t)w * h);
    cv_linear_axis(w, img_w, 1, xofs, alpha);
    cv_linear_axis(h, img_h, 0, yofs, beta);
    for (int dy = 0; dy < h; ++dy) {
        int sy0 = yofs[dy] < 0 ? 0 : (yofs[dy] > img_h - 1 ? img_h - 1 : yofs[dy]);
        int sy1 = yofs[dy] + 1 < 0 ? 0 : (yofs[dy] + 1 > img_h - 1 ? img_h - 1 : yofs[dy] + 1);
        const uint8_t* r0 = img + (size_t)sy0 * pitch;
        const uint8_t* r1 = img + (size_t)sy1 * pitch;
        for (int dx = 0; dx < w; ++dx) {
            int sx0 = xofs[dx], sx1 = xofs[dx] + 1 < img_w ? xofs[dx] + 1 : img_w - 1;
            for (int c = 0; c < 3; ++c) {
                S0[3 * dx + c] = r0[3 * sx0 + c] * alpha[2 * dx] + r0[3 * sx1 + c] * alpha[2 * dx + 1];
                S1[3 * dx + c] = r1[3 * sx0 + c] * alpha[2 * dx] + r1[3 * sx1 + c] * alpha[2 * dx + 1];
            }
        }
        int b0 = beta[2 * dy], b1 = beta[2 * dy + 1];
        for (int i = 0; i < 3 * w; ++i) {
            int v = (((b0 * (S0[i] >> 4)) >> 16) + ((b1 * (S1[i] >> 4)) >> 16) + 2) >> 2;
            re[(size_t)dy * 3 * w + i] = (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
        }
    }
    /* cv::Mat out(input_h, input_w, CV_8UC3, cv::Scalar(128, 128, 128)); re.copyTo(out(cv::Rect(X_LEFT_PAD, Y_TOP_PAD, w, h)));
     * then data[i] = (float)img.data[i] for every byte of the canvas */
    for (size_t i = 0; i < (size_t)net_h * net_w * 3; ++i) out[i] = 128.0f;
    for (int dy = 0; dy < h; ++dy)
        for (int i = 0; i < 3 * w; ++i)
            out[((size_t)(Y_TOP_PAD + dy) * net_w + X_LEFT_PAD) * 3 + i] = (float)re[(size_t)dy * 3 * w + i];
    free(xofs), free(yofs), free(alpha), free(beta), free(S0), free(S1), free(re);
    return 0;
}
