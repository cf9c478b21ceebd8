/*
 * cubic_oracle.c -- CPU ORACLE of the bicubic letterbox pre-process of yolov3-tiny and retinafaceAntiCov.  TEST INFRASTRUCTURE
 * ONLY, like trtx_oracle.c: plain C, single thread, built with -ffp-contract=off, independent of the library's code.
 *   preprocess_img   yolov3-tiny/yolov3-tiny.cpp:40-60, retinafaceAntiCov/retinafaceAntiCov.cpp:41-61 (the same function):
 *                    the letterbox rectangle, cv::resize(INTER_CUBIC) of the 8-bit frame into it, a 128-grey canvas
 *   the plane loops  yolov3-tiny.cpp:441-445 (u / 255.0) and retinafaceAntiCov.cpp:528-532 (((float)u - 127.5) * 0.0078125),
 *                    R, G, B planes
 * The resize is OpenCV 4.x's own code path (imgproc/src/resize.cpp, IPP off), restated: resizeGeneric_ with HResizeCubic and
 * VResizeCubic<uchar, int, short, FixedPtCast<int, uchar, 22>, VResizeCubicVec_32s8u>.  Its vertical pass runs the 8-lane
 * SSE loop of VResizeCubicVec_32s8u over the first (3 * dw) & ~7 bytes of a row (float, no FMA) and the scalar fixed-point
 * loop over the rest.  Pinned to cv2 with IPP off, bit for bit, by tests/test_cubic_pre_cpu.py.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORACLE_API __attribute__((visibility("default")))

/* interpolateCubic(x, coeffs), A = -0.75, in float */
static void interpolate_cubic(float x, float* c) {
    const float A = -0.75f;
    c[0] = ((A * (x + 1) - 5 * A) * (x + 1) + 8 * A) * (x + 1) - 4 * A;
    c[1] = ((A + 2) * x - (A + 3)) * x * x + 1;
    c[2] = ((A + 2) * (1 - x) - (A + 3)) * (1 - x) * (1 - x) + 1;
    c[3] = 1.f - c[0] - c[1] - c[2];
}

/* One axis of resizeGeneric_'s tables: for destination index d, the low tap ofs[d] = floor(fx) (not clamped: the fraction is kept
 * at the borders for INTER_CUBIC) and the 4 weights saturate_cast<short>(coeff * 2048) (cvRound: half to even). */
static void cubic_axis(int dn, int sn, int* ofs, int* w) {
    const double scale = 1. / ((double)dn / sn);
    for (int d = 0; d < dn; ++d) {
        float f = (float)((d + 0.5) * scale - 0.5);
        const int s = (int)floorf(f);
        f -= (float)s;
        float c[4];
        interpolate_cubic(f, c);
        ofs[d] = s;
        for (int k = 0; k < 4; ++k) w[4 * d + k] = (int)lrintf(c[k] * 2048.f);
    }
}

static int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

/* cv::resize(src, dst, Size(dw, dh), 0, 0, INTER_CUBIC) of an 8-bit 3-channel image, IPP off.  dst: dh rows of 3 * dw bytes. */
ORACLE_API void oracle_resize_cubic_u8(const uint8_t* src, int sw, int sh, size_t pitch, int dw, int dh, uint8_t* dst) {
    if (sw == dw && sh == dh) {  /* cv::resize copies */
        for (int y = 0; y < sh; ++y) memcpy(dst + (size_t)y * 3 * dw, src + (size_t)y * pitch, 3 * (size_t)dw);
        return;
    }
    const int W = 3 * dw, nvec = W & ~7;  /* bytes of a row: those of the 8-lane vector loop */
    int* xofs = (int*)malloc(sizeof(int) * (size_t)dw);
    int* yofs = (int*)malloc(sizeof(int) * (size_t)dh);
    int* alpha = (int*)malloc(sizeof(int) * 4 * (size_t)dw);
    int* beta = (int*)malloc(sizeof(int) * 4 * (size_t)dh);
    int* H = (int*)malloc(sizeof(int) * 4 * (size_t)W);
    cubic_axis(dw, sw, xofs, alpha);
    cubic_axis(dh, sh, yofs, beta);
    const float scale = 1.f / (2048 * 2048);
    for (int dy = 0; dy < dh; ++dy) {
        for (int k = 0; k < 4; ++k) {  /* HResizeCubic of the 4 clipped source rows */
            const uint8_t* S = src + (size_t)clampi(yofs[dy] - 1 + k, 0, sh - 1) * pitch;
            int* D = H + (size_t)k * W;
            for (int dx = 0; dx < dw; ++dx)
                for (int c = 0; c < 3; ++c) {
                    int v = 0;
                    for (int j = 0; j < 4; ++j) v += S[3 * clampi(xofs[dx] - 1 + j, 0, sw - 1) + c] * alpha[4 * dx + j];
                    D[3 * dx + c] = v;
                }
        }
        const int* b = beta + 4 * dy;
        const int *S0 = H, *S1 = H + W, *S2 = H + 2 * W, *S3 = H + 3 * W;
        const float b0 = (float)b[0] * scale, b1 = (float)b[1] * scale, b2 = (float)b[2] * scale, b3 = (float)b[3] * scale;
        uint8_t* out = dst + (size_t)dy * W;
        for (int x = 0; x < W; ++x) {
            int v;
            if (x < nvec)  /* v_muladd(S0, b0, v_muladd(S1, b1, v_muladd(S2, b2, S3 * b3))), v_round */
                v = (int)lrintf((float)S0[x] * b0 + ((float)S1[x] * b1 + ((float)S2[x] * b2 + (float)S3[x] * b3)));
            else  /* castOp(S0[x]*b0 + S1[x]*b1 + S2[x]*b2 + S3[x]*b3): FixedPtCast<int, uchar, 22> */
                v = (S0[x] * b[0] + S1[x] * b[1] + S2[x] * b[2] + S3[x] * b[3] + (1 << 21)) >> 22;
            out[x] = (uint8_t)clampi(v, 0, 255);
        }
    }
    free(xofs), free(yofs), free(alpha), free(beta), free(H);
}

/* The engine input value of byte u: variant 0 (yolov3-tiny) u / 255.0, variant 1 (retinafaceAntiCov)
 * ((float)u - 127.5) * 0.0078125, both in double and stored to float */
ORACLE_API float oracle_cubic_input_value(int variant, int u) {
    return variant == 0 ? (float)(u / 255.0) : (float)(((float)u - 127.5) * 0.0078125);
}

/* preprocess_img + the plane loop for one image: img_h rows of `pitch` bytes, u8 BGR -> out [3, net_h, net_w] fp32 planes
 * R, G, B; rect = {x, y, w, h} of the pasted resize.  Returns 0, or -1 where cv::resize or copyTo throws (an empty rectangle or
 * one that leaves the canvas); then `out` is not written. */
ORACLE_API int oracle_cubic_preprocess(int variant, const uint8_t* img, int img_w, int img_h, size_t pitch, int net_w,
                                       int net_h, float* out, int* rect) {
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
    if (rect) rect[0] = x, rect[1] = y, rect[2] = w, rect[3] = h;
    if (w <= 0 || h <= 0 || x < 0 || y < 0 || x + w > net_w || y + h > net_h) return -1;
    uint8_t* re = (uint8_t*)malloc((size_t)w * h * 3);
    oracle_resize_cubic_u8(img, img_w, img_h, pitch, w, h, re);
    const size_t plane = (size_t)net_w * net_h;
    float lut[256];
    for (int u = 0; u < 256; ++u) lut[u] = oracle_cubic_input_value(variant, u);
    for (int yy = 0; yy < net_h; ++yy)
        for (int xx = 0; xx < net_w; ++xx) {
            const int in = xx >= x && xx < x + w && yy >= y && yy < y + h;
            const uint8_t* p = in ? re + ((size_t)(yy - y) * w + (xx - x)) * 3 : NULL;
            for (int c = 0; c < 3; ++c) out[(size_t)c * plane + (size_t)yy * net_w + xx] = lut[p ? p[2 - c] : 128];
        }
    free(re);
    return 0;
}
