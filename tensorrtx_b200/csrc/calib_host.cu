// calib_host.cu -- the INT8 calibrator's host pre-process (SURVEY 8f rank 4: "INT8 calibrator path also reuses the CPU letterbox").
// Replaces, for Int8EntropyCalibrator2::getBatch (yolov8/src/calibrator.cpp:33-52, the same file in yolov5 / yolov7 / ...):
//     cv::Mat pr_img = preprocess_img(temp, input_w_, input_h_);                      // yolov8/include/utils.h:6-26
//     cv::Mat blob = cv::dnn::blobFromImages(input_imgs_, 1.0 / 255.0, size, cv::Scalar(0, 0, 0), true, false);
// i.e. cv::resize(INTER_LINEAR) of the 8-bit BGR image to the letterbox size, paste on a 128-grey canvas, swap R and B, scale by
// (float)(1 / 255.0), planar float output.  It is HOST code in the reference too (calibration runs once per engine build, not in
// the inference loop), and it is the one place on this path whose arithmetic lives in a third-party dependency that is not
// under /root/reference: OpenCV.  Restated here from OpenCV 4.x's 8-bit bilinear resize (imgproc/src/resize.cpp: fixed-point
// coefficients cvRound(c * 2048), horizontal pass in int, vertical pass ((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2,
// x taps clamped with zeroed fraction at the borders, y taps clipped with the fraction kept) and pinned bit for bit against
// cv2 4.13 (with and without IPP) by tests/test_calibrator_cpu.py.  No CUDA in this file.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

namespace trtx {

struct ResizeAxis {
    int* idx;    // source index of the low tap (x: clamped; y: NOT clamped, clipped when used)
    short* coef;  // 2 fixed-point weights per destination index, sum = 2048
};

static void resize_axis(ResizeAxis a, int dn, int sn, bool clamp) {
    const double scale = (double)sn / dn;
    for (int d = 0; d < dn; ++d) {
        const LinearTap t = cv_linear_tap(d, scale, sn, clamp);
        a.idx[d] = t.s;
        a.coef[2 * d] = t.c0;
        a.coef[2 * d + 1] = t.c1;
    }
}

}  // namespace trtx

using namespace trtx;

extern "C" {

// The letterbox rectangle of preprocess_img (utils.h:7-20): float ratios from a double division, products truncated to int.
TRTX_API int trtx_calib_letterbox_rect(int src_w, int src_h, int net_w, int net_h, int rect[4]) {
    if (src_w <= 0 || src_h <= 0 || net_w <= 0 || net_h <= 0 || !rect) return TRTX_ERR_INVALID;
    int w, h, x, y;
    float r_w = net_w / (src_w * 1.0);
    float r_h = net_h / (src_h * 1.0);
    if (r_h > r_w) {
        w = net_w;
        h = r_w * src_h;
        x = 0;
        y = (net_h - h) / 2;
    } else {
        w = r_h * src_w;
        h = net_h;
        x = (net_w - w) / 2;
        y = 0;
    }
    rect[0] = x, rect[1] = y, rect[2] = w, rect[3] = h;
    return TRTX_OK;
}

// The Python runners' preprocess_image (yolov8_det_trt.py:223-236): the ratios and products stay double, int() truncates;
// (net - h) is never negative, so int((net - h) / 2) is the integer division.
TRTX_API int trtx_pyrunner_letterbox_rect(int src_w, int src_h, int net_w, int net_h, int rect[4]) {
    if (src_w <= 0 || src_h <= 0 || net_w <= 0 || net_h <= 0 || !rect) return TRTX_ERR_INVALID;
    const double r_w = (double)net_w / src_w, r_h = (double)net_h / src_h;
    int w, h, x, y;
    if (r_h > r_w) {
        w = net_w;
        h = (int)(r_w * src_h);
        x = 0;
        y = (net_h - h) / 2;
    } else {
        w = (int)(r_h * src_w);
        h = net_h;
        x = (net_w - w) / 2;
        y = 0;
    }
    rect[0] = x, rect[1] = y, rect[2] = w, rect[3] = h;
    return TRTX_OK;
}

TRTX_API int trtx_calib_letterbox_host(const uint8_t* bgr, int src_w, int src_h, size_t src_pitch, int net_w, int net_h, float* out_chw) {
    if (!bgr || !out_chw || src_pitch < (size_t)src_w * 3) return TRTX_ERR_INVALID;
    int rc[4];
    const int e = trtx_calib_letterbox_rect(src_w, src_h, net_w, net_h, rc);
    if (e) return e;
    const int x0 = rc[0], y0 = rc[1], dw = rc[2], dh = rc[3];
    if (dw <= 0 || dh <= 0) return TRTX_ERR_UNSUPPORTED;  // cv::resize would throw on an empty destination
    float lut[256];
    const float s = (float)(1.0 / 255.0);  // blobFromImages: `image *= scalefactor` in float
    for (int v = 0; v < 256; ++v) lut[v] = (float)v * s;
    const size_t plane = (size_t)net_w * net_h;
    // canvas: cv::Scalar(128, 128, 128)
    for (size_t i = 0; i < 3 * plane; ++i) out_chw[i] = lut[128];
    int* xi = (int*)malloc(sizeof(int) * (size_t)dw);
    int* yi = (int*)malloc(sizeof(int) * (size_t)dh);
    short* xc = (short*)malloc(sizeof(short) * 2 * (size_t)dw);
    short* yc = (short*)malloc(sizeof(short) * 2 * (size_t)dh);
    int* rows[2] = {(int*)malloc(sizeof(int) * 3 * (size_t)dw), (int*)malloc(sizeof(int) * 3 * (size_t)dw)};
    if (!xi || !yi || !xc || !yc || !rows[0] || !rows[1]) {
        free(xi), free(yi), free(xc), free(yc), free(rows[0]), free(rows[1]);
        return TRTX_ERR_INVALID;
    }
    resize_axis(ResizeAxis{xi, xc}, dw, src_w, true);
    resize_axis(ResizeAxis{yi, yc}, dh, src_h, false);
    int have[2] = {-1, -1};  // source row held by rows[k]
    auto hresize = [&](int sy, int* dst) {
        const uint8_t* S = bgr + (size_t)sy * src_pitch;
        for (int dx = 0; dx < dw; ++dx) {
            const int sx = xi[dx], sx1 = sx + 1 < src_w ? sx + 1 : src_w - 1;
            const int a0 = xc[2 * dx], a1 = xc[2 * dx + 1];
            for (int c = 0; c < 3; ++c) dst[3 * dx + c] = S[3 * sx + c] * a0 + S[3 * sx1 + c] * a1;
        }
    };
    for (int dy = 0; dy < dh; ++dy) {
        int sy[2] = {yi[dy], yi[dy] + 1};
        for (int k = 0; k < 2; ++k) sy[k] = sy[k] < 0 ? 0 : (sy[k] > src_h - 1 ? src_h - 1 : sy[k]);
        // keep a row that is already resized (consecutive destination rows share source rows)
        if (have[0] != sy[0]) {
            if (have[1] == sy[0]) {
                int* t = rows[0];
                rows[0] = rows[1], rows[1] = t;
                have[1] = have[0], have[0] = sy[0];
            } else {
                hresize(sy[0], rows[0]);
                have[0] = sy[0];
            }
        }
        if (have[1] != sy[1]) {
            if (sy[1] == sy[0]) {
                memcpy(rows[1], rows[0], sizeof(int) * 3 * (size_t)dw);
            } else {
                hresize(sy[1], rows[1]);
            }
            have[1] = sy[1];
        }
        const int b0 = yc[2 * dy], b1 = yc[2 * dy + 1];
        float* o = out_chw + (size_t)(y0 + dy) * net_w + x0;
        for (int dx = 0; dx < dw; ++dx)
            for (int c = 0; c < 3; ++c) {
                int v = (((b0 * (rows[0][3 * dx + c] >> 4)) >> 16) + ((b1 * (rows[1][3 * dx + c] >> 4)) >> 16) + 2) >> 2;
                v = v < 0 ? 0 : (v > 255 ? 255 : v);
                o[(size_t)(2 - c) * plane + dx] = lut[v];  // swapRB: B, G, R -> planes 2, 1, 0
            }
    }
    free(xi), free(yi), free(xc), free(yc), free(rows[0]), free(rows[1]);
    return TRTX_OK;
}

}  // extern "C"
