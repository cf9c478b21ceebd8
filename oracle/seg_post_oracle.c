/* seg_post_oracle.c -- TEST INFRASTRUCTURE: the CPU oracle of the YOLO segmentation post-process, one image at a time.
 * Restates, in plain C, what the reference's segmentation drivers do after NMS (yolov8/yolov8_seg.cpp:289-297,
 * yolov5/yolov5_seg.cpp): process_mask (yolov8_seg.cpp:36-60, yolov5/src/postprocess.cpp:106-125), scale_mask
 * (yolov8/src/postprocess.cpp:207-226, yolov5 :127-146) and the mask selection of draw_mask_bbox (yolov8 :228-248,
 * yolov5 :148-167):
 *     img_mask = scale_mask(masks[i], img);  r = get_rect(img, dets[i].bbox);
 *     for x in [r.x, r.x + r.width), y in [r.y, r.y + r.height): if (img_mask.at<float>(y, x) <= 0.5) continue; -> pixel kept
 * process_mask, the bilinear resize and get_rect come from libtrtx_oracle.so (trtx_oracle.c).  Where the reference is
 * undefined the oracle does what the library documents: the selection is clipped to the image (a V5 rect may leave it), and a
 * box whose get_rect converts a non-finite or out-of-range float to int gets rect {0, 0, 0, 0} and an all-zero canvas. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORACLE_API __attribute__((visibility("default")))

void oracle_process_mask(int variant, const float* proto, int nm, int mh, int mw, int net_w, int net_h, const float* bbox,
                         const float* coeffs, float* out);
void oracle_resize_bilinear(const float* src, int sh, int sw, float* dst, int dh, int dw);
void oracle_get_rect(int variant, int net_w, int net_h, int img_w, int img_h, const float* bbox, int* rect);

static int fits_int(float v) {
    double r = round((double)v);
    return r >= -2147483648.0 && r <= 2147483647.0; /* false for NaN */
}

/* get_rect's four float -> int conversions (round(l), round(t), round(r - l), round(b - t)) are defined */
static int rect_defined(int variant, int net_w, int net_h, int img_w, int img_h, const float* bbox) {
    float r_w = (float)(net_w / (img_w * 1.0)), r_h = (float)(net_h / (img_h * 1.0));
    float l, r, t, b;
    if (variant == 0) {
        l = bbox[0], t = bbox[1], r = bbox[2], b = bbox[3];
    } else {
        l = bbox[0] - bbox[2] / 2.f, r = bbox[0] + bbox[2] / 2.f;
        t = bbox[1] - bbox[3] / 2.f, b = bbox[1] + bbox[3] / 2.f;
    }
    if (r_h > r_w) {
        t = (t - (net_h - r_w * img_h) / 2) / r_w, b = (b - (net_h - r_w * img_h) / 2) / r_w;
        l = l / r_w, r = r / r_w;
    } else {
        l = (l - (net_w - r_h * img_w) / 2) / r_h, r = (r - (net_w - r_h * img_w) / 2) / r_h;
        t = t / r_h, b = b / r_h;
    }
    if (variant == 0) {
        l = 0.0f > l ? 0.0f : l;
        t = 0.0f > t ? 0.0f : t;
    }
    return fits_int(l) && fits_int(t) && fits_int(r - l) && fits_int(b - t);
}

/* scale_mask's crop: `h = r_w * img.rows` truncates float -> int, `(kInputH - h) / 2` is an integer division */
ORACLE_API void oracle_scale_mask_rect(int net_w, int net_h, int img_w, int img_h, int* rect) {
    float r_w = (float)(net_w / (img_w * 1.0)), r_h = (float)(net_h / (img_h * 1.0));
    if (r_h > r_w) {
        rect[2] = net_w;
        rect[3] = (int)(r_w * img_h);
        rect[0] = 0;
        rect[1] = (net_h - rect[3]) / 2;
    } else {
        rect[2] = (int)(r_h * img_w);
        rect[3] = net_h;
        rect[0] = (net_w - rect[2]) / 2;
        rect[1] = 0;
    }
}

/* One image.  proto [nm, mh, mw]; dets [1 + max_rows * row_floats] = count, rows (box 0..3, conf 4, class 5, coefficients
 * at coeff_offset).  rows [1 + max_rows * 6]: n = min(count, max_rows), (x, y, w, h, conf, class) per row, zeros after.
 * canvases [max_masks, img_h, img_w] u8 or NULL: slots k < min(n, max_masks) are written, the others are left as they are.
 * scaled [max_masks, img_h, img_w] fp32 or NULL: scale_mask(M) of the same slots (the value the selection compares).
 * Returns 0, or -1 when the scale_mask crop is empty (the reference's cv::resize throws). */
ORACLE_API int oracle_seg_postprocess(int variant, const float* proto, int nm, int mh, int mw, int net_w, int net_h,
                                      const float* dets, int max_rows, int row_floats, int coeff_offset, int max_masks,
                                      int img_w, int img_h, float* rows, uint8_t* canvases, float* scaled) {
    const float c = dets[0];
    const int n = c > 0 ? (c < (float)max_rows ? (int)c : max_rows) : 0;
    memset(rows, 0, sizeof(float) * (1 + (size_t)max_rows * 6));
    rows[0] = (float)n;
    for (int i = 0; i < n; ++i) {
        const float* d = dets + 1 + (size_t)i * row_floats;
        float* r = rows + 1 + (size_t)i * 6;
        int rect[4] = {0, 0, 0, 0};
        if (rect_defined(variant, net_w, net_h, img_w, img_h, d)) oracle_get_rect(variant, net_w, net_h, img_w, img_h, d, rect);
        for (int e = 0; e < 4; ++e) r[e] = (float)rect[e];
        r[4] = d[4];
        r[5] = d[5];
    }
    if (!canvases && !scaled) return 0;
    int cr[4];
    oracle_scale_mask_rect(net_w, net_h, img_w, img_h, cr);
    if (cr[2] <= 0 || cr[3] <= 0) return -1;
    const size_t npix = (size_t)img_h * img_w;
    float* M = (float*)malloc(sizeof(float) * (size_t)net_w * net_h);
    float* crop = (float*)malloc(sizeof(float) * (size_t)cr[2] * cr[3]);
    float* S = (float*)malloc(sizeof(float) * npix);
    const int nmask = n < max_masks ? n : max_masks;
    for (int k = 0; k < nmask; ++k) {
        const float* d = dets + 1 + (size_t)k * row_floats;
        uint8_t* cv = canvases ? canvases + (size_t)k * npix : NULL;
        if (cv) memset(cv, 0, npix);
        if (!rect_defined(variant, net_w, net_h, img_w, img_h, d)) { /* nothing selected; S is reported as 0 */
            if (scaled) memset(scaled + (size_t)k * npix, 0, sizeof(float) * npix);
            continue;
        }
        oracle_process_mask(variant, proto, nm, mh, mw, net_w, net_h, d, d + coeff_offset, M);
        for (int y = 0; y < cr[3]; ++y) memcpy(crop + (size_t)y * cr[2], M + (size_t)(cr[1] + y) * net_w + cr[0], sizeof(float) * cr[2]);
        oracle_resize_bilinear(crop, cr[3], cr[2], S, img_h, img_w); /* cv::resize(mask(r), res, img.size()) */
        if (scaled) memcpy(scaled + (size_t)k * npix, S, sizeof(float) * npix);
        if (!cv) continue;
        int r[4];
        oracle_get_rect(variant, net_w, net_h, img_w, img_h, d, r);
        /* draw_mask_bbox's loops, clipped to the image */
        const long long x0 = r[0] > 0 ? r[0] : 0, x1 = (long long)r[0] + r[2] < img_w ? (long long)r[0] + r[2] : img_w;
        const long long y0 = r[1] > 0 ? r[1] : 0, y1 = (long long)r[1] + r[3] < img_h ? (long long)r[1] + r[3] : img_h;
        for (long long x = x0; x < x1; x++) {
            for (long long y = y0; y < y1; y++) {
                const float val = S[(size_t)y * img_w + x];
                if (val <= 0.5) continue;
                cv[(size_t)y * img_w + x] = 255;
            }
        }
    }
    free(M);
    free(crop);
    free(S);
    return 0;
}
