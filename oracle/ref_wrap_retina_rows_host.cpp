// ref_wrap_retina_rows_host.cpp -- TEST INFRASTRUCTURE.  The host loop of retinaface/retina_r50.cpp:373-388 over the compact
// NMS rows of one frame, on the reference's own get_rect_adapt_landmark (retinaface/common.hpp:65-89), for timing against
// the device face post-process.  oracle/face_obb26.mk builds it into oracle/_ref/libref_retina_rows_host.so.
#include <cstring>
#include <vector>

#include "common.hpp"

// n rows of row_floats floats (box4, conf, class, keep, 10 landmarks, ...): faces with class_confidence < conf_thresh are
// skipped, get_rect_adapt_landmark maps the rest into rect_out [n, 4] / lmk_out [n, 10].  Returns the number of faces mapped.
extern "C" __attribute__((visibility("default"))) int ref_retina_rows(int img_w, int img_h, int input_w, int input_h,
                                                                      const float* rows, int n, int row_floats,
                                                                      double conf_thresh, int* rect_out, float* lmk_out) {
    cv::Mat img(img_h, img_w, CV_8UC3, nullptr);
    int m = 0;
    for (int j = 0; j < n; ++j) {
        const float* d = rows + (size_t)j * row_floats;
        if (d[4] < conf_thresh) continue;
        float bbox[4] = {d[0], d[1], d[2], d[3]};
        float* lmk = lmk_out + 10 * m;
        memcpy(lmk, d + 7, 10 * sizeof(float));
        cv::Rect r = get_rect_adapt_landmark(img, input_w, input_h, bbox, lmk);
        rect_out[4 * m] = r.x, rect_out[4 * m + 1] = r.y, rect_out[4 * m + 2] = r.width, rect_out[4 * m + 3] = r.height;
        ++m;
    }
    return m;
}
