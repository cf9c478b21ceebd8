// ref_wrap_rcnn_host.cpp -- TEST INFRASTRUCTURE.  CPU-only wrapper around preprocessImg (rcnn/common.hpp:79-102): the four
// letterbox pads it writes through its int& outputs.  The image is a shim cv::Mat of the given size without pixels; the
// shim's resize and copyTo do no pixel work.
#include "common.hpp"

extern "C" {
// pads = {X_LEFT_PAD, X_RIGHT_PAD, Y_TOP_PAD, Y_BOTTOM_PAD}
__attribute__((visibility("default"))) void ref_rcnn_preprocess_pads(int img_w, int img_h, int input_w, int input_h, int* pads) {
    cv::Mat img(img_h, img_w, CV_8UC3, nullptr);
    int l = -1, r = -1, t = -1, b = -1;
    preprocessImg(img, input_w, input_h, l, r, t, b);
    pads[0] = l, pads[1] = r, pads[2] = t, pads[3] = b;
}
}
