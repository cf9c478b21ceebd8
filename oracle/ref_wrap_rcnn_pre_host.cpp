// ref_wrap_rcnn_pre_host.cpp -- TEST INFRASTRUCTURE.  CPU-only wrapper around preprocessImg (rcnn/common.hpp:79-110): the
// geometry of its resize and paste.  The image is a shim cv::Mat (oracle/shim_rcnn_pre) of the given size without pixels; the
// shim's resize and copyTo do no pixel work, they record their arguments.
#include "common.hpp"

extern "C" {
// geom = {resize width, resize height, paste x, paste y, paste width, paste height}: the size cv::resize is asked for and the
// rectangle of the 128-grey canvas that re.copyTo writes (:104-106)
__attribute__((visibility("default"))) void ref_rcnn_preprocess_geometry(int img_w, int img_h, int input_w, int input_h, int* geom) {
    cv::Mat img(img_h, img_w, CV_8UC3, nullptr);
    int l = -1, r = -1, t = -1, b = -1;
    for (int i = 0; i < 6; ++i) cv::Mat::shim_geometry()[i] = -1;
    preprocessImg(img, input_w, input_h, l, r, t, b);
    for (int i = 0; i < 6; ++i) geom[i] = cv::Mat::shim_geometry()[i];
}
}
