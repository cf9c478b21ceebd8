// SHIM, not OpenCV -- TEST INFRASTRUCTURE.  cv::dnn::blobFromImage as yolov3-spp.cpp names it; no pixel work.
#pragma once
#include "../opencv.hpp"
namespace cv {
namespace dnn {
inline Mat blobFromImage(const Mat& img, double = 1.0, const Size& = Size(), const Scalar& = Scalar(), bool = false,
                         bool = false) {
    return Mat(img.rows, img.cols, CV_32F);
}
}  // namespace dnn
}  // namespace cv
