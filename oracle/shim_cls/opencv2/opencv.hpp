// SHIM, not OpenCV -- TEST INFRASTRUCTURE.  The cv:: names that the YOLO cls drivers (yolov8/yolov8_cls.cpp, yolo11/yolo11_cls.cpp,
// yolov5/yolov5_cls.cpp, yolo26/yolo26_cls.cpp) and the headers they include mention, so that their batch_preprocess, softmax
// and topk compile where they lie (oracle/cls.mk, target `ref`).  An image is a (rows, cols, type) header; only a Mat made over
// caller memory has pixels.  resize, cvtColor, convertTo and split do no pixel work: the shim records the crop rectangle taken
// from an image and the size cv::resize is asked for (ref_cls_crop_geometry reads them back), and at<T> reads a dummy element.
#pragma once
#include <algorithm>
#include <cassert>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iostream>
#include <map>
#include <sstream>
#include <string>
#include <unordered_map>
#include <vector>

#define CV_8UC1 0
#define CV_8UC3 16
#define CV_32F 5
#define CV_32FC3 21

typedef unsigned char uchar;

namespace cv {
template <typename T>
struct Size_ {
    T width{}, height{};
    Size_() = default;
    Size_(T w, T h) : width(w), height(h) {}
};
using Size = Size_<int>;
template <typename T>
struct Rect_ {
    T x{}, y{}, width{}, height{};
    Rect_() = default;
    Rect_(T x_, T y_, T w, T h) : x(x_), y(y_), width(w), height(h) {}
};
using Rect = Rect_<int>;
struct Scalar {
    double val[4]{};
    Scalar() = default;
    Scalar(double a, double b = 0, double c = 0, double d = 0) : val{a, b, c, d} {}
};

class Mat {
   public:
    int rows{0}, cols{0}, type_{0};
    unsigned char* data{nullptr};
    size_t step{0};
    Mat() = default;
    Mat(int r, int c, int type) : rows(r), cols(c), type_(type) {}
    Mat(int r, int c, int type, const Scalar&) : Mat(r, c, type) {}
    Mat(int r, int c, int type, void* d, size_t s = 0)
        : rows(r), cols(c), type_(type), data(static_cast<unsigned char*>(d)), step(s ? s : (size_t)c * 3) {}
    Mat operator()(const Rect& r) const {
        int* g = shim_geometry();
        g[0] = r.x, g[1] = r.y, g[2] = r.width, g[3] = r.height;
        return Mat(r.height, r.width, type_);
    }
    // {rect x, rect y, rect width, rect height, resize width, resize height} of the last calls on this thread
    static int* shim_geometry() {
        static thread_local int v[6] = {0, 0, 0, 0, 0, 0};
        return v;
    }
    Size size() const { return Size(cols, rows); }
    bool empty() const { return rows <= 0 || cols <= 0; }
    int type() const { return type_; }
    void copyTo(Mat&&) const {}
    void copyTo(Mat&) const {}
    void convertTo(Mat& dst, int type, double = 1, double = 0) const {
        dst.rows = rows, dst.cols = cols, dst.type_ = type, dst.data = nullptr;
    }
    template <typename T>
    T& at(int, int) {
        static thread_local T dummy{};
        return dummy;
    }
};

enum { INTER_LINEAR = 1 };
enum { COLOR_BGR2RGB = 4 };

inline void resize(const Mat& src, Mat& dst, Size s, double = 0, double = 0, int = INTER_LINEAR) {
    Mat::shim_geometry()[4] = s.width;
    Mat::shim_geometry()[5] = s.height;
    dst.rows = s.height, dst.cols = s.width, dst.type_ = src.type_, dst.data = nullptr;
}
inline void cvtColor(const Mat& src, Mat& dst, int) { dst.rows = src.rows, dst.cols = src.cols, dst.type_ = src.type_; }
inline void split(const Mat& src, std::vector<Mat>& ch) {
    for (auto& m : ch) m = Mat(src.rows, src.cols, CV_32F);
}
inline Mat imread(const std::string&) { return Mat(); }
}  // namespace cv
