// SHIM, not OpenCV -- TEST INFRASTRUCTURE (oracle/Makefile).  Declares the cv:: names the reference's
// yolov8/src/postprocess.cpp and yolov5/src/postprocess.cpp mention, so that their draw_mask_bbox + scale_mask + get_rect run
// from where they lie.  Unlike oracle/shim, the cv::Mat here has real, shared (reference-counted) storage and ROI views with
// the parent's row step, and cv::resize of a CV_32F image is the oracle's restatement of OpenCV's float bilinear resize
// (oracle_resize_bilinear in trtx_oracle.c, pinned to cv2 in tests/test_oracle_cpu.py).  Drawing calls (rectangle, putText,
// line, circle, polylines) are no-ops and getTextSize returns an empty size: the pixels they would touch are not part of the
// mask selection.  Everything else aborts if ever called.
#pragma once
#include <algorithm>
#include <cassert>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <functional>
#include <iostream>
#include <map>
#include <math.h>
#include <memory>
#include <numeric>
#include <sstream>
#include <string>
#include <unordered_map>
#include <vector>

#define CV_8UC1 0
#define CV_8UC3 16
#define CV_32F 5
#define CV_32FC1 5
#define CV_PI 3.1415926535897932384626433832795

extern "C" void oracle_resize_bilinear(const float* src, int sh, int sw, float* dst, int dh, int dw);

namespace cv {
[[noreturn]] inline void shim_abort(const char* what) {
    std::fprintf(stderr, "opencv shim: %s is not implemented (test infrastructure)\n", what);
    std::abort();
}
template <typename T>
struct Point_ {
    T x{}, y{};
    Point_() = default;
    Point_(T x_, T y_) : x(x_), y(y_) {}
};
using Point = Point_<int>;
using Point2f = Point_<float>;
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
    Point_<T> tl() const { return {x, y}; }
    Point_<T> br() const { return {x + width, y + height}; }
    T area() const { return width * height; }
};
using Rect = Rect_<int>;
struct Scalar {
    double val[4]{};
    Scalar() = default;
    Scalar(double a, double b = 0, double c = 0, double d = 0) : val{a, b, c, d} {}
    static Scalar all(double v) { return Scalar(v, v, v, v); }
    double& operator[](int i) { return val[i]; }
    const double& operator[](int i) const { return val[i]; }
};
template <typename T, int N>
struct Vec {
    T val[N]{};
    T& operator[](int i) { return val[i]; }
    const T& operator[](int i) const { return val[i]; }
};
using Vec3b = Vec<unsigned char, 3>;
using Vec3f = Vec<float, 3>;

class Mat {
   public:
    int rows{0}, cols{0}, type_{0};
    unsigned char* data{nullptr};
    size_t step{0};
    std::shared_ptr<std::vector<unsigned char>> own;  // shared like cv::Mat's reference count
    Mat() = default;
    Mat(int r, int c, int type, void* d, size_t st = 0) : rows(r), cols(c), type_(type), data(static_cast<unsigned char*>(d)) {
        step = st ? st : (size_t)c * elemSize();
    }
    Mat(int r, int c, int type) : rows(r), cols(c), type_(type) {  // zero-filled
        step = (size_t)c * elemSize();
        own = std::make_shared<std::vector<unsigned char>>(step * r, 0);
        data = own->data();
    }
    Mat(int r, int c, int type, const Scalar&) { shim_abort("Mat(rows, cols, type, Scalar)"); }
    size_t elemSize() const { return type_ == CV_8UC3 ? 3 : (type_ == CV_32F ? 4 : 1); }
    static Mat zeros(int r, int c, int type) { return Mat(r, c, type); }
    static Mat zeros(Size s, int type) { return Mat(s.height, s.width, type); }
    template <typename T>
    T* ptr(int r = 0) { return reinterpret_cast<T*>(data + (size_t)r * step); }
    template <typename T>
    const T* ptr(int r = 0) const { return reinterpret_cast<const T*>(data + (size_t)r * step); }
    unsigned char* ptr(int r = 0) { return data + (size_t)r * step; }
    const unsigned char* ptr(int r = 0) const { return data + (size_t)r * step; }
    template <typename T>
    T& at(int r, int c) { return *reinterpret_cast<T*>(data + (size_t)r * step + (size_t)c * sizeof(T)); }
    template <typename T>
    const T& at(int r, int c) const { return *reinterpret_cast<const T*>(data + (size_t)r * step + (size_t)c * sizeof(T)); }
    // ROI: a view with the parent's step (Mat::operator()(Rect) asserts the rectangle lies inside; so does this)
    Mat operator()(const Rect& r) const {
        if (r.x < 0 || r.y < 0 || r.width < 0 || r.height < 0 || r.x + r.width > cols || r.y + r.height > rows)
            shim_abort("Mat::operator()(Rect) outside the image");
        Mat v(r.height, r.width, type_, data + (size_t)r.y * step + (size_t)r.x * elemSize(), step);
        v.own = own;
        return v;
    }
    Mat clone() const { shim_abort("Mat::clone"); }
    bool empty() const { return data == nullptr; }
    Size size() const { return Size(cols, rows); }
    int channels() const { return type_ == CV_8UC3 ? 3 : 1; }
    int type() const { return type_; }
    void copyTo(Mat&) const { shim_abort("Mat::copyTo"); }
    void copyTo(Mat&&) const { shim_abort("Mat::copyTo"); }
    void convertTo(Mat&, int, double = 1, double = 0) const { shim_abort("Mat::convertTo"); }
    Mat& setTo(const Scalar&) { shim_abort("Mat::setTo"); }
};

enum { FONT_HERSHEY_PLAIN = 1, FONT_HERSHEY_SIMPLEX = 0, LINE_AA = 16, INTER_LINEAR = 1, BORDER_CONSTANT = 0 };

inline void rectangle(Mat&, Rect, const Scalar&, int = 1, int = 8, int = 0) {}
inline void rectangle(Mat&, Point, Point, const Scalar&, int = 1, int = 8, int = 0) {}
inline void putText(Mat&, const std::string&, Point, int, double, const Scalar&, int = 1, int = 8, bool = false) {}
inline Size getTextSize(const std::string&, int, double, int, int*) { return Size(0, 0); }
// cv::resize(src, dst, dsize) of a single-channel float image, INTER_LINEAR; an empty size throws in OpenCV
inline void resize(const Mat& src, Mat& dst, Size s, double = 0, double = 0, int = 1) {
    if (src.type_ != CV_32F) shim_abort("resize of a non-float image");
    if (src.rows <= 0 || src.cols <= 0 || s.width <= 0 || s.height <= 0) shim_abort("resize of an empty image");
    std::vector<float> packed((size_t)src.rows * src.cols);
    for (int y = 0; y < src.rows; ++y) std::memcpy(&packed[(size_t)y * src.cols], src.ptr<float>(y), sizeof(float) * src.cols);
    Mat out(s.height, s.width, CV_32F);
    oracle_resize_bilinear(packed.data(), src.rows, src.cols, out.ptr<float>(0), s.height, s.width);
    dst = out;
}
inline void line(Mat&, Point, Point, const Scalar&, int = 1, int = 8, int = 0) {}
inline void circle(Mat&, Point, int, const Scalar&, int = 1, int = 8, int = 0) {}
inline void polylines(Mat&, const std::vector<std::vector<Point>>&, bool, const Scalar&, int = 1, int = 8, int = 0) {}
inline void polylines(Mat&, const std::vector<Point>&, bool, const Scalar&, int = 1, int = 8, int = 0) {}
inline Mat imread(const std::string&, int = 1) { shim_abort("imread"); }
inline bool imwrite(const std::string&, const Mat&) { shim_abort("imwrite"); }
inline void exp(const Mat&, Mat&) { shim_abort("exp"); }
inline void invertAffineTransform(const Mat&, Mat&) { shim_abort("invertAffineTransform"); }
}  // namespace cv
