// SHIM, not OpenCV -- TEST INFRASTRUCTURE (oracle/Makefile).  Declares the cv:: names the reference's
// yolov8/src/postprocess.cpp and yolo11/src/postprocess.cpp mention, so that their draw_bbox_keypoints_line and draw_bbox_obb
// run whole from where they lie.  Only the geometry those functions hand to the drawing calls matters here, so
// cv::rectangle(img, Rect, ...), cv::circle and cv::polylines RECORD their arguments (cv::shim_record(), cleared by the
// caller); the other drawing calls are no-ops, getTextSize returns an empty size, and everything else aborts if ever called.
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

// a size only: the functions driven here read img.cols / img.rows and draw
class Mat {
   public:
    int rows{0}, cols{0}, type_{0};
    unsigned char* data{nullptr};
    Mat() = default;
    Mat(int r, int c, int type) : rows(r), cols(c), type_(type) {}
    Mat(int r, int c, int type, void* d, size_t = 0) : rows(r), cols(c), type_(type), data(static_cast<unsigned char*>(d)) {}
    Mat(int, int, int, const Scalar&) { shim_abort("Mat(rows, cols, type, Scalar)"); }
    static Mat zeros(int r, int c, int type) { return Mat(r, c, type); }
    static Mat zeros(Size s, int type) { return Mat(s.height, s.width, type); }
    template <typename T>
    T& at(int, int) { shim_abort("Mat::at"); }
    unsigned char* ptr(int = 0) { shim_abort("Mat::ptr"); }
    Mat operator()(const Rect&) const { shim_abort("Mat::operator()(Rect)"); }
    Mat clone() const { shim_abort("Mat::clone"); }
    bool empty() const { return rows == 0 || cols == 0; }
    Size size() const { return Size(cols, rows); }
    int channels() const { return type_ == CV_8UC3 ? 3 : 1; }
    int type() const { return type_; }
    void copyTo(Mat&) const { shim_abort("Mat::copyTo"); }
    void copyTo(Mat&&) const { shim_abort("Mat::copyTo"); }
    void convertTo(Mat&, int, double = 1, double = 0) const { shim_abort("Mat::convertTo"); }
    Mat& setTo(const Scalar&) { shim_abort("Mat::setTo"); }
};

// what the recording drawing calls saw, in call order
struct ShimRecord {
    std::vector<Rect> rects;       // cv::rectangle(img, Rect, ...)
    std::vector<Point> circles;    // cv::circle centres
    std::vector<Point> polylines;  // every vertex of every cv::polylines call
};
inline ShimRecord& shim_record() {
    static ShimRecord r;
    return r;
}

enum { FONT_HERSHEY_PLAIN = 1, FONT_HERSHEY_SIMPLEX = 0, LINE_AA = 16, INTER_LINEAR = 1, BORDER_CONSTANT = 0 };

inline void rectangle(Mat&, Rect r, const Scalar&, int = 1, int = 8, int = 0) { shim_record().rects.push_back(r); }
inline void rectangle(Mat&, Point, Point, const Scalar&, int = 1, int = 8, int = 0) {}
inline void putText(Mat&, const std::string&, Point, int, double, const Scalar&, int = 1, int = 8, bool = false) {}
inline Size getTextSize(const std::string&, int, double, int, int*) { return Size(0, 0); }
inline void resize(const Mat&, Mat&, Size, double = 0, double = 0, int = 1) { shim_abort("resize"); }
inline void line(Mat&, Point, Point, const Scalar&, int = 1, int = 8, int = 0) {}
inline void circle(Mat&, Point c, int, const Scalar&, int = 1, int = 8, int = 0) { shim_record().circles.push_back(c); }
inline void polylines(Mat&, const std::vector<std::vector<Point>>& pts, bool, const Scalar&, int = 1, int = 8, int = 0) {
    for (const auto& poly : pts) shim_record().polylines.insert(shim_record().polylines.end(), poly.begin(), poly.end());
}
inline void polylines(Mat&, const std::vector<Point>& pts, bool, const Scalar&, int = 1, int = 8, int = 0) {
    shim_record().polylines.insert(shim_record().polylines.end(), pts.begin(), pts.end());
}
inline Mat imread(const std::string&, int = 1) { shim_abort("imread"); }
inline bool imwrite(const std::string&, const Mat&) { shim_abort("imwrite"); }
inline void exp(const Mat&, Mat&) { shim_abort("exp"); }
inline void invertAffineTransform(const Mat&, Mat&) { shim_abort("invertAffineTransform"); }
}  // namespace cv
