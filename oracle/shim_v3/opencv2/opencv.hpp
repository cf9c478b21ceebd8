// SHIM, not OpenCV -- TEST INFRASTRUCTURE.  The cv:: names that the yolov3 / yolov4 / scaled-yolov4 / yolov3-tiny / yolov3-spp
// drivers and their headers mention, so that their get_rect and yolov3-spp's letterbox compile where they lie (oracle/Makefile).
// An image is a (rows, cols, type) header with no pixels: get_rect reads rows and cols only; for the letterbox the shim records
// the last rectangle taken from an image and the last size cv::resize was asked for (Mat::shim_geometry), and the canvas
// letterbox returns carries its size.
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
#include <vector>

#define CV_8UC3 16
#define CV_32F 5

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
struct Point {
    int x{}, y{};
    Point(int x_, int y_) : x(x_), y(y_) {}
};
struct Scalar {
    double val[4]{};
    Scalar() = default;
    Scalar(double a, double b = 0, double c = 0, double d = 0) : val{a, b, c, d} {}
};
template <typename T, int n>
struct Vec {
    T v[n]{};
    T& operator[](int i) { return v[i]; }
};
using Vec3b = Vec<unsigned char, 3>;

class Mat {
   public:
    int rows{0}, cols{0}, type_{0};
    Mat() = default;
    Mat(int r, int c, int type) : rows(r), cols(c), type_(type) {}
    Mat(int r, int c, int type, const Scalar&) : Mat(r, c, type) {}
    // {rect x, rect y, rect width, rect height, resize width, resize height} of the last calls on this thread
    static int* shim_geometry() {
        static thread_local int v[6] = {0, 0, 0, 0, 0, 0};
        return v;
    }
    Mat operator()(const Rect& r) const {
        int* g = shim_geometry();
        g[0] = r.x, g[1] = r.y, g[2] = r.width, g[3] = r.height;
        return Mat(r.height, r.width, type_);
    }
    Size size() const { return Size(cols, rows); }
    bool empty() const { return rows <= 0 || cols <= 0; }
    void copyTo(Mat&&) const {}
    void copyTo(Mat&) const {}
    template <typename T>
    T& at(int) {
        static thread_local T dummy{};
        return dummy;
    }
    template <typename T>
    T* ptr(int) const { return nullptr; }
};

enum { INTER_LINEAR = 1, INTER_CUBIC = 2 };
enum { FONT_HERSHEY_PLAIN = 1 };

inline void resize(const Mat& src, Mat& dst, Size s, double = 0, double = 0, int = INTER_LINEAR) {
    Mat::shim_geometry()[4] = s.width;
    Mat::shim_geometry()[5] = s.height;
    dst.rows = s.height, dst.cols = s.width, dst.type_ = src.type_;
}
inline Mat imread(const std::string&) { return Mat(); }
inline bool imwrite(const std::string&, const Mat&) { return true; }
inline void rectangle(Mat&, const Rect&, const Scalar&, int = 1) {}
inline void putText(Mat&, const std::string&, Point, int, double, Scalar, int = 1) {}
}  // namespace cv
