// SHIM, not OpenCV -- TEST INFRASTRUCTURE.  The cv:: names that the reference's rcnn/common.hpp mentions, so that its
// preprocessImg (:79-102) compiles where it lies (oracle/Makefile, target `ref`) and can be called for its four pads.
// An image is a (rows, cols, type) header without pixels: resize, the 128-grey canvas and the copy into it do no pixel
// work, since only the int& pad outputs are read back.
#pragma once
#include <algorithm>
#include <cassert>
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

#define CV_8UC1 0
#define CV_8UC3 16

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
    Mat() = default;
    Mat(int r, int c, int type) : rows(r), cols(c), type_(type) {}
    Mat(int r, int c, int type, const Scalar&) : Mat(r, c, type) {}
    Mat(int r, int c, int type, void* d) : rows(r), cols(c), type_(type), data(static_cast<unsigned char*>(d)) {}
    Mat operator()(const Rect& r) const { return Mat(r.height, r.width, type_); }
    Size size() const { return Size(cols, rows); }
    bool empty() const { return rows <= 0 || cols <= 0; }
    void copyTo(Mat&&) const {}
};

enum { INTER_LINEAR = 1 };

inline void resize(const Mat&, Mat& dst, Size s, double = 0, double = 0, int = INTER_LINEAR) {
    dst.cols = s.width;
    dst.rows = s.height;
}
}  // namespace cv
