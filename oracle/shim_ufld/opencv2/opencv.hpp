// SHIM, not OpenCV -- TEST INFRASTRUCTURE.  The cv:: names that UFLD's driver (ufld/lane_det.cpp) and ufld/common.hpp mention,
// so that its argmax and softmax_mul compile where they lie (oracle/Makefile).  Type stubs only: no function here does pixel
// work, and prepareImage is never called (the tests pin the pre-process to cv2 itself).
#pragma once
#include <cassert>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#define CV_8UC3 16
#define CV_32FC3 21
#define CV_RGB(r, g, b) cv::Scalar((b), (g), (r))

namespace cv {
struct Size {
    int width{}, height{};
    Size() = default;
    Size(int w, int h) : width(w), height(h) {}
};
struct Point {
    int x{}, y{};
    Point() = default;
    Point(int x_, int y_) : x(x_), y(y_) {}
};
struct Scalar {
    double val[4]{};
    Scalar() = default;
    Scalar(double a, double b = 0, double c = 0, double d = 0) : val{a, b, c, d} {}
};
class Mat {
   public:
    unsigned char* data{nullptr};
    bool empty() const { return data == nullptr; }
    void convertTo(Mat&, int, double = 1, double = 0) const {}
};
struct MatExpr {
    operator Mat() const { return Mat(); }
};
inline MatExpr operator-(const Mat&, double) { return MatExpr(); }
inline MatExpr operator/(const MatExpr&, double) { return MatExpr(); }
enum { COLOR_BGR2RGB = 4 };
inline void cvtColor(const Mat&, Mat&, int) {}
inline void resize(const Mat&, Mat&, Size) {}
inline void split(const Mat&, std::vector<Mat>&) {}
inline Mat imread(const std::string&, int = 1) { return Mat(); }
inline void circle(Mat&, Point, int, const Scalar&, int = 1) {}
inline void imshow(const std::string&, const Mat&) {}
inline int waitKey(int = 0) { return -1; }
}  // namespace cv
