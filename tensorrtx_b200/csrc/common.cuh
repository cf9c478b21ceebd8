// common.cuh -- shared device helpers for libtrtx_hot (sm_90a only).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "trtx_hot.h"

namespace trtx {

constexpr int kWarp = 32;
constexpr size_t kAlign = 256;  // workspace sub-buffer alignment (rcnn/cuda_utils.h:7 uses the same)

__host__ __device__ inline size_t align_up(size_t v, size_t a = kAlign) { return (v + a - 1) / a * a; }

// thread-local last CUDA error (trtx_last_cuda_error)
extern thread_local int g_last_cuda_error;
inline int check_launch() {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        g_last_cuda_error = (int)e;
        return TRTX_ERR_CUDA;
    }
    return TRTX_OK;
}

// ---- streaming loads: read-once data bypasses L1 allocation (guide: Guideline 13/14) ----
__device__ __forceinline__ float4 ldg_stream_f4(const float* p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
                 : "l"(p));
    return r;
}
__device__ __forceinline__ float ldg_stream_f1(const float* p) {
    float r;
    asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(r) : "l"(p));
    return r;
}
// 4 halfs (8 bytes) -> 4 floats
__device__ __forceinline__ float4 ldg_stream_h4(const __half* p) {
    uint32_t a, b;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(a), "=r"(b) : "l"(p));
    __half2 h0 = *reinterpret_cast<__half2*>(&a);
    __half2 h1 = *reinterpret_cast<__half2*>(&b);
    float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
    return make_float4(f0.x, f0.y, f1.x, f1.y);
}
// 8 halfs (16 bytes), raw
__device__ __forceinline__ uint4 ldg_stream_h8(const __half* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ float ldg_stream_h1(const __half* p) {
    unsigned short r;
    asm volatile("ld.global.nc.L1::no_allocate.u16 %0, [%1];" : "=h"(r) : "l"(p));
    return __half2float(__ushort_as_half(r));
}

template <typename T>
struct Elem;
template <>
struct Elem<float> {
    static __device__ __forceinline__ float4 ld4(const float* p) { return ldg_stream_f4(p); }
    static __device__ __forceinline__ float ld1(const float* p) { return ldg_stream_f1(p); }
    static __device__ __forceinline__ float ld1_cached(const float* p) { return __ldg(p); }
};
template <>
struct Elem<__half> {
    static __device__ __forceinline__ float4 ld4(const __half* p) { return ldg_stream_h4(p); }
    static __device__ __forceinline__ float ld1(const __half* p) { return ldg_stream_h1(p); }
    static __device__ __forceinline__ float ld1_cached(const __half* p) { return __half2float(__ldg(p)); }
};

// The reference's Logist(): 1.0f / (1.0f + expf(-x)), IEEE division, CUDA expf
// (yolov8/plugin/yololayer.cu:174-176).  No fast-math anywhere in this library.
__device__ __forceinline__ float logist(float x) { return 1.0f / (1.0f + expf(-x)); }

// order-preserving float -> uint32 (larger float => larger key); -0.0 < +0.0 like cub's radix twiddle
__device__ __forceinline__ uint32_t float_key(float f) {
    uint32_t b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// One destination index d of OpenCV 4.x's 8-bit INTER_LINEAR resize (imgproc/src/resize.cpp) along an axis of `sn` source
// samples: fx = (float)((d + 0.5) * scale - 0.5), s = cvFloor(fx), fx -= s; with `clamp` (the x axis) a tap outside [0, sn - 1)
// moves to the border with a zero fraction, without it (the y axis) s and fx are kept and the rows are clipped where they are
// read; the weights are saturate_cast<short>((1 - fx) * 2048) and (fx * 2048), cvRound = round half to even.  The library's
// only floating-point step of that resize, shared by the host calibrator (calib_host.cu) and the R-CNN pre-process kernel
// (preprocess.cu).  The device spells the double expression with _rn intrinsics: left to itself nvcc may contract it into
// a DFMA, which rounds once where the host rounds twice.
struct LinearTap {
    int s;           // low tap (x: clamped; y: not clamped)
    short c0, c1;    // fixed-point weights, c0 + c1 = 2048
};
__host__ __device__ inline LinearTap cv_linear_tap(int d, double scale, int sn, bool clamp) {
#ifdef __CUDA_ARCH__
    float f = __double2float_rn(__dadd_rn(__dmul_rn(__dadd_rn((double)d, 0.5), scale), -0.5));
#else
    float f = (float)((d + 0.5) * scale - 0.5);
#endif
    int s = (int)floorf(f);
    f -= (float)s;
    if (clamp) {
        if (s < 0) f = 0, s = 0;
        if (s >= sn - 1) f = 0, s = sn - 1;
    }
    LinearTap t;
    t.s = s;
#ifdef __CUDA_ARCH__
    t.c0 = (short)__float2int_rn(__fmul_rn(__fsub_rn(1.f, f), 2048.f));
    t.c1 = (short)__float2int_rn(__fmul_rn(f, 2048.f));
#else
    t.c0 = (short)lrintf((1.f - f) * 2048.f);
    t.c1 = (short)lrintf(f * 2048.f);
#endif
    return t;
}

// Rounded float arithmetic spelled once for host and device: plain operators on the host (built without contraction),
// _rn intrinsics on the device so that nvcc cannot fuse a product into an FMA.
__host__ __device__ inline float f_mul(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
__host__ __device__ inline float f_sub(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fsub_rn(a, b);
#else
    return a - b;
#endif
}
__host__ __device__ inline float f_add(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}
__host__ __device__ inline float f_div(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fdiv_rn(a, b);
#else
    return a / b;
#endif
}

// round() of a float to int, false where the reference's int conversion is undefined (NaN, inf, outside the int range)
__host__ __device__ inline bool round_to_int(float v, int& out) {
    const double r = round((double)v);
    if (!(r >= -2147483648.0 && r <= 2147483647.0)) return false;
    out = (int)r;
    return true;
}

// The letterbox of an img_w x img_h frame inside the net_w x net_h input, as get_rect and get_rect_adapt_landmark
// (yolov8/src/postprocess.cpp:6-69) spell it: `kInputW / (img.cols * 1.0)` is a double division stored to float, the pad
// `(kInputH - r_w * img.rows) / 2` is float.
struct YoloLetterbox {
    float ratio;  // r_w where the width fills the input (by_w), else r_h
    float pad;    // the padding on the other axis, in network pixels
    bool by_w;    // r_h > r_w: vertical padding
};
__host__ __device__ inline YoloLetterbox yolo_letterbox(int net_w, int net_h, int img_w, int img_h) {
#ifdef __CUDA_ARCH__
    const float r_w = __double2float_rn(__ddiv_rn((double)net_w, (double)img_w));
    const float r_h = __double2float_rn(__ddiv_rn((double)net_h, (double)img_h));
#else
    const float r_w = (float)(net_w / (img_w * 1.0));
    const float r_h = (float)(net_h / (img_h * 1.0));
#endif
    YoloLetterbox lb;
    lb.by_w = r_h > r_w;
    lb.ratio = lb.by_w ? r_w : r_h;
    lb.pad = lb.by_w ? f_div(f_sub((float)net_h, f_mul(r_w, (float)img_h)), 2.0f)
                     : f_div(f_sub((float)net_w, f_mul(r_h, (float)img_w)), 2.0f);
    return lb;
}

// One keypoint coordinate of get_rect_adapt_landmark (yolov8/src/postprocess.cpp:47-61): axis 0 = x, 1 = y.  The padded axis
// loses the pad first, then both are divided by the ratio, all in float; the keypoint's confidence is not touched.
__host__ __device__ inline float yolo_map_landmark(const YoloLetterbox& lb, int axis, float v) {
    return (axis == 0) == lb.by_w ? f_div(v, lb.ratio) : f_div(f_sub(v, lb.pad), lb.ratio);
}

// get_rect: the inverse of the letterbox for a detection box -- yolov8/src/postprocess.cpp:6-36 (TRTX_YOLO_V8: l,t,r,b,
// clamped to the image) and yolov5/src/postprocess.cpp:4-29 (TRTX_YOLO_V5: cx,cy,w,h, not clamped).  Statement by statement:
// the two ratios are double divisions stored to float, the rest is float, round() sees doubles.  Shared by the host
// trtx_get_rect and trtx_get_rect_adapt_landmark (whose rectangle is the same float expressions as the V8 branch), the
// segmentation post-process kernels (mask.cu) and yolo_get_corner.  Returns false, with rect {0, 0, 0, 0}, where the
// reference's float -> int conversions are undefined (a non-finite box, or rescaled corners outside the int range).
__host__ __device__ inline bool yolo_get_rect(int variant, int net_w, int net_h, int img_w, int img_h, const float bbox[4],
                                              int rect[4]) {
    rect[0] = rect[1] = rect[2] = rect[3] = 0;
    const YoloLetterbox lb = yolo_letterbox(net_w, net_h, img_w, img_h);
    const bool by_w = lb.by_w;
    const float ratio = lb.ratio, pad = lb.pad;
    float l, r, t, b;
    if (variant == TRTX_YOLO_V8) {
        l = bbox[0];
        r = bbox[2];
        t = bbox[1];
        b = bbox[3];
    } else {
        l = f_sub(bbox[0], f_div(bbox[2], 2.f));
        r = f_add(bbox[0], f_div(bbox[2], 2.f));
        t = f_sub(bbox[1], f_div(bbox[3], 2.f));
        b = f_add(bbox[1], f_div(bbox[3], 2.f));
    }
    if (by_w) {
        t = f_sub(t, pad);
        b = f_sub(b, pad);
    } else {
        l = f_sub(l, pad);
        r = f_sub(r, pad);
    }
    l = f_div(l, ratio);
    r = f_div(r, ratio);
    t = f_div(t, ratio);
    b = f_div(b, ratio);
    if (variant == TRTX_YOLO_V8) {
        l = 0.0f > l ? 0.0f : l;
        t = 0.0f > t ? 0.0f : t;
    }
    int rl, rt, rw, rh;
    if (!round_to_int(l, rl) || !round_to_int(t, rt) || !round_to_int(f_sub(r, l), rw) || !round_to_int(f_sub(b, t), rh))
        return false;
    if (variant == TRTX_YOLO_V8) {  // l, t >= 0 here, so img - round(l) cannot overflow
        const int width = rw < img_w - rl ? rw : img_w - rl, height = rh < img_h - rt ? rh : img_h - rt;
        rw = width > 0 ? width : 0;
        rh = height > 0 ? height : 0;
    }
    rect[0] = rl;
    rect[1] = rt;
    rect[2] = rw;
    rect[3] = rh;
    return true;
}

// get_corner: the four corners of an oriented box in the original frame -- yolov8/src/postprocess.cpp:395-472 (net 640) and
// yolo11/src/postprocess.cpp:425-502 (get_rect_obb: net 1024), statement by statement without the debug prints:
//   angle = box.angle * 180.0f / CV_PI        float product, DOUBLE division, stored to float
//   h >= w: swap w, h and angle = fmod(angle + 90.0f, 180.0f) (float; fmod is exact); then angle < 0: += 360, > 180: -= 180
//   cos / sin of angle * CV_PI / 180.0f       double expression and double cos / sin, stored to float
//   rect = get_rect of the axis-aligned l, t, r, b (cx -/+ w / 2, cy -/+ h / 2)
//   x_ = (rect.x + rect.x + rect.width) / 2   INTEGER division (the sum wraps as the compiled x86-64 reference does)
//   corner = int(round(x_ +/- vec1x +/- vec2x)) (float sums in source order), clamped to [0, cols - 1] x [0, rows - 1].
// corners = {x0, y0, x1, y1, x2, y2, x3, y3} in get_corner's order.  Undefined cases of the reference, defined here as the
// compiled reference behaves on x86-64: a corner whose float -> int conversion is undefined (NaN, out of range) converts to
// INT_MIN there, which the clamp makes 0; a box whose get_rect is undefined gets four (0, 0) corners.  The device's double
// cos / sin are within 2 ulp of glibc's, not correctly rounded: a float can differ only where the double lies that close
// to a float rounding boundary.
__host__ __device__ inline void yolo_get_corner(int net_w, int net_h, int img_w, int img_h, const float box[4], float box_angle,
                                                int corners[8]) {
    constexpr double kPi = 3.1415926535897932384626433832795;  // CV_PI
    for (int k = 0; k < 8; ++k) corners[k] = 0;
    float w = box[2], h = box[3];
#ifdef __CUDA_ARCH__
    float angle = __double2float_rn(__ddiv_rn((double)__fmul_rn(box_angle, 180.0f), kPi));
#else
    float angle = (float)((double)(box_angle * 180.0f) / kPi);
#endif
    if (h >= w) {
        const float s = w;
        w = h;
        h = s;
        angle = fmodf(f_add(angle, 90.0f), 180.0f);
    }
    if (angle < 0) angle = f_add(angle, 360.0f);
    if (angle > 180.0f) angle = f_sub(angle, 180.0f);
#ifdef __CUDA_ARCH__
    const double rad = __ddiv_rn(__dmul_rn((double)angle, kPi), 180.0);
    const float cos_value = __double2float_rn(cos(rad)), sin_value = __double2float_rn(sin(rad));
#else
    const double rad = (double)angle * kPi / 180.0;
    const float cos_value = (float)cos(rad), sin_value = (float)sin(rad);
#endif
    const float bbox[4] = {f_sub(box[0], f_div(w, 2.0f)), f_sub(box[1], f_div(h, 2.0f)), f_add(box[0], f_div(w, 2.0f)),
                           f_add(box[1], f_div(h, 2.0f))};
    int rect[4];
    if (!yolo_get_rect(TRTX_YOLO_V8, net_w, net_h, img_w, img_h, bbox, rect)) return;
    const float x_ = (float)((int)((unsigned)rect[0] + (unsigned)rect[0] + (unsigned)rect[2]) / 2);
    const float y_ = (float)((int)((unsigned)rect[1] + (unsigned)rect[1] + (unsigned)rect[3]) / 2);
    const float width = (float)rect[2], height = (float)rect[3];
    const float vec1x = f_mul(f_div(width, 2.0f), cos_value);
    const float vec1y = f_mul(f_div(width, 2.0f), sin_value);
    const float vec2x = f_mul(f_div(-height, 2.0f), sin_value);
    const float vec2y = f_mul(f_div(height, 2.0f), cos_value);
    const float v[8] = {f_add(f_add(x_, vec1x), vec2x), f_add(f_add(y_, vec1y), vec2y),
                        f_sub(f_add(x_, vec1x), vec2x), f_sub(f_add(y_, vec1y), vec2y),
                        f_sub(f_sub(x_, vec1x), vec2x), f_sub(f_sub(y_, vec1y), vec2y),
                        f_add(f_sub(x_, vec1x), vec2x), f_add(f_sub(y_, vec1y), vec2y)};
    for (int k = 0; k < 8; ++k) {
        const int hi = (k & 1) ? img_h - 1 : img_w - 1;
        int c;
        if (!round_to_int(v[k], c)) c = 0;  // INT_MIN in the reference, then its clamp
        corners[k] = c < 0 ? 0 : (c > hi ? hi : c);
    }
}

__device__ __forceinline__ int warp_excl_scan(int v, int lane, int* total) {
    int x = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        int y = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= d) x += y;
    }
    *total = __shfl_sync(0xffffffffu, x, 31);
    return x - v;
}

}  // namespace trtx
