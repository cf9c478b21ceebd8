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

// Opts `kernel` in to `smem` bytes of dynamic shared memory where its current limit is lower.  Without an opt-in the limit is
// 48 KiB less the kernel's static shared memory (so a band kernel's 4 KiB of static arrays and tables leave it 44 KiB), not
// 48 KiB.  TRTX_ERR_CUDA, the error in g_last_cuda_error, where the limit cannot be read or raised.
template <class Kernel>
inline int opt_in_smem(Kernel* kernel, size_t smem) {
    cudaFuncAttributes fa;
    cudaError_t e = cudaFuncGetAttributes(&fa, kernel);
    if (e == cudaSuccess && smem > (size_t)fa.maxDynamicSharedSizeBytes)
        e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess) return TRTX_OK;
    g_last_cuda_error = (int)cudaGetLastError();
    return TRTX_ERR_CUDA;
}

// The frame descriptors every pre-process accepts: non-null u8 HWC BGR frames of positive size whose rows hold 3 * width bytes.
inline bool valid_images(const trtx_image_desc* images, int n) {
    for (int i = 0; i < n; ++i) {
        const trtx_image_desc& d = images[i];
        if (!d.data_dev || d.width <= 0 || d.height <= 0 || d.pitch < 3 * d.width) return false;
    }
    return true;
}

// Frames (or image descriptors) per launch of a per-frame entry: their data rides in the kernel's parameter block.
constexpr int kMaxFrames = 64;

// The sizes of the frames of one launch of a per-frame post-process, one CTA per frame.
struct FrameSizes {
    int w[kMaxFrames], h[kMaxFrames];  // of frame base + blockIdx.x
    int base;                          // frames [base, base + gridDim.x) of the call
};

// A per-frame post-process's frame_wh_host: `batch` (w, h) pairs in host memory, every side positive.
inline bool frames_valid(const int32_t* frame_wh_host, int batch) {
    for (int i = 0; i < batch; ++i)
        if (frame_wh_host[2 * i] <= 0 || frame_wh_host[2 * i + 1] <= 0) return false;
    return true;
}

// The size source of launch_frames for a frame_wh_host: frame i's (w, h), or 0 x 0 where frame_wh_host is null (a call
// without frame rows).
inline auto frame_wh(const int32_t* frame_wh_host) {
    return [frame_wh_host](int i, int& w, int& h) {
        w = frame_wh_host ? frame_wh_host[2 * i] : 0;
        h = frame_wh_host ? frame_wh_host[2 * i + 1] : 0;
    };
}

// One launch of `kernel` per <= kMaxFrames frames of a call, one CTA of `threads` per frame.  Before each launch, `base`
// gets the launch's first frame i0, and for frame j of the launch, frame i0 + j of the call, size(i0 + j, w, h) gives its
// size and frame(j, w, h) fills the caller's launch parameters.
template <class Args, class Size, class Frame>
int launch_frames(void (*kernel)(Args), Args& a, int& base, int batch, int threads, size_t smem, cudaStream_t st, Size size,
                  Frame frame) {
    for (int i0 = 0; i0 < batch; i0 += kMaxFrames) {
        const int n = min(batch - i0, kMaxFrames);
        base = i0;
        for (int j = 0; j < n; ++j) {
            int w, h;
            size(i0 + j, w, h);
            frame(j, w, h);
        }
        kernel<<<n, threads, smem, st>>>(a);
        const int rc = check_launch();
        if (rc) return rc;
    }
    return TRTX_OK;
}

// The same where a frame's launch parameters are its size alone, in `sizes`.
template <class Args, class Size>
int launch_frames(void (*kernel)(Args), Args& a, FrameSizes& sizes, int batch, int threads, size_t smem, cudaStream_t st,
                  Size size) {
    return launch_frames(kernel, a, sizes.base, batch, threads, smem, st, size,
                         [&](int j, int w, int h) { sizes.w[j] = w, sizes.h[j] = h; });
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

// order-preserving float -> uint32 (larger float => larger key).  -0.0 is mapped to +0.0 first, so the two zeros are one
// key and tie on the index like any other equal scores -- as in cub's radix sort ("positive and negative zeros are
// considered equivalent") and the reference's float comparisons.  Keys are only compared, never turned back into floats.
__device__ __forceinline__ uint32_t float_key(float f) {
    uint32_t b = __float_as_uint(f);
    b = b == 0x80000000u ? 0u : b;
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// One destination index d of OpenCV 4.x's 8-bit INTER_LINEAR resize (imgproc/src/resize.cpp) along an axis of `sn` source
// samples: fx = (float)((d + 0.5) * scale - 0.5), s = cvFloor(fx), fx -= s; with `clamp` (the x axis) a tap outside [0, sn - 1)
// moves to the border with a zero fraction, without it (the y axis) s and fx are kept and the rows are clipped where they are
// read; the weights are saturate_cast<short>((1 - fx) * 2048) and (fx * 2048), cvRound = round half to even.  The library's
// only floating-point step of that resize, shared by the host calibrator (calib_host.cu) and the R-CNN pre-process kernel
// (preprocess.cu).  The device spells the double expression with _rn intrinsics: left to itself nvcc may contract it into
// a DFMA, which rounds once where the host rounds twice.
// cv_linear_coord is the geometry alone, the low tap and its float fraction fx; the float64 resize of the CenterNet
// pre-process (centernet.cu) weights by (1 - fx, fx) in float.
struct LinearCoord {
    int s;    // low tap (clamped or not, as for LinearTap)
    float f;  // fraction, 0 where the tap was clamped
};
__host__ __device__ inline LinearCoord cv_linear_coord(int d, double scale, int sn, bool clamp) {
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
    return LinearCoord{s, f};
}
struct LinearTap {
    int s;           // low tap (x: clamped; y: not clamped)
    short c0, c1;    // fixed-point weights, c0 + c1 = 2048
};
__host__ __device__ inline LinearTap cv_linear_tap(int d, double scale, int sn, bool clamp) {
    const LinearCoord g = cv_linear_coord(d, scale, sn, clamp);
    const float f = g.f;
    LinearTap t;
    t.s = g.s;
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

// (int)v where it is defined: v truncated toward zero fits an int.  False for NaN, +-inf and values past the int range
// (in float, v >= -2^31 is the same as trunc(v) >= INT_MIN).  Shared by the truncating get_rects below and process_mask (mask.cu).
__host__ __device__ inline bool trunc_to_int(float v, int& out) {
    if (!(v >= -2147483648.0f && v < 2147483648.0f)) return false;
    out = (int)v;
    return true;
}

// The corners l, t, r, b of a cx, cy, w, h box as the truncating get_rect of yolov3 / yolov4 / scaled-yolov4 / yolov3-tiny and
// YOLOP (yolov3/yolov3.cpp:30-52, yolop/common.hpp:13-37; the same statements) compute them before their first int store:
// `bbox[0] - bbox[2]/2.f`, minus the pad `(INPUT_H - r_w * img.rows) / 2` on the padded axis, all in float.
__host__ __device__ inline void trunc_rect_corners(const YoloLetterbox& lb, const float bbox[4], float c[4]) {
    c[0] = f_sub(bbox[0], f_div(bbox[2], 2.f));
    c[1] = f_sub(bbox[1], f_div(bbox[3], 2.f));
    c[2] = f_add(bbox[0], f_div(bbox[2], 2.f));
    c[3] = f_add(bbox[1], f_div(bbox[3], 2.f));
    const int padded = lb.by_w ? 1 : 0;  // the axis that carries the pad: y when the width fills the input
    c[padded] = f_sub(c[padded], lb.pad);
    c[padded + 2] = f_sub(c[padded + 2], lb.pad);
}

// rect = {l, t, r - l, b - t} of four truncated corners; false where r - l or b - t overflows int.
__host__ __device__ inline bool int_rect(const int v[4], int rect[4]) {
    const long long w = (long long)v[2] - v[0], h = (long long)v[3] - v[1];
    if (w < INT32_MIN || w > INT32_MAX || h < INT32_MIN || h > INT32_MAX) return false;
    rect[0] = v[0];
    rect[1] = v[1];
    rect[2] = (int)w;
    rect[3] = (int)h;
    return true;
}

// get_rect of yolov3, yolov4, scaled-yolov4 and yolov3-tiny (yolov3/yolov3.cpp:30-52, yolov4/yolov4.cpp:55-77,
// scaled-yolov4/common.hpp:36-58, yolov3-tiny/yolov3-tiny.cpp:62-84): every assignment to `int l, r, t, b` truncates toward
// zero, so a corner is truncated after trunc_rect_corners and again after `l = l / r_w` (int -> float, a float division); no
// clamp.  Returns false, with rect {0, 0, 0, 0}, where the reference is undefined: a conversion of a NaN, an infinity or a
// float outside the int range, or an r - l that overflows.
__host__ __device__ inline bool yolov3_get_rect(const YoloLetterbox& lb, const float bbox[4], int rect[4]) {
    rect[0] = rect[1] = rect[2] = rect[3] = 0;
    float c[4];
    trunc_rect_corners(lb, bbox, c);
    int v[4];
    for (int k = 0; k < 4; ++k) {
        int t;
        if (!trunc_to_int(c[k], t) || !trunc_to_int(f_div((float)t, lb.ratio), v[k])) return false;
    }
    return int_rect(v, rect);
}

// yolov3-spp's letterbox (yolov3-spp/yolov3-spp.cpp:43-56) and the same lines at the top of its get_rect (:58-64), for MAX =
// max_size: r = std::min(MAX / (w * 1.0), MAX / (h * 1.0)) stored to float, r = std::min(r, 1.0f); unpad = (int)(r * w) in
// float; d = (MAX - unpad) % 32 per axis.  The canvas is (unpad_w + dw) x (unpad_h + dh), the resized frame sits at
// (dw / 2, dh / 2).
struct SppLetterbox {
    float ratio;
    int unpad_w, unpad_h, dw, dh;
};
__host__ __device__ inline SppLetterbox yolov3spp_letterbox(int max_size, int img_w, int img_h) {
#ifdef __CUDA_ARCH__
    const double a = __ddiv_rn((double)max_size, (double)img_w), b = __ddiv_rn((double)max_size, (double)img_h);
    float r = __double2float_rn(a < b ? a : b);
#else
    const double a = max_size / (img_w * 1.0), b = max_size / (img_h * 1.0);
    float r = (float)(a < b ? a : b);
#endif
    r = r < 1.0f ? r : 1.0f;
    SppLetterbox lb;
    lb.ratio = r;
    lb.unpad_w = (int)f_mul(r, (float)img_w);
    lb.unpad_h = (int)f_mul(r, (float)img_h);
    lb.dw = (max_size - lb.unpad_w) % 32;
    lb.dh = (max_size - lb.unpad_h) % 32;
    return lb;
}

// yolov3-spp's get_rect (yolov3-spp.cpp:58-75): `int l = bbox[0] - bbox[2]/2.f - dw / 2` (the pad an int division, the rest
// float, truncated), then `l /= ra` (int -> float, a float division, truncated); no clamp; undefined cases as yolov3_get_rect.
__host__ __device__ inline bool yolov3spp_get_rect(int max_size, int img_w, int img_h, const float bbox[4], int rect[4]) {
    rect[0] = rect[1] = rect[2] = rect[3] = 0;
    const SppLetterbox lb = yolov3spp_letterbox(max_size, img_w, img_h);
    const float px = (float)(lb.dw / 2), py = (float)(lb.dh / 2);
    const float c[4] = {f_sub(f_sub(bbox[0], f_div(bbox[2], 2.f)), px), f_sub(f_sub(bbox[1], f_div(bbox[3], 2.f)), py),
                        f_sub(f_add(bbox[0], f_div(bbox[2], 2.f)), px), f_sub(f_add(bbox[1], f_div(bbox[3], 2.f)), py)};
    int v[4];
    for (int k = 0; k < 4; ++k) {
        int t;
        if (!trunc_to_int(c[k], t) || !trunc_to_int(f_div((float)t, lb.ratio), v[k])) return false;
    }
    return int_rect(v, rect);
}

// get_rect: the inverse of the letterbox for a detection box -- yolov8/src/postprocess.cpp:6-36 (TRTX_YOLO_V8: l,t,r,b,
// clamped to the image) and yolov5/src/postprocess.cpp:4-29 (TRTX_YOLO_V5: cx,cy,w,h, not clamped).  Statement by statement:
// the two ratios are double divisions stored to float, the rest is float, round() sees doubles.  Shared by the host
// trtx_get_rect and trtx_get_rect_adapt_landmark (whose rectangle is the same float expressions as the V8 branch), the
// segmentation post-process kernels (mask.cu) and yolo_get_corner.  Returns false, with rect {0, 0, 0, 0}, where the
// reference's float -> int conversions are undefined (a non-finite box, or rescaled corners outside the int range).
// TRTX_YOLO_V3 is yolov3_get_rect, TRTX_RECT_YOLOV3_SPP yolov3spp_get_rect with MAX = net_w.
__host__ __device__ inline bool yolo_get_rect(int variant, int net_w, int net_h, int img_w, int img_h, const float bbox[4],
                                              int rect[4]) {
    if (variant == TRTX_YOLO_V3) return yolov3_get_rect(yolo_letterbox(net_w, net_h, img_w, img_h), bbox, rect);
    if (variant == TRTX_RECT_YOLOV3_SPP) return yolov3spp_get_rect(net_w, img_w, img_h, bbox, rect);
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

// A float -> int conversion as the compiled x86-64 reference performs it (cvttss2si): truncation toward zero, and INT_MIN
// for NaN, +-inf and values outside [-2^31, 2^31), where C++ leaves the conversion undefined.  Spelled out because the
// device's __float2int_rz saturates instead and maps NaN to 0.
__host__ __device__ inline int trunc_to_int_x86(float v) {
    return v >= -2147483648.0f && v < 2147483648.0f ? (int)v : INT32_MIN;
}

// RetinaFace's get_rect_adapt_landmark (retinaface/common.hpp:65-89; retinafaceAntiCov/retinafaceAntiCov.cpp:63-87 is the
// same statements at 640 x 640): every coordinate of the box and of the 5 landmarks is mapped as yolo_map_landmark maps it
// (the letterbox expressions are get_rect's), then the box corners are TRUNCATED to int (trunc_to_int_x86) and not clamped;
// w = r - l and h = b - t are int differences, which wrap modulo 2^32 as on x86-64.  rect = {l, t, w, h}; lmk (x, y pairs)
// is mapped in place.
__host__ __device__ inline void retina_get_rect(const YoloLetterbox& lb, const float bbox[4], int rect[4]) {
    const int l = trunc_to_int_x86(yolo_map_landmark(lb, 0, bbox[0])), t = trunc_to_int_x86(yolo_map_landmark(lb, 1, bbox[1]));
    const int r = trunc_to_int_x86(yolo_map_landmark(lb, 0, bbox[2])), b = trunc_to_int_x86(yolo_map_landmark(lb, 1, bbox[3]));
    rect[0] = l;
    rect[1] = t;
    rect[2] = (int)((uint32_t)r - (uint32_t)l);
    rect[3] = (int)((uint32_t)b - (uint32_t)t);
}
__host__ __device__ inline void retina_get_rect_adapt_landmark(int input_w, int input_h, int img_w, int img_h,
                                                               const float bbox[4], float lmk[10], int rect[4]) {
    const YoloLetterbox lb = yolo_letterbox(input_w, input_h, img_w, img_h);
    retina_get_rect(lb, bbox, rect);
    for (int i = 0; i < 10; ++i) lmk[i] = yolo_map_landmark(lb, i & 1, lmk[i]);
}

// YOLOP's get_rect (yolop/common.hpp:13-37): box cx, cy, w, h; the letterbox expressions are get_rect's (yolo_letterbox).
// Every statement stores to an int, so a corner is truncated twice: after `bbox[0] - bbox[2] / 2.f` (minus the pad on the
// padded axis, all float) and after its division by the ratio (int / float: a float division).  No clamp; rect =
// {l, t, r - l, b - t}.  Undefined cases as the compiled x86-64 reference behaves: trunc_to_int_x86, and int differences
// that wrap modulo 2^32.
__host__ __device__ inline void yolop_get_rect(const YoloLetterbox& lb, const float bbox[4], int rect[4]) {
    float c[4];  // l, t, r, b
    trunc_rect_corners(lb, bbox, c);
    int v[4];
    for (int k = 0; k < 4; ++k) v[k] = trunc_to_int_x86(f_div((float)trunc_to_int_x86(c[k]), lb.ratio));
    rect[0] = v[0];
    rect[1] = v[1];
    rect[2] = (int)((uint32_t)v[2] - (uint32_t)v[0]);
    rect[3] = (int)((uint32_t)v[3] - (uint32_t)v[1]);
}

// DETR's rectangle (detr/detr.cpp:795-803): box = cx, cy, w, h, normalised.  Each corner is a double expression stored to
// float, `float x1 = (cx - w / 2.0) * img.cols`; then cv::Rect r(x1, y1, x2 - x1, y2 - y1) converts four floats to int, the
// differences taken in float.  Undefined cases as the compiled x86-64 reference behaves: trunc_to_int_x86.  __dsub_rn /
// __dmul_rn on the device, so that nvcc cannot contract the corner into an FMA.
__host__ __device__ inline void detr_get_rect(int img_w, int img_h, const float box[4], int rect[4]) {
    float c[4];  // x1, y1, x2, y2
    for (int k = 0; k < 4; ++k) {
        const int a = k & 1;  // 0: x, 1: y
        const double centre = (double)box[a], half = (double)box[2 + a] / 2.0, size = (double)(a ? img_h : img_w);
#ifdef __CUDA_ARCH__
        c[k] = __double2float_rn(__dmul_rn(k < 2 ? __dsub_rn(centre, half) : __dadd_rn(centre, half), size));
#else
        c[k] = (float)((k < 2 ? centre - half : centre + half) * size);
#endif
    }
    rect[0] = trunc_to_int_x86(c[0]);
    rect[1] = trunc_to_int_x86(c[1]);
    rect[2] = trunc_to_int_x86(f_sub(c[2], c[0]));
    rect[3] = trunc_to_int_x86(f_sub(c[3], c[1]));
}

// UFLD's prepareImage after the resize (ufld/lane_det.cpp:194-221), the value of byte u in plane c (0 = R, 1 = G, 2 = B:
// cvtColor BGR2RGB, then cv::split), with the driver's `static float` mean and std:
//   convertTo(CV_32FC3, 1. / 255.)        s = (float)u * (float)(1. / 255.)
//   (channel - mean[c]) / std[c]          one convertTo(-1, 1 / std, -mean / std): OpenCV 4.x folds the MatExpr
//                                         (MatOp_AddEx), and cvtScale32f casts both coefficients to float and fuses them with
//                                         v_fma: fmaf(s, (float)(1 / std), (float)(-mean / std)), the quotients in double.
// The folding is read from OpenCV's source, not run (DESIGN §4.8); the fused product is pinned against cv2 4.13 on all
// 3 x 256 bytes (tests/test_ufld_cpu.py).
__device__ __forceinline__ float ufld_input_value(int c, uint32_t u) {
    const double mean = (double)(c == 0 ? 0.485f : (c == 1 ? 0.456f : 0.406f));
    const double sd = (double)(c == 0 ? 0.229f : (c == 1 ? 0.224f : 0.225f));
    const float s = __fmul_rn((float)u, (float)(1. / 255.));
    return __fmaf_rn(s, __double2float_rn(__ddiv_rn(1.0, sd)), __double2float_rn(__ddiv_rn(-mean, sd)));
}

// RefineDet's base_transform after the resize (refinedet/refinedet.cpp:822-839), the value of byte u in plane c (0 = R,
// 1 = G, 2 = B): (float)(u * 1.0 - mean) with mean 123, 117, 104, exact in float.
__device__ __forceinline__ float refinedet_input_value(int c, uint32_t u) {
    return __fsub_rn((float)u, c == 0 ? 123.f : (c == 1 ? 117.f : 104.f));
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
