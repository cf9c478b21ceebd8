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

// get_rect: the inverse of the letterbox for a detection box -- yolov8/src/postprocess.cpp:6-36 (TRTX_YOLO_V8: l,t,r,b,
// clamped to the image) and yolov5/src/postprocess.cpp:4-29 (TRTX_YOLO_V5: cx,cy,w,h, not clamped).  Statement by statement:
// the two ratios are double divisions stored to float, the rest is float, round() sees doubles.  Shared by the host
// trtx_get_rect and the segmentation post-process kernels (mask.cu).  Returns false, with rect {0, 0, 0, 0}, where the
// reference's float -> int conversions are undefined (a non-finite box, or rescaled corners outside the int range).
__host__ __device__ inline bool yolo_get_rect(int variant, int net_w, int net_h, int img_w, int img_h, const float bbox[4],
                                              int rect[4]) {
    rect[0] = rect[1] = rect[2] = rect[3] = 0;
#ifdef __CUDA_ARCH__
    const float r_w = __double2float_rn(__ddiv_rn((double)net_w, (double)img_w));
    const float r_h = __double2float_rn(__ddiv_rn((double)net_h, (double)img_h));
#else
    const float r_w = (float)(net_w / (img_w * 1.0));
    const float r_h = (float)(net_h / (img_h * 1.0));
#endif
    const bool by_w = r_h > r_w;  // the width fills the network input: vertical padding
    const float ratio = by_w ? r_w : r_h;
    const float pad = by_w ? f_div(f_sub((float)net_h, f_mul(r_w, (float)img_h)), 2.0f)
                           : f_div(f_sub((float)net_w, f_mul(r_h, (float)img_w)), 2.0f);
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
