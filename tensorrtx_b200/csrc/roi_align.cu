// roi_align.cu -- RoIAlign + MaskRcnnInference for sm_90a (SURVEY 8f rank 2).
// Replaces roiAlign / RoIAlignForward (rcnn/RoiAlign.cu:29-183) and maskRcnnInference / MaskRcnnInferenceKernel
// (rcnn/MaskRcnnInference.cu:8-63), which launch once per image and call cudaDeviceSynchronize() after every launch
// (RoiAlign.cu:178, MaskRcnnInference.cu:59) -- a full-device stall inside enqueue().  Here: one launch for the whole
// batch on the caller's stream, no synchronisation, no allocation.
//
// RoIAlign: a CTA owns one proposal and a chunk of channels.  The sample coordinates of RoIAlign are separable --
// (y_low, y_high, ly, hy, in-range) depends on (ph, iy) only, the x part on (pw, ix) only -- so the CTA tabulates them
// once in shared memory (<= 14*g entries each) instead of recomputing them for each of the 1024 channels; a thread
// then owns one output bin and walks its channels: 4 taps per sample from the L2-resident feature map, and the 196
// outputs of a (proposal, channel) pair are stored contiguously (coalesced).
// Roofline: HBM-write-bound: N*C*P*P*4 bytes per image (803 MB at N=1000, C=1024, P=14).
//
// Arithmetic mirrors the reference kernel statement by statement; where the compiler could contract it more than one way
// (the bilinear sum, bilinear_sum below) the contraction of the reference's own build is written out
// (tests/test_vs_reference_gpu.py compares against the reference kernel).
#include "common.cuh"

namespace trtx {

constexpr int kRoiMaxPooled = 32;   // pooler_resolution
constexpr int kRoiMaxTable = 256;   // pooler_resolution * sampling grid, per axis (larger grids: coordinates on the fly)
constexpr int kRoiChannelsPerCta = 64;

// T: the element type of the feature map and of the output, float or __half.  Proposals are fp32 in both modes (a half holds
// a coordinate up to 1067 to 0.5 px only).  A half tap is widened to float (exact), every sum is the fp32 one, and only the
// finished bin is rounded, once, with __float2half_rn: the half result is half(roi_align_fp32(float(features))) bit for bit.
template <typename T>
struct RoiArgs {
    const float4* rois;  // [B, N]
    const T* feat;       // [B, C, H, W]
    T* out;              // [B, N, C, P, P]
    int N, C, H, W, P, sampling_ratio;
    float spatial_scale;
};

template <typename T>
__device__ __forceinline__ T roi_bin(float v);
template <>
__device__ __forceinline__ float roi_bin<float>(float v) { return v; }
template <>
__device__ __forceinline__ __half roi_bin<__half>(float v) { return __float2half_rn(v); }

struct AxisTap {
    int low, high;  // clamped indices
    float l, h;     // fractions
    int valid;      // 0: the reference's bilinear_interpolate returns 0 for this coordinate
};

// one axis of bilinear_interpolate (RoiAlign.cu:29-69); `size` = height or width
__device__ __forceinline__ AxisTap axis_tap(float y, int size) {
    AxisTap t;
    t.valid = !(y < -1.0 || y > size);
    if (y <= 0) y = 0;
    int y_low = static_cast<int>(y);
    int y_high;
    if (y_low >= size - 1) {
        y_high = y_low = size - 1;
        y = (float)y_low;
    } else {
        y_high = y_low + 1;
    }
    t.low = y_low;
    t.high = y_high;
    t.l = y - y_low;
    t.h = 1. - t.l;
    return t;
}

// :76 `w1 * v1 + w2 * v2 + w3 * v3 + w4 * v4` as the reference's build for sm_90a contracts it: one multiply, then three
// fused multiply-adds in source order.  Left to nvcc, `w1 * v1 + w2 * v2` may fuse either product (for sm_90a it fuses the
// other one here), which moves sums of many samples by a few ulps.
__device__ __forceinline__ float bilinear_sum(float w1, float v1, float w2, float v2, float w3, float v3, float w4, float v4) {
    return __fmaf_rn(w4, v4, __fmaf_rn(w3, v3, __fmaf_rn(w2, v2, __fmul_rn(w1, v1))));
}

// Geometry of one proposal (RoiAlign.cu:104-127 -- "Do not using rounding; this implementation detail is critical")
struct RoiGeom {
    float start_w, start_h, bin_h, bin_w, count;
    int grid_h, grid_w;
    bool tabled;
};

template <typename T>
__device__ __forceinline__ RoiGeom roi_geom(const RoiArgs<T>& a, const float4 roi) {
    RoiGeom q;
    float roi_offset = 0.5f;
    float roi_start_w = roi.x * a.spatial_scale - roi_offset;
    float roi_start_h = roi.y * a.spatial_scale - roi_offset;
    float roi_end_w = roi.z * a.spatial_scale - roi_offset;
    float roi_end_h = roi.w * a.spatial_scale - roi_offset;
    float roi_width = roi_end_w - roi_start_w;
    float roi_height = roi_end_h - roi_start_h;
    q.start_w = roi_start_w;
    q.start_h = roi_start_h;
    q.bin_h = static_cast<float>(roi_height) / static_cast<float>(a.P);
    q.bin_w = static_cast<float>(roi_width) / static_cast<float>(a.P);
    q.grid_h = (a.sampling_ratio > 0) ? a.sampling_ratio : ceil(roi_height / a.P);
    q.grid_w = (a.sampling_ratio > 0) ? a.sampling_ratio : ceil(roi_width / a.P);
    q.count = q.grid_h * q.grid_w;
    q.tabled = q.grid_h > 0 && q.grid_w > 0 && a.P * q.grid_h <= kRoiMaxTable && a.P * q.grid_w <= kRoiMaxTable;
    return q;
}

// the sample coordinates of one axis (RoiAlign.cu:133-139)
__device__ __forceinline__ float roi_sample(float start, float bin, int p, int i, int grid) {
    return start + p * bin + static_cast<float>(i + .5f) * bin / static_cast<float>(grid);
}

// Direct form: taps straight from the (L2-resident) feature map.  One thread per output bin, CU channels per pass.
// `off_y(t)` / `off_x(t)`: how a tabulated tap turns into an offset -- absolute rows of the feature map here.
template <typename T>
__device__ __forceinline__ void roi_align_direct(const RoiArgs<T>& a, const RoiGeom& q, const AxisTap* s_y, const AxisTap* s_x, int n, int b,
                                                 int c_begin, int c_end) {
    const int P = a.P, PP = P * P;
    // thread = (bin, channel lane): bins are the fast index, so a warp writes consecutive floats
    const int nsub = max(1, (int)blockDim.x / PP);
    const int bin = threadIdx.x % PP, csub = threadIdx.x / PP;
    if (csub >= nsub) return;
    const int ph = bin / P, pw = bin - ph * P;
    const size_t plane = (size_t)a.H * a.W;
    const T* fb = a.feat + (size_t)b * a.C * plane;
    T* ob = a.out + (((size_t)b * a.N + n) * a.C) * PP + bin;
    constexpr int CU = 4;  // channels per thread and pass: the taps (shared-memory table reads, weights) are channel-independent
    for (int c0 = c_begin + csub * CU; c0 < c_end; c0 += nsub * CU) {
        float output_val[CU];
#pragma unroll
        for (int k = 0; k < CU; ++k) output_val[k] = 0.f;
        const T* fm = fb + (size_t)c0 * plane;
        const int nch = min(CU, c_end - c0);
        for (int iy = 0; iy < q.grid_h; iy++) {
            // degenerate or huge sampling grids: coordinates on the fly, as the reference does
            const AxisTap ty = q.tabled ? s_y[ph * q.grid_h + iy] : axis_tap(roi_sample(q.start_h, q.bin_h, ph, iy, q.grid_h), a.H);
            for (int ix = 0; ix < q.grid_w; ix++) {
                const AxisTap tx = q.tabled ? s_x[pw * q.grid_w + ix] : axis_tap(roi_sample(q.start_w, q.bin_w, pw, ix, q.grid_w), a.W);
                if (!(ty.valid && tx.valid)) continue;  // bilinear_interpolate returns 0: `output_val += 0`
                const float ly = ty.l, hy = ty.h, lx = tx.l, hx = tx.h;
                const float w1 = hy * hx, w2 = hy * lx, w3 = ly * hx, w4 = ly * lx;
                const int o1 = ty.low * a.W + tx.low, o2 = ty.low * a.W + tx.high, o3 = ty.high * a.W + tx.low,
                          o4 = ty.high * a.W + tx.high;
#pragma unroll
                for (int k = 0; k < CU; ++k) {
                    if (k < nch) {
                        const T* f = fm + (size_t)k * plane;
                        const float v1 = Elem<T>::ld1_cached(f + o1), v2 = Elem<T>::ld1_cached(f + o2), v3 = Elem<T>::ld1_cached(f + o3),
                                    v4 = Elem<T>::ld1_cached(f + o4);
                        const float val = bilinear_sum(w1, v1, w2, v2, w3, v3, w4, v4);  // :76
                        output_val[k] += val;
                    }
                }
            }
        }
#pragma unroll
        for (int k = 0; k < CU; ++k)
            if (k < nch) ob[(size_t)(c0 + k) * PP] = roi_bin<T>(output_val[k] / q.count);  // :147 (NaN for a degenerate proposal, like the reference)
    }
}

template <typename T>
__device__ __forceinline__ void roi_build_tables(const RoiArgs<T>& a, const RoiGeom& q, AxisTap* s_y, AxisTap* s_x) {
    for (int i = threadIdx.x; i < a.P * q.grid_h; i += blockDim.x) {
        const int ph = i / q.grid_h, iy = i - ph * q.grid_h;
        s_y[i] = axis_tap(roi_sample(q.start_h, q.bin_h, ph, iy, q.grid_h), a.H);
    }
    for (int i = threadIdx.x; i < a.P * q.grid_w; i += blockDim.x) {
        const int pw = i / q.grid_w, ix = i - pw * q.grid_w;
        s_x[i] = axis_tap(roi_sample(q.start_w, q.bin_w, pw, ix, q.grid_w), a.W);
    }
}

// round-1 kernel: every tap is a global load (the shapes the window kernel does not cover)
template <typename T>
__global__ void __launch_bounds__(256) roi_align_kernel(const __grid_constant__ RoiArgs<T> a) {
    __shared__ AxisTap s_y[kRoiMaxTable], s_x[kRoiMaxTable];
    const int n = blockIdx.x, b = blockIdx.z;
    const int c_begin = blockIdx.y * kRoiChannelsPerCta, c_end = min(a.C, c_begin + kRoiChannelsPerCta);
    const RoiGeom q = roi_geom(a, a.rois[(size_t)b * a.N + n]);
    if (q.tabled) roi_build_tables(a, q, s_y, s_x);
    __syncthreads();
    roi_align_direct(a, q, s_y, s_x, n, b, c_begin, c_end);
}

// --------------------------------------------------------------------------------------------
// Window kernel (round 2, default): the taps of a proposal touch only the feature-map window
// [y0..y1] x [x0..x1] that its sample coordinates span -- 169 cells for a 13x13-cell proposal against 196 output bins that
// each read 4..16 of them.  The CTA (one proposal, 64 channels) copies that window ONCE into shared memory, CHANNEL-MINOR
// (cell-major rows of `pitch` floats), with cp.async (4 bytes per element, every copy of a pass in flight together: the L2
// round trip is paid once per pass instead of once per dependent tap), and then takes every tap from shared memory: one
// LDS.128 fetches a tap for FOUR channels, the offsets and weights of a sample are read once per 16 channels.  A thread
// owns one output bin; per channel the samples are accumulated in the reference's order with the reference's expression,
// so the results stay bit-identical (test_roi_align_and_mask_rcnn_inference_vs_reference_functions).
//   fill: a warp item = 4 channels x 8 consecutive cells of a window row: four 32-byte global segments, 32 distinct banks;
//   taps: pitch = channels + 4 floats (pitch / 4 odd), so the 8 lanes of a quarter-warp -- neighbouring bins, i.e.
//         neighbouring or identical cells -- hit distinct 16-byte bank groups or broadcast.
// Shared memory: 2 tables (10 KB) + kRoiWindowBytes of window.
//
// Halves (T = __half): the window holds halves, channel-minor, so the same 64 KB hold twice the (cell, channel) items -- a
// proposal whose window does not fit with 64 channels takes half the passes -- and one LDS.128 fetches a tap for EIGHT
// channels; a thread takes 16 channels per tap round (two LDS.128 per tap), so the offsets and weights of a sample are
// read once per 16 channels.
//   fill: cp.async moves 4 bytes at least and the two halves of a window word come from two channel planes, so the fill
//         goes through registers: a warp item = 4 channel PAIRS x 8 consecutive cells; a lane loads its pair's two halves
//         (2-byte read-only loads, 16 of them in flight per lane) and stores them as one 32-bit word: 32 distinct banks.
//   taps: pitch = channels + 8 halves with channels % 16 == 0 (pitch bytes / 16 odd), the same quarter-warp argument.
//   stores: one 2-byte element per bin and channel; a thread row writes the 28 contiguous bytes of a row of 14 bins.
// --------------------------------------------------------------------------------------------
constexpr int kRoiWindowFloats = 16384;  // 64 KB
constexpr int kRoiWindowBytes = kRoiWindowFloats * (int)sizeof(float);
constexpr int kRoiWindowThreads = 224;   // 7 warps: 196 bins of a 14x14 pooler + 28 idle lanes in the tap phase

// The window layout of an element type.  kCU: channels per thread and tap round.  kGroup: the multiple a pass' channel count
// must be for pitch = channels + kPad elements to keep pitch bytes / 16 odd.  kMin: channels per pass (= pitch, 16 bytes per
// cell) when not even kGroup channels of the window fit -- 4096 cells at most, a whole 50 x 67 map: 3350.
template <typename T>
struct RoiWin;
template <>
struct RoiWin<float> {
    static constexpr int kCU = 8, kGroup = 8, kPad = 4, kMin = 4;
};
template <>
struct RoiWin<__half> {
    static constexpr int kCU = 16, kGroup = 16, kPad = 8, kMin = 8;
};

// one axis of a sample, window-relative: BYTE offsets of the low / high row (or column) in the window, the two fractions;
// lo < 0: the reference's bilinear_interpolate returns 0 for this coordinate
struct __align__(16) WinTap {
    int lo, hi;
    float l, h;
};

__device__ __forceinline__ void cp_async_4(void* smem_dst, const void* gmem_src) {
    const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(d), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_4s(uint32_t smem_dst, const void* gmem_src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_dst), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// 16 bytes of a window row -> the taps of its channels, widened to float
__device__ __forceinline__ void roi_tap16(const char* p, float (&v)[4]) {
    const float4 a = *reinterpret_cast<const float4*>(p);
    v[0] = a.x, v[1] = a.y, v[2] = a.z, v[3] = a.w;
}
__device__ __forceinline__ void roi_tap16(const char* p, float (&v)[8]) {
    const uint4 a = *reinterpret_cast<const uint4*>(p);
    const float2 f0 = __half22float2(*reinterpret_cast<const __half2*>(&a.x)), f1 = __half22float2(*reinterpret_cast<const __half2*>(&a.y));
    const float2 f2 = __half22float2(*reinterpret_cast<const __half2*>(&a.z)), f3 = __half22float2(*reinterpret_cast<const __half2*>(&a.w));
    v[0] = f0.x, v[1] = f0.y, v[2] = f1.x, v[3] = f1.y, v[4] = f2.x, v[5] = f2.y, v[6] = f3.x, v[7] = f3.y;
}

// POW2: the sample count is a power of two (1 for proposals of up to 14 x 14 cells), so `output_val / count` (:147) equals
// `output_val * (1 / count)` bit for bit (scaling by 2^-k is exact, or rounds the same real number once when it underflows)
template <typename T, bool FULL, bool POW2>
__device__ __forceinline__ void roi_window_taps(const char* win, const WinTap* ty_row, const WinTap* tx_row, int grid_h, int grid_w, int nch,
                                                float count, T* ob, const int PP) {
    constexpr int CU = RoiWin<T>::kCU, V = 16 / (int)sizeof(T);  // V: channels per 16-byte load
    float output_val[CU];
#pragma unroll
    for (int k = 0; k < CU; ++k) output_val[k] = 0.f;
    for (int iy = 0; iy < grid_h; iy++) {
        const WinTap ty = ty_row[iy];
        if (ty.lo < 0) continue;  // bilinear_interpolate returns 0: `output_val += 0`
        for (int ix = 0; ix < grid_w; ix++) {
            const WinTap tx = tx_row[ix];
            if (tx.lo < 0) continue;
            const float ly = ty.l, hy = ty.h, lx = tx.l, hx = tx.h;
            const float w1 = hy * hx, w2 = hy * lx, w3 = ly * hx, w4 = ly * lx;
            const char *p1 = win + (ty.lo + tx.lo), *p2 = win + (ty.lo + tx.hi), *p3 = win + (ty.hi + tx.lo), *p4 = win + (ty.hi + tx.hi);
#pragma unroll
            for (int g = 0; g < CU / V; ++g) {
                if (FULL || V * g < nch) {
                    float a1[V], a2[V], a3[V], a4[V];
                    roi_tap16(p1 + 16 * g, a1);
                    roi_tap16(p2 + 16 * g, a2);
                    roi_tap16(p3 + 16 * g, a3);
                    roi_tap16(p4 + 16 * g, a4);
#pragma unroll
                    for (int j = 0; j < V; ++j) {
                        const float v1 = a1[j], v2 = a2[j], v3 = a3[j], v4 = a4[j];
                        const float val = bilinear_sum(w1, v1, w2, v2, w3, v3, w4, v4);  // :76
                        output_val[V * g + j] += val;
                    }
                }
            }
        }
    }
#pragma unroll
    for (int k = 0; k < CU; ++k)
        if (FULL || k < nch) ob[(size_t)k * PP] = roi_bin<T>(POW2 ? output_val[k] * (1.0f / count) : output_val[k] / count);  // :147
}

// PT: the pooler resolution when it is the 14 of the Faster / Mask R-CNN heads (rcnn.cpp:44 POOLER_RESOLUTION) -- store offsets
// become immediates and a thread row of 16 owns one row of 14 bins, so that the 8 lanes of a quarter-warp read neighbouring
// cells of ONE window row (no shared-memory bank conflicts between bins of different rows); 0: any resolution, bin = thread.
template <int PT, typename T>
__global__ void __launch_bounds__(kRoiWindowThreads, 3) roi_align_window_kernel(const __grid_constant__ RoiArgs<T> a) {
    using Win = RoiWin<T>;
    constexpr int ES = (int)sizeof(T);
    __shared__ AxisTap s_y[kRoiMaxTable], s_x[kRoiMaxTable];   // 10 KB; rewritten in place as WinTap (16 of the 20 bytes)
    __shared__ int s_box[4];  // y0, y1, x0, x1 of the window (over the valid taps)
    extern __shared__ __align__(16) unsigned char s_win_bytes[];
    T* s_win = reinterpret_cast<T*>(s_win_bytes);
    const int n = blockIdx.x, b = blockIdx.z;
    const int c_begin = blockIdx.y * kRoiChannelsPerCta, c_end = min(a.C, c_begin + kRoiChannelsPerCta);
    const int P = PT ? PT : a.P, PP = P * P;
    const RoiGeom q = roi_geom(a, a.rois[(size_t)b * a.N + n]);
    if (!q.tabled) {  // block-uniform
        roi_align_direct(a, q, s_y, s_x, n, b, c_begin, c_end);
        return;
    }
    if (threadIdx.x == 0) {
        s_box[0] = a.H;
        s_box[1] = -1;
        s_box[2] = a.W;
        s_box[3] = -1;
    }
    roi_build_tables(a, q, s_y, s_x);
    __syncthreads();
    const int ny = P * q.grid_h, nx = P * q.grid_w;
    {   // window = hull of the valid taps (a handful of shared-memory atomics per CTA)
        int lo = a.H, hi = -1;
        for (int i = threadIdx.x; i < ny; i += blockDim.x)
            if (s_y[i].valid) lo = min(lo, s_y[i].low), hi = max(hi, s_y[i].high);
        if (hi >= 0) atomicMin(&s_box[0], lo), atomicMax(&s_box[1], hi);
        lo = a.W, hi = -1;
        for (int i = threadIdx.x; i < nx; i += blockDim.x)
            if (s_x[i].valid) lo = min(lo, s_x[i].low), hi = max(hi, s_x[i].high);
        if (hi >= 0) atomicMin(&s_box[2], lo), atomicMax(&s_box[3], hi);
    }
    __syncthreads();
    const int y0 = s_box[0], y1 = s_box[1], x0 = s_box[2], x1 = s_box[3];
    int ph, pw;
    bool has_bin;
    if (PT) {  // 16 threads per row of bins (kRoiWindowThreads = 14 * 16)
        ph = threadIdx.x >> 4, pw = threadIdx.x & 15;
        has_bin = pw < PT;
        if (!has_bin) pw = 0;
    } else {
        has_bin = (int)threadIdx.x < PP;
        ph = has_bin ? threadIdx.x / P : 0, pw = has_bin ? threadIdx.x - ph * P : 0;
    }
    T* ob = a.out + (((size_t)b * a.N + n) * a.C) * PP + (ph * P + pw);
    if (y1 < 0 || x1 < 0) {  // every sample is outside the map: the reference adds zeros
        if (has_bin)
            for (int c = c_begin; c < c_end; ++c) ob[(size_t)c * PP] = roi_bin<T>(0.f / q.count);
        return;
    }
    const int wh = y1 - y0 + 1, ww = x1 - x0 + 1, cells = wh * ww;
    // channels per pass: as many as fit, a multiple of kGroup (pitch = channels + kPad elements, pitch bytes / 16 odd) -- or
    // kMin with pitch kMin for the largest windows (floats: more than 20480 / 12 cells)
    int cpass = min(kRoiChannelsPerCta, (kRoiWindowBytes / ES / cells - Win::kPad) & ~(Win::kGroup - 1));
    int pitch = cpass + Win::kPad;
    if (cpass < Win::kGroup) cpass = Win::kMin, pitch = Win::kMin;
    // tables become window-relative byte offsets (AxisTap -> WinTap in place: each thread converts its own entries)
    WinTap* w_y = reinterpret_cast<WinTap*>(s_y);
    WinTap* w_x = reinterpret_cast<WinTap*>(s_x);
    {   // P * grid <= 256 entries per axis, 224 threads: at most 2 each (slots tid and tid + 224)
        const int i0 = threadIdx.x, i1 = threadIdx.x + kRoiWindowThreads;
        AxisTap ty0, ty1, tx0, tx1;
        if (i0 < ny) ty0 = s_y[i0];
        if (i1 < ny) ty1 = s_y[i1];
        if (i0 < nx) tx0 = s_x[i0];
        if (i1 < nx) tx1 = s_x[i1];
        __syncthreads();
        const int ymul = ww * pitch * ES, xmul = pitch * ES;
        auto conv = [](const AxisTap& t, int origin, int mul) {
            WinTap w;
            w.lo = t.valid ? (t.low - origin) * mul : -1;
            w.hi = (t.high - origin) * mul;
            w.l = t.l, w.h = t.h;
            return w;
        };
        if (i0 < ny) w_y[i0] = conv(ty0, y0, ymul);
        if (i1 < ny) w_y[i1] = conv(ty1, y0, ymul);
        if (i0 < nx) w_x[i0] = conv(tx0, x0, xmul);
        if (i1 < nx) w_x[i1] = conv(tx1, x0, xmul);
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const size_t plane = (size_t)a.H * a.W;
    const unsigned ngroups = (cells + 7) >> 3, m_ww = (65536 + ww - 1) / ww;
    const T* fwin = a.feat + (size_t)b * a.C * plane + (size_t)y0 * a.W + x0;
    const int fx = lane & 7, fc = lane >> 3;
    const int nsamp = q.grid_h * q.grid_w;
    const bool pow2 = (nsamp & (nsamp - 1)) == 0;
    for (int cb = c_begin; cb < c_end; cb += cpass) {
        const int nc = min(cpass, c_end - cb);
        __syncthreads();  // tables rewritten (first pass) / previous pass' taps done
        if constexpr (ES == 4) {
            // Fill.  An item = (cell, channel % 4): the lanes of a warp are 4 channels x 8 consecutive cells (four 32-byte global
            // segments unless the 8 cells wrap to the next window row; 32 distinct banks).  The item's source and destination are
            // worked out once, then one cp.async per channel quad with both addresses stepping by constants.
            const int plane4 = 4 * a.H * a.W;
            const int nq = nc >> 2, ntail = nc & 3;
            const T* fsrc = fwin + (size_t)(cb + fc) * plane;
            const uint32_t fdst = (uint32_t)__cvta_generic_to_shared(s_win + fc);
            for (unsigned e = threadIdx.x; e < ngroups * 32; e += kRoiWindowThreads) {
                const unsigned cell = (e >> 5) * 8 + fx;
                if (cell >= (unsigned)cells) continue;
                const unsigned y = cells * ww <= 65536 ? (cell * m_ww) >> 16 : cell / ww, x = cell - y * ww;  // exact: cell * (m_ww * ww - 2^16) < cells * ww <= 2^16
                const T* src = fsrc + (y * a.W + x);
                uint32_t dst = fdst + cell * pitch * 4;
#pragma unroll 4
                for (int cq = 0; cq < nq; ++cq) {
                    cp_async_4s(dst, src);
                    dst += 16;
                    src += plane4;
                }
                if (fc < ntail) cp_async_4s(dst, src);
            }
            cp_async_wait_all();
        } else {
            // Fill, halves.  An item = (cell, channel pair % 4): the lanes of a warp are 4 channel pairs x 8 consecutive cells;
            // one 32-bit store per 8 channels, both addresses stepping by constants (nc % 8 == 0: the dispatcher's rule).
            const int plane8 = 8 * a.H * a.W;
            const int n8 = nc >> 3;
            const unsigned short* fsrc = reinterpret_cast<const unsigned short*>(fwin + (size_t)(cb + 2 * fc) * plane);
            char* fdst = reinterpret_cast<char*>(s_win + 2 * fc);
            for (unsigned e = threadIdx.x; e < ngroups * 32; e += kRoiWindowThreads) {
                const unsigned cell = (e >> 5) * 8 + fx;
                if (cell >= (unsigned)cells) continue;
                const unsigned y = cells * ww <= 65536 ? (cell * m_ww) >> 16 : cell / ww, x = cell - y * ww;
                const unsigned short* src = fsrc + (y * a.W + x);
                char* dst = fdst + cell * pitch * 2;
#pragma unroll 8
                for (int cq = 0; cq < n8; ++cq) {
                    const uint32_t lo = __ldg(src), hi = __ldg(src + plane);
                    *reinterpret_cast<uint32_t*>(dst) = lo | (hi << 16);
                    dst += 16;
                    src += plane8;
                }
            }
        }
        __syncthreads();
        if (!has_bin) continue;
        for (int k0 = 0; k0 < nc; k0 += Win::kCU) {
            const int nch = nc - k0;
            const char* win = reinterpret_cast<const char*>(s_win + k0);
            T* o = ob + (size_t)(cb + k0) * PP;
            if (nch >= Win::kCU && pow2)
                roi_window_taps<T, true, true>(win, w_y + ph * q.grid_h, w_x + pw * q.grid_w, q.grid_h, q.grid_w, Win::kCU, q.count, o, PP);
            else if (nch >= Win::kCU)
                roi_window_taps<T, true, false>(win, w_y + ph * q.grid_h, w_x + pw * q.grid_w, q.grid_h, q.grid_w, Win::kCU, q.count, o, PP);
            else
                roi_window_taps<T, false, false>(win, w_y + ph * q.grid_h, w_x + pw * q.grid_w, q.grid_h, q.grid_w, nch, q.count, o, PP);
        }
    }
}

// MaskRcnnInferenceKernel (MaskRcnnInference.cu:8-33): out[d] = sigmoid(masks[d, class(d)]) -- one thread per OUTPUT
// element instead of one per (detection, class, pixel); detections whose class index is outside [0, num_classes)
// are left unwritten, as in the reference.  T: the masks' element type; a half is widened (exact), the output is fp32.
template <typename T>
__global__ void mask_rcnn_inference_kernel(const float* __restrict__ indices, const T* __restrict__ masks,
                                           float* __restrict__ out, int total_dets, int num_classes, int ss) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)total_dets * ss) return;
    const int ind = (int)(i / ss), px = (int)(i - (size_t)ind * ss);
    const int ind_class = indices[ind];  // float -> int, :19
    if (ind_class < 0 || ind_class >= num_classes) return;
    const float maskVal = masks[((size_t)ind * num_classes + ind_class) * ss + px];
    out[i] = logist(maskVal);
}

template <typename T>
static int roi_align_launch(int batch, const float* rois_dev, const void* features_dev, void* out_dev, int pooler_resolution,
                            float spatial_scale, int sampling_ratio, int num_proposals, int out_channels, int feature_h,
                            int feature_w, trtx_stream_t stream) {
    RoiArgs<T> a;
    a.rois = reinterpret_cast<const float4*>(rois_dev);
    a.feat = static_cast<const T*>(features_dev);
    a.out = static_cast<T*>(out_dev);
    a.N = num_proposals;
    a.C = out_channels;
    a.H = feature_h;
    a.W = feature_w;
    a.P = pooler_resolution;
    a.sampling_ratio = sampling_ratio;
    a.spatial_scale = spatial_scale;
    dim3 grid(num_proposals, (out_channels + kRoiChannelsPerCta - 1) / kRoiChannelsPerCta, batch);
    if (grid.y > 65535) return TRTX_ERR_UNSUPPORTED;
    // the window kernel is built for the 14 x 14 pooler of the reference's heads (rcnn.cpp:43), takes 16 bytes of channels
    // per shared-memory load (4 floats, 8 halves) and needs a map whose window fits its shared memory with 16 bytes per
    // cell; every other shape (other poolers, other channel counts, larger maps) takes the direct kernel
    constexpr int kChannelMultiple = 16 / (int)sizeof(T);
    const bool window_ok = pooler_resolution == 14 && out_channels % kChannelMultiple == 0 &&
                           (long long)feature_h * feature_w <= kRoiWindowFloats / 4;  // 16 bytes per cell in both modes
    if (!window_ok) {
        roi_align_kernel<T><<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(a);
        return check_launch();
    }
    constexpr int smem = kRoiWindowBytes;
    auto kernel = roi_align_window_kernel<14, T>;
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);  // idempotent
    if (e != cudaSuccess) {
        g_last_cuda_error = (int)e;
        return TRTX_ERR_CUDA;
    }
    kernel<<<grid, kRoiWindowThreads, smem, static_cast<cudaStream_t>(stream)>>>(a);
    return check_launch();
}

static bool aligned_to(const void* p, size_t n) { return reinterpret_cast<uintptr_t>(p) % n == 0; }

}  // namespace trtx

using namespace trtx;

extern "C" {

TRTX_API int trtx_roi_align_typed(int dtype, int batch, const float* rois_dev, const void* features_dev, void* out_dev,
                                  int pooler_resolution, float spatial_scale, int sampling_ratio, int num_proposals,
                                  int out_channels, int feature_h, int feature_w, trtx_stream_t stream) {
    if (dtype != TRTX_F32 && dtype != TRTX_F16) return TRTX_ERR_INVALID;
    if (batch <= 0 || !rois_dev || !features_dev || !out_dev) return TRTX_ERR_INVALID;
    if (pooler_resolution <= 0 || num_proposals <= 0 || out_channels <= 0 || feature_h <= 0 || feature_w <= 0) return TRTX_ERR_INVALID;
    // a proposal is one 16-byte load; features and bins are read and written element by element
    const size_t elem = dtype == TRTX_F16 ? sizeof(__half) : sizeof(float);
    if (!aligned_to(rois_dev, 16) || !aligned_to(features_dev, elem) || !aligned_to(out_dev, elem)) return TRTX_ERR_INVALID;
    if (pooler_resolution > kRoiMaxPooled || pooler_resolution * pooler_resolution > 256) return TRTX_ERR_UNSUPPORTED;
    if (batch > 65535) return TRTX_ERR_UNSUPPORTED;
    if (dtype == TRTX_F16)
        return roi_align_launch<__half>(batch, rois_dev, features_dev, out_dev, pooler_resolution, spatial_scale, sampling_ratio,
                                        num_proposals, out_channels, feature_h, feature_w, stream);
    return roi_align_launch<float>(batch, rois_dev, features_dev, out_dev, pooler_resolution, spatial_scale, sampling_ratio,
                                   num_proposals, out_channels, feature_h, feature_w, stream);
}

TRTX_API int trtx_roi_align(int batch, const float* rois_dev, const float* features_dev, float* out_dev, int pooler_resolution,
                            float spatial_scale, int sampling_ratio, int num_proposals, int out_channels, int feature_h,
                            int feature_w, trtx_stream_t stream) {
    return trtx_roi_align_typed(TRTX_F32, batch, rois_dev, features_dev, out_dev, pooler_resolution, spatial_scale, sampling_ratio,
                                num_proposals, out_channels, feature_h, feature_w, stream);
}

TRTX_API int trtx_mask_rcnn_inference_typed(int in_dtype, int batch, const float* indices_dev, const void* masks_dev, float* out_dev,
                                            int detections_per_im, int output_size, int num_classes, trtx_stream_t stream) {
    if (in_dtype != TRTX_F32 && in_dtype != TRTX_F16) return TRTX_ERR_INVALID;
    if (batch <= 0 || !indices_dev || !masks_dev || !out_dev) return TRTX_ERR_INVALID;
    if (detections_per_im <= 0 || output_size <= 0 || num_classes <= 0) return TRTX_ERR_INVALID;
    if (!aligned_to(indices_dev, sizeof(float)) || !aligned_to(out_dev, sizeof(float)) ||
        !aligned_to(masks_dev, in_dtype == TRTX_F16 ? sizeof(__half) : sizeof(float)))
        return TRTX_ERR_INVALID;
    const int ss = output_size * output_size;
    const long long total = (long long)batch * detections_per_im * ss;
    const long long blocks = (total + 255) / 256;
    if (blocks > 0x7fffffffLL) return TRTX_ERR_UNSUPPORTED;
    if (in_dtype == TRTX_F16)
        mask_rcnn_inference_kernel<__half><<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
            indices_dev, static_cast<const __half*>(masks_dev), out_dev, batch * detections_per_im, num_classes, ss);
    else
        mask_rcnn_inference_kernel<float><<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
            indices_dev, static_cast<const float*>(masks_dev), out_dev, batch * detections_per_im, num_classes, ss);
    return check_launch();
}

TRTX_API int trtx_mask_rcnn_inference(int batch, const float* indices_dev, const float* masks_dev, float* out_dev,
                                      int detections_per_im, int output_size, int num_classes, trtx_stream_t stream) {
    return trtx_mask_rcnn_inference_typed(TRTX_F32, batch, indices_dev, masks_dev, out_dev, detections_per_im, output_size,
                                          num_classes, stream);
}

}  // extern "C"
