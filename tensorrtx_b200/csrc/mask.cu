// mask.cu -- instance masks of the segmentation models for sm_90a (SURVEY 8f rank 1).
// Replaces the HOST function process_mask(): yolov8/yolov8_seg.cpp:17-60 (the same body in yolov5/src/postprocess.cpp:
// 94-125, yolo11/12 seg drivers), which runs on one CPU core after a D2H copy of the 32 x 160 x 160 prototype tensor:
//     rect   = get_downscale_rect(bbox, 4)
//     m[y,x] = sigmoid(sum_j coeff[j] * proto[j, y, x])        for (x, y) in rect, 0 elsewhere       (160 x 160)
//     mask   = cv::resize(m, 640 x 640)                        (bilinear, INTER_LINEAR)
// Here: ONE fused kernel for all kept detections of the batch.  A CTA owns a 16 x 16 tile of the low-resolution mask of
// one detection: it evaluates the 18 x 18 sigmoid(dot) values the tile's bilinear footprint needs into shared memory
// (tiles that do not touch the detection's rectangle skip the prototype reads entirely and only store zeros), then
// writes its 64 x 64 output pixels with 128-bit stores.  The low-resolution mask never goes to HBM.
//
// Roofline: HBM-bound on the mask WRITES: net_w*net_h*4 B per detection (1.6 MB at 640^2) against
// 32*(rect area)*4 B of prototype reads (L2-resident across the detections of an image).
//
// Arithmetic: the dot product accumulates j = 0..31 in order with separate multiply and add (the host code is built
// without FMA contraction), sigmoid is 1/(1+expf(-e)) (CUDA expf vs glibc expf: <= 2 ulp); the resize follows OpenCV's
// float bilinear kernel: fx = (dx + 0.5) * (src/dst) - 0.5, sx = floor(fx) clamped to [0, src-1] (fraction 0 when
// clamped), horizontal pass then vertical pass, every product and sum rounded to float.
//
// Also here: scale_mask of the yolov8 seg driver, and the Mask R-CNN post-process of rcnn/rcnn.cpp:516-550 (box rescale to
// the original image, mask paste into u8 canvases), which reuses the same resize taps.
#include "common.cuh"

namespace trtx {

constexpr int kMaskTile = 16;                // low-resolution cells per CTA edge
constexpr int kMaskHalo = kMaskTile + 2;     // + one cell on each side for the bilinear taps
constexpr int kMaxCoeffs = 64;
constexpr int kMaxFrames = 64;               // frames per launch of the per-frame entries (launch-parameter arrays)

struct MaskArgs {
    const float* proto;  // [B, nm, mh, mw]
    const float* dets;   // [B, 1 + max_rows * row_floats]
    float* out;          // [B, max_masks, net_h, net_w]
    int max_rows, row_floats, coeff_offset;
    int variant, nm, mw, mh, net_w, net_h, max_masks;
};

// get_downscale_rect: yolov8_seg.cpp:17-34 (bbox used as x, y, w, h; clamped to the network input; int() truncation),
// yolov5/src/postprocess.cpp:94-104 (cx, cy, w, h; round()).  The loops of process_mask are additionally clamped to
// the mask here (the reference would write out of bounds for a v5 box that leaves the image).
__device__ __forceinline__ void downscale_rect(int variant, const float* bbox, int net_w, int net_h, int& rx, int& ry,
                                               int& rw, int& rh) {
    float left, top, right, bottom;
    if (variant == TRTX_YOLO_V8) {
        left = bbox[0];
        top = bbox[1];
        right = __fadd_rn(bbox[0], bbox[2]);
        bottom = __fadd_rn(bbox[1], bbox[3]);
        left = left < 0 ? 0 : left;
        top = top < 0 ? 0 : top;
        right = right > net_w ? net_w : right;
        bottom = bottom > net_h ? net_h : bottom;
        left = __fdiv_rn(left, 4.0f);
        top = __fdiv_rn(top, 4.0f);
        right = __fdiv_rn(right, 4.0f);
        bottom = __fdiv_rn(bottom, 4.0f);
        rx = (int)left;
        ry = (int)top;
        rw = (int)__fsub_rn(right, left);
        rh = (int)__fsub_rn(bottom, top);
    } else {
        left = __fsub_rn(bbox[0], __fdiv_rn(bbox[2], 2.0f));
        top = __fsub_rn(bbox[1], __fdiv_rn(bbox[3], 2.0f));
        right = __fadd_rn(bbox[0], __fdiv_rn(bbox[2], 2.0f));
        bottom = __fadd_rn(bbox[1], __fdiv_rn(bbox[3], 2.0f));
        left = __fdiv_rn(left, 4.0f);
        top = __fdiv_rn(top, 4.0f);
        right = __fdiv_rn(right, 4.0f);
        bottom = __fdiv_rn(bottom, 4.0f);
        rx = (int)round((double)left);
        ry = (int)round((double)top);
        rw = (int)round((double)__fsub_rn(right, left));
        rh = (int)round((double)__fsub_rn(bottom, top));
    }
}

// OpenCV bilinear source coordinate for destination index d: (first tap, fraction)
__device__ __forceinline__ void resize_tap(int d, double scale, int src, int& s0, float& f) {
    float fx = (float)(((double)d + 0.5) * scale - 0.5);
    int sx = (int)floorf(fx);
    fx -= (float)sx;
    if (sx < 0) {
        fx = 0.0f;
        sx = 0;
    }
    if (sx >= src - 1) {
        fx = 0.0f;
        sx = src - 1;
    }
    s0 = sx;
    f = fx;
}

// OpenCV's float bilinear blend of the taps v00 v01 (upper row) and v10 v11 (lower row): HResizeLinear with the weights
// a0, a1, then VResizeLinear with b0, b1, every product and sum rounded to float.
__device__ __forceinline__ float bilinear(float v00, float v01, float v10, float v11, float a0, float a1, float b0, float b1) {
    const float h0 = __fadd_rn(__fmul_rn(v00, a0), __fmul_rn(v01, a1));  // HResizeLinear
    const float h1 = __fadd_rn(__fmul_rn(v10, a0), __fmul_rn(v11, a1));
    return __fadd_rn(__fmul_rn(h0, b0), __fmul_rn(h1, b1));             // VResizeLinear
}

// Bytes x0 .. x0 + 15 of a u8 canvas row (w[k]: bytes 4k .. 4k + 3): one 16-byte store when whole and aligned, else byte
// by byte up to img_w (odd width, pitch or base; the last chunk of a row), so a pitch byte is never written.
__device__ __forceinline__ void store_canvas_chunk(uint8_t* dst, const uint32_t w[4], int x0, int img_w) {
    if (x0 + 16 <= img_w && (reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
        *reinterpret_cast<uint4*>(dst) = make_uint4(w[0], w[1], w[2], w[3]);
    } else {
#pragma unroll
        for (int j = 0; j < 16; ++j)
            if (x0 + j < img_w) dst[j] = (uint8_t)(w[j >> 2] >> (8 * (j & 3)));
    }
}

// The frame owning this CTA in a flat grid over frames: the last j < n with first_cta[j] <= blockIdx.x (ascending, [0] = 0).
__device__ __forceinline__ int frame_of_cta(const int* first_cta, int n) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (first_cta[mid] <= (int)blockIdx.x) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

__global__ void __launch_bounds__(256) process_mask_kernel(const __grid_constant__ MaskArgs a) {
    __shared__ float s_m[kMaskHalo][kMaskHalo + 1];
    __shared__ float s_coeff[kMaxCoeffs];
    const int b = blockIdx.z / a.max_masks, m = blockIdx.z - b * a.max_masks;
    const float* img = a.dets + (size_t)b * (1 + (size_t)a.max_rows * a.row_floats);
    const int count = min(max((int)img[0], 0), min(a.max_rows, a.max_masks));
    if (m >= count) return;  // slots past the image's detections are left untouched
    const float* det = img + 1 + (size_t)m * a.row_floats;
    int rx, ry, rw, rh;
    downscale_rect(a.variant, det, a.net_w, a.net_h, rx, ry, rw, rh);
    const int x_lo = max(rx, 0), x_hi = min(rx + rw, a.mw), y_lo = max(ry, 0), y_hi = min(ry + rh, a.mh);
    const int cx0 = blockIdx.x * kMaskTile - 1, cy0 = blockIdx.y * kMaskTile - 1;  // first halo cell
    const int tid = threadIdx.x;
    const bool touches = x_lo < x_hi && y_lo < y_hi && cx0 < x_hi && cx0 + kMaskHalo > x_lo && cy0 < y_hi && cy0 + kMaskHalo > y_lo;
    if (touches) {
        if (tid < a.nm) s_coeff[tid] = det[a.coeff_offset + tid];
        __syncthreads();
        const size_t plane = (size_t)a.mh * a.mw;
        const float* proto = a.proto + (size_t)b * a.nm * plane;
        for (int c = tid; c < kMaskHalo * kMaskHalo; c += blockDim.x) {
            const int ly = c / kMaskHalo, lx = c - ly * kMaskHalo;
            const int x = cx0 + lx, y = cy0 + ly;
            float v = 0.0f;
            if (x >= x_lo && x < x_hi && y >= y_lo && y < y_hi) {
                const float* p = proto + (size_t)y * a.mw + x;
                float e = 0.0f;
                for (int j = 0; j < a.nm; ++j) e = __fadd_rn(e, __fmul_rn(s_coeff[j], p[(size_t)j * plane]));  // :47-49
                v = 1.0f / (1.0f + expf(-e));                                                                 // :50
            }
            s_m[ly][lx] = v;
        }
        __syncthreads();
    }
    // 64 x 64 output pixels of this tile, 4 adjacent pixels per thread and pass
    const double scale_x = (double)a.mw / (double)a.net_w, scale_y = (double)a.mh / (double)a.net_h;
    float* out = a.out + ((size_t)b * a.max_masks + m) * (size_t)a.net_h * a.net_w;
    const int ox0 = blockIdx.x * kMaskTile * 4 + (tid & 15) * 4;
    int sx[4];
    float fx[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) resize_tap(ox0 + k, scale_x, a.mw, sx[k], fx[k]);
#pragma unroll
    for (int pass = 0; pass < 4; ++pass) {
        const int oy = blockIdx.y * kMaskTile * 4 + pass * 16 + (tid >> 4);
        if (oy >= a.net_h || ox0 >= a.net_w) continue;
        float4 r = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (touches) {
            int sy;
            float fy;
            resize_tap(oy, scale_y, a.mh, sy, fy);
            const int ly0 = sy - cy0, ly1 = min(sy + 1, a.mh - 1) - cy0;
            const float b0 = 1.0f - fy, b1 = fy;
            float o[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int lx0 = sx[k] - cx0, lx1 = min(sx[k] + 1, a.mw - 1) - cx0;
                // bilinear() written out: as a call, its tap loads move ahead of the arithmetic and ptxas schedules the
                // kernel differently (0.15% slower measured on an H100 80GB HBM3, 700 W)
                const float a0 = 1.0f - fx[k], a1 = fx[k];
                const float h0 = __fadd_rn(__fmul_rn(s_m[ly0][lx0], a0), __fmul_rn(s_m[ly0][lx1], a1));  // HResizeLinear
                const float h1 = __fadd_rn(__fmul_rn(s_m[ly1][lx0], a0), __fmul_rn(s_m[ly1][lx1], a1));
                o[k] = __fadd_rn(__fmul_rn(h0, b0), __fmul_rn(h1, b1));                                   // VResizeLinear
            }
            r = make_float4(o[0], o[1], o[2], o[3]);
        }
        float* dst = out + (size_t)oy * a.net_w + ox0;
        if (ox0 + 3 < a.net_w && (reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
            *reinterpret_cast<float4*>(dst) = r;
        } else {
            const float rr[4] = {r.x, r.y, r.z, r.w};
            for (int k = 0; k < 4 && ox0 + k < a.net_w; ++k) dst[k] = rr[k];
        }
    }
}

// scale_mask (yolov8/src/postprocess.cpp:207-226): cv::resize(mask(r), img.size()) for n masks in one launch.  A thread
// produces 4 adjacent output pixels (one 16-byte store); OpenCV's float bilinear kernel as above (HResize then VResize).
struct ScaleMaskArgs {
    const float* in;  // [n, net_h, net_w]
    float* out;       // [n, img_h, img_w]
    int net_w, net_h, img_w, img_h;
    int rx, ry, rw, rh;
};
__global__ void __launch_bounds__(256) scale_mask_kernel(const __grid_constant__ ScaleMaskArgs a) {
    const int ox0 = (blockIdx.x * 64 + (threadIdx.x & 63)) * 4;
    const int oy = blockIdx.y * 4 + (threadIdx.x >> 6);
    if (ox0 >= a.img_w || oy >= a.img_h) return;
    const double scale_x = (double)a.rw / (double)a.img_w, scale_y = (double)a.rh / (double)a.img_h;
    const float* src = a.in + (size_t)blockIdx.z * a.net_h * a.net_w + (size_t)a.ry * a.net_w + a.rx;
    int sy;
    float fy;
    resize_tap(oy, scale_y, a.rh, sy, fy);
    const float* r0 = src + (size_t)sy * a.net_w;
    const float* r1 = src + (size_t)min(sy + 1, a.rh - 1) * a.net_w;
    const float b0 = 1.0f - fy, b1 = fy;
    float o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        int sx;
        float fx;
        resize_tap(min(ox0 + k, a.img_w - 1), scale_x, a.rw, sx, fx);
        const int sx1 = min(sx + 1, a.rw - 1);
        const float a0 = 1.0f - fx, a1 = fx;
        o[k] = bilinear(__ldg(r0 + sx), __ldg(r0 + sx1), __ldg(r1 + sx), __ldg(r1 + sx1), a0, a1, b0, b1);
    }
    float* dst = a.out + (size_t)blockIdx.z * a.img_h * a.img_w + (size_t)oy * a.img_w + ox0;
    if (ox0 + 3 < a.img_w && (reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
        *reinterpret_cast<float4*>(dst) = make_float4(o[0], o[1], o[2], o[3]);
    } else {
        for (int k = 0; k < 4 && ox0 + k < a.img_w; ++k) dst[k] = o[k];
    }
}

// Mask R-CNN post-process, rcnn/rcnn.cpp:516-550 (host code in the reference).  Two launches, stream-ordered, no workspace:
//   rcnn_rows_kernel  one warp per image: keeps slot i when score > thresh (ascending i), rescales its box to the original
//                     image, (box - pad) * ratio unfused (:523-526), and zeroes the rows past the count;
//   rcnn_paste_kernel one CTA per (image, mask slot, band of full-width rows): the canvas of the k-th kept row is 255 where
//                     cv::resize(mask, r.size()) > 0.5 inside the paste rectangle r (:543-550), 0 elsewhere.
// The paste is bound by HBM writes (one byte per canvas pixel).  Each thread owns 16 adjacent columns (one 16-byte store per
// row) and computes their horizontal taps once for all the rows of its band; a band that misses r's rows stores zeros only.
// The per-frame entry (trtx_rcnn_postprocess_frames_enqueue) runs the same two steps, rcnn_rows_frames_kernel and
// rcnn_paste_frames_kernel, with each frame's size, pads, canvases and pitch in the launch parameters; both pairs of kernels
// call the same per-image (rcnn_rows_image) and per-band (rcnn_paste_band) device functions.
constexpr int kRcnnRowFloats = 7;      // x1, y1, x2, y2, score, class, slot
constexpr int kRcnnMaxMask = 32;       // largest mask_size the shared-memory stage holds
constexpr int kPasteThreads = 256;
constexpr int kPastePasses = 8;        // row passes per CTA: band = kPastePasses * ty rows (~30 KB)

struct RcnnRowsArgs {
    const float* scores;   // [B, D]
    const float* boxes;    // [B, D, 4]
    const float* classes;  // [B, D]
    float* rows;           // [B, 1 + D * 7]
    int batch, dets;
    float thresh;
    int pad_l, pad_t;
    float w_ratio, h_ratio;
};

// One warp: the rows of image b (scores / boxes / classes / out already offset to it).
__device__ __forceinline__ void rcnn_rows_image(const float* scores, const float* boxes, const float* classes, float* out,
                                                int dets, float thresh, int pad_l, int pad_t, float w_ratio, float h_ratio,
                                                int lane) {
    int n = 0;
    for (int i0 = 0; i0 < dets; i0 += 32) {
        const int i = i0 + lane;
        const float s = i < dets ? scores[i] : 0.0f;
        const bool keep = i < dets && s > thresh;  // :522; a NaN score is not kept
        const unsigned m = __ballot_sync(0xffffffffu, keep);
        if (keep) {
            float* r = out + 1 + (size_t)(n + __popc(m & ((1u << lane) - 1u))) * kRcnnRowFloats;
            const float* bx = boxes + (size_t)i * 4;
            r[0] = __fmul_rn(__fsub_rn(bx[0], (float)pad_l), w_ratio);
            r[1] = __fmul_rn(__fsub_rn(bx[1], (float)pad_t), h_ratio);
            r[2] = __fmul_rn(__fsub_rn(bx[2], (float)pad_l), w_ratio);
            r[3] = __fmul_rn(__fsub_rn(bx[3], (float)pad_t), h_ratio);
            r[4] = s;
            r[5] = classes[i];
            r[6] = (float)i;
        }
        n += __popc(m);
    }
    for (int e = n * kRcnnRowFloats + lane; e < dets * kRcnnRowFloats; e += 32) out[1 + e] = 0.0f;
    if (lane == 0) out[0] = (float)n;
}

__global__ void __launch_bounds__(128) rcnn_rows_kernel(const __grid_constant__ RcnnRowsArgs a) {
    const int b = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (b >= a.batch) return;
    const size_t base = (size_t)b * a.dets;
    rcnn_rows_image(a.scores + base, a.boxes + base * 4, a.classes + base,
                    a.rows + (size_t)b * (1 + (size_t)a.dets * kRcnnRowFloats), a.dets, a.thresh, a.pad_l, a.pad_t, a.w_ratio,
                    a.h_ratio, lane);
}

// One axis of the paste rectangle (:543-546): floor(lo) - 1 clamped at 0, ceil(hi) + 1 clamped at `size`, then cv::Rect's
// normalisation (min corner, |delta|).  False where the reference throws: a corner outside the image makes
// Mat::operator()(Rect) throw, an empty size makes cv::resize throw.  In float, floor(c) - 1 is exact wherever it can
// land inside the image, so the comparisons match the reference's double ones.
__device__ __forceinline__ bool rcnn_rect_axis(float c0, float c1, int size, int& o, int& len) {
    float lo = floorf(c0) - 1.0f;
    lo = lo < 0.0f ? 0.0f : lo;
    float hi = ceilf(c1) + 1.0f;
    hi = hi > (float)size ? (float)size : hi;
    if (lo > (float)size || hi < 0.0f) return false;
    const int p = (int)lo, q = (int)hi;
    o = min(p, q);
    len = abs(q - p);
    return len > 0;
}

__device__ __forceinline__ bool rcnn_mask_rect(const float* r, int img_w, int img_h, int& rx, int& ry, int& rw, int& rh) {
    if (!(isfinite(r[0]) && isfinite(r[1]) && isfinite(r[2]) && isfinite(r[3]))) return false;
    return rcnn_rect_axis(r[0], r[2], img_w, rx, rw) && rcnn_rect_axis(r[1], r[3], img_h, ry, rh);
}

// Band `band` of canvas k of image b.  rows [B, 1 + D * 7] and masks [B, D, S, S] are the whole call's; the canvas is
// canvases + (canvas_image * max_masks + k) * img_h * pitch (the single-size entry passes the batch's canvases and b, the
// per-frame one the frame's own canvases and 0; computing the address here, after the barrier, keeps the single-size kernel at
// its 64 registers).  The CTA's threads form a tx x ty grid (tcol, trow): tx over the `chunks` 16-column chunks of a row, ty
// rows per pass, band_rows = kPastePasses * ty; threads with trow >= ty (a fixed block larger than tx * ty) only help stage
// the mask.  Every thread of the CTA calls this, since it may synchronise.
__device__ __forceinline__ void rcnn_paste_band(float* s_m, const float* rows, const float* masks, int b, int dets, int S,
                                                int max_masks, int k, int band, int img_w, int img_h, uint8_t* canvases,
                                                int canvas_image, int pitch, int tx, int ty, int tcol, int trow, int chunks,
                                                int band_rows) {
    const float* img = rows + (size_t)b * (1 + (size_t)dets * kRcnnRowFloats);
    const int count = min((int)img[0], min(dets, max_masks));
    if (k >= count) return;  // slots past the image's kept rows are left untouched
    const float* row = img + 1 + (size_t)k * kRcnnRowFloats;
    int rx = 0, ry = 0, rw = 1, rh = 1;
    const bool pasted = rcnn_mask_rect(row, img_w, img_h, rx, ry, rw, rh);
    const int y0 = band * band_rows, y1 = min(y0 + band_rows, img_h);
    const bool touches = pasted && ry < y1 && ry + rh > y0;  // uniform over the CTA
    if (touches) {
        const float* m = masks + ((size_t)b * dets + (int)row[6]) * S * S;
        const int nthreads = blockDim.x * blockDim.y;
        for (int e = threadIdx.y * blockDim.x + threadIdx.x; e < S * S; e += nthreads) s_m[e] = m[e];
        __syncthreads();
    }
    if (trow >= ty) return;
    const double scale_x = (double)S / (double)rw, scale_y = (double)S / (double)rh;
    uint8_t* plane = canvases + ((size_t)canvas_image * max_masks + k) * (size_t)img_h * pitch;
    for (int c = tcol; c < chunks; c += tx) {
        const int x0 = c * 16;
        int sx[16];
        float fx[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            sx[j] = -1;  // outside r: 0
            fx[j] = 0.0f;
            if (touches && x0 + j >= rx && x0 + j < rx + rw) resize_tap(x0 + j - rx, scale_x, S, sx[j], fx[j]);
        }
        for (int y = y0 + trow; y < y1; y += ty) {
            uint32_t w[4] = {0u, 0u, 0u, 0u};
            if (touches && y >= ry && y < ry + rh) {
                int sy;
                float fy;
                resize_tap(y - ry, scale_y, S, sy, fy);
                const float* r0 = s_m + sy * S;
                const float* r1 = s_m + min(sy + 1, S - 1) * S;
                const float b0 = 1.0f - fy, b1 = fy;
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    if (sx[j] < 0) continue;
                    const int sx1 = min(sx[j] + 1, S - 1);
                    const float a0 = 1.0f - fx[j], a1 = fx[j];
                    const float v = bilinear(r0[sx[j]], r0[sx1], r1[sx[j]], r1[sx1], a0, a1, b0, b1);
                    if (v > 0.5f) w[j >> 2] |= 0xffu << (8 * (j & 3));  // :549 threshold
                }
            }
            store_canvas_chunk(plane + (size_t)y * pitch + x0, w, x0, img_w);
        }
    }
}

struct RcnnPasteArgs {
    const float* rows;   // [B, 1 + D * 7], written by rcnn_rows_kernel
    const float* masks;  // [B, D, S, S]
    uint8_t* out;        // [B, max_masks, img_h, img_w]
    int dets, S, img_w, img_h, max_masks;
    int chunks, bands, band_rows;  // 16-column chunks per row; bands per canvas; rows per band
};

// One CTA of blockDim (tx, ty) per (image, mask slot, band); the host sizes the block to the image width.
__global__ void __launch_bounds__(kPasteThreads) rcnn_paste_kernel(const __grid_constant__ RcnnPasteArgs a) {
    __shared__ float s_m[kRcnnMaxMask * kRcnnMaxMask];
    const int item = blockIdx.x / a.bands, band = blockIdx.x - item * a.bands;
    const int b = item / a.max_masks, k = item - b * a.max_masks;
    rcnn_paste_band(s_m, a.rows, a.masks, b, a.dets, a.S, a.max_masks, k, band, a.img_w, a.img_h, a.out, b, a.img_w,
                    blockDim.x, blockDim.y, threadIdx.x, threadIdx.y, a.chunks, a.band_rows);
}

// The per-frame entry: frames [base, base + n_images) of the call, each with its own size, pads and canvases.
struct RcnnFrame {
    uint8_t* canvas;          // [max_masks, img_h, pitch] u8, or nullptr (rows only)
    int img_w, img_h, pitch;
    int pad_l, pad_t;
    float w_ratio, h_ratio;
    int tx, ty;               // paste threads over a row's 16-column chunks (min(chunks, 256)) and over rows (256 / tx)
    int bands;                // bands of kPastePasses * ty rows per canvas
};
struct RcnnFramesArgs {
    int first_cta[kMaxFrames];  // first CTA of each frame in the paste launch: prefix of max_masks * bands (searched by
                                // every CTA, so kept apart from the rest of the frame's parameters)
    RcnnFrame f[kMaxFrames];
    const float* scores;   // [B, D]
    const float* boxes;    // [B, D, 4]
    const float* classes;  // [B, D]
    const float* masks;    // [B, D, S, S]
    float* rows;           // [B, 1 + D * 7]
    int base, n_images, dets, S, max_masks;
    float thresh;
};

__global__ void __launch_bounds__(128) rcnn_rows_frames_kernel(const __grid_constant__ RcnnFramesArgs a) {
    const int j = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (j >= a.n_images) return;
    const RcnnFrame& f = a.f[j];
    const size_t base = (size_t)(a.base + j) * a.dets;
    rcnn_rows_image(a.scores + base, a.boxes + base * 4, a.classes + base,
                    a.rows + (size_t)(a.base + j) * (1 + (size_t)a.dets * kRcnnRowFloats), a.dets, a.thresh, f.pad_l, f.pad_t,
                    f.w_ratio, f.h_ratio, lane);
}

// Flat grid over (frame, slot, band), kPasteThreads threads per CTA.  Each frame keeps the band decomposition the
// single-size entry would launch for it (the host's tx, ty), the thread's place in it derived here from threadIdx.x.
__global__ void __launch_bounds__(kPasteThreads) rcnn_paste_frames_kernel(const __grid_constant__ RcnnFramesArgs a) {
    __shared__ float s_m[kRcnnMaxMask * kRcnnMaxMask];
    const int lo = frame_of_cta(a.first_cta, a.n_images);
    const RcnnFrame& f = a.f[lo];
    const int local = (int)blockIdx.x - a.first_cta[lo], k = local / f.bands, band = local - k * f.bands;
    const int tx = f.tx, ty = f.ty;
    rcnn_paste_band(s_m, a.rows, a.masks, a.base + lo, a.dets, a.S, a.max_masks, k, band, f.img_w, f.img_h, f.canvas, 0,
                    f.pitch, tx, ty, (int)threadIdx.x % tx, (int)threadIdx.x / tx, (f.img_w + 15) / 16, ty * kPastePasses);
}

// A per-frame entry's descriptors: canvases for all frames or none (-> `canvases`), sizes > 0, with canvases pitch >= img_w.
static int check_frames(const trtx_frame* frames, int batch, bool& canvases) {
    canvases = frames[0].masks_dev != nullptr;
    for (int i = 0; i < batch; ++i) {
        const trtx_frame& d = frames[i];
        if ((d.masks_dev != nullptr) != canvases || d.img_w <= 0 || d.img_h <= 0) return TRTX_ERR_INVALID;
        if (canvases && d.pitch < d.img_w) return TRTX_ERR_INVALID;
    }
    return TRTX_OK;
}

// The launch arguments of frames [i0, i0 + n) of a trtx_rcnn_postprocess_frames_enqueue call (n <= kMaxFrames): each
// frame's pads and ratios, and the band decomposition trtx_rcnn_postprocess_enqueue would launch for it.  ctas: the paste
// CTAs (0 without canvases); TRTX_ERR_UNSUPPORTED past INT_MAX of them.
static int rcnn_fill_frames(const trtx_rcnn_post_params* p, const trtx_frame* frames, int i0, int n, bool canvases,
                            RcnnFramesArgs& a, int& ctas) {
    a.base = i0;
    a.n_images = n;
    long long total = 0;
    for (int j = 0; j < n; ++j) {
        const trtx_frame& d = frames[i0 + j];
        RcnnFrame& f = a.f[j];
        int pads[4];
        trtx_rcnn_letterbox_pads(d.img_w, d.img_h, p->net_w, p->net_h, pads);
        f.canvas = d.masks_dev;
        f.img_w = d.img_w;
        f.img_h = d.img_h;
        f.pitch = d.pitch;
        f.pad_l = pads[0];
        f.pad_t = pads[2];
        f.h_ratio = (float)d.img_h / (float)(p->net_h - (pads[2] + pads[3]));  // as trtx_rcnn_postprocess_enqueue
        f.w_ratio = (float)d.img_w / (float)(p->net_w - (pads[0] + pads[1]));
        f.tx = min((d.img_w + 15) / 16, kPasteThreads);
        f.ty = kPasteThreads / f.tx;
        const int band_rows = f.ty * kPastePasses;
        f.bands = (d.img_h + band_rows - 1) / band_rows;
        a.first_cta[j] = (int)total;
        if (!canvases) continue;
        total += (long long)p->max_masks * f.bands;  // each term < 2^62: checked before the next
        if (total > 0x7fffffffLL) return TRTX_ERR_UNSUPPORTED;
    }
    ctas = (int)total;
    return TRTX_OK;
}

// YOLO segmentation post-process: process_mask (above) + draw_mask_bbox's mask selection (yolov8/src/postprocess.cpp:228-248,
// yolov5/src/postprocess.cpp:148-167), which the reference runs on one host core per image.  For detection k of image b:
//   M = process_mask's 640^2 mask, S = scale_mask(M) (crop trtx_scale_mask_rect, bilinear to img_w x img_h),
//   canvas[k](y, x) = 255 where (x, y) lies in get_rect(img, bbox_k) (clipped to the image) and !(S(y, x) <= 0.5), else 0.
// Two launches per <= 64 images, stream-ordered, no workspace:
//   seg_rows_kernel   one warp per image: count, then (get_rect x, y, w, h, conf, class) per row, zeroes the tail;
//   seg_canvas_kernel one CTA per (image, slot, band of kSegBand full-width canvas rows).  A band that misses get_rect's rows
//                     stores zeros and reads nothing.  Otherwise the band's y-taps of scale_mask name the rows of M it
//                     needs (at most 2 per canvas row) and get_rect's x-range the columns; their process_mask taps name
//                     the low-resolution cells.  The CTA evaluates those sigmoid(dot) values once into shared memory, then
//                     the needed M values with process_mask_kernel's expression, then S with scale_mask_kernel's, and
//                     stores the thresholded bytes with 16-byte stores.  Neither M nor S reaches HBM; every value is the
//                     same expression of the same inputs as in process_mask_kernel -> scale_mask_kernel, so the canvases
//                     are bit-identical to thresholding that composition.
constexpr int kSegBand = 8;                // canvas rows per CTA
constexpr int kSegThreads = 256;
constexpr int kSegMaxY = 2 * kSegBand;     // rows of M a band can need: two taps per canvas row
constexpr int kSegMaxLY = 2 * kSegMaxY;    // low-resolution rows those can need
constexpr int kSegRowFloats = 6;           // x, y, w, h, conf, class

struct SegImage {
    uint8_t* canvas;     // [max_masks, img_h, pitch] u8, or nullptr (rows only)
    int img_w, img_h, pitch;
    int cx, cy, cw, ch;  // scale_mask's crop of the net_w x net_h mask
    int bands;           // canvas row bands of kSegBand rows
};
struct SegArgs {
    int first_cta[kMaxFrames];  // first CTA of each image in the canvas launch: prefix of max_masks * bands
    SegImage img[kMaxFrames];
    const float* proto;  // [B, nm, mh, mw]
    const float* dets;   // [B, 1 + max_rows * row_floats]
    float* rows;         // [B, 1 + max_rows * 6]
    int base, n_images;  // images [base, base + n_images) of the call
    int max_rows, row_floats, coeff_offset, variant, nm, mw, mh, net_w, net_h, max_masks;
    int y_cap, x_cap, ly_cap, lx_cap;  // shared-memory regions of this launch: M [y_cap][x_cap], cells [ly_cap][lx_cap]
};

__global__ void __launch_bounds__(128) seg_rows_kernel(const __grid_constant__ SegArgs a) {
    const int j = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (j >= a.n_images) return;
    const SegImage& im = a.img[j];
    const int b = a.base + j;
    const float* src = a.dets + (size_t)b * (1 + (size_t)a.max_rows * a.row_floats);
    float* out = a.rows + (size_t)b * (1 + (size_t)a.max_rows * kSegRowFloats);
    const int n = min(max((int)src[0], 0), a.max_rows);
    for (int i = lane; i < a.max_rows; i += 32) {
        float* r = out + 1 + (size_t)i * kSegRowFloats;
        if (i < n) {
            const float* d = src + 1 + (size_t)i * a.row_floats;
            int rect[4];
            yolo_get_rect(a.variant, a.net_w, a.net_h, im.img_w, im.img_h, d, rect);  // {0, 0, 0, 0} where undefined
            r[0] = (float)rect[0];
            r[1] = (float)rect[1];
            r[2] = (float)rect[2];
            r[3] = (float)rect[3];
            r[4] = d[4];
            r[5] = d[5];
        } else {
#pragma unroll
            for (int e = 0; e < kSegRowFloats; ++e) r[e] = 0.0f;
        }
    }
    if (lane == 0) out[0] = (float)n;
}

// distinct-value list of at most a few dozen entries (thread 0 only)
__device__ __forceinline__ int seg_slot(int* list, int& n, int v) {
    for (int i = 0; i < n; ++i)
        if (list[i] == v) return i;
    list[n] = v;
    return n++;
}

__global__ void __launch_bounds__(kSegThreads) seg_canvas_kernel(const __grid_constant__ SegArgs a) {
    extern __shared__ __align__(16) float s_dyn[];  // M values [y_cap * x_cap], then sigmoid cells [ly_cap * lx_cap]
    __shared__ float s_coeff[kMaxCoeffs];
    __shared__ int s_yrow[kSegMaxY];      // row of M of each y slot
    __shared__ int s_ytap[kSegBand][2];   // y slots of the two scale_mask taps of band row k
    __shared__ float s_fy[kSegBand];
    __shared__ int s_lyrow[kSegMaxLY];    // low-resolution row of each cell slot
    __shared__ int s_mtap[kSegMaxY][2];   // cell slots of the two process_mask taps of y slot i
    __shared__ float s_mfy[kSegMaxY];
    __shared__ int s_ny, s_nly;
    const int lo = frame_of_cta(a.first_cta, a.n_images);
    const SegImage& im = a.img[lo];
    const int local = (int)blockIdx.x - a.first_cta[lo], k = local / im.bands, band = local - k * im.bands;
    const int b = a.base + lo, tid = threadIdx.x;
    const float* dets = a.dets + (size_t)b * (1 + (size_t)a.max_rows * a.row_floats);
    const int count = min(max((int)dets[0], 0), min(a.max_rows, a.max_masks));
    if (k >= count) return;  // slots past the image's detections are left untouched
    const float* det = dets + 1 + (size_t)k * a.row_floats;
    int rect[4];
    const bool defined = yolo_get_rect(a.variant, a.net_w, a.net_h, im.img_w, im.img_h, det, rect);
    // get_rect clipped to the image (a V5 rect may leave it; the reference's loop would read outside img_mask there)
    const int x_lo = max(rect[0], 0), x_hi = (int)min((long long)rect[0] + rect[2], (long long)im.img_w);
    const int y_lo = max(rect[1], 0), y_hi = (int)min((long long)rect[1] + rect[3], (long long)im.img_h);
    const int y0 = band * kSegBand, y1 = min(y0 + kSegBand, im.img_h);
    const int ya = max(y_lo, y0), yb = min(y_hi, y1);
    const bool touches = defined && x_lo < x_hi && ya < yb;  // uniform over the CTA
    const double sx_scale = (double)im.cw / (double)im.img_w, sy_scale = (double)im.ch / (double)im.img_h;  // scale_mask
    const double mx_scale = (double)a.mw / (double)a.net_w, my_scale = (double)a.mh / (double)a.net_h;      // process_mask
    float* s_M = s_dyn;
    int Xa = 0, nX = 1;
    if (touches) {
        if (tid == 0) {
            int ny = 0, nly = 0;
            for (int y = ya; y < yb; ++y) {
                int sy;
                float fy;
                resize_tap(y, sy_scale, im.ch, sy, fy);
                s_ytap[y - y0][0] = seg_slot(s_yrow, ny, im.cy + sy);
                s_ytap[y - y0][1] = seg_slot(s_yrow, ny, im.cy + min(sy + 1, im.ch - 1));
                s_fy[y - y0] = fy;
            }
            for (int i = 0; i < ny; ++i) {
                int ly;
                float fy;
                resize_tap(s_yrow[i], my_scale, a.mh, ly, fy);
                s_mtap[i][0] = seg_slot(s_lyrow, nly, ly);
                s_mtap[i][1] = seg_slot(s_lyrow, nly, min(ly + 1, a.mh - 1));
                s_mfy[i] = fy;
            }
            s_ny = ny;
            s_nly = nly;
        }
        if (tid < a.nm) s_coeff[tid] = det[a.coeff_offset + tid];
        // columns of M under get_rect's x-range and the low-resolution columns they need (the taps are monotonic)
        int s0, s1;
        float f;
        resize_tap(x_lo, sx_scale, im.cw, s0, f);
        resize_tap(x_hi - 1, sx_scale, im.cw, s1, f);
        Xa = im.cx + s0;
        nX = im.cx + min(s1 + 1, im.cw - 1) - Xa + 1;
        int lxa, lxb;
        resize_tap(Xa, mx_scale, a.mw, lxa, f);
        resize_tap(Xa + nX - 1, mx_scale, a.mw, lxb, f);
        const int nLX = min(lxb + 1, a.mw - 1) - lxa + 1;
        float* s_cell = s_dyn + a.y_cap * a.x_cap;
        __syncthreads();
        const int ny = s_ny, nly = s_nly;
        // low-resolution cells: sigmoid(coeffs . proto) inside get_downscale_rect, 0 outside (process_mask_kernel)
        int rx, ry, rw, rh;
        downscale_rect(a.variant, det, a.net_w, a.net_h, rx, ry, rw, rh);
        const int dx_lo = max(rx, 0), dx_hi = min(rx + rw, a.mw), dy_lo = max(ry, 0), dy_hi = min(ry + rh, a.mh);
        const size_t plane = (size_t)a.mh * a.mw;
        const float* proto = a.proto + (size_t)b * a.nm * plane;
        for (int c = tid; c < nly * nLX; c += blockDim.x) {
            const int i = c / nLX, x = lxa + (c - i * nLX), y = s_lyrow[i];
            float v = 0.0f;
            if (x >= dx_lo && x < dx_hi && y >= dy_lo && y < dy_hi) {
                const float* p = proto + (size_t)y * a.mw + x;
                float e = 0.0f;
                for (int j = 0; j < a.nm; ++j) e = __fadd_rn(e, __fmul_rn(s_coeff[j], __ldg(p + (size_t)j * plane)));
                v = 1.0f / (1.0f + expf(-e));
            }
            s_cell[c] = v;
        }
        __syncthreads();
        // the needed values of M: process_mask_kernel's horizontal then vertical pass
        for (int c = tid; c < ny * nX; c += blockDim.x) {
            const int i = c / nX, X = Xa + (c - i * nX);
            int lx0;
            float fx;
            resize_tap(X, mx_scale, a.mw, lx0, fx);
            const int lx1 = min(lx0 + 1, a.mw - 1) - lxa;
            lx0 -= lxa;
            const float* c0 = s_cell + s_mtap[i][0] * nLX;
            const float* c1 = s_cell + s_mtap[i][1] * nLX;
            // the blends and the canvas store of this kernel are bilinear() and store_canvas_chunk() written out: with the
            // helpers ptxas schedules the kernel differently and the call measured ~1% slower (H100 80GB HBM3, 700 W)
            const float a0 = 1.0f - fx, a1 = fx, fy = s_mfy[i];
            const float b0 = 1.0f - fy, b1 = fy;
            const float h0 = __fadd_rn(__fmul_rn(c0[lx0], a0), __fmul_rn(c0[lx1], a1));  // HResizeLinear
            const float h1 = __fadd_rn(__fmul_rn(c1[lx0], a0), __fmul_rn(c1[lx1], a1));
            s_M[c] = __fadd_rn(__fmul_rn(h0, b0), __fmul_rn(h1, b1));                   // VResizeLinear
        }
        __syncthreads();
    }
    // S = scale_mask_kernel's expression over M, thresholded; each thread owns 16-column chunks of the band's rows
    const int chunks = (im.img_w + 15) / 16;
    const int tx = min(chunks, kSegThreads), ty = kSegThreads / tx;
    const int tcol = tid % tx, trow = tid / tx;
    if (trow >= ty) return;
    uint8_t* plane = im.canvas + (size_t)k * im.img_h * im.pitch;
    for (int c = tcol; c < chunks; c += tx) {
        const int x0 = c * 16;
        int key[16];  // 2 * (first M column - Xa) + (second column != first), or -1 outside get_rect
        float fx[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            key[j] = -1;
            fx[j] = 0.0f;
            const int x = x0 + j;
            if (touches && x >= x_lo && x < x_hi) {
                int sx;
                resize_tap(x, sx_scale, im.cw, sx, fx[j]);
                key[j] = 2 * (im.cx + sx - Xa) + (sx + 1 < im.cw ? 1 : 0);
            }
        }
        for (int y = y0 + trow; y < y1; y += ty) {
            uint32_t w[4] = {0u, 0u, 0u, 0u};
            if (touches && y >= ya && y < yb) {
                const float* r0 = s_M + s_ytap[y - y0][0] * nX;
                const float* r1 = s_M + s_ytap[y - y0][1] * nX;
                const float fy = s_fy[y - y0];
                const float b0 = 1.0f - fy, b1 = fy;
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    if (key[j] < 0) continue;
                    const int m0 = key[j] >> 1, m1 = m0 + (key[j] & 1);
                    const float a0 = 1.0f - fx[j], a1 = fx[j];
                    const float h0 = __fadd_rn(__fmul_rn(r0[m0], a0), __fmul_rn(r0[m1], a1));
                    const float h1 = __fadd_rn(__fmul_rn(r1[m0], a0), __fmul_rn(r1[m1], a1));
                    const float v = __fadd_rn(__fmul_rn(h0, b0), __fmul_rn(h1, b1));
                    if (!(v <= 0.5f)) w[j >> 2] |= 0xffu << (8 * (j & 3));  // draw_mask_bbox: `if (val <= 0.5) continue;`
                }
            }
            uint8_t* dst = plane + (size_t)y * im.pitch + x0;
            if (x0 + 16 <= im.img_w && (reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
                *reinterpret_cast<uint4*>(dst) = make_uint4(w[0], w[1], w[2], w[3]);
            } else {
#pragma unroll
                for (int j = 0; j < 16; ++j)
                    if (x0 + j < im.img_w) dst[j] = (uint8_t)(w[j >> 2] >> (8 * (j & 3)));
            }
        }
    }
}

// Upper bounds of the y slots and cell slots a band can need (seg_canvas_kernel's lists), for a scale_mask row scale s:
// the band's kSegBand row taps span (kSegBand - 1) * s (+ float rounding), so they take at most floor(7 s) + 2 values, + 1
// for the upper taps; the rows of M they name span <= 7 s + 2, and process_mask's scale of 1/4 maps that onto at most
// floor((7 s + 2) / 4) + 3 low-resolution rows.  One more of slack each, capped by the hard limits.
static void seg_caps(double s, int& y_cap, int& ly_cap) {
    const double span = (kSegBand - 1) * s;
    y_cap = span + 4.0 < (double)kSegMaxY ? (int)span + 4 : kSegMaxY;
    ly_cap = (span + 3.0) / 4.0 + 4.0 < (double)kSegMaxLY ? (int)((span + 3.0) / 4.0) + 4 : kSegMaxLY;
    if (ly_cap > 2 * y_cap) ly_cap = 2 * y_cap;
}

// The launch arguments of images [i0, i0 + n) of a trtx_yolo_seg_postprocess_enqueue call (n <= kMaxFrames): sizes and
// canvases, and with canvases each image's scale_mask crop, the launch's shared-memory caps, its canvas CTAs `ctas` and
// dynamic shared memory `smem` (both 0 without canvases).  TRTX_ERR_UNSUPPORTED for an empty crop (the reference's
// cv::resize throws) or more than INT_MAX CTAs.
static int seg_fill_frames(const trtx_mask_params* p, const trtx_frame* frames, int i0, int n, bool canvases, SegArgs& a,
                           int& ctas, size_t& smem) {
    a.base = i0;
    a.n_images = n;
    a.y_cap = a.ly_cap = a.x_cap = 1;
    long long total = 0;
    for (int j = 0; j < n; ++j) {
        const trtx_frame& d = frames[i0 + j];
        SegImage& im = a.img[j];
        im.canvas = d.masks_dev;
        im.img_w = d.img_w;
        im.img_h = d.img_h;
        im.pitch = d.pitch;
        im.bands = (d.img_h + kSegBand - 1) / kSegBand;
        a.first_cta[j] = (int)total;
        if (!canvases) continue;
        int r[4];
        trtx_scale_mask_rect(p->net_w, p->net_h, d.img_w, d.img_h, r);
        if (r[2] <= 0 || r[3] <= 0 || r[0] < 0 || r[1] < 0 || r[0] + r[2] > p->net_w || r[1] + r[3] > p->net_h)
            return TRTX_ERR_UNSUPPORTED;
        im.cx = r[0];
        im.cy = r[1];
        im.cw = r[2];
        im.ch = r[3];
        int yc, lyc;
        seg_caps((double)r[3] / (double)d.img_h, yc, lyc);
        a.y_cap = max(a.y_cap, yc);
        a.ly_cap = max(a.ly_cap, lyc);
        a.x_cap = max(a.x_cap, r[2]);
        total += (long long)p->max_masks * im.bands;  // each term < 2^59: checked before the next
        if (total > 0x7fffffffLL) return TRTX_ERR_UNSUPPORTED;
    }
    a.lx_cap = min(p->mask_w, a.x_cap / 4 + 4);
    ctas = (int)total;
    smem = canvases ? ((size_t)a.y_cap * a.x_cap + (size_t)a.ly_cap * a.lx_cap) * sizeof(float) : 0;
    return TRTX_OK;
}

// Pose and oriented-box post-process: the per-detection geometry of draw_bbox_keypoints_line (get_rect_adapt_landmark,
// yolov8/src/postprocess.cpp:173-205) and draw_bbox_obb (get_corner, :474-507), which the reference runs on one host core
// after a D2H copy.  One CTA of kPoseObbThreads per frame, one launch per <= 64 frames, no workspace, no atomics:
//   the CTA walks the first min(count, max_rows) rows in passes of kPoseObbThreads, one row per thread; a ballot per warp
//   over the keep column and a scan of the warps' counts give each kept row its output slot (input order); the owning
//   thread computes the rectangle (yolo_get_rect) or the four corners (yolo_get_corner) into shared memory; then the whole
//   CTA writes the pass's kept rows as one contiguous run of floats (coalesced), mapping each keypoint coordinate with
//   yolo_map_landmark on the way.  Rows past the kept count are zeroed.
constexpr int kPoseObbThreads = 256;   // rows per pass
constexpr int kPoseObbWarps = kPoseObbThreads / kWarp;
constexpr int kPoseMaxKpts = 64;

struct PoseObbArgs {
    int img_w[kMaxFrames], img_h[kMaxFrames];
    const float* dets;  // [B, 1 + max_rows * row_floats]
    float* rows;        // [B, 1 + max_rows * out_floats]
    int base;           // frames [base, base + gridDim.x) of the call
    int pose, net_w, net_h, row_floats, extra_offset, num_kpts, out_floats, max_rows;
};

__global__ void __launch_bounds__(kPoseObbThreads) pose_obb_rows_kernel(const __grid_constant__ PoseObbArgs a) {
    __shared__ int s_src[kPoseObbThreads];      // input row of each kept row of the pass, by output slot
    __shared__ int s_geo[kPoseObbThreads * 8];  // its rectangle (pose: 4 ints) or corners (OBB: 8 ints)
    __shared__ int s_warp[kPoseObbWarps];       // kept rows per warp of the pass
    const int j = blockIdx.x, tid = threadIdx.x, lane = tid & (kWarp - 1), warp = tid / kWarp, b = a.base + j;
    const int img_w = a.img_w[j], img_h = a.img_h[j];
    const size_t R = (size_t)a.row_floats, F = (size_t)a.out_floats;
    const float* src = a.dets + (size_t)b * (1 + (size_t)a.max_rows * R);
    float* out = a.rows + (size_t)b * (1 + (size_t)a.max_rows * F);
    const int n = min(max((int)src[0], 0), a.max_rows);
    const YoloLetterbox lb = yolo_letterbox(a.net_w, a.net_h, img_w, img_h);
    const int geo = a.pose ? 4 : 8;  // floats of the row before conf and class
    int kept = 0;                    // rows written by the earlier passes
    for (int i0 = 0; i0 < n; i0 += kPoseObbThreads) {
        const int i = i0 + tid;
        const float* d = src + 1 + (size_t)i * R;
        const bool keep = i < n && (int)d[6] == 1;  // process_decode_ptr_host: `int keep_flag = ...; if (keep_flag == 1)`
        const unsigned m = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) s_warp[warp] = __popc(m);
        __syncthreads();
        int before = 0, total = 0;
#pragma unroll
        for (int w = 0; w < kPoseObbWarps; ++w) {
            const int c = s_warp[w];
            before += w < warp ? c : 0;
            total += c;
        }
        if (keep) {
            const int slot = before + __popc(m & ((1u << lane) - 1u));
            int g[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            if (a.pose)
                yolo_get_rect(TRTX_YOLO_V8, a.net_w, a.net_h, img_w, img_h, d, g);  // {0, 0, 0, 0} where undefined
            else
                yolo_get_corner(a.net_w, a.net_h, img_w, img_h, d, d[a.extra_offset], g);
            s_src[slot] = i;
#pragma unroll
            for (int e = 0; e < 8; ++e) s_geo[slot * 8 + e] = g[e];
        }
        __syncthreads();
        const size_t run = (size_t)total * F;
        float* o = out + 1 + (size_t)kept * F;
#pragma unroll 4
        for (size_t f = tid; f < run; f += kPoseObbThreads) {
            const int r = (int)(f / F), e = (int)(f - (size_t)r * F);
            const float* d2 = src + 1 + (size_t)s_src[r] * R;
            float v;
            if (e < geo) {
                v = (float)s_geo[r * 8 + e];
            } else if (e < geo + 2) {
                v = d2[4 + e - geo];  // conf, class
            } else {
                const int k = e - 6;  // keypoint float: x, y, conf
                const int c = k % 3;
                const float x = d2[a.extra_offset + k];
                v = c == 2 ? x : yolo_map_landmark(lb, c, x);
            }
            o[f] = v;
        }
        kept += total;
        __syncthreads();  // the next pass reuses the shared arrays
    }
    const size_t end = 1 + (size_t)a.max_rows * F;
    for (size_t f = 1 + (size_t)kept * F + tid; f < end; f += kPoseObbThreads) out[f] = 0.0f;
    if (tid == 0) out[0] = (float)kept;
}

}  // namespace trtx

using namespace trtx;

extern "C" {

TRTX_API int trtx_process_mask_enqueue(const trtx_mask_params* p, int batch, const float* proto_dev, const float* dets_dev,
                                       int max_rows, float* masks_dev, trtx_stream_t stream) {
    if (!p || batch <= 0 || !proto_dev || !dets_dev || !masks_dev || max_rows <= 0) return TRTX_ERR_INVALID;
    if (p->variant != TRTX_YOLO_V8 && p->variant != TRTX_YOLO_V5) return TRTX_ERR_INVALID;
    if (p->num_coeffs <= 0 || p->num_coeffs > kMaxCoeffs || p->max_masks <= 0 || p->row_floats < 4) return TRTX_ERR_INVALID;
    if (p->coeff_offset < 0 || p->coeff_offset + p->num_coeffs > p->row_floats) return TRTX_ERR_INVALID;
    if (p->mask_w <= 0 || p->mask_h <= 0) return TRTX_ERR_INVALID;
    // the reference hard-codes the factor 4 (get_downscale_rect(bbox, 4), kInputH / 4)
    if (p->net_w != 4 * p->mask_w || p->net_h != 4 * p->mask_h) return TRTX_ERR_UNSUPPORTED;
    if ((long long)batch * p->max_masks > 65535) return TRTX_ERR_UNSUPPORTED;
    MaskArgs a;
    a.proto = proto_dev;
    a.dets = dets_dev;
    a.out = masks_dev;
    a.max_rows = max_rows;
    a.row_floats = p->row_floats;
    a.coeff_offset = p->coeff_offset;
    a.variant = p->variant;
    a.nm = p->num_coeffs;
    a.mw = p->mask_w;
    a.mh = p->mask_h;
    a.net_w = p->net_w;
    a.net_h = p->net_h;
    a.max_masks = p->max_masks;
    dim3 grid((p->mask_w + kMaskTile - 1) / kMaskTile, (p->mask_h + kMaskTile - 1) / kMaskTile, batch * p->max_masks);
    process_mask_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(a);
    return check_launch();
}

// the crop of scale_mask, yolov8/src/postprocess.cpp:208-222: `h = r_w * img.rows` truncates float -> int, `(kInputH - h) / 2`
// is an integer division
TRTX_API int trtx_scale_mask_rect(int net_w, int net_h, int img_w, int img_h, int rect[4]) {
    if (!rect || net_w <= 0 || net_h <= 0 || img_w <= 0 || img_h <= 0) return TRTX_ERR_INVALID;
    int x, y, w, h;
    const float r_w = (float)(net_w / (img_w * 1.0));
    const float r_h = (float)(net_h / (img_h * 1.0));
    if (r_h > r_w) {
        w = net_w;
        h = (int)(r_w * img_h);
        x = 0;
        y = (net_h - h) / 2;
    } else {
        w = (int)(r_h * img_w);
        h = net_h;
        x = (net_w - w) / 2;
        y = 0;
    }
    rect[0] = x;
    rect[1] = y;
    rect[2] = w;
    rect[3] = h;
    return TRTX_OK;
}

TRTX_API int trtx_scale_mask_enqueue(const float* masks_dev, int n, int net_w, int net_h, int img_w, int img_h, float* out_dev,
                                     trtx_stream_t stream) {
    if (!masks_dev || !out_dev || n <= 0 || n > 65535) return TRTX_ERR_INVALID;
    int r[4];
    const int rc = trtx_scale_mask_rect(net_w, net_h, img_w, img_h, r);
    if (rc) return rc;
    if (r[2] <= 0 || r[3] <= 0 || r[0] < 0 || r[1] < 0 || r[0] + r[2] > net_w || r[1] + r[3] > net_h) return TRTX_ERR_UNSUPPORTED;
    ScaleMaskArgs a{masks_dev, out_dev, net_w, net_h, img_w, img_h, r[0], r[1], r[2], r[3]};
    dim3 grid((img_w + 255) / 256, (img_h + 3) / 4, n);
    scale_mask_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(a);
    return check_launch();
}

// preprocessImg's pads, rcnn/common.hpp:79-102: `input_w / (img.cols*1.0)` is a double division stored to float, `r_w *
// img.rows` a float product truncated to int, `(input_h - h) / 2.f` float; each pad is round() of that float -/+ 0.1 (double)
TRTX_API int trtx_rcnn_letterbox_pads(int img_w, int img_h, int net_w, int net_h, int pads[4]) {
    if (!pads || img_w <= 0 || img_h <= 0 || net_w <= 0 || net_h <= 0) return TRTX_ERR_INVALID;
    int w, h;
    float x, y;
    const float r_w = (float)(net_w / (img_w * 1.0));
    const float r_h = (float)(net_h / (img_h * 1.0));
    if (r_h > r_w) {
        w = net_w;
        h = (int)(r_w * (float)img_h);
        x = 0.0f;
        y = (float)(net_h - h) / 2.f;
    } else {
        w = (int)(r_h * (float)img_w);
        h = net_h;
        x = (float)(net_w - w) / 2.f;
        y = 0.0f;
    }
    (void)w;
    (void)h;
    pads[0] = (int)round(x - 0.1);
    pads[1] = (int)round(x + 0.1);
    pads[2] = (int)round(y - 0.1);
    pads[3] = (int)round(y + 0.1);
    return TRTX_OK;
}

TRTX_API int trtx_rcnn_postprocess_enqueue(const trtx_rcnn_post_params* p, int batch, const float* scores_dev,
                                           const float* boxes_dev, const float* classes_dev, const float* masks_dev,
                                           float* rows_dev, uint8_t* masks_out_dev, trtx_stream_t stream) {
    if (!p || batch <= 0 || !scores_dev || !boxes_dev || !classes_dev || !rows_dev) return TRTX_ERR_INVALID;
    if ((masks_dev == nullptr) != (masks_out_dev == nullptr)) return TRTX_ERR_INVALID;
    if (p->net_w <= 0 || p->net_h <= 0 || p->img_w <= 0 || p->img_h <= 0 || p->detections_per_im <= 0 || p->mask_size <= 0 ||
        p->max_masks <= 0)
        return TRTX_ERR_INVALID;
    if (p->mask_size > kRcnnMaxMask) return TRTX_ERR_INVALID;
    int pads[4];
    trtx_rcnn_letterbox_pads(p->img_w, p->img_h, p->net_w, p->net_h, pads);
    RcnnRowsArgs ra;
    ra.scores = scores_dev;
    ra.boxes = boxes_dev;
    ra.classes = classes_dev;
    ra.rows = rows_dev;
    ra.batch = batch;
    ra.dets = p->detections_per_im;
    ra.thresh = p->score_thresh;
    ra.pad_l = pads[0];
    ra.pad_t = pads[2];
    ra.h_ratio = (float)p->img_h / (float)(p->net_h - (pads[2] + pads[3]));  // rcnn.cpp:516-517
    ra.w_ratio = (float)p->img_w / (float)(p->net_w - (pads[0] + pads[1]));
    // bands of full-width rows: blockDim.x threads over the 16-column chunks, blockDim.y rows per pass
    const int chunks = (p->img_w + 15) / 16;
    const int tx = min(chunks, kPasteThreads), ty = kPasteThreads / tx;
    const int band_rows = ty * kPastePasses, bands = (p->img_h + band_rows - 1) / band_rows;
    const long long ctas = (long long)batch * p->max_masks * bands;
    if (masks_dev && ctas > 0x7fffffffLL) return TRTX_ERR_UNSUPPORTED;
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    rcnn_rows_kernel<<<(batch + 3) / 4, 128, 0, s>>>(ra);
    const int rc = check_launch();
    if (rc || !masks_dev) return rc;
    RcnnPasteArgs pa;
    pa.rows = rows_dev;
    pa.masks = masks_dev;
    pa.out = masks_out_dev;
    pa.dets = p->detections_per_im;
    pa.S = p->mask_size;
    pa.img_w = p->img_w;
    pa.img_h = p->img_h;
    pa.max_masks = p->max_masks;
    pa.chunks = chunks;
    pa.bands = bands;
    pa.band_rows = band_rows;
    rcnn_paste_kernel<<<(unsigned)ctas, dim3(tx, ty), 0, s>>>(pa);
    return check_launch();
}

TRTX_API int trtx_rcnn_postprocess_frames_enqueue(const trtx_rcnn_post_params* p, const trtx_frame* images_host,
                                                  int batch, const float* scores_dev, const float* boxes_dev,
                                                  const float* classes_dev, const float* masks_dev, float* rows_dev,
                                                  trtx_stream_t stream) {
    if (!p || !images_host || batch <= 0 || !scores_dev || !boxes_dev || !classes_dev || !rows_dev) return TRTX_ERR_INVALID;
    if (p->net_w <= 0 || p->net_h <= 0 || p->detections_per_im <= 0 || p->mask_size <= 0 || p->max_masks <= 0)
        return TRTX_ERR_INVALID;
    if (p->mask_size > kRcnnMaxMask) return TRTX_ERR_INVALID;
    bool canvases;
    int rc = check_frames(images_host, batch, canvases);
    if (rc) return rc;
    if (canvases && !masks_dev) return TRTX_ERR_INVALID;
    RcnnFramesArgs a;
    a.scores = scores_dev;
    a.boxes = boxes_dev;
    a.classes = classes_dev;
    a.masks = masks_dev;
    a.rows = rows_dev;
    a.dets = p->detections_per_im;
    a.S = p->mask_size;
    a.max_masks = p->max_masks;
    a.thresh = p->score_thresh;
    // every frame is checked before the first launch, so a rejected call writes nothing
    int ctas;
    for (int i0 = 0; i0 < batch; i0 += kMaxFrames)
        if ((rc = rcnn_fill_frames(p, images_host, i0, min(batch - i0, kMaxFrames), canvases, a, ctas))) return rc;
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    for (int i0 = 0; i0 < batch; i0 += kMaxFrames) {
        const int n = min(batch - i0, kMaxFrames);
        rcnn_fill_frames(p, images_host, i0, n, canvases, a, ctas);
        rcnn_rows_frames_kernel<<<(n + 3) / 4, 128, 0, s>>>(a);
        if ((rc = check_launch())) return rc;
        if (!canvases) continue;
        rcnn_paste_frames_kernel<<<(unsigned)ctas, kPasteThreads, 0, s>>>(a);
        if ((rc = check_launch())) return rc;
    }
    return TRTX_OK;
}

TRTX_API int trtx_yolo_seg_postprocess_enqueue(const trtx_mask_params* p, const trtx_frame* images_host, int batch,
                                               const float* proto_dev, const float* dets_dev, int max_rows,
                                               float* rows_dev, trtx_stream_t stream) {
    if (!p || !images_host || batch <= 0 || !dets_dev || !rows_dev || max_rows <= 0) return TRTX_ERR_INVALID;
    if (p->variant != TRTX_YOLO_V8 && p->variant != TRTX_YOLO_V5) return TRTX_ERR_INVALID;
    if (p->net_w <= 0 || p->net_h <= 0 || p->row_floats < kSegRowFloats) return TRTX_ERR_INVALID;
    bool masks;
    int rc = check_frames(images_host, batch, masks);
    if (rc) return rc;
    if (masks) {  // trtx_process_mask_enqueue's checks
        if (!proto_dev) return TRTX_ERR_INVALID;
        if (p->num_coeffs <= 0 || p->num_coeffs > kMaxCoeffs || p->max_masks <= 0) return TRTX_ERR_INVALID;
        if (p->coeff_offset < 0 || p->coeff_offset + p->num_coeffs > p->row_floats) return TRTX_ERR_INVALID;
        if (p->mask_w <= 0 || p->mask_h <= 0) return TRTX_ERR_INVALID;
        if (p->net_w != 4 * p->mask_w || p->net_h != 4 * p->mask_h) return TRTX_ERR_UNSUPPORTED;
    }
    SegArgs a;
    a.proto = proto_dev;
    a.dets = dets_dev;
    a.rows = rows_dev;
    a.max_rows = max_rows;
    a.row_floats = p->row_floats;
    a.coeff_offset = p->coeff_offset;
    a.variant = p->variant;
    a.nm = p->num_coeffs;
    a.mw = p->mask_w;
    a.mh = p->mask_h;
    a.net_w = p->net_w;
    a.net_h = p->net_h;
    a.max_masks = p->max_masks;
    // every image is checked before the first launch, so that a rejected call writes nothing
    int ctas;
    size_t smem, smem_max = 0;
    for (int i0 = 0; i0 < batch; i0 += kMaxFrames) {
        if ((rc = seg_fill_frames(p, images_host, i0, min(batch - i0, kMaxFrames), masks, a, ctas, smem))) return rc;
        smem_max = max(smem_max, smem);
    }
    if (smem_max > 48 * 1024 &&
        cudaFuncSetAttribute(seg_canvas_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_max) != cudaSuccess) {
        g_last_cuda_error = (int)cudaGetLastError();
        return TRTX_ERR_CUDA;
    }
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    for (int i0 = 0; i0 < batch; i0 += kMaxFrames) {
        const int n = min(batch - i0, kMaxFrames);
        seg_fill_frames(p, images_host, i0, n, masks, a, ctas, smem);
        seg_rows_kernel<<<(n + 3) / 4, 128, 0, st>>>(a);
        if ((rc = check_launch())) return rc;
        if (!masks) continue;
        seg_canvas_kernel<<<(unsigned)ctas, kSegThreads, smem, st>>>(a);
        if ((rc = check_launch())) return rc;
    }
    return TRTX_OK;
}

TRTX_API int trtx_yolo_pose_obb_postprocess_enqueue(const trtx_pose_obb_params* p, const int32_t* frame_wh_host, int batch,
                                                    const float* dets_dev, int max_rows, float* rows_dev,
                                                    trtx_stream_t stream) {
    if (!p || !frame_wh_host || batch <= 0 || !dets_dev || !rows_dev || max_rows <= 0) return TRTX_ERR_INVALID;
    if (p->task != TRTX_TASK_POSE && p->task != TRTX_TASK_OBB) return TRTX_ERR_INVALID;
    if (p->net_w <= 0 || p->net_h <= 0 || p->row_floats < 7 || p->extra_offset < 0) return TRTX_ERR_INVALID;
    const bool pose = p->task == TRTX_TASK_POSE;
    if (pose && (p->num_kpts < 0 || p->num_kpts > kPoseMaxKpts || p->extra_offset + 3 * p->num_kpts > p->row_floats))
        return TRTX_ERR_INVALID;
    if (!pose && p->extra_offset >= p->row_floats) return TRTX_ERR_INVALID;
    // every frame is checked before the first launch, so that a rejected call writes nothing
    for (int i = 0; i < batch; ++i)
        if (frame_wh_host[2 * i] <= 0 || frame_wh_host[2 * i + 1] <= 0) return TRTX_ERR_INVALID;
    PoseObbArgs a;
    a.dets = dets_dev;
    a.rows = rows_dev;
    a.pose = pose;
    a.net_w = p->net_w;
    a.net_h = p->net_h;
    a.row_floats = p->row_floats;
    a.extra_offset = p->extra_offset;
    a.num_kpts = pose ? p->num_kpts : 0;
    a.out_floats = pose ? 6 + 3 * p->num_kpts : 10;
    a.max_rows = max_rows;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    for (int i0 = 0; i0 < batch; i0 += kMaxFrames) {
        const int n = min(batch - i0, kMaxFrames);
        a.base = i0;
        for (int j = 0; j < n; ++j) {
            a.img_w[j] = frame_wh_host[2 * (i0 + j)];
            a.img_h[j] = frame_wh_host[2 * (i0 + j) + 1];
        }
        pose_obb_rows_kernel<<<n, kPoseObbThreads, 0, st>>>(a);
        const int rc = check_launch();
        if (rc) return rc;
    }
    return TRTX_OK;
}

}  // extern "C"
