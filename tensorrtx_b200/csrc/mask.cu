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

struct MaskArgs {
    const float* proto;  // [B, nm, mh, mw]
    const float* dets;   // [B, 1 + max_rows * row_floats]
    float* out;          // [B, max_masks, net_h, net_w]
    int max_rows, row_floats, coeff_offset;
    int variant, nm, mw, mh, net_w, net_h, max_masks;
};

// get_downscale_rect: yolov8_seg.cpp:17-34 (bbox used as x, y, w, h; clamped to the network input; int() truncation),
// yolov5/src/postprocess.cpp:94-104 (cx, cy, w, h; round()), as the cells [x_lo, x_hi) x [y_lo, y_hi) of the mw x mh mask
// that process_mask's loops visit.  The loops are clamped to the mask here (the reference would write out of bounds for a
// v5 box that leaves the image).  Where one of the four float -> int conversions is undefined (a non-finite box, or a
// corner or size past the int range in cells) the range is empty, so the mask is all zeros, as get_rect gives {0, 0, 0, 0}
// for such boxes; rx + rw is summed in 64 bits.
__device__ __forceinline__ void downscale_rect(int variant, const float* bbox, int net_w, int net_h, int mw, int mh,
                                               int& x_lo, int& x_hi, int& y_lo, int& y_hi) {
    float left, top, right, bottom;
    int rx, ry, rw, rh;
    bool defined;
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
        defined = trunc_to_int(left, rx) && trunc_to_int(top, ry) && trunc_to_int(__fsub_rn(right, left), rw) &&
                  trunc_to_int(__fsub_rn(bottom, top), rh);
    } else {
        left = __fsub_rn(bbox[0], __fdiv_rn(bbox[2], 2.0f));
        top = __fsub_rn(bbox[1], __fdiv_rn(bbox[3], 2.0f));
        right = __fadd_rn(bbox[0], __fdiv_rn(bbox[2], 2.0f));
        bottom = __fadd_rn(bbox[1], __fdiv_rn(bbox[3], 2.0f));
        left = __fdiv_rn(left, 4.0f);
        top = __fdiv_rn(top, 4.0f);
        right = __fdiv_rn(right, 4.0f);
        bottom = __fdiv_rn(bottom, 4.0f);
        defined = round_to_int(left, rx) && round_to_int(top, ry) && round_to_int(__fsub_rn(right, left), rw) &&
                  round_to_int(__fsub_rn(bottom, top), rh);
    }
    if (!defined) {
        x_lo = x_hi = y_lo = y_hi = 0;
        return;
    }
    // the 64-bit ends are clamped to [0, mw] and [0, mh] before they narrow: a V5 box with rx and rw both near INT_MIN
    // sums below INT_MIN, which would wrap to a large positive end
    x_lo = max(rx, 0);
    x_hi = (int)max(0LL, min((long long)rx + rw, (long long)mw));
    y_lo = max(ry, 0);
    y_hi = (int)max(0LL, min((long long)ry + rh, (long long)mh));
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
    int x_lo, x_hi, y_lo, y_hi;
    downscale_rect(a.variant, det, a.net_w, a.net_h, a.mw, a.mh, x_lo, x_hi, y_lo, y_hi);
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

// Outlines of the Mask R-CNN canvases: cv::findContours(curMask, RETR_EXTERNAL, CHAIN_APPROX_NONE) of rcnn/rcnn.cpp:551-552,
// OpenCV's Suzuki-Abe border following restated bit for bit (oracle_find_contours_external spells out the scan).  By the
// post-process's contract a canvas is 0 outside the paste rectangle r of its row, so the kernel reads r only.  A persistent
// grid: CTA i owns workspace slot i and walks canvases i, i + gridDim.x, ... of the launch.  Per canvas:
//   A. r -> the slot's padded int8 map (1 where nonzero, a zero frame around it), all threads;
//   B. bands of kContourBand rows: all warps list the band's runs of nonzero pixels (start, end) in raster order; warp 0 then
//      walks them in order.  A run start with value 1 (unvisited) is an outer-border start, followed by lane 0 unless the
//      value at lnbd (the last place in the row where the value changed to a mark) is positive; following marks the map and
//      appends (start, length) to the slot's contour list.  The lanes hold 32 runs' start / end values at a time (reloaded
//      after a trace), so the walk costs a few instructions per run;
//   C. contours in descending start order (cv2's): a suffix scan of the lengths gives each contour's first point, and one
//      thread per contour follows it again (the path reads zero / nonzero only) to write its points up to max_points.
// No atomics: the output depends only on the canvas.
constexpr int kContourThreads = 256;
constexpr int kContourWarps = kContourThreads / kWarp;
constexpr int kContourBand = 32;     // map rows per run-listing band
constexpr int kContourCtas = 128;    // CTAs (workspace slots) per launch at most
constexpr int kContourSmem = 200 * 1024;  // dynamic shared memory per CTA: the map of an r that fits goes here

struct ContourFrame {
    const uint8_t* canvas;  // [max_masks, img_h, pitch]
    int img_w, img_h, pitch;
};
struct ContourArgs {
    ContourFrame f[kMaxFrames];
    const float* rows;  // [B, 1 + D * 7]
    int32_t* counts;    // [B, max_masks, 2]
    int32_t* lengths;   // [B, max_masks, C]
    int32_t* points;    // [B, max_masks, P, 2]
    uint8_t* work;      // gridDim.x slots of slot_bytes
    size_t slot_bytes;
    long long map_bytes, list_bytes;  // offsets in a slot: map at 0, contour list at map_bytes, band runs at + list_bytes
    int base, n_images, dets, max_masks, max_contours, max_points;
};

// The regions of a workspace slot for a frame of w x h: the padded map; the contour list (at most ceil(w/2) * ceil(h/2)
// contours: a component and the zero pixels that part it from the next take 2 x 2 pixels); the runs of one band (at most
// ceil(w/2) per row).  A call's slot holds the largest of each region over its frames.
static void contour_regions(int w, int h, long long& map_bytes, long long& list_bytes, long long& band_bytes) {
    map_bytes = ((long long)(w + 2) * (h + 2) + 15) / 16 * 16;
    list_bytes = (long long)((w + 1) / 2) * ((h + 1) / 2) * 8;
    band_bytes = (long long)kContourBand * ((w + 1) / 2) * 8;
}

// Step s of the 3 x 3 neighbourhood (0 east, 1 north-east, ... counter-clockwise, y down), OpenCV's CV_INIT_3X3_DELTAS
__device__ __forceinline__ int code_dx(int s) { return ((36890 >> (2 * s)) & 3) - 1; }  // {1, 1, 0, -1, -1, -1, 0, 1}
__device__ __forceinline__ int code_dy(int s) { return ((43265 >> (2 * s)) & 3) - 1; }  // {0, -1, -1, -1, 0, 1, 1, 1}

// OpenCV's icvFetchContour for the outer border starting at map index i0 (map coordinates x, y): returns the number of
// points.  mark: write the visit marks (-2 where the search passed the right neighbour as 0, else 2 over a 1).  out: when not
// null, point q < limit goes to out[2q], out[2q + 1] as (x + ox, y + oy).
__device__ int contour_follow(int8_t* m, int stride, int i0, int x, int y, bool mark, int32_t* out, int limit, int ox, int oy) {
    int s = 4, i1;
    do {
        s = (s - 1) & 7;
        i1 = i0 + code_dx(s) + code_dy(s) * stride;
    } while (m[i1] == 0 && s != 4);
    if (s == 4) {  // a lone pixel
        if (mark) m[i0] = -2;
        if (out && limit > 0) out[0] = x + ox, out[1] = y + oy;
        return 1;
    }
    int i3 = i0, i4, n = 0;
    for (;;) {
        const int s_end = s;
        do {
            ++s;
            i4 = i3 + code_dx(s & 7) + code_dy(s & 7) * stride;
        } while (m[i4] == 0);
        s &= 7;
        if (mark) {
            if ((unsigned)(s - 1) < (unsigned)s_end) m[i3] = -2;
            else if (m[i3] == 1) m[i3] = 2;
        }
        if (out && n < limit) {
            out[2 * n] = x + ox;
            out[2 * n + 1] = y + oy;
        }
        ++n;
        x += code_dx(s);
        y += code_dy(s);
        if (i4 == i0 && i3 == i1) break;
        i3 = i4;
        s = (s + 4) & 7;
    }
    return n;
}

__device__ __forceinline__ bool is_mark(int v) { return (v & -2) != 0; }

__global__ void __launch_bounds__(kContourThreads) rcnn_contours_kernel(const __grid_constant__ ContourArgs a) {
    __shared__ int s_off[kContourBand + 1];  // first run of each band row in the band list
    __shared__ long long s_wsum[kContourWarps];
    __shared__ int s_n;                      // contours in the slot's list
    __shared__ long long s_carry;
    const int tid = threadIdx.x, lane = tid & (kWarp - 1), warp = tid / kWarp;
    uint8_t* slot = a.work + (size_t)blockIdx.x * a.slot_bytes;
    extern __shared__ __align__(16) int8_t s_map[];
    int2* list = reinterpret_cast<int2*>(slot + a.map_bytes);                 // (map index, length) in trace order
    int2* runs = reinterpret_cast<int2*>(slot + a.map_bytes + a.list_bytes);  // (start, end) of the band's runs
    for (int c = blockIdx.x; c < a.n_images * a.max_masks; c += gridDim.x) {
        const int j = c / a.max_masks, k = c - j * a.max_masks, b = a.base + j;
        const ContourFrame& f = a.f[j];
        const size_t canvas_id = (size_t)b * a.max_masks + k;
        const float* img = a.rows + (size_t)b * (1 + (size_t)a.dets * kRcnnRowFloats);
        const int count = min((int)img[0], min(a.dets, a.max_masks));  // as rcnn_paste_band
        int rx = 0, ry = 0, W = 0, H = 0;
        if (k >= count || !rcnn_mask_rect(img + 1 + (size_t)k * kRcnnRowFloats, f.img_w, f.img_h, rx, ry, W, H)) {
            if (tid == 0) a.counts[2 * canvas_id] = a.counts[2 * canvas_id + 1] = 0;
            continue;  // uniform over the CTA
        }
        const int stride = W + 2;
        // the map in shared memory when it fits (the follower's loads and marks then stay on chip), else in the slot
        int8_t* m = (long long)stride * (H + 2) <= kContourSmem ? s_map : reinterpret_cast<int8_t*>(slot);
        // A. the padded map of r
        const uint8_t* src = f.canvas + (size_t)k * f.img_h * f.pitch;
        for (int y = warp; y < H + 2; y += kContourWarps) {
            const uint8_t* row = src + (size_t)(ry + y - 1) * f.pitch + rx - 1;
            int8_t* dst = m + (size_t)y * stride;
            const bool inner = y >= 1 && y <= H;
            for (int x = lane; x < stride; x += kWarp) dst[x] = inner && x >= 1 && x <= W && row[x] != 0;
        }
        if (tid == 0) s_n = 0;
        __syncthreads();
        // B. bands of rows 1 .. H
        for (int y0 = 1; y0 <= H; y0 += kContourBand) {
            const int nrows = min(kContourBand, H + 1 - y0);
            // runs of each row: starts where a nonzero follows a zero, ends before a zero that follows a nonzero (the
            // map's frame closes every run); counted, then written at the row's offset
            for (int pass = 0; pass < 2; ++pass) {
                for (int r = warp; r < nrows; r += kContourWarps) {
                    const int8_t* row = m + (size_t)(y0 + r) * stride;
                    int n = pass ? s_off[r] : 0;
                    int ne = n;
                    unsigned carry = 0;
                    for (int x0 = 1; x0 <= W + 1; x0 += kWarp) {
                        const int x = x0 + lane;
                        const unsigned bits = __ballot_sync(0xffffffffu, x <= W + 1 && row[x] != 0);
                        const unsigned left = (bits << 1) | carry;
                        const unsigned st = bits & ~left, en = ~bits & left;
                        if (pass) {
                            const unsigned lt = (1u << lane) - 1u;
                            if (st >> lane & 1) runs[n + __popc(st & lt)].x = x;
                            if (en >> lane & 1) runs[ne + __popc(en & lt)].y = x - 1;
                        }
                        n += __popc(st);
                        ne += __popc(en);
                        carry = bits >> 31;
                    }
                    if (!pass && lane == 0) s_off[r + 1] = n;  // counts, summed below
                }
                __syncthreads();
                if (!pass) {
                    if (tid == 0) {
                        s_off[0] = 0;
                        for (int r = 0; r < nrows; ++r) s_off[r + 1] += s_off[r];
                    }
                    __syncthreads();
                }
            }
            // warp 0 walks the band's runs in raster order
            if (warp == 0) {
                const int nruns = s_off[nrows];
                int cur = -1, mval = 0, nc = s_n;
                for (int i0 = 0; i0 < nruns; i0 += kWarp) {
                    const int i = i0 + lane;
                    int ry_i = 0, s = 0, e = 0;
                    if (i < nruns) {
                        const int2 run = runs[i];
                        s = run.x;
                        e = run.y;
                        while (s_off[ry_i + 1] <= i) ++ry_i;
                    }
                    const int8_t* row = m + (size_t)(y0 + ry_i) * stride;
                    int vs = 0, ve = 0, ve1 = 0;
                    if (i < nruns) vs = row[s], ve = row[e], ve1 = row[e - 1];
                    const int cnt = min(kWarp, nruns - i0);
                    for (int q = 0; q < cnt; ++q) {
                        const int yq = __shfl_sync(0xffffffffu, ry_i, q), sq = __shfl_sync(0xffffffffu, s, q),
                                  eq = __shfl_sync(0xffffffffu, e, q);
                        if (yq != cur) cur = yq, mval = 0;  // lnbd starts on the frame at each row
                        int vsq = __shfl_sync(0xffffffffu, vs, q);
                        const bool traced = vsq == 1 && mval <= 0;
                        if (traced) {
                            const int y = y0 + yq, i0m = y * stride + sq;
                            if (lane == 0) {
                                const int len = contour_follow(m, stride, i0m, sq, y, true, nullptr, 0, 0, 0);
                                list[nc] = make_int2(i0m, len);
                            }
                            ++nc;
                            __syncwarp();
                            if (i < nruns) vs = row[s], ve = row[e], ve1 = row[e - 1];  // the trace marked the map
                            vsq = __shfl_sync(0xffffffffu, vs, q);
                        }
                        const int veq = __shfl_sync(0xffffffffu, ve, q), ve1q = __shfl_sync(0xffffffffu, ve1, q);
                        // lnbd: the last x of the run with a mark and a value change (the traced start itself excluded)
                        if (eq > sq && is_mark(veq) && veq != ve1q) {
                            mval = veq;
                        } else if (eq == sq) {
                            if (!traced && is_mark(vsq)) mval = vsq;
                        } else {
                            const int8_t* rq = m + (size_t)(y0 + yq) * stride;
                            const int lo = traced ? sq + 1 : sq;
                            for (int xh = eq; xh >= lo; xh -= kWarp) {
                                const int x = xh - lane;
                                const int v = x >= lo ? rq[x] : 0;
                                const bool hit = x >= lo && is_mark(v) && v != rq[x - 1];
                                const unsigned h = __ballot_sync(0xffffffffu, hit);
                                if (h) {
                                    mval = __shfl_sync(0xffffffffu, v, __ffs(h) - 1);
                                    break;
                                }
                            }
                        }
                    }
                }
                if (lane == 0) s_n = nc;
            }
            __syncthreads();
        }
        // C. outputs in descending start order: contour q of the output is list[n - 1 - q]
        const int n = s_n;
        if (tid == 0) s_carry = 0;
        __syncthreads();
        for (int q0 = 0; q0 < n; q0 += kContourThreads) {
            const int q = q0 + tid;
            const int2 cq = q < n ? list[n - 1 - q] : make_int2(0, 0);
            // exclusive prefix of the lengths over the output order
            long long v = cq.y;
#pragma unroll
            for (int d = 1; d < kWarp; d <<= 1) {
                const long long u = __shfl_up_sync(0xffffffffu, v, d);
                if (lane >= d) v += u;
            }
            if (lane == kWarp - 1) s_wsum[warp] = v;
            __syncthreads();
            long long before = s_carry, chunk = 0;
            for (int w = 0; w < kContourWarps; ++w) {
                before += w < warp ? s_wsum[w] : 0;
                chunk += s_wsum[w];
            }
            const long long off = before + v - cq.y;
            if (q < n) {
                if (q < a.max_contours) a.lengths[canvas_id * a.max_contours + q] = cq.y;
                if (off < a.max_points) {
                    const int y = cq.x / stride, x = cq.x - y * stride;
                    contour_follow(m, stride, cq.x, x, y, false, a.points + (canvas_id * a.max_points + off) * 2,
                                   (int)min((long long)cq.y, a.max_points - off), rx - 1, ry - 1);
                }
            }
            __syncthreads();
            if (tid == 0) s_carry += chunk;
            __syncthreads();
        }
        if (tid == 0) {
            a.counts[2 * canvas_id] = n;
            a.counts[2 * canvas_id + 1] = (int)s_carry;
        }
        __syncthreads();  // the slot is reused by the next canvas
    }
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
// dynamic shared memory of a canvas launch at most: 227 KB per CTA less a 1 KB margin for the kernel's static arrays
// (752 B today), so the limit does not move when they do.  The margin, not the hardware, makes 2408^2 the largest square
// net for a frame of a few pixels (2412^2 would need 231 552 B + 752 B, which an H100 could still launch).
constexpr size_t kSegMaxDynamicSmem = 227 * 1024 - 1024;

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
    const int x_lo = max(rect[0], 0), x_hi = (int)max(0LL, min((long long)rect[0] + rect[2], (long long)im.img_w));
    const int y_lo = max(rect[1], 0), y_hi = (int)max(0LL, min((long long)rect[1] + rect[3], (long long)im.img_h));
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
        int dx_lo, dx_hi, dy_lo, dy_hi;
        downscale_rect(a.variant, det, a.net_w, a.net_h, a.mw, a.mh, dx_lo, dx_hi, dy_lo, dy_hi);
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
// cv::resize throws), more than INT_MAX CTAs, or caps that need more than kSegMaxDynamicSmem (a net of more than 2408^2
// for a frame of a few pixels: M rows x crop width grows with the net).
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
    return smem > kSegMaxDynamicSmem ? TRTX_ERR_UNSUPPORTED : TRTX_OK;
}

// Per-row geometry post-processes: the per-detection host stage the reference runs on one core after a D2H copy, for a
// batch of frames of any sizes.  One CTA of kRowsThreads per frame, one launch per <= 64 frames, no workspace, no atomics.
// frame_rows() is the pass both kernels share; a small row policy says what differs:
//   Row::pass(d)            whether row d is used;
//   Row::geometry(d, g)     its integer geometry, Row::kGeo ints;
//   Row::value(d, g, e)     output float e of the row, from the row and its geometry.
// The CTA walks the first min(count, max_rows) rows in passes of kRowsThreads, one row per thread; a ballot per warp over
// pass() and a scan of the warps' counts give each used row its output slot (input order); the owning thread computes the
// geometry into shared memory; then the whole CTA writes the pass's rows as one contiguous run of floats (coalesced),
// calling value() per float.  Rows past the used count are zeroed, and float 0 gets the count.
constexpr int kRowsThreads = 256;  // rows per pass
constexpr int kRowsWarps = kRowsThreads / kWarp;
constexpr int kPoseMaxKpts = 64;

// What every launch of a per-row post-process carries besides the policy's own parameters.
struct RowFrames {
    FrameSizes sizes;   // its base next to row_floats: the prologue loads the two as one pair
    int row_floats, out_floats, max_rows;
    const float* dets;  // [B, 1 + max_rows * row_floats]
    float* rows;        // [B, 1 + max_rows * out_floats]
};

template <class Row, class Args>
__device__ __forceinline__ void frame_rows(const Args& args) {
    const RowFrames& a = args.f;
    __shared__ int s_src[kRowsThreads];               // input row of each used row of the pass, by output slot
    __shared__ int s_geo[kRowsThreads * Row::kGeo];   // its geometry
    __shared__ int s_warp[kRowsWarps];                // used rows per warp of the pass
    const int tid = threadIdx.x, lane = tid & (kWarp - 1), warp = tid / kWarp, b = a.sizes.base + blockIdx.x;
    const size_t R = (size_t)a.row_floats, F = (size_t)a.out_floats;
    const float* src = a.dets + (size_t)b * (1 + (size_t)a.max_rows * R);
    float* out = a.rows + (size_t)b * (1 + (size_t)a.max_rows * F);
    const int n = min(max((int)src[0], 0), a.max_rows);
    const Row row(args, blockIdx.x);  // after the count's load, so that the policy's set-up overlaps it
    int kept = 0;                     // rows written by the earlier passes
    for (int i0 = 0; i0 < n; i0 += kRowsThreads) {
        const int i = i0 + tid;
        const float* d = src + 1 + (size_t)i * R;
        const bool keep = i < n && row.pass(d);
        const unsigned m = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) s_warp[warp] = __popc(m);
        __syncthreads();
        int before = 0, total = 0;
#pragma unroll
        for (int w = 0; w < kRowsWarps; ++w) {
            const int c = s_warp[w];
            before += w < warp ? c : 0;
            total += c;
        }
        if (keep) {
            const int slot = before + __popc(m & ((1u << lane) - 1u));
            int g[Row::kGeo];
            row.geometry(d, g);
            s_src[slot] = i;
#pragma unroll
            for (int e = 0; e < Row::kGeo; ++e) s_geo[slot * Row::kGeo + e] = g[e];
        }
        __syncthreads();
        const size_t run = (size_t)total * F;
        float* o = out + 1 + (size_t)kept * F;
#pragma unroll 4
        for (size_t f = tid; f < run; f += kRowsThreads) {
            const int r = (int)(f / F), e = (int)(f - (size_t)r * F);
            o[f] = row.value(src + 1 + (size_t)s_src[r] * R, s_geo + r * Row::kGeo, e);
        }
        kept += total;
        __syncthreads();  // the next pass reuses the shared arrays
    }
    const size_t end = 1 + (size_t)a.max_rows * F;
    for (size_t f = 1 + (size_t)kept * F + tid; f < end; f += kRowsThreads) out[f] = 0.0f;
    if (tid == 0) out[0] = (float)kept;
}

// Pose and oriented boxes: draw_bbox_keypoints_line's get_rect_adapt_landmark (yolov8/src/postprocess.cpp:173-205) and
// draw_bbox_obb's get_corner (:474-507).  Pose rows: the rectangle (yolo_get_rect), conf, class, each keypoint coordinate
// mapped with yolo_map_landmark; OBB rows: the four corners (yolo_get_corner), conf, class.  The NMS-free yolo26 rows have
// no keep column and use every row.
struct PoseObbArgs {
    RowFrames f;
    int pose, nms_free, net_w, net_h, extra_offset, num_kpts;
};

struct PoseObbRow {
    static constexpr int kGeo = 8;  // the rectangle (pose: 4 ints) or the corners (OBB: 8 ints)
    const PoseObbArgs& a;
    int img_w, img_h;
    YoloLetterbox lb;
    int geo;  // floats of the output row before conf and class
    __device__ PoseObbRow(const PoseObbArgs& args, int j)
        : a(args), img_w(args.f.sizes.w[j]), img_h(args.f.sizes.h[j]),
          lb(yolo_letterbox(args.net_w, args.net_h, img_w, img_h)), geo(args.pose ? 4 : 8) {}
    // process_decode_ptr_host: `int keep_flag = ...; if (keep_flag == 1)`; yolo26's batch_decode_obb takes every row
    __device__ bool pass(const float* d) const { return a.nms_free || (int)d[6] == 1; }
    __device__ void geometry(const float* d, int g[8]) const {
#pragma unroll
        for (int e = 0; e < 8; ++e) g[e] = 0;
        if (a.pose)
            yolo_get_rect(TRTX_YOLO_V8, a.net_w, a.net_h, img_w, img_h, d, g);  // {0, 0, 0, 0} where undefined
        else
            yolo_get_corner(a.net_w, a.net_h, img_w, img_h, d, d[a.extra_offset], g);
    }
    __device__ float value(const float* d, const int* g, int e) const {
        if (e < geo) return (float)g[e];
        if (e < geo + 2) return d[4 + e - geo];  // conf, class
        const int k = e - 6;                     // keypoint float: x, y, conf
        const int c = k % 3;
        const float x = d[a.extra_offset + k];
        return c == 2 ? x : yolo_map_landmark(lb, c, x);
    }
};

__global__ void __launch_bounds__(kRowsThreads) pose_obb_rows_kernel(const __grid_constant__ PoseObbArgs a) {
    frame_rows<PoseObbRow>(a);
}

// Faces: the loop of retinaface/retina_r50.cpp:373-388 (retinafaceAntiCov/retinafaceAntiCov.cpp:540-552 without its
// threshold) over the compact NMS rows (box4, conf, class, keep, extras...): kept rows with !(conf < conf_thresh) become
// (x, y, w, h, conf, 10 landmark floats[, mask_conf]) by retina_get_rect_adapt_landmark.
struct FaceArgs {
    RowFrames f;
    int in_w, in_h, lmk_offset;
    float conf_thresh;
};

struct FaceRow {
    static constexpr int kGeo = 4;  // the rectangle
    const FaceArgs& a;
    YoloLetterbox lb;
    __device__ FaceRow(const FaceArgs& args, int j)
        : a(args), lb(yolo_letterbox(args.in_w, args.in_h, args.f.sizes.w[j], args.f.sizes.h[j])) {}
    // `if (res[j].class_confidence < CONF_THRESH) continue;`: a NaN confidence is kept
    __device__ bool pass(const float* d) const { return (int)d[6] == 1 && !(d[4] < a.conf_thresh); }
    __device__ void geometry(const float* d, int g[4]) const { retina_get_rect(lb, d, g); }
    __device__ float value(const float* d, const int* g, int e) const {
        if (e < 4) return (float)g[e];
        if (e == 4) return d[4];
        const int k = e - 5;  // landmark float, then mask_conf
        const float x = d[a.lmk_offset + k];
        return k < 10 ? yolo_map_landmark(lb, k & 1, x) : x;
    }
};

__global__ void __launch_bounds__(kRowsThreads) face_rows_kernel(const __grid_constant__ FaceArgs a) {
    frame_rows<FaceRow>(a);
}

// YOLOP: the driver's nms() result mapped by YOLOP's own get_rect (yolop/common.hpp:13-37, yolop.cpp:129-146) into
// (x, y, w, h, conf, class) rows.
struct YolopRowsArgs {
    RowFrames f;
    int net_w, net_h;
};

struct YolopRow {
    static constexpr int kGeo = 4;  // the rectangle
    YoloLetterbox lb;
    __device__ YolopRow(const YolopRowsArgs& args, int j) : lb(yolo_letterbox(args.net_w, args.net_h, args.f.sizes.w[j], args.f.sizes.h[j])) {}
    __device__ bool pass(const float* d) const { return (int)d[6] == 1; }  // every row of a greedy NMS output
    __device__ void geometry(const float* d, int g[4]) const { yolop_get_rect(lb, d, g); }
    __device__ float value(const float* d, const int* g, int e) const { return e < 4 ? (float)g[e] : d[e]; }  // conf, class
};

__global__ void __launch_bounds__(kRowsThreads) yolop_rows_kernel(const __grid_constant__ YolopRowsArgs a) {
    frame_rows<YolopRow>(a);
}

// yolov10: get_topk (yolov10/src/postprocess.cpp:35-44) keeps the plugin rows above the threshold, in plugin order, with no
// NMS; draw_bbox maps them by get_rect (:3-33, yolov8's) into (x, y, w, h, conf, class) rows.
struct TopkArgs {
    RowFrames f;
    int variant, net_w, net_h;
    float conf_thresh;
};

struct TopkRow {
    static constexpr int kGeo = 4;  // the rectangle
    const TopkArgs& a;
    int img_w, img_h;
    __device__ TopkRow(const TopkArgs& args, int j) : a(args), img_w(args.f.sizes.w[j]), img_h(args.f.sizes.h[j]) {}
    // `if (output[1 + det_size * i + 4] <= conf_thresh) continue;`: a NaN confidence is kept
    __device__ bool pass(const float* d) const { return !(d[4] <= a.conf_thresh); }
    // the variant as a literal in each call, so that only its own branch of yolo_get_rect is compiled
    __device__ void geometry(const float* d, int g[4]) const {
        if (a.variant == TRTX_YOLO_V8)
            yolo_get_rect(TRTX_YOLO_V8, a.net_w, a.net_h, img_w, img_h, d, g);
        else
            yolo_get_rect(TRTX_YOLO_V5, a.net_w, a.net_h, img_w, img_h, d, g);
    }
    __device__ float value(const float* d, const int* g, int e) const { return e < 4 ? (float)g[e] : d[e]; }  // conf, class
};

__global__ void __launch_bounds__(kRowsThreads) topk_rows_kernel(const __grid_constant__ TopkArgs a) {
    frame_rows<TopkRow>(a);
}

// YOLOP's labels (yolop/yolop.cpp:148-169): the drivable-area and lane maps resized to the frame with cv::resize(INTER_NEAREST)
// and combined per pixel, 2 = lane, else 1 = drivable area, else 0, into the frame's u8 canvas.  Bound by the canvas writes.
// A CTA owns a band of kLabelBand canvas rows of one frame (grid: bands x frames):
//   1. the nearest source column of every canvas column (sx, uint16 in shared memory) and the map row of every band row;
//      sy is non-decreasing in y, so the band's distinct map rows are consecutive;
//   2. the label of every map pixel of those rows, from the two int32 maps (small enough to stay in L2), as bytes in shared
//      memory;
//   3. each warp stages its row's bytes in shared memory, then writes the row with 16-byte stores (a head of 0..15 bytes up to
//      the first 16-byte boundary and a tail of 0..15 bytes are scalar: pitch and base may be anything); bytes past img_w are
//      not touched.
constexpr int kLabelBand = 8;  // canvas rows per CTA: small bands keep every SM busy at b8
constexpr int kLabelThreads = 256;
constexpr int kLabelWarps = kLabelThreads / kWarp;

struct YolopLabelFrame {
    uint8_t* canvas;
    double ifx, ify;  // cv::resize: 1. / ((double)dsize / ssize) per axis
    int img_w, img_h, pitch;
};
struct YolopLabelArgs {
    YolopLabelFrame fr[kMaxFrames];
    const int32_t* seg;   // [B, map_h, map_w]
    const int32_t* lane;
    int map_w, map_h, base;
    int sx_bytes;         // the sx table's bytes in dynamic shared memory (the widest frame, rounded to 16)
    int stage_bytes;      // bytes of a warp's staged row: the widest frame + 15, rounded to 16
};

__global__ void __launch_bounds__(kLabelThreads) yolop_label_kernel(const __grid_constant__ YolopLabelArgs a) {
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ int s_srow[kLabelBand];  // map row of each distinct slot
    __shared__ int s_slot[kLabelBand];  // slot of each band row
    __shared__ int s_nslots;
    const YolopLabelFrame& f = a.fr[blockIdx.y];
    const int y0 = blockIdx.x * kLabelBand;
    if (y0 >= f.img_h) return;  // uniform: a band past this frame's height (bands are sized for the tallest frame)
    const int rows = min(kLabelBand, f.img_h - y0), tid = threadIdx.x;
    const int warp = tid / kWarp, l = tid & (kWarp - 1);
    uint16_t* sx = reinterpret_cast<uint16_t*>(smem);
    uint8_t* lab = smem + a.sx_bytes;  // [slots][map_w], then the warps' staged rows
    if (warp == 0) {  // lane k: band row k; sy is non-decreasing, so a new slot starts where it changes
        const int sy = l < rows ? min((int)floor(__dmul_rn((double)(y0 + l), f.ify)), a.map_h - 1) : INT_MAX;
        const int prev = __shfl_up_sync(0xffffffffu, sy, 1);
        const unsigned starts = __ballot_sync(0xffffffffu, l < rows && (l == 0 || sy != prev));
        const int slot = __popc(starts & (0xffffffffu >> (31 - l))) - 1;
        if (l < rows) {
            s_slot[l] = slot;
            if ((starts >> l) & 1u) s_srow[slot] = sy;
        }
        if (l == 0) s_nslots = __popc(starts);
    }
    for (int x = tid; x < f.img_w; x += kLabelThreads) sx[x] = (uint16_t)min((int)floor(__dmul_rn((double)x, f.ifx)), a.map_w - 1);
    __syncthreads();
    const size_t map = (size_t)a.map_w * a.map_h, b = (size_t)(a.base + blockIdx.y);
    const int32_t* seg = a.seg + b * map;
    const int32_t* lane = a.lane + b * map;
    const int items = s_nslots * a.map_w;
#pragma unroll 4
    for (int i = tid; i < items; i += kLabelThreads) {
        const int s = i / a.map_w, m = i - s * a.map_w;
        const size_t o = (size_t)s_srow[s] * a.map_w + m;
        lab[i] = __ldg(lane + o) != 0 ? 2 : (__ldg(seg + o) != 0 ? 1 : 0);
    }
    __syncthreads();
    // each warp writes rows warp, warp + kLabelWarps, ...: its bytes staged so that the 16-byte runs of the canvas row are
    // 16-byte aligned in shared memory too (byte x at x + pad)
    uint8_t* stage = lab + ((kLabelBand * a.map_w + 15) & ~15) + warp * a.stage_bytes;
    const int w = f.img_w;
    for (int k = warp; k < rows; k += kLabelWarps) {
        const uint8_t* L = lab + s_slot[k] * a.map_w;
        uint8_t* row = f.canvas + (size_t)(y0 + k) * (size_t)f.pitch;
        const int head = min((int)((16u - (unsigned)(reinterpret_cast<uintptr_t>(row) & 15u)) & 15u), w);
        const int nvec = (w - head) >> 4, tail0 = head + 16 * nvec, pad = (16 - head) & 15;
        for (int x = l; x < w; x += kWarp) stage[x + pad] = L[sx[x]];  // consecutive lanes, consecutive x: no bank conflicts
        __syncwarp();
        if (l < head) row[l] = stage[l + pad];
        if (tail0 + l < w) row[tail0 + l] = stage[tail0 + l + pad];
        for (int q = l; q < nvec; q += kWarp)
            *reinterpret_cast<uint4*>(row + head + 16 * q) = *reinterpret_cast<const uint4*>(stage + head + pad + 16 * q);
        __syncwarp();  // the next row reuses the stage
    }
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

// The slots of a trtx_rcnn_contours_enqueue call and the bytes of one (sized for its largest frame); TRTX_ERR_INVALID /
// TRTX_ERR_UNSUPPORTED as documented there, in two passes over the frames so that TRTX_ERR_INVALID wins.
static int contour_plan(const trtx_rcnn_post_params* p, const trtx_frame* frames, int batch, int& slots,
                        long long& map_bytes, long long& list_bytes, long long& slot_bytes) {
    if (!p || !frames || batch <= 0 || p->detections_per_im <= 0 || p->max_masks <= 0) return TRTX_ERR_INVALID;
    for (int i = 0; i < batch; ++i) {
        const trtx_frame& d = frames[i];
        if (!d.masks_dev || d.img_w <= 0 || d.img_h <= 0 || d.pitch < d.img_w) return TRTX_ERR_INVALID;
    }
    long long band_bytes = 0;
    map_bytes = list_bytes = 0;
    for (int i = 0; i < batch; ++i) {
        const trtx_frame& d = frames[i];
        if ((long long)(d.img_w + 2) * (d.img_h + 2) > (1LL << 29)) return TRTX_ERR_UNSUPPORTED;
        long long mb, lb, bb;
        contour_regions(d.img_w, d.img_h, mb, lb, bb);
        map_bytes = max(map_bytes, mb);
        list_bytes = max(list_bytes, lb);
        band_bytes = max(band_bytes, bb);
    }
    slot_bytes = (map_bytes + list_bytes + band_bytes + 255) / 256 * 256;
    slots = (int)min((long long)min(batch, kMaxFrames) * p->max_masks, (long long)kContourCtas);
    return TRTX_OK;
}

TRTX_API size_t trtx_rcnn_contours_workspace_size(const trtx_rcnn_post_params* p, const trtx_frame* images_host, int batch) {
    int slots;
    long long map_bytes, list_bytes, slot_bytes;
    if (contour_plan(p, images_host, batch, slots, map_bytes, list_bytes, slot_bytes)) return 0;
    return (size_t)slots * (size_t)slot_bytes;
}

TRTX_API int trtx_rcnn_contours_enqueue(const trtx_rcnn_post_params* p, const trtx_frame* images_host, int batch,
                                        const float* rows_dev, int max_contours, int max_points, int32_t* counts_dev,
                                        int32_t* lengths_dev, int32_t* points_dev, void* workspace_dev,
                                        size_t workspace_bytes, trtx_stream_t stream) {
    if (!rows_dev || !counts_dev || !lengths_dev || !points_dev || !workspace_dev || max_contours <= 0 || max_points <= 0)
        return TRTX_ERR_INVALID;
    if (reinterpret_cast<uintptr_t>(workspace_dev) & 15) return TRTX_ERR_INVALID;
    int slots;
    long long map_bytes, list_bytes, slot_bytes;
    int rc = contour_plan(p, images_host, batch, slots, map_bytes, list_bytes, slot_bytes);
    if (rc) return rc;
    if (workspace_bytes < (size_t)slots * (size_t)slot_bytes) return TRTX_ERR_WORKSPACE;
    ContourArgs a;
    a.rows = rows_dev;
    a.counts = counts_dev;
    a.lengths = lengths_dev;
    a.points = points_dev;
    a.work = static_cast<uint8_t*>(workspace_dev);
    a.slot_bytes = (size_t)slot_bytes;
    a.map_bytes = map_bytes;
    a.list_bytes = list_bytes;
    a.dets = p->detections_per_im;
    a.max_masks = p->max_masks;
    a.max_contours = max_contours;
    a.max_points = max_points;
    if ((rc = opt_in_smem(rcnn_contours_kernel, kContourSmem))) return rc;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    for (int i0 = 0; i0 < batch; i0 += kMaxFrames) {
        const int n = min(batch - i0, kMaxFrames);
        for (int j = 0; j < n; ++j) {
            const trtx_frame& d = images_host[i0 + j];
            a.f[j] = ContourFrame{d.masks_dev, d.img_w, d.img_h, d.pitch};
        }
        a.base = i0;
        a.n_images = n;
        rcnn_contours_kernel<<<(unsigned)min(n * p->max_masks, kContourCtas), kContourThreads, kContourSmem, st>>>(a);
        if ((rc = check_launch())) return rc;
    }
    return TRTX_OK;
}

TRTX_API int trtx_yolo_seg_postprocess_enqueue(const trtx_mask_params* p, const trtx_frame* images_host, int batch,
                                               const float* proto_dev, const float* dets_dev, int max_rows,
                                               float* rows_dev, trtx_stream_t stream) {
    if (!p || !images_host || batch <= 0 || !dets_dev || !rows_dev || max_rows <= 0) return TRTX_ERR_INVALID;
    // TRTX_YOLO_V3 and TRTX_RECT_YOLOV3_SPP: rectangles only (their models have no masks)
    const bool rect_only = p->variant == TRTX_YOLO_V3 || p->variant == TRTX_RECT_YOLOV3_SPP;
    if (p->variant != TRTX_YOLO_V8 && p->variant != TRTX_YOLO_V5 && !rect_only) return TRTX_ERR_INVALID;
    if (p->net_w <= 0 || p->net_h <= 0 || p->row_floats < kSegRowFloats) return TRTX_ERR_INVALID;
    if (p->variant == TRTX_RECT_YOLOV3_SPP && p->net_w != p->net_h) return TRTX_ERR_INVALID;
    bool masks;
    int rc = check_frames(images_host, batch, masks);
    if (rc) return rc;
    if (masks) {  // trtx_process_mask_enqueue's checks
        if (rect_only || !proto_dev) return TRTX_ERR_INVALID;
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
    if ((rc = opt_in_smem(seg_canvas_kernel, smem_max))) return rc;
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

TRTX_API int trtx_yolo_seg_launch_caps(const trtx_mask_params* p, const trtx_frame* images_host, int batch, int32_t caps[5]) {
    if (!p || !images_host || !caps || batch <= 0) return TRTX_ERR_INVALID;
    if (p->net_w <= 0 || p->net_h <= 0 || p->mask_w <= 0 || p->mask_h <= 0) return TRTX_ERR_INVALID;
    for (int i = 0; i < batch; ++i)
        if (images_host[i].img_w <= 0 || images_host[i].img_h <= 0) return TRTX_ERR_INVALID;
    SegArgs a;
    int ctas, rc;
    size_t smem;
    caps[0] = caps[1] = caps[2] = caps[3] = caps[4] = 0;
    for (int i0 = 0; i0 < batch; i0 += kMaxFrames) {  // the launches trtx_yolo_seg_postprocess_enqueue makes
        a.lx_cap = 0;  // set last: still 0 where a frame is refused before
        smem = 0;
        rc = seg_fill_frames(p, images_host, i0, min(batch - i0, kMaxFrames), true, a, ctas, smem);
        caps[0] = max(caps[0], a.y_cap);
        caps[1] = max(caps[1], a.ly_cap);
        caps[2] = max(caps[2], a.x_cap);
        caps[3] = max(caps[3], a.lx_cap);
        caps[4] = max(caps[4], (int32_t)min(smem, (size_t)INT32_MAX));
        if (rc) return rc;
    }
    return TRTX_OK;
}

TRTX_API int trtx_yolo_pose_obb_postprocess_enqueue(const trtx_pose_obb_params* p, const int32_t* frame_wh_host, int batch,
                                                    const float* dets_dev, int max_rows, float* rows_dev,
                                                    trtx_stream_t stream) {
    if (!p || !frame_wh_host || batch <= 0 || !dets_dev || !rows_dev || max_rows <= 0) return TRTX_ERR_INVALID;
    if (p->task != TRTX_TASK_POSE && p->task != TRTX_TASK_OBB && p->task != TRTX_TASK_OBB_NMS_FREE) return TRTX_ERR_INVALID;
    if (p->net_w <= 0 || p->net_h <= 0 || p->row_floats < 7 || p->extra_offset < 0) return TRTX_ERR_INVALID;
    const bool pose = p->task == TRTX_TASK_POSE, nms_free = p->task == TRTX_TASK_OBB_NMS_FREE;
    if (pose && (p->num_kpts < 0 || p->num_kpts > kPoseMaxKpts || p->extra_offset + 3 * p->num_kpts > p->row_floats))
        return TRTX_ERR_INVALID;
    if (!pose && p->extra_offset >= p->row_floats) return TRTX_ERR_INVALID;
    // the NMS-free plugin row ends with the angle (yolo26/include/types.h: Detection::angle)
    if (nms_free && p->extra_offset != p->row_floats - 1) return TRTX_ERR_INVALID;
    if (!frames_valid(frame_wh_host, batch)) return TRTX_ERR_INVALID;
    PoseObbArgs a;
    a.f.dets = dets_dev;
    a.f.rows = rows_dev;
    a.f.row_floats = p->row_floats;
    a.f.out_floats = pose ? 6 + 3 * p->num_kpts : 10;
    a.f.max_rows = max_rows;
    a.pose = pose;
    a.nms_free = nms_free;
    a.net_w = p->net_w;
    a.net_h = p->net_h;
    a.extra_offset = p->extra_offset;
    a.num_kpts = pose ? p->num_kpts : 0;
    return launch_frames(pose_obb_rows_kernel, a, a.f.sizes, batch, kRowsThreads, 0, static_cast<cudaStream_t>(stream),
                         frame_wh(frame_wh_host));
}

TRTX_API int trtx_retina_postprocess_enqueue(const trtx_face_post_params* p, const int32_t* frame_wh_host, int batch,
                                             const float* dets_dev, int max_rows, float* rows_dev, trtx_stream_t stream) {
    if (!p || !frame_wh_host || batch <= 0 || !dets_dev || !rows_dev || max_rows <= 0) return TRTX_ERR_INVALID;
    if (p->variant != TRTX_RETINA_FACE && p->variant != TRTX_RETINA_ANTICOV) return TRTX_ERR_INVALID;
    const int extras = p->variant == TRTX_RETINA_ANTICOV ? 11 : 10;  // the landmarks (+ mask_confidence)
    if (p->in_w <= 0 || p->in_h <= 0 || p->row_floats < 7 || p->lmk_offset < 0 || p->lmk_offset > p->row_floats - extras)
        return TRTX_ERR_INVALID;
    if (!frames_valid(frame_wh_host, batch)) return TRTX_ERR_INVALID;
    FaceArgs a;
    a.f.dets = dets_dev;
    a.f.rows = rows_dev;
    a.f.row_floats = p->row_floats;
    a.f.out_floats = 5 + extras;
    a.f.max_rows = max_rows;
    a.in_w = p->in_w;
    a.in_h = p->in_h;
    a.lmk_offset = p->lmk_offset;
    a.conf_thresh = p->conf_thresh;
    return launch_frames(face_rows_kernel, a, a.f.sizes, batch, kRowsThreads, 0, static_cast<cudaStream_t>(stream),
                         frame_wh(frame_wh_host));
}

TRTX_API int trtx_yolo_topk_postprocess_enqueue(const trtx_yolo_topk_params* p, const int32_t* frame_wh_host, int batch,
                                                const float* dets_dev, int max_rows, float* rows_dev, trtx_stream_t stream) {
    if (!p || !frame_wh_host || batch <= 0 || !dets_dev || !rows_dev || max_rows <= 0) return TRTX_ERR_INVALID;
    if (p->variant != TRTX_YOLO_V8 && p->variant != TRTX_YOLO_V5) return TRTX_ERR_INVALID;
    if (p->net_w <= 0 || p->net_h <= 0 || p->row_floats < 6) return TRTX_ERR_INVALID;
    if (!frames_valid(frame_wh_host, batch)) return TRTX_ERR_INVALID;
    TopkArgs a;
    a.f.dets = dets_dev;
    a.f.rows = rows_dev;
    a.f.row_floats = p->row_floats;
    a.f.out_floats = 6;
    a.f.max_rows = max_rows;
    a.variant = p->variant;
    a.net_w = p->net_w;
    a.net_h = p->net_h;
    a.conf_thresh = p->conf_thresh;
    return launch_frames(topk_rows_kernel, a, a.f.sizes, batch, kRowsThreads, 0, static_cast<cudaStream_t>(stream),
                         frame_wh(frame_wh_host));
}

TRTX_API int trtx_yolop_postprocess_enqueue(const trtx_yolop_post_params* p, const trtx_frame* frames_host, int batch,
                                            const float* dets_dev, int max_rows, const int32_t* seg_dev,
                                            const int32_t* lane_dev, float* rows_dev, trtx_stream_t stream) {
    if (!p || !frames_host || batch <= 0 || !dets_dev || !rows_dev || max_rows <= 0) return TRTX_ERR_INVALID;
    if (p->net_w <= 0 || p->net_h <= 0 || p->map_w <= 0 || p->map_h <= 0 || p->row_floats < 7) return TRTX_ERR_INVALID;
    const bool labels = frames_host[0].masks_dev != nullptr;
    if (labels && (!seg_dev || !lane_dev)) return TRTX_ERR_INVALID;
    int w_max = 0;
    for (int i = 0; i < batch; ++i) {
        const trtx_frame& d = frames_host[i];
        if (d.img_w <= 0 || d.img_h <= 0 || (d.masks_dev != nullptr) != labels) return TRTX_ERR_INVALID;
        if (labels && d.pitch < d.img_w) return TRTX_ERR_INVALID;
        w_max = max(w_max, d.img_w);
    }
    // the sx table (uint16, so map_w <= 65536), the label rows of a band and the warps' staged rows in shared memory
    const int sx_bytes = (int)align_up(2 * (size_t)w_max, 16), stage_bytes = (int)align_up((size_t)w_max + 15, 16);
    const size_t smem = (size_t)sx_bytes + align_up((size_t)kLabelBand * p->map_w, 16) + (size_t)kLabelWarps * stage_bytes;
    if (labels && smem > 227 * 1024) return TRTX_ERR_UNSUPPORTED;
    int rc = labels ? opt_in_smem(yolop_label_kernel, smem) : TRTX_OK;
    if (rc) return rc;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    YolopRowsArgs r;
    r.f.dets = dets_dev;
    r.f.rows = rows_dev;
    r.f.row_floats = p->row_floats;
    r.f.out_floats = 6;
    r.f.max_rows = max_rows;
    r.net_w = p->net_w;
    r.net_h = p->net_h;
    rc = launch_frames(yolop_rows_kernel, r, r.f.sizes, batch, kRowsThreads, 0, st,
                       [&](int i, int& w, int& h) { w = frames_host[i].img_w, h = frames_host[i].img_h; });
    if (rc || !labels) return rc;
    YolopLabelArgs a;
    a.seg = seg_dev;
    a.lane = lane_dev;
    a.map_w = p->map_w;
    a.map_h = p->map_h;
    a.sx_bytes = sx_bytes;
    a.stage_bytes = stage_bytes;
    for (int i0 = 0; i0 < batch; i0 += kMaxFrames) {
        const int n = min(batch - i0, kMaxFrames);
        int bands = 0;
        a.base = i0;
        for (int j = 0; j < n; ++j) {
            const trtx_frame& d = frames_host[i0 + j];
            YolopLabelFrame& f = a.fr[j];
            f.canvas = d.masks_dev;
            f.img_w = d.img_w;
            f.img_h = d.img_h;
            f.pitch = d.pitch;
            f.ifx = 1. / ((double)d.img_w / p->map_w);
            f.ify = 1. / ((double)d.img_h / p->map_h);
            bands = max(bands, (d.img_h + kLabelBand - 1) / kLabelBand);
        }
        yolop_label_kernel<<<dim3(bands, n), kLabelThreads, smem, st>>>(a);
        if ((rc = check_launch())) return rc;
    }
    return TRTX_OK;
}

}  // extern "C"
