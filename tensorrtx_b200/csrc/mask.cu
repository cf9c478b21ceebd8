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
        const float h0 = __fadd_rn(__fmul_rn(__ldg(r0 + sx), a0), __fmul_rn(__ldg(r0 + sx1), a1));
        const float h1 = __fadd_rn(__fmul_rn(__ldg(r1 + sx), a0), __fmul_rn(__ldg(r1 + sx1), a1));
        o[k] = __fadd_rn(__fmul_rn(h0, b0), __fmul_rn(h1, b1));
    }
    float* dst = a.out + (size_t)blockIdx.z * a.img_h * a.img_w + (size_t)oy * a.img_w + ox0;
    if (ox0 + 3 < a.img_w && (reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
        *reinterpret_cast<float4*>(dst) = make_float4(o[0], o[1], o[2], o[3]);
    } else {
        for (int k = 0; k < 4 && ox0 + k < a.img_w; ++k) dst[k] = o[k];
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

}  // extern "C"
