// preprocess.cu -- batched letterbox warp-affine + BGR->RGB + /255 + HWC->CHW (+fp16) for sm_90a.
// Replaces warpaffine_kernel / cuda_preprocess / cuda_batch_preprocess, yolov8/src/preprocess.cu:7-127
// (identical bodies in yolov5/7/9/10/11/12/13/26), which launch once per image and synchronise the
// stream after every image (:119-127).  Here: ONE launch for the whole batch, per-image descriptors
// and affine matrices in the kernel parameter block (no H2D copy of metadata); a warp covers 32
// adjacent destination columns and every thread produces a strip of rows of its column.  Measured and
// rejected: 4 adjacent pixels per lane (L1 sector-bound), staging the source band in shared
// memory (2x slower).  Sources that are only translated / padded into the network input (scale 1, e.g. 640x640 -> 640x640)
// take letterbox_unit_kernel instead: full-width destination row bands whose source rows arrive by TMA (see below).
//
// Roofline: HBM-bound; algorithmic bytes per image = src_w*src_h*3 (u8 read once) +
// 3*dst_w*dst_h*sizeof(out) (SURVEY 8d: 6 144 000 B for 640x640 -> 640x640 fp32).
//
// Arithmetic follows the reference kernel statement by statement (including its `+0.5f` source
// offset without a matching `-0.5f`, preprocess.cu:22-23) and, like the reference's own nvcc build,
// leaves the bilinear sums to the default FMA contraction, which both paths of letterbox_kernel and the reference
// evaluate as fmaf(w4, v4, fmaf(w3, v3, fmaf(w1, v1, w2 * v2))).  The CPU oracle's contracted warpaffine
// (oracle/trtx_oracle.c) restates exactly that: it is the bit-exact expectation for every output of this file's
// letterbox (tests/test_letterbox_paths_gpu.py), fp16 outputs being its fp32 value rounded to nearest.
#include <limits.h>
#include <math.h>
#include <string.h>

#include "tma.cuh"

namespace trtx {

constexpr int kMaxImagesPerLaunch = 128;

struct PreImage {
    const uint8_t* src;
    int sw, sh, pitch;
    int dst_idx;  // image slot in dst
    float m[6];   // d2s
};
struct PreArgs {
    PreImage img[kMaxImagesPerLaunch];
    int dw, dh;
};

// x / 255.0f, correctly rounded, in 3 FP instructions instead of the IEEE division subroutine:
// q0 = x*r, e = fma(-255, q0, x), q = fma(e, r, q0) with r = RN(1/255).  Verified EXHAUSTIVELY against
// x/255.0f for every float in [0, 65536) (1.2e9 values, tools/verify_div255.c) -- bit-identical.
__device__ __forceinline__ float div255(float x) {
    const float r = 1.0f / 255.0f;
    const float q0 = __fmul_rn(x, r);
    return __fmaf_rn(__fmaf_rn(-255.0f, q0, x), r, q0);
}

// One thread = ONE destination column x kRowsPerThread destination rows; the 32 lanes of a warp are 32 adjacent
// columns, so a warp-level byte load spans 32 px * 3 B = 96 B = 3-4 sectors and the planar stores are 128 contiguous
// bytes per warp.  The kernel is bound by INSTRUCTION ISSUE (over a hundred SASS
// instructions per pixel before the fast path below), not by HBM, and a rolled, row-serial variant
// with fewer instructions was slower still (too few loads in flight): so everything is straight-line code that
// issues all of a strip's loads before the first use.
//   * the letterbox matrix has no rotation (m[1] = m[3] = -0.0f, preprocess.cu:99-104), so everything that depends on
//     the column only (src_x, x taps, horizontal weights, byte offsets, validity) is computed once per thread;
//   * the bilinear sum is written as the reference writes it and left to nvcc's default FMA contraction, exactly
//     like the reference's own build: the output is BIT-IDENTICAL to the reference kernel's
//     (tests/test_vs_reference_gpu.py::test_preprocess_vs_reference_kernel).

// u8 -> f32 without the conversion (XU) pipe: for 0 <= i < 2^23, 2^23 + i is exactly representable with i in the
// mantissa, so OR-ing i into the bits of 2^23 and subtracting 2^23 gives float(i) exactly (two full-rate instructions).
// The fast path converts every other sample this way so that neither the XU pipe nor the issue slots saturate.
__device__ __forceinline__ float u8_to_float_alu(uint32_t i) { return __uint_as_float(0x4B000000u | i) - 8388608.0f; }

constexpr int kRowsPerThread = 4;  // 8-row strips measured slower on an earlier GPU, not re-measured on H100 (tools/lb_probe.py)

// __launch_bounds__(256, 8): 32 registers -> 64 resident warps per SM.  The kernel is latency-bound once the instruction
// count is down, and occupancy is what hides it: fewer registers per thread measured faster (on an earlier GPU; not re-measured on H100).
template <typename OutT>
__global__ void __launch_bounds__(256, 8) letterbox_kernel(const __grid_constant__ PreArgs a, OutT* __restrict__ dst) {
    constexpr int R = kRowsPerThread;
    const int b = blockIdx.z;
    const PreImage& im = a.img[b];
    const int dx = blockIdx.x * blockDim.x + threadIdx.x;
    const int dy0 = (blockIdx.y * blockDim.y + threadIdx.y) * R;
    if (dx >= a.dw || dy0 >= a.dh) return;
    const size_t area = (size_t)a.dw * a.dh;
    OutT* base = dst + (size_t)im.dst_idx * 3 * area + (size_t)dy0 * a.dw + dx;
    const float cv = 128.0f;  // const_value_st (:115)
    const uint8_t* __restrict__ img = im.src;
    const int sw = im.sw, sh = im.sh;

    // preprocess.cu:22 (src_x), evaluated with the thread's first dy: m[1]*dy is +-0 for every dy
    const float src_x = im.m[0] * (float)dx + im.m[1] * (float)dy0 + im.m[2] + 0.5f;
    const bool x_out = src_x <= -1 || src_x >= sw;
    const int x_low = (int)floorf(src_x);
    const int x_high = x_low + 1;
    const float lx = src_x - (float)x_low, hx = 1 - lx;
    const bool xl = x_low >= 0, xh = x_high < sw;
    const float xm = im.m[3] * (float)dx;

    // bgr -> rgb, /255 (:64-74); planar stores, 128 B per warp and plane
    auto emit = [&](int r, float c0, float c1, float c2) {
        OutT* o = base + (size_t)r * a.dw;
        if constexpr (sizeof(OutT) == 4) {
            o[0] = div255(c2);
            o[area] = div255(c1);
            o[2 * area] = div255(c0);
        } else {
            o[0] = __float2half_rn(div255(c2));
            o[area] = __float2half_rn(div255(c1));
            o[2 * area] = __float2half_rn(div255(c0));
        }
    };

    float src_y[R];
    int y_low[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
        src_y[r] = xm + im.m[4] * (float)(dy0 + r) + im.m[5] + 0.5f;  // :23
        y_low[r] = (int)floorf(src_y[r]);
    }
    // Fast path (warp-uniform but for the image's left/right edge): a full strip whose rows step through CONSECUTIVE
    // source rows, all taps inside the image -- any letterbox that does not shrink the image, e.g. the 640x640 ->
    // 640x640 benchmark.  The R+1 source rows are loaded once (one address per row: the right tap is the next pixel)
    // and shared by neighbouring destination rows: (R+1)*6 loads and conversions instead of R*12, no clamps, no selects.
    bool fast = dy0 + R <= a.dh && xl && xh && y_low[0] >= 0 && y_low[0] + R < sh;
#pragma unroll
    for (int r = 1; r < R; ++r) fast = fast && y_low[r] == y_low[0] + r;
    if (fast) {
        const uint8_t* p = img + (size_t)y_low[0] * (size_t)im.pitch + (uint32_t)x_low * 3u;
        float t[R + 1][6];
#pragma unroll
        for (int s = 0; s <= R; ++s) {
#pragma unroll
            for (int k = 0; k < 6; ++k) {
                const uint32_t v = __ldg(p + k);
                t[s][k] = ((s * 6 + k) & 1) ? u8_to_float_alu(v) : (float)v;
            }
            p += im.pitch;
        }
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const float ly = src_y[r] - (float)y_low[r], hy = 1 - ly;
            const float w1 = hy * hx, w2 = hy * lx, w3 = ly * hx, w4 = ly * lx;
            // :59-61 (left-to-right; nvcc contracts to mul + 3 fma, as in the reference build)
            emit(r, w1 * t[r][0] + w2 * t[r][3] + w3 * t[r + 1][0] + w4 * t[r + 1][3],
                 w1 * t[r][1] + w2 * t[r][4] + w3 * t[r + 1][1] + w4 * t[r + 1][4],
                 w1 * t[r][2] + w2 * t[r][5] + w3 * t[r + 1][2] + w4 * t[r + 1][5]);
        }
        return;
    }

    // General path (borders, shrinking letterboxes): source coordinates are CLAMPED into the image and the 12 bytes
    // always loaded (one address per tap, channels through immediate offsets, no divergent border path); out-of-image
    // taps are then replaced by the border value with selects, which is what the reference's pointer redirection to
    // `const_value` does (preprocess.cu:38-57).
    const uint32_t o1 = (uint32_t)min(max(x_low, 0), sw - 1) * 3u, o2 = (uint32_t)min(max(x_high, 0), sw - 1) * 3u;
#pragma unroll
    for (int r = 0; r < R; ++r) {
        if (dy0 + r >= a.dh) break;
        float c0 = cv, c1 = cv, c2 = cv;
        if (!(x_out || src_y[r] <= -1 || src_y[r] >= sh)) {
            const int y_high = y_low[r] + 1;
            const float ly = src_y[r] - (float)y_low[r], hy = 1 - ly;
            const float w1 = hy * hx, w2 = hy * lx, w3 = ly * hx, w4 = ly * lx;
            const bool r0ok = y_low[r] >= 0, r1ok = y_high < sh;
            const uint32_t row0 = (uint32_t)max(y_low[r], 0) * (uint32_t)im.pitch;  // images < 4 GiB
            const uint32_t row1 = (uint32_t)min(y_high, sh - 1) * (uint32_t)im.pitch;
            const bool k1 = r0ok && xl, k2 = r0ok && xh, k3 = r1ok && xl, k4 = r1ok && xh;
            const uint8_t* p1 = img + (row0 + o1);
            const uint8_t* p2 = img + (row0 + o2);
            const uint8_t* p3 = img + (row1 + o1);
            const uint8_t* p4 = img + (row1 + o2);
            float v1[3], v2[3], v3[3], v4[3];
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const float t1 = (float)(uint32_t)__ldg(p1 + k);
                const float t2 = (float)(uint32_t)__ldg(p2 + k);
                const float t3 = (float)(uint32_t)__ldg(p3 + k);
                const float t4 = (float)(uint32_t)__ldg(p4 + k);
                v1[k] = k1 ? t1 : cv;
                v2[k] = k2 ? t2 : cv;
                v3[k] = k3 ? t3 : cv;
                v4[k] = k4 ? t4 : cv;
            }
            c0 = w1 * v1[0] + w2 * v2[0] + w3 * v3[0] + w4 * v4[0];
            c1 = w1 * v1[1] + w2 * v2[1] + w3 * v3[1] + w4 * v4[1];
            c2 = w1 * v1[2] + w2 * v2[2] + w3 * v3[2] + w4 * v4[2];
        }
        emit(r, c0, c1, c2);
    }
}


// =====================================================================================================================
// Unit-scale letterbox, streamed in full-width row bands (the 640x640 -> 640x640 benchmark and every source that fits the
// network input in one dimension: scale == 1, the image is only translated / padded).
//
// With scale == 1 the d2s matrix is {1, -0, tx, -0, 1, ty} with 2*tx, 2*ty integers (preprocess.cu:98-110), so for every
// destination pixel  x_low = dx + ox,  y_low = dy + oy  and the bilinear fractions lx, ly are image-wide constants in
// {0, 0.5}: the four weights are products of {0, 0.5, 1}, every product w*u8 and every partial sum of the reference's
// expression (preprocess.cu:59-61) is exact in fp32, hence the result does not depend on evaluation order or FMA
// contraction, and "tap outside the image -> 128" (preprocess.cu:38-57) also reproduces the fully-outside case
// (:25-30: the weights sum to exactly 1).  The kernel is therefore bit-identical to the reference by construction;
// tests assert array_equal against the reference's compiled kernel.
//
// The kernel is HBM-bound (4 output bytes per input byte for fp32) and streams at about the rate of a plain contiguous
// u8 -> fp32 expand of the same bytes (tools/lb_ceiling, DESIGN 8).  A CTA owns kUnitBand destination rows x ALL dw columns
// of one image: every plane of a CTA is one contiguous run of kUnitBand * dw outputs, every warp store instruction writes
// 512 contiguous bytes (32 lanes x 4 pixels x fp32), and the band's source window -- kUnitBand + 1 whole source rows --
// arrives by TMA tensor copies: a u8 tensor map over the image(s), boxes of [kUnitBoxBytes, kUnitBand + 1] laid side by side
// in shared memory (box k holds byte columns [256k, 256k + 256) of every window row).  Rows / columns outside the image
// arrive as zeros (hardware bounds check: no byte outside the image is read) and the taps there are replaced by 128 with
// selects.  Each thread produces 4 ADJACENT pixels x kUnitBand rows: per source row 4 conflict-free LDS.32 (15 bytes = 5 BGR
// pixels; lanes 12 bytes apart hit 32 distinct banks, and a box boundary moves the address by a multiple of 128 bytes),
// every byte converted once with one PRMT (byte -> mantissa of 2^23) + one FADD, a horizontal pass shared by the two
// destination rows that use the source row, and one 16-byte store per plane and row (8 bytes for fp16).  CTAs are
// short-lived (one band each, 10 KB of shared memory at 640 columns), so SMs free up for concurrent work as the grid drains.
constexpr int kUnitBand = 4;             // destination rows per CTA (8 measured slower)
constexpr int kUnitBoxBytes = 256;       // TMA inner box extent: the most one box may span
constexpr int kMaxUnitImages = 64;
constexpr int kUnitMaxThreads = 160;     // 640 columns = 160 threads x 4 pixels; wider inputs loop

struct UnitImage {
    int ox, oy;    // x_low(dx = 0), y_low(dy = 0)
    int sw, sh;
    int map, z;    // tensor map index, image coordinate inside that map
    int dst_idx;
    float lx, ly;  // bilinear fractions (0 or 0.5), constant over the image
};
struct alignas(64) UnitArgs {
    CUtensorMap map[kMaxUnitImages];
    UnitImage img[kMaxUnitImages];
    int dw, dh;
    int nbox;  // boxes per window row: nbox * kUnitBoxBytes >= 3 * dw + 4 (the last thread's 16 bytes)
};

template <typename OutT, int BAND>
__global__ void __launch_bounds__(kUnitMaxThreads) letterbox_unit_kernel(const __grid_constant__ UnitArgs a, OutT* __restrict__ dst) {
    constexpr int ROWS = BAND + 1, BOXW = kUnitBoxBytes, BOXB = ROWS * BOXW;
    extern __shared__ __align__(128) uint8_t win[];  // a.nbox boxes of [ROWS][BOXW]
    __shared__ uint64_t bar;
    const int tid = threadIdx.x, nt = blockDim.x;
    const UnitImage& im = a.img[blockIdx.y];
    const int dw = a.dw, dy0 = blockIdx.x * BAND;
    const int sx0 = im.ox, sy0 = dy0 + im.oy;  // source pixel under the band's first tap
    const int sw = im.sw, sh = im.sh;
    const int nbox = a.nbox;
    // window byte column c of window row r
    auto at = [&](int c, int r) { return (c >> 8) * BOXB + r * BOXW + (c & (BOXW - 1)); };

    if (sy0 + BAND >= 0 && sy0 < sh) {  // a pure padding band fetches nothing: every tap is the border value
        if (tid == 0) {
            mbar_init(&bar, 1);
            mbar_fence_init();
        }
        __syncthreads();
        if (tid < 32) {
            if (tid == 0) mbar_arrive_expect_tx(&bar, nbox * BOXB);
            __syncwarp();
            for (int k = tid; k < nbox; k += 32) tma_load_3d(win + k * BOXB, &a.map[im.map], sx0 * 3 + k * BOXW, sy0, im.z, &bar);
        }
        mbar_wait(&bar, 0);
    }
    const bool rows_in = sy0 >= 0 && sy0 + BAND < sh;  // every window row inside the image

    const float lx = im.lx, ly = im.ly, hx = 1 - lx, hy = 1 - ly;
    const size_t area = (size_t)dw * a.dh;
    const int rows = a.dh - dy0;  // destination rows of this band
    for (int x4 = tid; x4 < dw / 4; x4 += nt) {
        const int dx = 4 * x4;
        OutT* o = dst + (size_t)im.dst_idx * 3 * area + (size_t)dy0 * dw + dx;
        int off[4];  // the thread's 16 window bytes 12 * x4 .. 12 * x4 + 15, as 4 words (a word never straddles two boxes)
#pragma unroll
        for (int j = 0; j < 4; ++j) off[j] = at(12 * x4 + 4 * j, 0);
        unsigned xin = 0;  // bit p: the thread's window pixel p (source column sx0 + dx + p) lies inside the image
#pragma unroll
        for (int p = 0; p < 5; ++p) xin |= (unsigned)(sx0 + dx + p >= 0 && sx0 + dx + p < sw) << p;
        // horizontal pass of window row r: h[3j + c] = hx * px[j][c] + lx * px[j + 1][c] for the thread's 4 pixels (exact)
        auto hrow = [&](int r, float (&h)[12]) {
            uint32_t w[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) w[j] = *reinterpret_cast<const uint32_t*>(win + off[j] + r * BOXW);
            float t[15];
#pragma unroll
            for (int i = 0; i < 15; ++i)  // byte i -> float: 2^23 + v is exact with v in the mantissa
                t[i] = __uint_as_float(__byte_perm(w[i >> 2], 0x4B000000u, 0x7650u + (i & 3))) - 8388608.0f;
            if (!(rows_in && xin == 0x1fu)) {  // taps outside the image -> const_value_st = 128 (preprocess.cu:115)
                const bool yin = sy0 + r >= 0 && sy0 + r < sh;
#pragma unroll
                for (int i = 0; i < 15; ++i) t[i] = yin && (xin >> (i / 3) & 1u) ? t[i] : 128.0f;
            }
#pragma unroll
            for (int i = 0; i < 12; ++i) h[i] = hx * t[i] + lx * t[i + 3];
        };
        float top[12], bot[12];
        hrow(0, top);
#pragma unroll
        for (int r = 0; r < BAND; ++r) {
            hrow(r + 1, bot);
            if (r < rows) {
                float v[3][4];
#pragma unroll
                for (int j = 0; j < 4; ++j)
#pragma unroll
                    for (int c = 0; c < 3; ++c)  // :59-61 regrouped (exact), bgr -> rgb and /255 :64-74
                        v[c][j] = div255(hy * top[3 * j + c] + ly * bot[3 * j + c]);
                OutT* orow = o + (size_t)r * dw;
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    OutT* q = orow + (size_t)(2 - c) * area;
                    if constexpr (sizeof(OutT) == 4) {
                        *reinterpret_cast<float4*>(q) = make_float4(v[c][0], v[c][1], v[c][2], v[c][3]);
                    } else {
                        const __half2 h0 = __floats2half2_rn(v[c][0], v[c][1]), h1 = __floats2half2_rn(v[c][2], v[c][3]);
                        uint2 u;
                        u.x = *reinterpret_cast<const uint32_t*>(&h0);
                        u.y = *reinterpret_cast<const uint32_t*>(&h1);
                        *reinterpret_cast<uint2*>(q) = u;
                    }
                }
            }
#pragma unroll
            for (int i = 0; i < 12; ++i) top[i] = bot[i];
        }
    }
}

// Host: does this image take the unit-scale path?  (scale == 1 exactly, half-integer translation, TMA-compatible.)
static bool unit_scale_image(const trtx_image_desc& d, const float m[6], UnitImage* u) {
    if (!(m[0] == 1.0f && m[4] == 1.0f && m[1] == 0.0f && m[3] == 0.0f)) return false;
    const float tx = m[2] + 0.5f, ty = m[5] + 0.5f;
    if (!(fabsf(tx) < 1048576.0f && fabsf(ty) < 1048576.0f)) return false;
    if (2.0f * tx != rintf(2.0f * tx) || 2.0f * ty != rintf(2.0f * ty)) return false;
    if (reinterpret_cast<uintptr_t>(d.data_dev) % 16 != 0 || d.pitch % 16 != 0) return false;  // TMA base / stride
    u->ox = (int)floorf(tx);
    u->oy = (int)floorf(ty);
    // TMA fetches box k of a window from byte column 3 * ox + 256 * k: the start of a box must be 16-byte aligned in global
    // memory (an unaligned start is an illegal instruction on sm_90a), so horizontal offsets that are not a multiple of 16
    // pixels (e.g. a 624-wide source centred in 640) take the general kernel
    if (u->ox % 16 != 0) return false;
    u->lx = tx - floorf(tx);
    u->ly = ty - floorf(ty);
    u->sw = d.width;
    u->sh = d.height;
    return true;
}

static bool encode_image_map(CUtensorMap* map, const uint8_t* base, int sw, int sh, int pitch, int n, size_t image_stride) {
    EncodeTiledFn enc = tma_encoder();
    if (!enc) return false;
    const cuuint64_t gdim[3] = {(cuuint64_t)sw * 3u, (cuuint64_t)sh, (cuuint64_t)n};
    const cuuint64_t gstr[2] = {(cuuint64_t)pitch, (cuuint64_t)image_stride};
    const cuuint32_t bdim[3] = {(cuuint32_t)kUnitBoxBytes, (cuuint32_t)(kUnitBand + 1), 1u};
    const cuuint32_t estr[3] = {1u, 1u, 1u};
    return enc(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<uint8_t*>(base), gdim, gstr, bdim, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// Launch the unit-scale kernel for `n` images (descriptors d[i], unit info u[i] already filled but for map/z).
// Returns TRTX_ERR_UNSUPPORTED when no tensor map can be made or the window does not fit in shared memory (the caller
// falls back to the general kernel).
template <typename OutT>
static int launch_unit_t(const UnitArgs& a, int n, size_t smem, OutT* dst, cudaStream_t st) {
    auto* k = letterbox_unit_kernel<OutT, kUnitBand>;
    if (smem > 48 * 1024 && cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
        cudaGetLastError();
        return TRTX_ERR_UNSUPPORTED;
    }
    const int threads = min((a.dw / 4 + kWarp - 1) / kWarp * kWarp, kUnitMaxThreads);
    k<<<dim3((a.dh + kUnitBand - 1) / kUnitBand, n), threads, smem, st>>>(a, dst);
    return check_launch();
}

static int launch_unit(const trtx_image_desc* const* d, UnitImage* u, int n, void* dst, int dw, int dh, int out_dtype,
                       cudaStream_t st) {
    UnitArgs a;
    a.dw = dw;
    a.dh = dh;
    a.nbox = (3 * dw + 4 + kUnitBoxBytes - 1) / kUnitBoxBytes;
    const size_t smem = (size_t)a.nbox * kUnitBoxBytes * (kUnitBand + 1);
    if (smem > 227 * 1024) return TRTX_ERR_UNSUPPORTED;
    // one 3-D map for the whole group when the images are equally sized and equally spaced (a frame ring / one batch
    // tensor): one encode instead of n
    bool uniform = n > 1;
    const ptrdiff_t step = n > 1 ? d[1]->data_dev - d[0]->data_dev : 0;
    for (int i = 1; i < n && uniform; ++i)
        uniform = d[i]->width == d[0]->width && d[i]->height == d[0]->height && d[i]->pitch == d[0]->pitch &&
                  d[i]->data_dev - d[i - 1]->data_dev == step;
    uniform = uniform && step > 0 && step % 16 == 0 && (size_t)step >= (size_t)d[0]->pitch * (size_t)d[0]->height;
    if (uniform) {
        if (!encode_image_map(&a.map[0], d[0]->data_dev, d[0]->width, d[0]->height, d[0]->pitch, n, (size_t)step))
            return TRTX_ERR_UNSUPPORTED;
    }
    for (int i = 0; i < n; ++i) {
        if (uniform) {
            u[i].map = 0;
            u[i].z = i;
        } else {
            if (!encode_image_map(&a.map[i], d[i]->data_dev, d[i]->width, d[i]->height, d[i]->pitch, 1,
                                  (size_t)d[i]->pitch * (size_t)d[i]->height))
                return TRTX_ERR_UNSUPPORTED;
            u[i].map = i;
            u[i].z = 0;
        }
        a.img[i] = u[i];
    }
    if (out_dtype == TRTX_F32) return launch_unit_t(a, n, smem, static_cast<float*>(dst), st);
    return launch_unit_t(a, n, smem, static_cast<__half*>(dst), st);
}

// =====================================================================================================================
// Mask R-CNN pre-process: preprocessImg (rcnn/common.hpp:79-110) + the float widening of rcnn.cpp:504-505, i.e.
// cv::resize(INTER_LINEAR) of the 8-bit BGR image into the rectangle between the pads, pasted on a 128-grey canvas, every byte
// widened to float: [net_h, net_w, 3] fp32 BGR, 0..255 per image.  The resize is OpenCV 4.x's fixed-point one, as
// calib_host.cu restates it: taps and weights from cv_linear_tap, horizontal pass h = S[sx] * c0 + S[sx1] * c1 in int, vertical
// pass ((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2 saturated to 0..255 (VResizeLinearVec_32s8u).
//
// Bound by HBM writes: 4 output bytes per canvas byte (b8 at 1067 x 800: 81.9 MB written, 7.4 MB of u8 read).  A CTA owns a band
// of kRcnnPreBand full-width destination rows of one image (flat grid over images x bands), which in HWC is ONE contiguous run of
// band * net_w * 3 floats:
//   1. y taps: one per destination row of the band inside the rectangle; the distinct clipped source rows they read (at most
//      2 * band) become the band's slots;
//   2. horizontal pass: each thread computes the x taps of its columns once and runs them over every slot row; the results,
//      already >> 4 (all the vertical pass reads of them, <= 32640), are staged as int16 rows in shared memory and shared by
//      the destination rows that use the same source row;
//   3. stores: the run is written with 16-byte stores (a head of 0..3 floats up to the first 16-byte boundary and a tail
//      of 0..3 floats are scalar: rows are 12 * net_w bytes and dst may be only 4-byte aligned); an element outside the
//      rectangle is 128.0f.  A band wholly in the top / bottom padding skips 1 and 2 and reads nothing.
constexpr int kRcnnPreBand = 4;            // destination rows per CTA
constexpr int kRcnnPreSlots = 2 * kRcnnPreBand;  // staged source rows: two taps per destination row at most
constexpr int kRcnnPreThreads = 256;
constexpr int kMaxRcnnPreImages = 64;      // descriptors per launch (kernel parameter block)

struct RcnnPreImage {
    const uint8_t* src;
    double scale_x, scale_y;  // cv::resize: 1. / ((double)dsize / ssize)
    int sw, sh, pitch;
    int x0, y0, rw, rh;       // the resized rectangle on the canvas: (pad_left, pad_top, net - pads)
    int dst_idx;
};
struct RcnnPreArgs {
    RcnnPreImage img[kMaxRcnnPreImages];
    int net_w, net_h, bands;
    int stride;               // int16 per staged row: 3 * the widest rectangle of the launch
};

// Stages 1 and 2 of a band, shared by the R-CNN and the classification pre-process kernels; Store is stage 3:
// Store::run(a, im, y0, rows, k_lo, k_hi, pix, dst) writes band rows [0, rows), and pix(k, i), k_lo <= k < k_hi, is the
// resized byte i (B, G, R interleaved) of the rectangle's row under band row k.
template <class Store>
__device__ __forceinline__ void resize_band(const RcnnPreArgs& a, float* __restrict__ dst) {
    constexpr int R = kRcnnPreBand;
    extern __shared__ __align__(16) int16_t hrows[];  // [slots][a.stride]
    __shared__ int s_row[kRcnnPreSlots];              // source row of each slot
    __shared__ int s_slot[R][2];                      // slots of the two taps of destination row k
    __shared__ int s_coef[R][2];                      // their weights b0, b1
    __shared__ int s_nslots;
    const int item = blockIdx.x / a.bands, band = blockIdx.x - item * a.bands;
    const RcnnPreImage& im = a.img[item];
    const int y0 = band * R, rows = min(R, a.net_h - y0);
    const int k_lo = max(im.y0 - y0, 0), k_hi = min(im.y0 + im.rh - y0, rows);  // band rows inside the rectangle
    const int stride = a.stride;
    if (k_lo < k_hi) {  // uniform over the CTA
        if (threadIdx.x == 0) {
            int n = 0;
            for (int k = k_lo; k < k_hi; ++k) {
                const LinearTap t = cv_linear_tap(y0 + k - im.y0, im.scale_y, im.sh, false);
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const int sy = min(max(t.s + j, 0), im.sh - 1);  // y taps are clipped where they are read
                    int slot = -1;
                    for (int i = 0; i < n; ++i) slot = s_row[i] == sy ? i : slot;
                    if (slot < 0) {
                        s_row[n] = sy;
                        slot = n++;
                    }
                    s_slot[k][j] = slot;
                }
                s_coef[k][0] = t.c0;
                s_coef[k][1] = t.c1;
            }
            s_nslots = n;
        }
        __syncthreads();
        const int n = s_nslots;
        for (int x = threadIdx.x; x < im.rw; x += blockDim.x) {
            const LinearTap t = cv_linear_tap(x, im.scale_x, im.sw, true);
            const int o0 = 3 * t.s, o1 = 3 * min(t.s + 1, im.sw - 1);
            for (int j0 = 0; j0 < n; j0 += 4) {
                uint32_t px[4][6];  // the loads of 4 slot rows are in flight before the first use
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    if (j0 + j < n) {
                        const uint8_t* S = im.src + (size_t)s_row[j0 + j] * (size_t)im.pitch;
#pragma unroll
                        for (int c = 0; c < 3; ++c) px[j][c] = __ldg(S + o0 + c), px[j][3 + c] = __ldg(S + o1 + c);
                    }
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    if (j0 + j < n) {
                        int16_t* h = hrows + (j0 + j) * stride + 3 * x;
#pragma unroll
                        for (int c = 0; c < 3; ++c) h[c] = (int16_t)(((int)px[j][c] * t.c0 + (int)px[j][3 + c] * t.c1) >> 4);
                    }
            }
        }
        __syncthreads();
    }
    auto pix = [&](int k, int i) -> uint32_t {
        const int h0 = hrows[s_slot[k][0] * stride + i], h1 = hrows[s_slot[k][1] * stride + i];
        const int v = (((s_coef[k][0] * h0) >> 16) + ((s_coef[k][1] * h1) >> 16) + 2) >> 2;
        return (uint32_t)min(max(v, 0), 255);
    };
    Store::run(a, im, y0, rows, k_lo, k_hi, pix, dst);
}

// Stage 3's stores: the run base[0, total) of a band, float f = element e of band row k of rows of L floats, value(k, e),
// with 16-byte stores (a head of 0..3 floats up to the first 16-byte boundary and a tail of 0..3 floats are scalar: dst may be
// only 4-byte aligned).
template <class Value>
__device__ __forceinline__ void store_band_run(float* __restrict__ base, int total, int L, Value value) {
    const int head = min((int)(((16u - (unsigned)(reinterpret_cast<uintptr_t>(base) & 15u)) & 15u) >> 2), total);
    const int nvec = (total - head) >> 2, tail0 = head + 4 * nvec;
    if ((int)threadIdx.x < head) base[threadIdx.x] = value(threadIdx.x / L, threadIdx.x % L);
    if (tail0 + (int)threadIdx.x < total) {
        const int f = tail0 + threadIdx.x;
        base[f] = value(f / L, f % L);
    }
    int q = threadIdx.x;
    int k = (head + 4 * q) / L, e = (head + 4 * q) % L;  // row and element of the thread's first float4
    const int step = 4 * blockDim.x;
    for (; q < nvec; q += blockDim.x) {
        float v[4];
        int kk = k, ee = e;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            v[j] = value(kk, ee);
            if (++ee == L) ee = 0, ++kk;
        }
        *reinterpret_cast<float4*>(base + head + 4 * q) = make_float4(v[0], v[1], v[2], v[3]);
        for (e += step; e >= L; e -= L) ++k;
    }
}

// R-CNN: HWC, so the band is ONE contiguous run of band * net_w * 3 floats; 128.0f outside the rectangle.
struct RcnnHwcStore {
    template <class Pix>
    static __device__ __forceinline__ void run(const RcnnPreArgs& a, const RcnnPreImage& im, int y0, int rows, int k_lo, int k_hi,
                                               Pix pix, float* __restrict__ dst) {
        const int L = 3 * a.net_w;  // floats per canvas row
        float* base = dst + ((size_t)im.dst_idx * a.net_h + y0) * (size_t)L;
        const int e_lo = 3 * im.x0, e_n = 3 * im.rw;  // row elements [e_lo, e_lo + e_n) lie in the rectangle
        store_band_run(base, rows * L, L, [&](int k, int e) -> float {
            const int i = e - e_lo;
            if (k < k_lo || k >= k_hi || (unsigned)i >= (unsigned)e_n) return 128.0f;  // the canvas, Scalar(128, 128, 128)
            return u8_to_float_alu(pix(k, i));
        });
    }
};

__global__ void __launch_bounds__(kRcnnPreThreads) rcnn_preprocess_kernel(const __grid_constant__ RcnnPreArgs a,
                                                                          float* __restrict__ dst) {
    resize_band<RcnnHwcStore>(a, dst);
}

// ---------------------------------------------------------------------------------------------------------------------
// YOLO classification pre-process: batch_preprocess of the cls drivers (yolov8/yolov8_cls.cpp:19-46, the same code in yolo11 and
// yolo26; yolov5/yolov5_cls.cpp:19-36) into the engine's [B, 3, net_h, net_w] fp32 planar RGB input.  The resize is the band
// kernel's above, over RcnnPreImage descriptors that the host fills per variant:
//   TRTX_YOLO_V8: the centre square crop Rect((w - m) / 2, (h - m) / 2, m, m), m = min(w, h), as a descriptor offset (cv::resize
//                 of a ROI reads only the ROI), resized over the whole net_w x net_h;
//   TRTX_YOLO_V5: preprocess_img's letterbox (trtx_calib_letterbox_rect) on a 128-grey canvas.
// Only the store stage is new: the band is three contiguous planar runs of band * net_w floats, R, G, B, each written by
// store_band_run.  The value of byte u in plane c comes from a per-CTA table of 3 x 256 floats (cls_input_value).
// dynamic shared memory left beside the table and the band's other static arrays: rectangles up to 4 757 pixels wide
constexpr size_t kClsMaxDynamicSmem = 227 * 1024 - 3 * 256 * sizeof(float) - 1024;

// The engine input value of byte u in plane c (0 = R, 1 = G, 2 = B).
//   V8: convertTo(CV_32F, 1 / 255.0), i.e. (float)u * (float)(1 / 255.0), one rounded float product;
//   V5: ((float)u / 255.0 - mean_c) / std_c in double with the driver's literals (yolov5_cls.cpp:28-30), stored to float.
// _rn intrinsics: both are IEEE operations that nvcc must not contract.
__device__ __forceinline__ float cls_input_value(int variant, int c, uint32_t u) {
    if (variant == TRTX_YOLO_V8) return __fmul_rn((float)u, (float)(1 / 255.0));
    const double mean = c == 0 ? 0.485 : (c == 1 ? 0.456 : 0.406), std = c == 0 ? 0.229 : (c == 1 ? 0.224 : 0.225);
    return __double2float_rn(__ddiv_rn(__dsub_rn(__ddiv_rn((double)(float)u, 255.0), mean), std));
}

// YOLOP's preprocess_img (yolop/utils.h:11-36) after the resize, the value of byte u in plane c (0 = B, 1 = G, 2 = R: the
// driver copies the planes in BGR order, yolop/yolop.cpp:110-127, so Scalar(0.485, ...) meets B first):
//   convertTo(CV_32FC3, 1.f / 255.f)       t = (float)u * (1.f / 255.f)
//   cv::subtract(tensor, Scalar(mean))     s = t - (float)mean_c, in float
//   cv::divide(tensor, Scalar(std))        (float)((double)s / std_c), in double
// Pinned against cv2 4.13 on all 3 x 256 bytes (tests/test_yolop_cpu.py).
__device__ __forceinline__ float yolop_input_value(int c, uint32_t u) {
    const double mean = c == 0 ? 0.485 : (c == 1 ? 0.456 : 0.406), std = c == 0 ? 0.229 : (c == 1 ? 0.224 : 0.225);
    const float s = __fsub_rn(__fmul_rn((float)u, 1.f / 255.f), (float)mean);
    return __double2float_rn(__ddiv_rn((double)s, std));
}

// The input conventions of the planar stores: In::kCanvas is the byte of the letterbox canvas, In::channel(c) the BGR
// channel that plane c takes, In::value(c, u) the engine input value of byte u in plane c.
template <int kVariant>
struct ClsInput {
    static constexpr uint32_t kCanvas = 128u;  // the V5 canvas, Scalar(128, 128, 128); V8 has none
    static __device__ __forceinline__ int channel(int c) { return 2 - c; }  // cvtColor BGR2RGB / the driver's planes R, G, B
    static __device__ __forceinline__ float value(int c, uint32_t u) { return cls_input_value(kVariant, c, u); }
};
struct YolopInput {
    static constexpr uint32_t kCanvas = 114u;  // Scalar(114, 114, 114)
    static __device__ __forceinline__ int channel(int c) { return c; }
    static __device__ __forceinline__ float value(int c, uint32_t u) { return yolop_input_value(c, u); }
};
// DETR's preprocessImg (detr/common.hpp:81-89): cvtColor BGR2RGB, so plane c (0 = R) takes BGR channel 2 - c; then
// convertTo(CV_32FC3), `img /= 255` (convertTo(-1, 1. / 255): (float)u * (1.f / 255.f)), `img -= Scalar(mean)` (cv::subtract,
// float) and `img /= Scalar(std)` (cv::divide, double) -- YOLOP's chain with Scalar(0.485, ...) meeting R instead of B.
struct DetrInput {
    static constexpr uint32_t kCanvas = 0u;  // never read: the frame is stretched over the whole net
    static __device__ __forceinline__ int channel(int c) { return 2 - c; }
    static __device__ __forceinline__ float value(int c, uint32_t u) { return yolop_input_value(c, u); }
};
// UFLD's prepareImage (ufld/lane_det.cpp:194-221): cvtColor BGR2RGB and cv::split, so plane c (0 = R) takes BGR channel
// 2 - c; the value chain is ufld_input_value (common.cuh).
struct UfldInput {
    static constexpr uint32_t kCanvas = 0u;  // never read: the frame is stretched over the whole net
    static __device__ __forceinline__ int channel(int c) { return 2 - c; }
    static __device__ __forceinline__ float value(int c, uint32_t u) { return ufld_input_value(c, u); }
};
// RefineDet's base_transform (refinedet/refinedet.cpp:822-839): plane c (0 = R) reads BGR byte 2 - c of the resized frame;
// the value is refinedet_input_value (common.cuh).
struct RefinedetInput {
    static constexpr uint32_t kCanvas = 0u;  // never read: the frame is stretched over the whole net
    static __device__ __forceinline__ int channel(int c) { return 2 - c; }
    static __device__ __forceinline__ float value(int c, uint32_t u) { return refinedet_input_value(c, u); }
};

// [B, 3, net_h, net_w] planes: the band is three contiguous runs of band * net_w floats, each written by store_band_run; the
// value of a byte comes from a per-CTA table of 3 x 256 floats.
template <class In>
struct PlanarStore {
    template <class Pix>
    static __device__ __forceinline__ void run(const RcnnPreArgs& a, const RcnnPreImage& im, int y0, int rows, int k_lo, int k_hi,
                                               Pix pix, float* __restrict__ dst) {
        __shared__ float lut[3][256];
        for (int j = threadIdx.x; j < 3 * 256; j += blockDim.x) lut[j >> 8][j & 255] = In::value(j >> 8, j & 255);
        __syncthreads();
        const int W = a.net_w;
#pragma unroll 1
        for (int c = 0; c < 3; ++c) {
            const int ch = In::channel(c);
            float* base = dst + (((size_t)im.dst_idx * 3 + c) * a.net_h + y0) * (size_t)W;
            store_band_run(base, rows * W, W, [&](int k, int x) -> float {
                const int i = x - im.x0;
                const bool in = k >= k_lo && k < k_hi && (unsigned)i < (unsigned)im.rw;
                return lut[c][in ? pix(k, 3 * i + ch) : In::kCanvas];
            });
        }
    }
};

template <int kVariant>
__global__ void __launch_bounds__(kRcnnPreThreads) cls_preprocess_kernel(const __grid_constant__ RcnnPreArgs a,
                                                                         float* __restrict__ dst) {
    resize_band<PlanarStore<ClsInput<kVariant>>>(a, dst);
}

__global__ void __launch_bounds__(kRcnnPreThreads) yolop_preprocess_kernel(const __grid_constant__ RcnnPreArgs a,
                                                                           float* __restrict__ dst) {
    resize_band<PlanarStore<YolopInput>>(a, dst);
}

__global__ void __launch_bounds__(kRcnnPreThreads) detr_preprocess_kernel(const __grid_constant__ RcnnPreArgs a,
                                                                          float* __restrict__ dst) {
    resize_band<PlanarStore<DetrInput>>(a, dst);
}

__global__ void __launch_bounds__(kRcnnPreThreads) ufld_preprocess_kernel(const __grid_constant__ RcnnPreArgs a,
                                                                          float* __restrict__ dst) {
    resize_band<PlanarStore<UfldInput>>(a, dst);
}

__global__ void __launch_bounds__(kRcnnPreThreads) refinedet_preprocess_kernel(const __grid_constant__ RcnnPreArgs a,
                                                                               float* __restrict__ dst) {
    resize_band<PlanarStore<RefinedetInput>>(a, dst);
}

// One launch of `kernel` per kMaxRcnnPreImages frames: make(i, im) fills the band descriptor of frame i (validated before).
template <class Make>
static int launch_bands(void (*kernel)(RcnnPreArgs, float*), int batch, int net_w, int net_h, float* dst_dev, size_t smem_max,
                        cudaStream_t st, Make make) {
    if (smem_max > 48 * 1024 &&
        cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_max) != cudaSuccess) {
        g_last_cuda_error = (int)cudaGetLastError();
        return TRTX_ERR_CUDA;
    }
    RcnnPreArgs a;
    a.net_w = net_w;
    a.net_h = net_h;
    a.bands = (net_h + kRcnnPreBand - 1) / kRcnnPreBand;
    for (int i0 = 0; i0 < batch; i0 += kMaxRcnnPreImages) {
        const int n = batch - i0 < kMaxRcnnPreImages ? batch - i0 : kMaxRcnnPreImages;
        int wmax = 0;
        for (int j = 0; j < n; ++j) {
            RcnnPreImage& im = a.img[j];
            make(i0 + j, im);
            im.dst_idx = i0 + j;
            wmax = im.rw > wmax ? im.rw : wmax;
        }
        a.stride = 3 * wmax;
        const size_t smem = (size_t)kRcnnPreSlots * a.stride * sizeof(int16_t);
        kernel<<<(unsigned)(n * a.bands), kRcnnPreThreads, smem, st>>>(a, dst_dev);
        const int rc = check_launch();
        if (rc) return rc;
    }
    return TRTX_OK;
}

// The band descriptor of frame d for the classification pre-process; false where the reference's cv::resize or copyTo throws
// (an empty letterbox rectangle, or one that leaves the canvas).
static bool cls_band_image(int variant, const trtx_image_desc& d, int net_w, int net_h, RcnnPreImage& im) {
    im.src = d.data_dev;
    im.sw = d.width;
    im.sh = d.height;
    im.pitch = d.pitch;
    im.x0 = im.y0 = 0;
    im.rw = net_w;
    im.rh = net_h;
    if (variant == TRTX_YOLO_V8) {  // imgs[b](cv::Rect(left, top, m, m)), yolov8_cls.cpp:21-26
        const int m = d.width < d.height ? d.width : d.height;
        im.src += (size_t)((d.height - m) / 2) * (size_t)d.pitch + 3 * (size_t)((d.width - m) / 2);
        im.sw = im.sh = m;
    } else {
        int r[4];
        trtx_calib_letterbox_rect(d.width, d.height, net_w, net_h, r);
        im.x0 = r[0], im.y0 = r[1], im.rw = r[2], im.rh = r[3];
        if (im.rw <= 0 || im.rh <= 0 || im.x0 < 0 || im.y0 < 0 || im.x0 + im.rw > net_w || im.y0 + im.rh > net_h) return false;
    }
    im.scale_x = 1. / ((double)im.rw / im.sw);
    im.scale_y = 1. / ((double)im.rh / im.sh);
    return true;
}

// The band descriptor of frame d for a whole frame stretched over the whole net, cv::resize(img, dst, Size(net_w, net_h))
// (DETR's preprocessImg, UFLD's prepareImage), i.e. cls_band_image's V8 descriptor without the crop.
static void stretch_band_image(const trtx_image_desc& d, int net_w, int net_h, RcnnPreImage& im) {
    im.src = d.data_dev;
    im.sw = d.width;
    im.sh = d.height;
    im.pitch = d.pitch;
    im.x0 = im.y0 = 0;
    im.rw = net_w;
    im.rh = net_h;
    im.scale_x = 1. / ((double)net_w / d.width);
    im.scale_y = 1. / ((double)net_h / d.height);
}

// The whole-frame pre-processes (DETR, UFLD): one band descriptor per frame (stretch_band_image) into `kernel`'s planar store.
static int stretch_preprocess(void (*kernel)(RcnnPreArgs, float*), const trtx_image_desc* images_host, int batch, int net_w,
                              int net_h, float* dst_dev, cudaStream_t st) {
    if (!images_host || batch <= 0 || !dst_dev || net_w <= 0 || net_h <= 0) return TRTX_ERR_INVALID;
    if (reinterpret_cast<uintptr_t>(dst_dev) % sizeof(float) != 0) return TRTX_ERR_INVALID;
    // every descriptor is checked before the first launch, so that a rejected call writes nothing
    for (int i = 0; i < batch; ++i) {
        const trtx_image_desc& d = images_host[i];
        if (!d.data_dev || d.width <= 0 || d.height <= 0 || d.pitch < 3 * d.width) return TRTX_ERR_INVALID;
    }
    const size_t smem = (size_t)kRcnnPreSlots * 3 * (size_t)net_w * sizeof(int16_t);  // every rectangle is net_w wide
    if (smem > kClsMaxDynamicSmem) return TRTX_ERR_UNSUPPORTED;
    return launch_bands(kernel, batch, net_w, net_h, dst_dev, smem, st,
                        [&](int i, RcnnPreImage& im) { stretch_band_image(images_host[i], net_w, net_h, im); });
}

// ---------------------------------------------------------------------------------------------------------------------
// Bicubic letterbox pre-process: preprocess_img of yolov3-tiny (yolov3-tiny/yolov3-tiny.cpp:40-60) and retinafaceAntiCov
// (retinafaceAntiCov/retinafaceAntiCov.cpp:41-61) -- cv::resize(INTER_CUBIC) into trtx_calib_letterbox_rect's rectangle on a
// 128-grey canvas -- and the drivers' loops into R, G, B planes (:441-445, :528-532).  The resize is OpenCV 4.x's own 8-bit
// INTER_CUBIC (resizeGeneric_ with HResizeCubic and VResizeCubic; IPP's differs by 1 in a few % of the bytes, DESIGN §7):
//   taps:       fx = (float)((d + 0.5) * scale - 0.5), s = floor(fx), fx -= s (kept at the borders: cv_linear_coord without
//               clamp); taps s - 1 .. s + 2, clamped into the image; weights interpolateCubic(fx) (A = -0.75, float) and
//               saturate_cast<short>(c * 2048);
//   horizontal: h = the int sum of the 4 products (|h| reaches 2^19.3, so nothing is staged in int16);
//   vertical:   of the 3 * rw bytes of a destination row, the first (3 * rw) & ~7 are VResizeCubicVec_32s8u's 8-lane float loop:
//               h0 * b0' + (h1 * b1' + (h2 * b2' + h3 * b3')), b' = b / 2048^2 (exact), every product and sum rounded (no FMA),
//               then rounded half to even; the rest are the scalar tail's (sum h_k * b_k + 2^21) >> 22; both saturated to 0..255.
// The band structure is resize_band's with 4 y taps per destination row, the staged rows in int32 and up to 4 slots per row.
// The horizontal pass is shared by the band rows that read the same source row; stage 3 is PlanarStore.
constexpr int kCubicMaxSlots = 4 * kRcnnPreBand;

// interpolateCubic (imgproc/src/resize.cpp) statement by statement in float, then saturate_cast<short>(c * 2048)
__device__ __forceinline__ void cv_cubic_coeffs(float x, int (&c)[4]) {
    constexpr float A = -0.75f;
    const float x1 = __fadd_rn(x, 1.f), mx = __fsub_rn(1.f, x);
    const float c0 = __fsub_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fsub_rn(__fmul_rn(A, x1), 5 * A), x1), 8 * A), x1), 4 * A);
    const float c1 = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(A + 2, x), A + 3), x), x), 1.f);
    const float c2 = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(A + 2, mx), A + 3), mx), mx), 1.f);
    const float c3 = __fsub_rn(__fsub_rn(__fsub_rn(1.f, c0), c1), c2);
    c[0] = __float2int_rn(__fmul_rn(c0, 2048.f));
    c[1] = __float2int_rn(__fmul_rn(c1, 2048.f));
    c[2] = __float2int_rn(__fmul_rn(c2, 2048.f));
    c[3] = __float2int_rn(__fmul_rn(c3, 2048.f));
}

// Source rows a band of kRcnnPreBand destination rows can read at y scale `scale`: the low taps of its first and last rows are
// at most ceil(3 * scale) + 1 apart (the float rounding of fy moves a difference by far less than 1), and each row reads 4 rows
// from its low tap on.
static int cubic_band_slots(double scale) {
    return (int)fmin((double)kCubicMaxSlots, ceil((kRcnnPreBand - 1) * scale) + 5);
}

template <class Store>
__device__ __forceinline__ void cubic_band(const RcnnPreArgs& a, float* __restrict__ dst) {
    constexpr int R = kRcnnPreBand;
    extern __shared__ __align__(16) int hcub[];  // [slots][a.stride]
    __shared__ int s_row[kCubicMaxSlots];
    __shared__ int s_slot[R][4];
    __shared__ int s_coef[R][4];
    __shared__ int s_nslots;
    const int item = blockIdx.x / a.bands, band = blockIdx.x - item * a.bands;
    const RcnnPreImage& im = a.img[item];
    const int y0 = band * R, rows = min(R, a.net_h - y0);
    const int k_lo = max(im.y0 - y0, 0), k_hi = min(im.y0 + im.rh - y0, rows);
    const int stride = a.stride;
    if (k_lo < k_hi) {  // uniform over the CTA
        if (threadIdx.x == 0) {
            int n = 0;
            for (int k = k_lo; k < k_hi; ++k) {
                const LinearCoord g = cv_linear_coord(y0 + k - im.y0, im.scale_y, im.sh, false);
                int c[4];
                cv_cubic_coeffs(g.f, c);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int sy = min(max(g.s - 1 + j, 0), im.sh - 1);
                    int slot = -1;
                    for (int i = 0; i < n; ++i) slot = s_row[i] == sy ? i : slot;
                    if (slot < 0) {
                        s_row[n] = sy;
                        slot = n++;
                    }
                    s_slot[k][j] = slot;
                    s_coef[k][j] = c[j];
                }
            }
            s_nslots = n;
        }
        __syncthreads();
        const int n = s_nslots;
        for (int x = threadIdx.x; x < im.rw; x += blockDim.x) {
            const LinearCoord g = cv_linear_coord(x, im.scale_x, im.sw, false);
            int c[4], o[4];
            cv_cubic_coeffs(g.f, c);
#pragma unroll
            for (int t = 0; t < 4; ++t) o[t] = 3 * min(max(g.s - 1 + t, 0), im.sw - 1);
            for (int j0 = 0; j0 < n; j0 += 4) {
                uint32_t px[4][12];  // the loads of 4 slot rows are in flight before the first use
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    if (j0 + j < n) {
                        const uint8_t* S = im.src + (size_t)s_row[j0 + j] * (size_t)im.pitch;
#pragma unroll
                        for (int t = 0; t < 4; ++t)
#pragma unroll
                            for (int ch = 0; ch < 3; ++ch) px[j][3 * t + ch] = __ldg(S + o[t] + ch);
                    }
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    if (j0 + j < n) {
                        int* h = hcub + (j0 + j) * stride + 3 * x;
#pragma unroll
                        for (int ch = 0; ch < 3; ++ch)
                            h[ch] = (int)px[j][ch] * c[0] + (int)px[j][3 + ch] * c[1] + (int)px[j][6 + ch] * c[2] +
                                    (int)px[j][9 + ch] * c[3];
                    }
            }
        }
        __syncthreads();
    }
    const int nvec = (3 * im.rw) & ~7;  // bytes of a row that the 8-lane vector loop produces
    auto pix = [&](int k, int i) -> uint32_t {
        int h[4], b[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) h[j] = hcub[s_slot[k][j] * stride + i], b[j] = s_coef[k][j];
        int v;
        if (i < nvec) {
            constexpr float sc = 1.f / (2048.f * 2048.f);
            float t = __fmul_rn((float)h[3], (float)b[3] * sc);
            t = __fadd_rn(__fmul_rn((float)h[2], (float)b[2] * sc), t);
            t = __fadd_rn(__fmul_rn((float)h[1], (float)b[1] * sc), t);
            t = __fadd_rn(__fmul_rn((float)h[0], (float)b[0] * sc), t);
            v = __float2int_rn(t);
        } else {
            v = (h[0] * b[0] + h[1] * b[1] + h[2] * b[2] + h[3] * b[3] + (1 << 21)) >> 22;
        }
        return (uint32_t)min(max(v, 0), 255);
    };
    Store::run(a, im, y0, rows, k_lo, k_hi, pix, dst);
}

// The drivers' plane loops: data[i + c * H * W] = byte 2 - c of pixel i, as
//   TRTX_CUBIC_YOLOV3_TINY   u / 255.0 in double, stored to float;
//   TRTX_CUBIC_ANTICOV       ((float)u - 127.5) * 0.0078125 in double, stored to float (exact in float).
template <int kVariant>
struct CubicInput {
    static constexpr uint32_t kCanvas = 128u;  // Scalar(128, 128, 128)
    static __device__ __forceinline__ int channel(int c) { return 2 - c; }
    static __device__ __forceinline__ float value(int, uint32_t u) {
        if (kVariant == TRTX_CUBIC_YOLOV3_TINY) return __double2float_rn(__ddiv_rn((double)u, 255.0));
        return __double2float_rn(__dmul_rn(__dsub_rn((double)u, 127.5), 0.0078125));
    }
};

template <int kVariant>
__global__ void __launch_bounds__(kRcnnPreThreads) cubic_preprocess_kernel(const __grid_constant__ RcnnPreArgs a,
                                                                           float* __restrict__ dst) {
    cubic_band<PlanarStore<CubicInput<kVariant>>>(a, dst);
}

// ---------------------------------------------------------------------------------------------------------------------
// Bilinear letterbox pre-process of yolov3, yolov4, scaled-yolov4, yolov3-spp and RetinaFace: resize_band with a planar store;
// only the value conventions and the host-side rectangles are their own.
//   TRTX_LINEAR_YOLOV3      the yolov3-tiny chain, u / 255.0 in double (CubicInput<TRTX_CUBIC_YOLOV3_TINY>), planes R, G, B;
//   TRTX_LINEAR_PY          the same store over the Python runners' rectangle: their float32 u / 255.0f is that float;
//   TRTX_LINEAR_RETINA      RetinaInput below;
//   TRTX_LINEAR_YOLOV3_SPP  blobFromImage's (float)u * (float)(1 / 255.0), planes R, G, B: cls_preprocess_kernel<TRTX_YOLO_V8>,
//                           whose value chain it is, over yolov3-spp's rectangle.
// retina_r50.cpp:342-352: plane c (0 = B) takes BGR byte c, `pr_img.at<cv::Vec3b>(i)[c] - mean` in double with means 104, 117,
// 123, stored to float (exact).
struct RetinaInput {
    static constexpr uint32_t kCanvas = 128u;  // Scalar(128, 128, 128)
    static __device__ __forceinline__ int channel(int c) { return c; }
    static __device__ __forceinline__ float value(int c, uint32_t u) {
        return __fsub_rn((float)u, c == 0 ? 104.f : (c == 1 ? 117.f : 123.f));
    }
};

template <class In>
__global__ void __launch_bounds__(kRcnnPreThreads) linear_preprocess_kernel(const __grid_constant__ RcnnPreArgs a,
                                                                            float* __restrict__ dst) {
    resize_band<PlanarStore<In>>(a, dst);
}

// The band descriptor of frame d in yolov3-spp's letterbox: TRTX_ERR_UNSUPPORTED where the rectangle is empty (cv::resize
// throws), TRTX_ERR_INVALID where the canvas is not net_w x net_h (the call binds one input shape).
static int spp_band_image(const trtx_image_desc& d, int max_size, int net_w, int net_h, RcnnPreImage& im) {
    int g[6];
    const int rc = trtx_yolov3spp_letterbox(d.width, d.height, max_size, g);
    if (rc) return rc;
    if (g[0] != net_w || g[1] != net_h) return TRTX_ERR_INVALID;
    im.src = d.data_dev;
    im.sw = d.width;
    im.sh = d.height;
    im.pitch = d.pitch;
    im.x0 = g[2], im.y0 = g[3], im.rw = g[4], im.rh = g[5];
    im.scale_x = 1. / ((double)im.rw / im.sw);
    im.scale_y = 1. / ((double)im.rh / im.sh);
    return TRTX_OK;
}

// The band descriptor of frame d in the Python runners' preprocess_image: trtx_pyrunner_letterbox_rect's rectangle, which
// cv2.resize fills with the frame; TRTX_ERR_UNSUPPORTED where it is empty (cv2.resize raises).
static int py_band_image(const trtx_image_desc& d, int net_w, int net_h, RcnnPreImage& im) {
    int r[4];
    trtx_pyrunner_letterbox_rect(d.width, d.height, net_w, net_h, r);
    if (r[2] <= 0 || r[3] <= 0) return TRTX_ERR_UNSUPPORTED;
    im.src = d.data_dev;
    im.sw = d.width;
    im.sh = d.height;
    im.pitch = d.pitch;
    im.x0 = r[0], im.y0 = r[1], im.rw = r[2], im.rh = r[3];
    im.scale_x = 1. / ((double)im.rw / im.sw);
    im.scale_y = 1. / ((double)im.rh / im.sh);
    return TRTX_OK;
}

}  // namespace trtx

using namespace trtx;

extern "C" {

// preprocess.cu:98-110 + cv::invertAffineTransform (CV_32F branch)
TRTX_API void trtx_letterbox_matrix(int sw, int sh, int dw, int dh, float d2s[6]) {
    float a = dh / (float)sh, b = dw / (float)sw;
    float scale = a < b ? a : b;  // std::min
    float s2d[6];
    s2d[0] = scale;
    s2d[1] = 0;
    s2d[2] = (float)(-scale * sw * 0.5 + dw * 0.5);
    s2d[3] = 0;
    s2d[4] = scale;
    s2d[5] = (float)(-scale * sh * 0.5 + dh * 0.5);
    /* cv::invertAffineTransform, CV_32F branch, as OpenCV >= 4.x evaluates it with softfloat/softdouble
     * (pinned against cv2 4.13 on 3000 sizes, tests/test_oracle_cpu.py): the determinant and the
     * A = M*D products are FLOAT operations (softfloat::operator* converts D to float), 1/D and the
     * translation terms are double. */
    float p0 = s2d[0] * s2d[4], p1 = s2d[1] * s2d[3];
    float det = p0 - p1;
    double D = (double)det;
    D = D != 0 ? 1. / D : 0;
    float Df = (float)D;
    float fA11 = s2d[4] * Df, fA22 = s2d[0] * Df, fA12 = (-s2d[1]) * Df, fA21 = (-s2d[3]) * Df;
    double A11 = fA11, A22 = fA22, A12 = fA12, A21 = fA21;
    double b1 = -A11 * s2d[2] - A12 * s2d[5];
    double b2 = -A21 * s2d[2] - A22 * s2d[5];
    d2s[0] = (float)A11;
    d2s[1] = (float)A12;
    d2s[2] = (float)b1;
    d2s[3] = (float)A21;
    d2s[4] = (float)A22;
    d2s[5] = (float)b2;
}

// get_rect: the inverse of the letterbox for a detection box (yolo_get_rect in common.cuh, which the segmentation
// post-process kernels share).  Host function.
TRTX_API int trtx_get_rect(int variant, int net_w, int net_h, int img_w, int img_h, const float bbox[4], int rect[4]) {
    if (!bbox || !rect || net_w <= 0 || net_h <= 0 || img_w <= 0 || img_h <= 0) return TRTX_ERR_INVALID;
    if (variant != TRTX_YOLO_V8 && variant != TRTX_YOLO_V5 && variant != TRTX_YOLO_V3 && variant != TRTX_RECT_YOLOV3_SPP)
        return TRTX_ERR_INVALID;
    if (variant == TRTX_RECT_YOLOV3_SPP && net_w != net_h) return TRTX_ERR_INVALID;
    yolo_get_rect(variant, net_w, net_h, img_w, img_h, bbox, rect);
    return TRTX_OK;
}

// get_rect_adapt_landmark, yolov8/src/postprocess.cpp:38-69: its rectangle is get_rect's V8 branch (the same float
// expressions), its keypoints yolo_map_landmark (common.cuh, shared with the pose post-process kernel of mask.cu).
TRTX_API int trtx_get_rect_adapt_landmark(int net_w, int net_h, int img_w, int img_h, const float bbox[4], float* lmk,
                                          int num_kpts, int rect[4]) {
    if (!bbox || !rect || (num_kpts > 0 && !lmk) || num_kpts < 0 || net_w <= 0 || net_h <= 0 || img_w <= 0 || img_h <= 0)
        return TRTX_ERR_INVALID;
    const YoloLetterbox lb = yolo_letterbox(net_w, net_h, img_w, img_h);
    for (int i = 0; i < num_kpts * 3; i += 3) {
        lmk[i] = yolo_map_landmark(lb, 0, lmk[i]);
        lmk[i + 1] = yolo_map_landmark(lb, 1, lmk[i + 1]);
    }
    yolo_get_rect(TRTX_YOLO_V8, net_w, net_h, img_w, img_h, bbox, rect);  // {0, 0, 0, 0} where undefined
    return TRTX_OK;
}

// get_corner, yolov8/src/postprocess.cpp:395-472 / yolo11/src/postprocess.cpp:425-502 (yolo_get_corner in common.cuh, shared
// with the oriented-box post-process kernel of mask.cu).
TRTX_API int trtx_get_corner(int net_w, int net_h, int img_w, int img_h, const float cxcywh[4], float angle, int corners[8]) {
    if (!cxcywh || !corners || net_w <= 0 || net_h <= 0 || img_w <= 0 || img_h <= 0) return TRTX_ERR_INVALID;
    yolo_get_corner(net_w, net_h, img_w, img_h, cxcywh, angle, corners);
    return TRTX_OK;
}

// get_rect_adapt_landmark of RetinaFace, retinaface/common.hpp:65-89 (retina_get_rect_adapt_landmark in common.cuh, shared
// with the face post-process kernel of mask.cu).
TRTX_API int trtx_retina_get_rect_adapt_landmark(int input_w, int input_h, int img_w, int img_h, const float bbox[4], float lmk[10],
                                                 int rect[4]) {
    if (!bbox || !lmk || !rect || input_w <= 0 || input_h <= 0 || img_w <= 0 || img_h <= 0) return TRTX_ERR_INVALID;
    retina_get_rect_adapt_landmark(input_w, input_h, img_w, img_h, bbox, lmk, rect);
    return TRTX_OK;
}

// get_rect of YOLOP, yolop/common.hpp:13-37 (yolop_get_rect in common.cuh, shared with the YOLOP post-process kernel of mask.cu).
TRTX_API int trtx_yolop_get_rect(int net_w, int net_h, int img_w, int img_h, const float bbox[4], int rect[4]) {
    if (!bbox || !rect || net_w <= 0 || net_h <= 0 || img_w <= 0 || img_h <= 0) return TRTX_ERR_INVALID;
    yolop_get_rect(yolo_letterbox(net_w, net_h, img_w, img_h), bbox, rect);
    return TRTX_OK;
}

// process_decode_ptr_host, yolov8/src/postprocess.cpp:131-147
TRTX_API int trtx_process_decode_ptr_host(const float* decode_ptr_host, int bbox_element, int count, float* rows_out) {
    if (!decode_ptr_host || !rows_out || bbox_element < 7 || count < 0) return -TRTX_ERR_INVALID;
    int n = 0;
    for (int i = 0; i < count; ++i) {
        const float* p = decode_ptr_host + 1 + (size_t)i * bbox_element;
        if ((int)p[6] == 1) {  // `int keep_flag = decode_ptr_host[basic_pos + 6]`
            for (int k = 0; k < 6; ++k) rows_out[(size_t)n * 6 + k] = p[k];
            ++n;
        }
    }
    return n;
}

// process_decode_ptr_host_obb (yolov8/src/postprocess.cpp:273-290): the same for oriented boxes -- 7 floats per kept row, the angle
// from column 7 of the 8-float rows cuda_decode_obb writes (postprocess.cu:31-39)
TRTX_API int trtx_process_decode_ptr_host_obb(const float* decode_ptr_host, int bbox_element, int count, float* rows_out) {
    if (!decode_ptr_host || !rows_out || bbox_element < 8 || count < 0) return -TRTX_ERR_INVALID;
    int n = 0;
    for (int i = 0; i < count; ++i) {
        const float* p = decode_ptr_host + 1 + (size_t)i * bbox_element;
        if ((int)p[6] == 1) {
            for (int k = 0; k < 6; ++k) rows_out[(size_t)n * 7 + k] = p[k];
            rows_out[(size_t)n * 7 + 6] = p[7];
            ++n;
        }
    }
    return n;
}

TRTX_API int trtx_preprocess_batch_enqueue(const trtx_image_desc* images_host, int batch, void* dst_dev, int dst_w,
                                           int dst_h, int out_dtype, trtx_stream_t stream) {
    if (!images_host || batch <= 0 || !dst_dev || dst_w <= 0 || dst_h <= 0) return TRTX_ERR_INVALID;
    if (out_dtype != TRTX_F32 && out_dtype != TRTX_F16) return TRTX_ERR_INVALID;
    if (reinterpret_cast<uintptr_t>(dst_dev) % (out_dtype == TRTX_F32 ? sizeof(float) : sizeof(__half)) != 0) return TRTX_ERR_INVALID;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    for (int i = 0; i < batch; ++i) {
        const trtx_image_desc& d = images_host[i];
        if (!d.data_dev || d.width <= 0 || d.height <= 0 || d.pitch < 3 * d.width) return TRTX_ERR_INVALID;
    }
    // vector stores of the unit-scale kernel: 4 pixels per thread and plane
    const bool unit_ok = dst_w % 4 == 0 && reinterpret_cast<uintptr_t>(dst_dev) % 16 == 0;
    PreArgs g;  // general-path group
    g.dw = dst_w;
    g.dh = dst_h;
    int ng = 0;
    const trtx_image_desc* ud[kMaxUnitImages];
    UnitImage uu[kMaxUnitImages];
    int nu = 0;
    auto flush_general = [&]() -> int {
        if (!ng) return TRTX_OK;
        constexpr int R = kRowsPerThread;
        dim3 block(128, 2, 1);  // 128 columns x (2 x R) rows per block
        dim3 grid((dst_w + 127) / 128, (dst_h + 2 * R - 1) / (2 * R), ng);
        if (out_dtype == TRTX_F32)
            letterbox_kernel<float><<<grid, block, 0, st>>>(g, static_cast<float*>(dst_dev));
        else
            letterbox_kernel<__half><<<grid, block, 0, st>>>(g, static_cast<__half*>(dst_dev));
        ng = 0;
        return check_launch();
    };
    auto add_general = [&](int i) -> int {
        const trtx_image_desc& d = images_host[i];
        PreImage& im = g.img[ng++];
        im.src = d.data_dev;
        im.sw = d.width;
        im.sh = d.height;
        im.pitch = d.pitch;
        im.dst_idx = i;
        trtx_letterbox_matrix(d.width, d.height, dst_w, dst_h, im.m);
        return ng == kMaxImagesPerLaunch ? flush_general() : TRTX_OK;
    };
    auto flush_unit = [&]() -> int {
        if (!nu) return TRTX_OK;
        int rc = launch_unit(ud, uu, nu, dst_dev, dst_w, dst_h, out_dtype, st);
        if (rc == TRTX_ERR_UNSUPPORTED) {  // no tensor map (driver without the encoder): general kernel
            rc = TRTX_OK;
            for (int j = 0; j < nu && rc == TRTX_OK; ++j) rc = add_general(uu[j].dst_idx);
        }
        nu = 0;
        return rc;
    };
    for (int i = 0; i < batch; ++i) {
        const trtx_image_desc& d = images_host[i];
        float m[6];
        trtx_letterbox_matrix(d.width, d.height, dst_w, dst_h, m);
        int rc = TRTX_OK;
        if (unit_ok && unit_scale_image(d, m, &uu[nu])) {
            ud[nu] = &d;
            uu[nu].dst_idx = i;
            if (++nu == kMaxUnitImages) rc = flush_unit();
        } else {
            rc = add_general(i);
        }
        if (rc) return rc;
    }
    int rc = flush_unit();
    if (rc) return rc;
    return flush_general();
}

TRTX_API int trtx_rcnn_preprocess_enqueue(const trtx_image_desc* images_host, int batch, int net_w, int net_h, float* dst_dev,
                                          trtx_stream_t stream) {
    if (!images_host || batch <= 0 || !dst_dev || net_w <= 0 || net_h <= 0) return TRTX_ERR_INVALID;
    if (reinterpret_cast<uintptr_t>(dst_dev) % sizeof(float) != 0) return TRTX_ERR_INVALID;
    // every descriptor is checked before the first launch, so that a rejected call writes nothing
    size_t smem_max = 0;
    for (int i = 0; i < batch; ++i) {
        const trtx_image_desc& d = images_host[i];
        if (!d.data_dev || d.width <= 0 || d.height <= 0 || d.pitch < 3 * d.width) return TRTX_ERR_INVALID;
        int pads[4];
        trtx_rcnn_letterbox_pads(d.width, d.height, net_w, net_h, pads);
        const int rw = net_w - (pads[0] + pads[1]), rh = net_h - (pads[2] + pads[3]);
        if (rw <= 0 || rh <= 0 || pads[0] < 0 || pads[2] < 0) return TRTX_ERR_UNSUPPORTED;  // cv::resize / copyTo would throw
        const size_t smem = (size_t)kRcnnPreSlots * 3 * (size_t)rw * sizeof(int16_t);
        if (smem > 227 * 1024) return TRTX_ERR_UNSUPPORTED;
        smem_max = smem > smem_max ? smem : smem_max;
    }
    return launch_bands(rcnn_preprocess_kernel, batch, net_w, net_h, dst_dev, smem_max, static_cast<cudaStream_t>(stream),
                        [&](int i, RcnnPreImage& im) {
                            const trtx_image_desc& d = images_host[i];
                            int pads[4];
                            trtx_rcnn_letterbox_pads(d.width, d.height, net_w, net_h, pads);
                            im.src = d.data_dev;
                            im.sw = d.width;
                            im.sh = d.height;
                            im.pitch = d.pitch;
                            im.x0 = pads[0];
                            im.y0 = pads[2];
                            im.rw = net_w - (pads[0] + pads[1]);
                            im.rh = net_h - (pads[2] + pads[3]);
                            im.scale_x = 1. / ((double)im.rw / d.width);
                            im.scale_y = 1. / ((double)im.rh / d.height);
                        });
}

TRTX_API int trtx_cls_preprocess_enqueue(int variant, const trtx_image_desc* images_host, int batch, int net_w, int net_h,
                                         float* dst_dev, trtx_stream_t stream) {
    if (!images_host || batch <= 0 || !dst_dev || net_w <= 0 || net_h <= 0) return TRTX_ERR_INVALID;
    if (variant != TRTX_YOLO_V8 && variant != TRTX_YOLO_V5) return TRTX_ERR_INVALID;
    if (reinterpret_cast<uintptr_t>(dst_dev) % sizeof(float) != 0) return TRTX_ERR_INVALID;
    // every descriptor is checked before the first launch, so that a rejected call writes nothing
    size_t smem_max = 0;
    for (int i = 0; i < batch; ++i) {
        const trtx_image_desc& d = images_host[i];
        if (!d.data_dev || d.width <= 0 || d.height <= 0 || d.pitch < 3 * d.width) return TRTX_ERR_INVALID;
        RcnnPreImage im;
        if (!cls_band_image(variant, d, net_w, net_h, im)) return TRTX_ERR_UNSUPPORTED;
        const size_t smem = (size_t)kRcnnPreSlots * 3 * (size_t)im.rw * sizeof(int16_t);
        if (smem > kClsMaxDynamicSmem) return TRTX_ERR_UNSUPPORTED;
        smem_max = smem > smem_max ? smem : smem_max;
    }
    auto* kernel = variant == TRTX_YOLO_V8 ? cls_preprocess_kernel<TRTX_YOLO_V8> : cls_preprocess_kernel<TRTX_YOLO_V5>;
    return launch_bands(kernel, batch, net_w, net_h, dst_dev, smem_max, static_cast<cudaStream_t>(stream),
                        [&](int i, RcnnPreImage& im) { cls_band_image(variant, images_host[i], net_w, net_h, im); });
}

// YOLOP's preprocess_img letterbox is yolov5-cls's (the same statements, yolop/utils.h:13-25), so its band descriptor is
// cls_band_image's V5 one; only the store differs (canvas 114, BGR planes, its own value chain).
TRTX_API int trtx_yolop_preprocess_enqueue(const trtx_image_desc* images_host, int batch, int net_w, int net_h, float* dst_dev,
                                           trtx_stream_t stream) {
    if (!images_host || batch <= 0 || !dst_dev || net_w <= 0 || net_h <= 0) return TRTX_ERR_INVALID;
    if (reinterpret_cast<uintptr_t>(dst_dev) % sizeof(float) != 0) return TRTX_ERR_INVALID;
    // every descriptor is checked before the first launch, so that a rejected call writes nothing
    size_t smem_max = 0;
    for (int i = 0; i < batch; ++i) {
        const trtx_image_desc& d = images_host[i];
        if (!d.data_dev || d.width <= 0 || d.height <= 0 || d.pitch < 3 * d.width) return TRTX_ERR_INVALID;
        RcnnPreImage im;
        if (!cls_band_image(TRTX_YOLO_V5, d, net_w, net_h, im)) return TRTX_ERR_UNSUPPORTED;
        const size_t smem = (size_t)kRcnnPreSlots * 3 * (size_t)im.rw * sizeof(int16_t);
        if (smem > kClsMaxDynamicSmem) return TRTX_ERR_UNSUPPORTED;
        smem_max = smem > smem_max ? smem : smem_max;
    }
    return launch_bands(yolop_preprocess_kernel, batch, net_w, net_h, dst_dev, smem_max, static_cast<cudaStream_t>(stream),
                        [&](int i, RcnnPreImage& im) { cls_band_image(TRTX_YOLO_V5, images_host[i], net_w, net_h, im); });
}

// DETR's preprocessImg stretches the whole frame over the whole net: the planar store with DETR's R, G, B planes and value
// chain.
TRTX_API int trtx_detr_preprocess_enqueue(const trtx_image_desc* images_host, int batch, int net_w, int net_h, float* dst_dev,
                                          trtx_stream_t stream) {
    return stretch_preprocess(detr_preprocess_kernel, images_host, batch, net_w, net_h, dst_dev,
                              static_cast<cudaStream_t>(stream));
}

// UFLD's prepareImage, likewise, with UFLD's fused value chain.
TRTX_API int trtx_ufld_preprocess_enqueue(const trtx_image_desc* images_host, int batch, int net_w, int net_h, float* dst_dev,
                                          trtx_stream_t stream) {
    return stretch_preprocess(ufld_preprocess_kernel, images_host, batch, net_w, net_h, dst_dev,
                              static_cast<cudaStream_t>(stream));
}

// RefineDet's base_transform, likewise, on a square net with its mean-subtracted planes.
TRTX_API int trtx_refinedet_preprocess_enqueue(const trtx_image_desc* images_host, int batch, int net, float* dst_dev,
                                               trtx_stream_t stream) {
    return stretch_preprocess(refinedet_preprocess_kernel, images_host, batch, net, net, dst_dev,
                              static_cast<cudaStream_t>(stream));
}

// preprocess_img with INTER_CUBIC (yolov3-tiny, retinafaceAntiCov): cls_band_image's V5 rectangle, the bicubic band kernel.
// A launch's dynamic shared memory is its widest rectangle times its most slots, so every launch is sized (and checked against
// the budget) before the first one.
TRTX_API int trtx_cubic_preprocess_enqueue(int variant, const trtx_image_desc* images_host, int batch, int net_w, int net_h,
                                           float* dst_dev, trtx_stream_t stream) {
    if (!images_host || batch <= 0 || !dst_dev || net_w <= 0 || net_h <= 0) return TRTX_ERR_INVALID;
    if (variant != TRTX_CUBIC_YOLOV3_TINY && variant != TRTX_CUBIC_ANTICOV) return TRTX_ERR_INVALID;
    if (reinterpret_cast<uintptr_t>(dst_dev) % sizeof(float) != 0) return TRTX_ERR_INVALID;
    // every descriptor is checked before the first launch, so that a rejected call writes nothing
    for (int i = 0; i < batch; ++i) {
        const trtx_image_desc& d = images_host[i];
        if (!d.data_dev || d.width <= 0 || d.height <= 0 || d.pitch < 3 * d.width) return TRTX_ERR_INVALID;
    }
    size_t smem_max = 0;
    for (int i0 = 0; i0 < batch; i0 += kMaxRcnnPreImages) {
        int wmax = 0, slots = 0;
        for (int i = i0; i < batch && i < i0 + kMaxRcnnPreImages; ++i) {
            RcnnPreImage im;
            if (!cls_band_image(TRTX_YOLO_V5, images_host[i], net_w, net_h, im)) return TRTX_ERR_UNSUPPORTED;
            wmax = im.rw > wmax ? im.rw : wmax;
            const int s = cubic_band_slots(im.scale_y);
            slots = s > slots ? s : slots;
        }
        const size_t smem = (size_t)slots * 3 * (size_t)wmax * sizeof(int);
        if (smem > kClsMaxDynamicSmem) return TRTX_ERR_UNSUPPORTED;
        smem_max = smem > smem_max ? smem : smem_max;
    }
    auto* kernel = variant == TRTX_CUBIC_YOLOV3_TINY ? cubic_preprocess_kernel<TRTX_CUBIC_YOLOV3_TINY>
                                                     : cubic_preprocess_kernel<TRTX_CUBIC_ANTICOV>;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (smem_max > 48 * 1024 &&
        cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_max) != cudaSuccess) {
        g_last_cuda_error = (int)cudaGetLastError();
        return TRTX_ERR_CUDA;
    }
    RcnnPreArgs a;
    a.net_w = net_w;
    a.net_h = net_h;
    a.bands = (net_h + kRcnnPreBand - 1) / kRcnnPreBand;
    for (int i0 = 0; i0 < batch; i0 += kMaxRcnnPreImages) {
        const int n = batch - i0 < kMaxRcnnPreImages ? batch - i0 : kMaxRcnnPreImages;
        int wmax = 0, slots = 0;
        for (int j = 0; j < n; ++j) {
            RcnnPreImage& im = a.img[j];
            cls_band_image(TRTX_YOLO_V5, images_host[i0 + j], net_w, net_h, im);
            im.dst_idx = i0 + j;
            wmax = im.rw > wmax ? im.rw : wmax;
            const int s = cubic_band_slots(im.scale_y);
            slots = s > slots ? s : slots;
        }
        a.stride = 3 * wmax;
        kernel<<<(unsigned)(n * a.bands), kRcnnPreThreads, (size_t)slots * a.stride * sizeof(int), st>>>(a, dst_dev);
        const int rc = check_launch();
        if (rc) return rc;
    }
    return TRTX_OK;
}

TRTX_API int trtx_yolov3spp_letterbox(int img_w, int img_h, int max_size, int out[6]) {
    if (!out || img_w <= 0 || img_h <= 0 || max_size <= 0) return TRTX_ERR_INVALID;
    const SppLetterbox lb = yolov3spp_letterbox(max_size, img_w, img_h);
    out[0] = lb.unpad_w + lb.dw;
    out[1] = lb.unpad_h + lb.dh;
    out[2] = lb.dw / 2;
    out[3] = lb.dh / 2;
    out[4] = lb.unpad_w;
    out[5] = lb.unpad_h;
    return lb.unpad_w > 0 && lb.unpad_h > 0 ? TRTX_OK : TRTX_ERR_UNSUPPORTED;
}

// preprocess_img with INTER_LINEAR (yolov3, yolov4, scaled-yolov4, RetinaFace: cls_band_image's V5 rectangle), yolov3-spp's
// letterbox (spp_band_image) or the Python runners' preprocess_image (py_band_image), the bilinear band kernel with the
// variant's planar store.
TRTX_API int trtx_linear_preprocess_enqueue(int variant, const trtx_image_desc* images_host, int batch, int net_w, int net_h,
                                            int max_size, float* dst_dev, trtx_stream_t stream) {
    if (!images_host || batch <= 0 || !dst_dev || net_w <= 0 || net_h <= 0) return TRTX_ERR_INVALID;
    if (variant != TRTX_LINEAR_YOLOV3 && variant != TRTX_LINEAR_RETINA && variant != TRTX_LINEAR_YOLOV3_SPP &&
        variant != TRTX_LINEAR_PY)
        return TRTX_ERR_INVALID;
    if (variant == TRTX_LINEAR_YOLOV3_SPP && max_size <= 0) return TRTX_ERR_INVALID;
    if (reinterpret_cast<uintptr_t>(dst_dev) % sizeof(float) != 0) return TRTX_ERR_INVALID;
    auto make = [&](int i, RcnnPreImage& im) -> int {
        if (variant == TRTX_LINEAR_YOLOV3_SPP) return spp_band_image(images_host[i], max_size, net_w, net_h, im);
        if (variant == TRTX_LINEAR_PY) return py_band_image(images_host[i], net_w, net_h, im);
        return cls_band_image(TRTX_YOLO_V5, images_host[i], net_w, net_h, im) ? TRTX_OK : TRTX_ERR_UNSUPPORTED;
    };
    // every descriptor is checked before the first launch, so that a rejected call writes nothing
    for (int i = 0; i < batch; ++i) {
        const trtx_image_desc& d = images_host[i];
        if (!d.data_dev || d.width <= 0 || d.height <= 0 || d.pitch < 3 * d.width) return TRTX_ERR_INVALID;
    }
    size_t smem_max = 0;
    for (int i = 0; i < batch; ++i) {
        RcnnPreImage im;
        const int rc = make(i, im);
        if (rc) return rc;
        const size_t smem = (size_t)kRcnnPreSlots * 3 * (size_t)im.rw * sizeof(int16_t);
        if (smem > kClsMaxDynamicSmem) return TRTX_ERR_UNSUPPORTED;
        smem_max = smem > smem_max ? smem : smem_max;
    }
    auto* kernel = variant == TRTX_LINEAR_YOLOV3 || variant == TRTX_LINEAR_PY
                       ? linear_preprocess_kernel<CubicInput<TRTX_CUBIC_YOLOV3_TINY>>
                   : variant == TRTX_LINEAR_RETINA ? linear_preprocess_kernel<RetinaInput>
                                                   : cls_preprocess_kernel<TRTX_YOLO_V8>;
    return launch_bands(kernel, batch, net_w, net_h, dst_dev, smem_max, static_cast<cudaStream_t>(stream),
                        [&](int i, RcnnPreImage& im) { make(i, im); });
}

}  // extern "C"
