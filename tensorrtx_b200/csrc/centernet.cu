// centernet.cu -- CenterNet (ctdet) pre-process and decode for sm_90a.
// Replaces the host stages of centernet/sample/test.py:
//   pre_process (:34-41)     a float64 L x L zero canvas with the frame at the top-left, cv.resize to net x net on float64,
//                            ((v / 255.) - 0.5) / 0.5, CHW in the frame's B, G, R order      -> centernet_preprocess_kernel
//   ctdet_decode (:44-102)   sigmoid, the 3 x 3 max_pool2d peak test, the per-class topk, the topk over C * K, the gathers of
//                            reg and wh, and the boxes                                        -> the two decode kernels
//   the driver loop (:126-132)  rows with score > 0.5, scaled by 4 * s                       -> the optional frame rows
//
// Decode, two launches, no atomics on global memory:
//   1. centernet_peaks_kernel, one CTA per (image, class) map: the map streams through shared memory in strips of
//      kCnStripCells cells with a one-row halo; each cell's sigmoid is computed once and the peak test reads its 3 x 3
//      window there.  Positive or NaN suppressed values are appended to a shared list in cell order (ordered compaction,
//      a ballot per warp and a scan of the warps' counts), and so are the first K zero-valued cells.  When the next strip
//      could overflow the list it is cut to its K best (cn_select).  The class-local top-K -- the reference's first topk --
//      goes to the workspace in cell order.
//   2. centernet_select_kernel, one CTA per image: cn_select takes the K best of the C * K candidates, which lie in flat
//      index order, a bitonic sort orders them, and each thread gathers reg and wh for one detection and writes dets and,
//      when asked, the frame rows.
// Order everywhere: NaN first, then descending value, ties to the smaller flat index c * H * W + y * W + x.  cn_select is a
// radix select of the cut key (4 histogram passes) whose ties at the cut are taken in list order, so that a list kept in
// flat-index order needs no index passes.
#include "common.cuh"
#include "select_sort.cuh"

namespace trtx {

constexpr int kCnPeakThreads = 512;
constexpr int kCnSelectThreads = 1024;
constexpr int kCnStripCells = 4096;  // cells of one strip: its rows are max(1, kCnStripCells / W)
constexpr int kCnMaxK = 1024;
constexpr int kCnMaxSide = 1024;     // H, W
constexpr int kCnMaxCells = 1 << 20;  // H * W
constexpr int kCnMaxClasses = 1024;
constexpr int kCnListCap = kCnStripCells + kCnMaxK;       // the shared candidate list: K kept + one strip
constexpr int kCnSigFloats = kCnStripCells + 2 * kCnMaxSide;  // the strip's sigmoids with a halo row above and below
constexpr size_t kCnPeakSmem = (size_t)kCnSigFloats * 4 + (size_t)kCnListCap * 8 + (size_t)kCnMaxK * 4;
constexpr int kCnRow = 6;            // x1, y1, x2, y2, score, class

// The select key: NaN above everything, then float_key (values are sigmoids or +0, never negative).
__device__ __forceinline__ uint32_t cn_key(float v) { return v != v ? 0xffffffffu : float_key(v); }

struct CnSelectScratch {
    int hist[256];
    int warp[32];
    int need, bucket;
};

// Exclusive rank of each thread's flag among the CTA's set flags in thread order, and their total.
template <int kThreads>
__device__ __forceinline__ int cn_block_rank(bool flag, CnSelectScratch& sc, int* total) {
    const int lane = threadIdx.x & (kWarp - 1), warp = threadIdx.x / kWarp;
    const unsigned m = __ballot_sync(0xffffffffu, flag);
    if (lane == 0) sc.warp[warp] = __popc(m);
    __syncthreads();
    int before = 0, t = 0;
#pragma unroll
    for (int w = 0; w < kThreads / kWarp; ++w) {
        const int c = sc.warp[w];
        before += w < warp ? c : 0;
        t += c;
    }
    __syncthreads();  // sc.warp is reused by the next call
    *total = t;
    return before + __popc(m & ((1u << lane) - 1u));
}

// The k best of list elements [0, n) under (key descending, position ascending), 0 < k <= n, written in list order:
// load(i) reads element i into a register value, store(j, v) writes the j-th selected one.  All of a chunk's loads happen
// before any of its stores, and the j-th selected element comes from a position >= j, so the list may be cut in place.
// Returns the cut key, the key of the k-th best.
template <int kThreads, class Item, class KeyOf, class Load, class Store>
__device__ uint32_t cn_select(int n, int k, CnSelectScratch& sc, KeyOf key_of, Load load, Store store) {
    const int tid = threadIdx.x, lane = tid & (kWarp - 1);
    uint32_t prefix = 0, mask = 0;
    int need = k;
    for (int pass = 0; pass < 4; ++pass) {
        const int shift = 24 - 8 * pass;
        for (int j = tid; j < 256; j += kThreads) sc.hist[j] = 0;
        __syncthreads();
        for (int i0 = 0; i0 < n; i0 += kThreads) {  // uniform, so that the whole warp meets the match
            const int i = i0 + tid;
            const uint32_t kk = i < n ? key_of(load(i)) : 0u;
            const bool in = i < n && (kk & mask) == prefix;
            // candidates crowd into a few buckets (every sigmoid in [0.5, 1) shares its top byte): one atomic per bucket
            // and warp
            const uint32_t bucket = (kk >> shift) & 255;
            const unsigned peers = __match_any_sync(0xffffffffu, in ? bucket : 256u + lane);
            if (in && lane == __ffs(peers) - 1) atomicAdd(&sc.hist[bucket], __popc(peers));
        }
        __syncthreads();
        if (tid < kWarp) {  // lane l holds buckets 255 - 8l down to 248 - 8l; a scan over the lanes finds the cut bucket
            int c[8], sum = 0;
#pragma unroll
            for (int j = 0; j < 8; ++j) sum += (c[j] = sc.hist[255 - 8 * lane - j]);
            int incl = sum;
#pragma unroll
            for (int o = 1; o < kWarp; o <<= 1) {
                const int t = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += t;
            }
            int cum = incl - sum;
            if (cum < need && need <= incl) {
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    if (cum + c[j] >= need) {
                        sc.bucket = 255 - 8 * lane - j;
                        sc.need = need - cum;
                        break;
                    }
                    cum += c[j];
                }
            }
        }
        __syncthreads();
        need = sc.need;
        prefix |= (uint32_t)sc.bucket << shift;
        mask |= 255u << shift;
    }
    // selected: key > cut, or key == cut among the first `need` such elements in list order
    int eq_before = 0, sel_before = 0;
    for (int i0 = 0; i0 < n; i0 += kThreads) {  // uniform
        const int i = i0 + tid;
        Item v{};
        uint32_t kk = 0;
        if (i < n) v = load(i), kk = key_of(v);
        int eq_total, sel_total;
        const int eq_rank = eq_before + cn_block_rank<kThreads>(i < n && kk == prefix, sc, &eq_total);
        const bool sel = i < n && (kk > prefix || (kk == prefix && eq_rank < need));
        const int pos = sel_before + cn_block_rank<kThreads>(sel, sc, &sel_total);
        if (sel) store(pos, v);
        eq_before += eq_total;
        sel_before += sel_total;
    }
    __syncthreads();
    return prefix;
}

struct CnCand {
    float v;
    uint32_t cell;
};

struct CnDecodeArgs {
    const float* heat;  // [B, C, H, W]
    const float* wh;    // [B, 2, H, W]
    const float* reg;   // [B, 2, H, W]
    float* cand_v;      // workspace [B, C, K]: class-local top-K values, in cell order
    uint32_t* cand_cell;  //           [B, C, K]: their cells y * W + x
    float* dets;        // [B, K, 6]
    float* rows;        // [B, 1 + K * 6] or null
    int C, H, W, K;
    float score_thresh;
    int base;           // select launch: frames [base, base + gridDim.x)
    float scale[kMaxFrames];  // select launch: (float)(down * (L / net)) per frame
};

__global__ void __launch_bounds__(kCnPeakThreads) centernet_peaks_kernel(const __grid_constant__ CnDecodeArgs a) {
    constexpr int T = kCnPeakThreads;
    extern __shared__ __align__(16) unsigned char cn_smem[];
    float* sig = reinterpret_cast<float*>(cn_smem);                  // [kCnSigFloats]
    float* lv = sig + kCnSigFloats;                                  // [kCnListCap] candidate values
    uint32_t* lc = reinterpret_cast<uint32_t*>(lv + kCnListCap);     // [kCnListCap] their cells
    uint32_t* zc = lc + kCnListCap;                                  // [K] the first K zero-valued cells
    __shared__ CnSelectScratch sc;
    const int tid = threadIdx.x;
    const int H = a.H, W = a.W, K = a.K;
    const float* x = a.heat + (size_t)blockIdx.x * H * W;
    const int R = max(1, kCnStripCells / W);
    auto key_of = [](CnCand c) { return cn_key(c.v); };
    auto load = [&](int i) { return CnCand{lv[i], lc[i]}; };
    auto store = [&](int j, CnCand c) { lv[j] = c.v, lc[j] = c.cell; };
    int n = 0, nz = 0;  // list length, zero cells kept
    // once the list has been cut, a later cell needs a key above the cut: at the cut it would lose the tie to K earlier ones
    uint32_t floor_key = 0;
    for (int y0 = 0; y0 < H; y0 += R) {
        const int rows = min(R, H - y0), cells = rows * W;
        if (n + cells > kCnListCap) {  // uniform
            floor_key = cn_select<T, CnCand>(n, K, sc, key_of, load, store);
            n = K;
        }
        // sigmoids of rows y0 - 1 .. y0 + rows (clipped); row y0 - 1 + r of the map is row r of sig
        const int ya = max(y0 - 1, 0), yb = min(y0 + rows + 1, H);
        const int off = (ya - (y0 - 1)) * W, cnt = (yb - ya) * W;
        const float* src = x + (size_t)ya * W;
        for (int i = tid; i < cnt; i += 4 * T) {
            float v[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) v[j] = i + j * T < cnt ? ldg_stream_f1(src + i + j * T) : 0.f;
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (i + j * T < cnt) sig[off + i + j * T] = logist(v[j]);
        }
        __syncthreads();
        for (int i0 = 0; i0 < cells; i0 += T) {  // uniform
            const int i = i0 + tid;
            bool cand = false, zero = false;
            float v = 0.f;
            uint32_t cell = 0;
            if (i < cells) {
                const int r = i / W, cx = i - r * W, y = y0 + r;
                const float* c = sig + (r + 1) * W + cx;
                const float s = *c;
                // a peak iff s equals the max of its clipped 3 x 3 window: every neighbour <= s, which fails on any NaN
                bool peak = true;
#pragma unroll
                for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
                    for (int dx = -1; dx <= 1; ++dx)
                        if ((unsigned)(y + dy) < (unsigned)H && (unsigned)(cx + dx) < (unsigned)W) peak &= c[dy * W + dx] <= s;
                v = peak ? s : __fmul_rn(s, 0.f);  // heat * keep: +0, or NaN for a NaN cell
                zero = !(v > 0.f || v != v);
                cand = !zero && cn_key(v) > floor_key;
                cell = (uint32_t)(y * W + cx);
            }
            int tot, ztot;
            const int pos = n + cn_block_rank<T>(cand, sc, &tot);
            if (cand) lv[pos] = v, lc[pos] = cell;
            if (nz < K) {  // uniform
                const int zpos = nz + cn_block_rank<T>(zero, sc, &ztot);
                if (zero && zpos < K) zc[zpos] = cell;
                nz = min(K, nz + ztot);
            }
            n += tot;
        }
        __syncthreads();  // sig is rewritten by the next strip
    }
    float* ov = a.cand_v + (size_t)blockIdx.x * K;
    uint32_t* oc = a.cand_cell + (size_t)blockIdx.x * K;
    if (n >= K) {
        if (n > K) cn_select<T, CnCand>(n, K, sc, key_of, load, store);
        for (int i = tid; i < K; i += T) ov[i] = lv[i], oc[i] = lc[i];
    } else {
        // fewer than K positive or NaN cells: the rest are the first K - n zero-valued cells; merge the two lists, both in
        // cell order, by ranking each element in the other list
        const int nzu = K - n;
        for (int i = tid; i < n + nzu; i += T) {
            const bool from_list = i < n;
            const uint32_t cell = from_list ? lc[i] : zc[i - n];
            const uint32_t* other = from_list ? zc : lc;
            int lo = 0, hi = from_list ? nzu : n;  // elements of the other list with a smaller cell
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (other[mid] < cell) lo = mid + 1; else hi = mid;
            }
            const int pos = (from_list ? i : i - n) + lo;
            ov[pos] = from_list ? lv[i] : 0.f;
            oc[pos] = cell;
        }
    }
}

__global__ void __launch_bounds__(kCnSelectThreads) centernet_select_kernel(const __grid_constant__ CnDecodeArgs a) {
    constexpr int T = kCnSelectThreads;
    __shared__ unsigned long long s_key[kCnMaxK];  // (~key << 32) | slot, slots in flat-index order
    __shared__ int s_src[kCnMaxK];                 // candidate index c * K + j of each slot
    __shared__ CnSelectScratch sc;
    const int tid = threadIdx.x, b = a.base + blockIdx.x, K = a.K, n = a.C * K;
    const float* cv = a.cand_v + (size_t)b * n;
    cn_select<T, int>(n, K, sc, [&](int i) { return cn_key(cv[i]); }, [](int i) { return i; },
                      [&](int j, int i) { s_src[j] = i; });
    int S = 1;
    while (S < K) S <<= 1;
    for (int j = tid; j < S; j += T)
        s_key[j] = j < K ? ((unsigned long long)(~cn_key(cv[s_src[j]])) << 32) | (unsigned)j : ~0ull;
    __syncthreads();
    block_bitonic_sort_u64(s_key, S);
    const int HW = a.H * a.W;
    float score = 0.f;
    int keep_rank = 0;
    float box[4] = {0.f, 0.f, 0.f, 0.f}, cls = 0.f;
    if (tid < K) {
        const int src = s_src[(int)(s_key[tid] & 0xffffffffu)], c = src / K;
        const uint32_t cell = a.cand_cell[(size_t)b * n + src];
        score = cv[src];
        // (float)(int)((float)cell / (float)W) of the reference: the accepted H, W keep that equal to the integer quotient
        const float xs0 = (float)(cell % (uint32_t)a.W), ys0 = (float)(cell / (uint32_t)a.W);
        const float* reg = a.reg + (size_t)b * 2 * HW + cell;
        const float* wh = a.wh + (size_t)b * 2 * HW + cell;
        const float xs = __fadd_rn(xs0, __ldg(reg)), ys = __fadd_rn(ys0, __ldg(reg + HW));
        const float hw = __fdiv_rn(__ldg(wh), 2.f), hh = __fdiv_rn(__ldg(wh + HW), 2.f);
        box[0] = __fsub_rn(xs, hw);
        box[1] = __fsub_rn(ys, hh);
        box[2] = __fadd_rn(xs, hw);
        box[3] = __fadd_rn(ys, hh);
        cls = (float)c;
        float* d = a.dets + ((size_t)b * K + tid) * kCnRow;
#pragma unroll
        for (int e = 0; e < 4; ++e) d[e] = box[e];
        d[4] = score;
        d[5] = cls;
    }
    if (!a.rows) return;  // uniform
    // the driver's `if i[-2] > 0.5`: NaN scores come first and fail it, the kept ones follow as one run
    const bool keep = tid < K && score > a.score_thresh;
    const int nan = __syncthreads_count(tid < K && score != score), kept = __syncthreads_count(keep);
    keep_rank = tid - nan;
    float* out = a.rows + (size_t)b * (1 + (size_t)K * kCnRow);
    const float k = a.scale[blockIdx.x];
    if (keep) {
        float* o = out + 1 + (size_t)keep_rank * kCnRow;
#pragma unroll
        for (int e = 0; e < 4; ++e) o[e] = __fmul_rn(box[e], k);
        o[4] = score;
        o[5] = cls;
    }
    for (int f = 1 + kept * kCnRow + tid; f < 1 + K * kCnRow; f += T) out[f] = 0.f;
    if (tid == 0) out[0] = (float)kept;
}

// -------------------------------------------------------------------------------------------------------------------------
// pre_process: out(c, y, x) = (float)(((v / 255.) - 0.5) / 0.5) with v the float64 INTER_LINEAR resize of the L x L canvas,
// L = max(h, w, 3).  cv.resize on float64 is separable with float weights (1 - f, f) from cv_linear_coord, the tap clamped
// with its fraction zeroed at both ends on both axes; each pass is a0 * p0 + a1 * p1 in double.  _rn intrinsics so that nvcc
// cannot contract a product into a DFMA.  One thread per output pixel, three planes B, G, R.
constexpr int kCnPreThreads = 256;
constexpr int kCnMaxNet = 8192;

struct CnPreImage {
    const uint8_t* src;
    double scale;  // cv::resize: 1. / ((double)net / L)
    int w, h, pitch, L;
};
struct CnPreArgs {
    CnPreImage img[kMaxFrames];
    int net, base;
};

__global__ void __launch_bounds__(kCnPreThreads) centernet_preprocess_kernel(const __grid_constant__ CnPreArgs a,
                                                                              float* __restrict__ dst) {
    const CnPreImage& im = a.img[blockIdx.y];
    const int net = a.net, p = blockIdx.x * kCnPreThreads + threadIdx.x;
    if (p >= net * net) return;
    const int y = p / net, x = p - y * net;
    const LinearCoord tx = cv_linear_coord(x, im.scale, im.L, true), ty = cv_linear_coord(y, im.scale, im.L, true);
    const int xs[2] = {tx.s, min(tx.s + 1, im.L - 1)}, ys[2] = {ty.s, min(ty.s + 1, im.L - 1)};
    const double ax[2] = {(double)__fsub_rn(1.f, tx.f), (double)tx.f}, ay[2] = {(double)__fsub_rn(1.f, ty.f), (double)ty.f};
    // the canvas: the frame at the top-left, zeros elsewhere; a one-pixel-wide frame fills every column (numpy broadcasts it)
    double hrow[2][3];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const uint8_t* row = im.src + (size_t)ys[r] * im.pitch;
        double px[2][3];
#pragma unroll
        for (int t = 0; t < 2; ++t) {
            const bool in = ys[r] < im.h && (im.w == 1 || xs[t] < im.w);
            const int col = im.w == 1 ? 0 : xs[t];
#pragma unroll
            for (int c = 0; c < 3; ++c) px[t][c] = in ? (double)__ldg(row + 3 * col + c) : 0.0;
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) hrow[r][c] = __dadd_rn(__dmul_rn(px[0][c], ax[0]), __dmul_rn(px[1][c], ax[1]));
    }
    const size_t plane = (size_t)net * net;
    float* o = dst + (size_t)(a.base + blockIdx.y) * 3 * plane + p;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const double v = __dadd_rn(__dmul_rn(hrow[0][c], ay[0]), __dmul_rn(hrow[1][c], ay[1]));
        o[c * plane] = __double2float_rn(__ddiv_rn(__dsub_rn(__ddiv_rn(v, 255.0), 0.5), 0.5));
    }
}

}  // namespace trtx

using namespace trtx;

extern "C" {

// Everything in the parameters and the frame sizes (frame_wh_host, may be null) that can reject a decode call, before the
// first launch, in two passes so that TRTX_ERR_INVALID wins; TRTX_OK or the error code.
static int centernet_check(const trtx_centernet_params* p, int batch, const int32_t* frame_wh_host) {
    if (!p || batch <= 0) return TRTX_ERR_INVALID;
    if (p->num_classes <= 0 || p->height <= 0 || p->width <= 0 || p->k <= 0) return TRTX_ERR_INVALID;
    if ((int64_t)p->k > (int64_t)p->height * p->width) return TRTX_ERR_INVALID;  // the reference's topk raises
    if (frame_wh_host && (p->net <= 0 || p->down <= 0 || !(p->score_thresh == p->score_thresh) ||
                          !frames_valid(frame_wh_host, batch)))
        return TRTX_ERR_INVALID;
    if (p->num_classes > kCnMaxClasses || p->height > kCnMaxSide || p->width > kCnMaxSide ||
        (int64_t)p->height * p->width > kCnMaxCells || p->k > kCnMaxK)
        return TRTX_ERR_UNSUPPORTED;
    return TRTX_OK;
}

TRTX_API size_t trtx_centernet_workspace_size(const trtx_centernet_params* p, int batch) {
    if (centernet_check(p, batch, nullptr) != TRTX_OK) return 0;
    return align_up((size_t)batch * p->num_classes * p->k * sizeof(float)) * 2;
}

TRTX_API int trtx_centernet_decode_enqueue(const trtx_centernet_params* p, int batch, const float* heat_dev,
                                           const float* wh_dev, const float* reg_dev, void* workspace_dev,
                                           size_t workspace_bytes, float* dets_dev, const int32_t* frame_wh_host,
                                           float* rows_dev, trtx_stream_t stream) {
    if (!heat_dev || !wh_dev || !reg_dev || !workspace_dev || !dets_dev) return TRTX_ERR_INVALID;
    if (!frame_wh_host != !rows_dev) return TRTX_ERR_INVALID;  // the frame rows need both
    if (reinterpret_cast<uintptr_t>(workspace_dev) % kAlign) return TRTX_ERR_INVALID;
    int rc = centernet_check(p, batch, frame_wh_host);
    if (rc) return rc;
    if (workspace_bytes < trtx_centernet_workspace_size(p, batch)) return TRTX_ERR_WORKSPACE;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    if ((rc = opt_in_smem(centernet_peaks_kernel, kCnPeakSmem))) return rc;
    CnDecodeArgs a;
    a.heat = heat_dev;
    a.wh = wh_dev;
    a.reg = reg_dev;
    const size_t half = align_up((size_t)batch * p->num_classes * p->k * sizeof(float));
    a.cand_v = static_cast<float*>(workspace_dev);
    a.cand_cell = reinterpret_cast<uint32_t*>(static_cast<char*>(workspace_dev) + half);
    a.dets = dets_dev;
    a.rows = rows_dev;
    a.C = p->num_classes;
    a.H = p->height;
    a.W = p->width;
    a.K = p->k;
    a.score_thresh = p->score_thresh;
    a.base = 0;
    centernet_peaks_kernel<<<(unsigned)(batch * p->num_classes), kCnPeakThreads, kCnPeakSmem, st>>>(a);
    if ((rc = check_launch())) return rc;
    return launch_frames(centernet_select_kernel, a, a.base, batch, kCnSelectThreads, 0, st, frame_wh(frame_wh_host),
                         [&](int j, int w, int h) {
                             const int L = max(max(h, w), 3);  // max(image.shape): the channel count takes part
                             a.scale[j] = (float)((double)p->down * ((double)L / (double)p->net));
                         });
}

TRTX_API int trtx_centernet_preprocess_enqueue(const trtx_image_desc* images_host, int batch, int net, float* dst_dev,
                                               trtx_stream_t stream) {
    if (!images_host || batch <= 0 || !dst_dev || net <= 0) return TRTX_ERR_INVALID;
    if (reinterpret_cast<uintptr_t>(dst_dev) % sizeof(float) != 0) return TRTX_ERR_INVALID;
    // every descriptor is checked before the first launch, so that a rejected call writes nothing
    if (!valid_images(images_host, batch)) return TRTX_ERR_INVALID;
    if (net > kCnMaxNet) return TRTX_ERR_UNSUPPORTED;
    CnPreArgs a;
    a.net = net;
    for (int i0 = 0; i0 < batch; i0 += kMaxFrames) {
        const int n = min(batch - i0, kMaxFrames);
        a.base = i0;
        for (int j = 0; j < n; ++j) {
            const trtx_image_desc& d = images_host[i0 + j];
            CnPreImage& im = a.img[j];
            im.src = d.data_dev;
            im.w = d.width;
            im.h = d.height;
            im.pitch = d.pitch;
            im.L = max(max(d.width, d.height), 3);
            im.scale = 1. / ((double)net / im.L);
        }
        const dim3 grid((unsigned)(((size_t)net * net + kCnPreThreads - 1) / kCnPreThreads), (unsigned)n);
        centernet_preprocess_kernel<<<grid, kCnPreThreads, 0, static_cast<cudaStream_t>(stream)>>>(a, dst_dev);
        const int rc = check_launch();
        if (rc) return rc;
    }
    return TRTX_OK;
}

}  // extern "C"
