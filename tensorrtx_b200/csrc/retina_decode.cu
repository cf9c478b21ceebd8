// retina_decode.cu -- Decode_TRT (RetinaFace) for sm_90a.
// Replaces CalDetection/forwardGpu of retinaface/decode.cu:110-191 (3 launches + B memsets, float
// atomics on one counter per image) with one scan launch over all strides/images + one pack launch.
//
// Per level the input is [B, 32, g]: rows 0-7 bbox (2 priors x 4), 8-11 cls (2 x 2), 12-31 lmk (2 x 10)
// (decode.cu:121-123).  Only the 4 cls rows are streamed for every cell (128-bit loads along the
// cell axis); the 28 regression rows are touched only for priors that pass the gate.  Candidates go
// to per-tile slots (same atomic-free scheme as the YoloLayer scan), then a pack kernel writes the
// reference buffer [count, Detection(15 floats) rows] in ascending prior order.
//
// The reference's literals 0.5, 0.1, 0.2 are doubles: those expressions are evaluated in fp64 here too
// (a handful of DFMA per candidate; irrelevant for throughput).
//
// variant TRTX_RETINA_ANTICOV = retinafaceAntiCov/decode.cu:110-172 through the same two kernels: [B, 38, g] inputs
// (cls 4 | bbox 8 | lmk 20 | type 6; the network already soft-maxed cls/type, :124-127), 2 cls rows streamed, pixel-unit
// priors (7.5 + x*step, anchor*2/(k+1) in INTEGER arithmetic), 16-float rows ending in the mask confidence.  The
// reference handles batch 1 only (no image offset); here every image of the batch is decoded.
#include "common.cuh"

namespace trtx {

struct RetinaLevel {
    const void* in;  // [B, 32 | 38, g] of the scan's element type
    int g, w, h;
    int tile_begin;
    int slot_begin;
    int anchor;  // 16 * 4^level (decode.cu:170-189)
};
struct RetinaArgs {
    RetinaLevel lv[3];
    int det_floats;  // 15 (retinaface/decode.h:11-15) | 16 (retinafaceAntiCov/decode.h:13-18)
    int tiles_per_image, slots_per_image, tile_cells;
    int in_h, in_w;
    float gate;
    int* tile_count;
    float* cand;  // [B, slots, 16]
    int total_priors;
};

// T: the heads' element type (float | __half).  Every read goes through Elem<T>, which widens a half to float exactly, so
// the decode below -- the double-precision literals included -- is the same code on the same floats in both modes.
template <typename T, int VEC>
__global__ void __launch_bounds__(128) retina_scan_kernel(const __grid_constant__ RetinaArgs a, int batch) {
    constexpr int TILE = 32 * VEC;
    const int lane = threadIdx.x & 31;
    const int gw = blockIdx.x * 4 + (threadIdx.x >> 5);  // global warp = (image, tile)
    if (gw >= batch * a.tiles_per_image) return;
    const int b = gw / a.tiles_per_image;
    const int t = gw - b * a.tiles_per_image;
    int l = 0;
    while (l + 1 < 3 && t >= a.lv[l + 1].tile_begin) ++l;
    const RetinaLevel& L = a.lv[l];
    const int tile = t - L.tile_begin;
    const int a0 = tile * TILE + lane * VEC;
    const size_t g = (size_t)L.g;
    const bool active = a0 < L.g;
    const T* cur = static_cast<const T*>(L.in) + (size_t)b * 32 * g;
    const T* cls_reg = cur + 8 * g;

    float c[4][VEC];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
#pragma unroll
        for (int j = 0; j < VEC; ++j) c[r][j] = 0.0f;
        if (active) {
            if constexpr (VEC == 4) {
                float4 v = Elem<T>::ld4(cls_reg + (size_t)r * g + a0);
                c[r][0] = v.x;
                c[r][1] = v.y;
                c[r][2] = v.z;
                c[r][3] = v.w;
            } else {
                c[r][0] = Elem<T>::ld1(cls_reg + (size_t)r * g + a0);
            }
        }
    }
    unsigned flags = 0;
    float conf[VEC][2];
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const float conf1 = c[2 * k][j], conf2 = c[2 * k + 1][j];
            const float e1 = expf(conf1), e2 = expf(conf2);
            const float p = e2 / (e1 + e2);  // decode.cu:130
            conf[j][k] = p;
            // decode.cu:131 `if (conf2 <= 0.02) continue;` (gate already rounded for the double compare)
            if (active && (a0 + j < L.g) && !(p <= a.gate)) flags |= 1u << (j * 2 + k);
        }
    }
    int total;
    int off = warp_excl_scan(__popc(flags), lane, &total);
    if (lane == 0) a.tile_count[(size_t)b * a.tiles_per_image + t] = total;
    if (!flags) return;
    const size_t slot0 = (size_t)b * a.slots_per_image + L.slot_begin + (size_t)tile * TILE * 2;
    const T* bbox_reg = cur;
    const T* lmk_reg = cur + 12 * g;
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            if (!(flags & (1u << (j * 2 + k)))) continue;
            const int idx = a0 + j;
            const int y = idx / L.w, x = idx - y * L.w;
            float prior[4];  // decode.cu:138-142
            prior[0] = (float)(((double)(float)x + 0.5) / L.w);
            prior[1] = (float)(((double)(float)y + 0.5) / L.h);
            prior[2] = (float)L.anchor * (k + 1) / a.in_w;
            prior[3] = (float)L.anchor * (k + 1) / a.in_h;
            float d[15];
            const T* br = bbox_reg + idx + (size_t)k * 4 * g;
            d[0] = (float)(prior[0] + (double)Elem<T>::ld1_cached(br) * 0.1 * prior[2]);  // :145-156
            d[1] = (float)(prior[1] + (double)Elem<T>::ld1_cached(br + g) * 0.1 * prior[3]);
            d[2] = prior[2] * expf((float)((double)Elem<T>::ld1_cached(br + 2 * g) * 0.2));
            d[3] = prior[3] * expf((float)((double)Elem<T>::ld1_cached(br + 3 * g) * 0.2));
            d[0] -= d[2] / 2;
            d[1] -= d[3] / 2;
            d[2] += d[0];
            d[3] += d[1];
            d[0] *= a.in_w;
            d[1] *= a.in_h;
            d[2] *= a.in_w;
            d[3] *= a.in_h;
            d[4] = conf[j][k];
            const T* lr = lmk_reg + idx + (size_t)k * 10 * g;
#pragma unroll
            for (int i = 0; i < 10; i += 2) {  // :158-163
                d[5 + i] = (float)(prior[0] + (double)Elem<T>::ld1_cached(lr + (size_t)i * g) * 0.1 * prior[2]);
                d[5 + i + 1] = (float)(prior[1] + (double)Elem<T>::ld1_cached(lr + (size_t)(i + 1) * g) * 0.1 * prior[3]);
                d[5 + i] *= a.in_w;
                d[5 + i + 1] *= a.in_h;
            }
            float4* rec = reinterpret_cast<float4*>(a.cand + (slot0 + off) * 16);
            rec[0] = make_float4(d[0], d[1], d[2], d[3]);
            rec[1] = make_float4(d[4], d[5], d[6], d[7]);
            rec[2] = make_float4(d[8], d[9], d[10], d[11]);
            rec[3] = make_float4(d[12], d[13], d[14], __int_as_float(L.slot_begin + idx * 2 + k));
            ++off;
        }
    }
}

// retinafaceAntiCov/decode.cu:110-155.  Same tiling; the face probability of prior k is channel 2+k as it comes.
template <typename T, int VEC>
__global__ void __launch_bounds__(128) anticov_scan_kernel(const __grid_constant__ RetinaArgs a, int batch) {
    constexpr int TILE = 32 * VEC;
    const int lane = threadIdx.x & 31;
    const int gw = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (gw >= batch * a.tiles_per_image) return;
    const int b = gw / a.tiles_per_image;
    const int t = gw - b * a.tiles_per_image;
    int l = 0;
    while (l + 1 < 3 && t >= a.lv[l + 1].tile_begin) ++l;
    const RetinaLevel& L = a.lv[l];
    const int tile = t - L.tile_begin;
    const int a0 = tile * TILE + lane * VEC;
    const size_t g = (size_t)L.g;
    const bool active = a0 < L.g;
    const T* cur = static_cast<const T*>(L.in) + (size_t)b * 38 * g;
    const T* cls_reg = cur + 2 * g;  // :120
    float c[2][VEC];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
#pragma unroll
        for (int j = 0; j < VEC; ++j) c[r][j] = 0.0f;
        if (active) {
            if constexpr (VEC == 4) {
                float4 v = Elem<T>::ld4(cls_reg + (size_t)r * g + a0);
                c[r][0] = v.x;
                c[r][1] = v.y;
                c[r][2] = v.z;
                c[r][3] = v.w;
            } else {
                c[r][0] = Elem<T>::ld1(cls_reg + (size_t)r * g + a0);
            }
        }
    }
    unsigned flags = 0;
#pragma unroll
    for (int j = 0; j < VEC; ++j)
#pragma unroll
        for (int k = 0; k < 2; ++k)  // :127 `if (conf < 0.5) continue;` (0.5 is exact in fp32: the double compare is the float compare)
            if (active && (a0 + j < L.g) && !(c[k][j] < 0.5f)) flags |= 1u << (j * 2 + k);
    int total;
    int off = warp_excl_scan(__popc(flags), lane, &total);
    if (lane == 0) a.tile_count[(size_t)b * a.tiles_per_image + t] = total;
    if (!flags) return;
    const size_t slot0 = (size_t)b * a.slots_per_image + L.slot_begin + (size_t)tile * TILE * 2;
    const T* bbox_reg = cur + 4 * g;
    const T* lmk_reg = cur + 12 * g;
    const T* mask_reg = cur + 36 * g;
    // The level's fixed stride 8, 16, 32 (forwardGpu's base_step, :162-170).  Not in_w / w: with floor grids that is another
    // number whenever the stride does not divide in_w (in_w = 660 gives 33 at level 2), and it would move x and y alike.
    const int step = 8 << l;
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            if (!(flags & (1u << (j * 2 + k)))) continue;
            const int idx = a0 + j;
            const int y = idx / L.w, x = idx - y * L.w;
            float prior[4];  // :134-138
            prior[0] = (float)(7.5 + (double)(float)(x * step));
            prior[1] = (float)(7.5 + (double)(float)(y * step));
            prior[2] = (float)(L.anchor * 2 / (k + 1));
            prior[3] = prior[2];
            float d[16];
            const T* br = bbox_reg + idx + (size_t)k * 4 * g;
            d[0] = prior[0] + Elem<T>::ld1_cached(br) * prior[2];  // :141-148 (float; contracted like the reference build)
            d[1] = prior[1] + Elem<T>::ld1_cached(br + g) * prior[3];
            d[2] = prior[2] * expf(Elem<T>::ld1_cached(br + 2 * g));
            d[3] = prior[3] * expf(Elem<T>::ld1_cached(br + 3 * g));
            d[0] -= (d[2] - 1) / 2;
            d[1] -= (d[3] - 1) / 2;
            d[2] += d[0];
            d[3] += d[1];
            d[4] = c[k][j];
            const T* lr = lmk_reg + idx + (size_t)k * 10 * g;
#pragma unroll
            for (int i = 0; i < 10; i += 2) {  // :150-153: `* 0.2` promotes to double
                d[5 + i] = (float)(prior[0] + (double)Elem<T>::ld1_cached(lr + (size_t)i * g) * 0.2 * prior[2]);
                d[5 + i + 1] = (float)(prior[1] + (double)Elem<T>::ld1_cached(lr + (size_t)(i + 1) * g) * 0.2 * prior[3]);
            }
            d[15] = Elem<T>::ld1_cached(mask_reg + idx + (size_t)k * g);  // :154
            float4* rec = reinterpret_cast<float4*>(a.cand + (slot0 + off) * 16);
            rec[0] = make_float4(d[0], d[1], d[2], d[3]);
            rec[1] = make_float4(d[4], d[5], d[6], d[7]);
            rec[2] = make_float4(d[8], d[9], d[10], d[11]);
            rec[3] = make_float4(d[12], d[13], d[14], d[15]);
            ++off;
        }
    }
}

// Tiles whose row offsets one pass of the pack holds in shared memory.  An image of more tiles takes several passes, each
// starting from the rows of the passes before it, so no input size is refused for the pack and its shared memory is the
// same for every call (640x640 has 67 tiles per image: one pass).
constexpr int kPackChunk = 1024;

__global__ void __launch_bounds__(256) retina_pack_kernel(const __grid_constant__ RetinaArgs a, float* __restrict__ out) {
    __shared__ int s_prefix[kPackChunk + 1];
    const int b = blockIdx.x;
    const int T_ = a.tiles_per_image;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const int* cnt = a.tile_count + (size_t)b * T_;
    const int F = a.det_floats;
    float* o = out + (size_t)b * (1 + (size_t)a.total_priors * F);
    const int tile_slots = a.tile_cells * 2;
    int carry = 0;  // rows of the tiles before this pass
    for (int c0 = 0; c0 < T_; c0 += kPackChunk) {
        const int nt = min(kPackChunk, T_ - c0);
        if (warp == 0) {
            int run = carry;
            for (int base = 0; base < nt; base += 32) {
                int v = (base + lane < nt) ? cnt[c0 + base + lane] : 0;
                int tot;
                int ex = warp_excl_scan(v, lane, &tot);
                if (base + lane < nt) s_prefix[base + lane] = run + ex;
                run += tot;
            }
            if (lane == 0) s_prefix[nt] = run;
        }
        __syncthreads();
        for (int i = warp; i < nt; i += nwarps) {
            const int n = s_prefix[i + 1] - s_prefix[i];
            if (n == 0) continue;
            const int t = c0 + i;
            int l = 0;
            while (l + 1 < 3 && t >= a.lv[l + 1].tile_begin) ++l;
            const size_t slot0 =
                    (size_t)b * a.slots_per_image + a.lv[l].slot_begin + (size_t)(t - a.lv[l].tile_begin) * tile_slots;
            // n records x F floats, copied by the whole warp
            for (int e = lane; e < n * F; e += 32) {
                const int j = e / F, f = e - j * F;
                o[1 + (size_t)(s_prefix[i] + j) * F + f] = a.cand[(slot0 + j) * 16 + f];
            }
        }
        carry = s_prefix[nt];
        __syncthreads();  // the next pass rewrites s_prefix
    }
    if (threadIdx.x == 0) o[0] = (float)carry;
}

struct RetinaLayout {
    int vec, tile_cells, tiles, slots;
    int tile_begin[3], slot_begin[3];
    size_t off_cand, total;
};
static RetinaLayout retina_layout(const trtx_retina_params* p, int batch, int vec) {
    RetinaLayout L{};
    L.vec = vec;
    L.tile_cells = 32 * vec;
    int step = 8;
    for (int l = 0; l < 3; ++l, step *= 2) {
        int g = (p->in_h / step) * (p->in_w / step);
        L.tile_begin[l] = L.tiles;
        L.slot_begin[l] = L.slots;
        L.tiles += (g + L.tile_cells - 1) / L.tile_cells;
        L.slots += g * 2;
    }
    L.off_cand = align_up(sizeof(int) * (size_t)batch * L.tiles);
    L.total = L.off_cand + align_up(sizeof(float) * 16 * (size_t)batch * L.slots);
    return L;
}

template <typename T>
static void retina_scan_launch(bool anticov, int vec, const RetinaArgs& a, int batch, int warps, cudaStream_t st) {
    if (anticov) {
        if (vec == 4)
            anticov_scan_kernel<T, 4><<<(warps + 3) / 4, 128, 0, st>>>(a, batch);
        else
            anticov_scan_kernel<T, 1><<<(warps + 3) / 4, 128, 0, st>>>(a, batch);
    } else if (vec == 4)
        retina_scan_kernel<T, 4><<<(warps + 3) / 4, 128, 0, st>>>(a, batch);
    else
        retina_scan_kernel<T, 1><<<(warps + 3) / 4, 128, 0, st>>>(a, batch);
}

}  // namespace trtx

using namespace trtx;

extern "C" {

TRTX_API int trtx_retina_total_priors(const trtx_retina_params* p) {
    if (!p || p->in_h < 32 || p->in_w < 32) return 0;
    int n = 0;
    for (int s = 8; s <= 32; s *= 2) n += (p->in_h / s) * (p->in_w / s) * 2;  // decode.cu:33-41
    return n;
}

TRTX_API size_t trtx_retina_workspace_size(const trtx_retina_params* p, int batch) {
    if (!p || batch <= 0 || p->in_h < 32 || p->in_w < 32) return 0;
    return retina_layout(p, batch, 1).total;
}

TRTX_API int trtx_retina_decode_enqueue(const trtx_retina_params* p, int batch, const void* const* inputs_dev,
                                        float* output_dev, void* workspace_dev, size_t workspace_bytes,
                                        trtx_stream_t stream) {
    if (!p || batch <= 0 || !inputs_dev || !output_dev || !workspace_dev) return TRTX_ERR_INVALID;
    if (p->in_h < 32 || p->in_w < 32) return TRTX_ERR_INVALID;
    if (p->variant != TRTX_RETINA_FACE && p->variant != TRTX_RETINA_ANTICOV) return TRTX_ERR_INVALID;
    if (p->in_dtype != TRTX_F32 && p->in_dtype != TRTX_F16) return TRTX_ERR_INVALID;
    const size_t elem = p->in_dtype == TRTX_F16 ? sizeof(__half) : sizeof(float);
    if (reinterpret_cast<uintptr_t>(output_dev) % sizeof(float) != 0) return TRTX_ERR_INVALID;
    int vec = 4, step = 8;
    for (int l = 0; l < 3; ++l, step *= 2) {
        if (!inputs_dev[l] || reinterpret_cast<uintptr_t>(inputs_dev[l]) % elem != 0) return TRTX_ERR_INVALID;
        int g = (p->in_h / step) * (p->in_w / step);
        if (g % 4 != 0 || reinterpret_cast<uintptr_t>(inputs_dev[l]) % (4 * elem) != 0) vec = 1;  // four cells per load
    }
    RetinaLayout L = retina_layout(p, batch, vec);
    if (workspace_bytes < L.total) return TRTX_ERR_WORKSPACE;
    RetinaArgs a{};
    step = 8;
    int anchor = 16;
    for (int l = 0; l < 3; ++l, step *= 2, anchor *= 4) {
        a.lv[l].in = inputs_dev[l];
        a.lv[l].h = p->in_h / step;
        a.lv[l].w = p->in_w / step;
        a.lv[l].g = a.lv[l].h * a.lv[l].w;
        a.lv[l].tile_begin = L.tile_begin[l];
        a.lv[l].slot_begin = L.slot_begin[l];
        a.lv[l].anchor = anchor;
    }
    a.tiles_per_image = L.tiles;
    a.slots_per_image = L.slots;
    a.tile_cells = L.tile_cells;
    a.in_h = p->in_h;
    a.in_w = p->in_w;
    a.gate = p->gate;
    a.tile_count = static_cast<int*>(workspace_dev);
    a.cand = reinterpret_cast<float*>(static_cast<char*>(workspace_dev) + L.off_cand);
    a.total_priors = trtx_retina_total_priors(p);
    a.det_floats = p->variant == TRTX_RETINA_ANTICOV ? 16 : 15;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int warps = batch * L.tiles;
    const bool anticov = p->variant == TRTX_RETINA_ANTICOV;
    if (p->in_dtype == TRTX_F16)
        retina_scan_launch<__half>(anticov, vec, a, batch, warps, st);
    else
        retina_scan_launch<float>(anticov, vec, a, batch, warps, st);
    int rc = check_launch();
    if (rc) return rc;
    retina_pack_kernel<<<batch, 256, 0, st>>>(a, output_dev);
    return check_launch();
}

}  // extern "C"
