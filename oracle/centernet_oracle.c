/*
 * centernet_oracle.c -- CPU ORACLE of the CenterNet pre-process and decode.  TEST INFRASTRUCTURE ONLY, like trtx_oracle.c:
 * plain C, single thread, built with -ffp-contract=off, independent of the library's code.
 *   pre_process    centernet/sample/test.py:34-41 (float64 canvas, cv.resize INTER_LINEAR on float64, normalisation)
 *   ctdet_decode   centernet/sample/test.py:44-102 with reg, without cat_spec_wh, as the order the library defines
 *   the rows       the driver loop of centernet/sample/test.py:126-132 (`if i[-2] > 0.5: i[:4] *= 4*s`)
 * Pinned to the sample's own functions (or their stored outputs) and to cv2 by tests/test_centernet_cpu.py.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORACLE_API __attribute__((visibility("default")))

/* OpenCV 4.x's INTER_LINEAR geometry for one destination index: fx = (float)((d + 0.5) * scale - 0.5), s = floor, fx -= s;
 * on float64 both axes clamp the tap to [0, n - 1] with a zero fraction. */
static void linear_coord(int d, double scale, int n, int* s_out, float* f_out) {
    float f = (float)((d + 0.5) * scale - 0.5);
    int s = (int)floorf(f);
    f -= (float)s;
    if (s < 0) f = 0, s = 0;
    if (s >= n - 1) f = 0, s = n - 1;
    *s_out = s;
    *f_out = f;
}

/* the sample's canvas: the frame at the top-left of an L x L zero canvas; a w == 1 frame fills its rows (numpy broadcast) */
static double canvas(const uint8_t* img, int w, int h, size_t pitch, int y, int x, int c) {
    if (y >= h || (w != 1 && x >= w)) return 0.0;
    return (double)img[(size_t)y * pitch + 3 * (size_t)(w == 1 ? 0 : x) + c];
}

/* pre_process for one u8 BGR frame: out [3, net, net] float planes B, G, R. */
ORACLE_API void oracle_centernet_preprocess(const uint8_t* img, int w, int h, size_t pitch, int net, float* out) {
    const int L = (w > h ? w : h) > 3 ? (w > h ? w : h) : 3;
    const double scale = 1. / ((double)net / L);
    for (int y = 0; y < net; ++y) {
        int sy;
        float fy;
        linear_coord(y, scale, L, &sy, &fy);
        const int sy1 = sy + 1 < L ? sy + 1 : L - 1;
        const double b0 = (double)(1.f - fy), b1 = (double)fy;
        for (int x = 0; x < net; ++x) {
            int sx;
            float fx;
            linear_coord(x, scale, L, &sx, &fx);
            const int sx1 = sx + 1 < L ? sx + 1 : L - 1;
            const double a0 = (double)(1.f - fx), a1 = (double)fx;
            for (int c = 0; c < 3; ++c) {
                const double h0 = canvas(img, w, h, pitch, sy, sx, c) * a0 + canvas(img, w, h, pitch, sy, sx1, c) * a1;
                const double h1 = canvas(img, w, h, pitch, sy1, sx, c) * a0 + canvas(img, w, h, pitch, sy1, sx1, c) * a1;
                const double v = h0 * b0 + h1 * b1;
                out[((size_t)c * net + y) * net + x] = (float)(((v / 255.) - 0.5) / 0.5);
            }
        }
    }
}

typedef struct {
    float v;
    uint32_t idx;
} cand_t;

/* NaN first, then descending value, ties to the smaller flat index */
static int cand_cmp(const void* pa, const void* pb) {
    const cand_t* a = (const cand_t*)pa;
    const cand_t* b = (const cand_t*)pb;
    const int na = isnan(a->v), nb = isnan(b->v);
    if (na != nb) return na ? -1 : 1;
    if (!na && a->v != b->v) return a->v > b->v ? -1 : 1;
    return a->idx < b->idx ? -1 : (a->idx > b->idx);
}

/* ctdet_decode for one image: heat [C, H, W], wh [2, H, W], reg [2, H, W] -> dets [K, 6] (x1, y1, x2, y2, score, class). */
ORACLE_API void oracle_centernet_decode(const float* heat, const float* wh, const float* reg, int C, int H, int W, int K,
                                        float* dets) {
    const size_t HW = (size_t)H * W, N = (size_t)C * HW;
    float* s = (float*)malloc(N * sizeof(float));
    for (size_t i = 0; i < N; ++i) s[i] = 1.0f / (1.0f + expf(-heat[i]));
    cand_t* cand = (cand_t*)malloc(N * sizeof(cand_t));
    unsigned char* taken = (unsigned char*)calloc(N, 1);
    size_t n = 0;
    for (int c = 0; c < C; ++c)
        for (int y = 0; y < H; ++y)
            for (int x = 0; x < W; ++x) {
                const size_t i = (size_t)c * HW + (size_t)y * W + x;
                /* max_pool2d: the max of the clipped window, NaN as soon as one element is NaN */
                float m = -INFINITY;
                for (int dy = -1; dy <= 1; ++dy)
                    for (int dx = -1; dx <= 1; ++dx) {
                        const int yy = y + dy, xx = x + dx;
                        if (yy < 0 || yy >= H || xx < 0 || xx >= W) continue;
                        const float t = s[(size_t)c * HW + (size_t)yy * W + xx];
                        if (t > m || isnan(t)) m = isnan(m) ? m : t;
                    }
                const float v = s[i] * (float)(m == s[i]);  /* heat * (hmax == heat).float() */
                if (v > 0.f || isnan(v)) {
                    cand[n].v = v;
                    cand[n].idx = (uint32_t)i;
                    taken[i] = 1;
                    ++n;
                }
            }
    qsort(cand, n, sizeof(cand_t), cand_cmp);
    for (size_t i = 0; n < (size_t)K && i < N; ++i)  /* fewer than K positive or NaN cells: zero cells in flat order */
        if (!taken[i]) cand[n].v = 0.f, cand[n].idx = (uint32_t)i, ++n;
    for (int r = 0; r < K; ++r) {
        const uint32_t idx = cand[r].idx;
        const int c = (int)(idx / HW);
        const uint32_t cell = (uint32_t)(idx % HW);
        const float xs = (float)(cell % (uint32_t)W) + reg[cell];
        const float ys = (float)(int)((float)cell / (float)W) + reg[HW + cell];
        const float hw = wh[cell] / 2, hh = wh[HW + cell] / 2;
        float* d = dets + (size_t)r * 6;
        d[0] = xs - hw;
        d[1] = ys - hh;
        d[2] = xs + hw;
        d[3] = ys + hh;
        d[4] = cand[r].v;
        d[5] = (float)c;
    }
    free(taken);
    free(cand);
    free(s);
}

/* The driver loop over one frame's dets [K, 6]: rows [1 + K * 6] = the count of rows with score > thresh, then those rows
 * with x1, y1, x2, y2 times k = (float)(down * (L / (double)net)), L = max(img_h, img_w, 3); zeros past the count. */
ORACLE_API int oracle_centernet_rows(const float* dets, int K, int img_w, int img_h, int down, int net, float thresh,
                                     float* rows) {
    const int L = (img_w > img_h ? img_w : img_h) > 3 ? (img_w > img_h ? img_w : img_h) : 3;
    const float k = (float)(down * ((double)L / net));
    int n = 0;
    memset(rows, 0, sizeof(float) * (1 + (size_t)K * 6));
    for (int r = 0; r < K; ++r) {
        const float* d = dets + (size_t)r * 6;
        if (!(d[4] > thresh)) continue;
        float* o = rows + 1 + (size_t)n * 6;
        for (int e = 0; e < 4; ++e) o[e] = d[e] * k;
        o[4] = d[4];
        o[5] = d[5];
        ++n;
    }
    rows[0] = (float)n;
    return n;
}
