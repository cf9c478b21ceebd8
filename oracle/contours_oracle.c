/*
 * contours_oracle.c -- CPU ORACLE of cv::findContours(img, RETR_EXTERNAL, CHAIN_APPROX_NONE), the outlines the Mask R-CNN
 * driver takes of each pasted canvas (rcnn/rcnn.cpp:551-552).  TEST INFRASTRUCTURE ONLY, like trtx_oracle.c: plain C,
 * single thread.  Pinned to cv2 by tests/test_rcnn_contours_cpu.py; built by oracle/Makefile.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORACLE_API __attribute__((visibility("default")))

/* ------------------------------------------------------------------------------------------
 * cv::findContours(img, RETR_EXTERNAL, CHAIN_APPROX_NONE) of rcnn/rcnn.cpp:551-552, restated: Suzuki-Abe border following
 * as OpenCV implements it.  Pinned to cv2 by tests/test_rcnn_contours_cpu.py.
 * The image is copied into a padded int8 map (1 where nonzero, a zero frame around it).  A raster scan keeps `prev` (the value
 * left of x) and lnbd (the last place where the value changed to a traced-border mark); at prev == 0, p == 1 (an unvisited
 * outer-border start) it follows the border unless the value at lnbd is positive (the start lies inside a hole of a traced
 * component).  Following marks each visited pixel -2 when the search passed its right neighbour as 0, else 2 if it was 1;
 * holes are never followed.  Contours are returned in descending raster order of their starts, as cv2 does.
 * img: h rows of `pitch` bytes; lengths (capacity max_contours), points (x, y pairs, capacity max_points) get the first
 * entries in that order; *n_contours / *n_points get the totals.  Returns 0, or -1 when out of memory.
 * ------------------------------------------------------------------------------------------ */
static const int kCodeDx[8] = {1, 1, 0, -1, -1, -1, 0, 1};
static const int kCodeDy[8] = {0, -1, -1, -1, 0, 1, 1, 1};

/* Border following from the outer start i0 (OpenCV's icvFetchContour); returns the number of points, and writes them
 * (frame coordinates) to pts when it is not NULL. */
static long trace_outer(int8_t* m, long stride, long i0, int x, int y, int* pts) {
    long deltas[16];
    for (int k = 0; k < 8; ++k) deltas[k] = deltas[k + 8] = kCodeDx[k] + (long)kCodeDy[k] * stride;
    long n = 0;
    int s = 4, s_end = 4;
    long i1;
    do {
        s = (s - 1) & 7;
        i1 = i0 + deltas[s];
    } while (m[i1] == 0 && s != s_end);
    if (s == s_end) { /* a lone pixel */
        m[i0] = -2;
        if (pts) pts[0] = x, pts[1] = y;
        return 1;
    }
    long i3 = i0, i4;
    for (;;) {
        s_end = s;
        for (;;) {
            i4 = i3 + deltas[++s];
            if (m[i4] != 0) break;
        }
        s &= 7;
        if ((unsigned)(s - 1) < (unsigned)s_end) m[i3] = -2;
        else if (m[i3] == 1) m[i3] = 2;
        if (pts) pts[2 * n] = x, pts[2 * n + 1] = y;
        ++n;
        x += kCodeDx[s];
        y += kCodeDy[s];
        if (i4 == i0 && i3 == i1) break;
        i3 = i4;
        s = (s + 4) & 7;
    }
    return n;
}

ORACLE_API int oracle_find_contours_external(const uint8_t* img, int w, int h, int pitch, int max_contours, int max_points,
                                             int* n_contours, long* n_points, int* lengths, int* points) {
    const long stride = (long)w + 2;
    int8_t* m = (int8_t*)calloc((size_t)stride * (h + 2), 1);
    long cap = 16, n = 0;
    long* starts = (long*)malloc((size_t)cap * 2 * sizeof(long)); /* (start index, length) in trace order */
    if (!m || !starts) {
        free(m);
        free(starts);
        return -1;
    }
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) m[(y + 1) * stride + x + 1] = img[(size_t)y * pitch + x] != 0;
    for (int y = 1; y <= h; ++y) {
        int8_t* row = m + y * stride;
        int prev = 0;
        long lnbd = 0;
        for (int x = 1; x <= w; ++x) {
            const int p = row[x];
            if (p == prev) continue;
            if (prev == 0 && p == 1 && row[lnbd] <= 0) {
                if (n == cap) {
                    long* grown = (long*)realloc(starts, (size_t)cap * 4 * sizeof(long));
                    if (!grown) {
                        free(m);
                        free(starts);
                        return -1;
                    }
                    starts = grown;
                    cap *= 2;
                }
                starts[2 * n] = y * stride + x;
                starts[2 * n + 1] = trace_outer(m, stride, y * stride + x, x - 1, y - 1, NULL);
                ++n;
                prev = row[x]; /* the scan resumes after the start with its new mark; lnbd stays */
                continue;
            }
            prev = p;
            if (p & -2) lnbd = x;
        }
    }
    /* second pass: write in descending start order, on a fresh copy (the trace reads only zero / nonzero) */
    long total = 0, off = 0;
    for (long i = 0; i < n; ++i) total += starts[2 * i + 1];
    for (long i = n - 1; i >= 0; --i) {
        const long j = n - 1 - i, len = starts[2 * i + 1];
        if (j < max_contours) lengths[j] = (int)len;
        if (off < max_points) {
            const long s = starts[2 * i];
            if (off + len <= max_points) {
                trace_outer(m, stride, s, (int)(s % stride) - 1, (int)(s / stride) - 1, points + 2 * off);
            } else {
                int* tmp = (int*)malloc((size_t)len * 2 * sizeof(int));
                if (!tmp) {
                    free(m);
                    free(starts);
                    return -1;
                }
                trace_outer(m, stride, s, (int)(s % stride) - 1, (int)(s / stride) - 1, tmp);
                memcpy(points + 2 * off, tmp, (size_t)(max_points - off) * 2 * sizeof(int));
                free(tmp);
            }
        }
        off += len;
    }
    *n_contours = (int)n;
    *n_points = total;
    free(m);
    free(starts);
    return 0;
}
