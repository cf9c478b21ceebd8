/*
 * trtx_oracle.c -- CPU ORACLE for the tensorrtx detection hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is product code: only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * load it, and there only as the checker / the CPU comparator.
 *
 * PARITY STATUS: the reference (wang-xinyu/tensorrtx) ships NO tests, golden vectors or fixtures
 * for this path (SURVEY.md section 4 / 8c), so there is nothing of its own to check against.
 * The restatements are PINNED against the reference itself, compiled here from /root/reference:
 *   (a) CPU NMS functions: bit-identical rows, in identical order, to the reference's own
 *       nms()/iou()/cmp() -- oracle/_ref/libref_{yolov8,yolov5,retina}_host.so, built by
 *       oracle/Makefile from the reference's postprocess.cpp / common.hpp with header shims;
 *       tests/test_oracle_vs_ref_cpu.py (runs without a GPU).
 *   (b) GPU plugin kernels (decode, cuda_decode/cuda_nms, warpaffine, rcnn functions): the
 *       reference's .cu files compiled against tests/mock_trt/NvInfer.h into oracle/_ref/libref_*.so
 *       and run next to our kernels on the GPU box; tests/test_vs_reference_gpu.py.  The decode
 *       restatements below agree with those kernels to <= 2 ulp (glibc vs CUDA expf).
 *   (c) independent cross-checks: torchvision nms/batched_nms, cv2.invertAffineTransform, a numpy
 *       re-derivation of the v8 decode (tests/test_oracle_cpu.py).
 *
 * Every function cites the reference file:line (relative to /root/reference) it
 * restates.  Plain C, single thread, no FMA contraction (build with
 * -ffp-contract=off) so that the arithmetic is the straightforward IEEE fp32
 * sequence written in the reference source.
 *
 * Deterministic ordering: where the reference's order depends on atomicAdd arrival
 * (yololayer.cu:206) the oracle emits candidates in ascending (level, cell, anchor_k)
 * order and also returns that flat anchor id, so tests can compare as sets.
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORACLE_API __attribute__((visibility("default")))

/* yolov8/plugin/yololayer.cu:174-176 (Logist) and :23-25 (sigmoid) */
static inline float logist(float x) { return 1.0f / (1.0f + expf(-x)); }

/* ------------------------------------------------------------------------------------------
 * YOLOv8/11/12 anchor-free decode.  Restates CalDetection, yolov8/plugin/yololayer.cu:178-280,
 * and the launch loop of forwardGpu, :282-316.
 *
 * inputs[l]  : level l tensor, [B, info_len, gh_l*gw_l] fp32 channel-major (:187-190)
 * out        : [B, 1 + max_out*det_floats] fp32; out[b*out_elem] = candidate count as float
 *              (UNCLAMPED, like the reference's atomicAdd counter, :206), rows beyond
 *              max_out are dropped (:207-208).  Rows are zero-initialised here (the
 *              reference leaves untouched fields uninitialised).
 * anchor_idx : [B, max_out] int32 flat anchor id of each emitted row (level offset + cell),
 *              or NULL.
 * det_floats : sizeof(Detection)/4 = 90 for yolov8/include/types.h:4-12 (kNumberOfPoints=17).
 * gate       : 0.1 literal of :203.
 * ------------------------------------------------------------------------------------------ */
ORACLE_API void oracle_yolov8_decode(const float* const* inputs, int batch, int num_levels, const int* grid_h,
                                     const int* grid_w, const int* strides, int classes, int nk, float kpt_thresh,
                                     int is_seg, int is_pose, int is_obb, int max_out, int det_floats, float gate,
                                     float* out, int32_t* anchor_idx) {
    const int out_elem = 1 + max_out * det_floats; /* :283 */
    const int info_len = 4 + classes + (is_seg ? 32 : 0) + (is_pose ? nk * 3 : 0) + (is_obb ? 1 : 0); /* :186 */
    memset(out, 0, sizeof(float) * (size_t)batch * out_elem);
    int level_off = 0;
    for (int l = 0; l < num_levels; ++l) { /* :300 one launch per stride */
        const int gh = grid_h[l], gw = grid_w[l], stride = strides[l];
        const int total_grid = gh * gw;
        for (int idx = 0; idx < batch * total_grid; ++idx) { /* thread idx, :181 */
            const int b = idx / total_grid;
            const int e = idx % total_grid;
            const float* cur = inputs[l] + (size_t)b * total_grid * info_len; /* :189 */
            float* o = out + (size_t)b * out_elem;
            int class_id = 0;
            float max_cls_prob = 0.0f;
            for (int i = 4; i < 4 + classes; ++i) { /* :195-201 */
                float p = logist(cur[e + (size_t)i * total_grid]);
                if (p > max_cls_prob) {
                    max_cls_prob = p;
                    class_id = i - 4;
                }
            }
            if (max_cls_prob < gate) continue; /* :203 (0.1 double literal == 0.1f boundary) */
            int count = (int)o[0];
            o[0] += 1.0f; /* atomicAdd(float,1) :206 */
            if (count >= max_out) continue; /* :207 */
            float* det = o + 1 + (size_t)count * det_floats;
            if (anchor_idx) anchor_idx[(size_t)b * max_out + count] = level_off + e;
            const int row = e / gw, col = e % gw; /* :212-213 */
            const float d0 = cur[e + 0 * (size_t)total_grid], d1 = cur[e + 1 * (size_t)total_grid];
            const float d2 = cur[e + 2 * (size_t)total_grid], d3 = cur[e + 3 * (size_t)total_grid];
            det[4] = max_cls_prob;
            det[5] = (float)class_id;
            det[0] = (col + 0.5f - d0) * stride; /* :217-220 */
            det[1] = (row + 0.5f - d1) * stride;
            det[2] = (col + 0.5f + d2) * stride;
            det[3] = (row + 0.5f + d3) * stride;
            if (is_seg) { /* :222-227 */
                for (int k = 0; k < 32; ++k)
                    det[6 + k] =
                            cur[e + (size_t)(4 + classes + (is_pose ? nk * 3 : 0) + (is_obb ? 1 : 0) + k) * total_grid];
            }
            if (is_pose) { /* :229-253 ; keypoints live at Detection offset 6+32 */
                float* kp = det + 6 + 32;
                for (int k = 0; k < nk; ++k) {
                    const size_t base = (size_t)(4 + classes + (is_seg ? 32 : 0) + (is_obb ? 1 : 0) + k * 3);
                    float kc = logist(cur[e + (base + 2) * total_grid]);
                    /* "* 2.0" is a double literal: the expression is evaluated in double (:238-239) */
                    float kx = (float)(((double)cur[e + base * total_grid] * 2.0 + col) * stride);
                    float ky = (float)(((double)cur[e + (base + 1) * total_grid] * 2.0 + row) * stride);
                    int inside = kx >= det[0] && kx <= det[2] && ky >= det[1] && ky <= det[3];
                    if (kc < kpt_thresh || !inside) {
                        kp[k * 3] = -1;
                        kp[k * 3 + 1] = -1;
                        kp[k * 3 + 2] = -1;
                    } else {
                        kp[k * 3] = kx;
                        kp[k * 3 + 1] = ky;
                        kp[k * 3 + 2] = kc;
                    }
                }
            }
            if (is_obb) { /* :255-279, double-precision trig */
                const double pi = M_PI;
                float a_in = cur[e + (size_t)(4 + classes + (is_seg ? 32 : 0) + (is_pose ? nk * 3 : 0)) * total_grid];
                double angle = (double)(logist(a_in) - 0.25f) * pi;
                double cos1 = cos(angle), sin1 = sin(angle);
                float xf = (d2 - d0) / 2;
                float yf = (d3 - d1) / 2;
                double x = xf * cos1 - yf * sin1;
                double y = xf * sin1 + yf * cos1;
                float cx = (float)(((double)(col + 0.5f) + x) * stride);
                float cy = (float)(((double)(row + 0.5f) + y) * stride);
                float w1 = (d0 + d2) * stride;
                float h1 = (d1 + d3) * stride;
                det[0] = cx;
                det[1] = cy;
                det[2] = w1;
                det[3] = h1;
                det[det_floats - 1] = (float)angle; /* Detection::angle is the last float */
            }
        }
        level_off += total_grid;
    }
}

/* ------------------------------------------------------------------------------------------
 * YOLOv5 anchor-based decode.  Restates CalDetection, yolov5/plugin/yololayer.cu:161-210.
 * inputs[l] : [B, 3*(5+classes(+32)), gh*gw] fp32 (:171-172); anchors[l*6 + 2k (+1)] (:19 types.h).
 * out rows  : Detection of yolov5/src/types.h:11-16 = cx,cy,w,h,conf,cls,mask[32] -> det_floats 38.
 * Flat anchor id = level_off + cell*3 + k.
 * NOTE: the reference `return`s (not `continue`s) on overflow (:194) -- same effect per thread.
 * ------------------------------------------------------------------------------------------ */
ORACLE_API void oracle_yolov5_decode(const float* const* inputs, int batch, int num_levels, const int* grid_h,
                                     const int* grid_w, const float* anchors, int classes, int net_w, int net_h,
                                     int is_seg, int max_out, int det_floats, float ignore_thresh, float* out,
                                     int32_t* anchor_idx) {
    const int out_elem = 1 + max_out * det_floats;
    int info_len_i = 5 + classes;
    if (is_seg) info_len_i += 32;
    memset(out, 0, sizeof(float) * (size_t)batch * out_elem);
    int level_off = 0;
    for (int l = 0; l < num_levels; ++l) {
        const int yw = grid_w[l], yh = grid_h[l];
        const int total_grid = yw * yh;
        const float* anc = anchors + l * 6;
        for (int t = 0; t < batch * total_grid; ++t) {
            const int bn = t / total_grid;
            const int idx = t - total_grid * bn;
            const float* cur = inputs[l] + (size_t)bn * ((size_t)info_len_i * total_grid * 3);
            float* o = out + (size_t)bn * out_elem;
            for (int k = 0; k < 3; ++k) {
                const float* ck = cur + (size_t)k * info_len_i * total_grid;
                float box_prob = logist(ck[idx + 4 * (size_t)total_grid]); /* :176 */
                if (box_prob < ignore_thresh) continue;                     /* :177 */
                int class_id = 0;
                float max_cls_prob = 0.0f;
                for (int i = 5; i < 5 + classes; ++i) { /* :180-186 */
                    float p = logist(ck[idx + (size_t)i * total_grid]);
                    if (p > max_cls_prob) {
                        max_cls_prob = p;
                        class_id = i - 5;
                    }
                }
                int count = (int)o[0];
                o[0] += 1.0f;                /* :188 */
                if (count >= max_out) break; /* :189 `return` */
                float* det = o + 1 + (size_t)count * det_floats;
                if (anchor_idx) anchor_idx[(size_t)bn * max_out + count] = level_off + idx * 3 + k;
                const int row = idx / yw, col = idx % yw;
                /* :196-202, left-to-right evaluation: ((col-0.5f + 2σ) * netw) / yw */
                det[0] = (col - 0.5f + 2.0f * logist(ck[idx + 0 * (size_t)total_grid])) * net_w / yw;
                det[1] = (row - 0.5f + 2.0f * logist(ck[idx + 1 * (size_t)total_grid])) * net_h / yh;
                float w = 2.0f * logist(ck[idx + 2 * (size_t)total_grid]);
                det[2] = w * w * anc[2 * k];
                float h = 2.0f * logist(ck[idx + 3 * (size_t)total_grid]);
                det[3] = h * h * anc[2 * k + 1];
                det[4] = box_prob * max_cls_prob; /* :203 */
                det[5] = (float)class_id;
                for (int i = 0; is_seg && i < 32; ++i) /* :206-208 */
                    det[6 + i] = ck[idx + (size_t)(i + 5 + classes) * total_grid];
            }
        }
        level_off += total_grid * 3;
    }
}

/* ------------------------------------------------------------------------------------------
 * RetinaFace decode.  Restates CalDetection, retinaface/decode.cu:110-165 and forwardGpu
 * :167-191, with INPUT_H/INPUT_W (decode.h:16-17) made runtime.  The reference's literals
 * 0.5, 0.1, 0.2, 0.02 are doubles, so those expressions are evaluated in double.
 * inputs[l] : [B, 8+4+20, h*w] fp32 = [bbox 2x4 | cls 2x2 | lmk 2x10] (:121-123)
 * out       : [B, 1 + total_priors*15]; no capacity check in the reference (:133-136).
 * Flat anchor id = level_off + cell*2 + k.
 * ------------------------------------------------------------------------------------------ */
ORACLE_API void oracle_retina_decode(const float* const* inputs, int batch, int in_h, int in_w, double gate, float* out,
                                     int32_t* anchor_idx) {
    int total_priors = 0;
    for (int s = 8; s <= 32; s *= 2) total_priors += (in_h / s) * (in_w / s) * 2;
    const int out_elem = 1 + total_priors * 15; /* :175-178 */
    memset(out, 0, sizeof(float) * (size_t)batch * out_elem);
    int step = 8, anchor = 16, level_off = 0;
    for (int l = 0; l < 3; ++l) {
        const int h = in_h / step, w = in_w / step;
        const int total_grid = h * w;
        for (int t = 0; t < batch * total_grid; ++t) {
            const int bn = t / total_grid;
            const int idx = t - bn * total_grid;
            const int y = idx / w, x = idx % w;
            const float* cur = inputs[l] + (size_t)bn * (4 + 2 + 10) * 2 * total_grid;
            const float* bbox_reg = cur;
            const float* cls_reg = cur + 2 * 4 * (size_t)total_grid;
            const float* lmk_reg = cur + 2 * 4 * (size_t)total_grid + 2 * 2 * (size_t)total_grid;
            float* o = out + (size_t)bn * out_elem;
            for (int k = 0; k < 2; ++k) {
                float conf1 = cls_reg[idx + k * total_grid * 2];
                float conf2 = cls_reg[idx + k * total_grid * 2 + total_grid];
                conf2 = expf(conf2) / (expf(conf1) + expf(conf2)); /* :130 */
                if ((double)conf2 <= gate) continue;               /* :131, 0.02 is a double literal */
                int count = (int)o[0];
                o[0] += 1.0f;
                float* det = o + 1 + (size_t)count * 15;
                if (anchor_idx) anchor_idx[(size_t)bn * total_priors + count] = level_off + idx * 2 + k;
                float prior[4]; /* :138-142 */
                prior[0] = (float)(((double)(float)x + 0.5) / w);
                prior[1] = (float)(((double)(float)y + 0.5) / h);
                prior[2] = (float)anchor * (k + 1) / in_w;
                prior[3] = (float)anchor * (k + 1) / in_h;
                /* :145-156 */
                det[0] = (float)(prior[0] + (double)bbox_reg[idx + k * total_grid * 4] * 0.1 * prior[2]);
                det[1] = (float)(prior[1] + (double)bbox_reg[idx + k * total_grid * 4 + total_grid] * 0.1 * prior[3]);
                det[2] = prior[2] * expf((float)((double)bbox_reg[idx + k * total_grid * 4 + total_grid * 2] * 0.2));
                det[3] = prior[3] * expf((float)((double)bbox_reg[idx + k * total_grid * 4 + total_grid * 3] * 0.2));
                det[0] -= det[2] / 2;
                det[1] -= det[3] / 2;
                det[2] += det[0];
                det[3] += det[1];
                det[0] *= in_w;
                det[1] *= in_h;
                det[2] *= in_w;
                det[3] *= in_h;
                det[4] = conf2;
                for (int i = 0; i < 10; i += 2) { /* :158-163 */
                    det[5 + i] =
                            (float)(prior[0] + (double)lmk_reg[idx + k * total_grid * 10 + total_grid * i] * 0.1 * prior[2]);
                    det[5 + i + 1] = (float)(prior[1] + (double)lmk_reg[idx + k * total_grid * 10 + total_grid * (i + 1)] *
                                                                0.1 * prior[3]);
                    det[5 + i] *= in_w;
                    det[5 + i + 1] *= in_h;
                }
            }
        }
        level_off += total_grid * 2;
        step *= 2;
        anchor *= 4;
    }
}

/* ------------------------------------------------------------------------------------------
 * YOLOv3 / v3-spp / v4 anchor-based decode (SURVEY 8f rank 4).  Restates CalDetection,
 * yolov3-spp/yololayer.cu:148-191 (yolov3, yolov4 carry the same kernel).
 * inputs[l] : [B, 3*(5+classes), gh*gw] fp32 (:159-160), levels in the caller's order (the plugin's own order is
 *             stride 32, 16, 8, yololayer.h:27-44); anchors[l*6 + 2k (+1)]; strides[l].
 * out rows  : Detection of yololayer.h:47-53 = x,y,w,h, det_confidence, class_id, class_confidence -> 7 floats.
 * Class loop first (all classes, sigmoid, strict `>` from 0), THEN both gates (:171), exp() for w/h (:185-186).
 * Flat anchor id = level_off + cell*3 + k.
 * ------------------------------------------------------------------------------------------ */
ORACLE_API void oracle_yolov3_decode(const float* const* inputs, int batch, int num_levels, const int* grid_h,
                                     const int* grid_w, const int* strides, const float* anchors, int classes, int max_out,
                                     float ignore_thresh, float* out, int32_t* anchor_idx) {
    const int det_floats = 7;
    const int out_elem = 1 + max_out * det_floats;
    const int info_len_i = 5 + classes;
    memset(out, 0, sizeof(float) * (size_t)batch * out_elem);
    int level_off = 0;
    for (int l = 0; l < num_levels; ++l) {
        const int yw = grid_w[l], yh = grid_h[l];
        const int total_grid = yw * yh;
        const float* anc = anchors + l * 6;
        for (int t = 0; t < batch * total_grid; ++t) {
            const int bn = t / total_grid;
            const int idx = t - total_grid * bn;
            const float* cur = inputs[l] + (size_t)bn * ((size_t)info_len_i * total_grid * 3);
            float* o = out + (size_t)bn * out_elem;
            for (int k = 0; k < 3; ++k) {
                const float* ck = cur + (size_t)k * info_len_i * total_grid;
                int class_id = 0;
                float max_cls_prob = 0.0f;
                for (int i = 5; i < info_len_i; ++i) { /* :162-168 */
                    float p = logist(ck[idx + (size_t)i * total_grid]);
                    if (p > max_cls_prob) {
                        max_cls_prob = p;
                        class_id = i - 5;
                    }
                }
                float box_prob = logist(ck[idx + 4 * (size_t)total_grid]);             /* :170 */
                if (max_cls_prob < ignore_thresh || box_prob < ignore_thresh) continue; /* :171 */
                int count = (int)o[0];
                o[0] += 1.0f;                /* :174 */
                if (count >= max_out) break; /* :175 `return` */
                float* det = o + 1 + (size_t)count * det_floats;
                if (anchor_idx) anchor_idx[(size_t)bn * max_out + count] = level_off + idx * 3 + k;
                const int row = idx / yw, col = idx % yw;
                det[0] = (col + logist(ck[idx + 0 * (size_t)total_grid])) * strides[l]; /* :183-186 */
                det[1] = (row + logist(ck[idx + 1 * (size_t)total_grid])) * strides[l];
                det[2] = expf(ck[idx + 2 * (size_t)total_grid]) * anc[2 * k];
                det[3] = expf(ck[idx + 3 * (size_t)total_grid]) * anc[2 * k + 1];
                det[4] = box_prob;
                det[5] = (float)class_id;
                det[6] = max_cls_prob;
            }
        }
        level_off += total_grid * 3;
    }
}

/* ------------------------------------------------------------------------------------------
 * yolo26 NMS-free gather (SURVEY 8f rank 4).  Restates gatherKernel, yolo26/plugin/yololayer.cu:178-245.
 * input : [B, anchor_count, 4 + classes (+1 angle when is_obb)] fp32, ROW-major per anchor (AoS): xmin,ymin,xmax,ymax,
 *         class confidences (already probabilities), angle.  The reference handles batch index 0 only (:185 "TODO"); the
 *         restatement applies the same per-anchor code to every image.
 * out   : [B, 1 + max_out*det_floats] (Detection of yolo26/include/types.h: 90 floats, the angle is the last one);
 *         argmax: `conf > score` from score = 0, class_id = -1 (:201-209); gate `score < thresh` -> skip (:211).
 * ------------------------------------------------------------------------------------------ */
ORACLE_API void oracle_yolo26_gather(const float* input, int batch, int anchor_count, int classes, int is_obb, int max_out,
                                     int det_floats, float conf_thresh, float* out, int32_t* anchor_idx) {
    const int out_elem = 1 + max_out * det_floats;
    const int asz = (is_obb ? 5 : 4) + classes;
    memset(out, 0, sizeof(float) * (size_t)batch * out_elem);
    for (int b = 0; b < batch; ++b) {
        float* o = out + (size_t)b * out_elem;
        for (int idx = 0; idx < anchor_count; ++idx) {
            const float* a = input + ((size_t)b * anchor_count + idx) * asz;
            float score = 0.0f;
            int class_id = -1;
            for (int c = 0; c < classes; ++c) {
                float conf = a[4 + c];
                if (conf > score) {
                    score = conf;
                    class_id = c;
                }
            }
            if (score < conf_thresh) continue;
            int count = (int)o[0];
            o[0] += 1.0f;
            if (count >= max_out) continue;
            float* det = o + 1 + (size_t)count * det_floats;
            if (anchor_idx) anchor_idx[(size_t)b * max_out + count] = idx;
            det[0] = a[0];
            det[1] = a[1];
            det[2] = a[2];
            det[3] = a[3];
            det[4] = score;
            det[5] = (float)class_id;
            if (is_obb) det[det_floats - 1] = a[4 + classes];
        }
    }
}

/* ------------------------------------------------------------------------------------------
 * RetinaFace anti-cov decode (SURVEY 8f rank 4).  Restates CalDetection, retinafaceAntiCov/decode.cu:110-155 and
 * forwardGpu :157-172, with INPUT_H/INPUT_W (decode.h:20-21) made runtime and the batch index added (the reference is
 * batch 1 only: no image offset anywhere).
 * inputs[l] : [B, 38, h*w] fp32 = [cls 4 (softmaxed in the network; face prob of anchor k at channel 2+k) | bbox 2x4 |
 *             lmk 2x10 | type 6 (mask prob of anchor k at channel 36+k)] (:120-123)
 * out rows  : x1,y1,x2,y2, class_confidence, lmk[10], mask_confidence -> 16 floats (decode.h:13-18)
 * Literals 7.5, 0.2, 0.5 are doubles; `anchor * 2 / (k + 1)` is INTEGER arithmetic (:137).
 * ------------------------------------------------------------------------------------------ */
ORACLE_API void oracle_anticov_decode(const float* const* inputs, int batch, int in_h, int in_w, float* out,
                                      int32_t* anchor_idx) {
    int total_priors = 0;
    for (int s = 8; s <= 32; s *= 2) total_priors += (in_h / s) * (in_w / s) * 2;
    const int out_elem = 1 + total_priors * 16;
    memset(out, 0, sizeof(float) * (size_t)batch * out_elem);
    int step = 8, anchor = 16, level_off = 0;
    for (int l = 0; l < 3; ++l) {
        const int h = in_h / step, w = in_w / step;
        const int num_elem = h * w;
        for (int bn = 0; bn < batch; ++bn) {
            const float* input = inputs[l] + (size_t)bn * 38 * num_elem;
            const float* cls_reg = input + 2 * (size_t)num_elem;
            const float* bbox_reg = input + 4 * (size_t)num_elem;
            const float* lmk_reg = input + 12 * (size_t)num_elem;
            const float* mask_reg = input + 36 * (size_t)num_elem;
            float* o = out + (size_t)bn * out_elem;
            for (int idx = 0; idx < num_elem; ++idx) {
                const int y = idx / w, x = idx % w;
                for (int k = 0; k < 2; ++k) {
                    float conf = cls_reg[idx + k * num_elem];
                    if ((double)conf < 0.5) continue; /* :127 */
                    int count = (int)o[0];
                    o[0] += 1.0f;
                    float* det = o + 1 + (size_t)count * 16;
                    if (anchor_idx) anchor_idx[(size_t)bn * total_priors + count] = level_off + idx * 2 + k;
                    float prior[4]; /* :134-138 */
                    prior[0] = (float)(7.5 + (double)(float)(x * step));
                    prior[1] = (float)(7.5 + (double)(float)(y * step));
                    prior[2] = (float)(anchor * 2 / (k + 1));
                    prior[3] = prior[2];
                    det[0] = prior[0] + bbox_reg[idx + k * num_elem * 4] * prior[2]; /* :141-148 */
                    det[1] = prior[1] + bbox_reg[idx + k * num_elem * 4 + num_elem] * prior[3];
                    det[2] = prior[2] * expf(bbox_reg[idx + k * num_elem * 4 + num_elem * 2]);
                    det[3] = prior[3] * expf(bbox_reg[idx + k * num_elem * 4 + num_elem * 3]);
                    det[0] -= (det[2] - 1) / 2;
                    det[1] -= (det[3] - 1) / 2;
                    det[2] += det[0];
                    det[3] += det[1];
                    det[4] = conf;
                    for (int i = 0; i < 10; i += 2) { /* :150-153: float * 0.2 is a double product */
                        det[5 + i] = (float)(prior[0] + (double)lmk_reg[idx + k * num_elem * 10 + num_elem * i] * 0.2 * prior[2]);
                        det[5 + i + 1] =
                                (float)(prior[1] + (double)lmk_reg[idx + k * num_elem * 10 + num_elem * (i + 1)] * 0.2 * prior[3]);
                    }
                    det[15] = mask_reg[idx + k * num_elem];
                }
            }
        }
        level_off += num_elem * 2;
        step *= 2;
        anchor *= 4;
    }
}

/* ------------------------------------------------------------------------------------------
 * CPU greedy NMS.  Restates
 *   variant 0 (v8) : yolov8/src/postprocess.cpp:71-121  iou ltrb, cmp conf desc then bbox[0] asc,
 *                    filter `conf <= thr || isnan(conf)`
 *   variant 1 (v5) : yolov5/src/postprocess.cpp:30-73   iou cxcywh, cmp conf desc,
 *                    loop bound `i < output[0] && i < kMaxNumOutputBbox`
 *   variant 2 (retinaface): retinaface/common.hpp:91-130, single class, pre-filter conf<=0.1
 *                    (conf_thresh passed in), iou with +1e-6f in the denominator.
 * std::map<float,...> iterates classes ascending; std::sort is not stable, so full ties are
 * unspecified in the reference -- the oracle breaks them by input row order (a stable sort).
 *
 * plugin_out : one image, [1 + max_rows*det_floats]
 * res        : out rows, [<=max_rows, det_floats], in the reference's `res` order
 * res_src    : out, source row index (into plugin_out rows) of each kept row, or NULL
 * conf_thresh is a double: v8/v5 compare against the float constant (cast), retinaface against
 * the double literal 0.1.
 * returns number of kept rows.
 * ------------------------------------------------------------------------------------------ */
/* The four max / min of each IoU take their operands in the reference's order: std::max(a, b) is `a < b ? b : a` and
 * std::min(a, b) is `b < a ? b : a`, so a NaN in the later row `r` is ignored and one in the kept row `l` propagates. */
#define STD_MAX(a, b) ((a) < (b) ? (b) : (a))
#define STD_MIN(a, b) ((b) < (a) ? (b) : (a))
static float iou_ltrb(const float* l, const float* r) { /* yolov8/src/postprocess.cpp:71-85 */
    float ib0 = STD_MAX(l[0], r[0]);
    float ib1 = STD_MIN(l[2], r[2]);
    float ib2 = STD_MAX(l[1], r[1]);
    float ib3 = STD_MIN(l[3], r[3]);
    if (ib2 > ib3 || ib0 > ib1) return 0.0f;
    float inter = (ib1 - ib0) * (ib3 - ib2);
    float uni = (l[2] - l[0]) * (l[3] - l[1]) + (r[2] - r[0]) * (r[3] - r[1]) - inter;
    return inter / uni;
}
static float iou_cxcywh(const float* l, const float* r) { /* yolov5/src/postprocess.cpp:30-43 */
    float a0 = l[0] - l[2] / 2.f, b0 = r[0] - r[2] / 2.f;
    float a1 = l[0] + l[2] / 2.f, b1 = r[0] + r[2] / 2.f;
    float a2 = l[1] - l[3] / 2.f, b2 = r[1] - r[3] / 2.f;
    float a3 = l[1] + l[3] / 2.f, b3 = r[1] + r[3] / 2.f;
    float ib0 = STD_MAX(a0, b0);
    float ib1 = STD_MIN(a1, b1);
    float ib2 = STD_MAX(a2, b2);
    float ib3 = STD_MIN(a3, b3);
    if (ib2 > ib3 || ib0 > ib1) return 0.0f;
    float inter = (ib1 - ib0) * (ib3 - ib2);
    return inter / (l[2] * l[3] + r[2] * r[3] - inter);
}
static float iou_retina(const float* l, const float* r) { /* retinaface/common.hpp:91-104 */
    float ib0 = STD_MAX(l[0], r[0]);
    float ib1 = STD_MIN(l[2], r[2]);
    float ib2 = STD_MAX(l[1], r[1]);
    float ib3 = STD_MIN(l[3], r[3]);
    if (ib2 > ib3 || ib0 > ib1) return 0.0f;
    float inter = (ib1 - ib0) * (ib3 - ib2);
    return inter / ((l[2] - l[0]) * (l[3] - l[1]) + (r[2] - r[0]) * (r[3] - r[1]) - inter + 0.000001f);
}

/* yolov8-obb: convariance_matrix / probiou, yolov8/src/postprocess.cpp:303-355, with the C++ promotions spelled out:
 * `w * w / 12.0` divides in double; std::pow(float, int) is double; std::cos/sin/exp/sqrt(float) are the float
 * overloads; std::log and the last std::sqrt see double arguments.  d = Detection row, angle = d[89] (types.h:4-12). */
static void cov_host(const float* d, int angle_idx, float* a, float* b, float* c) {
    float w = d[2], h = d[3];
    float A = (float)((double)(w * w) / 12.0), B = (float)((double)(h * h) / 12.0);
    float r = d[angle_idx];
    float cos_r = cosf(r), sin_r = sinf(r);
    float cos_r2 = cos_r * cos_r, sin_r2 = sin_r * sin_r;
    *a = A * cos_r2 + B * sin_r2;
    *b = A * sin_r2 + B * cos_r2;
    *c = (A - B) * cos_r * sin_r;
}
static float probiou_host(const float* r1, const float* r2, int angle_idx) {
    const float eps = 1e-7;
    float a1, b1, c1, a2, b2, c2;
    cov_host(r1, angle_idx, &a1, &b1, &c1);
    cov_host(r2, angle_idx, &a2, &b2, &c2);
    float x1 = r1[0], y1 = r1[1], x2 = r2[0], y2 = r2[1];
    double py = pow((double)(y1 - y2), 2), px = pow((double)(x1 - x2), 2), pc = pow((double)(c1 + c2), 2);
    float t1 = (float)(((double)(a1 + a2) * py + (double)(b1 + b2) * px) / ((double)((a1 + a2) * (b1 + b2)) - pc + (double)eps));
    float t2 = (float)((double)((c1 + c2) * (x2 - x1) * (y1 - y2)) / ((double)((a1 + a2) * (b1 + b2)) - pc + (double)eps));
    float m1 = a1 * b1 - c1 * c1, m2 = a2 * b2 - c2 * c2;
    float den3 = 4 * sqrtf(m1 > 0.0f ? m1 : 0.0f) * sqrtf(m2 > 0.0f ? m2 : 0.0f) + eps; /* std::max(x, 0.0f) */
    float t3 = (float)log(((double)((a1 + a2) * (b1 + b2)) - pc) / (double)den3 + (double)eps);
    float bd = 0.25f * t1 + 0.5f * t2 + 0.5f * t3;
    bd = bd < 100.0f ? bd : 100.0f; /* std::min(bd, 100.0f) */
    bd = bd > eps ? bd : eps;       /* std::max(.., eps) */
    float hd = (float)sqrt(1.0 - (double)expf(-bd) + (double)eps);
    return 1 - hd;
}

typedef struct {
    float cls, conf, x0;
    int src;
} nms_key;
static int g_variant; /* comparator context (single-threaded oracle) */
static int nms_cmp(const void* pa, const void* pb) {
    const nms_key* a = (const nms_key*)pa;
    const nms_key* b = (const nms_key*)pb;
    if (a->cls != b->cls) return a->cls < b->cls ? -1 : 1;    /* std::map key order */
    if (a->conf != b->conf) return a->conf > b->conf ? -1 : 1; /* cmp: conf desc */
    if ((g_variant == 0 || g_variant == 3) && a->x0 != b->x0) return a->x0 < b->x0 ? -1 : 1; /* v8 :87-92 */
    return a->src < b->src ? -1 : (a->src > b->src ? 1 : 0);
}

ORACLE_API int oracle_nms(int variant, const float* plugin_out, int max_rows, int det_floats, double conf_thresh,
                          float nms_thresh, float* res, int32_t* res_src) {
    int n_in = (int)plugin_out[0]; /* `i < output[0]` */
    /* v5 clamps to kMaxNumOutputBbox (:51); v8/retina do not (and would overrun); the oracle
     * clamps always -- the buffer has no rows beyond max_rows. */
    if (n_in > max_rows) n_in = max_rows;
    if (n_in < 0) n_in = 0;
    nms_key* keys = (nms_key*)malloc(sizeof(nms_key) * (size_t)(n_in > 0 ? n_in : 1));
    int n = 0;
    for (int i = 0; i < n_in; ++i) {
        const float* d = plugin_out + 1 + (size_t)i * det_floats;
        float conf = d[4];
        if (variant == 2) {
            if ((double)conf <= conf_thresh) continue; /* common.hpp:113 `<= 0.1` double literal */
        } else {
            if (conf <= (float)conf_thresh) continue; /* kConfThresh is a float constant */
            if (variant == 0 && isnan(conf)) continue; /* v8 :99 */
        }
        keys[n].cls = (variant == 2) ? 0.0f : d[5];
        keys[n].conf = conf;
        keys[n].x0 = d[0];
        keys[n].src = i;
        ++n;
    }
    g_variant = variant;
    qsort(keys, (size_t)n, sizeof(nms_key), nms_cmp);
    char* erased = (char*)calloc((size_t)(n > 0 ? n : 1), 1);
    int n_keep = 0;
    for (int m = 0; m < n; ++m) {
        if (erased[m]) continue;
        const float* item = plugin_out + 1 + (size_t)keys[m].src * det_floats;
        memcpy(res + (size_t)n_keep * det_floats, item, sizeof(float) * det_floats);
        if (res_src) res_src[n_keep] = keys[m].src;
        ++n_keep;
        for (int q = m + 1; q < n && keys[q].cls == keys[m].cls; ++q) {
            if (erased[q]) continue;
            const float* other = plugin_out + 1 + (size_t)keys[q].src * det_floats;
            if (variant == 3) { /* nms_obb :357-385: probiou `>=` */
                if (probiou_host(item, other, det_floats - 1) >= nms_thresh) erased[q] = 1;
                continue;
            }
            float v = variant == 0 ? iou_ltrb(item, other) : (variant == 1 ? iou_cxcywh(item, other) : iou_retina(item, other));
            if (v > nms_thresh) erased[q] = 1; /* dets.erase(...) */
        }
    }
    free(erased);
    free(keys);
    return n_keep;
}

/* ------------------------------------------------------------------------------------------
 * GPU post-process of yolov8 (mode "g"): decode_kernel + nms_kernel,
 * yolov8/src/postprocess.cu:42-111, batch 1 in the reference.  ONE-SHOT (non-greedy) NMS:
 * a row is dropped if ANY same-class row with higher conf (ties: higher index wins, :100-102)
 * overlaps it, regardless of that row's own fate.
 * predict : plugin output of one image [1 + max_rows*det_floats]
 * parray  : [1 + max_objects*7] = count, (l,t,r,b,conf,cls,keep)*; rows emitted in input order
 *           (the reference's order is atomicAdd arrival); slots whose conf < thr stay zero (holes).
 * ------------------------------------------------------------------------------------------ */
static float box_iou_gpu(float al, float at, float ar, float ab, float bl, float bt, float br, float bb) { /* :74-87 */
    float cl = al > bl ? al : bl, ct = at > bt ? at : bt;
    float cr = ar < br ? ar : br, cb = ab < bb ? ab : bb;
    float cw = cr - cl > 0.0f ? cr - cl : 0.0f, ch = cb - ct > 0.0f ? cb - ct : 0.0f;
    float c_area = cw * ch;
    if (c_area == 0.0f) return 0.0f;
    float aw = ar - al > 0.0f ? ar - al : 0.0f, ah = ab - at > 0.0f ? ab - at : 0.0f;
    float bw = br - bl > 0.0f ? br - bl : 0.0f, bh = bb - bt > 0.0f ? bb - bt : 0.0f;
    return c_area / (aw * ah + bw * bh - c_area);
}
ORACLE_API void oracle_cuda_decode_nms(const float* predict, int max_rows, int det_floats, float conf_thresh,
                                       float nms_thresh, int max_objects, float* parray) {
    memset(parray, 0, sizeof(float) * (size_t)(1 + max_objects * 7));
    int count = (int)predict[0];
    if (count > max_rows) count = max_rows;
    int index = 0;
    for (int pos = 0; pos < count; ++pos) { /* decode_kernel :42-72 */
        const float* pitem = predict + 1 + (size_t)pos * det_floats;
        int my = index++; /* atomicAdd(parray,1) before the conf test (:50) */
        if (my >= max_objects) continue;
        if (pitem[4] < conf_thresh) continue;
        float* po = parray + 1 + my * 7;
        po[0] = pitem[0];
        po[1] = pitem[1];
        po[2] = pitem[2];
        po[3] = pitem[3];
        po[4] = pitem[4];
        po[5] = pitem[5];
        po[6] = 1;
    }
    parray[0] = (float)index;
    int n = index < max_objects ? index : max_objects; /* nms_kernel :91 */
    char* drop = (char*)calloc((size_t)(n > 0 ? n : 1), 1);
    for (int p = 0; p < n; ++p) {
        const float* pc = parray + 1 + p * 7;
        for (int i = 0; i < n; ++i) {
            const float* pi = parray + 1 + i * 7;
            if (i == p || pc[5] != pi[5]) continue;
            if (pi[4] >= pc[4]) {
                if (pi[4] == pc[4] && i < p) continue;
                float v = box_iou_gpu(pc[0], pc[1], pc[2], pc[3], pi[0], pi[1], pi[2], pi[3]);
                if (v > nms_thresh) {
                    drop[p] = 1;
                    break;
                }
            }
        }
    }
    for (int p = 0; p < n; ++p)
        if (drop[p]) parray[1 + p * 7 + 6] = 0;
    free(drop);
}

/* The oriented-box flavour of the same post-process: decode_kernel_obb + nms_kernel_obb, yolov8/src/postprocess.cu:7-40,
 * 113-166.  parray rows are 8 floats (cx,cy,w,h,conf,cls,keep,angle), angle = Detection float 89; box_probiou is all
 * float (powf/logf/expf/sqrtf/cosf/sinf); `>` threshold. */
static void cov_dev(float w, float h, float r, float* a, float* b, float* c) {
    float a_val = w * w / 12.0f, b_val = h * h / 12.0f;
    float cos_r = cosf(r), sin_r = sinf(r);
    *a = a_val * cos_r * cos_r + b_val * sin_r * sin_r;
    *b = a_val * sin_r * sin_r + b_val * cos_r * cos_r;
    *c = (a_val - b_val) * sin_r * cos_r;
}
static float box_probiou_gpu(const float* p, const float* q) {
    const float eps = 1e-7;
    float a1, b1, c1, a2, b2, c2;
    cov_dev(p[2], p[3], p[7], &a1, &b1, &c1);
    cov_dev(q[2], q[3], q[7], &a2, &b2, &c2);
    float cx1 = p[0], cy1 = p[1], cx2 = q[0], cy2 = q[1];
    float t1 = ((a1 + a2) * powf(cy1 - cy2, 2) + (b1 + b2) * powf(cx1 - cx2, 2)) / ((a1 + a2) * (b1 + b2) - powf(c1 + c2, 2) + eps);
    float t2 = ((c1 + c2) * (cx2 - cx1) * (cy1 - cy2)) / ((a1 + a2) * (b1 + b2) - powf(c1 + c2, 2) + eps);
    float t3 = logf(((a1 + a2) * (b1 + b2) - powf(c1 + c2, 2)) /
                            (4 * sqrtf(fmaxf(a1 * b1 - c1 * c1, 0.0f)) * sqrtf(fmaxf(a2 * b2 - c2 * c2, 0.0f)) + eps) +
                    eps);
    float bd = 0.25f * t1 + 0.5f * t2 + 0.5f * t3;
    bd = fmaxf(fminf(bd, 100.0f), eps);
    float hd = sqrtf(1.0f - expf(-bd) + eps);
    return 1 - hd;
}
ORACLE_API void oracle_cuda_decode_nms_obb(const float* predict, int max_rows, int det_floats, float conf_thresh,
                                           float nms_thresh, int max_objects, float* parray) {
    memset(parray, 0, sizeof(float) * (size_t)(1 + max_objects * 8));
    int count = (int)predict[0];
    if (count > max_rows) count = max_rows;
    int index = 0;
    for (int pos = 0; pos < count; ++pos) { /* decode_kernel_obb :7-40 */
        const float* pitem = predict + 1 + (size_t)pos * det_floats;
        int my = index++;
        if (my >= max_objects) continue;
        if (pitem[4] < conf_thresh) continue;
        float* po = parray + 1 + my * 8;
        po[0] = pitem[0];
        po[1] = pitem[1];
        po[2] = pitem[2];
        po[3] = pitem[3];
        po[4] = pitem[4];
        po[5] = pitem[5];
        po[6] = 1;
        po[7] = pitem[det_floats - 1]; /* pitem[89] */
    }
    parray[0] = (float)index;
    int n = index < max_objects ? index : max_objects;
    char* drop = (char*)calloc((size_t)(n > 0 ? n : 1), 1);
    for (int p = 0; p < n; ++p) { /* nms_kernel_obb :147-166 */
        const float* pc = parray + 1 + p * 8;
        for (int i = 0; i < n; ++i) {
            const float* pi = parray + 1 + i * 8;
            if (i == p || pc[5] != pi[5]) continue;
            if (pi[4] >= pc[4]) {
                if (pi[4] == pc[4] && i < p) continue;
                if (box_probiou_gpu(pc, pi) > nms_thresh) {
                    drop[p] = 1;
                    break;
                }
            }
        }
    }
    for (int p = 0; p < n; ++p)
        if (drop[p]) parray[1 + p * 8 + 6] = 0;
    free(drop);
}

/* ------------------------------------------------------------------------------------------
 * Letterbox warp-affine pre-process.  Restates warpaffine_kernel + cuda_preprocess,
 * yolov8/src/preprocess.cu:7-117 (cv::invertAffineTransform restated in closed form,
 * the reference computes it in double then stores float: OpenCV's implementation works on
 * doubles for CV_32F input and saturate-casts the result).
 * src : u8 HWC BGR [sh, sw, 3]; dst : fp32 CHW RGB [3, dh, dw], /255, border 128.
 * ------------------------------------------------------------------------------------------ */
ORACLE_API void oracle_letterbox_matrix(int sw, int sh, int dw, int dh, float* d2s /*[6]*/) {
    float scale = fminf(dh / (float)sh, dw / (float)sw); /* :98 */
    float s2d[6];
    s2d[0] = scale;
    s2d[1] = 0;
    s2d[2] = (float)(-scale * sw * 0.5 + dw * 0.5); /* double expr -> float (:102) */
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

/* The bilinear sum w1 * v1 + w2 * v2 + w3 * v3 + w4 * v4 (:59-61) as nvcc's default FMA contraction evaluates it in
 * the reference's compiled warpaffine_kernel and in both paths of letterbox_kernel (one FMUL, three FFMA in the SASS of
 * each): the product w2 * v2 is rounded, every other product is fused into the running sum. */
static float bilinear_contracted(float w1, float v1, float w2, float v2, float w3, float v3, float w4, float v4) {
    return fmaf(w4, v4, fmaf(w3, v3, fmaf(w1, v1, w2 * v2)));
}

/* src rows are `pitch` bytes apart.  contracted = 0: the sum evaluated left to right with every product rounded (the
 * plain IEEE restatement); contracted = 1: bilinear_contracted, the exact expectation for the device kernels (fp32
 * output; an fp16 output is this value rounded to nearest). */
ORACLE_API void oracle_warpaffine(const uint8_t* src, int sw, int sh, int pitch, float* dst, int dw, int dh,
                                  int contracted) {
    float m[6];
    oracle_letterbox_matrix(sw, sh, dw, dh, m);
    const size_t line = (size_t)pitch;
    const uint8_t cv = 128; /* :115 */
    const int area = dw * dh;
    for (int pos = 0; pos < area; ++pos) {
        int dx = pos % dw, dy = pos / dw;
        float src_x = m[0] * dx + m[1] * dy + m[2] + 0.5f; /* :22-23 */
        float src_y = m[3] * dx + m[4] * dy + m[5] + 0.5f;
        float c0, c1, c2;
        if (src_x <= -1 || src_x >= sw || src_y <= -1 || src_y >= sh) {
            c0 = c1 = c2 = cv;
        } else {
            int y_low = (int)floorf(src_y), x_low = (int)floorf(src_x);
            int y_high = y_low + 1, x_high = x_low + 1;
            const uint8_t cvv[3] = {cv, cv, cv};
            float ly = src_y - y_low, lx = src_x - x_low;
            float hy = 1 - ly, hx = 1 - lx;
            float w1 = hy * hx, w2 = hy * lx, w3 = ly * hx, w4 = ly * lx;
            const uint8_t *v1 = cvv, *v2 = cvv, *v3 = cvv, *v4 = cvv;
            if (y_low >= 0) {
                if (x_low >= 0) v1 = src + (size_t)y_low * line + x_low * 3;
                if (x_high < sw) v2 = src + (size_t)y_low * line + x_high * 3;
            }
            if (y_high < sh) {
                if (x_low >= 0) v3 = src + (size_t)y_high * line + x_low * 3;
                if (x_high < sw) v4 = src + (size_t)y_high * line + x_high * 3;
            }
            if (contracted) {
                c0 = bilinear_contracted(w1, v1[0], w2, v2[0], w3, v3[0], w4, v4[0]);
                c1 = bilinear_contracted(w1, v1[1], w2, v2[1], w3, v3[1], w4, v4[1]);
                c2 = bilinear_contracted(w1, v1[2], w2, v2[2], w3, v3[2], w4, v4[2]);
            } else {
                c0 = w1 * v1[0] + w2 * v2[0] + w3 * v3[0] + w4 * v4[0];
                c1 = w1 * v1[1] + w2 * v2[1] + w3 * v3[1] + w4 * v4[1];
                c2 = w1 * v1[2] + w2 * v2[2] + w3 * v3[2] + w4 * v4[2];
            }
        }
        float t = c2; /* bgr -> rgb :66-69 */
        c2 = c0;
        c0 = t;
        c0 = c0 / 255.0f;
        c1 = c1 / 255.0f;
        c2 = c2 / 255.0f;
        dst[(size_t)dy * dw + dx] = c0;
        dst[(size_t)area + (size_t)dy * dw + dx] = c1;
        dst[2 * (size_t)area + (size_t)dy * dw + dx] = c2;
    }
}

/* ==========================================================================================
 * Faster R-CNN plugins (rcnn/).  cub::DeviceRadixSort::SortPairsDescending is a STABLE
 * descending sort of fp32 keys with an iota payload => ties keep ascending original index.
 * ========================================================================================== */
typedef struct {
    float key;
    int idx;
} sort_pair;
static int sort_pair_desc(const void* pa, const void* pb) {
    const sort_pair* a = (const sort_pair*)pa;
    const sort_pair* b = (const sort_pair*)pb;
    if (a->key != b->key) return a->key > b->key ? -1 : 1;
    return a->idx < b->idx ? -1 : (a->idx > b->idx ? 1 : 0);
}
/* sort (keys[i], i) descending, stable */
static sort_pair* stable_sort_desc(const float* keys, int n) {
    sort_pair* p = (sort_pair*)malloc(sizeof(sort_pair) * (size_t)(n > 0 ? n : 1));
    for (int i = 0; i < n; ++i) {
        p[i].key = keys[i];
        p[i].idx = i;
    }
    qsort(p, (size_t)n, sizeof(sort_pair), sort_pair_desc);
    return p;
}

/* rcnn/RpnDecode.cu:27-143.  scores [B, A, H, W]; deltas [B, A*4, H, W]; anchors [A*4];
 * out_scores [B, top_n]; out_boxes [B, top_n, 4]. */
ORACLE_API void oracle_rpn_decode(int batch, const float* scores, const float* deltas, int height, int width,
                                  int image_height, int image_width, float stride, const float* anchors,
                                  int num_anchors, int top_n, float* out_scores, float* out_boxes) {
    const int scores_size = num_anchors * height * width;
    for (int b = 0; b < batch; ++b) {
        const float* in_scores = scores + (size_t)b * scores_size;
        const float* in_boxes = deltas + (size_t)b * scores_size * 4;
        float* os = out_scores + (size_t)b * top_n;
        float* ob = out_boxes + (size_t)b * top_n * 4;
        sort_pair* sp = NULL;
        int num_det = scores_size;
        if (num_det > top_n) { /* :79-86 */
            sp = stable_sort_desc(in_scores, scores_size);
            num_det = top_n;
        }
        for (int r = 0; r < num_det; ++r) {
            int i = sp ? sp[r].idx : r;
            int x = i % width;
            int y = (i / width) % height;
            int a = (i / height / width) % num_anchors;
            float bx = in_boxes[((size_t)(a * 4 + 0) * height + y) * width + x];
            float by = in_boxes[((size_t)(a * 4 + 1) * height + y) * width + x];
            float bz = in_boxes[((size_t)(a * 4 + 2) * height + y) * width + x];
            float bw = in_boxes[((size_t)(a * 4 + 3) * height + y) * width + x];
            if (num_anchors > 0 && anchors) { /* has_anchors :107-131 */
                float fx = (i % width) * stride;
                float fy = ((i / width) % height) * stride;
                const float* d = anchors + 4 * a;
                float x1 = fx + d[0], y1 = fy + d[1], x2 = fx + d[2], y2 = fy + d[3];
                float w = x2 - x1, h = y2 - y1;
                float pcx = bx * w + x1 + 0.5f * w;
                float pcy = by * h + y1 + 0.5f * h;
                float pw = expf(bz) * w;
                float ph = expf(bw) * h;
                bx = fmaxf(0.0f, pcx - 0.5f * pw);
                by = fmaxf(0.0f, pcy - 0.5f * ph);
                bz = fminf(pcx + 0.5f * pw, (float)image_width);
                bw = fminf(pcy + 0.5f * ph, (float)image_height);
            }
            ob[r * 4 + 0] = bx;
            ob[r * 4 + 1] = by;
            ob[r * 4 + 2] = bz;
            ob[r * 4 + 3] = bw;
            os[r] = (bz - bx <= 0.0f || bw - by <= 0.0f) ? -FLT_MAX : in_scores[i]; /* :129-132 */
        }
        for (int r = num_det; r < top_n; ++r) os[r] = -FLT_MAX; /* :136-139; boxes left untouched */
        free(sp);
    }
}

static float iou_plain(const float* i, const float* m) { /* rcnn/RpnNms.cu:38-50, BatchedNms.cu:43-55 */
    float x1 = fmaxf(i[0], m[0]), y1 = fmaxf(i[1], m[1]);
    float x2 = fminf(i[2], m[2]), y2 = fminf(i[3], m[3]);
    float w = fmaxf(0.0f, x2 - x1), h = fmaxf(0.0f, y2 - y1);
    float iarea = (i[2] - i[0]) * (i[3] - i[1]);
    float marea = (m[2] - m[0]) * (m[3] - m[1]);
    float inter = w * h;
    return inter / (iarea + marea - inter);
}

/* rcnn/RpnNms.cu:27-121 with the INTENDED (race-free, grid-synchronous) semantics of
 * rpn_nms_kernel: for m ascending, if scores[m] > -FLT_MAX, every i>m with IoU > thr gets
 * -FLT_MAX.  Then stable re-sort and gather the first post_nms_topk boxes (:111-117) -- so
 * when fewer than post_nms_topk survive, suppressed boxes follow in their sorted order. */
ORACLE_API void oracle_rpn_nms(int batch, const float* in_scores, const float* in_boxes, int pre_nms_topk,
                               int post_nms_topk, float nms_thresh, float* out_boxes) {
    for (int b = 0; b < batch; ++b) {
        const float* sc = in_scores + (size_t)b * pre_nms_topk;
        const float* bx = in_boxes + (size_t)b * pre_nms_topk * 4;
        float* ob = out_boxes + (size_t)b * post_nms_topk * 4;
        sort_pair* sp = stable_sort_desc(sc, pre_nms_topk);
        float* s = (float*)malloc(sizeof(float) * (size_t)pre_nms_topk);
        for (int i = 0; i < pre_nms_topk; ++i) s[i] = sp[i].key;
        for (int m = 0; m < pre_nms_topk; ++m) {
            if (!(s[m] > -FLT_MAX)) continue;
            const float* mbox = bx + (size_t)sp[m].idx * 4;
            for (int i = m + 1; i < pre_nms_topk; ++i) {
                if (iou_plain(bx + (size_t)sp[i].idx * 4, mbox) > nms_thresh) s[i] = -FLT_MAX;
            }
        }
        sort_pair* sp2 = stable_sort_desc(s, pre_nms_topk); /* idx here = position in first sort */
        int n = post_nms_topk < pre_nms_topk ? post_nms_topk : pre_nms_topk;
        for (int r = 0; r < n; ++r) memcpy(ob + r * 4, bx + (size_t)sp[sp2[r].idx].idx * 4, sizeof(float) * 4);
        free(sp2);
        free(s);
        free(sp);
    }
}

/* rcnn/PredictorDecode.cu:24-110.  scores [B, N, C]; deltas [B, N*C, 4]; proposals [B, N, 4].
 * NOTE the reference clips y2 with image_WIDTH (:99) -- restated as is. */
ORACLE_API void oracle_predictor_decode(int batch, const float* scores, const float* deltas, const float* proposals,
                                        int num_boxes, int num_classes, int image_height, int image_width,
                                        const float* w4, float* out_scores, float* out_boxes, float* out_classes) {
    (void)image_height;
    const int scores_size = num_boxes * num_classes;
    for (int b = 0; b < batch; ++b) {
        const float* in_scores = scores + (size_t)b * scores_size;
        const float* in_boxes = deltas + (size_t)b * scores_size * 4;
        const float* in_prop = proposals + (size_t)b * num_boxes * 4;
        sort_pair* sp = stable_sort_desc(in_scores, scores_size);
        for (int r = 0; r < num_boxes; ++r) {
            int i = sp[r].idx;
            int cls = i % num_classes;
            int n = i / num_classes;
            const float* d = in_boxes + (size_t)i * 4;
            const float* p = in_prop + (size_t)n * 4;
            float w = p[2] - p[0], h = p[3] - p[1];
            float pcx = (d[0] / w4[0]) * w + p[0] + 0.5f * w;
            float pcy = (d[1] / w4[1]) * h + p[1] + 0.5f * h;
            float pw = expf(d[2] / w4[2]) * w;
            float ph = expf(d[3] / w4[3]) * h;
            float bx = fmaxf(0.0f, pcx - 0.5f * pw);
            float by = fmaxf(0.0f, pcy - 0.5f * ph);
            float bz = fminf(pcx + 0.5f * pw, (float)image_width);
            float bw = fminf(pcy + 0.5f * ph, (float)image_width); /* sic, :99 */
            float* ob = out_boxes + ((size_t)b * num_boxes + r) * 4;
            ob[0] = bx;
            ob[1] = by;
            ob[2] = bz;
            ob[3] = bw;
            out_scores[(size_t)b * num_boxes + r] = (bz - bx <= 0.0f || bw - by <= 0.0f) ? 0.0f : in_scores[i];
            out_classes[(size_t)b * num_boxes + r] = (float)cls;
        }
        free(sp);
    }
}

/* rcnn/BatchedNms.cu:28-162, intended race-free semantics; nms_method 0 hard / 1 linear soft /
 * 2 gaussian soft (sigma 0.5), other = hard (:60-88).  `scores[m] > 0.0f` gates the suppressor. */
ORACLE_API void oracle_batched_nms(int nms_method, int batch, const float* in_scores, const float* in_boxes,
                                   const float* in_classes, int count, int detections_per_im, float nms_thresh,
                                   float* out_scores, float* out_boxes, float* out_classes) {
    for (int b = 0; b < batch; ++b) {
        const float* sc = in_scores + (size_t)b * count;
        const float* bx = in_boxes + (size_t)b * count * 4;
        const float* cl = in_classes + (size_t)b * count;
        sort_pair* sp = stable_sort_desc(sc, count);
        float* s = (float*)malloc(sizeof(float) * (size_t)count);
        for (int i = 0; i < count; ++i) s[i] = sp[i].key;
        for (int m = 0; m < count; ++m) {
            if (!(s[m] > 0.0f)) continue;
            int mcls = (int)cl[sp[m].idx];
            const float* mbox = bx + (size_t)sp[m].idx * 4;
            for (int i = m + 1; i < count; ++i) {
                int icls = (int)cl[sp[i].idx];
                if (mcls != icls) continue;
                float overlap = iou_plain(bx + (size_t)sp[i].idx * 4, mbox);
                const float sigma = 0.5f;
                if (overlap > nms_thresh) {
                    if (nms_method == 1)
                        s[i] = (1 - overlap) * s[i];
                    else if (nms_method == 2)
                        s[i] = expf(-(overlap * overlap) / sigma) * s[i];
                    else
                        s[i] = 0.0f;
                }
            }
        }
        sort_pair* sp2 = stable_sort_desc(s, count);
        int n = detections_per_im < count ? detections_per_im : count;
        for (int r = 0; r < n; ++r) {
            int src = sp[sp2[r].idx].idx;
            out_scores[(size_t)b * detections_per_im + r] = sp2[r].key;
            memcpy(out_boxes + ((size_t)b * detections_per_im + r) * 4, bx + (size_t)src * 4, sizeof(float) * 4);
            out_classes[(size_t)b * detections_per_im + r] = cl[src];
        }
        for (int r = n; r < detections_per_im; ++r) out_scores[(size_t)b * detections_per_im + r] = 0.0f; /* :152-154 */
        free(sp2);
        free(s);
        free(sp);
    }
}

/* ------------------------------------------------------------------------------------------
 * Timing helper for bench.py's cpu_baseline: decode + nms over `batch` images, returns the
 * number of kept rows (so the work cannot be optimised away).  Single thread; the caller
 * parallelises over images with one call per thread.
 * ------------------------------------------------------------------------------------------ */
ORACLE_API int oracle_yolov8_decode_nms_image(const float* const* inputs /* per level, ONE image */, int num_levels,
                                              const int* grid_h, const int* grid_w, const int* strides, int classes,
                                              int max_out, int det_floats, float gate, float conf_thresh,
                                              float nms_thresh, float* scratch_out /*[1+max_out*det_floats]*/,
                                              float* res /*[max_out*det_floats]*/) {
    oracle_yolov8_decode(inputs, 1, num_levels, grid_h, grid_w, strides, classes, 17, 0.0f, 0, 0, 0, max_out,
                         det_floats, gate, scratch_out, NULL);
    return oracle_nms(0, scratch_out, max_out, det_floats, conf_thresh, nms_thresh, res, NULL);
}

/* ------------------------------------------------------------------------------------------
 * process_mask: yolov8/yolov8_seg.cpp:17-60 (variant 0) and yolov5/src/postprocess.cpp:94-125 (variant 1), one
 * detection.  proto [nm, mh, mw]; bbox/coeffs = Detection.bbox / Detection.mask; out [net_h, net_w].
 * cv::resize(CV_32FC1, INTER_LINEAR) restated from OpenCV's resize.cpp (fx = (dx+0.5)*scale-0.5, floor, clamp with
 * zero fraction, horizontal pass then vertical pass in float); checked against cv2 4.13 in tests/test_oracle_cpu.py.
 * The x/y loops are clamped to the mask (the reference would index out of bounds for a yolov5 box leaving the image).
 * Where one of get_downscale_rect's float -> int conversions is undefined (NaN, +-inf, past the int range; x86 gives
 * INT_MIN) the mask stays all zeros, as the library documents; rx + rw is summed in 64 bits.
 * ------------------------------------------------------------------------------------------ */
static void resize_tap(int d, double scale, int src, int* s0, float* f) {
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
    *s0 = sx;
    *f = fx;
}
ORACLE_API void oracle_resize_bilinear(const float* src, int sh, int sw, float* dst, int dh, int dw) {
    double scale_x = (double)sw / dw, scale_y = (double)sh / dh;
    for (int y = 0; y < dh; ++y) {
        int sy;
        float fy;
        resize_tap(y, scale_y, sh, &sy, &fy);
        int sy1 = sy + 1 < sh ? sy + 1 : sh - 1;
        float b0 = 1.0f - fy, b1 = fy;
        for (int x = 0; x < dw; ++x) {
            int sx;
            float fx;
            resize_tap(x, scale_x, sw, &sx, &fx);
            int sx1 = sx + 1 < sw ? sx + 1 : sw - 1;
            float a0 = 1.0f - fx, a1 = fx;
            float h0 = src[(size_t)sy * sw + sx] * a0 + src[(size_t)sy * sw + sx1] * a1;
            float h1 = src[(size_t)sy1 * sw + sx] * a0 + src[(size_t)sy1 * sw + sx1] * a1;
            dst[(size_t)y * dw + x] = h0 * b0 + h1 * b1;
        }
    }
}
/* (int)v and (int)round(v) where they are defined */
static int trunc_fits(float v) { return v >= -2147483648.0f && v < 2147483648.0f; }
static int round_fits(float v) {
    double r = round((double)v);
    return r >= -2147483648.0 && r <= 2147483647.0;
}
ORACLE_API void oracle_process_mask(int variant, const float* proto, int nm, int mh, int mw, int net_w, int net_h,
                                    const float* bbox, const float* coeffs, float* out) {
    float* m = (float*)calloc((size_t)mh * mw, sizeof(float)); /* cv::Mat::zeros */
    float left, top, right, bottom;
    int rx = 0, ry = 0, rw = 0, rh = 0;
    if (variant == 0) { /* yolov8_seg.cpp:17-34 */
        left = bbox[0];
        top = bbox[1];
        right = bbox[0] + bbox[2];
        bottom = bbox[1] + bbox[3];
        left = left < 0 ? 0 : left;
        top = top < 0 ? 0 : top;
        right = right > net_w ? net_w : right;
        bottom = bottom > net_h ? net_h : bottom;
        left /= 4.0f;
        top /= 4.0f;
        right /= 4.0f;
        bottom /= 4.0f;
        if (trunc_fits(left) && trunc_fits(top) && trunc_fits(right - left) && trunc_fits(bottom - top)) {
            rx = (int)left;
            ry = (int)top;
            rw = (int)(right - left);
            rh = (int)(bottom - top);
        }
    } else { /* yolov5/src/postprocess.cpp:94-104 */
        left = bbox[0] - bbox[2] / 2;
        top = bbox[1] - bbox[3] / 2;
        right = bbox[0] + bbox[2] / 2;
        bottom = bbox[1] + bbox[3] / 2;
        left /= 4.0f;
        top /= 4.0f;
        right /= 4.0f;
        bottom /= 4.0f;
        if (round_fits(left) && round_fits(top) && round_fits(right - left) && round_fits(bottom - top)) {
            rx = (int)round(left);
            ry = (int)round(top);
            rw = (int)round(right - left);
            rh = (int)round(bottom - top);
        }
    }
    size_t plane = (size_t)mh * mw; /* proto_size / 32 */
    const long long x_hi = (long long)rx + rw < mw ? (long long)rx + rw : mw;
    const long long y_hi = (long long)ry + rh < mh ? (long long)ry + rh : mh;
    for (long long x = rx > 0 ? rx : 0; x < x_hi; ++x) {
        for (long long y = ry > 0 ? ry : 0; y < y_hi; ++y) {
            float e = 0.0f;
            for (int j = 0; j < nm; ++j) e += coeffs[j] * proto[(size_t)j * plane + (size_t)y * mw + x];
            m[(size_t)y * mw + x] = 1.0f / (1.0f + expf(-e));
        }
    }
    oracle_resize_bilinear(m, mh, mw, out, net_h, net_w);
    free(m);
}

/* ------------------------------------------------------------------------------------------
 * RoIAlign: RoIAlignForward + bilinear_interpolate, rcnn/RoiAlign.cu:29-149 (one image).
 * rois [N,4] x1,y1,x2,y2; feat [C,H,W]; out [N,C,P,P].  T = float; the double literals of the reference
 * (-1.0, `1. - ly`) are kept.
 * ------------------------------------------------------------------------------------------ */
static float roi_bilinear(const float* bottom, int height, int width, float y, float x) {
    if (y < -1.0 || y > height || x < -1.0 || x > width) return 0;
    if (y <= 0) y = 0;
    if (x <= 0) x = 0;
    int y_low = (int)y, x_low = (int)x, y_high, x_high;
    if (y_low >= height - 1) {
        y_high = y_low = height - 1;
        y = (float)y_low;
    } else {
        y_high = y_low + 1;
    }
    if (x_low >= width - 1) {
        x_high = x_low = width - 1;
        x = (float)x_low;
    } else {
        x_high = x_low + 1;
    }
    float ly = y - y_low, lx = x - x_low;
    float hy = (float)(1. - ly), hx = (float)(1. - lx);
    float v1 = bottom[y_low * width + x_low], v2 = bottom[y_low * width + x_high];
    float v3 = bottom[y_high * width + x_low], v4 = bottom[y_high * width + x_high];
    float w1 = hy * hx, w2 = hy * lx, w3 = ly * hx, w4 = ly * lx;
    return w1 * v1 + w2 * v2 + w3 * v3 + w4 * v4;
}
ORACLE_API void oracle_roi_align(const float* rois, const float* feat, float* out, int N, int C, int H, int W, int P,
                                 float spatial_scale, int sampling_ratio) {
    for (int n = 0; n < N; ++n) {
        const float* r = rois + 4 * n;
        float roi_offset = 0.5f;
        float roi_start_w = r[0] * spatial_scale - roi_offset, roi_start_h = r[1] * spatial_scale - roi_offset;
        float roi_end_w = r[2] * spatial_scale - roi_offset, roi_end_h = r[3] * spatial_scale - roi_offset;
        float roi_width = roi_end_w - roi_start_w, roi_height = roi_end_h - roi_start_h;
        float bin_size_h = roi_height / (float)P, bin_size_w = roi_width / (float)P;
        int gh = sampling_ratio > 0 ? sampling_ratio : (int)ceilf(roi_height / P);
        int gw = sampling_ratio > 0 ? sampling_ratio : (int)ceilf(roi_width / P);
        const float count = (float)(gh * gw);
        for (int c = 0; c < C; ++c) {
            const float* fm = feat + (size_t)c * H * W;
            for (int ph = 0; ph < P; ++ph)
                for (int pw = 0; pw < P; ++pw) {
                    float acc = 0.f;
                    for (int iy = 0; iy < gh; iy++) {
                        const float y = roi_start_h + ph * bin_size_h + (float)(iy + .5f) * bin_size_h / (float)gh;
                        for (int ix = 0; ix < gw; ix++) {
                            const float x = roi_start_w + pw * bin_size_w + (float)(ix + .5f) * bin_size_w / (float)gw;
                            acc += roi_bilinear(fm, H, W, y, x);
                        }
                    }
                    acc /= count;
                    out[(((size_t)n * C + c) * P + ph) * P + pw] = acc;
                }
        }
    }
}
/* MaskRcnnInferenceKernel, rcnn/MaskRcnnInference.cu:8-33 (one image); rows whose class index is out of range stay
 * as they are in `out`. */
ORACLE_API void oracle_mask_rcnn_inference(const float* indices, const float* masks, float* out, int D, int S, int nc) {
    for (int d = 0; d < D; ++d) {
        int cls = (int)indices[d];
        if (cls < 0 || cls >= nc) continue;
        for (int i = 0; i < S * S; ++i) out[(size_t)d * S * S + i] = logist(masks[((size_t)d * nc + cls) * S * S + i]);
    }
}

/* ------------------------------------------------------------------------------------------
 * get_rect: yolov8/src/postprocess.cpp:6-36 (variant 0: box l,t,r,b; result clamped to the image) and
 * yolov5/src/postprocess.cpp:4-29 (variant 1: box cx,cy,w,h; no clamping).  `kInputW / (img.cols * 1.0)` is a double
 * division stored to float; everything after it is float; round() is C round() on the float promoted to double.
 * ------------------------------------------------------------------------------------------ */
ORACLE_API void oracle_get_rect(int variant, int net_w, int net_h, int img_w, int img_h, const float* bbox, int* rect) {
    float l, r, t, b;
    float r_w = (float)(net_w / (img_w * 1.0));
    float r_h = (float)(net_h / (img_h * 1.0));
    if (variant == 0) {
        if (r_h > r_w) {
            l = bbox[0];
            r = bbox[2];
            t = bbox[1] - (net_h - r_w * img_h) / 2;
            b = bbox[3] - (net_h - r_w * img_h) / 2;
            l = l / r_w;
            r = r / r_w;
            t = t / r_w;
            b = b / r_w;
        } else {
            l = bbox[0] - (net_w - r_h * img_w) / 2;
            r = bbox[2] - (net_w - r_h * img_w) / 2;
            t = bbox[1];
            b = bbox[3];
            l = l / r_h;
            r = r / r_h;
            t = t / r_h;
            b = b / r_h;
        }
        l = 0.0f > l ? 0.0f : l; /* std::max(0.0f, l) */
        t = 0.0f > t ? 0.0f : t;
        int rw = (int)round(r - l), rl = (int)round(l), rh = (int)round(b - t), rt = (int)round(t);
        int width = rw < img_w - rl ? rw : img_w - rl;
        int height = rh < img_h - rt ? rh : img_h - rt;
        rect[0] = rl;
        rect[1] = rt;
        rect[2] = width > 0 ? width : 0;
        rect[3] = height > 0 ? height : 0;
    } else {
        if (r_h > r_w) {
            l = bbox[0] - bbox[2] / 2.f;
            r = bbox[0] + bbox[2] / 2.f;
            t = bbox[1] - bbox[3] / 2.f - (net_h - r_w * img_h) / 2;
            b = bbox[1] + bbox[3] / 2.f - (net_h - r_w * img_h) / 2;
            l = l / r_w;
            r = r / r_w;
            t = t / r_w;
            b = b / r_w;
        } else {
            l = bbox[0] - bbox[2] / 2.f - (net_w - r_h * img_w) / 2;
            r = bbox[0] + bbox[2] / 2.f - (net_w - r_h * img_w) / 2;
            t = bbox[1] - bbox[3] / 2.f;
            b = bbox[1] + bbox[3] / 2.f;
            l = l / r_h;
            r = r / r_h;
            t = t / r_h;
            b = b / r_h;
        }
        rect[0] = (int)round(l);
        rect[1] = (int)round(t);
        rect[2] = (int)round(r - l);
        rect[3] = (int)round(b - t);
    }
}

