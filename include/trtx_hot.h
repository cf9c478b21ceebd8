/*
 * trtx_hot.h -- C ABI of the H100-native detection hot path (libtrtx_hot.so).
 *
 * This is the drop-in boundary: every entry point below is what a TensorRT plugin's
 * enqueue()/getWorkspaceSize() (or the driver's cuda_* helper) in wang-xinyu/tensorrtx
 * binds to.  Plain pointers and sizes only; all pointers named *_dev are DEVICE pointers
 * owned by the caller (TensorRT owns inputs/outputs/workspace, SURVEY.md section 8b);
 * nothing is allocated, freed, retained or synchronised inside an enqueue; every call is
 * re-entrant and ordered on the given stream.  Return value: 0 = success (the reference's
 * enqueue() convention, yolov8/plugin/yololayer.cu:171), non-zero = TRTX_ERR_*; the library
 * never throws and never asserts.
 *
 * Reference citations are relative to the root of wang-xinyu/tensorrtx @ 3ff22bb4.
 * The header-only TensorRT adapters that forward the IPluginV2DynamicExt / IPluginV2IOExt /
 * IPluginV2Ext virtuals to these functions live in include/trtx_plugins.h; the binding a
 * maintainer adds on the reference side is shown in INTEGRATION.md.
 */
#ifndef TRTX_HOT_H
#define TRTX_HOT_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(_WIN32)
#define TRTX_API __declspec(dllexport)
#else
#define TRTX_API __attribute__((visibility("default")))
#endif

/* cudaStream_t, spelled without <cuda_runtime.h> so that C / cgo / ctypes callers can include this. */
typedef void* trtx_stream_t;

enum {
    TRTX_OK = 0,
    TRTX_ERR_INVALID = 1,     /* malformed params / null pointer */
    TRTX_ERR_WORKSPACE = 2,   /* workspace too small (the reference throws here, rcnn/cuda_utils.h:22-24) */
    TRTX_ERR_CUDA = 3,        /* a launch failed; see trtx_last_cuda_error() */
    TRTX_ERR_UNSUPPORTED = 4, /* parameter combination outside what the kernels cover */
};

#define TRTX_MAX_LEVELS 8

TRTX_API const char* trtx_version(void);
/* cudaError_t of the last failing launch on this thread (0 if none). */
TRTX_API int trtx_last_cuda_error(void);
/* sizeof() of the parameter structs as THIS library was compiled, so that an FFI binding (ctypes, cgo, ...) can check its
 * mirror of the layout: which = 0 trtx_yolo_params, 1 trtx_nms_params, 2 trtx_retina_params, 3 trtx_image_desc,
 * 4 trtx_mask_params, 5 trtx_rcnn_post_params, 6 trtx_frame, 7 trtx_pose_obb_params, 8 trtx_frame,
 * 9 trtx_face_post_params, 10 trtx_yolop_post_params, 11 trtx_detr_post_params, 12 trtx_centernet_params,
 * 13 trtx_ufld_post_params, 14 trtx_refinedet_params, 15 trtx_yolo_topk_params, 16 trtx_pyrunner_params;
 * anything else 0. */
TRTX_API size_t trtx_abi_sizeof(int which);

/* =====================================================================================
 * 1. YoloLayer_TRT  -- fused per-anchor sigmoid / argmax / gate / box decode / compaction
 *    replaces CalDetection + forwardGpu of
 *      yolov8/plugin/yololayer.cu:178-316 (anchor-free: yolov8, yolo11, yolov12; yolov9 with det_floats 38,
 *        yolov10 and yolov13 with det_floats 6 -- each of their CalDetection is yolov8's arithmetic)
 *      yolov5/plugin/yololayer.cu:161-227 (anchor-based: yolov5, yolov7, yolov5-lite, yolop)
 * ===================================================================================== */
enum {
    TRTX_YOLO_V8 = 0,
    TRTX_YOLO_V5 = 1,
    /* SURVEY 8f rank 4 -- older / other YoloLayer variants through the same scan / pack / NMS kernels: */
    TRTX_YOLO_V3 = 2,  /* yolov3-spp (yolov3-spp/yololayer.cu:148-191): anchor-based like V5, but box =
                          ((col + sigmoid(x)) * stride, ..., exp(w) * anchor_w, ...), class AND objectness gated, rows of 7
                          floats x,y,w,h, det_confidence, class_id, class_confidence (yololayer.h:47-53).  `strides` and
                          `anchors` are both used; det_floats >= 7.  The rectangle entry points (trtx_get_rect, the rows of
                          trtx_yolo_seg_postprocess_enqueue) take this value for the whole family below */
    TRTX_YOLO_V26 = 3, /* yolo26 NMS-free gatherKernel (yolo26/plugin/yololayer.cu:178-245): ONE input
                          [batch, anchors, 4 + num_classes (+1 angle when is_obb)], row-major per anchor, scores are
                          probabilities already; argmax `>` from (0, class -1), rows with score < gate dropped, 90-float
                          rows, everything the kernel does not write is zero (the reference memsets the buffer).
                          num_levels = 1, grid_h[0] * grid_w[0] = anchor count.  The reference decodes image 0 only
                          (":185 TODO"); this build decodes every image of the batch */
    /* The rest of the yolov3 family: TRTX_YOLO_V3's gates, rows, grids and anchors (`strides` unused), another box and sigmoid.
     * Every entry point that takes TRTX_YOLO_V3 for a decode takes these too, fp16 heads included. */
    TRTX_YOLO_V3_NET = 4, /* yolov3, yolov3-tiny (yolov3/yololayer.cu:173-176, yolov3-tiny/yololayer.cu:172-175):
                             x = ((float)col + sigmoid(x0)) * (float)net_w / (float)grid_w, in float left to right with an IEEE
                             divide (y with net_h, grid_h); w = expf(x2) * anchor_w.  Logist = 1.0f / (1.0f + expf(-x)) */
    TRTX_YOLO_V4 = 5,     /* yolov4 (yolov4/yololayer.cu:154, :191-194): TRTX_YOLO_V3_NET's box, but Logist = 1. / (1. + exp(-x))
                             in double, rounded to float -- for the gates, both confidences and the box */
    TRTX_YOLO_V4_CSP = 6, /* scaled-yolov4 (scaled-yolov4/yololayer.cu:154, :191-194): TRTX_YOLO_V4's double Logist;
                             x = (float)(((double)((float)col + 2.0f * sigmoid(x0)) - 0.5) * net_w / grid_w) in double (the
                             `- 0.5` is a double literal); w = powf(2.0f * sigmoid(x2), 2.0f) * anchor_w */
};
enum { TRTX_F32 = 0, TRTX_F16 = 1 };

typedef struct trtx_yolo_params {
    int32_t variant;     /* TRTX_YOLO_V8 | TRTX_YOLO_V5 | TRTX_YOLO_V3 | TRTX_YOLO_V26 | TRTX_YOLO_V3_NET | TRTX_YOLO_V4 |
                            TRTX_YOLO_V4_CSP */
    int32_t num_classes; /* combinedInfo[0] (yolov8/src/block.cpp:268) | netinfo[0] (yolov5/src/model.cpp:249) */
    int32_t net_w;       /* kInputW */
    int32_t net_h;       /* kInputH */
    int32_t max_out;     /* kMaxNumOutputBbox: capacity of the plugin output, rows per image */
    int32_t det_floats;  /* sizeof(Detection)/4 of the model dir: 90 (yolov8/include/types.h:4-12),
                            38 (yolov5/src/types.h:11-16), 6 (yolov7/10/13: yolov7/include/types.h:11-16),
                            7 (yolov3-spp/yololayer.h:47-53) */
    int32_t num_levels;  /* number of input tensors (strides) */
    int32_t grid_h[TRTX_MAX_LEVELS]; /* v8: net_h/stride (yololayer.cu:294); v5: YoloKernel.height */
    int32_t grid_w[TRTX_MAX_LEVELS];
    int32_t strides[TRTX_MAX_LEVELS];   /* v8 only (combinedInfo[9..]) */
    float anchors[TRTX_MAX_LEVELS][6];  /* v5 only: YoloKernel.anchors (yolov5/src/types.h:5-9) */
    int32_t is_seg;      /* copy 32 mask coefficients */
    int32_t is_pose;     /* v8: decode num_kpts keypoints */
    int32_t is_obb;      /* v8: rotated box */
    int32_t num_kpts;    /* combinedInfo[1] */
    float kpt_thresh;    /* combinedInfo[2] (int-truncated by the reference builder, block.cpp:271) */
    float gate;          /* 0.1f: literal of yolov8 yololayer.cu:203 / kIgnoreThresh yolov5 config.h:38 / IGNORE_THRESH
                            yolov3-spp yololayer.h:15; V26: the confidence threshold (d_confThreshold, yololayer.cu:9,32) */
    int32_t in_dtype;    /* TRTX_F32 (parity mode, what the reference accepts, yololayer.h:32-35) | TRTX_F16 */
    /* Launch tuning of the scan kernel.  Plain per-call data: the library keeps NO mutable state, so concurrent enqueues
     * (TensorRT calls enqueue() on clones from several threads, SURVEY 8b "Threading") with different tunings are
     * independent.  0 everywhere -- what memset / trtx_yolo_params_init_v8 leave -- selects the defaults chosen on an H100 for
     * the overlapped benchmark step (DESIGN.md section 4.1).  A combination that is not built returns TRTX_ERR_UNSUPPORTED. */
    int32_t tune_class_slices;   /* warps of a CTA splitting the class range: 1, 2, 4, 8; 0 = 4 (fp32 inputs, 4 anchors per lane), else 2 */
    int32_t tune_rows_in_flight; /* channel rows loaded per group; 0 = 10 (fp32 inputs with 4 anchors per lane, fp16 inputs with 8), else 5.  Built (slices, rows): (1,8) (1,16) (2,4) (2,5)
                                    (2,8) (2,10) (2,20) (4,4) (4,5) (4,10) (4,20) (8,5) (8,10) */
    int32_t tune_box_prefetch;   /* box rows of a tile: 1 on demand, 2 L2 prefetch, 3 into registers up front; 0 = 2 */
} trtx_yolo_params;

/* Fill grid_h/grid_w from net size and strides (v8) -- convenience, mirrors yololayer.cu:292-296. */
TRTX_API int trtx_yolo_params_init_v8(trtx_yolo_params* p, int num_classes, int net_w, int net_h, int max_out,
                                      const int* strides, int num_levels);

/* Scratch bytes for trtx_yolo_decode_enqueue / trtx_yolo_decode_nms_enqueue at `batch` images.
 * (The reference plugin needs none, yololayer.h:22; this build stages candidates per tile so that
 *  compaction is atomic-free and deterministic.) */
TRTX_API size_t trtx_yolo_workspace_size(const trtx_yolo_params* p, int batch);

/* Drop-in for YoloLayerPlugin::enqueue (yolov8/plugin/yololayer.cu:167-172, yolov5 :229-232).
 *  inputs_dev[l] : level-l tensor [batch, C_l, grid_h*grid_w], channel-major, fp32 (or fp16)
 *  output_dev    : [batch, 1 + max_out*det_floats] fp32: count, Detection rows.
 * Rows appear in ascending anchor order (deterministic; the reference's order is atomicAdd arrival).
 * count is clamped to max_out (the reference lets it run past, which overruns host readers). */
TRTX_API int trtx_yolo_decode_enqueue(const trtx_yolo_params* p, int batch, const void* const* inputs_dev,
                                      float* output_dev, void* workspace_dev, size_t workspace_bytes,
                                      trtx_stream_t stream);

/* =====================================================================================
 * 2. NMS -- sort + greedy class-aware NMS, one CTA per image, all images in one launch.
 *    replaces the host nms()/batch_nms() of yolov8/src/postprocess.cpp:94-129,
 *    yolov5/src/postprocess.cpp:49-80, retinaface/common.hpp:110-130 and the device
 *    cuda_decode()+cuda_nms() of yolov8/src/postprocess.cu:168-179 (batch 1 only there).
 * ===================================================================================== */
enum {
    TRTX_BOX_LTRB = 0,   /* yolov8 Detection: x1,y1,x2,y2; IoU of postprocess.cpp:71-85 */
    TRTX_BOX_CXCYWH = 1, /* yolov5 Detection: cx,cy,w,h;   IoU of yolov5 postprocess.cpp:30-43 */
    TRTX_BOX_RETINA = 2, /* retinaface: x1,y1,x2,y2, +1e-6f in the denominator, single class (common.hpp:91-104) */
    TRTX_BOX_OBB = 3,    /* yolov8-obb Detection: cx,cy,w,h + angle = the FIRST extra float (extra_floats >= 1,
                            extra_offset = 89 for plugin rows); greedy = nms_obb / probiou `>=`
                            (postprocess.cpp:303-385), one-shot = nms_kernel_obb / box_probiou `>`
                            (postprocess.cu:113-166).  Plugin-row source only (not the fused tile source). */
    TRTX_BOX_V9 = 4,     /* yolov9 (yolov9/src/postprocess.cpp:48-83): rows arrive x1,y1,x2,y2 and each becomes, in float,
                            cx = (x1 + x2) / 2, cy = (y1 + y2) / 2, w = x2 - x1, h = y2 - y1 before it is sorted or tested;
                            then TRTX_BOX_CXCYWH's IoU on the converted boxes, and the output rows hold the converted box
                            (what yolov9's get_rect receives).  Rounding in the conversion can decide a pair near nms_thresh
                            differently from TRTX_BOX_LTRB.  Greedy only: TRTX_NMS_ONESHOT is TRTX_ERR_UNSUPPORTED.  Both the
                            plugin-row and the fused / split tile sources */
};
enum {
    TRTX_NMS_GREEDY = 0,  /* CPU nms() semantics (the contract, SURVEY.md section 7 "Hard parts") */
    TRTX_NMS_ONESHOT = 1, /* nms_kernel semantics, yolov8/src/postprocess.cu:89-111 */
};

#define TRTX_NMS_MAX_ROWS 2048 /* rows per image the NMS kernel sorts on chip */

typedef struct trtx_nms_params {
    int32_t box_format;  /* TRTX_BOX_* */
    int32_t mode;        /* TRTX_NMS_* */
    float conf_thresh;   /* rows with !(conf > conf_thresh) are dropped (kConfThresh 0.5 / retinaface 0.1 rounded
                            so that the float compare equals the reference's double compare) */
    float nms_thresh;    /* kNmsThresh 0.45 / 0.4 */
    int32_t max_det;     /* K: rows of the compact output per image (kMaxNumOutputBbox) */
    int32_t class_aware; /* 1: only same-class rows interact (yolo); 0: single class (retinaface).  Class ids are
                            compared as floats, like the reference's std::map<float, ...> (-0.0 == +0.0; 2.0 and 2.5 are
                            two classes) and every row keeps its own class float; the order of NaN ids is unspecified. */
    int32_t tie_break_x0; /* 1: equal conf ordered by box[0] ascending (yolov8 cmp, postprocess.cpp:87-92); 0: none */
    int32_t extra_floats; /* floats copied verbatim from each source row into the output row after `keep`
                             (retinaface: 10 landmarks; yolo seg: 32 mask coefficients); 0 for plain det */
    int32_t extra_offset; /* offset (floats) of the first extra in the source row (retinaface 5, yolo seg 6) */
} trtx_nms_params;

/* Compact detection output: [batch, 1 + max_det*R] fp32, R = 7 + extra_floats:
 * count, (x0,x1,x2,x3,conf,cls,keep, extras...)*   (R = 7 is the layout of yolov8/include/types.h:18-19 +
 * postprocess.cu:64-71; box in the input's format).  Rows are ordered class asc then conf desc -- the
 * order of the reference's `res` vector (std::map iteration + std::sort).
 * GREEDY: only kept rows are written (keep=1), count = number kept.  ONESHOT: all rows above
 * conf_thresh, keep flag 0/1, count = rows.  Rows >= count are zero.
 * Rows entering NMS:
 *   trtx_nms_enqueue: every row i < min(count, max_rows) above conf_thresh, exactly like the reference's nms(), as long
 *     as max_rows <= TRTX_NMS_MAX_ROWS; with a larger max_rows (e.g. RetinaFace's 16800 priors) the TRTX_NMS_MAX_ROWS
 *     highest-confidence rows above conf_thresh enter (ties at the cut: lower row index first) -- the reference has no
 *     such cap, so results only differ when more than TRTX_NMS_MAX_ROWS rows of one image pass conf_thresh;
 *   fused / split calls: the first p->max_out candidates in ascending anchor order (= the rows the plugin buffer of
 *     trtx_yolo_decode_enqueue would hold), then the conf_thresh filter: both paths give identical results also when
 *     an image has more than max_out candidates (the reference's choice there is atomicAdd arrival order).
 *     p->max_out <= TRTX_NMS_MAX_ROWS or TRTX_ERR_UNSUPPORTED.
 * keep_index_dev (optional, may be NULL): [batch, max_det] int32 flat anchor id of each written row. */

/* NMS over a plugin-format buffer [batch, 1 + max_rows*det_floats] (drop-in for batch_nms()). */
TRTX_API size_t trtx_nms_workspace_size(const trtx_nms_params* p, int batch, int max_rows);
TRTX_API int trtx_nms_enqueue(const trtx_nms_params* p, int batch, const float* plugin_out_dev, int max_rows,
                              int det_floats, float* compact_out_dev, int32_t* keep_index_dev, void* workspace_dev,
                              size_t workspace_bytes, trtx_stream_t stream);

/* Fused decode + NMS: YoloLayer inputs -> compact detections, no plugin-format round trip. */
TRTX_API int trtx_yolo_decode_nms_enqueue(const trtx_yolo_params* p, const trtx_nms_params* q, int batch,
                                          const void* const* inputs_dev, float* compact_out_dev,
                                          int32_t* keep_index_dev, void* workspace_dev, size_t workspace_bytes,
                                          trtx_stream_t stream);

/* Split form of the fused call (same workspace, same stream order): scan = the HBM-bound streaming
 * kernel alone, then NMS over its tiles.  Used to time the scan kernel in isolation and to overlap the
 * scan of batch i+1 with the NMS of batch i on two streams. */
TRTX_API int trtx_yolo_scan_enqueue(const trtx_yolo_params* p, int batch, const void* const* inputs_dev,
                                    void* workspace_dev, size_t workspace_bytes, trtx_stream_t stream);
TRTX_API int trtx_yolo_nms_after_scan_enqueue(const trtx_yolo_params* p, const trtx_nms_params* q, int batch,
                                              const void* const* inputs_dev, float* compact_out_dev,
                                              int32_t* keep_index_dev, void* workspace_dev, size_t workspace_bytes,
                                              trtx_stream_t stream);

/* Multi-GPU gather of the compact detections over NVLink peer memory (SURVEY 8e: images shard by batch, the only exchange is
 * this gather).  One process per GPU on one NVSwitch node; every rank owns
 *   out   : [slots][world*batch][1 + max_det*R] fp32  -- the gathered detections (rank r's images at [r*batch, (r+1)*batch))
 *   flags : [world][slots] uint32, zero-initialised   -- flags[r][s] = how often rank r has published slot s
 *   ctrl  : [4] uint32, zero-initialised, local only  -- [1] scratch counter, [2] error (1 = a wait timed out)
 * allocated with trtx_peer_alloc (cudaMalloc + CUDA IPC handle) and mapped into the other ranks with trtx_peer_open, so
 * that out_dev[] / flags_dev[] hold, on every rank, the addresses of all ranks' buffers ([rank] = its own).  `slot` is chosen
 * by the caller per call (plain data: calls captured into CUDA graphs keep their slot).
 *   PUBLISH  trtx_gather_push_enqueue: gather_copy_kernel (one CTA per image) copies the live part [count, rows] of every image
 *            of a local compact output into `slot` of EVERY rank's `out` (lane-consecutive NVLink stores; no fence, no flag), then
 *            gather_publish_kernel (one warp) raises this rank's counter of the slot on every rank with relaxed system-scope
 *            stores: the kernel boundary between the two orders the rows before the counter, so no thread executes a system-scope
 *            fence.  Neither kernel waits for anybody.
 *            trtx_yolo_decode_nms_gather_enqueue publishes from inside nms_kernel instead (no extra launch; ONE system-scope
 *            fence by the last CTA; the NMS CTAs' 32 whole SMs stay occupied during the copy -- measured in DESIGN.md section 5).
 *   WAIT     trtx_gather_wait_enqueue (one warp, relaxed polls): returns on the stream once every rank's counter of `slot` has
 *            reached this rank's own, i.e. all ranks' rows of this round are in the local out[slot]; LATER work of the stream
 *            (kernels, copies) may read them.  Rows past an image's `count` are stale.  Gives up after ~2 s (ctrl[2] = 1) instead
 *            of hanging the GPU.
 * Reusing a slot overwrites it on every rank: a rank may publish into a slot again only after all ranks have finished
 * reading the previous round.  The pattern that guarantees it without further handshakes: 2*G slots used in halves; the G
 * publishes of a round go to one half, then the G waits, all on the streams of the round; the next round uses the other half.
 * (A rank cannot get two rounds ahead of a peer: its own waits need the peer's publishes of the round in between.)
 * Every rank must enqueue the same sequence.  world <= 8. */
typedef struct trtx_gather {
    int32_t world, rank, slots, slot;
    float* out_dev[8];
    uint32_t* flags_dev[8];
    uint32_t* ctrl_dev;
} trtx_gather;
TRTX_API int trtx_yolo_decode_nms_gather_enqueue(const trtx_yolo_params* p, const trtx_nms_params* q, int batch,
                                                 const void* const* inputs_dev, float* compact_out_dev,
                                                 int32_t* keep_index_dev, void* workspace_dev, size_t workspace_bytes,
                                                 const trtx_gather* gather, trtx_stream_t stream);
TRTX_API int trtx_gather_push_enqueue(const trtx_gather* gather, const float* compact_out_dev, int batch, int max_det,
                                      int extra_floats, trtx_stream_t stream);
TRTX_API int trtx_gather_wait_enqueue(const trtx_gather* gather, trtx_stream_t stream);
/* The same for n <= 8 consecutive slots slot .. slot+n-1 in ONE launch each (a round of n steps: one push kernel publishing
 * the n local outputs compact_outs_dev[0..n) -- a HOST array of device pointers -- with a single expensive release, one wait
 * kernel for the n slots; world * n <= 64).  A publish reads its sources when it runs: keep them unchanged until then (bench.py
 * double-buffers the compact outputs so that the next NMS never has to wait for the publish of the previous one). */
TRTX_API int trtx_gather_push_many_enqueue(const trtx_gather* gather, const float* const* compact_outs_dev, int n, int batch,
                                           int max_det, int extra_floats, trtx_stream_t stream);
TRTX_API int trtx_gather_wait_many_enqueue(const trtx_gather* gather, int nslots, trtx_stream_t stream);
/* Peer-mappable device memory (zero-initialised) + its 64-byte CUDA IPC handle; open / close a peer's handle; free. */
TRTX_API int trtx_peer_alloc(size_t bytes, void** dev_ptr, unsigned char handle[64]);
TRTX_API int trtx_peer_open(const unsigned char handle[64], void** dev_ptr);
TRTX_API int trtx_peer_close(void* dev_ptr);
TRTX_API int trtx_peer_free(void* dev_ptr);

/* =====================================================================================
 * 3. Decode_TRT (RetinaFace) -- replaces retinaface/decode.cu:110-199
 *    inputs_dev[l] : [batch, 32, (in_h/s)*(in_w/s)] fp32 (or fp16: in_dtype), s = 8,16,32, channels [bbox 2x4 | cls 2x2 | lmk 2x10]
 *    output_dev    : [batch, 1 + total_priors*15] fp32, rows x1,y1,x2,y2,conf,lmk[10]
 *    (TRTX_RETINA_ANTICOV: [batch, 38, g] inputs, [batch, 1 + total_priors*16] output)
 * ===================================================================================== */
enum {
    TRTX_RETINA_FACE = 0,    /* retinaface/decode.cu */
    TRTX_RETINA_ANTICOV = 1, /* retinafaceAntiCov/decode.cu:110-172 (SURVEY 8f rank 4): inputs [batch, 38, g] =
                                [cls 4 | bbox 2x4 | lmk 2x10 | type 6], all soft-maxed by the network; rows of 16 floats
                                x1,y1,x2,y2,conf,lmk[10],mask_conf (decode.h:13-18); gate is the literal `conf < 0.5`;
                                the reference decodes batch 1 only, this build every image */
};
typedef struct trtx_retina_params {
    int32_t in_h, in_w; /* decodeplugin::INPUT_H / INPUT_W (compile-time 480x640 in decode.h:16-17) */
    float gate;         /* 0.02 (decode.cu:131); compared as `conf <= gate`.  Unused by TRTX_RETINA_ANTICOV */
    int32_t variant;    /* TRTX_RETINA_FACE (0, what a zeroed struct selects) | TRTX_RETINA_ANTICOV */
    int32_t in_dtype;   /* element type of all three inputs: TRTX_F32 (0, what a zeroed struct selects; the reference's only
                           mode) | TRTX_F16.  A half is widened to float (exact) where the reference reads a float; the
                           arithmetic and the fp32 output rows are the same code, so the rows are those of the fp32 call on
                           the widened inputs */
} trtx_retina_params;

TRTX_API int trtx_retina_total_priors(const trtx_retina_params* p);
TRTX_API size_t trtx_retina_workspace_size(const trtx_retina_params* p, int batch);
/* TRTX_ERR_INVALID, before the first launch and with nothing written: a null argument, in_h or in_w < 32, an unknown variant
 * or in_dtype, an input pointer that is not a multiple of its element size (4 / 2 bytes), an output pointer that is not a
 * multiple of 4.  Inputs that are 16-byte (fp32) / 8-byte (fp16) aligned with grids of a multiple of 4 cells are read four
 * cells per load, any other one cell per load; the rows do not depend on which, and no input size is refused for either:
 * every in_h, in_w >= 32 decodes, with floor grids (in_h/s) x (in_w/s) per axis.  The priors are placed on the level's fixed
 * stride s = 8, 16, 32 (TRTX_RETINA_ANTICOV: 7.5 + x*s, 7.5 + y*s; not in_w / (in_w/s), which differs from s when s does not
 * divide in_w), as the reference's forwardGpu passes it. */
TRTX_API int trtx_retina_decode_enqueue(const trtx_retina_params* p, int batch, const void* const* inputs_dev,
                                        float* output_dev, void* workspace_dev, size_t workspace_bytes,
                                        trtx_stream_t stream);

/* =====================================================================================
 * 4. Faster R-CNN plugins -- same "null workspace returns the size" idiom as the reference
 *    free functions (rcnn/RpnNms.cu:63-80): call with workspace_dev == NULL to get bytes.
 *    All images of the batch are processed in one launch (the reference loops on the host).
 *    Outputs are the first entries of a stable descending sort of the scores: equal scores (-0.0 and +0.0 included)
 *    keep ascending input index.  Limits, beyond which a call returns -TRTX_ERR_UNSUPPORTED and writes nothing:
 *    num_anchors <= 64 and top_n <= 8192 (rpnDecode), pre_nms_topk <= 8192 (rpnNms), num_boxes <= 8192
 *    (predictorDecode), count <= 4096 (batchedNms).
 * ===================================================================================== */
/* rpnDecode, rcnn/RpnDecode.cu:27-143.  inputs: scores [B,A,H,W], deltas [B,A*4,H,W];
 * outputs: scores [B,top_n], boxes [B,top_n,4].  anchors_host: A*4 floats (host memory, copied
 * into the launch parameters -- no H2D copy per enqueue). */
TRTX_API int64_t trtx_rpn_decode(int batch, const float* scores_dev, const float* deltas_dev, float* out_scores_dev,
                                 float* out_boxes_dev, int height, int width, int image_height, int image_width,
                                 float stride, const float* anchors_host, int num_anchors, int top_n,
                                 void* workspace_dev, size_t workspace_bytes, trtx_stream_t stream);
/* rpnNms, rcnn/RpnNms.cu:59-121.  inputs: scores [B,pre], boxes [B,pre,4]; output boxes [B,post,4]. */
TRTX_API int64_t trtx_rpn_nms(int batch, const float* scores_dev, const float* boxes_dev, float* out_boxes_dev,
                              int pre_nms_topk, int post_nms_topk, float nms_thresh, void* workspace_dev,
                              size_t workspace_bytes, trtx_stream_t stream);
/* predictorDecode, rcnn/PredictorDecode.cu:24-110.  inputs: scores [B,N,C], deltas [B,N*C,4],
 * proposals [B,N,4]; outputs scores/boxes/classes [B,N,...]. */
TRTX_API int64_t trtx_predictor_decode(int batch, const float* scores_dev, const float* deltas_dev,
                                       const float* proposals_dev, float* out_scores_dev, float* out_boxes_dev,
                                       float* out_classes_dev, int num_boxes, int num_classes, int image_height,
                                       int image_width, const float* bbox_reg_weights_host, void* workspace_dev,
                                       size_t workspace_bytes, trtx_stream_t stream);
/* rpnDecode and predictorDecode with scores_dev AND deltas_dev of element type in_dtype: TRTX_F32 (= the untyped call, byte for
 * byte) or TRTX_F16, so that an FP16 engine hands both plugins the heads' half tensors without a reformat copy.  Every output
 * stays fp32 in both modes (scores, boxes up to the image size -- a half holds 1067 to 0.5 px only -- and classes: they feed
 * rpnNms, batchedNms and trtx_rcnn_postprocess*), and so do proposals_dev (rpnNms's output).  The half result is DEFINED as
 * the fp32 call on the widened tensors, bit for bit:
 *     trtx_*_decode_typed(TRTX_F16, h, ...) == trtx_*_decode(float(h), ...)
 * where float() is the device's exact widening; the order is the fp32 order (stable descending, -0.0 == +0.0, a NaN where its
 * widened value ranks).  The half select ranks 16-bit keys (two radix passes over 2-byte loads instead of four over 4-byte
 * ones).  The workspace query, limits and return codes are those of the untyped calls; the size does not depend on the type.
 * -TRTX_ERR_INVALID, before any launch and with nothing written: in_dtype not TRTX_F32 / TRTX_F16 (workspace query
 * included); in the half mode a scores_dev or deltas_dev not a multiple of 2 bytes, in predictorDecode a deltas_dev not a
 * multiple of 8 bytes (a candidate's 4 deltas are one load).  The fp32 mode checks what the untyped call checks, no more. */
TRTX_API int64_t trtx_rpn_decode_typed(int in_dtype, int batch, const void* scores_dev, const void* deltas_dev,
                                       float* out_scores_dev, float* out_boxes_dev, int height, int width, int image_height,
                                       int image_width, float stride, const float* anchors_host, int num_anchors, int top_n,
                                       void* workspace_dev, size_t workspace_bytes, trtx_stream_t stream);
TRTX_API int64_t trtx_predictor_decode_typed(int in_dtype, int batch, const void* scores_dev, const void* deltas_dev,
                                             const float* proposals_dev, float* out_scores_dev, float* out_boxes_dev,
                                             float* out_classes_dev, int num_boxes, int num_classes, int image_height,
                                             int image_width, const float* bbox_reg_weights_host, void* workspace_dev,
                                             size_t workspace_bytes, trtx_stream_t stream);
/* batchedNms, rcnn/BatchedNms.cu:92-162.  nms_method 0 hard / 1 soft-linear / 2 soft-gaussian. */
TRTX_API int64_t trtx_batched_nms(int nms_method, int batch, const float* scores_dev, const float* boxes_dev,
                                  const float* classes_dev, float* out_scores_dev, float* out_boxes_dev,
                                  float* out_classes_dev, int count, int detections_per_im, float nms_thresh,
                                  void* workspace_dev, size_t workspace_bytes, trtx_stream_t stream);

/* =====================================================================================
 * 5. Pre-process -- batched letterbox warp + BGR->RGB + /255 + HWC->CHW (+fp16)
 *    replaces warpaffine_kernel / cuda_preprocess / cuda_batch_preprocess,
 *    yolov8/src/preprocess.cu:7-127 (one launch + one stream sync PER IMAGE there).
 * ===================================================================================== */
typedef struct trtx_image_desc {
    const uint8_t* data_dev; /* u8 HWC BGR, row pitch = pitch bytes */
    int32_t width, height;
    int32_t pitch; /* bytes per row, >= 3*width */
    int32_t reserved;
} trtx_image_desc;

/* images_host: array of `batch` descriptors in HOST memory (copied into launch parameters);
 * dst_dev: [batch, 3, dst_h, dst_w] fp32 or fp16 (out_dtype TRTX_F32 | TRTX_F16). One launch per kernel and per
 * <= 64 scale-1 images / <= 128 other images.  Every argument is checked before the first launch (a rejected call writes
 * nothing): TRTX_ERR_INVALID for a null pointer, batch / dst sizes <= 0, an unknown out_dtype, pitch < 3 * width or a
 * dst_dev that is not aligned to its element size (4 bytes for TRTX_F32, 2 for TRTX_F16). */
TRTX_API int trtx_preprocess_batch_enqueue(const trtx_image_desc* images_host, int batch, void* dst_dev, int dst_w,
                                           int dst_h, int out_dtype, trtx_stream_t stream);
/* The band pre-processes: trtx_rcnn_, trtx_cls_, trtx_yolop_, trtx_detr_, trtx_ufld_, trtx_refinedet_, trtx_cubic_ and
 * trtx_linear_preprocess_enqueue.  Each resizes a batch of frames into the rectangle its model's driver gives each frame on
 * the engine input, by OpenCV 4.x's own 8-bit INTER_LINEAR (INTER_CUBIC for trtx_cubic_preprocess_enqueue), bit for bit,
 * and stores every byte as its model's value.  They share one contract:
 *   images_host: `batch` u8 HWC BGR descriptors in HOST memory (copied into launch parameters; any pitch and base alignment,
 *     mixed sizes allowed); dst_dev: the engine input, fp32.
 *   Everything is checked before the first launch, so a rejected call writes nothing, in two passes:
 *     1. TRTX_ERR_INVALID for a null pointer, batch / net sizes <= 0, pitch < 3 * width, an unknown variant or a dst_dev that
 *        is not 4-byte aligned;
 *     2. per frame, what the entry's rectangle rejects (TRTX_ERR_UNSUPPORTED where the reference's cv::resize throws, e.g. an
 *        empty rectangle for a 1 x 5000 frame); then TRTX_ERR_UNSUPPORTED where the staged source rows of a launch's widest
 *        rectangle exceed the kernel's shared memory: rectangles up to 4 840 pixels wide for trtx_rcnn_preprocess_enqueue,
 *        4 757 for the other bilinear entries and, for trtx_cubic_preprocess_enqueue, 1 189 at any scale, 2 378 when enlarging.
 *     So a call that both passes reject is TRTX_ERR_INVALID, whichever frame comes first.
 *   One launch per <= 64 frames, no workspace; can be captured in a CUDA graph. */

/* The reference's d2s matrix (preprocess.cu:98-110): scale, centre, cv::invertAffineTransform. */
TRTX_API void trtx_letterbox_matrix(int src_w, int src_h, int dst_w, int dst_h, float d2s[6]);
/* get_rect (yolov8/src/postprocess.cpp:6-36, yolov5/src/postprocess.cpp:4-29): maps a detection box from network-input
 * pixels back to the original image: rect = {x, y, width, height} as cv::Rect.  variant TRTX_YOLO_V8: box l,t,r,b,
 * result clamped to the image; TRTX_YOLO_V5: box cx,cy,w,h.
 * TRTX_YOLO_V3: the get_rect of yolov3, yolov4, scaled-yolov4 and yolov3-tiny (yolov3/yolov3.cpp:30-52, yolov4/yolov4.cpp:55-77,
 *   scaled-yolov4/common.hpp:36-58, yolov3-tiny/yolov3-tiny.cpp:62-84): box cx,cy,w,h; r_w = net_w / (img_w * 1.0) stored to
 *   float (r_h likewise), l = (int)(cx - w / 2.f) (minus the float pad (net_h - r_w * img_h) / 2 on the padded axis), then
 *   l = (int)((float)l / r_w); every int store truncates toward zero; no clamp; rect = {l, t, r - l, b - t}.
 * TRTX_RECT_YOLOV3_SPP: yolov3-spp's get_rect (yolov3-spp/yolov3-spp.cpp:58-75) with MAX_INPUT_SIZE = net_w = net_h: the
 *   letterbox of trtx_yolov3spp_letterbox, l = (int)(cx - w / 2.f - dw / 2) with dw / 2 an int division, then l /= ra
 *   (truncated); no clamp.
 * A box whose get_rect is undefined in the reference -- a NaN, an infinity or a float outside the int range converted to int,
 * or an r - l that overflows -- gets {0, 0, 0, 0} (TRTX_YOLO_V8 / V5: a non-finite box or rescaled corners outside the int
 * range).  TRTX_ERR_INVALID for a null pointer, a size <= 0, another variant, or net_w != net_h with TRTX_RECT_YOLOV3_SPP.
 * Host function (no device work). */
enum { TRTX_RECT_YOLOV3_SPP = 16 /* a rectangle variant only: no YoloLayer decodes with it */ };
TRTX_API int trtx_get_rect(int variant, int net_w, int net_h, int img_w, int img_h, const float bbox[4], int rect[4]);

/* get_rect_adapt_landmark (yolov8/src/postprocess.cpp:38-69): like get_rect for the pose models -- the box (l,t,r,b) becomes
 * a cv::Rect in the original image (trtx_get_rect's V8 result, {0, 0, 0, 0} where that is undefined) and the num_kpts
 * keypoints (x, y, conf triplets, `lmk`) are mapped IN PLACE, the confidences untouched.  Host function; the device form is
 * trtx_yolo_pose_obb_postprocess_enqueue. */
TRTX_API int trtx_get_rect_adapt_landmark(int net_w, int net_h, int img_w, int img_h, const float bbox[4], float* lmk,
                                          int num_kpts, int rect[4]);
/* get_corner (yolov8/src/postprocess.cpp:395-472 with net 640; yolo11/src/postprocess.cpp:425-502, whose get_rect_obb is
 * get_rect with net 1024): the four corners of an oriented box (cx, cy, w, h in network pixels, angle in radians) in the
 * original image, corners = {x0, y0, x1, y1, x2, y2, x3, y3} in get_corner's order, each clamped to the image.  A corner
 * whose float -> int conversion is undefined in the reference (NaN, out of range) is 0, as the compiled reference gives on
 * x86-64 after its clamp; a box whose get_rect is undefined gets four (0, 0) corners.  The reference's debug prints are
 * not reproduced.  Host function; the device form is trtx_yolo_pose_obb_postprocess_enqueue. */
TRTX_API int trtx_get_corner(int net_w, int net_h, int img_w, int img_h, const float cxcywh[4], float angle, int corners[8]);
/* RetinaFace's own get_rect_adapt_landmark (retinaface/common.hpp:65-89; retinafaceAntiCov's copy is the same statements with
 * input_w = input_h = 640): 5 landmarks as x, y pairs, modified in place; the box corners are truncated to int and not
 * clamped; rect = {x, y, w, h} in the original image.  Defined where the reference is not, as the compiled x86-64 reference
 * behaves: a corner that is NaN, infinite or outside [-2^31, 2^31) converts to INT_MIN, and w = r - l, h = b - t wrap
 * modulo 2^32.  Host function; the device form is trtx_retina_postprocess_enqueue. */
TRTX_API int trtx_retina_get_rect_adapt_landmark(int input_w, int input_h, int img_w, int img_h, const float bbox[4], float lmk[10],
                                                 int rect[4]);
/* process_decode_ptr_host (yolov8/src/postprocess.cpp:131-147): rows of a compact buffer [1 + K*bbox_element] (the output
 * of the ONESHOT mode / cuda_decode+cuda_nms) whose keep flag is 1 -> 6-float rows l,t,r,b,conf,cls.  Returns the number
 * of rows written (<= count), or a negative TRTX_ERR_*.  Host function on HOST memory. */
TRTX_API int trtx_process_decode_ptr_host(const float* decode_ptr_host, int bbox_element, int count, float* rows_out);
/* process_decode_ptr_host_obb (:273-290): rows_out gets 7 floats per kept row (l/cx, t/cy, r/w, b/h, conf, class, angle = column 7 of
 * the 8-float rows of the oriented-box decode); bbox_element >= 8. */
TRTX_API int trtx_process_decode_ptr_host_obb(const float* decode_ptr_host, int bbox_element, int count, float* rows_out);
/* scale_mask (yolov8/src/postprocess.cpp:207-226): the letterboxed region of a network-size mask, resized (cv::resize,
 * bilinear) to the original image.  trtx_scale_mask_rect = the crop rectangle {x, y, w, h} (host);
 * trtx_scale_mask_enqueue: masks_dev [n, net_h, net_w] fp32 -> out_dev [n, img_h, img_w] fp32, one launch, HBM-write-bound. */
TRTX_API int trtx_scale_mask_rect(int net_w, int net_h, int img_w, int img_h, int rect[4]);
TRTX_API int trtx_scale_mask_enqueue(const float* masks_dev, int n, int net_w, int net_h, int img_w, int img_h, float* out_dev,
                                     trtx_stream_t stream);

/* RoIAlign and MaskRcnnInference (SURVEY 8f rank 2): replace roiAlign (rcnn/RoiAlign.cu:150-183) and maskRcnnInference
 * (rcnn/MaskRcnnInference.cu:35-63); same argument meaning, whole batch in one launch, no cudaDeviceSynchronize().
 * rois_dev [batch, num_proposals, 4] x1,y1,x2,y2; features_dev [batch, out_channels, feature_h, feature_w];
 * out_dev [batch, num_proposals, out_channels, pooler_resolution, pooler_resolution].  sampling_ratio <= 0: adaptive.
 * The library picks the kernel from the shape; both are bit-identical to the reference's roiAlign.  The reference's
 * configuration class (pooler_resolution 14, out_channels % 4 == 0, feature_h * feature_w <= 4096) stages each proposal's
 * feature-map window in shared memory and takes the bilinear taps from there; any other shape takes every tap from global
 * memory.
 * Adaptive sampling (sampling_ratio <= 0) takes ceil(side / pooler_resolution) samples per bin and axis, as the reference
 * does: a proposal side of s feature cells costs about (s / pooler_resolution)^2 samples per bin, so a huge proposal does
 * that much work, and one with an infinite side an unbounded amount (its grid saturates at 2^31 - 1 per axis).  Pass finite
 * proposals of bounded size, or a fixed sampling_ratio. */
TRTX_API int trtx_roi_align(int batch, const float* rois_dev, const float* features_dev, float* out_dev, int pooler_resolution,
                            float spatial_scale, int sampling_ratio, int num_proposals, int out_channels, int feature_h,
                            int feature_w, trtx_stream_t stream);
/* The same with the element type of features_dev AND out_dev chosen by dtype: TRTX_F32 (= trtx_roi_align, byte for byte) or
 * TRTX_F16, so that an FP16 engine hands the plugin its half feature map and takes half bins without a reformat copy on
 * either side.  rois_dev stays fp32 in both modes (a half holds a coordinate up to 1067 to 0.5 px only).
 * The half result is DEFINED: every tap is widened to float (exact), sampled and summed exactly as in the fp32 mode, and
 * only the finished bin is rounded, once, to nearest-even (overflow to +-inf, NaN stays NaN):
 *     out = half(trtx_roi_align(float(features))), bit for bit.
 * In the half mode the shared-memory window kernel takes out_channels % 8 == 0 (pooler 14, feature_h * feature_w <= 4096 as
 * before); other shapes take every tap from global memory.
 * TRTX_ERR_INVALID, before any launch and with nothing written: dtype not TRTX_F32 / TRTX_F16; a null pointer or a
 * non-positive size; rois_dev not a multiple of 16 bytes (a proposal is one 16-byte load); features_dev or out_dev not a
 * multiple of the element size (4 / 2 bytes). */
TRTX_API int trtx_roi_align_typed(int dtype, int batch, const float* rois_dev, const void* features_dev, void* out_dev,
                                  int pooler_resolution, float spatial_scale, int sampling_ratio, int num_proposals,
                                  int out_channels, int feature_h, int feature_w, trtx_stream_t stream);
/* indices_dev [batch, detections_per_im] class index as float; masks_dev [batch, detections_per_im, num_classes, S, S];
 * out_dev [batch, detections_per_im, S, S] = sigmoid of the predicted class' mask (rows with an index outside
 * [0, num_classes) are left untouched, as in the reference). */
TRTX_API int trtx_mask_rcnn_inference(int batch, const float* indices_dev, const float* masks_dev, float* out_dev,
                                      int detections_per_im, int output_size, int num_classes, trtx_stream_t stream);
/* The same with masks_dev of element type in_dtype: TRTX_F32 (= trtx_mask_rcnn_inference) or TRTX_F16 (the mask head of an
 * FP16 engine).  A half is widened to float (exact) before the sigmoid; indices_dev and out_dev are fp32 in both modes
 * (out_dev feeds trtx_rcnn_postprocess*).  TRTX_ERR_INVALID, before the launch and with nothing written: in_dtype not
 * TRTX_F32 / TRTX_F16; a null pointer or a non-positive size; indices_dev or out_dev not a multiple of 4 bytes, masks_dev
 * not a multiple of its element size. */
TRTX_API int trtx_mask_rcnn_inference_typed(int in_dtype, int batch, const float* indices_dev, const void* masks_dev,
                                            float* out_dev, int detections_per_im, int output_size, int num_classes,
                                            trtx_stream_t stream);

/* The INT8 calibrator's host pre-process (SURVEY 8f rank 4): Int8EntropyCalibrator2::getBatch, yolov8/src/calibrator.cpp:33-52
 * = preprocess_img (yolov8/include/utils.h:6-26: cv::resize INTER_LINEAR of the 8-bit image into the letterbox rectangle, 128-grey
 * canvas) + cv::dnn::blobFromImages(1 / 255.0, swapRB).  HOST code, like the reference's (calibration is not in the inference loop):
 * bgr = 8-bit BGR rows of src_pitch bytes; out_chw = [3, net_h, net_w] fp32 RGB planes, ready for the cudaMemcpy of :48.  The
 * OpenCV arithmetic is restated (fixed-point bilinear resize, float scale) and pinned bit for bit against cv2 4.13.
 * trtx_calib_letterbox_rect: the rectangle {x, y, w, h} the resized image occupies. */
TRTX_API int trtx_calib_letterbox_rect(int src_w, int src_h, int net_w, int net_h, int rect[4]);
TRTX_API int trtx_calib_letterbox_host(const uint8_t* bgr, int src_w, int src_h, size_t src_pitch, int net_w, int net_h, float* out_chw);

/* =====================================================================================
 * 6. Instance masks of the segmentation models (SURVEY 8f rank 1)
 *    replaces the HOST function process_mask(), yolov8/yolov8_seg.cpp:17-60 and
 *    yolov5/src/postprocess.cpp:94-125: sigmoid(coeffs . prototypes) inside the detection's
 *    down-scaled rectangle, then cv::resize (bilinear) to the network input size.
 * ===================================================================================== */
typedef struct trtx_mask_params {
    int32_t variant;      /* TRTX_YOLO_V8: rect from (x, y, w, h) with int() truncation and clamping (yolov8_seg.cpp:17-34);
                             TRTX_YOLO_V5: rect from (cx, cy, w, h) with round() (yolov5 postprocess.cpp:94-104) */
    int32_t net_w, net_h; /* kInputW, kInputH: size of the masks written */
    int32_t mask_w, mask_h; /* prototype resolution; must be net/4 like the reference */
    int32_t num_coeffs;   /* 32 */
    int32_t row_floats;   /* floats per detection row of `dets_dev` */
    int32_t coeff_offset; /* first mask coefficient inside a row (box = floats 0..3) */
    int32_t max_masks;    /* masks written per image: the first min(count, max_masks) rows */
} trtx_mask_params;

/* proto_dev: [batch, num_coeffs, mask_h, mask_w] fp32 (the engine's "proto" output);
 * dets_dev : [batch, 1 + max_rows*row_floats] fp32 = count, rows (e.g. the compact NMS output with
 *            extra_floats = 32, extra_offset = 6: row_floats = 39, coeff_offset = 7);
 * masks_dev: [batch, max_masks, net_h, net_w] fp32; slots >= count are left untouched.  One launch.
 * A box for which one of get_downscale_rect's float -> int conversions is undefined in the reference (a non-finite box, or
 * a corner or size outside the int range in mask cells) gets an all-zero mask, as get_rect gives it {0, 0, 0, 0}.
 * TRTX_ERR_UNSUPPORTED for net != 4 * mask, or batch * max_masks > 65535 (nothing is launched). */
TRTX_API int trtx_process_mask_enqueue(const trtx_mask_params* p, int batch, const float* proto_dev, const float* dets_dev,
                                       int max_rows, float* masks_dev, trtx_stream_t stream);

/* One original frame of a per-frame post-process call (trtx_yolo_seg_postprocess_enqueue,
 * trtx_rcnn_postprocess_frames_enqueue): its size and its u8 canvases.  Passed in HOST memory, copied into launch parameters. */
typedef struct trtx_frame {
    int32_t img_w, img_h; /* the original frame (the reference's img / w_ori, h_ori) */
    uint8_t* masks_dev;   /* [max_masks, img_h, pitch] u8 canvases of this frame, or NULL (rows only) */
    int32_t pitch;        /* bytes per canvas row, >= img_w (any value, any base alignment) */
    int32_t reserved;
} trtx_frame;
typedef trtx_frame trtx_seg_image;  /* earlier names of trtx_frame, same type */
typedef trtx_frame trtx_rcnn_image;

/* The per-frame post-processes: trtx_yolo_seg_, trtx_yolo_pose_obb_, trtx_retina_, trtx_rcnn_ (frames), trtx_yolop_,
 * trtx_detr_, trtx_ufld_, trtx_refinedet_, trtx_yolo_topk_ and trtx_pyrunner_postprocess_enqueue, trtx_rcnn_contours_enqueue
 * and trtx_centernet_decode_enqueue.  Each maps its model's rows, masks or maps back to every original frame of a batch, and
 * they share one contract:
 *   the frames: frame_wh_host, `batch` (img_w, img_h) pairs, or images_host / frames_host, `batch` trtx_frame, in HOST
 *     memory, copied into launch parameters; sizes may differ in a call.
 *   Everything is checked before the first launch, so a rejected call writes nothing, in this order:
 *     1. TRTX_ERR_INVALID for a null pointer, a parameter outside its range, a frame size <= 0 or a bad descriptor, and a
 *        misaligned workspace;
 *     2. TRTX_ERR_UNSUPPORTED for a parameter or a frame past the entry's limits;
 *     3. TRTX_ERR_WORKSPACE for a workspace smaller than the entry's size function returns.
 *     So a call that fails two ways returns the first of these, whichever frame fails first.
 *   One launch of each kernel per <= 64 frames; can be captured in a CUDA graph.
 * Each entry's doc below lists its own cases. */

/* The segmentation models' last host stage on the device: process_mask + scale_mask + draw_mask_bbox's mask selection
 * (yolov8/src/postprocess.cpp:228-248, yolov5/src/postprocess.cpp:148-167), for a batch of original frames of any sizes. */

/* p: as for trtx_process_mask_enqueue (row_floats >= 6; with every masks_dev NULL only variant, net_w, net_h and row_floats
 *   are read, and variant may also be TRTX_YOLO_V3 or TRTX_RECT_YOLOV3_SPP: the rows of yolov3 / yolov4 / scaled-yolov4 /
 *   yolov3-tiny and yolov3-spp, whose models have no masks; with canvases those two are TRTX_ERR_INVALID).
 * dets_dev [B, 1 + max_rows*row_floats]: count, rows with the box at floats 0..3 in the variant's format, conf at 4, class
 *   at 5 (the compact NMS output with extra_floats = 32: row_floats 39, coeff_offset 7; plugin rows: 90 / 6).
 * rows_dev [B, 1 + max_rows*6]: n = min(count, max_rows), then per row i < n (x, y, w, h, conf, class) with x, y, w, h =
 *   get_rect(img, bbox) (trtx_get_rect: V8 clamped to the image, V5 not), rows past n zeroed.  A box whose get_rect is
 *   undefined in the reference (non-finite, or corners outside the int range) gets {0, 0, 0, 0}.
 * Canvas k < min(count, max_masks, max_rows) of image b: 255 where (x, y) lies in get_rect(img, bbox_k) clipped to the
 *   image and !(S(y, x) <= 0.5) -- draw_mask_bbox's `if (val <= 0.5) continue;`, so a NaN S is kept -- else 0, with
 *   S = scale_mask(M) (crop trtx_scale_mask_rect, bilinear to img_w x img_h) and M = process_mask's net_w x net_h mask.
 *   Bit-identical to thresholding trtx_process_mask_enqueue -> trtx_scale_mask_enqueue.  Canvases at or past that count are
 *   left untouched.
 * proto_dev [B, num_coeffs, mask_h, mask_w] may be NULL only when every masks_dev is NULL; NULL and non-NULL masks_dev in one
 * call is TRTX_ERR_INVALID.  A per-frame post-process: TRTX_ERR_INVALID for batch / max_rows <= 0, pitch < img_w;
 * TRTX_ERR_UNSUPPORTED for an image whose scale_mask crop is empty (e.g. 1 x 5000: the reference's cv::resize throws), and
 * for nets whose canvas launch would need more than 226 KB of shared memory (227 KB less a 1 KB margin for the kernel's
 * static arrays; square nets above 2408^2 with a frame of a few pixels).  Two kernels, no workspace. */
TRTX_API int trtx_yolo_seg_postprocess_enqueue(const trtx_mask_params* p, const trtx_frame* images_host, int batch,
                                               const float* proto_dev, const float* dets_dev, int max_rows,
                                               float* rows_dev, trtx_stream_t stream);

/* Host only, no device work: the shared memory the canvas launches of trtx_yolo_seg_postprocess_enqueue would use for these
 * frames (with canvases; masks_dev is not read), so a caller can check a set of frame sizes before enqueueing.  caps =
 * {M rows, low-resolution rows, M columns, low-resolution columns, dynamic shared-memory bytes}, each the largest over the
 * call's launches of 64 frames.  Returns what the enqueue would return for this geometry: TRTX_OK, TRTX_ERR_UNSUPPORTED for
 * an empty scale_mask crop or caps above 226 KB (caps then hold the launches sized so far), TRTX_ERR_INVALID for null
 * pointers or sizes <= 0. */
TRTX_API int trtx_yolo_seg_launch_caps(const trtx_mask_params* p, const trtx_frame* images_host, int batch, int32_t caps[5]);

/* The pose and oriented-box models' last host stage on the device: draw_bbox_keypoints_line's get_rect_adapt_landmark
 * (yolov8/src/postprocess.cpp:173-205) and draw_bbox_obb's get_corner (:474-507; yolo11/src/postprocess.cpp:504-537), for a
 * batch of original frames of any sizes.  The drawing itself stays with the caller. */
enum {
    TRTX_TASK_POSE = 1,         /* keypoints: rectangle + num_kpts (x, y, conf) mapped to the frame */
    TRTX_TASK_OBB = 2,          /* oriented boxes: four corners in the frame */
    TRTX_TASK_OBB_NMS_FREE = 3, /* the same corners from yolo26-obb's NMS-free plugin rows, which have no keep column */
};
typedef struct trtx_pose_obb_params {
    int32_t task;         /* TRTX_TASK_* */
    int32_t net_w, net_h; /* network input: kInputW / kInputH (640), or kObbInputW / kObbInputH (1024) of yolo11 / yolo26-obb */
    int32_t row_floats;   /* floats per row of dets_dev, >= 7 (box4, conf, class, keep, extras...) */
    int32_t extra_offset; /* POSE: first keypoint float in a row; OBB: the angle (radians); OBB_NMS_FREE: the angle,
                             which ends the row (row_floats - 1) */
    int32_t num_kpts;     /* POSE: keypoints per row, 0..64 (kNumberOfPoints = 17); OBB, OBB_NMS_FREE: not read */
} trtx_pose_obb_params;

/* dets_dev [B, 1 + max_rows*row_floats]: count, then rows (box4, conf, class, keep, extras...) -- the compact NMS output:
 *   pose: trtx_nms_enqueue(det_floats 90, extra_floats 51, extra_offset 38): row_floats 58, extra_offset 7, box l, t, r, b;
 *   OBB : batch_nms_obb (TRTX_BOX_OBB, greedy or one-shot): row_floats 8, extra_offset 7, box cx, cy, w, h.
 *   Of the first min(count, max_rows) rows only those with (int)keep == 1 are used (process_decode_ptr_host(_obb)): every
 *   greedy row, the kept rows of a one-shot output.
 *   OBB_NMS_FREE: the output of YoloLayerPlugin26 with is_obb (TRTX_YOLO_V26, det_floats 90): row_floats 90,
 *   extra_offset 89, box cx, cy, w, h; every one of the first min(count, max_rows) rows is used (yolo26's
 *   batch_decode_obb, yolo26/src/postprocess.cpp:310-326).
 * rows_dev [B, 1 + max_rows*F]: n kept rows in input order, then zeros up to max_rows:
 *   pose, F = 6 + 3*num_kpts: (x, y, w, h, conf, class, kx, ky, kc, ...) = trtx_get_rect_adapt_landmark;
 *   OBB and OBB_NMS_FREE, F = 10: (x0, y0, x1, y1, x2, y2, x3, y3, conf, class) = trtx_get_corner.
 * Bit-identical to those host functions (the device's double cos / sin are not correctly rounded, see trtx_get_corner).
 * A per-frame post-process: TRTX_ERR_INVALID for batch / max_rows <= 0, an unknown task, row_floats < 7 or extras outside
 * the row, num_kpts outside 0..64, an OBB_NMS_FREE angle that is not the row's last float.  One CTA per frame, no atomics
 * (deterministic), no workspace. */
TRTX_API int trtx_yolo_pose_obb_postprocess_enqueue(const trtx_pose_obb_params* p, const int32_t* frame_wh_host, int batch,
                                                    const float* dets_dev, int max_rows, float* rows_dev,
                                                    trtx_stream_t stream);

/* RetinaFace's last host stage on the device: the loop of retinaface/retina_r50.cpp:373-388 (CONF_THRESH, then
 * get_rect_adapt_landmark) and of retinafaceAntiCov/retinafaceAntiCov.cpp:540-552 (no threshold), for a batch of frames of
 * any sizes.  The drawing stays with the caller. */
typedef struct trtx_face_post_params {
    int32_t variant;    /* TRTX_RETINA_FACE: 15-float output rows | TRTX_RETINA_ANTICOV: 16 (+ mask_confidence) */
    int32_t in_w, in_h; /* decodeplugin::INPUT_W / INPUT_H (640x480 compiled into retinaface, 640x640 in AntiCov / config 3) */
    int32_t row_floats; /* floats per input row: 17 (compact NMS rows, extra_floats 10) / 18 (AntiCov, extra_floats 11) */
    int32_t lmk_offset; /* first landmark float of a row: 7; AntiCov's mask_confidence follows the 10 landmarks */
    float conf_thresh;  /* a row is skipped when conf < conf_thresh (retina_r50.cpp:381); -INFINITY = no filter (AntiCov).
                           For the reference's double threshold T, pass the smallest float >= T: a float c satisfies
                           c < T exactly when c < that float (0.75 is exact). */
} trtx_face_post_params;

/* dets_dev [B, 1 + max_rows*row_floats]: count, then (x1, y1, x2, y2, conf, class, keep, extras...) rows -- the compact
 *   output of trtx_nms_enqueue with TRTX_BOX_RETINA, extra_offset 5 (the landmarks, then AntiCov's mask_confidence).  Of the
 *   first min(count, max_rows) rows those with (int)keep == 1 and !(conf < conf_thresh) are used (a NaN conf is kept, as in
 *   the reference).
 * rows_dev [B, 1 + max_rows*F], F = 15 (FACE) or 16 (ANTICOV): the used count, then per used row in input order
 *   (x, y, w, h, conf, lx0, ly0, ..., lx4, ly4[, mask_conf]): the rectangle of trtx_retina_get_rect_adapt_landmark as
 *   floats (exact for |v| <= 2^24) and its mapped landmarks, bit-identical to that host function; rows past the count are
 *   zeroed.
 * A per-frame post-process: TRTX_ERR_INVALID for batch / max_rows <= 0, an unknown variant, row_floats < 7, landmarks or
 * mask_confidence outside the row.  One CTA per frame, no atomics, no workspace. */
TRTX_API int trtx_retina_postprocess_enqueue(const trtx_face_post_params* p, const int32_t* frame_wh_host, int batch,
                                             const float* dets_dev, int max_rows, float* rows_dev, trtx_stream_t stream);

/* =====================================================================================
 * 7. Mask R-CNN pre- and post-process
 *    replaces the HOST pre-process of rcnn/rcnn.cpp:497-506 (preprocessImg, a float widening loop, then an
 *    H2D copy of the fp32 batch) and the HOST loop of rcnn/rcnn.cpp:516-550, which runs after a D2H copy of
 *    BatchedNms's and MaskRcnnInference's outputs: rescale every box with score > SCORE_THRESH from the padded
 *    network input to the original image, and (MASK_ON) paste its mask into a w_ori x h_ori 8-bit canvas.
 * ===================================================================================== */
/* The four pads preprocessImg writes (rcnn/common.hpp:79-102), pads = {left, right, top, bottom}.  net_w / net_h are the
 * model input (INPUT_W / INPUT_H of calculateSize, rcnn/rcnn.cpp:349-366).  Host function. */
TRTX_API int trtx_rcnn_letterbox_pads(int img_w, int img_h, int net_w, int net_h, int pads[4]);

/* preprocessImg (rcnn/common.hpp:79-110) + the float widening of rcnn.cpp:504-505, a band pre-process (section 5):
 * dst_dev = [batch, net_h, net_w, 3] fp32 BGR, 0..255, 128 outside the resized rectangle: the engine input of
 * rcnn.cpp:259, ready for enqueue.  Image b is resized into the rectangle between the pads of trtx_rcnn_letterbox_pads, of
 * size (net_w - left - right) x (net_h - top - bottom). */
TRTX_API int trtx_rcnn_preprocess_enqueue(const trtx_image_desc* images_host, int batch, int net_w, int net_h,
                                          float* dst_dev, trtx_stream_t stream);

typedef struct trtx_rcnn_post_params {
    int32_t net_w, net_h;      /* INPUT_W, INPUT_H */
    int32_t img_w, img_h;      /* w_ori, h_ori: one original size per call; frames of mixed sizes go through
                                  trtx_rcnn_postprocess_frames_enqueue, which does not read these two */
    int32_t detections_per_im; /* DETECTIONS_PER_IMAGE (100): rows of BatchedNms's outputs */
    int32_t mask_size;         /* POOLER_RESOLUTION (14): masks are [S, S]; at most 32 */
    int32_t max_masks;         /* canvases written per image: the first min(count, max_masks) kept rows */
    float score_thresh;        /* SCORE_THRESH (0.6f); kept when score > score_thresh (a NaN score is not kept) */
} trtx_rcnn_post_params;

/* scores_dev [B, D], boxes_dev [B, D, 4] (x1, y1, x2, y2 in network-input pixels), classes_dev [B, D]: BatchedNms outputs;
 * masks_dev [B, D, S, S]: MaskRcnnInference output, or NULL for boxes only (Faster R-CNN, MASK_ON off).
 * rows_dev [B, 1 + D*7]: per image a count, then one row (x1, y1, x2, y2, score, class, slot) per slot i with
 *   score > score_thresh, in ascending i (the reference's loop order); slot = i indexes the inputs.  The box is
 *   (box - pad) * ratio with ratio = (float)img / (net - (pad_a + pad_b)) (rcnn.cpp:516-526).  Rows past the count are zeroed.
 * masks_out_dev [B, max_masks, img_h, img_w] u8, or NULL (both mask pointers NULL or both non-NULL): canvas k of image b is
 *   255 where cv::resize(mask, r.size()) (bilinear) > 0.5 inside the paste rectangle r of the k-th kept row (:543-550) and 0
 *   elsewhere; all zeros where the reference throws (empty r, r leaving the image, non-finite box).  Canvases at or past
 *   min(count, max_masks) are left untouched.  Two launches, no workspace. */
TRTX_API int trtx_rcnn_postprocess_enqueue(const trtx_rcnn_post_params* p, int batch, const float* scores_dev,
                                           const float* boxes_dev, const float* classes_dev, const float* masks_dev,
                                           float* rows_dev, uint8_t* masks_out_dev, trtx_stream_t stream);

/* The same post-process for a batch of frames of mixed original sizes, one trtx_frame per frame.
 * p: as for trtx_rcnn_postprocess_enqueue except img_w / img_h, which are not read.  scores_dev, boxes_dev, classes_dev, masks_dev and rows_dev: the layouts of
 *   trtx_rcnn_postprocess_enqueue (the engine input net_w x net_h is one size per call).
 * Image b is rescaled with its own pads, trtx_rcnn_letterbox_pads(img_w_b, img_h_b, net_w, net_h), and its own ratios, and
 *   its canvas k starts at masks_dev_b + k * img_h_b * pitch_b: image b of a call equals a batch-1
 *   trtx_rcnn_postprocess_enqueue of image b with its size.  Pixel rule, threshold and untouched canvases as there; the
 *   bytes of a row past img_w are never written.
 * Canvases for every frame or for none: NULL and non-NULL masks_dev in one call, or canvases with a NULL masks_dev input,
 *   is TRTX_ERR_INVALID (with no canvases masks_dev is not read).  A per-frame post-process: TRTX_ERR_INVALID for
 *   batch <= 0, pitch < img_w, mask_size > 32; TRTX_ERR_UNSUPPORTED for more than INT_MAX paste CTAs in one launch.  Two
 *   kernels, no workspace, no atomics. */
TRTX_API int trtx_rcnn_postprocess_frames_enqueue(const trtx_rcnn_post_params* p, const trtx_frame* images_host,
                                                  int batch, const float* scores_dev, const float* boxes_dev,
                                                  const float* classes_dev, const float* masks_dev, float* rows_dev,
                                                  trtx_stream_t stream);

/* The outlines of the pasted masks: cv::findContours(curMask, contours, RETR_EXTERNAL, CHAIN_APPROX_NONE) of
 * rcnn/rcnn.cpp:551-552 for every canvas k < min(count, max_masks) of every frame, bit for bit as cv2 4.13 returns it
 * (8-connected components of the nonzero pixels, the outer border of each component not inside a hole of another, each
 * starting at its component's first pixel in raster order and going down its left side first, the contours in descending
 * raster order of their starts).  The drawing (cv::drawContours) stays with the caller.
 * p: the parameters of the post-process call that wrote rows and canvases; only detections_per_im and max_masks are read.
 * images_host: each frame with its canvases (the single-size entry's dense canvases are frames of equal size with
 *   pitch = img_w).  rows_dev [B, 1 + D*7]: that call's rows.
 * The call reads only the paste rectangle r of each row (trtx_rcnn_postprocess_enqueue's), where the post-process writes;
 *   it returns the contours of the canvas restricted to r, which are those of the whole canvas, since the post-process
 *   leaves 0 outside r.  Where the reference throws (empty r, r leaving the image, a non-finite box) the canvas is all zeros
 *   and the call reports 0 contours.
 * Outputs, with C = max_contours and P = max_points capacities per canvas:
 *   counts_dev  [B, max_masks, 2] int32: (n_contours, n_points), the true totals even past the capacities; written for
 *               every slot, (0, 0) at or past the frame's min(count, max_masks);
 *   lengths_dev [B, max_masks, C] int32: the point counts of the first min(n_contours, C) contours;
 *   points_dev  [B, max_masks, P, 2] int32: (x, y) in frame pixels, the first min(n_points, P) points of the contours
 *               concatenated in order.
 *   Entries past those counts are not written.
 * Workspace: trtx_rcnn_contours_workspace_size(p, images_host, batch) bytes, 16-byte aligned; it depends on the arguments
 *   only: min(min(batch, 64) * max_masks, 128) slots of (W + 2)(H + 2) + 8 ceil(W/2) ceil(H/2) + 256 ceil(W/2) bytes
 *   (each term the largest over the frames, the sum rounded up to 256), about 3 bytes per frame pixel.  0 when the
 *   arguments are rejected.
 * A per-frame post-process: TRTX_ERR_INVALID for batch / detections_per_im / max_masks / max_contours / max_points <= 0,
 *   a frame without canvases, pitch < img_w, a workspace not 16-byte aligned; TRTX_ERR_UNSUPPORTED for a frame of more than
 *   2^29 pixels.  Launches of at most 128 CTAs with 200 KB of dynamic shared memory each, no atomics (deterministic). */
TRTX_API size_t trtx_rcnn_contours_workspace_size(const trtx_rcnn_post_params* p, const trtx_frame* images_host, int batch);
TRTX_API int trtx_rcnn_contours_enqueue(const trtx_rcnn_post_params* p, const trtx_frame* images_host, int batch,
                                        const float* rows_dev, int max_contours, int max_points, int32_t* counts_dev,
                                        int32_t* lengths_dev, int32_t* points_dev, void* workspace_dev,
                                        size_t workspace_bytes, trtx_stream_t stream);

/* =====================================================================================
 * 8. YOLO classification pre- and post-process
 *    replaces the HOST batch_preprocess of the cls drivers (yolov8/yolov8_cls.cpp:19-46, the same code in yolo11_cls.cpp and
 *    yolo26/yolo26_cls.cpp; yolov5/yolov5_cls.cpp:19-36) and the H2D copy of its fp32 batch, and the HOST softmax + topk
 *    (yolov8_cls.cpp:48-78, yolov5_cls.cpp:38-68, yolo26_cls.cpp:120-135) that run after a D2H copy of every logit.
 * ===================================================================================== */
/* batch_preprocess, a band pre-process (section 5): dst_dev = [batch, 3, net_h, net_w] fp32 planar RGB, the engine input.
 *   variant TRTX_YOLO_V8 (yolov8, yolo11, yolo26): the centre square crop Rect((w - m) / 2, (h - m) / 2, m, m), m = min(w, h),
 *     resized to net_w x net_h, then (float)u * (float)(1 / 255.0) per byte (convertTo(CV_32F, 1 / 255.0));
 *   variant TRTX_YOLO_V5: preprocess_img's letterbox (the rectangle of trtx_calib_letterbox_rect on a 128-grey canvas), then
 *     (float)(((float)u / 255.0 - mean) / std) in double with mean = 0.485, 0.456, 0.406 and std = 0.229, 0.224, 0.225 for
 *     R, G, B.
 * A V8 rectangle is the whole net_w x net_h; a V5 one can be empty. */
TRTX_API int trtx_cls_preprocess_enqueue(int variant, const trtx_image_desc* images_host, int batch, int net_w, int net_h,
                                         float* dst_dev, trtx_stream_t stream);

/* softmax + topk per image: logits_dev [batch, num_classes], the engine output.
 *   softmax = 1 (yolov8, yolo11, yolov5): res_i = expf(x_i) / sum, the sum in float in ascending i (softmax's loop);
 *   softmax = 0 (yolo26, whose output is already a sigmoid): res_i = x_i.
 * Outputs: index_dev [batch, k] int32, the first min(k, num_classes) indices in descending res; value_dev [batch, k], res at
 *   those indices; probs_dev [batch, num_classes], the whole res, or NULL.  Entries past min(k, num_classes) are not written.
 * Order: descending res with -0.0 == +0.0 and ties in ascending index; +NaN ranks above +inf and -NaN below -inf (an
 *   overflowing expf gives inf / inf = NaN, an all-underflow row 0 / 0).  The reference's std::sort is unstable there, and
 *   undefined with a NaN.  expf is CUDA's (within 2 ulp), so res is within a relative 2e-6 of the host's.
 * TRTX_ERR_INVALID for a null logits / index / value pointer, batch / num_classes / k <= 0 or softmax outside {0, 1};
 * TRTX_ERR_UNSUPPORTED for num_classes > 8 192; nothing is written then.  One launch, one 1024-thread CTA per image with up
 * to 96 KB of shared memory, no workspace; can be captured in a CUDA graph. */
TRTX_API int trtx_cls_postprocess_enqueue(int softmax, int batch, int num_classes, const float* logits_dev, int k,
                                          int32_t* index_dev, float* value_dev, float* probs_dev, trtx_stream_t stream);

/* =====================================================================================
 * 9. YOLOP pre- and post-process
 *    replaces the HOST preprocess_img of yolop/utils.h:11-36 with the driver's plane loop and H2D copy
 *    (yolop/yolop.cpp:110-127), and the HOST stages after inference: nms() + get_rect (yolop/common.hpp:13-83) on a D2H
 *    copy of the plugin rows, and the per-pixel loop over the drivable-area and lane maps (yolop/yolop.cpp:148-169).
 *    The detection head itself is YoloLayer_TRT with 6-float rows (TRTX_YOLO_V5, det_floats 6); its NMS is
 *    trtx_nms_enqueue with TRTX_BOX_CXCYWH, greedy.
 * ===================================================================================== */
/* preprocess_img + the plane loop, a band pre-process (section 5): dst_dev = [batch, 3, net_h, net_w] fp32 planes in the
 * driver's B, G, R order (Yolo::INPUT_W x INPUT_H = 640 x 384), the engine input.  The frame is resized into the rectangle of
 * trtx_calib_letterbox_rect on a 114-grey canvas; byte u of plane c (mean = 0.485, 0.456, 0.406 and std = 0.229, 0.224, 0.225
 * for planes 0, 1, 2) becomes
 *     s = (float)u * (1.f / 255.f) - (float)mean_c  (float),   (float)((double)s / std_c),
 * cv2 4.13's convertTo / subtract / divide chain. */
TRTX_API int trtx_yolop_preprocess_enqueue(const trtx_image_desc* images_host, int batch, int net_w, int net_h, float* dst_dev,
                                           trtx_stream_t stream);

/* YOLOP's get_rect (yolop/common.hpp:13-37): box cx, cy, w, h in network pixels (net_w x net_h = Yolo::INPUT_W x INPUT_H,
 * 640 x 384) -> rect = {x, y, w, h} in the img_w x img_h frame; each statement truncates to int, nothing is clamped.
 * Defined where the reference is not, as the compiled x86-64 reference behaves: a value that is NaN, infinite or outside
 * [-2^31, 2^31) converts to INT_MIN, and w = r - l, h = b - t wrap modulo 2^32.  Host function; the device form is
 * trtx_yolop_postprocess_enqueue. */
TRTX_API int trtx_yolop_get_rect(int net_w, int net_h, int img_w, int img_h, const float bbox[4], int rect[4]);

typedef struct trtx_yolop_post_params {
    int32_t net_w, net_h; /* Yolo::INPUT_W x INPUT_H (640 x 384): get_rect's letterbox */
    int32_t map_w, map_h; /* Yolo::IMG_W x IMG_H (640 x 360): the drivable-area and lane maps */
    int32_t row_floats;   /* floats per input row, >= 7: the compact NMS rows (cx, cy, w, h, conf, class, keep) */
} trtx_yolop_post_params;

/* dets_dev [B, 1 + max_rows*row_floats]: count, then (cx, cy, w, h, conf, class, keep, ...) rows -- the compact output of
 *   trtx_nms_enqueue (TRTX_BOX_CXCYWH, greedy, det_floats 6) over the plugin rows.  Of the first min(count, max_rows) rows
 *   those with (int)keep == 1 are used: every row of a greedy output.
 * rows_dev [B, 1 + max_rows*6]: the used count, then per used row in input order (x, y, w, h, conf, class) with x, y, w, h =
 *   trtx_yolop_get_rect as floats (exact for |v| <= 2^24); rows past the count are zeroed.
 * Labels, where frames_host[b].masks_dev is an [img_h, pitch] u8 canvas: pixel (x, y) of frame b gets 2 where
 *   lane_dev[b][sy][sx] != 0, else 1 where seg_dev[b][sy][sx] != 0, else 0 (yolop.cpp:148-169: `if (lane_idx) ... else if
 *   (seg_idx)`), with sx = min(floor(x * (1 / ((double)img_w / map_w))), map_w - 1) and sy likewise: cv::resize's
 *   INTER_NEAREST of OpenCV 4.x.  Bytes of a row past img_w are not written.  seg_dev and lane_dev are the engine's
 *   [B, map_h, map_w] int32 index maps.  Frame b reads maps b; the reference reads the first image's maps for every frame
 *   (yolop.cpp:90-92), which is the same at its BATCH_SIZE 1.  Colouring the frame stays with the caller.
 * Canvases for every frame or for none (then seg_dev and lane_dev may be NULL and are not read).  A per-frame post-process:
 * TRTX_ERR_INVALID for batch / max_rows <= 0, row_floats < 7, NULL and non-NULL masks_dev in one call, pitch < img_w;
 * TRTX_ERR_UNSUPPORTED where a CTA's shared-memory tables, 10 bytes per pixel of the widest frame's row + 8 * map_w bytes,
 * exceed 227 KB (with 640-wide maps: frames wider than about 22 000 pixels).  Two kernels, no workspace, no atomics. */
TRTX_API int trtx_yolop_postprocess_enqueue(const trtx_yolop_post_params* p, const trtx_frame* frames_host, int batch,
                                            const float* dets_dev, int max_rows, const int32_t* seg_dev,
                                            const int32_t* lane_dev, float* rows_dev, trtx_stream_t stream);

/* =====================================================================================
 * 10. DETR pre- and post-process
 *    replaces the HOST preprocessImg of detr/common.hpp:81-89 with the driver's plane loop and H2D copy
 *    (detr/detr.cpp:754-767, :638-641; the INT8 calibrator's getBatch, detr/calibrator.hpp:78-88, calls the same
 *    preprocessImg), and the HOST stage after inference: the D2H copy of the engine's scores and boxes (:643-648) and the
 *    per-query loop of detr/detr.cpp:777-806 (argmax, score threshold, no-object class, cv::Rect in the frame).
 * ===================================================================================== */
/* preprocessImg + the plane loop, a band pre-process (section 5): dst_dev = [batch, 3, net_h, net_w] fp32 planes in R, G, B
 * order (cvtColor BGR2RGB, then the driver's planes 0, 1, 2; INPUT_W x INPUT_H = 1066 x 800), the engine input.  The whole
 * frame is stretched over the whole net (no letterbox; an exact 2x downscale, where OpenCV takes INTER_AREA, gives the same
 * bytes); byte u of plane c (mean = 0.485, 0.456, 0.406 and std = 0.229, 0.224, 0.225 for planes 0, 1, 2) becomes
 *     s = (float)u * (1.f / 255.f) - (float)mean_c  (float),   (float)((double)s / std_c),
 * the driver's convertTo / `/= 255` / `-= Scalar` / `/= Scalar` chain.  Every rectangle is net_w wide. */
TRTX_API int trtx_detr_preprocess_enqueue(const trtx_image_desc* images_host, int batch, int net_w, int net_h, float* dst_dev,
                                          trtx_stream_t stream);

/* The rectangle of detr/detr.cpp:795-803 for one box cx, cy, w, h (normalised, the engine's sigmoid output) in an
 * img_w x img_h frame: x1 = (float)(((double)cx - (double)w / 2.0) * img_w), likewise y1 (cy, h), x2 and y2 (with +);
 * rect = {(int)x1, (int)y1, (int)(x2 - x1), (int)(y2 - y1)}, the differences in float.  Defined where the reference is
 * not, as the compiled x86-64 reference behaves: a value that is NaN, infinite or outside [-2^31, 2^31) converts to
 * INT_MIN.  Host function; the device form is trtx_detr_postprocess_enqueue. */
TRTX_API int trtx_detr_get_rect(int img_w, int img_h, const float box[4], int rect[4]);

typedef struct trtx_detr_post_params {
    int32_t num_queries;  /* Q: NUM_QUERIES (100) */
    int32_t num_classes;  /* C: NUM_CLASS (92), the last one the no-object class */
    float score_thresh;   /* SCORE_THRESH (0.5f) */
} trtx_detr_post_params;

/* scores_dev [B, Q, C] fp32: the engine's softmax scores; boxes_dev [B, Q, 4] fp32: its (cx, cy, w, h), normalised.
 * rows_dev [B, 1 + Q*6]: the kept count, then per kept query in query order (x, y, w, h, score, class) with x, y, w, h =
 *   trtx_detr_get_rect as floats (exact for |v| <= 2^24); rows past the count are zeroed.
 * Per query (detr.cpp:779-799): label = -1, score = -1.f; for j = 0 .. C-1 `if (score < s[j])` takes j, so the first
 * maximum wins and a NaN is never taken; the query is kept when score > score_thresh (float) and label != C - 1.  Frame b
 * reads queries b; the reference's loop runs over every query of the batch for every frame (detr.cpp:778), which is the
 * same at its BATCH_SIZE 1.  Drawing and labels stay with the caller.
 * A per-frame post-process: TRTX_ERR_INVALID for batch / Q <= 0, C < 2, or a score_thresh that is NaN or below -1 (which
 * would keep the reference's label -1 queries); TRTX_ERR_UNSUPPORTED for Q or C above 2^24 (the count and the class are
 * stored as floats).  One CTA per frame, no workspace, no atomics. */
TRTX_API int trtx_detr_postprocess_enqueue(const trtx_detr_post_params* p, const int32_t* frame_wh_host, int batch,
                                           const float* scores_dev, const float* boxes_dev, float* rows_dev,
                                           trtx_stream_t stream);

/* =====================================================================================
 * 11. CenterNet pre-process and decode
 *    replaces the HOST stages of centernet/sample/test.py (ctdet_coco_dla_2x): pre_process (:34-41) and the H2D copy of its
 *    input, and after inference the D2H copy of hm, wh and reg, ctdet_decode (:44-102) and the driver loop (:126-132).
 *    The DCNv2 plugin of the backbone is not part of this library.
 * ===================================================================================== */
/* pre_process for a whole batch, one launch per <= 64 images: images_host = `batch` u8 HWC BGR descriptors in HOST memory
 * (trtx_image_desc, any pitch and base alignment, mixed sizes allowed); dst_dev = [batch, 3, net, net] fp32 planes in the
 * frame's B, G, R order (the sample feeds cv.imread's BGR through transpose(2, 0, 1)), the engine input (net = 512).
 * Per frame: L = max(h, w, 3) (max(image.shape) includes the channel count); a float64 L x L zero canvas holds the frame at
 * its top-left; cv.resize(canvas, (net, net)) is OpenCV 4.x's INTER_LINEAR on float64, bit for bit: separable, weights
 * (1 - fx, fx) in float from fx = (float)((d + 0.5) * scale - 0.5) - floor, the tap clamped with fx = 0 at both ends of both
 * axes, each pass a0 * p0 + a1 * p1 in double; then (float)(((v / 255.) - 0.5) / 0.5) in double (the padding is -1.0f).
 * Defined where the sample raises: for 1 < w < L its `img[:h, :L] = image` fails, and the frame is placed at the top-left
 * with zeros elsewhere, the sample's evident intent; a frame with w == 1 fills every column of its rows, as numpy
 * broadcasts it there.  Every descriptor is checked before the first launch (a rejected call writes nothing):
 * TRTX_ERR_INVALID for a null pointer, batch / net <= 0, pitch < 3 * width or a dst_dev that is not 4-byte aligned;
 * TRTX_ERR_UNSUPPORTED for net > 8192.  No workspace; can be captured in a CUDA graph. */
TRTX_API int trtx_centernet_preprocess_enqueue(const trtx_image_desc* images_host, int batch, int net, float* dst_dev,
                                               trtx_stream_t stream);

typedef struct trtx_centernet_params {
    int32_t num_classes;  /* C: 80 */
    int32_t height, width; /* H, W of the heads: 128 x 128 */
    int32_t k;            /* K: 100, ctdet_decode's default */
    int32_t net;          /* frame rows only: the input side, 512 */
    int32_t down;         /* frame rows only: the heads' stride, 4 */
    float score_thresh;   /* frame rows only: 0.5f */
} trtx_centernet_params;

/* Workspace of trtx_centernet_decode_enqueue: 8 * B * C * K bytes (two 256-byte aligned halves); 0 for rejected params. */
TRTX_API size_t trtx_centernet_workspace_size(const trtx_centernet_params* p, int batch);

/* ctdet_decode(hm, wh, reg, K) for a batch: heat_dev [B, C, H, W], wh_dev [B, 2, H, W], reg_dev [B, 2, H, W], all fp32 (the
 * engine outputs hm, wh, reg) -> dets_dev [B, K, 6] fp32 (x1, y1, x2, y2, score, class) in map units.  Per image:
 *   1. s = 1 / (1 + expf(-x)) (the reference's CPU sigmoid may differ by a few ulps);
 *   2. a cell is a peak iff s equals the max of s over its 3 x 3 window clipped to the map (max_pool2d pads with -inf); the
 *      suppressed value is s at a peak and +0 elsewhere; a NaN in the window makes the max NaN, so the cell is no peak, and
 *      a NaN cell stays NaN; a saturated plateau (s == 1.0f) is a peak in every cell;
 *   3. the K largest suppressed values over all C * H * W cells, ordered NaN first, then by descending value, ties to the
 *      smaller flat index c * H * W + y * W + x.  This is the reference's two-stage topk under that order (a cell outside
 *      its class's top K has K cells above it); the reference's order among ties is implementation-defined, this one is not.  With
 *      fewer than K positive or NaN cells the rest are zero-valued cells in flat-index order;
 *   4. class = c, xs = x + reg[0, y, x], ys = y + reg[1, y, x], x1 = xs - wh[0] / 2, y1 = ys - wh[1] / 2, x2 = xs + wh[0] / 2,
 *      y2 = ys + wh[1] / 2, all float without contraction.  The accepted sizes keep the reference's float index divisions
 *      (true_divide(width), true_divide(K)) equal to integer divisions.
 * Frame rows (the driver loop), when frame_wh_host and rows_dev are both given:
 * rows_dev [B, 1 + K * 6] gets the count n of detections with score > score_thresh (a NaN score is dropped), then those
 * rows in order as (x1 * k, y1 * k, x2 * k, y2 * k, score, class), zeros past n, with k = (float)(down * (L / (double)net)),
 * L = max(img_h, img_w, 3) -- `i[:4] *= 4*s`, each product rounded once; int(), rectangles and text stay with the caller.
 * A per-frame post-process: TRTX_ERR_INVALID for batch, C, H, W or K <= 0, K > H * W (the reference's topk raises), only
 * one of frame_wh_host / rows_dev, with rows a net or down <= 0 or a NaN score_thresh, and a workspace that is not 256-byte
 * aligned; TRTX_ERR_UNSUPPORTED for C > 1024, H or W > 1024, H * W > 2^20 or K > 1024; TRTX_ERR_WORKSPACE for a workspace
 * short of trtx_centernet_workspace_size.  Two kernels, no host sync, no allocation. */
TRTX_API int trtx_centernet_decode_enqueue(const trtx_centernet_params* p, int batch, const float* heat_dev,
                                           const float* wh_dev, const float* reg_dev, void* workspace_dev,
                                           size_t workspace_bytes, float* dets_dev, const int32_t* frame_wh_host,
                                           float* rows_dev, trtx_stream_t stream);

/* =====================================================================================
 * 12. UFLD lane detection pre- and post-process
 *    replaces the HOST stages of ufld/lane_det.cpp (the Ultra-Fast Lane Detection row-anchor model): prepareImage (:194-221)
 *    and the H2D copy of its input, and after inference the D2H copy of `prob` and the driver's loops (:358-410: the row flip,
 *    argmax and softmax_mul of :223-270, the "no lane" zeroing, the lane choice and the points).  Drawing stays with the caller.
 * ===================================================================================== */
/* prepareImage, a band pre-process (section 5): dst_dev = [batch, 3, net_h, net_w] fp32 planes in R, G, B order (cvtColor
 * BGR2RGB, then cv::split; INPUT_W x INPUT_H = 800 x 288), the engine input.  The whole frame is stretched over the whole net
 * (an exact 2x downscale, where OpenCV takes INTER_AREA, gives the same bytes); byte u of plane c (the driver's
 * `static float` mean = 0.485f, 0.456f, 0.406f and std = 0.229f, 0.224f, 0.225f for planes 0, 1, 2) becomes
 *     s = (float)u * (float)(1. / 255.),   fmaf(s, (float)(1. / std_c), (float)(-mean_c / std_c))  (quotients in double),
 * the one convertTo that OpenCV 4.x makes of `(channel - mean[c]) / std[c]`, with the fused multiply-add of its AVX2 kernel.
 * The caller's frame is not converted in place, as the driver's cvtColor(img, img) does.  Every rectangle is net_w wide. */
TRTX_API int trtx_ufld_preprocess_enqueue(const trtx_image_desc* images_host, int batch, int net_w, int net_h, float* dst_dev,
                                          trtx_stream_t stream);

typedef struct trtx_ufld_post_params {
    int32_t num_cells;    /* C: OUTPUT_C = 101 (griding_num + 1); cell C - 1 is "no lane" (the driver's literal 100) */
    int32_t num_rows;     /* H: OUTPUT_H = 56 row anchors */
    int32_t num_lanes;    /* W: OUTPUT_W = 4 */
    int32_t net_w, net_h; /* INPUT_W 800, INPUT_H 288 */
    int32_t col_sample_w; /* 8 */
} trtx_ufld_post_params;

/* prob_dev [B, C, H, W] fp32: the engine output `prob`.  row_anchor_host: H ints in HOST memory (tusimple_row_anchor);
 * frame_wh_host: (w, h) of the picture the points are for ((1280, 720) is the driver's `vis`; a frame's own size gives the
 * points on that frame); the anchors are copied into launch parameters too.
 * rows_dev [B, 1 + H*W*3]: the point count n, then n rows (x, y, lane) as floats in the driver's draw order -- engine rows
 * j = H - 1 .. 0 (the driver flips the rows and indexes the anchors with H - 1 - k), the chosen lanes ascending in each --
 * then zeros.  Per cell (row j, lane l), reading prob[b, :, j, l], each statement of the driver rounded as there:
 *   argmax: int max = -10000000, max_ind = -1; for c: if (v > (float)max) max = (int)v, max_ind = c -- truncated, so a later
 *     value above the truncated running maximum wins ([3.7, 3.2] gives 1); (int)v is INT_MIN where the x86-64 conversion
 *     gives it (v >= 2^31 or +inf); a NaN is never taken; max_ind may stay -1;
 *   softmax_mul: e_c = (float)exp((double)v_c) for c < C - 1 (no max subtraction; the correctly rounded expf except within
 *     about 2^-29 of a rounding boundary), sum += e_c in float in c order, then expect += (e_c / sum) * (float)(c + 1) in c
 *     order; overflow and underflow give NaN as in the driver (inf / inf, 0 / 0);
 *   expect = 0 where max_ind == C - 1.
 * Per frame: lane l is chosen when more than 2 of its H cells have expect != 0 (a NaN counts); each chosen cell with
 * expect > 0 (NaN excluded) gives x = (int)(((expect * (float)col_sample_w) * (float)w) / (float)net_w) - 1 (float, left to
 * right; (int) as x86-64 converts, the - 1 wrapping) and y = h * anchor[j] / net_h - 1 in int; rows hold (float)x, exact for
 * |x| <= 2^24 (C * col_sample_w * w <= 2^24 * net_w suffices).
 * A per-frame post-process: TRTX_ERR_INVALID for batch, H, W, net_w, net_h or col_sample_w <= 0, or C < 2;
 * TRTX_ERR_UNSUPPORTED for H * W > 1024 or (C - 1) * H * W > 53 248 (one CTA per frame: a thread per cell, the exponentials
 * in shared memory), a frame side above 2^24, or a frame and anchor where h * anchor overflows int32 or |y| > 2^24.  No
 * workspace, no atomics. */
TRTX_API int trtx_ufld_postprocess_enqueue(const trtx_ufld_post_params* p, const int32_t* row_anchor_host,
                                           const int32_t* frame_wh_host, int batch, const float* prob_dev, float* rows_dev,
                                           trtx_stream_t stream);

/* =====================================================================================
 * 13. Bicubic letterbox pre-process (yolov3-tiny, retinafaceAntiCov)
 *    replaces the HOST preprocess_img with cv::resize(INTER_CUBIC) of yolov3-tiny/yolov3-tiny.cpp:40-60 and
 *    retinafaceAntiCov/retinafaceAntiCov.cpp:41-61, the drivers' plane loops (:441-445, :528-532) and the H2D copy of their
 *    fp32 input.
 * ===================================================================================== */
enum {
    TRTX_CUBIC_YOLOV3_TINY = 0, /* data = u / 255.0 (double), stored to float */
    TRTX_CUBIC_ANTICOV = 1,     /* data = ((float)u - 127.5) * 0.0078125 (double), stored to float: exact */
};

/* preprocess_img + the plane loop, a band pre-process (section 5): dst_dev = [batch, 3, net_h, net_w] fp32 planes in R, G, B
 * order (INPUT_W x INPUT_H = 608 x 608 for yolov3-tiny, 640 x 640 for retinafaceAntiCov), the engine input.  The frame is
 * resized into the rectangle of trtx_calib_letterbox_rect on a 128-grey canvas by OpenCV 4.x's own 8-bit INTER_CUBIC (the
 * build without IPP, which every non-x86 build runs):
 *   taps      fx = (float)((d + 0.5) * scale - 0.5), scale = 1. / ((double)dsize / ssize), s = floor(fx), fx -= s; taps
 *             s - 1 .. s + 2 clamped into the frame; weights saturate_cast<short>(interpolateCubic(fx) * 2048), A = -0.75;
 *   passes    horizontal: h = sum of the 4 products in int; vertical, for byte i of the 3 * w bytes of a resized row:
 *             i < (3 * w) & ~7: h0 * b0' + (h1 * b1' + (h2 * b2' + h3 * b3')) in float, b' = b / 2048^2, rounded half to even;
 *             otherwise (sum h_k * b_k + 2^21) >> 22; saturated to 0..255.
 * OpenCV with IPP (the default of x86 wheels) differs from this by 1 in a few % of the bytes of a non-integer-ratio resize.
 * Byte u then becomes the variant's value.  A launch stages 4 bytes per byte of its widest rectangle's row times at most 16
 * source rows (8 when enlarging). */
TRTX_API int trtx_cubic_preprocess_enqueue(int variant, const trtx_image_desc* images_host, int batch, int net_w, int net_h,
                                           float* dst_dev, trtx_stream_t stream);

/* =====================================================================================
 * 14. RefineDet pre- and post-process
 *    replaces base_transform of refinedet/refinedet.cpp (:822-839) and the H2D copy of its input, and the float64 tensor
 *    post-process of doInference (:730-815: PriorBox, the two decode steps, the ARM filter, the per-class nms() and the rows)
 *    with the driver's rectangles (:957-993 with RoiCorrect, :22-35).  Drawing and the text files stay with the caller.
 * ===================================================================================== */
/* base_transform, a band pre-process (section 5): dst_dev = [batch, 3, net, net] fp32 planes, the engine input (INPUT_W =
 * INPUT_H = 320; the reference indexes its planes with `i * INPUT_H + j`, right for square nets only, so the call takes one
 * side).  The whole frame is stretched over the net; plane 0 = R - 123, plane 1 = G - 117, plane 2 = B - 104 (exact in
 * float).  Gray frames are not accepted.  Every rectangle is net wide. */
TRTX_API int trtx_refinedet_preprocess_enqueue(const trtx_image_desc* images_host, int batch, int net, float* dst_dev,
                                               trtx_stream_t stream);

typedef struct trtx_refinedet_params {
    int32_t net;          /* S: the net side, 320; the priors are the four levels of side S / 8, S / 16, S / 32, S / 64 */
    int32_t num_classes;  /* C: num_class = 25, class 0 the background */
    float obj_thresh;     /* 0.01f: a prior keeps its ODM scores where arm_conf[p, 1] > obj_thresh */
    float conf_thresh;    /* 0.01f: a class score is a candidate where it is > conf_thresh */
    float nms_thresh;     /* 0.45f: overlap */
    int32_t top_k;        /* 1000: the highest candidates of a class that enter its NMS */
    int32_t max_det;      /* rows kept per frame; (C - 1) * top_k keeps every row the reference keeps */
    float score_thresh;   /* frame rows only: TH = 0.2f */
} trtx_refinedet_params;

/* Workspace of trtx_refinedet_postprocess_enqueue: B * (C - 1) * (4 + 2 * top_k) bytes in two 256-byte aligned parts; 0 for
 * rejected params. */
TRTX_API size_t trtx_refinedet_workspace_size(const trtx_refinedet_params* p, int batch);

/* doInference's post-process for a batch: arm_loc_dev [B, P, 4], arm_conf_dev [B, P, 2] (softmaxed), odm_loc_dev [B, P, 4],
 * odm_conf_dev [B, P, C] (softmaxed), all fp32, P = 3 * ((S/8)^2 + (S/16)^2 + (S/32)^2 + (S/64)^2) (6375 at S = 320), prior
 * index = level offset + (y * f + x) * 3 + k.
 * dets_dev [B, 1 + max_det * 6] fp32: n = min(total, max_det), then the reference's rows (x1, y1, x2, y2, score, label) in its
 * order -- classes ascending, each in keep order -- rounded to float as the driver's std::vector<float> holds them, zeros
 * past n.  Everything is the reference's float64 arithmetic, each tensor op rounded on its own (no contraction):
 *   priors   PriorBox (:553-597) in float: f_k = (float)(S / step), cx = (j + .5) / f_k, s_k = min_size / S (steps 8, 16, 32,
 *            64, min sizes 32, 64, 128, 256), anchors (s_k, s_k), (s_k * sqrt2, s_k / sqrt2), (s_k / sqrt2, s_k * sqrt2) in
 *            double rounded to float with sqrt2 = sqrtf(2.f), clamped to [0, 1].  The reference's headers decide which
 *            overload its `sqrt(ar)` names (with libstdc++, any <math.h> among them makes it the float one); the double
 *            overload gives the same table at S = 320 but differs in some anchors' last bit at S = 192, 384, 448 and
 *            704 .. 960;
 *   decode   d = (p01 + (l01 * v0) * p23, p23 * exp(l23 * v1)) over the prior with arm_loc, then the same over d with odm_loc,
 *            v0 = (double)0.1f, v1 = (double)0.2f, exp the CUDA double exp (ATen's); x1 = cx - w / 2, x2 = x1 + w;
 *   filter   score = odm_conf where arm_conf[p, 1] > obj_thresh, else odm_conf * 0.0 (inf and NaN become NaN); class c in
 *            1 .. C-1 takes the priors with score > conf_thresh (a NaN never) in the reference's order;
 *   nms      per class: the top_k highest candidates, then greedily the highest remaining box i is kept and every remaining j
 *            with !(IoU < nms_thresh) dropped (a NaN IoU drops j).  IoU clamps j's corners with i's rounded to float
 *            (`x1[i].item().toFloat()`; a finite value beyond the float range, where the reference throws, rounds to inf),
 *            as Tensor::clamp (a NaN bound gives NaN); w, h clamped to [0, INT_MAX]; inter = w * h;
 *            IoU = inter * 1.0 / ((area_j - inter) + area_i), areas (x2 - x1) * (y2 - y1) in double.
 *            Ties: the reference's CUDA sort leaves the order among equal scores, and the top_k cut at a tie, open; here a lower
 *            prior index ranks higher.
 * The reference's `score_my[0] < conf_thresh` class skip never fires (a kept score is above conf_thresh).
 * Frame rows, when frame_wh_host ((cols, rows) pairs) and rows_dev
 * [B, 1 + max_det * 6] are both given: the count, then per det row in order with score >= score_thresh (the driver's
 * `if (score < TH) continue`) (x, y, w, h, score, label) with x = (int)(x1 * cols) (a float product), w = (int)(x2 * cols -
 * x) in float, likewise y and h, then RoiCorrect: x < 0 -> 0, y < 0 -> 0, x >= cols - 1 -> 0, y >= rows - 1 -> 0, w <= 0 -> 1,
 * h <= 0 -> 1, x + w > cols - 1 -> w = cols - 1 - x, likewise h.  Conversions as x86-64 performs them (INT_MIN for NaN,
 * inf and out of range), x + w wrapping as there; zeros past the count.
 * A per-frame post-process: TRTX_ERR_INVALID for batch, net, top_k or max_det <= 0, C < 2, a NaN threshold, only one of
 * frame_wh_host / rows_dev, and a workspace that is not 256-byte aligned; TRTX_ERR_UNSUPPORTED for S not a multiple of 64,
 * P > 2^16 (S > 1024), top_k > 1024, C > 1024, max_det > 2^24 or a frame side above 2^24; TRTX_ERR_WORKSPACE for a
 * workspace short of trtx_refinedet_workspace_size.  Two kernels, no host sync, no allocation. */
TRTX_API int trtx_refinedet_postprocess_enqueue(const trtx_refinedet_params* p, int batch, const float* arm_loc_dev,
                                                const float* arm_conf_dev, const float* odm_loc_dev, const float* odm_conf_dev,
                                                void* workspace_dev, size_t workspace_bytes, float* dets_dev,
                                                const int32_t* frame_wh_host, float* rows_dev, trtx_stream_t stream);

/* =====================================================================================
 * 15. Bilinear letterbox pre-process (yolov3, yolov4, scaled-yolov4, yolov3-spp, RetinaFace)
 *    replaces the HOST preprocess_img with cv::resize(INTER_LINEAR) and the drivers' plane loops of yolov3
 *    (yolov3/utils.h:41-61, yolov3/yolov3.cpp:477-481), yolov4 (yolov4/yolov4.cpp:33-53, :637-641), scaled-yolov4
 *    (scaled-yolov4/common.hpp:14-34, yolov4_csp.cpp:466-468) and retina_r50 / retina_mnet (retinaface/common.hpp:21-41,
 *    retina_r50.cpp:342-352); yolov3-spp's letterbox + cv::dnn::blobFromImage (yolov3-spp/yolov3-spp.cpp:43-56, :533-536);
 *    and the H2D copy of their fp32 input.  The rectangles after NMS are trtx_get_rect's TRTX_YOLO_V3 and
 *    TRTX_RECT_YOLOV3_SPP, on the device trtx_yolo_seg_postprocess_enqueue's rows-only mode.
 * ===================================================================================== */
enum {
    TRTX_LINEAR_YOLOV3 = 0,     /* preprocess_img on a 128 canvas; planes R, G, B; data = u / 255.0 (double), stored to float */
    TRTX_LINEAR_RETINA = 1,     /* preprocess_img on a 128 canvas; planes B, G, R; data = u - 104.0, u - 117.0, u - 123.0
                                   (exact) */
    TRTX_LINEAR_YOLOV3_SPP = 2, /* yolov3-spp's letterbox; planes R, G, B; data = (float)u * (float)(1 / 255.0), as
                                   blobFromImage(pr, 1 / 255.0, size, Scalar(0, 0, 0), swapRB = true, crop = false) stores it */
    TRTX_LINEAR_PY = 4,         /* the Python runners' preprocess_image (section 17): trtx_pyrunner_letterbox_rect's rectangle
                                   on a 128 canvas; planes R, G, B; data as TRTX_LINEAR_YOLOV3 (float32 u / 255.0f is the same
                                   float for every byte) */
};

/* yolov3-spp's letterbox of an img_w x img_h frame for MAX_INPUT_SIZE = max_size (608 in the reference): r = std::min(max_size /
 * (img_w * 1.0), max_size / (img_h * 1.0)) stored to float, r = std::min(r, 1.0f), unpad = (int)(r * w) (a float product),
 * d = (max_size - unpad) % 32 per axis.  out = {canvas_w, canvas_h, x, y, w, h}: the (unpad_w + dw) x (unpad_h + dh) canvas the
 * engine's input shape is bound to, and the rectangle (dw / 2, dh / 2, unpad_w, unpad_h) the resized frame occupies (a frame no
 * larger than max_size keeps its size).  A caller skips frames whose canvas is below the engine profile's minimum (128, as
 * the driver does at :535).  TRTX_ERR_INVALID for a null out or a size <= 0; TRTX_ERR_UNSUPPORTED, with out filled, for an
 * empty rectangle (cv::resize throws there, e.g. 1 x 5000).  Host function. */
TRTX_API int trtx_yolov3spp_letterbox(int img_w, int img_h, int max_size, int out[6]);

/* The pre-process, a band pre-process (section 5): dst_dev = [batch, 3, net_h, net_w] fp32 planes, the engine input.  The
 * frame is resized into its rectangle on a 128-grey canvas (fx = (float)((d + 0.5) * scale - 0.5), weights
 * saturate_cast<short>((1 - fx) * 2048) and (fx * 2048), horizontal pass in int, vertical pass ((b0 * (S0 >> 4)) >> 16) +
 * ((b1 * (S1 >> 4)) >> 16) + 2) >> 2; cv2 4.13 gives these bytes with IPP on and off); a frame resized to its own size is
 * copied.  The rectangle is trtx_calib_letterbox_rect's for TRTX_LINEAR_YOLOV3 / RETINA
 * (INPUT_W x INPUT_H: 608 x 608 for yolov3 / yolov4, 512 x 512 for scaled-yolov4, 640 x 480 for RetinaFace) and
 * trtx_yolov3spp_letterbox's for TRTX_LINEAR_YOLOV3_SPP, trtx_pyrunner_letterbox_rect's for TRTX_LINEAR_PY (any net_w x
 * net_h).  max_size is read by TRTX_LINEAR_YOLOV3_SPP only; its engine binds one input shape per enqueue, so every frame's
 * canvas must be net_w x net_h: TRTX_ERR_INVALID in the first pass for max_size <= 0 and in the second for a frame whose
 * canvas is another. */
TRTX_API int trtx_linear_preprocess_enqueue(int variant, const trtx_image_desc* images_host, int batch, int net_w, int net_h,
                                            int max_size, float* dst_dev, trtx_stream_t stream);

/* =====================================================================================
 * 16. Rows of the NMS-free YOLO heads (yolov10)
 *    replaces the HOST batch_topk / get_topk of yolov10/src/postprocess.cpp:35-52, which run on one core after a D2H copy
 *    of the whole plugin buffer, and the rectangles draw_bbox takes from get_rect (:3-33).
 * ===================================================================================== */
typedef struct trtx_yolo_topk_params {
    int32_t variant;      /* the rectangle, as trtx_get_rect: TRTX_YOLO_V8 (yolov10: l, t, r, b rows, clamped to the frame)
                             or TRTX_YOLO_V5 (cx, cy, w, h rows, not clamped) */
    int32_t net_w, net_h; /* kInputW / kInputH (640) */
    int32_t row_floats;   /* floats per input row, >= 6 (box4, conf, class): 6 for yolov10's Detection */
    float conf_thresh;    /* a row is skipped when conf <= conf_thresh (kConfThresh 0.5f): a NaN confidence is kept */
} trtx_yolo_topk_params;

/* dets_dev [B, 1 + max_rows*row_floats]: the plugin output of trtx_yolo_decode_enqueue (TRTX_YOLO_V8, det_floats 6) or any
 *   buffer of that layout.  Of the first min(count, max_rows) rows, those with !(conf <= conf_thresh) are used, in input
 *   order, with no NMS and no sort (get_topk reads up to the count, which the reference's plugin lets run past maxOut; the
 *   library's decode clamps it).
 * rows_dev [B, 1 + max_rows*6]: the used count, then per used row (x, y, w, h, conf, class) with x, y, w, h = trtx_get_rect
 *   of the row's box for the variant ({0, 0, 0, 0} where that is undefined), bit-identical to it; rows past the count are
 *   zeroed.
 * A per-frame post-process: TRTX_ERR_INVALID for batch / max_rows <= 0, a variant other than the two above, row_floats < 6.
 * One CTA per frame, no atomics, no workspace. */
TRTX_API int trtx_yolo_topk_postprocess_enqueue(const trtx_yolo_topk_params* p, const int32_t* frame_wh_host, int batch,
                                                const float* dets_dev, int max_rows, float* rows_dev, trtx_stream_t stream);

/* =====================================================================================
 * 17. The Python runners' pre- and post-process (the *_trt.py scripts)
 *    replaces preprocess_image (yolov8/yolov8_det_trt.py:207-253, the same body in every yolov5, yolov7, yolov8, yolo11,
 *    yolov9, yolov10, yolov12-tubro and yolov13 runner) and the detection runners' post_process + non_max_suppression +
 *    bbox_iou + xywh2xyxy (yolov8_det_trt.py:255-381, yolov5/yolov5_det_trt.py:250-276), which run in numpy on one core per
 *    frame after a D2H copy of the whole plugin buffer.  The pre-process is trtx_linear_preprocess_enqueue(TRTX_LINEAR_PY).
 * ===================================================================================== */

/* preprocess_image's rectangle {x, y, w, h} of a src_w x src_h frame in a net_w x net_h input: r_w = net_w / src_w and
 * r_h = net_h / src_h in double; if r_h > r_w, w = net_w, h = (int)(r_w * src_h), x = 0, y = (net_h - h) / 2, else the
 * mirror case.  It differs from trtx_calib_letterbox_rect's float ratios for real frames (592 x 333 into 640 x 640: h = 360
 * here, 359 there).  TRTX_ERR_INVALID for a null rect or a size <= 0.  Host function. */
TRTX_API int trtx_pyrunner_letterbox_rect(int src_w, int src_h, int net_w, int net_h, int rect[4]);

typedef struct trtx_pyrunner_params {
    int32_t box_format;   /* how xywh2xyxy reads the plugin box: TRTX_BOX_LTRB (yolov8, yolo11, yolov9, yolov10,
                             yolov12-tubro, yolov13: l, t, r, b) or TRTX_BOX_CXCYWH (yolov3, yolov5, yolov7: cx, cy, w, h) */
    int32_t net_w, net_h; /* the runner's input_w / input_h */
    int32_t row_floats;   /* floats per plugin row: 90 (yolov8 det / 5u, yolo11, yolov12-tubro), 38 (yolov9, yolov5), 7 (yolov3),
                             6 (yolov7, yolov10, yolov13, yolov5 cuda-python) */
    int32_t label_col;    /* the float non_max_suppression compares as the label, boxes[:, -1]: row_floats - 1, or 5 where
                             the runner slices the row (yolov5 `pred[:, :6]`, yolov3); 5 <= label_col < row_floats */
    int32_t conf_col;     /* -1, or the column yolov3's post_process multiplies into the confidence (`pred[:, 4] *=
                             pred[:, 6]`): 6; 5 <= conf_col < row_floats, != label_col */
    float conf_thresh;    /* CONF_THRESH (0.5): a row is used when conf >= conf_thresh (a NaN conf never is) */
    float nms_thresh;     /* IOU_THRESHOLD (0.4): row j is removed by a kept row when IoU > nms_thresh and the labels are == */
} trtx_pyrunner_params;

/* The runner's post_process for a batch of frames of any sizes, one CTA per frame.
 * dets_dev [B, 1 + max_rows*row_floats]: the plugin output of trtx_yolo_decode_enqueue or any buffer of that layout;
 *   max_rows <= TRTX_NMS_MAX_ROWS.  The first n rows are read, n = the count float truncated and clamped to [0, max_rows]
 *   (a count below 1 or NaN reads none: the runner slices from the end for a negative count and raises on a NaN; the
 *   plugin writes neither).
 * Per frame, all in float32 as numpy computes it: conf = row[4] (times row[conf_col]); rows with conf >= conf_thresh; the
 *   box mapped by xywh2xyxy (the pad (net - r * origin) / 2 and the ratio r are computed in double and rounded to float,
 *   then y -= pad, y /= r) and clipped to [0, img_w - 1] x [0, img_h - 1] as np.clip does (a NaN stays NaN); sorted by
 *   descending conf, equal confs by ascending row (the runner's argsort leaves ties open); then greedy NMS: the front row
 *   is kept and always consumed, and removes every later row j with bbox_iou > nms_thresh (+1 on widths and heights,
 *   + 1e-16f in the denominator, no contraction) and row[label_col] == the front row's (a NaN label or box never
 *   matches).  The runner loops forever where a front row does not remove itself (a NaN label or box, an inverted box);
 *   the device defines that case by the consume rule and agrees with the runner wherever the runner returns.
 * rows_dev [B, 1 + max_rows*6]: the kept count, then the kept rows in order as (x1, y1, x2, y2, conf, row[5]) floats at
 *   the frame's size; floats past the count are zeroed.
 * A per-frame post-process: TRTX_ERR_INVALID for batch / max_rows / net sizes <= 0, another box format, columns outside
 * the ranges above, a NaN threshold, or dets_dev / rows_dev not 4-byte aligned; TRTX_ERR_UNSUPPORTED for
 * max_rows > TRTX_NMS_MAX_ROWS.  No atomics, no workspace, deterministic. */
TRTX_API int trtx_pyrunner_postprocess_enqueue(const trtx_pyrunner_params* p, const int32_t* frame_wh_host, int batch,
                                               const float* dets_dev, int max_rows, float* rows_dev, trtx_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* TRTX_HOT_H */
