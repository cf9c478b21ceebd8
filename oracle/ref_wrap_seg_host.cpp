// ref_wrap_seg_host.cpp -- TEST INFRASTRUCTURE.  The reference's own draw_mask_bbox + scale_mask + get_rect, run on the CPU:
// yolov8/src/postprocess.cpp (REF_SEG_V8) or yolov5/src/postprocess.cpp (REF_SEG_V5) is compiled into a namespace of its
// own (the two files define the same names), against the header shim oracle/shim_seg; oracle/Makefile builds this file
// once per variant and links both objects into oracle/_ref/libref_seg_host.so.
#include <dirent.h>

#include <cstdint>
#include <cstring>
#include <opencv2/opencv.hpp>
#include <string>
#include <unordered_map>
#include <vector>

#include "NvInfer.h"

#if defined(REF_SEG_V8)
#define REF_NS ref_seg_v8
#define REF_ENTRY ref_v8_draw_mask_select
#else
#define REF_NS ref_seg_v5
#define REF_ENTRY ref_v5_draw_mask_select
#endif

namespace REF_NS {
#include "postprocess.cpp"
}

// One detection (bbox in the variant's format, class 0, whose palette colour has every channel >= 2) with its 640 x 640
// process_mask output `mask`, drawn by draw_mask_bbox onto an all-zero img_w x img_h BGR image: sel = 1 where a pixel changed,
// i.e. exactly the pixels the reference's mask selection keeps (the rectangle and label calls are no-ops in the shim).
extern "C" __attribute__((visibility("default"))) void REF_ENTRY(int img_w, int img_h, const float* mask, const float* bbox,
                                                                 uint8_t* sel) {
    using namespace REF_NS;
    cv::Mat img(img_h, img_w, CV_8UC3);
    Detection det;
    std::memset(&det, 0, sizeof(det));
    std::memcpy(det.bbox, bbox, sizeof(det.bbox));
    det.conf = 0.9f;
    det.class_id = 0.0f;
    std::vector<Detection> dets{det};
    std::vector<cv::Mat> masks{cv::Mat(kInputH, kInputW, CV_32F, const_cast<float*>(mask))};
    std::unordered_map<int, std::string> labels{{0, "person"}};
    draw_mask_bbox(img, dets, masks, labels);
    for (int y = 0; y < img_h; ++y) {
        const unsigned char* p = img.ptr(y);
        for (int x = 0; x < img_w; ++x) sel[(size_t)y * img_w + x] = (p[3 * x] | p[3 * x + 1] | p[3 * x + 2]) != 0;
    }
}
