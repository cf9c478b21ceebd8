// ref_wrap_anchor_free_host.cpp -- TEST INFRASTRUCTURE.  CPU-only wrapper around one driver's own post-process
// (src/postprocess.cpp compiled where it lies by oracle/anchor_free.mk, against oracle/shim; unused code dropped with
// -Wl,--gc-sections): yolov9's and yolov13's nms() (REF_AF_NMS), yolov10's get_topk (REF_AF_TOPK), and each one's get_rect.
#include <cstring>
#include <vector>

#include "postprocess.h"
#include "types.h"

#ifdef REF_AF_TOPK
// defined in yolov10/src/postprocess.cpp (:35) without a declaration in postprocess.h
void get_topk(std::vector<Detection>& res, float* output, float conf_thresh, int tokp);
#endif

extern "C" {
#define REF_API __attribute__((visibility("default")))
REF_API int ref_af_host_det_floats() { return (int)(sizeof(Detection) / sizeof(float)); }

// output: one image's plugin buffer [count, rows]; the rows of `res`, in its order, go to res_out (room for max_rows rows)
REF_API int ref_af_rows(float* output, float conf_thresh, float nms_thresh, float* res_out, int max_rows) {
    std::vector<Detection> res;
#ifdef REF_AF_NMS
    nms(res, output, conf_thresh, nms_thresh);
#else
    (void)nms_thresh;
    get_topk(res, output, conf_thresh, 0);
#endif
    const int n = (int)res.size() < max_rows ? (int)res.size() : max_rows;
    if (n > 0) std::memcpy(res_out, res.data(), sizeof(Detection) * (size_t)n);
    return (int)res.size();
}

REF_API void ref_af_get_rect(int img_w, int img_h, float* bbox, int* rect) {
    cv::Mat img(img_h, img_w, CV_8UC3, nullptr);
    const cv::Rect r = get_rect(img, bbox);
    rect[0] = r.x;
    rect[1] = r.y;
    rect[2] = r.width;
    rect[3] = r.height;
}

REF_API void ref_af_consts(int* v) {
    v[0] = kInputW;
    v[1] = kInputH;
    v[2] = kMaxNumOutputBbox;
    v[3] = (int)(sizeof(Detection) / sizeof(float));
}
REF_API void ref_af_thresh(float* v) {
#ifdef REF_AF_TOPK
    v[0] = kConfThresh;
    v[1] = 0.0f;
#else
    v[0] = kConfThresh;
    v[1] = kNmsThresh;
#endif
}
}
