// ref_wrap_v3_host.cpp -- TEST INFRASTRUCTURE.  CPU-only wrapper around one driver of the yolov3 family compiled where it lies
// (oracle/Makefile: -DREF_V3_DRIVER=<the driver's .cpp> -Dmain=ref_v3_driver_main, against oracle/shim_v3), called with the
// test's arguments:
//   yolov3.cpp, yolov4.cpp, yolov4_csp.cpp (scaled-yolov4/common.hpp's get_rect), yolov3-tiny.cpp: get_rect(img, bbox) with the
//   driver's INPUT_W x INPUT_H; its own nms() with its own thresholds, called as its main calls it (yolov3.cpp:490,
//   yolov4.cpp:653, yolov3-tiny.cpp:453; REF_V3_CSP: yolov4_csp.cpp:480, whose nms() takes the thresholds as arguments); and
//   the blob its plugin's default constructor serializes, built from yololayer.h's own constants (REF_V3F_LEVELS = the number
//   of YoloKernel constants it declares);
//   yolov3-spp.cpp (REF_V3_SPP): get_rect(src_shape, pre_shape, bbox) and letterbox(img) with its MAX_INPUT_SIZE.
#include REF_V3_DRIVER

#include <cstring>
#include <vector>

#define REF_API extern "C" __attribute__((visibility("default")))

static void ref_v3_out(const cv::Rect& r, int* rect) {
    rect[0] = r.x;
    rect[1] = r.y;
    rect[2] = r.width;
    rect[3] = r.height;
}

#ifdef REF_V3_SPP
// {MAX_INPUT_SIZE, MAX_INPUT_SIZE}: the net the library's TRTX_RECT_YOLOV3_SPP takes
REF_API void ref_v3_net(int* wh) { wh[0] = wh[1] = MAX_INPUT_SIZE; }
REF_API void ref_v3_get_rect(int img_w, int img_h, float* bbox, int* rect) {
    ref_v3_out(get_rect(cv::Size(img_w, img_h), cv::Size(), bbox), rect);
}
// out = {canvas_w, canvas_h, x, y, w, h} of letterbox() on an img_w x img_h frame
REF_API void ref_v3_letterbox(int img_w, int img_h, int* out) {
    cv::Mat img(img_h, img_w, CV_8UC3);
    int* g = cv::Mat::shim_geometry();
    for (int i = 0; i < 6; ++i) g[i] = -1;
    cv::Mat pr = letterbox(img);
    out[0] = pr.cols;
    out[1] = pr.rows;
    for (int i = 0; i < 4; ++i) out[2 + i] = g[i];
}
#else
REF_API void ref_v3_net(int* wh) {
    wh[0] = INPUT_W;
    wh[1] = INPUT_H;
}
REF_API void ref_v3_get_rect(int img_w, int img_h, float* bbox, int* rect) {
    cv::Mat img(img_h, img_w, CV_8UC3);
    ref_v3_out(get_rect(img, bbox), rect);
}

// output: a plugin buffer [count, 7-float rows]; the kept rows, in the order of `res`, go to res_out (room for max_rows
// rows).  Returns their number.
REF_API int ref_v3_nms(float* output, float* res_out, int max_rows) {
    std::vector<Yolo::Detection> res;
#ifdef REF_V3_CSP
    nms(res, output, BBOX_CONF_THRESH, NMS_THRESH);
#else
    nms(res, output);
#endif
    const int n = (int)res.size() < max_rows ? (int)res.size() : max_rows;
    if (n > 0) std::memcpy(res_out, res.data(), sizeof(Yolo::Detection) * (size_t)n);
    return n;
}

// the blob the plugin's default constructor serializes (CLASS_NUM, threadCount 256, the YoloKernel table yolo1..yoloN,
// yolov4/yololayer.cu:11-17 and :58-70).  The constructor itself allocates device memory, so it is not called here.
REF_API int ref_v3f_header_blob(unsigned char* buf, int cap) {
    const Yolo::YoloKernel ks[] = {Yolo::yolo1, Yolo::yolo2
#if REF_V3F_LEVELS == 3
                                   , Yolo::yolo3
#endif
    };
    const int n = (int)(sizeof(ks) / sizeof(ks[0]));
    const int len = 12 + (int)sizeof(ks);
    if (len > cap) return -1;
    const int head[3] = {Yolo::CLASS_NUM, 256, n};
    std::memcpy(buf, head, 12);
    std::memcpy(buf + 12, ks, sizeof(ks));
    return len;
}
REF_API void ref_v3f_header_net(int* v) {
    v[0] = Yolo::INPUT_W;
    v[1] = Yolo::INPUT_H;
    v[2] = Yolo::MAX_OUTPUT_BBOX_COUNT;
    v[3] = (int)(sizeof(Yolo::Detection) / sizeof(float));
}
#endif
