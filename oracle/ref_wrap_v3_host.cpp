// ref_wrap_v3_host.cpp -- TEST INFRASTRUCTURE.  CPU-only wrapper around one driver of the yolov3 family compiled where it lies
// (oracle/linear.mk: -DREF_V3_DRIVER=<the driver's .cpp> -Dmain=ref_v3_driver_main, against oracle/shim_v3): its own get_rect,
// and with REF_V3_SPP yolov3-spp's own letterbox, called with the test's arguments.
//   yolov3.cpp, yolov4.cpp, yolov4_csp.cpp (scaled-yolov4/common.hpp's get_rect), yolov3-tiny.cpp: get_rect(img, bbox) with the
//   driver's INPUT_W x INPUT_H;  yolov3-spp.cpp (REF_V3_SPP): get_rect(src_shape, pre_shape, bbox) and letterbox(img) with its
//   MAX_INPUT_SIZE.
#include REF_V3_DRIVER

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
#endif
