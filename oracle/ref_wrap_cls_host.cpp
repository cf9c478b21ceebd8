// ref_wrap_cls_host.cpp -- TEST INFRASTRUCTURE.  CPU-only wrapper around one YOLO cls driver compiled where it lies
// (oracle/cls.mk: -DREF_CLS_DRIVER=<the driver's .cpp> -Dmain=ref_cls_driver_main, against oracle/shim_cls): its own
// batch_preprocess, softmax and topk, called with the test's arguments.
//   REF_CLS_V5       yolov5_cls.cpp: batch_preprocess calls preprocess_img (yolov5/src/calibrator.cpp, not compiled here); it is
//                    defined below as the identity, so that the driver's mean / std loop runs over the caller's bytes.
//   REF_CLS_SOFTMAX  the driver has a softmax (every one but yolo26).
#include <vector>

#include REF_CLS_DRIVER

#define REF_API __attribute__((visibility("default")))

#ifdef REF_CLS_V5
cv::Mat preprocess_img(cv::Mat& img, int, int) { return img; }
#endif

extern "C" {
#ifdef REF_CLS_V5
// out = [3, n]: the driver's R, G, B planes of n BGR pixels
REF_API void ref_cls_v5_normalize(const unsigned char* bgr, int n, float* out) {
    std::vector<cv::Mat> imgs{cv::Mat(1, n, CV_8UC3, const_cast<unsigned char*>(bgr), (size_t)n * 3)};
    batch_preprocess(imgs, out);
}
#else
// geom = {crop x, crop y, crop width, crop height, resize width, resize height} of batch_preprocess on one img_w x img_h image
REF_API void ref_cls_crop_geometry(int img_w, int img_h, int net_w, int net_h, int* geom) {
    std::vector<cv::Mat> imgs{cv::Mat(img_h, img_w, CV_8UC3)};
    std::vector<float> out((size_t)3 * net_w * net_h);
    for (int i = 0; i < 6; ++i) cv::Mat::shim_geometry()[i] = -1;
    batch_preprocess(imgs, out.data(), net_w, net_h);
    for (int i = 0; i < 6; ++i) geom[i] = cv::Mat::shim_geometry()[i];
}
#endif

#ifdef REF_CLS_SOFTMAX
REF_API void ref_cls_softmax(float* x, int n, float* res) {
    const std::vector<float> r = softmax(x, n);
    for (int i = 0; i < n; ++i) res[i] = r[i];
}
#endif

// the first min(k, n) indices topk returns; their count
REF_API int ref_cls_topk(const float* res, int n, int k, int* idx) {
    const std::vector<int> t = topk(std::vector<float>(res, res + n), k);
    for (size_t i = 0; i < t.size(); ++i) idx[i] = t[i];
    return (int)t.size();
}
}
