// ref_wrap_pose_obb_host.cpp -- TEST INFRASTRUCTURE.  The reference's own draw_bbox_obb (get_corner) and
// draw_bbox_keypoints_line (get_rect_adapt_landmark), run whole on the CPU: yolov8/src/postprocess.cpp (REF_POSE_OBB_V8,
// net 640) or yolo11/src/postprocess.cpp (REF_POSE_OBB_V11: get_corner calls get_rect_obb, net 1024) is compiled into a
// namespace of its own (the two files define the same names; the namespace also reaches the static get_corner's caller),
// against the header shim oracle/shim_pose_obb, whose cv::polylines / cv::rectangle record what they are handed.
// oracle/Makefile builds this file once per variant and links both objects into oracle/_ref/libref_pose_obb_host.so.
#include <dirent.h>

#include <cstdint>
#include <cstring>
#include <opencv2/opencv.hpp>
#include <sstream>
#include <string>
#include <vector>

#include "NvInfer.h"

#if defined(REF_POSE_OBB_V8)
#define REF_NS ref_pose_obb_v8
#define REF_DRAW_OBB ref_v8_draw_bbox_obb
#define REF_DRAW_POSE ref_v8_draw_bbox_keypoints_line
#else
#define REF_NS ref_pose_obb_v11
#define REF_DRAW_OBB ref_v11_draw_bbox_obb
#define REF_DRAW_POSE ref_v11_draw_bbox_keypoints_line
#endif

namespace REF_NS {
#include "postprocess.cpp"
}

namespace {
// std::cout of the reference (get_corner's debug prints) goes to `log` (at most log_cap bytes, NUL-terminated); returns the
// length of the whole text
template <typename Fn>
int with_cout(char* log, int log_cap, Fn fn) {
    std::ostringstream text;
    std::streambuf* old = std::cout.rdbuf(text.rdbuf());
    fn();
    std::cout.rdbuf(old);
    const std::string s = text.str();
    if (log && log_cap > 0) {
        const size_t k = std::min(s.size(), (size_t)log_cap - 1);
        std::memcpy(log, s.data(), k);
        log[k] = 0;
    }
    return (int)s.size();
}
}  // namespace

// n oriented boxes (cx, cy, w, h, angle in radians; network pixels) of one img_w x img_h frame through draw_bbox_obb:
// corners [n, 8] = the four points get_corner hands to cv::polylines, in its order.  Returns the length of the printed text.
extern "C" __attribute__((visibility("default"))) int REF_DRAW_OBB(int img_w, int img_h, int n, const float* boxes5, int* corners,
                                                                   char* log, int log_cap) {
    using namespace REF_NS;
    std::vector<cv::Mat> imgs{cv::Mat(img_h, img_w, CV_8UC3)};
    std::vector<std::vector<Detection>> res(1);
    for (int i = 0; i < n; ++i) {
        Detection det;
        std::memset(&det, 0, sizeof(det));
        std::memcpy(det.bbox, boxes5 + 5 * i, sizeof(det.bbox));
        det.angle = boxes5[5 * i + 4];
        det.conf = 0.9f;
        det.class_id = (float)(i % 15);
        res[0].push_back(det);
    }
    cv::shim_record() = cv::ShimRecord();
    const int len = with_cout(log, log_cap, [&] { draw_bbox_obb(imgs, res); });
    const auto& pts = cv::shim_record().polylines;
    for (size_t k = 0; k < pts.size() && k < (size_t)4 * n; ++k) {
        corners[2 * k] = pts[k].x;
        corners[2 * k + 1] = pts[k].y;
    }
    return pts.size() == (size_t)4 * n ? len : -1;
}

// n pose detections (l, t, r, b and kNumberOfPoints (x, y, conf) keypoints; network pixels) of one img_w x img_h frame
// through draw_bbox_keypoints_line: rects [n, 4] = the cv::Rect it draws (get_rect_adapt_landmark's), kpts [n, 51] = the
// keypoints it mapped in place.  Returns 0, or -1 when the drawing calls did not see n rectangles.
extern "C" __attribute__((visibility("default"))) int REF_DRAW_POSE(int img_w, int img_h, int n, const float* boxes4,
                                                                    const float* kpts_in, int* rects, float* kpts_out) {
    using namespace REF_NS;
    std::vector<cv::Mat> imgs{cv::Mat(img_h, img_w, CV_8UC3)};
    std::vector<std::vector<Detection>> res(1);
    for (int i = 0; i < n; ++i) {
        Detection det;
        std::memset(&det, 0, sizeof(det));
        std::memcpy(det.bbox, boxes4 + 4 * i, sizeof(det.bbox));
        std::memcpy(det.keypoints, kpts_in + (size_t)kNumberOfPoints * 3 * i, sizeof(det.keypoints));
        det.conf = 0.9f;
        res[0].push_back(det);
    }
    cv::shim_record() = cv::ShimRecord();
    with_cout(nullptr, 0, [&] { draw_bbox_keypoints_line(imgs, res); });
    const auto& r = cv::shim_record().rects;
    if (r.size() != (size_t)n) return -1;
    for (int i = 0; i < n; ++i) {
        rects[4 * i] = r[i].x;
        rects[4 * i + 1] = r[i].y;
        rects[4 * i + 2] = r[i].width;
        rects[4 * i + 3] = r[i].height;
        std::memcpy(kpts_out + (size_t)kNumberOfPoints * 3 * i, res[0][i].keypoints, sizeof(res[0][i].keypoints));
    }
    return 0;
}
