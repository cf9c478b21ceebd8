// ref_wrap_obb26_host.cpp -- TEST INFRASTRUCTURE.  yolo26's own draw_bbox_obb (get_corner over get_rect_obb, net 1024), run
// whole on the CPU: yolo26/src/postprocess.cpp is compiled into a namespace of its own against the header shim
// oracle/shim_pose_obb, whose cv::polylines records the points it is handed.  oracle/face_obb26.mk builds it into
// oracle/_ref/libref_obb26_host.so.
#include <cstdint>
#include <cstring>
#include <opencv2/opencv.hpp>
#include <sstream>
#include <string>
#include <vector>

#include "NvInfer.h"

namespace ref_obb26 {
#include "postprocess.cpp"
}

// n oriented boxes (cx, cy, w, h, angle in radians; network pixels) of one img_w x img_h frame through draw_bbox_obb:
// corners [n, 8] = the four points get_corner hands to cv::polylines, in its order.  The reference's std::cout goes to `log`
// (at most log_cap bytes, NUL-terminated).  Returns the length of the printed text, or -1 when the drawing calls did not
// see 4 points per box.
extern "C" __attribute__((visibility("default"))) int ref_v26_draw_bbox_obb(int img_w, int img_h, int n, const float* boxes5,
                                                                            int* corners, char* log, int log_cap) {
    using namespace ref_obb26;
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
    std::ostringstream text;
    std::streambuf* old = std::cout.rdbuf(text.rdbuf());
    draw_bbox_obb(imgs, res);
    std::cout.rdbuf(old);
    const std::string s = text.str();
    if (log && log_cap > 0) {
        const size_t k = std::min(s.size(), (size_t)log_cap - 1);
        std::memcpy(log, s.data(), k);
        log[k] = 0;
    }
    const auto& pts = cv::shim_record().polylines;
    for (size_t k = 0; k < pts.size() && k < (size_t)4 * n; ++k) {
        corners[2 * k] = pts[k].x;
        corners[2 * k + 1] = pts[k].y;
    }
    return pts.size() == (size_t)4 * n ? (int)s.size() : -1;
}
