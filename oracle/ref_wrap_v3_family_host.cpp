// ref_wrap_v3_family_host.cpp -- TEST INFRASTRUCTURE.  One yolov3-family driver's yololayer.h (yolov3, yolov4, scaled-yolov4,
// yolov3-tiny; REF_V3F_LEVELS = the number of YoloKernel constants it declares), compiled on the host against oracle/shim_v3 by
// oracle/v3family.mk: the blob its plugin's default constructor serializes (CLASS_NUM, threadCount 256, the YoloKernel
// table yolo1..yoloN, yolov4/yololayer.cu:11-17 and :58-70), built from the header's own constants.  The constructor itself
// allocates device memory, so it is not called here.
#include <cstring>

#include "yololayer.h"

extern "C" __attribute__((visibility("default"))) int ref_v3f_header_blob(unsigned char* buf, int cap) {
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
extern "C" __attribute__((visibility("default"))) void ref_v3f_header_net(int* v) {
    v[0] = Yolo::INPUT_W;
    v[1] = Yolo::INPUT_H;
    v[2] = Yolo::MAX_OUTPUT_BBOX_COUNT;
    v[3] = (int)(sizeof(Yolo::Detection) / sizeof(float));
}
