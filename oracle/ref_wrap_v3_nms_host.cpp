// ref_wrap_v3_nms_host.cpp -- TEST INFRASTRUCTURE.  CPU-only wrapper around one yolov3-family driver compiled where it lies
// (oracle/v3family.mk: -DREF_V3_DRIVER=<the driver's .cpp> -Dmain=ref_v3_driver_main, against oracle/shim_v3): the driver's
// own nms() with its own thresholds, called as its main calls it (yolov3.cpp:490, yolov4.cpp:653, yolov3-tiny.cpp:453;
// REF_V3_CSP: yolov4_csp.cpp:480, whose nms() takes the thresholds as arguments).
#include REF_V3_DRIVER

#include <cstring>
#include <vector>

// output: a plugin buffer [count, 7-float rows]; the kept rows, in the order of `res`, go to res_out (room for max_rows
// rows).  Returns their number.
extern "C" __attribute__((visibility("default"))) int ref_v3_nms(float* output, float* res_out, int max_rows) {
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
