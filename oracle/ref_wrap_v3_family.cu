// ref_wrap_v3_family.cu -- TEST INFRASTRUCTURE.  extern "C" entry points around the REFERENCE's own YoloLayer plugin of one
// yolov3-family driver (yolov3, yolov4, scaled-yolov4 or yolov3-tiny: yololayer.cu compiled where it lies by
// oracle/Makefile, IPluginV2IOExt of TensorRT 7), and the driver's compiled-in constants (yololayer.h).
// The plugin launches on the DEFAULT stream and memsets synchronously: the wrapper synchronises the device.
#include <cuda_runtime_api.h>

#include <cstddef>
#include <cstring>

#include "yololayer.h"

extern "C" {
#define REF_API __attribute__((visibility("default")))
REF_API int ref_v3f_det_floats() { return (int)(sizeof(Yolo::Detection) / sizeof(float)); }
REF_API int ref_v3f_num_classes() { return Yolo::CLASS_NUM; }
REF_API int ref_v3f_max_out() { return Yolo::MAX_OUTPUT_BBOX_COUNT; }
REF_API void ref_v3f_net(int* wh) {
    wh[0] = Yolo::INPUT_W;
    wh[1] = Yolo::INPUT_H;
}
REF_API float ref_v3f_ignore_thresh() { return Yolo::IGNORE_THRESH; }

// the default-constructed plugin's own serialize(): classCount, threadCount, kernelCount, its YoloKernel table.  Returns the
// length, or -1 when cap is too small.
REF_API int ref_v3f_serialize(unsigned char* buf, int cap) {
    nvinfer1::YoloLayerPlugin p;
    const int n = (int)p.getSerializationSize();
    if (n > cap) return -1;
    p.serialize(buf);
    return n;
}

// inputs_dev[i]: level i tensor [batch, 3*(5+CLASS_NUM), h_i, w_i] of the plugin's YoloKernel i; output [batch, 1 + 1000*7]
REF_API int ref_v3f_plugin_enqueue(int batch, const void* const* inputs_dev, float* output_dev) {
    nvinfer1::YoloLayerPlugin p;
    void* outs[1] = {output_dev};
    int rc = p.enqueue(batch, inputs_dev, outs, nullptr, 0);
    cudaError_t e = cudaDeviceSynchronize();
    return rc != 0 ? rc : (int)e;
}

// The plugin built by its deserialize constructor from `blob` (the layout ref_v3f_serialize writes), so that the driver's own
// CalDetection kernel runs on grids, anchors and a class count other than its compiled-in ones: those come from the blob;
// INPUT_W / INPUT_H and MAX_OUTPUT_BBOX_COUNT stay compiled in.  inputs_dev[i]: level i tensor [batch, 3*(5+classes),
// h_i, w_i]; output [batch, 1 + MAX_OUTPUT_BBOX_COUNT*7].  The yolov4 and scaled-yolov4 plugins allocate their anchor tables
// in that constructor and never free them (an empty destructor): each call leaks one small device buffer per level.
REF_API int ref_v3f_plugin_enqueue_blob(const void* blob, size_t len, int batch, const void* const* inputs_dev,
                                        float* output_dev) {
    nvinfer1::YoloLayerPlugin p(blob, len);
    void* outs[1] = {output_dev};
    int rc = p.enqueue(batch, inputs_dev, outs, nullptr, 0);
    cudaError_t e = cudaDeviceSynchronize();
    return rc != 0 ? rc : (int)e;
}
}
