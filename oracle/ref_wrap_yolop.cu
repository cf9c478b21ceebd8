// ref_wrap_yolop.cu -- TEST INFRASTRUCTURE.  extern "C" entry point around the REFERENCE's YOLOP YoloLayer plugin
// (yolop/yololayer.cu: CalDetection with 6-float Yolo::Detection rows), compiled from /root/reference.
#include <cuda_runtime_api.h>

#include <cstring>
#include <vector>

#include "yololayer.h"

extern "C" {
#define REF_API __attribute__((visibility("default")))
REF_API int ref_yolop_det_floats() { return (int)(sizeof(Yolo::Detection) / sizeof(float)); }

// kernels: nlevels x {int w, int h, float anchors[6]} = Yolo::YoloKernel (yololayer.h:13-18), in the plugin's input order
REF_API int ref_yolop_plugin_enqueue(int nc, int netw, int neth, int max_out, const void* kernels, int nlevels, int batch,
                                     const void* const* inputs_dev, float* output_dev, void* stream) {
    std::vector<Yolo::YoloKernel> ks(nlevels);
    memcpy(ks.data(), kernels, sizeof(Yolo::YoloKernel) * nlevels);
    nvinfer1::YoloLayerPlugin p(nc, netw, neth, max_out, ks);
    void* outs[1] = {output_dev};
    int rc = p.enqueue(batch, inputs_dev, outs, nullptr, static_cast<cudaStream_t>(stream));
    cudaError_t e = cudaStreamSynchronize(static_cast<cudaStream_t>(stream));
    return rc != 0 ? rc : (int)e;
}
}
