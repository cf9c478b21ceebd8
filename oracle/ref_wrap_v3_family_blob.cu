// ref_wrap_v3_family_blob.cu -- TEST INFRASTRUCTURE.  The REFERENCE's YoloLayer plugin of one yolov3-family driver built by
// its deserialize constructor, so that the driver's own CalDetection kernel runs on grids, anchors and a class count other
// than its compiled-in ones.  oracle/v3family.mk links it with ref_wrap_v3_family.cu into _ref/libref_v3f_blob_<driver>.so,
// libraries of their own: a build of the other entry points alone never leaves one without this symbol.
#include <cuda_runtime_api.h>

#include <cstddef>

#include "yololayer.h"

extern "C" {
#define REF_API __attribute__((visibility("default")))
// The plugin of `blob` (the layout ref_v3f_serialize writes): the grids, anchors and class count come from the blob;
// INPUT_W / INPUT_H and MAX_OUTPUT_BBOX_COUNT stay compiled in.  inputs_dev[i]: level i tensor [batch, 3*(5+classes),
// h_i, w_i]; output [batch, 1 + MAX_OUTPUT_BBOX_COUNT*7].  The plugin launches on the DEFAULT stream: the wrapper
// synchronises the device.  The yolov4 and scaled-yolov4 plugins allocate their anchor tables in that constructor and never
// free them (an empty destructor): each call leaks one small device buffer per level.
REF_API int ref_v3f_plugin_enqueue_blob(const void* blob, size_t len, int batch, const void* const* inputs_dev,
                                        float* output_dev) {
    nvinfer1::YoloLayerPlugin p(blob, len);
    void* outs[1] = {output_dev};
    int rc = p.enqueue(batch, inputs_dev, outs, nullptr, 0);
    cudaError_t e = cudaDeviceSynchronize();
    return rc != 0 ? rc : (int)e;
}
}
