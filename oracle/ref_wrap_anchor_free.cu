// ref_wrap_anchor_free.cu -- TEST INFRASTRUCTURE.  extern "C" entry points around the REFERENCE's own YoloLayer plugin of
// yolov9 (REF_AF_V9), yolov10 or yolov13 (plugin/yololayer.cu compiled where it lies by oracle/Makefile, IPluginV2IOExt).
// The plugin launches on the given stream and memsets there: the wrapper synchronises the stream.
#include <cuda_runtime_api.h>

#include "types.h"
#include "yololayer.h"

extern "C" {
#define REF_API __attribute__((visibility("default")))
REF_API int ref_af_det_floats() { return (int)(sizeof(Detection) / sizeof(float)); }

#ifdef REF_AF_V9
// YoloLayerPlugin(classCount, netW, netH, maxOut, is_seg) (yolov9/plugin/yololayer.cu:25-31); strides are ignored
#define REF_AF_PLUGIN(p) nvinfer1::YoloLayerPlugin p(nc, w, h, max_out, seg != 0)
#else
// YoloLayerPlugin(classCount, netW, netH, maxOut, strides, n) (yolov10/plugin/yololayer.cu:28-38); seg is ignored
#define REF_AF_PLUGIN(p) nvinfer1::YoloLayerPlugin p(nc, w, h, max_out, strides, n)
#endif

// the plugin's own serialize(); returns the length, or -1 when cap is too small
REF_API int ref_af_serialize(int nc, int w, int h, int max_out, int seg, const int* strides, int n, unsigned char* buf, int cap) {
    REF_AF_PLUGIN(p);
    const int len = (int)p.getSerializationSize();
    if (len > cap) return -1;
    p.serialize(buf);
    return len;
}

// YoloLayerPlugin::enqueue: inputs_dev[l] = level l [batch, C, grid], output [batch, 1 + max_out * det_floats]
REF_API int ref_af_enqueue(int nc, int w, int h, int max_out, int seg, const int* strides, int n, int batch,
                           const void* const* inputs_dev, float* output_dev, void* stream) {
    REF_AF_PLUGIN(p);
    void* outs[1] = {output_dev};
    const int rc = p.enqueue(batch, inputs_dev, outs, nullptr, static_cast<cudaStream_t>(stream));
    const cudaError_t e = cudaStreamSynchronize(static_cast<cudaStream_t>(stream));
    return rc != 0 ? rc : (int)e;
}
}
