// ref_wrap_yolop_host.cpp -- TEST INFRASTRUCTURE.  CPU-only wrapper around YOLOP's own nms() and get_rect
// (yolop/common.hpp:13-83), compiled where they lie against tests/mock_trt and the OpenCV type shim.
//
// common.hpp also defines YOLOP's builder helpers (convBlock, focus, SPP, addYoLoLayer, ...; :150-357).  They are never called
// here, but they must compile, and they use builder layers the mock does not declare.  The declarations below are those
// layers, from the public TensorRT 8.6 API documentation; common.hpp sees INetworkDefinition as the YolopNetwork class below,
// which adds the layer factories it calls to the mock's interface.
#include <cstring>
#include <vector>

#include "NvInfer.h"

namespace nvinfer1 {
enum class ActivationType : int32_t {
    kRELU = 0, kSIGMOID = 1, kTANH = 2, kLEAKY_RELU = 3, kELU = 4, kSELU = 5, kSOFTSIGN = 6, kSOFTPLUS = 7, kCLIP = 8,
    kHARD_SIGMOID = 9, kSCALED_TANH = 10, kTHRESHOLDED_RELU = 11
};
enum class ElementWiseOperation : int32_t { kSUM = 0, kPROD = 1, kMAX = 2, kMIN = 3, kSUB = 4, kDIV = 5, kPOW = 6 };
enum class PoolingType : int32_t { kMAX = 0, kAVERAGE = 1, kMAX_AVERAGE_BLEND = 2 };
enum class ResizeMode : int32_t { kNEAREST = 0, kLINEAR = 1 };
class IConvolutionLayer : public ILayer {
   public:
    virtual void setStrideNd(Dims stride) noexcept = 0;
    virtual void setPaddingNd(Dims padding) noexcept = 0;
    virtual void setNbGroups(int32_t nbGroups) noexcept = 0;
};
class IActivationLayer : public ILayer {
   public:
    virtual void setAlpha(float alpha) noexcept = 0;
    virtual void setBeta(float beta) noexcept = 0;
};
class IPoolingLayer : public ILayer {
   public:
    virtual void setStrideNd(Dims stride) noexcept = 0;
    virtual void setPaddingNd(Dims padding) noexcept = 0;
};
class IResizeLayer : public ILayer {
   public:
    virtual void setOutputDimensions(Dims dimensions) noexcept = 0;
    virtual void setResizeMode(ResizeMode resizeMode) noexcept = 0;
};
class IElementWiseLayer : public ILayer {};
class ISliceLayer : public ILayer {};
class IConcatenationLayer : public ILayer {};
class IPaddingLayer : public ILayer {};
class IConstantLayer : public ILayer {};
class IPluginV2Layer : public ILayer {};
class YolopNetwork : public INetworkDefinition {
   public:
    virtual IConvolutionLayer* addConvolutionNd(ITensor& input, int32_t nbOutputMaps, Dims kernelSize, Weights kernelWeights,
                                                Weights biasWeights) noexcept = 0;
    virtual IActivationLayer* addActivation(ITensor& input, ActivationType type) noexcept = 0;
    virtual IElementWiseLayer* addElementWise(ITensor& input1, ITensor& input2, ElementWiseOperation op) noexcept = 0;
    virtual ISliceLayer* addSlice(ITensor& input, Dims start, Dims size, Dims stride) noexcept = 0;
    virtual IConcatenationLayer* addConcatenation(ITensor* const* inputs, int32_t nbInputs) noexcept = 0;
    virtual IPoolingLayer* addPoolingNd(ITensor& input, PoolingType type, Dims windowSize) noexcept = 0;
    virtual IResizeLayer* addResize(ITensor& input) noexcept = 0;
    virtual IPaddingLayer* addPaddingNd(ITensor& input, Dims prePadding, Dims postPadding) noexcept = 0;
    virtual IConstantLayer* addConstant(Dims dimensions, Weights weights) noexcept = 0;
    virtual IPluginV2Layer* addPluginV2(ITensor* const* inputs, int32_t nbInputs, IPluginV2& plugin) noexcept = 0;
};
}  // namespace nvinfer1

#define INetworkDefinition YolopNetwork
#include "common.hpp"
#undef INetworkDefinition

extern "C" {
__attribute__((visibility("default"))) int ref_yolop_det_floats() { return (int)(sizeof(Yolo::Detection) / sizeof(float)); }
// nms(res, output, conf_thresh, nms_thresh): output = count, then 6-float rows (Yolo::Detection); res_out gets the kept rows
__attribute__((visibility("default"))) int ref_yolop_nms(float* output_host, float conf_thresh, float nms_thresh, float* res_out) {
    std::vector<Yolo::Detection> res;
    nms(res, output_host, conf_thresh, nms_thresh);
    for (size_t i = 0; i < res.size(); ++i) memcpy(res_out + i * (sizeof(Yolo::Detection) / 4), &res[i], sizeof(Yolo::Detection));
    return (int)res.size();
}
// get_rect(img, bbox): box cx, cy, w, h in network pixels (Yolo::INPUT_W x INPUT_H = 640 x 384) -> {x, y, w, h} in the frame
__attribute__((visibility("default"))) void ref_yolop_get_rect(int img_w, int img_h, float* bbox, int* rect_out) {
    cv::Mat img(img_h, img_w, CV_8UC3, nullptr);
    cv::Rect r = get_rect(img, bbox);
    rect_out[0] = r.x;
    rect_out[1] = r.y;
    rect_out[2] = r.width;
    rect_out[3] = r.height;
}
}
