// SHIM, not TensorRT -- TEST INFRASTRUCTURE.  tests/mock_trt/NvInfer.h (the plugin interfaces) plus the builder, network, engine
// and runtime names that the yolov3 / yolov4 / scaled-yolov4 / yolov3-tiny / yolov3-spp drivers mention outside the functions the
// tests call (get_rect, letterbox), so that those drivers compile where they lie (oracle/Makefile).  Declarations only: every
// builder and runtime call is a template that returns an empty value, and the linker drops the code that calls them
// (-Wl,--gc-sections), because nothing exported reaches it.
#pragma once
#include_next <NvInfer.h>

#ifndef TRTX_SHIM_V3_NVINFER_H
#define TRTX_SHIM_V3_NVINFER_H
namespace nvinfer1 {
enum class ActivationType : int32_t { kRELU = 0, kSIGMOID = 1, kTANH = 2, kLEAKY_RELU = 3 };
enum class ElementWiseOperation : int32_t { kSUM = 0, kPROD = 1, kMAX = 2, kMIN = 3, kSUB = 4, kDIV = 5, kPOW = 6 };
enum class PoolingType : int32_t { kMAX = 0, kAVERAGE = 1, kMAX_AVERAGE_BLEND = 2 };
enum class BuilderFlag : int32_t { kFP16 = 0, kINT8 = 1 };
enum class OptProfileSelector : int32_t { kMIN = 0, kOPT = 1, kMAX = 2 };
enum class NetworkDefinitionCreationFlag : int32_t { kEXPLICIT_BATCH = 0 };

// Every builder / network / layer / engine / runtime object of the drivers: the member names they call, returning nothing useful.
class ShimAny {
   public:
    struct Ret {  // converts to whatever the caller stores it in
        template <class T>
        operator T() const { return T(); }
        ShimAny* operator->() const { return nullptr; }
        ShimAny& operator*() const { return *static_cast<ShimAny*>(nullptr); }
        template <class T>
        bool operator==(const T&) const { return false; }
        template <class T>
        bool operator!=(const T&) const { return true; }
    };
#define TRTX_SHIM_ANY(name) \
    template <class... A>   \
    Ret name(A&&...) const { return Ret(); }
    TRTX_SHIM_ANY(addActivation) TRTX_SHIM_ANY(addConcatenation) TRTX_SHIM_ANY(addConvolutionNd)
    TRTX_SHIM_ANY(addDeconvolutionNd) TRTX_SHIM_ANY(addElementWise) TRTX_SHIM_ANY(addInput)
    TRTX_SHIM_ANY(addOptimizationProfile) TRTX_SHIM_ANY(addPaddingNd) TRTX_SHIM_ANY(addPoolingNd) TRTX_SHIM_ANY(addScale)
    TRTX_SHIM_ANY(addPluginV2) TRTX_SHIM_ANY(buildEngineWithConfig) TRTX_SHIM_ANY(createBuilderConfig)
    TRTX_SHIM_ANY(createExecutionContext) TRTX_SHIM_ANY(createOptimizationProfile) TRTX_SHIM_ANY(createNetworkV2)
    TRTX_SHIM_ANY(deserializeCudaEngine) TRTX_SHIM_ANY(destroy) TRTX_SHIM_ANY(markOutput) TRTX_SHIM_ANY(serialize)
    TRTX_SHIM_ANY(setAlpha) TRTX_SHIM_ANY(setDimensions) TRTX_SHIM_ANY(setFlag) TRTX_SHIM_ANY(setMaxBatchSize)
    TRTX_SHIM_ANY(setMaxWorkspaceSize) TRTX_SHIM_ANY(setName) TRTX_SHIM_ANY(setNbGroups) TRTX_SHIM_ANY(setOptimizationProfile)
    TRTX_SHIM_ANY(setPaddingNd) TRTX_SHIM_ANY(setStrideNd) TRTX_SHIM_ANY(setInt8Calibrator) TRTX_SHIM_ANY(enqueue)
    TRTX_SHIM_ANY(enqueueV2) TRTX_SHIM_ANY(getBindingIndex) TRTX_SHIM_ANY(getNbBindings) TRTX_SHIM_ANY(getEngine)
    TRTX_SHIM_ANY(setBindingDimensions)
#undef TRTX_SHIM_ANY
    ITensor* getOutput(int) const { return nullptr; }
    Dims getDimensions() const { return Dims(); }
    void* data() const { return nullptr; }
    size_t size() const { return 0; }
};
class ITensor : public ShimAny {};
using IBuilder = ShimAny;
using IBuilderConfig = ShimAny;
using ICudaEngine = ShimAny;
using IExecutionContext = ShimAny;
using IHostMemory = ShimAny;
using IRuntime = ShimAny;
using IOptimizationProfile = ShimAny;
using IConvolutionLayer = ShimAny;
using IDeconvolutionLayer = ShimAny;
using IActivationLayer = ShimAny;
using IPoolingLayer = ShimAny;
using IElementWiseLayer = ShimAny;
using IConcatenationLayer = ShimAny;
using IPaddingLayer = ShimAny;
using IPluginV2Layer = ShimAny;
using IShimScaleLayer = ShimAny;
class IInt8Calibrator {
   public:
    virtual ~IInt8Calibrator() {}
    virtual int32_t getBatchSize() const TRTX_NX = 0;
    virtual bool getBatch(void* bindings[], const char* names[], int32_t nbBindings) TRTX_NX = 0;
    virtual const void* readCalibrationCache(size_t& length) TRTX_NX = 0;
    virtual void writeCalibrationCache(const void* ptr, size_t length) TRTX_NX = 0;
};
class IInt8EntropyCalibrator2 : public IInt8Calibrator {};
inline ShimAny* createInferBuilder(ILogger&) { return nullptr; }
inline ShimAny* createInferRuntime(ILogger&) { return nullptr; }
}  // namespace nvinfer1
// the drivers' network and its scale layers are the shim's (the mock's INetworkDefinition serves the plugin headers)
#define INetworkDefinition ShimAny
#define IScaleLayer IShimScaleLayer
#endif
