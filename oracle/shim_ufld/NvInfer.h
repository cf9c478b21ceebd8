// SHIM, not TensorRT -- TEST INFRASTRUCTURE.  tests/mock_trt/NvInfer.h plus the builder, engine and runtime names that UFLD's
// driver (ufld/lane_det.cpp, ufld/common.hpp) mentions outside argmax and softmax_mul: declarations and null factories only,
// no behaviour.  The mock's INetworkDefinition declares only addScale; this one replaces it.
#pragma once
#define INetworkDefinition TrtxMockNetworkDefinition
#include_next <NvInfer.h>
#undef INetworkDefinition

#ifndef TRTX_SHIM_UFLD_NVINFER_H
#define TRTX_SHIM_UFLD_NVINFER_H
namespace nvinfer1 {
enum class ActivationType : int32_t { kRELU = 0 };
enum class PoolingType : int32_t { kMAX = 0 };
enum class ElementWiseOperation : int32_t { kSUM = 0 };
enum class MatrixOperation : int32_t { kNONE = 0, kTRANSPOSE = 1 };
enum class BuilderFlag : int32_t { kFP16 = 0 };
class ITensor {
   public:
    virtual void setName(const char*) TRTX_NX {}
    virtual Dims getDimensions() const TRTX_NX { return Dims{}; }
};
class IConvolutionLayer : public ILayer {
   public:
    virtual void setStride(DimsHW) TRTX_NX {}
    virtual void setPadding(DimsHW) TRTX_NX {}
    virtual void setNbGroups(int32_t) TRTX_NX {}
};
class IActivationLayer : public ILayer {};
class IPoolingLayer : public ILayer {
   public:
    virtual void setStride(DimsHW) TRTX_NX {}
    virtual void setPadding(DimsHW) TRTX_NX {}
};
class IShuffleLayer : public ILayer {
   public:
    virtual void setReshapeDimensions(Dims) TRTX_NX {}
};
class IConstantLayer : public ILayer {};
class IMatrixMultiplyLayer : public ILayer {};
class IElementWiseLayer : public ILayer {};
class INetworkDefinition {
   public:
    virtual ITensor* addInput(const char*, DataType, Dims) TRTX_NX = 0;
    virtual IScaleLayer* addScale(ITensor&, ScaleMode, Weights, Weights, Weights) TRTX_NX = 0;
    virtual IConvolutionLayer* addConvolution(ITensor&, int32_t, DimsHW, Weights, Weights) TRTX_NX = 0;
    virtual IActivationLayer* addActivation(ITensor&, ActivationType) TRTX_NX = 0;
    virtual IPoolingLayer* addPooling(ITensor&, PoolingType, DimsHW) TRTX_NX = 0;
    virtual IShuffleLayer* addShuffle(ITensor&) TRTX_NX = 0;
    virtual IConstantLayer* addConstant(Dims, Weights) TRTX_NX = 0;
    virtual IMatrixMultiplyLayer* addMatrixMultiply(ITensor&, MatrixOperation, ITensor&, MatrixOperation) TRTX_NX = 0;
    virtual IElementWiseLayer* addElementWise(ITensor&, ITensor&, ElementWiseOperation) TRTX_NX = 0;
    virtual void markOutput(ITensor&) TRTX_NX = 0;
    virtual void destroy() TRTX_NX = 0;
};
class IHostMemory {
   public:
    virtual ~IHostMemory() {}
    virtual void* data() const TRTX_NX { return nullptr; }
    virtual size_t size() const TRTX_NX { return 0; }
    virtual void destroy() TRTX_NX {}
};
class ICudaEngine;
class IExecutionContext {
   public:
    virtual ~IExecutionContext() {}
    virtual const ICudaEngine& getEngine() const TRTX_NX = 0;
    virtual bool enqueue(int32_t, void* const*, cudaStream_t, cudaEvent_t*) TRTX_NX { return false; }
};
class ICudaEngine {
   public:
    virtual ~ICudaEngine() {}
    virtual int32_t getNbBindings() const TRTX_NX { return 0; }
    virtual int32_t getBindingIndex(const char*) const TRTX_NX { return -1; }
    virtual IExecutionContext* createExecutionContext() TRTX_NX { return nullptr; }
    virtual IHostMemory* serialize() const TRTX_NX { return nullptr; }
    virtual void destroy() TRTX_NX {}
};
class IRuntime {
   public:
    virtual ~IRuntime() {}
    virtual ICudaEngine* deserializeCudaEngine(const void*, size_t) TRTX_NX { return nullptr; }
};
class IBuilderConfig {
   public:
    virtual ~IBuilderConfig() {}
    virtual void setMaxWorkspaceSize(size_t) TRTX_NX {}
    virtual void setFlag(BuilderFlag) TRTX_NX {}
};
class IBuilder {
   public:
    virtual ~IBuilder() {}
    virtual INetworkDefinition* createNetworkV2(uint32_t) TRTX_NX { return nullptr; }
    virtual IBuilderConfig* createBuilderConfig() TRTX_NX { return nullptr; }
    virtual void setMaxBatchSize(int32_t) TRTX_NX {}
    virtual bool platformHasFastFp16() const TRTX_NX { return false; }
    virtual ICudaEngine* buildEngineWithConfig(INetworkDefinition&, IBuilderConfig&) TRTX_NX { return nullptr; }
    virtual void destroy() TRTX_NX {}
};
inline IBuilder* createInferBuilder(ILogger&) TRTX_NX { return nullptr; }
inline IRuntime* createInferRuntime(ILogger&) TRTX_NX { return nullptr; }
}  // namespace nvinfer1
#endif
