// SHIM, not TensorRT -- TEST INFRASTRUCTURE.  tests/mock_trt/NvInfer.h (the plugin interfaces) plus the engine and runtime
// types that the YOLO cls drivers name outside the functions the tests call: declarations and null factories only, no behaviour.
#pragma once
#include_next <NvInfer.h>

#ifndef TRTX_SHIM_CLS_NVINFER_H
#define TRTX_SHIM_CLS_NVINFER_H
namespace nvinfer1 {
class IHostMemory {
   public:
    virtual ~IHostMemory() {}
    virtual void* data() const TRTX_NX { return nullptr; }
    virtual size_t size() const TRTX_NX { return 0; }
    virtual void destroy() TRTX_NX {}
};
class IExecutionContext {
   public:
    virtual ~IExecutionContext() {}
    virtual bool enqueue(int32_t, void* const*, cudaStream_t, cudaEvent_t*) TRTX_NX { return false; }
    virtual bool enqueueV2(void* const*, cudaStream_t, cudaEvent_t*) TRTX_NX { return false; }
    virtual void destroy() TRTX_NX {}
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
    virtual void destroy() TRTX_NX {}
};
class IBuilderConfig {
   public:
    virtual ~IBuilderConfig() {}
    virtual void destroy() TRTX_NX {}
};
class IBuilder {
   public:
    virtual ~IBuilder() {}
    virtual IBuilderConfig* createBuilderConfig() TRTX_NX { return nullptr; }
    virtual void destroy() TRTX_NX {}
};
class IInt8Calibrator {
   public:
    virtual ~IInt8Calibrator() {}
    virtual int32_t getBatchSize() const TRTX_NX = 0;
    virtual bool getBatch(void* bindings[], const char* names[], int32_t nbBindings) TRTX_NX = 0;
    virtual const void* readCalibrationCache(size_t& length) TRTX_NX = 0;
    virtual void writeCalibrationCache(const void* ptr, size_t length) TRTX_NX = 0;
};
class IInt8EntropyCalibrator2 : public IInt8Calibrator {};
inline IBuilder* createInferBuilder(ILogger&) TRTX_NX { return nullptr; }
inline IRuntime* createInferRuntime(ILogger&) TRTX_NX { return nullptr; }
}  // namespace nvinfer1
#endif
