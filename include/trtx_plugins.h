/*
 * trtx_plugins.h -- header-only TensorRT adapters for libtrtx_hot.so (the C ABI of include/trtx_hot.h).
 *
 * Same plugin names / versions / creator fields / serialization layouts as the reference plugins, so an engine
 * builder that does  getPluginRegistry()->getPluginCreator("YoloLayer_TRT", "1")  (yolov8/src/block.cpp:263,
 * yolov5/src/model.cpp:247), ("Decode_TRT", "1") (retinaface/retina_r50.cpp:204) or instantiates the rcnn plugin
 * classes by header (rcnn/rcnn.cpp:134,142,188,195) links this library instead of the reference's libmyplugins.so.
 *
 * Primary surface: IPluginV2DynamicExt (explicit batch; the interface TensorRT 10 / Blackwell requires -- the
 * reference's own template is yolov3-spp/yololayer.h:58-121).  Legacy adapters: IPluginV2IOExt for the YOLO /
 * RetinaFace builders that still use implicit batch (yolov8/plugin/yololayer.h:7) and IPluginV2Ext for rcnn
 * (rcnn/BatchedNmsPlugin.h:30).  Every enqueue() forwards to one C-ABI call; no state is mutated, nothing is
 * allocated or synchronised, the return value is the C ABI's (0 = success).
 *
 * Compile against the real <NvInfer.h>; this repository's tests compile it against tests/mock_trt/NvInfer.h
 * (interface declarations only) because the build image has no TensorRT.
 * Define TRTX_REGISTER_PLUGINS in exactly one translation unit to emit the REGISTER_TENSORRT_PLUGIN statics.
 */
#ifndef TRTX_PLUGINS_H
#define TRTX_PLUGINS_H

#include <NvInfer.h>

#include <cstring>
#include <string>
#include <vector>

#include "trtx_hot.h"

#if NV_TENSORRT_MAJOR >= 8
#define TRTX_NOEXCEPT noexcept
#define TRTX_CONST_ENQUEUE const
#else
#define TRTX_NOEXCEPT
#define TRTX_CONST_ENQUEUE
#endif

namespace trtx {

namespace detail {
template <typename T>
inline void write(char*& b, const T& v) {
    std::memcpy(b, &v, sizeof(T));
    b += sizeof(T);
}
template <typename T>
inline void read(const char*& b, T& v) {
    std::memcpy(&v, b, sizeof(T));
    b += sizeof(T);
}
// trtx_rpn_decode & co. answer a NULL / zero-sized workspace with the required size (> 0) and launch nothing
// (the reference idiom, rcnn/RpnNms.cu:63-80): inside enqueue that is a failure, not a success.
inline int rcnn_rc(int64_t rc) { return rc == 0 ? 0 : (rc < 0 ? (int)-rc : TRTX_ERR_WORKSPACE); }
}  // namespace detail

// ================================================================================================
// YoloLayer_TRT core (shared by the DynamicExt and IOExt adapters)
// ================================================================================================
struct YoloCore {
    trtx_yolo_params p{};
    int thread_count = 256;  // serialized by the reference (yololayer.cu:80); meaningless here, kept for layout
    std::string ns;

    // yolov8: fields of YoloLayerPlugin(classCount, nKpt, kptThr, W, H, maxOut, seg, pose, obb, strides...) (yololayer.cu:28-45)
    void init_v8(int nc, int nk, float kthr, int w, int h, int max_out, bool seg, bool pose, bool obb, const int* strides, int n) {
        trtx_yolo_params_init_v8(&p, nc, w, h, max_out, strides, n);
        p.num_kpts = nk;
        p.kpt_thresh = kthr;
        p.is_seg = seg;
        p.is_pose = pose;
        p.is_obb = obb;
    }
    // yolov5: YoloLayerPlugin(classCount, netW, netH, maxOut, is_seg, vector<YoloKernel>) (yolov5 yololayer.cu:22-39).
    // yolov7 and YOLOP: the same arithmetic with 6-float rows, YoloLayerPlugin(classCount, netW, netH, maxOut,
    // vector<YoloKernel>) (yolov7/plugin/yololayer.cu:21-36, yolop/yololayer.cu:28-44), det_floats = kV7Floats.
    static constexpr int kV5Floats = 38, kV7Floats = 6;
    void init_v5(int nc, int w, int h, int max_out, bool seg, const void* kernels /* {int w,h; float a[6]}[] */, int n,
                 int det_floats = kV5Floats) {
        std::memset(&p, 0, sizeof(p));
        p.variant = TRTX_YOLO_V5;
        p.num_classes = nc;
        p.net_w = w;
        p.net_h = h;
        p.max_out = max_out;
        p.det_floats = det_floats;
        p.num_levels = n;
        p.is_seg = seg;
        p.gate = 0.1f;
        const char* k = static_cast<const char*>(kernels);
        for (int i = 0; i < n && i < TRTX_MAX_LEVELS; ++i, k += 32) {
            std::memcpy(&p.grid_w[i], k, 4);
            std::memcpy(&p.grid_h[i], k + 4, 4);
            std::memcpy(p.anchors[i], k + 8, 24);
        }
    }
    int out_elems() const { return 1 + p.max_out * p.det_floats; }  // yololayer.cu:107-111
    // the yolov7 / YOLOP blob: the yolov5 one without the is_seg byte (yolov7/plugin/yololayer.cu:62-77,
    // yolop/yololayer.cu:81-101)
    bool v7_layout() const { return p.variant == TRTX_YOLO_V5 && p.det_floats == kV7Floats; }

    size_t serial_size() const {
        if (p.variant == TRTX_YOLO_V8) return 4 * 8 + 4 * (size_t)p.num_levels + 3;  // yololayer.cu:97-101
        return (v7_layout() ? 24 : 25) + 32 * (size_t)p.num_levels;                 // yolov5 yololayer.cu:72-83
    }
    void serialize(void* buffer) const {
        char* d = static_cast<char*>(buffer);
        if (p.variant == TRTX_YOLO_V8) {
            detail::write(d, p.num_classes);
            detail::write(d, p.num_kpts);
            detail::write(d, p.kpt_thresh);
            detail::write(d, thread_count);
            detail::write(d, p.net_w);
            detail::write(d, p.net_h);
            detail::write(d, p.max_out);
            detail::write(d, p.num_levels);
            for (int i = 0; i < p.num_levels; ++i) detail::write(d, p.strides[i]);
            detail::write(d, (bool)p.is_seg);
            detail::write(d, (bool)p.is_pose);
            detail::write(d, (bool)p.is_obb);
        } else {
            detail::write(d, p.num_classes);
            detail::write(d, thread_count);
            detail::write(d, p.num_levels);
            detail::write(d, p.net_w);
            detail::write(d, p.net_h);
            detail::write(d, p.max_out);
            if (!v7_layout()) detail::write(d, (bool)p.is_seg);
            for (int i = 0; i < p.num_levels; ++i) {
                detail::write(d, p.grid_w[i]);
                detail::write(d, p.grid_h[i]);
                for (int j = 0; j < 6; ++j) detail::write(d, p.anchors[i][j]);
            }
        }
    }
    // returns false on a malformed blob (the reference asserts, yololayer.cu:72).  variant TRTX_YOLO_V5 with v7 = true reads
    // the yolov7 / YOLOP layout.
    bool deserialize(const void* data, size_t length, int variant, bool v7 = false) {
        const char* d = static_cast<const char*>(data);
        if (variant == TRTX_YOLO_V8) {
            if (length < 35) return false;
            int nc, nk, tc, w, h, mo, ns;
            float kt;
            detail::read(d, nc);
            detail::read(d, nk);
            detail::read(d, kt);
            detail::read(d, tc);
            detail::read(d, w);
            detail::read(d, h);
            detail::read(d, mo);
            detail::read(d, ns);
            if (ns <= 0 || ns > TRTX_MAX_LEVELS || length != 32 + 4 * (size_t)ns + 3) return false;
            int st[TRTX_MAX_LEVELS];
            for (int i = 0; i < ns; ++i) detail::read(d, st[i]);
            bool seg, pose, obb;
            detail::read(d, seg);
            detail::read(d, pose);
            detail::read(d, obb);
            init_v8(nc, nk, kt, w, h, mo, seg, pose, obb, st, ns);
            thread_count = tc;
        } else {
            const size_t header = v7 ? 24 : 25;
            if (length < header) return false;
            int nc, tc, kc, w, h, mo;
            bool seg = false;
            detail::read(d, nc);
            detail::read(d, tc);
            detail::read(d, kc);
            detail::read(d, w);
            detail::read(d, h);
            detail::read(d, mo);
            if (!v7) detail::read(d, seg);
            if (kc <= 0 || kc > TRTX_MAX_LEVELS || length != header + 32 * (size_t)kc) return false;
            init_v5(nc, w, h, mo, seg, d, kc, v7 ? kV7Floats : kV5Floats);
            thread_count = tc;
        }
        return true;
    }
    // createPlugin field parsing: v8 "combinedInfo" (block.cpp:264-296); "netinfo" + "kernels" with a netinfo of 5 ints
    // (yolov5, model.cpp:249-277) or of 4 (yolov7, yolov7/src/block.cpp:224-241: 6-float rows); YOLOP's "netdata" +
    // "yolodata1".."yolodataN" (yolop/common.hpp:318-356).  Every field's declared length is checked before it is read,
    // except netdata's, whose fourth int lies past the declared 3 (below).
    bool from_fields(const nvinfer1::PluginFieldCollection* fc) {
        if (!fc || fc->nbFields <= 0 || !fc->fields) return false;
        const nvinfer1::PluginField* f = fc->fields;
        for (int i = 0; i < fc->nbFields; ++i)
            if (!f[i].name || !f[i].data) return false;
        if (fc->nbFields == 1 && std::strcmp(f[0].name, "combinedInfo") == 0) {
            const int* ci = static_cast<const int*>(f[0].data);
            const int n = f[0].length - 9;
            if (n <= 0 || n > TRTX_MAX_LEVELS) return false;
            init_v8(ci[0], ci[1], (float)ci[2], ci[3], ci[4], ci[5], ci[6] != 0, ci[7] != 0, ci[8] != 0, ci + 9, n);
            return true;
        }
        if (fc->nbFields == 2 && std::strcmp(f[0].name, "netinfo") == 0 && std::strcmp(f[1].name, "kernels") == 0) {
            const int* ni = static_cast<const int*>(f[0].data);
            const int n = f[1].length;
            if (f[0].length < 4 || n <= 0 || n > TRTX_MAX_LEVELS) return false;
            if (f[0].length == 4)
                init_v5(ni[0], ni[1], ni[2], ni[3], false, f[1].data, n, kV7Floats);
            else
                init_v5(ni[0], ni[1], ni[2], ni[3], ni[4] != 0, f[1].data, n);
            return true;
        }
        return yolop_fields(fc);
    }
    // YOLOP, parsed as yolop/yololayer.cu:289-320 parses it: fields in any order; "netdata" = {classCount, netW, netH,
    // maxOut}, declared with length 3 by YOLOP's builder (common.hpp:328-336) but read as 4 ints, as the reference reads
    // it; "yolodata1".."yolodata3" = {grid w, grid h, 6 anchors} as ints, each converted to a float anchor, yolodataK into
    // kernel slot 3 - K (the builder passes its stride-32 head first).  Rejected: a field of another name, a netdata
    // shorter than 3, a yolodataK whose length is not 8, a K outside 1..3 or given twice, a missing field.
    bool yolop_fields(const nvinfer1::PluginFieldCollection* fc) {
        constexpr int n = 3;  // the reference's yolo_kernels(3)
        if (fc->nbFields != n + 1) return false;
        const int* nd = nullptr;
        char kernels[n][32];
        bool seen[n] = {};
        for (int i = 0; i < fc->nbFields; ++i) {
            const nvinfer1::PluginField& f = fc->fields[i];
            if (std::strcmp(f.name, "netdata") == 0) {
                if (nd || f.length < 3) return false;
                nd = static_cast<const int*>(f.data);
                continue;
            }
            const int k = std::strncmp(f.name, "yolodata", 8) == 0 && f.name[9] == '\0' ? f.name[8] - '0' : 0;
            if (k < 1 || k > n || seen[k - 1] || f.length != 8) return false;
            seen[k - 1] = true;
            const int* v = static_cast<const int*>(f.data);
            char* o = kernels[n - k];
            std::memcpy(o, v, 8);  // grid w, h
            for (int j = 0; j < 6; ++j) {
                const float a = (float)v[2 + j];
                std::memcpy(o + 8 + 4 * j, &a, 4);
            }
        }
        if (!nd) return false;
        init_v5(nd[0], nd[1], nd[2], nd[3], false, kernels, n, kV7Floats);
        return true;
    }
};

// ------------------------------------------------------------------------------------------------
// Primary: IPluginV2DynamicExt (cf. yolov3-spp/yololayer.h:58-121)
// ------------------------------------------------------------------------------------------------
class YoloLayerPluginDynamic : public nvinfer1::IPluginV2DynamicExt {
   public:
    explicit YoloLayerPluginDynamic(const YoloCore& c) : core_(c) {}
    int getNbOutputs() const TRTX_NOEXCEPT override { return 1; }
    nvinfer1::DimsExprs getOutputDimensions(int, const nvinfer1::DimsExprs* inputs, int, nvinfer1::IExprBuilder& eb) TRTX_NOEXCEPT override {
        nvinfer1::DimsExprs de;
        de.nbDims = 2;
        de.d[0] = inputs[0].d[0];                   // batch (may be dynamic)
        de.d[1] = eb.constant(core_.out_elems());   // maxOut * sizeof(Detection)/4 + 1 (yolov3-spp/yololayer.cu:83-92)
        return de;
    }
    int initialize() TRTX_NOEXCEPT override { return 0; }
    void terminate() TRTX_NOEXCEPT override {}
    // TensorRT asks with the MAXIMUM dims of the optimisation profile; the layout is derived from the tensor dims exactly
    // as enqueue derives it, and the size grows with batch and grid, so what is granted here covers every runtime shape.
    size_t getWorkspaceSize(const nvinfer1::PluginTensorDesc* in, int, const nvinfer1::PluginTensorDesc*, int) const TRTX_NOEXCEPT override {
        const trtx_yolo_params p = bound_params(in);
        return trtx_yolo_workspace_size(&p, in[0].dims.d[0] > 0 ? in[0].dims.d[0] : 1);
    }
    int enqueue(const nvinfer1::PluginTensorDesc* in, const nvinfer1::PluginTensorDesc*, const void* const* inputs, void* const* outputs,
                void* workspace, cudaStream_t stream) TRTX_NOEXCEPT override {
        const trtx_yolo_params p = bound_params(in);  // per-call copy: enqueue never mutates the plugin
        const int batch = in[0].dims.d[0];
        return trtx_yolo_decode_enqueue(&p, batch, inputs, static_cast<float*>(outputs[0]), workspace,
                                        trtx_yolo_workspace_size(&p, batch), stream);
    }
    size_t getSerializationSize() const TRTX_NOEXCEPT override { return core_.serial_size(); }
    void serialize(void* buffer) const TRTX_NOEXCEPT override { core_.serialize(buffer); }
    bool supportsFormatCombination(int pos, const nvinfer1::PluginTensorDesc* io, int nbInputs, int) TRTX_NOEXCEPT override {
        if (io[pos].format != nvinfer1::TensorFormat::kLINEAR) return false;
        if (pos < nbInputs)  // fp32 is the reference's only mode (yololayer.h:32-35); fp16 inputs halve the HBM traffic
            return (io[pos].type == nvinfer1::DataType::kFLOAT || io[pos].type == nvinfer1::DataType::kHALF) && io[pos].type == io[0].type;
        return io[pos].type == nvinfer1::DataType::kFLOAT;
    }
    const char* getPluginType() const TRTX_NOEXCEPT override { return "YoloLayer_TRT"; }
    const char* getPluginVersion() const TRTX_NOEXCEPT override { return "1"; }
    void destroy() TRTX_NOEXCEPT override { delete this; }
    nvinfer1::IPluginV2DynamicExt* clone() const TRTX_NOEXCEPT override { return new YoloLayerPluginDynamic(core_); }
    void setPluginNamespace(const char* n) TRTX_NOEXCEPT override { core_.ns = n ? n : ""; }
    const char* getPluginNamespace() const TRTX_NOEXCEPT override { return core_.ns.c_str(); }
    nvinfer1::DataType getOutputDataType(int, const nvinfer1::DataType*, int) const TRTX_NOEXCEPT override { return nvinfer1::DataType::kFLOAT; }
    void attachToContext(cudnnContext*, cublasContext*, nvinfer1::IGpuAllocator*) TRTX_NOEXCEPT override {}
    void detachFromContext() TRTX_NOEXCEPT override {}
    void configurePlugin(const nvinfer1::DynamicPluginTensorDesc*, int, const nvinfer1::DynamicPluginTensorDesc*, int) TRTX_NOEXCEPT override {}
    const YoloCore& core() const { return core_; }

   private:
    // grid and input type from the bound tensors (yolov3-spp/yololayer.cu:207-216)
    trtx_yolo_params bound_params(const nvinfer1::PluginTensorDesc* in) const {
        trtx_yolo_params p = core_.p;
        for (int i = 0; i < p.num_levels; ++i) {
            if (in[i].dims.nbDims == 4) {
                p.grid_h[i] = in[i].dims.d[2];
                p.grid_w[i] = in[i].dims.d[3];
            }
            p.in_dtype = in[i].type == nvinfer1::DataType::kHALF ? TRTX_F16 : TRTX_F32;
        }
        return p;
    }
    YoloCore core_;
};

// ------------------------------------------------------------------------------------------------
// Legacy: IPluginV2IOExt, the interface of yolov8/plugin/yololayer.h:7 and yolov5/plugin/yololayer.h:10
// ------------------------------------------------------------------------------------------------
class YoloLayerPluginIOExt : public nvinfer1::IPluginV2IOExt {
   public:
    explicit YoloLayerPluginIOExt(const YoloCore& c) : core_(c) {}
    int getNbOutputs() const TRTX_NOEXCEPT override { return 1; }
    nvinfer1::Dims getOutputDimensions(int, const nvinfer1::Dims*, int) TRTX_NOEXCEPT override {
        return nvinfer1::Dims3(core_.out_elems(), 1, 1);  // yololayer.cu:107-111
    }
    int initialize() TRTX_NOEXCEPT override { return 0; }
    void terminate() TRTX_NOEXCEPT override {}
    size_t getWorkspaceSize(int maxBatchSize) const TRTX_NOEXCEPT override { return trtx_yolo_workspace_size(&core_.p, maxBatchSize); }
    int enqueue(int batchSize, const void* const* inputs, void* TRTX_CONST_ENQUEUE* outputs, void* workspace, cudaStream_t stream) TRTX_NOEXCEPT override {
        return trtx_yolo_decode_enqueue(&core_.p, batchSize, inputs, static_cast<float*>(outputs[0]), workspace,
                                        trtx_yolo_workspace_size(&core_.p, batchSize), stream);
    }
    size_t getSerializationSize() const TRTX_NOEXCEPT override { return core_.serial_size(); }
    void serialize(void* buffer) const TRTX_NOEXCEPT override { core_.serialize(buffer); }
    bool supportsFormatCombination(int pos, const nvinfer1::PluginTensorDesc* io, int, int) const TRTX_NOEXCEPT override {
        return io[pos].format == nvinfer1::TensorFormat::kLINEAR && io[pos].type == nvinfer1::DataType::kFLOAT;  // yololayer.h:32-35
    }
    const char* getPluginType() const TRTX_NOEXCEPT override { return "YoloLayer_TRT"; }
    const char* getPluginVersion() const TRTX_NOEXCEPT override { return "1"; }
    void destroy() TRTX_NOEXCEPT override { delete this; }
    nvinfer1::IPluginV2IOExt* clone() const TRTX_NOEXCEPT override { return new YoloLayerPluginIOExt(core_); }
    void setPluginNamespace(const char* n) TRTX_NOEXCEPT override { core_.ns = n ? n : ""; }
    const char* getPluginNamespace() const TRTX_NOEXCEPT override { return core_.ns.c_str(); }
    nvinfer1::DataType getOutputDataType(int, const nvinfer1::DataType*, int) const TRTX_NOEXCEPT override { return nvinfer1::DataType::kFLOAT; }
    bool isOutputBroadcastAcrossBatch(int, const bool*, int) const TRTX_NOEXCEPT override { return false; }
    bool canBroadcastInputAcrossBatch(int) const TRTX_NOEXCEPT override { return false; }
    void attachToContext(cudnnContext*, cublasContext*, nvinfer1::IGpuAllocator*) TRTX_NOEXCEPT override {}
    void configurePlugin(const nvinfer1::PluginTensorDesc*, int, const nvinfer1::PluginTensorDesc*, int) TRTX_NOEXCEPT override {}
    void detachFromContext() TRTX_NOEXCEPT override {}

   private:
    YoloCore core_;
};

// Creator for "YoloLayer_TRT"/"1".  Dynamic = true hands out IPluginV2DynamicExt objects (explicit-batch builders,
// yolo11/src/model.cpp:143-149); false the IPluginV2IOExt ones (implicit-batch builders).
template <bool Dynamic>
class YoloPluginCreatorT : public nvinfer1::IPluginCreator {
   public:
    YoloPluginCreatorT() { fc_.nbFields = 0; fc_.fields = nullptr; }
    const char* getPluginName() const TRTX_NOEXCEPT override { return "YoloLayer_TRT"; }
    const char* getPluginVersion() const TRTX_NOEXCEPT override { return "1"; }
    const nvinfer1::PluginFieldCollection* getFieldNames() TRTX_NOEXCEPT override { return &fc_; }
    nvinfer1::IPluginV2* createPlugin(const char*, const nvinfer1::PluginFieldCollection* fc) TRTX_NOEXCEPT override {
        YoloCore c;
        if (!c.from_fields(fc)) return nullptr;  // the reference asserts (yololayer.cu:340-341); we refuse instead
        return make(c);
    }
    nvinfer1::IPluginV2* deserializePlugin(const char*, const void* data, size_t len) TRTX_NOEXCEPT override {
        YoloCore c;
        // the three layouts differ in size modulo 4: v8 = 35 + 4n bytes (3), v5 = 25 + 32n (1), yolov7 / YOLOP = 24 + 32n (0)
        if (!c.deserialize(data, len, TRTX_YOLO_V8) && !c.deserialize(data, len, TRTX_YOLO_V5) &&
            !c.deserialize(data, len, TRTX_YOLO_V5, true))
            return nullptr;
        return make(c);
    }
    void setPluginNamespace(const char* n) TRTX_NOEXCEPT override { ns_ = n ? n : ""; }
    const char* getPluginNamespace() const TRTX_NOEXCEPT override { return ns_.c_str(); }

   private:
    nvinfer1::IPluginV2* make(YoloCore& c) const {
        c.ns = ns_;
        if (Dynamic) return new YoloLayerPluginDynamic(c);
        return new YoloLayerPluginIOExt(c);
    }
    std::string ns_;
    nvinfer1::PluginFieldCollection fc_;
};
using YoloPluginCreator = YoloPluginCreatorT<true>;
using YoloPluginCreatorImplicitBatch = YoloPluginCreatorT<false>;

// ================================================================================================
// Decode_TRT (RetinaFace), retinaface/decode.h:22-107.  The reference serializes nothing and bakes 480x640 in
// (decode.h:16-17); here the input size is plugin state (8 bytes), an empty blob means the reference's default.
// ================================================================================================
class DecodePluginDynamic : public nvinfer1::IPluginV2DynamicExt {
   public:
    explicit DecodePluginDynamic(int in_h = 480, int in_w = 640) { p_.in_h = in_h; p_.in_w = in_w; p_.gate = 0.02f; }
    int getNbOutputs() const TRTX_NOEXCEPT override { return 1; }
    nvinfer1::DimsExprs getOutputDimensions(int, const nvinfer1::DimsExprs* inputs, int, nvinfer1::IExprBuilder& eb) TRTX_NOEXCEPT override {
        nvinfer1::DimsExprs de;
        de.nbDims = 2;
        de.d[0] = inputs[0].d[0];
        de.d[1] = eb.constant(1 + trtx_retina_total_priors(&p_) * 15);  // decode.cu:33-41
        return de;
    }
    int initialize() TRTX_NOEXCEPT override { return 0; }
    void terminate() TRTX_NOEXCEPT override {}
    size_t getWorkspaceSize(const nvinfer1::PluginTensorDesc* in, int, const nvinfer1::PluginTensorDesc*, int) const TRTX_NOEXCEPT override {
        return trtx_retina_workspace_size(&p_, in[0].dims.d[0] > 0 ? in[0].dims.d[0] : 1);
    }
    int enqueue(const nvinfer1::PluginTensorDesc* in, const nvinfer1::PluginTensorDesc*, const void* const* inputs, void* const* outputs,
                void* workspace, cudaStream_t stream) TRTX_NOEXCEPT override {
        const int batch = in[0].dims.d[0];
        trtx_retina_params p = p_;  // per-call copy: enqueue never mutates the plugin
        p.in_dtype = in[0].type == nvinfer1::DataType::kHALF ? TRTX_F16 : TRTX_F32;
        return trtx_retina_decode_enqueue(&p, batch, inputs, static_cast<float*>(outputs[0]), workspace,
                                          trtx_retina_workspace_size(&p, batch), stream);
    }
    size_t getSerializationSize() const TRTX_NOEXCEPT override { return 8; }
    void serialize(void* buffer) const TRTX_NOEXCEPT override {
        char* d = static_cast<char*>(buffer);
        detail::write(d, p_.in_h);
        detail::write(d, p_.in_w);
    }
    bool supportsFormatCombination(int pos, const nvinfer1::PluginTensorDesc* io, int nbInputs, int) TRTX_NOEXCEPT override {
        if (io[pos].format != nvinfer1::TensorFormat::kLINEAR) return false;
        if (pos < nbInputs)  // the three heads: all fp32 (the reference's only mode) or all fp16, as YoloLayerPluginDynamic
            return (io[pos].type == nvinfer1::DataType::kFLOAT || io[pos].type == nvinfer1::DataType::kHALF) && io[pos].type == io[0].type;
        return io[pos].type == nvinfer1::DataType::kFLOAT;
    }
    const char* getPluginType() const TRTX_NOEXCEPT override { return "Decode_TRT"; }
    const char* getPluginVersion() const TRTX_NOEXCEPT override { return "1"; }
    void destroy() TRTX_NOEXCEPT override { delete this; }
    nvinfer1::IPluginV2DynamicExt* clone() const TRTX_NOEXCEPT override {
        auto* c = new DecodePluginDynamic(p_.in_h, p_.in_w);
        c->ns_ = ns_;
        return c;
    }
    void setPluginNamespace(const char* n) TRTX_NOEXCEPT override { ns_ = n ? n : ""; }
    const char* getPluginNamespace() const TRTX_NOEXCEPT override { return ns_.c_str(); }
    nvinfer1::DataType getOutputDataType(int, const nvinfer1::DataType*, int) const TRTX_NOEXCEPT override { return nvinfer1::DataType::kFLOAT; }
    void attachToContext(cudnnContext*, cublasContext*, nvinfer1::IGpuAllocator*) TRTX_NOEXCEPT override {}
    void detachFromContext() TRTX_NOEXCEPT override {}
    void configurePlugin(const nvinfer1::DynamicPluginTensorDesc*, int, const nvinfer1::DynamicPluginTensorDesc*, int) TRTX_NOEXCEPT override {}

   private:
    trtx_retina_params p_{};
    std::string ns_;
};

class DecodePluginCreator : public nvinfer1::IPluginCreator {
   public:
    DecodePluginCreator() { fc_.nbFields = 0; fc_.fields = nullptr; }
    const char* getPluginName() const TRTX_NOEXCEPT override { return "Decode_TRT"; }
    const char* getPluginVersion() const TRTX_NOEXCEPT override { return "1"; }
    const nvinfer1::PluginFieldCollection* getFieldNames() TRTX_NOEXCEPT override { return &fc_; }
    // no fields in the reference (retina_r50.cpp:205-206); optional "input_hw" = {h, w} makes the size runtime
    nvinfer1::IPluginV2* createPlugin(const char*, const nvinfer1::PluginFieldCollection* fc) TRTX_NOEXCEPT override {
        int h = 480, w = 640;
        if (fc && fc->nbFields == 1 && fc->fields[0].name && std::strcmp(fc->fields[0].name, "input_hw") == 0 && fc->fields[0].length == 2) {
            h = static_cast<const int*>(fc->fields[0].data)[0];
            w = static_cast<const int*>(fc->fields[0].data)[1];
        }
        auto* p = new DecodePluginDynamic(h, w);
        p->setPluginNamespace(ns_.c_str());
        return p;
    }
    nvinfer1::IPluginV2* deserializePlugin(const char*, const void* data, size_t len) TRTX_NOEXCEPT override {
        int h = 480, w = 640;
        if (len == 8) {
            const char* d = static_cast<const char*>(data);
            detail::read(d, h);
            detail::read(d, w);
        } else if (len != 0) {
            return nullptr;
        }
        auto* p = new DecodePluginDynamic(h, w);
        p->setPluginNamespace(ns_.c_str());
        return p;
    }
    void setPluginNamespace(const char* n) TRTX_NOEXCEPT override { ns_ = n ? n : ""; }
    const char* getPluginNamespace() const TRTX_NOEXCEPT override { return ns_.c_str(); }

   private:
    std::string ns_;
    nvinfer1::PluginFieldCollection fc_;
};

// ================================================================================================
// Faster R-CNN plugins: IPluginV2Ext with the reference's constructors (rcnn/*Plugin.h), names "RpnDecode",
// "RpnNms", "PredictorDecode", "BatchedNms", version "1", namespace "".  Implicit batch, fp32 linear only
// (the *PluginIOExt classes below also take fp16 feature maps / masks / scores and deltas).
// ================================================================================================
class RcnnPluginBase : public nvinfer1::IPluginV2Ext {
   public:
    bool supportsFormat(nvinfer1::DataType t, nvinfer1::PluginFormat f) const TRTX_NOEXCEPT override {
        return t == nvinfer1::DataType::kFLOAT && f == nvinfer1::PluginFormat::kLINEAR;  // BatchedNmsPlugin.h:98-100
    }
    int initialize() TRTX_NOEXCEPT override { return 0; }
    void terminate() TRTX_NOEXCEPT override {}
    void destroy() TRTX_NOEXCEPT override { delete this; }
    const char* getPluginVersion() const TRTX_NOEXCEPT override { return "1"; }
    const char* getPluginNamespace() const TRTX_NOEXCEPT override { return ""; }
    void setPluginNamespace(const char*) TRTX_NOEXCEPT override {}
    nvinfer1::DataType getOutputDataType(int, const nvinfer1::DataType*, int) const TRTX_NOEXCEPT override { return nvinfer1::DataType::kFLOAT; }
    bool isOutputBroadcastAcrossBatch(int, const bool*, int) const TRTX_NOEXCEPT override { return false; }
    bool canBroadcastInputAcrossBatch(int) const TRTX_NOEXCEPT override { return false; }
};

class RpnDecodePlugin : public RcnnPluginBase {
   public:
    RpnDecodePlugin(int top_n, const std::vector<float>& anchors, float stride, size_t image_height, size_t image_width)
        : top_n_(top_n), anchors_(anchors), stride_(stride), height_(0), width_(0), image_height_(image_height), image_width_(image_width) {}
    RpnDecodePlugin(int top_n, const std::vector<float>& anchors, float stride, size_t height, size_t width, size_t image_height, size_t image_width)
        : top_n_(top_n), anchors_(anchors), stride_(stride), height_(height), width_(width), image_height_(image_height), image_width_(image_width) {}
    RpnDecodePlugin(const void* data, size_t) {  // RpnDecodePlugin.h:42-58
        const char* d = static_cast<const char*>(data);
        detail::read(d, top_n_);
        size_t n;
        detail::read(d, n);
        anchors_.resize(n);
        for (size_t i = 0; i < n; ++i) detail::read(d, anchors_[i]);
        detail::read(d, stride_);
        detail::read(d, height_);
        detail::read(d, width_);
        detail::read(d, image_height_);
        detail::read(d, image_width_);
    }
    const char* getPluginType() const TRTX_NOEXCEPT override { return "RpnDecode"; }
    int getNbOutputs() const TRTX_NOEXCEPT override { return 2; }
    nvinfer1::Dims getOutputDimensions(int index, const nvinfer1::Dims*, int) TRTX_NOEXCEPT override { return nvinfer1::Dims2(top_n_, index == 1 ? 4 : 1); }
    size_t getWorkspaceSize(int maxBatchSize) const TRTX_NOEXCEPT override {
        return (size_t)trtx_rpn_decode(maxBatchSize, nullptr, nullptr, nullptr, nullptr, (int)height_, (int)width_, (int)image_height_,
                                       (int)image_width_, stride_, anchors_.data(), (int)anchors_.size() / 4, top_n_, nullptr, 0, nullptr);
    }
    int enqueue(int batchSize, const void* const* inputs, void* TRTX_CONST_ENQUEUE* outputs, void* workspace, cudaStream_t stream) TRTX_NOEXCEPT override {
        const int64_t rc = trtx_rpn_decode(batchSize, static_cast<const float*>(inputs[0]), static_cast<const float*>(inputs[1]),
                                           static_cast<float*>(outputs[0]), static_cast<float*>(outputs[1]), (int)height_, (int)width_,
                                           (int)image_height_, (int)image_width_, stride_, anchors_.data(), (int)anchors_.size() / 4,
                                           top_n_, workspace, getWorkspaceSize(batchSize), stream);
        return detail::rcnn_rc(rc);
    }
    size_t getSerializationSize() const TRTX_NOEXCEPT override {
        return sizeof(top_n_) + sizeof(size_t) + sizeof(float) * anchors_.size() + sizeof(stride_) + 4 * sizeof(size_t);
    }
    void serialize(void* buffer) const TRTX_NOEXCEPT override {
        char* d = static_cast<char*>(buffer);
        detail::write(d, top_n_);
        detail::write(d, anchors_.size());
        for (float v : anchors_) detail::write(d, v);
        detail::write(d, stride_);
        detail::write(d, height_);
        detail::write(d, width_);
        detail::write(d, image_height_);
        detail::write(d, image_width_);
    }
    void configurePlugin(const nvinfer1::Dims* inputDims, int, const nvinfer1::Dims*, int, const nvinfer1::DataType*, const nvinfer1::DataType*,
                         const bool*, const bool*, nvinfer1::PluginFormat, int) TRTX_NOEXCEPT override {
        height_ = inputDims[0].d[1];  // RpnDecodePlugin.h:148-157: scores dims {A, H, W}
        width_ = inputDims[0].d[2];
    }
    nvinfer1::IPluginV2Ext* clone() const TRTX_NOEXCEPT override {
        return new RpnDecodePlugin(top_n_, anchors_, stride_, height_, width_, image_height_, image_width_);
    }

   private:
    int top_n_;
    std::vector<float> anchors_;
    float stride_;
    size_t height_, width_, image_height_, image_width_;
};

class RpnNmsPlugin : public RcnnPluginBase {
   public:
    RpnNmsPlugin(float nms_thresh, int post_nms_topk, size_t pre_nms_topk = 1) : thresh_(nms_thresh), post_(post_nms_topk), pre_(pre_nms_topk) {}
    RpnNmsPlugin(const void* data, size_t) {  // RpnNmsPlugin.h:36-41
        const char* d = static_cast<const char*>(data);
        detail::read(d, thresh_);
        detail::read(d, post_);
        detail::read(d, pre_);
    }
    const char* getPluginType() const TRTX_NOEXCEPT override { return "RpnNms"; }
    int getNbOutputs() const TRTX_NOEXCEPT override { return 1; }
    nvinfer1::Dims getOutputDimensions(int, const nvinfer1::Dims*, int) TRTX_NOEXCEPT override { return nvinfer1::Dims2(post_, 4); }
    size_t getWorkspaceSize(int maxBatchSize) const TRTX_NOEXCEPT override {
        return (size_t)trtx_rpn_nms(maxBatchSize, nullptr, nullptr, nullptr, (int)pre_, post_, thresh_, nullptr, 0, nullptr);
    }
    int enqueue(int batchSize, const void* const* inputs, void* TRTX_CONST_ENQUEUE* outputs, void* workspace, cudaStream_t stream) TRTX_NOEXCEPT override {
        const int64_t rc = trtx_rpn_nms(batchSize, static_cast<const float*>(inputs[0]), static_cast<const float*>(inputs[1]),
                                        static_cast<float*>(outputs[0]), (int)pre_, post_, thresh_, workspace, getWorkspaceSize(batchSize), stream);
        return detail::rcnn_rc(rc);
    }
    size_t getSerializationSize() const TRTX_NOEXCEPT override { return sizeof(thresh_) + sizeof(post_) + sizeof(pre_); }
    void serialize(void* buffer) const TRTX_NOEXCEPT override {
        char* d = static_cast<char*>(buffer);
        detail::write(d, thresh_);
        detail::write(d, post_);
        detail::write(d, pre_);
    }
    void configurePlugin(const nvinfer1::Dims* inputDims, int, const nvinfer1::Dims*, int, const nvinfer1::DataType*, const nvinfer1::DataType*,
                         const bool*, const bool*, nvinfer1::PluginFormat, int) TRTX_NOEXCEPT override {
        pre_ = inputDims[0].d[0];
    }
    nvinfer1::IPluginV2Ext* clone() const TRTX_NOEXCEPT override { return new RpnNmsPlugin(thresh_, post_, pre_); }

   private:
    float thresh_;
    int post_;
    size_t pre_;
};

// rcnn/RoiAlignPlugin.h:27-170
class RoiAlignPlugin : public RcnnPluginBase {
   public:
    RoiAlignPlugin(int pooler_resolution, float spatial_scale, int sampling_ratio, int num_proposals, int out_channels,
                   int feature_h = 0, int feature_w = 0)
        : pooler_(pooler_resolution), scale_(spatial_scale), sampling_(sampling_ratio), proposals_(num_proposals),
          channels_(out_channels), fh_(feature_h), fw_(feature_w) {}
    RoiAlignPlugin(const void* data, size_t) {  // RoiAlignPlugin.h:37-46
        const char* d = static_cast<const char*>(data);
        detail::read(d, pooler_);
        detail::read(d, scale_);
        detail::read(d, sampling_);
        detail::read(d, proposals_);
        detail::read(d, channels_);
        detail::read(d, fh_);
        detail::read(d, fw_);
    }
    const char* getPluginType() const TRTX_NOEXCEPT override { return "RoiAlign"; }
    int getNbOutputs() const TRTX_NOEXCEPT override { return 1; }
    nvinfer1::Dims getOutputDimensions(int, const nvinfer1::Dims*, int) TRTX_NOEXCEPT override {
        return nvinfer1::Dims4(proposals_, channels_, pooler_, pooler_);
    }
    size_t getWorkspaceSize(int) const TRTX_NOEXCEPT override { return 0; }
    int enqueue(int batchSize, const void* const* inputs, void* TRTX_CONST_ENQUEUE* outputs, void*, cudaStream_t stream) TRTX_NOEXCEPT override {
        return trtx_roi_align(batchSize, static_cast<const float*>(inputs[0]), static_cast<const float*>(inputs[1]),
                              static_cast<float*>(outputs[0]), pooler_, scale_, sampling_, proposals_, channels_, fh_, fw_, stream);
    }
    size_t getSerializationSize() const TRTX_NOEXCEPT override { return 6 * sizeof(int) + sizeof(float); }
    void serialize(void* buffer) const TRTX_NOEXCEPT override {
        char* d = static_cast<char*>(buffer);
        detail::write(d, pooler_);
        detail::write(d, scale_);
        detail::write(d, sampling_);
        detail::write(d, proposals_);
        detail::write(d, channels_);
        detail::write(d, fh_);
        detail::write(d, fw_);
    }
    void configurePlugin(const nvinfer1::Dims* inputDims, int, const nvinfer1::Dims*, int, const nvinfer1::DataType*, const nvinfer1::DataType*,
                         const bool*, const bool*, nvinfer1::PluginFormat, int) TRTX_NOEXCEPT override {
        fh_ = inputDims[1].d[1];  // RoiAlignPlugin.h:151-152
        fw_ = inputDims[1].d[2];
    }
    nvinfer1::IPluginV2Ext* clone() const TRTX_NOEXCEPT override {
        return new RoiAlignPlugin(pooler_, scale_, sampling_, proposals_, channels_, fh_, fw_);
    }

   private:
    int pooler_;
    float scale_;
    int sampling_, proposals_, channels_, fh_, fw_;
};

// rcnn/MaskRcnnInferencePlugin.h:27-140
class MaskRcnnInferencePlugin : public RcnnPluginBase {
   public:
    MaskRcnnInferencePlugin(int detections_per_im, int output_size, int num_classes = 1)
        : dets_(detections_per_im), size_(output_size), classes_(num_classes) {}
    MaskRcnnInferencePlugin(const void* data, size_t) {  // MaskRcnnInferencePlugin.h:32-37
        const char* d = static_cast<const char*>(data);
        detail::read(d, dets_);
        detail::read(d, size_);
        detail::read(d, classes_);
    }
    const char* getPluginType() const TRTX_NOEXCEPT override { return "MaskRcnnInference"; }
    int getNbOutputs() const TRTX_NOEXCEPT override { return 1; }
    nvinfer1::Dims getOutputDimensions(int, const nvinfer1::Dims*, int) TRTX_NOEXCEPT override { return nvinfer1::Dims4(dets_, 1, size_, size_); }
    size_t getWorkspaceSize(int) const TRTX_NOEXCEPT override { return 0; }
    int enqueue(int batchSize, const void* const* inputs, void* TRTX_CONST_ENQUEUE* outputs, void*, cudaStream_t stream) TRTX_NOEXCEPT override {
        return trtx_mask_rcnn_inference(batchSize, static_cast<const float*>(inputs[0]), static_cast<const float*>(inputs[1]),
                                        static_cast<float*>(outputs[0]), dets_, size_, classes_, stream);
    }
    size_t getSerializationSize() const TRTX_NOEXCEPT override { return 3 * sizeof(int); }
    void serialize(void* buffer) const TRTX_NOEXCEPT override {
        char* d = static_cast<char*>(buffer);
        detail::write(d, dets_);
        detail::write(d, size_);
        detail::write(d, classes_);
    }
    void configurePlugin(const nvinfer1::Dims* inputDims, int, const nvinfer1::Dims*, int, const nvinfer1::DataType*, const nvinfer1::DataType*,
                         const bool*, const bool*, nvinfer1::PluginFormat, int) TRTX_NOEXCEPT override {
        classes_ = inputDims[1].d[1];  // MaskRcnnInferencePlugin.h:119
    }
    nvinfer1::IPluginV2Ext* clone() const TRTX_NOEXCEPT override { return new MaskRcnnInferencePlugin(dets_, size_, classes_); }

   private:
    int dets_, size_, classes_;
};

class PredictorDecodePlugin : public RcnnPluginBase {
   public:
    PredictorDecodePlugin(unsigned num_boxes, unsigned image_height, unsigned image_width, const std::vector<float>& w)
        : num_boxes_(num_boxes), num_classes_(0), image_height_(image_height), image_width_(image_width), w_(w) {}
    PredictorDecodePlugin(unsigned num_boxes, unsigned num_classes, unsigned image_height, unsigned image_width, const std::vector<float>& w)
        : num_boxes_(num_boxes), num_classes_(num_classes), image_height_(image_height), image_width_(image_width), w_(w) {}
    PredictorDecodePlugin(const void* data, size_t) {  // PredictorDecodePlugin.h:40-54
        const char* d = static_cast<const char*>(data);
        detail::read(d, num_boxes_);
        detail::read(d, num_classes_);
        detail::read(d, image_height_);
        detail::read(d, image_width_);
        size_t n;
        detail::read(d, n);
        w_.resize(n);
        for (size_t i = 0; i < n; ++i) detail::read(d, w_[i]);
    }
    const char* getPluginType() const TRTX_NOEXCEPT override { return "PredictorDecode"; }
    int getNbOutputs() const TRTX_NOEXCEPT override { return 3; }
    nvinfer1::Dims getOutputDimensions(int index, const nvinfer1::Dims*, int) TRTX_NOEXCEPT override { return nvinfer1::Dims2(num_boxes_, index == 1 ? 4 : 1); }
    size_t getWorkspaceSize(int maxBatchSize) const TRTX_NOEXCEPT override {
        return (size_t)trtx_predictor_decode(maxBatchSize, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, (int)num_boxes_, (int)num_classes_,
                                             (int)image_height_, (int)image_width_, w_.data(), nullptr, 0, nullptr);
    }
    int enqueue(int batchSize, const void* const* inputs, void* TRTX_CONST_ENQUEUE* outputs, void* workspace, cudaStream_t stream) TRTX_NOEXCEPT override {
        if (w_.size() < 4) return TRTX_ERR_INVALID;
        const int64_t rc = trtx_predictor_decode(batchSize, static_cast<const float*>(inputs[0]), static_cast<const float*>(inputs[1]),
                                                 static_cast<const float*>(inputs[2]), static_cast<float*>(outputs[0]), static_cast<float*>(outputs[1]),
                                                 static_cast<float*>(outputs[2]), (int)num_boxes_, (int)num_classes_, (int)image_height_,
                                                 (int)image_width_, w_.data(), workspace, getWorkspaceSize(batchSize), stream);
        return detail::rcnn_rc(rc);
    }
    size_t getSerializationSize() const TRTX_NOEXCEPT override { return 4 * sizeof(unsigned) + sizeof(size_t) + sizeof(float) * w_.size(); }
    void serialize(void* buffer) const TRTX_NOEXCEPT override {
        char* d = static_cast<char*>(buffer);
        detail::write(d, num_boxes_);
        detail::write(d, num_classes_);
        detail::write(d, image_height_);
        detail::write(d, image_width_);
        detail::write(d, w_.size());
        for (float v : w_) detail::write(d, v);
    }
    void configurePlugin(const nvinfer1::Dims* inputDims, int, const nvinfer1::Dims*, int, const nvinfer1::DataType*, const nvinfer1::DataType*,
                         const bool*, const bool*, nvinfer1::PluginFormat, int) TRTX_NOEXCEPT override {
        num_classes_ = inputDims[0].d[1];  // scores dims {N, C, 1, 1}
    }
    nvinfer1::IPluginV2Ext* clone() const TRTX_NOEXCEPT override {
        return new PredictorDecodePlugin(num_boxes_, num_classes_, image_height_, image_width_, w_);
    }

   private:
    unsigned num_boxes_, num_classes_, image_height_, image_width_;
    std::vector<float> w_;
};

class BatchedNmsPlugin : public RcnnPluginBase {
   public:
    BatchedNmsPlugin(int nms_method, float nms_thresh, int detections_per_im, size_t count = 1)
        : method_(nms_method), thresh_(nms_thresh), dets_(detections_per_im), count_(count) {}
    BatchedNmsPlugin(const void* data, size_t) {  // BatchedNmsPlugin.h:38-44
        const char* d = static_cast<const char*>(data);
        detail::read(d, method_);
        detail::read(d, thresh_);
        detail::read(d, dets_);
        detail::read(d, count_);
    }
    const char* getPluginType() const TRTX_NOEXCEPT override { return "BatchedNms"; }
    int getNbOutputs() const TRTX_NOEXCEPT override { return 3; }
    nvinfer1::Dims getOutputDimensions(int index, const nvinfer1::Dims*, int) TRTX_NOEXCEPT override { return nvinfer1::Dims2(dets_, index == 1 ? 4 : 1); }
    size_t getWorkspaceSize(int maxBatchSize) const TRTX_NOEXCEPT override {
        return (size_t)trtx_batched_nms(method_, maxBatchSize, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, (int)count_, dets_, thresh_, nullptr, 0, nullptr);
    }
    int enqueue(int batchSize, const void* const* inputs, void* TRTX_CONST_ENQUEUE* outputs, void* workspace, cudaStream_t stream) TRTX_NOEXCEPT override {
        const int64_t rc = trtx_batched_nms(method_, batchSize, static_cast<const float*>(inputs[0]), static_cast<const float*>(inputs[1]),
                                            static_cast<const float*>(inputs[2]), static_cast<float*>(outputs[0]), static_cast<float*>(outputs[1]),
                                            static_cast<float*>(outputs[2]), (int)count_, dets_, thresh_, workspace, getWorkspaceSize(batchSize), stream);
        return detail::rcnn_rc(rc);
    }
    size_t getSerializationSize() const TRTX_NOEXCEPT override { return sizeof(method_) + sizeof(thresh_) + sizeof(dets_) + sizeof(count_); }
    void serialize(void* buffer) const TRTX_NOEXCEPT override {
        char* d = static_cast<char*>(buffer);
        detail::write(d, method_);
        detail::write(d, thresh_);
        detail::write(d, dets_);
        detail::write(d, count_);
    }
    void configurePlugin(const nvinfer1::Dims* inputDims, int, const nvinfer1::Dims*, int, const nvinfer1::DataType*, const nvinfer1::DataType*,
                         const bool*, const bool*, nvinfer1::PluginFormat, int) TRTX_NOEXCEPT override {
        count_ = inputDims[0].d[0];  // BatchedNmsPlugin.h:148-157
    }
    nvinfer1::IPluginV2Ext* clone() const TRTX_NOEXCEPT override { return new BatchedNmsPlugin(method_, thresh_, dets_, count_); }

   private:
    int method_;
    float thresh_;
    int dets_;
    size_t count_;
};

template <typename P>
class RcnnCreator : public nvinfer1::IPluginCreator {
   public:
    explicit RcnnCreator(const char* name) : name_(name) {}
    const char* getPluginName() const TRTX_NOEXCEPT override { return name_; }
    const char* getPluginVersion() const TRTX_NOEXCEPT override { return "1"; }
    const char* getPluginNamespace() const TRTX_NOEXCEPT override { return ""; }
    void setPluginNamespace(const char*) TRTX_NOEXCEPT override {}
    const nvinfer1::PluginFieldCollection* getFieldNames() TRTX_NOEXCEPT override { return nullptr; }
    nvinfer1::IPluginV2* createPlugin(const char*, const nvinfer1::PluginFieldCollection*) TRTX_NOEXCEPT override { return nullptr; }  // as the reference
    nvinfer1::IPluginV2* deserializePlugin(const char*, const void* data, size_t len) TRTX_NOEXCEPT override { return new P(data, len); }

   private:
    const char* name_;
};
struct RpnDecodePluginCreator : RcnnCreator<RpnDecodePlugin> { RpnDecodePluginCreator() : RcnnCreator("RpnDecode") {} };
struct RpnNmsPluginCreator : RcnnCreator<RpnNmsPlugin> { RpnNmsPluginCreator() : RcnnCreator("RpnNms") {} };
struct PredictorDecodePluginCreator : RcnnCreator<PredictorDecodePlugin> { PredictorDecodePluginCreator() : RcnnCreator("PredictorDecode") {} };
struct BatchedNmsPluginCreator : RcnnCreator<BatchedNmsPlugin> { BatchedNmsPluginCreator() : RcnnCreator("BatchedNms") {} };
struct RoiAlignPluginCreator : RcnnCreator<RoiAlignPlugin> { RoiAlignPluginCreator() : RcnnCreator("RoiAlign") {} };
struct MaskRcnnInferencePluginCreator : RcnnCreator<MaskRcnnInferencePlugin> { MaskRcnnInferencePluginCreator() : RcnnCreator("MaskRcnnInference") {} };

// ------------------------------------------------------------------------------------------------
// RoiAlign, MaskRcnnInference, RpnDecode and PredictorDecode for an FP16 engine.  Each needs fp32 tensors next to half
// ones (proposals, class indices, fp32 outputs), which IPluginV2Ext::supportsFormat (one type for every tensor) cannot say;
// IPluginV2IOExt::supportsFormatCombination can.  Same plugin names, version, constructor arguments and namespace as the
// IPluginV2Ext classes above, which stay as they are.  The element type TensorRT chose arrives in configurePlugin, is
// carried through clone() and is appended to the serialized blob as one int32 (TRTX_F32 | TRTX_F16); a blob of the
// reference's length deserializes as fp32, a blob of any other length is refused.
// Exercised against tests/mock_trt only: how a real TensorRT builder drives these four classes is NOT verified.
// ------------------------------------------------------------------------------------------------
class RcnnIOExtBase : public nvinfer1::IPluginV2IOExt {
   public:
    int initialize() TRTX_NOEXCEPT override { return 0; }
    void terminate() TRTX_NOEXCEPT override {}
    void destroy() TRTX_NOEXCEPT override { delete this; }
    size_t getWorkspaceSize(int) const TRTX_NOEXCEPT override { return 0; }
    int getNbOutputs() const TRTX_NOEXCEPT override { return 1; }
    const char* getPluginVersion() const TRTX_NOEXCEPT override { return "1"; }
    const char* getPluginNamespace() const TRTX_NOEXCEPT override { return ""; }
    void setPluginNamespace(const char*) TRTX_NOEXCEPT override {}
    bool isOutputBroadcastAcrossBatch(int, const bool*, int) const TRTX_NOEXCEPT override { return false; }
    bool canBroadcastInputAcrossBatch(int) const TRTX_NOEXCEPT override { return false; }
    void attachToContext(cudnnContext*, cublasContext*, nvinfer1::IGpuAllocator*) TRTX_NOEXCEPT override {}
    void detachFromContext() TRTX_NOEXCEPT override {}
    int dtype() const { return dtype_; }

   protected:
    static bool float_or_half(nvinfer1::DataType t) { return t == nvinfer1::DataType::kFLOAT || t == nvinfer1::DataType::kHALF; }
    // the trailing int32 of a blob that is 4 bytes longer than the reference's; false: an unknown type
    bool read_dtype(const char* d, size_t length, size_t reference_length) {
        if (length == reference_length) return true;
        int32_t v;
        detail::read(d, v);
        if (v != TRTX_F32 && v != TRTX_F16) return false;
        dtype_ = v;
        return true;
    }
    int32_t dtype_ = TRTX_F32;  // of the half-capable inputs: the feature map / the masks / the scores and deltas
};

class RoiAlignPluginIOExt : public RcnnIOExtBase {
   public:
    RoiAlignPluginIOExt(int pooler_resolution, float spatial_scale, int sampling_ratio, int num_proposals, int out_channels,
                        int feature_h = 0, int feature_w = 0)
        : pooler_(pooler_resolution), scale_(spatial_scale), sampling_(sampling_ratio), proposals_(num_proposals),
          channels_(out_channels), fh_(feature_h), fw_(feature_w) {}
    RoiAlignPluginIOExt(const void* data, size_t length) {  // RoiAlignPlugin.h:37-46 (+ the element type)
        if (length != kReferenceBlob && length != kReferenceBlob + sizeof(int32_t)) {
            valid_ = false;
            return;
        }
        const char* d = static_cast<const char*>(data);
        detail::read(d, pooler_);
        detail::read(d, scale_);
        detail::read(d, sampling_);
        detail::read(d, proposals_);
        detail::read(d, channels_);
        detail::read(d, fh_);
        detail::read(d, fw_);
        valid_ = read_dtype(d, length, kReferenceBlob);
    }
    bool valid() const { return valid_; }  // false: the blob had neither the reference's length nor that + 4
    const char* getPluginType() const TRTX_NOEXCEPT override { return "RoiAlign"; }
    nvinfer1::Dims getOutputDimensions(int, const nvinfer1::Dims*, int) TRTX_NOEXCEPT override {
        return nvinfer1::Dims4(proposals_, channels_, pooler_, pooler_);
    }
    // proposals fp32; features fp32 or fp16; the bins in the features' type
    bool supportsFormatCombination(int pos, const nvinfer1::PluginTensorDesc* io, int, int) const TRTX_NOEXCEPT override {
        if (io[pos].format != nvinfer1::TensorFormat::kLINEAR) return false;
        if (pos == 0) return io[0].type == nvinfer1::DataType::kFLOAT;
        if (pos == 1) return float_or_half(io[1].type);
        return io[pos].type == io[1].type;
    }
    nvinfer1::DataType getOutputDataType(int, const nvinfer1::DataType* inputTypes, int nbInputs) const TRTX_NOEXCEPT override {
        return nbInputs > 1 ? inputTypes[1] : nvinfer1::DataType::kFLOAT;
    }
    void configurePlugin(const nvinfer1::PluginTensorDesc* in, int, const nvinfer1::PluginTensorDesc*, int) TRTX_NOEXCEPT override {
        fh_ = in[1].dims.d[1];  // RoiAlignPlugin.h:151-152
        fw_ = in[1].dims.d[2];
        dtype_ = in[1].type == nvinfer1::DataType::kHALF ? TRTX_F16 : TRTX_F32;
    }
    int enqueue(int batchSize, const void* const* inputs, void* TRTX_CONST_ENQUEUE* outputs, void*, cudaStream_t stream) TRTX_NOEXCEPT override {
        return trtx_roi_align_typed(dtype_, batchSize, static_cast<const float*>(inputs[0]), inputs[1], outputs[0], pooler_, scale_,
                                    sampling_, proposals_, channels_, fh_, fw_, stream);
    }
    size_t getSerializationSize() const TRTX_NOEXCEPT override { return kReferenceBlob + sizeof(int32_t); }
    void serialize(void* buffer) const TRTX_NOEXCEPT override {
        char* d = static_cast<char*>(buffer);
        detail::write(d, pooler_);
        detail::write(d, scale_);
        detail::write(d, sampling_);
        detail::write(d, proposals_);
        detail::write(d, channels_);
        detail::write(d, fh_);
        detail::write(d, fw_);
        detail::write(d, dtype_);
    }
    nvinfer1::IPluginV2IOExt* clone() const TRTX_NOEXCEPT override {
        auto* c = new RoiAlignPluginIOExt(pooler_, scale_, sampling_, proposals_, channels_, fh_, fw_);
        c->dtype_ = dtype_;
        return c;
    }

   private:
    static constexpr size_t kReferenceBlob = 6 * sizeof(int) + sizeof(float);
    int pooler_ = 0;
    float scale_ = 0.f;
    int sampling_ = 0, proposals_ = 0, channels_ = 0, fh_ = 0, fw_ = 0;
    bool valid_ = true;
};

class MaskRcnnInferencePluginIOExt : public RcnnIOExtBase {
   public:
    MaskRcnnInferencePluginIOExt(int detections_per_im, int output_size, int num_classes = 1)
        : dets_(detections_per_im), size_(output_size), classes_(num_classes) {}
    MaskRcnnInferencePluginIOExt(const void* data, size_t length) {  // MaskRcnnInferencePlugin.h:32-37 (+ the element type)
        if (length != kReferenceBlob && length != kReferenceBlob + sizeof(int32_t)) {
            valid_ = false;
            return;
        }
        const char* d = static_cast<const char*>(data);
        detail::read(d, dets_);
        detail::read(d, size_);
        detail::read(d, classes_);
        valid_ = read_dtype(d, length, kReferenceBlob);
    }
    bool valid() const { return valid_; }
    const char* getPluginType() const TRTX_NOEXCEPT override { return "MaskRcnnInference"; }
    nvinfer1::Dims getOutputDimensions(int, const nvinfer1::Dims*, int) TRTX_NOEXCEPT override { return nvinfer1::Dims4(dets_, 1, size_, size_); }
    // class indices fp32; masks fp32 or fp16; the probabilities fp32 (they feed trtx_rcnn_postprocess*)
    bool supportsFormatCombination(int pos, const nvinfer1::PluginTensorDesc* io, int, int) const TRTX_NOEXCEPT override {
        if (io[pos].format != nvinfer1::TensorFormat::kLINEAR) return false;
        if (pos == 1) return float_or_half(io[1].type);
        return io[pos].type == nvinfer1::DataType::kFLOAT;
    }
    nvinfer1::DataType getOutputDataType(int, const nvinfer1::DataType*, int) const TRTX_NOEXCEPT override { return nvinfer1::DataType::kFLOAT; }
    void configurePlugin(const nvinfer1::PluginTensorDesc* in, int, const nvinfer1::PluginTensorDesc*, int) TRTX_NOEXCEPT override {
        classes_ = in[1].dims.d[1];  // MaskRcnnInferencePlugin.h:119
        dtype_ = in[1].type == nvinfer1::DataType::kHALF ? TRTX_F16 : TRTX_F32;
    }
    int enqueue(int batchSize, const void* const* inputs, void* TRTX_CONST_ENQUEUE* outputs, void*, cudaStream_t stream) TRTX_NOEXCEPT override {
        return trtx_mask_rcnn_inference_typed(dtype_, batchSize, static_cast<const float*>(inputs[0]), inputs[1],
                                              static_cast<float*>(outputs[0]), dets_, size_, classes_, stream);
    }
    size_t getSerializationSize() const TRTX_NOEXCEPT override { return kReferenceBlob + sizeof(int32_t); }
    void serialize(void* buffer) const TRTX_NOEXCEPT override {
        char* d = static_cast<char*>(buffer);
        detail::write(d, dets_);
        detail::write(d, size_);
        detail::write(d, classes_);
        detail::write(d, dtype_);
    }
    nvinfer1::IPluginV2IOExt* clone() const TRTX_NOEXCEPT override {
        auto* c = new MaskRcnnInferencePluginIOExt(dets_, size_, classes_);
        c->dtype_ = dtype_;
        return c;
    }

   private:
    static constexpr size_t kReferenceBlob = 3 * sizeof(int);
    int dets_ = 0, size_ = 0, classes_ = 0;
    bool valid_ = true;
};

// RpnDecode and PredictorDecode for an FP16 engine: scores and deltas fp32 or fp16 (one type for both), PredictorDecode's
// proposals and every output fp32 (trtx_rpn_decode_typed / trtx_predictor_decode_typed).  Same names, version, constructor
// arguments and namespace as RpnDecodePlugin / PredictorDecodePlugin, same blob + the trailing int32 element type.
class RpnDecodePluginIOExt : public RcnnIOExtBase {
   public:
    RpnDecodePluginIOExt(int top_n, const std::vector<float>& anchors, float stride, size_t image_height, size_t image_width)
        : top_n_(top_n), anchors_(anchors), stride_(stride), height_(0), width_(0), image_height_(image_height), image_width_(image_width) {}
    RpnDecodePluginIOExt(int top_n, const std::vector<float>& anchors, float stride, size_t height, size_t width, size_t image_height,
                         size_t image_width)
        : top_n_(top_n), anchors_(anchors), stride_(stride), height_(height), width_(width), image_height_(image_height), image_width_(image_width) {}
    RpnDecodePluginIOExt(const void* data, size_t length) {  // RpnDecodePlugin.h:42-58 (+ the element type)
        const char* d = static_cast<const char*>(data);
        size_t n = 0;
        valid_ = length >= sizeof(top_n_) + sizeof(size_t);
        if (valid_) {
            detail::read(d, top_n_);
            detail::read(d, n);
            valid_ = n <= length / sizeof(float) &&
                     (length == reference_length(n) || length == reference_length(n) + sizeof(int32_t));
        }
        if (!valid_) return;
        anchors_.resize(n);
        for (size_t i = 0; i < n; ++i) detail::read(d, anchors_[i]);
        detail::read(d, stride_);
        detail::read(d, height_);
        detail::read(d, width_);
        detail::read(d, image_height_);
        detail::read(d, image_width_);
        valid_ = read_dtype(d, length, reference_length(n));
    }
    bool valid() const { return valid_; }  // false: the blob had neither the reference's length nor that + 4
    const char* getPluginType() const TRTX_NOEXCEPT override { return "RpnDecode"; }
    int getNbOutputs() const TRTX_NOEXCEPT override { return 2; }
    nvinfer1::Dims getOutputDimensions(int index, const nvinfer1::Dims*, int) TRTX_NOEXCEPT override { return nvinfer1::Dims2(top_n_, index == 1 ? 4 : 1); }
    size_t getWorkspaceSize(int maxBatchSize) const TRTX_NOEXCEPT override {
        return (size_t)trtx_rpn_decode_typed(dtype_, maxBatchSize, nullptr, nullptr, nullptr, nullptr, (int)height_, (int)width_,
                                             (int)image_height_, (int)image_width_, stride_, anchors_.data(), (int)anchors_.size() / 4,
                                             top_n_, nullptr, 0, nullptr);
    }
    // scores and deltas fp32 or fp16, one type; the scores and boxes fp32
    bool supportsFormatCombination(int pos, const nvinfer1::PluginTensorDesc* io, int nbInputs, int) const TRTX_NOEXCEPT override {
        if (io[pos].format != nvinfer1::TensorFormat::kLINEAR) return false;
        if (pos < nbInputs) return float_or_half(io[pos].type) && io[pos].type == io[0].type;
        return io[pos].type == nvinfer1::DataType::kFLOAT;
    }
    nvinfer1::DataType getOutputDataType(int, const nvinfer1::DataType*, int) const TRTX_NOEXCEPT override { return nvinfer1::DataType::kFLOAT; }
    void configurePlugin(const nvinfer1::PluginTensorDesc* in, int, const nvinfer1::PluginTensorDesc*, int) TRTX_NOEXCEPT override {
        height_ = in[0].dims.d[1];  // RpnDecodePlugin.h:148-157: scores dims {A, H, W}
        width_ = in[0].dims.d[2];
        dtype_ = in[0].type == nvinfer1::DataType::kHALF ? TRTX_F16 : TRTX_F32;
    }
    int enqueue(int batchSize, const void* const* inputs, void* TRTX_CONST_ENQUEUE* outputs, void* workspace, cudaStream_t stream) TRTX_NOEXCEPT override {
        const int64_t rc = trtx_rpn_decode_typed(dtype_, batchSize, inputs[0], inputs[1], static_cast<float*>(outputs[0]),
                                                 static_cast<float*>(outputs[1]), (int)height_, (int)width_, (int)image_height_,
                                                 (int)image_width_, stride_, anchors_.data(), (int)anchors_.size() / 4, top_n_, workspace,
                                                 getWorkspaceSize(batchSize), stream);
        return detail::rcnn_rc(rc);
    }
    size_t getSerializationSize() const TRTX_NOEXCEPT override { return reference_length(anchors_.size()) + sizeof(int32_t); }
    void serialize(void* buffer) const TRTX_NOEXCEPT override {
        char* d = static_cast<char*>(buffer);
        detail::write(d, top_n_);
        detail::write(d, anchors_.size());
        for (float v : anchors_) detail::write(d, v);
        detail::write(d, stride_);
        detail::write(d, height_);
        detail::write(d, width_);
        detail::write(d, image_height_);
        detail::write(d, image_width_);
        detail::write(d, dtype_);
    }
    nvinfer1::IPluginV2IOExt* clone() const TRTX_NOEXCEPT override {
        auto* c = new RpnDecodePluginIOExt(top_n_, anchors_, stride_, height_, width_, image_height_, image_width_);
        c->dtype_ = dtype_;
        return c;
    }

   private:
    static size_t reference_length(size_t num_anchor_floats) {
        return sizeof(int) + sizeof(size_t) + sizeof(float) * num_anchor_floats + sizeof(float) + 4 * sizeof(size_t);
    }
    int top_n_ = 0;
    std::vector<float> anchors_;
    float stride_ = 0.f;
    size_t height_ = 0, width_ = 0, image_height_ = 0, image_width_ = 0;
    bool valid_ = true;
};

class PredictorDecodePluginIOExt : public RcnnIOExtBase {
   public:
    PredictorDecodePluginIOExt(unsigned num_boxes, unsigned image_height, unsigned image_width, const std::vector<float>& w)
        : num_boxes_(num_boxes), num_classes_(0), image_height_(image_height), image_width_(image_width), w_(w) {}
    PredictorDecodePluginIOExt(unsigned num_boxes, unsigned num_classes, unsigned image_height, unsigned image_width, const std::vector<float>& w)
        : num_boxes_(num_boxes), num_classes_(num_classes), image_height_(image_height), image_width_(image_width), w_(w) {}
    PredictorDecodePluginIOExt(const void* data, size_t length) {  // PredictorDecodePlugin.h:40-54 (+ the element type)
        const char* d = static_cast<const char*>(data);
        size_t n = 0;
        valid_ = length >= 4 * sizeof(unsigned) + sizeof(size_t);
        if (valid_) {
            detail::read(d, num_boxes_);
            detail::read(d, num_classes_);
            detail::read(d, image_height_);
            detail::read(d, image_width_);
            detail::read(d, n);
            valid_ = n <= length / sizeof(float) &&
                     (length == reference_length(n) || length == reference_length(n) + sizeof(int32_t));
        }
        if (!valid_) return;
        w_.resize(n);
        for (size_t i = 0; i < n; ++i) detail::read(d, w_[i]);
        valid_ = read_dtype(d, length, reference_length(n));
    }
    bool valid() const { return valid_; }  // false: the blob had neither the reference's length nor that + 4
    const char* getPluginType() const TRTX_NOEXCEPT override { return "PredictorDecode"; }
    int getNbOutputs() const TRTX_NOEXCEPT override { return 3; }
    nvinfer1::Dims getOutputDimensions(int index, const nvinfer1::Dims*, int) TRTX_NOEXCEPT override { return nvinfer1::Dims2(num_boxes_, index == 1 ? 4 : 1); }
    size_t getWorkspaceSize(int maxBatchSize) const TRTX_NOEXCEPT override {
        return (size_t)trtx_predictor_decode_typed(dtype_, maxBatchSize, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, (int)num_boxes_,
                                                   (int)num_classes_, (int)image_height_, (int)image_width_, w_.data(), nullptr, 0, nullptr);
    }
    // scores and deltas fp32 or fp16, one type; the proposals and the scores, boxes and classes fp32
    bool supportsFormatCombination(int pos, const nvinfer1::PluginTensorDesc* io, int, int) const TRTX_NOEXCEPT override {
        if (io[pos].format != nvinfer1::TensorFormat::kLINEAR) return false;
        if (pos < 2) return float_or_half(io[pos].type) && io[pos].type == io[0].type;
        return io[pos].type == nvinfer1::DataType::kFLOAT;
    }
    nvinfer1::DataType getOutputDataType(int, const nvinfer1::DataType*, int) const TRTX_NOEXCEPT override { return nvinfer1::DataType::kFLOAT; }
    void configurePlugin(const nvinfer1::PluginTensorDesc* in, int, const nvinfer1::PluginTensorDesc*, int) TRTX_NOEXCEPT override {
        num_classes_ = in[0].dims.d[1];  // scores dims {N, C, 1, 1}
        dtype_ = in[0].type == nvinfer1::DataType::kHALF ? TRTX_F16 : TRTX_F32;
    }
    int enqueue(int batchSize, const void* const* inputs, void* TRTX_CONST_ENQUEUE* outputs, void* workspace, cudaStream_t stream) TRTX_NOEXCEPT override {
        if (w_.size() < 4) return TRTX_ERR_INVALID;
        const int64_t rc = trtx_predictor_decode_typed(dtype_, batchSize, inputs[0], inputs[1], static_cast<const float*>(inputs[2]),
                                                       static_cast<float*>(outputs[0]), static_cast<float*>(outputs[1]),
                                                       static_cast<float*>(outputs[2]), (int)num_boxes_, (int)num_classes_, (int)image_height_,
                                                       (int)image_width_, w_.data(), workspace, getWorkspaceSize(batchSize), stream);
        return detail::rcnn_rc(rc);
    }
    size_t getSerializationSize() const TRTX_NOEXCEPT override { return reference_length(w_.size()) + sizeof(int32_t); }
    void serialize(void* buffer) const TRTX_NOEXCEPT override {
        char* d = static_cast<char*>(buffer);
        detail::write(d, num_boxes_);
        detail::write(d, num_classes_);
        detail::write(d, image_height_);
        detail::write(d, image_width_);
        detail::write(d, w_.size());
        for (float v : w_) detail::write(d, v);
        detail::write(d, dtype_);
    }
    nvinfer1::IPluginV2IOExt* clone() const TRTX_NOEXCEPT override {
        auto* c = new PredictorDecodePluginIOExt(num_boxes_, num_classes_, image_height_, image_width_, w_);
        c->dtype_ = dtype_;
        return c;
    }

   private:
    static size_t reference_length(size_t num_weights) { return 4 * sizeof(unsigned) + sizeof(size_t) + sizeof(float) * num_weights; }
    unsigned num_boxes_ = 0, num_classes_ = 0, image_height_ = 0, image_width_ = 0;
    std::vector<float> w_;
    bool valid_ = true;
};

// deserializePlugin for the four classes above: a blob of neither accepted length is refused (nullptr)
template <typename P>
class RcnnIOExtCreator : public nvinfer1::IPluginCreator {
   public:
    explicit RcnnIOExtCreator(const char* name) : name_(name) {}
    const char* getPluginName() const TRTX_NOEXCEPT override { return name_; }
    const char* getPluginVersion() const TRTX_NOEXCEPT override { return "1"; }
    const char* getPluginNamespace() const TRTX_NOEXCEPT override { return ""; }
    void setPluginNamespace(const char*) TRTX_NOEXCEPT override {}
    const nvinfer1::PluginFieldCollection* getFieldNames() TRTX_NOEXCEPT override { return nullptr; }
    nvinfer1::IPluginV2* createPlugin(const char*, const nvinfer1::PluginFieldCollection*) TRTX_NOEXCEPT override { return nullptr; }  // as the reference
    nvinfer1::IPluginV2* deserializePlugin(const char*, const void* data, size_t len) TRTX_NOEXCEPT override {
        P* p = new P(data, len);
        if (p->valid()) return p;
        delete p;
        return nullptr;
    }

   private:
    const char* name_;
};
struct RoiAlignPluginIOExtCreator : RcnnIOExtCreator<RoiAlignPluginIOExt> { RoiAlignPluginIOExtCreator() : RcnnIOExtCreator("RoiAlign") {} };
struct MaskRcnnInferencePluginIOExtCreator : RcnnIOExtCreator<MaskRcnnInferencePluginIOExt> { MaskRcnnInferencePluginIOExtCreator() : RcnnIOExtCreator("MaskRcnnInference") {} };
struct RpnDecodePluginIOExtCreator : RcnnIOExtCreator<RpnDecodePluginIOExt> { RpnDecodePluginIOExtCreator() : RcnnIOExtCreator("RpnDecode") {} };
struct PredictorDecodePluginIOExtCreator : RcnnIOExtCreator<PredictorDecodePluginIOExt> { PredictorDecodePluginIOExtCreator() : RcnnIOExtCreator("PredictorDecode") {} };

}  // namespace trtx

#ifdef TRTX_REGISTER_PLUGINS
namespace trtx {
#ifdef TRTX_IMPLICIT_BATCH_PLUGINS
REGISTER_TENSORRT_PLUGIN(YoloPluginCreatorImplicitBatch);
#else
REGISTER_TENSORRT_PLUGIN(YoloPluginCreator);
#endif
REGISTER_TENSORRT_PLUGIN(DecodePluginCreator);
REGISTER_TENSORRT_PLUGIN(RpnNmsPluginCreator);
REGISTER_TENSORRT_PLUGIN(BatchedNmsPluginCreator);
#ifdef TRTX_RCNN_HALF_IO_PLUGINS  // the R-CNN plugins of an FP16 engine: "RpnDecode", "PredictorDecode", "RoiAlign" and
                                  // "MaskRcnnInference" that also accept fp16 scores and deltas / feature maps / masks
REGISTER_TENSORRT_PLUGIN(RpnDecodePluginIOExtCreator);
REGISTER_TENSORRT_PLUGIN(PredictorDecodePluginIOExtCreator);
REGISTER_TENSORRT_PLUGIN(RoiAlignPluginIOExtCreator);
REGISTER_TENSORRT_PLUGIN(MaskRcnnInferencePluginIOExtCreator);
#else
REGISTER_TENSORRT_PLUGIN(RpnDecodePluginCreator);
REGISTER_TENSORRT_PLUGIN(PredictorDecodePluginCreator);
REGISTER_TENSORRT_PLUGIN(RoiAlignPluginCreator);
REGISTER_TENSORRT_PLUGIN(MaskRcnnInferencePluginCreator);
#endif
}  // namespace trtx
#endif

#endif  // TRTX_PLUGINS_H
