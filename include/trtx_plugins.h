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
    // the yolov3 family (yolov3/yololayer.h:20-44 and its siblings): rows of 7 floats; the blob holds no net size, box formula
    // or maxOut, they are compile-time constants of each driver.  spp: a YoloKernel with a stride (36 bytes, grids -1 until
    // the tensors are bound); the others: {int w, h; float anchors[6]} (32 bytes).
    static constexpr int kV3Floats = 7;
    void init_v3(int variant, int nc, int w, int h, int max_out, const void* kernels, int n) {
        std::memset(&p, 0, sizeof(p));
        p.variant = variant;
        p.num_classes = nc;
        p.net_w = w;
        p.net_h = h;
        p.max_out = max_out;
        p.det_floats = kV3Floats;
        p.num_levels = n;
        p.gate = 0.1f;  // IGNORE_THRESH, yolov4/yololayer.h:11
        const int ks = v3_kernel_bytes();
        const char* k = static_cast<const char*>(kernels);
        for (int i = 0; i < n && i < TRTX_MAX_LEVELS; ++i, k += ks) {
            std::memcpy(&p.grid_w[i], k, 4);
            std::memcpy(&p.grid_h[i], k + 4, 4);
            if (ks == 36) std::memcpy(&p.strides[i], k + 8, 4);
            std::memcpy(p.anchors[i], k + ks - 24, 24);
        }
    }
    // bytes of one serialized YoloKernel of the yolov3 family, 0 for the other variants
    int v3_kernel_bytes() const {
        if (p.variant == TRTX_YOLO_V3) return 36;
        return p.variant == TRTX_YOLO_V3_NET || p.variant == TRTX_YOLO_V4 || p.variant == TRTX_YOLO_V4_CSP ? 32 : 0;
    }
    // the family's blob (yolov4/yololayer.cu:58-70, yolov3-spp/yololayer.cu:58-69): the variant, net size and maxOut come
    // from the caller; any length other than 12 + kernel bytes * kernelCount is refused
    bool deserialize_v3(const void* data, size_t length, int variant, int w, int h, int max_out) {
        if (length < 12) return false;
        const char* d = static_cast<const char*>(data);
        int nc, tc, kc;
        detail::read(d, nc);
        detail::read(d, tc);
        detail::read(d, kc);
        p.variant = variant;
        const size_t ks = (size_t)v3_kernel_bytes();
        if (ks == 0 || kc <= 0 || kc > TRTX_MAX_LEVELS || length != 12 + ks * (size_t)kc) return false;
        init_v3(variant, nc, w, h, max_out, d, kc);
        thread_count = tc;
        return true;
    }
    int out_elems() const { return 1 + p.max_out * p.det_floats; }  // yololayer.cu:107-111

    // yolov9, yolov10 and yolov13: yolov8's decode (TRTX_YOLO_V8) in another plugin class with another blob, so `blob` says
    // which layout serialize() writes: 0 the one the variant implies, 9 or 10 below.
    //   yolov9 (yolov9/plugin/yololayer.cu:25-63): YoloLayerPlugin(classCount, netW, netH, maxOut, is_seg); strides 8, 16, 32
    //   and grids net / stride are compiled in (:185-187); 38-float rows, the 32 mask coefficients at float 6; blob classCount,
    //   threadCount, netW, netH, maxOut, is_seg = 21 bytes.
    //   yolov10 / yolov13 (yolov10/plugin/yololayer.cu:28-84, yolov13's is the same): (classCount, netW, netH, maxOut, strides,
    //   n); 6-float rows; blob classCount, threadCount, netW, netH, maxOut, n, strides = 24 + 4n bytes.
    static constexpr int kV9Floats = 38, kV10Floats = 6;
    int blob = 0;
    void init_v9(int nc, int w, int h, int max_out, bool seg) {
        static const int st[3] = {8, 16, 32};
        init_v8(nc, 0, 0.0f, w, h, max_out, seg, false, false, st, 3);
        p.det_floats = kV9Floats;
        blob = 9;
    }
    // false for a level count outside 1..TRTX_MAX_LEVELS or a stride <= 0
    bool init_v10(int nc, int w, int h, int max_out, const int* strides, int n) {
        if (n < 1 || n > TRTX_MAX_LEVELS) return false;
        for (int i = 0; i < n; ++i)
            if (strides[i] <= 0) return false;
        init_v8(nc, 0, 0.0f, w, h, max_out, false, false, false, strides, n);
        p.det_floats = kV10Floats;
        blob = 10;
        return true;
    }
    // createPlugin: yolov9's one field "netinfo" = {nc, w, h, maxOut, is_seg}, read as ints whatever type it is declared with
    // (the builder declares kFLOAT32 for int data, block.cpp:405-410, and the plugin casts to int*, yololayer.cu:223)
    bool v9_fields(const nvinfer1::PluginFieldCollection* fc) {
        if (!fc || fc->nbFields != 1 || !fc->fields) return false;
        const nvinfer1::PluginField& f = fc->fields[0];
        if (!f.name || !f.data || std::strcmp(f.name, "netinfo") != 0 || f.length < 5) return false;
        const int* ni = static_cast<const int*>(f.data);
        init_v9(ni[0], ni[1], ni[2], ni[3], ni[4] != 0);
        return true;
    }
    // yolov10's / yolov13's one field "combinedInfo" = {nc, w, h, maxOut, strides...} (yolov10/src/block.cpp:235-262)
    bool v10_fields(const nvinfer1::PluginFieldCollection* fc) {
        if (!fc || fc->nbFields != 1 || !fc->fields) return false;
        const nvinfer1::PluginField& f = fc->fields[0];
        if (!f.name || !f.data || std::strcmp(f.name, "combinedInfo") != 0 || f.length < 5) return false;
        const int* ci = static_cast<const int*>(f.data);
        return init_v10(ci[0], ci[1], ci[2], ci[3], ci + 4, f.length - 4);
    }
    // the two blobs: exactly 21 bytes with an is_seg byte of 0 or 1; exactly 24 + 4n bytes with n and the strides valid
    bool deserialize_v9(const void* data, size_t length) {
        if (!data || length != 21) return false;
        const char* d = static_cast<const char*>(data);
        int nc, tc, w, h, mo;
        unsigned char seg;
        detail::read(d, nc);
        detail::read(d, tc);
        detail::read(d, w);
        detail::read(d, h);
        detail::read(d, mo);
        detail::read(d, seg);
        if (seg > 1) return false;
        init_v9(nc, w, h, mo, seg != 0);
        thread_count = tc;
        return true;
    }
    bool deserialize_v10(const void* data, size_t length) {
        if (!data || length < 24) return false;
        const char* d = static_cast<const char*>(data);
        int nc, tc, w, h, mo, n;
        detail::read(d, nc);
        detail::read(d, tc);
        detail::read(d, w);
        detail::read(d, h);
        detail::read(d, mo);
        detail::read(d, n);
        if (n < 1 || n > TRTX_MAX_LEVELS || length != 24 + 4 * (size_t)n) return false;
        int st[TRTX_MAX_LEVELS];
        for (int i = 0; i < n; ++i) detail::read(d, st[i]);
        if (!init_v10(nc, w, h, mo, st, n)) return false;
        thread_count = tc;
        return true;
    }
    // the yolov7 / YOLOP blob: the yolov5 one without the is_seg byte (yolov7/plugin/yololayer.cu:62-77,
    // yolop/yololayer.cu:81-101)
    bool v7_layout() const { return p.variant == TRTX_YOLO_V5 && p.det_floats == kV7Floats; }

    size_t serial_size() const {
        if (blob == 9) return 21;
        if (blob == 10) return 24 + 4 * (size_t)p.num_levels;
        if (p.variant == TRTX_YOLO_V8) return 4 * 8 + 4 * (size_t)p.num_levels + 3;  // yololayer.cu:97-101
        if (v3_kernel_bytes()) return 12 + (size_t)v3_kernel_bytes() * p.num_levels;
        return (v7_layout() ? 24 : 25) + 32 * (size_t)p.num_levels;                 // yolov5 yololayer.cu:72-83
    }
    void serialize(void* buffer) const {
        char* d = static_cast<char*>(buffer);
        if (blob == 9 || blob == 10) {
            detail::write(d, p.num_classes);
            detail::write(d, thread_count);
            detail::write(d, p.net_w);
            detail::write(d, p.net_h);
            detail::write(d, p.max_out);
            if (blob == 9) {
                detail::write(d, (bool)p.is_seg);
            } else {
                detail::write(d, p.num_levels);
                for (int i = 0; i < p.num_levels; ++i) detail::write(d, p.strides[i]);
            }
        } else if (p.variant == TRTX_YOLO_V8) {
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
        } else if (v3_kernel_bytes()) {
            detail::write(d, p.num_classes);
            detail::write(d, thread_count);
            detail::write(d, p.num_levels);
            for (int i = 0; i < p.num_levels; ++i) {
                detail::write(d, p.grid_w[i]);
                detail::write(d, p.grid_h[i]);
                if (p.variant == TRTX_YOLO_V3) detail::write(d, p.strides[i]);
                for (int j = 0; j < 6; ++j) detail::write(d, p.anchors[i][j]);
            }
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

// ------------------------------------------------------------------------------------------------
// "YoloLayer_TRT"/"1" of the yolov3 family.  Its creators take no fields (yolov4/yololayer.cu:258-263) and its plugins carry
// the driver's compiled-in constants, so the creator is configured with them: a traits struct of the driver's yololayer.h
// (CLASS_NUM, INPUT_W x INPUT_H, MAX_OUTPUT_BBOX_COUNT, the YoloKernel table in the plugin's level order) and its decode
// variant.  createPlugin ignores the field collection and returns the configured plugin, as the reference does;
// deserializePlugin accepts this driver's blob layout only, with the driver's kernel count (and strides, for spp).  A 3-level yolov3-spp blob (12 + 36 * 3 = 120 bytes) has the
// length of a 3-level yolov7 / YOLOP one (24 + 32 * 3): only a creator configured for the driver can tell them apart.
// ------------------------------------------------------------------------------------------------
struct YoloV3FamilyKernel {
    int w, h, stride;  // stride: yolov3-spp only (its grids are -1 until the tensors are bound)
    float anchors[6];
};
struct YoloV3Traits {  // yolov3/yololayer.h:11-39
    static constexpr int variant = TRTX_YOLO_V3_NET, classes = 80, net_w = 608, net_h = 608, max_out = 1000, levels = 3;
    static const YoloV3FamilyKernel* kernels() {
        static const YoloV3FamilyKernel k[3] = {{19, 19, 0, {116, 90, 156, 198, 373, 326}},
                                                {38, 38, 0, {30, 61, 62, 45, 59, 119}},
                                                {76, 76, 0, {10, 13, 16, 30, 33, 23}}};
        return k;
    }
};
struct YoloV4Traits {  // yolov4/yololayer.h:10-34
    static constexpr int variant = TRTX_YOLO_V4, classes = 80, net_w = 608, net_h = 608, max_out = 1000, levels = 3;
    static const YoloV3FamilyKernel* kernels() {
        static const YoloV3FamilyKernel k[3] = {{76, 76, 0, {12, 16, 19, 36, 40, 28}},
                                                {38, 38, 0, {36, 75, 76, 55, 72, 146}},
                                                {19, 19, 0, {142, 110, 192, 243, 459, 401}}};
        return k;
    }
};
struct ScaledYoloV4Traits {  // scaled-yolov4/yololayer.h:10-38
    static constexpr int variant = TRTX_YOLO_V4_CSP, classes = 80, net_w = 512, net_h = 512, max_out = 1000, levels = 3;
    static const YoloV3FamilyKernel* kernels() {
        static const YoloV3FamilyKernel k[3] = {{64, 64, 0, {12, 16, 19, 36, 40, 28}},
                                                {32, 32, 0, {36, 75, 76, 55, 72, 146}},
                                                {16, 16, 0, {142, 110, 192, 243, 459, 401}}};
        return k;
    }
};
struct YoloV3TinyTraits {  // yolov3-tiny/yololayer.h:11-34
    static constexpr int variant = TRTX_YOLO_V3_NET, classes = 80, net_w = 608, net_h = 608, max_out = 1000, levels = 2;
    static const YoloV3FamilyKernel* kernels() {
        static const YoloV3FamilyKernel k[2] = {{19, 19, 0, {81, 82, 135, 169, 344, 319}},
                                                {38, 38, 0, {23, 27, 37, 58, 81, 82}}};
        return k;
    }
};
struct YoloV3SppTraits {  // yolov3-spp/yololayer.h:11-44: dynamic input, the stride in the kernel, no net size
    static constexpr int variant = TRTX_YOLO_V3, classes = 80, net_w = 0, net_h = 0, max_out = 1000, levels = 3;
    static const YoloV3FamilyKernel* kernels() {
        static const YoloV3FamilyKernel k[3] = {{-1, -1, 32, {116, 90, 156, 198, 373, 326}},
                                                {-1, -1, 16, {30, 61, 62, 45, 59, 119}},
                                                {-1, -1, 8, {10, 13, 16, 30, 33, 23}}};
        return k;
    }
};

template <class Traits, bool Dynamic = true>
class YoloV3FamilyCreatorT : public nvinfer1::IPluginCreator {
   public:
    YoloV3FamilyCreatorT() { fc_.nbFields = 0; fc_.fields = nullptr; }
    const char* getPluginName() const TRTX_NOEXCEPT override { return "YoloLayer_TRT"; }
    const char* getPluginVersion() const TRTX_NOEXCEPT override { return "1"; }
    const nvinfer1::PluginFieldCollection* getFieldNames() TRTX_NOEXCEPT override { return &fc_; }
    // the reference's default constructor: CLASS_NUM, the YoloKernel table, threadCount 256
    static YoloCore configured() {
        YoloCore c;
        c.p.variant = Traits::variant;
        const int ks = c.v3_kernel_bytes();
        char blob[TRTX_MAX_LEVELS][36];
        for (int i = 0; i < Traits::levels; ++i) {
            const YoloV3FamilyKernel& k = Traits::kernels()[i];
            std::memcpy(blob[0] + i * ks, &k.w, 4);
            std::memcpy(blob[0] + i * ks + 4, &k.h, 4);
            if (ks == 36) std::memcpy(blob[0] + i * ks + 8, &k.stride, 4);
            std::memcpy(blob[0] + i * ks + ks - 24, k.anchors, 24);
        }
        c.init_v3(Traits::variant, Traits::classes, Traits::net_w, Traits::net_h, Traits::max_out, blob, Traits::levels);
        return c;
    }
    nvinfer1::IPluginV2* createPlugin(const char*, const nvinfer1::PluginFieldCollection*) TRTX_NOEXCEPT override {
        YoloCore c = configured();
        return make(c);
    }
    nvinfer1::IPluginV2* deserializePlugin(const char*, const void* data, size_t len) TRTX_NOEXCEPT override {
        YoloCore c;
        if (!data || !c.deserialize_v3(data, len, Traits::variant, Traits::net_w, Traits::net_h, Traits::max_out)) return nullptr;
        // the driver's plugin always serializes its own YoloKernel count and (spp) strides, which nothing changes: a blob
        // with other ones is not this driver's (a 3-level yolov7 / YOLOP blob has spp's length but maxOut where the
        // first stride lies)
        if (c.p.num_levels != Traits::levels) return nullptr;
        for (int i = 0; i < Traits::levels; ++i)
            if (Traits::variant == TRTX_YOLO_V3 && c.p.strides[i] != Traits::kernels()[i].stride) return nullptr;
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

// ------------------------------------------------------------------------------------------------
// "YoloLayer_TRT"/"1" of yolov9 (Driver = 9) and of yolov10 / yolov13 (Driver = 10).  yolov10's "combinedInfo" has 4 + n ints and
// yolov8's 9 + n: with up to TRTX_MAX_LEVELS strides the two length ranges overlap, so YoloPluginCreator cannot tell them
// apart, and it has no yolov9 layout at all.  These creators read their driver's field and blob only (YoloCore::v9_fields /
// v10_fields, deserialize_v9 / deserialize_v10) and refuse anything else with nullptr, where the reference asserts.
// ------------------------------------------------------------------------------------------------
template <int Driver, bool Dynamic = true>
class YoloAnchorFreeCreatorT : public nvinfer1::IPluginCreator {
    static_assert(Driver == 9 || Driver == 10, "Driver: 9 (yolov9) or 10 (yolov10, yolov13)");

   public:
    YoloAnchorFreeCreatorT() { fc_.nbFields = 0; fc_.fields = nullptr; }
    const char* getPluginName() const TRTX_NOEXCEPT override { return "YoloLayer_TRT"; }
    const char* getPluginVersion() const TRTX_NOEXCEPT override { return "1"; }
    const nvinfer1::PluginFieldCollection* getFieldNames() TRTX_NOEXCEPT override { return &fc_; }
    nvinfer1::IPluginV2* createPlugin(const char*, const nvinfer1::PluginFieldCollection* fc) TRTX_NOEXCEPT override {
        YoloCore c;
        if (!(Driver == 9 ? c.v9_fields(fc) : c.v10_fields(fc))) return nullptr;
        return make(c);
    }
    nvinfer1::IPluginV2* deserializePlugin(const char*, const void* data, size_t len) TRTX_NOEXCEPT override {
        YoloCore c;
        if (!(Driver == 9 ? c.deserialize_v9(data, len) : c.deserialize_v10(data, len))) return nullptr;
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
using YoloV9PluginCreator = YoloAnchorFreeCreatorT<9>;
using YoloV10PluginCreator = YoloAnchorFreeCreatorT<10>;

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
// Faster / Mask R-CNN plugins (rcnn/*Plugin.h): names "RpnDecode", "RpnNms", "PredictorDecode", "BatchedNms", "RoiAlign",
// "MaskRcnnInference", version "1", namespace "", implicit batch.  Each plugin is one parameter block (RpnDecodeParams, ...):
// the reference's fields with the reference's types (they fix the blob layout), its constructors, its blob, its output dims,
// its configurePlugin rule (on the dims of input kInput) and its C call.  RcnnPlugin<P> puts a block behind IPluginV2Ext (the
// reference's classes: RpnDecodePlugin, ...), RcnnPluginIOExt<P> behind IPluginV2IOExt (RpnDecodePluginIOExt, ...).
// ================================================================================================
namespace detail {
inline bool float_or_half(nvinfer1::DataType t) { return t == nvinfer1::DataType::kFLOAT || t == nvinfer1::DataType::kHALF; }

// A blob read front to back.  A read that does not fit in what is left fails the reader, and every read after it.
class BlobReader {
   public:
    BlobReader(const void* data, size_t length) : d_(static_cast<const char*>(data)), left_(data ? length : 0) {}
    // the next count * size bytes; nullptr when they do not fit
    const char* take(size_t count, size_t size) {
        if (!ok_ || count > left_ / size) {
            ok_ = false;
            return nullptr;
        }
        const char* p = d_;
        d_ += count * size;
        left_ -= count * size;
        return p;
    }
    template <typename T>
    void get(T& v) {
        if (const char* p = take(1, sizeof(T))) std::memcpy(&v, p, sizeof(T));
    }
    // every read fitted and no byte is left over
    bool done() const { return ok_ && left_ == 0; }

   private:
    const char* d_;
    size_t left_;
    bool ok_ = true;
};
// n floats that BlobReader::take has found in the blob
inline void assign(std::vector<float>& v, const char* p, size_t n) {
    v.resize(n);
    if (n) std::memcpy(v.data(), p, n * sizeof(float));
}

// Reads an R-CNN blob into p: the reference's blob (element type TRTX_F32) or, where tagged, the reference's blob followed by
// its element type as one int32 (TRTX_F32 | TRTX_F16).  False for any other blob.
template <class P>
bool read_dtype(P& p, const void* data, size_t length, bool tagged, int32_t& dtype) {
    int32_t t = TRTX_F32;
    if (!p.read(data, length)) {
        if (!tagged || length < sizeof(t) || !p.read(data, length - sizeof(t))) return false;
        std::memcpy(&t, static_cast<const char*>(data) + length - sizeof(t), sizeof(t));
        if (t != TRTX_F32 && t != TRTX_F16) return false;
    }
    dtype = t;
    return true;
}
}  // namespace detail

// rcnn/RpnDecodePlugin.h: scores [A, H, W] and deltas [4A, H, W] -> top_n scores [top_n, 1] and boxes [top_n, 4]
struct RpnDecodeParams {
    int top_n = 0;
    std::vector<float> anchors;
    float stride = 0.f;
    size_t height = 0, width = 0, image_height = 0, image_width = 0;

    RpnDecodeParams() = default;
    RpnDecodeParams(int top_n, const std::vector<float>& anchors, float stride, size_t image_height, size_t image_width)
        : RpnDecodeParams(top_n, anchors, stride, 0, 0, image_height, image_width) {}
    RpnDecodeParams(int top_n, const std::vector<float>& anchors, float stride, size_t height, size_t width, size_t image_height,
                    size_t image_width)
        : top_n(top_n), anchors(anchors), stride(stride), height(height), width(width), image_height(image_height),
          image_width(image_width) {}

    static const char* type() { return "RpnDecode"; }
    static constexpr int kOutputs = 2, kInput = 0;
    static constexpr bool kHasIOExt = true;
    size_t blob_size() const { return sizeof(int) + sizeof(size_t) + sizeof(float) * anchors.size() + sizeof(float) + 4 * sizeof(size_t); }
    void write(char*& d) const {  // RpnDecodePlugin.h:64-75
        detail::write(d, top_n);
        detail::write(d, anchors.size());
        for (float v : anchors) detail::write(d, v);
        detail::write(d, stride);
        detail::write(d, height);
        detail::write(d, width);
        detail::write(d, image_height);
        detail::write(d, image_width);
    }
    bool read(const void* data, size_t length) {  // RpnDecodePlugin.h:42-58
        detail::BlobReader r(data, length);
        size_t n = 0;
        r.get(top_n);
        r.get(n);
        const char* a = r.take(n, sizeof(float));
        r.get(stride);
        r.get(height);
        r.get(width);
        r.get(image_height);
        r.get(image_width);
        if (!r.done()) return false;
        detail::assign(anchors, a, n);
        return true;
    }
    nvinfer1::Dims dims(int index) const { return nvinfer1::Dims2(top_n, index == 1 ? 4 : 1); }
    void configure(const nvinfer1::Dims& scores) {  // RpnDecodePlugin.h:148-157: scores dims {A, H, W}
        height = scores.d[1];
        width = scores.d[2];
    }
    size_t workspace(int dtype, int batch) const {
        return (size_t)trtx_rpn_decode_typed(dtype, batch, nullptr, nullptr, nullptr, nullptr, (int)height, (int)width, (int)image_height,
                                             (int)image_width, stride, anchors.data(), (int)anchors.size() / 4, top_n, nullptr, 0, nullptr);
    }
    int run(int dtype, int batch, const void* const* in, void* const* out, void* ws, cudaStream_t stream) const {
        return detail::rcnn_rc(trtx_rpn_decode_typed(dtype, batch, in[0], in[1], static_cast<float*>(out[0]), static_cast<float*>(out[1]),
                                                     (int)height, (int)width, (int)image_height, (int)image_width, stride, anchors.data(),
                                                     (int)anchors.size() / 4, top_n, ws, workspace(dtype, batch), stream));
    }
    // IPluginV2IOExt: scores and deltas fp32 or fp16, one type; the scores and boxes fp32
    static bool io_type_ok(int pos, const nvinfer1::PluginTensorDesc* io, int nbInputs) {
        if (pos < nbInputs) return detail::float_or_half(io[pos].type) && io[pos].type == io[0].type;
        return io[pos].type == nvinfer1::DataType::kFLOAT;
    }
    static nvinfer1::DataType io_output_type(const nvinfer1::DataType*, int) { return nvinfer1::DataType::kFLOAT; }
};

// rcnn/RpnNmsPlugin.h: scores [pre, 1] and boxes [pre, 4] -> boxes [post, 4]
struct RpnNmsParams {
    float nms_thresh = 0.f;
    int post_nms_topk = 0;
    size_t pre_nms_topk = 1;

    RpnNmsParams() = default;
    RpnNmsParams(float nms_thresh, int post_nms_topk, size_t pre_nms_topk = 1)
        : nms_thresh(nms_thresh), post_nms_topk(post_nms_topk), pre_nms_topk(pre_nms_topk) {}

    static const char* type() { return "RpnNms"; }
    static constexpr int kOutputs = 1, kInput = 0;
    static constexpr bool kHasIOExt = false;
    size_t blob_size() const { return sizeof(float) + sizeof(int) + sizeof(size_t); }
    void write(char*& d) const {  // RpnNmsPlugin.h:48-52
        detail::write(d, nms_thresh);
        detail::write(d, post_nms_topk);
        detail::write(d, pre_nms_topk);
    }
    bool read(const void* data, size_t length) {  // RpnNmsPlugin.h:36-41
        detail::BlobReader r(data, length);
        r.get(nms_thresh);
        r.get(post_nms_topk);
        r.get(pre_nms_topk);
        return r.done();
    }
    nvinfer1::Dims dims(int) const { return nvinfer1::Dims2(post_nms_topk, 4); }
    void configure(const nvinfer1::Dims& scores) { pre_nms_topk = scores.d[0]; }
    size_t workspace(int, int batch) const {  // fp32 only
        return (size_t)trtx_rpn_nms(batch, nullptr, nullptr, nullptr, (int)pre_nms_topk, post_nms_topk, nms_thresh, nullptr, 0, nullptr);
    }
    int run(int dtype, int batch, const void* const* in, void* const* out, void* ws, cudaStream_t stream) const {
        return detail::rcnn_rc(trtx_rpn_nms(batch, static_cast<const float*>(in[0]), static_cast<const float*>(in[1]),
                                            static_cast<float*>(out[0]), (int)pre_nms_topk, post_nms_topk, nms_thresh, ws,
                                            workspace(dtype, batch), stream));
    }
};

// rcnn/RoiAlignPlugin.h:27-170: proposals [N, 4] and features [C, H, W] -> bins [N, C, P, P]
struct RoiAlignParams {
    int pooler_resolution = 0;
    float spatial_scale = 0.f;
    int sampling_ratio = 0, num_proposals = 0, out_channels = 0, feature_h = 0, feature_w = 0;

    RoiAlignParams() = default;
    RoiAlignParams(int pooler_resolution, float spatial_scale, int sampling_ratio, int num_proposals, int out_channels, int feature_h = 0,
                   int feature_w = 0)
        : pooler_resolution(pooler_resolution), spatial_scale(spatial_scale), sampling_ratio(sampling_ratio), num_proposals(num_proposals),
          out_channels(out_channels), feature_h(feature_h), feature_w(feature_w) {}

    static const char* type() { return "RoiAlign"; }
    static constexpr int kOutputs = 1, kInput = 1;
    static constexpr bool kHasIOExt = true;
    size_t blob_size() const { return 6 * sizeof(int) + sizeof(float); }
    void write(char*& d) const {  // RoiAlignPlugin.h:53-61
        detail::write(d, pooler_resolution);
        detail::write(d, spatial_scale);
        detail::write(d, sampling_ratio);
        detail::write(d, num_proposals);
        detail::write(d, out_channels);
        detail::write(d, feature_h);
        detail::write(d, feature_w);
    }
    bool read(const void* data, size_t length) {  // RoiAlignPlugin.h:37-46
        detail::BlobReader r(data, length);
        r.get(pooler_resolution);
        r.get(spatial_scale);
        r.get(sampling_ratio);
        r.get(num_proposals);
        r.get(out_channels);
        r.get(feature_h);
        r.get(feature_w);
        return r.done();
    }
    nvinfer1::Dims dims(int) const { return nvinfer1::Dims4(num_proposals, out_channels, pooler_resolution, pooler_resolution); }
    void configure(const nvinfer1::Dims& features) {  // RoiAlignPlugin.h:151-152
        feature_h = features.d[1];
        feature_w = features.d[2];
    }
    size_t workspace(int, int) const { return 0; }
    int run(int dtype, int batch, const void* const* in, void* const* out, void*, cudaStream_t stream) const {
        return trtx_roi_align_typed(dtype, batch, static_cast<const float*>(in[0]), in[1], out[0], pooler_resolution, spatial_scale,
                                    sampling_ratio, num_proposals, out_channels, feature_h, feature_w, stream);
    }
    // IPluginV2IOExt: proposals fp32; features fp32 or fp16; the bins in the features' type
    static bool io_type_ok(int pos, const nvinfer1::PluginTensorDesc* io, int) {
        if (pos == 0) return io[0].type == nvinfer1::DataType::kFLOAT;
        if (pos == 1) return detail::float_or_half(io[1].type);
        return io[pos].type == io[1].type;
    }
    static nvinfer1::DataType io_output_type(const nvinfer1::DataType* in, int nbInputs) {
        return nbInputs > 1 ? in[1] : nvinfer1::DataType::kFLOAT;
    }
};

// rcnn/MaskRcnnInferencePlugin.h:27-140: class indices [D] and masks [D, C, S, S] -> probabilities [D, 1, S, S]
struct MaskRcnnInferenceParams {
    int detections_per_im = 0, output_size = 0, num_classes = 1;

    MaskRcnnInferenceParams() = default;
    MaskRcnnInferenceParams(int detections_per_im, int output_size, int num_classes = 1)
        : detections_per_im(detections_per_im), output_size(output_size), num_classes(num_classes) {}

    static const char* type() { return "MaskRcnnInference"; }
    static constexpr int kOutputs = 1, kInput = 1;
    static constexpr bool kHasIOExt = true;
    size_t blob_size() const { return 3 * sizeof(int); }
    void write(char*& d) const {  // MaskRcnnInferencePlugin.h:41-45
        detail::write(d, detections_per_im);
        detail::write(d, output_size);
        detail::write(d, num_classes);
    }
    bool read(const void* data, size_t length) {  // MaskRcnnInferencePlugin.h:32-37
        detail::BlobReader r(data, length);
        r.get(detections_per_im);
        r.get(output_size);
        r.get(num_classes);
        return r.done();
    }
    nvinfer1::Dims dims(int) const { return nvinfer1::Dims4(detections_per_im, 1, output_size, output_size); }
    void configure(const nvinfer1::Dims& masks) { num_classes = masks.d[1]; }  // MaskRcnnInferencePlugin.h:119
    size_t workspace(int, int) const { return 0; }
    int run(int dtype, int batch, const void* const* in, void* const* out, void*, cudaStream_t stream) const {
        return trtx_mask_rcnn_inference_typed(dtype, batch, static_cast<const float*>(in[0]), in[1], static_cast<float*>(out[0]),
                                              detections_per_im, output_size, num_classes, stream);
    }
    // IPluginV2IOExt: class indices fp32; masks fp32 or fp16; the probabilities fp32 (they feed trtx_rcnn_postprocess*)
    static bool io_type_ok(int pos, const nvinfer1::PluginTensorDesc* io, int) {
        if (pos == 1) return detail::float_or_half(io[1].type);
        return io[pos].type == nvinfer1::DataType::kFLOAT;
    }
    static nvinfer1::DataType io_output_type(const nvinfer1::DataType*, int) { return nvinfer1::DataType::kFLOAT; }
};

// rcnn/PredictorDecodePlugin.h: scores [N, C, 1, 1], deltas [N, 4C, 1, 1] and proposals [N, 4] -> scores [N, 1], boxes [N, 4]
// and classes [N, 1]
struct PredictorDecodeParams {
    unsigned num_boxes = 0, num_classes = 0, image_height = 0, image_width = 0;
    std::vector<float> bbox_reg_weights;

    PredictorDecodeParams() = default;
    PredictorDecodeParams(unsigned num_boxes, unsigned image_height, unsigned image_width, const std::vector<float>& bbox_reg_weights)
        : PredictorDecodeParams(num_boxes, 0, image_height, image_width, bbox_reg_weights) {}
    PredictorDecodeParams(unsigned num_boxes, unsigned num_classes, unsigned image_height, unsigned image_width,
                          const std::vector<float>& bbox_reg_weights)
        : num_boxes(num_boxes), num_classes(num_classes), image_height(image_height), image_width(image_width),
          bbox_reg_weights(bbox_reg_weights) {}

    static const char* type() { return "PredictorDecode"; }
    static constexpr int kOutputs = 3, kInput = 0;
    static constexpr bool kHasIOExt = true;
    size_t blob_size() const { return 4 * sizeof(unsigned) + sizeof(size_t) + sizeof(float) * bbox_reg_weights.size(); }
    void write(char*& d) const {  // PredictorDecodePlugin.h:62-70
        detail::write(d, num_boxes);
        detail::write(d, num_classes);
        detail::write(d, image_height);
        detail::write(d, image_width);
        detail::write(d, bbox_reg_weights.size());
        for (float v : bbox_reg_weights) detail::write(d, v);
    }
    bool read(const void* data, size_t length) {  // PredictorDecodePlugin.h:40-54
        detail::BlobReader r(data, length);
        size_t n = 0;
        r.get(num_boxes);
        r.get(num_classes);
        r.get(image_height);
        r.get(image_width);
        r.get(n);
        const char* w = r.take(n, sizeof(float));
        if (!r.done()) return false;
        detail::assign(bbox_reg_weights, w, n);
        return true;
    }
    nvinfer1::Dims dims(int index) const { return nvinfer1::Dims2(num_boxes, index == 1 ? 4 : 1); }
    void configure(const nvinfer1::Dims& scores) { num_classes = scores.d[1]; }  // scores dims {N, C, 1, 1}
    size_t workspace(int dtype, int batch) const {
        return (size_t)trtx_predictor_decode_typed(dtype, batch, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, (int)num_boxes,
                                                   (int)num_classes, (int)image_height, (int)image_width, bbox_reg_weights.data(), nullptr,
                                                   0, nullptr);
    }
    int run(int dtype, int batch, const void* const* in, void* const* out, void* ws, cudaStream_t stream) const {
        if (bbox_reg_weights.size() < 4) return TRTX_ERR_INVALID;
        return detail::rcnn_rc(trtx_predictor_decode_typed(dtype, batch, in[0], in[1], static_cast<const float*>(in[2]),
                                                           static_cast<float*>(out[0]), static_cast<float*>(out[1]),
                                                           static_cast<float*>(out[2]), (int)num_boxes, (int)num_classes, (int)image_height,
                                                           (int)image_width, bbox_reg_weights.data(), ws, workspace(dtype, batch), stream));
    }
    // IPluginV2IOExt: scores and deltas fp32 or fp16, one type; the proposals and the scores, boxes and classes fp32
    static bool io_type_ok(int pos, const nvinfer1::PluginTensorDesc* io, int) {
        if (pos < 2) return detail::float_or_half(io[pos].type) && io[pos].type == io[0].type;
        return io[pos].type == nvinfer1::DataType::kFLOAT;
    }
    static nvinfer1::DataType io_output_type(const nvinfer1::DataType*, int) { return nvinfer1::DataType::kFLOAT; }
};

// rcnn/BatchedNmsPlugin.h: scores [count, 1], boxes [count, 4] and classes [count, 1] -> the same for detections_per_im
struct BatchedNmsParams {
    int nms_method = 0;
    float nms_thresh = 0.f;
    int detections_per_im = 0;
    size_t count = 1;

    BatchedNmsParams() = default;
    BatchedNmsParams(int nms_method, float nms_thresh, int detections_per_im, size_t count = 1)
        : nms_method(nms_method), nms_thresh(nms_thresh), detections_per_im(detections_per_im), count(count) {}

    static const char* type() { return "BatchedNms"; }
    static constexpr int kOutputs = 3, kInput = 0;
    static constexpr bool kHasIOExt = false;
    size_t blob_size() const { return sizeof(int) + sizeof(float) + sizeof(int) + sizeof(size_t); }
    void write(char*& d) const {  // BatchedNmsPlugin.h:51-56
        detail::write(d, nms_method);
        detail::write(d, nms_thresh);
        detail::write(d, detections_per_im);
        detail::write(d, count);
    }
    bool read(const void* data, size_t length) {  // BatchedNmsPlugin.h:38-44
        detail::BlobReader r(data, length);
        r.get(nms_method);
        r.get(nms_thresh);
        r.get(detections_per_im);
        r.get(count);
        return r.done();
    }
    nvinfer1::Dims dims(int index) const { return nvinfer1::Dims2(detections_per_im, index == 1 ? 4 : 1); }
    void configure(const nvinfer1::Dims& scores) { count = scores.d[0]; }  // BatchedNmsPlugin.h:148-157
    size_t workspace(int, int batch) const {  // fp32 only
        return (size_t)trtx_batched_nms(nms_method, batch, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, (int)count,
                                        detections_per_im, nms_thresh, nullptr, 0, nullptr);
    }
    int run(int dtype, int batch, const void* const* in, void* const* out, void* ws, cudaStream_t stream) const {
        return detail::rcnn_rc(trtx_batched_nms(nms_method, batch, static_cast<const float*>(in[0]), static_cast<const float*>(in[1]),
                                                static_cast<const float*>(in[2]), static_cast<float*>(out[0]), static_cast<float*>(out[1]),
                                                static_cast<float*>(out[2]), (int)count, detections_per_im, nms_thresh, ws,
                                                workspace(dtype, batch), stream));
    }
};

// IPluginV2Ext (rcnn/BatchedNmsPlugin.h:30) with the reference's constructors, fp32 linear tensors only and the reference's
// blob.  A blob is refused (valid() false) unless it is the reference's blob or, for a plugin that has an IPluginV2IOExt twin,
// that blob followed by a TRTX_F32 tag (what the twin writes in an fp32 engine).
template <class P>
class RcnnPlugin : public nvinfer1::IPluginV2Ext, private P {  // P is a base for its constructors (using P::P)
   public:
    using P::P;
    using P::type;  // the plugin name, for RcnnCreator
    RcnnPlugin(const void* data, size_t length) {
        int32_t dtype = -1;
        valid_ = detail::read_dtype<P>(*this, data, length, P::kHasIOExt, dtype) && dtype == TRTX_F32;
    }
    bool valid() const { return valid_; }
    const char* getPluginType() const TRTX_NOEXCEPT override { return P::type(); }
    const char* getPluginVersion() const TRTX_NOEXCEPT override { return "1"; }
    const char* getPluginNamespace() const TRTX_NOEXCEPT override { return ""; }
    void setPluginNamespace(const char*) TRTX_NOEXCEPT override {}
    int getNbOutputs() const TRTX_NOEXCEPT override { return P::kOutputs; }
    nvinfer1::Dims getOutputDimensions(int index, const nvinfer1::Dims*, int) TRTX_NOEXCEPT override { return P::dims(index); }
    bool supportsFormat(nvinfer1::DataType t, nvinfer1::PluginFormat f) const TRTX_NOEXCEPT override {
        return t == nvinfer1::DataType::kFLOAT && f == nvinfer1::PluginFormat::kLINEAR;  // BatchedNmsPlugin.h:98-100
    }
    nvinfer1::DataType getOutputDataType(int, const nvinfer1::DataType*, int) const TRTX_NOEXCEPT override { return nvinfer1::DataType::kFLOAT; }
    bool isOutputBroadcastAcrossBatch(int, const bool*, int) const TRTX_NOEXCEPT override { return false; }
    bool canBroadcastInputAcrossBatch(int) const TRTX_NOEXCEPT override { return false; }
    void configurePlugin(const nvinfer1::Dims* inputDims, int, const nvinfer1::Dims*, int, const nvinfer1::DataType*, const nvinfer1::DataType*,
                         const bool*, const bool*, nvinfer1::PluginFormat, int) TRTX_NOEXCEPT override {
        P::configure(inputDims[P::kInput]);
    }
    int initialize() TRTX_NOEXCEPT override { return 0; }
    void terminate() TRTX_NOEXCEPT override {}
    size_t getWorkspaceSize(int maxBatchSize) const TRTX_NOEXCEPT override { return P::workspace(TRTX_F32, maxBatchSize); }
    int enqueue(int batchSize, const void* const* inputs, void* TRTX_CONST_ENQUEUE* outputs, void* workspace, cudaStream_t stream) TRTX_NOEXCEPT override {
        return valid_ ? P::run(TRTX_F32, batchSize, inputs, outputs, workspace, stream) : TRTX_ERR_INVALID;
    }
    size_t getSerializationSize() const TRTX_NOEXCEPT override { return P::blob_size(); }
    void serialize(void* buffer) const TRTX_NOEXCEPT override {
        char* d = static_cast<char*>(buffer);
        P::write(d);
    }
    nvinfer1::IPluginV2Ext* clone() const TRTX_NOEXCEPT override { return new RcnnPlugin(*this); }
    void destroy() TRTX_NOEXCEPT override { delete this; }

   private:
    bool valid_ = true;
};

// ------------------------------------------------------------------------------------------------
// RoiAlign, MaskRcnnInference, RpnDecode and PredictorDecode for an FP16 engine.  Each needs fp32 tensors next to half
// ones (proposals, class indices, fp32 outputs), which IPluginV2Ext::supportsFormat (one type for every tensor) cannot say;
// IPluginV2IOExt::supportsFormatCombination can.  Same plugin names, version, constructor arguments and namespace as the
// IPluginV2Ext classes.  The element type TensorRT chose for input kInput arrives in configurePlugin, is carried through
// clone() and is appended to the serialized blob as one int32 (TRTX_F32 | TRTX_F16); a blob of the reference's length
// deserializes as fp32, a blob of any other length or with another tag is refused.
// Exercised against tests/mock_trt only: how a real TensorRT builder drives these four classes is NOT verified.
// ------------------------------------------------------------------------------------------------
template <class P>
class RcnnPluginIOExt : public nvinfer1::IPluginV2IOExt, private P {  // P is a base for its constructors (using P::P)
   public:
    using P::P;
    using P::type;  // the plugin name, for RcnnCreator
    RcnnPluginIOExt(const void* data, size_t length) { valid_ = detail::read_dtype<P>(*this, data, length, true, dtype_); }
    bool valid() const { return valid_; }
    int dtype() const { return dtype_; }  // of input kInput: the feature map / the masks / the scores and deltas
    const char* getPluginType() const TRTX_NOEXCEPT override { return P::type(); }
    const char* getPluginVersion() const TRTX_NOEXCEPT override { return "1"; }
    const char* getPluginNamespace() const TRTX_NOEXCEPT override { return ""; }
    void setPluginNamespace(const char*) TRTX_NOEXCEPT override {}
    int getNbOutputs() const TRTX_NOEXCEPT override { return P::kOutputs; }
    nvinfer1::Dims getOutputDimensions(int index, const nvinfer1::Dims*, int) TRTX_NOEXCEPT override { return P::dims(index); }
    bool supportsFormatCombination(int pos, const nvinfer1::PluginTensorDesc* io, int nbInputs, int) const TRTX_NOEXCEPT override {
        return io[pos].format == nvinfer1::TensorFormat::kLINEAR && P::io_type_ok(pos, io, nbInputs);
    }
    nvinfer1::DataType getOutputDataType(int, const nvinfer1::DataType* inputTypes, int nbInputs) const TRTX_NOEXCEPT override {
        return P::io_output_type(inputTypes, nbInputs);
    }
    bool isOutputBroadcastAcrossBatch(int, const bool*, int) const TRTX_NOEXCEPT override { return false; }
    bool canBroadcastInputAcrossBatch(int) const TRTX_NOEXCEPT override { return false; }
    void configurePlugin(const nvinfer1::PluginTensorDesc* in, int, const nvinfer1::PluginTensorDesc*, int) TRTX_NOEXCEPT override {
        P::configure(in[P::kInput].dims);
        dtype_ = in[P::kInput].type == nvinfer1::DataType::kHALF ? TRTX_F16 : TRTX_F32;
    }
    int initialize() TRTX_NOEXCEPT override { return 0; }
    void terminate() TRTX_NOEXCEPT override {}
    size_t getWorkspaceSize(int maxBatchSize) const TRTX_NOEXCEPT override { return P::workspace(dtype_, maxBatchSize); }
    int enqueue(int batchSize, const void* const* inputs, void* TRTX_CONST_ENQUEUE* outputs, void* workspace, cudaStream_t stream) TRTX_NOEXCEPT override {
        return valid_ ? P::run(dtype_, batchSize, inputs, outputs, workspace, stream) : TRTX_ERR_INVALID;
    }
    size_t getSerializationSize() const TRTX_NOEXCEPT override { return P::blob_size() + sizeof(dtype_); }
    void serialize(void* buffer) const TRTX_NOEXCEPT override {
        char* d = static_cast<char*>(buffer);
        P::write(d);
        detail::write(d, dtype_);
    }
    nvinfer1::IPluginV2IOExt* clone() const TRTX_NOEXCEPT override { return new RcnnPluginIOExt(*this); }
    void destroy() TRTX_NOEXCEPT override { delete this; }

   private:
    int32_t dtype_ = TRTX_F32;
    bool valid_ = true;
};

// The creator of an R-CNN plugin class.  No fields: createPlugin answers nullptr, as the reference's creators do; a blob the
// class refuses deserializes to nullptr.
template <class Plugin>
class RcnnCreator : public nvinfer1::IPluginCreator {
   public:
    const char* getPluginName() const TRTX_NOEXCEPT override { return Plugin::type(); }
    const char* getPluginVersion() const TRTX_NOEXCEPT override { return "1"; }
    const char* getPluginNamespace() const TRTX_NOEXCEPT override { return ""; }
    void setPluginNamespace(const char*) TRTX_NOEXCEPT override {}
    const nvinfer1::PluginFieldCollection* getFieldNames() TRTX_NOEXCEPT override { return nullptr; }
    nvinfer1::IPluginV2* createPlugin(const char*, const nvinfer1::PluginFieldCollection*) TRTX_NOEXCEPT override { return nullptr; }
    nvinfer1::IPluginV2* deserializePlugin(const char*, const void* data, size_t len) TRTX_NOEXCEPT override {
        Plugin* p = new Plugin(data, len);
        if (p->valid()) return p;
        delete p;
        return nullptr;
    }
};

using RpnDecodePlugin = RcnnPlugin<RpnDecodeParams>;
using RpnNmsPlugin = RcnnPlugin<RpnNmsParams>;
using PredictorDecodePlugin = RcnnPlugin<PredictorDecodeParams>;
using BatchedNmsPlugin = RcnnPlugin<BatchedNmsParams>;
using RoiAlignPlugin = RcnnPlugin<RoiAlignParams>;
using MaskRcnnInferencePlugin = RcnnPlugin<MaskRcnnInferenceParams>;
using RpnDecodePluginIOExt = RcnnPluginIOExt<RpnDecodeParams>;
using PredictorDecodePluginIOExt = RcnnPluginIOExt<PredictorDecodeParams>;
using RoiAlignPluginIOExt = RcnnPluginIOExt<RoiAlignParams>;
using MaskRcnnInferencePluginIOExt = RcnnPluginIOExt<MaskRcnnInferenceParams>;

using RpnDecodePluginCreator = RcnnCreator<RpnDecodePlugin>;
using RpnNmsPluginCreator = RcnnCreator<RpnNmsPlugin>;
using PredictorDecodePluginCreator = RcnnCreator<PredictorDecodePlugin>;
using BatchedNmsPluginCreator = RcnnCreator<BatchedNmsPlugin>;
using RoiAlignPluginCreator = RcnnCreator<RoiAlignPlugin>;
using MaskRcnnInferencePluginCreator = RcnnCreator<MaskRcnnInferencePlugin>;
using RpnDecodePluginIOExtCreator = RcnnCreator<RpnDecodePluginIOExt>;
using PredictorDecodePluginIOExtCreator = RcnnCreator<PredictorDecodePluginIOExt>;
using RoiAlignPluginIOExtCreator = RcnnCreator<RoiAlignPluginIOExt>;
using MaskRcnnInferencePluginIOExtCreator = RcnnCreator<MaskRcnnInferencePluginIOExt>;

}  // namespace trtx

#ifdef TRTX_REGISTER_PLUGINS
namespace trtx {
// TRTX_YOLO_V3_FAMILY=<traits> (YoloV3Traits, YoloV4Traits, ScaledYoloV4Traits, YoloV3TinyTraits, YoloV3SppTraits): the
// "YoloLayer_TRT" creator is that driver's family creator instead of YoloPluginCreator (only one creator can hold the name)
#if defined(TRTX_YOLO_V3_FAMILY) && defined(TRTX_IMPLICIT_BATCH_PLUGINS)
using YoloV3FamilyRegisteredCreator = YoloV3FamilyCreatorT<TRTX_YOLO_V3_FAMILY, false>;
REGISTER_TENSORRT_PLUGIN(YoloV3FamilyRegisteredCreator);
#elif defined(TRTX_YOLO_V3_FAMILY)
using YoloV3FamilyRegisteredCreator = YoloV3FamilyCreatorT<TRTX_YOLO_V3_FAMILY, true>;
REGISTER_TENSORRT_PLUGIN(YoloV3FamilyRegisteredCreator);
// TRTX_YOLO_ANCHOR_FREE=9 (yolov9) or 10 (yolov10, yolov13): that driver's creator instead of YoloPluginCreator
#elif defined(TRTX_YOLO_ANCHOR_FREE) && defined(TRTX_IMPLICIT_BATCH_PLUGINS)
using YoloAnchorFreeRegisteredCreator = YoloAnchorFreeCreatorT<TRTX_YOLO_ANCHOR_FREE, false>;
REGISTER_TENSORRT_PLUGIN(YoloAnchorFreeRegisteredCreator);
#elif defined(TRTX_YOLO_ANCHOR_FREE)
using YoloAnchorFreeRegisteredCreator = YoloAnchorFreeCreatorT<TRTX_YOLO_ANCHOR_FREE, true>;
REGISTER_TENSORRT_PLUGIN(YoloAnchorFreeRegisteredCreator);
#elif defined(TRTX_IMPLICIT_BATCH_PLUGINS)
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
