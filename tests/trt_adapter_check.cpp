// trt_adapter_check.cpp -- drives include/trtx_plugins.h through the TensorRT plugin surface exactly as an engine
// builder / the TensorRT runtime would: registry lookup by name, createPlugin with the reference's field layouts,
// (de)serialization, malformed R-CNN blobs refused, clone, getOutputDimensions, getWorkspaceSize, and (with --gpu) enqueue on
// the device.
// Compiled against tests/mock_trt/NvInfer.h (this image has no TensorRT) and linked with libtrtx_hot.so.
#define TRTX_REGISTER_PLUGINS
#include "trtx_plugins.h"

#include <cuda_runtime_api.h>

#include <cassert>
#include <cstdio>
#include <cstdlib>
#include <type_traits>
#include <vector>

#define CHECK(x)                                                          \
    do {                                                                  \
        if (!(x)) {                                                       \
            std::fprintf(stderr, "CHECK failed %s:%d: %s\n", __FILE__, __LINE__, #x); \
            std::exit(1);                                                 \
        }                                                                 \
    } while (0)

using namespace nvinfer1;

struct ConstExpr : IDimensionExpr {
    int v;
    explicit ConstExpr(int x) : v(x) {}
    bool isConstant() const TRTX_NX override { return true; }
    int32_t getConstantValue() const TRTX_NX override { return v; }
};
struct Builder : IExprBuilder {
    std::vector<ConstExpr*> pool;
    const IDimensionExpr* constant(int32_t value) TRTX_NX override {
        pool.push_back(new ConstExpr(value));
        return pool.back();
    }
    const IDimensionExpr* operation(DimensionOperation, const IDimensionExpr& a, const IDimensionExpr&) TRTX_NX override { return &a; }
};

// The blobs an IPluginV2Ext R-CNN class accepts: its reference blob ref and, where the class has an IPluginV2IOExt twin
// (f32_tag), ref + a TRTX_F32 tag; each deserializes, directly and through the registered creator, to a plugin that writes ref.
// Refused, with the creator answering nullptr and the plugin's enqueue TRTX_ERR_INVALID: an empty blob, ref one byte short or
// over, ref + a TRTX_F16 tag, and an anchor / weight count of 2^62 at byte count_at.
template <class P>
static void check_blobs(const std::vector<char>& ref, bool f32_tag, int count_at = -1) {
    static_assert(std::is_copy_constructible<P>::value && std::is_move_constructible<P>::value, "rcnn.cpp builds the plugins by value");
    IPluginCreator* c = getPluginRegistry()->getPluginCreator(P::type(), "1");
    CHECK(c != nullptr);
    auto accepted = [&](const std::vector<char>& b) {
        P direct(b.data(), b.size());
        IPluginV2* p = c->deserializePlugin(P::type(), b.data(), b.size());
        CHECK((p != nullptr) == direct.valid());
        if (!p) {
            CHECK(direct.enqueue(1, nullptr, nullptr, nullptr, nullptr) == TRTX_ERR_INVALID);
            return false;
        }
        std::vector<char> back(p->getSerializationSize());
        p->serialize(back.data());
        CHECK(back == ref);
        p->destroy();
        return true;
    };
    CHECK(accepted(ref));
    CHECK(!accepted({}));
    CHECK(!accepted(std::vector<char>(ref.begin(), ref.end() - 1)));
    std::vector<char> b = ref;
    b.push_back(0);
    CHECK(!accepted(b));
    for (int32_t tag : {TRTX_F32, TRTX_F16}) {
        b = ref;
        b.insert(b.end(), reinterpret_cast<const char*>(&tag), reinterpret_cast<const char*>(&tag) + sizeof(tag));
        CHECK(accepted(b) == (f32_tag && tag == TRTX_F32));
    }
    if (count_at >= 0) {
        b = ref;
        const size_t big = (size_t)1 << 62;
        std::memcpy(b.data() + count_at, &big, sizeof(big));
        CHECK(!accepted(b));
    }
}

int main(int argc, char** argv) {
    const bool gpu = argc > 1 && std::string(argv[1]) == "--gpu";
    const bool dump = argc > 1 && std::string(argv[1]) == "--dump";  // print every serialized blob as hex (compared with plugins.py)
    auto hex = [&](const char* name, const std::vector<char>& b) {
        if (!dump) return;
        std::printf("blob %s ", name);
        for (unsigned char c : b) std::printf("%02x", c);
        std::printf("\n");
    };
    // ---- what yolov8/src/block.cpp:262-296 does ----
    IPluginCreator* creator = getPluginRegistry()->getPluginCreator("YoloLayer_TRT", "1");
    CHECK(creator != nullptr);
    std::vector<int> combined = {80, 17, 0, 640, 640, 1000, 0, 0, 0, 8, 16, 32};
    PluginField pf("combinedInfo", combined.data(), PluginFieldType::kINT32, (int)combined.size());
    PluginFieldCollection fc{1, &pf};
    IPluginV2* obj = creator->createPlugin("yololayer", &fc);
    CHECK(obj != nullptr);
    CHECK(std::string(obj->getPluginType()) == "YoloLayer_TRT" && std::string(obj->getPluginVersion()) == "1");
    CHECK(obj->getNbOutputs() == 1);
    auto* dyn = static_cast<IPluginV2DynamicExt*>(obj);
    Builder eb;
    ConstExpr b32(32), c84(84), g0(6400);
    DimsExprs in0;
    in0.nbDims = 3;
    in0.d[0] = &b32;
    in0.d[1] = &c84;
    in0.d[2] = &g0;
    DimsExprs ins[3] = {in0, in0, in0};
    DimsExprs od = dyn->getOutputDimensions(0, ins, 3, eb);
    CHECK(od.nbDims == 2 && od.d[0]->getConstantValue() == 32 && od.d[1]->getConstantValue() == 1000 * 90 + 1);
    // serialization keeps the reference's byte layout (yololayer.cu:75-101): 8 ints/floats, strides, 3 bools
    CHECK(obj->getSerializationSize() == 4 * 8 + 4 * 3 + 3);
    std::vector<char> blob(obj->getSerializationSize());
    obj->serialize(blob.data());
    int first;
    std::memcpy(&first, blob.data(), 4);
    CHECK(first == 80);
    IPluginV2* back = creator->deserializePlugin("yololayer", blob.data(), blob.size());
    CHECK(back != nullptr && back->getSerializationSize() == blob.size());
    std::vector<char> blob2(blob.size());
    back->serialize(blob2.data());
    CHECK(blob == blob2);
    hex("yolov8", blob);
    CHECK(creator->deserializePlugin("yololayer", blob.data(), blob.size() - 1) == nullptr);  // malformed -> refused, no assert
    IPluginV2* cl = obj->clone();
    CHECK(cl != nullptr && cl != obj);
    PluginTensorDesc desc[4];
    for (int i = 0; i < 3; ++i) {
        desc[i].dims.nbDims = 3;
        desc[i].dims.d[0] = 32;
        desc[i].dims.d[1] = 84;
        desc[i].dims.d[2] = (640 >> (3 + i)) * (640 >> (3 + i));
        desc[i].type = DataType::kFLOAT;
        desc[i].format = TensorFormat::kLINEAR;
    }
    desc[3].dims.nbDims = 2;
    desc[3].dims.d[0] = 32;
    desc[3].dims.d[1] = 90001;
    desc[3].type = DataType::kFLOAT;
    desc[3].format = TensorFormat::kLINEAR;
    CHECK(dyn->supportsFormatCombination(0, desc, 3, 1) && dyn->supportsFormatCombination(3, desc, 3, 1));
    desc[3].type = DataType::kHALF;
    CHECK(!dyn->supportsFormatCombination(3, desc, 3, 1));
    desc[3].type = DataType::kFLOAT;
    const size_t ws_bytes = dyn->getWorkspaceSize(desc, 3, desc + 3, 1);
    CHECK(ws_bytes > 32u * 8400u * 32u);

    // ---- yolov5 fields (yolov5/src/model.cpp:249-277) through the implicit-batch creator ----
    trtx::YoloPluginCreatorImplicitBatch legacy;
    int netinfo[5] = {80, 640, 640, 1000, 0};
    struct K { int w, h; float a[6]; } kern[3] = {{80, 80, {10, 13, 16, 30, 33, 23}}, {40, 40, {30, 61, 62, 45, 59, 119}}, {20, 20, {116, 90, 156, 198, 373, 326}}};
    PluginField f5[2] = {PluginField("netinfo", netinfo, PluginFieldType::kFLOAT32, 5), PluginField("kernels", kern, PluginFieldType::kFLOAT32, 3)};
    PluginFieldCollection fc5{2, f5};
    IPluginV2* v5 = legacy.createPlugin("yololayer", &fc5);
    CHECK(v5 != nullptr && v5->getSerializationSize() == 25 + 3 * 32);
    Dims o5 = v5->getOutputDimensions(0, nullptr, 3);
    CHECK(o5.nbDims == 3 && o5.d[0] == 1000 * 38 + 1);
    std::vector<char> b5(v5->getSerializationSize());
    v5->serialize(b5.data());
    CHECK(legacy.deserializePlugin("yololayer", b5.data(), b5.size()) != nullptr);
    hex("yolov5", b5);

    // ---- Decode_TRT and the rcnn plugins ----
    IPluginCreator* dc = getPluginRegistry()->getPluginCreator("Decode_TRT", "1");
    CHECK(dc != nullptr);
    PluginFieldCollection none{0, nullptr};
    IPluginV2* dec = dc->createPlugin("decode", &none);
    CHECK(dec != nullptr && std::string(dec->getPluginType()) == "Decode_TRT");
    {
        std::vector<char> db(dec->getSerializationSize());
        dec->serialize(db.data());
        hex("decode", db);
    }
    trtx::RpnDecodePlugin rpn(6000, std::vector<float>(60, 1.f), 16.f, 50, 67, 800, 1067);
    CHECK(rpn.getNbOutputs() == 2 && rpn.getOutputDimensions(1, nullptr, 2).d[1] == 4 && rpn.getWorkspaceSize(8) > 0);
    std::vector<char> rb(rpn.getSerializationSize());
    rpn.serialize(rb.data());
    trtx::RpnDecodePlugin rpn2(rb.data(), rb.size());
    hex("rpn_decode", rb);
    check_blobs<trtx::RpnDecodePlugin>(rb, true, 4);
    {
        trtx::RpnNmsPlugin rn(0.7f, 1000);
        Dims nd[2];
        nd[0].nbDims = 2; nd[0].d[0] = 6000; nd[0].d[1] = 1; nd[1] = nd[0];
        rn.configurePlugin(nd, 2, nullptr, 1, nullptr, nullptr, nullptr, nullptr, PluginFormat::kLINEAR, 8);
        std::vector<char> nb(rn.getSerializationSize());
        rn.serialize(nb.data());
        hex("rpn_nms", nb);
        check_blobs<trtx::RpnNmsPlugin>(nb, false);
        trtx::PredictorDecodePlugin pd(1000, 800, 1067, std::vector<float>{10.f, 10.f, 5.f, 5.f});
        Dims pdm[3];
        pdm[0].nbDims = 4; pdm[0].d[0] = 1000; pdm[0].d[1] = 80; pdm[0].d[2] = 1; pdm[0].d[3] = 1; pdm[1] = pdm[0]; pdm[2] = pdm[0];
        pd.configurePlugin(pdm, 3, nullptr, 3, nullptr, nullptr, nullptr, nullptr, PluginFormat::kLINEAR, 8);
        std::vector<char> pb(pd.getSerializationSize());
        pd.serialize(pb.data());
        hex("predictor_decode", pb);
        check_blobs<trtx::PredictorDecodePlugin>(pb, true, 16);
    }
    CHECK(rpn2.getSerializationSize() == rb.size());
    trtx::BatchedNmsPlugin bn(1, 0.5f, 100);
    Dims cd[3];
    cd[0].nbDims = 2; cd[0].d[0] = 1000; cd[0].d[1] = 1; cd[1] = cd[0]; cd[2] = cd[0];
    bn.configurePlugin(cd, 3, nullptr, 3, nullptr, nullptr, nullptr, nullptr, PluginFormat::kLINEAR, 8);
    CHECK(bn.getSerializationSize() == 4 + 4 + 4 + sizeof(size_t) && bn.getWorkspaceSize(8) > 0);
    {
        std::vector<char> bb(bn.getSerializationSize());
        bn.serialize(bb.data());
        hex("batched_nms", bb);
        check_blobs<trtx::BatchedNmsPlugin>(bb, false);
    }
    CHECK(getPluginRegistry()->getPluginCreator("BatchedNms", "1") != nullptr && getPluginRegistry()->getPluginCreator("RpnNms", "1") != nullptr);
    trtx::RoiAlignPlugin ra(14, 1.f / 16, 0, 1000, 1024);
    Dims rd[2];
    rd[0].nbDims = 2; rd[0].d[0] = 1000; rd[0].d[1] = 4;
    rd[1].nbDims = 3; rd[1].d[0] = 1024; rd[1].d[1] = 50; rd[1].d[2] = 67;
    ra.configurePlugin(rd, 2, nullptr, 1, nullptr, nullptr, nullptr, nullptr, PluginFormat::kLINEAR, 8);
    std::vector<char> rab(ra.getSerializationSize());
    ra.serialize(rab.data());
    trtx::RoiAlignPlugin ra2(rab.data(), rab.size());
    hex("roi_align", rab);
    check_blobs<trtx::RoiAlignPlugin>(rab, true);
    CHECK(rab.size() == 28 && ra2.getOutputDimensions(0, nullptr, 2).d[3] == 14 && ra2.getWorkspaceSize(8) == 0);
    CHECK(std::string(ra2.getPluginType()) == "RoiAlign" && getPluginRegistry()->getPluginCreator("RoiAlign", "1") != nullptr);
    trtx::MaskRcnnInferencePlugin mi(100, 14);
    CHECK(mi.getSerializationSize() == 12 && mi.getOutputDimensions(0, nullptr, 2).d[0] == 100 &&
          getPluginRegistry()->getPluginCreator("MaskRcnnInference", "1") != nullptr);
    {
        std::vector<char> mb(mi.getSerializationSize());
        mi.serialize(mb.data());
        hex("mask_rcnn_inference", mb);
        check_blobs<trtx::MaskRcnnInferencePlugin>(mb, true);
    }

    if (gpu) {
        // ---- enqueue through both YOLO adapters on the same synthetic heads; outputs must be identical ----
        const int B = 4, C = 84;
        void* d_in[3];
        std::vector<std::vector<float>> h(3);
        int planted = 0;
        for (int l = 0; l < 3; ++l) {
            const int g = desc[l].dims.d[2];
            h[l].assign((size_t)B * C * g, -7.0f);
            for (int b = 0; b < B; ++b)
                for (int e = 0; e < g; e += 37) {  // one candidate every 37 cells, class e % 80, logit 2
                    h[l][((size_t)b * C + 4 + (e % 80)) * g + e] = 2.0f;
                    for (int k = 0; k < 4; ++k) h[l][((size_t)b * C + k) * g + e] = 1.5f;
                    if (b == 0) ++planted;
                }
            CHECK(cudaMalloc(&d_in[l], h[l].size() * 4) == cudaSuccess);
            CHECK(cudaMemcpy(d_in[l], h[l].data(), h[l].size() * 4, cudaMemcpyHostToDevice) == cudaSuccess);
            desc[l].dims.d[0] = B;
        }
        void *d_out, *d_out2, *d_ws;
        const size_t out_bytes = (size_t)B * 90001 * 4;
        CHECK(cudaMalloc(&d_out, out_bytes) == cudaSuccess && cudaMalloc(&d_out2, out_bytes) == cudaSuccess);
        CHECK(cudaMalloc(&d_ws, ws_bytes) == cudaSuccess);
        void* outs[1] = {d_out};
        CHECK(dyn->enqueue(desc, desc + 3, d_in, outs, d_ws, nullptr) == 0);
        trtx::YoloCore core;
        int st[3] = {8, 16, 32};
        core.init_v8(80, 17, 0.f, 640, 640, 1000, false, false, false, st, 3);
        trtx::YoloLayerPluginIOExt io(core);
        void* outs2[1] = {d_out2};
        CHECK(io.enqueue(B, d_in, outs2, d_ws, nullptr) == 0);
        CHECK(cudaDeviceSynchronize() == cudaSuccess);
        std::vector<float> r1((size_t)B * 90001), r2(r1.size());
        cudaMemcpy(r1.data(), d_out, out_bytes, cudaMemcpyDeviceToHost);
        cudaMemcpy(r2.data(), d_out2, out_bytes, cudaMemcpyDeviceToHost);
        for (int b = 0; b < B; ++b) {
            CHECK((int)r1[(size_t)b * 90001] == planted);
            for (int i = 0; i < planted; ++i)
                for (int k = 0; k < 6; ++k) CHECK(r1[(size_t)b * 90001 + 1 + i * 90 + k] == r2[(size_t)b * 90001 + 1 + i * 90 + k]);
            CHECK(r1[(size_t)b * 90001 + 1 + 4] > 0.88f && r1[(size_t)b * 90001 + 1 + 4] < 0.8809f);  // sigmoid(2)
        }
        std::printf("gpu enqueue ok: %d candidates per image through IPluginV2DynamicExt and IPluginV2IOExt\n", planted);
    }
    std::printf("trt adapter check ok\n");
    return 0;
}
