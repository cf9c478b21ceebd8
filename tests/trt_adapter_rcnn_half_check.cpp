// trt_adapter_rcnn_half_check.cpp -- RpnDecodePluginIOExt and PredictorDecodePluginIOExt of include/trtx_plugins.h driven as a
// TensorRT builder / runtime drives plugins: format combinations at every position, output data types, configurePlugin ->
// serialize -> deserialize -> clone with the trailing element type, a blob of the reference's length (what a plan serialized
// with the IPluginV2Ext classes holds) deserializing through the registry as an fp32 plugin, wrong lengths refused, and (with
// --gpu) enqueue through the adapters in both types, and through the IPluginV2Ext classes in fp32, against the direct C calls.  Compiled against tests/mock_trt/NvInfer.h
// with the R-CNN plugins of an FP16 engine registered, and linked with libtrtx_hot.so.
#define TRTX_REGISTER_PLUGINS
#define TRTX_RCNN_HALF_IO_PLUGINS
#include "trtx_plugins.h"

#include <cuda_fp16.h>
#include <cuda_runtime_api.h>

#include <cstdio>
#include <cstdlib>
#include <vector>

#define CHECK(x)                                                                      \
    do {                                                                              \
        if (!(x)) {                                                                   \
            std::fprintf(stderr, "CHECK failed %s:%d: %s\n", __FILE__, __LINE__, #x); \
            std::exit(1);                                                             \
        }                                                                             \
    } while (0)

using namespace nvinfer1;

static const DataType kTypes[] = {DataType::kFLOAT, DataType::kHALF, DataType::kINT8, DataType::kINT32};

static bool fh(DataType t) { return t == DataType::kFLOAT || t == DataType::kHALF; }

static PluginTensorDesc linear(DataType t) {
    PluginTensorDesc d{};
    d.type = t;
    d.format = TensorFormat::kLINEAR;
    return d;
}

template <typename P>
static std::vector<char> blob_of(const P& p) {
    std::vector<char> b(p.getSerializationSize());
    p.serialize(b.data());
    return b;
}

static std::vector<__half> to_half(const std::vector<float>& v) {
    std::vector<__half> h(v.size());
    for (size_t i = 0; i < v.size(); ++i) h[i] = __float2half(v[i]);
    return h;
}

template <typename T>
static T* upload(const std::vector<T>& v) {
    void* d;
    CHECK(cudaMalloc(&d, v.size() * sizeof(T)) == cudaSuccess);
    CHECK(cudaMemcpy(d, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice) == cudaSuccess);
    return static_cast<T*>(d);
}

static std::vector<uint32_t> download(const void* d, size_t n) {
    std::vector<uint32_t> v(n);
    CHECK(cudaMemcpy(v.data(), d, n * 4, cudaMemcpyDeviceToHost) == cudaSuccess);
    return v;
}

int main(int argc, char** argv) {
    const bool gpu = argc > 1 && std::string(argv[1]) == "--gpu";
    const int A = 3, H = 20, W = 27, TOP = 300;
    std::vector<float> anchors;
    for (int a = 0; a < A; ++a) {
        const float s = 16.f * (1 << a);
        anchors.insert(anchors.end(), {-s, -s / 2, s, s / 2});
    }

    // ---- RpnDecode: scores and deltas fp32 | fp16 of one type; scores and boxes fp32 ----
    IPluginCreator* rc = getPluginRegistry()->getPluginCreator("RpnDecode", "1");
    CHECK(rc != nullptr && dynamic_cast<trtx::RpnDecodePluginIOExtCreator*>(rc) != nullptr);
    trtx::RpnDecodePluginIOExt rd(TOP, anchors, 16.f, 320, 432);
    CHECK(std::string(rd.getPluginType()) == "RpnDecode" && std::string(rd.getPluginVersion()) == "1" && rd.getNbOutputs() == 2);
    CHECK(std::string(rd.getPluginNamespace()).empty() && rd.dtype() == TRTX_F32);
    CHECK(rd.getOutputDimensions(0, nullptr, 2).d[0] == TOP && rd.getOutputDimensions(1, nullptr, 2).d[1] == 4);
    for (DataType t0 : kTypes)
        for (DataType t1 : kTypes)
            for (DataType t2 : kTypes) {
                PluginTensorDesc io[4] = {linear(t0), linear(t1), linear(t2), linear(t2)};
                CHECK(rd.supportsFormatCombination(0, io, 2, 2) == fh(t0));
                CHECK(rd.supportsFormatCombination(1, io, 2, 2) == (fh(t1) && t1 == t0));
                CHECK(rd.supportsFormatCombination(2, io, 2, 2) == (t2 == DataType::kFLOAT));
                CHECK(rd.supportsFormatCombination(3, io, 2, 2) == (t2 == DataType::kFLOAT));
                for (PluginTensorDesc& d : io) d.format = TensorFormat::kCHW32;
                for (int pos = 0; pos < 4; ++pos) CHECK(!rd.supportsFormatCombination(pos, io, 2, 2));
            }
    {
        const DataType hh[2] = {DataType::kHALF, DataType::kHALF};
        CHECK(rd.getOutputDataType(0, hh, 2) == DataType::kFLOAT && rd.getOutputDataType(1, hh, 2) == DataType::kFLOAT);
    }
    PluginTensorDesc rio[4] = {linear(DataType::kHALF), linear(DataType::kHALF), linear(DataType::kFLOAT), linear(DataType::kFLOAT)};
    rio[0].dims.nbDims = 3; rio[0].dims.d[0] = A; rio[0].dims.d[1] = H; rio[0].dims.d[2] = W;
    rio[1].dims.nbDims = 3; rio[1].dims.d[0] = 4 * A; rio[1].dims.d[1] = H; rio[1].dims.d[2] = W;
    rd.configurePlugin(rio, 2, rio + 2, 2);
    CHECK(rd.dtype() == TRTX_F16);
    CHECK(rd.getWorkspaceSize(8) == (size_t)trtx_rpn_decode(8, nullptr, nullptr, nullptr, nullptr, H, W, 320, 432, 16.f, anchors.data(),
                                                            A, TOP, nullptr, 0, nullptr));
    const std::vector<char> rb = blob_of(rd);
    const size_t rref = 4 + 8 + 4 * anchors.size() + 4 + 4 * 8;  // RpnDecodePlugin.h:64-75
    CHECK(rb.size() == rref + 4);
    {
        int32_t last;
        std::memcpy(&last, rb.data() + rref, 4);
        CHECK(last == TRTX_F16);
        auto* back = static_cast<trtx::RpnDecodePluginIOExt*>(rc->deserializePlugin("rpn", rb.data(), rb.size()));
        CHECK(back != nullptr && back->dtype() == TRTX_F16 && blob_of(*back) == rb);
        auto* cl = static_cast<trtx::RpnDecodePluginIOExt*>(back->clone());
        CHECK(cl != nullptr && cl != back && cl->dtype() == TRTX_F16 && blob_of(*cl) == rb);
        // the IPluginV2Ext class writes the reference's bytes; through the registry they are an fp32 IOExt plugin
        trtx::RpnDecodePlugin legacy(TOP, anchors, 16.f, H, W, 320, 432);
        const std::vector<char> lb = blob_of(legacy);
        CHECK(lb == std::vector<char>(rb.begin(), rb.begin() + rref));
        IPluginV2* ref = rc->deserializePlugin("rpn", lb.data(), lb.size());
        auto* refx = dynamic_cast<trtx::RpnDecodePluginIOExt*>(ref);
        CHECK(refx != nullptr && refx->dtype() == TRTX_F32);
        const std::vector<char> refb = blob_of(*refx);
        CHECK(refb.size() == rref + 4 && std::memcmp(refb.data(), lb.data(), rref) == 0);
        // any other length, or an element type that does not exist: refused
        CHECK(rc->deserializePlugin("rpn", rb.data(), rref - 1) == nullptr && rc->deserializePlugin("rpn", rb.data(), rref + 1) == nullptr);
        CHECK(rc->deserializePlugin("rpn", rb.data(), rref + 8) == nullptr && rc->deserializePlugin("rpn", rb.data(), 4) == nullptr);
        std::vector<char> bad = rb;
        bad[rref] = 7;
        CHECK(rc->deserializePlugin("rpn", bad.data(), bad.size()) == nullptr);
        std::vector<char> huge = lb;  // an anchor count that does not fit the blob
        const size_t big = (size_t)1 << 62;
        std::memcpy(huge.data() + 4, &big, 8);
        CHECK(rc->deserializePlugin("rpn", huge.data(), huge.size()) == nullptr);
        rio[0].type = rio[1].type = DataType::kFLOAT;
        cl->configurePlugin(rio, 2, rio + 2, 2);
        CHECK(cl->dtype() == TRTX_F32);
        rio[0].type = rio[1].type = DataType::kHALF;
        cl->destroy();
        back->destroy();
        ref->destroy();
    }

    // ---- PredictorDecode: scores and deltas fp32 | fp16 of one type; proposals and the three outputs fp32 ----
    const int N = 100, NC = 8;
    const std::vector<float> w4 = {10.f, 10.f, 5.f, 5.f};
    IPluginCreator* pc = getPluginRegistry()->getPluginCreator("PredictorDecode", "1");
    CHECK(pc != nullptr && dynamic_cast<trtx::PredictorDecodePluginIOExtCreator*>(pc) != nullptr);
    trtx::PredictorDecodePluginIOExt pd(N, 320, 432, w4);
    CHECK(std::string(pd.getPluginType()) == "PredictorDecode" && pd.getNbOutputs() == 3 && pd.dtype() == TRTX_F32);
    CHECK(pd.getOutputDimensions(0, nullptr, 3).d[0] == N && pd.getOutputDimensions(1, nullptr, 3).d[1] == 4);
    for (DataType t0 : kTypes)
        for (DataType t1 : kTypes)
            for (DataType t2 : kTypes)
                for (DataType t3 : kTypes) {
                    PluginTensorDesc io[6] = {linear(t0), linear(t1), linear(t2), linear(t3), linear(t3), linear(t3)};
                    CHECK(pd.supportsFormatCombination(0, io, 3, 3) == fh(t0));
                    CHECK(pd.supportsFormatCombination(1, io, 3, 3) == (fh(t1) && t1 == t0));
                    CHECK(pd.supportsFormatCombination(2, io, 3, 3) == (t2 == DataType::kFLOAT));
                    for (int pos = 3; pos < 6; ++pos) CHECK(pd.supportsFormatCombination(pos, io, 3, 3) == (t3 == DataType::kFLOAT));
                    for (PluginTensorDesc& d : io) d.format = TensorFormat::kCHW32;
                    for (int pos = 0; pos < 6; ++pos) CHECK(!pd.supportsFormatCombination(pos, io, 3, 3));
                }
    {
        const DataType hhf[3] = {DataType::kHALF, DataType::kHALF, DataType::kFLOAT};
        for (int i = 0; i < 3; ++i) CHECK(pd.getOutputDataType(i, hhf, 3) == DataType::kFLOAT);
    }
    PluginTensorDesc pio[6] = {linear(DataType::kHALF), linear(DataType::kHALF), linear(DataType::kFLOAT),
                               linear(DataType::kFLOAT), linear(DataType::kFLOAT), linear(DataType::kFLOAT)};
    pio[0].dims.nbDims = 4; pio[0].dims.d[0] = N; pio[0].dims.d[1] = NC; pio[0].dims.d[2] = 1; pio[0].dims.d[3] = 1;
    pd.configurePlugin(pio, 3, pio + 3, 3);
    CHECK(pd.dtype() == TRTX_F16);
    const std::vector<char> pb = blob_of(pd);
    const size_t pref = 4 * 4 + 8 + 4 * 4;  // PredictorDecodePlugin.h:62-70
    CHECK(pb.size() == pref + 4);
    {
        unsigned classes;
        std::memcpy(&classes, pb.data() + 4, 4);
        CHECK(classes == (unsigned)NC);  // configurePlugin kept the reference's dimension read
        auto* back = static_cast<trtx::PredictorDecodePluginIOExt*>(pc->deserializePlugin("pred", pb.data(), pb.size()));
        CHECK(back != nullptr && back->dtype() == TRTX_F16 && blob_of(*back) == pb);
        auto* cl = static_cast<trtx::PredictorDecodePluginIOExt*>(back->clone());
        CHECK(cl != nullptr && cl->dtype() == TRTX_F16 && blob_of(*cl) == pb);
        trtx::PredictorDecodePlugin legacy(N, NC, 320, 432, w4);
        const std::vector<char> lb = blob_of(legacy);
        CHECK(lb == std::vector<char>(pb.begin(), pb.begin() + pref));
        IPluginV2* ref = pc->deserializePlugin("pred", lb.data(), lb.size());
        auto* refx = dynamic_cast<trtx::PredictorDecodePluginIOExt*>(ref);
        CHECK(refx != nullptr && refx->dtype() == TRTX_F32);
        CHECK(std::memcmp(blob_of(*refx).data(), lb.data(), pref) == 0);
        CHECK(pc->deserializePlugin("pred", pb.data(), pref - 1) == nullptr && pc->deserializePlugin("pred", pb.data(), pref + 2) == nullptr);
        CHECK(pc->deserializePlugin("pred", pb.data(), 12) == nullptr);
        std::vector<char> bad = pb;
        bad[pref] = 2;
        CHECK(pc->deserializePlugin("pred", bad.data(), bad.size()) == nullptr);
        cl->destroy();
        back->destroy();
        ref->destroy();
    }

    if (gpu) {
        const int B = 2;
        unsigned seed = 777u;
        auto rnd = [&]() {  // uniform in [-1, 1)
            seed = seed * 1664525u + 1013904223u;
            return (float)(seed >> 8) / 8388608.0f - 1.0f;
        };
        void* ws;
        CHECK(cudaMalloc(&ws, 4096) == cudaSuccess);
        // ---- RpnDecode through the adapter == trtx_rpn_decode_typed, halves and floats
        const int n = A * H * W;
        std::vector<float> sc((size_t)B * n), dl((size_t)B * n * 4);
        for (float& v : sc) v = rnd() * 4.f;
        for (float& v : dl) v = rnd() * 0.5f;
        const void* s32 = upload(sc);
        const void* d32 = upload(dl);
        const void* s16 = upload(to_half(sc));
        const void* d16 = upload(to_half(dl));
        void *o1, *o2, *r1, *r2;
        CHECK(cudaMalloc(&o1, B * TOP * 4) == cudaSuccess && cudaMalloc(&o2, B * TOP * 16) == cudaSuccess);
        CHECK(cudaMalloc(&r1, B * TOP * 4) == cudaSuccess && cudaMalloc(&r2, B * TOP * 16) == cudaSuccess);
        for (int half = 1; half >= 0; --half) {
            rio[0].type = rio[1].type = half ? DataType::kHALF : DataType::kFLOAT;
            rd.configurePlugin(rio, 2, rio + 2, 2);
            const void* ins[2] = {half ? s16 : s32, half ? d16 : d32};
            void* outs[2] = {o1, o2};
            CHECK(cudaMemset(o1, 0x11, B * TOP * 4) == cudaSuccess && cudaMemset(r1, 0x22, B * TOP * 4) == cudaSuccess);
            CHECK(rd.enqueue(B, ins, outs, ws, nullptr) == 0);
            CHECK(trtx_rpn_decode_typed(half ? TRTX_F16 : TRTX_F32, B, ins[0], ins[1], static_cast<float*>(r1), static_cast<float*>(r2), H, W,
                                        320, 432, 16.f, anchors.data(), A, TOP, ws, 4096, nullptr) == 0);
            CHECK(cudaDeviceSynchronize() == cudaSuccess);
            CHECK(download(o1, B * TOP) == download(r1, B * TOP) && download(o2, B * TOP * 4) == download(r2, B * TOP * 4));
        }
        {  // the IPluginV2Ext class configured with the same dims == the fp32 call
            trtx::RpnDecodePlugin legacy(TOP, anchors, 16.f, 320, 432);
            const Dims dims[2] = {rio[0].dims, rio[1].dims};
            legacy.configurePlugin(dims, 2, nullptr, 2, nullptr, nullptr, nullptr, nullptr, PluginFormat::kLINEAR, B);
            const void* ins[2] = {s32, d32};
            void* outs[2] = {o1, o2};
            CHECK(cudaMemset(o1, 0x11, B * TOP * 4) == cudaSuccess && cudaMemset(o2, 0x11, B * TOP * 16) == cudaSuccess);
            CHECK(legacy.enqueue(B, ins, outs, ws, nullptr) == 0);
            CHECK(cudaDeviceSynchronize() == cudaSuccess);
            CHECK(download(o1, B * TOP) == download(r1, B * TOP) && download(o2, B * TOP * 4) == download(r2, B * TOP * 4));
        }
        // ---- PredictorDecode through the adapter == trtx_predictor_decode_typed
        std::vector<float> ps((size_t)B * N * NC), pdl((size_t)B * N * NC * 4), props((size_t)B * N * 4);
        for (float& v : ps) v = (rnd() + 1.f) * 0.5f;
        for (float& v : pdl) v = rnd();
        for (int i = 0; i < B * N; ++i) {
            const float x = (rnd() + 1.f) * 150.f, y = (rnd() + 1.f) * 100.f;
            props[4 * i] = x, props[4 * i + 1] = y, props[4 * i + 2] = x + 20.f + (rnd() + 1.f) * 60.f, props[4 * i + 3] = y + 20.f + (rnd() + 1.f) * 50.f;
        }
        const void* p32 = upload(ps);
        const void* q32 = upload(pdl);
        const void* p16 = upload(to_half(ps));
        const void* q16 = upload(to_half(pdl));
        const float* dprops = upload(props);
        void *a[3], *b[3];
        for (int k = 0; k < 3; ++k) CHECK(cudaMalloc(&a[k], B * N * 16) == cudaSuccess && cudaMalloc(&b[k], B * N * 16) == cudaSuccess);
        for (int half = 1; half >= 0; --half) {
            pio[0].type = pio[1].type = half ? DataType::kHALF : DataType::kFLOAT;
            pd.configurePlugin(pio, 3, pio + 3, 3);
            const void* ins[3] = {half ? p16 : p32, half ? q16 : q32, dprops};
            void* outs[3] = {a[0], a[1], a[2]};
            for (int k = 0; k < 3; ++k) CHECK(cudaMemset(a[k], 0x11, B * N * 16) == cudaSuccess && cudaMemset(b[k], 0x22, B * N * 16) == cudaSuccess);
            CHECK(pd.enqueue(B, ins, outs, ws, nullptr) == 0);
            CHECK(trtx_predictor_decode_typed(half ? TRTX_F16 : TRTX_F32, B, ins[0], ins[1], dprops, static_cast<float*>(b[0]),
                                              static_cast<float*>(b[1]), static_cast<float*>(b[2]), N, NC, 320, 432, w4.data(), ws, 4096,
                                              nullptr) == 0);
            CHECK(cudaDeviceSynchronize() == cudaSuccess);
            CHECK(download(a[0], B * N) == download(b[0], B * N) && download(a[1], B * N * 4) == download(b[1], B * N * 4));
            CHECK(download(a[2], B * N) == download(b[2], B * N));
        }
        {  // the IPluginV2Ext class configured with the same dims == the fp32 call
            trtx::PredictorDecodePlugin legacy(N, 320, 432, w4);
            const Dims dims[3] = {pio[0].dims, pio[1].dims, pio[2].dims};
            legacy.configurePlugin(dims, 3, nullptr, 3, nullptr, nullptr, nullptr, nullptr, PluginFormat::kLINEAR, B);
            const void* ins[3] = {p32, q32, dprops};
            void* outs[3] = {a[0], a[1], a[2]};
            for (int k = 0; k < 3; ++k) CHECK(cudaMemset(a[k], 0x11, B * N * 16) == cudaSuccess);
            CHECK(legacy.enqueue(B, ins, outs, ws, nullptr) == 0);
            CHECK(cudaDeviceSynchronize() == cudaSuccess);
            for (int k = 0; k < 3; ++k) CHECK(download(a[k], B * N * (k == 1 ? 4 : 1)) == download(b[k], B * N * (k == 1 ? 4 : 1)));
        }
        std::printf("gpu rcnn half enqueue ok\n");
    }
    std::printf("trt adapter rcnn half check ok\n");
    return 0;
}
