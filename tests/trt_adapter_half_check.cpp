// trt_adapter_half_check.cpp -- the half-accepting adapters of include/trtx_plugins.h (DecodePluginDynamic,
// RoiAlignPluginIOExt, MaskRcnnInferencePluginIOExt) driven as a TensorRT builder / runtime drives plugins: format
// combinations at every position, output data types, configurePlugin -> serialize -> deserialize -> clone, and (with --gpu)
// enqueue through the adapter, and through the IPluginV2Ext RoiAlign / MaskRcnnInference classes in fp32, against the direct C
// call.  Compiled against tests/mock_trt/NvInfer.h (this image has no
// TensorRT) with the half-accepting rcnn creators registered, and linked with libtrtx_hot.so.
#define TRTX_REGISTER_PLUGINS
#define TRTX_RCNN_HALF_IO_PLUGINS
#include "trtx_plugins.h"

#include <cuda_fp16.h>
#include <cuda_runtime_api.h>

#include <cstdio>
#include <cstdlib>
#include <vector>

#define CHECK(x)                                                          \
    do {                                                                  \
        if (!(x)) {                                                       \
            std::fprintf(stderr, "CHECK failed %s:%d: %s\n", __FILE__, __LINE__, #x); \
            std::exit(1);                                                 \
        }                                                                 \
    } while (0)

using namespace nvinfer1;

static const DataType kTypes[] = {DataType::kFLOAT, DataType::kHALF, DataType::kINT8, DataType::kINT32};

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

template <typename T>
static std::vector<T> download(const void* d, size_t n) {
    std::vector<T> v(n);
    CHECK(cudaMemcpy(v.data(), d, n * sizeof(T), cudaMemcpyDeviceToHost) == cudaSuccess);
    return v;
}

int main(int argc, char** argv) {
    const bool gpu = argc > 1 && std::string(argv[1]) == "--gpu";

    // ---- Decode_TRT: the three heads all fp32 or all fp16, rows fp32 ----
    IPluginCreator* dc = getPluginRegistry()->getPluginCreator("Decode_TRT", "1");
    CHECK(dc != nullptr);
    PluginFieldCollection none{0, nullptr};
    auto* dec = static_cast<IPluginV2DynamicExt*>(dc->createPlugin("decode", &none));
    CHECK(dec != nullptr);
    for (DataType t0 : kTypes)
        for (DataType t : kTypes) {
            PluginTensorDesc io[4] = {linear(t0), linear(t), linear(t), linear(t)};
            const bool head_ok = (t0 == DataType::kFLOAT || t0 == DataType::kHALF);
            CHECK(dec->supportsFormatCombination(0, io, 3, 1) == head_ok);
            CHECK(dec->supportsFormatCombination(1, io, 3, 1) == (head_ok && t == t0));
            CHECK(dec->supportsFormatCombination(2, io, 3, 1) == (head_ok && t == t0));
            CHECK(dec->supportsFormatCombination(3, io, 3, 1) == (t == DataType::kFLOAT));
            io[1].format = io[3].format = TensorFormat::kCHW32;
            CHECK(!dec->supportsFormatCombination(1, io, 3, 1) && !dec->supportsFormatCombination(3, io, 3, 1));
        }
    {
        const DataType halves[3] = {DataType::kHALF, DataType::kHALF, DataType::kHALF};
        CHECK(dec->getOutputDataType(0, halves, 3) == DataType::kFLOAT);
        CHECK(dec->getSerializationSize() == 8);  // the element type is per call (the tensor descriptors), not plugin state
    }

    // ---- RoiAlign: proposals fp32, features fp32 | fp16, bins in the features' type ----
    CHECK(getPluginRegistry()->getPluginCreator("RoiAlign", "1") != nullptr);
    trtx::RoiAlignPluginIOExt ra(14, 1.f / 16, 2, 24, 16);
    CHECK(std::string(ra.getPluginType()) == "RoiAlign" && std::string(ra.getPluginVersion()) == "1" && ra.getNbOutputs() == 1);
    CHECK(ra.getOutputDimensions(0, nullptr, 2).d[1] == 16 && ra.getWorkspaceSize(8) == 0 && ra.dtype() == TRTX_F32);
    for (DataType t0 : kTypes)
        for (DataType t1 : kTypes)
            for (DataType t2 : kTypes) {
                PluginTensorDesc io[3] = {linear(t0), linear(t1), linear(t2)};
                CHECK(ra.supportsFormatCombination(0, io, 2, 1) == (t0 == DataType::kFLOAT));
                CHECK(ra.supportsFormatCombination(1, io, 2, 1) == (t1 == DataType::kFLOAT || t1 == DataType::kHALF));
                CHECK(ra.supportsFormatCombination(2, io, 2, 1) == (t2 == t1));
                io[0].format = io[1].format = io[2].format = TensorFormat::kCHW32;
                for (int pos = 0; pos < 3; ++pos) CHECK(!ra.supportsFormatCombination(pos, io, 2, 1));
            }
    {
        const DataType fh[2] = {DataType::kFLOAT, DataType::kHALF}, ff[2] = {DataType::kFLOAT, DataType::kFLOAT};
        CHECK(ra.getOutputDataType(0, fh, 2) == DataType::kHALF && ra.getOutputDataType(0, ff, 2) == DataType::kFLOAT);
    }
    const int N = 24, C = 16, H = 20, W = 27;
    PluginTensorDesc rio[3] = {linear(DataType::kFLOAT), linear(DataType::kHALF), linear(DataType::kHALF)};
    rio[0].dims.nbDims = 2; rio[0].dims.d[0] = N; rio[0].dims.d[1] = 4;
    rio[1].dims.nbDims = 3; rio[1].dims.d[0] = C; rio[1].dims.d[1] = H; rio[1].dims.d[2] = W;
    ra.configurePlugin(rio, 2, rio + 2, 1);
    CHECK(ra.dtype() == TRTX_F16);
    const std::vector<char> rab = blob_of(ra);
    CHECK(rab.size() == 28 + 4);  // the reference's seven fields (RoiAlignPlugin.h:53-61) + the element type
    {
        int32_t last;
        std::memcpy(&last, rab.data() + 28, 4);
        CHECK(last == TRTX_F16);
        trtx::RoiAlignPluginIOExtCreator rc;
        auto* back = static_cast<trtx::RoiAlignPluginIOExt*>(rc.deserializePlugin("roi", rab.data(), rab.size()));
        CHECK(back != nullptr && back->dtype() == TRTX_F16 && blob_of(*back) == rab);
        auto* cl = static_cast<trtx::RoiAlignPluginIOExt*>(back->clone());
        CHECK(cl != nullptr && cl != back && cl->dtype() == TRTX_F16 && blob_of(*cl) == rab);
        // a blob of the reference's length is an fp32 plugin with the same seven fields
        auto* ref = static_cast<trtx::RoiAlignPluginIOExt*>(rc.deserializePlugin("roi", rab.data(), 28));
        CHECK(ref != nullptr && ref->dtype() == TRTX_F32);
        const std::vector<char> refb = blob_of(*ref);
        CHECK(refb.size() == 32 && std::memcmp(refb.data(), rab.data(), 28) == 0);
        trtx::RoiAlignPlugin legacy(14, 1.f / 16, 2, N, C, H, W);  // the IPluginV2Ext class writes those 28 bytes
        CHECK(blob_of(legacy) == std::vector<char>(rab.begin(), rab.begin() + 28));
        // neither length, or an element type that does not exist: refused
        CHECK(rc.deserializePlugin("roi", rab.data(), 27) == nullptr && rc.deserializePlugin("roi", rab.data(), 3) == nullptr);
        std::vector<char> bad = rab;
        bad[28] = 7;
        CHECK(rc.deserializePlugin("roi", bad.data(), bad.size()) == nullptr);
        // configurePlugin with fp32 features turns the clone back into an fp32 plugin
        rio[1].type = rio[2].type = DataType::kFLOAT;
        cl->configurePlugin(rio, 2, rio + 2, 1);
        CHECK(cl->dtype() == TRTX_F32);
        rio[1].type = rio[2].type = DataType::kHALF;
        cl->destroy();
        back->destroy();
        ref->destroy();
    }

    // ---- MaskRcnnInference: indices fp32, masks fp32 | fp16, probabilities fp32 ----
    CHECK(getPluginRegistry()->getPluginCreator("MaskRcnnInference", "1") != nullptr);
    const int D = 10, NC = 5, S = 14;
    trtx::MaskRcnnInferencePluginIOExt mi(D, S);
    CHECK(std::string(mi.getPluginType()) == "MaskRcnnInference" && mi.getOutputDimensions(0, nullptr, 2).d[0] == D);
    for (DataType t0 : kTypes)
        for (DataType t1 : kTypes)
            for (DataType t2 : kTypes) {
                PluginTensorDesc io[3] = {linear(t0), linear(t1), linear(t2)};
                CHECK(mi.supportsFormatCombination(0, io, 2, 1) == (t0 == DataType::kFLOAT));
                CHECK(mi.supportsFormatCombination(1, io, 2, 1) == (t1 == DataType::kFLOAT || t1 == DataType::kHALF));
                CHECK(mi.supportsFormatCombination(2, io, 2, 1) == (t2 == DataType::kFLOAT));
            }
    {
        const DataType fh[2] = {DataType::kFLOAT, DataType::kHALF};
        CHECK(mi.getOutputDataType(0, fh, 2) == DataType::kFLOAT);
    }
    PluginTensorDesc mio[3] = {linear(DataType::kFLOAT), linear(DataType::kHALF), linear(DataType::kFLOAT)};
    mio[1].dims.nbDims = 4; mio[1].dims.d[0] = D; mio[1].dims.d[1] = NC; mio[1].dims.d[2] = S; mio[1].dims.d[3] = S;
    mi.configurePlugin(mio, 2, mio + 2, 1);
    CHECK(mi.dtype() == TRTX_F16);
    const std::vector<char> mib = blob_of(mi);
    CHECK(mib.size() == 12 + 4);
    {
        trtx::MaskRcnnInferencePluginIOExtCreator mc;
        auto* back = static_cast<trtx::MaskRcnnInferencePluginIOExt*>(mc.deserializePlugin("mask", mib.data(), mib.size()));
        CHECK(back != nullptr && back->dtype() == TRTX_F16 && blob_of(*back) == mib);
        auto* cl = static_cast<trtx::MaskRcnnInferencePluginIOExt*>(back->clone());
        CHECK(cl->dtype() == TRTX_F16 && blob_of(*cl) == mib);
        auto* ref = static_cast<trtx::MaskRcnnInferencePluginIOExt*>(mc.deserializePlugin("mask", mib.data(), 12));
        CHECK(ref != nullptr && ref->dtype() == TRTX_F32);
        trtx::MaskRcnnInferencePlugin legacy(D, S, NC);
        CHECK(blob_of(legacy) == std::vector<char>(mib.begin(), mib.begin() + 12));
        CHECK(mc.deserializePlugin("mask", mib.data(), 13) == nullptr);
        cl->destroy();
        back->destroy();
        ref->destroy();
    }

    if (gpu) {
        const int B = 2;
        unsigned seed = 12345u;
        auto rnd = [&]() {  // uniform in [-1, 1)
            seed = seed * 1664525u + 1013904223u;
            return (float)(seed >> 8) / 8388608.0f - 1.0f;
        };
        // ---- RoiAlign: half features through the adapter == trtx_roi_align_typed(TRTX_F16), and the fp32 adapter == trtx_roi_align
        std::vector<float> feat((size_t)B * C * H * W), rois((size_t)B * N * 4);
        for (float& v : feat) v = rnd() * 3.f;
        for (int i = 0; i < B * N; ++i) {
            const float x = (rnd() + 1.f) * 150.f, y = (rnd() + 1.f) * 100.f;
            rois[4 * i] = x, rois[4 * i + 1] = y, rois[4 * i + 2] = x + 16.f + (rnd() + 1.f) * 120.f, rois[4 * i + 3] = y + 16.f + (rnd() + 1.f) * 90.f;
        }
        const size_t nout = (size_t)B * N * C * 14 * 14;
        float* d_rois = upload(rois);
        float* d_feat = upload(feat);
        __half* d_feat_h = upload(to_half(feat));
        void *d_a, *d_b;
        CHECK(cudaMalloc(&d_a, nout * 4) == cudaSuccess && cudaMalloc(&d_b, nout * 4) == cudaSuccess);
        {
            const void* ins[2] = {d_rois, d_feat_h};
            void* outs[1] = {d_a};
            CHECK(cudaMemset(d_a, 0x11, nout * 4) == cudaSuccess && cudaMemset(d_b, 0x22, nout * 4) == cudaSuccess);
            CHECK(ra.enqueue(B, ins, outs, nullptr, nullptr) == 0);
            CHECK(trtx_roi_align_typed(TRTX_F16, B, d_rois, d_feat_h, d_b, 14, 1.f / 16, 2, N, C, H, W, nullptr) == 0);
            CHECK(cudaDeviceSynchronize() == cudaSuccess);
            CHECK(download<uint16_t>(d_a, nout) == download<uint16_t>(d_b, nout));
            rio[1].type = rio[2].type = DataType::kFLOAT;
            ra.configurePlugin(rio, 2, rio + 2, 1);
            ins[1] = d_feat;
            CHECK(ra.enqueue(B, ins, outs, nullptr, nullptr) == 0);
            CHECK(trtx_roi_align(B, d_rois, d_feat, static_cast<float*>(d_b), 14, 1.f / 16, 2, N, C, H, W, nullptr) == 0);
            CHECK(cudaDeviceSynchronize() == cudaSuccess);
            CHECK(download<uint32_t>(d_a, nout) == download<uint32_t>(d_b, nout));
            trtx::RoiAlignPlugin legacy(14, 1.f / 16, 2, N, C, H, W);  // the IPluginV2Ext class == the fp32 call
            CHECK(cudaMemset(d_a, 0x11, nout * 4) == cudaSuccess);
            CHECK(legacy.enqueue(B, ins, outs, nullptr, nullptr) == 0);
            CHECK(cudaDeviceSynchronize() == cudaSuccess);
            CHECK(download<uint32_t>(d_a, nout) == download<uint32_t>(d_b, nout));
        }
        // ---- MaskRcnnInference: half masks through the adapter == the typed C call
        std::vector<float> masks((size_t)B * D * NC * S * S), idx((size_t)B * D);
        for (float& v : masks) v = rnd() * 6.f;
        for (size_t i = 0; i < idx.size(); ++i) idx[i] = (float)(i % NC);
        idx[3] = -1.f;
        float* d_idx = upload(idx);
        __half* d_masks_h = upload(to_half(masks));
        const size_t mout = (size_t)B * D * S * S;
        {
            const void* ins[2] = {d_idx, d_masks_h};
            void* outs[1] = {d_a};
            CHECK(cudaMemset(d_a, 0x11, mout * 4) == cudaSuccess && cudaMemset(d_b, 0x11, mout * 4) == cudaSuccess);
            CHECK(mi.enqueue(B, ins, outs, nullptr, nullptr) == 0);
            CHECK(trtx_mask_rcnn_inference_typed(TRTX_F16, B, d_idx, d_masks_h, static_cast<float*>(d_b), D, S, NC, nullptr) == 0);
            CHECK(cudaDeviceSynchronize() == cudaSuccess);
            const std::vector<uint32_t> r = download<uint32_t>(d_a, mout);
            CHECK(r == download<uint32_t>(d_b, mout));
            CHECK(r[3 * S * S] == 0x11111111u && r[0] != 0x11111111u);  // the row of index -1 stays untouched
            trtx::MaskRcnnInferencePlugin legacy(D, S, NC);  // the IPluginV2Ext class == the fp32 call
            ins[1] = upload(masks);
            CHECK(cudaMemset(d_a, 0x11, mout * 4) == cudaSuccess && cudaMemset(d_b, 0x11, mout * 4) == cudaSuccess);
            CHECK(legacy.enqueue(B, ins, outs, nullptr, nullptr) == 0);
            CHECK(trtx_mask_rcnn_inference(B, d_idx, static_cast<const float*>(ins[1]), static_cast<float*>(d_b), D, S, NC, nullptr) == 0);
            CHECK(cudaDeviceSynchronize() == cudaSuccess);
            CHECK(download<uint32_t>(d_a, mout) == download<uint32_t>(d_b, mout));
        }
        // ---- Decode_TRT: half heads through the adapter == trtx_retina_decode_enqueue with in_dtype = TRTX_F16
        trtx_retina_params rp{};
        rp.in_h = 480, rp.in_w = 640, rp.gate = 0.02f, rp.in_dtype = TRTX_F16;
        PluginTensorDesc dio[4];
        const void* heads[3];
        for (int l = 0; l < 3; ++l) {
            const int g = (480 >> (3 + l)) * (640 >> (3 + l));
            std::vector<float> h((size_t)B * 32 * g);
            for (float& v : h) v = rnd();
            for (int b = 0; b < B; ++b)
                for (int e = l; e < g; e += 53) h[((size_t)b * 32 + 9) * g + e] = 4.f;  // a face every 53 cells (prior 0)
            heads[l] = upload(to_half(h));
            dio[l] = linear(DataType::kHALF);
            dio[l].dims.nbDims = 3; dio[l].dims.d[0] = B; dio[l].dims.d[1] = 32; dio[l].dims.d[2] = g;
        }
        dio[3] = linear(DataType::kFLOAT);
        const size_t row = 1 + (size_t)trtx_retina_total_priors(&rp) * 15;
        void *d_r1, *d_r2, *d_ws;
        const size_t ws = dec->getWorkspaceSize(dio, 3, dio + 3, 1);
        CHECK(ws == trtx_retina_workspace_size(&rp, B));
        CHECK(cudaMalloc(&d_r1, B * row * 4) == cudaSuccess && cudaMalloc(&d_r2, B * row * 4) == cudaSuccess && cudaMalloc(&d_ws, ws) == cudaSuccess);
        CHECK(cudaMemset(d_r1, 0, B * row * 4) == cudaSuccess && cudaMemset(d_r2, 0, B * row * 4) == cudaSuccess);
        void* outs[1] = {d_r1};
        CHECK(dec->enqueue(dio, dio + 3, heads, outs, d_ws, nullptr) == 0);
        CHECK(trtx_retina_decode_enqueue(&rp, B, heads, static_cast<float*>(d_r2), d_ws, ws, nullptr) == 0);
        CHECK(cudaDeviceSynchronize() == cudaSuccess);
        const std::vector<float> r1 = download<float>(d_r1, B * row), r2 = download<float>(d_r2, B * row);
        int faces = 0;
        for (int b = 0; b < B; ++b) {
            const int n = (int)r1[b * row];
            CHECK(n > 0 && n == (int)r2[b * row]);
            CHECK(std::memcmp(&r1[b * row], &r2[b * row], (1 + (size_t)n * 15) * 4) == 0);
            faces += n;
        }
        std::printf("gpu half enqueue ok: %d faces through DecodePluginDynamic with half heads\n", faces);
    }
    std::printf("trt adapter half check ok\n");
    return 0;
}
